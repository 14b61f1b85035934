// tf32 tensor-core weight gradient for sm_90a:  dW(tap, k, n) += sum_m pro(A[in_row(m, tap), k]) * prod(D[m, n])   (gemm_args.h, wgrad form)
//
// The reduction runs over the rows m, while wgmma reads tf32 operands from shared memory only K-major, so both operands are transposed on
// their way into shared memory: a stage holds 32 rows as A^T (64 k x 32 m) and D^T (N x 32 m), every line of 32 m-values one 128-byte
// SWIZZLE_128B row.  One warpgroup per CTA: it stores the next stage (LDG, prologue / dropout scale applied, rounded to tf32) while the MMAs
// of the current one run (wgmma m64n16k8, 4 K-steps per stage, N / 16 instructions per step), then adds its 64 x N tile into dW with
// atomics (the parameter-gradient buffer is zeroed once per step).  Grid: (taps x k tiles, row chunks).  The bias gradient is a
// separate column-sum pass.
#include "common.cuh"
#include "../../include/cmgan_b200.h"
#include "gemm_device.cuh"
#include "tc_ptx.cuh"

namespace {
using namespace cmgan_gemm;
using namespace cmgan_tc;

constexpr int WT = 128;              // one warpgroup
constexpr int RS = 32;               // rows per stage = one 128-byte line of m-values
constexpr int KT = 64;               // k values per tile = wgmma M
constexpr int A_BYTES = KT * 128;    // 8 KB

// byte offset of (line, m) in a K-major SWIZZLE_128B tile of 32-float lines
__device__ __forceinline__ uint32_t swz(int line, int m) { return (uint32_t)(line * 128 + ((((m >> 2) ^ line) & 7) << 4) + (m & 3) * 4); }

template <int NBMAX>
__global__ void __launch_bounds__(WT) gemm_wgrad_tc_kernel(const __grid_constant__ CmganGemmArgs g, int mch) {
    extern __shared__ uint8_t smem_raw[];
    const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;
    uint8_t* const bptr = smem_raw + (base - smem_u32(smem_raw));
    const int N = g.N, nb = N / 16;
    const uint32_t stage_bytes = (uint32_t)(A_BYTES + N * 128);
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int ktiles = (g.Cin + KT - 1) / KT;
    const int tap = blockIdx.x / ktiles, k0 = (blockIdx.x % ktiles) * KT;
    const long mbeg = (long)blockIdx.y * mch;
    const long mend = mbeg + mch < g.M ? mbeg + mch : g.M;
    const unsigned long long seed = eff_seed(g);
    // loader lanes: row m = (tid & 7) + 8 i, 4 consecutive columns (k or n) at 4 (tid >> 3) + 64 j -- 2-way bank conflicts on the transposed stores
    const int lm = tid & 7, lq = (tid >> 3) * 4;

    auto load_stage = [&](long mb, int buf) {
        uint8_t* sa = bptr + buf * stage_bytes;
        uint8_t* sd = sa + A_BYTES;
#pragma unroll
        for (int i = 0; i < RS / 8; ++i) {
            const int ml = lm + 8 * i;
            const long m = mb + ml;
            RowInfo ri = decode_row(g, (int)(m < mend ? m : g.M));
            if (m >= mend) ri.ok = false;
            float a[4];
            load_a4<4>(g, in_row_of(g, ri, tap), tap, k0 + lq, a);
#pragma unroll
            for (int j = 0; j < 4; ++j) *reinterpret_cast<float*>(sa + swz(lq + j, ml)) = to_tf32(a[j]);
            for (int n = lq; n < N; n += 64) {
                float4 d = make_float4(0.f, 0.f, 0.f, 0.f);
                if (m < mend) d = __ldg(reinterpret_cast<const float4*>(g.D + m * g.ldd + n));
                float dv[4] = {d.x, d.y, d.z, d.w};
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    if (g.prod == 1 && m < mend) dv[j] *= g.alpha * cmgan_drop_scale(seed, (uint64_t)m * N + n + j, g.drop_thr, g.inv_keep);
                    *reinterpret_cast<float*>(sd + swz(n + j, ml)) = to_tf32(dv[j]);
                }
            }
        }
        fence_proxy_async();          // generic-proxy stores -> visible to the tensor core's async proxy
    };

    float acc[NBMAX][8];
#pragma unroll
    for (int j = 0; j < NBMAX; ++j)
#pragma unroll
        for (int i = 0; i < 8; ++i) acc[j][i] = 0.f;
    const int nst = (int)((mend - mbeg + RS - 1) / RS);
    if (nst > 0) load_stage(mbeg, 0);
    __syncthreads();
    for (int st = 0; st < nst; ++st) {
        const uint32_t sa = base + (st & 1) * stage_bytes;
        wgmma_fence();
        mma_chunk_n<NBMAX>(nb, acc, gmma_desc_sw128(sa), gmma_desc_sw128(sa + A_BYTES), st == 0);
        wgmma_commit();
        if (st + 1 < nst) load_stage(mbeg + (long)(st + 1) * RS, (st + 1) & 1);     // the other buffer: its MMAs retired last iteration
        wgmma_wait<0>();
        __syncthreads();
    }
    if (nst == 0) return;
    // fragment of warp w: k = k0 + 16 w + lane / 4 (+ 8), n = 16 j + 8 i + 2 (lane % 4) (+ 1)
    const int kr = k0 + 16 * warp + (lane >> 2), nc = 2 * (lane & 3);
    float* const dst = g.C + (long)tap * g.sb_tap;
#pragma unroll
    for (int j = 0; j < NBMAX; ++j) {
        if (j >= nb) break;
#pragma unroll
        for (int i = 0; i < 2; ++i)
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int k = kr + 8 * h;
                if (k >= g.Cin) continue;
                const int n = 16 * j + 8 * i + nc;
                atomicAdd(dst + (long)k * g.sb_k + (long)n * g.sb_n, acc[j][4 * i + 2 * h]);
                atomicAdd(dst + (long)k * g.sb_k + (long)(n + 1) * g.sb_n, acc[j][4 * i + 2 * h + 1]);
            }
    }
}

// dbias[n] += sum_m prod(D[m, n])
__global__ void colsum_kernel(const float* __restrict__ D, long ldd, long M, int N, int prod, float alpha, unsigned long long seed, unsigned thr,
                              float inv_keep, int rows_per_block, float* __restrict__ out, const unsigned long long* __restrict__ seed_dev) {
    seed = cmgan_eff_seed(seed, seed_dev);
    __shared__ float sm[256];
    const int c = threadIdx.x % N, rg = threadIdx.x / N, nrg = blockDim.x / N;
    const long r_beg = (long)blockIdx.x * rows_per_block;
    const long r_end = r_beg + rows_per_block < M ? r_beg + rows_per_block : M;
    float s = 0.f;
    if (rg < nrg)
        for (long m = r_beg + rg; m < r_end; m += nrg) {
            float d = __ldg(D + m * ldd + c);
            if (prod == 1) d *= alpha * cmgan_drop_scale(seed, (uint64_t)m * N + c, thr, inv_keep);
            s += d;
        }
    sm[threadIdx.x] = s;
    __syncthreads();
    if (threadIdx.x < N) {
        float t = 0.f;
        for (int q = 0; q < nrg; ++q) t += sm[q * N + c];
        atomicAdd(out + c, t);
    }
}

int wgrad_tc_supported(const CmganGemmArgs* a) {
    if (a->N % 16 || a->N < 16 || a->N > 256) return 0;
    if (a->Cin % 4 || a->lda % 4 || ((uintptr_t)a->A & 15) || a->ldd % 4 || ((uintptr_t)a->D & 15)) return 0;
    for (int t = 0; t < a->ntaps; ++t)
        if (a->tap_off[t] % 4) return 0;
    return 1;
}

template <int NBMAX>
int launch(const CmganGemmArgs* a, dim3 grid, size_t smem, int mch, cudaStream_t st) {
    static bool attr_set = false;
    if (!attr_set) {
        cudaError_t e = cudaFuncSetAttribute(gemm_wgrad_tc_kernel<NBMAX>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(96 * 1024));
        if (e != cudaSuccess) { cmgan_set_error("gemm_wgrad_tc: cudaFuncSetAttribute: %s", cudaGetErrorString(e)); return -1; }
        attr_set = true;
    }
    gemm_wgrad_tc_kernel<NBMAX><<<grid, WT, smem, st>>>(*a, mch);
    return cmgan_check_launch("gemm_wgrad_tc_kernel");
}

}  // namespace

// tf32 tensor-core path of cmgan_gemm_wgrad (same contract).  Returns 1 if the shape is not covered (caller runs the fp32 kernels).
int cmgan_gemm_wgrad_tc_launch(const CmganGemmArgs* a, cudaStream_t st) {
    if (!wgrad_tc_supported(a)) return 1;
    const int ytiles = ((a->Cin + KT - 1) / KT) * a->ntaps;
    // rows per CTA: about four resident CTAs per SM in one wave (every CTA ends with one atomic pass over its dW tile), at least 8 stages
    long want = (4L * cmgan_num_sms()) / ytiles;
    if (want < 1) want = 1;
    long mch = (a->M + want - 1) / want;
    mch = ((mch + RS - 1) / RS) * RS;
    if (mch < 8 * RS) mch = 8 * RS;
    const dim3 grid((unsigned)ytiles, (unsigned)((a->M + mch - 1) / mch));
    const size_t smem = 1024 + 2 * (size_t)(A_BYTES + a->N * 128);
    const int rc = a->N <= 64 ? launch<4>(a, grid, smem, (int)mch, st) : launch<16>(a, grid, smem, (int)mch, st);
    if (rc) return rc;
    if (a->dbias) {
        const int rpb = 64 * (256 / a->N > 0 ? 256 / a->N : 1);     // ~64 rows per thread -> thousands of blocks
        colsum_kernel<<<cdiv(a->M, rpb), 256, 0, st>>>(a->D, a->ldd, a->M, a->N, a->prod, a->alpha, a->seed, a->drop_thr, a->inv_keep, rpb, a->dbias, a->seed_dev);
        return cmgan_check_launch("colsum_kernel");
    }
    return 0;
}
