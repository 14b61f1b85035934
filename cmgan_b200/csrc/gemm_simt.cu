// fp32 FFMA GEMMs with fused gather (implicit convolution), A-operand prologues and epilogues.
// These are the exact-fp32 baseline for every dense contraction of the path (see gemm_args.h for the
// contract); the tf32 wgmma kernels in gemm_tc.cu / gemm_wgrad_tc.cu implement the same contract for the hot shapes.
#include "common.cuh"
#include "../../include/cmgan_b200.h"
#include "gemm_args.h"
#include "gemm_device.cuh"

namespace {
using namespace cmgan_gemm;

constexpr int BM = 128, BN = 64, BK = 16, NT = 256;
constexpr int AS_LD = BM + 4;

template <int VEC>
__global__ void __launch_bounds__(NT, 2) gemm_rows_kernel(const __grid_constant__ CmganGemmArgs g) {
    __shared__ __align__(16) float As[BK][AS_LD];
    __shared__ __align__(16) float Bs[BK][BN];
    const int tid = threadIdx.x;
    const int m0 = blockIdx.x * BM, n0 = blockIdx.y * BN;
    const int ty = tid >> 4, tx = tid & 15;           // compute mapping: rows ty*8.., cols tx*4..
    const int lr = tid >> 2, lk = (tid & 3) * 4;        // A load mapping: rows lr, lr+64; k offset lk
    const int bk = tid >> 4, bn = (tid & 15) * 4;       // B load mapping
    const RowInfo ri0 = decode_row(g, m0 + lr), ri1 = decode_row(g, m0 + lr + 64);
    const int cpt = (g.Cin + BK - 1) / BK;              // chunks per tap
    const int nchunks = cpt * g.ntaps;

    float acc[8][4];
#pragma unroll
    for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;

    float ra0[4], ra1[4], rb[4];
    auto fetch = [&](int c) {
        int tap = c / cpt, k0 = (c - tap * cpt) * BK;
        load_a4<VEC>(g, in_row_of(g, ri0, tap), tap, k0 + lk, ra0);
        load_a4<VEC>(g, in_row_of(g, ri1, tap), tap, k0 + lk, ra1);
        int kk = k0 + bk;
        const float* bp = g.B + (long)tap * g.sb_tap + (long)kk * g.sb_k;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            int n = n0 + bn + j;
            rb[j] = (kk < g.Cin && n < g.N) ? __ldg(bp + (long)n * g.sb_n) : 0.f;
        }
    };
    fetch(0);
    for (int c = 0; c < nchunks; ++c) {
#pragma unroll
        for (int i = 0; i < 4; ++i) { As[lk + i][lr] = ra0[i]; As[lk + i][lr + 64] = ra1[i]; }
        *reinterpret_cast<float4*>(&Bs[bk][bn]) = make_float4(rb[0], rb[1], rb[2], rb[3]);
        __syncthreads();
        if (c + 1 < nchunks) fetch(c + 1);
#pragma unroll
        for (int k = 0; k < BK; ++k) {
            float4 a0 = *reinterpret_cast<const float4*>(&As[k][ty * 8]);
            float4 a1 = *reinterpret_cast<const float4*>(&As[k][ty * 8 + 4]);
            float4 b = *reinterpret_cast<const float4*>(&Bs[k][tx * 4]);
            float a[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
            float bb[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
            for (int i = 0; i < 8; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(a[i], bb[j], acc[i][j]);
        }
        __syncthreads();
    }
    // epilogue
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        long m = m0 + ty * 8 + i;
        if (m >= g.M) continue;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            int n = n0 + tx * 4 + j;
            if (n >= g.N) continue;
            float v = acc[i][j] + (g.bias ? __ldg(g.bias + n) : 0.f);
            if (g.epi == CMGAN_EPI_SWISH_DUAL) {
                g.C2[m * g.ldc2 + n] = swishf_(v) * cmgan_drop_scale(eff_seed(g), (uint64_t)m * g.N + n, g.drop_thr, g.inv_keep);
                if (g.C) g.C[m * g.ldc + n] = v;
            } else {
                float* cp = g.C + m * g.ldc + n;
                *cp = epilogue(g, v, m, n, cp);
            }
        }
    }
}

// ------------------------------------------------------------------------------------------------
// weight gradient:  dW(tap, k, n) += sum_m pro(A[in_row(m,tap), k]) * prod(D[m, n]);  dbias[n] += sum_m prod(D[m,n])
constexpr int WK = 64, WN = 64, WR = 16, MCH = 1024;

template <int VEC>
__global__ void __launch_bounds__(NT, 2) gemm_wgrad_kernel(const __grid_constant__ CmganGemmArgs g) {
    __shared__ __align__(16) float As[WR][WK];
    __shared__ __align__(16) float Ds[WR][WN];
    const int tid = threadIdx.x;
    const int ktiles = (g.Cin + WK - 1) / WK;
    const int tap = blockIdx.x / ktiles, k0 = (blockIdx.x % ktiles) * WK;
    const int n0 = blockIdx.y * WN;
    const long mbeg = (long)blockIdx.z * MCH;
    const long mend = mbeg + MCH < g.M ? mbeg + MCH : g.M;
    const int ty = tid >> 4, tx = tid & 15;
    const int lr = tid >> 4, lc = (tid & 15) * 4;
    float acc[4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
    float bsum = 0.f;
    const bool do_bias = g.dbias != nullptr && blockIdx.x == 0;

    float ra[4], rd[4];
    auto fetch = [&](long mb) {
        long m = mb + lr;
        RowInfo ri = decode_row(g, (int)(m < mend ? m : g.M));   // m >= mend -> masked (ri.ok false)
        if (m >= mend) ri.ok = false;
        load_a4<VEC>(g, in_row_of(g, ri, tap), tap, k0 + lc, ra);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            int n = n0 + lc + j;
            float d = 0.f;
            if (m < mend && n < g.N) {
                d = __ldg(g.D + m * g.ldd + n);
                if (g.prod == 1) d *= g.alpha * cmgan_drop_scale(eff_seed(g), (uint64_t)m * g.N + n, g.drop_thr, g.inv_keep);
            }
            rd[j] = d;
        }
    };
    if (mbeg < mend) fetch(mbeg);
    for (long mb = mbeg; mb < mend; mb += WR) {
        *reinterpret_cast<float4*>(&As[lr][lc]) = make_float4(ra[0], ra[1], ra[2], ra[3]);
        *reinterpret_cast<float4*>(&Ds[lr][lc]) = make_float4(rd[0], rd[1], rd[2], rd[3]);
        __syncthreads();
        if (mb + WR < mend) fetch(mb + WR);
#pragma unroll
        for (int r = 0; r < WR; ++r) {
            float4 a = *reinterpret_cast<const float4*>(&As[r][ty * 4]);
            float4 d = *reinterpret_cast<const float4*>(&Ds[r][tx * 4]);
            float aa[4] = {a.x, a.y, a.z, a.w}, dd[4] = {d.x, d.y, d.z, d.w};
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(aa[i], dd[j], acc[i][j]);
        }
        if (do_bias && tid < WN) {
#pragma unroll
            for (int r = 0; r < WR; ++r) bsum += Ds[r][tid];
        }
        __syncthreads();
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        int k = k0 + ty * 4 + i;
        if (k >= g.Cin) continue;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            int n = n0 + tx * 4 + j;
            if (n >= g.N) continue;
            atomicAdd(g.C + (long)tap * g.sb_tap + (long)k * g.sb_k + (long)n * g.sb_n, acc[i][j]);
        }
    }
    if (do_bias && tid < WN && n0 + tid < g.N) atomicAdd(g.dbias + n0 + tid, bsum);
}

// narrow forward / data gradient: N <= 16 output columns (the discriminator's first convolution and its input gradient, the decoders'
// 1- and 2-channel output convolutions).  Thread = one output row; the whole weight (ntaps * Cin x N, zero-padded to NP columns) sits in
// shared memory and is read with broadcast 128-bit loads; A is read once, as it lies.
template <int NP, int VEC>
__global__ void __launch_bounds__(NT) gemm_rows_narrow_kernel(const __grid_constant__ CmganGemmArgs g) {
    extern __shared__ __align__(16) float Ws[];           // [ntaps * Cin][NP]
    const int ktot = g.ntaps * g.Cin;
    for (int e = threadIdx.x; e < ktot * NP; e += NT) {
        const int kk = e / NP, n = e - kk * NP;
        const int tap = kk / g.Cin, k = kk - tap * g.Cin;
        Ws[e] = n < g.N ? __ldg(g.B + (long)tap * g.sb_tap + (long)k * g.sb_k + (long)n * g.sb_n) : 0.f;
    }
    __syncthreads();
    const long m = (long)blockIdx.x * NT + threadIdx.x;
    if (m >= g.M) return;
    const RowInfo ri = decode_row(g, (int)m);
    float acc[NP];
#pragma unroll
    for (int n = 0; n < NP; ++n) acc[n] = (g.bias && n < g.N) ? __ldg(g.bias + n) : 0.f;
    for (int tap = 0; tap < g.ntaps; ++tap) {
        const long ir = in_row_of(g, ri, tap);
        if (ir < 0) continue;
        const float* ap = g.A + g.tap_off[tap] + ir * g.lda;
        const float* wp = Ws + tap * g.Cin * NP;
        for (int k = 0; k < g.Cin; k += VEC) {
            float a[VEC];
            if (VEC == 4) {
                const float4 v = __ldg(reinterpret_cast<const float4*>(ap + k));
                a[0] = v.x; a[1] = v.y; a[2] = v.z; a[3] = v.w;
            } else {
                a[0] = __ldg(ap + k);
            }
#pragma unroll
            for (int i = 0; i < VEC; ++i)
#pragma unroll
                for (int n4 = 0; n4 < NP; n4 += 4) {
                    const float4 w = *reinterpret_cast<const float4*>(wp + (k + i) * NP + n4);
                    acc[n4] = fmaf(a[i], w.x, acc[n4]); acc[n4 + 1] = fmaf(a[i], w.y, acc[n4 + 1]);
                    acc[n4 + 2] = fmaf(a[i], w.z, acc[n4 + 2]); acc[n4 + 3] = fmaf(a[i], w.w, acc[n4 + 3]);
                }
        }
    }
    float* cp = g.C + m * g.ldc;
    if (NP == 16 && g.N == 16 && (g.ldc & 3) == 0 && (((uintptr_t)g.C) & 15) == 0) {
#pragma unroll
        for (int n4 = 0; n4 < 16; n4 += 4) *reinterpret_cast<float4*>(cp + n4) = make_float4(acc[n4], acc[n4 + 1], acc[n4 + 2], acc[n4 + 3]);
    } else {
#pragma unroll
        for (int n = 0; n < NP; ++n)
            if (n < g.N) cp[n] = acc[n];
    }
}

// narrow weight gradient: few input channels x taps and few outputs (the discriminator's first convolution: 2 channels, 4 x 4 taps,
// 16 outputs; the 64 x 64 tile above would be 99 % padding).  All ntaps * Cin <= 64 reduction columns and N <= 64 outputs of a row
// chunk are accumulated by one block: thread = up to 16 (k, n) products, 32 gathered rows per stage.
constexpr int NW_R = 32, NW_K = 64, NW_N = 64, NW_ACC = NW_K * NW_N / NT;
__global__ void __launch_bounds__(NT) gemm_wgrad_narrow_kernel(const __grid_constant__ CmganGemmArgs g, int mch) {
    __shared__ float As[NW_R][NW_K + 1];
    __shared__ float Ds[NW_R][NW_N + 1];
    const int tid = threadIdx.x;
    const int ktot = g.ntaps * g.Cin, nout = ktot * g.N;
    const long mbeg = (long)blockIdx.x * mch;
    const long mend = mbeg + mch < g.M ? mbeg + mch : g.M;
    float acc[NW_ACC];
#pragma unroll
    for (int j = 0; j < NW_ACC; ++j) acc[j] = 0.f;
    for (long mb = mbeg; mb < mend; mb += NW_R) {
        __syncthreads();
        for (int e = tid; e < NW_R * ktot; e += NT) {
            const int r = e / ktot, kk = e - r * ktot;
            const int tap = kk / g.Cin, k = kk - tap * g.Cin;
            const long m = mb + r;
            float v = 0.f;
            if (m < mend) {
                const long ir = in_row_of(g, decode_row(g, (int)m), tap);
                if (ir >= 0) v = __ldg(g.A + g.tap_off[tap] + ir * g.lda + k);
            }
            As[r][kk] = v;
        }
        for (int e = tid; e < NW_R * g.N; e += NT) {
            const int r = e / g.N, n = e - r * g.N;
            const long m = mb + r;
            Ds[r][n] = m < mend ? __ldg(g.D + m * g.ldd + n) : 0.f;
        }
        __syncthreads();
#pragma unroll
        for (int j = 0; j < NW_ACC; ++j) {
            const int o = tid + NT * j;
            if (o >= nout) break;
            const int kk = o / g.N, n = o - kk * g.N;
            float a = acc[j];
#pragma unroll 8
            for (int r = 0; r < NW_R; ++r) a = fmaf(As[r][kk], Ds[r][n], a);
            acc[j] = a;
        }
    }
#pragma unroll
    for (int j = 0; j < NW_ACC; ++j) {
        const int o = tid + NT * j;
        if (o >= nout) break;
        const int kk = o / g.N, n = o - kk * g.N;
        const int tap = kk / g.Cin, k = kk - tap * g.Cin;
        atomicAdd(g.C + (long)tap * g.sb_tap + (long)k * g.sb_k + (long)n * g.sb_n, acc[j]);
    }
}


bool vec_ok(const CmganGemmArgs& a) {
    if (a.lda % 4 || a.Cin % 4 || ((uintptr_t)a.A & 15)) return false;
    for (int t = 0; t < a.ntaps; ++t)
        if (a.tap_off[t] % 4) return false;
    return true;
}

int validate(const CmganGemmArgs* a, const char* who) {
    CMGAN_REQUIRE(a != nullptr, "%s: null args", who);
    CMGAN_REQUIRE(a->M >= 0 && a->N > 0 && a->Cin > 0, "%s: bad shape M=%d N=%d Cin=%d", who, a->M, a->N, a->Cin);
    CMGAN_REQUIRE(a->ntaps >= 1 && a->ntaps <= CMGAN_MAX_TAPS, "%s: ntaps=%d out of range", who, a->ntaps);
    CMGAN_REQUIRE(a->A && (a->C || (a->epi == CMGAN_EPI_SWISH_DUAL && a->C2)), "%s: null A/C pointer", who);
    if (a->epi == CMGAN_EPI_SWISH_DUAL) CMGAN_REQUIRE(a->C2 != nullptr, "%s: SWISH_DUAL epilogue needs C2", who);
    if (a->conv) {
        CMGAN_REQUIRE(a->OH > 0 && a->OW > 0 && a->IH > 0 && a->IW > 0, "%s: bad conv geometry", who);
        CMGAN_REQUIRE(a->mul_y >= 1 && a->mul_x >= 1 && a->div_y >= 1 && a->div_x >= 1, "%s: bad stride", who);
        CMGAN_REQUIRE((long)a->M % ((long)a->OH * a->OW) == 0, "%s: M=%d is not a multiple of OH*OW", who, a->M);
    }
    if (a->pro == CMGAN_PRO_LN) CMGAN_REQUIRE(a->p0 && a->p1 && a->p2, "%s: LN prologue needs stats/gamma/beta", who);
    if (a->pro == CMGAN_PRO_BN_SWISH) CMGAN_REQUIRE(a->p0 && a->p1, "%s: BN prologue needs scale/shift", who);
    if (a->pro == CMGAN_PRO_IN_PRELU) CMGAN_REQUIRE(a->p0 && a->p1 && a->p2 && a->rows_per_batch > 0, "%s: IN prologue params", who);
    return 0;
}

}  // namespace

int cmgan_gemm_rows_tc_launch(const CmganGemmArgs* a, cudaStream_t st);    // gemm_tc.cu
int cmgan_gemm_wgrad_tc_launch(const CmganGemmArgs* a, cudaStream_t st);   // gemm_wgrad_tc.cu

// C[M, N] = epi(bias + sum_taps pro(A) * B); see gemm_args.h.  Replaces every nn.Linear / nn.Conv1d(k=1) /
// nn.Conv2d of reference generator.py:24-32,53-63,108 and conformer.py:82-84,140-144,163,173 and their
// autograd data gradients.
CMGAN_API int cmgan_gemm_rows_f32(const CmganGemmArgs* a, void* stream) {
    if (validate(a, "cmgan_gemm_rows_f32")) return -1;
    CMGAN_REQUIRE(a->B != nullptr, "cmgan_gemm_rows_f32: null B");
    if (a->M == 0) return 0;
    if (a->epi == CMGAN_EPI_DSWISH_DROP || a->epi == CMGAN_EPI_DBNSWISH) CMGAN_REQUIRE(a->aux != nullptr, "gemm_rows: epilogue needs aux");
    if (a->precision == 1) {                       // tf32 wgmma path (gemm_tc.cu); 1 = shape not covered -> exact fp32 path below
        int rc = cmgan_gemm_rows_tc_launch(a, (cudaStream_t)stream);
        if (rc <= 0) return rc;
    }
    if (a->N <= 16 && a->pro == CMGAN_PRO_NONE && a->epi == CMGAN_EPI_NONE && (long)a->ntaps * a->Cin * 16 * 4 <= 48 * 1024) {
        const int np = a->N <= 4 ? 4 : 16;
        const int smem = a->ntaps * a->Cin * np * (int)sizeof(float);
        const unsigned grid_n = (unsigned)cdiv(a->M, NT);
        const bool v4 = vec_ok(*a);
        if (np == 4) {
            if (v4) gemm_rows_narrow_kernel<4, 4><<<grid_n, NT, smem, (cudaStream_t)stream>>>(*a);
            else gemm_rows_narrow_kernel<4, 1><<<grid_n, NT, smem, (cudaStream_t)stream>>>(*a);
        } else {
            if (v4) gemm_rows_narrow_kernel<16, 4><<<grid_n, NT, smem, (cudaStream_t)stream>>>(*a);
            else gemm_rows_narrow_kernel<16, 1><<<grid_n, NT, smem, (cudaStream_t)stream>>>(*a);
        }
        return cmgan_check_launch("gemm_rows_narrow_kernel");
    }
    dim3 grid(cdiv(a->M, BM), cdiv(a->N, BN));
    if (vec_ok(*a)) gemm_rows_kernel<4><<<grid, NT, 0, (cudaStream_t)stream>>>(*a);
    else gemm_rows_kernel<1><<<grid, NT, 0, (cudaStream_t)stream>>>(*a);
    return cmgan_check_launch("gemm_rows_kernel");
}

// dW += A^T D (accumulates with atomics into a[C], laid out like B in the forward call) and dbias += colsum(D).
CMGAN_API int cmgan_gemm_wgrad_f32(const CmganGemmArgs* a, void* stream) {
    if (validate(a, "cmgan_gemm_wgrad_f32")) return -1;
    CMGAN_REQUIRE(a->D != nullptr, "cmgan_gemm_wgrad_f32: null D");
    if (a->M == 0) return 0;
    if (a->precision == 1) {                       // tf32 wgmma path (gemm_wgrad_tc.cu); 1 = shape not covered -> exact fp32 path below
        int rc = cmgan_gemm_wgrad_tc_launch(a, (cudaStream_t)stream);
        if (rc <= 0) return rc;
    }
    if (a->ntaps * a->Cin <= NW_K && a->N <= NW_N && a->Cin < 16 && a->pro == CMGAN_PRO_NONE && a->prod == 0 && a->dbias == nullptr) {
        long mch = cdiv(a->M, (long)cmgan_num_sms() * 4);
        mch = cdiv(mch < 256 ? 256 : mch, NW_R) * NW_R;
        gemm_wgrad_narrow_kernel<<<(unsigned)cdiv(a->M, mch), NT, 0, (cudaStream_t)stream>>>(*a, (int)mch);
        return cmgan_check_launch("gemm_wgrad_narrow_kernel");
    }
    dim3 grid(cdiv(a->Cin, WK) * a->ntaps, cdiv(a->N, WN), cdiv(a->M, MCH));
    if (vec_ok(*a)) gemm_wgrad_kernel<4><<<grid, NT, 0, (cudaStream_t)stream>>>(*a);
    else gemm_wgrad_kernel<1><<<grid, NT, 0, (cudaStream_t)stream>>>(*a);
    return cmgan_check_launch("gemm_wgrad_kernel");
}
