// tf32 tensor-core weight and bias gradient for sm_90a   (gemm_args.h, wgrad form)
//     dW(tap, k, n) += sum_m pro(A[in_row(m, tap), k]) * prod(D[m, n])          dbias[n] += sum_m prod(D[m, n])
//
// The reduction runs over the rows m, and wgmma reads tf32 operands from shared memory only K-major, so both operands are transposed inside
// the SM.  One CTA owns a 64 x Q tile of dW (Q <= 256) and a range of rows, which it streams in stages of 32 rows:
//   - all 256 threads gather the stage's raw rows of A and D (row-major, as they lie in memory; convolution taps, strides and padding
//     resolved per row) with 16-byte cp.async into a ring of 3 .. 6 slabs, so that several stages of loads are in flight at any time;
//   - the same threads then read the oldest slab, apply the A prologue and D's dropout scale, add D into per-thread column sums for
//     dbias, round to tf32 and write the K-major SWIZZLE_128B image (one 128-byte line of 32 m-values per k or n) that the descriptors read;
//   - each warpgroup multiplies one half of the Q side of the image (m64n64k8 where Q allows, else m64n16k8) while the next image is
//     being written into the other buffer.
// The tile orientation is chosen per shape so that every CTA reads its rows of A and D once: either k on the wgmma M side and all N
// columns on the Q side (P = A), or n on the M side and all Cin columns on the Q side (P = D, Cin <= 256).  At the end each CTA adds its
// tile into dW (and, for one tile per tap-0 column range, its column sums into dbias) with atomics: the parameter-gradient buffer is
// zeroed once per step.  The grid is as many CTAs as are resident at once (one wave).
// The dense blocks' dilated 2 x 3 convolutions take a second plan that covers all six taps in one tile (gemm_wgrad_taps_kernel below).
#include "common.cuh"
#include "../../include/cmgan_b200.h"
#include "gemm_device.cuh"
#include "tc_ptx.cuh"

namespace {
using namespace cmgan_gemm;
using namespace cmgan_tc;

constexpr int NT = 256;              // two warpgroups
constexpr int RS = 32;               // rows per stage = one 128-byte line of m-values
constexpr int PT = 64;               // lines on the P side = wgmma M
constexpr int QMAX = 256;            // lines on the Q side, at most
constexpr int MAX_RING = 6;

struct Plan {
    int ydir;              // 0: P = 64 k of A, Q = the N columns of D;  1: P = 64 n of D, Q = the Cin columns of A
    int ptiles;            // 64-wide tiles along P per tap
    int qpad;              // Q lines, rounded up to 32 (two warpgroups x a multiple of 16)
    int wa, wd;            // raw row widths (floats) of the A and D slabs: multiples of 32
    int ring;              // slabs in the cp.async ring
    int mch;               // rows per CTA, a multiple of RS
    uint32_t raw_bytes;    // one slab: A rows, D rows, in_row of each row (int), LN statistics of each row (float2)
    uint32_t img_bytes;    // one operand image: P lines then Q lines, 128 bytes each
};

// byte offset of 16-byte chunk c of row r in a raw slab of row width w floats.  The chunk index is XOR-swizzled by the row's m-group, so
// that the eight lanes that read rows 4 g + i (g = 0..7) of one chunk hit eight different bank groups.
__device__ __forceinline__ uint32_t raw_off(int r, int c, int w) { return (uint32_t)(r * w * 4 + ((c ^ ((r >> 2) & 7)) << 4)); }

// one 32-row stage (4 K-steps of 8) of the warpgroup's 64 x 16 NB accumulator; `first` overwrites instead of accumulating
template <int NB>
__device__ __forceinline__ void mma_stage(float (&acc)[NB][8], uint64_t adesc, uint64_t bdesc, bool first) {
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const uint32_t accumulate = (first && k == 0) ? 0u : 1u;
        if constexpr (NB % 4 == 0) {
#pragma unroll
            for (int c = 0; c < NB / 4; ++c)
                wgmma_m64n64k8_tf32(reinterpret_cast<float(&)[4][8]>(acc[4 * c]), adesc + (uint64_t)(2 * k), bdesc + (uint64_t)(512 * c + 2 * k),
                                    accumulate);
        } else {
#pragma unroll
            for (int j = 0; j < NB; ++j) wgmma_m64n16k8_tf32(acc[j], adesc + (uint64_t)(2 * k), bdesc + (uint64_t)(128 * j + 2 * k), accumulate);
        }
    }
}
__device__ __forceinline__ void cp_async_wait_n(int n) {
    switch (n) {
        case 0: cp_async_wait<0>(); break;
        case 1: cp_async_wait<1>(); break;
        case 2: cp_async_wait<2>(); break;
        case 3: cp_async_wait<3>(); break;
        default: cp_async_wait<4>(); break;
    }
}

__device__ __forceinline__ float4 round4(float4 v) { return make_float4(to_tf32(v.x), to_tf32(v.y), to_tf32(v.z), to_tf32(v.w)); }

// NB = n16 accumulator blocks per warpgroup = qpad / 32.  Up to Q = 96 the shared memory holds two CTAs per SM, so the registers must too.
template <int NB>
__global__ void __launch_bounds__(NT, NB <= 3 ? 2 : 1) gemm_wgrad_tc_kernel(const __grid_constant__ CmganGemmArgs g, const Plan p) {
    extern __shared__ uint8_t smem_raw[];
    const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;
    uint8_t* const bptr = smem_raw + (base - smem_u32(smem_raw));
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, wg = tid >> 7;
    const int tap = blockIdx.x / p.ptiles, p0 = (blockIdx.x % p.ptiles) * PT;
    const int acol0 = p.ydir ? 0 : p0, na = p.ydir ? g.Cin : min(PT, g.Cin - p0);     // A columns of this tile
    const int dcol0 = p.ydir ? p0 : 0, nd = p.ydir ? min(PT, g.N - p0) : g.N;        // D columns of this tile
    const int la = p.ydir ? p.qpad : PT, ld = p.ydir ? PT : p.qpad;                   // image lines of A / D
    const uint32_t aimg = p.ydir ? PT * 128 : 0, dimg = p.ydir ? 0 : PT * 128;        // their offsets inside an image
    const long mbeg = (long)blockIdx.y * p.mch;
    const long mend = mbeg + p.mch < g.M ? mbeg + p.mch : g.M;
    const int nst = (int)((mend - mbeg + RS - 1) / RS);
    if (nst <= 0) return;
    const unsigned long long seed = eff_seed(g);
    const bool do_bias = g.dbias != nullptr && tap == 0 && (p.ydir || p0 == 0);
    uint8_t* const img0 = bptr;
    uint8_t* const ring = bptr + 2 * p.img_bytes;
    const uint32_t dslab = (uint32_t)(RS * p.wa * 4), rows_off = (uint32_t)(RS * (p.wa + p.wd) * 4), stats_off = rows_off + RS * 4;

    // stage s -> slab `slot`: thread t gathers row t / 8 of the stage, 16-byte chunks t % 8, t % 8 + 8, ... of its A and D columns
    auto issue = [&](int s, int slot) {
        uint8_t* const sl = ring + slot * p.raw_bytes;
        const int row = tid >> 3, c8 = tid & 7;
        const long m = mbeg + (long)s * RS + row;
        long r = -1;
        if (m < mend) r = in_row_of(g, decode_row(g, (int)m), tap);
        if (c8 == 0) reinterpret_cast<int*>(sl + rows_off)[row] = (int)r;
        if (r >= 0) {
            const float* src = g.A + g.tap_off[tap] + r * g.lda + acol0;
            for (int c = c8; c < na / 4; c += 8) cp_async16(smem_u32(sl + raw_off(row, c, p.wa)), src + 4 * c, 16);
            if (g.pro == CMGAN_PRO_LN && c8 == 0) cp_async8(smem_u32(sl + stats_off + row * 8), g.p0 + 2 * r);
        }
        if (m < mend) {
            const float* src = g.D + m * g.ldd + dcol0;
            for (int c = c8; c < nd / 4; c += 8) cp_async16(smem_u32(sl + dslab + raw_off(row, c, p.wd)), src + 4 * c, 16);
        }
    };

    // item it < 2 ld: D lines 4 lb .. 4 lb + 3 x rows 4 q .. 4 q + 3 (lb = it / 8, q = it % 8); then the same for A.  A thread keeps its
    // D items from stage to stage, so it keeps their column sums in registers (at most 2 items: ld <= 256).
    float cs[2][4] = {};
    auto colsum = [](float (&c)[4], const float4 (&v)[4]) {
#pragma unroll
        for (int i = 0; i < 4; ++i) { c[0] += v[i].x; c[1] += v[i].y; c[2] += v[i].z; c[3] += v[i].w; }
    };
    auto transform = [&](int s, int slot, uint8_t* img) {
        const uint8_t* const sl = ring + slot * p.raw_bytes;
        const int* const rows = reinterpret_cast<const int*>(sl + rows_off);
        const float2* const stats = reinterpret_cast<const float2*>(sl + stats_off);
        const long mb = mbeg + (long)s * RS;
#pragma unroll 1
        for (int u = 0; u < 3; ++u) {
            const int it = tid + u * NT;
            if (it >= 2 * (ld + la)) break;
            const bool isd = it < 2 * ld;
            const int j = isd ? it : it - 2 * ld, lb = j >> 3, q = j & 7;
            float4 v[4];
            if (4 * lb < (isd ? nd : na)) {
                const uint8_t* const src = isd ? sl + dslab : sl;
                const int w = isd ? p.wd : p.wa;
#pragma unroll
                for (int i = 0; i < 4; ++i) v[i] = *reinterpret_cast<const float4*>(src + raw_off(4 * q + i, lb, w));
                if (isd) {
#pragma unroll
                    for (int i = 0; i < 4; ++i) {
                        const long m = mb + 4 * q + i;
                        if (m >= mend) { v[i] = make_float4(0.f, 0.f, 0.f, 0.f); continue; }
                        if (g.prod == 1) {
                            float ds[4];
                            cmgan_drop_scale4(seed, (uint64_t)m * g.N + dcol0 + 4 * lb, g.drop_thr, g.inv_keep, ds);
                            v[i].x *= g.alpha * ds[0]; v[i].y *= g.alpha * ds[1]; v[i].z *= g.alpha * ds[2]; v[i].w *= g.alpha * ds[3];
                        }
                    }
                    if (do_bias) {
                        if (u == 0) colsum(cs[0], v);
                        else colsum(cs[1], v);
                    }
                } else {
                    const int k = acol0 + 4 * lb;
                    ChunkParams cp;
                    load_chunk_params(g, k, cp);
#pragma unroll
                    for (int i = 0; i < 4; ++i) {
                        const int r = rows[4 * q + i];
                        if (r < 0) { v[i] = make_float4(0.f, 0.f, 0.f, 0.f); continue; }
                        if (g.pro != CMGAN_PRO_NONE) {
                            const float2 st = g.pro == CMGAN_PRO_LN ? stats[4 * q + i] : make_float2(0.f, 0.f);
                            v[i] = transform4(g, v[i], r, k, st.x, st.y, cp);
                        }
                    }
                }
            } else {
#pragma unroll
                for (int i = 0; i < 4; ++i) v[i] = make_float4(0.f, 0.f, 0.f, 0.f);
            }
#pragma unroll
            for (int i = 0; i < 4; ++i) v[i] = round4(v[i]);
            // line L = 4 lb + e of the image holds (v[0].e, v[1].e, v[2].e, v[3].e) at m-group q
            uint8_t* const dst = img + (isd ? dimg : aimg);
            const int L = 4 * lb;
            *reinterpret_cast<float4*>(dst + (L + 0) * 128 + (((q ^ (L + 0)) & 7) << 4)) = make_float4(v[0].x, v[1].x, v[2].x, v[3].x);
            *reinterpret_cast<float4*>(dst + (L + 1) * 128 + (((q ^ (L + 1)) & 7) << 4)) = make_float4(v[0].y, v[1].y, v[2].y, v[3].y);
            *reinterpret_cast<float4*>(dst + (L + 2) * 128 + (((q ^ (L + 2)) & 7) << 4)) = make_float4(v[0].z, v[1].z, v[2].z, v[3].z);
            *reinterpret_cast<float4*>(dst + (L + 3) * 128 + (((q ^ (L + 3)) & 7) << 4)) = make_float4(v[0].w, v[1].w, v[2].w, v[3].w);
        }
        fence_proxy_async();          // generic-proxy stores -> visible to the tensor core's async proxy
    };

    float acc[NB][8];      // written first by the MMAs of stage 0 (nst >= 1)
    const int qh = NB * 16;

    // one commit group per stage (empty past the end), so that "stage s has landed" is always "at most ring - 2 groups pending"
    for (int s = 0; s < p.ring - 1; ++s) {
        if (s < nst) issue(s, s);
        cp_async_commit();
    }
    for (int s = 0; s < nst; ++s) {
        cp_async_wait_n(p.ring - 2);
        __syncthreads();              // stage s visible to all; the slab and image of stage s - 2 / s - 1 are no longer read
        if (s + p.ring - 1 < nst) issue(s + p.ring - 1, (s + p.ring - 1) % p.ring);
        cp_async_commit();
        uint8_t* const img = img0 + (s & 1) * p.img_bytes;
        transform(s, s % p.ring, img);
        __syncthreads();
        const uint32_t ia = smem_u32(img);
        wgmma_fence();
        mma_stage<NB>(acc, gmma_desc_sw128(ia), gmma_desc_sw128(ia + PT * 128 + wg * qh * 128), s == 0);
        wgmma_commit();
        wgmma_wait<1>();              // the MMAs of stage s - 1 are done: its image buffer is written next
    }
    wgmma_wait<0>();

    // fragment of warp w of warpgroup h: P line 16 (w % 4) + lane / 4 (+ 8), Q line h qh + 16 j + 8 i + 2 (lane % 4) (+ 1)
    const int pl = 16 * (warp & 3) + (lane >> 2), ql = wg * qh + 2 * (lane & 3);
    float* const dst = g.C + (long)tap * g.sb_tap;
#pragma unroll
    for (int j = 0; j < NB; ++j) {
#pragma unroll
        for (int e = 0; e < 8; ++e) {
            const int pe = p0 + pl + 8 * ((e >> 1) & 1), qe = ql + 16 * j + 8 * (e >> 2) + (e & 1);
            const int k = p.ydir ? qe : pe, n = p.ydir ? pe : qe;
            if (k < g.Cin && n < g.N) atomicAdd(dst + (long)k * g.sb_k + (long)n * g.sb_n, acc[j][e]);
        }
    }
    if (do_bias) {
#pragma unroll
        for (int u = 0; u < 2; ++u) {
            const int it = tid + u * NT;
            if (it >= 2 * ld) break;                    // uniform per warp: 2 ld is a multiple of 64
            const int lb = it >> 3;
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                float v = cs[u][e];
                v += __shfl_xor_sync(0xffffffffu, v, 1);
                v += __shfl_xor_sync(0xffffffffu, v, 2);
                v += __shfl_xor_sync(0xffffffffu, v, 4);
                if ((it & 7) == 0 && 4 * lb + e < nd) atomicAdd(g.dbias + dcol0 + 4 * lb + e, v);
            }
        }
    }
}

// ---- the dense block's causal dilated 2 x 3 convolution: all six taps in one tile -------------------------------------------------
// Taps (dy, dx) = ((kh - 1) dil, kw - 1), tap = 3 kh + kw, stride 1, same size.  Indexed by the input row r instead of the output row m,
//     dW(tap, k, n) = sum_r A[r, k] D[r - dy IW - dx, n]      (only where row r - dy IW - dx reads r through the tap)
// so one K-major image of a stage's 32 A rows serves every tap, and each tap reads D shifted by its offset.  The shift is along the
// wgmma K dimension, which a shared-memory descriptor cannot offset by single rows, so D^T goes to the M side from registers: each
// thread loads its fragment straight from a row-major D window at the tap's row, masks it and rounds it.  Warpgroup h takes the taps
// kh = h (three m64n64 accumulators, 96 registers): kh = 1 reads the window of the stage's own rows, kh = 0 one dil IW rows further,
// each with a one-row halo for dx = +-1.  A CTA owns 64 A columns and a range of A rows; dbias comes from tap (0, 0) of column tile 0.
constexpr int TQ = 64;               // A columns per CTA
constexpr int DWP = 72;              // D window row pitch (floats): 72 = 8 mod 32 banks, so the fragment loads are conflict-free
constexpr int DWR = RS + 2;          // D window rows: the stage's 32 and one each side
constexpr uint32_t TAPS_A = RS * TQ * 4, TAPS_WIN = DWR * DWP * 4, TAPS_MASK = 2 * TAPS_WIN + TAPS_A;
constexpr uint32_t TAPS_RAW = TAPS_MASK + RS * 4, TAPS_IMG = TQ * 128;

struct TapsPlan {
    int ring;              // slabs in the cp.async ring
    int mch;               // A rows per CTA, a multiple of RS
};

// bit t: A row r feeds tap t, i.e. row m = r - dy IW - dx lies in the same image row (x - dx inside [0, IW)), the same utterance and < M
__device__ __forceinline__ uint32_t taps_mask(const CmganGemmArgs& g, int r, int dil) {
    const int x = r % g.IW, y = (r / g.IW) % g.IH;
    uint32_t mk = 0;
#pragma unroll
    for (int t = 0; t < 6; ++t) {
        const int kh = t / 3, dx = t % 3 - 1;
        const long m = (long)r + (kh ? 0 : (long)dil * g.IW) - dx;
        if (x - dx >= 0 && x - dx < g.IW && (kh || y + dil < g.IH) && m < g.M) mk |= 1u << t;
    }
    return mk;
}

__global__ void __launch_bounds__(NT, 1) gemm_wgrad_taps_kernel(const __grid_constant__ CmganGemmArgs g, const TapsPlan p) {
    extern __shared__ uint8_t smem_raw[];
    const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;
    uint8_t* const bptr = smem_raw + (base - smem_u32(smem_raw));
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, wg = tid >> 7;
    const int acol0 = blockIdx.x * TQ, dil = -g.dy[0];
    const long shift = (long)dil * g.IW;
    const long rbeg = (long)blockIdx.y * p.mch;
    const long rend = rbeg + p.mch < g.M ? rbeg + p.mch : g.M;
    const int nst = (int)((rend - rbeg + RS - 1) / RS);
    if (nst <= 0) return;
    const bool do_bias = g.dbias != nullptr && blockIdx.x == 0;
    uint8_t* const img0 = bptr;
    uint8_t* const ring = bptr + 2 * TAPS_IMG;

    // stage s -> slab: thread t copies A row t / 8 (16-byte chunks t % 8, t % 8 + 8), the last warp writes the rows' tap masks; then
    // the 2 x 34 rows of the two D windows (window kh starts at D row r0 - 1 + (1 - kh) dil IW), 16 chunks each, rows outside [0, M)
    // left unwritten
    auto issue = [&](int s, int slot) {
        uint8_t* const sl = ring + slot * TAPS_RAW;
        const long r0 = rbeg + (long)s * RS;
        const int row = tid >> 3, c8 = tid & 7;
        const long r = r0 + row;
        if (r < rend) {
            const float* src = g.A + g.tap_off[0] + r * g.lda + acol0;
            cp_async16(smem_u32(sl + raw_off(row, c8, TQ)), src + 4 * c8, 16);
            cp_async16(smem_u32(sl + raw_off(row, c8 + 8, TQ)), src + 4 * c8 + 32, 16);
        }
        if (warp == NT / 32 - 1) {    // one warp decodes the stage's 32 rows: a divergent branch in every warp would cost each of them
            const long rl = r0 + lane;
            reinterpret_cast<uint32_t*>(sl + TAPS_MASK)[lane] = rl < rend ? taps_mask(g, (int)rl, dil) : 0u;
        }
        for (int i = tid; i < 2 * DWR * 16; i += NT) {
            const int kh = i / (DWR * 16), j = i % (DWR * 16), wr = j >> 4, c = j & 15;
            const long m = r0 - 1 + wr + (kh ? 0 : shift);
            if (m >= 0 && m < g.M) cp_async16(smem_u32(sl + TAPS_A + kh * TAPS_WIN + (wr * DWP + 4 * c) * 4), g.D + m * g.ldd + 4 * c, 16);
        }
    };

    // A rows -> K-major SWIZZLE_128B image: thread t < 128 transposes A lines 4 lb .. 4 lb + 3 x rows 4 q .. 4 q + 3 (lb = t / 8, q = t % 8)
    auto transform = [&](int s, int slot, uint8_t* img) {
        if (tid >= 2 * TQ) return;
        const uint8_t* const sl = ring + slot * TAPS_RAW;
        const long mb = rbeg + (long)s * RS;
        const int lb = tid >> 3, q = tid & 7;
        float4 v[4];
#pragma unroll
        for (int i = 0; i < 4; ++i)         // rows past the CTA's range are zero: another CTA owns them
            v[i] = mb + 4 * q + i < rend ? round4(*reinterpret_cast<const float4*>(sl + raw_off(4 * q + i, lb, TQ)))
                                         : make_float4(0.f, 0.f, 0.f, 0.f);
        const int L = 4 * lb;
        *reinterpret_cast<float4*>(img + (L + 0) * 128 + (((q ^ (L + 0)) & 7) << 4)) = make_float4(v[0].x, v[1].x, v[2].x, v[3].x);
        *reinterpret_cast<float4*>(img + (L + 1) * 128 + (((q ^ (L + 1)) & 7) << 4)) = make_float4(v[0].y, v[1].y, v[2].y, v[3].y);
        *reinterpret_cast<float4*>(img + (L + 2) * 128 + (((q ^ (L + 2)) & 7) << 4)) = make_float4(v[0].z, v[1].z, v[2].z, v[3].z);
        *reinterpret_cast<float4*>(img + (L + 3) * 128 + (((q ^ (L + 3)) & 7) << 4)) = make_float4(v[0].w, v[1].w, v[2].w, v[3].w);
    };

    // fragment of this thread: D columns n0, n0 + 8 (the M side), A rows 8 j + 4 h + tq of the stage (the K side)
    const int n0 = 16 * (warp & 3) + (lane >> 2), tq = lane & 3;
    float acc[3][4][8];                    // written first by the MMAs of stage 0 (nst >= 1)
    // dbias: columns n0, n0 + 8 (warpgroup 1, tap (0, 0)), compensated sums: a thread adds up to a quarter of its CTA's rows
    float cs0 = 0.f, cs1 = 0.f, cc0 = 0.f, cc1 = 0.f;
    auto kahan = [](float& sum, float& c, float v) {
        const float y = v - c, t = sum + y;
        c = (t - sum) - y;
        sum = t;
    };

    for (int s = 0; s < p.ring - 1; ++s) {
        if (s < nst) issue(s, s);
        cp_async_commit();
    }
    for (int s = 0; s < nst; ++s) {
        cp_async_wait_n(p.ring - 2);
        __syncthreads();              // stage s visible to all; slab s - 1 and image s - 2 are no longer read
        if (s + p.ring - 1 < nst) issue(s + p.ring - 1, (s + p.ring - 1) % p.ring);
        cp_async_commit();
        uint8_t* const img = img0 + (s & 1) * TAPS_IMG;
        transform(s, s % p.ring, img);
        fence_proxy_async();
        __syncthreads();
        wgmma_wait<0>();              // the MMAs of stage s - 1 are done: their fragment registers may be overwritten
        const uint8_t* const sl = ring + (s % p.ring) * TAPS_RAW;
        const float* const win = reinterpret_cast<const float*>(sl + TAPS_A + wg * TAPS_WIN) + n0;
        const uint32_t* const mask = reinterpret_cast<const uint32_t*>(sl + TAPS_MASK);
        uint32_t fr[4][3][4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int kk = 8 * j + 4 * h + tq;
                const uint32_t mk = mask[kk] >> (3 * wg);
#pragma unroll
                for (int kw = 0; kw < 3; ++kw) {
                    const float* const src = win + (kk + 2 - kw) * DWP;      // D row r - dx, window row r - r0 + 1 - dx
                    const bool ok = (mk >> kw) & 1u;
                    const float v0 = ok ? src[0] : 0.f, v1 = ok ? src[8] : 0.f;
                    fr[j][kw][2 * h] = __float_as_uint(to_tf32(v0));
                    fr[j][kw][2 * h + 1] = __float_as_uint(to_tf32(v1));
                    if (kw == 1 && wg == 1 && do_bias) { kahan(cs0, cc0, v0); kahan(cs1, cc1, v1); }
                }
            }
        }
        const uint64_t bdesc = gmma_desc_sw128(smem_u32(img));
        wgmma_fence();
#pragma unroll
        for (int j = 0; j < 4; ++j)
#pragma unroll
            for (int kw = 0; kw < 3; ++kw) wgmma_m64n64k8_tf32_rs(acc[kw], fr[j][kw], bdesc + (uint64_t)(2 * j), (s == 0 && j == 0) ? 0u : 1u);
        wgmma_commit();
    }
    wgmma_wait<0>();

    // accumulator fragment: M row n0 + 8 ((e >> 1) & 1), N column 16 b + 8 (e >> 2) + 2 tq + (e & 1)
    const int kh = wg;
#pragma unroll
    for (int kw = 0; kw < 3; ++kw) {
        float* const dst = g.C + (long)(3 * kh + kw) * g.sb_tap;
#pragma unroll
        for (int b = 0; b < 4; ++b)
#pragma unroll
            for (int e = 0; e < 8; ++e) {
                const int n = n0 + 8 * ((e >> 1) & 1), k = acol0 + 16 * b + 8 * (e >> 2) + 2 * tq + (e & 1);
                atomicAdd(dst + (long)k * g.sb_k + (long)n * g.sb_n, acc[kw][b][e]);
            }
    }
    if (do_bias && wg == 1) {
        cs0 += __shfl_xor_sync(0xffffffffu, cs0, 1);
        cs0 += __shfl_xor_sync(0xffffffffu, cs0, 2);
        cs1 += __shfl_xor_sync(0xffffffffu, cs1, 1);
        cs1 += __shfl_xor_sync(0xffffffffu, cs1, 2);
        if (tq == 0) { atomicAdd(g.dbias + n0, cs0); atomicAdd(g.dbias + n0 + 8, cs1); }
    }
}

// the dense block's convolution, which the taps plan covers: stride 1, same size, taps ((kh - 1) dil, kw - 1) in kh-major order, one A
// pointer for every tap, no prologue and no scale on D, N = 64 and whole 64-column tiles of A
bool taps_plan_fits(const CmganGemmArgs* a) {
    if (!a->conv || a->ntaps != 6 || a->mul_y != 1 || a->mul_x != 1 || a->div_y != 1 || a->div_x != 1) return false;
    if (a->OH != a->IH || a->OW != a->IW || a->pro != CMGAN_PRO_NONE || a->prod != 0 || a->N != 64 || a->Cin % TQ) return false;
    const int dil = -a->dy[0];
    if (dil < 1) return false;
    for (int t = 0; t < 6; ++t)
        if (a->dy[t] != (t / 3 - 1) * dil || a->dx[t] != t % 3 - 1 || a->tap_off[t] != a->tap_off[0]) return false;
    return true;
}

int wgrad_tc_supported(const CmganGemmArgs* a) {
    if (a->N % 16 || a->N < 16 || a->N > QMAX) return 0;
    if (a->Cin % 4 || a->lda % 4 || ((uintptr_t)a->A & 15) || a->ldd % 4 || ((uintptr_t)a->D & 15)) return 0;
    for (int t = 0; t < a->ntaps; ++t)
        if (a->tap_off[t] % 4) return 0;
    return 1;
}

// shared memory of an SM and the opt-in limit of one CTA (queried once)
int smem_limits(int* per_sm, int* per_block) {
    static int sm = 0, blk = 0;
    if (!sm) {
        int dev = 0;
        cudaError_t e = cudaGetDevice(&dev);
        if (e == cudaSuccess) e = cudaDeviceGetAttribute(&sm, cudaDevAttrMaxSharedMemoryPerMultiprocessor, dev);
        if (e == cudaSuccess) e = cudaDeviceGetAttribute(&blk, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev);
        if (e != cudaSuccess) { sm = 0; cmgan_set_error("gemm_wgrad_tc: device attributes: %s", cudaGetErrorString(e)); return -1; }
    }
    *per_sm = sm;
    *per_block = blk;
    return 0;
}

template <int NB>
int launch(const CmganGemmArgs* a, Plan p, size_t smem, int smem_blk, cudaStream_t st) {
    static bool attr_set = false;
    if (!attr_set) {
        cudaError_t e = cudaFuncSetAttribute(gemm_wgrad_tc_kernel<NB>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_blk);
        if (e != cudaSuccess) { cmgan_set_error("gemm_wgrad_tc: cudaFuncSetAttribute: %s", cudaGetErrorString(e)); return -1; }
        attr_set = true;
    }
    int occ = 0;
    cudaError_t e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, gemm_wgrad_tc_kernel<NB>, NT, smem);
    if (e != cudaSuccess || occ < 1) { cmgan_set_error("gemm_wgrad_tc: occupancy query: %s (%d CTAs)", cudaGetErrorString(e), occ); return -1; }
    // one wave: the resident CTAs split the rows evenly between them
    const long tiles = (long)a->ntaps * p.ptiles;
    long chunks = ((long)occ * cmgan_num_sms()) / tiles;
    if (chunks < 1) chunks = 1;
    const long max_chunks = (a->M + RS - 1) / RS;
    if (chunks > max_chunks) chunks = max_chunks;
    const long mch = (a->M + chunks - 1) / chunks;
    p.mch = (int)(((mch + RS - 1) / RS) * RS);
    const dim3 grid((unsigned)tiles, (unsigned)((a->M + p.mch - 1) / p.mch));
    gemm_wgrad_tc_kernel<NB><<<grid, NT, smem, st>>>(*a, p);
    return cmgan_check_launch("gemm_wgrad_tc_kernel");
}

// one CTA per SM (the accumulators take 96 registers a thread), one wave: the column tiles x row chunks fill the SMs once
int launch_taps(const CmganGemmArgs* a, int smem_blk, cudaStream_t st) {
    TapsPlan p{};
    const long ring = (smem_blk - 1024 - 2L * TAPS_IMG) / TAPS_RAW;
    if (ring < 3) { cmgan_set_error("gemm_wgrad_taps: the ring does not fit in shared memory"); return -1; }
    p.ring = ring > MAX_RING ? MAX_RING : (int)ring;
    const size_t smem = 1024 + 2 * (size_t)TAPS_IMG + (size_t)p.ring * TAPS_RAW;
    static bool attr_set = false;
    if (!attr_set) {
        cudaError_t e = cudaFuncSetAttribute(gemm_wgrad_taps_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_blk);
        if (e != cudaSuccess) { cmgan_set_error("gemm_wgrad_taps: cudaFuncSetAttribute: %s", cudaGetErrorString(e)); return -1; }
        attr_set = true;
    }
    const long tiles = a->Cin / TQ;
    long chunks = (long)cmgan_num_sms() / tiles;
    if (chunks < 1) chunks = 1;
    const long max_chunks = (a->M + RS - 1) / RS;
    if (chunks > max_chunks) chunks = max_chunks;
    const long mch = (a->M + chunks - 1) / chunks;
    p.mch = (int)(((mch + RS - 1) / RS) * RS);
    const dim3 grid((unsigned)tiles, (unsigned)((a->M + p.mch - 1) / p.mch));
    gemm_wgrad_taps_kernel<<<grid, NT, smem, st>>>(*a, p);
    return cmgan_check_launch("gemm_wgrad_taps_kernel");
}

}  // namespace

// tf32 tensor-core path of cmgan_gemm_wgrad (same contract, bias gradient included).  Returns 1 if the shape is not covered (the caller
// runs the fp32 kernels).
int cmgan_gemm_wgrad_tc_launch(const CmganGemmArgs* a, cudaStream_t st) {
    if (!wgrad_tc_supported(a)) return 1;
    if (a->M <= 0) return 0;
    int smem_sm, smem_blk;
    if (smem_limits(&smem_sm, &smem_blk)) return -1;
    if (taps_plan_fits(a)) return launch_taps(a, smem_blk, st);
    Plan p{};
    // orientation: the one that reads fewer bytes of A and D in total (every tile reads all rows of its columns)
    const long cost_x = (long)cdiv(a->Cin, PT) * (PT + a->N), cost_y = (long)cdiv(a->N, PT) * (a->Cin + PT);
    p.ydir = a->Cin <= QMAX && cost_y < cost_x;
    p.ptiles = p.ydir ? cdiv(a->N, PT) : cdiv(a->Cin, PT);
    p.qpad = (((p.ydir ? a->Cin : a->N) + 31) / 32) * 32;
    p.wa = p.ydir ? p.qpad : PT;
    p.wd = p.ydir ? PT : p.qpad;
    p.raw_bytes = (uint32_t)(RS * (p.wa + p.wd) * 4 + RS * 4 + RS * 8);
    p.img_bytes = (uint32_t)((PT + p.qpad) * 128);
    // two CTAs per SM when a ring of at least 3 slabs fits in half the shared memory, else one CTA with a deeper ring
    long ring = (smem_sm / 2 - 2048 - 2L * p.img_bytes) / p.raw_bytes;     // per-CTA reservation + alignment slack + the two images
    if (ring < 3) ring = (smem_blk - 1024 - 2L * p.img_bytes) / p.raw_bytes;
    if (ring < 3) { cmgan_set_error("gemm_wgrad_tc: %d x %d tile does not fit in shared memory", PT, p.qpad); return -1; }
    p.ring = ring > MAX_RING ? MAX_RING : (int)ring;
    const size_t smem = 1024 + 2 * (size_t)p.img_bytes + (size_t)p.ring * p.raw_bytes;
    switch (p.qpad / 32) {
        case 1: return launch<1>(a, p, smem, smem_blk, st);
        case 2: return launch<2>(a, p, smem, smem_blk, st);
        case 3: return launch<3>(a, p, smem, smem_blk, st);
        case 4: return launch<4>(a, p, smem, smem_blk, st);
        case 5: return launch<5>(a, p, smem, smem_blk, st);
        case 6: return launch<6>(a, p, smem, smem_blk, st);
        case 7: return launch<7>(a, p, smem, smem_blk, st);
        default: return launch<8>(a, p, smem, smem_blk, st);
    }
}
