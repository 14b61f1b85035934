// Fused macaron feed-forward of the conformer block (reference conformer.py:54-72,136-148,211-212) for sm_90a:
//
//     out = x + alpha * drop2( W2 ( swish(W1 LN(x) + b1) * drop1 ) + b2 )                alpha = 0.5, C = 64, hidden = 256
//
// Both kernels run a persistent CTA per SM with TWO consumer warpgroups that share the CTA's resident weight images (K-major
// SWIZZLE_128B tf32) and walk different 64-row tiles: consumer w of CTA b takes tiles b + gridDim.x (2 k + w).  The two synchronise
// only through their own named barriers, so while one is in its Swish / dropout epilogue the other issues its loads and MMAs.
//
// Forward: ONE kernel, both weight images (2 x 64 KB) resident.  Per consumer and tile: LayerNorm (two threads per row) -> the
// normalised tile as the A operand -> per 128-column half of the hidden layer: wgmma into a 64 x 128 register accumulator -> bias,
// Swish, dropout, tf32 rounding -> the half as the A operand (32 KB of shared memory per consumer; it never reaches HBM) of K chunks
// 4 hf .. 4 hf + 3 of the second contraction into one 64 x 64 accumulator, so its K order is that of the whole hidden layer -> bias,
// dropout, alpha, residual -> store.  Only the module input is kept for the backward pass.
//
// Backward: ONE kernel, three weight images (3 x 64 KB) resident.  It recomputes the hidden pre-activation h (LN + first contraction,
// xn from shared memory) and forms dh = (dz W2) * swish'(h) * drop1 one 64-column quarter of the hidden layer at a time (two 64 x 64
// accumulators in registers; dz, already a tf32 operand, is loaded straight into register A fragments, which leaves room for two
// consumers' xn tiles), writing the operands of the two weight-gradient GEMMs (xn, a = swish(h) * drop1, dh) and the LayerNorm
// statistics.  The rounded dh quarter stays in registers as the A operand of dLN += dh_q W1_q (a third 64 x 64 accumulator; W1^T is the
// third image), and the LayerNorm backward runs on that accumulator in the same consumer, so neither dh nor dLN is read back from HBM.
// Dropout masks are the counter-based hash of the GEMM epilogues (csrc/gemm_tc.cu): pair (m * N + n) / 2, 16 bits per element.
#include "common.cuh"
#include "../../include/cmgan_b200.h"
#include "tc_ptx.cuh"

namespace {
using namespace cmgan_tc;

constexpr int BM = 64, C = 64, HID = 256;
constexpr int NT = 128;                         // one consumer warpgroup
constexpr int NCONS = 2, NTHR = NCONS * NT;     // two consumers per CTA, each on its own 64-row tiles
constexpr int CHUNK = BM * 128;                 // 64 rows x 32 floats = 8 KB
constexpr int W_BYTES = 64 * 1024;              // one packed 64 x 256 weight image

// barrier of one consumer's 128 threads (id 0 is __syncthreads')
__device__ __forceinline__ void consumer_sync(int w) { asm volatile("bar.sync %0, %1;" ::"r"(1 + w), "n"(NT) : "memory"); }

// byte offset of (row r, float column c of a 32-float chunk) in a K-major SWIZZLE_128B chunk
__device__ __forceinline__ uint32_t swz(int r, int c) { return (uint32_t)(r * 128 + ((((c >> 2) ^ r) & 7) << 4) + (c & 3) * 4); }

// dropout scales of the element pair (m, n), (m, n + 1), n even
__device__ __forceinline__ float2 drop_pair(long m, int n, int N, uint32_t seed32, uint32_t thr16, float inv_keep, bool on) {
    if (!on) return make_float2(1.f, 1.f);
    const uint32_t pr = (uint32_t)(((unsigned long long)m * (unsigned long long)N + (unsigned long long)n) >> 1);
    const uint32_t h = cmgan_mix32((pr * 0x9E3779B1u) ^ seed32);
    return make_float2((h & 0xFFFFu) >= thr16 ? inv_keep : 0.f, (h >> 16) >= thr16 ? inv_keep : 0.f);
}

__device__ __forceinline__ void copy_image(uint8_t* dst, const float* src, int bytes) {
    const uint4* s = reinterpret_cast<const uint4*>(src);
    uint4* d = reinterpret_cast<uint4*>(dst);
    for (int i = threadIdx.x; i < bytes / 16; i += NTHR) d[i] = __ldg(s + i);
}

// LayerNorm of the tile's rows (two threads per row, 32 channels each; t: thread of the consumer) -> tf32 A operand (2 chunks); rows
// past M are zero.  Returns (mean, rstd) of the thread's row.
__device__ __forceinline__ float2 ln_tile(const float* __restrict__ x, long ldx, long m0, long M, const float* __restrict__ g,
                                          const float* __restrict__ b, uint8_t* sXn, float* xn_out, int t) {
    const int r = t >> 1, half = t & 1;
    const long m = m0 + r;
    float v[32];
#pragma unroll
    for (int q = 0; q < 8; ++q) {
        float4 t = m < M ? __ldg(reinterpret_cast<const float4*>(x + m * ldx + half * 32 + 4 * q)) : make_float4(0.f, 0.f, 0.f, 0.f);
        v[4 * q] = t.x; v[4 * q + 1] = t.y; v[4 * q + 2] = t.z; v[4 * q + 3] = t.w;
    }
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < 32; ++i) s += v[i];
    s += __shfl_xor_sync(0xffffffffu, s, 1);
    const float mean = s * (1.f / C);
    float q2 = 0.f;
#pragma unroll
    for (int i = 0; i < 32; ++i) { const float d = v[i] - mean; q2 += d * d; }
    q2 += __shfl_xor_sync(0xffffffffu, q2, 1);
    const float rstd = rsqrtf(q2 * (1.f / C) + 1e-5f);
#pragma unroll
    for (int q = 0; q < 8; ++q) {
        float o[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int c = half * 32 + 4 * q + j;
            o[j] = m < M ? to_tf32((v[4 * q + j] - mean) * rstd * __ldg(g + c) + __ldg(b + c)) : 0.f;
        }
        *reinterpret_cast<float4*>(sXn + half * CHUNK + swz(r, 4 * q)) = make_float4(o[0], o[1], o[2], o[3]);
        if (xn_out && m < M) *reinterpret_cast<float4*>(xn_out + m * C + half * 32 + 4 * q) = make_float4(o[0], o[1], o[2], o[3]);
    }
    return make_float2(mean, rstd);
}

// one 32-float K chunk (4 K steps) into 64 x (64 NB) accumulators, one m64n64k8 instruction per 64 columns: the A rows are read from
// shared memory once per 64 columns instead of once per 16.  Same fragment layout as mma_chunk<4 NB> (acc[4 b + c] = columns 64 b + 16 c ..).
template <int NB>
__device__ __forceinline__ void mma_chunk64(float (&acc)[4 * NB][8], uint64_t adesc, uint64_t bdesc, bool first) {
#pragma unroll
    for (int k = 0; k < 4; ++k)
#pragma unroll
        for (int b = 0; b < NB; ++b)
            wgmma_m64n64k8_tf32(*reinterpret_cast<float(*)[4][8]>(&acc[4 * b]), adesc + (uint64_t)(2 * k), bdesc + (uint64_t)(512 * b + 2 * k),
                                (first && k == 0) ? 0u : 1u);
}

// start pulling the rows [m0, m0 + 64) of an array into L2 ahead of their use: one 128-byte line per thread of the consumer
__device__ __forceinline__ void prefetch_rows_l2(const float* p, long ld, long m0, long M, int t) {
    const long m = m0 + (t >> 1);
    if (m < M) asm volatile("prefetch.global.L2 [%0];" ::"l"(p + m * ld + (t & 1) * 32));
}

struct FfnFwdArgs {
    const float* x; long long ldx; float* out; long long ldo;
    const float* ln_g; const float* ln_b; const float* W1p; const float* b1; const float* W2p; const float* b2;
    long long M; float alpha; unsigned long long seed1, seed2; unsigned int thr; float inv_keep; const unsigned long long* seed_dev;
};

__global__ void __launch_bounds__(NTHR, 1) ffn_fwd_kernel(const __grid_constant__ FfnFwdArgs g) {
    extern __shared__ uint8_t smem_raw[];
    const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;
    uint8_t* const bp = smem_raw + (base - smem_u32(smem_raw));
    uint8_t* const sW1 = bp;                       // 2 chunks x 256 rows
    uint8_t* const sW2 = bp + W_BYTES;             // 8 chunks x 64 rows
    const int w = threadIdx.x / NT, t = threadIdx.x % NT;
    const uint32_t xa = base + 2 * W_BYTES + w * 6 * CHUNK, ha = xa + 2 * CHUNK;
    uint8_t* const sXn = bp + (xa - base);         // the consumer's 2 chunks x 64 rows
    uint8_t* const sH = bp + (ha - base);          // the consumer's hidden half: 4 chunks x 64 rows
    const int warp = t >> 5, lane = t & 31, fg = lane >> 2, ft = lane & 3;
    const bool drop_on = g.thr != 0u;
    const uint32_t thr16 = g.thr >> 16;
    const uint32_t s1 = cmgan_seed32(cmgan_eff_seed(g.seed1, g.seed_dev)), s2 = cmgan_seed32(cmgan_eff_seed(g.seed2, g.seed_dev));
    copy_image(sW1, g.W1p, W_BYTES);
    copy_image(sW2, g.W2p, W_BYTES);
    fence_proxy_async();
    __syncthreads();
    const long ntiles = (g.M + BM - 1) / BM, stride = (long)NCONS * gridDim.x;
    for (long tile = blockIdx.x + (long)w * gridDim.x; tile < ntiles; tile += stride) {
        const long m0 = tile * BM;
        prefetch_rows_l2(g.x, g.ldx, m0 + stride * BM, g.M, t);       // the consumer's next tile
        ln_tile(g.x, g.ldx, m0, g.M, g.ln_g, g.ln_b, sXn, nullptr, t);
        fence_proxy_async();
        consumer_sync(w);
        // the hidden layer one 128-column half at a time; the second contraction adds its K chunks in the same order as a whole tile
        float acc2[4][8];
#pragma unroll
        for (int hf = 0; hf < 2; ++hf) {
            float acc[8][8];
            wgmma_fence();
            mma_chunk64<2>(acc, gmma_desc_sw128(xa), gmma_desc_sw128(base + hf * 128 * 128), true);
            mma_chunk64<2>(acc, gmma_desc_sw128(xa + CHUNK), gmma_desc_sw128(base + 256 * 128 + hf * 128 * 128), false);
            wgmma_commit();
            wgmma_wait<0>();              // for hf = 1 also the second contraction of half 0, the last reader of sH
            if (hf == 1) consumer_sync(w);
            // hidden activation -> second A operand (fragment rows 16 warp + fg (+ 8), columns 128 hf + 16 j + 8 i + 2 ft (+ 1))
#pragma unroll
            for (int j = 0; j < 8; ++j)
#pragma unroll
                for (int i = 0; i < 2; ++i)
#pragma unroll
                    for (int hh = 0; hh < 2; ++hh) {
                        const int r = 16 * warp + fg + 8 * hh, n = 128 * hf + 16 * j + 8 * i + 2 * ft;
                        const float2 bb = __ldg(reinterpret_cast<const float2*>(g.b1 + n));
                        const float2 ds = drop_pair(m0 + r, n, HID, s1, thr16, g.inv_keep, drop_on);
                        const float h0 = acc[j][4 * i + 2 * hh] + bb.x, h1 = acc[j][4 * i + 2 * hh + 1] + bb.y;
                        *reinterpret_cast<float2*>(sH + ((n >> 5) - 4 * hf) * CHUNK + swz(r, n & 31)) =
                            make_float2(to_tf32(swishf_(h0) * ds.x), to_tf32(swishf_(h1) * ds.y));
                    }
            fence_proxy_async();
            consumer_sync(w);
            wgmma_fence();
#pragma unroll
            for (int c = 0; c < 4; ++c)
                mma_chunk64<1>(acc2, gmma_desc_sw128(ha + c * CHUNK), gmma_desc_sw128(base + W_BYTES + (4 * hf + c) * CHUNK), hf == 0 && c == 0);
            wgmma_commit();
        }
        wgmma_wait<0>();
#pragma unroll
        for (int j = 0; j < 4; ++j)
#pragma unroll
            for (int i = 0; i < 2; ++i)
#pragma unroll
                for (int hh = 0; hh < 2; ++hh) {
                    const long m = m0 + 16 * warp + fg + 8 * hh;
                    if (m >= g.M) continue;
                    const int n = 16 * j + 8 * i + 2 * ft;
                    const float2 bb = __ldg(reinterpret_cast<const float2*>(g.b2 + n));
                    const float2 ds = drop_pair(m, n, C, s2, thr16, g.inv_keep, drop_on);
                    const float2 xr = __ldg(reinterpret_cast<const float2*>(g.x + m * g.ldx + n));
                    *reinterpret_cast<float2*>(g.out + m * g.ldo + n) =
                        make_float2(xr.x + g.alpha * (acc2[j][4 * i + 2 * hh] + bb.x) * ds.x, xr.y + g.alpha * (acc2[j][4 * i + 2 * hh + 1] + bb.y) * ds.y);
                }
        // no barrier: sXn's last readers were waited for before half 1's barrier, sH's are waited for above and the next tile's
        // barrier after its LayerNorm orders them before its first write to sH
    }
}

struct FfnBwdArgs {
    const float* x; long long ldx; const float* dz; long long lddz; const float* dout; long long lddo; const float* res2; long long ldr2;
    const float* ln_g; const float* ln_b; const float* W1p; const float* b1; const float* W2tp; const float* W1tp;
    long long M; unsigned long long seed1; unsigned int thr; float inv_keep; const unsigned long long* seed_dev;
    float* a_out; float* dh_out; float* xn_out; float* stats; float* dx; long long lddx; float* dgamma; float* dbeta;
};

// The W1^T image (64 channel rows x 256 hidden, K-major SWIZZLE_128B) with K permuted inside each group of 8, so that the rounded dh
// accumulator fragment is the register A operand of dLN = dh W1 as it stands: a thread holds hidden columns 2 t, 2 t + 1 of a group,
// where the A fragment wants columns t, t + 4, so slot s of a group holds hidden column 2 s (s < 4) or 2 (s - 4) + 1.
__device__ __forceinline__ void copy_image_kperm(uint8_t* dst, const float* __restrict__ src) {
    for (int u = threadIdx.x; u < W_BYTES / 16; u += NTHR) {
        const int c = u >> 9, n = (u >> 3) & 63, cu = u & 7;     // chunk, row, 16-byte unit (slots 4 cu .. 4 cu + 3) of the row
        float v[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int k = 8 * (cu >> 1) + 2 * j + (cu & 1);
            v[j] = __ldg(src + c * (CHUNK / 4) + n * 32 + (((k >> 2) ^ (n & 7)) << 2) + (k & 3));
        }
        *reinterpret_cast<float4*>(dst + c * CHUNK + swz(n, 4 * cu)) = make_float4(v[0], v[1], v[2], v[3]);
    }
}

// one 64-column quarter of the hidden layer: h (acc) = xn W1^T (xn at xa in shared memory) and dz W2 (dacc; dz as register A fragments)
// on hidden columns 64 qt .. 64 qt + 63
__device__ __forceinline__ void bwd_quarter_mmas(float (&acc)[4][8], float (&dacc)[4][8], const uint32_t (&dzf)[8][4], uint32_t base, uint32_t xa,
                                                 int qt) {
    const uint32_t wrow = (uint32_t)qt * 64 * 128;
    mma_chunk64<1>(acc, gmma_desc_sw128(xa), gmma_desc_sw128(base + wrow), true);
    mma_chunk64<1>(acc, gmma_desc_sw128(xa + CHUNK), gmma_desc_sw128(base + 256 * 128 + wrow), false);
    const uint64_t bdesc = gmma_desc_sw128(base + W_BYTES + wrow);
#pragma unroll
    for (int kk = 0; kk < 8; ++kk)
        wgmma_m64n64k8_tf32_rs(dacc, dzf[kk], bdesc + (uint64_t)((kk >> 2) * (256 * 128 >> 4) + 2 * (kk & 3)), kk > 0 ? 1u : 0u);
}

// Per 64-row tile: LayerNorm (xn, stats out), then per hidden quarter h and dz W2 -> a, dh out, and dLN += rna(dh) W1 with dh taken from
// registers; the quarter's dLN MMAs are issued together with the next quarter's.  Then the LayerNorm backward on the 64 x 64 dLN
// accumulator, row sums over the quad that holds a row: dx = rstd (dLN g - mean(dLN g) - xhat mean(dLN g xhat)) + dout (+ res2).
// dgamma / dbeta: per-thread column partials over the consumer's tiles, reduced in the CTA, one atomic per column per CTA.
__global__ void __launch_bounds__(NTHR, 1) ffn_bwd_kernel(const __grid_constant__ FfnBwdArgs g) {
    extern __shared__ uint8_t smem_raw[];
    const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;
    uint8_t* const bp = smem_raw + (base - smem_u32(smem_raw));
    uint8_t* const sW1 = bp;                       // W1 image: 2 chunks x 256 rows (h = xn W1^T)
    uint8_t* const sW2t = bp + W_BYTES;            // W2^T image: 2 chunks x 256 rows (dz W2)
    uint8_t* const sW1t = bp + 2 * W_BYTES;        // K-permuted W1^T image: 8 chunks x 64 rows (dLN = dh W1)
    const int w = threadIdx.x / NT, t = threadIdx.x % NT;
    const uint32_t xa = base + 3 * W_BYTES + w * 2 * CHUNK;
    uint8_t* const sXn = bp + (xa - base);         // the consumer's 2 chunks x 64 rows
    float2* const sStats = reinterpret_cast<float2*>(bp + 3 * W_BYTES + NCONS * 2 * CHUNK) + w * BM;     // the consumer's 64 x (mean, rstd)
    const int warp = t >> 5, lane = t & 31, fg = lane >> 2, ft = lane & 3;
    const bool drop_on = g.thr != 0u;
    const uint32_t thr16 = g.thr >> 16;
    const uint32_t s1 = cmgan_seed32(cmgan_eff_seed(g.seed1, g.seed_dev));
    copy_image(sW1, g.W1p, W_BYTES);
    copy_image(sW2t, g.W2tp, W_BYTES);
    copy_image_kperm(sW1t, g.W1tp);
    fence_proxy_async();
    __syncthreads();
    float pg[4][4], pb[4][4];                      // dgamma / dbeta partials of columns 16 j + 8 (e >> 1) + 2 ft + (e & 1)
#pragma unroll
    for (int j = 0; j < 4; ++j)
#pragma unroll
        for (int e = 0; e < 4; ++e) pg[j][e] = pb[j][e] = 0.f;
    const long ntiles = (g.M + BM - 1) / BM, stride = (long)NCONS * gridDim.x;
    for (long tile = blockIdx.x + (long)w * gridDim.x; tile < ntiles; tile += stride) {
        const long m0 = tile * BM, mn = m0 + stride * BM;                // mn: the consumer's next tile
        prefetch_rows_l2(g.x, g.ldx, mn, g.M, t);
        prefetch_rows_l2(g.dz, g.lddz, mn, g.M, t);
        prefetch_rows_l2(g.dout, g.lddo, mn, g.M, t);
        if (g.res2) prefetch_rows_l2(g.res2, g.ldr2, mn, g.M, t);
        const float2 st = ln_tile(g.x, g.ldx, m0, g.M, g.ln_g, g.ln_b, sXn, g.xn_out, t);
        if ((t & 1) == 0) {   // statistics for the LayerNorm backward
            const long m = m0 + (t >> 1);
            sStats[t >> 1] = st;
            if (m < g.M) reinterpret_cast<float2*>(g.stats)[m] = st;
        }
        // dz (already a tf32 operand) straight into the A fragments of the 8 K steps of dz W2; rows past M are zero
        uint32_t dzf[8][4];
#pragma unroll
        for (int hh = 0; hh < 2; ++hh) {
            const long m = m0 + 16 * warp + fg + 8 * hh;
#pragma unroll
            for (int kk = 0; kk < 8; ++kk)
#pragma unroll
                for (int e = 0; e < 2; ++e)
                    dzf[kk][hh + 2 * e] = m < g.M ? __float_as_uint(__ldg(g.dz + m * g.lddz + 8 * kk + ft + 4 * e)) : 0u;
        }
        fence_proxy_async();
        consumer_sync(w);
        float acc[4][8], dacc[4][8], dln[4][8];
        wgmma_fence();
        bwd_quarter_mmas(acc, dacc, dzf, base, xa, 0);
        wgmma_commit();
        wgmma_wait<0>();
        uint32_t dha[8][4];                        // rna(dh) as the A fragments of the quarter's 8 K steps (columns permuted as sW1t)
        // a, dh of quarter qt out, then its dLN MMAs issued
        auto quarter_dh = [&](int qt) {
#pragma unroll
            for (int j = 0; j < 4; ++j)
#pragma unroll
                for (int i = 0; i < 2; ++i)
#pragma unroll
                    for (int hh = 0; hh < 2; ++hh) {
                        const long m = m0 + 16 * warp + fg + 8 * hh;
                        const int n = 64 * qt + 16 * j + 8 * i + 2 * ft;
                        const float2 bb = __ldg(reinterpret_cast<const float2*>(g.b1 + n));
                        const float2 ds = drop_pair(m, n, HID, s1, thr16, g.inv_keep, drop_on);
                        const float h0 = acc[j][4 * i + 2 * hh] + bb.x, h1 = acc[j][4 * i + 2 * hh + 1] + bb.y;
                        // rows past M have xn = dz = 0, so their dh is 0 and they add nothing to dLN
                        const float d0 = to_tf32(dacc[j][4 * i + 2 * hh] * dswishf_(h0) * ds.x);
                        const float d1 = to_tf32(dacc[j][4 * i + 2 * hh + 1] * dswishf_(h1) * ds.y);
                        dha[2 * j + i][hh] = __float_as_uint(d0);
                        dha[2 * j + i][2 + hh] = __float_as_uint(d1);
                        if (m >= g.M) continue;
                        *reinterpret_cast<float2*>(g.a_out + m * HID + n) = make_float2(to_tf32(swishf_(h0) * ds.x), to_tf32(swishf_(h1) * ds.y));
                        *reinterpret_cast<float2*>(g.dh_out + m * HID + n) = make_float2(d0, d1);
                    }
            wgmma_fence();
            const uint64_t bdesc = gmma_desc_sw128(base + 2 * W_BYTES + 2 * qt * CHUNK);
#pragma unroll
            for (int kk = 0; kk < 8; ++kk)
                wgmma_m64n64k8_tf32_rs(dln, dha[kk], bdesc + (uint64_t)((kk >> 2) * (CHUNK >> 4) + 2 * (kk & 3)), (qt > 0 || kk > 0) ? 1u : 0u);
        };
        // the last quarter is peeled: a wgmma under a run-time branch would make ptxas serialize them
#pragma unroll 1
        for (int qt = 0; qt < 3; ++qt) {
            quarter_dh(qt);
            bwd_quarter_mmas(acc, dacc, dzf, base, xa, qt + 1);
            wgmma_commit();
            wgmma_wait<0>();
        }
        quarter_dh(3);
        wgmma_commit();
        wgmma_wait<0>();
        // LayerNorm backward, as ln_bwd_kernel: rows 16 warp + fg + 8 hh, 16 columns per thread, the row's 64 over the quad
#pragma unroll
        for (int hh = 0; hh < 2; ++hh) {
            const int r = 16 * warp + fg + 8 * hh;
            const long m = m0 + r;
            const bool ok = m < g.M;
            const float2 s = ok ? sStats[r] : make_float2(0.f, 0.f);
            float xh[4][4], dg[4][4], s1r = 0.f, s2r = 0.f;
#pragma unroll
            for (int j = 0; j < 4; ++j)
#pragma unroll
                for (int i = 0; i < 2; ++i) {
                    const int n = 16 * j + 8 * i + 2 * ft;
                    const float2 v = ok ? __ldg(reinterpret_cast<const float2*>(g.x + m * g.ldx + n)) : make_float2(0.f, 0.f);
                    const float2 gm = __ldg(reinterpret_cast<const float2*>(g.ln_g + n));
                    xh[j][2 * i] = (v.x - s.x) * s.y;
                    xh[j][2 * i + 1] = (v.y - s.x) * s.y;
                    dg[j][2 * i] = dln[j][4 * i + 2 * hh] * gm.x;
                    dg[j][2 * i + 1] = dln[j][4 * i + 2 * hh + 1] * gm.y;
                    s1r += dg[j][2 * i] + dg[j][2 * i + 1];
                    s2r += dg[j][2 * i] * xh[j][2 * i] + dg[j][2 * i + 1] * xh[j][2 * i + 1];
                }
            s1r += __shfl_xor_sync(0xffffffffu, s1r, 1);
            s1r += __shfl_xor_sync(0xffffffffu, s1r, 2);
            s2r += __shfl_xor_sync(0xffffffffu, s2r, 1);
            s2r += __shfl_xor_sync(0xffffffffu, s2r, 2);
            const float m1 = s1r * (1.0f / C), m2 = s2r * (1.0f / C);
#pragma unroll
            for (int j = 0; j < 4; ++j)
#pragma unroll
                for (int i = 0; i < 2; ++i) {
                    const int n = 16 * j + 8 * i + 2 * ft;
                    if (ok) {
                        float2 rr = __ldg(reinterpret_cast<const float2*>(g.dout + m * g.lddo + n));
                        if (g.res2) {
                            const float2 r2 = __ldg(reinterpret_cast<const float2*>(g.res2 + m * g.ldr2 + n));
                            rr.x += r2.x; rr.y += r2.y;
                        }
                        *reinterpret_cast<float2*>(g.dx + m * g.lddx + n) =
                            make_float2(s.y * (dg[j][2 * i] - m1 - xh[j][2 * i] * m2) + rr.x, s.y * (dg[j][2 * i + 1] - m1 - xh[j][2 * i + 1] * m2) + rr.y);
                    }
#pragma unroll
                    for (int e = 0; e < 2; ++e) {
                        const float d = dln[j][4 * i + 2 * hh + e];
                        pg[j][2 * i + e] = fmaf(d, xh[j][2 * i + e], pg[j][2 * i + e]);
                        pb[j][2 * i + e] += d;
                    }
                }
        }
        consumer_sync(w);         // sXn / sStats are rewritten by the next tile
    }
    // dgamma / dbeta: over the 8 row groups of the warp (butterfly), the 8 warps of the CTA (pairwise), then one atomic per column
    float* const red = reinterpret_cast<float*>(bp + 3 * W_BYTES);          // [warp][dgamma 64 | dbeta 64] over consumer 0's xn tile
    const int cw = threadIdx.x >> 5;
    __syncthreads();
#pragma unroll
    for (int j = 0; j < 4; ++j)
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            float a = pg[j][e], b = pb[j][e];
#pragma unroll
            for (int o = 4; o < 32; o <<= 1) {
                a += __shfl_xor_sync(0xffffffffu, a, o);
                b += __shfl_xor_sync(0xffffffffu, b, o);
            }
            if (fg == 0) {
                const int n = 16 * j + 8 * (e >> 1) + 2 * ft + (e & 1);
                red[cw * 2 * C + n] = a;
                red[cw * 2 * C + C + n] = b;
            }
        }
    __syncthreads();
    if (threadIdx.x < C) {
        const int n = threadIdx.x;
        float v[2][NTHR / 32];
#pragma unroll
        for (int u = 0; u < NTHR / 32; ++u) v[0][u] = red[u * 2 * C + n], v[1][u] = red[u * 2 * C + C + n];
#pragma unroll
        for (int o = 1; o < NTHR / 32; o <<= 1)
#pragma unroll
            for (int u = 0; u < NTHR / 32; u += 2 * o) v[0][u] += v[0][u + o], v[1][u] += v[1][u + o];
        atomicAdd(g.dgamma + n, v[0][0]);
        atomicAdd(g.dbeta + n, v[1][0]);
    }
}

template <typename K>
int prepare(K kernel, size_t smem, const char* name) {
    static bool set = false;
    if (!set) {
        cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) { cmgan_set_error("%s: cudaFuncSetAttribute: %s", name, cudaGetErrorString(e)); return -1; }
        set = true;
    }
    return 0;
}

}  // namespace

// out = x + alpha * drop2(W2 (swish(W1 LN(x) + b1) * drop1) + b2); W1p / W2p: cmgan_pack_weight images of W1 (256 x 64) and W2 (64 x 256)
CMGAN_API int cmgan_ffn_fwd(const float* x, long long ldx, long long M, const float* ln_g, const float* ln_b, const float* W1p, const float* b1,
                            const float* W2p, const float* b2, float alpha, unsigned long long seed1, unsigned long long seed2, unsigned int thr,
                            float inv_keep, const unsigned long long* seed_dev, float* out, long long ldo, void* stream) {
    CMGAN_REQUIRE(x && out && ln_g && ln_b && W1p && b1 && W2p && b2 && M >= 0 && ldx % 4 == 0 && ldo % 2 == 0, "cmgan_ffn_fwd: bad arguments");
    if (M == 0) return 0;
    const size_t smem = 1024 + 2 * W_BYTES + NCONS * (2 * CHUNK + 4 * CHUNK);
    if (prepare(ffn_fwd_kernel, smem, "ffn_fwd_kernel")) return -1;
    FfnFwdArgs a{x, ldx, out, ldo, ln_g, ln_b, W1p, b1, W2p, b2, M, alpha, seed1, seed2, thr, inv_keep, seed_dev};
    const long ntiles = (M + BM - 1) / BM, half_tiles = (ntiles + 1) / 2;       // one tile per consumer and pass
    const int grid = (int)(half_tiles < cmgan_num_sms() ? half_tiles : cmgan_num_sms());
    ffn_fwd_kernel<<<grid, NTHR, smem, (cudaStream_t)stream>>>(a);
    return cmgan_check_launch("ffn_fwd_kernel");
}

// Data gradients of the feed-forward from its input x and dz = alpha * drop2-mask * dout (a tf32 operand): dx = LN-backward(dh W1) + dout
// (+ res2), dgamma / dbeta accumulated; leaves the weight-gradient operands a = swish(h) * drop1, dh and xn.  W1p: image of W1,
// W2tp: image of W2 read transposed (256 x 64), W1tp: image of W1 read transposed (64 x 256).  ws: M * 66 floats of scratch.
CMGAN_API int cmgan_ffn_bwd(const float* x, long long ldx, const float* dz, long long lddz, const float* dout, long long lddo, const float* res2,
                            long long ldr2, long long M, const float* ln_g, const float* ln_b, const float* W1p, const float* b1, const float* W2tp,
                            const float* W1tp, unsigned long long seed1, unsigned int thr, float inv_keep, const unsigned long long* seed_dev,
                            float* dx, long long lddx, float* a_out, float* dh_out, float* xn_out, float* dgamma, float* dbeta, float* ws,
                            void* stream) {
    CMGAN_REQUIRE(x && dz && dout && ln_g && ln_b && W1p && b1 && W2tp && W1tp && dx && a_out && dh_out && xn_out && dgamma && dbeta && ws && M >= 0 &&
                  ldx % 4 == 0 && lddz % 4 == 0, "cmgan_ffn_bwd: bad arguments");
    CMGAN_REQUIRE(lddo % 2 == 0 && (!res2 || ldr2 % 2 == 0) && lddx % 2 == 0, "cmgan_ffn_bwd: bad arguments");
    if (M == 0) return 0;
    const size_t smem = 1024 + 3 * W_BYTES + NCONS * (2 * CHUNK + BM * sizeof(float2));
    if (prepare(ffn_bwd_kernel, smem, "ffn_bwd_kernel")) return -1;
    float* stats = ws + C * M;       // M x (mean, rstd); ws[0, 64 M) is unused
    FfnBwdArgs a{x, ldx, dz, lddz, dout, lddo, res2, res2 ? ldr2 : 0, ln_g, ln_b, W1p, b1, W2tp, W1tp, M, seed1, thr, inv_keep, seed_dev,
                 a_out, dh_out, xn_out, stats, dx, lddx, dgamma, dbeta};
    // At most ceil(ntiles / 2) CTAs, so while grid < SMs each consumer has at most one tile.  A consumer adds the dgamma / dbeta terms
    // of its rows in a chain of 2 T (T = its tiles) and 3 butterfly adds, the CTA's 8 warps are summed pairwise (3 adds), then one
    // atomic: a term sees at most 2 T + 7 + grid roundings.  With X = ceil(M / 128) >= grid that is never longer than ln_bwd_kernel's
    // 8 + 16 + X: T <= 1 while grid < SMs, and when grid = SMs (X >= SMs), T = ceil(ntiles / (2 SMs)) <= ceil(X / SMs), so
    // 2 T + 7 + SMs <= 24 + X (2 ceil(X / SMs) grows by 2 for every SMs that X grows by).
    const long ntiles = (M + BM - 1) / BM, half_tiles = (ntiles + 1) / 2;
    const int grid = (int)(half_tiles < cmgan_num_sms() ? half_tiles : cmgan_num_sms());
    ffn_bwd_kernel<<<grid, NTHR, smem, (cudaStream_t)stream>>>(a);
    return cmgan_check_launch("ffn_bwd_kernel");
}
