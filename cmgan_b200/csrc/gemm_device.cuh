// Device helpers shared by the FFMA (gemm_simt.cu) and wgmma (gemm_tc.cu) implementations of the GEMM contract
// in gemm_args.h: row decoding / implicit-convolution gather, A-operand prologues, epilogues.
#pragma once
#include "common.cuh"
#include "gemm_args.h"

namespace cmgan_gemm {

// dropout seeds: the per-site constant plus an optional device-resident step counter
__device__ __forceinline__ unsigned long long eff_seed(const CmganGemmArgs& g) { return cmgan_eff_seed(g.seed, g.seed_dev); }
__device__ __forceinline__ unsigned long long eff_pro_seed(const CmganGemmArgs& g) { return cmgan_eff_seed(g.pro_seed, g.seed_dev); }

struct RowInfo { int b, y, x; bool ok; };

__device__ __forceinline__ RowInfo decode_row(const CmganGemmArgs& g, int m) {
    RowInfo r;
    r.ok = m < g.M;
    if (g.conv) {
        int x = m % g.OW; int t = m / g.OW;
        r.x = x; r.y = t % g.OH; r.b = t / g.OH;
    } else { r.b = 0; r.y = 0; r.x = m; }
    return r;
}

// in_row for (row, tap) or -1 when the tap falls into padding / a stride hole
__device__ __forceinline__ long in_row_of(const CmganGemmArgs& g, const RowInfo& r, int tap) {
    if (!r.ok) return -1;
    if (!g.conv) return r.x;
    int iy = r.y * g.mul_y + g.dy[tap];
    int ix = r.x * g.mul_x + g.dx[tap];
    if (iy < 0 || ix < 0) return -1;
    if (g.div_y > 1) { if (iy % g.div_y) return -1; iy /= g.div_y; }
    if (g.div_x > 1) { if (ix % g.div_x) return -1; ix /= g.div_x; }
    if (iy >= g.IH || ix >= g.IW) return -1;
    return ((long)r.b * g.IH + iy) * g.IW + ix;
}

__device__ __forceinline__ float apply_pro(const CmganGemmArgs& g, float a, long r, int k, float mean, float rstd) {
    switch (g.pro) {
        case CMGAN_PRO_LN: return (a - mean) * rstd * __ldg(g.p1 + k) + __ldg(g.p2 + k);
        case CMGAN_PRO_SWISH_DROP: return swishf_(a) * cmgan_drop_scale(eff_pro_seed(g), (uint64_t)r * g.Cin + k, g.pro_thr, g.pro_inv_keep);
        case CMGAN_PRO_BN_SWISH: return swishf_(a * __ldg(g.p0 + k) + __ldg(g.p1 + k));
        case CMGAN_PRO_DROP: return a * g.pro_alpha * cmgan_drop_scale(eff_pro_seed(g), (uint64_t)r * g.Cin + k, g.pro_thr, g.pro_inv_keep);
        case CMGAN_PRO_IN_PRELU: {
            long b = r / g.rows_per_batch;
            float z = a * __ldg(g.p0 + b * g.pstride + k) + __ldg(g.p1 + b * g.pstride + k);
            return z >= 0.f ? z : z * __ldg(g.p2 + k);
        }
        default: return a;
    }
}

// loads 4 consecutive k of one A row (prologue applied); zeros where masked
template <int VEC>
__device__ __forceinline__ void load_a4(const CmganGemmArgs& g, long r, int tap, int k, float out[4]) {
    out[0] = out[1] = out[2] = out[3] = 0.f;
    if (r < 0 || k >= g.Cin) return;
    const float* p = g.A + g.tap_off[tap] + r * g.lda + k;
    float mean = 0.f, rstd = 0.f;
    if (g.pro == CMGAN_PRO_LN) { float2 st = __ldg(reinterpret_cast<const float2*>(g.p0) + r); mean = st.x; rstd = st.y; }
    if (VEC == 4 && k + 3 < g.Cin) {
        float4 v = __ldg(reinterpret_cast<const float4*>(p));
        out[0] = v.x; out[1] = v.y; out[2] = v.z; out[3] = v.w;
        if (g.pro != CMGAN_PRO_NONE) {
#pragma unroll
            for (int i = 0; i < 4; ++i) out[i] = apply_pro(g, out[i], r, k + i, mean, rstd);
        }
    } else {
#pragma unroll
        for (int i = 0; i < 4; ++i)
            if (k + i < g.Cin) out[i] = apply_pro(g, __ldg(p + i), r, k + i, mean, rstd);
    }
}

__device__ __forceinline__ float epilogue(const CmganGemmArgs& g, float v, long m, int n, const float* cptr) {
    switch (g.epi) {
        case CMGAN_EPI_DROP_RES: {
            float o = g.alpha * v * cmgan_drop_scale(eff_seed(g), (uint64_t)m * g.N + n, g.drop_thr, g.inv_keep);
            if (g.R) o += __ldg(g.R + m * g.ldr + n);
            return o;
        }
        case CMGAN_EPI_DSWISH_DROP: {
            float h = __ldg(g.aux + m * g.ldaux + n);
            return v * dswishf_(h) * cmgan_drop_scale(eff_seed(g), (uint64_t)m * g.N + n, g.drop_thr, g.inv_keep);
        }
        case CMGAN_EPI_DBNSWISH: {
            float z = __ldg(g.aux + m * g.ldaux + n) * __ldg(g.e0 + n) + __ldg(g.e1 + n);
            return v * dswishf_(z);
        }
        case CMGAN_EPI_ACC: return g.alpha * v + *cptr;
        default: return v;
    }
}


// ---- prologue on 4 consecutive k with hoisted per-chunk parameters -----------------------------------
struct ChunkParams { float4 a, b; };     // LN: gamma, beta;  BN: scale, shift

__device__ __forceinline__ void load_chunk_params(const CmganGemmArgs& g, int k, ChunkParams& cp) {
    if (g.pro == CMGAN_PRO_LN) { cp.a = __ldg(reinterpret_cast<const float4*>(g.p1 + k)); cp.b = __ldg(reinterpret_cast<const float4*>(g.p2 + k)); }
    else if (g.pro == CMGAN_PRO_BN_SWISH) { cp.a = __ldg(reinterpret_cast<const float4*>(g.p0 + k)); cp.b = __ldg(reinterpret_cast<const float4*>(g.p1 + k)); }
}

__device__ __forceinline__ float4 transform4(const CmganGemmArgs& g, float4 v, long r, int k, float mean, float rstd, const ChunkParams& cp) {
    switch (g.pro) {
        case CMGAN_PRO_LN:
            v.x = (v.x - mean) * rstd * cp.a.x + cp.b.x; v.y = (v.y - mean) * rstd * cp.a.y + cp.b.y;
            v.z = (v.z - mean) * rstd * cp.a.z + cp.b.z; v.w = (v.w - mean) * rstd * cp.a.w + cp.b.w;
            break;
        case CMGAN_PRO_BN_SWISH:
            v.x = swishf_(fmaf(v.x, cp.a.x, cp.b.x)); v.y = swishf_(fmaf(v.y, cp.a.y, cp.b.y));
            v.z = swishf_(fmaf(v.z, cp.a.z, cp.b.z)); v.w = swishf_(fmaf(v.w, cp.a.w, cp.b.w));
            break;
        case CMGAN_PRO_SWISH_DROP: {
            v.x = swishf_(v.x); v.y = swishf_(v.y); v.z = swishf_(v.z); v.w = swishf_(v.w);
            if (g.pro_thr) {
                float ds[4];
                cmgan_drop_scale4(eff_pro_seed(g), (uint64_t)r * g.Cin + k, g.pro_thr, g.pro_inv_keep, ds);
                v.x *= ds[0]; v.y *= ds[1]; v.z *= ds[2]; v.w *= ds[3];
            }
            break;
        }
        case CMGAN_PRO_DROP: {
            float ds[4];
            cmgan_drop_scale4(eff_pro_seed(g), (uint64_t)r * g.Cin + k, g.pro_thr, g.pro_inv_keep, ds);
            v.x *= g.pro_alpha * ds[0]; v.y *= g.pro_alpha * ds[1]; v.z *= g.pro_alpha * ds[2]; v.w *= g.pro_alpha * ds[3];
            break;
        }
        case CMGAN_PRO_IN_PRELU: {
            long b = r / g.rows_per_batch;
            const float4 sc = __ldg(reinterpret_cast<const float4*>(g.p0 + b * g.pstride + k));
            const float4 sh = __ldg(reinterpret_cast<const float4*>(g.p1 + b * g.pstride + k));
            const float4 sl = __ldg(reinterpret_cast<const float4*>(g.p2 + k));
            v.x = fmaf(v.x, sc.x, sh.x); v.y = fmaf(v.y, sc.y, sh.y); v.z = fmaf(v.z, sc.z, sh.z); v.w = fmaf(v.w, sc.w, sh.w);
            v.x = v.x >= 0.f ? v.x : v.x * sl.x; v.y = v.y >= 0.f ? v.y : v.y * sl.y;
            v.z = v.z >= 0.f ? v.z : v.z * sl.z; v.w = v.w >= 0.f ? v.w : v.w * sl.w;
            break;
        }
        default: break;
    }
    return v;
}

// ---- vectorised epilogue on 4 consecutive columns; `ex` = the pre-loaded auxiliary operand of the same 4 positions
// (R for DROP_RES, aux for DSWISH_DROP / DBNSWISH, the old C for ACC), `e0v`/`e1v` = per-column scale/shift (DBNSWISH)
__device__ __forceinline__ bool epi_needs_extra(const CmganGemmArgs& g) {
    return (g.epi == CMGAN_EPI_DROP_RES && g.R != nullptr) || g.epi == CMGAN_EPI_DSWISH_DROP || g.epi == CMGAN_EPI_DBNSWISH || g.epi == CMGAN_EPI_ACC;
}
__device__ __forceinline__ const float* epi_extra_ptr(const CmganGemmArgs& g, long m, int n) {
    switch (g.epi) {
        case CMGAN_EPI_DROP_RES: return g.R + m * g.ldr + n;
        case CMGAN_EPI_DSWISH_DROP:
        case CMGAN_EPI_DBNSWISH: return g.aux + m * g.ldaux + n;
        default: return g.C + m * g.ldc + n;
    }
}
__device__ __forceinline__ void epilogue4(const CmganGemmArgs& g, float v[4], long m, int n, const float4& ex, const float4& e0v, const float4& e1v) {
    const float x[4] = {ex.x, ex.y, ex.z, ex.w};
    switch (g.epi) {
        case CMGAN_EPI_DROP_RES: {
            float ds[4];
            cmgan_drop_scale4(eff_seed(g), (uint64_t)m * g.N + n, g.drop_thr, g.inv_keep, ds);
#pragma unroll
            for (int j = 0; j < 4; ++j) v[j] = g.alpha * v[j] * ds[j] + (g.R ? x[j] : 0.f);
            break;
        }
        case CMGAN_EPI_DSWISH_DROP: {
            float ds[4];
            cmgan_drop_scale4(eff_seed(g), (uint64_t)m * g.N + n, g.drop_thr, g.inv_keep, ds);
#pragma unroll
            for (int j = 0; j < 4; ++j) v[j] = v[j] * dswishf_(x[j]) * ds[j];
            break;
        }
        case CMGAN_EPI_DBNSWISH: {
            const float a[4] = {e0v.x, e0v.y, e0v.z, e0v.w}, b[4] = {e1v.x, e1v.y, e1v.z, e1v.w};
#pragma unroll
            for (int j = 0; j < 4; ++j) v[j] = v[j] * dswishf_(fmaf(x[j], a[j], b[j]));
            break;
        }
        case CMGAN_EPI_ACC:
#pragma unroll
            for (int j = 0; j < 4; ++j) v[j] = g.alpha * v[j] + x[j];
            break;
        default: break;
    }
}

}  // namespace cmgan_gemm
