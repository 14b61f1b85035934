// tf32 tensor-core implementation of the row-parallel GEMM contract (gemm_args.h) for sm_90a (H100).
// Persistent, warp-specialised, one CTA of three warpgroups per SM: each CTA loops over 128-row output tiles through a ring of
// shared-memory stages.  Each stage holds the tile's 128 A rows of one K chunk (two 64-row K-major SWIZZLE_128B halves) and, for
// streamed weights, the chunk's weight tile, which both consumers read: a weight chunk crosses L2 -> SM once per 128 rows.
// One exception (template NC = 1, TileShape): the cp.async gather with N <= 64 runs 64-row tiles with one consumer warpgroup and two
// CTAs per SM, since that producer is bound by its issue rate and gains from a second producer warpgroup on the SM.
//
//   warps 0-3   A producers (register budget cut by setmaxnreg, RegSplit), three modes:
//               * TMA (cfg.tma = 1): dense row-major A, one thread issues cp.async.bulk.tensor.2d boxes of 128 rows x 32 floats that
//                 land directly in the K-major SWIZZLE_128B layout; rows past M are zero-filled by the unit.
//               * TMA patches (cfg.tma = 2, template PATCH): same-size convolutions; a tile is a 16 x 8 (h x w) patch of one image and
//                 a chunk is one (tap, 32 channels) box of a 4-D (C, W, H, B) tensor map with the tap's (dy, dx) added to the
//                 coordinates -- padding is the unit's out-of-bounds zero fill.  Rows 0-63 (consumer 0) are image lines 0-7.
//               * cp.async (LDGSTS 16 B, zero fill) for strided / transposed convolutions, and LDG -> registers -> transform ->
//                 st.shared for operands with a prologue (BatchNorm+Swish / Swish+dropout / dropout / LayerNorm / InstanceNorm+PReLU);
//                 8 rows per thread.
//               Thread 0 also issues the weight tiles: cp.async.bulk of pre-tiled, pre-swizzled (N x 128 B) blocks, all K chunks once
//               per CTA when the whole weight fits in shared memory ("resident", every conformer GEMM), else per K chunk through the
//               stage ring ("streamed", the dilated dense convolutions).
//   warps 4-7   consumer 0: tile rows 0-63;  warps 8-11  consumer 1: tile rows 64-127 (register budget raised by setmaxnreg).
//               Each runs wgmma (M = 64, K = 8, one instruction per K step over N rounded up to a multiple of 64) over every K chunk
//               of its half, one wgmma group in flight (a stage is released when the next chunk's MMAs have been issued and its own
//               have retired; the empty barrier takes one arrival per consumer warp, 8 in all, so a stage returns to the producers
//               only when both halves are done with it), then the epilogue (compile-time kind): accumulator fragments -> per-warp
//               shared-memory staging -> coalesced float4 rows: bias, dropout, residual, activation gradients, Swish dual output ->
//               global.  A half with no row below M still runs its MMAs on the zero rows and releases its stages; it stores nothing.
//
// The weight operand is re-tiled once per call by pack_b_kernel into the scratch the caller passes (any source layout:
// Linear (N,K), Conv2d (N,C,kh,kw), and the transposed forms used for data gradients).
// All waits are bounded (a protocol bug traps instead of hanging the GPU).
#include <cuda.h>      // CUtensorMap (types only; the encoder is fetched from the driver at run time)

#include "common.cuh"
#include "../../include/cmgan_b200.h"
#include "gemm_device.cuh"
#include "tc_ptx.cuh"

namespace {
using namespace cmgan_gemm;
using namespace cmgan_tc;

constexpr int BM = 64;               // rows per consumer warpgroup = wgmma M
constexpr int NCONS = 2;             // consumer warpgroups of the 128-row plans
constexpr int TILE_M = NCONS * BM;   // rows per tile
constexpr int KC = 32;               // floats per K chunk = one 128-byte swizzle row
constexpr int A_HALF_BYTES = BM * KC * 4;           // 8 KB: one consumer's rows of a chunk
constexpr int NPROD = 128;           // producer threads (warps 0-3)
constexpr int SLAB = 64;             // epilogue column slab
constexpr int STG_LD = SLAB + 4;     // staging row stride (floats): conflict-free 128-bit accesses
// the tile of a kernel instance with NC consumer warpgroups: NC = 2 (128 rows, 384 threads, one CTA per SM) everywhere but the narrow
// cp.async plan (NC = 1: 64-row tiles, 256 threads, two CTAs per SM; make_plan).  The cp.async / register producers take 8 threads per
// 128-byte row; the epilogue stages 16 rows x (64 + 4) floats per consumer warp.
template <int NC> struct TileShape {
    static constexpr int rows = NC * BM, stage_bytes = NC * A_HALF_BYTES, threads = NPROD + NC * 128;
    static constexpr int rows_per_thread = rows / (NPROD / 8), stg_bytes = NC * 4 * 16 * STG_LD * 4;
};
constexpr int ENTRY_REGS = 168;      // 65536 / 384 rounded down to a multiple of 8 (__launch_bounds__(384, 1))
// setmaxnreg split per producer kind: 128 x PROD + 256 x CONS <= 128 x ENTRY + 256 x ENTRY = 64512.  The register producer keeps 8
// rows' decoded positions and normalisation statistics live across the K loop.
template <bool ASYNC_A> struct RegSplit { static constexpr int prod = ASYNC_A ? 72 : 120, cons = ASYNC_A ? 216 : 192; };
static_assert(128 * RegSplit<true>::prod + 256 * RegSplit<true>::cons <= TileShape<2>::threads * ENTRY_REGS, "register split");
static_assert(128 * RegSplit<false>::prod + 256 * RegSplit<false>::cons <= TileShape<2>::threads * ENTRY_REGS, "register split");
constexpr int SMEM_LIMIT = 227 * 1024;
constexpr int SMEM_LIMIT2 = 112 * 1024;             // per CTA when two share an SM (the narrow cp.async plan)
constexpr int RESIDENT_MAX = 96 * 1024;

// ---- weight re-tiling ------------------------------------------------------------------------------
// out[chunk][n][swizzled 32 floats], chunk = tap * (Cin/32) + kc;  rows n >= N are zero
__global__ void pack_b_kernel(const float* __restrict__ B, long sb_tap, long sb_k, long sb_n, int Cin, int ntaps, int N, int BN,
                              float* __restrict__ out) {
    long total = (long)ntaps * (Cin / KC) * BN * KC;
    long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= total) return;
    int kk = (int)(i % KC); long t = i / KC; int n = (int)(t % BN); long chunk = t / BN;
    int cpt = Cin / KC;
    int tap = (int)(chunk / cpt), kc = (int)(chunk % cpt);
    float v = 0.f;
    if (n < N) v = to_tf32(__ldg(B + (long)tap * sb_tap + (long)(kc * KC + kk) * sb_k + (long)n * sb_n));
    int c = kk >> 2, j = kk & 3;
    out[(chunk * BN + n) * KC + ((c ^ (n & 7)) << 2) + j] = v;
}

// every weight of a network in one launch (after the optimiser step): blockIdx.y = descriptor
__global__ void pack_all_kernel(const CmganPackDesc* __restrict__ descs) {
    const CmganPackDesc d = descs[blockIdx.y];
    const int Cin = (int)d.Cin, N = (int)d.N;
    const long total = d.ntaps * (Cin / KC) * (long)N * KC;
    for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
        int kk = (int)(i % KC); long t = i / KC; int n = (int)(t % N); long chunk = t / N;
        int cpt = Cin / KC;
        int tap = (int)(chunk / cpt), kc = (int)(chunk % cpt);
        float v = to_tf32(__ldg(d.src + (long)tap * d.sb_tap + (long)(kc * KC + kk) * d.sb_k + (long)n * d.sb_n));
        int c = kk >> 2, j = kk & 3;
        d.dst[(chunk * N + n) * KC + ((c ^ (n & 7)) << 2) + j] = v;
    }
}

// tma: 0 = cp.async / register producers, 1 = dense 2-D tensor map, 2 = same-size convolution: tiles are 16 x 8 (h x w) patches of one
// image (PW = 8 positions along w, PH = 16 lines), fetched through a 4-D tensor map with the tap offset added to the coordinates
struct TcCfg { int BN, stages, resident, ntiles, tma, nfx, nty, W, H; };
constexpr int PW = 8, PH = 16;
static_assert(PW * PH == TILE_M, "a patch tile is one tile");

// one consumer's view of the stage ring: its 64-row half of each A stage at sA (stage base + c x 8 KB), B stages (streamed) or all K
// chunks (resident) at sB, full barriers at bars, empty barriers at bars + 8 stages
struct TileRing { uint32_t sA, sB, bars; int stages, a_stage_bytes, b_tile_bytes, nchunks, resident, lane; };

// every K chunk of one tile into acc, NB 16-column blocks wide (compile time, so the wgmma pipeline is one straight K loop).  One wgmma
// group stays in flight: chunk q's MMAs are committed before the wait for chunk q - 1, whose stage is then released, so the tensor pipe
// does not drain at every chunk.  The tile's last group is waited for before returning (the epilogue reads acc).  q counts chunks
// over the CTA's tiles.  Since chunk q - 1 is released only after full(q) has been waited for, a producer may make full(q) depend on
// at most the release of chunk q - 2: TMA and register producers wait for the release of chunk q - stages before filling chunk q
// (stages >= 2); the cp.async producer signals full(q) LAG chunks later, so it needs stages >= LAG + 2.
template <int NB, int NBMAX>
__device__ __forceinline__ void tile_mma(float (&acc)[NBMAX][8], const TileRing& r, long& q) {
    auto empty_bar = [&](long qq) { return r.bars + 8u * (r.stages + (int)(qq % r.stages)); };
    for (int ch = 0; ch < r.nchunks; ++ch, ++q) {
        const int s = (int)(q % r.stages);
        const uint32_t par = (uint32_t)((q / r.stages) & 1);
        mbar_wait(r.bars + 8u * s, par);
        const uint64_t adesc = gmma_desc_sw128(r.sA + s * r.a_stage_bytes);
        const uint64_t bdesc = gmma_desc_sw128(r.sB + (r.resident ? ch : s) * r.b_tile_bytes);
        wgmma_fence();
        mma_chunk<NB, NBMAX>(acc, adesc, bdesc, ch == 0);
        wgmma_commit();
        wgmma_wait<1>();
        if (ch > 0) {
            __syncwarp();
            if (r.lane == 0) mbar_arrive(empty_bar(q - 1));      // this warp's share of chunk q - 1's stage has been read
        }
    }
    wgmma_wait<0>();
    __syncwarp();
    if (r.lane == 0) mbar_arrive(empty_bar(q - 1));
}
// the same at run time: N rounded up to 64 columns (nw = 1 .. NBMAX / 4 wgmma m64n64 widths), one branch per tile outside the wgmma
// pipeline.  Each accumulator column is its own dot product, so the columns past N change nothing in the first N, and the epilogue never
// reads them.  Their B rows (at most 48 rows = 6 KB past the tile, inside the allocation) are whatever lies there: the next ring stage,
// possibly while TMA or cp.async is writing it, the next resident chunk, or the epilogue staging.  Widths that are not a multiple of 64
// (an m64n64 block plus an n16 / n32 / n48 tail) would mix accumulator register groups of different sizes across the branches, and
// ptxas then serializes every wgmma of the kernel (advisory C7511, "insufficient register resources").
template <int NBMAX, int I = 1>
__device__ __forceinline__ void tile_mma_nw(int nw, float (&acc)[NBMAX][8], const TileRing& r, long& q) {
    if constexpr (4 * I <= NBMAX) {
        if (nw == I) tile_mma<4 * I, NBMAX>(acc, r, q);
        else tile_mma_nw<NBMAX, I + 1>(nw, acc, r, q);
    }
}

// NBMAX: 16-column blocks the accumulator has room for (N <= 256).  NC: consumer warpgroups = 64-row halves of a tile (TileShape)
template <bool ASYNC_A, int NBMAX, int EPI, bool PATCH, int NC>
__global__ void __launch_bounds__(TileShape<NC>::threads, NC == 1 ? 2 : 1) gemm_rows_tc_kernel(const __grid_constant__ CmganGemmArgs g, const float* __restrict__ Bp,
                                                                 const TcCfg cfg, const __grid_constant__ CUtensorMap tmA) {
    static_assert(NC == 2 || (ASYNC_A && !PATCH && NBMAX == 4), "64-row tiles only for the narrow cp.async plan");
    using TS = TileShape<NC>;
    extern __shared__ uint8_t smem_raw[];
    const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;        // SWIZZLE_128B tiles need 1024-byte alignment
    uint8_t* base_ptr = smem_raw + (base - smem_u32(smem_raw));
    const int BN = cfg.BN, stages = cfg.stages;
    const int b_tile_bytes = BN * KC * 4;
    const int cpt = g.Cin / KC;
    const int nchunks = cpt * g.ntaps;
    const uint32_t sA = base;
    const uint32_t sB = sA + stages * TS::stage_bytes;
    const uint32_t b_region = (uint32_t)(cfg.resident ? nchunks : stages) * b_tile_bytes;
    const uint32_t sStg = sB + b_region;
    const uint32_t bars = sStg + TS::stg_bytes;
    auto full_bar = [&](int s) { return bars + 8u * s; };
    auto empty_bar = [&](int s) { return bars + 8u * (stages + s); };
    const uint32_t bready_bar = bars + 8u * (2 * stages);

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int ntiles = cfg.ntiles;
    const int my_tiles = (ntiles - (int)blockIdx.x + (int)gridDim.x - 1) / (int)gridDim.x;

    if (tid == 0) {
        for (int s = 0; s < stages; ++s) { mbar_init(full_bar(s), cfg.tma ? 1 : NPROD + (cfg.resident ? 0 : 1)); mbar_init(empty_bar(s), 4 * NC); }
        mbar_init(bready_bar, 1);
        fence_barrier_init();
    }
    __syncthreads();

    if (warp < 4) {
        // ================================ A producers ================================
        if constexpr (NC == 2) setmaxnreg_dec<RegSplit<ASYNC_A>::prod>();
        const int c = tid & 7;            // 16-byte chunk within the 128-byte row
        const int rr = tid >> 3;          // rows rr + 16 i, i < 8: (rr + 16 i) & 7 == rr & 7, so row i lies 16 i x 128 bytes after row 0
        const uint32_t dst_off0 = rr * 128 + ((c ^ (rr & 7)) << 4);
        const long total = (long)my_tiles * nchunks;
        // weight tiles by cp.async.bulk of pre-tiled, pre-swizzled (N x 128 B) blocks, issued by thread 0: all K chunks once when they
        // fit ("resident"), else one per stage next to the A chunk ("streamed"; B_STAGE is a no-op when resident)
        if (tid == 0 && cfg.resident) {
            mbar_arrive_expect_tx(bready_bar, (uint32_t)(nchunks * b_tile_bytes));
            for (int ch = 0; ch < nchunks; ++ch)
                bulk_g2s(sB + ch * b_tile_bytes, Bp + (long)ch * BN * KC, (uint32_t)b_tile_bytes, bready_bar);
        }
#define B_STAGE(q, s)                                                                                                    \
        if (tid == 0 && !cfg.resident) {                                                                                 \
            if (!cfg.tma) mbar_arrive_expect_tx(full_bar(s), (uint32_t)b_tile_bytes);                                    \
            bulk_g2s(sB + (s) * b_tile_bytes, Bp + (long)((q) % nchunks) * BN * KC, (uint32_t)b_tile_bytes, full_bar(s)); \
        }

        if (ASYNC_A && cfg.tma) {
            // dense row-major A (no gather): one thread drives TMA, a 128-row x 32-float box per K chunk written straight into the
            // SWIZZLE_128B layout (rows past M are zero-filled by the unit); every stage of the ring can be in flight
            if (tid == 0) {
                for (long q = 0; q < total; ++q) {
                    const int lt = (int)(q / nchunks), ch = (int)(q - (long)lt * nchunks);
                    const int s = (int)(q % stages);
                    const uint32_t par = (uint32_t)((q / stages) & 1);
                    mbar_wait(empty_bar(s), par ^ 1u);
                    mbar_arrive_expect_tx(full_bar(s), (uint32_t)(TS::stage_bytes + (cfg.resident ? 0 : b_tile_bytes)));
                    B_STAGE(q, s)
                    const int tile = blockIdx.x + lt * gridDim.x;
                    if (!PATCH) {
                        tma_load_2d(sA + s * TS::stage_bytes, &tmA, ch * KC, tile * TS::rows, full_bar(s));
                    } else {        // patch (bimg, ty, fx): rows r = 8 * line + position; padding and ragged edges come back as zeros
                        const int fx = tile % cfg.nfx, ty = (tile / cfg.nfx) % cfg.nty, bimg = tile / (cfg.nfx * cfg.nty);
                        const int tap = ch / cpt, kc = ch - tap * cpt;
                        tma_load_4d(sA + s * TS::stage_bytes, &tmA, kc * KC, fx * PW + g.dx[tap], ty * PH + g.dy[tap], bimg, full_bar(s));
                    }
                }
            }
            __syncwarp();
        } else if (ASYNC_A) {
            // full(q) is signalled after the wait for the release of chunk q + LAG - stages, which must come before the consumer's
            // release of chunk q - 1 (one chunk late, see tile_mma): LAG <= stages - 2.  The launcher gives this producer >= 3 stages.
            const int LAG = stages >= 4 ? 2 : 1;
            long rowoff[TS::rows_per_thread];
            RowInfo ri[TS::rows_per_thread];
            int cur_tile = -1, cur_tap = -1;
            for (long q = 0; q < total + LAG; ++q) {
                if (q < total) {
                    const int lt = (int)(q / nchunks), ch = (int)(q - (long)lt * nchunks);
                    const int s = (int)(q % stages);
                    const uint32_t par = (uint32_t)((q / stages) & 1);
                    const int tap = ch / cpt, k0 = (ch - tap * cpt) * KC + c * 4;
                    if (lt != cur_tile) {
                        cur_tile = lt; cur_tap = -1;
                        const int m0 = (blockIdx.x + lt * gridDim.x) * TS::rows;
#pragma unroll
                        for (int i = 0; i < TS::rows_per_thread; ++i) ri[i] = decode_row(g, m0 + rr + 16 * i);
                    }
                    if (tap != cur_tap) {
                        cur_tap = tap;
#pragma unroll
                        for (int i = 0; i < TS::rows_per_thread; ++i) {
                            long r = in_row_of(g, ri[i], tap);
                            rowoff[i] = r < 0 ? -1 : g.tap_off[tap] + r * g.lda;
                        }
                    }
                    mbar_wait(empty_bar(s), par ^ 1u);
                    B_STAGE(q, s)
                    const uint32_t sbase = sA + s * TS::stage_bytes + dst_off0;
#pragma unroll
                    for (int i = 0; i < TS::rows_per_thread; ++i) {
                        const bool ok = rowoff[i] >= 0;
                        cp_async16(sbase + i * 16 * 128, g.A + (ok ? rowoff[i] + k0 : 0), ok ? 16u : 0u);
                    }
                }
                cp_async_commit();
                const long done = q - LAG;
                if (done >= 0) {
                    if (LAG == 2) cp_async_wait<2>(); else cp_async_wait<1>();
                    fence_proxy_async();
                    mbar_arrive(full_bar((int)(done % stages)));
                }
            }
        } else {
            float mean[TS::rows_per_thread], rstd[TS::rows_per_thread];
            RowInfo ri[TS::rows_per_thread];
            int cur_tile = -1;
            for (long q = 0; q < total; ++q) {
                const int lt = (int)(q / nchunks), ch = (int)(q - (long)lt * nchunks);
                const int s = (int)(q % stages);
                const uint32_t par = (uint32_t)((q / stages) & 1);
                const int tap = ch / cpt, k0 = (ch - tap * cpt) * KC + c * 4;
                if (lt != cur_tile) {
                    cur_tile = lt;
                    const int m0 = (blockIdx.x + lt * gridDim.x) * TS::rows;
#pragma unroll
                    for (int i = 0; i < TS::rows_per_thread; ++i) {
                        ri[i] = decode_row(g, m0 + rr + 16 * i);
                        mean[i] = 0.f; rstd[i] = 1.f;
                        if (g.pro == CMGAN_PRO_LN) {        // ntaps == 1: in_row is constant over the K loop
                            long r = in_row_of(g, ri[i], 0);
                            if (r >= 0) { float2 st = __ldg(reinterpret_cast<const float2*>(g.p0) + r); mean[i] = st.x; rstd[i] = st.y; }
                        }
                    }
                }
                ChunkParams cp;
                load_chunk_params(g, k0, cp);
                const uint32_t sbase = sA + s * TS::stage_bytes + dst_off0;
                // two passes of 4 rows (one consumer's half each), so that the loads in flight fit the producer's register budget
#pragma unroll
                for (int h = 0; h < NC; ++h) {
                    float4 v[4];
                    long rows[4];
#pragma unroll
                    for (int i = 0; i < 4; ++i) {
                        rows[i] = in_row_of(g, ri[4 * h + i], tap);
                        v[i] = rows[i] >= 0 ? __ldg(reinterpret_cast<const float4*>(g.A + g.tap_off[tap] + rows[i] * g.lda + k0)) : make_float4(0.f, 0.f, 0.f, 0.f);
                    }
#pragma unroll
                    for (int i = 0; i < 4; ++i)
                        if (rows[i] >= 0) v[i] = transform4(g, v[i], rows[i], k0, mean[4 * h + i], rstd[4 * h + i], cp);
                    if (h == 0) {
                        mbar_wait(empty_bar(s), par ^ 1u);
                        B_STAGE(q, s)
                    }
#pragma unroll
                    for (int i = 0; i < 4; ++i)
                        asm volatile("st.shared.v4.f32 [%0], {%1, %2, %3, %4};" ::"r"(sbase + (4 * h + i) * 16 * 128), "f"(to_tf32(v[i].x)),
                                     "f"(to_tf32(v[i].y)), "f"(to_tf32(v[i].z)), "f"(to_tf32(v[i].w)) : "memory");
                }
                fence_proxy_async();
                mbar_arrive(full_bar(s));
            }
        }
#undef B_STAGE
    } else {
        // ======================= consumer warpgroups (warps 4-7: rows 0-63, warps 8-11: rows 64-127): MMAs, then the epilogue =======================
        // warp cw owns tile rows 16 cw .. 16 cw + 15.  Per 64-column slab: fragments -> st.shared (own rows) -> the warp re-reads the slab
        // as coalesced 256-byte row segments (16 lanes x float4, 2 rows per pass, 8 passes), applies the compile-time epilogue and stores.
        if constexpr (NC == 2) setmaxnreg_inc<RegSplit<ASYNC_A>::cons>();
        const int cw = warp - 4;
        const int cons = cw >> 2;
        const int nb = BN / 16;
        float acc[NBMAX][8];
#pragma unroll
        for (int j = 0; j < NBMAX; ++j)
#pragma unroll
            for (int i = 0; i < 8; ++i) acc[j][i] = 0.f;
        float* stg = reinterpret_cast<float*>(base_ptr + (sStg - base)) + cw * 16 * STG_LD;
        const int col4 = (lane & 15) * 4;
        const int rsub = lane >> 4;
        const int fg = lane >> 2, ft = lane & 3;       // fragment row / column pair
        constexpr bool DROPS = EPI == CMGAN_EPI_DROP_RES || EPI == CMGAN_EPI_DSWISH_DROP || EPI == CMGAN_EPI_SWISH_DUAL;
        const uint32_t seed32 = DROPS ? cmgan_seed32(eff_seed(g)) : 0u;
        const uint32_t thr16 = g.drop_thr >> 16;
        const bool drop_on = DROPS && g.drop_thr != 0u;
        constexpr bool patch = PATCH;          // compile-time: the flat-tile epilogue keeps its simple row arithmetic
        const float inv_keep = g.inv_keep, alpha = g.alpha;
        // auxiliary operand read at the output position: R (DROP_RES, optional), aux (DSWISH_DROP / DBNSWISH), old C (ACC)
        const float* xbase = nullptr;
        long ldx = 0;
        if (EPI == CMGAN_EPI_DROP_RES) { xbase = g.R; ldx = g.ldr; }
        else if (EPI == CMGAN_EPI_DSWISH_DROP || EPI == CMGAN_EPI_DBNSWISH) { xbase = g.aux; ldx = g.ldaux; }
        else if (EPI == CMGAN_EPI_ACC) { xbase = g.C; ldx = g.ldc; }
        if (cfg.resident) mbar_wait(bready_bar, 0);
        const TileRing ring{sA + cons * A_HALF_BYTES, sB, bars, stages, TS::stage_bytes, b_tile_bytes, nchunks, cfg.resident, lane};
        long q = 0;
        for (int lt = 0; lt < my_tiles; ++lt) {
            tile_mma_nw<NBMAX>((nb + 3) / 4, acc, ring, q);
            // rows of this warp.  Flat tiles: 16 consecutive rows.  Patch tiles (cfg.tma == 2): 2 image lines x 8 positions.
            // Pass ps handles rows 2 ps + rsub; its row index is mfirst + (ps >> 2) * hi_rows + 2 * (ps & 3).
            const int tile = blockIdx.x + lt * gridDim.x;
            long mfirst;
            int hi_rows, vhi, vlo;          // valid: flat: 8 (ps >> 2) + 2 (ps & 3) + rsub < vlo;  patch: (ps >> 2) < vhi && 2 (ps & 3) + rsub < vlo
            if (patch) {
                const int fx = tile % cfg.nfx, ty = (tile / cfg.nfx) % cfg.nty, bimg = tile / (cfg.nfx * cfg.nty);
                const int y0 = ty * PH + cw * 2, x0 = fx * PW;
                mfirst = ((long)bimg * cfg.H + y0) * cfg.W + x0 + rsub;
                hi_rows = cfg.W; vhi = cfg.H - y0; vlo = cfg.W - x0;
            } else {
                const int mrow0 = tile * TS::rows + cw * 16;
                mfirst = (long)mrow0 + rsub;
                hi_rows = 8; vhi = 2; vlo = g.M - mrow0;
            }
            auto row_ok = [&](int ps) { return patch ? ((ps >> 2) < vhi && 2 * (ps & 3) + rsub < vlo) : (2 * ps + rsub < vlo); };
            auto row_delta = [&](int ps) { return (long)(ps >> 2) * hi_rows + 2 * (ps & 3); };
            const bool any_row = row_ok(0);
#pragma unroll
            for (int sl = 0; sl < NBMAX / 4; ++sl) {
                const int n0 = sl * SLAB;
                if (n0 >= BN) break;
                const int ncols = min(SLAB, BN - n0);
#pragma unroll
                for (int jj = 0; jj < 4; ++jj) {
                    if (16 * jj >= ncols) break;
                    const float* d = acc[4 * sl + jj];
#pragma unroll
                    for (int i = 0; i < 2; ++i) {
                        const int col = 16 * jj + 8 * i + 2 * ft;
                        *reinterpret_cast<float2*>(stg + fg * STG_LD + col) = make_float2(d[4 * i], d[4 * i + 1]);
                        *reinterpret_cast<float2*>(stg + (fg + 8) * STG_LD + col) = make_float2(d[4 * i + 2], d[4 * i + 3]);
                    }
                }
                __syncwarp();
                if (col4 < ncols && any_row) {
                    const int n = n0 + col4;
                    float4 bias4 = make_float4(0.f, 0.f, 0.f, 0.f), e0v = bias4, e1v = bias4;
                    if (g.bias) bias4 = __ldg(reinterpret_cast<const float4*>(g.bias + n));
                    if (EPI == CMGAN_EPI_DBNSWISH) { e0v = __ldg(reinterpret_cast<const float4*>(g.e0 + n)); e1v = __ldg(reinterpret_cast<const float4*>(g.e1 + n)); }
                    float* cptr = g.C ? g.C + mfirst * g.ldc + n : nullptr;
                    float* c2ptr = EPI == CMGAN_EPI_SWISH_DUAL ? g.C2 + mfirst * g.ldc2 + n : nullptr;
                    const float* xp = xbase ? xbase + mfirst * ldx + n : nullptr;
                    const float* sptr = stg + rsub * STG_LD + col4;
                    const long ldc = g.ldc, ldc2 = g.ldc2;
                    const uint32_t pair = (uint32_t)(((unsigned long long)mfirst * (unsigned long long)g.N + (unsigned long long)n) >> 1);
                    const uint32_t phalf = (uint32_t)g.N >> 1;       // one row further = N / 2 pairs further
#pragma unroll
                    for (int b4 = 0; b4 < 2; ++b4) {
                        float4 ex[4];          // auxiliary operand of the 4 rows of this batch: all loads in flight before the first use
#pragma unroll
                        for (int u = 0; u < 4; ++u)
                            ex[u] = (xp && row_ok(b4 * 4 + u)) ? __ldg(reinterpret_cast<const float4*>(xp + row_delta(b4 * 4 + u) * ldx))
                                                                : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
                        for (int u = 0; u < 4; ++u) {
                            const int ps = b4 * 4 + u;
                            if (!row_ok(ps)) continue;
                            const long rd = row_delta(ps);
                            const float4 a = *reinterpret_cast<const float4*>(sptr + ps * 2 * STG_LD);
                            float v[4] = {a.x + bias4.x, a.y + bias4.y, a.z + bias4.z, a.w + bias4.w};
                            float ds[4] = {1.f, 1.f, 1.f, 1.f};
                            if (DROPS && drop_on) {
                                const uint32_t pr = pair + (uint32_t)rd * phalf;
                                const uint32_t h0 = cmgan_mix32((pr * 0x9E3779B1u) ^ seed32), h1 = cmgan_mix32(((pr + 1u) * 0x9E3779B1u) ^ seed32);
                                ds[0] = (h0 & 0xFFFFu) >= thr16 ? inv_keep : 0.f; ds[1] = (h0 >> 16) >= thr16 ? inv_keep : 0.f;
                                ds[2] = (h1 & 0xFFFFu) >= thr16 ? inv_keep : 0.f; ds[3] = (h1 >> 16) >= thr16 ? inv_keep : 0.f;
                            }
                            const float x[4] = {ex[u].x, ex[u].y, ex[u].z, ex[u].w};
                            if (EPI == CMGAN_EPI_SWISH_DUAL) {
                                if (cptr) *reinterpret_cast<float4*>(cptr + rd * ldc) = make_float4(v[0], v[1], v[2], v[3]);
#pragma unroll
                                for (int j = 0; j < 4; ++j) v[j] = to_tf32(swishf_(v[j]) * ds[j]);      // operand of the next contraction: round, the tensor core would truncate
                                *reinterpret_cast<float4*>(c2ptr + rd * ldc2) = make_float4(v[0], v[1], v[2], v[3]);
                                continue;
                            }
                            if (EPI == CMGAN_EPI_DROP_RES) {
#pragma unroll
                                for (int j = 0; j < 4; ++j) v[j] = alpha * v[j] * ds[j] + (xbase ? x[j] : 0.f);
                            } else if (EPI == CMGAN_EPI_DSWISH_DROP) {
#pragma unroll
                                for (int j = 0; j < 4; ++j) v[j] = to_tf32(v[j] * dswishf_(x[j]) * ds[j]);   // feeds the next data-gradient GEMM and a weight-gradient GEMM
                            } else if (EPI == CMGAN_EPI_DBNSWISH) {
                                const float sa[4] = {e0v.x, e0v.y, e0v.z, e0v.w}, sb[4] = {e1v.x, e1v.y, e1v.z, e1v.w};
#pragma unroll
                                for (int j = 0; j < 4; ++j) v[j] = v[j] * dswishf_(fmaf(x[j], sa[j], sb[j]));
                            } else if (EPI == CMGAN_EPI_ACC) {
#pragma unroll
                                for (int j = 0; j < 4; ++j) v[j] = alpha * v[j] + x[j];
                            }
                            *reinterpret_cast<float4*>(cptr + rd * ldc) = make_float4(v[0], v[1], v[2], v[3]);
                        }
                    }
                }
                __syncwarp();
            }
        }
    }
}

int tc_supported(const CmganGemmArgs* a) {
    if (a->N % 16 || a->N < 16 || a->N > 256) return 0;
    if (a->Cin % KC) return 0;
    if (a->lda % 4 || ((uintptr_t)a->A & 15)) return 0;
    if (a->C && (a->ldc % 4 || ((uintptr_t)a->C & 15))) return 0;
    if (a->epi == CMGAN_EPI_SWISH_DUAL && (a->ldc2 % 4 || ((uintptr_t)a->C2 & 15))) return 0;
    if (a->bias && ((uintptr_t)a->bias & 15)) return 0;
    for (int t = 0; t < a->ntaps; ++t)
        if (a->tap_off[t] % 4) return 0;
    if (!a->ws || a->ws_floats < (long long)a->N * a->Cin * a->ntaps) return 0;
    if ((uintptr_t)a->ws & 127) return 0;
    if (a->pro == CMGAN_PRO_LN && (((uintptr_t)a->p1 & 15) || ((uintptr_t)a->p2 & 15) || a->ntaps != 1)) return 0;
    if (a->pro == CMGAN_PRO_BN_SWISH && (((uintptr_t)a->p0 & 15) || ((uintptr_t)a->p1 & 15))) return 0;
    if (a->pro == CMGAN_PRO_IN_PRELU && (((uintptr_t)a->p0 & 15) || ((uintptr_t)a->p1 & 15) || ((uintptr_t)a->p2 & 15) || a->pstride % 4)) return 0;
    return 1;
}

int g_num_sms = 0;

using PFN_encodeTiled = CUresult (*)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                      const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
PFN_encodeTiled get_encoder() {
    static PFN_encodeTiled encode = nullptr;
    static bool tried = false;
    if (!tried) {
        tried = true;
        void* fn = nullptr;
        cudaDriverEntryPointQueryResult qres;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres) == cudaSuccess && qres == cudaDriverEntryPointSuccess)
            encode = reinterpret_cast<PFN_encodeTiled>(fn);
    }
    return encode;
}

// Every launch decision of the row GEMM, made on the host from the arguments alone.  One CTA of three warpgroups per SM (the producer
// and two consumers, 128-row tiles); the stage ring fills the shared memory left after the epilogue staging and, when the whole weight
// fits in RESIDENT_MAX, the resident weight image.  The cp.async producer needs 3 stages (gemm_rows_tc_kernel, LAG) and the TMA plans
// fall back to it, so no plan takes fewer: the largest stage (N = 256, streamed, 48 KB) still leaves room for 3.
void make_plan(const CmganGemmArgs* a, CmganGemmRowsPlan* p) {
    memset(p, 0, sizeof(*p));
    if (!tc_supported(a)) return;
    bool same_off = true;
    for (int t = 1; t < a->ntaps; ++t) same_off = same_off && a->tap_off[t] == a->tap_off[0];
    const long long img = (long long)a->OH * a->OW;
    if (a->pro != CMGAN_PRO_NONE) {
        p->mode = CMGAN_ROWS_REGISTER;
    } else if ((a->epi == CMGAN_EPI_NONE || a->epi == CMGAN_EPI_ACC) && a->conv && a->mul_y == 1 && a->mul_x == 1 && a->div_y == 1 &&
               a->div_x == 1 && a->OH == a->IH && a->OW == a->IW && same_off && img > 0 && a->M % img == 0 &&
               a->M / img * cdiv((long long)a->OW, (long long)PW) * cdiv((long long)a->OH, (long long)PH) < (1ll << 30)) {
        // same-size convolution: taps = coordinate offsets of a (C, W, H, B) tensor, padding = out-of-bounds zero fill
        p->mode = CMGAN_ROWS_PATCH;
    } else if (!a->conv && a->ntaps == 1) {
        p->mode = CMGAN_ROWS_TMA2D;
    } else {
        p->mode = CMGAN_ROWS_CPASYNC;
    }
    p->b_tile_bytes = a->N * KC * 4;
    p->nchunks = (a->Cin / KC) * a->ntaps;
    p->resident = (long)p->nchunks * p->b_tile_bytes <= RESIDENT_MAX ? 1 : 0;
    const int resident_bytes = p->resident ? p->nchunks * p->b_tile_bytes : 0;
    const int b_stage = p->resident ? 0 : p->b_tile_bytes;
    const int fixed1 = 1024 /*alignment*/ + TileShape<1>::stg_bytes + 256 /*barriers*/ + resident_bytes;
    // the cp.async gather is bound by its producer's issue rate (one 16-byte copy per row and 16 bytes of K): with N <= 64 it runs 64-row
    // tiles, two CTAs per SM, so that two producer warpgroups gather on each SM; every other plan runs 128-row tiles, one CTA per SM
    const bool narrow = p->mode == CMGAN_ROWS_CPASYNC && a->N <= 64 && fixed1 + 3 * (TileShape<1>::stage_bytes + b_stage) <= SMEM_LIMIT2;
    const int nc = narrow ? 1 : 2;
    p->tile_rows = narrow ? TileShape<1>::rows : TileShape<2>::rows;
    p->consumers = nc;
    p->threads = narrow ? TileShape<1>::threads : TileShape<2>::threads;
    p->ctas_per_sm = narrow ? 2 : 1;
    p->entry_regs = narrow ? 128 : ENTRY_REGS;
    const int per_stage = (narrow ? TileShape<1>::stage_bytes : TileShape<2>::stage_bytes) + b_stage;
    const int fixed = narrow ? fixed1 : 1024 + TileShape<2>::stg_bytes + 256 + resident_bytes;
    p->stages = ((narrow ? SMEM_LIMIT2 : SMEM_LIMIT) - fixed) / per_stage;
    if (p->stages > 8) p->stages = 8;
    p->smem_bytes = fixed + p->stages * per_stage;
    p->ntiles = cdiv((long long)a->M, (long long)p->tile_rows);
    if (p->mode == CMGAN_ROWS_PATCH) {
        p->patch_w = PW;
        p->patch_h = PH;
        p->ntiles = a->M / img * cdiv((long long)a->OW, (long long)PW) * cdiv((long long)a->OH, (long long)PH);
    }
    const bool async_a = p->mode != CMGAN_ROWS_REGISTER;
    p->producer_regs = narrow ? p->entry_regs : async_a ? RegSplit<true>::prod : RegSplit<false>::prod;
    p->consumer_regs = narrow ? p->entry_regs : async_a ? RegSplit<true>::cons : RegSplit<false>::cons;
    p->supported = p->stages >= 3 ? 1 : 0;
}

template <bool ASYNC_A, int NBMAX, int EPI, bool PATCH = false, int NC = 2>
int launch_variant(const CmganGemmArgs& a, const TcCfg& cfg, int grid, size_t smem, cudaStream_t st, const CUtensorMap& tm) {
    static bool attr_set = false;
    if (!attr_set) {
        cudaError_t e = cudaFuncSetAttribute(gemm_rows_tc_kernel<ASYNC_A, NBMAX, EPI, PATCH, NC>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_LIMIT);
        if (e != cudaSuccess) { cmgan_set_error("gemm_rows_tc: cudaFuncSetAttribute: %s", cudaGetErrorString(e)); return -1; }
        attr_set = true;
    }
    gemm_rows_tc_kernel<ASYNC_A, NBMAX, EPI, PATCH, NC><<<grid, TileShape<NC>::threads, smem, st>>>(a, a.ws, cfg, tm);
    return 0;
}

}  // namespace

// tf32 tensor-core path of cmgan_gemm_rows (same contract).  Returns 1 if the shape is not covered (caller falls back).
int cmgan_gemm_rows_tc_launch(const CmganGemmArgs* a, cudaStream_t st) {
    CmganGemmRowsPlan p;
    make_plan(a, &p);
    if (!p.supported) return 1;
    TcCfg cfg;
    cfg.BN = a->N;
    cfg.stages = p.stages;
    cfg.resident = p.resident;
    cfg.ntiles = (int)cdiv(a->M, TILE_M);      // the 64-row plan has no TMA mode: p.ntiles
    if (p.tile_rows != TILE_M) cfg.ntiles = (int)p.ntiles;
    cfg.tma = 0;
    cfg.nfx = cfg.nty = 1; cfg.W = cfg.H = 0;
    if (g_num_sms == 0) {
        int dev = 0;
        cudaGetDevice(&dev);
        cudaDeviceGetAttribute(&g_num_sms, cudaDevAttrMultiProcessorCount, dev);
    }
    // the TMA plans describe A to the unit (SWIZZLE_128B, zero fill out of bounds); if the driver cannot encode the map, the cp.async
    // producer gathers the same rows (make_plan gives every plan the 3 stages it needs)
    alignas(64) CUtensorMap tm;
    memset(&tm, 0, sizeof(tm));
    if (p.mode == CMGAN_ROWS_TMA2D) {           // dense row-major A: box = 32 floats x 128 rows
        PFN_encodeTiled encode = get_encoder();
        if (encode) {
            const cuuint64_t gdim[2] = {(cuuint64_t)a->Cin, (cuuint64_t)a->M};
            const cuuint64_t gstride[1] = {(cuuint64_t)a->lda * sizeof(float)};
            const cuuint32_t box[2] = {(cuuint32_t)KC, (cuuint32_t)TILE_M};
            const cuuint32_t estr[2] = {1, 1};
            CUresult r = encode(&tm, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<float*>(a->A + a->tap_off[0]), gdim, gstride, box, estr,
                                CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                                CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
            if (r == CUDA_SUCCESS) cfg.tma = 1;
        }
    } else if (p.mode == CMGAN_ROWS_PATCH) {    // (C, W, H, B) tensor, box = 32 channels x PW positions x PH lines x 1 image
        PFN_encodeTiled encode = get_encoder();
        if (encode) {
            const long long Bn = a->M / ((long long)a->OH * a->OW);
            const cuuint64_t gdim[4] = {(cuuint64_t)a->Cin, (cuuint64_t)a->IW, (cuuint64_t)a->IH, (cuuint64_t)Bn};
            const cuuint64_t gstride[3] = {(cuuint64_t)a->lda * sizeof(float), (cuuint64_t)a->IW * a->lda * sizeof(float),
                                           (cuuint64_t)a->IH * a->IW * a->lda * sizeof(float)};
            const cuuint32_t box[4] = {(cuuint32_t)KC, (cuuint32_t)PW, (cuuint32_t)PH, 1};
            const cuuint32_t estr[4] = {1, 1, 1, 1};
            CUresult r = encode(&tm, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, const_cast<float*>(a->A + a->tap_off[0]), gdim, gstride, box, estr,
                                CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                                CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
            if (r == CUDA_SUCCESS) {
                cfg.tma = 2; cfg.nfx = (int)cdiv(a->OW, PW); cfg.nty = (int)cdiv(a->OH, PH); cfg.W = a->OW; cfg.H = a->OH;
                cfg.ntiles = (int)p.ntiles;
            }
        }
    }
    if (!a->b_packed) {
        long total = (long)p.nchunks * cfg.BN * KC;
        pack_b_kernel<<<cdiv(total, 256), 256, 0, st>>>(a->B, a->sb_tap, a->sb_k, a->sb_n, a->Cin, a->ntaps, a->N, cfg.BN, a->ws);
        if (cmgan_check_launch("pack_b_kernel")) return -1;
    }
    const int grid = cfg.ntiles < p.ctas_per_sm * g_num_sms ? cfg.ntiles : p.ctas_per_sm * g_num_sms;
    const size_t smem = (size_t)p.smem_bytes;
    int rc = -2;
#define CMGAN_TC_LAUNCH(E)                                                                                            \
    case E:                                                                                                           \
        rc = a->pro != CMGAN_PRO_NONE ? launch_variant<false, 16, E>(*a, cfg, grid, smem, st, tm)                     \
             : p.consumers == 1       ? launch_variant<true, 4, E, false, 1>(*a, cfg, grid, smem, st, tm)             \
                                      : launch_variant<true, 16, E>(*a, cfg, grid, smem, st, tm);                     \
        break;
    if (cfg.tma == 2) {      // patch tiles (same-size convolutions): forward (plain) and data-gradient (accumulating) epilogues
        rc = a->epi == CMGAN_EPI_NONE ? launch_variant<true, 16, CMGAN_EPI_NONE, true>(*a, cfg, grid, smem, st, tm)
                                      : launch_variant<true, 16, CMGAN_EPI_ACC, true>(*a, cfg, grid, smem, st, tm);
    } else
    switch (a->epi) {
        CMGAN_TC_LAUNCH(CMGAN_EPI_NONE)
        CMGAN_TC_LAUNCH(CMGAN_EPI_DROP_RES)
        CMGAN_TC_LAUNCH(CMGAN_EPI_DSWISH_DROP)
        CMGAN_TC_LAUNCH(CMGAN_EPI_DBNSWISH)
        CMGAN_TC_LAUNCH(CMGAN_EPI_ACC)
        CMGAN_TC_LAUNCH(CMGAN_EPI_SWISH_DUAL)
        default: break;
    }
#undef CMGAN_TC_LAUNCH
    if (rc == -2) { cmgan_set_error("gemm_rows_tc: unknown epilogue %d", a->epi); return -1; }
    if (rc) return -1;
    return cmgan_check_launch("gemm_rows_tc_kernel");
}

// the launch plan of one argument block, computed on the host without touching the device
CMGAN_API int cmgan_gemm_rows_tc_plan(const CmganGemmArgs* a, CmganGemmRowsPlan* out) {
    CMGAN_REQUIRE(a && out, "cmgan_gemm_rows_tc_plan: null argument");
    make_plan(a, out);
    return 0;
}

// Re-tile n weights (device table of CmganPackDesc) for the tensor-core path in one launch: called once after the optimiser step, so that the
// GEMM launches of the next step find their B operand ready (CmganGemmArgs.b_packed = 1).
// one weight -> its K-major SWIZZLE_128B tile image (the layout cmgan_ffn_fwd / the b_packed GEMM path consume): N * Cin * ntaps floats
CMGAN_API int cmgan_pack_weight(const float* src, float* dst, long long sb_tap, long long sb_k, long long sb_n, int Cin, int ntaps, int N, void* stream) {
    CMGAN_REQUIRE(src && dst && Cin > 0 && Cin % KC == 0 && ntaps >= 1 && N > 0, "cmgan_pack_weight: bad arguments (Cin must be a multiple of %d)", KC);
    const long total = (long)ntaps * Cin * N;
    pack_b_kernel<<<cdiv(total, 256), 256, 0, (cudaStream_t)stream>>>(src, sb_tap, sb_k, sb_n, Cin, ntaps, N, N, dst);
    return cmgan_check_launch("pack_b_kernel");
}

CMGAN_API int cmgan_pack_weights(const CmganPackDesc* descs, int n, void* stream) {
    CMGAN_REQUIRE(descs || n == 0, "cmgan_pack_weights: null table");
    if (n == 0) return 0;
    pack_all_kernel<<<dim3(48, n), 256, 0, (cudaStream_t)stream>>>(descs);
    return cmgan_check_launch("pack_all_kernel");
}
