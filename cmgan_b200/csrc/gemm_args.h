// Argument block shared by the row-parallel GEMM (cmgan_gemm_rows), the weight-gradient GEMM
// (cmgan_gemm_wgrad) and their tensor-core variants.  Plain C layout (mirrored by ctypes in
// cmgan_b200/_lib.py); no torch types.
//
// One call computes, for every output row m < M and column n < N,
//     C[m, n] = epi( bias[n] + sum_{tap < ntaps} sum_{k < Cin}  pro(A[in_row(m, tap), k]) * B(tap, k, n) )
// with   B(tap, k, n) = B[tap * sb_tap + k * sb_k + n * sb_n]      (any weight layout, no repacking)
// and    in_row(m, tap) = m                                          (conv == 0)
//        m = (b * OH + y) * OW + x,  iy = y * mul_y + dy[tap],  ix = x * mul_x + dx[tap],
//        (iy, ix) must be divisible by (div_y, div_x) and land inside [0, IH) x [0, IW) after the
//        division, else the tap contributes zero (zero padding / transposed-conv holes);
//        in_row = (b * IH + iy) * IW + ix                            (conv == 1)
// A row r starts at A + tap_off[tap] + r * lda.  This one form covers: Linear / 1x1 conv (forward and
// data gradient), the causal dilated (2,3) dense convolutions, the strided (1,3) and 4x4 convolutions and
// their data gradients, the sub-pixel (1,3) convolution, and the framed DFT / inverse DFT of the
// STFT front/back end (overlapping rows: lda = hop < Cin).
#pragma once
#include <stdint.h>

#define CMGAN_MAX_TAPS 16

enum CmganPro {          // applied to every A element before the product
    CMGAN_PRO_NONE = 0,
    CMGAN_PRO_LN = 1,          // (a - mean[r]) * rstd[r] * p1[k] + p2[k];  p0 = float2 stats per in_row
    CMGAN_PRO_SWISH_DROP = 2,  // swish(a) * drop(r * Cin + k)
    CMGAN_PRO_BN_SWISH = 3,    // z = a * p0[k] + p1[k]; swish(z)
    CMGAN_PRO_DROP = 4,        // a * drop(r * Cin + k) * pro_alpha
    CMGAN_PRO_IN_PRELU = 5     // z = a * p0[b*pstride + k] + p1[b*pstride + k]; prelu(z, p2[k]);  b = r / rows_per_batch
};
enum CmganEpi {
    CMGAN_EPI_NONE = 0,        // C = v
    CMGAN_EPI_DROP_RES = 1,    // C = alpha * drop(m * N + n) * v + R[m, n]   (R may be null)
    CMGAN_EPI_DSWISH_DROP = 2, // C = v * dswish(aux[m, n]) * drop(m * N + n)
    CMGAN_EPI_DBNSWISH = 3,    // z = aux[m, n] * e0[n] + e1[n];  C = v * dswish(z)
    CMGAN_EPI_ACC = 4,         // C = alpha * v + C
    CMGAN_EPI_SWISH_DUAL = 5   // C = v (skipped when C is null);  C2[m, n] = swish(v) * drop(m * N + n)   (feed-forward: pre-activation kept for
                               // the backward pass, activated copy consumed by the next GEMM without a prologue)
};

typedef struct CmganGemmArgs {
    const float* A; long long lda;
    const float* B; long long sb_tap, sb_k, sb_n;
    const float* bias;
    float* C; long long ldc;
    int M, N, Cin, ntaps;
    int conv, OH, OW, IH, IW, mul_y, mul_x, div_y, div_x;
    int dy[CMGAN_MAX_TAPS], dx[CMGAN_MAX_TAPS];
    long long tap_off[CMGAN_MAX_TAPS];
    int pro; float pro_alpha; const float* p0; const float* p1; const float* p2; long long rows_per_batch; long long pstride;
    int epi; float alpha; const float* R; long long ldr; const float* aux; long long ldaux; const float* e0; const float* e1;
    unsigned long long seed; unsigned int drop_thr; float inv_keep;              // epilogue / wgrad-D dropout
    unsigned long long pro_seed; unsigned int pro_thr; float pro_inv_keep;       // prologue dropout
    // wgrad only: D = upstream gradient rows (M x N), prod: 0 none, 1 = alpha * drop(m*N+n); dbias may be null
    const float* D; long long ldd; int prod; float* dbias;
    int precision;             // 0 = fp32 FFMA, 1 = tf32 wgmma tensor cores (shapes the tensor path does not cover fall back to fp32 FFMA)
    float* ws; long long ws_floats;   // tf32 path: scratch for the re-tiled weight operand, >= N_pad * Cin * ntaps floats (caller-owned)
    float* C2; long long ldc2;        // second output of CMGAN_EPI_SWISH_DUAL
    const unsigned long long* seed_dev;   // optional device counter added to both dropout seeds (CUDA-graph replays draw fresh masks)
    int b_packed;              // tf32 path: 1 = ws already holds the re-tiled weight (cmgan_pack_weights after the optimiser step), skip the re-tiling
} CmganGemmArgs;

// launch plan of the tf32 row GEMM for one argument block (cmgan_gemm_rows_tc_plan; computed on the host, no device involved)
enum CmganRowsMode {
    CMGAN_ROWS_REGISTER = 0,   // LDG -> prologue -> st.shared (pro != NONE)
    CMGAN_ROWS_CPASYNC = 1,    // cp.async row gather (strided / transposed convolutions, epilogues the patch plan does not take)
    CMGAN_ROWS_TMA2D = 2,      // dense rows, one 2-D TMA box per K chunk
    CMGAN_ROWS_PATCH = 3       // same-size convolutions, one 4-D TMA box (patch_w x patch_h positions) per tap and K chunk
};
typedef struct CmganGemmRowsPlan {
    int supported;             // 0: the tensor path does not take these arguments (cmgan_gemm_rows_f32 runs the fp32 FFMA kernel)
    int mode;                  // CmganRowsMode (TMA modes fall back to CMGAN_ROWS_CPASYNC at launch if the driver cannot encode the map)
    int tile_rows, consumers, threads, ctas_per_sm;
    int stages, resident, nchunks, b_tile_bytes;
    int smem_bytes;            // dynamic shared memory per CTA, alignment slack included
    int producer_regs, consumer_regs;   // per thread after the warpgroup register split; entry_regs = the launch-bounds count
    int entry_regs;
    int patch_w, patch_h;      // positions x lines of a patch tile (mode PATCH), else 0
    long long ntiles;
} CmganGemmRowsPlan;

// one weight to re-tile for the tensor-core path (cmgan_pack_weights): same meaning as the B / sb_* / Cin / ntaps / N fields above
typedef struct CmganPackDesc {
    const float* src; float* dst; long long sb_tap, sb_k, sb_n; long long Cin, ntaps, N;
} CmganPackDesc;
