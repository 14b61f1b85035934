/* cmgan_b200 -- C ABI of the H100-native (sm_90a) CMGAN hot path (libcmgan_b200.so).
 *
 * The reference (ruizhecao96/CMGAN) has no FFI layer: its boundary for this path is the nn.Module
 * interface (TSCNet.forward generator.py:174-196, Discriminator.forward discriminator.py:62-64,
 * power_compress / power_uncompress utils.py:20-39, torch.stft / torch.istft call sites
 * train.py:81-112).  These entry points are what a binding for that path calls; every function
 *   - takes raw DEVICE pointers, explicit sizes / strides (in elements) and a cudaStream_t (void*),
 *   - allocates nothing and never synchronises (re-entrant per stream, CUDA-graph capturable),
 *   - returns 0 on success, -1 on error with the message available from cmgan_last_error().
 * Activations are channel-last: row index (b*T + t)*F + f, channels contiguous.
 * One declaration per line (cmgan_b200/_lib.py parses this file to build the ctypes prototypes).
 */
#ifndef CMGAN_B200_H
#define CMGAN_B200_H
#include "../cmgan_b200/csrc/gemm_args.h"

#ifdef __cplusplus
extern "C" {
#endif

const char* cmgan_last_error(void);
int cmgan_abi_version(void);
int cmgan_gemm_args_size(void);
int cmgan_set_tf32_rounding(int on);

/* ---- dense contractions (replace nn.Linear / nn.Conv1d(k=1) / nn.Conv2d and their autograd; gemm_args.h) */
int cmgan_gemm_rows_f32(const CmganGemmArgs* a, void* stream);
int cmgan_gemm_wgrad_f32(const CmganGemmArgs* a, void* stream);
int cmgan_gemm_rows_tc_plan(const CmganGemmArgs* a, CmganGemmRowsPlan* out);
int cmgan_pack_weights(const CmganPackDesc* descs, int n, void* stream);
int cmgan_pack_weight(const float* src, float* dst, long long sb_tap, long long sb_k, long long sb_n, int Cin, int ntaps, int N, void* stream);



/* ---- fused macaron feed-forward (conformer.py:54-72,136-148,211-212): LN -> 64x256 -> Swish, dropout -> 256x64 -> dropout, alpha, residual in ONE wgmma kernel; backward recomputes the hidden layer (ws: M * 66 floats) */
int cmgan_ffn_fwd(const float* x, long long ldx, long long M, const float* ln_g, const float* ln_b, const float* W1p, const float* b1, const float* W2p, const float* b2, float alpha, unsigned long long seed1, unsigned long long seed2, unsigned int thr, float inv_keep, const unsigned long long* seed_dev, float* out, long long ldo, void* stream);
int cmgan_ffn_bwd(const float* x, long long ldx, const float* dz, long long lddz, const float* dout, long long lddo, const float* res2, long long ldr2, long long M, const float* ln_g, const float* ln_b, const float* W1p, const float* b1, const float* W2tp, const float* W1tp, unsigned long long seed1, unsigned int thr, float inv_keep, const unsigned long long* seed_dev, float* dx, long long lddx, float* a_out, float* dh_out, float* xn_out, float* dgamma, float* dbeta, float* ws, void* stream);

/* ---- LayerNorm (conformer.py:68,161,214), InstanceNorm2d (generator.py:35,55,61,128,148), BatchNorm1d (conformer.py:169) */
int cmgan_ln_stats(const float* x, long long ldx, long long M, float* stats, void* stream);
int cmgan_ln_apply(const float* x, long long ldx, long long M, const float* gamma, const float* beta, const float* res, long long ldr, float* y, long long ldy, float* stats, int round_tf32, void* stream);
int cmgan_ln_bwd(const float* dy, long long lddy, const float* x, long long ldx, const float* stats, const float* gamma, long long M, const float* res, long long ldr, const float* res2, long long ldr2, float* dx, long long lddx, float* dgamma, float* dbeta, void* stream);
int cmgan_ln_bwd_drop(const float* dy, long long lddy, const float* x, long long ldx, const float* stats, const float* gamma, long long M, const float* res, long long ldr, const float* res2, long long ldr2, float* dx, long long lddx, float* dgamma, float* dbeta, float* dz, long long lddz, float alpha, unsigned long long seed, unsigned int thr, float inv_keep, const unsigned long long* seed_dev, void* stream);
int cmgan_norm_stats(const float* x, long long ldx, int G, long long rows_per_group, int C, double* sums, void* stream);
int cmgan_norm_finalize(const double* sums, long long n, int G, int C, int mode, const float* gamma, const float* beta, float* running_mean, float* running_var, float momentum, float* scale, float* shift, float* mean_out, float* rstd_out, long long tstride, void* stream);
int cmgan_norm_bwd_reduce(const float* x, long long ldx, const float* dact, long long ldd, int G, long long rows_per_group, int C, int act, const float* scale, const float* shift, const float* mean, const float* rstd, long long tstride, const float* slope, double* S, float* dslope, void* stream);
int cmgan_norm_bwd_apply(const float* x, long long ldx, const float* dact, long long ldd, int G, long long rows_per_group, int C, int act, int use_batch_stats, const float* scale, const float* shift, const float* mean, const float* rstd, long long tstride, const float* slope, const double* S, float* dx, long long lddx, float* dgamma, float* dbeta, void* stream);
int cmgan_norm_apply(const float* x, long long ldx, int G, long long rows_per_group, int C, int act, const float* scale, const float* shift, long long tstride, const float* slope, float* y, long long ldy, void* stream);
int cmgan_norm_stats_ragged(const float* x, long long ldx, int G, long long rows_per_group, int C, long long rows_per_frame, const int* frames, double* sums, void* stream);
int cmgan_norm_finalize_ragged(const double* sums, long long rows_per_frame, int T, const int* frames, int G, int C, const float* gamma, const float* beta, float* scale, float* shift, float* mean_out, float* rstd_out, long long tstride, void* stream);
int cmgan_fill(float* p, long long n, float v, void* stream);
int cmgan_copy_rows(const float* src, long long lds, float* dst, long long ldd, long long M, int C, void* stream);
int cmgan_copy_rows_operand(const float* src, long long lds, float* dst, long long ldd, long long M, int C, void* stream);
int cmgan_add_rows(const float* src, long long lds, float* dst, long long ldd, long long M, int C, void* stream);

/* ---- attention with Shaw relative positions (conformer.py:100-131); axis 0 = time sequences, 1 = frequency sequences */
int cmgan_attention_fwd(const float* qkv, const float* E, int B, int T, int F, int axis, float* ctx, float* lse, void* stream);
int cmgan_attention_fwd_tf32(const float* qkv, const float* E, int B, int T, int F, int axis, float* ctx, float* lse, void* stream);
int cmgan_attention_fwd_ragged(const float* qkv, const float* E, int B, int T, int F, int axis, const int* frames, float* ctx, float* lse, void* stream);
int cmgan_attention_fwd_tf32_ragged(const float* qkv, const float* E, int B, int T, int F, int axis, const int* frames, float* ctx, float* lse, void* stream);
int cmgan_attention_fwd_tf32_nbuf(const float* qkv, const float* E, int B, int T, int F, int axis, float* ctx, float* lse, int nbuf, void* stream);
int cmgan_attention_bwd(const float* qkv, const float* E, const float* ctx, const float* dctx, const float* lse, int B, int T, int F, int axis, float* delta, float* dqkv, float* dE, void* stream);
int cmgan_attention_bwd_tf32_parts(const float* qkv, const float* E, const float* ctx, const float* dctx, const float* lse, int B, int T, int F, int axis, float* delta, float* dqkv, float* dE, int parts, void* stream);
long long cmgan_attention_bwd_ws_floats(int B, int T, int F, int axis);
int cmgan_attention_bwd_tf32_ws(const float* qkv, const float* E, const float* ctx, const float* dctx, const float* lse, int B, int T, int F, int axis, float* delta, float* dqkv, float* dE, int parts, float* scratch, long long scratch_floats, void* stream);
int cmgan_attention_bwd_tf32(const float* qkv, const float* E, const float* ctx, const float* dctx, const float* lse, int B, int T, int F, int axis, float* delta, float* dqkv, float* dE, void* stream);

/* ---- GLU + depthwise conv k=31 (conformer.py:30-48,164-168) */
int cmgan_glu_dwconv_fwd(const float* g, const float* w, const float* bias, int B, int T, int F, int axis, float* out, double* bn_sums, void* stream);
int cmgan_glu_dwconv_fwd_ragged(const float* g, const float* w, const float* bias, int B, int T, int F, int axis, const int* frames, float* out, void* stream);
int cmgan_glu_dwconv_bwd(const float* g, const float* dz, const float* w, int B, int T, int F, int axis, float* dg, float* dw, float* dbias, void* stream);

/* ---- signal front / back end (train.py:75-112, evaluation.py:21-51, utils.py:20-39) */
int cmgan_rms_scale(const float* x, long long ldx, int B, int L, float* c, void* stream);
int cmgan_pad_reflect(const float* x, long long ldx, int B, int L, const float* c, float* xp, int Lp, void* stream);
int cmgan_rms_scale_ragged(const float* x, long long ldx, int B, int L, const int* lengths, float* c, void* stream);
int cmgan_pad_wrap_reflect_ragged(const float* x, long long ldx, int B, int L, const int* lengths, const float* c, float* xp, int Lp, void* stream);
int cmgan_compress(const float* S, int B, int T, float* X, void* stream);
int cmgan_uncompress(const float* re, const float* im, long long sb, long long st, long long sf, int B, int T, float* U, void* stream);
int cmgan_uncompress_bwd(const float* re, const float* im, long long sb, long long st, long long sf, int B, int T, const float* dU, float* dre, float* dim_, int accumulate, void* stream);
int cmgan_power_law(const float* re, const float* im, long long i0, long long i1, long long i2, float* ore, float* oim, long long o0, long long o1, long long o2, int d0, int d1, int d2, float p, void* stream);
int cmgan_power_law_bwd(const float* re, const float* im, long long i0, long long i1, long long i2, const float* gre, const float* gim, long long o0, long long o1, long long o2, float* dre, float* dim_, long long q0, long long q1, long long q2, int d0, int d1, int d2, float p, void* stream);
int cmgan_ola(const float* frames, int B, int T, const float* inv_env, const float* c_div, float* y, long long ldy, void* stream);
int cmgan_ola_ragged(const float* frames, int B, int T, const int* tlen, const float* inv_env, const float* inv_tail, const float* c_div, float* y, long long ldy, void* stream);
int cmgan_ola_bwd(const float* dy, long long lddy, int B, int T, const float* inv_env, float* dframes, void* stream);
/* STFT tables (n_fft 400, hop 100, periodic Hamming), built on the device from float64 arithmetic and rounded to fp32 once; any output may
 * be null.  fwd_basis (400, 402) = [w cos | -w sin]; inv_basis (402, 400) = the one-sided inverse DFT (weights 1, 2, ..., 2, 1; / 400) times
 * the window; inv_env = 1 / overlap-add envelope of T >= 2 frames (100 (T - 1) samples); inv_tail = its last 100 samples for any T >= 3. */
int cmgan_stft_tables(float* fwd_basis, float* inv_basis, int T, float* inv_env, float* inv_tail, void* stream);
/* Crossfade of overlapping windows (cmgan_enhance_overlap; signal.enhance with overlap > 0 runs the same launches).
 * cmgan_crossfade_table: w[m] = sin^2(pi (m + 0.5) / (2 overlap)), m < overlap, computed in float64 on the device and rounded to fp32 once.
 * cmgan_crossfade: window j of k covers samples [j H, j H + S) of a clip of L samples, H = S - overlap, 0 < overlap <= S / 2; y (rows, S)
 *   contiguous holds windows j0 .. j0 + rows - 1.  For n with j = min(n / H, k - 1) in that range and m = n - j H: out[n] = fp32(w[overlap - 1 - m]
 *   y_{j-1}[m + H]) + fp32(w[m] y_j[m]) (two rounded products, a rounded sum) when j >= 1 and m < overlap, else y_j[m].  Unless j0 + rows = k,
 *   the call also writes the first half fp32(w[overlap - 1 - m] y_{j0+rows-1}[m + H]) of the next window's crossfade into out, and the call for
 *   windows from j0 + rows on adds its own half to it: call it for j0 = 0, 1, ... in order.  Writes out[j0 H, ...) and never past L; needs
 *   (k - 1) H + overlap <= L <= (k - 1) H + S (k > 1) and L <= 2^30. */
int cmgan_crossfade_table(float* w, int overlap, void* stream);
int cmgan_crossfade(const float* y, int rows, int j0, int k, int S, int overlap, const float* w, float* out, long long L, void* stream);

/* ---- generator head and tails (generator.py:53,126,136-139,150,175-196) */
int cmgan_head_conv(const float* x, long long sb, long long sc, long long st, long long sf, int B, int T, int F, const float* w, const float* bias, float* out, long long ldo, void* stream);
int cmgan_head_conv_wgrad(const float* x, long long sb, long long sc, long long st, long long sf, int B, int T, int F, const float* draw, long long ldd, float* dw, float* db, void* stream);
int cmgan_rowdot_fwd(const float* in, int B, int T, int Fout, int nout, const float* scale, const float* shift, const float* slope, const float* w, const float* bias, float* out, void* stream);
int cmgan_rowdot_bwd(const float* in, int B, int T, int Fout, int nout, const float* scale, const float* shift, const float* slope, const float* w, const float* dout, float* dact, float* dw, float* dbias, void* stream);
int cmgan_recombine(const float* m1, const float* in_scale, const float* in_shift, const float* a1, const float* fcw, const float* fcb, const float* slope_f, const float* x, long long sb, long long sc, long long st, long long sf, const float* cplx, int B, int T, int F, float* fr, float* fi, void* stream);
int cmgan_recombine_bwd(const float* m1, const float* in_scale, const float* in_shift, const float* a1, const float* fcw, const float* fcb, const float* slope_f, const float* x, long long sb, long long sc, long long st, long long sf, const float* dfr, const float* dfi, long long gb, long long gt, long long gf, int B, int T, int F, float* dcplx, float* dz, float* dslope_f, float* dfcw, float* dfcb, void* stream);

/* ---- input gradients: TSCNet and the signal front end differentiated wrt their inputs (dc / dc_div are accumulated: zero them first).
 * cmgan_tscnet_input_grad: dx (B, 2, T, F) contiguous from dfr / dfi, the mask tail (as cmgan_recombine_bwd) and draw (M, ldd), the gradient of
 *   the raw head-convolution output (16-byte aligned, ldd % 4 == 0); w = the head weight (64, 3).  Where |x| = 0 the magnitude term is 0.
 * cmgan_rms_scale_bwd: dx (+)= -dc c^3 x / L.  cmgan_pad_reflect_bwd: dframes (B*T, 400), T = L / 100 + 1, -> dx = c g and dc += sum g x, the
 *   adjoint of cmgan_pad_reflect and the DFT's framing (c, dc may be null).  cmgan_ola_div_bwd: the gradient of cmgan_ola with c_div (y = its
 *   output; dc may be null). */
int cmgan_tscnet_input_grad(const float* m1, const float* in_scale, const float* in_shift, const float* a1, const float* fcw, const float* fcb, const float* slope_f, const float* x, long long sb, long long sc, long long st, long long sf, const float* dfr, const float* dfi, long long gb, long long gt, long long gf, const float* draw, long long ldd, const float* w, int B, int T, int F, float* dx, void* stream);
int cmgan_rms_scale_bwd(const float* x, long long ldx, int B, int L, const float* c, const float* dc, float* dx, long long lddx, int accumulate, void* stream);
int cmgan_pad_reflect_bwd(const float* dframes, int B, int T, const float* x, long long ldx, int L, const float* c, float* dx, long long lddx, float* dc, void* stream);
int cmgan_ola_div_bwd(const float* dy, long long lddy, int B, int T, const float* inv_env, const float* c_div, const float* y, long long ldy, float* dframes, float* dc, void* stream);

/* ---- discriminator-only pieces (discriminator.py:29-64, utils.py:42-50) and dropout-mask export */
int cmgan_dropout_mask(float* out, long long n, unsigned long long seed, unsigned int thr, void* stream);
int cmgan_stack2(const float* x, long long xb, long long xh, long long xw, const float* y, long long yb, long long yh, long long yw, int B, int H, int W, float* out, void* stream);
int cmgan_unstack2(const float* dxy, long long n, float* dx, float* dy, void* stream);
int cmgan_spectral_norm(const float* W, int R, int Cc, float* u, float* v, int training, float* w_sn, float* sigma, float* uv_out, void* stream);
int cmgan_spectral_norm_bwd(const float* w_sn, const float* dw_sn, int R, int Cc, const float* u, const float* v, const float* sigma, float* dW, void* stream);
int cmgan_norm_maxpool(const float* x, int B, long long rows, int C, const float* scale, const float* shift, const float* slope, float* out, int* arg, void* stream);
int cmgan_maxpool_bwd(const float* dout, const int* arg, int B, long long rows, int C, float* dact, void* stream);
int cmgan_drop_prelu(const float* x, long long n, int C, const float* slope, unsigned long long seed, unsigned int thr, float inv_keep, float* y, const unsigned long long* seed_dev, void* stream);
int cmgan_drop_prelu_bwd(const float* x, const float* dy, long long n, int C, const float* slope, unsigned long long seed, unsigned int thr, float inv_keep, float* dx, float* dslope, const unsigned long long* seed_dev, void* stream);
int cmgan_lsigmoid(const float* x, long long n, const float* slope, float* y, void* stream);
int cmgan_lsigmoid_bwd(const float* x, const float* y, const float* dy, long long n, const float* slope, float* dx, float* dslope, void* stream);

/* ---- losses with fused gradients (train.py:124-174) and flat AdamW (train.py:63-66) */
int cmgan_spec_loss(const float* er, const float* ei, const float* cr, const float* ci, long long per, long long cb, long long n, float w_ri, float w_mag, double* acc, float* d_er, float* d_ei, float* est_mag, float* clean_mag, void* stream);
int cmgan_time_loss(const float* ea, long long lde, const float* clean, long long ldc, int B, int L, float w_t, double* acc, float* d_ea, void* stream);
int cmgan_gen_loss_finalize(const double* acc, double n_spec, double n_time, float w_ri, float w_mag, float w_t, float w_gan, const float* fake, int B, float* loss, float* d_fake, void* stream);
int cmgan_disc_loss(const float* d_max, const float* d_enh, const float* target, int B, float* loss, float* g_max, float* g_enh, void* stream);
int cmgan_mag_bwd_add(const float* er, const float* ei, const float* d_mag, long long gb, long long gt, long long gf, int B, int T, int F, float* d_er, float* d_ei, void* stream);
int cmgan_adamw(float* p, const float* g, float* m, float* v, long long n, float lr, float beta1, float beta2, float eps, float wd, int step, const unsigned long long* step_dev, const float* lr_dev, void* stream);
int cmgan_counter_add(unsigned long long* p, unsigned long long v, void* stream);

/* ---- PESQ-free scoring on the GPU (src/tools/compute_metrics.py: segmental SNR :350-397, STOI :400-471, LLR :277-347, WSS :80-274), float64 like the numpy reference */
int cmgan_ssnr_f64(const double* clean, const double* proc, long long L, int W, int skip, int nfr, double* out, void* stream);
long long cmgan_stoi_scratch_doubles(long long L);
int cmgan_llr_f64(const double* clean, const double* proc, long long L, int W, int skip, int order, int nfr, double* out, void* stream);
int cmgan_wss_f64(const double* clean, const double* proc, long long L, int W, int skip, int nfft, const double* filt, int nfr, double* out, void* stream);
int cmgan_stoi_f64(const double* clean, const double* proc, long long L, const double* h, const int* band_lo, const int* band_hi, double* scratch, double* out, void* stream);

/* ---- module level: TSCNet.forward, inference mode (generator.py:160-196; eval BatchNorm, no dropout) as one call.
 * params = every floating-point state_dict tensor of the reference TSCNet(64, 201) in state_dict order, each starting at a multiple of 4
 * floats (cmgan_tscnet_param_info enumerates key / offset / numel; cmgan_tscnet_param_floats = size of the block).  x is (B, 2, T, F) with
 * element strides (the reference passes a permuted view, train.py:95); outputs are contiguous (B, 1, T, F).  The workspace is caller-owned,
 * 256-byte aligned, at least cmgan_tscnet_workspace_bytes(B, T, F, precision) bytes; precision 0 = exact fp32, 1 = tf32 tensor cores. */
int cmgan_tscnet_param_count(void);
long long cmgan_tscnet_param_floats(void);
int cmgan_tscnet_param_info(int index, const char** key, long long* offset, long long* numel);
long long cmgan_tscnet_workspace_bytes(int B, int T, int F, int precision);
int cmgan_tscnet_fwd(const float* params, const float* x, long long sxb, long long sxc, long long sxt, long long sxf, int B, int T, int F, float* final_real, float* final_imag, void* workspace, long long workspace_bytes, int precision, void* stream);
/* Ragged batch: utterance b occupies frames t < frames[b] of the (B, 2, T, F) grid (frames: device int32[B], 1 <= T_b <= T; values are
 * clamped to [0, T] on the device).  Input frames t >= T_b are never read and may hold anything, NaN included; output frames t >= T_b are
 * unspecified.  Every valid output frame is what cmgan_tscnet_fwd computes for that utterance alone (same kernels, same order; only the
 * order of the double-precision atomic additions of the InstanceNorm statistics may differ).  The workspace is
 * cmgan_tscnet_workspace_bytes(B, T, F, precision): the same buffers as the uniform call.  Returns -1 when B * T * F * 320 >= 2^31 (the
 * encoder's concat buffer is indexed with 32-bit element counts). */
int cmgan_tscnet_fwd_ragged(const float* params, const float* x, long long sxb, long long sxc, long long sxt, long long sxf, int B, int T, int F, const int* frames, float* final_real, float* final_imag, void* workspace, long long workspace_bytes, int precision, void* stream);

/* ---- module level, training: TSCNet.forward with its activations saved, and TSCNet's backward (parameter and input gradients), one call each.
 * cmgan_tscnet_fwd_train, training = 1: the train-mode forward (generator.py:160-196 under model.train()).  Dropout p = 0.2 at the five sites of
 *   every conformer block, with the masks of the counter-based generator (cmgan_dropout_mask) at seed (seed * 1000003 + block * 16 + site + 1)
 *   mod 2^64 (block = 2 (i - 1) + axis for TSCB_i, site 0..4 = ff1 hidden, ff1 out, attention out, ff2 hidden, ff2 out) plus *seed_dev when
 *   seed_dev is not null (a device counter: CUDA-graph replays draw fresh masks).  BatchNorm uses batch statistics and updates running_mean /
 *   running_var in params in place (momentum 0.1, unbiased variance).  num_batches_tracked is not in the block: the caller owns it (at
 *   momentum 0.1 it affects no value).  training = 0: the eval-mode forward (running statistics, no dropout; params untouched) with the
 *   activations saved, for input gradients through a frozen eval-mode model.
 * The workspace (256-byte aligned, >= cmgan_tscnet_train_workspace_bytes(B, T, F, precision), the same for both modes) keeps everything the
 *   backward reads -- the encoder's concat buffer, raw outputs and normalisation tables, every conformer's input and saved activations, the
 *   decoders' concat buffers, raw outputs, tables and sub-pixel outputs, the mask tail -- in a region at its start; scratch lies above it.
 * cmgan_tscnet_bwd: gradients given dfr / dfi (B, 1, T, F) with element strides (sgb, sgt, sgf) (either may be null: zeros, laid out with the
 *   other's strides, which must then span at most B * T * F elements).  grads: a block laid out like params (cmgan_tscnet_param_info);
 *   every parameter gradient is ACCUMULATED into it (+=), running-statistic slots are never written.  grads == NULL: frozen weights, no
 *   weight-gradient GEMM and no head weight gradient runs.  dx: the input gradient, contiguous (B, 2, T, F), or NULL.  Not both NULL.
 *   Preconditions (not checked on the device): it follows a cmgan_tscnet_fwd_train with the same workspace, B, T, F, training, seed, precision,
 *   an unchanged *seed_dev, unchanged params (including the running statistics that forward wrote) and an unchanged x; nothing in between
 *   wrote to the workspace.  Both return -1 (no launch) for null or misaligned pointers (params, grads 16-byte; workspace 256-byte), F != 201,
 *   B or T <= 0, precision not 0 / 1, training not 0 / 1, a workspace smaller than the query, or B * T * F * 320 >= 2^31. */
long long cmgan_tscnet_train_workspace_bytes(int B, int T, int F, int precision);
int cmgan_tscnet_fwd_train(float* params, const float* x, long long sxb, long long sxc, long long sxt, long long sxf, int B, int T, int F, int training, unsigned long long seed, const unsigned long long* seed_dev, float* final_real, float* final_imag, void* workspace, long long workspace_bytes, int precision, void* stream);
int cmgan_tscnet_bwd(const float* params, const float* x, long long sxb, long long sxc, long long sxt, long long sxf, int B, int T, int F, int training, unsigned long long seed, const unsigned long long* seed_dev, const float* dfr, const float* dfi, long long sgb, long long sgt, long long sgf, float* grads, float* dx, void* workspace, long long workspace_bytes, int precision, void* stream);

/* ---- module level, training: the metric discriminator (discriminator.py:29-64, ndf = 16 as train.py:55) forward with its activations saved, and
 * its backward (parameter gradients through the spectral norm, input gradients), one call each.
 * params = the 34 floating-point state_dict tensors of the reference Discriminator(16) in state_dict order, the spectral-norm triplets
 *   weight_orig / weight_u / weight_v included, each starting at a multiple of 4 floats (cmgan_disc_param_info enumerates key / offset / numel).
 * cmgan_disc_fwd: x, y are (B, 1, H, W) magnitudes with element strides (the trainer passes (B, 1, F, T) permuted views of (B, 1, T, F)
 *   buffers; x == y is allowed); out is (B, 1).  H, W >= 16.  training = 1: one power iteration per spectrally normalised weight, weight_u /
 *   weight_v updated in place in params (as torch's spectral_norm in train mode); Dropout(0.3) with the mask of the counter-based generator
 *   (cmgan_dropout_mask) at seed, plus *seed_dev when seed_dev is not null.  training = 0: stored u / v, no dropout, params untouched; the
 *   activations are still saved, so a frozen eval-mode discriminator can be differentiated.
 * The workspace (256-byte aligned, >= cmgan_disc_workspace_bytes(B, H, W, precision), the same for both modes) keeps everything the backward
 *   reads -- the stacked input, every layer's input, raw output and InstanceNorm tables, W / sigma, sigma and the [u | v] THIS forward used for
 *   all six spectrally normalised weights, the pooled features and their arg-max, both linear layers' outputs and out -- in a region at its
 *   start.  Each forward whose backward is still to come needs its own workspace: a later train-mode forward iterates u / v in params again.
 * cmgan_disc_bwd: dout (B, 1) contiguous.  grads: a block laid out like params; every parameter gradient is ACCUMULATED into it (+=), the
 *   weight_u / weight_v slots are never written.  grads == NULL: frozen weights, no weight-gradient GEMM and no spectral-norm backward runs.
 *   dx, dy: the input gradients, contiguous (B, 1, H, W), either may be NULL; not all three NULL.  Preconditions (not checked on the device): it
 *   follows a cmgan_disc_fwd with the same workspace, B, H, W, training, seed, precision and an unchanged *seed_dev; the non-buffer parameters
 *   are unchanged; nothing in between wrote to the workspace.  The backward reads nothing else: x, y, weight_u and weight_v may have changed.
 * precision 0 = exact fp32, 1 = tf32 tensor cores for the convolutions (the two linear layers always run exact fp32).  Both return -1 (no
 *   launch) for null or misaligned pointers (params, grads 16-byte; workspace 256-byte), B <= 0, H or W < 16, precision not 0 / 1, training
 *   not 0 / 1, a workspace smaller than the query, or B * H * W > 2^31 - 128 (the GEMMs count rows in 32 bits). */
int cmgan_disc_param_count(void);
long long cmgan_disc_param_floats(void);
int cmgan_disc_param_info(int index, const char** key, long long* offset, long long* numel);
long long cmgan_disc_workspace_bytes(int B, int H, int W, int precision);
int cmgan_disc_fwd(float* params, const float* x, long long sxb, long long sxh, long long sxw, const float* y, long long syb, long long syh, long long syw, int B, int H, int W, int training, unsigned long long seed, const unsigned long long* seed_dev, float* out, void* workspace, long long workspace_bytes, int precision, void* stream);
int cmgan_disc_bwd(const float* params, int B, int H, int W, int training, unsigned long long seed, const unsigned long long* seed_dev, const float* dout, float* grads, float* dx, float* dy, void* workspace, long long workspace_bytes, int precision, void* stream);

/* ---- module level, training from waveforms: the generator's side of train.py:72-151 around the TSCNet pair above, one call each way.
 * cmgan_gen_wave_fwd: clean, noisy (B, L) fp32 with row strides ldc, ldn >= L.  Runs: c = the noisy batch's RMS scale; the STFT (n_fft 400,
 *   hop 100, exact fp32) and power compression of the noisy and of the clean batch, both scaled by c; TSCNet.forward on the noisy spectrogram
 *   (training / seed / seed_dev / params as cmgan_tscnet_fwd_train, running statistics updated in place in train mode); un-compression and the
 *   inverse STFT into est_audio (B, Lo), Lo = 100 floor(L / 100), row stride lde >= Lo, left at the RMS-scaled level; the spectral loss
 *   (cmgan_spec_loss with w_ri, w_mag), writing est_mag and clean_mag as contiguous (B, 1, T, 201), T = L / 100 + 1; the time loss (cmgan_time_loss
 *   with w_t) of est_audio against the UN-scaled clean[:, :Lo], as the reference's train_step compares them (train.py:188).  acc (3 doubles) is
 *   zeroed by the call and holds the loss sums cmgan_gen_loss_finalize(acc, B * T * 201, B * Lo, ...) turns into the loss.
 * Between the two calls the host runs the GAN term: cmgan_disc_fwd on (B, 1, 201, T) views of clean_mag / est_mag, cmgan_gen_loss_finalize, and
 *   cmgan_disc_bwd with grads = NULL for d_mag; without a discriminator, finalize with fake = NULL and pass d_mag = NULL.
 * cmgan_gen_wave_bwd: d_mag, the gradient wrt est_mag in a (B, 1, 201, T) layout with element strides (sgb along B, sgt along T, sgf along F), or
 *   NULL.  Adds the magnitude term to the spectral-loss gradients, runs the inverse STFT's backward into them and the TSCNet backward; every
 *   parameter gradient is ACCUMULATED into grads (non-null, laid out like params; running-statistic slots never written).  No waveform gradient.
 *   It reads only params, d_mag and the workspace: clean, noisy, est_audio, est_mag and clean_mag may have changed since the forward.  Otherwise
 *   the preconditions of cmgan_tscnet_bwd hold: the same workspace, B, L, training, seed, precision, *seed_dev and unchanged params.
 * The workspace (256-byte aligned, >= cmgan_gen_wave_workspace_bytes(B, L, precision), the same for both modes) starts with a region holding
 *   the STFT tables (regenerated by every forward), the RMS scales, both compressed spectrograms, fr / fi, the spectral-loss gradients and the
 *   time-loss gradient; TSCNet's training layout lies above it.  All three return -1 (no launch) for B <= 0, L <= 200, precision not 0 / 1, or
 *   B * T * 201 * 320 >= 2^31; the calls also for null or misaligned pointers (params, grads 16-byte; workspace 256-byte; d_mag may be NULL),
 *   ldc or ldn < L, lde < Lo, est_audio overlapping clean or noisy, training not 0 / 1 or a workspace smaller than the query.
 * cmgan_cut_batch: the data loader's cut (dataloader.py:32-49) on the device.  Utterance b is corpus[offsets[b] : offsets[b] + lengths[b]]
 *   (offsets, lengths, starts: device arrays); out[b, n], n < cut_len, row stride ldo >= cut_len, is corpus[off + n % len] when len < cut_len
 *   (whole copies, then the first cut_len % len samples), else corpus[off + start + n] with start = starts[b] clamped to [0, len - cut_len]; a
 *   row with len <= 0 is zero-filled.  Nothing outside an utterance is read.  Call it once for the clean and once for the noisy corpus. */
long long cmgan_gen_wave_workspace_bytes(int B, int L, int precision);
int cmgan_gen_wave_fwd(float* params, const float* clean, long long ldc, const float* noisy, long long ldn, int B, int L, int training, unsigned long long seed, const unsigned long long* seed_dev, float w_ri, float w_mag, float w_t, float* est_audio, long long lde, float* est_mag, float* clean_mag, double* acc, void* workspace, long long workspace_bytes, int precision, void* stream);
int cmgan_gen_wave_bwd(const float* params, int B, int L, int training, unsigned long long seed, const unsigned long long* seed_dev, const float* d_mag, long long sgb, long long sgt, long long sgf, float* grads, void* workspace, long long workspace_bytes, int precision, void* stream);
int cmgan_cut_batch(const float* corpus, const long long* offsets, const int* lengths, const int* starts, int B, int cut_len, float* out, long long ldo, void* stream);

/* ---- module level, waveform in / waveform out: evaluation.py:21-53 (enhance_one_track between load and save) as one call.
 * wav (B, L) fp32 with row stride ldw; out (B, L) fp32 with row stride ldo; neither range may overlap the other.  Per clip: RMS scale,
 * wrap padding to a multiple of 100, the STFT, power compression, TSCNet.forward (params / precision as cmgan_tscnet_fwd), un-compression,
 * the inverse STFT, de-normalisation, truncation to the clip's length.  Each clip gets what it would get enhanced alone.
 *   lengths == NULL: B clips of exactly L samples.  A clip whose padded length exceeds cut_len is folded into k segments as the reference
 *     does (k = ceil(padded / cut_len), raised until it divides 100); every out[b, :L] is written.
 *   lengths != NULL: device int32[B], clip b is wav[b, :lengths[b]] (values clamped to [0, L] on the device); wav[b, n >= len_b] is never
 *     read and out[b, n >= len_b] never written.  Needs ceil(L / 100) * 100 <= cut_len (longer clips take the uniform, folding call).  Every
 *     length must satisfy the wrap-padding precondition: padded_b = ceil(len_b / 100) * 100 > 200 and padded_b - len_b <= len_b (any
 *     len_b >= 201 does).  A clip that breaks it gets an unspecified output; nothing out of bounds is touched.
 * The workspace (256-byte aligned) holds the STFT tables, regenerated on every call, and every intermediate; cmgan_enhance_workspace_bytes
 * sizes it for both modes and returns -1 (message in cmgan_last_error) for any shape cmgan_enhance rejects: B <= 0, L <= 200, a folded
 * segment of 200 samples or fewer, a fold that yields fewer than L samples, or rows * T * 201 * 320 >= 2^31 (rows = B, or B k folded; T =
 * segment length / 100 + 1 frames).  Allocates nothing, never synchronises, CUDA-graph capturable. */
long long cmgan_enhance_workspace_bytes(int B, int L, int cut_len, int precision);
int cmgan_enhance(const float* params, const float* wav, long long ldw, int B, int L, const int* lengths, int cut_len, float* out, long long ldo, void* workspace, long long workspace_bytes, int precision, void* stream);

/* ---- module level, waveform in / waveform out for ONE clip of any length in bounded memory: cmgan_enhance's fold, run a few segments at a time.
 * wav, out: L samples on the device; only wav[:L] is read and only out[:L] written; the ranges may not overlap.  The RMS scale is computed once
 * over the whole clip (the kernel and summation order of cmgan_enhance), then the k segments of the fold run in passes of at most max_segments
 * rows through one workspace: padding, STFT, compression, TSCNet.forward, un-compression, inverse STFT and overlap-add into the pass's range
 * of out.  Segments share nothing but the scale, so a pass computes exactly what the single-batch fold computes for its rows.
 *   Fold: padded = ceil(L / 100) * 100.  padded <= cut_len: one segment.  Otherwise the reference's rule (k = ceil(padded / cut_len) raised
 *   until it divides 100, S = padded / k), as cmgan_enhance, wherever it gives a fold: k <= 100 and k 100 floor(S / 100) >= L samples out.
 *   Where it does not -- padded > 100 cut_len, where the reference loops forever, or segments that yield fewer than L samples (any k that does
 *   not divide padded / 100; the reference's own length assertion fails and cmgan_enhance rejects the clip) -- an extension with no reference
 *   behaviour to match: S_max = 100 floor(cut_len / 100), k = ceil(padded / S_max), S = 100 ceil(padded / (100 k)); the clip is wrap-padded
 *   with its own head to k S <= 2 L and the segment outputs tile it without a gap.
 * cmgan_enhance_long_workspace_bytes(cut_len, max_segments, precision) depends on neither L nor the clip: one buffer serves every length.
 * Both return -1 (message in cmgan_last_error; nothing launched) for null or misaligned pointers (params 16-byte, workspace 256-byte),
 * L <= 200 or L > 2^30, cut_len < 300 (no segment of more than 200 samples), max_segments <= 0, max_segments * T_max * 201 * 320 >= 2^31
 * (T_max = floor(cut_len / 100) + 1; 13 segments at cut_len = 16 s), overlapping wav / out, precision not 0 / 1, a workspace smaller than
 * the query, or a fold into segments of 200 samples or fewer (small cut_len only).  Allocates nothing,
 * never synchronises, CUDA-graph capturable. */
long long cmgan_enhance_long_workspace_bytes(int cut_len, int max_segments, int precision);
int cmgan_enhance_long(const float* params, const float* wav, int L, int cut_len, int max_segments, float* out, void* workspace, long long workspace_bytes, int precision, void* stream);

/* ---- sample-rate conversion: scipy.signal.resample_poly(x, up, down) with its default filter, up / down = sr_out / sr_in in lowest terms.
 * Supported: 8000 <= sr_in, sr_out <= 192000 Hz with up, down <= 1024 -- the standard rates 8, 11.025, 12, 16, 22.05, 24, 32, 44.1, 48, 88.2,
 * 96, 176.4 and 192 kHz to and from 16 kHz, and most pairs among them (not 11.025 <-> 32 kHz and its multiples, 1280 / 441); any other pair
 * returns -1 with a message.
 * cmgan_resample_taps_floats: 2 half + 1, half = 10 max(up, down) (12 801 at 11.025 <-> 16 kHz, the largest).
 * cmgan_resample_taps: writes the taps h[m] = firwin(2 half + 1, 1 / max(up, down), window=('kaiser', 5.0))[m] * up into h (device, that many
 *   floats), computed in float64 on the device (sinc times a Kaiser(5) window with a series I0, normalised by its sum) and rounded to fp32 once.
 * cmgan_resample: x (B, L) with row stride ldx >= L -> y (B, ceil(L up / down)) with row stride ldy >= ceil(L up / down); x and y may not
 *   overlap; h = the taps of (sr_in, sr_out).  y[b, n] = sum_i x[b, i] h[down n + half - up i] over the i in [0, len_b) the filter reaches
 *   (zero padding at both ends), summed in increasing i.  lengths == NULL: every len_b = L.  Otherwise device int32[B], clamped to [0, L]:
 *   row b reads only x[b, :len_b] and writes only y[b, :ceil(len_b up / down)]. */
int cmgan_resample_taps_floats(int sr_in, int sr_out);
int cmgan_resample_taps(int sr_in, int sr_out, float* h, void* stream);
int cmgan_resample(const float* x, long long ldx, int B, long long L, const int* lengths, int sr_in, int sr_out, const float* h, float* y, long long ldy, void* stream);

/* ---- module level, waveform in / waveform out at any supported sample rate sr (the list above): the entries above around the 16 kHz model.
 * cmgan_enhance_sr: the clips are resampled to 16 kHz into the workspace (L16 = ceil(L 16000 / sr) samples; a ragged batch's 16 kHz lengths
 *   are computed on the device), cmgan_enhance runs on them in the rest of the workspace, and its 16 kHz output is resampled back into out and
 *   cut to each clip's length: out[b, :L] (ragged: out[b, :lengths[b]], nothing past it written).  The result is bit for bit cmgan_resample ->
 *   cmgan_enhance -> cmgan_resample.  The fold, the ragged limit and every rejection of cmgan_enhance apply to L16; cut_len counts 16 kHz
 *   samples.  Also -1 for an unsupported sr or L16 >= 2^31.
 * cmgan_enhance_long_sr: the same around cmgan_enhance_long for one clip of L samples at sr; L may pass 2^30 as long as L16 <= 2^30.  The
 *   workspace is cmgan_enhance_long's pass workspace, whose size does not depend on L, plus the 16 kHz copies of the whole clip, in and out
 *   (8 bytes per 16 kHz sample: about 460 MB per hour).  Both copies are needed: the wrap padding of the fold reads the clip's head in the
 *   last pass.  The activations stay bounded by max_segments as in cmgan_enhance_long; only the copies grow with L.
 * At sr = 16000 each entry is exactly its 16 kHz counterpart (the same launches) and each query returns the same size.  The queries return -1
 * for any shape their entry rejects.  Allocates nothing, never synchronises, CUDA-graph capturable. */
long long cmgan_enhance_sr_workspace_bytes(int B, int L, int sr, int cut_len, int precision);
int cmgan_enhance_sr(const float* params, const float* wav, long long ldw, int B, int L, const int* lengths, int sr, int cut_len, float* out, long long ldo, void* workspace, long long workspace_bytes, int precision, void* stream);
long long cmgan_enhance_long_sr_workspace_bytes(long long L, int sr, int cut_len, int max_segments, int precision);
int cmgan_enhance_long_sr(const float* params, const float* wav, long long L, int sr, int cut_len, int max_segments, float* out, void* workspace, long long workspace_bytes, int precision, void* stream);

/* ---- module level, ONE clip of any length at any supported sample rate, with overlapping windows joined by a crossfade: no output sample
 * depends on a window edge alone.  All lengths below count 16 kHz samples; at another sr the clip is resampled to 16 kHz first and back
 * afterwards, exactly as cmgan_enhance_long_sr does (the workspace holds the same 16 kHz copies).
 *   overlap = 0: cmgan_enhance_long_sr (at 16 kHz cmgan_enhance_long): the same launches, and the query returns the same size.
 *   overlap = O > 0: a multiple of 100 with 100 <= O and 2 O <= S_max = 100 floor(cut_len / 100), cut_len >= 300.  With padded =
 *   ceil(L / 100) * 100 (200 < L <= 2^30, padded - L <= L):
 *     padded <= S_max: one window of S = padded samples, the one-segment case of cmgan_enhance_long (the same launches);
 *     otherwise S = S_max, hop H = S - O, k = 1 + ceil((padded - S) / H) windows, window j covering [j H, j H + S) of the clip wrap-padded
 *     with its own head to Lw = (k - 1) H + S (rejected when Lw - L > L).
 *   Window j: scaled by the RMS scale c of the WHOLE clip (cmgan_enhance_long's kernel and order), reflect-padded by 200 at its own edges,
 *   STFT, compression, TSCNet.forward, un-compression, inverse STFT and overlap-add divided by c: y_j, S samples.  The windows are joined by
 *   cmgan_crossfade with w = cmgan_crossfade_table(O): out[n] = fp32(w[O - 1 - m] y_{j-1}[m + H]) + fp32(w[m] y_j[m]) in the first O samples
 *   of every window but the first, y_j[m] elsewhere (j = min(n / H, k - 1), m = n - j H).
 *   The windows run at most max_segments at a time (the 2^31 bound of cmgan_enhance_long: 13 at cut_len = 16 s); the output does not depend
 *   on max_segments.  At 16 kHz the workspace does not depend on L.  Only wav[:L] is read and only out[:L] written; the ranges may not overlap.
 * Both return -1 (message in cmgan_last_error; nothing launched) for a bad overlap or cut_len, L out of range, an unsupported sr, null or
 * misaligned pointers (params 16-byte, workspace 256-byte), max_segments <= 0 or past the 2^31 bound, precision not 0 / 1, overlapping wav /
 * out, or a workspace smaller than the query.  Allocates nothing, never synchronises, CUDA-graph capturable. */
long long cmgan_enhance_overlap_workspace_bytes(long long L, int sr, int cut_len, int overlap, int max_segments, int precision);
int cmgan_enhance_overlap(const float* params, const float* wav, long long L, int sr, int cut_len, int overlap, int max_segments, float* out, void* workspace, long long workspace_bytes, int precision, void* stream);

#ifdef __cplusplus
}
#endif
#endif
