// Whole-clip front / back end launchers of frontend.cu used by the module-level enhance walk (tscnet_module.cu).  Library-internal (hidden
// visibility): the C ABI exposes them only through cmgan_enhance.  Each returns 0 or -1 with cmgan_last_error() set.
#pragma once
#include <cuda_runtime.h>

// cmgan_rms_scale_ragged that also writes each clip's frame count tlen[b] = ceil(L_b / 100) + 1 (L_b = lengths[b] clamped to [0, L])
int cmgan_rms_scale_frames(const float* x, long long ldx, int B, int L, const int* lengths, float* c, int* tlen, cudaStream_t st);
// B clips of L samples, each wrap-padded with its own head and cut into segments of S samples, segment r starting at sample r hop (hop = S:
// the fold; hop < S: overlapping windows): segments [seg0, seg0 + k) of every clip become rows (B k, Lp)
int cmgan_pad_wrap_reflect_fold(const float* x, long long ldx, int B, int L, int k, int S, int seg0, int hop, const float* c, float* xp,
                                int Lp, cudaStream_t st);
// overlap-add of rows = B k folded segments of T frames, written into y (B, L) at row stride ldy, de-normalised by c_div[clip]; a pass that
// starts at segment seg0 of one clip passes y + seg0 * 100 (T - 1) and L - seg0 * 100 (T - 1)
int cmgan_ola_fold(const float* frames, int rows, int T, int k, const float* inv_env, const float* c_div, float* y, long long ldy, int L,
                   cudaStream_t st);
// ragged overlap-add written into y (B, L): clip b gets its samples n < lengths[b] (clamped to [0, L]), nothing past them
int cmgan_ola_ragged_lengths(const float* frames, int B, int T, const int* tlen, const int* lengths, int L, const float* inv_env,
                             const float* inv_tail, const float* c_div, float* y, long long ldy, cudaStream_t st);
