/* Speech enhancement from a non-Python host (plain C99): one noisy mono clip in, the enhanced clip out, through the waveform-level entry
 * cmgan_enhance of libcmgan_b200.so (evaluation.py:21-53 as one call), or through cmgan_enhance_long, which runs a clip of any length a few
 * folded segments at a time in a workspace whose size does not depend on the length; at a sample rate other than 16 kHz through
 * cmgan_enhance_sr / cmgan_enhance_long_sr, which resample on the device around them; or, given an overlap, through cmgan_enhance_overlap,
 * which cuts the long clip into overlapping windows and joins them with a raised-cosine crossfade instead of folding it.
 *   Build:  gcc -std=c99 -Iinclude examples/c_enhance.c -o c_enhance -Lcmgan_b200 -lcmgan_b200 -Wl,-rpath,$PWD/cmgan_b200
 *           (add -DWITH_CUDA -I/usr/local/cuda/include -L/usr/local/cuda/lib64 -lcudart to enhance a clip).
 *   Run:    c_enhance [params.f32 noisy.f32 enhanced.f32 [precision [cut_len [max_segments [sr [overlap]]]]]]
 *           (max_segments > 0 switches to cmgan_enhance_long with passes of at most that many segments; sr = the clip's sample rate, 16000
 *           by default; cut_len counts 16 kHz samples; overlap > 0, in 16 kHz samples, a multiple of 100, switches the long mode to
 *           cmgan_enhance_overlap)
 *           c_enhance sr  only prints the workspace queries, those of the sample-rate entries at sr.
 * params.f32 is a raw little-endian float32 dump of the parameter block (cmgan_b200.module_abi.pack_params(...).cpu().numpy().tofile(path));
 * noisy.f32 / enhanced.f32 are raw little-endian float32 samples at sr (the reference reads 16-bit wav files and divides by 32768).
 * Without WITH_CUDA only the host-side workspace queries and argument checks run (no GPU needed). */
#include <stdio.h>
#include <stdlib.h>

#include "cmgan_b200.h"

#ifdef WITH_CUDA
#include <cuda_runtime.h>
#endif

static int query(int B, int L, int cut_len, const char* what) {
    const long long ws = cmgan_enhance_workspace_bytes(B, L, cut_len, 1);
    if (ws < 0) {
        fprintf(stderr, "%s\n", cmgan_last_error());
        return 1;
    }
    printf("workspace %s B=%d L=%d cut_len=%d tf32: %lld bytes\n", what, B, L, cut_len, ws);
    return 0;
}

int main(int argc, char** argv) {
    if (query(1, 16000, 16000 * 16, "uniform") || query(16, 32000, 16000 * 16, "uniform / ragged") || query(1, 3950, 1000, "folded"))
        return 1;
    /* a fold of 1700 samples into 2 segments of 850 yields 2 * 800 samples: rejected, as the reference's own length assertion would */
    if (cmgan_enhance_workspace_bytes(1, 1700, 1000, 1) >= 0) { fprintf(stderr, "a short fold must be rejected\n"); return 1; }
    printf("rejected L=1700 cut_len=1000: %s\n", cmgan_last_error());
    if (cmgan_enhance(NULL, NULL, 0, 1, 16000, NULL, 16000 * 16, NULL, 0, NULL, 0, 1, NULL) == 0) { fprintf(stderr, "null pointers must be rejected\n"); return 1; }
    printf("rejected call: %s\n", cmgan_last_error());
    /* the long entry's workspace depends on cut_len, max_segments and precision only; at 16 s, 13 segments are the most one pass takes */
    const int segs[4] = {1, 4, 8, 13};
    for (int i = 0; i < 4; ++i) {
        const int m = segs[i];
        const long long ws = cmgan_enhance_long_workspace_bytes(16000 * 16, m, 1);
        if (ws < 0) { fprintf(stderr, "%s\n", cmgan_last_error()); return 1; }
        printf("workspace long cut_len=%d max_segments=%d tf32: %lld bytes\n", 16000 * 16, m, ws);
    }
    if (cmgan_enhance_long_workspace_bytes(16000 * 16, 14, 1) >= 0) { fprintf(stderr, "14 segments of 16 s must be rejected\n"); return 1; }
    printf("rejected max_segments=14: %s\n", cmgan_last_error());
    /* the sample-rate entries: at 16 kHz the same sizes as above; the long one grows with the clip (its 16 kHz copies, in and out) */
    const int qsr = argc == 2 ? atoi(argv[1]) : 48000;
    const long long ws_sr = cmgan_enhance_sr_workspace_bytes(1, qsr, qsr, 16000 * 16, 1);
    const long long ws_long_sr = cmgan_enhance_long_sr_workspace_bytes(3600LL * qsr, qsr, 16000 * 16, 13, 1);
    if (ws_sr < 0 || ws_long_sr < 0) { fprintf(stderr, "%s\n", cmgan_last_error()); return 1; }
    printf("workspace sr=%d uniform B=1 L=%d cut_len=%d tf32: %lld bytes\n", qsr, qsr, 16000 * 16, ws_sr);
    printf("workspace sr=%d long L=%lld cut_len=%d max_segments=13 tf32: %lld bytes\n", qsr, 3600LL * qsr, 16000 * 16, ws_long_sr);
    /* the crossfaded windows: at 16 kHz one size for every length, as the long entry; overlap 0 is the long entry itself */
    const int ovl[3] = {0, 8000, 16000};
    for (int i = 0; i < 3; ++i) {
        const long long ws = cmgan_enhance_overlap_workspace_bytes(3600LL * 16000, 16000, 16000 * 16, ovl[i], 13, 1);
        if (ws < 0) { fprintf(stderr, "%s\n", cmgan_last_error()); return 1; }
        printf("workspace overlap=%d cut_len=%d max_segments=13 tf32: %lld bytes\n", ovl[i], 16000 * 16, ws);
    }
    if (cmgan_enhance_overlap_workspace_bytes(3600LL * 16000, 16000, 16000 * 16, 150, 13, 1) >= 0) { fprintf(stderr, "overlap 150 must be rejected\n"); return 1; }
    printf("rejected overlap=150: %s\n", cmgan_last_error());
#ifdef WITH_CUDA
    if (argc > 3) {
        const int precision = argc > 4 ? atoi(argv[4]) : 1, cut_len = argc > 5 ? atoi(argv[5]) : 16000 * 16;
        const int max_segments = argc > 6 ? atoi(argv[6]) : 0, sr = argc > 7 ? atoi(argv[7]) : 16000, overlap = argc > 8 ? atoi(argv[8]) : 0;
        const long long total = cmgan_tscnet_param_floats();
        float* hp = (float*)malloc((size_t)total * 4);
        FILE* f = fopen(argv[1], "rb");
        if (!f || fread(hp, 4, (size_t)total, f) != (size_t)total) { fprintf(stderr, "cannot read %s\n", argv[1]); return 1; }
        fclose(f);
        f = fopen(argv[2], "rb");
        if (!f) { fprintf(stderr, "cannot read %s\n", argv[2]); return 1; }
        fseek(f, 0, SEEK_END);
        const int L = (int)(ftell(f) / 4);
        fseek(f, 0, SEEK_SET);
        float* hx = (float*)malloc((size_t)L * 4);
        if (L <= 0 || fread(hx, 4, (size_t)L, f) != (size_t)L) { fprintf(stderr, "cannot read %s\n", argv[2]); return 1; }
        fclose(f);
        const long long ws = max_segments > 0 ? (overlap > 0 ? cmgan_enhance_overlap_workspace_bytes(L, sr, cut_len, overlap, max_segments, precision)
                                                             : cmgan_enhance_long_sr_workspace_bytes(L, sr, cut_len, max_segments, precision))
                                              : cmgan_enhance_sr_workspace_bytes(1, L, sr, cut_len, precision);
        if (ws < 0) { fprintf(stderr, "%s\n", cmgan_last_error()); return 1; }
        float *params, *x, *y;
        void* wsp;
        if (cudaMalloc((void**)&params, (size_t)total * 4) != cudaSuccess || cudaMalloc((void**)&x, (size_t)L * 4) != cudaSuccess ||
            cudaMalloc((void**)&y, (size_t)L * 4) != cudaSuccess || cudaMalloc(&wsp, (size_t)ws) != cudaSuccess) {
            fprintf(stderr, "cudaMalloc failed\n");
            return 1;
        }
        cudaMemcpy(params, hp, (size_t)total * 4, cudaMemcpyHostToDevice);
        cudaMemcpy(x, hx, (size_t)L * 4, cudaMemcpyHostToDevice);
        const int rc = max_segments > 0 ? (overlap > 0 ? cmgan_enhance_overlap(params, x, L, sr, cut_len, overlap, max_segments, y, wsp, ws, precision, 0)
                                                       : cmgan_enhance_long_sr(params, x, L, sr, cut_len, max_segments, y, wsp, ws, precision, 0))
                                        : cmgan_enhance_sr(params, x, L, 1, L, NULL, sr, cut_len, y, L, wsp, ws, precision, 0);
        if (rc) { fprintf(stderr, "%s\n", cmgan_last_error()); return 1; }
        if (cudaMemcpy(hx, y, (size_t)L * 4, cudaMemcpyDeviceToHost) != cudaSuccess) { fprintf(stderr, "device error\n"); return 1; }
        f = fopen(argv[3], "wb");
        if (!f || fwrite(hx, 4, (size_t)L, f) != (size_t)L) { fprintf(stderr, "cannot write %s\n", argv[3]); return 1; }
        fclose(f);
        printf("enhanced %d samples (precision %d, workspace %lld bytes%s)\n", L, precision, ws, max_segments > 0 ? ", long entry" : "");
        if (max_segments > 0 && overlap > 0) printf("crossfaded windows: overlap %d samples at 16 kHz\n", overlap);
        cudaFree(params); cudaFree(x); cudaFree(y); cudaFree(wsp);
        free(hp); free(hx);
    }
#endif
    return 0;
}
