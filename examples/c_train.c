/* Training the generator from a non-Python host (plain C99): K steps of the spectral loss on one batch, each step one train-mode forward
 * (cmgan_tscnet_fwd_train), the loss and its gradient (cmgan_spec_loss, cmgan_gen_loss_finalize), one backward (cmgan_tscnet_bwd) and AdamW
 * (cmgan_adamw) over the parameter block, all on one stream of libcmgan_b200.so.
 *   Build:  gcc -std=c99 -Iinclude examples/c_train.c -o c_train -Lcmgan_b200 -lcmgan_b200 -Wl,-rpath,$PWD/cmgan_b200
 *           (add -DWITH_CUDA -I/usr/local/cuda/include -L/usr/local/cuda/lib64 -lcudart to train).
 *   Run:    c_train [params.f32 x.f32 target.f32 B T steps precision out.f32 [lr]]
 * params.f32 is a raw little-endian float32 dump of the parameter block (cmgan_b200.module_abi.pack_params(...).cpu().numpy().tofile(path));
 * x.f32 / target.f32 are contiguous (B, 2, T, 201) float32 compressed spectrograms of the noisy and the clean batch (real, imaginary planes).
 * The trained block (running statistics included) is written to out.f32.  Without WITH_CUDA only the host-side workspace queries and argument
 * checks run (no GPU needed). */
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "cmgan_b200.h"

#ifdef WITH_CUDA
#include <cuda_runtime.h>
#endif

#define NF 201

static int query(int B, int T, int precision) {
    const long long ws = cmgan_tscnet_train_workspace_bytes(B, T, NF, precision);
    if (ws < 0) {
        fprintf(stderr, "%s\n", cmgan_last_error());
        return 1;
    }
    printf("training workspace B=%d T=%d %s: %lld bytes\n", B, T, precision ? "tf32" : "fp32", ws);
    return 0;
}

#ifdef WITH_CUDA
static float* read_floats(const char* path, long long n) {
    float* h = (float*)malloc((size_t)n * 4);
    FILE* f = fopen(path, "rb");
    if (!h || !f || fread(h, 4, (size_t)n, f) != (size_t)n) {
        fprintf(stderr, "cannot read %lld floats from %s\n", n, path);
        exit(1);
    }
    fclose(f);
    return h;
}

static void* dev_alloc(size_t bytes) {
    void* p = NULL;
    if (cudaMalloc(&p, bytes) != cudaSuccess) {
        fprintf(stderr, "cudaMalloc of %zu bytes failed\n", bytes);
        exit(1);
    }
    return p;
}

#define CHECK(call)                                                  \
    do {                                                             \
        if ((call) != 0) {                                           \
            fprintf(stderr, "%s\n", cmgan_last_error());             \
            return 1;                                                \
        }                                                            \
    } while (0)

/* AdamW over every parameter; the BatchNorm running statistics are buffers, not parameters: the segments skip them */
static int adamw_segments(float* p, const float* g, float* m, float* v, float lr, const unsigned long long* step_dev) {
    const int n = cmgan_tscnet_param_count();
    long long start = 0;
    for (int i = 0; i <= n; ++i) {
        const char* key = NULL;
        long long off = cmgan_tscnet_param_floats(), numel = 0;
        if (i < n) cmgan_tscnet_param_info(i, &key, &off, &numel);
        if (i == n || strstr(key, "running_")) {
            if (off > start && cmgan_adamw(p + start, g + start, m + start, v + start, off - start, lr, 0.9f, 0.999f, 1e-8f, 0.01f, 1, step_dev, NULL, 0))
                return 1;
            if (i < n) start = off + (numel + 3) / 4 * 4;
        }
    }
    return 0;
}

static int train(char** argv, int argc) {
    const int B = atoi(argv[4]), T = atoi(argv[5]), K = atoi(argv[6]), precision = atoi(argv[7]);
    const float lr = argc > 9 ? (float)atof(argv[9]) : 5e-4f;
    const float w_ri = 0.1f, w_mag = 0.9f;             /* loss weights of the reference trainer (train.py:124-174), w_t = w_gan = 0 here */
    const unsigned long long seed = 1234;
    const long long total = cmgan_tscnet_param_floats(), plane = (long long)T * NF, n = (long long)B * plane;
    const long long ws = cmgan_tscnet_train_workspace_bytes(B, T, NF, precision);
    if (ws < 0) { fprintf(stderr, "%s\n", cmgan_last_error()); return 1; }
    float* hp = read_floats(argv[1], total);
    float* hx = read_floats(argv[2], 2 * n);
    float* ht = read_floats(argv[3], 2 * n);
    float *p = (float*)dev_alloc((size_t)total * 4), *g = (float*)dev_alloc((size_t)total * 4), *m = (float*)dev_alloc((size_t)total * 4),
          *v = (float*)dev_alloc((size_t)total * 4);
    float *x = (float*)dev_alloc((size_t)n * 8), *tg = (float*)dev_alloc((size_t)n * 8);
    float *fr = (float*)dev_alloc((size_t)n * 4), *fi = (float*)dev_alloc((size_t)n * 4), *der = (float*)dev_alloc((size_t)n * 4),
          *dei = (float*)dev_alloc((size_t)n * 4), *loss = (float*)dev_alloc(4);
    double* acc = (double*)dev_alloc(3 * sizeof(double));
    unsigned long long* step = (unsigned long long*)dev_alloc(8);
    void* wsp = dev_alloc((size_t)ws);
    cudaMemcpy(p, hp, (size_t)total * 4, cudaMemcpyHostToDevice);
    cudaMemcpy(x, hx, (size_t)n * 8, cudaMemcpyHostToDevice);
    cudaMemcpy(tg, ht, (size_t)n * 8, cudaMemcpyHostToDevice);
    cudaMemset(m, 0, (size_t)total * 4);
    cudaMemset(v, 0, (size_t)total * 4);
    cudaMemset(step, 0, 8);
    for (int k = 0; k < K; ++k) {
        CHECK(cmgan_fill(g, total, 0.f, 0));
        CHECK(cmgan_counter_add(step, 1, 0));          /* AdamW's step and the dropout seed offset */
        CHECK(cmgan_tscnet_fwd_train(p, x, 2 * plane, plane, NF, 1, B, T, NF, 1, seed, step, fr, fi, wsp, ws, precision, 0));
        if (cudaMemsetAsync(acc, 0, 3 * sizeof(double), 0) != cudaSuccess) { fprintf(stderr, "cudaMemsetAsync failed\n"); return 1; }
        CHECK(cmgan_spec_loss(fr, fi, tg, tg + plane, plane, 2 * plane, n, w_ri, w_mag, acc, der, dei, NULL, NULL, 0));
        CHECK(cmgan_gen_loss_finalize(acc, (double)n, 1.0, w_ri, w_mag, 0.f, 0.f, NULL, B, loss, NULL, 0));
        CHECK(cmgan_tscnet_bwd(p, x, 2 * plane, plane, NF, 1, B, T, NF, 1, seed, step, der, dei, plane, NF, 1, g, NULL, wsp, ws, precision, 0));
        CHECK(adamw_segments(p, g, m, v, lr, step));
        float hl = 0.f;
        if (cudaMemcpy(&hl, loss, 4, cudaMemcpyDeviceToHost) != cudaSuccess) { fprintf(stderr, "device error\n"); return 1; }
        printf("step %d loss %.9g\n", k + 1, hl);
    }
    if (cudaMemcpy(hp, p, (size_t)total * 4, cudaMemcpyDeviceToHost) != cudaSuccess) { fprintf(stderr, "device error\n"); return 1; }
    FILE* f = fopen(argv[8], "wb");
    if (!f || fwrite(hp, 4, (size_t)total, f) != (size_t)total) { fprintf(stderr, "cannot write %s\n", argv[8]); return 1; }
    fclose(f);
    printf("trained %d steps (B=%d T=%d precision %d, workspace %lld bytes)\n", K, B, T, precision, ws);
    cudaFree(p); cudaFree(g); cudaFree(m); cudaFree(v); cudaFree(x); cudaFree(tg); cudaFree(fr); cudaFree(fi); cudaFree(der); cudaFree(dei);
    cudaFree(loss); cudaFree(acc); cudaFree(step); cudaFree(wsp);
    free(hp); free(hx); free(ht);
    return 0;
}
#endif

int main(int argc, char** argv) {
    for (int precision = 0; precision <= 1; ++precision)
        if (query(4, 321, precision) || query(16, 321, precision)) return 1;
    if (cmgan_tscnet_train_workspace_bytes(4, 321, 200, 1) >= 0) { fprintf(stderr, "F = 200 must be rejected\n"); return 1; }
    printf("rejected F=200: %s\n", cmgan_last_error());
    if (cmgan_tscnet_bwd(NULL, NULL, 0, 0, 0, 0, 1, 101, NF, 1, 0, NULL, NULL, NULL, 0, 0, 0, NULL, NULL, NULL, 0, 1, NULL) == 0) {
        fprintf(stderr, "a call with nothing to compute must be rejected\n");
        return 1;
    }
    printf("rejected call: %s\n", cmgan_last_error());
#ifdef WITH_CUDA
    if (argc > 8) return train(argv, argc);
#else
    (void)argc;
    (void)argv;
#endif
    return 0;
}
