/* One MetricGAN training loop from a non-Python host (plain C99): K steps on one spectrogram batch, all on one stream of libcmgan_b200.so.
 * Each step is the reference train_step (train.py:176-205) without the time-domain loss, as examples/c_train.c:
 *   generator step:     cmgan_tscnet_fwd_train, cmgan_spec_loss (which also writes est_mag / clean_mag), the train-mode discriminator on
 *                       (clean_mag, est_mag) (cmgan_disc_fwd), cmgan_gen_loss_finalize with w_gan = 0.05, the discriminator's input gradient with
 *                       frozen weights (cmgan_disc_bwd, grads = NULL), cmgan_mag_bwd_add, cmgan_tscnet_bwd, AdamW over the generator block
 *                       (skipping the BatchNorm running statistics);
 *   discriminator step: on the same, detached est_mag: cmgan_disc_fwd on (clean, est) and on (clean, clean) into two workspaces,
 *                       cmgan_disc_loss against the PESQ target, both cmgan_disc_bwd into the discriminator's gradient block, AdamW at 2 lr
 *                       (skipping the spectral-norm vectors weight_u / weight_v, which weight decay would otherwise move).
 * What stays with the host: the PESQ scores (here one constant target for the whole batch, given on the command line), the time-domain loss
 * through the inverse STFT, and any all-reduce across GPUs.
 *   Build:  gcc -std=c99 -Iinclude examples/c_gan_train.c -o c_gan_train -Lcmgan_b200 -lcmgan_b200 -Wl,-rpath,$PWD/cmgan_b200
 *           (add -DWITH_CUDA -I/usr/local/cuda/include -L/usr/local/cuda/lib64 -lcudart to train).
 *   Run:    c_gan_train [gen.f32 disc.f32 x.f32 target.f32 B T steps precision pesq gen_out.f32 disc_out.f32 [lr]]
 * gen.f32 / disc.f32 are raw little-endian float32 dumps of the two parameter blocks (cmgan_b200.module_abi.pack_params(...) and
 * pack_disc_params(...), .cpu().numpy().tofile(path)); x.f32 / target.f32 are contiguous (B, 2, T, 201) float32 compressed spectrograms of
 * the noisy and the clean batch (real, imaginary planes).  Both trained blocks are written out.  Without WITH_CUDA only the host-side
 * workspace queries and argument checks run (no GPU needed). */
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "cmgan_b200.h"

#ifdef WITH_CUDA
#include <cuda_runtime.h>
#endif

#define NF 201

static int query(int B, int T, int precision) {
    const long long wg = cmgan_tscnet_train_workspace_bytes(B, T, NF, precision), wd = cmgan_disc_workspace_bytes(B, NF, T, precision);
    if (wg < 0 || wd < 0) {
        fprintf(stderr, "%s\n", cmgan_last_error());
        return 1;
    }
    printf("workspaces B=%d T=%d %s: generator %lld bytes, discriminator %lld bytes\n", B, T, precision ? "tf32" : "fp32", wg, wd);
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

static int write_floats(const char* path, const float* d, long long n) {
    float* h = (float*)malloc((size_t)n * 4);
    if (!h || cudaMemcpy(h, d, (size_t)n * 4, cudaMemcpyDeviceToHost) != cudaSuccess) { fprintf(stderr, "device error\n"); return 1; }
    FILE* f = fopen(path, "wb");
    if (!f || fwrite(h, 4, (size_t)n, f) != (size_t)n) { fprintf(stderr, "cannot write %s\n", path); return 1; }
    fclose(f);
    free(h);
    return 0;
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

typedef int (*InfoFn)(int, const char**, long long*, long long*);

/* AdamW over every parameter of a block; the slots whose key contains `skip1` or `skip2` are buffers, not parameters: the segments skip them */
static int adamw_segments(float* p, const float* g, float* m, float* v, int n, long long total, InfoFn info, const char* skip1, const char* skip2,
                          float lr, const unsigned long long* step_dev) {
    long long start = 0;
    for (int i = 0; i <= n; ++i) {
        const char* key = NULL;
        long long off = total, numel = 0;
        if (i < n) info(i, &key, &off, &numel);
        if (i == n || strstr(key, skip1) || (skip2 && strstr(key, skip2))) {
            if (off > start && cmgan_adamw(p + start, g + start, m + start, v + start, off - start, lr, 0.9f, 0.999f, 1e-8f, 0.01f, 1, step_dev, NULL, 0))
                return 1;
            if (i < n) start = off + (numel + 3) / 4 * 4;
        }
    }
    return 0;
}

static int train(char** argv, int argc) {
    const int B = atoi(argv[5]), T = atoi(argv[6]), K = atoi(argv[7]), precision = atoi(argv[8]);
    const float pesq = (float)atof(argv[9]);
    const float lr = argc > 12 ? (float)atof(argv[12]) : 5e-4f;
    const float w_ri = 0.1f, w_mag = 0.9f, w_gan = 0.05f;     /* loss weights of the reference trainer (train.py:124-174); w_t = 0 here */
    const unsigned long long seed = 1234, dseed = 1234 * 31 + 5;
    const long long ng = cmgan_tscnet_param_floats(), nd = cmgan_disc_param_floats(), plane = (long long)T * NF, n = (long long)B * plane;
    const long long wsg = cmgan_tscnet_train_workspace_bytes(B, T, NF, precision), wsd = cmgan_disc_workspace_bytes(B, NF, T, precision);
    if (wsg < 0 || wsd < 0) { fprintf(stderr, "%s\n", cmgan_last_error()); return 1; }
    float* hg = read_floats(argv[1], ng);
    float* hd = read_floats(argv[2], nd);
    float* hx = read_floats(argv[3], 2 * n);
    float* ht = read_floats(argv[4], 2 * n);
    float *pg = (float*)dev_alloc((size_t)ng * 4), *gg = (float*)dev_alloc((size_t)ng * 4), *mg = (float*)dev_alloc((size_t)ng * 4),
          *vg = (float*)dev_alloc((size_t)ng * 4);
    float *pd = (float*)dev_alloc((size_t)nd * 4), *gd = (float*)dev_alloc((size_t)nd * 4), *md = (float*)dev_alloc((size_t)nd * 4),
          *vd = (float*)dev_alloc((size_t)nd * 4);
    float *x = (float*)dev_alloc((size_t)n * 8), *tg = (float*)dev_alloc((size_t)n * 8);
    float *fr = (float*)dev_alloc((size_t)n * 4), *fi = (float*)dev_alloc((size_t)n * 4), *der = (float*)dev_alloc((size_t)n * 4),
          *dei = (float*)dev_alloc((size_t)n * 4), *est = (float*)dev_alloc((size_t)n * 4), *cln = (float*)dev_alloc((size_t)n * 4),
          *dmag = (float*)dev_alloc((size_t)n * 4);
    float* sc = (float*)dev_alloc(64 * 4 + (size_t)B * 4 * 8);        /* two losses, then seven (B,) vectors */
    float *gloss = sc, *dloss = sc + 32, *fake = sc + 64, *dfake = fake + B, *denh = dfake + B, *dmax = denh + B, *genh = dmax + B, *gmax = genh + B,
          *target = gmax + B;
    double* acc = (double*)dev_alloc(3 * sizeof(double));
    unsigned long long* step = (unsigned long long*)dev_alloc(8);
    void* wg = dev_alloc((size_t)wsg);
    void* wd1 = dev_alloc((size_t)wsd);
    void* wd2 = dev_alloc((size_t)wsd);
    float* ht_pesq = (float*)malloc((size_t)B * 4);
    for (int b = 0; b < B; ++b) ht_pesq[b] = pesq;
    cudaMemcpy(pg, hg, (size_t)ng * 4, cudaMemcpyHostToDevice);
    cudaMemcpy(pd, hd, (size_t)nd * 4, cudaMemcpyHostToDevice);
    cudaMemcpy(x, hx, (size_t)n * 8, cudaMemcpyHostToDevice);
    cudaMemcpy(tg, ht, (size_t)n * 8, cudaMemcpyHostToDevice);
    cudaMemcpy(target, ht_pesq, (size_t)B * 4, cudaMemcpyHostToDevice);
    cudaMemset(mg, 0, (size_t)ng * 4); cudaMemset(vg, 0, (size_t)ng * 4);
    cudaMemset(md, 0, (size_t)nd * 4); cudaMemset(vd, 0, (size_t)nd * 4);
    cudaMemset(step, 0, 8);
    /* the discriminator reads est_mag / clean_mag, written (B, 1, T, F), as (B, 1, F, T) views: H = F (stride 1), W = T (stride F) */
    const long long sb = plane, sh = 1, sw = NF;
    for (int k = 0; k < K; ++k) {
        /* ---- generator step */
        CHECK(cmgan_fill(gg, ng, 0.f, 0));
        CHECK(cmgan_counter_add(step, 1, 0));          /* AdamW's step and the dropout seed offset */
        CHECK(cmgan_tscnet_fwd_train(pg, x, 2 * plane, plane, NF, 1, B, T, NF, 1, seed, step, fr, fi, wg, wsg, precision, 0));
        if (cudaMemsetAsync(acc, 0, 3 * sizeof(double), 0) != cudaSuccess) { fprintf(stderr, "cudaMemsetAsync failed\n"); return 1; }
        CHECK(cmgan_spec_loss(fr, fi, tg, tg + plane, plane, 2 * plane, n, w_ri, w_mag, acc, der, dei, est, cln, 0));
        CHECK(cmgan_disc_fwd(pd, cln, sb, sh, sw, est, sb, sh, sw, B, NF, T, 1, dseed, step, fake, wd1, wsd, precision, 0));
        CHECK(cmgan_gen_loss_finalize(acc, (double)n, 1.0, w_ri, w_mag, 0.f, w_gan, fake, B, gloss, dfake, 0));
        CHECK(cmgan_disc_bwd(pd, B, NF, T, 1, dseed, step, dfake, NULL, NULL, dmag, wd1, wsd, precision, 0));
        CHECK(cmgan_mag_bwd_add(fr, fi, dmag, plane, 1, T, B, T, NF, der, dei, 0));       /* dmag is contiguous (B, 1, F, T) */
        CHECK(cmgan_tscnet_bwd(pg, x, 2 * plane, plane, NF, 1, B, T, NF, 1, seed, step, der, dei, plane, NF, 1, gg, NULL, wg, wsg, precision, 0));
        CHECK(adamw_segments(pg, gg, mg, vg, cmgan_tscnet_param_count(), ng, cmgan_tscnet_param_info, "running_", NULL, lr, step));
        /* ---- discriminator step on the same est_mag (computed before the generator update, as the reference detaches it) */
        CHECK(cmgan_fill(gd, nd, 0.f, 0));
        CHECK(cmgan_disc_fwd(pd, cln, sb, sh, sw, est, sb, sh, sw, B, NF, T, 1, dseed + 1, step, denh, wd1, wsd, precision, 0));
        CHECK(cmgan_disc_fwd(pd, cln, sb, sh, sw, cln, sb, sh, sw, B, NF, T, 1, dseed + 2, step, dmax, wd2, wsd, precision, 0));
        CHECK(cmgan_disc_loss(dmax, denh, target, B, dloss, gmax, genh, 0));
        CHECK(cmgan_disc_bwd(pd, B, NF, T, 1, dseed + 1, step, genh, gd, NULL, NULL, wd1, wsd, precision, 0));
        CHECK(cmgan_disc_bwd(pd, B, NF, T, 1, dseed + 2, step, gmax, gd, NULL, NULL, wd2, wsd, precision, 0));
        CHECK(adamw_segments(pd, gd, md, vd, cmgan_disc_param_count(), nd, cmgan_disc_param_info, "weight_u", "weight_v", 2.f * lr, step));
        float hl[2] = {0.f, 0.f};
        if (cudaMemcpy(&hl[0], gloss, 4, cudaMemcpyDeviceToHost) != cudaSuccess || cudaMemcpy(&hl[1], dloss, 4, cudaMemcpyDeviceToHost) != cudaSuccess) {
            fprintf(stderr, "device error\n");
            return 1;
        }
        printf("step %d generator loss %.9g discriminator loss %.9g\n", k + 1, hl[0], hl[1]);
    }
    if (write_floats(argv[10], pg, ng) || write_floats(argv[11], pd, nd)) return 1;
    printf("trained %d steps (B=%d T=%d precision %d, workspaces %lld + 2 x %lld bytes)\n", K, B, T, precision, wsg, wsd);
    cudaFree(pg); cudaFree(gg); cudaFree(mg); cudaFree(vg); cudaFree(pd); cudaFree(gd); cudaFree(md); cudaFree(vd); cudaFree(x); cudaFree(tg);
    cudaFree(fr); cudaFree(fi); cudaFree(der); cudaFree(dei); cudaFree(est); cudaFree(cln); cudaFree(dmag); cudaFree(sc); cudaFree(acc);
    cudaFree(step); cudaFree(wg); cudaFree(wd1); cudaFree(wd2);
    free(hg); free(hd); free(hx); free(ht); free(ht_pesq);
    return 0;
}
#endif

int main(int argc, char** argv) {
    for (int precision = 0; precision <= 1; ++precision)
        if (query(4, 321, precision) || query(16, 321, precision)) return 1;
    if (cmgan_disc_workspace_bytes(4, NF, 15, 1) >= 0) { fprintf(stderr, "W = 15 must be rejected\n"); return 1; }
    printf("rejected W=15: %s\n", cmgan_last_error());
    if (cmgan_disc_bwd(NULL, 1, NF, 101, 1, 0, NULL, NULL, NULL, NULL, NULL, NULL, 0, 1, NULL) == 0) {
        fprintf(stderr, "a call with nothing to compute must be rejected\n");
        return 1;
    }
    printf("rejected call: %s\n", cmgan_last_error());
#ifdef WITH_CUDA
    if (argc > 11) return train(argv, argc);
#else
    (void)argc;
    (void)argv;
#endif
    return 0;
}
