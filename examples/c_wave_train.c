/* MetricGAN training from a packed waveform corpus by a non-Python host (plain C99): K steps of the reference train_step (train.py:176-205),
 * time-domain loss included, all on one stream of libcmgan_b200.so.  Each step:
 *   batch:              two cmgan_cut_batch (clean, noisy) with the step's (utterance, start) pairs: the data loader's cut (dataloader.py:32-49);
 *   generator step:     cmgan_gen_wave_fwd (RMS scale, both STFTs, the train-mode TSCNet, the inverse STFT, spectral and time-domain losses), the
 *                       train-mode discriminator on (clean_mag, est_mag) (cmgan_disc_fwd), cmgan_gen_loss_finalize with the weights (0.1, 0.9,
 *                       0.2, 0.05), the discriminator's input gradient with frozen weights (cmgan_disc_bwd, grads = NULL), cmgan_gen_wave_bwd,
 *                       AdamW over the generator block (skipping the BatchNorm running statistics);
 *   discriminator step: as examples/c_gan_train.c, on the same est_mag: (clean, est) and (clean, clean) forwards, cmgan_disc_loss against the
 *                       PESQ target, both backwards, AdamW at 2 lr (skipping weight_u / weight_v).
 * Seeds follow FusedTrainer(seed = s) on one GPU: gseed = s * 65537 * 7919 for TSCNet, gseed * 31 + 5 for the discriminator inside the generator
 * step, gseed * 131 + 17 + {1, 2} for the discriminator step; one device counter offsets every dropout seed and counts AdamW's steps.
 * What stays with the host: the PESQ scores (here one constant target, given on the command line) and any all-reduce across GPUs.
 *   Build:  gcc -std=c99 -Iinclude examples/c_wave_train.c -o c_wave_train -Lcmgan_b200 -lcmgan_b200 -Wl,-rpath,$PWD/cmgan_b200
 *           (add -DWITH_CUDA -I/usr/local/cuda/include -L/usr/local/cuda/lib64 -lcudart to train).
 *   Run:    c_wave_train [gen.f32 disc.f32 clean.f32 noisy.f32 lengths.i32 schedule.i32 B cut_len steps precision pesq gen_out.f32 disc_out.f32
 *                         [lr [seed]]]
 * gen.f32 / disc.f32 are raw little-endian float32 dumps of the two parameter blocks (cmgan_b200.module_abi.pack_params / pack_disc_params);
 * clean.f32 / noisy.f32 hold the utterances back to back (float32 samples, the same lengths in both); lengths.i32 holds one int32 length per
 * utterance; schedule.i32 holds steps x B int32 pairs (utterance index, start sample).  Both trained blocks are written out.  Without WITH_CUDA
 * only the host-side workspace queries and argument checks run (no GPU needed). */
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "cmgan_b200.h"

#ifdef WITH_CUDA
#include <cuda_runtime.h>
#endif

#define NF 201

static int query(int B, int L, int precision) {
    const int T = L / 100 + 1;
    const long long wg = cmgan_gen_wave_workspace_bytes(B, L, precision), wd = cmgan_disc_workspace_bytes(B, NF, T, precision);
    if (wg < 0 || wd < 0) {
        fprintf(stderr, "%s\n", cmgan_last_error());
        return 1;
    }
    printf("workspaces B=%d L=%d %s: generator %lld bytes, discriminator %lld bytes\n", B, L, precision ? "tf32" : "fp32", wg, wd);
    return 0;
}

#ifdef WITH_CUDA
static void* read_file(const char* path, size_t elem, long long* count) {
    FILE* f = fopen(path, "rb");
    if (!f || fseek(f, 0, SEEK_END) != 0) { fprintf(stderr, "cannot open %s\n", path); exit(1); }
    const long size = ftell(f);
    rewind(f);
    void* h = malloc(size > 0 ? (size_t)size : 1);
    if (!h || size < 0 || fread(h, 1, (size_t)size, f) != (size_t)size) { fprintf(stderr, "cannot read %s\n", path); exit(1); }
    fclose(f);
    *count = (long long)((size_t)size / elem);
    return h;
}

static float* read_floats(const char* path, long long n) {
    long long have = 0;
    float* h = (float*)read_file(path, 4, &have);
    if (have != n) { fprintf(stderr, "%s holds %lld floats, expected %lld\n", path, have, n); exit(1); }
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

static void* dev_copy(const void* h, size_t bytes) {
    void* d = dev_alloc(bytes);
    if (cudaMemcpy(d, h, bytes, cudaMemcpyHostToDevice) != cudaSuccess) { fprintf(stderr, "cudaMemcpy failed\n"); exit(1); }
    return d;
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
    const int B = atoi(argv[7]), cut = atoi(argv[8]), K = atoi(argv[9]), precision = atoi(argv[10]);
    const float pesq = (float)atof(argv[11]);
    const float lr = argc > 14 ? (float)atof(argv[14]) : 5e-4f;
    const unsigned long long s = argc > 15 ? strtoull(argv[15], NULL, 10) : 0;
    const float w_ri = 0.1f, w_mag = 0.9f, w_t = 0.2f, w_gan = 0.05f;       /* train.py:124-151 */
    const unsigned long long gseed = s * 65537ull * 7919ull, dseed = gseed * 31ull + 5ull, dstep = gseed * 131ull + 17ull;
    if (B <= 0 || cut <= 200 || K <= 0) { fprintf(stderr, "need B > 0, cut_len > 200, steps > 0\n"); return 1; }
    const int T = cut / 100 + 1, Lo = cut / 100 * 100;
    const long long ng = cmgan_tscnet_param_floats(), nd = cmgan_disc_param_floats(), plane = (long long)T * NF, n = (long long)B * plane;
    const long long wsg = cmgan_gen_wave_workspace_bytes(B, cut, precision), wsd = cmgan_disc_workspace_bytes(B, NF, T, precision);
    if (wsg < 0 || wsd < 0) { fprintf(stderr, "%s\n", cmgan_last_error()); return 1; }
    float* hg = read_floats(argv[1], ng);
    float* hd = read_floats(argv[2], nd);
    long long nutt = 0, nsched = 0, total = 0;
    int* hlen = (int*)read_file(argv[5], 4, &nutt);
    int* hsched = (int*)read_file(argv[6], 4, &nsched);
    if (nsched != 2LL * K * B) { fprintf(stderr, "the schedule holds %lld ints, expected %lld\n", nsched, 2LL * K * B); return 1; }
    long long* hoff = (long long*)malloc((size_t)nutt * 8);
    for (long long u = 0; u < nutt; ++u) { hoff[u] = total; total += hlen[u]; }
    float* hclean = read_floats(argv[3], total);
    float* hnoisy = read_floats(argv[4], total);
    /* the per-step index arrays of cmgan_cut_batch, for all K steps: offsets (int64), lengths and starts (int32) */
    long long* hso = (long long*)malloc((size_t)K * B * 8);
    int *hsl = (int*)malloc((size_t)K * B * 4), *hss = (int*)malloc((size_t)K * B * 4);
    for (long long i = 0; i < (long long)K * B; ++i) {
        const int u = hsched[2 * i];
        if (u < 0 || u >= nutt) { fprintf(stderr, "schedule entry %lld names utterance %d of %lld\n", i, u, nutt); return 1; }
        hso[i] = hoff[u]; hsl[i] = hlen[u]; hss[i] = hsched[2 * i + 1];
    }
    float* corpus_c = (float*)dev_copy(hclean, (size_t)total * 4);
    float* corpus_n = (float*)dev_copy(hnoisy, (size_t)total * 4);
    long long* so = (long long*)dev_copy(hso, (size_t)K * B * 8);
    int* sl = (int*)dev_copy(hsl, (size_t)K * B * 4);
    int* ss = (int*)dev_copy(hss, (size_t)K * B * 4);
    float* pg = (float*)dev_copy(hg, (size_t)ng * 4);
    float* pd = (float*)dev_copy(hd, (size_t)nd * 4);
    float *gg = (float*)dev_alloc((size_t)ng * 4), *mg = (float*)dev_alloc((size_t)ng * 4), *vg = (float*)dev_alloc((size_t)ng * 4);
    float *gd = (float*)dev_alloc((size_t)nd * 4), *md = (float*)dev_alloc((size_t)nd * 4), *vd = (float*)dev_alloc((size_t)nd * 4);
    float *clean = (float*)dev_alloc((size_t)B * cut * 4), *noisy = (float*)dev_alloc((size_t)B * cut * 4), *est_audio = (float*)dev_alloc((size_t)B * Lo * 4);
    float *est = (float*)dev_alloc((size_t)n * 4), *cln = (float*)dev_alloc((size_t)n * 4), *dmag = (float*)dev_alloc((size_t)n * 4);
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
    cudaMemcpy(target, ht_pesq, (size_t)B * 4, cudaMemcpyHostToDevice);
    cudaMemset(mg, 0, (size_t)ng * 4); cudaMemset(vg, 0, (size_t)ng * 4);
    cudaMemset(md, 0, (size_t)nd * 4); cudaMemset(vd, 0, (size_t)nd * 4);
    cudaMemset(step, 0, 8);
    /* the discriminator reads est_mag / clean_mag, written (B, 1, T, F), as (B, 1, F, T) views: H = F (stride 1), W = T (stride F) */
    const long long sb = plane, sh = 1, sw = NF;
    for (int k = 0; k < K; ++k) {
        const long long i0 = (long long)k * B;
        CHECK(cmgan_cut_batch(corpus_c, so + i0, sl + i0, ss + i0, B, cut, clean, cut, 0));
        CHECK(cmgan_cut_batch(corpus_n, so + i0, sl + i0, ss + i0, B, cut, noisy, cut, 0));
        /* ---- generator step */
        CHECK(cmgan_counter_add(step, 1, 0));          /* AdamW's step and the dropout seed offset */
        CHECK(cmgan_fill(gg, ng, 0.f, 0));
        CHECK(cmgan_gen_wave_fwd(pg, clean, cut, noisy, cut, B, cut, 1, gseed, step, w_ri, w_mag, w_t, est_audio, Lo, est, cln, acc, wg, wsg, precision, 0));
        CHECK(cmgan_disc_fwd(pd, cln, sb, sh, sw, est, sb, sh, sw, B, NF, T, 1, dseed, step, fake, wd1, wsd, precision, 0));
        CHECK(cmgan_gen_loss_finalize(acc, (double)n, (double)B * Lo, w_ri, w_mag, w_t, w_gan, fake, B, gloss, dfake, 0));
        CHECK(cmgan_disc_bwd(pd, B, NF, T, 1, dseed, step, dfake, NULL, NULL, dmag, wd1, wsd, precision, 0));
        /* dmag is contiguous (B, 1, F, T): stride T * F along B, 1 along T, T along F */
        CHECK(cmgan_gen_wave_bwd(pg, B, cut, 1, gseed, step, dmag, plane, 1, T, gg, wg, wsg, precision, 0));
        CHECK(adamw_segments(pg, gg, mg, vg, cmgan_tscnet_param_count(), ng, cmgan_tscnet_param_info, "running_", NULL, lr, step));
        /* ---- discriminator step on the same est_mag (computed before the generator update, as the reference detaches it) */
        CHECK(cmgan_fill(gd, nd, 0.f, 0));
        CHECK(cmgan_disc_fwd(pd, cln, sb, sh, sw, est, sb, sh, sw, B, NF, T, 1, dstep + 1, step, denh, wd1, wsd, precision, 0));
        CHECK(cmgan_disc_fwd(pd, cln, sb, sh, sw, cln, sb, sh, sw, B, NF, T, 1, dstep + 2, step, dmax, wd2, wsd, precision, 0));
        CHECK(cmgan_disc_loss(dmax, denh, target, B, dloss, gmax, genh, 0));
        CHECK(cmgan_disc_bwd(pd, B, NF, T, 1, dstep + 1, step, genh, gd, NULL, NULL, wd1, wsd, precision, 0));
        CHECK(cmgan_disc_bwd(pd, B, NF, T, 1, dstep + 2, step, gmax, gd, NULL, NULL, wd2, wsd, precision, 0));
        CHECK(adamw_segments(pd, gd, md, vd, cmgan_disc_param_count(), nd, cmgan_disc_param_info, "weight_u", "weight_v", 2.f * lr, step));
        float hl[2] = {0.f, 0.f};
        if (cudaMemcpy(&hl[0], gloss, 4, cudaMemcpyDeviceToHost) != cudaSuccess || cudaMemcpy(&hl[1], dloss, 4, cudaMemcpyDeviceToHost) != cudaSuccess) {
            fprintf(stderr, "device error\n");
            return 1;
        }
        printf("step %d generator loss %.9g discriminator loss %.9g\n", k + 1, hl[0], hl[1]);
    }
    if (write_floats(argv[12], pg, ng) || write_floats(argv[13], pd, nd)) return 1;
    printf("trained %d steps (B=%d cut_len=%d precision %d, workspaces %lld + 2 x %lld bytes)\n", K, B, cut, precision, wsg, wsd);
    cudaFree(corpus_c); cudaFree(corpus_n); cudaFree(so); cudaFree(sl); cudaFree(ss);
    cudaFree(pg); cudaFree(gg); cudaFree(mg); cudaFree(vg); cudaFree(pd); cudaFree(gd); cudaFree(md); cudaFree(vd);
    cudaFree(clean); cudaFree(noisy); cudaFree(est_audio); cudaFree(est); cudaFree(cln); cudaFree(dmag); cudaFree(sc); cudaFree(acc);
    cudaFree(step); cudaFree(wg); cudaFree(wd1); cudaFree(wd2);
    free(hg); free(hd); free(hlen); free(hsched); free(hoff); free(hclean); free(hnoisy); free(hso); free(hsl); free(hss); free(ht_pesq);
    return 0;
}
#endif

int main(int argc, char** argv) {
    for (int precision = 0; precision <= 1; ++precision)
        if (query(4, 32000, precision) || query(16, 32000, precision)) return 1;
    if (cmgan_gen_wave_workspace_bytes(4, 200, 1) >= 0) { fprintf(stderr, "L = 200 must be rejected\n"); return 1; }
    printf("rejected L=200: %s\n", cmgan_last_error());
    if (cmgan_gen_wave_bwd(NULL, 2, 16000, 1, 0, NULL, NULL, 0, 0, 0, NULL, NULL, 0, 1, NULL) == 0) {
        fprintf(stderr, "a backward without a gradient block must be rejected\n");
        return 1;
    }
    printf("rejected call: %s\n", cmgan_last_error());
#ifdef WITH_CUDA
    if (argc > 13) return train(argv, argc);
#else
    (void)argc;
    (void)argv;
#endif
    return 0;
}
