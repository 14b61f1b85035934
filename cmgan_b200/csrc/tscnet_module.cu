// Module-level entry point: TSCNet.forward in inference mode (eval: BatchNorm running statistics, no dropout) as ONE C call over the
// kernels of this library -- the boundary SURVEY 8(b) asks for a non-Python host: raw device pointers, explicit strides, a caller-owned
// workspace sized by a query, int status + cmgan_last_error(), everything enqueued on the caller's stream, no allocation, no sync.
// Reference: generator.py:160-196 (TSCNet), :50-69 (DenseEncoder), :6-47 (DilatedDenseNet), :72-99 (TSCB), :122-156 (decoders),
// conformer.py:182-222 (ConformerBlock).  The launch sequence is the one cmgan_b200/network.py + conformer_block.py issue from Python
// (same kernels, same order), so the results are bit-identical to the nn.Module path.
//
// Parameters: one flat fp32 block holding every floating-point tensor of the reference's state_dict, in state_dict order, each tensor
// starting at a multiple of 4 floats (cmgan_tscnet_param_info enumerates key / offset / element count; the int64 num_batches_tracked
// buffers are not part of it).
#include <algorithm>
#include <cstring>
#include <string>
#include <unordered_map>
#include <vector>

#include "common.cuh"
#include "frontend.cuh"
#include "module_walk.cuh"
#include "resample.cuh"
#include "../../include/cmgan_b200.h"

namespace {

using namespace cmgan_walk;

constexpr int C = 64, CAT = 320, NFEAT = 201;

struct Table : ParamTable {
    void norm_prelu(const std::string& p, const char* norm, const char* prelu) {
        add(p + norm + ".weight", C); add(p + norm + ".bias", C); add(p + prelu + ".weight", C);
    }
    void dense_block(const std::string& p) {            // generator.py:6-37
        for (int i = 1; i <= 4; ++i) {
            const std::string s = std::to_string(i);
            add(p + "conv" + s + ".weight", (long long)C * C * i * 6); add(p + "conv" + s + ".bias", C);
            add(p + "norm" + s + ".weight", C); add(p + "norm" + s + ".bias", C); add(p + "prelu" + s + ".weight", C);
        }
    }
    void feed_forward(const std::string& p) {           // conformer.py:136-148 wrapped by Scale(PreNorm(...)) :54-72
        add(p + "fn.fn.net.0.weight", 4 * C * C); add(p + "fn.fn.net.0.bias", 4 * C);
        add(p + "fn.fn.net.3.weight", 4 * C * C); add(p + "fn.fn.net.3.bias", C);
        add(p + "fn.norm.weight", C); add(p + "fn.norm.bias", C);
    }
    void conformer(const std::string& p) {              // conformer.py:182-214
        feed_forward(p + "ff1.");
        add(p + "attn.fn.to_q.weight", C * C); add(p + "attn.fn.to_kv.weight", 2 * C * C);
        add(p + "attn.fn.to_out.weight", C * C); add(p + "attn.fn.to_out.bias", C);
        add(p + "attn.fn.rel_pos_emb.weight", 1025 * 16);
        add(p + "attn.norm.weight", C); add(p + "attn.norm.bias", C);
        add(p + "conv.net.0.weight", C); add(p + "conv.net.0.bias", C);
        add(p + "conv.net.2.weight", 4 * C * C); add(p + "conv.net.2.bias", 4 * C);
        add(p + "conv.net.4.conv.weight", 2 * C * 31); add(p + "conv.net.4.conv.bias", 2 * C);
        add(p + "conv.net.5.weight", 2 * C); add(p + "conv.net.5.bias", 2 * C);
        add(p + "conv.net.5.running_mean", 2 * C); add(p + "conv.net.5.running_var", 2 * C);
        add(p + "conv.net.7.weight", 2 * C * C); add(p + "conv.net.7.bias", C);
        feed_forward(p + "ff2.");
        add(p + "post_norm.weight", C); add(p + "post_norm.bias", C);
    }
    Table() {
        add("dense_encoder.conv_1.0.weight", C * 3); add("dense_encoder.conv_1.0.bias", C);
        norm_prelu("dense_encoder.conv_1.", "1", "2");
        dense_block("dense_encoder.dilated_dense.");
        add("dense_encoder.conv_2.0.weight", C * C * 3); add("dense_encoder.conv_2.0.bias", C);
        norm_prelu("dense_encoder.conv_2.", "1", "2");
        for (int i = 1; i <= 4; ++i) {
            conformer("TSCB_" + std::to_string(i) + ".time_conformer.");
            conformer("TSCB_" + std::to_string(i) + ".freq_conformer.");
        }
        dense_block("mask_decoder.dense_block.");
        add("mask_decoder.sub_pixel.conv.weight", 2 * C * C * 3); add("mask_decoder.sub_pixel.conv.bias", 2 * C);
        add("mask_decoder.conv_1.weight", C * 2); add("mask_decoder.conv_1.bias", 1);
        add("mask_decoder.norm.weight", 1); add("mask_decoder.norm.bias", 1);
        add("mask_decoder.prelu.weight", 1);
        add("mask_decoder.final_conv.weight", 1); add("mask_decoder.final_conv.bias", 1);
        add("mask_decoder.prelu_out.weight", NFEAT);
        dense_block("complex_decoder.dense_block.");
        add("complex_decoder.sub_pixel.conv.weight", 2 * C * C * 3); add("complex_decoder.sub_pixel.conv.bias", 2 * C);
        add("complex_decoder.prelu.weight", C);
        add("complex_decoder.norm.weight", C); add("complex_decoder.norm.bias", C);
        add("complex_decoder.conv.weight", 2 * C * 2); add("complex_decoder.conv.bias", 2);
    }
};

const Table& table() {
    static const Table t;
    return t;
}

// ---- what the backward reads, kept by a training forward (cmgan_tscnet_fwd_train) in the saved region of the workspace
struct FfSaved { float *xn = nullptr, *st = nullptr, *h = nullptr, *a = nullptr; };      // fp32 feed-forward only (tf32 recomputes its hidden layer)
struct ConfSaved {
    const float* x;             // block input (the previous block's output)
    float *x1, *xn2, *st2, *qkv, *ctx, *lse, *x2, *xn3, *st3, *g, *d, *dsw, *x3, *x4, *st5;
    Tabs bn;
    FfSaved f1, f2;
};
struct DenseSaved { float* raw[4]; Tabs tab[4]; };
struct Saved {
    float *catE, *raw0, *e2;
    Tabs tab0, tab2;
    DenseSaved enc;
    ConfSaved conf[8];
    float *cat[2], *sp[2];
    DenseSaved dec[2];
    float* m1;
    Tabs tabM, tabC;
};

// counter-based dropout parameters (ops.drop_params) and per-site seeds (conformer_block._site_seed)
constexpr double P_DROP = 0.2;          // generator.py:81-82,88-89: attention and feed-forward dropout
unsigned drop_thr(bool on) { return on ? (unsigned)std::min(P_DROP * 4294967296.0, 4294967295.0) : 0u; }
float drop_inv(bool on) { return on ? (float)(1.0 / (1.0 - P_DROP)) : 1.f; }
unsigned long long site_seed(unsigned long long seed, int block_id, int site) { return seed * 1000003ull + (unsigned long long)(block_id * 16 + site + 1); }

// ---- one forward pass = a walk over the launch list; `dry` only sizes the workspace
struct Run : Walk {
    Saved* sv = nullptr;        // forward: record where the saved activations are (set together with `saving`)
    Run() { tab = &table(); tag = "cmgan_tscnet"; who = "cmgan_tscnet_fwd"; }
};

// InstanceNorm2d(affine) + PReLU of a raw (M, 64) tensor, written into dst (generator.py:35-37)
Tabs norm_prelu_to(Run& r, const float* raw, int G, long long rows, long long rows_per_t, const float* gamma, const float* beta, const float* slope,
                   float* dst, long long ldd, double*& sums) {
    Tabs t = make_tabs(r, G, C);
    inst_norm_site(r, raw, C, G, rows, rows_per_t, C, gamma, beta, t, sums);
    if (r.live()) r.ok(cmgan_norm_apply(raw, C, G, rows, C, 1 | (r.precision == 1 ? 16 : 0), t.scale, t.shift, C, slope, dst, ldd, r.st));
    return t;
}

const int W3_DY[3] = {0, 0, 0}, W3_DX[3] = {-1, 0, 1}, W3T_DX[3] = {1, 0, -1};     // (1, 3) convolutions and their data gradients

// DilatedDenseNet (generator.py:39-47) on the concat buffer cat = [out4 | out3 | out2 | out1 | x]; `ds` records the raw outputs and tables
void dense_block(Run& r, float* cat, const std::string& p, int B, int T, int Fw, double*& sums, DenseSaved* ds = nullptr) {
    const long long M = (long long)B * T * Fw, rows = (long long)T * Fw;
    for (int i = 1; i <= 4; ++i) {
        const int dil = 1 << (i - 1), c0 = (5 - i) * C, Cin = C * i, co = (4 - i) * C;
        const std::string s = std::to_string(i);
        float* raw = r.keep((size_t)M * C);
        const int dy[6] = {-dil, -dil, -dil, 0, 0, 0}, dx[6] = {-1, 0, 1, -1, 0, 1};         // tap = kh * 3 + kw, causal in time (generator.py:12-21)
        Gemm(off(cat, c0), CAT, r.w(p + "conv" + s + ".weight"), 1, 6, (long long)Cin * 6, r.w(p + "conv" + s + ".bias"), raw, C, M, C, Cin)
            .taps(6, dy, dx).conv(T, Fw, T, Fw).run(r);
        const Tabs t = norm_prelu_to(r, raw, B, rows, Fw, r.w(p + "norm" + s + ".weight"), r.w(p + "norm" + s + ".bias"), r.w(p + "prelu" + s + ".weight"),
                                     off(cat, co), CAT, sums);
        if (ds) { ds->raw[i - 1] = raw; ds->tab[i - 1] = t; }
    }
}

// 0.5 * FF(LN(x)) + x  (conformer.py:54-72,136-148,211-212); dropout (training) with the site seeds s1 (hidden layer) and s2 (output)
float* feed_forward(Run& r, const float* xin, long long M, const std::string& p, unsigned long long s1 = 0, unsigned long long s2 = 0, FfSaved* fs = nullptr) {
    const unsigned thr = drop_thr(r.training);
    const float inv = drop_inv(r.training);
    float* out = r.keep((size_t)M * C);
    if (r.precision == 1) {          // fused kernel: the hidden activation stays on the SM (ffn_fused.cu)
        float* w1p = r.alloc((size_t)4 * C * C);
        float* w2p = r.alloc((size_t)4 * C * C);
        if (r.live()) {
            r.ok(cmgan_pack_weight(r.w(p + "fn.fn.net.0.weight"), w1p, 0, 1, C, C, 1, 4 * C, r.st));
            r.ok(cmgan_pack_weight(r.w(p + "fn.fn.net.3.weight"), w2p, 0, 1, 4 * C, 4 * C, 1, C, r.st));
            r.ok(cmgan_ffn_fwd(xin, C, M, r.w(p + "fn.norm.weight"), r.w(p + "fn.norm.bias"), w1p, r.w(p + "fn.fn.net.0.bias"), w2p,
                               r.w(p + "fn.fn.net.3.bias"), 0.5f, s1, s2, thr, inv, r.seed_dev, out, C, r.st));
        }
        return out;
    }
    float* xn = r.keep((size_t)M * C);
    float* stt = r.keep((size_t)M * 2);
    float* h = fs ? r.keep((size_t)M * 4 * C) : nullptr;           // pre-activation: only the backward reads it
    float* a = r.keep((size_t)M * 4 * C);
    if (r.live()) r.ok(cmgan_ln_apply(xin, C, M, r.w(p + "fn.norm.weight"), r.w(p + "fn.norm.bias"), nullptr, 0, xn, C, stt, r.precision == 1 ? 1 : 0, r.st));
    Gemm g1(xn, C, r.w(p + "fn.fn.net.0.weight"), 0, 1, C, r.w(p + "fn.fn.net.0.bias"), h, 4 * C, M, 4 * C, C);
    g1.a.epi = CMGAN_EPI_SWISH_DUAL; g1.a.C2 = a; g1.a.ldc2 = 4 * C;
    g1.drop(s1, thr, inv).run(r);
    Gemm g2(a, 4 * C, r.w(p + "fn.fn.net.3.weight"), 0, 1, 4 * C, r.w(p + "fn.fn.net.3.bias"), out, C, M, C, 4 * C);
    g2.residual(xin, C).drop(s2, thr, inv).a.alpha = 0.5f;
    g2.run(r);
    if (fs) { fs->xn = xn; fs->st = stt; fs->h = h; fs->a = a; }
    return out;
}

// ConformerBlock + the outer TSCB residual (conformer.py:216-222, generator.py:95,97): returns LN(x4) + x in `y`.
// Training: dropout at the five sites (seeds from block_id), BatchNorm batch statistics from the depthwise kernel's epilogue sums.
void conformer(Run& r, const float* x, float* y, const std::string& p, int B, int T, int F2, int axis, int block_id = 0, double** sums = nullptr,
               ConfSaved* cs = nullptr) {
    const long long M = (long long)B * T * F2;
    const size_t mark = r.top;
    const int rnd = r.precision == 1 ? 1 : 0;
    unsigned long long sd[5] = {0, 0, 0, 0, 0};
    if (r.training)
        for (int i = 0; i < 5; ++i) sd[i] = site_seed(r.seed, block_id, i);
    float* x1 = feed_forward(r, x, M, p + "ff1.", sd[0], sd[1], cs ? &cs->f1 : nullptr);
    // ---- attention (conformer.py:90-133)
    float* xn2 = r.keep((size_t)M * C);
    float* st2 = r.keep((size_t)M * 2);
    if (r.live()) r.ok(cmgan_ln_apply(x1, C, M, r.w(p + "attn.norm.weight"), r.w(p + "attn.norm.bias"), nullptr, 0, xn2, C, st2, rnd, r.st));
    float* qkv = r.keep((size_t)M * 3 * C);
    // to_q and to_kv are adjacent in the parameter block: one (192, 64) projection
    Gemm(xn2, C, r.w(p + "attn.fn.to_q.weight"), 0, 1, C, nullptr, qkv, 3 * C, M, 3 * C, C).run(r);
    float* ctx = r.keep((size_t)M * C);
    float* lse = r.keep((size_t)M * 4);
    if (r.live()) {
        const float* E = r.w(p + "attn.fn.rel_pos_emb.weight");
        if (r.frames)
            r.ok(r.precision == 1 ? cmgan_attention_fwd_tf32_ragged(qkv, E, B, T, F2, axis, r.frames, ctx, lse, r.st)
                                  : cmgan_attention_fwd_ragged(qkv, E, B, T, F2, axis, r.frames, ctx, lse, r.st));
        else
            r.ok(r.precision == 1 ? cmgan_attention_fwd_tf32(qkv, E, B, T, F2, axis, ctx, lse, r.st) : cmgan_attention_fwd(qkv, E, B, T, F2, axis, ctx, lse, r.st));
    }
    float* x2 = r.keep((size_t)M * C);
    Gemm(ctx, C, r.w(p + "attn.fn.to_out.weight"), 0, 1, C, r.w(p + "attn.fn.to_out.bias"), x2, C, M, C, C).residual(x1, C)
        .drop(sd[2], drop_thr(r.training), drop_inv(r.training)).run(r);
    // ---- convolution module (conformer.py:160-173)
    float* xn3 = r.keep((size_t)M * C);
    float* st3 = r.keep((size_t)M * 2);
    if (r.live()) r.ok(cmgan_ln_apply(x2, C, M, r.w(p + "conv.net.0.weight"), r.w(p + "conv.net.0.bias"), nullptr, 0, xn3, C, st3, rnd, r.st));
    float* g = r.keep((size_t)M * 4 * C);
    Gemm(xn3, C, r.w(p + "conv.net.2.weight"), 0, 1, C, r.w(p + "conv.net.2.bias"), g, 4 * C, M, 4 * C, C).run(r);
    float* d = r.keep((size_t)M * 2 * C);
    Tabs bn = make_tabs(r, 1, 2 * C);
    float* dsw = r.keep((size_t)M * 2 * C);
    double* bs = nullptr;        // training: per-channel sum and sum of squares of d, from the depthwise kernel's epilogue
    if (r.training) { bs = *sums; *sums += 2 * C * 2; }
    if (r.live()) {
        float* rmean = const_cast<float*>(r.w(p + "conv.net.5.running_mean"));
        float* rvar = const_cast<float*>(r.w(p + "conv.net.5.running_var"));
        if (r.frames)
            r.ok(cmgan_glu_dwconv_fwd_ragged(g, r.w(p + "conv.net.4.conv.weight"), r.w(p + "conv.net.4.conv.bias"), B, T, F2, axis, r.frames, d, r.st));
        else
            r.ok(cmgan_glu_dwconv_fwd(g, r.w(p + "conv.net.4.conv.weight"), r.w(p + "conv.net.4.conv.bias"), B, T, F2, axis, d, bs, r.st));
        if (r.training)     // batch statistics; the running statistics are updated in place (momentum 0.1, unbiased variance)
            r.ok(cmgan_norm_finalize(bs, M, 1, 2 * C, 0, r.w(p + "conv.net.5.weight"), r.w(p + "conv.net.5.bias"), rmean, rvar, 0.1f,
                                     bn.scale, bn.shift, bn.mean, bn.rstd, 2 * C, r.st));
        else                // eval: BatchNorm1d folds to scale / shift from the running statistics (mode 1; they are only read)
            r.ok(cmgan_norm_finalize(nullptr, M, 1, 2 * C, 1, r.w(p + "conv.net.5.weight"), r.w(p + "conv.net.5.bias"), rmean, rvar, 0.1f,
                                     bn.scale, bn.shift, bn.mean, bn.rstd, 2 * C, r.st));
        r.ok(cmgan_norm_apply(d, 2 * C, 1, M, 2 * C, 2 | (16 * rnd), bn.scale, bn.shift, 2 * C, nullptr, dsw, 2 * C, r.st));
    }
    float* x3 = r.keep((size_t)M * C);
    Gemm(dsw, 2 * C, r.w(p + "conv.net.7.weight"), 0, 1, 2 * C, r.w(p + "conv.net.7.bias"), x3, C, M, C, 2 * C).residual(x2, C).run(r);
    // ---- second feed-forward, post norm, outer residual
    float* x4 = feed_forward(r, x3, M, p + "ff2.", sd[3], sd[4], cs ? &cs->f2 : nullptr);
    float* st5 = r.keep((size_t)M * 2);
    if (r.live()) r.ok(cmgan_ln_apply(x4, C, M, r.w(p + "post_norm.weight"), r.w(p + "post_norm.bias"), x, C, y, C, st5, 0, r.st));
    if (cs) {
        cs->x = x; cs->x1 = x1; cs->xn2 = xn2; cs->st2 = st2; cs->qkv = qkv; cs->ctx = ctx; cs->lse = lse; cs->x2 = x2; cs->xn3 = xn3; cs->st3 = st3;
        cs->g = g; cs->d = d; cs->dsw = dsw; cs->bn = bn; cs->x3 = x3; cs->x4 = x4; cs->st5 = st5;
    }
    r.top = mark;            // everything but `y` (owned by the caller) and the saved activations is released
}

const char* conformer_name(int k) {         // k = (i - 1) * 2 + axis: the block_id of conformer_block._site_seed
    static const char* n[8] = {"TSCB_1.time_conformer.", "TSCB_1.freq_conformer.", "TSCB_2.time_conformer.", "TSCB_2.freq_conformer.",
                               "TSCB_3.time_conformer.", "TSCB_3.freq_conformer.", "TSCB_4.time_conformer.", "TSCB_4.freq_conformer."};
    return n[k];
}
const char* const DEC_NAMES[2] = {"mask_decoder.", "complex_decoder."};

// statistics scratch of one pass (network._sums_size): every InstanceNorm site, plus the BatchNorm sums of the conformers in training
size_t sums_size(int B, bool training) { return (size_t)(16 * C + 2) * B * 2 + 64 + (training ? 8 * 2 * C * 2 : 0); }

void forward(Run& r, const float* x, long long sxb, long long sxc, long long sxt, long long sxf, int B, int T, int F, float* fr, float* fi) {
    const int F2 = (F - 1) / 2 + 1;
    const long long M = (long long)B * T * F, M2 = (long long)B * T * F2;
    Saved* sv = r.sv;
    const size_t n_sums = sums_size(B, r.training);
    double* sums0 = r.alloc<double>(n_sums);
    double* sums = sums0;
    if (r.live()) {
        cudaError_t e = cudaMemsetAsync(sums0, 0, n_sums * sizeof(double), r.st);
        if (e != cudaSuccess) { cmgan_set_error("cmgan_tscnet_fwd: cudaMemsetAsync: %s", cudaGetErrorString(e)); r.rc = -1; }
    }
    // TSCB activations ping-pong between these two; when saving, every block's input is kept instead
    float* hA = sv ? r.keep((size_t)M2 * C) : r.alloc((size_t)M2 * C);
    float* hB = sv ? nullptr : r.alloc((size_t)M2 * C);
    // ---- dense encoder (generator.py:50-69)
    {
        const size_t mark = r.top;
        const std::string pe = "dense_encoder.";
        float* catE = r.keep((size_t)M * CAT);
        float* raw0 = r.keep((size_t)M * C);
        if (r.live()) r.ok(cmgan_head_conv(x, sxb, sxc, sxt, sxf, B, T, F, r.w(pe + "conv_1.0.weight"), r.w(pe + "conv_1.0.bias"), raw0, C, r.st));
        const Tabs t0 = norm_prelu_to(r, raw0, B, (long long)T * F, F, r.w(pe + "conv_1.1.weight"), r.w(pe + "conv_1.1.bias"),
                                      r.w(pe + "conv_1.2.weight"), off(catE, 4 * C), CAT, sums);
        dense_block(r, catE, pe + "dilated_dense.", B, T, F, sums, sv ? &sv->enc : nullptr);
        float* e2 = r.keep((size_t)M2 * C);
        Gemm(catE, CAT, r.w(pe + "conv_2.0.weight"), 1, 3, 3 * C, r.w(pe + "conv_2.0.bias"), e2, C, M2, C, C).taps(3, W3_DY, W3_DX).conv(T, F2, T, F, 2).run(r);
        Tabs t2 = make_tabs(r, B, C);
        inst_norm_site(r, e2, C, B, (long long)T * F2, F2, C, r.w(pe + "conv_2.1.weight"), r.w(pe + "conv_2.1.bias"), t2, sums);
        if (r.live()) r.ok(cmgan_norm_apply(e2, C, B, (long long)T * F2, C, 1, t2.scale, t2.shift, C, r.w(pe + "conv_2.2.weight"), hA, C, r.st));
        if (sv) { sv->catE = catE; sv->raw0 = raw0; sv->tab0 = t0; sv->e2 = e2; sv->tab2 = t2; }
        r.top = mark;
    }
    // ---- 4 x TSCB (generator.py:92-99): time conformer then frequency conformer on the same rows
    float *h = hA, *hn = hB;
    for (int k = 0; k < 8; ++k) {
        if (sv) hn = r.keep((size_t)M2 * C);
        conformer(r, h, hn, conformer_name(k), B, T, F2, k % 2, k, &sums, sv ? &sv->conf[k] : nullptr);
        float* t = h; h = hn; hn = t;
    }
    // ---- decoders (generator.py:122-156)
    float* sp[2];
    for (int dd = 0; dd < 2; ++dd) {
        const std::string pd = DEC_NAMES[dd];
        sp[dd] = r.keep((size_t)M2 * 2 * C);          // (B, T, 2 F2, 64): the sub-pixel shuffle is a reinterpretation
        const size_t mark = r.top;
        float* cat = r.keep((size_t)M2 * CAT);
        if (r.live()) r.ok(cmgan_copy_rows_operand(h, C, cat + 4 * C, CAT, M2, C, r.st));
        dense_block(r, cat, pd + "dense_block.", B, T, F2, sums, sv ? &sv->dec[dd] : nullptr);
        Gemm(cat, CAT, r.w(pd + "sub_pixel.conv.weight"), 1, 3, 3 * C, r.w(pd + "sub_pixel.conv.bias"), sp[dd], 2 * C, M2, 2 * C, C)
            .taps(3, W3_DY, W3_DX).conv(T, F2, T, F2).run(r);
        if (sv) { sv->cat[dd] = cat; sv->sp[dd] = sp[dd]; }
        r.top = mark;
    }
    const std::string pm = "mask_decoder.", pc = "complex_decoder.";
    float* m1 = r.keep((size_t)M);
    Tabs tabM = make_tabs(r, B, 1), tabC = make_tabs(r, B, C);
    if (sv) { sv->m1 = m1; sv->tabM = tabM; sv->tabC = tabC; }
    float* cplx = r.alloc((size_t)M * 2);
    if (r.live()) r.ok(cmgan_rowdot_fwd(sp[0], B, T, F, 1, nullptr, nullptr, nullptr, r.w(pm + "conv_1.weight"), r.w(pm + "conv_1.bias"), m1, r.st));
    inst_norm_site(r, m1, 1, B, (long long)T * F, F, 1, r.w(pm + "norm.weight"), r.w(pm + "norm.bias"), tabM, sums);
    inst_norm_site(r, sp[1], C, B, (long long)T * 2 * F2, 2 * F2, C, r.w(pc + "norm.weight"), r.w(pc + "norm.bias"), tabC, sums);
    if (r.live()) {
        r.ok(cmgan_rowdot_fwd(sp[1], B, T, F, 2, tabC.scale, tabC.shift, r.w(pc + "prelu.weight"), r.w(pc + "conv.weight"), r.w(pc + "conv.bias"), cplx, r.st));
        r.ok(cmgan_recombine(m1, tabM.scale, tabM.shift, r.w(pm + "prelu.weight"), r.w(pm + "final_conv.weight"), r.w(pm + "final_conv.bias"),
                             r.w(pm + "prelu_out.weight"), x, sxb, sxc, sxt, sxf, cplx, B, T, F, fr, fi, r.st));
    }
    if ((size_t)(sums - sums0) > n_sums && r.rc == 0) { cmgan_set_error("cmgan_tscnet_fwd: statistics scratch exhausted"); r.rc = -1; }
}

// ==================================================================================== backward (network.tscnet_bwd, conformer_block.conformer_bwd)
// The launch sequence of the Python walk on one stream (ops.WGRAD_STREAM = ops.AUX_STREAM = None, no weight-pack cache, ATTN_BWD_WS off).

// LayerNorm backward (+ residual gradients); with dz also the dropout-scaled copy dz = zalpha * mask(zseed) * dx that enters the next branch
void ln_bwd(Run& r, long long M, const float* dy, const float* x, const float* st, const std::string& name, const float* res, const float* res2,
            float* dx, float* dz = nullptr, float zalpha = 0.f, unsigned long long zseed = 0) {
    if (!r.live()) return;
    const float* gam = r.w(name + ".weight");
    float *dg = r.g(name + ".weight"), *db = r.g(name + ".bias");
    if (!dz)
        r.ok(cmgan_ln_bwd(dy, C, x, C, st, gam, M, res, res ? C : 0, res2, res2 ? C : 0, dx, C, dg, db, r.st));
    else
        r.ok(cmgan_ln_bwd_drop(dy, C, x, C, st, gam, M, res, res ? C : 0, res2, res2 ? C : 0, dx, C, dg, db, dz, C, zalpha, zseed, drop_thr(r.training),
                               drop_inv(r.training), r.seed_dev, r.st));
}

// out = xin + 0.5 * drop2(W2 a + b2), a = swish(h) * drop1, h = W1 LN(xin) + b1;  dz = 0.5 * drop2-mask * dout  ->  dx (+ res2)
void feed_forward_bwd(Run& r, long long M, const std::string& p, const FfSaved& f, const float* xin, const float* dout, const float* dz,
                      const float* res2, unsigned long long s1, float* dx) {
    const size_t mark = r.top;
    const float *W1 = r.w(p + "fn.fn.net.0.weight"), *W2 = r.w(p + "fn.fn.net.3.weight");
    if (r.precision == 1) {      // hidden activation recomputed, dh formed in the same kernel; it leaves a, dh and xn for the weight gradients
        float* w1p = r.alloc((size_t)4 * C * C);
        float* w2tp = r.alloc((size_t)4 * C * C);
        float* w1tp = r.alloc((size_t)4 * C * C);
        float* a = r.alloc((size_t)M * 4 * C);
        float* dh = r.alloc((size_t)M * 4 * C);
        float* xn = r.alloc((size_t)M * C);
        float* ws = r.alloc((size_t)M * (2 + C));
        if (r.live()) {
            r.ok(cmgan_pack_weight(W1, w1p, 0, 1, C, C, 1, 4 * C, r.st));
            r.ok(cmgan_pack_weight(W2, w2tp, 0, 4 * C, 1, C, 1, 4 * C, r.st));
            r.ok(cmgan_pack_weight(W1, w1tp, 0, C, 1, 4 * C, 1, C, r.st));
            r.ok(cmgan_ffn_bwd(xin, C, dz, C, dout, C, res2, res2 ? C : 0, M, r.w(p + "fn.norm.weight"), r.w(p + "fn.norm.bias"), w1p,
                               r.w(p + "fn.fn.net.0.bias"), w2tp, w1tp, s1, drop_thr(r.training), drop_inv(r.training), r.seed_dev, dx, C, a, dh, xn,
                               r.g(p + "fn.norm.weight"), r.g(p + "fn.norm.bias"), ws, r.st));
        }
        Gemm(a, 4 * C, nullptr, 0, 1, 4 * C, nullptr, r.g(p + "fn.fn.net.3.weight"), 0, M, C, 4 * C).wgrad(dz, C, r.g(p + "fn.fn.net.3.bias")).run(r);
        Gemm(xn, C, nullptr, 0, 1, C, nullptr, r.g(p + "fn.fn.net.0.weight"), 0, M, 4 * C, C).wgrad(dh, 4 * C, r.g(p + "fn.fn.net.0.bias")).run(r);
        r.top = mark;
        return;
    }
    float* dh = r.alloc((size_t)M * 4 * C);
    Gemm(dz, C, W2, 0, 4 * C, 1, nullptr, dh, 4 * C, M, 4 * C, C).epi(CMGAN_EPI_DSWISH_DROP, f.h, 4 * C)
        .drop(s1, drop_thr(r.training), drop_inv(r.training)).run(r);
    Gemm(f.a, 4 * C, nullptr, 0, 1, 4 * C, nullptr, r.g(p + "fn.fn.net.3.weight"), 0, M, C, 4 * C).wgrad(dz, C, r.g(p + "fn.fn.net.3.bias")).run(r);
    float* dln = r.alloc((size_t)M * C);
    Gemm(dh, 4 * C, W1, 0, C, 1, nullptr, dln, C, M, C, 4 * C).run(r);
    Gemm(f.xn, C, nullptr, 0, 1, C, nullptr, r.g(p + "fn.fn.net.0.weight"), 0, M, 4 * C, C).wgrad(dh, 4 * C, r.g(p + "fn.fn.net.0.bias")).run(r);
    ln_bwd(r, M, dln, xin, f.st, p + "fn.norm", dout, res2, dx);
    r.top = mark;
}

// gradient of conformer(): dy (M, 64) -> dx (M, 64)
void conformer_bwd(Run& r, const ConfSaved& s, const float* dy, float* dx, const std::string& p, int B, int T, int F2, int axis, int block_id,
                   double*& sums) {
    const long long M = (long long)B * T * F2;
    const size_t mark = r.top;
    unsigned long long sd[5];
    for (int i = 0; i < 5; ++i) sd[i] = site_seed(r.seed, block_id, i);
    // y = LN(x4) * g + b + x
    float* dx4 = r.alloc((size_t)M * C);
    float* dz4 = r.alloc((size_t)M * C);
    ln_bwd(r, M, dy, s.x4, s.st5, p + "post_norm", nullptr, nullptr, dx4, dz4, 0.5f, sd[4]);
    float* dx3 = r.alloc((size_t)M * C);
    feed_forward_bwd(r, M, p + "ff2.", s.f2, s.x3, dx4, dz4, nullptr, sd[3], dx3);
    // ---- convolution module: x3 = x2 + W7 swish(bn(d)) + b7
    float* dbn = r.alloc((size_t)M * 2 * C);
    const float* dx3_op = dx3;
    if (r.precision == 1) {      // dx3 also carries the residual gradient at full precision: the tensor-core operand is a rounded copy
        float* t = r.alloc((size_t)M * C);
        if (r.live()) r.ok(cmgan_copy_rows_operand(dx3, C, t, C, M, C, r.st));
        dx3_op = t;
    }
    Gemm gb(dx3_op, C, r.w(p + "conv.net.7.weight"), 0, 2 * C, 1, nullptr, dbn, 2 * C, M, 2 * C, C);
    gb.epi(CMGAN_EPI_DBNSWISH, s.d, 2 * C);
    gb.a.e0 = s.bn.scale; gb.a.e1 = s.bn.shift;
    gb.run(r);
    Gemm(s.dsw, 2 * C, nullptr, 0, 1, 2 * C, nullptr, r.g(p + "conv.net.7.weight"), 0, M, C, 2 * C).wgrad(dx3, C, r.g(p + "conv.net.7.bias")).run(r);
    float* dd = r.alloc((size_t)M * 2 * C);
    norm_bwd(r, s.d, 2 * C, dbn, 2 * C, 1, M, 2 * C, 0, r.training ? 1 : 0, s.bn, nullptr, dd, 2 * C, r.g(p + "conv.net.5.weight"),
             r.g(p + "conv.net.5.bias"), nullptr, sums, false);
    float* dg = r.alloc((size_t)M * 4 * C);
    if (r.live())
        r.ok(cmgan_glu_dwconv_bwd(s.g, dd, r.w(p + "conv.net.4.conv.weight"), B, T, F2, axis, dg, r.g(p + "conv.net.4.conv.weight"),
                                  r.g(p + "conv.net.4.conv.bias"), r.st));
    float* dln3 = r.alloc((size_t)M * C);
    Gemm(dg, 4 * C, r.w(p + "conv.net.2.weight"), 0, C, 1, nullptr, dln3, C, M, C, 4 * C).run(r);
    Gemm(s.xn3, C, nullptr, 0, 1, C, nullptr, r.g(p + "conv.net.2.weight"), 0, M, 4 * C, C).wgrad(dg, 4 * C, r.g(p + "conv.net.2.bias")).run(r);
    float* dx2 = r.alloc((size_t)M * C);
    float* dz2 = r.training ? r.alloc((size_t)M * C) : dx2;     // attention dropout: the to_out branch sees mask * dx2
    ln_bwd(r, M, dln3, s.x2, s.st3, p + "conv.net.0", dx3, nullptr, dx2, r.training ? dz2 : nullptr, 1.f, sd[2]);
    // ---- attention: x2 = x1 + drop(ctx Wo^T + bo)
    float* dctx = r.alloc((size_t)M * C);
    Gemm(dz2, C, r.w(p + "attn.fn.to_out.weight"), 0, C, 1, nullptr, dctx, C, M, C, C).run(r);
    Gemm(s.ctx, C, nullptr, 0, 1, C, nullptr, r.g(p + "attn.fn.to_out.weight"), 0, M, C, C).wgrad(dz2, C, r.g(p + "attn.fn.to_out.bias")).run(r);
    float* dqkv = r.alloc((size_t)M * 3 * C);
    float* delta = r.alloc((size_t)M * 4);
    if (r.live()) {
        const float* E = r.w(p + "attn.fn.rel_pos_emb.weight");
        float* dE = r.g(p + "attn.fn.rel_pos_emb.weight");
        r.ok(r.precision == 1 ? cmgan_attention_bwd_tf32_ws(s.qkv, E, s.ctx, dctx, s.lse, B, T, F2, axis, delta, dqkv, dE, 7, nullptr, 0, r.st)
                              : cmgan_attention_bwd(s.qkv, E, s.ctx, dctx, s.lse, B, T, F2, axis, delta, dqkv, dE, r.st));
    }
    // to_q and to_kv (and their gradients) are adjacent in the blocks: one (192, 64) projection
    float* dln2 = r.alloc((size_t)M * C);
    Gemm(dqkv, 3 * C, r.w(p + "attn.fn.to_q.weight"), 0, C, 1, nullptr, dln2, C, M, C, 3 * C).run(r);
    Gemm(s.xn2, C, nullptr, 0, 1, C, nullptr, r.g(p + "attn.fn.to_q.weight"), 0, M, 3 * C, C).wgrad(dqkv, 3 * C, nullptr).run(r);
    float* dx1 = r.alloc((size_t)M * C);
    float* dz1 = r.alloc((size_t)M * C);
    ln_bwd(r, M, dln2, s.x1, s.st2, p + "attn.norm", dx2, nullptr, dx1, dz1, 0.5f, sd[1]);
    // ---- first feed-forward; the outer residual adds dy
    feed_forward_bwd(r, M, p + "ff1.", s.f1, s.x, dx1, dz1, dy, sd[0], dx);
    r.top = mark;
}

// dcat slot 0 holds the gradient wrt act(out4); on return dcat slot 4 holds the gradient wrt the block input (network.dense_block_bwd)
void dense_block_bwd(Run& r, const float* cat, const DenseSaved& s, float* dcat, const std::string& p, int B, int T, int Fw, double*& sums) {
    const long long M = (long long)B * T * Fw, rows = (long long)T * Fw;
    for (int i = 4; i >= 1; --i) {
        const int dil = 1 << (i - 1), c0 = (5 - i) * C, Cin = C * i, co = (4 - i) * C;
        const std::string n = std::to_string(i);
        const size_t mark = r.top;
        float* draw = r.alloc((size_t)M * C);
        norm_bwd(r, s.raw[i - 1], C, off(dcat, co), CAT, B, rows, C, 1, 1, s.tab[i - 1], r.w(p + "prelu" + n + ".weight"), draw, C,
                 r.g(p + "norm" + n + ".weight"), r.g(p + "norm" + n + ".bias"), r.g(p + "prelu" + n + ".weight"), sums, true);
        const int dy[6] = {-dil, -dil, -dil, 0, 0, 0}, dx[6] = {-1, 0, 1, -1, 0, 1};
        const int ndy[6] = {dil, dil, dil, 0, 0, 0}, ndx[6] = {1, 0, -1, 1, 0, -1};
        Gemm(off(cat, c0), CAT, nullptr, 1, 6, (long long)Cin * 6, nullptr, r.g(p + "conv" + n + ".weight"), 0, M, C, Cin).taps(6, dy, dx)
            .conv(T, Fw, T, Fw).wgrad(draw, C, r.g(p + "conv" + n + ".bias")).run(r);
        Gemm dg(draw, C, r.w(p + "conv" + n + ".weight"), 1, (long long)Cin * 6, 6, nullptr, off(dcat, c0), CAT, M, Cin, C);
        dg.taps(6, ndy, ndx).conv(T, Fw, T, Fw).a.epi = i == 4 ? CMGAN_EPI_NONE : CMGAN_EPI_ACC;
        dg.run(r);
        r.top = mark;
    }
}

// dfr / dfi (B, 1, T, F) with strides (sgb, sgt, sgf), null = zero; dx (B, 2, T, F) contiguous or null
void backward(Run& r, const Saved& sv, const float* x, long long sxb, long long sxc, long long sxt, long long sxf, int B, int T, int F, const float* dfr,
              const float* dfi, long long sgb, long long sgt, long long sgf, float* dx) {
    const int F2 = (F - 1) / 2 + 1;
    const long long M = (long long)B * T * F, M2 = (long long)B * T * F2;
    const size_t n_sums = sums_size(B, true);
    double* sums0 = r.alloc<double>(n_sums);
    double* sums = sums0;
    float* zero = r.alloc((size_t)M);            // stands in for a null dfr / dfi (laid out with the given strides: span <= B T F, checked on entry)
    if (r.live()) {
        cudaError_t e = cudaMemsetAsync(sums0, 0, n_sums * sizeof(double), r.st);
        if (e == cudaSuccess && (!dfr || !dfi)) e = cudaMemsetAsync(zero, 0, (size_t)M * sizeof(float), r.st);
        if (e != cudaSuccess) { cmgan_set_error("cmgan_tscnet_bwd: cudaMemsetAsync: %s", cudaGetErrorString(e)); r.rc = -1; }
    }
    if (!dfr) dfr = zero;
    if (!dfi) dfi = zero;
    const std::string pm = "mask_decoder.", pc = "complex_decoder.", pe = "dense_encoder.";
    // ---- tails: final = mask * x + cplx (generator.py:136-139,150,191-196)
    float* dsp[2] = {r.alloc((size_t)M2 * 2 * C), r.alloc((size_t)M2 * 2 * C)};
    float *dh = r.alloc((size_t)M2 * C), *dh2 = r.alloc((size_t)M2 * C);      // TSCB gradients ping-pong between these two
    {
        const size_t mark = r.top;
        float* dcplx = r.alloc((size_t)M * 2);
        float* dz = r.alloc((size_t)M);
        if (r.live())
            r.ok(cmgan_recombine_bwd(sv.m1, sv.tabM.scale, sv.tabM.shift, r.w(pm + "prelu.weight"), r.w(pm + "final_conv.weight"), r.w(pm + "final_conv.bias"),
                                     r.w(pm + "prelu_out.weight"), x, sxb, sxc, sxt, sxf, dfr, dfi, sgb, sgt, sgf, B, T, F, dcplx, dz, r.g(pm + "prelu_out.weight"),
                                     r.g(pm + "final_conv.weight"), r.g(pm + "final_conv.bias"), r.st));
        float* dm1 = r.alloc((size_t)M);
        norm_bwd(r, sv.m1, 1, dz, 1, B, (long long)T * F, 1, 1, 1, sv.tabM, r.w(pm + "prelu.weight"), dm1, 1, r.g(pm + "norm.weight"), r.g(pm + "norm.bias"),
                 r.g(pm + "prelu.weight"), sums, false);
        if (r.live()) {
            r.ok(cmgan_rowdot_bwd(sv.sp[0], B, T, F, 1, nullptr, nullptr, nullptr, r.w(pm + "conv_1.weight"), dm1, dsp[0], r.g(pm + "conv_1.weight"),
                                  r.g(pm + "conv_1.bias"), r.st));
            r.ok(cmgan_copy_rows_operand(dsp[0], 2 * C, dsp[0], 2 * C, M2, 2 * C, r.st));      // operand of the sub-pixel convolution's gradient GEMMs
        }
        float* dactc = r.alloc((size_t)M2 * 2 * C);
        if (r.live())
            r.ok(cmgan_rowdot_bwd(sv.sp[1], B, T, F, 2, sv.tabC.scale, sv.tabC.shift, r.w(pc + "prelu.weight"), r.w(pc + "conv.weight"), dcplx, dactc,
                                  r.g(pc + "conv.weight"), r.g(pc + "conv.bias"), r.st));
        norm_bwd(r, sv.sp[1], C, dactc, C, B, (long long)T * 2 * F2, C, 1, 1, sv.tabC, r.w(pc + "prelu.weight"), dsp[1], C, r.g(pc + "norm.weight"),
                 r.g(pc + "norm.bias"), r.g(pc + "prelu.weight"), sums, true);
        r.top = mark;
    }
    // ---- decoders: sub-pixel convolution, dense block; both add into the gradient of the last TSCB's output
    for (int dd = 0; dd < 2; ++dd) {
        const std::string pd = DEC_NAMES[dd];
        const size_t mark = r.top;
        float* dcat = r.alloc((size_t)M2 * CAT);
        Gemm(sv.cat[dd], CAT, nullptr, 1, 3, 3 * C, nullptr, r.g(pd + "sub_pixel.conv.weight"), 0, M2, 2 * C, C).taps(3, W3_DY, W3_DX).conv(T, F2, T, F2)
            .wgrad(dsp[dd], 2 * C, r.g(pd + "sub_pixel.conv.bias")).run(r);
        Gemm(dsp[dd], 2 * C, r.w(pd + "sub_pixel.conv.weight"), 1, 3 * C, 3, nullptr, dcat, CAT, M2, C, 2 * C).taps(3, W3_DY, W3T_DX).conv(T, F2, T, F2).run(r);
        dense_block_bwd(r, sv.cat[dd], sv.dec[dd], dcat, pd + "dense_block.", B, T, F2, sums);
        if (r.live()) r.ok((dd == 0 ? cmgan_copy_rows : cmgan_add_rows)(dcat + 4 * C, CAT, dh, C, M2, C, r.st));
        r.top = mark;
    }
    // ---- TSCBs in reverse
    for (int k = 7; k >= 0; --k) {
        conformer_bwd(r, sv.conf[k], dh, dh2, conformer_name(k), B, T, F2, k % 2, k, sums);
        float* t = dh; dh = dh2; dh2 = t;
    }
    // ---- encoder
    float* de2 = r.alloc((size_t)M2 * C);
    norm_bwd(r, sv.e2, C, dh, C, B, (long long)T * F2, C, 1, 1, sv.tab2, r.w(pe + "conv_2.2.weight"), de2, C, r.g(pe + "conv_2.1.weight"),
             r.g(pe + "conv_2.1.bias"), r.g(pe + "conv_2.2.weight"), sums, true);
    Gemm(sv.catE, CAT, nullptr, 1, 3, 3 * C, nullptr, r.g(pe + "conv_2.0.weight"), 0, M2, C, C).taps(3, W3_DY, W3_DX).conv(T, F2, T, F, 2)
        .wgrad(de2, C, r.g(pe + "conv_2.0.bias")).run(r);
    float* dcatE = r.alloc((size_t)M * CAT);
    Gemm(de2, C, r.w(pe + "conv_2.0.weight"), 1, 3 * C, 3, nullptr, dcatE, CAT, M, C, C).taps(3, W3_DY, W3T_DX).conv(T, F, T, F2, 1, 2).run(r);
    dense_block_bwd(r, sv.catE, sv.enc, dcatE, pe + "dilated_dense.", B, T, F, sums);
    float* draw1 = r.alloc((size_t)M * C);
    norm_bwd(r, sv.raw0, C, off(dcatE, 4 * C), CAT, B, (long long)T * F, C, 1, 1, sv.tab0, r.w(pe + "conv_1.2.weight"), draw1, C,
             r.g(pe + "conv_1.1.weight"), r.g(pe + "conv_1.1.bias"), r.g(pe + "conv_1.2.weight"), sums, false);
    if (r.wgrad && r.live())
        r.ok(cmgan_head_conv_wgrad(x, sxb, sxc, sxt, sxf, B, T, F, draw1, C, r.g(pe + "conv_1.0.weight"), r.g(pe + "conv_1.0.bias"), r.st));
    if (dx && r.live())         // final = mask x + cplx and the head reads [|x|, re, im]: one pass over draw1 and the recomputed mask
        r.ok(cmgan_tscnet_input_grad(sv.m1, sv.tabM.scale, sv.tabM.shift, r.w(pm + "prelu.weight"), r.w(pm + "final_conv.weight"),
                                     r.w(pm + "final_conv.bias"), r.w(pm + "prelu_out.weight"), x, sxb, sxc, sxt, sxf, dfr, dfi, sgb, sgt, sgf, draw1, C,
                                     r.w(pe + "conv_1.0.weight"), B, T, F, dx, r.st));
    if ((size_t)(sums - sums0) > n_sums && r.rc == 0) { cmgan_set_error("cmgan_tscnet_bwd: statistics scratch exhausted"); r.rc = -1; }
}

// ---- waveform in, waveform out (evaluation.py:21-53): the launch sequence of signal.enhance / enhance_ragged around forward()
constexpr int NFFT = 400, HOP = 100;

// k segments of S samples per clip, T frames per segment, Lp padded samples per row, rows = B k in all, run `pass` rows at a time
struct EnhanceGeom { int k, S, T, Lp, rows, pass; };

// The fold of a clip of L samples (signal.fold_geometry restates it): padded = ceil(L / 100) * 100, wrap-padded with the clip's own head.
//   1. padded <= cut_len: one segment.
//   2. the reference's rule (evaluation.py:30-34): k = ceil(padded / cut_len), raised until it divides 100, S = padded / k; each segment
//      yields 100 floor(S / 100) samples, concatenated and cut to L.
//   3. extend only, where rule 2 fails -- its loop never ends (k would pass 100) or its segments yield fewer than L samples (the reference's
//      own length assertion fails): S_max = 100 floor(cut_len / 100) >= 300, k = ceil(padded / S_max), S = 100 ceil(padded / (100 k))
//      <= S_max, wrap-padded to k S <= 2 L; the segments tile the clip without a gap.  The reference has no behaviour to match here.
// 0, or -1 with the message set.  The 2^31 bound on rows * T is checked here for a single pass only (!extend).
int enhance_geom(int B, int L, int cut_len, bool ragged, bool extend, EnhanceGeom& g, const char* who) {
    CMGAN_REQUIRE(B > 0, "%s: B must be positive (B=%d)", who, B);
    CMGAN_REQUIRE(L > NFFT / 2, "%s: L=%d samples; a clip needs more than the 200-sample reflect padding of the STFT", who, L);
    CMGAN_REQUIRE(cut_len > 0, "%s: cut_len must be positive (cut_len=%d)", who, cut_len);
    const long long padded = ((long long)L + HOP - 1) / HOP * HOP;
    CMGAN_REQUIRE(padded - L <= L, "%s: wrap padding L=%d to %lld is longer than the clip", who, L, padded);
    long long k = 1, S = padded;
    if (padded > cut_len) {
        CMGAN_REQUIRE(!ragged, "%s: a ragged batch needs ceil(L / 100) * 100 <= cut_len (L=%d, cut_len=%d); longer clips take the uniform call, "
                      "which folds them", who, L, cut_len);
        k = (padded + cut_len - 1) / cut_len;
        while (k <= HOP && HOP % k != 0) ++k;
        if (k <= HOP) S = padded / k;
        if (k > HOP || (extend && k * HOP * (S / HOP) < L)) {
            CMGAN_REQUIRE(extend, "%s: L=%d with cut_len=%d folds into more than 100 segments", who, L, cut_len);
            const long long smax = cut_len / HOP * HOP;
            CMGAN_REQUIRE(smax >= 3 * HOP, "%s: cut_len=%d gives segments of at most %lld samples; a segment needs more than 200", who, cut_len, smax);
            k = (padded + smax - 1) / smax;
            S = (padded + HOP * k - 1) / (HOP * k) * HOP;
            CMGAN_REQUIRE(k * S - L <= L, "%s: wrap padding L=%d to %lld segments of %lld samples is longer than the clip", who, L, k, S);
        }
    }
    g.k = (int)k;
    g.S = (int)S;
    CMGAN_REQUIRE(g.S > NFFT / 2, "%s: L=%d with cut_len=%d folds into %d segments of %d samples; a segment needs more than 200", who, L,
                  cut_len, g.k, g.S);
    g.T = g.S / HOP + 1;
    CMGAN_REQUIRE(k * HOP * (g.T - 1) >= L, "%s: L=%d with cut_len=%d folds into %d segments of %d samples, which yield only %lld samples", who,
                  L, cut_len, g.k, g.S, k * HOP * (g.T - 1));
    if (!extend) {
        const long long elems = (long long)B * k * g.T * NFEAT * CAT;
        CMGAN_REQUIRE(elems < (1ll << 31), "%s: rows * T * 201 * %d = %lld elements reach 2^31 (32-bit indexing of the encoder concat buffer); "
                      "split the batch", who, CAT, elems);
    }
    g.rows = (int)(B * k);
    g.pass = g.rows;
    g.Lp = (g.S + NFFT + HOP - 1) / HOP * HOP;
    return 0;
}

// The overlapping windows of cmgan_enhance_overlap (signal.overlap_geometry restates it), one clip of L samples, padded = ceil(L / 100) * 100,
// S_max = 100 floor(cut_len / 100).  Needs overlap O a multiple of 100 with 100 <= O and 2 O <= S_max, cut_len >= 300, L > 200 and
// padded - L <= L.
//   padded <= S_max: one window of S = padded samples, the one-segment case of cmgan_enhance_long (h = S).
//   otherwise: S = S_max, hop h = S - O, k = 1 + ceil((padded - S) / h) windows, window j covering [j h, j h + S) of the clip wrap-padded with
//   its own head to Lw = (k - 1) h + S; needs Lw - L <= L.
// 0, or -1 with the message set.
int overlap_geom(int L, int cut_len, int overlap, EnhanceGeom& g, int& h, const char* who) {
    CMGAN_REQUIRE(cut_len >= 3 * HOP, "%s: cut_len=%d gives windows of at most %d samples; a window needs more than 200", who, cut_len,
                  cut_len / HOP * HOP);
    const int smax = cut_len / HOP * HOP;
    CMGAN_REQUIRE(overlap >= HOP && overlap % HOP == 0 && 2LL * overlap <= smax,
                  "%s: overlap=%d must be a multiple of 100 with 100 <= overlap <= %d (half of the %d-sample windows at cut_len=%d)", who, overlap,
                  smax / 2, smax, cut_len);
    CMGAN_REQUIRE(L > NFFT / 2, "%s: L=%d samples; a clip needs more than the 200-sample reflect padding of the STFT", who, L);
    const long long padded = ((long long)L + HOP - 1) / HOP * HOP;
    CMGAN_REQUIRE(padded - L <= L, "%s: wrap padding L=%d to %lld is longer than the clip", who, L, padded);
    long long k = 1, S = padded, H = padded;
    if (padded > smax) {
        S = smax;
        H = S - overlap;
        k = 1 + (padded - S + H - 1) / H;
        CMGAN_REQUIRE((k - 1) * H + S - L <= L, "%s: wrap padding L=%d to %lld windows of %lld samples at hop %lld is longer than the clip", who,
                      L, k, S, H);
    }
    g.k = (int)k;
    g.S = (int)S;
    g.T = g.S / HOP + 1;
    g.rows = g.k;
    g.pass = g.rows;
    g.Lp = (g.S + NFFT + HOP - 1) / HOP * HOP;
    h = (int)H;
    return 0;
}

// the crossfade of overlapping windows: overlap O samples, hop S - O
struct Crossfade { int overlap, hop; };

// The launch sequence of signal.enhance / enhance_ragged around forward(): the STFT tables and the RMS scales of the whole clips, then the
// rows in passes of g.pass -- padding, DFT, compression, TSCNet, un-compression, inverse DFT, overlap-add into that pass's range of `out`.
// Several passes only for one clip (B = 1): the segments share nothing but c.
// xf (B = 1 only): the rows are overlapping windows, starting xf->hop samples apart; each pass overlap-adds its windows into a staging buffer
// and cmgan_crossfade joins them into its range of `out`.
void enhance_walk(Run& r, const float* wav, long long ldw, int B, int L, const int* lengths, const EnhanceGeom& g, float* out, long long ldo,
                  const Crossfade* xf = nullptr) {
    const int T = g.T, F = NFEAT;
    float* fwd = r.alloc((size_t)NFFT * 2 * F);
    float* inv = r.alloc((size_t)2 * F * NFFT);
    float* env = r.alloc((size_t)HOP * (T - 1));
    float* tail = r.alloc(HOP);
    float* c = r.alloc(B);
    int* tlen = r.alloc<int>(B);
    float* X = r.alloc((size_t)g.pass * T * 2 * F);
    float* fr = r.alloc((size_t)g.pass * T * F);
    float* fi = r.alloc((size_t)g.pass * T * F);
    if (r.live()) r.ok(cmgan_stft_tables(fwd, inv, T, env, tail, r.st));
    if (r.live()) r.ok(lengths ? cmgan_rms_scale_frames(wav, ldw, B, L, lengths, c, tlen, r.st) : cmgan_rms_scale(wav, ldw, B, L, c, r.st));
    float* xw = xf ? r.alloc(xf->overlap) : nullptr;
    if (xf && r.live()) r.ok(cmgan_crossfade_table(xw, xf->overlap, r.st));
    const size_t mark = r.top;
    const long long Lout = (long long)HOP * (T - 1);        // samples each segment yields
    for (int s0 = 0; s0 < g.rows; s0 += g.pass) {
        const int rows = std::min(g.pass, g.rows - s0), kp = rows / B;       // rows of this pass, segments per clip in it
        const long long MT = (long long)rows * T;
        // ---- signal._stft_padded: wrap + reflect (+ fold) padding, framed DFT (exact fp32 FFMA), power compression
        {
            float* xp = r.alloc((size_t)rows * g.Lp);
            float* S = r.alloc((size_t)MT * 2 * F);
            if (r.live())
                r.ok(lengths ? cmgan_pad_wrap_reflect_ragged(wav, ldw, B, L, lengths, c, xp, g.Lp, r.st)
                             : cmgan_pad_wrap_reflect_fold(wav, ldw, B, L, kp, g.S, s0, xf ? xf->hop : g.S, c, xp, g.Lp, r.st));
            Gemm dft(xp, HOP, fwd, 0, 2 * F, 1, nullptr, S, 2 * F, MT, 2 * F, NFFT);
            dft.conv(1, T, 1, g.Lp / HOP);
            if (r.live()) r.ok(cmgan_gemm_rows_f32(&dft.a, r.st));          // precision 0 (memset by Gemm): the DFTs stay exact fp32
            if (r.live()) r.ok(cmgan_compress(S, rows, T, X, r.st));
            r.top = mark;
        }
        // ---- TSCNet.forward on (rows, 2, T, F) contiguous; a ragged batch passes its frame counts
        r.frames = lengths ? tlen : nullptr;
        forward(r, X, 2LL * T * F, (long long)T * F, F, 1, rows, T, F, fr, fi);
        r.frames = nullptr;
        r.top = mark;
        // ---- signal.uncompress_istft_fwd: un-compression, inverse DFT (exact fp32 FFMA), overlap-add straight into `out`
        float* U = r.alloc((size_t)MT * 2 * F);
        float* frames = r.alloc((size_t)MT * NFFT);
        if (r.live()) r.ok(cmgan_uncompress(fr, fi, (long long)T * F, F, 1, rows, T, U, r.st));
        Gemm idft(U, 2 * F, inv, 0, NFFT, 1, nullptr, frames, NFFT, MT, NFFT, 2 * F);
        if (r.live()) r.ok(cmgan_gemm_rows_f32(&idft.a, r.st));
        if (xf) {           // the windows' de-normalised outputs, (rows, S) contiguous, then the crossfade into out
            float* y = r.alloc((size_t)rows * g.S);
            if (r.live()) r.ok(cmgan_ola_fold(frames, rows, T, rows, env, c, y, 0, rows * g.S, r.st));
            if (r.live()) r.ok(cmgan_crossfade(y, rows, s0, g.k, g.S, xf->overlap, xw, out, L, r.st));
        } else if (r.live()) {
            r.ok(lengths ? cmgan_ola_ragged_lengths(frames, B, T, tlen, lengths, L, env, tail, c, out, ldo, r.st)
                         : cmgan_ola_fold(frames, rows, T, kp, env, c, out + s0 * Lout, ldo, (int)(L - s0 * Lout), r.st));
        }
        r.top = mark;
    }
}

}  // namespace

CMGAN_API int cmgan_tscnet_param_count(void) { return (int)table().e.size(); }
CMGAN_API long long cmgan_tscnet_param_floats(void) { return table().total; }

CMGAN_API int cmgan_tscnet_param_info(int index, const char** key, long long* offset, long long* numel) {
    CMGAN_REQUIRE(index >= 0 && index < (int)table().e.size(), "cmgan_tscnet_param_info: index %d out of range", index);
    const Entry& e = table().e[index];
    if (key) *key = e.key.c_str();
    if (offset) *offset = e.off;
    if (numel) *numel = e.numel;
    return 0;
}

CMGAN_API long long cmgan_tscnet_workspace_bytes(int B, int T, int F, int precision) {
    if (B <= 0 || T <= 0 || F != NFEAT || (precision != 0 && precision != 1)) { cmgan_set_error("cmgan_tscnet_workspace_bytes: bad arguments"); return -1; }
    Run r;
    r.P = nullptr; r.ws = nullptr; r.dry = true; r.precision = precision; r.st = nullptr;
    forward(r, nullptr, 0, 0, 0, 0, B, T, F, nullptr, nullptr);
    return (long long)r.peak + 256;
}

static int tscnet_fwd(const float* params, const float* x, long long sxb, long long sxc, long long sxt, long long sxf, int B, int T, int F,
                      const int* frames, float* final_real, float* final_imag, void* workspace, long long workspace_bytes, int precision, void* stream) {
    CMGAN_REQUIRE(params && x && final_real && final_imag && workspace, "cmgan_tscnet_fwd: null pointer");
    CMGAN_REQUIRE(B > 0 && T > 0 && F == NFEAT, "cmgan_tscnet_fwd: expected x of shape (B, 2, T, %d), got B=%d T=%d F=%d", NFEAT, B, T, F);
    CMGAN_REQUIRE(precision == 0 || precision == 1, "cmgan_tscnet_fwd: precision must be 0 (fp32) or 1 (tf32)");
    CMGAN_REQUIRE((((uintptr_t)params) & 15) == 0 && (((uintptr_t)workspace) & 255) == 0, "cmgan_tscnet_fwd: params must be 16-byte, workspace 256-byte aligned");
    cmgan_set_tf32_rounding(precision);       // producers of tensor-core operands round to nearest on store (library-wide switch)
    Run r;
    r.P = params; r.ws = static_cast<char*>(workspace); r.cap = (size_t)workspace_bytes; r.dry = false; r.precision = precision;
    r.st = (cudaStream_t)stream;
    r.frames = frames;
    forward(r, x, sxb, sxc, sxt, sxf, B, T, F, final_real, final_imag);
    return r.rc;
}

CMGAN_API int cmgan_tscnet_fwd(const float* params, const float* x, long long sxb, long long sxc, long long sxt, long long sxf, int B, int T, int F,
                               float* final_real, float* final_imag, void* workspace, long long workspace_bytes, int precision, void* stream) {
    return tscnet_fwd(params, x, sxb, sxc, sxt, sxf, B, T, F, nullptr, final_real, final_imag, workspace, workspace_bytes, precision, stream);
}

// ragged batch: utterance b occupies frames t < frames[b]; the InstanceNorms, the attention and the depthwise convolutions see only those
// frames, everything else works per row or causally in time (the dense blocks' dilated convolutions pad only the past)
CMGAN_API int cmgan_tscnet_fwd_ragged(const float* params, const float* x, long long sxb, long long sxc, long long sxt, long long sxf, int B, int T,
                                      int F, const int* frames, float* final_real, float* final_imag, void* workspace, long long workspace_bytes,
                                      int precision, void* stream) {
    CMGAN_REQUIRE(frames, "cmgan_tscnet_fwd_ragged: frames is null");
    CMGAN_REQUIRE(B > 0 && T > 0 && (long long)B * T * F * CAT < (1ll << 31),
                  "cmgan_tscnet_fwd_ragged: B * T * F * %d = %lld elements reach 2^31 (32-bit indexing of the encoder concat buffer); split the batch",
                  CAT, (long long)B * T * F * CAT);
    return tscnet_fwd(params, x, sxb, sxc, sxt, sxf, B, T, F, frames, final_real, final_imag, workspace, workspace_bytes, precision, stream);
}

// one size for the uniform and the ragged call at (B, L, cut_len): the walk allocates the same buffers in both modes
static long long enhance_bytes(int B, int L, const EnhanceGeom& g, int precision) {
    Run r;
    r.P = nullptr; r.ws = nullptr; r.dry = true; r.precision = precision; r.st = nullptr;
    enhance_walk(r, nullptr, L, B, L, nullptr, g, nullptr, L);
    return (long long)r.peak + 256;
}

CMGAN_API long long cmgan_enhance_workspace_bytes(int B, int L, int cut_len, int precision) {
    if (precision != 0 && precision != 1) { cmgan_set_error("cmgan_enhance_workspace_bytes: precision must be 0 (fp32) or 1 (tf32)"); return -1; }
    EnhanceGeom g;
    if (enhance_geom(B, L, cut_len, false, false, g, "cmgan_enhance_workspace_bytes") != 0) return -1;
    return enhance_bytes(B, L, g, precision);
}

CMGAN_API int cmgan_enhance(const float* params, const float* wav, long long ldw, int B, int L, const int* lengths, int cut_len, float* out,
                            long long ldo, void* workspace, long long workspace_bytes, int precision, void* stream) {
    CMGAN_REQUIRE(params && wav && out && workspace, "cmgan_enhance: null pointer");
    CMGAN_REQUIRE(precision == 0 || precision == 1, "cmgan_enhance: precision must be 0 (fp32) or 1 (tf32)");
    CMGAN_REQUIRE((((uintptr_t)params) & 15) == 0 && (((uintptr_t)workspace) & 255) == 0, "cmgan_enhance: params must be 16-byte, workspace 256-byte aligned");
    EnhanceGeom g;
    if (enhance_geom(B, L, cut_len, lengths != nullptr, false, g, "cmgan_enhance") != 0) return -1;
    CMGAN_REQUIRE(ldw >= L && ldo >= L, "cmgan_enhance: row strides must cover a clip (L=%d ldw=%lld ldo=%lld)", L, ldw, ldo);
    const uintptr_t w0 = (uintptr_t)wav, w1 = (uintptr_t)(wav + (B - 1) * ldw + L), o0 = (uintptr_t)out, o1 = (uintptr_t)(out + (B - 1) * ldo + L);
    CMGAN_REQUIRE(w1 <= o0 || o1 <= w0, "cmgan_enhance: wav and out overlap");
    const long long need = enhance_bytes(B, L, g, precision);
    CMGAN_REQUIRE(workspace_bytes >= need, "cmgan_enhance: workspace too small (%lld bytes needed, %lld given)", need, workspace_bytes);
    cmgan_set_tf32_rounding(precision);       // as cmgan_tscnet_fwd: producers of tensor-core operands round to nearest on store
    Run r;
    r.P = params; r.ws = static_cast<char*>(workspace); r.cap = (size_t)workspace_bytes; r.dry = false; r.precision = precision;
    r.st = (cudaStream_t)stream;
    enhance_walk(r, wav, ldw, B, L, lengths, g, out, ldo);
    return r.rc;
}

// one clip of any length in passes of at most max_segments segments: the workspace is that of one pass of max_segments segments of the
// longest S a fold can give at this cut_len (T_max = floor(cut_len / 100) + 1 frames), whatever L is
static long long enhance_long_bytes(int cut_len, int max_segments, int precision, const char* who) {
    CMGAN_REQUIRE(precision == 0 || precision == 1, "%s: precision must be 0 (fp32) or 1 (tf32)", who);
    CMGAN_REQUIRE(cut_len >= 3 * HOP, "%s: cut_len=%d gives segments of at most %d samples; a segment needs more than 200", who, cut_len,
                  cut_len / HOP * HOP);
    CMGAN_REQUIRE(max_segments > 0, "%s: max_segments must be positive (max_segments=%d)", who, max_segments);
    const int T = cut_len / HOP + 1;
    const long long elems = (long long)max_segments * T * NFEAT * CAT;
    CMGAN_REQUIRE(elems < (1ll << 31), "%s: max_segments * T * 201 * %d = %lld elements reach 2^31 (32-bit indexing of the encoder concat buffer; "
                  "T = %d frames at cut_len=%d); lower max_segments", who, CAT, elems, T, cut_len);
    const EnhanceGeom g{max_segments, cut_len, T, (cut_len + NFFT + HOP - 1) / HOP * HOP, max_segments, max_segments};
    return enhance_bytes(1, cut_len, g, precision);
}

CMGAN_API long long cmgan_enhance_long_workspace_bytes(int cut_len, int max_segments, int precision) {
    return enhance_long_bytes(cut_len, max_segments, precision, "cmgan_enhance_long_workspace_bytes");
}

CMGAN_API int cmgan_enhance_long(const float* params, const float* wav, int L, int cut_len, int max_segments, float* out, void* workspace,
                                 long long workspace_bytes, int precision, void* stream) {
    const char* who = "cmgan_enhance_long";
    CMGAN_REQUIRE(params && wav && out && workspace, "%s: null pointer", who);
    CMGAN_REQUIRE((((uintptr_t)params) & 15) == 0 && (((uintptr_t)workspace) & 255) == 0, "%s: params must be 16-byte, workspace 256-byte aligned", who);
    CMGAN_REQUIRE(L <= (1 << 30), "%s: L=%d samples; at most 2^30 (18.6 hours at 16 kHz) keeps every sample index in 32 bits", who, L);
    const long long need = enhance_long_bytes(cut_len, max_segments, precision, who);
    if (need < 0) return -1;
    EnhanceGeom g;
    if (enhance_geom(1, L, cut_len, false, true, g, who) != 0) return -1;
    const uintptr_t w0 = (uintptr_t)wav, w1 = (uintptr_t)(wav + L), o0 = (uintptr_t)out, o1 = (uintptr_t)(out + L);
    CMGAN_REQUIRE(w1 <= o0 || o1 <= w0, "%s: wav and out overlap", who);
    CMGAN_REQUIRE(workspace_bytes >= need, "%s: workspace too small (%lld bytes needed, %lld given)", who, need, workspace_bytes);
    g.pass = std::min(max_segments, g.k);
    EnhanceGeom first = g;          // every pass starts from the same mark, and the first one is the largest
    first.rows = g.pass;
    const long long run = enhance_bytes(1, L, first, precision);
    CMGAN_REQUIRE(run <= need, "%s: internal error: L=%d needs %lld workspace bytes, more than the query's %lld", who, L, run, need);
    cmgan_set_tf32_rounding(precision);       // as cmgan_tscnet_fwd: producers of tensor-core operands round to nearest on store
    Run r;
    r.P = params; r.ws = static_cast<char*>(workspace); r.cap = (size_t)workspace_bytes; r.dry = false; r.precision = precision;
    r.st = (cudaStream_t)stream; r.who = who;
    enhance_walk(r, wav, L, 1, L, nullptr, g, out, L);
    return r.rc;
}

// ==================================================================================== any sample rate: resample, the 16 kHz walk, resample back
// The model runs at 16 kHz.  At another rate sr the entries resample the clips to 16 kHz into the workspace, run cmgan_enhance /
// cmgan_enhance_long there on the rest of the workspace, and resample the 16 kHz result back into the caller's out, cut to each clip's
// length: a composition of public entries, so it computes exactly what the caller would get by chaining them.
namespace {

constexpr int SR_MODEL = 16000;

// what lies in front of the 16 kHz walk's workspace: both tap tables, the 16 kHz input and output (B rows of L16) and the 16 kHz lengths
struct SrRegion { float *h_in, *h_out, *x16, *y16; int* len16; };

// places the region at ws (null: sizes it only); returns its size, a multiple of 256 bytes
size_t sr_region(char* ws, const resample::Ratio& q, int B, long long L16, SrRegion& s) {
    Walk k;
    k.dry = ws == nullptr; k.ws = ws; k.cap = SIZE_MAX;
    const size_t taps = 2 * (size_t)q.half + 1;
    s.h_in = k.alloc(taps);
    s.h_out = k.alloc(taps);
    s.x16 = k.alloc((size_t)B * L16);
    s.y16 = k.alloc((size_t)B * L16);
    s.len16 = k.alloc<int>(B);
    return (k.top + 255) & ~(size_t)255;
}

// sr -> 16 kHz ratio and the 16 kHz length ceil(L up / down); 0, or -1 with the message set
int sr_geom(int sr, long long L, long long max16, resample::Ratio& q, long long& L16, const char* who) {
    if (resample::ratio(sr, SR_MODEL, q, who) != 0) return -1;
    CMGAN_REQUIRE(L > 0, "%s: L must be positive (L=%lld)", who, L);
    L16 = (L * q.up + q.down - 1) / q.down;
    CMGAN_REQUIRE(L16 <= max16, "%s: L=%lld samples at %d Hz are %lld at 16 kHz; at most %lld", who, L, sr, L16, max16);
    return 0;
}

}  // namespace

CMGAN_API long long cmgan_enhance_sr_workspace_bytes(int B, int L, int sr, int cut_len, int precision) {
    if (sr == SR_MODEL) return cmgan_enhance_workspace_bytes(B, L, cut_len, precision);
    const char* who = "cmgan_enhance_sr_workspace_bytes";
    if (precision != 0 && precision != 1) { cmgan_set_error("%s: precision must be 0 (fp32) or 1 (tf32)", who); return -1; }
    resample::Ratio q;
    long long L16;
    EnhanceGeom g;
    if (sr_geom(sr, L, INT32_MAX, q, L16, who) != 0 || enhance_geom(B, (int)L16, cut_len, false, false, g, who) != 0) return -1;
    SrRegion s;
    return (long long)sr_region(nullptr, q, B, L16, s) + enhance_bytes(B, (int)L16, g, precision);
}

CMGAN_API int cmgan_enhance_sr(const float* params, const float* wav, long long ldw, int B, int L, const int* lengths, int sr, int cut_len, float* out,
                               long long ldo, void* workspace, long long workspace_bytes, int precision, void* stream) {
    if (sr == SR_MODEL) return cmgan_enhance(params, wav, ldw, B, L, lengths, cut_len, out, ldo, workspace, workspace_bytes, precision, stream);
    const char* who = "cmgan_enhance_sr";
    CMGAN_REQUIRE(params && wav && out && workspace, "%s: null pointer", who);
    CMGAN_REQUIRE(precision == 0 || precision == 1, "%s: precision must be 0 (fp32) or 1 (tf32)", who);
    CMGAN_REQUIRE((((uintptr_t)params) & 15) == 0 && (((uintptr_t)workspace) & 255) == 0, "%s: params must be 16-byte, workspace 256-byte aligned", who);
    resample::Ratio q;
    long long L16;
    EnhanceGeom g;
    if (sr_geom(sr, L, INT32_MAX, q, L16, who) != 0 || enhance_geom(B, (int)L16, cut_len, lengths != nullptr, false, g, who) != 0) return -1;
    CMGAN_REQUIRE(ldw >= L && ldo >= L, "%s: row strides must cover a clip (L=%d ldw=%lld ldo=%lld)", who, L, ldw, ldo);
    const uintptr_t w0 = (uintptr_t)wav, w1 = (uintptr_t)(wav + (B - 1) * ldw + L), o0 = (uintptr_t)out, o1 = (uintptr_t)(out + (B - 1) * ldo + L);
    CMGAN_REQUIRE(w1 <= o0 || o1 <= w0, "%s: wav and out overlap", who);
    SrRegion s;
    const size_t region = sr_region(nullptr, q, B, L16, s);
    const long long need = (long long)region + enhance_bytes(B, (int)L16, g, precision);
    CMGAN_REQUIRE(workspace_bytes >= need, "%s: workspace too small (%lld bytes needed, %lld given)", who, need, workspace_bytes);
    sr_region(static_cast<char*>(workspace), q, B, L16, s);
    const cudaStream_t st = (cudaStream_t)stream;
    int* len16 = lengths ? s.len16 : nullptr;
    if (cmgan_resample_taps(sr, SR_MODEL, s.h_in, stream) != 0 || cmgan_resample_taps(SR_MODEL, sr, s.h_out, stream) != 0) return -1;
    if (resample::launch<float>(wav, ldw, B, L, lengths, q.up, q.down, q.half, s.h_in, s.x16, L16, L16, nullptr, len16, st) != 0) return -1;
    if (cmgan_enhance(params, s.x16, L16, B, (int)L16, len16, cut_len, s.y16, L16, static_cast<char*>(workspace) + region,
                      workspace_bytes - (long long)region, precision, stream) != 0)
        return -1;
    return resample::launch<float>(s.y16, L16, B, L16, len16, q.down, q.up, q.half, s.h_out, out, ldo, L, lengths, nullptr, st);
}

// ==================================================================================== one long clip, overlapping windows joined by a crossfade
// The pass workspace of cmgan_enhance_overlap at 16 kHz: one pass of max_segments windows of S_max samples plus the crossfade table and the
// staging rows, and never less than cmgan_enhance_long's (the one-window case runs that entry).  Independent of L.
static long long overlap_bytes(int cut_len, int overlap, int max_segments, int precision, const char* who) {
    const long long base = enhance_long_bytes(cut_len, max_segments, precision, who);
    if (base < 0) return -1;
    EnhanceGeom g;
    int h;
    if (overlap_geom(1 << 30, cut_len, overlap, g, h, who) != 0) return -1;          // a clip long enough for windows of S_max samples
    g.rows = g.pass = max_segments;
    const Crossfade xf{overlap, h};
    Run r;
    r.P = nullptr; r.ws = nullptr; r.dry = true; r.precision = precision; r.st = nullptr;
    enhance_walk(r, nullptr, g.S, 1, g.S, nullptr, g, nullptr, g.S, &xf);
    return std::max(base, (long long)r.peak + 256);
}

// cmgan_enhance_overlap at 16 kHz, overlap > 0; every check before the first launch
static int enhance_overlap16(const float* params, const float* wav, long long L, int cut_len, int overlap, int max_segments, float* out,
                             void* workspace, long long workspace_bytes, int precision, void* stream, const char* who) {
    CMGAN_REQUIRE(params && wav && out && workspace, "%s: null pointer", who);
    CMGAN_REQUIRE((((uintptr_t)params) & 15) == 0 && (((uintptr_t)workspace) & 255) == 0, "%s: params must be 16-byte, workspace 256-byte aligned", who);
    CMGAN_REQUIRE(L <= (1 << 30), "%s: L=%lld samples; at most 2^30 (18.6 hours at 16 kHz) keeps every sample index in 32 bits", who, L);
    const long long need = overlap_bytes(cut_len, overlap, max_segments, precision, who);
    if (need < 0) return -1;
    EnhanceGeom g;
    int h;
    if (overlap_geom((int)std::max(L, 0LL), cut_len, overlap, g, h, who) != 0) return -1;
    const uintptr_t w0 = (uintptr_t)wav, w1 = (uintptr_t)(wav + L), o0 = (uintptr_t)out, o1 = (uintptr_t)(out + L);
    CMGAN_REQUIRE(w1 <= o0 || o1 <= w0, "%s: wav and out overlap", who);
    CMGAN_REQUIRE(workspace_bytes >= need, "%s: workspace too small (%lld bytes needed, %lld given)", who, need, workspace_bytes);
    if (g.k == 1)           // one window: the one-segment case of the long entry, the same launches
        return cmgan_enhance_long(params, wav, (int)L, cut_len, max_segments, out, workspace, workspace_bytes, precision, stream);
    g.pass = std::min(max_segments, g.k);
    const Crossfade xf{overlap, h};
    cmgan_set_tf32_rounding(precision);       // as cmgan_tscnet_fwd: producers of tensor-core operands round to nearest on store
    Run r;
    r.P = params; r.ws = static_cast<char*>(workspace); r.cap = (size_t)workspace_bytes; r.dry = false; r.precision = precision;
    r.st = (cudaStream_t)stream; r.who = who;
    enhance_walk(r, wav, L, 1, (int)L, nullptr, g, out, L, &xf);
    return r.rc;
}

// One clip at sr: resample to 16 kHz into the workspace, the 16 kHz long walk (overlap 0: cmgan_enhance_long's fold, else the crossfaded
// windows) on the rest of it, resample back.  sr = 16000 is the 16 kHz walk itself.
static long long long_sr_bytes(long long L, int sr, int cut_len, int overlap, int max_segments, int precision, const char* who) {
    resample::Ratio q;
    long long L16 = L;
    if (sr != SR_MODEL && sr_geom(sr, L, 1ll << 30, q, L16, who) != 0) return -1;
    const long long walk = overlap == 0 ? enhance_long_bytes(cut_len, max_segments, precision, who)
                                        : overlap_bytes(cut_len, overlap, max_segments, precision, who);
    if (walk < 0 || sr == SR_MODEL) return walk;
    SrRegion s;
    return (long long)sr_region(nullptr, q, 1, L16, s) + walk;
}

static int enhance_long_sr(const float* params, const float* wav, long long L, int sr, int cut_len, int overlap, int max_segments, float* out,
                           void* workspace, long long workspace_bytes, int precision, void* stream, const char* who) {
    if (sr == SR_MODEL) {
        if (overlap != 0)
            return enhance_overlap16(params, wav, L, cut_len, overlap, max_segments, out, workspace, workspace_bytes, precision, stream, who);
        CMGAN_REQUIRE(L >= 0 && L <= (1ll << 30), "%s: L=%lld samples; at most 2^30 (18.6 hours at 16 kHz) keeps every sample index in 32 bits", who, L);
        return cmgan_enhance_long(params, wav, (int)L, cut_len, max_segments, out, workspace, workspace_bytes, precision, stream);
    }
    CMGAN_REQUIRE(params && wav && out && workspace, "%s: null pointer", who);
    CMGAN_REQUIRE((((uintptr_t)params) & 15) == 0 && (((uintptr_t)workspace) & 255) == 0, "%s: params must be 16-byte, workspace 256-byte aligned", who);
    resample::Ratio q;
    long long L16;
    if (sr_geom(sr, L, 1ll << 30, q, L16, who) != 0) return -1;
    const long long walk = overlap == 0 ? enhance_long_bytes(cut_len, max_segments, precision, who)
                                        : overlap_bytes(cut_len, overlap, max_segments, precision, who);
    if (walk < 0) return -1;
    EnhanceGeom g;
    int h;
    if ((overlap == 0 ? enhance_geom(1, (int)L16, cut_len, false, true, g, who) : overlap_geom((int)L16, cut_len, overlap, g, h, who)) != 0)
        return -1;
    const uintptr_t w0 = (uintptr_t)wav, w1 = (uintptr_t)(wav + L), o0 = (uintptr_t)out, o1 = (uintptr_t)(out + L);
    CMGAN_REQUIRE(w1 <= o0 || o1 <= w0, "%s: wav and out overlap", who);
    SrRegion s;
    const size_t region = sr_region(nullptr, q, 1, L16, s);
    const long long need = (long long)region + walk;
    CMGAN_REQUIRE(workspace_bytes >= need, "%s: workspace too small (%lld bytes needed, %lld given)", who, need, workspace_bytes);
    sr_region(static_cast<char*>(workspace), q, 1, L16, s);
    const cudaStream_t st = (cudaStream_t)stream;
    if (cmgan_resample_taps(sr, SR_MODEL, s.h_in, stream) != 0 || cmgan_resample_taps(SR_MODEL, sr, s.h_out, stream) != 0) return -1;
    if (resample::launch<float>(wav, L, 1, L, nullptr, q.up, q.down, q.half, s.h_in, s.x16, L16, L16, nullptr, nullptr, st) != 0) return -1;
    char* ws16 = static_cast<char*>(workspace) + region;
    const long long bytes16 = workspace_bytes - (long long)region;
    if ((overlap == 0 ? cmgan_enhance_long(params, s.x16, (int)L16, cut_len, max_segments, s.y16, ws16, bytes16, precision, stream)
                      : enhance_overlap16(params, s.x16, L16, cut_len, overlap, max_segments, s.y16, ws16, bytes16, precision, stream, who)) != 0)
        return -1;
    return resample::launch<float>(s.y16, L16, 1, L16, nullptr, q.down, q.up, q.half, s.h_out, out, L, L, nullptr, nullptr, st);
}

CMGAN_API long long cmgan_enhance_long_sr_workspace_bytes(long long L, int sr, int cut_len, int max_segments, int precision) {
    if (sr == SR_MODEL) return cmgan_enhance_long_workspace_bytes(cut_len, max_segments, precision);
    return long_sr_bytes(L, sr, cut_len, 0, max_segments, precision, "cmgan_enhance_long_sr_workspace_bytes");
}

CMGAN_API int cmgan_enhance_long_sr(const float* params, const float* wav, long long L, int sr, int cut_len, int max_segments, float* out,
                                    void* workspace, long long workspace_bytes, int precision, void* stream) {
    return enhance_long_sr(params, wav, L, sr, cut_len, 0, max_segments, out, workspace, workspace_bytes, precision, stream, "cmgan_enhance_long_sr");
}

CMGAN_API long long cmgan_enhance_overlap_workspace_bytes(long long L, int sr, int cut_len, int overlap, int max_segments, int precision) {
    const char* who = "cmgan_enhance_overlap_workspace_bytes";
    CMGAN_REQUIRE(overlap >= 0, "%s: overlap=%d must be 0 (the fold of cmgan_enhance_long) or a positive multiple of 100", who, overlap);
    if (overlap == 0) return cmgan_enhance_long_sr_workspace_bytes(L, sr, cut_len, max_segments, precision);
    return long_sr_bytes(L, sr, cut_len, overlap, max_segments, precision, who);
}

CMGAN_API int cmgan_enhance_overlap(const float* params, const float* wav, long long L, int sr, int cut_len, int overlap, int max_segments, float* out,
                                    void* workspace, long long workspace_bytes, int precision, void* stream) {
    const char* who = "cmgan_enhance_overlap";
    CMGAN_REQUIRE(overlap >= 0, "%s: overlap=%d must be 0 (the fold of cmgan_enhance_long) or a positive multiple of 100", who, overlap);
    if (overlap == 0) return cmgan_enhance_long_sr(params, wav, L, sr, cut_len, max_segments, out, workspace, workspace_bytes, precision, stream);
    return enhance_long_sr(params, wav, L, sr, cut_len, overlap, max_segments, out, workspace, workspace_bytes, precision, stream, who);
}

// ==================================================================================== training: train-mode (or saving eval-mode) forward, backward
// Workspace of a training call: the saved region (what the backward reads, fixed by the shape), then the scratch of whichever call runs --
// the forward's or the backward's, which starts with a parameter-gradient stand-in for frozen weights.  Both walks derive the saved layout
// from the same forward walk, so the backward finds every saved activation where the forward left it.
struct TrainLayout { size_t keep, fwd, bwd; };

static TrainLayout train_layout(int B, int T, int F, int precision, bool training) {
    Saved sv;
    Run f;
    f.P = nullptr; f.ws = nullptr; f.dry = true; f.precision = precision; f.st = nullptr; f.sv = &sv; f.saving = true; f.training = training;
    forward(f, nullptr, 0, 0, 0, 0, B, T, F, nullptr, nullptr);
    Run b;
    b.P = nullptr; b.ws = nullptr; b.dry = true; b.precision = precision; b.st = nullptr; b.training = training;
    b.alloc((size_t)table().total);
    backward(b, sv, nullptr, 0, 0, 0, 0, B, T, F, nullptr, nullptr, 0, 0, 0, nullptr);
    return {(f.ktop + 255) & ~(size_t)255, f.peak, b.peak};
}

CMGAN_API long long cmgan_tscnet_train_workspace_bytes(int B, int T, int F, int precision) {
    if (B <= 0 || T <= 0 || F != NFEAT || (precision != 0 && precision != 1)) {
        cmgan_set_error("cmgan_tscnet_train_workspace_bytes: bad arguments (B=%d T=%d F=%d precision=%d; F must be %d, precision 0 or 1)", B, T, F,
                        precision, NFEAT);
        return -1;
    }
    if ((long long)B * T * F * CAT >= (1ll << 31)) {
        cmgan_set_error("cmgan_tscnet_train_workspace_bytes: B * T * F * %d = %lld elements reach 2^31 (32-bit indexing of the encoder concat buffer); "
                        "split the batch", CAT, (long long)B * T * F * CAT);
        return -1;
    }
    const TrainLayout L = train_layout(B, T, F, precision, true);      // eval mode keeps the same buffers and needs less statistics scratch
    return (long long)(L.keep + std::max(L.fwd, L.bwd)) + 256;
}

// checks shared by both training entries; on success `r` is set up for the walk (saved region at the workspace base, scratch above it)
static int train_setup(Run& r, Saved& sv, const char* who, const float* params, const float* x, int B, int T, int F, int training,
                       unsigned long long seed, const unsigned long long* seed_dev, void* workspace, long long workspace_bytes, int precision, void* stream) {
    CMGAN_REQUIRE(params && x && workspace, "%s: null pointer", who);
    CMGAN_REQUIRE(B > 0 && T > 0 && F == NFEAT, "%s: expected x of shape (B, 2, T, %d), got B=%d T=%d F=%d", who, NFEAT, B, T, F);
    CMGAN_REQUIRE(precision == 0 || precision == 1, "%s: precision must be 0 (fp32) or 1 (tf32)", who);
    CMGAN_REQUIRE(training == 0 || training == 1, "%s: training must be 0 (eval) or 1 (train)", who);
    CMGAN_REQUIRE((((uintptr_t)params) & 15) == 0 && (((uintptr_t)workspace) & 255) == 0, "%s: params must be 16-byte, workspace 256-byte aligned", who);
    CMGAN_REQUIRE((long long)B * T * F * CAT < (1ll << 31),
                  "%s: B * T * F * %d = %lld elements reach 2^31 (32-bit indexing of the encoder concat buffer); split the batch", who, CAT,
                  (long long)B * T * F * CAT);
    const long long need = cmgan_tscnet_train_workspace_bytes(B, T, F, precision);
    CMGAN_REQUIRE(workspace_bytes >= need, "%s: workspace too small (%lld bytes needed, %lld given)", who, need, workspace_bytes);
    const TrainLayout L = train_layout(B, T, F, precision, training == 1);
    cmgan_set_tf32_rounding(precision);       // as cmgan_tscnet_fwd: producers of tensor-core operands round to nearest on store
    r.P = params; r.dry = false; r.precision = precision; r.st = (cudaStream_t)stream;
    r.sv = &sv; r.saving = true; r.kws = static_cast<char*>(workspace);
    r.ws = r.kws + L.keep; r.cap = (size_t)workspace_bytes - L.keep;
    r.training = training == 1; r.seed = seed; r.seed_dev = seed_dev;
    return 0;
}

// the backward call's first half: a forward walk that launches nothing and only places the saved activations where the forward call left them
static int place_saved(Run& r, const float* x, long long sxb, long long sxc, long long sxt, long long sxf, int B, int T, int F) {
    r.quiet = true;
    forward(r, x, sxb, sxc, sxt, sxf, B, T, F, nullptr, nullptr);
    r.quiet = false;
    r.top = r.peak = 0;
    return r.rc;
}

// the backward walk from the scratch position `r` is at; grads null = frozen weights
static void backward_pass(Run& r, const Saved& sv, const float* x, long long sxb, long long sxc, long long sxt, long long sxf, int B, int T, int F,
                          const float* dfr, const float* dfi, long long sgb, long long sgt, long long sgf, float* grads, float* dx) {
    float* gscratch = r.alloc((size_t)table().total);       // frozen weights: the gradient atomics fused into the data-gradient kernels land here
    r.G = grads ? grads : gscratch;
    r.wgrad = grads != nullptr;
    backward(r, sv, x, sxb, sxc, sxt, sxf, B, T, F, dfr, dfi, sgb, sgt, sgf, dx);
}

CMGAN_API int cmgan_tscnet_fwd_train(float* params, const float* x, long long sxb, long long sxc, long long sxt, long long sxf, int B, int T, int F,
                                     int training, unsigned long long seed, const unsigned long long* seed_dev, float* final_real, float* final_imag,
                                     void* workspace, long long workspace_bytes, int precision, void* stream) {
    const char* who = "cmgan_tscnet_fwd_train";
    CMGAN_REQUIRE(final_real && final_imag, "%s: null pointer", who);
    Run r;
    Saved sv;
    if (train_setup(r, sv, who, params, x, B, T, F, training, seed, seed_dev, workspace, workspace_bytes, precision, stream) != 0) return -1;
    forward(r, x, sxb, sxc, sxt, sxf, B, T, F, final_real, final_imag);
    return r.rc;
}

CMGAN_API int cmgan_tscnet_bwd(const float* params, const float* x, long long sxb, long long sxc, long long sxt, long long sxf, int B, int T, int F,
                               int training, unsigned long long seed, const unsigned long long* seed_dev, const float* dfr, const float* dfi, long long sgb,
                               long long sgt, long long sgf, float* grads, float* dx, void* workspace, long long workspace_bytes, int precision,
                               void* stream) {
    const char* who = "cmgan_tscnet_bwd";
    CMGAN_REQUIRE(grads || dx, "%s: grads and dx are both null: nothing to compute", who);
    CMGAN_REQUIRE((((uintptr_t)grads) & 15) == 0, "%s: grads must be 16-byte aligned", who);
    CMGAN_REQUIRE(sgb >= 0 && sgt >= 0 && sgf >= 0, "%s: gradient strides must be non-negative", who);
    CMGAN_REQUIRE((dfr && dfi) || (long long)(B - 1) * sgb + (long long)(T - 1) * sgt + (long long)(F - 1) * sgf < (long long)B * T * F,
                  "%s: a null dfr / dfi stands for zeros laid out with the strides of the other; those strides span more than B * T * F elements", who);
    Run r;
    Saved sv;
    if (train_setup(r, sv, who, params, x, B, T, F, training, seed, seed_dev, workspace, workspace_bytes, precision, stream) != 0) return -1;
    if (place_saved(r, x, sxb, sxc, sxt, sxf, B, T, F) != 0) return r.rc;
    backward_pass(r, sv, x, sxb, sxc, sxt, sxf, B, T, F, dfr, dfi, sgb, sgt, sgf, grads, dx);
    return r.rc;
}

// ==================================================================================== training from waveforms (train.py:72-151)
// The launch sequence of FusedTrainer.generator_step around the TSCNet pair: RMS scale, the STFT front end of both batches, the TSCNet
// forward, the inverse STFT, the spectral and time-domain losses; then the magnitude term's gradient, the inverse STFT's backward and the
// TSCNet backward.  Workspace: the waveform region first, then TSCNet's training layout (saved region, scratch).  The front end and the
// inverse STFT (and its backward) take their scratch from TSCNet's scratch area: nothing of TSCNet's is live there at those points.
namespace {

// what the waveform ends keep across the TSCNet forward or for the backward: the STFT tables, the RMS scales, both compressed spectrograms
// (the noisy one is TSCNet's x), fr / fi, the spectral-loss gradients and the time-loss gradient d_audio (B, Lo)
struct WaveKeep { float *fwd, *inv, *env, *c, *xn, *xc, *fr, *fi, *der, *dei, *dau; };

// places the region at k's base (k.dry: sizes it only); returns its size rounded up to 256 bytes
size_t wave_keep(Run& k, int B, int T, WaveKeep& w) {
    const size_t MT = (size_t)B * T, F = NFEAT;
    w.fwd = k.alloc((size_t)NFFT * 2 * F);
    w.inv = k.alloc((size_t)2 * F * NFFT);
    w.env = k.alloc((size_t)HOP * (T - 1));
    w.c = k.alloc(B);
    w.xn = k.alloc(MT * 2 * F);
    w.xc = k.alloc(MT * 2 * F);
    w.fr = k.alloc(MT * F);
    w.fi = k.alloc(MT * F);
    w.der = k.alloc(MT * F);
    w.dei = k.alloc(MT * F);
    w.dau = k.alloc((size_t)B * HOP * (T - 1));
    return (k.top + 255) & ~(size_t)255;
}

struct WaveArgs {
    const float *clean, *noisy;
    long long ldc, ldn;
    float w_ri, w_mag, w_t;
    float *est_audio, *est_mag, *clean_mag;
    long long lde;
    double* acc;
};

void gen_wave_fwd_walk(Run& r, const WaveKeep& w, int B, int L, const WaveArgs& a) {
    const int T = L / HOP + 1, F = NFEAT, Lo = HOP * (T - 1), Lp = (L + NFFT + HOP - 1) / HOP * HOP;
    const long long MT = (long long)B * T, TF = (long long)T * F;
    if (r.live()) r.ok(cmgan_stft_tables(w.fwd, w.inv, T, w.env, nullptr, r.st));
    if (r.live()) r.ok(cmgan_rms_scale(a.noisy, a.ldn, B, L, w.c, r.st));
    // signal.stft_compress of the noisy batch, then of the clean batch, both scaled by the noisy batch's c (train.py:75-79); exact fp32 DFTs
    const float* src[2] = {a.noisy, a.clean};
    const long long lds[2] = {a.ldn, a.ldc};
    float* dst[2] = {w.xn, w.xc};
    const size_t mark = r.top;
    for (int i = 0; i < 2; ++i) {
        float* xp = r.alloc((size_t)B * Lp);
        float* S = r.alloc((size_t)MT * 2 * F);
        if (r.live()) r.ok(cmgan_pad_reflect(src[i], lds[i], B, L, w.c, xp, Lp, r.st));
        Gemm(xp, HOP, w.fwd, 0, 2 * F, 1, nullptr, S, 2 * F, MT, 2 * F, NFFT).conv(1, T, 1, Lp / HOP).precision(0).run(r);
        if (r.live()) r.ok(cmgan_compress(S, B, T, dst[i], r.st));
        r.top = mark;
    }
    forward(r, w.xn, 2 * TF, TF, F, 1, B, T, F, w.fr, w.fi);
    r.top = mark;
    // signal.uncompress_istft_fwd without de-normalisation: est_audio stays at the RMS-scaled level (train.py:106-112)
    float* U = r.alloc((size_t)MT * 2 * F);
    float* frames = r.alloc((size_t)MT * NFFT);
    float* ea = r.alloc((size_t)B * Lo);
    if (r.live()) r.ok(cmgan_uncompress(w.fr, w.fi, TF, F, 1, B, T, U, r.st));
    Gemm(U, 2 * F, w.inv, 0, NFFT, 1, nullptr, frames, NFFT, MT, NFFT, 2 * F).precision(0).run(r);
    if (r.live()) r.ok(cmgan_ola(frames, B, T, w.env, nullptr, ea, Lo, r.st));
    r.zero(a.acc, 3 * sizeof(double));
    if (r.live())
        r.ok(cmgan_spec_loss(w.fr, w.fi, w.xc, w.xc + TF, TF, 2 * TF, MT * F, a.w_ri, a.w_mag, a.acc, w.der, w.dei, a.est_mag, a.clean_mag, r.st));
    // against the un-scaled clean batch, as the reference's train_step stores it (train.py:188)
    if (r.live()) r.ok(cmgan_time_loss(ea, Lo, a.clean, a.ldc, B, Lo, a.w_t, a.acc, w.dau, r.st));
    if (r.live()) {          // d_audio keeps the row stride Lo whatever lde is: est_audio leaves the workspace by one 2-D copy
        const cudaError_t e = cudaMemcpy2DAsync(a.est_audio, (size_t)a.lde * 4, ea, (size_t)Lo * 4, (size_t)Lo * 4, B, cudaMemcpyDeviceToDevice, r.st);
        if (e != cudaSuccess) { cmgan_set_error("%s: cudaMemcpy2DAsync: %s", r.who, cudaGetErrorString(e)); r.rc = -1; }
    }
    r.top = mark;
}

// d_mag (B, 1, F, T) with element strides (sgb, sgt, sgf), or null
void gen_wave_bwd_walk(Run& r, const Saved& sv, const WaveKeep& w, int B, int T, const float* d_mag, long long sgb, long long sgt, long long sgf,
                       float* grads) {
    const int F = NFEAT, Lo = HOP * (T - 1);
    const long long MT = (long long)B * T, TF = (long long)T * F;
    if (d_mag && r.live()) r.ok(cmgan_mag_bwd_add(w.fr, w.fi, d_mag, sgb, sgt, sgf, B, T, F, w.der, w.dei, r.st));
    // signal.uncompress_istft_bwd, accumulated into the spectral-loss gradients
    const size_t mark = r.top;
    float* dframes = r.alloc((size_t)MT * NFFT);
    float* dU = r.alloc((size_t)MT * 2 * F);
    if (r.live()) r.ok(cmgan_ola_bwd(w.dau, Lo, B, T, w.env, dframes, r.st));
    Gemm(dframes, NFFT, w.inv, 0, 1, NFFT, nullptr, dU, 2 * F, MT, 2 * F, NFFT).precision(0).run(r);
    if (r.live()) r.ok(cmgan_uncompress_bwd(w.fr, w.fi, TF, F, 1, B, T, dU, w.der, w.dei, 1, r.st));
    r.top = mark;
    backward_pass(r, sv, w.xn, 2 * TF, TF, F, 1, B, T, F, w.der, w.dei, TF, F, 1, grads, nullptr);
}

struct WaveLayout { size_t wave; TrainLayout t; };

// an exact dry run of both walks
WaveLayout wave_layout(int B, int L, int precision, bool training) {
    const int T = L / HOP + 1;
    WaveKeep w;
    Run k;
    const size_t wave = wave_keep(k, B, T, w);
    Saved sv;
    Run f;
    f.P = nullptr; f.ws = nullptr; f.dry = true; f.precision = precision; f.st = nullptr; f.sv = &sv; f.saving = true; f.training = training;
    WaveArgs a{};
    a.lde = a.ldc = a.ldn = L;
    gen_wave_fwd_walk(f, w, B, L, a);
    Run b;
    b.P = nullptr; b.ws = nullptr; b.dry = true; b.precision = precision; b.st = nullptr; b.training = training;
    gen_wave_bwd_walk(b, sv, w, B, T, nullptr, 0, 0, 0, nullptr);
    return {wave, {(f.ktop + 255) & ~(size_t)255, f.peak, b.peak}};
}

int wave_shape_check(const char* who, int B, int L, int precision) {
    CMGAN_REQUIRE(B > 0, "%s: B must be positive (B=%d)", who, B);
    CMGAN_REQUIRE(L > NFFT / 2, "%s: L=%d samples; a clip needs more than the 200-sample reflect padding of the STFT", who, L);
    CMGAN_REQUIRE(precision == 0 || precision == 1, "%s: precision must be 0 (fp32) or 1 (tf32)", who);
    const long long T = L / HOP + 1, elems = (long long)B * T * NFEAT * CAT;
    CMGAN_REQUIRE(elems < (1ll << 31), "%s: B * T * 201 * %d = %lld elements reach 2^31 (32-bit indexing of the encoder concat buffer); split the "
                  "batch", who, CAT, elems);
    return 0;
}

long long wave_bytes(int B, int L, int precision) {
    const WaveLayout l = wave_layout(B, L, precision, true);      // eval mode keeps the same buffers and needs less statistics scratch
    return (long long)(l.wave + l.t.keep + std::max(l.t.fwd, l.t.bwd)) + 256;
}

// checks shared by both entries; on success `r` walks the workspace (waveform region `w`, TSCNet's saved region, scratch)
int wave_setup(Run& r, Saved& sv, WaveKeep& w, const char* who, const float* params, int B, int L, int training, unsigned long long seed,
               const unsigned long long* seed_dev, void* workspace, long long workspace_bytes, int precision, void* stream) {
    CMGAN_REQUIRE(params && workspace, "%s: null pointer", who);
    CMGAN_REQUIRE((((uintptr_t)params) & 15) == 0 && (((uintptr_t)workspace) & 255) == 0, "%s: params must be 16-byte, workspace 256-byte aligned", who);
    if (wave_shape_check(who, B, L, precision) != 0) return -1;
    CMGAN_REQUIRE(training == 0 || training == 1, "%s: training must be 0 (eval) or 1 (train)", who);
    const long long need = wave_bytes(B, L, precision);
    CMGAN_REQUIRE(workspace_bytes >= need, "%s: workspace too small (%lld bytes needed, %lld given)", who, need, workspace_bytes);
    const WaveLayout l = wave_layout(B, L, precision, training == 1);
    cmgan_set_tf32_rounding(precision);       // as cmgan_tscnet_fwd: producers of tensor-core operands round to nearest on store
    Run k;
    k.dry = false; k.ws = static_cast<char*>(workspace); k.cap = (size_t)workspace_bytes;
    wave_keep(k, B, L / HOP + 1, w);
    r.P = params; r.dry = false; r.precision = precision; r.st = (cudaStream_t)stream; r.who = who;
    r.sv = &sv; r.saving = true; r.kws = static_cast<char*>(workspace) + l.wave;
    r.ws = r.kws + l.t.keep; r.cap = (size_t)workspace_bytes - l.wave - l.t.keep;
    r.training = training == 1; r.seed = seed; r.seed_dev = seed_dev;
    return 0;
}

}  // namespace

CMGAN_API long long cmgan_gen_wave_workspace_bytes(int B, int L, int precision) {
    if (wave_shape_check("cmgan_gen_wave_workspace_bytes", B, L, precision) != 0) return -1;
    return wave_bytes(B, L, precision);
}

CMGAN_API int cmgan_gen_wave_fwd(float* params, const float* clean, long long ldc, const float* noisy, long long ldn, int B, int L, int training,
                                 unsigned long long seed, const unsigned long long* seed_dev, float w_ri, float w_mag, float w_t, float* est_audio,
                                 long long lde, float* est_mag, float* clean_mag, double* acc, void* workspace, long long workspace_bytes,
                                 int precision, void* stream) {
    const char* who = "cmgan_gen_wave_fwd";
    CMGAN_REQUIRE(clean && noisy && est_audio && est_mag && clean_mag && acc, "%s: null pointer", who);
    const int Lo = L / HOP * HOP;
    CMGAN_REQUIRE(ldc >= L && ldn >= L && lde >= Lo, "%s: row strides must cover a row (L=%d Lo=%d ldc=%lld ldn=%lld lde=%lld)", who, L, Lo, ldc, ldn,
                  lde);
    if (B > 0 && L > 0) {
        const uintptr_t e0 = (uintptr_t)est_audio, e1 = (uintptr_t)(est_audio + (B - 1) * lde + Lo);
        for (const auto& s : {std::make_pair(clean, ldc), std::make_pair(noisy, ldn)}) {
            const uintptr_t s0 = (uintptr_t)s.first, s1 = (uintptr_t)(s.first + (B - 1) * s.second + L);
            CMGAN_REQUIRE(e1 <= s0 || s1 <= e0, "%s: est_audio overlaps clean or noisy", who);
        }
    }
    Run r;
    Saved sv;
    WaveKeep w;
    if (wave_setup(r, sv, w, who, params, B, L, training, seed, seed_dev, workspace, workspace_bytes, precision, stream) != 0) return -1;
    WaveArgs a{clean, noisy, ldc, ldn, w_ri, w_mag, w_t, est_audio, est_mag, clean_mag, lde, acc};
    gen_wave_fwd_walk(r, w, B, L, a);
    return r.rc;
}

CMGAN_API int cmgan_gen_wave_bwd(const float* params, int B, int L, int training, unsigned long long seed, const unsigned long long* seed_dev,
                                 const float* d_mag, long long sgb, long long sgt, long long sgf, float* grads, void* workspace, long long workspace_bytes,
                                 int precision, void* stream) {
    const char* who = "cmgan_gen_wave_bwd";
    CMGAN_REQUIRE(grads, "%s: null pointer (grads)", who);
    CMGAN_REQUIRE((((uintptr_t)grads) & 15) == 0, "%s: grads must be 16-byte aligned", who);
    CMGAN_REQUIRE(sgb >= 0 && sgt >= 0 && sgf >= 0, "%s: d_mag strides must be non-negative", who);
    Run r;
    Saved sv;
    WaveKeep w;
    if (wave_setup(r, sv, w, who, params, B, L, training, seed, seed_dev, workspace, workspace_bytes, precision, stream) != 0) return -1;
    const int T = L / HOP + 1;
    const long long TF = (long long)T * NFEAT;
    if (place_saved(r, w.xn, 2 * TF, TF, NFEAT, 1, B, T, NFEAT) != 0) return r.rc;
    gen_wave_bwd_walk(r, sv, w, B, T, d_mag, sgb, sgt, sgf, grads);
    return r.rc;
}
