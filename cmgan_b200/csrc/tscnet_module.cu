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
#include <cstring>
#include <string>
#include <unordered_map>
#include <vector>

#include "common.cuh"
#include "frontend.cuh"
#include "../../include/cmgan_b200.h"

namespace {

constexpr int C = 64, CAT = 320, NFEAT = 201;

struct Entry { std::string key; long long off, numel; };

struct Table {
    std::vector<Entry> e;
    long long total = 0;
    void add(const std::string& k, long long n) {
        e.push_back({k, total, n});
        total += (n + 3) / 4 * 4;
    }
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
const std::unordered_map<std::string, long long>& offsets() {
    static const std::unordered_map<std::string, long long> m = [] {
        std::unordered_map<std::string, long long> o;
        for (const Entry& e : table().e) o.emplace(e.key, e.off);
        return o;
    }();
    return m;
}

// ---- one forward pass = a walk over the launch list; `dry` only sizes the workspace
struct Run {
    const float* P;             // parameter block (null in a dry run)
    char* ws;                   // workspace base
    size_t top = 0, peak = 0, cap = 0;
    bool dry;
    int precision;
    cudaStream_t st;
    const int* frames = nullptr;      // ragged batch: valid frames per utterance (device); null = every utterance fills the grid
    int rc = 0;

    const float* w(const std::string& key) const {
        if (dry) return nullptr;
        const auto it = offsets().find(key);
        if (it != offsets().end()) return P + it->second;
        cmgan_set_error("cmgan_tscnet_fwd: unknown parameter %s", key.c_str());
        const_cast<Run*>(this)->rc = -1;
        return nullptr;
    }
    template <typename T = float>
    T* alloc(size_t n) {
        top = (top + 255) & ~(size_t)255;
        T* p = dry ? nullptr : reinterpret_cast<T*>(ws + top);
        top += n * sizeof(T);
        if (top > peak) peak = top;
        if (!dry && top > cap && rc == 0) { cmgan_set_error("cmgan_tscnet_fwd: workspace too small (%zu bytes needed so far, %zu given)", top, cap); rc = -1; }
        return p;
    }
    void ok(int r) { if (r != 0 && rc == 0) rc = r; }
    bool live() const { return !dry && rc == 0; }
};

struct Tabs { float *scale, *shift, *mean, *rstd; int width; };
Tabs make_tabs(Run& r, int G, int width) {
    Tabs t;
    t.scale = r.alloc((size_t)G * width); t.shift = r.alloc((size_t)G * width);
    t.mean = r.alloc((size_t)G * width); t.rstd = r.alloc((size_t)G * width);
    t.width = width;
    return t;
}

struct Gemm {
    CmganGemmArgs a;
    Gemm(const float* A, long long lda, const float* W, long long sb_tap, long long sb_k, long long sb_n, const float* bias, float* Cout,
         long long ldc, long long M, int N, int Cin) {
        memset(&a, 0, sizeof(a));
        a.A = A; a.lda = lda; a.B = W; a.sb_tap = sb_tap; a.sb_k = sb_k; a.sb_n = sb_n; a.bias = bias; a.C = Cout; a.ldc = ldc;
        a.M = (int)M; a.N = N; a.Cin = Cin; a.ntaps = 1;
        a.mul_y = a.mul_x = a.div_y = a.div_x = 1;
        a.inv_keep = 1.f; a.pro_inv_keep = 1.f; a.alpha = 1.f; a.pro_alpha = 1.f;
    }
    Gemm& conv(int OH, int OW, int IH, int IW, int mul_x = 1) {
        a.conv = 1; a.OH = OH; a.OW = OW; a.IH = IH; a.IW = IW; a.mul_x = mul_x;
        return *this;
    }
    Gemm& taps(int n, const int* dy, const int* dx) {
        a.ntaps = n;
        for (int i = 0; i < n; ++i) { a.dy[i] = dy[i]; a.dx[i] = dx[i]; }
        return *this;
    }
    Gemm& residual(const float* R, long long ldr) { a.epi = CMGAN_EPI_DROP_RES; a.R = R; a.ldr = ldr; return *this; }
    void run(Run& r) {
        a.precision = r.precision;
        if (r.precision == 1 && a.N % 16 == 0 && a.N <= 256 && a.Cin % 32 == 0) {      // scratch for the re-tiled weight (gemm_args.h)
            a.ws_floats = (long long)a.N * a.Cin * a.ntaps;
            a.ws = r.alloc((size_t)a.ws_floats);
        }
        if (r.live()) r.ok(cmgan_gemm_rows_f32(&a, r.st));
    }
};

// rows_per_t: rows of one frame within a group (row = t * rows_per_t + f); a ragged batch normalises over the valid frames only
void inst_norm_site(Run& r, const float* x, long long ldx, int G, long long rows, long long rows_per_t, int Cn, const float* gamma, const float* beta,
                    const Tabs& t, double*& sums) {
    double* s = sums;
    sums += (size_t)G * Cn * 2;
    if (!r.live()) return;
    if (r.frames) {
        r.ok(cmgan_norm_stats_ragged(x, ldx, G, rows, Cn, rows_per_t, r.frames, s, r.st));
        r.ok(cmgan_norm_finalize_ragged(s, rows_per_t, (int)(rows / rows_per_t), r.frames, G, Cn, gamma, beta, t.scale, t.shift, t.mean, t.rstd,
                                        t.width, r.st));
        return;
    }
    r.ok(cmgan_norm_stats(x, ldx, G, rows, Cn, s, r.st));
    r.ok(cmgan_norm_finalize(s, rows, G, Cn, 0, gamma, beta, nullptr, nullptr, 0.f, t.scale, t.shift, t.mean, t.rstd, t.width, r.st));
}

// InstanceNorm2d(affine) + PReLU of a raw (M, 64) tensor, written into dst (generator.py:35-37)
void norm_prelu_to(Run& r, const float* raw, int G, long long rows, long long rows_per_t, const float* gamma, const float* beta, const float* slope,
                   float* dst, long long ldd, double*& sums) {
    Tabs t = make_tabs(r, G, C);
    inst_norm_site(r, raw, C, G, rows, rows_per_t, C, gamma, beta, t, sums);
    if (r.live()) r.ok(cmgan_norm_apply(raw, C, G, rows, C, 1 | (r.precision == 1 ? 16 : 0), t.scale, t.shift, C, slope, dst, ldd, r.st));
}

// DilatedDenseNet (generator.py:39-47) on the concat buffer cat = [out4 | out3 | out2 | out1 | x]
void dense_block(Run& r, float* cat, const std::string& p, int B, int T, int Fw, double*& sums) {
    const long long M = (long long)B * T * Fw, rows = (long long)T * Fw;
    for (int i = 1; i <= 4; ++i) {
        const int dil = 1 << (i - 1), c0 = (5 - i) * C, Cin = C * i, co = (4 - i) * C;
        const std::string s = std::to_string(i);
        float* raw = r.alloc((size_t)M * C);
        const int dy[6] = {-dil, -dil, -dil, 0, 0, 0}, dx[6] = {-1, 0, 1, -1, 0, 1};         // tap = kh * 3 + kw, causal in time (generator.py:12-21)
        Gemm(cat ? cat + c0 : nullptr, CAT, r.w(p + "conv" + s + ".weight"), 1, 6, (long long)Cin * 6, r.w(p + "conv" + s + ".bias"), raw, C, M, C, Cin)
            .taps(6, dy, dx).conv(T, Fw, T, Fw).run(r);
        norm_prelu_to(r, raw, B, rows, Fw, r.w(p + "norm" + s + ".weight"), r.w(p + "norm" + s + ".bias"), r.w(p + "prelu" + s + ".weight"),
                      cat ? cat + co : nullptr, CAT, sums);
    }
}

// 0.5 * FF(LN(x)) + x  (conformer.py:54-72,136-148,211-212)
float* feed_forward(Run& r, const float* xin, long long M, const std::string& p) {
    float* out = r.alloc((size_t)M * C);
    if (r.precision == 1) {          // fused kernel: the hidden activation stays on the SM (ffn_fused.cu)
        float* w1p = r.alloc((size_t)4 * C * C);
        float* w2p = r.alloc((size_t)4 * C * C);
        if (r.live()) {
            r.ok(cmgan_pack_weight(r.w(p + "fn.fn.net.0.weight"), w1p, 0, 1, C, C, 1, 4 * C, r.st));
            r.ok(cmgan_pack_weight(r.w(p + "fn.fn.net.3.weight"), w2p, 0, 1, 4 * C, 4 * C, 1, C, r.st));
            r.ok(cmgan_ffn_fwd(xin, C, M, r.w(p + "fn.norm.weight"), r.w(p + "fn.norm.bias"), w1p, r.w(p + "fn.fn.net.0.bias"), w2p,
                               r.w(p + "fn.fn.net.3.bias"), 0.5f, 0ull, 0ull, 0u, 1.f, nullptr, out, C, r.st));
        }
        return out;
    }
    float* xn = r.alloc((size_t)M * C);
    float* stt = r.alloc((size_t)M * 2);
    float* a = r.alloc((size_t)M * 4 * C);
    if (r.live()) r.ok(cmgan_ln_apply(xin, C, M, r.w(p + "fn.norm.weight"), r.w(p + "fn.norm.bias"), nullptr, 0, xn, C, stt, r.precision == 1 ? 1 : 0, r.st));
    Gemm g1(xn, C, r.w(p + "fn.fn.net.0.weight"), 0, 1, C, r.w(p + "fn.fn.net.0.bias"), nullptr, 4 * C, M, 4 * C, C);
    g1.a.epi = CMGAN_EPI_SWISH_DUAL; g1.a.C2 = a; g1.a.ldc2 = 4 * C;
    g1.run(r);
    Gemm g2(a, 4 * C, r.w(p + "fn.fn.net.3.weight"), 0, 1, 4 * C, r.w(p + "fn.fn.net.3.bias"), out, C, M, C, 4 * C);
    g2.residual(xin, C).a.alpha = 0.5f;
    g2.run(r);
    return out;
}

// ConformerBlock + the outer TSCB residual (conformer.py:216-222, generator.py:95,97): returns LN(x4) + x in `y`
void conformer(Run& r, const float* x, float* y, const std::string& p, int B, int T, int F2, int axis) {
    const long long M = (long long)B * T * F2;
    const size_t mark = r.top;
    const int rnd = r.precision == 1 ? 1 : 0;
    float* x1 = feed_forward(r, x, M, p + "ff1.");
    // ---- attention (conformer.py:90-133)
    float* xn2 = r.alloc((size_t)M * C);
    float* st2 = r.alloc((size_t)M * 2);
    if (r.live()) r.ok(cmgan_ln_apply(x1, C, M, r.w(p + "attn.norm.weight"), r.w(p + "attn.norm.bias"), nullptr, 0, xn2, C, st2, rnd, r.st));
    float* qkv = r.alloc((size_t)M * 3 * C);
    // to_q and to_kv are adjacent in the parameter block: one (192, 64) projection
    Gemm(xn2, C, r.w(p + "attn.fn.to_q.weight"), 0, 1, C, nullptr, qkv, 3 * C, M, 3 * C, C).run(r);
    float* ctx = r.alloc((size_t)M * C);
    float* lse = r.alloc((size_t)M * 4);
    if (r.live()) {
        const float* E = r.w(p + "attn.fn.rel_pos_emb.weight");
        if (r.frames)
            r.ok(r.precision == 1 ? cmgan_attention_fwd_tf32_ragged(qkv, E, B, T, F2, axis, r.frames, ctx, lse, r.st)
                                  : cmgan_attention_fwd_ragged(qkv, E, B, T, F2, axis, r.frames, ctx, lse, r.st));
        else
            r.ok(r.precision == 1 ? cmgan_attention_fwd_tf32(qkv, E, B, T, F2, axis, ctx, lse, r.st) : cmgan_attention_fwd(qkv, E, B, T, F2, axis, ctx, lse, r.st));
    }
    float* x2 = r.alloc((size_t)M * C);
    Gemm(ctx, C, r.w(p + "attn.fn.to_out.weight"), 0, 1, C, r.w(p + "attn.fn.to_out.bias"), x2, C, M, C, C).residual(x1, C).run(r);
    // ---- convolution module (conformer.py:160-173)
    float* xn3 = r.alloc((size_t)M * C);
    float* st3 = r.alloc((size_t)M * 2);
    if (r.live()) r.ok(cmgan_ln_apply(x2, C, M, r.w(p + "conv.net.0.weight"), r.w(p + "conv.net.0.bias"), nullptr, 0, xn3, C, st3, rnd, r.st));
    float* g = r.alloc((size_t)M * 4 * C);
    Gemm(xn3, C, r.w(p + "conv.net.2.weight"), 0, 1, C, r.w(p + "conv.net.2.bias"), g, 4 * C, M, 4 * C, C).run(r);
    float* d = r.alloc((size_t)M * 2 * C);
    Tabs bn = make_tabs(r, 1, 2 * C);
    float* dsw = r.alloc((size_t)M * 2 * C);
    if (r.live()) {
        if (r.frames)
            r.ok(cmgan_glu_dwconv_fwd_ragged(g, r.w(p + "conv.net.4.conv.weight"), r.w(p + "conv.net.4.conv.bias"), B, T, F2, axis, r.frames, d, r.st));
        else
            r.ok(cmgan_glu_dwconv_fwd(g, r.w(p + "conv.net.4.conv.weight"), r.w(p + "conv.net.4.conv.bias"), B, T, F2, axis, d, nullptr, r.st));
        // eval: BatchNorm1d folds to scale / shift from the running statistics (mode 1; they are only read)
        r.ok(cmgan_norm_finalize(nullptr, M, 1, 2 * C, 1, r.w(p + "conv.net.5.weight"), r.w(p + "conv.net.5.bias"),
                                 const_cast<float*>(r.w(p + "conv.net.5.running_mean")), const_cast<float*>(r.w(p + "conv.net.5.running_var")), 0.1f,
                                 bn.scale, bn.shift, bn.mean, bn.rstd, 2 * C, r.st));
        r.ok(cmgan_norm_apply(d, 2 * C, 1, M, 2 * C, 2 | (16 * rnd), bn.scale, bn.shift, 2 * C, nullptr, dsw, 2 * C, r.st));
    }
    float* x3 = r.alloc((size_t)M * C);
    Gemm(dsw, 2 * C, r.w(p + "conv.net.7.weight"), 0, 1, 2 * C, r.w(p + "conv.net.7.bias"), x3, C, M, C, 2 * C).residual(x2, C).run(r);
    // ---- second feed-forward, post norm, outer residual
    float* x4 = feed_forward(r, x3, M, p + "ff2.");
    float* st5 = r.alloc((size_t)M * 2);
    if (r.live()) r.ok(cmgan_ln_apply(x4, C, M, r.w(p + "post_norm.weight"), r.w(p + "post_norm.bias"), x, C, y, C, st5, 0, r.st));
    r.top = mark;            // everything but `y` (owned by the caller) is released
}

void forward(Run& r, const float* x, long long sxb, long long sxc, long long sxt, long long sxf, int B, int T, int F, float* fr, float* fi) {
    const int F2 = (F - 1) / 2 + 1;
    const long long M = (long long)B * T * F, M2 = (long long)B * T * F2;
    const size_t n_sums = (size_t)(16 * C + 2) * B * 2 + 64;
    double* sums0 = r.alloc<double>(n_sums);
    double* sums = sums0;
    if (r.live()) {
        cudaError_t e = cudaMemsetAsync(sums0, 0, n_sums * sizeof(double), r.st);
        if (e != cudaSuccess) { cmgan_set_error("cmgan_tscnet_fwd: cudaMemsetAsync: %s", cudaGetErrorString(e)); r.rc = -1; }
    }
    float* hA = r.alloc((size_t)M2 * C);          // TSCB activations ping-pong between these two
    float* hB = r.alloc((size_t)M2 * C);
    // ---- dense encoder (generator.py:50-69)
    {
        const size_t mark = r.top;
        const std::string pe = "dense_encoder.";
        float* catE = r.alloc((size_t)M * CAT);
        float* raw0 = r.alloc((size_t)M * C);
        if (r.live()) r.ok(cmgan_head_conv(x, sxb, sxc, sxt, sxf, B, T, F, r.w(pe + "conv_1.0.weight"), r.w(pe + "conv_1.0.bias"), raw0, C, r.st));
        norm_prelu_to(r, raw0, B, (long long)T * F, F, r.w(pe + "conv_1.1.weight"), r.w(pe + "conv_1.1.bias"), r.w(pe + "conv_1.2.weight"),
                      catE ? catE + 4 * C : nullptr, CAT, sums);
        dense_block(r, catE, pe + "dilated_dense.", B, T, F, sums);
        float* e2 = r.alloc((size_t)M2 * C);
        const int dy[3] = {0, 0, 0}, dx[3] = {-1, 0, 1};
        Gemm(catE, CAT, r.w(pe + "conv_2.0.weight"), 1, 3, 3 * C, r.w(pe + "conv_2.0.bias"), e2, C, M2, C, C).taps(3, dy, dx).conv(T, F2, T, F, 2).run(r);
        Tabs t2 = make_tabs(r, B, C);
        inst_norm_site(r, e2, C, B, (long long)T * F2, F2, C, r.w(pe + "conv_2.1.weight"), r.w(pe + "conv_2.1.bias"), t2, sums);
        if (r.live()) r.ok(cmgan_norm_apply(e2, C, B, (long long)T * F2, C, 1, t2.scale, t2.shift, C, r.w(pe + "conv_2.2.weight"), hA, C, r.st));
        r.top = mark;
    }
    // ---- 4 x TSCB (generator.py:92-99): time conformer then frequency conformer on the same rows
    float *h = hA, *hn = hB;
    for (int i = 1; i <= 4; ++i)
        for (int axis = 0; axis < 2; ++axis) {
            conformer(r, h, hn, "TSCB_" + std::to_string(i) + (axis == 0 ? ".time_conformer." : ".freq_conformer."), B, T, F2, axis);
            float* t = h; h = hn; hn = t;
        }
    // ---- decoders (generator.py:122-156)
    float* sp[2];
    const char* names[2] = {"mask_decoder.", "complex_decoder."};
    for (int dd = 0; dd < 2; ++dd) {
        const std::string pd = names[dd];
        sp[dd] = r.alloc((size_t)M2 * 2 * C);          // (B, T, 2 F2, 64): the sub-pixel shuffle is a reinterpretation
        const size_t mark = r.top;
        float* cat = r.alloc((size_t)M2 * CAT);
        if (r.live()) r.ok(cmgan_copy_rows_operand(h, C, cat + 4 * C, CAT, M2, C, r.st));
        dense_block(r, cat, pd + "dense_block.", B, T, F2, sums);
        const int dy[3] = {0, 0, 0}, dx[3] = {-1, 0, 1};
        Gemm(cat, CAT, r.w(pd + "sub_pixel.conv.weight"), 1, 3, 3 * C, r.w(pd + "sub_pixel.conv.bias"), sp[dd], 2 * C, M2, 2 * C, C)
            .taps(3, dy, dx).conv(T, F2, T, F2).run(r);
        r.top = mark;
    }
    const std::string pm = "mask_decoder.", pc = "complex_decoder.";
    float* m1 = r.alloc((size_t)M);
    Tabs tabM = make_tabs(r, B, 1), tabC = make_tabs(r, B, C);
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

// ---- waveform in, waveform out (evaluation.py:21-53): the launch sequence of signal.enhance / enhance_ragged around forward()
constexpr int NFFT = 400, HOP = 100;

struct EnhanceGeom { int k, S, T, Lp, rows; };

// evaluation.py:25-34: wrap padding to padded = ceil(L / 100) * 100; past cut_len the clip is folded into k segments of S = padded / k
// samples, k = ceil(padded / cut_len) raised until it divides 100.  0, or -1 with the message set.
int enhance_geom(int B, int L, int cut_len, bool ragged, EnhanceGeom& g, const char* who) {
    CMGAN_REQUIRE(B > 0, "%s: B must be positive (B=%d)", who, B);
    CMGAN_REQUIRE(L > NFFT / 2, "%s: L=%d samples; a clip needs more than the 200-sample reflect padding of the STFT", who, L);
    CMGAN_REQUIRE(cut_len > 0, "%s: cut_len must be positive (cut_len=%d)", who, cut_len);
    const long long padded = ((long long)L + HOP - 1) / HOP * HOP;
    CMGAN_REQUIRE(padded - L <= L, "%s: wrap padding L=%d to %lld is longer than the clip", who, L, padded);
    long long k = 1;
    if (padded > cut_len) {
        CMGAN_REQUIRE(!ragged, "%s: a ragged batch needs ceil(L / 100) * 100 <= cut_len (L=%d, cut_len=%d); longer clips take the uniform call, "
                      "which folds them", who, L, cut_len);
        k = (padded + cut_len - 1) / cut_len;
        while (k <= HOP && HOP % k != 0) ++k;
        CMGAN_REQUIRE(k <= HOP, "%s: L=%d with cut_len=%d folds into more than 100 segments", who, L, cut_len);
    }
    g.k = (int)k;
    g.S = (int)(padded / k);
    CMGAN_REQUIRE(g.S > NFFT / 2, "%s: L=%d with cut_len=%d folds into %d segments of %d samples; a segment needs more than 200", who, L,
                  cut_len, g.k, g.S);
    g.T = g.S / HOP + 1;
    CMGAN_REQUIRE(k * HOP * (g.T - 1) >= L, "%s: L=%d with cut_len=%d folds into %d segments of %d samples, which yield only %lld samples", who,
                  L, cut_len, g.k, g.S, k * HOP * (g.T - 1));
    const long long elems = (long long)B * k * g.T * NFEAT * CAT;
    CMGAN_REQUIRE(elems < (1ll << 31), "%s: rows * T * 201 * %d = %lld elements reach 2^31 (32-bit indexing of the encoder concat buffer); split "
                  "the batch", who, CAT, elems);
    g.rows = (int)(B * k);
    g.Lp = (g.S + NFFT + HOP - 1) / HOP * HOP;
    return 0;
}

void enhance_walk(Run& r, const float* wav, long long ldw, int B, int L, const int* lengths, const EnhanceGeom& g, float* out, long long ldo) {
    const int T = g.T, rows = g.rows, F = NFEAT;
    const long long MT = (long long)rows * T;
    float* fwd = r.alloc((size_t)NFFT * 2 * F);
    float* inv = r.alloc((size_t)2 * F * NFFT);
    float* env = r.alloc((size_t)HOP * (T - 1));
    float* tail = r.alloc(HOP);
    float* c = r.alloc(B);
    int* tlen = r.alloc<int>(B);
    float* X = r.alloc((size_t)MT * 2 * F);
    float* fr = r.alloc((size_t)MT * F);
    float* fi = r.alloc((size_t)MT * F);
    if (r.live()) r.ok(cmgan_stft_tables(fwd, inv, T, env, tail, r.st));
    if (r.live()) r.ok(lengths ? cmgan_rms_scale_frames(wav, ldw, B, L, lengths, c, tlen, r.st) : cmgan_rms_scale(wav, ldw, B, L, c, r.st));
    const size_t mark = r.top;
    // ---- signal._stft_padded: wrap + reflect (+ fold) padding, framed DFT (exact fp32 FFMA), power compression
    {
        float* xp = r.alloc((size_t)rows * g.Lp);
        float* S = r.alloc((size_t)MT * 2 * F);
        if (r.live())
            r.ok(lengths ? cmgan_pad_wrap_reflect_ragged(wav, ldw, B, L, lengths, c, xp, g.Lp, r.st)
                         : cmgan_pad_wrap_reflect_fold(wav, ldw, B, L, g.k, c, xp, g.Lp, r.st));
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
    if (r.live())
        r.ok(lengths ? cmgan_ola_ragged_lengths(frames, B, T, tlen, lengths, L, env, tail, c, out, ldo, r.st)
                     : cmgan_ola_fold(frames, rows, T, g.k, env, c, out, ldo, L, r.st));
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
    if (enhance_geom(B, L, cut_len, false, g, "cmgan_enhance_workspace_bytes") != 0) return -1;
    return enhance_bytes(B, L, g, precision);
}

CMGAN_API int cmgan_enhance(const float* params, const float* wav, long long ldw, int B, int L, const int* lengths, int cut_len, float* out,
                            long long ldo, void* workspace, long long workspace_bytes, int precision, void* stream) {
    CMGAN_REQUIRE(params && wav && out && workspace, "cmgan_enhance: null pointer");
    CMGAN_REQUIRE(precision == 0 || precision == 1, "cmgan_enhance: precision must be 0 (fp32) or 1 (tf32)");
    CMGAN_REQUIRE((((uintptr_t)params) & 15) == 0 && (((uintptr_t)workspace) & 255) == 0, "cmgan_enhance: params must be 16-byte, workspace 256-byte aligned");
    EnhanceGeom g;
    if (enhance_geom(B, L, cut_len, lengths != nullptr, g, "cmgan_enhance") != 0) return -1;
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
