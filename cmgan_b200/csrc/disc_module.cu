// Module-level entry points of the metric discriminator (reference discriminator.py:29-64, ndf = 16 as train.py:55 builds it): the train-mode
// (or saving eval-mode) forward with one spectral-norm power iteration per weight, and its backward with parameter gradients through the
// spectral norm and input gradients, one C call each.  The launch sequence is the one cmgan_b200/discriminator.py (disc_fwd / disc_bwd) issues
// from Python with no side stream and no weight-pack cache: same kernels, same arguments, same order.
//
// Parameters: one flat fp32 block holding the 34 floating-point state_dict tensors of the reference Discriminator(16) in state_dict order
// (the spectral-norm triplets weight_orig / weight_u / weight_v included), each starting at a multiple of 4 floats.
#include <algorithm>
#include <string>

#include "common.cuh"
#include "module_walk.cuh"
#include "../../include/cmgan_b200.h"

namespace {

using namespace cmgan_walk;

constexpr int NDF = 16, NCONV = 4, MIN_HW = 16;
constexpr int CONV_IDX[NCONV] = {0, 3, 6, 9};
constexpr double P_DROP = 0.3;          // discriminator.py:55: Dropout(0.3) in front of PReLU(64)
unsigned drop_thr(bool on) { return on ? (unsigned)std::min(P_DROP * 4294967296.0, 4294967295.0) : 0u; }      // ops.drop_params
float drop_inv(bool on) { return on ? (float)(1.0 / (1.0 - P_DROP)) : 1.f; }
// the GEMMs count rows in 32-bit ints (CmganGemmArgs.M, the kernels' row decoding), in whole tiles of up to 128 rows; the largest row count of
// the walk is the first convolution's data gradient, B * H * W rows of the stacked input
constexpr long long MAX_ROWS = (1ll << 31) - 128;

struct DiscTable : ParamTable {
    DiscTable() {           // discriminator.py:29-64 (spectral_norm registers weight_orig after the bias, u / v as buffers after both)
        int cin = 2;
        for (int i = 0; i < NCONV; ++i) {
            const int idx = CONV_IDX[i], cout = NDF << i;
            const std::string k = "layers." + std::to_string(idx);
            add(k + ".weight_orig", (long long)cout * cin * 16); add(k + ".weight_u", cout); add(k + ".weight_v", cin * 16);
            add("layers." + std::to_string(idx + 1) + ".weight", cout); add("layers." + std::to_string(idx + 1) + ".bias", cout);
            add("layers." + std::to_string(idx + 2) + ".weight", cout);
            cin = cout;
        }
        add("layers.14.bias", NDF * 4); add("layers.14.weight_orig", NDF * 4 * NDF * 8); add("layers.14.weight_u", NDF * 4);
        add("layers.14.weight_v", NDF * 8); add("layers.16.weight", NDF * 4);
        add("layers.17.bias", 1); add("layers.17.weight_orig", NDF * 4); add("layers.17.weight_u", 1); add("layers.17.weight_v", NDF * 4);
        add("layers.18.slope", 1);
    }
};

const DiscTable& table() {
    static const DiscTable t;
    return t;
}

// W / sigma of one spectrally normalised weight and the [u | v] this forward used (discriminator._spectral)
struct Spectral { float *w_sn, *sigma, *uv; int R, Cc; std::string key; };
struct ConvSaved { const float* a_in; float* raw; Tabs tab; Spectral sn; int Cin, Cout, ih, iw, oh, ow; };
struct DSaved {
    float* xy;
    ConvSaved conv[NCONV];
    float* pooled;
    int* arg;
    Spectral s14, s17;
    float *h1, *a1, *h2, *out;
};

struct DRun : Walk {
    DRun() { tab = &table(); tag = "cmgan_disc"; who = "cmgan_disc_fwd"; }
};

size_t sums_size(int B) { return (size_t)(16 + 32 + 64 + 128) * B * 2 * 2 + 64; }       // discriminator._Sums

const int TAP_DY[16] = {-1, -1, -1, -1, 0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 2, 2}, TAP_DX[16] = {-1, 0, 1, 2, -1, 0, 1, 2, -1, 0, 1, 2, -1, 0, 1, 2};
const int TAPT_DY[16] = {1, 1, 1, 1, 0, 0, 0, 0, -1, -1, -1, -1, -2, -2, -2, -2}, TAPT_DX[16] = {1, 0, -1, -2, 1, 0, -1, -2, 1, 0, -1, -2, 1, 0, -1, -2};

Spectral spectral(DRun& r, const std::string& key, int R, int Cc) {
    Spectral s{r.keep((size_t)R * Cc), r.keep(1), r.keep((size_t)(R + Cc)), R, Cc, key};
    if (r.live()) {
        float* P = const_cast<float*>(r.P);            // training: u / v are updated in place in the block (the forward entry's params is writable)
        r.ok(cmgan_spectral_norm(r.w(key + ".weight_orig"), R, Cc, P + r.find(key + ".weight_u"), P + r.find(key + ".weight_v"), r.training ? 1 : 0,
                                 s.w_sn, s.sigma, s.uv, r.st));
    }
    return s;
}

// discriminator._disc_fwd; out: the caller's (B, 1) output (null in the backward's re-walk)
void forward(DRun& r, DSaved& sv, const float* x, long long sxb, long long sxh, long long sxw, const float* y, long long syb, long long syh,
             long long syw, int B, int H, int W, float* out) {
    const size_t n_sums = sums_size(B);
    double* sums0 = r.alloc<double>(n_sums);
    double* sums = sums0;
    r.zero(sums0, n_sums * sizeof(double));
    sv.xy = r.keep((size_t)B * H * W * 2);
    if (r.live()) r.ok(cmgan_stack2(x, sxb, sxh, sxw, y, syb, syh, syw, B, H, W, sv.xy, r.st));
    const float* act = sv.xy;
    int Cin = 2, ih = H, iw = W;
    for (int li = 0; li < NCONV; ++li) {
        const int idx = CONV_IDX[li], Cout = NDF << li;
        const std::string key = "layers." + std::to_string(idx);
        ConvSaved& L = sv.conv[li];
        L.sn = spectral(r, key, Cout, Cin * 16);
        const int oh = (ih + 2 - 4) / 2 + 1, ow = (iw + 2 - 4) / 2 + 1;
        const long long M = (long long)B * oh * ow;
        L.raw = r.keep((size_t)M * Cout);
        Gemm(act, Cin, L.sn.w_sn, 1, 16, (long long)Cin * 16, nullptr, L.raw, Cout, M, Cout, Cin).taps(16, TAP_DY, TAP_DX).conv(oh, ow, ih, iw, 2, 1, 2, 1)
            .run(r);
        L.tab = make_tabs(r, B, Cout);
        inst_norm_site(r, L.raw, Cout, B, (long long)oh * ow, Cout, Cout, r.w("layers." + std::to_string(idx + 1) + ".weight"),
                       r.w("layers." + std::to_string(idx + 1) + ".bias"), L.tab, sums);
        const float* slope = r.w("layers." + std::to_string(idx + 2) + ".weight");
        L.a_in = act; L.Cin = Cin; L.Cout = Cout; L.ih = ih; L.iw = iw; L.oh = oh; L.ow = ow;
        if (li < NCONV - 1) {
            float* nxt = r.keep((size_t)M * Cout);
            if (r.live())
                r.ok(cmgan_norm_apply(L.raw, Cout, B, (long long)oh * ow, Cout, 1 | (r.precision == 1 ? 16 : 0), L.tab.scale, L.tab.shift, Cout, slope,
                                      nxt, Cout, r.st));
            act = nxt; Cin = Cout; ih = oh; iw = ow;
        } else {
            sv.pooled = r.keep((size_t)B * Cout);
            sv.arg = r.keep<int>((size_t)B * Cout);
            if (r.live()) r.ok(cmgan_norm_maxpool(L.raw, B, (long long)oh * ow, Cout, L.tab.scale, L.tab.shift, slope, sv.pooled, sv.arg, r.st));
        }
    }
    // ---- SN Linear(128 -> 64) + Dropout(0.3) + PReLU(64) + SN Linear(64 -> 1) + LearnableSigmoid, exact fp32 whatever the precision
    const int n1 = NDF * 4, n0 = NDF * 8;
    sv.s14 = spectral(r, "layers.14", n1, n0);
    sv.h1 = r.keep((size_t)B * n1);
    Gemm(sv.pooled, n0, sv.s14.w_sn, 0, 1, n0, r.w("layers.14.bias"), sv.h1, n1, B, n1, n0).precision(0).run(r);
    sv.a1 = r.keep((size_t)B * n1);
    if (r.live())
        r.ok(cmgan_drop_prelu(sv.h1, (long long)B * n1, n1, r.w("layers.16.weight"), r.seed, drop_thr(r.training), drop_inv(r.training), sv.a1,
                              r.seed_dev, r.st));
    sv.s17 = spectral(r, "layers.17", 1, n1);
    sv.h2 = r.keep(B);
    Gemm(sv.a1, n1, sv.s17.w_sn, 0, 1, n1, r.w("layers.17.bias"), sv.h2, 1, B, 1, n1).precision(0).run(r);
    sv.out = r.keep(B);
    if (r.live()) r.ok(cmgan_lsigmoid(sv.h2, B, r.w("layers.18.slope"), sv.out, r.st));
    if (out && r.live()) {          // the backward reads the saved copy: the caller may reuse its output buffer
        const cudaError_t e = cudaMemcpyAsync(out, sv.out, (size_t)B * sizeof(float), cudaMemcpyDeviceToDevice, r.st);
        if (e != cudaSuccess) { cmgan_set_error("cmgan_disc_fwd: cudaMemcpyAsync: %s", cudaGetErrorString(e)); r.rc = -1; }
    }
    if ((size_t)(sums - sums0) > n_sums && r.rc == 0) { cmgan_set_error("cmgan_disc_fwd: statistics scratch exhausted"); r.rc = -1; }
}

// discriminator._sn_bwd: dW_orig += the spectral-norm backward of dW_sn with this forward's sigma and [u | v]
void sn_bwd(DRun& r, const Spectral& s, const float* dw_sn) {
    if (r.live()) r.ok(cmgan_spectral_norm_bwd(s.w_sn, dw_sn, s.R, s.Cc, s.uv, s.uv + s.R, s.sigma, r.g(s.key + ".weight_orig"), r.st));
}

// discriminator._disc_bwd; dx / dy (B, 1, H, W) contiguous or null
void backward(DRun& r, const DSaved& sv, int B, int H, int W, const float* dout, float* dx, float* dy) {
    const size_t n_sums = sums_size(B);
    double* sums0 = r.alloc<double>(n_sums);
    double* sums = sums0;
    r.zero(sums0, n_sums * sizeof(double));
    const int n1 = NDF * 4, n0 = NDF * 8;
    float* dh2 = r.alloc(B);
    if (r.live()) r.ok(cmgan_lsigmoid_bwd(sv.h2, sv.out, dout, B, r.w("layers.18.slope"), dh2, r.g("layers.18.slope"), r.st));
    float* dw17 = r.alloc(n1);
    if (r.wgrad) {
        r.zero(dw17, (size_t)n1 * sizeof(float));
        Gemm(sv.a1, n1, nullptr, 0, 1, n1, nullptr, dw17, 0, B, 1, n1).wgrad(dh2, 1, r.g("layers.17.bias")).precision(0).run(r);
        sn_bwd(r, sv.s17, dw17);
    }
    float* da1 = r.alloc((size_t)B * n1);
    Gemm(dh2, 1, sv.s17.w_sn, 0, n1, 1, nullptr, da1, n1, B, n1, 1).precision(0).run(r);
    float* dh1 = r.alloc((size_t)B * n1);
    if (r.live())
        r.ok(cmgan_drop_prelu_bwd(sv.h1, da1, (long long)B * n1, n1, r.w("layers.16.weight"), r.seed, drop_thr(r.training), drop_inv(r.training), dh1,
                                  r.g("layers.16.weight"), r.seed_dev, r.st));
    float* dw14 = r.alloc((size_t)n1 * n0);
    if (r.wgrad) {
        r.zero(dw14, (size_t)n1 * n0 * sizeof(float));
        Gemm(sv.pooled, n0, nullptr, 0, 1, n0, nullptr, dw14, 0, B, n1, n0).wgrad(dh1, n1, r.g("layers.14.bias")).precision(0).run(r);
        sn_bwd(r, sv.s14, dw14);
    }
    float* dpool = r.alloc((size_t)B * n0);
    Gemm(dh1, n1, sv.s14.w_sn, 0, n0, 1, nullptr, dpool, n0, B, n0, n1).precision(0).run(r);
    // ---- conv stack in reverse
    float* dact = nullptr;
    for (int li = NCONV - 1; li >= 0; --li) {
        const ConvSaved& L = sv.conv[li];
        const int idx = CONV_IDX[li], Cout = L.Cout, Cin = L.Cin;
        const long long M = (long long)B * L.oh * L.ow;
        if (li == NCONV - 1) {
            dact = r.alloc((size_t)M * Cout);
            if (r.live()) r.ok(cmgan_maxpool_bwd(dpool, sv.arg, B, (long long)L.oh * L.ow, Cout, dact, r.st));
        }
        float* draw = r.alloc((size_t)M * Cout);
        const std::string pn = "layers." + std::to_string(idx + 1), ps = "layers." + std::to_string(idx + 2);
        norm_bwd(r, L.raw, Cout, dact, Cout, B, (long long)L.oh * L.ow, Cout, 1, 1, L.tab, r.w(ps + ".weight"), draw, Cout, r.g(pn + ".weight"),
                 r.g(pn + ".bias"), r.g(ps + ".weight"), sums, true);
        float* dw_sn = r.alloc((size_t)Cout * Cin * 16);
        if (r.wgrad) {
            r.zero(dw_sn, (size_t)Cout * Cin * 16 * sizeof(float));
            Gemm(L.a_in, Cin, nullptr, 1, 16, (long long)Cin * 16, nullptr, dw_sn, 0, M, Cout, Cin).taps(16, TAP_DY, TAP_DX)
                .conv(L.oh, L.ow, L.ih, L.iw, 2, 1, 2, 1).wgrad(draw, Cout, nullptr).run(r);
            sn_bwd(r, L.sn, dw_sn);
        }
        if (li > 0 || dx || dy) {
            const long long Min = (long long)B * L.ih * L.iw;
            dact = r.alloc((size_t)Min * Cin);
            Gemm(draw, Cout, L.sn.w_sn, 1, (long long)Cin * 16, 16, nullptr, dact, Cin, Min, Cin, Cout).taps(16, TAPT_DY, TAPT_DX)
                .conv(L.ih, L.iw, L.oh, L.ow, 1, 2, 1, 2).run(r);
        }
    }
    if ((dx || dy) && r.live()) r.ok(cmgan_unstack2(dact, (long long)B * H * W, dx, dy, r.st));
    if ((size_t)(sums - sums0) > n_sums && r.rc == 0) { cmgan_set_error("cmgan_disc_bwd: statistics scratch exhausted"); r.rc = -1; }
}

// Workspace: the saved region (what the backward reads, fixed by the shape), then the scratch of whichever call runs -- the forward's or the
// backward's, which starts with a parameter-gradient stand-in for frozen weights.  Both calls derive the saved layout from the same walk.
struct Layout { size_t keep, fwd, bwd; };

Layout layout(int B, int H, int W, int precision) {
    DSaved sv;
    DRun f;
    f.precision = precision; f.saving = true;
    forward(f, sv, nullptr, 0, 0, 0, nullptr, 0, 0, 0, B, H, W, nullptr);
    DRun b;
    b.precision = precision;
    b.alloc((size_t)table().total);
    float one;
    backward(b, sv, B, H, W, nullptr, &one, &one);       // dry: sized with the input gradients (nothing is written)
    return {(f.ktop + 255) & ~(size_t)255, f.peak, b.peak};
}

int check_shape(const char* who, int B, int H, int W, int precision) {
    CMGAN_REQUIRE(B > 0 && H >= MIN_HW && W >= MIN_HW, "%s: expected inputs of shape (B, 1, H, W) with B > 0 and H, W >= %d (four 4x4 stride-2 "
                  "convolutions), got B=%d H=%d W=%d", who, MIN_HW, B, H, W);
    CMGAN_REQUIRE(precision == 0 || precision == 1, "%s: precision must be 0 (fp32) or 1 (tf32)", who);
    CMGAN_REQUIRE((long long)B * H * W <= MAX_ROWS, "%s: B * H * W = %lld rows exceed 2^31 - 128 (the GEMMs count rows in 32 bits; the first "
                  "convolution's data gradient has B * H * W rows); split the batch", who, (long long)B * H * W);
    return 0;
}

// checks shared by both entries; on success `r` is set up for the walk (saved region at the workspace base, scratch above it)
int setup(DRun& r, const char* who, const float* params, int B, int H, int W, int training, unsigned long long seed,
          const unsigned long long* seed_dev, void* workspace, long long workspace_bytes, int precision, void* stream) {
    CMGAN_REQUIRE(params && workspace, "%s: null pointer", who);
    if (check_shape(who, B, H, W, precision) != 0) return -1;
    CMGAN_REQUIRE(training == 0 || training == 1, "%s: training must be 0 (eval) or 1 (train)", who);
    CMGAN_REQUIRE((((uintptr_t)params) & 15) == 0 && (((uintptr_t)workspace) & 255) == 0, "%s: params must be 16-byte, workspace 256-byte aligned", who);
    const long long need = cmgan_disc_workspace_bytes(B, H, W, precision);
    CMGAN_REQUIRE(workspace_bytes >= need, "%s: workspace too small (%lld bytes needed, %lld given)", who, need, workspace_bytes);
    const Layout L = layout(B, H, W, precision);
    cmgan_set_tf32_rounding(precision);       // as cmgan_tscnet_fwd_train: producers of tensor-core operands round to nearest on store
    r.P = params; r.dry = false; r.precision = precision; r.st = (cudaStream_t)stream; r.who = who;
    r.saving = true; r.kws = static_cast<char*>(workspace);
    r.ws = r.kws + L.keep; r.cap = (size_t)workspace_bytes - L.keep;
    r.training = training == 1; r.seed = seed; r.seed_dev = seed_dev;
    return 0;
}

}  // namespace

CMGAN_API int cmgan_disc_param_count(void) { return (int)table().e.size(); }
CMGAN_API long long cmgan_disc_param_floats(void) { return table().total; }

CMGAN_API int cmgan_disc_param_info(int index, const char** key, long long* offset, long long* numel) {
    CMGAN_REQUIRE(index >= 0 && index < (int)table().e.size(), "cmgan_disc_param_info: index %d out of range", index);
    const Entry& e = table().e[index];
    if (key) *key = e.key.c_str();
    if (offset) *offset = e.off;
    if (numel) *numel = e.numel;
    return 0;
}

CMGAN_API long long cmgan_disc_workspace_bytes(int B, int H, int W, int precision) {
    if (check_shape("cmgan_disc_workspace_bytes", B, H, W, precision) != 0) return -1;
    const Layout L = layout(B, H, W, precision);
    return (long long)(L.keep + std::max(L.fwd, L.bwd)) + 256;
}

CMGAN_API int cmgan_disc_fwd(float* params, const float* x, long long sxb, long long sxh, long long sxw, const float* y, long long syb, long long syh,
                             long long syw, int B, int H, int W, int training, unsigned long long seed, const unsigned long long* seed_dev, float* out,
                             void* workspace, long long workspace_bytes, int precision, void* stream) {
    const char* who = "cmgan_disc_fwd";
    CMGAN_REQUIRE(x && y && out, "%s: null pointer", who);
    DRun r;
    DSaved sv;
    if (setup(r, who, params, B, H, W, training, seed, seed_dev, workspace, workspace_bytes, precision, stream) != 0) return -1;
    forward(r, sv, x, sxb, sxh, sxw, y, syb, syh, syw, B, H, W, out);
    return r.rc;
}

CMGAN_API int cmgan_disc_bwd(const float* params, int B, int H, int W, int training, unsigned long long seed, const unsigned long long* seed_dev,
                             const float* dout, float* grads, float* dx, float* dy, void* workspace, long long workspace_bytes, int precision,
                             void* stream) {
    const char* who = "cmgan_disc_bwd";
    CMGAN_REQUIRE(grads || dx || dy, "%s: grads, dx and dy are all null: nothing to compute", who);
    CMGAN_REQUIRE(dout, "%s: null pointer", who);
    CMGAN_REQUIRE((((uintptr_t)grads) & 15) == 0, "%s: grads must be 16-byte aligned", who);
    DRun r;
    DSaved sv;
    if (setup(r, who, params, B, H, W, training, seed, seed_dev, workspace, workspace_bytes, precision, stream) != 0) return -1;
    r.quiet = true;          // the forward walk launches nothing here: it only places the saved activations where the forward call left them
    forward(r, sv, nullptr, 0, 0, 0, nullptr, 0, 0, 0, B, H, W, nullptr);
    if (r.rc != 0) return r.rc;
    r.quiet = false;
    r.top = r.peak = 0;
    float* gscratch = r.alloc((size_t)table().total);       // frozen weights: the gradient atomics fused into the data-gradient kernels land here
    r.G = grads ? grads : gscratch;
    r.wgrad = grads != nullptr;
    backward(r, sv, B, H, W, dout, dx, dy);
    return r.rc;
}
