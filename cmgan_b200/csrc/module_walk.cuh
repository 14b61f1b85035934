// Pieces shared by the module-level entry points (tscnet_module.cu, disc_module.cu): the flat parameter table, the workspace walk with its
// bump allocator and saved region, the GEMM argument builder and the normalisation sites.  A module entry is one walk over its launch list;
// the same walk in `dry` mode sizes the workspace, and in `quiet` mode re-derives where a forward left its saved activations.
#pragma once
#include <cstring>
#include <string>
#include <unordered_map>
#include <vector>

#include "common.cuh"
#include "../../include/cmgan_b200.h"

namespace cmgan_walk {

struct Entry { std::string key; long long off, numel; };

// one flat fp32 block of state_dict tensors in state_dict order, each starting at a multiple of 4 floats
struct ParamTable {
    std::vector<Entry> e;
    std::unordered_map<std::string, long long> at;
    long long total = 0;
    void add(const std::string& k, long long n) {
        e.push_back({k, total, n});
        at.emplace(k, total);
        total += (n + 3) / 4 * 4;
    }
};

struct Tabs { float *scale, *shift, *mean, *rstd; int width; };

template <typename T>
T* off(T* p, long long n) { return p ? p + n : nullptr; }

struct Walk {
    const ParamTable* tab = nullptr;
    const char* tag = "";       // prefix of the unknown-parameter message
    const char* who = "";       // prefix of the workspace-too-small message
    const float* P = nullptr;   // parameter block (null in a dry run)
    char* ws = nullptr;         // workspace base (of the scratch region when saving)
    size_t top = 0, peak = 0, cap = 0;
    bool dry = true;
    int precision = 0;
    cudaStream_t st = nullptr;
    const int* frames = nullptr;      // ragged batch: valid frames per utterance (device); null = every utterance fills the grid
    int rc = 0;
    // training entries only (the inference walks leave these alone)
    bool saving = false;        // forward: keep what the backward reads in the saved region (below the scratch)
    char* kws = nullptr;        // saved region base
    size_t ktop = 0;
    bool quiet = false;         // walk for the addresses only: the backward re-derives the saved layout this way, nothing is launched
    bool training = false;
    unsigned long long seed = 0;
    const unsigned long long* seed_dev = nullptr;
    float* G = nullptr;         // backward: parameter-gradient block (scratch when the weights are frozen)
    bool wgrad = true;          // backward: run the weight-gradient GEMMs

    long long find(const std::string& key) const {
        const auto it = tab->at.find(key);
        if (it != tab->at.end()) return it->second;
        cmgan_set_error("%s: unknown parameter %s", tag, key.c_str());
        const_cast<Walk*>(this)->rc = -1;
        return -1;
    }
    const float* w(const std::string& key) const {
        if (dry) return nullptr;
        const long long o = find(key);
        return o < 0 ? nullptr : P + o;
    }
    float* g(const std::string& key) const {
        if (dry) return nullptr;
        const long long o = find(key);
        return o < 0 ? nullptr : G + o;
    }
    template <typename T = float>
    T* alloc(size_t n) {
        top = (top + 255) & ~(size_t)255;
        T* p = dry ? nullptr : reinterpret_cast<T*>(ws + top);
        top += n * sizeof(T);
        if (top > peak) peak = top;
        if (!dry && top > cap && rc == 0) { cmgan_set_error("%s: workspace too small (%zu bytes needed so far, %zu given)", who, top, cap); rc = -1; }
        return p;
    }
    // an activation the backward reads: in the saved region when saving, else scratch like any other buffer
    template <typename T = float>
    T* keep(size_t n) {
        if (!saving) return alloc<T>(n);
        ktop = (ktop + 255) & ~(size_t)255;
        T* p = dry ? nullptr : reinterpret_cast<T*>(kws + ktop);
        ktop += n * sizeof(T);
        return p;
    }
    void ok(int r) { if (r != 0 && rc == 0) rc = r; }
    bool live() const { return !dry && !quiet && rc == 0; }
    // zero n bytes on the walk's stream (statistics scratch, gradient accumulators)
    void zero(void* p, size_t n) {
        if (!live()) return;
        const cudaError_t e = cudaMemsetAsync(p, 0, n, st);
        if (e != cudaSuccess) { cmgan_set_error("%s: cudaMemsetAsync: %s", who, cudaGetErrorString(e)); rc = -1; }
    }
};

inline Tabs make_tabs(Walk& r, int G, int width) {
    Tabs t;
    t.scale = r.keep((size_t)G * width); t.shift = r.keep((size_t)G * width);
    t.mean = r.keep((size_t)G * width); t.rstd = r.keep((size_t)G * width);
    t.width = width;
    return t;
}

struct Gemm {
    CmganGemmArgs a;
    bool wg = false;
    int prec = -1;              // >= 0: this call's precision instead of the walk's (the discriminator's linears always run exact fp32)
    Gemm(const float* A, long long lda, const float* W, long long sb_tap, long long sb_k, long long sb_n, const float* bias, float* Cout,
         long long ldc, long long M, int N, int Cin) {
        memset(&a, 0, sizeof(a));
        a.A = A; a.lda = lda; a.B = W; a.sb_tap = sb_tap; a.sb_k = sb_k; a.sb_n = sb_n; a.bias = bias; a.C = Cout; a.ldc = ldc;
        a.M = (int)M; a.N = N; a.Cin = Cin; a.ntaps = 1;
        a.mul_y = a.mul_x = a.div_y = a.div_x = 1;
        a.inv_keep = 1.f; a.pro_inv_keep = 1.f; a.alpha = 1.f; a.pro_alpha = 1.f;
    }
    Gemm& conv(int OH, int OW, int IH, int IW, int mul_x = 1, int div_x = 1, int mul_y = 1, int div_y = 1) {
        a.conv = 1; a.OH = OH; a.OW = OW; a.IH = IH; a.IW = IW; a.mul_x = mul_x; a.div_x = div_x; a.mul_y = mul_y; a.div_y = div_y;
        return *this;
    }
    Gemm& taps(int n, const int* dy, const int* dx) {
        a.ntaps = n;
        for (int i = 0; i < n; ++i) { a.dy[i] = dy[i]; a.dx[i] = dx[i]; }
        return *this;
    }
    Gemm& residual(const float* R, long long ldr) { a.epi = CMGAN_EPI_DROP_RES; a.R = R; a.ldr = ldr; return *this; }
    Gemm& drop(unsigned long long seed, unsigned thr, float inv_keep) { a.seed = seed; a.drop_thr = thr; a.inv_keep = inv_keep; return *this; }
    Gemm& epi(int e, const float* aux, long long ldaux) { a.epi = e; a.aux = aux; a.ldaux = ldaux; return *this; }
    Gemm& precision(int p) { prec = p; return *this; }
    // weight gradient: accumulates dW (laid out like W: C = dW, ldc = 0) from A and the upstream gradient rows D
    Gemm& wgrad(const float* D, long long ldd, float* dbias) { wg = true; a.D = D; a.ldd = ldd; a.dbias = dbias; return *this; }
    void run(Walk& r) {
        a.precision = prec >= 0 ? prec : r.precision;
        a.seed_dev = r.seed_dev;
        if (wg) {
            if (r.wgrad && r.live()) r.ok(cmgan_gemm_wgrad_f32(&a, r.st));
            return;
        }
        if (a.precision == 1 && a.N % 16 == 0 && a.N <= 256 && a.Cin % 32 == 0) {      // scratch for the re-tiled weight (gemm_args.h)
            a.ws_floats = (long long)a.N * a.Cin * a.ntaps;
            a.ws = r.alloc((size_t)a.ws_floats);
        }
        if (r.live()) r.ok(cmgan_gemm_rows_f32(&a, r.st));
    }
};

// InstanceNorm statistics -> tables; rows_per_t: rows of one frame within a group (row = t * rows_per_t + f); a ragged batch normalises over
// the valid frames only.  Every site takes its own G * Cn * 2 doubles of the pass's zeroed statistics scratch.
inline void inst_norm_site(Walk& r, const float* x, long long ldx, int G, long long rows, long long rows_per_t, int Cn, const float* gamma,
                           const float* beta, const Tabs& t, double*& sums) {
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

// InstanceNorm / BatchNorm (+ PReLU) backward of one site (conformer_block._norm_bwd); `operand`: dx feeds tensor-core contractions
inline void norm_bwd(Walk& r, const float* x, long long ldx, const float* dact, long long ldd, int G, long long rows, int Cn, int act, int batch_stats,
                     const Tabs& t, const float* slope, float* dx, long long lddx, float* dgamma, float* dbeta, float* dslope, double*& sums,
                     bool operand) {
    double* s = sums;
    sums += (size_t)G * Cn * 2;
    if (!r.live()) return;
    r.ok(cmgan_norm_bwd_reduce(x, ldx, dact, ldd, G, rows, Cn, act, t.scale, t.shift, t.mean, t.rstd, t.width, slope, s, dslope, r.st));
    r.ok(cmgan_norm_bwd_apply(x, ldx, dact, ldd, G, rows, Cn, act | (operand && r.precision == 1 ? 16 : 0), batch_stats, t.scale, t.shift, t.mean,
                              t.rstd, t.width, slope, s, dx, lddx, dgamma, dbeta, r.st));
}

}  // namespace cmgan_walk
