// Signal front/back end and the small HBM-bound ends of TSCNet:
//   RMS normalise + reflect pad (train.py:75-87), power-law compression / un-compression (utils.py:20-39),
//   overlap-add of the inverse STFT (train.py:106-112), the generator head (generator.py:175-179 + conv_1 :53),
//   the (1,2) output convolutions of both decoders (generator.py:126,150) and the final recombination
//   (generator.py:136-139,188-196).  The framed DFT / inverse DFT themselves are GEMMs (gemm_args.h).
#include "common.cuh"
#include "frontend.cuh"
#include "../../include/cmgan_b200.h"

namespace {

constexpr int NFFT = 400, HOP = 100, NF = 201;

// ------------------------------------------------------------------ STFT tables
// The window-folded DFT bases and the inverse overlap-add envelopes, built the way signal.py built them in torch float64 and rounded to
// fp32 once: angle(r) = (2 pi r) / 400 with r = (n k) mod 400, window w[n] = 0.54 - 0.46 cos(angle(n)).  Every product, sum and quotient
// is an explicit _rn intrinsic, so nvcc cannot contract a pair into an FMA: each step is the IEEE float64 operation torch performs, in
// the same order, and only cos / sin of the 400 angles come from a different (device) libm.
__device__ __forceinline__ double inv_envelope64(const double* w, int n, int T) {
    const int p = n + NFFT / 2;                     // position in the un-trimmed envelope: sum_t w^2[p - 100 t], t increasing from 0.0
    const int t_lo = p >= NFFT ? (p - NFFT) / HOP + 1 : 0, t_hi = min(p / HOP, T - 1);          // the frames that cover p
    double e = 0.0;
    for (int t = t_lo; t <= t_hi; ++t) {
        const int m = p - t * HOP;
        e = __dadd_rn(e, __dmul_rn(w[m], w[m]));
    }
    return __ddiv_rn(1.0, e);
}

__global__ void stft_tables_kernel(float* __restrict__ fwd, float* __restrict__ inv, int T, float* __restrict__ env, float* __restrict__ tail) {
    __shared__ double cs[NFFT], sn[NFFT], w[NFFT];
    for (int r = threadIdx.x; r < NFFT; r += blockDim.x) {
        const double a = __ddiv_rn(__dmul_rn(2.0 * 3.141592653589793, (double)r), (double)NFFT);
        cs[r] = cos(a);
        sn[r] = sin(a);
        w[r] = __dsub_rn(0.54, __dmul_rn(0.46, cs[r]));
    }
    __syncthreads();
    const long nb = (long)NFFT * 2 * NF, nenv = env ? (long)HOP * (T - 1) : 0, total = 2 * nb + nenv + HOP;
    for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
        if (i < nb) {                               // fwd (400, 402): [w cos | -w sin]
            if (!fwd) continue;
            const int n = (int)(i / (2 * NF)), col = (int)(i % (2 * NF)), k = col < NF ? col : col - NF, r = n * k % NFFT;
            fwd[i] = (float)(col < NF ? __dmul_rn(w[n], cs[r]) : __dmul_rn(-w[n], sn[r]));
        } else if (i < 2 * nb) {                    // inv (402, 400): [wk cos w / 400 ; -wk sin w / 400], wk = 1, 2, ..., 2, 1
            if (!inv) continue;
            const long j = i - nb;
            const int row = (int)(j / NFFT), n = (int)(j % NFFT), k = row < NF ? row : row - NF, r = n * k % NFFT;
            const double wk = (k == 0 || k == NF - 1) ? 1.0 : 2.0;
            const double v = row < NF ? __dmul_rn(__dmul_rn(wk, cs[r]), w[n]) : __dmul_rn(__dmul_rn(-wk, sn[r]), w[n]);
            inv[j] = (float)__ddiv_rn(v, (double)NFFT);
        } else if (i < 2 * nb + nenv) {             // 1 / envelope(T), n < 100 (T - 1)
            const int n = (int)(i - 2 * nb);
            env[n] = (float)inv_envelope64(w, n, T);
        } else if (tail) {                          // the last 100 samples of 1 / envelope(T), any T >= 3: those of T = 8
            const int n = (int)(i - 2 * nb - nenv);
            tail[n] = (float)inv_envelope64(w, 6 * HOP + n, 8);
        }
    }
}

// ------------------------------------------------------------------ RMS scale: c[b] = sqrt(L / sum x^2)
// RAGGED: row b has its own length lens[b] (clamped to [0, L]); tlen (optional) receives its frame count ceil(L_b / 100) + 1
template <bool RAGGED>
__global__ void rms_scale_kernel(const float* __restrict__ x, long ldx, int L, float* __restrict__ c, const int* __restrict__ lens,
                                 int* __restrict__ tlen) {
    __shared__ double sm[32];
    if (RAGGED) L = clamp_len(__ldg(lens + blockIdx.x), L);
    const float* p = x + (long)blockIdx.x * ldx;
    double s = 0.0;
    for (int i = threadIdx.x; i < L; i += blockDim.x) { float v = __ldg(p + i); s += (double)v * v; }
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if ((threadIdx.x & 31) == 0) sm[threadIdx.x >> 5] = s;
    __syncthreads();
    if (threadIdx.x == 0) {
        double t = 0.0;
        for (int w = 0; w < (blockDim.x >> 5); ++w) t += sm[w];
        c[blockIdx.x] = (float)sqrt((double)L / t);
        if (RAGGED && tlen) tlen[blockIdx.x] = (L + HOP - 1) / HOP + 1;
    }
}

// xp[b, i] = c[b] * x[b, reflect(i - 200)], i < L + 400; zero up to Lp
__global__ void pad_reflect_kernel(const float* __restrict__ x, long ldx, int L, const float* __restrict__ c, float* __restrict__ xp, int Lp) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    int b = blockIdx.y;
    if (i >= Lp) return;
    float v = 0.f;
    if (i < L + NFFT) {
        int j = i - NFFT / 2;
        if (j < 0) j = -j;
        if (j >= L) j = 2 * (L - 1) - j;
        v = __ldg(x + (long)b * ldx + j) * (c ? c[b] : 1.f);
    }
    xp[(long)b * Lp + i] = v;
}

// ragged front end of evaluation.py:21-29 + the STFT's centre padding: utterance b (L_b = lens[b] samples, clamped to [0, L]) is wrap-padded
// with its own head to Lw = ceil(L_b / 100) * 100, reflect-padded by 200 on both sides and scaled by c[b]; zero from Lw + 400 up to Lp.
// Needs L_b >= Lw - L_b and Lw > 200 (checked on the host); the value of every element is the one cmgan_pad_reflect gives the padded
// utterance alone.
// FOLD (evaluation.py:25-34): every clip has L samples and lens is unused; clip b, wrap-padded with its own head, is cut into segments of
// S samples, and this launch fills k rows per clip: row b k + r is segment seg0 + r, reflect-padded by 200 on each side (its own edges) and
// scaled by c[b] -- the rows signal.enhance feeds its DFT after the reshape, without the wrapped copy.  Needs S > 200 and a wrapped length
// (seg0 + k) S <= 2 L (checked on the host).  Segment r starts at sample r hop of the wrapped clip: hop = S is the fold, hop < S the
// overlapping windows of cmgan_enhance_overlap, which need (seg0 + k - 1) hop + S <= 2 L.
template <bool FOLD>
__global__ void pad_wrap_reflect_kernel(const float* __restrict__ x, long ldx, int L, const int* __restrict__ lens, int k, int S, int seg0,
                                        int hop, const float* __restrict__ c, float* __restrict__ xp, int Lp) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    const int row = blockIdx.y;
    if (i >= Lp) return;
    const int b = FOLD ? row / k : row;
    const int Lb = FOLD ? L : clamp_len(__ldg(lens + b), L);
    const int Lw = FOLD ? S : (Lb + HOP - 1) / HOP * HOP;
    float v = 0.f;
    if (Lb > 0 && i < Lw + NFFT) {
        int j = i - NFFT / 2;
        if (j < 0) j = -j;
        if (j >= Lw) j = 2 * (Lw - 1) - j;
        if (FOLD) j += (seg0 + row - b * k) * hop;    // segment r starts at sample r hop of the wrapped clip
        if (j >= Lb) j -= Lb;                         // wrap padding: sample Lb + k is sample k
        j = clamp_len(j, Lb - 1);                     // only reachable for lengths the host rejects
        v = __ldg(x + (long)b * ldx + j) * (c ? c[b] : 1.f);
    }
    xp[(long)row * Lp + i] = v;
}

// S (B*T, 402) = [re | im]  ->  planes X[b, 0/1, t, f] = S * |S|^-0.7
__global__ void compress_kernel(const float* __restrict__ S, long total /*B*T*F*/, int T, float* __restrict__ X) {
    long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= total) return;
    int f = (int)(i % NF);
    long bt = i / NF;
    long b = bt / T; int t = (int)(bt % T);
    float re = __ldg(S + bt * (2 * NF) + f), im = __ldg(S + bt * (2 * NF) + NF + f);
    float m2 = re * re + im * im;
    float sc = m2 > 0.f ? powf(m2, -0.35f) : 0.f;
    long o = ((b * 2) * T + t) * NF + f;
    X[o] = re * sc;
    X[o + (long)T * NF] = im * sc;
}

// un-compression of (re, im) planes (each (B, T, F) with explicit strides) -> U (B*T, 402) = [re | im] * |.|^(7/3)
__global__ void uncompress_kernel(const float* __restrict__ re_p, const float* __restrict__ im_p, long sb, long st, long sf, long total, int T,
                                  float* __restrict__ U) {
    long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= total) return;
    int f = (int)(i % NF);
    long bt = i / NF;
    long b = bt / T; int t = (int)(bt % T);
    long o = b * sb + t * st + f * sf;
    float re = __ldg(re_p + o), im = __ldg(im_p + o);
    float m2 = re * re + im * im;
    float sc = m2 > 0.f ? powf(m2, 7.0f / 6.0f) : 0.f;
    U[bt * (2 * NF) + f] = re * sc;
    U[bt * (2 * NF) + NF + f] = im * sc;
}

// gradient of the un-compression: dU (B*T, 402) -> d_re, d_im planes (B, T, F) contiguous
__global__ void uncompress_bwd_kernel(const float* __restrict__ re_p, const float* __restrict__ im_p, long sb, long st, long sf, long total, int T,
                                      const float* __restrict__ dU, float* __restrict__ dre, float* __restrict__ dim_, int accumulate) {
    long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= total) return;
    int f = (int)(i % NF);
    long bt = i / NF;
    long b = bt / T; int t = (int)(bt % T);
    long o = b * sb + t * st + f * sf;
    float re = __ldg(re_p + o), im = __ldg(im_p + o);
    float gr = __ldg(dU + bt * (2 * NF) + f), gi = __ldg(dU + bt * (2 * NF) + NF + f);
    float m2 = re * re + im * im;
    float dr = 0.f, di = 0.f;
    if (m2 > 0.f) {
        const float p = 7.0f / 3.0f;
        float mp = powf(m2, 0.5f * p);            // m^p
        float mp2 = p * mp / m2;                  // p m^(p-2)
        dr = gr * (mp + mp2 * re * re) + gi * (mp2 * re * im);
        di = gr * (mp2 * re * im) + gi * (mp + mp2 * im * im);
    }
    if (accumulate) { dre[i] += dr; dim_[i] += di; }
    else { dre[i] = dr; dim_[i] = di; }
}

// generic strided power law  Y = X * |X|^p  over a (d0, d1, d2) index space (power_compress p = -0.7, power_uncompress p = 7/3)
__global__ void power_law_kernel(const float* __restrict__ re, const float* __restrict__ im, long i0, long i1, long i2, float* __restrict__ ore,
                                 float* __restrict__ oim, long o0, long o1, long o2, int d1, int d2, long n, float half_p) {
    long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    int c = (int)(i % d2); long t = i / d2; int b = (int)(t % d1); long a = t / d1;
    long io = a * i0 + b * i1 + c * i2, oo = a * o0 + b * o1 + c * o2;
    float r = __ldg(re + io), m = __ldg(im + io);
    float m2 = r * r + m * m;
    float sc = m2 > 0.f ? powf(m2, half_p) : 0.f;
    ore[oo] = r * sc; oim[oo] = m * sc;
}
// gradient: (gre, gim) at the output strides -> (dre, dim) at the input strides
__global__ void power_law_bwd_kernel(const float* __restrict__ re, const float* __restrict__ im, long i0, long i1, long i2,
                                     const float* __restrict__ gre, const float* __restrict__ gim, long o0, long o1, long o2,
                                     float* __restrict__ dre, float* __restrict__ dim_, long q0, long q1, long q2, int d1, int d2, long n, float p) {
    long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    int c = (int)(i % d2); long t = i / d2; int b = (int)(t % d1); long a = t / d1;
    long io = a * i0 + b * i1 + c * i2, oo = a * o0 + b * o1 + c * o2, qo = a * q0 + b * q1 + c * q2;
    float r = __ldg(re + io), m = __ldg(im + io), gr = __ldg(gre + oo), gi = __ldg(gim + oo);
    float m2 = r * r + m * m;
    float dr = 0.f, di = 0.f;
    if (m2 > 0.f) {
        float mp = powf(m2, 0.5f * p), mp2 = p * mp / m2;
        dr = gr * (mp + mp2 * r * r) + gi * (mp2 * r * m);
        di = gr * (mp2 * r * m) + gi * (mp + mp2 * m * m);
    }
    dre[qo] = dr; dim_[qo] = di;
}

// overlap-add: y[b, n] = (sum_t frames[b, t, n + 200 - 100 t]) / env[n],  n < 100 (T - 1)
// MAP (the folded clips of evaluation.py:30-34,52): row b is segment r = b % k of clip b / k; its samples go to y[b / k, r 100 (T - 1) + n]
// below L (the reference's flatten()[:length]), de-normalised by c_div[b / k].  k = 1 writes y[b, n], n < L.
template <bool MAP>
__global__ void ola_kernel(const float* __restrict__ frames, int T, const float* __restrict__ inv_env, const float* __restrict__ c_div,
                           float* __restrict__ y, long ldy, int k_seg, int L) {
    int n = blockIdx.x * blockDim.x + threadIdx.x;
    int b = blockIdx.y;
    int Lout = HOP * (T - 1);
    if (n >= Lout) return;
    int p = n + NFFT / 2;                         // position in the un-trimmed signal
    int t_hi = p / HOP; if (t_hi > T - 1) t_hi = T - 1;
    int t_lo = (p - NFFT + HOP) / HOP; if (p - NFFT + 1 <= 0) t_lo = 0;
    float s = 0.f;
    for (int t = t_lo; t <= t_hi; ++t) {
        int k = p - t * HOP;
        if (k >= 0 && k < NFFT) s += __ldg(frames + ((long)b * T + t) * NFFT + k);
    }
    s *= inv_env[n];
    if (MAP) {
        const int clip = b / k_seg, o = (b - clip * k_seg) * Lout + n;
        if (o >= L) return;
        if (c_div) s /= c_div[clip];
        y[(long)clip * ldy + o] = s;
        return;
    }
    if (c_div) s /= c_div[b];
    y[(long)b * ldy + n] = s;
}

// overlap-add of a ragged batch: utterance b sums only its frames t < T_b = tlen[b] (clamped to [0, T]) into y[b, n], n < 100 (T_b - 1),
// with its own inverse envelope: 1 / envelope(T_b) equals inv_env (the table of the full T-frame grid) except over the last 100 samples,
// where frame T_b is missing; there it is inv_tail[n - 100 (T_b - 2)], the same for every T_b >= 4 (signal._inv_envelope_tail).
// Samples n >= 100 (T_b - 1) are written as zero.
// MAP: y is the caller's (B, L) output; only the clip's own samples n < lens[b] (clamped to [0, L]) are written, nothing past them.
template <bool MAP>
__global__ void ola_ragged_kernel(const float* __restrict__ frames, int T, const int* __restrict__ tlen, const float* __restrict__ inv_env,
                                  const float* __restrict__ inv_tail, const float* __restrict__ c_div, float* __restrict__ y, long ldy,
                                  const int* __restrict__ lens, int L) {
    const int n = blockIdx.x * blockDim.x + threadIdx.x;
    const int b = blockIdx.y;
    if (n >= HOP * (T - 1)) return;
    if (MAP && n >= clamp_len(__ldg(lens + b), L)) return;
    const int Tb = clamp_len(__ldg(tlen + b), T);
    const int Lout = HOP * (Tb - 1);
    float s = 0.f;
    if (n < Lout) {
        const int p = n + NFFT / 2;
        int t_hi = p / HOP; if (t_hi > Tb - 1) t_hi = Tb - 1;
        int t_lo = (p - NFFT + HOP) / HOP; if (p - NFFT + 1 <= 0) t_lo = 0;
        for (int t = t_lo; t <= t_hi; ++t) {
            const int k = p - t * HOP;
            if (k >= 0 && k < NFFT) s += __ldg(frames + ((long)b * T + t) * NFFT + k);
        }
        const int tail0 = Lout - HOP;
        s *= n >= tail0 ? inv_tail[n - tail0] : inv_env[n];
        if (c_div) s /= c_div[b];
    }
    y[(long)b * ldy + n] = s;
}

// ------------------------------------------------------------------ crossfade of overlapping windows (cmgan_enhance_overlap)
// w[m] = fp32(sin^2(pi (m + 0.5) / (2 O))), m < O: float64 on the device, each step an explicit _rn intrinsic (the order numpy evaluates
// np.sin(np.pi * (m + 0.5) / (2 * O)) ** 2 in), rounded to fp32 once.  w[m] + w[O - 1 - m] = 1 in exact arithmetic.
__global__ void crossfade_table_kernel(float* __restrict__ w, int O) {
    for (int m = blockIdx.x * blockDim.x + threadIdx.x; m < O; m += gridDim.x * blockDim.x) {
        const double s = sin(__ddiv_rn(__dmul_rn(3.141592653589793, __dadd_rn((double)m, 0.5)), (double)(2 * O)));
        w[m] = (float)__dmul_rn(s, s);
    }
}

// Windows j0 .. j0 + rows - 1 of k, window j covering samples [j H, j H + S), H = S - O, staged as y (rows, S).  For n in [n0, n1), with
// j = min(n / H, k - 1) and m = n - j H:
//   j >= 1 and m < O:  out[n] = fp32(w[O - 1 - m] y_{j-1}[m + H]) + fp32(w[m] y_j[m])    (two rounded products, a rounded sum: no FMA)
//   otherwise:         out[n] = y_j[m]
// The pass's range is n0 = j0 H up to n1 = L after the last window, else n1 = (j0 + rows) H + O: the first O samples of the next window
// j0 + rows, where only its predecessor's half, fp32(w[O - 1 - m] y_{j0+rows-1}[m + H]), is known.  That half is written into out and the
// next pass adds its own to it (its first window finds y_{j-1} there), so nothing is carried outside out.
__global__ void crossfade_kernel(const float* __restrict__ y, int rows, int j0, int k, int S, int O, const float* __restrict__ w,
                                 float* __restrict__ out, int n0, int n1) {
    const int n = n0 + blockIdx.x * blockDim.x + threadIdx.x;
    if (n >= n1) return;
    const int H = S - O;
    const int j = min(n / H, k - 1), m = n - j * H, r = j - j0;
    if (r == rows) {                                            // the next pass's first window: hand on the predecessor's half
        out[n] = __fmul_rn(__ldg(w + O - 1 - m), __ldg(y + (long)(r - 1) * S + m + H));
        return;
    }
    float v = __ldg(y + (long)r * S + m);
    if (j >= 1 && m < O) {
        const float a = r > 0 ? __fmul_rn(__ldg(w + O - 1 - m), __ldg(y + (long)(r - 1) * S + m + H)) : out[n];
        v = __fadd_rn(a, __fmul_rn(__ldg(w + m), v));
    }
    out[n] = v;
}

// gradient of overlap-add: dframes[b, t, k] = dy[b, 100 t + k - 200] / env (zero outside the trimmed range)
__global__ void ola_bwd_kernel(const float* __restrict__ dy, long lddy, int T, const float* __restrict__ inv_env, float* __restrict__ dframes) {
    long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    int b = blockIdx.y;
    if (i >= (long)T * NFFT) return;
    int t = (int)(i / NFFT), k = (int)(i % NFFT);
    int n = t * HOP + k - NFFT / 2;
    float v = 0.f;
    if (n >= 0 && n < HOP * (T - 1)) v = __ldg(dy + (long)b * lddy + n) * inv_env[n];
    dframes[(long)b * T * NFFT + i] = v;
}

// ------------------------------------------------------------------ generator head: mag + 1x1 conv 3 -> 64 (raw, pre-norm)
// x (B, 2, T, F) with strides; out rows (b, t, f) with leading dimension ldo
__global__ void head_conv_kernel(const float* __restrict__ x, long sb, long sc, long st, long sf, int T, int F, long M,
                                 const float* __restrict__ w /*(64,3)*/, const float* __restrict__ bias, float* __restrict__ out, long ldo) {
    long idx = (long)blockIdx.x * blockDim.x + threadIdx.x;
    long m = idx >> 4; int c4 = (int)(idx & 15) * 4;
    if (m >= M) return;
    int f = (int)(m % F); long bt = m / F; int t = (int)(bt % T); long b = bt / T;
    long o = b * sb + t * st + f * sf;
    float re = __ldg(x + o), im = __ldg(x + o + sc);
    float mag = sqrtf(re * re + im * im);
    float r[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        int n = c4 + j;
        r[j] = fmaf(__ldg(w + n * 3), mag, fmaf(__ldg(w + n * 3 + 1), re, fmaf(__ldg(w + n * 3 + 2), im, __ldg(bias + n))));
    }
    *reinterpret_cast<float4*>(out + m * ldo + c4) = make_float4(r[0], r[1], r[2], r[3]);
}

// dW (64,3) += sum_m draw[m, n] * in_j[m];  dbias[n] += sum_m draw[m, n]
__global__ void head_conv_wgrad_kernel(const float* __restrict__ x, long sb, long sc, long st, long sf, int T, int F, long M,
                                       const float* __restrict__ draw, long ldd, int rows_per_block, float* __restrict__ dw, float* __restrict__ db) {
    __shared__ float sm[4][4][64];
    int n = threadIdx.x & 63, rg = threadIdx.x >> 6;       // 256 threads: 4 row groups x 64 channels
    long m_beg = (long)blockIdx.x * rows_per_block, m_end = m_beg + rows_per_block < M ? m_beg + rows_per_block : M;
    float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
    for (long m = m_beg + rg; m < m_end; m += 4) {
        int f = (int)(m % F); long bt = m / F; int t = (int)(bt % T); long b = bt / T;
        long o = b * sb + t * st + f * sf;
        float re = __ldg(x + o), im = __ldg(x + o + sc);
        float mag = sqrtf(re * re + im * im);
        float d = __ldg(draw + m * ldd + n);
        a0 = fmaf(d, mag, a0); a1 = fmaf(d, re, a1); a2 = fmaf(d, im, a2); a3 += d;
    }
    sm[rg][0][n] = a0; sm[rg][1][n] = a1; sm[rg][2][n] = a2; sm[rg][3][n] = a3;
    __syncthreads();
    if (rg == 0) {
        float s0 = 0, s1 = 0, s2 = 0, s3 = 0;
        for (int g = 0; g < 4; ++g) { s0 += sm[g][0][n]; s1 += sm[g][1][n]; s2 += sm[g][2][n]; s3 += sm[g][3][n]; }
        atomicAdd(dw + n * 3, s0); atomicAdd(dw + n * 3 + 1, s1); atomicAdd(dw + n * 3 + 2, s2); atomicAdd(db + n, s3);
    }
}

// ------------------------------------------------------------------ (1,2) output convolutions, 64 -> NOUT (1 or 2)
// in rows (b, t, f'), f' < Fin = Fout + 1, 64 channels, optional InstanceNorm+PReLU prologue (scale/shift per (b, c)).
// out[(b,t,f), j] = bias[j] + sum_{dj<2} sum_c act(in[(b,t,f+dj), c]) * w[j, c, 0, dj].  One warp per output pixel.
template <int NOUT>
__global__ void rowdot_fwd_kernel(const float* __restrict__ in, int T, int Fout, long npix, const float* __restrict__ scale,
                                  const float* __restrict__ shift, const float* __restrict__ slope, const float* __restrict__ w,
                                  const float* __restrict__ bias, float* __restrict__ out) {
    long pix = (long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    int lane = threadIdx.x & 31;
    if (pix >= npix) return;
    int f = (int)(pix % Fout); long bt = pix / Fout; long b = bt / T;
    const int Fin = Fout + 1;
    int k = lane * 4, dj = k >> 6, c = k & 63;
    float4 v = __ldg(reinterpret_cast<const float4*>(in + (bt * Fin + f) * 64) + lane);
    float a[4] = {v.x, v.y, v.z, v.w};
    if (scale) {
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            float z = a[i] * __ldg(scale + b * 64 + c + i) + __ldg(shift + b * 64 + c + i);
            a[i] = z >= 0.f ? z : z * __ldg(slope + c + i);
        }
    }
#pragma unroll
    for (int j = 0; j < NOUT; ++j) {
        float s = 0.f;
#pragma unroll
        for (int i = 0; i < 4; ++i) s = fmaf(a[i], __ldg(w + (j * 64 + c + i) * 2 + dj), s);
        s = warp_sum(s);
        if (lane == 0) out[pix * NOUT + j] = s + __ldg(bias + j);
    }
}

// backward of the above.  dact (B,T,Fin,64) = grad wrt act(in) (overwritten); dw (NOUT,64,1,2), dbias accumulated.
// One warp per input row (b, t, f'); lane owns channels 2*lane, 2*lane+1.
template <int NOUT>
__global__ void rowdot_bwd_kernel(const float* __restrict__ in, int T, int Fout, long nrows, const float* __restrict__ scale,
                                  const float* __restrict__ shift, const float* __restrict__ slope, const float* __restrict__ w,
                                  const float* __restrict__ dout, int rows_per_warp, float* __restrict__ dact, float* __restrict__ dw,
                                  float* __restrict__ dbias) {
    __shared__ float sm[8][NOUT * 2 * 64];
    int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
    const int Fin = Fout + 1;
    float wr[NOUT][2][2];     // [j][dj][ch]
    float acc[NOUT][2][2];
    float bacc[NOUT];
#pragma unroll
    for (int j = 0; j < NOUT; ++j) {
        bacc[j] = 0.f;
#pragma unroll
        for (int dj = 0; dj < 2; ++dj)
#pragma unroll
            for (int e = 0; e < 2; ++e) { wr[j][dj][e] = __ldg(w + (j * 64 + 2 * lane + e) * 2 + dj); acc[j][dj][e] = 0.f; }
    }
    long r0 = ((long)blockIdx.x * nw + warp) * rows_per_warp;
    for (int it = 0; it < rows_per_warp; ++it) {
        long row = r0 + it;
        if (row >= nrows) break;
        int fp = (int)(row % Fin); long bt = row / Fin; long b = bt / T;
        float2 v = __ldg(reinterpret_cast<const float2*>(in + row * 64) + lane);
        float a[2] = {v.x, v.y};
        if (scale) {
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                int c = 2 * lane + e;
                float z = a[e] * __ldg(scale + b * 64 + c) + __ldg(shift + b * 64 + c);
                a[e] = z >= 0.f ? z : z * __ldg(slope + c);
            }
        }
        float g[2] = {0.f, 0.f};
#pragma unroll
        for (int j = 0; j < NOUT; ++j) {
            float d0 = fp < Fout ? __ldg(dout + (bt * Fout + fp) * NOUT + j) : 0.f;      // this row is tap dj = 0 of pixel fp
            float d1 = fp >= 1 ? __ldg(dout + (bt * Fout + fp - 1) * NOUT + j) : 0.f;    // and tap dj = 1 of pixel fp - 1
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                g[e] = fmaf(d0, wr[j][0][e], fmaf(d1, wr[j][1][e], g[e]));
                acc[j][0][e] = fmaf(d0, a[e], acc[j][0][e]);
                acc[j][1][e] = fmaf(d1, a[e], acc[j][1][e]);
            }
            if (lane == 0) bacc[j] += d0;
        }
        reinterpret_cast<float2*>(dact + row * 64)[lane] = make_float2(g[0], g[1]);
    }
#pragma unroll
    for (int j = 0; j < NOUT; ++j)
#pragma unroll
        for (int dj = 0; dj < 2; ++dj)
#pragma unroll
            for (int e = 0; e < 2; ++e) sm[warp][(j * 2 + dj) * 64 + 2 * lane + e] = acc[j][dj][e];
    __syncthreads();
    for (int i = threadIdx.x; i < NOUT * 2 * 64; i += blockDim.x) {
        float s = 0.f;
        for (int wv = 0; wv < nw; ++wv) s += sm[wv][i];
        int j = i / 128, dj = (i / 64) & 1, c = i & 63;
        atomicAdd(dw + (j * 64 + c) * 2 + dj, s);
    }
    if (lane == 0) {
#pragma unroll
        for (int j = 0; j < NOUT; ++j) atomicAdd(dbias + j, bacc[j]);
    }
}

// ------------------------------------------------------------------ recombination (mask tail + complex add)
// m1 (B*T*F) raw (1,2)-conv output of the mask branch; IN(1) scale/shift per b; PReLU(1) a1; 1x1 conv (fcw, fcb);
// PReLU with one slope per frequency; final = mask * x + cplx.
struct MaskTail { const float* scale; const float* shift; const float* a1; const float* fcw; const float* fcb; const float* slope_f; };

__global__ void recombine_kernel(const float* __restrict__ m1, MaskTail mt, const float* __restrict__ x, long sb, long sc, long st, long sf,
                                 const float* __restrict__ cplx, int T, int F, long M, float* __restrict__ fr, float* __restrict__ fi) {
    long m = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (m >= M) return;
    int f = (int)(m % F); long bt = m / F; int t = (int)(bt % T); long b = bt / T;
    float z = __ldg(m1 + m) * mt.scale[b] + mt.shift[b];
    if (z < 0.f) z *= mt.a1[0];
    float z2 = fmaf(mt.fcw[0], z, mt.fcb[0]);
    float mask = z2 >= 0.f ? z2 : z2 * __ldg(mt.slope_f + f);
    long o = b * sb + t * st + f * sf;
    float re = __ldg(x + o), im = __ldg(x + o + sc);
    float2 c = __ldg(reinterpret_cast<const float2*>(cplx) + m);
    fr[m] = fmaf(mask, re, c.x);
    fi[m] = fmaf(mask, im, c.y);
}

// backward: dfr, dfi with strides (gb, gt, gf) -> dcplx (M, 2), dz (M) = grad wrt the IN(1)+PReLU(1) output;
// dslope_f (F), dfcw, dfcb accumulated.  At z2 = 0 the slope branch, as torch's PReLU backward.
__global__ void recombine_bwd_kernel(const float* __restrict__ m1, MaskTail mt, const float* __restrict__ x, long sb, long sc, long st, long sf,
                                     const float* __restrict__ dfr, const float* __restrict__ dfi, long gb, long gt, long gf, int T, int F,
                                     long M, float* __restrict__ dcplx, float* __restrict__ dz, float* __restrict__ dslope_f,
                                     float* __restrict__ dfcw, float* __restrict__ dfcb) {
    long m = (long)blockIdx.x * blockDim.x + threadIdx.x;
    float pw = 0.f, pb = 0.f;
    if (m < M) {
        int f = (int)(m % F); long bt = m / F; int t = (int)(bt % T); long b = bt / T;
        float z = __ldg(m1 + m) * mt.scale[b] + mt.shift[b];
        if (z < 0.f) z *= mt.a1[0];
        float z2 = fmaf(mt.fcw[0], z, mt.fcb[0]);
        long o = b * sb + t * st + f * sf;
        float re = __ldg(x + o), im = __ldg(x + o + sc);
        long go = b * gb + t * gt + f * gf;
        float gr = __ldg(dfr + go), gi = __ldg(dfi + go);
        reinterpret_cast<float2*>(dcplx)[m] = make_float2(gr, gi);
        float dmask = gr * re + gi * im;
        float dz2 = dmask;
        if (!(z2 > 0.f)) { dz2 = dmask * __ldg(mt.slope_f + f); atomicAdd(dslope_f + f, dmask * z2); }
        pw = dz2 * z; pb = dz2;
        dz[m] = dz2 * mt.fcw[0];
    }
    pw = warp_sum(pw); pb = warp_sum(pb);
    if ((threadIdx.x & 31) == 0) { atomicAdd(dfcw, pw); atomicAdd(dfcb, pb); }
}

// ------------------------------------------------------------------ input gradients (differentiable front end)
// *dst += sum of v over the block (blockDim.x a multiple of 32, at most 1024); every thread of the block must call it
__device__ __forceinline__ void block_sum_atomic(float v, float* dst) {
    __shared__ float sm[32];
    v = warp_sum(v);
    if ((threadIdx.x & 31) == 0) sm[threadIdx.x >> 5] = v;
    __syncthreads();
    if (threadIdx.x == 0) {
        float s = 0.f;
        for (int w = 0; w < (int)(blockDim.x >> 5); ++w) s += sm[w];
        atomicAdd(dst, s);
    }
}

// gradient of TSCNet wrt its input x (B, 2, T, F).  final = mask x + cplx (recombine_kernel) and the head convolution reads [|x|, re, im]
// (head_conv_kernel), so with draw = the gradient of the raw head output (rows m, 64 channels) and w the head weight (64, 3):
//   dre = mask dfr + sum_n draw[m, n] (w[n, 1] + w[n, 0] re / |x|),   dim = mask dfi + sum_n draw[m, n] (w[n, 2] + w[n, 0] im / |x|).
// At |x| = 0 the magnitude term contributes 0 (the reference's autograd gives NaN there: the derivative of sqrt at 0).  The mask is
// recomputed from m1 as recombine_bwd_kernel does.  16 threads per row, 4 channels each; dx is contiguous (B, 2, T, F).
__global__ void tscnet_input_grad_kernel(const float* __restrict__ m1, MaskTail mt, const float* __restrict__ x, long sb, long sc, long st,
                                         long sf, const float* __restrict__ dfr, const float* __restrict__ dfi, long gb, long gt, long gf,
                                         const float* __restrict__ draw, long ldd, const float* __restrict__ w, int T, int F, long M,
                                         float* __restrict__ dx) {
    const long idx = (long)blockIdx.x * blockDim.x + threadIdx.x;
    const long m = idx >> 4;
    const int c4 = (int)(idx & 15) * 4;
    float s0 = 0.f, s1 = 0.f, s2 = 0.f;
    if (m < M) {
        const float4 d = __ldg(reinterpret_cast<const float4*>(draw + m * ldd + c4));
        const float dv[4] = {d.x, d.y, d.z, d.w};
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int n = c4 + j;
            s0 = fmaf(dv[j], __ldg(w + n * 3), s0);
            s1 = fmaf(dv[j], __ldg(w + n * 3 + 1), s1);
            s2 = fmaf(dv[j], __ldg(w + n * 3 + 2), s2);
        }
    }
#pragma unroll
    for (int o = 8; o > 0; o >>= 1) {           // the 16 threads of a row are 16 consecutive lanes
        s0 += __shfl_xor_sync(0xffffffffu, s0, o);
        s1 += __shfl_xor_sync(0xffffffffu, s1, o);
        s2 += __shfl_xor_sync(0xffffffffu, s2, o);
    }
    if (m >= M || c4 != 0) return;
    const int f = (int)(m % F); const long bt = m / F; const int t = (int)(bt % T); const long b = bt / T;
    float z = __ldg(m1 + m) * mt.scale[b] + mt.shift[b];
    if (z < 0.f) z *= mt.a1[0];
    const float z2 = fmaf(mt.fcw[0], z, mt.fcb[0]);
    const float mask = z2 >= 0.f ? z2 : z2 * __ldg(mt.slope_f + f);
    const long o = b * sb + t * st + f * sf;
    const float re = __ldg(x + o), im = __ldg(x + o + sc);
    const float mag = sqrtf(re * re + im * im);
    const float sm = mag > 0.f ? s0 / mag : 0.f;
    const long go = b * gb + t * gt + f * gf;
    const long q = ((b * 2) * T + t) * F + f;
    dx[q] = fmaf(mask, __ldg(dfr + go), fmaf(sm, re, s1));
    dx[q + (long)T * F] = fmaf(mask, __ldg(dfi + go), fmaf(sm, im, s2));
}

// gradient of c[b] = sqrt(L / sum x^2):  dc / dx_i = -c^3 x_i / L,  dx[b, i] (+)= -dc[b] c[b]^3 x[b, i] / L
__global__ void rms_scale_bwd_kernel(const float* __restrict__ x, long ldx, int L, const float* __restrict__ c, const float* __restrict__ dc,
                                     float* __restrict__ dx, long lddx, int accumulate) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    const int b = blockIdx.y;
    if (i >= L) return;
    const float cb = c[b];
    const float k = -dc[b] * cb * cb * cb / (float)L;
    const float v = k * __ldg(x + (long)b * ldx + i);
    float* p = dx + (long)b * lddx + i;
    *p = accumulate ? *p + v : v;
}

// adjoint of the framing + reflect padding + scaling in front of the DFT (pad_reflect_kernel, frame t = xp[100 t, 100 t + 400)).
// dframes (B*T, 400) -> g[b, j] = sum over the padded positions p that read x[b, j] (p = j + 200, p = 200 - j for j <= 200, p = 2 (L - 1) - j
// + 200 for j >= L - 201) of sum over the frames t that cover p of dframes[b, t, p - 100 t];  dx[b, j] = c[b] g[b, j] (c null: 1) and
// dc[b] += sum_j g[b, j] x[b, j] (dc optional, zeroed by the caller).  Needs L > 200 (one reflection per side) and T = L / 100 + 1.
__device__ __forceinline__ float frames_at(const float* __restrict__ df, int T, int p) {
    const int t_lo = p >= NFFT ? (p - NFFT) / HOP + 1 : 0, t_hi = min(p / HOP, T - 1);
    float s = 0.f;
    for (int t = t_lo; t <= t_hi; ++t) s += __ldg(df + (long)t * NFFT + p - t * HOP);
    return s;
}

__global__ void pad_reflect_bwd_kernel(const float* __restrict__ dframes, int T, const float* __restrict__ x, long ldx, int L,
                                       const float* __restrict__ c, float* __restrict__ dx, long lddx, float* __restrict__ dc) {
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    const int b = blockIdx.y;
    const float* df = dframes + (long)b * T * NFFT;
    float gx = 0.f;
    if (j < L) {
        float g = frames_at(df, T, j + NFFT / 2);
        if (j >= 1 && j <= NFFT / 2) g += frames_at(df, T, NFFT / 2 - j);
        if (j >= L - 1 - NFFT / 2 && j <= L - 2) g += frames_at(df, T, 2 * (L - 1) - j + NFFT / 2);
        dx[(long)b * lddx + j] = c ? c[b] * g : g;
        gx = g * __ldg(x + (long)b * ldx + j);
    }
    if (dc) block_sum_atomic(gx, dc + b);
}

// gradient of the de-normalised overlap-add y = ola(frames) / c_div (ola_kernel with c_div): dframes[b, t, k] = dy[b, n] inv_env[n] / c_div[b]
// (n = 100 t + k - 200, zero outside the trimmed range) and dc[b] += -sum_n dy[b, n] y[b, n] / c_div[b] (dc optional, zeroed by the caller)
__global__ void ola_div_bwd_kernel(const float* __restrict__ dy, long lddy, int T, const float* __restrict__ inv_env, const float* __restrict__ c_div,
                                   const float* __restrict__ y, long ldy, float* __restrict__ dframes, float* __restrict__ dc) {
    const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    const int b = blockIdx.y;
    const int Lout = HOP * (T - 1);
    const float cb = c_div[b];
    if (i < (long)T * NFFT) {
        const int t = (int)(i / NFFT), k = (int)(i % NFFT);
        const int n = t * HOP + k - NFFT / 2;
        float v = 0.f;
        if (n >= 0 && n < Lout) v = __ldg(dy + (long)b * lddy + n) * inv_env[n] / cb;
        dframes[(long)b * T * NFFT + i] = v;
    }
    if (dc) {
        const float p = i < Lout ? __ldg(dy + (long)b * lddy + i) * __ldg(y + (long)b * ldy + i) : 0.f;
        block_sum_atomic(-p / cb, dc + b);
    }
}

}  // namespace

// ------------------------------------------------------------------ C ABI
// any output may be null; inv_env (100 (T - 1) samples) needs T >= 2
CMGAN_API int cmgan_stft_tables(float* fwd_basis, float* inv_basis, int T, float* inv_env, float* inv_tail, void* stream) {
    CMGAN_REQUIRE(!inv_env || T >= 2, "cmgan_stft_tables: inv_env needs T >= 2 (T=%d)", T);
    if (!fwd_basis && !inv_basis && !inv_env && !inv_tail) return 0;
    stft_tables_kernel<<<128, 256, 0, (cudaStream_t)stream>>>(fwd_basis, inv_basis, T, inv_env, inv_tail);
    return cmgan_check_launch("stft_tables_kernel");
}

int cmgan_rms_scale_frames(const float* x, long long ldx, int B, int L, const int* lengths, float* c, int* tlen, cudaStream_t st) {
    CMGAN_REQUIRE(x && c && lengths && tlen && L > 0, "cmgan_rms_scale_frames: bad arguments");
    if (B == 0) return 0;
    rms_scale_kernel<true><<<B, 256, 0, st>>>(x, ldx, L, c, lengths, tlen);
    return cmgan_check_launch("rms_scale_kernel");
}

int cmgan_pad_wrap_reflect_fold(const float* x, long long ldx, int B, int L, int k, int S, int seg0, int hop, const float* c, float* xp,
                                int Lp, cudaStream_t st) {
    CMGAN_REQUIRE(x && xp && k > 0 && seg0 >= 0 && S > NFFT / 2 && hop > 0 && hop <= S && Lp >= S + NFFT &&
                      (long long)(seg0 + k - 1) * hop + S <= 2LL * L,
                  "cmgan_pad_wrap_reflect_fold: need S > 200, 0 < hop <= S, Lp >= S + 400 and (seg0 + k - 1) hop + S <= 2 L (L=%d k=%d S=%d "
                  "seg0=%d hop=%d Lp=%d)", L, k, S, seg0, hop, Lp);
    if (B == 0) return 0;
    dim3 grid(cdiv(Lp, 256), B * k);
    pad_wrap_reflect_kernel<true><<<grid, 256, 0, st>>>(x, ldx, L, nullptr, k, S, seg0, hop, c, xp, Lp);
    return cmgan_check_launch("pad_wrap_reflect_kernel");
}

int cmgan_ola_fold(const float* frames, int rows, int T, int k, const float* inv_env, const float* c_div, float* y, long long ldy, int L,
                   cudaStream_t st) {
    CMGAN_REQUIRE(frames && inv_env && y && T >= 2 && k > 0 && rows % k == 0, "cmgan_ola_fold: bad arguments");
    if (rows == 0) return 0;
    dim3 grid(cdiv((long)HOP * (T - 1), 256), rows);
    ola_kernel<true><<<grid, 256, 0, st>>>(frames, T, inv_env, c_div, y, ldy, k, L);
    return cmgan_check_launch("ola_kernel");
}

int cmgan_ola_ragged_lengths(const float* frames, int B, int T, const int* tlen, const int* lengths, int L, const float* inv_env,
                             const float* inv_tail, const float* c_div, float* y, long long ldy, cudaStream_t st) {
    CMGAN_REQUIRE(frames && tlen && lengths && inv_env && inv_tail && y && T >= 2, "cmgan_ola_ragged_lengths: bad arguments");
    if (B == 0) return 0;
    dim3 grid(cdiv((long)HOP * (T - 1), 256), B);
    ola_ragged_kernel<true><<<grid, 256, 0, st>>>(frames, T, tlen, inv_env, inv_tail, c_div, y, ldy, lengths, L);
    return cmgan_check_launch("ola_ragged_kernel");
}

CMGAN_API int cmgan_rms_scale(const float* x, long long ldx, int B, int L, float* c, void* stream) {
    CMGAN_REQUIRE(x && c && L > 0, "cmgan_rms_scale: bad arguments");
    if (B == 0) return 0;
    rms_scale_kernel<false><<<B, 256, 0, (cudaStream_t)stream>>>(x, ldx, L, c, nullptr, nullptr);
    return cmgan_check_launch("rms_scale_kernel");
}

// c[b] = sqrt(L_b / sum_{i < L_b} x[b, i]^2), L_b = lengths[b] clamped to [0, L]
CMGAN_API int cmgan_rms_scale_ragged(const float* x, long long ldx, int B, int L, const int* lengths, float* c, void* stream) {
    CMGAN_REQUIRE(x && c && lengths && L > 0, "cmgan_rms_scale_ragged: bad arguments");
    if (B == 0) return 0;
    rms_scale_kernel<true><<<B, 256, 0, (cudaStream_t)stream>>>(x, ldx, L, c, lengths, nullptr);
    return cmgan_check_launch("rms_scale_kernel");
}

// xp (B, Lp): utterance b wrap-padded to a multiple of 100, reflect-padded by 200 each side, scaled by c[b] (may be null), zero beyond;
// Lp >= ceil(L / 100) * 100 + 400 covers every utterance
CMGAN_API int cmgan_pad_wrap_reflect_ragged(const float* x, long long ldx, int B, int L, const int* lengths, const float* c, float* xp, int Lp,
                                            void* stream) {
    CMGAN_REQUIRE(x && xp && lengths && L > 0 && Lp >= (L + HOP - 1) / HOP * HOP + NFFT,
                  "cmgan_pad_wrap_reflect_ragged: need Lp >= ceil(L / 100) * 100 + 400 (L=%d Lp=%d)", L, Lp);
    if (B == 0) return 0;
    dim3 grid(cdiv(Lp, 256), B);
    pad_wrap_reflect_kernel<false><<<grid, 256, 0, (cudaStream_t)stream>>>(x, ldx, L, lengths, 1, 0, 0, 0, c, xp, Lp);
    return cmgan_check_launch("pad_wrap_reflect_kernel");
}

// xp (B, Lp): reflect-padded (200 each side) and scaled by c[b] (c may be null); Lp >= L + 400, zero filled beyond
CMGAN_API int cmgan_pad_reflect(const float* x, long long ldx, int B, int L, const float* c, float* xp, int Lp, void* stream) {
    CMGAN_REQUIRE(x && xp && L > 200 && Lp >= L + 400, "cmgan_pad_reflect: need L > 200 and Lp >= L + 400 (L=%d Lp=%d)", L, Lp);
    if (B == 0) return 0;
    dim3 grid(cdiv(Lp, 256), B);
    pad_reflect_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(x, ldx, L, c, xp, Lp);
    return cmgan_check_launch("pad_reflect_kernel");
}

CMGAN_API int cmgan_compress(const float* S, int B, int T, float* X, void* stream) {
    CMGAN_REQUIRE(S && X, "cmgan_compress: null pointer");
    long total = (long)B * T * NF;
    if (total == 0) return 0;
    compress_kernel<<<cdiv(total, 256), 256, 0, (cudaStream_t)stream>>>(S, total, T, X);
    return cmgan_check_launch("compress_kernel");
}

CMGAN_API int cmgan_uncompress(const float* re, const float* im, long long sb, long long st, long long sf, int B, int T, float* U, void* stream) {
    CMGAN_REQUIRE(re && im && U, "cmgan_uncompress: null pointer");
    long total = (long)B * T * NF;
    if (total == 0) return 0;
    uncompress_kernel<<<cdiv(total, 256), 256, 0, (cudaStream_t)stream>>>(re, im, sb, st, sf, total, T, U);
    return cmgan_check_launch("uncompress_kernel");
}

CMGAN_API int cmgan_uncompress_bwd(const float* re, const float* im, long long sb, long long st, long long sf, int B, int T, const float* dU,
                                   float* dre, float* dim_, int accumulate, void* stream) {
    CMGAN_REQUIRE(re && im && dU && dre && dim_, "cmgan_uncompress_bwd: null pointer");
    long total = (long)B * T * NF;
    if (total == 0) return 0;
    uncompress_bwd_kernel<<<cdiv(total, 256), 256, 0, (cudaStream_t)stream>>>(re, im, sb, st, sf, total, T, dU, dre, dim_, accumulate);
    return cmgan_check_launch("uncompress_bwd_kernel");
}

CMGAN_API int cmgan_ola(const float* frames, int B, int T, const float* inv_env, const float* c_div, float* y, long long ldy, void* stream) {
    CMGAN_REQUIRE(frames && inv_env && y && T >= 2, "cmgan_ola: bad arguments");
    if (B == 0) return 0;
    dim3 grid(cdiv((long)HOP * (T - 1), 256), B);
    ola_kernel<false><<<grid, 256, 0, (cudaStream_t)stream>>>(frames, T, inv_env, c_div, y, ldy, 1, 0);
    return cmgan_check_launch("ola_kernel");
}

CMGAN_API int cmgan_crossfade_table(float* w, int overlap, void* stream) {
    CMGAN_REQUIRE(w && overlap > 0, "cmgan_crossfade_table: need w and overlap > 0 (overlap=%d)", overlap);
    crossfade_table_kernel<<<cdiv(overlap, 256), 256, 0, (cudaStream_t)stream>>>(w, overlap);
    return cmgan_check_launch("crossfade_table_kernel");
}

CMGAN_API int cmgan_crossfade(const float* y, int rows, int j0, int k, int S, int overlap, const float* w, float* out, long long L, void* stream) {
    CMGAN_REQUIRE(y && w && out, "cmgan_crossfade: null pointer");
    CMGAN_REQUIRE(overlap > 0 && 2LL * overlap <= S, "cmgan_crossfade: need 0 < overlap <= S / 2 (S=%d overlap=%d)", S, overlap);
    CMGAN_REQUIRE(rows > 0 && j0 >= 0 && (long long)j0 + rows <= k, "cmgan_crossfade: need rows > 0 and 0 <= j0, j0 + rows <= k (rows=%d j0=%d k=%d)",
                  rows, j0, k);
    const long long H = S - overlap;
    const long long lo = k == 1 ? 1 : (k - 1) * H + overlap;
    CMGAN_REQUIRE(L <= (1LL << 30) && L >= lo && L <= (k - 1) * H + S,
                  "cmgan_crossfade: L=%lld must lie in [%lld, (k - 1) H + S = %lld] (the last window's crossfade inside the clip) and be at most "
                  "2^30 (k=%d H=%lld S=%d)", L, lo, (k - 1) * H + S, k, H, S);
    const long long n0 = (long long)j0 * H, n1 = j0 + rows == k ? L : (j0 + rows) * H + overlap;
    crossfade_kernel<<<cdiv(n1 - n0, 256), 256, 0, (cudaStream_t)stream>>>(y, rows, j0, k, S, overlap, w, out, (int)n0, (int)n1);
    return cmgan_check_launch("crossfade_kernel");
}

CMGAN_API int cmgan_ola_ragged(const float* frames, int B, int T, const int* tlen, const float* inv_env, const float* inv_tail, const float* c_div,
                               float* y, long long ldy, void* stream) {
    CMGAN_REQUIRE(frames && tlen && inv_env && inv_tail && y && T >= 2, "cmgan_ola_ragged: bad arguments");
    if (B == 0) return 0;
    dim3 grid(cdiv((long)HOP * (T - 1), 256), B);
    ola_ragged_kernel<false><<<grid, 256, 0, (cudaStream_t)stream>>>(frames, T, tlen, inv_env, inv_tail, c_div, y, ldy, nullptr, 0);
    return cmgan_check_launch("ola_ragged_kernel");
}

CMGAN_API int cmgan_ola_bwd(const float* dy, long long lddy, int B, int T, const float* inv_env, float* dframes, void* stream) {
    CMGAN_REQUIRE(dy && inv_env && dframes && T >= 2, "cmgan_ola_bwd: bad arguments");
    if (B == 0) return 0;
    dim3 grid(cdiv((long)T * NFFT, 256), B);
    ola_bwd_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(dy, lddy, T, inv_env, dframes);
    return cmgan_check_launch("ola_bwd_kernel");
}

CMGAN_API int cmgan_head_conv(const float* x, long long sb, long long sc, long long st, long long sf, int B, int T, int F, const float* w,
                              const float* bias, float* out, long long ldo, void* stream) {
    CMGAN_REQUIRE(x && w && bias && out && ldo % 4 == 0, "cmgan_head_conv: bad arguments");
    long M = (long)B * T * F;
    if (M == 0) return 0;
    head_conv_kernel<<<cdiv(M * 16, 256), 256, 0, (cudaStream_t)stream>>>(x, sb, sc, st, sf, T, F, M, w, bias, out, ldo);
    return cmgan_check_launch("head_conv_kernel");
}

CMGAN_API int cmgan_head_conv_wgrad(const float* x, long long sb, long long sc, long long st, long long sf, int B, int T, int F,
                                    const float* draw, long long ldd, float* dw, float* db, void* stream) {
    CMGAN_REQUIRE(x && draw && dw && db, "cmgan_head_conv_wgrad: null pointer");
    long M = (long)B * T * F;
    if (M == 0) return 0;
    const int rpb = 512;
    head_conv_wgrad_kernel<<<cdiv(M, rpb), 256, 0, (cudaStream_t)stream>>>(x, sb, sc, st, sf, T, F, M, draw, ldd, rpb, dw, db);
    return cmgan_check_launch("head_conv_wgrad_kernel");
}

CMGAN_API int cmgan_rowdot_fwd(const float* in, int B, int T, int Fout, int nout, const float* scale, const float* shift, const float* slope,
                               const float* w, const float* bias, float* out, void* stream) {
    CMGAN_REQUIRE(in && w && bias && out && (nout == 1 || nout == 2), "cmgan_rowdot_fwd: bad arguments");
    long npix = (long)B * T * Fout;
    if (npix == 0) return 0;
    if (nout == 1) rowdot_fwd_kernel<1><<<cdiv(npix, 8), 256, 0, (cudaStream_t)stream>>>(in, T, Fout, npix, scale, shift, slope, w, bias, out);
    else rowdot_fwd_kernel<2><<<cdiv(npix, 8), 256, 0, (cudaStream_t)stream>>>(in, T, Fout, npix, scale, shift, slope, w, bias, out);
    return cmgan_check_launch("rowdot_fwd_kernel");
}

CMGAN_API int cmgan_rowdot_bwd(const float* in, int B, int T, int Fout, int nout, const float* scale, const float* shift, const float* slope,
                               const float* w, const float* dout, float* dact, float* dw, float* dbias, void* stream) {
    CMGAN_REQUIRE(in && w && dout && dact && dw && dbias && (nout == 1 || nout == 2), "cmgan_rowdot_bwd: bad arguments");
    long nrows = (long)B * T * (Fout + 1);
    if (nrows == 0) return 0;
    const int rpw = 32;
    if (nout == 1) rowdot_bwd_kernel<1><<<cdiv(nrows, 8 * rpw), 256, 0, (cudaStream_t)stream>>>(in, T, Fout, nrows, scale, shift, slope, w, dout, rpw, dact, dw, dbias);
    else rowdot_bwd_kernel<2><<<cdiv(nrows, 8 * rpw), 256, 0, (cudaStream_t)stream>>>(in, T, Fout, nrows, scale, shift, slope, w, dout, rpw, dact, dw, dbias);
    return cmgan_check_launch("rowdot_bwd_kernel");
}

CMGAN_API int cmgan_recombine(const float* m1, const float* in_scale, const float* in_shift, const float* a1, const float* fcw, const float* fcb,
                              const float* slope_f, const float* x, long long sb, long long sc, long long st, long long sf, const float* cplx,
                              int B, int T, int F, float* fr, float* fi, void* stream) {
    CMGAN_REQUIRE(m1 && in_scale && in_shift && a1 && fcw && fcb && slope_f && x && cplx && fr && fi, "cmgan_recombine: null pointer");
    long M = (long)B * T * F;
    if (M == 0) return 0;
    MaskTail mt{in_scale, in_shift, a1, fcw, fcb, slope_f};
    recombine_kernel<<<cdiv(M, 256), 256, 0, (cudaStream_t)stream>>>(m1, mt, x, sb, sc, st, sf, cplx, T, F, M, fr, fi);
    return cmgan_check_launch("recombine_kernel");
}

CMGAN_API int cmgan_recombine_bwd(const float* m1, const float* in_scale, const float* in_shift, const float* a1, const float* fcw,
                                  const float* fcb, const float* slope_f, const float* x, long long sb, long long sc, long long st, long long sf,
                                  const float* dfr, const float* dfi, long long gb, long long gt, long long gf, int B, int T, int F,
                                  float* dcplx, float* dz, float* dslope_f, float* dfcw, float* dfcb, void* stream) {
    CMGAN_REQUIRE(m1 && in_scale && in_shift && a1 && fcw && fcb && slope_f && x && dfr && dfi && dcplx && dz && dslope_f && dfcw && dfcb,
                  "cmgan_recombine_bwd: null pointer");
    long M = (long)B * T * F;
    if (M == 0) return 0;
    MaskTail mt{in_scale, in_shift, a1, fcw, fcb, slope_f};
    recombine_bwd_kernel<<<cdiv(M, 256), 256, 0, (cudaStream_t)stream>>>(m1, mt, x, sb, sc, st, sf, dfr, dfi, gb, gt, gf, T, F, M, dcplx, dz,
                                                                        dslope_f, dfcw, dfcb);
    return cmgan_check_launch("recombine_bwd_kernel");
}

// Y = X |X|^p with explicit element strides (utils.power_compress / power_uncompress as free functions)
CMGAN_API int cmgan_power_law(const float* re, const float* im, long long i0, long long i1, long long i2, float* ore, float* oim, long long o0,
                              long long o1, long long o2, int d0, int d1, int d2, float p, void* stream) {
    CMGAN_REQUIRE(re && im && ore && oim, "cmgan_power_law: null pointer");
    long n = (long)d0 * d1 * d2;
    if (n == 0) return 0;
    power_law_kernel<<<cdiv(n, 256), 256, 0, (cudaStream_t)stream>>>(re, im, i0, i1, i2, ore, oim, o0, o1, o2, d1, d2, n, 0.5f * p);
    return cmgan_check_launch("power_law_kernel");
}

CMGAN_API int cmgan_power_law_bwd(const float* re, const float* im, long long i0, long long i1, long long i2, const float* gre, const float* gim,
                                  long long o0, long long o1, long long o2, float* dre, float* dim_, long long q0, long long q1, long long q2,
                                  int d0, int d1, int d2, float p, void* stream) {
    CMGAN_REQUIRE(re && im && gre && gim && dre && dim_, "cmgan_power_law_bwd: null pointer");
    long n = (long)d0 * d1 * d2;
    if (n == 0) return 0;
    power_law_bwd_kernel<<<cdiv(n, 256), 256, 0, (cudaStream_t)stream>>>(re, im, i0, i1, i2, gre, gim, o0, o1, o2, dre, dim_, q0, q1, q2, d1, d2, n, p);
    return cmgan_check_launch("power_law_bwd_kernel");
}

// ------------------------------------------------------------------ input gradients (differentiable front end)
// dx (B, 2, T, F) contiguous = the gradient of TSCNet wrt its input x (see tscnet_input_grad_kernel); draw (M, ldd) 16-byte aligned, ldd % 4 == 0
CMGAN_API int cmgan_tscnet_input_grad(const float* m1, const float* in_scale, const float* in_shift, const float* a1, const float* fcw,
                                      const float* fcb, const float* slope_f, const float* x, long long sb, long long sc, long long st,
                                      long long sf, const float* dfr, const float* dfi, long long gb, long long gt, long long gf,
                                      const float* draw, long long ldd, const float* w, int B, int T, int F, float* dx, void* stream) {
    CMGAN_REQUIRE(m1 && in_scale && in_shift && a1 && fcw && fcb && slope_f && x && dfr && dfi && draw && w && dx,
                  "cmgan_tscnet_input_grad: null pointer");
    CMGAN_REQUIRE(ldd >= 64 && ldd % 4 == 0 && ((uintptr_t)draw & 15) == 0,
                  "cmgan_tscnet_input_grad: draw needs 16-byte alignment and ldd >= 64, ldd %% 4 == 0 (ldd=%lld)", ldd);
    CMGAN_REQUIRE(B >= 0 && T >= 0 && F >= 0, "cmgan_tscnet_input_grad: negative size (B=%d T=%d F=%d)", B, T, F);
    const long M = (long)B * T * F;
    if (M == 0) return 0;
    MaskTail mt{in_scale, in_shift, a1, fcw, fcb, slope_f};
    tscnet_input_grad_kernel<<<cdiv(M * 16, 256), 256, 0, (cudaStream_t)stream>>>(m1, mt, x, sb, sc, st, sf, dfr, dfi, gb, gt, gf, draw, ldd, w,
                                                                                  T, F, M, dx);
    return cmgan_check_launch("tscnet_input_grad_kernel");
}

// dx[b, i] (+)= -dc[b] c[b]^3 x[b, i] / L: the gradient of cmgan_rms_scale
CMGAN_API int cmgan_rms_scale_bwd(const float* x, long long ldx, int B, int L, const float* c, const float* dc, float* dx, long long lddx,
                                  int accumulate, void* stream) {
    CMGAN_REQUIRE(x && c && dc && dx, "cmgan_rms_scale_bwd: null pointer");
    CMGAN_REQUIRE(B >= 0 && L > 0 && ldx >= L && lddx >= L, "cmgan_rms_scale_bwd: need L > 0 and row strides >= L (L=%d ldx=%lld lddx=%lld)",
                  L, ldx, lddx);
    if (B == 0) return 0;
    dim3 grid(cdiv(L, 256), B);
    rms_scale_bwd_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(x, ldx, L, c, dc, dx, lddx, accumulate);
    return cmgan_check_launch("rms_scale_bwd_kernel");
}

// adjoint of cmgan_pad_reflect + the framing of the DFT: dframes (B*T, 400), T = L / 100 + 1 -> dx (B, L) = c g (c may be null: 1) and
// dc[b] += sum_j g[b, j] x[b, j] (dc may be null; the caller zeroes it)
CMGAN_API int cmgan_pad_reflect_bwd(const float* dframes, int B, int T, const float* x, long long ldx, int L, const float* c, float* dx,
                                    long long lddx, float* dc, void* stream) {
    CMGAN_REQUIRE(dframes && x && dx, "cmgan_pad_reflect_bwd: null pointer");
    CMGAN_REQUIRE(B >= 0 && L > NFFT / 2 && T == L / HOP + 1, "cmgan_pad_reflect_bwd: need L > 200 and T = L / 100 + 1 (L=%d T=%d)", L, T);
    CMGAN_REQUIRE(ldx >= L && lddx >= L, "cmgan_pad_reflect_bwd: row strides must be >= L (L=%d ldx=%lld lddx=%lld)", L, ldx, lddx);
    if (B == 0) return 0;
    dim3 grid(cdiv(L, 256), B);
    pad_reflect_bwd_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(dframes, T, x, ldx, L, c, dx, lddx, dc);
    return cmgan_check_launch("pad_reflect_bwd_kernel");
}

// gradient of cmgan_ola with c_div: dframes (B*T, 400) from dy / c_div, and dc[b] += -sum_n dy[b, n] y[b, n] / c_div[b] (y the forward output;
// dc may be null; the caller zeroes it)
CMGAN_API int cmgan_ola_div_bwd(const float* dy, long long lddy, int B, int T, const float* inv_env, const float* c_div, const float* y,
                                long long ldy, float* dframes, float* dc, void* stream) {
    CMGAN_REQUIRE(dy && inv_env && c_div && y && dframes, "cmgan_ola_div_bwd: null pointer");
    CMGAN_REQUIRE(B >= 0 && T >= 2 && lddy >= (long long)HOP * (T - 1) && ldy >= (long long)HOP * (T - 1),
                  "cmgan_ola_div_bwd: need T >= 2 and row strides >= 100 (T - 1) (T=%d lddy=%lld ldy=%lld)", T, lddy, ldy);
    if (B == 0) return 0;
    dim3 grid(cdiv((long)T * NFFT, 256), B);
    ola_div_bwd_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(dy, lddy, T, inv_env, c_div, y, ldy, dframes, dc);
    return cmgan_check_launch("ola_div_bwd_kernel");
}

// ------------------------------------------------------------------ training batch cut (dataloader.py:32-49) on the device
namespace {

__global__ void cut_batch_kernel(const float* __restrict__ corpus, const long long* __restrict__ offsets, const int* __restrict__ lengths,
                                 const int* __restrict__ starts, int cut_len, float* __restrict__ out, long long ldo) {
    const int b = blockIdx.y;
    const long long off = offsets[b];
    const int len = lengths[b];
    const int start = len >= cut_len ? min(max(starts[b], 0), len - cut_len) : 0;
    float* o = out + (long long)b * ldo;
    for (int n = blockIdx.x * blockDim.x + threadIdx.x; n < cut_len; n += gridDim.x * blockDim.x) {
        float v = 0.f;
        if (len > 0) v = len < cut_len ? corpus[off + n % len] : corpus[off + start + n];
        o[n] = v;
    }
}

}  // namespace

// out[b, :cut_len] from utterance b = corpus[offsets[b] : offsets[b] + lengths[b]]: shorter utterances repeat whole and end with their first
// cut_len % len samples, longer ones give cut_len samples from starts[b] clamped to [0, len - cut_len]; len <= 0 gives zeros
CMGAN_API int cmgan_cut_batch(const float* corpus, const long long* offsets, const int* lengths, const int* starts, int B, int cut_len, float* out,
                              long long ldo, void* stream) {
    CMGAN_REQUIRE(corpus && offsets && lengths && starts && out, "cmgan_cut_batch: null pointer");
    CMGAN_REQUIRE(B > 0 && cut_len > 0, "cmgan_cut_batch: B and cut_len must be positive (B=%d cut_len=%d)", B, cut_len);
    CMGAN_REQUIRE(ldo >= cut_len, "cmgan_cut_batch: ldo=%lld is shorter than cut_len=%d", ldo, cut_len);
    CMGAN_REQUIRE(B <= 65535, "cmgan_cut_batch: B=%d exceeds 65535 rows", B);
    dim3 grid(min(cdiv(cut_len, 256), 1024), B);
    cut_batch_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(corpus, offsets, lengths, starts, cut_len, out, ldo);
    return cmgan_check_launch("cut_batch_kernel");
}
