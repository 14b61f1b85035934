// PESQ-free quality metrics of the reference's scoring tool on the GPU (reference src/tools/compute_metrics.py): segmental SNR
// (compute_metrics.py:350-397) and STOI (:400-471 with thirdoct :474-519, stdft :522-545, removeSilentFrames :548-583, taa_corr :586-599).
// Everything is float64 like the numpy reference (tiny work: what matters is that 824 test files can be scored without leaving the GPU);
// intermediate sizes that depend on the data (number of non-silent frames) stay on the device -- every kernel is launched over the
// worst case and exits early -- so the entry points never synchronise.
#include <cstdlib>

#include "common.cuh"
#include "resample.cuh"
#include "../../include/cmgan_b200.h"

namespace {

constexpr int NF = 256, HOPF = 128, NFFT = 512, NBIN = 257, NBAND = 15, NSEG = 30;

__device__ double block_sum_d(double v, double* sm) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    __syncthreads();
    if ((threadIdx.x & 31) == 0) sm[threadIdx.x >> 5] = v;
    __syncthreads();
    double t = 0.0;
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) t += sm[w];
    return t;
}

// numpy's minimum / maximum: NaN when either operand is NaN (CUDA's fmin / fmax return the other operand).  The reference clips and
// floors with NaN-propagating operations, so a silent or non-finite processed signal scores NaN there and must score NaN here too.
__device__ __forceinline__ double np_min(double a, double b) { return (isnan(a) || isnan(b)) ? a + b : fmin(a, b); }
__device__ __forceinline__ double np_max(double a, double b) { return (isnan(a) || isnan(b)) ? a + b : fmax(a, b); }

// ---- segmental SNR: one block per frame; out[0] += clipped frame value / nfr
__global__ void ssnr_kernel(const double* __restrict__ c, const double* __restrict__ p, int W, int skip, int nfr, double* __restrict__ out) {
    __shared__ double sm[32];
    const int f = blockIdx.x;
    const long s0 = (long)f * skip;
    const double PI = 3.14159265358979323846;
    double se = 0.0, ne = 0.0;
    for (int i = threadIdx.x; i < W; i += blockDim.x) {
        const double w = 0.5 * (1.0 - cos(2.0 * PI * (double)(i + 1) / (double)(W + 1)));
        const double a = c[s0 + i] * w, b = p[s0 + i] * w;
        se += a * a; ne += (a - b) * (a - b);
    }
    se = block_sum_d(se, sm);
    ne = block_sum_d(ne, sm);
    if (threadIdx.x == 0) {
        const double eps = 2.220446049250313e-16;
        double v = 10.0 * log10(se / (ne + eps) + eps);
        v = np_min(np_max(v, -10.0), 35.0);
        atomicAdd(out, v / (double)nfr);
    }
}

__device__ __forceinline__ double hann_inner(int i) {      // scipy.signal.windows.hann(N + 2)[1 : N + 1], N = 256 (symmetric window of 258 points)
    const double PI = 3.14159265358979323846;
    return 0.5 - 0.5 * cos(2.0 * PI * (double)(i + 1) / 257.0);
}

// ---- frame levels of the clean signal (removeSilentFrames): frame j covers samples j K - 1 .. j K + N - 2 (the reference's index shift; index -1 wraps)
__global__ void frame_level_kernel(const double* __restrict__ x, long len, int nframes, double* __restrict__ lev) {
    __shared__ double sm[32];
    const int j = blockIdx.x;
    if (j >= nframes) return;
    double e = 0.0;
    for (int i = threadIdx.x; i < NF; i += blockDim.x) {
        long idx = (long)j * HOPF - 1 + i;
        if (idx < 0) idx += len;
        const double v = x[idx] * hann_inner(i);
        e += v * v;
    }
    e = block_sum_d(e, sm);
    if (threadIdx.x == 0) lev[j] = 20.0 * log10(sqrt(e) / 16.0);       // / sqrt(N), N = 256
}

// one block: max level, keep mask, compaction map.  kept[c] = source frame of the c-th kept frame; cnt[0] = number kept.  Fully silent
// frames (level -inf) lie below the -1e300 start and are dropped; a NaN level makes the maximum NaN (np.max) and then no frame is kept.
__global__ void silent_mask_kernel(const double* __restrict__ lev, int nframes, double dyn, int* __restrict__ kept, int* __restrict__ cnt) {
    __shared__ double smx[32];
    __shared__ int soff;
    double m = -1e300;
    for (int j = threadIdx.x; j < nframes; j += blockDim.x) m = np_max(m, lev[j]);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = np_max(m, __shfl_xor_sync(0xffffffffu, m, o));
    if ((threadIdx.x & 31) == 0) smx[threadIdx.x >> 5] = m;
    if (threadIdx.x == 0) soff = 0;
    __syncthreads();
    m = smx[0];
    for (int w = 1; w < (int)(blockDim.x >> 5); ++w) m = np_max(m, smx[w]);
    // ordered compaction, 1024 frames per pass (one thread per frame, warp ballots + a serial pass over the 32 warp totals)
    __shared__ int wtot[32];
    for (int base = 0; base < nframes; base += blockDim.x) {
        const int j = base + threadIdx.x;
        const bool k = j < nframes && (lev[j] - m + dyn) > 0.0;
        const unsigned bal = __ballot_sync(0xffffffffu, k);
        const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
        if (lane == 0) wtot[w] = __popc(bal);
        __syncthreads();
        int before = soff;
        for (int i = 0; i < w; ++i) before += wtot[i];
        if (k) kept[before + __popc(bal & ((1u << lane) - 1u))] = j;
        __syncthreads();
        if (threadIdx.x == 0) { int t = 0; for (int i = 0; i < (int)(blockDim.x >> 5); ++i) t += wtot[i]; soff += t; }
        __syncthreads();
    }
    if (threadIdx.x == 0) cnt[0] = soff;
}

// overlap-add of the kept, windowed frames back to back (gather form): output sample o gets slots c = o / K - 1 and o / K
__global__ void compact_kernel(const double* __restrict__ x, const double* __restrict__ y, const int* __restrict__ kept, const int* __restrict__ cnt,
                               double* __restrict__ xs, double* __restrict__ ys, long max_out) {
    const long o = (long)blockIdx.x * blockDim.x + threadIdx.x;
    const int count = cnt[0];
    const long len_out = count > 0 ? (long)(count - 1) * HOPF + NF : 0;
    if (o >= max_out) return;
    if (o >= len_out) { xs[o] = 0.0; ys[o] = 0.0; return; }
    double ax = 0.0, ay = 0.0;
    const int c1 = (int)(o / HOPF);
#pragma unroll
    for (int d = 0; d < 2; ++d) {
        const int c = c1 - d;
        if (c < 0 || c >= count) continue;
        const int i = (int)(o - (long)c * HOPF);
        if (i >= NF) continue;
        const long src = (long)kept[c] * HOPF + i;
        const double w = hann_inner(i);
        ax += x[src] * w; ay += y[src] * w;
    }
    xs[o] = ax; ys[o] = ay;
}

// ---- third-octave band envelopes: X[band, frame] = sqrt(sum_{bins of band} |DFT_512(frame * hann)|^2).  Block = one frame of one signal;
// the 257 bins are computed directly (256-term sums in float64) and folded into the 15 bands through shared memory.
__global__ void band_env_kernel(const double* __restrict__ xs, const double* __restrict__ ys, const int* __restrict__ cnt, const int* __restrict__ band_lo,
                                const int* __restrict__ band_hi, double* __restrict__ X, double* __restrict__ Y, int max_frames) {
    __shared__ double fr[NF];
    __shared__ double mag2[NBIN];
    const int m = blockIdx.x, which = blockIdx.y;
    const int nfr = cnt[0] - 1;                       // int((len - N) / K) with len = (count - 1) K + N
    if (m >= nfr) return;
    const double* s = which ? ys : xs;
    const double PI = 3.14159265358979323846;
    double wsum = 0.0;
    for (int i = 0; i < NF; ++i) wsum += hann_inner(i);          // scipy's stft scales by 1 / sum(window)
    for (int i = threadIdx.x; i < NF; i += blockDim.x) fr[i] = s[(long)m * HOPF + i] * hann_inner(i);
    __syncthreads();
    for (int k = threadIdx.x; k < NBIN; k += blockDim.x) {
        double re = 0.0, im = 0.0;
        for (int i = 0; i < NF; ++i) {
            const int ph = (k * i) & (NFFT - 1);
            double sn, cs;
            sincos(2.0 * PI * (double)ph / (double)NFFT, &sn, &cs);
            re += fr[i] * cs; im -= fr[i] * sn;
        }
        re /= wsum; im /= wsum;
        mag2[k] = re * re + im * im;
    }
    __syncthreads();
    if (threadIdx.x < NBAND) {
        double e = 0.0;
        for (int k = band_lo[threadIdx.x]; k < band_hi[threadIdx.x]; ++k) e += mag2[k];
        (which ? Y : X)[(long)threadIdx.x * max_frames + m] = sqrt(e);
    }
}

// ---- intermediate intelligibility of one 30-frame segment (all 15 bands), accumulated into out[0] (sum) and out[1] (count)
__global__ void stoi_segment_kernel(const double* __restrict__ X, const double* __restrict__ Y, const int* __restrict__ cnt, int max_frames,
                                    double* __restrict__ out) {
    const int nfr = cnt[0] - 1;
    const int m = blockIdx.x + NSEG - 1;
    if (m >= nfr) return;
    __shared__ double part[NBAND];
    const int j = threadIdx.x;
    if (j < NBAND) {
        const double* xr = X + (long)j * max_frames + (m - NSEG + 1);
        const double* yr = Y + (long)j * max_frames + (m - NSEG + 1);
        double sx = 0.0, sy = 0.0;
        for (int n = 0; n < NSEG; ++n) { sx += xr[n] * xr[n]; sy += yr[n] * yr[n]; }
        const double alpha = sqrt(sx / sy);
        const double c = 5.623413251903491;          // 10^(15/20)
        double yp[NSEG];
        double mx = 0.0, my = 0.0;
        // a processed band that is zero over the segment gives alpha = inf and 0 * inf = NaN: the segment, like the reference's, is NaN
        for (int n = 0; n < NSEG; ++n) { yp[n] = np_min(yr[n] * alpha, xr[n] + xr[n] * c); mx += xr[n]; my += yp[n]; }
        mx /= NSEG; my /= NSEG;
        double nx = 0.0, ny = 0.0, dot = 0.0;
        for (int n = 0; n < NSEG; ++n) { const double a = xr[n] - mx, b = yp[n] - my; nx += a * a; ny += b * b; dot += a * b; }
        part[j] = dot / (sqrt(nx) * sqrt(ny));
    }
    __syncthreads();
    if (j == 0) {
        double d = 0.0;
        for (int b = 0; b < NBAND; ++b) d += part[b];
        atomicAdd(out, d / NBAND);
        atomicAdd(out + 1, 1.0);
    }
}

// ---- log-likelihood ratio (compute_metrics.py:277-347: llr + lpcoeff): one block per frame.  Windowed frames in shared memory, the 17
// autocorrelation lags of both signals by one warp each (strided + shuffle reduction), Levinson-Durbin (order P <= 16) by one thread per
// signal in shared memory and the two quadratic forms a R_c a^T by thread 0 (a few hundred flops).  out[f] = log(a_p R_c a_p^T / a_c R_c a_c^T).
constexpr int LLR_MAXW = 512, LLR_P = 16;
__global__ void llr_kernel(const double* __restrict__ c, const double* __restrict__ p, int W, int skip, int P, double* __restrict__ out, int serial) {
    __shared__ double fc[LLR_MAXW], fp[LLR_MAXW], Rc[LLR_P + 1], Rp[LLR_P + 1];
    const int f = blockIdx.x, tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, nw = blockDim.x >> 5;
    const long s0 = (long)f * skip;
    const double PI = 3.14159265358979323846;
    for (int i = tid; i < W; i += blockDim.x) {
        const double w = 0.5 * (1.0 - cos(2.0 * PI * (double)(i + 1) / (double)(W + 1)));
        fc[i] = c[s0 + i] * w;
        fp[i] = p[s0 + i] * w;
    }
    __syncthreads();
    if (serial) {                      // one thread per lag (diagnostic / fallback variant: no warp-level reduction)
        if (tid < 2 * (P + 1)) {
            const int k = tid % (P + 1);
            const double* x = tid <= P ? fc : fp;
            double acc = 0.0;
            for (int i = 0; i < W - k; ++i) acc += x[i] * x[i + k];
            if (tid <= P) Rc[k] = acc; else Rp[k] = acc;
        }
    } else {
        for (int job = warp; job < 2 * (P + 1); job += nw) {
            const int k = job % (P + 1);
            const double* x = job <= P ? fc : fp;
            double acc = 0.0;
            for (int i = lane; i < W - k; i += 32) acc += x[i] * x[i + k];
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
            if (lane == 0) { if (job <= P) Rc[k] = acc; else Rp[k] = acc; }
        }
    }
    __syncthreads();
    // Levinson-Durbin in shared memory, one thread per signal (thread 0: clean, thread 1: processed), ping-pong coefficient arrays:
    //   k_i = (R[i+1] - sum_{j<i} a_j R[i-j]) / E_i;   a'_j = a_j - k_i a_{i-1-j} (j < i), a'_i = k_i;   E_{i+1} = (1 - k_i^2) E_i
    __shared__ double lev[2][2][LLR_P + 1], poly[2][LLR_P + 1];
    if (tid < 2) {
        const double* R = tid == 0 ? Rc : Rp;
        int cur = 0;
        double err = R[0];
        for (int i = 0; i < P; ++i) {
            double acc = 0.0;
            for (int j = 0; j < i; ++j) acc += lev[tid][cur][j] * R[i - j];
            const double k = (R[i + 1] - acc) / err;
            for (int j = 0; j < i; ++j) lev[tid][cur ^ 1][j] = lev[tid][cur][j] - lev[tid][cur][i - 1 - j] * k;
            lev[tid][cur ^ 1][i] = k;
            err = (1.0 - k * k) * err;
            cur ^= 1;
        }
        poly[tid][0] = 1.0;
        for (int i = 0; i < P; ++i) poly[tid][i + 1] = -lev[tid][cur][i];
    }
    __syncthreads();
    if (tid == 0) {
        double num = 0.0, den = 0.0;
        for (int i = 0; i <= P; ++i)
            for (int j = 0; j <= P; ++j) {
                const double r = Rc[i > j ? i - j : j - i];
                num += poly[1][i] * r * poly[1][j];
                den += poly[0][i] * r * poly[0][j];
            }
        out[f] = log(num / den);
    }
}

// ---- weighted spectral slope (compute_metrics.py:80-274): one block per frame.  Windowed frame / 32768 -> power spectrum of the first
// nfft / 2 bins by a direct DFT against a shared twiddle table (nfft = 1024: 512 bins x 480 samples per signal) -> 25 critical-band
// energies in dB (filter matrix supplied by the caller, floor 1e-10) -> slopes, nearest-peak search and Klatt weights by thread 0.
constexpr int WSS_NB = 25, WSS_MAXFFT = 1024;
__device__ void wss_peaks(const double* e, const double* sl, double* pk) {
    for (int i = 0; i < WSS_NB - 1; ++i) {
        int n = i;
        if (sl[i] > 0) {
            while (n < WSS_NB - 1 && sl[n] > 0) ++n;
            pk[i] = e[n - 1];
        } else {
            while (n >= 0 && sl[n] <= 0) --n;
            pk[i] = e[n + 1];
        }
    }
}

__global__ void wss_kernel(const double* __restrict__ c, const double* __restrict__ p, int W, int skip, int nfft, const double* __restrict__ filt,
                           double* __restrict__ out, int serial) {
    extern __shared__ double sm[];
    double* fc = sm;                     // [W]
    double* fp = fc + LLR_MAXW;          // [W]
    double* tw = fp + LLR_MAXW;          // cos, sin tables [nfft] each
    double* sc = tw + 2 * WSS_MAXFFT;    // power spectra [nfft / 2] each
    double* sp = sc + WSS_MAXFFT / 2;
    __shared__ double ec[WSS_NB], ep[WSS_NB];
    const int f = blockIdx.x, tid = threadIdx.x, half = nfft / 2;
    const long s0 = (long)f * skip;
    const double PI = 3.14159265358979323846;
    for (int i = tid; i < W; i += blockDim.x) {
        const double w = 0.5 * (1.0 - cos(2.0 * PI * (double)(i + 1) / (double)(W + 1)));
        fc[i] = c[s0 + i] / 32768.0 * w;
        fp[i] = p[s0 + i] / 32768.0 * w;
    }
    for (int i = tid; i < nfft; i += blockDim.x) {
        double sn, cs;
        sincospi(2.0 * (double)i / (double)nfft, &sn, &cs);
        tw[i] = cs; tw[WSS_MAXFFT + i] = sn;
    }
    __syncthreads();
    for (int k = tid; k < half; k += blockDim.x) {
        double cr = 0.0, ci = 0.0, pr = 0.0, pi = 0.0;
        int ph = 0;
        for (int n = 0; n < W; ++n) {
            const double cs = tw[ph], sn = tw[WSS_MAXFFT + ph];
            cr += fc[n] * cs; ci -= fc[n] * sn;
            pr += fp[n] * cs; pi -= fp[n] * sn;
            ph += k;
            if (ph >= nfft) ph -= nfft;
        }
        sc[k] = cr * cr + ci * ci;
        sp[k] = pr * pr + pi * pi;
    }
    __syncthreads();
    if (serial) {
        if (tid < 2 * WSS_NB) {
            const int b = tid % WSS_NB;
            const double* spec = tid < WSS_NB ? sc : sp;
            double acc = 0.0;
            for (int j = 0; j < half; ++j) acc += filt[b * half + j] * spec[j];
            const double v = 10.0 * log10(np_max(acc, 1e-10));
            if (tid < WSS_NB) ec[b] = v; else ep[b] = v;
        }
    } else {
        for (int job = tid >> 5; job < 2 * WSS_NB; job += blockDim.x >> 5) {
            const int b = job % WSS_NB, lane = tid & 31;
            const double* spec = job < WSS_NB ? sc : sp;
            double acc = 0.0;
            for (int j = lane; j < half; j += 32) acc += filt[b * half + j] * spec[j];
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
            const double v = 10.0 * log10(np_max(acc, 1e-10));
            if (lane == 0) { if (job < WSS_NB) ec[b] = v; else ep[b] = v; }
        }
    }
    __syncthreads();
    if (tid == 0) {
        double csl[WSS_NB - 1], psl[WSS_NB - 1], cpk[WSS_NB - 1], ppk[WSS_NB - 1];
        double cmax = ec[0], pmax = ep[0];
        for (int i = 0; i < WSS_NB - 1; ++i) { csl[i] = ec[i + 1] - ec[i]; psl[i] = ep[i + 1] - ep[i]; }
        for (int i = 1; i < WSS_NB; ++i) { cmax = np_max(cmax, ec[i]); pmax = np_max(pmax, ep[i]); }
        wss_peaks(ec, csl, cpk);
        wss_peaks(ep, psl, ppk);
        double num = 0.0, den = 0.0;
        for (int i = 0; i < WSS_NB - 1; ++i) {
            const double wc = (20.0 / (20.0 + cmax - ec[i])) * (1.0 / (1.0 + cpk[i] - ec[i]));
            const double wp = (20.0 / (20.0 + pmax - ep[i])) * (1.0 / (1.0 + ppk[i] - ep[i]));
            const double w = 0.5 * (wc + wp), d = csl[i] - psl[i];
            num += w * d * d;
            den += w;
        }
        out[f] = num / den;
    }
}

}  // namespace

// mean segmental SNR (dB) of `proc` against `clean` (float64, L samples), added to out[0]: zero it on entry for the mean itself.  nfr =
// int(L / skip - W / skip) is the caller's (it is a host-side float expression in the reference); nfr = 0 writes nothing.
CMGAN_API int cmgan_ssnr_f64(const double* clean, const double* proc, long long L, int W, int skip, int nfr, double* out, void* stream) {
    CMGAN_REQUIRE(clean && proc && out && W > 0 && skip > 0, "cmgan_ssnr_f64: bad arguments");
    CMGAN_REQUIRE(nfr >= 0 && (long long)(nfr - 1) * skip + W <= L, "cmgan_ssnr_f64: frames exceed the signal");
    if (nfr == 0) return 0;
    ssnr_kernel<<<nfr, 128, 0, (cudaStream_t)stream>>>(clean, proc, W, skip, nfr, out);
    return cmgan_check_launch("ssnr_kernel");
}

// STOI of `proc` against `clean` (float64, L samples at 16 kHz).  h: the 161-tap resampling filter (already x 5); band_lo / band_hi: first and
// one-past-last DFT bin of the 15 third-octave bands; scratch: >= cmgan_stoi_scratch_doubles(L) doubles; out[0] / out[1] (zero on entry) receive
// the sum of the segment scores and their number (STOI = out[0] / out[1]).
CMGAN_API long long cmgan_stoi_scratch_doubles(long long L) {
    const long long n10 = (L * 5 + 7) / 8;
    const long long nframes = n10 / HOPF + 2;
    return 4 * (n10 + NF) + nframes * (1 + 2 * NBAND) + nframes + 64;       // x10, y10, xs, ys, levels, X, Y, (kept + cnt as ints)
}
CMGAN_API int cmgan_stoi_f64(const double* clean, const double* proc, long long L, const double* h, const int* band_lo, const int* band_hi,
                             double* scratch, double* out, void* stream) {
    CMGAN_REQUIRE(clean && proc && h && band_lo && band_hi && scratch && out && L > 16 * NF, "cmgan_stoi_f64: bad arguments");
    cudaStream_t st = (cudaStream_t)stream;
    const long n10 = (long)((L * 5) / 8 + ((L * 5) % 8 != 0));
    const int nframes = (int)((n10 - NF + HOPF - 1) / HOPF);            // len(arange(0, n10 - N, K))
    const long max_out = (long)(nframes - 1) * HOPF + NF;
    double* x10 = scratch; double* y10 = x10 + n10 + NF; double* xs = y10 + n10 + NF; double* ys = xs + n10 + NF;
    double* lev = ys + n10 + NF; double* X = lev + nframes + 1; double* Y = X + (long)NBAND * nframes;
    int* kept = reinterpret_cast<int*>(Y + (long)NBAND * nframes); int* cnt = kept + nframes + 1;
    // scipy.signal.resample_poly(x, 10000, 16000): up 5, down 8, the 161 taps of h (already x 5)
    if (resample::launch<double>(clean, L, 1, L, nullptr, 5, 8, 80, h, x10, n10, n10, nullptr, nullptr, st) != 0) return -1;
    if (resample::launch<double>(proc, L, 1, L, nullptr, 5, 8, 80, h, y10, n10, n10, nullptr, nullptr, st) != 0) return -1;
    frame_level_kernel<<<nframes, 128, 0, st>>>(x10, n10, nframes, lev);
    silent_mask_kernel<<<1, 1024, 0, st>>>(lev, nframes, 40.0, kept, cnt);
    compact_kernel<<<cdiv(max_out, 256), 256, 0, st>>>(x10, y10, kept, cnt, xs, ys, max_out);
    band_env_kernel<<<dim3(nframes, 2), 128, 0, st>>>(xs, ys, cnt, band_lo, band_hi, X, Y, nframes);
    if (nframes > NSEG) stoi_segment_kernel<<<nframes - NSEG + 1, 32, 0, st>>>(X, Y, cnt, nframes, out);
    return cmgan_check_launch("stoi kernels");
}

// per-frame log-likelihood ratios (compute_metrics.py:277-318); nfr = int((L - W) / skip) frames, out[nfr]; the caller sorts / trims (:52-55)
CMGAN_API int cmgan_llr_f64(const double* clean, const double* proc, long long L, int W, int skip, int order, int nfr, double* out, void* stream) {
    CMGAN_REQUIRE(clean && proc && out, "cmgan_llr_f64: null pointer");
    CMGAN_REQUIRE(W > 0 && W <= LLR_MAXW && skip > 0 && order >= 1 && order <= LLR_P && order < W, "cmgan_llr_f64: W=%d order=%d unsupported", W, order);
    CMGAN_REQUIRE(nfr >= 0 && (long long)(nfr - 1) * skip + W <= L, "cmgan_llr_f64: %d frames do not fit %lld samples", nfr, L);
    if (nfr == 0) return 0;
    llr_kernel<<<nfr, 256, 0, (cudaStream_t)stream>>>(clean, proc, W, skip, order, out, getenv("CMGAN_METRICS_SERIAL") != nullptr);
    return cmgan_check_launch("llr_kernel");
}

// per-frame weighted-spectral-slope distances (compute_metrics.py:80-274); filt = (25, nfft / 2) critical-band filter matrix, out[nfr]
CMGAN_API int cmgan_wss_f64(const double* clean, const double* proc, long long L, int W, int skip, int nfft, const double* filt, int nfr,
                            double* out, void* stream) {
    CMGAN_REQUIRE(clean && proc && filt && out, "cmgan_wss_f64: null pointer");
    CMGAN_REQUIRE(W > 0 && W <= LLR_MAXW && skip > 0 && nfft >= W && nfft <= WSS_MAXFFT && (nfft & (nfft - 1)) == 0, "cmgan_wss_f64: W=%d nfft=%d unsupported", W, nfft);
    CMGAN_REQUIRE(nfr >= 0 && (long long)(nfr - 1) * skip + W <= L, "cmgan_wss_f64: %d frames do not fit %lld samples", nfr, L);
    if (nfr == 0) return 0;
    const int smem = (2 * LLR_MAXW + 2 * WSS_MAXFFT + WSS_MAXFFT) * (int)sizeof(double);
    static bool attr_set = false;
    if (!attr_set) {
        cudaError_t e = cudaFuncSetAttribute(wss_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
        CMGAN_REQUIRE(e == cudaSuccess, "cmgan_wss_f64: cudaFuncSetAttribute: %s", cudaGetErrorString(e));
        attr_set = true;
    }
    wss_kernel<<<nfr, 256, smem, (cudaStream_t)stream>>>(clean, proc, W, skip, nfft, filt, out, getenv("CMGAN_METRICS_SERIAL") != nullptr);
    return cmgan_check_launch("wss_kernel");
}
