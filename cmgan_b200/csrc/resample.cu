// Sample-rate conversion between the standard audio rates: scipy.signal.resample_poly with its default filter (firwin(2 half + 1,
// 1 / max(up, down), window=('kaiser', 5.0)) * up, half = 10 max(up, down)), the tap table built on the device and the float instance of
// the polyphase kernel (resample.cuh).  The module-level entries cmgan_enhance_sr / cmgan_enhance_long_sr run it around the 16 kHz walk.
#include <cmath>

#include "resample.cuh"
#include "../../include/cmgan_b200.h"

namespace resample {

constexpr int SR_MIN = 8000, SR_MAX = 192000, MAX_FACTOR = 1024;

static int gcd(int a, int b) {
    while (b) { const int t = a % b; a = b; b = t; }
    return a;
}

int ratio(int sr_in, int sr_out, Ratio& q, const char* who) {
    CMGAN_REQUIRE(sr_in >= SR_MIN && sr_in <= SR_MAX && sr_out >= SR_MIN && sr_out <= SR_MAX,
                  "%s: sample rates must lie in [%d, %d] Hz (sr_in=%d sr_out=%d)", who, SR_MIN, SR_MAX, sr_in, sr_out);
    const int g = gcd(sr_in, sr_out);
    q.up = sr_out / g;
    q.down = sr_in / g;
    CMGAN_REQUIRE(q.up <= MAX_FACTOR && q.down <= MAX_FACTOR,
                  "%s: %d -> %d Hz reduces to up=%d down=%d; at most %d each (the standard rates 8, 11.025, 12, 16, 22.05, 24, 32, 44.1, 48, "
                  "88.2, 96, 176.4 and 192 kHz to and from 16 kHz all qualify)", who, sr_in, sr_out, q.up, q.down, MAX_FACTOR);
    q.half = 10 * std::max(q.up, q.down);
    return 0;
}

namespace {

// modified Bessel function of the first kind, order 0, by its power series (z <= 5 here: 20 terms reach float64 precision)
__device__ double bessel_i0(double z) {
    const double q = 0.25 * z * z;
    double term = 1.0, sum = 1.0;
    for (int k = 1; k < 64; ++k) {
        term *= q / ((double)k * (double)k);
        sum += term;
        if (term < 1e-17 * sum) break;
    }
    return sum;
}

// the un-normalised firwin tap m: fc sinc(fc (m - half)) * kaiser(2 half + 1, 5)[m], fc = 1 / max(up, down)
__device__ double raw_tap(int m, int half, double fc) {
    const double d = (double)(m - half);
    const double a = fc * d;
    const double sinc = d == 0.0 ? 1.0 : sinpi(a) / (3.141592653589793 * a);
    const double r = d / (double)half;
    const double w = bessel_i0(5.0 * sqrt(fmax(0.0, 1.0 - r * r))) / bessel_i0(5.0);
    return fc * sinc * w;
}

// one block: the taps' sum (firwin normalises the pass band's DC gain to 1), then h[m] = raw_tap(m) / sum * up, rounded to fp32 once
__global__ void taps_kernel(int half, int up, double fc, float* __restrict__ h) {
    __shared__ double part[32];
    const int ntaps = 2 * half + 1;
    double s = 0.0;
    for (int m = threadIdx.x; m < ntaps; m += blockDim.x) s += raw_tap(m, half, fc);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5] = s;
    __syncthreads();
    double sum = 0.0;
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) sum += part[w];
    for (int m = threadIdx.x; m < ntaps; m += blockDim.x) h[m] = (float)(raw_tap(m, half, fc) / sum * (double)up);
}

}  // namespace
}  // namespace resample

using namespace resample;

CMGAN_API int cmgan_resample_taps_floats(int sr_in, int sr_out) {
    Ratio q;
    if (ratio(sr_in, sr_out, q, "cmgan_resample_taps_floats") != 0) return -1;
    return 2 * q.half + 1;
}

CMGAN_API int cmgan_resample_taps(int sr_in, int sr_out, float* h, void* stream) {
    Ratio q;
    if (ratio(sr_in, sr_out, q, "cmgan_resample_taps") != 0) return -1;
    CMGAN_REQUIRE(h, "cmgan_resample_taps: h is null");
    taps_kernel<<<1, 1024, 0, (cudaStream_t)stream>>>(q.half, q.up, 1.0 / (double)std::max(q.up, q.down), h);
    return cmgan_check_launch("taps_kernel");
}

CMGAN_API int cmgan_resample(const float* x, long long ldx, int B, long long L, const int* lengths, int sr_in, int sr_out, const float* h, float* y,
                             long long ldy, void* stream) {
    const char* who = "cmgan_resample";
    Ratio q;
    if (ratio(sr_in, sr_out, q, who) != 0) return -1;
    CMGAN_REQUIRE(x && h && y, "%s: null pointer", who);
    CMGAN_REQUIRE(B > 0 && L > 0, "%s: B and L must be positive (B=%d L=%lld)", who, B, L);
    const long long n_out = (L * q.up + q.down - 1) / q.down;
    CMGAN_REQUIRE(ldx >= L && ldy >= n_out, "%s: row strides must cover a row (L=%lld ldx=%lld, %lld outputs, ldy=%lld)", who, L, ldx, n_out, ldy);
    const uintptr_t x0 = (uintptr_t)x, x1 = (uintptr_t)(x + (B - 1) * ldx + L), y0 = (uintptr_t)y, y1 = (uintptr_t)(y + (B - 1) * ldy + n_out);
    CMGAN_REQUIRE(x1 <= y0 || y1 <= x0, "%s: x and y overlap", who);
    return launch<float>(x, ldx, B, L, lengths, q.up, q.down, q.half, h, y, ldy, n_out, nullptr, nullptr, (cudaStream_t)stream);
}
