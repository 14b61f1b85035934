// Polyphase resampling: scipy.signal.resample_poly(x, up, down) with zero padding at both ends, in the index form
//   y[n] = sum_i x[i] h[down n + half - up i],  i in [max(0, ceil((down n - half) / up)), min(n_in - 1, floor((down n + half) / up))],
// h = the 2 half + 1 taps of the low-pass filter (already multiplied by up).  One template serves both users: the float instance behind
// cmgan_resample / cmgan_enhance_sr (resample.cu) and the double instance of STOI's 16 -> 10 kHz step (metrics.cu, up 5, down 8).
#pragma once
#include <algorithm>

#include "common.cuh"

namespace resample {

constexpr int THREADS = 256;
constexpr int MAX_BLOCKS_X = 1024;       // blocks per row: each stages the tap table once and strides over the row's outputs

// Block (x, b) works on row b; one output sample per thread per step, the block's tap table in shared memory.  Row b reads
// x[b, :len_b] with len_b = lens[b] clamped to [0, n_in] (n_in when lens is null) and writes y[b, :m_b], m_b = ceil(len_b up / down)
// limited to n_out and, when cap is not null, to cap[b] clamped to [0, n_out].  lens_out (optional) receives the m_b.  The sum runs
// over increasing i from 0.0 as acc += x[i] * h[.] (one fused multiply-add per tap, the order of the original STOI kernel).
template <typename T>
__global__ void __launch_bounds__(THREADS) resample_kernel(const T* __restrict__ x, long ldx, long n_in, const int* __restrict__ lens,
                                                           int up, int down, int half, const T* __restrict__ h, T* __restrict__ y, long ldy,
                                                           long n_out, const int* __restrict__ cap, int* __restrict__ lens_out) {
    extern __shared__ __align__(16) unsigned char resample_smem[];
    T* hs = reinterpret_cast<T*>(resample_smem);
    const int ntaps = 2 * half + 1;
    for (int i = threadIdx.x; i < ntaps; i += blockDim.x) hs[i] = h[i];
    __syncthreads();
    const int b = blockIdx.y;
    long len = n_in;
    if (lens) len = min(max((long)lens[b], 0L), n_in);
    long m = (len * up + down - 1) / down;
    m = min(m, n_out);
    if (cap) m = min(m, min(max((long)cap[b], 0L), n_out));
    if (lens_out && blockIdx.x == 0 && threadIdx.x == 0) lens_out[b] = (int)m;
    const T* xb = x + (long)b * ldx;
    T* yb = y + (long)b * ldy;
    for (long n = (long)blockIdx.x * blockDim.x + threadIdx.x; n < m; n += (long)gridDim.x * blockDim.x) {
        const long t = (long)down * n + half;
        long i_lo = t - 2 * half <= 0 ? 0 : (t - 2 * half + up - 1) / up;
        long i_hi = t / up;
        if (i_hi > len - 1) i_hi = len - 1;
        T acc = 0.0;
        for (long i = i_lo; i <= i_hi; ++i) acc += xb[i] * hs[t - up * i];
        yb[n] = acc;
    }
}

// enqueue resample_kernel over B rows; the caller has checked the arguments.  Tables above 48 KB (float taps at max(up, down) > 960)
// need the opt-in shared-memory size, set once per instance.
template <typename T>
int launch(const T* x, long ldx, int B, long n_in, const int* lens, int up, int down, int half, const T* h, T* y, long ldy, long n_out,
           const int* cap, int* lens_out, cudaStream_t st) {
    const size_t smem = (size_t)(2 * half + 1) * sizeof(T);
    static size_t smem_set = 48 * 1024;
    if (smem > smem_set) {
        const cudaError_t e = cudaFuncSetAttribute(resample_kernel<T>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) { cmgan_set_error("resample_kernel: cudaFuncSetAttribute(%zu bytes): %s", smem, cudaGetErrorString(e)); return -1; }
        smem_set = smem;
    }
    const long most = std::min((n_in * up + down - 1) / down, n_out);        // outputs of the longest row
    const int gx = (int)std::min<long>(std::max<long>(cdiv(most, THREADS), 1), MAX_BLOCKS_X);
    resample_kernel<T><<<dim3(gx, B), THREADS, smem, st>>>(x, ldx, n_in, lens, up, down, half, h, y, ldy, n_out, cap, lens_out);
    return cmgan_check_launch("resample_kernel");
}

// sr_in -> sr_out as up / down in lowest terms, half = 10 max(up, down); 0, or -1 with the message set for an unsupported pair
struct Ratio { int up, down, half; };
int ratio(int sr_in, int sr_out, Ratio& q, const char* who);

}  // namespace resample
