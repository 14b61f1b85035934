// Error channel, library info, dropout-mask export, and the small discriminator-only kernels
// (input stacking, spectral normalisation, global max pool, dropout+PReLU, learnable sigmoid).
#include <stdarg.h>

#include "common.cuh"
#include "../../include/cmgan_b200.h"

static thread_local char g_err[512] = "";

int g_cmgan_round_tf32 = 0;
CMGAN_API int cmgan_set_tf32_rounding(int on) { g_cmgan_round_tf32 = on ? 1 : 0; return 0; }

void cmgan_set_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}

int cmgan_check_launch(const char* what) {
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) {
        cmgan_set_error("%s: %s", what, cudaGetErrorString(e));
        return -1;
    }
    return 0;
}

int cmgan_num_sms() {
    static int n = 0;
    if (n == 0) {
        int dev = 0;
        if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) n = 132;
    }
    return n;
}

CMGAN_API const char* cmgan_last_error(void) { return g_err; }
CMGAN_API int cmgan_abi_version(void) { return 1; }
CMGAN_API int cmgan_gemm_args_size(void) { return (int)sizeof(CmganGemmArgs); }

namespace {

__global__ void dropout_mask_kernel(float* out, long n, unsigned long long seed, unsigned thr) {
    long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = cmgan_drop_scale(seed, (uint64_t)i, thr, 1.0f);
}

// (x, y) each (B, 1, H, W) with strides -> xy (B, H, W, 2)
__global__ void stack2_kernel(const float* __restrict__ x, long xb, long xh, long xw, const float* __restrict__ y, long yb, long yh, long yw,
                              int H, int W, long n, float* __restrict__ out) {
    long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    int w = (int)(i % W); long t = i / W; int h = (int)(t % H); long b = t / H;
    reinterpret_cast<float2*>(out)[i] = make_float2(__ldg(x + b * xb + h * xh + w * xw), __ldg(y + b * yb + h * yh + w * yw));
}
// d(x), d(y) planes (B, H, W) contiguous from dxy (B, H, W, 2)
__global__ void unstack2_kernel(const float* __restrict__ dxy, long n, float* __restrict__ dx, float* __restrict__ dy) {
    long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    float2 v = __ldg(reinterpret_cast<const float2*>(dxy) + i);
    if (dx) dx[i] = v.x;
    if (dy) dy[i] = v.y;
}

// ---- spectral normalisation (reference discriminator.py:33-58 via torch.nn.utils.spectral_norm, 1 power iteration)
// W (R, Cc) row-major = weight_orig.view(out, -1).  One block.  train: v = normalize(W^T u); u = normalize(W v).
// sigma = u^T W v;  w_sn = W / sigma.
__device__ float block_sum(float v, float* sm) {
    v = warp_sum(v);
    __syncthreads();
    if ((threadIdx.x & 31) == 0) sm[threadIdx.x >> 5] = v;
    __syncthreads();
    float t = 0.f;
    for (int w = 0; w < (blockDim.x >> 5); ++w) t += sm[w];
    return t;
}

__global__ void spectral_norm_kernel(const float* __restrict__ W, int R, int Cc, float* __restrict__ u, float* __restrict__ v, int training,
                                     float* __restrict__ w_sn, float* __restrict__ sigma_out, float* __restrict__ uv_out) {
    __shared__ float sm[32];
    extern __shared__ float dyn[];      // su[R], sv[Cc], swv[R]
    float* su = dyn; float* sv = dyn + R; float* swv = sv + Cc;
    const float eps = 1e-12f;
    for (int i = threadIdx.x; i < R; i += blockDim.x) su[i] = u[i];
    for (int j = threadIdx.x; j < Cc; j += blockDim.x) sv[j] = v[j];
    __syncthreads();
    if (training) {
        float part = 0.f;
        for (int j = threadIdx.x; j < Cc; j += blockDim.x) {
            float a = 0.f;
            for (int i = 0; i < R; ++i) a = fmaf(__ldg(W + (long)i * Cc + j), su[i], a);
            sv[j] = a; part = fmaf(a, a, part);
        }
        float nrm = fmaxf(sqrtf(block_sum(part, sm)), eps);
        for (int j = threadIdx.x; j < Cc; j += blockDim.x) sv[j] /= nrm;
        __syncthreads();
    }
    // W v (needed for sigma in both modes, and for the u update in training)
    {
        int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
        for (int i = warp; i < R; i += nw) {
            float a = 0.f;
            for (int j = lane; j < Cc; j += 32) a = fmaf(__ldg(W + (long)i * Cc + j), sv[j], a);
            a = warp_sum(a);
            if (lane == 0) swv[i] = a;
        }
        __syncthreads();
    }
    if (training) {
        float part = 0.f;
        for (int i = threadIdx.x; i < R; i += blockDim.x) part = fmaf(swv[i], swv[i], part);
        float nrm = fmaxf(sqrtf(block_sum(part, sm)), eps);
        for (int i = threadIdx.x; i < R; i += blockDim.x) su[i] = swv[i] / nrm;
        __syncthreads();
    }
    float part = 0.f;
    for (int i = threadIdx.x; i < R; i += blockDim.x) part = fmaf(su[i], swv[i], part);
    float sigma = block_sum(part, sm);
    float inv = 1.f / sigma;
    for (long k = threadIdx.x; k < (long)R * Cc; k += blockDim.x) w_sn[k] = __ldg(W + k) * inv;
    if (training) {
        for (int i = threadIdx.x; i < R; i += blockDim.x) u[i] = su[i];
        for (int j = threadIdx.x; j < Cc; j += blockDim.x) v[j] = sv[j];
    }
    if (uv_out) {       // the (u, v) this forward's sigma / W_sn were formed with: the backward of THIS forward must use them, not the live buffers
        for (int i = threadIdx.x; i < R; i += blockDim.x) uv_out[i] = su[i];
        for (int j = threadIdx.x; j < Cc; j += blockDim.x) uv_out[R + j] = sv[j];
    }
    if (threadIdx.x == 0) sigma_out[0] = sigma;
}

// dW_orig += (dW_sn - <dW_sn, W_sn> u v^T) / sigma.  One block (the dot product is a block-wide reduction over <= 131 k elements):
// 1024 threads, 128-bit loads when the row length allows (every layer of the reference discriminator: Cc = 32 .. 1024).
__global__ void __launch_bounds__(1024) spectral_norm_bwd_kernel(const float* __restrict__ w_sn, const float* __restrict__ dw_sn, int R, int Cc,
                                                                 const float* __restrict__ u, const float* __restrict__ v,
                                                                 const float* __restrict__ sigma, float* __restrict__ dW) {
    __shared__ float sm[32];
    const long n = (long)R * Cc;
    const bool v4 = (Cc & 3) == 0 && ((((uintptr_t)w_sn) | ((uintptr_t)dw_sn) | ((uintptr_t)dW) | ((uintptr_t)v)) & 15) == 0;
    float part = 0.f;
    if (v4) {
#pragma unroll 4
        for (long k = threadIdx.x; k < n / 4; k += blockDim.x) {
            const float4 a = __ldg(reinterpret_cast<const float4*>(dw_sn) + k), b = __ldg(reinterpret_cast<const float4*>(w_sn) + k);
            part += a.x * b.x + a.y * b.y + a.z * b.z + a.w * b.w;
        }
    } else {
        for (long k = threadIdx.x; k < n; k += blockDim.x) part = fmaf(__ldg(dw_sn + k), __ldg(w_sn + k), part);
    }
    const float dot = block_sum(part, sm);
    const float inv = 1.f / sigma[0];
    if (v4) {
        const int c4 = Cc / 4;
#pragma unroll 4
        for (long k = threadIdx.x; k < n / 4; k += blockDim.x) {
            const int i = (int)(k / c4), j = (int)(k % c4);
            const float4 a = __ldg(reinterpret_cast<const float4*>(dw_sn) + k), vv = __ldg(reinterpret_cast<const float4*>(v) + j);
            const float du = dot * u[i];
            float4 o = reinterpret_cast<float4*>(dW)[k];
            o.x += (a.x - du * vv.x) * inv; o.y += (a.y - du * vv.y) * inv; o.z += (a.z - du * vv.z) * inv; o.w += (a.w - du * vv.w) * inv;
            reinterpret_cast<float4*>(dW)[k] = o;
        }
    } else {
        for (long k = threadIdx.x; k < n; k += blockDim.x) {
            const int i = (int)(k / Cc), j = (int)(k % Cc);
            dW[k] += (__ldg(dw_sn + k) - dot * u[i] * v[j]) * inv;
        }
    }
}

// out[b, c] = max over rows of prelu(x*scale+shift);  arg[b, c] = row index (within the group) of the max: the first of tied rows, and
// as in torch's adaptive_max_pool2d a NaN wins (the last NaN of the window), so the output is NaN and its gradient goes to that row
__global__ void norm_maxpool_kernel(const float* __restrict__ x, long rows, int C, const float* __restrict__ scale, const float* __restrict__ shift,
                                    const float* __restrict__ slope, float* __restrict__ out, int* __restrict__ arg) {
    int b = blockIdx.x, c = threadIdx.x;
    if (c >= C) return;
    float sc = scale[b * C + c], sh = shift[b * C + c], a = slope[c];
    float best = -INFINITY; int bi = 0;
    for (long r = 0; r < rows; ++r) {
        float z = __ldg(x + ((long)b * rows + r) * C + c) * sc + sh;
        if (z < 0.f) z *= a;
        if (z > best || isnan(z)) { best = z; bi = (int)r; }
    }
    out[b * C + c] = best;
    if (arg) arg[b * C + c] = bi;
}
// dact (B*rows, C) = zero except at the arg-max row
__global__ void maxpool_bwd_kernel(const float* __restrict__ dout, const int* __restrict__ arg, long rows, int C, long total, float* __restrict__ dact) {
    long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= total) return;
    int c = (int)(i % C); long row = i / C; long b = row / rows; long r = row % rows;
    dact[i] = (arg[b * C + c] == (int)r) ? dout[b * C + c] : 0.f;
}

// y = prelu(x * drop(i), slope[c])   (Dropout(0.3) then PReLU(64), discriminator.py:55-56); in place allowed.  The backward takes the slope
// branch at z = 0, as torch's PReLU backward does.
__global__ void drop_prelu_kernel(const float* __restrict__ x, long n, int C, const float* __restrict__ slope, unsigned long long seed,
                                  unsigned thr, float inv_keep, float* __restrict__ y, const unsigned long long* __restrict__ seed_dev) {
    long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    seed = cmgan_eff_seed(seed, seed_dev);
    float z = x[i] * cmgan_drop_scale(seed, (uint64_t)i, thr, inv_keep);
    y[i] = z >= 0.f ? z : z * slope[i % C];
}
__global__ void drop_prelu_bwd_kernel(const float* __restrict__ x, const float* __restrict__ dy, long n, int C, const float* __restrict__ slope,
                                      unsigned long long seed, unsigned thr, float inv_keep, float* __restrict__ dx, float* __restrict__ dslope,
                                      const unsigned long long* __restrict__ seed_dev) {
    long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    seed = cmgan_eff_seed(seed, seed_dev);
    float ds = cmgan_drop_scale(seed, (uint64_t)i, thr, inv_keep);
    float z = x[i] * ds;
    float g = dy[i];
    if (!(z > 0.f)) { atomicAdd(dslope + (i % C), g * z); g *= slope[i % C]; }
    dx[i] = g * ds;
}
// y = sigmoid(slope * x)  (LearnableSigmoid(1), utils.py:42-50)
__global__ void lsigmoid_kernel(const float* __restrict__ x, long n, const float* __restrict__ slope, float* __restrict__ y) {
    long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) y[i] = sigmoidf_(slope[0] * x[i]);
}
__global__ void lsigmoid_bwd_kernel(const float* __restrict__ x, const float* __restrict__ y, const float* __restrict__ dy, long n,
                                    const float* __restrict__ slope, float* __restrict__ dx, float* __restrict__ dslope) {
    long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    float p = 0.f;
    if (i < n) {
        float g = dy[i] * y[i] * (1.f - y[i]);
        dx[i] = g * slope[0];
        p = g * x[i];
    }
    p = warp_sum(p);
    if ((threadIdx.x & 31) == 0 && p != 0.f) atomicAdd(dslope, p);
}

__global__ void counter_add_kernel(unsigned long long* p, unsigned long long v) { *p += v; }

}  // namespace

// *p += v on the device (step counters that CUDA-graph replays advance)
CMGAN_API int cmgan_counter_add(unsigned long long* p, unsigned long long v, void* stream) {
    CMGAN_REQUIRE(p != nullptr, "cmgan_counter_add: null pointer");
    counter_add_kernel<<<1, 1, 0, (cudaStream_t)stream>>>(p, v);
    return cmgan_check_launch("counter_add_kernel");
}

// out[i] = 1 if element i is kept by dropout(seed, p) else 0  (tests: feed the exact masks to the oracle)
CMGAN_API int cmgan_dropout_mask(float* out, long long n, unsigned long long seed, unsigned int thr, void* stream) {
    if (n == 0) return 0;
    dropout_mask_kernel<<<cdiv(n, 256), 256, 0, (cudaStream_t)stream>>>(out, n, seed, thr);
    return cmgan_check_launch("dropout_mask_kernel");
}

CMGAN_API int cmgan_stack2(const float* x, long long xb, long long xh, long long xw, const float* y, long long yb, long long yh, long long yw,
                           int B, int H, int W, float* out, void* stream) {
    CMGAN_REQUIRE(x && y && out, "cmgan_stack2: null pointer");
    long n = (long)B * H * W;
    if (n == 0) return 0;
    stack2_kernel<<<cdiv(n, 256), 256, 0, (cudaStream_t)stream>>>(x, xb, xh, xw, y, yb, yh, yw, H, W, n, out);
    return cmgan_check_launch("stack2_kernel");
}

CMGAN_API int cmgan_unstack2(const float* dxy, long long n, float* dx, float* dy, void* stream) {
    CMGAN_REQUIRE(dxy, "cmgan_unstack2: null pointer");
    if (n == 0) return 0;
    unstack2_kernel<<<cdiv(n, 256), 256, 0, (cudaStream_t)stream>>>(dxy, n, dx, dy);
    return cmgan_check_launch("unstack2_kernel");
}

CMGAN_API int cmgan_spectral_norm(const float* W, int R, int Cc, float* u, float* v, int training, float* w_sn, float* sigma, float* uv_out,
                                  void* stream) {
    CMGAN_REQUIRE(W && u && v && w_sn && sigma && R > 0 && Cc > 0, "cmgan_spectral_norm: bad arguments");
    size_t smem = (size_t)(2 * R + Cc) * sizeof(float);
    CMGAN_REQUIRE(smem <= 40000, "cmgan_spectral_norm: matrix too large (%d x %d)", R, Cc);
    spectral_norm_kernel<<<1, 512, smem, (cudaStream_t)stream>>>(W, R, Cc, u, v, training, w_sn, sigma, uv_out);
    return cmgan_check_launch("spectral_norm_kernel");
}

CMGAN_API int cmgan_spectral_norm_bwd(const float* w_sn, const float* dw_sn, int R, int Cc, const float* u, const float* v, const float* sigma,
                                      float* dW, void* stream) {
    CMGAN_REQUIRE(w_sn && dw_sn && u && v && sigma && dW, "cmgan_spectral_norm_bwd: null pointer");
    spectral_norm_bwd_kernel<<<1, 1024, 0, (cudaStream_t)stream>>>(w_sn, dw_sn, R, Cc, u, v, sigma, dW);
    return cmgan_check_launch("spectral_norm_bwd_kernel");
}

CMGAN_API int cmgan_norm_maxpool(const float* x, int B, long long rows, int C, const float* scale, const float* shift, const float* slope,
                                 float* out, int* arg, void* stream) {
    CMGAN_REQUIRE(x && scale && shift && slope && out && C <= 1024, "cmgan_norm_maxpool: bad arguments");
    if (B == 0) return 0;
    norm_maxpool_kernel<<<B, C, 0, (cudaStream_t)stream>>>(x, rows, C, scale, shift, slope, out, arg);
    return cmgan_check_launch("norm_maxpool_kernel");
}

CMGAN_API int cmgan_maxpool_bwd(const float* dout, const int* arg, int B, long long rows, int C, float* dact, void* stream) {
    CMGAN_REQUIRE(dout && arg && dact, "cmgan_maxpool_bwd: null pointer");
    long total = (long)B * rows * C;
    if (total == 0) return 0;
    maxpool_bwd_kernel<<<cdiv(total, 256), 256, 0, (cudaStream_t)stream>>>(dout, arg, rows, C, total, dact);
    return cmgan_check_launch("maxpool_bwd_kernel");
}

CMGAN_API int cmgan_drop_prelu(const float* x, long long n, int C, const float* slope, unsigned long long seed, unsigned int thr, float inv_keep,
                               float* y, const unsigned long long* seed_dev, void* stream) {
    CMGAN_REQUIRE(x && slope && y, "cmgan_drop_prelu: null pointer");
    if (n == 0) return 0;
    drop_prelu_kernel<<<cdiv(n, 256), 256, 0, (cudaStream_t)stream>>>(x, n, C, slope, seed, thr, inv_keep, y, seed_dev);
    return cmgan_check_launch("drop_prelu_kernel");
}

CMGAN_API int cmgan_drop_prelu_bwd(const float* x, const float* dy, long long n, int C, const float* slope, unsigned long long seed,
                                   unsigned int thr, float inv_keep, float* dx, float* dslope, const unsigned long long* seed_dev, void* stream) {
    CMGAN_REQUIRE(x && dy && slope && dx && dslope, "cmgan_drop_prelu_bwd: null pointer");
    if (n == 0) return 0;
    drop_prelu_bwd_kernel<<<cdiv(n, 256), 256, 0, (cudaStream_t)stream>>>(x, dy, n, C, slope, seed, thr, inv_keep, dx, dslope, seed_dev);
    return cmgan_check_launch("drop_prelu_bwd_kernel");
}

CMGAN_API int cmgan_lsigmoid(const float* x, long long n, const float* slope, float* y, void* stream) {
    CMGAN_REQUIRE(x && slope && y, "cmgan_lsigmoid: null pointer");
    if (n == 0) return 0;
    lsigmoid_kernel<<<cdiv(n, 256), 256, 0, (cudaStream_t)stream>>>(x, n, slope, y);
    return cmgan_check_launch("lsigmoid_kernel");
}

CMGAN_API int cmgan_lsigmoid_bwd(const float* x, const float* y, const float* dy, long long n, const float* slope, float* dx, float* dslope,
                                 void* stream) {
    CMGAN_REQUIRE(x && y && dy && slope && dx && dslope, "cmgan_lsigmoid_bwd: null pointer");
    if (n == 0) return 0;
    lsigmoid_bwd_kernel<<<cdiv(n, 256), 256, 0, (cudaStream_t)stream>>>(x, y, dy, n, slope, dx, dslope);
    return cmgan_check_launch("lsigmoid_bwd_kernel");
}
