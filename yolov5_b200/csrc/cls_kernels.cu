// Classification head and loss: global average pool (forward / backward) over NHWC channel-slice views, and the
// label-smoothed cross-entropy of nn.CrossEntropyLoss(label_smoothing=eps) with its gradient.
// Reference: models/common.py:1120-1140 (Classify: conv -> AdaptiveAvgPool2d(1) -> Dropout -> Linear),
// utils/torch_utils.py:52-57 (smartCrossEntropyLoss), classify/train.py:223-227 (autocast forward, scaled backward).
// Every reduction runs in a fixed order with fp32 accumulators and no atomics, so results repeat bit for bit.
#include <math.h>

#include "../../include/y5b200.h"
#include "common.cuh"
#include "host_util.h"

namespace y5 {

// ---------------------------------------------------------------------------------------------------------------------
// pooled[b][c] = round(sum_{p < HW} x[b][p][c] / HW): one thread per (image, 8-channel vector), pixels summed in order.
// ---------------------------------------------------------------------------------------------------------------------
__global__ void gap_fwd_kernel(const uint16_t* __restrict__ x, int x_pitch, uint16_t* __restrict__ y, int y_pitch, int B, int HW, int C,
                               int bf16) {
    const int cv = C >> 3;
    const long long total = static_cast<long long>(B) * cv;
    for (long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; idx < total;
         idx += static_cast<long long>(gridDim.x) * blockDim.x) {
        const int c8 = static_cast<int>(idx % cv);
        const int b = static_cast<int>(idx / cv);
        const uint16_t* p = x + static_cast<long long>(b) * HW * x_pitch + c8 * 8;
        float acc[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[j] = 0.0f;
#pragma unroll 4
        for (int q = 0; q < HW; ++q) {
            const uint4 v = *reinterpret_cast<const uint4*>(p + static_cast<long long>(q) * x_pitch);
            const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const float2 t = unpack2(w[j], bf16);
                acc[2 * j] += t.x;
                acc[2 * j + 1] += t.y;
            }
        }
        const float n = static_cast<float>(HW);
        uint4 o;
        o.x = pack2(acc[0] / n, acc[1] / n, bf16);
        o.y = pack2(acc[2] / n, acc[3] / n, bf16);
        o.z = pack2(acc[4] / n, acc[5] / n, bf16);
        o.w = pack2(acc[6] / n, acc[7] / n, bf16);
        *reinterpret_cast<uint4*>(y + static_cast<long long>(b) * y_pitch + c8 * 8) = o;
    }
}

// dx[b][p][c] = round(dy[b][c] / HW) for every pixel p: one thread per (pixel, 8-channel vector).
__global__ void gap_bwd_kernel(const uint16_t* __restrict__ dy, int dy_pitch, uint16_t* __restrict__ dx, int dx_pitch, int B, int HW, int C,
                               int bf16) {
    const int cv = C >> 3;
    const long long total = static_cast<long long>(B) * HW * cv;
    const float n = static_cast<float>(HW);
    for (long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; idx < total;
         idx += static_cast<long long>(gridDim.x) * blockDim.x) {
        const int c8 = static_cast<int>(idx % cv);
        const long long pix = idx / cv;
        const int b = static_cast<int>(pix / HW);
        const uint4 v = *reinterpret_cast<const uint4*>(dy + static_cast<long long>(b) * dy_pitch + c8 * 8);
        const uint32_t w[4] = {v.x, v.y, v.z, v.w};
        uint32_t o[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const float2 t = unpack2(w[j], bf16);
            o[j] = pack2(t.x / n, t.y / n, bf16);
        }
        *reinterpret_cast<uint4*>(dx + pix * dx_pitch + c8 * 8) = make_uint4(o[0], o[1], o[2], o[3]);
    }
}

// ---------------------------------------------------------------------------------------------------------------------
// Cross-entropy with label smoothing, one CTA per row.  With lse = max + log(sum exp(x - max)):
//   -log p_c = lse - x_c,   row loss = (1 - eps) (lse - x_y) + (eps / nc) (nc lse - sum_c x_c)
// and, when dlogits is given, dlogits_c = g (softmax_c - q_c) / B with q_c = (1 - eps) [c == y] + eps / nc, g the upstream
// gradient (a device scalar, 1 when absent) multiplied in fp32 before the single rounding to the logits dtype.
// ---------------------------------------------------------------------------------------------------------------------
constexpr int kCeThreads = 256;

template <typename T>
__device__ __forceinline__ float ld(const T* p);
template <> __device__ __forceinline__ float ld<__half>(const __half* p) { return __half2float(*p); }
template <> __device__ __forceinline__ float ld<__nv_bfloat16>(const __nv_bfloat16* p) { return __bfloat162float(*p); }
template <> __device__ __forceinline__ float ld<float>(const float* p) { return *p; }
template <typename T>
__device__ __forceinline__ T st(float v);
template <> __device__ __forceinline__ __half st<__half>(float v) { return __float2half_rn(v); }
template <> __device__ __forceinline__ __nv_bfloat16 st<__nv_bfloat16>(float v) { return __float2bfloat16_rn(v); }
template <> __device__ __forceinline__ float st<float>(float v) { return v; }

// fixed-order block reduction (shuffle tree inside each warp, then warp 0 over the warp partials); every thread gets the result
template <bool kMax>
__device__ __forceinline__ float block_reduce(float v, float* red) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const float u = __shfl_xor_sync(0xffffffffu, v, o);
        v = kMax ? fmaxf(v, u) : v + u;
    }
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    __syncthreads();  // `red` may still be read by the previous reduction
    if (lane == 0) red[warp] = v;
    __syncthreads();
    if (warp == 0) {
        v = lane < kCeThreads / 32 ? red[lane] : (kMax ? -INFINITY : 0.0f);
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            const float u = __shfl_xor_sync(0xffffffffu, v, o);
            v = kMax ? fmaxf(v, u) : v + u;
        }
        if (lane == 0) red[0] = v;
    }
    __syncthreads();
    return red[0];
}

template <typename T>
__global__ void __launch_bounds__(kCeThreads) ce_row_kernel(const T* __restrict__ logits, long long row_stride, int nc,
                                                             const long long* __restrict__ labels, float eps, const float* __restrict__ g_scale,
                                                             T* __restrict__ dlogits, long long d_stride, float* __restrict__ row_loss, int B) {
    __shared__ float red[32];
    const int b = blockIdx.x;
    const T* x = logits + static_cast<long long>(b) * row_stride;
    const long long yl = labels[b];
    const bool valid = yl >= 0 && yl < nc;
    float mx = -INFINITY, sx = 0.0f;
    for (int c = threadIdx.x; c < nc; c += kCeThreads) {
        const float v = ld<T>(x + c);
        mx = fmaxf(mx, v);
        sx += v;
    }
    mx = block_reduce<true>(mx, red);
    sx = block_reduce<false>(sx, red);
    float se = 0.0f;
    for (int c = threadIdx.x; c < nc; c += kCeThreads) se += expf(ld<T>(x + c) - mx);
    se = block_reduce<false>(se, red);
    const float lse = mx + logf(se);
    if (threadIdx.x == 0) {
        const float xy = valid ? ld<T>(x + yl) : NAN;
        row_loss[b] = (1.0f - eps) * (lse - xy) + (eps / static_cast<float>(nc)) * (static_cast<float>(nc) * lse - sx);
    }
    if (dlogits == nullptr) return;
    const float g = (g_scale != nullptr ? *g_scale : 1.0f) / static_cast<float>(B);
    const float off = eps / static_cast<float>(nc);
    T* d = dlogits + static_cast<long long>(b) * d_stride;
    for (int c = threadIdx.x; c < nc; c += kCeThreads) {
        const float sm = expf(ld<T>(x + c) - lse);
        const float q = (c == yl ? 1.0f - eps : 0.0f) + off;
        d[c] = st<T>(valid ? g * (sm - q) : NAN);
    }
}

// loss = sum_b row_loss[b] / B, summed by one CTA in a fixed order (strided per-thread partials, then the block tree)
__global__ void __launch_bounds__(kCeThreads) ce_mean_kernel(const float* __restrict__ row_loss, int B, float* __restrict__ loss) {
    __shared__ float red[32];
    float s = 0.0f;
    for (int b = threadIdx.x; b < B; b += kCeThreads) s += row_loss[b];
    s = block_reduce<false>(s, red);
    if (threadIdx.x == 0) *loss = s / static_cast<float>(B);
}

}  // namespace y5

using namespace y5;

extern "C" Y5_API int y5_global_avg_pool(const void* x, int32_t x_pitch, void* y, int32_t y_pitch, int32_t batch, int32_t h, int32_t w, int32_t c,
                                         int32_t dtype, void* stream) {
    if (!x || !y || batch <= 0 || h <= 0 || w <= 0 || c <= 0 || x_pitch < c || y_pitch < c) return set_error(Y5_E_INVALID, "global_avg_pool: bad arguments");
    if (c % 8 || x_pitch % 8 || y_pitch % 8 || (dtype != Y5_F16 && dtype != Y5_BF16))
        return set_error(Y5_E_UNSUPPORTED, "global_avg_pool: c/pitch %% 8, fp16/bf16 only");
    const long long total = static_cast<long long>(batch) * (c / 8);
    const int threads = 128, grid = grid_stride_ctas(total, threads, 16);
    return launch("global_avg_pool", gap_fwd_kernel, {grid, threads, 0, static_cast<cudaStream_t>(stream)}, static_cast<const uint16_t*>(x),
                  x_pitch, static_cast<uint16_t*>(y), y_pitch, batch, h * w, c, dtype == Y5_BF16);
}

extern "C" Y5_API int y5_global_avg_pool_bwd(const void* dy, int32_t dy_pitch, void* dx, int32_t dx_pitch, int32_t batch, int32_t h, int32_t w,
                                             int32_t c, int32_t dtype, void* stream) {
    if (!dy || !dx || batch <= 0 || h <= 0 || w <= 0 || c <= 0 || dy_pitch < c || dx_pitch < c)
        return set_error(Y5_E_INVALID, "global_avg_pool_bwd: bad arguments");
    if (c % 8 || dy_pitch % 8 || dx_pitch % 8 || (dtype != Y5_F16 && dtype != Y5_BF16))
        return set_error(Y5_E_UNSUPPORTED, "global_avg_pool_bwd: c/pitch %% 8, fp16/bf16 only");
    const long long total = static_cast<long long>(batch) * h * w * (c / 8);
    const int threads = 256, grid = grid_stride_ctas(total, threads, 16);
    return launch("global_avg_pool_bwd", gap_bwd_kernel, {grid, threads, 0, static_cast<cudaStream_t>(stream)},
                  static_cast<const uint16_t*>(dy), dy_pitch, static_cast<uint16_t*>(dx), dx_pitch, batch, h * w, c, dtype == Y5_BF16);
}

extern "C" Y5_API int y5_cross_entropy(const void* logits, int32_t dtype, int32_t batch, int32_t nc, int64_t row_stride, const int64_t* labels,
                                       float label_smoothing, const float* grad_scale, void* dlogits, int64_t dlogits_stride, float* row_loss,
                                       float* loss, void* stream) {
    if (!logits || !labels || !row_loss || !loss || batch <= 0 || nc < 2 || row_stride < nc || (dlogits && dlogits_stride < nc))
        return set_error(Y5_E_INVALID, "cross_entropy: bad arguments");
    if (!(label_smoothing >= 0.0f && label_smoothing <= 1.0f)) return set_error(Y5_E_INVALID, "cross_entropy: label_smoothing outside [0, 1]");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const long long* lab = reinterpret_cast<const long long*>(labels);
    int e;
    switch (dtype) {
        case Y5_F16:
            e = launch("cross_entropy", ce_row_kernel<__half>, {batch, kCeThreads, 0, st}, static_cast<const __half*>(logits), row_stride, nc,
                       lab, label_smoothing, grad_scale, static_cast<__half*>(dlogits), dlogits_stride, row_loss, batch);
            break;
        case Y5_BF16:
            e = launch("cross_entropy", ce_row_kernel<__nv_bfloat16>, {batch, kCeThreads, 0, st}, static_cast<const __nv_bfloat16*>(logits),
                       row_stride, nc, lab, label_smoothing, grad_scale, static_cast<__nv_bfloat16*>(dlogits), dlogits_stride, row_loss, batch);
            break;
        case Y5_F32:
            e = launch("cross_entropy", ce_row_kernel<float>, {batch, kCeThreads, 0, st}, static_cast<const float*>(logits), row_stride, nc,
                       lab, label_smoothing, grad_scale, static_cast<float*>(dlogits), dlogits_stride, row_loss, batch);
            break;
        default: return set_error(Y5_E_UNSUPPORTED, "cross_entropy: logits dtype %d (fp16 / bf16 / fp32)", dtype);
    }
    if (e) return e;
    return launch("cross_entropy mean", ce_mean_kernel, {1, kCeThreads, 0, st}, row_loss, batch, loss);
}
