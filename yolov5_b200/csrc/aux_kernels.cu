// HBM-bound data-movement kernels of the forward path: stem space-to-depth (+ u8 -> fp16 /255), SPPF pooling,
// 2x nearest upsample into a concat slice, strided view copy, NHWC -> NCHW export.
// All of them move 16-byte vectors (8 fp16/bf16 channels) per thread with the channel index fastest, so a warp
// touches 512 contiguous bytes.  max() on fp16/bf16 bit patterns is done in fp32 (exact).  SPPF's max propagates NaN the way
// F.max_pool2d does: a NaN anywhere in a window makes that window's maximum NaN.
#include "../../include/y5b200.h"
#include "common.cuh"
#include "host_util.h"

namespace y5 {

// ---------------------------------------------------------------------------------------------------------------------
// stem: NCHW image -> 2x2 space-to-depth NHWC, 16 channels ((dy*2+dx)*3 + c, 12 used)
// Replaces detect.py:206-208 / val.py:259-262 (`im.half(); im /= 255`) and turns the 6x6/s2/p2 stem conv
// (models/yolov5s.yaml:20) into a 3x3/s1/p1 conv: input pixel (2i+dy, 2j+dx) lands in cell (i,j).
// ---------------------------------------------------------------------------------------------------------------------
template <typename T>
__device__ __forceinline__ float load_px(const T* p);
template <> __device__ __forceinline__ float load_px<uint8_t>(const uint8_t* p) { return static_cast<float>(*p) / 255.0f; }
template <> __device__ __forceinline__ float load_px<__half>(const __half* p) { return __half2float(*p); }
template <> __device__ __forceinline__ float load_px<__nv_bfloat16>(const __nv_bfloat16* p) { return __bfloat162float(*p); }
template <> __device__ __forceinline__ float load_px<float>(const float* p) { return *p; }

template <typename T>
__global__ void stem_s2d_kernel(const T* __restrict__ img, uint4* __restrict__ out, int B, int H, int W, int bf16, int row_px,
                                int x_off) {
    const int Wo = W >> 1, Ho = H >> 1;
    const long long total = static_cast<long long>(B) * Ho * Wo;
    for (long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; idx < total;
         idx += static_cast<long long>(gridDim.x) * blockDim.x) {
        const int ox = static_cast<int>(idx % Wo);
        const int oy = static_cast<int>((idx / Wo) % Ho);
        const int b = static_cast<int>(idx / (static_cast<long long>(Wo) * Ho));
        float v[16];
#pragma unroll
        for (int dy = 0; dy < 2; ++dy)
#pragma unroll
            for (int dx = 0; dx < 2; ++dx)
#pragma unroll
                for (int c = 0; c < 3; ++c)
                    v[(dy * 2 + dx) * 3 + c] =
                        load_px<T>(img + ((static_cast<long long>(b) * 3 + c) * H + (2 * oy + dy)) * W + (2 * ox + dx));
        v[12] = v[13] = v[14] = v[15] = 0.0f;
        uint4 lo, hi;
        lo.x = pack2(v[0], v[1], bf16); lo.y = pack2(v[2], v[3], bf16); lo.z = pack2(v[4], v[5], bf16); lo.w = pack2(v[6], v[7], bf16);
        hi.x = pack2(v[8], v[9], bf16); hi.y = pack2(v[10], v[11], bf16); hi.z = pack2(v[12], v[13], bf16); hi.w = pack2(v[14], v[15], bf16);
        const long long opx = (static_cast<long long>(b) * Ho + oy) * row_px + x_off + ox;  // row_px >= Wo: zero border columns
        out[opx * 2] = lo;
        out[opx * 2 + 1] = hi;
    }
}

// ---------------------------------------------------------------------------------------------------------------------
// plain first layer (models/hub/yolov3*.yaml: Conv(3, c, 3, 1)): NCHW image -> NHWC [B][H][W][out_c], channels 0..2 the
// image, the rest zero, so the conv GEMM reads it as an out_c-channel map.  One thread per (pixel, 8-channel vector).
// ---------------------------------------------------------------------------------------------------------------------
template <typename T>
__global__ void image_nhwc_kernel(const T* __restrict__ img, uint4* __restrict__ out, int B, int H, int W, int cv, int bf16) {
    const long long total = static_cast<long long>(B) * H * W * cv;
    for (long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; idx < total;
         idx += static_cast<long long>(gridDim.x) * blockDim.x) {
        const int c8 = static_cast<int>(idx % cv);
        const long long pix = idx / cv;
        uint4 o = make_uint4(0, 0, 0, 0);
        if (c8 == 0) {
            const long long hw = static_cast<long long>(H) * W, n = pix / hw, p = pix - n * hw;
            const T* src = img + n * 3 * hw + p;
            o.x = pack2(load_px<T>(src), load_px<T>(src + hw), bf16);
            o.y = pack2(load_px<T>(src + 2 * hw), 0.0f, bf16);
        }
        out[idx] = o;
    }
}

// ---------------------------------------------------------------------------------------------------------------------
// SPPF: y1 = maxpool_k(x), y2 = maxpool_k(y1), y3 = maxpool_k(y2) with stride 1, pad k/2 (implicit -inf padding).
// Chained stride-1 max pools compose: y2 is the (2k-1)-window max, y3 the (3k-2)-window max of x, so all three
// come from one pass over the 13x13 neighbourhood (k=5).  One thread per (pixel, 8-channel vector).
// ---------------------------------------------------------------------------------------------------------------------
// max that keeps NaN (fmaxf returns the other operand): once acc is NaN, 'v > acc' is false and acc stays NaN
__device__ __forceinline__ float max_nan(float acc, float v) { return (v > acc || v != v) ? v : acc; }
__device__ __forceinline__ void vmax8(float (&acc)[8], const uint4& v, bool bf16) {
    const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        const float2 t = unpack2(w[j], bf16);
        acc[2 * j] = max_nan(acc[2 * j], t.x);
        acc[2 * j + 1] = max_nan(acc[2 * j + 1], t.y);
    }
}
__device__ __forceinline__ uint4 pack8(const float (&f)[8], bool bf16) {
    uint4 o;
    o.x = pack2(f[0], f[1], bf16); o.y = pack2(f[2], f[3], bf16); o.z = pack2(f[4], f[5], bf16); o.w = pack2(f[6], f[7], bf16);
    return o;
}

__global__ void sppf_pool_kernel(const uint16_t* __restrict__ x, int x_pitch, uint16_t* y1, uint16_t* y2, uint16_t* y3,
                                 int y_pitch, int B, int H, int W, int C, int k, int bf16) {
    const int cv = C >> 3;
    const long long total = static_cast<long long>(B) * H * W * cv;
    const int r1 = k / 2, r2 = 2 * (k / 2), r3 = 3 * (k / 2);
    for (long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; idx < total;
         idx += static_cast<long long>(gridDim.x) * blockDim.x) {
        const int c8 = static_cast<int>(idx % cv);
        const long long pix = idx / cv;
        const int px = static_cast<int>(pix % W);
        const int py = static_cast<int>((pix / W) % H);
        const int b = static_cast<int>(pix / (static_cast<long long>(W) * H));
        float m1[8], m2[8], m3[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) m1[j] = m2[j] = m3[j] = -INFINITY;
        for (int dy = -r3; dy <= r3; ++dy) {
            const int yy = py + dy;
            if (yy < 0 || yy >= H) continue;
            const int ady = dy < 0 ? -dy : dy;
            for (int dx = -r3; dx <= r3; ++dx) {
                const int xx = px + dx;
                if (xx < 0 || xx >= W) continue;
                const int adx = dx < 0 ? -dx : dx;
                const int cheb = ady > adx ? ady : adx;
                const uint4 v = *reinterpret_cast<const uint4*>(
                    x + ((static_cast<long long>(b) * H + yy) * W + xx) * x_pitch + c8 * 8);
                vmax8(m3, v, bf16);
                if (cheb <= r2) vmax8(m2, v, bf16);
                if (cheb <= r1) vmax8(m1, v, bf16);
            }
        }
        const long long o = pix * y_pitch + c8 * 8;
        *reinterpret_cast<uint4*>(y1 + o) = pack8(m1, bf16);
        *reinterpret_cast<uint4*>(y2 + o) = pack8(m2, bf16);
        *reinterpret_cast<uint4*>(y3 + o) = pack8(m3, bf16);
    }
}

// Shared-memory version: one CTA per (image, 8-channel vector).  The H x W plane of that vector sits in smem
// (uint4 per pixel) and each k x k / stride-1 max-pool is done separably (row max then column max), three times in a
// row exactly as the reference chains them; y1, y2, y3 are written as they are produced.  Reads each input element
// once from HBM and writes 3 outputs: the algorithmic minimum.  __hmax2_nan, not __hmax2, so NaN propagates.
__device__ __forceinline__ uint4 max8(const uint4& a, const uint4& b, bool bf16) {
    const uint32_t aw[4] = {a.x, a.y, a.z, a.w}, bw[4] = {b.x, b.y, b.z, b.w};
    uint32_t o[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        if (bf16) {
            __nv_bfloat162 r = __hmax2_nan(*reinterpret_cast<const __nv_bfloat162*>(&aw[j]), *reinterpret_cast<const __nv_bfloat162*>(&bw[j]));
            o[j] = *reinterpret_cast<uint32_t*>(&r);
        } else {
            __half2 r = __hmax2_nan(*reinterpret_cast<const __half2*>(&aw[j]), *reinterpret_cast<const __half2*>(&bw[j]));
            o[j] = *reinterpret_cast<uint32_t*>(&r);
        }
    }
    return make_uint4(o[0], o[1], o[2], o[3]);
}

__global__ void sppf_pool_smem_kernel(const uint16_t* __restrict__ x, int x_pitch, uint16_t* y1, uint16_t* y2, uint16_t* y3,
                                      int y_pitch, int H, int W, int C, int k, int bf16) {
    extern __shared__ uint4 plane[];  // [2][H*W]
    const int cv = C >> 3;
    const int b = blockIdx.x / cv, c8 = blockIdx.x - b * cv;
    const int HW = H * W, r = k / 2;
    uint4* cur = plane;
    uint4* tmp = plane + HW;
    const long long base = static_cast<long long>(b) * HW;
    for (int i = threadIdx.x; i < HW; i += blockDim.x) cur[i] = *reinterpret_cast<const uint4*>(x + (base + i) * x_pitch + c8 * 8);
    __syncthreads();
    uint16_t* outs[3] = {y1, y2, y3};
    for (int pass = 0; pass < 3; ++pass) {
        for (int i = threadIdx.x; i < HW; i += blockDim.x) {  // row max
            const int py = i / W, px = i - py * W;
            uint4 m = cur[i];
            for (int d = 1; d <= r; ++d) {
                if (px - d >= 0) m = max8(m, cur[i - d], bf16);
                if (px + d < W) m = max8(m, cur[i + d], bf16);
            }
            tmp[i] = m;
        }
        __syncthreads();
        for (int i = threadIdx.x; i < HW; i += blockDim.x) {  // column max
            const int py = i / W;
            uint4 m = tmp[i];
            for (int d = 1; d <= r; ++d) {
                if (py - d >= 0) m = max8(m, tmp[i - d * W], bf16);
                if (py + d < H) m = max8(m, tmp[i + d * W], bf16);
            }
            cur[i] = m;  // safe: this pass reads only tmp
            *reinterpret_cast<uint4*>(outs[pass] + (base + i) * y_pitch + c8 * 8) = m;
        }
        __syncthreads();
    }
}

// ---------------------------------------------------------------------------------------------------------------------
// nearest 2x upsample into a (strided) view; one thread per (output pixel, 8-channel vector)
// ---------------------------------------------------------------------------------------------------------------------
__global__ void upsample2x_kernel(const uint16_t* __restrict__ x, int x_pitch, uint16_t* __restrict__ y, int y_pitch, int B,
                                  int H, int W, int C) {
    griddep_wait();  // PDL: the predecessor kernel has completed and flushed beyond this point
    griddep_launch_dependents();
    const int cv = C >> 3;
    const int Ho = 2 * H, Wo = 2 * W;
    const long long total = static_cast<long long>(B) * Ho * Wo * cv;
    for (long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; idx < total;
         idx += static_cast<long long>(gridDim.x) * blockDim.x) {
        const int c8 = static_cast<int>(idx % cv);
        const long long pix = idx / cv;
        const int ox = static_cast<int>(pix % Wo);
        const int oy = static_cast<int>((pix / Wo) % Ho);
        const int b = static_cast<int>(pix / (static_cast<long long>(Wo) * Ho));
        const uint4 v = *reinterpret_cast<const uint4*>(
            x + ((static_cast<long long>(b) * H + (oy >> 1)) * W + (ox >> 1)) * x_pitch + c8 * 8);
        *reinterpret_cast<uint4*>(y + pix * y_pitch + c8 * 8) = v;
    }
}

__global__ void copy_view_kernel(const uint16_t* __restrict__ x, int x_pitch, uint16_t* __restrict__ y, int y_pitch,
                                 long long pixels, int C) {
    griddep_wait();  // PDL: the predecessor kernel has completed and flushed beyond this point
    griddep_launch_dependents();
    const int cv = C >> 3;
    const long long total = pixels * cv;
    for (long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; idx < total;
         idx += static_cast<long long>(gridDim.x) * blockDim.x) {
        const int c8 = static_cast<int>(idx % cv);
        const long long pix = idx / cv;
        *reinterpret_cast<uint4*>(y + pix * y_pitch + c8 * 8) = *reinterpret_cast<const uint4*>(x + pix * x_pitch + c8 * 8);
    }
}

// NHWC view -> dense NCHW through a 32x32 shared-memory transpose tile (coalesced on both sides)
__global__ void nhwc_to_nchw_kernel(const uint16_t* __restrict__ x, int x_pitch, uint16_t* __restrict__ y, int HW, int C) {
    __shared__ uint16_t tile[32][33];
    const int b = blockIdx.z;
    const int p0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
    for (int i = threadIdx.y; i < 32; i += blockDim.y) {
        const int p = p0 + i, c = c0 + threadIdx.x;
        if (p < HW && c < C) tile[i][threadIdx.x] = x[(static_cast<long long>(b) * HW + p) * x_pitch + c];
    }
    __syncthreads();
    for (int i = threadIdx.y; i < 32; i += blockDim.y) {
        const int c = c0 + i, p = p0 + threadIdx.x;
        if (p < HW && c < C) y[(static_cast<long long>(b) * C + c) * HW + p] = tile[threadIdx.x][i];
    }
}

}  // namespace y5

using namespace y5;

static bool half_dtype(int d) { return d == Y5_F16 || d == Y5_BF16; }
// a view the kernels read or write in 16-byte vectors: aligned base, pitch covering its channels
static bool vec_view(const void* p, int pitch, int c) { return !(reinterpret_cast<uintptr_t>(p) & 15) && pitch >= c; }

extern "C" Y5_API int y5_stem_s2d(const void* img, int32_t img_dtype, void* out, int32_t out_dtype, int32_t batch, int32_t h, int32_t w,
                                  int32_t out_row_px, int32_t out_x_off, void* stream) {
    const int row_px = out_row_px > 0 ? out_row_px : w / 2;
    if (out_x_off < 0 || out_x_off + w / 2 > row_px) return set_error(Y5_E_INVALID, "stem_s2d: output row pitch/offset do not cover the row");
    if (!img || !out || batch <= 0 || h <= 0 || w <= 0 || (h & 1) || (w & 1)) return set_error(Y5_E_INVALID, "stem_s2d: bad arguments (h, w must be even)");
    if (!half_dtype(out_dtype)) return set_error(Y5_E_UNSUPPORTED, "stem_s2d: output dtype must be fp16/bf16");
    if (reinterpret_cast<uintptr_t>(out) & 15) return set_error(Y5_E_INVALID, "stem_s2d: output must be 16-byte aligned");
    const long long total = static_cast<long long>(batch) * (h / 2) * (w / 2);
    const int threads = 256, grid = grid_stride_ctas(total, threads, 16);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const int bf = out_dtype == Y5_BF16;
    uint4* o = static_cast<uint4*>(out);
    switch (img_dtype) {
        case Y5_U8: return launch("stem_s2d", stem_s2d_kernel<uint8_t>, {grid, threads, 0, st}, static_cast<const uint8_t*>(img), o, batch, h, w, bf, row_px, out_x_off);
        case Y5_F16: return launch("stem_s2d", stem_s2d_kernel<__half>, {grid, threads, 0, st}, static_cast<const __half*>(img), o, batch, h, w, bf, row_px, out_x_off);
        case Y5_BF16: return launch("stem_s2d", stem_s2d_kernel<__nv_bfloat16>, {grid, threads, 0, st}, static_cast<const __nv_bfloat16*>(img), o, batch, h, w, bf, row_px, out_x_off);
        case Y5_F32: return launch("stem_s2d", stem_s2d_kernel<float>, {grid, threads, 0, st}, static_cast<const float*>(img), o, batch, h, w, bf, row_px, out_x_off);
        default: return set_error(Y5_E_UNSUPPORTED, "stem_s2d: image dtype %d", img_dtype);
    }
}

extern "C" Y5_API int y5_image_nhwc(const void* img, int32_t img_dtype, void* out, int32_t out_dtype, int32_t batch, int32_t h, int32_t w,
                                    int32_t out_c, void* stream) {
    if (!img || !out || batch <= 0 || h <= 0 || w <= 0 || out_c < 8 || out_c % 8) return set_error(Y5_E_INVALID, "image_nhwc: bad arguments (out_c a multiple of 8)");
    if (!half_dtype(out_dtype)) return set_error(Y5_E_UNSUPPORTED, "image_nhwc: output dtype must be fp16/bf16");
    if (reinterpret_cast<uintptr_t>(out) & 15) return set_error(Y5_E_INVALID, "image_nhwc: output must be 16-byte aligned");
    const int cv = out_c / 8;
    const long long total = static_cast<long long>(batch) * h * w * cv;
    const int threads = 256, grid = grid_stride_ctas(total, threads, 16);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const int bf = out_dtype == Y5_BF16;
    uint4* o = static_cast<uint4*>(out);
    switch (img_dtype) {
        case Y5_U8: return launch("image_nhwc", image_nhwc_kernel<uint8_t>, {grid, threads, 0, st}, static_cast<const uint8_t*>(img), o, batch, h, w, cv, bf);
        case Y5_F16: return launch("image_nhwc", image_nhwc_kernel<__half>, {grid, threads, 0, st}, static_cast<const __half*>(img), o, batch, h, w, cv, bf);
        case Y5_BF16: return launch("image_nhwc", image_nhwc_kernel<__nv_bfloat16>, {grid, threads, 0, st}, static_cast<const __nv_bfloat16*>(img), o, batch, h, w, cv, bf);
        case Y5_F32: return launch("image_nhwc", image_nhwc_kernel<float>, {grid, threads, 0, st}, static_cast<const float*>(img), o, batch, h, w, cv, bf);
        default: return set_error(Y5_E_UNSUPPORTED, "image_nhwc: image dtype %d", img_dtype);
    }
}

extern "C" Y5_API int y5_sppf_pool(const void* x, int32_t x_pitch, void* y1, void* y2, void* y3, int32_t y_pitch, int32_t batch, int32_t h,
                            int32_t w, int32_t c, int32_t ksize, int32_t dtype, void* stream) {
    if (!x || !y1 || !y2 || !y3 || batch <= 0 || h <= 0 || w <= 0 || c <= 0) return set_error(Y5_E_INVALID, "sppf_pool: bad arguments");
    if (c % 8 || x_pitch % 8 || y_pitch % 8 || !half_dtype(dtype) || !(ksize & 1)) return set_error(Y5_E_UNSUPPORTED, "sppf_pool: c/pitch %% 8, odd k, fp16/bf16 only");
    if (!vec_view(x, x_pitch, c) || !vec_view(y1, y_pitch, c) || !vec_view(y2, y_pitch, c) || !vec_view(y3, y_pitch, c))
        return set_error(Y5_E_INVALID, "sppf_pool: views must be 16-byte aligned with pitch >= c");
    const size_t smem = static_cast<size_t>(2) * h * w * sizeof(uint4);
    if (smem <= 96 * 1024 && static_cast<long long>(batch) * (c / 8) < 0x7fffffff) {
        if (ensure_dyn_smem(reinterpret_cast<const void*>(sppf_pool_smem_kernel), 96 * 1024) != cudaSuccess)
            return set_error(Y5_E_DRIVER, "sppf_pool: cudaFuncSetAttribute(MaxDynamicSharedMemorySize) failed");
        return launch("sppf_pool", sppf_pool_smem_kernel, {batch * (c / 8), 256, smem, static_cast<cudaStream_t>(stream)},
                      static_cast<const uint16_t*>(x), x_pitch, static_cast<uint16_t*>(y1), static_cast<uint16_t*>(y2),
                      static_cast<uint16_t*>(y3), y_pitch, h, w, c, ksize, dtype == Y5_BF16);
    }
    const long long total = static_cast<long long>(batch) * h * w * (c / 8);
    const int threads = 128, grid = grid_stride_ctas(total, threads, 16);
    return launch("sppf_pool", sppf_pool_kernel, {grid, threads, 0, static_cast<cudaStream_t>(stream)}, static_cast<const uint16_t*>(x),
                  x_pitch, static_cast<uint16_t*>(y1), static_cast<uint16_t*>(y2), static_cast<uint16_t*>(y3), y_pitch, batch, h, w, c,
                  ksize, dtype == Y5_BF16);
}

extern "C" Y5_API int y5_upsample2x(const void* x, int32_t x_pitch, void* y, int32_t y_pitch, int32_t batch, int32_t h, int32_t w, int32_t c,
                             int32_t dtype, void* stream) {
    if (!x || !y || batch <= 0 || h <= 0 || w <= 0 || c <= 0) return set_error(Y5_E_INVALID, "upsample2x: bad arguments");
    if (c % 8 || x_pitch % 8 || y_pitch % 8 || !half_dtype(dtype)) return set_error(Y5_E_UNSUPPORTED, "upsample2x: c/pitch %% 8, fp16/bf16 only");
    if (!vec_view(x, x_pitch, c) || !vec_view(y, y_pitch, c)) return set_error(Y5_E_INVALID, "upsample2x: views must be 16-byte aligned with pitch >= c");
    const long long total = static_cast<long long>(batch) * 4 * h * w * (c / 8);
    const int threads = 256, grid = grid_stride_ctas(total, threads, 16);
    return launch("upsample2x", upsample2x_kernel, {grid, threads, 0, static_cast<cudaStream_t>(stream), /*pdl=*/true},
                  static_cast<const uint16_t*>(x), x_pitch, static_cast<uint16_t*>(y), y_pitch, batch, h, w, c);
}

extern "C" Y5_API int y5_copy_view(const void* x, int32_t x_pitch, void* y, int32_t y_pitch, int64_t pixels, int32_t c, int32_t dtype,
                            void* stream) {
    if (!x || !y || pixels <= 0 || c <= 0) return set_error(Y5_E_INVALID, "copy_view: bad arguments");
    if (c % 8 || x_pitch % 8 || y_pitch % 8 || !half_dtype(dtype)) return set_error(Y5_E_UNSUPPORTED, "copy_view: c/pitch %% 8, fp16/bf16 only");
    if (!vec_view(x, x_pitch, c) || !vec_view(y, y_pitch, c)) return set_error(Y5_E_INVALID, "copy_view: views must be 16-byte aligned with pitch >= c");
    const long long total = pixels * (c / 8);
    const int threads = 256, grid = grid_stride_ctas(total, threads, 16);
    return launch("copy_view", copy_view_kernel, {grid, threads, 0, static_cast<cudaStream_t>(stream), /*pdl=*/true},
                  static_cast<const uint16_t*>(x), x_pitch, static_cast<uint16_t*>(y), y_pitch, pixels, c);
}

extern "C" Y5_API int y5_nhwc_to_nchw(const void* x, int32_t x_pitch, void* y, int32_t batch, int32_t h, int32_t w, int32_t c, int32_t dtype,
                               void* stream) {
    if (!x || !y || batch <= 0 || h <= 0 || w <= 0 || c <= 0 || !half_dtype(dtype)) return set_error(Y5_E_INVALID, "nhwc_to_nchw: bad arguments");
    if (batch > 65535) return set_error(Y5_E_UNSUPPORTED, "nhwc_to_nchw: batch > 65535");
    const int HW = h * w;
    dim3 grid((HW + 31) / 32, (c + 31) / 32, batch), block(32, 8);
    return launch("nhwc_to_nchw", nhwc_to_nchw_kernel, {grid, block, 0, static_cast<cudaStream_t>(stream)}, static_cast<const uint16_t*>(x),
                  x_pitch, static_cast<uint16_t*>(y), HW, c);
}
