// Max-pool kernels of the YOLOv3 models (models/hub/yolov3*.yaml) over NHWC channel-slice views, fp16 / bf16 / fp32:
//   Y5_POOL_K2S2       nn.MaxPool2d(2, 2, 0): (h, w) -> (h/2, w/2), floor
//   Y5_POOL_K2S1_ZPAD  nn.ZeroPad2d((0, 1, 0, 1)) then nn.MaxPool2d(2, 1, 0): (h, w) -> (h, w).  The pad cells right of and
//                      below the map hold 0, so a border window's maximum includes 0 (and is 0 when its cells are negative).
// and the backward of SPP's three stride-1 pools (windows k, 2k-1, 3k-2 with -inf padding; the forward is y5_sppf_pool).
//
// Tie rule of every backward: a window's gradient goes to its first maximum in row-major window order, and a NaN takes it
// from any earlier cell -- torch's max_pool2d (`val > max || isnan(val)`).  A window whose maximum is a zero-pad cell routes
// its gradient nowhere.  Every backward is a gather: each input element sums, in fp32 and in a fixed order, the gradients
// of the windows that chose it and is rounded once.  No atomics, so the result does not depend on scheduling.
//
// One thread per (pixel, 8-channel vector); the channel index is fastest, so a warp reads contiguous bytes.
#include "../../include/y5b200.h"
#include "common.cuh"
#include "host_util.h"

namespace {

using namespace y5;

template <typename T> struct Vec8;
template <> struct Vec8<uint16_t> {  // fp16 / bf16 bit patterns: one 16-byte vector
    static __device__ __forceinline__ void load(const uint16_t* p, bool bf16, float (&f)[8]) {
        const uint4 v = *reinterpret_cast<const uint4*>(p);
        const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const float2 t = unpack2(w[j], bf16);
            f[2 * j] = t.x;
            f[2 * j + 1] = t.y;
        }
    }
    static __device__ __forceinline__ void store(uint16_t* p, bool bf16, const float (&f)[8]) {
        *reinterpret_cast<uint4*>(p) = make_uint4(pack2(f[0], f[1], bf16), pack2(f[2], f[3], bf16), pack2(f[4], f[5], bf16), pack2(f[6], f[7], bf16));
    }
};
template <> struct Vec8<float> {  // two 16-byte vectors
    static __device__ __forceinline__ void load(const float* p, bool, float (&f)[8]) {
        const float4 a = *reinterpret_cast<const float4*>(p), b = *reinterpret_cast<const float4*>(p + 4);
        f[0] = a.x; f[1] = a.y; f[2] = a.z; f[3] = a.w; f[4] = b.x; f[5] = b.y; f[6] = b.z; f[7] = b.w;
    }
    static __device__ __forceinline__ void store(float* p, bool, const float (&f)[8]) {
        *reinterpret_cast<float4*>(p) = make_float4(f[0], f[1], f[2], f[3]);
        *reinterpret_cast<float4*>(p + 4) = make_float4(f[4], f[5], f[6], f[7]);
    }
};

// torch's scan step: take v when it is larger than the running maximum or NaN
__device__ __forceinline__ bool takes(float v, float best) { return v > best || v != v; }

// the 2x2 window of output (oy, ox): top-left input cell, and the value of window cell j = dy*2 + dx (0 for a zero-pad cell)
template <typename T, int MODE>
__device__ __forceinline__ void window_cell(const T* x, int x_pitch, long long img, int H, int W, int y0, int x0, int j, int c8, bool bf16,
                                            float (&v)[8]) {
    const int yy = y0 + (j >> 1), xx = x0 + (j & 1);
    if (MODE == Y5_POOL_K2S1_ZPAD && (yy >= H || xx >= W)) {
#pragma unroll
        for (int i = 0; i < 8; ++i) v[i] = 0.f;
        return;
    }
    Vec8<T>::load(x + ((img * H + yy) * W + xx) * x_pitch + c8 * 8, bf16, v);
}

template <typename T, int MODE>
__global__ void maxpool2_fwd_kernel(const T* __restrict__ x, int x_pitch, T* __restrict__ y, int y_pitch, int B, int H, int W, int Ho,
                                    int Wo, int C, int bf16) {
    const int cv = C >> 3;
    const long long total = static_cast<long long>(B) * Ho * Wo * cv;
    for (long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; idx < total;
         idx += static_cast<long long>(gridDim.x) * blockDim.x) {
        const int c8 = static_cast<int>(idx % cv);
        const long long pix = idx / cv;
        const int ox = static_cast<int>(pix % Wo);
        const int oy = static_cast<int>((pix / Wo) % Ho);
        const long long n = pix / (static_cast<long long>(Wo) * Ho);
        const int s = MODE == Y5_POOL_K2S2 ? 2 : 1;
        float m[8], v[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) m[i] = -INFINITY;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            window_cell<T, MODE>(x, x_pitch, n, H, W, oy * s, ox * s, j, c8, bf16 != 0, v);
#pragma unroll
            for (int i = 0; i < 8; ++i)
                if (takes(v[i], m[i])) m[i] = v[i];
        }
        Vec8<T>::store(y + pix * y_pitch + c8 * 8, bf16 != 0, m);
    }
}

// dx of one input pixel: the windows containing it, in row-major output order (as torch's backward sums them)
template <typename T, int MODE>
__global__ void maxpool2_bwd_kernel(const T* __restrict__ x, int x_pitch, const T* __restrict__ dy, int dy_pitch, T* __restrict__ dx,
                                    int dx_pitch, int B, int H, int W, int Ho, int Wo, int C, int bf16) {
    const int cv = C >> 3;
    const long long total = static_cast<long long>(B) * H * W * cv;
    const int s = MODE == Y5_POOL_K2S2 ? 2 : 1;
    for (long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; idx < total;
         idx += static_cast<long long>(gridDim.x) * blockDim.x) {
        const int c8 = static_cast<int>(idx % cv);
        const long long pix = idx / cv;
        const int ix = static_cast<int>(pix % W);
        const int iy = static_cast<int>((pix / W) % H);
        const long long n = pix / (static_cast<long long>(W) * H);
        float acc[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) acc[i] = 0.f;
        const int oy0 = MODE == Y5_POOL_K2S2 ? iy / 2 : max(iy - 1, 0), oy1 = MODE == Y5_POOL_K2S2 ? iy / 2 : iy;
        const int ox0 = MODE == Y5_POOL_K2S2 ? ix / 2 : max(ix - 1, 0), ox1 = MODE == Y5_POOL_K2S2 ? ix / 2 : ix;
        for (int oy = oy0; oy <= oy1 && oy < Ho; ++oy)
            for (int ox = ox0; ox <= ox1 && ox < Wo; ++ox) {
                const int self = (iy - oy * s) * 2 + (ix - ox * s);
                float best[8], v[8];
                int arg[8];
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    window_cell<T, MODE>(x, x_pitch, n, H, W, oy * s, ox * s, j, c8, bf16 != 0, v);
#pragma unroll
                    for (int i = 0; i < 8; ++i)
                        if (j == 0 || takes(v[i], best[i])) {
                            best[i] = v[i];
                            arg[i] = j;
                        }
                }
                float g[8];
                Vec8<T>::load(dy + ((n * Ho + oy) * Wo + ox) * dy_pitch + c8 * 8, bf16 != 0, g);
#pragma unroll
                for (int i = 0; i < 8; ++i)
                    if (arg[i] == self) acc[i] += g[i];
            }
        Vec8<T>::store(dx + pix * dx_pitch + c8 * 8, bf16 != 0, acc);
    }
}

// SPP backward, pass 1: for every position q and each window size (k, 2k-1, 3k-2) around it, the offset of the window's
// arg-max, coded (dy + R) * (2R + 1) + (dx + R) with R = the largest radius.  The windows are concentric, so one row-major
// scan of the largest visits each smaller window's cells in its own row-major order.
template <typename T>
__global__ void spp_argmax_kernel(const T* __restrict__ a, int a_pitch, uint16_t* __restrict__ code, int B, int H, int W, int C, int k,
                                  int bf16) {
    const int cv = C >> 3;
    const long long total = static_cast<long long>(B) * H * W * cv;
    const long long plane = static_cast<long long>(B) * H * W * C;
    const int r1 = k / 2, r2 = 2 * (k / 2), R = 3 * (k / 2), side = 2 * R + 1;
    for (long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; idx < total;
         idx += static_cast<long long>(gridDim.x) * blockDim.x) {
        const int c8 = static_cast<int>(idx % cv);
        const long long pix = idx / cv;
        const int px = static_cast<int>(pix % W);
        const int py = static_cast<int>((pix / W) % H);
        const long long n = pix / (static_cast<long long>(W) * H);
        float best[3][8];
        int arg[3][8];
#pragma unroll
        for (int s = 0; s < 3; ++s)
#pragma unroll
            for (int i = 0; i < 8; ++i) {
                best[s][i] = -INFINITY;
                arg[s][i] = -1;
            }
        for (int dy = -R; dy <= R; ++dy) {
            const int yy = py + dy;
            if (yy < 0 || yy >= H) continue;
            const int ady = dy < 0 ? -dy : dy;
            for (int dx = -R; dx <= R; ++dx) {
                const int xx = px + dx;
                if (xx < 0 || xx >= W) continue;
                const int adx = dx < 0 ? -dx : dx;
                const int cheb = ady > adx ? ady : adx;
                const int cell = (dy + R) * side + (dx + R);
                float v[8];
                Vec8<T>::load(a + ((n * H + yy) * W + xx) * a_pitch + c8 * 8, bf16 != 0, v);
#pragma unroll
                for (int s = 0; s < 3; ++s) {
                    if (cheb > (s == 0 ? r1 : s == 1 ? r2 : R)) continue;
#pragma unroll
                    for (int i = 0; i < 8; ++i)
                        if (arg[s][i] < 0 || takes(v[i], best[s][i])) {
                            best[s][i] = v[i];
                            arg[s][i] = cell;
                        }
                }
            }
        }
#pragma unroll
        for (int s = 0; s < 3; ++s) {
            uint4 o;
            o.x = static_cast<uint32_t>(arg[s][0]) | (static_cast<uint32_t>(arg[s][1]) << 16);
            o.y = static_cast<uint32_t>(arg[s][2]) | (static_cast<uint32_t>(arg[s][3]) << 16);
            o.z = static_cast<uint32_t>(arg[s][4]) | (static_cast<uint32_t>(arg[s][5]) << 16);
            o.w = static_cast<uint32_t>(arg[s][6]) | (static_cast<uint32_t>(arg[s][7]) << 16);
            *reinterpret_cast<uint4*>(code + s * plane + pix * C + c8 * 8) = o;
        }
    }
}

// SPP backward, pass 2: da = dcat[0] + the gradients of every k / 2k-1 / 3k-2 window whose arg-max is this element
template <typename T>
__global__ void spp_gather_kernel(const T* __restrict__ dcat, int dcat_pitch, const uint16_t* __restrict__ code, T* __restrict__ da,
                                  int da_pitch, int B, int H, int W, int C, int k, int bf16) {
    const int cv = C >> 3;
    const long long total = static_cast<long long>(B) * H * W * cv;
    const long long plane = static_cast<long long>(B) * H * W * C;
    const int R = 3 * (k / 2), side = 2 * R + 1;
    for (long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; idx < total;
         idx += static_cast<long long>(gridDim.x) * blockDim.x) {
        const int c8 = static_cast<int>(idx % cv);
        const long long pix = idx / cv;
        const int px = static_cast<int>(pix % W);
        const int py = static_cast<int>((pix / W) % H);
        const long long n = pix / (static_cast<long long>(W) * H);
        float acc[8];
        Vec8<T>::load(dcat + pix * dcat_pitch + c8 * 8, bf16 != 0, acc);
        for (int s = 0; s < 3; ++s) {
            const int r = (s + 1) * (k / 2);
            for (int qy = max(py - r, 0); qy <= min(py + r, H - 1); ++qy)
                for (int qx = max(px - r, 0); qx <= min(px + r, W - 1); ++qx) {
                    const long long q = (n * H + qy) * W + qx;
                    const uint4 o = *reinterpret_cast<const uint4*>(code + s * plane + q * C + c8 * 8);
                    const uint32_t self = static_cast<uint32_t>((py - qy + R) * side + (px - qx + R));
                    const uint32_t w[4] = {o.x, o.y, o.z, o.w};
                    bool any = false;
#pragma unroll
                    for (int i = 0; i < 4; ++i) any |= (w[i] & 0xffffu) == self || (w[i] >> 16) == self;
                    if (!any) continue;
                    float g[8];
                    Vec8<T>::load(dcat + q * dcat_pitch + (s + 1) * C + c8 * 8, bf16 != 0, g);
#pragma unroll
                    for (int i = 0; i < 8; ++i)
                        if (((w[i >> 1] >> (16 * (i & 1))) & 0xffffu) == self) acc[i] += g[i];
                }
        }
        Vec8<T>::store(da + pix * da_pitch + c8 * 8, bf16 != 0, acc);
    }
}

// a view the kernels move in 16-byte vectors: aligned base, pitch covering its channels and a multiple of 8 elements
bool vec_view(const void* p, int pitch, int c) { return p && !(reinterpret_cast<uintptr_t>(p) & 15) && pitch >= c && pitch % 8 == 0; }

bool pool_dtype(int d) { return d == Y5_F16 || d == Y5_BF16 || d == Y5_F32; }

int pool_out(int mode, int h, int w, int* ho, int* wo) {
    if (mode == Y5_POOL_K2S2) {
        *ho = h / 2;
        *wo = w / 2;
    } else if (mode == Y5_POOL_K2S1_ZPAD) {
        *ho = h;
        *wo = w;
    } else {
        return set_error(Y5_E_UNSUPPORTED, "maxpool2d: mode %d (Y5_POOL_K2S2 or Y5_POOL_K2S1_ZPAD)", mode);
    }
    if (*ho <= 0 || *wo <= 0) return set_error(Y5_E_INVALID, "maxpool2d: %dx%d input gives an empty output", h, w);
    return 0;
}

template <typename T>
int fwd_launch(int mode, const void* x, int xp, void* y, int yp, int B, int H, int W, int Ho, int Wo, int C, int bf, cudaStream_t st) {
    const int threads = 256, grid = grid_stride_ctas(static_cast<long long>(B) * Ho * Wo * (C / 8), threads, 16);
    auto* kernel = mode == Y5_POOL_K2S2 ? maxpool2_fwd_kernel<T, Y5_POOL_K2S2> : maxpool2_fwd_kernel<T, Y5_POOL_K2S1_ZPAD>;
    return launch("maxpool2d", kernel, {grid, threads, 0, st}, static_cast<const T*>(x), xp, static_cast<T*>(y), yp, B, H, W, Ho, Wo, C, bf);
}

template <typename T>
int bwd_launch(int mode, const void* x, int xp, const void* dy, int dyp, void* dx, int dxp, int B, int H, int W, int Ho, int Wo, int C, int bf,
               cudaStream_t st) {
    const int threads = 256, grid = grid_stride_ctas(static_cast<long long>(B) * H * W * (C / 8), threads, 16);
    auto* kernel = mode == Y5_POOL_K2S2 ? maxpool2_bwd_kernel<T, Y5_POOL_K2S2> : maxpool2_bwd_kernel<T, Y5_POOL_K2S1_ZPAD>;
    return launch("maxpool2d_bwd", kernel, {grid, threads, 0, st}, static_cast<const T*>(x), xp, static_cast<const T*>(dy), dyp,
                  static_cast<T*>(dx), dxp, B, H, W, Ho, Wo, C, bf);
}

template <typename T>
int spp_launch(const void* a, int ap, const void* dcat, int dp, void* da, int dap, int B, int H, int W, int C, int k, int bf, uint16_t* code,
               cudaStream_t st) {
    const int threads = 128, grid = grid_stride_ctas(static_cast<long long>(B) * H * W * (C / 8), threads, 16);
    if (int e = launch("spp_pool_bwd", spp_argmax_kernel<T>, {grid, threads, 0, st}, static_cast<const T*>(a), ap, code, B, H, W, C, k, bf)) return e;
    return launch("spp_pool_bwd", spp_gather_kernel<T>, {grid, threads, 0, st}, static_cast<const T*>(dcat), dp, code, static_cast<T*>(da), dap,
                  B, H, W, C, k, bf);
}

}  // namespace

extern "C" Y5_API int y5_maxpool2d(const void* x, int32_t x_pitch, void* y, int32_t y_pitch, int32_t batch, int32_t h, int32_t w, int32_t c,
                                   int32_t mode, int32_t dtype, void* stream) {
    if (batch <= 0 || h <= 0 || w <= 0 || c <= 0) return set_error(Y5_E_INVALID, "maxpool2d: bad arguments");
    if (c % 8 || !pool_dtype(dtype)) return set_error(Y5_E_UNSUPPORTED, "maxpool2d: c %% 8 and fp16/bf16/fp32 only");
    if (!vec_view(x, x_pitch, c) || !vec_view(y, y_pitch, c))
        return set_error(Y5_E_INVALID, "maxpool2d: views must be non-null, 16-byte aligned, with pitch >= c and a multiple of 8");
    int ho, wo;
    if (int e = pool_out(mode, h, w, &ho, &wo)) return e;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    if (dtype == Y5_F32) return fwd_launch<float>(mode, x, x_pitch, y, y_pitch, batch, h, w, ho, wo, c, 0, st);
    return fwd_launch<uint16_t>(mode, x, x_pitch, y, y_pitch, batch, h, w, ho, wo, c, dtype == Y5_BF16, st);
}

extern "C" Y5_API int y5_maxpool2d_bwd(const void* x, int32_t x_pitch, const void* dy, int32_t dy_pitch, void* dx, int32_t dx_pitch, int32_t batch,
                                       int32_t h, int32_t w, int32_t c, int32_t mode, int32_t dtype, void* stream) {
    if (batch <= 0 || h <= 0 || w <= 0 || c <= 0) return set_error(Y5_E_INVALID, "maxpool2d_bwd: bad arguments");
    if (c % 8 || !pool_dtype(dtype)) return set_error(Y5_E_UNSUPPORTED, "maxpool2d_bwd: c %% 8 and fp16/bf16/fp32 only");
    if (!vec_view(x, x_pitch, c) || !vec_view(dy, dy_pitch, c) || !vec_view(dx, dx_pitch, c))
        return set_error(Y5_E_INVALID, "maxpool2d_bwd: views must be non-null, 16-byte aligned, with pitch >= c and a multiple of 8");
    int ho, wo;
    if (int e = pool_out(mode, h, w, &ho, &wo)) return e;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    if (dtype == Y5_F32) return bwd_launch<float>(mode, x, x_pitch, dy, dy_pitch, dx, dx_pitch, batch, h, w, ho, wo, c, 0, st);
    return bwd_launch<uint16_t>(mode, x, x_pitch, dy, dy_pitch, dx, dx_pitch, batch, h, w, ho, wo, c, dtype == Y5_BF16, st);
}

extern "C" Y5_API int64_t y5_spp_bwd_workspace_bytes(int32_t batch, int32_t h, int32_t w, int32_t c) {
    return 3LL * batch * h * w * c * static_cast<int64_t>(sizeof(uint16_t));
}

extern "C" Y5_API int y5_spp_pool_bwd(const void* a, int32_t a_pitch, const void* dcat, int32_t dcat_pitch, void* da, int32_t da_pitch,
                                      int32_t batch, int32_t h, int32_t w, int32_t c, int32_t ksize, int32_t dtype, void* workspace,
                                      void* stream) {
    if (batch <= 0 || h <= 0 || w <= 0 || c <= 0 || !workspace) return set_error(Y5_E_INVALID, "spp_pool_bwd: bad arguments");
    if (c % 8 || !pool_dtype(dtype)) return set_error(Y5_E_UNSUPPORTED, "spp_pool_bwd: c %% 8 and fp16/bf16/fp32 only");
    if (ksize < 1 || !(ksize & 1) || 3 * (ksize / 2) > 127)
        return set_error(Y5_E_UNSUPPORTED, "spp_pool_bwd: ksize %d (odd, with 3 * (ksize / 2) <= 127)", ksize);
    if (!vec_view(a, a_pitch, c) || !vec_view(dcat, dcat_pitch, 4 * c) || !vec_view(da, da_pitch, c) || (reinterpret_cast<uintptr_t>(workspace) & 15))
        return set_error(Y5_E_INVALID, "spp_pool_bwd: views must be non-null, 16-byte aligned, with pitch >= their channels (4c for dcat) "
                                       "and a multiple of 8; workspace 16-byte aligned");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    uint16_t* code = static_cast<uint16_t*>(workspace);
    if (dtype == Y5_F32) return spp_launch<float>(a, a_pitch, dcat, dcat_pitch, da, da_pitch, batch, h, w, c, ksize, 0, code, st);
    return spp_launch<uint16_t>(a, a_pitch, dcat, dcat_pitch, da, da_pitch, batch, h, w, c, ksize, dtype == Y5_BF16, code, st);
}
