// Depthwise 5x5 / stride 1 / pad 2 convolution: the cheap half of GhostConv (reference models/common.py GhostConv.cv2 =
// Conv(c_, c_, 5, 1, None, c_)) over NHWC channel-slice views, fp16 / bf16, fp32 accumulation.
//
//   y5_dwconv_fwd    y = act(fp32(sum of the 25 taps) + bias) + res, rounded once -- conv_gemm's epilogue order.  With `flip`
//                    the taps are rotated 180 degrees: with no bias and no activation that is the data gradient of the same
//                    conv, and `res` then adds the gradient that reaches x by another path.  Optionally the same launch writes
//                    x_out = x + x_res at every output pixel (GhostBottleneck's first concat half, or a plain copy of x).
//   y5_dwconv_wgrad  dW[c][ky][kx] = sum over (n, y, x) of x[n, y+ky-2, x+kx-2, c] * dy[n, y, x, c] in fp32.
//
// A depthwise conv has no reduction over channels: each output is 25 MACs over one channel, so both kernels stream NHWC
// bytes and are bound by memory bandwidth (DESIGN.md, "Depthwise conv").  A thread owns one channel PAIR (a 32-bit word of two fp16 /
// bf16 values); pairs are the fastest index, so a warp touches contiguous bytes of a pixel.
//   forward: a block of 256 threads covers 8 pairs x 32 columns (4 x 64 when the channel count is not a multiple of 16) x kRows
//            rows.  It stages the (kRows + 4) x (columns + 4) halo tile of its channels in shared memory with 16-byte loads,
//            zero-filling cells outside the map (the padding), then each thread computes the kRows outputs of one (pair,
//            column): it reads the kRows + 4 rows of its 5-column window once and scatters each word into the accumulators of
//            the (up to) five output rows that use it.  The pair's 50 fp32 weights and 2 x kRows accumulators stay in registers;
//            kRows = 6 with three blocks per SM measured fastest among the configurations that do not spill.
//   wgrad:   the thread walks a strip of rows of its column with a 5x5 register window of the input (five new words per
//            row) and accumulates the pair's 50 tap sums in registers.  Lanes of a warp that hold the same pair (channel
//            counts below 64) add theirs by shuffles, the block sums the rest in shared memory, and adds its totals to dW
//            with one global fp32 atomic per (channel, tap).  The atomics make the summation
//            order depend on scheduling, as y5_conv_wgrad's split-K does (DESIGN.md section 3b): the result is not
//            bit-reproducible run to run, and is exact whenever every partial sum is (integer data).
#include <cmath>

#include "../../include/y5b200.h"
#include "common.cuh"
#include "host_util.h"

// kernels in a named namespace, so their symbols (what a profiler trace shows) do not depend on the build path
namespace y5 {

constexpr int kTaps = 25;
constexpr int kRows = 6;          // output rows per forward thread
constexpr int kFwdThreads = 256;
constexpr int kWgThreads = 128;   // wgrad: the block's shared partials are kWgThreads pairs x 50 floats (25.6 KB)

__device__ __forceinline__ float act_f(float v, int act, float slope, bool bf16) {
    if (act == Y5_ACT_SILU) {
        const float kTail = bf16 ? 8.0f : 4.0f;  // silu_from_half is faithful down to -kTail (common.cuh); conv_gemm's rule
        const float h = 0.5f * v;                // exactly fp32(acc + bias) / 2
        return h < -0.5f * kTail ? silu_tail(v) : silu_from_half(h);
    }
    if (act == Y5_ACT_LEAKY) return v > 0.0f ? v : slope * v;
    return v;
}

// x, y, res, x_res, x_out: views as 32-bit words (channel pairs), pitches in words.  y may alias res and x_out may alias x_res
// (in-place adds: each element is read and written by one thread); x must alias neither output.
// CP channel pairs x TW = kFwdThreads / CP columns x kRows rows of outputs per block; the block stages its (kRows + 4) x (TW + 4)
// x CP halo tile in shared memory with 16-byte loads (zeros outside the map: the padding), then each thread computes the kRows
// outputs of one (pair, column).
template <bool FLIP, int CP>
__global__ void __launch_bounds__(kFwdThreads, 3) dwconv5_fwd_kernel(const uint32_t* __restrict__ x, int xp, const uint16_t* __restrict__ w,
                                                                  const float* __restrict__ bias, const uint32_t* res, int rp, uint32_t* y, int yp,
                                                                  const uint32_t* x_res, int xrp, uint32_t* x_out, int xop, int H, int W, int cp,
                                                                  int strips, int act, float slope, int bf16) {
    constexpr int TW = kFwdThreads / CP, HW = TW + 4, VPP = CP / 4;  // tile width, halo width, 16-byte vectors per pixel
    __shared__ uint4 tile[(kRows + 4) * HW * VPP];
    const int chunks = cp / CP, chunk = blockIdx.x % chunks, col0 = (blockIdx.x / chunks) * TW;
    const int n = blockIdx.y / strips, y0 = (blockIdx.y % strips) * kRows;
    const long long img = static_cast<long long>(n) * H;
    for (int i = threadIdx.x; i < (kRows + 4) * HW * VPP; i += kFwdThreads) {
        const int v = i % VPP, px = i / VPP, iy = y0 - 2 + px / HW, ix = col0 - 2 + px % HW;
        tile[i] = (iy >= 0 && iy < H && ix >= 0 && ix < W)
                      ? __ldg(reinterpret_cast<const uint4*>(x + ((img + iy) * W + ix) * xp + chunk * CP) + v)
                      : make_uint4(0u, 0u, 0u, 0u);
    }
    const int lp = threadIdx.x % CP, lc = threadIdx.x / CP, pair = chunk * CP + lp, col = col0 + lc;
    const bool bf = bf16 != 0;
    float w0[kTaps], w1[kTaps];
#pragma unroll
    for (int t = 0; t < kTaps; ++t) {
        const int src = FLIP ? kTaps - 1 - t : t;
        w0[t] = unpack1(w[(2 * pair) * kTaps + src], bf);
        w1[t] = unpack1(w[(2 * pair + 1) * kTaps + src], bf);
    }
    __syncthreads();
    if (col >= W) return;
    const uint32_t* sw = reinterpret_cast<const uint32_t*>(tile);
    float a0[kRows], a1[kRows];
#pragma unroll
    for (int o = 0; o < kRows; ++o) a0[o] = a1[o] = 0.0f;
#pragma unroll
    for (int r = 0; r < kRows + 4; ++r) {
#pragma unroll
        for (int dx = 0; dx < 5; ++dx) {
            const float2 f = unpack2(sw[(r * HW + lc + dx) * CP + lp], bf);
#pragma unroll
            for (int ky = 0; ky < 5; ++ky) {
                const int o = r - ky;  // output row o reads input row o + ky: taps in row-major order
                if (o >= 0 && o < kRows) {
                    a0[o] = fmaf(f.x, w0[ky * 5 + dx], a0[o]);
                    a1[o] = fmaf(f.y, w1[ky * 5 + dx], a1[o]);
                }
            }
        }
    }
    const float b0 = bias ? bias[2 * pair] : 0.0f, b1 = bias ? bias[2 * pair + 1] : 0.0f;
#pragma unroll
    for (int o = 0; o < kRows; ++o) {
        const int yy = y0 + o;
        if (yy >= H) break;
        const long long pix = (img + yy) * W + col;
        float v0 = act_f(a0[o] + b0, act, slope, bf), v1 = act_f(a1[o] + b1, act, slope, bf);
        if (res) {
            const float2 t = unpack2(res[pix * rp + pair], bf);
            v0 += t.x;
            v1 += t.y;
        }
        y[pix * yp + pair] = pack2(v0, v1, bf);
        if (x_out) {
            const uint32_t xv = sw[((o + 2) * HW + lc + 2) * CP + lp];
            if (x_res) {
                const float2 s = unpack2(xv, bf), t = unpack2(x_res[pix * xrp + pair], bf);
                x_out[pix * xop + pair] = pack2(s.x + t.x, s.y + t.y, bf);
            } else {
                x_out[pix * xop + pair] = xv;
            }
        }
    }
}

__global__ void __launch_bounds__(kWgThreads) dwconv5_wgrad_kernel(const uint32_t* __restrict__ x, int xp, const uint32_t* __restrict__ dy, int dyp,
                                                                   float* __restrict__ dw, int H, int W, int cp, int rows_per, int strips, int bf16) {
    __shared__ float part[kWgThreads * 2 * kTaps];
    const int pairs_in_block = cp < kWgThreads ? cp : kWgThreads;
    for (int i = threadIdx.x; i < pairs_in_block * 2 * kTaps; i += kWgThreads) part[i] = 0.0f;
    __syncthreads();
    const long long g0 = static_cast<long long>(blockIdx.x) * kWgThreads, g = g0 + threadIdx.x;
    const int pair = static_cast<int>(g % cp), col = static_cast<int>(g / cp);
    const int pair0 = static_cast<int>(g0 % cp);
    const int n = blockIdx.y / strips, ys = (blockIdx.y % strips) * rows_per;
    const int ye = min(ys + rows_per, H);
    const bool bf = bf16 != 0;
    float a0[kTaps], a1[kTaps];
#pragma unroll
    for (int t = 0; t < kTaps; ++t) a0[t] = a1[t] = 0.0f;
    if (col < W) {
        const long long img = static_cast<long long>(n) * H;
        auto load_row = [&](int iy, float2 (&row)[5]) {
#pragma unroll
            for (int dx = 0; dx < 5; ++dx) {
                const int ix = col - 2 + dx;
                const uint32_t v = (iy >= 0 && iy < H && ix >= 0 && ix < W) ? __ldg(x + ((img + iy) * W + ix) * xp + pair) : 0u;
                row[dx] = unpack2(v, bf);
            }
        };
        float2 win[5][5];  // win[ky] = input row yy + ky - 2 of the current output row yy
#pragma unroll
        for (int k = 1; k < 5; ++k) load_row(ys - 3 + k, win[k]);
        for (int yy = ys; yy < ye; ++yy) {
#pragma unroll
            for (int k = 0; k < 4; ++k)
#pragma unroll
                for (int dx = 0; dx < 5; ++dx) win[k][dx] = win[k + 1][dx];
            load_row(yy + 2, win[4]);
            const float2 d = unpack2(__ldg(dy + ((img + yy) * W + col) * dyp + pair), bf);
#pragma unroll
            for (int ky = 0; ky < 5; ++ky)
#pragma unroll
                for (int dx = 0; dx < 5; ++dx) {
                    a0[ky * 5 + dx] = fmaf(win[ky][dx].x, d.x, a0[ky * 5 + dx]);
                    a1[ky * 5 + dx] = fmaf(win[ky][dx].y, d.y, a1[ky * 5 + dx]);
                }
        }
    }
    // lanes l, l + cp, l + 2cp, ... of a warp hold the same pair: lanes 0 .. cp-1 take their sums first, so fewer threads meet
    // at the same shared-memory words (a column of zeros for lanes past the map)
    const int lane = threadIdx.x & 31;
    if (cp < 32) {
#pragma unroll
        for (int t = 0; t < kTaps; ++t) {
            float s0 = a0[t], s1 = a1[t];
            for (int d = cp; d < 32; d += cp) {
                const float v0 = __shfl_down_sync(0xffffffffu, a0[t], d), v1 = __shfl_down_sync(0xffffffffu, a1[t], d);
                if (lane + d < 32) {  // past the warp's last lane the shuffle returns the caller's own value
                    s0 += v0;
                    s1 += v1;
                }
            }
            a0[t] = s0;
            a1[t] = s1;
        }
    }
    if (col < W && (cp >= 32 || lane < cp)) {
        const int lp = cp < kWgThreads ? pair : (pair - pair0 + cp) % cp;  // < pairs_in_block
#pragma unroll
        for (int t = 0; t < kTaps; ++t) {
            atomicAdd(&part[lp * 2 * kTaps + t], a0[t]);
            atomicAdd(&part[lp * 2 * kTaps + kTaps + t], a1[t]);
        }
    }
    __syncthreads();
    for (int i = threadIdx.x; i < pairs_in_block * 2 * kTaps; i += kWgThreads) {
        const int lp = i / (2 * kTaps), j = i % (2 * kTaps);
        const int p = cp < kWgThreads ? lp : (pair0 + lp) % cp;
        atomicAdd(&dw[(2 * p + j / kTaps) * kTaps + j % kTaps], part[i]);  // dW laid out [c][5][5], like the (c, 1, 5, 5) parameter
    }
}

}  // namespace y5

namespace {

using namespace y5;

int launched(const char* what) {
    count_launch();
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return set_error(int(e), "%s launch failed: %s", what, cudaGetErrorString(e));
    return 0;
}

// a view the kernels read in 32-bit words and that the 16-byte rule of the ABI allows: aligned base, pitch >= c, pitch % 8 == 0
bool dw_view(const void* p, int pitch, int c) { return p && !(reinterpret_cast<uintptr_t>(p) & 15) && pitch >= c && pitch % 8 == 0; }

int check_common(const char* what, int batch, int h, int w, int c, int ksize, int stride, int dtype) {
    if (ksize != 5 || stride != 1)
        return set_error(Y5_E_INVALID, "%s: kernel size %d, stride %d (built: the 5x5 stride-1 depthwise conv of GhostConv)", what, ksize, stride);
    if (batch <= 0 || h <= 0 || w <= 0 || c <= 0 || c % 8)
        return set_error(Y5_E_INVALID, "%s: batch %d, %dx%d, %d channels (channels a positive multiple of 8)", what, batch, h, w, c);
    if (dtype != Y5_F16 && dtype != Y5_BF16) return set_error(Y5_E_UNSUPPORTED, "%s: dtype must be fp16 or bf16", what);
    return 0;
}

}  // namespace

extern "C" Y5_API int y5_dwconv_fwd(const void* x, int32_t x_pitch, const void* weight, const float* bias, void* y, int32_t y_pitch,
                                    const void* residual, int32_t res_pitch, const void* x_res, int32_t x_res_pitch, void* x_out,
                                    int32_t x_out_pitch, int32_t batch, int32_t h, int32_t w, int32_t c, int32_t ksize, int32_t stride,
                                    int32_t act, float act_slope, int32_t flip, int32_t dtype, void* stream) {
    if (int e = check_common("dwconv_fwd", batch, h, w, c, ksize, stride, dtype)) return e;
    if (act != Y5_ACT_NONE && act != Y5_ACT_SILU && act != Y5_ACT_LEAKY) return set_error(Y5_E_INVALID, "dwconv_fwd: activation code %d", act);
    if (act == Y5_ACT_LEAKY && !std::isfinite(act_slope)) return set_error(Y5_E_INVALID, "dwconv_fwd: LeakyReLU slope must be finite");
    if (!weight || (reinterpret_cast<uintptr_t>(weight) & 3) || (reinterpret_cast<uintptr_t>(bias) & 3))
        return set_error(Y5_E_INVALID, "dwconv_fwd: weight must be non-null and 4-byte aligned, bias 4-byte aligned");
    if (!dw_view(x, x_pitch, c) || !dw_view(y, y_pitch, c) || (residual && !dw_view(residual, res_pitch, c)) ||
        (x_out && !dw_view(x_out, x_out_pitch, c)) || (x_res && (!x_out || !dw_view(x_res, x_res_pitch, c))))
        return set_error(Y5_E_INVALID, "dwconv_fwd: views must be non-null, 16-byte aligned, with pitch >= c (%d) and a multiple of 8; "
                                       "x_res needs x_out", c);
    if (x == y || x == x_out) return set_error(Y5_E_INVALID, "dwconv_fwd: x is read by neighbouring outputs and cannot be written in place");
    const int cp = c / 2, strips = (h + kRows - 1) / kRows;
    if (static_cast<long long>(batch) * strips > 65535) return set_error(Y5_E_UNSUPPORTED, "dwconv_fwd: batch x ceil(h / %d) > 65535", kRows);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    auto* xw = static_cast<const uint32_t*>(x);
    auto* wp = static_cast<const uint16_t*>(weight);
    auto* rw = static_cast<const uint32_t*>(residual);
    auto* yw = static_cast<uint32_t*>(y);
    auto* xrw = static_cast<const uint32_t*>(x_res);
    auto* xow = static_cast<uint32_t*>(x_out);
    // 8 pairs (16 channels) x 32 columns per block where the channels allow, else 4 pairs x 64 columns (c = 8, 24, 40, ...)
    auto launch = [&](auto kern, int pairs_per_block) {
        const int tw = kFwdThreads / pairs_per_block;
        const dim3 grid(static_cast<unsigned>((cp / pairs_per_block) * ((w + tw - 1) / tw)), static_cast<unsigned>(batch * strips));
        kern<<<grid, kFwdThreads, 0, st>>>(xw, x_pitch / 2, wp, bias, rw, res_pitch / 2, yw, y_pitch / 2, xrw, x_res_pitch / 2, xow, x_out_pitch / 2,
                                           h, w, cp, strips, act, act_slope, dtype == Y5_BF16);
    };
    if (cp % 8 == 0)
        flip ? launch(dwconv5_fwd_kernel<true, 8>, 8) : launch(dwconv5_fwd_kernel<false, 8>, 8);
    else
        flip ? launch(dwconv5_fwd_kernel<true, 4>, 4) : launch(dwconv5_fwd_kernel<false, 4>, 4);
    return launched("dwconv_fwd");
}

extern "C" Y5_API int y5_dwconv_wgrad(const void* x, int32_t x_pitch, const void* dy, int32_t dy_pitch, float* dweight, int32_t batch, int32_t h,
                                      int32_t w, int32_t c, int32_t ksize, int32_t stride, int32_t dtype, void* stream) {
    if (int e = check_common("dwconv_wgrad", batch, h, w, c, ksize, stride, dtype)) return e;
    if (!dw_view(x, x_pitch, c) || !dw_view(dy, dy_pitch, c))
        return set_error(Y5_E_INVALID, "dwconv_wgrad: views must be non-null, 16-byte aligned, with pitch >= c (%d) and a multiple of 8", c);
    if (!dweight || (reinterpret_cast<uintptr_t>(dweight) & 3)) return set_error(Y5_E_INVALID, "dwconv_wgrad: dweight must be non-null and 4-byte aligned");
    const int cp = c / 2;
    const long long gx = (static_cast<long long>(w) * cp + kWgThreads - 1) / kWgThreads;
    // rows per thread: enough blocks for ~8 per SM, each thread walking as many rows as that allows (fewer partials to add up)
    const long long want = static_cast<long long>(sm_count()) * 8;
    long long strips = (want + gx * batch - 1) / (gx * batch);
    strips = strips < 1 ? 1 : (strips > h ? h : strips);
    const int rows_per = static_cast<int>((h + strips - 1) / strips);
    strips = (h + rows_per - 1) / rows_per;
    if (batch * strips > 65535) return set_error(Y5_E_UNSUPPORTED, "dwconv_wgrad: batch %d too large", batch);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    cudaMemsetAsync(dweight, 0, static_cast<size_t>(c) * kTaps * sizeof(float), st);
    count_launch();
    dwconv5_wgrad_kernel<<<dim3(static_cast<unsigned>(gx), static_cast<unsigned>(batch * strips)), kWgThreads, 0, st>>>(
        static_cast<const uint32_t*>(x), x_pitch / 2, static_cast<const uint32_t*>(dy), dy_pitch / 2, dweight, h, w, cp, rows_per,
        static_cast<int>(strips), dtype == Y5_BF16);
    return launched("dwconv_wgrad");
}
