// Training augmentation of the detection dataloader (reference utils/dataloaders.py:696-855, utils/augmentations.py:69-233)
// on the device, byte-exact with the reference's OpenCV / numpy arithmetic (oracle/aug_ref.py):
//   aug_gather_kernel : one thread per output pixel (per 2x2 cell for the stem's space-to-depth output).  Undo the flips,
//                       run cv2.warpAffine's fixed-point coordinate arithmetic against the VIRTUAL mosaic canvas (each
//                       bilinear tap reads whichever placed tile covers it, or 114 -- the 2s x 2s canvas is never
//                       built), blend a second mosaic for mixup, apply BGR->HSV, the LUTs and HSV->BGR, write CHW.
//   aug_labels_kernel : the label path (xywhn2xyxy, clip, the corners through M, box_candidates, xyxy2xywhn, flips) and
//                       a stable compaction of the kept rows, in one block.
// Compiled with -fmad=false; every rounding point the reference has is an explicit _rn intrinsic, and the two fused
// multiply-adds the references contain (OpenCV's AVX2 HSV->BGR, OpenBLAS's `xy @ M.T`) are explicit fma.
#include <math.h>

#include "../../include/y5b200.h"
#include "common.cuh"
#include "host_util.h"

namespace y5 {

constexpr int kAugBorder = 114;
constexpr int kLabelThreads = 1024;

// canvas pixel (x, y) of mosaic m, channel-strided BGR; 114 outside the canvas and outside every tile
__device__ __forceinline__ void canvas_tap(const y5_aug_image& im, int m, int x, int y, int v[3]) {
    v[0] = v[1] = v[2] = kAugBorder;
    if (x < 0 || y < 0 || x >= im.canvas_w || y >= im.canvas_h) return;
    const int t0 = m * 4, t1 = m * 4 + im.n_tiles[m];
    for (int t = t0; t < t1; ++t) {
        const y5_aug_tile& T = im.tiles[t];
        if (x >= T.x1a && x < T.x2a && y >= T.y1a && y < T.y2a) {
            const uint8_t* p = static_cast<const uint8_t*>(T.src) + static_cast<long long>(y + T.dy) * T.row_bytes +
                               static_cast<long long>(x + T.dx) * T.pixel_stride;
            v[0] = p[0];
            v[1] = p[T.channel_stride];
            v[2] = p[2 * T.channel_stride];
            return;
        }
    }
}

// cv2.warpAffine(canvas, M, dsize, INTER_LINEAR, BORDER_CONSTANT 114) at output pixel (x, y): imgwarp.cpp's fixed point
// (AB_BITS 10, INTER_BITS 5) and remap's bilinear weights scaled by 2^15
__device__ __forceinline__ void warp_sample(const y5_aug_image& im, int m, int x, int y, int v[3]) {
    if (!im.warp[m]) {
        canvas_tap(im, m, x, y, v);
        return;
    }
    const double* iM = im.inv_m[m];
    const int adelta = __double2int_rn(__dmul_rn(__dmul_rn(iM[0], static_cast<double>(x)), 1024.0));
    const int bdelta = __double2int_rn(__dmul_rn(__dmul_rn(iM[3], static_cast<double>(x)), 1024.0));
    const int X0 = __double2int_rn(__dmul_rn(__dadd_rn(__dmul_rn(iM[1], static_cast<double>(y)), iM[2]), 1024.0)) + 16;
    const int Y0 = __double2int_rn(__dmul_rn(__dadd_rn(__dmul_rn(iM[4], static_cast<double>(y)), iM[5]), 1024.0)) + 16;
    const int X = (X0 + adelta) >> 5, Y = (Y0 + bdelta) >> 5;
    const int sx = min(max(X >> 5, -32768), 32767), sy = min(max(Y >> 5, -32768), 32767);
    const int fx = X & 31, fy = Y & 31;
    const int w00 = (32 - fy) * (32 - fx) * 32, w01 = (32 - fy) * fx * 32, w10 = fy * (32 - fx) * 32, w11 = fy * fx * 32;
    int a[3], b[3], c[3], d[3];
    canvas_tap(im, m, sx, sy, a);
    canvas_tap(im, m, sx + 1, sy, b);
    canvas_tap(im, m, sx, sy + 1, c);
    canvas_tap(im, m, sx + 1, sy + 1, d);
#pragma unroll
    for (int k = 0; k < 3; ++k) v[k] = min(max((a[k] * w00 + b[k] * w01 + c[k] * w10 + d[k] * w11 + (1 << 14)) >> 15, 0), 255);
}

// COLOR_BGR2HSV on uint8: OpenCV's integer path (hsv_shift 12, sdiv / hdiv tables rounded from double)
__device__ __forceinline__ void bgr_to_hsv(const int bgr[3], int hsv[3]) {
    const int b = bgr[0], g = bgr[1], r = bgr[2];
    const int v = max(max(b, g), r);
    const int diff = v - min(min(b, g), r);
    const int sdiv = v ? __double2int_rn(__ddiv_rn(static_cast<double>(255 << 12), static_cast<double>(v))) : 0;
    const int hdiv = diff ? __double2int_rn(__ddiv_rn(static_cast<double>(180 << 12), __dmul_rn(6.0, static_cast<double>(diff)))) : 0;
    const bool vr = v == r, vg = !vr && v == g;
    int h = vr ? g - b : (vg ? b - r + 2 * diff : r - g + 4 * diff);
    h = (h * hdiv + (1 << 11)) >> 12;
    if (h < 0) h += 180;
    hsv[0] = h;
    hsv[1] = (diff * sdiv + (1 << 11)) >> 12;
    hsv[2] = v;
}

// COLOR_HSV2BGR on uint8 as OpenCV's AVX2 build computes it: float32, 1 - s*h and 1 - s*(1 - h) fused, times 255, then
// truncated inside the row's 32-pixel SIMD blocks and rounded in the scalar tail
__device__ __forceinline__ void hsv_to_bgr(const int hsv[3], bool truncate, int bgr[3]) {
    const float h = __fmul_rn(static_cast<float>(hsv[0]), static_cast<float>(6.0 / 180.0));
    const float s = __fmul_rn(static_cast<float>(hsv[1]), static_cast<float>(1.0 / 255.0));
    const float v = __fmul_rn(static_cast<float>(hsv[2]), static_cast<float>(1.0 / 255.0));
    const int sec = static_cast<int>(floorf(h));
    const float fr = __fsub_rn(h, static_cast<float>(sec));
    const float t1 = __fmul_rn(v, __fsub_rn(1.0f, s));
    const float t2 = __fmul_rn(v, __fmaf_rn(-s, fr, 1.0f));
    const float t3 = __fmul_rn(v, __fmaf_rn(-s, __fsub_rn(1.0f, fr), 1.0f));
    // OpenCV's sector table {1,3,0},{1,0,2},{3,0,1},{0,2,1},{0,1,3},{2,1,0}: 2 bits per channel, 6 bits per sector
    const unsigned code = static_cast<unsigned>((0x1b461384dull >> (6 * (sec % 6))) & 63u);
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const unsigned i = (code >> (2 * k)) & 3u;
        const float o = __fmul_rn(i == 0 ? v : (i == 1 ? t1 : (i == 2 ? t2 : t3)), 255.0f);
        bgr[k] = min(max(truncate ? static_cast<int>(o) : __float2int_rn(o), 0), 255);
    }
}

// the finished BGR pixel at output (x, y) of image im
__device__ __forceinline__ void aug_pixel(const y5_aug_image& im, int x, int y, int out_h, int out_w, int simd_cols, int v[3]) {
    const int px = im.fliplr ? out_w - 1 - x : x;
    const int py = im.flipud ? out_h - 1 - y : y;
    warp_sample(im, 0, px, py, v);
    if (im.n_mosaic == 2) {
        int v2[3];
        warp_sample(im, 1, px, py, v2);
        const double r = im.mix_r, r1 = __dsub_rn(1.0, r);
#pragma unroll
        for (int k = 0; k < 3; ++k)
            v[k] = static_cast<int>(__dadd_rn(__dmul_rn(static_cast<double>(v[k]), r), __dmul_rn(static_cast<double>(v2[k]), r1)));
    }
    if (im.hsv) {
        int hsv[3];
        bgr_to_hsv(v, hsv);
#pragma unroll
        for (int k = 0; k < 3; ++k) hsv[k] = im.lut[k][hsv[k]];
        hsv_to_bgr(hsv, px < simd_cols, v);
    }
}

// OUT: 0 = uint8 NCHW, 1 = fp16/bf16 NCHW (/255), 2 = fp32 NCHW (/255), 3 = stem space-to-depth cells (16 channels)
template <int OUT>
__global__ void aug_gather_kernel(const y5_aug_image* __restrict__ table, int out_h, int out_w, int simd_cols, int swap_rb,
                                  void* __restrict__ out, int bf16, int row_px, int x_off) {
    const int b = blockIdx.z;
    const y5_aug_image& im = table[b];
    const int step = OUT == 3 ? 2 : 1;
    const int cx = (blockIdx.x * blockDim.x + threadIdx.x) * step;
    const int cy = (blockIdx.y * blockDim.y + threadIdx.y) * step;
    if (cx >= out_w || cy >= out_h) return;
    float cell[16];
#pragma unroll
    for (int q = 0; q < 16; ++q) cell[q] = 0.f;
#pragma unroll
    for (int dy = 0; dy < step; ++dy)
#pragma unroll
        for (int dx = 0; dx < step; ++dx) {
            const int ox = cx + dx, oy = cy + dy;
            int v[3];
            aug_pixel(im, ox, oy, out_h, out_w, simd_cols, v);
            if (swap_rb) { const int t = v[0]; v[0] = v[2]; v[2] = t; }
            if (OUT == 3) {
#pragma unroll
                for (int c = 0; c < 3; ++c) cell[(dy * 2 + dx) * 3 + c] = static_cast<float>(v[c]) / 255.0f;
            } else {
                const long long plane = static_cast<long long>(out_h) * out_w;
                const long long o = (static_cast<long long>(b) * 3) * plane + static_cast<long long>(oy) * out_w + ox;
#pragma unroll
                for (int c = 0; c < 3; ++c) {
                    if (OUT == 0) static_cast<uint8_t*>(out)[o + c * plane] = static_cast<uint8_t>(v[c]);
                    else if (OUT == 1) static_cast<uint16_t*>(out)[o + c * plane] = pack1(static_cast<float>(v[c]) / 255.0f, bf16 != 0);
                    else static_cast<float*>(out)[o + c * plane] = static_cast<float>(v[c]) / 255.0f;
                }
            }
        }
    if (OUT == 3) {
        uint4 lo, hi;
        const bool bf = bf16 != 0;
        lo.x = pack2(cell[0], cell[1], bf); lo.y = pack2(cell[2], cell[3], bf); lo.z = pack2(cell[4], cell[5], bf); lo.w = pack2(cell[6], cell[7], bf);
        hi.x = pack2(cell[8], cell[9], bf); hi.y = pack2(cell[10], cell[11], bf); hi.z = pack2(cell[12], cell[13], bf); hi.w = pack2(cell[14], cell[15], bf);
        const long long opx = (static_cast<long long>(b) * (out_h >> 1) + (cy >> 1)) * row_px + x_off + (cx >> 1);
        static_cast<uint4*>(out)[opx * 2] = lo;
        static_cast<uint4*>(out)[opx * 2 + 1] = hi;
    }
}

// x' = x*M0 + y*M1 + M2 as OpenBLAS's dgemm forms `xy @ M.T` (K = 3): product, fma, add
__device__ __forceinline__ double affine_row(const double* Mr, double x, double y) {
    return __dadd_rn(__fma_rn(y, Mr[1], __dmul_rn(x, Mr[0])), Mr[2]);
}

// one label row -> keep flag and the output row (utils/augmentations.py:163-197 with utils/dataloaders.py:734-756)
__device__ bool aug_label_row(const y5_aug_image* table, const y5_aug_label& L, int out_h, int out_w, float row[6]) {
    const y5_aug_image& im = table[L.image];
    const int m = L.mosaic;
    float x1 = L.x, y1 = L.y, x2 = L.w, y2 = L.h;
    if (!(L.flags & Y5_AUG_IN_XYXY)) {  // xywhn2xyxy, float32
        const float hw = __fdiv_rn(L.w, 2.0f), hh = __fdiv_rn(L.h, 2.0f);
        x1 = __fadd_rn(__fmul_rn(L.tile_w, __fsub_rn(L.x, hw)), L.pad_w);
        y1 = __fadd_rn(__fmul_rn(L.tile_h, __fsub_rn(L.y, hh)), L.pad_h);
        x2 = __fadd_rn(__fmul_rn(L.tile_w, __fadd_rn(L.x, hw)), L.pad_w);
        y2 = __fadd_rn(__fmul_rn(L.tile_h, __fadd_rn(L.y, hh)), L.pad_h);
    }
    if (L.flags & Y5_AUG_CLIP) {
        x1 = fminf(fmaxf(x1, 0.f), im.clip_max); y1 = fminf(fmaxf(y1, 0.f), im.clip_max);
        x2 = fminf(fmaxf(x2, 0.f), im.clip_max); y2 = fminf(fmaxf(y2, 0.f), im.clip_max);
    }
    // the corners x1y1, x2y2, x1y2, x2y1 through M, in double
    const double* M0 = im.m[m];
    const double* M1 = im.m[m] + 3;
    const double cxs[4] = {x1, x2, x1, x2}, cys[4] = {y1, y2, y2, y1};
    double nx1 = INFINITY, ny1 = INFINITY, nx2 = -INFINITY, ny2 = -INFINITY;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const double px = affine_row(M0, cxs[k], cys[k]), py = affine_row(M1, cxs[k], cys[k]);
        nx1 = fmin(nx1, px); nx2 = fmax(nx2, px); ny1 = fmin(ny1, py); ny2 = fmax(ny2, py);
    }
    const double W = static_cast<double>(out_w), H = static_cast<double>(out_h);
    nx1 = fmin(fmax(nx1, 0.0), W); nx2 = fmin(fmax(nx2, 0.0), W);
    ny1 = fmin(fmax(ny1, 0.0), H); ny2 = fmin(fmax(ny2, 0.0), H);
    // box_candidates(targets[:, 1:5].T * s, new.T): box1 in float32, box2 in float64
    const float s = im.scale[m];
    const float w1 = __fsub_rn(__fmul_rn(x2, s), __fmul_rn(x1, s)), h1 = __fsub_rn(__fmul_rn(y2, s), __fmul_rn(y1, s));
    const double w2 = __dsub_rn(nx2, nx1), h2 = __dsub_rn(ny2, ny1);
    const double ar = fmax(__ddiv_rn(w2, __dadd_rn(h2, 1e-16)), __ddiv_rn(h2, __dadd_rn(w2, 1e-16)));
    const float area1 = __fadd_rn(__fmul_rn(w1, h1), static_cast<float>(1e-16));
    const bool keep = w2 > 2.0 && h2 > 2.0 && __ddiv_rn(__dmul_rn(w2, h2), static_cast<double>(area1)) > 0.1 && ar < 100.0;
    // targets[:, 1:5] = new[i]: float64 -> float32
    float b0 = __double2float_rn(nx1), b1 = __double2float_rn(ny1), b2 = __double2float_rn(nx2), b3 = __double2float_rn(ny2);
    row[0] = static_cast<float>(L.image);
    row[1] = L.cls;
    if (L.flags & Y5_AUG_OUT_XYXY) {
        row[2] = b0; row[3] = b1; row[4] = b2; row[5] = b3;
        return keep;
    }
    // xyxy2xywhn(w, h, clip=True, eps=1e-3), float32, then the flips
    const float cw = __double2float_rn(__dsub_rn(W, 1e-3)), ch = __double2float_rn(__dsub_rn(H, 1e-3));
    b0 = fminf(fmaxf(b0, 0.f), cw); b2 = fminf(fmaxf(b2, 0.f), cw);
    b1 = fminf(fmaxf(b1, 0.f), ch); b3 = fminf(fmaxf(b3, 0.f), ch);
    const float Wf = static_cast<float>(out_w), Hf = static_cast<float>(out_h);
    float xc = __fdiv_rn(__fdiv_rn(__fadd_rn(b0, b2), 2.0f), Wf);
    float yc = __fdiv_rn(__fdiv_rn(__fadd_rn(b1, b3), 2.0f), Hf);
    if (im.flipud) yc = __fsub_rn(1.0f, yc);
    if (im.fliplr) xc = __fsub_rn(1.0f, xc);
    row[2] = xc;
    row[3] = yc;
    row[4] = __fdiv_rn(__fsub_rn(b2, b0), Wf);
    row[5] = __fdiv_rn(__fsub_rn(b3, b1), Hf);
    return keep;
}

// one block: chunks of kLabelThreads rows, kept rows written in input order (ballot + warp-total scan per chunk)
__global__ void __launch_bounds__(kLabelThreads) aug_labels_kernel(const y5_aug_image* __restrict__ table, const y5_aug_label* __restrict__ labels,
                                                                   int n_labels, int n_images, int out_h, int out_w,
                                                                   float* __restrict__ targets, int* __restrict__ count) {
    __shared__ int s_warp[kLabelThreads / 32];
    __shared__ int s_base;
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    if (tid == 0) s_base = 0;
    __syncthreads();
    for (int c0 = 0; c0 < n_labels; c0 += kLabelThreads) {
        const int i = c0 + tid;
        float row[6];
        // a row naming no image of the table, or no mosaic of it, is dropped
        const bool valid = i < n_labels && labels[i].image >= 0 && labels[i].image < n_images && labels[i].mosaic >= 0 &&
                           labels[i].mosaic < table[labels[i].image].n_mosaic;
        const bool keep = valid && aug_label_row(table, labels[i], out_h, out_w, row);
        const unsigned mask = __ballot_sync(0xffffffffu, keep);
        if (lane == 0) s_warp[wid] = __popc(mask);
        __syncthreads();
        int before = s_base;
        for (int w = 0; w < wid; ++w) before += s_warp[w];
        before += __popc(mask & ((1u << lane) - 1u));
        if (keep) {
#pragma unroll
            for (int k = 0; k < 6; ++k) targets[static_cast<long long>(before) * 6 + k] = row[k];
        }
        __syncthreads();
        if (tid == 0) {
            int total = 0;
            for (int w = 0; w < kLabelThreads / 32; ++w) total += s_warp[w];
            s_base += total;
        }
        __syncthreads();
    }
    if (tid == 0) *count = s_base;
}

}  // namespace y5

using namespace y5;

extern "C" Y5_API int y5_aug_gather(const y5_aug_image* table, int32_t n_images, int32_t out_h, int32_t out_w, int32_t hsv_simd_cols,
                                    int32_t swap_rb, void* out, int32_t out_dtype, int32_t s2d, int32_t out_row_px, int32_t out_x_off,
                                    void* stream) {
    if (!table || !out || n_images <= 0 || out_h <= 0 || out_w <= 0) return set_error(Y5_E_INVALID, "aug_gather: bad argument");
    if (hsv_simd_cols < 0 || hsv_simd_cols > out_w) return set_error(Y5_E_INVALID, "aug_gather: hsv_simd_cols outside [0, out_w]");
    if (n_images > 65535 || out_h > 32767 || out_w > 32767) return set_error(Y5_E_UNSUPPORTED, "aug_gather: batch or image too large");
    if (s2d && ((out_h | out_w) & 1)) return set_error(Y5_E_INVALID, "aug_gather: space-to-depth output needs even height/width");
    if (s2d && out_dtype != Y5_F16 && out_dtype != Y5_BF16) return set_error(Y5_E_UNSUPPORTED, "aug_gather: s2d output is fp16/bf16");
    if (!s2d && out_dtype != Y5_U8 && out_dtype != Y5_F16 && out_dtype != Y5_BF16 && out_dtype != Y5_F32)
        return set_error(Y5_E_UNSUPPORTED, "aug_gather: output dtype");
    if (s2d && (out_x_off < 0 || (out_row_px && out_x_off + out_w / 2 > out_row_px)))
        return set_error(Y5_E_INVALID, "aug_gather: output row pitch/offset do not cover the row");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const int step = s2d ? 2 : 1;
    const dim3 block(32, 8);
    const dim3 grid((out_w / step + block.x - 1) / block.x, (out_h / step + block.y - 1) / block.y, n_images);
    const int bf = out_dtype == Y5_BF16;
    if (s2d) {
        const int row_px = out_row_px ? out_row_px : out_w / 2;
        return launch("aug_gather", aug_gather_kernel<3>, {grid, block, 0, st}, table, out_h, out_w, hsv_simd_cols, swap_rb, out, bf, row_px,
                      out_x_off);
    }
    auto* kernel = out_dtype == Y5_U8 ? aug_gather_kernel<0> : out_dtype == Y5_F32 ? aug_gather_kernel<2> : aug_gather_kernel<1>;
    return launch("aug_gather", kernel, {grid, block, 0, st}, table, out_h, out_w, hsv_simd_cols, swap_rb, out, bf, 0, 0);
}

extern "C" Y5_API int y5_aug_labels(const y5_aug_image* table, int32_t n_images, const y5_aug_label* labels, int32_t n_labels, int32_t out_h,
                                    int32_t out_w, float* targets, int32_t* count, void* stream) {
    if (!table || !count || n_images <= 0 || n_labels < 0 || out_h <= 0 || out_w <= 0 || (n_labels > 0 && (!labels || !targets)))
        return set_error(Y5_E_INVALID, "aug_labels: bad argument");
    return launch("aug_labels", aug_labels_kernel, {1, kLabelThreads, 0, static_cast<cudaStream_t>(stream)}, table, labels, n_labels, n_images,
                  out_h, out_w, targets, count);
}
