// The callers either side of the hot path (SURVEY.md section 8f), batched on the device with no host synchronisation:
//   pre : letterbox (cv2.resize INTER_LINEAR fixed-point bilinear + 114 border) + BGR->RGB + HWC->CHW + /255, written
//         as a uint8 / fp16 / bf16 / fp32 NCHW batch or straight into the stem's space-to-depth buffer
//         (reference utils/augmentations.py:85-115, utils/dataloaders.py:354-357, detect.py:205-208)
//   post: process_mask / crop_mask (utils/segment/general.py:10-52), scale_boxes + clip_boxes (utils/general.py:613-626),
//         xywh2xyxy + process_batch's detection<->label matching for a whole batch (utils/metrics.py:224-265,
//         val.py:282-318), ConfusionMatrix.process_batch's counts for a whole batch (utils/metrics.py:139-183)
// Integer / index results (letterboxed bytes, match matrices) are bit-exact w.r.t. oracle/pre_ref.py / oracle/post_ref.py;
// this file is compiled with -fmad=false and uses explicit _rn intrinsics wherever a rounding point matters; fmaf() is
// used only where the reference itself is a BLAS dot product (mask logits).
#include <math.h>

#include "../../include/y5b200.h"
#include "common.cuh"
#include "host_util.h"
#include "match_rule.cuh"

namespace y5 {

// ---------------------------------------------------------------------------------------------------------------------
// letterbox
// ---------------------------------------------------------------------------------------------------------------------
constexpr int kLbMaxImages = 24;  // descriptors travel by value in the kernel parameter block

struct LbBatch {
    y5_letterbox_image im[kLbMaxImages];
};

// OpenCV resize.cpp coefficient rule: f = (float)((d + 0.5) * scale - 0.5) in double, split into floor + fraction;
// weights = cvRound(w * 2048) as int16.  Horizontal taps collapse onto the border pixel; vertical taps keep their weights
// and clamp the two row indices individually.
__device__ __forceinline__ void lb_coeff(int d, double scale, int src, bool horizontal, int& i0, int& i1, int& w0, int& w1) {
    const float f0 = static_cast<float>(__dsub_rn(__dmul_rn(__dadd_rn(static_cast<double>(d), 0.5), scale), 0.5));
    int s = static_cast<int>(floorf(f0));
    float f = __fsub_rn(f0, static_cast<float>(s));
    if (horizontal) {
        if (s < 0) { f = 0.f; s = 0; }
        if (s >= src - 1) { f = 0.f; s = src - 1; }
    }
    w1 = __float2int_rn(__fmul_rn(f, 2048.0f));
    w0 = __float2int_rn(__fmul_rn(__fsub_rn(1.0f, f), 2048.0f));
    i0 = min(max(s, 0), src - 1);
    i1 = min(max(s + 1, 0), src - 1);
}

// cv2.resize INTER_LINEAR (uint8, 3 channels) of a src_h x src_w image to dst_h x dst_w, at destination pixel (rx, ry)
__device__ __forceinline__ void linear_px(const uint8_t* src, int row_bytes, int src_h, int src_w, int dst_h, int dst_w, int rx, int ry,
                                          int (&v)[3]) {
    const double sx = 1.0 / (static_cast<double>(dst_w) / static_cast<double>(src_w));
    const double sy = 1.0 / (static_cast<double>(dst_h) / static_cast<double>(src_h));
    int x0, x1, a0, a1, y0, y1, b0, b1;
    lb_coeff(rx, sx, src_w, true, x0, x1, a0, a1);
    lb_coeff(ry, sy, src_h, false, y0, y1, b0, b1);
    const uint8_t* r0 = src + static_cast<long long>(y0) * row_bytes;
    const uint8_t* r1 = src + static_cast<long long>(y1) * row_bytes;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        const int s0 = r0[x0 * 3 + c] * a0 + r0[x1 * 3 + c] * a1;
        const int s1 = r1[x0 * 3 + c] * a0 + r1[x1 * 3 + c] * a1;
        const int o = (((b0 * (s0 >> 4)) >> 16) + ((b1 * (s1 >> 4)) >> 16) + 2) >> 2;
        v[c] = min(max(o, 0), 255);
    }
}

// OUT: 0 = uint8 NCHW, 1 = fp16/bf16 NCHW (/255), 2 = fp32 NCHW (/255), 3 = stem space-to-depth cells (16 channels)
template <int OUT>
__global__ void letterbox_kernel(const LbBatch L, int n_img, int out_h, int out_w, int swap_rb, int pad_value, void* __restrict__ out,
                                 int bf16, int row_px, int x_off) {
    const int b = blockIdx.z;
    if (b >= n_img) return;
    const y5_letterbox_image im = L.im[b];
    const uint8_t* src = static_cast<const uint8_t*>(im.data);
    // OUT 3 handles a 2x2 block of output pixels per thread (one s2d cell); the others one pixel per thread
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
            int v[3] = {pad_value, pad_value, pad_value};
            const int rx = ox - im.left, ry = oy - im.top;
            if (rx >= 0 && rx < im.new_w && ry >= 0 && ry < im.new_h) linear_px(src, im.row_bytes, im.src_h, im.src_w, im.new_h, im.new_w, rx, ry, v);
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

// ---------------------------------------------------------------------------------------------------------------------
// validation batch: load_image's resize + letterbox(scaleup=False)
// ---------------------------------------------------------------------------------------------------------------------
constexpr int kValMaxImages = 64;  // descriptors travel by value in the kernel parameter block (64 x 56 bytes)

// kVal*: to the canvas at (top, left), HWC BGR to `dst` (the scratch of a letterbox that resizes again), or not at all
enum : int { kValCanvas = 0, kValScratch = 1, kValSkip = 2 };

struct ValDesc {
    const uint8_t* src;
    uint8_t* dst;
    int src_h, src_w, row_bytes, res_h, res_w, interp, top, left, mode, reserved;
};

struct ValBatch {
    ValDesc im[kValMaxImages];
};

// OpenCV's computeResizeAreaTab for one destination index: the source cell [d s, d s + s) with s = 1 / (dst / src) as
// taps s1 - first .. s2 - 1 + last; whole pixels weigh 1 / w, a partial first / last one its covered fraction / w
struct AreaAxis {
    int s1, n;
    float w_first, w_mid, w_last;
    bool first, last;
};

__device__ __forceinline__ AreaAxis area_axis(int d, double scale, int src) {
    AreaAxis a;
    const double f1 = __dmul_rn(static_cast<double>(d), scale);
    const double f2 = __dadd_rn(f1, scale);
    const double cw = fmin(scale, __dsub_rn(static_cast<double>(src), f1));
    int s2 = min(static_cast<int>(floor(f2)), src - 1);
    const int s1 = min(static_cast<int>(ceil(f1)), s2);
    const double head = __dsub_rn(static_cast<double>(s1), f1), tail = __dsub_rn(f2, static_cast<double>(s2));
    a.first = head > 1e-3;
    a.last = tail > 1e-3;
    a.w_first = static_cast<float>(__ddiv_rn(head, cw));
    a.w_mid = static_cast<float>(__ddiv_rn(1.0, cw));
    a.w_last = static_cast<float>(__ddiv_rn(fmin(fmin(tail, 1.0), cw), cw));
    a.s1 = s1 - (a.first ? 1 : 0);
    a.n = (s2 - s1) + (a.first ? 1 : 0) + (a.last ? 1 : 0);
    return a;
}

__device__ __forceinline__ float area_weight(const AreaAxis& a, int t) {
    return a.first && t == 0 ? a.w_first : (a.last && t == a.n - 1 ? a.w_last : a.w_mid);
}

__device__ __forceinline__ int round_u8(float f) { return min(max(__float2int_rn(f), 0), 255); }

// cv2.resize INTER_AREA (uint8, 3 channels, shrinking in both axes) at destination pixel (rx, ry)
__device__ void area_px(const uint8_t* src, int row_bytes, int src_h, int src_w, int dst_h, int dst_w, int rx, int ry, int (&v)[3]) {
    const double sx = 1.0 / (static_cast<double>(dst_w) / static_cast<double>(src_w));
    const double sy = 1.0 / (static_cast<double>(dst_h) / static_cast<double>(src_h));
    const int kx = __double2int_rn(sx), ky = __double2int_rn(sy);
    if (fabs(sx - kx) < 2.220446049250313e-16 && fabs(sy - ky) < 2.220446049250313e-16) {
        // "area fast": integer cells summed exactly; 2 x 2 rounds as (sum + 2) >> 2, others as cvRound(sum * (1.f / area))
        const uint8_t* p = src + static_cast<long long>(ry) * ky * row_bytes + rx * kx * 3;
        int s[3] = {0, 0, 0};
        for (int y = 0; y < ky; ++y)
            for (int x = 0; x < kx; ++x)
#pragma unroll
                for (int c = 0; c < 3; ++c) s[c] += p[static_cast<long long>(y) * row_bytes + x * 3 + c];
        const float inv = __fdiv_rn(1.0f, static_cast<float>(kx * ky));
#pragma unroll
        for (int c = 0; c < 3; ++c) v[c] = kx == 2 && ky == 2 ? (s[c] + 2) >> 2 : round_u8(__fmul_rn(static_cast<float>(s[c]), inv));
        return;
    }
    // weighted cells: each source row summed across its x taps, then the rows across their y taps, in float32 in tap order
    const AreaAxis ax = area_axis(rx, sx, src_w), ay = area_axis(ry, sy, src_h);
    float sum[3] = {0.f, 0.f, 0.f};
    for (int ty = 0; ty < ay.n; ++ty) {
        const uint8_t* row = src + static_cast<long long>(ay.s1 + ty) * row_bytes;
        const float beta = area_weight(ay, ty);
        float buf[3] = {0.f, 0.f, 0.f};
        for (int tx = 0; tx < ax.n; ++tx) {
            const float alpha = area_weight(ax, tx);
            const uint8_t* q = row + (ax.s1 + tx) * 3;
#pragma unroll
            for (int c = 0; c < 3; ++c) buf[c] = __fadd_rn(buf[c], __fmul_rn(static_cast<float>(q[c]), alpha));
        }
#pragma unroll
        for (int c = 0; c < 3; ++c) sum[c] = __fadd_rn(sum[c], __fmul_rn(beta, buf[c]));
    }
#pragma unroll
    for (int c = 0; c < 3; ++c) v[c] = round_u8(sum[c]);
}

// OUT: 0 = uint8, 1 = fp16/bf16, 2 = fp32 (float32(v) * float32(1/255), rounded once); CHW RGB
template <int OUT>
__global__ void val_letterbox_kernel(const ValBatch L, int out_h, int out_w, void* __restrict__ out, int bf16) {
    const int b = blockIdx.z;
    const ValDesc& im = L.im[b];
    const int ox = blockIdx.x * blockDim.x + threadIdx.x, oy = blockIdx.y * blockDim.y + threadIdx.y;
    if (im.mode == kValSkip) return;
    const bool to_scratch = im.mode == kValScratch;
    const int rx = to_scratch ? ox : ox - im.left, ry = to_scratch ? oy : oy - im.top;
    if (to_scratch ? (rx >= im.res_w || ry >= im.res_h) : (ox >= out_w || oy >= out_h)) return;
    int v[3] = {114, 114, 114};
    if (rx >= 0 && rx < im.res_w && ry >= 0 && ry < im.res_h) {
        if (im.interp == Y5_VAL_AREA) {
            area_px(im.src, im.row_bytes, im.src_h, im.src_w, im.res_h, im.res_w, rx, ry, v);
        } else if (im.interp == Y5_VAL_LINEAR) {
            linear_px(im.src, im.row_bytes, im.src_h, im.src_w, im.res_h, im.res_w, rx, ry, v);
        } else {
            const uint8_t* p = im.src + static_cast<long long>(ry) * im.row_bytes + rx * 3;
            v[0] = p[0]; v[1] = p[1]; v[2] = p[2];
        }
    }
    if (to_scratch) {
        uint8_t* d = im.dst + (static_cast<long long>(ry) * im.res_w + rx) * 3;
        d[0] = static_cast<uint8_t>(v[0]); d[1] = static_cast<uint8_t>(v[1]); d[2] = static_cast<uint8_t>(v[2]);
        return;
    }
    const long long plane = static_cast<long long>(out_h) * out_w;
    const long long o = static_cast<long long>(b) * 3 * plane + static_cast<long long>(oy) * out_w + ox;
    const float inv255 = 1.0f / 255.0f;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        const int x = v[2 - c];  // BGR -> RGB
        if (OUT == 0) static_cast<uint8_t*>(out)[o + c * plane] = static_cast<uint8_t>(x);
        else if (OUT == 1) static_cast<uint16_t*>(out)[o + c * plane] = pack1(__fmul_rn(static_cast<float>(x), inv255), bf16 != 0);
        else static_cast<float*>(out)[o + c * plane] = __fmul_rn(static_cast<float>(x), inv255);
    }
}

// ---------------------------------------------------------------------------------------------------------------------
// classification batch: CenterCrop's resize + ToTensor + Normalize
// ---------------------------------------------------------------------------------------------------------------------
struct ClsNorm {
    float mean[3], std[3];
};

// OUT: 1 = fp16/bf16, 2 = fp32; CHW RGB.  The descriptor table is in device memory: every thread of a block reads the
// same 16 bytes, so the loads are broadcasts
template <int OUT>
__global__ void cls_batch_kernel(const y5_cls_image* __restrict__ images, int out_h, int out_w, const ClsNorm N, void* __restrict__ out, int bf16) {
    const int b = blockIdx.z;
    const int ox = blockIdx.x * blockDim.x + threadIdx.x, oy = blockIdx.y * blockDim.y + threadIdx.y;
    if (ox >= out_w || oy >= out_h) return;
    const y5_cls_image im = images[b];
    if (im.side <= 0 || im.row_bytes < 3 * im.side) return;
    int v[3];
    linear_px(static_cast<const uint8_t*>(im.data), im.row_bytes, im.side, im.side, out_h, out_w, ox, oy, v);
    const long long plane = static_cast<long long>(out_h) * out_w;
    const long long o = static_cast<long long>(b) * 3 * plane + static_cast<long long>(oy) * out_w + ox;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        // ToTensor's `/= 255` on a CPU float32 tensor is a true division (not a multiply by 1/255), then Normalize
        const float x = __fdiv_rn(static_cast<float>(v[2 - c]), 255.0f);  // BGR -> RGB
        const float y = __fdiv_rn(__fsub_rn(x, N.mean[c]), N.std[c]);
        if (OUT == 1) static_cast<uint16_t*>(out)[o + c * plane] = pack1(y, bf16 != 0);
        else static_cast<float*>(out)[o + c * plane] = y;
    }
}

// ---------------------------------------------------------------------------------------------------------------------
// process_mask
// ---------------------------------------------------------------------------------------------------------------------
constexpr int kMaskDets = 8;     // detections per thread pass (prototype vector stays in registers)
constexpr int kMaskMaxC = 64;    // prototype channels

__device__ __forceinline__ float load_proto(const void* p, long long i, int dtype) {
    if (dtype == Y5_F32) return static_cast<const float*>(p)[i];
    return unpack1(static_cast<const uint16_t*>(p)[i], dtype == Y5_BF16);
}

// low-resolution masks: sigmoid(coef . protos[:, pixel]) cropped to the (down-scaled) box.
// FINAL: 1 = threshold here and write the final {0,1} mask, 0 = write the cropped fp32 values for the up-sampling pass
template <int FINAL>
__global__ void mask_lowres_kernel(const void* __restrict__ protos, int pdtype, int c, int mh, int mw, const float* __restrict__ coef,
                                   int coef_stride, const float* __restrict__ boxes, int box_stride, const int32_t* __restrict__ img_index,
                                   int n, float sxw, float syh, int crop, void* __restrict__ out, int out_u8) {
    extern __shared__ float s_coef[];  // [kMaskDets][c] + boxes [kMaskDets][4] + image [kMaskDets]
    float* s_box = s_coef + kMaskDets * c;
    int* s_img = reinterpret_cast<int*>(s_box + kMaskDets * 4);
    const int hw = mh * mw;
    const int d0 = blockIdx.y * kMaskDets;
    const int nd = min(kMaskDets, n - d0);
    for (int i = threadIdx.x; i < nd * c; i += blockDim.x) s_coef[i] = coef[static_cast<long long>(d0 + i / c) * coef_stride + (i % c)];
    for (int i = threadIdx.x; i < nd; i += blockDim.x) {
        const float* bp = boxes + static_cast<long long>(d0 + i) * box_stride;
        // downsampled_bboxes[:, 0] *= mw / iw ... (utils/segment/general.py:43-47): one fp32 multiply each
        s_box[i * 4 + 0] = __fmul_rn(bp[0], sxw);
        s_box[i * 4 + 1] = __fmul_rn(bp[1], syh);
        s_box[i * 4 + 2] = __fmul_rn(bp[2], sxw);
        s_box[i * 4 + 3] = __fmul_rn(bp[3], syh);
        s_img[i] = img_index ? img_index[d0 + i] : 0;
    }
    __syncthreads();
    const int pix = blockIdx.x * blockDim.x + threadIdx.x;
    if (pix >= hw) return;
    const float fx = static_cast<float>(pix % mw), fy = static_cast<float>(pix / mw);
    float pv[kMaskMaxC];
    int cur_img = -1;
    for (int j = 0; j < nd; ++j) {
        if (s_img[j] != cur_img) {  // detections arrive grouped by image: reload the prototype vector only when it changes
            cur_img = s_img[j];
            const long long base = static_cast<long long>(cur_img) * c * hw + pix;
#pragma unroll
            for (int k = 0; k < kMaskMaxC; ++k)
                if (k < c) pv[k] = load_proto(protos, base + static_cast<long long>(k) * hw, pdtype);
        }
        float acc = 0.f;
#pragma unroll
        for (int k = 0; k < kMaskMaxC; ++k)
            if (k < c) acc = fmaf(s_coef[j * c + k], pv[k], acc);
        float m = __fdiv_rn(1.0f, __fadd_rn(1.0f, expf(-acc)));
        const bool in = fx >= s_box[j * 4 + 0] && fx < s_box[j * 4 + 2] && fy >= s_box[j * 4 + 1] && fy < s_box[j * 4 + 3];
        if (crop && !in) m = 0.f;
        const long long o = static_cast<long long>(d0 + j) * hw + pix;
        if (FINAL) {
            const bool on = m > 0.5f;
            if (out_u8) static_cast<uint8_t*>(out)[o] = on ? 1 : 0;
            else static_cast<float*>(out)[o] = on ? 1.0f : 0.0f;
        } else {
            static_cast<float*>(out)[o] = m;
        }
    }
}

// F.interpolate(mode='bilinear', align_corners=False) of a window [y_off, y_off+win_h) x [x_off, x_off+win_w) of the low
// resolution masks to (oh, ow), optional crop to full-resolution boxes (process_mask_native), then > 0.5
__global__ void mask_upsample_kernel(const float* __restrict__ low, int n, int mh, int mw, int y_off, int x_off, int win_h, int win_w, int oh,
                                     int ow, const float* __restrict__ boxes, int box_stride, void* __restrict__ out, int out_u8) {
    const float scale_y = __fdiv_rn(static_cast<float>(win_h), static_cast<float>(oh));
    const float scale_x = __fdiv_rn(static_cast<float>(win_w), static_cast<float>(ow));
    const long long total = static_cast<long long>(n) * oh * ow;
    for (long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; idx < total;
         idx += static_cast<long long>(gridDim.x) * blockDim.x) {
        const int ox = static_cast<int>(idx % ow);
        const int oy = static_cast<int>((idx / ow) % oh);
        const int d = static_cast<int>(idx / (static_cast<long long>(ow) * oh));
        const float srcy = fmaxf(__fsub_rn(__fmul_rn(__fadd_rn(static_cast<float>(oy), 0.5f), scale_y), 0.5f), 0.f);
        const float srcx = fmaxf(__fsub_rn(__fmul_rn(__fadd_rn(static_cast<float>(ox), 0.5f), scale_x), 0.5f), 0.f);
        const int y0 = min(static_cast<int>(srcy), win_h - 1), x0 = min(static_cast<int>(srcx), win_w - 1);
        const int y1 = min(y0 + 1, win_h - 1), x1 = min(x0 + 1, win_w - 1);
        const float ly = __fsub_rn(srcy, static_cast<float>(y0)), lx = __fsub_rn(srcx, static_cast<float>(x0));
        const float* p = low + static_cast<long long>(d) * mh * mw + static_cast<long long>(y_off) * mw + x_off;
        const float v00 = p[y0 * mw + x0], v01 = p[y0 * mw + x1], v10 = p[y1 * mw + x0], v11 = p[y1 * mw + x1];
        const float hx = __fsub_rn(1.0f, lx), hy = __fsub_rn(1.0f, ly);
        const float top = __fadd_rn(__fmul_rn(v00, hx), __fmul_rn(v01, lx));
        const float bot = __fadd_rn(__fmul_rn(v10, hx), __fmul_rn(v11, lx));
        float v = __fadd_rn(__fmul_rn(top, hy), __fmul_rn(bot, ly));
        if (boxes) {
            const float* b = boxes + static_cast<long long>(d) * box_stride;
            const float fx = static_cast<float>(ox), fy = static_cast<float>(oy);
            if (!(fx >= b[0] && fx < b[2] && fy >= b[1] && fy < b[3])) v = 0.f;
        }
        const bool on = v > 0.5f;
        if (out_u8) static_cast<uint8_t*>(out)[idx] = on ? 1 : 0;
        else static_cast<float*>(out)[idx] = on ? 1.0f : 0.0f;
    }
}

// crop_mask (utils/segment/general.py:10-22) on its own: masks (n,h,w) fp32 times the box indicator, out of place
__global__ void crop_mask_kernel(const float* __restrict__ masks, const float* __restrict__ boxes, int box_stride, int n, int h, int w,
                                 float* __restrict__ out) {
    const long long total = static_cast<long long>(n) * h * w;
    for (long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; idx < total;
         idx += static_cast<long long>(gridDim.x) * blockDim.x) {
        const int x = static_cast<int>(idx % w);
        const int y = static_cast<int>((idx / w) % h);
        const float* b = boxes + (idx / (static_cast<long long>(w) * h)) * box_stride;
        const float fx = static_cast<float>(x), fy = static_cast<float>(y);
        const bool in = fx >= b[0] && fx < b[2] && fy >= b[1] && fy < b[3];
        out[idx] = in ? masks[idx] : __fmul_rn(masks[idx], 0.0f);
    }
}

// ---------------------------------------------------------------------------------------------------------------------
// scale_boxes / labels to native space / process_batch
// ---------------------------------------------------------------------------------------------------------------------
// meta per image: [gain, pad_x, pad_y, w0, h0]  (img0 = the original image, utils/general.py:613-626)
__device__ __forceinline__ void scale_clip(float (&b)[4], const float* m) {
    b[0] = __fdiv_rn(__fsub_rn(b[0], m[1]), m[0]);
    b[2] = __fdiv_rn(__fsub_rn(b[2], m[1]), m[0]);
    b[1] = __fdiv_rn(__fsub_rn(b[1], m[2]), m[0]);
    b[3] = __fdiv_rn(__fsub_rn(b[3], m[2]), m[0]);
    b[0] = fminf(fmaxf(b[0], 0.f), m[3]);
    b[2] = fminf(fmaxf(b[2], 0.f), m[3]);
    b[1] = fminf(fmaxf(b[1], 0.f), m[4]);
    b[3] = fminf(fmaxf(b[3], 0.f), m[4]);
}

// boxes: n rows of `stride` floats, xyxy in the first 4; img_index NULL -> rows_per_image > 0 gives image = row / rows_per_image
__global__ void scale_boxes_kernel(float* __restrict__ boxes, int stride, long long n, const int32_t* __restrict__ img_index, int rows_per_image,
                                   const int32_t* __restrict__ count, const float* __restrict__ meta) {
    for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += static_cast<long long>(gridDim.x) * blockDim.x) {
        int img = 0;
        if (img_index) img = img_index[i];
        else if (rows_per_image > 0) {
            img = static_cast<int>(i / rows_per_image);
            if (count && static_cast<int>(i - static_cast<long long>(img) * rows_per_image) >= count[img]) continue;  // padding rows stay untouched
        }
        float b[4];
        float* p = boxes + i * stride;
#pragma unroll
        for (int k = 0; k < 4; ++k) b[k] = p[k];
        scale_clip(b, meta + img * 5);
#pragma unroll
        for (int k = 0; k < 4; ++k) p[k] = b[k];
    }
}

// targets (nt,6) [img, cls, cx, cy, w, h] in network-input pixels -> (nt,6) [img, cls, x1, y1, x2, y2] in native pixels:
// xywh2xyxy (val.py:304) then scale_boxes (val.py:305)
__global__ void labels_native_kernel(const float* __restrict__ tg, int nt, const float* __restrict__ meta, float* __restrict__ out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= nt) return;
    const float* t = tg + static_cast<long long>(i) * 6;
    const int img = static_cast<int>(t[0]);
    const float hw = __fdiv_rn(t[4], 2.0f), hh = __fdiv_rn(t[5], 2.0f);
    float b[4] = {__fsub_rn(t[2], hw), __fsub_rn(t[3], hh), __fadd_rn(t[2], hw), __fadd_rn(t[3], hh)};
    scale_clip(b, meta + img * 5);
    float* o = out + static_cast<long long>(i) * 6;
    o[0] = t[0];
    o[1] = t[1];
    o[2] = b[0]; o[3] = b[1]; o[4] = b[2]; o[5] = b[3];
}

__device__ __forceinline__ float iou_label_det(const float* l, const float* d, float eps) {  // box_iou(labels, detections) element
    const float a1 = __fmul_rn(__fsub_rn(l[2], l[0]), __fsub_rn(l[3], l[1]));
    const float a2 = __fmul_rn(__fsub_rn(d[2], d[0]), __fsub_rn(d[3], d[1]));
    const float w = fmaxf(__fsub_rn(fminf(l[2], d[2]), fmaxf(l[0], d[0])), 0.0f);
    const float h = fmaxf(__fsub_rn(fminf(l[3], d[3]), fmaxf(l[1], d[1])), 0.0f);
    const float inter = __fmul_rn(w, h);
    return __fdiv_rn(inter, __fadd_rn(__fsub_rn(__fadd_rn(a1, a2), inter), eps));
}

// One block per image.  Detection d's best label = the same-class label with the highest IoU (first label on ties: the
// reference's stable descending sort keeps (label, detection) scan order); then match_assign (match_rule.cuh).
__global__ void match_kernel(const float* __restrict__ det, long long img_stride, int row_stride, const int32_t* __restrict__ count,
                             int max_det, const float* __restrict__ labels, int nt, const float* __restrict__ iouv, int niou, float eps,
                             uint8_t* __restrict__ correct) {
    __shared__ int s_best[kMatchMaxDet];
    __shared__ float s_iou[kMatchMaxDet];
    const int b = blockIdx.x;
    const int n = min(count ? count[b] : max_det, max_det);
    const float* dbase = det + static_cast<long long>(b) * img_stride;
    for (int d = threadIdx.x; d < n; d += blockDim.x) {
        const float* dp = dbase + static_cast<long long>(d) * row_stride;
        const float db[4] = {dp[0], dp[1], dp[2], dp[3]};
        const float dcls = dp[5];
        int best = -1;
        float best_iou = -1.0f;
        for (int l = 0; l < nt; ++l) {
            const float* lp = labels + static_cast<long long>(l) * 6;
            if (static_cast<int>(lp[0]) != b || lp[1] != dcls) continue;
            const float v = iou_label_det(lp + 2, db, eps);
            if (v > best_iou) { best_iou = v; best = l; }
        }
        s_best[d] = best;
        s_iou[d] = best_iou;
    }
    __syncthreads();
    match_assign(s_best, s_iou, n, max_det, iouv, niou, correct + static_cast<long long>(b) * max_det * niou);
}

// ConfusionMatrix.process_batch (utils/metrics.py:139-183) for one image per block, counts added into `matrix` (nc+1)^2.
// Kept detections: conf > conf_thres.  Candidates: iou > iou_thres, any classes.  Each kept detection keeps its best label
// (highest IoU, first label on ties), then each label keeps, among the detections whose best it is, the one with the highest
// IoU (first detection on ties).  A class is `.int()` of its value: values outside (-1, nc) set an error bit, never a write.
constexpr int kConfusionLabelErr = 1, kConfusionDetErr = 2;  // bits of the error word
constexpr int kNoLabel = -1, kDropped = -2;  // s_best of a kept detection without a candidate, of a detection at or below conf_thres

__device__ __forceinline__ bool confusion_class(float c, int nc) { return c > -1.0f && c < static_cast<float>(nc); }  // .int() in [0, nc)

__device__ __forceinline__ void confusion_add(unsigned long long* matrix, int nc, int row, int col) {
    atomicAdd(matrix + static_cast<long long>(row) * (nc + 1) + col, 1ull);
}

__global__ void confusion_kernel(const float* __restrict__ det, long long img_stride, int row_stride, const int32_t* __restrict__ count,
                                 int max_det, const float* __restrict__ labels, int nt, int nc, float conf_thres, float iou_thres, float eps,
                                 unsigned long long* __restrict__ matrix, int* __restrict__ error) {
    __shared__ int s_best[kMatchMaxDet];
    __shared__ float s_iou[kMatchMaxDet];
    __shared__ uint8_t s_won[kMatchMaxDet];
    __shared__ int s_any;
    const int b = blockIdx.x;
    const int n = max(0, min(count ? count[b] : max_det, max_det));
    const float* dbase = det + static_cast<long long>(b) * img_stride;
    if (threadIdx.x == 0) s_any = 0;
    for (int d = threadIdx.x; d < n; d += blockDim.x) {
        const float* dp = dbase + static_cast<long long>(d) * row_stride;
        s_won[d] = 0;
        if (!(dp[4] > conf_thres)) {
            s_best[d] = kDropped;
            continue;
        }
        const float db[4] = {dp[0], dp[1], dp[2], dp[3]};
        int best = kNoLabel;
        float best_iou = 0.0f;
        for (int l = 0; l < nt; ++l) {
            const float* lp = labels + static_cast<long long>(l) * 6;
            if (static_cast<int>(lp[0]) != b) continue;
            const float v = iou_label_det(lp + 2, db, eps);
            if (v > iou_thres && (best == kNoLabel || v > best_iou)) { best_iou = v; best = l; }
        }
        s_best[d] = best;
        s_iou[d] = best_iou;
    }
    __syncthreads();
    // one count per label of this image: at [class of its winning detection, class] or, without one, at [nc, class]
    for (int l = threadIdx.x; l < nt; l += blockDim.x) {
        const float* lp = labels + static_cast<long long>(l) * 6;
        if (static_cast<int>(lp[0]) != b) continue;
        int win = -1;
        float win_iou = 0.0f;
        for (int d = 0; d < n; ++d)
            if (s_best[d] == l && (win < 0 || s_iou[d] > win_iou)) { win_iou = s_iou[d]; win = d; }
        if (win >= 0) {
            s_won[win] = 1;
            s_any = 1;
        }
        const float gc = lp[1];
        const float dc = win >= 0 ? dbase[static_cast<long long>(win) * row_stride + 5] : 0.0f;
        if (!confusion_class(gc, nc)) atomicOr(error, kConfusionLabelErr);
        else if (!confusion_class(dc, nc)) atomicOr(error, kConfusionDetErr);
        else confusion_add(matrix, nc, win >= 0 ? static_cast<int>(dc) : nc, static_cast<int>(gc));
    }
    __syncthreads();
    if (!s_any) return;  // the reference counts unmatched detections only in an image with at least one match
    for (int d = threadIdx.x; d < n; d += blockDim.x) {
        if (s_best[d] == kDropped || s_won[d]) continue;
        const float dc = dbase[static_cast<long long>(d) * row_stride + 5];
        if (confusion_class(dc, nc)) confusion_add(matrix, nc, static_cast<int>(dc), nc);
        else atomicOr(error, kConfusionDetErr);
    }
}

}  // namespace y5

using namespace y5;

extern "C" Y5_API int y5_letterbox_max_images(void) { return kLbMaxImages; }

extern "C" Y5_API int y5_letterbox(const y5_letterbox_image* images, int32_t n_images, int32_t out_h, int32_t out_w, int32_t swap_rb,
                                   int32_t pad_value, void* out, int32_t out_dtype, int32_t s2d, int32_t out_row_px, int32_t out_x_off,
                                   void* stream) {
    if (!images || !out || n_images <= 0 || out_h <= 0 || out_w <= 0) return set_error(Y5_E_INVALID, "letterbox: bad argument");
    if (pad_value < 0 || pad_value > 255) return set_error(Y5_E_INVALID, "letterbox: pad value must be a byte");
    if (s2d && ((out_h | out_w) & 1)) return set_error(Y5_E_INVALID, "letterbox: space-to-depth output needs even height/width");
    if (s2d && out_dtype != Y5_F16 && out_dtype != Y5_BF16) return set_error(Y5_E_UNSUPPORTED, "letterbox: s2d output is fp16/bf16");
    if (!s2d && out_dtype != Y5_U8 && out_dtype != Y5_F16 && out_dtype != Y5_BF16 && out_dtype != Y5_F32)
        return set_error(Y5_E_UNSUPPORTED, "letterbox: output dtype");
    for (int i = 0; i < n_images; ++i) {
        const y5_letterbox_image& im = images[i];
        if (!im.data || im.src_h <= 0 || im.src_w <= 0 || im.new_h <= 0 || im.new_w <= 0 || im.row_bytes < im.src_w * 3 || im.top < 0 ||
            im.left < 0 || im.top + im.new_h > out_h || im.left + im.new_w > out_w)
            return set_error(Y5_E_INVALID, "letterbox: image %d does not fit the %dx%d output (src %dx%d new %dx%d top %d left %d)", i, out_h, out_w,
                             im.src_h, im.src_w, im.new_h, im.new_w, im.top, im.left);
    }
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const int step = s2d ? 2 : 1;
    const dim3 block(32, 8);
    const size_t img_elems = static_cast<size_t>(3) * out_h * out_w;
    for (int i0 = 0; i0 < n_images; i0 += kLbMaxImages) {
        const int nb = n_images - i0 < kLbMaxImages ? n_images - i0 : kLbMaxImages;
        LbBatch L;
        for (int i = 0; i < nb; ++i) L.im[i] = images[i0 + i];
        const dim3 grid((out_w / step + block.x - 1) / block.x, (out_h / step + block.y - 1) / block.y, nb);
        const int bf = out_dtype == Y5_BF16;
        int e;
        if (s2d) {
            const int row_px = out_row_px ? out_row_px : out_w / 2;
            uint8_t* o = static_cast<uint8_t*>(out) + static_cast<size_t>(i0) * (out_h / 2) * row_px * 32;
            e = launch("letterbox", letterbox_kernel<3>, {grid, block, 0, st}, L, nb, out_h, out_w, swap_rb, pad_value, o, bf, row_px, out_x_off);
        } else if (out_dtype == Y5_U8) {
            e = launch("letterbox", letterbox_kernel<0>, {grid, block, 0, st}, L, nb, out_h, out_w, swap_rb, pad_value,
                       static_cast<uint8_t*>(out) + i0 * img_elems, bf, 0, 0);
        } else if (out_dtype == Y5_F32) {
            e = launch("letterbox", letterbox_kernel<2>, {grid, block, 0, st}, L, nb, out_h, out_w, swap_rb, pad_value,
                       static_cast<float*>(out) + i0 * img_elems, bf, 0, 0);
        } else {
            e = launch("letterbox", letterbox_kernel<1>, {grid, block, 0, st}, L, nb, out_h, out_w, swap_rb, pad_value,
                       static_cast<uint16_t*>(out) + i0 * img_elems, bf, 0, 0);
        }
        if (e) return e;
    }
    return 0;
}

static int launch_val(const ValBatch& L, int nb, int grid_w, int grid_h, int out_h, int out_w, void* out, int out_dtype, cudaStream_t st) {
    const dim3 block(32, 8);
    const dim3 grid((grid_w + block.x - 1) / block.x, (grid_h + block.y - 1) / block.y, nb);
    auto* kernel = out_dtype == Y5_U8 ? val_letterbox_kernel<0> : out_dtype == Y5_F32 ? val_letterbox_kernel<2> : val_letterbox_kernel<1>;
    return launch("val_letterbox", kernel, {grid, block, 0, st}, L, out_h, out_w, out, out_dtype == Y5_BF16);
}

extern "C" Y5_API int y5_val_letterbox(const y5_val_image* images, int32_t n_images, int32_t out_h, int32_t out_w, void* out, int32_t out_dtype,
                                       void* stream) {
    if (!images || !out || n_images <= 0 || out_h <= 0 || out_w <= 0) return set_error(Y5_E_INVALID, "val_letterbox: bad argument");
    if (out_dtype != Y5_U8 && out_dtype != Y5_F16 && out_dtype != Y5_BF16 && out_dtype != Y5_F32)
        return set_error(Y5_E_UNSUPPORTED, "val_letterbox: output dtype");
    constexpr int kMaxSide = 1 << 15;
    if (out_h > kMaxSide || out_w > kMaxSide) return set_error(Y5_E_UNSUPPORTED, "val_letterbox: canvas larger than %d", kMaxSide);
    for (int i = 0; i < n_images; ++i) {
        const y5_val_image& im = images[i];
        const bool again = im.new_h != im.res_h || im.new_w != im.res_w;
        if (!im.data || im.src_h <= 0 || im.src_w <= 0 || im.res_h <= 0 || im.res_w <= 0 || im.new_h <= 0 || im.new_w <= 0 ||
            im.row_bytes < im.src_w * 3 || im.top < 0 || im.left < 0 || im.top + im.new_h > out_h || im.left + im.new_w > out_w ||
            (again && !im.scratch))
            return set_error(Y5_E_INVALID, "val_letterbox: image %d does not fit the %dx%d output (src %dx%d load %dx%d new %dx%d top %d left %d%s)", i,
                             out_h, out_w, im.src_h, im.src_w, im.res_h, im.res_w, im.new_h, im.new_w, im.top, im.left,
                             again && !im.scratch ? ", no scratch" : "");
        if (im.src_h > kMaxSide || im.src_w > kMaxSide || im.res_h > kMaxSide || im.res_w > kMaxSide)
            return set_error(Y5_E_UNSUPPORTED, "val_letterbox: image %d larger than %d", i, kMaxSide);
        const bool ok = im.interp == Y5_VAL_COPY ? im.res_h == im.src_h && im.res_w == im.src_w
                      : im.interp == Y5_VAL_AREA ? im.res_h <= im.src_h && im.res_w <= im.src_w
                                                 : im.interp == Y5_VAL_LINEAR;
        if (!ok) return set_error(Y5_E_UNSUPPORTED, "val_letterbox: image %d: interp %d from %dx%d to %dx%d", i, im.interp, im.src_h, im.src_w, im.res_h,
                                  im.res_w);
    }
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const size_t elem = out_dtype == Y5_U8 ? 1 : (out_dtype == Y5_F32 ? 4 : 2);
    const size_t img_bytes = static_cast<size_t>(3) * out_h * out_w * elem;
    for (int i0 = 0; i0 < n_images; i0 += kValMaxImages) {
        const int nb = n_images - i0 < kValMaxImages ? n_images - i0 : kValMaxImages;
        ValBatch L, A;  // L: load_image (+ letterbox when it only pads); A: letterbox's own resize from the scratch
        int gw = out_w, gh = out_h, again = 0;
        for (int i = 0; i < nb; ++i) {
            const y5_val_image& im = images[i0 + i];
            ValDesc& d = L.im[i];
            d = ValDesc{static_cast<const uint8_t*>(im.data), static_cast<uint8_t*>(im.scratch), im.src_h, im.src_w, im.row_bytes, im.res_h, im.res_w,
                        im.interp, im.top, im.left, kValCanvas, 0};
            A.im[i] = ValDesc{nullptr, nullptr, 0, 0, 0, 0, 0, 0, 0, 0, kValSkip, 0};
            if (im.new_h != im.res_h || im.new_w != im.res_w) {
                d.mode = kValScratch;
                gw = gw > im.res_w ? gw : im.res_w;
                gh = gh > im.res_h ? gh : im.res_h;
                A.im[i] = ValDesc{static_cast<const uint8_t*>(im.scratch), nullptr, im.res_h, im.res_w, im.res_w * 3, im.new_h, im.new_w, Y5_VAL_LINEAR,
                                  im.top, im.left, kValCanvas, 0};
                again = 1;
            }
        }
        void* o = static_cast<uint8_t*>(out) + static_cast<size_t>(i0) * img_bytes;
        if (int e = launch_val(L, nb, gw, gh, out_h, out_w, o, out_dtype, st)) return e;
        if (again)
            if (int e = launch_val(A, nb, out_w, out_h, out_h, out_w, o, out_dtype, st)) return e;
    }
    return 0;
}

extern "C" Y5_API int y5_cls_batch(const y5_cls_image* images, int32_t n_images, int32_t out_h, int32_t out_w, const float* mean, const float* std,
                                   void* out, int32_t out_dtype, void* stream) {
    if (!images || !out || !mean || !std || n_images <= 0 || out_h <= 0 || out_w <= 0) return set_error(Y5_E_INVALID, "cls_batch: bad argument");
    if (out_dtype != Y5_F16 && out_dtype != Y5_BF16 && out_dtype != Y5_F32) return set_error(Y5_E_UNSUPPORTED, "cls_batch: output dtype");
    constexpr int kMaxSide = 1 << 14, kMaxImages = 65535;  // grid.z carries the image
    if (out_h > kMaxSide || out_w > kMaxSide) return set_error(Y5_E_UNSUPPORTED, "cls_batch: output larger than %d", kMaxSide);
    if (n_images > kMaxImages) return set_error(Y5_E_UNSUPPORTED, "cls_batch: %d images (max %d per launch)", n_images, kMaxImages);
    ClsNorm N;
    for (int c = 0; c < 3; ++c) {
        if (!(std[c] != 0.0f)) return set_error(Y5_E_INVALID, "cls_batch: std[%d] is zero", c);
        N.mean[c] = mean[c];
        N.std[c] = std[c];
    }
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const dim3 block(32, 8);
    const dim3 grid((out_w + block.x - 1) / block.x, (out_h + block.y - 1) / block.y, n_images);
    return launch("cls_batch", out_dtype == Y5_F32 ? cls_batch_kernel<2> : cls_batch_kernel<1>, {grid, block, 0, st}, images, out_h, out_w, N, out,
                  out_dtype == Y5_BF16);
}

extern "C" Y5_API int64_t y5_process_mask_workspace_bytes(int32_t n, int32_t mh, int32_t mw, int32_t mode) {
    return mode != 0 ? static_cast<int64_t>(n) * mh * mw * 4 + 256 : 0;
}

extern "C" Y5_API int y5_process_mask(const void* protos, int32_t proto_dtype, int32_t batch, int32_t c, int32_t mh, int32_t mw,
                                      const float* coef, int32_t coef_stride, const float* boxes, int32_t box_stride,
                                      const int32_t* img_index, int32_t n, int32_t in_h, int32_t in_w, int32_t mode, const int32_t* window,
                                      void* out, int32_t out_dtype, void* workspace, int64_t workspace_bytes, void* stream) {
    if (n == 0) return 0;
    if (!protos || !coef || !boxes || !out || n < 0 || batch <= 0 || mh <= 0 || mw <= 0 || in_h <= 0 || in_w <= 0)
        return set_error(Y5_E_INVALID, "process_mask: bad argument");
    if (mode < 0 || mode > 2) return set_error(Y5_E_INVALID, "process_mask: mode must be 0 (mask resolution), 1 (up-sampled) or 2 (native)");
    if (c <= 0 || c > kMaskMaxC) return set_error(Y5_E_UNSUPPORTED, "process_mask: %d prototype channels (max %d)", c, kMaskMaxC);
    if (proto_dtype != Y5_F16 && proto_dtype != Y5_BF16 && proto_dtype != Y5_F32) return set_error(Y5_E_UNSUPPORTED, "process_mask: proto dtype");
    if (out_dtype != Y5_F32 && out_dtype != Y5_U8) return set_error(Y5_E_UNSUPPORTED, "process_mask: output dtype must be fp32 or uint8");
    if (mode != 0 && (!workspace || workspace_bytes < y5_process_mask_workspace_bytes(n, mh, mw, mode)))
        return set_error(Y5_E_INVALID, "process_mask: workspace too small");
    int wy = 0, wx = 0, wh = mh, ww = mw;
    if (mode == 2) {
        if (!window) return set_error(Y5_E_INVALID, "process_mask: native mode needs the prototype window [top, left, height, width]");
        wy = window[0]; wx = window[1]; wh = window[2]; ww = window[3];
        if (wy < 0 || wx < 0 || wh <= 0 || ww <= 0 || wy + wh > mh || wx + ww > mw) return set_error(Y5_E_INVALID, "process_mask: bad window");
    }
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const int hw = mh * mw;
    const dim3 grid((hw + 255) / 256, (n + kMaskDets - 1) / kMaskDets);
    const size_t smem = static_cast<size_t>(kMaskDets) * (c + 4) * sizeof(float) + kMaskDets * sizeof(int);
    // python-float ratios rounded once to fp32, as `tensor *= mw / iw` does
    const float sxw = static_cast<float>(static_cast<double>(mw) / static_cast<double>(in_w));
    const float syh = static_cast<float>(static_cast<double>(mh) / static_cast<double>(in_h));
    if (mode == 0)
        return launch("process_mask", mask_lowres_kernel<1>, {grid, 256, smem, st}, protos, proto_dtype, c, mh, mw, coef, coef_stride, boxes,
                      box_stride, img_index, n, sxw, syh, 1, out, out_dtype == Y5_U8);
    float* low = reinterpret_cast<float*>((reinterpret_cast<uintptr_t>(workspace) + 255) & ~uintptr_t(255));
    if (int e = launch("process_mask", mask_lowres_kernel<0>, {grid, 256, smem, st}, protos, proto_dtype, c, mh, mw, coef, coef_stride, boxes,
                       box_stride, img_index, n, sxw, syh, mode == 1, low, 0))
        return e;
    const long long total = static_cast<long long>(n) * in_h * in_w;
    return launch("process_mask", mask_upsample_kernel, {grid_stride_ctas(total, 256, 32), 256, 0, st}, low, n, mh, mw, wy, wx, wh, ww, in_h, in_w,
                  mode == 2 ? boxes : nullptr, box_stride, out, out_dtype == Y5_U8);
}

extern "C" Y5_API int y5_crop_mask(const float* masks, const float* boxes, int32_t box_stride, int32_t n, int32_t h, int32_t w, float* out,
                                   void* stream) {
    if (n == 0) return 0;
    if (!masks || !boxes || !out || n < 0 || h <= 0 || w <= 0 || box_stride < 4) return set_error(Y5_E_INVALID, "crop_mask: bad argument");
    const long long total = static_cast<long long>(n) * h * w;
    return launch("crop_mask", crop_mask_kernel, {grid_stride_ctas(total, 256, 16), 256, 0, static_cast<cudaStream_t>(stream)}, masks, boxes,
                  box_stride, n, h, w, out);
}

extern "C" Y5_API int y5_scale_boxes(float* boxes, int32_t row_stride, int64_t n_rows, const int32_t* img_index, int32_t rows_per_image,
                                     const int32_t* count, const float* meta, void* stream) {
    if (n_rows == 0) return 0;
    if (!boxes || !meta || n_rows < 0 || row_stride < 4) return set_error(Y5_E_INVALID, "scale_boxes: bad argument");
    return launch("scale_boxes", scale_boxes_kernel, {grid_stride_ctas(n_rows, 256, 8), 256, 0, static_cast<cudaStream_t>(stream)}, boxes,
                  row_stride, n_rows, img_index, rows_per_image, count, meta);
}

extern "C" Y5_API int y5_labels_native(const float* targets, int32_t nt, const float* meta, float* out, void* stream) {
    if (nt == 0) return 0;
    if (!targets || !meta || !out || nt < 0) return set_error(Y5_E_INVALID, "labels_native: bad argument");
    return launch("labels_native", labels_native_kernel, {(nt + 127) / 128, 128, 0, static_cast<cudaStream_t>(stream)}, targets, nt, meta, out);
}

extern "C" Y5_API int y5_match_batch(const float* det, int64_t img_stride, int32_t row_stride, const int32_t* count, int32_t batch,
                                     int32_t max_det, const float* labels, int32_t nt, const float* iouv, int32_t niou, float eps,
                                     uint8_t* correct, void* stream) {
    if (batch <= 0 || max_det <= 0) return 0;
    if (!det || !iouv || !correct || niou <= 0 || row_stride < 6 || nt < 0 || (nt > 0 && !labels))
        return set_error(Y5_E_INVALID, "match_batch: bad argument");
    if (max_det > kMatchMaxDet) return set_error(Y5_E_UNSUPPORTED, "match_batch: max_det %d > %d", max_det, kMatchMaxDet);
    return launch("match_batch", match_kernel, {batch, 256, 0, static_cast<cudaStream_t>(stream)}, det, img_stride, row_stride, count, max_det,
                  labels, nt, iouv, niou, eps, correct);
}

extern "C" Y5_API int y5_confusion_batch(const float* det, int64_t img_stride, int32_t row_stride, const int32_t* count, int32_t batch,
                                         int32_t max_det, const float* labels, int32_t nt, int32_t nc, float conf_thres, float iou_thres,
                                         float eps, int64_t* matrix, int32_t* error, void* stream) {
    if (batch == 0) return 0;
    if (batch < 0 || max_det < 0 || nt < 0 || nc <= 0 || row_stride < 6 || !matrix || !error || (max_det > 0 && !det) || (nt > 0 && !labels))
        return set_error(Y5_E_INVALID, "confusion_batch: bad argument");
    if (max_det > kMatchMaxDet) return set_error(Y5_E_UNSUPPORTED, "confusion_batch: max_det %d > %d", max_det, kMatchMaxDet);
    if (nc > (1 << 15)) return set_error(Y5_E_UNSUPPORTED, "confusion_batch: nc %d > %d", nc, 1 << 15);
    return launch("confusion_batch", confusion_kernel, {batch, 256, 0, static_cast<cudaStream_t>(stream)}, det, img_stride, row_stride, count,
                  max_det, labels, nt, nc, conf_thres, iou_thres, eps, reinterpret_cast<unsigned long long*>(matrix), error);
}
