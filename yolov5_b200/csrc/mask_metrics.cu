// Mask-IoU matching of segment/val.py (utils/metrics.py:239-265 process_batch(masks=True), ultralytics' mask_iou) for a whole
// batch, with no host synchronisation:
//   mask_labels_kernel : each label's row in the per-image label blocks (target order inside an image), on the device
//   mask_pack_kernel   : masks -> bit rows + popcounts; direct 0/1 masks or overlap index images, optionally resized
//                        (F.interpolate bilinear, align_corners=False, then > 0.5) on the way.  One block per bit row: an
//                        overlap index plane is read once per label of its image (L2-resident after the first read)
//   mask_iou_kernel    : intersections as a 1-bit GEMM on the tensor cores (mma.sync m16n8k256 .and.popc, int32 accumulators),
//                        then the reference's single fp32 division
//   match_iou_kernel   : the matching rule of match_kernel (match_rule.cuh) on that IoU matrix
// Every quantity before the division is an integer count, so the results are bit-exact.  Compiled with -fmad=false; the
// resize weights follow mask_upsample_kernel (post_kernels.cu) with explicit _rn intrinsics.
#include "../../include/y5b200.h"
#include "common.cuh"
#include "host_util.h"
#include "match_rule.cuh"

namespace y5 {

constexpr int kMaskMaxPixels = 1 << 23;  // 2*H*W <= 2^24: the reference's fp32 pixel sums are exact up to here
constexpr int kPackThreads = 256;
constexpr int kIouWarps = 8;              // a block covers 8 * kIouWarps predictions of one image

__device__ __forceinline__ float load_mask(const void* p, long long i, int dtype) {
    if (dtype == Y5_U8) return static_cast<float>(static_cast<const uint8_t*>(p)[i]);
    if (dtype == Y5_F32) return static_cast<const float*>(p)[i];
    return unpack1(static_cast<const uint16_t*>(p)[i], dtype == Y5_BF16);
}

// image of target i, or -1 when its image column is not an integer in [0, batch) (`targets[:, 0] == si` never holds)
__device__ __forceinline__ int target_image(const float* timg, int ts, int i, int batch) {
    const float f = timg[static_cast<long long>(i) * ts];
    if (!(f >= 0.f && f < static_cast<float>(batch))) return -1;
    const int b = static_cast<int>(f);
    return static_cast<float>(b) == f ? b : -1;
}

// One block.  label_index = [off (batch+1)][row_target (nt)][row_img (nt)]: image b's labels are rows off[b]..off[b+1]-1 in
// target order; targets of no image follow off[batch] with row_img -1.  One warp per image, ballots over the targets.
__global__ void mask_labels_kernel(const float* __restrict__ timg, int ts, int nt, int batch, int* __restrict__ label_index) {
    int* off = label_index;
    int* row_target = off + batch + 1;
    int* row_img = row_target + nt;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
    for (int b = warp; b < batch; b += nw) {
        int c = 0;
        for (int i0 = 0; i0 < nt; i0 += 32) {
            const int i = i0 + lane;
            c += __popc(__ballot_sync(0xffffffffu, i < nt && target_image(timg, ts, i, batch) == b));
        }
        if (lane == 0) off[b + 1] = c;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        off[0] = 0;
        for (int b = 0; b < batch; ++b) off[b + 1] += off[b];
    }
    __syncthreads();
    for (int b = warp; b <= batch; b += nw) {
        const int want = b == batch ? -1 : b;
        int r = off[b];
        for (int i0 = 0; i0 < nt; i0 += 32) {
            const int i = i0 + lane;
            const bool mine = i < nt && target_image(timg, ts, i, batch) == want;
            const unsigned m = __ballot_sync(0xffffffffu, mine);
            if (mine) {
                const int g = r + __popc(m & ((1u << lane) - 1u));
                row_target[g] = i;
                row_img[g] = want;
            }
            r += __popc(m);
        }
    }
}

// One block per bit row.  Pixel p of the (oh, ow) mask is bit p%32 of word p/32; words >= ceil(oh*ow/32) are zero.
//   OVERLAP 0: the row is source plane `plane`, its values taken as they are (non-{0,1} values counted when not resized)
//   OVERLAP 1: the row is the indicator `plane == value` (label k of an overlap index image is value k+1)
//   RESIZE   : the per-row values are interpolated bilinearly (align_corners=False) to (oh, ow) and kept where > 0.5
template <int OVERLAP, int RESIZE>
__global__ void __launch_bounds__(kPackThreads) mask_pack_kernel(const void* __restrict__ src, int dtype, int sh, int sw, int oh, int ow,
                                                                  const int* __restrict__ label_index, int batch, int n_rows, int words,
                                                                  uint32_t* __restrict__ bits, int* __restrict__ popcount,
                                                                  int* __restrict__ nonbinary) {
    __shared__ int s_red[2][kPackThreads / 32];
    const int row = blockIdx.x;
    long long plane = OVERLAP ? 0 : row;
    float value = static_cast<float>(row + 1);
    bool active = true;
    if (label_index) {
        const int img = label_index[batch + 1 + n_rows + row];
        if (OVERLAP) {
            plane = img;
            value = static_cast<float>(row - (img >= 0 ? label_index[img] : 0) + 1);
            active = img >= 0;
        } else {
            plane = label_index[batch + 1 + row];
        }
    }
    const long long src_hw = static_cast<long long>(sh) * sw;
    const long long base = plane * src_hw;
    const int hw = oh * ow;
    const float scale_y = __fdiv_rn(static_cast<float>(sh), static_cast<float>(oh));
    const float scale_x = __fdiv_rn(static_cast<float>(sw), static_cast<float>(ow));
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    int pop = 0, bad = 0;
    for (int w0 = warp * 32; w0 < words; w0 += kPackThreads) {
        uint32_t mine = 0;
        for (int j = 0; j < 32; ++j) {
            const int p = (w0 + j) * 32 + lane;
            bool on = false;
            if (active && p < hw) {
                if (RESIZE) {
                    const int ox = p % ow, oy = p / ow;
                    const float srcy = fmaxf(__fsub_rn(__fmul_rn(__fadd_rn(static_cast<float>(oy), 0.5f), scale_y), 0.5f), 0.f);
                    const float srcx = fmaxf(__fsub_rn(__fmul_rn(__fadd_rn(static_cast<float>(ox), 0.5f), scale_x), 0.5f), 0.f);
                    const int y0 = min(static_cast<int>(srcy), sh - 1), x0 = min(static_cast<int>(srcx), sw - 1);
                    const int y1 = min(y0 + 1, sh - 1), x1 = min(x0 + 1, sw - 1);
                    const float ly = __fsub_rn(srcy, static_cast<float>(y0)), lx = __fsub_rn(srcx, static_cast<float>(x0));
                    float v00 = load_mask(src, base + static_cast<long long>(y0) * sw + x0, dtype);
                    float v01 = load_mask(src, base + static_cast<long long>(y0) * sw + x1, dtype);
                    float v10 = load_mask(src, base + static_cast<long long>(y1) * sw + x0, dtype);
                    float v11 = load_mask(src, base + static_cast<long long>(y1) * sw + x1, dtype);
                    if (OVERLAP) {  // the expanded per-label 0/1 masks are what the reference interpolates
                        v00 = v00 == value ? 1.f : 0.f;
                        v01 = v01 == value ? 1.f : 0.f;
                        v10 = v10 == value ? 1.f : 0.f;
                        v11 = v11 == value ? 1.f : 0.f;
                    }
                    const float hx = __fsub_rn(1.0f, lx), hy = __fsub_rn(1.0f, ly);
                    const float top = __fadd_rn(__fmul_rn(v00, hx), __fmul_rn(v01, lx));
                    const float bot = __fadd_rn(__fmul_rn(v10, hx), __fmul_rn(v11, lx));
                    on = __fadd_rn(__fmul_rn(top, hy), __fmul_rn(bot, ly)) > 0.5f;  // gt_(0.5): exactly 0.5 stays 0
                } else {
                    const float v = load_mask(src, base + p, dtype);
                    if (OVERLAP) {
                        on = v == value;
                    } else {
                        on = v != 0.f;
                        bad += (v != 0.f && v != 1.f) ? 1 : 0;
                    }
                }
            }
            const uint32_t word = __ballot_sync(0xffffffffu, on);
            if (lane == j) mine = word;
        }
        if (w0 + lane < words) {
            bits[static_cast<long long>(row) * words + w0 + lane] = mine;
            pop += __popc(mine);
        }
    }
    for (int o = 16; o > 0; o >>= 1) {
        pop += __shfl_xor_sync(0xffffffffu, pop, o);
        bad += __shfl_xor_sync(0xffffffffu, bad, o);
    }
    if (lane == 0) { s_red[0][warp] = pop; s_red[1][warp] = bad; }
    __syncthreads();
    if (threadIdx.x == 0) {
        int tp = 0, tb = 0;
        for (int i = 0; i < kPackThreads / 32; ++i) { tp += s_red[0][i]; tb += s_red[1][i]; }
        popcount[row] = tp;
        if (tb) atomicAdd(nonbinary, tb);
    }
}

// D(16x8, s32) += popc(A(16x256, b1) AND B(256x8, b1))
__device__ __forceinline__ void bmma_and_popc(int (&c)[4], const uint32_t (&a)[4], const uint32_t (&b)[2]) {
    asm volatile(
        "mma.sync.aligned.m16n8k256.row.col.s32.b1.b1.s32.and.popc {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
        : "+r"(c[0]), "+r"(c[1]), "+r"(c[2]), "+r"(c[3])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
}

// grid (ceil(rows_per_image / (8 * kIouWarps)), n_img).  Image img0 + y: labels l0..l0+nl-1 (label_index offsets, or all n_gt
// rows of a single image), predictions 0..n-1 at pred rows y*rows_per_image + d.  Each warp owns 8 predictions and walks the
// label rows 16 at a time; K advances 256 pixels per mma.  Fragment layout (PTX ISA, m16n8k256 .b1): thread (g = lane/4,
// t = lane%4) holds A rows g, g+8 and B column g at words t and t+4 of the 8-word K tile; D rows g, g+8, columns 2t, 2t+1.
// iou[(l0 + r) * rows_per_image + d] = inter / (|gt_r| + |pred_d| - inter + eps), the reference's mask_iou.
__global__ void __launch_bounds__(kIouWarps * 32) mask_iou_kernel(const uint32_t* __restrict__ gt, const int* __restrict__ gt_pop,
                                                                   const int* __restrict__ label_index, int n_gt,
                                                                   const uint32_t* __restrict__ pred, const int* __restrict__ pred_pop,
                                                                   const int* __restrict__ count, int img0, int rows_per_image, int words,
                                                                   float eps, float* __restrict__ iou) {
    const int y = blockIdx.y, b = img0 + y;
    int l0 = 0, nl = n_gt;
    if (label_index) {
        l0 = label_index[b];
        nl = label_index[b + 1] - l0;
    }
    const int n = count ? min(count[b], rows_per_image) : rows_per_image;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
    const int d0 = (blockIdx.x * kIouWarps + warp) * 8;
    if (d0 >= n || nl <= 0) return;
    const long long prow = static_cast<long long>(y) * rows_per_image;
    const uint32_t* pb = pred + (prow + min(d0 + g, n - 1)) * words;
    for (int m0 = 0; m0 < nl; m0 += 16) {
        const uint32_t* pa0 = gt + static_cast<long long>(l0 + min(m0 + g, nl - 1)) * words;
        const uint32_t* pa1 = gt + static_cast<long long>(l0 + min(m0 + g + 8, nl - 1)) * words;
        int c[4] = {0, 0, 0, 0};
#pragma unroll 4
        for (int k = 0; k < words; k += 8) {
            const uint32_t a[4] = {__ldg(pa0 + k + t), __ldg(pa1 + k + t), __ldg(pa0 + k + 4 + t), __ldg(pa1 + k + 4 + t)};
            const uint32_t bb[2] = {__ldg(pb + k + t), __ldg(pb + k + 4 + t)};
            bmma_and_popc(c, a, bb);
        }
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            const int r = m0 + g + (q >> 1) * 8, d = d0 + 2 * t + (q & 1);
            if (r < nl && d < n) {
                const float inter = static_cast<float>(c[q]);
                const float uni = __fsub_rn(__fadd_rn(static_cast<float>(gt_pop[l0 + r]), static_cast<float>(pred_pop[prow + d])), inter);
                iou[static_cast<long long>(l0 + r) * rows_per_image + d] = __fdiv_rn(inter, __fadd_rn(uni, eps));
            }
        }
    }
}

// One block per image: detection d's best label = the same-class label of its image with the highest mask IoU (first in
// target order on ties), then match_assign.  Labels: label_index blocks, or all nt rows for a single image.
__global__ void match_iou_kernel(const float* __restrict__ det, long long img_stride, int row_stride, const int32_t* __restrict__ count,
                                 int max_det, const float* __restrict__ label_cls, int cls_stride, const int* __restrict__ label_index,
                                 int batch, int nt, const float* __restrict__ iou, const float* __restrict__ iouv, int niou,
                                 uint8_t* __restrict__ correct) {
    __shared__ int s_best[kMatchMaxDet];
    __shared__ float s_iou[kMatchMaxDet];
    const int b = blockIdx.x;
    const int n = min(count ? count[b] : max_det, max_det);
    const int l0 = label_index && nt > 0 ? label_index[b] : 0;
    const int l1 = label_index && nt > 0 ? min(label_index[b + 1], nt) : nt;
    const float* dbase = det + static_cast<long long>(b) * img_stride;
    for (int d = threadIdx.x; d < n; d += blockDim.x) {
        const float dcls = dbase[static_cast<long long>(d) * row_stride + 5];
        int best = -1;
        float best_iou = -1.0f;
        for (int l = l0; l < l1; ++l) {
            const int tg = label_index ? label_index[batch + 1 + l] : l;
            if (label_cls[static_cast<long long>(tg) * cls_stride] != dcls) continue;
            const float v = iou[static_cast<long long>(l) * max_det + d];
            if (v > best_iou) { best_iou = v; best = l; }
        }
        s_best[d] = best;
        s_iou[d] = best_iou;
    }
    __syncthreads();
    match_assign(s_best, s_iou, n, max_det, iouv, niou, correct + static_cast<long long>(b) * max_det * niou);
}

}  // namespace y5

using namespace y5;

extern "C" Y5_API int32_t y5_mask_row_words(int32_t h, int32_t w) {
    if (h <= 0 || w <= 0) return set_error(Y5_E_INVALID, "mask_row_words: bad shape %dx%d", h, w);
    if (static_cast<long long>(h) * w > kMaskMaxPixels)
        return set_error(Y5_E_UNSUPPORTED, "mask_row_words: %dx%d masks exceed 2^23 pixels (fp32 pixel counts stop being exact)", h, w);
    return static_cast<int32_t>((static_cast<long long>(h) * w + 255) / 256 * 8);
}

extern "C" Y5_API int y5_mask_pack(const void* src, int32_t src_dtype, int32_t src_h, int32_t src_w, int32_t overlap, const float* target_img,
                                   int32_t target_stride, int32_t batch, int32_t n_rows, int32_t out_h, int32_t out_w, int32_t* label_index,
                                   uint32_t* bits, int32_t* popcount, int32_t* nonbinary, void* stream) {
    if (n_rows < 0 || src_h <= 0 || src_w <= 0 || out_h <= 0 || out_w <= 0) return set_error(Y5_E_INVALID, "mask_pack: bad shape");
    const int words = y5_mask_row_words(out_h, out_w);
    if (words < 0) return words;
    if (static_cast<long long>(src_h) * src_w > (1LL << 30)) return set_error(Y5_E_UNSUPPORTED, "mask_pack: %dx%d source", src_h, src_w);
    if (src_dtype != Y5_U8 && src_dtype != Y5_F32 && src_dtype != Y5_F16 && src_dtype != Y5_BF16)
        return set_error(Y5_E_UNSUPPORTED, "mask_pack: source dtype %d", src_dtype);
    if (target_img && !label_index) return set_error(Y5_E_INVALID, "mask_pack: targets need label_index");
    if (label_index && (batch <= 0 || (n_rows > 0 && (!target_img || target_stride <= 0))))
        return set_error(Y5_E_INVALID, "mask_pack: label_index needs batch > 0 and, with targets, their image column and stride");
    if (n_rows == 0 && !label_index) return 0;
    if (n_rows > 0 && (!src || !bits || !popcount || !nonbinary)) return set_error(Y5_E_INVALID, "mask_pack: null pointer");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const int* li = nullptr;
    if (label_index) {  // also with no targets at all: every image then owns an empty label block
        if (int e = launch("mask_pack", mask_labels_kernel, {1, 1024, 0, st}, target_img, target_stride, n_rows, batch, label_index)) return e;
        li = label_index;
        if (n_rows == 0) return 0;
    }
    const bool resize = src_h != out_h || src_w != out_w;
    const int ov = overlap != 0;
    auto* kernel = ov ? (resize ? mask_pack_kernel<1, 1> : mask_pack_kernel<1, 0>) : (resize ? mask_pack_kernel<0, 1> : mask_pack_kernel<0, 0>);
    return launch("mask_pack", kernel, {n_rows, kPackThreads, 0, st}, src, src_dtype, src_h, src_w, out_h, out_w, li, batch, n_rows, words, bits,
                  popcount, nonbinary);
}

extern "C" Y5_API int y5_mask_iou(const uint32_t* gt_bits, const int32_t* gt_pop, const int32_t* label_index, int32_t n_gt, const uint32_t* pred_bits,
                                  const int32_t* pred_pop, const int32_t* count, int32_t img0, int32_t n_img, int32_t rows_per_image, int32_t words,
                                  float eps, float* iou, void* stream) {
    if (n_img == 0 || rows_per_image == 0) return 0;
    if (n_img < 0 || rows_per_image < 0 || img0 < 0 || n_gt < 0 || words <= 0 || (words & 7)) return set_error(Y5_E_INVALID, "mask_iou: bad shape");
    if (words > kMaskMaxPixels / 32) return set_error(Y5_E_UNSUPPORTED, "mask_iou: %d words per row exceed 2^23 pixels", words);
    if (!label_index && (n_img != 1 || count)) return set_error(Y5_E_INVALID, "mask_iou: without label_index there is one image and no count");
    if (!label_index && n_gt == 0) return 0;
    if (!gt_bits || !gt_pop || !pred_bits || !pred_pop || !iou) return set_error(Y5_E_INVALID, "mask_iou: null pointer");
    const dim3 grid((rows_per_image + 8 * kIouWarps - 1) / (8 * kIouWarps), n_img);
    return launch("mask_iou", mask_iou_kernel, {grid, kIouWarps * 32, 0, static_cast<cudaStream_t>(stream)}, gt_bits, gt_pop, label_index, n_gt,
                  pred_bits, pred_pop, count, img0, rows_per_image, words, eps, iou);
}

extern "C" Y5_API int y5_mask_match_batch(const float* det, int64_t img_stride, int32_t row_stride, const int32_t* count, int32_t batch,
                                          int32_t max_det, const float* label_cls, int32_t cls_stride, const int32_t* label_index, int32_t nt,
                                          const float* iou, const float* iouv, int32_t niou, uint8_t* correct, void* stream) {
    if (batch <= 0 || max_det <= 0) return 0;
    if (!det || !iouv || !correct || niou <= 0 || row_stride < 6 || nt < 0 || cls_stride <= 0 || (nt > 0 && (!label_cls || !iou)))
        return set_error(Y5_E_INVALID, "mask_match_batch: bad argument");
    if (!label_index && batch != 1) return set_error(Y5_E_INVALID, "mask_match_batch: more than one image needs label_index");
    if (max_det > kMatchMaxDet) return set_error(Y5_E_UNSUPPORTED, "mask_match_batch: max_det %d > %d", max_det, kMatchMaxDet);
    return launch("mask_match_batch", match_iou_kernel, {batch, 256, 0, static_cast<cudaStream_t>(stream)}, det, img_stride, row_stride, count,
                  max_det, label_cls, cls_stride, label_index, batch, nt, iou, iouv, niou, correct);
}
