// Segmentation training augmentation (reference utils/segment/dataloaders.py:130-301, utils/segment/augmentations.py:26-91)
// on the device: the segment path of random_perspective, the label filter and the polygon masks, exact with the
// reference's numpy / OpenCV arithmetic (oracle/seg_aug_ref.py).  The image itself goes through aug_kernels.cu.
//   seg_warp_kernel    : one block per label.  xyn2xy (float32), load_mosaic's clip, resample_segments(n=1000) (float64
//                        np.linspace + np.interp), `xy @ M.T` as OpenBLAS forms it, segment2box, box_candidates
//                        (area_thr 0.01), xyxy2xywhn + flips; the polygon as the int32 vertices polygon2mask casts it to.
//   seg_raster_kernel  : one block per (kept label, mask row): cv2.fillPoly(zeros(s, s), [poly], 1) rows, then
//                        cv2.resize(INTER_LINEAR) to s / r (r = 4 reads source rows and columns 4k+1, 4k+2), and the area.
//   seg_order_kernel   : one block per image: stable compaction of the kept labels, the overlap order (argsort(-areas) on
//                        uint64, ties by label order) and the target rows in that order.
//   seg_compose_kernel : the batch's mask tensor: overlap planes (clip(v + m_i * (i + 1), 0, i + 1) in uint8 or int32) or
//                        one plane per label, with the flips.
// Compiled with -fmad=false; every rounding point of the reference is an explicit _rn intrinsic.
#include <math.h>
#include <stdint.h>

#include "../../include/y5b200.h"
#include "common.cuh"
#include "host_util.h"

namespace y5 {

constexpr int kSegThreads = 256;
constexpr int kSegOrderThreads = 256;
constexpr int kXYShift = 16;  // cv2 drawing's fixed point

// x' = x*M0 + y*M1 + M2 as OpenBLAS's dgemm forms `xy @ M.T` (K = 3): product, fma, add (same at 4 and 1000 rows)
__device__ __forceinline__ double seg_affine(const double* Mr, double x, double y) {
    return __dadd_rn(__fma_rn(y, Mr[1], __dmul_rn(x, Mr[0])), Mr[2]);
}

// np.interp(x, arange(L), d) at x = np.linspace(0, L - 1, 1000)[i], for the closed polygon's float32 values d
__device__ __forceinline__ double seg_interp(const float* d, int L, int i, double step) {
    if (i == Y5_SEG_POINTS - 1) return static_cast<double>(d[L - 1]);
    const double x = __dmul_rn(static_cast<double>(i), step);
    const int j = static_cast<int>(floor(x));
    if (j >= L - 1) return static_cast<double>(d[L - 1]);
    const double dj = static_cast<double>(d[j]);
    if (x == static_cast<double>(j)) return dj;
    const double slope = __dsub_rn(static_cast<double>(d[j + 1]), dj);
    return __dadd_rn(__dmul_rn(slope, __dsub_rn(x, static_cast<double>(j))), dj);
}

__device__ __forceinline__ double warp_min(double v) {
    for (int o = 16; o; o >>= 1) v = fmin(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}

__device__ __forceinline__ double warp_max(double v) {
    for (int o = 16; o; o >>= 1) v = fmax(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}

// one block per label: polygon -> 1000 int32 vertices, segment box, keep flag and the output row
__global__ void __launch_bounds__(kSegThreads) seg_warp_kernel(const y5_aug_image* __restrict__ table, int n_images,
                                                              const y5_aug_label* __restrict__ labels,
                                                              const y5_aug_segment* __restrict__ segments,
                                                              const float* __restrict__ points, int max_points, int out_h, int out_w,
                                                              int32_t* __restrict__ verts, float* __restrict__ rows,
                                                              int32_t* __restrict__ keep) {
    extern __shared__ float s_xy[];  // 2 * (n_points + 1): x values, then y values, of the closed polygon
    __shared__ double s_red[4][kSegThreads / 32];
    __shared__ int s_any[kSegThreads / 32];
    const int li = blockIdx.x, tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    const y5_aug_label L = labels[li];
    const y5_aug_segment S = segments[li];
    const bool valid = L.image >= 0 && L.image < n_images && L.mosaic >= 0 && L.mosaic < table[L.image].n_mosaic &&
                       S.n_points >= 1 && S.n_points <= max_points;
    if (!valid) {  // a row naming no image / mosaic, or an empty polygon, is dropped
        if (tid == 0) keep[li] = 0;
        return;
    }
    const y5_aug_image& im = table[L.image];
    const int n = S.n_points, np1 = n + 1;
    float* sx = s_xy;
    float* sy = s_xy + np1;
    // xyn2xy in float32 (w * x + padw with w, padw already float32), then load_mosaic's clip to [0, 2s]
    for (int k = tid; k < n; k += blockDim.x) {
        const float* p = points + 2 * (static_cast<long long>(S.point_offset) + k);
        float x = __fadd_rn(__fmul_rn(L.tile_w, p[0]), L.pad_w);
        float y = __fadd_rn(__fmul_rn(L.tile_h, p[1]), L.pad_h);
        if (L.flags & Y5_AUG_CLIP) {
            x = fminf(fmaxf(x, 0.f), im.clip_max);
            y = fminf(fmaxf(y, 0.f), im.clip_max);
        }
        sx[k] = x;
        sy[k] = y;
        if (k == 0) {  // resample_segments closes the polygon with its first point
            sx[n] = x;
            sy[n] = y;
        }
    }
    __syncthreads();
    const double step = __ddiv_rn(static_cast<double>(np1 - 1), static_cast<double>(Y5_SEG_POINTS - 1));
    const double* M0 = im.m[L.mosaic];
    const double* M1 = im.m[L.mosaic] + 3;
    const double W = static_cast<double>(out_w), H = static_cast<double>(out_h);
    double bx1 = INFINITY, by1 = INFINITY, bx2 = -INFINITY, by2 = -INFINITY;
    int any = 0;
    int32_t* v = verts + static_cast<long long>(li) * Y5_SEG_POINTS * 2;
    for (int i = tid; i < Y5_SEG_POINTS; i += blockDim.x) {
        const double x = seg_interp(sx, np1, i, step), y = seg_interp(sy, np1, i, step);
        const double px = seg_affine(M0, x, y), py = seg_affine(M1, x, y);
        if (px >= 0.0 && py >= 0.0 && px <= W && py <= H) {  // segment2box's inside filter
            bx1 = fmin(bx1, px); bx2 = fmax(bx2, px); by1 = fmin(by1, py); by2 = fmax(by2, py);
            any = 1;
        }
        v[2 * i] = __double2int_rz(px);  // np.asarray(polygons, dtype=np.int32): truncation toward zero
        v[2 * i + 1] = __double2int_rz(py);
    }
    bx1 = warp_min(bx1); by1 = warp_min(by1); bx2 = warp_max(bx2); by2 = warp_max(by2);
    any = __any_sync(0xffffffffu, any);
    if (lane == 0) {
        s_red[0][wid] = bx1; s_red[1][wid] = by1; s_red[2][wid] = bx2; s_red[3][wid] = by2;
        s_any[wid] = any;
    }
    __syncthreads();
    if (tid != 0) return;
    for (int w = 1; w < kSegThreads / 32; ++w) {
        bx1 = fmin(bx1, s_red[0][w]); by1 = fmin(by1, s_red[1][w]);
        bx2 = fmax(bx2, s_red[2][w]); by2 = fmax(by2, s_red[3][w]);
        any |= s_any[w];
    }
    if (!any) bx1 = by1 = bx2 = by2 = 0.0;  // segment2box: zeros when no point is inside
    // box1 = the label's xywhn2xyxy box (clipped in a mosaic) times the scale draw, float32
    const float hw = __fdiv_rn(L.w, 2.0f), hh = __fdiv_rn(L.h, 2.0f);
    float x1 = __fadd_rn(__fmul_rn(L.tile_w, __fsub_rn(L.x, hw)), L.pad_w);
    float y1 = __fadd_rn(__fmul_rn(L.tile_h, __fsub_rn(L.y, hh)), L.pad_h);
    float x2 = __fadd_rn(__fmul_rn(L.tile_w, __fadd_rn(L.x, hw)), L.pad_w);
    float y2 = __fadd_rn(__fmul_rn(L.tile_h, __fadd_rn(L.y, hh)), L.pad_h);
    if (L.flags & Y5_AUG_CLIP) {
        x1 = fminf(fmaxf(x1, 0.f), im.clip_max); y1 = fminf(fmaxf(y1, 0.f), im.clip_max);
        x2 = fminf(fmaxf(x2, 0.f), im.clip_max); y2 = fminf(fmaxf(y2, 0.f), im.clip_max);
    }
    const float s = im.scale[L.mosaic];
    const float w1 = __fsub_rn(__fmul_rn(x2, s), __fmul_rn(x1, s)), h1 = __fsub_rn(__fmul_rn(y2, s), __fmul_rn(y1, s));
    const double w2 = __dsub_rn(bx2, bx1), h2 = __dsub_rn(by2, by1);
    const double ar = fmax(__ddiv_rn(w2, __dadd_rn(h2, 1e-16)), __ddiv_rn(h2, __dadd_rn(w2, 1e-16)));
    const float area1 = __fadd_rn(__fmul_rn(w1, h1), static_cast<float>(1e-16));
    keep[li] = w2 > 2.0 && h2 > 2.0 && __ddiv_rn(__dmul_rn(w2, h2), static_cast<double>(area1)) > 0.01 && ar < 100.0;
    // targets[:, 1:5] = new (float64 -> float32), xyxy2xywhn(clip=True, eps=1e-3) in float32, then the flips
    float b0 = __double2float_rn(bx1), b1 = __double2float_rn(by1), b2 = __double2float_rn(bx2), b3 = __double2float_rn(by2);
    const float cw = __double2float_rn(__dsub_rn(W, 1e-3)), ch = __double2float_rn(__dsub_rn(H, 1e-3));
    b0 = fminf(fmaxf(b0, 0.f), cw); b2 = fminf(fmaxf(b2, 0.f), cw);
    b1 = fminf(fmaxf(b1, 0.f), ch); b3 = fminf(fmaxf(b3, 0.f), ch);
    const float Wf = static_cast<float>(out_w), Hf = static_cast<float>(out_h);
    float xc = __fdiv_rn(__fdiv_rn(__fadd_rn(b0, b2), 2.0f), Wf);
    float yc = __fdiv_rn(__fdiv_rn(__fadd_rn(b1, b3), 2.0f), Hf);
    if (im.flipud) yc = __fsub_rn(1.0f, yc);
    if (im.fliplr) xc = __fsub_rn(1.0f, xc);
    float* row = rows + static_cast<long long>(li) * 6;
    row[0] = static_cast<float>(L.image);
    row[1] = L.cls;
    row[2] = xc;
    row[3] = yc;
    row[4] = __fdiv_rn(__fsub_rn(b2, b0), Wf);
    row[5] = __fdiv_rn(__fsub_rn(b3, b1), Hf);
}

// cv2.clipLine on int64 points against [0, w) x [0, h) (the double-precision intercepts truncated toward zero).  The
// points are updated even when the line misses the image, as cv2 does; returns whether the clipped line is inside.
__device__ bool clip_line(long long w, long long h, long long& x1, long long& y1, long long& x2, long long& y2) {
    const long long right = w - 1, bottom = h - 1;
    int c1 = (x1 < 0) + (x1 > right) * 2 + (y1 < 0) * 4 + (y1 > bottom) * 8;
    int c2 = (x2 < 0) + (x2 > right) * 2 + (y2 < 0) * 4 + (y2 > bottom) * 8;
    if ((c1 & c2) == 0 && (c1 | c2) != 0) {
        long long a;
        if (c1 & 12) {
            a = c1 < 8 ? 0 : bottom;
            x1 += static_cast<long long>(__ddiv_rn(__dmul_rn(static_cast<double>(a - y1), static_cast<double>(x2 - x1)), static_cast<double>(y2 - y1)));
            y1 = a;
            c1 = (x1 < 0) + (x1 > right) * 2;
        }
        if (c2 & 12) {
            a = c2 < 8 ? 0 : bottom;
            x2 += static_cast<long long>(__ddiv_rn(__dmul_rn(static_cast<double>(a - y2), static_cast<double>(x2 - x1)), static_cast<double>(y2 - y1)));
            y2 = a;
            c2 = (x2 < 0) + (x2 > right) * 2;
        }
        if ((c1 & c2) == 0 && (c1 | c2) != 0) {
            if (c1) {
                a = c1 == 1 ? 0 : right;
                y1 += static_cast<long long>(__ddiv_rn(__dmul_rn(static_cast<double>(a - x1), static_cast<double>(y2 - y1)), static_cast<double>(x2 - x1)));
                x1 = a;
                c1 = 0;
            }
            if (c2) {
                a = c2 == 1 ? 0 : right;
                y2 += static_cast<long long>(__ddiv_rn(__dmul_rn(static_cast<double>(a - x2), static_cast<double>(y2 - y1)), static_cast<double>(x2 - x1)));
                x2 = a;
                c2 = 0;
            }
        }
    }
    return (c1 | c2) == 0;
}

__device__ __forceinline__ long long ceil_div(long long a, long long b) {  // b > 0
    return a >= 0 ? (a + b - 1) / b : -((-a) / b);
}

// one source row's pixel set: `mark` (outline pixels and spans' exact-integer ends) and `par` (parity of the span
// crossings whose floor is each column), `below` (parity of crossings left of column 0)
struct RowAcc {
    uint8_t* mark;
    int* par;
    int* below;
};

// polygon edge e (from vertex e-1 to vertex e) at source row y: its 8-connected outline pixels (cv2's Line, clipped,
// drawn left to right) and its fill crossing (cv2's CollectPolyEdges / FillEdgeCollection in 16.16 fixed point)
__device__ void edge_row(const int32_t* v, int n, int e, int y, int w, int h, RowAcc acc) {
    const int p = e == 0 ? n - 1 : e - 1;
    const long long ax = v[2 * p], ay = v[2 * p + 1], bx = v[2 * e], by = v[2 * e + 1];
    long long x1 = ax, y1 = ay, x2 = bx, y2 = by;
    const bool outside = ax < 0 || ax >= w || bx < 0 || bx >= w || ay < 0 || ay >= h || by < 0 || by >= h;
    const bool in = !outside || clip_line(w, h, x1, y1, x2, y2);
    // outline: Bresenham with err = dx - 2dy; after n major steps the minor offset is floor((2 dy n + dx - 1) / (2 dx))
    if (in) {
        long long lx1 = x1, ly1 = y1, lx2 = x2, ly2 = y2;
        if (lx2 < lx1) {
            const long long tx = lx1, ty = ly1;
            lx1 = lx2; ly1 = ly2; lx2 = tx; ly2 = ty;
        }
        const long long dx = lx2 - lx1, dy = ly2 - ly1, ady = dy < 0 ? -dy : dy;
        const long long k = dy < 0 ? ly1 - y : y - ly1;  // minor (or major) steps to reach row y
        if (k >= 0 && k <= ady) {
            if (ady > dx) {  // y-major: one pixel per row
                const long long xx = lx1 + (2 * dx * k + ady - 1) / (2 * ady);
                if (xx >= 0 && xx < w) acc.mark[xx] = 1;
            } else {
                long long lo = 0, hi = dx;
                if (ady > 0) {
                    lo = max(lo, ceil_div(2 * dx * k - dx + 1, 2 * ady));
                    hi = min(hi, ceil_div(2 * dx * k + dx + 1, 2 * ady) - 1);
                }
                for (long long t = max(lo, -lx1); t <= hi && lx1 + t < w; ++t) acc.mark[lx1 + t] = 1;
            }
        }
    }
    // fill: edges with y0 <= y < y1 (horizontal edges skipped); an edge touching the outside starts from its clipped x
    if (ay == by) return;
    long long p0x = (ax << kXYShift), p0y = ay, p1x = (bx << kXYShift), p1y = by;
    if (outside) {
        p0x = x1 << kXYShift;
        p1x = x2 << kXYShift;
        if (y1 != y2) {
            p0y = y1;
            p1y = y2;
        }
    }
    const long long dxe = (p1x - p0x) / (p1y - p0y);  // C division: truncation toward zero
    long long ey0, ey1, ex;
    if (ay < by) {
        ey0 = ay; ey1 = by; ex = p0x + (ey0 - p0y) * dxe;
    } else {
        ey0 = by; ey1 = ay; ex = p1x + (ey0 - p1y) * dxe;
    }
    if (y < ey0 || y >= ey1) return;
    const long long x = ex + (y - ey0) * dxe;
    const long long F = x >> kXYShift;  // a span covers columns ceil(left) .. floor(right)
    if (F < 0) {
        atomicXor(acc.below, 1);
    } else if (F < w) {
        atomicXor(acc.par + F, 1);
        if ((x & ((1LL << kXYShift) - 1)) == 0) acc.mark[F] = 1;  // an integer left end is inside its own span
    }
}

// column c of the row is set iff it is on the outline, is an integer span end, or an odd number of crossings lie left
// of it (the sorted crossings pair up into spans [ceil(x_2k), floor(x_2k+1)])
__device__ void row_scan(int w, RowAcc acc, int* s_chunk) {
    const int tid = threadIdx.x, nt = blockDim.x;
    const int per = (w + nt - 1) / nt;
    const int c0 = min(tid * per, w), c1 = min(c0 + per, w);
    int x = 0;
    for (int c = c0; c < c1; ++c) x ^= acc.par[c];
    s_chunk[tid] = x;
    __syncthreads();
    for (int o = 1; o < nt; o <<= 1) {  // inclusive xor scan over the chunks
        const int t = tid >= o ? s_chunk[tid - o] : 0;
        __syncthreads();
        s_chunk[tid] ^= t;
        __syncthreads();
    }
    int run = (tid ? s_chunk[tid - 1] : 0) ^ *acc.below;
    for (int c = c0; c < c1; ++c) {
        const int here = acc.par[c];
        acc.par[c] = acc.mark[c] | run;  // becomes the pixel value
        run ^= here;
    }
    __syncthreads();
}

// grid (mask rows, labels): fillPoly + resize of one mask row of one kept label; masks[label] is (h / r, w / r) uint8
__global__ void __launch_bounds__(kSegThreads) seg_raster_kernel(const int32_t* __restrict__ verts, int n_verts, const int32_t* __restrict__ keep,
                                                                int out_h, int out_w, int ratio, uint8_t* __restrict__ masks,
                                                                int32_t* __restrict__ areas) {
    extern __shared__ int s_dyn[];
    __shared__ int s_chunk[kSegThreads];
    __shared__ int s_below[2];
    __shared__ int s_sum;
    const int li = blockIdx.y, orow = blockIdx.x;
    if (!keep[li]) return;
    const int w = out_w, h = out_h, mw = out_w / ratio;
    const int nsrc = ratio == 1 ? 1 : 2;
    int* par = s_dyn;                                               // nsrc * w
    uint8_t* mark = reinterpret_cast<uint8_t*>(s_dyn + nsrc * w);  // nsrc * w
    for (int i = threadIdx.x; i < nsrc * w; i += blockDim.x) {
        par[i] = 0;
        mark[i] = 0;
    }
    if (threadIdx.x < 2) s_below[threadIdx.x] = 0;
    if (threadIdx.x == 0) s_sum = 0;
    __syncthreads();
    const int32_t* v = verts + static_cast<long long>(li) * n_verts * 2;
    for (int r = 0; r < nsrc; ++r) {
        const int y = ratio == 1 ? orow : orow * ratio + 1 + r;
        const RowAcc acc{mark + r * w, par + r * w, s_below + r};
        for (int e = threadIdx.x; e < n_verts; e += blockDim.x) edge_row(v, n_verts, e, y, w, h, acc);
    }
    __syncthreads();
    for (int r = 0; r < nsrc; ++r) row_scan(w, RowAcc{mark + r * w, par + r * w, s_below + r}, s_chunk);
    // cv2.resize INTER_LINEAR, uint8: at r = 4 every output pixel weighs source rows/cols 4k+1, 4k+2 by 1/2 each,
    // (sum * 2^20 + 2^21) >> 22 of 0/1 values is 1 iff at least two of the four are set
    uint8_t* out = masks + (static_cast<long long>(li) * (out_h / ratio) + orow) * mw;
    int cnt = 0;
    for (int j = threadIdx.x; j < mw; j += blockDim.x) {
        int val;
        if (ratio == 1) {
            val = par[j];
        } else {
            const int c = j * ratio + 1;
            val = (par[c] + par[c + 1] + par[w + c] + par[w + c + 1]) >= 2;
        }
        out[j] = static_cast<uint8_t>(val);
        cnt += val;
    }
    for (int o = 16; o; o >>= 1) cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
    if ((threadIdx.x & 31) == 0 && cnt) atomicAdd(&s_sum, cnt);
    __syncthreads();
    if (threadIdx.x == 0 && s_sum) atomicAdd(areas + li, s_sum);
}

// overlap order key: np.argsort(-areas) on uint64 puts zero areas first, then larger areas first
__device__ __forceinline__ bool seg_before(int32_t ai, int i, int32_t aj, int j) {
    const long long ki = ai == 0 ? -(1LL << 40) : -static_cast<long long>(ai);
    const long long kj = aj == 0 ? -(1LL << 40) : -static_cast<long long>(aj);
    return kj < ki || (kj == ki && j < i);
}

__device__ __forceinline__ int block_sum(int v, int* s_red) {
    for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    __syncthreads();
    if ((threadIdx.x & 31) == 0) s_red[threadIdx.x >> 5] = v;
    __syncthreads();
    int t = 0;
    for (int w = 0; w < static_cast<int>(blockDim.x >> 5); ++w) t += s_red[w];
    return t;
}

// one block per image: kept labels of rows [image_rows[b], image_rows[b+1]) -> output positions
__global__ void __launch_bounds__(kSegOrderThreads) seg_order_kernel(const int32_t* __restrict__ image_rows, int n_images,
                                                                    const int32_t* __restrict__ keep, const int32_t* __restrict__ areas,
                                                                    const float* __restrict__ rows, int overlap, float* __restrict__ targets,
                                                                    int32_t* __restrict__ plane, int32_t* __restrict__ counts) {
    __shared__ int s_red[kSegOrderThreads / 32];
    const int b = blockIdx.x, tid = threadIdx.x;
    const int r0 = image_rows[b], r1 = image_rows[b + 1];
    int before = 0, mine = 0;
    for (int i = tid; i < r0; i += blockDim.x) before += keep[i] != 0;
    for (int i = r0 + tid; i < r1; i += blockDim.x) mine += keep[i] != 0;
    const int base = block_sum(before, s_red);
    const int nk = block_sum(mine, s_red);
    for (int i = r0 + tid; i < r1; i += blockDim.x) {
        if (!keep[i]) continue;
        int rank = 0;
        for (int j = r0; j < r1; ++j) {
            if (j == i || !keep[j]) continue;
            rank += overlap ? seg_before(areas[i], i, areas[j], j) : j < i;
        }
        const int pos = base + rank;
#pragma unroll
        for (int k = 0; k < 6; ++k) targets[static_cast<long long>(pos) * 6 + k] = rows[static_cast<long long>(i) * 6 + k];
        plane[pos] = i;
    }
    if (tid == 0) {
        counts[1 + b] = nk;
        if (b == n_images - 1) counts[0] = base + nk;
    }
}

// overlap: grid (pixel blocks, images), out (n_images, mh, mw); planes: grid (pixel blocks, kept labels), out (nt, mh, mw)
template <typename T>
__device__ __forceinline__ void seg_store(void* out, long long o, int v) {
    static_cast<T*>(out)[o] = static_cast<T>(v);
}

__global__ void seg_compose_kernel(const y5_aug_image* __restrict__ table, const y5_aug_label* __restrict__ labels,
                                   const int32_t* __restrict__ counts, const int32_t* __restrict__ plane,
                                   const uint8_t* __restrict__ masks, int mh, int mw, int overlap, void* __restrict__ out, int out_dtype) {
    const long long npx = static_cast<long long>(mh) * mw;
    const long long px = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (px >= npx) return;
    const int oy = static_cast<int>(px / mw), ox = static_cast<int>(px % mw);
    const int z = blockIdx.y;
    const y5_aug_image& im = table[overlap ? z : labels[plane[z]].image];
    const long long src = static_cast<long long>(im.flipud ? mh - 1 - oy : oy) * mw + (im.fliplr ? mw - 1 - ox : ox);
    int v = 0;
    if (overlap) {
        int start = 0;
        for (int c = 0; c < z; ++c) start += counts[1 + c];
        const int n = counts[1 + z];
        const bool u8 = n <= 255;  // polygons2masks_overlap: uint8 up to 255 labels, else int32
        for (int i = 0; i < n; ++i) {
            const int m = masks[static_cast<long long>(plane[start + i]) * npx + src];
            v = v + m * (i + 1);
            if (u8) v &= 0xff;  // uint8 wrap-around before the clip
            v = min(max(v, 0), i + 1);
        }
    } else {
        v = masks[static_cast<long long>(plane[z]) * npx + src];
    }
    const long long o = static_cast<long long>(z) * npx + px;
    if (out_dtype == Y5_U8) seg_store<uint8_t>(out, o, v);
    else if (out_dtype == Y5_F32) seg_store<float>(out, o, v);
    else seg_store<int32_t>(out, o, v);
}

}  // namespace y5

using namespace y5;

extern "C" Y5_API int y5_seg_warp(const y5_aug_image* table, int32_t n_images, const y5_aug_label* labels, const y5_aug_segment* segments,
                                  const float* points, int32_t max_points, int32_t n_labels, int32_t out_h, int32_t out_w, int32_t* verts,
                                  float* rows, int32_t* keep, void* stream) {
    if (!table || n_images <= 0 || n_labels < 0 || out_h <= 0 || out_w <= 0 || max_points < 1 ||
        (n_labels > 0 && (!labels || !segments || !points || !verts || !rows || !keep)))
        return set_error(Y5_E_INVALID, "seg_warp: bad argument");
    if (out_h > 16384 || out_w > 16384 || max_points > 8192) return set_error(Y5_E_UNSUPPORTED, "seg_warp: image or polygon too large");
    if (n_labels == 0) return 0;
    const size_t smem = sizeof(float) * 2 * (static_cast<size_t>(max_points) + 1);
    return launch("seg_warp", seg_warp_kernel, {n_labels, kSegThreads, smem, static_cast<cudaStream_t>(stream)}, table, n_images, labels, segments,
                  points, max_points, out_h, out_w, verts, rows, keep);
}

extern "C" Y5_API int y5_seg_raster(const int32_t* verts, int32_t n_verts, const int32_t* keep, int32_t n_labels, int32_t out_h, int32_t out_w,
                                    int32_t ratio, uint8_t* masks, int32_t* areas, void* stream) {
    if (n_labels < 0 || n_verts < 1 || out_h <= 0 || out_w <= 0 || (n_labels > 0 && (!verts || !keep || !masks || !areas)))
        return set_error(Y5_E_INVALID, "seg_raster: bad argument");
    if (ratio != 1 && ratio != 4) return set_error(Y5_E_UNSUPPORTED, "seg_raster: downsample ratio %d (1 or 4)", ratio);
    if (out_h % ratio || out_w % ratio) return set_error(Y5_E_UNSUPPORTED, "seg_raster: image size not a multiple of the ratio");
    if (out_w > 4096 || out_h > 4096 || n_labels > 65535) return set_error(Y5_E_UNSUPPORTED, "seg_raster: image or label count too large");
    if (n_labels == 0) return 0;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    cudaMemsetAsync(areas, 0, sizeof(int32_t) * n_labels, st);
    const int nsrc = ratio == 1 ? 1 : 2;
    const size_t smem = static_cast<size_t>(nsrc) * out_w * (sizeof(int) + 1);
    if (smem > 48 * 1024) cudaFuncSetAttribute(seg_raster_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem));
    return launch("seg_raster", seg_raster_kernel, {dim3(out_h / ratio, n_labels), kSegThreads, smem, st}, verts, n_verts, keep, out_h, out_w, ratio,
                  masks, areas);
}

extern "C" Y5_API int y5_seg_order(const int32_t* image_rows, int32_t n_images, const int32_t* keep, const int32_t* areas, const float* rows,
                                   int32_t overlap, float* targets, int32_t* plane, int32_t* counts, void* stream) {
    if (!image_rows || !counts || n_images <= 0) return set_error(Y5_E_INVALID, "seg_order: bad argument");
    if (n_images > 65535) return set_error(Y5_E_UNSUPPORTED, "seg_order: batch too large");
    return launch("seg_order", seg_order_kernel, {n_images, kSegOrderThreads, 0, static_cast<cudaStream_t>(stream)}, image_rows, n_images, keep,
                  areas, rows, overlap, targets, plane, counts);
}

extern "C" Y5_API int y5_seg_compose(const y5_aug_image* table, const y5_aug_label* labels, const int32_t* counts, const int32_t* plane,
                                     const uint8_t* masks, int32_t n_out, int32_t mask_h, int32_t mask_w, int32_t overlap, void* out,
                                     int32_t out_dtype, void* stream) {
    if (!table || !counts || n_out < 0 || mask_h <= 0 || mask_w <= 0 || (n_out > 0 && (!out || !plane || !masks || (!overlap && !labels))))
        return set_error(Y5_E_INVALID, "seg_compose: bad argument");
    if (out_dtype != Y5_U8 && out_dtype != Y5_F32 && out_dtype != Y5_SEG_I32) return set_error(Y5_E_UNSUPPORTED, "seg_compose: output dtype");
    if (n_out > 65535) return set_error(Y5_E_UNSUPPORTED, "seg_compose: too many planes");
    if (n_out == 0) return 0;
    const long long npx = static_cast<long long>(mask_h) * mask_w;
    const dim3 grid(static_cast<unsigned>((npx + 255) / 256), n_out);
    return launch("seg_compose", seg_compose_kernel, {grid, 256, 0, static_cast<cudaStream_t>(stream)}, table, labels, counts, plane, masks, mask_h,
                  mask_w, overlap, out, out_dtype);
}
