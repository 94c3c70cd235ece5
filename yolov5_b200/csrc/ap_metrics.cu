// Validation AP of val.py / segment/val.py (utils/metrics.py:25-126 ap_per_class with compute_ap, and
// utils/segment/metrics.py:17-64 ap_per_class_box_and_mask) on the device, in float64 and step for step:
//   ap_setup_kernel   : label count per class, the ascending unique-class list, the row offset of every image (padded form)
//   ap_gather_kernel  : the rows in (image, row) order -> sort key, confidence, tp bit mask (one bit per IoU threshold),
//                       prediction count per class
//   radix_*_kernel    : stable LSD radix sort of the key (class << 32 | descending-confidence key), 6 passes of 8 bits: rows
//                       grouped by class, inside a class np.argsort(-conf, kind="stable") order (ties in input order, NaN last)
//   ap_permute_kernel : confidences and tp masks in sorted order
//   ap_class_kernel   : one block per (class, threshold): integer cumsum of tp, the p / r curves at the 1000 points of
//                       np.linspace(0, 1, 1000) (threshold 0), compute_ap (precision envelope, np.interp at the 101 points of
//                       np.linspace(0, 1, 101), np.trapezoid summed in numpy's pairwise order)
//   ap_tail_kernel    : f1, its class mean in class order, smooth(0.1) + first argmax, and p, r, f1, tp, fp at that index
// Every value but the smoothed mean-F1 curve (whose np.convolve summation order is BLAS's) is the reference's, bit for bit;
// the smoothed curve only picks the index.  Compiled with -fmad=false, with explicit _rn arithmetic where it matters; there
// are no floating-point atomics, so two runs give the same bits.  No allocation, no host synchronisation.
#include "../../include/y5b200.h"
#include "common.cuh"
#include "host_util.h"

namespace y5 {

constexpr int kApMaxClasses = 4096;  // nms.cu kMaxClasses
constexpr int kApMaxIou = 32;        // one bit per threshold in a uint32 mask
constexpr int kApPx = 1000, kApX = 101;
constexpr int kRowThreads = 256;
constexpr int kSortThreads = 256, kSortItems = 8, kSortTile = kSortThreads * kSortItems, kSortPasses = 6;
constexpr int kClassThreads = 256, kClassItems = 4, kClassChunk = kClassThreads * kClassItems;
constexpr int kOneBlock = 1024;
constexpr int kFlagPredClass = 1, kFlagTargetClass = 2;

// class value -> class index, or -1 unless it is an integer in [0, kApMaxClasses)
__device__ __forceinline__ int class_index(float c) {
    if (!(c >= 0.f && c < static_cast<float>(kApMaxClasses))) return -1;
    const int k = static_cast<int>(c);
    return static_cast<float>(k) == c ? k : -1;
}

// ascending order of the key == ascending order of -conf as numpy sorts it: -0 ties with +0, every NaN last
__device__ __forceinline__ uint32_t conf_key(float conf) {
    float v = -conf;
    if (v != v) return 0xffffffffu;
    if (v == 0.f) v = 0.f;
    const uint32_t u = __float_as_uint(v);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

// exclusive prefix sum over the block (THREADS threads); `total` gets the block's sum
template <int THREADS>
__device__ __forceinline__ int block_exclusive_scan(int v, int& total) {
    __shared__ int s_w[THREADS / 32];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    int x = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int y = __shfl_up_sync(0xffffffffu, x, o);
        if (lane >= o) x += y;
    }
    if (lane == 31) s_w[warp] = x;
    __syncthreads();
    if (warp == 0) {
        int w = lane < THREADS / 32 ? s_w[lane] : 0;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int y = __shfl_up_sync(0xffffffffu, w, o);
            if (lane >= o) w += y;
        }
        if (lane < THREADS / 32) s_w[lane] = w;
    }
    __syncthreads();
    const int before = warp ? s_w[warp - 1] : 0;
    total = s_w[THREADS / 32 - 1];
    __syncthreads();
    return before + x - v;
}

// numpy's binary_search_with_guess on an ascending xp of n >= 1 values: n when x > xp[n-1], -1 when x < xp[0], else the
// largest j with xp[j] <= x
template <class XP>
__device__ __forceinline__ int interp_search(double x, int n, XP xp) {
    if (x > xp(n - 1)) return n;
    if (x < xp(0)) return -1;
    int lo = 0, hi = n;
    while (lo < hi) {
        const int mid = lo + ((hi - lo) >> 1);
        if (x >= xp(mid)) lo = mid + 1;
        else hi = mid;
    }
    return lo - 1;
}

// numpy's interp at x given j = interp_search(...): xj, fj at j and xj1, fj1 at j + 1 (read only when j + 1 < n)
__device__ __forceinline__ double interp_value(double x, int j, int n, double xj, double fj, double xj1, double fj1, double lval, double rval) {
    if (j < 0) return lval;
    if (j >= n) return rval;
    if (j == n - 1 || xj == x) return fj;
    const double s = __ddiv_rn(__dsub_rn(fj1, fj), __dsub_rn(xj1, xj));
    double y = __dadd_rn(__dmul_rn(s, __dsub_rn(x, xj)), fj);
    if (isnan(y)) {
        y = __dadd_rn(__dmul_rn(s, __dsub_rn(x, xj1)), fj1);
        if (isnan(y) && fj == fj1) y = fj;
    }
    return y;
}

// 2 * p * r / (p + r + eps), left to right
__device__ __forceinline__ double f1_score(double p, double r, double eps) {
    return __ddiv_rn(__dmul_rn(__dmul_rn(2.0, p), r), __dadd_rn(__dadd_rn(p, r), eps));
}

// One block.  meta = [n, nc, flags, argmax 0, argmax 1, unique classes...]; img_off[b] = rows of images before b.
__global__ void __launch_bounds__(kOneBlock) ap_setup_kernel(const float* __restrict__ target_cls, int nt, const int32_t* __restrict__ count,
                                                              int n_img, int rows_per_image, int* __restrict__ img_off,
                                                              int* __restrict__ label_count, int* __restrict__ pred_count,
                                                              int32_t* __restrict__ meta) {
    __shared__ int s_hist[kApMaxClasses];
    __shared__ int s_flag;
    const int tid = threadIdx.x;
    for (int c = tid; c < kApMaxClasses; c += kOneBlock) {
        s_hist[c] = 0;
        pred_count[c] = 0;
    }
    if (tid == 0) s_flag = 0;
    __syncthreads();
    for (int i = tid; i < nt; i += kOneBlock) {
        const int k = class_index(target_cls[i]);
        if (k < 0) atomicOr(&s_flag, kFlagTargetClass);
        else atomicAdd(&s_hist[k], 1);
    }
    __syncthreads();
    constexpr int per = kApMaxClasses / kOneBlock;
    int present = 0;
#pragma unroll
    for (int q = 0; q < per; ++q) present += s_hist[tid * per + q] > 0;
    int nc;
    int ci = block_exclusive_scan<kOneBlock>(present, nc);
#pragma unroll
    for (int q = 0; q < per; ++q) {
        const int c = tid * per + q;
        label_count[c] = s_hist[c];
        if (s_hist[c] > 0) meta[Y5_AP_META + ci++] = c;
    }
    const int chunk = (n_img + kOneBlock - 1) / kOneBlock;
    const int b0 = min(tid * chunk, n_img), b1 = min(b0 + chunk, n_img);
    int rows = 0;
    for (int b = b0; b < b1; ++b) rows += count ? min(max(count[b], 0), rows_per_image) : rows_per_image;
    int n;
    int run = block_exclusive_scan<kOneBlock>(rows, n);
    for (int b = b0; b < b1; ++b) {
        img_off[b] = run;
        run += count ? min(max(count[b], 0), rows_per_image) : rows_per_image;
    }
    if (tid == 0) {
        img_off[n_img] = n;
        meta[0] = n;
        meta[1] = nc;
        meta[2] = s_flag;
        meta[3] = meta[4] = 0;
    }
}

// One thread per (image, row) slot; rows at or past count[image] are not read.
__global__ void __launch_bounds__(kRowThreads) ap_gather_kernel(const uint8_t* __restrict__ tp, const uint8_t* __restrict__ tp2, long long tp_img_stride,
                                                                 int tp_row_stride, const float* __restrict__ conf, const float* __restrict__ pred_cls,
                                                                 long long img_stride, int row_stride, const int32_t* __restrict__ count,
                                                                 long long slots, int rows_per_image, int niou, const int* __restrict__ img_off,
                                                                 unsigned long long* __restrict__ keys, int* __restrict__ vals,
                                                                 float* __restrict__ conf_flat, uint32_t* __restrict__ tpm,
                                                                 uint32_t* __restrict__ tpm2, int* __restrict__ pred_count, int32_t* __restrict__ meta) {
    const long long s = static_cast<long long>(blockIdx.x) * kRowThreads + threadIdx.x;
    int k = -1;
    if (s < slots) {
        const int img = static_cast<int>(s / rows_per_image), r = static_cast<int>(s % rows_per_image);
        const int cnt = count ? min(max(count[img], 0), rows_per_image) : rows_per_image;
        if (r < cnt) {
            const int flat = img_off[img] + r;
            const long long pe = img * img_stride + static_cast<long long>(r) * row_stride;
            const float f = conf[pe];
            k = class_index(pred_cls[pe]);
            if (k < 0) {
                atomicOr(&meta[2], kFlagPredClass);
                k = 0;
            }
            keys[flat] = (static_cast<unsigned long long>(k) << 32) | conf_key(f);
            vals[flat] = flat;
            conf_flat[flat] = f;
            const long long te = img * tp_img_stride + static_cast<long long>(r) * tp_row_stride;
            uint32_t m = 0, m2 = 0;
            for (int t = 0; t < niou; ++t) {
                m |= static_cast<uint32_t>(tp[te + t] != 0) << t;
                if (tp2) m2 |= static_cast<uint32_t>(tp2[te + t] != 0) << t;
            }
            tpm[flat] = m;
            if (tp2) tpm2[flat] = m2;
        }
    }
    // one atomic per class present in the warp
    const unsigned peers = __match_any_sync(0xffffffffu, k);
    if (k >= 0 && (threadIdx.x & 31) == __ffs(peers) - 1) atomicAdd(&pred_count[k], __popc(peers));
}

// hist[digit * ntiles + tile] = rows of the tile with that digit
__global__ void __launch_bounds__(kSortThreads) radix_hist_kernel(const unsigned long long* __restrict__ keys, const int32_t* __restrict__ meta,
                                                                   int shift, int ntiles, int* __restrict__ hist) {
    __shared__ int s_count[256];
    const int n = meta[0];
    s_count[threadIdx.x] = 0;
    __syncthreads();
    const long long base = static_cast<long long>(blockIdx.x) * kSortTile;
#pragma unroll
    for (int q = 0; q < kSortItems; ++q) {
        const long long i = base + q * kSortThreads + threadIdx.x;
        if (i < n) atomicAdd(&s_count[(keys[i] >> shift) & 255], 1);
    }
    __syncthreads();
    hist[static_cast<long long>(threadIdx.x) * ntiles + blockIdx.x] = s_count[threadIdx.x];
}

// One block: exclusive prefix sum of hist in place (digit-major, so a tile's rows of a digit land after every earlier
// tile's rows of that digit and after all rows of smaller digits)
__global__ void __launch_bounds__(kOneBlock) radix_scan_kernel(int* __restrict__ hist, int total) {
    const int chunk = (total + kOneBlock - 1) / kOneBlock;
    const int b0 = min(static_cast<int>(threadIdx.x) * chunk, total), b1 = min(b0 + chunk, total);
    int sum = 0;
    for (int i = b0; i < b1; ++i) sum += hist[i];
    int all;
    int run = block_exclusive_scan<kOneBlock>(sum, all);
    for (int i = b0; i < b1; ++i) {
        const int v = hist[i];
        hist[i] = run;
        run += v;
    }
}

// Stable scatter of one tile: rounds of 256 rows in order; inside a round, rows of one digit keep thread order
// (warp peers by __match_any_sync, earlier warps' counts of the digit in shared memory).
__global__ void __launch_bounds__(kSortThreads) radix_scatter_kernel(const unsigned long long* __restrict__ kin, const int* __restrict__ vin,
                                                                      unsigned long long* __restrict__ kout, int* __restrict__ vout,
                                                                      const int32_t* __restrict__ meta, int shift, int ntiles,
                                                                      const int* __restrict__ hist) {
    constexpr int kWarps = kSortThreads / 32;
    __shared__ int s_base[256];
    __shared__ int s_warp[kWarps][256];
    const int n = meta[0];
    const long long base = static_cast<long long>(blockIdx.x) * kSortTile;
    if (base >= n) return;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    s_base[tid] = hist[static_cast<long long>(tid) * ntiles + blockIdx.x];
    for (int q = 0; q < kSortItems; ++q) {
        const long long i = base + q * kSortThreads + tid;
        const bool valid = i < n;
#pragma unroll
        for (int w = 0; w < kWarps; ++w) s_warp[w][tid] = 0;
        __syncthreads();
        unsigned long long key = 0;
        int val = 0, digit = 256;
        if (valid) {
            key = kin[i];
            val = vin[i];
            digit = static_cast<int>((key >> shift) & 255);
        }
        const unsigned peers = __match_any_sync(0xffffffffu, digit);
        const int rank = __popc(peers & ((1u << lane) - 1u));
        if (valid && lane == __ffs(peers) - 1) s_warp[warp][digit] = __popc(peers);
        __syncthreads();
        if (valid) {
            int off = s_base[digit] + rank;
            for (int w = 0; w < warp; ++w) off += s_warp[w][digit];
            kout[off] = key;
            vout[off] = val;
        }
        __syncthreads();
        int add = 0;
#pragma unroll
        for (int w = 0; w < kWarps; ++w) add += s_warp[w][tid];
        s_base[tid] += add;
        __syncthreads();
    }
}

__global__ void __launch_bounds__(kRowThreads) ap_permute_kernel(const int* __restrict__ vals, const int32_t* __restrict__ meta,
                                                                  const float* __restrict__ conf_flat, const uint32_t* __restrict__ tpm,
                                                                  const uint32_t* __restrict__ tpm2, float* __restrict__ conf_s,
                                                                  uint32_t* __restrict__ tpm_s, uint32_t* __restrict__ tpm2_s) {
    const long long i = static_cast<long long>(blockIdx.x) * kRowThreads + threadIdx.x;
    if (i >= meta[0]) return;
    const int v = vals[i];
    conf_s[i] = conf_flat[v];
    tpm_s[i] = tpm[v];
    if (tpm2) tpm2_s[i] = tpm2[v];
}

// grid (nc_cap, niou): block (ci, t) handles unique class ci at threshold t.  tpc (niou rows of n_cap int32) gets the class
// segment's cumulative tp counts; curves (threshold 0 blocks) p_curve / r_curve rows of kApPx values; ap[ci * niou + t].
// grid = [np.linspace(0, 1, 1000), np.linspace(0, 1, 101)].
__global__ void __launch_bounds__(kClassThreads) ap_class_kernel(const int32_t* __restrict__ meta, const int* __restrict__ label_count,
                                                                  const int* __restrict__ pred_count, const float* __restrict__ conf_s,
                                                                  const uint32_t* __restrict__ tpm_s, int* __restrict__ tpc_all, long long n_cap,
                                                                  const double* __restrict__ grid, double eps, int niou,
                                                                  double* __restrict__ p_curve, double* __restrict__ r_curve, double* __restrict__ ap) {
    constexpr int kWarps = kClassThreads / 32;
    __shared__ double s_chunk[kClassChunk];
    __shared__ double s_wmax[kWarps];
    __shared__ int s_j[kApX];
    __shared__ double s_e0[kApX], s_e1[kApX], s_y[kApX];
    const int ci = blockIdx.x, t = blockIdx.y, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if (ci >= meta[1]) return;
    const int c = meta[Y5_AP_META + ci];
    const int n_l = label_count[c], n_p = pred_count[c];
    int part = 0;
    for (int q = tid; q < c; q += kClassThreads) part += pred_count[q];
    int start;
    block_exclusive_scan<kClassThreads>(part, start);
    double* pc = p_curve + static_cast<long long>(ci) * kApPx;
    double* rc = r_curve + static_cast<long long>(ci) * kApPx;
    if (n_p == 0) {  // the reference skips the class: zero curves and AP
        if (t == 0)
            for (int k = tid; k < kApPx; k += kClassThreads) pc[k] = rc[k] = 0.0;
        if (tid == 0) ap[static_cast<long long>(ci) * niou + t] = 0.0;
        return;
    }
    const float* cs = conf_s + start;
    const uint32_t* tm = tpm_s + start;
    int* tpc = tpc_all + t * n_cap + start;

    // tpc = tp[:, t].cumsum(0) (fpc = row + 1 - tpc)
    int carry = 0;
    for (int b = 0; b < n_p; b += kClassChunk) {
        int v[kClassItems], sum = 0;
#pragma unroll
        for (int q = 0; q < kClassItems; ++q) {
            const int i = b + tid * kClassItems + q;
            v[q] = i < n_p ? static_cast<int>((tm[i] >> t) & 1u) : 0;
            sum += v[q];
        }
        int all;
        int run = carry + block_exclusive_scan<kClassThreads>(sum, all);
#pragma unroll
        for (int q = 0; q < kClassItems; ++q) {
            const int i = b + tid * kClassItems + q;
            run += v[q];
            if (i < n_p) tpc[i] = run;
        }
        carry += all;
    }
    __syncthreads();
    const double den = __dadd_rn(static_cast<double>(n_l), eps);
    auto recall = [&](int i) { return __ddiv_rn(static_cast<double>(tpc[i]), den); };
    auto precision = [&](int i) { return __ddiv_rn(static_cast<double>(tpc[i]), static_cast<double>(i + 1)); };

    // r = np.interp(-px, -conf, recall[:, 0], left=0), p = np.interp(-px, -conf, precision[:, 0], left=1)
    if (t == 0) {
        auto xp = [&](int i) { return -static_cast<double>(cs[i]); };
        for (int k = tid; k < kApPx; k += kClassThreads) {
            const double x = -grid[k];
            const int j = interp_search(x, n_p, xp);
            const bool in = j >= 0 && j < n_p, next = in && j + 1 < n_p;
            const double xj = in ? xp(j) : 0.0, xj1 = next ? xp(j + 1) : 0.0;
            rc[k] = interp_value(x, j, n_p, xj, in ? recall(j) : 0.0, xj1, next ? recall(j + 1) : 0.0, 0.0, recall(n_p - 1));
            pc[k] = interp_value(x, j, n_p, xj, in ? precision(j) : 0.0, xj1, next ? precision(j + 1) : 0.0, 1.0, precision(n_p - 1));
        }
    }

    // compute_ap: mrec = [0, recall, 1], mpre = [1, precision, 0] (m = n_p + 2 points), envelope env = suffix max of mpre
    const int m = n_p + 2;
    auto mrec = [&](int j) { return j == 0 ? 0.0 : (j == m - 1 ? 1.0 : recall(j - 1)); };
    for (int k = tid; k < kApX; k += kClassThreads) {
        s_j[k] = interp_search(grid[kApPx + k], m, mrec);
        s_e0[k] = s_e1[k] = 0.0;
    }
    __syncthreads();
    // env at the points 1..n_p the interpolation reads, from the last chunk backwards; env(m - 1) = 0, env(0) = max(1, env(1))
    double after = 0.0;
    for (int hi = n_p; hi >= 1; hi -= kClassChunk) {
        const int lo = max(1, hi - kClassChunk + 1);
        double v[kClassItems], run = 0.0;
#pragma unroll
        for (int q = kClassItems - 1; q >= 0; --q) {
            const int pos = lo + tid * kClassItems + q;
            const double x = pos <= hi ? precision(pos - 1) : 0.0;
            run = x > run ? x : run;
            v[q] = run;
        }
        double incl = run;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const double y = __shfl_down_sync(0xffffffffu, incl, o);
            if (lane + o < 32) incl = y > incl ? y : incl;
        }
        double later = __shfl_down_sync(0xffffffffu, incl, 1);
        if (lane == 31) later = 0.0;
        if (lane == 0) s_wmax[warp] = incl;
        __syncthreads();
        for (int w = warp + 1; w < kWarps; ++w) later = s_wmax[w] > later ? s_wmax[w] : later;
        later = after > later ? after : later;
#pragma unroll
        for (int q = 0; q < kClassItems; ++q) {
            const int pos = lo + tid * kClassItems + q;
            if (pos <= hi) s_chunk[pos - lo] = v[q] > later ? v[q] : later;
        }
        __syncthreads();
        for (int k = tid; k < kApX; k += kClassThreads) {
            const int j = s_j[k];
            if (j >= lo && j <= hi) s_e0[k] = s_chunk[j - lo];
            if (j + 1 >= lo && j + 1 <= hi) s_e1[k] = s_chunk[j + 1 - lo];
        }
        after = s_chunk[0];
        __syncthreads();
    }
    const double env0 = after > 1.0 ? after : 1.0;
    for (int k = tid; k < kApX; k += kClassThreads) {
        const int j = s_j[k];
        const double e0 = j == 0 ? env0 : s_e0[k];  // j == m - 1 reads env(m - 1) = 0, as initialised
        const double e1 = j + 1 == 0 ? env0 : s_e1[k];
        const bool next = j >= 0 && j + 1 < m;
        s_y[k] = interp_value(grid[kApPx + k], j, m, j >= 0 && j < m ? mrec(j) : 0.0, e0, next ? mrec(j + 1) : 0.0, e1, env0, 0.0);
    }
    __syncthreads();
    if (tid == 0) {  // np.trapezoid: d * (y[1:] + y[:-1]) / 2.0 summed as numpy's pairwise_sum (8 accumulators, then the tail)
        const double* x = grid + kApPx;
        auto term = [&](int i) { return __ddiv_rn(__dmul_rn(__dsub_rn(x[i + 1], x[i]), __dadd_rn(s_y[i + 1], s_y[i])), 2.0); };
        constexpr int nterm = kApX - 1, full = nterm - nterm % 8;
        double r[8];
#pragma unroll
        for (int q = 0; q < 8; ++q) r[q] = term(q);
        for (int i = 8; i < full; i += 8)
#pragma unroll
            for (int q = 0; q < 8; ++q) r[q] = __dadd_rn(r[q], term(i + q));
        double res = __dadd_rn(__dadd_rn(__dadd_rn(r[0], r[1]), __dadd_rn(r[2], r[3])), __dadd_rn(__dadd_rn(r[4], r[5]), __dadd_rn(r[6], r[7])));
        for (int i = full; i < nterm; ++i) res = __dadd_rn(res, term(i));
        ap[static_cast<long long>(ci) * niou + t] = res;
    }
}

// One block.  out (one set) = [tp, fp, p, r, f1] (nc_cap each), ap follows and is written by ap_class_kernel.
__global__ void __launch_bounds__(kOneBlock) ap_tail_kernel(int32_t* __restrict__ meta, int set, const int* __restrict__ label_count,
                                                             const double* __restrict__ p_curve, const double* __restrict__ r_curve, double eps,
                                                             int nc_cap, double* __restrict__ out) {
    constexpr int pad = 50;  // smooth(f=0.1): 101 taps, 50 edge copies each side
    __shared__ double s_y[kApPx + 2 * pad];
    __shared__ double s_s[kApPx];
    const int nc = meta[1], tid = threadIdx.x;
    for (int k = tid; k < kApPx; k += kOneBlock) {
        double acc = 0.0;
        for (int ci = 0; ci < nc; ++ci) {  // f1.mean(0): classes added in class order, then one division
            const long long e = static_cast<long long>(ci) * kApPx + k;
            const double f = f1_score(p_curve[e], r_curve[e], eps);
            acc = ci ? __dadd_rn(acc, f) : f;
        }
        s_y[pad + k] = nc ? __ddiv_rn(acc, static_cast<double>(nc)) : __longlong_as_double(0x7ff8000000000000LL);
    }
    __syncthreads();
    if (tid < pad) {
        s_y[tid] = s_y[pad];
        s_y[pad + kApPx + tid] = s_y[pad + kApPx - 1];
    }
    __syncthreads();
    const double w = 1.0 / (2 * pad + 1);
    for (int k = tid; k < kApPx; k += kOneBlock) {
        double s = 0.0;
        for (int q = 0; q <= 2 * pad; ++q) s = __dadd_rn(s, __dmul_rn(s_y[k + q], w));
        s_s[k] = s;
    }
    __syncthreads();
    __shared__ int s_i;
    if (tid == 0) {  // np.argmax: the first maximum, and a NaN beats everything
        int best = 0;
        for (int k = 1; k < kApPx && !isnan(s_s[best]); ++k)
            if (isnan(s_s[k]) || s_s[k] > s_s[best]) best = k;
        s_i = best;
        meta[3 + set] = best;
    }
    __syncthreads();
    const int i = s_i;
    for (int ci = tid; ci < nc; ci += kOneBlock) {
        const long long e = static_cast<long long>(ci) * kApPx + i;
        const double p = p_curve[e], r = r_curve[e];
        const double tp = rint(__dmul_rn(r, static_cast<double>(label_count[meta[Y5_AP_META + ci]])));
        out[ci] = tp;
        out[nc_cap + ci] = rint(__dsub_rn(__ddiv_rn(tp, __dadd_rn(p, eps)), tp));
        out[2 * nc_cap + ci] = p;
        out[3 * nc_cap + ci] = r;
        out[4 * nc_cap + ci] = f1_score(p, r, eps);
    }
}

struct ApWorkspace {
    int* img_off;
    unsigned long long* keys[2];
    int* vals[2];
    float *conf, *conf_s;
    uint32_t *tpm[2], *tpm_s[2];
    int *hist, *label_count, *pred_count, *tpc;
    double *p_curve, *r_curve;
    long long bytes;
};

static long long sort_tiles(long long n_cap) { return (n_cap + kSortTile - 1) / kSortTile; }

// base == nullptr: sizes only
static ApWorkspace ap_workspace(char* base, long long n_cap, int n_img, int niou, int nc_cap, int sets) {
    ApWorkspace w{};
    long long off = 0;
    auto take = [&](long long bytes) {
        char* p = base ? base + off : nullptr;
        off += (bytes + 255) / 256 * 256;
        return p;
    };
    w.img_off = reinterpret_cast<int*>(take(4LL * (n_img + 1)));
    for (int q = 0; q < 2; ++q) w.keys[q] = reinterpret_cast<unsigned long long*>(take(8 * n_cap));
    for (int q = 0; q < 2; ++q) w.vals[q] = reinterpret_cast<int*>(take(4 * n_cap));
    w.conf = reinterpret_cast<float*>(take(4 * n_cap));
    w.conf_s = reinterpret_cast<float*>(take(4 * n_cap));
    for (int q = 0; q < sets; ++q) {
        w.tpm[q] = reinterpret_cast<uint32_t*>(take(4 * n_cap));
        w.tpm_s[q] = reinterpret_cast<uint32_t*>(take(4 * n_cap));
    }
    w.hist = reinterpret_cast<int*>(take(4LL * 256 * sort_tiles(n_cap)));
    w.label_count = reinterpret_cast<int*>(take(4LL * kApMaxClasses));
    w.pred_count = reinterpret_cast<int*>(take(4LL * kApMaxClasses));
    w.tpc = reinterpret_cast<int*>(take(4LL * niou * n_cap));
    w.p_curve = reinterpret_cast<double*>(take(8LL * kApPx * nc_cap));
    w.r_curve = reinterpret_cast<double*>(take(8LL * kApPx * nc_cap));
    w.bytes = off;
    return w;
}

static int ap_shape_error(int32_t n_img, int32_t rows_per_image, int32_t niou, int32_t nt, int32_t sets) {
    if (n_img < 0 || rows_per_image < 0 || nt < 0 || niou < 1 || sets < 1 || sets > 2)
        return set_error(Y5_E_INVALID, "ap_per_class: bad shape (images %d, rows %d, niou %d, labels %d, sets %d)", n_img, rows_per_image,
                         niou, nt, sets);
    if (niou > kApMaxIou) return set_error(Y5_E_UNSUPPORTED, "ap_per_class: %d IoU thresholds > %d", niou, kApMaxIou);
    if (static_cast<long long>(n_img) * rows_per_image >= (1LL << 31))
        return set_error(Y5_E_UNSUPPORTED, "ap_per_class: %d x %d rows reach 2^31", n_img, rows_per_image);
    return 0;
}

}  // namespace y5

using namespace y5;

extern "C" Y5_API int64_t y5_ap_workspace_bytes(int32_t n_img, int32_t rows_per_image, int32_t niou, int32_t nt, int32_t sets) {
    if (int e = ap_shape_error(n_img, rows_per_image, niou, nt, sets)) return e;
    return ap_workspace(nullptr, static_cast<long long>(n_img) * rows_per_image, n_img, niou, min(nt, kApMaxClasses), sets).bytes;
}

extern "C" Y5_API int y5_ap_per_class(const uint8_t* tp, const uint8_t* tp2, int64_t tp_img_stride, int32_t tp_row_stride, const float* conf,
                                      const float* pred_cls, int64_t img_stride, int32_t row_stride, const int32_t* count, int32_t n_img,
                                      int32_t rows_per_image, int32_t niou, const float* target_cls, int32_t nt, const double* grid, double eps,
                                      void* workspace, int64_t workspace_bytes, double* out, int32_t* meta, void* stream) {
    const int sets = tp2 ? 2 : 1;
    if (int e = ap_shape_error(n_img, rows_per_image, niou, nt, sets)) return e;
    const long long slots = static_cast<long long>(n_img) * rows_per_image;
    if (slots > 0 && (!tp || !conf || !pred_cls || tp_row_stride < niou || row_stride < 1 || (n_img > 1 && (img_stride < 1 || tp_img_stride < 1))))
        return set_error(Y5_E_INVALID, "ap_per_class: null rows or bad strides");
    if ((nt > 0 && !target_cls) || !grid || !workspace || !out || !meta) return set_error(Y5_E_INVALID, "ap_per_class: null pointer");
    const int nc_cap = min(nt, kApMaxClasses);
    const ApWorkspace w = ap_workspace(static_cast<char*>(workspace), slots, n_img, niou, nc_cap, sets);
    if (workspace_bytes < w.bytes)
        return set_error(Y5_E_INVALID, "ap_per_class: workspace of %lld bytes, %lld needed", static_cast<long long>(workspace_bytes), w.bytes);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const char* what = "ap_per_class";
    if (int e = launch(what, ap_setup_kernel, {1, kOneBlock, 0, st}, target_cls, nt, count, n_img, rows_per_image, w.img_off, w.label_count,
                       w.pred_count, meta))
        return e;
    if (slots > 0) {
        const long long ntiles = sort_tiles(slots);
        if (256 * ntiles > (1LL << 31) - 1) return set_error(Y5_E_UNSUPPORTED, "ap_per_class: %lld rows", slots);
        if (int e = launch(what, ap_gather_kernel, {static_cast<unsigned>((slots + kRowThreads - 1) / kRowThreads), kRowThreads, 0, st}, tp, tp2,
                           tp_img_stride, tp_row_stride, conf, pred_cls, img_stride, row_stride, count, slots, rows_per_image, niou, w.img_off,
                           w.keys[0], w.vals[0], w.conf, w.tpm[0], tp2 ? w.tpm[1] : nullptr, w.pred_count, meta))
            return e;
        for (int pass = 0; pass < kSortPasses; ++pass) {
            const int in = pass & 1, shift = 8 * pass;
            if (int e = launch(what, radix_hist_kernel, {static_cast<unsigned>(ntiles), kSortThreads, 0, st}, w.keys[in], meta, shift,
                               static_cast<int>(ntiles), w.hist))
                return e;
            if (int e = launch(what, radix_scan_kernel, {1, kOneBlock, 0, st}, w.hist, static_cast<int>(256 * ntiles))) return e;
            if (int e = launch(what, radix_scatter_kernel, {static_cast<unsigned>(ntiles), kSortThreads, 0, st}, w.keys[in], w.vals[in],
                               w.keys[in ^ 1], w.vals[in ^ 1], meta, shift, static_cast<int>(ntiles), w.hist))
                return e;
        }
        static_assert(kSortPasses % 2 == 0, "the sorted rows end in buffer 0");
        if (int e = launch(what, ap_permute_kernel, {static_cast<unsigned>((slots + kRowThreads - 1) / kRowThreads), kRowThreads, 0, st}, w.vals[0],
                           meta, w.conf, w.tpm[0], tp2 ? w.tpm[1] : nullptr, w.conf_s, w.tpm_s[0], tp2 ? w.tpm_s[1] : nullptr))
            return e;
    }
    if (nc_cap > 0) {
        for (int s = 0; s < sets; ++s) {
            double* o = out + static_cast<long long>(s) * nc_cap * (5 + niou);
            if (int e = launch(what, ap_class_kernel, {dim3(nc_cap, niou), kClassThreads, 0, st}, meta, w.label_count, w.pred_count, w.conf_s,
                               w.tpm_s[s], w.tpc, slots, grid, eps, niou, w.p_curve, w.r_curve, o + 5LL * nc_cap))
                return e;
            if (int e = launch(what, ap_tail_kernel, {1, kOneBlock, 0, st}, meta, s, w.label_count, w.p_curve, w.r_curve, eps, nc_cap, o)) return e;
        }
    }
    return 0;
}
