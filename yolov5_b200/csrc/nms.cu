// Batched non_max_suppression for sm_90a -- whole batch, no host synchronisation, bit-exact indices.
// Replaces reference utils/general.py:658-767 (+ torchvision.ops.nms called at :750) and ultralytics box_iou.
//
// Pipeline (every kernel is launched unconditionally; per-image early exits happen on the device):
//   1 count      warp per 32-row segment: obj > thr, conf = obj*cls (rounded to the input dtype) > thr -> #candidates
//   2 scan       per image: exclusive prefix over segments, total; decide whether the max_nms cut is needed
//   3-6 select   (only images with total > max_nms) two-level radix select on the fp32 score bits -> exact
//                threshold score T and how many candidates equal to T survive (lowest candidate ids first)
//   7 write      ordered compaction of the selected candidates (candidate id = row*nc + cls, ascending)
//   8 sort       per image bitonic sort in shared memory by (score desc, candidate order asc)  == stable argsort
//   9 greedy     per image: 64-candidate chunks against the kept list, early exit at max_det; writes rows + ids
// dtype flow follows the reference exactly: compares / obj*cls / xywh->xyxy are evaluated in fp32 and rounded to
// the INPUT dtype after every operation; scores, class offset (cls*max_wh) and IoU are fp32.  This file is
// compiled with -fmad=false and uses explicit _rn intrinsics: no FMA contraction anywhere on the index path.
#include <math.h>

#include "../../include/y5b200.h"
#include "common.cuh"
#include "host_util.h"

namespace y5 {

constexpr int kSegRows = 32;      // rows per warp segment
constexpr int kCandCap = 32768;   // >= max_nms (30000), power of two for the bitonic sort
constexpr int kMaxDetCap = 4096;
constexpr int kMaxClasses = 4096;

struct NmsArgs {
    const void* pred;
    int B, N, no, nc, nm, dtype;
    float thr;        // conf threshold rounded to the input dtype
    float iou_thr;    // largest float <= the double iou threshold (torchvision's CPU kernel compares in double)
    int multi_label, agnostic, max_det, max_nms;
    float max_wh;
    const int* classes;
    int n_classes;
    int nseg;
    // workspace
    int* seg_cnt;        // [B][nseg]   candidates per segment (pass 1), later selected per segment
    int* seg_eq;         // [B][nseg]   candidates equal to T per segment
    int* seg_off;        // [B][nseg]   exclusive prefix of selected candidates
    int* seg_eq_off;     // [B][nseg]   exclusive prefix of == T candidates
    int* img;            // [B][8]      0 total, 1 need_select, 2 t_hi, 3 cnt_gt_hi, 4 T bits, 5 need_eq, 6 n_sel
    unsigned* hist;      // [B][2][65536]
    float* cand_score;   // [B][kCandCap]
    unsigned* cand_id;   // [B][kCandCap]
    float4* sorted_box;  // [B][kCandCap]  class-offset boxes in score order
    unsigned* sorted_id; // [B][kCandCap]
    float* sorted_score; // [B][kCandCap]
    // outputs
    float* out_rows;
    long long* out_idx;
    int* out_count;
};

__device__ __forceinline__ float ld_elem(const void* base, long long i, int dtype) {
    if (dtype == Y5_F32) return reinterpret_cast<const float*>(base)[i];
    const uint16_t u = reinterpret_cast<const uint16_t*>(base)[i];
    return unpack1(u, dtype == Y5_BF16);
}
__device__ __forceinline__ float rnd(float x, int dtype) {
    if (dtype == Y5_F32) return x;
    return unpack1(pack1(x, dtype == Y5_BF16), dtype == Y5_BF16);
}
__device__ __forceinline__ bool class_allowed(const unsigned* cls_mask, int j) { return (cls_mask[j >> 5] >> (j & 31)) & 1u; }

// Enumerates the candidates of one 32-row segment in candidate-id order.  The whole warp calls
//   f(ok, score, cand_id, before, group_mask)
// convergently once per group of <= 32 potential candidates: `ok` marks the lanes that hold a real candidate,
// `group_mask` is the ballot of ok, `before` the number of candidates of this segment in earlier groups; the
// segment-local rank of a candidate is before + popc(group_mask & lanes_below).  Returns the segment's count.
template <typename F>
__device__ __forceinline__ int for_each_candidate(const NmsArgs& a, int b, int seg, const unsigned* cls_mask, F&& f) {
    const int lane = threadIdx.x & 31;
    const int row0 = seg * kSegRows;
    const long long img_base = static_cast<long long>(b) * a.N * a.no;
    const int my_row = row0 + lane;
    bool pass = false;
    if (my_row < a.N) pass = ld_elem(a.pred, img_base + static_cast<long long>(my_row) * a.no + 4, a.dtype) > a.thr;
    unsigned rows = __ballot_sync(0xffffffffu, pass);
    int count = 0;
    if (a.multi_label) {
        while (rows) {  // warp-uniform loop: one passing row at a time, lanes stride over the classes
            const int rl = __ffs(rows) - 1;
            rows &= rows - 1;
            const int r = row0 + rl;
            const long long rb = img_base + static_cast<long long>(r) * a.no;
            const float obj = ld_elem(a.pred, rb + 4, a.dtype);
            for (int j0 = 0; j0 < a.nc; j0 += 32) {
                const int j = j0 + lane;
                float conf = 0.0f;
                bool ok = false;
                if (j < a.nc) {
                    conf = rnd(__fmul_rn(ld_elem(a.pred, rb + 5 + j, a.dtype), obj), a.dtype);
                    ok = conf > a.thr && class_allowed(cls_mask, j);
                }
                const unsigned m = __ballot_sync(0xffffffffu, ok);
                f(ok, conf, static_cast<unsigned>(r) * a.nc + (ok ? j : 0), count, m);
                count += __popc(m);
            }
        }
    } else {
        // best class per row: maximum of the rounded products, first index on ties (torch.max).  Four passing rows are
        // handled per iteration, eight lanes each (ascending row order == ascending lane-group order, so ballot ranks stay
        // in candidate order); this cuts the dependent load rounds per segment by 4.
        const int sub = lane >> 3, sl = lane & 7;
        while (rows) {
            const unsigned rl = __fns(rows, 0, sub + 1);  // position of this group's row among the set bits (0xffffffff: none)
            const bool has = rl < 32u;
            float best = -INFINITY;
            int bj = 0x7fffffff;
            int r = 0;
            bool nan = false;  // torch.max propagates NaN: a row with any NaN product has a NaN best score and is dropped
            if (has) {
                r = row0 + static_cast<int>(rl);
                const long long rb = img_base + static_cast<long long>(r) * a.no;
                const float obj = ld_elem(a.pred, rb + 4, a.dtype);
                for (int j = sl; j < a.nc; j += 8) {
                    const float conf = rnd(__fmul_rn(ld_elem(a.pred, rb + 5 + j, a.dtype), obj), a.dtype);
                    nan |= isnan(conf);
                    if (bj == 0x7fffffff || conf > best) { best = conf; bj = j; }
                }
            }
#pragma unroll
            for (int o = 4; o > 0; o >>= 1) {  // reduce inside the 8-lane group
                const float ob = __shfl_xor_sync(0xffffffffu, best, o);
                const int oj = __shfl_xor_sync(0xffffffffu, bj, o);
                nan |= __shfl_xor_sync(0xffffffffu, static_cast<int>(nan), o) != 0;
                if (oj != 0x7fffffff && (bj == 0x7fffffff || ob > best || (ob == best && oj < bj))) { best = ob; bj = oj; }
            }
            const bool okrow = has && !nan && bj != 0x7fffffff && best > a.thr && class_allowed(cls_mask, bj);
            const bool ok = okrow && sl == 0;
            const unsigned m = __ballot_sync(0xffffffffu, ok);
            f(ok, best, static_cast<unsigned>(r) * a.nc + (okrow ? bj : 0), count, m);
            count += __popc(m);
#pragma unroll
            for (int q = 0; q < 4; ++q) rows &= rows - 1;  // drop the (up to) four rows just handled
        }
    }
    return count;
}

__device__ __forceinline__ void load_class_mask(const NmsArgs& a, unsigned* cls_mask) {
    const int words = (a.nc + 31) / 32;
    for (int w = threadIdx.x; w < words; w += blockDim.x) cls_mask[w] = a.classes ? 0u : 0xffffffffu;
    __syncthreads();
    if (a.classes)
        for (int i = threadIdx.x; i < a.n_classes; i += blockDim.x) {
            const int c = a.classes[i];
            if (c >= 0 && c < a.nc) atomicOr(&cls_mask[c >> 5], 1u << (c & 31));
        }
    __syncthreads();
}

// pass kinds: 0 count all, 1 histogram (hi or lo 16 bits), 2 count (> T, == T), 3 write selected
template <int KIND>
__global__ void nms_pass_kernel(const NmsArgs a, int level) {
    __shared__ unsigned cls_mask[kMaxClasses / 32];
    load_class_mask(a, cls_mask);
    const int b = blockIdx.y;
    const int seg = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (seg >= a.nseg) return;  // warp-uniform
    const int lane = threadIdx.x & 31;
    const unsigned lt = (1u << lane) - 1u;
    int* img = a.img + b * 8;
    const int sidx = b * a.nseg + seg;
    if (KIND == 0) {
        const int c = for_each_candidate(a, b, seg, cls_mask, [](bool, float, unsigned, int, unsigned) {});
        if (lane == 0) a.seg_cnt[sidx] = c;
        return;
    }
    const bool need_select = img[1] != 0;
    if (KIND == 1) {
        if (!need_select) return;
        unsigned* hist = a.hist + (static_cast<size_t>(b) * 2 + level) * 65536;
        const unsigned t_hi = static_cast<unsigned>(img[2]);
        for_each_candidate(a, b, seg, cls_mask, [&](bool ok, float s, unsigned, int, unsigned) {
            if (!ok) return;
            const unsigned u = __float_as_uint(s);
            if (level == 0) atomicAdd(&hist[u >> 16], 1u);
            else if ((u >> 16) == t_hi) atomicAdd(&hist[u & 0xffffu], 1u);
        });
        return;
    }
    if (KIND == 2) {
        if (!need_select) return;  // seg_cnt already holds the selected count (= all)
        const unsigned T = static_cast<unsigned>(img[4]);
        int gt = 0, eq = 0;  // warp-uniform (built from ballots)
        for_each_candidate(a, b, seg, cls_mask, [&](bool ok, float s, unsigned, int, unsigned) {
            const unsigned u = __float_as_uint(s);
            gt += __popc(__ballot_sync(0xffffffffu, ok && u > T));
            eq += __popc(__ballot_sync(0xffffffffu, ok && u == T));
        });
        if (lane == 0) { a.seg_cnt[sidx] = gt; a.seg_eq[sidx] = eq; }
        return;
    }
    if (KIND == 3) {
        const int base = a.seg_off[sidx];
        float* cs = a.cand_score + static_cast<size_t>(b) * kCandCap;
        unsigned* ci = a.cand_id + static_cast<size_t>(b) * kCandCap;
        if (!need_select) {
            for_each_candidate(a, b, seg, cls_mask, [&](bool ok, float s, unsigned id, int before, unsigned m) {
                const int pos = base + before + __popc(m & lt);
                if (ok && pos < kCandCap) { cs[pos] = s; ci[pos] = id; }
            });
            return;
        }
        // selected = score > T, or score == T and among the first need_eq such candidates in candidate order
        const unsigned T = static_cast<unsigned>(img[4]);
        const int eq_allowed = max(0, img[5] - a.seg_eq_off[sidx]);  // == T candidates this segment may still take
        int run_gt = 0, run_eq = 0;                                    // warp-uniform running counts
        for_each_candidate(a, b, seg, cls_mask, [&](bool ok, float s, unsigned id, int, unsigned) {
            const unsigned u = __float_as_uint(s);
            const bool is_gt = ok && u > T, is_eq = ok && u == T;
            const unsigned gt_m = __ballot_sync(0xffffffffu, is_gt);
            const unsigned eq_m = __ballot_sync(0xffffffffu, is_eq);
            const int gt_before = run_gt + __popc(gt_m & lt);
            const int eq_before = run_eq + __popc(eq_m & lt);
            if (is_gt || (is_eq && eq_before < eq_allowed)) {
                const int pos = base + gt_before + min(eq_before, eq_allowed);
                if (pos < kCandCap) { cs[pos] = s; ci[pos] = id; }
            }
            run_gt += __popc(gt_m);
            run_eq += __popc(eq_m);
        });
    }
}

// per image: exclusive scan over segments.  MODE 0: after pass 0 (decide selection); MODE 1: after pass 2.
template <int MODE>
__global__ void nms_scan_kernel(const NmsArgs a) {
    const int b = blockIdx.x;
    int* img = a.img + b * 8;
    __shared__ int part[1024];
    __shared__ int part2[1024];
    const int t = threadIdx.x, nt = blockDim.x;
    const int per = (a.nseg + nt - 1) / nt;
    const int s0 = t * per, s1 = min(a.nseg, s0 + per);
    if (MODE == 1 && img[1] == 0) return;
    int* cnt = a.seg_cnt + b * a.nseg;
    int* eqc = a.seg_eq + b * a.nseg;
    int sum = 0, sum2 = 0;
    for (int s = s0; s < s1; ++s) { sum += cnt[s]; if (MODE == 1) sum2 += eqc[s]; }
    part[t] = sum;
    part2[t] = sum2;
    __syncthreads();
    // Hillis-Steele inclusive scan over the per-thread partials
    for (int o = 1; o < nt; o <<= 1) {
        const int v = t >= o ? part[t - o] : 0;
        const int v2 = t >= o ? part2[t - o] : 0;
        __syncthreads();
        part[t] += v;
        part2[t] += v2;
        __syncthreads();
    }
    int run = part[t] - sum;      // exclusive prefix of (all | > T) counts
    int run2 = part2[t] - sum2;   // exclusive prefix of == T counts
    const int total = part[nt - 1];
    if (MODE == 0) {
        for (int s = s0; s < s1; ++s) { a.seg_off[b * a.nseg + s] = run; run += cnt[s]; }
        if (t == 0) {
            img[0] = total;
            img[1] = total > a.max_nms ? 1 : 0;
            img[6] = total > a.max_nms ? a.max_nms : total;
        }
        if (total > a.max_nms) {  // clear both histograms for the select passes
            unsigned* h = a.hist + static_cast<size_t>(b) * 2 * 65536;
            for (int i = t; i < 2 * 65536; i += nt) h[i] = 0u;
        }
    } else {
        // selected in segment = gt + clamp(need_eq - eq_before, 0, eq); offsets over the selected counts need a second
        // scan: do it serially per thread range after computing each thread's selected sum.
        const int need_eq = img[5];
        int sel_sum = 0;
        {
            int e = run2;
            for (int s = s0; s < s1; ++s) {
                const int take = max(0, min(eqc[s], need_eq - e));
                sel_sum += cnt[s] + take;
                e += eqc[s];
            }
        }
        __syncthreads();
        part[t] = sel_sum;
        __syncthreads();
        for (int o = 1; o < nt; o <<= 1) {
            const int v = t >= o ? part[t - o] : 0;
            __syncthreads();
            part[t] += v;
            __syncthreads();
        }
        int off = part[t] - sel_sum;
        int e = run2;
        for (int s = s0; s < s1; ++s) {
            a.seg_off[b * a.nseg + s] = off;
            a.seg_eq_off[b * a.nseg + s] = e;
            const int take = max(0, min(eqc[s], need_eq - e));
            off += cnt[s] + take;
            e += eqc[s];
        }
    }
}

// per image: walk the 65536-bin histogram from the top to find the bin holding the max_nms-th largest score
__global__ void nms_pick_kernel(const NmsArgs a, int level) {
    const int b = blockIdx.x;
    int* img = a.img + b * 8;
    if (img[1] == 0) return;
    const unsigned* hist = a.hist + (static_cast<size_t>(b) * 2 + level) * 65536;
    __shared__ unsigned part[1024];
    const int t = threadIdx.x;  // blockDim.x == 1024, 64 bins per thread, thread 0 owns the TOP bins
    const int hi_bin = 65535 - t * 64;
    unsigned sum = 0;
    for (int i = 0; i < 64; ++i) sum += hist[hi_bin - i];
    part[t] = sum;
    __syncthreads();
    for (int o = 1; o < 1024; o <<= 1) {
        const unsigned v = t >= o ? part[t - o] : 0;
        __syncthreads();
        part[t] += v;
        __syncthreads();
    }
    const unsigned before = part[t] - sum;  // candidates in bins above this thread's range
    const unsigned want = static_cast<unsigned>(level == 0 ? a.max_nms : a.max_nms - img[3]);  // rank to locate (1-based)
    if (before < want && before + sum >= want) {
        unsigned acc = before;
        for (int i = 0; i < 64; ++i) {
            const unsigned h = hist[hi_bin - i];
            if (acc + h >= want) {
                if (level == 0) { img[2] = hi_bin - i; img[3] = static_cast<int>(acc); }
                else {
                    img[4] = static_cast<int>((static_cast<unsigned>(img[2]) << 16) | static_cast<unsigned>(hi_bin - i));
                    img[5] = a.max_nms - (img[3] + static_cast<int>(acc));  // == T candidates to keep
                }
                break;
            }
            acc += h;
        }
    }
}

// per image: bitonic sort of (score desc, position asc) in shared memory, then materialise the sorted boxes
__global__ void nms_sort_kernel(const NmsArgs a) {
    extern __shared__ unsigned char sm[];
    const int b = blockIdx.x;
    const int n = min(a.img[b * 8 + 6], kCandCap);
    int P = 64;
    while (P < n) P <<= 1;
    unsigned* key = reinterpret_cast<unsigned*>(sm);
    unsigned short* pos = reinterpret_cast<unsigned short*>(sm + static_cast<size_t>(P) * 4);
    const float* cs = a.cand_score + static_cast<size_t>(b) * kCandCap;
    const unsigned* ci = a.cand_id + static_cast<size_t>(b) * kCandCap;
    if (n == 0) return;
    for (int i = threadIdx.x; i < P; i += blockDim.x) {
        key[i] = i < n ? __float_as_uint(cs[i]) : 0u;  // scores are > thr >= 0, so uint order == float order
        pos[i] = static_cast<unsigned short>(i < n ? i : 0xffff);
    }
    __syncthreads();
    for (int k = 2; k <= P; k <<= 1) {
        for (int j = k >> 1; j > 0; j >>= 1) {
            for (int i = threadIdx.x; i < P; i += blockDim.x) {
                const int l = i ^ j;
                if (l > i) {
                    const unsigned ki = key[i], kl = key[l];
                    const unsigned short pi = pos[i], pl = pos[l];
                    const bool i_first = ki > kl || (ki == kl && pi < pl);  // "i precedes l" in the target order
                    const bool up = (i & k) == 0;
                    if (up ? !i_first : i_first) { key[i] = kl; key[l] = ki; pos[i] = pl; pos[l] = pi; }
                }
            }
            __syncthreads();
        }
    }
    float4* sb = a.sorted_box + static_cast<size_t>(b) * kCandCap;
    unsigned* sid = a.sorted_id + static_cast<size_t>(b) * kCandCap;
    float* ssc = a.sorted_score + static_cast<size_t>(b) * kCandCap;
    const long long img_base = static_cast<long long>(b) * a.N * a.no;
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
        const unsigned id = ci[pos[i]];
        const unsigned r = id / a.nc, c = id - r * a.nc;
        const long long rb = img_base + static_cast<long long>(r) * a.no;
        const float cx = ld_elem(a.pred, rb + 0, a.dtype), cy = ld_elem(a.pred, rb + 1, a.dtype);
        const float hw = rnd(__fdiv_rn(ld_elem(a.pred, rb + 2, a.dtype), 2.0f), a.dtype);
        const float hh = rnd(__fdiv_rn(ld_elem(a.pred, rb + 3, a.dtype), 2.0f), a.dtype);
        const float off = a.agnostic ? __fmul_rn(static_cast<float>(c), 0.0f) : __fmul_rn(static_cast<float>(c), a.max_wh);
        float4 bx;
        bx.x = __fadd_rn(rnd(__fsub_rn(cx, hw), a.dtype), off);
        bx.y = __fadd_rn(rnd(__fsub_rn(cy, hh), a.dtype), off);
        bx.z = __fadd_rn(rnd(__fadd_rn(cx, hw), a.dtype), off);
        bx.w = __fadd_rn(rnd(__fadd_rn(cy, hh), a.dtype), off);
        sb[i] = bx;
        sid[i] = id;
        ssc[i] = __uint_as_float(key[i]);
    }
}

__device__ __forceinline__ bool iou_gt(const float4& p, float parea, const float4& q, float thr) {
    const float xx1 = fmaxf(p.x, q.x), yy1 = fmaxf(p.y, q.y);
    const float xx2 = fminf(p.z, q.z), yy2 = fminf(p.w, q.w);
    const float w = fmaxf(0.0f, __fsub_rn(xx2, xx1)), h = fmaxf(0.0f, __fsub_rn(yy2, yy1));
    const float inter = __fmul_rn(w, h);
    const float qarea = __fmul_rn(__fsub_rn(q.z, q.x), __fsub_rn(q.w, q.y));
    const float ovr = __fdiv_rn(inter, __fsub_rn(__fadd_rn(parea, qarea), inter));
    return ovr > thr;  // NaN -> false: never suppresses
}

constexpr int kChunk = 64;
constexpr int kGreedyThreads = 1024;               // 16 threads per candidate of a chunk
constexpr int kParts = kGreedyThreads / kChunk;    // 16

// per image greedy suppression over the sorted candidates + output
__global__ void __launch_bounds__(kGreedyThreads) nms_greedy_kernel(const NmsArgs a) {
    extern __shared__ unsigned char sm[];
    float4* kept_box = reinterpret_cast<float4*>(sm);                                  // [max_det]
    int* kept_pos = reinterpret_cast<int*>(sm + static_cast<size_t>(a.max_det) * 16);  // [max_det]
    __shared__ unsigned long long mask[kChunk];
    __shared__ unsigned alive_w[2];
    __shared__ int n_kept_s;
    const int b = blockIdx.x;
    const int n = min(a.img[b * 8 + 6], kCandCap);
    const float4* sb = a.sorted_box + static_cast<size_t>(b) * kCandCap;
    const int t = threadIdx.x;
    if (t == 0) n_kept_s = 0;
    __syncthreads();
    const int ci = t & (kChunk - 1);   // candidate within chunk
    const int part = t >> 6;           // 0..15
    for (int c0 = 0; c0 < n; c0 += kChunk) {
        const int n_kept = n_kept_s;
        if (n_kept >= a.max_det) break;
        if (t < kChunk) mask[t] = 0ull;
        if (t < 2) alive_w[t] = 0xffffffffu;
        __syncthreads();
        const int idx = c0 + ci;
        const bool in_range = idx < n;
        float4 me = make_float4(0.f, 0.f, 0.f, 0.f);
        if (in_range) me = sb[idx];
        // (1) against the kept list: kept box i suppresses me when IoU(kept_i, me) > thr
        bool dead = false;
        if (in_range) {
            for (int k = part; k < n_kept && !dead; k += kParts) {
                const float4 kb = kept_box[k];
                const float karea = __fmul_rn(__fsub_rn(kb.z, kb.x), __fsub_rn(kb.w, kb.y));
                dead = iou_gt(kb, karea, me, a.iou_thr);
            }
        }
        if (dead || (!in_range && part == 0)) atomicAnd(&alive_w[ci >> 5], ~(1u << (ci & 31)));
        // (2) pairwise inside the chunk: bit j of mask[i] set when earlier candidate j (j < i) would suppress i
        if (in_range) {
            unsigned long long m = 0ull;
            const int j0 = part * (kChunk / kParts);
            for (int j = j0; j < j0 + kChunk / kParts && j < ci; ++j) {
                const float4 ob = sb[c0 + j];
                const float oarea = __fmul_rn(__fsub_rn(ob.z, ob.x), __fsub_rn(ob.w, ob.y));
                if (iou_gt(ob, oarea, me, a.iou_thr)) m |= 1ull << j;
            }
            if (m) atomicOr(&mask[ci], m);
        }
        __syncthreads();
        // (3) serial resolve inside warp 0: lane l holds the masks of candidates l and l+32; every lane runs the same
        // 64-step recurrence on broadcast values (registers + shuffles only)
        if (t < 32) {
            const unsigned long long m_lo = mask[t], m_hi = mask[t + 32];
            const unsigned long long alive = static_cast<unsigned long long>(alive_w[0]) | (static_cast<unsigned long long>(alive_w[1]) << 32);
            unsigned long long keptbits = 0ull;
            int nk = n_kept;
#pragma unroll 8
            for (int i = 0; i < kChunk; ++i) {
                const unsigned long long mi = __shfl_sync(0xffffffffu, i < 32 ? m_lo : m_hi, i & 31);
                if (((alive >> i) & 1ull) && (mi & keptbits) == 0ull && nk < a.max_det) {
                    keptbits |= 1ull << i;
                    ++nk;
                }
            }
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int i = t + 32 * h;
                if ((keptbits >> i) & 1ull) kept_pos[n_kept + __popcll(keptbits & ((1ull << i) - 1ull))] = c0 + i;
            }
            if (t == 0) n_kept_s = nk;
        }
        __syncthreads();
        const int nk2 = n_kept_s;
        for (int k = n_kept + t; k < nk2; k += blockDim.x) kept_box[k] = sb[kept_pos[k]];
        __syncthreads();
    }
    __syncthreads();
    // output rows: [x1,y1,x2,y2 (input-dtype rounding, no class offset), conf, cls, masks*obj]
    const int nk = n_kept_s;
    if (t == 0) a.out_count[b] = nk;
    const int width = 6 + a.nm;
    const unsigned* sid = a.sorted_id + static_cast<size_t>(b) * kCandCap;
    const float* ssc = a.sorted_score + static_cast<size_t>(b) * kCandCap;
    const long long img_base = static_cast<long long>(b) * a.N * a.no;
    for (int e = t; e < nk * width; e += blockDim.x) {
        const int k = e / width, col = e - k * width;
        const int p = kept_pos[k];
        const unsigned id = sid[p];
        const unsigned r = id / a.nc, c = id - r * a.nc;
        const long long rb = img_base + static_cast<long long>(r) * a.no;
        float v;
        if (col < 4) {
            const float ctr = ld_elem(a.pred, rb + (col & 1), a.dtype);
            const float half = rnd(__fdiv_rn(ld_elem(a.pred, rb + 2 + (col & 1), a.dtype), 2.0f), a.dtype);
            v = rnd(col < 2 ? __fsub_rn(ctr, half) : __fadd_rn(ctr, half), a.dtype);
        } else if (col == 4) v = ssc[p];
        else if (col == 5) v = static_cast<float>(c);
        else v = rnd(__fmul_rn(ld_elem(a.pred, rb + 5 + a.nc + (col - 6), a.dtype), ld_elem(a.pred, rb + 4, a.dtype)), a.dtype);
        a.out_rows[(static_cast<size_t>(b) * a.max_det + k) * width + col] = v;
        if (col == 0) a.out_idx[static_cast<size_t>(b) * a.max_det + k] = static_cast<long long>(id);
    }
}

__global__ void box_iou_kernel(const float* __restrict__ A, int n, const float* __restrict__ Bx, int m, float eps, float* out) {
    const long long total = static_cast<long long>(n) * m;
    for (long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; idx < total;
         idx += static_cast<long long>(gridDim.x) * blockDim.x) {
        const int i = static_cast<int>(idx / m), j = static_cast<int>(idx - static_cast<long long>(i) * m);
        const float4 p = reinterpret_cast<const float4*>(A)[i];
        const float4 q = reinterpret_cast<const float4*>(Bx)[j];
        const float a1 = __fmul_rn(__fsub_rn(p.z, p.x), __fsub_rn(p.w, p.y));
        const float a2 = __fmul_rn(__fsub_rn(q.z, q.x), __fsub_rn(q.w, q.y));
        const float w = fmaxf(__fsub_rn(fminf(p.z, q.z), fmaxf(p.x, q.x)), 0.0f);
        const float h = fmaxf(__fsub_rn(fminf(p.w, q.w), fmaxf(p.y, q.y)), 0.0f);
        const float inter = __fmul_rn(w, h);
        out[idx] = __fdiv_rn(inter, __fadd_rn(__fsub_rn(__fadd_rn(a1, a2), inter), eps));
    }
}

}  // namespace y5

using namespace y5;

namespace {
struct WsLayout {
    size_t seg_cnt, seg_eq, seg_off, seg_eq_off, img, hist, cand_score, cand_id, sorted_box, sorted_id, sorted_score, total;
};
WsLayout ws_layout(int B, int nseg) {
    WsLayout L;
    size_t o = 0;
    auto take = [&](size_t bytes) { size_t r = o; o += (bytes + 255) & ~size_t(255); return r; };
    L.seg_cnt = take(sizeof(int) * B * nseg);
    L.seg_eq = take(sizeof(int) * B * nseg);
    L.seg_off = take(sizeof(int) * B * nseg);
    L.seg_eq_off = take(sizeof(int) * B * nseg);
    L.img = take(sizeof(int) * B * 8);
    L.hist = take(sizeof(unsigned) * B * 2 * 65536);
    L.cand_score = take(sizeof(float) * B * kCandCap);
    L.cand_id = take(sizeof(unsigned) * B * kCandCap);
    L.sorted_box = take(sizeof(float4) * B * kCandCap);
    L.sorted_id = take(sizeof(unsigned) * B * kCandCap);
    L.sorted_score = take(sizeof(float) * B * kCandCap);
    L.total = o;
    return L;
}
int validate_nms(const y5_nms_params* p) {
    if (!p) return set_error(Y5_E_INVALID, "nms: null params");
    if (p->batch <= 0 || p->n_rows <= 0 || p->nc <= 0 || p->nm < 0 || p->no != 5 + p->nc + p->nm)
        return set_error(Y5_E_INVALID, "nms: inconsistent shape (batch %d rows %d no %d nc %d nm %d)", p->batch, p->n_rows, p->no, p->nc, p->nm);
    if (p->dtype != Y5_F16 && p->dtype != Y5_BF16 && p->dtype != Y5_F32) return set_error(Y5_E_UNSUPPORTED, "nms: dtype");
    if (!(p->conf_thres >= 0.f && p->conf_thres <= 1.f) || !(p->iou_thres >= 0.f && p->iou_thres <= 1.f))
        return set_error(Y5_E_INVALID, "nms: thresholds must be in [0,1]");  // reference asserts, utils/general.py:675-676
    if (p->max_det <= 0 || p->max_det > kMaxDetCap) return set_error(Y5_E_UNSUPPORTED, "nms: max_det must be in [1,%d]", kMaxDetCap);
    if (p->max_nms <= 0 || p->max_nms > kCandCap) return set_error(Y5_E_UNSUPPORTED, "nms: max_nms must be in [1,%d]", kCandCap);
    if (p->nc > kMaxClasses) return set_error(Y5_E_UNSUPPORTED, "nms: more than %d classes", kMaxClasses);
    if (static_cast<long long>(p->n_rows) * p->nc > 0xffffffffLL) return set_error(Y5_E_UNSUPPORTED, "nms: rows*nc exceeds 2^32");
    if (p->batch > 65535) return set_error(Y5_E_UNSUPPORTED, "nms: batch > 65535");
    return 0;
}
float round_thr_to_dtype(float t, int dtype) {
    if (dtype == Y5_F16) return __half2float(__float2half_rn(t));
    if (dtype == Y5_BF16) return __bfloat162float(__float2bfloat16_rn(t));
    return t;
}
}  // namespace

extern "C" Y5_API int64_t y5_nms_workspace_bytes(const y5_nms_params* p) {
    if (validate_nms(p)) return -1;
    return static_cast<int64_t>(ws_layout(p->batch, (p->n_rows + kSegRows - 1) / kSegRows).total);
}

extern "C" Y5_API int y5_nms_batched(const y5_nms_params* p, const void* pred, float* out_rows, int64_t* out_idx, int32_t* out_count,
                              void* workspace, int64_t workspace_bytes, void* stream) {
    if (int e = validate_nms(p)) return e;
    if (!pred || !out_rows || !out_idx || !out_count || !workspace) return set_error(Y5_E_INVALID, "nms: null pointer");
    const int nseg = (p->n_rows + kSegRows - 1) / kSegRows;
    const WsLayout L = ws_layout(p->batch, nseg);
    if (workspace_bytes < static_cast<int64_t>(L.total)) return set_error(Y5_E_INVALID, "nms: workspace too small (%lld < %zu)", (long long)workspace_bytes, L.total);
    if (reinterpret_cast<uintptr_t>(workspace) & 255) return set_error(Y5_E_INVALID, "nms: workspace must be 256-byte aligned");
    unsigned char* ws = static_cast<unsigned char*>(workspace);
    NmsArgs a{};
    a.pred = pred;
    a.B = p->batch; a.N = p->n_rows; a.no = p->no; a.nc = p->nc; a.nm = p->nm; a.dtype = p->dtype;
    a.thr = round_thr_to_dtype(p->conf_thres, p->dtype);
    // torchvision's CPU kernel evaluates (float ratio) > (double threshold): equivalent float threshold = largest float
    // not above the double value.  The caller passes the python float narrowed to fp32, so recover the double rule from
    // the decimal the user most plausibly meant is impossible here; the Python binding passes iou_thres already adjusted
    // (see yolov5_b200/utils/general.py::_iou_threshold_f32) and we use it verbatim.
    a.iou_thr = p->iou_thres;
    a.multi_label = (p->multi_label && p->nc > 1) ? 1 : 0;  // reference :693
    a.agnostic = p->agnostic; a.max_det = p->max_det; a.max_nms = p->max_nms; a.max_wh = p->max_wh;
    a.classes = p->n_classes > 0 ? p->classes : nullptr; a.n_classes = p->n_classes;
    a.nseg = nseg;
    a.seg_cnt = reinterpret_cast<int*>(ws + L.seg_cnt);
    a.seg_eq = reinterpret_cast<int*>(ws + L.seg_eq);
    a.seg_off = reinterpret_cast<int*>(ws + L.seg_off);
    a.seg_eq_off = reinterpret_cast<int*>(ws + L.seg_eq_off);
    a.img = reinterpret_cast<int*>(ws + L.img);
    a.hist = reinterpret_cast<unsigned*>(ws + L.hist);
    a.cand_score = reinterpret_cast<float*>(ws + L.cand_score);
    a.cand_id = reinterpret_cast<unsigned*>(ws + L.cand_id);
    a.sorted_box = reinterpret_cast<float4*>(ws + L.sorted_box);
    a.sorted_id = reinterpret_cast<unsigned*>(ws + L.sorted_id);
    a.sorted_score = reinterpret_cast<float*>(ws + L.sorted_score);
    a.out_rows = out_rows; a.out_idx = reinterpret_cast<long long*>(out_idx); a.out_count = out_count;

    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const int threads = 256, wpb = threads / 32;
    dim3 grid((nseg + wpb - 1) / wpb, p->batch);
    if (ensure_dyn_smem(reinterpret_cast<const void*>(nms_sort_kernel), kCandCap * 6) != cudaSuccess ||
        ensure_dyn_smem(reinterpret_cast<const void*>(nms_greedy_kernel), kMaxDetCap * 20) != cudaSuccess)
        return set_error(Y5_E_DRIVER, "nms: cudaFuncSetAttribute(MaxDynamicSharedMemorySize) failed");
    nms_pass_kernel<0><<<grid, threads, 0, st>>>(a, 0);
    nms_scan_kernel<0><<<p->batch, 1024, 0, st>>>(a);
    int launches = 2;
    const long long max_cands = a.multi_label ? static_cast<long long>(p->n_rows) * p->nc : p->n_rows;
    if (max_cands > p->max_nms) {  // the cut can only trigger when more candidates than max_nms are possible at all
        nms_pass_kernel<1><<<grid, threads, 0, st>>>(a, 0);
        nms_pick_kernel<<<p->batch, 1024, 0, st>>>(a, 0);
        nms_pass_kernel<1><<<grid, threads, 0, st>>>(a, 1);
        nms_pick_kernel<<<p->batch, 1024, 0, st>>>(a, 1);
        nms_pass_kernel<2><<<grid, threads, 0, st>>>(a, 0);
        nms_scan_kernel<1><<<p->batch, 1024, 0, st>>>(a);
        launches += 6;
    }
    nms_pass_kernel<3><<<grid, threads, 0, st>>>(a, 0);
    nms_sort_kernel<<<p->batch, 1024, kCandCap * 6, st>>>(a);
    nms_greedy_kernel<<<p->batch, kGreedyThreads, static_cast<size_t>(p->max_det) * 20, st>>>(a);
    launches += 3;
    count_launch(launches);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return set_error(int(e), "nms launch failed: %s", cudaGetErrorString(e));
    return 0;
}

extern "C" Y5_API int y5_box_iou(const float* a, int32_t n, const float* b, int32_t m, float eps, float* out, void* stream) {
    if (n < 0 || m < 0 || (n > 0 && m > 0 && (!a || !b || !out))) return set_error(Y5_E_INVALID, "box_iou: bad arguments");
    if (n == 0 || m == 0) return 0;
    if ((reinterpret_cast<uintptr_t>(a) & 15) || (reinterpret_cast<uintptr_t>(b) & 15)) return set_error(Y5_E_INVALID, "box_iou: boxes must be 16-byte aligned");
    const long long total = static_cast<long long>(n) * m;
    const int threads = 256;
    long long blocks = (total + threads - 1) / threads;
    if (blocks > sm_count() * 16) blocks = sm_count() * 16;
    box_iou_kernel<<<static_cast<int>(blocks), threads, 0, static_cast<cudaStream_t>(stream)>>>(a, n, b, m, eps, out);
    count_launch();
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return set_error(int(e), "box_iou launch failed: %s", cudaGetErrorString(e));
    return 0;
}
