// ComputeLoss on the device: build_targets (index work, bit-exact and ordered like the reference) and the fused
// gather + CIoU + objectness scatter + BCE forward/backward.  Replaces reference utils/loss.py:134-247.
//
//   1 zero        clear the dense objectness-target planes and counters
//   2 targets     one CTA per level: enumerate (offset k, anchor a, target t) in the reference's order, apply the
//                 anchor-ratio test and the 5-neighbour rule, ordered compaction -> (b, a, gj, gi, cls), tbox
//   3 match       per match: gather 4 box logits, CIoU + its gradient (forward-mode duals), deterministic
//                 last-writer-wins scatter of clamp(iou,0) into the objectness target (64-bit atomicMax on
//                 (match order, value)), per-block partial sums of (1 - iou)
//   4 dense       flat pass over every logit: objectness BCE (partials) and, if requested, the full gradient tensor
//                 (zeros + objectness gradient)
//   5 cls         warp per match: class BCE (partials); adds box + class gradients into the gradient tensor
//   6 finalize    fixed-order reduction of the partials, gains, `* batch` -> out_loss[4]
// Index arithmetic uses explicit _rn intrinsics and the file is compiled with -fmad=false, so the fp32 compares
// that decide the match set round exactly like the reference's separate torch ops.
#include <math.h>

#include "../../include/y5b200.h"
#include "common.cuh"
#include "host_util.h"

namespace y5 {

constexpr int kMaxLevels = 5;
constexpr int kPartials = 256;  // per level partial-sum slots (fixed -> deterministic final reduction)

struct LossArgs {
    int nl, B, na, no, nc, dtype, nt;
    int ny[kMaxLevels], nx[kMaxLevels];
    const void* p[kMaxLevels];
    void* grad[kMaxLevels];
    const float* targets;
    const float* anchors;
    float anchor_t, box_gain, obj_gain, cls_gain, cls_pw, obj_pw, cp, cn, grad_scale;
    const float* grad_scale_dev;              // optional upstream gradient of the loss (device scalar), multiplied in fp32
    float balance[kMaxLevels];
    int cap;                                  // matches capacity per level = 5*na*nt
    int* count;                               // [nl]
    int* midx;                                // [nl][5][cap]  b, a, gj, gi, cls
    float4* tbox;                             // [nl][cap]
    float4* bgrad;                            // [nl][cap]     d(1-ciou)/d(box logits)
    unsigned long long* tobj[kMaxLevels];     // dense (B,na,ny,nx): (order+1)<<32 | float bits
    long long cells[kMaxLevels];              // B*na*ny*nx
    float* part_box;                          // [nl][kPartials]
    float* part_obj;                          // [nl][kPartials]
    float* part_cls;                          // [nl][kPartials]
    float* out_loss;
    int* trow;                                // optional [nl][cap]: target row of each match (segmentation loss)
};

__device__ __forceinline__ float ldp(const void* base, long long i, int dtype) {
    if (dtype == Y5_F32) return reinterpret_cast<const float*>(base)[i];
    return unpack1(reinterpret_cast<const uint16_t*>(base)[i], dtype == Y5_BF16);
}
__device__ __forceinline__ float rnd_dt(float x, int dtype) {
    if (dtype == Y5_F32) return x;
    return unpack1(pack1(x, dtype == Y5_BF16), dtype == Y5_BF16);
}
__device__ __forceinline__ void stg(void* base, long long i, float v, int dtype) {
    if (dtype == Y5_F32) reinterpret_cast<float*>(base)[i] = v;
    else reinterpret_cast<uint16_t*>(base)[i] = pack1(v, dtype == Y5_BF16);
}
__device__ __forceinline__ void atomic_add_elem(void* base, long long i, float v, int dtype) {
    if (dtype == Y5_F32) atomicAdd(reinterpret_cast<float*>(base) + i, v);
    else if (dtype == Y5_F16) atomicAdd(reinterpret_cast<__half*>(base) + i, __float2half_rn(v));
    else atomicAdd(reinterpret_cast<__nv_bfloat16*>(base) + i, __float2bfloat16_rn(v));
}

__global__ void loss_zero_kernel(LossArgs a) {
    const long long stride = static_cast<long long>(gridDim.x) * blockDim.x;
    const long long tid = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
    for (int l = 0; l < a.nl; ++l)
        for (long long i = tid; i < a.cells[l]; i += stride) a.tobj[l][i] = 0ull;
    if (tid < a.nl) a.count[tid] = 0;
}

// ---------------------------------------------------------------------------------------------------------------------
// build_targets: reference utils/loss.py:185-247
// ---------------------------------------------------------------------------------------------------------------------
__global__ void loss_targets_kernel(LossArgs a) {
    const int l = blockIdx.x;
    const int nx = a.nx[l], ny = a.ny[l];
    const int total = 5 * a.na * a.nt;
    __shared__ int warp_cnt[32];
    __shared__ int base_s;
    if (threadIdx.x == 0) base_s = 0;
    __syncthreads();
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
    int* mi = a.midx + static_cast<size_t>(l) * 5 * a.cap;
    float4* tb = a.tbox + static_cast<size_t>(l) * a.cap;
    const float fnx = static_cast<float>(nx), fny = static_cast<float>(ny);
    for (int c0 = 0; c0 < total; c0 += blockDim.x) {
        const int c = c0 + threadIdx.x;
        bool ok = false;
        int b = 0, cls = 0, an = 0, gi = 0, gj = 0, t = 0;
        float gx = 0, gy = 0, gw = 0, gh = 0;
        if (c < total) {
            const int k = c / (a.na * a.nt);
            const int rem = c - k * (a.na * a.nt);
            an = rem / a.nt;
            t = rem - an * a.nt;
            const float* tg = a.targets + static_cast<size_t>(t) * 6;
            // t = targets * gain  (gain = [1,1,nx,ny,nx,ny,1]); image / class columns are multiplied by 1.0
            gx = __fmul_rn(tg[2], fnx); gy = __fmul_rn(tg[3], fny);
            gw = __fmul_rn(tg[4], fnx); gh = __fmul_rn(tg[5], fny);
            const float aw = a.anchors[(l * a.na + an) * 2], ah = a.anchors[(l * a.na + an) * 2 + 1];
            const float rw = __fdiv_rn(gw, aw), rh = __fdiv_rn(gh, ah);
            const float mw = fmaxf(rw, __fdiv_rn(1.0f, rw)), mh = fmaxf(rh, __fdiv_rn(1.0f, rh));
            ok = fmaxf(mw, mh) < a.anchor_t;                                                         // :219-220
            float ox = 0.f, oy = 0.f;
            if (ok && k > 0) {
                const float gxi = __fsub_rn(fnx, gx), gyi = __fsub_rn(fny, gy);
                if (k == 1) { ok = fmodf(gx, 1.0f) < 0.5f && gx > 1.0f; ox = 0.5f; }               // j  -> ( .5, 0)
                else if (k == 2) { ok = fmodf(gy, 1.0f) < 0.5f && gy > 1.0f; oy = 0.5f; }          // k  -> (0,  .5)
                else if (k == 3) { ok = fmodf(gxi, 1.0f) < 0.5f && gxi > 1.0f; ox = -0.5f; }       // l  -> (-.5, 0)
                else { ok = fmodf(gyi, 1.0f) < 0.5f && gyi > 1.0f; oy = -0.5f; }                   // m  -> (0, -.5)
            }
            if (ok) {
                b = static_cast<int>(tg[0]);    // .long(): truncation
                cls = static_cast<int>(tg[1]);
                // the reference raises IndexError for an image index >= batch or a class >= nc; a kernel cannot, and must
                // not write out of bounds: such rows are ignored
                if (b < 0 || b >= a.B || cls < 0 || cls >= a.nc) ok = false;
                const int ix = static_cast<int>(__fsub_rn(gx, ox)), iy = static_cast<int>(__fsub_rn(gy, oy));
                gi = min(max(ix, 0), nx - 1);   // clamp_ aliases gij (:242), so tbox below uses the clamped cell
                gj = min(max(iy, 0), ny - 1);
            }
        }
        // ordered compaction across the block
        const unsigned m = __ballot_sync(0xffffffffu, ok);
        if (lane == 0) warp_cnt[warp] = __popc(m);
        __syncthreads();
        int before = base_s;
        for (int w = 0; w < warp; ++w) before += warp_cnt[w];
        if (ok) {
            const int pos = before + __popc(m & ((1u << lane) - 1u));
            mi[0 * a.cap + pos] = b; mi[1 * a.cap + pos] = an; mi[2 * a.cap + pos] = gj; mi[3 * a.cap + pos] = gi;
            mi[4 * a.cap + pos] = cls;
            tb[pos] = make_float4(__fsub_rn(gx, static_cast<float>(gi)), __fsub_rn(gy, static_cast<float>(gj)), gw, gh);
            if (a.trow) a.trow[static_cast<size_t>(l) * a.cap + pos] = t;
        }
        __syncthreads();
        if (threadIdx.x == 0) {
            int s = base_s;
            for (int w = 0; w < nwarps; ++w) s += warp_cnt[w];
            base_s = s;
        }
        __syncthreads();
    }
    if (threadIdx.x == 0) a.count[l] = base_s;
}

// ---------------------------------------------------------------------------------------------------------------------
// forward-mode dual numbers over the 4 box parameters (x, y, w, h) of the prediction
// ---------------------------------------------------------------------------------------------------------------------
struct D4 {
    float v, d[4];
};
__device__ __forceinline__ D4 dconst(float v) { return {v, {0.f, 0.f, 0.f, 0.f}}; }
__device__ __forceinline__ D4 dvar(float v, int i) { D4 r = dconst(v); r.d[i] = 1.f; return r; }
__device__ __forceinline__ D4 operator+(const D4& a, const D4& b) { D4 r; r.v = a.v + b.v; for (int i = 0; i < 4; ++i) r.d[i] = a.d[i] + b.d[i]; return r; }
__device__ __forceinline__ D4 operator-(const D4& a, const D4& b) { D4 r; r.v = a.v - b.v; for (int i = 0; i < 4; ++i) r.d[i] = a.d[i] - b.d[i]; return r; }
__device__ __forceinline__ D4 operator*(const D4& a, const D4& b) { D4 r; r.v = a.v * b.v; for (int i = 0; i < 4; ++i) r.d[i] = a.d[i] * b.v + a.v * b.d[i]; return r; }
__device__ __forceinline__ D4 operator/(const D4& a, const D4& b) { D4 r; r.v = a.v / b.v; const float inv = 1.0f / b.v; for (int i = 0; i < 4; ++i) r.d[i] = (a.d[i] - r.v * b.d[i]) * inv; return r; }
__device__ __forceinline__ D4 dscale(const D4& a, float s) { D4 r; r.v = a.v * s; for (int i = 0; i < 4; ++i) r.d[i] = a.d[i] * s; return r; }
// torch.minimum / maximum backward: the gradient goes to the selected operand, and on a tie half to each
// (a predicted box equal to its target, e.g. logits 0 on an anchor-sized target, ties every edge)
__device__ __forceinline__ D4 dtie(const D4& a, const D4& b) { D4 r; r.v = a.v; for (int i = 0; i < 4; ++i) r.d[i] = 0.5f * (a.d[i] + b.d[i]); return r; }
__device__ __forceinline__ D4 dmin(const D4& a, const D4& b) { return a.v < b.v ? a : b.v < a.v ? b : dtie(a, b); }
__device__ __forceinline__ D4 dmax(const D4& a, const D4& b) { return a.v > b.v ? a : b.v > a.v ? b : dtie(a, b); }
// clamp(min=0) backward passes the gradient where v >= 0 (touching boxes: intersection width exactly 0)
__device__ __forceinline__ D4 dclamp0(const D4& a) { return a.v >= 0.f ? a : dconst(0.f); }
__device__ __forceinline__ D4 datan(const D4& a) { D4 r; r.v = atanf(a.v); const float g = 1.0f / (1.0f + a.v * a.v); for (int i = 0; i < 4; ++i) r.d[i] = a.d[i] * g; return r; }

// CIoU(pred xywh, target xywh), eps 1e-7  (ultralytics bbox_iou, SURVEY.md Appendix C); alpha is a constant (no_grad)
__device__ __forceinline__ D4 ciou_dual(float px, float py, float pw, float ph, const float4& t) {
    const float eps = 1e-7f;
    const D4 x1 = dvar(px, 0), y1 = dvar(py, 1), w1 = dvar(pw, 2), h1 = dvar(ph, 3);
    const D4 x2 = dconst(t.x), y2 = dconst(t.y), w2 = dconst(t.z), h2 = dconst(t.w);
    const D4 hw1 = dscale(w1, 0.5f), hh1 = dscale(h1, 0.5f), hw2 = dscale(w2, 0.5f), hh2 = dscale(h2, 0.5f);
    const D4 b1x1 = x1 - hw1, b1x2 = x1 + hw1, b1y1 = y1 - hh1, b1y2 = y1 + hh1;
    const D4 b2x1 = x2 - hw2, b2x2 = x2 + hw2, b2y1 = y2 - hh2, b2y2 = y2 + hh2;
    const D4 inter = dclamp0(dmin(b1x2, b2x2) - dmax(b1x1, b2x1)) * dclamp0(dmin(b1y2, b2y2) - dmax(b1y1, b2y1));
    const D4 uni = w1 * h1 + w2 * h2 - inter + dconst(eps);
    const D4 iou = inter / uni;
    const D4 cw = dmax(b1x2, b2x2) - dmin(b1x1, b2x1);
    const D4 ch = dmax(b1y2, b2y2) - dmin(b1y1, b2y1);
    const D4 c2 = cw * cw + ch * ch + dconst(eps);
    const D4 dx = b2x1 + b2x2 - b1x1 - b1x2, dy = b2y1 + b2y2 - b1y1 - b1y2;
    const D4 rho2 = dscale(dx * dx + dy * dy, 0.25f);
    const D4 da = datan(w2 / h2) - datan(w1 / h1);
    const D4 v = dscale(da * da, 0.40528473456935108578f);  // 4 / pi^2
    const float alpha = v.v / (v.v - iou.v + (1.0f + eps));
    return iou - (rho2 / c2 + dscale(v, alpha));
}

__global__ void loss_match_kernel(LossArgs a) {
    const int l = blockIdx.y;
    const int n = a.count[l];
    const int nx = a.nx[l], ny = a.ny[l];
    const int* mi = a.midx + static_cast<size_t>(l) * 5 * a.cap;
    const float4* tb = a.tbox + static_cast<size_t>(l) * a.cap;
    float4* bg = a.bgrad + static_cast<size_t>(l) * a.cap;
    float local = 0.0f;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const int b = mi[i], an = mi[a.cap + i], gj = mi[2 * a.cap + i], gi = mi[3 * a.cap + i];
        const long long cell = ((static_cast<long long>(b) * a.na + an) * ny + gj) * nx + gi;
        const long long e = cell * a.no;
        const float s0 = sigmoid_f(ldp(a.p[l], e + 0, a.dtype)), s1 = sigmoid_f(ldp(a.p[l], e + 1, a.dtype));
        const float s2 = sigmoid_f(ldp(a.p[l], e + 2, a.dtype)), s3 = sigmoid_f(ldp(a.p[l], e + 3, a.dtype));
        const float aw = a.anchors[(l * a.na + an) * 2], ah = a.anchors[(l * a.na + an) * 2 + 1];
        const float px = s0 * 2.0f - 0.5f, py = s1 * 2.0f - 0.5f;                    // :148
        const float pw = (s2 * 2.0f) * (s2 * 2.0f) * aw, ph = (s3 * 2.0f) * (s3 * 2.0f) * ah;  // :149
        const D4 ci = ciou_dual(px, py, pw, ph, tb[i]);
        local += 1.0f - ci.v;
        // d(1 - ciou)/d logit = -dciou/dbox * dbox/dlogit
        float4 g;
        g.x = -ci.d[0] * 2.0f * s0 * (1.0f - s0);
        g.y = -ci.d[1] * 2.0f * s1 * (1.0f - s1);
        g.z = -ci.d[2] * 8.0f * s2 * s2 * (1.0f - s2) * aw;
        g.w = -ci.d[3] * 8.0f * s3 * s3 * (1.0f - s3) * ah;
        bg[i] = g;
        // tobj[b,a,gj,gi] = iou.detach().clamp(0).type(tobj.dtype)   (:155-160); duplicates: highest match index wins
        const float tv = rnd_dt(fmaxf(ci.v, 0.0f), a.dtype);
        const unsigned long long key = (static_cast<unsigned long long>(i + 1) << 32) | __float_as_uint(tv);
        atomicMax(a.tobj[l] + cell, key);
    }
    // deterministic block sum -> partial slot
    __shared__ float red[32];
    for (int o = 16; o > 0; o >>= 1) local += __shfl_xor_sync(0xffffffffu, local, o);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = local;
    __syncthreads();
    if (threadIdx.x == 0) {
        float s = 0.f;
        for (int w = 0; w < (blockDim.x >> 5); ++w) s += red[w];
        a.part_box[l * kPartials + blockIdx.x] = s;
    }
}

__device__ __forceinline__ float bce_logits(float x, float t, float pw) {
    // torch.nn.functional.binary_cross_entropy_with_logits with pos_weight
    const float lw = 1.0f + (pw - 1.0f) * t;
    return (1.0f - t) * x + lw * (log1pf(expf(-fabsf(x))) + fmaxf(-x, 0.0f));
}
__device__ __forceinline__ float bce_logits_grad(float x, float t, float pw) {
    const float lw = 1.0f + (pw - 1.0f) * t;
    return (1.0f - t) - lw * (1.0f - sigmoid_f(x));
}

__global__ void loss_dense_kernel(LossArgs a) {
    const int l = blockIdx.y;
    const long long total = a.cells[l] * a.no;
    // d(loss*bs*grad_scale)/d obj logit = obj_gain * balance / cells * bs * grad_scale * dBCE
    const float up = a.grad_scale_dev ? *a.grad_scale_dev : 1.0f;
    const float gscale = a.obj_gain * a.balance[l] * static_cast<float>(a.B) * a.grad_scale * up / static_cast<float>(a.cells[l]);
    float local = 0.0f;
    const bool want_grad = a.grad[l] != nullptr;
    for (long long e = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; e < total;
         e += static_cast<long long>(gridDim.x) * blockDim.x) {
        const long long cell = e / a.no;
        const int o = static_cast<int>(e - cell * a.no);
        float g = 0.0f;
        if (o == 4) {
            const float x = ldp(a.p[l], e, a.dtype);
            const float t = __uint_as_float(static_cast<unsigned>(a.tobj[l][cell] & 0xffffffffull));
            local += bce_logits(x, t, a.obj_pw);
            g = bce_logits_grad(x, t, a.obj_pw) * gscale;
        }
        if (want_grad) stg(a.grad[l], e, g, a.dtype);
    }
    __shared__ float red[32];
    for (int o = 16; o > 0; o >>= 1) local += __shfl_xor_sync(0xffffffffu, local, o);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = local;
    __syncthreads();
    if (threadIdx.x == 0) {
        float s = 0.f;
        for (int w = 0; w < (blockDim.x >> 5); ++w) s += red[w];
        a.part_obj[l * kPartials + blockIdx.x] = s;
    }
}

// warp per match: class BCE + scatter-add of box/class gradients
__global__ void loss_cls_kernel(LossArgs a) {
    const int l = blockIdx.y;
    const int n = a.count[l];
    const int nx = a.nx[l], ny = a.ny[l];
    const int* mi = a.midx + static_cast<size_t>(l) * 5 * a.cap;
    const float4* bg = a.bgrad + static_cast<size_t>(l) * a.cap;
    const int lane = threadIdx.x & 31;
    const int wpb = blockDim.x >> 5;
    const bool want_grad = a.grad[l] != nullptr;
    // lbox_l = mean(1-iou): each match contributes 1/n; lcls_l = mean over n*nc
    const float fb = static_cast<float>(a.B) * a.grad_scale * (a.grad_scale_dev ? *a.grad_scale_dev : 1.0f);
    const float gbox = n > 0 ? a.box_gain * fb / static_cast<float>(n) : 0.f;
    const float gcls = n > 0 ? a.cls_gain * fb / (static_cast<float>(n) * static_cast<float>(a.nc)) : 0.f;
    float local = 0.0f;
    for (int i = blockIdx.x * wpb + (threadIdx.x >> 5); i < n; i += gridDim.x * wpb) {
        const int b = mi[i], an = mi[a.cap + i], gj = mi[2 * a.cap + i], gi = mi[3 * a.cap + i], cls = mi[4 * a.cap + i];
        const long long e = (((static_cast<long long>(b) * a.na + an) * ny + gj) * nx + gi) * a.no;
        if (want_grad && lane < 4) {
            const float4 g = bg[i];
            const float gv = lane == 0 ? g.x : lane == 1 ? g.y : lane == 2 ? g.z : g.w;
            atomic_add_elem(a.grad[l], e + lane, gv * gbox, a.dtype);
        }
        if (a.nc > 1) {  // :163
            for (int j = lane; j < a.nc; j += 32) {
                const float x = ldp(a.p[l], e + 5 + j, a.dtype);
                const float t = j == cls ? a.cp : a.cn;
                local += bce_logits(x, t, a.cls_pw);
                if (want_grad) atomic_add_elem(a.grad[l], e + 5 + j, bce_logits_grad(x, t, a.cls_pw) * gcls, a.dtype);
            }
        }
    }
    __shared__ float red[32];
    for (int o = 16; o > 0; o >>= 1) local += __shfl_xor_sync(0xffffffffu, local, o);
    if (lane == 0) red[threadIdx.x >> 5] = local;
    __syncthreads();
    if (threadIdx.x == 0) {
        float s = 0.f;
        for (int w = 0; w < wpb; ++w) s += red[w];
        a.part_cls[l * kPartials + blockIdx.x] = s;
    }
}

__global__ void loss_finalize_kernel(LossArgs a, int match_blocks, int dense_blocks, int cls_blocks) {
    if (threadIdx.x != 0) return;
    float lbox = 0.f, lobj = 0.f, lcls = 0.f;
    for (int l = 0; l < a.nl; ++l) {
        const int n = a.count[l];
        float sb = 0.f, so = 0.f, sc = 0.f;
        for (int i = 0; i < match_blocks; ++i) sb += a.part_box[l * kPartials + i];
        for (int i = 0; i < dense_blocks; ++i) so += a.part_obj[l * kPartials + i];
        for (int i = 0; i < cls_blocks; ++i) sc += a.part_cls[l * kPartials + i];
        if (n > 0) {
            lbox += sb / static_cast<float>(n);
            if (a.nc > 1) lcls += sc / (static_cast<float>(n) * static_cast<float>(a.nc));
        }
        lobj += so / static_cast<float>(a.cells[l]) * a.balance[l];
    }
    lbox *= a.box_gain;
    lobj *= a.obj_gain;
    lcls *= a.cls_gain;
    a.out_loss[0] = (lbox + lobj + lcls) * static_cast<float>(a.B);
    a.out_loss[1] = lbox;
    a.out_loss[2] = lobj;
    a.out_loss[3] = lcls;
}

// ---------------------------------------------------------------------------------------------------------------------
// Segmentation loss: the mask term of reference utils/segment/loss.py:88-99,116-120 on top of the launch set above.
//
//   7 seg_prep      one CTA: per-image target counts -> tidx (global row, or with `overlap` the position's value in the
//                   concatenation [1..n_0, 1..n_1, ...]), xywhn = (t*nx)/nx; per (level, image) match counts and the
//                   start of every image's match list
//   8 seg_bucket    CTA per image: ordered compaction of that image's matches, level by level (stable)
//   9 seg_match     CTA per match: crop bounds, BCE over the crop's pixels only, the mask-coefficient gradient
//                   (fixed-order block reduction), added into grad[l] like the class gradients
//  10 seg_proto     CTA per (image, 16x16 pixel tile): dproto = sum_j g_j(p) coef_j over the image's matches whose crop
//                   meets the tile, recomputed in registers; every element written once (no atomics)
//  11 seg_finalize  fixed-order reduction: per (level, image) mean, sum, gains -> out[5]
// Pixels outside a crop contribute exactly zero, so the work is ~3*nm FMAs per pixel of crop summed over the matches.
// ---------------------------------------------------------------------------------------------------------------------
constexpr int kSegMaxNm = 32;
constexpr int kSegMaxBatch = 1024;  // seg_prep keeps per-image counters in shared memory
constexpr int kSegTile = 16;

struct SegArgs {
    int nl, B, na, no, nc, nm, mh, mw, gt_h, gt_w, overlap, nt, cap, dtype, pdtype;
    int ny[kMaxLevels], nx[kMaxLevels];
    const void* p[kMaxLevels];
    void* grad[kMaxLevels];
    const void* proto;
    long long ps_b, ps_k, ps_y, ps_x;         // proto element strides (NCHW or channels_last)
    void* grad_proto;                         // same dtype and strides as proto
    const float* masks;                       // (n_masks, gt_h, gt_w)
    const float* targets;
    const float* grad_scale_dev;
    float box_gain, grad_scale;
    const int* count;                         // [nl]           detection workspace
    const int* midx;                          // [nl][5][cap]   detection workspace
    const int* trow;                          // [nl][cap]
    int* tidx;                                // [nl][cap]
    float4* xywhn;                            // [nl][cap]
    int* nimg;                                // [nl][B]        matches of image b at level l
    int* ioff;                                // [B+1]          start of image b's list
    int* list;                                // [nl*cap]       l*cap + i, by image, then level, then match order
    int4* crop;                               // [nl][cap]      x0, x1, y0, y1 (half-open, clipped to the map)
    float* gs;                                // [nl][cap]      d(loss * upstream)/d logit = gs * (sigmoid - gt)
    float* val;                               // [nl][cap]      crop BCE sum / (mh*mw) / area
    const float* det_out;                     // [4]            detection items
    float* out;                               // [5]
};

// gt of pixel (y, x) at proto resolution: F.interpolate(mode="nearest") folded into the read,
// source index min(floor(dst * (in / out)), in - 1) in fp32
__device__ __forceinline__ float seg_gt(const SegArgs& a, int b, int tidx, int y, int x) {
    const float sy = __fdiv_rn(static_cast<float>(a.gt_h), static_cast<float>(a.mh));
    const float sx = __fdiv_rn(static_cast<float>(a.gt_w), static_cast<float>(a.mw));
    const int iy = min(static_cast<int>(floorf(__fmul_rn(static_cast<float>(y), sy))), a.gt_h - 1);
    const int ix = min(static_cast<int>(floorf(__fmul_rn(static_cast<float>(x), sx))), a.gt_w - 1);
    const int m = a.overlap ? b : tidx;
    const float v = a.masks[(static_cast<long long>(m) * a.gt_h + iy) * a.gt_w + ix];
    return a.overlap ? (v == static_cast<float>(tidx) ? 1.0f : 0.0f) : v;
}

__device__ __forceinline__ float seg_logit(const float* coef, const float* pr, int nm) {
    float acc = 0.0f;
#pragma unroll
    for (int k = 0; k < kSegMaxNm; ++k)
        if (k < nm) acc = __fmaf_rn(coef[k], pr[k], acc);
    return acc;
}

__device__ __forceinline__ void seg_load_proto(const SegArgs& a, int b, int y, int x, float* pr) {
    const long long base = b * a.ps_b + y * a.ps_y + x * a.ps_x;
#pragma unroll
    for (int k = 0; k < kSegMaxNm; ++k) pr[k] = k < a.nm ? ldp(a.proto, base + k * a.ps_k, a.pdtype) : 0.0f;
}

__global__ void seg_prep_kernel(SegArgs a) {
    __shared__ int s_start[kSegMaxBatch + 1];
    __shared__ int s_cnt[kMaxLevels * kSegMaxBatch];
    for (int i = threadIdx.x; i <= a.B; i += blockDim.x) s_start[i] = 0;
    for (int i = threadIdx.x; i < a.nl * a.B; i += blockDim.x) s_cnt[i] = 0;
    __syncthreads();
    // (targets[:, 0] == i).sum() per image (segment/loss.py:134)
    for (int t = threadIdx.x; t < a.nt; t += blockDim.x) {
        const float f = a.targets[static_cast<size_t>(t) * 6];
        const int b = static_cast<int>(f);
        if (f == static_cast<float>(b) && b >= 0 && b < a.B) atomicAdd(&s_start[b + 1], 1);
    }
    for (int l = 0; l < a.nl; ++l) {
        const int n = a.count[l];
        const int* mb = a.midx + static_cast<size_t>(l) * 5 * a.cap;
        for (int i = threadIdx.x; i < n; i += blockDim.x) atomicAdd(&s_cnt[l * a.B + mb[i]], 1);
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        int off = 0;
        for (int b = 0; b < a.B; ++b) {
            s_start[b + 1] += s_start[b];
            a.ioff[b] = off;
            for (int l = 0; l < a.nl; ++l) off += s_cnt[l * a.B + b];
        }
        a.ioff[a.B] = off;
    }
    for (int i = threadIdx.x; i < a.nl * a.B; i += blockDim.x) a.nimg[i] = s_cnt[i];
    __syncthreads();
    for (int l = 0; l < a.nl; ++l) {
        const int n = a.count[l];
        const float fnx = static_cast<float>(a.nx[l]), fny = static_cast<float>(a.ny[l]);
        for (int i = threadIdx.x; i < n; i += blockDim.x) {
            const size_t q = static_cast<size_t>(l) * a.cap + i;
            const int t = a.trow[q];
            int v = t;
            if (a.overlap) {  // value at position t of cat([arange(n_b) + 1 for b in range(B)]): the image is the POSITION's
                int lo = 0, hi = a.B - 1;
                while (lo < hi) {
                    const int mid = (lo + hi + 1) >> 1;
                    if (s_start[mid] <= t) lo = mid; else hi = mid - 1;
                }
                v = t - s_start[lo] + 1;
            }
            a.tidx[q] = v;
            const float* tg = a.targets + static_cast<size_t>(t) * 6;
            // xywhn = cat(gxy, gwh) / gain[2:6] with gxy, gwh = targets * gain: (t * nx) / nx, not always t in fp32
            a.xywhn[q] = make_float4(__fdiv_rn(__fmul_rn(tg[2], fnx), fnx), __fdiv_rn(__fmul_rn(tg[3], fny), fny),
                                     __fdiv_rn(__fmul_rn(tg[4], fnx), fnx), __fdiv_rn(__fmul_rn(tg[5], fny), fny));
        }
    }
}

__global__ void seg_bucket_kernel(SegArgs a) {
    const int b = blockIdx.x;
    __shared__ int warp_cnt[32];
    __shared__ int base_s;
    if (threadIdx.x == 0) base_s = a.ioff[b];
    __syncthreads();
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
    for (int l = 0; l < a.nl; ++l) {
        const int n = a.count[l];
        const int* mb = a.midx + static_cast<size_t>(l) * 5 * a.cap;
        for (int c0 = 0; c0 < n; c0 += blockDim.x) {
            const int i = c0 + threadIdx.x;
            const bool ok = i < n && mb[i] == b;
            const unsigned m = __ballot_sync(0xffffffffu, ok);
            if (lane == 0) warp_cnt[warp] = __popc(m);
            __syncthreads();
            int before = base_s;
            for (int w = 0; w < warp; ++w) before += warp_cnt[w];
            if (ok) a.list[before + __popc(m & ((1u << lane) - 1u))] = l * a.cap + i;
            __syncthreads();
            if (threadIdx.x == 0) {
                int s = base_s;
                for (int w = 0; w < nwarps; ++w) s += warp_cnt[w];
                base_s = s;
            }
            __syncthreads();
        }
    }
}

// fixed-order block sum of v[0..nv) (blockDim.x == 256): result valid in red_out[0..nv) after the call
template <int NV>
__device__ __forceinline__ void block_sum(float (&v)[NV], float (*red)[NV], float* red_out) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int k = 0; k < NV; ++k)
        for (int o = 16; o > 0; o >>= 1) v[k] += __shfl_xor_sync(0xffffffffu, v[k], o);
    if (lane == 0)
#pragma unroll
        for (int k = 0; k < NV; ++k) red[warp][k] = v[k];
    __syncthreads();
    if (threadIdx.x < NV) {
        float s = 0.0f;
        for (int w = 0; w < (blockDim.x >> 5); ++w) s += red[w][threadIdx.x];
        red_out[threadIdx.x] = s;
    }
    __syncthreads();
}

__global__ void __launch_bounds__(256) seg_match_kernel(SegArgs a) {
    const int l = blockIdx.y;
    const int n = a.count[l];
    const int nx = a.nx[l], ny = a.ny[l];
    const int* mi = a.midx + static_cast<size_t>(l) * 5 * a.cap;
    const float up = a.grad_scale * (a.grad_scale_dev ? *a.grad_scale_dev : 1.0f);
    const float hw = static_cast<float>(a.mh) * static_cast<float>(a.mw);
    __shared__ float s_coef[kSegMaxNm];
    __shared__ float red[8][kSegMaxNm + 1];
    __shared__ float tot[kSegMaxNm + 1];
    for (int i = blockIdx.x; i < n; i += gridDim.x) {
        const size_t q = static_cast<size_t>(l) * a.cap + i;
        const int b = mi[i], an = mi[a.cap + i], gj = mi[2 * a.cap + i], gi = mi[3 * a.cap + i];
        const long long e = (((static_cast<long long>(b) * a.na + an) * ny + gj) * nx + gi) * a.no + 5 + a.nc;
        if (threadIdx.x < a.nm) s_coef[threadIdx.x] = ldp(a.p[l], e + threadIdx.x, a.dtype);
        const float4 xn = a.xywhn[q];
        // mxyxy = xywh2xyxy(xywhn * [mw, mh, mw, mh]); crop_mask keeps r >= x1 & r < x2 -> columns [ceil(x1), ceil(x2))
        const float bx = __fmul_rn(xn.x, static_cast<float>(a.mw)), by = __fmul_rn(xn.y, static_cast<float>(a.mh));
        const float bw = __fdiv_rn(__fmul_rn(xn.z, static_cast<float>(a.mw)), 2.0f);
        const float bh = __fdiv_rn(__fmul_rn(xn.w, static_cast<float>(a.mh)), 2.0f);
        const int x0 = static_cast<int>(fminf(fmaxf(ceilf(__fsub_rn(bx, bw)), 0.0f), static_cast<float>(a.mw)));
        const int x1 = static_cast<int>(fminf(fmaxf(ceilf(__fadd_rn(bx, bw)), 0.0f), static_cast<float>(a.mw)));
        const int y0 = static_cast<int>(fminf(fmaxf(ceilf(__fsub_rn(by, bh)), 0.0f), static_cast<float>(a.mh)));
        const int y1 = static_cast<int>(fminf(fmaxf(ceilf(__fadd_rn(by, bh)), 0.0f), static_cast<float>(a.mh)));
        const float area = __fmul_rn(xn.z, xn.w);
        const float nb = static_cast<float>(a.nimg[l * a.B + b]);
        const float s = __fdiv_rn(__fdiv_rn(__fdiv_rn(__fmul_rn(up, a.box_gain), nb), hw), area);
        const int tidx = a.tidx[q];
        __syncthreads();
        float coef[kSegMaxNm];
#pragma unroll
        for (int k = 0; k < kSegMaxNm; ++k) coef[k] = k < a.nm ? s_coef[k] : 0.0f;
        float acc[kSegMaxNm + 1];
#pragma unroll
        for (int k = 0; k <= kSegMaxNm; ++k) acc[k] = 0.0f;
        const int cw = max(x1 - x0, 0), ch = max(y1 - y0, 0);
        const int npix = cw * ch;
        for (int pix = threadIdx.x; pix < npix; pix += blockDim.x) {
            const int y = y0 + pix / cw, x = x0 + pix % cw;
            float pr[kSegMaxNm];
            seg_load_proto(a, b, y, x, pr);
            const float xl = seg_logit(coef, pr, a.nm);
            const float gt = seg_gt(a, b, tidx, y, x);
            acc[kSegMaxNm] += bce_logits(xl, gt, 1.0f);
            const float g = __fmul_rn(__fsub_rn(sigmoid_f(xl), gt), s);
#pragma unroll
            for (int k = 0; k < kSegMaxNm; ++k) acc[k] = __fmaf_rn(g, pr[k], acc[k]);
        }
        block_sum<kSegMaxNm + 1>(acc, red, tot);
        if (threadIdx.x < a.nm && a.grad[l]) atomic_add_elem(a.grad[l], e + threadIdx.x, tot[threadIdx.x], a.dtype);
        if (threadIdx.x == 0) {
            a.val[q] = __fdiv_rn(__fdiv_rn(tot[kSegMaxNm], hw), area);
            a.crop[q] = make_int4(x0, x1, y0, y1);
            a.gs[q] = s;
        }
        __syncthreads();
    }
}

__global__ void __launch_bounds__(256) seg_proto_kernel(SegArgs a) {
    constexpr int kBatch = 32;
    const int b = blockIdx.y;
    const int tiles_x = (a.mw + kSegTile - 1) / kSegTile;
    const int tx0 = (blockIdx.x % tiles_x) * kSegTile, ty0 = (blockIdx.x / tiles_x) * kSegTile;
    const int x = tx0 + (threadIdx.x % kSegTile), y = ty0 + (threadIdx.x / kSegTile);
    const bool inside = x < a.mw && y < a.mh;
    __shared__ float s_coef[kBatch][kSegMaxNm];
    __shared__ int4 s_crop[kBatch];
    __shared__ float s_gs[kBatch];
    __shared__ int s_tidx[kBatch];
    __shared__ int s_hit[kBatch];
    float pr[kSegMaxNm], acc[kSegMaxNm];
    seg_load_proto(a, b, inside ? y : 0, inside ? x : 0, pr);
#pragma unroll
    for (int k = 0; k < kSegMaxNm; ++k) acc[k] = 0.0f;
    const int beg = a.ioff[b], end = a.ioff[b + 1];
    for (int j0 = beg; j0 < end; j0 += kBatch) {
        const int nb = min(kBatch, end - j0);
        if (threadIdx.x < nb) {
            const int q = a.list[j0 + threadIdx.x];
            const int4 c = a.crop[q];
            s_crop[threadIdx.x] = c;
            s_gs[threadIdx.x] = a.gs[q];
            s_tidx[threadIdx.x] = a.tidx[q];
            s_hit[threadIdx.x] = max(c.x, tx0) < min(c.y, tx0 + kSegTile) && max(c.z, ty0) < min(c.w, ty0 + kSegTile);
        }
        __syncthreads();
        for (int idx = threadIdx.x; idx < nb * kSegMaxNm; idx += blockDim.x) {
            const int jj = idx / kSegMaxNm, k = idx % kSegMaxNm;
            if (!s_hit[jj] || k >= a.nm) continue;
            const int q = a.list[j0 + jj];
            const int l = q / a.cap, i = q - l * a.cap;
            const int* mi = a.midx + static_cast<size_t>(l) * 5 * a.cap;
            const long long e = (((static_cast<long long>(mi[i]) * a.na + mi[a.cap + i]) * a.ny[l] + mi[2 * a.cap + i]) * a.nx[l] +
                                 mi[3 * a.cap + i]) * a.no + 5 + a.nc;
            s_coef[jj][k] = ldp(a.p[l], e + k, a.dtype);
        }
        __syncthreads();
        for (int jj = 0; jj < nb; ++jj) {
            if (!s_hit[jj]) continue;
            const int4 c = s_crop[jj];
            if (!inside || x < c.x || x >= c.y || y < c.z || y >= c.w) continue;
            const float xl = seg_logit(s_coef[jj], pr, a.nm);
            const float g = __fmul_rn(__fsub_rn(sigmoid_f(xl), seg_gt(a, b, s_tidx[jj], y, x)), s_gs[jj]);
#pragma unroll
            for (int k = 0; k < kSegMaxNm; ++k) acc[k] = __fmaf_rn(g, s_coef[jj][k < a.nm ? k : 0], acc[k]);
        }
        __syncthreads();
    }
    if (!inside) return;
    const long long base = b * a.ps_b + y * a.ps_y + x * a.ps_x;
#pragma unroll
    for (int k = 0; k < kSegMaxNm; ++k)
        if (k < a.nm) stg(a.grad_proto, base + k * a.ps_k, acc[k], a.pdtype);
}

__global__ void seg_finalize_kernel(SegArgs a) {
    __shared__ float red[256];
    float local = 0.0f;
    for (int b = threadIdx.x; b < a.B; b += blockDim.x) {
        // the image's list is level-ordered: mean per (level, image), as the reference's `for bi in b.unique()`
        float cur = 0.0f;
        int cur_l = -1;
        for (int j = a.ioff[b]; j < a.ioff[b + 1]; ++j) {
            const int q = a.list[j];
            const int l = q / a.cap;
            if (l != cur_l) {
                if (cur_l >= 0) local += cur / static_cast<float>(a.nimg[cur_l * a.B + b]);
                cur = 0.0f;
                cur_l = l;
            }
            cur += a.val[q];
        }
        if (cur_l >= 0) local += cur / static_cast<float>(a.nimg[cur_l * a.B + b]);
    }
    red[threadIdx.x] = local;
    __syncthreads();
    if (threadIdx.x != 0) return;
    float lseg = 0.0f;
    for (int w = 0; w < blockDim.x; ++w) lseg += red[w];
    lseg *= a.box_gain / static_cast<float>(a.B);
    const float lbox = a.det_out[1], lobj = a.det_out[2], lcls = a.det_out[3];
    a.out[0] = (lbox + lobj + lcls + lseg) * static_cast<float>(a.B);
    a.out[1] = lbox;
    a.out[2] = lseg;
    a.out[3] = lobj;
    a.out[4] = lcls;
}

}  // namespace y5

using namespace y5;

namespace {
struct LossWs {
    size_t count, midx, tbox, bgrad, tobj[kMaxLevels], part_box, part_obj, part_cls, total;
};
LossWs loss_ws(const y5_loss_params* p) {
    LossWs L;
    size_t o = 0;
    auto take = [&](size_t bytes) { size_t r = o; o += (bytes + 255) & ~size_t(255); return r; };
    const size_t cap = static_cast<size_t>(5) * p->na * (p->nt > 0 ? p->nt : 1);
    L.count = take(sizeof(int) * kMaxLevels);
    L.midx = take(sizeof(int) * p->nl * 5 * cap);
    L.tbox = take(sizeof(float4) * p->nl * cap);
    L.bgrad = take(sizeof(float4) * p->nl * cap);
    for (int l = 0; l < p->nl; ++l) L.tobj[l] = take(sizeof(unsigned long long) * static_cast<size_t>(p->batch) * p->na * p->ny[l] * p->nx[l]);
    L.part_box = take(sizeof(float) * kMaxLevels * kPartials);
    L.part_obj = take(sizeof(float) * kMaxLevels * kPartials);
    L.part_cls = take(sizeof(float) * kMaxLevels * kPartials);
    L.total = o;
    return L;
}
int validate_loss(const y5_loss_params* p) {
    if (!p) return set_error(Y5_E_INVALID, "loss: null params");
    if (p->nl < 1 || p->nl > kMaxLevels || p->batch < 1 || p->na < 1 || p->nc < 1 || p->no < 5 + p->nc || p->nt < 0)
        return set_error(Y5_E_INVALID, "loss: bad shape (nl %d batch %d na %d no %d nc %d nt %d)", p->nl, p->batch, p->na, p->no, p->nc, p->nt);
    if (p->dtype != Y5_F16 && p->dtype != Y5_BF16 && p->dtype != Y5_F32) return set_error(Y5_E_UNSUPPORTED, "loss: dtype");
    for (int l = 0; l < p->nl; ++l)
        if (p->ny[l] < 1 || p->nx[l] < 1) return set_error(Y5_E_INVALID, "loss: bad grid at level %d", l);
    if (static_cast<long long>(5) * p->na * p->nt > 0x3fffffff) return set_error(Y5_E_UNSUPPORTED, "loss: too many targets");
    return 0;
}
void fill_args(LossArgs& a, const y5_loss_params* p, void* workspace, const LossWs& L) {
    unsigned char* ws = static_cast<unsigned char*>(workspace);
    a.nl = p->nl; a.B = p->batch; a.na = p->na; a.no = p->no; a.nc = p->nc; a.dtype = p->dtype; a.nt = p->nt;
    for (int l = 0; l < p->nl; ++l) {
        a.ny[l] = p->ny[l]; a.nx[l] = p->nx[l]; a.balance[l] = p->balance[l];
        a.cells[l] = static_cast<long long>(p->batch) * p->na * p->ny[l] * p->nx[l];
        a.tobj[l] = reinterpret_cast<unsigned long long*>(ws + L.tobj[l]);
    }
    a.anchor_t = p->anchor_t; a.box_gain = p->box_gain; a.obj_gain = p->obj_gain; a.cls_gain = p->cls_gain;
    a.cls_pw = p->cls_pw; a.obj_pw = p->obj_pw; a.cp = p->cp; a.cn = p->cn; a.grad_scale = p->grad_scale;
    a.cap = 5 * p->na * (p->nt > 0 ? p->nt : 1);
    a.count = reinterpret_cast<int*>(ws + L.count);
    a.midx = reinterpret_cast<int*>(ws + L.midx);
    a.tbox = reinterpret_cast<float4*>(ws + L.tbox);
    a.bgrad = reinterpret_cast<float4*>(ws + L.bgrad);
    a.part_box = reinterpret_cast<float*>(ws + L.part_box);
    a.part_obj = reinterpret_cast<float*>(ws + L.part_obj);
    a.part_cls = reinterpret_cast<float*>(ws + L.part_cls);
}
}  // namespace

extern "C" Y5_API int64_t y5_loss_workspace_bytes(const y5_loss_params* p) {
    if (validate_loss(p)) return -1;
    return static_cast<int64_t>(loss_ws(p).total);
}

namespace {
// the detection launch set; `trow` (segmentation loss only) receives each match's target row
int loss_launch(const y5_loss_params* p, const void* const* pl, const float* targets, const float* anchors, float* out_loss,
                void* const* grad, const float* grad_scale_dev, void* workspace, int64_t workspace_bytes, void* stream, int* trow) {
    if (int e = validate_loss(p)) return e;
    if (!pl || !anchors || !out_loss || !workspace || (p->nt > 0 && !targets)) return set_error(Y5_E_INVALID, "loss: null pointer");
    const LossWs L = loss_ws(p);
    if (workspace_bytes < static_cast<int64_t>(L.total)) return set_error(Y5_E_INVALID, "loss: workspace too small");
    if (reinterpret_cast<uintptr_t>(workspace) & 255) return set_error(Y5_E_INVALID, "loss: workspace must be 256-byte aligned");
    LossArgs a{};
    fill_args(a, p, workspace, L);
    for (int l = 0; l < p->nl; ++l) {
        if (!pl[l]) return set_error(Y5_E_INVALID, "loss: null prediction level %d", l);
        a.p[l] = pl[l];
        a.grad[l] = grad ? grad[l] : nullptr;
    }
    a.targets = targets; a.anchors = anchors; a.out_loss = out_loss;
    a.grad_scale_dev = grad_scale_dev;
    a.trow = trow;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const int sms = sm_count();
    if (int e = launch("loss", loss_zero_kernel, {sms * 4, 256, 0, st}, a)) return e;
    if (int e = launch("loss", loss_targets_kernel, {p->nl, 1024, 0, st}, a)) return e;
    const int match_blocks = min(kPartials, max(1, (a.cap + 127) / 128));
    if (int e = launch("loss", loss_match_kernel, {dim3(match_blocks, p->nl), 128, 0, st}, a)) return e;
    const int dense_blocks = kPartials;
    if (int e = launch("loss", loss_dense_kernel, {dim3(dense_blocks, p->nl), 512, 0, st}, a)) return e;
    const int cls_blocks = min(kPartials, max(1, (a.cap + 7) / 8));
    if (int e = launch("loss", loss_cls_kernel, {dim3(cls_blocks, p->nl), 256, 0, st}, a)) return e;
    return launch("loss", loss_finalize_kernel, {1, 32, 0, st}, a, match_blocks, dense_blocks, cls_blocks);
}
}  // namespace

extern "C" Y5_API int y5_loss_fwd_bwd_scaled(const y5_loss_params* p, const void* const* pl, const float* targets, const float* anchors,
                                             float* out_loss, void* const* grad, const float* grad_scale_dev, void* workspace,
                                             int64_t workspace_bytes, void* stream) {
    return loss_launch(p, pl, targets, anchors, out_loss, grad, grad_scale_dev, workspace, workspace_bytes, stream, nullptr);
}

// Copies one level's build_targets result to host memory (synchronises the stream: test / debugging helper).
extern "C" Y5_API int y5_loss_read_targets(const y5_loss_params* p, const void* workspace, int32_t level, int64_t* idx5_host,
                                           float* tbox_host, int32_t* count_host, void* stream) {
    if (int e = validate_loss(p)) return e;
    if (!workspace || level < 0 || level >= p->nl || !count_host) return set_error(Y5_E_INVALID, "loss_read_targets: bad arguments");
    const LossWs L = loss_ws(p);
    const unsigned char* ws = static_cast<const unsigned char*>(workspace);
    const size_t cap = static_cast<size_t>(5) * p->na * (p->nt > 0 ? p->nt : 1);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    int counts[kMaxLevels];
    cudaError_t e = cudaMemcpyAsync(counts, ws + L.count, sizeof(int) * kMaxLevels, cudaMemcpyDeviceToHost, st);
    if (e == cudaSuccess) e = cudaStreamSynchronize(st);
    if (e != cudaSuccess) return set_error(int(e), "loss_read_targets: %s", cudaGetErrorString(e));
    const int n = counts[level];
    *count_host = n;
    if (n > 0 && idx5_host) {
        int* tmp = new int[5 * cap];
        e = cudaMemcpyAsync(tmp, ws + L.midx + sizeof(int) * level * 5 * cap, sizeof(int) * 5 * cap, cudaMemcpyDeviceToHost, st);
        if (e == cudaSuccess) e = cudaStreamSynchronize(st);
        if (e == cudaSuccess)
            for (int q = 0; q < 5; ++q)
                for (int i = 0; i < n; ++i) idx5_host[static_cast<size_t>(q) * n + i] = tmp[q * cap + i];
        delete[] tmp;
        if (e != cudaSuccess) return set_error(int(e), "loss_read_targets: %s", cudaGetErrorString(e));
    }
    if (n > 0 && tbox_host) {
        e = cudaMemcpyAsync(tbox_host, ws + L.tbox + sizeof(float4) * level * cap, sizeof(float4) * n, cudaMemcpyDeviceToHost, st);
        if (e == cudaSuccess) e = cudaStreamSynchronize(st);
        if (e != cudaSuccess) return set_error(int(e), "loss_read_targets: %s", cudaGetErrorString(e));
    }
    return 0;
}

// ---------------------------------------------------------------------------------------------------------------------
// segmentation loss: detection workspace layout unchanged, the seg scratch follows it
// ---------------------------------------------------------------------------------------------------------------------
namespace {
struct SegWs {
    size_t trow, tidx, xywhn, nimg, ioff, list, crop, gs, val, det_out, total;
};
SegWs seg_ws(const y5_loss_params* p) {
    SegWs S;
    size_t o = loss_ws(p).total;
    auto take = [&](size_t bytes) { size_t r = o; o += (bytes + 255) & ~size_t(255); return r; };
    const size_t m = static_cast<size_t>(p->nl) * 5 * p->na * (p->nt > 0 ? p->nt : 1);
    S.trow = take(sizeof(int) * m);
    S.tidx = take(sizeof(int) * m);
    S.xywhn = take(sizeof(float4) * m);
    S.nimg = take(sizeof(int) * kMaxLevels * p->batch);
    S.ioff = take(sizeof(int) * (p->batch + 1));
    S.list = take(sizeof(int) * m);
    S.crop = take(sizeof(int4) * m);
    S.gs = take(sizeof(float) * m);
    S.val = take(sizeof(float) * m);
    S.det_out = take(sizeof(float) * 4);
    S.total = o;
    return S;
}
int validate_seg(const y5_loss_params* p) {
    if (int e = validate_loss(p)) return e;
    if (p->batch > kSegMaxBatch) return set_error(Y5_E_INVALID, "seg_loss: batch %d > %d", p->batch, kSegMaxBatch);
    if (static_cast<long long>(p->nl) * 5 * p->na * (p->nt > 0 ? p->nt : 1) > 0x3fffffff)
        return set_error(Y5_E_UNSUPPORTED, "seg_loss: too many targets");
    return 0;
}
}  // namespace

extern "C" Y5_API int64_t y5_seg_loss_workspace_bytes(const y5_loss_params* p) {
    if (validate_seg(p)) return -1;
    return static_cast<int64_t>(seg_ws(p).total);
}

extern "C" Y5_API int y5_seg_loss_fwd_bwd_scaled(const y5_loss_params* p, const void* const* pl, const float* targets,
                                                 const float* anchors, const void* proto, int32_t proto_dtype, int64_t ps_b,
                                                 int64_t ps_k, int64_t ps_y, int64_t ps_x, int32_t nm, int32_t mh, int32_t mw,
                                                 const float* masks, int32_t n_masks, int32_t gt_h, int32_t gt_w, int32_t overlap,
                                                 float* out_loss, void* const* grad, void* grad_proto, const float* grad_scale_dev,
                                                 void* workspace, int64_t workspace_bytes, void* stream) {
    if (int e = validate_seg(p)) return e;
    if (nm < 1 || nm > kSegMaxNm) return set_error(Y5_E_INVALID, "seg_loss: nm %d outside [1, %d]", nm, kSegMaxNm);
    if (p->no != 5 + p->nc + nm) return set_error(Y5_E_INVALID, "seg_loss: no %d != 5 + nc %d + nm %d", p->no, p->nc, nm);
    if (mh < 1 || mw < 1 || gt_h < 1 || gt_w < 1)
        return set_error(Y5_E_INVALID, "seg_loss: bad mask sizes (proto %dx%d, masks %dx%d)", mh, mw, gt_h, gt_w);
    if (overlap != 0 && overlap != 1) return set_error(Y5_E_INVALID, "seg_loss: overlap must be 0 or 1");
    if (overlap ? n_masks != p->batch : n_masks < p->nt)
        return set_error(Y5_E_INVALID, "seg_loss: %d masks for batch %d / %d targets (overlap %d)", n_masks, p->batch, p->nt, overlap);
    if (proto_dtype != Y5_F16 && proto_dtype != Y5_BF16 && proto_dtype != Y5_F32) return set_error(Y5_E_UNSUPPORTED, "seg_loss: proto dtype");
    if (ps_b < 0 || ps_k < 0 || ps_y < 0 || ps_x < 0) return set_error(Y5_E_INVALID, "seg_loss: negative proto stride");
    if (!proto || !out_loss || !workspace || (p->nt > 0 && !masks)) return set_error(Y5_E_INVALID, "seg_loss: null pointer");
    const SegWs S = seg_ws(p);
    if (workspace_bytes < static_cast<int64_t>(S.total)) return set_error(Y5_E_INVALID, "seg_loss: workspace too small");
    unsigned char* ws = static_cast<unsigned char*>(workspace);
    if (int e = loss_launch(p, pl, targets, anchors, reinterpret_cast<float*>(ws + S.det_out), grad, grad_scale_dev, workspace,
                            workspace_bytes, stream, reinterpret_cast<int*>(ws + S.trow)))
        return e;
    const LossWs L = loss_ws(p);
    SegArgs a{};
    a.nl = p->nl; a.B = p->batch; a.na = p->na; a.no = p->no; a.nc = p->nc; a.nm = nm; a.mh = mh; a.mw = mw;
    a.gt_h = gt_h; a.gt_w = gt_w; a.overlap = overlap; a.nt = p->nt; a.cap = 5 * p->na * (p->nt > 0 ? p->nt : 1);
    a.dtype = p->dtype; a.pdtype = proto_dtype;
    for (int l = 0; l < p->nl; ++l) {
        a.ny[l] = p->ny[l]; a.nx[l] = p->nx[l];
        a.p[l] = pl[l];
        a.grad[l] = grad ? grad[l] : nullptr;
    }
    a.proto = proto; a.ps_b = ps_b; a.ps_k = ps_k; a.ps_y = ps_y; a.ps_x = ps_x;
    a.grad_proto = grad_proto; a.masks = masks; a.targets = targets; a.grad_scale_dev = grad_scale_dev;
    a.box_gain = p->box_gain; a.grad_scale = p->grad_scale;
    a.count = reinterpret_cast<const int*>(ws + L.count);
    a.midx = reinterpret_cast<const int*>(ws + L.midx);
    a.trow = reinterpret_cast<const int*>(ws + S.trow);
    a.tidx = reinterpret_cast<int*>(ws + S.tidx);
    a.xywhn = reinterpret_cast<float4*>(ws + S.xywhn);
    a.nimg = reinterpret_cast<int*>(ws + S.nimg);
    a.ioff = reinterpret_cast<int*>(ws + S.ioff);
    a.list = reinterpret_cast<int*>(ws + S.list);
    a.crop = reinterpret_cast<int4*>(ws + S.crop);
    a.gs = reinterpret_cast<float*>(ws + S.gs);
    a.val = reinterpret_cast<float*>(ws + S.val);
    a.det_out = reinterpret_cast<const float*>(ws + S.det_out);
    a.out = out_loss;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    if (int e = launch("seg_loss", seg_prep_kernel, {1, 1024, 0, st}, a)) return e;
    if (int e = launch("seg_loss", seg_bucket_kernel, {p->batch, 256, 0, st}, a)) return e;
    if (int e = launch("seg_loss", seg_match_kernel, {dim3(min(a.cap, 4 * sm_count()), p->nl), 256, 0, st}, a)) return e;
    if (grad_proto) {
        const int tiles = ((mw + kSegTile - 1) / kSegTile) * ((mh + kSegTile - 1) / kSegTile);
        if (int e = launch("seg_loss", seg_proto_kernel, {dim3(tiles, p->batch), kSegTile * kSegTile, 0, st}, a)) return e;
    }
    return launch("seg_loss", seg_finalize_kernel, {1, 256, 0, st}, a);
}

// Copies one level's tidx (int64) and xywhn (fp32 x4) to host memory (synchronises the stream: test / debugging helper).
extern "C" Y5_API int y5_seg_loss_read_targets(const y5_loss_params* p, const void* workspace, int32_t level, int64_t* tidx_host,
                                               float* xywhn_host, int32_t* count_host, void* stream) {
    if (int e = validate_seg(p)) return e;
    if (!workspace || level < 0 || level >= p->nl || !count_host) return set_error(Y5_E_INVALID, "seg_loss_read_targets: bad arguments");
    const LossWs L = loss_ws(p);
    const SegWs S = seg_ws(p);
    const unsigned char* ws = static_cast<const unsigned char*>(workspace);
    const size_t cap = static_cast<size_t>(5) * p->na * (p->nt > 0 ? p->nt : 1);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    int counts[kMaxLevels];
    cudaError_t e = cudaMemcpyAsync(counts, ws + L.count, sizeof(int) * kMaxLevels, cudaMemcpyDeviceToHost, st);
    if (e == cudaSuccess) e = cudaStreamSynchronize(st);
    if (e != cudaSuccess) return set_error(int(e), "seg_loss_read_targets: %s", cudaGetErrorString(e));
    const int n = counts[level];
    *count_host = n;
    if (n > 0 && tidx_host) {
        int* tmp = new int[n];
        e = cudaMemcpyAsync(tmp, ws + S.tidx + sizeof(int) * level * cap, sizeof(int) * n, cudaMemcpyDeviceToHost, st);
        if (e == cudaSuccess) e = cudaStreamSynchronize(st);
        if (e == cudaSuccess)
            for (int i = 0; i < n; ++i) tidx_host[i] = tmp[i];
        delete[] tmp;
        if (e != cudaSuccess) return set_error(int(e), "seg_loss_read_targets: %s", cudaGetErrorString(e));
    }
    if (n > 0 && xywhn_host) {
        e = cudaMemcpyAsync(xywhn_host, ws + S.xywhn + sizeof(float4) * level * cap, sizeof(float4) * n, cudaMemcpyDeviceToHost, st);
        if (e == cudaSuccess) e = cudaStreamSynchronize(st);
        if (e != cudaSuccess) return set_error(int(e), "seg_loss_read_targets: %s", cudaGetErrorString(e));
    }
    return 0;
}
