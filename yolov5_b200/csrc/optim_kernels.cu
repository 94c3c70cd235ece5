// The step right after backward (SURVEY.md section 8f rank 4): reference train.py:413-421 --
//     scaler.unscale_(optimizer); clip_grad_norm_(model.parameters(), 10.0); scaler.step(optimizer); optimizer.zero_grad(); ema.update(model)
// with optimizer = SGD(momentum, nesterov=True) over 3 parameter groups (utils/torch_utils.py:256-289) and
// ModelEMA.update (utils/torch_utils.py:359-368) -- as TWO multi-tensor launches over every parameter of the model:
//   1. grad_norm : per-chunk partial sums of (g * inv_scale)^2 and a non-finite flag (deterministic: fixed chunk order)
//   2. step      : clip coefficient from the partials, un-scale, weight decay, momentum / Nesterov update, EMA of the new
//                  weights (and of the floating-point buffers), gradient zeroing -- one read of g, one read+write of
//                  p / momentum / ema per element instead of ~10 passes of foreach kernels.  A non-finite gradient skips
//                  the parameter update (what GradScaler.step does) but still advances the EMA, like the reference.
// y5_adam_step is the same step with torch.optim.Adam / AdamW (utils/torch_utils.py:276-279) in place of SGD: the same norm
// pass, one element pass over g / p / exp_avg / exp_avg_sq / ema, and a tail that advances the per-tensor step counters.
// Hyper-parameters live in DEVICE memory (per-group lr / momentum / weight decay, loss-scale reciprocal, EMA decay
// constants, update counter), so a captured CUDA graph sees schedule changes without re-capture and never syncs.
#include <math.h>

#include "../../include/y5b200.h"
#include "common.cuh"
#include "host_util.h"

namespace y5 {

constexpr int kOptChunk = 16384;   // elements per block
constexpr int kOptThreads = 256;

__device__ __forceinline__ float block_sum(float v, float* sh) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = v;
    __syncthreads();
    float r = 0.f;
    if (threadIdx.x < 32) {
        r = threadIdx.x < kOptThreads / 32 ? sh[threadIdx.x] : 0.f;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) r += __shfl_xor_sync(0xffffffffu, r, o);
    }
    return r;  // valid in thread 0
}

// partial[2*chunk] = sum of squares of the un-scaled gradient chunk, partial[2*chunk+1] = 1 if any element is inf/nan
__global__ void __launch_bounds__(kOptThreads) opt_grad_norm_kernel(const y5_opt_tensor* __restrict__ tab, const int32_t* __restrict__ chunk_tensor,
                                                                    const int32_t* __restrict__ chunk_index, const float* __restrict__ hyper,
                                                                    float* __restrict__ partial) {
    __shared__ float sh[kOptThreads / 32];
    __shared__ int bad;
    if (threadIdx.x == 0) bad = 0;
    __syncthreads();
    const y5_opt_tensor t = tab[chunk_tensor[blockIdx.x]];
    const float inv_scale = hyper[Y5_OPT_INV_SCALE];
    float acc = 0.f;
    int nonfinite = 0;
    if (t.grad) {
        const long long e0 = static_cast<long long>(chunk_index[blockIdx.x]) * kOptChunk;
        const long long e1 = min(static_cast<long long>(t.numel), e0 + kOptChunk);
        const float* g = static_cast<const float*>(t.grad);
        for (long long i = e0 + threadIdx.x; i < e1; i += kOptThreads) {
            const float v = g[i] * inv_scale;
            if (!isfinite(v)) nonfinite = 1;
            acc = fmaf(v, v, acc);
        }
    }
    if (nonfinite) bad = 1;
    const float s = block_sum(acc, sh);
    __syncthreads();
    if (threadIdx.x == 0) {
        partial[2 * blockIdx.x] = s;
        partial[2 * blockIdx.x + 1] = bad ? 1.f : 0.f;
    }
}

// The step's scalars, shared by the update kernels: clip coefficient, overflow skip flag and EMA decay.  Every block
// re-reduces the per-chunk partials in the same fixed order: deterministic, no second launch, no atomics.  Block 0 publishes
// the norm and the skip flag to `hyper`.  s_coef / s_skip / s_decay are __shared__ and valid after the call.
__device__ __forceinline__ void opt_step_scalars(float* __restrict__ hyper, const float* __restrict__ partial, int n_chunks, int do_step,
                                                 float* sh, float& s_coef, float& s_skip, float& s_decay) {
    float acc = 0.f, badf = 0.f;
    if (do_step)
        for (int i = threadIdx.x; i < n_chunks; i += kOptThreads) {
            acc += partial[2 * i];
            badf = fmaxf(badf, partial[2 * i + 1]);
        }
    const float total = block_sum(acc, sh);
    __syncthreads();
    const float anybad = block_sum(badf, sh);
    if (threadIdx.x == 0) {
        const float norm = sqrtf(total);
        const float max_norm = hyper[Y5_OPT_MAX_NORM];
        // torch.nn.utils.clip_grad_norm_: coef = max_norm / (norm + 1e-6), clamped to 1
        s_coef = max_norm > 0.f ? fminf(max_norm / (norm + 1e-6f), 1.0f) : 1.0f;
        s_skip = (anybad > 0.f || !isfinite(norm)) ? 1.f : 0.f;
        const float upd = hyper[Y5_OPT_EMA_UPDATES] + 1.0f;  // ModelEMA.update: self.updates += 1; d = decay * (1 - exp(-updates / tau))
        s_decay = hyper[Y5_OPT_EMA_DECAY] * (1.0f - expf(-upd / hyper[Y5_OPT_EMA_TAU]));
        if (blockIdx.x == 0 && do_step) {
            hyper[Y5_OPT_OUT_NORM] = norm;
            hyper[Y5_OPT_OUT_SKIPPED] = s_skip;
        }
    }
    __syncthreads();
}

__global__ void __launch_bounds__(kOptThreads) opt_step_kernel(const y5_opt_tensor* __restrict__ tab, const int32_t* __restrict__ chunk_tensor,
                                                               const int32_t* __restrict__ chunk_index, int n_chunks, float* __restrict__ hyper,
                                                               const float* __restrict__ partial, int do_step, int do_ema, int zero_grad) {
    __shared__ float sh[kOptThreads / 32];
    __shared__ float s_coef, s_skip, s_decay;
    opt_step_scalars(hyper, partial, n_chunks, do_step, sh, s_coef, s_skip, s_decay);
    const y5_opt_tensor t = tab[chunk_tensor[blockIdx.x]];
    const long long e0 = static_cast<long long>(chunk_index[blockIdx.x]) * kOptChunk;
    const long long e1 = min(static_cast<long long>(t.numel), e0 + kOptChunk);
    const bool step = do_step && t.grad && t.mom && s_skip == 0.f;
    const float* hg = hyper + Y5_OPT_GROUPS + 4 * t.group;
    const float lr = hg[0], mom = hg[1], wd = hg[2], nesterov = hg[3];
    const float gscale = hyper[Y5_OPT_INV_SCALE] * s_coef;
    const float d = s_decay;
    float* p = static_cast<float*>(t.param);
    float* g = static_cast<float*>(t.grad);
    float* m = static_cast<float*>(t.mom);
    float* e = static_cast<float*>(t.ema);
    for (long long i = e0 + threadIdx.x; i < e1; i += kOptThreads) {
        float w = p[i];
        if (step) {
            float gi = g[i] * gscale;
            gi = fmaf(wd, w, gi);                    // d_p = d_p.add(p, alpha=weight_decay)
            const float b = fmaf(mom, m[i], gi);     // buf.mul_(momentum).add_(d_p)   (first step: buf = d_p, momentum buffer starts at 0)
            m[i] = b;
            if (nesterov != 0.f) gi = fmaf(mom, b, gi);  // d_p = d_p.add(buf, alpha=momentum)
            else gi = b;
            w = fmaf(-lr, gi, w);                    // p.add_(d_p, alpha=-lr)
            p[i] = w;
        }
        if (g && zero_grad) g[i] = 0.f;
        if (do_ema && e) e[i] = fmaf(d, e[i], (1.0f - d) * w);  // v *= d; v += (1 - d) * msd[k]
    }
}

// advances the EMA update counter once per step (separate 1-thread tail so every block of the step kernel reads the same value)
__global__ void opt_tick_kernel(float* hyper, int do_ema) {
    if (do_ema) hyper[Y5_OPT_EMA_UPDATES] += 1.0f;
}

// Adam / AdamW (torch.optim.Adam's foreach CUDA path, amsgrad = maximize = False) with the same un-scale, clip, skip and EMA as
// opt_step_kernel.  exp_avg is t.mom, exp_avg_sq sits `sq_offset` elements behind it; steps[t] is tensor t's step count BEFORE
// this step (adam_tick_kernel advances it afterwards, so every block of a tensor sees the same count).
__global__ void __launch_bounds__(kOptThreads) opt_adam_step_kernel(const y5_opt_tensor* __restrict__ tab, const int32_t* __restrict__ chunk_tensor,
                                                                    const int32_t* __restrict__ chunk_index, int n_chunks, float* __restrict__ hyper,
                                                                    const double* __restrict__ group_hyper, long long sq_offset,
                                                                    const float* __restrict__ steps, const float* __restrict__ partial, int do_ema,
                                                                    int zero_grad) {
    __shared__ float sh[kOptThreads / 32];
    __shared__ float s_coef, s_skip, s_decay;
    __shared__ float s_step_size, s_bc2_sqrt, s_w1, s_beta2, s_w2, s_eps, s_wd_mul, s_wd_add;
    const int ti = chunk_tensor[blockIdx.x];
    const y5_opt_tensor t = tab[ti];
    if (threadIdx.x == 0 && t.mom) {
        // torch computes these in Python doubles and hands fp32 scalars to its kernels: same doubles, same rounding points
        const double* h = group_hyper + Y5_ADAM_STRIDE * t.group;
        const double lr = h[Y5_ADAM_LR], b1 = h[Y5_ADAM_BETA1], b2 = h[Y5_ADAM_BETA2], wd = h[Y5_ADAM_WEIGHT_DECAY];
        const double step = static_cast<double>(steps[ti] + 1.0f);  // state["step"] += 1 (fp32), then step.item()
        s_step_size = static_cast<float>(-(lr / (1.0 - pow(b1, step))));
        s_bc2_sqrt = static_cast<float>(sqrt(1.0 - pow(b2, step)));
        s_w1 = static_cast<float>(1.0 - b1);
        s_beta2 = static_cast<float>(b2);
        s_w2 = static_cast<float>(1.0 - b2);
        s_eps = static_cast<float>(h[Y5_ADAM_EPS]);
        const bool decoupled = h[Y5_ADAM_DECOUPLED] != 0.0;
        s_wd_mul = decoupled ? static_cast<float>(1.0 - lr * wd) : 1.0f;  // AdamW: p.mul_(1 - lr * weight_decay)
        s_wd_add = decoupled ? 0.0f : static_cast<float>(wd);              // Adam:  grad = grad.add(p, alpha=weight_decay)
    }
    opt_step_scalars(hyper, partial, n_chunks, 1, sh, s_coef, s_skip, s_decay);  // ends with __syncthreads
    const long long e0 = static_cast<long long>(chunk_index[blockIdx.x]) * kOptChunk;
    const long long e1 = min(static_cast<long long>(t.numel), e0 + kOptChunk);
    const bool step = t.grad && t.mom && s_skip == 0.f;
    const float gscale = hyper[Y5_OPT_INV_SCALE] * s_coef;
    const float d = s_decay;
    const float step_size = s_step_size, bc2_sqrt = s_bc2_sqrt, w1 = s_w1, beta2 = s_beta2, w2 = s_w2, eps = s_eps;
    const float wd_mul = s_wd_mul, wd_add = s_wd_add;
    float* p = static_cast<float*>(t.param);
    float* g = static_cast<float*>(t.grad);
    float* m = static_cast<float*>(t.mom);
    float* v = m + sq_offset;
    float* e = static_cast<float*>(t.ema);
    for (long long i = e0 + threadIdx.x; i < e1; i += kOptThreads) {
        float w = p[i];
        if (step) {
            float gi = g[i] * gscale;
            w *= wd_mul;
            if (wd_add != 0.f) gi = fmaf(wd_add, w, gi);
            float mi = m[i];
            const float dm = gi - mi;
            mi = w1 < 0.5f ? fmaf(w1, dm, mi) : fmaf(-dm, 1.0f - w1, gi);  // torch's lerp(m, g, 1 - beta1)
            const float vi = fmaf(w2, gi * gi, v[i] * beta2);              // v.mul_(beta2).addcmul_(g, g, value=1 - beta2)
            const float den = sqrtf(vi) / bc2_sqrt + eps;                  // (v.sqrt() / sqrt(bc2)).add_(eps)
            w = fmaf(step_size, mi / den, w);                              // p.addcdiv_(m, den, value=-lr / bc1)
            m[i] = mi;
            v[i] = vi;
            p[i] = w;
        }
        if (g && zero_grad) g[i] = 0.f;
        if (do_ema && e) e[i] = fmaf(d, e[i], (1.0f - d) * w);
    }
}

// the Adam step's tail: tensor t's step count advances when it had a gradient and the step was not skipped; the EMA counter
// advances like opt_tick_kernel's
__global__ void adam_tick_kernel(const y5_opt_tensor* __restrict__ tab, int n_tensors, float* __restrict__ steps, float* __restrict__ hyper,
                                 int do_ema) {
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t < n_tensors && tab[t].grad && tab[t].mom && hyper[Y5_OPT_OUT_SKIPPED] == 0.f) steps[t] += 1.0f;
    if (t == 0 && do_ema) hyper[Y5_OPT_EMA_UPDATES] += 1.0f;
}

// Data-parallel gradient exchange, device side (reference utils/torch_utils.py:61-70 wraps the model in DistributedDataParallel;
// train.py:404-414): every gradient is copied where autograd left it into ONE contiguous fp32 arena -- a single multi-tensor
// launch -- so that the all-reduce is ONE NCCL call over the arena (85 MB for yolov5m: ~0.2 ms over NVLink) instead of
// per-parameter autograd hooks, bucket copies and copy-backs; y5_opt_step then reads the averaged gradients from the arena.
// Tensors without a gradient this step contribute zeros (what DDP's find-unused path reduces for them).
__global__ void __launch_bounds__(kOptThreads) grad_pack_kernel(const y5_opt_tensor* __restrict__ tab, const int32_t* __restrict__ chunk_tensor,
                                                                const int32_t* __restrict__ chunk_index, const int64_t* __restrict__ arena_offset,
                                                                float* __restrict__ arena, float* __restrict__ present) {
    const int ti = chunk_tensor[blockIdx.x];
    const y5_opt_tensor t = tab[ti];
    if (!t.mom) return;  // EMA-only entries (buffers) have no gradient slot
    if (chunk_index[blockIdx.x] == 0 && threadIdx.x == 0) present[ti] = t.grad ? 1.0f : 0.0f;
    const long long e0 = static_cast<long long>(chunk_index[blockIdx.x]) * kOptChunk;
    const long long e1 = min(static_cast<long long>(t.numel), e0 + kOptChunk);
    float* dst = arena + arena_offset[ti];  // offsets are multiples of 4 elements and the arena is 16-byte aligned
    const float* g = static_cast<const float*>(t.grad);
    if (g && (reinterpret_cast<uintptr_t>(g) & 15) == 0) {
        const long long v1 = e0 + ((e1 - e0) & ~3LL);
        for (long long i = e0 + 4LL * threadIdx.x; i < v1; i += 4LL * kOptThreads)
            *reinterpret_cast<float4*>(dst + i) = __ldg(reinterpret_cast<const float4*>(g + i));
        for (long long i = v1 + threadIdx.x; i < e1; i += kOptThreads) dst[i] = g[i];
    } else {
        for (long long i = e0 + threadIdx.x; i < e1; i += kOptThreads) dst[i] = g ? g[i] : 0.0f;
    }
}

// after the all-reduce: a tensor whose gradient was absent on EVERY rank (present[] averaged to 0) keeps a NULL gradient in the
// arena table, so y5_opt_step skips it exactly like the single-process step skips a parameter without .grad
__global__ void grad_bind_kernel(y5_opt_tensor* __restrict__ arena_tab, int n_tensors, const int64_t* __restrict__ arena_offset,
                                 float* __restrict__ arena, const float* __restrict__ present) {
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n_tensors || !arena_tab[t].mom) return;
    arena_tab[t].grad = present[t] > 0.0f ? static_cast<void*>(arena + arena_offset[t]) : nullptr;
}

}  // namespace y5

using namespace y5;

extern "C" Y5_API int32_t y5_opt_chunk_elems(void) { return kOptChunk; }

extern "C" Y5_API int y5_opt_step(const y5_opt_tensor* table, const int32_t* chunk_tensor, const int32_t* chunk_index, int32_t n_chunks,
                                  float* hyper, float* partial, int32_t do_step, int32_t do_ema, int32_t zero_grad, void* stream) {
    if (n_chunks <= 0) return 0;
    if (!table || !chunk_tensor || !chunk_index || !hyper || (do_step && !partial)) return set_error(Y5_E_INVALID, "opt_step: null pointer");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    if (do_step)
        if (int e = launch("opt_step", opt_grad_norm_kernel, {n_chunks, kOptThreads, 0, st}, table, chunk_tensor, chunk_index, hyper, partial)) return e;
    if (int e = launch("opt_step", opt_step_kernel, {n_chunks, kOptThreads, 0, st}, table, chunk_tensor, chunk_index, n_chunks, hyper, partial,
                       do_step, do_ema, zero_grad))
        return e;
    return launch("opt_step", opt_tick_kernel, {1, 1, 0, st}, hyper, do_ema);
}

extern "C" Y5_API int y5_adam_step(const y5_opt_tensor* table, int32_t n_tensors, const int32_t* chunk_tensor, const int32_t* chunk_index,
                                   int32_t n_chunks, float* hyper, const double* group_hyper, int64_t sq_offset, float* steps, float* partial,
                                   int32_t do_ema, int32_t zero_grad, void* stream) {
    if (n_chunks <= 0) return 0;
    if (!table || !chunk_tensor || !chunk_index || !hyper || !group_hyper || !steps || !partial)
        return set_error(Y5_E_INVALID, "adam_step: null pointer");
    if (n_tensors <= 0 || sq_offset < 0) return set_error(Y5_E_INVALID, "adam_step: n_tensors %d, sq_offset %lld", n_tensors, (long long)sq_offset);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    if (int e = launch("adam_step", opt_grad_norm_kernel, {n_chunks, kOptThreads, 0, st}, table, chunk_tensor, chunk_index, hyper, partial)) return e;
    if (int e = launch("adam_step", opt_adam_step_kernel, {n_chunks, kOptThreads, 0, st}, table, chunk_tensor, chunk_index, n_chunks, hyper,
                       group_hyper, sq_offset, steps, partial, do_ema, zero_grad))
        return e;
    return launch("adam_step", adam_tick_kernel, {(n_tensors + 255) / 256, 256, 0, st}, table, n_tensors, steps, hyper, do_ema);
}

extern "C" Y5_API int y5_grad_pack(const y5_opt_tensor* table, const int32_t* chunk_tensor, const int32_t* chunk_index, int32_t n_chunks,
                                   const int64_t* arena_offset, float* arena, float* present, void* stream) {
    if (n_chunks <= 0) return 0;
    if (!table || !chunk_tensor || !chunk_index || !arena_offset || !arena || !present) return set_error(Y5_E_INVALID, "grad_pack: null pointer");
    if (reinterpret_cast<uintptr_t>(arena) & 15) return set_error(Y5_E_INVALID, "grad_pack: the arena must be 16-byte aligned");
    return launch("grad_pack", grad_pack_kernel, {n_chunks, kOptThreads, 0, static_cast<cudaStream_t>(stream)}, table, chunk_tensor, chunk_index,
                  arena_offset, arena, present);
}

extern "C" Y5_API int y5_grad_bind(y5_opt_tensor* arena_table, int32_t n_tensors, const int64_t* arena_offset, float* arena, const float* present,
                                   void* stream) {
    if (n_tensors <= 0) return 0;
    if (!arena_table || !arena_offset || !arena || !present) return set_error(Y5_E_INVALID, "grad_bind: null pointer");
    return launch("grad_bind", grad_bind_kernel, {(n_tensors + 255) / 256, 256, 0, static_cast<cudaStream_t>(stream)}, arena_table, n_tensors,
                  arena_offset, arena, present);
}
