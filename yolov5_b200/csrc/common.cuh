// Thin inline-PTX layer for sm_90a: mbarrier, TMA (tiled + im2col), wgmma descriptors / fences, register reallocation.
// Everything the kernels in this directory need from the Hopper programming model lives here; there is no dependency
// on CUTLASS/CuTe.  Descriptor bit layouts follow the PTX ISA "matrix descriptor" table of the wgmma section.
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

namespace y5 {

// ---------------------------------------------------------------------------------------------------------------------
// small helpers
// ---------------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return static_cast<uint32_t>(__cvta_generic_to_shared(p)); }

__device__ __forceinline__ bool elect_one() {
    uint32_t pred = 0;
    asm volatile(
        "{\n\t.reg .pred P;\n\t"
        "elect.sync _|P, 0xffffffff;\n\t"
        "selp.b32 %0, 1, 0, P;\n\t}"
        : "=r"(pred));
    return pred != 0;
}

// ---------------------------------------------------------------------------------------------------------------------
// mbarrier
// ---------------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("{\n\t.reg .b64 st;\n\tmbarrier.arrive.shared::cta.b64 st, [%0];\n\t}" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("{\n\t.reg .b64 st;\n\tmbarrier.arrive.expect_tx.shared::cta.b64 st, [%0], %1;\n\t}" ::"r"(smem_u32(bar)),
                 "r"(bytes)
                 : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n\t.reg .pred P;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 P, [%1], %2;\n\t"
        "selp.b32 %0, 1, 0, P;\n\t}"
        : "=r"(ok)
        : "r"(smem_u32(bar)), "r"(parity)
        : "memory");
    return ok != 0;
}
// try_wait with a suspend-time hint: the thread sleeps in hardware until the phase completes or ~`ns` nanoseconds pass, instead of
// re-issuing the probe (the round-1 spin loop cost 17 % of all issued instructions of the store-bound layers under ncu)
__device__ __forceinline__ bool mbar_try_wait_hint(uint64_t* bar, uint32_t parity, uint32_t ns) {
    uint32_t ok;
    asm volatile(
        "{\n\t.reg .pred P;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 P, [%1], %2, %3;\n\t"
        "selp.b32 %0, 1, 0, P;\n\t}"
        : "=r"(ok)
        : "r"(smem_u32(bar)), "r"(parity), "r"(ns)
        : "memory");
    return ok != 0;
}
// Bounded wait: a pipeline bug must surface as a trapped kernel (launch error), never as a hung GPU.  No printf here: a
// function call inside a kernel that issues wgmma makes ptxas serialise every wgmma of the kernel.
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    if (mbar_try_wait(bar, parity)) return;
    uint32_t spins = 0;
    while (!mbar_try_wait_hint(bar, parity, 20000u)) {       // <= 20 us asleep per probe
        if (++spins > 200000u) __trap();                     // ~4 s
    }
}

// ---------------------------------------------------------------------------------------------------------------------
// TMA
// ---------------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* m) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
__device__ __forceinline__ void tma_load_2d(const CUtensorMap* m, uint64_t* bar, void* dst, int c0, int c1) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];" ::"r"(
            smem_u32(dst)),
        "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
        : "memory");
}
__device__ __forceinline__ void tma_load_4d(const CUtensorMap* m, uint64_t* bar, void* dst, int c0, int c1, int c2, int c3) {
    asm volatile(
        "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];" ::"r"(
            smem_u32(dst)),
        "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
        : "memory");
}
// multicast variant: the tile lands at the same CTA-relative smem offset of every CTA in `mask`, and each of those
// CTAs' mbarrier (same offset) receives the complete_tx
__device__ __forceinline__ void tma_load_2d_mcast(const CUtensorMap* m, uint64_t* bar, void* dst, int c0, int c1, uint16_t mask) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster"
        " [%0], [%1, {%3, %4}], [%2], %5;" ::"r"(smem_u32(dst)),
        "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "h"(mask)
        : "memory");
}
// shared::cluster address of `p` (a shared-memory object of this CTA) as seen in CTA `rank` of the cluster (same offset)
__device__ __forceinline__ uint32_t mapa_u32(const void* p, uint32_t rank) {
    uint32_t r;
    asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(smem_u32(p)), "r"(rank));
    return r;
}
// arrive (count 1) on a barrier anywhere in the cluster
__device__ __forceinline__ void mbar_arrive_cluster(uint32_t bar_addr) {
    asm volatile("mbarrier.arrive.release.cluster.shared::cluster.b64 _, [%0];" ::"r"(bar_addr) : "memory");
}
__device__ __forceinline__ uint32_t cluster_ctarank() { uint32_t r; asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r)); return r; }
__device__ __forceinline__ uint32_t cluster_nctarank() { uint32_t r; asm volatile("mov.u32 %0, %%cluster_nctarank;" : "=r"(r)); return r; }
__device__ __forceinline__ void cluster_sync_all() {
    asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");
    asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");
}
// im2col mode over an NHWC tensor (dims C,W,H,N): {c,w,h,n} is the base pixel of the first filter window of the tile,
// {off_w, off_h} the filter tap.  The unit walks `pixelsPerColumn` windows in (w,h,n) order, zero-filling padding.
__device__ __forceinline__ void tma_load_im2col_4d(const CUtensorMap* m, uint64_t* bar, void* dst, int c, int w, int h,
                                                   int n, uint16_t off_w, uint16_t off_h) {
    asm volatile(
        "cp.async.bulk.tensor.4d.shared::cluster.global.im2col.mbarrier::complete_tx::bytes"
        " [%0], [%1, {%3, %4, %5, %6}], [%2], {%7, %8};" ::"r"(smem_u32(dst)),
        "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c), "r"(w), "r"(h), "r"(n), "h"(off_w), "h"(off_h)
        : "memory");
}
__device__ __forceinline__ void tma_store_2d(const CUtensorMap* m, const void* src, int c0, int c1) {
    asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];" ::"l"(
                     reinterpret_cast<uint64_t>(m)),
                 "r"(smem_u32(src)), "r"(c0), "r"(c1)
                 : "memory");
}
__device__ __forceinline__ void tma_store_4d(const CUtensorMap* m, const void* src, int c0, int c1, int c2, int c3) {
    asm volatile("cp.async.bulk.tensor.4d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5}], [%1];" ::"l"(
                     reinterpret_cast<uint64_t>(m)),
                 "r"(smem_u32(src)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
                 : "memory");
}
__device__ __forceinline__ void tma_store_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
__device__ __forceinline__ void tma_store_wait_read0() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
__device__ __forceinline__ void tma_store_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }

// ---------------------------------------------------------------------------------------------------------------------
// wgmma (warpgroup MMA) -- the instruction wrappers themselves are in wgmma.cuh
// ---------------------------------------------------------------------------------------------------------------------
// K-major shared-memory operand descriptor.  Tile rows are `row_bytes` (32/64/128) wide with the matching TMA swizzle,
// 8-row groups packed back to back (SBO = 8*row_bytes); LBO is unused for swizzled K-major layouts (encoded 1).
// Stepping 16 elements along K is +32 bytes on the start address (+2 on the low word).
__device__ __forceinline__ uint32_t gmma_desc_hi(uint32_t row_bytes) {
    const uint32_t layout = row_bytes == 128 ? 1u : (row_bytes == 64 ? 2u : 3u);  // SW128 / SW64 / SW32
    return (((8u * row_bytes) >> 4) & 0x3FFFu) | (layout << 30);
}
__device__ __forceinline__ uint32_t gmma_desc_lo(uint32_t saddr) { return ((saddr >> 4) & 0x3FFFu) | (1u << 16); }
__device__ __forceinline__ uint64_t gmma_desc(uint32_t lo, uint32_t hi) { return (static_cast<uint64_t>(hi) << 32) | lo; }

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// the accumulator registers must not be touched by other instructions while a wgmma that uses them is in flight
template <int N>
__device__ __forceinline__ void fence_regs(float (&d)[N]) {
#pragma unroll
    for (int i = 0; i < N; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// per-warpgroup register budget: the producer warpgroup gives registers back, the MMA / epilogue warpgroups take them
template <uint32_t R>
__device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(R)); }
template <uint32_t R>
__device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(R)); }

// Programmatic dependent launch: `wait` blocks until the grid this one depends on has completed and its writes are
// visible; `launch_dependents` lets the next grid in the stream start its prologue as soon as SMs free up.
__device__ __forceinline__ void griddep_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void griddep_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

__device__ __forceinline__ uint32_t ld_shared_u32(uint32_t addr) {
    uint32_t v;
    asm volatile("ld.shared.b32 %0, [%1];" : "=r"(v) : "r"(addr) : "memory");
    return v;
}
__device__ __forceinline__ void st_shared_u32(uint32_t addr, uint32_t v) {
    asm volatile("st.shared.b32 [%0], %1;" ::"r"(addr), "r"(v) : "memory");
}

__device__ __forceinline__ void named_bar_sync(uint32_t id, uint32_t nthreads) {
    asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}

// ---------------------------------------------------------------------------------------------------------------------
// numeric helpers
// ---------------------------------------------------------------------------------------------------------------------
#ifndef Y5_SILU_EXACT
// x*sigmoid(x) = h + h*tanh(h), h = x/2: one MUFU op per element (tanh.approx) instead of two (ex2 + rcp).  Faithfully rounded
// to fp16 for x >= -4 and to bf16 for x >= -8 (at most 0.58 / 0.82 ulp, measured on an H100 over every input value), but not
// below: there the two terms cancel, tanh.approx's absolute error near -1 becomes most of the result (all of it once tanh
// rounds to -1, x < -17), up to 30 ulp in fp16 and 255 in bf16.  The conv epilogue takes silu_tail for those inputs.
// -DY5_SILU_EXACT restores the ex2 + rcp form.
__device__ __forceinline__ float silu_f(float x) {
    const float h = 0.5f * x;
    float t;
    asm("tanh.approx.f32 %0, %1;" : "=f"(t) : "f"(h));
    return fmaf(h, t, h);
}
// same with h = x / 2 already formed (the conv epilogue folds the halving into its bias FMA)
__device__ __forceinline__ float silu_from_half(float h) {
    float t;
    asm("tanh.approx.f32 %0, %1;" : "=f"(t) : "f"(h));
    return fmaf(h, t, h);
}
#else
__device__ __forceinline__ float silu_f(float x) { return __fdividef(x, 1.0f + __expf(-x)); }
__device__ __forceinline__ float silu_from_half(float h) { return silu_f(2.0f * h); }
#endif
// x*sigmoid(x) for x <= -4 without cancellation: e = e^x <= 0.0184, sigmoid = e / (1 + e) = e (1 - e + e^2 - e^3) to e^4 < 2^-23
// relative.  ex2 without .ftz keeps the subnormal e of x < -87, which bf16 results still resolve.
__device__ __forceinline__ float silu_tail(float x) {
    float e;
    asm("ex2.approx.f32 %0, %1;" : "=f"(e) : "f"(1.44269504088896341f * x));
    return x * e * fmaf(e, fmaf(e, 1.0f - e, -1.0f), 1.0f);
}
__device__ __forceinline__ float sigmoid_f(float x) { return __fdividef(1.0f, 1.0f + __expf(-x)); }

__device__ __forceinline__ uint32_t pack2(float a, float b, bool bf16) {
    if (bf16) {
        __nv_bfloat162 t = __floats2bfloat162_rn(a, b);
        return *reinterpret_cast<uint32_t*>(&t);
    }
    __half2 t = __floats2half2_rn(a, b);
    return *reinterpret_cast<uint32_t*>(&t);
}
__device__ __forceinline__ float2 unpack2(uint32_t u, bool bf16) {
    if (bf16) return __bfloat1622float2(*reinterpret_cast<__nv_bfloat162*>(&u));
    return __half22float2(*reinterpret_cast<__half2*>(&u));
}
__device__ __forceinline__ uint16_t pack1(float a, bool bf16) {
    if (bf16) {
        __nv_bfloat16 t = __float2bfloat16_rn(a);
        return *reinterpret_cast<uint16_t*>(&t);
    }
    __half t = __float2half_rn(a);
    return *reinterpret_cast<uint16_t*>(&t);
}
__device__ __forceinline__ float unpack1(uint16_t u, bool bf16) {
    if (bf16) return __bfloat162float(*reinterpret_cast<__nv_bfloat16*>(&u));
    return __half2float(*reinterpret_cast<__half*>(&u));
}

}  // namespace y5
