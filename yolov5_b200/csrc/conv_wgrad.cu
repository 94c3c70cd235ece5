// Weight gradient of a convolution for sm_90a:
//     dW[co][r][s][ci] = sum over output pixels m of  dY[m][co] * X[pixel(m) shifted by tap (r,s)][ci]
// i.e. per filter tap a GEMM  dW_tap[Cout, Cin] = dY[M, Cout]^T * X_tap[M, Cin]  whose reduction dimension is the pixel
// index -- the dimension that is OUTERMOST in the NHWC activations.  Both operands are therefore fed to wgmma as
// MN-major shared-memory tiles (transpose flags set): a TMA box of [P pixels][64 channels] (128-byte rows, 128-byte
// swizzle) is exactly the canonical MN-major SW128 layout ((8,n),(8,k)):((1,LBO),(8,SBO)) in 16-byte units -- each pixel is
// one 128-byte line of 64 channels, 8 pixels form a 1024-byte swizzle atom (SBO).  So neither dY nor X is ever transposed
// in memory; the tensor core does it on the fly.
//   A (dY)   : 1-2 boxes [P px][64 co] per stage -> 128 output channels per CTA, one 64-channel box per consumer warpgroup
//              (the upper box is not fetched, and its warpgroup idles, when the layer has <= 64 of them left)
//   B (X_tap): n boxes [P px][64 ci] per stage per tap (n <= 4); hardware im2col for k > 1 or strided convs (same tensor
//              map type as the forward kernel), plain 2-D tiles for 1x1/s1
// One CTA = one (co tile, tap group, ci tile, pixel range) work item.  A tap group is up to G filter taps whose
// accumulators sit side by side in registers (G * n <= 4 blocks of m64 x n64 = 128 fp32 registers per thread): the dY tile
// of a pixel block is fetched once and multiplied with the G shifted X tiles, which divides the dY traffic of 3x3 layers
// by G.  P (pixels per pipeline stage) is 128 when a stage of 128-pixel boxes stays within 56 KB -- one dY box pair and one
// X box, i.e. 1x1 filters with Cin <= 64 -- and 64 otherwise, which amortises the per-stage barrier / TMA issue costs.
// The fp32 tiles are added to the fp32 gradient with vector reductions (red.global.add.v2.f32); the pixel range is split
// so the grid is about one CTA per SM (one wave).
// Summation order across pixel ranges is not fixed (fp32 atomics), like cuDNN's default wgrad.
//
// Gradient of reference models/common.py:86-88 (Conv.forward, the nn.Conv2d weight) / models/yolo.py:97 (Detect.m[i]).
#include <cstdio>
#include <cstdlib>
#include <mutex>

#include "../../include/y5b200.h"
#include "common.cuh"
#include "host_util.h"
#include "wgmma.cuh"

namespace y5 {

constexpr int kWgThreads = 128 + 256;  // warpgroup 0: TMA producer (warp 0), warpgroups 1-2: MMA + reductions, 64 co each
constexpr int kWgCo = 128;            // output channels per tile
constexpr int kWgSlots = 4;           // accumulator blocks (tap, 64-channel ci block) per thread: 4 x 32 fp32 registers
constexpr int kWgStagesMax = 6;

struct WgradParams {
    int M, Cout, Cin;
    int kh, kw, stride, pad_h, pad_w, Wo, HoWo;
    int linear;                 // 1x1 / stride 1 / no padding: X tiles are plain 2-D boxes of the [M, Cin] matrix
    int n_blocks;               // 64-channel blocks of Cin per tile
    int ci_tiles, taps;
    int group, tap_groups;      // taps per CTA, number of tap groups
    int pix;                    // pixels (GEMM K) per pipeline stage: 64 | 128
    int kblocks, splits, kb_per_split;
    int stages;
    uint32_t box_bytes, stage_bytes;
    int is_bf16;
    float* dw;
};

template <bool BF16>
__device__ __forceinline__ void wgrad_mma(float (&acc)[kWgSlots][32], int nslots, int n_blocks, uint32_t a16, uint32_t b16, uint32_t box16,
                                          uint32_t lbo, uint32_t dhi, int ksteps, uint32_t first) {
#pragma unroll
    for (int t = 0; t < kWgSlots; ++t) {
        if (t < nslots) {
            const int g = t / n_blocks, j = t - g * n_blocks;
            const uint32_t bt16 = b16 + (g * n_blocks + j) * box16;
            for (int k = 0; k < ksteps; ++k)  // 16 pixels = two 8-pixel swizzle atoms = +2048 bytes
                Wgmma<64>::run<BF16, 1, 1>(acc[t], gmma_desc((a16 + k * 128) | lbo, dhi), gmma_desc((bt16 + k * 128) | lbo, dhi),
                                           (first == 0 || k != 0) ? 1u : 0u);
        }
    }
}

__global__ void __launch_bounds__(kWgThreads, 1)
conv_wgrad_kernel(const __grid_constant__ CUtensorMap tmDy, const __grid_constant__ CUtensorMap tmX, const WgradParams p) {
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint8_t* ring = smem;
    uint64_t* full = reinterpret_cast<uint64_t*>(smem + p.stages * p.stage_bytes);
    uint64_t* empty = full + kWgStagesMax;

    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;

    // work item
    int t = blockIdx.x;
    const int split = t % p.splits;
    t /= p.splits;
    const int ci_tile = t % p.ci_tiles;
    t /= p.ci_tiles;
    const int tg = t % p.tap_groups;
    const int co_tile = t / p.tap_groups;
    const int tap0 = tg * p.group;
    const int ntaps = min(p.group, p.taps - tap0);
    const int co0 = co_tile * kWgCo;
    const int a_boxes = p.Cout - co0 > 64 ? 2 : 1;
    const int bn = p.n_blocks * 64;
    const int ci0 = ci_tile * bn;
    const int kb0 = split * p.kb_per_split;
    const int kb1 = min(p.kblocks, kb0 + p.kb_per_split);
    const int nkb = kb1 - kb0;
    // stage layout: [A box 0][A box 1][tap 0: n boxes][tap 1: n boxes]...
    const uint32_t tx_bytes = (a_boxes + ntaps * p.n_blocks) * p.box_bytes;

    if (threadIdx.x == 0) {
        tma_prefetch_desc(&tmDy);
        tma_prefetch_desc(&tmX);
        for (int s = 0; s < kWgStagesMax; ++s) {
            mbar_init(&full[s], 1);
            mbar_init(&empty[s], a_boxes);  // one arrival per working consumer warpgroup
        }
        fence_barrier_init();
    }
    __syncthreads();
    griddep_wait();  // PDL: barrier init above overlaps the predecessor's tail
    griddep_launch_dependents();

    if (warp < 4) {
        setmaxnreg_dec<40>();
        if (warp != 0) return;
        // ===================================== TMA producer =====================================
        int st = 0;
        uint32_t ph = 0;
        for (int kb = kb0; kb < kb1; ++kb) {
            const int m0 = kb * p.pix;
            int img = 0, y0 = 0, x0 = 0;
            if (!p.linear) {
                img = m0 / p.HoWo;
                const int rem = m0 - img * p.HoWo;
                const int oy = rem / p.Wo;
                y0 = oy * p.stride - p.pad_h;
                x0 = (rem - oy * p.Wo) * p.stride - p.pad_w;
            }
            mbar_wait(&empty[st], ph ^ 1);
            if (elect_one()) {
                uint8_t* dst = ring + st * p.stage_bytes;
                mbar_arrive_expect_tx(&full[st], tx_bytes);
                tma_load_2d(&tmDy, &full[st], dst, co0, m0);
                if (a_boxes == 2) tma_load_2d(&tmDy, &full[st], dst + p.box_bytes, co0 + 64, m0);
                for (int g = 0; g < ntaps; ++g) {
                    const int tap = tap0 + g;
                    const int r = tap / p.kw, s = tap - r * p.kw;
                    for (int j = 0; j < p.n_blocks; ++j) {
                        uint8_t* b_dst = dst + (2 + g * p.n_blocks + j) * p.box_bytes;
                        if (p.linear) tma_load_2d(&tmX, &full[st], b_dst, ci0 + j * 64, m0);
                        else
                            tma_load_im2col_4d(&tmX, &full[st], b_dst, ci0 + j * 64, x0, y0, img, static_cast<uint16_t>(s),
                                               static_cast<uint16_t>(r));
                    }
                }
            }
            __syncwarp();
            if (++st == p.stages) { st = 0; ph ^= 1; }
        }
        return;
    }

    // ===================================== MMA + fp32 reductions =====================================
    setmaxnreg_inc<232>();
    const int wg = (warp >> 2) - 1;  // output channels [co0 + 64 wg, co0 + 64 wg + 64): dY box wg
    if (wg >= a_boxes || nkb <= 0) return;
    // MN-major SW128 descriptors: SBO = 1024 B between 8-pixel groups, LBO = one [P px][64 ch] box between 64-channel blocks
    const uint32_t dhi = ((1024u >> 4) & 0x3FFFu) | (1u << 30);
    const uint32_t lbo = ((p.box_bytes >> 4) & 0x3FFFu) << 16;
    const uint32_t ring16 = (smem_u32(ring) >> 4) & 0x3FFFu;
    const uint32_t box16 = p.box_bytes >> 4;
    const int ksteps = p.pix / 16;
    const int nslots = ntaps * p.n_blocks;
    const bool signal = (threadIdx.x & 127) == 0;
    float acc[kWgSlots][32];
#pragma unroll
    for (int s = 0; s < kWgSlots; ++s)
#pragma unroll
        for (int i = 0; i < 32; ++i) acc[s][i] = 0.0f;
    int st = 0;
    uint32_t ph = 0;
    for (int i = 0; i < nkb; ++i) {
        mbar_wait(&full[st], ph);
        const uint32_t a16 = ring16 + ((st * p.stage_bytes) >> 4);
#pragma unroll
        for (int s = 0; s < kWgSlots; ++s) fence_regs(acc[s]);
        wgmma_fence();
        if (p.is_bf16) wgrad_mma<true>(acc, nslots, p.n_blocks, a16 + wg * box16, a16 + 2 * box16, box16, lbo, dhi, ksteps, i == 0);
        else wgrad_mma<false>(acc, nslots, p.n_blocks, a16 + wg * box16, a16 + 2 * box16, box16, lbo, dhi, ksteps, i == 0);
        wgmma_commit();
        wgmma_wait<0>();
#pragma unroll
        for (int s = 0; s < kWgSlots; ++s) fence_regs(acc[s]);
        if (signal) mbar_arrive(&empty[st]);
        if (++st == p.stages) { st = 0; ph ^= 1; }
    }
    // accumulator fragment: rows (co) 16*warp + lane/4 + 8h, columns (ci) 8q + 2*(lane%4) + e of each 64 x 64 block
    const bool vec_ok = (p.Cin & 1) == 0;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        const int co = co0 + wg * 64 + (warp & 3) * 16 + (lane >> 2) + 8 * h;
        if (co >= p.Cout) continue;
#pragma unroll
        for (int s = 0; s < kWgSlots; ++s) {
            if (s >= nslots) continue;
            const int g = s / p.n_blocks, j = s - g * p.n_blocks;
            float* row = p.dw + (static_cast<size_t>(co) * p.taps + tap0 + g) * p.Cin;
#pragma unroll
            for (int q = 0; q < 8; ++q) {
                const int ci = ci0 + j * 64 + q * 8 + 2 * (lane & 3);
                const float v0 = acc[s][4 * q + 2 * h], v1 = acc[s][4 * q + 2 * h + 1];
                if (vec_ok && ci + 1 < p.Cin) {
                    asm volatile("red.global.add.v2.f32 [%0], {%1, %2};" ::"l"(row + ci), "f"(v0), "f"(v1) : "memory");
                } else {
                    if (ci < p.Cin) atomicAdd(row + ci, v0);
                    if (ci + 1 < p.Cin) atomicAdd(row + ci + 1, v1);
                }
            }
        }
    }
}

}  // namespace y5

using namespace y5;

extern "C" Y5_API int y5_conv_wgrad(const y5_wgrad_desc* d, void* stream) {
    if (!d || !d->in || !d->dout || !d->dweight) return set_error(Y5_E_INVALID, "wgrad: null pointer");
    if (d->dtype != Y5_F16 && d->dtype != Y5_BF16) return set_error(Y5_E_UNSUPPORTED, "wgrad: dtype must be fp16 or bf16");
    if (d->batch <= 0 || d->in_h <= 0 || d->in_w <= 0 || d->in_c <= 0 || d->out_c <= 0 || d->ksize <= 0 || d->stride <= 0 || d->pad < 0)
        return set_error(Y5_E_INVALID, "wgrad: bad shape");
    if ((d->in_pitch % 8) || (d->dout_pitch % 8) || (reinterpret_cast<uintptr_t>(d->in) & 15) || (reinterpret_cast<uintptr_t>(d->dout) & 15) ||
        (reinterpret_cast<uintptr_t>(d->dweight) & 15))
        return set_error(Y5_E_INVALID, "wgrad: views must be 16-byte aligned with pitches that are multiples of 8 elements");
    const bool strided_view = d->in_x_stride || d->in_y_stride || d->in_n_stride;
    if ((!strided_view && d->in_pitch < d->in_c) || d->dout_pitch < d->out_c)
        return set_error(Y5_E_INVALID, "wgrad: pitch smaller than channel count");
    if ((d->in_x_stride % 8) || (d->in_y_stride % 8) || (d->in_n_stride % 8) || d->kw < 0 || d->pad_w < 0)
        return set_error(Y5_E_INVALID, "wgrad: strides must be multiples of 8 elements");
    const int k = d->ksize;                       // filter rows
    const int kw = d->kw ? d->kw : d->ksize;      // filter columns
    const int pad_w = d->kw ? d->pad_w : d->pad;
    const int Ho = (d->in_h + 2 * d->pad - k) / d->stride + 1, Wo = (d->in_w + 2 * pad_w - kw) / d->stride + 1;
    if (Ho <= 0 || Wo <= 0) return set_error(Y5_E_INVALID, "wgrad: empty output");
    const long long M = static_cast<long long>(d->batch) * Ho * Wo;
    if (M > 0x7fffffffLL) return set_error(Y5_E_UNSUPPORTED, "wgrad: too many pixels");
    cudaStream_t st = static_cast<cudaStream_t>(stream);

    WgradParams p{};
    p.M = static_cast<int>(M);
    p.Cout = d->out_c;
    p.Cin = d->in_c;
    p.kh = k;
    p.kw = kw;
    p.stride = d->stride;
    p.pad_h = d->pad;
    p.pad_w = pad_w;
    p.Wo = Wo;
    p.HoWo = Ho * Wo;
    p.linear = (k == 1 && kw == 1 && d->stride == 1 && d->pad == 0 && pad_w == 0 && !strided_view) ? 1 : 0;
    p.taps = k * kw;
    const int blocks_total = (d->in_c + 63) / 64;
    p.n_blocks = blocks_total < 4 ? blocks_total : 4;
    p.ci_tiles = (blocks_total + p.n_blocks - 1) / p.n_blocks;
    // balance the blocks over the ci tiles (e.g. 5 blocks -> 3 + 2, not 4 + 1)
    p.n_blocks = (blocks_total + p.ci_tiles - 1) / p.ci_tiles;
    const int co_tiles = (d->out_c + kWgCo - 1) / kWgCo;
    const int bn = p.n_blocks * 64;
    // taps per CTA: the accumulators of a group share the consumer threads' registers (kWgSlots blocks of 64 ci); groups are
    // balanced (9 taps, limit 4 -> 3 + 3 + 3)
    const unsigned stage_kb = 56u;
    int gmax = kWgSlots / p.n_blocks;
    if (gmax < 1) gmax = 1;
    p.tap_groups = (p.taps + gmax - 1) / gmax;
    p.group = (p.taps + p.tap_groups - 1) / p.tap_groups;
    // pixels per stage: 128 if such a stage stays within ~56 KB (>= 3 stages in flight), else 64.  (A stage holds two dY boxes
    // and at least one X box, so 256-pixel stages, 3 x 32 KB, never fit.)
    p.pix = static_cast<uint32_t>(2 + p.group * p.n_blocks) * 128u * 128u <= stage_kb * 1024u ? 128 : 64;
    p.box_bytes = p.pix * 128u;
    p.kblocks = (p.M + p.pix - 1) / p.pix;
    const long long items = static_cast<long long>(co_tiles) * p.tap_groups * p.ci_tiles;
    long long want = (sm_count() + items - 1) / items;  // pixel ranges per tile: one CTA per SM, one wave
    if (want < 1) want = 1;
    if (want > p.kblocks) want = p.kblocks;
    p.kb_per_split = static_cast<int>((p.kblocks + want - 1) / want);
    p.splits = (p.kblocks + p.kb_per_split - 1) / p.kb_per_split;  // no empty range
    p.stage_bytes = (2 + p.group * p.n_blocks) * p.box_bytes;
    p.stages = static_cast<int>((200u * 1024u) / p.stage_bytes);
    if (p.stages > kWgStagesMax) p.stages = kWgStagesMax;
    if (p.stages < 2) return set_error(Y5_E_UNSUPPORTED, "wgrad: stage does not fit shared memory");
    p.is_bf16 = d->dtype == Y5_BF16;
    p.dw = d->dweight;

    CUtensorMap tmDy, tmX;
    {
        cuuint64_t dims[2] = {(cuuint64_t)d->out_c, (cuuint64_t)M};
        cuuint64_t str[1] = {(cuuint64_t)d->dout_pitch * 2};
        cuuint32_t box[2] = {64, (cuuint32_t)p.pix};
        int e = encode_tiled(&tmDy, d->dtype, d->dout, 2, dims, str, box, CU_TENSOR_MAP_SWIZZLE_128B, "wgrad dY");
        if (e) return e;
    }
    if (p.linear) {
        cuuint64_t dims[2] = {(cuuint64_t)d->in_c, (cuuint64_t)M};
        cuuint64_t str[1] = {(cuuint64_t)d->in_pitch * 2};
        cuuint32_t box[2] = {64, (cuuint32_t)p.pix};
        int e = encode_tiled(&tmX, d->dtype, d->in, 2, dims, str, box, CU_TENSOR_MAP_SWIZZLE_128B, "wgrad X");
        if (e) return e;
    } else {
        const long long xs = d->in_x_stride ? d->in_x_stride : d->in_pitch;
        const long long ys = d->in_y_stride ? d->in_y_stride : xs * d->in_w;
        const long long ns = d->in_n_stride ? d->in_n_stride : ys * d->in_h;
        int e = encode_im2col(&tmX, d->dtype, d->in, d->in_c, d->in_w, d->in_h, d->batch, xs, ys, ns, k, kw, d->stride, d->pad, pad_w, 64,
                              p.pix, CU_TENSOR_MAP_SWIZZLE_128B);
        if (e) return e;
    }
    const size_t dw_bytes = static_cast<size_t>(d->out_c) * p.taps * d->in_c * sizeof(float);
    if (!d->accumulate) {
        cudaError_t me = cudaMemsetAsync(d->dweight, 0, dw_bytes, st);
        if (me != cudaSuccess) return set_error(int(me), "wgrad: memset failed: %s", cudaGetErrorString(me));
    }
    const uint32_t smem = p.stages * p.stage_bytes + 2 * kWgStagesMax * 8 + 1024;
    const cudaError_t attr_err = ensure_dyn_smem(reinterpret_cast<const void*>(conv_wgrad_kernel), 227 * 1024);
    if (attr_err != cudaSuccess) return set_error(int(attr_err), "wgrad: cudaFuncSetAttribute failed");
    const long long grid = items * p.splits;
    return launch("wgrad", conv_wgrad_kernel, {static_cast<unsigned>(grid), kWgThreads, smem, st, /*pdl=*/true}, tmDy, tmX, p);
}
