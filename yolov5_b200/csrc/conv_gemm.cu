// Implicit-GEMM convolution for sm_90a:  D[M = B*Ho*Wo, N = Cout] = im2col(X)[M, K = kh*kw*Cin] * W[N, K]^T
//
// Activation (A) fetch, three modes -- all by the TMA unit, all landing in 32/64/128-byte-swizzled K-major smem tiles
// that wgmma reads through shared-memory descriptors:
//   LINEAR  1x1/s1 convs: 2-D tiles [128 pixels x BLOCK_K channels] of the [M, Cin] matrix.
//   IM2COL  hardware im2col mode (cp.async.bulk.tensor.4d...im2col): a tile is 128 consecutive output pixels in
//           (n,y,x) order whatever the row/image boundaries; padding zero-filled; stride via elementStrides.  One
//           copy per filter tap: the input is re-read kh*kw times (from L2).  Used for stride-2 and small maps.
//   PATCH   stride-1 convs: the tile is a th x tw block of output pixels (th*tw = 128) and, per channel chunk and
//           horizontal tap s, ONE copy brings the (th+kh-1) x tw input patch; the kh vertical taps are the same smem
//           patch read at row offsets r*tw (a plain descriptor offset, still aligned to the 8-row swizzle pattern
//           because tw % 8 == 0).  L2->smem traffic for A drops from kh*kw to kw*(th+kh-1)/th reads per input element.
//   PATCH, wide (64-channel chunks = 128-byte rows, kw > 1): tile = 16 rows x 8 pixels, ONE copy per channel chunk brings the
//           (16+kh-1) x PW patch (PW = 8*MT + 8 pixels: the MT sub-tiles sit side by side in it) and ALL kh*kw taps are read
//           from it: tap (r, s) = descriptor start + (r*PW + s) rows, the 8 pixels of an output row are one 8-row swizzle group,
//           consecutive output rows are PW*128 bytes apart (the descriptor's group stride).
// Weights (B): 2-D TMA tiles of the packed [Cout][kh][kw][Cin_pad] matrix, one per (tap, channel chunk); A and B
// have separate mbarrier rings because one A patch feeds kh B tiles (PATCH mode: the kh tiles of a group may share one stage).
// MMA + epilogue: two consumer warpgroups.  Warpgroup w owns rows [64w, 64w + 64) of every 128-row sub-tile and issues
// wgmma m64 x BLOCK_N x k16 (fp32 accumulators in registers) for them; after the tile's last K block it applies the
// folded-BN bias -> SiLU or LeakyReLU -> (+ residual) -> fp16/bf16 and stores straight from the registers to the NHWC (slice) view.
// Epilogue stores: by default the tile is staged in shared memory in swizzled 64-row boxes, with its residual TMA-loaded there by
// the producer warp, and leaves by TMA bulk stores (the TMA unit clips the tails).  Direct mode (reserved bit 16, and plans where
// the staging block does not fit or costs too much): each thread stores its 4-byte pairs straight from the registers, with the
// residual words loaded in batches ahead of the stores (the residual may alias the output, so interleaving would serialise); the
// OPT instantiation can instead stage each warpgroup's block and write whole 16-byte row segments.
// Tiles: MT sub-tiles of 128 rows x BLOCK_N with MT * BLOCK_N <= 256 (128 accumulator registers per thread), so one weight
// tile feeds MT sub-tiles and narrow layers do as much work per barrier round as wide ones.
// Clusters (2 or 4 CTAs along M): the CTAs of a cluster work on different M super-tiles of the SAME N tile in lock-step, each
// fetches 1/csize of every weight tile and TMA-multicasts it to all of them, so the L2 -> smem weight traffic per CTA drops by
// the cluster size.  A weight stage is free again only when the consumers of every CTA of the cluster have released it.
// EPI=2 is the conv epilogue with LeakyReLU (ReLU: slope 0) in place of SiLU: an instantiation of its own, so the SiLU / linear
// instantiations (EPI=0) compile to exactly the code they had without it.
// Detect head (EPI=1): an anchor's `no` outputs are tpa = ceil(no / 128) N tiles (weights packed npad = 128 * tpa rows per anchor).
// no <= 128 (one tile per anchor): raw logits and decoded predictions are staged in smem in the exact global layout and copied out
// with 16-byte vectors.  Wider heads stage [128 rows][128 columns] blocks and copy each row segment to its column offset, with 16-,
// 4- or 2-byte stores as `no` and the output alignment allow, and read their bias per tile instead of preloading it.
// Mainloop: one K block of a tile is one wgmma batch (block_k / 16 k16 steps x MT sub-tiles, issued back to back; the dtype is a
// template parameter, the step count a per-block switch into unrolled batches).  One batch stays in flight: after issuing batch i a
// consumer waits (wgmma.wait_group 1) only for batch i-1 and then releases the stages i-1 was the last reader of, so the tensor
// pipe is not drained between K blocks.  At the end of a tile it drains (wait_group 0) and releases what is still pending before
// the epilogue, so the producer fills the next tile's stages while the epilogue runs.
// Limits: both warpgroups run the epilogue of the same tile, so the tensor cores idle during each epilogue; overlapping them (two
// accumulator sets or ping-pong warpgroups) is the next step for this kernel.
// Persistent grid (<= one CTA per SM), warp-specialised: warp 0 TMA producer (its warpgroup hands its registers to the
// consumers through setmaxnreg), warpgroups 1 and 2 MMA + epilogue.
//
// Replaces reference models/common.py:86-92 (Conv), :181 (Bottleneck add), :246/:340/:453 (cat, via strided
// output views) and models/yolo.py:95-113 (Detect level).
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <mutex>
#include <type_traits>

#include "../../include/y5b200.h"
#include "common.cuh"
#include "host_util.h"
#include "wgmma.cuh"

namespace y5 {

constexpr int kBlockM = 128;
constexpr int kConsumers = 2;                          // MMA + epilogue warpgroups (64 rows of each sub-tile each)
constexpr int kConsumerThreads = 128 * kConsumers;
constexpr int kThreads = 128 + kConsumerThreads;       // warpgroup 0: TMA producer (warp 0 only)
constexpr int kMaxStages = 8;
constexpr int kHeadN = 128;                 // head GEMM: N tile width; an anchor takes ceil(no / 128) of them
constexpr int kHeadMaxNo = 8192;            // head outputs per anchor (5 + nc + nm), with nc <= kHeadMaxNc
constexpr int kHeadMaxNc = 4096;            // classes: the NMS / AP class limit

// head staging: [128 rows][cols] per block, cols = no for one N tile per anchor (the global layout), else one 128-column tile
__host__ __device__ inline int head_stage_cols(int no) { return no < kHeadN ? no : kHeadN; }

enum AMode { A_LINEAR = 0, A_IM2COL = 1, A_PATCH = 2 };

struct ConvParams {
    int M, N;                   // GEMM rows (B*Ho*Wo), output channels
    int num_m_tiles;            // 128-row sub-tiles
    int num_m_super, num_n_tiles;
    int kh, kw, c_chunks;       // K loop = kh*kw*c_chunks blocks of block_k
    int block_k;                // 16 | 32 | 64 elements (row bytes 32/64/128)
    int a_mode;
    int Ho, Wo, HoWo, stride, pad_h, pad_w;
    int tw, th, tiles_x, tiles_y;  // PATCH: spatial sub-tile th x tw (= 128 pixels), sub-tiles per image
    int b_grouped;              // PATCH: a weight stage holds all kh tiles of one (chunk, horizontal tap) group: one barrier round per group
    int patch_pw;               // > 0: wide patch mode, patch row pitch in pixels (8*MT + 8); one A copy per channel chunk feeds kh*kw taps
    int cluster_n;              // CTAs per cluster (1, 2, 4): weight tiles are split between them and multicast
    uint32_t stg_bytes;         // EPI 0: shared-memory staging of the epilogue (0 = direct stores)
    int tma_epi;                // EPI 0, default instantiation: the tile is staged in smem (residual TMA-loaded into it) and TMA-stored
    uint32_t b_sub_bytes;       // bytes of one weight tile inside a (possibly grouped) stage
    float rcp_per_img, rcp_tiles_x, rcp_HoWo, rcp_Wo;  // reciprocals for fdiv(): exact small-integer division in ~7 instructions
    int a_stages, b_stages;
    uint32_t a_sub_bytes, a_stage_bytes, b_stage_bytes;
    int is_bf16, act;           // act: SiLU (EPI 0)
    const float* bias;
    int bias_n;                 // floats preloaded into smem (0: a wide head reads each tile's bias from global memory)
    // EPI 0
    void* out;
    int out_pitch;
    const void* res;
    int res_pitch;
    // EPI 1 (detect head)
    void* raw;
    void* z;
    int na, no, nc, nx, z_rows, z_row0;
    float det_stride;
    float anchor_wh[8];
    // EPI 2 (conv with LeakyReLU / ReLU): v > 0 ? v : slope * v on v = fp32(acc + bias).  Last, so the other instantiations read
    // their parameters at the offsets they always had
    float slope;
};

struct SmemLayout {
    uint32_t off_a, off_b, off_out, off_bias, off_bars, total;
};

__host__ __device__ inline SmemLayout smem_layout(int epi, int no, int bias_n, int a_stages, int b_stages, uint32_t a_bytes,
                                                   uint32_t b_bytes, uint32_t stg_bytes) {
    SmemLayout L;
    uint32_t o = 0;
    L.off_a = o;
    o += a_stages * a_bytes;
    L.off_b = o;
    o += b_stages * b_bytes;
    o = (o + 1023) & ~1023u;
    L.off_out = o;
    if (epi == 1) o += 4 * ((kBlockM * head_stage_cols(no) * 2 + 1023) & ~1023u);  // head: 2 sets x {raw, decoded} blocks
    else o += stg_bytes;                                            // EPI 0 staging: per warpgroup [64 rows][BLOCK_N] (staged) or the tile (TMA)
    L.off_bias = o;
    o += ((bias_n + 3) & ~3) * 4;
    o = (o + 7) & ~7u;
    L.off_bars = o;
    o += (4 * kMaxStages + 2) * 8;  // A / B rings, then the TMA epilogue's res_full / stg_free pair
    L.total = o;
    return L;
}

// floor(n / d) for 0 <= n < 2^23, d >= 1, with rd = 1.0f / d: the float estimate is off by at most one, corrected exactly.
// (ptxas expands a 32-bit integer division into ~30 instructions; the tile decodes below run per tile in every role.)
__device__ __forceinline__ int fdiv(int n, int d, float rd) {
    if (n >= (1 << 23)) return n / d;  // beyond float's exact-integer range: the slow path (warp-uniform, rare)
    int q = __float2int_rz(__int2float_rz(n) * rd);
    const int r = n - q * d;
    if (r >= d) ++q;
    else if (r < 0) --q;
    return q;
}

// TMA epilogue: a warpgroup's 64 rows of a sub-tile are kNB boxes of [64 rows][kCols columns] with kRB-byte rows and the TMA
// swizzle of that row size (64 or 128 bytes), placed [warpgroup][sub-tile][box] in the staging block.
template <int BLOCK_N>
struct EpiBox {
    static constexpr int kRB = BLOCK_N * 2 < 128 ? BLOCK_N * 2 : 128;
    static constexpr int kCols = kRB / 2;
    static constexpr int kNB = BLOCK_N / kCols;
    static constexpr uint32_t kBytes = 64u * kRB;
};
struct EpiOrigin {
    int x, y, img;  // 2-D map: y = first row; PATCH (4-D map): first pixel x, y of image img
};
// where warpgroup wg's 64 rows of sub-tile mt start in the output / residual map; a PATCH box is [min(tw, 64)] x [max(64 / tw, 1)]
// pixels.  Rows past M, pixels past Wo / Ho and sub-tiles past the last one land out of bounds: the TMA unit clips the stores and
// zero-fills the loads.
__device__ __forceinline__ EpiOrigin epi_origin(const ConvParams& p, int mt, int wg) {
    if (p.a_mode != A_PATCH) return {0, mt * kBlockM + 64 * wg, 0};
    const int per_img = p.tiles_x * p.tiles_y;
    const int img = fdiv(mt, per_img, p.rcp_per_img);
    const int rem = mt - img * per_img;
    const int ty = fdiv(rem, p.tiles_x, p.rcp_tiles_x);
    const int x = (rem - ty * p.tiles_x) * p.tw, y = ty * p.th;
    return p.tw > 64 ? EpiOrigin{x + 64 * wg, y, img} : EpiOrigin{x, y + wg * (64 / p.tw), img};
}

// One K block (KS k16 steps) for all MT sub-tiles as one wgmma batch: fence, KS * MT back-to-back wgmmas, commit.  Nothing
// between the wgmmas touches their registers, so ptxas issues them as one chain (only the last waits on the scoreboard).
// scale_first == 0 overwrites the accumulators with the first k16 step (the tile's first K block).
template <int BLOCK_N, int MT, int KS, bool BF16>
__device__ __forceinline__ void mma_batch(float (&acc)[MT][BLOCK_N / 2], uint32_t a_lo, uint32_t a_sub16, uint32_t a_hi, uint32_t b_lo,
                                          uint32_t b_hi, uint32_t scale_first) {
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < KS; ++k)
#pragma unroll
        for (int mi = 0; mi < MT; ++mi)
            Wgmma<BLOCK_N>::template run<BF16, 0, 0>(acc[mi], gmma_desc(a_lo + mi * a_sub16 + 2 * k, a_hi), gmma_desc(b_lo + 2 * k, b_hi),
                                                     k == 0 ? scale_first : 1u);
    wgmma_commit();
}

// OPT: the instantiation that supports the optional modes (clusters, wide patch, staged stores); the default one compiles them out,
// which keeps their run-time tests and live registers out of the hot loops (measured 8 % on yolov5l's conv stack).
// BF16: activation / weight dtype (bf16 or fp16), fixed per instantiation so the MMA batches and the epilogue carry no dtype branch.
template <int BLOCK_N, int EPI, int MT, bool OPT, bool BF16>
__global__ void __launch_bounds__(kThreads, 1)
conv_gemm_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const __grid_constant__ CUtensorMap tmO,
                 const __grid_constant__ CUtensorMap tmR, const ConvParams p) {
    static_assert(MT * BLOCK_N <= 256, "accumulators: at most 128 fp32 registers per consumer thread");
    constexpr bool kConv = EPI != 1;   // EPI 0 and 2: the conv epilogue
    constexpr bool kLeaky = EPI == 2;  // ... with LeakyReLU instead of SiLU / none
    constexpr int kAcc = BLOCK_N / 2;  // accumulator registers per sub-tile and thread (64 x BLOCK_N over a warpgroup)
    using Box = EpiBox<BLOCK_N>;
    const bool tma_epi = kConv && !OPT && p.tma_epi;

    extern __shared__ __align__(1024) uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    const SmemLayout L = smem_layout(EPI, p.no, p.bias_n, p.a_stages, p.b_stages, p.a_stage_bytes, p.b_stage_bytes, p.stg_bytes);
    uint8_t* sA = smem + L.off_a;
    uint8_t* sB = smem + L.off_b;
    float* sBias = reinterpret_cast<float*>(smem + L.off_bias);
    uint64_t* a_full = reinterpret_cast<uint64_t*>(smem + L.off_bars);
    uint64_t* a_empty = a_full + kMaxStages;
    uint64_t* b_full = a_empty + kMaxStages;
    uint64_t* b_empty = b_full + kMaxStages;
    // TMA epilogue: the producer fills the staging block with a tile's residual (or just arrives, without one) on res_full once the
    // previous tile's bulk stores have finished reading it (stg_free, one arrival per consumer warpgroup)
    uint64_t* res_full = b_empty + kMaxStages;
    uint64_t* stg_free = res_full + 1;
    uint8_t* stg = smem + L.off_out;

    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;
    const int csize = OPT ? static_cast<int>(cluster_nctarank()) : 1;
    const uint32_t crank = OPT ? cluster_ctarank() : 0u;

    if (threadIdx.x == 0) {
        tma_prefetch_desc(&tmA);
        tma_prefetch_desc(&tmB);
        for (int s = 0; s < kMaxStages; ++s) {
            mbar_init(&a_full[s], 1);
            mbar_init(&a_empty[s], kConsumers);  // one arrival per consumer warpgroup
            mbar_init(&b_full[s], 1);
            mbar_init(&b_empty[s], kConsumers * csize);  // multicast stages: released by the consumers of every CTA of the cluster
        }
        mbar_init(res_full, 1);
        mbar_init(stg_free, kConsumers);
        if (tma_epi) {
            tma_prefetch_desc(&tmO);
            if (p.res) tma_prefetch_desc(&tmR);
        }
        fence_barrier_init();
    }
    if (threadIdx.x >= 128)  // whole folded-BN bias vector once: no per-tile global loads in the epilogue
        for (int i = threadIdx.x - 128; i < p.bias_n; i += kConsumerThreads) {
            // SiLU layers keep HALF the bias: the epilogue forms h = (acc + b) / 2 with one FMA and silu = h + h * tanh(h)
            const float b = i < p.N ? __ldg(p.bias + i) : 0.0f;
            sBias[i] = (kConv && p.act) ? 0.5f * b : b;
        }
    __syncthreads();
    if (csize > 1) cluster_sync_all();  // peers' barriers are initialised before anyone multicasts into them or arrives on them
    // PDL: everything above (barrier init, descriptor prefetch, bias preload) may overlap the tail of the previous kernel in
    // the stream; activations are only touched after this point.
    griddep_wait();
    griddep_launch_dependents();

    // tile = (group of csize M super-tiles, N tile), N fastest: CTAs running at the same time share the activation rows through L2;
    // this CTA takes super-tile group * csize + crank
    const int nn = p.num_n_tiles;
    const int num_tiles = ((p.num_m_super + csize - 1) / csize) * nn;
    const int tile0 = blockIdx.x / csize, tile_step = gridDim.x / csize;
    const uint32_t row_bytes = p.block_k * 2;
    const bool patch = p.a_mode == A_PATCH;
    // K iteration: "A groups" each feeding `grp` consecutive B tiles.
    //   PATCH : groups = (chunk cc, horizontal tap s), members r = 0..kh-1   -> k-block (r*kw + s)*c_chunks + cc
    //   else  : groups = k-blocks in (r, s, cc) order, one member each
    //   PATCH wide: groups = channel chunks cc, members (r, s) in weight order   -> k-block (r*kw + s)*c_chunks + cc
    const bool wide = OPT && p.patch_pw > 0;
    const int grp = wide ? p.kh * p.kw : (patch ? p.kh : 1);
    const int num_groups = wide ? p.c_chunks : (patch ? p.c_chunks * p.kw : p.kh * p.kw * p.c_chunks);

    if (warp < 4) {
        setmaxnreg_dec<56>();  // 56 / 224: no spills in any instantiation (40 / 232 spilled the producer's tile decode)
    }
    if (warp == 0) {
        // ===================================== TMA producer =====================================
        // the whole warp runs the loop with warp-uniform state; one elected lane issues the copies
        int as = 0, bs = 0;
        uint32_t aph = 0, bph = 0, sph = 0;
        for (int tile = tile0; tile < num_tiles; tile += tile_step) {
            const int ms = (tile / nn) * csize + static_cast<int>(crank);
            const int n0 = (tile - (tile / nn) * nn) * BLOCK_N;
            int img[MT], y0[MT], x0[MT];  // IM2COL: base pixel of the first window; PATCH: sub-tile origin
#pragma unroll
            for (int mi = 0; mi < MT; ++mi) {
                const int mt = ms * MT + mi;
                img[mi] = y0[mi] = x0[mi] = 0;
                if (p.a_mode == A_IM2COL) {
                    const int m0 = mt * kBlockM;
                    img[mi] = fdiv(m0, p.HoWo, p.rcp_HoWo);
                    const int rem = m0 - img[mi] * p.HoWo;
                    const int oy = fdiv(rem, p.Wo, p.rcp_Wo);
                    y0[mi] = oy * p.stride - p.pad_h;
                    x0[mi] = (rem - oy * p.Wo) * p.stride - p.pad_w;
                } else if (patch) {
                    const int per_img = p.tiles_x * p.tiles_y;
                    img[mi] = fdiv(mt, per_img, p.rcp_per_img);
                    const int rem = mt - img[mi] * per_img;
                    const int ty = fdiv(rem, p.tiles_x, p.rcp_tiles_x);
                    y0[mi] = ty * p.th - p.pad_h;
                    x0[mi] = (rem - ty * p.tiles_x) * p.tw - p.pad_w;
                }
            }
            // one A group + its B tiles; PATCH walks (cc, s){r}, the other modes walk (r, s, cc)
            auto issue_group = [&](int cc, int s, int r0) {
                mbar_wait(&a_empty[as], aph ^ 1);
                if (elect_one()) {
                    mbar_arrive_expect_tx(&a_full[as], p.a_stage_bytes);
#pragma unroll
                    for (int mi = 0; mi < MT; ++mi) {
                        uint8_t* a_dst = sA + as * p.a_stage_bytes + mi * p.a_sub_bytes;
                        if (wide) {  // one patch for all sub-tiles and taps (sub-tile mi starts 8 pixels = 1024 bytes into it)
                            if (mi == 0) tma_load_4d(&tmA, &a_full[as], a_dst, cc * p.block_k, x0[0], y0[0], img[0]);
                        } else if (p.a_mode == A_LINEAR) tma_load_2d(&tmA, &a_full[as], a_dst, cc * p.block_k, (ms * MT + mi) * kBlockM);
                        else if (p.a_mode == A_IM2COL)
                            tma_load_im2col_4d(&tmA, &a_full[as], a_dst, cc * p.block_k, x0[mi], y0[mi], img[mi], static_cast<uint16_t>(s),
                                               static_cast<uint16_t>(r0));
                        else tma_load_4d(&tmA, &a_full[as], a_dst, cc * p.block_k, x0[mi] + s, y0[mi], img[mi]);
                    }
                }
                __syncwarp();
                if (++as == p.a_stages) { as = 0; aph ^= 1; }
                for (int j = 0; j < grp; ++j) {
                    const int r = patch ? j : r0;
                    const int kb = wide ? j * p.c_chunks + cc : (r * p.kw + s) * p.c_chunks + cc;
                    // grouped stages: the kh tiles of this group share one stage (one wait, one expect_tx covering all of them)
                    const bool stage_first = !p.b_grouped || j == 0, stage_last = !p.b_grouped || j == grp - 1;
                    if (stage_first) mbar_wait(&b_empty[bs], bph ^ 1);
                    if (elect_one()) {
                        if (stage_first) mbar_arrive_expect_tx(&b_full[bs], p.b_stage_bytes);
                        uint8_t* b_dst = sB + bs * p.b_stage_bytes + (p.b_grouped ? j * p.b_sub_bytes : 0u);
                        if (csize == 1) tma_load_2d(&tmB, &b_full[bs], b_dst, kb * p.block_k, n0);
                        else {  // my slice of the rows, delivered to every CTA of the cluster
                            const int slice_rows = BLOCK_N / csize;
                            tma_load_2d_mcast(&tmB, &b_full[bs], b_dst + crank * slice_rows * row_bytes, kb * p.block_k,
                                              n0 + static_cast<int>(crank) * slice_rows, static_cast<uint16_t>((1u << csize) - 1u));
                        }
                    }
                    __syncwarp();
                    if (stage_last && ++bs == p.b_stages) { bs = 0; bph ^= 1; }
                }
            };
            if (wide) {
                for (int cc = 0; cc < p.c_chunks; ++cc) issue_group(cc, 0, 0);
            } else if (patch) {
                for (int cc = 0; cc < p.c_chunks; ++cc)
                    for (int s = 0; s < p.kw; ++s) issue_group(cc, s, 0);
            } else {
                for (int r = 0; r < p.kh; ++r)
                    for (int s = 0; s < p.kw; ++s)
                        for (int cc = 0; cc < p.c_chunks; ++cc) issue_group(cc, s, r);
            }
            // the tile's residual, after its last K block: by then the consumers have started this tile (its first batch frees the
            // staging block of the previous one), so the wait rarely blocks and the copy lands while the tile's MMAs run
            if (tma_epi) {
                mbar_wait(stg_free, sph ^ 1);
                if (elect_one()) {
                    if (p.res) {
                        mbar_arrive_expect_tx(res_full, p.stg_bytes);
#pragma unroll 1
                        for (int i = 0; i < kConsumers * MT; ++i) {
                            const EpiOrigin o = epi_origin(p, ms * MT + i % MT, i / MT);
#pragma unroll
                            for (int b = 0; b < Box::kNB; ++b) {
                                uint8_t* dst = stg + (i * Box::kNB + b) * Box::kBytes;
                                if (patch) tma_load_4d(&tmR, res_full, dst, n0 + b * Box::kCols, o.x, o.y, o.img);
                                else tma_load_2d(&tmR, res_full, dst, n0 + b * Box::kCols, o.y);
                            }
                        }
                    } else {
                        mbar_arrive(res_full);
                    }
                }
                __syncwarp();
                sph ^= 1;
            }
        }
    } else if (warp >= 4) {
    // ===================================== MMA + epilogue (warpgroups 1, 2) =====================================
    setmaxnreg_inc<224>();
    const int wg = (warp >> 2) - 1;                       // rows [64 wg, 64 wg + 64) of every sub-tile
    const int ct = threadIdx.x - 128;                     // 0 .. kConsumerThreads-1
    const int wrow = wg * 64 + (warp & 3) * 16 + (lane >> 2);  // this thread's first accumulator row (the second is +8)
    const int ccol = 2 * (lane & 3);                      // this thread's first column inside every 8-column group
    const bool signal = (threadIdx.x & 127) == 0;         // the warpgroup's thread that releases smem stages
    constexpr bool bf16 = BF16;
    const uint32_t dhi = gmma_desc_hi(row_bytes);
    // wide patch: group stride = one patch row (PW pixels); warpgroup wg starts 8 output rows = 8 patch rows down
    const uint32_t a_hi = wide ? (dhi & ~0x3FFFu) | (((static_cast<uint32_t>(p.patch_pw) * row_bytes) >> 4) & 0x3FFFu) : dhi;
    const uint32_t a_base = gmma_desc_lo(smem_u32(sA) + (wide ? wg * 8 * p.patch_pw : wg * 64) * row_bytes), b_base = gmma_desc_lo(smem_u32(sB));
    const uint32_t row16 = row_bytes >> 4;
    const uint32_t a_stage16 = p.a_stage_bytes >> 4, b_stage16 = p.b_stage_bytes >> 4, a_sub16 = p.a_sub_bytes >> 4;
    const uint32_t b_sub16 = p.b_sub_bytes >> 4;
    const uint32_t a_shift16 = patch ? (p.tw * row_bytes) >> 4 : 0;  // between vertical taps inside a patch
    const int k_steps = p.block_k / 16;
    const int per_img = p.tiles_x * p.tiles_y;
    const int tw_shift = patch ? __ffs(p.tw) - 1 : 0;
    int as = 0, bs = 0, head_set = 0;
    uint32_t aph = 0, bph = 0, rph = 0;
    float acc[MT][kAcc];
#pragma unroll
    for (int mi = 0; mi < MT; ++mi)
#pragma unroll
        for (int i = 0; i < kAcc; ++i) acc[mi][i] = 0.0f;

    // Stage release, deferred by one batch: the stages a batch reads are handed back to the producer only once the NEXT batch has
    // been issued and wgmma.wait_group 1 has confirmed this one complete, so the tensor pipe never drains between K blocks.  The
    // record of the batch in flight: its A stage and whether it is that stage's last reader, its B stage and whether it is that
    // stage's last reader (a grouped B stage feeds kh members, a wide-patch A stage kh*kw).
    int pend_as = 0, pend_bs = 0;
    bool pend_a_last = false, pend_b_last = false;
    auto release_pending = [&]() {
        if (!signal) return;
        if (pend_b_last) {
            if (csize == 1) mbar_arrive(&b_empty[pend_bs]);
            else  // multicast stage: every CTA of the cluster waits for the consumers of all of them
                for (int r = 0; r < csize; ++r) mbar_arrive_cluster(mapa_u32(&b_empty[pend_bs], static_cast<uint32_t>(r)));
        }
        if (pend_a_last) mbar_arrive(&a_empty[pend_as]);
    };

    for (int tile = tile0; tile < num_tiles; tile += tile_step) {
        const int ms = (tile / nn) * csize + static_cast<int>(crank);
        const int nt = tile - (tile / nn) * nn;
        const int n0 = nt * BLOCK_N;
        for (int g = 0; g < num_groups; ++g) {
            mbar_wait(&a_full[as], aph);
            const uint32_t a_stage_lo = a_base + as * a_stage16;
            uint32_t a_lo = a_stage_lo;
            for (int j = 0; j < grp; ++j) {
                if (wide) {  // tap (r, s) of the shared patch
                    const int tr = j / p.kw, ts = j - tr * p.kw;
                    a_lo = a_stage_lo + (tr * p.patch_pw + ts) * row16;
                }
                const bool stage_first = !p.b_grouped || j == 0, stage_last = !p.b_grouped || j == grp - 1;
                if (stage_first) mbar_wait(&b_full[bs], bph);
                const uint32_t b_lo = b_base + bs * b_stage16 + (p.b_grouped ? j * b_sub16 : 0u);
                const uint32_t scale_first = (g | j) != 0 ? 1u : 0u;  // the tile's first K step overwrites the accumulators
#pragma unroll
                for (int mi = 0; mi < MT; ++mi) fence_regs(acc[mi]);
                switch (k_steps) {  // block_k 64 / 32 / 16
                    case 4: mma_batch<BLOCK_N, MT, 4, BF16>(acc, a_lo, a_sub16, a_hi, b_lo, dhi, scale_first); break;
                    case 2: mma_batch<BLOCK_N, MT, 2, BF16>(acc, a_lo, a_sub16, a_hi, b_lo, dhi, scale_first); break;
                    default: mma_batch<BLOCK_N, MT, 1, BF16>(acc, a_lo, a_sub16, a_hi, b_lo, dhi, scale_first); break;
                }
                wgmma_wait<1>();  // the previous batch (not this one) is complete: its stages can go back to the producer
#pragma unroll
                for (int mi = 0; mi < MT; ++mi) fence_regs(acc[mi]);
                if (g | j) release_pending();  // the tile's first batch: everything before it was released at the previous tile's end
                else if (tma_epi && signal && tile != tile0) {
                    // the previous tile's bulk stores have read the staging block (waited for under this batch): the producer may
                    // load this tile's residual into it
                    tma_store_wait_read0();
                    mbar_arrive(stg_free);
                }
                pend_as = as;
                pend_a_last = j == grp - 1;
                pend_bs = bs;
                pend_b_last = stage_last;
                if (stage_last && ++bs == p.b_stages) { bs = 0; bph ^= 1; }
                a_lo += a_shift16;
            }
            if (++as == p.a_stages) { as = 0; aph ^= 1; }
        }
        // drain before the epilogue reads the accumulators; the last stages go back now, so the producer fills the next tile's
        // stages while this tile's epilogue runs
        wgmma_wait<0>();
#pragma unroll
        for (int mi = 0; mi < MT; ++mi) fence_regs(acc[mi]);
        release_pending();

        if (kConv) {
            const bool staged = OPT && p.stg_bytes != 0;
            const uint32_t stg_pitch = BLOCK_N * 2 + 16;  // +16 bytes: the fragment's 8 rows x 4 column pairs hit 32 distinct banks
            uint8_t* stg_wg = stg + wg * 64 * stg_pitch;
            // TMA epilogue: shared address of the word of column pair (8 j + ccol) of row half h of sub-tile mi in its swizzled box
            // (16-byte chunk index XOR the row's offset bits 7.., as the TMA unit lays it out; the fragment's 8 rows x 4 column pairs
            // hit 32 distinct banks).  The thread's row base and XOR term are laundered per tile, so the compiler does not hoist
            // every word address out of the tile loop and hold them next to the accumulators.
            constexpr int kChunks = Box::kRB / 16;
            uint32_t stg_row = smem_u32(stg) + wg * MT * Box::kNB * Box::kBytes + (wrow - wg * 64) * Box::kRB + ccol * 2;
            uint32_t stg_swz = ((((wrow - wg * 64) * Box::kRB) >> 7) & (kChunks - 1)) << 4;
            asm volatile("" : "+r"(stg_row), "+r"(stg_swz));
            auto stg_word = [&](int mi, int h, int j) -> uint32_t {
                return stg_row + (mi * Box::kNB + j / kChunks) * Box::kBytes + h * 8 * Box::kRB + (((j % kChunks) << 4) ^ stg_swz);
            };
            // global output pixel of row `row` of sub-tile `mt`, -1 outside the output
            auto pixel_of = [&](int mt, int row) -> long long {
                if (patch) {  // image + origin of the th x tw block
                    const int img = fdiv(mt, per_img, p.rcp_per_img);
                    const int rem = mt - img * per_img;
                    const int tyi = fdiv(rem, p.tiles_x, p.rcp_tiles_x);
                    const int oy = tyi * p.th + (row >> tw_shift), ox = (rem - tyi * p.tiles_x) * p.tw + (row & ((1 << tw_shift) - 1));
                    return (mt < p.num_m_tiles && oy < p.Ho && ox < p.Wo) ? static_cast<long long>(img) * p.HoWo + oy * p.Wo + ox : -1;
                }
                const long long m = static_cast<long long>(mt) * kBlockM + row;
                return m < p.M ? m : -1;
            };
            // The residual may alias the output (the in-place Bottleneck add), so a load placed after a store cannot be moved above
            // it: read and written group by group, every 8-column group would cost one dependent global round trip.  Instead the
            // thread's rows (MT sub-tiles x 2 row halves) go in batches of kBatch, and every residual word of a batch is loaded before
            // its first store: one round trip per batch, and at most 2 per tile.  Legal in place because each thread reads only the
            // elements it writes itself.  kBatch keeps the loaded words to 32 registers (64 spill next to 128 accumulators), 16 in
            // the OPT instantiations, whose optional modes hold more live state.
            constexpr float kTail = BF16 ? 8.0f : 4.0f;  // silu_from_half is faithful down to -kTail (see common.cuh)
            constexpr int kRows = 2 * MT, kWords = (OPT ? 128 : 256) / BLOCK_N;
            constexpr int kBatch = kWords < 1 ? 1 : (kWords < kRows ? kWords : kRows);
            // TMA epilogue: the residual words (zero outside the output) are in the staging block and the tile is written there; no
            // global access and no bounds test per element, the TMA unit clips the stores
            const bool has_res = p.res != nullptr;
            if (tma_epi) {
                mbar_wait(res_full, rph);
                rph ^= 1;
            }
            // the two store paths as separate straight-line code: run-time tests of the path inside the unrolled loops made ptxas spill
            auto rows = [&](auto tma_path) {
                constexpr bool TMA = decltype(tma_path)::value;
#pragma unroll
                for (int q0 = 0; q0 < kRows; q0 += kBatch) {
                    uint32_t rv[kBatch][BLOCK_N / 8];
                    long long gp[kBatch];  // output pixel of each row half of the batch, -1 outside the output
#pragma unroll
                    for (int q = 0; q < kBatch; ++q) gp[q] = TMA ? 0 : pixel_of(ms * MT + (q0 + q) / 2, wrow + 8 * ((q0 + q) & 1));
                    if (has_res && TMA) {
#pragma unroll
                        for (int q = 0; q < kBatch; ++q)
#pragma unroll
                            for (int j = 0; j < BLOCK_N / 8; ++j) rv[q][j] = ld_shared_u32(stg_word((q0 + q) / 2, (q0 + q) & 1, j));
                    } else if (has_res) {
#pragma unroll
                        for (int q = 0; q < kBatch; ++q) {
                            const uint16_t* rp = reinterpret_cast<const uint16_t*>(p.res) + (gp[q] < 0 ? 0 : gp[q] * p.res_pitch) + n0 + ccol;
#pragma unroll
                            for (int j = 0; j < BLOCK_N / 8; ++j)
                                rv[q][j] = (gp[q] >= 0 && n0 + 8 * j < p.N) ? *reinterpret_cast<const uint32_t*>(rp + 8 * j) : 0u;
                        }
                    }
#pragma unroll
                    for (int q = 0; q < kBatch; ++q) {
                        const int mi = (q0 + q) / 2, h = (q0 + q) & 1;  // sub-tile, row half
                        const int mt = ms * MT + mi;
                        const int row = wrow + 8 * h;
                        const long long gpix = gp[q];
                        if (gpix >= 0 || staged) {
                            uint16_t* op = reinterpret_cast<uint16_t*>(p.out) + gpix * p.out_pitch + n0 + ccol;
                            uint8_t* sp = stg_wg + (row - wg * 64) * stg_pitch + ccol * 2;
                            float hmin = 0.0f;  // smallest SiLU input / 2 of the row half
                            // the row half's 8-column groups: bias -> SiLU -> + residual -> pack -> store.  TAIL: the pass that recomputes
                            // the SiLU inputs below -kTail with silu_tail (silu_from_half is not faithful there) and stores the row again
                            auto row_half = [&](auto tail_pass) {
                                constexpr bool TAIL = decltype(tail_pass)::value;
#pragma unroll
                                for (int j = 0; j < BLOCK_N / 8; ++j) {
                                    if (n0 + 8 * j >= p.N) continue;  // N % 8 == 0: an 8-column group is all in or all out
                                    const float2 b = *reinterpret_cast<const float2*>(sBias + n0 + 8 * j + ccol);
                                    const float a0 = acc[mi][4 * j + 2 * h], a1 = acc[mi][4 * j + 2 * h + 1];
                                    float f0, f1;
                                    if (p.act) {  // b holds bias / 2 (see the preload)
                                        const float h0 = fmaf(a0, 0.5f, b.x), h1 = fmaf(a1, 0.5f, b.y);  // exactly fp32(acc + bias) / 2
                                        f0 = silu_from_half(h0);
                                        f1 = silu_from_half(h1);
                                        if (TAIL) {
                                            if (h0 < -0.5f * kTail) f0 = silu_tail(2.0f * h0);
                                            if (h1 < -0.5f * kTail) f1 = silu_tail(2.0f * h1);
                                        } else {
                                            hmin = fminf(hmin, fminf(h0, h1));
                                        }
                                    } else {
                                        f0 = a0 + b.x;
                                        f1 = a1 + b.y;
                                        if (kLeaky) {
                                            f0 = f0 > 0.0f ? f0 : p.slope * f0;
                                            f1 = f1 > 0.0f ? f1 : p.slope * f1;
                                        }
                                    }
                                    if (has_res && gpix >= 0) {
                                        const float2 t = unpack2(rv[q][j], bf16);
                                        f0 += t.x;
                                        f1 += t.y;
                                    }
                                    if (TMA) st_shared_u32(stg_word(mi, h, j), pack2(f0, f1, bf16));
                                    else if (staged) *reinterpret_cast<uint32_t*>(sp + 16 * j) = pack2(f0, f1, bf16);
                                    else *reinterpret_cast<uint32_t*>(op + 8 * j) = pack2(f0, f1, bf16);
                                }
                            };
                            row_half(std::false_type{});
                            // inputs below -kTail are rare: one vote per row half, and only the warps holding some take the second pass
                            // (the residual comes from the registers, so an in-place residual stays right)
                            if (p.act && __any_sync(__activemask(), hmin < -0.5f * kTail)) row_half(std::true_type{});
                        }
                        if (staged && h == 1) {  // the sub-tile is complete: the warpgroup's 64 rows leave as whole 16-byte row segments
                            named_bar_sync(2 + wg, 128);
                            constexpr int kSeg = BLOCK_N / 8;
                            for (int i = threadIdx.x & 127; i < 64 * kSeg; i += 128) {
                                const int lrow = i / kSeg, c = i - lrow * kSeg;
                                const long long gp = pixel_of(mt, wg * 64 + lrow);
                                if (gp >= 0 && n0 + 8 * c < p.N)
                                    *reinterpret_cast<uint4*>(reinterpret_cast<uint16_t*>(p.out) + gp * p.out_pitch + n0 + 8 * c) =
                                        *reinterpret_cast<const uint4*>(stg_wg + lrow * stg_pitch + c * 16);
                            }
                            named_bar_sync(2 + wg, 128);  // the staging block is rewritten by the next sub-tile / tile
                        }
                    }
                }
            };
            if (tma_epi) rows(std::true_type{});
            else rows(std::false_type{});
            if (tma_epi) {
                // the warpgroup's rows are in the staging block: make them visible to the async proxy, then one thread stores them and
                // goes on to the next tile; it waits for the stores to have read the block under the next tile's first MMA batch
                fence_proxy_async_smem();
                named_bar_sync(2 + wg, 128);
                if (signal) {
#pragma unroll 1
                    for (int mi = 0; mi < MT; ++mi) {
                        const EpiOrigin o = epi_origin(p, ms * MT + mi, wg);
#pragma unroll
                        for (int b = 0; b < Box::kNB; ++b) {
                            const uint8_t* src = stg + ((wg * MT + mi) * Box::kNB + b) * Box::kBytes;
                            if (patch) tma_store_4d(&tmO, src, n0 + b * Box::kCols, o.x, o.y, o.img);
                            else tma_store_2d(&tmO, src, n0 + b * Box::kCols, o.y);
                        }
                    }
                    tma_store_commit();
                    // the next layer reads this output (under PDL, as soon as this grid completes): the CTA's last stores are complete
                    // before it exits.  (Placed here: the same wait after the tile loop made ptxas serialise the wgmmas and spill.)
                    if (tile + tile_step >= num_tiles) tma_store_wait_all();
                }
            }
        } else {
            // ---- Detect head (models/yolo.py:95-113): N tile `nt` is tile nt % tpa of anchor nt / tpa, its output columns
            // [c0, c0 + 128).  The accumulators give the raw logits AND the decoded predictions, written into two smem blocks, one
            // barrier of the consumer warpgroups, then the copy-out.  One tile per anchor (no <= 128): the blocks are laid out exactly
            // like their global destinations ([128 pixels][no] contiguous per anchor) and leave as 16-byte vectors.  Wider heads: the
            // blocks are [128 pixels][128 columns] and every row segment goes to column c0 of its pixel's row.  Two staging sets
            // alternate per tile, so the barrier of tile i+1 also fences the reuse of tile i-1's set.
            const int no = p.no;
            const int tpa = (no + kHeadN - 1) / kHeadN;
            const int scols = head_stage_cols(no);
            const uint32_t blk = (kBlockM * scols * 2 + 1023) & ~1023u;
            const int set = head_set;
            head_set ^= 1;
            uint16_t* stage_raw = reinterpret_cast<uint16_t*>(smem + L.off_out + (2 * set) * blk);
            uint16_t* stage_z = reinterpret_cast<uint16_t*>(smem + L.off_out + (2 * set + 1) * blk);
            const int a = tpa == 1 ? nt : nt / tpa;  // (no integer division on the one-tile path)
            const int c0 = (nt - a * tpa) * kHeadN;
            const int ncol = min(kHeadN, no - c0);  // columns of the anchor's outputs in this tile
            const float aw = p.anchor_wh[a * 2], ah = p.anchor_wh[a * 2 + 1];
            const int m0 = ms * kBlockM;
            const int rows_here = min(kBlockM, p.M - m0);
            // the two staging paths as separate straight-line code (a run-time test of the path inside the unrolled loop slowed the
            // one-tile head by 9 %, measured on yolov5l's nc = 80 levels).  WIDE: the tile's bias is read from global memory once
            // (bias_n == 0), columns are offset by c0 and only the anchor's first tile holds the box columns.
            auto stage = [&](auto wide_path) {
                constexpr bool WIDE = decltype(wide_path)::value;
                float bcol[BLOCK_N / 8][2];
                if (WIDE) {
#pragma unroll
                    for (int j = 0; j < BLOCK_N / 8; ++j)
#pragma unroll
                        for (int e = 0; e < 2; ++e) {
                            const int o = 8 * j + ccol + e;
                            bcol[j][e] = o < ncol ? __ldg(p.bias + n0 + o) : 0.0f;
                        }
                }
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const int row = wrow + 8 * h;
                    const int m = m0 + row;
                    int gx = 0, gy = 0;
                    if (m < p.M && (!WIDE || c0 == 0)) {
                        const int pix = m - fdiv(m, p.HoWo, p.rcp_HoWo) * p.HoWo;
                        gy = fdiv(pix, p.nx, p.rcp_Wo);
                        gx = pix - gy * p.nx;
                    }
                    const float fgx = static_cast<float>(gx) - 0.5f, fgy = static_cast<float>(gy) - 0.5f;
#pragma unroll
                    for (int j = 0; j < BLOCK_N / 8; ++j) {
#pragma unroll
                        for (int e = 0; e < 2; ++e) {
                            const int o = 8 * j + ccol + e;  // column in the tile
                            if (o >= (WIDE ? ncol : no)) continue;
                            const int oc = WIDE ? c0 + o : o;  // column of the anchor's outputs
                            const float x = acc[0][4 * j + 2 * h + e] + (WIDE ? bcol[j][e] : sBias[n0 + o]);
                            float d = x;
                            if (oc < 5 + p.nc) {
                                const float sg = sigmoid_f(x);
                                if (oc == 0) d = (sg * 2.0f + fgx) * p.det_stride;
                                else if (oc == 1) d = (sg * 2.0f + fgy) * p.det_stride;
                                else if (oc == 2) { const float u = sg * 2.0f; d = u * u * aw; }
                                else if (oc == 3) { const float u = sg * 2.0f; d = u * u * ah; }
                                else d = sg;
                            }
                            const int si = row * (WIDE ? kHeadN : no) + o;
                            stage_raw[si] = pack1(x, bf16);
                            stage_z[si] = pack1(d, bf16);
                        }
                    }
                }
            };
            if (tpa > 1) stage(std::true_type{});
            else stage(std::false_type{});
            named_bar_sync(1, kConsumerThreads);
            if (tpa > 1) {
                // wide head: row r of the block is ncol elements at column c0 of global row (b, a, pix) of raw and (b, z_row0 + a
                // HoWo + pix) of z.  16-byte vectors when no % 8 == 0 (c0 is a multiple of 128, so every segment is then aligned),
                // 4-byte words when no is even, else half-words.
#pragma unroll 1
                for (int which = 0; which < 2; ++which) {
                    uint16_t* base = reinterpret_cast<uint16_t*>(which == 0 ? p.raw : p.z);
                    const uint16_t* src = which == 0 ? stage_raw : stage_z;
                    auto copy = [&](auto vec) {
                        constexpr int V = decltype(vec)::value;  // elements per store
                        using T = std::conditional_t<V == 8, uint4, std::conditional_t<V == 2, uint32_t, uint16_t>>;
                        const int segs = ncol / V;
                        // one warp per row: the row's destination is computed once, the lanes store its segment
                        for (int r = ct >> 5; r < rows_here; r += kConsumerThreads / 32) {
                            const int m = m0 + r;
                            const int b = fdiv(m, p.HoWo, p.rcp_HoWo), pix = m - b * p.HoWo;
                            const long long grow = which == 0 ? (static_cast<long long>(b) * p.na + a) * p.HoWo + pix
                                                              : static_cast<long long>(b) * p.z_rows + p.z_row0 + static_cast<long long>(a) * p.HoWo + pix;
                            T* d = reinterpret_cast<T*>(base + grow * no + c0);
                            const T* s = reinterpret_cast<const T*>(src + r * kHeadN);
                            for (int c = lane; c < segs; c += 32) d[c] = s[c];
                        }
                    };
                    const uintptr_t ba = reinterpret_cast<uintptr_t>(base);
                    if ((no & 7) == 0 && (ba & 15) == 0) copy(std::integral_constant<int, 8>{});
                    else if ((no & 1) == 0 && (ba & 3) == 0) copy(std::integral_constant<int, 2>{});
                    else copy(std::integral_constant<int, 1>{});
                }
                continue;
            }
            // copy out: for each image the tile touches, rows [r_lo, r_hi) are one contiguous global block per output
            const int b_lo = fdiv(m0, p.HoWo, p.rcp_HoWo), b_hi = fdiv(m0 + rows_here - 1, p.HoWo, p.rcp_HoWo);
            for (int b = b_lo; b <= b_hi; ++b) {
                const int r_lo = max(b * p.HoWo - m0, 0), r_hi = min((b + 1) * p.HoWo - m0, rows_here);
                const int pix_lo = m0 + r_lo - b * p.HoWo;
                const int n_el = (r_hi - r_lo) * no;
#pragma unroll
                for (int which = 0; which < 2; ++which) {
                    const long long dst_el = which == 0
                        ? ((static_cast<long long>(b) * p.na + a) * p.HoWo + pix_lo) * no
                        : (static_cast<long long>(b) * p.z_rows + p.z_row0 + static_cast<long long>(a) * p.HoWo + pix_lo) * no;
                    uint16_t* dst = reinterpret_cast<uint16_t*>(which == 0 ? p.raw : p.z) + dst_el;
                    const uint16_t* src = (which == 0 ? stage_raw : stage_z) + r_lo * no;
                    if ((((reinterpret_cast<uintptr_t>(dst) | reinterpret_cast<uintptr_t>(src)) & 15) == 0) && (n_el & 7) == 0) {
                        const uint4* s4 = reinterpret_cast<const uint4*>(src);
                        uint4* d4 = reinterpret_cast<uint4*>(dst);
                        for (int i = ct; i < n_el / 8; i += kConsumerThreads) d4[i] = s4[i];
                    } else {
                        for (int i = ct; i < n_el; i += kConsumerThreads) dst[i] = src[i];
                    }
                }
            }
        }
    }
    }
    if (csize > 1) cluster_sync_all();  // no CTA leaves while a peer may still multicast into it or arrive on its barriers
}

// ---------------------------------------------------------------------------------------------------------------------
// Independent CUDA-core direct convolution (cross-check on device; also documents the packed weight layout).
// ---------------------------------------------------------------------------------------------------------------------
__global__ void conv_direct_kernel(const uint16_t* __restrict__ in, long long xs, long long ys, long long ns, int B, int H,
                                   int W, int Cin, const uint16_t* __restrict__ w, int cin_pad, const float* __restrict__ bias,
                                   uint16_t* out, int out_pitch, int Cout, const uint16_t* res, int res_pitch, int kh, int kw,
                                   int stride, int pad_h, int pad_w, int Ho, int Wo, int act, float slope, int bf16) {
    const long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
    const long long total = static_cast<long long>(B) * Ho * Wo * Cout;
    if (idx >= total) return;
    const int n = static_cast<int>(idx % Cout);
    const long long m = idx / Cout;
    const int ox = static_cast<int>(m % Wo);
    const int oy = static_cast<int>((m / Wo) % Ho);
    const int b = static_cast<int>(m / (static_cast<long long>(Wo) * Ho));
    float acc = 0.0f;
    for (int r = 0; r < kh; ++r) {
        const int iy = oy * stride - pad_h + r;
        if (iy < 0 || iy >= H) continue;
        for (int s = 0; s < kw; ++s) {
            const int ix = ox * stride - pad_w + s;
            if (ix < 0 || ix >= W) continue;
            const uint16_t* ip = in + b * ns + iy * ys + ix * xs;
            const uint16_t* wp = w + (static_cast<long long>(n) * kh * kw + r * kw + s) * cin_pad;
            for (int c = 0; c < Cin; ++c) acc += unpack1(ip[c], bf16) * unpack1(wp[c], bf16);
        }
    }
    float x = acc + bias[n];
    if (act == Y5_ACT_SILU) x = x / (1.0f + expf(-x));
    else if (act == Y5_ACT_LEAKY) x = x > 0.0f ? x : slope * x;
    if (res) x += unpack1(res[m * res_pitch + n], bf16);
    out[m * out_pitch + n] = pack1(x, bf16);
}

}  // namespace y5

// =====================================================================================================================
// host side
// =====================================================================================================================
using namespace y5;

namespace {

int pick_block_k(int in_c) {
    // 64-channel chunks (128-byte rows, 4 K steps per barrier round) for everything wider than 16 channels: the zero padding of
    // K (the copy engine zero-fills the channels beyond in_c, the packed weights carry zeros there) costs less than the extra
    // barrier rounds of narrower chunks.  Only very narrow inputs (the 16-channel stem) keep 16-channel chunks.
    return in_c > 16 ? 64 : 16;
}

// Tile shape (block_n, sub-tiles per tile), MT * block_n <= 256 (the accumulators live in the consumer warpgroups' registers).
// Narrow layers fill the 256 columns with 128-row sub-tiles that share each weight tile (one barrier round feeds MT of them);
// wider layers take 128 x 256 tiles when the layer has enough of them to keep every SM busy for two waves, else 128 x 128.
void pick_tile(int out_c, int64_t m_tiles, int* block_n, int* mt) {
    const int64_t sms = sm_count();
    if (out_c <= 32) { *block_n = 32; *mt = 4; return; }
    if (out_c <= 64) { *block_n = 64; *mt = 2; return; }
    if (out_c <= 128) {
        *block_n = 128;
        *mt = ((m_tiles + 1) / 2) >= sms ? 2 : 1;  // 256 x 128 tiles only while they still make a full wave
        return;
    }
    const int64_t tiles256 = m_tiles * ((out_c + 255) / 256);
    *block_n = (tiles256 >= 2 * sms && (out_c % 256 == 0 || out_c > 384)) ? 256 : 128;
    *mt = 1;
}

int pick_block_n(int out_c, int64_t m_rows) {
    int bn, mt;
    pick_tile(out_c, m_rows > 0 ? (m_rows + kBlockM - 1) / kBlockM : 1, &bn, &mt);
    return bn;
}

template <int BN, int EPI, int MT, bool OPT>
int launch_conv(const CUtensorMap& a, const CUtensorMap& b, const CUtensorMap& o, const CUtensorMap& r, const ConvParams& p, int grid,
                int cluster, uint32_t smem, cudaStream_t st) {
    auto* kernel = p.is_bf16 ? conv_gemm_kernel<BN, EPI, MT, OPT, true> : conv_gemm_kernel<BN, EPI, MT, OPT, false>;
    const cudaError_t attr_err = ensure_dyn_smem(reinterpret_cast<const void*>(kernel), 227 * 1024);
    if (attr_err != cudaSuccess) return set_error(int(attr_err), "conv_gemm launch failed: %s", cudaGetErrorString(attr_err));
    return launch("conv_gemm", kernel, {grid, kThreads, smem, st, /*pdl=*/true, static_cast<unsigned>(cluster)}, a, b, o, r, p);
}

struct PlanCommon {
    CUtensorMap tmA, tmB;
    CUtensorMap tmO, tmR;  // TMA epilogue: output and residual views
    ConvParams p;
    int block_n, epi, mt, grid, cluster;
    uint32_t smem_bytes;
};

// stage counts from the shared-memory budget; fills p.a_stages/b_stages and pc.smem_bytes/grid.
// Expects p.a_sub_bytes, p.b_stage_bytes, p.num_m_tiles set.
int finish_plan(PlanCommon& pc, int block_n, int epi, int mt, int cluster = 1) {
    ConvParams& p = pc.p;
    p.cluster_n = cluster;
    p.a_stage_bytes = mt * p.a_sub_bytes;
    if (p.patch_pw > 0) p.a_stage_bytes = static_cast<uint32_t>(p.th + p.kh - 1) * p.patch_pw * p.block_k * 2;  // one shared patch per stage
    p.num_m_super = (p.num_m_tiles + mt - 1) / mt;
    p.num_n_tiles = (p.N + block_n - 1) / block_n;  // head: na * ceil(no / 128), p.N being the padded na * npad rows
    // a wide head reads each tile's bias in the epilogue: na * npad floats would not fit beside the staging at the class limit
    p.bias_n = (epi == 1 && p.no > kHeadN) ? 0 : p.num_n_tiles * block_n;
    const uint32_t budget = 225 * 1024 - 1024;
    const bool patch = p.a_mode == A_PATCH;
    int a_st = 0, b_st = 0;
    if (!patch) {
        for (int s = kMaxStages; s >= 2; --s)
            if (smem_layout(epi, p.no, p.bias_n, s, s, p.a_stage_bytes, p.b_stage_bytes, p.stg_bytes).total <= budget) { a_st = b_st = s; break; }
    } else {
        const int b_min = p.b_grouped ? 2 : 3, b_max = p.b_grouped ? 4 : kMaxStages;  // a grouped stage holds kh tiles
        for (int a = 3; a >= 2 && !a_st; --a)
            for (int b = b_max; b >= b_min; --b)
                if (smem_layout(epi, p.no, p.bias_n, a, b, p.a_stage_bytes, p.b_stage_bytes, p.stg_bytes).total <= budget) { a_st = a; b_st = b; break; }
    }
    if (a_st < 2 || b_st < 2) return set_error(Y5_E_UNSUPPORTED, "conv tile does not fit shared memory (block_n %d a %u b %u)", block_n,
                                                p.a_stage_bytes, p.b_stage_bytes);
    p.a_stages = a_st;
    p.b_stages = b_st;
    pc.smem_bytes = smem_layout(epi, p.no, p.bias_n, a_st, b_st, p.a_stage_bytes, p.b_stage_bytes, p.stg_bytes).total + 1024;
    pc.block_n = block_n;
    pc.epi = epi;
    pc.mt = mt;
    pc.cluster = cluster;
    const long long tiles = static_cast<long long>((p.num_m_super + cluster - 1) / cluster) * p.num_n_tiles;  // per cluster
    const int max_clusters = sm_count() / cluster;  // 1 CTA per SM (shared memory), persistent
    pc.grid = static_cast<int>(tiles < max_clusters ? tiles : max_clusters) * cluster;
    return 0;
}

// the optional modes run in the OPT instantiation (see conv_gemm_kernel)
bool plan_staged(const PlanCommon& pc) { return pc.p.stg_bytes > 0 && !pc.p.tma_epi; }
bool plan_opt(const PlanCommon& pc) { return pc.cluster > 1 || pc.p.patch_pw > 0 || plan_staged(pc); }

int run_plan(const PlanCommon& pc, cudaStream_t st) {
    const int key = (plan_opt(pc) ? 100000 : 0) + pc.epi * 10000 + pc.block_n * 10 + pc.mt;
    switch (key) {
        case 324: return launch_conv<32, 0, 4, false>(pc.tmA, pc.tmB, pc.tmO, pc.tmR, pc.p, pc.grid, pc.cluster, pc.smem_bytes, st);
        case 642: return launch_conv<64, 0, 2, false>(pc.tmA, pc.tmB, pc.tmO, pc.tmR, pc.p, pc.grid, pc.cluster, pc.smem_bytes, st);
        case 1281: return launch_conv<128, 0, 1, false>(pc.tmA, pc.tmB, pc.tmO, pc.tmR, pc.p, pc.grid, pc.cluster, pc.smem_bytes, st);
        case 1282: return launch_conv<128, 0, 2, false>(pc.tmA, pc.tmB, pc.tmO, pc.tmR, pc.p, pc.grid, pc.cluster, pc.smem_bytes, st);
        case 2561: return launch_conv<256, 0, 1, false>(pc.tmA, pc.tmB, pc.tmO, pc.tmR, pc.p, pc.grid, pc.cluster, pc.smem_bytes, st);
        case 11281: return launch_conv<kHeadN, 1, 1, false>(pc.tmA, pc.tmB, pc.tmO, pc.tmR, pc.p, pc.grid, pc.cluster, pc.smem_bytes, st);
        case 100324: return launch_conv<32, 0, 4, true>(pc.tmA, pc.tmB, pc.tmO, pc.tmR, pc.p, pc.grid, pc.cluster, pc.smem_bytes, st);
        case 100642: return launch_conv<64, 0, 2, true>(pc.tmA, pc.tmB, pc.tmO, pc.tmR, pc.p, pc.grid, pc.cluster, pc.smem_bytes, st);
        case 101281: return launch_conv<128, 0, 1, true>(pc.tmA, pc.tmB, pc.tmO, pc.tmR, pc.p, pc.grid, pc.cluster, pc.smem_bytes, st);
        case 101282: return launch_conv<128, 0, 2, true>(pc.tmA, pc.tmB, pc.tmO, pc.tmR, pc.p, pc.grid, pc.cluster, pc.smem_bytes, st);
        case 102561: return launch_conv<256, 0, 1, true>(pc.tmA, pc.tmB, pc.tmO, pc.tmR, pc.p, pc.grid, pc.cluster, pc.smem_bytes, st);
        // conv with LeakyReLU (EPI 2)
        case 20324: return launch_conv<32, 2, 4, false>(pc.tmA, pc.tmB, pc.tmO, pc.tmR, pc.p, pc.grid, pc.cluster, pc.smem_bytes, st);
        case 20642: return launch_conv<64, 2, 2, false>(pc.tmA, pc.tmB, pc.tmO, pc.tmR, pc.p, pc.grid, pc.cluster, pc.smem_bytes, st);
        case 21281: return launch_conv<128, 2, 1, false>(pc.tmA, pc.tmB, pc.tmO, pc.tmR, pc.p, pc.grid, pc.cluster, pc.smem_bytes, st);
        case 21282: return launch_conv<128, 2, 2, false>(pc.tmA, pc.tmB, pc.tmO, pc.tmR, pc.p, pc.grid, pc.cluster, pc.smem_bytes, st);
        case 22561: return launch_conv<256, 2, 1, false>(pc.tmA, pc.tmB, pc.tmO, pc.tmR, pc.p, pc.grid, pc.cluster, pc.smem_bytes, st);
        case 120324: return launch_conv<32, 2, 4, true>(pc.tmA, pc.tmB, pc.tmO, pc.tmR, pc.p, pc.grid, pc.cluster, pc.smem_bytes, st);
        case 120642: return launch_conv<64, 2, 2, true>(pc.tmA, pc.tmB, pc.tmO, pc.tmR, pc.p, pc.grid, pc.cluster, pc.smem_bytes, st);
        case 121281: return launch_conv<128, 2, 1, true>(pc.tmA, pc.tmB, pc.tmO, pc.tmR, pc.p, pc.grid, pc.cluster, pc.smem_bytes, st);
        case 121282: return launch_conv<128, 2, 2, true>(pc.tmA, pc.tmB, pc.tmO, pc.tmR, pc.p, pc.grid, pc.cluster, pc.smem_bytes, st);
        case 122561: return launch_conv<256, 2, 1, true>(pc.tmA, pc.tmB, pc.tmO, pc.tmR, pc.p, pc.grid, pc.cluster, pc.smem_bytes, st);
        default: return set_error(Y5_E_UNSUPPORTED, "conv: no kernel for block_n %d mt %d epi %d", pc.block_n, pc.mt, pc.epi);
    }
}

struct Geo {
    int kh, kw, pad_h, pad_w, Ho, Wo;
    long long xs, ys, ns;
};
Geo geometry(const y5_conv_desc* d) {
    Geo g;
    g.kh = d->ksize;
    g.kw = d->kw ? d->kw : d->ksize;
    g.pad_h = d->pad;
    g.pad_w = d->kw ? d->pad_w : d->pad;
    g.xs = d->in_x_stride ? d->in_x_stride : d->in_pitch;
    g.ys = d->in_y_stride ? d->in_y_stride : static_cast<long long>(d->in_w) * g.xs;
    g.ns = d->in_n_stride ? d->in_n_stride : static_cast<long long>(d->in_h) * g.ys;
    g.Ho = (d->in_h + 2 * g.pad_h - g.kh) / d->stride + 1;
    g.Wo = (d->in_w + 2 * g.pad_w - g.kw) / d->stride + 1;
    return g;
}

// TMA epilogue view of the output or the residual (EpiBox boxes, the swizzle of their row size): 2-D [M rows][N] for LINEAR and
// IM2COL tiles, 4-D (N, Wo, Ho, batch) for PATCH tiles
int encode_epi_map(CUtensorMap* map, int dtype, const void* base, int pitch, const ConvParams& p, int batch, int bn, const char* what) {
    const int rb = bn * 2 < 128 ? bn * 2 : 128;
    const cuuint64_t px = static_cast<cuuint64_t>(pitch) * 2;
    if (p.a_mode == A_PATCH) {
        cuuint64_t dims[4] = {(cuuint64_t)p.N, (cuuint64_t)p.Wo, (cuuint64_t)p.Ho, (cuuint64_t)batch};
        cuuint64_t str[3] = {px, px * p.Wo, px * p.HoWo};
        cuuint32_t box[4] = {(cuuint32_t)(rb / 2), (cuuint32_t)(p.tw < 64 ? p.tw : 64), (cuuint32_t)(p.tw < 64 ? 64 / p.tw : 1), 1};
        return encode_tiled(map, dtype, base, 4, dims, str, box, swizzle_for_row_bytes(rb), what);
    }
    cuuint64_t dims[2] = {(cuuint64_t)p.N, (cuuint64_t)p.M};
    cuuint64_t str[1] = {px};
    cuuint32_t box[2] = {(cuuint32_t)(rb / 2), 64};
    return encode_tiled(map, dtype, base, 2, dims, str, box, swizzle_for_row_bytes(rb), what);
}

}  // namespace

struct y5_conv_plan {
    PlanCommon pc;
};
struct y5_detect_plan {
    PlanCommon pc;
};

extern "C" Y5_API int y5_conv_pick(int32_t in_c, int32_t out_c, int64_t m_rows, int32_t* block_k, int32_t* block_n) {
    if (in_c <= 0 || out_c <= 0) return set_error(Y5_E_INVALID, "y5_conv_pick: non-positive channel count");
    if (block_k) *block_k = pick_block_k(in_c);
    if (block_n) *block_n = pick_block_n(out_c, m_rows);
    return 0;
}

static int validate_conv(const y5_conv_desc* d) {
    if (!d || !d->in || !d->weight || !d->bias || !d->out) return set_error(Y5_E_INVALID, "conv: null pointer");
    if (d->dtype != Y5_F16 && d->dtype != Y5_BF16) return set_error(Y5_E_UNSUPPORTED, "conv: dtype must be fp16/bf16");
    if (d->batch <= 0 || d->in_h <= 0 || d->in_w <= 0 || d->in_c <= 0 || d->out_c <= 0)
        return set_error(Y5_E_INVALID, "conv: non-positive dimension");
    const long long xs = d->in_x_stride ? d->in_x_stride : d->in_pitch;
    if (xs <= 0 || xs % 8 || (d->in_y_stride % 8) || (d->in_n_stride % 8) || d->out_pitch < d->out_c || d->out_pitch % 8 || d->out_c % 8)
        return set_error(Y5_E_INVALID, "conv: strides/pitches/out_c must be multiples of 8 elements and cover the view");
    if (!d->in_x_stride && d->in_pitch < d->in_c) return set_error(Y5_E_INVALID, "conv: in_pitch smaller than in_c");
    if (!aligned16(d->in) || !aligned16(d->out) || !aligned16(d->weight) || (d->residual && !aligned16(d->residual)))
        return set_error(Y5_E_INVALID, "conv: pointers must be 16-byte aligned");
    if (d->residual && (d->res_pitch < d->out_c || d->res_pitch % 8)) return set_error(Y5_E_INVALID, "conv: bad residual pitch");
    if (d->act != Y5_ACT_NONE && d->act != Y5_ACT_SILU && d->act != Y5_ACT_LEAKY)
        return set_error(Y5_E_UNSUPPORTED, "conv: activation code %d unsupported", d->act);
    if (d->act == Y5_ACT_LEAKY && !std::isfinite(d->act_slope)) return set_error(Y5_E_INVALID, "conv: LeakyReLU slope must be finite");
    const int kw = d->kw ? d->kw : d->ksize, pw = d->kw ? d->pad_w : d->pad;
    if (d->ksize < 1 || d->ksize > 7 || kw < 1 || kw > 7 || d->stride < 1 || d->stride > 8 || d->pad < 0 || d->pad > d->ksize || pw < 0 ||
        pw > kw)
        return set_error(Y5_E_UNSUPPORTED, "conv: kernel %dx%d stride %d pad %d,%d unsupported", d->ksize, kw, d->stride, d->pad, pw);
    return 0;
}

extern "C" Y5_API int y5_conv_plan_create(const y5_conv_desc* d, y5_conv_plan** out) {
    if (!out) return set_error(Y5_E_INVALID, "conv: null plan out");
    *out = nullptr;
    if (int e = validate_conv(d)) return e;
    const Geo g = geometry(d);
    if (g.Ho <= 0 || g.Wo <= 0) return set_error(Y5_E_INVALID, "conv: empty output");
    const int64_t M64 = static_cast<int64_t>(d->batch) * g.Ho * g.Wo;
    if (M64 > 0x7fffffff - 256) return set_error(Y5_E_UNSUPPORTED, "conv: more than 2^31 output pixels");
    const int bk = d->block_k ? d->block_k : pick_block_k(d->in_c);
    if (bk != 16 && bk != 32 && bk != 64) return set_error(Y5_E_INVALID, "conv: block_k must be 16/32/64");
    const bool plain = g.kh == 1 && g.kw == 1 && d->stride == 1 && g.pad_h == 0 && g.pad_w == 0 && !d->in_x_stride && !d->in_y_stride &&
                       !d->in_n_stride;
    // spatial tile for PATCH mode: th x tw = 128 with tw in {8..128}; pick the shape wasting the fewest pixels
    int best_tw = 0;
    double best_eff = 0.0;
    if (d->stride == 1 && !plain) {
        for (int tw = 8; tw <= 128; tw <<= 1) {
            const int th = 128 / tw;
            const double eff = (double)g.Wo * g.Ho / ((double)((g.Wo + tw - 1) / tw * tw) * ((g.Ho + th - 1) / th * th));
            if (eff > best_eff + 1e-9) { best_eff = eff; best_tw = tw; }
        }
    }
    int a_mode_sel;
    if (plain) a_mode_sel = A_LINEAR;
    else if (d->a_mode == 2 && d->stride != 1) return set_error(Y5_E_INVALID, "conv: patch mode needs stride 1");
    else if (d->a_mode == 2 || (d->a_mode == 0 && d->stride == 1 && best_eff >= 0.75)) a_mode_sel = A_PATCH;
    else a_mode_sel = A_IM2COL;

    int bn = d->block_n, mt_sel = 0, cl_sel = 1;
    {
        int bn_auto = 0;
        pick_tile(d->out_c, (M64 + kBlockM - 1) / kBlockM, &bn_auto, &mt_sel);
        if (!bn) bn = bn_auto;
        else {  // forced block_n (tests / tuning): narrow tiles fill 128 columns, reserved bit 1 asks for 256 x 128 tiles,
                // bit 2 for CTA pairs (a 2-CTA cluster sharing every weight tile), bits 8.. for the cluster size (2 | 4)
            mt_sel = bn < 128 ? 128 / bn : ((d->reserved & 2) && bn == 128 ? 2 : 1);
            cl_sel = (d->reserved >> 8) > 1 ? (d->reserved >> 8) : 1;
            if (d->reserved & 4) cl_sel = 2;
            if (cl_sel != 1 && cl_sel != 2 && cl_sel != 4) return set_error(Y5_E_INVALID, "conv: cluster size must be 1, 2 or 4");
        }
    }
    if (bn != 32 && bn != 64 && bn != 128 && bn != 256) return set_error(Y5_E_INVALID, "conv: block_n must be 32/64/128/256");
    auto* plan = new y5_conv_plan();
    PlanCommon& pc = plan->pc;
    std::memset(&pc.p, 0, sizeof(pc.p));
    ConvParams& p = pc.p;
    p.M = static_cast<int>(M64);
    p.N = d->out_c;
    p.kh = g.kh; p.kw = g.kw;
    p.Ho = g.Ho; p.Wo = g.Wo; p.HoWo = g.Ho * g.Wo;
    p.rcp_HoWo = 1.0f / static_cast<float>(p.HoWo);
    p.rcp_Wo = 1.0f / static_cast<float>(p.Wo);
    p.stride = d->stride;
    p.pad_h = g.pad_h; p.pad_w = g.pad_w;
    p.is_bf16 = d->dtype == Y5_BF16;
    p.act = d->act == Y5_ACT_SILU;
    p.slope = d->act_slope;
    p.bias = d->bias;
    p.out = d->out;
    p.out_pitch = d->out_pitch;
    p.res = d->residual;
    p.res_pitch = d->res_pitch;
    p.block_k = bk;
    p.c_chunks = (d->in_c + bk - 1) / bk;
    const int row_bytes = bk * 2;
    p.b_sub_bytes = bn * row_bytes;
    p.b_stage_bytes = p.b_sub_bytes;
    p.a_mode = a_mode_sel;

    const CUtensorMapSwizzle sw = swizzle_for_row_bytes(row_bytes);
    int e = 0;
    if (p.a_mode == A_LINEAR) {
        p.num_m_tiles = (p.M + kBlockM - 1) / kBlockM;
        p.a_sub_bytes = kBlockM * row_bytes;
        cuuint64_t dims[2] = {(cuuint64_t)d->in_c, (cuuint64_t)p.M};
        cuuint64_t str[1] = {(cuuint64_t)d->in_pitch * 2};
        cuuint32_t box[2] = {(cuuint32_t)bk, kBlockM};
        e = encode_tiled(&pc.tmA, d->dtype, d->in, 2, dims, str, box, sw, "A linear");
    } else if (p.a_mode == A_IM2COL) {
        p.num_m_tiles = (p.M + kBlockM - 1) / kBlockM;
        p.a_sub_bytes = kBlockM * row_bytes;
        e = encode_im2col(&pc.tmA, d->dtype, d->in, d->in_c, d->in_w, d->in_h, d->batch, g.xs, g.ys, g.ns, g.kh, g.kw, d->stride, g.pad_h,
                          g.pad_w, bk, kBlockM, sw);
    } else {
        p.tw = best_tw;
        p.th = 128 / best_tw;
        // wide patch mode (see the header): 128-byte rows, horizontal taps, and an 8-pixel-wide tiling that wastes no more than the
        // chosen one; with MT = 2 the two sub-tiles must be neighbours in x (even number of 8-pixel tiles per row).  Opt-in (reserved
        // bit 7, 128); bit 5 (32) wins and keeps one patch copy per horizontal tap.
        {
            const int tx8 = (g.Wo + 7) / 8, ty16 = (g.Ho + 15) / 16;
            const double eff8 = (double)g.Wo * g.Ho / ((double)tx8 * 8 * ty16 * 16);
            if ((d->reserved & 128) && !(d->reserved & 32) && row_bytes == 128 && g.kw > 1 && (mt_sel == 1 || (mt_sel == 2 && tx8 % 2 == 0)) &&
                eff8 >= best_eff - 1e-9) {
                p.tw = 8;
                p.th = 16;
                p.patch_pw = 8 * mt_sel + 8;
            }
        }
        // grouped weight stages: the kh tiles of a (chunk, horizontal tap) group travel in ONE stage -- one full/empty barrier round
        // per group instead of per tile; 256-wide weight tiles are too large to group kh of them.
        if (!p.patch_pw && g.kh > 1 && bn <= 128) {
            p.b_grouped = 1;
            p.b_stage_bytes = g.kh * p.b_sub_bytes;
        }
        p.tiles_x = (g.Wo + p.tw - 1) / p.tw;
        p.tiles_y = (g.Ho + p.th - 1) / p.th;
        p.rcp_tiles_x = 1.0f / static_cast<float>(p.tiles_x);
        p.rcp_per_img = 1.0f / static_cast<float>(p.tiles_x * p.tiles_y);
        p.num_m_tiles = d->batch * p.tiles_x * p.tiles_y;
        p.a_sub_bytes = p.patch_pw ? 8 * row_bytes : (p.th + g.kh - 1) * p.tw * row_bytes;
        cuuint64_t dims[4] = {(cuuint64_t)d->in_c, (cuuint64_t)d->in_w, (cuuint64_t)d->in_h, (cuuint64_t)d->batch};
        cuuint64_t str[3] = {(cuuint64_t)g.xs * 2, (cuuint64_t)g.ys * 2, (cuuint64_t)g.ns * 2};
        cuuint32_t box[4] = {(cuuint32_t)bk, (cuuint32_t)(p.patch_pw ? p.patch_pw : p.tw), (cuuint32_t)(p.th + g.kh - 1), 1};
        e = encode_tiled(&pc.tmA, d->dtype, d->in, 4, dims, str, box, sw, "A patch");
    }
    if (e) { delete plan; return e; }
    const uint64_t ktot = static_cast<uint64_t>(p.kh) * p.kw * p.c_chunks * bk;
    {
        cuuint64_t dims[2] = {ktot, (cuuint64_t)d->out_c};
        cuuint64_t str[1] = {ktot * 2};
        cuuint32_t box[2] = {(cuuint32_t)bk, (cuuint32_t)(bn / cl_sel)};  // cluster: each CTA fetches its slice of the rows
        e = encode_tiled(&pc.tmB, d->dtype, d->weight, 2, dims, str, box, sw, "B");
    }
    if (e) { delete plan; return e; }
    // Epilogue stores.  Default: the TMA epilogue (the tile staged in shared memory with its residual TMA-loaded there, then TMA
    // bulk stores).  Reserved bit 4 (16) forces direct stores from the registers; bit 3 (8) asks for the staged 16-byte row segments
    // of the OPT instantiation, whose optional modes (clusters, wide patch) also keep direct stores.  Either staging falls back to
    // direct stores when its block does not fit next to the pipeline stages.
    // The staging block costs the 128 x 256 tiles a pipeline stage (4 -> 3): on the stride-2 IM2COL convs, whose K loops are long and
    // whose epilogue is a small share of the tile, that measured 4-7 % slower per layer (yolov5l, H100), so they keep direct stores.
    const bool opt_modes = cl_sel > 1 || p.patch_pw > 0 || (d->reserved & 8);
    const bool stages_first = p.a_mode == A_IM2COL && bn == 256;
    if (!(d->reserved & 16) && !opt_modes && !stages_first) {
        p.tma_epi = 1;
        p.stg_bytes = static_cast<uint32_t>(mt_sel * bn * 256);  // the whole tile: MT sub-tiles x 128 rows x bn columns
        e = encode_epi_map(&pc.tmO, d->dtype, d->out, d->out_pitch, p, d->batch, bn, "output");
        if (!e && d->residual) e = encode_epi_map(&pc.tmR, d->dtype, d->residual, d->res_pitch, p, d->batch, bn, "residual");
        if (e) { delete plan; return e; }
    } else if ((d->reserved & 8) && !(d->reserved & 16)) {
        p.stg_bytes = static_cast<uint32_t>(kConsumers * 64 * (bn * 2 + 16));
    }
    const int epi = d->act == Y5_ACT_LEAKY ? 2 : 0;
    int e2 = finish_plan(pc, bn, epi, mt_sel, cl_sel);
    if (e2 && p.stg_bytes) {
        p.stg_bytes = 0;
        p.tma_epi = 0;
        e2 = finish_plan(pc, bn, epi, mt_sel, cl_sel);
    }
    if (e2) { delete plan; return e2; }
    *out = plan;
    return 0;
}

extern "C" Y5_API int y5_conv_plan_run(const y5_conv_plan* plan, void* stream) {
    if (!plan) return set_error(Y5_E_INVALID, "conv: null plan");
    return run_plan(plan->pc, static_cast<cudaStream_t>(stream));
}
extern "C" Y5_API void y5_conv_plan_destroy(y5_conv_plan* plan) { delete plan; }

extern "C" Y5_API int y5_conv_plan_info(const y5_conv_plan* plan, struct y5_conv_plan_info* out) {
    if (!plan || !out) return set_error(Y5_E_INVALID, "conv: null plan/info");
    const PlanCommon& pc = plan->pc;
    const ConvParams& p = pc.p;
    out->a_mode = p.a_mode;
    out->tw = p.tw;
    out->th = p.th;
    out->block_k = p.block_k;
    out->block_n = pc.block_n;
    out->mt = pc.mt;
    out->cluster = pc.cluster;
    out->patch_pw = p.patch_pw;
    out->b_grouped = p.b_grouped;
    out->staged = plan_staged(pc);
    out->tma_epi = p.tma_epi;
    out->opt = plan_opt(pc);
    out->epi = pc.epi;
    out->a_stages = p.a_stages;
    out->b_stages = p.b_stages;
    out->grid = pc.grid;
    return 0;
}

extern "C" Y5_API int y5_conv_bn_silu_fwd(const y5_conv_desc* d, void* stream) {
    y5_conv_plan* plan = nullptr;
    if (int e = y5_conv_plan_create(d, &plan)) return e;
    const int e = y5_conv_plan_run(plan, stream);
    y5_conv_plan_destroy(plan);
    return e;
}

extern "C" Y5_API int y5_conv_direct_fwd(const y5_conv_desc* d, void* stream) {
    if (int e = validate_conv(d)) return e;
    const Geo g = geometry(d);
    const int bk = d->block_k ? d->block_k : pick_block_k(d->in_c);
    const int cin_pad = (d->in_c + bk - 1) / bk * bk;
    const long long total = static_cast<long long>(d->batch) * g.Ho * g.Wo * d->out_c;
    const int threads = 256;
    const long long blocks = (total + threads - 1) / threads;
    return launch("conv_direct", conv_direct_kernel, {static_cast<unsigned>(blocks), threads, 0, static_cast<cudaStream_t>(stream)},
                  static_cast<const uint16_t*>(d->in), g.xs, g.ys, g.ns, d->batch, d->in_h, d->in_w, d->in_c,
                  static_cast<const uint16_t*>(d->weight), cin_pad, d->bias, static_cast<uint16_t*>(d->out), d->out_pitch, d->out_c,
                  static_cast<const uint16_t*>(d->residual), d->res_pitch, g.kh, g.kw, d->stride, g.pad_h, g.pad_w, g.Ho, g.Wo, d->act,
                  d->act_slope, d->dtype == Y5_BF16);
}

extern "C" Y5_API int y5_detect_plan_create(const y5_detect_desc* d, y5_detect_plan** out) {
    if (!out) return set_error(Y5_E_INVALID, "detect: null plan out");
    *out = nullptr;
    if (!d || !d->in || !d->weight || !d->bias) return set_error(Y5_E_INVALID, "detect: null pointer");
    if (d->dtype != Y5_F16 && d->dtype != Y5_BF16) return set_error(Y5_E_UNSUPPORTED, "detect: dtype must be fp16/bf16");
    if (d->na < 1 || d->na > 4 || d->no < 6 || d->no > kHeadMaxNo || d->nc < 1 || d->nc > kHeadMaxNc || 5 + d->nc > d->no)
        return set_error(Y5_E_UNSUPPORTED, "detect: na %d no %d nc %d unsupported (no <= %d, nc <= %d, na <= 4)", d->na, d->no, d->nc,
                         kHeadMaxNo, kHeadMaxNc);
    if (d->in_pitch < d->in_c || d->in_pitch % 8 || !aligned16(d->in) || !aligned16(d->weight))
        return set_error(Y5_E_INVALID, "detect: bad input view");
    const int64_t M64 = static_cast<int64_t>(d->batch) * d->ny * d->nx;
    if (M64 <= 0 || M64 > 0x7fffffff - 256) return set_error(Y5_E_INVALID, "detect: bad pixel count");
    const int bk = d->block_k ? d->block_k : pick_block_k(d->in_c);
    auto* plan = new y5_detect_plan();
    PlanCommon& pc = plan->pc;
    std::memset(&pc.p, 0, sizeof(pc.p));
    ConvParams& p = pc.p;
    p.M = static_cast<int>(M64);
    p.N = d->na * kHeadN * ((d->no + kHeadN - 1) / kHeadN);  // weights / bias are packed with every anchor padded to npad rows
    p.kh = p.kw = 1;
    p.Ho = d->ny; p.Wo = d->nx; p.HoWo = d->ny * d->nx;
    p.rcp_HoWo = 1.0f / static_cast<float>(p.HoWo);
    p.rcp_Wo = 1.0f / static_cast<float>(p.Wo);
    p.stride = 1;
    p.is_bf16 = d->dtype == Y5_BF16;
    p.bias = d->bias;
    p.na = d->na; p.no = d->no; p.nc = d->nc; p.nx = d->nx;
    p.z_rows = d->z_rows; p.z_row0 = d->z_row0;
    p.det_stride = d->stride;
    for (int i = 0; i < 8; ++i) p.anchor_wh[i] = d->anchor_wh[i];
    p.a_mode = A_LINEAR;
    p.block_k = bk;
    p.c_chunks = (d->in_c + bk - 1) / bk;
    const int row_bytes = bk * 2;
    p.a_sub_bytes = kBlockM * row_bytes;
    p.b_stage_bytes = kHeadN * row_bytes;
    p.num_m_tiles = (p.M + kBlockM - 1) / kBlockM;
    const CUtensorMapSwizzle sw = swizzle_for_row_bytes(row_bytes);
    cuuint64_t dims[2] = {(cuuint64_t)d->in_c, (cuuint64_t)p.M};
    cuuint64_t str[1] = {(cuuint64_t)d->in_pitch * 2};
    cuuint32_t box[2] = {(cuuint32_t)bk, kBlockM};
    int e = encode_tiled(&pc.tmA, d->dtype, d->in, 2, dims, str, box, sw, "head A");
    if (e) { delete plan; return e; }
    const uint64_t ktot = static_cast<uint64_t>(p.c_chunks) * bk;
    cuuint64_t bdims[2] = {ktot, (cuuint64_t)p.N};
    cuuint64_t bstr[1] = {ktot * 2};
    cuuint32_t bbox[2] = {(cuuint32_t)bk, (cuuint32_t)kHeadN};
    e = encode_tiled(&pc.tmB, d->dtype, d->weight, 2, bdims, bstr, bbox, sw, "head B");
    if (e) { delete plan; return e; }
    if (int e2 = finish_plan(pc, kHeadN, 1, 1)) { delete plan; return e2; }
    *out = plan;
    return 0;
}
extern "C" Y5_API int y5_detect_plan_run_to(const y5_detect_plan* plan, void* raw, void* z, void* stream) {
    if (!plan || !raw || !z) return set_error(Y5_E_INVALID, "detect: null plan/output");
    PlanCommon pc = plan->pc;
    pc.p.raw = raw;
    pc.p.z = z;
    return run_plan(pc, static_cast<cudaStream_t>(stream));
}
extern "C" Y5_API void y5_detect_plan_destroy(y5_detect_plan* plan) { delete plan; }
