// Training-mode pieces of Conv = SiLU(BN(conv(x)))  (reference models/common.py:86-88, BN eps 1e-3 / momentum 0.03 set by
// initialize_weights, models/yolo.py:259) that are not GEMMs: batch statistics, normalise + activate, and their backward.
// All of them are HBM-bound passes over a [rows = B*H*W][channels] fp16/bf16 view (NHWC, possibly a channel slice of a
// wider buffer): one thread owns 8 consecutive channels (one 16-byte access per row) and walks rows, so per-channel
// partial sums live in registers; blocks combine through shared memory and publish with fp64 atomics (the fp64 total
// keeps E[y^2] - E[y]^2 well conditioned over millions of rows).
//
// Numerics follow the reference under torch.autocast: BN math in fp32 on the low-precision conv output, its result
// rounded to the activation dtype, SiLU on that rounded value, gradients rounded to the activation dtype between ops.
#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstdlib>

#include "../../include/y5b200.h"
#include "common.cuh"
#include "host_util.h"

namespace y5 {

constexpr int kRedThreads = 256;
constexpr int kUnroll = 4;  // rows a thread has in flight per loop trip (4 x 16 B per operand)

struct RowGeom {
    int cgx;   // channel groups (of 8) handled side by side by one block
    int rows;  // thread rows per block
    int rpb;   // tensor rows per block
};
static inline int env_int(const char* name, int dflt) {
    const char* e = getenv(name);
    return e && atoi(e) > 0 ? atoi(e) : dflt;
}
// Block geometry of the row-walking passes.  `reduce` passes end with 2 x (channels of the block) fp64 atomics per block and
// the L2 retires only ~14 G of those per second (measured: 6400 x 512 statistics took 14.5 us with 400 blocks, 7.9 us with 200),
// so they want FEW row blocks: at least Y5_BN_RED_MIN_ROWS rows per block, and the block count comes from narrowing the
// channel span of a block (down to 4 groups = 64 contiguous bytes per row) instead of from shortening it.  Elementwise passes
// only pay a per-block prologue (per-channel constants), so they keep the widest span and at least two loop trips per thread.
static inline RowGeom row_geom(int channels, long long nrows, bool reduce, int resident = 4) {
    // blocks per SM the grids aim for: whole waves of the kernel's residency (4 blocks/SM forward, 3 backward)
    static const int red_env = env_int("Y5_BN_RED_BPS", 0), elt_waves = env_int("Y5_BN_ELT_WAVES", 2);
    const int elt_bps = elt_waves * resident;
    const int red_bps = red_env ? red_env : resident;  // reductions: one wave
    static const int red_min_rows = env_int("Y5_BN_RED_MIN_ROWS", 512);
    const int cg = channels / 8;
    const long long target = static_cast<long long>(sm_count()) * (reduce ? red_bps : elt_bps);
    int cgx = cg >= 32 ? 32 : (cg >= 16 ? 16 : (cg >= 8 ? 8 : (cg >= 4 ? 4 : (cg >= 2 ? 2 : 1))));
    RowGeom g;
    for (;; cgx >>= 1) {
        g.cgx = cgx;
        g.rows = kRedThreads / cgx;
        const long long gx = (cg + cgx - 1) / cgx;
        const long long quantum = static_cast<long long>(g.rows) * kUnroll;
        long long rpb = (nrows * gx + target - 1) / target;
        const long long floor_rows = reduce ? std::max<long long>(red_min_rows, quantum) : 2 * quantum;
        if (rpb < floor_rows) rpb = floor_rows;
        rpb = (rpb + quantum - 1) / quantum * quantum;
        g.rpb = static_cast<int>(rpb);
        const long long blocks = gx * ((nrows + rpb - 1) / rpb);
        if (!reduce || cgx <= 4 || blocks * 5 >= target * 3) break;
    }
    return g;
}

__device__ __forceinline__ uint4 ld16(const void* base, long long elem_off) {
    return *reinterpret_cast<const uint4*>(static_cast<const uint16_t*>(base) + elem_off);
}
__device__ __forceinline__ void st16(void* base, long long elem_off, const uint4& u) {
    *reinterpret_cast<uint4*>(static_cast<uint16_t*>(base) + elem_off) = u;
}
__device__ __forceinline__ void unpack8(const uint4& u, bool bf16, float (&v)[8]) {
    const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const float2 f = unpack2(w[i], bf16);
        v[2 * i] = f.x;
        v[2 * i + 1] = f.y;
    }
}
__device__ __forceinline__ uint4 pack8(const float (&v)[8], bool bf16) {
    uint4 u;
    u.x = pack2(v[0], v[1], bf16);
    u.y = pack2(v[2], v[3], bf16);
    u.z = pack2(v[4], v[5], bf16);
    u.w = pack2(v[6], v[7], bf16);
    return u;
}
__device__ __forceinline__ void load8(const void* base, long long elem_off, bool bf16, float (&v)[8]) { unpack8(ld16(base, elem_off), bf16, v); }
__device__ __forceinline__ void store8(void* base, long long elem_off, bool bf16, const float (&v)[8]) { st16(base, elem_off, pack8(v, bf16)); }
__device__ __forceinline__ float round_lowp(float x, bool bf16) { return unpack1(pack1(x, bf16), bf16); }

// block-level combine of NV per-thread vectors of 8 channels over the thread rows, then fp64 atomics.  The scratch is
// [channel-in-group][thread] with a row pitch of 256 + cgx words: stores and the column walk are both bank-conflict free.
template <int NV>
__device__ __forceinline__ void block_publish(float (&acc)[NV][8], int cgx, int nrows, int channels, double* const (&dst)[NV]) {
    __shared__ float red[8 * (kRedThreads + 32)];
    const int tx = threadIdx.x % cgx, ty = threadIdx.x / cgx;
    const int pitch = kRedThreads + cgx;
#pragma unroll
    for (int v = 0; v < NV; ++v) {
        __syncthreads();
#pragma unroll
        for (int i = 0; i < 8; ++i) red[i * pitch + threadIdx.x] = acc[v][i];
        __syncthreads();
        // thread (tx, ty < 8) sums channel ty of group tx over all thread rows
        if (ty < 8) {
            const float* col = red + ty * pitch + tx;
            float s0 = 0.f, s1 = 0.f;
            int r = 0;
            for (; r + 1 < nrows; r += 2) {
                s0 += col[r * cgx];
                s1 += col[(r + 1) * cgx];
            }
            if (r < nrows) s0 += col[r * cgx];
            const int c = (blockIdx.x * cgx + tx) * 8 + ty;
            if (c < channels) atomicAdd(dst[v] + c, static_cast<double>(s0 + s1));
        }
    }
}

// mode 0: sum, sum of squares;  mode 1: sum only
template <int MODE>
__global__ void __launch_bounds__(kRedThreads) col_stats_kernel(const void* __restrict__ y, int pitch, long long rows, int channels, int bf16,
                                                                int cgx, int rpb, double* __restrict__ ws, double* __restrict__ count) {
    griddep_wait();  // PDL: the predecessor kernel has completed and flushed beyond this point
    griddep_launch_dependents();
    if (count && blockIdx.x == 0 && blockIdx.y == 0 && threadIdx.x == 0) *count += static_cast<double>(rows);  // SyncBN: this rank's rows
    const int nrows = kRedThreads / cgx;
    const int tx = threadIdx.x % cgx, ty = threadIdx.x / cgx;
    const int cg = blockIdx.x * cgx + tx;
    const bool active = cg * 8 < channels;
    const bool b = bf16 != 0;
    float acc[MODE == 0 ? 2 : 1][8] = {};
    const long long r0 = static_cast<long long>(blockIdx.y) * rpb;
    const long long r1 = min(rows, r0 + rpb);
    if (active)
        for (long long r = r0 + ty; r < r1; r += kUnroll * nrows) {
            uint4 raw[kUnroll];
#pragma unroll
            for (int u = 0; u < kUnroll; ++u) {
                const long long rr = r + u * nrows;
                raw[u] = rr < r1 ? ld16(y, rr * pitch + cg * 8) : make_uint4(0u, 0u, 0u, 0u);  // +0.0 in both formats
            }
#pragma unroll
            for (int u = 0; u < kUnroll; ++u) {
                float v[8];
                unpack8(raw[u], b, v);
#pragma unroll
                for (int i = 0; i < 8; ++i) {
                    acc[0][i] += v[i];
                    if (MODE == 0) acc[1][i] = fmaf(v[i], v[i], acc[1][i]);
                }
            }
        }
    if constexpr (MODE == 0) {
        double* const dst[2] = {ws, ws + channels};
        block_publish<2>(acc, cgx, nrows, channels, dst);
    } else {
        double* const dst[1] = {ws};
        block_publish<1>(acc, cgx, nrows, channels, dst);
    }
}

// dbeta / dgamma of the reduce pass alone (SyncBN): this rank's sums, rounded as the apply pass rounds them
__global__ void bn_affine_grad_kernel(const double* __restrict__ ws, int channels, float* __restrict__ dgamma, float* __restrict__ dbeta) {
    griddep_wait();  // PDL: the predecessor kernel has completed and flushed beyond this point
    griddep_launch_dependents();
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c < channels) {
        dbeta[c] = static_cast<float>(ws[c]);
        dgamma[c] = static_cast<float>(ws[channels + c]);
    }
}

__global__ void col_sum_finalize_kernel(const double* __restrict__ ws, int channels, float* __restrict__ out) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c < channels) out[c] = static_cast<float>(ws[c]);
}

// Per-channel constants of the three passes live in shared memory:
//   a = invstd*gamma, b = beta - mean*a           -> t = round(y*a + b) is the BN output
//   forward : z = silu(t)  or  leaky(t) = t > 0 ? t : slope*t
//   reduce  : xh = y*is + m2 (m2 = -mean*invstd);  du = dz*act'(t);  sum du, sum du*xh
//   apply   : dy = du*a + y*c1 + c0  with c1 = -invstd*(dgamma/rows)*a,  c0 = -(dbeta/rows + m2*dgamma/rows)*a
// which is (du - dbeta/rows - xh*dgamma/rows)*gamma*invstd written so that four constants per channel suffice; keeping
// them out of registers lets 3-4 blocks share an SM.  Layout: two float2 tables indexed [channel-in-group * cgx + group] --
// the threads of a warp own consecutive groups, so every read is one conflict-free wavefront.  (Round 1 kept one 16-byte
// struct per channel, i.e. a 128-byte stride between the threads of a warp: 16-way bank conflicts on every constant read made
// shared memory, not HBM, the bound of these passes for layers with >= 64 channels -- 1.7 TB/s at 128 channels vs 3.5 TB/s at 32.)
struct ChanTables {
    float2 ab[kRedThreads];
    float2 cd[kRedThreads];
};
__device__ __forceinline__ int chan_slot(int i, int cgx) { return (i & 7) * cgx + (i >> 3); }  // i = channel inside the block's span

// du = dz * act'(t) rounded to the activation dtype.  LeakyReLU: torch's leaky_relu_backward (t > 0 ? dz : dz * slope)
template <int ACT>
__device__ __forceinline__ float act_bwd(float dz, float t, float slope, bool bf16) {
    if (ACT == Y5_ACT_NONE) return dz;
    if (ACT == Y5_ACT_LEAKY) return round_lowp(t > 0.0f ? dz : dz * slope, bf16);
    const float sg = __fdividef(1.0f, 1.0f + __expf(-t));
    return round_lowp(dz * sg * (1.0f + t * (1.0f - sg)), bf16);
}

// LEAKY: z = t > 0 ? t : slope * t (a template parameter, so the SiLU / linear instantiations carry none of it)
template <bool RES, bool LEAKY>
__global__ void __launch_bounds__(kRedThreads, RES ? 3 : 4) bn_act_fwd_kernel(const void* __restrict__ y, int y_pitch, void* __restrict__ z, int z_pitch,
                                                                    long long rows, int channels, int bf16, int act, int cgx, int rpb,
                                                                    float* __restrict__ mean, float* __restrict__ invstd,
                                                                    const float* __restrict__ gamma, const float* __restrict__ beta,
                                                                    const double* __restrict__ sums, const double* __restrict__ count,
                                                                    double inv_rows, double unbias, float eps,
                                                                    float momentum, float* __restrict__ running_mean,
                                                                    float* __restrict__ running_var, const void* __restrict__ res, int res_pitch,
                                                                    float slope) {
    griddep_wait();  // PDL: the predecessor kernel has completed and flushed beyond this point
    griddep_launch_dependents();
    if (count) {  // SyncBN: the row count N of all ranks, summed with the column sums; the same double arithmetic as the host's
        const double n = *count;
        inv_rows = 1.0 / n;
        unbias = n > 1.0 ? n / (n - 1.0) : 1.0;
    }
    __shared__ float2 tab[kRedThreads];
    const int nrows = kRedThreads / cgx;
    const int tx = threadIdx.x % cgx, ty = threadIdx.x / cgx;
    const int cg = blockIdx.x * cgx + tx;
    for (int i = threadIdx.x; i < cgx * 8; i += kRedThreads) {
        const int c = blockIdx.x * cgx * 8 + i;
        float2 k = make_float2(0.f, 0.f);
        if (c < channels) {
            float mu, is;
            if (sums) {  // batch statistics from the column sums of y5_bn_stats (every block derives what it needs; row-block 0 publishes)
                const double m = sums[c] * inv_rows;
                double var = fma(sums[channels + c], inv_rows, -m * m);
                if (var < 0.0) var = 0.0;
                mu = static_cast<float>(m);
                is = static_cast<float>(rsqrt(var + static_cast<double>(eps)));
                if (blockIdx.y == 0) {
                    mean[c] = mu;
                    invstd[c] = is;
                    if (running_mean) running_mean[c] = (1.f - momentum) * running_mean[c] + momentum * mu;
                    if (running_var) running_var[c] = (1.f - momentum) * running_var[c] + momentum * static_cast<float>(var * unbias);
                }
            } else {
                mu = mean[c];
                is = invstd[c];
            }
            k.x = is * gamma[c];
            k.y = beta[c] - mu * k.x;
        }
        tab[chan_slot(i, cgx)] = k;
    }
    __syncthreads();
    if (cg * 8 >= channels) return;
    const bool b = bf16 != 0;
    const float2* kt = tab + tx;  // this thread's 8 channels: kt[i * cgx], one conflict-free wavefront per read
    const long long r0 = static_cast<long long>(blockIdx.y) * rpb;
    const long long r1 = min(rows, r0 + rpb);
    for (long long r = r0 + ty; r < r1; r += kUnroll * nrows) {
        uint4 yv[kUnroll], qv[kUnroll];
#pragma unroll
        for (int u = 0; u < kUnroll; ++u) {
            const long long rr = r + u * nrows;
            if (rr < r1) {
                yv[u] = ld16(y, rr * y_pitch + cg * 8);
                if (RES) qv[u] = ld16(res, rr * res_pitch + cg * 8);  // Bottleneck shortcut (models/common.py:181)
            }
        }
#pragma unroll
        for (int u = 0; u < kUnroll; ++u) {
            const long long rr = r + u * nrows;
            if (rr < r1) {
                float v[8], q[8];
                unpack8(yv[u], b, v);
                if (RES) unpack8(qv[u], b, q);
#pragma unroll
                for (int i = 0; i < 8; ++i) {
                    const float2 k = kt[i * cgx];
                    const float t = round_lowp(fmaf(v[i], k.x, k.y), b);
                    if (LEAKY) v[i] = t > 0.0f ? t : slope * t;
                    else v[i] = act ? __fdividef(t, 1.0f + __expf(-t)) : t;
                    if (RES) v[i] = round_lowp(v[i], b) + q[i];  // z = x + act(BN(y)), each term rounded like the reference's add
                }
                st16(z, rr * z_pitch + cg * 8, pack8(v, b));
            }
        }
    }
}

// U rows in flight per thread.  This pass is bound by its instruction stream (exp + reciprocal + ~18 more per element), not by
// HBM: the constants of a channel pair are read once per loop trip and used for all U rows, and the loop nest is
// channel-pair-major so that nothing but the raw 16-byte words of the U rows stays live across it.
template <int U, bool BF16, int ACT>
__global__ void __launch_bounds__(kRedThreads, U == 4 ? 2 : 3) bn_act_bwd_reduce_kernel(const void* __restrict__ y, int y_pitch, const void* __restrict__ dz,
                                                                           int dz_pitch, long long rows, int channels,
                                                                           int cgx, int rpb, const float* __restrict__ mean,
                                                                           const float* __restrict__ invstd, const float* __restrict__ gamma,
                                                                           const float* __restrict__ beta, double* __restrict__ ws,
                                                                           void* __restrict__ du_out, int du_pitch, float slope) {
    griddep_wait();  // PDL: the predecessor kernel has completed and flushed beyond this point
    griddep_launch_dependents();
    __shared__ ChanTables tab;
    const int nrows = kRedThreads / cgx;
    const int tx = threadIdx.x % cgx, ty = threadIdx.x / cgx;
    const int cg = blockIdx.x * cgx + tx;
    for (int i = threadIdx.x; i < cgx * 8; i += kRedThreads) {
        const int c = blockIdx.x * cgx * 8 + i;
        float2 ab = make_float2(0.f, 0.f), cd = make_float2(0.f, 0.f);
        if (c < channels) {
            ab.x = invstd[c] * gamma[c];
            ab.y = beta[c] - mean[c] * ab.x;
            cd.x = invstd[c];
            cd.y = -mean[c] * invstd[c];
        }
        tab.ab[chan_slot(i, cgx)] = ab;
        tab.cd[chan_slot(i, cgx)] = cd;
    }
    __syncthreads();
    const bool active = cg * 8 < channels;
    constexpr bool b = BF16;
    float acc[2][8] = {};
    if (active) {
        const float2* kab = tab.ab + tx;
        const float2* kcd = tab.cd + tx;
        const long long r0 = static_cast<long long>(blockIdx.y) * rpb;
        const int n_here = static_cast<int>(min(rows - r0, static_cast<long long>(rpb)));  // rows of this block
        // block-relative 32-bit element offsets (rpb * pitch < 2^31): one 64-bit base per tensor instead of 64-bit row arithmetic
        const uint16_t* yb = static_cast<const uint16_t*>(y) + (r0 * y_pitch + cg * 8);
        const uint16_t* gb = static_cast<const uint16_t*>(dz) + (r0 * dz_pitch + cg * 8);
        uint16_t* ob = du_out ? static_cast<uint16_t*>(du_out) + (r0 * du_pitch + cg * 8) : nullptr;
        for (int r = ty; r < n_here; r += U * nrows) {
            {
                constexpr int h = 0;
                uint4 yv[U], gv[U];
                uint32_t duw[U][4];
#pragma unroll
                for (int u = 0; u < U; ++u) {
                    const int rr = r + (h + u) * nrows;
                    if (rr < n_here) {
                        yv[u] = *reinterpret_cast<const uint4*>(yb + static_cast<uint32_t>(rr) * static_cast<uint32_t>(y_pitch));
                        gv[u] = *reinterpret_cast<const uint4*>(gb + static_cast<uint32_t>(rr) * static_cast<uint32_t>(dz_pitch));
                    }
                }
#pragma unroll
                for (int p = 0; p < 4; ++p) {
                    const float2 ab0 = kab[(2 * p) * cgx], cd0 = kcd[(2 * p) * cgx];
                    const float2 ab1 = kab[(2 * p + 1) * cgx], cd1 = kcd[(2 * p + 1) * cgx];
#pragma unroll
                    for (int u = 0; u < U; ++u) {
                        if (r + (h + u) * nrows < n_here) {
                            const uint32_t yw[4] = {yv[u].x, yv[u].y, yv[u].z, yv[u].w};
                            const uint32_t gw[4] = {gv[u].x, gv[u].y, gv[u].z, gv[u].w};
                            const float2 yy = unpack2(yw[p], b), gg = unpack2(gw[p], b);
                            const float t0 = round_lowp(fmaf(yy.x, ab0.x, ab0.y), b), t1 = round_lowp(fmaf(yy.y, ab1.x, ab1.y), b);
                            const float du0 = act_bwd<ACT>(gg.x, t0, slope, b), du1 = act_bwd<ACT>(gg.y, t1, slope, b);
                            acc[0][2 * p] += du0;
                            acc[0][2 * p + 1] += du1;
                            acc[1][2 * p] = fmaf(du0, fmaf(yy.x, cd0.x, cd0.y), acc[1][2 * p]);
                            acc[1][2 * p + 1] = fmaf(du1, fmaf(yy.y, cd1.x, cd1.y), acc[1][2 * p + 1]);
                            duw[u][p] = pack2(du0, du1, b);
                        }
                    }
                }
                // du is already a value of the activation dtype (act_bwd rounds it): the apply pass reads it back instead of
                // re-deriving it from y and dz (exp + reciprocal + ~15 more instructions per element, which bound that pass)
                if (ob) {
#pragma unroll
                    for (int u = 0; u < U; ++u) {
                        const int rr = r + (h + u) * nrows;
                        if (rr < n_here)
                            *reinterpret_cast<uint4*>(ob + static_cast<uint32_t>(rr) * static_cast<uint32_t>(du_pitch)) =
                                make_uint4(duw[u][0], duw[u][1], duw[u][2], duw[u][3]);
                    }
                }
            }
        }
    }
    double* const dst[2] = {ws, ws + channels};
    block_publish<2>(acc, cgx, nrows, channels, dst);
}

__global__ void __launch_bounds__(kRedThreads, 4) bn_act_bwd_apply_kernel(const void* __restrict__ y, int y_pitch, const void* du, int du_pitch,
                                                                          void* dy, int dy_pitch, long long rows, int channels, int bf16,
                                                                          int cgx, int rpb, const float* __restrict__ mean,
                                                                          const float* __restrict__ invstd, const float* __restrict__ gamma,
                                                                          const double* __restrict__ ws, const double* __restrict__ count,
                                                                          float* __restrict__ dgamma, float* __restrict__ dbeta) {
    // dy = du*a + y*c1 + c0 (see the table above).  du = dz * act'(t) comes from the reduce pass (stored in the dy buffer itself
    // for SiLU layers -- each thread reads its 16 bytes before it overwrites them -- or is dz for linear layers): no
    // transcendental work is left here, the pass is a pure 2-read 1-write stream.
    griddep_wait();  // PDL: the predecessor kernel has completed and flushed beyond this point
    griddep_launch_dependents();
    __shared__ float2 tab_ac[kRedThreads];  // {a, c1}
    __shared__ float tab_d[kRedThreads];    // c0
    const int nrows = kRedThreads / cgx;
    const int tx = threadIdx.x % cgx, ty = threadIdx.x / cgx;
    const int cg = blockIdx.x * cgx + tx;
    // count != NULL (SyncBN): ws holds the sums of all ranks and *count their row count N
    const float inv_rows = 1.0f / (count ? static_cast<float>(*count) : static_cast<float>(rows));
    for (int i = threadIdx.x; i < cgx * 8; i += kRedThreads) {
        const int c = blockIdx.x * cgx * 8 + i;
        float2 ac = make_float2(0.f, 0.f);
        float d = 0.f;
        if (c < channels) {
            const float db = static_cast<float>(ws[c]), dg = static_cast<float>(ws[channels + c]);
            if (blockIdx.y == 0 && dgamma) {
                dbeta[c] = db;
                dgamma[c] = dg;
            }
            const float is = invstd[c], m2 = -mean[c] * is;
            ac.x = is * gamma[c];
            ac.y = -is * (dg * inv_rows) * ac.x;
            d = -(db * inv_rows + m2 * (dg * inv_rows)) * ac.x;
        }
        tab_ac[chan_slot(i, cgx)] = ac;
        tab_d[chan_slot(i, cgx)] = d;
    }
    __syncthreads();
    if (cg * 8 >= channels) return;
    const bool b = bf16 != 0;
    const float2* kac = tab_ac + tx;  // channel i of this thread: [i * cgx], conflict-free
    const float* kd = tab_d + tx;
    const long long r0 = static_cast<long long>(blockIdx.y) * rpb;
    const long long r1 = min(rows, r0 + rpb);
    for (long long r = r0 + ty; r < r1; r += kUnroll * nrows) {
        uint4 yv[kUnroll], gv[kUnroll];
#pragma unroll
        for (int u = 0; u < kUnroll; ++u) {
            const long long rr = r + u * nrows;
            if (rr < r1) {
                yv[u] = ld16(y, rr * y_pitch + cg * 8);
                gv[u] = ld16(du, rr * du_pitch + cg * 8);
            }
        }
#pragma unroll
        for (int u = 0; u < kUnroll; ++u) {
            const long long rr = r + u * nrows;
            if (rr < r1) {
                float v[8], g[8];
                unpack8(yv[u], b, v);
                unpack8(gv[u], b, g);
#pragma unroll
                for (int i = 0; i < 8; ++i) {
                    const float2 ac = kac[i * cgx];
                    v[i] = fmaf(g[i], ac.x, fmaf(v[i], ac.y, kd[i * cgx]));
                }
                st16(dy, rr * dy_pitch + cg * 8, pack8(v, b));
            }
        }
    }
}

// out[n, 2y, 2x, :] = in[n, y, x, :], every other pixel zero: turns the data gradient of a stride-2 conv into a
// stride-1 conv over the stuffed tensor
__global__ void zero_stuff2x_kernel(const uint4* __restrict__ in, int in_pitch16, uint4* __restrict__ out, int out_pitch16, int batch, int h,
                                    int w, int c16) {
    griddep_wait();  // PDL: the predecessor kernel has completed and flushed beyond this point
    griddep_launch_dependents();
    const long long total = static_cast<long long>(batch) * (2 * h) * (2 * w) * c16;
    for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total; i += static_cast<long long>(gridDim.x) * blockDim.x) {
        const int cc = static_cast<int>(i % c16);
        long long px = i / c16;
        const int ox = static_cast<int>(px % (2 * w));
        px /= 2 * w;
        const int oy = static_cast<int>(px % (2 * h));
        const int n = static_cast<int>(px / (2 * h));
        uint4 v = make_uint4(0, 0, 0, 0);
        if (!(ox & 1) && !(oy & 1)) v = in[((static_cast<long long>(n) * h + (oy >> 1)) * w + (ox >> 1)) * in_pitch16 + cc];
        out[((static_cast<long long>(n) * 2 * h + oy) * 2 * w + ox) * out_pitch16 + cc] = v;
    }
}

// OIHW master weights (fp32 / fp16 / bf16) -> the two K-major packings the GEMM kernel wants, in one pass:
//   fwd  [co][r][s][ci_pad]            = w[co][ci][r][s]                  (forward conv)
//   dgrad[ci][r][s][co_pad]            = w[co][ci][k-1-r][k-1-s]          (data gradient = conv with the flipped, transposed filter)
__device__ __forceinline__ float load_w(const void* w, long long i, int src_dtype) {
    if (src_dtype == Y5_F32) return static_cast<const float*>(w)[i];
    return unpack1(static_cast<const uint16_t*>(w)[i], src_dtype == Y5_BF16);
}
// element i of the concatenated [forward packing | data-gradient packing] of one OIHW filter
__device__ __forceinline__ void pack_elem(const void* __restrict__ w, int src_dtype, int cout, int cin, int k, uint16_t* __restrict__ fwd,
                                          int ci_pad, uint16_t* __restrict__ dgrad, int co_pad, bool bf16, long long n_fwd, long long i) {
    if (i < n_fwd) {
        const int ci = static_cast<int>(i % ci_pad);
        long long t = i / ci_pad;
        const int s_ = static_cast<int>(t % k);
        t /= k;
        const int r = static_cast<int>(t % k);
        const int co = static_cast<int>(t / k);
        const float v = ci < cin ? load_w(w, ((static_cast<long long>(co) * cin + ci) * k + r) * k + s_, src_dtype) : 0.f;
        fwd[i] = pack1(v, bf16);
    } else {
        const long long j = i - n_fwd;
        const int co = static_cast<int>(j % co_pad);
        long long t = j / co_pad;
        const int s_ = static_cast<int>(t % k);
        t /= k;
        const int r = static_cast<int>(t % k);
        const int ci = static_cast<int>(t / k);
        const float v = co < cout ? load_w(w, ((static_cast<long long>(co) * cin + ci) * k + (k - 1 - r)) * k + (k - 1 - s_), src_dtype) : 0.f;
        dgrad[j] = pack1(v, bf16);
    }
}
__global__ void weight_pack_kernel(const void* __restrict__ w, int src_dtype, int cout, int cin, int k, uint16_t* __restrict__ fwd, int ci_pad,
                                   uint16_t* __restrict__ dgrad, int co_pad, int bf16) {
    griddep_wait();  // PDL: the predecessor kernel has completed and flushed beyond this point
    griddep_launch_dependents();
    const long long n_fwd = fwd ? static_cast<long long>(cout) * k * k * ci_pad : 0;
    const long long n_dg = dgrad ? static_cast<long long>(cin) * k * k * co_pad : 0;
    for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < n_fwd + n_dg;
         i += static_cast<long long>(gridDim.x) * blockDim.x)
        pack_elem(w, src_dtype, cout, cin, k, fwd, ci_pad, dgrad, co_pad, bf16 != 0, n_fwd, i);
}
// every filter of a model in ONE launch (the per-step re-packing of the fp32 master weights): block b works on piece
// chunk_index[b] (kPackChunk elements) of item chunk_item[b]
constexpr int kPackChunk = 8192;
__global__ void __launch_bounds__(256) weight_pack_multi_kernel(const y5_pack_item* __restrict__ items, const int32_t* __restrict__ chunk_item,
                                                                const int32_t* __restrict__ chunk_index, int bf16) {
    griddep_wait();  // PDL: the predecessor kernel has completed and flushed beyond this point
    griddep_launch_dependents();
    const y5_pack_item it = items[chunk_item[blockIdx.x]];
    const long long n_fwd = it.fwd ? static_cast<long long>(it.out_c) * it.ksize * it.ksize * it.in_c_pad : 0;
    const long long n_dg = it.dgrad ? static_cast<long long>(it.in_c) * it.ksize * it.ksize * it.out_c_pad : 0;
    const long long i0 = static_cast<long long>(chunk_index[blockIdx.x]) * kPackChunk;
    const long long i1 = min(n_fwd + n_dg, i0 + kPackChunk);
    for (long long i = i0 + threadIdx.x; i < i1; i += blockDim.x)
        pack_elem(it.w, it.w_dtype, it.out_c, it.in_c, it.ksize, static_cast<uint16_t*>(it.fwd), it.in_c_pad, static_cast<uint16_t*>(it.dgrad),
                  it.out_c_pad, bf16 != 0, n_fwd, i);
}

// eval-mode BatchNorm folded into the conv weights + K-major packing, one launch (reference utils/torch_utils.py:224-254):
// scale = gamma / sqrt(var + eps) in fp32 (same operation order as torch's expression), W' = W * scale rounded once to the
// activation dtype, b' = beta + (b - mean) * scale in fp32.
__device__ __forceinline__ float load_any(const void* p, long long i, int dtype) {
    if (dtype == Y5_F32) return static_cast<const float*>(p)[i];
    return unpack1(static_cast<const uint16_t*>(p)[i], dtype == Y5_BF16);
}
__global__ void fold_pack_kernel(const void* __restrict__ w, int w_dtype, int cout, int cin, int kh, int kw, const void* __restrict__ cbias,
                                 const void* __restrict__ gamma, const void* __restrict__ beta, const void* __restrict__ mean,
                                 const void* __restrict__ var, int bn_dtype, float eps, uint16_t* __restrict__ packed, int ci_pad, int co_pad,
                                 float* __restrict__ bias_out, int bf16) {
    const long long n = static_cast<long long>(co_pad) * kh * kw * ci_pad;
    for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < n; i += static_cast<long long>(gridDim.x) * blockDim.x) {
        const int ci = static_cast<int>(i % ci_pad);
        long long t = i / ci_pad;
        const int s_ = static_cast<int>(t % kw);
        t /= kw;
        const int r = static_cast<int>(t % kh);
        const int co = static_cast<int>(t / kh);
        float v = 0.f;
        if (ci < cin && co < cout) {
            v = load_any(w, ((static_cast<long long>(co) * cin + ci) * kh + r) * kw + s_, w_dtype);
            if (gamma) v = __fmul_rn(v, __fdiv_rn(load_any(gamma, co, bn_dtype), __fsqrt_rn(__fadd_rn(load_any(var, co, bn_dtype), eps))));
        }
        packed[i] = pack1(v, bf16 != 0);
    }
    if (bias_out)
        for (int co = blockIdx.x * blockDim.x + threadIdx.x; co < co_pad; co += gridDim.x * blockDim.x) {
            float b = 0.f;
            if (co < cout) {
                const float b0 = cbias ? load_any(cbias, co, w_dtype) : 0.f;
                if (gamma) {
                    const float sc = __fdiv_rn(load_any(gamma, co, bn_dtype), __fsqrt_rn(__fadd_rn(load_any(var, co, bn_dtype), eps)));
                    b = __fadd_rn(load_any(beta, co, bn_dtype), __fmul_rn(__fsub_rn(b0, load_any(mean, co, bn_dtype)), sc));
                } else {
                    b = b0;
                }
            }
            bias_out[co] = b;
        }
}

// backward of nn.Upsample(scale_factor=2, 'nearest'): dx[n,y,x,:] = sum of the 2x2 block of dy (fp32 sum, one rounding)
__global__ void upsample2x_bwd_kernel(const void* __restrict__ dy, int dy_pitch, void* __restrict__ dx, int dx_pitch, int B, int H, int W, int C,
                                      int bf16) {
    griddep_wait();  // PDL: the predecessor kernel has completed and flushed beyond this point
    griddep_launch_dependents();
    const int cv = C >> 3;
    const long long total = static_cast<long long>(B) * H * W * cv;
    const bool b = bf16 != 0;
    for (long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; idx < total;
         idx += static_cast<long long>(gridDim.x) * blockDim.x) {
        const int c8 = static_cast<int>(idx % cv);
        const long long pix = idx / cv;
        const int x = static_cast<int>(pix % W);
        const int y = static_cast<int>((pix / W) % H);
        const int n = static_cast<int>(pix / (static_cast<long long>(W) * H));
        float acc[8] = {};
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            float v[8];
            load8(dy, ((static_cast<long long>(n) * 2 * H + 2 * y + (j >> 1)) * 2 * W + 2 * x + (j & 1)) * dy_pitch + c8 * 8, b, v);
#pragma unroll
            for (int i = 0; i < 8; ++i) acc[i] += v[i];
        }
        store8(dx, pix * dx_pitch + c8 * 8, b, acc);
    }
}

// ---- backward of SPPF's pooling chain  cat = [a, y1 = m(a), y2 = m(y1), y3 = m(y2)], m = MaxPool2d(k, 1, k/2) ----
// acc_j (fp32, dense [B*H*W][c]) start as the incoming gradients of slices 0..2; then, last stage first, every output
// position routes its gradient to the arg-max of its window (first maximum in row-major scan order, strict '>', as
// torch's max_pool2d_with_indices picks it):  g3 -> acc2 through y2's windows, acc2 -> acc1 through y1's, acc1 -> acc0
// through a's.  acc0 rounded is da.
__global__ void sppf_bwd_init_kernel(const void* __restrict__ dcat, int dcat_pitch, float* __restrict__ acc, long long pixels, int c, int bf16) {
    const long long total = pixels * c;
    for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < 3 * total;
         i += static_cast<long long>(gridDim.x) * blockDim.x) {
        const int j = static_cast<int>(i / total);
        const long long e = i - j * total;
        const long long pix = e / c;
        const int ch = static_cast<int>(e - pix * c);
        acc[i] = unpack1(static_cast<const uint16_t*>(dcat)[pix * dcat_pitch + j * c + ch], bf16 != 0);
    }
}
template <bool G_LOWP>
__global__ void sppf_bwd_scatter_kernel(const void* __restrict__ src, int src_pitch, const void* __restrict__ g, int g_pitch,
                                        float* __restrict__ acc, int B, int H, int W, int c, int k, int bf16) {
    const long long total = static_cast<long long>(B) * H * W * c;
    const int r = k / 2;
    const bool b = bf16 != 0;
    const uint16_t* s = static_cast<const uint16_t*>(src);
    for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < total;
         i += static_cast<long long>(gridDim.x) * blockDim.x) {
        const int ch = static_cast<int>(i % c);
        const long long pix = i / c;
        const int x = static_cast<int>(pix % W);
        const int y = static_cast<int>((pix / W) % H);
        const int n = static_cast<int>(pix / (static_cast<long long>(W) * H));
        const float gv = G_LOWP ? unpack1(static_cast<const uint16_t*>(g)[pix * g_pitch + ch], b) : static_cast<const float*>(g)[pix * g_pitch + ch];
        float best = -INFINITY;
        long long arg = -1;
        for (int yy = max(0, y - r); yy <= min(H - 1, y + r); ++yy)
            for (int xx = max(0, x - r); xx <= min(W - 1, x + r); ++xx) {
                const long long q = (static_cast<long long>(n) * H + yy) * W + xx;
                const float v = unpack1(s[q * src_pitch + ch], b);
                if (v > best || arg < 0 || v != v) {
                    best = v;
                    arg = q;
                }
            }
        if (gv != 0.f) atomicAdd(acc + arg * c + ch, gv);
    }
}
__global__ void f32_to_lowp_kernel(const float* __restrict__ in, void* __restrict__ out, int out_pitch, long long pixels, int c, int bf16) {
    const long long total = pixels * c;
    for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < total; i += static_cast<long long>(gridDim.x) * blockDim.x) {
        const long long pix = i / c;
        static_cast<uint16_t*>(out)[pix * out_pitch + (i - pix * c)] = pack1(in[i], bf16 != 0);
    }
}

static int check_view(const void* p, int pitch, int channels, const char* what) {
    if (!p) return set_error(Y5_E_INVALID, "%s: null pointer", what);
    if ((reinterpret_cast<uintptr_t>(p) & 15) || (pitch % 8) || (channels % 8) || channels <= 0 || pitch < channels)
        return set_error(Y5_E_INVALID, "%s: views must be 16-byte aligned, channels and pitch multiples of 8", what);
    return 0;
}
static dim3 row_grid(const RowGeom& g, int channels, long long rows) {
    return dim3((channels / 8 + g.cgx - 1) / g.cgx, static_cast<unsigned>((rows + g.rpb - 1) / g.rpb));
}

}  // namespace y5

using namespace y5;

extern "C" Y5_API int64_t y5_bn_workspace_bytes(int32_t channels) { return static_cast<int64_t>(channels) * 2 * sizeof(double); }

// the activation of a BN pass: Y5_ACT_NONE | Y5_ACT_SILU | Y5_ACT_LEAKY with a finite slope
static int check_act(const char* what, int32_t act, float slope) {
    if (act != Y5_ACT_NONE && act != Y5_ACT_SILU && act != Y5_ACT_LEAKY) return set_error(Y5_E_UNSUPPORTED, "%s: activation code %d unsupported", what, act);
    if (act == Y5_ACT_LEAKY && !std::isfinite(slope)) return set_error(Y5_E_INVALID, "%s: LeakyReLU slope must be finite", what);
    return 0;
}

// check_view with the operand named after the entry point ("bn_act_fwd y")
static int check_operand(const char* what, const char* operand, const void* p, int pitch, int channels) {
    char name[64];
    snprintf(name, sizeof(name), "%s %s", what, operand);
    return check_view(p, pitch, channels, name);
}

// `count` (SyncBatchNorm) is one fp64 row count, the slot after the 2*channels column sums: y5_bn_stats adds this rank's
// rows to it, and after the caller's SUM all-reduce of the whole workspace it holds N, which y5_bn_act_fwd and
// y5_bn_act_bwd_apply divide by instead of the host's `rows`.  NULL: `rows` is the whole batch.
extern "C" Y5_API int y5_bn_stats(const void* y, int32_t pitch, int64_t rows, int32_t channels, int32_t dtype, void* workspace, double* count,
                                  void* stream) {
    if (int e = check_view(y, pitch, channels, "bn_stats")) return e;
    if (dtype != Y5_F16 && dtype != Y5_BF16) return set_error(Y5_E_UNSUPPORTED, "bn_stats: dtype must be fp16 or bf16");
    if (!workspace || rows <= 0) return set_error(Y5_E_INVALID, "bn_stats: bad argument");
    const RowGeom g = row_geom(channels, rows, true);
    return launch("bn_stats", col_stats_kernel<0>, {row_grid(g, channels, rows), kRedThreads, 0, static_cast<cudaStream_t>(stream), /*pdl=*/true},
                  y, pitch, rows, channels, dtype == Y5_BF16, g.cgx, g.rpb, static_cast<double*>(workspace), count);
}

extern "C" Y5_API int y5_bn_act_fwd(const void* y, int32_t y_pitch, void* z, int32_t z_pitch, int64_t rows, int32_t channels, int32_t dtype,
                                    float* mean, float* invstd, const float* gamma, const float* beta, int32_t act, float slope,
                                    const void* sums, const void* count, float eps, float momentum, float* running_mean, float* running_var,
                                    const void* residual, int32_t res_pitch, void* stream) {
    const char* what = "bn_act_fwd";
    if (int e = check_act(what, act, slope)) return e;
    if (int e = check_operand(what, "y", y, y_pitch, channels)) return e;
    if (int e = check_operand(what, "z", z, z_pitch, channels)) return e;
    if (dtype != Y5_F16 && dtype != Y5_BF16) return set_error(Y5_E_UNSUPPORTED, "%s: dtype must be fp16 or bf16", what);
    if (!mean || !invstd || !gamma || !beta || rows <= 0) return set_error(Y5_E_INVALID, "%s: bad argument", what);
    if (count && !sums) return set_error(Y5_E_INVALID, "%s: count needs the column sums", what);
    if (residual)
        if (int e = check_operand(what, "residual", residual, res_pitch, channels)) return e;
    const RowGeom g = row_geom(channels, rows, false, residual ? 3 : 4);
    const double inv_rows = 1.0 / static_cast<double>(rows);
    const double unbias = rows > 1 ? static_cast<double>(rows) / static_cast<double>(rows - 1) : 1.0;
    const double* s = static_cast<const double*>(sums);
    const bool leaky = act == Y5_ACT_LEAKY;
    auto* kernel = residual ? (leaky ? bn_act_fwd_kernel<true, true> : bn_act_fwd_kernel<true, false>)
                            : (leaky ? bn_act_fwd_kernel<false, true> : bn_act_fwd_kernel<false, false>);
    return launch(what, kernel, {row_grid(g, channels, rows), kRedThreads, 0, static_cast<cudaStream_t>(stream), /*pdl=*/true}, y, y_pitch, z,
                  z_pitch, rows, channels, dtype == Y5_BF16, act, g.cgx, g.rpb, mean, invstd, gamma, beta, s, static_cast<const double*>(count),
                  inv_rows, unbias, eps, momentum, running_mean, running_var, residual, res_pitch, slope);
}

static int bn_bwd_check(const char* what, const void* y, int32_t y_pitch, const void* dz, int32_t dz_pitch, void* dy, int32_t dy_pitch, int64_t rows,
                        int32_t channels, int32_t dtype, const float* mean, const float* invstd, const float* gamma, const void* workspace) {
    if (int e = check_operand(what, "y", y, y_pitch, channels)) return e;
    if (int e = check_operand(what, "dz", dz, dz_pitch, channels)) return e;
    if (int e = check_operand(what, "dy", dy, dy_pitch, channels)) return e;
    if (dtype != Y5_F16 && dtype != Y5_BF16) return set_error(Y5_E_UNSUPPORTED, "%s: dtype must be fp16 or bf16", what);
    if (!mean || !invstd || !gamma || !workspace || rows <= 0) return set_error(Y5_E_INVALID, "%s: bad argument", what);
    return 0;
}

// reduce pass: du = dz * act'(t) and its two column sums into the workspace.  SiLU and LeakyReLU layers: du is left in the dy
// buffer and the apply pass finishes it in place; linear layers have du == dz
static int bn_bwd_reduce_launch(const char* what, const void* y, int32_t y_pitch, const void* dz, int32_t dz_pitch, void* dy, int32_t dy_pitch,
                                int64_t rows, int32_t channels, int32_t dtype, const float* mean, const float* invstd, const float* gamma,
                                const float* beta, int32_t act, float slope, void* workspace, cudaStream_t st) {
    static const int red_u = env_int("Y5_BN_RED_U", 4);
    const RowGeom g = row_geom(channels, rows, true, red_u == 2 ? 3 : 2);
    using RedFn = void (*)(const void*, int, const void*, int, long long, int, int, int, const float*, const float*, const float*, const float*,
                           double*, void*, int, float);
    constexpr int N = Y5_ACT_NONE, S = Y5_ACT_SILU, L = Y5_ACT_LEAKY;
    static const RedFn table[2][2][3] = {
        {{bn_act_bwd_reduce_kernel<4, false, N>, bn_act_bwd_reduce_kernel<4, false, S>, bn_act_bwd_reduce_kernel<4, false, L>},
         {bn_act_bwd_reduce_kernel<4, true, N>, bn_act_bwd_reduce_kernel<4, true, S>, bn_act_bwd_reduce_kernel<4, true, L>}},
        {{bn_act_bwd_reduce_kernel<2, false, N>, bn_act_bwd_reduce_kernel<2, false, S>, bn_act_bwd_reduce_kernel<2, false, L>},
         {bn_act_bwd_reduce_kernel<2, true, N>, bn_act_bwd_reduce_kernel<2, true, S>, bn_act_bwd_reduce_kernel<2, true, L>}}};
    return launch(what, table[red_u == 2 ? 1 : 0][dtype == Y5_BF16 ? 1 : 0][act], {row_grid(g, channels, rows), kRedThreads, 0, st, /*pdl=*/true},
                  y, y_pitch, dz, dz_pitch, rows, channels, g.cgx, g.rpb, mean, invstd, gamma, beta, static_cast<double*>(workspace),
                  act ? dy : static_cast<void*>(nullptr), dy_pitch, slope);
}

// apply pass: dy from du and the column sums (count == NULL: divided by this call's rows); dgamma / dbeta written when non-NULL
static int bn_bwd_apply_launch(const char* what, const void* y, int32_t y_pitch, const void* dz, int32_t dz_pitch, void* dy, int32_t dy_pitch,
                               int64_t rows, int32_t channels, int32_t dtype, const float* mean, const float* invstd, const float* gamma, int32_t act,
                               const double* sums, const double* count, float* dgamma, float* dbeta, cudaStream_t st) {
    const RowGeom ga = row_geom(channels, rows, false, 4);
    return launch(what, bn_act_bwd_apply_kernel, {row_grid(ga, channels, rows), kRedThreads, 0, st, /*pdl=*/true}, y, y_pitch,
                  act ? static_cast<const void*>(dy) : dz, act ? dy_pitch : dz_pitch, dy, dy_pitch, rows, channels, dtype == Y5_BF16, ga.cgx,
                  ga.rpb, mean, invstd, gamma, sums, count, dgamma, dbeta);
}

extern "C" Y5_API int y5_col_sum(const void* y, int32_t pitch, int64_t rows, int32_t channels, int32_t dtype, float* out, void* workspace,
                                 void* stream) {
    if (int e = check_view(y, pitch, channels, "col_sum")) return e;
    if (dtype != Y5_F16 && dtype != Y5_BF16) return set_error(Y5_E_UNSUPPORTED, "col_sum: dtype must be fp16 or bf16");
    if (!out || !workspace || rows <= 0) return set_error(Y5_E_INVALID, "col_sum: bad argument");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    cudaMemsetAsync(workspace, 0, static_cast<size_t>(channels) * sizeof(double), st);
    const RowGeom g = row_geom(channels, rows, true);
    if (int e = launch("col_sum", col_stats_kernel<1>, {row_grid(g, channels, rows), kRedThreads, 0, st, /*pdl=*/true}, y, pitch, rows, channels,
                       dtype == Y5_BF16, g.cgx, g.rpb, static_cast<double*>(workspace), static_cast<double*>(nullptr)))
        return e;
    return launch("col_sum", col_sum_finalize_kernel, {(channels + 127) / 128, 128, 0, st}, static_cast<const double*>(workspace), channels, out);
}

extern "C" Y5_API int y5_bn_act_bwd(const void* y, int32_t y_pitch, const void* dz, int32_t dz_pitch, void* dy, int32_t dy_pitch, int64_t rows,
                                    int32_t channels, int32_t dtype, const float* mean, const float* invstd, const float* gamma,
                                    const float* beta, int32_t act, float slope, float* dgamma, float* dbeta, void* workspace, void* stream) {
    const char* what = "bn_act_bwd";
    if (int e = check_act(what, act, slope)) return e;
    if (int e = bn_bwd_check(what, y, y_pitch, dz, dz_pitch, dy, dy_pitch, rows, channels, dtype, mean, invstd, gamma, workspace)) return e;
    if (!beta || !dgamma || !dbeta) return set_error(Y5_E_INVALID, "%s: bad argument", what);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    if (int e = bn_bwd_reduce_launch(what, y, y_pitch, dz, dz_pitch, dy, dy_pitch, rows, channels, dtype, mean, invstd, gamma, beta, act, slope,
                                     workspace, st))
        return e;
    return bn_bwd_apply_launch(what, y, y_pitch, dz, dz_pitch, dy, dy_pitch, rows, channels, dtype, mean, invstd, gamma, act,
                               static_cast<const double*>(workspace), nullptr, dgamma, dbeta, st);
}

extern "C" Y5_API int y5_bn_act_bwd_reduce(const void* y, int32_t y_pitch, const void* dz, int32_t dz_pitch, void* dy, int32_t dy_pitch,
                                           int64_t rows, int32_t channels, int32_t dtype, const float* mean, const float* invstd,
                                           const float* gamma, const float* beta, int32_t act, float slope, float* dgamma, float* dbeta,
                                           void* workspace, void* stream) {
    const char* what = "bn_act_bwd_reduce";
    if (int e = check_act(what, act, slope)) return e;
    if (int e = bn_bwd_check(what, y, y_pitch, dz, dz_pitch, dy, dy_pitch, rows, channels, dtype, mean, invstd, gamma, workspace)) return e;
    if (!beta || !dgamma || !dbeta) return set_error(Y5_E_INVALID, "%s: bad argument", what);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    if (int e = bn_bwd_reduce_launch(what, y, y_pitch, dz, dz_pitch, dy, dy_pitch, rows, channels, dtype, mean, invstd, gamma, beta, act, slope,
                                     workspace, st))
        return e;
    return launch(what, bn_affine_grad_kernel, {(channels + 127) / 128, 128, 0, st, /*pdl=*/true}, static_cast<const double*>(workspace),
                  static_cast<int>(channels), dgamma, dbeta);
}

extern "C" Y5_API int y5_bn_act_bwd_apply(const void* y, int32_t y_pitch, const void* dz, int32_t dz_pitch, void* dy, int32_t dy_pitch,
                                          int64_t rows, int32_t channels, int32_t dtype, const float* mean, const float* invstd,
                                          const float* gamma, int32_t act, const void* sums, const void* count, void* stream) {
    if (int e = check_act("bn_act_bwd_apply", act, 0.0f)) return e;
    if (int e = bn_bwd_check("bn_act_bwd_apply", y, y_pitch, dz, dz_pitch, dy, dy_pitch, rows, channels, dtype, mean, invstd, gamma, sums)) return e;
    if (!count) return set_error(Y5_E_INVALID, "bn_act_bwd_apply: bad argument");
    return bn_bwd_apply_launch("bn_act_bwd_apply", y, y_pitch, dz, dz_pitch, dy, dy_pitch, rows, channels, dtype, mean, invstd, gamma, act,
                               static_cast<const double*>(sums), static_cast<const double*>(count), nullptr, nullptr, static_cast<cudaStream_t>(stream));
}

extern "C" Y5_API int y5_zero_stuff2x(const void* x, int32_t x_pitch, void* y, int32_t y_pitch, int32_t batch, int32_t h, int32_t w, int32_t c,
                                      int32_t dtype, void* stream) {
    if (int e = check_view(x, x_pitch, c, "zero_stuff2x x")) return e;
    if (int e = check_view(y, y_pitch, c, "zero_stuff2x y")) return e;
    if (dtype != Y5_F16 && dtype != Y5_BF16) return set_error(Y5_E_UNSUPPORTED, "zero_stuff2x: dtype must be fp16 or bf16");
    if (batch <= 0 || h <= 0 || w <= 0) return set_error(Y5_E_INVALID, "zero_stuff2x: bad shape");
    const long long total = static_cast<long long>(batch) * 4 * h * w * (c / 8);
    return launch("zero_stuff2x", zero_stuff2x_kernel, {grid_stride_ctas(total, 256, 16), 256, 0, static_cast<cudaStream_t>(stream), /*pdl=*/true},
                  static_cast<const uint4*>(x), x_pitch / 8, static_cast<uint4*>(y), y_pitch / 8, batch, h, w, c / 8);
}

extern "C" Y5_API int y5_weight_pack(const void* w, int32_t w_dtype, int32_t out_c, int32_t in_c, int32_t ksize, void* fwd, int32_t in_c_pad,
                                     void* dgrad, int32_t out_c_pad, int32_t dtype, void* stream) {
    if (!w || (!fwd && !dgrad)) return set_error(Y5_E_INVALID, "weight_pack: null pointer");
    if (w_dtype != Y5_F32 && w_dtype != Y5_F16 && w_dtype != Y5_BF16) return set_error(Y5_E_UNSUPPORTED, "weight_pack: source dtype");
    if (dtype != Y5_F16 && dtype != Y5_BF16) return set_error(Y5_E_UNSUPPORTED, "weight_pack: packed dtype must be fp16 or bf16");
    if (out_c <= 0 || in_c <= 0 || ksize <= 0 || (fwd && in_c_pad < in_c) || (dgrad && out_c_pad < out_c))
        return set_error(Y5_E_INVALID, "weight_pack: bad shape");
    const long long total = (fwd ? static_cast<long long>(out_c) * ksize * ksize * in_c_pad : 0) +
                            (dgrad ? static_cast<long long>(in_c) * ksize * ksize * out_c_pad : 0);
    return launch("weight_pack", weight_pack_kernel, {grid_stride_ctas(total, 256, 8), 256, 0, static_cast<cudaStream_t>(stream), /*pdl=*/true}, w,
                  w_dtype, out_c, in_c, ksize, static_cast<uint16_t*>(fwd), in_c_pad, static_cast<uint16_t*>(dgrad), out_c_pad, dtype == Y5_BF16);
}


extern "C" Y5_API int32_t y5_weight_pack_chunk_elems(void) { return kPackChunk; }

extern "C" Y5_API int y5_weight_pack_multi(const y5_pack_item* items, const int32_t* chunk_item, const int32_t* chunk_index, int32_t n_chunks,
                                           int32_t dtype, void* stream) {
    if (n_chunks == 0) return 0;
    if (!items || !chunk_item || !chunk_index || n_chunks < 0) return set_error(Y5_E_INVALID, "weight_pack_multi: bad argument");
    if (dtype != Y5_F16 && dtype != Y5_BF16) return set_error(Y5_E_UNSUPPORTED, "weight_pack_multi: packed dtype must be fp16 or bf16");
    return launch("weight_pack_multi", weight_pack_multi_kernel, {static_cast<unsigned>(n_chunks), 256, 0, static_cast<cudaStream_t>(stream), /*pdl=*/true},
                  items, chunk_item, chunk_index, dtype == Y5_BF16);
}

extern "C" Y5_API int y5_fold_pack(const void* w, int32_t w_dtype, int32_t out_c, int32_t in_c, int32_t kh, int32_t kw, const void* conv_bias,
                                   const void* gamma, const void* beta, const void* mean, const void* var, int32_t bn_dtype, float eps,
                                   void* packed, int32_t in_c_pad, int32_t out_c_pad, float* bias_out, int32_t dtype, void* stream) {
    if (!w || !packed) return set_error(Y5_E_INVALID, "fold_pack: null pointer");
    if (w_dtype != Y5_F32 && w_dtype != Y5_F16 && w_dtype != Y5_BF16) return set_error(Y5_E_UNSUPPORTED, "fold_pack: weight dtype");
    if (bn_dtype != Y5_F32 && bn_dtype != Y5_F16 && bn_dtype != Y5_BF16) return set_error(Y5_E_UNSUPPORTED, "fold_pack: BatchNorm dtype");
    if (dtype != Y5_F16 && dtype != Y5_BF16) return set_error(Y5_E_UNSUPPORTED, "fold_pack: packed dtype must be fp16 or bf16");
    if (out_c <= 0 || in_c <= 0 || kh <= 0 || kw <= 0 || in_c_pad < in_c || out_c_pad < out_c) return set_error(Y5_E_INVALID, "fold_pack: bad shape");
    if (gamma && (!beta || !mean || !var)) return set_error(Y5_E_INVALID, "fold_pack: BatchNorm needs gamma, beta, mean and var");
    const long long total = static_cast<long long>(out_c_pad) * kh * kw * in_c_pad;
    return launch("fold_pack", fold_pack_kernel, {grid_stride_ctas(total, 256, 8), 256, 0, static_cast<cudaStream_t>(stream)}, w, w_dtype, out_c,
                  in_c, kh, kw, conv_bias, gamma, beta, mean, var, bn_dtype, eps, static_cast<uint16_t*>(packed), in_c_pad, out_c_pad, bias_out,
                  dtype == Y5_BF16);
}

extern "C" Y5_API int y5_upsample2x_bwd(const void* dy, int32_t dy_pitch, void* dx, int32_t dx_pitch, int32_t batch, int32_t h, int32_t w, int32_t c,
                                        int32_t dtype, void* stream) {
    if (int e = check_view(dy, dy_pitch, c, "upsample2x_bwd dy")) return e;
    if (int e = check_view(dx, dx_pitch, c, "upsample2x_bwd dx")) return e;
    if (dtype != Y5_F16 && dtype != Y5_BF16) return set_error(Y5_E_UNSUPPORTED, "upsample2x_bwd: dtype must be fp16 or bf16");
    if (batch <= 0 || h <= 0 || w <= 0) return set_error(Y5_E_INVALID, "upsample2x_bwd: bad shape");
    const long long total = static_cast<long long>(batch) * h * w * (c / 8);
    return launch("upsample2x_bwd", upsample2x_bwd_kernel, {grid_stride_ctas(total, 256, 16), 256, 0, static_cast<cudaStream_t>(stream), /*pdl=*/true},
                  dy, dy_pitch, dx, dx_pitch, batch, h, w, c, dtype == Y5_BF16);
}

extern "C" Y5_API int64_t y5_sppf_bwd_workspace_bytes(int32_t batch, int32_t h, int32_t w, int32_t c) {
    return static_cast<int64_t>(3) * batch * h * w * c * sizeof(float);
}

extern "C" Y5_API int y5_sppf_pool_bwd(const void* cat, int32_t cat_pitch, const void* dcat, int32_t dcat_pitch, void* da, int32_t da_pitch,
                                       int32_t batch, int32_t h, int32_t w, int32_t c, int32_t ksize, int32_t dtype, void* workspace,
                                       void* stream) {
    if (int e = check_view(cat, cat_pitch, c, "sppf_pool_bwd cat")) return e;
    if (int e = check_view(dcat, dcat_pitch, c, "sppf_pool_bwd dcat")) return e;
    if (int e = check_view(da, da_pitch, c, "sppf_pool_bwd da")) return e;
    if (dtype != Y5_F16 && dtype != Y5_BF16) return set_error(Y5_E_UNSUPPORTED, "sppf_pool_bwd: dtype must be fp16 or bf16");
    if (!workspace || batch <= 0 || h <= 0 || w <= 0 || ksize < 1 || !(ksize & 1) || cat_pitch < 4 * c || dcat_pitch < 4 * c)
        return set_error(Y5_E_INVALID, "sppf_pool_bwd: bad argument");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const long long pixels = static_cast<long long>(batch) * h * w, total = pixels * c;
    const int bf = dtype == Y5_BF16;
    const int blocks = grid_stride_ctas(total, 256, 16);
    float* acc = static_cast<float*>(workspace);
    const uint16_t* cat16 = static_cast<const uint16_t*>(cat);
    const uint16_t* dcat16 = static_cast<const uint16_t*>(dcat);
    const char* what = "sppf_pool_bwd";
    if (int e = launch(what, sppf_bwd_init_kernel, {blocks, 256, 0, st}, dcat, dcat_pitch, acc, pixels, c, bf)) return e;
    // g3 -> acc2 through the windows of y2 (slice 2);  acc2 -> acc1 through y1 (slice 1);  acc1 -> acc0 through a (slice 0)
    if (int e = launch(what, sppf_bwd_scatter_kernel<true>, {blocks, 256, 0, st}, cat16 + 2 * c, cat_pitch, dcat16 + 3 * c, dcat_pitch,
                       acc + 2 * total, batch, h, w, c, ksize, bf))
        return e;
    if (int e = launch(what, sppf_bwd_scatter_kernel<false>, {blocks, 256, 0, st}, cat16 + c, cat_pitch, acc + 2 * total, c, acc + total, batch,
                       h, w, c, ksize, bf))
        return e;
    if (int e = launch(what, sppf_bwd_scatter_kernel<false>, {blocks, 256, 0, st}, cat16, cat_pitch, acc + total, c, acc, batch, h, w, c, ksize, bf))
        return e;
    return launch(what, f32_to_lowp_kernel, {blocks, 256, 0, st}, acc, da, da_pitch, pixels, c, bf);
}
