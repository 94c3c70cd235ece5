// Fused multi-head softmax attention of the C3TR transformer layers (reference models/common.py:115-135:
// nn.MultiheadAttention with dropout 0), forward and backward, for NHWC token rows.
//
// Tokens are the rows of an NHWC view: token l of image b is row b*L + l, and head h of Q, K, V, O, dQ, dK, dV owns the
// channels [h*dh, (h+1)*dh) of its view.  One CTA of four warps owns a 64-row tile (queries in the forward and dQ passes,
// keys in the dK/dV pass); each warp owns 16 of its rows and runs mma.sync m16n8k16 tensor-core tiles with fp32
// accumulators.  The forward keeps an online softmax (running max and sum in fp32, exp2 domain) and rounds O once; it can
// write the per-row natural logsumexp, from which the backward recomputes P tile by tile, so no pass holds an L x L tensor
// in HBM.  Rows past L are zero-filled in shared memory and their columns masked with -inf, so any L >= 1 works.
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <math.h>

#include "../../include/y5b200.h"
#include "host_util.h"

namespace y5 {
namespace {

constexpr int kAttnThreads = 128;  // four warps, 16 rows each
constexpr int kTile = 64;          // rows per CTA; key columns per step of the forward and dQ passes
constexpr float kLog2e = 1.4426950408889634f;
constexpr float kLn2 = 0.6931471805599453f;

template <bool BF16>
__device__ __forceinline__ void mma16816(float* c, const uint32_t* a, uint32_t b0, uint32_t b1) {
    if constexpr (BF16) {
        asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
                     : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
                     : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
    } else {
        asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
                     : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
                     : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
    }
}

template <bool BF16>
__device__ __forceinline__ uint32_t pack(float lo, float hi) {
    if constexpr (BF16) {
        __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
        return *reinterpret_cast<uint32_t*>(&v);
    } else {
        __half2 v = __floats2half2_rn(lo, hi);
        return *reinterpret_cast<uint32_t*>(&v);
    }
}

__device__ __forceinline__ uint32_t ld32(const uint16_t* p) { return *reinterpret_cast<const uint32_t*>(p); }
__device__ __forceinline__ uint32_t ld2x16(const uint16_t* p0, const uint16_t* p1) {
    return static_cast<uint32_t>(*p0) | (static_cast<uint32_t>(*p1) << 16);
}

// Shared-memory tiles are [rows][DH + 8] elements: the 16-byte row skew keeps the fragment loads (nearly) bank-conflict free.
template <int DH>
struct Tile {
    static constexpr int kStride = DH + 8;
};

// rows [r0, r0 + R) of one head's channel slice (`src` already offset to the head's first channel) into a smem tile; rows at
// or past L are zero
template <int DH, int R>
__device__ __forceinline__ void load_tile(uint16_t* dst, const uint16_t* __restrict__ src, int pitch, long long row_base, int r0, int L) {
    constexpr int kChunks = DH / 8;
    for (int i = threadIdx.x; i < R * kChunks; i += kAttnThreads) {
        const int r = i / kChunks, c = i % kChunks;
        uint4 v = make_uint4(0, 0, 0, 0);
        if (r0 + r < L) v = *reinterpret_cast<const uint4*>(src + (row_base + r0 + r) * pitch + c * 8);
        *reinterpret_cast<uint4*>(dst + r * Tile<DH>::kStride + c * 8) = v;
    }
}

// A fragment (16 x 16, row-major) of rows [r0, r0+16), columns [k0, k0+16) of a smem tile
template <int DH>
__device__ __forceinline__ void frag_a(uint32_t* a, const uint16_t* X, int r0, int k0, int g, int t) {
    constexpr int S = Tile<DH>::kStride;
    a[0] = ld32(X + (r0 + g) * S + k0 + 2 * t);
    a[1] = ld32(X + (r0 + g + 8) * S + k0 + 2 * t);
    a[2] = ld32(X + (r0 + g) * S + k0 + 8 + 2 * t);
    a[3] = ld32(X + (r0 + g + 8) * S + k0 + 8 + 2 * t);
}

// B fragment (16 x 8) with B(k, n) = Y[n0 + n][k0 + k]: the transpose of a row-major tile (Q K^T, dO V^T)
template <int DH>
__device__ __forceinline__ void frag_bt(uint32_t& b0, uint32_t& b1, const uint16_t* Y, int n0, int k0, int g, int t) {
    constexpr int S = Tile<DH>::kStride;
    b0 = ld32(Y + (n0 + g) * S + k0 + 2 * t);
    b1 = ld32(Y + (n0 + g) * S + k0 + 8 + 2 * t);
}

// B fragment (16 x 8) with B(k, n) = Y[k0 + k][n0 + n]: a row-major tile as it is (P V, dS K, P^T dO, dS^T Q)
template <int DH>
__device__ __forceinline__ void frag_bn(uint32_t& b0, uint32_t& b1, const uint16_t* Y, int k0, int n0, int g, int t) {
    constexpr int S = Tile<DH>::kStride;
    const uint16_t* p = Y + (k0 + 2 * t) * S + n0 + g;
    b0 = ld2x16(p, p + S);
    b1 = ld2x16(p + 8 * S, p + 9 * S);
}

// The accumulator layout of two adjacent 8-column tiles is the A-fragment layout of one 16-column k step: P and dS feed the
// next product straight from registers (rounded to the dtype once).
template <bool BF16>
__device__ __forceinline__ void acc_to_a(uint32_t* a, const float* c0, const float* c1) {
    a[0] = pack<BF16>(c0[0], c0[1]);
    a[1] = pack<BF16>(c0[2], c0[3]);
    a[2] = pack<BF16>(c1[0], c1[1]);
    a[3] = pack<BF16>(c1[2], c1[3]);
}

// ---------------------------------------------------------------------------------------------------------------------
// Forward: grid (ceil(L/64), heads, B).  O = softmax(scale * Q K^T) V per (image, head); lse (optional) = the natural
// logsumexp of each row's scaled logits, [B][heads][L] fp32.
// ---------------------------------------------------------------------------------------------------------------------
template <int DH, bool BF16>
__global__ void __launch_bounds__(kAttnThreads) attn_fwd_kernel(const uint16_t* __restrict__ q, const uint16_t* __restrict__ k,
                                                                const uint16_t* __restrict__ v, int qkv_pitch, uint16_t* __restrict__ o,
                                                                int o_pitch, float* __restrict__ lse, int L, float scale_log2) {
    constexpr int S = Tile<DH>::kStride;
    extern __shared__ uint4 smem_u4[];
    uint16_t* sQ = reinterpret_cast<uint16_t*>(smem_u4);
    uint16_t* sK = sQ + kTile * S;
    uint16_t* sV = sK + kTile * S;
    const int qt = blockIdx.x, h = blockIdx.y, b = blockIdx.z, heads = gridDim.y;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
    const long long base = static_cast<long long>(b) * L;
    const int col = h * DH;
    load_tile<DH, kTile>(sQ, q + col, qkv_pitch, base, qt * kTile, L);

    float acc[DH / 8][4];
#pragma unroll
    for (int j = 0; j < DH / 8; ++j) acc[j][0] = acc[j][1] = acc[j][2] = acc[j][3] = 0.0f;
    float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.0f, 0.0f};
    const int nkt = (L + kTile - 1) / kTile;
    for (int kt = 0; kt < nkt; ++kt) {
        __syncthreads();  // the previous step is done with sK / sV
        load_tile<DH, kTile>(sK, k + col, qkv_pitch, base, kt * kTile, L);
        load_tile<DH, kTile>(sV, v + col, qkv_pitch, base, kt * kTile, L);
        __syncthreads();
        float s[8][4];
#pragma unroll
        for (int j = 0; j < 8; ++j) s[j][0] = s[j][1] = s[j][2] = s[j][3] = 0.0f;
#pragma unroll
        for (int kk = 0; kk < DH / 16; ++kk) {
            uint32_t a[4];
            frag_a<DH>(a, sQ, warp * 16, kk * 16, g, t);
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                uint32_t b0, b1;
                frag_bt<DH>(b0, b1, sK, j * 8, kk * 16, g, t);
                mma16816<BF16>(s[j], a, b0, b1);
            }
        }
        float mx[2] = {m[0], m[1]};
#pragma unroll
        for (int j = 0; j < 8; ++j) {
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const int key = kt * kTile + j * 8 + 2 * t + (e & 1);
                s[j][e] = key < L ? s[j][e] * scale_log2 : -INFINITY;
                mx[e >> 1] = fmaxf(mx[e >> 1], s[j][e]);
            }
        }
#pragma unroll
        for (int r = 0; r < 2; ++r) {
            mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 1));
            mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 2));
        }
        float alpha[2];
#pragma unroll
        for (int r = 0; r < 2; ++r) {  // every key tile holds at least one valid key: mx is finite from the first tile on
            alpha[r] = exp2f(m[r] - mx[r]);
            m[r] = mx[r];
            l[r] *= alpha[r];
        }
#pragma unroll
        for (int j = 0; j < DH / 8; ++j) {
            acc[j][0] *= alpha[0];
            acc[j][1] *= alpha[0];
            acc[j][2] *= alpha[1];
            acc[j][3] *= alpha[1];
        }
#pragma unroll
        for (int j = 0; j < 8; ++j) {
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                s[j][e] = exp2f(s[j][e] - m[e >> 1]);
                l[e >> 1] += s[j][e];
            }
        }
#pragma unroll
        for (int kk = 0; kk < kTile / 16; ++kk) {
            uint32_t a[4];
            acc_to_a<BF16>(a, s[2 * kk], s[2 * kk + 1]);
#pragma unroll
            for (int j = 0; j < DH / 8; ++j) {
                uint32_t b0, b1;
                frag_bn<DH>(b0, b1, sV, kk * 16, j * 8, g, t);
                mma16816<BF16>(acc[j], a, b0, b1);
            }
        }
    }
#pragma unroll
    for (int r = 0; r < 2; ++r) {
        l[r] += __shfl_xor_sync(0xffffffffu, l[r], 1);
        l[r] += __shfl_xor_sync(0xffffffffu, l[r], 2);
    }
#pragma unroll
    for (int r = 0; r < 2; ++r) {
        const int row = qt * kTile + warp * 16 + g + 8 * r;
        if (row >= L) continue;
        const float inv = 1.0f / l[r];
        uint16_t* dst = o + (base + row) * o_pitch + col + 2 * t;
#pragma unroll
        for (int j = 0; j < DH / 8; ++j) *reinterpret_cast<uint32_t*>(dst + j * 8) = pack<BF16>(acc[j][2 * r] * inv, acc[j][2 * r + 1] * inv);
        if (lse && t == 0) lse[(static_cast<long long>(b) * heads + h) * L + row] = (m[r] + log2f(l[r])) * kLn2;
    }
}

// ---------------------------------------------------------------------------------------------------------------------
// Backward.  With S = scale * Q K^T, P = softmax(S), dP = dO V^T and D_i = sum_d dO[i][d] O[i][d]:
//   dS = P * (dP - D),  dQ = scale * dS K,  dK = scale * dS^T Q,  dV = P^T dO.
// P is recomputed from the saved logsumexp.  Three launches: D, then dQ (CTA per query tile, looping over key tiles) and
// dK / dV (CTA per key tile, looping over query tiles); no atomics, so the gradients repeat bit for bit.
// ---------------------------------------------------------------------------------------------------------------------
template <bool BF16>
__device__ __forceinline__ float to_f(uint16_t u) {
    if constexpr (BF16) return __uint_as_float(static_cast<uint32_t>(u) << 16);
    else return __half2float(__ushort_as_half(u));
}

// delta[(b*heads + h)*L + l] = sum over the head's channels of dO * O in fp32: one warp per (token, head)
template <bool BF16>
__global__ void __launch_bounds__(256) attn_delta_kernel(const uint16_t* __restrict__ o, int o_pitch, const uint16_t* __restrict__ dout,
                                                         int do_pitch, float* __restrict__ delta, int B, int L, int heads, int dh) {
    const long long total = static_cast<long long>(B) * L * heads;
    const long long wid = (static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (wid >= total) return;
    const int h = static_cast<int>(wid % heads);
    const long long row = wid / heads;  // b*L + l
    const uint16_t* po = o + row * o_pitch + h * dh;
    const uint16_t* pd = dout + row * do_pitch + h * dh;
    float s = 0.0f;
    for (int c = lane; c < dh; c += 32) s += to_f<BF16>(po[c]) * to_f<BF16>(pd[c]);
#pragma unroll
    for (int off = 16; off; off >>= 1) s += __shfl_xor_sync(0xffffffffu, s, off);
    if (lane == 0) {
        const long long b = row / L, l = row % L;
        delta[(b * heads + h) * L + l] = s;
    }
}

// dQ: grid (ceil(L/64), heads, B)
template <int DH, bool BF16>
__global__ void __launch_bounds__(kAttnThreads) attn_dq_kernel(const uint16_t* __restrict__ q, const uint16_t* __restrict__ k,
                                                               const uint16_t* __restrict__ v, int qkv_pitch, const uint16_t* __restrict__ dout,
                                                               int do_pitch, const float* __restrict__ lse, const float* __restrict__ delta,
                                                               uint16_t* __restrict__ dq, int dqkv_pitch, int L, float scale) {
    constexpr int S = Tile<DH>::kStride;
    extern __shared__ uint4 smem_u4[];
    uint16_t* sQ = reinterpret_cast<uint16_t*>(smem_u4);
    uint16_t* sdO = sQ + kTile * S;
    uint16_t* sK = sdO + kTile * S;
    uint16_t* sV = sK + kTile * S;
    const int qt = blockIdx.x, h = blockIdx.y, b = blockIdx.z, heads = gridDim.y;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
    const long long base = static_cast<long long>(b) * L;
    const int col = h * DH;
    const float scale_log2 = scale * kLog2e;
    load_tile<DH, kTile>(sQ, q + col, qkv_pitch, base, qt * kTile, L);
    load_tile<DH, kTile>(sdO, dout + col, do_pitch, base, qt * kTile, L);
    float lse2[2], dlt[2];
#pragma unroll
    for (int r = 0; r < 2; ++r) {
        const int row = qt * kTile + warp * 16 + g + 8 * r;
        const long long idx = (static_cast<long long>(b) * heads + h) * L + row;
        lse2[r] = row < L ? lse[idx] * kLog2e : 0.0f;
        dlt[r] = row < L ? delta[idx] : 0.0f;
    }
    float acc[DH / 8][4];
#pragma unroll
    for (int j = 0; j < DH / 8; ++j) acc[j][0] = acc[j][1] = acc[j][2] = acc[j][3] = 0.0f;
    const int nkt = (L + kTile - 1) / kTile;
    for (int kt = 0; kt < nkt; ++kt) {
        __syncthreads();
        load_tile<DH, kTile>(sK, k + col, qkv_pitch, base, kt * kTile, L);
        load_tile<DH, kTile>(sV, v + col, qkv_pitch, base, kt * kTile, L);
        __syncthreads();
        float s[8][4], dp[8][4];
#pragma unroll
        for (int j = 0; j < 8; ++j)
#pragma unroll
            for (int e = 0; e < 4; ++e) s[j][e] = dp[j][e] = 0.0f;
#pragma unroll
        for (int kk = 0; kk < DH / 16; ++kk) {
            uint32_t aq[4], ad[4];
            frag_a<DH>(aq, sQ, warp * 16, kk * 16, g, t);
            frag_a<DH>(ad, sdO, warp * 16, kk * 16, g, t);
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                uint32_t b0, b1;
                frag_bt<DH>(b0, b1, sK, j * 8, kk * 16, g, t);
                mma16816<BF16>(s[j], aq, b0, b1);
                frag_bt<DH>(b0, b1, sV, j * 8, kk * 16, g, t);
                mma16816<BF16>(dp[j], ad, b0, b1);
            }
        }
#pragma unroll
        for (int j = 0; j < 8; ++j) {
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const int key = kt * kTile + j * 8 + 2 * t + (e & 1);
                const float p = key < L ? exp2f(s[j][e] * scale_log2 - lse2[e >> 1]) : 0.0f;
                s[j][e] = p * (dp[j][e] - dlt[e >> 1]);
            }
        }
#pragma unroll
        for (int kk = 0; kk < kTile / 16; ++kk) {
            uint32_t a[4];
            acc_to_a<BF16>(a, s[2 * kk], s[2 * kk + 1]);
#pragma unroll
            for (int j = 0; j < DH / 8; ++j) {
                uint32_t b0, b1;
                frag_bn<DH>(b0, b1, sK, kk * 16, j * 8, g, t);
                mma16816<BF16>(acc[j], a, b0, b1);
            }
        }
    }
#pragma unroll
    for (int r = 0; r < 2; ++r) {
        const int row = qt * kTile + warp * 16 + g + 8 * r;
        if (row >= L) continue;
        uint16_t* dst = dq + (base + row) * dqkv_pitch + col + 2 * t;
#pragma unroll
        for (int j = 0; j < DH / 8; ++j) *reinterpret_cast<uint32_t*>(dst + j * 8) = pack<BF16>(acc[j][2 * r] * scale, acc[j][2 * r + 1] * scale);
    }
}

// query rows per step of the dK / dV pass: two dh-wide accumulators per warp leave room for a 32-column step only when dh > 64
template <int DH>
__host__ __device__ constexpr int dkv_bq() { return DH <= 64 ? 64 : 32; }

// dK, dV: grid (ceil(L/64), heads, B), a CTA per 64-key tile
template <int DH, bool BF16>
__global__ void __launch_bounds__(kAttnThreads) attn_dkv_kernel(const uint16_t* __restrict__ q, const uint16_t* __restrict__ k,
                                                                const uint16_t* __restrict__ v, int qkv_pitch, const uint16_t* __restrict__ dout,
                                                                int do_pitch, const float* __restrict__ lse, const float* __restrict__ delta,
                                                                uint16_t* __restrict__ dk, uint16_t* __restrict__ dv, int dqkv_pitch, int L,
                                                                float scale) {
    constexpr int S = Tile<DH>::kStride;
    constexpr int BQ = dkv_bq<DH>();
    extern __shared__ uint4 smem_u4[];
    uint16_t* sK = reinterpret_cast<uint16_t*>(smem_u4);
    uint16_t* sV = sK + kTile * S;
    uint16_t* sQ = sV + kTile * S;
    uint16_t* sdO = sQ + BQ * S;
    float* sL = reinterpret_cast<float*>(sdO + BQ * S);
    float* sD = sL + BQ;
    const int kt = blockIdx.x, h = blockIdx.y, b = blockIdx.z, heads = gridDim.y;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
    const long long base = static_cast<long long>(b) * L;
    const long long stat = (static_cast<long long>(b) * heads + h) * L;
    const int col = h * DH;
    const float scale_log2 = scale * kLog2e;
    load_tile<DH, kTile>(sK, k + col, qkv_pitch, base, kt * kTile, L);
    load_tile<DH, kTile>(sV, v + col, qkv_pitch, base, kt * kTile, L);
    float ak[DH / 8][4], av[DH / 8][4];
#pragma unroll
    for (int j = 0; j < DH / 8; ++j)
#pragma unroll
        for (int e = 0; e < 4; ++e) ak[j][e] = av[j][e] = 0.0f;
    const int nqt = (L + BQ - 1) / BQ;
    for (int qt = 0; qt < nqt; ++qt) {
        __syncthreads();
        load_tile<DH, BQ>(sQ, q + col, qkv_pitch, base, qt * BQ, L);
        load_tile<DH, BQ>(sdO, dout + col, do_pitch, base, qt * BQ, L);
        for (int i = threadIdx.x; i < BQ; i += kAttnThreads) {
            const int row = qt * BQ + i;  // a query past L gets P = 0 through lse = +inf
            sL[i] = row < L ? lse[stat + row] * kLog2e : INFINITY;
            sD[i] = row < L ? delta[stat + row] : 0.0f;
        }
        __syncthreads();
        float st[BQ / 8][4], dpt[BQ / 8][4];  // S^T and dP^T: rows = this warp's 16 keys, columns = BQ queries
#pragma unroll
        for (int j = 0; j < BQ / 8; ++j)
#pragma unroll
            for (int e = 0; e < 4; ++e) st[j][e] = dpt[j][e] = 0.0f;
#pragma unroll
        for (int kk = 0; kk < DH / 16; ++kk) {
            uint32_t akf[4], avf[4];
            frag_a<DH>(akf, sK, warp * 16, kk * 16, g, t);
            frag_a<DH>(avf, sV, warp * 16, kk * 16, g, t);
#pragma unroll
            for (int j = 0; j < BQ / 8; ++j) {
                uint32_t b0, b1;
                frag_bt<DH>(b0, b1, sQ, j * 8, kk * 16, g, t);
                mma16816<BF16>(st[j], akf, b0, b1);
                frag_bt<DH>(b0, b1, sdO, j * 8, kk * 16, g, t);
                mma16816<BF16>(dpt[j], avf, b0, b1);
            }
        }
#pragma unroll
        for (int j = 0; j < BQ / 8; ++j) {
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const int i = j * 8 + 2 * t + (e & 1);
                const float p = exp2f(st[j][e] * scale_log2 - sL[i]);
                st[j][e] = p;
                dpt[j][e] = p * (dpt[j][e] - sD[i]);
            }
        }
#pragma unroll
        for (int kk = 0; kk < BQ / 16; ++kk) {
            uint32_t ap[4], as[4];
            acc_to_a<BF16>(ap, st[2 * kk], st[2 * kk + 1]);
            acc_to_a<BF16>(as, dpt[2 * kk], dpt[2 * kk + 1]);
#pragma unroll
            for (int j = 0; j < DH / 8; ++j) {
                uint32_t b0, b1;
                frag_bn<DH>(b0, b1, sdO, kk * 16, j * 8, g, t);
                mma16816<BF16>(av[j], ap, b0, b1);
                frag_bn<DH>(b0, b1, sQ, kk * 16, j * 8, g, t);
                mma16816<BF16>(ak[j], as, b0, b1);
            }
        }
    }
#pragma unroll
    for (int r = 0; r < 2; ++r) {
        const int row = kt * kTile + warp * 16 + g + 8 * r;
        if (row >= L) continue;
        uint16_t* pk = dk + (base + row) * dqkv_pitch + col + 2 * t;
        uint16_t* pv = dv + (base + row) * dqkv_pitch + col + 2 * t;
#pragma unroll
        for (int j = 0; j < DH / 8; ++j) {
            *reinterpret_cast<uint32_t*>(pk + j * 8) = pack<BF16>(ak[j][2 * r] * scale, ak[j][2 * r + 1] * scale);
            *reinterpret_cast<uint32_t*>(pv + j * 8) = pack<BF16>(av[j][2 * r], av[j][2 * r + 1]);
        }
    }
}

template <int DH>
constexpr int fwd_smem() { return 3 * kTile * Tile<DH>::kStride * 2; }
template <int DH>
constexpr int dq_smem() { return 4 * kTile * Tile<DH>::kStride * 2; }
template <int DH>
constexpr int dkv_smem() { return (2 * kTile + 2 * dkv_bq<DH>()) * Tile<DH>::kStride * 2 + 2 * dkv_bq<DH>() * 4; }

template <int DH, bool BF16>
int launch_fwd(const void* q, const void* k, const void* v, int qkv_pitch, void* o, int o_pitch, float* lse, int B, int L, int heads, float scale,
               cudaStream_t st) {
    auto kern = attn_fwd_kernel<DH, BF16>;
    constexpr int smem = fwd_smem<DH>();
    cudaError_t e = ensure_dyn_smem(reinterpret_cast<const void*>(kern), smem);
    if (e != cudaSuccess) return set_error(int(e), "attention_fwd: shared memory attribute: %s", cudaGetErrorString(e));
    dim3 grid((L + kTile - 1) / kTile, heads, B);
    return launch("attention_fwd", kern, {grid, kAttnThreads, smem, st}, static_cast<const uint16_t*>(q), static_cast<const uint16_t*>(k),
                  static_cast<const uint16_t*>(v), qkv_pitch, static_cast<uint16_t*>(o), o_pitch, lse, L, scale * kLog2e);
}

template <int DH, bool BF16>
int launch_bwd(const void* q, const void* k, const void* v, int qkv_pitch, const void* dout, int do_pitch, const float* lse, const float* delta,
               void* dq, void* dk, void* dv, int dqkv_pitch, int B, int L, int heads, float scale, cudaStream_t st) {
    auto kq = attn_dq_kernel<DH, BF16>;
    auto kkv = attn_dkv_kernel<DH, BF16>;
    constexpr int smem_q = dq_smem<DH>(), smem_kv = dkv_smem<DH>();
    cudaError_t e = ensure_dyn_smem(reinterpret_cast<const void*>(kq), smem_q);
    if (e == cudaSuccess) e = ensure_dyn_smem(reinterpret_cast<const void*>(kkv), smem_kv);
    if (e != cudaSuccess) return set_error(int(e), "attention_bwd: shared memory attribute: %s", cudaGetErrorString(e));
    dim3 grid((L + kTile - 1) / kTile, heads, B);
    const uint16_t *q16 = static_cast<const uint16_t*>(q), *k16 = static_cast<const uint16_t*>(k), *v16 = static_cast<const uint16_t*>(v);
    const uint16_t* d16 = static_cast<const uint16_t*>(dout);
    if (int r = launch("attention_bwd dq", kq, {grid, kAttnThreads, smem_q, st}, q16, k16, v16, qkv_pitch, d16, do_pitch, lse, delta,
                       static_cast<uint16_t*>(dq), dqkv_pitch, L, scale))
        return r;
    return launch("attention_bwd dk dv", kkv, {grid, kAttnThreads, smem_kv, st}, q16, k16, v16, qkv_pitch, d16, do_pitch, lse, delta,
                  static_cast<uint16_t*>(dk), static_cast<uint16_t*>(dv), dqkv_pitch, L, scale);
}

// common argument checks of both passes; returns 0 or the error code (message recorded)
int check_common(const char* what, const void* q, const void* k, const void* v, int qkv_pitch, int batch, int seq, int heads, int head_dim,
                 float scale, int dtype) {
    if (!q || !k || !v || batch < 1 || seq < 1 || heads < 1) return set_error(Y5_E_INVALID, "%s: null pointer, batch < 1, seq < 1 or heads < 1", what);
    if (head_dim != 32 && head_dim != 64 && head_dim != 96 && head_dim != 128 && head_dim != 160)
        return set_error(Y5_E_UNSUPPORTED, "%s: head_dim %d (32, 64, 96, 128 and 160 are built)", what, head_dim);
    if (dtype != Y5_F16 && dtype != Y5_BF16) return set_error(Y5_E_UNSUPPORTED, "%s: dtype %d (fp16 / bf16 only)", what, dtype);
    if (!(scale > 0.0f) || !isfinite(scale)) return set_error(Y5_E_INVALID, "%s: scale must be finite and > 0", what);
    if (qkv_pitch < heads * head_dim || qkv_pitch % 8) return set_error(Y5_E_INVALID, "%s: qkv_pitch %d (>= heads*head_dim, multiple of 8)", what, qkv_pitch);
    if (!aligned16(q) || !aligned16(k) || !aligned16(v)) return set_error(Y5_E_INVALID, "%s: q, k and v must be 16-byte aligned", what);
    return 0;
}

}  // namespace
}  // namespace y5

using namespace y5;

#define Y5_ATTN_DISPATCH(CALL)                                                    \
    switch (head_dim * 2 + (dtype == Y5_BF16)) {                                  \
        case 64: return CALL(32, false);                                          \
        case 65: return CALL(32, true);                                           \
        case 128: return CALL(64, false);                                         \
        case 129: return CALL(64, true);                                          \
        case 192: return CALL(96, false);                                         \
        case 193: return CALL(96, true);                                          \
        case 256: return CALL(128, false);                                        \
        case 257: return CALL(128, true);                                         \
        case 320: return CALL(160, false);                                        \
        case 321: return CALL(160, true);                                         \
        default: return set_error(Y5_E_UNSUPPORTED, "attention: head_dim %d", head_dim); \
    }

extern "C" Y5_API int y5_attention_fwd(const void* q, const void* k, const void* v, int32_t qkv_pitch, void* o, int32_t o_pitch, float* lse,
                                       int32_t batch, int32_t seq, int32_t heads, int32_t head_dim, float scale, int32_t dtype, void* stream) {
    int r = check_common("attention_fwd", q, k, v, qkv_pitch, batch, seq, heads, head_dim, scale, dtype);
    if (r) return r;
    if (!o || o_pitch < heads * head_dim || o_pitch % 8 || !aligned16(o))
        return set_error(Y5_E_INVALID, "attention_fwd: o must be 16-byte aligned with o_pitch >= heads*head_dim, a multiple of 8");
    if (lse && (reinterpret_cast<uintptr_t>(lse) & 3)) return set_error(Y5_E_INVALID, "attention_fwd: lse must be 4-byte aligned");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
#define Y5_FWD(DH, BF) launch_fwd<DH, BF>(q, k, v, qkv_pitch, o, o_pitch, lse, batch, seq, heads, scale, st)
    Y5_ATTN_DISPATCH(Y5_FWD)
#undef Y5_FWD
}

extern "C" Y5_API int y5_attention_bwd(const void* q, const void* k, const void* v, int32_t qkv_pitch, const void* o, int32_t o_pitch,
                                       const void* dout, int32_t dout_pitch, const float* lse, float* delta, void* dq, void* dk, void* dv,
                                       int32_t dqkv_pitch, int32_t batch, int32_t seq, int32_t heads, int32_t head_dim, float scale,
                                       int32_t dtype, void* stream) {
    int r = check_common("attention_bwd", q, k, v, qkv_pitch, batch, seq, heads, head_dim, scale, dtype);
    if (r) return r;
    const int hd = heads * head_dim;
    if (!o || !dout || !lse || !delta || !dq || !dk || !dv) return set_error(Y5_E_INVALID, "attention_bwd: null pointer");
    if (o_pitch < hd || dout_pitch < hd || dqkv_pitch < hd || o_pitch % 8 || dout_pitch % 8 || dqkv_pitch % 8)
        return set_error(Y5_E_INVALID, "attention_bwd: o_pitch, dout_pitch and dqkv_pitch must be >= heads*head_dim and multiples of 8");
    if (!aligned16(o) || !aligned16(dout) || !aligned16(dq) || !aligned16(dk) || !aligned16(dv) || (reinterpret_cast<uintptr_t>(lse) & 3) ||
        (reinterpret_cast<uintptr_t>(delta) & 3))
        return set_error(Y5_E_INVALID, "attention_bwd: o, dout, dq, dk, dv must be 16-byte aligned, lse and delta 4-byte aligned");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const long long warps = static_cast<long long>(batch) * seq * heads;
    const long long blocks = (warps * 32 + 255) / 256;
    r = launch("attention_bwd delta", dtype == Y5_BF16 ? attn_delta_kernel<true> : attn_delta_kernel<false>,
               {static_cast<unsigned>(blocks), 256, 0, st}, static_cast<const uint16_t*>(o), o_pitch, static_cast<const uint16_t*>(dout), dout_pitch,
               delta, batch, seq, heads, head_dim);
    if (r) return r;
#define Y5_BWD(DH, BF) launch_bwd<DH, BF>(q, k, v, qkv_pitch, dout, dout_pitch, lse, delta, dq, dk, dv, dqkv_pitch, batch, seq, heads, scale, st)
    Y5_ATTN_DISPATCH(Y5_BWD)
#undef Y5_BWD
}
