// SPDX-License-Identifier: Apache-2.0
// Fused scaled-dot-product attention for sm_90a (wgmma + TMA), forward and backward.
//
// Replaces: diffusers Attention (AttnProcessor2_0 -> F.scaled_dot_product_attention, or xFormers when
// `enable_xformers`, reference hcpdiff/train_ac.py:258-263) inside BasicTransformerBlock.attn1/attn2
// (module structure: reference cfgs/unet_struct.txt:17-43) and its autograd backward.
//
// Layout: Q/K/V/O are token-major bf16 matrices [B, L, ld] in which head h occupies columns [h*d, (h+1)*d) -- the
// layout the (fused) projection GEMMs write and the out-projection GEMM reads, so no head permute ever exists in
// HBM.  A 4D TMA map (d, H, L, B) with box (64, 1, rows, 1) lands a [rows x 64] K-major SWIZZLE_128B tile of one head
// in shared memory; columns >= d and rows >= L are zero-filled by the TMA unit.
//
// Forward, one CTA per (128 query rows, head, image): two MMA warpgroups of 64 query rows each + one TMA warp.
//   S = Q K^T            wgmma SS, fp32 S in registers
//   online softmax       on the accumulator fragments (a row lives in the four lanes of a quad); exp2 with folded scale
//   O += P V             wgmma RS: P (bf16) goes from the S registers straight into the A operand; V is used from its
//                        row-major TMA box as an MN-major operand
// Backward, one CTA per (128 kv rows, head, image, output column slice of 64) looping over 64-row query tiles; warpgroup g owns
// kv rows [64g, 64g+64):
//   S^T = K Q^T, dP^T = V dO^T (registers) -> P^T, dS^T -> dV += P^T dO, dK += dS^T Q (wgmma RS, accumulators in registers),
//   dQ_i += dS K over all 128 kv rows of the CTA (dS^T of both warpgroups staged in shared memory as one MN-major operand; the
//   warpgroups take turns per query tile), reduced into an fp32 buffer with vector red.global: one contribution per CTA, so a
//   short kv range (<= 2 tiles) sums dQ in an order-independent way.
#include <stdlib.h>
#include "common.cuh"
#include "host_util.h"
#include "../../include/hcp_b200.h"

namespace hcp {

constexpr int kAttnThreads = 288;          // warps 0-7: two MMA warpgroups, warp 8: TMA
constexpr int BOX_BYTES = 128 * 128;       // one [128 rows x 64 cols] bf16 box
constexpr float kLog2e = 1.4426950408889634f;
constexpr float kLn2 = 0.6931471805599453f;

// offset (in 16-byte units) of k-step ks inside a K-major operand made of 64-column SWIZZLE_128B boxes of `box_bytes` each
__device__ __forceinline__ uint32_t kmajor_off(int ks, int box_bytes) { return (uint32_t)((ks >> 2) * (box_bytes >> 4) + (ks & 3) * 2); }
__device__ __forceinline__ float quad_max(float v) {
    v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 1));
    return fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 2));
}
__device__ __forceinline__ float quad_sum(float v) {
    v += __shfl_xor_sync(0xffffffffu, v, 1);
    return v + __shfl_xor_sync(0xffffffffu, v, 2);
}

// =============================================================================================
// forward
// =============================================================================================
struct alignas(64) AttnFwdParams {
    CUtensorMap tmQ, tmK, tmV;   // Q: boxes of 128 rows; K / V: boxes of KVT rows
    int B, H, Lq, Lkv, d;
    int nks;             // 16-wide k-steps of Q K^T: ceil(d / 16)
    float scale_log2;    // softmax scale * log2(e)
    const float* kv_bias;   // [B, Lkv] additive bias (natural-log units) or nullptr
    __nv_bfloat16* O;
    int64_t ldo;
    float* lse;          // [B, H, Lq], natural log
};

// NB = 64-column boxes per head row (ceil(d / 64)), KVT = kv rows per tile.  Per thread: KVT / 2 S registers + 32 NB O registers.
template <int NB, int KVT>
struct AttnFwdCfg {
    static constexpr int Q_BYTES = NB * BOX_BYTES;
    static constexpr int KV_BOX = KVT * 128;
    static constexpr int KV_BYTES = NB * KV_BOX;          // one K (or V) tile
    static constexpr int STAGES = 2;
    static constexpr int SMEM_BYTES = Q_BYTES + 2 * STAGES * KV_BYTES + 256 + 1024;
};

template <int NB, int KVT>
__global__ void __launch_bounds__(kAttnThreads, 1) attn_fwd_kernel(const __grid_constant__ AttnFwdParams p) {
    using Cfg = AttnFwdCfg<NB, KVT>;
    constexpr int STAGES = Cfg::STAGES;
    constexpr int DN = 64 * NB;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint8_t* sQ = smem;
    uint8_t* sK = sQ + Cfg::Q_BYTES;                     // [STAGES]
    uint8_t* sV = sK + STAGES * Cfg::KV_BYTES;           // [STAGES]
    uint64_t* bars = reinterpret_cast<uint64_t*>(sV + STAGES * Cfg::KV_BYTES);
    uint64_t* q_full = bars;
    uint64_t* kv_full = bars + 1;                        // [STAGES]
    uint64_t* kv_empty = bars + 1 + STAGES;              // [STAGES]

    const int warp = warp_id_uniform(), lane = threadIdx.x & 31;
    const int qt = blockIdx.x, h = blockIdx.y, b = blockIdx.z;
    const int nkv = (p.Lkv + KVT - 1) / KVT;

    if (threadIdx.x == 0) {
        mbar_init(q_full, 1);
        for (int s = 0; s < STAGES; ++s) { mbar_init(&kv_full[s], 1); mbar_init(&kv_empty[s], 256); }
        fence_mbar_init();
    }
    __syncthreads();
    pdl_trigger();
    pdl_wait();

    if (warp == 8) {
        if (elect_one()) {
            mbar_arrive_expect_tx(q_full, Cfg::Q_BYTES);
            for (int bx = 0; bx < NB; ++bx) tma_load_4d(sQ + bx * BOX_BYTES, &p.tmQ, q_full, bx * 64, h, qt * 128, b);
            for (int j = 0; j < nkv; ++j) {
                const int st = j % STAGES;
                mbar_wait(&kv_empty[st], ((j / STAGES) & 1) ^ 1);
                mbar_arrive_expect_tx(&kv_full[st], 2 * Cfg::KV_BYTES);
                for (int bx = 0; bx < NB; ++bx) {
                    tma_load_4d(sK + st * Cfg::KV_BYTES + bx * Cfg::KV_BOX, &p.tmK, &kv_full[st], bx * 64, h, j * KVT, b);
                    tma_load_4d(sV + st * Cfg::KV_BYTES + bx * Cfg::KV_BOX, &p.tmV, &kv_full[st], bx * 64, h, j * KVT, b);
                }
            }
        }
        return;
    }

    // ------------------------------ MMA warpgroups: rows of a quad's thread are g and g + 8 ------------------------------
    const int wg = warp >> 2;
    const int g = lane >> 2, cq = 2 * (lane & 3);
    const int row0 = wg * 64 + (warp & 3) * 16 + g;      // tile rows row0 and row0 + 8
    const float* bias = p.kv_bias ? p.kv_bias + (int64_t)b * p.Lkv : nullptr;
    const float sl2 = p.scale_log2;
    float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};
    float o[DN / 2];
#pragma unroll
    for (int i = 0; i < DN / 2; ++i) o[i] = 0.f;
    const uint64_t qdesc = make_smem_desc(smem_u32(sQ) + wg * 64 * 128, 16, 1024);
    mbar_wait(q_full, 0);
    for (int j = 0; j < nkv; ++j) {
        const int st = j % STAGES;
        const int kv0 = j * KVT;
        const int ncols = min(KVT, p.Lkv - kv0);
        mbar_wait(&kv_full[st], (j / STAGES) & 1);
        // ---- S = Q K^T
        float s[KVT / 2];
        const uint64_t kdesc = make_smem_desc(smem_u32(sK + st * Cfg::KV_BYTES), 16, 1024);
        wgmma_fence();
        wgmma_ss<KVT, 0, 0>(s, qdesc, kdesc, 0u);
        for (int ks = 1; ks < p.nks; ++ks)
            wgmma_ss<KVT, 0, 0>(s, desc_adv(qdesc, kmajor_off(ks, BOX_BYTES)), desc_adv(kdesc, kmajor_off(ks, Cfg::KV_BOX)), 1u);
        wgmma_commit();
        wgmma_wait<0>();
        wgmma_fence_acc(s);
        // ---- online softmax (log2 domain)
        float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
        for (int c8 = 0; c8 < KVT / 8; ++c8) {
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                const int col = c8 * 8 + cq + e;
                const float bv = (bias && col < ncols) ? bias[kv0 + col] * kLog2e : 0.f;
#pragma unroll
                for (int hh = 0; hh < 2; ++hh) {
                    float v = s[4 * c8 + 2 * hh + e] * sl2 + bv;
                    v = (col < ncols) ? v : -INFINITY;
                    s[4 * c8 + 2 * hh + e] = v;
                    mx[hh] = fmaxf(mx[hh], v);
                }
            }
        }
        float mu[2];
#pragma unroll
        for (int hh = 0; hh < 2; ++hh) {
            const float m_new = fmaxf(m[hh], quad_max(mx[hh]));
            mu[hh] = (m_new == -INFINITY) ? 0.f : m_new;             // a row with no finite score so far: P = 0, nothing to rescale
            const float alpha = fast_exp2(m[hh] - mu[hh]);           // exp2(-inf) = 0 on the first tile
            l[hh] *= alpha;
#pragma unroll
            for (int c8 = 0; c8 < DN / 8; ++c8) { o[4 * c8 + 2 * hh] *= alpha; o[4 * c8 + 2 * hh + 1] *= alpha; }
            m[hh] = m_new;
        }
        // ---- P = exp2(s - m) as bf16 A fragments; the row sums use the bf16-rounded values the MMA sees
        uint32_t pa[KVT / 16][4];
#pragma unroll
        for (int kk = 0; kk < KVT / 16; ++kk) {
#pragma unroll
            for (int r = 0; r < 4; ++r) {
                const int hh = r & 1;
                const int i = 8 * kk + 4 * (r >> 1) + 2 * hh;
                const uint32_t u = pack_bf16x2(fast_exp2(s[i] - mu[hh]), fast_exp2(s[i + 1] - mu[hh]));
                const float2 f = unpack_bf16x2(u);
                l[hh] += f.x + f.y;
                pa[kk][r] = u;
            }
        }
        // ---- O += P V   (V tile: MN-major B operand; LBO = distance between its 64-column boxes)
        const uint64_t vdesc = make_smem_desc(smem_u32(sV + st * Cfg::KV_BYTES), Cfg::KV_BOX, 1024);
        wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < KVT / 16; ++kk) wgmma_rs<DN, 1>(o, pa[kk], desc_adv(vdesc, kk * 128), 1u);
        wgmma_commit();
        wgmma_wait<0>();
        wgmma_fence_acc(o);
        mbar_arrive(&kv_empty[st]);
    }
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
        const float lt = quad_sum(l[hh]);
        const int qrow = qt * 128 + row0 + 8 * hh;
        if (qrow >= p.Lq) continue;
        const float inv = 1.f / lt;
        __nv_bfloat16* orow = p.O + ((int64_t)b * p.Lq + qrow) * p.ldo + (int64_t)h * p.d;
#pragma unroll
        for (int c8 = 0; c8 < DN / 8; ++c8) {
            const int col = c8 * 8 + cq;
            if (col < p.d) *reinterpret_cast<uint32_t*>(orow + col) = pack_bf16x2(o[4 * c8 + 2 * hh] * inv, o[4 * c8 + 2 * hh + 1] * inv);
        }
        if (cq == 0 && p.lse) p.lse[((int64_t)b * p.H + h) * p.Lq + qrow] = ((m[hh] == -INFINITY ? 0.f : m[hh]) + log2f(lt)) * kLn2;
    }
}

// =============================================================================================
// backward
// =============================================================================================
struct alignas(64) AttnBwdParams {
    CUtensorMap tmQ, tmK, tmV, tmdO;   // K / V: boxes of 128 rows; Q / dO: boxes of 64 rows
    int B, H, Lq, Lkv, d;
    int nks;                 // 16-wide k-steps over d
    int col0;                // output column slice [col0, col0 + 64) of this launch
    float scale, scale_log2;
    const float* kv_bias;
    const float* lse;        // [B,H,Lq]
    const float* delta;      // [B,H,Lq]  rowsum(dO * O)
    float* dq_acc;           // [B,H,dq_ld/4,Lq,4] fp32
    int dq_ld;
    int qsplit;              // CTAs per kv tile along the query dimension
    float* dkv_acc;          // [B,H,Lkv,2,dq_ld] fp32 partial dK/dV when qsplit > 1, else nullptr
    __nv_bfloat16 *dK, *dV;
    int64_t lddk, lddv;
};

template <int NB>
struct AttnBwdCfg {
    static constexpr int KV_BYTES = NB * BOX_BYTES;       // K or V: 128 rows
    static constexpr int QBOX = 64 * 128;
    static constexpr int Q_BYTES = NB * QBOX;             // Q or dO: 64 rows
    static constexpr int STAGES = 2;
    static constexpr int DS_BYTES = 64 * 128;             // dS^T of one warpgroup: [64 kv][64 q] bf16 (the two are contiguous)
    static constexpr int SMEM_BYTES = 2 * KV_BYTES + 2 * STAGES * Q_BYTES + 2 * DS_BYTES + 256 + 1024;
};

template <int NB>
__global__ void __launch_bounds__(kAttnThreads, 1) attn_bwd_kernel(const __grid_constant__ AttnBwdParams p) {
    using Cfg = AttnBwdCfg<NB>;
    constexpr int STAGES = Cfg::STAGES;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint8_t* sK = smem;
    uint8_t* sV = sK + Cfg::KV_BYTES;
    uint8_t* sQ = sV + Cfg::KV_BYTES;                     // [STAGES]
    uint8_t* sdO = sQ + STAGES * Cfg::Q_BYTES;            // [STAGES]
    uint8_t* sDS = sdO + STAGES * Cfg::Q_BYTES;           // [2 warpgroups]
    uint64_t* bars = reinterpret_cast<uint64_t*>(sDS + 2 * Cfg::DS_BYTES);
    uint64_t* kv_full = bars;
    uint64_t* q_full = bars + 1;                          // [STAGES]
    uint64_t* q_empty = bars + 1 + STAGES;                // [STAGES]

    // Register-bound: 288 threads cap every thread at 168 registers, and S, dP, their bf16 fragments and the dV / dK / dQ accumulators
    // do not fit; ptxas spills (~0.3 KB per thread) and serializes the wgmmas (C7512).  The thread-index form of the warp index below
    // measured faster than warp_id_uniform() here (the latter spilled more).
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int kt = blockIdx.x / p.qsplit, qs = blockIdx.x % p.qsplit;
    const int h = blockIdx.y, b = blockIdx.z;
    const int nq = (p.Lq + 63) / 64;
    const int per = 2 * (((nq + 1) / 2 + p.qsplit - 1) / p.qsplit);     // whole 128-row units per split (plan_qsplit)
    const int i0 = qs * per, i1 = min(nq, i0 + per);

    if (threadIdx.x == 0) {
        mbar_init(kv_full, 1);
        for (int s = 0; s < STAGES; ++s) { mbar_init(&q_full[s], 1); mbar_init(&q_empty[s], 256); }
        fence_mbar_init();
    }
    __syncthreads();
    pdl_trigger();
    pdl_wait();

    if (warp == 8) {
        if (elect_one()) {
            mbar_arrive_expect_tx(kv_full, 2 * Cfg::KV_BYTES);
            for (int bx = 0; bx < NB; ++bx) {
                tma_load_4d(sK + bx * BOX_BYTES, &p.tmK, kv_full, bx * 64, h, kt * 128, b);
                tma_load_4d(sV + bx * BOX_BYTES, &p.tmV, kv_full, bx * 64, h, kt * 128, b);
            }
            for (int i = i0; i < i1; ++i) {
                const int st = (i - i0) % STAGES;
                mbar_wait(&q_empty[st], (((i - i0) / STAGES) & 1) ^ 1);
                mbar_arrive_expect_tx(&q_full[st], 2 * Cfg::Q_BYTES);
                for (int bx = 0; bx < NB; ++bx) {
                    tma_load_4d(sQ + st * Cfg::Q_BYTES + bx * Cfg::QBOX, &p.tmQ, &q_full[st], bx * 64, h, i * 64, b);
                    tma_load_4d(sdO + st * Cfg::Q_BYTES + bx * Cfg::QBOX, &p.tmdO, &q_full[st], bx * 64, h, i * 64, b);
                }
            }
        }
        return;
    }

    const int wg = warp >> 2;
    const int g = lane >> 2, cq = 2 * (lane & 3);
    const int r0 = (warp & 3) * 16 + g;                  // rows r0, r0 + 8 of this warpgroup's 64 kv rows
    const int kvw = kt * 128 + wg * 64;
    const int64_t bh = (int64_t)b * p.H + h;
    const float sl2 = p.scale_log2, scale = p.scale;
    const int cbox = p.col0 / 64;                        // box holding the output column slice
    float kvb[2];
    bool kv_ok[2];
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
        const int kv = kvw + r0 + 8 * hh;
        kv_ok[hh] = kv < p.Lkv;
        kvb[hh] = (p.kv_bias && kv_ok[hh]) ? p.kv_bias[(int64_t)b * p.Lkv + kv] * kLog2e : 0.f;
    }
    float dv[32], dk[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) { dv[i] = 0.f; dk[i] = 0.f; }
    const uint64_t kdesc = make_smem_desc(smem_u32(sK) + wg * 64 * 128, 16, 1024);
    const uint64_t vdesc = make_smem_desc(smem_u32(sV) + wg * 64 * 128, 16, 1024);
    // dQ: A = dS^T of all 128 kv rows read transposed, B = the 128 K rows, output columns of the slice (both MN-major)
    const uint64_t kdesc_mn = make_smem_desc(smem_u32(sK) + cbox * BOX_BYTES, BOX_BYTES, 1024);
    const uint32_t ds_base = smem_u32(sDS) + wg * Cfg::DS_BYTES;
    const uint64_t dsdesc = make_smem_desc(smem_u32(sDS), 2 * Cfg::DS_BYTES, 1024);
    mbar_wait(kv_full, 0);
    for (int i = i0; i < i1; ++i) {
        const int st = (i - i0) % STAGES;
        mbar_wait(&q_full[st], ((i - i0) / STAGES) & 1);
        const uint32_t qb = smem_u32(sQ + st * Cfg::Q_BYTES), dob = smem_u32(sdO + st * Cfg::Q_BYTES);
        const uint64_t qdesc = make_smem_desc(qb, 16, 1024), dodesc = make_smem_desc(dob, 16, 1024);
        // ---- S^T = K Q^T, dP^T = V dO^T  (rows: kv, columns: q)
        float s[32], dp[32];
        wgmma_fence();
        wgmma_ss<64, 0, 0>(s, kdesc, qdesc, 0u);
        for (int ks = 1; ks < p.nks; ++ks)
            wgmma_ss<64, 0, 0>(s, desc_adv(kdesc, kmajor_off(ks, BOX_BYTES)), desc_adv(qdesc, kmajor_off(ks, Cfg::QBOX)), 1u);
        wgmma_ss<64, 0, 0>(dp, vdesc, dodesc, 0u);
        for (int ks = 1; ks < p.nks; ++ks)
            wgmma_ss<64, 0, 0>(dp, desc_adv(vdesc, kmajor_off(ks, BOX_BYTES)), desc_adv(dodesc, kmajor_off(ks, Cfg::QBOX)), 1u);
        wgmma_commit();
        wgmma_wait<0>();
        wgmma_fence_acc(s);
        wgmma_fence_acc(dp);
        // ---- P^T, dS^T = scale * P^T (dP^T - delta) as bf16 A fragments (K = q); dS^T also to shared memory for dQ
        uint32_t pa[4][4], da[4][4];
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) {
            // per-column (query) statistics of the four columns of this k-step this thread holds
            float lq[4], dq_[4];
#pragma unroll
            for (int c = 0; c < 4; ++c) {
                const int q = i * 64 + 16 * kk + 8 * (c >> 1) + cq + (c & 1);
                const bool ok = q < p.Lq;
                lq[c] = ok ? __ldg(p.lse + bh * p.Lq + q) * kLog2e : INFINITY;   // masked query: P = exp2(-inf) = 0
                dq_[c] = ok ? __ldg(p.delta + bh * p.Lq + q) : 0.f;
            }
#pragma unroll
            for (int r = 0; r < 4; ++r) {
                const int hh = r & 1;
                const int c = 2 * (r >> 1);                     // index into lq / dq_ of the first of the two columns
                const int idx = 8 * kk + 4 * (r >> 1) + 2 * hh;
                float pv[2], dsv[2];
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    const float pe = kv_ok[hh] ? fast_exp2(s[idx + e] * sl2 + kvb[hh] - lq[c + e]) : 0.f;
                    pv[e] = pe;
                    dsv[e] = scale * pe * (dp[idx + e] - dq_[c + e]);
                }
                pa[kk][r] = pack_bf16x2(pv[0], pv[1]);
                da[kk][r] = pack_bf16x2(dsv[0], dsv[1]);
                // dS^T element (kv row, q col) of the [64 kv][64 q] MN-major SWIZZLE_128B tile
                const int row = r0 + 8 * hh, col = 16 * kk + 8 * (r >> 1) + cq;
                asm volatile("st.shared.b32 [%0], %1;" ::"r"(ds_base + sw128_offset(row, col >> 3) + (col & 7) * 2), "r"(da[kk][r]) : "memory");
            }
        }
        fence_proxy_async_smem();
        asm volatile("bar.sync 1, 256;" ::: "memory");                   // dS^T of both warpgroups in shared memory
        // ---- dV += P^T dO, dK += dS^T Q (slice columns; MN-major B); one warpgroup: dQ_i = dS K over the CTA's 128 kv rows
        const bool dq_here = ((i - i0) & 1) == wg;
        const uint64_t dodesc_mn = make_smem_desc(dob + cbox * Cfg::QBOX, Cfg::QBOX, 1024);
        const uint64_t qdesc_mn = make_smem_desc(qb + cbox * Cfg::QBOX, Cfg::QBOX, 1024);
        float dqa[32];
        wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) wgmma_rs<64, 1>(dv, pa[kk], desc_adv(dodesc_mn, kk * 128), 1u);
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) wgmma_rs<64, 1>(dk, da[kk], desc_adv(qdesc_mn, kk * 128), 1u);
        wgmma_commit();
        wgmma_wait<0>();                                 // P^T / dS^T registers free before the dQ accumulator is live
        wgmma_fence_acc(dv);
        wgmma_fence_acc(dk);
        if (dq_here) {
            wgmma_fence();
            wgmma_ss<64, 1, 1>(dqa, dsdesc, kdesc_mn, 0u);
#pragma unroll
            for (int kk = 1; kk < 8; ++kk) wgmma_ss<64, 1, 1>(dqa, desc_adv(dsdesc, kk * 128), desc_adv(kdesc_mn, kk * 128), 1u);
        }
        wgmma_commit();
        wgmma_wait<0>();
        wgmma_fence_acc(dqa);
        mbar_arrive(&q_empty[st]);
        asm volatile("bar.sync 1, 256;" ::: "memory");                   // the dS^T tiles may be overwritten by the next query tile
        if (!dq_here) continue;
        // ---- dQ of the CTA's kv rows -> fp32 accumulator [B,H,dq_ld/4,Lq,4]
#pragma unroll
        for (int hh = 0; hh < 2; ++hh) {
            const int q = i * 64 + r0 + 8 * hh;
            if (q >= p.Lq) continue;
#pragma unroll
            for (int c8 = 0; c8 < 8; ++c8) {
                const int col = p.col0 + 8 * c8 + cq;
                if (col < p.d) red_add_v2(p.dq_acc + ((bh * (p.dq_ld / 4) + col / 4) * p.Lq + q) * 4 + (col & 3), dqa[4 * c8 + 2 * hh], dqa[4 * c8 + 2 * hh + 1]);
            }
        }
    }
    // ---- dK / dV of this warpgroup's kv rows
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
        if (!kv_ok[hh]) continue;
        const int kv = kvw + r0 + 8 * hh;
#pragma unroll
        for (int c8 = 0; c8 < 8; ++c8) {
            const int col = p.col0 + 8 * c8 + cq;
            if (col >= p.d) continue;
            const float v0 = dv[4 * c8 + 2 * hh], v1 = dv[4 * c8 + 2 * hh + 1];
            const float k0 = dk[4 * c8 + 2 * hh], k1 = dk[4 * c8 + 2 * hh + 1];
            if (p.dkv_acc) {
                float* base = p.dkv_acc + ((bh * p.Lkv + kv) * 2) * p.dq_ld + col;
                red_add_v2(base, v0, v1);
                red_add_v2(base + p.dq_ld, k0, k1);
            } else {
                *reinterpret_cast<uint32_t*>(p.dV + ((int64_t)b * p.Lkv + kv) * p.lddv + (int64_t)h * p.d + col) = pack_bf16x2(v0, v1);
                *reinterpret_cast<uint32_t*>(p.dK + ((int64_t)b * p.Lkv + kv) * p.lddk + (int64_t)h * p.d + col) = pack_bf16x2(k0, k1);
            }
        }
    }
}

// delta[b,h,q] = sum_e dO*O ; also zero-fills the fp32 dQ / dK,dV accumulators (when present).  One thread per (b,q,h): the
// d elements of a head are contiguous (d % 8 == 0 -> 16-byte loads) and adjacent threads read adjacent heads of the same token
// row, so a warp streams contiguous memory.
__global__ void __launch_bounds__(256) attn_bwd_prep_kernel(const __nv_bfloat16* __restrict__ O, int64_t ldo,
                                                            const __nv_bfloat16* __restrict__ dO, int64_t lddo, int B, int H, int Lq,
                                                            int d, float* __restrict__ delta, float* __restrict__ dq_acc,
                                                            int64_t dq_n, float* __restrict__ dkv_acc, int64_t dkv_n) {
    pdl_trigger();
    pdl_wait();
    const int64_t gtid = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    const int64_t nthreads = (int64_t)gridDim.x * blockDim.x;
    if (dq_acc) {
        float4* z = reinterpret_cast<float4*>(dq_acc);
        for (int64_t i = gtid; i < dq_n / 4; i += nthreads) z[i] = make_float4(0.f, 0.f, 0.f, 0.f);
    }
    if (dkv_acc) {
        float4* z = reinterpret_cast<float4*>(dkv_acc);
        for (int64_t i = gtid; i < dkv_n / 4; i += nthreads) z[i] = make_float4(0.f, 0.f, 0.f, 0.f);
    }
    const int64_t total = (int64_t)B * Lq * H;
    if (gtid >= total) return;
    const int h = (int)(gtid % H);
    const int64_t bq = gtid / H;
    const int q = (int)(bq % Lq);
    const int b = (int)(bq / Lq);
    const uint4* o = reinterpret_cast<const uint4*>(O + bq * ldo + (int64_t)h * d);
    const uint4* g = reinterpret_cast<const uint4*>(dO + bq * lddo + (int64_t)h * d);
    float acc = 0.f;
    for (int e = 0; e < d / 8; ++e) {
        const uint4 a = o[e], c = g[e];
        float2 x, y;
        x = unpack_bf16x2(a.x); y = unpack_bf16x2(c.x); acc += x.x * y.x + x.y * y.y;
        x = unpack_bf16x2(a.y); y = unpack_bf16x2(c.y); acc += x.x * y.x + x.y * y.y;
        x = unpack_bf16x2(a.z); y = unpack_bf16x2(c.z); acc += x.x * y.x + x.y * y.y;
        x = unpack_bf16x2(a.w); y = unpack_bf16x2(c.w); acc += x.x * y.x + x.y * y.y;
    }
    delta[((int64_t)b * H + h) * Lq + q] = acc;
}

// dQ bf16 [B, Lq, lddq] <- fp32 accumulator [B,H,dq_ld/4,Lq,4]
__global__ void attn_bwd_post_kernel(const float* __restrict__ dq_acc, int dq_ld, int B, int H, int Lq, int d,
                                     __nv_bfloat16* __restrict__ dQ, int64_t lddq) {
    pdl_trigger();
    pdl_wait();
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;   // one thread per 4 elements
    const int d4 = d / 4;
    const int64_t total = (int64_t)B * Lq * H * d4;
    if (i >= total) return;
    const int e = (int)(i % d4) * 4;
    const int64_t r = i / d4;
    const int h = (int)(r % H);
    const int64_t bq = r / H;
    const int q = (int)(bq % Lq);
    const int b = (int)(bq / Lq);
    const float4 v = *reinterpret_cast<const float4*>(dq_acc + ((((int64_t)b * H + h) * (dq_ld / 4) + e / 4) * Lq + q) * 4);   // [B,H,d/4,Lq,4]
    uint2 o;
    o.x = pack_bf16x2(v.x, v.y);
    o.y = pack_bf16x2(v.z, v.w);
    *reinterpret_cast<uint2*>(dQ + bq * lddq + (int64_t)h * d + e) = o;
}

// dK / dV bf16 [B, Lkv, ld] <- fp32 partial sums [B,H,Lkv,2,dq_ld]  (only when the query range was split)
__global__ void attn_bwd_post_kv_kernel(const float* __restrict__ acc, int dq_ld, int B, int H, int Lkv, int d,
                                        __nv_bfloat16* __restrict__ dK, int64_t lddk, __nv_bfloat16* __restrict__ dV, int64_t lddv) {
    pdl_trigger();
    pdl_wait();
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    const int d4 = d / 4;
    const int64_t total = (int64_t)B * Lkv * H * 2 * d4;
    if (i >= total) return;
    const int e = (int)(i % d4) * 4;
    int64_t r = i / d4;
    const int which = (int)(r % 2); r /= 2;
    const int h = (int)(r % H);
    const int64_t bk = r / H;
    const int kv = (int)(bk % Lkv);
    const int b = (int)(bk / Lkv);
    const float4 v = *reinterpret_cast<const float4*>(acc + ((((int64_t)b * H + h) * Lkv + kv) * 2 + which) * dq_ld + e);
    uint2 o;
    o.x = pack_bf16x2(v.x, v.y);
    o.y = pack_bf16x2(v.z, v.w);
    __nv_bfloat16* dst = which ? dK : dV;
    const int64_t ld = which ? lddk : lddv;
    *reinterpret_cast<uint2*>(dst + bk * ld + (int64_t)h * d + e) = o;
}

static int make_head_map(CUtensorMap* m, const void* base, int64_t ld, int64_t B, int64_t H, int64_t L, int64_t d, uint32_t rows) {
    uint64_t dims[4] = {(uint64_t)d, (uint64_t)H, (uint64_t)L, (uint64_t)B};
    uint64_t strides[3] = {(uint64_t)d * 2, (uint64_t)ld * 2, (uint64_t)L * ld * 2};
    uint32_t box[4] = {64, 1, rows, 1};
    return make_tmap_nd(m, base, 4, dims, strides, box);
}

static int check_common(int64_t B, int64_t H, int64_t Lq, int64_t Lkv, int64_t d) {
    if (B <= 0 || H <= 0 || Lq <= 0 || Lkv <= 0) return set_error(HCP_ERR_INVALID, "attention: empty problem");
    if (d % 8 != 0 || d < 8 || d > 192) return set_error(HCP_ERR_INVALID, "attention: head dim must be a multiple of 8 in [8,192]");
    return HCP_OK;
}

template <int NB, int KVT>
static int launch_attn_fwd(const AttnFwdParams& p, dim3 grid, cudaStream_t stream) {
    using Cfg = AttnFwdCfg<NB, KVT>;
    static bool configured = false;
    if (!configured) {
        cudaError_t e = cudaFuncSetAttribute(attn_fwd_kernel<NB, KVT>, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM_BYTES);
        if (e != cudaSuccess) return set_cuda_error(e, "cudaFuncSetAttribute(attn_fwd)");
        configured = true;
    }
    launch_k(attn_fwd_kernel<NB, KVT>, grid, dim3(kAttnThreads), Cfg::SMEM_BYTES, stream, p);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return set_cuda_error(e, "attn_fwd launch");
    return HCP_OK;
}

template <int NB>
static int launch_attn_bwd(const AttnBwdParams& p, dim3 grid, cudaStream_t stream) {
    using Cfg = AttnBwdCfg<NB>;
    static bool configured = false;
    if (!configured) {
        cudaError_t e = cudaFuncSetAttribute(attn_bwd_kernel<NB>, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM_BYTES);
        if (e != cudaSuccess) return set_cuda_error(e, "cudaFuncSetAttribute(attn_bwd)");
        configured = true;
    }
    launch_k(attn_bwd_kernel<NB>, grid, dim3(kAttnThreads), Cfg::SMEM_BYTES, stream, p);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return set_cuda_error(e, "attn_bwd launch");
    return HCP_OK;
}

}  // namespace hcp

using namespace hcp;

extern "C" int hcp_attn_fwd_bf16(const hcp_attn_args* a, hcp_stream_t stream_) {
    if (!a || !a->q || !a->k || !a->v || !a->o) return set_error(HCP_ERR_INVALID, "attn_fwd: null pointer");
    int rc = check_common(a->B, a->H, a->Lq, a->Lkv, a->d);
    if (rc) return rc;
    const int nb = (int)((a->d + 63) / 64);
    // kv tile: 128 rows, 64 when the O accumulator of d > 128 leaves no registers for a 128-column S tile
    const uint32_t kvt = nb == 3 ? 64 : 128;
    AttnFwdParams p;
    memset(&p, 0, sizeof(p));
    if ((rc = make_head_map(&p.tmQ, a->q, a->ldq, a->B, a->H, a->Lq, a->d, 128))) return rc;
    if ((rc = make_head_map(&p.tmK, a->k, a->ldk, a->B, a->H, a->Lkv, a->d, kvt))) return rc;
    if ((rc = make_head_map(&p.tmV, a->v, a->ldv, a->B, a->H, a->Lkv, a->d, kvt))) return rc;
    p.B = (int)a->B; p.H = (int)a->H; p.Lq = (int)a->Lq; p.Lkv = (int)a->Lkv; p.d = (int)a->d;
    p.nks = (int)((a->d + 15) / 16);
    p.scale_log2 = a->scale * kLog2e;
    p.kv_bias = a->kv_bias;
    p.O = (__nv_bfloat16*)a->o; p.ldo = a->ldo;
    p.lse = a->lse;
    const dim3 grid((unsigned)((a->Lq + 127) / 128), (unsigned)a->H, (unsigned)a->B);
    cudaStream_t stream = (cudaStream_t)stream_;
    if (nb == 1) return launch_attn_fwd<1, 128>(p, grid, stream);
    if (nb == 2) return launch_attn_fwd<2, 128>(p, grid, stream);
    return launch_attn_fwd<3, 64>(p, grid, stream);
}

// CTAs per kv tile along the query dimension: when the (kv tile, head, image) CTAs fill less than one wave, the query range is split
// so that about two CTAs per SM run; the partial dK / dV sums then go through an fp32 buffer
// (in units of 128 query rows, i.e. two of the kernel's query tiles: two splits -- an order-independent fp32 sum -- cover Lq <= 256)
static int plan_qsplit(int64_t B, int64_t H, int64_t Lq, int64_t Lkv) {
    const int64_t base = ((Lkv + 127) / 128) * H * B;
    const int64_t nq = (Lq + 127) / 128;
    const int64_t sms = num_sms();
    if (base >= sms * 4 / 5 || nq < 2) return 1;
    int64_t qs = (2 * sms + base - 1) / base;
    if (qs > nq) qs = nq;
    const int64_t per = (nq + qs - 1) / qs;
    return (int)((nq + per - 1) / per);                 // every split owns at least one 128-row unit
}

extern "C" size_t hcp_attn_bwd_workspace_bytes(int64_t B, int64_t H, int64_t Lq, int64_t Lkv, int64_t d) {
    const int64_t dq_ld = (d + 3) / 4 * 4;
    size_t n = (size_t)((B * H * Lq + 3) / 4 * 4) + (size_t)(B * H * Lq * dq_ld);   // delta (padded to 16 bytes) + dQ accumulator
    if (plan_qsplit(B, H, Lq, Lkv) > 1) n += (size_t)(B * H * Lkv * 2 * dq_ld);
    return n * sizeof(float);
}

extern "C" int hcp_attn_bwd_bf16(const hcp_attn_bwd_args* a, hcp_stream_t stream_) {
    if (!a || !a->q || !a->k || !a->v || !a->o || !a->dout || !a->lse || !a->dq || !a->dk || !a->dv || !a->workspace)
        return set_error(HCP_ERR_INVALID, "attn_bwd: null pointer");
    int rc = check_common(a->B, a->H, a->Lq, a->Lkv, a->d);
    if (rc) return rc;
    if (a->workspace_bytes < hcp_attn_bwd_workspace_bytes(a->B, a->H, a->Lq, a->Lkv, a->d))
        return set_error(HCP_ERR_INVALID, "attn_bwd: workspace too small");
    if ((a->ldo % 8) != 0 || (a->lddo % 8) != 0 || (a->lddq % 8) != 0) return set_error(HCP_ERR_INVALID, "attn_bwd: leading dimensions must be multiples of 8");
    cudaStream_t stream = (cudaStream_t)stream_;
    const int dq_ld = (int)((a->d + 3) / 4 * 4);
    float* delta = a->workspace;
    float* dq_acc = a->workspace + (a->B * a->H * a->Lq + 3) / 4 * 4;
    const int qsplit = plan_qsplit(a->B, a->H, a->Lq, a->Lkv);
    const int64_t dkv_n = qsplit > 1 ? a->B * a->H * a->Lkv * 2 * dq_ld : 0;
    float* dkv_acc = qsplit > 1 ? dq_acc + a->B * a->H * a->Lq * dq_ld : nullptr;
    {
        const int64_t total = a->B * a->Lq * a->H;
        const int threads = 256;
        const int64_t blocks = (total + threads - 1) / threads;
        launch_k(attn_bwd_prep_kernel, dim3((unsigned)blocks), dim3(threads), 0, stream, (const __nv_bfloat16*)a->o, a->ldo,
                 (const __nv_bfloat16*)a->dout, a->lddo, (int)a->B, (int)a->H, (int)a->Lq, (int)a->d, delta,
                 dq_acc, (int64_t)(a->B * a->H * a->Lq * dq_ld), dkv_acc, dkv_n);
    }
    AttnBwdParams p;
    memset(&p, 0, sizeof(p));
    if ((rc = make_head_map(&p.tmQ, a->q, a->ldq, a->B, a->H, a->Lq, a->d, 64))) return rc;
    if ((rc = make_head_map(&p.tmK, a->k, a->ldk, a->B, a->H, a->Lkv, a->d, 128))) return rc;
    if ((rc = make_head_map(&p.tmV, a->v, a->ldv, a->B, a->H, a->Lkv, a->d, 128))) return rc;
    if ((rc = make_head_map(&p.tmdO, a->dout, a->lddo, a->B, a->H, a->Lq, a->d, 64))) return rc;
    p.B = (int)a->B; p.H = (int)a->H; p.Lq = (int)a->Lq; p.Lkv = (int)a->Lkv; p.d = (int)a->d;
    p.nks = (int)((a->d + 15) / 16);
    p.scale = a->scale;
    p.scale_log2 = a->scale * kLog2e;
    p.kv_bias = a->kv_bias;
    p.lse = a->lse;
    p.delta = delta;
    p.dq_acc = dq_acc;
    p.dq_ld = dq_ld;
    p.qsplit = qsplit;
    p.dkv_acc = dkv_acc;
    p.dK = (__nv_bfloat16*)a->dk; p.lddk = a->lddk;
    p.dV = (__nv_bfloat16*)a->dv; p.lddv = a->lddv;
    const int nb = (int)((a->d + 63) / 64);
    const dim3 grid((unsigned)(((a->Lkv + 127) / 128) * qsplit), (unsigned)a->H, (unsigned)a->B);
    // output column slices of 64 (one box): dK / dV / dQ accumulators of a slice stay in registers; S and dP are recomputed per slice
    for (int col0 = 0; col0 < a->d; col0 += 64) {
        p.col0 = col0;
        rc = nb == 1 ? launch_attn_bwd<1>(p, grid, stream) : nb == 2 ? launch_attn_bwd<2>(p, grid, stream) : launch_attn_bwd<3>(p, grid, stream);
        if (rc) return rc;
    }
    {
        const int64_t n = a->B * a->Lq * a->H * (a->d / 4);
        launch_k(attn_bwd_post_kernel, dim3((unsigned)((n + 255) / 256)), dim3(256), 0, stream, dq_acc, dq_ld, (int)a->B, (int)a->H, (int)a->Lq,
                 (int)a->d, (__nv_bfloat16*)a->dq, a->lddq);
    }
    if (qsplit > 1) {
        const int64_t n = a->B * a->Lkv * a->H * 2 * (a->d / 4);
        launch_k(attn_bwd_post_kv_kernel, dim3((unsigned)((n + 255) / 256)), dim3(256), 0, stream, dkv_acc, dq_ld, (int)a->B, (int)a->H, (int)a->Lkv, (int)a->d,
                                                                                (__nv_bfloat16*)a->dk, a->lddk, (__nv_bfloat16*)a->dv, a->lddv);
    }
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return set_cuda_error(e, "attn_bwd post launch");
    return HCP_OK;
}
