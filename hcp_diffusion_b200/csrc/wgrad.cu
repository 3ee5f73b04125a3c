// SPDX-License-Identifier: Apache-2.0
// Weight gradients of the base model (full fine-tune, reference `unet:` config items: hcpdiff/utils/cfg_net_tools.py:96-106,
// cfgs/train/examples/DreamBooth.yaml:6-10) for sm_90a:
//   * wgrad_tc_kernel<SN>: dW = dY^T . X on the tensor cores (wgmma TN GEMM, both operands read MN-major straight from the row-major
//     activations through TMA; the X operand of a 3x3 convolution is the shifted NHWC box of the forward kernel), fp32 atomics into
//     the flat gradient buffer;
//   * column sums (bias gradients, per-image time-embedding gradients), GroupNorm / LayerNorm affine gradients;
//   * the 4-channel boundary convolutions' weight gradients, the small fp32 linears of the time-embedding path (M = batch rows);
//   * the per-step fp32 -> bf16 repack of the trained weights into the operand layouts of the forward / dgrad kernels.
// Replaces autograd of nn.Linear / nn.Conv2d / nn.GroupNorm / nn.LayerNorm parameters in the reference's full fine-tune.
#include "common.cuh"
#include "host_util.h"
#include "../../include/hcp_b200.h"

namespace hcp {

#define LAUNCH_CHECK(what)                                              \
    do {                                                                \
        cudaError_t e_ = cudaGetLastError();                            \
        if (e_ != cudaSuccess) return set_cuda_error(e_, what);         \
    } while (0)

// =============================================================================================
// D[j, n] += scale * sum_m S[m, j0 + j] * X[m, n0 + n]        (reduction over the M token / pixel rows)
//   linear:  dW[o, k] : S = dY [M, N], X = x [M, K]
//   conv3x3: dW[co, ci, kh, kw] : S = dY, X = x shifted by the tap (4-D / 5-D NHWC box, zero padding by TMA)
//   LoRA:    dW_down[j, k] = sum_m U[m, c0+j] x[m, k]  (S = U = dY . (alpha B), X = x, or the shifted box of a Conv2d LoRA)
//            dW_up[o, j]   = alpha * sum_m dY[m, o0+o] T[m, c0+j]  (S = T = x . A^T, X = dY)
// Both operands are read straight from their row-major [M, *] tensors as MN-major wgmma operands (TMA boxes of 64 columns x
// 128 rows), so no transpose ever exists.  One CTA owns 128 columns of X and SN columns of S over a slice of the rows; MMA warpgroup
// g computes X columns [64g, 64g+64) (wgmma M = 64, N = SN, K = 16 rows per instruction) and reduces its 64 x SN fp32 block into
// the flat gradient buffer with atomics: dense, dst[j * ld_j + n * ld_n], or (kTable, SN = 64) through a table of up to 8 LoRA
// blocks, each a rank range of the 64 S columns and an X column range with its own destination layout and scale.
// =============================================================================================
constexpr int kWgThreads = 288;   // warps 0-7: two MMA warpgroups, warp 8: TMA
constexpr int LG_MAX_BLOCKS = 8;

struct LGBlock {
    int32_t n_lo, n_hi, c0, rank, transpose_out, dst_ld;
    int32_t n_stride;        // element stride of the X-column index in the destination (1; 9 for the taps of a 3x3 W_down)
    float scale;
    float* dst;
};
struct LGTable {
    int32_t nblocks;
    LGBlock blk[LG_MAX_BLOCKS];
};
// X operand = shifted im2col box of a 3x3 convolution: the same boxes as the forward convolution's A operand
struct WgConv {
    int32_t rank;            // 0: plain [M, ldx] matrix; 4 / 5: rank of the NHWC tensor map
    ConvBox box;
    ConvTap tap;
};
struct WgProblem {
    CUtensorMap tmX, tmS;
    int32_t n_begin, n_end;          // X columns [n_begin, n_end)
    int32_t j_cols;                  // valid S columns (dense epilogue)
    int32_t n_tiles, j_tiles, splits, tiles_per_cta, ctas;
    // dense epilogue
    int64_t ld_j, ld_n;
    float scale;
    float* dst;
    // table epilogue
    LGTable tab;
};
struct alignas(64) WgradParams {
    WgProblem prob[2];               // up to two independent problems per launch (dW_down and dW_up of one LoRA group)
    int32_t M, nprob;
    WgConv conv;                     // X geometry of the launch (a convolution launch carries one problem)
};

template <int SN>
struct WgCfg {
    static constexpr int X_BYTES = 2 * 128 * 128;             // two 64-column boxes of 128 rows
    static constexpr int S_BYTES = (SN / 64) * 128 * 128;
    static constexpr int STAGE_BYTES = X_BYTES + S_BYTES;
    static constexpr int STAGES = 3;
    static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + 256 + 1024;
};

template <int SN, bool kTable>
__global__ void __launch_bounds__(kWgThreads, 1) wgrad_tc_kernel(const __grid_constant__ WgradParams p) {
    static_assert(!kTable || SN == 64, "the block table covers one 64-column slab of S");
    using Cfg = WgCfg<SN>;
    constexpr int STAGES = Cfg::STAGES;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + STAGES * Cfg::STAGE_BYTES);
    uint64_t* empty_bar = full_bar + STAGES;
    const int warp = warp_id_uniform(), lane = threadIdx.x & 31;
    // flat grid over (problem, row split, j tile, n tile): n fastest so that concurrent CTAs share the S tile in L2.  Only the LoRA
    // launches carry two problems; the dense variant keeps problem 0 a compile-time choice (90 instead of 94 registers at SN = 128).
    int bid = blockIdx.x, z = 0;
    if (kTable && p.nprob == 2 && bid >= p.prob[0].ctas) { bid -= p.prob[0].ctas; z = 1; }
    const WgProblem& q = z ? p.prob[1] : p.prob[0];
    const int nt = bid % q.n_tiles, jt = (bid / q.n_tiles) % q.j_tiles, sp = bid / (q.n_tiles * q.j_tiles);
    const int ncol0 = q.n_begin + nt * 128, jcol0 = jt * SN;
    const int total_tiles = (p.M + 127) / 128;
    const int t0 = sp * q.tiles_per_cta;
    const int t1 = min(total_tiles, t0 + q.tiles_per_cta);

    if (threadIdx.x == 0) {
        for (int s = 0; s < STAGES; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], 256); }
        fence_mbar_init();
        tma_prefetch_desc(&q.tmX);
        tma_prefetch_desc(&q.tmS);
    }
    __syncthreads();
    pdl_trigger();
    pdl_wait();

    if (warp == 8) {
        if (elect_one()) {
            int stage = 0; uint32_t phase = 0;
            for (int t = t0; t < t1; ++t) {
                mbar_wait(&empty_bar[stage], phase ^ 1);
                mbar_arrive_expect_tx(&full_bar[stage], Cfg::STAGE_BYTES);
                uint8_t* base = smem + stage * Cfg::STAGE_BYTES;
                if (p.conv.rank == 0) {
                    tma_load_2d(base, &q.tmX, &full_bar[stage], ncol0, t * 128);
                    tma_load_2d(base + 128 * 128, &q.tmX, &full_bar[stage], ncol0 + 64, t * 128);
                } else {
                    const ConvBox& bx = p.conv.box;
                    const ConvTap& tp = p.conv.tap;
                    int img0, h0 = 0, w0 = 0;
                    if (bx.bn == 1) {
                        const int per_img = bx.tiles_w * bx.tiles_h, r = t % per_img;
                        img0 = t / per_img;
                        h0 = (r / bx.tiles_w) * bx.bh;
                        w0 = (r % bx.tiles_w) * bx.bw;
                    } else {
                        img0 = t * bx.bn;
                    }
                    for (int hf = 0; hf < 2; ++hf) {
                        const int c = tp.c0_off + ncol0 + hf * 64;
                        if (p.conv.rank == 4) tma_load_4d(base + hf * 128 * 128, &q.tmX, &full_bar[stage], c, w0 + tp.dw, h0 + tp.dh, img0);
                        else tma_load_5d(base + hf * 128 * 128, &q.tmX, &full_bar[stage], c, w0 + tp.dw, tp.c2, h0 + tp.dh, img0);
                    }
                }
#pragma unroll
                for (int s = 0; s < SN / 64; ++s)
                    tma_load_2d(base + Cfg::X_BYTES + s * 128 * 128, &q.tmS, &full_bar[stage], jcol0 + s * 64, t * 128);
                if (++stage == STAGES) { stage = 0; phase ^= 1; }
            }
        }
        return;
    }
    // The table epilogue walks `q.tab.blk[b]` with run-time z and b (dynamically indexed constant-bank loads): the MMA threads copy
    // the table to shared memory first.
    __shared__ LGTable stab;
    if constexpr (kTable) {
        const uint32_t* src = reinterpret_cast<const uint32_t*>(&q.tab);
        uint32_t* dst = reinterpret_cast<uint32_t*>(&stab);
        for (int i = threadIdx.x; i < (int)(sizeof(LGTable) / 4); i += 256) dst[i] = src[i];
        asm volatile("bar.sync 1, 256;" ::: "memory");
    }
    const int wg = warp >> 2;
    float acc[SN / 2];
#pragma unroll
    for (int i = 0; i < SN / 2; ++i) acc[i] = 0.f;
    int stage = 0; uint32_t phase = 0;
    for (int t = t0; t < t1; ++t) {
        mbar_wait(&full_bar[stage], phase);
        const uint32_t xb = smem_u32(smem + stage * Cfg::STAGE_BYTES) + wg * 128 * 128;   // this warpgroup's 64 X columns
        const uint32_t sb = smem_u32(smem + stage * Cfg::STAGE_BYTES) + Cfg::X_BYTES;
        wgmma_fence();
#pragma unroll
        for (int ks = 0; ks < 8; ++ks)       // 16 rows per k-step = 2048 B inside each 64-column box
            // MN-major SWIZZLE_128B: LBO = distance between 64-wide MN chunks (one box = 16 KB), SBO = 8 k rows = 1024 B
            wgmma_ss<SN, 1, 1>(acc, make_smem_desc(xb + ks * 2048, 128 * 128, 1024), make_smem_desc(sb + ks * 2048, 128 * 128, 1024), 1u);
        wgmma_commit();
        wgmma_wait<0>();
        mbar_arrive(&empty_bar[stage]);
        if (++stage == STAGES) { stage = 0; phase ^= 1; }
    }
    wgmma_fence_acc(acc);
    if (t1 <= t0) return;
    const int n_row = ncol0 + wg * 64 + (warp & 3) * 16 + (lane >> 2);
    if constexpr (kTable) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int n = n_row + 8 * h;                                     // column of X
            if (n >= q.n_end) continue;
            for (int b = 0; b < stab.nblocks; ++b) {
                const LGBlock& k = stab.blk[b];
                if (n < k.n_lo || n >= k.n_hi) continue;
#pragma unroll
                for (int i = 0; i < 16; ++i) {
                    const int jj = 8 * (i >> 1) + 2 * (lane & 3) + (i & 1);   // column of S
                    const int j = jj - k.c0;
                    if (j >= 0 && j < k.rank) {
                        const float val = acc[4 * (i >> 1) + 2 * h + (i & 1)] * k.scale;
                        float* dst = k.transpose_out ? k.dst + (int64_t)(n - k.n_lo) * k.dst_ld + j
                                                     : k.dst + (int64_t)j * k.dst_ld + (int64_t)(n - k.n_lo) * k.n_stride;
                        atomicAdd(dst, val);
                    }
                }
            }
        }
    } else {
        const float scale = q.scale;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int n = n_row + 8 * h;                                     // column of X
            if (n >= q.n_end) continue;
            float* dcol = q.dst + (int64_t)n * q.ld_n;
#pragma unroll
            for (int i = 0; i < SN / 4; ++i) {
                const int j = jcol0 + 8 * (i >> 1) + 2 * (lane & 3) + (i & 1);      // column of S
                if (j < q.j_cols) atomicAdd(dcol + (int64_t)j * q.ld_j, acc[4 * (i >> 1) + 2 * h + (i & 1)] * scale);
            }
        }
    }
}

// ---------------------------------------------------------------------------------------------
// out[g, c] += scale * sum_{r in group g} x[r, c]      x bf16 [M, ld], groups of rows_per_group rows (bias gradient: one group;
// time-embedding gradient of a resnet: one group per image)
// ---------------------------------------------------------------------------------------------
// block = 8 column vectors (8 bf16 = 16 bytes each: a 64-column slab) x 32 row lanes; four rows in flight per thread
__device__ __forceinline__ void unpack8f(const uint4& u, float (&f)[8]) {
    float2 t;
    t = unpack_bf16x2(u.x); f[0] = t.x; f[1] = t.y;
    t = unpack_bf16x2(u.y); f[2] = t.x; f[3] = t.y;
    t = unpack_bf16x2(u.z); f[4] = t.x; f[5] = t.y;
    t = unpack_bf16x2(u.w); f[6] = t.x; f[7] = t.y;
}
__global__ void __launch_bounds__(256) colsum_bf16_kernel(const __nv_bfloat16* __restrict__ x, int64_t ld, int64_t M, int N, int64_t rows_per_group,
                                                          int chunk, float scale, float* __restrict__ out, int64_t ldo) {
    pdl_trigger();
    pdl_wait();
    const int vx = threadIdx.x & 7, ry = threadIdx.x >> 3;
    const int c = blockIdx.x * 64 + vx * 8;
    const int64_t r0 = (int64_t)blockIdx.y * chunk;
    const int64_t r1 = min(M, r0 + chunk);
    __shared__ float part[32][65];
    float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    if (c < N) {
        // a chunk never straddles a group boundary (host picks chunk | rows_per_group)
        for (int64_t r = r0 + ry; r < r1; r += 128) {
            uint4 u[4];
#pragma unroll
            for (int j = 0; j < 4; ++j) u[j] = (r + 32 * j < r1) ? *reinterpret_cast<const uint4*>(x + (r + 32 * j) * ld + c) : make_uint4(0u, 0u, 0u, 0u);
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                float f[8];
                unpack8f(u[j], f);
#pragma unroll
                for (int e = 0; e < 8; ++e) acc[e] += f[e];
            }
        }
    }
#pragma unroll
    for (int e = 0; e < 8; ++e) part[ry][vx * 8 + e] = acc[e];
    __syncthreads();
    if (threadIdx.x < 64 && blockIdx.x * 64 + (int)threadIdx.x < N) {
        float sum = 0.f;
#pragma unroll 8
        for (int i = 0; i < 32; ++i) sum += part[i][threadIdx.x];
        atomicAdd(out + (r0 / rows_per_group) * ldo + blockIdx.x * 64 + threadIdx.x, sum * scale);
    }
}

// ---------------------------------------------------------------------------------------------
// GroupNorm / LayerNorm affine gradients:  dgamma[c] += sum dz * xhat,  dbeta[c] += sum dz,
//   xhat = (x - mean) * rstd,  dz = dy (no activation)  or  dy * silu'(gamma xhat + beta)
// x = [x1 | x2] concatenated along channels (GroupNorm of the up blocks); stats fp32 [rows_or_groups, 2] = (mean, rstd)
// Same block shape as the column sums: 8 vectors of 8 channels x 32 row lanes, two rows in flight per thread.  A GroupNorm chunk lies
// inside one image (host: chunk | rows_per_image), so the statistics of a thread's eight channels are loop constants.
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) norm_affine_grad_kernel(const __nv_bfloat16* __restrict__ x1, const __nv_bfloat16* __restrict__ x2, int C1, int C2,
                                                               const __nv_bfloat16* __restrict__ dy, const float* __restrict__ stats,
                                                               const float* __restrict__ gamma, const float* __restrict__ beta, int64_t rows,
                                                               int64_t rows_per_image, int ch_per_group, int groups, int silu, int chunk,
                                                               float* __restrict__ dgamma, float* __restrict__ dbeta) {
    pdl_trigger();
    pdl_wait();
    const int C = C1 + C2;
    const int vx = threadIdx.x & 7, ry = threadIdx.x >> 3;
    const int c = blockIdx.x * 64 + vx * 8;
    const int64_t r0 = (int64_t)blockIdx.y * chunk, r1 = min(rows, r0 + chunk);
    __shared__ float part[32][2 * 64 + 1];
    float ag[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f}, ab[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    if (c < C) {
        float g[8], bt[8], mean[8], rstd[8];
#pragma unroll
        for (int e = 0; e < 8; ++e) {
            const int ce = min(c + e, C - 1);
            g[e] = gamma[ce]; bt[e] = beta[ce];
            mean[e] = 0.f; rstd[e] = 0.f;
            if (groups > 0) {
                const int64_t si = ((r0 / rows_per_image) * groups + ce / ch_per_group) * 2;
                mean[e] = stats[si]; rstd[e] = stats[si + 1];
            }
        }
        const bool first = c < C1;
        const __nv_bfloat16* xb = first ? x1 + c : x2 + (c - C1);
        const int64_t xld = first ? C1 : C2;
        for (int64_t r = r0 + ry; r < r1; r += 64) {
            uint4 ux[2], ud[2];
            float lm[2] = {0.f, 0.f}, lr[2] = {0.f, 0.f};
#pragma unroll
            for (int j = 0; j < 2; ++j) {
                const int64_t rr = r + 32 * j;
                ux[j] = ud[j] = make_uint4(0u, 0u, 0u, 0u);
                if (rr < r1) {
                    ux[j] = *reinterpret_cast<const uint4*>(xb + rr * xld);
                    ud[j] = *reinterpret_cast<const uint4*>(dy + rr * C + c);
                    if (groups == 0) { lm[j] = stats[rr * 2]; lr[j] = stats[rr * 2 + 1]; }
                }
            }
#pragma unroll
            for (int j = 0; j < 2; ++j) {
                float xv[8], dv[8];
                unpack8f(ux[j], xv);
                unpack8f(ud[j], dv);             // rows past the chunk: dv = 0 -> no contribution
#pragma unroll
                for (int e = 0; e < 8; ++e) {
                    const float h = (groups > 0) ? (xv[e] - mean[e]) * rstd[e] : (xv[e] - lm[j]) * lr[j];
                    float d = dv[e];
                    if (silu) {
                        const float z = g[e] * h + bt[e];
                        const float sg = 1.f / (1.f + __expf(-z));
                        d *= sg * (1.f + z * (1.f - sg));
                    }
                    ag[e] += d * h;
                    ab[e] += d;
                }
            }
        }
    }
#pragma unroll
    for (int e = 0; e < 8; ++e) { part[ry][vx * 8 + e] = ag[e]; part[ry][64 + vx * 8 + e] = ab[e]; }
    __syncthreads();
    if (threadIdx.x < 128) {
        const int which = threadIdx.x >> 6, cl = threadIdx.x & 63;
        const int cc = blockIdx.x * 64 + cl;
        if (cc < C) {
            float sum = 0.f;
#pragma unroll 8
            for (int i = 0; i < 32; ++i) sum += part[i][which * 64 + cl];
            atomicAdd((which ? dbeta : dgamma) + cc, sum);
        }
    }
}

// ---------------------------------------------------------------------------------------------
// small fp32 linears of the time-embedding path (M = batch rows <= 64): y = x W^T + b is hcp_skinny_linear; here its backward
//   dx[m, k] = sum_n dy[m, n] W[n, k]          (W bf16 [N, K]: the operand the forward used)
//   dW[n, k] += sum_m dy[m, n] x[m, k],  db[n] += sum_m dy[m, n]      (fp32 master gradients)
// and SiLU forward / backward on fp32 vectors.
// ---------------------------------------------------------------------------------------------
// dx: every thread owns one k and a slice of the n range for up to 16 rows at a time: the weight is streamed ONCE (the first version
// re-read all of W per row: 840 MB for the 22 stacked time_emb_proj layers at batch 16), partial sums leave through atomics
constexpr int SLDX_ROWS = 16;
__global__ void __launch_bounds__(128) small_linear_dx_kernel(const float* __restrict__ dy, int64_t ldy, const __nv_bfloat16* __restrict__ w, int M, int N,
                                                              int K, int n_chunk, float* __restrict__ dx) {
    pdl_trigger();
    pdl_wait();
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    const int n0 = blockIdx.y * n_chunk, n1 = min(N, n0 + n_chunk);
    const int m0 = blockIdx.z * SLDX_ROWS;
    const int rows = min(SLDX_ROWS, M - m0);
    __shared__ float sdy[SLDX_ROWS][128];
    float acc[SLDX_ROWS];
#pragma unroll
    for (int r = 0; r < SLDX_ROWS; ++r) acc[r] = 0.f;
    for (int nb = n0; nb < n1; nb += 128) {
        __syncthreads();
        for (int i = threadIdx.x; i < SLDX_ROWS * 128; i += blockDim.x) {
            const int r = i >> 7, n = nb + (i & 127);
            sdy[r][i & 127] = (r < rows && n < n1) ? dy[(int64_t)(m0 + r) * ldy + n] : 0.f;
        }
        __syncthreads();
        if (k < K) {
            const int lim = min(128, n1 - nb);
            for (int j = 0; j < lim; ++j) {
                const float wv = __bfloat162float(w[(int64_t)(nb + j) * K + k]);     // coalesced over k
#pragma unroll
                for (int r = 0; r < SLDX_ROWS; ++r) acc[r] = fmaf(sdy[r][j], wv, acc[r]);
            }
        }
    }
    if (k < K)
        for (int r = 0; r < rows; ++r) atomicAdd(dx + (int64_t)(m0 + r) * K + k, acc[r]);
}
__global__ void small_linear_dw_kernel(const float* __restrict__ dy, int64_t ldy, const float* __restrict__ x, int M, int N, int K,
                                       float* __restrict__ dw, float* __restrict__ db) {
    pdl_trigger();
    pdl_wait();
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    const int n = blockIdx.y;
    if (k >= K) return;
    float acc = 0.f, bsum = 0.f;
    for (int m = 0; m < M; ++m) {
        const float d = dy[(int64_t)m * ldy + n];
        acc += d * x[(int64_t)m * K + k];
        bsum += d;
    }
    dw[(int64_t)n * K + k] += acc;            // one thread per element: no atomics needed (gradient ACCUMULATES across micro-steps)
    if (db && k == 0) db[n] += bsum;
}
__global__ void silu_f32_kernel(const float* __restrict__ x, const float* __restrict__ dy, int64_t n, float* __restrict__ out) {
    pdl_trigger();
    pdl_wait();
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float z = x[i], s = 1.f / (1.f + __expf(-z));
    out[i] = dy ? dy[i] * s * (1.f + z * (1.f - s)) : z * s;
}

// ---------------------------------------------------------------------------------------------
// boundary convolutions (4 latent channels): weight gradients in the nn.Conv2d layout [Cout, Cin, 3, 3]
//   conv_in : dW[co, ci, kh, kw] += sum_{b,y,x} dh[b, y, x, co] * lat[b, ci, y+kh-1, x+kw-1]     dh bf16 NHWC, lat fp32 NCHW
//   conv_out: dW[co, ci, kh, kw] += sum_{b,y,x} dy[b, co, y, x] * act[b, y+kh-1, x+kw-1, ci]     dy fp32 NCHW, act bf16 NHWC
// block = one (small-channel index, tap) pair and a chunk of pixels; threads = the wide channel (coalesced bf16 rows)
// ---------------------------------------------------------------------------------------------
// One block owns a chunk of WIDE pixels (rows of the bf16 NHWC tensor) and ALL Cn x 9 (narrow channel, tap) pairs: the 36 fp32
// narrow values that meet each wide pixel are gathered into shared memory once (zero outside the image), then every thread (= wide
// channel) reads its bf16 value of a pixel once and feeds 36 accumulators.  (The first version gave every (channel, tap) pair its own
// blocks and re-read the wide tensor 36 times with a division chain per pixel: 3.6 ms per launch at batch 16.)
//   conv_in  (wide_is_out = 1): wide = dh (output gradient), narrow = latent; input pixel = output pixel + (kh-1, kw-1)
//   conv_out (wide_is_out = 0): wide = activation (input),  narrow = dy;     output pixel = input pixel - (kh-1, kw-1)
constexpr int CEW_PX = 128;          // wide pixels per block
constexpr int CEW_MAX_PAIRS = 36;    // Cn <= 4
__global__ void __launch_bounds__(320) conv_edge_wgrad_kernel(const __nv_bfloat16* __restrict__ wide, const float* __restrict__ narrow, int B, int H, int W,
                                                              int Cw, int Cn, int wide_is_out, int chunk, float* __restrict__ dw,
                                                              float* __restrict__ db_wide) {
    pdl_trigger();
    pdl_wait();
    (void)chunk;
    __shared__ float tbl[CEW_PX][CEW_MAX_PAIRS + 1];
    const int npairs = Cn * 9;
    const int64_t npx = (int64_t)B * H * W;
    const int64_t p0 = (int64_t)blockIdx.x * CEW_PX;
    const int np = (int)min((int64_t)CEW_PX, npx - p0);
    const int sgn = wide_is_out ? 1 : -1;
    for (int i = threadIdx.x; i < CEW_PX * npairs; i += blockDim.x) {
        const int pl = i / npairs, pr = i % npairs;
        float v = 0.f;
        if (pl < np) {
            const int64_t px = p0 + pl;
            const int xw = (int)(px % W), yh = (int)((px / W) % H), b = (int)(px / ((int64_t)H * W));
            const int cn = pr / 9, tap = pr % 9;
            const int ih = yh + sgn * (tap / 3 - 1), iw = xw + sgn * (tap % 3 - 1);
            if (ih >= 0 && ih < H && iw >= 0 && iw < W) v = narrow[(((int64_t)b * Cn + cn) * H + ih) * W + iw];
        }
        tbl[pl][pr] = v;
    }
    __syncthreads();
    for (int cw = threadIdx.x; cw < Cw; cw += blockDim.x) {
        float acc[CEW_MAX_PAIRS];
#pragma unroll
        for (int j = 0; j < CEW_MAX_PAIRS; ++j) acc[j] = 0.f;
        float bsum = 0.f;
        for (int pl = 0; pl < np; ++pl) {
            const float wv = __bfloat162float(wide[(p0 + pl) * Cw + cw]);        // coalesced over cw
            bsum += wv;
#pragma unroll
            for (int j = 0; j < CEW_MAX_PAIRS; ++j) acc[j] = fmaf(wv, tbl[pl][j], acc[j]);   // pairs >= npairs: table column unused, acc ignored
        }
        for (int j = 0; j < npairs; ++j) {
            const int cn = j / 9, tap = j % 9;
            // nn.Conv2d layout [Cout, Cin, 3, 3]
            float* dst = wide_is_out ? dw + ((int64_t)cw * Cn + cn) * 9 + tap : dw + ((int64_t)cn * Cw + cw) * 9 + tap;
            atomicAdd(dst, acc[j]);
        }
        if (wide_is_out && db_wide) atomicAdd(db_wide + cw, bsum);
    }
}
// db[c] += sum over (b, y, x) of a fp32 NCHW tensor (conv_out bias gradient)
__global__ void nchw_channel_sum_kernel(const float* __restrict__ x, int B, int C, int64_t hw, float* __restrict__ out) {
    pdl_trigger();
    pdl_wait();
    const int c = blockIdx.x;
    float acc = 0.f;
    for (int b = 0; b < B; ++b)
        for (int64_t i = threadIdx.x; i < hw; i += blockDim.x) acc += x[((int64_t)b * C + c) * hw + i];
    acc = warp_sum(acc);
    __shared__ float s[32];
    if ((threadIdx.x & 31) == 0) s[threadIdx.x >> 5] = acc;
    __syncthreads();
    if (threadIdx.x < 32) {
        float v = (threadIdx.x < (blockDim.x >> 5)) ? s[threadIdx.x] : 0.f;
        v = warp_sum(v);
        if (threadIdx.x == 0) atomicAdd(out + c, v);
    }
}

// ---------------------------------------------------------------------------------------------
// per-step repack of trained fp32 master weights into the bf16 operand layouts (one launch for every trained layer)
//   kind 0  linear / 1x1 conv  W [rows, K]            -> W_bf16 rows [o0, o0+rows) of [*, K]  and  WT_bf16 [K, n_tot] columns [o0, ...)
//   kind 1  conv 3x3           W [Cout, Cin, 3, 3]    -> Wf [Cout, 3, 3, Cin]  and  Wd [Cin, 3, 3, Cout] (taps flipped when flip)
//   kind 2  fp32 vector copy   (fused-group biases, concatenated time_emb_proj biases)
//   kind 3  fp32 -> bf16 rows  W [rows, K] -> dst rows [o0, ...) of [*, K]   (time-embedding skinny-linear operands)
// ---------------------------------------------------------------------------------------------
struct RepackJob {
    const float* src;
    void* dst0;
    void* dst1;
    int32_t kind, rows, K, o0, n_tot, flip;
};
// Tiled: a block walks tiles of its job (blockIdx.y); both destinations are written in runs of consecutive elements.
//   kind 0 / 3: 64 x 64 tiles of W [rows, K]: rows of dst0 directly, the transposed tile through shared memory
//   kind 1: 16 output channels x 64 input channels x 9 taps of a 3x3 weight [Cout, Cin, 3, 3]: the 16 x 576 fp32 source rows are read
//           contiguously; dst0 [co][tap][ci] leaves in 64-element rows, dst1 [ci][tap'][co] in 16-element runs
// (The element-wise first version scattered 2-byte writes at a stride of n_tot: 11.6 ms for the 859 M parameters of the full UNet.)
__global__ void __launch_bounds__(256) repack_kernel(const RepackJob* __restrict__ jobs) {
    pdl_trigger();
    pdl_wait();
    const RepackJob jb = jobs[blockIdx.y];
    __shared__ __align__(16) uint8_t sraw[16 * 576 * 4 + 64];
    if (jb.kind == 2) {
        for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < jb.rows; i += (int64_t)gridDim.x * blockDim.x)
            reinterpret_cast<float*>(jb.dst0)[jb.o0 + i] = jb.src[i];
        return;
    }
    const int tid = threadIdx.x;
    if (jb.kind == 0 || jb.kind == 3) {
        __nv_bfloat16 (*st)[72] = reinterpret_cast<__nv_bfloat16 (*)[72]>(sraw);          // [64 k][64 rows + pad]
        const int K = jb.K, rows = jb.rows;
        const int tiles_k = (K + 63) / 64, ntiles = ((rows + 63) / 64) * tiles_k;
        __nv_bfloat16* d0 = reinterpret_cast<__nv_bfloat16*>(jb.dst0);
        __nv_bfloat16* d1 = reinterpret_cast<__nv_bfloat16*>(jb.dst1);
        const int tx = tid & 15, ty = tid >> 4;                                            // 4 consecutive k, rows ty + 16 i
        for (int t = blockIdx.x; t < ntiles; t += gridDim.x) {
            const int r_base = (t / tiles_k) * 64, k_base = (t % tiles_k) * 64;
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const int rl = ty + 16 * i, r = r_base + rl, k = k_base + tx * 4;
                float v[4] = {0.f, 0.f, 0.f, 0.f};
                if (r < rows) {
                    if (k + 4 <= K && (K & 3) == 0) {
                        const float4 f = *reinterpret_cast<const float4*>(jb.src + (int64_t)r * K + k);
                        v[0] = f.x; v[1] = f.y; v[2] = f.z; v[3] = f.w;
                    } else {
                        for (int e = 0; e < 4; ++e) if (k + e < K) v[e] = jb.src[(int64_t)r * K + k + e];
                    }
                    if (k + 4 <= K && (K & 3) == 0) {
                        uint2 pk;
                        pk.x = pack_bf16x2(v[0], v[1]); pk.y = pack_bf16x2(v[2], v[3]);
                        *reinterpret_cast<uint2*>(d0 + (int64_t)(jb.o0 + r) * K + k) = pk;
                    } else {
                        for (int e = 0; e < 4; ++e)
                            if (k + e < K) d0[(int64_t)(jb.o0 + r) * K + k + e] = __float2bfloat16(v[e]);
                    }
                }
                if (d1) for (int e = 0; e < 4; ++e) st[tx * 4 + e][rl] = __float2bfloat16(v[e]);
            }
            if (d1) {
                __syncthreads();
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                    const int kl = ty + 16 * i, k = k_base + kl;
                    if (k < K) {
                        const int r4 = r_base + tx * 4;
                        if (r4 + 4 <= rows && ((jb.n_tot | jb.o0) & 3) == 0) {
                            *reinterpret_cast<uint2*>(d1 + (int64_t)k * jb.n_tot + jb.o0 + r4) = *reinterpret_cast<const uint2*>(&st[kl][tx * 4]);
                        } else {
                            for (int e = 0; e < 4; ++e)
                                if (r4 + e < rows) d1[(int64_t)k * jb.n_tot + jb.o0 + r4 + e] = st[kl][tx * 4 + e];
                        }
                    }
                }
                __syncthreads();
            }
        }
        return;
    }
    // kind 1: rows = Cout, K = Cin; src index = ((co * Cin + ci) * 9 + tap)
    float (*sf)[577] = reinterpret_cast<float (*)[577]>(sraw);                              // [16 co][64 ci * 9 taps] (+1: bank spread)
    static_assert(sizeof(sraw) >= 16 * 577 * 4, "kind-1 tile");
    const int Cin = jb.K, Cout = jb.rows;
    const int tiles_ci = (Cin + 63) / 64, ntiles = ((Cout + 15) / 16) * tiles_ci;
    __nv_bfloat16* d0 = reinterpret_cast<__nv_bfloat16*>(jb.dst0);
    __nv_bfloat16* d1 = reinterpret_cast<__nv_bfloat16*>(jb.dst1);
    for (int t = blockIdx.x; t < ntiles; t += gridDim.x) {
        const int co_base = (t / tiles_ci) * 16, ci_base = (t % tiles_ci) * 64;
        const int nci = min(64, Cin - ci_base), nco = min(16, Cout - co_base);
        for (int i = tid; i < 16 * 576; i += 256) {
            const int col = i / 576, e = i % 576;                                          // e = ci_local * 9 + tap
            sf[col][e] = (col < nco && e < nci * 9) ? jb.src[((int64_t)(co_base + col) * Cin + ci_base) * 9 + e] : 0.f;
        }
        __syncthreads();
        // dst0 [co][tap][ci]: consecutive threads -> consecutive ci
        for (int i = tid; i < 16 * 9 * 64; i += 256) {
            const int cil = i & 63, tap = (i >> 6) % 9, col = i / 576;
            if (col < nco && cil < nci) d0[((int64_t)(co_base + col) * 9 + tap) * Cin + ci_base + cil] = __float2bfloat16(sf[col][cil * 9 + tap]);
        }
        // dst1 [ci][tap'][co]: consecutive threads -> consecutive co (16-element runs)
        for (int i = tid; i < 64 * 9 * 16; i += 256) {
            const int col = i & 15, tap = (i >> 4) % 9, cil = i / 144;
            if (col < nco && cil < nci) {
                const int tap_d = jb.flip ? 8 - tap : tap;
                d1[((int64_t)(ci_base + cil) * 9 + tap_d) * Cout + co_base + col] = __float2bfloat16(sf[col][cil * 9 + tap]);
            }
        }
        __syncthreads();
    }
}

template <int SN, bool kTable>
static int launch_wgrad(const WgradParams& p, cudaStream_t stream) {
    using Cfg = WgCfg<SN>;
    static bool configured = false;
    if (!configured) {
        cudaError_t e = cudaFuncSetAttribute(wgrad_tc_kernel<SN, kTable>, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM_BYTES);
        if (e != cudaSuccess) return set_cuda_error(e, "cudaFuncSetAttribute(wgrad)");
        configured = true;
    }
    const int ctas = p.prob[0].ctas + (p.nprob == 2 ? p.prob[1].ctas : 0);
    launch_k(wgrad_tc_kernel<SN, kTable>, dim3(ctas), dim3(kWgThreads), Cfg::SMEM_BYTES, stream, p);
    LAUNCH_CHECK("wgrad launch");
    return HCP_OK;
}

// `splits` CTAs (at least one 128-row tile each) share the rows of every output tile of the problem
static void split_rows(WgProblem& q, int M, int splits) {
    const int total_tiles = (M + 127) / 128;
    if (splits < 1) splits = 1;
    if (splits > total_tiles) splits = total_tiles;
    q.tiles_per_cta = (total_tiles + splits - 1) / splits;
    q.splits = (total_tiles + q.tiles_per_cta - 1) / q.tiles_per_cta;
    q.ctas = q.n_tiles * q.j_tiles * q.splits;
}

// dense problem over S columns [0, j_cols) and X columns [0, n_cols): about two waves of CTAs
static int run_wgrad(WgradParams& p, int64_t j_cols, int64_t n_cols, cudaStream_t stream) {
    WgProblem& q = p.prob[0];
    const int sn = (j_cols > 64) ? 128 : 64;
    p.nprob = 1;
    q.n_tiles = (int)((n_cols + 127) / 128);
    q.j_tiles = (int)((j_cols + sn - 1) / sn);
    q.n_end = (int)n_cols; q.j_cols = (int)j_cols;
    const int out_tiles = q.n_tiles * q.j_tiles;
    split_rows(q, p.M, (2 * num_sms() + out_tiles - 1) / out_tiles);
    if (sn == 128) return launch_wgrad<128, false>(p, stream);
    return launch_wgrad<64, false>(p, stream);
}

// X operand of a 3x3 / pad 1 convolution's weight gradient: the shifted boxes of the forward convolution, one row per output pixel
static int conv_x(WgradParams& p, const void* x, int64_t B, int64_t Hin, int64_t Win, int64_t Cin, int stride, const char* who) {
    const int64_t oH = Hin / stride, oW = Win / stride;
    int rc = plan_conv_box(oH, oW, who, p.conv.box);
    if (rc) return rc;
    p.M = (int)(B * oH * oW);
    p.conv.rank = stride == 1 ? 4 : 5;
    return make_tmap_nhwc(&p.prob[0].tmX, x, B, Hin, Win, Cin, stride, p.conv.box);
}

// LoRA problem: the 64 S columns of one slab against X columns [n_begin, n_end) in 128-column chunks, `target_ctas` CTAs in all
static void lg_problem(WgProblem& q, int M, int64_t n_begin, int64_t n_end, int target_ctas) {
    q.n_begin = (int)n_begin; q.n_end = (int)n_end;
    q.n_tiles = (int)((n_end - n_begin + 127) / 128);
    q.j_tiles = 1;
    split_rows(q, M, target_ctas / q.n_tiles);
}

static int lg_table(LGTable& t, const hcp_lora_grad_block* blocks, int32_t nblocks, const char* err) {
    t.nblocks = nblocks;
    for (int i = 0; i < nblocks; ++i) {
        const hcp_lora_grad_block& k = blocks[i];
        if (k.rank < 1 || k.c0 < 0 || k.c0 + k.rank > 64 || !k.dst) return set_error(HCP_ERR_INVALID, err);
        t.blk[i].n_lo = (int)k.n_lo; t.blk[i].n_hi = (int)k.n_hi; t.blk[i].c0 = k.c0; t.blk[i].rank = k.rank;
        t.blk[i].transpose_out = k.transpose_out; t.blk[i].dst_ld = (int)k.dst_ld; t.blk[i].scale = k.scale; t.blk[i].dst = k.dst;
        t.blk[i].n_stride = 1;
    }
    return HCP_OK;
}

// X-column ranges and destination pitches of a linear launch's blocks.  The kernel reduces only X columns [n_begin, n_end), so a
// block reaching outside them would silently lose those columns; a pitch below the row length would make destination rows overlap.
static int lg_check_ranges(const hcp_lora_grad_block* blocks, int32_t nblocks, int64_t n_begin, int64_t n_end) {
    for (int i = 0; i < nblocks; ++i) {
        const hcp_lora_grad_block& k = blocks[i];
        if (k.n_lo >= k.n_hi || k.n_lo < n_begin || k.n_hi > n_end)
            return set_error(HCP_ERR_INVALID, "lora_grad: block columns [n_lo, n_hi) must be a non-empty part of [n_begin, n_end)");
        if (k.dst_ld < (k.transpose_out ? (int64_t)k.rank : k.n_hi - k.n_lo))
            return set_error(HCP_ERR_INVALID, "lora_grad: block dst_ld below its row length (rank, or n_hi - n_lo without transpose)");
    }
    return HCP_OK;
}

static int lg_fill(WgradParams& p, int z, const void* S, int64_t lds, const void* X, int64_t ldx, int64_t M, int64_t n_begin,
                   int64_t n_end, const hcp_lora_grad_block* blocks, int32_t nblocks, int target_ctas) {
    if (!S || !X || !blocks || nblocks < 1 || nblocks > LG_MAX_BLOCKS) return set_error(HCP_ERR_INVALID, "lora_grad: 1..8 blocks per problem");
    if (n_begin < 0 || n_end <= n_begin || (ldx % 8) != 0 || (n_begin % 8) != 0 || lds < 64 || (lds % 8) != 0)
        return set_error(HCP_ERR_INVALID, "lora_grad: shape");
    // the X tensor map is ldx columns wide: columns past it would read as zeros
    if (n_end > ldx) return set_error(HCP_ERR_INVALID, "lora_grad: n_end > ldx");
    int rc = lg_check_ranges(blocks, nblocks, n_begin, n_end);
    if (rc) return rc;
    WgProblem& q = p.prob[z];
    rc = make_tmap_2d(&q.tmX, X, (uint64_t)ldx, (uint64_t)M, (uint64_t)ldx, 64, 128);
    if (rc) return rc;
    rc = make_tmap_2d(&q.tmS, S, 64, (uint64_t)M, (uint64_t)lds, 64, 128);     // the 64 columns of S this launch reduces
    if (rc) return rc;
    lg_problem(q, p.M, n_begin, n_end, target_ctas);
    return lg_table(q.tab, blocks, nblocks, "lora_grad: block descriptor");
}

}  // namespace hcp

using namespace hcp;

extern "C" int hcp_wgrad_bf16(const void* S, int64_t lds, int64_t j_cols, const void* X, int64_t ldx, int64_t n_cols, int64_t M,
                              float scale, float* dst, int64_t ld_j, int64_t ld_n, hcp_stream_t stream_) {
    if (!S || !X || !dst || M <= 0 || j_cols <= 0 || n_cols <= 0) return set_error(HCP_ERR_INVALID, "wgrad: arguments");
    if ((lds % 8) || (ldx % 8)) return set_error(HCP_ERR_INVALID, "wgrad: row pitches must be multiples of 8 elements");
    WgradParams p;
    memset(&p, 0, sizeof(p));
    WgProblem& q = p.prob[0];
    p.M = (int)M; q.scale = scale; q.dst = dst; q.ld_j = ld_j; q.ld_n = ld_n;
    int rc = make_tmap_2d(&q.tmX, X, (uint64_t)n_cols, (uint64_t)M, (uint64_t)ldx, 64, 128);
    if (rc) return rc;
    rc = make_tmap_2d(&q.tmS, S, (uint64_t)j_cols, (uint64_t)M, (uint64_t)lds, 64, 128);
    if (rc) return rc;
    return run_wgrad(p, j_cols, n_cols, (cudaStream_t)stream_);
}

// dW [Cout, Cin, 3, 3] (nn.Conv2d layout, fp32, accumulated) of a 3x3 / pad 1 / stride 1|2 convolution: nine launches, one per tap
extern "C" int hcp_wgrad_conv3x3_bf16(const void* dy, int64_t Cout, const void* x, int64_t B, int64_t Hin, int64_t Win, int64_t Cin,
                                      int32_t stride, float scale, float* dw, hcp_stream_t stream_) {
    if (!dy || !x || !dw) return set_error(HCP_ERR_INVALID, "wgrad_conv: null pointer");
    if (Cin % 64 != 0 || Cout % 8 != 0 || (stride != 1 && stride != 2)) return set_error(HCP_ERR_INVALID, "wgrad_conv: shape");
    if (stride == 2 && ((Hin | Win) & 1)) return set_error(HCP_ERR_INVALID, "wgrad_conv: odd extent with stride 2");
    WgradParams p;
    memset(&p, 0, sizeof(p));
    WgProblem& q = p.prob[0];
    q.scale = scale; q.ld_j = Cin * 9; q.ld_n = 9;
    int rc = conv_x(p, x, B, Hin, Win, Cin, stride, "wgrad_conv");
    if (rc) return rc;
    rc = make_tmap_2d(&q.tmS, dy, (uint64_t)Cout, (uint64_t)p.M, (uint64_t)Cout, 64, 128);
    if (rc) return rc;
    for (int kh = 0; kh < 3; ++kh)
        for (int kw = 0; kw < 3; ++kw) {
            p.conv.tap = conv_tap(kh, kw, stride, Cin);
            q.dst = dw + (kh * 3 + kw);
            rc = run_wgrad(p, Cout, Cin, (cudaStream_t)stream_);
            if (rc) return rc;
        }
    return HCP_OK;
}

extern "C" int hcp_lora_grad(const void* S, int64_t lds, const void* X, int64_t ldx, int64_t M, int64_t n_begin, int64_t n_end,
                             const hcp_lora_grad_block* blocks, int32_t nblocks, hcp_stream_t stream_) {
    if (M <= 0) return set_error(HCP_ERR_INVALID, "lora_grad: M");
    WgradParams p;
    memset(&p, 0, sizeof(p));
    p.M = (int)M; p.nprob = 1;
    int rc = lg_fill(p, 0, S, lds, X, ldx, M, n_begin, n_end, blocks, nblocks, num_sms());     // one wave of CTAs
    if (rc) return rc;
    return launch_wgrad<64, true>(p, (cudaStream_t)stream_);
}

// dW_down of a Conv2d LoRA: nine launches (one per tap) with the shifted NHWC box as X operand.
extern "C" int hcp_lora_grad_conv3x3(const void* S, int64_t lds, const void* x, int64_t B, int64_t Hin, int64_t Win, int64_t Cin,
                                     int32_t stride, const hcp_lora_grad_block* blocks, int32_t nblocks, hcp_stream_t stream_) {
    if (!S || !x || !blocks || nblocks < 1 || nblocks > LG_MAX_BLOCKS) return set_error(HCP_ERR_INVALID, "lora_grad_conv: arguments");
    if (Cin % 64 != 0 || (stride != 1 && stride != 2) || lds < 64 || (lds % 8) != 0) return set_error(HCP_ERR_INVALID, "lora_grad_conv: shape");
    if (stride == 2 && ((Hin | Win) & 1)) return set_error(HCP_ERR_INVALID, "lora_grad_conv: odd extent with stride 2");
    WgradParams p;
    memset(&p, 0, sizeof(p));
    WgProblem& q = p.prob[0];
    p.nprob = 1;
    int rc = conv_x(p, x, B, Hin, Win, Cin, stride, "lora_grad_conv");
    if (rc) return rc;
    rc = make_tmap_2d(&q.tmS, S, 64, (uint64_t)p.M, (uint64_t)lds, 64, 128);
    if (rc) return rc;
    lg_problem(q, p.M, 0, Cin, num_sms());
    if ((rc = lg_table(q.tab, blocks, nblocks, "lora_grad_conv: block descriptor"))) return rc;
    for (int i = 0; i < nblocks; ++i) {      // dW_down [r, Cin, 3, 3]: X column ci of tap t lands at dst[j * 9 Cin + 9 ci + t]
        LGBlock& k = q.tab.blk[i];
        k.n_lo = 0; k.n_hi = (int)Cin; k.transpose_out = 0; k.dst_ld = (int)(Cin * 9); k.n_stride = 9;
    }
    for (int kh = 0; kh < 3; ++kh)
        for (int kw = 0; kw < 3; ++kw) {
            p.conv.tap = conv_tap(kh, kw, stride, Cin);
            for (int i = 0; i < nblocks; ++i) q.tab.blk[i].dst = blocks[i].dst + (kh * 3 + kw);
            rc = launch_wgrad<64, true>(p, (cudaStream_t)stream_);
            if (rc) return rc;
        }
    return HCP_OK;
}

// dW_down and dW_up of one LoRA group in ONE launch (two independent TN GEMMs over the same M token rows).
extern "C" int hcp_lora_grad_pair(const void* U, const void* x, int64_t ldx, int64_t K, const hcp_lora_grad_block* down,
                                  const void* T, const void* dy, int64_t lddy, int64_t N, const hcp_lora_grad_block* up,
                                  int32_t nblocks, int64_t M, int64_t lds, hcp_stream_t stream_) {
    if (M <= 0) return set_error(HCP_ERR_INVALID, "lora_grad_pair: M");
    WgradParams p;
    memset(&p, 0, sizeof(p));
    p.M = (int)M; p.nprob = 2;
    // split the SMs between the two problems in proportion to their column counts (one CTA per SM: 147 KB of smem each)
    const int64_t ck = (K + 127) / 128, cn = (N + 127) / 128;
    const int sms = num_sms();
    int t0 = (int)((sms * ck + (ck + cn) / 2) / (ck + cn));
    if (t0 < 1) t0 = 1;
    if (t0 > sms - 1) t0 = sms - 1;
    int rc = lg_fill(p, 0, U, lds, x, ldx, M, 0, K, down, nblocks, t0);
    if (rc) return rc;
    rc = lg_fill(p, 1, T, lds, dy, lddy, M, 0, N, up, nblocks, sms - t0);
    if (rc) return rc;
    return launch_wgrad<64, true>(p, (cudaStream_t)stream_);
}

extern "C" int hcp_colsum_bf16(const void* x, int64_t ld, int64_t M, int64_t N, int64_t rows_per_group, float scale, float* out,
                               int64_t ldo, hcp_stream_t st) {
    if (!x || !out || M <= 0 || N <= 0 || (N % 8) || (ld % 8) || ((uintptr_t)x & 15))
        return set_error(HCP_ERR_INVALID, "colsum: arguments (N, ld multiples of 8; 16-byte aligned x)");
    if (rows_per_group <= 0) rows_per_group = M;
    if (M % rows_per_group) return set_error(HCP_ERR_INVALID, "colsum: M must be a multiple of rows_per_group");
    int64_t chunk = rows_per_group;
    while (chunk > 512 && (chunk % 2) == 0) chunk /= 2;        // chunk divides rows_per_group: a block never straddles two groups
    dim3 grid((unsigned)((N + 63) / 64), (unsigned)(M / chunk));
    launch_k(colsum_bf16_kernel, grid, dim3(256), 0, (cudaStream_t)st, (const __nv_bfloat16*)x, ld, M, (int)N, rows_per_group, (int)chunk, scale, out, ldo);
    LAUNCH_CHECK("colsum launch");
    return HCP_OK;
}

extern "C" int hcp_norm_affine_grad_bf16(const void* x1, const void* x2, int64_t C1, int64_t C2, const void* dy, const float* stats,
                                         const float* gamma, const float* beta, int64_t rows, int64_t rows_per_image, int64_t groups,
                                         int32_t silu, float* dgamma, float* dbeta, hcp_stream_t st) {
    const int64_t C = C1 + C2;
    if (!x1 || !dy || !stats || !gamma || !beta || !dgamma || !dbeta || rows <= 0 || C <= 0 || (C1 % 8) || (C2 % 8) || (C2 && !x2))
        return set_error(HCP_ERR_INVALID, "norm_affine_grad: arguments (channel counts must be multiples of 8)");
    int cpg = 0;
    if (groups > 0) {
        if (C % groups || ((C / groups) & 1) || rows_per_image <= 0) return set_error(HCP_ERR_INVALID, "norm_affine_grad: groups");
        cpg = (int)(C / groups);
    }
    int64_t chunk = 1024;
    if (groups > 0) {                       // a block stays inside one image: its statistics are loop constants
        if (rows % rows_per_image) return set_error(HCP_ERR_INVALID, "norm_affine_grad: rows must be a multiple of rows_per_image");
        chunk = rows_per_image;
        while (chunk > 1024 && (chunk % 2) == 0) chunk /= 2;
    }
    dim3 grid((unsigned)((C + 63) / 64), (unsigned)((rows + chunk - 1) / chunk));
    launch_k(norm_affine_grad_kernel, grid, dim3(256), 0, (cudaStream_t)st, (const __nv_bfloat16*)x1, (const __nv_bfloat16*)x2, (int)C1, (int)C2,
             (const __nv_bfloat16*)dy, stats, gamma, beta, rows, rows_per_image, cpg, (int)groups, (int)silu, (int)chunk, dgamma, dbeta);
    LAUNCH_CHECK("norm_affine_grad launch");
    return HCP_OK;
}

extern "C" int hcp_small_linear_bwd_f32(const float* dy, int64_t ldy, const float* x, const void* w_bf16, int64_t M, int64_t N, int64_t K,
                                        float* dx, float* dw, float* db, hcp_stream_t st) {
    if (!dy || M <= 0 || N <= 0 || K <= 0 || M > 4096 || ldy < N) return set_error(HCP_ERR_INVALID, "small_linear_bwd: arguments");
    if (dx) {
        if (!w_bf16) return set_error(HCP_ERR_INVALID, "small_linear_bwd: dx needs the weight");
        cudaError_t ez = cudaMemsetAsync(dx, 0, (size_t)M * K * sizeof(float), (cudaStream_t)st);      // the kernel accumulates n slices
        if (ez != cudaSuccess) return set_cuda_error(ez, "small_linear dx memset");
        const int kb = (int)((K + 127) / 128);
        int n_chunk = 512;
        while (n_chunk < N && (int64_t)kb * ((N + n_chunk - 1) / n_chunk) > 592) n_chunk *= 2;
        launch_k(small_linear_dx_kernel, dim3((unsigned)kb, (unsigned)((N + n_chunk - 1) / n_chunk), (unsigned)((M + SLDX_ROWS - 1) / SLDX_ROWS)), dim3(128), 0,
                 (cudaStream_t)st, dy, ldy, (const __nv_bfloat16*)w_bf16, (int)M, (int)N, (int)K, n_chunk, dx);
        LAUNCH_CHECK("small_linear dx launch");
    }
    if (dw) {
        if (!x) return set_error(HCP_ERR_INVALID, "small_linear_bwd: dW needs the input");
        launch_k(small_linear_dw_kernel, dim3((unsigned)((K + 127) / 128), (unsigned)N), dim3(128), 0, (cudaStream_t)st, dy, ldy, x, (int)M, (int)N, (int)K, dw, db);
        LAUNCH_CHECK("small_linear dW launch");
    }
    return HCP_OK;
}

extern "C" int hcp_silu_f32(const float* x, const float* dy, int64_t n, float* out, hcp_stream_t st) {
    if (!x || !out || n <= 0) return set_error(HCP_ERR_INVALID, "silu: arguments");
    launch_k(silu_f32_kernel, dim3((unsigned)((n + 255) / 256)), dim3(256), 0, (cudaStream_t)st, x, dy, n, out);
    LAUNCH_CHECK("silu launch");
    return HCP_OK;
}

extern "C" int hcp_conv_in_wgrad_f32(const void* dh_nhwc_bf16, const float* x_nchw, int64_t B, int64_t Cin, int64_t H, int64_t W, int64_t Cout,
                                     float* dw, float* db, hcp_stream_t st) {
    if (!dh_nhwc_bf16 || !x_nchw || !dw) return set_error(HCP_ERR_INVALID, "conv_in_wgrad: null pointer");
    const int64_t npx = B * H * W;
    if (Cin > 4) return set_error(HCP_ERR_INVALID, "conv_in_wgrad: at most 4 input channels");
    const int chunk = CEW_PX;
    dim3 grid((unsigned)((npx + chunk - 1) / chunk));
    launch_k(conv_edge_wgrad_kernel, grid, dim3(320), 0, (cudaStream_t)st, (const __nv_bfloat16*)dh_nhwc_bf16, x_nchw, (int)B, (int)H, (int)W, (int)Cout,
             (int)Cin, 1, chunk, dw, db);
    LAUNCH_CHECK("conv_in_wgrad launch");
    return HCP_OK;
}

extern "C" int hcp_conv_out_wgrad_f32(const float* dy_nchw, const void* x_nhwc_bf16, int64_t B, int64_t H, int64_t W, int64_t Cin, int64_t Cout,
                                      float* dw, float* db, hcp_stream_t st) {
    if (!dy_nchw || !x_nhwc_bf16 || !dw) return set_error(HCP_ERR_INVALID, "conv_out_wgrad: null pointer");
    const int64_t npx = B * H * W;
    if (Cout > 4) return set_error(HCP_ERR_INVALID, "conv_out_wgrad: at most 4 output channels");
    const int chunk = CEW_PX;
    dim3 grid((unsigned)((npx + chunk - 1) / chunk));
    launch_k(conv_edge_wgrad_kernel, grid, dim3(320), 0, (cudaStream_t)st, (const __nv_bfloat16*)x_nhwc_bf16, dy_nchw, (int)B, (int)H, (int)W, (int)Cin,
             (int)Cout, 0, chunk, dw, (float*)nullptr);
    LAUNCH_CHECK("conv_out_wgrad launch");
    if (db) {
        launch_k(nchw_channel_sum_kernel, dim3((unsigned)Cout), dim3(256), 0, (cudaStream_t)st, dy_nchw, (int)B, (int)Cout, H * W, db);
        LAUNCH_CHECK("conv_out bias grad launch");
    }
    return HCP_OK;
}

extern "C" int hcp_repack_weights(const hcp_repack_job* jobs_device, int64_t njobs, hcp_stream_t st) {
    if (!jobs_device || njobs <= 0) return set_error(HCP_ERR_INVALID, "repack: jobs");
    static_assert(sizeof(hcp_repack_job) == sizeof(RepackJob), "hcp_repack_job layout");
    dim3 grid(64, (unsigned)njobs);
    launch_k(repack_kernel, grid, dim3(256), 0, (cudaStream_t)st, reinterpret_cast<const RepackJob*>(jobs_device));
    LAUNCH_CHECK("repack launch");
    return HCP_OK;
}
