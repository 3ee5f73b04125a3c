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
// One CTA owns 128 columns of X and SN columns of S over a slice of the rows; MMA warpgroup g computes X columns [64g, 64g+64)
// (wgmma M = 64, N = SN, K = 16 rows per instruction) and reduces its 64 x SN fp32 block into dst[j * ld_j + n * ld_n] with atomics.
// =============================================================================================
constexpr int kWgThreads = 288;   // warps 0-7: two MMA warpgroups, warp 8: TMA

struct WgConv {
    int32_t rank;            // 0: plain [M, ldx] matrix; 4 / 5: rank of the NHWC tensor map
    int32_t bw, bh, bn, tiles_w, tiles_h;
    int32_t c0_off, dw, dh, c2;
};
struct alignas(64) WgradParams {
    CUtensorMap tmX, tmS;
    int32_t M;
    int32_t n_tiles, j_tiles, splits, tiles_per_cta;
    int32_t n_cols, j_cols;          // valid X / S columns
    int64_t ld_j, ld_n;
    float scale;
    float* dst;
    WgConv conv;
};

template <int SN>
struct WgCfg {
    static constexpr int X_BYTES = 2 * 128 * 128;             // two 64-column boxes of 128 rows
    static constexpr int S_BYTES = (SN / 64) * 128 * 128;
    static constexpr int STAGE_BYTES = X_BYTES + S_BYTES;
    static constexpr int STAGES = 3;
    static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + 256 + 1024;
};

template <int SN>
__global__ void __launch_bounds__(kWgThreads, 1) wgrad_tc_kernel(const __grid_constant__ WgradParams p) {
    using Cfg = WgCfg<SN>;
    constexpr int STAGES = Cfg::STAGES;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + STAGES * Cfg::STAGE_BYTES);
    uint64_t* empty_bar = full_bar + STAGES;
    const int warp = warp_id_uniform(), lane = threadIdx.x & 31;
    // flat grid over (row split, j tile, n tile): n fastest so that concurrent CTAs share the S tile in L2
    const int bid = blockIdx.x;
    const int nt = bid % p.n_tiles, jt = (bid / p.n_tiles) % p.j_tiles, sp = bid / (p.n_tiles * p.j_tiles);
    const int ncol0 = nt * 128, jcol0 = jt * SN;
    const int total_tiles = (p.M + 127) / 128;
    const int t0 = sp * p.tiles_per_cta;
    const int t1 = min(total_tiles, t0 + p.tiles_per_cta);

    if (threadIdx.x == 0) {
        for (int s = 0; s < STAGES; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], 256); }
        fence_mbar_init();
        tma_prefetch_desc(&p.tmX);
        tma_prefetch_desc(&p.tmS);
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
                    tma_load_2d(base, &p.tmX, &full_bar[stage], ncol0, t * 128);
                    tma_load_2d(base + 128 * 128, &p.tmX, &full_bar[stage], ncol0 + 64, t * 128);
                } else {
                    const WgConv& cv = p.conv;
                    int img0, h0 = 0, w0 = 0;
                    if (cv.bn == 1) {
                        const int per_img = cv.tiles_w * cv.tiles_h, r = t % per_img;
                        img0 = t / per_img;
                        h0 = (r / cv.tiles_w) * cv.bh;
                        w0 = (r % cv.tiles_w) * cv.bw;
                    } else {
                        img0 = t * cv.bn;
                    }
                    for (int hf = 0; hf < 2; ++hf) {
                        const int c = cv.c0_off + ncol0 + hf * 64;
                        if (cv.rank == 4) tma_load_4d(base + hf * 128 * 128, &p.tmX, &full_bar[stage], c, w0 + cv.dw, h0 + cv.dh, img0);
                        else tma_load_5d(base + hf * 128 * 128, &p.tmX, &full_bar[stage], c, w0 + cv.dw, cv.c2, h0 + cv.dh, img0);
                    }
                }
#pragma unroll
                for (int q = 0; q < SN / 64; ++q)
                    tma_load_2d(base + Cfg::X_BYTES + q * 128 * 128, &p.tmS, &full_bar[stage], jcol0 + q * 64, t * 128);
                if (++stage == STAGES) { stage = 0; phase ^= 1; }
            }
        }
        return;
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
    const float scale = p.scale;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        const int n = ncol0 + wg * 64 + (warp & 3) * 16 + (lane >> 2) + 8 * h;     // column of X
        if (n >= p.n_cols) continue;
        float* dcol = p.dst + (int64_t)n * p.ld_n;
#pragma unroll
        for (int i = 0; i < SN / 4; ++i) {
            const int j = jcol0 + 8 * (i >> 1) + 2 * (lane & 3) + (i & 1);          // column of S
            if (j < p.j_cols) atomicAdd(dcol + (int64_t)j * p.ld_j, acc[4 * (i >> 1) + 2 * h + (i & 1)] * scale);
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

template <int SN>
static int launch_wgrad(const WgradParams& p, int ctas, cudaStream_t stream) {
    using Cfg = WgCfg<SN>;
    static bool configured = false;
    if (!configured) {
        cudaError_t e = cudaFuncSetAttribute(wgrad_tc_kernel<SN>, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM_BYTES);
        if (e != cudaSuccess) return set_cuda_error(e, "cudaFuncSetAttribute(wgrad)");
        configured = true;
    }
    launch_k(wgrad_tc_kernel<SN>, dim3(ctas), dim3(kWgThreads), Cfg::SMEM_BYTES, stream, p);
    LAUNCH_CHECK("wgrad launch");
    return HCP_OK;
}

static int run_wgrad(WgradParams& p, int64_t j_cols, int64_t n_cols, cudaStream_t stream) {
    const int sn = (j_cols > 64) ? 128 : 64;
    p.n_tiles = (int)((n_cols + 127) / 128);
    p.j_tiles = (int)((j_cols + sn - 1) / sn);
    p.n_cols = (int)n_cols; p.j_cols = (int)j_cols;
    const int total_tiles = (p.M + 127) / 128;
    const int out_tiles = p.n_tiles * p.j_tiles;
    int splits = (2 * num_sms() + out_tiles - 1) / out_tiles;    // about two waves of CTAs
    if (splits < 1) splits = 1;
    if (splits > total_tiles) splits = total_tiles;
    p.tiles_per_cta = (total_tiles + splits - 1) / splits;
    p.splits = (total_tiles + p.tiles_per_cta - 1) / p.tiles_per_cta;
    const int ctas = out_tiles * p.splits;
    if (sn == 128) return launch_wgrad<128>(p, ctas, stream);
    return launch_wgrad<64>(p, ctas, stream);
}

}  // namespace hcp

using namespace hcp;

extern "C" int hcp_wgrad_bf16(const void* S, int64_t lds, int64_t j_cols, const void* X, int64_t ldx, int64_t n_cols, int64_t M,
                              float scale, float* dst, int64_t ld_j, int64_t ld_n, hcp_stream_t stream_) {
    if (!S || !X || !dst || M <= 0 || j_cols <= 0 || n_cols <= 0) return set_error(HCP_ERR_INVALID, "wgrad: arguments");
    if ((lds % 8) || (ldx % 8)) return set_error(HCP_ERR_INVALID, "wgrad: row pitches must be multiples of 8 elements");
    WgradParams p;
    memset(&p, 0, sizeof(p));
    p.M = (int)M; p.scale = scale; p.dst = dst; p.ld_j = ld_j; p.ld_n = ld_n;
    int rc = make_tmap_2d(&p.tmX, X, (uint64_t)n_cols, (uint64_t)M, (uint64_t)ldx, 64, 128);
    if (rc) return rc;
    rc = make_tmap_2d(&p.tmS, S, (uint64_t)j_cols, (uint64_t)M, (uint64_t)lds, 64, 128);
    if (rc) return rc;
    return run_wgrad(p, j_cols, n_cols, (cudaStream_t)stream_);
}

// dW [Cout, Cin, 3, 3] (nn.Conv2d layout, fp32, accumulated) of a 3x3 / pad 1 / stride 1|2 convolution: nine launches, one per tap
extern "C" int hcp_wgrad_conv3x3_bf16(const void* dy, int64_t Cout, const void* x, int64_t B, int64_t Hin, int64_t Win, int64_t Cin,
                                      int32_t stride, float scale, float* dw, hcp_stream_t stream_) {
    if (!dy || !x || !dw) return set_error(HCP_ERR_INVALID, "wgrad_conv: null pointer");
    if (Cin % 64 != 0 || Cout % 8 != 0 || (stride != 1 && stride != 2)) return set_error(HCP_ERR_INVALID, "wgrad_conv: shape");
    if (stride == 2 && ((Hin | Win) & 1)) return set_error(HCP_ERR_INVALID, "wgrad_conv: odd extent with stride 2");
    const int64_t oH = Hin / stride, oW = Win / stride;
    int bw, bh, bnimg;                       // same 128-pixel tiles as hcp_conv3x3_bf16 (mode 0)
    if (oW >= 128) { bw = 128; bh = 1; bnimg = 1; if (oW % 128) return set_error(HCP_ERR_INVALID, "wgrad_conv: W"); }
    else {
        bw = (int)oW;
        if (128 % bw) return set_error(HCP_ERR_INVALID, "wgrad_conv: W must divide 128");
        bh = 128 / bw;
        if (bh <= oH) { if (oH % bh) return set_error(HCP_ERR_INVALID, "wgrad_conv: H tiling"); bnimg = 1; }
        else { bh = (int)oH; if (128 % (bw * bh)) return set_error(HCP_ERR_INVALID, "wgrad_conv: H*W must divide 128"); bnimg = 128 / (bw * bh); }
    }
    WgradParams p;
    memset(&p, 0, sizeof(p));
    const int64_t M = B * oH * oW;
    p.M = (int)M; p.scale = scale;
    p.ld_j = Cin * 9; p.ld_n = 9;
    int rc;
    if (stride == 1) {
        uint64_t dims[4] = {(uint64_t)Cin, (uint64_t)Win, (uint64_t)Hin, (uint64_t)B};
        uint64_t strides[3] = {(uint64_t)Cin * 2, (uint64_t)Win * Cin * 2, (uint64_t)Hin * Win * Cin * 2};
        uint32_t box[4] = {64, (uint32_t)bw, (uint32_t)bh, (uint32_t)bnimg};
        rc = make_tmap_nd(&p.tmX, x, 4, dims, strides, box);
        p.conv.rank = 4;
    } else {
        uint64_t dims[5] = {(uint64_t)(2 * Cin), (uint64_t)(Win / 2), 2, (uint64_t)(Hin / 2), (uint64_t)B};
        uint64_t strides[4] = {(uint64_t)(2 * Cin) * 2, (uint64_t)Win * Cin * 2, (uint64_t)(2 * Win * Cin) * 2, (uint64_t)Hin * Win * Cin * 2};
        uint32_t box[5] = {64, (uint32_t)bw, 1, (uint32_t)bh, (uint32_t)bnimg};
        rc = make_tmap_nd(&p.tmX, x, 5, dims, strides, box);
        p.conv.rank = 5;
    }
    if (rc) return rc;
    rc = make_tmap_2d(&p.tmS, dy, (uint64_t)Cout, (uint64_t)M, (uint64_t)Cout, 64, 128);
    if (rc) return rc;
    p.conv.bw = bw; p.conv.bh = bh; p.conv.bn = bnimg;
    p.conv.tiles_w = (int)(oW / bw); p.conv.tiles_h = (int)(oH / bh);
    for (int kh = 0; kh < 3; ++kh)
        for (int kw = 0; kw < 3; ++kw) {
            if (stride == 1) { p.conv.c0_off = 0; p.conv.dw = kw - 1; p.conv.dh = kh - 1; p.conv.c2 = 0; }
            else {          // input row 2*oh + kh - 1 -> (phase, index) of the [H/2][2][W/2][2C] view, as in the forward conv
                p.conv.c0_off = (int)(((kw == 1) ? 0 : 1) * Cin);
                p.conv.dw = (kw == 0) ? -1 : 0;
                p.conv.c2 = (kh == 1) ? 0 : 1;
                p.conv.dh = (kh == 0) ? -1 : 0;
            }
            p.dst = dw + (kh * 3 + kw);
            rc = run_wgrad(p, Cout, Cin, (cudaStream_t)stream_);
            if (rc) return rc;
        }
    return HCP_OK;
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
