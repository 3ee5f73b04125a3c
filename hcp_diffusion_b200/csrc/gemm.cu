// SPDX-License-Identifier: Apache-2.0
// wgmma + TMA GEMM / implicit-GEMM 3x3 convolution for sm_90a.
//
//   out[M,N] = sum_s A_s[M,K_s] . B_s[N,K_s]^T + bias[N] + rowbias[row/rows_per_group, N] + residual[M,N]
//
// Persistent kernel, one CTA per SM walking 128 x BN work items.  Warp roles (288 threads):
//   warps 0-7 : two MMA warpgroups; warpgroup g issues wgmma.mma_async for rows [64g, 64g+64) of the tile (fp32 accumulators in
//               registers) and runs the epilogue of those rows (fused bias / per-image bias / residual, bf16 stores)
//   warp 8    : TMA producer (one elected lane; A and B tiles of 64 K-elements per stage, SWIZZLE_128B), which runs ahead into the
//               next work item while the warpgroups drain the current one
//
// hcpdiff's LoRA (reference: hcpdiff/models/lora_layers_patch.py:44-57) reaches this kernel in two forms: adapters that apply to all
// rows are merged into the weight operand once per step (misc.cu: lora_merge_kernel) and their rank products T / U leave as a second
// output (`out2`: extra rows of the operand); DreamArtist++ adapters enter as an extra K-segment A_1 = (x . W_down^T) [M, 64-padded],
// B_1 = alpha * W_up [N, 64-padded], of which only ceil(r/16) k-steps are issued.
//
// The 3x3 convolution uses the same pipeline: the A tile of tap (kh,kw) and channel block c is a 4D (or 5D
// for stride 2) TMA box over the NHWC activation at a shifted coordinate; coordinates outside the image are
// zero-filled by the TMA unit, which IS the padding.  B is the weight matrix [Cout, 9*Cin].
#include <stdlib.h>
#include "common.cuh"
#include "host_util.h"
#include "../../include/hcp_b200.h"

namespace hcp {

constexpr int BLOCK_M = 128;
constexpr int BLOCK_K = 64;
constexpr int A_STAGE_BYTES = BLOCK_M * BLOCK_K * 2;
constexpr int kGemmMmaThreads = 256;     // two MMA warpgroups
constexpr int kGemmThreads = kGemmMmaThreads + 32;   // + the TMA producer warp
constexpr int kMaxTaps = 9;

struct TapEntry {
    int32_t c0_off;   // added to the innermost (channel) coordinate of A (stride-2: phase_w * Cin)
    int32_t dw;       // added to the W coordinate
    int32_t dh;       // added to the H coordinate
    int32_t c2;       // 5D only: the H-phase coordinate
    int32_t wk_off;   // K offset of this tap inside the weight matrix
};

struct alignas(64) GemmKParams {
    CUtensorMap tmA[HCP_GEMM_MAX_SEG];
    CUtensorMap tmB[HCP_GEMM_MAX_SEG];
    int32_t nkb[HCP_GEMM_MAX_SEG];     // 64-wide k-blocks per segment (conv: per tap)
    int32_t klast[HCP_GEMM_MAX_SEG];   // 16-wide k-steps issued in the last k-block of the segment (1..4)
    int32_t nseg;
    int32_t btile;                     // bit s: B of segment s is k-block-major [K/64][rows][64] (3D tensor map, coordinate 2 = k-block)
    int32_t M, N;
    int32_t tiles_n, tiles_m;
    // convolution geometry (conv == 0: plain GEMM)
    int32_t conv;                      // 0 none, 4 = 4D A map, 5 = 5D A map
    int32_t ntaps;
    TapEntry taps[kMaxTaps];
    int32_t bw, bh, bn;                // box (w, h, images) of one M tile, bw*bh*bn == 128
    int32_t tiles_w, tiles_h;          // tiles per image
    int32_t oW, oH;                    // output feature-map extent (rows of `out` are (img, y, x))
    int32_t sh, sw, oh0, ow0;          // output pixel of tile pixel (h,w) is (h*sh+oh0, w*sw+ow0)
    // epilogue
    const float* bias;
    const float* rowbias;
    int32_t rows_per_group;
    int64_t rowbias_ld;
    const __nv_bfloat16* residual;
    int64_t ldr;
    __nv_bfloat16* out;
    int64_t ldo;
    // columns >= n_main of the result are a SECOND output (the rank-r LoRA products T = x A^T / U = dY (alpha B) riding the layer's own
    // GEMM as extra rows of its weight operand): stored raw (no bias / residual) to out2[row, col - n_main]; out2 == NULL: n_main = N
    __nv_bfloat16* out2;
    int64_t ldo2;
    int32_t n_main;
    // split-K: CTA (x, y) reduces the k-blocks [y*kb_per_split, (y+1)*kb_per_split) and stores raw fp32 partials
    int32_t splits, kb_per_split;
    float* ws;                         // [splits, M, N] fp32
};

// BN = columns of a work item = N of every wgmma (a multiple of 16, at most 256); each MMA warpgroup holds 64 x BN fp32
// accumulators (BN / 2 registers per thread).
template <int BN>
struct GemmCfg {
    static constexpr int B_STAGE_BYTES = BN * BLOCK_K * 2;
    static constexpr int STAGE_BYTES = A_STAGE_BYTES + B_STAGE_BYTES;
    static constexpr int FIXED_BYTES = 256 /*barriers*/ + 1024 /*align*/;
    static constexpr int MAX_STAGES = (227 * 1024 - FIXED_BYTES) / STAGE_BYTES;
    // one CTA per SM: the ring must cover the TMA latency alone
    static constexpr int STAGES = MAX_STAGES > 6 ? 6 : MAX_STAGES;
    static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + FIXED_BYTES;
    static_assert(BN % 16 == 0 && BN <= 256, "wgmma N");
    static_assert(STAGES >= 3, "pipeline too shallow");
};

struct TileOrigin {
    int m0, img0, h0, w0;
};

// The output geometry of a launch, copied out of the parameter block BEFORE griddepcontrol.wait, so that the first touch of the
// constant-bank lines of the parameter block overlaps the previous kernel's tail.
struct TileGeom {
    int conv, bw, bh, bn, tiles_w, tiles_h, oW, oH, sh, sw, oh0, ow0, rows_per_group;
    __device__ __forceinline__ explicit TileGeom(const GemmKParams& p)
        : conv(p.conv), bw(p.bw), bh(p.bh), bn(p.bn), tiles_w(p.tiles_w), tiles_h(p.tiles_h), oW(p.oW), oH(p.oH), sh(p.sh), sw(p.sw),
          oh0(p.oh0), ow0(p.ow0), rows_per_group(p.rows_per_group) {}
};

__device__ __forceinline__ TileOrigin tile_origin(const TileGeom& p, int m_tile) {
    TileOrigin o{m_tile * BLOCK_M, 0, 0, 0};
    if (p.conv) {
        if (p.bn == 1) {
            const int per_img = p.tiles_w * p.tiles_h;
            o.img0 = m_tile / per_img;
            const int r = m_tile % per_img;
            o.h0 = (r / p.tiles_w) * p.bh;
            o.w0 = (r % p.tiles_w) * p.bw;
        } else {
            o.img0 = m_tile * p.bn;
        }
    }
    return o;
}
// row r of the tile -> row of `out` (and the per-image bias group)
__device__ __forceinline__ int64_t tile_row(const TileGeom& p, const TileOrigin& o, int r, int& group) {
    if (p.conv) {
        const int per = p.bw * p.bh;
        const int im = o.img0 + r / per;
        const int rr = r % per;
        const int hh = o.h0 + rr / p.bw;
        const int ww = o.w0 + rr % p.bw;
        group = im;
        return (int64_t)im * p.oH * p.oW + (int64_t)(hh * p.sh + p.oh0) * p.oW + (ww * p.sw + p.ow0);
    }
    const int64_t g = o.m0 + r;
    group = p.rows_per_group > 0 ? (int)(g / p.rows_per_group) : 0;
    return g;
}

// Position of a k-block inside a work item's reduction: (segment s, tap t of the convolution segment, k-block kb of nkb_s).
struct KPos {
    int s, t, kb, nkb_s;
};
// The reduction of a work item, held in REGISTERS of the producer and the MMA warpgroups: dynamically indexed loads from the
// kernel-parameter block (p.nkb[s], p.klast[s], p.taps[t]...) are slow constant-bank accesses.  A split seeks its first k-block
// directly and advances incrementally.
struct KPlan {
    int nkb0, nkb1, nkb2, kl0, kl1, kl2, ntap0, seg0, total_kb, conv, btile, kb_per_split;
    __device__ __forceinline__ explicit KPlan(const GemmKParams& p) {
        nkb0 = p.nkb[0]; nkb1 = p.nkb[1]; nkb2 = p.nkb[2];
        kl0 = p.klast[0]; kl1 = p.klast[1]; kl2 = p.klast[2];
        conv = p.conv; btile = p.btile; kb_per_split = p.kb_per_split;
        ntap0 = conv ? p.ntaps : 1;
        seg0 = nkb0 * ntap0;
        total_kb = seg0 + nkb1 + nkb2;
    }
    __device__ __forceinline__ int klast(int s) const { return s == 0 ? kl0 : (s == 1 ? kl1 : kl2); }
    __device__ __forceinline__ KPos seek(int it) const {
        KPos q;
        if (it < seg0) { q.s = 0; q.nkb_s = nkb0; q.t = it / nkb0; q.kb = it - q.t * nkb0; }
        else if (it < seg0 + nkb1) { q.s = 1; q.nkb_s = nkb1; q.t = 0; q.kb = it - seg0; }
        else { q.s = 2; q.nkb_s = nkb2; q.t = 0; q.kb = it - seg0 - nkb1; }
        return q;
    }
    // next k-block; true when a new tap of the convolution segment begins (the caller reloads its TapEntry)
    __device__ __forceinline__ bool advance(KPos& q) const {
        if (++q.kb < q.nkb_s) return false;
        q.kb = 0;
        if (q.s == 0 && q.t + 1 < ntap0) { ++q.t; return true; }
        ++q.s; q.t = 0;
        q.nkb_s = (q.s == 1) ? nkb1 : nkb2;
        return false;
    }
};

// Persistent kernel: grid = min(#work items, #SMs) CTAs; a work item is (split, m_tile, n_tile) with n fastest so that the CTAs
// running concurrently share A tiles in L2.  The producer runs up to STAGES k-blocks ahead, across work items, so the next item's
// operands stream in while the warpgroups run the epilogue of the current one.  Split-K items store raw fp32 partials
// (splitk_finalize_kernel applies bias / residual).
template <int BN>
__global__ void __launch_bounds__(kGemmThreads, 1) gemm_wgmma_kernel(const __grid_constant__ GemmKParams p) {
    using Cfg = GemmCfg<BN>;
    constexpr int STAGES = Cfg::STAGES;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint8_t* sA = smem;
    uint8_t* sB = smem + STAGES * A_STAGE_BYTES;
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(sB + STAGES * Cfg::B_STAGE_BYTES);
    uint64_t* empty_bar = full_bar + STAGES;

    const int warp = warp_id_uniform();
    const int lane = threadIdx.x & 31;
    const int tiles_mn = p.tiles_n * p.tiles_m;      // work items per split
    const int total_work = tiles_mn * p.splits;

    if (threadIdx.x == 0) {
        for (int s = 0; s < STAGES; ++s) {
            mbar_init(&full_bar[s], 1);
            mbar_init(&empty_bar[s], kGemmMmaThreads);
        }
        fence_mbar_init();
        for (int s = 0; s < p.nseg; ++s) {
            tma_prefetch_desc(&p.tmA[s]);
            tma_prefetch_desc(&p.tmB[s]);
        }
    }
    __syncthreads();
    // parameter block -> registers while the previous kernel of the stream is still draining
    const KPlan kq(p);
    const TileGeom geo(p);
    const int tiles_n = p.tiles_n;
    pdl_trigger();
    pdl_wait();     // the set-up above overlapped the previous kernel's tail; its results are visible from here on

    if (warp == kGemmMmaThreads / 32) {
        // ===================================== TMA producer =====================================
        if (elect_one()) {
            int stage = 0;
            uint32_t phase = 0;
            for (int w = blockIdx.x; w < total_work; w += gridDim.x) {
                const int split = w / tiles_mn, mn = w % tiles_mn;
                const int n0 = (mn % tiles_n) * BN;
                const TileOrigin o = tile_origin(geo, mn / tiles_n);
                const int kb_lo = split * kq.kb_per_split, kb_hi = min(kb_lo + kq.kb_per_split, kq.total_kb);
                KPos q = kq.seek(kb_lo);
                TapEntry te = p.taps[q.t];
                for (int it = kb_lo; it < kb_hi; ++it) {
                    const int s = q.s, kb = q.kb;
                    const bool tap_seg = kq.conv && s == 0;
                    mbar_wait(&empty_bar[stage], phase ^ 1);
                    void* dA = sA + stage * A_STAGE_BYTES;
                    void* dB = sB + stage * Cfg::B_STAGE_BYTES;
                    const int kcol = (tap_seg ? te.wk_off : 0) + kb * BLOCK_K;
                    mbar_arrive_expect_tx(&full_bar[stage], Cfg::STAGE_BYTES);
                    if (tap_seg) {
                        if (kq.conv == 4)
                            tma_load_4d(dA, &p.tmA[0], &full_bar[stage], te.c0_off + kb * BLOCK_K, o.w0 + te.dw, o.h0 + te.dh, o.img0);
                        else
                            tma_load_5d(dA, &p.tmA[0], &full_bar[stage], te.c0_off + kb * BLOCK_K, o.w0 + te.dw, te.c2, o.h0 + te.dh, o.img0);
                    } else {
                        tma_load_2d(dA, &p.tmA[s], &full_bar[stage], kb * BLOCK_K, o.m0);
                    }
                    if ((kq.btile >> s) & 1) tma_load_3d(dB, &p.tmB[s], &full_bar[stage], 0, n0, kcol / BLOCK_K);
                    else tma_load_2d(dB, &p.tmB[s], &full_bar[stage], kcol, n0);
                    if (++stage == STAGES) { stage = 0; phase ^= 1; }
                    if (kq.advance(q)) te = p.taps[q.t];
                }
            }
        }
        return;
    }

    // ===================================== MMA warpgroups + epilogue =====================================
    const int wg = warp >> 2;                     // rows [64 wg, 64 wg + 64) of the tile
    const int r_lo = wg * 64 + (warp & 3) * 16 + (lane >> 2);   // accumulator rows of this thread: r_lo and r_lo + 8
    const int cq = 2 * (lane & 3);                       // first of the two adjacent columns per 8-column group
    const int N = p.N, n_main = p.n_main;
    const int64_t Mrows = p.M, ldo = p.ldo, ldr = p.ldr, ldo2 = p.ldo2, rowbias_ld = p.rowbias_ld;
    const float* const bias = p.bias;
    const float* const rowbias = p.rowbias;
    const __nv_bfloat16* const res = p.residual;
    __nv_bfloat16* const out = p.out;
    __nv_bfloat16* const out2 = p.out2;
    float* const ws = p.ws;
    const bool split_k = p.splits > 1;
    int stage = 0;
    uint32_t phase = 0;
    for (int w = blockIdx.x; w < total_work; w += gridDim.x) {
        const int split = w / tiles_mn, mn = w % tiles_mn;
        const int n0 = (mn % tiles_n) * BN;
        const int kb_lo = split * kq.kb_per_split, kb_hi = min(kb_lo + kq.kb_per_split, kq.total_kb);
        float acc[BN / 2];
#pragma unroll
        for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
        KPos q = kq.seek(kb_lo);
        int held = -1;                                   // stage whose operands the wgmma group in flight still reads
        for (int it = kb_lo; it < kb_hi; ++it) {
            mbar_wait(&full_bar[stage], phase);
            const uint64_t adesc = make_smem_desc(smem_u32(sA + stage * A_STAGE_BYTES + wg * 64 * 128), 16, 1024);
            const uint64_t bdesc = make_smem_desc(smem_u32(sB + stage * Cfg::B_STAGE_BYTES), 16, 1024);
            const int ksteps = (q.kb == q.nkb_s - 1) ? kq.klast(q.s) : (BLOCK_K / 16);
            wgmma_fence();
            // +32 bytes (= 2 in descriptor units) per 16-element k-step inside the swizzle atom
            wgmma_ss<BN, 0, 0>(acc, adesc, bdesc, 1u);
            for (int k = 1; k < ksteps; ++k) wgmma_ss<BN, 0, 0>(acc, desc_adv(adesc, 2 * k), desc_adv(bdesc, 2 * k), 1u);
            wgmma_commit();
            wgmma_wait<1>();                             // the previous k-block's group has retired: its stage goes back to the producer
            if (held >= 0) mbar_arrive(&empty_bar[held]);
            held = stage;
            if (++stage == STAGES) { stage = 0; phase ^= 1; }
            kq.advance(q);
        }
        wgmma_wait<0>();
        wgmma_fence_acc(acc);
        if (held >= 0) mbar_arrive(&empty_bar[held]);

        // rows of `out` behind this thread's two accumulator rows (-1: beyond M)
        const TileOrigin o = tile_origin(geo, mn / tiles_n);
        int64_t grow[2];
        int group[2];
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            grow[h] = tile_row(geo, o, r_lo + 8 * h, group[h]);
            if (grow[h] >= Mrows) grow[h] = -1;
        }
        if (split_k) {
#pragma unroll
            for (int j = 0; j < BN / 8; ++j) {
                const int col = n0 + 8 * j + cq;
                if (col >= N) continue;
#pragma unroll
                for (int h = 0; h < 2; ++h)
                    if (grow[h] >= 0)
                        *reinterpret_cast<float2*>(ws + ((int64_t)split * Mrows + grow[h]) * N + col) = make_float2(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]);
            }
            continue;
        }
#pragma unroll
        for (int j = 0; j < BN / 8; ++j) {
            const int col = n0 + 8 * j + cq;
            if (col >= N) continue;
            if (col < n_main) {
                float b0 = 0.f, b1 = 0.f;
                if (bias) { b0 = __ldg(bias + col); b1 = __ldg(bias + col + 1); }
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    if (grow[h] < 0) continue;
                    float f0 = acc[4 * j + 2 * h] + b0, f1 = acc[4 * j + 2 * h + 1] + b1;
                    if (rowbias) {
                        const float* rb = rowbias + (int64_t)group[h] * rowbias_ld + col;
                        f0 += __ldg(rb); f1 += __ldg(rb + 1);
                    }
                    if (res) {
                        const float2 t = unpack_bf16x2(*reinterpret_cast<const uint32_t*>(res + grow[h] * ldr + col));
                        f0 += t.x; f1 += t.y;
                    }
                    *reinterpret_cast<uint32_t*>(out + grow[h] * ldo + col) = pack_bf16x2(f0, f1);
                }
            } else {
#pragma unroll
                for (int h = 0; h < 2; ++h)
                    if (grow[h] >= 0)
                        *reinterpret_cast<uint32_t*>(out2 + grow[h] * ldo2 + (col - n_main)) = pack_bf16x2(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]);
            }
        }
    }
}

// out = sum_s ws[s] + bias + rowbias + residual  (bf16), 8 columns per thread
__global__ void splitk_finalize_kernel(const float* __restrict__ ws, int splits, int64_t M, int N, const float* __restrict__ bias,
                                       const float* __restrict__ rowbias, int rows_per_group, int64_t rowbias_ld,
                                       const __nv_bfloat16* __restrict__ residual, int64_t ldr, __nv_bfloat16* __restrict__ out, int64_t ldo) {
    pdl_trigger();
    pdl_wait();
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    const int nv = N / 8;
    if (i >= M * nv) return;
    const int64_t row = i / nv;
    const int col = (int)(i % nv) * 8;
    float f[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    for (int s0 = 0; s0 < splits; s0 += 4) {                     // four partials in flight per thread (fixed summation order)
        float4 a[4], b[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int s = (s0 + j < splits) ? s0 + j : s0;         // clamp: the duplicate is not added below
            const float* src = ws + ((int64_t)s * M + row) * N + col;
            a[j] = *reinterpret_cast<const float4*>(src);
            b[j] = *reinterpret_cast<const float4*>(src + 4);
        }
#pragma unroll
        for (int j = 0; j < 4; ++j)
            if (s0 + j < splits) {
                f[0] += a[j].x; f[1] += a[j].y; f[2] += a[j].z; f[3] += a[j].w;
                f[4] += b[j].x; f[5] += b[j].y; f[6] += b[j].z; f[7] += b[j].w;
            }
    }
    if (bias) {
#pragma unroll
        for (int j = 0; j < 8; ++j) f[j] += bias[col + j];
    }
    if (rowbias) {
        const float* rb = rowbias + (rows_per_group > 0 ? row / rows_per_group : 0) * rowbias_ld + col;
#pragma unroll
        for (int j = 0; j < 8; ++j) f[j] += rb[j];
    }
    if (residual) {
        const uint4 rv = *reinterpret_cast<const uint4*>(residual + row * ldr + col);
        float2 t;
        t = unpack_bf16x2(rv.x); f[0] += t.x; f[1] += t.y;
        t = unpack_bf16x2(rv.y); f[2] += t.x; f[3] += t.y;
        t = unpack_bf16x2(rv.z); f[4] += t.x; f[5] += t.y;
        t = unpack_bf16x2(rv.w); f[6] += t.x; f[7] += t.y;
    }
    uint4 o;
    o.x = pack_bf16x2(f[0], f[1]); o.y = pack_bf16x2(f[2], f[3]); o.z = pack_bf16x2(f[4], f[5]); o.w = pack_bf16x2(f[6], f[7]);
    *reinterpret_cast<uint4*>(out + row * ldo + col) = o;
}

// number of K-splits for a launch with `ctas` output tiles and `total_kb` 64-wide k-blocks (1 = no split)
static int plan_splits(int64_t ctas, int64_t total_kb, int64_t N) {
    // splitting costs a second (finalize) launch and an fp32 round trip: never for the skinny LoRA projections or short reductions
    if (total_kb < 8 || N <= 64) return 1;
    const int64_t sms = num_sms();
    if (ctas >= sms / 3) {
        // a third to a half of the SMs busy for the whole reduction: two K halves fill them, worth it when each half is still a long
        // main loop (>= 20 k-blocks): the 16x16 / 8x8 level convolutions and the K >= 2560 linears at M = 1024
        return (ctas <= sms / 2 && total_kb >= 40) ? 2 : 1;
    }
    int64_t s = sms / ctas;                 // persistent grid: keep the work items within one wave of SMs
    if (s > total_kb / 4) s = total_kb / 4;
    if (s > 16) s = 16;
    return s < 2 ? 1 : (int)s;
}

// =============================================================================================
// LoRA gradients on the tensor pipe:  D[n, j] = sum_m X[m, n] * S[m, j]   (reduction over the M token rows)
//   dW_down[j, k] = sum_m U[m, c0+j] x[m, k]          S = U = dY . (alpha B),  X = x
//   dW_up[o, j]   = alpha * sum_m dY[m, o0+o] T[m, c0+j]   S = T = x . A^T,        X = dY
// Both operands are read straight from their row-major [M, *] tensors as MN-major wgmma operands (TMA boxes of 64 columns x
// 128 rows), so no transpose ever exists.  One CTA owns 128 columns of X and a slice of the rows (split-K); MMA warpgroup g
// accumulates the 64 x 64 fp32 block of X columns [64g, 64g+64) and reduces it into the flat gradient buffer with atomics.
// =============================================================================================
constexpr int kLgThreads = 288;   // warps 0-7: two MMA warpgroups, warp 8: TMA
constexpr int LG_STAGES = 3;
constexpr int LG_STAGE_BYTES = 3 * 128 * 128;      // two X boxes + one S box
constexpr int LG_SMEM_BYTES = LG_STAGES * LG_STAGE_BYTES + 256 + 1024;
constexpr int LG_MAX_BLOCKS = 8;

struct LGBlock {
    int32_t n_lo, n_hi, c0, rank, transpose_out, dst_ld;
    int32_t n_stride;        // element stride of the X-column index in the destination (1; 9 for the taps of a 3x3 W_down)
    float scale;
    float* dst;
};
// X operand = shifted im2col box of a 3x3 convolution (dW_down of a Conv2d LoRA): same boxes as the forward conv's A operand
struct LGConv {
    int32_t rank;            // 0: plain [M, ldx] matrix; 4 / 5: rank of the NHWC tensor map
    int32_t bw, bh, bn, tiles_w, tiles_h;
    int32_t c0_off, dw, dh, c2;
};
struct LGProblem {
    int32_t n_begin, n_end, tiles_per_cta, nblocks, col_chunks, splits;
    LGBlock blk[LG_MAX_BLOCKS];
};
struct alignas(64) LoraGradParams {
    CUtensorMap tmX[2], tmS[2];        // up to two independent problems per launch (dW_down and dW_up of one group)
    int32_t M, nprob;
    LGProblem prob[2];
    LGConv conv;
};

__global__ void __launch_bounds__(kLgThreads, 1) lora_grad_tc_kernel(const __grid_constant__ LoraGradParams p) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + LG_STAGES * LG_STAGE_BYTES);
    uint64_t* empty_bar = full_bar + LG_STAGES;
    const int warp = warp_id_uniform(), lane = threadIdx.x & 31;
    // flat grid over (problem, column chunk, row split)
    int bid = blockIdx.x, z = 0;
    if (p.nprob == 2 && bid >= p.prob[0].col_chunks * p.prob[0].splits) { bid -= p.prob[0].col_chunks * p.prob[0].splits; z = 1; }
    // The reduction epilogue walks `p.prob[z].blk[b]` with run-time z and b (dynamically indexed constant-bank loads): the MMA
    // threads copy the descriptor to shared memory first; the producer only needs the scalars read here.
    __shared__ LGProblem sq;
    const LGProblem& q = z ? p.prob[1] : p.prob[0];
    const CUtensorMap* tmX = z ? &p.tmX[1] : &p.tmX[0];
    const CUtensorMap* tmS = z ? &p.tmS[1] : &p.tmS[0];
    const int ncol0 = q.n_begin + (bid % q.col_chunks) * 128;
    const int total_tiles = (p.M + 127) / 128;
    const int t0 = (bid / q.col_chunks) * q.tiles_per_cta;
    const int t1 = min(total_tiles, t0 + q.tiles_per_cta);

    if (threadIdx.x == 0) {
        for (int s = 0; s < LG_STAGES; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], 256); }
        fence_mbar_init();
    }
    __syncthreads();
    pdl_trigger();
    pdl_wait();

    if (warp == 8) {
        if (elect_one()) {
            int stage = 0; uint32_t phase = 0;
            for (int t = t0; t < t1; ++t) {
                mbar_wait(&empty_bar[stage], phase ^ 1);
                mbar_arrive_expect_tx(&full_bar[stage], LG_STAGE_BYTES);
                uint8_t* base = smem + stage * LG_STAGE_BYTES;
                if (p.conv.rank == 0) {
                    tma_load_2d(base, tmX, &full_bar[stage], ncol0, t * 128);
                    tma_load_2d(base + 128 * 128, tmX, &full_bar[stage], ncol0 + 64, t * 128);
                } else {
                    const LGConv& cv = p.conv;
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
                        if (cv.rank == 4) tma_load_4d(base + hf * 128 * 128, tmX, &full_bar[stage], c, w0 + cv.dw, h0 + cv.dh, img0);
                        else tma_load_5d(base + hf * 128 * 128, tmX, &full_bar[stage], c, w0 + cv.dw, cv.c2, h0 + cv.dh, img0);
                    }
                }
                tma_load_2d(base + 2 * 128 * 128, tmS, &full_bar[stage], 0, t * 128);
                if (++stage == LG_STAGES) { stage = 0; phase ^= 1; }
            }
        }
        return;
    }
    {   // descriptor -> shared memory
        const uint32_t* src = reinterpret_cast<const uint32_t*>(&q);
        uint32_t* dst = reinterpret_cast<uint32_t*>(&sq);
        for (int i = threadIdx.x; i < (int)(sizeof(LGProblem) / 4); i += 256) dst[i] = src[i];
        asm volatile("bar.sync 1, 256;" ::: "memory");
    }
    const int wg = warp >> 2;
    float acc[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) acc[i] = 0.f;
    int stage = 0; uint32_t phase = 0;
    for (int t = t0; t < t1; ++t) {
        mbar_wait(&full_bar[stage], phase);
        const uint32_t xb = smem_u32(smem + stage * LG_STAGE_BYTES) + wg * 128 * 128;   // this warpgroup's 64 X columns
        const uint32_t sb = smem_u32(smem + stage * LG_STAGE_BYTES) + 2 * 128 * 128;
        wgmma_fence();
#pragma unroll
        for (int ks = 0; ks < 8; ++ks)                                   // 16 token rows per k-step = 2048 B
            wgmma_ss<64, 1, 1>(acc, make_smem_desc(xb + ks * 2048, 128 * 128, 1024), make_smem_desc(sb + ks * 2048, 128 * 128, 1024), 1u);
        wgmma_commit();
        wgmma_wait<0>();
        mbar_arrive(&empty_bar[stage]);
        if (++stage == LG_STAGES) { stage = 0; phase ^= 1; }
    }
    wgmma_fence_acc(acc);
    if (t1 <= t0) return;
    const LGProblem& qs = sq;
    const int n_lo_row = ncol0 + wg * 64 + (warp & 3) * 16 + (lane >> 2);
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        const int n = n_lo_row + 8 * h;                                  // column of X
        if (n >= qs.n_end) continue;
        for (int b = 0; b < qs.nblocks; ++b) {
            const LGBlock& k = qs.blk[b];
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
}

// ---------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------
template <int BN>
static int launch_gemm(const GemmKParams& kp, cudaStream_t stream) {
    using Cfg = GemmCfg<BN>;
    static bool configured = false;
    if (!configured) {
        cudaError_t e = cudaFuncSetAttribute(gemm_wgmma_kernel<BN>, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM_BYTES);
        if (e != cudaSuccess) return set_cuda_error(e, "cudaFuncSetAttribute(gemm)");
        configured = true;
    }
    const int total = kp.tiles_n * kp.tiles_m * kp.splits;
    const int workers = num_sms();
    launch_k(gemm_wgmma_kernel<BN>, dim3(total < workers ? total : workers), dim3(kGemmThreads), Cfg::SMEM_BYTES, stream, kp);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return set_cuda_error(e, "gemm launch");
    return HCP_OK;
}

static int pick_bn(int64_t N) {
    if (N <= 32) return 32;
    if (N <= 64) return 64;
    if (N % 64 == 0 && N < 256 && N % 128 != 0) return 64;
    // 160 divides every channel count of the UNet; 176 covers a layer whose weight operand carries its LoRA down-projection as extra
    // rows (N + 8..16 per 160 columns) without an extra column tile; the least padded width wins, ties go to the fewer tiles
    int best = 128;
    int64_t best_w = (N + 127) / 128 * 128;
    const int cand[2] = {160, 176};
    for (int c : cand) {
        const int64_t w = (N + c - 1) / c * c;
        if (w < best_w || (w == best_w && c > best)) { best = c; best_w = w; }
    }
    return best;
}

static int dispatch_gemm(int bn, GemmKParams& kp, int m_tiles, cudaStream_t stream) {
    kp.tiles_m = m_tiles;
    switch (bn) {
        case 32: return launch_gemm<32>(kp, stream);
        case 64: return launch_gemm<64>(kp, stream);
        case 128: return launch_gemm<128>(kp, stream);
        case 160: return launch_gemm<160>(kp, stream);
        case 176: return launch_gemm<176>(kp, stream);
        default: return set_error(HCP_ERR_INVALID, "unsupported BLOCK_N");
    }
}

// plain or split-K launch (+ finalize).  `ws` may be NULL / too small: then the launch is not split.
static int run_gemm(int bn, GemmKParams& kp, int m_tiles, int64_t total_kb, float* ws, size_t ws_bytes, bool allow_split, cudaStream_t stream) {
    int splits = !allow_split ? 1 : plan_splits((int64_t)m_tiles * kp.tiles_n, total_kb, kp.N);
    if (splits > 1 && (!ws || ws_bytes < (size_t)splits * kp.M * kp.N * sizeof(float))) splits = 1;
    if (splits > 1) {
        kp.kb_per_split = (int)((total_kb + splits - 1) / splits);
        splits = (int)((total_kb + kp.kb_per_split - 1) / kp.kb_per_split);
    }
    if (splits <= 1) {
        kp.splits = 1;
        kp.kb_per_split = 1 << 30;
        kp.ws = nullptr;
        return dispatch_gemm(bn, kp, m_tiles, stream);
    }
    kp.splits = splits;
    kp.ws = ws;
    int rc = dispatch_gemm(bn, kp, m_tiles, stream);
    if (rc) return rc;
    const int64_t n = (int64_t)kp.M * (kp.N / 8);
    launch_k(splitk_finalize_kernel, dim3((unsigned)((n + 255) / 256)), dim3(256), 0, stream, ws, splits, kp.M, kp.N, kp.bias, kp.rowbias,
                                                                            kp.conv ? kp.oH * kp.oW : kp.rows_per_group, kp.rowbias_ld,
                                                                            kp.residual, kp.ldr, kp.out, kp.ldo);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return set_cuda_error(e, "splitk finalize launch");
    return HCP_OK;
}

}  // namespace hcp

using namespace hcp;

extern "C" size_t hcp_splitk_workspace_bytes(int64_t M, int64_t N, int64_t total_k) {
    const int bn = pick_bn(N);
    const int64_t m_tiles = (M + BLOCK_M - 1) / BLOCK_M;
    const int64_t ctas = m_tiles * ((N + bn - 1) / bn);
    const int splits = plan_splits(ctas, (total_k + BLOCK_K - 1) / BLOCK_K, N);
    return splits > 1 ? (size_t)splits * M * N * sizeof(float) : 0;
}
extern "C" int hcp_gemm_bf16(const hcp_gemm_args* a, hcp_stream_t stream_) {
    if (!a || a->nseg < 1 || a->nseg > HCP_GEMM_MAX_SEG) return set_error(HCP_ERR_INVALID, "gemm: nseg");
    if (a->M <= 0 || a->N <= 0 || (a->N % 8) != 0) return set_error(HCP_ERR_INVALID, "gemm: M/N (N must be a multiple of 8)");
    if (!a->out || (a->ldo % 8) != 0) return set_error(HCP_ERR_INVALID, "gemm: out/ldo");
    if (a->residual && (a->ldr % 8) != 0) return set_error(HCP_ERR_INVALID, "gemm: ldr");
    GemmKParams kp;
    memset(&kp, 0, sizeof(kp));
    const int bn = pick_bn(a->N);
    const int b_box_rows = bn;       // rows of one TMA box of B
    for (int s = 0; s < a->nseg; ++s) {
        if (a->k[s] <= 0) return set_error(HCP_ERR_INVALID, "gemm: k must be positive");
        if ((a->lda[s] % 8) != 0 || (((a->flags >> s) & 1) == 0 && (a->ldb[s] % 8) != 0)) return set_error(HCP_ERR_INVALID, "gemm: lda/ldb");
        const int64_t nrb = a->n_rows_b[s] > 0 ? a->n_rows_b[s] : a->N;
        int rc = make_tmap_2d(&kp.tmA[s], a->a[s], (uint64_t)a->k[s], (uint64_t)a->M, (uint64_t)a->lda[s], BLOCK_K, BLOCK_M);
        if (rc) return rc;
        if ((a->flags >> s) & 1) {
            // k-block-major B: element (n, k) at b + ((k / 64) * ldb + n) * 64 + k % 64 -- every TMA box is ONE contiguous run of memory
            if (a->k[s] % BLOCK_K) return set_error(HCP_ERR_INVALID, "gemm: a k-block-major B operand needs k % 64 == 0");
            uint64_t dims[3] = {BLOCK_K, (uint64_t)nrb, (uint64_t)(a->k[s] / BLOCK_K)};
            uint64_t strides[2] = {BLOCK_K * 2, (uint64_t)a->ldb[s] * BLOCK_K * 2};
            uint32_t box[3] = {BLOCK_K, (uint32_t)b_box_rows, 1};
            rc = make_tmap_nd(&kp.tmB[s], a->b[s], 3, dims, strides, box);
            kp.btile |= 1 << s;
        } else {
            rc = make_tmap_2d(&kp.tmB[s], a->b[s], (uint64_t)a->k[s], (uint64_t)nrb, (uint64_t)a->ldb[s], BLOCK_K, b_box_rows);
        }
        if (rc) return rc;
        kp.nkb[s] = (int)((a->k[s] + BLOCK_K - 1) / BLOCK_K);
        const int64_t rem = a->k[s] - (int64_t)(kp.nkb[s] - 1) * BLOCK_K;
        kp.klast[s] = (int)((rem + 15) / 16);
    }
    kp.nseg = a->nseg;
    kp.M = (int)a->M;
    kp.N = (int)a->N;
    kp.tiles_n = (int)((a->N + bn - 1) / bn);
    kp.conv = 0;
    kp.bias = a->bias;
    kp.rowbias = a->rowbias;
    kp.rows_per_group = (int)a->rows_per_group;
    kp.rowbias_ld = a->rowbias_ld > 0 ? a->rowbias_ld : a->N;
    kp.residual = (const __nv_bfloat16*)a->residual;
    kp.ldr = a->ldr;
    kp.out = (__nv_bfloat16*)a->out;
    kp.ldo = a->ldo;
    kp.n_main = kp.N;
    if (a->out2) {
        if (a->n_main <= 0 || a->n_main >= a->N || (a->n_main % 8) != 0 || (a->ldo2 % 8) != 0) return set_error(HCP_ERR_INVALID, "gemm: out2 / n_main / ldo2");
        kp.out2 = (__nv_bfloat16*)a->out2;
        kp.ldo2 = a->ldo2;
        kp.n_main = (int)a->n_main;
    }
    const int m_tiles = (int)((a->M + BLOCK_M - 1) / BLOCK_M);
    int64_t total_kb = 0;
    for (int s = 0; s < a->nseg; ++s) total_kb += kp.nkb[s];
    return run_gemm(bn, kp, m_tiles, total_kb, a->workspace, a->workspace_bytes, a->out2 == nullptr, (cudaStream_t)stream_);
}

// Conv2d LoRA: out += T . Bl^T as K-segment 1 (plain 2D operands; the rows of an M tile of the convolution are contiguous pixels)
static int conv_lora_segment(const hcp_conv3x3_args* a, GemmKParams& kp, int b_box_rows) {
    if (!a->lora_t) return HCP_OK;
    if (!a->lora_b || a->lora_r <= 0 || a->lora_r > a->lora_ld || (a->lora_ld % 8) != 0)
        return set_error(HCP_ERR_INVALID, "conv3x3: LoRA segment (lora_b / lora_r / lora_ld)");
    int rc = make_tmap_2d(&kp.tmA[1], a->lora_t, (uint64_t)a->lora_r, (uint64_t)kp.M, (uint64_t)a->lora_ld, BLOCK_K, BLOCK_M);
    if (rc) return rc;
    rc = make_tmap_2d(&kp.tmB[1], a->lora_b, (uint64_t)a->lora_r, (uint64_t)a->Cout, (uint64_t)a->lora_ld, BLOCK_K, b_box_rows);
    if (rc) return rc;
    kp.nseg = 2;
    kp.nkb[1] = (int)((a->lora_r + BLOCK_K - 1) / BLOCK_K);
    kp.klast[1] = (int)((a->lora_r - (int64_t)(kp.nkb[1] - 1) * BLOCK_K + 15) / 16);
    return HCP_OK;
}

extern "C" int hcp_conv3x3_bf16(const hcp_conv3x3_args* a, hcp_stream_t stream_) {
    if (!a || !a->x || !a->w || !a->out) return set_error(HCP_ERR_INVALID, "conv3x3: null pointer");
    if (a->Cin % 64 != 0 || a->Cout % 8 != 0) return set_error(HCP_ERR_INVALID, "conv3x3: Cin %% 64, Cout %% 8 required");
    if (a->stride != 1 && a->stride != 2) return set_error(HCP_ERR_INVALID, "conv3x3: stride");
    if (a->mode != 0 && !(a->mode == 1)) return set_error(HCP_ERR_INVALID, "conv3x3: mode");
    GemmKParams kp;
    memset(&kp, 0, sizeof(kp));
    const int bn = pick_bn(a->Cout);
    const int64_t Cin = a->Cin;

    // geometry of the "tile grid" (the grid the 128-pixel M tiles walk over) and of the output map
    int64_t tH, tW;   // extent of the tile grid per image
    int64_t oH, oW;   // output feature map
    if (a->mode == 0) {
        if (a->stride == 2 && ((a->Hin | a->Win) & 1)) return set_error(HCP_ERR_INVALID, "conv3x3: odd extent with stride 2");
        oH = a->Hin / a->stride; oW = a->Win / a->stride;
        tH = oH; tW = oW;
    } else {
        oH = a->Hin * 2; oW = a->Win * 2;
        tH = a->Hin; tW = a->Win;   // one launch per output phase, tiles walk the dY grid
    }
    // box: bw*bh*bn == 128
    int bw, bh, bnimg;
    if (tW >= 128) { bw = 128; bh = 1; bnimg = 1; if (tW % 128) return set_error(HCP_ERR_INVALID, "conv3x3: W"); }
    else {
        bw = (int)tW;
        if (128 % bw) return set_error(HCP_ERR_INVALID, "conv3x3: W must divide 128");
        bh = 128 / bw;
        if (bh <= tH) { if (tH % bh) return set_error(HCP_ERR_INVALID, "conv3x3: H tiling"); bnimg = 1; }
        else { bh = (int)tH; if (128 % (bw * bh)) return set_error(HCP_ERR_INVALID, "conv3x3: H*W must divide 128"); bnimg = 128 / (bw * bh); }
    }
    kp.bw = bw; kp.bh = bh; kp.bn = bnimg;
    kp.tiles_w = (int)(tW / bw);
    kp.tiles_h = (int)(tH / bh);
    kp.oW = (int)oW; kp.oH = (int)oH;
    kp.nseg = 1;
    kp.nkb[0] = (int)(Cin / BLOCK_K);
    kp.klast[0] = 4;
    kp.N = (int)a->Cout;
    kp.M = (int)(a->B * oH * oW);
    kp.tiles_n = (int)((a->Cout + bn - 1) / bn);
    kp.bias = a->bias;
    kp.rowbias = a->rowbias;
    kp.rows_per_group = 0;
    kp.rowbias_ld = a->rowbias_ld > 0 ? a->rowbias_ld : a->Cout;
    kp.residual = (const __nv_bfloat16*)a->residual;
    kp.ldr = a->Cout;
    kp.out = (__nv_bfloat16*)a->out;
    kp.ldo = a->Cout;
    kp.n_main = (int)a->Cout;
    const int m_tiles = (bnimg == 1) ? (int)(a->B * kp.tiles_w * kp.tiles_h) : (int)((a->B + bnimg - 1) / bnimg);
    const int b_box_rows = bn;
    int rc;
    if (a->w_tiled) {          // k-block-major weights [9*Cin/64][Cout][64]
        uint64_t dims[3] = {BLOCK_K, (uint64_t)a->Cout, (uint64_t)(9 * Cin / BLOCK_K)};
        uint64_t strides[2] = {BLOCK_K * 2, (uint64_t)a->Cout * BLOCK_K * 2};
        uint32_t box[3] = {BLOCK_K, (uint32_t)b_box_rows, 1};
        rc = make_tmap_nd(&kp.tmB[0], a->w, 3, dims, strides, box);
        kp.btile = 1;
    } else {
        rc = make_tmap_2d(&kp.tmB[0], a->w, (uint64_t)(9 * Cin), (uint64_t)a->Cout, (uint64_t)(9 * Cin), BLOCK_K, b_box_rows);
    }
    if (rc) return rc;
    cudaStream_t stream = (cudaStream_t)stream_;

    if (a->mode == 0 && a->stride == 1) {
        kp.conv = 4;
        uint64_t dims[4] = {(uint64_t)Cin, (uint64_t)a->Win, (uint64_t)a->Hin, (uint64_t)a->B};
        uint64_t strides[3] = {(uint64_t)Cin * 2, (uint64_t)a->Win * Cin * 2, (uint64_t)a->Hin * a->Win * Cin * 2};
        uint32_t box[4] = {BLOCK_K, (uint32_t)bw, (uint32_t)bh, (uint32_t)bnimg};
        rc = make_tmap_nd(&kp.tmA[0], a->x, 4, dims, strides, box);
        if (rc) return rc;
        kp.ntaps = 9;
        for (int kh = 0; kh < 3; ++kh)
            for (int kw = 0; kw < 3; ++kw) {
                TapEntry& t = kp.taps[kh * 3 + kw];
                t.c0_off = 0; t.dw = kw - 1; t.dh = kh - 1; t.c2 = 0;
                t.wk_off = (int)((kh * 3 + kw) * Cin);
            }
        kp.sh = kp.sw = 1; kp.oh0 = kp.ow0 = 0;
        if ((rc = conv_lora_segment(a, kp, b_box_rows))) return rc;
        return run_gemm(bn, kp, m_tiles, (int64_t)9 * kp.nkb[0] + (kp.nseg > 1 ? kp.nkb[1] : 0), a->workspace, a->workspace_bytes, true, stream);
    }
    if (a->mode == 0 && a->stride == 2) {
        // view x as [B][Hin/2][2][Win/2][2*Cin]: input row ih = 2*oh + kh - 1 -> (phase, index)
        kp.conv = 5;
        uint64_t dims[5] = {(uint64_t)(2 * Cin), (uint64_t)(a->Win / 2), 2, (uint64_t)(a->Hin / 2), (uint64_t)a->B};
        uint64_t strides[4] = {(uint64_t)(2 * Cin) * 2, (uint64_t)a->Win * Cin * 2, (uint64_t)(2 * a->Win * Cin) * 2,
                               (uint64_t)a->Hin * a->Win * Cin * 2};
        uint32_t box[5] = {BLOCK_K, (uint32_t)bw, 1, (uint32_t)bh, (uint32_t)bnimg};
        rc = make_tmap_nd(&kp.tmA[0], a->x, 5, dims, strides, box);
        if (rc) return rc;
        kp.ntaps = 9;
        for (int kh = 0; kh < 3; ++kh)
            for (int kw = 0; kw < 3; ++kw) {
                TapEntry& t = kp.taps[kh * 3 + kw];
                const int pw = (kw == 1) ? 0 : 1, ph = (kh == 1) ? 0 : 1;
                t.c0_off = (int)(pw * Cin);
                t.dw = (kw == 0) ? -1 : 0;
                t.c2 = ph;
                t.dh = (kh == 0) ? -1 : 0;
                t.wk_off = (int)((kh * 3 + kw) * Cin);
            }
        kp.sh = kp.sw = 1; kp.oh0 = kp.ow0 = 0;
        if ((rc = conv_lora_segment(a, kp, b_box_rows))) return rc;
        return run_gemm(bn, kp, m_tiles, (int64_t)9 * kp.nkb[0] + (kp.nseg > 1 ? kp.nkb[1] : 0), a->workspace, a->workspace_bytes, true, stream);
    }
    if (a->lora_t) return set_error(HCP_ERR_INVALID, "conv3x3: the LoRA segment is only available in mode 0");
    // mode 1: dgrad of the stride-2 conv.  x = dY [B, Hin, Win, Cin] (Cin = Cout of the fwd conv),
    // out = dX [B, 2Hin, 2Win, Cout].  Output pixel (2i+ph, 2j+pw) gathers dY[i+dh, j+dw] over the taps whose
    // parity matches:  ph=0: kh=1 (dh=0);  ph=1: kh=0 (dh=+1), kh=2 (dh=0).   w[co][kh][kw][ci] here is the
    // dgrad weight = W_fwd[ci][kh][kw][co] (NOT flipped; the tap choice below does the bookkeeping).
    kp.conv = 4;
    {
        uint64_t dims[4] = {(uint64_t)Cin, (uint64_t)a->Win, (uint64_t)a->Hin, (uint64_t)a->B};
        uint64_t strides[3] = {(uint64_t)Cin * 2, (uint64_t)a->Win * Cin * 2, (uint64_t)a->Hin * a->Win * Cin * 2};
        uint32_t box[4] = {BLOCK_K, (uint32_t)bw, (uint32_t)bh, (uint32_t)bnimg};
        rc = make_tmap_nd(&kp.tmA[0], a->x, 4, dims, strides, box);
        if (rc) return rc;
    }
    kp.sh = kp.sw = 2;
    for (int ph = 0; ph < 2; ++ph)
        for (int pw = 0; pw < 2; ++pw) {
            int nt = 0;
            for (int kh = 0; kh < 3; ++kh) {
                if (((ph + 1 - kh) & 1) != 0) continue;
                for (int kw = 0; kw < 3; ++kw) {
                    if (((pw + 1 - kw) & 1) != 0) continue;
                    TapEntry& t = kp.taps[nt++];
                    t.c0_off = 0; t.c2 = 0;
                    t.dh = (ph + 1 - kh) / 2;
                    t.dw = (pw + 1 - kw) / 2;
                    t.wk_off = (int)((kh * 3 + kw) * Cin);
                }
            }
            kp.ntaps = nt;
            kp.oh0 = ph; kp.ow0 = pw;
            rc = run_gemm(bn, kp, m_tiles, 0, nullptr, 0, false, stream);
            if (rc) return rc;
        }
    return HCP_OK;
}

static int lg_fill(LoraGradParams& p, int z, const void* S, int64_t lds, const void* X, int64_t ldx, int64_t M, int64_t n_begin,
                   int64_t n_end, const hcp_lora_grad_block* blocks, int32_t nblocks, int target_ctas) {
    if (!S || !X || !blocks || nblocks < 1 || nblocks > LG_MAX_BLOCKS) return set_error(HCP_ERR_INVALID, "lora_grad: 1..8 blocks per problem");
    if (n_end <= n_begin || (ldx % 8) != 0 || (n_begin % 8) != 0 || lds < 64 || (lds % 8) != 0) return set_error(HCP_ERR_INVALID, "lora_grad: shape");
    int rc = make_tmap_2d(&p.tmX[z], X, (uint64_t)ldx, (uint64_t)M, (uint64_t)ldx, 64, 128);
    if (rc) return rc;
    rc = make_tmap_2d(&p.tmS[z], S, 64, (uint64_t)M, (uint64_t)lds, 64, 128);     // the 64 columns of S this launch reduces
    if (rc) return rc;
    LGProblem& q = p.prob[z];
    q.n_begin = (int)n_begin; q.n_end = (int)n_end; q.nblocks = nblocks;
    q.col_chunks = (int)((n_end - n_begin + 127) / 128);
    const int total_tiles = (int)((M + 127) / 128);
    int splits = target_ctas / q.col_chunks;     // at most one wave of CTAs over all problems of the launch
    if (splits < 1) splits = 1;
    if (splits > total_tiles) splits = total_tiles;
    q.tiles_per_cta = (total_tiles + splits - 1) / splits;
    q.splits = (total_tiles + q.tiles_per_cta - 1) / q.tiles_per_cta;
    for (int i = 0; i < nblocks; ++i) {
        const hcp_lora_grad_block& k = blocks[i];
        if (k.rank < 1 || k.c0 < 0 || k.c0 + k.rank > 64 || !k.dst) return set_error(HCP_ERR_INVALID, "lora_grad: block descriptor");
        q.blk[i].n_lo = (int)k.n_lo; q.blk[i].n_hi = (int)k.n_hi; q.blk[i].c0 = k.c0; q.blk[i].rank = k.rank;
        q.blk[i].transpose_out = k.transpose_out; q.blk[i].dst_ld = (int)k.dst_ld; q.blk[i].scale = k.scale; q.blk[i].dst = k.dst;
        q.blk[i].n_stride = 1;
    }
    return HCP_OK;
}

static int lg_launch(LoraGradParams& p, cudaStream_t stream) {
    static bool configured = false;
    if (!configured) {
        cudaError_t e = cudaFuncSetAttribute(lora_grad_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, LG_SMEM_BYTES);
        if (e != cudaSuccess) return set_cuda_error(e, "cudaFuncSetAttribute(lora_grad)");
        configured = true;
    }
    int ctas = 0;
    for (int z = 0; z < p.nprob; ++z) ctas += p.prob[z].col_chunks * p.prob[z].splits;
    launch_k(lora_grad_tc_kernel, dim3(ctas), dim3(kLgThreads), LG_SMEM_BYTES, stream, p);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return set_cuda_error(e, "lora_grad launch");
    return HCP_OK;
}

extern "C" int hcp_lora_grad(const void* S, int64_t lds, const void* X, int64_t ldx, int64_t M, int64_t n_begin, int64_t n_end,
                             const hcp_lora_grad_block* blocks, int32_t nblocks, hcp_stream_t stream_) {
    if (M <= 0) return set_error(HCP_ERR_INVALID, "lora_grad: M");
    LoraGradParams p;
    memset(&p, 0, sizeof(p));
    p.M = (int)M; p.nprob = 1;
    int rc = lg_fill(p, 0, S, lds, X, ldx, M, n_begin, n_end, blocks, nblocks, num_sms());
    if (rc) return rc;
    return lg_launch(p, (cudaStream_t)stream_);
}

// dW_down of a Conv2d LoRA: nine launches (one per tap) of the gradient kernel with the shifted NHWC box as X operand.
extern "C" int hcp_lora_grad_conv3x3(const void* S, int64_t lds, const void* x, int64_t B, int64_t Hin, int64_t Win, int64_t Cin,
                                     int32_t stride, const hcp_lora_grad_block* blocks, int32_t nblocks, hcp_stream_t stream_) {
    if (!S || !x || !blocks || nblocks < 1 || nblocks > LG_MAX_BLOCKS) return set_error(HCP_ERR_INVALID, "lora_grad_conv: arguments");
    if (Cin % 64 != 0 || (stride != 1 && stride != 2) || lds < 64 || (lds % 8) != 0) return set_error(HCP_ERR_INVALID, "lora_grad_conv: shape");
    if (stride == 2 && ((Hin | Win) & 1)) return set_error(HCP_ERR_INVALID, "lora_grad_conv: odd extent with stride 2");
    const int64_t oH = Hin / stride, oW = Win / stride;
    int bw, bh, bnimg;                       // same 128-pixel tiles as hcp_conv3x3_bf16 (mode 0)
    if (oW >= 128) { bw = 128; bh = 1; bnimg = 1; if (oW % 128) return set_error(HCP_ERR_INVALID, "lora_grad_conv: W"); }
    else {
        bw = (int)oW;
        if (128 % bw) return set_error(HCP_ERR_INVALID, "lora_grad_conv: W must divide 128");
        bh = 128 / bw;
        if (bh <= oH) { if (oH % bh) return set_error(HCP_ERR_INVALID, "lora_grad_conv: H tiling"); bnimg = 1; }
        else { bh = (int)oH; if (128 % (bw * bh)) return set_error(HCP_ERR_INVALID, "lora_grad_conv: H*W must divide 128"); bnimg = 128 / (bw * bh); }
    }
    LoraGradParams p;
    memset(&p, 0, sizeof(p));
    const int64_t M = B * oH * oW;
    p.M = (int)M; p.nprob = 1;
    int rc;
    if (stride == 1) {
        uint64_t dims[4] = {(uint64_t)Cin, (uint64_t)Win, (uint64_t)Hin, (uint64_t)B};
        uint64_t strides[3] = {(uint64_t)Cin * 2, (uint64_t)Win * Cin * 2, (uint64_t)Hin * Win * Cin * 2};
        uint32_t box[4] = {64, (uint32_t)bw, (uint32_t)bh, (uint32_t)bnimg};
        rc = make_tmap_nd(&p.tmX[0], x, 4, dims, strides, box);
        p.conv.rank = 4;
    } else {
        uint64_t dims[5] = {(uint64_t)(2 * Cin), (uint64_t)(Win / 2), 2, (uint64_t)(Hin / 2), (uint64_t)B};
        uint64_t strides[4] = {(uint64_t)(2 * Cin) * 2, (uint64_t)Win * Cin * 2, (uint64_t)(2 * Win * Cin) * 2, (uint64_t)Hin * Win * Cin * 2};
        uint32_t box[5] = {64, (uint32_t)bw, 1, (uint32_t)bh, (uint32_t)bnimg};
        rc = make_tmap_nd(&p.tmX[0], x, 5, dims, strides, box);
        p.conv.rank = 5;
    }
    if (rc) return rc;
    rc = make_tmap_2d(&p.tmS[0], S, 64, (uint64_t)M, (uint64_t)lds, 64, 128);
    if (rc) return rc;
    p.conv.bw = bw; p.conv.bh = bh; p.conv.bn = bnimg;
    p.conv.tiles_w = (int)(oW / bw); p.conv.tiles_h = (int)(oH / bh);
    LGProblem& q = p.prob[0];
    q.n_begin = 0; q.n_end = (int)Cin; q.nblocks = nblocks;
    q.col_chunks = (int)((Cin + 127) / 128);
    const int total_tiles = (int)((M + 127) / 128);
    int splits = num_sms() / q.col_chunks;
    if (splits < 1) splits = 1;
    if (splits > total_tiles) splits = total_tiles;
    q.tiles_per_cta = (total_tiles + splits - 1) / splits;
    q.splits = (total_tiles + q.tiles_per_cta - 1) / q.tiles_per_cta;
    for (int kh = 0; kh < 3; ++kh)
        for (int kw = 0; kw < 3; ++kw) {
            if (stride == 1) { p.conv.c0_off = 0; p.conv.dw = kw - 1; p.conv.dh = kh - 1; p.conv.c2 = 0; }
            else {          // input row 2*oh + kh - 1 -> (phase, index) of the [H/2][2][W/2][2C] view, as in the forward conv
                p.conv.c0_off = (int)(((kw == 1) ? 0 : 1) * Cin);
                p.conv.dw = (kw == 0) ? -1 : 0;
                p.conv.c2 = (kh == 1) ? 0 : 1;
                p.conv.dh = (kh == 0) ? -1 : 0;
            }
            for (int i = 0; i < nblocks; ++i) {
                const hcp_lora_grad_block& k = blocks[i];
                if (k.rank < 1 || k.c0 < 0 || k.c0 + k.rank > 64 || !k.dst) return set_error(HCP_ERR_INVALID, "lora_grad_conv: block descriptor");
                q.blk[i].n_lo = 0; q.blk[i].n_hi = (int)Cin; q.blk[i].c0 = k.c0; q.blk[i].rank = k.rank;
                q.blk[i].transpose_out = 0; q.blk[i].dst_ld = (int)(Cin * 9); q.blk[i].n_stride = 9;
                q.blk[i].scale = k.scale; q.blk[i].dst = k.dst + (kh * 3 + kw);
            }
            rc = lg_launch(p, (cudaStream_t)stream_);
            if (rc) return rc;
        }
    return HCP_OK;
}

// dW_down and dW_up of one LoRA group in ONE launch (two independent TN GEMMs over the same M token rows).
extern "C" int hcp_lora_grad_pair(const void* U, const void* x, int64_t ldx, int64_t K, const hcp_lora_grad_block* down,
                                  const void* T, const void* dy, int64_t lddy, int64_t N, const hcp_lora_grad_block* up,
                                  int32_t nblocks, int64_t M, int64_t lds, hcp_stream_t stream_) {
    if (M <= 0) return set_error(HCP_ERR_INVALID, "lora_grad_pair: M");
    LoraGradParams p;
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
    return lg_launch(p, (cudaStream_t)stream_);
}
