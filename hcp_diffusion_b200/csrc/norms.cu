// SPDX-License-Identifier: Apache-2.0
// HBM-bound kernels of the UNet hot path (sm_90a): GroupNorm(+SiLU) and LayerNorm forward/backward with
// warp-shuffle reductions, GEGLU, nearest-2x upsample.  All activations are bf16 NHWC / token-major, statistics
// and accumulation fp32, 16-byte vector accesses.
//
// Replaces (reference module structure cfgs/unet_struct.txt): ResnetBlock2D.norm1/norm2 + nonlinearity (:93-99),
// Transformer2DModel.norm (:13), conv_norm_out (:929), BasicTransformerBlock.norm1/2/3 (:44-46), GEGLU (:27-30),
// Upsample2D's F.interpolate(scale_factor=2, mode='nearest') (:392) -- and their autograd backward.
#include <stdlib.h>
#include "common.cuh"
#include "host_util.h"
#include "../../include/hcp_b200.h"

namespace hcp {

__device__ __forceinline__ float silu_f(float z) { return z / (1.f + __expf(-z)); }
__device__ __forceinline__ float silu_grad(float z) {
    const float s = 1.f / (1.f + __expf(-z));
    return s * (1.f + z * (1.f - s));
}
__device__ __forceinline__ float gelu_f(float x) { return 0.5f * x * (1.f + erff(x * 0.70710678118654752f)); }
__device__ __forceinline__ float gelu_grad(float x) {
    const float cdf = 0.5f * (1.f + erff(x * 0.70710678118654752f));
    const float pdf = 0.3989422804014327f * __expf(-0.5f * x * x);
    return cdf + x * pdf;
}

__device__ __forceinline__ void unpack8(const uint4& u, float* f) {
    float2 t;
    t = unpack_bf16x2(u.x); f[0] = t.x; f[1] = t.y;
    t = unpack_bf16x2(u.y); f[2] = t.x; f[3] = t.y;
    t = unpack_bf16x2(u.z); f[4] = t.x; f[5] = t.y;
    t = unpack_bf16x2(u.w); f[6] = t.x; f[7] = t.y;
}
__device__ __forceinline__ uint4 pack8(const float* o) {
    uint4 w;
    w.x = pack_bf16x2(o[0], o[1]); w.y = pack_bf16x2(o[2], o[3]); w.z = pack_bf16x2(o[4], o[5]); w.w = pack_bf16x2(o[6], o[7]);
    return w;
}

// =============================================================================================
// GroupNorm.  x is the channel-concatenation of x1 [B,HW,C1] and (optionally) x2 [B,HW,C2].
// Pass A: per-(image, pixel-chunk) partial sums per group.  Pass B: finalise the statistics of the image
// (every CTA re-reduces the few partials), then normalise / back-propagate its own pixel chunk.
// =============================================================================================
constexpr int GN_MAX_THREADS = 1024;
constexpr int GN_MAX_G = 32;
constexpr int GN_MAX_PT = 4;          // channel pairs per thread (C <= 8192)

// Thread mapping: a CTA owns `rows_per_cta` pixels of one image.  Its threads form a [R row-lanes] x [TP channel-pair
// columns] grid (TP = C/2/PT, R = blockDim/TP): lane (r, tp) walks rows r, r+R, ... and always touches the same PT channel
// pairs, so gamma/beta/group statistics stay in registers and one warp reads 128 contiguous bytes of a pixel row.
struct GNParams {
    const __nv_bfloat16* x1; const __nv_bfloat16* x2;
    int C1, C2, C, G, cg;
    int B, HW, rows_per_cta, nchunks;
    int TP, R, PT, vec8;
    const float* gamma; const float* beta;
    float eps; int silu;
    float* partial;            // [B, nchunks, G, 2]
    float* stats;              // [B, G, 2] (mean, rstd)
    __nv_bfloat16* y;          // fwd out [B,HW,C]
    // backward
    const __nv_bfloat16* dy;   // [B,HW,C]
    const __nv_bfloat16* add1; const __nv_bfloat16* add2;   // optional grads to add to dx1 / dx2
    __nv_bfloat16* dx1; __nv_bfloat16* dx2;
};

__device__ __forceinline__ float2 gn_load2(const GNParams& p, int64_t pix, int c) {
    // channel pair (c, c+1) of concatenated pixel `pix` (C1, C2 even)
    const __nv_bfloat16* src = (c < p.C1) ? p.x1 + pix * p.C1 + c : p.x2 + pix * p.C2 + (c - p.C1);
    return __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(src));
}

template <bool BWD>
__global__ void __launch_bounds__(GN_MAX_THREADS) gn_partial_kernel(const GNParams p) {
    pdl_trigger();
    pdl_wait();
    // per-(row-lane, channel-pair) partial sums, then ONE thread per group adds them in a fixed order: deterministic
    // (no floating-point atomics), which the batch-invariance property test relies on.
    extern __shared__ float s_pair[];     // [R][C/2][2]
    const int b = blockIdx.y, chunk = blockIdx.x;
    const int r0 = chunk * p.rows_per_cta;
    const int r1 = min(p.HW, r0 + p.rows_per_cta);
    const int npair = p.C / 2;
    const int tp = threadIdx.x % p.TP, rl = threadIdx.x / p.TP;
    const bool active = threadIdx.x < p.TP * p.R;          // the block is padded to whole warps
    const float* st = BWD ? p.stats + (int64_t)b * p.G * 2 : nullptr;
    float a0[GN_MAX_PT], a1[GN_MAX_PT];
    float gm0[GN_MAX_PT], gm1[GN_MAX_PT], bt0[GN_MAX_PT], bt1[GN_MAX_PT], mean[GN_MAX_PT], rstd[GN_MAX_PT];
#pragma unroll
    for (int k = 0; k < GN_MAX_PT; ++k) {
        a0[k] = a1[k] = 0.f;
        if (BWD && k < p.PT) {
            const int c = (tp + k * p.TP) * 2;
            const int g = c / p.cg;
            gm0[k] = p.gamma[c]; gm1[k] = p.gamma[c + 1]; bt0[k] = p.beta[c]; bt1[k] = p.beta[c + 1];
            mean[k] = st[g * 2]; rstd[k] = st[g * 2 + 1];
        }
    }
    for (int r = r0 + rl; active && r < r1; r += p.R) {
        const int64_t pix = (int64_t)b * p.HW + r;
#pragma unroll
        for (int k = 0; k < GN_MAX_PT; ++k) {
            if (k < p.PT) {
                const int c = (tp + k * p.TP) * 2;
                const float2 v = gn_load2(p, pix, c);
                if (!BWD) {
                    a0[k] += v.x + v.y;
                    a1[k] += v.x * v.x + v.y * v.y;
                } else {
                    const float2 d = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(p.dy + pix * p.C + c));
                    const float xh0 = (v.x - mean[k]) * rstd[k], xh1 = (v.y - mean[k]) * rstd[k];
                    float g0 = d.x * gm0[k], g1 = d.y * gm1[k];
                    if (p.silu) {
                        g0 *= silu_grad(xh0 * gm0[k] + bt0[k]);
                        g1 *= silu_grad(xh1 * gm1[k] + bt1[k]);
                    }
                    a0[k] += g0 + g1;
                    a1[k] += g0 * xh0 + g1 * xh1;
                }
            }
        }
    }
#pragma unroll
    for (int k = 0; k < GN_MAX_PT; ++k)
        if (active && k < p.PT) {
            const int cp = tp + k * p.TP;
            s_pair[(rl * npair + cp) * 2] = a0[k];
            s_pair[(rl * npair + cp) * 2 + 1] = a1[k];
        }
    __syncthreads();
    float* out = p.partial + ((int64_t)b * p.nchunks + chunk) * p.G * 2;
    const int ppg = p.cg / 2;             // pairs per group
    for (int i = threadIdx.x; i < p.G * 2; i += blockDim.x) {
        const int g = i >> 1, which = i & 1;
        float acc = 0.f;
        for (int r = 0; r < p.R; ++r)
            for (int k = 0; k < ppg; ++k) acc += s_pair[(r * npair + g * ppg + k) * 2 + which];
        out[i] = acc;
    }
}

template <bool BWD>
__global__ void __launch_bounds__(GN_MAX_THREADS) gn_apply_kernel(const GNParams p) {
    pdl_trigger();
    pdl_wait();
    __shared__ float s_a[GN_MAX_G], s_b[GN_MAX_G];
    const int b = blockIdx.y, chunk = blockIdx.x;
    const float n = (float)p.HW * (float)p.cg;
    // finalise: warp w reduces group w, w+nwarps, ... over the chunk partials with a shuffle reduction
    {
        const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nwarps = blockDim.x >> 5;
        for (int g = warp; g < p.G; g += nwarps) {
            float a0 = 0.f, a1 = 0.f;
            for (int ch = lane; ch < p.nchunks; ch += 32) {
                const float* src = p.partial + (((int64_t)b * p.nchunks + ch) * p.G + g) * 2;
                a0 += src[0];
                a1 += src[1];
            }
            a0 = warp_sum(a0);
            a1 = warp_sum(a1);
            if (lane == 0) {
                if (!BWD) {
                    const float mean = a0 / n;
                    const float var = fmaxf(a1 / n - mean * mean, 0.f);
                    const float rstd = rsqrtf(var + p.eps);
                    s_a[g] = mean;
                    s_b[g] = rstd;
                    if (chunk == 0) {
                        p.stats[((int64_t)b * p.G + g) * 2] = mean;
                        p.stats[((int64_t)b * p.G + g) * 2 + 1] = rstd;
                    }
                } else {
                    s_a[g] = a0 / n;   // mean(g)
                    s_b[g] = a1 / n;   // mean(g * xhat)
                }
            }
        }
    }
    __syncthreads();
    const int r0 = chunk * p.rows_per_cta;
    const int r1 = min(p.HW, r0 + p.rows_per_cta);
    const int tp = threadIdx.x % p.TP, rl = threadIdx.x / p.TP;
    const float* st = BWD ? p.stats + (int64_t)b * p.G * 2 : nullptr;
    float gm0[GN_MAX_PT], gm1[GN_MAX_PT], bt0[GN_MAX_PT], bt1[GN_MAX_PT], sa[GN_MAX_PT], sb[GN_MAX_PT], mean[GN_MAX_PT], rstd[GN_MAX_PT];
#pragma unroll
    for (int k = 0; k < GN_MAX_PT; ++k)
        if (k < p.PT) {
            const int c = (tp + k * p.TP) * 2;
            const int g = c / p.cg;
            gm0[k] = p.gamma[c]; gm1[k] = p.gamma[c + 1]; bt0[k] = p.beta[c]; bt1[k] = p.beta[c + 1];
            sa[k] = s_a[g]; sb[k] = s_b[g];
            if (BWD) { mean[k] = st[g * 2]; rstd[k] = st[g * 2 + 1]; }
        }
    for (int r = r0 + rl; threadIdx.x < p.TP * p.R && r < r1; r += p.R) {
        const int64_t pix = (int64_t)b * p.HW + r;
#pragma unroll
        for (int k = 0; k < GN_MAX_PT; ++k) {
            if (k >= p.PT) continue;
            const int c = (tp + k * p.TP) * 2;
            const float2 v = gn_load2(p, pix, c);
            if (!BWD) {
                float z0 = (v.x - sa[k]) * sb[k] * gm0[k] + bt0[k];
                float z1 = (v.y - sa[k]) * sb[k] * gm1[k] + bt1[k];
                if (p.silu) { z0 = silu_f(z0); z1 = silu_f(z1); }
                *reinterpret_cast<__nv_bfloat162*>(p.y + pix * p.C + c) = __floats2bfloat162_rn(z0, z1);
            } else {
                const float2 d = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(p.dy + pix * p.C + c));
                const float xh0 = (v.x - mean[k]) * rstd[k], xh1 = (v.y - mean[k]) * rstd[k];
                float g0 = d.x * gm0[k], g1 = d.y * gm1[k];
                if (p.silu) {
                    g0 *= silu_grad(xh0 * gm0[k] + bt0[k]);
                    g1 *= silu_grad(xh1 * gm1[k] + bt1[k]);
                }
                float o0 = rstd[k] * (g0 - sa[k] - xh0 * sb[k]);
                float o1 = rstd[k] * (g1 - sa[k] - xh1 * sb[k]);
                __nv_bfloat16* dst;
                const __nv_bfloat16* add;
                if (c < p.C1) {
                    dst = p.dx1 + pix * p.C1 + c;
                    add = p.add1 ? p.add1 + pix * p.C1 + c : nullptr;
                } else {
                    dst = p.dx2 + pix * p.C2 + (c - p.C1);
                    add = p.add2 ? p.add2 + pix * p.C2 + (c - p.C1) : nullptr;
                }
                if (add) {
                    const float2 a = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(add));
                    o0 += a.x; o1 += a.y;
                }
                *reinterpret_cast<__nv_bfloat162*>(dst) = __floats2bfloat162_rn(o0, o1);
            }
        }
    }
}

// ---------------------------------------------------------------------------------------------
// 16-byte-vector variant (8 channels per thread and row) for layers with >= 8 channels per group.  A vector may straddle
// ONE group boundary: its first `nb` channels belong to group g_lo, the rest to g_lo + 1; both sets of statistics live in
// registers.  Same two-pass structure and the same deterministic fixed-order reductions as the scalar-pair kernels.
// ---------------------------------------------------------------------------------------------
struct GN8Thread {
    int c0, g_lo, nb;      // first channel, its group, number of channels (of 8) that belong to g_lo
};
__device__ __forceinline__ GN8Thread gn8_thread(const GNParams& p, int vec) {
    GN8Thread t;
    t.c0 = vec * 8;
    t.g_lo = t.c0 / p.cg;
    t.nb = min(8, (t.g_lo + 1) * p.cg - t.c0);
    return t;
}
__device__ __forceinline__ void gn8_load(const GNParams& p, int64_t pix, int c0, float* f) {
    const __nv_bfloat16* src = (c0 < p.C1) ? p.x1 + pix * p.C1 + c0 : p.x2 + pix * p.C2 + (c0 - p.C1);
    unpack8(*reinterpret_cast<const uint4*>(src), f);
}

template <bool BWD>
__global__ void __launch_bounds__(GN_MAX_THREADS) gn8_partial_kernel(const GNParams p) {
    pdl_trigger();
    pdl_wait();
    extern __shared__ float s_vec[];      // [R][C/8][4] : (lo a0, lo a1, hi a0, hi a1)
    const int b = blockIdx.y, chunk = blockIdx.x;
    const int r0 = chunk * p.rows_per_cta;
    const int r1 = min(p.HW, r0 + p.rows_per_cta);
    const int nvec = p.C / 8;
    const int tv = threadIdx.x % p.TP, rl = threadIdx.x / p.TP;
    const GN8Thread t = gn8_thread(p, tv);
    const float* st = BWD ? p.stats + (int64_t)b * p.G * 2 : nullptr;
    float gm[8], bt[8], mean[2] = {0.f, 0.f}, rstd[2] = {0.f, 0.f};
    if (BWD) {
#pragma unroll
        for (int e = 0; e < 8; ++e) { gm[e] = p.gamma[t.c0 + e]; bt[e] = p.beta[t.c0 + e]; }
        mean[0] = st[t.g_lo * 2]; rstd[0] = st[t.g_lo * 2 + 1];
        if (t.nb < 8) { mean[1] = st[t.g_lo * 2 + 2]; rstd[1] = st[t.g_lo * 2 + 3]; }
    }
    float a0[2] = {0.f, 0.f}, a1[2] = {0.f, 0.f};
    const bool active = threadIdx.x < p.TP * p.R;          // the block is padded to whole warps
    for (int r = r0 + rl; active && r < r1; r += p.R) {
        const int64_t pix = (int64_t)b * p.HW + r;
        float x[8];
        gn8_load(p, pix, t.c0, x);
        if (!BWD) {
#pragma unroll
            for (int e = 0; e < 8; ++e) {
                const bool lo = e < t.nb;     // selects, not runtime-indexed arrays (those live in local memory)
                if (lo) a0[0] += x[e]; else a0[1] += x[e];
                if (lo) a1[0] += x[e] * x[e]; else a1[1] += x[e] * x[e];
            }
        } else {
            float d[8];
            unpack8(*reinterpret_cast<const uint4*>(p.dy + pix * p.C + t.c0), d);
#pragma unroll
            for (int e = 0; e < 8; ++e) {
                const bool lo = e < t.nb;     // selects, not runtime-indexed arrays (those live in local memory)
                const float xh = (x[e] - (lo ? mean[0] : mean[1])) * (lo ? rstd[0] : rstd[1]);
                float g = d[e] * gm[e];
                if (p.silu) g *= silu_grad(xh * gm[e] + bt[e]);
                if (lo) a0[0] += g; else a0[1] += g;
                if (lo) a1[0] += g * xh; else a1[1] += g * xh;
            }
        }
    }
    if (active) {
        float* dst = s_vec + ((size_t)rl * nvec + tv) * 4;
        dst[0] = a0[0]; dst[1] = a1[0]; dst[2] = a0[1]; dst[3] = a1[1];
    }
    __syncthreads();
    float* out = p.partial + ((int64_t)b * p.nchunks + chunk) * p.G * 2;
    for (int i = threadIdx.x; i < p.G * 2; i += blockDim.x) {
        const int g = i >> 1, which = i & 1;
        const int v_lo = (g * p.cg) / 8, v_hi = ((g + 1) * p.cg - 1) / 8;
        float acc = 0.f;
        for (int r = 0; r < p.R; ++r)
            for (int v = v_lo; v <= v_hi; ++v) {
                const int vg = (v * 8) / p.cg;                    // g_lo of that vector
                const float* src = s_vec + ((size_t)r * nvec + v) * 4;
                if (vg == g) acc += src[which];
                else if (vg + 1 == g) acc += src[2 + which];
            }
        out[i] = acc;
    }
}

template <bool BWD>
__global__ void __launch_bounds__(GN_MAX_THREADS) gn8_apply_kernel(const GNParams p) {
    pdl_trigger();
    pdl_wait();
    __shared__ float s_a[GN_MAX_G], s_b[GN_MAX_G];
    const int b = blockIdx.y, chunk = blockIdx.x;
    const float n = (float)p.HW * (float)p.cg;
    {
        const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nwarps = blockDim.x >> 5;
        for (int g = warp; g < p.G; g += nwarps) {
            float a0 = 0.f, a1 = 0.f;
            for (int ch = lane; ch < p.nchunks; ch += 32) {
                const float* src = p.partial + (((int64_t)b * p.nchunks + ch) * p.G + g) * 2;
                a0 += src[0];
                a1 += src[1];
            }
            a0 = warp_sum(a0);
            a1 = warp_sum(a1);
            if (lane == 0) {
                if (!BWD) {
                    const float mean = a0 / n;
                    const float var = fmaxf(a1 / n - mean * mean, 0.f);
                    const float rstd = rsqrtf(var + p.eps);
                    s_a[g] = mean;
                    s_b[g] = rstd;
                    if (chunk == 0) {
                        p.stats[((int64_t)b * p.G + g) * 2] = mean;
                        p.stats[((int64_t)b * p.G + g) * 2 + 1] = rstd;
                    }
                } else {
                    s_a[g] = a0 / n;
                    s_b[g] = a1 / n;
                }
            }
        }
    }
    __syncthreads();
    const int r0 = chunk * p.rows_per_cta;
    const int r1 = min(p.HW, r0 + p.rows_per_cta);
    const int tv = threadIdx.x % p.TP, rl = threadIdx.x / p.TP;
    const GN8Thread t = gn8_thread(p, tv);
    const float* st = BWD ? p.stats + (int64_t)b * p.G * 2 : nullptr;
    float gm[8], bt[8], sa[2], sb[2], mean[2] = {0.f, 0.f}, rstd[2] = {0.f, 0.f};
#pragma unroll
    for (int e = 0; e < 8; ++e) { gm[e] = p.gamma[t.c0 + e]; bt[e] = p.beta[t.c0 + e]; }
    const int g_hi = min(t.g_lo + 1, p.G - 1);
    sa[0] = s_a[t.g_lo]; sb[0] = s_b[t.g_lo]; sa[1] = s_a[g_hi]; sb[1] = s_b[g_hi];
    if (BWD) { mean[0] = st[t.g_lo * 2]; rstd[0] = st[t.g_lo * 2 + 1]; mean[1] = st[g_hi * 2]; rstd[1] = st[g_hi * 2 + 1]; }
    for (int r = r0 + rl; threadIdx.x < p.TP * p.R && r < r1; r += p.R) {
        const int64_t pix = (int64_t)b * p.HW + r;
        float x[8], o[8];
        gn8_load(p, pix, t.c0, x);
        if (!BWD) {
#pragma unroll
            for (int e = 0; e < 8; ++e) {
                const bool lo = e < t.nb;     // selects, not runtime-indexed arrays (those live in local memory)
                float z = (x[e] - (lo ? sa[0] : sa[1])) * (lo ? sb[0] : sb[1]) * gm[e] + bt[e];
                if (p.silu) z = silu_f(z);
                o[e] = z;
            }
            *reinterpret_cast<uint4*>(p.y + pix * p.C + t.c0) = pack8(o);
        } else {
            float d[8];
            unpack8(*reinterpret_cast<const uint4*>(p.dy + pix * p.C + t.c0), d);
#pragma unroll
            for (int e = 0; e < 8; ++e) {
                const bool lo = e < t.nb;     // selects, not runtime-indexed arrays (those live in local memory)
                const float xh = (x[e] - (lo ? mean[0] : mean[1])) * (lo ? rstd[0] : rstd[1]);
                float g = d[e] * gm[e];
                if (p.silu) g *= silu_grad(xh * gm[e] + bt[e]);
                o[e] = (lo ? rstd[0] : rstd[1]) * (g - (lo ? sa[0] : sa[1]) - xh * (lo ? sb[0] : sb[1]));
            }
            __nv_bfloat16* dst;
            const __nv_bfloat16* add;
            if (t.c0 < p.C1) {
                dst = p.dx1 + pix * p.C1 + t.c0;
                add = p.add1 ? p.add1 + pix * p.C1 + t.c0 : nullptr;
            } else {
                dst = p.dx2 + pix * p.C2 + (t.c0 - p.C1);
                add = p.add2 ? p.add2 + pix * p.C2 + (t.c0 - p.C1) : nullptr;
            }
            if (add) {
                float a[8];
                unpack8(*reinterpret_cast<const uint4*>(add), a);
#pragma unroll
                for (int e = 0; e < 8; ++e) o[e] += a[e];
            }
            *reinterpret_cast<uint4*>(dst) = pack8(o);
        }
    }
}

// =============================================================================================
// Single-pass GroupNorm: one read and one write of the activation (fwd), two reads and one write (bwd).
//
// The statistics of a group only involve that group's channels, so the work is cut along CHANNELS first: a channel block is
// CB = lcm(8, C/G) channels (whole groups AND whole 16-byte vectors: 40 / 80 / 120 channels for the SD widths), and the HW
// pixels of one (image, channel block) are split over a thread-block cluster of S CTAs.  Each CTA brings its [P pixels x CB
// channels] slab into shared memory with a few TMA box loads (all in flight at once), reduces it, the S partial sums per
// group are exchanged through distributed shared memory (fixed rank order -> deterministic and independent of the batch
// neighbours), and the slab is normalised / back-propagated straight from shared memory.
// Replaces the two-pass kernels above whenever the concatenation boundary C1 falls on a channel-block boundary.
// =============================================================================================
constexpr int GNF_LANES = 64;        // pixel lanes per CTA: blockDim = (CB / 8) * lanes, lanes = 64 (narrow blocks) or 32; <= 512 threads

struct alignas(64) GNFParams {
    CUtensorMap tmX1, tmX2, tmDY;    // [B*HW, C*] row-major, box [CB, RB], no swizzle
    int C1, C2, C, G, cg, CB, V, gpb;
    int HW, P, RB, nbox, S, lanes;
    float inv_n;                     // 1 / (HW * cg)
    const float* gamma; const float* beta;
    float eps; int silu;
    float* stats;                    // [B, G, 2] (mean, rstd): written by fwd, read by bwd
    __nv_bfloat16* y;
    const __nv_bfloat16* add1; const __nv_bfloat16* add2;
    __nv_bfloat16* dx1; __nv_bfloat16* dx2;
};

template <bool BWD>
__global__ void __maxnreg__(96) gnf_kernel(const __grid_constant__ GNFParams p) {   // <= 512 threads; 96 registers keep two 320-thread CTAs per SM
    extern __shared__ uint8_t gnf_smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(gnf_smem_raw) + 127) & ~uintptr_t(127));
    const int tile_bytes = p.P * p.CB * 2;
    uint8_t* sX = smem;
    uint8_t* sDY = sX + tile_bytes;                                     // BWD only
    float* s_part = reinterpret_cast<float*>(sX + (BWD ? 2 : 1) * tile_bytes);   // [GNF_LANES][V][4]
    float* s_cta = s_part + p.lanes * p.V * 4;                         // [gpb*2] partial sums of this CTA (read by the cluster)
    float* s_raw = s_cta + 16;                                           // [gpb*2] cluster totals
    float* s_fin = s_raw + 16;                                           // [gpb*2] (mean, rstd) or (mean g, mean g*xhat)
    uint64_t* bar = reinterpret_cast<uint64_t*>(s_fin + 16);

    const int rank = (int)cluster_ctarank();
    const int cb = blockIdx.y, b = blockIdx.z;
    const int c0 = cb * p.CB;                                            // first channel of the block (in the concatenation)
    const int tv = threadIdx.x % p.V, rl = threadIdx.x / p.V;
    const int64_t row0 = (int64_t)b * p.HW + (int64_t)rank * p.P;
    if (threadIdx.x == 0) {
        mbar_init(bar, 1);
        fence_mbar_init();
    }
    __syncthreads();
    pdl_trigger();
    pdl_wait();
    const bool first = c0 < p.C1;
    if (threadIdx.x == 0) {
        const CUtensorMap* tx = first ? &p.tmX1 : &p.tmX2;
        const int cc = first ? c0 : c0 - p.C1;
        mbar_arrive_expect_tx(bar, (BWD ? 2 : 1) * tile_bytes);
        for (int i = 0; i < p.nbox; ++i) {
            tma_load_2d(sX + (size_t)i * p.RB * p.CB * 2, tx, bar, cc, (int)(row0 + i * p.RB));
            if (BWD) tma_load_2d(sDY + (size_t)i * p.RB * p.CB * 2, &p.tmDY, bar, c0, (int)(row0 + i * p.RB));
        }
    }
    // per-thread constants: 8 consecutive channels, which may straddle ONE group boundary
    const int ch = c0 + tv * 8;
    const int g_lo = (tv * 8) / p.cg;                                    // group index inside the block
    const int nb = min(8, (g_lo + 1) * p.cg - tv * 8);
    const int g_hi = min(g_lo + 1, p.gpb - 1);
    const int gbase = c0 / p.cg;
    float gm[8], bt[8], mean[2] = {0.f, 0.f}, rstd[2] = {0.f, 0.f};
#pragma unroll
    for (int e = 0; e < 8; ++e) { gm[e] = p.gamma[ch + e]; bt[e] = p.beta[ch + e]; }
    if (BWD) {
        const float* st = p.stats + ((int64_t)b * p.G + gbase) * 2;
        mean[0] = st[g_lo * 2]; rstd[0] = st[g_lo * 2 + 1];
        mean[1] = st[g_hi * 2]; rstd[1] = st[g_hi * 2 + 1];
    }
    // explicit shared-space reads of the slab (the aligned-base pointer arithmetic would make them generic loads)
    const uint32_t sx_addr = smem_u32(sX), sdy_addr = smem_u32(sDY);
    mbar_wait(bar, 0);

    // ---- pass 1: partial sums of this CTA's slab
    float a0[2] = {0.f, 0.f}, a1[2] = {0.f, 0.f};
    for (int pp = rl; pp < p.P; pp += p.lanes) {
        float x[8];
        unpack8(lds128(sx_addr + (uint32_t)(pp * p.CB + tv * 8) * 2u), x);
        if (!BWD) {
#pragma unroll
            for (int e = 0; e < 8; ++e) {
                const bool lo = e < nb;       // selects, not runtime-indexed arrays (those live in local memory)
                if (lo) a0[0] += x[e]; else a0[1] += x[e];
                if (lo) a1[0] += x[e] * x[e]; else a1[1] += x[e] * x[e];
            }
        } else {
            float d[8];
            unpack8(lds128(sdy_addr + (uint32_t)(pp * p.CB + tv * 8) * 2u), d);
#pragma unroll
            for (int e = 0; e < 8; ++e) {
                const bool lo = e < nb;       // selects, not runtime-indexed arrays (those live in local memory)
                const float xh = (x[e] - (lo ? mean[0] : mean[1])) * (lo ? rstd[0] : rstd[1]);
                float g = d[e] * gm[e];
                if (p.silu) g *= silu_grad(xh * gm[e] + bt[e]);
                if (lo) a0[0] += g; else a0[1] += g;
                if (lo) a1[0] += g * xh; else a1[1] += g * xh;
            }
        }
    }
    {
        float* dst = s_part + ((size_t)rl * p.V + tv) * 4;
        dst[0] = a0[0]; dst[1] = a1[0]; dst[2] = a0[1]; dst[3] = a1[1];
    }
    __syncthreads();
    if ((int)(threadIdx.x >> 5) < p.gpb * 2) {                           // one warp per (group, moment); fixed summation tree
        const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
        const int g = w >> 1, which = w & 1;
        const int v_lo = (g * p.cg) / 8, v_hi = ((g + 1) * p.cg - 1) / 8;
        float acc = 0.f;
        for (int r = lane; r < p.lanes; r += 32)
            for (int v = v_lo; v <= v_hi; ++v) {
                const int vg = (v * 8) / p.cg;
                const float* src = s_part + ((size_t)r * p.V + v) * 4;
                if (vg == g) acc += src[which];
                else if (vg + 1 == g) acc += src[2 + which];
            }
        acc = warp_sum(acc);
        if (lane == 0) s_cta[w] = acc;
    }
    // ---- cluster exchange of the partial sums (rank order: deterministic)
    cluster_arrive();
    cluster_wait();
    if ((int)threadIdx.x < p.gpb * 2) {
        float tot = 0.f;
        for (int r = 0; r < p.S; ++r) tot += ld_dsmem_f32(smem_u32(&s_cta[threadIdx.x]), (uint32_t)r);
        s_raw[threadIdx.x] = tot;
    }
    __syncthreads();
    if ((int)threadIdx.x < p.gpb) {
        const int g = threadIdx.x;
        if (!BWD) {
            const float m = s_raw[2 * g] * p.inv_n;
            const float var = fmaxf(s_raw[2 * g + 1] * p.inv_n - m * m, 0.f);
            const float rs = rsqrtf(var + p.eps);
            s_fin[2 * g] = m;
            s_fin[2 * g + 1] = rs;
            if (rank == 0) {
                p.stats[((int64_t)b * p.G + gbase + g) * 2] = m;
                p.stats[((int64_t)b * p.G + gbase + g) * 2 + 1] = rs;
            }
        } else {
            s_fin[2 * g] = s_raw[2 * g] * p.inv_n;
            s_fin[2 * g + 1] = s_raw[2 * g + 1] * p.inv_n;
        }
    }
    cluster_arrive();                // this CTA no longer reads its neighbours' shared memory (matched by the wait before exit)
    __syncthreads();

    // ---- pass 2: normalise / back-propagate the slab from shared memory
    const float sa[2] = {s_fin[g_lo * 2], s_fin[g_hi * 2]};
    const float sb[2] = {s_fin[g_lo * 2 + 1], s_fin[g_hi * 2 + 1]};
    for (int pb = rl; pb < p.P; pb += 2 * p.lanes) {
        uint4 av[2];
        if (BWD) {                       // residual-branch gradients of two pixels in flight before the first store
#pragma unroll
            for (int j = 0; j < 2; ++j) {
                const int pp = pb + j * p.lanes;
                av[j] = make_uint4(0u, 0u, 0u, 0u);
                if (pp < p.P) {
                    const int64_t pix = row0 + pp;
                    const __nv_bfloat16* add = first ? (p.add1 ? p.add1 + pix * p.C1 + ch : nullptr)
                                                     : (p.add2 ? p.add2 + pix * p.C2 + (ch - p.C1) : nullptr);
                    if (add) av[j] = *reinterpret_cast<const uint4*>(add);
                }
            }
        }
#pragma unroll
        for (int j = 0; j < 2; ++j) {
            const int pp = pb + j * p.lanes;
            if (pp >= p.P) break;
            const int64_t pix = row0 + pp;
            float x[8], o[8];
            unpack8(lds128(sx_addr + (uint32_t)(pp * p.CB + tv * 8) * 2u), x);
            if (!BWD) {
#pragma unroll
                for (int e = 0; e < 8; ++e) {
                    const bool lo = e < nb;
                    float z = (x[e] - (lo ? sa[0] : sa[1])) * (lo ? sb[0] : sb[1]) * gm[e] + bt[e];
                    if (p.silu) z = silu_f(z);
                    o[e] = z;
                }
                *reinterpret_cast<uint4*>(p.y + pix * p.C + ch) = pack8(o);
            } else {
                float d[8], a[8];
                unpack8(lds128(sdy_addr + (uint32_t)(pp * p.CB + tv * 8) * 2u), d);
                unpack8(av[j], a);
#pragma unroll
                for (int e = 0; e < 8; ++e) {
                    const bool lo = e < nb;
                    const float xh = (x[e] - (lo ? mean[0] : mean[1])) * (lo ? rstd[0] : rstd[1]);
                    float g = d[e] * gm[e];
                    if (p.silu) g *= silu_grad(xh * gm[e] + bt[e]);
                    o[e] = (lo ? rstd[0] : rstd[1]) * (g - (lo ? sa[0] : sa[1]) - xh * (lo ? sb[0] : sb[1])) + a[e];
                }
                __nv_bfloat16* dst = first ? p.dx1 + pix * p.C1 + ch : p.dx2 + pix * p.C2 + (ch - p.C1);
                *reinterpret_cast<uint4*>(dst) = pack8(o);
            }
        }
    }
    cluster_wait();                  // nobody in the cluster still reads this CTA's partial sums
}

static int gcd_int(int a, int b) { while (b) { const int t = a % b; a = b; b = t; } return a; }

// Geometry of the single-pass kernel; returns false when the shape must take the two-pass kernels.
static bool gnf_plan(const hcp_groupnorm_args* a, bool bwd, GNFParams& p, dim3& grid, int& threads, size_t& smem, int& rc) {
    rc = HCP_OK;
    static const bool off = getenv("HCP_GN_TWO_PASS") != nullptr;
    if (off) return false;
    const int64_t C = a->C1 + a->C2;
    if (a->G <= 0 || C % a->G != 0) return false;
    const int cg = (int)(C / a->G);
    if (cg < 8 || (cg & 1) || (a->C1 % 8) != 0 || (a->C2 % 8) != 0) return false;
    const int CB = cg / gcd_int(cg, 8) * 8;                      // lcm(8, cg)
    if (C % CB != 0 || (a->C2 > 0 && a->C1 % CB != 0)) return false;
    const int V = CB / 8, gpb = CB / cg;
    const int lanes = V <= 5 ? GNF_LANES : 32;
    if (V * lanes > 512 || gpb > 8 || CB > 256) return false;
    const int64_t HW = a->HW;
    if (HW * a->B >= (int64_t)1 << 31) return false;
    const int nblk = (int)(C / CB);
    const size_t per_pixel = (size_t)CB * 2 * (bwd ? 2 : 1);
    // cluster size: a function of HW only (never of the batch), so the summation order -- and every bit of the result -- of one
    // image does not depend on its batch neighbours; at least one pixel per lane and CTA
    int S = 1;
    while (S < 8 && HW % (2 * S) == 0 && HW / (2 * S) >= GNF_LANES) S *= 2;
    const int P = (int)(HW / S);
    if (P * per_pixel > 180 * 1024) return false;
    int RB = P < 256 ? P : 256;                                   // rows per TMA box: a multiple of 8 (128-byte aligned slabs)
    while (RB >= 8 && (P % RB != 0 || RB % 8 != 0)) --RB;
    if (RB < 8) return false;
    memset(&p, 0, sizeof(p));
    p.C1 = (int)a->C1; p.C2 = (int)a->C2; p.C = (int)C; p.G = (int)a->G; p.cg = cg; p.CB = CB; p.V = V; p.gpb = gpb;
    p.HW = (int)HW; p.P = P; p.RB = RB; p.nbox = P / RB; p.S = S; p.lanes = lanes;
    p.inv_n = 1.f / ((float)HW * (float)cg);
    p.gamma = a->gamma; p.beta = a->beta; p.eps = a->eps; p.silu = a->silu;
    p.stats = a->stats;
    const uint64_t rows = (uint64_t)a->B * HW;
    {
        uint64_t dims[2] = {(uint64_t)a->C1, rows};
        uint64_t strides[1] = {(uint64_t)a->C1 * 2};
        uint32_t box[2] = {(uint32_t)CB, (uint32_t)RB};
        if ((rc = make_tmap_nd(&p.tmX1, a->x1, 2, dims, strides, box, false))) return false;
    }
    if (a->C2 > 0) {
        uint64_t dims[2] = {(uint64_t)a->C2, rows};
        uint64_t strides[1] = {(uint64_t)a->C2 * 2};
        uint32_t box[2] = {(uint32_t)CB, (uint32_t)RB};
        if ((rc = make_tmap_nd(&p.tmX2, a->x2, 2, dims, strides, box, false))) return false;
    } else {
        p.tmX2 = p.tmX1;
    }
    if (bwd) {
        uint64_t dims[2] = {(uint64_t)C, rows};
        uint64_t strides[1] = {(uint64_t)C * 2};
        uint32_t box[2] = {(uint32_t)CB, (uint32_t)RB};
        if ((rc = make_tmap_nd(&p.tmDY, a->dy, 2, dims, strides, box, false))) return false;
    } else {
        p.tmDY = p.tmX1;
    }
    grid = dim3((unsigned)S, (unsigned)nblk, (unsigned)a->B);
    threads = V * lanes;
    smem = (size_t)P * per_pixel + (size_t)lanes * V * 4 * sizeof(float) + 3 * 16 * sizeof(float) + 64 + 128;
    return true;
}

template <bool BWD>
static int gnf_launch(const GNFParams& p, dim3 grid, int threads, size_t smem, cudaStream_t stream) {
    static bool configured = false;
    if (!configured) {
        cudaError_t e = cudaFuncSetAttribute(gnf_kernel<BWD>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
        if (e != cudaSuccess) return set_cuda_error(e, "cudaFuncSetAttribute(gnf)");
        configured = true;
    }
    cudaError_t e = launch_cluster(gnf_kernel<BWD>, grid, dim3(threads), smem, stream, grid.x, p);
    if (e != cudaSuccess) return set_cuda_error(e, "groupnorm single-pass launch");
    return HCP_OK;
}

static int gn_geometry(const hcp_groupnorm_args* a, GNParams& p) {
    if (!a || !a->x1 || !a->gamma || !a->beta || !a->workspace || !a->stats) return set_error(HCP_ERR_INVALID, "groupnorm: null pointer");
    const int64_t C = a->C1 + a->C2;
    if (a->G <= 0 || a->G > GN_MAX_G || C % a->G != 0) return set_error(HCP_ERR_INVALID, "groupnorm: groups");
    const int64_t cg = C / a->G;
    if ((cg & 1) || (a->C1 & 1) || (a->C2 & 1)) return set_error(HCP_ERR_INVALID, "groupnorm: channels per group must be even");
    const int npair = (int)(C / 2);
    int PT = (npair + GN_MAX_THREADS - 1) / GN_MAX_THREADS;
    while (PT <= GN_MAX_PT && npair % PT != 0) ++PT;
    if (PT > GN_MAX_PT) return set_error(HCP_ERR_INVALID, "groupnorm: unsupported channel count");
    if (a->C2 > 0 && !a->x2) return set_error(HCP_ERR_INVALID, "groupnorm: x2");
    memset(&p, 0, sizeof(p));
    p.x1 = (const __nv_bfloat16*)a->x1; p.x2 = (const __nv_bfloat16*)a->x2;
    p.C1 = (int)a->C1; p.C2 = (int)a->C2; p.C = (int)C; p.G = (int)a->G; p.cg = (int)cg;
    p.B = (int)a->B; p.HW = (int)a->HW;
    // <= 32 pixel chunks per image (one wave of ~1000-thread CTAs at batch 4), at least 4 rows per CTA.  The chunking depends on HW only, never on the batch size, so
    // the summation order (and therefore every bit of the result) of one image is independent of its batch neighbours.
    int rows = (int)((a->HW + 31) / 32);
    if (rows < 4) rows = 4;
    if (rows > a->HW) rows = (int)a->HW;
    p.rows_per_cta = rows;
    p.nchunks = (int)((a->HW + rows - 1) / rows);
    p.vec8 = (cg >= 8 && (a->C1 % 8) == 0 && (a->C2 % 8) == 0 && C / 8 <= GN_MAX_THREADS) ? 1 : 0;
    p.PT = PT;
    p.TP = p.vec8 ? (int)(C / 8) : npair / PT;
    p.R = GN_MAX_THREADS / p.TP;
    if (p.R > rows) p.R = rows;
    if (p.R < 1) p.R = 1;
    p.gamma = a->gamma; p.beta = a->beta; p.eps = a->eps; p.silu = a->silu;
    p.partial = a->workspace; p.stats = a->stats;
    if (a->workspace_bytes < (size_t)a->B * p.nchunks * p.G * 2 * sizeof(float)) return set_error(HCP_ERR_INVALID, "groupnorm: workspace too small");
    return HCP_OK;
}

// =============================================================================================
// LayerNorm: one warp per row, the row lives in registers (C <= 2048)
// =============================================================================================
constexpr int LN_MAX_C = 2048;

// NVPL = ceil((C/8) / 32): 16-byte vectors per lane (compile time so the row stays in registers)
template <bool BWD, int NVPL, bool PIPE>
__global__ void __launch_bounds__(256) layernorm_kernel(const __nv_bfloat16* __restrict__ x, const __nv_bfloat16* __restrict__ dy,
                                                        const __nv_bfloat16* __restrict__ add, const float* __restrict__ gamma,
                                                        const float* __restrict__ beta, float eps, int64_t M, int C,
                                                        float* __restrict__ stats, __nv_bfloat16* __restrict__ out, int rows_per_warp) {
    pdl_trigger();
    pdl_wait();
    const int64_t warp_g = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    const int nv = C / 8;
    // a warp walks `rows_per_warp` consecutive rows: the affine parameters of its columns are loaded once and stay in registers
    float gm[NVPL][8], bt[NVPL][8];
#pragma unroll
    for (int k = 0; k < NVPL; ++k) {
        const int i = lane + 32 * k;
#pragma unroll
        for (int e = 0; e < 8; ++e) { gm[k][e] = 0.f; bt[k][e] = 0.f; }
        if (i < nv) {
            const float4 g0 = *reinterpret_cast<const float4*>(gamma + i * 8), g1 = *reinterpret_cast<const float4*>(gamma + i * 8 + 4);
            gm[k][0] = g0.x; gm[k][1] = g0.y; gm[k][2] = g0.z; gm[k][3] = g0.w; gm[k][4] = g1.x; gm[k][5] = g1.y; gm[k][6] = g1.z; gm[k][7] = g1.w;
            if (!BWD) {
                const float4 b0 = *reinterpret_cast<const float4*>(beta + i * 8), b1 = *reinterpret_cast<const float4*>(beta + i * 8 + 4);
                bt[k][0] = b0.x; bt[k][1] = b0.y; bt[k][2] = b0.z; bt[k][3] = b0.w; bt[k][4] = b1.x; bt[k][5] = b1.y; bt[k][6] = b1.z; bt[k][7] = b1.w;
            }
        }
    }
    // Software pipeline over the rows of this warp: the raw 16-byte vectors of row r+1 (x, and dY / the residual gradient in the
    // backward) are requested BEFORE row r is reduced, normalised and stored, so a warp never waits one full memory round trip per row.
    const int64_t row_begin = warp_g * rows_per_warp;
    if (row_begin >= M) return;
    const int64_t row_end = (row_begin + rows_per_warp < M) ? row_begin + rows_per_warp : M;
    uint4 xn[NVPL], dn[NVPL], an[NVPL];
    auto fetch = [&](int64_t row) {
#pragma unroll
        for (int k = 0; k < NVPL; ++k) {
            const int i = lane + 32 * k;
            xn[k] = dn[k] = an[k] = make_uint4(0u, 0u, 0u, 0u);
            if (i < nv) {
                xn[k] = *reinterpret_cast<const uint4*>(x + row * C + i * 8);
                if (BWD) {
                    dn[k] = *reinterpret_cast<const uint4*>(dy + row * C + i * 8);
                    if (add) an[k] = *reinterpret_cast<const uint4*>(add + row * C + i * 8);
                }
            }
        }
    };
    if (PIPE) fetch(row_begin);
    for (int64_t row = row_begin; row < row_end; ++row) {
    if (!PIPE) fetch(row);                    // wide rows / one or two rows per warp: no second register set
    float v[NVPL][8];
    uint4 dcur[NVPL], av[NVPL];
    float s = 0.f;
#pragma unroll
    for (int k = 0; k < NVPL; ++k) {
        unpack8(xn[k], v[k]);                 // lanes beyond the row hold zeros
        dcur[k] = dn[k];
        av[k] = an[k];
#pragma unroll
        for (int e = 0; e < 8; ++e) s += v[k][e];
    }
    float mean_b = 0.f, rstd_b = 0.f;
    if (BWD) { mean_b = stats[row * 2]; rstd_b = stats[row * 2 + 1]; }
    if (PIPE && row + 1 < row_end) fetch(row + 1);    // next row's loads are in flight while this row is processed
    if (!BWD) {
        const float mean = warp_sum(s) / C;
        float q = 0.f;
#pragma unroll
        for (int k = 0; k < NVPL; ++k)
            if (lane + 32 * k < nv) {
#pragma unroll
                for (int e = 0; e < 8; ++e) { const float d = v[k][e] - mean; q += d * d; }
            }
        const float rstd = rsqrtf(warp_sum(q) / C + eps);
        if (lane == 0 && stats) { stats[row * 2] = mean; stats[row * 2 + 1] = rstd; }
#pragma unroll
        for (int k = 0; k < NVPL; ++k) {
            const int i = lane + 32 * k;
            if (i < nv) {
                float o[8];
#pragma unroll
                for (int e = 0; e < 8; ++e) o[e] = (v[k][e] - mean) * rstd * gm[k][e] + bt[k][e];
                *reinterpret_cast<uint4*>(out + row * C + i * 8) = pack8(o);
            }
        }
    } else {
        const float mean = mean_b, rstd = rstd_b;
        float g[NVPL][8];
        float s1 = 0.f, s2 = 0.f;
#pragma unroll
        for (int k = 0; k < NVPL; ++k) {
            const int i = lane + 32 * k;
            if (i < nv) {
                float d[8];
                unpack8(dcur[k], d);
#pragma unroll
                for (int e = 0; e < 8; ++e) {
                    const float xh = (v[k][e] - mean) * rstd;
                    v[k][e] = xh;
                    g[k][e] = d[e] * gm[k][e];
                    s1 += g[k][e];
                    s2 += g[k][e] * xh;
                }
            }
        }
        s1 = warp_sum(s1) / C;
        s2 = warp_sum(s2) / C;
#pragma unroll
        for (int k = 0; k < NVPL; ++k) {
            const int i = lane + 32 * k;
            if (i < nv) {
                float o[8], a[8];
                unpack8(av[k], a);
#pragma unroll
                for (int e = 0; e < 8; ++e) o[e] = rstd * (g[k][e] - s1 - v[k][e] * s2) + a[e];
                *reinterpret_cast<uint4*>(out + row * C + i * 8) = pack8(o);
            }
        }
    }
    }   // rows of this warp
}

template <bool BWD>
static void launch_layernorm(const __nv_bfloat16* x, const __nv_bfloat16* dy, const __nv_bfloat16* add, const float* gamma,
                             const float* beta, float eps, int64_t M, int C, float* stats, __nv_bfloat16* out, cudaStream_t st) {
    // one wave of CTAs: SMs x 2 resident CTAs (the register-resident rows + affine parameters cost 75-190 registers) x 8 warps
    const int64_t wave = (int64_t)num_sms() * 2 * 8;
    int rpw = (int)((M + wave - 1) / wave);
    if (rpw < 1) rpw = 1;
    if (rpw > 32) rpw = 32;
    const int64_t warps = (M + rpw - 1) / rpw;
    const unsigned blocks = (unsigned)((warps * 32 + 255) / 256);
    const int nvpl = (C / 8 + 31) / 32;
#define LN_CASE(N) case N: launch_k(layernorm_kernel<BWD, N, false>, dim3(blocks), dim3(256), 0, st, x, dy, add, gamma, beta, eps, M, C, stats, out, rpw); break;
    if (rpw >= 3 && nvpl <= 2) {              // many narrow rows per warp (the 64x64 level): software-pipelined variant
        if (nvpl == 1) launch_k(layernorm_kernel<BWD, 1, true>, dim3(blocks), dim3(256), 0, st, x, dy, add, gamma, beta, eps, M, C, stats, out, rpw);
        else launch_k(layernorm_kernel<BWD, 2, true>, dim3(blocks), dim3(256), 0, st, x, dy, add, gamma, beta, eps, M, C, stats, out, rpw);
        return;
    }
    switch (nvpl) {
        LN_CASE(1) LN_CASE(2) LN_CASE(3) LN_CASE(4) LN_CASE(5) LN_CASE(6) LN_CASE(7) LN_CASE(8)
    }
#undef LN_CASE
}

// =============================================================================================
// GEGLU: u = [a | g] (each F wide);  h = a * gelu(g)
// =============================================================================================
__global__ void geglu_fwd_kernel(const __nv_bfloat16* __restrict__ u, int64_t M, int F, __nv_bfloat16* __restrict__ h) {
    pdl_trigger();
    pdl_wait();
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;   // one thread per 8 outputs
    const int nv = F / 8;
    if (i >= M * nv) return;
    const int64_t m = i / nv;
    const int c = (int)(i % nv) * 8;
    const uint4 ua = *reinterpret_cast<const uint4*>(u + m * 2 * F + c);
    const uint4 ug = *reinterpret_cast<const uint4*>(u + m * 2 * F + F + c);
    const uint32_t aa[4] = {ua.x, ua.y, ua.z, ua.w}, gg[4] = {ug.x, ug.y, ug.z, ug.w};
    uint32_t o[4];
#pragma unroll
    for (int e = 0; e < 4; ++e) {
        const float2 a = unpack_bf16x2(aa[e]), g = unpack_bf16x2(gg[e]);
        o[e] = pack_bf16x2(a.x * gelu_f(g.x), a.y * gelu_f(g.y));
    }
    *reinterpret_cast<uint4*>(h + m * F + c) = make_uint4(o[0], o[1], o[2], o[3]);
}
__global__ void geglu_bwd_kernel(const __nv_bfloat16* __restrict__ u, const __nv_bfloat16* __restrict__ dh, int64_t M, int F,
                                 __nv_bfloat16* __restrict__ du) {
    pdl_trigger();
    pdl_wait();
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    const int nv = F / 8;
    if (i >= M * nv) return;
    const int64_t m = i / nv;
    const int c = (int)(i % nv) * 8;
    const uint4 ua = *reinterpret_cast<const uint4*>(u + m * 2 * F + c);
    const uint4 ug = *reinterpret_cast<const uint4*>(u + m * 2 * F + F + c);
    const uint4 ud = *reinterpret_cast<const uint4*>(dh + m * F + c);
    const uint32_t aa[4] = {ua.x, ua.y, ua.z, ua.w}, gg[4] = {ug.x, ug.y, ug.z, ug.w}, dd[4] = {ud.x, ud.y, ud.z, ud.w};
    uint32_t oa[4], og[4];
#pragma unroll
    for (int e = 0; e < 4; ++e) {
        const float2 a = unpack_bf16x2(aa[e]), g = unpack_bf16x2(gg[e]), d = unpack_bf16x2(dd[e]);
        oa[e] = pack_bf16x2(d.x * gelu_f(g.x), d.y * gelu_f(g.y));
        og[e] = pack_bf16x2(d.x * a.x * gelu_grad(g.x), d.y * a.y * gelu_grad(g.y));
    }
    *reinterpret_cast<uint4*>(du + m * 2 * F + c) = make_uint4(oa[0], oa[1], oa[2], oa[3]);
    *reinterpret_cast<uint4*>(du + m * 2 * F + F + c) = make_uint4(og[0], og[1], og[2], og[3]);
}

// =============================================================================================
// quick-GELU (CLIP MLP): y = x * sigmoid(1.702 x);  dx = dy * (s + 1.702 x s (1 - s))
// =============================================================================================
__device__ __forceinline__ float qgelu_sig(float x) { return 1.f / (1.f + __expf(-1.702f * x)); }

__global__ void quick_gelu_fwd_kernel(const __nv_bfloat16* __restrict__ x, int64_t n8, __nv_bfloat16* __restrict__ y) {
    pdl_trigger();
    pdl_wait();
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;   // one thread per 8 elements
    if (i >= n8) return;
    const uint4 ux = reinterpret_cast<const uint4*>(x)[i];
    const uint32_t xx[4] = {ux.x, ux.y, ux.z, ux.w};
    uint32_t o[4];
#pragma unroll
    for (int e = 0; e < 4; ++e) {
        const float2 v = unpack_bf16x2(xx[e]);
        o[e] = pack_bf16x2(v.x * qgelu_sig(v.x), v.y * qgelu_sig(v.y));
    }
    reinterpret_cast<uint4*>(y)[i] = make_uint4(o[0], o[1], o[2], o[3]);
}
__global__ void quick_gelu_bwd_kernel(const __nv_bfloat16* __restrict__ x, const __nv_bfloat16* __restrict__ dy, int64_t n8,
                                      __nv_bfloat16* __restrict__ dx) {
    pdl_trigger();
    pdl_wait();
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= n8) return;
    const uint4 ux = reinterpret_cast<const uint4*>(x)[i], ud = reinterpret_cast<const uint4*>(dy)[i];
    const uint32_t xx[4] = {ux.x, ux.y, ux.z, ux.w}, dd[4] = {ud.x, ud.y, ud.z, ud.w};
    uint32_t o[4];
#pragma unroll
    for (int e = 0; e < 4; ++e) {
        const float2 v = unpack_bf16x2(xx[e]), d = unpack_bf16x2(dd[e]);
        const float s0 = qgelu_sig(v.x), s1 = qgelu_sig(v.y);
        o[e] = pack_bf16x2(d.x * (s0 + 1.702f * v.x * s0 * (1.f - s0)), d.y * (s1 + 1.702f * v.y * s1 * (1.f - s1)));
    }
    reinterpret_cast<uint4*>(dx)[i] = make_uint4(o[0], o[1], o[2], o[3]);
}

// =============================================================================================
// exact GELU (OpenCLIP-bigG MLP, transformers hidden_act='gelu'): y = 0.5 x (1 + erf(x / sqrt 2));
// dx = dy * (Phi(x) + x phi(x))  -- gelu_f / gelu_grad, the same functions GEGLU uses
// =============================================================================================
__global__ void gelu_fwd_kernel(const __nv_bfloat16* __restrict__ x, int64_t n8, __nv_bfloat16* __restrict__ y) {
    pdl_trigger();
    pdl_wait();
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;   // one thread per 8 elements
    if (i >= n8) return;
    const uint4 ux = reinterpret_cast<const uint4*>(x)[i];
    const uint32_t xx[4] = {ux.x, ux.y, ux.z, ux.w};
    uint32_t o[4];
#pragma unroll
    for (int e = 0; e < 4; ++e) {
        const float2 v = unpack_bf16x2(xx[e]);
        o[e] = pack_bf16x2(gelu_f(v.x), gelu_f(v.y));
    }
    reinterpret_cast<uint4*>(y)[i] = make_uint4(o[0], o[1], o[2], o[3]);
}
__global__ void gelu_bwd_kernel(const __nv_bfloat16* __restrict__ x, const __nv_bfloat16* __restrict__ dy, int64_t n8,
                                __nv_bfloat16* __restrict__ dx) {
    pdl_trigger();
    pdl_wait();
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= n8) return;
    const uint4 ux = reinterpret_cast<const uint4*>(x)[i], ud = reinterpret_cast<const uint4*>(dy)[i];
    const uint32_t xx[4] = {ux.x, ux.y, ux.z, ux.w}, dd[4] = {ud.x, ud.y, ud.z, ud.w};
    uint32_t o[4];
#pragma unroll
    for (int e = 0; e < 4; ++e) {
        const float2 v = unpack_bf16x2(xx[e]), d = unpack_bf16x2(dd[e]);
        o[e] = pack_bf16x2(d.x * gelu_grad(v.x), d.y * gelu_grad(v.y));
    }
    reinterpret_cast<uint4*>(dx)[i] = make_uint4(o[0], o[1], o[2], o[3]);
}

// =============================================================================================
// fp32 sum of up to kSumSrcs bf16 arrays, in source order: the fan-in of the text embedding's gradient over the cross-attentions
// =============================================================================================
constexpr int kSumSrcs = 32;
struct SumSrcs { const __nv_bfloat16* p[kSumSrcs]; };

__global__ void sum_bf16_f32_kernel(const __grid_constant__ SumSrcs s, int nsrc, int64_t n8, int accumulate, float* __restrict__ out) {
    pdl_trigger();
    pdl_wait();
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;   // one thread per 8 elements
    if (i >= n8) return;
    float acc[8];
    float4* o = reinterpret_cast<float4*>(out) + 2 * i;
    if (accumulate) {
        const float4 a = o[0], b = o[1];
        acc[0] = a.x; acc[1] = a.y; acc[2] = a.z; acc[3] = a.w; acc[4] = b.x; acc[5] = b.y; acc[6] = b.z; acc[7] = b.w;
    } else {
#pragma unroll
        for (int e = 0; e < 8; ++e) acc[e] = 0.f;
    }
    for (int k = 0; k < nsrc; ++k) {
        const uint4 u = reinterpret_cast<const uint4*>(s.p[k])[i];
        const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            const float2 f = unpack_bf16x2(w[e]);
            acc[2 * e] += f.x;
            acc[2 * e + 1] += f.y;
        }
    }
    o[0] = make_float4(acc[0], acc[1], acc[2], acc[3]);
    o[1] = make_float4(acc[4], acc[5], acc[6], acc[7]);
}

// =============================================================================================
// token + position embedding gather (CLIPTextEmbeddings): out[r] = bf16(tok[clamp(ids[r])] + pos[clamp(pos_ids[l] or l)]),
// r = b * L + l.  Ids outside the tables read the nearest valid row; they are never read out of bounds.
// =============================================================================================
__global__ void embed_gather_kernel(const int64_t* __restrict__ ids, const int64_t* __restrict__ pos_ids, const float* __restrict__ tok,
                                    int64_t V, const float* __restrict__ pos, int64_t P, int64_t rows, int L, int C,
                                    __nv_bfloat16* __restrict__ out) {
    pdl_trigger();
    pdl_wait();
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;   // one thread per 8 outputs
    const int nv = C / 8;
    if (i >= rows * nv) return;
    const int64_t r = i / nv;
    const int c = (int)(i % nv) * 8;
    const int l = (int)(r % L);
    const int64_t t = min(max(ids[r], (int64_t)0), V - 1);
    const int64_t pr = min(max(pos_ids ? pos_ids[l] : (int64_t)l, (int64_t)0), P - 1);
    const float4* a = reinterpret_cast<const float4*>(tok + t * C + c);
    const float4* b = reinterpret_cast<const float4*>(pos + pr * C + c);
    const float4 a0 = a[0], a1 = a[1], b0 = b[0], b1 = b[1];
    *reinterpret_cast<uint4*>(out + r * C + c) = make_uint4(pack_bf16x2(a0.x + b0.x, a0.y + b0.y), pack_bf16x2(a0.z + b0.z, a0.w + b0.w),
                                                            pack_bf16x2(a1.x + b1.x, a1.y + b1.y), pack_bf16x2(a1.z + b1.z, a1.w + b1.w));
}

// =============================================================================================
// nearest 2x upsample (NHWC) and its backward (sum of the 2x2 block)
// =============================================================================================
__global__ void upsample2x_fwd_kernel(const __nv_bfloat16* __restrict__ x, int B, int H, int W, int C, __nv_bfloat16* __restrict__ y) {
    pdl_trigger();
    pdl_wait();
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;   // one thread per 8 output channels
    const int nv = C / 8;
    const int64_t total = (int64_t)B * 4 * H * W * nv;
    if (i >= total) return;
    const int c = (int)(i % nv) * 8;
    const int64_t pix = i / nv;
    const int wo = (int)(pix % (2 * W)), ho = (int)((pix / (2 * W)) % (2 * H)), b = (int)(pix / ((int64_t)4 * H * W));
    const uint4 v = *reinterpret_cast<const uint4*>(x + (((int64_t)b * H + ho / 2) * W + wo / 2) * C + c);
    *reinterpret_cast<uint4*>(y + pix * C + c) = v;
}
__global__ void upsample2x_bwd_kernel(const __nv_bfloat16* __restrict__ dy, int B, int H, int W, int C, __nv_bfloat16* __restrict__ dx) {
    pdl_trigger();
    pdl_wait();
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;   // one thread per 8 input channels
    const int nv = C / 8;
    const int64_t total = (int64_t)B * H * W * nv;
    if (i >= total) return;
    const int c = (int)(i % nv) * 8;
    const int64_t pix = i / nv;
    const int w = (int)(pix % W), h = (int)((pix / W) % H), b = (int)(pix / ((int64_t)H * W));
    float acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
#pragma unroll
    for (int dh = 0; dh < 2; ++dh)
#pragma unroll
        for (int dw = 0; dw < 2; ++dw) {
            const uint4 v = *reinterpret_cast<const uint4*>(dy + (((int64_t)b * 2 * H + 2 * h + dh) * 2 * W + 2 * w + dw) * C + c);
            float2 t;
            t = unpack_bf16x2(v.x); acc[0] += t.x; acc[1] += t.y;
            t = unpack_bf16x2(v.y); acc[2] += t.x; acc[3] += t.y;
            t = unpack_bf16x2(v.z); acc[4] += t.x; acc[5] += t.y;
            t = unpack_bf16x2(v.w); acc[6] += t.x; acc[7] += t.y;
        }
    uint4 o;
    o.x = pack_bf16x2(acc[0], acc[1]); o.y = pack_bf16x2(acc[2], acc[3]); o.z = pack_bf16x2(acc[4], acc[5]); o.w = pack_bf16x2(acc[6], acc[7]);
    *reinterpret_cast<uint4*>(dx + pix * C + c) = o;
}

// out = a + b (bf16), used where autograd fan-in cannot be folded into a producer kernel
__global__ void add_bf16_kernel(const __nv_bfloat16* __restrict__ a, const __nv_bfloat16* __restrict__ b, int64_t n8,
                                __nv_bfloat16* __restrict__ out) {
    pdl_trigger();
    pdl_wait();
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= n8) return;
    const uint4 x = reinterpret_cast<const uint4*>(a)[i], y = reinterpret_cast<const uint4*>(b)[i];
    const uint32_t xa[4] = {x.x, x.y, x.z, x.w}, ya[4] = {y.x, y.y, y.z, y.w};
    uint32_t o[4];
#pragma unroll
    for (int e = 0; e < 4; ++e) {
        const float2 p = unpack_bf16x2(xa[e]), q = unpack_bf16x2(ya[e]);
        o[e] = pack_bf16x2(p.x + q.x, p.y + q.y);
    }
    reinterpret_cast<uint4*>(out)[i] = make_uint4(o[0], o[1], o[2], o[3]);
}

}  // namespace hcp

using namespace hcp;

#define LAUNCH_CHECK(what)                                              \
    do {                                                                \
        cudaError_t e_ = cudaGetLastError();                            \
        if (e_ != cudaSuccess) return set_cuda_error(e_, what);         \
    } while (0)

extern "C" size_t hcp_groupnorm_workspace_bytes(int64_t B, int64_t HW, int64_t G) {
    int64_t rows = (HW + 31) / 32;
    if (rows < 4) rows = 4;
    if (rows > HW) rows = HW;
    const int64_t nchunks = (HW + rows - 1) / rows;
    return (size_t)(B * nchunks * G * 2) * sizeof(float);
}

extern "C" int hcp_groupnorm_fwd_bf16(const hcp_groupnorm_args* a, hcp_stream_t stream_) {
    GNParams p;
    int rc = gn_geometry(a, p);
    if (rc) return rc;
    if (!a->y) return set_error(HCP_ERR_INVALID, "groupnorm_fwd: y");
    {
        GNFParams f;
        dim3 fgrid;
        int fthreads = 0, frc = HCP_OK;
        size_t fsmem = 0;
        if (gnf_plan(a, false, f, fgrid, fthreads, fsmem, frc)) {
            f.y = (__nv_bfloat16*)a->y;
            return gnf_launch<false>(f, fgrid, fthreads, fsmem, (cudaStream_t)stream_);
        }
        if (frc) return frc;
    }
    p.y = (__nv_bfloat16*)a->y;
    dim3 grid(p.nchunks, p.B);
    const int threads = (p.TP * p.R + 31) & ~31;          // whole warps: the finalize step uses full-warp shuffles
    if (p.vec8) {
        const size_t smem = (size_t)p.R * (p.C / 8) * 4 * sizeof(float);
        launch_k(gn8_partial_kernel<false>, dim3(grid), dim3(threads), smem, (cudaStream_t)stream_, p);
        launch_k(gn8_apply_kernel<false>, dim3(grid), dim3(threads), 0, (cudaStream_t)stream_, p);
    } else {
        const size_t smem = (size_t)p.R * (p.C / 2) * 2 * sizeof(float);
        launch_k(gn_partial_kernel<false>, dim3(grid), dim3(threads), smem, (cudaStream_t)stream_, p);
        launch_k(gn_apply_kernel<false>, dim3(grid), dim3(threads), 0, (cudaStream_t)stream_, p);
    }
    LAUNCH_CHECK("groupnorm_fwd launch");
    return HCP_OK;
}

extern "C" int hcp_groupnorm_bwd_bf16(const hcp_groupnorm_args* a, hcp_stream_t stream_) {
    GNParams p;
    int rc = gn_geometry(a, p);
    if (rc) return rc;
    if (!a->dy || !a->dx1 || (a->C2 > 0 && !a->dx2)) return set_error(HCP_ERR_INVALID, "groupnorm_bwd: dy/dx");
    {
        GNFParams f;
        dim3 fgrid;
        int fthreads = 0, frc = HCP_OK;
        size_t fsmem = 0;
        if (gnf_plan(a, true, f, fgrid, fthreads, fsmem, frc)) {
            f.add1 = (const __nv_bfloat16*)a->add1; f.add2 = (const __nv_bfloat16*)a->add2;
            f.dx1 = (__nv_bfloat16*)a->dx1; f.dx2 = (__nv_bfloat16*)a->dx2;
            return gnf_launch<true>(f, fgrid, fthreads, fsmem, (cudaStream_t)stream_);
        }
        if (frc) return frc;
    }
    p.dy = (const __nv_bfloat16*)a->dy;
    p.add1 = (const __nv_bfloat16*)a->add1; p.add2 = (const __nv_bfloat16*)a->add2;
    p.dx1 = (__nv_bfloat16*)a->dx1; p.dx2 = (__nv_bfloat16*)a->dx2;
    dim3 grid(p.nchunks, p.B);
    const int threads = (p.TP * p.R + 31) & ~31;          // whole warps: the finalize step uses full-warp shuffles
    if (p.vec8) {
        const size_t smem = (size_t)p.R * (p.C / 8) * 4 * sizeof(float);
        launch_k(gn8_partial_kernel<true>, dim3(grid), dim3(threads), smem, (cudaStream_t)stream_, p);
        launch_k(gn8_apply_kernel<true>, dim3(grid), dim3(threads), 0, (cudaStream_t)stream_, p);
    } else {
        const size_t smem = (size_t)p.R * (p.C / 2) * 2 * sizeof(float);
        launch_k(gn_partial_kernel<true>, dim3(grid), dim3(threads), smem, (cudaStream_t)stream_, p);
        launch_k(gn_apply_kernel<true>, dim3(grid), dim3(threads), 0, (cudaStream_t)stream_, p);
    }
    LAUNCH_CHECK("groupnorm_bwd launch");
    return HCP_OK;
}

extern "C" int hcp_layernorm_fwd_bf16(const void* x, const float* gamma, const float* beta, float eps, int64_t M, int64_t C,
                                      float* stats, void* y, hcp_stream_t stream_) {
    if (!x || !gamma || !beta || !y) return set_error(HCP_ERR_INVALID, "layernorm_fwd: null pointer");
    if (C % 8 != 0 || C > LN_MAX_C || C <= 0) return set_error(HCP_ERR_INVALID, "layernorm: C must be a multiple of 8, <= 2048");
    launch_layernorm<false>((const __nv_bfloat16*)x, nullptr, nullptr, gamma, beta, eps, M, (int)C, stats, (__nv_bfloat16*)y,
                            (cudaStream_t)stream_);
    LAUNCH_CHECK("layernorm_fwd launch");
    return HCP_OK;
}

extern "C" int hcp_layernorm_bwd_bf16(const void* x, const void* dy, const void* add, const float* gamma, const float* stats,
                                      int64_t M, int64_t C, void* dx, hcp_stream_t stream_) {
    if (!x || !dy || !gamma || !stats || !dx) return set_error(HCP_ERR_INVALID, "layernorm_bwd: null pointer");
    if (C % 8 != 0 || C > LN_MAX_C || C <= 0) return set_error(HCP_ERR_INVALID, "layernorm: C must be a multiple of 8, <= 2048");
    launch_layernorm<true>((const __nv_bfloat16*)x, (const __nv_bfloat16*)dy, (const __nv_bfloat16*)add, gamma, nullptr, 0.f, M, (int)C,
                           const_cast<float*>(stats), (__nv_bfloat16*)dx, (cudaStream_t)stream_);
    LAUNCH_CHECK("layernorm_bwd launch");
    return HCP_OK;
}

extern "C" int hcp_geglu_fwd_bf16(const void* u, int64_t M, int64_t F, void* h, hcp_stream_t stream_) {
    if (!u || !h || F % 8 != 0) return set_error(HCP_ERR_INVALID, "geglu_fwd");
    const int64_t n = M * (F / 8);
    launch_k(geglu_fwd_kernel, dim3((unsigned)((n + 255) / 256)), dim3(256), 0, (cudaStream_t)stream_, (const __nv_bfloat16*)u, M, (int)F, (__nv_bfloat16*)h);
    LAUNCH_CHECK("geglu_fwd launch");
    return HCP_OK;
}
extern "C" int hcp_geglu_bwd_bf16(const void* u, const void* dh, int64_t M, int64_t F, void* du, hcp_stream_t stream_) {
    if (!u || !dh || !du || F % 8 != 0) return set_error(HCP_ERR_INVALID, "geglu_bwd");
    const int64_t n = M * (F / 8);
    launch_k(geglu_bwd_kernel, dim3((unsigned)((n + 255) / 256)), dim3(256), 0, (cudaStream_t)stream_, (const __nv_bfloat16*)u, (const __nv_bfloat16*)dh, M,
                                                                                   (int)F, (__nv_bfloat16*)du);
    LAUNCH_CHECK("geglu_bwd launch");
    return HCP_OK;
}
extern "C" int hcp_quick_gelu_fwd_bf16(const void* x, int64_t M, int64_t F, void* y, hcp_stream_t stream_) {
    if (!x || !y || M < 0 || F % 8 != 0) return set_error(HCP_ERR_INVALID, "quick_gelu_fwd");
    const int64_t n8 = M * (F / 8);
    if (n8 == 0) return HCP_OK;
    launch_k(quick_gelu_fwd_kernel, dim3((unsigned)((n8 + 255) / 256)), dim3(256), 0, (cudaStream_t)stream_, (const __nv_bfloat16*)x, n8,
             (__nv_bfloat16*)y);
    LAUNCH_CHECK("quick_gelu_fwd launch");
    return HCP_OK;
}
extern "C" int hcp_quick_gelu_bwd_bf16(const void* x, const void* dy, int64_t M, int64_t F, void* dx, hcp_stream_t stream_) {
    if (!x || !dy || !dx || M < 0 || F % 8 != 0) return set_error(HCP_ERR_INVALID, "quick_gelu_bwd");
    const int64_t n8 = M * (F / 8);
    if (n8 == 0) return HCP_OK;
    launch_k(quick_gelu_bwd_kernel, dim3((unsigned)((n8 + 255) / 256)), dim3(256), 0, (cudaStream_t)stream_, (const __nv_bfloat16*)x,
             (const __nv_bfloat16*)dy, n8, (__nv_bfloat16*)dx);
    LAUNCH_CHECK("quick_gelu_bwd launch");
    return HCP_OK;
}
extern "C" int hcp_gelu_fwd_bf16(const void* x, int64_t M, int64_t F, void* y, hcp_stream_t stream_) {
    if (!x || !y || M < 0 || F % 8 != 0) return set_error(HCP_ERR_INVALID, "gelu_fwd");
    const int64_t n8 = M * (F / 8);
    if (n8 == 0) return HCP_OK;
    launch_k(gelu_fwd_kernel, dim3((unsigned)((n8 + 255) / 256)), dim3(256), 0, (cudaStream_t)stream_, (const __nv_bfloat16*)x, n8,
             (__nv_bfloat16*)y);
    LAUNCH_CHECK("gelu_fwd launch");
    return HCP_OK;
}
extern "C" int hcp_gelu_bwd_bf16(const void* x, const void* dy, int64_t M, int64_t F, void* dx, hcp_stream_t stream_) {
    if (!x || !dy || !dx || M < 0 || F % 8 != 0) return set_error(HCP_ERR_INVALID, "gelu_bwd");
    const int64_t n8 = M * (F / 8);
    if (n8 == 0) return HCP_OK;
    launch_k(gelu_bwd_kernel, dim3((unsigned)((n8 + 255) / 256)), dim3(256), 0, (cudaStream_t)stream_, (const __nv_bfloat16*)x,
             (const __nv_bfloat16*)dy, n8, (__nv_bfloat16*)dx);
    LAUNCH_CHECK("gelu_bwd launch");
    return HCP_OK;
}
extern "C" int hcp_sum_bf16_to_f32(const void* const* srcs, int64_t nsrc, int64_t n, float* out, hcp_stream_t stream_) {
    if (!srcs || !out || nsrc <= 0 || n % 8 != 0) return set_error(HCP_ERR_INVALID, "sum_bf16_to_f32: need sources and n % 8 == 0");
    for (int64_t k = 0; k < nsrc; ++k)
        if (!srcs[k]) return set_error(HCP_ERR_INVALID, "sum_bf16_to_f32: null source");
    const int64_t n8 = n / 8;
    if (n8 == 0) return HCP_OK;
    for (int64_t k0 = 0; k0 < nsrc; k0 += kSumSrcs) {
        SumSrcs s;
        memset(&s, 0, sizeof(s));
        const int cnt = (int)(nsrc - k0 < kSumSrcs ? nsrc - k0 : kSumSrcs);
        for (int k = 0; k < cnt; ++k) s.p[k] = (const __nv_bfloat16*)srcs[k0 + k];
        launch_k(sum_bf16_f32_kernel, dim3((unsigned)((n8 + 255) / 256)), dim3(256), 0, (cudaStream_t)stream_, s, cnt, n8, (int)(k0 > 0), out);
        LAUNCH_CHECK("sum_bf16_to_f32 launch");
    }
    return HCP_OK;
}
extern "C" int hcp_embed_gather_bf16(const int64_t* ids, const int64_t* pos_ids, const float* tok_emb, int64_t V, const float* pos_emb,
                                     int64_t P, int64_t B, int64_t L, int64_t C, void* out, hcp_stream_t stream_) {
    if (!ids || !tok_emb || !pos_emb || !out) return set_error(HCP_ERR_INVALID, "embed_gather: null pointer");
    if (V <= 0 || P <= 0 || B <= 0 || L <= 0 || C <= 0 || C % 8 != 0)
        return set_error(HCP_ERR_INVALID, "embed_gather: empty table or C not a multiple of 8");
    if (!pos_ids && L > P) return set_error(HCP_ERR_INVALID, "embed_gather: sequence longer than the position table");
    const int64_t n = B * L * (C / 8);
    launch_k(embed_gather_kernel, dim3((unsigned)((n + 255) / 256)), dim3(256), 0, (cudaStream_t)stream_, ids, pos_ids, tok_emb, V, pos_emb, P,
             B * L, (int)L, (int)C, (__nv_bfloat16*)out);
    LAUNCH_CHECK("embed_gather launch");
    return HCP_OK;
}
extern "C" int hcp_upsample2x_fwd_bf16(const void* x, int64_t B, int64_t H, int64_t W, int64_t C, void* y, hcp_stream_t stream_) {
    if (!x || !y || C % 8 != 0) return set_error(HCP_ERR_INVALID, "upsample2x_fwd");
    const int64_t n = B * 4 * H * W * (C / 8);
    launch_k(upsample2x_fwd_kernel, dim3((unsigned)((n + 255) / 256)), dim3(256), 0, (cudaStream_t)stream_, (const __nv_bfloat16*)x, (int)B, (int)H, (int)W,
                                                                                        (int)C, (__nv_bfloat16*)y);
    LAUNCH_CHECK("upsample2x_fwd launch");
    return HCP_OK;
}
extern "C" int hcp_upsample2x_bwd_bf16(const void* dy, int64_t B, int64_t H, int64_t W, int64_t C, void* dx, hcp_stream_t stream_) {
    if (!dy || !dx || C % 8 != 0) return set_error(HCP_ERR_INVALID, "upsample2x_bwd");
    const int64_t n = B * H * W * (C / 8);
    launch_k(upsample2x_bwd_kernel, dim3((unsigned)((n + 255) / 256)), dim3(256), 0, (cudaStream_t)stream_, (const __nv_bfloat16*)dy, (int)B, (int)H, (int)W,
                                                                                        (int)C, (__nv_bfloat16*)dx);
    LAUNCH_CHECK("upsample2x_bwd launch");
    return HCP_OK;
}
extern "C" int hcp_add_bf16(const void* a, const void* b, int64_t n, void* out, hcp_stream_t stream_) {
    if (!a || !b || !out || n % 8 != 0) return set_error(HCP_ERR_INVALID, "add_bf16");
    const int64_t n8 = n / 8;
    launch_k(add_bf16_kernel, dim3((unsigned)((n8 + 255) / 256)), dim3(256), 0, (cudaStream_t)stream_, (const __nv_bfloat16*)a, (const __nv_bfloat16*)b, n8,
                                                                                   (__nv_bfloat16*)out);
    LAUNCH_CHECK("add_bf16 launch");
    return HCP_OK;
}
