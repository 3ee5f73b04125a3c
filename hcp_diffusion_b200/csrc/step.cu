// SPDX-License-Identifier: Apache-2.0
// Training-step kernels either side of the UNet call (sm_90a; the clip and optimizer kernels are in misc.cu and optim.cu):
//   * the eps loss, plain MSE or SNR-weighted (reference hcpdiff/loss/min_snr_loss.py:5-52: MinSNR / SoftMinSNR / KDiffMinSNR /
//     EDM weights), over the data groups of one step with per-sample weights and a per-pixel mask (prior preservation, att_mask;
//     reference hcpdiff/train_ac.py:467-482, 506-515), reduced in a fixed order
//   * exponential moving average of the flat trainable buffer (reference hcpdiff/utils/ema.py:18-32)
//   * nn.Dropout on a patched layer's output (reference hcpdiff/models/lora_base_patch.py:74), counter-based RNG so that the
//     backward pass regenerates the forward mask instead of storing it, and CUDA-graph replays draw fresh masks
//   * the DreamArtist classifier-free-guidance mix of the two UNet halves (reference hcpdiff/models/cfg_context.py:23-39)
//   * pyramid noise (reference hcpdiff/noise/pyramid_noise.py:17-32): device-drawn level sizes, the level grids, their bilinear
//     sum onto the base noise with a per-group std, and add_noise on the normalised sum (1/std = 1: DDPMScheduler.add_noise)
// All of them are HBM-bound elementwise kernels over at most a few MB.
#include <algorithm>
#include <cmath>

#include "common.cuh"
#include "host_util.h"
#include "../../include/hcp_b200.h"

namespace hcp {

#define LAUNCH_CHECK(what)                                              \
    do {                                                                \
        cudaError_t e_ = cudaGetLastError();                            \
        if (e_ != cudaSuccess) return set_cuda_error(e_, what);         \
    } while (0)

// ---------------------------------------------------------------------------------------------
// Min-SNR family loss weights w(t_b) of the eps loss below:
//   snr = acp / (1 - acp)  ( = (alpha/sigma)^2 of min_snr_loss.py:16-19 )
//   mode 0 MinSNR      w = min(gamma / snr, 1)
//   mode 1 SoftMinSNR  w = gamma^3 / (snr^2 + gamma^3)
//   mode 2 KDiffMinSNR w = 4 (gamma snr)^2 / (snr^2 + gamma^2)^2
//   mode 3 EDM         w = (sigma^2 + gamma^2) / (snr (sigma gamma)^2),  sigma = sqrt(1 - acp)
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ float snr_weight(float acp, float gamma, int mode) {
    const float snr = acp / (1.f - acp);
    if (mode == 0) return fminf(gamma / snr, 1.f);
    if (mode == 1) { const float g3 = gamma * gamma * gamma; return g3 / (snr * snr + g3); }
    if (mode == 2) { const float a = gamma * snr, b = snr * snr + gamma * gamma; return 4.f * (a * a) / (b * b); }
    const float s2 = 1.f - acp;
    return (s2 + gamma * gamma) / (snr * (s2 * gamma * gamma));
}

// ---------------------------------------------------------------------------------------------
// Grouped, masked eps loss: the reference's get_loss with its per-pixel mask, (criterion(pred, target) * mask).mean()
// (train_ac.py:506-515), weighted per data group and summed over the groups of one step (train_ac.py:467-482):
//   group_loss[g] += sum_{b in g} scale_b * sum_{c,p} w(t_b) M[b,p] (pred - target)^2,   scale_b = loss_weight_g / (B_g C HW)
//   dpred = 2 w M d scale_b grad_scale
// Grid (chunks, B): block (c, b) covers elements [c * EPS_CHUNK, (c + 1) * EPS_CHUNK) of sample b and writes its partial to
// ws[b * chunks + c]; eps_loss_reduce_kernel then sums ws per group in index order, so the loss bits do not depend on which
// block finishes first (CUDA-graph replays are bit-identical).
// ---------------------------------------------------------------------------------------------
constexpr int64_t EPS_CHUNK = 4096;             // elements per block: 256 threads x 4 float4

template <bool VEC>
__global__ void eps_loss_grouped_kernel(const float* __restrict__ pred, const float* __restrict__ target, const int64_t* __restrict__ t,
                                        const float* __restrict__ acp, const float* __restrict__ mask, const float* __restrict__ scale,
                                        int mode, float gamma, int64_t per_image, int64_t HW, float grad_scale, float* __restrict__ ws,
                                        float* __restrict__ dpred) {
    pdl_trigger();
    pdl_wait();
    __shared__ float s_part[8];
    const int64_t b = blockIdx.y;
    const float w = mode < 0 ? 1.f : snr_weight(acp[t[b]], gamma, mode);
    const float sc = scale[b];
    const float gs = 2.f * w * sc * grad_scale;
    const float* __restrict__ p_s = pred + b * per_image;
    const float* __restrict__ q_s = target + b * per_image;
    float* __restrict__ d_s = dpred ? dpred + b * per_image : nullptr;
    const float* __restrict__ m_s = mask ? mask + b * HW : nullptr;
    const int64_t lo = blockIdx.x * EPS_CHUNK;
    const int64_t hi = min(lo + EPS_CHUNK, per_image);
    float acc = 0.f;
    if (VEC) {                                  // per_image % 4 == 0 and 16-byte aligned operands: lo, hi, i are multiples of 4
        for (int64_t i = lo + 4 * (int64_t)threadIdx.x; i < hi; i += 4 * (int64_t)blockDim.x) {
            const float4 pv = *reinterpret_cast<const float4*>(p_s + i), qv = *reinterpret_cast<const float4*>(q_s + i);
            float4 mv = make_float4(1.f, 1.f, 1.f, 1.f);
            if (m_s) {
                const int64_t px = i % HW;
                if ((HW & 3) == 0) mv = *reinterpret_cast<const float4*>(m_s + px);
                else {                          // the 4 elements may straddle a channel boundary: the pixel index wraps
                    mv.x = m_s[px];
                    mv.y = m_s[px + 1 < HW ? px + 1 : px + 1 - HW];
                    mv.z = m_s[px + 2 < HW ? px + 2 : px + 2 - HW];
                    mv.w = m_s[px + 3 < HW ? px + 3 : px + 3 - HW];
                }
            }
            const float dx = pv.x - qv.x, dy = pv.y - qv.y, dz = pv.z - qv.z, dw = pv.w - qv.w;
            const float mx = mv.x * dx, my = mv.y * dy, mz = mv.z * dz, mw = mv.w * dw;
            acc += mx * dx + my * dy + mz * dz + mw * dw;
            if (d_s) *reinterpret_cast<float4*>(d_s + i) = make_float4(gs * mx, gs * my, gs * mz, gs * mw);
        }
    } else {
        for (int64_t i = lo + threadIdx.x; i < hi; i += blockDim.x) {
            const float d = p_s[i] - q_s[i];
            const float md = (m_s ? m_s[i % HW] : 1.f) * d;
            acc += md * d;
            if (d_s) d_s[i] = gs * md;
        }
    }
    acc = warp_sum(acc);
    if ((threadIdx.x & 31) == 0) s_part[threadIdx.x >> 5] = acc;
    __syncthreads();
    if (threadIdx.x < 32) {
        float v = (threadIdx.x < (blockDim.x >> 5)) ? s_part[threadIdx.x] : 0.f;
        v = warp_sum(v);
        if (threadIdx.x == 0) ws[b * gridDim.x + blockIdx.x] = v * w * sc;
    }
}

// group_loss[g] += sum of ws[b * chunks + c] over samples b of group g, in a fixed order (one block)
__global__ void eps_loss_reduce_kernel(const float* __restrict__ ws, const int32_t* __restrict__ sample_group, int64_t B, int64_t chunks,
                                       int ngroups, float* __restrict__ group_loss) {
    pdl_trigger();
    pdl_wait();
    __shared__ float s_part[8];
    const int64_t n = B * chunks;
    for (int g = 0; g < ngroups; ++g) {
        float acc = 0.f;
        for (int64_t k = threadIdx.x; k < n; k += blockDim.x)
            if (sample_group[k / chunks] == g) acc += ws[k];
        acc = warp_sum(acc);
        if ((threadIdx.x & 31) == 0) s_part[threadIdx.x >> 5] = acc;
        __syncthreads();
        if (threadIdx.x < 32) {
            float v = (threadIdx.x < (blockDim.x >> 5)) ? s_part[threadIdx.x] : 0.f;
            v = warp_sum(v);
            if (threadIdx.x == 0) group_loss[g] += v;
        }
        __syncthreads();
    }
}

// ---------------------------------------------------------------------------------------------
// ema <- lerp(ema, p, 1 - decay),  decay = clip(1 - (1 + step / inv_gamma)^(-power), 0, decay_max)   (ema.py:18-27; `step`
// is the optimizer's device-side step counter AFTER its increment, i.e. ModelEMA.step after `self.step += 1`)
// ---------------------------------------------------------------------------------------------
__global__ void ema_flat_kernel(float* __restrict__ ema, const float* __restrict__ p, int64_t n, const int* __restrict__ step_ptr,
                                float decay_max, float inv_gamma, float power) {
    pdl_trigger();
    pdl_wait();
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= n) return;
    float decay = 1.f - powf(1.f + (float)(*step_ptr) / inv_gamma, -power);
    decay = fminf(fmaxf(decay, 0.f), decay_max);
    const float e = ema[i];
    ema[i] = e + (1.f - decay) * (p[i] - e);
}

// ---------------------------------------------------------------------------------------------
// Philox4x32-10 (Salmon et al. 2011): counter (element group, site, draw), key (seed) -> 4 x 32 random bits
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ uint4 philox4x32_10(uint4 ctr, uint2 key) {
#pragma unroll
    for (int r = 0; r < 10; ++r) {
        const uint32_t hi0 = __umulhi(0xD2511F53u, ctr.x), lo0 = 0xD2511F53u * ctr.x;
        const uint32_t hi1 = __umulhi(0xCD9E8D57u, ctr.z), lo1 = 0xCD9E8D57u * ctr.z;
        ctr = make_uint4(hi1 ^ ctr.y ^ key.x, lo1, hi0 ^ ctr.w ^ key.y, lo0);
        key.x += 0x9E3779B9u;
        key.y += 0xBB67AE85u;
    }
    return ctr;
}

// out[r, c] = keep(r, c) * x[r, c] / (1 - p) (+ res[r, c]) (+ rowbias[r / rows_per_group, c]) for the columns [0, ncols) of a
// row-major bf16 matrix (ncols % 8 == 0).
// keep is a function of (seed, draw counter, site, r, c) only: calling the kernel on the gradient with the same state[] and site
// applies the forward mask.  state = {seed, draw}: `draw` is advanced once per training step by hcp_counter_add_u64.
__global__ void dropout_bf16_kernel(const __nv_bfloat16* __restrict__ x, int64_t ldx, const __nv_bfloat16* __restrict__ res, int64_t ldr,
                                    const float* __restrict__ rowbias, int64_t rowbias_ld, int64_t rows_per_group,
                                    int64_t rows, int ncols, float p, const unsigned long long* __restrict__ state, uint32_t site,
                                    __nv_bfloat16* __restrict__ out, int64_t ldo) {
    pdl_trigger();
    pdl_wait();
    const int vec_per_row = ncols >> 3;
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= rows * vec_per_row) return;
    const int64_t r = i / vec_per_row;
    const int c = (int)(i % vec_per_row) * 8;
    const unsigned long long seed = state[0], draw = state[1];
    const uint4 rnd = philox4x32_10(make_uint4((uint32_t)i, (uint32_t)(i >> 32), site, (uint32_t)draw),
                                    make_uint2((uint32_t)seed, (uint32_t)(seed >> 32) ^ (uint32_t)(draw >> 32)));
    const uint32_t thr = (uint32_t)(p * 65536.f);          // element dropped when its 16 random bits are < thr
    const float inv = 1.f / (1.f - p);
    const uint4 xv = *reinterpret_cast<const uint4*>(x + r * ldx + c);
    uint4 rv = make_uint4(0u, 0u, 0u, 0u);
    if (res) rv = *reinterpret_cast<const uint4*>(res + r * ldr + c);
    const uint32_t xs[4] = {xv.x, xv.y, xv.z, xv.w}, rs[4] = {rv.x, rv.y, rv.z, rv.w}, rn[4] = {rnd.x, rnd.y, rnd.z, rnd.w};
    float rb[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    if (rowbias) {
        const float* src = rowbias + (r / rows_per_group) * rowbias_ld + c;
        const float4 b0 = *reinterpret_cast<const float4*>(src), b1 = *reinterpret_cast<const float4*>(src + 4);
        rb[0] = b0.x; rb[1] = b0.y; rb[2] = b0.z; rb[3] = b0.w; rb[4] = b1.x; rb[5] = b1.y; rb[6] = b1.z; rb[7] = b1.w;
    }
    uint32_t os[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        const float2 v = unpack_bf16x2(xs[j]);
        const float2 a = unpack_bf16x2(rs[j]);
        const float lo = ((rn[j] & 0xFFFFu) >= thr ? v.x * inv : 0.f) + a.x + rb[2 * j];
        const float hi = ((rn[j] >> 16) >= thr ? v.y * inv : 0.f) + a.y + rb[2 * j + 1];
        os[j] = pack_bf16x2(lo, hi);
    }
    *reinterpret_cast<uint4*>(out + r * ldo + c) = make_uint4(os[0], os[1], os[2], os[3]);
}

__global__ void counter_add_u64_kernel(unsigned long long* ctr, unsigned long long inc) {
    pdl_trigger();
    pdl_wait();
    *ctr += inc;
}

// ---------------------------------------------------------------------------------------------
// DreamArtist CFG mix (cfg_context.py:23-39): pred[b] = e_u[b] + s(t_b) (e_c[b] - e_u[b]),  eps2 = [e_u | e_c] (2B images)
//   s = (hi - lo) * rate + lo,  rate = t / (T - 1) shaped by mode: 0 'ln' (linear), 1 'cos' cos((rate-1) pi/2), 2 'cos2' 1 - cos(rate pi/2);
//   lo == hi gives the constant scale.  fwd: out = mix;  bwd (dout given): d_eps2 = [(1 - s) dout | s dout]
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ float cfg_scale_of(int64_t t, float lo, float hi, int mode, int num_train_timesteps) {
    if (lo == hi) return lo;
    float rate = (float)t / (float)(num_train_timesteps - 1);
    if (mode == 1) rate = cosf((rate - 1.f) * 1.5707963267948966f);
    else if (mode == 2) rate = 1.f - cosf(rate * 1.5707963267948966f);
    return (hi - lo) * rate + lo;
}
__global__ void cfg_mix_fwd_kernel(const float* __restrict__ eps2, const int64_t* __restrict__ t, int64_t B, int64_t per_image, float lo,
                                   float hi, int mode, int T, float* __restrict__ out) {
    pdl_trigger();
    pdl_wait();
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= B * per_image) return;
    const float s = cfg_scale_of(t[i / per_image], lo, hi, mode, T);
    const float u = eps2[i], c = eps2[B * per_image + i];
    out[i] = u + s * (c - u);
}
__global__ void cfg_mix_bwd_kernel(const float* __restrict__ dout, const int64_t* __restrict__ t, int64_t B, int64_t per_image, float lo,
                                   float hi, int mode, int T, float* __restrict__ deps2) {
    pdl_trigger();
    pdl_wait();
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= B * per_image) return;
    const float s = cfg_scale_of(t[i / per_image], lo, hi, mode, T);
    const float g = dout[i];
    deps2[i] = (1.f - s) * g;
    deps2[B * per_image + i] = s * g;
}

// ---------------------------------------------------------------------------------------------
// Pyramid (multi-resolution) noise, PyramidNoiseScheduler.add_noise (reference hcpdiff/noise/pyramid_noise.py:17-32), per data
// group g (batch rows [group_start[g], group_start[g + 1])):
//   for i in 1 .. level-1:  r = 2 U + step_size;  hn, wn = max(1, int(h / r^i)), max(1, int(w / r^i))    (float64, truncation)
//                           noise += bilinear(randn(b_g, c, hn, wn), (h, w)) * fp32(discount^i);  break after wn == 1 or hn == 1
//   inv_std[g] = 1 / std(noise over the group's b_g c h w elements, unbiased)
// Random numbers: Philox4x32-10 on a {seed, draw} state of its own (not the dropout state), key (seed_lo, seed_hi ^ draw_hi):
//   U of level i         counter (i, 0xFFFFFFFF, g, draw_lo), U = ((w0 >> 5) 2^26 + (w1 >> 6)) / 2^53  (53-bit double)
//   grid of level i      counter (q, i, g, draw_lo) for elements 4q .. 4q+3 of the group's [b_g, c, hn, wn] grid; Box-Muller in
//                        float64 on (w0, w1) and (w2, w3): u1 = (w + 1) 2^-32, u2 = w' 2^-32, z = sqrt(-2 ln u1) (cos, sin)(2 pi u2)
// ---------------------------------------------------------------------------------------------
constexpr int PYR_MAX_LEVEL = HCP_PYRAMID_MAX_LEVEL;
constexpr int PYR_MAX_GROUPS = HCP_PYRAMID_MAX_GROUPS;
constexpr int PYR_ROW = HCP_PYRAMID_PLAN_INTS;
constexpr int64_t PYR_CHUNK = 4096;             // output elements per block of the sum kernel

// Worst-case grid sizes (r = step_size, the smallest ratio): every level grid has a fixed slot in the workspace.  Computed on the
// host only and passed by value, so the kernels that write and read the grids agree on the layout.
struct PyrCaps {
    int32_t nlev;                               // levels of the worst case, early break included
    int32_t h[PYR_MAX_LEVEL], w[PYR_MAX_LEVEL];
    int64_t slot[PYR_MAX_LEVEL];                // floats per sample: C * h * w
    int64_t off[PYR_MAX_LEVEL];                 // first float of the level's [B, slot] block
    int64_t grid_floats;
};

static PyrCaps pyramid_caps(int64_t B, int64_t C, int64_t H, int64_t W, int level, double step_size) {
    PyrCaps c;
    memset(&c, 0, sizeof(c));
    int64_t off = 0;
    for (int i = 1; i < level; ++i) {
        const double p = pow(step_size, (double)i);
        const int64_t hn = std::max<int64_t>(1, (int64_t)((double)H / p)), wn = std::max<int64_t>(1, (int64_t)((double)W / p));
        c.h[i - 1] = (int32_t)hn;
        c.w[i - 1] = (int32_t)wn;
        c.slot[i - 1] = C * hn * wn;
        c.off[i - 1] = off;
        off += B * C * hn * wn;
        c.nlev = i;
        if (hn == 1 || wn == 1) break;
    }
    c.grid_floats = off;
    return c;
}

__device__ __forceinline__ uint2 pyramid_key(const unsigned long long* state) {
    const unsigned long long seed = state[0], draw = state[1];
    return make_uint2((uint32_t)seed, (uint32_t)(seed >> 32) ^ (uint32_t)(draw >> 32));
}

__global__ void pyramid_plan_kernel(const unsigned long long* __restrict__ state, int ngroups, int level, double step_size, int64_t H,
                                    int64_t W, int32_t* __restrict__ plan) {
    pdl_trigger();
    pdl_wait();
    const int g = threadIdx.x;
    if (g >= ngroups) return;
    const uint2 key = pyramid_key(state);
    const uint32_t draw_lo = (uint32_t)state[1];
    int32_t* row = plan + g * PYR_ROW;
    int n = 0;
    for (int i = 1; i < level; ++i) {
        const uint4 w = philox4x32_10(make_uint4((uint32_t)i, 0xFFFFFFFFu, (uint32_t)g, draw_lo), key);
        const double u = ((double)(w.x >> 5) * 67108864.0 + (double)(w.y >> 6)) / 9007199254740992.0;
        const double r = u * 2.0 + step_size;
        const double p = pow(r, (double)i);
        const int64_t wn = max((int64_t)1, (int64_t)((double)W / p)), hn = max((int64_t)1, (int64_t)((double)H / p));
        row[2 * i] = (int32_t)hn;
        row[2 * i + 1] = (int32_t)wn;
        n = i;
        if (wn == 1 || hn == 1) break;
    }
    row[0] = n;
    row[1] = 0;
    for (int k = 2 * n + 2; k < PYR_ROW; ++k) row[k] = 0;
}

__device__ __forceinline__ int pyramid_group_of(const int32_t* __restrict__ group_start, int ngroups, int64_t b) {
    int g = 0;
    while (g + 1 < ngroups && b >= group_start[g + 1]) ++g;
    return g;
}

// Plan row of a group as the sum kernels read it: the level count clamped to [0, caps.nlev], each size to [1, its worst case]
__device__ __forceinline__ int pyramid_levels(const int32_t* __restrict__ row, const PyrCaps& caps) {
    return min(max(row[0], 0), caps.nlev);
}
__device__ __forceinline__ void pyramid_size(const int32_t* __restrict__ row, const PyrCaps& caps, int k, int* hn, int* wn) {
    *hn = min(max(row[2 + 2 * k], 1), caps.h[k]);
    *wn = min(max(row[3 + 2 * k], 1), caps.w[k]);
}

// One thread per 4 grid elements of (level blockIdx.y + 1, group blockIdx.z)
__global__ void pyramid_grid_kernel(const int32_t* __restrict__ plan, const int32_t* __restrict__ group_start,
                                    const unsigned long long* __restrict__ state, PyrCaps caps, int64_t C, float* __restrict__ grid) {
    pdl_trigger();
    pdl_wait();
    const int k = blockIdx.y, g = blockIdx.z;
    const int32_t* row = plan + g * PYR_ROW;
    if (k >= pyramid_levels(row, caps)) return;
    int hn, wn;
    pyramid_size(row, caps, k, &hn, &wn);
    const int64_t b0 = group_start[g], bg = group_start[g + 1] - b0;
    const int64_t per = C * hn * wn;
    const int64_t q = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (4 * q >= bg * per) return;
    const uint4 w = philox4x32_10(make_uint4((uint32_t)q, (uint32_t)(k + 1), (uint32_t)g, (uint32_t)state[1]), pyramid_key(state));
    const uint32_t ws[4] = {w.x, w.y, w.z, w.w};
    float z[4];
#pragma unroll
    for (int j = 0; j < 4; j += 2) {
        const double u1 = ((double)ws[j] + 1.0) * 2.3283064365386963e-10, u2 = (double)ws[j + 1] * 2.3283064365386963e-10;
        const double rad = sqrt(-2.0 * log(u1));
        double s, c;
        sincospi(2.0 * u2, &s, &c);
        z[j] = (float)(rad * c);
        z[j + 1] = (float)(rad * s);
    }
    float* base = grid + caps.off[k];
    for (int j = 0; j < 4; ++j) {
        const int64_t e = 4 * q + j;
        if (e >= bg * per) break;
        const int64_t b = b0 + e / per;
        base[b * caps.slot[k] + e % per] = z[j];
    }
}

// PyTorch's bilinear source index (align_corners=False, fp32): src = max(scale (dst + 0.5) - 0.5, 0), scale = in / out, with the
// single rounding of the fused multiply-add torch's compiled kernels use (two roundings are up to 2e-5 off near in == out)
__device__ __forceinline__ void bilinear_index(float scale, int64_t dst, int in, int* i0, int* i1, float* l0, float* l1) {
    float src = __fmaf_rn(scale, (float)dst + 0.5f, -0.5f);
    src = fmaxf(src, 0.f);
    const int i = min((int)floorf(src), in - 1);
    const float l = fminf(fmaxf(src - (float)i, 0.f), 1.f);
    *i0 = i;
    *i1 = i + (i < in - 1 ? 1 : 0);
    *l1 = l;
    *l0 = 1.f - l;
}

// target = noise + sum_k bilinear(grid_k) * d_k (fp32, level order) per element; block (chunk, sample) writes its fp64 (sum, sum sq)
// to part[2 * (b * chunks + chunk)]
__global__ void pyramid_sum_kernel(const float* __restrict__ noise, const int32_t* __restrict__ plan, const int32_t* __restrict__ group_start,
                                   int ngroups, double discount, PyrCaps caps, int64_t C, int64_t H, int64_t W, const float* __restrict__ grid,
                                   float* __restrict__ target, double* __restrict__ part) {
    pdl_trigger();
    pdl_wait();
    __shared__ double s_part[2][8];
    __shared__ int s_n, s_hn[PYR_MAX_LEVEL], s_wn[PYR_MAX_LEVEL];
    __shared__ float s_d[PYR_MAX_LEVEL];
    const int64_t b = blockIdx.y;
    if (threadIdx.x == 0) {
        const int32_t* row = plan + pyramid_group_of(group_start, ngroups, b) * PYR_ROW;
        s_n = pyramid_levels(row, caps);
        for (int k = 0; k < s_n; ++k) {
            pyramid_size(row, caps, k, &s_hn[k], &s_wn[k]);
            s_d[k] = (float)pow(discount, (double)(k + 1));     // Python's discount**i, then rounded to fp32 as torch does
        }
    }
    __syncthreads();
    const int n = s_n;
    const int* hn = s_hn;
    const int* wn = s_wn;
    const int64_t HW = H * W, per_image = C * HW;
    const int64_t lo = blockIdx.x * PYR_CHUNK, hi = min(lo + PYR_CHUNK, per_image);
    double s = 0.0, sq = 0.0;
    for (int64_t i = lo + threadIdx.x; i < hi; i += blockDim.x) {
        const int64_t c = i / HW, p = i % HW, y = p / W, x = p % W;
        float v = noise[b * per_image + i];
        for (int k = 0; k < n; ++k) {
            int y0, y1, x0, x1;
            float ly0, ly1, lx0, lx1;
            bilinear_index((float)hn[k] / (float)H, y, hn[k], &y0, &y1, &ly0, &ly1);
            bilinear_index((float)wn[k] / (float)W, x, wn[k], &x0, &x1, &lx0, &lx1);
            const float* gk = grid + caps.off[k] + b * caps.slot[k] + c * hn[k] * wn[k];
            const float t0 = __fadd_rn(__fmul_rn(gk[y0 * wn[k] + x0], lx0), __fmul_rn(gk[y0 * wn[k] + x1], lx1));
            const float t1 = __fadd_rn(__fmul_rn(gk[y1 * wn[k] + x0], lx0), __fmul_rn(gk[y1 * wn[k] + x1], lx1));
            const float up = __fadd_rn(__fmul_rn(t0, ly0), __fmul_rn(t1, ly1));
            v = __fadd_rn(v, __fmul_rn(up, s_d[k]));
        }
        target[b * per_image + i] = v;
        s += (double)v;
        sq += (double)v * (double)v;
    }
    for (int o = 16; o > 0; o >>= 1) {
        s += __shfl_down_sync(0xFFFFFFFFu, s, o);
        sq += __shfl_down_sync(0xFFFFFFFFu, sq, o);
    }
    if ((threadIdx.x & 31) == 0) {
        s_part[0][threadIdx.x >> 5] = s;
        s_part[1][threadIdx.x >> 5] = sq;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        double a = 0.0, q = 0.0;
        for (int w = 0; w < (int)(blockDim.x >> 5); ++w) {
            a += s_part[0][w];
            q += s_part[1][w];
        }
        part[2 * (b * gridDim.x + blockIdx.x)] = a;
        part[2 * (b * gridDim.x + blockIdx.x) + 1] = q;
    }
}

// inv_std[g] = 1 / sqrt((sum sq - sum^2 / N) / (N - 1)) over the group's partials, summed in a fixed order (one block)
__global__ void pyramid_std_kernel(const double* __restrict__ part, const int32_t* __restrict__ group_start, int ngroups, int64_t chunks,
                                   int64_t per_image, float* __restrict__ inv_std) {
    pdl_trigger();
    pdl_wait();
    __shared__ double s_part[2][8];
    for (int g = 0; g < ngroups; ++g) {
        const int64_t k0 = group_start[g] * chunks, k1 = group_start[g + 1] * chunks;
        double s = 0.0, sq = 0.0;
        for (int64_t k = k0 + threadIdx.x; k < k1; k += blockDim.x) {
            s += part[2 * k];
            sq += part[2 * k + 1];
        }
        for (int o = 16; o > 0; o >>= 1) {
            s += __shfl_down_sync(0xFFFFFFFFu, s, o);
            sq += __shfl_down_sync(0xFFFFFFFFu, sq, o);
        }
        if ((threadIdx.x & 31) == 0) {
            s_part[0][threadIdx.x >> 5] = s;
            s_part[1][threadIdx.x >> 5] = sq;
        }
        __syncthreads();
        if (threadIdx.x == 0) {
            double a = 0.0, q = 0.0;
            for (int w = 0; w < (int)(blockDim.x >> 5); ++w) {
                a += s_part[0][w];
                q += s_part[1][w];
            }
            const double N = (double)((group_start[g + 1] - group_start[g]) * per_image);
            inv_std[g] = (float)(1.0 / sqrt((q - a * (a / N)) / (N - 1.0)));
        }
        __syncthreads();
    }
}

// x_t = sqrt(acp[t]) x0 + sqrt(1 - acp[t]) (noise inv_std[group(b)])   (DDPMScheduler.add_noise on the normalised pyramid noise)
__global__ void add_noise_scaled_kernel(const float* __restrict__ x0, const float* __restrict__ noise, const int64_t* __restrict__ t,
                                        const float* __restrict__ acp, const float* __restrict__ inv_std, const int32_t* __restrict__ group_start,
                                        int ngroups, int64_t per_image, int64_t n, float* __restrict__ xt) {
    pdl_trigger();
    pdl_wait();
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int64_t b = i / per_image;
    const float a = acp[t[b]];
    const float nz = noise[i] * inv_std[pyramid_group_of(group_start, ngroups, b)];
    xt[i] = sqrtf(a) * x0[i] + sqrtf(1.f - a) * nz;
}

}  // namespace hcp

using namespace hcp;

extern "C" size_t hcp_eps_loss_grouped_workspace_bytes(int64_t B, int64_t per_image) {
    if (B <= 0 || per_image <= 0) return 0;
    return (size_t)B * (size_t)((per_image + EPS_CHUNK - 1) / EPS_CHUNK) * sizeof(float);
}

extern "C" int hcp_eps_loss_grouped(const float* pred, const float* target, const int64_t* t, const float* alphas_cumprod, const float* mask,
                                    const float* sample_scale, const int32_t* sample_group, int32_t ngroups, int32_t mode, float gamma,
                                    int64_t B, int64_t C, int64_t HW, float grad_scale, float* group_loss, float* dpred, void* workspace,
                                    size_t workspace_bytes, hcp_stream_t st) {
    if (!pred || !target || !sample_scale || !sample_group || !group_loss || !workspace)
        return set_error(HCP_ERR_INVALID, "eps_loss_grouped: null pointer");
    if (mode < -1 || mode > 3 || (mode >= 0 && (!t || !alphas_cumprod || !(gamma > 0.f))))
        return set_error(HCP_ERR_INVALID, "eps_loss_grouped: mode -1 (MSE) or 0..3 (SNR weights with t, alphas_cumprod and gamma > 0)");
    if (B <= 0 || B > 65535 || C <= 0 || HW <= 0 || ngroups <= 0)
        return set_error(HCP_ERR_INVALID, "eps_loss_grouped: shape (0 < B <= 65535, C, HW, ngroups > 0)");
    const int64_t per_image = C * HW;
    const int64_t chunks = (per_image + EPS_CHUNK - 1) / EPS_CHUNK;
    if (workspace_bytes < hcp_eps_loss_grouped_workspace_bytes(B, per_image))
        return set_error(HCP_ERR_INVALID, "eps_loss_grouped: workspace smaller than hcp_eps_loss_grouped_workspace_bytes(B, C * HW)");
    const bool aligned = ((uintptr_t)pred | (uintptr_t)target | (uintptr_t)(dpred ? dpred : pred) | (uintptr_t)(mask ? mask : pred)) % 16 == 0;
    const bool vec = aligned && (per_image % 4) == 0 && HW >= 4;
    const dim3 grid((unsigned)chunks, (unsigned)B);
    float* ws = (float*)workspace;
    if (vec) launch_k(eps_loss_grouped_kernel<true>, grid, dim3(256), 0, (cudaStream_t)st, pred, target, t, alphas_cumprod, mask, sample_scale,
                      (int)mode, gamma, per_image, HW, grad_scale, ws, dpred);
    else launch_k(eps_loss_grouped_kernel<false>, grid, dim3(256), 0, (cudaStream_t)st, pred, target, t, alphas_cumprod, mask, sample_scale,
                  (int)mode, gamma, per_image, HW, grad_scale, ws, dpred);
    LAUNCH_CHECK("eps_loss_grouped launch");
    launch_k(eps_loss_reduce_kernel, dim3(1), dim3(256), 0, (cudaStream_t)st, (const float*)ws, sample_group, B, chunks, (int)ngroups, group_loss);
    LAUNCH_CHECK("eps_loss_grouped reduce launch");
    return HCP_OK;
}

extern "C" int hcp_ema_flat(float* ema, const float* p, int64_t n, const int* step_device, float decay_max, float inv_gamma, float power,
                            hcp_stream_t st) {
    if (!ema || !p || !step_device || n <= 0) return set_error(HCP_ERR_INVALID, "ema_flat: arguments");
    launch_k(ema_flat_kernel, dim3((unsigned)((n + 255) / 256)), dim3(256), 0, (cudaStream_t)st, ema, p, n, step_device, decay_max, inv_gamma, power);
    LAUNCH_CHECK("ema_flat launch");
    return HCP_OK;
}

extern "C" int hcp_dropout_bf16(const void* x, int64_t ldx, const void* residual, int64_t ldr, const float* rowbias, int64_t rowbias_ld,
                                int64_t rows_per_group, int64_t rows, int64_t ncols, float p, const uint64_t* state_device, uint32_t site,
                                void* out, int64_t ldo, hcp_stream_t st) {
    if (!x || !out || !state_device) return set_error(HCP_ERR_INVALID, "dropout: null pointer");
    if (rows <= 0 || ncols <= 0 || (ncols % 8) || (ldx % 8) || (ldo % 8) || (residual && (ldr % 8)) || !(p >= 0.f && p < 1.f) ||
        (rowbias && (rows_per_group <= 0 || (rowbias_ld % 4))))
        return set_error(HCP_ERR_INVALID, "dropout: shape (columns and pitches in multiples of 8, 0 <= p < 1)");
    if (!aligned16(x, residual, rowbias, out))
        return set_error(HCP_ERR_INVALID, "dropout: buffers must be 16-byte aligned");
    const int64_t n = rows * (ncols / 8);
    launch_k(dropout_bf16_kernel, dim3((unsigned)((n + 255) / 256)), dim3(256), 0, (cudaStream_t)st, (const __nv_bfloat16*)x, ldx,
             (const __nv_bfloat16*)residual, ldr, rowbias, rowbias_ld, rows_per_group, rows, (int)ncols, p, (const unsigned long long*)state_device, site, (__nv_bfloat16*)out, ldo);
    LAUNCH_CHECK("dropout launch");
    return HCP_OK;
}

extern "C" int hcp_counter_add_u64(uint64_t* counter_device, uint64_t inc, hcp_stream_t st) {
    if (!counter_device) return set_error(HCP_ERR_INVALID, "counter_add: null pointer");
    launch_k(counter_add_u64_kernel, dim3(1), dim3(1), 0, (cudaStream_t)st, (unsigned long long*)counter_device, (unsigned long long)inc);
    LAUNCH_CHECK("counter_add launch");
    return HCP_OK;
}

extern "C" int hcp_cfg_mix_f32(const float* eps2, const float* dout, const int64_t* t, int64_t B, int64_t per_image, float scale_lo,
                               float scale_hi, int32_t mode, int32_t num_train_timesteps, float* out, hcp_stream_t st) {
    if (!t || !out || (!eps2 && !dout) || B <= 0 || per_image <= 0 || mode < 0 || mode > 2 || num_train_timesteps < 2)
        return set_error(HCP_ERR_INVALID, "cfg_mix: arguments");
    const int64_t n = B * per_image;
    const dim3 grid((unsigned)((n + 255) / 256));
    if (dout) launch_k(cfg_mix_bwd_kernel, grid, dim3(256), 0, (cudaStream_t)st, dout, t, B, per_image, scale_lo, scale_hi, (int)mode, (int)num_train_timesteps, out);
    else launch_k(cfg_mix_fwd_kernel, grid, dim3(256), 0, (cudaStream_t)st, eps2, t, B, per_image, scale_lo, scale_hi, (int)mode, (int)num_train_timesteps, out);
    LAUNCH_CHECK("cfg_mix launch");
    return HCP_OK;
}

template <typename T>
static bool aligned_to(const T* p) {
    return ((uintptr_t)p % sizeof(T)) == 0;
}

static int pyramid_check(int32_t ngroups, int32_t level, double step_size, int64_t H, int64_t W) {
    if (ngroups < 1 || ngroups > PYR_MAX_GROUPS) return set_error(HCP_ERR_INVALID, "pyramid: ngroups in [1, HCP_PYRAMID_MAX_GROUPS]");
    if (level < 1 || level > PYR_MAX_LEVEL) return set_error(HCP_ERR_INVALID, "pyramid: level in [1, HCP_PYRAMID_MAX_LEVEL]");
    if (!(step_size >= 1.0) || !std::isfinite(step_size))
        return set_error(HCP_ERR_INVALID, "pyramid: step_size must be >= 1 (a ratio below 1 makes grids larger than the latent)");
    if (H <= 0 || W <= 0 || H > INT32_MAX || W > INT32_MAX) return set_error(HCP_ERR_INVALID, "pyramid: latent height and width");
    return HCP_OK;
}

extern "C" int hcp_pyramid_plan(const uint64_t* state_device, int32_t ngroups, int32_t level, double step_size, int64_t H, int64_t W,
                                int32_t* plan, hcp_stream_t st) {
    if (!state_device || !plan) return set_error(HCP_ERR_INVALID, "pyramid_plan: null pointer");
    if (!aligned_to(state_device) || !aligned_to(plan)) return set_error(HCP_ERR_INVALID, "pyramid_plan: misaligned pointer");
    const int rc = pyramid_check(ngroups, level, step_size, H, W);
    if (rc != HCP_OK) return rc;
    launch_k(pyramid_plan_kernel, dim3(1), dim3(PYR_MAX_GROUPS), 0, (cudaStream_t)st, (const unsigned long long*)state_device, (int)ngroups,
             (int)level, step_size, H, W, plan);
    LAUNCH_CHECK("pyramid_plan launch");
    return HCP_OK;
}

static size_t pyramid_part_bytes(int64_t B, int64_t per_image) {
    return (size_t)B * (size_t)((per_image + PYR_CHUNK - 1) / PYR_CHUNK) * 2 * sizeof(double);
}

extern "C" size_t hcp_pyramid_workspace_bytes(int64_t B, int64_t C, int64_t H, int64_t W, int32_t level, double step_size) {
    if (B <= 0 || C <= 0 || H <= 0 || W <= 0 || level < 1 || level > PYR_MAX_LEVEL || !(step_size >= 1.0) || !std::isfinite(step_size))
        return 0;
    return pyramid_part_bytes(B, C * H * W) + (size_t)pyramid_caps(B, C, H, W, level, step_size).grid_floats * sizeof(float);
}

extern "C" int hcp_pyramid_noise(const float* noise, const int32_t* plan, const int32_t* group_start, int32_t ngroups,
                                 const uint64_t* state_device, int32_t level, double discount, double step_size, int64_t B, int64_t C,
                                 int64_t H, int64_t W, float* target, float* inv_std, void* workspace, size_t workspace_bytes,
                                 hcp_stream_t st) {
    if (!noise || !plan || !group_start || !state_device || !target || !inv_std || !workspace)
        return set_error(HCP_ERR_INVALID, "pyramid_noise: null pointer");
    if (!aligned_to(noise) || !aligned_to(plan) || !aligned_to(group_start) || !aligned_to(state_device) || !aligned_to(target) ||
        !aligned_to(inv_std) || ((uintptr_t)workspace % 16))
        return set_error(HCP_ERR_INVALID, "pyramid_noise: misaligned pointer (elements at their size, workspace at 16 bytes)");
    int rc = pyramid_check(ngroups, level, step_size, H, W);
    if (rc != HCP_OK) return rc;
    if (!std::isfinite(discount)) return set_error(HCP_ERR_INVALID, "pyramid_noise: discount must be finite");
    if (B < 0 || C <= 0 || B > 65535) return set_error(HCP_ERR_INVALID, "pyramid_noise: shape (0 <= B <= 65535, C > 0)");
    if (B == 0) return HCP_OK;
    if (ngroups > B) return set_error(HCP_ERR_INVALID, "pyramid_noise: more groups than samples");
    if (workspace_bytes < hcp_pyramid_workspace_bytes(B, C, H, W, level, step_size))
        return set_error(HCP_ERR_INVALID, "pyramid_noise: workspace smaller than hcp_pyramid_workspace_bytes");
    const PyrCaps caps = pyramid_caps(B, C, H, W, level, step_size);
    const int64_t per_image = C * H * W, chunks = (per_image + PYR_CHUNK - 1) / PYR_CHUNK;
    double* part = (double*)workspace;
    float* grid = (float*)((char*)workspace + pyramid_part_bytes(B, per_image));
    if (caps.nlev > 0) {
        int64_t quads = 0;
        for (int k = 0; k < caps.nlev; ++k) quads = std::max(quads, (B * caps.slot[k] + 3) / 4);
        launch_k(pyramid_grid_kernel, dim3((unsigned)((quads + 255) / 256), (unsigned)caps.nlev, (unsigned)ngroups), dim3(256), 0,
                 (cudaStream_t)st, plan, group_start, (const unsigned long long*)state_device, caps, C, grid);
        LAUNCH_CHECK("pyramid_noise grid launch");
    }
    launch_k(pyramid_sum_kernel, dim3((unsigned)chunks, (unsigned)B), dim3(256), 0, (cudaStream_t)st, noise, plan, group_start, (int)ngroups,
             discount, caps, C, H, W, (const float*)grid, target, part);
    LAUNCH_CHECK("pyramid_noise sum launch");
    launch_k(pyramid_std_kernel, dim3(1), dim3(256), 0, (cudaStream_t)st, (const double*)part, group_start, (int)ngroups, chunks, per_image,
             inv_std);
    LAUNCH_CHECK("pyramid_noise std launch");
    return HCP_OK;
}

extern "C" int hcp_add_noise_scaled(const float* x0, const float* noise, const int64_t* t, const float* alphas_cumprod, const float* inv_std,
                                    const int32_t* group_start, int32_t ngroups, int64_t B, int64_t per_image, float* xt, hcp_stream_t st) {
    if (!x0 || !noise || !t || !alphas_cumprod || !inv_std || !group_start || !xt)
        return set_error(HCP_ERR_INVALID, "add_noise_scaled: null pointer");
    if (!aligned_to(x0) || !aligned_to(noise) || !aligned_to(t) || !aligned_to(alphas_cumprod) || !aligned_to(inv_std) ||
        !aligned_to(group_start) || !aligned_to(xt))
        return set_error(HCP_ERR_INVALID, "add_noise_scaled: misaligned pointer");
    if (B < 0 || per_image < 0 || ngroups < 1 || ngroups > PYR_MAX_GROUPS)
        return set_error(HCP_ERR_INVALID, "add_noise_scaled: sizes (B, per_image >= 0, ngroups in [1, HCP_PYRAMID_MAX_GROUPS])");
    const int64_t n = B * per_image;
    if (n == 0) return HCP_OK;
    launch_k(add_noise_scaled_kernel, dim3((unsigned)((n + 255) / 256)), dim3(256), 0, (cudaStream_t)st, x0, noise, t, alphas_cumprod, inv_std,
             group_start, (int)ngroups, per_image, n, xt);
    LAUNCH_CHECK("add_noise_scaled launch");
    return HCP_OK;
}
