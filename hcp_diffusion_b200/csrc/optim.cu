// SPDX-License-Identifier: Apache-2.0
// Adafactor (transformers.optimization.Adafactor.step) over the flat fp32 parameter buffer of the training step (sm_90a), and
// Lion (lion_pytorch.Lion.step, one elementwise kernel at the end of this file).
//
// Every trainable tensor keeps its module shape: a tensor with two or more dims is factored over its LAST TWO dims, viewed as
// [P, R, C] with the leading dims a batch (a Conv2d weight [O, I, 3, 3] is P = O*I slabs of 3 x 3); a 1-D tensor keeps an
// elementwise second moment.  Per tensor p with (scaled, clipped) gradient g:
//   rms_p = sqrt(mean(p^2)) (before the update),  lr_t = (relative_step ? min(warmup ? 1e-6 step : 1e-2, 1/sqrt(step)) : lr)
//                                                        * (scale_parameter ? max(eps2, rms_p) : 1)
//   q = g^2 + eps1;  row = b2 row + (1-b2) mean_C(q);  col = b2 col + (1-b2) mean_R(q);  u = g rsqrt(row / mean_R(row)) rsqrt(col)
//   (1-D: v = b2 v + (1-b2) q;  u = g rsqrt(v)),   u = u / max(1, rms(u) / clip_threshold) * lr_t,   [m = b1 m + (1-b1) u; u = m]
//   p = p - weight_decay lr_t p - u
//
// One launch per pass covers every tensor.  The host cuts each tensor into tiles ("items", about 64K elements: up to 256 rows x
// 256 columns of one slab, or whole small slabs side by side) and passes the list; one CTA per item.
//   (a) stats:  q of the tile staged 16 rows at a time in shared memory; row sums by groups of lanes, column sums in registers,
//               the tile's sum of p^2.  A row (column) sum that the tile holds completely updates the EMA in place; otherwise the
//               partial sum goes to the work buffer ([rows, column tiles] / [row chunks, columns]).
//   (b) factors: partial sums -> EMAs, and mean_R(row) per slab (one CTA per slab when R >= 32, else one thread per slab).
//   (c) rms:    sum of u^2 per tile (u recomputed from g and the factors).
//   (d) apply:  per-tensor totals of (a) and (c) summed in a fixed order, then the update; u is recomputed, never stored.
// Every reduction has a fixed order, so two runs from the same state give bit-identical results.  Only elements of the tensors are
// written: the 16-byte padding between tensors in the flat buffer and the gradient are never touched.
#include "common.cuh"
#include "host_util.h"
#include "../../include/hcp_b200.h"

namespace hcp {

#define LAUNCH_CHECK(what)                                              \
    do {                                                                \
        cudaError_t e_ = cudaGetLastError();                            \
        if (e_ != cudaSuccess) return set_cuda_error(e_, what);         \
    } while (0)

constexpr int AF_T = 256;        // threads per CTA = columns of a tile
constexpr int AF_RS = 16;        // rows staged in shared memory at a time
constexpr int AF_RCH = 256;      // rows of a tile (row chunk)

enum { AF_SCALE_PARAMETER = 1, AF_RELATIVE_STEP = 2, AF_WARMUP_INIT = 4, AF_BETA1 = 8 };

__device__ __forceinline__ float af_grad_scale(float gscale, const float* __restrict__ sumsq, float max_norm) {
    float clip = 1.f;
    if (sumsq && max_norm > 0.f) {                     // clip_grad_norm_ exactly as adamw_flat_dev_kernel applies it
        const float norm = sqrtf(*sumsq) * gscale;
        clip = fminf(1.f, max_norm / (norm + 1e-6f));
    }
    return gscale * clip;
}

__device__ __forceinline__ float af_beta2t(const float* hy, const int* steps, int group) {
    return 1.f - powf((float)steps[group], hy[4]);
}

template <typename TV>
__device__ __forceinline__ TV af_block_sum(TV v, TV* s_red) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if ((threadIdx.x & 31) == 0) s_red[threadIdx.x >> 5] = v;
    __syncthreads();
    TV t = 0;
    if (threadIdx.x == 0)
        for (int w = 0; w < AF_T / 32; ++w) t += s_red[w];
    __syncthreads();
    return t;                                          // valid in thread 0
}

// Element walk of one item shared by passes (c) and (d): f(element index within the tensor, slab, row, column).
template <typename F>
__device__ __forceinline__ void af_for_each(const hcp_adafactor_item& it, const hcp_adafactor_tensor& T, F&& f) {
    const int cw = it.c1 - it.c0, k = AF_T / cw;
    const int pi = threadIdx.x / cw, c = it.c0 + threadIdx.x % cw;
    for (int pb = it.p0; pb < it.p1; pb += k) {
        if (pi >= min(k, it.p1 - pb)) continue;
        const int64_t p = pb + pi;
        for (int r = it.r0; r < it.r1; ++r) {
            const int64_t e = (p * T.R + r) * T.C + c;
            if (T.factored || e < T.numel) f(e, p, (int64_t)r, (int64_t)c);
        }
    }
}

__device__ __forceinline__ float af_precond(const hcp_adafactor_tensor& T, const float* __restrict__ state, const float* __restrict__ work,
                                            int64_t e, int64_t p, int64_t r, int64_t c) {
    if (!T.factored) return rsqrtf(state[T.row + e]);
    const float rf = rsqrtf(state[T.row + p * T.R + r] / work[T.rmean + p]);
    return rf * rsqrtf(state[T.col + p * T.C + c]);
}

// (a) ---------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(AF_T) adafactor_stats_kernel(const float* __restrict__ p, const float* __restrict__ g, float* __restrict__ state,
                                                               float* __restrict__ work, const hcp_adafactor_tensor* __restrict__ tensors,
                                                               const hcp_adafactor_item* __restrict__ items, const float* __restrict__ hyper,
                                                               const int* __restrict__ steps, float gscale, const float* __restrict__ sumsq,
                                                               float max_norm) {
    pdl_trigger();
    pdl_wait();
    __shared__ float s_q[AF_RS][AF_T];
    __shared__ float s_red[AF_T / 32];
    const hcp_adafactor_item it = items[blockIdx.x];
    const hcp_adafactor_tensor T = tensors[it.tensor];
    const float* hy = hyper + 8 * T.group;
    const float eps1 = hy[1], b2 = af_beta2t(hy, steps, T.group), gs = af_grad_scale(gscale, sumsq, max_norm);
    const float* pt = p + T.offset;
    const float* gt = g + T.offset;
    float* row = state + T.row;
    const int tid = threadIdx.x, cw = it.c1 - it.c0, k = AF_T / cw;
    const int pi = tid / cw, c = it.c0 + tid % cw;
    int L = 1;                                         // lanes per row segment (a power of two, at most a warp)
    while (L < cw && L < 32) L <<= 1;
    const int ngroups = AF_T / L, gid = tid / L, lane = tid % L;
    float p2 = 0.f;
    for (int pb = it.p0; pb < it.p1; pb += k) {
        const int kk = min(k, it.p1 - pb);
        const bool act = pi < kk;
        const int64_t ps = pb + pi;
        float cacc = 0.f;
        for (int rb = it.r0; rb < it.r1; rb += AF_RS) {
            const int nr = min(AF_RS, it.r1 - rb);
            for (int j = 0; j < nr; ++j) {
                float q = 0.f;
                if (act) {
                    const int64_t e = (ps * T.R + rb + j) * T.C + c;
                    if (T.factored || e < T.numel) {
                        const float w = pt[e], gv = gt[e] * gs;
                        p2 += w * w;
                        q = gv * gv + eps1;
                        if (!T.factored) row[e] = b2 * row[e] + (1.f - b2) * q;
                    }
                }
                s_q[j][tid] = q;
                cacc += q;
            }
            if (!T.factored) continue;                 // uniform across the CTA
            __syncthreads();
            const int nseg = nr * kk;                  // (slab, row) segments of cw staged values each
            for (int base = 0; base < nseg; base += ngroups) {
                const int seg = base + gid;
                float s = 0.f;
                if (seg < nseg) {
                    const int si = seg / nr, j = seg % nr;
                    for (int x = lane; x < cw; x += L) s += s_q[j][si * cw + x];
                }
                for (int o = L >> 1; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
                if (lane == 0 && seg < nseg) {
                    const int si = seg / nr, j = seg % nr;
                    const int64_t ri = (int64_t)(pb + si) * T.R + rb + j;
                    if (T.nct == 1) row[ri] = b2 * row[ri] + (1.f - b2) * (s / (float)T.C);
                    else work[T.rowpart + ri * T.nct + it.c0 / AF_T] = s;
                }
            }
            __syncthreads();
        }
        if (T.factored && act) {
            const int64_t ci = ps * T.C + c;
            if (T.nrch == 1) state[T.col + ci] = b2 * state[T.col + ci] + (1.f - b2) * (cacc / (float)T.R);
            else work[T.colpart + (int64_t)(it.r0 / AF_RCH) * T.P * T.C + ci] = cacc;
        }
    }
    p2 = af_block_sum(p2, s_red);
    if (tid == 0) work[blockIdx.x] = p2;
}

// (b) ---------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(AF_T) adafactor_factor_kernel(float* __restrict__ state, float* __restrict__ work,
                                                                const hcp_adafactor_tensor* __restrict__ tensors,
                                                                const hcp_adafactor_item* __restrict__ items, const float* __restrict__ hyper,
                                                                const int* __restrict__ steps) {
    pdl_trigger();
    pdl_wait();
    __shared__ float s_red[AF_T / 32];
    const hcp_adafactor_item it = items[blockIdx.x];
    const hcp_adafactor_tensor T = tensors[it.tensor];
    const float b2 = af_beta2t(hyper + 8 * T.group, steps, T.group);
    auto row_of = [&](int64_t ps, int64_t r) -> float {
        const int64_t ri = ps * T.R + r;
        float v = state[T.row + ri];
        if (T.nct > 1) {
            float s = 0.f;
            for (int ct = 0; ct < T.nct; ++ct) s += work[T.rowpart + ri * T.nct + ct];
            v = b2 * v + (1.f - b2) * (s / (float)T.C);
            state[T.row + ri] = v;
        }
        return v;
    };
    auto col_update = [&](int64_t ps, int64_t c) {
        if (T.nrch == 1) return;
        const int64_t ci = ps * T.C + c;
        float s = 0.f;
        for (int rc = 0; rc < T.nrch; ++rc) s += work[T.colpart + (int64_t)rc * T.P * T.C + ci];
        state[T.col + ci] = b2 * state[T.col + ci] + (1.f - b2) * (s / (float)T.R);
    };
    if (it.mode == 0) {                                // one CTA per slab
        const int64_t ps = it.p0;
        float acc = 0.f;
        for (int64_t r = threadIdx.x; r < T.R; r += AF_T) acc += row_of(ps, r);
        for (int64_t c = threadIdx.x; c < T.C; c += AF_T) col_update(ps, c);
        acc = af_block_sum(acc, s_red);
        if (threadIdx.x == 0) work[T.rmean + ps] = acc / (float)T.R;
    } else {                                           // one thread per slab
        for (int64_t ps = it.p0 + threadIdx.x; ps < it.p1; ps += AF_T) {
            float acc = 0.f;
            for (int64_t r = 0; r < T.R; ++r) acc += row_of(ps, r);
            for (int64_t c = 0; c < T.C; ++c) col_update(ps, c);
            work[T.rmean + ps] = acc / (float)T.R;
        }
    }
}

// (c) ---------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(AF_T) adafactor_rms_kernel(const float* __restrict__ g, const float* __restrict__ state, float* __restrict__ work,
                                                             const hcp_adafactor_tensor* __restrict__ tensors,
                                                             const hcp_adafactor_item* __restrict__ items, int nitems, float gscale,
                                                             const float* __restrict__ sumsq, float max_norm) {
    pdl_trigger();
    pdl_wait();
    __shared__ float s_red[AF_T / 32];
    const hcp_adafactor_item it = items[blockIdx.x];
    const hcp_adafactor_tensor T = tensors[it.tensor];
    const float gs = af_grad_scale(gscale, sumsq, max_norm);
    const float* gt = g + T.offset;
    float u2 = 0.f;
    af_for_each(it, T, [&](int64_t e, int64_t ps, int64_t r, int64_t c) {
        const float u = af_precond(T, state, work, e, ps, r, c) * (gt[e] * gs);
        u2 += u * u;
    });
    u2 = af_block_sum(u2, s_red);
    if (threadIdx.x == 0) work[nitems + blockIdx.x] = u2;
}

// (d) ---------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(AF_T) adafactor_apply_kernel(float* __restrict__ p, const float* __restrict__ g, const float* __restrict__ state,
                                                               float* __restrict__ exp_avg, const float* __restrict__ work,
                                                               const hcp_adafactor_tensor* __restrict__ tensors,
                                                               const hcp_adafactor_item* __restrict__ items, int nitems,
                                                               const float* __restrict__ hyper, const int* __restrict__ steps, float gscale,
                                                               const float* __restrict__ sumsq, float max_norm) {
    pdl_trigger();
    pdl_wait();
    __shared__ double s_red[AF_T / 32];
    __shared__ float s_scale[2];
    const hcp_adafactor_item it = items[blockIdx.x];
    const hcp_adafactor_tensor T = tensors[it.tensor];
    const float* hy = hyper + 8 * T.group;
    const int flags = (int)hy[7];
    double sp = 0.0, su = 0.0;                         // per-tensor totals of the tiles' partial sums, in item order
    for (int i = threadIdx.x; i < T.nitems; i += AF_T) {
        sp += (double)work[T.item0 + i];
        su += (double)work[nitems + T.item0 + i];
    }
    sp = af_block_sum(sp, s_red);
    su = af_block_sum(su, s_red);
    if (threadIdx.x == 0) {
        const float step = (float)steps[T.group];
        const float rms_p = (float)sqrt(sp / (double)T.numel), rms_u = (float)sqrt(su / (double)T.numel);
        float lr = hy[0];
        if (flags & AF_RELATIVE_STEP) lr = fminf((flags & AF_WARMUP_INIT) ? 1e-6f * step : 1e-2f, 1.f / sqrtf(step));
        if (flags & AF_SCALE_PARAMETER) lr *= fmaxf(hy[2], rms_p);
        s_scale[0] = lr;
        s_scale[1] = fmaxf(1.f, rms_u / hy[3]);
    }
    __syncthreads();
    const float lr = s_scale[0], denom = s_scale[1], wd = hy[6], beta1 = hy[5];
    const bool use_m = (flags & AF_BETA1) != 0;
    const float gs = af_grad_scale(gscale, sumsq, max_norm);
    float* pt = p + T.offset;
    const float* gt = g + T.offset;
    float* mt = use_m ? exp_avg + T.offset : nullptr;
    af_for_each(it, T, [&](int64_t e, int64_t ps, int64_t r, int64_t c) {
        float u = af_precond(T, state, work, e, ps, r, c) * (gt[e] * gs);
        u = u / denom * lr;
        if (use_m) {
            u = beta1 * mt[e] + (1.f - beta1) * u;
            mt[e] = u;
        }
        float w = pt[e];
        if (wd != 0.f) w = w + w * (-wd * lr);
        pt[e] = w - u;
    });
}

__global__ void adafactor_incr_kernel(int* steps, int ngroups) {
    pdl_trigger();
    pdl_wait();
    if ((int)threadIdx.x < ngroups) steps[threadIdx.x] += 1;
}

// Lion (lion_pytorch.Lion.step; Chen et al. 2023, Program 1) over one segment of the flat buffer, hyper = {lr, beta1, beta2, eps
// (unused), weight_decay} as adamw_flat_dev_kernel reads it.  Per element, in this order and in fp32:
//   p = p (1 - lr wd);  c = b1 m + (1 - b1) g;  p = p - lr sign(c)  (sign(0) = 0);  m = b2 m + (1 - b2) g
// One moment, no bias correction: the step counter is only advanced (by block 0), for hcp_ema_flat.  Four elements per thread
// and iteration (16-byte accesses: 20 B of traffic per element), the n % 4 tail in block 0.
__global__ void __launch_bounds__(256) lion_flat_dev_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m,
                                                            int64_t n, const float* __restrict__ hyper, float gscale,
                                                            const float* __restrict__ sumsq, float max_norm, int* __restrict__ step_ptr) {
    pdl_trigger();
    pdl_wait();
    if (blockIdx.x == 0 && threadIdx.x == 0) *step_ptr += 1;
    const float gs = af_grad_scale(gscale, sumsq, max_norm);
    const float lr = hyper[0], beta1 = hyper[1], beta2 = hyper[2], wd = hyper[4];
    const float decay = __fsub_rn(1.f, __fmul_rn(lr, wd));      // 1 - lr * wd rounded twice, as lion-pytorch's fp32 tensors see it
    auto upd = [&](float& w, float grad, float& mi) {
        grad *= gs;
        w *= decay;
        const float c = beta1 * mi + (1.f - beta1) * grad;
        w -= lr * (float)((c > 0.f) - (c < 0.f));
        mi = beta2 * mi + (1.f - beta2) * grad;
    };
    const int64_t n4 = n >> 2, stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n4; i += stride) {
        float4 w4 = reinterpret_cast<float4*>(p)[i], m4 = reinterpret_cast<float4*>(m)[i];
        const float4 g4 = reinterpret_cast<const float4*>(g)[i];
        upd(w4.x, g4.x, m4.x); upd(w4.y, g4.y, m4.y); upd(w4.z, g4.z, m4.z); upd(w4.w, g4.w, m4.w);
        reinterpret_cast<float4*>(p)[i] = w4; reinterpret_cast<float4*>(m)[i] = m4;
    }
    if (blockIdx.x == 0 && threadIdx.x < (n & 3)) {
        const int64_t i = (n4 << 2) + threadIdx.x;
        float w = p[i], mi = m[i];
        upd(w, g[i], mi);
        p[i] = w; m[i] = mi;
    }
}

}  // namespace hcp

using namespace hcp;

extern "C" int hcp_adafactor_flat(float* p, const float* g, float* state, float* exp_avg, float* work, const hcp_adafactor_tensor* tensors_device,
                                  const hcp_adafactor_item* items_device, int64_t nitems, const hcp_adafactor_item* factor_items_device,
                                  int64_t nfactor_items, const float* hyper_device, int* steps_device, int32_t ngroups, float grad_scale,
                                  const float* sumsq_device, float max_norm, hcp_stream_t st) {
    if (!p || !g || !state || !work || !tensors_device || !items_device || !hyper_device || !steps_device)
        return set_error(HCP_ERR_INVALID, "adafactor: null pointer");
    if (nitems <= 0 || nitems > (1ll << 30) || nfactor_items < 0 || nfactor_items > (1ll << 30) || (nfactor_items && !factor_items_device) ||
        ngroups <= 0 || ngroups > AF_T)
        return set_error(HCP_ERR_INVALID, "adafactor: item or group count");
    const cudaStream_t s = (cudaStream_t)st;
    launch_k(adafactor_incr_kernel, dim3(1), dim3(AF_T), 0, s, steps_device, (int)ngroups);
    launch_k(adafactor_stats_kernel, dim3((unsigned)nitems), dim3(AF_T), 0, s, p, g, state, work, tensors_device, items_device, hyper_device,
             (const int*)steps_device, grad_scale, sumsq_device, max_norm);
    if (nfactor_items)
        launch_k(adafactor_factor_kernel, dim3((unsigned)nfactor_items), dim3(AF_T), 0, s, state, work, tensors_device, factor_items_device,
                 hyper_device, (const int*)steps_device);
    launch_k(adafactor_rms_kernel, dim3((unsigned)nitems), dim3(AF_T), 0, s, g, (const float*)state, work, tensors_device, items_device,
             (int)nitems, grad_scale, sumsq_device, max_norm);
    launch_k(adafactor_apply_kernel, dim3((unsigned)nitems), dim3(AF_T), 0, s, p, g, (const float*)state, exp_avg, (const float*)work,
             tensors_device, items_device, (int)nitems, hyper_device, (const int*)steps_device, grad_scale, sumsq_device, max_norm);
    LAUNCH_CHECK("adafactor launch");
    return HCP_OK;
}

extern "C" int hcp_lion_flat_dev(float* p, const float* g, float* m, int64_t n, const float* hyper_device, float grad_scale,
                                 const float* sumsq_device, float max_norm, int* step_device, hcp_stream_t st) {
    if (!p || !g || !m || !hyper_device || !step_device) return set_error(HCP_ERR_INVALID, "lion_dev: null pointer");
    if (n < 0) return set_error(HCP_ERR_INVALID, "lion_dev: negative size");
    if (((uintptr_t)p | (uintptr_t)g | (uintptr_t)m) & 15) return set_error(HCP_ERR_INVALID, "lion_dev: buffers must be 16-byte aligned");
    if (n == 0) return HCP_OK;
    int64_t blocks = ((n >> 2) + 255) / 256;
    if (blocks > num_sms() * 16) blocks = num_sms() * 16;
    if (blocks < 1) blocks = 1;
    launch_k(lion_flat_dev_kernel, dim3((unsigned)blocks), dim3(256), 0, (cudaStream_t)st, p, g, m, n, hyper_device, grad_scale,
             sumsq_device, max_norm, step_device);
    LAUNCH_CHECK("lion_dev launch");
    return HCP_OK;
}
