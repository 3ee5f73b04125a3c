// SPDX-License-Identifier: Apache-2.0
// Adafactor (transformers.optimization.Adafactor.step) over the flat fp32 parameter buffer of the training step (sm_90a), and
// Lion (lion_pytorch.Lion.step, one elementwise kernel), Prodigy (prodigyopt.Prodigy, a device-side step size d from a global
// reduction) and AdamW8bit (bitsandbytes.optim.AdamW8bit, blockwise 8-bit moments), near the end of this file.
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

// AdamW8bit (bitsandbytes.optim.AdamW8bit: Optimizer2State, optim_bits 8, block_wise; kOptimizerStatic8bit2StateBlockwise and
// kOptimizer32bit2State) over the tensors of a host-built table, hyper = fp32 [ngroups, 5] rows {lr, beta1, beta2, eps,
// weight_decay} as adamw_flat_dev_kernel reads them, steps int32 [ngroups] already advanced by adafactor_incr_kernel.
//
// A work item is a run of whole 256-element blocks of one tensor; CTAs walk the items grid-stride, four blocks at a time, one
// quarter (64 threads, two warps) per block and four consecutive elements per thread.  Per element, in fp32 with every product
// and sum rounded on its own (no contraction, so the moments, scales and codes are reproducible from fp32 on any machine):
//   g' = g * gscale_clip;   s1 = map1[c1] * absmax1;  s2 = map2[c2] * absmax2                       (8-bit; 32-bit: s1 = m, s2 = v)
//   s1 = s1 b1 + (1 - b1) g';  s2 = s2 b2 + ((1 - b2) g') g'
//   p = p + (-lr sqrt(1 - b2^t) / (1 - b1^t)) s1 / (sqrt(s2) + eps sqrt(1 - b2^t));  if wd > 0: p = p (1 - lr wd)
// 8-bit only: a non-finite g sets s1 = s2 = 0 and leaves p; the block's new scale is max |s| over its elements (a warp max, then
// the two warps of the quarter -- an exact, order-free reduction inside the CTA), and each s / scale (0 for an all-zero block) is
// re-encoded with bitsandbytes' binary search and midpoint rule (an exact midpoint goes to the last probed entry); a first-moment
// code whose value has the other sign bit than s1 moves one step toward s1's sign.  The maps live in shared memory at index
// k + k / 32, which spreads the search's probes (entries 32 apart) over different banks.
constexpr int A8_T = 256;
constexpr int A8_BLOCK = 256;

__host__ __device__ constexpr int a8_idx(int k) { return k + (k >> 5); }

__device__ __forceinline__ float a8_grad_scale(float gscale, const float* __restrict__ sumsq, float max_norm) {
    float clip = 1.f;
    if (sumsq && max_norm > 0.f) {                     // clip_grad_norm_ as af_grad_scale, each operation rounded on its own
        const float norm = __fmul_rn(sqrtf(*sumsq), gscale);
        clip = fminf(1.f, __fdiv_rn(max_norm, __fadd_rn(norm, 1e-6f)));
    }
    return __fmul_rn(gscale, clip);
}

template <bool SIGNED>
__device__ __forceinline__ int a8_quantize(const float* __restrict__ s_map, float x) {
    int pivot = 127, upper_pivot = 255, lower_pivot = 0;
    float lower = SIGNED ? -1.f : 0.f, upper = 1.f;
    float val = s_map[a8_idx(pivot)];
#pragma unroll
    for (int i = 64; i > 0; i >>= 1) {
        if (x > val) { lower_pivot = pivot; lower = val; pivot += i; }
        else { upper_pivot = pivot; upper = val; pivot -= i; }
        val = s_map[a8_idx(pivot)];
    }
    if (x > val) return x > __fmul_rn(__fadd_rn(upper, val), 0.5f) ? upper_pivot : pivot;
    return x < __fmul_rn(__fadd_rn(lower, val), 0.5f) ? lower_pivot : pivot;
}

__global__ void __launch_bounds__(A8_T, 4) adamw8bit_kernel(float* __restrict__ p, const float* __restrict__ g, uint8_t* __restrict__ code1,
                                                         uint8_t* __restrict__ code2, float* __restrict__ absmax1, float* __restrict__ absmax2,
                                                         float* __restrict__ m32, float* __restrict__ v32, const float* __restrict__ maps,
                                                         const hcp_adamw8bit_tensor* __restrict__ tensors,
                                                         const hcp_adamw8bit_item* __restrict__ items, int nitems,
                                                         const float* __restrict__ hyper, const int* __restrict__ steps, float gscale,
                                                         const float* __restrict__ sumsq, float max_norm) {
    pdl_trigger();
    pdl_wait();
    __shared__ float s_map1[a8_idx(256)], s_map2[a8_idx(256)];
    __shared__ float s_max[2][A8_T / 32][2];           // [parity][warp][moment]
    for (int k = threadIdx.x; k < 256; k += A8_T) {
        s_map1[a8_idx(k)] = maps[k];
        s_map2[a8_idx(k)] = maps[256 + k];
    }
    __syncthreads();
    const float gs = a8_grad_scale(gscale, sumsq, max_norm);
    const int q = threadIdx.x >> 6, lane64 = threadIdx.x & 63, warp = threadIdx.x >> 5;
    int parity = 0;
    for (int ii = blockIdx.x; ii < nitems; ii += gridDim.x) {
        const hcp_adamw8bit_item it = items[ii];
        const hcp_adamw8bit_tensor T = tensors[it.tensor];
        const float* hy = hyper + 5 * T.group;
        const float lr = hy[0], b1 = hy[1], b2 = hy[2], eps = hy[3], wd = hy[4];
        const float t = (float)steps[T.group];
        const float corr1 = 1.f - powf(b1, t), corr2 = sqrtf(1.f - powf(b2, t));
        const float step_size = __fdiv_rn(__fmul_rn(-lr, corr2), corr1);
        const float eps_c = __fmul_rn(eps, corr2);
        const float omb1 = 1.f - b1, omb2 = 1.f - b2, decay = __fsub_rn(1.f, __fmul_rn(lr, wd));
        const bool q8 = T.mode == 1;
        float* pt = p + T.offset;
        const float* gt = g + T.offset;
        for (int b0 = it.block0; b0 < it.block1; b0 += 4) {
            const int64_t b = b0 + q;
            const bool active = b < it.block1;
            const int64_t e0 = b * A8_BLOCK + lane64 * 4;
            const int nv = active ? (int)max((int64_t)0, min((int64_t)4, T.numel - e0)) : 0;
            float w[4] = {0.f, 0.f, 0.f, 0.f}, gr[4] = {0.f, 0.f, 0.f, 0.f}, s1[4] = {0.f, 0.f, 0.f, 0.f}, s2[4] = {0.f, 0.f, 0.f, 0.f};
            uint8_t c1[4] = {0, 0, 0, 0}, c2[4] = {0, 0, 0, 0};
            if (nv == 4) {
                const float4 w4 = *reinterpret_cast<const float4*>(pt + e0), g4 = *reinterpret_cast<const float4*>(gt + e0);
                w[0] = w4.x; w[1] = w4.y; w[2] = w4.z; w[3] = w4.w;
                gr[0] = g4.x; gr[1] = g4.y; gr[2] = g4.z; gr[3] = g4.w;
                if (q8) {
                    const uchar4 a = *reinterpret_cast<const uchar4*>(code1 + T.state + e0), c = *reinterpret_cast<const uchar4*>(code2 + T.state + e0);
                    c1[0] = a.x; c1[1] = a.y; c1[2] = a.z; c1[3] = a.w;
                    c2[0] = c.x; c2[1] = c.y; c2[2] = c.z; c2[3] = c.w;
                } else {
                    const float4 m4 = *reinterpret_cast<const float4*>(m32 + T.state + e0), v4 = *reinterpret_cast<const float4*>(v32 + T.state + e0);
                    s1[0] = m4.x; s1[1] = m4.y; s1[2] = m4.z; s1[3] = m4.w;
                    s2[0] = v4.x; s2[1] = v4.y; s2[2] = v4.z; s2[3] = v4.w;
                }
            } else {
                for (int j = 0; j < nv; ++j) {
                    w[j] = pt[e0 + j];
                    gr[j] = gt[e0 + j];
                    if (q8) { c1[j] = code1[T.state + e0 + j]; c2[j] = code2[T.state + e0 + j]; }
                    else { s1[j] = m32[T.state + e0 + j]; s2[j] = v32[T.state + e0 + j]; }
                }
            }
            float am1 = 0.f, am2 = 0.f;
            if (q8 && active) { am1 = absmax1[T.absmax + b]; am2 = absmax2[T.absmax + b]; }
            float mx1 = 0.f, mx2 = 0.f;
            bool fin[4];
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                fin[j] = !q8 || isfinite(gr[j]);
                if (j >= nv) continue;
                if (fin[j]) {
                    const float gv = __fmul_rn(gr[j], gs);
                    float a = s1[j], c = s2[j];
                    if (q8) { a = __fmul_rn(s_map1[a8_idx(c1[j])], am1); c = __fmul_rn(s_map2[a8_idx(c2[j])], am2); }
                    s2[j] = __fadd_rn(__fmul_rn(c, b2), __fmul_rn(__fmul_rn(omb2, gv), gv));
                    s1[j] = __fadd_rn(__fmul_rn(a, b1), __fmul_rn(omb1, gv));
                    float wj = __fadd_rn(w[j], __fmul_rn(step_size, __fdiv_rn(s1[j], __fadd_rn(sqrtf(s2[j]), eps_c))));
                    if (wd > 0.f) wj = __fmul_rn(wj, decay);
                    w[j] = wj;
                } else {
                    s1[j] = 0.f;
                    s2[j] = 0.f;
                }
                mx1 = fmaxf(mx1, fabsf(s1[j]));
                mx2 = fmaxf(mx2, fabsf(s2[j]));
            }
            if (q8) {                                      // uniform across the CTA: every item of one CTA step is one tensor's
#pragma unroll
                for (int o = 16; o > 0; o >>= 1) {
                    mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, o));
                    mx2 = fmaxf(mx2, __shfl_xor_sync(0xffffffffu, mx2, o));
                }
                if ((threadIdx.x & 31) == 0) { s_max[parity][warp][0] = mx1; s_max[parity][warp][1] = mx2; }
                __syncthreads();
                mx1 = fmaxf(s_max[parity][2 * q][0], s_max[parity][2 * q + 1][0]);
                mx2 = fmaxf(s_max[parity][2 * q][1], s_max[parity][2 * q + 1][1]);
                parity ^= 1;                               // the next write goes to the other half: one barrier per step
                if (active && lane64 == 0) { absmax1[T.absmax + b] = mx1; absmax2[T.absmax + b] = mx2; }
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    const float x1 = mx1 > 0.f ? __fdiv_rn(s1[j], mx1) : 0.f, x2 = mx2 > 0.f ? __fdiv_rn(s2[j], mx2) : 0.f;
                    int k1 = a8_quantize<true>(s_map1, x1);
                    if (signbit(s_map1[a8_idx(k1)]) != signbit(s1[j])) k1 = (k1 + (s1[j] > 0.f ? 1 : -1)) & 255;
                    c1[j] = (uint8_t)k1;
                    c2[j] = (uint8_t)a8_quantize<false>(s_map2, x2);
                }
            }
            if (nv == 4) {
                *reinterpret_cast<float4*>(pt + e0) = make_float4(w[0], w[1], w[2], w[3]);
                if (q8) {
                    *reinterpret_cast<uchar4*>(code1 + T.state + e0) = make_uchar4(c1[0], c1[1], c1[2], c1[3]);
                    *reinterpret_cast<uchar4*>(code2 + T.state + e0) = make_uchar4(c2[0], c2[1], c2[2], c2[3]);
                } else {
                    *reinterpret_cast<float4*>(m32 + T.state + e0) = make_float4(s1[0], s1[1], s1[2], s1[3]);
                    *reinterpret_cast<float4*>(v32 + T.state + e0) = make_float4(s2[0], s2[1], s2[2], s2[3]);
                }
            } else {
                for (int j = 0; j < nv; ++j) {
                    pt[e0 + j] = w[j];
                    if (q8) { code1[T.state + e0 + j] = c1[j]; code2[T.state + e0 + j] = c2[j]; }
                    else { m32[T.state + e0 + j] = s1[j]; v32[T.state + e0 + j] = s2[j]; }
                }
            }
        }
    }
}

// Prodigy (prodigyopt.Prodigy.step; Mishchenko & Defazio 2023) over segments of the flat buffer, in three launches:
//   (1) prodigy_stats_kernel: per element of every segment, g' = g * gscale_clip (+ wd p when decay is coupled); on the first call
//       p0 = p and s = m = v = 0; in a segment with lr > 0:  m = b1 m + d (1 - b1) g';  v = b2 v + d^2 (1 - b2) g'^2;
//       s = b3 s + (d / d0) (safeguard_warmup ? d : dlr) g'.  Per-CTA fp64 partials of sum g' (p0 - p) and sum |s| go to the
//       workspace (per thread in element order, then a fixed shuffle tree).
//   (2) prodigy_scalars_kernel: one CTA sums the partials in a fixed order and updates d, d_max, D_num, k (or marks the call
//       skipped when sum |s| == 0), and advances the EMA step counter.
//   (3) prodigy_apply_kernel: unless skipped, p = p - wd dlr p (decoupled decay) and p = p - dlr m / (sqrt(v) + d eps) with the
//       old dlr and the new d, read from the scalar block.
// d, dlr and the other scalars are fp64 (the reference keeps them as Python floats); the coefficients an element sees are rounded
// to fp32 once, as torch's fp32 ops round a Python scalar.  16-byte accesses, the count % 4 tail of a segment by one CTA.
constexpr int PD_T = 256;
enum { PD_BIAS_CORRECTION = 1, PD_SAFEGUARD_WARMUP = 2, PD_DECOUPLE = 4 };
enum { PD_D = 0, PD_DMAX = 1, PD_DNUM = 2, PD_K = 3, PD_INIT = 4, PD_SKIP = 5, PD_DLR = 6 };

// the largest segment lr, over the whole CTA (every thread gets it)
__device__ __forceinline__ double pd_max_lr(const hcp_prodigy_segment* __restrict__ segs, int nsegs, double* s_red) {
    double mx = 0.0;
    for (int i = threadIdx.x; i < nsegs; i += PD_T) mx = fmax(mx, segs[i].lr);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) mx = fmax(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    if ((threadIdx.x & 31) == 0) s_red[threadIdx.x >> 5] = mx;
    __syncthreads();
    mx = s_red[0];
    for (int w = 1; w < PD_T / 32; ++w) mx = fmax(mx, s_red[w]);
    __syncthreads();
    return mx;
}

// dlr = d lr bc of the step about to run (old d, k), identical in launches (1) and (2)
__device__ __forceinline__ double pd_dlr(const double* __restrict__ hy, const double* __restrict__ st, double lr) {
    double bc = 1.0;
    if ((int)hy[7] & PD_BIAS_CORRECTION) {
        const double k1 = st[PD_K] + 1.0;
        bc = sqrt(1.0 - pow(hy[1], k1)) / (1.0 - pow(hy[0], k1));
    }
    return st[PD_D] * lr * bc;
}

template <typename TV>
__device__ __forceinline__ TV pd_block_sum(TV v, TV* s_red) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if ((threadIdx.x & 31) == 0) s_red[threadIdx.x >> 5] = v;
    __syncthreads();
    TV t = 0;
    if (threadIdx.x == 0)
        for (int w = 0; w < PD_T / 32; ++w) t += s_red[w];
    __syncthreads();
    return t;                                          // valid in thread 0
}

__global__ void __launch_bounds__(PD_T) prodigy_stats_kernel(const float* __restrict__ p, const float* __restrict__ g, float* __restrict__ p0,
                                                             float* __restrict__ s, float* __restrict__ m, float* __restrict__ v,
                                                             const hcp_prodigy_segment* __restrict__ segs, int nsegs,
                                                             const double* __restrict__ hy, const double* __restrict__ st,
                                                             double* __restrict__ work, float gscale, const float* __restrict__ sumsq,
                                                             float max_norm) {
    pdl_trigger();
    pdl_wait();
    __shared__ double s_red[PD_T / 32];
    const double lr = pd_max_lr(segs, nsegs, s_red);
    const double d = st[PD_D], dlr = pd_dlr(hy, st, lr), d0 = hy[4];
    const int flags = (int)hy[7];
    const bool first = st[PD_INIT] == 0.0, coupled = !(flags & PD_DECOUPLE);
    const float b1 = (float)hy[0], b2 = (float)hy[1], b3 = (float)hy[2];
    const float cm = (float)(d * (1.0 - hy[0])), cv = (float)(d * d * (1.0 - hy[1]));
    const float cs = (float)((d / d0) * ((flags & PD_SAFEGUARD_WARMUP) ? d : dlr));
    const float gs = af_grad_scale(gscale, sumsq, max_norm);
    double dot = 0.0, den = 0.0;
    for (int si = 0; si < nsegs; ++si) {
        const hcp_prodigy_segment sg = segs[si];
        const bool live = sg.lr > 0.0;
        if (!live && !first) continue;                 // an lr-0 segment only decays, in (3)
        const float wd = coupled ? (float)sg.weight_decay : 0.f;
        auto upd = [&](float w, float gr, float& q0, float& si_, float& mi, float& vi) {
            gr *= gs;
            if (wd != 0.f) gr += wd * w;
            if (first) { q0 = w; si_ = 0.f; mi = 0.f; vi = 0.f; }
            if (live) {
                dot += (double)gr * ((double)q0 - (double)w);
                mi = b1 * mi + cm * gr;
                vi = b2 * vi + cv * gr * gr;
                si_ = b3 * si_ + cs * gr;
                den += fabs((double)si_);
            }
        };
        const float* ps = p + sg.offset;
        const float* gg = g + sg.offset;
        float *q = p0 + sg.offset, *ss = s + sg.offset, *ms = m + sg.offset, *vs = v + sg.offset;
        const int64_t n4 = sg.count >> 2, stride = (int64_t)gridDim.x * PD_T;
        for (int64_t i = blockIdx.x * (int64_t)PD_T + threadIdx.x; i < n4; i += stride) {
            const float4 w4 = reinterpret_cast<const float4*>(ps)[i], g4 = reinterpret_cast<const float4*>(gg)[i];
            float4 q4 = make_float4(0.f, 0.f, 0.f, 0.f), s4 = q4, m4 = q4, v4 = q4;
            if (!first) {
                q4 = reinterpret_cast<const float4*>(q)[i]; s4 = reinterpret_cast<const float4*>(ss)[i];
                m4 = reinterpret_cast<const float4*>(ms)[i]; v4 = reinterpret_cast<const float4*>(vs)[i];
            }
            upd(w4.x, g4.x, q4.x, s4.x, m4.x, v4.x); upd(w4.y, g4.y, q4.y, s4.y, m4.y, v4.y);
            upd(w4.z, g4.z, q4.z, s4.z, m4.z, v4.z); upd(w4.w, g4.w, q4.w, s4.w, m4.w, v4.w);
            if (first) reinterpret_cast<float4*>(q)[i] = q4;
            reinterpret_cast<float4*>(ss)[i] = s4; reinterpret_cast<float4*>(ms)[i] = m4; reinterpret_cast<float4*>(vs)[i] = v4;
        }
        if ((int)blockIdx.x == si % (int)gridDim.x && threadIdx.x < (sg.count & 3)) {
            const int64_t i = (n4 << 2) + threadIdx.x;
            float q0 = first ? 0.f : q[i], si_ = first ? 0.f : ss[i], mi = first ? 0.f : ms[i], vi = first ? 0.f : vs[i];
            upd(ps[i], gg[i], q0, si_, mi, vi);
            if (first) q[i] = q0;
            ss[i] = si_; ms[i] = mi; vs[i] = vi;
        }
    }
    dot = pd_block_sum(dot, s_red);
    den = pd_block_sum(den, s_red);
    if (threadIdx.x == 0) {
        work[2 * blockIdx.x] = dot;
        work[2 * blockIdx.x + 1] = den;
    }
}

__global__ void __launch_bounds__(PD_T) prodigy_scalars_kernel(const hcp_prodigy_segment* __restrict__ segs, int nsegs,
                                                               const double* __restrict__ hy, double* __restrict__ st,
                                                               const double* __restrict__ work, int nblocks, int* __restrict__ step_ptr) {
    pdl_trigger();
    pdl_wait();
    __shared__ double s_red[PD_T / 32];
    const double lr = pd_max_lr(segs, nsegs, s_red);
    double dot = 0.0, den = 0.0;
    for (int b = threadIdx.x; b < nblocks; b += PD_T) {
        dot += work[2 * b];
        den += work[2 * b + 1];
    }
    dot = pd_block_sum(dot, s_red);
    den = pd_block_sum(den, s_red);
    if (threadIdx.x != 0) return;
    *step_ptr += 1;                                    // ModelEMA counts every optimizer call, skipped or not
    double d = st[PD_D], d_max = st[PD_DMAX];
    const double d0 = hy[4], dlr = pd_dlr(hy, st, lr);
    const double d_num = hy[2] * st[PD_DNUM] + (d / d0) * dlr * dot;
    st[PD_INIT] = 1.0;
    if (den == 0.0) {                                  // no progress: p, d, d_max, D_num and k stay
        st[PD_SKIP] = 1.0;
        return;
    }
    if (lr > 0.0) {
        const double d_hat = hy[5] * d_num / den;
        if (d == d0) d = fmax(d, d_hat);
        d_max = fmax(d_max, d_hat);
        d = fmin(d_max, d * hy[6]);
    }
    st[PD_D] = d;
    st[PD_DMAX] = d_max;
    st[PD_DNUM] = d_num;
    st[PD_K] += 1.0;
    st[PD_SKIP] = 0.0;
    st[PD_DLR] = dlr;
}

__global__ void __launch_bounds__(PD_T) prodigy_apply_kernel(float* __restrict__ p, const float* __restrict__ m, const float* __restrict__ v,
                                                             const hcp_prodigy_segment* __restrict__ segs, int nsegs,
                                                             const double* __restrict__ hy, const double* __restrict__ st) {
    pdl_trigger();
    pdl_wait();
    if (st[PD_SKIP] != 0.0) return;
    const double dlr = st[PD_DLR];
    const float step = (float)(-dlr), deps = (float)(st[PD_D] * hy[3]);
    const bool decouple = (int)hy[7] & PD_DECOUPLE;
    for (int si = 0; si < nsegs; ++si) {
        const hcp_prodigy_segment sg = segs[si];
        const float decay = (decouple && sg.weight_decay != 0.0) ? (float)(-sg.weight_decay * dlr) : 0.f;
        auto upd = [&](float& w, float mi, float vi) {
            if (decay != 0.f) w = w + w * decay;
            w = w + step * (mi / (sqrtf(vi) + deps));
        };
        float* ps = p + sg.offset;
        const float *ms = m + sg.offset, *vs = v + sg.offset;
        const int64_t n4 = sg.count >> 2, stride = (int64_t)gridDim.x * PD_T;
        for (int64_t i = blockIdx.x * (int64_t)PD_T + threadIdx.x; i < n4; i += stride) {
            float4 w4 = reinterpret_cast<float4*>(ps)[i];
            const float4 m4 = reinterpret_cast<const float4*>(ms)[i], v4 = reinterpret_cast<const float4*>(vs)[i];
            upd(w4.x, m4.x, v4.x); upd(w4.y, m4.y, v4.y); upd(w4.z, m4.z, v4.z); upd(w4.w, m4.w, v4.w);
            reinterpret_cast<float4*>(ps)[i] = w4;
        }
        if ((int)blockIdx.x == si % (int)gridDim.x && threadIdx.x < (sg.count & 3)) {
            const int64_t i = (n4 << 2) + threadIdx.x;
            float w = ps[i];
            upd(w, ms[i], vs[i]);
            ps[i] = w;
        }
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

extern "C" int hcp_prodigy_flat(float* p, const float* g, float* p0, float* s, float* m, float* v, int64_t n,
                                const hcp_prodigy_segment* segs_host, const hcp_prodigy_segment* segs_device, int32_t nsegs,
                                const double* hyper_device, double* state_device, double* workspace, size_t workspace_bytes,
                                float grad_scale, const float* sumsq_device, float max_norm, int* step_device, hcp_stream_t st) {
    if (!p || !g || !p0 || !s || !m || !v || !segs_host || !segs_device || !hyper_device || !state_device || !workspace || !step_device)
        return set_error(HCP_ERR_INVALID, "prodigy: null pointer");
    if (n < 0 || nsegs < 0) return set_error(HCP_ERR_INVALID, "prodigy: negative size");
    if (!aligned16(p, g, p0, s, m, v) || ((uintptr_t)workspace & 7) || ((uintptr_t)hyper_device & 7) || ((uintptr_t)state_device & 7) ||
        ((uintptr_t)segs_device & 7))
        return set_error(HCP_ERR_INVALID, "prodigy: p / g / p0 / s / m / v must be 16-byte aligned, the tables 8-byte aligned");
    if (workspace_bytes < (size_t)HCP_PRODIGY_WORKSPACE_BYTES) return set_error(HCP_ERR_INVALID, "prodigy: workspace too small");
    int64_t end = 0, total = 0;
    for (int32_t i = 0; i < nsegs; ++i) {
        const hcp_prodigy_segment& sg = segs_host[i];
        if (sg.count < 0 || sg.offset < end || (sg.offset & 3) || sg.count > n - sg.offset)
            return set_error(HCP_ERR_INVALID, "prodigy: segment outside [0, n), overlapping, negative or off 16-byte alignment");
        end = sg.offset + sg.count;
        total += sg.count;
    }
    if (total == 0) return HCP_OK;
    const cudaStream_t cs = (cudaStream_t)st;
    int64_t blocks = ((total >> 2) + PD_T - 1) / PD_T;
    if (blocks > num_sms() * 4) blocks = num_sms() * 4;          // one resident wave: the partials are one per CTA
    if (blocks > HCP_PRODIGY_WORKSPACE_BYTES / 16) blocks = HCP_PRODIGY_WORKSPACE_BYTES / 16;
    if (blocks < 1) blocks = 1;
    int64_t ablocks = ((total >> 2) + PD_T - 1) / PD_T;          // the update has no partials: lion's grid
    if (ablocks > num_sms() * 16) ablocks = num_sms() * 16;
    if (ablocks < 1) ablocks = 1;
    launch_k(prodigy_stats_kernel, dim3((unsigned)blocks), dim3(PD_T), 0, cs, (const float*)p, g, p0, s, m, v, segs_device, (int)nsegs,
             hyper_device, (const double*)state_device, workspace, grad_scale, sumsq_device, max_norm);
    launch_k(prodigy_scalars_kernel, dim3(1), dim3(PD_T), 0, cs, segs_device, (int)nsegs, hyper_device, state_device,
             (const double*)workspace, (int)blocks, step_device);
    launch_k(prodigy_apply_kernel, dim3((unsigned)ablocks), dim3(PD_T), 0, cs, p, (const float*)m, (const float*)v, segs_device, (int)nsegs,
             hyper_device, (const double*)state_device);
    LAUNCH_CHECK("prodigy launch");
    return HCP_OK;
}

// Host-side check of the tables the kernel will read (their device copies are the caller's): every tensor inside p / g and its
// state inside the buffers, aligned for 16-byte (p, g, m, v) and 4-byte (codes) accesses, tensors and states in increasing,
// non-overlapping order, and the items tiling each tensor's blocks once, in table order.
static int adamw8bit_check_tables(const hcp_adamw8bit_tensor* T, int32_t ntensors, const hcp_adamw8bit_item* I, int64_t nitems, int64_t n,
                                  int64_t code_bytes, int64_t nblocks, int64_t small_numel, int32_t ngroups) {
    int64_t p_end = 0, code_end = 0, blk_end = 0, small_end = 0;
    for (int32_t i = 0; i < ntensors; ++i) {
        const hcp_adamw8bit_tensor& t = T[i];
        if (t.numel <= 0 || t.offset < p_end || (t.offset & 3) || t.numel > n - t.offset)
            return set_error(HCP_ERR_INVALID, "adamw8bit: tensor outside p / g, overlapping, or off 16-byte alignment");
        if (t.group < 0 || t.group >= ngroups) return set_error(HCP_ERR_INVALID, "adamw8bit: tensor group out of range");
        const int64_t nb = (t.numel + A8_BLOCK - 1) / A8_BLOCK;
        if (t.mode == 1) {
            if (t.state < code_end || (t.state & 3) || t.numel > code_bytes - t.state || t.absmax < blk_end || nb > nblocks - t.absmax)
                return set_error(HCP_ERR_INVALID, "adamw8bit: 8-bit state outside the code / absmax buffers, overlapping or misaligned");
            code_end = t.state + t.numel;
            blk_end = t.absmax + nb;
        } else if (t.mode == 0) {
            if (t.state < small_end || (t.state & 3) || t.numel > small_numel - t.state)
                return set_error(HCP_ERR_INVALID, "adamw8bit: 32-bit state outside state32, overlapping or misaligned");
            small_end = t.state + t.numel;
        } else {
            return set_error(HCP_ERR_INVALID, "adamw8bit: tensor mode must be 0 (32-bit) or 1 (8-bit)");
        }
        p_end = t.offset + t.numel;
    }
    int32_t cur = 0;
    int64_t next = 0;                                  // the next block of tensor `cur` an item must start at
    for (int64_t k = 0; k < nitems; ++k) {
        const hcp_adamw8bit_item& it = I[k];
        if (it.tensor == cur + 1 && cur + 1 < ntensors && next == (T[cur].numel + A8_BLOCK - 1) / A8_BLOCK) { cur += 1; next = 0; }
        if (it.tensor != cur || it.block0 != next || it.block1 <= it.block0 ||
            it.block1 > (T[cur].numel + A8_BLOCK - 1) / A8_BLOCK)
            return set_error(HCP_ERR_INVALID, "adamw8bit: items must tile every tensor's blocks once, in table order");
        next = it.block1;
    }
    if (cur != ntensors - 1 || next != (T[cur].numel + A8_BLOCK - 1) / A8_BLOCK)
        return set_error(HCP_ERR_INVALID, "adamw8bit: items leave blocks uncovered");
    return HCP_OK;
}

extern "C" int hcp_adamw8bit_flat(float* p, const float* g, uint8_t* codes, float* absmax, float* state32, const float* maps_device,
                                  const hcp_adamw8bit_tensor* tensors_host, const hcp_adamw8bit_tensor* tensors_device, int32_t ntensors,
                                  const hcp_adamw8bit_item* items_host, const hcp_adamw8bit_item* items_device, int64_t nitems, int64_t n,
                                  int64_t code_bytes, int64_t nblocks, int64_t small_numel, const float* hyper_device, int* steps_device,
                                  int32_t ngroups, float grad_scale, const float* sumsq_device, float max_norm, hcp_stream_t st) {
    if (ntensors < 0 || nitems < 0 || n < 0 || code_bytes < 0 || nblocks < 0 || small_numel < 0)
        return set_error(HCP_ERR_INVALID, "adamw8bit: negative size");
    if (ntensors == 0) return HCP_OK;
    if (!p || !g || !maps_device || !tensors_host || !tensors_device || !items_host || !items_device || !hyper_device || !steps_device ||
        ((code_bytes || nblocks) && (!codes || !absmax)) || (small_numel && !state32))
        return set_error(HCP_ERR_INVALID, "adamw8bit: null pointer");
    if (((uintptr_t)p | (uintptr_t)g | (uintptr_t)state32) & 15 || ((uintptr_t)codes & 15) || ((uintptr_t)absmax & 3) || (code_bytes & 15) ||
        (small_numel & 3))
        return set_error(HCP_ERR_INVALID, "adamw8bit: p / g / state32 / codes must be 16-byte aligned, code_bytes a multiple of 16 and "
                                          "small_numel of 4");
    if (ngroups <= 0 || ngroups > A8_T) return set_error(HCP_ERR_INVALID, "adamw8bit: group count");
    if (nitems == 0 || nitems >= (1ll << 31) || nblocks >= (1ll << 40))
        return set_error(HCP_ERR_INVALID, "adamw8bit: item count");
    const int rc = adamw8bit_check_tables(tensors_host, ntensors, items_host, nitems, n, code_bytes, nblocks, small_numel, ngroups);
    if (rc != HCP_OK) return rc;
    const cudaStream_t s = (cudaStream_t)st;
    int64_t blocks = nitems;                           // persistent: 64 registers per thread keep 4 CTAs of 256 on an SM
    if (blocks > num_sms() * 4) blocks = num_sms() * 4;
    launch_k(adafactor_incr_kernel, dim3(1), dim3(AF_T), 0, s, steps_device, (int)ngroups);
    launch_k(adamw8bit_kernel, dim3((unsigned)blocks), dim3(A8_T), 0, s, p, g, codes, codes + code_bytes, absmax, absmax + nblocks,
             state32, state32 + small_numel, maps_device, tensors_device, items_device, (int)nitems, hyper_device,
             (const int*)steps_device, grad_scale, sumsq_device, max_norm);
    LAUNCH_CHECK("adamw8bit launch");
    return HCP_OK;
}
