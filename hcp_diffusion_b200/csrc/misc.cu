// SPDX-License-Identifier: Apache-2.0
// Small kernels at the edges of the UNet hot path (sm_90a): the 4-channel convolutions conv_in / conv_out
// (NCHW fp32 at the module boundary <-> bf16 NHWC inside), the timestep-embedding MLP and all ResnetBlock2D
// time_emb_proj layers as one skinny linear, LoRA parameter packing and LoRA gradient reduction, and the loss /
// optimizer kernels either side of the UNet call.
//
// Replaces (reference): diffusers conv_in / conv_out / Timesteps / TimestepEmbedding / time_emb_proj
// (cfgs/unet_struct.txt:2-8,95,931); LoraBlock.get_weight's alpha*W_up@W_down materialisation
// (hcpdiff/models/lora_base_patch.py:61-62) -> packed low-rank operands; autograd of W_down/W_up;
// Trainer.get_loss (hcpdiff/train_ac.py:506-515) and the AdamW step on the LoRA parameters (train_ac.py:485-494).
#include "common.cuh"
#include "host_util.h"
#include "../../include/hcp_b200.h"

namespace hcp {

// ---------------------------------------------------------------------------------------------
// conv_in: x NCHW fp32 [B,Cin(<=8),H,W] -> y NHWC bf16 [B,H,W,Cout];  w fp32 TAP-MAJOR [Cin,3,3,Cout]
// one thread per (pixel, output channel): the 9*Cin input taps are broadcast loads shared by the warp, the weights of a tap
// are contiguous over the output channels (coalesced; the [Cout,Cin,3,3] parameter layout made them 144-byte strided)
// ---------------------------------------------------------------------------------------------
__global__ void conv_in_kernel(const float* __restrict__ x, const float* __restrict__ w, const float* __restrict__ bias, int B,
                               int Cin, int H, int W, int Cout, __nv_bfloat16* __restrict__ y) {
    pdl_trigger();
    pdl_wait();
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    const int64_t total = (int64_t)B * H * W * Cout;
    if (i >= total) return;
    const int co = (int)(i % Cout);
    const int64_t pix = i / Cout;
    const int xw = (int)(pix % W), yh = (int)((pix / W) % H), b = (int)(pix / ((int64_t)H * W));
    float acc = bias ? bias[co] : 0.f;
    for (int ci = 0; ci < Cin; ++ci)
#pragma unroll
        for (int kh = 0; kh < 3; ++kh) {
            const int ih = yh + kh - 1;
            if (ih < 0 || ih >= H) continue;
#pragma unroll
            for (int kw = 0; kw < 3; ++kw) {
                const int iw = xw + kw - 1;
                if (iw < 0 || iw >= W) continue;
                acc += x[(((int64_t)b * Cin + ci) * H + ih) * W + iw] * w[((ci * 3 + kh) * 3 + kw) * Cout + co];
            }
        }
    y[i] = __float2bfloat16(acc);
}

// ---------------------------------------------------------------------------------------------
// conv_out: x NHWC bf16 [B,H,W,Cin] -> y NCHW fp32 [B,Cout(<=8),H,W];  w fp32 TAP-MAJOR [3,3,Cout,Cin] (contiguous over ci)
// one warp per output pixel: lanes split the channels, shuffle-reduce the Cout partial sums
// ---------------------------------------------------------------------------------------------
template <int COUT>
__global__ void conv_out_kernel(const __nv_bfloat16* __restrict__ x, const float* __restrict__ w, const float* __restrict__ bias,
                                int B, int H, int W, int Cin, float* __restrict__ y) {
    pdl_trigger();
    pdl_wait();
    const int64_t warp = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (warp >= (int64_t)B * H * W) return;
    const int xw = (int)(warp % W), yh = (int)((warp / W) % H), b = (int)(warp / ((int64_t)H * W));
    float acc[COUT];
#pragma unroll
    for (int c = 0; c < COUT; ++c) acc[c] = 0.f;
    for (int kh = 0; kh < 3; ++kh) {
        const int ih = yh + kh - 1;
        if (ih < 0 || ih >= H) continue;
        for (int kw = 0; kw < 3; ++kw) {
            const int iw = xw + kw - 1;
            if (iw < 0 || iw >= W) continue;
            const __nv_bfloat16* xp = x + (((int64_t)b * H + ih) * W + iw) * Cin;
            for (int ci = lane * 2; ci < Cin; ci += 64) {
                const float2 v = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(xp + ci));
#pragma unroll
                for (int c = 0; c < COUT; ++c) {
                    const float2 wv = *reinterpret_cast<const float2*>(w + ((kh * 3 + kw) * COUT + c) * Cin + ci);
                    acc[c] += v.x * wv.x + v.y * wv.y;
                }
            }
        }
    }
#pragma unroll
    for (int c = 0; c < COUT; ++c) {
        const float s = warp_sum(acc[c]);
        if (lane == 0) y[(((int64_t)b * COUT + c) * H + yh) * W + xw] = s + (bias ? bias[c] : 0.f);
    }
}

// dgrad of conv_out: dy NCHW fp32 [B,Cout,H,W] -> dx NHWC bf16 [B,H,W,Cin]; one thread per (pixel, ci); w TAP-MAJOR [3,3,Cout,Cin]
template <int COUT>
__global__ void conv_out_dgrad_kernel(const float* __restrict__ dy, const float* __restrict__ w, int B, int H, int W, int Cin,
                                      __nv_bfloat16* __restrict__ dx) {
    pdl_trigger();
    pdl_wait();
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    const int64_t total = (int64_t)B * H * W * Cin;
    if (i >= total) return;
    const int ci = (int)(i % Cin);
    const int64_t pix = i / Cin;
    const int xw = (int)(pix % W), yh = (int)((pix / W) % H), b = (int)(pix / ((int64_t)H * W));
    float acc = 0.f;
    // dx[ih,iw,ci] = sum_{co,kh,kw} dy[co, ih-kh+1, iw-kw+1] * w[co,ci,kh,kw]
#pragma unroll
    for (int kh = 0; kh < 3; ++kh) {
        const int oh = yh - kh + 1;
        if (oh < 0 || oh >= H) continue;
#pragma unroll
        for (int kw = 0; kw < 3; ++kw) {
            const int ow = xw - kw + 1;
            if (ow < 0 || ow >= W) continue;
#pragma unroll
            for (int c = 0; c < COUT; ++c)
                acc += dy[(((int64_t)b * COUT + c) * H + oh) * W + ow] * w[((kh * 3 + kw) * COUT + c) * Cin + ci];
        }
    }
    dx[i] = __float2bfloat16(acc);
}

// ---------------------------------------------------------------------------------------------
// skinny linear for M <= 16 rows: y[m,n] = sum_k f(x[m,k]) * W[n,k] + bias[n]   (one warp per output column n)
// in_mode: 0 identity, 1 SiLU, 2 x is the timestep [M] and the K inputs are its sinusoidal embedding
//          ([cos | sin], flip_sin_to_cos=True, downscale_freq_shift=0 -- diffusers Timesteps for SD1.x)
// ---------------------------------------------------------------------------------------------
constexpr int SK_MAX_M = 16;
__global__ void skinny_linear_kernel(const float* __restrict__ x, const __nv_bfloat16* __restrict__ Wt, const float* __restrict__ bias,
                                     int M, int K, int N, int in_mode, int out_silu, float* __restrict__ y) {
    pdl_trigger();
    pdl_wait();
    extern __shared__ float sx[];   // [M][K] transformed inputs
    for (int i = threadIdx.x; i < M * K; i += blockDim.x) {
        const int m = i / K, k = i % K;
        float v;
        if (in_mode == 2) {
            const int half = K / 2;
            const int j = (k < half) ? k : k - half;
            const float freq = expf(-9.210340371976184f * (float)j / (float)half);   // ln(10000)
            const float a = x[m] * freq;
            v = (k < half) ? cosf(a) : sinf(a);
        } else {
            v = x[(int64_t)m * K + k];
            if (in_mode == 1) v = v / (1.f + __expf(-v));
        }
        sx[i] = v;
    }
    __syncthreads();
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int n = blockIdx.x * (blockDim.x >> 5) + warp;
    if (n >= N) return;
    float acc[SK_MAX_M];
#pragma unroll
    for (int m = 0; m < SK_MAX_M; ++m) acc[m] = 0.f;
    const __nv_bfloat16* wr = Wt + (int64_t)n * K;
    for (int k = lane * 2; k < K; k += 64) {
        const float2 wv = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(wr + k));
#pragma unroll
        for (int m = 0; m < SK_MAX_M; ++m)
            if (m < M) acc[m] += sx[m * K + k] * wv.x + sx[m * K + k + 1] * wv.y;
    }
#pragma unroll
    for (int m = 0; m < SK_MAX_M; ++m) {
        if (m < M) {
            float s = warp_sum(acc[m]);
            if (lane == 0) {
                s += bias ? bias[n] : 0.f;
                if (out_silu) s = s / (1.f + __expf(-s));
                y[(int64_t)m * N + n] = s;
            }
        }
    }
}

// ---------------------------------------------------------------------------------------------
// fp32 -> bf16 cast (weights once, encoder_hidden_states per step); four elements per thread, 16-byte loads when VEC (x 16-byte
// and y 8-byte aligned), element by element otherwise (a user tensor or a slice of one may start anywhere)
// ---------------------------------------------------------------------------------------------
template <bool VEC>
__global__ void cast_f32_bf16_kernel(const float* __restrict__ x, int64_t n, __nv_bfloat16* __restrict__ y) {
    pdl_trigger();
    pdl_wait();
    const int64_t i = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) * 4;
    if (VEC && i + 3 < n) {
        const float4 v = *reinterpret_cast<const float4*>(x + i);
        uint2 o;
        o.x = pack_bf16x2(v.x, v.y);
        o.y = pack_bf16x2(v.z, v.w);
        *reinterpret_cast<uint2*>(y + i) = o;
    } else {
        for (int64_t j = i; j < n && j < i + 4; ++j) y[j] = __float2bfloat16(x[j]);
    }
}

// ---------------------------------------------------------------------------------------------
// LoRA operand packing.  For every LoRA block (one launch for ALL blocks of the model, driven by a job table):
//   A   [r_tot, in]  rows [c0, c0+r)            = bf16(W_down)               (B operand of T = x . A^T)
//   AT  [in, 64]     cols [c0, c0+r)            = bf16(W_down^T)             (B operand of dX += U . A)
//   Bl  [out_tot,64] rows [o0,o0+out), cols [c0,c0+r) = bf16(alpha * W_up)   (B operand of y += T . Bl^T)
//   BlT [r_tot,out_tot] rows [c0,c0+r), cols [o0,o0+out) = bf16(alpha*W_up^T)(B operand of U = dY . Bl)
// Buffers are zero-initialised once by the caller; blocks of one fused group tile them block-diagonally.
// ---------------------------------------------------------------------------------------------
__global__ void lora_pack_kernel(const hcp_lora_job* __restrict__ jobs, int njobs) {
    pdl_trigger();
    pdl_wait();
    const int j = blockIdx.y;
    if (j >= njobs) return;
    const hcp_lora_job jb = jobs[j];
    const float alpha = jb.alpha;
    const int r = jb.rank, in = jb.in_dim, out = jb.out_dim;
    const int64_t n_down = (int64_t)r * in, n_up = (int64_t)out * r;
    __nv_bfloat16* A = (__nv_bfloat16*)jb.A;
    __nv_bfloat16* AT = (__nv_bfloat16*)jb.AT;
    __nv_bfloat16* Bl = (__nv_bfloat16*)jb.Bl;
    __nv_bfloat16* BlT = (__nv_bfloat16*)jb.BlT;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n_down + n_up; i += (int64_t)gridDim.x * blockDim.x) {
        if (i < n_down) {
            const int rr = (int)(i / in), k = (int)(i % in);
            const __nv_bfloat16 v = __float2bfloat16(jb.w_down[i]);
            A[(int64_t)(jb.c0 + rr) * in + k] = v;
            AT[(int64_t)k * jb.ld_r + jb.c0 + rr] = v;
        } else {
            const int64_t t = i - n_down;
            const int o = (int)(t / r), rr = (int)(t % r);
            const __nv_bfloat16 v = __float2bfloat16(alpha * jb.w_up[t]);
            Bl[(int64_t)(jb.o0 + o) * jb.ld_r + jb.c0 + rr] = v;
            BlT[(int64_t)(jb.c0 + rr) * jb.out_tot + jb.o0 + o] = v;
        }
    }
}

// out[m / per_row, (m % per_row) * dim + j] = cos(x[m] f_j) (j < dim/2) | sin(x[m] f_{j-dim/2}),  f_j = 10000^(-j/(dim/2)):
// diffusers Timesteps(flip_sin_to_cos=True, downscale_freq_shift=0) for the SDXL `time_ids` (add_time_proj), written straight
// into the column slot of the add_embedding input
__global__ void sinusoid_kernel(const float* __restrict__ x, int64_t M, int dim, int per_row, float* __restrict__ out, int64_t ld_out) {
    pdl_trigger();
    pdl_wait();
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= M * dim) return;
    const int64_t m = i / dim;
    const int j = (int)(i % dim), half = dim / 2;
    const int jj = j < half ? j : j - half;
    const float a = x[m] * expf(-9.210340371976184f * (float)jj / (float)half);
    out[(m / per_row) * ld_out + (m % per_row) * dim + j] = j < half ? cosf(a) : sinf(a);
}

// Conv2d LoRA down-projection: fp32 [rank, Cin, 3, 3] -> bf16 wt [R,3,3,Cin] (rows c0..) and wd [Cin,3,3,R] (columns c0..);
// wd is the dgrad arrangement: taps flipped for the stride-1 conv, as-is for the stride-2 phase kernels (hcp_conv3x3_bf16 mode 1)
__global__ void lora_pack_conv_kernel(const hcp_lora_conv_job* __restrict__ jobs, int njobs) {
    pdl_trigger();
    pdl_wait();
    const int j = blockIdx.y;
    if (j >= njobs) return;
    const hcp_lora_conv_job jb = jobs[j];
    const int64_t n = (int64_t)jb.rank * jb.cin * 9;
    __nv_bfloat16* wt = (__nv_bfloat16*)jb.wt;
    __nv_bfloat16* wd = (__nv_bfloat16*)jb.wd;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const int tap = (int)(i % 9);
        const int ci = (int)((i / 9) % jb.cin);
        const int rr = (int)(i / (9 * (int64_t)jb.cin));
        const __nv_bfloat16 v = __float2bfloat16(jb.w_down[i]);
        wt[((int64_t)(jb.c0 + rr) * 9 + tap) * jb.cin + ci] = v;
        const int tap_d = jb.flip ? 8 - tap : tap;
        wd[((int64_t)ci * 9 + tap_d) * jb.ld_r + jb.c0 + rr] = v;
    }
}

// ---------------------------------------------------------------------------------------------
// LoRA weight merge: W_eff = bf16(W_host + sum_b alpha_b * W_up_b . W_down_b), written as the forward operand W [out_tot, in]
// (rows o0 .. o0+out of a fused group) and as the dgrad operand WT [in, out_tot].  This is what the reference layer computes every
// forward -- LoraBlock.get_weight (alpha * mm(W_up, W_down), lora_layers_patch.py:44-45) summed over the stacked blocks by
// LoraPatchContainer.forward (lora_base_patch.py:21-35) and added to the host weight in LinearLayer.forward (:47-57) -- with the
// sum formed in fp32 from the fp32 masters and rounded to bf16 ONCE (autocast's cast of the summed weight).  One launch per step
// covers every patched Linear of the model: a flat grid over the 64x64 tiles of all jobs (tile0 = running tile count, ascending).
// ---------------------------------------------------------------------------------------------
constexpr int MG_T = 64;          // tile edge
constexpr int MG_RMAX = 64;       // sum of the ranks stacked on one host
// Shared memory is sized by the launch for `rcap` = the largest rank sum of any job rounded up to 8 (9 KB + rcap * 528 B: 13 KB for
// rank 8 instead of the 43 KB a rank-64 layout needs), so that 16 instead of 5 blocks share an SM and their load / compute / store
// phases overlap.
__global__ void __launch_bounds__(256) lora_merge_kernel(const hcp_lora_merge_job* __restrict__ jobs, int njobs, const int32_t* __restrict__ tile_job,
                                                         int rcap) {
    extern __shared__ __align__(16) uint8_t mg_smem[];
    __nv_bfloat16 (*s_t)[MG_T + 8] = reinterpret_cast<__nv_bfloat16 (*)[MG_T + 8]>(mg_smem);                  // the merged tile (transposed store)
    float (*s_dn)[MG_T + 4] = reinterpret_cast<float (*)[MG_T + 4]>(mg_smem + MG_T * (MG_T + 8) * 2);          // [rcap] W_down rows over the tile's k range
    float* s_up_base = reinterpret_cast<float*>(mg_smem + MG_T * (MG_T + 8) * 2 + rcap * (MG_T + 4) * 4);      // [64][rcap + 1] alpha * W_up rows
    const int up_ld = rcap + 1;
#define s_up(o, r) s_up_base[(o) * up_ld + (r)]
    pdl_trigger();
    pdl_wait();
    // job of this tile: one load from the caller's tile -> job table, or (no table) the last job with tile0 <= blockIdx.x by a
    // binary search -- seven DEPENDENT global loads per CTA
    int lo = 0;
    if (tile_job) {
        lo = tile_job[blockIdx.x];
    } else {
        int hi = njobs - 1;
        while (lo < hi) {
            const int mid = (lo + hi + 1) >> 1;
            if (jobs[mid].tile0 <= (int)blockIdx.x) lo = mid; else hi = mid - 1;
        }
    }
    const hcp_lora_merge_job& jb = jobs[lo];
    const int in = jb.in_dim, out = jb.out_dim;
    const int tiles_k = (in + MG_T - 1) / MG_T;
    const int t = (int)blockIdx.x - jb.tile0;
    const int o_base = (t / tiles_k) * MG_T, k_base = (t % tiles_k) * MG_T;
    if (o_base >= out) return;
    const int tid = threadIdx.x;
    // this thread's share of the host tile: 8 consecutive k of rows ty and ty + 32, requested before anything else (the fp32 masters
    // are 2/3 of the kernel's traffic and nothing below depends on the low-rank factors until the FMAs)
    const int tx = tid & 7, ty = tid >> 3;
    float4 w[2][2];
#pragma unroll
    for (int i = 0; i < 2; ++i) {
        const int o = o_base + ty + 32 * i, k = k_base + tx * 8;
#pragma unroll
        for (int h = 0; h < 2; ++h)
            w[i][h] = (o < out && k + 4 * h < in) ? __ldg(reinterpret_cast<const float4*>(jb.w_host + (int64_t)o * in + k + 4 * h)) : make_float4(0.f, 0.f, 0.f, 0.f);
    }
    int rtot = 0;
    for (int b = 0; b < jb.nblocks; ++b) {
        const int r = jb.rank[b];
        const float* dn = jb.w_down[b];
        const float* up = jb.w_up[b];
        const float alpha = jb.alpha[b];
        for (int i = tid; i < r * MG_T; i += 256) {
            const int rr = i / MG_T, k = k_base + i % MG_T;
            s_dn[rtot + rr][i % MG_T] = (k < in) ? dn[(int64_t)rr * in + k] : 0.f;
        }
        for (int i = tid; i < MG_T * r; i += 256) {
            const int o = o_base + i / r, rr = i % r;
            s_up(i / r, rtot + rr) = (o < out) ? alpha * up[(int64_t)o * r + rr] : 0.f;
        }
        rtot += r;
    }
    __syncthreads();
    __nv_bfloat16* W = (__nv_bfloat16*)jb.W;
    __nv_bfloat16* WT = (__nv_bfloat16*)jb.WT;
#pragma unroll
    for (int i = 0; i < 2; ++i) {
        const int ol = ty + 32 * i, o = o_base + ol, k = k_base + tx * 8;
        float d[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
        for (int r = 0; r < rtot; ++r) {
            const float u = s_up(ol, r);
            const float4 d0 = *reinterpret_cast<const float4*>(&s_dn[r][tx * 8]), d1 = *reinterpret_cast<const float4*>(&s_dn[r][tx * 8 + 4]);
            d[0] = fmaf(u, d0.x, d[0]); d[1] = fmaf(u, d0.y, d[1]); d[2] = fmaf(u, d0.z, d[2]); d[3] = fmaf(u, d0.w, d[3]);
            d[4] = fmaf(u, d1.x, d[4]); d[5] = fmaf(u, d1.y, d[5]); d[6] = fmaf(u, d1.z, d[6]); d[7] = fmaf(u, d1.w, d[7]);
        }
        uint4 v;
        v.x = pack_bf16x2(w[i][0].x + d[0], w[i][0].y + d[1]);
        v.y = pack_bf16x2(w[i][0].z + d[2], w[i][0].w + d[3]);
        v.z = pack_bf16x2(w[i][1].x + d[4], w[i][1].y + d[5]);
        v.w = pack_bf16x2(w[i][1].z + d[6], w[i][1].w + d[7]);
        if (o < out && k < in) {
            // k-block-major: ((k / 64) * out_tot + row) * 64 + k % 64 (the 8 consecutive k of a thread never straddle a 64-block)
            __nv_bfloat16* dst = jb.tiled ? W + ((int64_t)(k >> 6) * jb.out_tot + jb.o0 + o) * 64 + (k & 63) : W + (int64_t)(jb.o0 + o) * in + k;
            if (k + 8 <= in) *reinterpret_cast<uint4*>(dst) = v;
            else *reinterpret_cast<uint2*>(dst) = make_uint2(v.x, v.y);            // in % 8 == 4 tail
        }
        const __nv_bfloat16* e = reinterpret_cast<const __nv_bfloat16*>(&v);
#pragma unroll
        for (int j = 0; j < 8; ++j) s_t[tx * 8 + j][ol] = e[j];
    }
    __syncthreads();
    if (WT) {
#pragma unroll
        for (int i = 0; i < 2; ++i) {
            const int kl = ty + 32 * i, k = k_base + kl, o = o_base + tx * 8;
            if (k < in && o < out) {
                const int oo = jb.o0 + o;
                __nv_bfloat16* dst = jb.tiled ? WT + ((int64_t)(oo >> 6) * in + k) * 64 + (oo & 63) : WT + (int64_t)k * jb.out_tot + oo;
                const uint4 v = *reinterpret_cast<const uint4*>(&s_t[kl][tx * 8]);
                if (o + 8 <= out) *reinterpret_cast<uint4*>(dst) = v;
                else *reinterpret_cast<uint2*>(dst) = make_uint2(v.x, v.y);
            }
        }
    }
}

#undef s_up

// ---------------------------------------------------------------------------------------------
// loss = mean((pred - target)^2) (fp32, reference train_ac.py:506-515 with loss.type == 'eps'), dpred = 2(pred-target)/n
// ---------------------------------------------------------------------------------------------
__global__ void mse_loss_kernel(const float* __restrict__ pred, const float* __restrict__ target, int64_t n, float grad_scale,
                                float* __restrict__ loss_sum, float* __restrict__ dpred) {
    pdl_trigger();
    pdl_wait();
    __shared__ float s_part[8];
    float acc = 0.f;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const float d = pred[i] - target[i];
        acc += d * d;
        if (dpred) dpred[i] = 2.f * d * grad_scale / (float)n;
    }
    acc = warp_sum(acc);
    if ((threadIdx.x & 31) == 0) s_part[threadIdx.x >> 5] = acc;
    __syncthreads();
    if (threadIdx.x < 32) {
        float v = (threadIdx.x < (blockDim.x >> 5)) ? s_part[threadIdx.x] : 0.f;
        v = warp_sum(v);
        if (threadIdx.x == 0) atomicAdd(loss_sum, v / (float)n);
    }
}

// x_t = sqrt(acp[t]) * x0 + sqrt(1 - acp[t]) * noise   (DDPMScheduler.add_noise, reference train_ac.py:437-447)
__global__ void add_noise_kernel(const float* __restrict__ x0, const float* __restrict__ noise, const int64_t* __restrict__ t,
                                 const float* __restrict__ acp, int64_t per_image, int64_t n, float* __restrict__ xt) {
    pdl_trigger();
    pdl_wait();
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float a = acp[t[i / per_image]];
    xt[i] = sqrtf(a) * x0[i] + sqrtf(1.f - a) * noise[i];
}

// sum of squares of a flat fp32 buffer (for clip_grad_norm_, reference train_ac.py:485-490)
__global__ void sumsq_kernel(const float* __restrict__ g, int64_t n, float* __restrict__ out) {
    pdl_trigger();
    pdl_wait();
    __shared__ float s_part[8];
    float acc = 0.f;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) acc += g[i] * g[i];
    acc = warp_sum(acc);
    if ((threadIdx.x & 31) == 0) s_part[threadIdx.x >> 5] = acc;
    __syncthreads();
    if (threadIdx.x < 32) {
        float v = (threadIdx.x < (blockDim.x >> 5)) ? s_part[threadIdx.x] : 0.f;
        v = warp_sum(v);
        if (threadIdx.x == 0) atomicAdd(out, v);
    }
}

// AdamW over one flat fp32 parameter buffer; grad is first scaled by gscale and clipped to max_norm using the
// device-side sum of squares (no host sync).  step_count lives on the device so the kernel is CUDA-graph replayable.
__global__ void adamw_flat_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m, float* __restrict__ v,
                                  int64_t n, const float* __restrict__ lr_ptr, float beta1, float beta2, float eps, float wd,
                                  float gscale, const float* __restrict__ sumsq, float max_norm, const int* __restrict__ step_ptr) {
    pdl_trigger();
    pdl_wait();
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= n) return;
    float clip = 1.f;
    if (sumsq && max_norm > 0.f) {
        const float norm = sqrtf(*sumsq) * gscale;
        clip = fminf(1.f, max_norm / (norm + 1e-6f));
    }
    const float lr = *lr_ptr;
    const int step = *step_ptr;
    const float grad = g[i] * gscale * clip;
    const float mi = beta1 * m[i] + (1.f - beta1) * grad;
    const float vi = beta2 * v[i] + (1.f - beta2) * grad * grad;
    m[i] = mi;
    v[i] = vi;
    const float bc1 = 1.f - powf(beta1, (float)step);
    const float bc2 = 1.f - powf(beta2, (float)step);
    float w = p[i];
    w -= lr * wd * w;
    w -= lr * (mi / bc1) / (sqrtf(vi / bc2) + eps);
    p[i] = w;
}
// same update with every hyper-parameter read from device memory: hyper = {lr, beta1, beta2, eps, weight_decay}.  LR schedulers
// (OneCycleLR also cycles beta1) then only write five floats; the captured CUDA graph stays valid.  Four elements per thread and
// iteration (16-byte accesses), the bias corrections (two powf) once per thread: the full fine-tune moves 24 GB through this kernel.
__global__ void __launch_bounds__(256) adamw_flat_dev_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m,
                                                             float* __restrict__ v, int64_t n, const float* __restrict__ hyper, float gscale,
                                                             const float* __restrict__ sumsq, float max_norm, const int* __restrict__ step_ptr) {
    pdl_trigger();
    pdl_wait();
    float clip = 1.f;
    if (sumsq && max_norm > 0.f) {
        const float norm = sqrtf(*sumsq) * gscale;
        clip = fminf(1.f, max_norm / (norm + 1e-6f));
    }
    const float lr = hyper[0], beta1 = hyper[1], beta2 = hyper[2], eps = hyper[3], wd = hyper[4];
    const int step = *step_ptr;
    const float gs = gscale * clip;
    const float ibc1 = 1.f / (1.f - powf(beta1, (float)step)), ibc2 = 1.f / (1.f - powf(beta2, (float)step));
    const float decay = 1.f - lr * wd;
    auto upd = [&](float& w, float grad, float& mi, float& vi) {
        grad *= gs;
        mi = beta1 * mi + (1.f - beta1) * grad;
        vi = beta2 * vi + (1.f - beta2) * grad * grad;
        w = w * decay - lr * (mi * ibc1) / (sqrtf(vi * ibc2) + eps);
    };
    const int64_t n4 = n >> 2, stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n4; i += stride) {
        float4 w4 = reinterpret_cast<float4*>(p)[i], m4 = reinterpret_cast<float4*>(m)[i], v4 = reinterpret_cast<float4*>(v)[i];
        const float4 g4 = reinterpret_cast<const float4*>(g)[i];
        upd(w4.x, g4.x, m4.x, v4.x); upd(w4.y, g4.y, m4.y, v4.y); upd(w4.z, g4.z, m4.z, v4.z); upd(w4.w, g4.w, m4.w, v4.w);
        reinterpret_cast<float4*>(p)[i] = w4; reinterpret_cast<float4*>(m)[i] = m4; reinterpret_cast<float4*>(v)[i] = v4;
    }
    if (blockIdx.x == 0 && threadIdx.x < (n & 3)) {             // tail (the flat buffers are 16-byte aligned; n need not be a multiple of 4)
        const int64_t i = (n4 << 2) + threadIdx.x;
        float w = p[i], mi = m[i], vi = v[i];
        upd(w, g[i], mi, vi);
        p[i] = w; m[i] = mi; v[i] = vi;
    }
}
__global__ void incr_step_kernel(int* step) {
    pdl_trigger();
    pdl_wait(); *step += 1; }

}  // namespace hcp

using namespace hcp;

#define LAUNCH_CHECK(what)                                              \
    do {                                                                \
        cudaError_t e_ = cudaGetLastError();                            \
        if (e_ != cudaSuccess) return set_cuda_error(e_, what);         \
    } while (0)

extern "C" int hcp_conv_in_f32(const float* x, const float* w, const float* bias, int64_t B, int64_t Cin, int64_t H, int64_t W,
                               int64_t Cout, void* y, hcp_stream_t st) {
    if (!x || !w || !y) return set_error(HCP_ERR_INVALID, "conv_in: null pointer");
    const int64_t n = B * H * W * Cout;
    launch_k(conv_in_kernel, dim3((unsigned)((n + 255) / 256)), dim3(256), 0, (cudaStream_t)st, x, w, bias, (int)B, (int)Cin, (int)H, (int)W, (int)Cout,
                                                                            (__nv_bfloat16*)y);
    LAUNCH_CHECK("conv_in launch");
    return HCP_OK;
}

extern "C" int hcp_conv_out_f32(const void* x, const float* w, const float* bias, int64_t B, int64_t H, int64_t W, int64_t Cin,
                                int64_t Cout, float* y, hcp_stream_t st) {
    if (!x || !w || !y) return set_error(HCP_ERR_INVALID, "conv_out: null pointer");
    if (Cout != 4 || (Cin & 1)) return set_error(HCP_ERR_INVALID, "conv_out: only Cout == 4, even Cin");
    const int64_t n = B * H * W * 32;
    launch_k(conv_out_kernel<4>, dim3((unsigned)((n + 255) / 256)), dim3(256), 0, (cudaStream_t)st, (const __nv_bfloat16*)x, w, bias, (int)B, (int)H, (int)W,
                                                                                (int)Cin, y);
    LAUNCH_CHECK("conv_out launch");
    return HCP_OK;
}

extern "C" int hcp_conv_out_dgrad_f32(const float* dy, const float* w, int64_t B, int64_t H, int64_t W, int64_t Cin, int64_t Cout,
                                      void* dx, hcp_stream_t st) {
    if (!dy || !w || !dx) return set_error(HCP_ERR_INVALID, "conv_out_dgrad: null pointer");
    if (Cout != 4) return set_error(HCP_ERR_INVALID, "conv_out_dgrad: only Cout == 4");
    const int64_t n = B * H * W * Cin;
    launch_k(conv_out_dgrad_kernel<4>, dim3((unsigned)((n + 255) / 256)), dim3(256), 0, (cudaStream_t)st, dy, w, (int)B, (int)H, (int)W, (int)Cin,
                                                                                      (__nv_bfloat16*)dx);
    LAUNCH_CHECK("conv_out_dgrad launch");
    return HCP_OK;
}

extern "C" int hcp_skinny_linear(const float* x, const void* w_bf16, const float* bias, int64_t M, int64_t K, int64_t N, int in_mode,
                                 int out_silu, float* y, hcp_stream_t st) {
    if (!x || !w_bf16 || !y) return set_error(HCP_ERR_INVALID, "skinny_linear: null pointer");
    if (M < 1 || M > SK_MAX_M || (K & 1)) return set_error(HCP_ERR_INVALID, "skinny_linear: 1 <= M <= 16, even K");
    const size_t smem = (size_t)M * K * sizeof(float);
    if (smem > 96 * 1024) return set_error(HCP_ERR_INVALID, "skinny_linear: M*K too large");
    static bool configured = false;
    if (!configured) {
        cudaError_t e = cudaFuncSetAttribute(skinny_linear_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 96 * 1024);
        if (e != cudaSuccess) return set_cuda_error(e, "cudaFuncSetAttribute(skinny_linear)");
        configured = true;
    }
    const int warps = 8;
    launch_k(skinny_linear_kernel, dim3((unsigned)((N + warps - 1) / warps)), dim3(warps * 32), smem, (cudaStream_t)st, 
        x, (const __nv_bfloat16*)w_bf16, bias, (int)M, (int)K, (int)N, in_mode, out_silu, y);
    LAUNCH_CHECK("skinny_linear launch");
    return HCP_OK;
}

extern "C" int hcp_cast_f32_to_bf16(const float* x, int64_t n, void* y, hcp_stream_t st) {
    if (!x || !y) return set_error(HCP_ERR_INVALID, "cast: null pointer");
    if (n < 0) return set_error(HCP_ERR_INVALID, "cast: negative size");
    if (n == 0) return HCP_OK;
    const int64_t threads = (n + 3) / 4;
    const dim3 grid((unsigned)((threads + 255) / 256));
    if ((((uintptr_t)x & 15) | ((uintptr_t)y & 7)) == 0)
        launch_k(cast_f32_bf16_kernel<true>, grid, dim3(256), 0, (cudaStream_t)st, x, n, (__nv_bfloat16*)y);
    else
        launch_k(cast_f32_bf16_kernel<false>, grid, dim3(256), 0, (cudaStream_t)st, x, n, (__nv_bfloat16*)y);
    LAUNCH_CHECK("cast launch");
    return HCP_OK;
}

extern "C" int hcp_lora_pack(const hcp_lora_job* jobs_device, int64_t njobs, hcp_stream_t st) {
    if (!jobs_device || njobs <= 0) return set_error(HCP_ERR_INVALID, "lora_pack: jobs");
    dim3 grid(16, (unsigned)njobs);
    launch_k(lora_pack_kernel, dim3(grid), dim3(256), 0, (cudaStream_t)st, jobs_device, (int)njobs);
    LAUNCH_CHECK("lora_pack launch");
    return HCP_OK;
}

extern "C" int hcp_lora_merge(const hcp_lora_merge_job* jobs_device, int64_t njobs, int64_t total_tiles, const int32_t* tile_job_device,
                              int32_t max_rank_sum, hcp_stream_t st) {
    if (!jobs_device || njobs <= 0 || total_tiles <= 0) return set_error(HCP_ERR_INVALID, "lora_merge: jobs");
    if (max_rank_sum <= 0 || max_rank_sum > MG_RMAX) max_rank_sum = MG_RMAX;
    const int rcap = (max_rank_sum + 7) / 8 * 8;
    const size_t smem = (size_t)MG_T * (MG_T + 8) * 2 + (size_t)rcap * (MG_T + 4) * 4 + (size_t)MG_T * (rcap + 1) * 4;
    launch_k(lora_merge_kernel, dim3((unsigned)total_tiles), dim3(256), smem, (cudaStream_t)st, jobs_device, (int)njobs, tile_job_device, rcap);
    LAUNCH_CHECK("lora_merge launch");
    return HCP_OK;
}

extern "C" int hcp_sinusoid_f32(const float* x, int64_t M, int64_t dim, int64_t per_row, float* out, int64_t ld_out, hcp_stream_t st) {
    if (!x || !out || M <= 0 || dim <= 0 || (dim & 1) || per_row <= 0) return set_error(HCP_ERR_INVALID, "sinusoid: arguments");
    const int64_t n = M * dim;
    launch_k(sinusoid_kernel, dim3((unsigned)((n + 255) / 256)), dim3(256), 0, (cudaStream_t)st, x, M, (int)dim, (int)per_row, out, ld_out);
    LAUNCH_CHECK("sinusoid launch");
    return HCP_OK;
}

extern "C" int hcp_lora_pack_conv(const hcp_lora_conv_job* jobs_device, int64_t njobs, hcp_stream_t st) {
    if (!jobs_device || njobs <= 0) return set_error(HCP_ERR_INVALID, "lora_pack_conv: jobs");
    dim3 grid(16, (unsigned)njobs);
    launch_k(lora_pack_conv_kernel, dim3(grid), dim3(256), 0, (cudaStream_t)st, jobs_device, (int)njobs);
    LAUNCH_CHECK("lora_pack_conv launch");
    return HCP_OK;
}

extern "C" int hcp_mse_loss(const float* pred, const float* target, int64_t n, float grad_scale, float* loss_sum, float* dpred,
                            hcp_stream_t st) {
    if (!pred || !target || !loss_sum) return set_error(HCP_ERR_INVALID, "mse_loss: null pointer");
    if (n < 0) return set_error(HCP_ERR_INVALID, "mse_loss: negative size");
    if (n == 0) return HCP_OK;
    int blocks = (int)((n + 255) / 256);
    if (blocks > 592) blocks = 592;
    launch_k(mse_loss_kernel, dim3(blocks), dim3(256), 0, (cudaStream_t)st, pred, target, n, grad_scale, loss_sum, dpred);
    LAUNCH_CHECK("mse_loss launch");
    return HCP_OK;
}

extern "C" int hcp_add_noise(const float* x0, const float* noise, const int64_t* t, const float* alphas_cumprod, int64_t B,
                             int64_t per_image, float* xt, hcp_stream_t st) {
    if (!x0 || !noise || !t || !alphas_cumprod || !xt) return set_error(HCP_ERR_INVALID, "add_noise: null pointer");
    if (B < 0 || per_image < 0) return set_error(HCP_ERR_INVALID, "add_noise: negative size");
    const int64_t n = B * per_image;
    if (n == 0) return HCP_OK;
    launch_k(add_noise_kernel, dim3((unsigned)((n + 255) / 256)), dim3(256), 0, (cudaStream_t)st, x0, noise, t, alphas_cumprod, per_image, n, xt);
    LAUNCH_CHECK("add_noise launch");
    return HCP_OK;
}

extern "C" int hcp_sumsq(const float* g, int64_t n, float* out, hcp_stream_t st) {
    if (!g || !out) return set_error(HCP_ERR_INVALID, "sumsq: null pointer");
    if (n < 0) return set_error(HCP_ERR_INVALID, "sumsq: negative size");
    if (n == 0) return HCP_OK;
    int blocks = (int)((n + 255) / 256);
    if (blocks > 592) blocks = 592;
    launch_k(sumsq_kernel, dim3(blocks), dim3(256), 0, (cudaStream_t)st, g, n, out);
    LAUNCH_CHECK("sumsq launch");
    return HCP_OK;
}

extern "C" int hcp_adamw_flat(float* p, const float* g, float* m, float* v, int64_t n, const float* lr_device, float beta1, float beta2,
                              float eps, float weight_decay, float grad_scale, const float* sumsq_device, float max_norm,
                              int* step_device, hcp_stream_t st) {
    if (!p || !g || !m || !v || !lr_device || !step_device) return set_error(HCP_ERR_INVALID, "adamw: null pointer");
    if (n < 0) return set_error(HCP_ERR_INVALID, "adamw: negative size");
    if (n == 0) return HCP_OK;
    launch_k(incr_step_kernel, dim3(1), dim3(1), 0, (cudaStream_t)st, step_device);
    launch_k(adamw_flat_kernel, dim3((unsigned)((n + 255) / 256)), dim3(256), 0, (cudaStream_t)st, p, g, m, v, n, lr_device, beta1, beta2, eps, weight_decay,
                                                                               grad_scale, sumsq_device, max_norm, step_device);
    LAUNCH_CHECK("adamw launch");
    return HCP_OK;
}

extern "C" int hcp_adamw_flat_dev(float* p, const float* g, float* m, float* v, int64_t n, const float* hyper_device, float grad_scale,
                                  const float* sumsq_device, float max_norm, int* step_device, hcp_stream_t st) {
    if (!p || !g || !m || !v || !hyper_device || !step_device) return set_error(HCP_ERR_INVALID, "adamw_dev: null pointer");
    if (n < 0) return set_error(HCP_ERR_INVALID, "adamw_dev: negative size");
    if (((uintptr_t)p | (uintptr_t)g | (uintptr_t)m | (uintptr_t)v) & 15) return set_error(HCP_ERR_INVALID, "adamw_dev: buffers must be 16-byte aligned");
    if (n == 0) return HCP_OK;
    int64_t blocks = ((n >> 2) + 255) / 256;
    if (blocks > num_sms() * 16) blocks = num_sms() * 16;
    if (blocks < 1) blocks = 1;
    launch_k(incr_step_kernel, dim3(1), dim3(1), 0, (cudaStream_t)st, step_device);
    launch_k(adamw_flat_dev_kernel, dim3((unsigned)blocks), dim3(256), 0, (cudaStream_t)st, p, g, m, v, n, hyper_device, grad_scale,
             sumsq_device, max_norm, step_device);
    LAUNCH_CHECK("adamw_dev launch");
    return HCP_OK;
}
