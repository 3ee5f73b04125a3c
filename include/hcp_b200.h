/* SPDX-License-Identifier: Apache-2.0
 *
 * libhcpb200 -- C ABI of the H100 (sm_90a) kernels behind the HCP-Diffusion UNet denoising hot path.
 *
 * The reference (IrisRainbowNeko/HCP-Diffusion @ 404f0e85) has NO native code and NO FFI: every op
 * below replaces a PyTorch call made from the pure-Python hot path.  Each entry point cites the
 * reference call it replaces (paths relative to the reference root).
 *
 * Conventions
 *   - every function returns 0 on success, a negative hcp_status otherwise; nothing throws across the ABI;
 *     hcp_last_error_string() describes the last failure on the calling thread.
 *   - the caller owns every buffer (activations, outputs, workspaces); the library never allocates device
 *     memory, never synchronises and only enqueues work on the `stream` argument (a cudaStream_t).
 *   - activations are bf16, row-major "NHWC": a [B,H,W,C] feature map is the same memory as the [B*H*W, C]
 *     token matrix the transformer blocks use.  Accumulation is fp32.  `ld*` are row pitches in ELEMENTS.
 *   - all device pointers must be 16-byte aligned, all row pitches multiples of 8 elements.  The elementwise bf16 kernels (GEGLU,
 *     GELU, quick-GELU, upsample, add, the bf16 sum, dropout) and hcp_adamw_flat_dev refuse a pointer off 16-byte alignment with
 *     HCP_ERR_INVALID before any launch; hcp_cast_f32_to_bf16 takes an element-wise path for it instead.
 *   - the elementwise and training-step kernels refuse a negative size with HCP_ERR_INVALID; an empty one (n, M or B == 0) returns
 *     HCP_OK and launches nothing.  A refused call launches nothing and changes no device state (step counters included).
 */
#ifndef HCP_B200_H_
#define HCP_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef void* hcp_stream_t; /* cudaStream_t */

enum hcp_status {
    HCP_OK = 0,
    HCP_ERR_INVALID = -1,   /* bad argument / unsupported shape */
    HCP_ERR_CUDA = -2,      /* CUDA runtime or driver error (see hcp_last_error_string) */
    HCP_ERR_NO_DEVICE = -3, /* no sm_90 device / driver entry point missing */
};

int hcp_version(void);                     /* ABI version, bumps on any signature change */
const char* hcp_last_error_string(void);   /* thread-local, never NULL */
int hcp_device_check(void);                /* HCP_OK iff the current device is compute capability 10.x */
/* Number of kernels the library has launched in this process (every launch goes through one counter; kernels captured into a
 * CUDA graph are counted once, at capture).  bench.py reports differences of this value as `gpu_launches`. */
unsigned long long hcp_launch_count(void);

/* ------------------------------------------------------------------------------------------------
 * GEMM family (wgmma + TMA).  out[M,N] = sum_s A_s[M,K_s] . B_s[N,K_s]^T  (+ epilogue)
 *
 * Replaces: LinearLayer.forward -> torch.mm(x2d, (W_host + dW).T)   hcpdiff/models/lora_layers_patch.py:50-57
 *           LinearLayer.get_weight -> alpha*mm(W_up, W_down)         hcpdiff/models/lora_layers_patch.py:44-45
 *           LoraPatchContainer.forward / LoraBlock.post_forward       hcpdiff/models/lora_base_patch.py:21-35,68-74
 *           nn.Linear / 1x1 nn.Conv2d inside diffusers' UNet2DConditionModel (structure: cfgs/unet_struct.txt)
 * The rank-r LoRA product is never materialised as a [out,in] matrix: segment 1 is (x.W_down^T)[M,rpad] times
 * (alpha*W_up)[N,rpad], i.e. extra K-blocks of the same tensor-core pipeline.
 * ---------------------------------------------------------------------------------------------- */
#define HCP_GEMM_MAX_SEG 3

typedef struct hcp_gemm_args {
    int32_t nseg;                          /* 1..3 K-segments */
    const void* a[HCP_GEMM_MAX_SEG];       /* bf16 [M, k[s]] row-major, pitch lda[s] */
    const void* b[HCP_GEMM_MAX_SEG];       /* bf16 [n_rows_b[s], k[s]] row-major, pitch ldb[s]; rows >= n_rows_b read as 0 */
    int64_t lda[HCP_GEMM_MAX_SEG];
    int64_t ldb[HCP_GEMM_MAX_SEG];
    int64_t k[HCP_GEMM_MAX_SEG];           /* reduction extent; the TMA box is 64 wide, tails read as zero */
    int64_t n_rows_b[HCP_GEMM_MAX_SEG];    /* valid rows of b[s] (== N normally; < N for the LoRA down-projection) */
    int64_t M, N;
    const float* bias;                     /* fp32 [N] or NULL */
    const float* rowbias;                  /* fp32 [ceil(M/rows_per_group), N] or NULL (time-embedding bias per image) */
    int64_t rows_per_group;
    int64_t rowbias_ld;                    /* row pitch of rowbias in floats (0 -> N) */
    const void* residual;                  /* bf16 [M,N] pitch ldr, or NULL: added in the epilogue */
    int64_t ldr;
    void* out;                             /* bf16 [M,N] pitch ldo */
    int64_t ldo;
    int32_t flags;                         /* bit s: b[s] is K-BLOCK-MAJOR -- element (n, k) at b + ((k/64)*ldb[s] + n)*64 + k%64, i.e.
                                            * [k[s]/64][ldb[s] rows][64]: every 64-wide TMA box of B is one contiguous run of memory
                                            * (weight streaming at small M reads whole DRAM pages); needs k[s] % 64 == 0 */
    float* workspace;                      /* optional split-K scratch (see hcp_splitk_workspace_bytes); NULL = never split */
    size_t workspace_bytes;
    /* Second output: columns [n_main, N) of the product go, raw (no bias / rowbias / residual), to out2[row*ldo2 + col - n_main].
     * This is how the rank-r LoRA products ride the layer's own GEMM: the weight operand carries W_down (forward: T = x W_down^T) or
     * alpha*W_up^T (dgrad: U = dY alpha W_up) as rows n_main.. of b[].  out2 == NULL: single output.  n_main, ldo2 multiples of 8. */
    void* out2;
    int64_t ldo2;
    int64_t n_main;
} hcp_gemm_args;

int hcp_gemm_bf16(const hcp_gemm_args* args, hcp_stream_t stream);
/* Bytes of fp32 scratch that let a GEMM / conv with this output and total reduction extent (sum of K over segments;
 * 9*Cin for a 3x3 conv) split its reduction over several CTAs when the output alone cannot fill the SMs; 0 = no split. */
size_t hcp_splitk_workspace_bytes(int64_t M, int64_t N, int64_t total_k);

/* ------------------------------------------------------------------------------------------------
 * 3x3 convolution as implicit GEMM (wgmma; the im2col gather is done by 4D/5D TMA boxes with
 * out-of-bounds zero fill standing in for the padding).
 *
 * Replaces: F.conv2d inside diffusers ResnetBlock2D.conv1/conv2, Downsample2D.conv (stride 2),
 *           Upsample2D.conv (after nearest x2) -- module shapes pinned by cfgs/unet_struct.txt;
 *           and its dgrad (autograd of the same call) for the backward pass.
 *   mode 0: y[b,ho,wo,:] = sum_{kh,kw} x[b, ho*s+kh-1, wo*s+kw-1, :] . w[:, kh, kw, :]^T   (s = stride, pad 1)
 *   mode 1: transposed conv of a stride-2 conv (dgrad): x is dY [B,H/2,W/2,Cin'], output [B,H,W,Cout'];
 *           w must already be the "dgrad" arrangement (see hcp_conv3x3_args.w).
 * ---------------------------------------------------------------------------------------------- */
typedef struct hcp_conv3x3_args {
    const void* x;       /* bf16 [B, Hin, Win, Cin] */
    const void* w;       /* bf16 [Cout, 3, 3, Cin] (tap-major, channel-minor "K-major" layout) */
    int64_t B, Hin, Win, Cin, Cout;
    int32_t stride;      /* 1 or 2 */
    int32_t mode;        /* 0 = forward conv, 1 = dgrad of the stride-2 conv */
    const float* bias;   /* fp32 [Cout] or NULL */
    const float* rowbias;/* fp32 [B, Cout] or NULL (time embedding projection, broadcast over H,W) */
    int64_t rowbias_ld;  /* row pitch of rowbias in floats (0 -> Cout) */
    const void* residual;/* bf16 [B,Hout,Wout,Cout] or NULL */
    void* out;           /* bf16 [B,Hout,Wout,Cout] */
    float* workspace;    /* optional split-K scratch, hcp_splitk_workspace_bytes(B*Hout*Wout, Cout, 9*Cin) */
    size_t workspace_bytes;
    /* Conv2d LoRA (LoCon, reference lora_layers_patch.py:64-100), mode 0 only: out += T . Bl^T as one more K-segment, where
     * T = conv3x3(x, W_down) [B*Hout*Wout, lora_ld] was produced by a previous call and Bl = alpha*W_up [Cout, lora_ld]. */
    const void* lora_t;  /* bf16 or NULL */
    const void* lora_b;  /* bf16 */
    int64_t lora_r;      /* rank columns in use (<= lora_ld) */
    int64_t lora_ld;     /* row pitch of lora_t / lora_b: the 64-padded rank */
    int32_t w_tiled;     /* 1: w is K-BLOCK-MAJOR [9*Cin/64][Cout][64] (k = (kh*3+kw)*Cin + ci): every weight box is one contiguous 128*rows-byte run */
} hcp_conv3x3_args;

int hcp_conv3x3_bf16(const hcp_conv3x3_args* args, hcp_stream_t stream);

/* ------------------------------------------------------------------------------------------------
 * Fused attention (wgmma flash-style forward, and backward).
 *
 * Replaces: diffusers Attention -> F.scaled_dot_product_attention / xformers.memory_efficient_attention
 *           (selected at reference hcpdiff/train_ac.py:258-263) for BasicTransformerBlock.attn1 / attn2
 *           (reference cfgs/unet_struct.txt:17-43), and its autograd backward.
 * q/k/v/o/dout/dq/dk/dv: bf16 [B, L, ld] token-major, head h in columns [h*d, (h+1)*d); d % 8 == 0, d <= 192.
 * kv_bias: optional fp32 [B, Lkv] additive logit bias = (1 - encoder_attention_mask) * -10000
 *          (the diffusers convention restated at reference hcpdiff/models/controlnet.py:99-103).
 * lse: fp32 [B, H, Lq] natural-log sum-exp of the scaled logits (saved for backward; may be NULL in fwd).
 * ---------------------------------------------------------------------------------------------- */
typedef struct hcp_attn_args {
    const void* q; int64_t ldq;
    const void* k; int64_t ldk;
    const void* v; int64_t ldv;
    int64_t B, H, Lq, Lkv, d;
    float scale;
    const float* kv_bias;
    void* o; int64_t ldo;
    float* lse;
} hcp_attn_args;

int hcp_attn_fwd_bf16(const hcp_attn_args* args, hcp_stream_t stream);

typedef struct hcp_attn_bwd_args {
    const void* q; int64_t ldq;
    const void* k; int64_t ldk;
    const void* v; int64_t ldv;
    const void* o; int64_t ldo;
    const void* dout; int64_t lddo;
    int64_t B, H, Lq, Lkv, d;
    float scale;
    const float* kv_bias;
    const float* lse;
    void* dq; int64_t lddq;
    void* dk; int64_t lddk;
    void* dv; int64_t lddv;
    float* workspace;            /* >= hcp_attn_bwd_workspace_bytes(B,H,Lq,Lkv,d) bytes, caller-owned scratch */
    size_t workspace_bytes;
} hcp_attn_bwd_args;

size_t hcp_attn_bwd_workspace_bytes(int64_t B, int64_t H, int64_t Lq, int64_t Lkv, int64_t d);
int hcp_attn_bwd_bf16(const hcp_attn_bwd_args* args, hcp_stream_t stream);

/* Causal self-attention: the same arguments with Lq == Lkv (else HCP_ERR_INVALID before any launch); query row i attends to kv
 * columns <= i, kv_bias (if given) still adds on top.  The backward uses the same workspace size.
 * Replaces: transformers CLIPAttention with CLIPTextTransformer's causal_attention_mask (text encoder self_attn, reference
 *           cfgs/te_struct.txt; run every step when `lora_text_encoder` is set, hcpdiff/models/wrapper.py:14-30) and its backward. */
int hcp_attn_fwd_causal_bf16(const hcp_attn_args* args, hcp_stream_t stream);
int hcp_attn_bwd_causal_bf16(const hcp_attn_bwd_args* args, hcp_stream_t stream);

/* ------------------------------------------------------------------------------------------------
 * GroupNorm (+SiLU) over NHWC bf16, optionally over the channel concatenation [x1 | x2] (up-block skip
 * connections: the concat is never materialised un-normalised), forward and backward.
 *
 * Replaces: ResnetBlock2D.norm1/norm2 + SiLU (reference cfgs/unet_struct.txt:93-99), Transformer2DModel.norm
 *           (:13, eps 1e-6, no SiLU), conv_norm_out + SiLU (:929) and torch.cat([h, skip], dim=1) in the up blocks.
 * fwd: y[B,HW,C1+C2] = act(GN(cat(x1,x2))); stats[B,G,2] = (mean, rstd) saved for backward.
 * bwd: dx1 = dGN/dx1 (+ add1), dx2 = dGN/dx2 (+ add2); gamma/beta gradients are not produced (frozen base).
 * workspace: >= hcp_groupnorm_workspace_bytes(B, HW, G) bytes of caller-owned scratch.
 * ---------------------------------------------------------------------------------------------- */
typedef struct hcp_groupnorm_args {
    const void* x1; const void* x2;     /* bf16 [B,HW,C1], [B,HW,C2] (x2 may be NULL with C2 == 0) */
    int64_t B, HW, C1, C2, G;
    const float* gamma; const float* beta;   /* fp32 [C1+C2] */
    float eps;
    int32_t silu;
    float* stats;                       /* fp32 [B,G,2]: written by fwd, read by bwd */
    float* workspace; size_t workspace_bytes;
    void* y;                            /* fwd: bf16 [B,HW,C1+C2] */
    const void* dy;                     /* bwd: bf16 [B,HW,C1+C2] */
    const void* add1; const void* add2; /* bwd: optional bf16 gradients accumulated into dx1 / dx2 */
    void* dx1; void* dx2;               /* bwd outputs */
} hcp_groupnorm_args;

size_t hcp_groupnorm_workspace_bytes(int64_t B, int64_t HW, int64_t G);
int hcp_groupnorm_fwd_bf16(const hcp_groupnorm_args* args, hcp_stream_t stream);
int hcp_groupnorm_bwd_bf16(const hcp_groupnorm_args* args, hcp_stream_t stream);

/* LayerNorm over the last dim of a bf16 [M,C] matrix (BasicTransformerBlock.norm1/2/3, cfgs/unet_struct.txt:44-46).
 * stats fp32 [M,2] (mean, rstd).  bwd: dx = dLN/dx (+ add). */
int hcp_layernorm_fwd_bf16(const void* x, const float* gamma, const float* beta, float eps, int64_t M, int64_t C, float* stats,
                           void* y, hcp_stream_t stream);
int hcp_layernorm_bwd_bf16(const void* x, const void* dy, const void* add, const float* gamma, const float* stats, int64_t M,
                           int64_t C, void* dx, hcp_stream_t stream);

/* GEGLU (cfgs/unet_struct.txt:27-30): u bf16 [M,2F] = [a | g];  h = a * gelu_erf(g);  du = [dh*gelu(g) | dh*a*gelu'(g)] */
int hcp_geglu_fwd_bf16(const void* u, int64_t M, int64_t F, void* h, hcp_stream_t stream);
int hcp_geglu_bwd_bf16(const void* u, const void* dh, int64_t M, int64_t F, void* du, hcp_stream_t stream);

/* quick-GELU (transformers QuickGELUActivation, CLIPMLP.activation_fn, reference cfgs/te_struct.txt): x, y, dy, dx bf16 [M,F],
 * F % 8 == 0;  y = x * sigmoid(1.702 x);  dx = dy * (s + 1.702 x s (1 - s)), s = sigmoid(1.702 x).  fp32 arithmetic. */
int hcp_quick_gelu_fwd_bf16(const void* x, int64_t M, int64_t F, void* y, hcp_stream_t stream);
int hcp_quick_gelu_bwd_bf16(const void* x, const void* dy, int64_t M, int64_t F, void* dx, hcp_stream_t stream);

/* exact GELU (transformers GELUActivation, hidden_act='gelu': the MLP of SDXL's second text encoder, OpenCLIP ViT-bigG/14): x, y, dy,
 * dx bf16 [M,F], F % 8 == 0;  y = 0.5 x (1 + erf(x / sqrt 2));  dx = dy * (Phi(x) + x phi(x)) from the saved pre-activation x.
 * fp32 arithmetic, Phi(x) = erfc(-x / sqrt 2) / 2 (accurate in the lower tail, where 1 + erf cancels). */
int hcp_gelu_fwd_bf16(const void* x, int64_t M, int64_t F, void* y, hcp_stream_t stream);
int hcp_gelu_bwd_bf16(const void* x, const void* dy, int64_t M, int64_t F, void* dx, hcp_stream_t stream);

/* out fp32 [n] = srcs[0] + srcs[1] + ... + srcs[nsrc-1] (bf16 [n] each, n % 8 == 0), summed in fp32 in source order.
 * Replaces: autograd's fp32 accumulation of the gradient of the fp32 text embedding, which the reference casts to bf16 separately for
 *           every cross-attention under autocast (attn2.to_k / to_v, reference cfgs/unet_struct.txt:35-38; TEUnetWrapper.forward,
 *           hcpdiff/models/wrapper.py:14-30). */
int hcp_sum_bf16_to_f32(const void* const* srcs, int64_t nsrc, int64_t n, float* out, hcp_stream_t stream);

/* Token + position embedding (transformers CLIPTextEmbeddings.forward, reference cfgs/te_struct.txt):
 * out[b, l, :] = bf16(tok_emb[ids[b, l]] + pos_emb[pos_ids ? pos_ids[l] : l]).  ids int64 [B, L] and pos_ids int64 [L] (or NULL)
 * live on the device, so the call can be captured in a CUDA graph; an id outside [0, V) (position outside [0, P)) is clamped to
 * the nearest valid row -- the tables are never read out of bounds.  tok_emb fp32 [V, C], pos_emb fp32 [P, C], C % 8 == 0;
 * without pos_ids, L <= P.  out bf16 [B, L, C]. */
int hcp_embed_gather_bf16(const int64_t* ids, const int64_t* pos_ids, const float* tok_emb, int64_t V, const float* pos_emb, int64_t P,
                          int64_t B, int64_t L, int64_t C, void* out, hcp_stream_t stream);

/* Backward of hcp_embed_gather_bf16 (the embedding tables trained: `text_encoder:` full fine-tuning, reference
 * hcpdiff/train_ac.py:324-340 through autograd's embedding backward).  dH bf16 [B, L, C]; with ids and positions clamped as the gather
 * clamps them:  dtok[v, :] += sum of dH[r, :] over the rows r = b L + l with id v   (fp32 [V, C], or NULL: not trained)
 *               dpos[p, :] += sum of dH[r, :] over the rows at position p           (fp32 [P, C], or NULL), at least one given.
 * Deterministic without float atomics: the rows of one table row are taken in row order and cut into pieces at every multiple of 32
 * of their position in the stable (table row, row) order of all B L rows; each piece is summed from 0 in row order, the pieces are
 * added in order, and the total is added to the table row once.  Repeats and graph replays are bit-identical.  Ids stay on the
 * device (no host sync, graph-capturable).  C % 8 == 0, V, P <= INT32_MAX; without pos_ids (and dpos given) L <= P.  dH, dtok,
 * dpos and the workspace 16-byte aligned, ids / pos_ids 8-byte; workspace_bytes >= hcp_embed_grad_workspace_bytes(B, L, C)
 * (0 for a non-positive size).  Three launches. */
size_t hcp_embed_grad_workspace_bytes(int64_t B, int64_t L, int64_t C);
int hcp_embed_grad_bf16(const int64_t* ids, const int64_t* pos_ids, const void* dH, int64_t B, int64_t L, int64_t C, float* dtok, int64_t V,
                        float* dpos, int64_t P, void* workspace, size_t workspace_bytes, hcp_stream_t stream);

/* nearest x2 upsample of NHWC bf16 [B,H,W,C] (Upsample2D, cfgs/unet_struct.txt:392) and its backward */
int hcp_upsample2x_fwd_bf16(const void* x, int64_t B, int64_t H, int64_t W, int64_t C, void* y, hcp_stream_t stream);
int hcp_upsample2x_bwd_bf16(const void* dy, int64_t B, int64_t H, int64_t W, int64_t C, void* dx, hcp_stream_t stream);
int hcp_add_bf16(const void* a, const void* b, int64_t n, void* out, hcp_stream_t stream);

/* ------------------------------------------------------------------------------------------------
 * Module-boundary kernels: the UNet call takes NCHW fp32 latents and returns NCHW fp32 noise_pred
 * (reference hcpdiff/models/wrapper.py:29); inside everything is bf16 NHWC.  Weights are fp32 and TAP-MAJOR so that a warp reads
 * them contiguously: conv_in  w[Cin][3][3][Cout]  (= nn.Conv2d weight.permute(1,2,3,0));
 *                    conv_out w[3][3][Cout][Cin]  (= weight.permute(2,3,0,1)), also for its dgrad.
 * ---------------------------------------------------------------------------------------------- */
/* Sinusoidal embedding of M scalars (diffusers Timesteps, flip_sin_to_cos, shift 0): element m lands in row m / per_row at
 * column (m % per_row) * dim of `out` (row pitch ld_out floats) -- the SDXL time_ids slot of the add_embedding input
 * (diffusers add_time_proj; reference hcpdiff/models/wrapper.py:66 supplies the ids as `crop_info`). */
int hcp_sinusoid_f32(const float* x, int64_t M, int64_t dim, int64_t per_row, float* out, int64_t ld_out, hcp_stream_t stream);
int hcp_conv_in_f32(const float* x_nchw, const float* w, const float* bias, int64_t B, int64_t Cin, int64_t H, int64_t W,
                    int64_t Cout, void* y_nhwc_bf16, hcp_stream_t stream);
int hcp_conv_out_f32(const void* x_nhwc_bf16, const float* w, const float* bias, int64_t B, int64_t H, int64_t W, int64_t Cin,
                     int64_t Cout, float* y_nchw, hcp_stream_t stream);
int hcp_conv_out_dgrad_f32(const float* dy_nchw, const float* w, int64_t B, int64_t H, int64_t W, int64_t Cin, int64_t Cout,
                           void* dx_nhwc_bf16, hcp_stream_t stream);
/* y[M,N] fp32 = f(x)[M,K] . W[N,K]^T + bias, any M >= 1 (16 rows per CTA row of the grid, K staged in 512-column chunks; every row
 * is summed in the same order whatever M is, so a row's result does not depend on the rows launched with it).  in_mode 0: f = id, 1: f = SiLU, 2: x is timesteps [M] and f is the
 * sinusoidal embedding (diffusers Timesteps: [cos | sin], freq = exp(-ln(1e4) * j / (K/2))).  W is bf16. */
int hcp_skinny_linear(const float* x, const void* w_bf16, const float* bias, int64_t M, int64_t K, int64_t N, int in_mode,
                      int out_silu, float* y, hcp_stream_t stream);
/* y bf16 [n] = x fp32 [n] rounded to nearest even; any alignment (16-byte x and 8-byte y take the vector path) */
int hcp_cast_f32_to_bf16(const float* x, int64_t n, void* y, hcp_stream_t stream);

/* ------------------------------------------------------------------------------------------------
 * LoRA operand packing / gradient reduction.
 * Replaces LoraBlock.get_weight (alpha * mm(W_up, W_down), reference lora_base_patch.py:61-62,
 * lora_layers_patch.py:44-45) and autograd of W_down / W_up.  One job per LoRA block; blocks that share a fused
 * GEMM (to_q/to_k/to_v on the same input; several stacked blocks on one layer) tile the packed operands
 * block-diagonally via (c0, o0).  c0 is the block's first column inside the group's R-wide T / U buffers.
 * ---------------------------------------------------------------------------------------------- */
typedef struct hcp_lora_job {
    const float* w_down;     /* fp32 [rank, in_dim]  (LoraLayer.LinearLayer.W_down) */
    const float* w_up;       /* fp32 [out_dim, rank] (W_up) */
    float alpha;             /* LoraBlock.alpha buffer = alpha / rank */
    int32_t rank, in_dim, out_dim;
    int32_t c0;              /* first rank column of this block inside the group's R-wide T / U buffers */
    int32_t o0;              /* first output row of this block inside the group's fused output */
    int32_t out_tot;         /* fused output width of the group */
    int32_t ld_r;            /* R: rank columns of the group padded to a multiple of 64 (row pitch of AT / Bl, of T / U) */
    void* A;                 /* bf16 [R, in_dim]   (DAPP: the buffer of this block's branch) */
    void* AT;                /* bf16 [in_dim, R] */
    void* Bl;                /* bf16 [out_tot, R] */
    void* BlT;               /* bf16 [R, out_tot]  (DAPP: the buffer of this block's branch) */
} hcp_lora_job;

int hcp_lora_pack(const hcp_lora_job* jobs_device, int64_t njobs, hcp_stream_t stream);
/* LoRA weight merge, one launch per step for every patched Linear / 1x1 Conv2d whose adapters apply to all rows (no DreamArtist++
 * branches): W_eff = bf16(W_host + sum_b alpha_b * W_up_b . W_down_b) -- LoraBlock.get_weight + LoraPatchContainer.forward +
 * LinearLayer.forward (reference lora_base_patch.py:21-35,61-62, lora_layers_patch.py:44-57), summed in fp32 and rounded once.
 * Written as W [out_tot, in_dim] rows [o0, o0+out_dim) (forward B operand) and WT [in_dim, out_tot] (dgrad B operand; may be NULL).
 * The forward and the input gradient of the layer are then plain GEMMs.  Requirements: in_dim, out_dim, o0, out_tot multiples of
 * 8; at most 4 stacked blocks whose ranks sum to <= 64.  tile0 = number of 64x64 tiles of the jobs before this one
 * (ceil(out_dim/64) * ceil(in_dim/64) each); total_tiles = their sum. */
typedef struct hcp_lora_merge_job {
    const float* w_host;     /* fp32 [out_dim, in_dim] */
    const float* w_down[4];  /* fp32 [rank_b, in_dim] */
    const float* w_up[4];    /* fp32 [out_dim, rank_b] */
    float alpha[4];
    int32_t rank[4];
    int32_t nblocks, in_dim, out_dim, o0, out_tot, tile0;
    int32_t tiled;           /* 1: W / WT are k-block-major ([in_dim/64][out_tot][64] / [out_tot/64][in_dim][64], see hcp_gemm_args.flags) */
    int32_t pad_;
    void* W;
    void* WT;
} hcp_lora_merge_job;
/* tile_job_device: optional int32 [total_tiles] table, tile index -> job index (NULL: the kernel searches the job table itself);
 * max_rank_sum: the largest sum of stacked ranks of any job (sizes the kernel's shared memory; <= 0: assume 64). */
int hcp_lora_merge(const hcp_lora_merge_job* jobs_device, int64_t njobs, int64_t total_tiles, const int32_t* tile_job_device,
                   int32_t max_rank_sum, hcp_stream_t stream);
/* Conv2d LoRA down-projection W_down fp32 [rank, Cin, 3, 3] -> the two bf16 operands the 3x3 kernels take:
 *   wt [R, 3, 3, Cin]  forward weights of T = conv3x3(x, W_down) (rows c0 .. c0+rank of the group's R-row matrix)
 *   wd [Cin, 3, 3, R]  dgrad arrangement of the same taps (flipped for stride 1, as-is for the stride-2 phase kernels)
 * (the up-projection [Cout, rank, 1, 1] goes through hcp_lora_pack with in_dim = 0). */
typedef struct hcp_lora_conv_job {
    const float* w_down;
    int32_t rank, cin, c0, ld_r, flip, pad_;
    void* wt;
    void* wd;
} hcp_lora_conv_job;
int hcp_lora_pack_conv(const hcp_lora_conv_job* jobs_device, int64_t njobs, hcp_stream_t stream);
/* Gradients of the LoRA factors on the tensor pipe: for every block b and every column n in [n_lo_b, n_hi_b) of X,
 *     D[n, j] = scale_b * sum_m X[m, n] * S[m, c0_b + j],   j < rank_b      (S bf16 [M,64] with row pitch lds >= 64: one 64-column
 *     slab of the group's T / U buffer -- wider groups call once per slab with S advanced by 64 columns; X bf16 [M,ldx])
 * is ACCUMULATED (fp32 atomics) into  dst_b[j*dst_ld + (n-n_lo)]  (transpose_out = 0: dW_down[r,in], S = dY.(alpha B), X = x)
 *                               or   dst_b[(n-n_lo)*dst_ld + j]  (transpose_out = 1: dW_up[out,r],  S = x.A^T, X = dY).
 * hcp_lora_grad and hcp_lora_grad_pair refuse, before any launch:
 *   - 0 <= n_begin < n_end <= ldx not holding (X columns past ldx would read as zeros);
 *   - a block with n_lo >= n_hi or [n_lo, n_hi) not inside [n_begin, n_end) (the columns outside would be dropped);
 *   - a block with dst_ld < rank (transpose_out = 1) or dst_ld < n_hi - n_lo (transpose_out = 0): rows would overlap. */
typedef struct hcp_lora_grad_block {
    int64_t n_lo, n_hi;
    int32_t c0, rank;
    float scale;
    int32_t transpose_out;
    float* dst;
    int64_t dst_ld;
} hcp_lora_grad_block;
int hcp_lora_grad(const void* S, int64_t lds, const void* X, int64_t ldx, int64_t M, int64_t n_begin, int64_t n_end,
                  const hcp_lora_grad_block* blocks, int32_t nblocks, hcp_stream_t stream);     /* nblocks <= 8 */
/* dW_down of a Conv2d LoRA: for every tap (kh,kw) and block b,
 *     dst_b[(j*Cin + n)*9 + kh*3 + kw] += sum_m S[m, c0_b + j] * x[pixel(m) shifted by the tap, n]
 * S = U = dY . (alpha W_up) bf16 [B*Hout*Wout, lds]; x bf16 NHWC [B,Hin,Win,Cin]; zero padding and stride as in the forward conv.
 * Nine launches of the gradient kernel whose X operand is the shifted 4-D / 5-D TMA box of the convolution.  Block fields used:
 * c0, rank, scale, dst (fp32 [rank, Cin, 3, 3]); n_lo/n_hi/transpose_out/dst_ld are ignored. */
int hcp_lora_grad_conv3x3(const void* S, int64_t lds, const void* x, int64_t B, int64_t Hin, int64_t Win, int64_t Cin, int32_t stride,
                          const hcp_lora_grad_block* blocks, int32_t nblocks, hcp_stream_t stream);
/* Both gradients of one LoRA group in a single launch: dW_down from (U [M,64], x [M,K]) and dW_up from (T [M,64], dY [M,N]). */
int hcp_lora_grad_pair(const void* U, const void* x, int64_t ldx, int64_t K, const hcp_lora_grad_block* down,
                       const void* T, const void* dy, int64_t lddy, int64_t N, const hcp_lora_grad_block* up,
                       int32_t nblocks, int64_t M, int64_t lds /* row pitch of U and T */, hcp_stream_t stream);

/* ------------------------------------------------------------------------------------------------
 * The step either side of the UNet call (reference hcpdiff/train_ac.py:437-447, 485-494, 506-515).
 * ---------------------------------------------------------------------------------------------- */
int hcp_sumsq(const float* g, int64_t n, float* out /* += */, hcp_stream_t stream);
int hcp_adamw_flat(float* p, const float* g, float* m, float* v, int64_t n, const float* lr_device, float beta1, float beta2,
                   float eps, float weight_decay, float grad_scale, const float* sumsq_device, float max_norm,
                   int* step_device, hcp_stream_t stream);
/* The same step with the hyper-parameters in device memory: hyper_device = {lr, beta1, beta2, eps, weight_decay} (fp32 [5]); an LR
 * scheduler (OneCycleLR cycles lr AND beta1) rewrites them between CUDA-graph replays.  p, g, m, v 16-byte aligned (a segment of a
 * flat buffer starts at a multiple of 4 elements).  Both AdamW calls advance *step_device once per call with n > 0; n == 0 is a
 * no-op and leaves it. */
int hcp_adamw_flat_dev(float* p, const float* g, float* m, float* v, int64_t n, const float* hyper_device, float grad_scale,
                       const float* sumsq_device, float max_norm, int* step_device, hcp_stream_t stream);
/* Lion (lion_pytorch.Lion.step) with the contract of hcp_adamw_flat_dev: the same hyper row (eps unused), gradient g * grad_scale
 * clipped with sumsq_device, *step_device advanced once per call with n > 0 (Lion itself has no bias correction; hcp_ema_flat
 * reads it), 16-byte aligned p / g / m, n == 0 a no-op, no host synchronisation.  Per element, in fp32:
 *   p = p (1 - lr wd);  c = beta1 m + (1 - beta1) g;  p = p - lr sign(c) (sign(0) = 0);  m = beta2 m + (1 - beta2) g.  One launch. */
int hcp_lion_flat_dev(float* p, const float* g, float* m, int64_t n, const float* hyper_device, float grad_scale,
                      const float* sumsq_device, float max_norm, int* step_device, hcp_stream_t stream);

/* Prodigy (prodigyopt.Prodigy.step) over segments (parameter groups) of the flat buffers p, g, p0, s, m, v (fp32, 16-byte
 * aligned; p0 / s / m / v are Prodigy's per-element state).  segs: [nsegs] in increasing, non-overlapping order inside [0, n), each
 * offset a multiple of 4; segs_host is checked before any launch, segs_device (its device copy) is what the kernels read, so a
 * scheduler rewrites `lr` there between CUDA-graph replays.  Every segment's lr must be the table's largest lr or 0 (prodigyopt
 * raises otherwise; the caller keeps that rule).
 * hyper_device fp64 [HCP_PRODIGY_HYPER] = {beta1, beta2, beta3, eps, d0, d_coef, growth_rate, flags}, flags = 1 use_bias_correction
 * | 2 safeguard_warmup | 4 decouple (beta1 may be rewritten between replays: OneCycleLR).  state_device fp64 [HCP_PRODIGY_STATE] =
 * {d, d_max, D_num, k, initialised, skipped, dlr, unused}, set to {d0, d0, 0, 0, 0, 0, 0, 0} before the first call.  Per call, with
 * g' = g * grad_scale clipped to max_norm with the device-side sumsq (as hcp_adamw_flat_dev), lr = the largest segment lr and
 * dlr = d lr (use_bias_correction ? sqrt(1 - beta2^(k+1)) / (1 - beta1^(k+1)) : 1):
 *   coupled decay (decouple == 0): g' += wd p.  First call: p0 = p, s = m = v = 0 (every segment).
 *   segments with lr > 0: D_num' = beta3 D_num + (d / d0) dlr sum g' (p0 - p);  m = beta1 m + d (1 - beta1) g';
 *     v = beta2 v + d^2 (1 - beta2) g'^2;  s = beta3 s + (d / d0) (safeguard_warmup ? d : dlr) g';  D_den = sum |s|.
 *   D_den == 0: nothing else changes (p, d, d_max, D_num, k stay; "skipped" is set).  Otherwise, when lr > 0:
 *     d_hat = d_coef D_num' / D_den;  d = max(d, d_hat) if d == d0;  d_max = max(d_max, d_hat);  d = min(d_max, d growth_rate);
 *     then every segment: p = p - wd dlr p (decouple), p = p - dlr m / (sqrt(v) + d eps) (old dlr, new d);  k += 1.
 * *step_device (hcp_ema_flat's counter) is advanced on every call, skipped or not.  The sums are fp64 partials per CTA in
 * `workspace` (at least HCP_PRODIGY_WORKSPACE_BYTES, 8-byte aligned), added in a fixed order: replays are bit-identical.  An
 * empty table is a no-op.  Three launches; no host synchronisation (CUDA-graph capturable). */
typedef struct {
    int64_t offset;
    int64_t count;
    double lr;
    double weight_decay;
} hcp_prodigy_segment;
#define HCP_PRODIGY_HYPER 8
#define HCP_PRODIGY_STATE 8
#define HCP_PRODIGY_WORKSPACE_BYTES 16384
int hcp_prodigy_flat(float* p, const float* g, float* p0, float* s, float* m, float* v, int64_t n, const hcp_prodigy_segment* segs_host,
                     const hcp_prodigy_segment* segs_device, int32_t nsegs, const double* hyper_device, double* state_device,
                     double* workspace, size_t workspace_bytes, float grad_scale, const float* sumsq_device, float max_norm,
                     int* step_device, hcp_stream_t stream);

/* AdamW8bit (bitsandbytes.optim.AdamW8bit: blockwise 8-bit Adam moments) over the tensors of a table.  A tensor in mode 1 keeps
 * its first and second moments as uint8 codes, code1 at codes + state and code2 at codes + code_bytes + state (numel each), with one
 * fp32 scale per 256-element block counted from the tensor's first element: absmax1 at absmax + absmax_row, absmax2 at absmax +
 * nblocks + absmax_row.  Codes decode through maps_device (fp32 [2, 256]: bitsandbytes' signed dynamic map for the first moment,
 * the unsigned one for the second).  A tensor in mode 0 keeps fp32 m at state32 + state and v at state32 + small_numel + state. */
typedef struct {
    int64_t offset;     /* first element in p and g (a multiple of 4) */
    int64_t numel;
    int64_t state;      /* mode 1: first code (a multiple of 4); mode 0: first element of m / v (a multiple of 4) */
    int64_t absmax;     /* mode 1: first block scale; mode 0: unused */
    int32_t mode;       /* 1: 8-bit blockwise, 0: 32-bit */
    int32_t group;
} hcp_adamw8bit_tensor;
/* Blocks [block0, block1) of one tensor, walked by one CTA.  The items tile every tensor's blocks once, in table order. */
typedef struct {
    int32_t tensor, block0, block1, pad;
} hcp_adamw8bit_item;
/* The contract of hcp_adamw_flat_dev per group: hyper_device fp32 [ngroups, 5] = {lr, beta1, beta2, eps, weight_decay} rows,
 * steps_device int32 [ngroups] each advanced once per call (the bias corrections read it; hcp_ema_flat reads group 0's), the gradient
 * g * grad_scale clipped to max_norm with the device-side sumsq.  Per element, in fp32 (each operation rounded on its own):
 *   s1 = b1 s1 + (1 - b1) g;  s2 = b2 s2 + (1 - b2) g^2;  p += -lr sqrt(1 - b2^t) / (1 - b1^t) s1 / (sqrt(s2) + eps sqrt(1 - b2^t));
 *   then, when weight_decay > 0, p *= 1 - lr weight_decay (after the step, as bitsandbytes).
 * Mode 1: a non-finite g sets both moments to 0 and leaves p; each block's new scale is max |s| over the block after the update,
 * and s / scale (0 when the scale is 0) is re-encoded with bitsandbytes' search and midpoint rule; a first-moment code of the other
 * sign than s1 moves one step toward it.  Mode 0 (bitsandbytes' 32-bit path) has no non-finite guard.  tensors_host / items_host
 * are checked before any launch (inside the buffers, aligned, increasing, the items tiling each tensor once); tensors_device /
 * items_device are their device copies, which the kernel reads.  p, g, state32 and codes 16-byte aligned, code_bytes a multiple of
 * 16, small_numel of 4.  An empty table is a no-op.  Two launches; no host synchronisation (CUDA-graph capturable). */
int hcp_adamw8bit_flat(float* p, const float* g, uint8_t* codes, float* absmax, float* state32, const float* maps_device,
                       const hcp_adamw8bit_tensor* tensors_host, const hcp_adamw8bit_tensor* tensors_device, int32_t ntensors,
                       const hcp_adamw8bit_item* items_host, const hcp_adamw8bit_item* items_device, int64_t nitems, int64_t n,
                       int64_t code_bytes, int64_t nblocks, int64_t small_numel, const float* hyper_device, int* steps_device,
                       int32_t ngroups, float grad_scale, const float* sumsq_device, float max_norm, hcp_stream_t stream);

/* Adafactor (transformers.optimization.Adafactor.step) over the flat buffer, per tensor of the module's shape.  A tensor with two or
 * more dims is factored over its last two: view [P, R, C], exp_avg_sq_row [P, R] at state+row, exp_avg_sq_col [P, C] at state+col.
 * A 1-D tensor has exp_avg_sq [numel] at state+row, and is walked as P = 1, R = ceil(numel / 256), C = 256. */
typedef struct {
    int64_t offset;     /* first element in p, g and exp_avg */
    int64_t numel;
    int64_t P, R, C;
    int64_t row, col;   /* state offsets (col = -1 when not factored) */
    int64_t rowpart;    /* work offset of the partial row sums [P*R, nct] (used when nct > 1) */
    int64_t colpart;    /* work offset of the partial column sums [nrch, P*C] (used when nrch > 1) */
    int64_t rmean;      /* work offset of mean_R(exp_avg_sq_row) [P] (factored) */
    int32_t factored, group;
    int32_t nct, nrch;  /* column tiles of 256 (wide rows) and row chunks of 256 of the tensor's items */
    int32_t item0, nitems;  /* the tensor's range in the item list */
} hcp_adafactor_tensor;
/* One CTA of 256 threads: slabs [p0, p1), columns [c0, c1) (c1 - c0 <= 256; columns of 256 / (c1 - c0) slabs side by side), rows
 * [r0, r1) (at most 256, starting at a multiple of 256; wide column tiles start at a multiple of 256).  Factor items (pass b): mode 0
 * one CTA for slab p0, mode 1 one thread per slab of [p0, p1). */
typedef struct {
    int32_t tensor, p0, p1, c0, c1, r0, r1, mode;
} hcp_adafactor_item;
/* hyper_device: fp32 [ngroups, 8] = {lr, eps1, eps2, clip_threshold, decay_rate, beta1, weight_decay, flags} with flags = 1
 * scale_parameter | 2 relative_step | 4 warmup_init | 8 beta1 set; steps_device int32 [ngroups] (incremented here).  work: fp32,
 * [2 * nitems] tile partial sums followed by the per-tensor scratch the table points at.  exp_avg (flat, like p) may be NULL when
 * no group sets beta1.  The gradient is g * grad_scale, clipped to max_norm with the device-side sumsq (as hcp_adamw_flat_dev).
 * Five launches whatever the tensor count; no host synchronisation (CUDA-graph capturable). */
int hcp_adafactor_flat(float* p, const float* g, float* state, float* exp_avg, float* work, const hcp_adafactor_tensor* tensors_device,
                       const hcp_adafactor_item* items_device, int64_t nitems, const hcp_adafactor_item* factor_items_device,
                       int64_t nfactor_items, const float* hyper_device, int* steps_device, int32_t ngroups, float grad_scale,
                       const float* sumsq_device, float max_norm, hcp_stream_t stream);

/* The eps loss over the data groups of one step (reference train_ac.py:467-482, get_loss :506-515 with its per-pixel mask):
 *   group_loss[g] += sum_{b: sample_group[b] == g} sample_scale[b] * sum_{c,p} w(t_b) mask[b,p] (pred - target)^2
 *   dpred = 2 w(t_b) mask[b,p] (pred - target) sample_scale[b] grad_scale
 * pred / target / dpred fp32 [B, C, HW]; mask fp32 [B, HW] broadcast over channels (NULL = ones); sample_scale fp32 [B] =
 * loss_weight_g / (B_g C HW) (mean over all elements, not over the mask); sample_group int32 [B] in [0, ngroups); mode -1 plain
 * MSE, w = 1 (t / alphas_cumprod unused, may be NULL); modes 0..3 the SNR weights of reference hcpdiff/loss/min_snr_loss.py:5-52,
 * snr = acp/(1-acp): 0 MinSNRLoss w = min(gamma/snr, 1), 1 SoftMinSNRLoss, 2 KDiffMinSNRLoss, 3 EDMLoss (t int64 [B]).  All
 * tables are in device memory (CUDA-graph capturable).  workspace: hcp_eps_loss_grouped_workspace_bytes(B, C * HW) bytes of block partials, summed per group in a fixed
 * order by a second launch, so repeated calls give bit-identical losses. */
size_t hcp_eps_loss_grouped_workspace_bytes(int64_t B, int64_t per_image);
int hcp_eps_loss_grouped(const float* pred, const float* target, const int64_t* t, const float* alphas_cumprod, const float* mask,
                         const float* sample_scale, const int32_t* sample_group, int32_t ngroups, int32_t mode, float gamma, int64_t B,
                         int64_t C, int64_t HW, float grad_scale, float* group_loss /* fp32 [ngroups], += */, float* dpred /* may be NULL */,
                         void* workspace, size_t workspace_bytes, hcp_stream_t stream);
/* ModelEMA.update on a flat fp32 buffer (reference hcpdiff/utils/ema.py:18-27): decay = clip(1 - (1 + step/inv_gamma)^-power, 0,
 * decay_max), ema = lerp(ema, p, 1 - decay); `step_device` is the optimizer's device-side step counter (already incremented). */
int hcp_ema_flat(float* ema, const float* p, int64_t n, const int* step_device, float decay_max, float inv_gamma, float power,
                 hcp_stream_t stream);
/* nn.Dropout on a patched layer's output (reference hcpdiff/models/lora_base_patch.py:74), optionally followed by the residual
 * add the GEMM epilogue would otherwise fuse: out[r, c] = keep * x[r, c] / (1 - p) (+ residual[r, c]), c < ncols (% 8 == 0),
 * row pitches ldx / ldr / ldo in elements.  keep = f(state_device[0] seed, state_device[1] draw, site, r, c) (Philox4x32-10):
 * the backward pass calls the same function on the gradient with the same (state, site); hcp_counter_add_u64 on
 * &state_device[1] once per step makes CUDA-graph replays draw fresh masks. */
int hcp_dropout_bf16(const void* x, int64_t ldx, const void* residual /* may be NULL */, int64_t ldr,
                     const float* rowbias /* fp32 [rows / rows_per_group, rowbias_ld], may be NULL: added after the dropout */,
                     int64_t rowbias_ld, int64_t rows_per_group, int64_t rows, int64_t ncols, float p, const uint64_t* state_device,
                     uint32_t site, void* out, int64_t ldo, hcp_stream_t stream);
int hcp_counter_add_u64(uint64_t* counter_device, uint64_t inc, hcp_stream_t stream);
/* DreamArtistPTContext.post (reference hcpdiff/models/cfg_context.py:23-39) on fp32 NCHW predictions of the doubled batch
 * eps2 = [uncond (B) | cond (B)]: out[b] = e_u + s(t_b) (e_c - e_u), s = (hi - lo) rate(t_b) + lo, rate = t/(T-1) shaped by
 * mode (0 'ln', 1 'cos', 2 'cos2'); lo == hi: constant scale.  Forward: eps2 given, dout NULL, out [B*per_image].
 * Backward: dout given (eps2 ignored), out = d eps2 [2*B*per_image] = [(1-s) dout | s dout]. */
int hcp_cfg_mix_f32(const float* eps2, const float* dout, const int64_t* t, int64_t B, int64_t per_image, float scale_lo,
                    float scale_hi, int32_t mode, int32_t num_train_timesteps, float* out, hcp_stream_t stream);

/* Pyramid (multi-resolution) noise: PyramidNoiseScheduler(base, level, discount, step_size, 'bilinear').add_noise (reference
 * hcpdiff/noise/pyramid_noise.py:17-32), called once per data group and micro-step by Trainer.make_noise (hcpdiff/train_ac.py:437-447).
 * Three calls, all CUDA-graph capturable (no host synchronisation, no allocation); bad pointers and sizes are refused before any
 * launch.  Random numbers come from Philox4x32-10 on state_device = {seed, draw} (uint64 [2], its own state, not the dropout one):
 * the caller advances `draw` once per micro-step with hcp_counter_add_u64, and the data group g is the Philox site.
 *
 * Plan: plan int32 [ngroups, HCP_PYRAMID_PLAN_INTS], row g = {n, 0, hn_1, wn_1, .., hn_n, wn_n, 0 ..}: for i = 1 .. level-1,
 * r_i = 2 U + step_size (U a 53-bit double), hn_i, wn_i = max(1, int(H / r_i^i)), max(1, int(W / r_i^i)) in float64, stopping after
 * the first level with hn_i == 1 or wn_i == 1 (pyramid_noise.py:26-31).  A caller may write its own plan instead; the sum clamps
 * n to the level count and each size to [1, the size at r = step_size], the largest grid the workspace holds. */
#define HCP_PYRAMID_MAX_LEVEL 16
#define HCP_PYRAMID_MAX_GROUPS 64
#define HCP_PYRAMID_PLAN_INTS 32
int hcp_pyramid_plan(const uint64_t* state_device, int32_t ngroups, int32_t level /* 1 .. HCP_PYRAMID_MAX_LEVEL */,
                     double step_size /* >= 1 */, int64_t H, int64_t W, int32_t* plan, hcp_stream_t stream);
/* Sum: target = noise + sum_i bilinear(N(0,1) [b_g, C, hn_i, wn_i] -> [H, W]) * fp32(discount^i), per element in fp32 in level
 * order (F.interpolate, align_corners=False), and inv_std[g] = 1 / std(target over group g), unbiased, from fp64 partials summed in
 * a fixed order (replays are bit-identical).  target is the reference's loss target: its `noise +=` runs in place on make_noise's
 * tensor, and only the x_t input sees the normalised noise.  target may alias noise.  group_start int32 [ngroups + 1] (device):
 * group g is batch rows [group_start[g], group_start[g+1]), 0 = group_start[0] < .. < group_start[ngroups] = B.  Grid values of
 * level i: counter (q, i, g, draw_lo), key (seed_lo, seed_hi ^ draw_hi), Box-Muller in float64 on words (0, 1) and (2, 3) for
 * elements 4q .. 4q+3 of the group's grid.  Each level grid is generated once into the workspace.  B == 0 is a no-op. */
size_t hcp_pyramid_workspace_bytes(int64_t B, int64_t C, int64_t H, int64_t W, int32_t level, double step_size);
int hcp_pyramid_noise(const float* noise, const int32_t* plan, const int32_t* group_start, int32_t ngroups, const uint64_t* state_device,
                      int32_t level, double discount, double step_size, int64_t B, int64_t C, int64_t H, int64_t W, float* target,
                      float* inv_std /* fp32 [ngroups] */, void* workspace, size_t workspace_bytes, hcp_stream_t stream);
/* x_t = sqrt(acp[t]) x0 + sqrt(1 - acp[t]) (noise * inv_std[g(b)])  (the base scheduler's DDPMScheduler.add_noise on the normalised
 * pyramid noise, pyramid_noise.py:32), g(b) from group_start as above.  With inv_std = 1 it is DDPMScheduler.add_noise (reference
 * make_noise, train_ac.py:437-447), bit for bit. */
int hcp_add_noise_scaled(const float* x0, const float* noise, const int64_t* t, const float* alphas_cumprod, const float* inv_std,
                         const int32_t* group_start, int32_t ngroups, int64_t B, int64_t per_image, float* xt, hcp_stream_t stream);

/* ------------------------------------------------------------------------------------------------
 * Full fine-tune (reference `unet:` config items, hcpdiff/utils/cfg_net_tools.py:96-106; cfgs/train/examples/DreamBooth.yaml:6-10):
 * gradients of the base model's own parameters and the per-step repack of the trained fp32 masters.  Every gradient is ACCUMULATED
 * (fp32, atomics / read-modify-write) into caller-owned buffers -- the flat gradient buffer of the engine -- so that
 * gradient accumulation over micro-batches needs nothing extra.
 * ---------------------------------------------------------------------------------------------- */
/* dst[j * ld_j + n * ld_n] += scale * sum_m S[m, j] X[m, n],  j < j_cols, n < n_cols   (wgmma TN GEMM; S, X bf16 row-major [M, *])
 * nn.Linear weight gradient dW[out, in] = dY^T x:  S = dY (lds = N), X = x (ldx = K), ld_j = K, ld_n = 1. */
int hcp_wgrad_bf16(const void* S, int64_t lds, int64_t j_cols, const void* X, int64_t ldx, int64_t n_cols, int64_t M, float scale,
                   float* dst, int64_t ld_j, int64_t ld_n, hcp_stream_t stream);
/* nn.Conv2d(3x3, pad 1, stride 1|2) weight gradient dw[Cout, Cin, 3, 3] += scale * dY^T x_shifted(tap); dy bf16 [B*Hout*Wout, Cout],
 * x bf16 NHWC [B, Hin, Win, Cin] (Cin % 64 == 0).  Nine launches (one per tap) with the shifted TMA box of the forward kernel. */
int hcp_wgrad_conv3x3_bf16(const void* dy, int64_t Cout, const void* x, int64_t B, int64_t Hin, int64_t Win, int64_t Cin, int32_t stride,
                           float scale, float* dw, hcp_stream_t stream);
/* out[r / rows_per_group, c] += scale * x[r, c]  (x bf16 [M, ld]; bias gradients: one group; per-image time-embedding gradient of a
 * ResnetBlock2D: rows_per_group = H*W).  rows_per_group <= 0 means M. */
int hcp_colsum_bf16(const void* x, int64_t ld, int64_t M, int64_t N, int64_t rows_per_group, float scale, float* out, int64_t ldo,
                    hcp_stream_t stream);
/* GroupNorm (groups > 0: stats fp32 [B, groups, 2] = (mean, rstd), rows_per_image = H*W) / LayerNorm (groups == 0: stats [rows, 2])
 * affine gradients: dgamma[c] += sum dz xhat, dbeta[c] += sum dz with dz = dy or dy * silu'(gamma xhat + beta) (silu != 0: the fused
 * GroupNorm+SiLU of ResnetBlock2D).  The input is the channel concatenation [x1 | x2] (x2 may be NULL, C2 = 0). */
int hcp_norm_affine_grad_bf16(const void* x1, const void* x2, int64_t C1, int64_t C2, const void* dy, const float* stats,
                              const float* gamma, const float* beta, int64_t rows, int64_t rows_per_image, int64_t groups, int32_t silu,
                              float* dgamma, float* dbeta, hcp_stream_t stream);
/* Backward of the small fp32 linears of the time-embedding path (y = x W^T + b, M = batch rows): dx[M,K] = dy W (W bf16 [N,K], the
 * operand the forward used; dx may be NULL), dw[N,K] += dy^T x, db[N] += colsum(dy) (fp32 masters; dw / db may be NULL).
 * dy fp32 [M, N] with row pitch ldy (a column slice of a wider matrix: the 22 time_emb_proj layers share one input). */
int hcp_small_linear_bwd_f32(const float* dy, int64_t ldy, const float* x, const void* w_bf16, int64_t M, int64_t N, int64_t K, float* dx,
                             float* dw, float* db, hcp_stream_t stream);
/* out = silu(x) (dy NULL) or dy * silu'(x), fp32 vectors */
int hcp_silu_f32(const float* x, const float* dy, int64_t n, float* out, hcp_stream_t stream);
/* Weight / bias gradients of the 4-channel boundary convolutions in the nn.Conv2d layout [Cout, Cin, 3, 3] (fp32, accumulated):
 * conv_in: dh bf16 NHWC [B,H,W,Cout] (gradient of its output), x fp32 NCHW latent; conv_out: dy fp32 NCHW [B,Cout,H,W], x bf16 NHWC. */
int hcp_conv_in_wgrad_f32(const void* dh_nhwc_bf16, const float* x_nchw, int64_t B, int64_t Cin, int64_t H, int64_t W, int64_t Cout,
                          float* dw, float* db /* may be NULL */, hcp_stream_t stream);
int hcp_conv_out_wgrad_f32(const float* dy_nchw, const void* x_nhwc_bf16, int64_t B, int64_t H, int64_t W, int64_t Cin, int64_t Cout,
                           float* dw, float* db /* may be NULL */, hcp_stream_t stream);
/* Per-step repack of trained fp32 master weights into the bf16 operand layouts (one launch for every trained layer):
 *   kind 0  W [rows, K] -> dst0 bf16 rows [o0, o0+rows) of [*, K]  and  dst1 bf16 [K, n_tot] columns [o0, o0+rows)   (linear, 1x1 conv)
 *   kind 1  W [rows = Cout, K = Cin, 3, 3] -> dst0 [Cout, 3, 3, Cin]  and  dst1 [Cin, 3, 3, Cout] (taps flipped when flip != 0)
 *   kind 2  fp32 vector of `rows` elements (K = 1) -> dst0 fp32 at element offset o0
 *   kind 3  W [rows, K] -> dst0 bf16 rows [o0, o0+rows) of [*, K] */
typedef struct hcp_repack_job {
    const float* src;
    void* dst0;
    void* dst1;
    int32_t kind, rows, K, o0, n_tot, flip;
} hcp_repack_job;
int hcp_repack_weights(const hcp_repack_job* jobs_device, int64_t njobs, hcp_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* HCP_B200_H_ */
