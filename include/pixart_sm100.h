/* pixart_sm100.h -- C ABI of libpixart_sm100.so: hand-written sm_90a (H100) kernels for the
 * PixArt-Sigma DiT denoiser hot path  PixArtMS.forward -> 28 x PixArtMSBlock.forward.
 *
 * The reference (PixArt-alpha/PixArt-sigma) is pure Python and has NO FFI / plugin interface; its GPU math is
 * reached through library calls (torch nn.Linear / LayerNorm / GELU, xformers memory_efficient_attention).
 * Each entry point below replaces one such call site (file:line relative to the reference root) and is what a
 * ctypes binding inside diffusion/model/nets/PixArt_blocks.py would bind (see INTEGRATION.md).
 *
 * Contract (all entry points):
 *   - plain pointers and sizes only; every buffer (inputs, outputs, workspace) is owned by the caller and is
 *     DEVICE memory; the library never allocates, frees or synchronises and launches only on `stream`
 *     (a cudaStream_t passed as void*), so calls are CUDA-graph capturable;
 *   - returns 0 on success, a negative PXA_ERR_* otherwise; pxa_last_error() gives the message (thread local);
 *   - bf16 operands, fp32 accumulation / statistics / softmax; pointers must be 16-byte aligned;
 *   - requires an sm_90 device (PXA_ERR_ARCH otherwise). There is no CPU or non-Hopper path.
 */
#ifndef PIXART_SM100_H_
#define PIXART_SM100_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define PXA_OK 0
#define PXA_ERR_ARG (-1)     /* bad shape / null pointer / unsupported option */
#define PXA_ERR_ALIGN (-2)   /* pointer or stride not 16-byte aligned */
#define PXA_ERR_ARCH (-3)    /* device is not sm_90 */
#define PXA_ERR_CUDA (-4)    /* CUDA runtime / driver error (launch, tensor-map encode) */

#define PXA_DTYPE_BF16 0
#define PXA_DTYPE_F32 1
#define PXA_DTYPE_F16 2      /* accepted only where an entry point says so (pxa_iddpm_step) */

int pxa_version(void);
const char* pxa_last_error(void);
/* Number of kernel launches issued by this library since load (all streams) -- bench.py's `gpu_launches`. */
uint64_t pxa_launch_count(void);

/* ------------------------------------------------------------------------------------------------- GEMM
 * out = epilogue( A[M,K] . W[N,K]^T + bias[N] ),  A/W bf16 K-contiguous (W is the nn.Linear weight as stored).
 * wgmma (m64 x BN/2 x 16 per consumer warpgroup, fp32 accumulators in registers), TMA-fed smem ring, persistent, warp-specialised.
 *
 * Replaces: attn.qkv PixArt_blocks.py:130 | attn.proj + gate + residual PixArt_blocks.py:155, PixArtMS.py:75 |
 *   cross_attn.q_linear / kv_linear / proj (+residual) PixArt_blocks.py:47,48,55, PixArtMS.py:76 |
 *   mlp.fc1 + GELU(tanh) / fc2 + gate + residual (timm Mlp; PixArtMS.py:67,77) | y_embedder.y_proj PixArt_blocks.py:406.
 */
#define PXA_EPI_BIAS 0          /* out = acc + bias                                   */
#define PXA_EPI_BIAS_GELU 1     /* out = gelu_tanh(acc + bias)                        */
#define PXA_EPI_BIAS_RESIDUAL 2 /* out = residual + gate[row/rows_per_batch, n] * (acc + bias); gate NULL -> 1 */
/* Training fusions of the MLP (timm Mlp, PixArtMS.py:67,77), used by the block backward of pixart_sigma_b200.autograd. */
#define PXA_EPI_BIAS_GELU_AUX 3 /* out = gelu_tanh(acc + bias), out_aux_bf16 = acc + bias (pre-activation kept for the backward) */
#define PXA_EPI_MUL_DGELU 4     /* out = acc * gelu_tanh'(pre), pre = `residual` as bf16 [M, N] row stride ldo; bias must be NULL  */
/* adaLN-single modulate FUSED into the projection that follows it (norm1 + t2i_modulate + attn.qkv, PixArtMS.py:75 with
 * PixArt_blocks.py:24-25,130; norm2 + t2i_modulate + mlp.fc1, PixArtMS.py:77): the LayerNorm'ed, modulated activations
 * are never materialised.  With mu_r / rstd_r the LayerNorm statistics of row r of the fp32 residual stream x and
 * (shift_b, scale_b) the modulation of its sample b,
 *     sum_k [ (x[r,k] - mu_r) rstd_r (1 + scale_b[k]) + shift_b[k] ] W[n,k] + bias[n]
 *   = rstd_r * ( acc[r,n] - mu_r * u_b[n] ) + v_b[n],     acc = A W^T,  A[r,k] = bf16( x[r,k] (1 + scale_b[k]) ),
 *     u_b[n] = sum_k (1 + scale_b[k]) W[n,k],   v_b[n] = sum_k shift_b[k] W[n,k] + bias[n].
 * A and the per-row statistics are by-products of the residual epilogue that produced x (`aux_scale`, `row_stats_out`
 * below) or of pxa_ln_prepare; u_b / v_b are two tiny per-sample GEMVs per forward.
 * Accuracy trade-off: A is rounded to bf16 relative to |x|, not to the normalised x - mu, and the row variance comes from
 * one-pass fp32 sums.  The error against the unfused LayerNorm therefore grows like 1 + |mu_r| rstd_r (about
 * 2^-9 rstd sum_k |x_k (1 + scale_k) W[n,k]| at worst, tests/test_numerics_gpu.py); the unfused pxa_ln_modulate path
 * (two-pass statistics, the default) has no such dependence on the mean. */
#define PXA_EPI_LN_BIAS 5       /* out = rstd*(acc - mu*u) + v            (`ln_*` fields; bias must be NULL: it is inside v) */
#define PXA_EPI_LN_BIAS_GELU 6  /* out = gelu_tanh(rstd*(acc - mu*u) + v)                                                   */
#define PXA_LN_STAT_PARTS 8     /* row statistics are kept as 8 partial (sum x, sum x^2) pairs per row: fp32 [M][8][2]      */

/* The structure keeps the layout it had when the library offered several kernel forms per call.  On sm_90 there is one GEMM
 * kernel (128 x BN tiles on one CTA), so `cta_pair`, `res_epilogue`, `epi_warps` and `debug_trace` are validated where noted and
 * otherwise ignored. */
typedef struct PxaGemmArgs {
  const void* a;        /* bf16 [M, K], row stride lda (elements)                                   */
  const void* w;        /* bf16 [N, K], row stride ldw (elements)                                   */
  const void* bias;     /* bf16 [N] or NULL                                                         */
  void* out;            /* [M, N], row stride ldo (elements), dtype out_dtype                       */
  void* out_aux_bf16;   /* optional second bf16 copy of out (row stride ldo) or NULL                */
  const void* residual; /* EPI_BIAS_RESIDUAL: [M, N] row stride ldo, dtype out_dtype (may alias out)*/
  const float* gate;    /* EPI_BIAS_RESIDUAL: fp32, element (b, n) at gate[b*gate_batch_stride + n], or NULL */
  int64_t gate_batch_stride;
  int32_t rows_per_batch; /* rows of A per sample (tokens N); row r belongs to sample r / rows_per_batch */
  int32_t M, N, K;
  int32_t lda, ldw, ldo;
  int32_t epilogue;     /* PXA_EPI_*            */
  int32_t out_dtype;    /* PXA_DTYPE_*          */
  int32_t block_n;      /* 0 = auto (192 when it divides N, else 128); or 128 / 192 / 256 (fp32 out: 256 runs as 128) */
  int32_t max_ctas;     /* 0 = one CTA per SM; >0 caps the persistent grid (tests)                  */
  int32_t cta_pair;     /* (ignored, see above; must be 0, 1 or 2) */
  int64_t* debug_trace; /* (ignored) */
  int32_t operands_mn_major; /* 1: weight-gradient form out[M, N] += A^T . W with a = [K, M] (row stride lda) and
                                w = [K, N] (row stride ldw), i.e. the contraction runs over the ROWS of both operands
                                (dW = dY^T X straight from the activations' natural layouts; no transposes).  Requires
                                EPI_BIAS_RESIDUAL, fp32 out, residual == out (in-place accumulate), no bias / gate / aux. */
  int32_t k_splits;     /* operands_mn_major only: 0 = auto (fill the 132 SMs), else the number of K splits        */
  int32_t aux_is_branch; /* EPI_BIAS_RESIDUAL with out_aux_bf16: 1 = the aux output receives acc + bias (the un-gated
                            branch output, which the backward of the gate needs) instead of a bf16 copy of out          */
  /* --- producer side of the fused LayerNorm-modulate (EPI_BIAS_RESIDUAL, fp32 out, out_aux_bf16 set) */
  const float* aux_scale;   /* fp32 or NULL: the bf16 aux copy becomes out[r,n] * aux_scale[b*aux_scale_batch_stride + n]
                               (pass 1 + scale of the NEXT modulate: the aux output is then the A operand above)          */
  int64_t aux_scale_batch_stride;
  float* row_stats_out;     /* fp32 [M][PXA_LN_STAT_PARTS][2] or NULL: partial (sum, sum of squares) of each row of `out`
                               over the columns of one output tile, part = the tile's column index; unused parts zeroed     */
  /* --- consumer side (EPI_LN_BIAS / EPI_LN_BIAS_GELU) */
  const float* ln_stats;    /* fp32 [M][PXA_LN_STAT_PARTS][2] partial sums of the rows of x (row_stats_out / pxa_ln_prepare) */
  const float* ln_u;        /* fp32, u_b[n] at ln_u[b*ln_uv_batch_stride + n]                                                */
  const float* ln_v;        /* fp32, v_b[n] at ln_v[b*ln_uv_batch_stride + n]                                                */
  int64_t ln_uv_batch_stride;
  int32_t ln_dim;           /* row length C of x the statistics were taken over                                              */
  float ln_eps;
  int32_t res_epilogue;     /* (ignored; must be 0, 1 or 2) */
  int32_t epi_warps;        /* (ignored) */
  int32_t reverse_tiles;    /* 1: visit the output tiles from the LAST row block to the first.  A GEMM whose A operand was
                               written front to back by the previous kernel (mlp.fc2 after mlp.fc1) then starts on the rows
                               that are still in the 50 MB L2 instead of the ones already evicted to HBM                   */
} PxaGemmArgs;
int pxa_gemm_bf16(const PxaGemmArgs* args, void* stream);

/* ------------------------------------------------------------------------------------------- GEMM with a K-tail (LoRA)
 * out = epilogue( A W^T + tail_a tail_w^T + bias ): the same kernel as pxa_gemm_bf16 with ceil(tail_k / 64) more K-blocks,
 * read from tail_a [M, tail_k] and tail_w [N, tail_k] (bf16, K-contiguous) into the same operand ring after the last
 * K-block of A W^T, so that the epilogue sees the sum.  Columns past tail_k are TMA zero fill.  For a LoRA projection
 * tail_a = u = x A^T and tail_w = s B (block-diagonal over fused projections): the adapter's up-projection lands in the
 * accumulator before the bias / GELU / gated-residual epilogue.  In the backward, tail_a = v = s dY B and tail_w = A^T.
 * Accepts every PxaGemmArgs form except the fused LayerNorm epilogues (EPI_LN_*) and operands_mn_major
 * (PXA_ERR_ARG); the convolution (pxa_conv3x3_nhwc_bf16) has no tail.  tail_k must be a multiple of 8 (PXA_ERR_ARG);
 * tail_a / tail_w 16-byte aligned and lda_tail / ldw_tail multiples of 8 (PXA_ERR_ALIGN).  With a tail, block_n 256 runs at
 * 192 and fp32 output at 128 (the wider tail instantiations would spill registers). */
typedef struct PxaGemmTail {
  const void* tail_a;   /* bf16 [M, tail_k], row stride lda_tail (elements) */
  const void* tail_w;   /* bf16 [N, tail_k], row stride ldw_tail (elements) */
  int32_t tail_k;
  int32_t lda_tail, ldw_tail;
} PxaGemmTail;
int pxa_gemm_lora_bf16(const PxaGemmArgs* args, const PxaGemmTail* tail, void* stream);

/* ------------------------------------------------------------------------------------------- fused Mlp
 * x32[r, :] += gate[b, :] * ( gelu_tanh(x[r, :] W1^T + b1) W2^T + b2 )        b = r / rows_per_batch
 * The timm Mlp of PixArtMSBlock with its gate and residual (PixArtMS.py:67,77), run in groups of `group` 256-row panels: per group
 * one fc1 + GELU launch and one fc2 + gate + residual launch of the GEMM kernel, back to back on the stream, so that the group's
 * [rows, N1] hidden activations sit in a slot of a small ring (hidden_ws) that lives in L2 instead of streaming through HBM
 * (mlp_sm90.cu; 2 * ceil(M / (256 group)) launches, not one kernel).  x = the normalised, modulated bf16 activations
 * (pxa_ln_modulate output); x32 = the fp32 residual stream, updated in place.
 */
typedef struct PxaMlpArgs {
  const void* x;         /* bf16 [M, K1], row stride ldx                                   */
  const void* w1;        /* bf16 [N1, K1] (mlp.fc1.weight), row stride ldw1                 */
  const void* b1;        /* bf16 [N1] or NULL                                              */
  const void* w2;        /* bf16 [N2, N1] (mlp.fc2.weight), row stride ldw2                 */
  const void* b2;        /* bf16 [N2] or NULL                                              */
  float* x32;            /* fp32 [M, N2], row stride ldo: residual stream, updated in place */
  const float* gate;     /* fp32 (b, n) at gate[b*gate_batch_stride + n], or NULL           */
  int64_t gate_batch_stride;
  void* hidden_ws;       /* bf16 scratch, >= ring * group * 256 * N1 elements               */
  int64_t hidden_ws_bytes;
  void* flags_ws;        /* unused (may be NULL); kept for binary compatibility                                   */
  int64_t flags_ws_bytes;
  int32_t rows_per_batch;
  int32_t M, K1, N1, N2; /* N1 % 256 == 0, N2 % 192 == 0                                   */
  int32_t ldx, ldw1, ldw2, ldo;
  int32_t group;         /* 256-row panels per group (0 = 4)                               */
  int32_t ring;          /* groups held by hidden_ws (0 = 2): group g uses slot g % ring   */
  int32_t max_ctas;      /* 0 = one CTA per SM; > 0 caps the persistent grid (tests)       */
  int32_t lag;           /* unused */
  int32_t k_splits;      /* unused */
} PxaMlpArgs;
int pxa_mlp_fused_bf16(const PxaMlpArgs* args, void* stream);

/* ------------------------------------------------------------------------------------ LayerNorm + modulate
 * out[r,:] = LN(x[r,:]; eps, no affine) * (1 + scale[b,:]) + shift[b,:]  with b = r / rows_per_batch, bf16 out.
 * Replaces norm1/norm2 + t2i_modulate (PixArtMS.py:58,64,75,77; PixArt_blocks.py:24-25) and the final-layer
 * modulate (PixArt_blocks.py:218-219).  HBM-bound: reads x once, writes out once.
 */
typedef struct PxaLnModArgs {
  const void* x;        /* [M, C] row stride ldx, dtype x_dtype */
  void* out;            /* bf16 [M, C] contiguous                */
  const float* shift;   /* fp32, (b, c) at shift[b*mod_batch_stride + c] */
  const float* scale;   /* fp32, same addressing                  */
  int64_t mod_batch_stride;
  int32_t rows_per_batch;
  int32_t M, C, ldx;
  int32_t x_dtype;      /* PXA_DTYPE_* */
  float eps;
  int32_t reverse_rows; /* 1: CTAs take the rows from the last to the first (start on the rows of x that the front-to-back
                           residual GEMM before it wrote last, i.e. the ones still in L2)                        */
  int32_t max_ctas;     /* 0 = auto: a grid-stride launch of two 8-warp CTAs per SM, every warp prefetching its next row;
                           > 0 caps / widens the grid (M / 8 or more = one row per warp)                               */
} PxaLnModArgs;
int pxa_ln_modulate(const PxaLnModArgs* args, void* stream);

/* First link of the fused LayerNorm-modulate chain (see PXA_EPI_LN_BIAS): for the residual stream x as the patch embedding
 * leaves it (PixArtMS.py:184), writes the A operand  a[r,:] = bf16( x[r,:] * mult[b,:] ), mult = 1 + scale (the same
 * multiplier PxaGemmArgs.aux_scale takes), and the row statistics
 * stats[r][0] = (sum_k x[r,k], sum_k x[r,k]^2), stats[r][1..7] = 0  that the QKV GEMM of block 0 consumes.  Later links
 * get both from the residual epilogues (PxaGemmArgs.aux_scale / row_stats_out).  HBM-bound: one read of x, one bf16 write.
 */
typedef struct PxaLnPrepareArgs {
  const float* x;       /* fp32 [M, C] row stride ldx                 */
  void* a_out;          /* bf16 [M, C] contiguous                     */
  float* stats_out;     /* fp32 [M][PXA_LN_STAT_PARTS][2]             */
  const float* scale;   /* fp32 multiplier 1 + scale_b, (b, c) at scale[b*mod_batch_stride + c] */
  int64_t mod_batch_stride;
  int32_t rows_per_batch;
  int32_t M, C, ldx;
} PxaLnPrepareArgs;
int pxa_ln_prepare(const PxaLnPrepareArgs* args, void* stream);

/* In-place LayerNorm(C = 1152, affine weight / bias bf16, fp32 statistics) on M bf16 rows of stride ld (elements):
 * q_norm / k_norm of AttentionKVCompress (`qk_norm=True`, PixArt_blocks.py:91-95,133-134) on the q and k column slices
 * of the qkv GEMM output.  HBM-bound: one read and one write of the slice. */
int pxa_layernorm_affine_bf16(void* x, const void* weight, const void* bias, int32_t M, int32_t C, int64_t ld, float eps,
                              void* stream);

/* RMS norm of the T5-v1.1-XXL caption encoder (transformers `T5LayerNorm`, eps 1e-6; reference call site diffusion/model/t5.py:107-110):
 * out[r, c] = bf16(x[r, c] * rsqrt(mean_c(x[r, :]^2) + eps) * weight[c]) on M rows of the fp32 residual stream (row strides ldx /
 * ldo in elements, C a multiple of 4).  HBM-bound: 4 C + 2 C bytes per row. */
int pxa_rmsnorm_bf16(const float* x, const void* weight, void* out, int32_t M, int32_t C, int64_t ldx, int64_t ldo, float eps,
                     void* stream);

/* Self-attention of the T5-v1.1-XXL caption encoder (transformers `T5Attention.forward`; reference call site
 * diffusion/model/t5.py:107-110): out[b, i, h, :] = softmax_j(q_i . k_j * scale + bias[h, i, j] + key_bias[b, j]) v_j for head_dim 64
 * and L <= 384 tokens per sample (T5 uses scale = 1 and a learned relative-position bias; key_bias carries the additive padding mask:
 * 0 for real tokens, a large negative number for padding).  q / k / v: bf16, element (b, i, h, d) at x[(b*L + i)*x_sn + h*x_sh + d]
 * (strided views of a fused qkv GEMM output are fine); out: bf16 [(b*L + i)*ldo + h*64 + d].  Logits, bias add, softmax and the
 * accumulation are fp32; P enters P V as bf16. */
typedef struct PxaT5AttnArgs {
  const void* q; const void* k; const void* v;
  void* out;
  const float* bias;      /* fp32 [H, L, L]; may be NULL when rel_bias is given                                              */
  const float* key_bias;  /* fp32 [B, L] or NULL                                                                             */
  int64_t q_sn, q_sh, k_sn, k_sh, v_sn, v_sh, ldo;
  int32_t B, H, L;
  float scale;
  const float* rel_bias;  /* fp32 [H, 2L-1] or NULL: the Toeplitz form bias[h, i, j] = rel_bias[h, j - i + L - 1] that T5's relative
                             position bias has; staged in shared memory (used instead of `bias` when non-NULL)              */
} PxaT5AttnArgs;
int pxa_t5_attn_d64_bf16(const PxaT5AttnArgs* args, void* stream);

/* GroupNorm (+ SiLU) on an NHWC bf16 image: the prologue of each 3x3 convolution of the SDXL-VAE decoder ResnetBlock2D
 * (diffusers GroupNorm(32, eps 1e-6) -> SiLU; reference call site scripts/inference.py:136).  out[b,p,c] =
 * silu((x[b,p,c] - mean[b,g]) * rstd[b,g] * gamma[c] + beta[c]), g = c / (C / groups), statistics over the HW pixels and the
 * C / groups channels of the group (fp32).  stats_ws: caller-owned fp32 [B][groups][2] scratch (zeroed by the call, on the
 * stream).  Two launches: statistics, apply.  HBM-bound: 2 reads + 1 write of the image. */
int pxa_groupnorm_silu_nhwc_bf16(const void* x, void* out, const void* gamma, const void* beta, float* stats_ws, int32_t B,
                                 int32_t HW, int32_t C, int32_t groups, float eps, int32_t silu, void* stream);

/* AdamW on a flat fp32 bucket (torch.optim.AdamW semantics: decoupled weight decay, bias-corrected moments) -- the optimizer
 * of the PixArt-alpha configs (configs/PixArt_xl2_internal.py:48 `AdamW(lr=1e-4, weight_decay=3e-2, eps=1e-10)`, built by
 * diffusion/utils/optimizer.py:236-245; the PixArt-Sigma configs train with CAME, pxa_came_flat below), applied to the
 * gradient buckets of pixart_sigma_b200.parallel.GradBucketReducer in one launch per bucket; optionally writes the bf16 copy of
 * the updated parameters that the GEMMs read.  All pointers device. */
typedef struct PxaAdamWArgs {
  float* param;          /* fp32 [n], updated in place          */
  const float* grad;     /* fp32 [n]                            */
  float* exp_avg;        /* fp32 [n], updated in place          */
  float* exp_avg_sq;     /* fp32 [n], updated in place          */
  void* shadow_bf16;     /* bf16 [n] or NULL                    */
  int64_t n;             /* multiple of 4                       */
  int32_t step;          /* 1-based step count (bias correction) */
  float grad_scale;      /* gradients are multiplied by this first (1 / loss scale, or 1) */
  double lr, beta1, beta2, eps, weight_decay;   /* as torch.optim.AdamW takes them: 1 - beta and the bias corrections
                                                   are formed in double, then rounded once to fp32 */
} PxaAdamWArgs;
int pxa_adamw_flat(const PxaAdamWArgs* args, void* stream);

/* Gradient-norm clipping over flat gradient buckets (torch.nn.utils.clip_grad_norm_, which train_scripts/train.py:181-182
 * reaches through accelerate):  g *= grad_scale;  total = ||g||_2 over every bucket;  g *= min(max_norm / (total + 1e-6), 1).
 * Two launches: per-CTA partial sums of squares into `partials` (PXA_GRAD_CLIP_PARTS slots), then every CTA reduces the
 * partials in the same fixed order, reads the coefficient on the device and scales its share.  No atomics, no host read:
 * `total_norm` (fp32 0-d, device) receives the norm.  Bucket pointers are 16-byte aligned; the elements past `n` (padding)
 * are not touched. */
#define PXA_GRAD_CLIP_PARTS 1024
#define PXA_GRAD_CLIP_MAX_BUCKETS 128
typedef struct PxaGradBucket {
  float* ptr;            /* fp32 [n], device, scaled in place */
  int64_t n;
} PxaGradBucket;
typedef struct PxaGradClipArgs {
  const PxaGradBucket* buckets;   /* HOST array [n_buckets] (passed to the kernels by value) */
  int32_t n_buckets;              /* 1 .. PXA_GRAD_CLIP_MAX_BUCKETS */
  float max_norm;
  float grad_scale;               /* multiplied in first (1 / loss scale, or 1) */
  float* partials;                /* fp32 [PXA_GRAD_CLIP_PARTS] workspace */
  float* total_norm;              /* fp32 [1] out: the norm after grad_scale, before clipping */
} PxaGradClipArgs;
int pxa_grad_clip_flat(const PxaGradClipArgs* args, void* stream);

/* CAME (came_pytorch.CAME.step, which every config under configs/pixart_sigma_config selects as `CAMEWrapper`,
 * diffusion/utils/optimizer.py:242-246) over every parameter of every flat bucket.  Per parameter p with gradient g, no bias
 * correction, state starting at zero:
 *   u = g^2 + eps1;  factored (ndim >= 2, p viewed as `lead` matrices R x C):  row = b2 row + (1-b2) mean_C u,
 *   col = b2 col + (1-b2) mean_R u,  u = rsqrt(row / mean_R row) rsqrt(col) g;   1-D:  v = b2 v + (1-b2) u,  u = rsqrt(v) g;
 *   u /= max(RMS(u) / clip_threshold, 1);  m = b1 m + (1-b1) u;
 *   factored: res = (u - m)^2 + eps2, rrow / rcol EMAs with b3 as above, upd = rsqrt(rrow / mean rrow) rsqrt(rcol) m;  1-D: upd = m;
 *   p -= weight_decay * lr * p (if weight_decay != 0);  p -= lr * upd;  rms[e] = ||p_before||_2 / sqrt(numel).
 * The parameter table (one PxaCameParam per parameter, built on the host and planned by pxa_came_workspace_bytes) is read
 * from device memory, so one launch per pass covers every bucket: 7 launches per step whatever the bucket count.  Work is
 * split into tiles: 2048 elements of a 1-D parameter; 256 whole matrices of a parameter whose matrices are at most 4 x 4 (one
 * thread each); 128 x 128 blocks of a larger matrix, whose row / column partial sums go to the workspace and are reduced in
 * a fixed order (no floating-point atomics: the same inputs give bitwise-equal results).  u is recomputed where needed,
 * .grad is only read.  Parameters need no alignment (scalar coalesced accesses), the bucket padding is not touched.
 * `lr` is read from device memory (a schedule can change it between CUDA-graph replays).  HBM-bound: 32 B per parameter
 * (g read 4 times, exp_avg read + written, p read + written). */
typedef struct PxaCameParam {
  float* param;          /* device: the parameter's first element in its flat fp32 parameter bucket               */
  const float* grad;     /* device: its gradient in the gradient bucket                                           */
  float* exp_avg;        /* device: its first moment in the exp_avg bucket                                        */
  int64_t numel;         /* lead * R * C                                                                          */
  int64_t offset;        /* element offset of the parameter in its bucket ...                                     */
  int64_t bucket_numel;  /* ... and the bucket's length: offset + numel <= bucket_numel is checked                */
  int64_t sq_off;        /* factored: offset of its lead * R row statistics in sq_row / res_row;
                            1-D: offset of its numel second moments in exp_avg_sq                                 */
  int64_t col_off;       /* factored: offset of its lead * C column statistics in sq_col / res_col                */
  int32_t lead, R, C;    /* 1-D: lead = 1, R = 1, C = numel                                                       */
  int32_t factored;      /* 1: ndim >= 2                                                                          */
  int64_t tile_begin;    /* plan, written by pxa_came_workspace_bytes: first tile ...                             */
  int64_t fin_begin;     /* ... first statistics-finalisation work item ...                                       */
  int64_t ws_off;        /* ... and workspace offset (floats) of the parameter                                    */
} PxaCameParam;
typedef struct PxaCameArgs {
  const PxaCameParam* table;  /* DEVICE copy of the planned table [n_entries]                                     */
  float* exp_avg_sq;          /* fp32 [n_vec]: second moments of the 1-D parameters                              */
  float* sq_row; float* res_row;   /* fp32 [n_row]                                                                */
  float* sq_col; float* res_col;   /* fp32 [n_col]                                                                */
  float* rms;                 /* fp32 [n_entries] out                                                             */
  const float* lr;            /* fp32 [1], device                                                                 */
  void* workspace;            /* caller-owned, workspace_bytes >= what pxa_came_workspace_bytes returned          */
  int64_t workspace_bytes;
  int64_t n_vec, n_row, n_col;
  int32_t n_entries;
  int32_t step;               /* 1-based step count (CAME applies no bias correction; must be positive)           */
  double eps1, eps2, clip_threshold, beta1, beta2, beta3, weight_decay;
  int64_t n_tiles, n_fin, ws_floats;   /* plan totals, written by pxa_came_workspace_bytes                       */
} PxaCameArgs;
/* Checks every entry of the HOST table against `args` (shapes, bucket bounds, state offsets), writes its plan fields and
 * args->n_tiles / n_fin / ws_floats, and returns the workspace size in *bytes.  Host only; call once, then copy the table
 * to the device. */
int pxa_came_workspace_bytes(PxaCameArgs* args, PxaCameParam* table_host, int64_t* bytes);
int pxa_came_flat(const PxaCameArgs* args, void* stream);

/* ------------------------------------------------------------------------------------------- attention
 * out[b, i, h, :] = softmax_j( q[b,i,h,:] . k[b,j,h,:] * scale ) v[b,j,h,:],  j < kv_len[b],  head_dim 72.
 * Flash-style: TMA-staged K/V ring, S = QK^T and O += PV on wgmma with S/P/O in registers, fp32 online softmax.
 * One kernel serves self-attention (PixArt_blocks.py:153, optionally KV-compressed: Nk < Nq) and the packed
 * var-len T5 cross-attention (PixArt_blocks.py:50-53, BlockDiagonalMask semantics via kv_off/kv_len).
 * Rows with kv_len == 0 produce zeros (xformers behaviour).
 */
typedef struct PxaAttnArgs {
  const void* q;  /* bf16, element (b, i, h, d) at q[(b*Nq + i)*q_sn + h*q_sh + d] */
  const void* k;  /* bf16, element (row, h, d) at k[row*k_sn + h*k_sh + d], row = kv_off[b] + j (see below) */
  const void* v;  /* bf16, same addressing as k with v_sn / v_sh */
  void* out;      /* bf16, element (b, i, h, d) at out[(b*Nq + i)*ldo + h*72 + d] */
  const int32_t* kv_len; /* device [B] or NULL (-> Nk for every sample)                                */
  const int32_t* kv_off; /* device [B] first key row of sample b, or NULL (-> b*Nk: padded/unpacked)   */
  int64_t q_sn, q_sh;
  int64_t k_sn, k_sh, v_sn, v_sh;
  int64_t kv_rows;  /* total rows addressable through k / v (B*Nk unpacked, sum(kv_len) packed)          */
  int32_t B, H, Nq, Nk; /* Nk = max keys per sample (loop bound) */
  int32_t ldo;
  float scale;      /* softmax scale, 72^-0.5 */
  int64_t* debug_trace; /* ignored (kept for binary compatibility) */
  float* lse;       /* optional fp32 [B, H, Nq]: log2-domain log-sum-exp of the scaled scores, the softmax statistic the
                       backward pass recomputes P from (training); NULL for inference                              */
  int32_t reverse_batch; /* 1: CTAs take the samples from the last to the first (same L2 argument as PxaGemmArgs.reverse_tiles:
                            the qkv rows of the last samples are the ones the QKV GEMM has just written)                   */
  int32_t variant;  /* 0 or 2..7: accepted for compatibility; one kernel (attn_fwd.cuh) serves them all with identical arithmetic */
  int32_t p_precision; /* 0 = P rounded to bf16 before P V (up to 2^-8 relative; the default).
                          1 = `fp32_attention` semantics (PixArt_blocks.py:145-147: q / k / v and hence P kept in fp32): P enters
                              the tensor pipe as bf16 hi + lo terms (2^-17 relative), two P V products per 16 keys; logits,
                              softmax and accumulation are fp32 in both modes.  Rejected together with variant 3.                  */
  int32_t reserved0;   /* must be 0 */
} PxaAttnArgs;
int pxa_flash_attn_d72_bf16(const PxaAttnArgs* args, void* stream);

/* ------------------------------------------------------------------------------------- KV token compression
 * out[b, p, c] = LN_c( bias[c] + sum_{dy,dx<2} w[c,dy,dx] * in[b, (2py+dy)*W + 2px+dx, c] ) * gamma[c] + beta[c]
 * Depthwise conv k=s=2 + LayerNorm(affine, eps 1e-5) on K and V (PixArt_blocks.py:84-89, 115-117), both tensors in
 * one launch.  in: bf16 rows of `ld_in` elements (k and v are column slices of the qkv GEMM output).
 */
typedef struct PxaKvCompressArgs {
  const void* k_in; const void* v_in; /* bf16, token row stride ld_in, batch stride H*W*ld_in */
  void* k_out; void* v_out;           /* bf16 [B, (H/2)*(W/2), C] contiguous                   */
  const void* conv_w;   /* bf16 [C, 1, 2, 2] */
  const void* conv_b;   /* bf16 [C]          */
  const void* ln_w;     /* bf16 [C]          */
  const void* ln_b;     /* bf16 [C]          */
  int32_t B, H, W, C, ld_in;
  float eps;
} PxaKvCompressArgs;
int pxa_kv_compress_conv2_ln(const PxaKvCompressArgs* args, void* stream);

/* ------------------------------------------------------------------------------------ 3x3 convolution (SDXL-VAE decoder)
 * out[b,y,x,:] = (residual[b,y,x,:] +) bias + sum_{dy,dx,c} w[:, dy, dx, c] * x[b, y+dy-1, x+dx-1, c]   (zero padding 1)
 * Implicit GEMM on the wgmma GEMM kernel: M = B*H*W pixels, N = Cout, K = 9*Cin; the A tiles are 128-pixel blocks of
 * the NHWC image fetched by a 4-D TMA tensor map whose out-of-bounds fill implements the padding (no im2col buffer).
 * Replaces the conv1 / conv2 of the decoder ResBlocks of diffusers' AutoencoderKL (reference call site
 * scripts/inference.py:136 `vae.decode`; GroupNorm + SiLU stay PyTorch).
 * Requirements: Cin % 64 == 0, Cout % 8 == 0.  Any H x W: widths that are a power of two <= 128 (with H a multiple of 128 / W) or a
 * multiple of 128 tile exactly; the others run over a virtual width rounded up to 128 (W / Wp of the MMA work is useful).
 */
typedef struct PxaConv3x3Args {
  const void* x;        /* bf16 NHWC [B, H, W, Cin] contiguous (torch channels_last)                         */
  const void* w;        /* bf16 [Cout, 3, 3, Cin] contiguous = checkpoint weight [Cout, Cin, 3, 3] permuted    */
  const void* bias;     /* bf16 [Cout] or NULL                                                               */
  void* out;            /* bf16 NHWC [B, H, W, Cout]                                                         */
  const void* residual; /* bf16 NHWC [B, H, W, Cout] or NULL                                                 */
  int32_t B, H, W, Cin, Cout;
} PxaConv3x3Args;
int pxa_conv3x3_nhwc_bf16(const PxaConv3x3Args* args, void* stream);

/* ------------------------------------------------------------------------------------ VAE output head to uint8 pixels
 * The decoder's conv_out (Cin -> 3 channels, 3x3, zero padding 1) on the NHWC bf16 output of conv_norm_out + SiLU, then
 * torchvision.utils.save_image's arithmetic (normalize=True, value_range=(-1, 1); call site scripts/inference.py:136-143):
 *     y[b,i,j,o] = bias[o] + sum_{dy,dx,c} w[o, dy, dx, c] * x[b, i+dy-1, j+dx-1, c]        (fp32 accumulation)
 *     u8         = trunc(clamp(((clamp(y, -1, 1) + 1) / 2) * 255 + 0.5, 0, 255))         (op by op in fp32, round to nearest)
 * x is addressed as x[b * x_sb + i * x_sh + j * x_sw + c] (elements; a channels_last tensor or a view with padded strides).
 * Requirements: B, H, W >= 1 (any H, W); Cin a multiple of 8; x 16-byte aligned with strides multiples of 8 elements.
 * Direct convolution on CUDA cores with an 8 x 32-pixel tile plus one-pixel halo staged in shared memory.
 */
typedef struct PxaVaeOutArgs {
  const void* x;        /* bf16 [B, H, W, Cin] with the strides below                                          */
  const void* w;        /* bf16 [3, 3, 3, Cin] contiguous = checkpoint weight [3, Cin, 3, 3] permuted            */
  const float* bias;    /* fp32 [3]                                                                            */
  uint8_t* out_u8;      /* uint8 [B, H, W, 3] contiguous                                                       */
  float* out_f32;       /* fp32 [B, H, W, 3] contiguous (y before the conversion), or NULL                     */
  int64_t x_sb, x_sh, x_sw;
  int32_t B, H, W, Cin;
} PxaVaeOutArgs;
int pxa_vae_out_u8(const PxaVaeOutArgs* args, void* stream);

/* ------------------------------------------------------------------------------------ DPM-Solver++ sampler step
 * One fused elementwise pass per sampling step of the multistep DPM-Solver++ (2M) loop the reference runs in PyTorch
 * (diffusion/model/dpm_solver.py: CFG combine :326-332, data prediction :435-444, first-order update :565-577,
 * second-order multistep update :822-840; loop :1196-1241; call site scripts/inference.py:102-118):
 *     eps   = eps_uncond + cfg_scale * (eps_cond - eps_uncond)
 *     x0    = (x - sigma_s * eps) * inv_alpha_s                      (data prediction at the current time s)
 *     x    <- a * x - b * x0 - c * (x0 - x0_prev)                    (c = 0: first-order update)
 *     x0_prev <- x0
 * with host-computed scalars a = sigma_t / sigma_s, b = alpha_t * expm1(-h), c = 0.5 * b / r0.
 * `model_out` is the denoiser output of the CFG batch [uncond (n) ; cond (n)]: element (i, ch, p) at
 * model_out[i * out_batch_stride + ch * hw + p], ch < 4 (so the 8-channel learn-sigma output can be passed as is).
 * fp32 arithmetic; x, x0_prev: fp32 [n, 4, hw] contiguous, updated in place.  HBM-bound: 24 (fp32 out) / 16 (bf16 out)
 * algorithmic bytes per latent element.
 */
typedef struct PxaDpmStepArgs {
  const void* model_out;    /* [2n, >=4, hw], dtype out_dtype                         */
  float* x;                 /* fp32 [n, 4, hw] in/out                                 */
  float* x0_prev;           /* fp32 [n, 4, hw] in/out (ignored on input when c == 0)  */
  int64_t out_batch_stride; /* elements                                               */
  int32_t n, hw;
  int32_t out_dtype;        /* PXA_DTYPE_*                                            */
  float cfg_scale, sigma_s, inv_alpha_s, a, b, c;
} PxaDpmStepArgs;
int pxa_dpm_solver_pp_step(const PxaDpmStepArgs* args, void* stream);

/* ------------------------------------------------------------------------------------ SA-Solver sampler step
 * One fused elementwise pass per denoiser evaluation of the SA-Solver loop the reference runs in PyTorch as
 * `SASolverSampler.sample` calls it (diffusion/sa_sampler.py:30-94: mode 'few_steps', skip_type 'time', predictor and
 * corrector order 2, PEC, data prediction; call site scripts/inference.py:119-133).  Evaluation i (0 <= i < S) at time t_i:
 *     eps      = eps_uncond + cfg_scale * (eps_cond - eps_uncond)    (guided; else the n conditional rows alone)
 *     m        = (x_pred - sigma * eps) * inv_alpha                  (data prediction, diffusion/model/sa_solver.py:377-386)
 *     x       <- c_x * x + c_m0 * m + c_m1 * m_prev + c_noise * noise_c      (corrector giving x_i, :700-753)
 *     x_pred  <- p_x * x + p_m0 * m + p_m1 * m_prev + p_noise * noise_p      (predictor giving x~_{i+1}, :644-698)
 *     m_prev  <- m
 * (the predictor reads the corrected x).  The host computes every scalar once per evaluation: c_x = exp(-tau_i^2 h_i)
 * sigma_i / sigma_{i-1}, c_noise = sigma_i sqrt(1 - exp(-2 tau_i^2 h_i)), c_m* the order-2 corrector gradient
 * coefficients, and p_* the same for the step to t_{i+1} (order 1 at the first and the last step, tau = 0 at the last);
 * i = 0 passes the identity corrector (c_x = 1, the others 0).  The loop driver: :841-897.
 * `model_out` rows as in PxaDpmStepArgs (guided: [uncond (n) ; cond (n)]).  A term whose coefficient is 0 is not read, so
 * m_prev may be uninitialised at i = 0 and noise_c / noise_p may be NULL when c_noise / p_noise is 0.
 * fp32 arithmetic; x, x_pred, m_prev, noise_*: fp32 [n, 4, hw] contiguous.  HBM-bound: 48 (fp32 out) / 40 (bf16 out)
 * algorithmic bytes per latent element with both noise terms.
 */
typedef struct PxaSaStepArgs {
  const void* model_out;    /* [2n (guided) or n, >=4, hw], dtype out_dtype                          */
  float* x;                 /* fp32 [n, 4, hw] in/out: x_{i-1} -> x_i                                */
  float* x_pred;            /* fp32 [n, 4, hw] in/out: x~_i (the denoiser input) -> x~_{i+1}         */
  float* m_prev;            /* fp32 [n, 4, hw] in/out: m_{i-1} -> m_i                                */
  const float* noise_c;     /* fp32 [n, 4, hw] xi_i, or NULL when c_noise == 0                       */
  const float* noise_p;     /* fp32 [n, 4, hw] xi_{i+1}, or NULL when p_noise == 0                   */
  int64_t out_batch_stride; /* elements                                                              */
  int32_t n, hw;
  int32_t out_dtype;        /* PXA_DTYPE_*                                                           */
  int32_t guided;           /* 1: CFG batch of 2n rows; 0: n conditional rows, cfg_scale ignored      */
  float cfg_scale, sigma, inv_alpha;
  float c_x, c_m0, c_m1, c_noise;
  float p_x, p_m0, p_m1, p_noise;
} PxaSaStepArgs;
int pxa_sa_solver_step(const PxaSaStepArgs* args, void* stream);

/* ------------------------------------------------------------------------------------ IDDPM ancestral step
 * One fused elementwise pass per step of the IDDPM sampling loop the reference runs in PyTorch as scripts/inference.py:89-101
 * calls it (`IDDPM(str(steps)).p_sample_loop(model.forward_with_cfg, ...)`): p_mean_variance with LEARNED_RANGE variance and
 * EPSILON prediction (diffusion/model/gaussian_diffusion.py:280-361), p_sample (:405-446), and the CFG mix of
 * forward_with_cfg (diffusion/model/nets/PixArtMS.py:221-234).  Per element of row r (fp32 arithmetic):
 *     eps      = model_out[r, c]                      c = 0..3; guided and c < 3: eps_u + cfg_scale (eps_c - eps_u), the
 *                                                     same mixed value for both rows of the pair (channel 3 stays the row's own)
 *     frac     = (model_out[r, 4 + c] + 1) / 2        (the row's own variance channel)
 *     logvar   = frac * log_beta + (1 - frac) * post_logvar
 *     pred_x0  = sqrt_recip_ac * img - sqrt_recipm1_ac * eps,   clamped to [-1, 1] when clip
 *     img     <- post_c1 * pred_x0 + post_c2 * img  (+ exp(0.5 * logvar) * noise when noise != NULL, i.e. t != 0)
 * Guided: N = 2n rows ordered [cond (n) ; uncond (n)] (inference.py:93, the reverse of the DPM / SA steps), both halves of
 * img are updated, and next_in receives the next model input [img[:n] ; img[:n]] (forward_with_cfg's cat([half, half])).
 * Unguided: N = n rows used as they are; next_in is not written (the next model input is img itself) and may be NULL.
 * The host computes every scalar once per step, as the fp64 tables rounded to fp32 (`_extract_into_tensor`).
 * model_out: [N, 8, hw] in out_dtype (fp32, bf16 or fp16), row r at r * out_batch_stride, channel c at c * hw.  img, noise,
 * next_in: fp32 [N, 4, hw] contiguous, 4-byte aligned.  Any hw.  HBM-bound: 16 (fp32 out) / 12 (bf16 / fp16 out) + 4 (noise)
 * + 4 (guided: next_in) algorithmic bytes per latent element.
 */
typedef struct PxaIddpmStepArgs {
  const void* model_out;    /* [N, 8, hw], dtype out_dtype                                          */
  float* img;               /* fp32 [N, 4, hw] in/out: x_t -> x_{t-1}                                */
  const float* noise;       /* fp32 [N, 4, hw], or NULL at t == 0                                    */
  float* next_in;           /* fp32 [N, 4, hw] out (guided), ignored when unguided                   */
  int64_t out_batch_stride; /* elements                                                              */
  int32_t n, hw;            /* n images: N = 2n rows guided, n unguided                              */
  int32_t out_dtype;        /* PXA_DTYPE_F32, PXA_DTYPE_BF16 or PXA_DTYPE_F16                        */
  int32_t guided;           /* 1: CFG pairs [cond ; uncond], cfg_scale used; 0: rows as they are     */
  int32_t clip;             /* 1: clamp pred_x0 to [-1, 1] (clip_denoised)                           */
  float cfg_scale, sqrt_recip_ac, sqrt_recipm1_ac, post_c1, post_c2, log_beta, post_logvar;
} PxaIddpmStepArgs;
int pxa_iddpm_step(const PxaIddpmStepArgs* args, void* stream);

/* ------------------------------------------------------------------------------------ LCM sampler step
 * One step of the reference's 4-step LCM sampler (`LCMScheduler.step`, diffusion/lcm_scheduler.py:310-410, epsilon
 * prediction; loop: train_scripts/train_pixart_lcm.py:105-135) in one elementwise pass:
 *     x0       = (x - sqrt_beta * eps) / sqrt_alpha            (sqrt(1 - ac_t), sqrt(ac_t))
 *     denoised = c_out * x0 + c_skip * x
 *     x_next   = c_prev * denoised + c_noise * noise           (sqrt(ac_prev), sqrt(1 - ac_prev); 1-step: c_prev = 1, c_noise = 0)
 * Every scalar comes from the host plan (float32 values computed with the reference's float32 torch operations).  Each
 * product, sum and the division is rounded separately (no FMA contraction), which is the reference's sequence of fp32
 * tensor operations.  `noise` is not read when c_noise == 0 (it may be NULL).  eps is `model_out` channels 0..3 (a
 * channel slice of the 8-channel learn-sigma output is fine), fp32 or bf16.  x, noise, denoised, x_next: fp32
 * [n, 4, hw] contiguous; x_next may alias x.  HBM-bound: 20 (bf16 eps, no noise) .. 28 algorithmic bytes per element. */
typedef struct PxaLcmStepArgs {
  const void* model_out;    /* [n, >=4, hw], dtype out_dtype, sample b at b * out_batch_stride              */
  const float* x;           /* fp32 [n, 4, hw]: the sample at t                                              */
  const float* noise;       /* fp32 [n, 4, hw], or NULL when c_noise == 0                                    */
  float* denoised;          /* fp32 [n, 4, hw] out                                                           */
  float* x_next;            /* fp32 [n, 4, hw] out (may alias x)                                             */
  int64_t out_batch_stride; /* elements                                                                      */
  int32_t n, hw;
  int32_t out_dtype;        /* PXA_DTYPE_*                                                                   */
  float sqrt_alpha, sqrt_beta, c_skip, c_out, c_prev, c_noise;
} PxaLcmStepArgs;
int pxa_lcm_step(const PxaLcmStepArgs* args, void* stream);

/* ------------------------------------------------------------------------------------ LCM consistency distillation
 * The per-step glue of train_scripts/train_pixart_lcm.py:223-303 (IDDPM with return_startx, DDIMSolver, boundary
 * scalings) as two kernels over a device table of PXA_LCM_MAX_ROWS rows, one per DDIM index (num_ddim_timesteps rows,
 * uploaded once and indexed on the device by `index`, so a step never reads anything back to the host):
 *   start = ddim_timesteps[index], t = max(start - k, 0) with k = train_timesteps / num_ddim_timesteps
 *   row.sra_s, row.srm1_s   = fp32 sqrt(1 / ac[start]), sqrt(1 / ac[start] - 1)      (IDDPM's fp64 tables, rounded)
 *   row.cskip_s, row.cout_s = the fp32 boundary scalings at start (scalings_for_boundary_conditions on int64 steps)
 *   row.sra_t .. row.cout_t = the same at t
 *   row.sqrt_acp, row.sqrt_1macp = fp64 sqrt(ac_prev[index]), sqrt(1 - ac_prev[index])  (DDIMSolver.ddim_alpha_cumprods_prev)
 * An index outside [0, n_rows) gives NaN for that sample. */
#define PXA_LCM_MAX_ROWS 1000
#define PXA_LCM_LOSS_PARTS 512
#define PXA_LCM_HUBER 0
#define PXA_LCM_L2 1
typedef struct PxaLcmRow {
  float sra_s, srm1_s, cskip_s, cout_s;
  float sra_t, srm1_t, cskip_t, cout_t;
  double sqrt_acp, sqrt_1macp;
} PxaLcmRow;

/* pxa_lcm_teacher_target: guided DDIM target from the teacher's batch-2b output [cond (b) ; uncond (b)] at x_t:
 *     x0_c = sra_s x_t - srm1_s eps_c,   x0_u = sra_s x_t - srm1_s eps_u                  (fp32, as the reference)
 *     x0   = x0_c + w (x0_c - x0_u),     eps = eps_c + w (eps_c - eps_u)                  (fp32, as the reference)
 *     x_prev = fp32( sqrt_acp * x0 + sqrt_1macp * eps )                                     (fp64 products and sum)
 * The reference's DDIM step multiplies by fp64 (b,1,1,1) tables, so its x_prev is fp64 and is rounded to fp32 only where
 * it is used (`x_prev.float()`, the loss).  Here that step is evaluated in fp64 with the same fp64 coefficients and
 * rounded once, so x_prev equals the reference's `x_prev.float()` exactly for the same fp32 x0 and eps.  The one place the
 * reference keeps more: its target uses the fp64 x_prev (c_skip(t) x_prev), the loss kernel the fp32 one (a relative
 * difference of at most 2^-24 in that term).  teacher_out: fp32 or bf16, channel slices fine; x_t, x_prev fp32 [b, 4, hw]. */
typedef struct PxaLcmTeacherArgs {
  const void* teacher_out;  /* [2b, >=4, hw], dtype out_dtype, sample r at r * out_batch_stride              */
  const float* x_t;         /* fp32 [b, 4, hw]                                                               */
  const int64_t* index;     /* DEVICE [b] DDIM indices                                                       */
  const PxaLcmRow* table;   /* DEVICE [n_rows]                                                               */
  float* x_prev;            /* fp32 [b, 4, hw] out                                                           */
  int64_t out_batch_stride;
  int32_t b, hw, out_dtype, n_rows;
  float w;                  /* guidance scale (config cfg_scale)                                             */
} PxaLcmTeacherArgs;
int pxa_lcm_teacher_target(const PxaLcmTeacherArgs* args, void* stream);

/* pxa_lcm_consistency_loss: the consistency loss and its gradient with respect to the student's output, per element
 *     model_pred = cskip_s x_t + cout_s (sra_s x_t - srm1_s eps_s)                         (fp32, as the reference)
 *     target     = fp32( cskip_t x_prev + fp32(cout_t (sra_t x_prev - srm1_t eps_e)) )     (fp64 sum, as the reference)
 *     d = model_pred - target;   huber: l = sqrt(d^2 + c^2) - c, evaluated as d^2 / (sqrt(d^2 + c^2) + c) (no cancellation
 *     for |d| << c);  l2: l = d^2
 *     loss = mean(l) over b * 4 * hw  ->  *loss (fp32)
 *     d_student_out[:, 0:4] = dl/dd * (-cout_s srm1_s) / (b * 4 * hw),   d_student_out[:, 4:out_channels] = 0 exactly
 * Launch 1: one pass over the elements by PXA_LCM_LOSS_PARTS CTAs, each writing the fp64 sum of its elements' l to
 * partials[cta]; launch 2: one CTA sums the partials in index order.  No floating-point atomics: the result is bitwise
 * reproducible.  eps_s: fp32 (the student's output); eps_e: fp32 or bf16; both channel slices of [*, >=4, hw] outputs. */
typedef struct PxaLcmLossArgs {
  const float* student_out;   /* fp32 [b, >=4, hw], sample b at b * student_batch_stride                     */
  const void* ema_out;        /* [b, >=4, hw], dtype ema_dtype, sample b at b * ema_batch_stride               */
  const float* x_t;           /* fp32 [b, 4, hw]                                                             */
  const float* x_prev;        /* fp32 [b, 4, hw]                                                             */
  const int64_t* index;       /* DEVICE [b]                                                                  */
  const PxaLcmRow* table;     /* DEVICE [n_rows]                                                             */
  float* d_student_out;       /* fp32 [b, out_channels, hw] contiguous out                                   */
  float* loss;                /* fp32 [1] out                                                                */
  double* partials;           /* fp64 [PXA_LCM_LOSS_PARTS] workspace                                         */
  int64_t student_batch_stride, ema_batch_stride;
  int32_t b, hw, ema_dtype, n_rows;
  int32_t out_channels;       /* 4 or 8                                                                      */
  int32_t loss_type;          /* PXA_LCM_HUBER or PXA_LCM_L2                                                 */
  float huber_c;
} PxaLcmLossArgs;
int pxa_lcm_consistency_loss(const PxaLcmLossArgs* args, void* stream);

/* ------------------------------------------------------------------------------------ flat EMA update
 * ema_update(model_ema, model, rate) of train_scripts/train_pixart_lcm.py:48-53 (`d.mul_(rate).add_((1 - rate) * s)`) over
 * every bucket in ONE launch (grid: x = CTAs per bucket, y = bucket), reading a DEVICE table of buckets:
 *     master[i] = fp32(fp32(master[i] * rate) + fp32(src[i] * (1 - rate)))      (three roundings, no FMA: bitwise torch's)
 *     shadow[i] = bf16(master[i])                                                 (round to nearest even)
 * for i < n only: the padding of a bucket is never read or written.  rate and 1 - rate are rounded to fp32 from the double
 * `rate` as torch does for a Python scalar.  master, src: 16-byte aligned; shadow: 8-byte aligned.  14 B of HBM traffic
 * per parameter (read 4 + 4, write 4 + 2). */
typedef struct PxaEmaBucket {
  float* master;            /* fp32 [n] EMA master values, in / out                                          */
  const float* src;         /* fp32 [n] the online model's parameters                                        */
  void* shadow;             /* bf16 [n] out: the EMA model's forward weights (NULL: not written)             */
  int64_t n;                /* parameter elements of the bucket (its padding excluded)                       */
} PxaEmaBucket;
typedef struct PxaEmaArgs {
  const PxaEmaBucket* table;  /* DEVICE [n_buckets]                                                         */
  int32_t n_buckets;          /* 1 .. 65535                                                                  */
  int64_t max_n;              /* max over the buckets of n (sizes the grid)                                  */
  double rate;
} PxaEmaArgs;
int pxa_ema_flat(const PxaEmaArgs* args, void* stream);

/* ------------------------------------------------------------------------------------ DMD distribution-matching loss
 * The glue of one distribution-matching step (train_scripts/train_pixart_dmd.py:519-561, `use_dm`, `snr_gamma=None`) between
 * the one-step generator's x0 (`latents`), the frozen real model's CFG batch and the fake model's output, per element:
 *     a = alphas_cumprod[t[i]],  sa = sqrt(a),  sb = sqrt(1 - a)                  (fp32; t outside [0, n_timesteps): NaN)
 *     score_real = -(eps_u + cfg (eps_c - eps_u)),  score_fake = -eps_f
 *     coeff  = (score_fake - score_real) sb / sa,   pred = (noisy + sb score_real) / sa
 *     weight[i] = 1 / (mean_i |latents - pred| + 1e-5)                            (per sample; the mean from an fp64 sum)
 *     target = latents - weight coeff,   d = latents - target,   loss = mean(d^2) over b * 4 * hw
 *     d_gen_out[:, 0:4] = (2 d / (b * 4 * hw)) / gen_sqrt_alpha * (-gen_sqrt_beta)   (dL/deps of x0 = (x - sb_g eps) / sa_g)
 *     d_gen_out[:, 4:out_channels] = 0 exactly
 * Every product, sum and division is rounded once, in the reference's fp32 order (the mean over a sample and the loss are
 * summed in fp64).  Launch 1: PXA_DMD_PARTS CTAs per sample write fp64 partial sums of |latents - pred|; launch 2: each CTA
 * folds its sample's partials in index order into weight and writes the gradient and fp64 loss partials; launch 3: one CTA
 * sums the loss partials in index order.  No floating-point atomics: bitwise reproducible, never syncs the host.
 * real_out: [2b, >=4, hw] with rows 0..b-1 unconditional; fake_out: [b, >=4, hw]; both fp32 or bf16, channel slices fine.
 * latents, noisy: fp32 [b, 4, hw] contiguous. */
#define PXA_DMD_PARTS 64
typedef struct PxaDmdLossArgs {
  const float* latents;         /* fp32 [b, 4, hw]: the generator's x0                                          */
  const float* noisy;           /* fp32 [b, 4, hw]: add_noise(latents, noise, t)                                */
  const int64_t* timesteps;     /* DEVICE [b]                                                                  */
  const float* alphas_cumprod;  /* DEVICE fp32 [n_timesteps]                                                   */
  const void* real_out;         /* [2b, >=4, hw], dtype real_dtype, row r at r * real_batch_stride             */
  const void* fake_out;         /* [b, >=4, hw], dtype fake_dtype, row r at r * fake_batch_stride              */
  float* d_gen_out;             /* fp32 [b, out_channels, hw] contiguous out                                   */
  float* loss;                  /* fp32 [1] out                                                                */
  float* weight;                /* fp32 [b] out                                                                */
  double* partials;             /* fp64 [2 * b * PXA_DMD_PARTS] workspace                                      */
  int64_t real_batch_stride, fake_batch_stride;
  int32_t b, hw, n_timesteps;
  int32_t out_channels;         /* 4 or 8                                                                      */
  int32_t real_dtype, fake_dtype;
  float cfg;                    /* guidance scale of the real model                                            */
  float gen_sqrt_alpha, gen_sqrt_beta;  /* fp32 sqrt(ac[t_g]), sqrt(1 - ac[t_g]) of the generator's step       */
} PxaDmdLossArgs;
int pxa_dmd_loss(const PxaDmdLossArgs* args, void* stream);

/* =============================================================================================== training backward
 * The reference trains through torch autograd (train_scripts/train.py:197 `accelerator.backward(loss)`, per-block
 * activation checkpointing diffusion/model/utils.py:28-45).  The entry points below are the backward twins of the forward
 * ops above; `pixart_sigma_b200/autograd.py` binds them as torch.autograd.Function s.  The dgrad / wgrad matrix products
 * run on pxa_gemm_bf16 itself (dX = dY . W  ==  gemm(A = dY, W' = W^T);  dW += dY^T . X  ==  gemm(A = dY^T, W' = X^T) with the
 * fp32 residual epilogue adding into the gradient buffer), fed by pxa_transpose_bf16.
 */

/* out[C, R] = in[R, C]^T (bf16; 32-bit accesses when R, C, ldi, ldo are even, element-wise otherwise). */
int pxa_transpose_bf16(const void* in, void* out, int32_t R, int32_t C, int64_t ldi, int64_t ldo, void* stream);

/* GELU(approximate='tanh') on n bf16 elements (n % 8 == 0): dh == NULL: out = gelu(pre);  else out = dh * gelu'(pre).
 * Replaces timm Mlp.act (PixArtMS.py:67) forward (training path, which keeps `pre` for the backward) and backward. */
int pxa_gelu_tanh_bf16(const void* pre, const void* dh, void* out, int64_t n, void* stream);

/* Gated residual add of the block (PixArtMS.py:75-77) on the fp32 residual stream, and its backward.
 *   fwd: out[r,:] = x[r,:] + gate[b,:] * y[r,:]                      (x, out fp32; y bf16; gate NULL -> 1)
 *   bwd: x = dout (fp32), out = dy (bf16) = dout * gate[b,:];  dgate[b,:] += sum_{r in b} dout[r,:] * y[r,:]  (if dgate)  */
typedef struct PxaGateResidualArgs {
  const void* x;        /* fp32 [M, C] contiguous (fwd: residual stream; bwd: incoming gradient)               */
  const void* y;        /* bf16 [M, C] contiguous branch output (bwd: only needed with dgate)                   */
  const float* gate;    /* fp32 (b, c) at gate[b*gate_batch_stride + c], or NULL                                */
  void* out;            /* fwd: fp32 [M, C];  bwd: bf16 [M, C]                                                  */
  float* dgate;         /* bwd only: fp32 [B, C] contiguous, accumulated into (atomics); or NULL                */
  int64_t gate_batch_stride;
  int32_t rows_per_batch;
  int32_t M, C;
} PxaGateResidualArgs;
int pxa_gate_residual_fwd(const PxaGateResidualArgs* args, void* stream);
int pxa_gate_residual_bwd(const PxaGateResidualArgs* args, void* stream);

/* Backward of pxa_ln_modulate w.r.t. x, shift and scale (C = 1152):
 *   dx = LN-backward((1 + scale[b]) * dxn);  dshift[b,:] += sum_r dxn[r,:];  dscale[b,:] += sum_r dxn[r,:] * xhat[r,:]  */
typedef struct PxaLnModBwdArgs {
  const void* x;        /* fp32 [M, C] contiguous: the forward input                                            */
  const void* dxn;      /* bf16 [M, C] contiguous: gradient of the forward output                               */
  const float* scale;   /* fp32 (b, c) at scale[b*mod_batch_stride + c]                                         */
  void* dx;             /* fp32 [M, C] contiguous (written)                                                     */
  float* dshift;        /* fp32 [B, C] contiguous (accumulated, atomics)                                        */
  float* dscale;        /* fp32 [B, C] contiguous (accumulated, atomics)                                        */
  int64_t mod_batch_stride;
  int32_t rows_per_batch;
  int32_t M, C;
  float eps;
  const float* add_in;  /* optional fp32 [M, C]: dx = add_in + (gradient through the LayerNorm): the gradient of the residual
                           stream that by-passes the norm (x feeds both the norm and the residual add), folded in       */
} PxaLnModBwdArgs;
int pxa_ln_modulate_bwd(const PxaLnModBwdArgs* args, void* stream);

/* Backward of pxa_kv_compress_conv2_ln (depthwise conv k=s=2 + LayerNorm(affine) on K and V, PixArt_blocks.py:84-89,
 * 115-117): input gradients written to the 4 input rows of every output token, parameter gradients (shared by K and V)
 * ACCUMULATED into fp32 buffers (atomics).  The LN bias does not influence any gradient and is not needed. */
typedef struct PxaKvCompressBwdArgs {
  const void* k_in; const void* v_in;     /* bf16 forward inputs, token row stride ld_in                           */
  const void* dk_out; const void* dv_out; /* bf16 [B, (H/2)*(W/2), C] gradients of the compressed K / V             */
  void* dk_in; void* dv_in;               /* bf16 gradients of the inputs, token row stride ld_din (written)        */
  const void* conv_w; const void* conv_b; const void* ln_w;   /* bf16 parameters as in the forward                  */
  float* d_conv_w;      /* fp32 [C, 1, 2, 2] accumulated */
  float* d_conv_b;      /* fp32 [C] accumulated           */
  float* d_ln_w;        /* fp32 [C] accumulated           */
  float* d_ln_b;        /* fp32 [C] accumulated           */
  int32_t B, H, W, C, ld_in, ld_din;
  float eps;
} PxaKvCompressBwdArgs;
int pxa_kv_compress_conv2_ln_bwd(const PxaKvCompressBwdArgs* args, void* stream);

/* out[c] += sum_r a[r, c]  (bias gradients; a bf16 [M, N] row stride lda, N % 8 == 0; out fp32 [N], atomics). */
int pxa_colsum_bf16(const void* a, float* out, int32_t M, int32_t N, int64_t lda, void* stream);

/* delta[(b*H + h)*Nq + i] = sum_d dO[b,i,h,d] * O[b,i,h,d]  (o / dO bf16 [B*Nq, H*72] with row strides ldo / lddo). */
int pxa_attn_delta_d72(const void* o, const void* d_o, float* delta, int32_t B, int32_t H, int32_t Nq, int64_t ldo,
                       int64_t lddo, void* stream);

/* Backward of pxa_flash_attn_d72_bf16: dq, dk, dv from (q, k, v, o, dO, lse).  Flash-attention-2 recomputation on
 * wgmma (two passes: dK/dV per key tile, dQ per query tile); nothing N x N reaches HBM.  Same addressing as the
 * forward (strided bf16 views, packed var-len keys through kv_off / kv_len), any Nq / Nk.
 * dk / dv rows of keys >= kv_len[b] are not written.  `delta` is caller-owned workspace.                         */
typedef struct PxaAttnBwdArgs {
  const void* q; const void* k; const void* v;   /* as PxaAttnArgs                                              */
  const void* o;        /* bf16 forward output, (b, i, h, d) at o[(b*Nq + i)*ldo + h*72 + d]                      */
  const void* d_o;      /* bf16 gradient of o, row stride lddo                                                   */
  const float* lse;     /* fp32 [B, H, Nq] written by the forward (PxaAttnArgs.lse)                              */
  float* delta;         /* fp32 [B, H, Nq] workspace                                                             */
  void* dq; void* dk; void* dv;                  /* bf16, addressed like q / k / v with the strides below        */
  const int32_t* kv_len; const int32_t* kv_off;
  int64_t q_sn, q_sh, k_sn, k_sh, v_sn, v_sh;
  int64_t dq_sn, dq_sh, dk_sn, dk_sh, dv_sn, dv_sh;
  int64_t ldo, lddo;
  int64_t kv_rows;
  int32_t B, H, Nq, Nk;
  float scale;
} PxaAttnBwdArgs;
int pxa_flash_attn_d72_bwd_bf16(const PxaAttnBwdArgs* args, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* PIXART_SM100_H_ */
