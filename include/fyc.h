/*
 * libfyc_sm90a.so - C ABI of the H100-native FollowYourClick denoising engine.
 *
 * The reference (mayuelala/FollowYourClick) has no FFI: every GPU instruction it issues comes from
 * PyTorch/cuDNN/cuBLAS call sites inside Python modules.  Each entry point below replaces one family of
 * those call sites (cited as reference file:line, relative to the reference repo root); the Python classes
 * in followyourclick_b200/ keep the reference call surface and hand raw device pointers to these functions.
 *
 * Conventions (SURVEY.md section 8b):
 *   - caller owns every buffer (inputs, outputs, workspace); the library never allocates device memory,
 *     never synchronises, never touches the default stream: all work is enqueued on `stream`;
 *   - return value 0 = OK, non-zero = error, message via fyc_last_error() (thread-local);
 *   - activations are channels-last "tokens": [images(B*F), H*W, C] contiguous unless a leading dimension
 *     is passed; `dtype` selects the storage type of activations/weights (accumulation is always fp32); "16-bit" below means
 *     FYC_BF16 or FYC_F16;
 *   - small per-channel vectors (bias, norm gamma/beta) are always fp32.
 */
#ifndef FYC_H_
#define FYC_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define FYC_VERSION 100 /* 0.1.0 */

enum { FYC_OK = 0, FYC_ERR_INVALID = 1, FYC_ERR_CUDA = 2, FYC_ERR_UNSUPPORTED = 3 };
/* storage dtypes.  FYC_F16 (IEEE half) is accepted wherever FYC_BF16 is, with the same layouts and eligibility rules: its 11
 * significand bits round about 8x finer than bf16's 8, and its range ends at 65504 (the caller keeps activations within it). */
enum { FYC_F32 = 0, FYC_BF16 = 1, FYC_F16 = 2 };
/* GEMM / conv implementation selector */
enum { FYC_IMPL_AUTO = 0, FYC_IMPL_SIMT = 1, FYC_IMPL_TCGEN05 = 2 };
/* epilogue flags */
enum {
  FYC_EPI_BIAS = 1,      /* + bias[n]                                  */
  FYC_EPI_RESIDUAL = 2,  /* + residual[m, n]                           */
  FYC_EPI_ROWBIAS = 4,   /* + rowbias[m / rows_per_group, n]  (time embedding broadcast, resnet.py:307,319) */
  FYC_EPI_GEGLU = 8,     /* out[m, j] = a * gelu_erf(gate); weight rows pre-interleaved in 128-col granules */
  FYC_EPI_OUT_F32 = 16,  /* write fp32 output regardless of `dtype`    */
  FYC_EPI_LNFOLD = 32    /* A is the RAW input x of a LayerNorm whose output this GEMM consumes (attention.py:383,412,418, motion_module.py:261,
                            267: norm1/2/3, norms.j, ff_norm -> to_q/k/v, ff.net.0.proj).  The caller packs W" = gamma (.) W with every row
                            CENTRED (W"[n, k] -= mean_k of the row): since mean_m = (1/C) sum_k x[m, k],
                              x W"^T = x W'^T - mean_m * colsum(W')[n]   and   LN(x) W^T + b = rstd_m * (x W"^T)[m, n] + (beta W^T + b)[n],
                            i.e. the mean subtraction lives in the weights, the tensor core computes the bracket, and the epilogue only scales
                            by rstd_m (ln_rowstats, from fyc_layernorm_stats) and adds the bias: the GEMM costs what the plain one costs,
                            and LayerNorm's read + write pass shrinks to one read-only statistics pass.  tensor-core path; alpha = 1, no fp32
                            output, no residual; with FYC_EPI_ROWBIAS (the temporal position table P W^T) rows_per_group % 128 == 0. */
};
enum { FYC_PRED_EPSILON = 0, FYC_PRED_SAMPLE = 1, FYC_PRED_V = 2 };

int32_t fyc_version(void);
const char* fyc_last_error(void);
/* 1 if the tensor-core (wgmma / TMA) kernels can run (driver entry point for cuTensorMapEncodeTiled resolved); the name is kept
 * for ABI stability. */
int32_t fyc_tcgen05_available(void);

/* ---- linear / 1x1 conv / batched matmul ---------------------------------------------------------------
 * out[b][m, n] = alpha * sum_k A[b][m, k] * W[b][n, k]  (+ epilogue).  Replaces F.linear / 1x1 F.conv2d /
 * baddbmm call sites: diffusers/models/attention.py:560-569,654-660,672 (q,k,v,out, scores), :733-821 (FF),
 * animatediff/models/attention.py:182,215 (proj_in/out), resnet.py:286 (shortcut), motion_module.py:128,155.
 * A: [M, K] lda; W: [N, K] ldw; out: [M, N_out] ldo where N_out = N (or N/2 with FYC_EPI_GEGLU).
 */
typedef struct {
  const void* A; const void* W; void* out;
  const float* bias;            /* [N] fp32 (FYC_EPI_BIAS) */
  const void* residual;         /* [M, N_out] ldr, same dtype as out unless residual_f32 */
  const float* rowbias;         /* [M / rows_per_group, N] fp32 (FYC_EPI_ROWBIAS) */
  int64_t M, N, K;
  int64_t lda, ldw, ldo, ldr;
  int64_t batch, strideA, strideW, strideO;   /* batch >= 1; strides in elements */
  int64_t rows_per_group;
  float alpha;
  int32_t dtype, epilogue, impl;
  const void* A2;               /* optional second K segment (NULL: none): A[:, :K1] comes from A (lda), A[:, K1:] from A2 (lda2) - the GEMM over
                                   a channel concatenation that is never written (the up blocks' conv_shortcut on cat([x, skip]),
                                   resnet.py:286 after unet_blocks.py:763,885).  tensor-core path: K1 % 64 == 0.  W stays [N, K]. */
  int64_t lda2, K1;
  const float* ln_rowstats;     /* FYC_EPI_LNFOLD: [M] fp32 rstd per row, from fyc_layernorm_stats */
} fyc_gemm_args;
int32_t fyc_gemm(const fyc_gemm_args* a, void* stream);

/* ---- 3x3 convolution as implicit GEMM (NHWC) ----------------------------------------------------------
 * Replaces InflatedConv3d / nn.Conv2d 3x3 call sites: animatediff/models/resnet.py:19-27,245,270,
 * unet.py:124,351, Downsample3D resnet.py:184 (stride 2), Upsample3D :155,168 (nearest x2 folded into the
 * input index), diffusers/models/vae.py:160,205, resnet.py:407,423, Upsample2D :139.
 * x: [NB, H, W, Cin]; w: [Cout, 3, 3, Cin] (re-packed once from the reference [Cout, Cin, 3, 3]);
 * out: [NB, Ho, Wo, Cout], Ho = (H*up + 2 - 3)/stride + 1.
 */
typedef struct {
  const void* x; const void* w; void* out;
  const float* bias; const void* residual; const float* rowbias;
  int64_t NB, H, W, Cin, Cout;
  int32_t stride;               /* 1 or 2 */
  int32_t upsample;             /* 1 or 2: nearest-neighbour upsampling of x before the conv */
  int64_t images_per_group;     /* rowbias row = image / images_per_group  (= F, frames per clip) */
  int32_t dtype, epilogue, impl;
  void* workspace;              /* fyc_conv3x3_workspace_bytes() bytes (stride-2 / upsample on the tensor-core path) */
  size_t workspace_bytes;
  int32_t pad_mode;             /* 0: zero pad 1 on every side.  1 (stride 2, even H and W, upsample 1 only): pad 1 on the bottom /
                                   right only - diffusers Downsample2D with padding=0, F.pad(x, (0,1,0,1)) + valid conv
                                   (diffusers/models/resnet.py:183-188), the VAE Encoder's downsamplers (vae.py:95);
                                   Ho = H/2 either way, input row = 2*oh + kh instead of 2*oh + kh - 1 */
  const void* w_phases;         /* optional (upsample == 2, 16-bit): the filter pre-summed per output parity, [4 phases = 2*py+px]
                                   [Cout][2][2][Cin].  nearest-x2 followed by a padded 3x3 conv is, for each output parity (py, px),
                                   a 2x2 conv on the LOW-resolution image: rows {oh-1 | w[0], oh | w[1]+w[2]} for py = 0 and
                                   {oh | w[0]+w[1], oh+1 | w[2]} for py = 1 (columns alike) - 16 instead of 36 MACs per input
                                   pixel and channel pair, and the upsampled tensor is never written.  The tensor-core path runs the
                                   four phases as four 4-tap implicit GEMMs whose rows are written interleaved; without it (or on
                                   the CUDA-core path) `w` is used with the upsample folded into the input index. */
  int64_t ld_rowbias;           /* row stride of `rowbias` in elements; 0 = Cout.  > Cout when rowbias points into a wider table -
                                   all ResnetBlock3D time-embedding projections of a forward (resnet.py:307-313) come out of ONE
                                   fused GEMV as [B, sum Cout], each conv reading its own column block */
} fyc_conv3x3_args;
size_t fyc_conv3x3_workspace_bytes(const fyc_conv3x3_args* a);
int32_t fyc_conv3x3(const fyc_conv3x3_args* a, void* stream);
/* 1 when a (upsample == 2, w_phases != NULL) call will take the four-phase tensor-core path, else 0 (the caller then either
 * materialises the upsample and runs the plain 3x3 path, or lets fyc_conv3x3 fold it into the CUDA-core kernel's index). */
int32_t fyc_conv3x3_up2_eligible(const fyc_conv3x3_args* a);
/* 1 when fyc_conv3x3 will run this call (workspace as given) on the tensor-core kernel, else 0 (the CUDA-core kernels).  A shape whose
 * output grid has no 128-pixel patch bw x bh x bn of powers of two dividing Wo, Ho and NB (e.g. 5 x 9 pixels over 32 images) is not
 * tensor-core eligible even when its channel counts are. */
int32_t fyc_conv3x3_tc_route(const fyc_conv3x3_args* a);

/* ---- normalisation ------------------------------------------------------------------------------------
 * GroupNorm (+ optional SiLU) over x viewed as [NB, R, C]: statistics per (nb, group) over R rows x C/G
 * channels.  Cross-frame statistics of ResnetBlock3D (resnet.py:240,263; nn.GroupNorm on the 5-D tensor):
 * NB = clips, R = F*H*W.  Per-frame statistics (attention.py:178,269; motion_module.py:127,188; VAE): NB =
 * images, R = H*W.  workspace: fyc_groupnorm_workspace_bytes().
 */
size_t fyc_groupnorm_workspace_bytes(int64_t NB, int64_t C, int64_t G);
int32_t fyc_groupnorm(const void* x, const float* gamma, const float* beta, void* out, int64_t NB, int64_t R,
                      int64_t C, int64_t G, float eps, int32_t silu, int32_t dtype, void* workspace,
                      size_t workspace_bytes, void* stream);
/* GroupNorm of the channel concatenation [x1 (C1) | x2 (C2)] WITHOUT materialising it: the up blocks' `torch.cat([hidden_states,
 * res_hidden_states], dim=1)` (animatediff/models/unet_blocks.py:763,885) feeds ResnetBlock3D.norm1 (and the 1x1 shortcut, see
 * fyc_gemm_args.A2); both read the two tensors in place.  out: [NB, R, C1 + C2].  Same workspace as fyc_groupnorm with C = C1 + C2. */
int32_t fyc_groupnorm_concat(const void* x1, int64_t C1, const void* x2, int64_t C2, const float* gamma, const float* beta, void* out,
                             int64_t NB, int64_t R, int64_t G, float eps, int32_t silu, int32_t dtype, void* workspace,
                             size_t workspace_bytes, void* stream);
/* LayerNorm over the last dim (attention.py:383,412,418; motion_module.py:261,267), optional sinusoidal
 * position table added AFTER the norm: out = LN(x) + pe[(row / rows_per_frame) % frames]  (motion_module.py:303,378). */
int32_t fyc_layernorm(const void* x, const float* gamma, const float* beta, void* out, int64_t M, int64_t C,
                      float eps, const float* pe, int64_t rows_per_frame, int64_t frames, int32_t dtype,
                      void* stream);

/* LayerNorm statistics only (biased variance + eps like nn.LayerNorm) for a GEMM launched with FYC_EPI_LNFOLD: rstd[m] (fp32).  `aug` is
 * optional (NULL: not written): [m][8] in `dtype` (bf16 for fp32 rows) = [m_hi, m_hi, m_lo, m_lo, 0, 0, 0, 0] with mean_m = m_hi + m_lo, for callers that want the
 * row mean as a second K segment of a GEMM (fyc_gemm_args.A2) instead of centred weights. */
int32_t fyc_layernorm_stats(const void* x, float* rstd, void* aug, int64_t M, int64_t C, float eps, int32_t dtype, void* stream);

/* ---- attention ----------------------------------------------------------------------------------------
 * out[n, i, h*D + :] (=|+=) out_alpha * softmax_j(scale * q[n,i,h] . k[n',j,h]) v[n',j,h],  n' = n / kv_batch_div.
 * Replaces CrossAttention._attention (diffusers/models/attention.py:649-678) for attn1/attn2 and the two
 * softmaxes of IPCrossAttention.forward (animatediff/models/attention.py:98-120; second call with
 * accumulate=1, out_alpha = ip scale - or both at once through k2 / v2 / alpha2).  Never materialises the score matrix.
 */
typedef struct {
  const void* q; const void* k; const void* v; void* out;
  int64_t batch, heads, Lq, Lk, D;
  int64_t ldq, ldk, ldv, ldo;            /* row strides in elements */
  int64_t bsq, bsk, bsv, bso;            /* batch strides in elements */
  int64_t kv_batch_div;                  /* >= 1: context shared by F consecutive images (attention.py:264) */
  float scale, out_alpha;
  int32_t accumulate, dtype, impl;
  /* optional SECOND context, fused (NULL: none): out = out_alpha * softmax(scale q k^T) v + alpha2 * softmax(scale q k2^T) v2, written once.
     The IP-Adapter cross-attention - text keys [:, :-T] and image keys [:, -T:] with their own to_k_ip / to_v_ip projections, two
     softmaxes, `hidden_states + self.scale * ip_hidden_states` (animatediff/models/attention.py:92-120,
     ip_adapter/attention_processor.py:137-168) - as ONE kernel instead of two attention passes and an add.  Same batch / heads / D /
     kv_batch_div as the first context. */
  const void* k2; const void* v2;
  int64_t Lk2, ldk2, ldv2, bsk2, bsv2;
  float alpha2;
} fyc_attention_args;
int32_t fyc_attention(const fyc_attention_args* a, void* stream);

/* Temporal self-attention over the frame axis (VersatileAttention.forward, motion_module.py:371-464 +
 * mm_attn_cross.py:148-177): qkv [B, F, HW, 3C] (q | k | v packed per token), out [B, F, HW, C].  The
 * '(b f) d c -> (b d) f c' regrouping (motion_module.py:376,462) is absorbed into the addressing. */
int32_t fyc_temporal_attention(const void* qkv, void* out, int64_t B, int64_t F, int64_t HW, int64_t heads,
                               int64_t D, float scale, int32_t dtype, void* stream);
/* Spatial self-attention on the tensor cores (wgmma; S, O accumulators in registers) for head dim 40 or 64, L % 128 == 0 - the level-0
 * attn1 of an SD-1.5 UNet, every attn1 of an SD-2.x UNet (diffusers/models/attention.py:649-678 via animatediff/models/attention.py:507).
 * qk: [NB, L, ldqk] bf16, q head h at columns [q_col0 + 64h, +64), k head h at [k_col0 + 64h, +64): for D = 40 columns 40..63 of each
 * head ZERO (zero rows in the packed projection weight), for D = 64 the fused [q | k | v] projection as is; vt: [NB, heads*D, L]
 * (V transposed per image, fyc_transpose_tokens); out: [NB, L, ldo], head h at columns [h*D, (h+1)*D). */
int32_t fyc_self_attention_tc(const void* qk, int64_t ldqk, int64_t q_col0, int64_t k_col0, const void* vt, void* out,
                              int64_t ldo, int64_t NB, int64_t heads, int64_t L, int64_t D, float scale, void* stream);
/* The same with fp16 operands and output (FYC_F16 storage). */
int32_t fyc_self_attention_tc_f16(const void* qk, int64_t ldqk, int64_t q_col0, int64_t k_col0, const void* vt, void* out,
                                  int64_t ldo, int64_t NB, int64_t heads, int64_t L, int64_t D, float scale, void* stream);
/* The same for head dim 80, L % 256 == 0 - the level-1 attn1 (1024 tokens at cfg2, 2304 at cfg5).  qkv: [NB, L, ldqkv] bf16, the fused
 * [q | k | v] projection UNPADDED: q head h at columns [q_col0 + 80 h, +80), k at [k_col0 + 80 h, +80); each head's second 64-column
 * TMA atom overlaps the next head, whose columns are never multiplied (QK^T issues 5 k-steps of 16), so the row only has to extend 48
 * columns past the last k head (the v block does).  vt: [NB, heads * 80, L]; out: [NB, L, ldo]. */
int32_t fyc_self_attention_tc_d80(const void* qkv, int64_t ldqkv, int64_t q_col0, int64_t k_col0, const void* vt, void* out,
                                  int64_t ldo, int64_t NB, int64_t heads, int64_t L, float scale, void* stream);
/* The same with fp16 operands and output. */
int32_t fyc_self_attention_tc_d80_f16(const void* qkv, int64_t ldqkv, int64_t q_col0, int64_t k_col0, const void* vt, void* out,
                                      int64_t ldo, int64_t NB, int64_t heads, int64_t L, float scale, void* stream);
/* Cross-attention against a SHORT, step-invariant context on the tensor cores (head dim 40, 64 or 80; bf16): attn2 of every transformer block
 * (diffusers/models/attention.py:649-678) and, with the second context, the whole IP-Adapter cross-attention in one launch
 * (animatediff/models/attention.py:92-120, ip_adapter/attention_processor.py:137-168):
 *   out[n, i, h D + :] = out_alpha softmax_{j < Lk}(scale q k^T) v + alpha2 softmax_{j < Lk2}(scale q k2^T) v2,   context n / kv_batch_div.
 * One CTA per (image, head) keeps K, V^T (and K2, V2^T) in shared memory and ping-pongs two softmax warpgroups over its query tiles; S and
 * O live in registers, the probabilities are normalised in registers (one key tile: no online rescaling) and both contexts accumulate into ONE
 * O accumulator, written once.  Operands, packed once per clip by the caller:
 *   q   [NB, Lq, ldq], head h at columns [q_col0 + D h, +D), unpadded (for D = 40 the 64-column q box of head h also holds the first 24
 *       columns of head h + 1, which meet the zero key columns 40..63: a NaN in those columns of head h + 1 makes head h's row NaN too;
 *       the box of the last head ends at column heads D, past which nothing is read);
 *   k   [NBc, 80, ldk], head h at columns [DKP h, +D) with DKP = 64 for D = 40 (columns D..63 of every head ZERO) | 64 for D = 64 | 80 for
 *       D = 80, rows Lk..79 zero;
 *   vt  [NBc, heads D, 80] (V transposed: keys contiguous), columns Lk..79 zero;
 *   k2  [NBc, 16, ldk2], vt2 [NBc, heads D, 16] likewise (NULL / Lk2 = 0: no second context). */
int32_t fyc_cross_attention_tc(const void* q, int64_t ldq, int64_t q_col0, const void* k, int64_t ldk, const void* vt, const void* k2,
                               int64_t ldk2, const void* vt2, void* out, int64_t ldo, int64_t NB, int64_t heads, int64_t Lq, int64_t D,
                               int64_t Lk, int64_t Lk2, int64_t kv_batch_div, float scale, float out_alpha, float alpha2, void* stream);
/* The same with fp16 operands and output. */
int32_t fyc_cross_attention_tc_f16(const void* q, int64_t ldq, int64_t q_col0, const void* k, int64_t ldk, const void* vt, const void* k2,
                                   int64_t ldk2, const void* vt2, void* out, int64_t ldo, int64_t NB, int64_t heads, int64_t Lq, int64_t D,
                                   int64_t Lk, int64_t Lk2, int64_t kv_batch_div, float scale, float out_alpha, float alpha2, void* stream);
/* in [NB, L, ld] columns [col0, col0 + C) (any 16-bit type: the values are moved, not converted) -> out [NB, C, L] */
int32_t fyc_transpose_tokens(const void* in, void* out, int64_t NB, int64_t L, int64_t C, int64_t ld, int64_t col0,
                             void* stream);
/* Row softmax of fp32 scores (VAE AttentionBlock, diffusers/models/attention.py:366), output in `dtype`. */
int32_t fyc_softmax_rows(const float* scores, void* probs, int64_t rows, int64_t L, int32_t dtype, void* stream);

/* ---- embeddings / glue --------------------------------------------------------------------------------*/
/* get_timestep_embedding (diffusers/models/embeddings.py:21-61): out[n, dim] fp32; freqs[dim/2] fp32 is
 * exp(-ln(1e4) k / (half - shift)) computed once on the host. */
int32_t fyc_timestep_embed(const int64_t* t, const float* freqs, float* out, int64_t n, int64_t dim,
                           int32_t flip_sin_to_cos, void* stream);
int32_t fyc_silu(const void* x, void* out, int64_t n, int32_t dtype, void* stream);
/* exact-erf GELU, elementwise (nn.GELU of the IP-Adapter Perceiver Resampler, ip_adapter/resampler.py:14-21) */
int32_t fyc_gelu(const void* x, void* out, int64_t n, int32_t dtype, void* stream);
/* GEGLU for the SIMT path: in [M, 2*Hd] (128-col granule interleave) -> out [M, Hd]. */
int32_t fyc_geglu(const void* in, void* out, int64_t M, int64_t Hd, int32_t dtype, void* stream);
int32_t fyc_upsample_nearest2x(const void* x, void* out, int64_t NB, int64_t H, int64_t W, int64_t C,
                               int32_t dtype, void* stream);
/* torch.cat([a, b], dim=channels) (unet_blocks.py:763,885): a [M, C1], b [M, C2] -> out [M, C1+C2]. */
int32_t fyc_concat_channels(const void* a, const void* b, void* out, int64_t M, int64_t C1, int64_t C2,
                            int32_t dtype, void* stream);
/* fp32 (b, c, f, h, w) <-> dtype [b, f, h, w, c]; the forward direction multiplies by `scale` in fp32 first
 * (1/0.18215 latent scaling of decode_latents, pipeline_animation.py:402). */
int32_t fyc_ncfhw_to_nfhwc(const float* in, void* out, int64_t B, int64_t C, int64_t F, int64_t HW, float scale,
                           int32_t dtype, void* stream);
/* `ldc` = channel stride of `in` in elements (0 or C: packed); ldc > C reads the first C of ldc channels - the 4-channel
 * conv_out head runs on the tensor cores with its output channels zero-padded to 16 (unet.py:351). */
int32_t fyc_nfhwc_to_ncfhw(const void* in, float* out, int64_t B, int64_t C, int64_t F, int64_t HW, int64_t ldc,
                           int32_t dtype, void* stream);
/* AnimationPipeline.__call__ step prologue (pipeline_animation.py:625-635,693-711): builds the channels-last
 * UNet input [dup*b, F, H, W, Cin] from latents (b,4,F,H,W) fp32, mask (b,1,1,H,W) fp32 (NULL -> 1 on frame 0)
 * and first-frame latents (b,4,H,W) fp32 (NULL -> Cin = 4, plain latents).  c_pad >= Cin: channels Cin..c_pad-1 are
 * written as zeros (lets the 9-channel stem run on the tensor-core path with a 16-channel, zero-extended filter). */
int32_t fyc_build_unet_input(const float* latents, const float* mask, const float* first, void* out, int64_t b,
                             int64_t F, int64_t HW, int32_t dup, int32_t c_pad, int32_t dtype, void* stream);
/* The same step prologue for the first-frame-conditioned motion models; `mode` is a bit set, first (b,4,H,W) fp32 the clean first-image
 * latents:
 *   FYC_FIRST_CONCAT (use_first_frame_condition_concat): out = [latents(4) | first(4) on every frame], Cin = 8.  Replaces the CFG
 *       duplication `torch.cat([latents] * 2)` (pipeline_animation.py:709) followed by the UNet's own concat of the duplicated
 *       first-image latents repeated over the frames (`torch.cat([first_image_latents] * 2)`, :717-719; unet.py:578-583);
 *   FYC_FIRST_FRAME (use_first_frame_condition): frame 0 of `latents` is overwritten IN PLACE with `first`, then out = latents, Cin = 4.
 *       Replaces `latents[:, :, 0, :, :] = first_image_latents` (pipeline_animation.py:691-692), which writes the tensor the DDIM step
 *       of the same iteration reads as its sample: the caller passes its persistent latents.
 * Both bits together do both (the reference runs that combination too).  Channels Cin..c_pad-1 are written as zeros. */
enum { FYC_FIRST_CONCAT = 1, FYC_FIRST_FRAME = 2 };
int32_t fyc_build_unet_input_first(float* latents, const float* first, void* out, int64_t b, int64_t F, int64_t HW, int32_t dup,
                                   int32_t mode, int32_t c_pad, int32_t dtype, void* stream);
/* Time-embedding row table of use_first_frame_condition (unet.py:523-524 appends a zero timestep, so emb has B + 1 rows; resnet.py:304-320
 * adds row B to frame 0 of every clip and row b to frames 1.. of clip b): temb [B + 1, N] fp32 (the fused time_emb_proj GEMV of all
 * ResnetBlock3Ds, t = 0 row last) -> out [B * F, N], out[b F + f] = temb[f == 0 ? B : b].  conv1 reads it as its row bias with
 * images_per_group = 1. */
int32_t fyc_first_frame_temb_rows(const float* temb, float* out, int64_t B, int64_t F, int64_t N, void* stream);
/* CFG combine + DDIMScheduler.step (pipeline_animation.py:763-764 + scheduling_ddim.py:308-349), fp32, exact
 * reference operation order (no FMA contraction).  pred: [2, n] (uncond, cond) when c->cfg_pair else [1, n]. */
typedef struct {
  float guidance;                 /* CFG scale (read only when cfg_pair != 0) */
  float sqrt_alpha_t, sqrt_beta_t, sqrt_alpha_prev, dir_coef, noise_coef;
  int32_t prediction_type, clip_sample;
  int32_t cfg_pair;               /* 1: pred holds [uncond; cond] (2n values) and n = u + guidance (c - u); 0: pred holds n values.  Set by the
                                     host from ITS decision `guidance_scale > 1.0` (a Python double: pipeline_animation.py:599) - the kernel must
                                     not re-derive it from the fp32-rounded `guidance`, which is 1.0f for every scale in (1, 1 + 2^-24] */
} fyc_ddim_coefs;
int32_t fyc_cfg_ddim_step(const float* pred, const float* sample, const float* noise, float* prev, int64_t n,
                          const fyc_ddim_coefs* c, void* stream);
/* The video_scale > 0 variant (pipeline_animation.py:738-761): `single` [n] is the UNet's prediction on the clip's frames
 * taken one at a time (F = 1, no temporal context); n = s + video_scale * (u - s) + guidance * (c - u), then the same step. */
int32_t fyc_cfg_video_ddim_step(const float* pred, const float* single, float video_scale, const float* sample,
                                const float* noise, float* prev, int64_t n, const fyc_ddim_coefs* c, void* stream);
/* decode_latents epilogue (pipeline_animation.py:409-410): x [b*F, HW, ldc >= 3] -> video (b, 3, F, H, W) fp32,
 * (x / 2 + 0.5).clamp(0, 1)  (ldc 0 or 3: packed RGB; 16 when the VAE's 3-channel head ran zero-padded on the tensor cores). */
int32_t fyc_frames_finalize(const void* x, float* video, int64_t b, int64_t F, int64_t HW, int64_t ldc, int32_t dtype,
                            void* stream);

/* Output side (SURVEY 8f row 4), save_videos_grid's tiling + 8-bit conversion (animatediff/utils/util.py:18-27): video (b, 3, F, H, W)
 * fp32 -> out [F, Hg, Wg, 3] uint8 where frame t tiles the b clips like torchvision.utils.make_grid(nrow, padding, pad_value 0)
 * (b == 1: the image unpadded; else xmaps = min(nrow, b), Hg = (H + padding) * ceil(b / xmaps) + padding, Wg alike) and each value is
 * trunc(((x + 1) / 2 if rescale else x) * 255). */
int32_t fyc_video_grid_u8(const float* video, uint8_t* out, int64_t b, int64_t F, int64_t H, int64_t W, int64_t nrow,
                          int64_t padding, int32_t rescale, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* FYC_H_ */
