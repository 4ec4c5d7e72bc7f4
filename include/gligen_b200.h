/* gligen_b200 C ABI  --  libgligen_b200.so
 *
 * Drop-in boundary for the GLIGEN per-timestep denoiser (SURVEY 8b).  The reference is pure
 * Python/PyTorch and has no FFI of its own; each entry point below replaces the torch library call(s)
 * the reference makes at the cited file:line (paths relative to the reference checkout).  Signatures
 * are plain C: device pointers, sizes, a cudaStream_t passed as void*.  No torch types cross the ABI.
 *
 * Conventions
 *   - every function returns 0 on success, <0 on error; glg_last_error() returns a thread-local message.
 *   - all work is enqueued on `stream`; nothing synchronises the device; every call is CUDA-graph
 *     capture safe (no allocation, no host sync) once the tensor-map cache is warm (first call per
 *     distinct (pointer, shape) creates a CUtensorMap on the host - also capture safe).
 *   - activations are bf16, channels-last: [B, H*W, C] == [B*T, C] row-major with an explicit leading
 *     dimension (ld, in elements) so that channel-concatenated buffers are addressed in place.
 *   - weights are bf16 [N, K] row-major (nn.Linear layout); 3x3 conv weights are packed [9][Cout][Cin].
 *   - statistics, biases, gates and sampler state are fp32.
 */
#ifndef GLIGEN_B200_H_
#define GLIGEN_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define GLG_ABI_VERSION 4

#define GLG_ACT_NONE 0
#define GLG_ACT_SILU 1
#define GLG_ACT_GELU 2        /* exact (erf) GELU: nn.GELU() of the ConvNeXt blocks (convnext.py:32) */
#define GLG_ACT_QUICK_GELU 3  /* x * sigmoid(1.702 x): the CLIP text encoder's MLP activation */

/* ---- library ------------------------------------------------------------------------------- */
int glg_abi_version(void);
const char* glg_last_error(void);
/* number of kernels launched by this library since load / since the last reset (bench gpu_launches). */
int64_t glg_launch_count(void);
void glg_reset_launch_count(void);

/* ---- tensor-core GEMM / implicit-GEMM convolution -------------------------------------------
 * out[M,N] = epilogue( A[M,K] * W[N,K]^T )      wgmma (bf16 x bf16 -> fp32 in registers), TMA-fed.
 *
 * Replaces: nn.Linear (attention.py:110-115,161-165,42,61,239), nn.Conv2d 1x1 (attention.py:349,360;
 * openaimodel.py:194), nn.Conv2d 3x3 stride 1 (openaimodel.py:157,183,70; conv_mode=1), the
 * PositionNet / time-embed MLPs (text_grounding_net.py:18-24, openaimodel.py:282-286,171-177).
 *
 * epilogue, in this order:  v = acc + bias[n] + rowbias[row / rows_per_batch][n];
 *                           v = act(v);   v *= *gate;   v += residual[row][n];
 * geglu=1 (attention.py:42-44): W/bias rows are packed per 256-row tile as [128 x-rows | 128 gate-rows]
 *   and out[M, N/2] = (x + bx) * gelu_erf(g + bg); act/gate/residual are not applied.
 * conv_mode=1: A is an NHWC activation [B, H, W, C=K] (ld = pixel stride); W is [9][N][K]; zero padding 1; any H, W.
 *
 * LayerNorm fold (attention.py:309-311,225-226 nn.LayerNorm feeding a Linear): with W' = W * gamma (per input
 *   channel, folded into W by the caller), colsum[n] = sum_k W'[n,k] and bias' = bias + W beta,
 *       LN(x) W^T + bias = rstd_r * (x W'^T - mu_r * colsum) + bias'
 *   so the GEMM runs on the RAW activations and the normalisation is two per-row scalars in the epilogue:
 *   ln_stats[ln_slots][rows][2] holds partial (sum, sum of squares) of every A row over its K columns (summed in
 *   slot order); they are produced for free by the GEMM that wrote A when its stats_out is set
 *   (stats_out[N/32][rows][2]: one partial per (row, 32-column chunk) of the bf16-rounded stored values - a layout
 *   independent of the tile shape, so results are bit-reproducible; slot-major so that the 32 rows a warp owns are
 *   contiguous).  No LayerNorm kernel, no normalised copy in HBM.
 * out_rows_per_batch > 0: output row r is written at (r / orpb) * out_batch_stride + (r % orpb) * ldc.
 * splitk_ws: when the tile grid would leave most SMs idle (M = 64 * batch at the 8x8 level) up to 8 CTAs share an
 *   output tile, each reducing a contiguous K range into an fp32 slab; a second kernel sums the slabs in a fixed
 *   order and applies the epilogue (deterministic).
 */
typedef struct GlgGemmArgs {
  const void* A;          /* bf16 */
  int64_t lda;            /* elements between consecutive rows (pixels) of A */
  const void* W;          /* bf16 [N(*9), K] row-major, contiguous */
  void* out;              /* bf16 (or fp32 if out_fp32) */
  int64_t ldc;
  int32_t M, N, K;
  int32_t out_fp32;
  const float* bias;      /* [N] or NULL */
  const float* rowbias;   /* [M / rows_per_batch, ld_rowbias] fp32 or NULL (ResBlock emb add, openaimodel.py:221-230) */
  int64_t ld_rowbias;
  int32_t rows_per_batch;
  int32_t act;            /* GLG_ACT_* */
  const float* gate;      /* device scalar (scale * tanh(alpha), attention.py:241-242) or NULL */
  const void* residual;   /* bf16 [M, ldr] or NULL */
  int64_t ldr;
  int32_t geglu;
  int32_t conv_mode;      /* 0 = plain GEMM, 1 = 3x3 stride-1 pad-1 convolution */
  int32_t H, Wd, Bn;      /* conv_mode: spatial dims and batch; M == Bn*H*Wd */
  const float* ln_stats;  /* LayerNorm fold: SLOT-major [ln_slots][ln_slot_stride rows][2] fp32 or NULL */
  const float* ln_colsum; /* [N] fp32 */
  int32_t ln_slots;
  float ln_eps;
  float* stats_out;       /* SLOT-major [stats_slots][stats_slot_stride rows][2] fp32 or NULL */
  int32_t stats_slots;
  int32_t out_rows_per_batch;
  int64_t out_batch_stride;
  void* splitk_ws;        /* optional fp32 scratch for split-K (small-M, long-K problems); NULL disables it */
  int64_t splitk_ws_bytes;
  int64_t ln_slot_stride;    /* rows between consecutive slots of ln_stats (0 = M): lets a consumer read a row range of a */
  int64_t stats_slot_stride; /* larger producer's statistics (the grounding-token streams) */
} GlgGemmArgs;
int glg_gemm(const GlgGemmArgs* args, void* stream);

/* ---- fused attention --------------------------------------------------------------------------
 * O[b, i, h*d:(h+1)*d] = softmax_j( Q[b,i,h,:] . K[b,j,h,:] * d^-1/2 ) V[b,j,h,:]      (flash style, online
 * softmax in fp32, scores never leave the SM).  Replaces the two einsums + softmax of
 * attention.py:142-146 (CrossAttention) and :180-183 (SelfAttention; also GatedSelfAttentionDense's
 * attention over [visual ; grounding] tokens with only the first Lq query rows kept, :241).
 * q/k/v are bf16 with independent row strides (elements) and batch strides so that packed QKV / KV
 * GEMM outputs are consumed in place.  d_head in {8,16,...,160}, multiple of 8.
 * Kernel selection (csrc/attention.cu): Lk <= 128 (the 77-token text context) -> K/V-resident mma.sync kernel;
 * longer key sets -> wgmma + TMA flash kernel.  All kernels give the same result to bf16 round-off
 * (tests/test_kernels_gpu.py::test_attention runs each against the same reference).
 */
typedef struct GlgAttnArgs {
  const void* q; const void* k; const void* v; void* out;   /* bf16 */
  int64_t q_row, k_row, v_row, o_row;        /* row strides (elements) */
  int64_t q_batch, k_batch, v_batch, o_batch;/* batch strides (elements) */
  int32_t B, heads, d_head, Lq, Lk;
  float scale;                               /* d_head^-0.5 */
  int32_t causal;                            /* ABI v4: 1 = query row i attends to keys [0, i] only (the CLIP text encoder's causal
                                                mask, transformers CLIPTextTransformer); needs Lk <= 128 (short-key kernel) */
} GlgAttnArgs;
int glg_attention(const GlgAttnArgs* args, void* stream);

/* ---- normalisation ---------------------------------------------------------------------------
 * GroupNorm over channels-last input (32 groups in the reference): fp32 statistics, affine, optional
 * SiLU, bf16 out.  Replaces GroupNorm32+SiLU (util.py:208-226, openaimodel.py:155-156,179-180,392-393;
 * eps 1e-5) and Normalize (attention.py:76-77; eps 1e-6, no SiLU).  `stats` is a caller-provided fp32
 * scratch of GLG_GN_SCRATCH_FLOATS(B, groups) floats whose first 128 words must be ZERO before the first call (they
 * hold the self-resetting counters of a sample-wide barrier inside the single kernel; per-CTA partial moments -
 * accumulated on data shifted by a per-group pivot, so large-mean activations do not cancel - are reduced in a fixed
 * order: results are bit-reproducible).  B <= 64.  One launch; the grid is sized so that all CTAs are co-resident.
 */
#define GLG_GN_SCRATCH_FLOATS(B, groups) (128 + 2 * (groups) * (8 * 148 + (B)))
int glg_groupnorm(const void* x, int64_t ldx, void* y, int64_t ldy, const float* gamma, const float* beta,
                  float* stats, int32_t B, int32_t HW, int32_t C, int32_t groups, float eps, int32_t silu,
                  void* stream);
/* LayerNorm over the last dim C (attention.py:309-311,225-226; eps 1e-5).  Row r of batch b is read at
 * x + b*x_batch + r*C and written at y + b*y_batch + r*C (lets the fuser build LN(cat[x, objs]) in place). */
int glg_layernorm(const void* x, int64_t x_batch, void* y, int64_t y_batch, const float* gamma, const float* beta,
                  int32_t B, int32_t rows, int32_t C, float eps, void* stream);

/* ---- data movement / small ops ------------------------------------------------------------- */
/* First conv: NCHW fp32 x (+ optional extra channels, inpainting openaimodel.py:444-447) -> NHWC bf16.
 * w fp32 packed [9][Cin][Cout] (tap-major), Cin = C0 + C1.  openaimodel.py:305,454. */
int glg_conv_in(const float* x, int32_t C0, const float* extra, int32_t C1, const float* w, const float* bias,
                void* out, int64_t ldo, int32_t B, int32_t H, int32_t Wd, int32_t Cout, void* stream);
/* Last conv: NHWC bf16 (already GN+SiLU'd) -> NCHW fp32 eps.  w fp32 packed [9][Cout][Cin], Cout in {3, 4, 8}.  openaimodel.py:391-395;
 * Cout = 3 is the VAE decoder's conv_out (model.py:529-533). */
int glg_conv_out(const void* x, int64_t ldx, const float* w, const float* bias, float* out,
                 int32_t B, int32_t H, int32_t Wd, int32_t Cin, int32_t Cout, void* stream);
/* nearest 2x upsample, NHWC bf16 (openaimodel.py:79 F.interpolate). */
int glg_upsample2x(const void* x, int64_t ldx, void* y, int64_t ldy, int32_t B, int32_t H, int32_t Wd, int32_t C, void* stream);
/* im2col for the 3x3 stride-2 pad-1 downsample conv (openaimodel.py:104-106): y[B*Ho*Wo, 9*C], k = tap*C + c. */
int glg_im2col_s2(const void* x, int64_t ldx, void* y, int32_t B, int32_t H, int32_t Wd, int32_t C, void* stream);
/* same with the zero padding chosen: pad_lo = 1 is glg_im2col_s2; pad_lo = 0 pads only right / bottom, which is the VAE
 * encoder's Downsample (ldm/modules/diffusionmodules/model.py:73-77: F.pad (0,1,0,1) then 3x3 stride-2 pad-0). */
int glg_im2col_s2_pad(const void* x, int64_t ldx, void* y, int32_t B, int32_t H, int32_t Wd, int32_t C, int32_t pad_lo, void* stream);
/* strided 2-D copy of bf16 rows: y[r, 0:C] = x[r, 0:C] (used to place skip tensors; C % 8 == 0). */
int glg_copy_rows(const void* x, int64_t ldx, void* y, int64_t ldy, int64_t rows, int32_t C, void* stream);
/* timestep_embedding (util.py:160-180): out bf16 [B, dim] = [cos(t f) | sin(t f)], f_k = exp(-ln(1e4) k / (dim/2)). */
int glg_timestep_embedding(const int64_t* t, void* out, int32_t B, int32_t dim, void* stream);
/* PositionNet input rows (text_grounding_net.py:33-45, text_image_grounding_net.py:44-60,
 * keypoint_grounding_net.py:38-55): out bf16 [B*N, F + P] = [feat*m_f + (1-m_f)*null_f | fourier(coords)*m + (1-m)*null_p]
 * feat: fp32 [B, N, F] (feat_batch_stride = 0 broadcasts one [N, F] table over the batch); coords fp32 [B, N, ncoord];
 * P = freqs*2*ncoord laid out per frequency as [sin(f*coords) | cos(f*coords)] (util.py:20-26);
 * rows have stride ldo >= F + P and columns [F+P, ldo) are zero (pads K to a multiple of 64 for glg_gemm). */
int glg_position_features(const float* feat, int64_t feat_batch_stride, const float* feat_mask, const float* null_feat,
                          const float* coords, const float* pos_mask, const float* null_pos, void* out, int64_t ldo,
                          int32_t B, int32_t N, int32_t F, int32_t ncoord, int32_t freqs, void* stream);
/* Row softmax: p[r, c] = softmax_c(scale * s[r, c]) as bf16 (fp32 scores in, rows normalised before rounding).  The VAE
 * decoder's single-head attention over H*W tokens (model.py:178-202: torch.bmm + softmax + torch.bmm; head dim 512).
 * cols, lds and ldp are multiples of 4; s is 16-byte and p 8-byte aligned. */
int glg_softmax_rows(const float* s, int64_t lds, void* p, int64_t ldp, int64_t rows, int32_t cols, float scale, void* stream);
/* fp32 -> bf16 cast of a contiguous buffer (context / weights staging). */
int glg_cast_f32_bf16(const float* x, void* y, int64_t n, void* stream);

/* ---- spatial grounding modalities: ConvNeXt tokenizer + grounding downsamplers (once per sample) --------------------
 * k x k stride-k patches as GEMM rows, so that Conv2d(k, stride=k) (convnext.py:71-72,79-81: stem 4x4/4, downsample 2x2/2) is a
 * glg_gemm with the weight packed [Cout, (ky, kx, c)]:  out[(b,oy,ox)][(ky*k+kx)*C + c], bf16, columns [k*k*C, ldo) zero.
 * _nchw: fp32 NCHW source resampled by nearest onto a virtual Hv x Wv grid first (F.interpolate(x, resize_input),
 *        hed_grounding_net.py:42 - fused here);  _nhwc: bf16 channels-last source (row stride ldx, C % 8 == 0). */
int glg_patchify_nchw(const float* x, void* out, int64_t ldo, int32_t B, int32_t C, int32_t Hs, int32_t Ws, int32_t Hv, int32_t Wv,
                      int32_t k, void* stream);
int glg_patchify_nhwc(const void* x, int64_t ldx, void* out, int64_t ldo, int32_t B, int32_t H, int32_t Wd, int32_t C, int32_t k, void* stream);
/* LayerNorm over the first C columns of `rows` strided bf16 rows (the channels_first LayerNorm of convnext.py:119-139 on a
 * channels-last tensor; two-pass statistics in registers); y columns [C, Cpad) are written as zeros (K padding). In place is fine. */
int glg_layernorm_rows(const void* x, int64_t ldx, void* y, int64_t ldy, const float* gamma, const float* beta, int64_t rows,
                       int32_t C, int32_t Cpad, float eps, void* stream);
/* same, fp32 output (no padding columns): the final LayerNorm of the CLIP text encoder -> last_hidden_state. */
int glg_layernorm_rows_f32(const void* x, int64_t ldx, float* y, int64_t ldy, const float* gamma, const float* beta, int64_t rows,
                           int32_t C, float eps, void* stream);
/* Text-encoder input rows (ldm/modules/encoders/modules.py:157-160 -> transformers CLIPTextEmbeddings):
 * out[b, l, :] = bf16(table[ids[b, l], :] + pos[l, :]);  ids int64 [B, L], table fp32 [vocab, C], pos fp32 [L, C]. */
int glg_embed_tokens(const int64_t* ids, const float* table, int64_t vocab, const float* pos, void* out, int64_t ldo, int32_t B, int32_t L,
                     int32_t C, void* stream);
/* Image-tower input rows (gligen_inference.py:151-153,110 -> transformers CLIPVisionEmbeddings.forward + CLIPVisionTransformer
 * pre_layrnorm): for image n of N with P patches, row n*(P+1) of x is LN(cls + pos[0]) and row n*(P+1)+1+p is
 * LN(patch[n*P + p] + pos[1+p]).  patch fp32 [N*P, ldp] (the patch-embedding GEMM's fp32 output), cls fp32 [C], pos fp32 [P+1, C];
 * the add is fp32, the statistics two-pass fp32, x bf16 rows of stride ldx.  One launch replaces cat + position add + LayerNorm. */
int glg_clip_vision_embed(const float* patch, int64_t ldp, const float* cls, const float* pos, const float* gamma, const float* beta,
                          void* x, int64_t ldx, int32_t N, int32_t P, int32_t C, float eps, void* stream);
/* Image-tower head, fp32 on CUDA cores, one CTA per image (transformers CLIPVisionTransformer pooled_output = post_layernorm(CLS),
 * CLIPVisionModelWithProjection visual_projection; gligen_inference.py:110 outputs.image_embeds, :114-116 the reprojection):
 *   pooled[n]  = LN(x[n*x_batch + 0 : C])                              (bf16 CLS row in, two-pass fp32 statistics)
 *   embeds[n]  = pooled[n] . w_proj^T                                  (w_proj fp32 [D, C], no bias)
 *   feature[n] = f * target_norm / |f|_2,  f = embeds[n] . proj        (proj fp32 [D, D] as torch.load('projection_matrix'); optional:
 *                                                                       proj and feature both NULL skips it)
 * Reductions run in a fixed order: results are bit-reproducible.  (C + D) * 4 bytes of shared memory, <= 48 KiB. */
int glg_clip_image_head(const void* x, int64_t x_batch, const float* gamma, const float* beta, const float* w_proj, const float* proj,
                        float target_norm, float* pooled, float* embeds, float* feature, int32_t N, int32_t C, int32_t D, float eps,
                        void* stream);
/* ConvNeXt block front (convnext.py:40-43): depthwise 7x7 pad 3 + bias, then LayerNorm over channels, one pass.
 * x / y NHWC bf16; w fp32 packed [49][C] (tap-major); y columns [C, Cpad) are zeros. */
int glg_dwconv7_ln(const void* x, int64_t ldx, void* y, int64_t ldy, const float* w, const float* bias, const float* gamma,
                   const float* beta, int32_t B, int32_t H, int32_t Wd, int32_t C, int32_t Cpad, float eps, void* stream);
/* Grounding tokens of a spatial map before the PositionNet MLP (hed_grounding_net.py:47-56): for the n tokens of sample b
 * y[b, t, :] = x[b, t, :] * mask[b] + null_feat * (1 - mask[b]) + pos[t, :]   (x, y bf16 rows; mask [B], null_feat [C], pos [n, C] fp32). */
int glg_spatial_tokens(const void* x, int64_t ldx, const float* mask, const float* null_feat, const float* pos, void* y, int64_t ldy,
                       int32_t B, int32_t n, int32_t C, void* stream);
/* F.interpolate on fp32 NCHW planes: y[B, C, Ho, Wo] from channels 0..C-1 of x (batch stride x_batch_stride elements).
 * mode 0 = nearest, 1 = bicubic (align_corners=False; hed/canny/depth/normal_grounding_downsampler.py). */
int glg_resize_plane(const float* x, int64_t x_batch_stride, float* y, int32_t B, int32_t C, int32_t Hs, int32_t Ws, int32_t Ho, int32_t Wo,
                     int32_t mode, void* stream);
/* Direct Conv2d with Cout in {3, 4, 8, 16} on fp32 NCHW (the downsamplers' Conv2d(.,.,4,2,1) pairs, sem_grounding_net.py:21
 * in_conv 3x3): the input is the source resampled by nearest onto a virtual Hv x Wv grid (Hv = Hs, Wv = Ws: as is);
 * w fp32 packed [Cin*k*k][Cout]; optional SiLU; y [B, Cout, Ho, Wo]. */
int glg_conv2d_small(const float* x, const float* w, const float* bias, float* y, int32_t B, int32_t Cin, int32_t Hs, int32_t Ws, int32_t Hv,
                     int32_t Wv, int32_t Cout, int32_t k, int32_t stride, int32_t pad, int32_t silu, void* stream);

/* ---- gatedSA2 fuser residual (attention.py:283-291: the grounding rows of the fuser's self-attention, reshaped to a g x g
 * grid, F.interpolate(mode='bicubic') onto the n x n visual grid, then the gated add x + scale*tanh(alpha_attn)*residual) ------
 *   x[b, y*n + x', c] = bf16( x[b, y*n + x', c] + gate[0] * bicubic_{g->n}(grid[b])[y, x', c] )      in place
 * grid fp32 [B][g*g][C] (row-major tokens, batch stride grid_batch_stride elements, 16-byte aligned); x bf16 rows b*n*n + p of
 * stride ldx (>= C, multiple of 8, 16-byte aligned); gate a device fp32 scalar (scale * tanh(alpha_attn)).  Bicubic as
 * glg_resize_plane: align_corners = False, A = -0.75, border-clamped taps (n < g is an unfiltered downsample, n == g the identity).
 * stats_out SLOT-major [C/32][stats_slot_stride rows][2]: per (row, 32-column slot) the sum and sum of squares of the stored
 * bf16 values - the stats_out contract of glg_gemm, so the norm2-folded FF GEMM that follows reads them as ln_stats.
 * C a multiple of 32, g <= 19. */
int glg_grid_resample_gate(const float* grid, int64_t grid_batch_stride, void* x, int64_t ldx, const float* gate, float* stats_out,
                           int64_t stats_slot_stride, int32_t B, int32_t g, int32_t n, int32_t C, void* stream);

/* ---- sampler update (plms.py:121-158, ddim.py:113-134), one fused fp32 kernel ---------------
 * e      = e_u + g*(e_c - e_u)                       (if e_uncond != NULL, else e = e_cond)
 * e'     = c0*e + c1*old1 + c2*old2 + c3*old3        (Adams-Bashforth / identity / improved Euler)
 * x_prev = sqrt(a_prev) * (x - sqrt(1-a_t) e')/sqrt(a_t) + sqrt(1-a_prev) * e'        (sigma = 0)
 * e_out (nullable) receives e (the CFG-combined epsilon, kept for the multistep history). */
int glg_sampler_update(const float* x, const float* e_cond, const float* e_uncond, float guidance,
                       const float* old1, const float* old2, const float* old3,
                       float c0, float c1, float c2, float c3,
                       float a_t, float a_prev, float* e_out, float* x_prev, int64_t n, void* stream);

/* ---- DPM-Solver++ multistep update (Lu et al. 2022, "DPM-Solver++: Fast Solver for Guided Sampling of Diffusion
 * Probabilistic Models", Algorithm 2), one fused fp32 kernel --------------------------------------------------------------
 * e      = e_u + g*(e_c - e_u)                       (if e_uncond != NULL, else e = e_cond)
 * x0_out = m0 = (x - sigma*e) / alpha                 data prediction at the evaluated timestep s0
 * x_prev = cx*x + k0*m0 + k1*m1 + k2*m2               (m1, m2 nullable: the two previous data predictions, read as 0)
 * alpha = sqrt(ac_s0), sigma = sqrt(1 - ac_s0).  With lambda = log(alpha/sigma), h = lambda_t - lambda_s0,
 * r0 = (lambda_s0 - lambda_s1)/h, r1 = (lambda_s1 - lambda_s2)/h, phi = -alpha_t expm1(-h), D1_0 = (m0 - m1)/r0,
 * D1_1 = (m1 - m2)/r1, the host expands into (cx, k0, k1, k2) (in float64, passed as fp32):
 *   order 1:  x_t = (sigma_t/sigma_s0) x + phi m0                                        (DDIM, eta = 0)
 *   order 2:  x_t = (sigma_t/sigma_s0) x + phi (m0 + D1_0/2)
 *   order 3:  x_t = (sigma_t/sigma_s0) x + phi m0 + alpha_t (expm1(-h)/h + 1) D1 - alpha_t ((expm1(-h) + h)/h^2 - 1/2) D2,
 *             D1 = D1_0 + r0/(r0 + r1) (D1_0 - D1_1), D2 = (D1_0 - D1_1)/(r0 + r1).
 * x0_out and x_prev must not alias any input or each other.  Any n >= 0; 16-byte-aligned pointers take 16-byte accesses. */
int glg_dpm_update(const float* x, const float* e_cond, const float* e_uncond, float guidance, const float* m1, const float* m2,
                   float alpha, float sigma, float cx, float k0, float k1, float k2, float* x0_out, float* x_prev, int64_t n, void* stream);

/* ---- UniPC predictor-corrector update (Zhao et al. 2023, "UniPC: A Unified Predictor-Corrector Framework for Fast Sampling
 * of Diffusion Models"; data prediction, B(h) = expm1(-h)), one fused fp32 kernel per step i ------------------------------
 * e      = e_u + g*(e_c - e_u)                                      (if e_uncond != NULL, else e = e_cond)
 * m_out  = m0 = (x - sigma*e) / alpha                                data prediction at point i (x = x_i)
 * xc_out = xc = cc*xc_prev + c0*m0 + c1*m1 + c2*m2 + c3*m3           UniC from point i-1 (xc_prev NULL: xc = x, the first step)
 * x_next = pc*xc + p0*m0 + p1*m1 + p2*m2                             UniP to point i+1, from the fp32 xc stored in xc_out
 * m1, m2, m3 (nullable, read as 0): the data predictions at points i-1, i-2, i-3.  alpha = sqrt(ac_i), sigma = sqrt(1 - ac_i).
 * With lambda = log(alpha/sigma), a step from s to t of order p has h = lambda_t - lambda_s, B = expm1(-h),
 * r_k = (lambda_{s-k} - lambda_s)/h, D_k = (m_{s-k} - m_s)/r_k (k < p), r_p = 1, R[a] = (r_1 .. r_p)^a and
 * b[a] = g_{a+1} (a+1)!/B with g_1 = B/(-h) - 1, g_{a+1} = g_a/(-h) - 1/(a+1)!; the host expands in float64 (passed as fp32)
 *   UniP:  x_t = (sigma_t/sigma_s) x_s - alpha_t B m_s - alpha_t B sum_k rhoP_k D_k
 *          rhoP = [] (p = 1), [1/2] (p = 2: DPM-Solver++ 2M), solve(R[:2,:2], b[:2]) (p = 3)
 *   UniC:  x_t = (sigma_t/sigma_s) x_s - alpha_t B m_s - alpha_t B (sum_{k<p} rhoC_k D_k + rhoC_p (m_t - m_s))
 *          rhoC = [1/2] (p = 1), solve(R, b) (p >= 2).
 * The outputs must not alias any input or each other.  Any n >= 0; 16-byte-aligned pointers take 16-byte accesses. */
int glg_unipc_update(const float* x, const float* xc_prev, const float* e_cond, const float* e_uncond, float guidance,
                     const float* m1, const float* m2, const float* m3, float alpha, float sigma,
                     float cc, float c0, float c1, float c2, float c3, float pc, float p0, float p1, float p2,
                     float* m_out, float* xc_out, float* x_next, int64_t n, void* stream);

/* ---- engine level: a whole UNet forward from an exported plan ----------------------------------
 * Replaces UNetModel.forward (openaimodel.py:420-464) for hosts that cannot embed Python.  gligen_b200/export.py writes one
 * (batch rows, grounding slots, context length) plan of the engine to a file: packed weights, workspace sizes and the ordered
 * op-level calls above with every pointer as (buffer, offset).  Named buffers: inputs "in:x" fp32 [rows,C,H,W], "in:t" int64
 * [rows], "in:context" fp32 [rows,77,768], "in:coords" / "in:masks" / "in:feat0" / "in:fmask0" (/ "in:feat1" / "in:fmask1",
 * "in:extra") as GroundingNetInput.prepare lays them out, "out" fp32 [rows,C,H,W]; weights "W:<name>" ("W:gates" holds
 * scale * tanh(alpha) per fuser, "W:conv_in.w" / "W:conv_in.b" the first conv that restore_first_conv_from_SD swaps).
 * glg_engine_load checks every op of the file against the calls above (name, argument count and kinds, struct sizes, every pointer
 * inside its buffer) before it allocates anything; a plan that fails a check is refused (< 0, glg_last_error names the op index and
 * the problem) and glg_engine_run only ever replays checked ops.
 * Not thread-safe per handle; all work is enqueued on `stream`; CUDA-graph capturable (no allocation inside run). */
typedef struct GlgEngine GlgEngine;
int glg_engine_load(const char* path, GlgEngine** out);
int glg_engine_buffer(GlgEngine* e, const char* name, void** dev_ptr, int64_t* bytes);
int glg_engine_write(GlgEngine* e, const char* name, const void* src, int64_t bytes, void* stream);   /* host or device src */
int glg_engine_read(GlgEngine* e, const char* name, void* dst, int64_t bytes, void* stream);
int glg_engine_run(GlgEngine* e, int32_t static_part, int32_t fuser_on, void* stream);
int64_t glg_engine_num_ops(GlgEngine* e);
int glg_engine_destroy(GlgEngine* e);

#ifdef __cplusplus
}
#endif
#endif /* GLIGEN_B200_H_ */
