/*
 * virtex_b200 -- C ABI of the H100-native (sm_90a) kernels behind the VirTex bicaptioning pretraining step.
 *
 * The reference (kdexd/virtex) has no FFI of its own: its hot path is `VirTexModel.forward` + autograd
 * (virtex/models/captioning.py:71-143) executed by torch / torchvision library calls (SURVEY.md section 8b).
 * Each entry point below replaces one family of those library calls; the file:line it stands in for is cited.
 *
 * Conventions
 *   - plain pointers + sizes, no torch types; every pointer is a DEVICE pointer unless stated otherwise
 *   - `stream` is a cudaStream_t passed as void*
 *   - returns 0 on success, a negative VTX_E* code on failure; vtx_last_error() gives a message (thread local)
 *   - no allocation, no synchronisation, no global state beyond cached device properties
 *   - activations are bf16 (NHWC for the backbone, [tokens, features] row-major for the head); statistics,
 *     master parameters, gradients and the decoder residual stream are fp32
 */
#ifndef VIRTEX_B200_H_
#define VIRTEX_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define VTX_OK 0
#define VTX_EINVAL (-1)
#define VTX_ECUDA (-2)
#define VTX_EUNSUPPORTED (-3)

const char* vtx_last_error(void);
int vtx_version(void);
/* Number of SMs of the current device (cached). */
int vtx_num_sms(void);

/* ------------------------------------------------------------------------------------------------------------------
 * wgmma GEMM:  D[M,N] = epilogue( sum_k A[m,k] * B[n,k] )       bf16 x bf16 -> fp32 accumulate in registers
 * Replaces every cuBLASLt / cuDNN GEMM-shaped call on the path: nn.Linear fwd/dgrad/wgrad
 * (virtex/modules/textual_heads.py:168-170,199,245,277; torch/nn/modules/transformer.py:1158-1199) and the 1x1 /
 * im2col'd convolutions of torchvision Bottleneck (torchvision/models/resnet.py:146-158).
 *   a_mn = 0: A is stored [M, K] row major (K contiguous, leading dim lda)     ("K-major")
 *   a_mn = 1: A is stored [K, M] row major (M contiguous, leading dim lda)     ("MN-major", used by wgrad)
 *   b_mn = 0: B is stored [N, K] row major;   b_mn = 1: B is stored [K, N] row major.
 * Epilogue order: acc -> (stats: per-column sum / sum of squares of acc, fp32 atomics) -> *alpha -> +bias[n]
 *                 -> +residual[m,n] (bf16) -> activation -> store (bf16 or fp32; or fp32 atomic accumulate).
 * split_k > 1 requires atomic = 1 (fp32 output, caller zero-initialises).
 * A bf16 output is stored by the TMA unit in 16-byte chunks: when N % 8 != 0, columns N .. round_up(N, 8) - 1 of every
 * output row are overwritten too, so D's rows must own that padding.
 * ------------------------------------------------------------------------------------------------------------------ */
typedef struct VtxGemm {
  const void* A;
  const void* B;
  void* D;
  const float* bias;    /* [N] or NULL */
  const void* residual; /* bf16 [M, ldr] or NULL */
  float* stats;         /* [2, N]: sum, sumsq  or NULL */
  int64_t lda, ldb, ldd, ldr;
  int32_t M, N, K;
  int32_t a_mn, b_mn;
  int32_t out_f32; /* 0: bf16 output, 1: fp32 output */
  int32_t atomic;  /* 1: D += result with fp32 atomics (needs out_f32) */
  int32_t act;     /* 0 none, 1 relu, 2 gelu(erf) */
  int32_t split_k; /* >= 1 */
  int32_t tile_n;  /* 0 = auto; else multiple of 16 (64 if b_mn) and <= 256 */
  float alpha;
  /* implicit 3x3 / stride 1 / pad 1 convolution over an NHWC bf16 tensor (conv_c > 0):
     A is the activation [conv_n, conv_h, conv_w, conv_c]; M = n*h*w, K = 9*conv_c, B = weights [N, (kh,kw,c)].
     conv_wgrad = 1 swaps roles for the weight gradient (see gemm_tc.cu). */
  int32_t conv_n, conv_h, conv_w, conv_c;
  int32_t conv_mode; /* 0 = plain GEMM, 1 = implicit fprop/dgrad gather on A (any conv_c -> N, 3x3 / stride 1 or 2),
                        2 = wgrad gather on B,
                        4 = wgrad for C = Cout = 64 in the transposed layout: A = dy, B = x, D[9*C, Cout] fp32 +=
                            (atomic), i.e. the TRANSPOSE of mode 2's [Cout, 9*C] output,
                        5 = 7x7/2 stem fprop over the space-to-depth view S written by vtx_stem_s2d: A = S
                            [conv_n, conv_h + 3, conv_w + 3, 16] (conv_h x conv_w = OUTPUT size, conv_c = 64 = 4 pixels
                            x 16 channels), B = packed weights [64, 256] (vtx_stem_s2d_w_pack), D [n*h*w, 64] NHWC
                            (torchvision resnet.py:197 conv1 forward, BN statistics through `stats`),
                        6 = stem wgrad: A = dy [conv_n, conv_h, conv_w, 64], B = S; D [64, 256] fp32 += (atomic) */
  int32_t conv_stride;          /* conv_mode 1 / 2 only: 0 or 1 = unit stride; 2 = stride-2 convolution -- conv_h / conv_w
                                   are the INPUT extent, outputs (M, K of the wgrad) run over (h-1)/2+1 x (w-1)/2+1; the
                                   gather uses TMA traversal strides (torchvision resnet.py:133-138, 239-243) */
  int32_t conv_taps;            /* 0 or 9 = 3x3 / pad 1 taps; 1 = a single tap (1x1 / pad 0: the strided downsample) */
  /* conv_mode 1, explicit tap grid (conv_taps_h > 0): conv_taps_h x conv_taps_w taps, tap (a, b) reads (h + a - conv_pad,
     w + b - conv_pad); K = taps * conv_c.  With the output view below this is one parity class of a stride-2 dgrad. */
  int32_t conv_taps_h, conv_taps_w, conv_pad;
  /* conv_mode 1, output view (conv_out_w > 0): D is the strided sub-grid [conv_n, conv_out_h, conv_out_w, N] of a larger
     NHWC tensor with element strides ldd_n / ldd_h / ldd_w (D points at its first element); rows of the conv_h x conv_w
     tile grid that fall outside the view are clipped. */
  int32_t conv_out_h, conv_out_w;
  int64_t ldd_w, ldd_h, ldd_n;
  const uint8_t* residual_mask; /* optional (bf16 output, N % 32 == 0; a plain GEMM, or conv_mode 1 without an output
                                   view, whose row m is the NHWC output pixel): bit (m, n) of a [M, N/8] bit mask in the
                                   layout vtx_bn_act writes; residual[m, n] is added only where the bit is set.  This is
                                   the shortcut gradient dz = dOut * [block output > 0] of a residual block without dz
                                   ever being written to memory (torchvision resnet.py:100-103, 160-161 backward): the
                                   1x1 conv1 dgrad of a bottleneck, the 3x3 conv1 dgrad of a basic block. */
  /* BatchNorm-backward reduction fused into the epilogue (bnr_y != NULL; bf16 output, N % 8 == 0, no bias / activation /
     stats): D is the gradient w.r.t. the output of a train-mode BN (+ReLU) whose pre-BN input is bnr_y (same geometry as
     D: leading dimension bnr_ldy, or D's view strides for conv_mode 1 output views) and whose forward parameters are
     bnr_bnp [4, N] = mean, invstd, scale, shift (vtx_bn_finalize).  With dz = D * mask, mask = bit (m, n) of bnr_mask
     (layout of vtx_bn_act's mask; plain GEMMs, or conv_mode 1 without an output view, rows as for residual_mask) or,
     when bnr_mask is NULL, [bnr_y * scale + shift > 0],
         bnr_sums[0, n] += sum_m dz[m, n],    bnr_sums[1, n] += sum_m dz[m, n] * (bnr_y[m, n] - mean[n]) * invstd[n]
     -- exactly what vtx_bn_bwd_reduce computes in a separate pass over D and y (torch batch_norm backward, first half);
     D itself is stored unmasked, vtx_bn_bwd_finalize_apply consumes the sums. */
  const void* bnr_y;
  const float* bnr_bnp;
  float* bnr_sums;
  const uint8_t* bnr_mask;
  int64_t bnr_ldy;
  /* Eval-mode BatchNorm folded into the epilogue (col_scale and col_shift both non-NULL, fp32 [N], 8-byte aligned): the
         D[m, n] = bf16( act( fmaf(acc, col_scale[n], col_shift[n]) + residual[m, n] ) )
     of a torchvision Bottleneck conv + BN (+ shortcut) (+ ReLU) in eval mode (torchvision resnet.py:146-163), with
     scale / shift = rows 2 / 3 of the bnp vtx_bn_finalize writes with training = 0.  Needs a bf16 output, alpha 1,
     act 0 or 1, N % 2 == 0, conv_mode 0 or 1 without an output view, no bias / stats / bnr_* / residual_mask, and a
     residual (optional) that is 16-byte aligned with ldr % 8 == 0; anything else is rejected.  Both NULL: the epilogue
     order above. */
  const float* col_scale;
  const float* col_shift;
} VtxGemm;

int vtx_gemm(const VtxGemm* g, void* stream);
/* Tile schedule of the persistent GEMM.  0 (default): static round robin, tile t of CTA c = c + i * #CTAs -- the fastest
   when the GEMM has the GPU to itself.  1: every CTA takes its tiles from a per-launch atomic counter, so that an SM held
   by another stream's kernel (NCCL's all-reduce CTAs during the overlapped gradient exchange of the data-parallel step,
   scripts/pretrain_virtex.py:121-123) does not own a fixed share of every GEMM issued meanwhile.  Process-wide. */
int vtx_gemm_set_dynamic_schedule(int on);
/* sizeof(VtxGemm) of the built library (a binding compares it with its own struct definition) */
int vtx_sizeof_gemm(void);

/* ------------------------------------------------------------------------------------------------------------------
 * Backbone auxiliaries (NHWC bf16 activations).  Replace cuDNN BatchNorm / ATen elementwise + pooling kernels called by
 * torchvision/models/resnet.py:143-163,268-276 and the im2col side of strided convolutions.
 * ------------------------------------------------------------------------------------------------------------------ */
/* 7x7/stride 2/pad 3 stem: image fp32 NCHW -> cols bf16 [N*Ho*Wo, ldc], k = (kh*7+kw)*3 + c, zero padded to ldc */
int vtx_stem_im2col(const float* img, void* cols, int N, int H, int W, int ldc, void* stream);
/* space-to-depth view of the image for the 4-tap implicit stem conv (vtx_gemm conv_mode 5 / 6):
   image fp32 NCHW [N, 3, H, W] -> S bf16 [N, H/2 + 3, W/2 + 3, 16],
   S[n, i, j, (r*2+q)*3 + c] = img[n, c, 2i + r - 3, 2j + q - 3], zero outside the image and in channels 12..15 */
int vtx_stem_s2d(const float* img, void* S, int N, int H, int W, void* stream);
/* conv1.weight fp32 [O, 3, 7, 7] -> bf16 [O, 256], k = a*64 + b*16 + (r*2+q)*3 + c for tap (kh, kw) = (2a+r, 2b+q) */
int vtx_stem_s2d_w_pack(const float* w, void* wp, int O, void* stream);
/* grad fp32 [O, 3, 7, 7] += dwp fp32 [O, 256] (same index map) */
int vtx_stem_s2d_w_unpack_add(const float* dwp, float* grad, int O, void* stream);
/* 3x3 / pad 1 / given stride: x [N,H,W,C] -> cols [N*Ho*Wo, 9*C] (k = tap*C + c) and its adjoint */
int vtx_im2col3x3(const void* x, void* cols, int N, int H, int W, int C, int stride, void* stream);
int vtx_col2im3x3(const void* dcols, void* dx, int N, int H, int W, int C, int stride, void* stream);
/* strided 1x1 (downsample) gather and its adjoint (dx += scatter(dxs)) */
int vtx_subsample(const void* x, void* xs, int N, int H, int W, int C, int stride, void* stream);
int vtx_upsample_add(const void* dxs, void* dx, int N, int H, int W, int C, int stride, void* stream);
/* stats [2,C] (sum, sumsq from the GEMM epilogue) -> bnp [4,C] = mean, invstd, scale, shift; updates running stats */
int vtx_bn_finalize(const float* stats, float count, const float* gamma, const float* beta, float* running_mean,
                    float* running_var, int64_t* num_batches_tracked, float momentum, float eps, int training,
                    float* bnp, int C, void* stream);
/* out = act(y*scale + shift [+ res | + res*scale_r + shift_r]).  relu_mask (optional, relu only): uint8 [M, C/8], bit j
   of byte (m, g) = [pre-activation of channel 8g + j > 0] -- all that BN backward needs of `out` (1/16 of its bytes).
   C/8 must divide 256 (C = 8, 16, 32, ..., 2048); any other C is rejected with VTX_EINVAL. */
int vtx_bn_act(const void* y, const float* bnp, const void* res, const float* bnp_res, void* out, uint8_t* relu_mask,
               int64_t M, int C, int relu, void* stream);
/* vtx_bn_finalize + vtx_bn_act fused into one launch; C/8 must divide 256, as for vtx_bn_act */
int vtx_bn_finalize_act(const float* stats, float count, const float* gamma, const float* beta, float* running_mean,
                        float* running_var, int64_t* num_batches_tracked, float momentum, float eps, int training,
                        float* bnp, const void* y, const void* res, const float* bnp_res, void* out, uint8_t* relu_mask,
                        int64_t M, int C, int relu, void* stream);
int vtx_bn_relu_maxpool(const void* y, const float* bnp, void* out, uint8_t* idx, int N, int H, int W, int C,
                        void* stream);
int vtx_maxpool_bwd(const void* dpool, const uint8_t* idx, void* da, int N, int H, int W, int C, void* stream);
/* BN backward in three steps: per-channel sums of dz and dz*xhat (dz = dA*[relu_mask bit]); coefficients + dgamma/dbeta;
   dy = scale*(dz - mean(dz) - xhat*mean(dz*xhat)).  A second BN sharing dz (downsample branch) rides along.
   relu_mask: the uint8 bit mask written by vtx_bn_act / vtx_bn_finalize_act, or NULL;
   relu_mask == NULL && mask_from_y: the ReLU mask is recomputed as [y*scale + shift > 0] instead of being read.
   vtx_bn_bwd_reduce takes any C % 8 == 0 with C/8 <= 256; vtx_bn_bwd_apply and vtx_bn_bwd_finalize_apply need C/8 to
   divide 256 (C = 8, 16, 32, ..., 2048) and reject any other C with VTX_EINVAL. */
int vtx_bn_bwd_reduce(const void* dA, const uint8_t* relu_mask, const void* y, const float* bnp, const void* y2,
                      const float* bnp2, float* sums, float* sums2, int64_t M, int C, int mask_from_y,
                      void* stream);
int vtx_bn_bwd_finalize(const float* sums, const float* bnp, float count, float* coef, float* dgamma, float* dbeta,
                        int C, void* stream);
int vtx_bn_bwd_apply(const void* dA, const uint8_t* relu_mask, const void* y, const float* bnp, const float* coef, void* dy,
                     const void* y2, const float* bnp2, const float* coef2, void* dy2, void* dz_out, int64_t M, int C,
                     int mask_from_y, void* stream);
/* vtx_bn_bwd_finalize + vtx_bn_bwd_apply fused into one launch (dgamma/dbeta accumulated by the first thread block) */
int vtx_bn_bwd_finalize_apply(const float* sums, const float* sums2, float count, float* dgamma, float* dbeta,
                              float* dgamma2, float* dbeta2, const void* dA, const uint8_t* relu_mask, const void* y,
                              const float* bnp, void* dy, const void* y2, const float* bnp2, void* dy2, void* dz_out,
                              int64_t M, int C, int mask_from_y, void* stream);
/* conv weight layouts: fp32 OIHW <-> bf16 [O, (kh,kw,I)] GEMM operand; flipped/transposed dgrad operand */
int vtx_conv_w_pack(const float* w, void* out, int O, int I, int KH, int KW, int ldk, void* stream);
int vtx_conv_w_pack_dgrad(const float* w, void* out, int O, int I, void* stream);
int vtx_conv_w_unpack_add(const float* dwp, float* grad, int O, int I, int KH, int KW, int ldk, void* stream);
/* same for the transposed [(tap, I), O] weight-gradient layout written by vtx_gemm conv_mode 4 */
int vtx_conv_w_unpack_add_t(const float* dwt, float* grad, int O, int I, int KH, int KW, void* stream);
/* Batched form of the six weight-layout kernels above (and of vtx_stem_s2d_w_pack / _unpack_add): one launch executes a
   DEVICE-resident table of jobs.  kind: 0 pack, 1 pack_dgrad, 2 unpack_add, 3 unpack_add_t, 4 stem s2d pack,
   5 stem s2d unpack_add, 6 pack for parity class (KH, KW) of a stride-2 3x3 dgrad ([I, taps*O], see backbone.cu), 7 transpose of a 1x1 weight ([O, I] -> bf16 [I, O]); total = number of output elements of the job; block0 = first thread block of the job (jobs are
   sorted by block0, every block handles vtx_weight_job_block_elems() consecutive elements). */
typedef struct VtxWeightJob {
  const void* src;
  void* dst;
  int64_t total;
  int32_t O, I, KH, KW, ldk, kind, block0, reserved;
} VtxWeightJob;
int vtx_conv_w_jobs(const VtxWeightJob* jobs, int njobs, int total_blocks, void* stream);
int vtx_weight_job_block_elems(void);
int vtx_cast_bf16(const float* in, void* out, int64_t n, void* stream);
int vtx_nhwc_to_nchw_f32(const void* in, float* out, int N, int HW, int C, void* stream);

/* ------------------------------------------------------------------------------------------------------------------
 * Textual-head auxiliaries.  `seed` is a DEVICE pointer to the 64-bit dropout seed of the current step (so a captured
 * CUDA graph can be replayed with fresh masks); `site` distinguishes dropout call sites; p = 0 disables dropout.
 * Replace nn.Embedding/LayerNorm/Dropout (virtex/modules/embedding.py:58-73), F.scaled_dot_product_attention with
 * the merged float mask (torch/nn/functional.py:6608-6682), GELU, nn.CrossEntropyLoss (virtex/models/captioning.py:69).
 * ------------------------------------------------------------------------------------------------------------------ */
int vtx_embed_fwd(const int64_t* tokens, const float* words, const float* positions, const float* gamma,
                  const float* beta, float* z, float* stats, float* out, void* out_bf, int M, int T, int H, int pad,
                  float eps, float p, const uint64_t* seed, uint32_t site, void* stream);
int vtx_embed_bwd(const float* dy_a, const void* dy_b, const int64_t* tokens, const float* z, const float* stats,
                  const float* gamma, float* d_words, float* d_pos, float* d_gamma, float* d_beta, int M, int T, int H,
                  int pad, float p, const uint64_t* seed, uint32_t site, void* stream);
/* z = res + dropout(branch); out = LN(z) (ln=1) or z (ln=0) */
int vtx_add_ln_fwd(const float* res, const void* branch, const float* gamma, const float* beta, float* z, float* stats,
                   float* out, void* out_bf, int M, int H, float eps, float p, const uint64_t* seed, uint32_t site,
                   int ln, void* stream);
int vtx_ln_bwd(const float* dy_a, const void* dy_b, const float* z, const float* stats, const float* gamma,
               const float* d_skip, float* d_res, void* d_branch, float* d_gamma, float* d_beta, int M, int H, float p,
               const uint64_t* seed, uint32_t site, int ln, void* stream);
/* Attention core, head_dim 64, 1 <= Tq, Tk <= VTX_ATTN_MAX_T (larger shapes: VTX_EINVAL); bf16 q / k / v / out with
   leading dimensions that are multiples of 8.  causal = 1: key j visible to query i iff j <= i and j < lengths[b];
   causal = 2: iff j < lengths[b] (key-padding mask only: masked language modelling); causal = 0: every key.
   With Qs = Tq rounded up to a multiple of 32 and Ks = Tk rounded up to a multiple of 64, `lse` holds B * heads * Qs
   fp32 rows (row (b * heads + h) * Qs + i; rows i >= Tq are not written) and the dropout mask of the probabilities is
   the counter hash of element ((b * heads + h) * Qs + i) * Ks + j.  Tq <= 32 and Tk <= 64 run on one warp per
   (b, h); longer shapes stream 64-row tiles (one CTA per (b, h, 64 queries) forward, per (b, h) backward).  Both are
   deterministic and allocate nothing. */
#define VTX_ATTN_MAX_T 1024
int vtx_attn_fwd(const void* q, int64_t ldq, const void* k, int64_t ldk, const void* v, int64_t ldv, void* out,
                 int64_t ldo, float* lse, int B, int heads, int Tq, int Tk, const int64_t* lengths, int causal,
                 float p, const uint64_t* seed, uint32_t site, void* stream);
int vtx_attn_bwd(const void* q, int64_t ldq, const void* k, int64_t ldk, const void* v, int64_t ldv, const void* dout,
                 int64_t ldo, const float* lse, void* dq, int64_t lddq, void* dk, int64_t lddk, void* dv, int64_t lddv,
                 int B, int heads, int Tq, int Tk, const int64_t* lengths, int causal, float p, const uint64_t* seed,
                 uint32_t site, void* stream);
int vtx_gelu_dropout_fwd(const void* u, void* h, int64_t n, float p, const uint64_t* seed, uint32_t site, void* stream);
int vtx_gelu_dropout_bwd(const void* dh, const void* u, void* du, int64_t n, float p, const uint64_t* seed,
                         uint32_t site, void* stream);
/* shift = 1: the target of position t is tokens[b, t+1] (captioning.py:111-114); shift = 0: tokens[b, t] is the label of
   position t itself (masked_labels of virtex/models/masked_lm.py:68-72).  Targets equal to pad are ignored. */
int vtx_count_valid(const int64_t* tokens, int B, int T, int pad, int shift, float* count, void* stream);
/* logits bf16 [B*T, ldl]; loss += mean NLL over valid targets; write_grad: logits := dlogits in place */
int vtx_cross_entropy(void* logits, int64_t ldl, const int64_t* tokens, int B, int T, int V, int pad, int shift,
                      const float* count, float* loss, int write_grad, void* stream);
int vtx_colsum(const void* X, int64_t ld, int M, int N, float* out, void* stream);
int vtx_argmax_rows(const float* X, int64_t ld, int M, int N, int64_t* out, void* stream);

/* ------------------------------------------------------------------------------------------------------------------
 * Classification pretext heads (csrc/classify.cu): LinearTextualHead's global average pool and the K-hot loss of
 * ClassificationModel (virtex/modules/textual_heads.py:46-95, virtex/models/classification.py:43-108).  The linear layer
 * is vtx_gemm; its bf16 logits use a leading dimension of V rounded up to 8 (the GEMM's bf16 row alignment).
 * ------------------------------------------------------------------------------------------------------------------ */
/* pooled bf16 [B, C] = mean over the HW rows of each image of feat bf16 [B*HW, C] (NHWC backbone output), fp32 sums;
   C % 8 == 0 */
int vtx_group_mean_fwd(const void* feat, void* pooled, int B, int HW, int C, void* stream);
/* dfeat bf16 [B*HW, C] = dpooled[b, c] / HW for every row of image b */
int vtx_group_mean_bwd(const void* dpooled, void* dfeat, int B, int HW, int C, void* stream);
/* Largest V the loss's shared-memory label bitmap covers; a larger V is rejected with VTX_EUNSUPPORTED. */
#define VTX_KHOT_MAX_V 65536
/* K-hot cross entropy over bf16 logits [B, ldl] (V valid columns) and int64 labels [B, ldlab] (L used columns).
   U_b = distinct labels of row b in [0, V) that are not in the device array ignore[n_ignore]; labels outside [0, V)
   are skipped, never read as a column.  loss[0] += (1/B) * (logsumexp_b - mean_{u in U_b} z[b, u]), which is NaN for
   an empty U_b.  write_grad: logits := (softmax - [v in U_b] / |U_b|) / B in place, a zero row for an empty U_b. */
int vtx_khot_xent(void* logits, int64_t ldl, const int64_t* labels, int64_t ldlab, int B, int L, int V,
                  const int64_t* ignore, int n_ignore, float* loss, int write_grad, void* stream);
/* out int64 [M, k] = column indices of the k largest values of each row of fp32 X [M, ld] (N columns), in descending
   order; equal values in ascending index order; NaN ranks as -inf.  Needs k <= N. */
int vtx_topk_rows(const float* X, int64_t ld, int M, int N, int k, int64_t* out, void* stream);

/* ------------------------------------------------------------------------------------------------------------------
 * Incremental beam-search decoding (csrc/decode.cu): AutoRegressiveBeamSearch over CaptioningModel.decoding_step
 * (virtex/utils/beam_search.py:52-238, virtex/models/captioning.py:144-213) with a key/value cache instead of a full
 * recompute per step.  Step tables are step-major: pred int64 [steps, R] and index int32 [steps, R], R = B * beam, so
 * that step t of every row is one contiguous row (the token input of the next step's vtx_embed_fwd with T = 1).
 * ------------------------------------------------------------------------------------------------------------------ */
#define VTX_DECODE_MAX_KEYS 64
/* One query per row, head_dim 64, 1 <= Tk <= VTX_DECODE_MAX_KEYS keys, no mask, no dropout.  Query row m = b * group + g
   (g < group) of head h attends over the Tk keys of block b:
       key j  = k + blk * ldb + j * ldkv + 64 h,   value j = v + blk * ldb + j * ldkv + 64 h,
       blk    = b, or kv_index[j * ld_index + b] when kv_index != NULL (needs group == 1),
   out[m, 64h .. 64h+63] = softmax_j(q_m . key_j / 8) . value_j (fp32 softmax, bf16 output).
   Self-attention over the cache: group 1, ldb = the cache's row stride, kv_index = the step-major index table.
   Cross-attention: group = beam, Tk = h * w, ldb = Tk * ldkv over K|V projected once per image. */
int vtx_attn_decode(const void* q, int64_t ldq, const void* k, const void* v, int64_t ldkv, int64_t ldb,
                    const int32_t* kv_index, int64_t ld_index, void* out, int64_t ldo, int blocks, int heads, int group,
                    int Tk, void* stream);
/* Row half of a beam step, one row of fp32 logits [R, ldl] (V columns, bias included) per CTA: scores = log_softmax
   in fp32, then exactly -10000 at the row's last token last[row], then -- when last[row] == eos -- 0 at eos and -inf
   elsewhere, unnormalised (beam_search.py:152-172).  last == NULL: log_softmax only (the first step).  Writes the k
   best scores and their columns, cand_val fp32 / cand_idx int32 [R, k], in descending order, equal scores in ascending
   column order (as vtx_topk_rows); NaN ranks as -inf.  k <= min(V, 32). */
int vtx_beam_rows(const float* logits, int64_t ldl, int R, int V, const int64_t* last, int eos, int k, float* cand_val,
                  int32_t* cand_idx, void* stream);
/* Image half of a beam step, one warp per image b < B.  Candidate c < parents * k of image b is row candidate c % k of
   parent row p = b * parents + c / k, scored cand_val + scores_in[p] (0 when scores_in is NULL).  The beam best
   candidates (descending, ties in ascending c) become rows i = b * beam + r:
       scores_out[i] = score,  parent_out[i] = p (optional),  pred_out[s, i] = cand_idx,  index_out[s, i] = i,
       pred_out[j, i] = pred_in[j, p] and index_out[j, i] = index_in[j, p] for j < s,
   and alive[s] = 1 if any new token is not eos (alive is zeroed by the caller).  scores_in may alias scores_out;
   the tables may not alias (ping-pong them).  beam <= parents * k <= 32. */
int vtx_beam_select(const float* cand_val, const int32_t* cand_idx, int parents, int k, int beam, const float* scores_in,
                    float* scores_out, int32_t* parent_out, const int64_t* pred_in, int64_t* pred_out,
                    const int32_t* index_in, int32_t* index_out, int B, int s, int eos, int32_t* alive, void* stream);
/* One step of nucleus sampling (AutoRegressiveNucleusSampling, virtex/utils/nucleus_sampling.py:58-115), one row of
   fp32 logits [R, ldl] (V columns) per CTA, last token last[row].  In (descending value, ascending column) order, with
   fp32 probabilities from a one-pass log-sum-exp, the nucleus keeps every token whose preceding cumulative probability
   is <= p (the first token always); the last token is then banned, and the new token is drawn from the softmax of
   the remaining nucleus by the inverse CDF in ascending column order at the uniform
       u = (hash_u64(*seed, 4000, s * R + row) >> 40) / 2^24        (vtx_common.cuh; 24 bits, exact in fp32).
   When the nucleus is the last token alone, every logit is -1e12 in the reference and the draw is uniform over all
   V tokens: floor(u * V).  A row whose last token is eos draws eos.  Writes pred[s * R + row] of the step-major int64
   table [steps, R] and sets alive[s] = 1 if the new token is not eos (alive is zeroed by the caller).  Cumulative
   masses are fixed-point integers: bitwise deterministic for a seed.  The seed is read on the device, so a captured
   launch stays valid.  0 <= p <= 1, V <= VTX_NUCLEUS_MAX_V (the row is staged in shared memory). */
#define VTX_NUCLEUS_MAX_V 32768
int vtx_nucleus_sample(const float* logits, int64_t ldl, int R, int V, const int64_t* last, int eos, float p,
                       const uint64_t* seed, int s, int64_t* pred, int32_t* alive, void* stream);

/* ------------------------------------------------------------------------------------------------------------------
 * GPU input pipeline (csrc/input_pipe.cu): decoded uint8 HWC images -> fp32 NCHW network input, token lists -> padded
 * matrices.  Replaces the per-sample albumentations / cv2 transforms and the collate of
 * virtex/data/datasets/captioning.py:51-100 with the transform lists of virtex/factories.py:131-155.  Random parameters
 * are sampled on the host.  src: all images of the batch back to back (uint8, RGB, HWC), image n at src + src_off[n];
 * geom_i [B,8] = {H, W, region y0, x0, h, w, window offset y, x}; geom_d [B,2] = {region h / resized h, region w /
 * resized w}; jit_i [B,6] = {flip, apply-jitter, op order[4] (0 brightness, 1 contrast, 2 saturation, 3 hue)};
 * jit_d [B,4] = the four factors.  Integer paths are bit-exact with OpenCV's uint8 resize / cvtColor / addWeighted.
 * ------------------------------------------------------------------------------------------------------------------ */
/* crop + cv2.resize(INTER_LINEAR) (+ horizontal flip): out uint8 [B, S, S, 3] */
int vtx_image_resample(const uint8_t* src, const int64_t* src_off, const int32_t* geom_i, const double* geom_d,
                       const int32_t* jit_i, uint8_t* out, int B, int S, void* stream);
/* gray_sum[n] += sum of grey values of image n at the contrast stage of its jitter (caller zero-initialises) */
int vtx_image_gray_sum(const uint8_t* img, const int32_t* jit_i, const double* jit_d, uint64_t* gray_sum, int B, int S,
                       void* stream);
/* colour jitter in the sampled op order + (v - mean*255) / (std*255), written as fp32 NCHW; norm = {m[3], 1/s[3]} */
int vtx_image_jitter_normalize(const uint8_t* img, const int32_t* jit_i, const double* jit_d, const uint64_t* gray_sum,
                               const float* norm, float* out, int B, int S, void* stream);
/* flat token ids + offsets [B+1] -> caption / reversed caption [B, T] right-padded with pad, lengths [B] (<= max_len) */
int vtx_collate_tokens(const int64_t* flat, const int64_t* offs, int64_t* cap, int64_t* rev, int64_t* lengths, int B,
                       int T, int max_len, int64_t pad, void* stream);
/* The masked-LM collate (MaskedLmDataset.__getitem__ + collate_fn, virtex/data/datasets/masked_lm.py:64-119): the
   trim + right-pad of vtx_collate_tokens into cap, then, per caption of trimmed length n, k = ceil((n - 2) * proportion)
   (float64) distinct positions of 1 .. n-2 -- the k smallest (key, position), key = hash_u64(*seed, 5000, ctr) -- each
   turned into mask_id with labels = the original id when k == 1 or u <= mask_prob, into the id
   mulhi(hash_u64(*seed, 5002, ctr), vocab) of [0, vocab) when u <= mask_prob + replace_prob (float64 sum), and left
   as it is otherwise; u = (hash_u64(*seed, 5001, ctr) >> 11) * 2^-53, ctr = caption << 32 | position.  labels [B, T]
   holds pad everywhere else.  The seed is read on the device.  T <= VTX_MLM_MAX_T (one CTA per caption); proportion,
   mask_prob and replace_prob in [0, 1]; vocab > 0. */
#define VTX_MLM_MAX_T 1024
int vtx_collate_masked_lm(const int64_t* flat, const int64_t* offs, int64_t* cap, int64_t* labels, int64_t* lengths,
                          int B, int T, int max_len, int64_t pad, int64_t mask_id, int64_t vocab, double proportion,
                          double mask_prob, double replace_prob, const uint64_t* seed, void* stream);

/* ------------------------------------------------------------------------------------------------------------------
 * JPEG decoding (csrc/jpeg.cu): compressed baseline / extended-sequential Huffman JPEGs -> uint8 HWC RGB, bit-exact
 * with cv2.cvtColor(cv2.imdecode(buf, IMREAD_COLOR), COLOR_BGR2RGB), the reference's image reads.  One interleaved
 * scan, 8-bit, 1 component or YCbCr with luma sampling 1x1 / 2x1 / 1x2 / 2x2 and 1x1 chroma, restart markers optional.
 * The host parses the headers (virtex_b200/jpeg.py) into, per image n:
 *   info int32 [B, VTX_JPEG_NI]: the VTX_JPEG_I_* fields; component c at VTX_JPEG_I_COMP + 8c = {h, v, quant table,
 *     DC table, AC table (indices into quant / huff), blocks per plane row, plane rows of blocks, first block in MCU}
 *   info64 int64 [B, VTX_JPEG_N64]: the VTX_JPEG_Q_* byte / block offsets
 *   quant uint16 [*, 64] in natural order;  huff: VTX_JPEG_HUFF_BYTES per table (layout in csrc/jpeg.cu)
 * Workspaces (sized from the headers by the caller): ent (unstuffed bytes, >= entropy length per image), segments
 * (seg_start, seg_len, seg_chunk0: VTX_JPEG_I_NSEG per image), chunk slots (VTX_JPEG_I_CHUNK_CAP per image: two
 * state buffers of int4 and one int32 scan), coef int16 [blocks, 64] (zeroed), planes uint8.  status int32 [B]
 * (zeroed) collects VTX_JPEG_ST_* bits; rounds int32 [B] (zeroed) the last synchronisation round that changed a chunk.
 * ------------------------------------------------------------------------------------------------------------------ */
#define VTX_JPEG_NI 48
#define VTX_JPEG_I_H 0           /* frame height, width */
#define VTX_JPEG_I_W 1
#define VTX_JPEG_I_ORIENT 2      /* EXIF orientation 1..8 */
#define VTX_JPEG_I_NCOMP 3
#define VTX_JPEG_I_MCUX 4        /* MCUs per row, MCU rows */
#define VTX_JPEG_I_MCUY 5
#define VTX_JPEG_I_RI 6          /* restart interval in MCUs, 0 = none */
#define VTX_JPEG_I_BPM 7         /* blocks per MCU */
#define VTX_JPEG_I_NSEG 8        /* restart segments = ceil(MCUs / RI), 1 without restarts */
#define VTX_JPEG_I_SEG_BASE 9    /* first segment slot of the image */
#define VTX_JPEG_I_CHUNK_BASE 10 /* first chunk slot (ascending over the batch) */
#define VTX_JPEG_I_CHUNK_CAP 11  /* chunk slots: ceil(entropy bytes * 8 / chunk_bits) + segments */
#define VTX_JPEG_I_OH 12         /* oriented output height, width */
#define VTX_JPEG_I_OW 13
#define VTX_JPEG_I_COMP 16
#define VTX_JPEG_N64 8
#define VTX_JPEG_Q_ENT_SRC 0     /* entropy data (after SOS) in src; the EOI marker follows it */
#define VTX_JPEG_Q_ENT_LEN 1
#define VTX_JPEG_Q_ENT_DST 2     /* the image's region of ent */
#define VTX_JPEG_Q_COEF 3        /* first block in coef (ascending over the batch) */
#define VTX_JPEG_Q_PLANE 4       /* 3 plane offsets in planes */
#define VTX_JPEG_Q_OUT 7         /* RGB output offset in out */
#define VTX_JPEG_HUFF_BYTES 1536
#define VTX_JPEG_ST_MARKER 1     /* unexpected marker, RSTn out of order or restart count mismatch */
#define VTX_JPEG_ST_BADCODE 2    /* a code missing from the Huffman table */
#define VTX_JPEG_ST_RUN 4        /* a run past coefficient 63 */
#define VTX_JPEG_ST_OUT 8        /* a restart segment ran out of bits */
#define VTX_JPEG_ST_UNSYNCED 16  /* some chunk had not synchronised: run more rounds and decode again */
/* one CTA per image: strip stuffing, split at RSTn, count chunks of chunk_bits bits per segment */
int vtx_jpeg_unstuff(const uint8_t* src, const int32_t* info, const int64_t* info64, int B, uint8_t* ent,
                     int32_t* seg_start, int32_t* seg_len, int32_t* seg_chunk0, int32_t* nchunks, int32_t* status,
                     int chunk_bits, void* stream);
/* synchronisation round `round` (0 = speculative decode of every chunk) from st_in into st_out (int4 per slot) */
int vtx_jpeg_sync(const uint8_t* ent, const int32_t* info, const int64_t* info64, const void* huff,
                  const int32_t* seg_start, const int32_t* seg_len, const int32_t* seg_chunk0, const int32_t* nchunks,
                  int B, int slots, const void* st_in, void* st_out, int round, int32_t* rounds, int chunk_bits,
                  void* stream);
/* excl [slots] = exclusive scan of the blocks each chunk completes, per image */
int vtx_jpeg_count_scan(const int32_t* info, const int32_t* nchunks, const void* st, int32_t* excl, int B,
                        void* stream);
/* final decode: coefficients (DC as differences) into coef, verification of every chunk's recorded state */
int vtx_jpeg_coefs(const uint8_t* ent, const int32_t* info, const int64_t* info64, const void* huff,
                   const int32_t* seg_start, const int32_t* seg_len, const int32_t* seg_chunk0, const int32_t* nchunks,
                   int B, int slots, const void* st, const int32_t* excl, int16_t* coef, int32_t* status,
                   int chunk_bits, void* stream);
/* DC differences -> absolute DC, per component and restart interval */
int vtx_jpeg_dc_scan(const int32_t* info, const int64_t* info64, int16_t* coef, int B, void* stream);
/* dequantise + islow IDCT of nblocks blocks into the component planes */
int vtx_jpeg_idct(const int32_t* info, const int64_t* info64, const int16_t* coef, const uint16_t* quant,
                  uint8_t* planes, int B, int64_t nblocks, void* stream);
/* upsampling + YCbCr -> RGB (or grey x 3) + EXIF orientation into out (uint8 HWC RGB at out + info64 Q_OUT) */
int vtx_jpeg_color(const int32_t* info, const int64_t* info64, const uint8_t* planes, uint8_t* out, int B,
                   int64_t max_pixels, void* stream);

/* ------------------------------------------------------------------------------------------------------------------
 * Fused optimiser tail over flat fp32 arenas (scripts/pretrain_virtex.py:157-162; virtex/factories.py:529-545;
 * virtex/optim/lookahead.py:82-102).  segs: device array of {int64 begin, int64 end, float lr, float wd}.
 * ctl[0] = gradient scale (clip / world size), ctl[1] = gradient norm; hyper = {lr multiplier, first step, lookahead}.
 * ------------------------------------------------------------------------------------------------------------------ */
/* *out += sum of x[i]^2 over n elements (n = 0 leaves *out untouched); x must be 16-byte aligned (read as float4). */
int vtx_sumsq(const float* x, int64_t n, float* out, void* stream);
/* norm = sqrt(*sumsq) / world_size; ctl = {min(1, max_norm / (norm + 1e-6)) / world_size, norm}.  Non-finite norms
 * follow torch.nn.utils.clip_grad_norm_: an inf norm gives the coefficient 0 and a NaN norm a NaN coefficient, so the
 * step writes NaN into every updated parameter (the step is not skipped, as a GradScaler would).  max_norm <= 0
 * disables clipping (coefficient 1 / world_size), where clip_grad_norm_ would scale every gradient by <= 0. */
int vtx_clip_coef(const float* sumsq, int world_size, float max_norm, float* ctl, void* stream);
int vtx_sgd_step(float* p, const float* g, float* mom, float* slow, void* p_bf, const void* segs, int nseg,
                 const float* ctl, const float* hyper, float momentum, float la_alpha, void* stream);
/* torch.optim.AdamW (decoupled weight decay, no amsgrad) over the same segments; elements outside every segment and
 * their moments are left untouched.  hyper = {lr multiplier, 1/(1-beta1^t), 1/sqrt(1-beta2^t), lookahead}. */
int vtx_adamw_step(float* p, const float* g, float* exp_avg, float* exp_avg_sq, float* slow, void* p_bf,
                   const void* segs, int nseg, const float* ctl, const float* hyper, double beta1, double beta2,
                   float eps, float la_alpha, void* stream);

/* ------------------------------------------------------------------------------------------------------------------
 * VOC07 linear SVMs (csrc/svm.cu): the per-class LinearSVC(C, class_weight={1: 2, -1: 1}, loss="squared_hinge")
 * cost sweep with 3-fold cross_val_score(scoring="average_precision") of scripts/clf_voc07.py:56-105 (run once per
 * class by pool.map, :216-229), with the labels of virtex/data/datasets/downstream.py:151-165.  All P problems
 * (class, cost, fold-or-full fit) are columns of one truncated-Newton solve of liblinear's L2R_L2LOSS_SVC objective
 *     f_p(w) = 1/2 |w|^2 + sum_i c_ip max(0, 1 - y_ip w . x~_i)^2,    x~_i = [x_i, 1, 0 ...] (intercept_scaling = 1),
 * c_ip = 0 on the held-out fold of a cross-validation problem.  Per-problem vectors are fp32 [rows, P] (P % 64 == 0);
 * the products with X~ are vtx_gemm calls over the split operands written here (x = hi + lo in bf16, the three-term
 * product hi.hi + hi.lo + lo.hi concatenated along K):
 *     Z [n_pad, P]  = xcat [n_pad, 3 dp] . op [3 dp, P]          (a_mn 0, b_mn 1),  op = [hi; lo; hi] of W
 *     G [dp, P]     = xstk [3 n_pad, dp]^T . op [3 n_pad, P]     (a_mn 1, b_mn 1),  op = [hi; lo; hi] of U
 * Column reductions write partial sums double [k][VTX_SVM_SLICES][P] (k = 1 or 3 quantities) that their consumers
 * add in a fixed order.  Per-problem state: double scal [VTX_SVM_NSCAL, P] and int32 flags [VTX_SVM_NFLAGS, P], rows
 * named below; the caller zero-initialises both and W before the first Newton step.
 * ------------------------------------------------------------------------------------------------------------------ */
#define VTX_SVM_SLICES 32
#define VTX_SVM_MAX_N 16384 /* samples per problem (line search) and per scored column (average precision) */
/* scal rows: objective at the start of the Newton step, |grad f|, |grad f(0)|, CG |r|^2, CG tolerance |r|^2, CG beta,
   line-search step */
#define VTX_SVM_F 0
#define VTX_SVM_GNORM 1
#define VTX_SVM_GNORM0 2
#define VTX_SVM_RR 3
#define VTX_SVM_CG_TOL2 4
#define VTX_SVM_BETA 5
#define VTX_SVM_STEP 6
#define VTX_SVM_NSCAL 7
/* flags rows: status (0 running, 1 converged, 2 Newton-step cap), Newton steps taken, CG done in this step, CG
   iterations in this step, CG iterations in total, CG iteration cap ever hit */
#define VTX_SVM_STATUS 0
#define VTX_SVM_NEWTON 1
#define VTX_SVM_CG_DONE 2
#define VTX_SVM_CG_ITERS 3
#define VTX_SVM_CG_TOTAL 4
#define VTX_SVM_CG_CAPPED 5
#define VTX_SVM_NFLAGS 6
/* x fp32 [n, ldx] (d features) -> x~ = [x, 1, 0 ... 0] with rows n .. n_pad-1 zero, written as xcat bf16 [n_pad, 3 dp]
   = [hi | hi | lo] and / or xstk bf16 [3 n_pad, dp] = [hi; hi; lo] (either may be NULL); n_pad, dp % 64 == 0, dp > d */
int vtx_svm_split_x(const float* x, int64_t ldx, int n, int d, int n_pad, int dp, void* xcat, void* xstk, void* stream);
/* op bf16 [3 rows, P] = [hi; lo; hi] of v fp32 [rows, P] */
int vtx_svm_split_cols(const float* v, int rows, int P, void* op, void* stream);
/* From Z and cy = y * c [n, P]: uop = split of u = 2 c (z - y) [y z < 1] (grad f = w + X~^T u), dact = c [y z < 1]
   (generalised Hessian H = I + 2 X~^T diag(dact) X~), part [1][S][P] = loss sum_i c max(0, 1 - y z)^2 */
int vtx_svm_margin(const float* z, const float* cy, int n, int P, void* uop, float* dact, double* part, void* stream);
/* y += x when add; part [3][S][P] = sum y^2, sum x y, sum x^2 (after the add) */
int vtx_svm_axpy_dot(float* y, const float* x, int rows, int P, int add, double* part, void* stream);
/* vop = split of 2 dact t */
int vtx_svm_hess_mid(const float* t, const float* dact, int n, int P, void* vop, void* stream);
/* One thread per problem, from the margin's loss and the axpy_dot of g += w: objective, |g|, convergence
   (|g| <= eps |g(0)| -> status 1; max_newton steps taken -> status 2) and the CG set-up (|r|^2 = |g|^2, tolerance
   0.01 |g|^2: forcing term 0.1); *n_running = problems still running (the one value the host reads per Newton step) */
int vtx_svm_newton_begin(const double* part_loss, const double* part_g, int P, double* scal, int32_t* flags,
                         double eps, int max_newton, int32_t* n_running, void* stream);
/* r = -g, d = r, s = 0 (all zero for problems not running), dop = split of d */
int vtx_svm_cg_start(const float* g, float* r, float* d, float* s, const int32_t* flags, int rows, int P, void* dop,
                     void* stream);
/* CG iteration for problems with CG not done: alpha = rr / (d . Hd) from part_dhd (axpy_dot of Hd = X~^T v + d, row
   1), s += alpha d, r -= alpha Hd; part_rr [1][S][P] = |r|^2 */
int vtx_svm_cg_update(float* s, float* r, const float* d, const float* hd, const double* part_dhd, const double* scal,
                      const int32_t* flags, int rows, int P, double* part_rr, void* stream);
/* One thread per problem: beta = |r_new|^2 / |r|^2, CG done at |r|^2 <= tolerance or max_cg iterations (CG_CAPPED);
   *n_running = problems still in CG */
int vtx_svm_cg_scalars(const double* part_rr, int P, double* scal, int32_t* flags, int max_cg, int32_t* n_running,
                       void* stream);
/* d = r + beta d for problems in CG; dop = split of d */
int vtx_svm_cg_direction(const float* r, float* d, const double* scal, const int32_t* flags, int rows, int P, void* dop,
                         void* stream);
/* Exact line search along s, one CTA per running problem, in double: the root of phi'(a) for the convex piecewise
   quadratic phi(a) = f(w + a s), from z = X~ w, t = X~ s, cy and part_dots (axpy_dot with y = s, x = w: s.s, w.s);
   writes scal STEP, counts the Newton step, and sets status 1 when phi(0) - phi(step) <= decrease_tol * f.
   n <= VTX_SVM_MAX_N (z, t, cy staged in shared memory). */
int vtx_svm_line_search(const float* z, const float* t, const float* cy, int n, int P, const double* part_dots,
                        double* scal, int32_t* flags, double decrease_tol, void* stream);
/* w += step s; wop = split of w */
int vtx_svm_newton_step(float* w, const float* s, const double* scal, int rows, int P, void* wop, void* stream);
/* sklearn's average_precision_score (sklearn/metrics/_ranking.py: step-wise over distinct thresholds, tied scores one
   step), one CTA per scored column j: cols int32 [ncols, 3] = (score column, label column, fold).  Sample i < n counts
   when labels[i * ldl + label column] is 1 (positive) or 0 (negative) and, for fold >= 0, folds[i * ldf + label column]
   == fold; ap[j] in double, 0 without a positive.  n > VTX_SVM_MAX_N is rejected with VTX_EUNSUPPORTED. */
int vtx_svm_average_precision(const float* scores, int64_t lds, int n, const int8_t* labels, int64_t ldl,
                              const int8_t* folds, int64_t ldf, const int32_t* cols, int ncols, double* ap,
                              void* stream);

/* ------------------------------------------------------------------------------------------------------------------
 * Caption metrics (CIDEr) (csrc/cider.cu): cider(predictions, ground_truth, n=4, sigma) of virtex/utils/metrics.py:
 * 177-264, the score of CocoCaptionsEvaluator.evaluate.  Sentences are int32 word ids in CSR form: words [W] and
 * sent_off [S + 1].  Image i owns reference sentences img_off[i] .. img_off[i + 1] - 1 and hypothesis sentence i.
 * Per-occurrence arrays are [W, 4]: entry (w, k - 1) is the k-gram starting at word w (k = 1..4); an entry past its
 * sentence's end holds gid -1, tf 0, ent -1.
 * An n-gram's identity is a slot of a device hash table (keys uint64 [capacity], capacity a power of two, zeroed by the
 * caller): a k-gram is the full key (slot of its (k-1)-gram, last word), so equal slots mean equal n-grams.
 * Every float reduction runs in a fixed order on one thread: two calls are bit-identical.
 * ------------------------------------------------------------------------------------------------------------------ */
#define VTX_CIDER_MAX_REFS 32                /* references per image */
#define VTX_CIDER_MAX_WORDS 256              /* words per sentence */
#define VTX_CIDER_MAX_IMAGE_WORDS 1024       /* reference words of one image (shared-memory df deduplication) */
#define VTX_CIDER_MAX_TOTAL_WORDS (1 << 24)  /* reference words, and hypothesis words, of one corpus */
/* gid [W, 4] = slot of every n-gram, inserted (insert = 1) or looked up (insert = 0: -1 when absent).  The table
   must have at least twice as many slots as it will hold n-grams. */
int vtx_cider_intern(const int32_t* words, const int32_t* sent_off, int n_sent, unsigned long long* keys,
                     int64_t capacity, int insert, int32_t* gid, void* stream);
/* df [capacity] (zeroed by the caller) += 1 per image for every distinct n-gram of its references, one CTA per image */
int vtx_cider_df(const int32_t* gid, const int32_t* sent_off, const int32_t* img_off, int n_img, int32_t* df,
                 void* stream);
/* One warp per sentence: at the first occurrence of each distinct n-gram (by words) tf = its count in the sentence and
   ent = tf * (log n_img - log max(1, df[gid])) (df 0 when gid < 0); later occurrences tf 0, ent -1.
   norm [S, 4] = sqrt(sum of ent^2) per order, summed in position order. */
int vtx_cider_vectors(const int32_t* words, const int32_t* gid, const int32_t* sent_off, int n_sent, const int32_t* df,
                      int n_img, int32_t* tf, double* ent, double* norm, void* stream);
/* img_score [n_img] = 10 * mean_k(sum over references of sim_k) / references, with sim_k of the reference's cider():
   sum over the hypothesis's distinct k-grams of min(vh, vr) * vr, divided by (|h|_k |r|_k) or 1, times
   e^(-(len_h - len_r)^2 / (2 sigma^2)), len = max(words - 1, 0).  hyp_off [n_img + 1]; one warp per image. */
int vtx_cider_score(const int32_t* hyp_gid, const double* hyp_ent, const double* hyp_norm, const int32_t* hyp_off,
                    const int32_t* ref_gid, const double* ref_ent, const double* ref_norm, const int32_t* ref_off,
                    const int32_t* img_off, int n_img, double sigma, double* img_score, void* stream);
/* out[0] = mean of x [n], one CTA in a fixed order */
int vtx_cider_mean(const double* x, int n, double* out, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* VIRTEX_B200_H_ */
