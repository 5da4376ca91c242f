/* pg_b200.h — C ABI of libpg_b200.so, the sm_90a kernel library behind the drop-in
 * `pytorch_generative.nn.*` / `models.*` Module API.
 *
 * The reference (EugenHotaj/pytorch-generative) ships no native interface: its hot path is Python
 * nn.Modules whose arithmetic is delegated to torch (SURVEY.md §8b).  The entry points below are
 * therefore what a maintainer's ctypes binding would call in place of those torch ops; each one
 * cites the reference call site it replaces.  Conventions:
 *   - every pointer is a raw device pointer unless stated otherwise; the caller owns all memory;
 *   - `stream` is a cudaStream_t passed as void* (NULL = legacy default stream);
 *   - return value 0 = success, non-zero = failure with a message available from pg_last_error();
 *   - no allocation, no global stream state, no torch/pybind types;
 *   - the streaming kernels move 16 bytes per access, so pg_layernorm_fwd / _bwd when C % 128 == 0 and C <= 1024,
 *     pg_gated_act_fwd / _bwd and pg_gated_res_fwd when C % 8 == 0, pg_act_cast_bf16 when C and ld_out are multiples
 *     of 8 and ld_x is a multiple of 4 (fp32 x) or 8 (bf16 x), pg_dact_from_out, pg_tap_gather and pg_tap_scatter
 *     need every tensor base they access 16-byte aligned (a column view may not start mid-row; pitches as stated per
 *     function); a misaligned base is an error return, never a kernel launch;
 *   - activations are "pixel-major": a [P, C] row-major matrix with P = N*H*W pixels (NHWC), which is
 *     the layout every GEMM-shaped op wants; NCHW<->pixel-major converters are provided for the
 *     module boundary.
 */
#ifndef PG_B200_H_
#define PG_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define PG_ABI_VERSION 1

int pg_abi_version(void);
const char* pg_last_error(void);
/* Number of SMs of the current device (132 on an H100 SXM); used by callers to size split-K. */
int pg_sm_count(void);
/* Leaves `n` SMs out of every persistent grid from now on (returns the previous setting; 0 = use them all): room for the
 * NCCL kernels of the gradient all-reduce that run concurrently with the backward pass under data parallelism. */
int pg_reserve_sms(int n);
/* Number of kernels this library has launched in this process (all threads); bench.py's gpu_launches. */
unsigned long long pg_launch_count(void);

/* Activation ids (shared by the GEMM epilogue and the elementwise kernels). */
enum { PG_ACT_NONE = 0, PG_ACT_RELU = 1, PG_ACT_GELU = 2, PG_ACT_ELU = 3, PG_ACT_TANH = 4,
       /* pg_gemm_epilogue.dact only: `aux` already holds the derivative (see PG_ACT_STORE_DERIV) */
       PG_ACT_GIVEN = 5,
       /* pg_gemm_epilogue.dact only: `aux` holds the ACTIVATED value (relu(pre) / elu(pre)), from which the derivative
        * follows without the pre-activation: relu' = [a > 0], elu' = a > 0 ? 1 : a + 1 */
       PG_ACT_RELU_OUT = 6, PG_ACT_ELU_OUT = 7 };
/* OR-ed into pg_gemm_epilogue.act: out_pre receives act'(pre) instead of pre, so that the matching dgrad epilogue
 * (dact = PG_ACT_GIVEN) is a single multiply. */
#define PG_ACT_STORE_DERIV 0x100
/* OR-ed into pg_gemm_epilogue.act: res0 / res1 point to bf16 [M,N] matrices (pitch ld_res in bf16 elements, a multiple of 8)
 * instead of fp32 ones — short-lived sums (GatedPixelCNN's vertical-to-horizontal link) that are not a residual stream. */
#define PG_ACT_RES_BF16 0x200

/* ---------------------------------------------------------------------------------------------
 * Channel contraction (every nn.Conv2d 1x1 on the path and, per live tap, every masked conv):
 *   reference: torch.nn.Conv2d.forward at nn/attention.py:105-118,140-144,161;
 *   models/autoregressive/image_gpt.py:40-48,101-103; pixel_cnn.py:35-49,95-103;
 *   gated_pixel_cnn.py:79-99,176-182; pixel_snail.py:86-87,173-180 — and their autograd
 *   (dgrad / wgrad).
 *
 *   acc[m,n] = sum_k A(m,k) * B(n,k)            bf16 inputs, fp32 accumulation on wgmma
 *   t        = alpha * acc + bias[n]
 *   t       *= act'(aux[m,n])                   if dact != PG_ACT_NONE   (backward through an activation)
 *   pre      = t + res0[m,n] + res1[m,n]
 *   out_f32[m,n]  = pre  (or += pre when accumulate=1; bias/res only added by split 0)
 *   out_pre[m,n]  = bf16(pre)
 *   out_bf16[m,n] = bf16(act(pre))
 *
 * Operand layouts: a_mn_major=0 -> A is [M,K] row-major with pitch lda (K contiguous);
 *                  a_mn_major=1 -> A is [K,M] row-major with pitch lda (M contiguous).
 *                  b_mn_major=0 -> B is [N,K] row-major (a conv weight [Cout,Cin]);
 *                  b_mn_major=1 -> B is [K,N] row-major.
 * So forward = (0,0) with B = W; dgrad = (0,1) with B = W; wgrad = (1,1) with A = dY, B = X.
 * Pitches must be multiples of 8 elements and bases 16-byte aligned (TMA requirement).
 * ------------------------------------------------------------------------------------------- */
typedef struct pg_gemm_epilogue {
  const float* bias;   /* [N] or NULL */
  const void* aux;     /* bf16 [M,N] pre-activation (or the derivative itself, dact = PG_ACT_GIVEN), used when dact != 0 */
  const float* res0;   /* fp32 [M,N] or NULL */
  const float* res1;   /* fp32 [M,N] or NULL */
  void* out_bf16;      /* bf16 [M,N] or NULL */
  void* out_pre;       /* bf16 [M,N] or NULL: pre-activation (act'(pre) with PG_ACT_STORE_DERIV) */
  float* out_f32;      /* fp32 [M,N] or NULL */
  int64_t ld_aux, ld_res, ld_out_bf16, ld_out_pre, ld_out_f32; /* row pitches, elements */
  int32_t act;         /* activation applied to out_bf16 */
  int32_t dact;        /* activation whose derivative (at aux) scales the accumulator */
  int32_t accumulate;  /* 1: out_f32 is accumulated with fp32 atomics (split-K / grad accumulation) */
  float alpha;
  float* bias_grad;    /* weight-gradient GEMMs only (a_mn_major = 1, impl 0), or NULL: fp32 [M] += sum_k A(m,k), i.e. the
                        * bias gradient sum_p dY[p, cout] of the same layer, reduced from the staged A tiles */
} pg_gemm_epilogue;

/* impl: 0 = wgmma/TMA kernel (the product); 1 = plain SIMT kernel kept as an on-device cross-check
 * for the tests (same epilogue code); 2 = skinny-rows kernel for M <= 32 (the per-pixel step of incremental
 * sampling: one warp per output column, weights streamed once).  split_k > 1 only with accumulate=1 into out_f32
 * alone (no bias, residuals, activation or bf16 outputs); the K slices are added to out_f32 in slice order. */
int pg_gemm_bf16(const void* A, int a_mn_major, int64_t lda, const void* B, int b_mn_major, int64_t ldb,
                 int M, int N, int K, int split_k, const pg_gemm_epilogue* epi, int impl, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Tap-loop convolution, im2col-free (CausalConv2d with wide channels — reference nn/convolution.py:41-43;
 * GatedPixelCNN 1xN / Nx1 stacks — gated_pixel_cnn.py:63-99 with the crops at 115,121; PixelSNAIL 2x2 —
 * pixel_snail.py:41-56), forward and both gradients on the pg_gemm_bf16 kernel:
 *   conv(x)[p] = sum_t W_t . x[p + (dy_t, dx_t)], zero outside the image (the reference's pad + front crop).
 * The shifted operand is never materialised: for every tap the TMA unit loads the [C, W, H, N] box displaced by
 * (dy_t, dx_t) from the pixel-major tensor (out-of-image elements arrive as zeros) and the tensor core accumulates
 * one K slab per (tap, 64 channels).  Epilogue semantics are pg_gemm_bf16's.
 *   PG_CONV_FWD:   A = x  [P, >=C] bf16, C = Cin;  B = packed weight [Cout, T*Cin] (tap-major columns);
 *                  M = P, N = Cout, K = T*Cin.
 *   PG_CONV_DGRAD: A = dy [P, >=C] bf16, C = Cout, taps negated by the caller;  B = the same packed weight;
 *                  M = P, N = Cin (= the per-tap column stride of the packed weight), K = T*Cout.
 *   PG_CONV_WGRAD: A = dy [P, Cout] bf16;  B = x [P, >=C] bf16, C = Cin;  M = Cout, N = T*Cin, K = P;
 *                  out_f32 [Cout, T*Cin] accumulated (split_k as pg_gemm_bf16).
 * Geometry limits (else use pg_tap_gather): C % 64 == 0, W | 64, H*W % 128 == 0, 1..225 taps, |offset| <= 64.
 * pg_gemm_bf16_conv_taps takes the offsets as host arrays dy[n_taps], dx[n_taps] (up to 225 taps: a 15 x 15 kernel, of
 * any dilation whose offsets stay within 64); pg_gemm_bf16_conv is the same call with the geometry in a pg_conv_geom,
 * whose arrays hold 32 taps.  The kernel receives the offsets as int8 in its parameters (450 bytes at 225 taps).
 * ------------------------------------------------------------------------------------------- */
enum { PG_CONV_FWD = 1, PG_CONV_DGRAD = 2, PG_CONV_WGRAD = 3 };
typedef struct pg_conv_geom {
  int32_t mode;        /* PG_CONV_* */
  int32_t N, H, W;     /* images, rows, columns: P = N*H*W pixels */
  int32_t C;           /* channels of the shifted tensor (per-tap K extent for fwd / dgrad, per-tap N extent for wgrad) */
  int32_t n_taps;
  int32_t dy[32], dx[32];
} pg_conv_geom;
int pg_gemm_bf16_conv(const void* A, int64_t lda, const void* B, int64_t ldb, int M, int N, int K, int split_k,
                      const pg_gemm_epilogue* epi, const pg_conv_geom* geom, void* stream);
int pg_gemm_bf16_conv_taps(const void* A, int64_t lda, const void* B, int64_t ldb, int M, int N, int K, int split_k,
                           const pg_gemm_epilogue* epi, int mode, int n_img, int H, int W, int C, int n_taps,
                           const int* dy /* host */, const int* dx /* host */, void* stream);

/* Column sums of a bf16 [P, C] matrix into fp32 out[C] (bias gradients; accumulate=1 adds). */
int pg_colsum_bf16(const void* x, int64_t ld, int P, int C, float* out, int accumulate, void* stream);
int pg_colsum_f32(const float* x, int64_t ld, int P, int C, float* out, int accumulate, void* stream);

/* ---------------------------------------------------------------------------------------------
 * ReZero — reference nn/utils.py ReZeroWrapper: y = x + alpha f, alpha a [1] fp32 tensor read on the device (no host
 * read: the call can be captured in a CUDA graph).  x, f, y, dy, df are contiguous fp32 arrays of `numel` elements.
 * Every product and sum is a separately rounded fp32 operation (no FMA), so y and df equal torch's `x + alpha * f` and
 * its gradient bit for bit.
 *   pg_rezero_fwd: y = x + alpha f.  One launch.
 *   pg_rezero_bwd: df = alpha dy (df may be NULL); dalpha[0] = sum(dy f) (dalpha may be NULL; it is overwritten).  Block
 *     b sums elements [b PG_REZERO_CHUNK, (b + 1) PG_REZERO_CHUNK) into the library's scratch and pg_sum_partials adds
 *     the blocks in block order: two launches, one when dalpha is NULL.  No atomics: every run gives the same bits.
 * ------------------------------------------------------------------------------------------- */
#define PG_REZERO_CHUNK 8192
int pg_rezero_fwd(const float* x, const float* f, const float* alpha, int64_t numel, float* y, void* stream);
int pg_rezero_bwd(const float* dy, const float* f, const float* alpha, int64_t numel, float* df, float* dalpha,
                  void* stream);

/* ---------------------------------------------------------------------------------------------
 * NCHWLayerNorm — reference nn/convolution.py:69-75 (permute -> nn.LayerNorm(C) -> permute).
 * Pixel-major x [P, C] fp32 (the residual stream) -> y bf16 and/or fp32; eps as nn.LayerNorm (1e-5),
 * biased variance; mean/rstd [P] fp32 are saved for backward.
 * Backward: dx = rstd * (g - mean_c(g) - xhat * mean_c(g * xhat)), g = dy * gamma;
 *   dx_out_f32 = dx + dres0 + dres1 (fused residual-gradient adds), optional bf16 copy for the next
 *   dgrad GEMM; dgamma/dbeta are accumulated (atomics) into fp32 [C] buffers that the caller zeroed;
 *   dx_colsum (optional, [C], caller-zeroed) receives the column sums of dx_out = the bias gradient of the
 *   layer whose output x is (saves a separate pass over the gradient).
 * ------------------------------------------------------------------------------------------- */
int pg_layernorm_fwd(const float* x, const float* gamma, const float* beta, int P, int C, float eps,
                     void* y_bf16, float* y_f32, float* mean, float* rstd, void* stream);
int pg_layernorm_bwd(const void* dy_bf16, const float* dy_f32, const float* x, const float* gamma,
                     const float* mean, const float* rstd, int P, int C, const float* dres0,
                     const float* dres1, float* dx_f32, void* dx_bf16, float* dgamma, float* dbeta,
                     float* dx_colsum, void* stream);
/* The same LayerNorm on rows of pitch ld >= C (x, y, dy, dres0 / dres1 and dx all [P, ld]): the statistics, dgamma,
 * dbeta and dx_colsum cover the first C columns, and columns C..ld of y and dx are written as zeros.  This keeps a
 * stream of C channels in a 16-byte operand pitch (ld = round_up(C, 8)) with exactly-zero pad columns.
 * pg_layernorm_fwd / _bwd are these calls with ld = C; ld > C takes the generic (4-byte access) kernels. */
int pg_layernorm_fwd_ld(const float* x, const float* gamma, const float* beta, int P, int C, int ld, float eps,
                        void* y_bf16, float* y_f32, float* mean, float* rstd, void* stream);
int pg_layernorm_bwd_ld(const void* dy_bf16, const float* dy_f32, const float* x, const float* gamma,
                        const float* mean, const float* rstd, int P, int C, int ld, const float* dres0,
                        const float* dres1, float* dx_f32, void* dx_bf16, float* dgamma, float* dbeta,
                        float* dx_colsum, void* stream);

/* ---------------------------------------------------------------------------------------------
 * GatedActivation — reference nn/convolution.py:46-66: act(x[:, :C]) * sigmoid(x[:, C:]).
 * Pixel-major x [P, 2C] (bf16 or fp32) -> y [P, C].  act is PG_ACT_TANH (GatedPixelCNN) or
 * PG_ACT_NONE (PixelSNAIL's nn.Identity).  Backward writes dx [P, 2C].  Any C >= 1: C % 8 == 0 takes 16-byte
 * accesses (aligned bases required), any other C goes element by element (no alignment requirement); the same holds for
 * pg_gated_res_fwd.
 * ------------------------------------------------------------------------------------------- */
int pg_gated_act_fwd(const void* x, int x_is_f32, int P, int C, int act, void* y, int y_is_f32, void* stream);
int pg_gated_act_bwd(const void* x, int x_is_f32, const void* dy, int dy_is_f32, int P, int C, int act,
                     void* dx, int dx_is_f32, void* stream);
/* y = res + act(x[:, :C]) * sigmoid(x[:, C:]) in one pass: the residual sum around PixelSNAIL's gated residual block
 * (reference pixel_snail.py:52-56), res / y fp32 [P, C]. */
int pg_gated_res_fwd(const void* x, int x_is_f32, const float* res, int P, int C, int act, float* y, void* stream);
/* out = bf16(dy * act'(pre)) given the ACTIVATED value ya = act(pre) (relu / elu; elu'(pre) = ya + 1 for pre <= 0): the
 * backward of an activation whose output, not input, was kept (elu(conv(.)) outputs, pixel_snail.py:27-28,115-119). */
int pg_dact_from_out(const void* dy, int dy_is_f32, const void* ya_bf16, int64_t numel, int act, void* out_bf16, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Recipe loss — reference models/autoregressive/image_gpt.py:158-162 (identical in the other three):
 * BCEWithLogits(preds, x, reduction="none").sum(1).mean().  logits/target are [N, D] fp32 in any
 * common memory order (elementwise); loss_sum receives sum over all elements (caller divides by N);
 * dlogits = (sigmoid(l) - t) * scale.
 * ------------------------------------------------------------------------------------------- */
int pg_bce_logits_fwd_bwd(const float* logits, const float* target, int64_t numel, float grad_scale,
                          float* loss_sum /* 1 float, accumulated */, float* dlogits /* or NULL */,
                          void* stream);

/* Layout converters for the Module boundary (NCHW fp32 <-> pixel-major). */
int pg_nchw_to_pm(const float* x_nchw, int N, int C, int HW, void* out, int out_is_f32, int64_t ld_out,
                  void* stream);
/* act (PG_ACT_*) is applied on the way out: used for activations that follow a convolution. */
int pg_pm_to_nchw(const void* x_pm, int x_is_f32, int64_t ld_x, int N, int C, int HW, int act, float* out_nchw,
                  void* stream);
/* out = bf16(dy * act'(pre)): gradient through such an output activation. */
int pg_dact_mul(const void* dy_bf16, int64_t ld_dy, const float* pre_f32, int64_t ld_pre, int P, int C, int act,
                void* out_bf16, int64_t ld_out, void* stream);
/* out = bf16(act(x)) over a pitched pixel-major [P, C] matrix (fp32 or bf16 in): builds the tensor-core operand of a
 * convolution whose input activation (ReLU / ELU in front of the conv: pixel_cnn.py:35-49, pixel_snail.py:27-28) was not
 * already emitted by the producing GEMM's epilogue.  Any C: with C and ld_out multiples of 8 and ld_x a multiple of 4
 * (fp32 x) or 8 (bf16 x) it takes 16-byte accesses, anything else goes element by element. */
int pg_act_cast_bf16(const void* x, int x_is_f32, int64_t ld_x, int P, int C, int act, void* out_bf16, int64_t ld_out,
                     void* stream);
/* fp32 -> bf16 cast of a dense buffer (weights packing; masked taps already zeroed by the caller). */
int pg_cast_f32_to_bf16(const float* x, void* y, int64_t numel, void* stream);

/* ---------------------------------------------------------------------------------------------
 * CausalAttention core — reference nn/attention.py:147-160 (mask, q@k^T/sqrt(dk), masked softmax,
 * re-zero, attn@v, head concat).  q/k/v/o are pixel-major bf16 with per-image sequences of length S
 * (seq index = row*W+col), heads are contiguous channel blocks of dk (q,k) / dv (v,o) channels.
 * strict=1 is mask_center=True (position i attends j<i; row 0 yields zeros), strict=0 attends j<=i.
 * `scale` multiplies q.k (the reference uses 1/sqrt(embed_channels/n_heads); it is passed explicitly so
 * that head slots may be zero-padded: the tensor-core kernels require dk in {64, 128} and dv in {64, 128},
 * other heads are laid out in the smallest of those slots that holds them, with zero extra columns).
 * lse [N, H, S] fp32 (log-sum-exp of scaled scores; rows without keys store 0 and o = 0).
 * impl: 0 = wgmma kernel, 1 = SIMT cross-check (any dk, dv <= 128, S <= 1024).
 * ------------------------------------------------------------------------------------------- */
int pg_causal_attn_fwd(const void* q, int64_t ld_q, const void* k, int64_t ld_k, const void* v, int64_t ld_v,
                       void* o, int64_t ld_o, float* lse, int N, int S, int H, int dk, int dv, float scale,
                       int strict, int impl, void* stream);
/* Scratch: delta [N, H, S] fp32.  dq_accum is not used (kept for ABI compatibility; may be NULL).  dq/dk/dv are bf16
 * pixel-major.  Every output element is summed in a fixed order: the results are the same on every run.
 * impl (backward): 0 = wgmma kernels, 3 = the same kernels (one CTA per key tile for dK / dV), 1 = SIMT cross-check. */
int pg_causal_attn_bwd(const void* q, int64_t ld_q, const void* k, int64_t ld_k, const void* v, int64_t ld_v,
                       const void* o, int64_t ld_o, const void* d_o, int64_t ld_do, const float* lse,
                       float* delta, float* dq_accum, void* dq, int64_t ld_dq, void* dk_, int64_t ld_dk,
                       void* dv_, int64_t ld_dv, int N, int S, int H, int dk, int dv, float scale, int strict,
                       int impl, void* stream);

/* Incremental (KV-cached) attention for AutoregressiveModel.sample (reference models/base.py:97-120 recomputes the full
 * forward per pixel; causality makes the per-position update exact): appends the current position's k / v rows
 * ([N, H*d]) to the caches ([N*S, H*d]) at row *pos_dev and attends over cache rows [0, pos] ([0, pos) if strict).
 * pos_dev is a device int so that one captured CUDA graph serves the whole raster scan.  S (the cache capacity) is
 * unbounded; dk, dv <= 128, dk % 8 == 0.  For S > 1024 each (image, head) is split into ceil(S / 1024) blocks of 1024
 * keys whose partial (max, sum, output) go through the library's reduction scratch and are merged in a fixed order;
 * the scratch grows outside CUDA-graph capture only, so run one step with the same S before capturing it. */
int pg_attn_decode(const void* q, int64_t ld_q, const void* k_new, int64_t ld_kn, const void* v_new, int64_t ld_vn,
                   void* k_cache, int64_t ld_kc, void* v_cache, int64_t ld_vc, void* o, int64_t ld_o,
                   const int* pos_dev, int N, int S, int H, int dk, int dv, float scale, int strict, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Tap-list convolution for small channel counts (CausalConv2d input layers, Cin in {1,3}):
 * reference nn/convolution.py:41-43 (weight.data *= mask; F.conv2d).  x is NCHW fp32 (the model
 * input), w is the masked OIHW fp32 weight, output pixel-major.  taps are all kh*kw positions; masked
 * taps contribute zero because the caller zeroes the weight in place exactly as the reference does.
 * wgrad is dense over kh*kw (masked taps receive gradient, as autograd does in the reference).
 * The _d variants take a dilation: kernel position (i, j) reads the input at (y + i*dil_h - pad_h, x + j*dil_w - pad_w)
 * (nn.Conv2d's `dilation`); pg_conv_small_fwd / _bwd are these calls with dil_h = dil_w = 1.
 * ------------------------------------------------------------------------------------------- */
int pg_conv_small_fwd(const float* x_nchw, const float* w_oihw, const float* bias, int N, int Cin, int H, int W,
                      int Cout, int kh, int kw, int pad_h, int pad_w, int pre_act /* applied to x */, float* out_f32,
                      void* out_bf16, int act_bf16, void* stream);
int pg_conv_small_bwd(const float* x_nchw, const float* w_oihw, const float* dy_pm /* [P,Cout] fp32 */, int N,
                      int Cin, int H, int W, int Cout, int kh, int kw, int pad_h, int pad_w, int pre_act,
                      float* dw_oihw /* accumulated */, float* dbias /* accumulated */,
                      float* dx_nchw /* or NULL; overwritten */, void* stream);
int pg_conv_small_fwd_d(const float* x_nchw, const float* w_oihw, const float* bias, int N, int Cin, int H, int W,
                        int Cout, int kh, int kw, int pad_h, int pad_w, int dil_h, int dil_w, int pre_act,
                        float* out_f32, void* out_bf16, int act_bf16, void* stream);
int pg_conv_small_bwd_d(const float* x_nchw, const float* w_oihw, const float* dy_pm, int N, int Cin, int H, int W,
                        int Cout, int kh, int kw, int pad_h, int pad_w, int dil_h, int dil_w, int pre_act,
                        float* dw_oihw, float* dbias, float* dx_nchw, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Wide-channel tap-list convolutions (CausalConv2d with Cin >= 8; GatedPixelCNN 1xN / Nx1 — reference
 * gated_pixel_cnn.py:63-99 with the crops at 115,121; PixelSNAIL 2x2 — pixel_snail.py:41-56).
 * conv(x)[p] = sum_t W_t . x[p + (dy_t, dx_t)], zero outside the image (= the reference's pad + front crop).
 * pg_tap_gather builds X_cat[p, t*C + c] = act(x[p + off_t, c]) in bf16; the contraction over K = T*C is
 * pg_gemm_bf16 (forward, dgrad to dX_cat, wgrad from X_cat); pg_tap_scatter folds dX_cat back:
 * dx[p, c] = act'(x_pre[p, c]) * sum_t dX_cat[p - off_t, t*C + c].  C % 8 == 0, 1 <= T <= 225 (a 15 x 15 kernel), any
 * offsets; the kernels receive them as int32 in their parameters (1800 bytes at 225 taps).
 * These are the stride-1 case of pg_strided_gather / pg_strided_scatter below, with rows = spatial = (N, H, W), and run
 * on the same kernels (pg_tap_gather adds act; pg_tap_scatter is dact = act with no bias and no output activation), so
 * they take the same checks: pitches (ld_x; ld_dx, and ld_pre when act != PG_ACT_NONE) at least C, and N = 0 returns 0
 * without a launch.
 * ------------------------------------------------------------------------------------------- */
int pg_tap_gather(const void* x_pm, int64_t ld_x, int N, int H, int W, int C, int T, const int* dy /* host */,
                  const int* dx /* host */, int act, void* out /* bf16 [P, T*C] */, void* stream);
int pg_tap_scatter(const void* dxcat /* bf16 [P, T*C] */, int N, int H, int W, int C, int T, const int* dy,
                   const int* dx, int act, const void* x_pre /* bf16 [P, ld_pre] or NULL */, int64_t ld_pre,
                   float* dx_f32, void* dx_bf16, int64_t ld_dx, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Strided tap gather / scatter — the stride-2 Conv2d and ConvTranspose2d of reference models/vae/vaes.py (Encoder,
 * Decoder).  Two geometries: the grid of GEMM rows (N, Hg, Wg) and the spatial tensor (N, Hs, Ws), both pixel-major.
 * With the taps of every kernel position (dy_t, dx_t) = (i - pad, j - pad):
 *   pg_strided_gather:  X_cat[p_o, t*C + c] = x[(yo*s + dy_t, xo*s + dx_t), c]   (bf16, zero outside the spatial tensor);
 *   pg_strided_scatter: its adjoint, v[q, c] = sum over the (p_o, t) that land on q, in ascending t, of Y_cat[p_o, t*C + c]
 *     (Y_cat fp32 when ycat_f32, else bf16; contiguous [N*Hg*Wg, T*C]); then v += bias[c] for c < n_bias (bias may be
 *     NULL), v *= dact'(x_pre[q, c]) when x_pre is not NULL; out_f32 = v and out_bf16 = act(v), either may be NULL.
 *     A spatial pixel no tap reaches gets v = bias (or 0).  No atomics.
 * Conv2d(k, s, p): rows = output pixels, spatial = input; forward = gather -> GEMM, dgrad = GEMM -> scatter (with the
 * input activation's derivative), wgrad = GEMM over X_cat.  ConvTranspose2d(k, s, p): rows = input pixels, spatial =
 * output; forward = GEMM into Y_cat -> scatter (bias and the next layer's activation), dgrad = gather of dY -> GEMM,
 * wgrad = GEMM of the gathered dY against X.  C % 8 == 0, 1 <= T <= 225, s >= 1, pitches multiples of 8.
 * ------------------------------------------------------------------------------------------- */
int pg_strided_gather(const void* x_pm, int64_t ld_x, int N, int Hg, int Wg, int Hs, int Ws, int C, int T, int stride,
                      const int* dy /* host */, const int* dx /* host */, void* out /* bf16 [N*Hg*Wg, T*C] */,
                      void* stream);
int pg_strided_scatter(const void* ycat, int ycat_f32, int N, int Hg, int Wg, int Hs, int Ws, int C, int T, int stride,
                       const int* dy, const int* dx, const float* bias, int n_bias, int act, int dact,
                       const void* x_pre /* bf16 [N*Hs*Ws, ld_pre] or NULL */, int64_t ld_pre, float* out_f32,
                       void* out_bf16, int64_t ld_out, void* stream);

/* ---------------------------------------------------------------------------------------------
 * LinearCausalAttention numerator — reference nn/attention.py:168-200 (`_UnnormalizedLinearCausalAttention`: a Python loop
 * over the sequence, forward and backward).  q, k: [B, L, d] fp32, v / g / out: [B, L, dv] fp32, B = images x heads,
 * contiguous.  out_i = q_i . S_i,  S_i = sum_{j <= i} k_j^T v_j.  Backward: dq_i = g_i S_i^T; with R_i = sum_{j >= i}
 * q_j^T g_j: dv_i = k_i R_i, dk_i = v_i R_i^T.  Any d, dv, L >= 1.  Each product is one chunked fp32 scan: per chunk of
 * 64 positions, out_c = X_c S + tril(X_c Y_c^T) Z_c, then S += Y_c^T Z_c; one CTA per 64 output columns recomputes
 * X_c Y_c^T, so only a (d or dv) x 64 slice of the state is live.  When B x column blocks leaves SMs idle the sequence is
 * also split into segments that start from the fixed-order sum of the segments before them.  Deterministic (no atomics),
 * O(L (d + dv)) memory plus a pg_scratch area that does not grow with L.
 * ------------------------------------------------------------------------------------------- */
int pg_linear_attn_fwd(const float* q, const float* k, const float* v, float* out, int B, int L, int d, int dv, void* stream);
int pg_linear_attn_bwd(const float* q, const float* k, const float* v, const float* g, float* dq, float* dk, float* dv_out,
                       int B, int L, int d, int dv, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Optimizer part of the training step — reference trainer.py:182-191 (`clip_grad_norm_(model.parameters(), max_norm)`
 * then `optimizer.step()` with torch.optim.Adam as every recipe builds it, e.g. image_gpt.py:155) over ALL parameters in
 * two launches.  Tensors are given as device arrays of device pointers (one entry per parameter, fp32, contiguous);
 * `numel` [n_tensors] int64 (device); `chunks` [n_chunks] pairs of int32 (tensor index, chunk index) (device): block b
 * handles elements [chunk * chunk_elems, +chunk_elems) of its tensor.
 *   pg_grad_sqnorm: partials[b] = sum of g^2 over block b's chunk.
 *   pg_adam_step:   norm = sqrt(sum partials) (same order in every block: deterministic); norm_out[0] = norm;
 *                   if skip_above > 0 and not (norm <= skip_above), a NaN norm included: nothing is updated and
 *                   norm_out[1] = 0 (the trainer's skip_grad_norm rule), else norm_out[1] = 1 and, with
 *                   c = min(1, max_norm / (norm + 1e-6)) (NaN when the norm is NaN, as in torch's clip_grad_norm_):
 *                   g *= c (written back unless c == 1), m = b1 m + (1-b1) g, v = b2 v + (1-b2) g^2,
 *                   p -= lr / (1-b1^step) * m / (sqrt(v) / sqrt(1-b2^step) + eps)      (torch.optim.Adam, no amsgrad).
 * ------------------------------------------------------------------------------------------- */
/* dst[t][i] = bf16(src[t][i]) for many fp32 tensors in one launch (same pointer-array / chunk-table convention): the
 * per-step refresh of the bf16 tensor-core copies of the fp32 master weights. */
int pg_cast_multi_bf16(const void* src_ptrs, const void* dst_ptrs, const int64_t* numel, const void* chunks, int n_chunks,
                       int chunk_elems, void* stream);
int pg_grad_sqnorm(const void* grad_ptrs, const int64_t* numel, const void* chunks, int n_chunks, int chunk_elems,
                   float* partials, void* stream);
int pg_adam_step(const void* param_ptrs, const void* grad_ptrs, const void* exp_avg_ptrs, const void* exp_avg_sq_ptrs,
                 const int64_t* numel, const void* chunks, int n_chunks, int chunk_elems, const float* partials,
                 float max_norm, float skip_above, double lr, double beta1, double beta2, double eps, int step,
                 float* norm_out /* [2] */, void* stream);
/* pg_adabelief_step: the reference's AdaBelief update (optim.py, with its tuple unpack corrected) after the same norm and
 *   clip / skip rule as pg_adam_step, per element in fp32:
 *     g *= c;  m = b1 m + (1-b1) g;  e = g - m;  v = b2 v + (1-b2) e^2 + 1e-10;
 *     p -= lr * (m / (1-b1^step)) / (sqrt(v / (1-b2^step)) + 1e-10)
 *   lr, b1, b2, 1-b1, 1-b2 and both bias corrections are computed in double and rounded to fp32.  `chunks` / n_chunks
 *   are this launch's slice of the chunk table (one launch per parameter group, each with its own lr / betas / step);
 *   the norm is the sum of all n_partials partials of one pg_grad_sqnorm pass over every group, so every launch sees
 *   the same norm and writes the same norm_out[0..1] (meaning as in pg_adam_step). */
int pg_adabelief_step(const void* param_ptrs, const void* grad_ptrs, const void* ema_avg_ptrs, const void* ema_var_ptrs,
                      const int64_t* numel, const void* chunks, int n_chunks, int chunk_elems, const float* partials,
                      int n_partials, float max_norm, float skip_above, double lr, double beta1, double beta2, int step,
                      float* norm_out, void* stream);

/* ---------------------------------------------------------------------------------------------
 * MADE — reference models/autoregressive/made.py (MaskedLinear: `weight.data *= mask` then F.linear; MADE._sample_masks
 * builds every mask on the host from connectivity vectors; MADE._sample runs one full forward per input dimension).
 *
 * pg_made_mask_cast: the connectivity mask of one layer, mask[o, i] = conn_in[i] <= conn_out[o] (strict = 1: <, the
 *   output layer), applied to the fp32 weight w [rows, cols] (row-major) in place (w *= mask) and, in the same pass, the
 *   bf16 GEMM operand w_bf16 [rows_p >= rows, ld_bf16 >= cols] = bf16(w * mask), zero in the pad rows and columns.
 *   mask (fp32 [rows, cols], or NULL): receives the 0/1 mask (the layer's `mask` buffer).  conn_in [cols] and
 *   conn_out [rows] are int32 device vectors.
 *
 * pg_made_sample_step: one dimension of incremental sampling for a batch of n images of D dimensions, one block per image.
 *   The step index is read from *pos (device memory) so that one captured CUDA graph serves every step; order [D] lists
 *   the dimensions in sampling order.  h1 [n, H] fp32 holds the first layer's pre-activation W1 x_in + b1, kept in step
 *   with the canvas [n, D] fp32 through x_in [n, D] (the canvas values h1 was computed from):
 *     update = 2: h1 += W1 (canvas - x_in) over every dimension, then x_in = canvas (the start of a sampling call);
 *     update = 1: the same for the dimension order[t - 1] only, t = *pos (nothing at t = 0);
 *     update = 0: h1 is not touched.
 *   w1t [D, H] fp32 is the masked first-layer weight transposed, so a dimension's column is contiguous.
 *   a1 (bf16 [n, ld_a1], or NULL) receives relu(h1) (the operand of a second hidden layer).
 *   logits (fp32 [n], or NULL) receive, for d = order[t], b_out[d] + sum_k act[k] * w_out[d, k] with w_out [D, K] fp32
 *   and act = relu(h1) (K == H) or, when hl is given, the bf16 activations hl [n, ld_hl] of the last hidden layer.
 * ------------------------------------------------------------------------------------------- */
int pg_made_mask_cast(float* w, int rows, int cols, const int* conn_in, const int* conn_out, int strict, void* w_bf16,
                      int rows_p, int64_t ld_bf16, float* mask, void* stream);
int pg_made_sample_step(const int64_t* pos, const int* order, int D, int n, const float* canvas, float* x_in,
                        const float* w1t, float* h1, int H, int update, void* a1_bf16, int64_t ld_a1, const void* hl_bf16,
                        int64_t ld_hl, const float* w_out, int K, const float* b_out, float* logits, void* stream);

/* ---------------------------------------------------------------------------------------------
 * NADE — reference models/autoregressive/nade.py (`_forward`: a Python loop over the D input dimensions, about ten
 * tiny ops per dimension, replayed by autograd).  Parameters in_w [H, D], in_b [H], h_w [D, H], h_b [D], fp32
 * row-major; x [n, D] fp32.  Per image, with x~ the effective input:
 *   a_0 = in_b,  a_d = a_{d-1} + x~_{d-1} * in_w[:, d-1]  (a separately rounded multiply and add, in index order),
 *   p_d = sigmoid(h_w[d] . relu(a_d) + h_b[d]),  x~_d = x_d where x_d >= 0, else (u_d < p_d ? 1 : 0).
 *
 * pg_nade_fwd: the whole scan in one launch (after a transpose of in_w into the library's scratch).  u [n, D]: uniforms
 *   for the entries to draw.  Writes p [n, D] (or NULL), x~ into xt [n, D] and, when ckpt is not NULL, the checkpoints
 *   ckpt [n, ceil(D / PG_NADE_CHUNK), H] = a_{c * PG_NADE_CHUNK} for the backward.  One image's results do not depend
 *   on the other images of the batch.  Any H: above 16384 units `a` is kept in the scratch instead of registers.
 *   n = 0 (both functions) does nothing.
 * pg_nade_bwd: the gradients of one forward, from its x, xt, p and ckpt and g = dL/dp [n, D]:
 *   d_h_w[d, h] += sum_n gz[n,d] relu(a[n,d,h]),  d_h_b[d] += sum_n gz[n,d],  gz = g (1 - p) p,
 *   d_in_w[h, i] += sum_n x~[n,i] s_i[n,h],  d_in_b[h] += sum_n s_{-1}[n,h],  s_i = sum_{d > i} gz_d h_w[d] [a_d > 0],
 *   dx[n, i] += in_w[:, i] . s_i[n] where x[n, i] >= 0 (no gradient flows through a drawn entry); dx may be NULL.
 *   Partial sums go through the library's scratch and are added in a fixed order.
 * ------------------------------------------------------------------------------------------- */
#define PG_NADE_CHUNK 16
int pg_nade_fwd(const float* x, const float* u, const float* in_w, const float* in_b, const float* h_w, const float* h_b,
                int n, int D, int H, float* p, float* xt, float* ckpt, void* stream);
int pg_nade_bwd(const float* x, const float* xt, const float* p, const float* g, const float* ckpt, const float* in_w,
                const float* h_w, int n, int D, int H, float* d_in_w, float* d_in_b, float* d_h_w, float* d_h_b,
                float* dx, void* stream);

/* ---------------------------------------------------------------------------------------------
 * FVBN — reference models/autoregressive/fvbn.py (`FullyVisibleBeliefNetwork`: D modules nn.Linear(max(1, i), 1), a
 * Python loop of D tiny GEMMs and a stack).  Row i has len(i) = max(1, i) weights W_i [len(i)] and a bias b_i; the
 * parameters stay separate tensors and the kernels read them through a device table of addresses:
 * params [2 * D] int64 = (address of W_0, ..., W_{D-1}, address of b_0, ..., b_{D-1}), fp32 contiguous each.
 * x [n, D] fp32 row-major.  Row 0 takes the constant input 0 (PyTorch has no zero-width Linear), rows i >= 1 take
 * x[:, :i]:
 *   logit[b, i] = b_i + sum_{j < len(i)} W_i[j] xin[b, i, j],   xin = 0 for i = 0, x[b, j] otherwise.
 * Summation order (the forward and the sample step share it, so their logits are bit-identical): one fmaf chain per
 * output, acc = 0, acc = fmaf(W_i[j], xin, acc) for j = 0, 1, ..., len(i) - 1 in ascending order, then acc + b_i.  Row 0
 * is computed with real arithmetic (fmaf(W_0[0], 0, 0)), so a non-finite W_0 propagates as in the reference.
 * Packed weight-gradient layout: row i starts at off(i) = 0 for i = 0 and 1 + i (i - 1) / 2 otherwise, len(i) entries,
 * T = 1 + D (D - 1) / 2 in all.
 *
 * pg_fvbn_fwd: logits [n, D].  One launch; one image's logits do not depend on the other images of the batch.
 * pg_fvbn_bwd: from g = dL/dlogits [n, D]:
 *   dw [T] += packed dW_i[j] = sum_b g[b, i] xin[b, i, j],   db [D] += sum_b g[b, i],
 *   dx [n, D] = dx[b, j] = sum_{i > j} g[b, i] W_i[j]   (written, not added; dx may be NULL: no input gradient).
 *   Every sum runs in a fixed order: over images in index order within a batch slice, the slices' partials written to
 *   the library's scratch and added by pg_sum_partials; over rows i in ascending order for dx.  No atomics.  Two
 *   launches at any D and n when db directly follows dw in memory (db == dw + T: the tile kernel and one sum over both),
 *   three otherwise (a sum per output); the results are the same bits either way.
 * pg_fvbn_sample_step: the c logits of one pixel for raster-order sampling of images [c, hw] (D = c * hw): for the
 *   pixel p = *pos (an int64 in device memory, so that one captured CUDA graph serves every step) and each channel ch,
 *   logits[b, ch] = logit[b, ch * hw + p] of the live canvas [n, D], in the forward's order.
 * Any D >= 1, any n >= 0 (n = 0 does nothing).
 * ------------------------------------------------------------------------------------------- */
int pg_fvbn_fwd(const int64_t* params, const float* x, int n, int D, float* logits, void* stream);
int pg_fvbn_bwd(const int64_t* params, const float* x, const float* g, int n, int D, float* dw, float* db, float* dx,
                void* stream);
int pg_fvbn_sample_step(const int64_t* params, const int64_t* pos, const float* canvas, int n, int c, int hw,
                        float* logits, void* stream);

/* ---------------------------------------------------------------------------------------------
 * NICE — reference models/flow/nice.py (`AdditiveCouplingBlock`, `ScalingLayer`, the recipe's logistic prior).  The
 * coupling networks run on pg_gemm_bf16; these are the elementwise ends of the flow.  The flow's stream is two fp32
 * half buffers of x [n, D] (row-major, fp32):
 *   lo [n, ld] = x[:, :D/2],  hi [n, ld] = x[:, D/2:]   (h_lo = D/2, h_hi = D - D/2 columns; ld >= h_hi, the GEMM
 *   operand pitch round_up(h_hi, 8); columns beyond a half's width are written as zeros).
 * s = log_scale [D] fp32; NULL = no scaling.  `bf16_half` 0 / 1 names the half (lo / hi) whose bf16 copy [n, ld] is
 * written (pads zero) when the bf16 pointer is not NULL.
 *
 * pg_nice_split: lo, hi from x, each entry x[b, j] * expf(sign * s[j]) when s is given (the inverse's entry, sign = -1),
 *   copied exactly otherwise.
 * pg_nice_join: z [n, D] = [lo | hi] * expf(sign * s) (an exact copy without s); with log_det (a device scalar, needs s)
 *   also log_det = sum_j s[j], one fp32 chain in ascending j.  n = 0 with log_det writes log_det alone.
 * pg_nice_scale_bwd: the scaling's backward from dz [n, D], its output z [n, D] and g_log_det (a device scalar, the
 *   gradient of log_det; NULL = 0):
 *   d_lo, d_hi = dz * expf(s) (split as above), the bf16 copy of half bf16_half into dm_bf16,
 *   d_log_scale [D] = g_log_det + sum_b dz[b, j] z[b, j]   (written, not added).
 *   The sum over images runs in index order within batch slices of up to 128 images (one fmaf chain per column), and
 *   the slices' partials are added in slice order by pg_sum_partials: two launches.  n = 0 gives d_log_scale = g_log_det.
 * pg_logistic_prior_fwd_bwd: per image log_prob[b] = -sum_j (softplus(z) + softplus(-z)), computed as
 *   |z| + 2 log1p(exp(-|z|)); one CTA per image, each thread sums its columns j = t, t + 256, ... in ascending order and
 *   the 256 threads' sums are combined by a fixed tree.  In the same pass dz [n, D] = grad_scale * tanh(z / 2) (the
 *   gradient of -log_prob[b] is tanh(z / 2)) when dz is not NULL.
 * expf / log1pf / tanhf throughout (no fast-math intrinsics).  No atomics.
 * ------------------------------------------------------------------------------------------- */
int pg_nice_split(const float* x, int n, int D, const float* log_scale, float sign, float* lo, float* hi, int64_t ld,
                  int bf16_half, void* out_bf16, void* stream);
int pg_nice_join(const float* lo, const float* hi, int64_t ld, int n, int D, const float* log_scale, float sign, float* z,
                 float* log_det, void* stream);
int pg_nice_scale_bwd(const float* dz, const float* z, const float* log_scale, const float* g_log_det, int n, int D,
                      float* d_lo, float* d_hi, int64_t ld, int bf16_half, void* dm_bf16, float* d_log_scale,
                      void* stream);
int pg_logistic_prior_fwd_bwd(const float* z, int n, int D, float grad_scale, float* log_prob, float* dz, void* stream);

/* ---------------------------------------------------------------------------------------------
 * VAE — the Gaussian latent of reference models/vae/vae.py (`forward`) and vaes.py (`unit_gaussian_kl_div`,
 * `sample_from_gaussian`).  h: the encoder's last convolution output, pixel-major fp32 [n*hw, ld_h >= 2L]: columns
 * [0, L) the mean, [L, 2L) log_std.  eps: the noise in the reference's NCHW order, fp32 [n, L, hw].
 * pg_vae_latent_fwd: z = mean + exp(log_std) * eps as bf16 [n*hw, ld_z] (ld_z % 8 == 0, zero in columns >= L) and
 *   kl[b] = sum over image b of -0.5 (1 + 2 log_std - exp(log_std)^2 - mean^2).  One CTA per image: each thread sums
 *   its entries in ascending order and the threads are combined by a fixed tree.  Every product and sum is rounded on
 *   its own, as in the reference.
 * pg_vae_latent_bwd: from dz (bf16 [n*hw, ld_dz]) and g_kl (fp32 [n], the gradient of kl; NULL = 0) writes
 *   dh (bf16 [n*hw, ld_dh], ld_dh % 8 == 0, zero in columns >= 2L):
 *   dmean = dz + g mean,  dlog_std = dz exp(log_std) eps + g (exp(log_std)^2 - 1).
 * Both write every column up to their output's pitch (z up to ld_z, dh up to ld_dh), zeros beyond L / 2L: the output
 * must own those columns.  n = 0 does nothing.  No atomics.
 * ------------------------------------------------------------------------------------------- */
int pg_vae_latent_fwd(const float* h, int64_t ld_h, const float* eps, int n, int L, int hw, void* z, int64_t ld_z,
                      float* kl, void* stream);
int pg_vae_latent_bwd(const float* h, int64_t ld_h, const float* eps, const void* dz, int64_t ld_dz, const float* g_kl,
                      int n, int L, int hw, void* dh, int64_t ld_dh, void* stream);

/* ---------------------------------------------------------------------------------------------
 * VeryDeepVAE — the stages of reference models/vae/vd_vae.py between its convolutions.  Streams are pixel-major fp32
 * [n*h*w, ld >= C].  Every access is scalar: no operand needs an aligned base, and column views are fine.  Every sum
 * runs in a fixed order, no kernel uses atomics, and nothing synchronises with the host.
 * pg_gelu_cast: g = bf16(GELU(x)) and d = bf16(GELU'(x)) from fp32 x [P, ld_x >= C] into columns [0, width) of two
 *   bf16 matrices with pitch ld_out (g and d may point into a wider operand, e.g. its second half); columns [C, width)
 *   get 0.  The same GELU fit and derivative as the GEMM epilogue's PG_ACT_GELU | PG_ACT_STORE_DERIV.
 * pg_vd_latent_fwd: a TopDownBlock's latent.  prior: fp32 [n*hw, ld_prior >= 2L + C], columns p_mean | p_log_std | p_h;
 *   post: fp32 [n*hw, ld_post >= 2L], q_mean | q_log_std, or NULL to sample from the prior; x: the block's input
 *   stream [n*hw, ld_x >= C]; eps: fp32 [n, L, hw] (NCHW).  Writes z = mean + exp(log_std) eps as bf16
 *   [n*hw, ld_z] (zero in columns [L, ld_z)), s = x + p_h (fp32 [n*hw, ld_s >= C]) and, with post,
 *   kl_out[b] = kl_in[b] + sum over image b of KL(q || p) = -0.5 + (t - s) + (e^{2s} + (m_q - m_p)^2) / (2 e^{2t})
 *   (kl_in NULL = 0; kl_out may be kl_in).  Each operation is rounded on its own, in the reference's order.  One CTA per
 *   image: each thread sums its entries in ascending order and the threads are combined by a fixed tree.
 * pg_vd_latent_bwd: from dz (bf16 [n*hw, ld_dz >= L], NULL = 0), g_kl (fp32 [n], NULL = 0) and dsum (the fp32
 *   gradient of s, [n*hw, ld_dsum >= C]) writes dprior = [dp_mean | dp_log_std | bf16(dsum)] (bf16 [n*hw, ld_dprior])
 *   and dpost = [dq_mean | dq_log_std] (bf16 [n*hw, ld_dpost]; NULL exactly when post is), zero up to each pitch.
 *   With d = m_q - m_p and v = e^{2t}: dm_q = dz + g d / v, d(q_log_std) = dz e^s eps + g (e^{2s} / v - 1),
 *   dm_p = -g d / v, d(p_log_std) = g (1 - (e^{2s} + d^2) / v).  From the prior: dm_p = dz, d(p_log_std) = dz e^t eps.
 * pg_avg_pool2_fwd / _bwd: nn.AvgPool2d(2, 2) of x [n*h*w, C] into y [n*(h/2)*(w/2), C] (odd sides floored), and its
 *   adjoint: dx = dy / 4 under each window, 0 at the pixels no window covers.
 * pg_bias_unpool_fwd: y = up_f(x + bias), f = 1 or 2 (nearest neighbour): x [n*s*s, C] or NULL (= 0), bias the NCHW
 *   parameter [1, C, s, s], y [n*(f s)^2, C].  _bwd: dx (NULL = not wanted) = the sum of each pixel's f x f children
 *   in raster order, dbias[c, i, j] = that sum added over the images in ascending order (overwritten, not accumulated).
 * ------------------------------------------------------------------------------------------- */
int pg_gelu_cast(const float* x, int64_t ld_x, int P, int C, int width, void* g, void* d, int64_t ld_out, void* stream);
int pg_vd_latent_fwd(const float* prior, int64_t ld_prior, const float* post, int64_t ld_post, const float* x,
                     int64_t ld_x, const float* eps, int n, int L, int C, int hw, void* z, int64_t ld_z, float* s,
                     int64_t ld_s, const float* kl_in, float* kl_out, void* stream);
int pg_vd_latent_bwd(const float* prior, int64_t ld_prior, const float* post, int64_t ld_post, const float* eps,
                     const void* dz, int64_t ld_dz, const float* g_kl, const float* dsum, int64_t ld_dsum, int n, int L,
                     int C, int hw, void* dprior, int64_t ld_dprior, void* dpost, int64_t ld_dpost, void* stream);
int pg_avg_pool2_fwd(const float* x, int64_t ld_x, int n, int h, int w, int C, float* y, int64_t ld_y, void* stream);
int pg_avg_pool2_bwd(const float* dy, int64_t ld_dy, int n, int h, int w, int C, float* dx, int64_t ld_dx, void* stream);
int pg_bias_unpool_fwd(const float* x, int64_t ld_x, const float* bias, int n, int s, int C, int f, float* y,
                       int64_t ld_y, void* stream);
int pg_bias_unpool_bwd(const float* dy, int64_t ld_dy, int n, int s, int C, int f, float* dx, int64_t ld_dx,
                       float* dbias, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Vector quantizer — reference nn/utils.py `VectorQuantizer` (VQ-VAE, VQ-VAE-2).  x: pixel-major fp32 rows [P, ld_x]
 * (the reference's flat_x, d = embedding_dim columns); emb: the codebook, fp32 [K, d] contiguous.  Every sum runs in a
 * fixed order and no kernel uses atomics: every run is bit-identical.
 * pg_vq_assign: idx[r] (int32) = argmin over k of (|x_r|^2 + |e_k|^2) - 2 x_r.e_k, in fp32 on the CUDA cores, the first
 *   minimal index on ties (codes scanned in ascending order with a strict <).  The codebook is staged in shared memory in
 *   chunks.  When out is not NULL it writes x + (q - x) (q = emb[idx[r]]) to columns [col0, col0 + d) of out (bf16, or
 *   fp32 when out_f32) with row pitch ld_out, and zeros to [col0 + d, col0 + out_cols).  When loss_sum is not NULL,
 *   *loss_sum += sum over rows and columns of (x - q)^2 (per-CTA partials added by pg_sum_partials: two launches).
 * pg_vq_code_sums: counts[k] = rows assigned to k (may be NULL; exact up to 2^24 rows) and sums[k, :] (fp32 [K, d],
 *   overwritten) = sum over those rows, in ascending row order, of x_r, or, when emb is not NULL, of
 *   ((q_r - x_r) scale) g[0] (the codebook gradient of mse(q, x) with scale = 2 / numel).  A code with no rows gets 0.
 * pg_vq_ema_update: per code, cs = decay cs + one_minus_decay counts, avg = decay avg + one_minus_decay sums,
 *   emb = avg / (cs + 1e-5), in place.
 * pg_vq_bwd: dx[r, c] = dq[r, col0 + c] + ((x - q) scale) g[0] for c < d, 0 for d <= c < ld_dx (dq NULL = 0, g NULL = 0);
 *   dq and dx are bf16, or fp32 when f32.
 * ------------------------------------------------------------------------------------------- */
int pg_vq_assign(const float* x, int64_t ld_x, int P, int d, const float* emb, int K, int* idx, void* out, int out_f32,
                 int64_t ld_out, int col0, int out_cols, float* loss_sum, void* stream);
int pg_vq_code_sums(const float* x, int64_t ld_x, int P, int d, const int* idx, int K, const float* emb, const float* g,
                    float scale, float* counts, float* sums, void* stream);
int pg_vq_ema_update(const float* counts, const float* sums, int K, int d, float decay, float one_minus_decay,
                     float* cluster_size, float* embedding_avg, float* embedding, void* stream);
int pg_vq_bwd(const float* x, int64_t ld_x, int P, int d, const float* emb, const int* idx, const void* dq, int64_t ld_dq,
              int col0, const float* g, float scale, int f32, void* dx, int64_t ld_dx, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Mean squared error — F.mse_loss(a, b) of the VQ-VAE recipes and of VQ-VAE-2's mse(decoded_t, encoded_b).  a, b: fp32
 * [rows, cols] with pitches ld_a, ld_b (pixel-major, or NCHW seen as [n*c*h, w]).
 *   forward (loss_sum given, g NULL): *loss_sum += sum of (a - b)^2 (per-CTA partials added by pg_sum_partials);
 *   backward (g given, loss_sum NULL): da = ((a - b) scale) g[0] (pitch ld_da) and db = -da (pitch ld_db), each zero in
 *   its columns [cols, pitch); either may be NULL.  scale = 2 / numel.
 * ------------------------------------------------------------------------------------------- */
int pg_mse_mean(const float* a, int64_t ld_a, const float* b, int64_t ld_b, int rows, int cols, const float* g,
                float scale, float* loss_sum, float* da, int64_t ld_da, float* db, int64_t ld_db, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Density estimators — reference models/kde.py (`GaussianKernel`, `ParzenWindowKernel`) and models/mixture_models.py
 * (`GaussianMixtureModel`, `BernoulliMixtureModel`).  Queries x: fp32 [N, D] contiguous; training points t: fp32
 * [M, D] contiguous; mixture parameters fp32 [K, D] contiguous.  Every kernel runs in fp32 on the CUDA cores over
 * 64 x 64 tiles of (query, codebook row) pairs with D streamed through shared memory in chunks of 32: nothing of N x M
 * (or N x K x D) elements is ever allocated.  Splits write partials to the library scratch and are added in split order:
 * of the codebook rows for the KDE (up to 32 from M alone; 8 for the backward), of D for the mixture forward (up to 8
 * from D alone), so a query's result does not depend on its batch; of the batch for the mixture backward (from K, D
 * and the SM count).  No atomics: every run is bit-identical.  N = 0 launches nothing.
 *
 * pg_kde_gauss_fwd: s_nm = (-0.5 / h^2) * sum_d (x_nd - t_md)^2 (direct differences, one fmaf chain per pair in
 *   ascending d), lse[n] = logsumexp_m s_nm from per-split online (max, sum) states merged in split order with each
 *   sum rescaled by exp(m_s - max); out[n] = lse[n] - Z.  lse may be NULL.  Two launches.
 * pg_kde_gauss_bwd: dx[n, d] += -(g_n / h^2) sum_m w_nm (x_nd - t_md), w_nm = exp(s_nm - lse_n) recomputed per
 *   training tile (each tile read twice: the pair sums over all of D, then the weighted D-chunks); per-split partials
 *   [splits, N, D] added by pg_sum_partials.  dx is added to (zero it first).  Two launches.
 * pg_kde_parzen_count: count[n] = the training rows with fl(|x_nd - t_md| / h) <= 0.5 (IEEE fp32 division, h rounded to
 *   fp32) for every d, evaluated exactly as |x_nd - t_md| <= a*, a* the largest fp32 whose quotient rounds to <= 0.5;
 *   out[n] = log(count) - log(M) - D log(h) in fp64, rounded to fp32 (-inf for a zero count).  Either output may be
 *   NULL.  M < 2^24.  Two launches.
 * pg_mixture_fwd (kind PG_MIXTURE_GAUSSIAN: p0 = mean, p1 = log_std; PG_MIXTURE_BERNOULLI: p0 = logits, p1 unused):
 *   a[n, k] = log_softmax(mixture_logits)_k + sum_d term(x_nd; k, d), out[n] = logsumexp_k a[n, k];
 *   Gaussian term (-log_std - 0.5 log 2pi) - 0.5 ((x - mean) / exp(log_std))^2 with an IEEE division; Bernoulli term
 *   l x - (max(l, 0) + log1p(exp(-|l|))).  Feature splits when the batch tiles alone cannot fill the GPU; the splits'
 *   sums are added in split order by the second launch.  K <= 8192.  Two launches.
 * pg_mixture_bwd: with r = exp(a - out) and the cotangent g [N]:
 *   dparams (fp32, added to) = [dmean (K D) | dlog_std (K D) | dmixture_logits (K)] (Gaussian) or
 *   [dlogits (K D) | dmixture_logits (K)] (Bernoulli), each sum over n of g r times (x - mean) / std^2,
 *   ((x - mean) / std)^2 - 1, x - sigmoid(l); dmixture_logits_k = sum_n g_n r_nk - softmax_k sum_n g_n.  Batch-slice
 *   partials added by pg_sum_partials.  dx [N, D] (written; NULL = none) = sum_k g r (mean - x) / std^2 or g r l.
 *   Two launches, three with dx.
 * ------------------------------------------------------------------------------------------- */
#define PG_MIXTURE_GAUSSIAN 0
#define PG_MIXTURE_BERNOULLI 1
int pg_kde_gauss_fwd(const float* x, int N, const float* t, int M, int D, float bandwidth, float Z, float* lse,
                     float* out, void* stream);
int pg_kde_gauss_bwd(const float* x, int N, const float* t, int M, int D, float bandwidth, const float* lse,
                     const float* g, float* dx, void* stream);
int pg_kde_parzen_count(const float* x, int N, const float* t, int M, int D, double bandwidth, int* count, float* out,
                        void* stream);
int pg_mixture_fwd(int kind, const float* x, int N, int D, int K, const float* mixture_logits, const float* p0,
                   const float* p1, float* a, float* out, void* stream);
int pg_mixture_bwd(int kind, const float* x, int N, int D, int K, const float* mixture_logits, const float* p0,
                   const float* p1, const float* a, const float* out, const float* g, float* dparams, float* dx,
                   void* stream);

/* ---------------------------------------------------------------------------------------------
 * Gaussian process — the dense fp64 linear algebra of reference models/gaussian_process.py.  Row-major fp64 device
 * buffers, 64-bit offsets, no atomics, no host synchronisation; every sum runs in a fixed order.
 *
 * pg_gemm_f64: C = alpha op(A) op(B) + beta C, op(A) [m, k], op(B) [k, n]; op(A)[i][p] = A[i lda + p] (transA = 0) or
 *   A[p lda + i] (transA = 1), likewise B.  FP64 tensor cores (mma.sync m16n8k16 .f64) on 64 x 64 tiles; each element
 *   sums over k in ascending chunks of 16, so its bits depend on k alone, not on m, n or its tile.  beta == 0 does not
 *   read C; alpha == 0 gives beta C.  lower_only: only elements (i, j) with j <= i are written (the SYRK form).  One
 *   launch (none when m or n is 0).
 * pg_gp_potrf: A [n, n] (pitch lda) gets noise added to its diagonal and its strict upper triangle zeroed, then is
 *   factored in place into its lower Cholesky factor L, blocked by 64: per block column a one-CTA diagonal factor, a
 *   panel solve and a lower_only trailing update on pg_gemm_f64.  A pivot d with isfinite(d) && d <= tau, tau =
 *   n 2^-52 max_i A_ii (after the noise; LAPACK dpstrf's default tolerance), is dropped: its whole column of L is 0 and
 *   it is counted in the device int *dropped (reset by the call).  A NaN pivot propagates.  tau lives in the library
 *   scratch.  3 ceil(n / 64) - 1 launches.
 * pg_gp_trsm: solves L X = B (transpose = 0) or L^T X = B (transpose = 1) in place, L [n, n] lower (pitch n), B
 *   [n, ncols] (pitch ncols): 64-row diagonal-block solves with the off-diagonal updates on pg_gemm_f64.  A zero
 *   diagonal entry gives a zero row of X.  Columns are independent: a subset of B's columns gives the same bits.
 *   2 ceil(n / 64) - 1 launches.
 * ------------------------------------------------------------------------------------------- */
int pg_gemm_f64(int transA, int transB, int m, int n, int k, double alpha, const double* A, int64_t lda, const double* B,
                int64_t ldb, double beta, double* C, int64_t ldc, int lower_only, void* stream);
int pg_gp_potrf(double* A, int n, int64_t lda, double noise, int* dropped, void* stream);
int pg_gp_trsm(const double* L, int n, double* B, int ncols, int transpose, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* PG_B200_H_ */
