/*
 * micronet_b200 — C-ABI of the H100 (sm_90a) fake-quant conv/linear engine.
 *
 * The reference (666DZY666/micronet) has no FFI: its hot path is Python
 * nn.Module code that composes ATen ops.  This header is the boundary a
 * maintainer binds instead (ctypes stub in INTEGRATION.md): plain device
 * pointers, sizes and a cudaStream_t — no torch types.  Every entry point
 * cites the reference lines it replaces; aliases:
 *   DF  = micronet/compression/quantization/wqaq/dorefa/quantize.py
 *   WB  = micronet/compression/quantization/wbwtab/quantize.py
 *   IAO = micronet/compression/quantization/wqaq/iao/quantize.py
 *
 * Conventions
 *   - all pointers are DEVICE pointers unless the name ends in _host;
 *   - tensors are contiguous fp32 NCHW (weights KCRS) as at the reference's
 *     module surface; "codes" are u8 integer levels (level - qmin);
 *   - every call is asynchronous on `stream`, allocates nothing and keeps no
 *     pointer after returning; scratch is passed in by the caller;
 *   - return value: 0 = ok, <0 = invalid argument (MNB_E_*), >0 = cudaError_t;
 *     mnb_last_error() gives a thread-local message.
 */
#ifndef MICRONET_B200_H
#define MICRONET_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef void* mnb_stream_t; /* cudaStream_t */

#define MNB_E_ARG (-1)         /* bad shape / null pointer / unsupported bits */
#define MNB_E_UNSUPPORTED (-2) /* valid request this build has no kernel for  */

int mnb_version(void);
const char* mnb_last_error(void);
/* number of kernel launches issued through this library since load (bench.py's gpu_launches) */
int64_t mnb_launch_count(void);

/* ------------------------------------------------------------------------
 * Convolution geometry (F.conv2d arguments: WB:186-194, DF:113-121, IAO:498-506)
 * ---------------------------------------------------------------------- */
typedef struct {
  int32_t batch, in_c, in_h, in_w;
  int32_t out_c, ker_h, ker_w;
  int32_t stride_h, stride_w, pad_h, pad_w, dil_h, dil_w, groups;
} mnb_conv_shape;

/* ------------------------------------------------------------------------
 * Activation fake-quantizers
 * ---------------------------------------------------------------------- */
#define MNB_ACT_DOREFA 1 /* DF:36-46   clamp(0.1x,0,1) -> round(./s), s = 1/(2^a-1)      */
#define MNB_ACT_IAO 2    /* IAO:214-240 clamp(round(x/s - zp), qmin, qmax)              */
#define MNB_ACT_SIGN 3   /* WB:11-36   sign(x) with 0 -> +1, saturate-STE               */

typedef struct {
  int32_t mode;        /* MNB_ACT_*                                                    */
  int32_t bits;        /* DoReFa a_bits (2..8)                                         */
  int32_t qmin, qmax;  /* IAO level range (IAO:243-288)                                */
  int32_t q_type;      /* IAO: 0 symmetric / 1 asymmetric STE range (IAO:148-157)      */
  const float* scale;  /* IAO: device scalar `scale`                                   */
  const float* zero_point; /* IAO: device scalar `zero_point`                          */
  const float* obs_min;    /* IAO: device scalar observer.min_val                      */
  const float* obs_max;    /* IAO: device scalar observer.max_val                      */
} mnb_act_qparams;

/* Forward.  Any of the three outputs may be NULL.
 *   codes    u8[n]      level - level_min   (DoReFa/IAO; SIGN: 0 or 2 so that e = code-1)
 *   pass_bits u32[ceil(n/32)]  bit i set  <=>  the STE passes the gradient at element i
 *   xq       f32[n]     the fake-quantized tensor the reference module returns           */
int mnb_act_quant_fwd(const float* x, int64_t n, const mnb_act_qparams* qp, uint8_t* codes,
                      uint32_t* pass_bits, float* xq, mnb_stream_t stream);
/* Backward of the same op (autograd of DF:43-45 / IAO:227-239 / WB:22-36):
 *   DoReFa dx = (((g*s)/s) * pass) * 0.1 ; IAO dx = ((g*s) * pass) / s ; SIGN dx = g * pass   */
int mnb_act_quant_bwd(const float* g, const uint32_t* pass_bits, int64_t n, const mnb_act_qparams* qp,
                      float* dx, mnb_stream_t stream);

/* IAO QuantBNFuseConv2d (IAO:858-945): fold BatchNorm statistics into (weight, bias) before quantization, one launch:
 *   ratio = gamma / sqrt(var + eps);  w_fused[k, :] = w[k, :] * ratio[k];  b_fused = beta + (bias - mean) * ratio  (bias may
 *   be NULL).  Backward: dw = dw_fused * ratio and out6[k] = {dgamma, dbeta, dbias, dmean, dvar, 0}.
 * mnb_bn_fold_running: running_mean / running_var <- batch statistics (first call) or (1 - momentum) r + momentum batch. */
int mnb_bn_fold_fwd(const float* w, int32_t out_c, int32_t per_channel, const float* gamma, const float* beta,
                    const float* bias, const float* mean, const float* var, double eps, float* w_fused, float* b_fused,
                    mnb_stream_t stream);
int mnb_bn_fold_bwd(const float* dw_fused, const float* db_fused, const float* w, int32_t out_c, int32_t per_channel,
                    const float* gamma, const float* bias, const float* mean, const float* var, double eps, float* dw,
                    float* out6, mnb_stream_t stream);
int mnb_bn_fold_running(float* running_mean, float* running_var, const float* batch_mean, const float* batch_var, int32_t n,
                        double momentum, int32_t first, mnb_stream_t stream);

/* IAO QuantAdd (IAO:1441-1498) in one pass: out = Q(a) + Q(b) with the shared union-range quantizer (read both addends
 * once, write the sum; pass masks for the backward pass, either may be NULL).  Backward: da = STE_a(g), db = STE_b(g). */
int mnb_quant_add_fwd(const float* a, const float* b, int64_t n, const mnb_act_qparams* qp, float* out,
                      uint32_t* pass_bits_a, uint32_t* pass_bits_b, int32_t relu /* out = max(., 0): inference graphs */,
                      mnb_stream_t stream);
int mnb_quant_add_bwd(const float* g, const uint32_t* pass_bits_a, const uint32_t* pass_bits_b, int64_t n,
                      const mnb_act_qparams* qp, float* da, float* db, mnb_stream_t stream);

/* ------------------------------------------------------------------------
 * IAO observers + update_qparams (IAO:15-139, 292-321), all on device, no host sync.
 *   observer kinds: 0 = MinMaxObserver (running extremum), 1 = MovingAverageMinMaxObserver,
 *                   2 = HistogramObserver (EMA of the k-th smallest |x|, k=int(p*n))
 *   `first` = 1 on the observer's first call (the reference's num_flag == 0 branch).
 *   `rows`  = 1 for q_level "L"; = out_channels for "C"/"FC" (x viewed as [rows, n/rows]).
 *   min_val/max_val/scale/zero_point: the module's registered buffers (rows floats each).
 *   symmetric: 1 -> SymmetricQuantizer, 0 -> AsymmetricQuantizer.  update_qparams=0 only observes.
 *   scratch: >= mnb_observe_scratch_bytes(n, rows) bytes, zero-initialised once by the caller
 *   (the kernels leave it zeroed again).                                                   */
int64_t mnb_observe_scratch_bytes(int64_t n, int32_t rows);
int mnb_iao_observe(const float* x, int64_t n, int32_t rows, int32_t observer_kind, int32_t first,
                    double momentum, double percentile, float* min_val, float* max_val,
                    int32_t update_qparams, int32_t symmetric, int32_t qmin, int32_t qmax,
                    float* scale, float* zero_point, void* scratch, mnb_stream_t stream);
/* update_qparams only (QuantAdd's union range, IAO:1487-1494). */
int mnb_iao_update_qparams(const float* min_val, const float* max_val, int32_t rows, int32_t symmetric,
                           int32_t qmin, int32_t qmax, float* scale, float* zero_point,
                           mnb_stream_t stream);

/* ------------------------------------------------------------------------
 * Weight quantizers.  Forward writes
 *   w_int   i16[numel]  effective integer e with  wq = e * w_scale[k]   (exact)
 *   w_scale f32[K]      per-output-channel dequantization scale
 *   wq      f32[numel]  the fake-quantized weight the reference feeds F.conv2d
 * and whatever the closed-form backward needs in `aux`.
 * ---------------------------------------------------------------------- */
/* DF:61-73.  aux: f32[numel + 4] (tanh values, then {max|t|, #ties, s, -}).  scratch as above. */
int mnb_dorefa_weight_fwd(const float* w, int64_t numel, int32_t out_c, int32_t w_bits, int16_t* w_int,
                          float* w_scale, float* wq, float* aux, void* scratch, mnb_stream_t stream);
int mnb_dorefa_weight_bwd(const float* g_wq, const float* aux, int64_t numel, int32_t w_bits, float* dw,
                          void* scratch, mnb_stream_t stream);
/* WB:98-149.  W = 2 (binary; MUTATES w in place: mean-centre over dim 1 + clamp, WB:98-102)
 *             W = 3 (ternary).  w is [out_c, in_c_per_group, kh*kw].
 * aux: f32[3*out_c] = {alpha_k, threshold_k, count_k}.                                          */
int mnb_wb_weight_fwd(float* w, int32_t out_c, int32_t in_c_per_group, int32_t ker_hw, int32_t W,
                      int16_t* w_int, float* w_scale, float* wq, float* aux, mnb_stream_t stream);
int mnb_wb_weight_bwd(const float* g_wq, const float* w, const float* aux, int32_t out_c,
                      int32_t in_c_per_group, int32_t ker_hw, int32_t W, float* dw, mnb_stream_t stream);
/* IAO:214-240 on a weight tensor with per-row (rows = out_c) or per-layer (rows = 1) qparams that
 * were just refreshed by mnb_iao_observe.  pass: u8[numel] STE mask.                           */
int mnb_iao_weight_fwd(const float* w, int64_t numel, int32_t out_c, int32_t rows, const float* scale,
                       const float* zero_point, const float* obs_min, const float* obs_max,
                       int32_t q_type, int32_t qmin, int32_t qmax, int16_t* w_int, float* w_scale,
                       float* wq, uint8_t* pass, mnb_stream_t stream);
int mnb_iao_weight_bwd(const float* g_wq, const uint8_t* pass, const float* scale, int64_t numel,
                       int32_t out_c, int32_t rows, float* dw, mnb_stream_t stream);

/* ------------------------------------------------------------------------
 * Fake-quantized convolution (WB:186, DF:113, IAO:498/947) and its autograd (ATen
 * convolution_backward).  F.linear (DF:198, IAO:1156) is the 1x1 case on a [B, C, 1, 1] view.
 *
 * Activation operand:  a_codes != NULL : u8 codes, effective integer e_a = code + a_offset,
 *                                        value = e_a * a_scale[0]; a_offset_zp (device scalar,
 *                                        may be NULL) is added to a_offset (IAO zero_point);
 *                      else            : a_f32 raw fp32 activations.
 * Weight operand:      w_int != NULL && a_codes != NULL : exact integer path, s64 accumulate,
 *                                        y = bias + acc * (a_scale * w_scale[k]), acc rounded once;
 *                      else            : w_f32 fp32 weights, fp32 accumulate.
 * ---------------------------------------------------------------------- */
typedef struct {
  const uint8_t* a_codes;
  const float* a_f32;
  int32_t a_offset;
  const float* a_offset_zp;
  const float* a_scale; /* device scalar or NULL (= 1) */
  const int16_t* w_int;
  const float* w_scale; /* f32[out_c] */
  const float* w_f32;
  const float* bias; /* f32[out_c] or NULL */
} mnb_conv_operands;

int mnb_conv2d_fwd(const mnb_conv_shape* s, const mnb_conv_operands* op, float* y, mnb_stream_t stream);
/* dX = conv_transpose(dY, Wq) fused with the activation STE:  pass_bits/qp may be NULL (plain dgrad). */
int mnb_conv2d_dgrad(const mnb_conv_shape* s, const float* dy, const float* wq, const uint32_t* pass_bits,
                     const mnb_act_qparams* qp, float* dx, mnb_stream_t stream);
/* dWq = corr(Xq, dY); Xq given as codes (+offset, *a_scale) or fp32.  scratch >= mnb_wgrad_scratch_bytes. */
int64_t mnb_wgrad_scratch_bytes(const mnb_conv_shape* s);
int mnb_conv2d_wgrad(const mnb_conv_shape* s, const float* dy, const mnb_conv_operands* op, float* dwq,
                     void* scratch, mnb_stream_t stream);
/* per-channel sums over (B, H, W) of a [B, C, HW] tensor:
 *   stats[0..C) = sum, stats[C..2C) = sum of squares (both accumulated in fp64, stored fp32 as
 *   mean and UNBIASED variance when `as_mean_var` != 0 — torch.mean / torch.var of IAO:854-855). */
int mnb_channel_stats(const float* x, int32_t batch, int32_t channels, int32_t hw, int32_t as_mean_var,
                      float* stats, void* scratch, mnb_stream_t stream);
/* backward of (mean, var):  dx = dmean/N + dvar * 2 (x - mean)/(N-1) */
int mnb_channel_stats_bwd(const float* x, const float* mean, const float* dmean, const float* dvar,
                          int32_t batch, int32_t channels, int32_t hw, float* dx, mnb_stream_t stream);

/* ------------------------------------------------------------------------
 * Fused tensor-core forward (wgmma + TMA): fake-quantize the fp32 NCHW input on the fly while
 * it is staged for the MMA, convolve exact integer levels, scale + bias in the epilogue.
 *   qp == NULL : x is used as it is (wbwtab: +-1 or plain fp32 activations, exact 3-term bf16 split)
 *   qp != NULL : DoReFa / IAO quantizer; `codes` (u8, same shape as x) and `pass_bits`
 *                (u32[ceil(numel/32)], ZERO-INITIALISED by the caller) receive what backward needs.
 * Replaces activation_quantizer(input) + F.conv2d of DF:108-121 / IAO:493-506 / WB:186-194.
 * Returns MNB_E_UNSUPPORTED (and launches nothing) for geometries outside the kernel's cover
 * (see mnb_conv_tc.cu); the caller then composes mnb_act_quant_fwd + mnb_conv2d_fwd.
 * err_flag: device int, stays 0 unless a bounded pipeline wait timed out (a bug, never expected).
 * ---------------------------------------------------------------------- */
int mnb_fq_conv2d_fwd_tc(const mnb_conv_shape* s, const float* x, const mnb_act_qparams* qp,
                         const int16_t* w_int, const float* w_scale, const float* bias, float* y,
                         uint8_t* codes, uint32_t* pass_bits, void* wpack_scratch, int32_t* err_flag,
                         mnb_stream_t stream);
/* wpack_scratch: >= 2 * numel(w_int) bytes, 16-byte aligned (bf16 operand image of the weights). */

/* Data gradient of the same convolution on the tensor-core path (ATen convolution_backward's
 * grad_input): dx = STE( conv_transpose(dy, w_scale[k] * w_int) ), the per-channel weight scale folded
 * into dy while it is staged (exact 3-term bf16 split of the fp32 product).  pass_bits / qp NULL:
 * plain dgrad (wbwtab).  Same geometry cover and error conventions as mnb_fq_conv2d_fwd_tc.   */
int mnb_conv2d_dgrad_tc(const mnb_conv_shape* s, const float* dy, const int16_t* w_int, const float* w_scale,
                        const uint32_t* pass_bits, const mnb_act_qparams* qp, float* dx, void* wpack_scratch,
                        int32_t* err_flag, mnb_stream_t stream);
/* host only, the plan mnb_fq_conv2d_fwd_tc (dgrad = 0; quant_mode 0 = raw fp32 input, else the quantizer's mode) or
 * mnb_conv2d_dgrad_tc (dgrad != 0; quant_mode ignored) runs, from the function its launcher uses: the first min(n, 17) of
 * {NG (output channels per group: the kernel instance), TB (images per tile), TH (rows per tile), row_tiles, n_tiles, CC
 * (channels per chunk), nchunk, nst (staging slots), nop (operand buffers), slab_groups, n_slabs, collapsed (1: the
 * (H*W, C, B) tensor map of a 1x1 filter), smem_bytes, BW (padded row), npos_in (operand positions), grid (CTAs),
 * n_mma_off (entries of the per-(tap, k-step) offset table)}.  Refusals as for the launchers (MNB_E_UNSUPPORTED, the
 * reason in mnb_last_error). */
int mnb_tc_conv_plan(const mnb_conv_shape* s, int32_t dgrad, int32_t quant_mode, int32_t* out, int32_t n);

/* Weight gradient on the tensor-core path: dWq = s_a * corr(e_a, dy) with e_a re-quantized from the
 * fp32 input x on the fly (qp as in the forward; NULL = raw x, which must be bf16-exact such as the
 * +-1 activations of wbwtab - otherwise *inexact_flag is set on the device and the result is to be
 * replaced by mnb_conv2d_wgrad_cond(..., inexact_flag), which runs only when the flag is non-zero,
 * so no host synchronisation is needed).  scratch >= mnb_wgrad_tc_scratch_bytes(s) (-1: unsupported). */
int64_t mnb_wgrad_tc_scratch_bytes(const mnb_conv_shape* s);
/* host only, the plan mnb_conv2d_wgrad_tc runs, from the function its launcher uses: the first min(n, 16) of {Gb (groups
 * per channel block), nsplit (128-channel slices of one group), tap_groups, tpc (taps per CTA), n_block (activation
 * channels per CTA), CC (channels per chunk), TH, TB, nbuf (operand buffers), nst (staging slots), ranks (CTAs per
 * block), n_slabs (channel blocks x tap groups), smem_bytes, npos_d, npos_x, n_tiles}.  Refusals as for the launcher. */
int mnb_wgrad_tc_plan(const mnb_conv_shape* s, int32_t quant_mode, int32_t* out, int32_t n);
int mnb_conv2d_wgrad_tc(const mnb_conv_shape* s, const float* dy, const float* x, const mnb_act_qparams* qp,
                        float* dwq, void* scratch, int32_t* inexact_flag, int32_t* err_flag, mnb_stream_t stream);
int mnb_conv2d_wgrad_cond(const mnb_conv_shape* s, const float* dy, const mnb_conv_operands* op, float* dwq,
                          void* scratch, const int32_t* run_if_nonzero, mnb_stream_t stream);

/* Producer-side fusions of a wbwtab block (SURVEY.md 8 f2):
 *   conv -> nn.BatchNorm2d -> ActivationQuantizer(A=2) [-> nn.MaxPool2d] -> channel_shuffle -> next conv
 * (nin_gc.py:9-21 shuffle, :53-59 block, WB:79-94 binarizer).
 *
 * mnb_bn_sign_fwd / _bwd replace BatchNorm2d + binarizer:
 *   fwd : y = sign(gamma (x - mean) invstd + beta), 0 -> +1; pass bit = |bn| < 1 (saturate STE)
 *   bwd : training-mode batch-norm backward of the masked gradient (dgamma, dbeta, dx); `training` = 0
 *         uses fixed statistics (dx = gamma invstd g pass).  dx_channel_sum (may be NULL) receives
 *         sum_{b,h,w} dx per channel: the bias gradient of the convolution that produced x.
 * mean / invstd come from mnb_channel_stats(as_mean_var = 2: mean, biased var, unbiased var).
 *
 * out_shuffle_groups = sg > 1 folds the NEXT block's channel shuffle into the producer: the output is
 * written as out[:, a*sg + b] = result[:, b*(C/sg) + a] and the incoming gradient is read through the same
 * permutation; pass bits / argmax stay in the producer's own channel order.  sg = 1: no permutation.   */
/* nn.BatchNorm2d's training-mode statistics in one launch: mean_invstd[0..C) = batch mean,
 * mean_invstd[C..2C) = 1/sqrt(biased var + eps); running_mean / running_var are updated in place with `momentum`
 * (unbiased variance, torch semantics) and *num_batches_tracked (may be NULL) is incremented.              */
int mnb_bn_batch_stats(const float* x, int32_t batch, int32_t channels, int32_t hw, double eps, double momentum,
                       float* running_mean, float* running_var, int64_t* num_batches_tracked, float* mean_invstd,
                       void* scratch, mnb_stream_t stream);
int mnb_bn_sign_fwd(const float* x, int32_t batch, int32_t channels, int32_t hw, const float* mean, const float* invstd,
                    const float* gamma, const float* beta, int32_t out_shuffle_groups, float* y, uint32_t* pass_bits,
                    mnb_stream_t stream);
/* training: 1 batch statistics, 0 running statistics, 2 = reduce pass only (dgamma / dbeta; the caller applies them with
 * mnb_bn_sign_bwd_pack, which writes dx as a packed operand) */
int mnb_bn_sign_bwd(const float* g, const uint32_t* pass_bits, const float* x, int32_t batch, int32_t channels, int32_t hw,
                    const float* mean, const float* invstd, const float* gamma, int32_t training,
                    int32_t out_shuffle_groups, float* dx, float* dgamma, float* dbeta, float* dx_channel_sum,
                    void* scratch, mnb_stream_t stream);

/* BatchNorm2d + binarizer + nn.MaxPool2d(2, 2) in one pass (the block before a 2x2 pool: nin_gc.py:84-85, :88-89): the
 * full-resolution +-1 tensor and the un-pooled gradient are never materialised.  y / g: [B, C, H/2, W/2] (through the
 * output permutation), pass_bits: B*C*H*W bits, argmax: B*C*(H/2)*(W/2) bytes (window index, ATen's first-maximum
 * rule).  Needs even H and W % 8 == 0, else MNB_E_UNSUPPORTED (run mnb_bn_sign_* and mnb_maxpool2d_* instead).   */
int mnb_bn_sign_pool_fwd(const float* x, int32_t batch, int32_t channels, int32_t H, int32_t W, const float* mean,
                         const float* invstd, const float* gamma, const float* beta, int32_t out_shuffle_groups, float* y,
                         uint32_t* pass_bits, uint8_t* argmax, mnb_stream_t stream);
int mnb_bn_sign_pool_bwd(const float* g, const uint32_t* pass_bits, const uint8_t* argmax, const float* x, int32_t batch,
                         int32_t channels, int32_t H, int32_t W, const float* mean, const float* invstd, const float* gamma,
                         int32_t training, int32_t out_shuffle_groups, float* dx, float* dgamma, float* dbeta,
                         float* dx_channel_sum, void* scratch, mnb_stream_t stream);

/* nn.MaxPool2d (square kernel <= 15, dilation 1, floor mode; nin_gc.py:85,89 / nin.py pools) with a one-byte
 * window index per output instead of int64 indices.  Same first-maximum tie rule and gradient accumulation
 * order as ATen, so results are bit-identical.  argmax: batch*channels*OH*OW bytes.                   */
int mnb_maxpool2d_fwd(const float* x, int32_t batch, int32_t channels, int32_t H, int32_t W, int32_t kernel, int32_t stride,
                      int32_t pad, int32_t out_shuffle_groups, float* y, uint8_t* argmax, mnb_stream_t stream);
int mnb_maxpool2d_bwd(const float* g, const uint8_t* argmax, int32_t batch, int32_t channels, int32_t H, int32_t W,
                      int32_t kernel, int32_t stride, int32_t pad, int32_t out_shuffle_groups, float* dx,
                      mnb_stream_t stream);

/* mnb_bn_sign_fwd that additionally writes its +-1 output as the bf16 operand plane of the packed-operand tensor-core
 * family (below): x_packed = bf16 [B][C/8][H][W][8] in the OUTPUT channel order (B*C*H*W*2 bytes, 16-byte aligned); needs
 * C % 8 == 0 and H*W % 32 == 0, else MNB_E_UNSUPPORTED.  y may be NULL (the consumer reads only the plane).           */
int mnb_bn_sign_fwd_packed(const float* x, int32_t batch, int32_t channels, int32_t hw, const float* mean,
                           const float* invstd, const float* gamma, const float* beta, int32_t out_shuffle_groups, float* y,
                           uint32_t* pass_bits, void* x_packed, mnb_stream_t stream);

/* fp32 convolution with few input channels on the tensor-core path: the un-quantized first layer of the QAT
 * models (plain nn.Conv2d in the reference: nin_gc.py:82, nin.py:60, resnet.py first conv; WB:300-317 leaves it
 * unquantized).  im2col operand built in shared memory, exact 3-piece bf16 split of both fp32 operands, the six
 * leading piece products accumulated in fp32 (error <= 2^-23 relative, i.e. that of an fp32 convolution).
 * Cover: groups 1, stride 1, dilation 1, 'same' odd square filter, C*R*S <= 128, Cout <= 256, 128 % W == 0,
 * (H*W) % 128 == 0; anything else returns MNB_E_UNSUPPORTED (-2).
 *   fwd   : y = conv2d(x, w) + bias (bias may be NULL)
 *   wgrad : dw = corr(x, dy);  scratch >= mnb_fconv2d_wgrad_tc_scratch_bytes(s) (-1: unsupported)
 *   mnb_fconv2d_plan: host only, the plan the forward (wgrad = 0) or weight gradient (wgrad != 0) will run; the first
 *                     min(n, 8) of  NP (padded Cout), KP (padded C*R*S), TH (rows per 128-position tile), n_tiles, grid
 *                     (CTAs), nbuf_a (forward operand buffers), smem_bytes, patch_floats (C * (TH + R - 1) * (W + R - 1))
 *                     are written.  Refusals as for the launching entry points.                                          */
int mnb_fconv2d_plan(const mnb_conv_shape* s, int32_t wgrad, int32_t* out, int32_t n);
int mnb_fconv2d_fwd_tc(const mnb_conv_shape* s, const float* x, const float* w, const float* bias, float* y,
                       int32_t* err_flag, mnb_stream_t stream);
/* mnb_fconv2d_fwd_wg: the same forward on two MMA warpgroups, 64-position tiles and one MMA over all output channels;
 * bit for bit mnb_fconv2d_fwd_tc's y.  Cover: that of mnb_fconv2d_fwd_tc with W <= 64, Cout > 128, where 3 im2col
 * buffers fit in shared memory (the 3 -> 192 / 256 5x5 stems at 32 x 32); anything else returns MNB_E_UNSUPPORTED before
 * any launch.
 *   mnb_fconv2d_wg_plan: host only, its plan in the fields of mnb_fconv2d_plan (TH: rows per 64-position tile, NP: the MMA
 *                        width 192 or 256, nbuf_a: im2col buffers).                                                          */
int mnb_fconv2d_wg_plan(const mnb_conv_shape* s, int32_t* out, int32_t n);
int mnb_fconv2d_fwd_wg(const mnb_conv_shape* s, const float* x, const float* w, const float* bias, float* y,
                       int32_t* err_flag, mnb_stream_t stream);
int64_t mnb_fconv2d_wgrad_tc_scratch_bytes(const mnb_conv_shape* s);
/* mnb_fconv2d_wgrad_wg: the same weight gradient on two MMA warpgroups with the running sums in registers; bit for bit
 * mnb_fconv2d_wgrad_tc's dw (same plan, partials and reduction).  Cover: that of mnb_fconv2d_wgrad_tc with 65 <= C*R*S <= 80
 * and Cout > 128 (the 3 -> 192 / 256 5x5 stems); scratch >= mnb_fconv2d_wgrad_wg_scratch_bytes(s) (-1: unsupported).                          */
int64_t mnb_fconv2d_wgrad_wg_scratch_bytes(const mnb_conv_shape* s);
int mnb_fconv2d_wgrad_wg(const mnb_conv_shape* s, const float* dy, const float* x, float* dw, void* scratch,
                         int32_t* err_flag, mnb_stream_t stream);
int mnb_fconv2d_wgrad_tc(const mnb_conv_shape* s, const float* dy, const float* x, float* dw, void* scratch,
                         int32_t* err_flag, mnb_stream_t stream);

/* ------------------------------------------------------------------------
 * Packed-operand ("pk") tensor-core family (mnb_pk.cu): every conv geometry of the QAT models on wgmma - weights
 * streamed per K-chunk, N / W tiling, stride 1 and 2 (space-to-depth), any filter with <= 64 taps.  Same math as
 * F.conv2d of the fake-quantized tensors (WB:186, DF:113, IAO:498/843/947) and ATen convolution_backward.
 *
 * Operands are bf16 "term planes"  pk[t][b][ceil(C/8)][h][w][8] : t = 0..T-1 exact pieces of an fp32 value
 * (x = p0 + p1 + p2, 8 significand bits each) or ONE plane of exact integer levels.
 *   mnb_pk_pack_act   : fp32 NCHW -> term planes.  qp != NULL: fake-quantize (DF:36-46 / IAO:214-240 / WB:11-36), planes
 *                       hold the integer level e (value = e * scale), bits8[b][c/8][h][w] bit j = STE pass flag of channel
 *                       8*(c/8)+j.  qp == NULL: exact split of x (* ch_scale[c] when given).  phase_split: the four
 *                       (h%2, w%2) planes become channel octets (h%2*2 + w%2)*ceil(C/8) + c/8 of an [H/2, W/2] tensor
 *                       (the form a stride-2 consumer reads).  out_pk: mnb_pk_act_bytes() bytes, 16-byte aligned.
 *   mnb_pk_pack_weight: w_int (i16 levels) or w_f32 [K, C/g, R, S] -> the bf16 operand image of (shape, mode);
 *                       mode 0 forward, 1 data gradient.  kzero[k] == 0 zeroes channel k (dgrad of a zero-scale channel).
 *                       w_img: mnb_pk_wimage_bytes() bytes.  terms_a / terms_w must match the later mnb_pk_conv call.
 *   mnb_pk_conv       : mode 0: y = bias + (a_scale * n_scale[n]) * conv2d(A, W);  mode 1: dx = STE(conv_transpose(A = dy, W)),
 *                       bits8 / gain: STE mask of the quantizer that fed the forward conv and its gradient factor (0.1 DoReFa).
 *                       a_scale: device scalar or NULL (then a_scale_const); n_scale NULL = 1.
 *   mnb_pk_wgrad      : dw[k][c][r][s] = (a_scale / kdiv[k]) * corr(x, dy); kdiv = the ch_scale dy_pk was packed with.
 * All return MNB_E_UNSUPPORTED (nothing launched) outside the cover (dilation, > 64 taps, odd sizes with stride 2, ...).
 * ---------------------------------------------------------------------- */
int64_t mnb_pk_act_bytes(int32_t batch, int32_t channels, int32_t h, int32_t w, int32_t terms);
int mnb_pk_pack_act(const float* x, int32_t batch, int32_t channels, int32_t h, int32_t w, const mnb_act_qparams* qp,
                    int32_t terms, const float* ch_scale, int32_t phase_split, void* out_pk, uint8_t* bits8,
                    mnb_stream_t stream);
/* BatchNorm2d + ReLU + DoReFa activation quantizer (DF:36-46) of the NEXT conv + operand packing in one pass (the DoReFa
 * block conv -> nn.BatchNorm2d -> nn.ReLU -> [channel_shuffle] -> QuantConv2d, nin_gc.py:53-59): x_packed = that conv's packed
 * bf16 level plane [B][C/8][H][W][8] in the output channel order of the folded shuffle; pass_bits = relu'(bn) * [0.1 bn <= 1]
 * as flat NCHW bits in the producer's own channel order (what mnb_bn_sign_bwd consumes for the backward pass).
 * Needs C % 8 == 0 and H*W % 32 == 0, else MNB_E_UNSUPPORTED. */
int mnb_bn_relu_quant_pack_fwd(const float* x, int32_t batch, int32_t channels, int32_t hw, const float* mean,
                               const float* invstd, const float* gamma, const float* beta, const mnb_act_qparams* qp,
                               int32_t out_shuffle_groups, void* x_packed, uint32_t* pass_bits, mnb_stream_t stream);
/* Second pass of mnb_bn_sign_bwd for a producing conv that runs on the packed-operand family (nn.BatchNorm2d backward +
 * saturate STE of WB:11-36, after dgamma / dbeta were reduced): writes  dx * ch_scale[c]  (ch_scale NULL: dx) as `terms`
 * exact bf16 pieces in the plane layout of mnb_pk_pack_act - the dy operand of that conv's mnb_pk_conv (mode 1) and
 * mnb_pk_wgrad (kdiv = ch_scale) - and, when dx != NULL, plain fp32 dx.  Training-mode statistics only.  channels % 8 == 0. */
int mnb_bn_sign_bwd_pack(const float* g, const uint32_t* pass_bits, const float* x, int32_t batch, int32_t channels, int32_t hw,
                         const float* mean, const float* invstd, const float* gamma, const float* dgamma, const float* dbeta,
                         int32_t out_shuffle_groups, const float* ch_scale, int32_t terms, float* dx, void* dy_packed,
                         mnb_stream_t stream);
/* The same for a producer with the 2x2 max-pool folded in: second pass of mnb_bn_sign_pool_bwd (call that one with
 * training = 2 first: reduce pass only, dgamma / dbeta) writing the full-resolution gradient [batch, channels, H, W] as the
 * producing conv's packed operand.  argmax / pass_bits as written by mnb_bn_sign_pool_fwd; g is the pooled gradient
 * [batch, channels, H/2, W/2] in the shuffled order.  Needs even H, W % 8 == 0, channels % 8 == 0.                  */
int mnb_bn_sign_pool_bwd_pack(const float* g, const uint32_t* pass_bits, const uint8_t* argmax, const float* x, int32_t batch,
                              int32_t channels, int32_t H, int32_t W, const float* mean, const float* invstd,
                              const float* gamma, const float* dgamma, const float* dbeta, int32_t out_shuffle_groups,
                              const float* ch_scale, int32_t terms, void* dy_packed, mnb_stream_t stream);
/* Int16 hand-off between a wbwtab conv and its BatchNorm + binarizer (the conv's only reader).  On a +-1 activation plane
 * and integer weight levels the conv's sums are exact integers; mnb_pk_conv_codes stores them as int16 `codes`
 * [B][K][OH][OW] instead of the fp32 output, plus dec[2][K] = (a_scale * n_scale[k], bias[k]), the epilogue's pair, so that
 * x = fmaf(code, dec[k], dec[K + k]) is mnb_pk_conv's fp32 output bit for bit.  Refused with MNB_E_UNSUPPORTED (nothing
 * launched) unless (C/g) * R * S * level_bound <= 32767 (level_bound = max |weight level|), terms_a = terms_w = 1 and the
 * plan is not segmented.  The _codes producers below are their fp32 namesakes reading x through that decode, with the
 * same element-to-thread mapping and summation order (identical results); codes need half the alignment x needs there. */
int mnb_pk_conv_codes(const mnb_conv_shape* s, const void* a_pk, int32_t terms_a, const void* w_img, int32_t terms_w,
                      const float* n_scale, const float* a_scale, float a_scale_const, const float* bias, int32_t level_bound,
                      int16_t* codes, float* dec, int32_t* err_flag, mnb_stream_t stream);
/* x = fmaf(codes, dec[c], dec[C + c]) as fp32 [batch, channels, hw] */
int mnb_codes_decode(const int16_t* codes, const float* dec, int32_t batch, int32_t channels, int32_t hw, float* x,
                     mnb_stream_t stream);
int mnb_bn_batch_stats_codes(const int16_t* codes, const float* dec, int32_t batch, int32_t channels, int32_t hw, double eps,
                             double momentum, float* running_mean, float* running_var, int64_t* num_batches_tracked,
                             float* mean_invstd, void* scratch, mnb_stream_t stream);
int mnb_bn_sign_fwd_packed_codes(const int16_t* codes, const float* dec, int32_t batch, int32_t channels, int32_t hw,
                                 const float* mean, const float* invstd, const float* gamma, const float* beta,
                                 int32_t out_shuffle_groups, float* y, uint32_t* pass_bits, void* x_packed, mnb_stream_t stream);
int mnb_bn_sign_bwd_codes(const float* g, const uint32_t* pass_bits, const int16_t* codes, const float* dec, int32_t batch,
                          int32_t channels, int32_t hw, const float* mean, const float* invstd, const float* gamma,
                          int32_t training, int32_t out_shuffle_groups, float* dx, float* dgamma, float* dbeta,
                          float* dx_channel_sum, void* scratch, mnb_stream_t stream);
int mnb_bn_sign_pool_fwd_codes(const int16_t* codes, const float* dec, int32_t batch, int32_t channels, int32_t H, int32_t W,
                               const float* mean, const float* invstd, const float* gamma, const float* beta,
                               int32_t out_shuffle_groups, float* y, uint32_t* pass_bits, uint8_t* argmax, mnb_stream_t stream);
int mnb_bn_sign_pool_bwd_codes(const float* g, const uint32_t* pass_bits, const uint8_t* argmax, const int16_t* codes,
                               const float* dec, int32_t batch, int32_t channels, int32_t H, int32_t W, const float* mean,
                               const float* invstd, const float* gamma, int32_t training, int32_t out_shuffle_groups, float* dx,
                               float* dgamma, float* dbeta, float* dx_channel_sum, void* scratch, mnb_stream_t stream);
int mnb_bn_sign_bwd_pack_codes(const float* g, const uint32_t* pass_bits, const int16_t* codes, const float* dec, int32_t batch,
                               int32_t channels, int32_t hw, const float* mean, const float* invstd, const float* gamma,
                               const float* dgamma, const float* dbeta, int32_t out_shuffle_groups, const float* ch_scale,
                               int32_t terms, float* dx, void* dy_packed, mnb_stream_t stream);
int mnb_bn_sign_pool_bwd_pack_codes(const float* g, const uint32_t* pass_bits, const uint8_t* argmax, const int16_t* codes,
                                    const float* dec, int32_t batch, int32_t channels, int32_t H, int32_t W, const float* mean,
                                    const float* invstd, const float* gamma, const float* dgamma, const float* dbeta,
                                    int32_t out_shuffle_groups, const float* ch_scale, int32_t terms, void* dy_packed,
                                    mnb_stream_t stream);
/* mnb_pk_pack_act with a preceding nn.ReLU folded in (relu != 0: x is clamped at 0 before it is quantized / split) */
int mnb_pk_pack_act_relu(const float* x, int32_t batch, int32_t channels, int32_t h, int32_t w, const mnb_act_qparams* qp,
                         int32_t terms, const float* ch_scale, int32_t phase_split, int32_t relu, void* out_pk,
                         uint8_t* bits8, mnb_stream_t stream);
/* Group-padded planes of a grouped conv (DESIGN.md 4.17): mnb_pk_pack_act_relu for the operand of a conv with `groups` groups.
 * Group g's channel j sits at plane channel g * round_up(channels / groups, 8) + j; the padding channels are zero in every
 * plane and in bits8 [b][groups * ceil(channels / groups / 8)][h][w].  With channels / groups % 8 == 0 (or groups == 1) this
 * is the plane of mnb_pk_pack_act.  mnb_pk_conv, mnb_pk_wgrad and mnb_pk_pack_weight read grouped operands in this layout
 * (mode 0: the input's channels per group, mode 1 and the weight gradient's dy: the output's).  out_pk:
 * mnb_pk_grouped_act_bytes() bytes (-1: groups do not divide channels). */
int64_t mnb_pk_grouped_act_bytes(int32_t batch, int32_t channels, int32_t h, int32_t w, int32_t terms, int32_t groups);
int mnb_pk_pack_act_grouped(const float* x, int32_t batch, int32_t channels, int32_t h, int32_t w, const mnb_act_qparams* qp,
                            int32_t terms, const float* ch_scale, int32_t phase_split, int32_t relu, void* out_pk,
                            uint8_t* bits8, int32_t groups, mnb_stream_t stream);
int mnb_pk_conv_plan(const mnb_conv_shape* s, int32_t mode, int32_t terms_a, int32_t terms_w, int32_t* out16); /* host only */
/* host only, the plan mnb_pk_conv / mnb_pk_wgrad will run (same MNB_PK_* environment knobs); the first min(n, 31) resp.
 * min(n, 16) fields are written.  Each query (and mnb_pk_conv_plan, mnb_pk_wimage_bytes, mnb_pk_wgrad_scratch_bytes)
 * refuses exactly what its launch refuses on the host, with the same code and error text:
 *   mnb_pk_conv_plan_ex: the 16 fields of mnb_pk_conv_plan, then segmented, seg_len (stages per segment, 0 when not
 *                        segmented), npairs (piece products per K-step), col_tiles, n_mgroups, stage templates (tap groups)
 *                        of output phases 0..3, filter taps of output phases 0..3, MMA program words, stages of the last
 *                        accumulation segment of a phase-0 item (0 when not segmented)
 *   mnb_pk_wgrad_plan  : Nc, n_ctiles, tpg (taps per CTA), n_tg (tap groups), gm (merged groups), splits (batch splits),
 *                        NI (sub-blocks per stage), nstage, BW, TH, n_ktiles, nkph_used (k-phase planes read),
 *                        stg_per_split, nsub (row-tile sub-blocks), issue-program entries, nstg_total */
int mnb_pk_conv_plan_ex(const mnb_conv_shape* s, int32_t mode, int32_t terms_a, int32_t terms_w, int32_t* out, int32_t n);
int mnb_pk_wgrad_plan(const mnb_conv_shape* s, int32_t terms_dy, int32_t terms_x, int32_t* out, int32_t n);
int64_t mnb_pk_wimage_bytes(const mnb_conv_shape* s, int32_t mode, int32_t terms_a, int32_t terms_w);
int mnb_pk_pack_weight(const mnb_conv_shape* s, int32_t mode, int32_t terms_a, int32_t terms_w, const int16_t* w_int,
                       const float* w_f32, const float* kzero, void* w_img, mnb_stream_t stream);
int mnb_pk_conv(const mnb_conv_shape* s, int32_t mode, const void* a_pk, int32_t terms_a, const void* w_img, int32_t terms_w,
                const float* n_scale, const float* a_scale, float a_scale_const, const float* bias, const uint8_t* bits8,
                float gain, float* out, int32_t* err_flag, mnb_stream_t stream);
/* Inference graphs with frozen quantizers (BASELINE.json configs[4], iao/main.py:511-519: eval forward of a calibrated model):
 * the producer writes the operand plane of its consumer, so the fp32 activation between two quantized convs is neither
 * written nor re-read nor packed in a separate pass.
 *   mnb_pk_conv_post        : forward conv (mode 0 of mnb_pk_conv) whose epilogue also computes
 *                             level = Q_consumer([ReLU](y)) (IAO:214-240 / DF:36-46 of the NEXT layer's activation quantizer)
 *                             and stores it as that layer's bf16 plane; out may be NULL (plane only).
 *   mnb_quant_add_pack_fwd  : IAO QuantAdd (IAO:1441-1498: out = Q(a) + Q(b) [-> ReLU]) that additionally quantizes its
 *                             result for the consuming conv and writes that conv's plane (a, b, out: fp32 [B, C, H, W]).
 * phase_split: the consumer is a stride-2 conv (space-to-depth plane order of mnb_pk_pack_act). */
typedef struct mnb_pk_post {
  const mnb_act_qparams* q; /* the consumer's activation quantizer, 2..8 bits, DoReFa or IAO */
  int32_t relu;             /* an nn.ReLU sits between producer and consumer */
  int32_t phase_split;
  void* out_pk;             /* mnb_pk_act_bytes(B, C_out, OH, OW, 1) bytes, 16-byte aligned */
  /* Trailing fields, zero = absent (mnb_pk_conv_post and mnb_pk_i8_conv only; the QuantAdd producers ignore them):
   * eval BatchNorm2d between the conv and the [ReLU +] quantizer, y' = fmaf(y - mean, gamma * invstd, beta) - the op
   * sequence of mnb_bn_relu_quant_pack_fwd, so a DoReFa block conv -> nn.BatchNorm2d -> nn.ReLU -> QuantConv2d
   * (nin.py / nin_gc.py conv-bn-relu blocks, DF:36-46) writes the levels that producer writes from the fp32 output, bit for
   * bit.  All four NULL or all four [C_out]; a partial set is MNB_E_ARG.
   * shuffle_groups > 1: the consumer block's channel_shuffle (nin_gc.py:14-22) - producer channel c is stored as consumer
   * channel (c % cpg) * sg + c / cpg, cpg = C_out / sg.  MNB_E_UNSUPPORTED unless sg divides C_out, C_out fills whole
   * 16-byte units (8 bf16 / 16 int8 channels) and phase_split is 0. */
  const float* bn_mean;
  const float* bn_invstd;
  const float* bn_gamma;
  const float* bn_beta;
  int32_t shuffle_groups;
  /* terms_out > 0 with q == NULL (mnb_pk_conv_post only): no consumer quantizer - the consumer reads the fp32 value
   * [ReLU](BatchNorm(y)) itself as terms_out (1..3) exact bf16 pieces, the term planes mnb_pk_pack_act writes from that
   * tensor (qp == NULL), out_pk then holding terms_out planes of mnb_pk_act_bytes(B, C_out, OH, OW, 1) bytes each.  The
   * frozen wbwtab graphs of fp32-activation models (prepare(A=32, W=2|3)): a binary / ternary conv -> nn.BatchNorm2d ->
   * ReLU (WB:79-94, A=32) -> [channel_shuffle] -> the next QuantConv2d, which feeds its fp32 input to F.conv2d (WB:181-195).
   * Same cover and refusals as the quantized consumer plane, and output channels per group % 8 != 0 (grouped or not) is
   * MNB_E_UNSUPPORTED; q == NULL with terms_out == 0 (or q with terms_out != 0) and terms_out > 3 are MNB_E_ARG. */
  int32_t terms_out;
} mnb_pk_post;
int mnb_pk_conv_post(const mnb_conv_shape* s, const void* a_pk, int32_t terms_a, const void* w_img, int32_t terms_w,
                     const float* n_scale, const float* a_scale, float a_scale_const, const float* bias, float* out,
                     const mnb_pk_post* post, int32_t* err_flag, mnb_stream_t stream);
int mnb_quant_add_pack_fwd(const float* a, const float* b, int32_t batch, int32_t channels, int32_t h, int32_t w,
                           const mnb_act_qparams* qp, int32_t relu, float* out, const mnb_pk_post* post, mnb_stream_t stream);
/* Host only: the route of a forward conv of the family with consumer `post` (NULL: none) - the checks mnb_pk_conv_post
 * (cpu 8) or mnb_pk_i8_conv (cpu 16, terms 1 x 1) make before launching, with the same return code and mnb_last_error
 * text on a refusal.  The pointers of post are compared and checked for alignment, never dereferenced (post->q is read).
 * out = {epilogue path, Nt, MT, n_mtiles, n_items, ny, col_tiles, n_ntiles, CTAs per output phase, segmented}, the first
 * min(n, 10) written; path 0 plain bf16 levels (or no consumer), 1 segmented (no consumer), 2 int8 (levels or none),
 * 3 bf16 levels behind BatchNorm / shuffle, 4 the same into an int8 plane, 5 term planes. */
int mnb_pk_conv_post_plan(const mnb_conv_shape* s, int32_t terms_a, int32_t terms_w, int32_t cpu, const mnb_pk_post* post,
                          int32_t* out, int32_t n);
/* int8 operands for frozen inference graphs (symmetric IAO, IAO:214-240 with q_type 0): the forward conv of the family on
 * s8 x s8 -> s32 wgmma (K32 MMAs, exact integer sums).  The result is  y = fmaf(float(sum), a_scale * n_scale[n], bias[n]),
 * bit-identical to mnb_pk_conv on the same levels whenever its fp32 partial sums stay below 2^24, and exact (one rounding of
 * the integer sum) above.  Cover: everything mnb_pk_conv covers in mode 0 with one piece per operand, grouped convs with
 * C/g % 16 == 0, kg * R * S * 128 * 127 < 2^31; the quantizers must be symmetric IAO with 2..8 bits (levels in [-128, 127]),
 * weight levels in [-127, 127].  Outside the cover every entry point returns MNB_E_UNSUPPORTED (or MNB_E_ARG for bad
 * pointers) before launching anything.
 *   int8 plane: pk8[b][ceil(C/16)][h][w][16] s8 levels (the byte geometry of the bf16 plane with 16 channels per 16 bytes);
 *               phase_split: unit (h%2*2 + w%2)*ceil(C/16) + c/16 of an [H/2, W/2] tensor, as in mnb_pk_pack_act.
 *   mnb_pk_i8_act_bytes        : bytes of one int8 plane.
 *   mnb_pk_i8_pack_act         : fp32 NCHW [-> ReLU when relu != 0] -> int8 level plane (no STE bits: inference only).
 *   mnb_pk_i8_conv_plan        : host only, the plan mnb_pk_i8_conv runs; same fields as mnb_pk_conv_plan_ex (CC counts
 *                                channels: 32 per K-step).
 *   mnb_pk_i8_wimage_bytes     : bytes of the int8 weight image (-1 outside the cover).
 *   mnb_pk_i8_pack_weight      : i16 levels [K, C/g, R, S] -> int8 image [n-tile][group][stage][tap][c/16][n][16].
 *   mnb_pk_i8_conv             : forward conv of an int8 plane; out may be NULL when post is given.  post: the consumer's
 *                                plane is written as int8 (its quantizer symmetric IAO; producer and consumer channel
 *                                offsets multiples of 16, i.e. grouped producers need K/g % 16 == 0).
 *   mnb_quant_add_pack_i8_fwd  : mnb_quant_add_pack_fwd writing the consumer's int8 plane. */
int64_t mnb_pk_i8_act_bytes(int32_t batch, int32_t channels, int32_t h, int32_t w);
int mnb_pk_i8_pack_act(const float* x, int32_t batch, int32_t channels, int32_t h, int32_t w, const mnb_act_qparams* qp,
                       int32_t phase_split, int32_t relu, void* out_pk, mnb_stream_t stream);
int mnb_pk_i8_conv_plan(const mnb_conv_shape* s, int32_t* out, int32_t n);
int64_t mnb_pk_i8_wimage_bytes(const mnb_conv_shape* s);
int mnb_pk_i8_pack_weight(const mnb_conv_shape* s, const int16_t* w_int, void* w_img, mnb_stream_t stream);
int mnb_pk_i8_conv(const mnb_conv_shape* s, const void* a_pk, const void* w_img, const float* n_scale, const float* a_scale,
                   float a_scale_const, const float* bias, float* out, const mnb_pk_post* post, int32_t* err_flag,
                   mnb_stream_t stream);
int mnb_quant_add_pack_i8_fwd(const float* a, const float* b, int32_t batch, int32_t channels, int32_t h, int32_t w,
                              const mnb_act_qparams* qp, int32_t relu, float* out, const mnb_pk_post* post, mnb_stream_t stream);
/* Frozen DoReFa inference graphs (the reference's quant_inference flow, wqaq/dorefa/quant_model_test/quant_model_test.py:185-194).
 * int8 planes also hold DoReFa levels 0 .. 2^a - 1 for a = 2..7 (DF:36-46); weight levels +-(2^w - 1) fit s8 for w <= 7.
 * 8-bit DoReFa activations stay on the bf16 planes: every int8 entry point refuses them with MNB_E_UNSUPPORTED.
 *   mnb_bn_relu_quant_pack_i8_fwd : mnb_bn_relu_quant_pack_fwd (same BatchNorm, ReLU and shuffle sequence) writing the int8
 *                                   plane of a DoReFa quantizer with 2..7 bits; no STE bits (inference only).  Needs
 *                                   C % 16 == 0 and H*W % 32 == 0, else MNB_E_UNSUPPORTED.
 *   mnb_pk_plane_maxpool          : max_pool2d(k, stride s, padding p) of a level plane (int8 != 0: int8 [b][c/16][h][w][16],
 *                                   else bf16 [b][c/8][h][w][8]) into the same layout at the pooled size, padding skipped.
 *                                   Exact for every plane a quantizer writes: DoReFa's floor(clamp(0.1 x, 0, 1) / s + 0.5)
 *                                   and ReLU are monotone non-decreasing, so Q(maxpool(relu(y))) == maxpool(Q(relu(y))).
 *                                   Square windows with 2 * p <= k (nin.py:51/56, nin_gc.py:126/131); the output feeds a
 *                                   stride-1 consumer (no phase split). */
int mnb_bn_relu_quant_pack_i8_fwd(const float* x, int32_t batch, int32_t channels, int32_t hw, const float* mean,
                                  const float* invstd, const float* gamma, const float* beta, const mnb_act_qparams* qp,
                                  int32_t out_shuffle_groups, void* x_packed, mnb_stream_t stream);
int mnb_pk_plane_maxpool(const void* in_pk, int32_t batch, int32_t channels, int32_t h, int32_t w, int32_t k, int32_t s, int32_t p,
                         int32_t int8, void* out_pk, mnb_stream_t stream);
/* Frozen IAO inference graphs of NIN / NIN-GC (nin.py:51/55, nin_gc.py:88/119): the pool between two conv-bn-relu blocks is a
 * QuantMaxPool2d (IAO:1285-1343) with a quantizer of its own, so the producer's epilogue writes the POOL quantizer's levels
 * L and the next conv quantizes the pooled values again.  Both maps are exact functions of L: the pool writes
 * v = fl((L + zp_p) * s_p) (ActQuantFn), and the consumer's level of v is monotone non-decreasing in L (s_p > 0), so
 * Q_c(maxpool(Q_p(relu(y)))) == T[maxpool(L)] with a 256-entry table T.
 *   mnb_pk_plane_maxpool_requant : mnb_pk_plane_maxpool of a plane of the pool quantizer's levels (same layouts, same cover,
 *                                  int8 in -> int8 out, bf16 in -> bf16 out), each window max written through T as the
 *                                  consumer's plane.  Every CTA builds T in shared memory from the device scalars with the
 *                                  fp32 op sequence of the engine's IAO quantizer (__fdiv_rn, round half away, clamp), so
 *                                  the result is the consumer's pack_act of max_pool2d(ActQuantFn(x)) bit for bit.  Both
 *                                  quantizers must be IAO with q_type 0 and 2..8 bits (zero_point 0, levels in
 *                                  [-128, 127]); anything else returns MNB_E_UNSUPPORTED before launching. */
int mnb_pk_plane_maxpool_requant(const void* in_pk, int32_t batch, int32_t channels, int32_t h, int32_t w, int32_t k, int32_t s,
                                 int32_t p, int32_t int8, const mnb_act_qparams* q_in, const mnb_act_qparams* q_out, void* out_pk,
                                 mnb_stream_t stream);
/* Frozen wbwtab inference graphs with fp32 activations (prepare(A=32, W=2|3), WB:79-94: the "activation quantizer" is a ReLU):
 * activations cross between layers as term planes (terms exact bf16 pieces, the mnb_pk_pack_act layout with qp == NULL).
 *   mnb_pk_plane_maxpool_terms : max_pool2d(k, s, p) of the fp32 tensor a term plane holds (nin.py:51/56 3x3/2/1, nin_gc.py
 *                                2x2/2/0, replacing ATen's max-pool of the ReLU output and the next conv's pack): values
 *                                rebuilt exactly, window max with ATen's rule (first of equal values, NaN propagates),
 *                                written as `terms` pieces of the pooled size.  Bitwise mnb_pk_pack_act of ATen max_pool2d of
 *                                the decoded tensor.  Same cover as mnb_pk_plane_maxpool (square windows, 2 * p <= k, stride-1
 *                                consumer); MNB_E_UNSUPPORTED outside it.
 *   mnb_bn_relu_pack_terms_fwd : eval BatchNorm y' = fmaf(y - mean, gamma * invstd, beta) (all four NULL: none) [-> ReLU]
 *                                [-> the consumer block's channel shuffle] of an fp32 NCHW tensor written as the consumer's
 *                                `terms` term planes: the stem producer (fp32 stem conv -> nn.BatchNorm2d -> ReLU ->
 *                                first QuantConv2d), the op sequence of mnb_pk_conv_post with terms_out.  channels % 8 == 0,
 *                                shuffle groups dividing channels, else MNB_E_UNSUPPORTED; a partial BatchNorm set is MNB_E_ARG. */
int mnb_pk_plane_maxpool_terms(const void* in_pk, int32_t batch, int32_t channels, int32_t h, int32_t w, int32_t k, int32_t s,
                               int32_t p, int32_t terms, void* out_pk, mnb_stream_t stream);
int mnb_bn_relu_pack_terms_fwd(const float* x, int32_t batch, int32_t channels, int32_t hw, const float* mean,
                               const float* invstd, const float* gamma, const float* beta, int32_t relu,
                               int32_t out_shuffle_groups, int32_t terms, void* x_packed, mnb_stream_t stream);
int64_t mnb_pk_wgrad_scratch_bytes(const mnb_conv_shape* s, int32_t terms_dy, int32_t terms_x);
int mnb_pk_wgrad(const mnb_conv_shape* s, const void* dy_pk, int32_t terms_dy, const void* x_pk, int32_t terms_x,
                 const float* a_scale, const float* kdiv, float* dw, void* scratch, int32_t* err_flag, mnb_stream_t stream);
/* mnb_pk_wgrad for narrow grouped 3x3 layers (stride 1, 16 input / 32 output channels per group, groups % 4 == 0): one CTA
 * keeps all nine taps of four groups in registers, so every operand byte is loaded once.  Same arguments as mnb_pk_wgrad
 * and the same result bit for bit (same accumulation chains, batch splits and reduction order); MNB_E_UNSUPPORTED (nothing
 * launched) outside that cover.
 * mnb_pk_wgrad_taps_plan (host only): out = {blocks, splits, NI, nstage, BW, TH, stages per split, smem bytes,
 * accumulators per MMA thread, scratch bytes (lo 31 bits), scratch bytes (hi), npairs}; the first min(n, 12) are written. */
int mnb_pk_wgrad_taps_plan(const mnb_conv_shape* s, int32_t terms_dy, int32_t terms_x, int32_t* out, int32_t n);
int mnb_pk_wgrad_taps(const mnb_conv_shape* s, const void* dy_pk, int32_t terms_dy, const void* x_pk, int32_t terms_x,
                      const float* a_scale, const float* kdiv, float* dw, void* scratch, int32_t* err_flag, mnb_stream_t stream);
/* Data gradient (mnb_pk_conv mode 1) and weight gradient (mnb_pk_wgrad) of a 1x1 convolution in one pass over dy: stride
 * 1, no padding, <= 128 input and output channels per group, not group-padded, on the weight gradient's own raster, stages
 * and batch splits.  w_img: the data-gradient weight image of mnb_pk_pack_weight (mode 1, terms_dy, terms_w).  dx is
 * mnb_pk_conv's result without n_scale, a_scale or bias (dx = acc * a_scale_const; with the STE mask bits8,
 * dx = pass ? acc * gain : 0) and dw mnb_pk_wgrad's (a_scale, kdiv), both bit for bit.  MNB_E_UNSUPPORTED (nothing launched)
 * outside that cover.
 * mnb_pk_bwd1x1_plan (host only): out = {groups, splits, NI, nstage, BW, TH, stages per split, smem bytes, sub-blocks,
 * stages, data-gradient MMAs per chain, scratch bytes (lo 31 bits), scratch bytes (hi), npairs, N tile}; the first
 * min(n, 15) are written. */
int mnb_pk_bwd1x1_plan(const mnb_conv_shape* s, int32_t terms_dy, int32_t terms_x, int32_t terms_w, int32_t* out, int32_t n);
int mnb_pk_bwd1x1(const mnb_conv_shape* s, const void* dy_pk, int32_t terms_dy, const void* x_pk, int32_t terms_x,
                  const void* w_img, int32_t terms_w, float a_scale_const, const uint8_t* bits8, float gain, float* dx,
                  const float* a_scale, const float* kdiv, float* dw, void* scratch, int32_t* err_flag, mnb_stream_t stream);
/* Forward and data gradient of the same narrow grouped 3x3 layers (stride 1, padding 0..2, 16 input / 32 output channels per
 * group, groups % 4 == 0) with whole images as M tiles and a CTA per block of groups whose weights stay in shared memory.
 * Forward: one activation piece and one weight piece (mnb_pk_gc3_conv mode 0 = mnb_pk_conv mode 0, mnb_pk_gc3_conv_codes =
 * mnb_pk_conv_codes); data gradient: two dy pieces and one weight piece on an un-segmented plan (mnb_pk_gc3_conv mode 1 =
 * mnb_pk_conv mode 1).  Same arguments, same weight image (mnb_pk_pack_weight) and the same result bit for bit: every
 * element sees the MMA chain of mnb_pk_conv's plan.  MNB_E_UNSUPPORTED (nothing launched) outside that cover.
 * mnb_pk_gc3_plan (host only): out[0..9] = {groups per CTA block, images per M tile, m64 blocks per M tile, stages, smem
 * bytes, CTAs, image tiles, MMAs per chain, N tile, MMA warpgroups (stages are a multiple of it)}, then per MMA of the chain in issue order (tap r * 3 + s,
 * streamed-operand piece, weight piece, 16-channel K-step); the first n are written. */
int mnb_pk_gc3_plan(const mnb_conv_shape* s, int32_t mode, int32_t terms_a, int32_t terms_w, int32_t* out, int32_t n);
int mnb_pk_gc3_conv(const mnb_conv_shape* s, int32_t mode, const void* a_pk, int32_t terms_a, const void* w_img, int32_t terms_w,
                    const float* n_scale, const float* a_scale, float a_scale_const, const float* bias, const uint8_t* bits8,
                    float gain, float* out, int32_t* err_flag, mnb_stream_t stream);
int mnb_pk_gc3_conv_codes(const mnb_conv_shape* s, const void* a_pk, int32_t terms_a, const void* w_img, int32_t terms_w,
                          const float* n_scale, const float* a_scale, float a_scale_const, const float* bias, int32_t level_bound,
                          int16_t* codes, float* dec, int32_t* err_flag, mnb_stream_t stream);

/* ------------------------------------------------------------------------
 * Bit-packed XNOR-popcount forward for wbwtab layers (mnb_xnor.cu): binary activations (WB:11-36, sign with 0 -> +1)
 * times binary / ternary weights (WB:40-75, 98-146) as sum = popc(N) - 2 popc(N & (A ^ S)) on 1-bit planes; the integer
 * sum is exact, y = fmaf(sum, alpha[k], bias[k]) equals mnb_pk_conv's result bit for bit.  Forward only (the gradients
 * of a QAT step multiply real-valued dy).  functional.py picks it per layer (functional.xnor_preferred).
 *   a_bits : u32 [B][G][ceil(C/g / 32)][H][W], bit j of word n = [x[b][g*C/g + 32 n + j][h][w] is not < 0]
 *   w_img  : mnb_xnor_wimage_bytes() bytes, built from the i16 levels {-1, 0, +1} [K][C/g][R][S] of mnb_wb_weight_fwd
 * Cover: square filter 1/3/5, equal strides / pads, dilation 1, C/g <= 128 (3x3), <= 64 (5x5), <= 256 (1x1); else
 * MNB_E_UNSUPPORTED (mnb_xnor_supported: 1 / 0).                                                                      */
int mnb_xnor_supported(const mnb_conv_shape* s);
int64_t mnb_xnor_act_bytes(int32_t batch, int32_t channels, int32_t h, int32_t w, int32_t groups);
int mnb_xnor_pack_act(const float* x, int32_t batch, int32_t channels, int32_t h, int32_t w, int32_t groups, void* out_bits,
                      mnb_stream_t stream);
int64_t mnb_xnor_wimage_bytes(const mnb_conv_shape* s);
int mnb_xnor_pack_weight(const mnb_conv_shape* s, const int16_t* w_int, void* w_img, mnb_stream_t stream);
int mnb_xnor_conv_fwd(const mnb_conv_shape* s, const void* a_bits, const void* w_img, const float* alpha, const float* bias,
                      float* y, mnb_stream_t stream);
/* Frozen wbwtab inference graphs (wbwtab.freeze_inference): the producer writes its consumer's operand, so no fp32 tensor
 * crosses between two binarized layers.  The value v = fmaf(sum, alpha[k], bias[k]) of mnb_xnor_conv_fwd goes through
 *   [eval BatchNorm: v = fmaf(v - mean[k], gamma[k] * invstd[k], beta[k]), the op sequence of mnb_bn_sign_fwd_packed]
 *   -> sign bit !(v < 0) (WB:11-36: 0 and -0.0 -> +1) [-> MaxPool2d(2, 2): OR of the window's bits] [-> channel shuffle:
 *   channel c to (c mod C/sg) * sg + c div (C/sg), the producers' out_shuffle_groups]
 * and is stored in the consumer's format:
 *   MNB_XNOR_BITS       the bit plane of mnb_xnor_pack_act for a consumer with out_groups groups (zeroed and OR-ed into on
 *                       the stream: bitwise deterministic);
 *   MNB_XNOR_PM1_BF16   the +-1 bf16 plane [b][c/8][h][w][8] of mnb_bn_sign_fwd_packed (no pool; C % 8 == 0, 16-byte aligned).
 *   mnb_xnor_post_bytes    : bytes of conv_post's output (-1 outside the cover: conv shape, odd plane under a pool, ...).
 *   mnb_xnor_conv_post     : the convolution with that epilogue.
 *   mnb_xnor_pack_act_post : fp32 NCHW [B, C, H, W] (the un-quantized stem's output) -> the same epilogue -> bit plane.
 * Refusals (nothing launched): MNB_E_ARG for a malformed description (format, shuffle / consumer groups that do not divide C,
 * partial BatchNorm pointers), MNB_E_UNSUPPORTED outside the cover (conv shape, a pool over an odd plane, bf16 with a pool). */
#define MNB_XNOR_BITS 0
#define MNB_XNOR_PM1_BF16 1
typedef struct mnb_xnor_post {
  int32_t format;          /* MNB_XNOR_BITS or MNB_XNOR_PM1_BF16 (mnb_b1_*: also MNB_XNOR_B1_PLANE) */
  int32_t out_groups;      /* bits: the consumer conv's group count (C_out % out_groups == 0) */
  int32_t shuffle_groups;  /* 1 = none */
  int32_t pool2;           /* 1: MaxPool2d(2, 2) folded in (even P and Q) */
  const float* bn_mean;    /* NULL: no BatchNorm; otherwise all four, [C_out] */
  const float* bn_invstd;
  const float* bn_gamma;
  const float* bn_beta;
} mnb_xnor_post;
int64_t mnb_xnor_post_bytes(const mnb_conv_shape* s, const mnb_xnor_post* post);
int mnb_xnor_conv_post(const mnb_conv_shape* s, const void* a_bits, const void* w_img, const float* alpha, const float* bias,
                       const mnb_xnor_post* post, void* out, mnb_stream_t stream);
int mnb_xnor_pack_act_post(const float* x, int32_t batch, int32_t channels, int32_t h, int32_t w, const mnb_xnor_post* post,
                           void* out_bits, mnb_stream_t stream);
/* host only, the plan mnb_xnor_conv_fwd (post NULL) / mnb_xnor_conv_post runs, from the function their launcher uses:
 * out[0..9] = {R, NW (32-channel words per group), border, px (pixels per thread), post, ksplit (k-slices per group),
 * kb (output channels per k-slice, the last one ragged when K/g % kb != 0), pblocks (pixel blocks), shared-memory bytes,
 * refused}.  refused = 1: the launch returns MNB_E_UNSUPPORTED although mnb_xnor_supported is 1 (shared memory over 48 KB
 * or more than 65535 (group, k-slice) blocks).  Returns MNB_E_UNSUPPORTED outside the cover and check_post's refusals. */
int mnb_xnor_plan(const mnb_conv_shape* s, const mnb_xnor_post* post, int32_t* out);

/* ------------------------------------------------------------------------
 * Binary tensor-core forward for wbwtab layers (mnb_b1.cu): the exact integer sum of mnb_xnor_conv_fwd / mnb_pk_conv
 * (WB:11-36, 55-75, 181-195) on wgmma m64nNk256.s32.b1.b1.and.popc, for the layers outside the XNOR kernel's cover
 * (NIN's 1x1 / 3x3 / 5x5 layers of 160 and 192 channels, models/nin.py; deployed as by wbwtab/bn_fuse).
 *   b1 plane : [B][G * u][H][W][16 bytes], u = ceil(C/g / 64) units per group; a unit holds 64 channels of one pixel,
 *              bits 0-63 p = [value is +1], bits 64-127 n = [value is -1] (bit j of the 64 = channel 64 i + j of the group).
 *              p = n = 0 is a 0: image halo (zero-filled by the TMA unit), channel padding up to a whole unit, and each
 *              group starting on a unit boundary - the zero padding of the reference's +-1 tensor, with no border tables.
 *   w_img    : mnb_b1_wimage_bytes() bytes from the i16 levels {-1, 0, +1} [K][C/g][R][S]: P = [w == +1], M = [w == -1];
 *              output channel k owns two adjacent B columns plus = [P | M] and minus = [M | P], so
 *              D_plus - D_minus = sum (P - M)(p - n) = sum w * a exactly.
 * y = fmaf(sum, alpha[k], bias[k]) equals mnb_xnor_conv_fwd's and mnb_pk_conv's result bit for bit.  Cover: stride 1,
 * dilation 1, square filters up to 7 x 7 with pad <= R / 2, any C/g and K/g; else MNB_E_UNSUPPORTED (mnb_b1_supported: 1 / 0).
 *   mnb_b1_pack_act       : fp32 NCHW -> b1 plane (sign with 0 -> +1, NaN -> +1, like the engine's other binarizers).
 *   mnb_b1_pack_act_post  : fp32 NCHW -> [eval BatchNorm] -> sign [-> 2x2 max-pool] [-> channel shuffle] -> the consumer's
 *                           b1 plane (format MNB_XNOR_B1_PLANE, out_groups = the consumer's groups).
 *   mnb_b1_conv_fwd       : fp32 NCHW output.  err_flag: device int set on a pipeline timeout (as mnb_pk_conv's).
 *   mnb_b1_conv_post      : the epilogue of mnb_xnor_conv_post (BatchNorm, sign, OR-pool, shuffle) into MNB_XNOR_BITS,
 *                           MNB_XNOR_PM1_BF16 or MNB_XNOR_B1_PLANE (bitwise deterministic: the plane is pre-filled, then
 *                           OR / AND-ed into, one word per output pixel and run of channels).
 *   mnb_b1_plane_maxpool  : MaxPool2d(k, s, p) (2p <= k, floor mode) on a b1 plane: p = OR of the in-image p bits,
 *                           n = (OR n) & !p - the max of +-1 values, padding channels stay zero.
 * mnb_xnor_conv_post / mnb_xnor_pack_act_post refuse MNB_XNOR_B1_PLANE (MNB_E_ARG).                                     */
#define MNB_XNOR_B1_PLANE 2
int mnb_b1_supported(const mnb_conv_shape* s);
int64_t mnb_b1_act_bytes(int32_t batch, int32_t channels, int32_t h, int32_t w, int32_t groups);
int mnb_b1_pack_act(const float* x, int32_t batch, int32_t channels, int32_t h, int32_t w, int32_t groups, void* out_plane,
                    mnb_stream_t stream);
int mnb_b1_pack_act_post(const float* x, int32_t batch, int32_t channels, int32_t h, int32_t w, const mnb_xnor_post* post,
                         void* out_plane, mnb_stream_t stream);
int64_t mnb_b1_wimage_bytes(const mnb_conv_shape* s);
int mnb_b1_pack_weight(const mnb_conv_shape* s, const int16_t* w_int, void* w_img, mnb_stream_t stream);
int mnb_b1_conv_fwd(const mnb_conv_shape* s, const void* a_plane, const void* w_img, const float* alpha, const float* bias,
                    float* y, int32_t* err_flag, mnb_stream_t stream);
/* host only, the plan mnb_b1_conv_fwd (post NULL) / mnb_b1_conv_post runs (the launcher's own plan function):
 * out[0..16] = {Nt (B columns of the N tile: kernel instance), n_ntiles, u (64-channel units per group), ksteps, G,
 * col_tiles, Wt (output columns per tile), BW (box width with halo), TH (output rows per tile), TB (images per M tile),
 * row_tiles, n_mtiles, TG (taps per stage), ntg (tap groups), nstage (pipeline stages), post, dynamic shared-memory bytes}.
 * Returns MNB_E_UNSUPPORTED outside the cover and check_post's refusals. */
int mnb_b1_plan(const mnb_conv_shape* s, const mnb_xnor_post* post, int32_t* out);
int64_t mnb_b1_post_bytes(const mnb_conv_shape* s, const mnb_xnor_post* post);
int mnb_b1_conv_post(const mnb_conv_shape* s, const void* a_plane, const void* w_img, const float* alpha, const float* bias,
                     const mnb_xnor_post* post, void* out, int32_t* err_flag, mnb_stream_t stream);
int mnb_b1_plane_maxpool(const void* in_plane, int32_t batch, int32_t channels, int32_t groups, int32_t h, int32_t w, int32_t k,
                         int32_t s, int32_t p, void* out_plane, mnb_stream_t stream);

/* Optimizer step of the QAT loop (torch.optim.Adam semantics, L2 weight decay, no amsgrad;
 * wbwtab/main.py:84,331-339) over one flat fp32 parameter / gradient bucket: a single launch. */
int mnb_adam_step(float* params, const float* grads, float* exp_avg, float* exp_avg_sq, int64_t n, float lr,
                  float beta1, float beta2, float eps, float weight_decay, int32_t step, mnb_stream_t stream);

/* Debug hook: 16 int64 device counters [role: tma, mma, epilogue, converter][wait a, wait b, wait c,
 * total cycles], accumulated by the fwd/dgrad tensor-core kernel while the pointer is non-NULL.  */
void mnb_set_tc_profile_buffer(void* dev_int64x16);

/* ------------------------------------------------------------------------
 * Hardware self-tests of the sm_90a building blocks (run by tests/test_gpu_tc_selftest.py).
 * Bounded waits: a wrong descriptor sets *err_flag (device int) instead of hanging the GPU.
 * ---------------------------------------------------------------------- */
/* D[128 x N] = A[128 x K] * B[N x K]^T through wgmma (bf16 -> f32, or s8 -> s32), two 64-row halves, with
 * thread-written no-swizzle operands; A/B/D are fp32 row-major device arrays.
 * int8: 0 = bf16 K-major operands, 1 = int8 K-major, 2 = bf16 MN-major (the wgrad kernel's form).    */
int mnb_selftest_umma(const float* A, const float* B, float* D, int32_t N, int32_t K, int32_t int8,
                      int32_t* err_flag, mnb_stream_t stream);
/* one cp.async.bulk.tensor.3d box (dims/box/coord innermost-first, fp32) copied to `out`;
 * elements outside the tensor must read back as 0.                                              */
int mnb_selftest_tma3d(const float* src, const int64_t* dims3_host, const int32_t* box3_host,
                       const int32_t* coord3_host, float* out, int32_t* err_flag, mnb_stream_t stream);

/* micro-benchmark: `iters` back-to-back M64 x N x K16 bf16 wgmma (N = 32, 64 or 128) from one warpgroup into one
 * register accumulator (n_acc >= 1 is accepted and ignored); out2[0] = cycles until all have retired, out2[1] = cycles
 * spent issuing.                                                                                   */
int mnb_selftest_mma_rate(int32_t N, int32_t n_acc, int32_t a_shift16, int32_t iters, int32_t mn_major,
                          int64_t* out2, int32_t* err_flag, mnb_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* MICRONET_B200_H */
