/* unicorn_b200 — C ABI of the H100-native Unicorn per-frame inference hot path.
 *
 * Every entry point takes plain device pointers, sizes and a CUDA stream (passed as void* so the header
 * needs no CUDA include).  No entry point allocates, synchronises or keeps state between calls (apart from
 * a lazily resolved driver entry point), so all of them are CUDA-graph capturable.  All return 0 on success
 * and a negative UC_E* / positive cudaError_t code otherwise; uc_last_error() gives the text.
 * There is NO CPU fallback: on a machine without an sm_90 device every launch returns an error.
 *
 * Reference interfaces replaced (paths relative to MasterBin-IIAU/Unicorn):
 *   uc_msda_forward_*      unicorn/models/ops/src/ms_deform_attn.h:20-39  (ms_deform_attn_forward)
 *                          -> unicorn/models/ops/src/cuda/ms_deform_attn_cuda.cu:20-80
 *                          -> ms_deformable_im2col_gpu_kernel, ms_deform_im2col_cuda.cuh:237-299
 *   uc_conv2d              nn.Conv2d / nn.Linear call sites of the backbone, neck, heads:
 *                          backbone/convnext.py:41-54,82-87; network_blocks.py:50-51; unicorn.py:36-44;
 *                          unicorn_head.py:267-336; ops/modules/ms_deform_attn.py:94-113
 *   uc_stem_ln             backbone/convnext.py:77-80 (conv4x4s4 + channels_first LayerNorm)
 *   uc_resnet_stem         backbone/resnet.py:148-152,209-212 (conv7x7s2 + BatchNorm + ReLU + maxpool3x3s2)
 *   uc_dwconv7_ln          backbone/convnext.py:43-45 (dwconv 7x7 + LayerNorm)
 *   uc_layernorm           backbone/convnext.py:176-184; deformable_transformer.py:113,121
 *   uc_groupnorm_*         GroupNorm(16,eps 1e-3) from exp/unicorn_track.py:450-470; unicorn.py:38
 *   uc_corr_propagate      external/lib/test/tracker/unicorn_sot.py:95-100, unicorn_vos.py:171-181
 *   uc_head_decode         unicorn_head.py:332-334,467-482
 *   uc_nms_*               utils/boxes.py:33-77 (torchvision.ops.batched_nms)
 */
#ifndef UNICORN_B200_H_
#define UNICORN_B200_H_
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#if defined(__GNUC__)
#define UC_API __attribute__((visibility("default")))
#else
#define UC_API
#endif

#define UC_OK 0
#define UC_EINVAL (-1)   /* bad argument (shape / alignment / dtype) */
#define UC_EDRIVER (-2)  /* driver entry point (cuTensorMapEncodeTiled) unavailable */
#define UC_ENODEV (-3)   /* no sm_90 device */

/* dtypes of activation tensors */
#define UC_BF16 0
#define UC_F32 1
#define UC_F16 2

/* fused activations */
#define UC_ACT_NONE 0
#define UC_ACT_RELU 1
#define UC_ACT_GELU 2 /* exact erf GELU (nn.GELU()), evaluated as x*sigmoid(x*P(x^2)), |error| < 4e-6 */
#define UC_ACT_SILU 3
#define UC_ACT_SIGMOID 4

UC_API const char* uc_last_error(void);
UC_API int uc_version(void);
/* 0 if the current device is sm_90 and the driver entry points resolve, else a UC_E* code */
UC_API int uc_check_device(void);

/* Dense convolution / linear layer as an implicit GEMM on wgmma tensor cores (TMA-fed, register accumulators).
 *   x : NHWC activations, 16-bit (bf16 or f16 per x_dtype), pixel stride ldx elements (ldx >= Cin, ldx % 8 == 0)
 *   w : packed weights [Cout][KH*KW][Cin] in the same 16-bit type as x (K-major)
 *   y : NHWC output, pixel stride ldy, dtype y_dtype; y = act(conv(x) + bias) ; then y = res + gamma * y if given
 *       (act_after_res: y = relu(conv(x) + bias + res))
 * A Linear layer on [M, Cin] rows is B=1, H=1, W=M, KH=KW=1.  stride in {1,2}; pad < KH.
 * Cin % 8 == 0, Cout % 8 == 0 (pad the weight rows / output channels otherwise).  x, w, y and res are 16-byte aligned.  A 16-bit
 * y tile is staged in shared memory and written by TMA stores, and the residual is read by TMA into the same tile; fp32 y is stored
 * straight from the accumulator registers (64 bits per lane, row and 8-channel chunk).  Every launch is CUDA-graph capturable and
 * uses programmatic dependent launch.
 */
typedef struct UcConv2d {
  const void* x;
  int x_dtype;
  int B, H, W, Cin, ldx;
  const void* w;
  int Cout, KH, KW, stride, pad;
  const float* bias;  /* [Cout] or NULL */
  int act;            /* UC_ACT_* */
  const float* gamma; /* [Cout] layer scale or NULL */
  const void* res;    /* residual, 16-bit like x, rows of ldres elements, or NULL */
  int ldres;
  void* y;
  int ldy;
  int y_dtype;
  int block_n; /* 0 = auto; else force the N tile (16,32,64,96,128,192,256); +1000 (1128,1192,1256) = the 2-CTA
                  cluster variant: two CTAs with consecutive M tiles share one weight stream (TMA multicast) */
  /* Optional GroupNorm statistics of the (pre-activation) output, accumulated per (image, group):
   * gn_stats[b][g] = {sum, sumsq} as int64 fixed point (value * 2^22; integer atomics => order independent,
   * bit-reproducible); must be zeroed by the caller; NULL = off.  Consumed by uc_groupnorm_apply. */
  void* gn_stats;
  int gn_groups;
  /* Optional LayerNorm folded into a 1x1 conv (ConvNeXt block, convnext.py:45-46): x is the UN-normalised map, w = W * diag(ln_w),
   * bias = W @ ln_b + b, col_s[n] = sum_k w[n][k] (of the 16-bit weights), row_stats = per-pixel {sum, sumsq} over Cin of x as
   * written by uc_dwconv7 (int64 fixed point 2^22): y = act(rstd * (w x) - rstd * mu * col_s + bias).  NULL = off. */
  const void* row_stats;
  const float* col_s;
  float row_eps;
  /* 1 = the activation comes after the residual: y = relu(conv(x) + bias + res) (ResNet Bottleneck, resnet.py:115-122: bn3 folded
   * into w / bias, identity added, then ReLU).  Needs act = UC_ACT_RELU, res and bf16 x; rejected (UC_EINVAL) otherwise and with
   * gamma, gn_stats or row_stats.  0 = as above. */
  int act_after_res;
} UcConv2d;
UC_API int uc_conv2d(const UcConv2d* d, void* stream);

/* ConvNeXt stem: Conv2d(3,C0,k4,s4)+bias then channels_first LayerNorm (backbone/convnext.py:77-80,179-184).
 * img: fp32 NCHW [B,3,H,W] (PreprocessorX output, unicorn_sot.py:114-123) or, with img_is_u8_hwc = 1, the uint8 HWC
 * BGR frame [B,H,W,3] as cv2 delivers it (the permute / float conversion is fused into the load);
 * w48 fp32 [48][C0] with k=(ci*4+kh)*4+kw; out NHWC bf16 [B,H/4,W/4,C0]. */
UC_API int uc_stem_ln(const void* img, int img_is_u8_hwc, const float* w48, const float* bias, const float* lnw, const float* lnb,
                      void* out_bf16, int B, int H, int W, int C0, float eps, void* stream);

/* ResNet-50 stem in ONE launch (backbone/resnet.py:148-152,209-212): conv 7x7 stride 2 pad 3 (3 -> 64) with the eval-mode
 * BatchNorm folded into the weights and bias, ReLU, max-pool 3x3 stride 2 pad 1.  The H/2 x W/2 x 64 map before the pool stays in
 * shared memory; only the pooled map is written.  The conv runs on tensor cores (mma.sync m16n8k16, fp16 operands, fp32 accumulate):
 * the 0-255 integer pixels are exact in fp16, so the only roundings are those of the folded weights (fp16: 11-bit significand, 8x finer
 * than bf16) and of the bf16 output.  img: fp32 NCHW [B,3,H,W] or, with img_is_u8_hwc = 1, the uint8 HWC BGR frame [B,H,W,3] (same
 * forms as uc_stem_ln); w_f16 [64][160] fp16, k = ci*49 + kh*7 + kw, zero for k >= 147 (unicorn_b200.ops.pack_resnet_stem_weight);
 * bias fp32 [64]; out NHWC bf16 [B,H/4,W/4,64], 16-byte aligned.  H % 4 == 0, W % 4 == 0. */
UC_API int uc_resnet_stem(const void* img, int img_is_u8_hwc, const void* w_f16, const float* bias, void* out_bf16, int B, int H, int W,
                          void* stream);

/* ConvNeXt block front half in ONE launch: depthwise 7x7 (pad 3)+bias then LayerNorm over C (convnext.py:43-45); the
 * intermediate map stays in shared memory (C % 64 == 0; other C use a one-warp-row kernel).  Not in place.  The engine uses
 * uc_dwconv7 + uc_layernorm instead, which is faster on ConvNeXt-L's shapes (DESIGN.md 4.3).
 * x,y NHWC bf16 contiguous [B,H,W,C]; w49 fp32 [49][C] (k = kh*7+kw). */
UC_API int uc_dwconv7_ln(const void* x_bf16, const float* w49, const float* bias, const float* lnw, const float* lnb,
                         void* y_bf16, int B, int H, int W, int C, float eps, void* stream);

/* Depthwise 7x7 (pad 3) + bias of the ConvNeXt block (convnext.py:43), TMA staged (csrc/dwconv_tma.cu); follow with uc_layernorm,
 * or give ln_stats and fold the LayerNorm into pwconv1 (UcConv2d.row_stats).  x, y NHWC bf16 contiguous, not in place; w49 fp32 [49][C].
 * C % 8 == 0; x, y and w49 16-byte aligned, bias 8-byte aligned (UC_EINVAL otherwise).
 * ln_stats (optional, may be NULL): [B*H*W][2] int64 fixed point (value * 2^22), zeroed by the caller; receives the per-pixel
 * {sum, sum of squares} over C of the stored outputs.  work_counter (optional, may be NULL): one device int, ZERO before the launch,
 * used to hand out the tiles dynamically (balanced SM loads on small maps); NULL = static round-robin. */
UC_API int uc_dwconv7(const void* x_bf16, const float* w49, const float* bias, void* y_bf16, int B, int H, int W, int C,
                      void* ln_stats, int* work_counter, void* stream);

/* The same depthwise 7x7 + bias on tensor cores (csrc/dwconv_mma.cu): every filter row is a banded 16 x 8 Toeplitz block applied with
 * mma.sync.m16n8k16 to a channel-planar copy of the input tile.  qtab = per 32-channel chunk {int32 [32][7][8]: the filter as bf16
 * tap pairs {f[kh][j-1], f[kh][j]}, j = 0..7, zero outside the row; fp32 [32]: the biases}, zero for the channels that pad C to a
 * multiple of 32 (unicorn_b200.ops.pack_dw_weight_mma); C % 8 == 0.  Same x / y / work_counter conventions as uc_dwconv7; no ln_stats. */
UC_API int uc_dwconv7_mma(const void* x_bf16, const void* qtab, void* y_bf16, int B, int H, int W, int C, int* work_counter, void* stream);

/* Fused back half of a ConvNeXt block (unicorn/models/backbone/convnext.py:45-52: norm -> pwconv1 -> GELU -> pwconv2 -> gamma ->
 * residual) in one launch, for C = 96 / 192 / 256 / 384 (uc_convnext_mlp_supported): x[M][C] += gamma * (W2 . GELU(W1f . LN0(t) + c1) + b2), LN0 =
 * LayerNorm without affine (eps = ln_eps) over the C channels of a row of t[M][C] (the depthwise-conv output), W1f[4C][C] = pwconv1
 * weight with the LayerNorm weight folded in (W1 diag(g)), c1[4C] = b1 + W1 beta, W2[C][4C].  bf16 maps and weights, fp32 vectors;
 * t / weights 16-byte, x / vectors 32-byte aligned.  The 4C hidden activations stay in shared / tensor memory (csrc/mlp_fused.cu). */
UC_API int uc_convnext_mlp_supported(int C);
UC_API int uc_convnext_mlp(const void* t_bf16, const void* w1f_bf16, const float* c1, const void* w2_bf16, const float* b2, const float* gamma,
                           void* x_bf16, int M, int C, float ln_eps, void* stream);

/* Row LayerNorm: y[m,:] = LN(x[m,:] + res[m,:]) * w + b  (res may be NULL).  16-bit rows with element strides.
 * convnext.py:176-184 (downsample / out norms), deformable_transformer.py:113,121,127-130 (post-norm). */
UC_API int uc_layernorm(const void* x, int ldx, const void* res, int ldres, const float* w, const float* b, void* y,
                        int ldy, long M, int C, float eps, int dtype, void* stream);

/* GroupNorm apply with the statistics accumulated by uc_conv2d (gn_stats = [B][G]{sum,sumsq}):
 * y = act((x-mean)*rstd*w+b) [+ prior[pix]*beta[c]] ; optional second output y2 = y + add2.
 * network_blocks.py:50-51 with exp/unicorn_track.py:450-470 (GN16, eps 1e-3, SiLU); unicorn.py:38 (GN32, eps 1e-5);
 * unicorn_head.py:272-275 (prior fusion).  x,y,add2,y2 bf16 NHWC with pixel strides, 16-byte aligned; stats 8-byte aligned.
 * act is UC_ACT_NONE, UC_ACT_RELU or UC_ACT_SILU; G >= 1, C % G == 0, C <= 4096 (UC_EINVAL otherwise). */
UC_API int uc_groupnorm_apply(const void* x, int ldx, const void* stats, const float* w, const float* b, void* y,
                              int ldy, int B, long HW, int C, int G, float eps, int act, const float* prior,
                              const float* beta, const void* add2, int ldadd2, void* y2, int ldy2, void* stream);
/* The same normalisation with the source image of each output image taken from a device table (a head stem shared by several head
 * images, of one video or of several): x holds n_src images [n_src][HW pixels] (row stride ldx, image stride HW * ldx) and stats
 * their [n_src][G]{sum,sumsq}; src_of is a device int32 [B] table read when the kernel runs, so a captured graph follows its current
 * contents.  y holds B images [B][HW pixels], image stride HW * ldy.  Output image b normalises image src_of[b] with that image's
 * statistics; b < n_plain = act((x-mean)*rstd*w+b) (the no-prior path: adding a zero prior would turn a -0 into +0), b >= n_plain
 * adds prior[(b - n_plain) * HW + pix] * beta[c].  Every image equals uc_groupnorm_apply at B = 1 on image src_of[b], with or
 * without its prior, bit for bit.  A table entry outside [0, n_src) leaves output image b untouched and reads nothing of x, stats or
 * prior.  1 <= n_src, B <= 65535, 0 <= n_plain <= B; src_of non-null and 4-byte aligned; prior (4-byte aligned) and beta are given
 * exactly when n_plain < B; x (all n_src images) and y must not overlap; otherwise the conventions of uc_groupnorm_apply (UC_EINVAL
 * before any launch). */
UC_API int uc_groupnorm_apply_gather(const void* x, int ldx, int n_src, const void* stats, const float* w, const float* b, void* y,
                                     int ldy, int B, int n_plain, const int* src_of, long HW, int C, int G, float eps, int act,
                                     const float* prior, const float* beta, void* stream);

/* dst[b,oh,ow,:C] = src[b,oh/up,ow/up,:C], up in {1,2} (nearest upsample + concat slice; yolo_pafpn_new.py:139-146).
 * 16-bit NHWC; C, lds, ldd multiples of 8; src and dst 16-byte aligned. */
UC_API int uc_copy_upsample(const void* src, int lds, void* dst, int ldd, int B, int Hs, int Ws, int C, int up, void* stream);
/* nn.PixelShuffle(2) in NHWC (unicorn.py:41): in [B,H,W,4*Co] -> out [B,2H,2W,Co], 16-bit. */
UC_API int uc_pixel_shuffle2(const void* in, int ldi, void* out, int ldo, int B, int H, int W, int Co, void* stream);
/* F.interpolate(bilinear, align_corners=False) on fp32 planes [P,Hs,Ws]->[P,Hd,Wd]; scale_* = 1/scale_factor or 0. */
UC_API int uc_bilinear_f32(const float* src, float* dst, int P, int Hs, int Ws, int Hd, int Wd, float scale_h,
                           float scale_w, void* stream);
/* Letterbox preprocessing on the device (PreprocessorX.process, external/lib/test/tracker/unicorn_sot.py:114-123; preproc,
 * unicorn/data/data_augment.py:194-214): dst[0:rh,0:rw] = cv2.resize(src,(rw,rh),INTER_LINEAR) — bit-exact restatement of
 * OpenCV's 8-bit fixed-point bilinear —, the rest = pad (114); swap_rb does cv2.COLOR_RGB2BGR.  uint8 HWC, 3 channels. */
UC_API int uc_letterbox_u8(const uint8_t* src_hwc, int Hs, int Ws, uint8_t* dst_hwc, int Hd, int Wd, int rh, int rw,
                           int swap_rb, int pad, void* stream);
/* uc_letterbox_u8's output (swap_rb = 1) for the BGR frame cv2.cvtColor(COLOR_YUV2BGR_NV12) makes of an NV12 frame (BT.601 limited
 * range, OpenCV's 20-bit fixed point), bit-exact, without storing that frame: y = the Hs x Ws luma plane, uv = the interleaved
 * Hs/2 x Ws chroma plane (U, V pairs), both with row pitch ld >= Ws bytes (decoder surfaces: the planes may be apart).  Hs, Ws even;
 * 1 <= rh <= Hd, 1 <= rw <= Wd; 0 <= pad <= 255.  BGR uint8 HWC out, top-left placement. */
UC_API int uc_letterbox_nv12(const uint8_t* y, const uint8_t* uv, int ld, int Hs, int Ws, uint8_t* dst_hwc, int Hd, int Wd, int rh,
                             int rw, int pad, void* stream);
/* y = a + b on 16-bit (UC_BF16 / UC_F16) rows; C and the strides multiples of 8; a, b and y 16-byte aligned. */
UC_API int uc_add(const void* a, int lda, const void* b, int ldb, void* y, int ldy, long M, int C, int dtype, void* stream);
/* Conditional strided row copy decided on the device: rows are copied when (*flag_dev != 0) != invert.  The MOT drivers use it for
 * "pre_dict = cur_dict only when this frame produced detections" (unicorn/evaluators/mot_evaluator.py:1005,1014-1020) so that the
 * frame needs no host decision (CUDA-graph replay).  16-byte aligned rows / strides. */
UC_API int uc_copy_rows_if(const int* flag_dev, int invert, const void* src, long src_ld_bytes, void* dst, long dst_ld_bytes, long rows,
                           int row_bytes, void* stream);
/* The same for B >= 1 images in one launch: image b copies its rows (src + b * src_bs_bytes -> dst + b * dst_bs_bytes) when
 * (gate_dev == NULL || gate_dev[b] != 0) && ((flag_dev[b] != 0) != invert); flag_dev / gate_dev device int32 [B].  The multi-sequence
 * MOT driver gates with the step's active-slot table so that an idle slot keeps its pre_dict.  Rows and strides as uc_copy_rows_if
 * (16-byte aligned), per-image strides multiples of 16 and >= rows * ld.  B < 1, null pointers or smaller strides: UC_EINVAL. */
UC_API int uc_copy_rows_if_batched(const int* flag_dev, const int* gate_dev, int invert, const void* src, long src_ld_bytes, long src_bs_bytes,
                                   void* dst, long dst_ld_bytes, long dst_bs_bytes, long rows, int row_bytes, int B, void* stream);
UC_API int uc_nchw_f32_to_nhwc(const float* src, void* dst, int ldd, int B, int C, long HW, int dtype, void* stream);
UC_API int uc_nhwc_to_nchw_f32(const void* src, int lds, float* dst, int B, int C, long HW, int dtype, void* stream);

/* Drop-in for MultiScaleDeformableAttention.ms_deform_attn_forward (ops/src/ms_deform_attn.h:20-39):
 * value [B,S,M,D] f32, spatial_shapes [L,2] i64 (device), level_start_index [L] i64 (device),
 * sampling_loc [B,Lq,M,L,P,2] f32 normalised (x,y), attn_weight [B,Lq,M,L,P] f32 -> out [B,Lq,M*D] f32. */
UC_API int uc_msda_forward_f32(const float* value, const int64_t* spatial_shapes, const int64_t* level_start_index,
                               const float* sampling_loc, const float* attn_weight, int B, int S, int M, int D, int L,
                               int Lq, int P, float* out, void* stream);
/* Fused form used by the H100 path (head dim 32): value bf16 [S, M*32]; offlog f32 [Lq, ld] = raw
 * sampling_offsets (M*L*P*2) followed by attention logits (M*L*P); queries = concatenated level grids;
 * level_hw host int[2L] (h,w).  out bf16 [Lq, M*32]. */
UC_API int uc_msda_fused_bf16(const void* value, const float* offlog, int ld_offlog, void* out, const int* level_hw,
                              int L, int M, int P, void* stream);
/* The same for B >= 1 images in one launch.  Rows of value / offlog / out are level-major with the images inside each level:
 * level l of image b starts at row B * (h_0*w_0 + ... + h_{l-1}*w_{l-1}) + b * h_l*w_l (B = 1 is uc_msda_fused_bf16's layout).
 * Every image samples only its own value rows.  B < 1: UC_EINVAL. */
UC_API int uc_msda_fused_bf16_batched(const void* value, const float* offlog, int ld_offlog, void* out, const int* level_hw,
                                      int L, int M, int P, int B, void* stream);

/* Fused correlation + softmax over reference positions + label propagation
 * (external/lib/test/tracker/unicorn_sot.py:95-100; unicorn_vos.py:171-181):
 *   out[o,j] = sum_i values[o,i] * softmax_i(<embed_ref[i,:], embed_cur[j,:]>)
 * embed_* [n, C=128] 16-bit rows (NHWC embedding maps), values f32 [n_obj, ldv], out f32 [n_obj, ldo]; n_obj <= 8. */
UC_API int uc_corr_propagate(const void* embed_ref, int ld_ref, int n_ref, const void* embed_cur, int ld_cur, int n_cur,
                             int C, int dtype, const float* values, int ldv, int n_obj, float* out, int ldo, void* stream);
/* B >= 1 independent (embed_ref, embed_cur, values) -> out problems in one launch (grid: current-position tiles x sequences).
 * bs_* are the element strides from one sequence to the next: bs_ref, bs_cur multiples of 8 and >= ld * n; bs_values >= ldv * n_obj;
 * bs_out >= ldo * n_obj (UC_EINVAL otherwise; ignored when B = 1).  Each sequence's output equals its own uc_corr_propagate. */
UC_API int uc_corr_propagate_batched(const void* embed_ref, int ld_ref, long bs_ref, int n_ref, const void* embed_cur, int ld_cur,
                                     long bs_cur, int n_cur, int C, int dtype, const float* values, int ldv, long bs_values, int n_obj,
                                     float* out, int ldo, long bs_out, int B, void* stream);

/* Head decode (unicorn_head.py:332-334,467-482): per level regobj f32 [HW, ld_ro] = reg(4), obj logit;
 * cls f32 [HW, ld_cls] = class logits.  regobj/cls/hw/strides are HOST arrays of 3 device pointers / ints.
 * out f32 [sum HW, 5+ncls] = cx,cy,w,h,sigmoid(obj),sigmoid(cls..). */
UC_API int uc_head_decode(const float* const* regobj, const float* const* cls, const int* hw, const int* strides,
                          int ld_ro, int ld_cls, int ncls, float* out, void* stream);
/* B >= 1 images: image b of level k starts at regobj[k] + b * bs_ro[k] / cls[k] + b * bs_cls[k] (HOST arrays of 3 element
 * strides, each >= h_k*w_k*ld; ignored when B = 1); out f32 [B, sum HW, 5+ncls]. */
UC_API int uc_head_decode_batched(const float* const* regobj, const float* const* cls, const int* hw, const int* strides,
                                  int ld_ro, int ld_cls, const long* bs_ro, const long* bs_cls, int ncls, int B, float* out,
                                  void* stream);

/* postprocess (utils/boxes.py:33-77) on the device: out_dets f32 [<=A, 7] rows (x1,y1,x2,y2,obj,cls_conf,cls_id)
 * in descending score order, *out_count (device int) = number of rows.  max_keep > 0 stops the greedy scan once that
 * many boxes are kept: the rows returned are exactly the first max_keep rows of the full result (the SOT driver only
 * consumes output[:max_inst], external/lib/test/tracker/unicorn_sot.py:69-70); max_keep <= 0 = no limit.
 * out_anchor (device int[A], may be NULL) receives the anchor index of every returned row — what postprocess_inst
 * (utils/boxes.py:125-128) needs to pick each instance's location / dynamic parameters / FPN level.
 * Decisions are pinned bit for bit: a row passes when rn(obj * cls_conf) >= conf_thre (cls_conf the first maximum), and the
 * NMS of each class equals torchvision.ops.nms on CUDA (devIoU: union = fmaf(w_later, h_later, area_earlier) - inter, IEEE
 * divide, IoU > (float)nms_thre suppresses), rows of equal score in ascending candidate order. */
UC_API long uc_postprocess_workspace_bytes(int max_anchors);
UC_API int uc_postprocess(const float* pred, int A, int ncls, float conf_thre, float nms_thre, int max_keep, void* workspace,
                          long workspace_bytes, float* out_dets, int* out_count, int* out_anchor, void* stream);
/* The same for B >= 1 images in one launch sequence (one CTA per image in each of the four kernels): pred f32 [B, A, 5+ncls],
 * out_dets [B, A, 7], out_count [B], out_anchor [B, A] (or NULL); max_keep applies per image.  The workspace holds B per-image
 * slices: uc_postprocess_workspace_bytes_batched(A, B) bytes (0 for B < 1).  B < 1 or a smaller workspace: UC_EINVAL. */
UC_API long uc_postprocess_workspace_bytes_batched(int max_anchors, int B);
UC_API int uc_postprocess_batched(const float* pred, int A, int ncls, float conf_thre, float nms_thre, int max_keep, int B,
                                  void* workspace, long workspace_bytes, float* out_dets, int* out_count, int* out_anchor, void* stream);

/* Flags of the *_ex / *_nms entry points.  UC_POST_CLASS_AGNOSTIC: NMS over all classes (postprocess(..., class_agnostic=True),
 * torchvision.ops.nms); without it NMS is class-aware as in uc_postprocess.  Unknown bits: UC_EINVAL. */
#define UC_POST_CLASS_AGNOSTIC 1
UC_API int uc_postprocess_batched_ex(const float* pred, int A, int ncls, float conf_thre, float nms_thre, int max_keep, int B, int flags,
                                     void* workspace, long workspace_bytes, float* out_dets, int* out_count, int* out_anchor, void* stream);
/* Decode + score filter of B images read straight from the per-level head maps (the arguments of uc_head_decode_batched), without
 * the [B, A, 5+ncls] tensor: fills the workspace (uc_postprocess_workspace_bytes_batched(A, B), A = sum h*w) with exactly the
 * candidates, keys and anchor ids that uc_head_decode_batched followed by the filter of uc_postprocess_batched leave there.
 * uc_postprocess_nms_batched then runs the sort, gather and greedy NMS of uc_postprocess_batched on that workspace. */
UC_API int uc_det_candidates_batched(const float* const* regobj, const float* const* cls, const int* hw, const int* strides, int ld_ro,
                                     int ld_cls, const long* bs_ro, const long* bs_cls, int ncls, int B, float conf_thre, void* workspace,
                                     long workspace_bytes, void* stream);
UC_API int uc_postprocess_nms_batched(int A, float nms_thre, int max_keep, int B, int flags, void* workspace, long workspace_bytes,
                                      float* out_dets, int* out_count, int* out_anchor, void* stream);

/* Instance-embedding sampling at box centres (unicorn/evaluators/mot_evaluator.py:1024-1034): embed NHWC 16-bit
 * [h,w,C] (pixel stride ld), boxes f32 [n,ldb] xyxy in network-input pixels, stride = 8; grid_sample(bilinear,
 * border, align_corners=False) semantics incl. the reference's clamp/normalise step.  n = min(*count_dev, n_max)
 * (count_dev may be NULL).  out f32 [n_max, C]. */
UC_API int uc_sample_embed(const void* embed, int ld, int h, int w, int C, int dtype, const float* boxes, int ldb,
                           const int* count_dev, int n_max, float stride, float* out, void* stream);
/* The same for B >= 1 images in one launch (grid: boxes x images): image b samples embed + b * bs_embed at the boxes
 * boxes + b * bs_boxes (the [B, A, 7] NMS output of uc_postprocess_batched) for its first min(count_dev[b], n_max) rows and writes
 * out + b * bs_out; rows at or past that count are not written.  Element strides bs_embed >= h*w*ld, bs_boxes >= n_max*ldb,
 * bs_out >= n_max*C.  B < 1, null pointers (count_dev included) or smaller strides: UC_EINVAL.  Each image's rows equal its own
 * uc_sample_embed call. */
UC_API int uc_sample_embed_batched(const void* embed, int ld, long bs_embed, int h, int w, int C, int dtype, const float* boxes, int ldb,
                                   long bs_boxes, const int* count_dev, int n_max, float stride, float* out, long bs_out, int B, void* stream);
/* Quasi-dense association score (unicorn/tracker/quasi_dense_embed_tracker.py:166-175): scores = (softmax_rows(F) +
 * softmax_cols(F)) / 2 with F = E M^T, zeroed where labels differ (labels may be NULL).  workspace >= N*M+2N+2M floats. */
UC_API int uc_bisoftmax(const float* det_embeds, const float* memo_embeds, int N, int M, int C, const float* det_labels,
                        const float* memo_labels, float* workspace, float* scores, void* stream);
/* Greedy assignment of QuasiDenseEmbedTracker.match (unicorn/tracker/quasi_dense_embed_tracker.py:188-199) on the device: rows =
 * detections in descending score order, scores f32 [N,M] from uc_bisoftmax, memo_ids int64 [M] (-1 = backdrop), det_scores f32
 * (element stride ld_det: column 4 of the [N,5] box rows).  ids_out int64 [N]: the tracklet id, -2 (duplicate of a tracklet, dropped)
 * or -1 (unmatched).  taken_ws: M bytes of scratch.  One CTA; torch.max tie-breaking (first maximum). */
UC_API int uc_qd_assign(const float* scores, int N, int M, const long long* memo_ids, const float* det_scores, int ld_det, float match_thr,
                        float obj_thr, float nms_conf_thr, long long* ids_out, uint8_t* taken_ws, void* stream);
/* Pairwise IoU out[i,j] of xyxy f32 boxes with row strides.  plus_one = 0: torchvision.ops.box_iou
 * (quasi_dense_embed_tracker.py:80,146); plus_one = 1: cython_bbox.bbox_overlaps' inclusive-pixel convention
 * (unicorn/tracker/matching.py:65-68, ByteTrack).  Every fp32 step is rounded on its own (no fused multiply-add), so
 * plus_one = 0 equals torchvision.ops.box_iou bit for bit; plus_one = 1 is that order in fp32 where bbox_overlaps uses float64. */
UC_API int uc_box_iou(const float* a, int lda, int N, const float* b, int ldb, int M, float* out, int plus_one, void* stream);

/* dst += aligned_bilinear(src, factor) on NHWC bf16 maps (condinst/comm.py:5-27; mask_branch.py:81-96). */
UC_API int uc_aligned_bilinear_add(const void* src, int lds, int hs, int ws, void* dst, int ldd, int C, int factor, void* stream);
/* The same for B >= 1 images in one launch: image b reads src + b * bs_src and updates dst + b * bs_dst (element strides, even,
 * bs_src >= hs*ws*lds, bs_dst >= hs*f*ws*f*ldd).  B < 1, null pointers or smaller strides: UC_EINVAL. */
UC_API int uc_aligned_bilinear_add_batched(const void* src, int lds, long bs_src, int hs, int ws, void* dst, int ldd, long bs_dst, int C,
                                           int factor, int B, void* stream);
/* Per-instance CondInst masks (condinst/dynamic_mask_head.py:61-87,159-225,284; utils/boxes.py:138-145) for the first
 * min(*count_dev, n_max) rows of the NMS output: mask_feats f32 [h,w,8], up_masks f32 [h,w,9*up_rate^2],
 * dyn_levels = HOST array of 3 device pointers to the controller outputs [h_k*w_k, ld_dyn] (169 used), level_hw /
 * level_strides / level_soi host arrays; anchors_dev = out_anchor of uc_postprocess; scratch >= n_max*h*w*(1+up^2)
 * floats; out_masks f32 [n_max, h*up*d, w*up*d] = sigmoid scores. */
UC_API int uc_dynamic_masks(const float* mask_feats, const float* up_masks, int h, int w, int up_rate, int d_rate,
                            const float* const* dyn_levels, int ld_dyn, const int* level_hw, const int* level_strides,
                            const float* level_soi, const int* anchors_dev, const int* count_dev, int n_max, float* scratch,
                            float* out_masks, void* stream);
/* The same for B >= 1 head images in one launch sequence (grid: pixels x instances x images).  Head image b has its controller
 * outputs at dyn_levels[k] + b * bs_dyn[k] (HOST array of 3 element strides, each >= h_k*w_k*ld_dyn), its NMS result at
 * anchors_dev + b * bs_anchors (bs_anchors >= the anchor count sum h_k*w_k) and count_dev[b] (the [B, A] / [B] layout of
 * uc_postprocess_batched), and reads mask-branch image image_of[b] (device int32 [B]) of the S images mask_feats f32 [S,h,w,8] /
 * up_masks f32 [S,h,w,9*up_rate^2]; an image_of entry outside [0, S) skips head image b (nothing is read or written for it).
 * scratch >= B*n_max*h*w*(1+up^2) floats; out_masks f32 [B, n_max, h*up*d, w*up*d].  Each image's masks equal its own
 * uc_dynamic_masks call.  B < 1, S < 1, null pointers (image_of and bs_dyn included) or smaller strides: UC_EINVAL. */
UC_API int uc_dynamic_masks_batched(const float* mask_feats, const float* up_masks, int S, int h, int w, int up_rate, int d_rate,
                                    const float* const* dyn_levels, int ld_dyn, const long* bs_dyn, const int* level_hw,
                                    const int* level_strides, const float* level_soi, const int* anchors_dev, long bs_anchors,
                                    const int* count_dev, const int* image_of, int B, int n_max, float* scratch, float* out_masks,
                                    void* stream);

/* VOS result assembly on the device (external/lib/test/tracker/unicorn_vos.py:129-155 mask resize to the original frame,
 * :105-121 soft aggregation + argmax): for every object either `mask` (f32 [Hin,Win] soft mask at network resolution, resized
 * with F.interpolate(scale_factor=1/r, bilinear, align_corners=False)[:H,:W]) or `init_mask` (uint8 [H,W] label map of the
 * frame the object first appears in; object = label == id) or neither (no detection: zeros).  objs is a HOST array in the
 * reference's list order (the float32 background product follows it).  soft_out (may be NULL) f32 [n,H,W]; seg_out uint8 [H,W]. */
typedef struct UcVosObject {
  const float* mask;
  const uint8_t* init_mask;
  int id;
} UcVosObject;
UC_API int uc_vos_aggregate(const UcVosObject* objs, int n, int Hin, int Win, int H, int W, float r, float* soft_out,
                            uint8_t* seg_out, void* stream);

/* uc_vos_aggregate of B videos (1 <= B <= UC_VOS_MAX_VIDEOS) in one launch, all at the network resolution Hin x Win.  Video b has
 * its own objects (objs: HOST array of n, 1 <= n <= 16, ids 1..255, in the reference's list order), original size H x W, letterbox
 * ratio r > 0 and outputs (soft_out may be NULL; seg_out may not).  videos is a HOST array of B.  Video b's seg and soft equal those
 * of uc_vos_aggregate called on video b alone, bit for bit; uc_vos_aggregate is this call with B = 1.  Every argument is validated
 * before any CUDA call; no allocation, no synchronisation, one launch. */
#define UC_VOS_MAX_VIDEOS UC_MOTS_MAX_IMAGES
typedef struct UcVosVideo {
  const UcVosObject* objs;
  int n;
  int H, W;
  float r;
  float* soft_out;
  uint8_t* seg_out;
} UcVosVideo;
UC_API int uc_vos_aggregate_batched(const UcVosVideo* videos, int B, int Hin, int Win, void* stream);

/* MOTS result encoding on the device (unicorn/evaluators/mot_evaluator.py:804-805, :858-866, :884-888): for the k instances of
 * one frame, masks f32 [n_max,Hin,Win] (the uc_dynamic_masks output) are resized to the original H x W frame as in uc_vos_aggregate
 * (only the hm x wm corner F.interpolate produces, hm = min(H, floor(Hin/r)), is encoded), thresholded (> thr), made overlap free
 * (instance j keeps the pixels no instance before it in `order` had in its thresholded mask) and written as COCO compressed RLE
 * strings (column-major runs from the zero run, unicorn_b200.results.rle_encode).  order: device int32 [k], the mask rows in
 * ascending track id; emit: device uint8 [k], 0 = the instance still hides pixels from the later ones but gets an empty string.
 * r is the letterbox ratio in double precision (the output size floor(Hin/r) depends on its last bits).  offsets: device int64
 * [k+1], string j is chars[offsets[j] .. offsets[j+1]), offsets[k] = the chars needed; chars: device buffer of `capacity` bytes,
 * nothing at or past capacity is written (re-run with a larger buffer: the call is idempotent).  workspace: device, 16-byte
 * aligned, uc_mots_encode_workspace_bytes(k, H, W) bytes.  Three launches for k > 0, one for k = 0. */
UC_API long uc_mots_encode_workspace_bytes(int k_max, int H, int W);
UC_API int uc_mots_encode(const float* masks, int n_max, int Hin, int Win, const int* order, const uint8_t* emit, int k, float thr,
                          double r, int H, int W, void* workspace, long workspace_bytes, char* chars, long capacity,
                          long long* offsets, void* stream);

/* uc_mots_encode over the instances of B images (1 <= B <= UC_MOTS_MAX_IMAGES) in one set of launches: each image has its own
 * original size H[b] x W[b], letterbox ratio r[b] and k[b] instances (0 <= k[b] <= n_max); k, H, W and r are HOST arrays of B.
 * masks: f32 image b at masks + b * bs_masks, [n_max,Hin,Win] (the uc_dynamic_masks_batched output).  order / emit: device, one flat
 * list of K = sum k[b] entries grouped by image; image b's order entries are mask rows within its own block.  Overlap removal stays
 * within an image.  offsets: device int64 [K+1] over all images, so image b's strings are contiguous; every string is byte-identical
 * to a uc_mots_encode call on that image alone (that call's offsets are image b's minus offsets[k[0] + ... + k[b-1]]).  chars and
 * capacity as in uc_mots_encode.  workspace: uc_mots_encode_workspace_bytes(K, max H[b], max W[b]) bytes suffice.  No allocation,
 * no synchronisation, graph-capturable; three launches for K > 0, one for K = 0. */
#define UC_MOTS_MAX_IMAGES 64
UC_API int uc_mots_encode_batched(const float* masks, long bs_masks, int n_max, int Hin, int Win, int B, const int* k, const int* H,
                                  const int* W, const double* r, const int* order, const uint8_t* emit, float thr, void* workspace,
                                  long workspace_bytes, char* chars, long capacity, long long* offsets, void* stream);

/* COCO instance-segmentation result encoding on the device (unicorn/evaluators/coco_inst_evaluator.py convert_to_coco_format): one
 * COCO compressed RLE string per (image, row) slot of B images (1 <= B <= UC_MOTS_MAX_IMAGES), without the full-resolution masks.
 * maps: f32 image b at maps + b * bs_maps, [n_max, hs, ws], the sigmoid masks uc_dynamic_masks_batched writes with d_rate = 1 for
 * NMS rows row0 .. row0 + n_max - 1.  Slot j = b * n_max + i holds row row0 + i of image b; it is emitted (emit[j] = 1, written by
 * the call: device uint8 [B * n_max]) when row0 + i < count_dev[b] (device int32 [B], read on the device), else it gets an empty
 * string.  Each emitted mask is upsampled by aligned_bilinear(x d_rate) to the network input (hs * d_rate) x (ws * d_rate), bit for
 * bit as uc_dynamic_masks stores it, resized by 1/r[b] to the original frame as in uc_mots_encode, thresholded (> thr) and encoded
 * over the whole H[b] x W[b] frame: pixels outside the hm x wm corner the resize covers are background.  There is no overlap removal.
 * H, W, r: HOST arrays of B.  offsets: device int64 [B * n_max + 1]; chars / capacity as in uc_mots_encode (idempotent: re-run with a
 * larger buffer).  workspace: uc_mots_encode_workspace_bytes(B * n_max, max H[b], max W[b]) bytes, 16-byte aligned.  B * n_max <= 65535.
 * Every argument is validated before any CUDA call; no allocation, no synchronisation, graph-capturable; three launches. */
UC_API int uc_inst_encode_batched(const float* maps, long bs_maps, int n_max, int hs, int ws, int d_rate, int B, const int* count_dev,
                                  int row0, const int* H, const int* W, const double* r, float thr, void* workspace, long workspace_bytes,
                                  uint8_t* emit, char* chars, long capacity, long long* offsets, void* stream);

/* BDD100K MOTS bitmasks on the device (qdtrack core/to_bdd100k/utils.py:15-38, mask_prepare + mask_merge; the seg_track result of
 * tools/to_bdd100k.py): for B frames (1 <= B <= UC_MOTS_MAX_IMAGES), frame b with k[b] tracked instances (0 <= k[b] <= 65535) and size
 * H[b] x W[b] (H * W < 2^31), the uint8 row-major [H, W, 4] RGBA array mask_merge saves as PNG, at out + out_offsets[b] (byte offsets
 * into the out_bytes bytes of out, 4-byte aligned, frames not overlapping).  k, H, W, out_offsets: HOST arrays of B.
 * DEVICE inputs, one flat list of K = sum k[b] instances grouped by frame: string j = chars[offsets[j] .. offsets[j+1]) (offsets int64
 * [K+1] into the n_chars chars) is instance j's COCO compressed RLE counts over its frame (column-major, pycocotools' string form);
 * colors[j] its packed colour, byte 0 = R at the lowest address (label + 1, 0, id >> 8, id & 255 as uint8); ranks[j] its position in
 * the paint order of its frame (np.argsort of the scores: 0 is painted first), a permutation of 0 .. k[b]-1.  A pixel takes the
 * colour of the covering instance of highest rank (all four channels, zeros included); a pixel no instance covers is 0.  The ranks are
 * used as given: the call does not sort.  A frame without instances is all zeros.
 * status: device int32 [B], written by the call: frame b's UC_BDD_* flags, 0 when every string of the frame is well formed.  A
 * malformed string paints nothing and never writes outside its frame.  workspace: device, 16-byte aligned,
 * uc_bdd_bitmask_workspace_bytes(B, k, H, W, n_chars) bytes (-1 for bad arguments).  Every argument is validated before any CUDA
 * call; no allocation, no synchronisation, graph-capturable: two memsets and three launches for K > 0, one memset and one launch
 * for K = 0. */
#define UC_BDD_BAD_CHARS 1 /* a char outside '0' .. 'o', a count of more than 7 chars, or a string that ends inside a count */
#define UC_BDD_BAD_RUNS 2  /* a negative count, or counts whose sum is not H * W */
#define UC_BDD_BAD_INDEX 4 /* offsets[j] > offsets[j+1], an offset outside [0, n_chars], or a rank outside [0, k[b]) */
UC_API long uc_bdd_bitmask_workspace_bytes(int B, const int* k, const int* H, const int* W, long n_chars);
UC_API int uc_bdd_bitmask_batched(int B, const int* k, const int* H, const int* W, const long* out_offsets, const char* chars, long n_chars,
                                  const long long* offsets, const uint32_t* colors, const int* ranks, void* workspace, long workspace_bytes,
                                  uint8_t* out, long out_bytes, int* status, void* stream);

#ifdef __cplusplus
}
#endif
#endif
