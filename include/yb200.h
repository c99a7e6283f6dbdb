/* yb200 -- C ABI of the H100 (sm_90a) YOLOX hot path.
 *
 * The reference (lucasjinreal/yolov7_d2) has no FFI of its own: every entry point below replaces a
 * PyTorch / torchvision call the reference makes on its hot path (file:line cited per function, paths
 * relative to the reference tree).  All pointers are DEVICE pointers unless stated otherwise, all tensors
 * are caller-allocated, every call is asynchronous on `stream` (a cudaStream_t passed as void*), performs no
 * host synchronisation and returns 0 on success or a negative yb200_status.  No global state except a
 * lazily resolved driver entry point (cuTensorMapEncodeTiled) and the per-device SM count.
 *
 * Activation layout: NHWC bf16 with a channel pitch, so that channel slices of a concat buffer are views:
 *   element (n,y,x,c) of a view = ptr[((n*h + y)*w + x)*c_pitch + c_off + c]
 */
#ifndef YB200_H_
#define YB200_H_
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define YB200_VERSION 100

typedef enum {
  YB200_OK = 0,
  YB200_ERR_INVALID = -1,     /* bad argument (null pointer, negative size, misaligned pitch) */
  YB200_ERR_UNSUPPORTED = -2, /* shape outside what the kernels implement */
  YB200_ERR_CUDA = -3,        /* a CUDA runtime / driver call failed; see yb200_last_error() */
} yb200_status;

typedef struct {
  void* ptr;        /* base of the underlying NHWC bf16 buffer (16-byte aligned) */
  int32_t n, h, w;  /* logical extents */
  int32_t c;        /* channels of this view (multiple of 8) */
  int32_t c_pitch;  /* channels of the underlying buffer (multiple of 8) */
  int32_t c_off;    /* first channel of the view inside the buffer (multiple of 8) */
} yb200_act;

int yb200_version(void);
const char* yb200_last_error(void);

/* ---- weights ------------------------------------------------------------------------------------- */
/* nn.Conv2d.weight (fp32 OIHW, wrappers.py:67-75) -> the two bf16 GEMM operands used by the kernels:
 *   w_fwd  [cout_pad][k*k][cin_pad]  (forward / weight-gradient order),  zero padded
 *   w_dgrad[cin_pad][k*k][cout_pad]  (data-gradient order); may be NULL.                                 */
int yb200_pack_conv_weight(const float* w_oihw, int cout, int cin, int ksize, int cout_pad, int cin_pad,
                           void* w_fwd, void* w_dgrad, void* stream);

/* ---- convolution (implicit GEMM on wgmma) -------------------------------------------------------- */
/* z = conv2d(x, w) without bias, padding (k-1)/2 -- BaseConv.conv, wrappers.py:67-80.
 * ksize in {1,3}, stride in {1,2} (stride 2 only with ksize 3).  z is the pre-BatchNorm output, stored as **fp16**
 * (same 2-byte NHWC view; BatchNorm's mean subtraction makes this tensor the precision-critical one).
 * If stat_sum/stat_sqsum are non-NULL the per-channel sum and sum of squares of the *stored* z are
 * accumulated into them (fp64, must be zeroed by the caller) -- the batch statistics nn.BatchNorm2d
 * (wrappers.py:76) computes in training mode.                                                          */
int yb200_conv2d_fwd(const yb200_act* x, const void* w_fwd, const yb200_act* z, int ksize, int stride,
                     double* stat_sum, double* stat_sqsum, void* stream);

/* Eval-mode BaseConv in one kernel: out = SiLU(conv2d(x, w)*scale + shift) [+ residual], bf16 -- nn.Conv2d + nn.BatchNorm2d
 * (running statistics) + nn.SiLU of wrappers.py:60-83 with the BatchNorm folded as in utils/checkpoint.py:11-43
 * (scale / shift from yb200_bn_eval_affine); the Bottleneck shortcut (wrappers.py:119-123) is added after the activation. */
int yb200_conv2d_bn_silu_fwd(const yb200_act* x, const void* w_fwd, const float* scale, const float* shift,
                             const yb200_act* residual, const yb200_act* out, int ksize, int stride, void* stream);

/* yb200_conv2d_fwd on a PIXEL-GROUPED view: when g horizontally adjacent pixels are viewed as one pixel of g*C channels (same memory), a
 * convolution becomes a convolution of the grouped tensors with an expanded weight matrix; output column k is channel k % stat_fold of one of
 * the g pixels, and the BatchNorm sums accumulate per channel.  For ksize 3 the weights MUST be such an expansion: the kernel skips the products of
 * the left / right neighbour group that the expansion makes zero (all but its last / first pixel).  Used for the stem (12 -> 32 channels at 320x320: 32-byte pixel rows are bound by
 * the TMA row rate; grouped by 4 they are 128-byte rows), `BaseConv` of `backbone.stem.conv` (darknetx.py:117, wrappers.py:60-80).            */
int yb200_conv2d_fwd_fold(const yb200_act* x, const void* w_fwd, const yb200_act* z, int ksize, int stride,
                          double* stat_sum, double* stat_sqsum, int stat_fold, void* stream);

/* out[n, a_off + y*w + x, c_off + c] = conv1x1(x, w)[n,y,x,c] + bias[c] in fp32 -- the prediction convs
 * yolox_head.py:103-129 fused with the cat/flatten/permute of yolox_head.py:175,238-244.
 * out is [n][a_total][c_total] fp32.                                                                    */
int yb200_conv1x1_bias_f32(const yb200_act* x, const void* w_fwd, const float* bias, int cout, float* out,
                           int a_total, int a_off, int c_total, int c_off, void* stream);

/* dx = conv_transpose(dz, w) [+ addend] -- autograd of the convolution w.r.t. its input.  dx/addend have the
 * input's shape, dz the output's.  addend may be NULL.                                                   */
int yb200_conv2d_dgrad(const yb200_act* dz, const void* w_dgrad, const yb200_act* dx, const yb200_act* addend,
                       int ksize, int stride, void* stream);

/* grad_oihw (+)= d loss / d weight, fp32 [cout][cin_real][k][k] -- autograd of the convolution w.r.t. its weight.
 * workspace: at least yb200_conv2d_wgrad_workspace() bytes.                                              */
int64_t yb200_conv2d_wgrad_workspace(const yb200_act* x, const yb200_act* dz, int ksize, int stride);
int yb200_conv2d_wgrad(const yb200_act* x, const yb200_act* dz, int ksize, int stride, int cin_real,
                       float* grad_oihw, int accumulate, void* workspace, int64_t workspace_bytes, void* stream);
/* The same for the PIXEL-GROUPED stem (x, dz = the grouped views of yb200_conv2d_fwd_fold, `group` pixels per group): grad_oihw is the gradient of
 * the EXPANDED weight matrix, valid at the positions the expansion fills (the caller folds them onto the [cout, cin, 3, 3] parameter); positions
 * that the expansion leaves zero are not computed (side taps multiply one neighbour pixel instead of the whole group).                      */
int yb200_conv2d_wgrad_grouped(const yb200_act* x, const yb200_act* dz, int ksize, int stride, int cin_real, int group,
                               float* grad_oihw, int accumulate, void* workspace, int64_t workspace_bytes, void* stream);

/* ---- preprocessing ------------------------------------------------------------------------------- */
/* uint8 NCHW images -> Focus (space-to-depth) NHWC bf16 [n, h/2, w/2, 16]: channel = patch*3 + rgb with patch order
 * (top-left, bottom-left, top-right, bottom-right) as wrappers.py:210-220, channels 12..15 zero.  No mean/std
 * normalisation (yolox.py:98).  hw_valid (device int32 [n][2], may be NULL) gives each image's true (h, w); pixels
 * beyond it read as pad_value = MODEL.PADDED_VALUE 114 (yolox.py:100-101, detectron2 ImageList.from_tensors).   */
int yb200_preprocess_focus(const uint8_t* images_nchw, int n, int h, int w, const int32_t* hw_valid, float pad_value,
                           const yb200_act* out, void* stream);

/* ---- BatchNorm + SiLU (nn.BatchNorm2d + nn.SiLU of BaseConv, wrappers.py:76-80; eps/momentum yolox.py:85-90) ---- */
/* Training statistics -> per-channel affine: scale = gamma*invstd, shift = beta - mean*scale (biased variance);
 * updates running_mean / running_var (unbiased variance, momentum) and num_batches_tracked in place when given;
 * zeroes stat_sum / stat_sqsum for the next step.                                                          */
int yb200_bn_finalize(double* stat_sum, double* stat_sqsum, int c, int64_t count, const float* gamma, const float* beta,
                      float eps, float momentum, float* running_mean, float* running_var, int64_t* num_batches_tracked,
                      float* scale, float* shift, float* save_mean, float* save_invstd, void* stream);
/* Eval mode: scale/shift from running statistics (the folding of utils/checkpoint.py:11-43 as an epilogue).   */
int yb200_bn_eval_affine(int c, const float* gamma, const float* beta, const float* running_mean,
                         const float* running_var, float eps, float* scale, float* shift, void* stream);
/* z is the fp16 tensor written by yb200_conv2d_fwd; every other activation / gradient view is bf16.
 * out = SiLU(z*scale + shift) [+ residual]  (Bottleneck shortcut, wrappers.py:119-123); when out_up2x is given the
 * result is also written nearest-upsampled x2 into that view (nn.Upsample + torch.cat of yolo_pafpn.py:96-102). */
int yb200_bn_apply_silu(const yb200_act* z, const float* scale, const float* shift, const yb200_act* residual,
                        const yb200_act* out, const yb200_act* out_up2x, void* stream);
/* yb200_bn_finalize + yb200_bn_apply_silu in ONE launch (training): every block derives scale / shift of its channels from the batch
 * sums, block 0 publishes scale / shift / save_mean / save_invstd (read by the backward pass) and updates the running statistics.
 * All pointers are per-channel arrays of this view's channels.  stat_sum / stat_sqsum are NOT cleared (clear them once per step).      */
int yb200_bn_train_apply_silu(const yb200_act* z, const double* stat_sum, const double* stat_sqsum, int64_t count,
                              const float* gamma, const float* beta, float eps, float momentum, float* running_mean,
                              float* running_var, float* scale, float* shift, float* save_mean, float* save_invstd,
                              const yb200_act* residual, const yb200_act* out, const yb200_act* out_up2x, void* stream);
/* Backward of SiLU(BN(z)) in training mode.  The incoming gradient is da [+ da2] [+ 2x2 sum-pool of da_up2x]
 * (fan-out of the activation / backward of the upsample).  Writes dz (bf16) and dgamma / dbeta (fp32, optionally
 * accumulated).  acc_dgamma / acc_dbeta: fp64 scratch [c], must be zero on entry, are zero on exit.          */
int yb200_bn_silu_bwd(const yb200_act* z, const yb200_act* da, const yb200_act* da2, const yb200_act* da_up2x,
                      const float* scale, const float* shift, const float* save_mean, const float* save_invstd,
                      double* acc_dgamma, double* acc_dbeta, const yb200_act* dz, float* dgamma, float* dbeta,
                      int accumulate, void* stream);

/* yb200_bn_silu_bwd with dgamma == dbeta == NULL leaves its sums in the fp64 accumulators; this call converts the accumulators of a
 * run of c channels (several layers) in one launch: grad_base[gamma_off[i]] (+)= dgamma_i, grad_base[beta_off[i]] (+)= dbeta_i, accumulators
 * zeroed.  Replaces the tail of torch's batch_norm backward for every BaseConv of a plan (wrappers.py:60-80).                        */
int yb200_bn_param_grads(double* acc_dgamma, double* acc_dbeta, int c, const int32_t* gamma_off, const int32_t* beta_off,
                         float* grad_base, int accumulate, void* stream);

/* ---- SPP / concat helpers ------------------------------------------------------------------------ */
/* nn.MaxPool2d(k, 1, k//2) for k = 5, 9, 13 written into three channel slices (SPPBottleneck, wrappers.py:150-160).
 * argmax (may be NULL): uint8 [3][n][h][w][c] window offsets for the backward.                                */
int yb200_spp_pool(const yb200_act* x, const yb200_act* o5, const yb200_act* o9, const yb200_act* o13, uint8_t* argmax,
                   void* stream);
/* dx = d0 + maxpool-backward(d5, d9, d13);  scratch: fp32 [n*h*w*c].
 * Bit-reproducible only on the shared-memory path (c % 16 == 0 and h*w*16*7 B <= 200 KiB, i.e. maps up to 42x42 for a square map): it adds
 * the gradients routed to each input in a fixed order.  Other shapes scatter them with fp32 atomics into `scratch`, in an order that can
 * change from run to run, so the last bits of dx can too.                                                         */
int yb200_spp_pool_bwd(const yb200_act* d0, const yb200_act* d5, const yb200_act* d9, const yb200_act* d13,
                       const uint8_t* argmax, float* scratch, const yb200_act* dx, void* stream);
int yb200_copy_view(const yb200_act* src, const yb200_act* dst, void* stream);

/* ---- YOLOX head tail: decode, SimOTA, losses ----------------------------------------------------- */
/* level_hw_stride: HOST int32 [num_levels][3] = (h, w, stride) of each FPN level, anchors ordered level by level,
 * row-major (yolox_head.py:226-245).  outputs: [batch][num_anchors][5+C] fp32 = (x, y, w, h, obj, cls...).     */
/* In place: xy = (xy + grid)*stride, wh = exp(wh)*stride (yolox_head.py:238-244); eval_mode also applies sigmoid to
 * obj / cls (yolox_head.py:209-211, 247-272).                                                                  */
int yb200_yolox_decode(float* outputs, int batch, int num_anchors, int channels, const int32_t* level_hw_stride,
                       int num_levels, int eval_mode, void* stream);
/* Training decode that also keeps the RAW regression outputs: raw_reg [batch][num_anchors][4] fp32 (16-byte aligned) = `origin_preds` of the
 * L1 branch (`use_l1`, yolox_head.py:186-195).                                                                                           */
int yb200_yolox_decode_keep_raw(float* outputs, int batch, int num_anchors, int channels, const int32_t* level_hw_stride,
                                int num_levels, float* raw_reg, void* stream);
/* SimOTA dynamic-k assignment for the whole batch (get_assignments + get_in_boxes_info + dynamic_k_matching,
 * yolox_head.py:450-669) on DECODED outputs and labels [batch][max_gt][5] = (cls, cx, cy, w, h), zero padded.
 * Per anchor: fg_mask (u8), matched_gt (-1 when background), matched_iou, matched_cls; per image num_gt / num_fg;
 * totals[0] = number of foreground anchors in the batch, totals[1] = number of gts.                            */
int64_t yb200_simota_workspace(int batch, int num_anchors);
int yb200_simota_assign(const float* outputs, const float* labels, int batch, int num_anchors, int channels, int max_gt,
                        const int32_t* level_hw_stride, int num_levels, void* workspace, int32_t* num_gt,
                        uint8_t* fg_mask, int32_t* matched_gt, float* matched_iou, int32_t* matched_cls,
                        int32_t* num_fg_img, int32_t* totals, void* stream);
/* Losses of get_losses (yolox_head.py:412-441) and/or their gradient w.r.t. the RAW (pre-decode) head outputs.
 *   losses6 (device float[6], may be NULL): total, 5*iou, obj, cls, l1 (= 0), num_fg/num_gt.
 *   weights3 (device float[3], NULL = no gradient): d objective / d (loss_iou, loss_obj, loss_cls)  (5, 1, 1 for `total`).
 *   d_cls[l] / d_regobj[l] (HOST arrays of device pointers, one per level): bf16 NHWC [batch][h][w][C] / [..][16]
 *   (reg 0-3, obj 4, zero padding) -- the dz tensors of the prediction convs.  d_dense: optional fp32 [batch][A][5+C].
 *   bias_acc: optional fp64 [num_levels][5+C] accumulators (zeroed by the caller) of the summed gradients.
 *   loss_acc3: fp64 scratch [3], zero on entry and exit.                                                        */
int yb200_yolox_loss(const float* outputs, const float* labels, int batch, int num_anchors, int channels, int max_gt,
                     const int32_t* level_hw_stride, int num_levels, const uint8_t* fg_mask, const int32_t* matched_gt,
                     const float* matched_iou, const int32_t* matched_cls, const int32_t* totals, const float* weights3,
                     double* loss_acc3, float* losses6, void* const* d_cls, void* const* d_regobj, float* d_dense,
                     double* bias_acc, void* stream);
/* The same with the L1 branch (`use_l1`, yolox_head.py:389-429, 443-448): loss_l1 = sum |raw_reg[fg] - l1_target| / num_fg with
 * l1_target = (gt_xy / stride - grid, log(gt_wh / stride + 1e-8)); total = 5*iou + obj + cls + l1, losses6[4] = l1; weights4[3] = d objective /
 * d loss_l1; the gradient sign(raw - target) * weight / num_fg is added to the regression gradients.  loss_acc4: fp64 scratch [4].          */
int yb200_yolox_loss_l1(const float* outputs, const float* raw_reg, const float* labels, int batch, int num_anchors, int channels,
                        int max_gt, const int32_t* level_hw_stride, int num_levels, const uint8_t* fg_mask,
                        const int32_t* matched_gt, const float* matched_iou, const int32_t* matched_cls, const int32_t* totals,
                        const float* weights4, double* loss_acc4, float* losses6, void* const* d_cls, void* const* d_regobj,
                        float* d_dense, double* bias_acc, void* stream);
/* bias gradients of reg_preds / obj_preds / cls_preds of one level out of bias_acc (which is re-zeroed).          */
int yb200_head_bias_grad(double* bias_acc, int num_levels, int channels, int level, float* grad_reg_bias4,
                         float* grad_obj_bias1, float* grad_cls_bias, int accumulate, void* stream);

/* All convolution weights of a plan repacked in ONE launch (same result as n calls of yb200_pack_conv_weight).  table / prefix live in
 * DEVICE memory and are built once per plan: prefix[i] = sum of cout_pad*k*k*cin_pad over layers < i, prefix[n] = total.               */
typedef struct yb200_pack_desc {
  const float* w_oihw;
  void* w_fwd;      /* [cout_pad][k*k][cin_pad] bf16, may be NULL */
  void* w_dgrad;    /* [cin_pad][k*k][cout_pad] bf16, may be NULL */
  int32_t cout, cin, ksize, cout_pad, cin_pad, reserved;
} yb200_pack_desc;
int yb200_pack_conv_weights_batched(const yb200_pack_desc* table_dev, const int64_t* prefix_dev, int n, int64_t total, void* stream);

/* ---- strict mode: fp32-grade forward on the same tensor-core kernels -------------------------------- */
/* SPLIT storage: an activation a is the sum of `planes` bf16 values a0 = bf16(a), a1 = bf16(a - a0) [, a2 = bf16(a - a0 - a1)]:
 * 16 significant bits with planes = 2, the full 24 bits of fp32 with planes = 3.  All planes live in one NHWC bf16 buffer,
 * lo_delta channels apart, so a yb200_act describes plane 0 and (view, lo_delta, planes) the value.  The convolution keeps
 * every partial product a_i * w_j with i + j < planes (3 / 6 taps per spatial tap of the SAME wgmma implicit GEMM, one
 * fp32 accumulator); the pre-BatchNorm output z is fp32 NHWC [n][h/stride][w/stride][z_pitch], channels [z_off, z_off+cout).
 * Used to check the reference's fp32 logits / losses to 1e-3 (tests/test_strict_gpu.py); forward only.
 * yb200_pack_conv_weight_split: fp32 OIHW -> [cout_pad][planes][k*k][cin_pad], `nn.Conv2d.weight` of wrappers.py:67-75.
 * yb200_conv2d_fwd_split: `BaseConv.conv` (wrappers.py:79).  yb200_conv1x1_bias_f32_split: the prediction convolutions
 * (yolox_head.py:103-129,175), same output geometry as yb200_conv1x1_bias_f32.                                           */
int yb200_pack_conv_weight_split(const float* w_oihw, int cout, int cin, int ksize, int cout_pad, int cin_pad, int planes,
                                 void* w_split, void* stream);
int yb200_conv2d_fwd_split(const yb200_act* x, int lo_delta, int planes, const void* w_split, int cout, int ksize,
                           int stride, float* z, int z_pitch, int z_off, void* stream);
int yb200_conv1x1_bias_f32_split(const yb200_act* x, int lo_delta, int planes, const void* w_split, const float* bias,
                                 int cout, float* out, int a_total, int a_off, int c_total, int c_off, void* stream);
/* BatchNorm batch statistics of an fp32 slice (sum, sum of squares in fp64; feed yb200_bn_finalize), then
 * out = SiLU(z*scale + shift) [+ residual] as split planes, optionally also 2x nearest-upsampled (wrappers.py:76-80,
 * 119-123; yolo_pafpn.py:96-102); SPP max-pools 5/9/13 on split values (wrappers.py:150-160).                        */
int yb200_strict_bn_stats(const float* z, int64_t npix, int z_pitch, int z_off, int c, double* stat_sum,
                          double* stat_sqsum, void* stream);
int yb200_strict_bn_apply_silu(const float* z, int z_pitch, int z_off, const float* scale, const float* shift,
                               const yb200_act* residual, int residual_lo, const yb200_act* out, int out_lo,
                               const yb200_act* out_up2x, int up_lo, int planes, void* stream);
int yb200_strict_spp_pool(const yb200_act* x, const yb200_act* o5, const yb200_act* o9, const yb200_act* o13,
                          int lo_delta, int planes, void* stream);

/* ---- post-processing ----------------------------------------------------------------------------- */
/* `postprocess` (boxes.py:171-210) for the whole batch: prediction [batch][A][5+C] = (cx, cy, w, h, obj, cls...) with
 * probabilities already applied.  Per image: class_conf / class_pred = max / first argmax over classes; candidates have
 * obj*class_conf >= conf_thre; per-class NMS (torchvision batched_nms, "vanilla" semantics: stable descending score
 * order, suppress when IoU > nms_thre on un-offset fp32 xyxy boxes); survivors ordered by descending score.
 * detections [batch][A][7] = (x1, y1, x2, y2, obj_conf, class_conf, class_pred), det_count[batch] rows are valid.
 * mutate_prediction != 0 also rewrites prediction[..., :4] to xyxy in place, as the reference does (boxes.py:177).     */
int64_t yb200_nms_workspace(int batch, int num_anchors);
int yb200_postprocess_nms(float* prediction, int batch, int num_anchors, int num_classes, float conf_thre, float nms_thre,
                          int mutate_prediction, void* workspace, float* detections, int32_t* det_count, void* stream);
/* Same, plus (both nullable): det_anchor [batch][A] = anchor index of every emitted row, and tie_count[batch] = number of
 * adjacent emitted rows with bit-identical scores.  Equal scores are emitted lower-anchor-first (the stable order of
 * torchvision's `nms`, i.e. the reference on CUDA and on CPU with <= 1000 candidates); the CPU `_batched_nms_vanilla`
 * path ends with an UNSTABLE torch.sort whose permutation of ties a caller can re-apply from det_anchor when
 * tie_count > 0 (yolov7_d2_b200.modeling.postprocess(tie_order="torch_cpu_sort")).                                      */
int yb200_postprocess_nms_indexed(float* prediction, int batch, int num_anchors, int num_classes, float conf_thre,
                                  float nms_thre, int mutate_prediction, void* workspace, float* detections,
                                  int32_t* det_count, int32_t* det_anchor, int32_t* tie_count, void* stream);

/* ---- box regression losses ----------------------------------------------------------------------- */
/* loss[i] and d loss[i] / d pred[i] for n matched (prediction, target) pairs of (cx, cy, w, h) boxes (device fp32 [n][4]).
 * mode 0: IOUloss "iou" = 1 - iou^2 (boxes.py:125-151, the YOLOX-s loss, yolox_head.py:134); 1: IOUloss "giou" (boxes.py:152-161);
 * 2 / 3 / 4: IOUlossV6 giou / diou / ciou with eps 1e-7 (boxes.py:666-752, YOLOv6 head).  dloss_dpred may be NULL.            */
int yb200_iou_loss(const float* pred_cxcywh, const float* target_cxcywh, int n, int mode, float* loss, float* dloss_dpred,
                   void* stream);

/* ---- parameter update on the flat fp32 buffers (SURVEY.md par.8f rank 1) -------------------------------------------------------
 * Per-parameter hyper-parameters come from a segment table in device memory: seg_begin[nseg] ascending element offsets
 * (seg_begin[0] == 0), seg_wd[nseg] weight decay, seg_lr_mult[nseg] learning-rate multiplier (NULL = 1): the param groups that
 * yolov7/optimizer/build.py:77-170 builds (norm / bias / embedding decay, bias_lr_factor, lr_multipliers_overwrite).
 * grad_scale multiplies every gradient first (1/world_size of the DDP mean); total_norm (device scalar from yb200_grad_norm, may be
 * NULL) with max_norm > 0 applies clip_grad_norm_ over the whole model (FullModelGradientClippingOptimizer, build.py:206-223).       */
int64_t yb200_grad_norm_workspace(void);
/* out_norm[0] = || grad * grad_scale ||_2, deterministic two-stage reduction (fp64 accumulation) */
int yb200_grad_norm(const float* grad, int64_t n, float grad_scale, void* workspace, float* out_norm, void* stream);
/* torch.optim.SGD.step (build.py:234-245): d = g + wd*p; buf = first_step ? d : momentum*buf + (1-dampening)*d;
 * d = nesterov ? d + momentum*buf : buf; p -= lr*d.  momentum_buf may be NULL when momentum == 0.                                   */
int yb200_sgd_step(float* param, const float* grad, float* momentum_buf, int64_t n, const int64_t* seg_begin, const float* seg_wd,
                   const float* seg_lr_mult, int nseg, float lr, float momentum, float dampening, int nesterov, int first_step,
                   float grad_scale, const float* total_norm, float max_norm, void* stream);
/* torch.optim.AdamW.step (build.py:248-256): p *= 1 - lr*wd; m, v moments; p -= lr/(1-b1^t) * m / (sqrt(v)/sqrt(1-b2^t) + eps); step t >= 1 */
int yb200_adamw_step(float* param, const float* grad, float* exp_avg, float* exp_avg_sq, int64_t n, const int64_t* seg_begin,
                     const float* seg_wd, const float* seg_lr_mult, int nseg, float lr, float beta1, float beta2, float eps, int step,
                     float grad_scale, const float* total_norm, float max_norm, void* stream);

/* ---- ConvNeXt block (SURVEY.md par.8a row C1: yolov7/modeling/backbone/convnext.py) ------------------------------------------------
 * The two Linear layers of the block and the 2x2 / 4x4 strided convolutions run on the implicit-GEMM kernels above with these
 * epilogues; everything else is in csrc/convnext.cu.  Linear weights [out][in] are packed with yb200_pack_conv_weight(ksize 1).      */
/* as yb200_pack_conv_weight with every output row scaled by cout_scale[co] first (layer scale gamma folded into pwconv2, convnext.py:54-56);
 * scaled_bias[co] = cout_scale[co] * bias[co] (both NULL or both given): the shift of the matching yb200_conv2d_affine_fwd call              */
int yb200_pack_conv_weight_scaled(const float* w_oihw, const float* cout_scale, const float* bias, int cout, int cin, int ksize, int cout_pad,
                                  int cin_pad, void* w_fwd, void* w_dgrad, float* scaled_bias, void* stream);
/* out = bf16(conv(x) * scale[c] + shift[c] [+ residual]); scale / shift may be NULL (1 / 0).  ksize/stride: 1/1, 3/1, 3/2 or 2/2 (no padding:
 * the downsample convolutions, convnext.py:86-91).  nn.Conv2d / nn.Linear with bias: shift = bias.                                      */
int yb200_conv2d_affine_fwd(const yb200_act* x, const void* w_fwd, const float* scale, const float* shift, const yb200_act* residual,
                            const yb200_act* out, int ksize, int stride, void* stream);
/* pwconv1 + GELU (convnext.py:52-53): u = bf16(x W^T + bias) -> u_out (may be NULL), h = bf16(GELU(u)) -> h_out (exact erf form)       */
int yb200_linear_gelu_fwd(const yb200_act* x, const void* w_fwd, const float* bias, const yb200_act* u_out, const yb200_act* h_out, void* stream);
/* du = bf16((dz W) * GELU'(u)) and, when bias_grad_sum != NULL, bias_grad_sum[c] += sum over pixels of the stored bf16 du[.., c] (fp32 per
 * CTA, then fp64 atomics into the caller's accumulator):
 * the data gradient of pwconv2 fused with the GELU backward and the bias gradient of pwconv1.                                            */
int yb200_linear_dgrad_gelu(const yb200_act* dz, const void* w_dgrad, const yb200_act* u, const yb200_act* du, double* bias_grad_sum,
                            void* stream);
/* depthwise 7x7, stride 1, zero padding 3 (convnext.py:41,49): out = dwconv(x; w) [+ bias] [+ addend].  w_c49: fp32 [C][7][7] (the
 * nn.Conv2d(groups=C) weight [C][1][7][7]).  flip != 0 correlates with the flipped kernel = the data gradient (addend: the residual branch). */
int yb200_dwconv7(const yb200_act* x, const float* w_c49, const float* bias, const yb200_act* addend, const yb200_act* out, int flip,
                  void* stream);
int64_t yb200_dwconv7_wgrad_workspace(const yb200_act* x);
/* grad_w_c49[c][ky][kx] = sum dy[p][c] x[p + (ky-3, kx-3)][c]; grad_bias[c] = sum dy[p][c] (may be NULL); fixed summation order          */
int yb200_dwconv7_wgrad(const yb200_act* x, const yb200_act* dy, float* grad_w_c49, float* grad_bias, int accumulate, void* workspace,
                        void* stream);
/* LayerNorm over the channel dimension of every pixel (convnext.py:196-206, both data formats; biased variance, eps inside the sqrt).
 * stats_mean_rstd: fp32 [pixels][2], may be NULL in forward-only use.                                                                    */
int yb200_layernorm_fwd(const yb200_act* x, const float* gamma, const float* beta, float eps, const yb200_act* y, float* stats_mean_rstd,
                        void* stream);
int64_t yb200_layernorm_bwd_workspace(const yb200_act* x);
/* dx = LayerNorm-backward(dy) [+ addend]; grad_gamma / grad_beta fp32 [C], fixed summation order                                         */
int yb200_layernorm_bwd(const yb200_act* dy, const yb200_act* x, const float* stats_mean_rstd, const float* gamma, const yb200_act* addend,
                        const yb200_act* dx, float* grad_gamma, float* grad_beta, int accumulate, void* workspace, void* stream);
int64_t yb200_colsum_workspace(const yb200_act* x);
/* out[c] = scale * sum over pixels of x[.., c] (bias gradients), fixed summation order                                                    */
int yb200_colsum(const yb200_act* x, float scale, float* out, int accumulate, void* workspace, void* stream);
/* Layer scale gamma (convnext.py:44-45,55-56) folded into pwconv2: given raw_wgrad = dOut^T h (weight gradient w.r.t. the UNscaled output
 * gradient, [C][hidden]) and gout_colsum[c] = sum of dOut:  grad_w2 = gamma[c] * raw, grad_gamma[c] = <w2[c], raw[c]> + b2[c] * colsum[c],
 * grad_b2[c] = gamma[c] * colsum[c].  raw_wgrad may alias grad_w2.                                                                         */
int yb200_layer_scale_grad(const float* raw_wgrad, const float* w2, const float* b2, const float* gamma, const float* gout_colsum, int channels,
                           int hidden, float* grad_w2, float* grad_gamma, float* grad_b2, int accumulate, void* stream);
/* stem input (convnext.py:81-84): uint8 (is_f32 = 0) or fp32 NCHW image -> [N][H/4][W/4][48] bf16 patches, channel = c*16 + kh*4 + kw (the OIHW flattening of
 * the 4x4 stride-4 stem weight), so the stem is a K = 48 GEMM (yb200_conv2d_affine_fwd, ksize 1).                                          */
int yb200_patchify4(const void* images_nchw, int is_f32, int n, int h, int w, const yb200_act* out, void* stream);
/* dst[i] = (accumulate ? dst[i] : 0) + (float)src[i]; src[i] = 0 when zero_src (fp64 accumulators of the GEMM epilogues -> fp32 gradients) */
int yb200_f64_to_f32(double* src, int n, float* dst, int accumulate, int zero_src, void* stream);

/* ---- DETR transformer attention (SURVEY.md par.8a row T1: yolov7/modeling/backbone/detr_backbone.py:140,157-161,200-236) -------------
 * The core of nn.MultiheadAttention between in_proj and out_proj, head dimension 32:
 *   out[b, i, h, :] = softmax_j(scale * <q[b,i,h,:], k[b,j,h,:]> + (key_padding_mask[b,j] ? -inf : 0)) . v[b,j,h,:]
 * q / out: views [B][1][Lq][heads*32], k / v: [B][1][Lk][heads*32] (token-major, head h = channels [32h, 32h+32) of the view; q, k, v may be
 * slices of one packed in_proj output).  key_padding_mask: uint8 [B][Lk], 1 = ignore, or NULL.  scale: head_dim^-0.5 in the reference.
 * lse (fp32 [B][heads][Lq], may be NULL) receives log sum_j exp(scaled masked score), the statistic a backward pass needs.
 * A query whose keys are all masked yields zeros (torch yields NaN).  in_proj / out_proj / FFN are yb200_conv2d_affine_fwd calls.          */
int yb200_attention_fwd(const yb200_act* q, const yb200_act* k, const yb200_act* v, const uint8_t* key_padding_mask, float scale,
                        const yb200_act* out, float* lse, void* stream);
/* Linear + ReLU of the transformer FFN (detr_backbone.py:167, 239): h = bf16(max(x W^T + bias, 0))                                        */
int yb200_linear_relu_fwd(const yb200_act* x, const void* w_fwd, const float* bias, const yb200_act* h_out, void* stream);
/* du = bf16(h > 0 ? dz W : 0) (h > 0: positive and non-zero; -0 and negatives mask) and optionally bias_grad_sum[c] += column sums of the
 * STORED bf16 du (summed in fp32 inside each CTA, added to the caller's fp64 accumulator with one atomic per CTA and column: the order of
 * those additions is not fixed): data gradient of linear2 fused with the ReLU backward and the bias gradient of linear1               */
int yb200_linear_dgrad_relu(const yb200_act* dz, const void* w_dgrad, const yb200_act* h, const yb200_act* du, double* bias_grad_sum, void* stream);
/* out = a + b (bf16 views of equal shape): tensor + positional embedding (detr_backbone.py:154-155, 218-219)                                */
int yb200_add(const yb200_act* a, const yb200_act* b, const yb200_act* out, void* stream);

/* ---- SparseInst IAM decoder forward (SURVEY.md par.8a row S1: yolov7/modeling/transcoders/decoder_sparseinst.py:27-169) ------------------
 * 3x3 convolution + bias + ReLU (`_make_stack_3x3_convs` :18-24); ksize / stride as yb200_conv2d_affine_fwd                                 */
int yb200_conv2d_relu_fwd(const yb200_act* x, const void* w_fwd, const float* bias, const yb200_act* out, int ksize, int stride, void* stream);
/* 1x1 convolution with fp32 NCHW output [N][cout][H][W] (+ bias, may be NULL): with per-image weights = pred_kernel[b] this is
 * `torch.bmm(pred_kernel, mask_features.view(B, C, HW))` (:143-146); cout <= 128                                                            */
int yb200_conv1x1_nchw_f32(const yb200_act* x, const void* w_fwd, const float* bias, int cout, float* out_nchw, void* stream);
/* The same for a whole batch with ONE WEIGHT MATRIX PER IMAGE (w_fwd: [x->n][cout][x->c] bf16 = the batch's predicted kernels): the batched
 * `torch.bmm` of :143-146 in one launch.  Accepted when the 128-pixel tile choose_tile picks for (n, h, w) holds one image (tile width x
 * height = 128: e.g. 80x80, 64x64, 72x96, any map at n = 1, and maps like 1x65 whose tiles overhang the image); otherwise (e.g. 40x40 or
 * 60x80 at n = 2, two images per tile) YB200_ERR_UNSUPPORTED, the output untouched: call yb200_conv1x1_nchw_f32 per image.                */
int yb200_conv1x1_nchw_f32_batched(const yb200_act* x, const void* w_fwd, int cout, float* out_nchw, void* stream);
/* F.interpolate(x, scale_factor=2, mode="bilinear", align_corners=False) on fp32 planes [planes][h][w] -> [planes][2h][2w]: the mask logits
 * (:148-153)                                                                                                                                  */
int yb200_upsample_bilinear2x_f32(const float* in, float* out, int64_t planes, int h, int w, void* stream);
/* out = sigmoid(x): instance activation maps (:67)                                                                                           */
int yb200_sigmoid(const yb200_act* x, const yb200_act* out, void* stream);
/* inst[r][c] = raw[r][c] / max(normalizer[r], 1e-6) -> bf16 [1][1][rows][cols] view (:75-76).  raw = iam_prob^T features of one image is
 * yb200_conv2d_wgrad(x = features, dz = iam_prob, ksize 1) (the pixel contraction of :74), normalizer = yb200_colsum(iam_prob).              */
int yb200_iam_normalize(const float* raw, const float* normalizer, int rows, int cols, const yb200_act* out, void* stream);

/* ---- SparseInst IAM decoder backward (decoder_sparseinst.py:27-250) -------------------------------------------------------------------------
 * Fixed summation order and no atomics in every call below: bit-reproducible.
 * yb200_conv2d_dgrad_relu: dx = bf16((h > 0 ? dz W : 0) + addend) -- the data gradient of a convolution whose input h is a ReLU output
 *   (`_make_stack_3x3_convs` :18-24), masked before addend (may be NULL) is added: pass an addend that is already masked.  ksize 1 or 3,
 *   stride 1; h and dx have the same shape and channel pitch.
 * yb200_upsample_bilinear2x_bwd_f32: the adjoint of yb200_upsample_bilinear2x_f32 (:148-153): dout fp32 [dx->n][maps][2h][2w] -> dx bf16
 *   [n][h][w][c] view (maps <= c; channels >= maps written as 0), the NHWC operand of the mask GEMM's gradients.  Each element sums its
 *   (up to 16) up-sampled contributions.
 * yb200_iam_normalize_bwd: backward of yb200_iam_normalize for a batch (:75-76, group :225-235).  g: bf16 [n][1][R][(rows / rows_per_group) *
 *   cols] view, the gradient of inst; raw row r reads row r % rows_per_group, columns from (r / rows_per_group) * cols (the grouped decoder's
 *   reshape(B, G, N, C).transpose(1, 2); rows of r % rows_per_group >= R read as 0).  raw fp32 [n][rows][cols], normalizer fp32 [n][rows].
 *   Writes d raw = g / max(normalizer, 1e-6) as bf16 draw [n][rows][cols] and draw_t [n][cols][rows], and dnorm fp32 [n][rows] =
 *   -sum_c draw raw / max(normalizer, 1e-6) (= -sum_c g raw / max(normalizer, 1e-6)^2, summed from the stored bf16 d raw so that the
 *   normalisation's invariance to a common scale of the probabilities holds for the operands the aggregation backward reads; 0 where
 *   normalizer < 1e-6, the clamp).  cols <= 2048.
 * yb200_sigmoid_bwd: dx = dy * sigmoid'(x) with sigmoid' recomputed in fp32 from x (:67), the channels regrouped: dx channel
 *   k * group_out + i = (i < group_in ? dy * sigmoid'(x) at channel k * group_in + i : 0).  dy and x have the same shape; dx the same
 *   pixels and dy->c / group_in * group_out channels; group_in, group_out multiples of 8.                                                       */
int yb200_conv2d_dgrad_relu(const yb200_act* dz, const void* w_dgrad, const yb200_act* h, const yb200_act* dx, const yb200_act* addend, int ksize,
                            int stride, void* stream);
int yb200_upsample_bilinear2x_bwd_f32(const float* dout, int maps, const yb200_act* dx, void* stream);
int yb200_iam_normalize_bwd(const yb200_act* g, const float* raw, const float* normalizer, int rows, int cols, int rows_per_group, void* draw,
                            void* draw_t, float* dnorm, void* stream);
int yb200_sigmoid_bwd(const yb200_act* dy, const yb200_act* x, const yb200_act* dx, int group_in, int group_out, void* stream);
/* Backward of yb200_attention_fwd: given out, its gradient dout and the saved lse, dq / dk / dv (bf16 views shaped like q / k / k; they may be
 * slices of one packed buffer).  P is recomputed from lse; two kernels (per key tile: dK, dV; per query tile: dQ), accumulation in registers,
 * no atomics.  workspace: yb200_attention_bwd_workspace(q) bytes (D = <dout, out> per query row and head).                                     */
int64_t yb200_attention_bwd_workspace(const yb200_act* q);
int yb200_attention_bwd(const yb200_act* q, const yb200_act* k, const yb200_act* v, const yb200_act* out, const yb200_act* dout,
                        const uint8_t* key_padding_mask, float scale, const float* lse, const yb200_act* dq, const yb200_act* dk,
                        const yb200_act* dv, void* workspace, void* stream);

/* Dropout of the transformer layers (detr_backbone.py:132-152, 200-214).  The masks are a counter-based hash of (seed, element index) evaluated
 * inside the kernels -- keep(element) with probability 1 - p_drop, kept values scaled by 1 / (1 - p_drop) -- so the backward calls regenerate the
 * mask of the forward from the same seed; p_drop = 0 is exactly the dropout-free kernel.  (Not torch's Philox stream: same distribution, different
 * bits; oracle/detr_oracle.py restates the hash for the parity tests.)
 *   yb200_attention_fwd_dropout / _bwd_dropout: nn.MultiheadAttention(dropout = p) -- the mask multiplies the softmax probabilities (index: image, head,
 *     query, key); lse stays the log-sum-exp of the undropped scores.
 *   yb200_dropout: out = residual + x * mask(seed) / (1 - p) * extra_scale on [B][1][L][C] bf16 views (index: logical element ((b L + l) C + c));
 *     residual may be NULL; the backward of nn.Dropout is the same call on the gradient.                                                          */
int yb200_attention_fwd_dropout(const yb200_act* q, const yb200_act* k, const yb200_act* v, const uint8_t* key_padding_mask, float scale,
                                const yb200_act* out, float* lse, float p_drop, uint32_t seed, void* stream);
int yb200_attention_bwd_dropout(const yb200_act* q, const yb200_act* k, const yb200_act* v, const yb200_act* out, const yb200_act* dout,
                                const uint8_t* key_padding_mask, float scale, const float* lse, const yb200_act* dq, const yb200_act* dk,
                                const yb200_act* dv, void* workspace, float p_drop, uint32_t seed, void* stream);
int yb200_dropout(const yb200_act* x, const yb200_act* residual, const yb200_act* out, float p_drop, uint32_t seed, float extra_scale,
                  void* stream);

/* ---- mosaic / random_perspective / mixup of the YOLOX training mapper ------------------------------------------------------------------------ */
/* MyDatasetMapper2.__call__ (yolov7/data/dataset_mapper.py:477-611, mixup :686-767) with random_perspective (data_augment.py:31-102): the host
 * (yolov7_d2_b200/augment.py) makes the random draws and computes the boxes; these two calls render the pixels of a whole batch.  One descriptor
 * per sample in DEVICE memory; the sources are HWC uint8 (BGR) images packed in one buffer, the outputs CHW uint8 (the reference's
 * `img.transpose(2, 0, 1)`, :637-638) packed in another.  Bit-reproducible (no atomics), no host synchronisation.
 *   yb200_mosaic_warp: mode 1 -- the four tiles cv2.resize'd (INTER_LINEAR) into the 2h x 2w canvas of 114 (:529-566), then
 *     cv2.warpAffine(canvas, M[:2], (out_w, out_h), borderValue 114) with minv = the inverse of M (data_augment.py:62-74); mode 0 -- a sample
 *     without mosaic (pool still filling, or mosaic_flag 0): source 0 copied HWC -> CHW.
 *   yb200_mosaic_mixup: for samples with mode 1 and mix 1, the mixup image (:701-739: resize of source 4 into the in_h x in_w canvas of 114,
 *     float64 resize to jit_h x jit_w, optional horizontal flip, zero padding, crop at (y_off, x_off)) blended into the output in place,
 *     (a + b) / 2 truncated (:763-767).  Run it after yb200_mosaic_warp on the same stream.
 * max_h / max_w bound the output sizes of the batch (they size the grid).                                                                      */
typedef struct yb200_mosaic_desc {
  int64_t src_off[5];          /* byte offsets of the sources in `src`: tiles 0-3 (top left, top right, bottom left, bottom right), mixup 4 */
  int64_t out_off;             /* byte offset of the sample's [3][out_h][out_w] output in `out` */
  double minv[6];              /* inverse of the 2x3 affine map: output pixel -> canvas pixel */
  int32_t src_h[5], src_w[5];
  int32_t tile_h[4], tile_w[4];  /* resized tile size: (int(h0 * s), int(w0 * s)), s = min(h / h0, w / w0) */
  int32_t rect[16];            /* per tile: canvas rectangle x1a, y1a, x2a, y2a */
  int32_t pad[8];              /* per tile: padw, padh (canvas position of the tile's pixel (0, 0)) */
  int32_t in_h, in_w;          /* mosaic size (h, w); the canvas is 2h x 2w */
  int32_t out_h, out_w;
  int32_t mode;                /* 0: copy source 0, 1: mosaic */
  int32_t mix;                 /* 1: blend the mixup image */
  int32_t mix_h, mix_w;        /* resized mixup source inside the in_h x in_w canvas */
  int32_t jit_h, jit_w;        /* jittered canvas size */
  int32_t flip, x_off, y_off, reserved;
} yb200_mosaic_desc;
int yb200_mosaic_warp(const yb200_mosaic_desc* table_dev, int n, const uint8_t* src, uint8_t* out, int max_h, int max_w, void* stream);
int yb200_mosaic_mixup(const yb200_mosaic_desc* table_dev, int n, const uint8_t* src, uint8_t* out, int max_h, int max_w, void* stream);

/* ---- DETR matching cost and SetCriterion (yolov7/utils/detr_utils.py:12-91, yolov7/modeling/meta_arch/detr.py:475-647) ----------------------
 * Every call covers all L decoder layers.  logits: fp32 [L][B][Q][K1] (K1 = num_classes + 1, the last class is "no object"), boxes: fp32
 * [L][B][Q][4] post-sigmoid (cx, cy, w, h).  The targets of the batch are packed: labels int32 [G], target_boxes fp32 [G][4] (cx, cy, w, h),
 * offsets int32 [B+1] (image b owns targets [offsets[b], offsets[b+1]), offsets[B] = G).  labels / target_boxes must not be NULL even when G = 0.
 *   yb200_detr_match_cost: HungarianMatcher's cost w_bbox * L1 + w_class * (-softmax[label]) + w_giou * (-GIoU) (detr_utils.py:65-86), only the
 *     per-image blocks: block (l, b) is [Q][G_b] row-major at cost + l*Q*G + Q*offsets[b].  cost has L*Q*G + 1 floats: the last one is an int32
 *     status word, bit 0 = a label outside [0, K1), bit 1 = a target box whose corners are out of order (generalized_box_iou's assert).
 *   yb200_detr_set_loss: match int32 [L][B][Q] = the matched target's index within its image, or -1.  out fp32 [L][5] = (loss_ce, loss_bbox,
 *     loss_giou, cardinality_error, class_error) of each layer, unweighted, as loss_labels / loss_boxes / loss_cardinality (detr.py:507-570)
 *     compute them; the cross entropy is weighted by eos_coef on the no-object class and normalised by its weight sum; num_boxes as detr.py:620-624.
 *   yb200_detr_set_loss_bwd: grad fp32 [L][3] = upstream gradients of (loss_ce, loss_bbox, loss_giou) per layer (device memory); writes
 *     dlogits [L][B][Q][K1] and dboxes [L][B][Q][4] (zero on unmatched queries).
 * Fixed summation order (bit-reproducible), no host synchronisation.                                                                            */
int yb200_detr_match_cost(const float* logits, const float* boxes, const int32_t* labels, const float* target_boxes, const int32_t* offsets, int L,
                          int B, int Q, int K1, int G, float w_class, float w_bbox, float w_giou, float* cost, void* stream);
int yb200_detr_set_loss(const float* logits, const float* boxes, const int32_t* match, const int32_t* labels, const float* target_boxes,
                        const int32_t* offsets, int L, int B, int Q, int K1, float eos_coef, float num_boxes, float* out, void* stream);
int yb200_detr_set_loss_bwd(const float* logits, const float* boxes, const int32_t* match, const int32_t* labels, const float* target_boxes,
                            const int32_t* offsets, int L, int B, int Q, int K1, float eos_coef, float num_boxes, const float* grad, float* dlogits,
                            float* dboxes, void* stream);

/* ---- SparseInst matcher and criterion (yolov7/modeling/loss/sparseinst_loss.py) --------------------------------------------------------------
 * pred_logits fp32 [B][N][K], pred_masks fp32 [B][N][H*W] (HW = H*W), pred_scores fp32 [B][N].  The targets of the batch are packed: labels int32
 * [G], offsets int32 [B+1] (image b owns targets [offsets[b], offsets[b+1]), offsets[B] = G), the resized masks tmasks fp32 [G][HW] and their
 * Σt² tsq [G] (yb200_sparseinst_target_masks).  labels / tmasks / tsq must not be NULL even when G = 0.  N <= 4096, B*N < 65536.
 *   yb200_sparseinst_target_masks: masks = the uint8 masks of the batch in one buffer; table int64 [G][3] = (byte offset, h, w) of each.  out
 *     [G][H][W] = the mask zero-padded to in_h x in_w (nested_masks_from_list, :320-322) and resized by F.interpolate(bilinear,
 *     align_corners=False) (:326-331) with ATen's index and weight formula; tsq[g] = Σ out[g]².  Every mask needs h <= in_h, w <= in_w.
 *   yb200_sparseinst_match_cost: SparseInstMatcher's C = dice^alpha * sigmoid(logit[label])^beta (:336-340), dice = 2 Σσ(m)t / (Σσ(m)² + Σt² +
 *     1e-4), only the per-image blocks: block b is [N][G_b] row-major at cost + N*offsets[b].  cost has N*G + 1 floats: the last one is an int32
 *     status word, bit 0 = a label outside [0, K), bit 1 = an image with more than N targets (its block is not written).
 *   yb200_sparseinst_set_loss: match int32 [B][N] = the matched target's index within its image, or -1; num_pairs = matched rows.  out fp32 [4]
 *     = (loss_ce, loss_objectness, loss_dice, loss_mask) weighted by (w_ce, w_obj, w_dice, w_mask), as loss_labels and
 *     loss_masks_with_iou_objectness (:89-184) compute them; the three mask terms are 0 when num_pairs = 0.  save fp32 [B][N][8]: per-row sums
 *     the backward reads.
 *   yb200_sparseinst_set_loss_bwd: grad fp32 [4] = upstream gradients of out (device memory); writes dlogits [B][N][K], dmasks [B][N][HW] (zero
 *     on unmatched rows) and dscores [B][N] (zero on unmatched rows).  The IoU target carries no gradient.
 * Fixed summation order (bit-reproducible), no host synchronisation.                                                                            */
int yb200_sparseinst_target_masks(const uint8_t* masks, const int64_t* table, int G, int in_h, int in_w, int H, int W, float* out, float* tsq,
                                  void* stream);
int yb200_sparseinst_match_cost(const float* logits, const float* masks, const int32_t* labels, const int32_t* offsets, const float* tmasks,
                                const float* tsq, int B, int N, int K, int HW, int G, float alpha, float beta, float* cost, void* stream);
int yb200_sparseinst_set_loss(const float* logits, const float* masks, const float* scores, const int32_t* match, const int32_t* labels,
                              const int32_t* offsets, const float* tmasks, const float* tsq, int B, int N, int K, int HW, int num_pairs, float w_ce,
                              float w_obj, float w_dice, float w_mask, float num_instances, float* save, float* out, void* stream);
int yb200_sparseinst_set_loss_bwd(const float* logits, const float* masks, const float* scores, const int32_t* match, const int32_t* labels,
                                  const int32_t* offsets, const float* tmasks, const float* tsq, const float* save, int B, int N, int K, int HW,
                                  int num_pairs, float w_ce, float w_obj, float w_dice, float w_mask, float num_instances, const float* grad,
                                  float* dlogits, float* dmasks, float* dscores, void* stream);

/* ---- SparseInst InstanceContextEncoder (yolov7/modeling/transcoders/encoder_sparseinst.py:18-127) -----------------------------------------
 * The non-GEMM steps of the encoder and their adjoints, on NHWC bf16 views (channel slices of the concat buffers).  The convolutions are
 * yb200_conv2d_affine_fwd / yb200_conv2d_relu_fwd, their gradients yb200_conv2d_dgrad[_relu], yb200_conv2d_wgrad and yb200_colsum.  Every sum
 * runs in fp32 in a fixed order, rounded to bf16 once; no atomics: bit-reproducible.
 *   yb200_avg_pool2d: MyAdaptiveAvgPool2d (:18-39), which is F.avg_pool2d with kernel = stride = (kh, kw) = (ceil(H/s), ceil(W/s)), floor
 *     mode, no padding: out [n][h/kh][w/kw][c] = window sum / (kh * kw).
 *   yb200_ppm_input_grad: the gradient of the PPM's input (:56-68): dx = dcat + sum over the stages i < nstages, in order, of the adjoint of
 *     the pool, dpooled[i] / (kh * kw) at every pixel of the window that covers it (pixels beyond the last full window get dcat only).
 *     dpooled: HOST array of nstages (<= 8) views, each [dx->n][dx->h / kh][dx->w / kw][dx->c]; kernel_hw: HOST int32 [nstages][2] = (kh, kw).
 *   yb200_resize_bilinear: F.interpolate(x, size=(out->h, out->w), mode="bilinear", align_corners=False) (:58-66, :121-125) with ATen's index
 *     arithmetic: scale = in / out, src = max(scale * (dst + 0.5) - 0.5, 0), i1 = i0 + (i0 < in - 1), fp32 weights.
 *   yb200_resize_bilinear_bwd: its adjoint, dx (the input's shape) = for every input pixel the weighted sum of the d out pixels whose taps
 *     reach it; h (may be NULL, dx's shape): dx = h > 0 ? sum : 0, the gradient of z in interpolate(relu(z)).
 *   yb200_upsample_nearest2x_add: the top-down path (:114-118), out = lat + F.interpolate(coarse, scale_factor=2, mode="nearest"); out may
 *     be lat.
 *   yb200_upsample_nearest2x_bwd: its adjoint, dx [n][h/2][w/2][c] = the 2x2 sums of dy; h (may be NULL, dx's shape): dx = h > 0 ? sum : 0. */
int yb200_avg_pool2d(const yb200_act* x, int kh, int kw, const yb200_act* out, void* stream);
int yb200_ppm_input_grad(const yb200_act* dcat, const yb200_act* dpooled, const int32_t* kernel_hw, int nstages, const yb200_act* dx, void* stream);
int yb200_resize_bilinear(const yb200_act* x, const yb200_act* out, void* stream);
int yb200_resize_bilinear_bwd(const yb200_act* dout, const yb200_act* h, const yb200_act* dx, void* stream);
int yb200_upsample_nearest2x_add(const yb200_act* lat, const yb200_act* coarse, const yb200_act* out, void* stream);
int yb200_upsample_nearest2x_bwd(const yb200_act* dy, const yb200_act* h, const yb200_act* dx, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* YB200_H_ */
