/*
 * libmyolo_sm90a — C ABI of the H100-native (sm_90a) joint detection+segmentation hot path.
 *
 * The reference (TomMao23/multiyolov5) is pure Python: the interfaces this library sits behind are
 *   - models.yolo.Model.forward / forward_once          (reference models/yolo.py:273-316)
 *   - models.yolo.Model.fuse  (BN folding)              (reference models/yolo.py:339-347, utils/torch_utils.py:182-202)
 *   - utils.general.non_max_suppression                 (reference utils/general.py:421-509)
 *   - detect.py's seg upsample + argmax                 (reference detect.py:191-193)
 * so the "FFI binding" a maintainer adds on the reference side is a ctypes stub (INTEGRATION.md).
 *
 * Conventions
 *   - every entry point returns 0 on success, a negative MYOLO_E_* code otherwise; myolo_last_error()
 *     returns a thread-local human readable message.  No C++ exceptions cross the ABI.
 *   - all data pointers are DEVICE pointers unless the name says `host_`; the library never frees caller memory.
 *   - `stream` is a cudaStream_t passed as void* (torch.cuda.current_stream().cuda_stream); the library never
 *     synchronises the device on its own.
 *   - there is NO CPU fallback: every function needs an sm_90 (H100) device and fails loudly otherwise.
 */
#ifndef MYOLO_H_
#define MYOLO_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define MYOLO_ABI_VERSION 1

/* error codes */
#define MYOLO_OK 0
#define MYOLO_E_INVALID (-1)  /* bad argument / unsupported shape           */
#define MYOLO_E_CUDA (-2)     /* CUDA runtime / driver error                */
#define MYOLO_E_NODEVICE (-3) /* no sm_90 device                            */
#define MYOLO_E_STATE (-4)    /* call order (e.g. forward before weights)   */

/* dtypes */
#define MYOLO_F16 0
#define MYOLO_F32 1
#define MYOLO_U8 2
#define MYOLO_I64 3

/* activation of a conv op */
#define MYOLO_ACT_NONE 0
#define MYOLO_ACT_SILU 1    /* nn.SiLU, reference models/common.py:40 */
#define MYOLO_ACT_SIGMOID 2 /* nn.Sigmoid in FFM attention, reference models/common.py:220 */

/* op kinds of the layer plan (what Model.forward_once executes, reference models/yolo.py:293-316) */
#define MYOLO_OP_INPUT_FOCUS 1   /* NCHW image -> 2x2 space-to-depth NHWC fp16 (Focus.forward, models/common.py:549-550) */
#define MYOLO_OP_CONV 2          /* conv(+folded BN)+bias+act(+residual): Conv/Bottleneck, models/common.py:42-46,104-105 */
#define MYOLO_OP_UPSAMPLE_NEAREST 3 /* nn.Upsample(None,2,'nearest'), yaml layers 11/15 */
#define MYOLO_OP_SPP_POOL 4      /* cascaded stride-1 max pools 5/9/13, models/common.py:170-174 */
#define MYOLO_OP_BILINEAR 5      /* bilinear align_corners=True NHWC->NHWC, models/yolo.py:163,170,174; models/common.py:534-537 */
#define MYOLO_OP_REGION_SUM 6    /* fp32 sums over rectangular atoms (stage 1 of AdaptiveAvgPool2d / GAP) */
#define MYOLO_OP_REGION_COMBINE 7 /* bins = sum(atoms)/count   (stage 2; models/common.py:521-524, :214) */
#define MYOLO_OP_CHANNEL_SCALE 8 /* FFM: feat*att+feat in place, models/common.py:228-229 */
#define MYOLO_OP_ADD 9           /* elementwise add (SegMaskBiSe m16 + up32, models/yolo.py:83) */
#define MYOLO_OP_DETECT_DECODE 10 /* Detect.forward view/permute/sigmoid/decode, models/yolo.py:211-225 */
#define MYOLO_OP_SEG_UPSAMPLE 11 /* final x8 bilinear of the seg head -> NCHW logits, models/yolo.py:163 */
#define MYOLO_OP_BROADCAST 12    /* F.interpolate(nearest) of a 1x1 map (RFB2 global branch), models/common.py:509 */
#define MYOLO_OP_BN_ACT 14       /* train mode: batch-statistics BatchNorm + activation (+ residual) on a raw conv output; aux[0] = bn slot */
#define MYOLO_OP_ACT 15          /* train mode: standalone activation (FFM attention SiLU / Sigmoid) so the pre-activation is kept */
#define MYOLO_OP_DROPOUT 17      /* train mode: out = in * keep / (1-p), keep ~ Bernoulli(1-p) from a counter-based hash of (seed, forward step, op, element); faux[0] = p, aux[0] = op salt.  nn.Dropout(0.1) of the Base / BiSe heads (reference models/yolo.py:65,140) */
#define MYOLO_OP_CHANNEL_SCALE_OOP 16 /* train mode: out = in * (1 + in2) out of place (in is needed by the backward pass) */
#define MYOLO_OP_FOCUS_CONV 13   /* whole layer 0 fused: Focus slicing + Conv3x3+BN+SiLU from the NCHW image, models/common.py:542-551 */

/* conv op flags */
#define MYOLO_CONV_FORCE_SIMT 1 /* run on the generic CUDA-core kernel (tiny M / odd shapes / debugging) */
/* op flags (any kind): a run of 2..4 CONSECUTIVE ops of one kind (REGION_COMBINE of one atom grid, small CONVs, BILINEARs with equal output
 * extents) may be executed as ONE launch: the first op carries GROUP_HEAD and the member count in aux[7], the others GROUP_MEMBER */
#define MYOLO_OP_GROUP_HEAD 2
#define MYOLO_OP_GROUP_MEMBER 4

typedef struct {
  int32_t h, w, c; /* per-image NHWC extents; batch is the plan's B */
  int32_t dtype;   /* MYOLO_F16 or MYOLO_F32 */
  int64_t offset;  /* byte offset inside the plan workspace (liveness-packed by the host-side planner) */
} myolo_buf_desc;

typedef struct {
  int32_t buf;   /* index into the buffer table, -1 = none */
  int32_t c_off; /* first channel of the slice */
  int32_t c;     /* channels in the slice */
} myolo_view;

typedef struct {
  int32_t kind;
  myolo_view in;  /* main input                                      */
  myolo_view in2; /* residual (CONV) / second addend (ADD) / attention (CHANNEL_SCALE) */
  myolo_view out;
  int32_t k, stride, dil; /* CONV geometry; pad = dil*(k/2)             */
  int32_t act;
  int32_t flags;
  int32_t weight_slot;    /* CONV: index used with myolo_plan_set_conv_weights */
  int32_t aux[8];         /* kind specific (documented in multiyolov5_b200/plan.py) */
  float faux[4];
} myolo_op;

typedef struct myolo_plan myolo_plan;

/* ---- library ---- */
int myolo_abi_version(void);
const char* myolo_last_error(void);
/* fills name (<=255 chars), SM count, compute capability major/minor of the current device */
int myolo_device_info(char* name, int* sm_count, int* cc_major, int* cc_minor);

/* ---- layer plan: what Model.__init__/fuse + forward_once become ---- */
int myolo_plan_create(const myolo_op* ops, int n_ops, const myolo_buf_desc* bufs, int n_bufs,
                      const int32_t* extra, int n_extra, /* variable-length tables referenced by aux[] */
                      int B, int H, int W, int64_t workspace_bytes, int n_weight_slots, myolo_plan** out);
void myolo_plan_destroy(myolo_plan* plan);
/* folds BN (eval: w' = w*g/sqrt(var+eps), b' = beta - g*mean/sqrt(var+eps); reference utils/torch_utils.py:182-202),
 * converts to fp16 and packs [Co][Ci][k][k] fp32 -> [Co_pad][k*k][Ci_pad].  gamma..var / bias may be NULL. */
int myolo_plan_set_conv_weights(myolo_plan* plan, int weight_slot, const float* w, int co, int ci, int k,
                                const float* gamma, const float* beta, const float* mean, const float* var, float eps,
                                const float* bias, void* stream);
/* Re-packs EVERY slot from the pointers the last myolo_plan_set_conv_weights calls registered, in one launch (training: the fp32
 * parameters changed in place - optimizer.step() reference train.py:396-398 - and every fp16 copy, forward and data-gradient, follows).
 * The pointers must still be valid; call myolo_plan_set_conv_weights again for a slot whose tensors moved. */
int myolo_plan_repack_weights(myolo_plan* plan, void* stream);
/* One forward pass.  x: (B,3,H,W) NCHW of x_dtype (F32/F16 in [0,1], or U8 scaled by 1/255 like detect.py:137).
 * z: (B, sum_i 3*ny_i*nx_i, 5+nc) fp32;  raw[i]: (B,3,ny_i,nx_i,5+nc) fp32 (nullable);
 * seg: (B,n_segcls,H,W) of seg_dtype (nullable); seg_argmax: (B,H,W) int64 class ids (nullable, fused path). */
int myolo_plan_forward(myolo_plan* plan, const void* x, int x_dtype, float* z, float* const* raw, void* seg, int seg_dtype,
                       int64_t* seg_argmax, void* stream);
/* debugging / per-layer parity: copies the NHWC buffer slice of a view into dst as (B,C,H,W) fp32 */
int myolo_plan_read_view(myolo_plan* plan, myolo_view view, float* dst_nchw, void* stream);
/* number of kernels the last myolo_plan_forward launched (bench.py's gpu_launches) */
int64_t myolo_plan_last_launch_count(const myolo_plan* plan);
/* which kernel conv op `op_index` takes and its tiling: info[12] = {1 wgmma / 0 CUDA-core, grid, smem bytes, BN, stages, mode (always 0:
 * one TMA box per tap), weights-stationary (0), tiles per round (1), tiles, N tiles, kc, CTAs per SM (1)}.  Feeds bench.py's roofline record. */
int myolo_plan_conv_info(myolo_plan* plan, int op_index, int32_t* info);
/* per-op device time of the next forward (CUDA events around every op; host array of n_ops floats, ms) */
int myolo_plan_profile(myolo_plan* plan, const void* x, int x_dtype, float* z, float* const* raw, void* seg, int seg_dtype,
                       int64_t* seg_argmax, float* host_ms_per_op, void* stream);

/* ---- training (SURVEY.md section 8 row a13): plans built with train-mode ops; no buffer aliasing; no CUDA graph ---- */
/* BatchNorm parameters of bn_slot: device fp32 pointers owned by the caller (updated in place by its optimiser); running stats are
 * updated by the forward with `momentum` (reference utils/torch_utils.py:150-152: eps 1e-3, momentum 0.03); d_gamma/d_beta nullable */
int myolo_plan_set_bn(myolo_plan* plan, int bn_slot, int channels, float* gamma, float* beta, float* running_mean, float* running_var,
                      float* d_gamma, float* d_beta, float momentum, float eps);
/* where the conv parameter gradients are accumulated (fp32, PyTorch layout [Co][Ci][k][k]; d_bias nullable) */
int myolo_plan_set_conv_grad(myolo_plan* plan, int weight_slot, float* d_weight, float* d_bias);
/* seed of the train-mode dropout masks (default 0); masks change with every train forward */
int myolo_plan_set_seed(myolo_plan* plan, uint64_t seed);
/* Concurrent train-mode forwards of one model on two plans (the det and the seg pass of reference train.py:364-392): a plan with
 * defer != 0 leaves running_mean / running_var untouched in its forward and keeps the batch sums; myolo_plan_apply_running then performs
 * the momentum update of every BN layer in one launch - call it after the other plan's forward so the statistics move in the
 * reference's order (det batch first, then seg batch). */
int myolo_plan_set_defer_running(myolo_plan* plan, int defer);
int myolo_plan_apply_running(myolo_plan* plan, void* stream);
/* train-mode forward: raw[i] (B,na,ny,nx,no) fp32 and seg (B,n_segcls,H,W) fp32, like Model.forward in training (models/yolo.py:225,316) */
int myolo_plan_train_forward(myolo_plan* plan, const void* x, int x_dtype, float* const* raw, float* seg, void* stream);
/* backward of the last train forward: grad_raw[i] / grad_seg are dL/d(raw[i]) / dL/d(seg) (fp32, nullable); parameter gradients are
 * ACCUMULATED into the registered pointers (the reference accumulates the det and the seg pass, train.py:371,392) */
int myolo_plan_backward(myolo_plan* plan, const float* const* grad_raw, const float* grad_seg, void* stream);
/* BiSe head in train mode returns three seg outputs [out, aux16, aux32] (reference models/yolo.py:70-79,86): seg[k] / grad_seg[k]
 * are arrays of three fp32 (B,n_segcls,H,W) pointers (nullable entries; k = 0 is the main output) */
int myolo_plan_train_forward_multi(myolo_plan* plan, const void* x, int x_dtype, float* const* raw, float* const* seg, void* stream);
int myolo_plan_backward_multi(myolo_plan* plan, const float* const* grad_raw, const float* const* grad_seg, void* stream);
/* Fused segmentation loss (SURVEY.md section 8f rank 3): mean CrossEntropyLoss(ignore_index) of the bilinear(align_corners) upsample of the
 * last train forward's low-resolution logits against `labels` (B,H,W) int64, WITHOUT materialising the full-resolution logits or their
 * gradient (reference models/yolo.py:163 + utils/loss.py:237 + autograd), followed by the backward pass seeded with
 * factor * (*scale_dev) * d(loss)/d(logits).  loss_out (device float, nullable) receives the mean CE.  scale_dev: device float, nullable. */
int myolo_plan_backward_seg_ce(myolo_plan* plan, const int64_t* labels, int ignore_index, float factor, const float* scale_dev,
                               float* loss_out, void* stream);
/* debug: like myolo_plan_read_view, from the gradient workspace of the last backward */
int myolo_plan_read_grad_view(myolo_plan* plan, myolo_view view, float* dst_nchw_f32, void* stream);
/* Optimiser step over FLAT fp32 buffers (all parameters of the model laid out back to back; `group[i]` in 0..n_groups-1 selects the
 * lr / weight decay of element i): torch.optim.SGD(momentum, nesterov) as configured by reference train.py:108-126 (pg0 BN weights,
 * pg1 conv weights + decay, pg2 biases).  Gradients are multiplied by *inv_scale (device scalar: 1 / (loss scale x world size),
 * nullable = 1); when *found_inf != 0 the update is skipped (amp.GradScaler.step, train.py:396); zero_grad clears the gradients in the
 * same pass (optimizer.zero_grad, train.py:398).  lr / weight_decay are HOST arrays of n_groups (<= 4) floats. */
/* standalone weight gradient of one conv (per-op parity tests / ncu): x (B,H,W,ci) and dy (B,Ho,Wo,co) NHWC fp16, "same" padding
 * dil*(k/2); dW fp32 [co][ci][k][k] is ACCUMULATED into.  path 0: mma.sync kernel, 1: wgmma kernel (needs ci % 64 == 0, Wo % 16 == 0) */
int myolo_conv_wgrad(const void* x, const void* dy, int B, int H, int W, int ci, int co, int k, int stride, int dil, float* dW, int path,
                     void* stream);
int myolo_grads_check_finite(const float* grad, int64_t n, int32_t* found_inf /* device */, void* stream);
int myolo_sgd_step(float* param, float* grad, float* momentum_buf, const uint8_t* group, int64_t n, const float* lr,
                   const float* weight_decay, int n_groups, float momentum, int nesterov, const float* inv_scale /* device */,
                   const int32_t* found_inf /* device, nullable */, int zero_grad, void* stream);

/* Detection loss forward + backward in four launches (reference utils/loss.py:115-217 `ComputeLoss.__call__` / `build_targets` + autograd):
 * p[l] / dp[l]: the nl raw head outputs (B, na, ny[l], nx[l], no) fp32 and their gradients (overwritten); targets (nt, 6) [image, class,
 * x, y, w, h] normalised, all-zero rows never match; anchors_grid: nl*na*2 floats in grid units (host); balance: nl floats (host).
 * d loss / d p = mult * (*scale_dev) * d[bs-free ComputeLoss value]/dp with mult = batch * world * detgain chosen by the caller; items_out (device
 * float[4]) = lbox, lobj, lcls, their sum (detached, as the reference's loss_items).  fl_gamma = 0, cls_pw = obj_pw = 1 only. */
int64_t myolo_det_loss_workspace_bytes(int B, int na, int nl, const int32_t* ny, const int32_t* nx);
int myolo_det_loss(const float* const* p, float* const* dp, const float* targets, int nt, int B, int na, int no, int nl, const int32_t* ny,
                   const int32_t* nx, const float* anchors_grid, const float* balance, float hyp_box, float hyp_obj, float hyp_cls,
                   float anchor_t, float gr, float cp, float cn, float mult, const float* scale_dev, float* items_out, void* workspace,
                   int64_t workspace_bytes, void* stream);

/* The path's ONE exchange step (SURVEY.md section 8b/8e; reference train.py:243-245 wraps the model in DistributedDataParallel): in-place
 * SUM all-reduce of the flat fp32 gradient buffer over the ranks of `nccl_comm` (an ncclComm_t; averaging is folded into myolo_sgd_step's
 * inv_scale), enqueued on `stream`.  The library does not link NCCL: it binds ncclAllReduce from the libnccl the host process has already
 * loaded (torch's); MYOLO_E_INVALID if no NCCL is loaded.  Python binding: parallel.allreduce_flat_grads. */
int myolo_allreduce_grads(float* flat_grad, int64_t n, void* nccl_comm, void* stream);

/* ---- pre-process (SURVEY.md section 8f rank 1) ----
 * `letterbox` of reference utils/datasets.py:818-848 (cv2.resize INTER_LINEAR to resized_w x resized_h, constant border) on uint8 HWC
 * frames (B,H0,W0,3), bit exact with OpenCV's 8-bit path; optionally fused with the BGR->RGB swap, HWC->CHW transpose
 * (utils/datasets.py:185-189) and the uint8 -> fp16/fp32 /255 conversion (detect.py:135-137).  The caller computes the geometry
 * (resized size, top/left offsets, output H x W) with the reference's host arithmetic.  pad_bgr: 3 ints in SOURCE channel order (NULL =
 * 114).  out: (B,3,H,W) if chw else (B,H,W,3), dtype MYOLO_U8 / MYOLO_F16 / MYOLO_F32 (float = value / 255). */
int myolo_letterbox(const uint8_t* src, int B, int H0, int W0, int resized_w, int resized_h, int top, int left, int H, int W,
                    const int32_t* pad_bgr, void* out, int out_dtype, int chw, int swap_rb, void* stream);

/* ---- consumers of the seg output (SURVEY.md section 8f rank 2) ----
 * myolo_seg_lut_blend: out[i][c] = lut[class_map[i]][c] (label2image / trainid2id, reference detect.py:69-77; reverse_channels gives the
 * BGR order of detect.py:193) and, if `blend` is given, blend[i][c] = cv2.addWeighted(out, alpha, image, beta, 0) (detect.py:194).
 * class_map: uint8 or int64 (dtype code); lut: device (n_entries x channels) uint8; out / blend: (n_pixels x channels) uint8, each nullable.
 * myolo_seg_metrics: the counters of utils/metrics.py:234-275 from a class map and int64 labels (-1 = ignore), ACCUMULATED into
 * counters[2 + 3*n_classes] (device uint64): [correct, labeled, intersection[n], prediction area[n], label area[n]]. */
int myolo_seg_lut_blend(const void* class_map, int map_dtype, int64_t n_pixels, const uint8_t* lut, int n_entries, int channels,
                        int reverse_channels, uint8_t* out, const uint8_t* image, float alpha, float beta, uint8_t* blend, void* stream);
int myolo_seg_metrics(const void* pred, int pred_dtype, const int64_t* target, int64_t n_pixels, int n_classes, uint64_t* counters,
                      void* stream);

/* ---- post-process ---- */
/* utils.general.non_max_suppression (reference utils/general.py:421-509).  pred: (B,A,no) fp32.
 * out: (B,max_det,6) fp32 rows [x1,y1,x2,y2,conf,cls] in the reference's order; out_count: (B) int32.
 * classes: device int32 list or NULL.  workspace: >= myolo_nms_workspace_bytes(B,A,no,multi_label). */
int64_t myolo_nms_workspace_bytes(int B, int A, int no, int multi_label);
int myolo_nms(const float* pred, int B, int A, int no, float conf_thres, float iou_thres, const int32_t* classes,
              int n_classes, int agnostic, int multi_label, int max_det, int max_nms, float max_wh, float* out,
              int32_t* out_count, void* workspace, int64_t workspace_bytes, void* stream);
/* detect.py:191-193: bilinear(align_corners=True) to (H,W) then argmax over C (first max wins).
 * logits: (B,C,h,w) NCHW fp32/fp16.  out: (B,H,W) int64 (out_dtype I64) or uint8 (U8). */
int myolo_seg_upsample_argmax(const void* logits, int dtype, int B, int C, int h, int w, int H, int W, void* out,
                              int out_dtype, void* stream);
/* F.interpolate(seg,(H,W),'bilinear',align_corners=True) on NCHW fp32 (materialised logits) */
int myolo_bilinear_nchw(const float* src, int B, int C, int h, int w, int H, int W, float* dst, void* stream);

/* ---- standalone kernels for per-op parity tests and ncu captures ---- */
/* SiLU(conv(x)*bnscale+bnshift) on NHWC fp16: x (B,H,W,Ci) -> y (B,Ho,Wo,Co); w fp32 [Co][Ci][k][k]; path: 0 auto, 1 wgmma, 2 simt, 3 wgmma (same kernel as 1) */
int myolo_conv_bn_silu(const void* x_nhwc_f16, int B, int H, int W, int ci, const float* w, int co, int k, int stride,
                       int dil, const float* gamma, const float* beta, const float* mean, const float* var, float eps,
                       const float* bias, int act, const void* residual_nhwc_f16, void* y_nhwc_f16, int path, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* MYOLO_H_ */
