/*
 * libmyolo_sm90a — C ABI of the H100-native (sm_90a) joint detection+segmentation hot path.
 *
 * The reference (TomMao23/multiyolov5) is pure Python: the interfaces this library sits behind are
 *   - models.yolo.Model.forward / forward_once          (reference models/yolo.py:273-316)
 *   - models.yolo.Model.fuse  (BN folding)              (reference models/yolo.py:339-347, utils/torch_utils.py:182-202)
 *   - utils.general.non_max_suppression                 (reference utils/general.py:421-509)
 *   - detect.py's seg upsample + argmax                 (reference detect.py:191-193)
 *   - the training batch loaders: LoadImagesAndLabels.__getitem__ (utils/datasets.py:518-593) and the segmentation
 *     datasets' `_sync_transform` + ColorJitter + ToTensor (SegmentationDataset.py:118-151, :458-531)
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
#define MYOLO_F64 4   /* myolo_anchor_metric only */

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
/* 13 is retired (it was a fused Focus + conv layer 0) */
#define MYOLO_OP_BN_ACT 14       /* train mode: batch-statistics BatchNorm + activation (+ residual) on a raw conv output; aux[0] = bn slot */
#define MYOLO_OP_ACT 15          /* train mode: standalone activation (FFM attention SiLU / Sigmoid) so the pre-activation is kept */
#define MYOLO_OP_DROPOUT 17      /* train mode: out = in * keep / (1-p), keep ~ Bernoulli(1-p) from a counter-based hash of (seed, forward step, op, element); faux[0] = p, aux[0] = op salt.  nn.Dropout(0.1) of the Base / BiSe heads (reference models/yolo.py:65,140) */
#define MYOLO_OP_CHANNEL_SCALE_OOP 16 /* train mode: out = in * (1 + in2) out of place (in is needed by the backward pass) */

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

/* ---- layer plan: what Model.__init__/fuse + forward_once become ---- */
int myolo_plan_create(const myolo_op* ops, int n_ops, const myolo_buf_desc* bufs, int n_bufs,
                      const int32_t* extra, int n_extra, /* variable-length tables referenced by aux[] */
                      int B, int H, int W, int64_t workspace_bytes, int n_weight_slots, myolo_plan** out);
/* Like myolo_plan_create, but the plan binds to caller-owned activation / gradient workspaces `ws` / `gws` of `capacity` bytes each
 * (256-byte aligned) instead of allocating private ones: train plans of several input shapes that run one after another on one stream
 * (--multi-scale, reference train.py:354-359) share one pair sized for the largest.  MYOLO_E_INVALID when workspace_bytes > capacity.
 * The addresses are baked into the plan's tensor maps and captured graphs: they must stay valid, at the same address, for the plan's life.
 * The caller zeroes `ws` before the plan's first forward and again whenever another plan has written it since (the plan reads some
 * never-written bytes, e.g. zero-padded channels, as zeros).  myolo_plan_destroy never frees them.
 * The library does not track which plan wrote the shared workspaces last: a backward (myolo_plan_backward_multi, myolo_plan_backward_seg_*)
 * after ANOTHER plan's train forward on the same pair reads that plan's activations as its own and returns wrong gradients without an
 * error.  The caller keeps one outstanding train forward per pair: forward, backward, then the next plan's forward (the Python engine
 * refuses such a stale backward before it launches). */
int myolo_plan_create_shared(const myolo_op* ops, int n_ops, const myolo_buf_desc* bufs, int n_bufs, const int32_t* extra, int n_extra,
                             int B, int H, int W, int64_t workspace_bytes, int n_weight_slots, void* ws, void* gws, int64_t capacity,
                             myolo_plan** out);
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
/* Overwrites n words of the plan's extra table (the `extra` of myolo_plan_create) from offset on, with n int32 / fp32 words read from
 * DEVICE memory `src`, stream-ordered and at the table's device address (captured graphs stay valid).  Inference plans refresh each
 * DETECT_DECODE op's anchors with it when the model's anchor_grid moved (an EMA averages it).  MYOLO_E_INVALID out of range. */
int myolo_plan_set_extra(myolo_plan* plan, int offset, const void* src, int n, void* stream);
/* One forward pass.  x: (B,3,H,W) NCHW of x_dtype (F32/F16 in [0,1], or U8 scaled by 1/255 like detect.py:137).
 * z: (B, sum_i 3*ny_i*nx_i, 5+nc) fp32;  raw[i]: (B,3,ny_i,nx_i,5+nc) fp32 (nullable);
 * seg: (B,n_segcls,H,W) of seg_dtype (nullable); seg_argmax: (B,H,W) int64 class ids (nullable, fused path). */
int myolo_plan_forward(myolo_plan* plan, const void* x, int x_dtype, float* z, float* const* raw, void* seg, int seg_dtype,
                       int64_t* seg_argmax, void* stream);
/* One pass of test-time augmentation (reference models/yolo.py:274-289): myolo_plan_forward without raw outputs, whose Detect decodes write
 * the plan's rows into rows [z_row_offset, z_row_offset + plan rows) of z (B, z_rows_total, 5+nc) fp32, with the four box columns
 * multiplied by z_inv_scale (`yi[..., :4] /= si` with z_inv_scale = 1.0f / (float)si) and, for z_flip_w > 0, column 0 replaced by
 * (float)z_flip_w - x (`yi[..., 0] = img_size[1] - yi[..., 0]`), each rounded once.  (z_rows_total = plan rows, 0, 1.0f, 0) is
 * myolo_plan_forward's z bit for bit.  The arguments reach only the decodes, which run after the captured graph: changing them between
 * calls captures nothing again.  MYOLO_E_INVALID when the rows do not fit, z_inv_scale is not positive and finite or z_flip_w < 0. */
int myolo_plan_forward_pass(myolo_plan* plan, const void* x, int x_dtype, float* z, int z_rows_total, int z_row_offset, float z_inv_scale,
                            int z_flip_w, void* seg, int seg_dtype, int64_t* seg_argmax, void* stream);
/* The seg output of a model ensemble (models.experimental.Ensemble) over plans[0..K) of K <= MYOLO_ENSEMBLE_MAX members, after each
 * plan's latest forward on the same input (myolo_plan_forward_pass with seg = seg_argmax = NULL leaves its low-res logits in its
 * workspace).  Per output pixel and class: each member's x8 upsampled logit as its own forward would store it in seg_dtype, the fp32
 * mean of those K values as torch's CUDA `torch.stack(maps).mean(0)` computes it (its per-thread partial sums, and the member groups it
 * reduces separately when the stacked maps exceed 32-bit byte offsets), then seg (B,n_segcls,H,W) of seg_dtype (nullable)
 * and/or seg_argmax (B,H,W) int64, the argmax of the fp32 mean, first maximum wins (nullable, not both null).  The plans must share
 * B, H, W, n_segcls and the low-res size.  MYOLO_E_INVALID when they do not, or when K members' staged source rows exceed the device's
 * shared memory per block. */
#define MYOLO_ENSEMBLE_MAX 8
int myolo_seg_ensemble(myolo_plan* const* plans, int K, void* seg, int seg_dtype, int64_t* seg_argmax, void* stream);
/* debugging / per-layer parity: copies the NHWC buffer slice of a view into dst as (B,C,H,W) fp32 */
int myolo_plan_read_view(myolo_plan* plan, myolo_view view, float* dst_nchw, void* stream);
/* number of kernels the last myolo_plan_forward launched (bench.py's gpu_launches) */
int64_t myolo_plan_last_launch_count(const myolo_plan* plan);
/* which kernel conv op `op_index` takes and its tiling: info[12] = {1 wgmma / 0 CUDA-core, grid, smem bytes, BN, stages, strip (1: one
 * input strip per filter row, 0: one TMA box per tap), resident (1: the CTA keeps its weight slice in shared memory), always 1, tiles,
 * N tiles, kc, CTAs per SM (1 or 2)}.  Feeds bench.py's roofline record. */
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
/* Synchronised BatchNorm (torch.nn.SyncBatchNorm, the reference's --sync-bn, train.py:190-193): every train-mode BN layer normalises with
 * the mean and biased variance over the batches of all ranks, updates its running statistics with them and the global count, and its
 * backward uses {sum dz, sum dz*xhat} summed over ranks (d_gamma / d_beta stay local).
 *   nccl_comm (ncclComm_t): ncclAllGather of each layer's {count, mean, var} record in the forward and ncclAllReduce of the two sums in
 *     the backward, on this communicator and the plan's stream; world size and rank from ncclCommCount / ncclCommUserRank.  Every rank must
 *     run the same plans in the same order (NCCL matches collectives by sequence).
 *   rank_images[n_groups] (nccl_comm null): one-GPU rank emulation.  The batch is n_groups consecutive groups of images, each treated
 *     as one rank's batch (unequal counts allowed; the counts sum to the plan's batch).
 * Both null: off.  Both set: MYOLO_E_INVALID.  Not with myolo_plan_set_defer_running.  A synchronised plan runs its forward and backward
 * in order on the caller's stream, without CUDA-graph replay.  Every BN layer must have C % 8 == 0 and C <= 2048. */
int myolo_plan_set_bn_sync(myolo_plan* plan, void* nccl_comm, const int32_t* rank_images, int n_groups);
/* train-mode forward: raw[i] (B,na,ny,nx,no) fp32 and the seg outputs, like Model.forward in training (models/yolo.py:225,316).  seg is
 * nullable or an array of three fp32 (B,n_segcls,H,W) pointers (nullable entries; k = 0 is the main output): the BiSe head in train mode
 * returns three seg outputs [out, aux16, aux32] (reference models/yolo.py:70-79,86). */
int myolo_plan_train_forward_multi(myolo_plan* plan, const void* x, int x_dtype, float* const* raw, float* const* seg, void* stream);
/* backward of the last train forward: grad_raw[i] / grad_seg[k] are dL/d(raw[i]) / dL/d(seg[k]) (fp32, nullable; grad_seg as seg above);
 * parameter gradients are ACCUMULATED into the registered pointers (the reference accumulates the det and the seg pass, train.py:371,392) */
int myolo_plan_backward_multi(myolo_plan* plan, const float* const* grad_raw, const float* const* grad_seg, void* stream);
/* Fused segmentation loss (SURVEY.md section 8f rank 3): mean CrossEntropyLoss(ignore_index) of the bilinear(align_corners) upsample of the
 * last train forward's low-resolution logits against `labels` (B,H,W) int64, WITHOUT materialising the full-resolution logits or their
 * gradient (reference models/yolo.py:163 + utils/loss.py:237 + autograd), followed by the backward pass seeded with
 * factor * (*scale_dev) * d(loss)/d(logits).  loss_out (device float, nullable) receives the mean CE.  scale_dev: device float, nullable. */
int myolo_plan_backward_seg_ce(myolo_plan* plan, const int64_t* labels, int ignore_index, float factor, const float* scale_dev,
                               float* loss_out, void* stream);
/* The same fused pass with the reference's OhemCELoss (utils/loss.py:303-328) in place of the mean CE: with n_min = (valid pixels) // 16,
 * the pixels whose CE exceeds thresh_t (= -log(thresh), fp32) when there are at least n_min of them, else the n_min largest CEs (ignored
 * pixels take part with CE 0; among pixels tied at the n_min-th value the lowest flat indices b*H*W + y*W + x), averaged over the pixels
 * taken.  No hard pixel with n_min = 0 gives NaN and no gradient, as the reference does; a non-finite CE gives a NaN loss and NaN
 * gradients.  The selection runs on the device with a fixed launch sequence (no host synchronisation; capturable, either branch on replay).
 * Scratch of 4 bytes per full-resolution pixel plus ~5 KB is allocated on the first call and kept by the plan. */
int myolo_plan_backward_seg_ohem(myolo_plan* plan, const int64_t* labels, int ignore_index, float thresh_t, float factor,
                                 const float* scale_dev, float* loss_out, void* stream);
/* The same fused pass with the class-weighted CE and the focal loss in place of the mean CE: SegFocalLoss(gamma, alpha=class_weights,
 * reduction='mean') (reference utils/loss.py:279-297) as myolo_seg_focal_loss defines it, which with gamma = 0 is
 * CrossEntropyLoss(weight=class_weights) (SegmentationLosses(weight=...), train.py:269-278).  class_weights: n_segcls device floats owned
 * by the caller, nullable (unit weights); gamma finite and >= 0.  With gamma > 0 the ignored pixels' softmax enters the loss, against
 * class 0, as in the reference.  No host synchronisation.  Scratch of 8 bytes per full-resolution pixel plus 256 bytes is allocated on
 * the first call and kept by the plan. */
int myolo_plan_backward_seg_loss(myolo_plan* plan, const int64_t* labels, int ignore_index, const float* class_weights, float gamma,
                                 float factor, const float* scale_dev, float* loss_out, void* stream);
/* debug: like myolo_plan_read_view, from the gradient workspace of the last backward */
int myolo_plan_read_grad_view(myolo_plan* plan, myolo_view view, float* dst_nchw_f32, void* stream);
int myolo_grads_check_finite(const float* grad, int64_t n, int32_t* found_inf /* device */, void* stream);
/* Optimiser step over FLAT fp32 buffers (all parameters of the model laid out back to back; `group[i]` in 0..n_groups-1 selects the
 * lr / weight decay of element i): torch.optim.SGD(momentum, nesterov) as configured by reference train.py:108-126 (pg0 BN weights,
 * pg1 conv weights + decay, pg2 biases).  Gradients are multiplied by *inv_scale (device scalar: 1 / (loss scale x world size),
 * nullable = 1); when *found_inf != 0 the update is skipped (amp.GradScaler.step, train.py:396); zero_grad clears the gradients in the
 * same pass (optimizer.zero_grad, train.py:398).  lr / weight_decay are HOST arrays of n_groups (<= 4) floats. */
int myolo_sgd_step(float* param, float* grad, float* momentum_buf, const uint8_t* group, int64_t n, const float* lr,
                   const float* weight_decay, int n_groups, float momentum, int nesterov, const float* inv_scale /* device */,
                   const int32_t* found_inf /* device, nullable */, int zero_grad, void* stream);
/* torch.optim.Adam(betas=(beta1, beta2), eps) as reference train.py:128-137 builds it for --adam, behind amp.GradScaler, over the same
 * flat buffers as myolo_sgd_step: bit-identical with GradScaler.unscale_ + torch's default CUDA Adam (foreach, capturable=False).
 * exp_avg / exp_avg_sq: flat fp32 moments.  lr: HOST array of n_groups DOUBLES (torch divides the Python lr by the bias correction
 * before rounding the step size to fp32); weight_decay: host floats, 0 = no decay term (torch's `if weight_decay != 0`).
 * steps: device int32, the steps taken so far; the launch uses step *steps + 1 for the bias corrections and does NOT advance it: the caller
 * adds (*found_inf == 0) after the launch.  When *found_inf != 0 nothing moves.  zero_grad clears the gradients in both cases.
 * Every buffer 16-byte aligned, group 4-byte aligned; n need not be a multiple of 4. */
int myolo_adam_step(float* param, float* grad, float* exp_avg, float* exp_avg_sq, const uint8_t* group, int64_t n, const double* lr,
                    const float* weight_decay, int n_groups, double beta1, double beta2, double eps, const int32_t* steps /* device */,
                    const float* inv_scale /* device */, const int32_t* found_inf /* device, nullable */, int zero_grad, void* stream);
/* The scalars myolo_adam_step uses at step k = steps[i] (device int32, k >= 1), from the same device code: the double bias corrections
 * bc1[i] = 1 - beta1^k and bc2[i] = 1 - beta2^k, and the fp32 scalars step_size[i] = (float)(-(lr / bc1[i])), bc2_sqrt[i] =
 * (float)sqrt(bc2[i]). */
int myolo_adam_scalars(const int32_t* steps, int64_t n, double lr, double beta1, double beta2, float* step_size, float* bc2_sqrt,
                       double* bc1, double* bc2, void* stream);
/* ModelEMA.update (reference utils/torch_utils.py:290-300) over every floating-point state_dict entry in one launch, bit-identical with
 * its three torch statements `v *= d; v += (1. - d) * msd[k]`, each rounding to its own dtype.  With df = (float)decay and
 * d1f = (float)(1.0 - decay) (torch rounds a Python scalar to the op's fp32 math type):
 *   fp32 EMA:  v = rn(rn(v * df) + rn(d1f * m))
 *   fp16 EMA:  v = half_rn(rn(float(half_rn(float(v) * df)) + rn(d1f * m)))      (after the reference's ema.half() of test.py:45,124)
 * chunks: DEVICE array of n_chunks pieces, each n (1 .. any) elements of one entry; the EMA side is MYOLO_F32 or MYOLO_F16, the source
 * (the training model's entry) is always fp32.  The caller cuts entries at multiples of MYOLO_EMA_CHUNK elements (one CTA per chunk).  A
 * chunk whose two pointers are 16-byte (fp16 EMA: 8-byte) aligned runs 4-wide; any other runs element by element.  MYOLO_E_INVALID for
 * a null table, n_chunks < 1 or decay outside [0, 1]; the table's contents are the caller's to validate (Python: ValueError). */
#define MYOLO_EMA_CHUNK 8192
typedef struct {
  void* ema;           /* fp32 or fp16 EMA elements, updated in place */
  const float* src;    /* fp32 training-model elements */
  int32_t n;           /* elements in this chunk */
  int32_t dtype;       /* MYOLO_F32 or MYOLO_F16: the EMA side's dtype */
} myolo_ema_chunk;
int myolo_ema_update(const myolo_ema_chunk* chunks /* device */, int n_chunks, double decay, void* stream);

/* Detection loss forward + backward in four launches (reference utils/loss.py:115-217 `ComputeLoss.__call__` / `build_targets` + autograd):
 * p[l] / dp[l]: the nl raw head outputs (B, na, ny[l], nx[l], no) fp32 and their gradients (overwritten); targets (nt, 6) [image, class,
 * x, y, w, h] normalised, all-zero rows never match; anchors_grid: nl*na*2 floats in grid units (host); balance: nl floats (host).
 * d loss / d p = mult * (*scale_dev) * d[bs-free ComputeLoss value]/dp with mult = batch * world * detgain chosen by the caller; items_out (device
 * float[4]) = lbox, lobj, lcls, their sum (detached, as the reference's loss_items).  fl_gamma = 0, cls_pw = obj_pw = 1 only; 1 <= nl <= 3,
 * 1 <= na <= MYOLO_DET_LOSS_NA_MAX (the range of --evolve's `anchors` hyp). */
#define MYOLO_DET_LOSS_NA_MAX 10
int64_t myolo_det_loss_workspace_bytes(int B, int na, int nl, const int32_t* ny, const int32_t* nx);
int myolo_det_loss(const float* const* p, float* const* dp, const float* targets, int nt, int B, int na, int no, int nl, const int32_t* ny,
                   const int32_t* nx, const float* anchors_grid, const float* balance, float hyp_box, float hyp_obj, float hyp_cls,
                   float anchor_t, float gr, float cp, float cn, float mult, const float* scale_dev, float* items_out, void* workspace,
                   int64_t workspace_bytes, void* stream);

/* ---- autoanchor (reference utils/autoanchor.py:23-160; Python: utils.autoanchor) ---- */
#define MYOLO_ANCHOR_MAX 32   /* anchors (na * nl) per call */
typedef struct {
  int64_t n_best;        /* labels whose best ratio x over the anchors is > thr */
  int64_t n_x;           /* (label, anchor) pairs with x > thr */
  double sum_x, sum_best, sum_x_above;   /* fp64 sums of x, of best, and of x over pairs with x > thr (fixed order: the same every run) */
} myolo_anchor_stats;
/* The reference's ratio metric of n labels' wh (n, 2) against na anchors (na, 2): r = wh / k, x = min(r, 1 / r) over both sides (correct
 * rounding: torch's `1. / r` is r.reciprocal()), best = max over the anchors.  The arithmetic and the comparisons with thr (1 / anchor_t,
 * cast to the compute dtype) run in fp64 when either input is MYOLO_F64 (torch promotes an fp32 tensor divided by a float64 numpy array),
 * else in fp32.  wh_dtype, k_dtype: MYOLO_F32 or MYOLO_F64; device pointers; out: device myolo_anchor_stats.  workspace: device, at least
 * myolo_anchor_metric_workspace_bytes().  No host synchronisation. */
int64_t myolo_anchor_metric_workspace_bytes(void);
int myolo_anchor_metric(const void* wh, int wh_dtype, int64_t n, const void* k, int k_dtype, int na, double thr, myolo_anchor_stats* out,
                        void* workspace, int64_t workspace_bytes, void* stream);
/* kmean_anchors' genetic evolution (utils/autoanchor.py:146-158) in one persistent cooperative kernel.  wh: (n, 2) fp32 device labels;
 * k0: (na, 2) fp64 device start anchors (the sorted k-means result); v: (gen, na, 2) fp64 device mutation factors drawn on the host;
 * thr: 1 / anchor_t.  Per generation kg = max(k * v, 2.0) in fp64, its fp32 cast scores fg = fp32(sum of best over labels with best > thr,
 * summed exactly in fp64) / n in fp32, and kg replaces k when fg > f.  Outputs (device): k_out (na, 2) fp64, f_out[2] fp32 (the fitness
 * of k0, the final fitness), fg_out (gen) fp32, accepted_out int32 (generations taken).  Needs 1 <= n < 2^26, 1 <= na <= MYOLO_ANCHOR_MAX and fp32(thr) >= 1/16 (anchor_t <= 16):
 * the bounds of the exact sum; else MYOLO_E_INVALID.  workspace: device, at least myolo_anchor_evolve_workspace_bytes(n) (it depends on
 * the current device).  A cooperative launch sized from the kernel's occupancy: a grid that cannot be co-resident is refused, never run. */
int64_t myolo_anchor_evolve_workspace_bytes(int64_t n);
int myolo_anchor_evolve(const float* wh, int64_t n, const double* k0, int na, const double* v, int gen, double thr, double* k_out,
                        float* f_out, float* fg_out, int32_t* accepted_out, void* workspace, int64_t workspace_bytes, void* stream);
/* scipy.cluster.vq.kmeans(obs, k, iter=restarts, thresh) with an int k (kmean_anchors' `kmeans(wh / s, n, iter=30)`,
 * utils/autoanchor.py:125), bit for bit with scipy >= 1.17: one CTA per restart, all restarts in one ordinary launch.  obs: (n, d) fp64
 * device; init_idx: (restarts, k) int64 device, each restart's start rows (numpy.random's `choice(n, k, replace=False)`, drawn by the
 * caller as scipy's `_kpoints` draws them).  Per restart: Lloyd iterations (vq without fused multiply-adds, the first nearest code;
 * numpy's pairwise mean of the distances; per-cluster sequential fp64 member sums in observation order, empty clusters dropped) while
 * |prev - cur| > thresh from prev = inf, then one more vq with the final book for its distortion.  Outputs (device): books
 * (restarts, k, d) fp64 (the first book_k[r] rows valid, the rest zero), book_k (restarts) int32, dists (restarts) fp64, iters (restarts)
 * int32 (Lloyd iterations), best int32 (the first restart with the smallest distortion: scipy's winner), status int32 (zeroed by the call;
 * bits MYOLO_KMEANS_MAX_ITER: a restart was still moving after max_iter iterations, MYOLO_KMEANS_BAD_INDEX: an init_idx row outside
 * [0, n)).  Needs d == 2, 1 <= k <= MYOLO_KMEANS_KMAX, k <= n < 2^30, max_iter >= 1 and restarts at most the co-resident CTA count of
 * the current device; else MYOLO_E_INVALID.  workspace: device, at least myolo_kmeans_workspace_bytes(n, k, restarts).  No host
 * synchronisation. */
#define MYOLO_KMEANS_KMAX 32
#define MYOLO_KMEANS_MAX_ITER 1
#define MYOLO_KMEANS_BAD_INDEX 2
int64_t myolo_kmeans_workspace_bytes(int64_t n, int k, int restarts);
int myolo_kmeans(const double* obs, int64_t n, int d, const int64_t* init_idx, int k, int restarts, double thresh, int max_iter,
                 double* books, int32_t* book_k, double* dists, int32_t* iters, int32_t* best, int32_t* status, void* workspace,
                 int64_t workspace_bytes, void* stream);

/* --image-weights (reference train.py:255,305-316, utils/general.py:216-240), bit for bit with numpy 2 and Python 3.12's random.  A label's
 * class is its float32 class value truncated toward zero, as astype(int) does; a class outside [0, nc) is skipped and sets
 * MYOLO_IW_BAD_CLASS.  Every sum over the nc classes is numpy's np.add.reduce order (pairwise blocks of 8 accumulators, added to the
 * initial 0.0), in fp64 without fused multiply-adds.  status: int32 device word, only OR-ed (the caller zeroes it).  Needs
 * 1 <= nc <= MYOLO_IW_NC_MAX; else MYOLO_E_INVALID.  All pointers are device pointers; no host synchronisation.
 *   myolo_class_weights   labels_to_class_weights(labels, nc): cls is the (n_labels) float32 class column of every label; counts (nc) int64
 *                         the exact per-class counts; weights (nc) fp64 = (1 / max(count, 1)) / their sum.
 *   myolo_image_weights   labels_to_image_weights(labels, nc, cw): image i's labels are cls[offsets[i] .. offsets[i + 1]) (offsets:
 *                         n + 1 int64); iw (n) fp64 = the sum over c of cw[c] * count_i(c).
 *   myolo_weighted_draw   random.choices(range(n), weights=w, k=n) given its n random() values u (fp64): cum (n) fp64 the sequential
 *                         cumulative sums (itertools.accumulate), total (1) fp64 = cum[n - 1] + 0.0; total <= 0 sets MYOLO_IW_TOTAL_NONPOS,
 *                         a non-finite total MYOLO_IW_TOTAL_NONFINITE, and then idx is left unwritten; else idx (n) int32 =
 *                         bisect_right(cum, u[i] * total, 0, n - 1).  Needs 1 <= n < 2^31. */
#define MYOLO_IW_NC_MAX 1024
#define MYOLO_IW_BAD_CLASS 1
#define MYOLO_IW_TOTAL_NONPOS 2
#define MYOLO_IW_TOTAL_NONFINITE 4
int myolo_class_weights(const float* cls, int64_t n_labels, int nc, int64_t* counts, double* weights, int32_t* status, void* stream);
int myolo_image_weights(const float* cls, const int64_t* offsets, int64_t n, const double* cw, int nc, double* iw, int32_t* status,
                        void* stream);
int myolo_weighted_draw(const double* w, const double* u, int64_t n, double* cum, double* total, int32_t* idx, int32_t* status,
                        void* stream);

/* OhemCELoss.forward_once (reference utils/loss.py:321-328) over full-resolution logits (B, C, H, W) fp32 NCHW, any C, and labels (B, H, W)
 * int64, with the selection of myolo_plan_backward_seg_ohem.  myolo_seg_ohem_loss writes the loss to loss_out (device float) and leaves
 * its selection in the workspace; myolo_seg_ohem_loss_backward then writes grad_logits = (*grad_out) * d loss / d logits (grad_out: device
 * float) from the same logits, labels and workspace.  Labels outside [0, C) other than ignore_index count as ignored.  No host
 * synchronisation in either call.  Python: utils.loss.OhemCELoss. */
int64_t myolo_seg_ohem_loss_workspace_bytes(int B, int H, int W);
int myolo_seg_ohem_loss(const float* logits, const int64_t* labels, int B, int C, int H, int W, int ignore_index, float thresh_t,
                        float* loss_out, void* workspace, int64_t workspace_bytes, void* stream);
int myolo_seg_ohem_loss_backward(const float* logits, const int64_t* labels, int B, int C, int H, int W, int ignore_index,
                                 const float* grad_out, float* grad_logits, const void* workspace, int64_t workspace_bytes, void* stream);

/* SegFocalLoss(gamma, alpha=class_weights, ignore_index, reduction) (reference utils/loss.py:279-297) over full-resolution logits
 * (B, C, H, W) fp32 NCHW, any C, and labels (B, H, W) int64.  With t' = t on valid pixels and 0 on ignored ones, p = softmax over C and
 * N = B*H*W: loss = A * F, A = sum_valid w[t] CE / sum_valid w[t] and F = sum_all (1 - p_t')^gamma / N for MYOLO_REDUCTION_MEAN, the
 * two sums themselves for MYOLO_REDUCTION_SUM (the reference's CE takes the outer reduction).  gamma = 0 with the mean is the class-weighted
 * CrossEntropyLoss(weight=class_weights).  class_weights: C device floats, nullable (unit weights); gamma finite and >= 0.
 * myolo_seg_focal_loss writes the loss to loss_out (device float) and leaves its coefficients in the workspace; myolo_seg_focal_loss_backward
 * then writes grad_logits = (*grad_out) * d loss / d logits from the same logits, labels, weights, gamma and workspace.  Labels outside
 * [0, C) other than ignore_index count as ignored.  No host synchronisation in either call.  Python: utils.loss.SegFocalLoss. */
#define MYOLO_REDUCTION_MEAN 0
#define MYOLO_REDUCTION_SUM 1
int64_t myolo_seg_focal_loss_workspace_bytes(void);
int myolo_seg_focal_loss(const float* logits, const int64_t* labels, int B, int C, int H, int W, int ignore_index, const float* class_weights,
                         float gamma, int reduction, float* loss_out, void* workspace, int64_t workspace_bytes, void* stream);
int myolo_seg_focal_loss_backward(const float* logits, const int64_t* labels, int B, int C, int H, int W, int ignore_index,
                                  const float* class_weights, float gamma, const float* grad_out, float* grad_logits, const void* workspace,
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

/* ---- autoShape's pre-process of a ragged batch (reference models/common.py:636-658) ----
 * myolo_letterbox_items: B RGB uint8 HWC sources of different sizes, packed in one device buffer `src`, each letterboxed to the shared
 * H x W (`letterbox(im, new_shape=shape1, auto=False)`, cv2.resize INTER_LINEAR bit exact with OpenCV's 8-bit path, border 114, no
 * channel swap) into out (B,3,H,W): MYOLO_U8, or MYOLO_F16 / MYOLO_F32 holding value / 255 as torch's CPU division of
 * `.type_as(p) / 255.` gives.  items: DEVICE array of B myolo_letterbox_item built on the host (multiyolov5_b200/utils/datasets.py
 * letterbox_item_table); the kernel trusts its geometry (top + rh <= H, left + rw <= W, sources inside src). */
typedef struct {
  int64_t offset;            /* byte offset of the item's (H0, W0, 3) source in src */
  double scale_x, scale_y;   /* cv2's 1 / (rw / W0) and 1 / (rh / H0), in double */
  int32_t H0, W0;
  int32_t mode;              /* 0: copy (rw == W0 and rh == H0), 1: bilinear, 2: exact 2x down-scale (cv2's 2x2 area mean) */
  int32_t rw, rh;            /* resized (un-padded) size */
  int32_t top, left;         /* border offsets inside H x W */
  int32_t reserved;
} myolo_letterbox_item;
int myolo_letterbox_items(const uint8_t* src, const myolo_letterbox_item* items, int B, int H, int W, void* out, int out_dtype,
                          void* stream);

/* ---- detection training batches (reference utils/datasets.py:518-593 LoadImagesAndLabels.__getitem__, augment=True) ----
 * myolo_resize_u8: cv2.resize(src, (W, H), INTER_LINEAR) of one uint8 HWC image (H0,W0,3) into dst (H,W,3), bit exact with OpenCV's
 * 8-bit path (exact 2x down-scaling takes its area path): `load_image`'s resize to long side img_size (:629-643) for the device cache.
 * myolo_augment_det_hw: one batch of B augmented H x W images: the S x S batches of H = W = S, or the `--rect` batches at their batch
 * shape (`LoadImagesAndLabels(augment=True, rect=True)`: a letterbox to the batch shape, random_perspective at (W, H), flips over H and W).
 * items: DEVICE array of B myolo_aug_item, built on the host from the reference's random draws (multiyolov5_b200/utils/datasets.py
 * DetAugmenter, DetRectLoader).  Per output pixel: cv2.warpAffine (INTER_LINEAR, border 114) of the virtual canvas of warp[0] (mosaic
 * tiles or a letterboxed image, 114 elsewhere), optionally mixed with warp[1] (trunc(a*mix_r + b*mix_q) in double), augment_hsv through
 * the three LUTs, flipud / fliplr, BGR->RGB.
 * out: (B,3,H,W) of out_dtype MYOLO_U8 / MYOLO_F16 / MYOLO_F32 (float = value / 255, as imgs.float() / 255 on the GPU). */
typedef struct {
  const uint8_t* src[4];  /* tile images: HWC BGR uint8, device */
  int32_t rect[4][4];     /* canvas rectangle [x1, x2) x [y1, y2) covered by tile t: x1, y1, x2, y2 */
  int32_t off[4][2];      /* source pixel of canvas pixel (x, y): (x - off[t][0], y - off[t][1]) */
  int32_t src_w[4];       /* source row length in pixels */
  int32_t n_tiles;        /* 1..4 */
  int32_t reserved;
  double minv[6];         /* the affine M inverted the way cv2.warpAffine inverts it: canvas = minv * (x, y, 1) */
} myolo_aug_warp;

typedef struct {
  myolo_aug_warp warp[2];
  double mix_r, mix_q;    /* mixup ratio r and 1 - r (computed by the caller) */
  int32_t n_warps;        /* 1, or 2 with mixup */
  int32_t flipud, fliplr;
  int32_t reserved;
  uint8_t lut[3][256];    /* augment_hsv LUTs: hue, saturation, value */
} myolo_aug_item;

int myolo_resize_u8(const uint8_t* src, int H0, int W0, uint8_t* dst, int H, int W, void* stream);

/* myolo_resize_area_u8: cv2.resize(src, (W, H), INTER_AREA) of one uint8 HWC image (H0,W0,3) into dst (H,W,3), bit exact with OpenCV's
 * 8-bit path: `load_image`'s augment=False cache resize when it shrinks (validation, :639).  Down-scaling only: H > H0 or W > W0 is
 * MYOLO_E_INVALID.  cv2's choice of path: a copy at equal size, the 2x2 mean at exact 2x, the integer block sum times the float
 * reciprocal of its area at other integral scales, else the general float32 area-weight arithmetic. */
int myolo_resize_area_u8(const uint8_t* src, int H0, int W0, uint8_t* dst, int H, int W, void* stream);

/* myolo_resize_bilinear: the det batch rescale of --multi-scale (reference train.py:354-359), F.interpolate(x, (Ho, Wo), mode='bilinear',
 * align_corners=False) of NCHW src (B,C,H,W) into NCHW dst (B,C,Ho,Wo), bit exact with torch's CUDA kernel on fp32 input.  src_dtype
 * MYOLO_U8 (each tap converted as imgs.float() / 255.0 converts it on the device: v * fp32(1/255)), MYOLO_F16 or MYOLO_F32; dst_dtype
 * MYOLO_F16 (the fp32 result rounded to nearest) or MYOLO_F32.  Equal sizes convert only. */
int myolo_resize_bilinear(const void* src, int src_dtype, int B, int C, int H, int W, void* dst, int dst_dtype, int Ho, int Wo, void* stream);
/* myolo_scale_img: scale_img of test-time augmentation (reference utils/torch_utils.py:248-258) in one launch: F.interpolate of NCHW src
 * (B,C,H,W) to (Ho, Wo), bilinear, align_corners=False, as myolo_resize_bilinear computes it, then F.pad on the right and bottom to
 * dst (B,C,Hp,Wp) with pad_value (the caller rounds it to the dtype, as torch's fill does); Hp < Ho or Wp < Wo crops.  flip_lr != 0
 * resamples src.flip(3) instead.  src and dst share dtype, MYOLO_F16 or MYOLO_F32. */
int myolo_scale_img(const void* src, int dtype, int B, int C, int H, int W, void* dst, int Ho, int Wo, int Hp, int Wp, int flip_lr,
                    float pad_value, void* stream);
int myolo_augment_det_hw(const myolo_aug_item* items, int B, int H, int W, void* out, int out_dtype, void* stream);

/* myolo_collate_quad: the pixels of `--quad`'s LoadImagesAndLabels.collate_fn4 (reference utils/datasets.py:602-625) over one drawn batch,
 * one launch on `stream`, no synchronisation.  imgs: DEVICE uint8 (B,3,H,W) RGB, B >= 4; tile: HOST array of B/4 flags,
 * one per quad in order (the caller's `random.random() >= 0.5`), at most MYOLO_QUAD_MAX; they travel as kernel parameters.  Quad q of
 * out (B/4,3,2H,2W) is the 2x2 tile of items 4q (top left), 4q+1 (bottom left), 4q+2 (top right), 4q+3 (bottom right)
 * when tile[q], else F.interpolate(item 4q, scale_factor=2., mode='bilinear', align_corners=False) truncated to uint8, in integer
 * arithmetic that equals torch's bit for bit.  Items past 4 * (B/4) are not read.  out_dtype MYOLO_U8 / MYOLO_F16 / MYOLO_F32 (float =
 * value / 255, as imgs.float() / 255 on the GPU).  W % 8 == 0 with imgs 8-byte and out 16-byte aligned takes 8 pixels per thread. */
#define MYOLO_QUAD_MAX 1024
int myolo_collate_quad(const uint8_t* imgs, int B, int H, int W, const uint8_t* tile, void* out, int out_dtype, void* stream);

/* ---- segmentation training batches (reference SegmentationDataset.py:118-151 `_sync_transform` + ColorJitter + ToTensor, and the
 * testval items of :81-94) ----
 * myolo_augment_seg: B items in two launches on `stream`.  Per item: Pillow's bilinear Image.resize of the source (mirrored when `flip`)
 * evaluated over the h x w crop window only, right/bottom pad 0, the ColorJitter ops in `order`, ToTensor; the mask through Pillow's
 * NEAREST resize (pad 255) and `lut` into out_mask (B,mh,mw) int64.  items: DEVICE array, built on the host
 * (multiyolov5_b200/utils/datasets.py SegAugmenter); lsum must be 0 on entry (the kernel accumulates into it).  tables: DEVICE int32
 * array the items' offsets index.  scratch: B*h*w*3 bytes.  out_img: (B,3,h,w) of out_dtype MYOLO_U8 / MYOLO_F16 / MYOLO_F32
 * (float = v / 255 as ToTensor divides, fp16 that value rounded).  All arithmetic is bit exact with Pillow's. */
typedef struct {
  const uint8_t* img;     /* source (H0, W0, 3) RGB uint8, device */
  const uint8_t* mask;    /* source (H0, W0) uint8, device */
  int32_t H0, W0;
  int32_t flip;           /* mirror: source column x is read as W0-1-x */
  int32_t kx, ky;         /* coefficients per column / row entry */
  int32_t col, row;       /* offsets in `tables` of w column / h row entries {first source index, taps (0 = pad), kx|ky int32
                             coefficients with 22 fraction bits} */
  int32_t mcol, mrow;     /* offsets in `tables` of mw / mh mask source indices (-1 = pad) */
  int32_t order[4];       /* jitter ops in application order, -1 = none: 0 brightness, 1 contrast, 2 saturation, 3 hue */
  float factor[3];        /* brightness, contrast, saturation factors (C float, as Image.blend narrows them) */
  int32_t hue_shift;      /* added to H modulo 256 */
  int32_t reserved;
  uint64_t lsum;          /* sum of convert("L") of the image entering contrast: 0 on entry */
  int32_t lut[256];       /* mask value -> label */
} myolo_seg_item;

int myolo_augment_seg(myolo_seg_item* items, int B, int h, int w, int mh, int mw, const int32_t* tables, uint8_t* scratch, void* out_img,
                      int out_dtype, int64_t* out_mask, void* stream);

/* ---- consumers of the seg output (SURVEY.md section 8f rank 2) ----
 * myolo_seg_lut_blend: out[i][c] = lut[class_map[i]][c] (label2image / trainid2id, reference detect.py:69-77; reverse_channels gives the
 * BGR order of detect.py:193) and, if `blend` is given, blend[i][c] = cv2.addWeighted(out, alpha, image, beta, 0) (detect.py:194).
 * class_map: uint8 or int64 (dtype code); lut: device (n_entries x channels) uint8; out / blend: (n_pixels x channels) uint8, each nullable.
 * lut2 / out2 (nullable): a second table (n_entries x channels2, read in its own channel order) written to out2 (n_pixels x channels2)
 * from the same read of the class map: detect.py's mask, blend and trainid2id ids (detect.py:193-194,206) in one pass.
 * myolo_seg_metrics: the counters of utils/metrics.py:234-275 from a class map and int64 labels (-1 = ignore), ACCUMULATED into
 * counters[2 + 3*n_classes] (device uint64): [correct, labeled, intersection[n], prediction area[n], label area[n]]. */
int myolo_seg_lut_blend(const void* class_map, int map_dtype, int64_t n_pixels, const uint8_t* lut, int n_entries, int channels,
                        int reverse_channels, uint8_t* out, const uint8_t* image, float alpha, float beta, uint8_t* blend,
                        const uint8_t* lut2, int channels2, uint8_t* out2, void* stream);
int myolo_seg_metrics(const void* pred, int pred_dtype, const int64_t* target, int64_t n_pixels, int n_classes, uint64_t* counters,
                      void* stream);

/* ---- detect.py's boxes in frame space (reference detect.py:166-177; multiyolov5_b200/detect.py) ----
 * myolo_detect_boxes: for each of B frames, rows [0, counts[b]) of the padded NMS output rows (B, max_det, 6) fp32 are scaled IN PLACE to
 * the frame: scale_coords(img_shape, rows[:, :4], im0_shape).round() (x -= pad, x /= gain, clamp to [0, w0] / [0, h0], round half to
 * even), in fp32 IEEE arithmetic, equal to torch's CPU statements.  geom: device (B, 5) fp32 {pad_x, pad_y, gain, w0, h0}, the Python
 * scalars of scale_coords rounded to fp32.  xywhn (nullable): (B, max_det, 4) fp32, xyxy2xywh(box) / (w0, h0, w0, h0) of --save-txt.
 * class_counts (nullable): (B, nc) int32, each frame's rows per class id (ids that are not an integer in [0, nc) are not counted). */
int myolo_detect_boxes(float* rows, const int32_t* counts, int B, int max_det, const float* geom, int nc, float* xywhn,
                       int32_t* class_counts, void* stream);
/* myolo_scale_boxes: autoShape's boxes in image space (reference models/common.py:668-669,680-688).  Rows [0, counts[b]) of the padded
 * NMS rows (B, max_det, 6) fp32 become scale_coords(shape1, rows[:, :4], shape0[b]) IN PLACE (x -= pad, x /= gain, clamp to [0, w0] /
 * [0, h0], no rounding), fp32 IEEE arithmetic equal to torch's CPU statements; geom as in myolo_detect_boxes.  Each nullable output is
 * (B, max_det, 6) fp32 written for the same rows: xywh = xyxy2xywh(row), xyxyn = row / gn, xywhn = xywh / gn with
 * gn = (w0, h0, w0, h0, 1, 1) (a division, as Detections.__init__ does).  Rows past the count are not touched. */
int myolo_scale_boxes(float* rows, const int32_t* counts, int B, int max_det, const float* geom, float* xywh, float* xyxyn, float* xywhn,
                      void* stream);

/* ---- detection validation statistics (reference test.py:175,183-265 and utils/metrics.py:24-112; multiyolov5_b200/utils/metrics.py
 * DetectionStats) ----
 * The stats store holds one slot per (image, NMS row): correct (uint16, bit k = IoU > iouv[k]), conf (fp32) and class (uint8), plus the
 * image's row count, and per-class target counts (uint64[256]).
 * myolo_det_match: one launch for a batch of B images, written to images img_base .. img_base+B-1 of the store.  dets: (B,max_det,6)
 * NMS rows, counts: (B) int32, targets: (n_targets,6) fp32 [image, class, x, y, w, h] normalised, all device.  geom: device (B,5) fp32
 * (h0, w0, gain, padw, padh) of each image's loader shapes; iouv: device fp32[10].  Class ids outside [0,256) or not integral set bits of
 * *err (MYOLO_DET_ERR_*), as do more than 1024 targets in one image; the kernel never indexes out of bounds.
 * myolo_det_ap: ap_per_class over images 0 .. n_images-1 of the store, using the lowest `ncol` (<= 16) correct bits.  px: device
 * float64[1000] and x101: float64[101], numpy's linspace(0, 1, 1000 | 101).  Outputs, one row per class with tcount > 0 in class order:
 * out_ap (rows, ncol), out_p / out_r (rows, 1000) float64; out_info int32[2] = {any correct bit, number of predictions}.  Predictions of
 * one class with equal conf keep their (image, row) order.  workspace: >= myolo_det_ap_workspace_bytes(n_images, max_det, ncol). */
#define MYOLO_DET_ERR_TARGET_CLASS 1
#define MYOLO_DET_ERR_PRED_CLASS 2
#define MYOLO_DET_ERR_LABELS 4
int myolo_det_match(const float* dets, const int32_t* counts, int B, int max_det, const float* targets, int n_targets, int H, int W,
                    const float* geom, const float* iouv, int img_base, uint16_t* st_correct, float* st_conf, uint8_t* st_cls,
                    int32_t* st_rows, uint64_t* tcount, int32_t* err, void* stream);
/* utils.metrics.ConfusionMatrix.process_batch (the fork's utils/metrics.py:115-162) for a batch of B images in one launch, into
 * matrix: device int64 (nc+1, nc+1), row = true class (the fork's order), accumulated.  With geom != NULL the inputs are those of
 * myolo_det_match (padded NMS rows in network space, normalised targets, H, W, geom) and are scaled to native space as test.py does;
 * with geom == NULL, dets rows and targets [image, class, x1, y1, x2, y2] are native-space boxes already.  Detections with
 * conf <= conf_thres are dropped; pairs with IoU > iou_thres match, each detection keeping its best label and then each label its
 * best remaining detection (ties: lower label index, then lower detection index).  require_rows != 0 skips images without labels
 * or without rows, as test() only calls process_batch for those.  Classes outside [0, nc) set MYOLO_DET_ERR_TARGET_CLASS /
 * MYOLO_DET_ERR_PRED_CLASS in *err and are not counted; more than 1024 labels in one image sets MYOLO_DET_ERR_LABELS. */
int myolo_confusion_update(const float* dets, const int32_t* counts, int B, int max_det, const float* targets, int n_targets, int H,
                           int W, const float* geom, int nc, float conf_thres, float iou_thres, int require_rows, int64_t* matrix,
                           int32_t* err, void* stream);
int64_t myolo_det_ap_workspace_bytes(int n_images, int max_det, int ncol);
int myolo_det_ap(const uint16_t* correct, const float* conf, const uint8_t* cls, const int32_t* rows, int n_images, int max_det, int ncol,
                 const uint64_t* tcount, const double* px, const double* x101, double* out_ap, double* out_p, double* out_r,
                 int32_t* out_info, void* workspace, int64_t workspace_bytes, void* stream);

/* ---- post-process ---- */
/* utils.general.non_max_suppression (reference utils/general.py:421-509).  pred: (B,A,no) fp32.
 * out: (B,max_det,6) fp32 rows [x1,y1,x2,y2,conf,cls] in the reference's order; out_count: (B) int32.
 * classes: device int32 list or NULL.  workspace: >= myolo_nms_workspace_bytes(B,A,no,multi_label). */
int64_t myolo_nms_workspace_bytes(int B, int A, int no, int multi_label);
int myolo_nms(const float* pred, int B, int A, int no, float conf_thres, float iou_thres, const int32_t* classes,
              int n_classes, int agnostic, int multi_label, int max_det, int max_nms, float max_wh, float* out,
              int32_t* out_count, void* workspace, int64_t workspace_bytes, void* stream);
/* non_max_suppression(..., labels=lb) (utils/general.py:448-455, test.py --save-hybrid): as myolo_nms, with image b's apriori labels
 * labels[label_offsets[b] .. label_offsets[b+1]) appended after its candidates.  labels: device (n,5) fp32 [cls, x, y, w, h] in network
 * input pixels; label_offsets: device (B+1) int32.  max_labels bounds every image's label count (the number of rows n is always a
 * valid bound; labels may be NULL when it is 0).  A label whose class id truncates to a value outside [0, nc) is dropped and sets
 * MYOLO_NMS_ERR_LABEL_CLASS in *err; an image with more than max_labels labels sets MYOLO_NMS_ERR_LABEL_COUNT (its first max_labels
 * labels are used).  *err is OR-ed into, never cleared, so one word can serve many calls.
 * workspace: >= myolo_nms_labels_workspace_bytes(B,A,no,multi_label,max_labels). */
#define MYOLO_NMS_ERR_LABEL_CLASS 1
#define MYOLO_NMS_ERR_LABEL_COUNT 2
int64_t myolo_nms_labels_workspace_bytes(int B, int A, int no, int multi_label, int max_labels);
int myolo_nms_labels(const float* pred, int B, int A, int no, float conf_thres, float iou_thres, const int32_t* classes,
                     int n_classes, int agnostic, int multi_label, int max_det, int max_nms, float max_wh, const float* labels,
                     const int32_t* label_offsets, int max_labels, int32_t* err, float* out, int32_t* out_count, void* workspace,
                     int64_t workspace_bytes, void* stream);
/* detect.py:191-193: bilinear(align_corners=True) to (H,W) then argmax over C (first max wins).
 * logits: (B,C,h,w) NCHW fp32/fp16.  out: (B,H,W) int64 (out_dtype I64) or uint8 (U8). */
int myolo_seg_upsample_argmax(const void* logits, int dtype, int B, int C, int h, int w, int H, int W, void* out,
                              int out_dtype, void* stream);
/* autoShape's per-image class maps: for item b, F.interpolate(logits[b:b+1, :, top:top+rh, left:left+rw], (h0, w0), 'bilinear',
 * align_corners=True).argmax(1) (ties -> lowest class id; fp16 logits compare the fp16-rounded values, as torch's half interpolate returns
 * them) written as uint8 (h0, w0) at out + offset.  logits: (B,C,H,W) NCHW fp32/fp16, C <= 256.  items: DEVICE array of B
 * myolo_seg_crop_item, each window inside H x W; max_pixels: the largest h0 * w0, which sizes the grid.  One launch. */
typedef struct {
  int64_t offset;            /* byte offset of the item's (h0, w0) map in out */
  int32_t top, left, rh, rw; /* the window of the letterboxed image in the logits */
  int32_t h0, w0;            /* output size: the original image */
} myolo_seg_crop_item;
int myolo_seg_crop_upsample_argmax(const void* logits, int dtype, int B, int C, int H, int W, const myolo_seg_crop_item* items,
                                   int64_t max_pixels, uint8_t* out, void* stream);
/* F.interpolate(seg,(H,W),'bilinear',align_corners=True) on NCHW fp32 (materialised logits) */
int myolo_bilinear_nchw(const float* src, int B, int C, int h, int w, int H, int W, float* dst, void* stream);

/* ---- standalone kernels for per-op parity tests and ncu captures ---- */
/* standalone forward of one conv through the plan's own routing and launches: y = act(conv(x, W) + b) (+ residual), W and b the fp16 pack
 * and fp32 bias of fp32 master weights w [co][ci][k][k] with BatchNorm (gamma, beta, mean, var, eps; all four or none) folded in and the
 * conv bias (nullable) added, as myolo_plan_set_conv_weights packs them.  Views are channel slices of NHWC buffers (base of the buffer,
 * channels per pixel ctot, first channel c_off), as the plan passes them:
 *   x    (B,H,W) fp16 / fp32, ci rounded up to 16 channels (the padding channels hold zeros);
 *   y    (B,Ho,Wo) fp16 / fp32, co channels: exactly those are written;
 *   res  nullable, (B,Ho,Wo) fp16, co channels, added after the activation; it may alias y.
 * "same" padding dil*(k/2).  path: 0 as the plan, 1 wgmma (error when the op is not eligible), 2 CUDA-core, 3 wgmma with streamed weights
 * and one A box per tap (the layout path 1's weight residency and strip are checked against).  info (nullable): the 12 slots of
 * myolo_plan_conv_info. */
int myolo_conv_forward(const void* x, int x_dtype, int B, int H, int W, int x_ctot, int x_coff, void* y, int y_dtype, int y_ctot, int y_coff,
                       const void* res, int res_ctot, int res_coff, const float* w, int co, int ci, int k, int stride, int dil,
                       const float* gamma, const float* beta, const float* mean, const float* var, float eps, const float* bias, int act,
                       int path, int32_t* info, void* stream);
/* standalone backward of one conv through the train plan's own routing and launches (per-op tests).  Views are channel slices of NHWC
 * buffers (base of the buffer, channels per pixel ctot, first channel c_off), as the plan passes them:
 *   x     (B,H,W) fp16 / fp32, ci rounded up to 16 channels (the padding channels hold zeros);
 *   dy    (B,Ho,Wo) fp16 with co channels, or an fp32 head gradient with co rounded up to 16 (zero padding);
 *   gin   grad(in), nullable (no data gradient), x's dtype and channel count: ACCUMULATED into;
 *   w     fp32 master weights [co][ci][k][k]; dW (same layout) and dbias [co] (nullable) are ACCUMULATED into.
 * "same" padding dil*(k/2).  route: 0 as the plan, or MYOLO_CONV_BWD_* bits.  info (nullable) receives 16 slots:
 *   0  data gradient: 0 none, 1 small (generic kernel, fp32 weights), 2 wgmma conv, 3 CUDA-core conv
 *   1  weight gradient: 1 small, 2 mma.sync, 3 wgmma into dW, 4 wgmma through a packed buffer
 *   2  bias gradient: 0 none, 1 summed from fp32 dY, 2 from fp16 dY
 *   3-7  wgmma data gradient: kc, BN, CTAs per SM, weights resident, strip mode;  13-14: N tiles, padded output channels of the pack
 *   8-12 wgmma weight gradient: pixels per step Kc, N, row slabs, rows per slab, rows in all */
#define MYOLO_CONV_BWD_SIMT 1          /* data gradient on the CUDA-core conv (as MYOLO_FORCE_SIMT=1 does for a plan) */
#define MYOLO_CONV_BWD_NO_WGRAD_TC 2   /* weight gradient on the mma.sync kernel where the wgmma one would run */
int myolo_conv_backward(const void* x, int x_dtype, int B, int H, int W, int x_ctot, int x_coff, const void* dy, int dy_dtype, int dy_ctot,
                        int dy_coff, void* gin, int gin_ctot, int gin_coff, const float* w, int co, int ci, int k, int stride, int dil,
                        float* dW, float* dbias, int route, int32_t* info, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* MYOLO_H_ */
