"""ctypes binding of libmyolo_sm90a.so (C ABI: include/myolo.h).

There is no CPU / PyTorch fallback: if the shared library is missing or no sm_90 (H100) device is present every entry
point raises.  Build with `python -c "import __graft_entry__ as g; g.build()"` or `make -C multiyolov5_b200/csrc`.
"""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("MYOLO_LIB") or os.path.join(_HERE, "libmyolo_sm90a.so")   # MYOLO_LIB: developer builds (e.g. the clock64 timeline variant)

F16, F32, U8, I64, F64 = 0, 1, 2, 3, 4     # F64: myolo_anchor_metric only
ACT_NONE, ACT_SILU, ACT_SIGMOID = 0, 1, 2
OP_INPUT_FOCUS = 1
OP_CONV = 2
OP_UPSAMPLE_NEAREST = 3
OP_SPP_POOL = 4
OP_BILINEAR = 5
OP_REGION_SUM = 6
OP_REGION_COMBINE = 7
OP_CHANNEL_SCALE = 8
OP_ADD = 9
OP_DETECT_DECODE = 10
OP_SEG_UPSAMPLE = 11
OP_BROADCAST = 12
OP_BN_ACT = 14      # 13 is retired
OP_ACT = 15
OP_CHANNEL_SCALE_OOP = 16
OP_DROPOUT = 17
OP_GROUP_HEAD, OP_GROUP_MEMBER = 2, 4      # include/myolo.h: consecutive ops of one kind executed as one launch

EXPORTS = [
    "myolo_abi_version", "myolo_last_error", "myolo_plan_create", "myolo_plan_destroy",
    "myolo_plan_set_conv_weights", "myolo_plan_repack_weights", "myolo_plan_forward", "myolo_plan_read_view", "myolo_plan_last_launch_count",
    "myolo_plan_profile", "myolo_nms_workspace_bytes", "myolo_nms", "myolo_seg_upsample_argmax", "myolo_bilinear_nchw",
    "myolo_plan_set_bn", "myolo_plan_set_conv_grad", "myolo_grads_check_finite", "myolo_sgd_step", "myolo_letterbox", "myolo_seg_lut_blend", "myolo_seg_metrics", "myolo_plan_backward_seg_ce", "myolo_plan_read_grad_view", "myolo_plan_set_seed", "myolo_plan_train_forward_multi", "myolo_plan_backward_multi", "myolo_plan_conv_info", "myolo_allreduce_grads", "myolo_det_loss", "myolo_det_loss_workspace_bytes", "myolo_plan_set_defer_running", "myolo_plan_apply_running",
    "myolo_resize_u8", "myolo_augment_seg", "myolo_det_match", "myolo_det_ap", "myolo_det_ap_workspace_bytes",
    "myolo_resize_area_u8", "myolo_resize_bilinear", "myolo_plan_create_shared", "myolo_augment_det_hw", "myolo_adam_step",
    "myolo_adam_scalars", "myolo_ema_update", "myolo_plan_set_extra", "myolo_collate_quad", "myolo_plan_set_bn_sync",
    "myolo_plan_backward_seg_ohem", "myolo_seg_ohem_loss", "myolo_seg_ohem_loss_backward", "myolo_seg_ohem_loss_workspace_bytes",
    "myolo_anchor_metric", "myolo_anchor_metric_workspace_bytes", "myolo_anchor_evolve", "myolo_anchor_evolve_workspace_bytes",
    "myolo_kmeans", "myolo_kmeans_workspace_bytes", "myolo_class_weights", "myolo_image_weights", "myolo_weighted_draw",
    "myolo_plan_backward_seg_loss", "myolo_seg_focal_loss", "myolo_seg_focal_loss_backward", "myolo_seg_focal_loss_workspace_bytes",
    "myolo_conv_backward", "myolo_conv_forward", "myolo_plan_forward_pass", "myolo_scale_img", "myolo_detect_boxes",
    "myolo_letterbox_items", "myolo_scale_boxes", "myolo_seg_crop_upsample_argmax", "myolo_nms_labels", "myolo_nms_labels_workspace_bytes",
    "myolo_confusion_update", "myolo_seg_ensemble",
]
REDUCTION_MEAN, REDUCTION_SUM = 0, 1        # include/myolo.h: MYOLO_REDUCTION_* of myolo_seg_focal_loss
DET_ERR_TARGET_CLASS, DET_ERR_PRED_CLASS, DET_ERR_LABELS = 1, 2, 4     # include/myolo.h: bits of myolo_det_match's error word
NMS_ERR_LABEL_CLASS, NMS_ERR_LABEL_COUNT = 1, 2                          # include/myolo.h: bits of myolo_nms_labels' error word
KMEANS_MAX_ITER, KMEANS_BAD_INDEX = 1, 2                                 # include/myolo.h: bits of myolo_kmeans' status word
IW_BAD_CLASS, IW_TOTAL_NONPOS, IW_TOTAL_NONFINITE = 1, 2, 4              # include/myolo.h: bits of the image-weights status word
ENSEMBLE_MAX = 8                                                         # include/myolo.h MYOLO_ENSEMBLE_MAX
IW_NC_MAX = 1024                                                         # include/myolo.h MYOLO_IW_NC_MAX
DET_LOSS_NA_MAX = 10                                                     # include/myolo.h MYOLO_DET_LOSS_NA_MAX
CONV_BWD_SIMT, CONV_BWD_NO_WGRAD_TC = 1, 2                               # include/myolo.h: route bits of myolo_conv_backward


class BufDesc(C.Structure):
    _fields_ = [("h", C.c_int32), ("w", C.c_int32), ("c", C.c_int32), ("dtype", C.c_int32), ("offset", C.c_int64)]


class View(C.Structure):
    _fields_ = [("buf", C.c_int32), ("c_off", C.c_int32), ("c", C.c_int32)]


class Op(C.Structure):
    _fields_ = [("kind", C.c_int32), ("in_", View), ("in2", View), ("out", View), ("k", C.c_int32), ("stride", C.c_int32),
                ("dil", C.c_int32), ("act", C.c_int32), ("flags", C.c_int32), ("weight_slot", C.c_int32),
                ("aux", C.c_int32 * 8), ("faux", C.c_float * 4)]


class AugWarp(C.Structure):
    _fields_ = [("src", C.c_void_p * 4), ("rect", (C.c_int32 * 4) * 4), ("off", (C.c_int32 * 2) * 4), ("src_w", C.c_int32 * 4),
                ("n_tiles", C.c_int32), ("reserved", C.c_int32), ("minv", C.c_double * 6)]


class AugItem(C.Structure):
    _fields_ = [("warp", AugWarp * 2), ("mix_r", C.c_double), ("mix_q", C.c_double), ("n_warps", C.c_int32), ("flipud", C.c_int32),
                ("fliplr", C.c_int32), ("reserved", C.c_int32), ("lut", (C.c_uint8 * 256) * 3)]


class SegItem(C.Structure):
    _fields_ = [("img", C.c_void_p), ("mask", C.c_void_p), ("H0", C.c_int32), ("W0", C.c_int32), ("flip", C.c_int32), ("kx", C.c_int32),
                ("ky", C.c_int32), ("col", C.c_int32), ("row", C.c_int32), ("mcol", C.c_int32), ("mrow", C.c_int32),
                ("order", C.c_int32 * 4), ("factor", C.c_float * 3), ("hue_shift", C.c_int32), ("reserved", C.c_int32),
                ("lsum", C.c_uint64), ("lut", C.c_int32 * 256)]


class EmaChunk(C.Structure):
    """include/myolo.h myolo_ema_chunk: elements [ema, ema + n) of one EMA entry (dtype F32 / F16) and [src, src + n) of its fp32 source"""
    _fields_ = [("ema", C.c_void_p), ("src", C.c_void_p), ("n", C.c_int32), ("dtype", C.c_int32)]


EMA_CHUNK = 8192        # include/myolo.h MYOLO_EMA_CHUNK: entries are cut at multiples of it, one CTA per chunk


class MyoloError(RuntimeError):
    pass


_lib = None


def lib():
    """Loads the shared library (once).  Fails loudly when it has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.isfile(LIB_PATH):
        raise MyoloError(f"{LIB_PATH} is missing - build it first (`make -C multiyolov5_b200/csrc` or __graft_entry__.build()); "
                         "this package has no CPU/PyTorch fallback path")
    L = C.CDLL(LIB_PATH)
    vp, i32, i64, f32 = C.c_void_p, C.c_int, C.c_int64, C.c_float
    L.myolo_abi_version.restype = i32
    L.myolo_last_error.restype = C.c_char_p
    L.myolo_plan_create.argtypes = [C.POINTER(Op), i32, C.POINTER(BufDesc), i32, C.POINTER(C.c_int32), i32, i32, i32, i32, i64,
                                    i32, C.POINTER(vp)]
    L.myolo_plan_create_shared.argtypes = [C.POINTER(Op), i32, C.POINTER(BufDesc), i32, C.POINTER(C.c_int32), i32, i32, i32, i32, i64,
                                           i32, vp, vp, i64, C.POINTER(vp)]
    L.myolo_plan_destroy.argtypes = [vp]
    L.myolo_plan_destroy.restype = None
    L.myolo_plan_set_conv_weights.argtypes = [vp, i32, vp, i32, i32, i32, vp, vp, vp, vp, f32, vp, vp]
    L.myolo_plan_repack_weights.argtypes = [vp, vp]
    L.myolo_plan_forward.argtypes = [vp, vp, i32, vp, C.POINTER(vp), vp, i32, vp, vp]
    L.myolo_plan_forward_pass.argtypes = [vp, vp, i32, vp, i32, i32, f32, i32, vp, i32, vp, vp]
    L.myolo_seg_ensemble.argtypes = [C.POINTER(vp), i32, vp, i32, vp, vp]
    L.myolo_plan_read_view.argtypes = [vp, View, vp, vp]
    L.myolo_plan_last_launch_count.argtypes = [vp]
    L.myolo_plan_last_launch_count.restype = i64
    L.myolo_plan_profile.argtypes = [vp, vp, i32, vp, C.POINTER(vp), vp, i32, vp, C.POINTER(f32), vp]
    L.myolo_plan_set_bn.argtypes = [vp, i32, i32, vp, vp, vp, vp, vp, vp, f32, f32]
    L.myolo_plan_set_conv_grad.argtypes = [vp, i32, vp, vp]
    L.myolo_letterbox.argtypes = [vp, i32, i32, i32, i32, i32, i32, i32, i32, i32, vp, vp, i32, i32, i32, vp]
    L.myolo_resize_u8.argtypes = [vp, i32, i32, vp, i32, i32, vp]
    L.myolo_resize_area_u8.argtypes = [vp, i32, i32, vp, i32, i32, vp]
    L.myolo_resize_bilinear.argtypes = [vp, i32, i32, i32, i32, i32, vp, i32, i32, i32, vp]
    L.myolo_scale_img.argtypes = [vp, i32, i32, i32, i32, i32, vp, i32, i32, i32, i32, i32, f32, vp]
    L.myolo_augment_det_hw.argtypes = [vp, i32, i32, i32, vp, i32, vp]
    L.myolo_collate_quad.argtypes = [vp, i32, i32, i32, vp, vp, i32, vp]
    L.myolo_augment_seg.argtypes = [vp, i32, i32, i32, i32, i32, vp, vp, vp, i32, vp, vp]
    L.myolo_seg_lut_blend.argtypes = [vp, i32, i64, vp, i32, i32, i32, vp, vp, f32, f32, vp, vp, i32, vp, vp]
    L.myolo_detect_boxes.argtypes = [vp, vp, i32, i32, vp, i32, vp, vp, vp]
    L.myolo_scale_boxes.argtypes = [vp, vp, i32, i32, vp, vp, vp, vp, vp]
    L.myolo_letterbox_items.argtypes = [vp, vp, i32, i32, i32, vp, i32, vp]
    L.myolo_seg_crop_upsample_argmax.argtypes = [vp, i32, i32, i32, i32, i32, vp, i64, vp, vp]
    L.myolo_seg_metrics.argtypes = [vp, i32, vp, i64, i32, vp, vp]
    L.myolo_det_match.argtypes = [vp, vp, i32, i32, vp, i32, i32, i32, vp, vp, i32, vp, vp, vp, vp, vp, vp, vp]
    L.myolo_confusion_update.argtypes = [vp, vp, i32, i32, vp, i32, i32, i32, vp, i32, f32, f32, i32, vp, vp, vp]
    L.myolo_det_ap_workspace_bytes.argtypes = [i32, i32, i32]
    L.myolo_det_ap_workspace_bytes.restype = i64
    L.myolo_det_ap.argtypes = [vp, vp, vp, vp, i32, i32, i32, vp, vp, vp, vp, vp, vp, vp, vp, i64, vp]
    L.myolo_plan_backward_seg_ce.argtypes = [vp, vp, i32, f32, vp, vp, vp]
    L.myolo_plan_backward_seg_ohem.argtypes = [vp, vp, i32, f32, f32, vp, vp, vp]
    L.myolo_seg_ohem_loss_workspace_bytes.argtypes = [i32, i32, i32]
    L.myolo_seg_ohem_loss_workspace_bytes.restype = i64
    L.myolo_seg_ohem_loss.argtypes = [vp, vp, i32, i32, i32, i32, i32, f32, vp, vp, i64, vp]
    L.myolo_seg_ohem_loss_backward.argtypes = [vp, vp, i32, i32, i32, i32, i32, vp, vp, vp, i64, vp]
    L.myolo_plan_backward_seg_loss.argtypes = [vp, vp, i32, vp, f32, f32, vp, vp, vp]
    L.myolo_seg_focal_loss_workspace_bytes.argtypes = []
    L.myolo_seg_focal_loss_workspace_bytes.restype = i64
    L.myolo_seg_focal_loss.argtypes = [vp, vp, i32, i32, i32, i32, i32, vp, f32, i32, vp, vp, i64, vp]
    L.myolo_seg_focal_loss_backward.argtypes = [vp, vp, i32, i32, i32, i32, i32, vp, f32, vp, vp, vp, i64, vp]
    L.myolo_anchor_metric_workspace_bytes.argtypes = []
    L.myolo_anchor_metric_workspace_bytes.restype = i64
    L.myolo_anchor_metric.argtypes = [vp, i32, i64, vp, i32, i32, C.c_double, vp, vp, i64, vp]
    L.myolo_anchor_evolve_workspace_bytes.argtypes = [i64]
    L.myolo_anchor_evolve_workspace_bytes.restype = i64
    L.myolo_anchor_evolve.argtypes = [vp, i64, vp, i32, vp, i32, C.c_double, vp, vp, vp, vp, vp, i64, vp]
    L.myolo_kmeans_workspace_bytes.argtypes = [i64, i32, i32]
    L.myolo_kmeans_workspace_bytes.restype = i64
    L.myolo_kmeans.argtypes = [vp, i64, i32, vp, i32, i32, C.c_double, i32, vp, vp, vp, vp, vp, vp, vp, i64, vp]
    L.myolo_class_weights.argtypes = [vp, i64, i32, vp, vp, vp, vp]
    L.myolo_image_weights.argtypes = [vp, vp, i64, vp, i32, vp, vp, vp]
    L.myolo_weighted_draw.argtypes = [vp, vp, i64, vp, vp, vp, vp, vp]
    L.myolo_plan_read_grad_view.argtypes = [vp, View, vp, vp]
    L.myolo_plan_set_seed.argtypes = [vp, C.c_uint64]
    L.myolo_plan_set_defer_running.argtypes = [vp, i32]
    L.myolo_plan_apply_running.argtypes = [vp, vp]
    L.myolo_plan_set_bn_sync.argtypes = [vp, vp, C.POINTER(C.c_int32), i32]
    L.myolo_plan_train_forward_multi.argtypes = [vp, vp, i32, C.POINTER(vp), C.POINTER(vp), vp]
    L.myolo_plan_backward_multi.argtypes = [vp, C.POINTER(vp), C.POINTER(vp), vp]
    L.myolo_conv_backward.argtypes = [vp, i32, i32, i32, i32, i32, i32, vp, i32, i32, i32, vp, i32, i32, vp, i32, i32, i32, i32, i32, vp, vp,
                                      i32, C.POINTER(C.c_int32), vp]
    L.myolo_grads_check_finite.argtypes = [vp, i64, vp, vp]
    L.myolo_sgd_step.argtypes = [vp, vp, vp, vp, i64, C.POINTER(f32), C.POINTER(f32), i32, f32, i32, vp, vp, i32, vp]
    L.myolo_adam_step.argtypes = [vp, vp, vp, vp, vp, i64, C.POINTER(C.c_double), C.POINTER(f32), i32, C.c_double, C.c_double, C.c_double,
                                  vp, vp, vp, i32, vp]
    L.myolo_adam_scalars.argtypes = [vp, i64, C.c_double, C.c_double, C.c_double, vp, vp, vp, vp, vp]
    L.myolo_ema_update.argtypes = [vp, i32, C.c_double, vp]
    L.myolo_plan_set_extra.argtypes = [vp, i32, vp, i32, vp]
    L.myolo_allreduce_grads.argtypes = [vp, i64, vp, vp]
    L.myolo_det_loss_workspace_bytes.argtypes = [i32, i32, i32, C.POINTER(C.c_int32), C.POINTER(C.c_int32)]
    L.myolo_det_loss_workspace_bytes.restype = i64
    L.myolo_det_loss.argtypes = [C.POINTER(vp), C.POINTER(vp), vp, i32, i32, i32, i32, i32, C.POINTER(C.c_int32), C.POINTER(C.c_int32),
                                 C.POINTER(f32), C.POINTER(f32), f32, f32, f32, f32, f32, f32, f32, f32, vp, vp, vp, i64, vp]
    L.myolo_plan_conv_info.argtypes = [vp, i32, C.POINTER(C.c_int32)]
    L.myolo_nms_workspace_bytes.argtypes = [i32, i32, i32, i32]
    L.myolo_nms_workspace_bytes.restype = i64
    L.myolo_nms.argtypes = [vp, i32, i32, i32, f32, f32, vp, i32, i32, i32, i32, i32, f32, vp, vp, vp, i64, vp]
    L.myolo_nms_labels_workspace_bytes.argtypes = [i32, i32, i32, i32, i32]
    L.myolo_nms_labels_workspace_bytes.restype = i64
    L.myolo_nms_labels.argtypes = [vp, i32, i32, i32, f32, f32, vp, i32, i32, i32, i32, i32, f32, vp, vp, i32, vp, vp, vp, vp, i64, vp]
    L.myolo_seg_upsample_argmax.argtypes = [vp, i32, i32, i32, i32, i32, i32, i32, vp, i32, vp]
    L.myolo_bilinear_nchw.argtypes = [vp, i32, i32, i32, i32, i32, i32, vp, vp]
    L.myolo_conv_forward.argtypes = [vp, i32, i32, i32, i32, i32, i32, vp, i32, i32, i32, vp, i32, i32, vp, i32, i32, i32, i32, i32, vp, vp, vp,
                                     vp, f32, vp, i32, i32, C.POINTER(C.c_int32), vp]
    for name in EXPORTS:
        getattr(L, name)  # AttributeError here == header / library mismatch
    if L.myolo_abi_version() != 1:
        raise MyoloError("libmyolo_sm90a ABI version mismatch")
    _lib = L
    return L


def check(rc: int):
    if rc != 0:
        raise MyoloError(f"libmyolo_sm90a error {rc}: {lib().myolo_last_error().decode(errors='replace')}")


def stream_ptr():
    import torch
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def ptr(t):
    return C.c_void_p(t.data_ptr()) if t is not None else C.c_void_p(0)


def torch_dtype_code(dt):
    import torch
    return {torch.float16: F16, torch.float32: F32, torch.uint8: U8, torch.int64: I64}[dt]
