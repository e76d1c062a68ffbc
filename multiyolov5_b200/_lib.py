"""ctypes binding of libmyolo_sm90a.so (C ABI: include/myolo.h).

There is no CPU / PyTorch fallback: if the shared library is missing or no sm_90 (H100) device is present every entry
point raises.  Build with `python -c "import __graft_entry__ as g; g.build()"` or `make -C multiyolov5_b200/csrc`.
"""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("MYOLO_LIB") or os.path.join(_HERE, "libmyolo_sm90a.so")   # MYOLO_LIB: developer builds (e.g. the clock64 timeline variant)

F16, F32, U8, I64 = 0, 1, 2, 3
ACT_NONE, ACT_SILU, ACT_SIGMOID = 0, 1, 2
(OP_INPUT_FOCUS, OP_CONV, OP_UPSAMPLE_NEAREST, OP_SPP_POOL, OP_BILINEAR, OP_REGION_SUM, OP_REGION_COMBINE, OP_CHANNEL_SCALE,
 OP_ADD, OP_DETECT_DECODE, OP_SEG_UPSAMPLE, OP_BROADCAST, OP_FOCUS_CONV, OP_BN_ACT, OP_ACT, OP_CHANNEL_SCALE_OOP, OP_DROPOUT) = range(1, 18)
CONV_FORCE_SIMT = 1
OP_GROUP_HEAD, OP_GROUP_MEMBER = 2, 4      # include/myolo.h: consecutive ops of one kind executed as one launch

EXPORTS = [
    "myolo_abi_version", "myolo_last_error", "myolo_device_info", "myolo_plan_create", "myolo_plan_destroy",
    "myolo_plan_set_conv_weights", "myolo_plan_repack_weights", "myolo_plan_forward", "myolo_plan_read_view", "myolo_plan_last_launch_count",
    "myolo_plan_profile", "myolo_nms_workspace_bytes", "myolo_nms", "myolo_seg_upsample_argmax", "myolo_bilinear_nchw",
    "myolo_conv_bn_silu", "myolo_plan_set_bn", "myolo_plan_set_conv_grad", "myolo_plan_train_forward", "myolo_plan_backward",
    "myolo_grads_check_finite", "myolo_sgd_step", "myolo_conv_wgrad", "myolo_letterbox", "myolo_seg_lut_blend", "myolo_seg_metrics", "myolo_plan_backward_seg_ce", "myolo_plan_read_grad_view", "myolo_plan_set_seed", "myolo_plan_train_forward_multi", "myolo_plan_backward_multi", "myolo_plan_conv_info", "myolo_allreduce_grads", "myolo_det_loss", "myolo_det_loss_workspace_bytes", "myolo_plan_set_defer_running", "myolo_plan_apply_running",
]


class BufDesc(C.Structure):
    _fields_ = [("h", C.c_int32), ("w", C.c_int32), ("c", C.c_int32), ("dtype", C.c_int32), ("offset", C.c_int64)]


class View(C.Structure):
    _fields_ = [("buf", C.c_int32), ("c_off", C.c_int32), ("c", C.c_int32)]


class Op(C.Structure):
    _fields_ = [("kind", C.c_int32), ("in_", View), ("in2", View), ("out", View), ("k", C.c_int32), ("stride", C.c_int32),
                ("dil", C.c_int32), ("act", C.c_int32), ("flags", C.c_int32), ("weight_slot", C.c_int32),
                ("aux", C.c_int32 * 8), ("faux", C.c_float * 4)]


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
    L.myolo_device_info.argtypes = [C.c_char_p, C.POINTER(i32), C.POINTER(i32), C.POINTER(i32)]
    L.myolo_plan_create.argtypes = [C.POINTER(Op), i32, C.POINTER(BufDesc), i32, C.POINTER(C.c_int32), i32, i32, i32, i32, i64,
                                    i32, C.POINTER(vp)]
    L.myolo_plan_destroy.argtypes = [vp]
    L.myolo_plan_destroy.restype = None
    L.myolo_plan_set_conv_weights.argtypes = [vp, i32, vp, i32, i32, i32, vp, vp, vp, vp, f32, vp, vp]
    L.myolo_plan_repack_weights.argtypes = [vp, vp]
    L.myolo_plan_forward.argtypes = [vp, vp, i32, vp, C.POINTER(vp), vp, i32, vp, vp]
    L.myolo_plan_read_view.argtypes = [vp, View, vp, vp]
    L.myolo_plan_last_launch_count.argtypes = [vp]
    L.myolo_plan_last_launch_count.restype = i64
    L.myolo_plan_profile.argtypes = [vp, vp, i32, vp, C.POINTER(vp), vp, i32, vp, C.POINTER(f32), vp]
    L.myolo_plan_set_bn.argtypes = [vp, i32, i32, vp, vp, vp, vp, vp, vp, f32, f32]
    L.myolo_plan_set_conv_grad.argtypes = [vp, i32, vp, vp]
    L.myolo_plan_train_forward.argtypes = [vp, vp, i32, C.POINTER(vp), vp, vp]
    L.myolo_plan_backward.argtypes = [vp, C.POINTER(vp), vp, vp]
    L.myolo_letterbox.argtypes = [vp, i32, i32, i32, i32, i32, i32, i32, i32, i32, vp, vp, i32, i32, i32, vp]
    L.myolo_seg_lut_blend.argtypes = [vp, i32, i64, vp, i32, i32, i32, vp, vp, f32, f32, vp, vp]
    L.myolo_seg_metrics.argtypes = [vp, i32, vp, i64, i32, vp, vp]
    L.myolo_plan_backward_seg_ce.argtypes = [vp, vp, i32, f32, vp, vp, vp]
    L.myolo_plan_read_grad_view.argtypes = [vp, View, vp, vp]
    L.myolo_plan_set_seed.argtypes = [vp, C.c_uint64]
    L.myolo_plan_set_defer_running.argtypes = [vp, i32]
    L.myolo_plan_apply_running.argtypes = [vp, vp]
    L.myolo_plan_train_forward_multi.argtypes = [vp, vp, i32, C.POINTER(vp), C.POINTER(vp), vp]
    L.myolo_plan_backward_multi.argtypes = [vp, C.POINTER(vp), C.POINTER(vp), vp]
    L.myolo_conv_wgrad.argtypes = [vp, vp, i32, i32, i32, i32, i32, i32, i32, i32, vp, i32, vp]
    L.myolo_grads_check_finite.argtypes = [vp, i64, vp, vp]
    L.myolo_sgd_step.argtypes = [vp, vp, vp, vp, i64, C.POINTER(f32), C.POINTER(f32), i32, f32, i32, vp, vp, i32, vp]
    L.myolo_allreduce_grads.argtypes = [vp, i64, vp, vp]
    L.myolo_det_loss_workspace_bytes.argtypes = [i32, i32, i32, C.POINTER(C.c_int32), C.POINTER(C.c_int32)]
    L.myolo_det_loss_workspace_bytes.restype = i64
    L.myolo_det_loss.argtypes = [C.POINTER(vp), C.POINTER(vp), vp, i32, i32, i32, i32, i32, C.POINTER(C.c_int32), C.POINTER(C.c_int32),
                                 C.POINTER(f32), C.POINTER(f32), f32, f32, f32, f32, f32, f32, f32, f32, vp, vp, vp, i64, vp]
    L.myolo_plan_conv_info.argtypes = [vp, i32, C.POINTER(C.c_int32)]
    L.myolo_nms_workspace_bytes.argtypes = [i32, i32, i32, i32]
    L.myolo_nms_workspace_bytes.restype = i64
    L.myolo_nms.argtypes = [vp, i32, i32, i32, f32, f32, vp, i32, i32, i32, i32, i32, f32, vp, vp, vp, i64, vp]
    L.myolo_seg_upsample_argmax.argtypes = [vp, i32, i32, i32, i32, i32, i32, i32, vp, i32, vp]
    L.myolo_bilinear_nchw.argtypes = [vp, i32, i32, i32, i32, i32, i32, vp, vp]
    L.myolo_conv_bn_silu.argtypes = [vp, i32, i32, i32, i32, vp, i32, i32, i32, i32, vp, vp, vp, vp, f32, vp, i32, vp, vp, i32, vp]
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
