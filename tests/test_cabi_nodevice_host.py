"""CPU: without a CUDA device every standalone C entry point that launches work fails with MYOLO_E_NODEVICE and says why, once its
arguments pass the checks that come before the device check; the workspace-size queries that need no device return their sizes."""
import ctypes as C

import pytest
import torch

if torch.cuda.is_available():
    pytest.skip("these calls pass host buffers where the library expects device memory", allow_module_level=True)

from multiyolov5_b200 import _lib

E_INVALID, E_NODEVICE = -1, -3
_BUF = C.create_string_buffer(1 << 12)
P = C.addressof(_BUF)                     # non-null, 16-byte aligned: never dereferenced, the device check comes first
LR32, WD32, LR64 = (C.c_float * 4)(0.01, 0.01, 0.01), (C.c_float * 4)(0.0, 5e-4, 0.0), (C.c_double * 4)(0.01, 0.01, 0.01)
WS = 1 << 30                              # workspace_bytes: more than any call below needs
U8, F32, F64 = _lib.U8, _lib.F32, _lib.F64
CALLS = {
    "myolo_letterbox": (P, 1, 8, 8, 8, 8, 0, 0, 8, 8, None, P, U8, 1, 1, None),
    "myolo_letterbox_items": (P, P, 1, 8, 8, P, U8, None),
    "myolo_resize_u8": (P, 8, 8, P, 4, 4, None),
    "myolo_resize_area_u8": (P, 8, 8, P, 4, 4, None),
    "myolo_augment_det_hw": (P, 1, 8, 8, P, U8, None),
    "myolo_resize_bilinear": (P, U8, 1, 3, 8, 8, P, F32, 4, 4, None),
    "myolo_scale_img": (P, F32, 1, 3, 8, 8, P, 4, 4, 8, 8, 0, 0.447, None),
    "myolo_collate_quad": (P, 4, 8, 8, P, P, U8, None),
    "myolo_augment_seg": (P, 1, 8, 8, 8, 8, P, P, P, F32, P, None),
    "myolo_seg_lut_blend": (P, U8, 64, P, 19, 3, 0, P, None, 0.4, 0.6, None, None, 0, None, None),
    "myolo_detect_boxes": (P, P, 1, 300, P, 10, None, None, None),
    "myolo_scale_boxes": (P, P, 1, 300, P, None, None, None, None),
    "myolo_seg_metrics": (P, U8, P, 64, 19, P, None),
    "myolo_det_match": (P, P, 1, 300, P, 0, 64, 64, P, P, 0, P, P, P, P, P, P, None),
    "myolo_confusion_update": (P, P, 1, 300, P, 0, 64, 64, P, 10, 0.25, 0.45, 1, P, P, None),
    "myolo_det_ap": (P, P, P, P, 1, 300, 10, P, P, P, P, P, P, P, P, WS, None),
    "myolo_grads_check_finite": (P, 64, P, None),
    "myolo_sgd_step": (P, P, P, P, 64, LR32, WD32, 3, 0.937, 1, P, None, 1, None),
    "myolo_adam_step": (P, P, P, P, P, 64, LR64, WD32, 3, 0.937, 0.999, 1e-8, P, P, None, 1, None),
    "myolo_adam_scalars": (P, 1, 0.01, 0.937, 0.999, P, P, P, P, None),
    "myolo_ema_update": (P, 1, 0.999, None),
    "myolo_seg_ohem_loss": (P, P, 1, 19, 8, 8, 255, 0.36, P, P, WS, None),
    "myolo_seg_ohem_loss_backward": (P, P, 1, 19, 8, 8, 255, P, P, P, WS, None),
    "myolo_seg_focal_loss": (P, P, 1, 19, 8, 8, 255, None, 2.0, _lib.REDUCTION_MEAN, P, P, WS, None),
    "myolo_seg_focal_loss_backward": (P, P, 1, 19, 8, 8, 255, None, 2.0, P, P, P, WS, None),
    "myolo_anchor_metric": (P, F32, 100, P, F64, 9, 0.25, P, P, WS, None),
    "myolo_anchor_evolve": (P, 100, P, 9, P, 10, 0.25, P, P, P, P, P, WS, None),
    "myolo_kmeans": (P, 100, 2, P, 9, 4, 1e-5, 30, P, P, P, P, P, P, P, WS, None),
    "myolo_class_weights": (P, 100, 10, P, P, P, None),
    "myolo_image_weights": (P, P, 10, P, 10, P, P, None),
    "myolo_weighted_draw": (P, P, 10, P, P, P, P, None),
}


def _set_other_error(L):
    """leaves a known message behind (a host-side argument check), so a message read afterwards is the next call's own"""
    assert L.myolo_nms(None, 1, 1, 6, 0.25, 0.45, None, 0, 0, 0, 1, 1, 0.0, None, None, None, 0, None) == E_INVALID
    return L.myolo_last_error()


@pytest.mark.parametrize("name", sorted(CALLS))
def test_entry_point_without_device_fails_with_nodevice(name):
    L = _lib.lib()
    other = _set_other_error(L)
    assert getattr(L, name)(*CALLS[name]) == E_NODEVICE
    msg = L.myolo_last_error()
    assert msg and msg != other, msg


def test_anchor_evolve_workspace_bytes_without_device_is_minus_one():
    L = _lib.lib()                        # the size depends on the device's SM count and occupancy
    other = _set_other_error(L)
    assert L.myolo_anchor_evolve_workspace_bytes(1000) == -1
    msg = L.myolo_last_error()
    assert msg and msg != other, msg


@pytest.mark.parametrize("name,args,expected", [
    ("myolo_det_ap_workspace_bytes", (1, 1, 1), 11264),
    ("myolo_det_ap_workspace_bytes", (8, 300, 10), 355584),
    ("myolo_det_ap_workspace_bytes", (5000, 300, 10), 216546048),
    ("myolo_det_ap_workspace_bytes", (0, 300, 10), 0),
    ("myolo_det_ap_workspace_bytes", (8, 0, 10), 0),
    ("myolo_det_ap_workspace_bytes", (8, 300, 0), 0),
    ("myolo_seg_ohem_loss_workspace_bytes", (1, 1, 1), 4612),
    ("myolo_seg_ohem_loss_workspace_bytes", (2, 64, 128), 70144),
    ("myolo_seg_ohem_loss_workspace_bytes", (16, 512, 1024), 33566976),
    ("myolo_seg_focal_loss_workspace_bytes", (), 256),
    ("myolo_anchor_metric_workspace_bytes", (), 10240),
    ("myolo_kmeans_workspace_bytes", (1, 1, 1), 512),
    ("myolo_kmeans_workspace_bytes", (1000, 9, 32), 41216),
    ("myolo_kmeans_workspace_bytes", (100000, 9, 64), 7192832),
    ("myolo_kmeans_workspace_bytes", ((1 << 30) - 1, 9, 1), 1174405632),
    ("myolo_kmeans_workspace_bytes", (0, 9, 1), -1),
    ("myolo_kmeans_workspace_bytes", (1 << 30, 9, 1), -1),
    ("myolo_kmeans_workspace_bytes", (10, 0, 1), -1),
    ("myolo_kmeans_workspace_bytes", (10, 9, 0), -1),
])
def test_workspace_bytes_need_no_device(name, args, expected):
    assert getattr(_lib.lib(), name)(*args) == expected
