"""Device-side pre-process behind the reference's names (SURVEY.md section 8f rank 1):

    letterbox(img, new_shape, color, auto, scaleFill, scaleup, stride) -> (img, ratio, (dw, dh))     reference utils/datasets.py:818-848
    preprocess(img0, img_size, stride, half)  -> (1|B,3,H,W) float tensor in [0,1]                     :185-189 + detect.py:135-137

`img` is a uint8 HWC BGR frame (numpy array or torch tensor; a CPU input is uploaded as uint8 - 4x less than the fp32 the reference
ships to the GPU); the resize (OpenCV's 8-bit INTER_LINEAR arithmetic, bit exact), the 114 border, the channel swap, the transpose and
the /255 run in ONE kernel of libmyolo_sm90a.  The host only does the reference's shape arithmetic.
"""
import ctypes as C

import numpy as np
import torch

from .. import _lib


def letterbox_geometry(shape, new_shape=(640, 640), auto=True, scaleFill=False, scaleup=True, stride=32):
    """host arithmetic of the reference's letterbox: ((new_w, new_h), ratio, (dw, dh), (top, bottom, left, right))"""
    if isinstance(new_shape, int):
        new_shape = (new_shape, new_shape)
    r = min(new_shape[0] / shape[0], new_shape[1] / shape[1])
    if not scaleup:
        r = min(r, 1.0)
    ratio = r, r
    new_unpad = int(round(shape[1] * r)), int(round(shape[0] * r))
    dw, dh = new_shape[1] - new_unpad[0], new_shape[0] - new_unpad[1]
    if auto:
        dw, dh = np.mod(dw, stride), np.mod(dh, stride)
    elif scaleFill:
        dw, dh = 0.0, 0.0
        new_unpad = (new_shape[1], new_shape[0])
        ratio = new_shape[1] / shape[1], new_shape[0] / shape[0]
    dw /= 2
    dh /= 2
    top, bottom = int(round(dh - 0.1)), int(round(dh + 0.1))
    left, right = int(round(dw - 0.1)), int(round(dw + 0.1))
    return new_unpad, ratio, (dw, dh), (top, bottom, left, right)


def _as_device_frames(img):
    t = torch.from_numpy(np.ascontiguousarray(img)) if isinstance(img, np.ndarray) else img
    assert t.dtype == torch.uint8 and t.dim() in (3, 4) and t.shape[-1] == 3, "expected uint8 (H,W,3) or (B,H,W,3) BGR frames"
    if not t.is_cuda:
        t = t.pin_memory().cuda(non_blocking=True) if torch.cuda.is_available() else t
    if not t.is_cuda:
        raise _lib.MyoloError("letterbox needs a CUDA device: multiyolov5_b200 has no CPU path")
    return t.contiguous()


def _run(frames, geom, color, out_dtype, chw, swap_rb):
    batched = frames.dim() == 4
    f4 = frames if batched else frames[None]
    B, H0, W0, _ = f4.shape
    (rw, rh), _, _, (top, bottom, left, right) = geom
    H, W = rh + top + bottom, rw + left + right
    shape = (B, 3, H, W) if chw else (B, H, W, 3)
    out = torch.empty(shape, dtype=out_dtype, device=frames.device)
    pad = (C.c_int32 * 3)(*[int(c) for c in color])
    _lib.check(_lib.lib().myolo_letterbox(_lib.ptr(f4), B, H0, W0, rw, rh, top, left, H, W, pad, _lib.ptr(out), _lib.torch_dtype_code(out_dtype),
                                          int(chw), int(swap_rb), _lib.stream_ptr()))
    return out if batched else out[0]


def letterbox(img, new_shape=(640, 640), color=(114, 114, 114), auto=True, scaleFill=False, scaleup=True, stride=32):
    """Resize and pad while meeting stride-multiple constraints; returns (uint8 HWC frame on the GPU, ratio, (dw, dh))"""
    frames = _as_device_frames(img)
    geom = letterbox_geometry(tuple(frames.shape[-3:-1]), new_shape, auto, scaleFill, scaleup, stride)
    return _run(frames, geom, color, torch.uint8, chw=False, swap_rb=False), geom[1], geom[2]


def preprocess(img0, img_size=640, stride=32, half=True, color=(114, 114, 114), auto=True):
    """LoadImages.__next__ + the conversion at the top of detect.py's loop in one kernel: BGR uint8 frame(s) -> RGB (B,3,H,W) fp16/fp32
    in [0,1], letterboxed to `img_size`.  Returns (tensor, ratio, (dw, dh))."""
    frames = _as_device_frames(img0)
    geom = letterbox_geometry(tuple(frames.shape[-3:-1]), img_size, auto, False, True, stride)
    out = _run(frames, geom, color, torch.float16 if half else torch.float32, chw=True, swap_rb=True)
    return (out if out.dim() == 4 else out[None]), geom[1], geom[2]
