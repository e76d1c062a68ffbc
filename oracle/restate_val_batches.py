"""TEST INFRASTRUCTURE - numpy restatement of the detection validation batches (reference utils/datasets.py `LoadImagesAndLabels`
with augment=False, rect=True): `cv2_resize_area_u8` (load_image's INTER_AREA cache resize) and `val_batch_images` (the cached
images letterboxed to the batch shapes, BGR -> RGB, CHW, stacked as collate_fn stacks them).

cv2.resize(INTER_AREA) down-scaling of 8-bit images chooses its path as OpenCV does:
  * equal size: a copy;
  * scale = 1 / (dst / src) in double, integral in both axes (|scale - round(scale)| < DBL_EPSILON): the kx x ky block sum in int32,
    then (sum + 2) >> 2 at 2x2 and rint(float(sum) * (1.f / (kx * ky))) otherwise (resizeAreaFast);
  * otherwise computeResizeAreaTab + ResizeArea_Invoker: per axis and destination index the taps s1 - 1 (partial), s1 .. s2 - 1 and
    s2 (partial) with float32 weights computed in double; per y tap buf = sum of src * alpha over the x taps in order, then
    sum = beta * buf for the first y tap and sum + beta * buf after it, all in float32; rint and saturate at the end.
This file loops over the tap index and vectorises over pixels, so that full-size frames take well under a second.
"""
import numpy as np

from oracle import restate

_DBL_EPS = np.finfo(np.float64).eps


def _area_taps(d_size, s_size, scale):
    """computeResizeAreaTab of one axis: first source (d_size,), tap count (d_size,) and float32 weights (d_size, kmax), zero past the
    count"""
    fs1 = np.arange(d_size, dtype=np.float64) * scale
    fs2 = fs1 + scale
    cell = np.minimum(scale, s_size - fs1)
    s2 = np.minimum(np.floor(fs2), s_size - 1).astype(np.int64)
    s1 = np.minimum(np.ceil(fs1).astype(np.int64), s2)
    first = (s1 - fs1) > 1e-3
    last = (fs2 - s2) > 1e-3
    n = first.astype(np.int64) + (s2 - s1) + last.astype(np.int64)
    k = np.arange(int(n.max()))[None, :]
    w_first = ((s1 - fs1) / cell).astype(np.float32)[:, None]
    w_mid = (1.0 / cell).astype(np.float32)[:, None]
    w_last = (np.minimum(np.minimum(fs2 - s2, 1.0), cell) / cell).astype(np.float32)[:, None]
    w = np.where(k < n[:, None], w_mid, np.float32(0))
    w = np.where((k == 0) & first[:, None], w_first, w)
    w = np.where((k == n[:, None] - 1) & last[:, None], w_last, w)
    return np.where(first, s1 - 1, s1), n, w.astype(np.float32)


def area_path(H0, W0, H, W):
    """'copy', 'fast2', 'fast' or 'general': the arithmetic cv2.resize(INTER_AREA) uses for (H0, W0) -> (H, W)"""
    if (H, W) == (H0, W0):
        return "copy"
    sx, sy = 1.0 / (W / W0), 1.0 / (H / H0)
    kx, ky = int(round(sx)), int(round(sy))
    if abs(sx - kx) < _DBL_EPS and abs(sy - ky) < _DBL_EPS:
        return "fast2" if kx == ky == 2 else "fast"
    return "general"


def cv2_resize_area_u8(img, dw, dh):
    """cv2.resize(img, (dw, dh), interpolation=cv2.INTER_AREA) of a uint8 (H0, W0, 3) image, down-scaling only, bit for bit"""
    H0, W0 = img.shape[:2]
    if dw > W0 or dh > H0:
        raise ValueError(f"cv2_resize_area_u8: down-scaling only ({W0}x{H0} -> {dw}x{dh})")
    path = area_path(H0, W0, dh, dw)
    if path == "copy":
        return img.copy()
    sx, sy = 1.0 / (dw / W0), 1.0 / (dh / H0)
    if path != "general":
        kx, ky = int(round(sx)), int(round(sy))
        s = img[:dh * ky, :dw * kx].astype(np.int32).reshape(dh, ky, dw, kx, 3).sum((1, 3))
        if path == "fast2":
            return ((s + 2) >> 2).astype(np.uint8)
        return np.clip(np.rint(s.astype(np.float32) * (np.float32(1) / np.float32(kx * ky))), 0, 255).astype(np.uint8)
    x0, _, xw = _area_taps(dw, W0, sx)
    y0, _, yw = _area_taps(dh, H0, sy)
    src = img.astype(np.float32)
    out = None
    for j in range(yw.shape[1]):             # a tap past an index's count has weight 0: it adds +0 and changes nothing
        rows = src[np.minimum(y0 + j, H0 - 1)]
        buf = np.zeros((dh, dw, 3), np.float32)
        for k in range(xw.shape[1]):
            buf = buf + rows[:, np.minimum(x0 + k, W0 - 1)] * xw[None, :, k, None]
        t = yw[:, j, None, None] * buf
        out = t if out is None else out + t
    return np.clip(np.rint(out), 0, 255).astype(np.uint8)


def load_image_val(img, img_size):
    """load_image with augment=False: long side to img_size, INTER_AREA when shrinking, INTER_LINEAR when growing"""
    h0, w0 = img.shape[:2]
    r = img_size / max(h0, w0)
    if r == 1:
        return img.copy()
    w, h = int(w0 * r), int(h0 * r)
    return cv2_resize_area_u8(img, w, h) if r < 1 else restate.cv2_resize_linear_u8(img, w, h)


def val_batch_images(cached, batch_shape):
    """collate_fn's image tensor of one batch: each cached image letterboxed (auto=False, scaleup=False) to batch_shape (h, w), BGR ->
    RGB, HWC -> CHW, stacked; uint8 (B, 3, h, w)"""
    shape = (int(batch_shape[0]), int(batch_shape[1]))
    out = [restate.letterbox_np(im, shape, auto=False, scaleup=False)[0] for im in cached]
    return np.stack([np.ascontiguousarray(o[:, :, ::-1].transpose(2, 0, 1)) for o in out], 0)
