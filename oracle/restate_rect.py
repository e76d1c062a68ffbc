"""Numpy restatement of the reference's `--rect` training dataset: LoadImagesAndLabels(augment=True, rect=True) (reference
utils/datasets.py:410-439 the aspect-ratio sort and batch shapes, :518-592 `__getitem__` without mosaic).  The pixel arithmetic (cv2's
resize, warpAffine, HSV conversions) is oracle/restate_augment.py's; this module adds the rect plan and the rect item, and is pinned to
the reference by tests/golden/rect_cases.npz (oracle/make_golden_rect.py).
"""
import random

import numpy as np

from oracle.restate import letterbox_np
from oracle.restate_augment import _boxes_to_pixels, augment_hsv_np, warp


def rect_batch_shapes(shapes0, img_size, batch_size, stride=32, pad=0.0):
    """LoadImagesAndLabels.__init__ with rect=True (reference :410-439) over the original (h, w) shapes: (irect, bi, batch_shapes [h, w])"""
    wh = np.array([(w, h) for h, w in shapes0], np.float64)
    ar = wh[:, 1] / wh[:, 0]
    irect = ar.argsort()
    ar = ar[irect]
    bi = np.floor(np.arange(len(ar)) / batch_size).astype(int)
    shapes = []
    for i in range(bi[-1] + 1):
        lo, hi = ar[bi == i].min(), ar[bi == i].max()
        shapes.append([hi, 1] if hi < 1 else [1, 1 / lo] if lo > 1 else [1, 1])
    return irect, bi, np.ceil(np.array(shapes) * img_size / stride + pad).astype(int) * stride


def getitem_rect(ds, index, shape):
    """one item of LoadImagesAndLabels(augment=True, rect=True) (reference :518-592 without mosaic): letterbox to the batch `shape`
    (a numpy [h, w] row of batch_shapes), random_perspective at that size (skipped for the identity), augment_hsv, the label path, the
    flips, BGR -> RGB and HWC -> CHW.  `ds` is a restate_augment.Source.  Returns (uint8 (3, h, w) RGB image, (n, 5) float32 labels)."""
    hyp = ds.hyp
    im = ds.cache[index]
    h, w = im.shape[:2]
    img, ratio, (dw, dh) = letterbox_np(im, shape, auto=False, scaleup=True)
    lab = ds.labels[index].copy()
    if lab.size:
        lab[:, 1:] = _boxes_to_pixels(lab[:, 1:], ratio[0] * w, ratio[1] * h, dw, dh)
    img, lab = warp(img, lab, hyp)
    img = augment_hsv_np(img, hyp["hsv_h"], hyp["hsv_s"], hyp["hsv_v"])
    if len(lab):
        xyxy = lab[:, 1:5].copy()
        lab[:, 1] = (xyxy[:, 0] + xyxy[:, 2]) / 2
        lab[:, 2] = (xyxy[:, 1] + xyxy[:, 3]) / 2
        lab[:, 3] = xyxy[:, 2] - xyxy[:, 0]
        lab[:, 4] = xyxy[:, 3] - xyxy[:, 1]
        lab[:, [2, 4]] /= img.shape[0]
        lab[:, [1, 3]] /= img.shape[1]
    if random.random() < hyp["flipud"]:
        img = img[::-1]
        if len(lab):
            lab[:, 2] = 1 - lab[:, 2]
    if random.random() < hyp["fliplr"]:
        img = img[:, ::-1]
        if len(lab):
            lab[:, 1] = 1 - lab[:, 1]
    return np.ascontiguousarray(img[:, :, ::-1].transpose(2, 0, 1)), lab
