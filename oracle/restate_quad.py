"""Numpy restatement of the reference's `--quad` collate, LoadImagesAndLabels.collate_fn4 (reference utils/datasets.py:602-625), pinned to
the reference by tests/golden/quad_cases.npz (oracle/make_golden_quad.py).

The x2 bilinear up-scale is restated in integers: F.interpolate(scale_factor=2., mode='bilinear', align_corners=False) reads output row Y
at Y/2 - 1/4 (clamped at 0), so the weights are 1/4 and 3/4 (1 at the clamped first row and the last odd row), and torch's float32 sum
is exact (tests/test_quad_host.py proves it); `.type(uint8)` truncates it.
"""
import random

import numpy as np

HO = np.array([[0., 0, 0, 1, 0, 0]], np.float32)      # collate_fn4's ho, wo and s (float32, as its torch.tensor literals)
WO = np.array([[0., 0, 1, 0, 0, 0]], np.float32)
S = np.array([[1, 1, .5, .5, .5, .5]], np.float32)


def _taps(n):
    """per output index of a x2 axis of n inputs: first input, second input, weight of the first (of 4)"""
    d = np.arange(2 * n)
    r, odd = d >> 1, (d & 1).astype(bool)
    a = np.where(odd, r, np.maximum(r - 1, 0))
    b = np.where(odd, np.minimum(r + 1, n - 1), r)
    return a, b, np.where(odd, 3, 1)


def upsample2x_u8(img: np.ndarray) -> np.ndarray:
    """F.interpolate(img.float()[None], scale_factor=2., mode='bilinear', align_corners=False)[0].type(uint8) of a uint8 (C, H, W)"""
    v = img.astype(np.int64)
    ya, yb, wy = _taps(img.shape[1])
    xa, xb, wx = _taps(img.shape[2])
    rows = wy[:, None] * v[:, ya] + (4 - wy)[:, None] * v[:, yb]          # (C, 2H, W), weights in quarters
    out = wx * rows[:, :, xa] + (4 - wx) * rows[:, :, xb]                  # (C, 2H, 2W), in sixteenths
    return (out >> 4).astype(np.uint8)


def collate_quad_np(imgs: np.ndarray, targets: np.ndarray, rng=random):
    """collate_fn4 of a collated batch: uint8 (B, 3, h, w) images and (n, 6) float32 targets whose column 0 is the item index.  Returns
    (uint8 (B // 4, 3, 2h, 2w), (m, 6) float32), one rng.random() per quad in quad order.  ValueError below 4 items."""
    n = len(imgs) // 4
    if n == 0:
        raise ValueError(f"a batch of {len(imgs)} items has no quad")
    labels = [targets[targets[:, 0] == i] for i in range(len(imgs))]
    img4, label4 = [], []
    for q in range(n):
        i = 4 * q
        if rng.random() < 0.5:
            im, lb = upsample2x_u8(imgs[i]), labels[i].copy()
        else:
            im = np.concatenate((np.concatenate((imgs[i], imgs[i + 1]), 1), np.concatenate((imgs[i + 2], imgs[i + 3]), 1)), 2)
            lb = np.concatenate((labels[i], labels[i + 1] + HO, labels[i + 2] + WO, labels[i + 3] + HO + WO), 0) * S
        lb[:, 0] = q
        img4.append(im)
        label4.append(lb)
    return np.stack(img4), np.concatenate(label4, 0).astype(np.float32)
