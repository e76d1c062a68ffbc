"""Restatement of the reference's test-time augmentation (reference models/yolo.py:274-289, `Model.forward(x, augment=True)`, and
utils/torch_utils.py:248-258 `scale_img`) over `restate.model_forward`.

The fork's loop takes `forward_once(xi)[0]`, which in this fork is the pair (z, raw list), and cannot de-scale it; the loop restated here
takes z, `forward_once(xi)[0][0]`, which is what upstream YOLOv5's loop (where forward_once returns z first) computes.  Three passes:
the input itself, its left-right mirror resized by 0.83, and the input resized by 0.67; every resized input is padded on the right and
bottom to a multiple of the largest stride with 0.447.  Each pass's box columns are divided by its scale, the mirrored pass's centre x is
mirrored back at the input width, and the three predictions are concatenated along the rows.
"""
import math

import torch
import torch.nn.functional as F

from oracle import restate

PASSES = ((1, False), (0.83, True), (0.67, False))      # (scale, left-right mirror)
PAD = 0.447


def scale_img(img: torch.Tensor, ratio=1.0, same_shape=False, gs=32) -> torch.Tensor:
    """bilinear resize (half-pixel centres) to the truncated scaled size, then a constant pad on the right and bottom up to the scaled
    size rounded up to a multiple of gs (or back to the input size with same_shape; a negative pad crops).  Ratio 1: the input as is."""
    if ratio == 1.0:
        return img
    h, w = img.shape[-2:]
    rh, rw = int(h * ratio), int(w * ratio)
    resized = F.interpolate(img, size=(rh, rw), mode="bilinear", align_corners=False)
    oh, ow = (h, w) if same_shape else (math.ceil(h * ratio / gs) * gs, math.ceil(w * ratio / gs) * gs)
    return F.pad(resized, [0, ow - rw, 0, oh - rh], value=PAD)


def tta(z_of, x: torch.Tensor, gs=32) -> torch.Tensor:
    """the augment loop over any single-pass detector `z_of(x) -> z (B, rows, no)`"""
    width = x.shape[-1]
    zs = []
    for si, mirror in PASSES:
        z = z_of(scale_img(x.flip(3) if mirror else x, si, gs=gs)).clone()
        z[..., :4] /= si
        if mirror:
            z[..., 0] = width - z[..., 0]
        zs.append(z)
    return torch.cat(zs, 1)


def model_forward_tta(cfg: dict, sd, x: torch.Tensor, half: bool = False, gs=32) -> torch.Tensor:
    """z of the augmented forward: fp32 on the CPU, or (half=True, CUDA input) the torch fp16 yardstick of restate.model_forward"""
    if half:
        x = x.half()
    return tta(lambda xi: restate.model_forward(cfg, sd, xi, half=half)["z"], x, gs=gs)
