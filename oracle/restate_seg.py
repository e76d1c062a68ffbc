"""TEST INFRASTRUCTURE - numpy restatement of one segmentation training item and one testval item of the reference's PIL loader
(SegmentationDataset.py:118-151 `_sync_transform`, :81-94 `_testval_img_transform`, :182-189 / :219-222 `_mask_transform`, and the
loader functions' `ColorJitter` + `ToTensor`, :458-531).  Every operation is written out as Pillow's C code computes it:

  * Image.resize(BILINEAR): `precompute_coeffs` in double, the 8-bpc fixed-point coefficients (22 fraction bits), a horizontal pass whose
    rows are rounded and clipped to uint8, then a vertical pass; an unchanged axis is an identity pass, an identity resize a copy;
  * Image.resize(NEAREST): the affine-scale path, whose source coordinate is accumulated in double;
  * convert("L"): (19595 R + 38470 G + 7471 B + 0x8000) >> 16;
  * Image.blend: in1 + alpha * (in2 - in1) in C float, alpha narrowed to float, truncated for 0 <= alpha <= 1 and clipped otherwise;
  * convert("HSV") / HSV -> RGB: Pillow's mixed float / double arithmetic of rgb2hsv_row / hsv2rgb;
  * ToTensor: float32(v) / 255.

tests/test_seg_augment_host.py pins each piece to Pillow / torchvision over its input domain and the whole item to the reference's
own output (tests/golden/seg_augment_cases.npz); the GPU tests compare the device path with this module.
"""
import math
import random

import numpy as np
import torch

PRECISION_BITS = 32 - 8 - 2

# Cityscapes label ids -> train ids (the reference's `_key`, indexed by id + 1 after np.digitize over range(-1, 34))
CITYSCAPES_KEY = np.array([-1, -1, -1, -1, -1, -1, -1, -1, 0, 1, -1, -1, 2, 3, 4, -1, -1, -1, 5, -1, 6, 7, 8, 9, 10, 11, 12, 13, 14,
                           15, -1, -1, 16, 17, 18])

# the reference's three loader functions: ColorJitter(brightness, contrast, saturation, hue), get_long_size(low, high, std), crop
PRESETS = {
    "citys": dict(jitter=(0.45, 0.45, 0.45, 0.15), low=0.65, high=3.0, std=25),
    "citysbdd": dict(jitter=(0.4, 0.4, 0.4, 0.05), low=0.65, high=2.0, std=40),
    "custom": dict(jitter=(0.4, 0.4, 0.4, 0.0), low=0.75, high=1.5, std=35),
}


def mask_lut(kind):
    """256-entry uint8 -> int64 label map: 'cityscapes' (_class_to_index: 255 -> 0, id -> trainId; ids above 33 invalid, marked
    -2) or 'trainid' (255 -> -1)"""
    lut = np.full(256, -2, np.int64)
    if kind == "cityscapes":
        lut[:34] = CITYSCAPES_KEY[1:35]
        lut[255] = CITYSCAPES_KEY[1]
    elif kind == "trainid":
        lut[:] = np.arange(256)
        lut[255] = -1
    else:
        raise ValueError(kind)
    return lut


# ---------------------------------------------------------------------------------------------------------------- random draws
def norm_pdf(x, mean, std):
    """scipy.stats.norm.pdf(x, mean, std) as scipy computes it"""
    y = (np.asarray(x, np.float64) - mean) / std
    return np.exp(-y ** 2 / 2.0) / np.sqrt(2 * np.pi) / std


def range_and_prob(base_size, low, high, std):
    lo = math.ceil((base_size * low) / 32)
    hi = math.ceil((base_size * high) / 32)
    mean = math.ceil(base_size / 32) - 4
    x = np.array(list(range(lo, hi + 1)))
    p = norm_pdf(x, mean, std)
    p = p / p.sum()
    return x, np.cumsum(p)


def jitter_ranges(b, c, s, h):
    """ColorJitter's (min, max) per factor; None where the factor is off (hue 0)"""
    def rng(v, center, clip):
        lo, hi = center - v, center + v
        if clip:
            lo = max(lo, 0.0)
        return None if lo == hi == center else (float(lo), float(hi))
    return rng(b, 1, True), rng(c, 1, True), rng(s, 1, True), rng(h, 0, False)


def jitter_params(ranges):
    """ColorJitter.get_params on torch's CPU generator: (order, [b, c, s, h] with None where off)"""
    order = torch.randperm(4).tolist()
    f = [None if r is None else float(torch.empty(1).uniform_(r[0], r[1])) for r in ranges]
    return order, f


def draw_train(w, h, base_size, crop, low, high, std, ranges):
    """the draws of one `_sync_transform` + ColorJitter, in the reference's order: mirror, long side, x1, y1, jitter"""
    flip = random.random() < 0.5
    x, cum_p = range_and_prob(base_size, low, high, std)
    long_size = random.choices(population=x, cum_weights=cum_p, k=1)[0] * 32
    if h > w:
        oh = long_size
        ow = int(1.0 * w * long_size / h + 0.5)
    else:
        ow = long_size
        oh = int(1.0 * h * long_size / w + 0.5)
    cw, ch = crop
    pw, ph = max(ow, cw), max(oh, ch)
    x1 = random.randint(0, pw - cw)
    y1 = random.randint(0, ph - ch)
    order, f = jitter_params(ranges)
    return dict(flip=flip, ow=int(ow), oh=int(oh), x1=x1, y1=y1, order=order, factors=f)


# ---------------------------------------------------------------------------------------------------------------- Pillow arithmetic
def precompute_coeffs(in_size, out_size):
    """Pillow's bilinear precompute_coeffs + normalize_coeffs_8bpc: (xmin[out], count[out], int32 coefficients[out, ksize])"""
    scale = float(np.float32(in_size)) / out_size
    filterscale = max(scale, 1.0)
    support = 1.0 * filterscale
    ksize = int(math.ceil(support)) * 2 + 1
    bounds = np.zeros((out_size, 2), np.int64)
    kk = np.zeros((out_size, ksize), np.int32)
    ss = 1.0 / filterscale
    for xx in range(out_size):
        center = 0.0 + (xx + 0.5) * scale
        xmin = max(int(center - support + 0.5), 0)
        xmax = min(int(center + support + 0.5), in_size) - xmin
        w = []
        for x in range(xmax):
            t = abs((x + xmin - center + 0.5) * ss)
            w.append(1.0 - t if t < 1.0 else 0.0)
        ww = 0.0
        for v in w:
            ww += v
        for x in range(xmax):
            k = w[x] / ww if ww != 0.0 else w[x]
            kk[xx, x] = int(-0.5 + k * (1 << PRECISION_BITS)) if k < 0 else int(0.5 + k * (1 << PRECISION_BITS))
        bounds[xx] = xmin, xmax
    return bounds[:, 0], bounds[:, 1], kk


def _pass(src, axis, out_size):
    """one 8-bpc resampling pass of uint8 (H, W, C) along axis 1 (horizontal) or 0 (vertical)"""
    xmin, cnt, kk = precompute_coeffs(src.shape[axis], out_size)
    s = np.moveaxis(src.astype(np.int64), axis, 0)
    acc = np.full((out_size,) + s.shape[1:], 1 << (PRECISION_BITS - 1), np.int64)
    for k in range(kk.shape[1]):
        idx = np.minimum(xmin + k, s.shape[0] - 1)
        c = np.where(k < cnt, kk[:, k], 0).astype(np.int64).reshape((-1,) + (1,) * (s.ndim - 1))
        acc += s[idx] * c
    return np.moveaxis(np.clip(acc >> PRECISION_BITS, 0, 255).astype(np.uint8), 0, axis)


def resize_bilinear(img, ow, oh):
    """Image.resize((ow, oh), BILINEAR) of uint8 (H, W, 3)"""
    h, w = img.shape[:2]
    out = img
    if ow != w:
        out = _pass(out, 1, ow)
    if oh != h:
        out = _pass(out, 0, oh)
    return out.copy()


def nearest_index(in_size, out_size):
    """source index of each output position of Image.resize(NEAREST): xo = a/2, xo += a, accumulated in double"""
    a = float(np.float32(in_size)) / out_size
    idx = np.empty(out_size, np.int64)
    xo = 0.0 + a * 0.5
    for x in range(out_size):
        idx[x] = -1 if xo < 0.0 else int(xo)
        xo += a
    return idx


def resize_nearest(mask, ow, oh):
    h, w = mask.shape[:2]
    if (ow, oh) == (w, h):
        return mask.copy()
    return mask[nearest_index(h, oh)][:, nearest_index(w, ow)]


def to_l(img):
    """convert('L')"""
    r, g, b = (img[..., c].astype(np.int64) for c in range(3))
    return ((r * 19595 + g * 38470 + b * 7471 + 0x8000) >> 16).astype(np.uint8)


def blend(in1, in2, alpha):
    """Image.blend(in1, in2, alpha) of uint8 arrays"""
    a = np.float32(alpha)
    i1 = in1.astype(np.float32)
    t = i1 + a * (in2.astype(np.float32) - i1)
    if 0.0 <= alpha <= 1.0:
        return t.astype(np.uint8)
    return np.where(t <= 0.0, 0, np.where(t >= 255.0, 255, np.clip(t, 0, 255).astype(np.uint8))).astype(np.uint8)


def rgb2hsv(img):
    """convert('HSV'): Pillow's rgb2hsv_row (float variables, double constants)"""
    r, g, b = (img[..., c].astype(np.int64) for c in range(3))
    mx, mn = np.maximum(r, np.maximum(g, b)), np.minimum(r, np.minimum(g, b))
    cr = (mx - mn).astype(np.float32)
    crs = np.where(cr == 0, np.float32(1), cr)
    s = cr / np.maximum(mx, 1).astype(np.float32)
    rc = (mx - r).astype(np.float32) / crs
    gc = (mx - g).astype(np.float32) / crs
    bc = (mx - b).astype(np.float32) / crs
    h = np.where(r == mx, (bc - gc).astype(np.float64),
                 np.where(g == mx, (2.0 + rc.astype(np.float64)) - bc.astype(np.float64),
                          (4.0 + gc.astype(np.float64)) - rc.astype(np.float64))).astype(np.float32)
    h = np.fmod(h.astype(np.float64) / 6.0 + 1.0, 1.0).astype(np.float32)
    uh = np.clip((h.astype(np.float64) * 255.0).astype(np.int64), 0, 255)
    us = np.clip((s.astype(np.float64) * 255.0).astype(np.int64), 0, 255)
    grey = mx == mn
    return np.stack([np.where(grey, 0, uh), np.where(grey, 0, us), mx], -1).astype(np.uint8)


def _round_half_away(x):
    t = np.trunc(x)
    return (t + np.sign(x) * (np.abs(x - t) >= 0.5)).astype(np.int64)


def hsv2rgb(hsv):
    """HSV -> RGB: Pillow's hsv2rgb"""
    h, s, v = (hsv[..., c].astype(np.int64) for c in range(3))
    hd = h.astype(np.float32).astype(np.float64) * 6.0 / 255.0
    i = np.floor(hd).astype(np.int64)
    f = (hd - i.astype(np.float32).astype(np.float64)).astype(np.float32)
    fs = f * s.astype(np.float32)
    vf = v.astype(np.float32).astype(np.float64)
    p = np.clip(_round_half_away(vf * (1.0 - s.astype(np.float32).astype(np.float64) / 255.0)), 0, 255)
    q = np.clip(_round_half_away(vf * (1.0 - fs.astype(np.float64) / 255.0)), 0, 255)
    t = np.clip(_round_half_away(vf * (1.0 - (s.astype(np.float32) - fs).astype(np.float64) / 255.0)), 0, 255)
    sel = i % 6
    table = [(v, t, p), (q, v, p), (p, v, t), (p, q, v), (t, p, v), (v, p, q)]
    out = [np.choose(sel, [tb[c] for tb in table]) for c in range(3)]
    grey = s == 0
    return np.stack([np.where(grey, v, o) for o in out], -1).astype(np.uint8)


def hue_shift(hue_factor):
    """np.int32(hue_factor * 255).astype(np.uint8) of adjust_hue"""
    return int(np.int32(hue_factor * 255).astype(np.uint8))


def adjust_hue(img, hue_factor):
    hsv = rgb2hsv(img)
    hsv[..., 0] = (hsv[..., 0].astype(np.int64) + hue_shift(hue_factor)) & 255
    return hsv2rgb(hsv)


def color_jitter(img, order, factors):
    """ColorJitter.forward on a uint8 (H, W, 3) RGB image with drawn (order, factors)"""
    for fn in order:
        f = factors[fn]
        if f is None:
            continue
        if fn == 0:
            img = blend(np.zeros_like(img), img, f)
        elif fn == 1:
            mean = int(float(to_l(img).astype(np.int64).sum()) / img[..., 0].size + 0.5)
            img = blend(np.full_like(img, mean), img, f)
        elif fn == 2:
            img = blend(np.repeat(to_l(img)[..., None], 3, -1), img, f)
        else:
            img = adjust_hue(img, f)
    return img


def to_tensor(img):
    """ToTensor of uint8 (H, W, 3): float32 (3, H, W) = v / 255"""
    return np.ascontiguousarray(img.transpose(2, 0, 1)).astype(np.float32) / np.float32(255)


# ---------------------------------------------------------------------------------------------------------------- items
def crop_of(img, mask, p, crop):
    """mirror, resize, pad (image 0, mask 255) and crop of `_sync_transform` with drawn parameters p"""
    if p["flip"]:
        img, mask = img[:, ::-1], mask[:, ::-1]
    img = resize_bilinear(np.ascontiguousarray(img), p["ow"], p["oh"])
    mask = resize_nearest(np.ascontiguousarray(mask), p["ow"], p["oh"])
    cw, ch = crop
    ph, pw = max(p["oh"], ch), max(p["ow"], cw)
    im2 = np.zeros((ph, pw, 3), np.uint8)
    m2 = np.full((ph, pw), 255, np.uint8)
    im2[:p["oh"], :p["ow"]] = img
    m2[:p["oh"], :p["ow"]] = mask
    x1, y1 = p["x1"], p["y1"]
    return im2[y1:y1 + ch, x1:x1 + cw], m2[y1:y1 + ch, x1:x1 + cw]


def train_item(img, mask, lut, p, crop):
    """dataset[i] for mode='train' from drawn parameters: (float32 (3, h, w), int64 (h, w))"""
    im, m = crop_of(img, mask, p, crop)
    return to_tensor(color_jitter(im, p["order"], p["factors"])), lut[m]


def getitem(img, mask, lut, base_size, crop, low, high, std, ranges):
    """dataset[i] for mode='train', consuming the reference's draws from `random` and torch's CPU generator"""
    p = draw_train(img.shape[1], img.shape[0], base_size, crop, low, high, std, ranges)
    return train_item(img, mask, lut, p, crop)


def make_divisible(x, divisor):
    return math.ceil(x / divisor) * divisor


def testval_size(w, h, base_size):
    """(ow, oh) of `_testval_img_transform`"""
    outlong = make_divisible(base_size, 32)
    if w > h:
        ow = outlong
        oh = make_divisible(int(1.0 * h * ow / w), 32)
    else:
        oh = outlong
        ow = make_divisible(int(1.0 * w * oh / h), 32)
    return ow, oh


def testval_item(img, mask, lut, base_size):
    """dataset[i] for mode='testval': (float32 (3, oh, ow), int64 (H, W))"""
    ow, oh = testval_size(img.shape[1], img.shape[0], base_size)
    return to_tensor(resize_bilinear(img, ow, oh)), lut[mask]
