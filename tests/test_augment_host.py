"""CPU: the detection training-item restatement (oracle/restate_augment.py) against the reference's own output
(tests/golden/augment_cases.npz, oracle/make_golden_augment.py), the colour conversions against cv2 over their whole input domain, and the
host half of DetAugmenter (random draws, labels, kernel parameters) against the restatement."""
import json
import os
import random

import numpy as np
import pytest

from oracle import restate_augment as ra

GOLD = os.path.join(os.path.dirname(__file__), "golden")


def _golden():
    g = np.load(os.path.join(GOLD, "augment_cases.npz"))
    return g, json.loads(bytes(g["meta_json"]).decode())


def _source(g, meta, name):
    n = len(meta["shapes"])
    c = meta["cases"][name]
    return ra.Source([g[f"src_{k}"] for k in range(n)], [g[f"labels_{k}"] for k in range(n)], c["img_size"], c["hyp"])


@pytest.mark.parametrize("name", ["scratch", "stress", "mixup", "flipud", "single"])
def test_restatement_matches_reference_items(name):
    g, meta = _golden()
    c = meta["cases"][name]
    src = _source(g, meta, name)
    for i in range(src.n):                       # load_image's resize (the cache; stored for one size, the items pin the other)
        key = f"cache{c['img_size']}_{i}"
        assert key in g.files or c["img_size"] != 96
        assert key not in g.files or np.array_equal(src.cache[i], g[key]), (name, i)
    random.seed(c["seed"])
    np.random.seed(c["seed"])
    for i in c["items"]:
        img, lab = ra.getitem(src, i)
        ref_img, ref_lab = g[f"{name}_img_{i}"], g[f"{name}_lab_{i}"]
        assert img.shape == ref_img.shape and np.array_equal(img, ref_img), (name, i, int((img != ref_img).sum()))
        assert lab.dtype == np.float32 and np.array_equal(lab, ref_lab), (name, i, lab, ref_lab)
    assert random.random() == c["next_random"] and float(np.random.random()) == c["next_np"], "random number consumption differs"


def test_fixtures_cover_every_branch():
    g, meta = _golden()
    cases = meta["cases"]
    assert cases["single"]["hyp"]["mosaic"] == 0 and cases["mixup"]["hyp"]["mixup"] == 1 and cases["flipud"]["hyp"]["flipud"] > 0
    assert cases["stress"]["hyp"]["degrees"] == 10 and cases["stress"]["hyp"]["shear"] == 5
    assert any(min(s) < 64 for s in meta["shapes"]) and any(h > w for h, w in meta["shapes"])
    assert cases["flipud"]["hyp"]["flipud"] == 1 and cases["scratch"]["hyp"]["fliplr"] > 0


def _cv2():
    return pytest.importorskip("cv2")


def test_hsv2bgr_exhaustive_against_cv2():
    cv2 = _cv2()
    h, s, v = np.meshgrid(np.arange(180), np.arange(256), np.arange(256), indexing="ij")
    hsv = np.stack([h, s, v], -1).astype(np.uint8).reshape(180 * 256, 256, 3)
    want = cv2.cvtColor(hsv, cv2.COLOR_HSV2BGR)
    got = ra.hsv2bgr_u8(hsv)
    assert np.array_equal(got, want), int((got != want).sum())


def test_bgr2hsv_exhaustive_against_cv2():
    cv2 = _cv2()
    bgr = np.arange(1 << 24, dtype=np.uint32)
    bgr = np.stack([bgr & 255, (bgr >> 8) & 255, bgr >> 16], -1).astype(np.uint8).reshape(4096, 4096, 3)
    want = cv2.cvtColor(bgr, cv2.COLOR_BGR2HSV)
    got = ra.bgr2hsv_u8(bgr)
    assert np.array_equal(got, want), int((got != want).sum())


def test_warp_affine_model_against_cv2():
    cv2 = _cv2()
    rs = np.random.RandomState(0)
    canvas = rs.randint(0, 256, (150, 170, 3), dtype=np.uint8)
    for k in range(6):
        a = np.deg2rad(rs.uniform(-10, 10))
        sc = rs.uniform(0.5, 1.5)
        M = np.array([[np.cos(a) * sc, np.sin(a) * sc + rs.uniform(-0.1, 0.1), rs.uniform(-40, 40)],
                      [-np.sin(a) * sc, np.cos(a) * sc, rs.uniform(-40, 40)]])
        want = cv2.warpAffine(canvas, M, dsize=(128, 120), borderValue=(114, 114, 114))
        assert np.array_equal(ra.warp_affine_u8(canvas, M, 128, 120), want), k


def test_bilinear_table_needs_no_correction():
    t = ra.bilinear_tab()
    fy, fx = np.meshgrid(np.arange(32), np.arange(32), indexing="ij")
    want = np.stack([(32 - fy) * (32 - fx), (32 - fy) * fx, fy * (32 - fx), fy * fx], -1) * 32     # what the kernel computes
    assert np.array_equal(t, want) and (t.sum(-1) == 32768).all()


class _HostCache:
    """what DetAugmenter reads from a DeviceImageCache, without a device (pointers are placeholders)"""

    def __init__(self, src):
        self.img_size, self.n, self.labels = src.img_size, src.n, src.labels
        self.shapes = [im.shape[:2] for im in src.cache]

    def ptr(self, i):
        return 4096 * (i + 1)


def test_aug_struct_layout():
    import ctypes as C
    from multiyolov5_b200 import _lib
    assert C.sizeof(_lib.AugWarp) == 200 and C.sizeof(_lib.AugItem) == 1200     # static_assert in csrc/augment.cu


@pytest.mark.parametrize("name", ["scratch", "stress", "mixup", "flipud", "single"])
def test_host_draws_match_restatement(name):
    """DetAugmenter.item (host half of the device path) consumes the same draws and produces the same labels as the restatement;
    its warp parameters are the restatement's inverse matrix"""
    from multiyolov5_b200.utils.datasets import DetAugmenter
    g, meta = _golden()
    c = meta["cases"][name]
    src = _source(g, meta, name)
    aug = DetAugmenter(_HostCache(src), c["hyp"])
    for i in c["items"]:
        random.seed(c["seed"] + 100 * i)
        np.random.seed(c["seed"] + 100 * i)
        _, want = ra.getitem(src, i)
        r_state, n_state = random.getstate(), np.random.get_state()[1].copy()
        random.seed(c["seed"] + 100 * i)
        np.random.seed(c["seed"] + 100 * i)
        it, lab = aug.item(i)
        assert np.array_equal(lab, want), (name, i)
        assert random.getstate() == r_state and np.array_equal(np.random.get_state()[1], n_state), (name, i)
        assert it.n_warps in (1, 2) and (it.n_warps == 2) == (c["hyp"]["mixup"] > 0 and c["hyp"]["mosaic"] > 0)
    random.seed(7)
    M, _, _, _ = ra.affine_params(2 * src.img_size, 2 * src.img_size, (-src.img_size // 2,) * 2, c["hyp"])
    random.seed(7)
    M2, _ = aug._perspective(2 * src.img_size, 2 * src.img_size, np.zeros((0, 5), np.float32), border=aug.mosaic_border)
    assert np.array_equal(M, M2)
    w = aug._warp([(4096, 10, 0, 0, 10, 10, 0, 0)], M2)
    assert list(w.minv) == list(ra.invert_affine(M[:2]))


def test_unsupported_settings_raise():
    from multiyolov5_b200.utils.datasets import DetAugmenter
    g, meta = _golden()
    src = _source(g, meta, "scratch")
    hyp = dict(meta["cases"]["scratch"]["hyp"])
    with pytest.raises(NotImplementedError):
        DetAugmenter(_HostCache(src), dict(hyp, perspective=0.001))
    with pytest.raises(NotImplementedError):
        DetAugmenter(_HostCache(src), hyp, mosaic9=True)
    with pytest.raises(NotImplementedError):
        DetAugmenter(_HostCache(src), hyp, quad=True)
