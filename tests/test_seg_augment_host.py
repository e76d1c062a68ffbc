"""CPU: the segmentation training-item restatement (oracle/restate_seg.py) against the reference's own items
(tests/golden/seg_augment_cases.npz, oracle/make_golden_seg.py), each Pillow operation it restates against Pillow / torchvision over its
input domain, and the host half of SegAugmenter (random draws, resampling tables, mask maps) against the restatement and the fixtures."""
import json
import os
import random

import numpy as np
import pytest
import torch

from oracle import restate_seg as rs

GOLD = os.path.join(os.path.dirname(__file__), "golden")


def _golden():
    g = np.load(os.path.join(GOLD, "seg_augment_cases.npz"))
    return g, json.loads(bytes(g["meta_json"]).decode())["cases"]


def _kind(c, i):
    if c["loader"] == "citys" or (c["loader"] == "citysbdd" and c["files"][i].endswith("png")):
        return "cityscapes"
    return "trainid"


def _item_sources(g, c, i):
    si, mi = c["sources"][i]
    return g[f"src_{si}"], g[f"mask_{mi}"]


@pytest.mark.parametrize("name", ["citys", "citysbdd", "custom", "testval"])
def test_restatement_matches_reference_items(name):
    g, cases = _golden()
    c = cases[name]
    pre = rs.PRESETS[c["loader"]]
    random.seed(c["seed"])
    torch.manual_seed(c["seed"])
    for j, i in enumerate(c["items"]):
        img, mask = _item_sources(g, c, i)
        lut = rs.mask_lut(_kind(c, i))
        if c["mode"] == "train":
            im, lab = rs.getitem(img, mask, lut, c["base_size"], tuple(c["crop_size"]), pre["low"], pre["high"], pre["std"],
                                 rs.jitter_ranges(*pre["jitter"]))
        else:
            im, lab = rs.testval_item(img, mask, lut, c["base_size"])
        ref = g[f"{name}_img_{j}"].astype(np.float32) / np.float32(255)
        assert im.dtype == np.float32 and im.shape == ref.shape and np.array_equal(im, ref), (name, j, int((im != ref).sum()))
        assert lab.dtype == np.int64 and np.array_equal(lab, g[f"{name}_lab_{j}"].astype(np.int64)), (name, j)
    assert random.random() == c["next_random"] and float(torch.rand(1)) == c["next_torch"], "random number consumption differs"


def test_fixtures_cover_every_branch():
    """the fixture items between them mirror, pad, shrink and grow the source, use several jitter orders, and the City+BDD case maps
    one JPEG item as train ids"""
    g, cases = _golden()
    seen = dict(flip=set(), pad=False, down=False, up=False, orders=set())
    for name in ("citys", "citysbdd", "custom"):
        c = cases[name]
        pre = rs.PRESETS[c["loader"]]
        random.seed(c["seed"])
        torch.manual_seed(c["seed"])
        for i in c["items"]:
            h, w = _item_sources(g, c, i)[0].shape[:2]
            p = rs.draw_train(w, h, c["base_size"], tuple(c["crop_size"]), pre["low"], pre["high"], pre["std"],
                              rs.jitter_ranges(*pre["jitter"]))
            seen["flip"].add(p["flip"])
            seen["pad"] |= p["ow"] < c["crop_size"][0] or p["oh"] < c["crop_size"][1]
            seen["down"] |= p["ow"] < w
            seen["up"] |= p["ow"] > w
            seen["orders"].add(tuple(p["order"]))
    assert seen["flip"] == {False, True} and seen["pad"] and seen["down"] and seen["up"] and len(seen["orders"]) >= 6, seen
    assert any(f.endswith(".jpg") for f in cases["citysbdd"]["files"])


# ------------------------------------------------------------------------------------------------ restatement vs Pillow / torchvision
def _pil():
    return pytest.importorskip("PIL.Image")


def _all_colours():
    v = np.arange(1 << 24, dtype=np.uint32)
    return np.stack([v & 255, (v >> 8) & 255, v >> 16], -1).astype(np.uint8).reshape(4096, 4096, 3)


def test_resize_sweep_against_pillow():
    """bilinear and NEAREST resizes up, down, along one axis, identity, and of a mirrored source"""
    Image = _pil()
    r = np.random.RandomState(0)
    src = r.randint(0, 256, (64, 96, 3)).astype(np.uint8)
    mask = r.randint(0, 256, (64, 96)).astype(np.uint8)
    for ow, oh in [(96, 64), (200, 133), (31, 21), (96, 30), (40, 64), (97, 65), (192, 128), (48, 32), (17, 90), (300, 7), (95, 63)]:
        for flip in (False, True):
            s = np.ascontiguousarray(src[:, ::-1]) if flip else src
            m = np.ascontiguousarray(mask[:, ::-1]) if flip else mask
            assert np.array_equal(rs.resize_bilinear(s, ow, oh), np.array(Image.fromarray(s).resize((ow, oh), Image.BILINEAR))), (ow, oh)
            assert np.array_equal(rs.resize_nearest(m, ow, oh), np.array(Image.fromarray(m).resize((ow, oh), Image.NEAREST))), (ow, oh)


def test_resize_full_size_extremes_against_pillow():
    """2048x1024 to the long sides 672 (about 7 taps per axis) and 3072 (2 taps)"""
    Image = _pil()
    big = np.random.RandomState(1).randint(0, 256, (1024, 2048, 3)).astype(np.uint8)
    for ow, oh in [(672, 336), (3072, 1536)]:
        assert np.array_equal(rs.resize_bilinear(big, ow, oh), np.array(Image.fromarray(big).resize((ow, oh), Image.BILINEAR))), ow


def test_l_conversion_all_colours_against_pillow():
    Image = _pil()
    rgb = _all_colours()
    assert np.array_equal(rs.to_l(rgb), np.array(Image.fromarray(rgb).convert("L")))


def test_hsv_round_trip_all_colours_against_pillow():
    Image = _pil()
    rgb = _all_colours()
    assert np.array_equal(rs.rgb2hsv(rgb), np.array(Image.fromarray(rgb).convert("HSV")))
    assert np.array_equal(rs.hsv2rgb(rgb), np.array(Image.fromarray(rgb, "HSV").convert("RGB")))     # every (h, s, v)


@pytest.mark.parametrize("hue", [-0.5, -0.15, -0.0039, 0.002, 0.07, 0.15, 0.5])
def test_adjust_hue_all_colours_against_torchvision(hue):
    Image = _pil()
    F = pytest.importorskip("torchvision.transforms.functional")
    rgb = _all_colours()
    assert np.array_equal(rs.adjust_hue(rgb, hue), np.array(F.adjust_hue(Image.fromarray(rgb), hue))), hue


@pytest.mark.parametrize("alpha", [0.0, 0.13, 0.55, 0.9999999, 1.0, 1.0000001, 1.37, 1.45, 3.0, -0.2])
def test_blend_all_pairs_against_pillow(alpha):
    Image = _pil()
    a, b = np.meshgrid(np.arange(256), np.arange(256), indexing="ij")
    i1 = np.repeat(a[..., None], 3, -1).astype(np.uint8)
    i2 = np.repeat(b[..., None], 3, -1).astype(np.uint8)
    alpha = float(np.float32(alpha))                         # the factors are float32 draws
    assert np.array_equal(rs.blend(i1, i2, alpha), np.array(Image.blend(Image.fromarray(i1), Image.fromarray(i2), alpha)))


def test_color_jitter_against_torchvision():
    """every op in all 24 orders, contrast factors on both sides of 1, against ColorJitter's own functions"""
    import itertools
    Image = _pil()
    F = pytest.importorskip("torchvision.transforms.functional")
    img = np.random.RandomState(2).randint(0, 256, (40, 56, 3)).astype(np.uint8)
    fns = [F.adjust_brightness, F.adjust_contrast, F.adjust_saturation, F.adjust_hue]
    for k, order in enumerate(itertools.permutations(range(4))):
        factors = [float(np.float32(v)) for v in ([0.55, 1.45][k % 2], [0.6, 1.4][(k // 2) % 2], [0.7, 1.3][(k // 4) % 2],
                                                  [-0.15, 0.15][(k // 3) % 2])]
        want = Image.fromarray(img)
        for fn in order:
            want = fns[fn](want, factors[fn])
        assert np.array_equal(rs.color_jitter(img, list(order), factors), np.array(want)), order


def test_to_tensor_division_against_torchvision():
    F = pytest.importorskip("torchvision.transforms.functional")
    img = np.arange(256, dtype=np.uint8).reshape(16, 16, 1).repeat(3, -1)
    assert np.array_equal(rs.to_tensor(img), F.to_tensor(img).numpy())
    assert not np.array_equal(rs.to_tensor(img), img.transpose(2, 0, 1).astype(np.float32) * np.float32(1 / 255))


# ------------------------------------------------------------------------------------------------ host half of SegAugmenter
@pytest.mark.parametrize("preset", ["citys", "citysbdd", "custom"])
@pytest.mark.parametrize("base", [128, 1024])
def test_range_and_prob_equals_scipy(preset, base):
    stats = pytest.importorskip("scipy.stats")
    import math
    from multiyolov5_b200.utils.datasets import SEG_PRESETS, range_and_prob
    p = SEG_PRESETS[preset]
    x, cum_p = range_and_prob(base, p["low"], p["high"], p["std"])
    lo, hi, mean = math.ceil(base * p["low"] / 32), math.ceil(base * p["high"] / 32), math.ceil(base / 32) - 4
    want = stats.norm.pdf(np.array(list(range(lo, hi + 1))), mean, p["std"])
    want = want / want.sum()
    assert np.array_equal(x, np.arange(lo, hi + 1)) and np.array_equal(cum_p, np.cumsum(want))


def test_tables_equal_restatement():
    from multiyolov5_b200.utils.datasets import _bilinear_table, _nearest_index
    for n_in, n_out in [(2048, 672), (2048, 3072), (1024, 336), (1024, 1536), (96, 200), (256, 96), (120, 7), (64, 64), (250, 384)]:
        t = _bilinear_table(n_in, n_out)
        if n_in == n_out:
            assert (t[:, 0] == np.arange(n_out)).all() and (t[:, 1] == 1).all() and (t[:, 2] == 1 << 22).all()
        else:
            xmin, cnt, kk = rs.precompute_coeffs(n_in, n_out)
            assert np.array_equal(t[:, 0], xmin) and np.array_equal(t[:, 1], cnt) and np.array_equal(t[:, 2:], kk), (n_in, n_out)
        assert np.array_equal(_nearest_index(n_in, n_out), rs.nearest_index(n_in, n_out)), (n_in, n_out)


class _HostCache:
    """what SegAugmenter.draw reads from a DeviceSegCache, without a device"""

    def __init__(self, shapes):
        self.shapes = shapes


@pytest.mark.parametrize("name", ["citys", "citysbdd", "custom"])
def test_host_draws_match_fixtures(name):
    """SegAugmenter.draw consumes the reference's draws: the same parameters as the restatement, and the fixtures' next draws after"""
    from multiyolov5_b200.utils.datasets import SegAugmenter
    g, cases = _golden()
    c = cases[name]
    pre = rs.PRESETS[c["loader"]]
    shapes = [g[f"src_{si}"].shape[:2] for si, _ in c["sources"]]
    aug = SegAugmenter(_HostCache(shapes), base_size=c["base_size"], crop_size=tuple(c["crop_size"]), preset=c["loader"])
    random.seed(c["seed"])
    torch.manual_seed(c["seed"])
    want = [rs.draw_train(shapes[i][1], shapes[i][0], c["base_size"], tuple(c["crop_size"]), pre["low"], pre["high"], pre["std"],
                          rs.jitter_ranges(*pre["jitter"])) for i in c["items"]]
    random.seed(c["seed"])
    torch.manual_seed(c["seed"])
    got = [aug.draw(i) for i in c["items"]]
    assert got == want
    assert random.random() == c["next_random"] and float(torch.rand(1)) == c["next_torch"]
    if name == "custom":
        assert aug.crop_size == (c["base_size"],) * 2 and aug.jitter_ranges[3] is None


def test_preset_override():
    from multiyolov5_b200.utils.datasets import SegAugmenter
    aug = SegAugmenter(_HostCache([(8, 8)]), base_size=512, preset="citysbdd", hue=0.0, low=0.5, crop_size=(256, 128))
    assert aug.jitter_ranges == ((0.6, 1.4), (0.6, 1.4), (0.6, 1.4), None) and aug.low == 0.5 and aug.high == 2.0
    assert aug.crop_size == (256, 128)
    with pytest.raises(ValueError):
        SegAugmenter(_HostCache([(8, 8)]), preset="voc")


def test_mask_maps():
    from multiyolov5_b200.utils.datasets import seg_mask_lut
    for kind in ("cityscapes", "trainid"):
        assert np.array_equal(seg_mask_lut(kind), rs.mask_lut(kind))
    lut = seg_mask_lut("cityscapes")
    ids = np.arange(34)
    key = np.array([-1, -1, -1, -1, -1, -1, -1, -1, 0, 1, -1, -1, 2, 3, 4, -1, -1, -1, 5, -1, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15, -1,
                    -1, 16, 17, 18])
    assert np.array_equal(lut[ids], key[np.digitize(ids, np.arange(-1, 34), right=True)]) and lut[255] == -1
    t = seg_mask_lut("trainid")
    assert t[255] == -1 and np.array_equal(t[:255], np.arange(255))
    with pytest.raises(ValueError):
        seg_mask_lut("ade20k")


def test_mask_validation_raises_before_upload():
    """a Cityscapes mask with an id outside the reference's mapping fails at construction, on the host"""
    from multiyolov5_b200.utils.datasets import DeviceSegCache
    img = np.zeros((4, 6, 3), np.uint8)
    bad = np.zeros((4, 6), np.uint8)
    bad[1, 2] = 40
    with pytest.raises(ValueError, match="40"):
        DeviceSegCache([img], [bad], mask_map="cityscapes")
    with pytest.raises(ValueError):
        DeviceSegCache([img, img], [bad, bad], mask_map=["trainid"])
    with pytest.raises(ValueError):
        DeviceSegCache([img], [np.zeros((4, 5), np.uint8)])
    with pytest.raises(ValueError):
        DeviceSegCache([img.astype(np.int16)], [bad], mask_map="trainid")


def test_seg_item_layout():
    import ctypes as C
    from multiyolov5_b200 import _lib
    assert C.sizeof(_lib.SegItem) == 1120 and _lib.SegItem.lsum.offset == 88 and _lib.SegItem.lut.offset == 96
