"""CPU: the mode='val' segmentation item restatement (oracle/restate_seg_val.py) against the reference's own items
(tests/golden/seg_val_cases.npz, oracle/make_golden_seg_val.py), the host geometry of SegAugmenter.val against the geometry the reference
used, the tuple crop_size refusal, and the batch order of train.SegValBatches."""
import json
import os
import random

import numpy as np
import pytest
import torch

from oracle import restate_seg_val as rv

GOLD = os.path.join(os.path.dirname(__file__), "golden")
CASES = ["citys", "citys_c63", "citysbdd"]


def _golden():
    g = np.load(os.path.join(GOLD, "seg_val_cases.npz"))
    return g, json.loads(bytes(g["meta_json"]).decode())


def _kind(c, j):
    """CitySegmentation maps every item as Cityscapes ids; CityBddSegmentation its .jpg items as train ids"""
    return "trainid" if c["loader"] == "citysbdd" and c["files"][j].endswith("jpg") else "cityscapes"


def _item_sources(g, c, j):
    si, mi = c["sources"][j]
    return g[f"src_{si}"], g[f"mask_{mi}"]


@pytest.mark.parametrize("name", CASES)
def test_restatement_matches_reference_items(name):
    """every item bit for bit, and mode='val' consumes no `random` or torch draw"""
    g, meta = _golden()
    c = meta["cases"][name]
    random.seed(c["seed"])
    torch.manual_seed(c["seed"])
    for j in range(len(c["files"])):
        img, mask = _item_sources(g, c, j)
        im, lab = rv.val_item(img, mask, rv.mask_lut(_kind(c, j)), c["crop_size"])
        ref = g[f"{name}_img_{j}"].astype(np.float32) / np.float32(255)
        assert im.dtype == np.float32 and im.shape == ref.shape and np.array_equal(im, ref), (name, j, int((im != ref).sum()))
        assert lab.dtype == np.int64 and np.array_equal(lab, g[f"{name}_lab_{j}"].astype(np.int64)), (name, j)
    assert random.random() == c["next_random"] and float(torch.rand(1)) == c["next_torch"], "mode='val' drew random numbers"
    random.seed(c["seed"])
    torch.manual_seed(c["seed"])
    assert random.random() == c["next_random"] and float(torch.rand(1)) == c["next_torch"]


@pytest.mark.parametrize("name", CASES)
def test_host_geometry_equals_the_references(name):
    """the reference's Image.resize sizes (image BILINEAR, mask NEAREST) and crop boxes against seg_val_geometry and the restatement"""
    Image = pytest.importorskip("PIL.Image")
    from multiyolov5_b200.utils.datasets import seg_val_geometry
    g, meta = _golden()
    c = meta["cases"][name]
    crop = c["crop_size"]
    for j, calls in enumerate(c["geometry"]):
        h, w = _item_sources(g, c, j)[0].shape[:2]
        ow, oh, x1, y1 = seg_val_geometry(w, h, crop)
        assert (ow, oh, x1, y1) == rv.val_geometry(w, h, crop)
        box = [x1, y1, x1 + crop, y1 + crop]
        assert calls == [["resize", [ow, oh], int(Image.BILINEAR)], ["resize", [ow, oh], int(Image.NEAREST)], ["crop", box],
                         ["crop", box]], (name, j, calls)


def test_geometry_rounds_half_to_even():
    """(w' - c) / 2 = k + 0.5 goes to the even neighbour: 0.5 -> 0, 1.5 -> 2, 24.5 -> 24, 33.5 -> 34; squares go the portrait way"""
    from multiyolov5_b200.utils.datasets import seg_val_geometry
    assert seg_val_geometry(49, 48, 64) == (65, 64, 0, 0)
    assert seg_val_geometry(268, 256, 64) == (67, 64, 2, 0)
    assert seg_val_geometry(40, 71, 64) == (64, 113, 0, 24)
    assert seg_val_geometry(262, 128, 64) == (131, 64, 34, 0)
    assert seg_val_geometry(2048, 1024, 512) == (1024, 512, 256, 0)
    assert seg_val_geometry(1280, 720, 512) == (910, 512, 199, 0)
    assert seg_val_geometry(7, 7, 5) == (5, 5, 0, 0)
    for w, h, c in [(1000, 999, 37), (333, 1001, 64), (1280, 720, 513), (3, 2, 64)]:
        assert seg_val_geometry(w, h, c) == rv.val_geometry(w, h, c)


class _HostCache:
    """what SegAugmenter and SegValBatches read from a DeviceSegCache, without a device"""

    def __init__(self, shapes):
        self.shapes, self.n = shapes, len(shapes)


def test_tuple_crop_raises():
    """the reference raises TypeError on a tuple crop_size (recorded for get_citys_loader's default and get_custom_loader);
    SegAugmenter.val and SegValBatches refuse it with ValueError naming that, before any device work"""
    from multiyolov5_b200.train import SegValBatches
    from multiyolov5_b200.utils.datasets import SegAugmenter
    _, meta = _golden()
    assert meta["raises"]["get_citys_loader"]["type"] == "TypeError" and meta["raises"]["get_citys_loader"]["crop_size"] == [1024, 512]
    assert meta["raises"]["get_custom_loader"]["type"] == "TypeError" and meta["raises"]["get_custom_loader"]["crop_size"] == [64, 64]
    cache = _HostCache([(100, 200)])
    aug = SegAugmenter(cache, base_size=128, preset="citysbdd")
    for crop in [(1024, 512), [64, 64]]:
        with pytest.raises(ValueError, match="TypeError"):
            aug.val([0], crop)
        with pytest.raises(ValueError, match="TypeError"):
            SegValBatches(aug, 4, mode="val", crop_size=crop)
    for crop in [None, 0, -4, 64.0, "64", True]:
        with pytest.raises(ValueError):
            aug.val([0], crop)
        with pytest.raises(ValueError):
            SegValBatches(aug, 4, mode="val", crop_size=crop)
    with pytest.raises(ValueError):
        SegValBatches(aug, 4, mode="train", crop_size=64)
    with pytest.raises(ValueError):
        SegValBatches(aug, 0, mode="val", crop_size=64)


class _FakeSegAug:
    """records each batch's indices and which mode built it"""

    def __init__(self, shapes):
        self.cache = _HostCache(shapes)
        self.calls = []

    def val(self, indices, crop_size, out_dtype=torch.float32):
        self.calls.append(("val", list(indices), crop_size, out_dtype))
        return indices, crop_size

    def testval(self, indices, out_dtype=torch.float32):
        self.calls.append(("testval", list(indices), None, out_dtype))
        return indices, None


@pytest.mark.parametrize("n,B", [(10, 4), (9, 4), (8, 4), (5, 1), (3, 8)])
def test_seg_val_batches_order_is_the_dataloaders(n, B):
    """DataLoader(shuffle=False, drop_last=False): items in order, the last batch partial; iterable again for every pass"""
    from multiyolov5_b200.train import SegValBatches
    aug = _FakeSegAug([(720, 1280) if k % 3 else (1024, 2048) for k in range(n)])
    sv = SegValBatches(aug, B, mode="val", crop_size=512, out_dtype=torch.float16)
    want = [idx.tolist() for idx in torch.utils.data.DataLoader(range(n), batch_size=B, shuffle=False, drop_last=False)]
    for _ in range(2):
        assert [b[0] for b in sv] == want
    assert aug.calls == [("val", w, 512, torch.float16) for w in want] * 2 and len(sv) == len(want)


def test_seg_val_batches_draw_nothing():
    """the order is fixed: no DataLoader sampler draws from torch's generator"""
    from multiyolov5_b200.train import SegValBatches
    sv = SegValBatches(_FakeSegAug([(8, 8)] * 7), 3, mode="val", crop_size=8)
    random.seed(3)
    torch.manual_seed(3)
    list(sv)
    a, t = random.random(), float(torch.rand(1))
    random.seed(3)
    torch.manual_seed(3)
    assert a == random.random() and t == float(torch.rand(1))


def test_seg_val_batches_testval():
    """mode='testval' builds aug.testval batches, the scripts' batch 4 over one source size and batch 1 over sizes that vary; a testval
    batch whose items differ in source size raises at construction, as default_collate would at that batch"""
    from multiyolov5_b200.train import SegValBatches
    aug = _FakeSegAug([(1024, 2048)] * 6)
    sv = SegValBatches(aug, 4, mode="testval")
    assert [b[0] for b in sv] == [[0, 1, 2, 3], [4, 5]] and all(c[0] == "testval" for c in aug.calls)
    mixed = _FakeSegAug([(1024, 2048), (1024, 2048), (720, 1280), (600, 800), (600, 800)])
    assert [b[0] for b in SegValBatches(mixed, 1, mode="testval")] == [[k] for k in range(5)]
    assert [b[0] for b in SegValBatches(mixed, 2, mode="val", crop_size=64)] == [[0, 1], [2, 3], [4]]
    with pytest.raises(ValueError, match="source sizes"):
        SegValBatches(mixed, 2, mode="testval")
    with pytest.raises(ValueError, match="source sizes"):
        SegValBatches(mixed, 4, mode="testval")


def test_fixtures_cover_every_branch():
    """landscape, portrait and square sources; down-scales of 2x and more and up-scales from a short side below the crop; centre crops
    at k + 0.5 for even and odd k and at whole numbers; a City+BDD .jpg item whose mask holds 255; Cityscapes masks with every id and 255"""
    g, meta = _golden()
    seen = dict(landscape=False, portrait=False, square=False, down2=False, up=False, half_even=False, half_odd=False, whole=False,
                jpg255=False, ids=set())
    for name in CASES:
        c = meta["cases"][name]
        crop = c["crop_size"]
        for j in range(len(c["files"])):
            img, mask = _item_sources(g, c, j)
            h, w = img.shape[:2]
            seen["landscape"] |= w > h
            seen["portrait"] |= h > w
            seen["square"] |= h == w
            seen["down2"] |= min(h, w) >= 2 * crop
            seen["up"] |= min(h, w) < crop
            ow, oh = rv.val_geometry(w, h, crop)[:2]
            for d in (ow - crop, oh - crop):
                k, odd = divmod(d, 2)
                seen["half_even"] |= bool(odd) and k % 2 == 0
                seen["half_odd"] |= bool(odd) and k % 2 == 1
                seen["whole"] |= d > 0 and not odd
            if _kind(c, j) == "trainid":
                seen["jpg255"] |= bool((mask == 255).any()) and bool((g[f"{name}_lab_{j}"] == -1).any())
            else:
                seen["ids"] |= set(np.unique(mask).tolist())
    ids = seen.pop("ids")
    assert all(seen.values()), seen
    assert ids == set(range(34)) | {255}
    assert any(min(g[f"src_{si}"].shape[:2]) >= 4 * meta["cases"]["citys"]["crop_size"] for si, _ in meta["cases"]["citys"]["sources"])
    assert set(meta["raises"]) == {"get_citys_loader", "get_custom_loader"}
