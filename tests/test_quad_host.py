"""CPU: `--quad`'s collate (LoadImagesAndLabels.collate_fn4).  The numpy restatement (oracle/restate_quad.py) against every batch the
reference collated (tests/golden/quad_cases.npz, oracle/make_golden_quad.py), with its draw order; the labels of both branches and of the
partial batch; the error below 4 items; and the integer x2 up-scale, proven exact against torch's float32 arithmetic and checked against
torch's CPU F.interpolate."""
import json
import os
import random

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import restate_quad as rq

GOLD = os.path.join(os.path.dirname(__file__), "golden")
CASES = ["mosaic", "mixup", "rect"]


def _golden():
    g = np.load(os.path.join(GOLD, "quad_cases.npz"))
    return g, json.loads(bytes(g["meta_json"]).decode())


def _rng(g, name, b):
    """a random.Random in the state collate_fn4 started batch b from"""
    r = random.Random()
    r.setstate((3, tuple(int(v) for v in g[f"{name}_state_{b}"]), None))
    return r


@pytest.mark.parametrize("name", CASES)
def test_restatement_matches_reference_batches_and_draws(name):
    g, meta = _golden()
    c = meta["cases"][name]
    for b in range(c["n_batches"]):
        rng = _rng(g, name, b)
        img4, t4 = rq.collate_quad_np(g[f"{name}_items_{b}"], g[f"{name}_targets_{b}"], rng)
        ref_img, ref_t = g[f"{name}_img4_{b}"], g[f"{name}_targets4_{b}"]
        assert img4.shape == ref_img.shape and np.array_equal(img4, ref_img), (name, b)
        assert t4.dtype == ref_t.dtype == np.float32 and np.array_equal(t4, ref_t), (name, b)
        assert rng.random() == c["next_random"][b], (name, b)      # one draw per quad, none more


def test_fixtures_cover_both_branches_full_and_partial_batches():
    g, meta = _golden()
    for name in CASES:
        c = meta["cases"][name]
        assert [len(g[f"{name}_items_{b}"]) for b in range(c["n_batches"])] == [8, 6]
        assert [len(t) for t in c["tiles"]] == [2, 1]
        flat = sum(c["tiles"], [])
        assert any(flat) and not all(flat), name
        for b, tiles in enumerate(c["tiles"]):
            rng = _rng(g, name, b)
            assert [rng.random() >= 0.5 for _ in tiles] == tiles
    shapes = [tuple(s) for s in g["rect_batch_shapes"].tolist()]
    assert shapes == [(32, 64), (64, 32)]
    assert g["rect_img4_0"].shape[2:] == (64, 128) and g["rect_img4_1"].shape[2:] == (128, 64)


@pytest.mark.parametrize("name", CASES)
def test_labels_of_each_branch(name):
    """upsampled quad: item 4q's rows unchanged; tiled quad: the four items' rows shifted by (x + 1 for the right column, y + 1 for the
    bottom row) and halved; the partial batch keeps only items 0..3 and column 0 is the quad index"""
    g, meta = _golden()
    c = meta["cases"][name]
    for b, tiles in enumerate(c["tiles"]):
        t, t4 = g[f"{name}_targets_{b}"], g[f"{name}_targets4_{b}"]
        assert t4[:, 0].tolist() == sorted(t4[:, 0].tolist()) and set(t4[:, 0].astype(int)) <= set(range(len(tiles)))
        for q, tile in enumerate(tiles):
            got = t4[t4[:, 0] == q]
            if not tile:
                want = t[t[:, 0] == 4 * q].copy()
            else:
                parts = []
                for k in range(4):
                    lb = t[t[:, 0] == 4 * q + k].copy()
                    lb[:, 3] += np.float32(k % 2)
                    lb[:, 2] += np.float32(k // 2)
                    lb[:, 2:] *= np.float32(0.5)
                    parts.append(lb)
                want = np.concatenate(parts, 0)
            want[:, 0] = q
            assert np.array_equal(got, want), (name, b, q, tile)
        if len(g[f"{name}_items_{b}"]) == 6:                     # the partial batch: items 4 and 5 are dropped
            assert len(t4) == sum(len(t[t[:, 0] == i]) for i in (range(4) if tiles[0] else [0]))


def test_fewer_than_four_items_raise():
    imgs = np.zeros((3, 3, 8, 8), np.uint8)
    with pytest.raises(ValueError):
        rq.collate_quad_np(imgs, np.zeros((0, 6), np.float32))


def test_bilinear_x2_arithmetic_is_exact_in_float32():
    """Why floor(integer sum / 16) equals torch's float32 result whatever its evaluation order.
    1. The source coordinates torch computes (area_pixel_compute_source_index with scale 1/2, in float32) give the weights {0, 1/4, 3/4, 1}
       at every output index of axes up to 4096, and the two taps of each index are the ones of restate_quad._taps.
    2. So every product of a uint8 value with a 1-D weight or with a product of two weights is k / 16 for an integer 0 <= k < 4096, and
       every partial sum of such non-negative products with weights summing to at most 1 stays below 256; differences (a lerp form) stay
       above -256.  Every such multiple of 1/16 in (-256, 256) is a float32, so each operation's exact result is representable and IEEE
       rounding returns it unchanged: the float32 result is the exact rational sum, and the uint8 cast truncates it."""
    for n in (1, 2, 3, 7, 64, 1023, 1024, 4096):
        d = np.arange(2 * n, dtype=np.float32)
        src = np.maximum(np.float32(0.5) * (d + np.float32(0.5)) - np.float32(0.5), np.float32(0))
        i1 = src.astype(np.int64)
        l1 = src - i1.astype(np.float32)
        i2 = np.minimum(i1 + 1, n - 1)                   # torch's h1p: the second tap repeats the first at the last index
        l0 = np.float32(1) - l1
        assert set(np.unique(l1).tolist()) <= {0.0, 0.25, 0.75}
        a, b, wa = rq._taps(n)
        for j in range(2 * n):                           # restate_quad's (a, b, wa / 4) is the same combination of the same inputs
            torch_taps, mine = {}, {}
            for idx, wt in ((i1[j], l0[j]), (i2[j], l1[j])):
                torch_taps[int(idx)] = torch_taps.get(int(idx), 0.0) + float(wt)
            for idx, wt in ((a[j], wa[j] / 4), (b[j], (4 - wa[j]) / 4)):
                mine[int(idx)] = mine.get(int(idx), 0.0) + float(wt)
            assert {k: v for k, v in torch_taps.items() if v} == {k: v for k, v in mine.items() if v}, (n, j)
    k = np.arange(-4095, 4096)
    assert np.array_equal(np.float32(k / 16).astype(np.float64), k / 16)
    w = np.array([0, 1, 3, 4], np.float32) / np.float32(4)
    w2 = (w[:, None] * w[None, :]).ravel()
    v = np.arange(256, dtype=np.float32)
    prods = (v[:, None] * np.concatenate([w, w2])[None, :]).astype(np.float64)
    assert np.array_equal(prods * 16, np.round(prods * 16)) and prods.max() <= 255


@pytest.mark.parametrize("shape", [(1, 1), (2, 3), (7, 5), (16, 16), (33, 64), (48, 31), (64, 96)])
def test_integer_x2_equals_torch_cpu_interpolate(shape):
    rs = np.random.RandomState(shape[0] * 100 + shape[1])
    img = rs.randint(0, 256, (3,) + shape).astype(np.uint8)
    img[:, ::3] = 255                                                # extremes next to each other
    img[:, 1::5] = 0
    t = torch.from_numpy(img)
    ref = F.interpolate(t.float()[None], scale_factor=2., mode='bilinear', align_corners=False)[0].type(t.type())
    assert np.array_equal(rq.upsample2x_u8(img), ref.numpy()), shape
