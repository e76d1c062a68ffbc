"""CPU: the detection validation batches' host side.  The INTER_AREA restatement (oracle/restate_val_batches.py) is pinned to cv2 itself
and to the unmodified reference's cached images (tests/golden/val_batch_cases.npz); the loader's host arithmetic (det_val_plan: order,
batch shapes, letterbox geometry, labels, shapes) and the restated batch images are pinned to the reference's batches.  numpy's argsort
is not stable and its tie order depends on the CPU, so items are compared keyed by source index, and the order is checked against
np.argsort on this host."""
import json
import os

import numpy as np
import pytest

from multiyolov5_b200.utils.datasets import det_val_plan
from oracle import restate_val_batches as RV

GOLD = os.path.join(os.path.dirname(__file__), "golden", "val_batch_cases.npz")


def _cases():
    z = np.load(GOLD)
    return z, json.loads(bytes(z["meta_json"]).decode())


def _sources(z, meta):
    n = len(meta["shapes"])
    return [z[f"src_{k}"] for k in range(n)], [z[f"labels_{k}"] for k in range(n)]


def _sweep():
    out = [(13, W0, 5, W) for W0 in range(1, 24) for W in range(1, W0 + 1)]        # every residue of W0 mod W
    out += [(H0, 7, H, 3) for H0 in range(1, 20) for H in range(1, H0 + 1)]
    out += [(720, 1280, 576, 1024), (100, 125, 80, 100),                            # 1.25
            (1024, 2048, 320, 640), (320, 640, 100, 200), (330, 512, 103, 160),     # 3.2
            (1080, 1920, 360, 640), (96, 129, 32, 43), (64, 128, 16, 32),           # 3, 4
            (60, 90, 30, 30), (90, 60, 30, 30), (41, 37, 40, 36), (37, 41, 36, 1)]  # mixed integral, near 1, one column
    return out


def test_area_restatement_matches_cv2():
    cv2 = pytest.importorskip("cv2")
    rs = np.random.RandomState(0)
    for H0, W0, H, W in _sweep():
        img = rs.randint(0, 256, (H0, W0, 3)).astype(np.uint8)
        ref = cv2.resize(img, (W, H), interpolation=cv2.INTER_AREA)
        assert np.array_equal(RV.cv2_resize_area_u8(img, W, H), ref), (H0, W0, H, W, RV.area_path(H0, W0, H, W))


def test_area_restatement_paths_and_limits():
    assert RV.area_path(1024, 2048, 320, 640) == "general" and RV.area_path(1080, 1920, 360, 640) == "fast"
    assert RV.area_path(96, 192, 48, 96) == "fast2" and RV.area_path(50, 70, 50, 70) == "copy"
    with pytest.raises(ValueError):
        RV.cv2_resize_area_u8(np.zeros((10, 10, 3), np.uint8), 11, 5)


def test_load_image_restatement_matches_reference_cache():
    z, meta = _cases()
    srcs, _ = _sources(z, meta)
    for name, c in meta["cases"].items():
        for k, src in enumerate(srcs):
            assert np.array_equal(RV.load_image_val(src, c["img_size"]), z[f"{name}_cache_{k}"]), (name, k)


def _plan(z, meta, name):
    c = meta["cases"][name]
    srcs, labels = _sources(z, meta)
    shapes0 = [s.shape[:2] for s in srcs]
    shapes = [z[f"{name}_cache_{k}"].shape[:2] for k in range(len(srcs))]
    return det_val_plan(shapes0, shapes, labels, c["img_size"], c["batch_size"], 32, 0.5, c["single_cls"])


def _rows(t, pos):
    return t[t[:, 0] == pos, 1:]


@pytest.mark.parametrize("name", ["main", "single_cls", "big_batch"])
def test_plan_matches_reference(name):
    z, meta = _cases()
    c = meta["cases"][name]
    order, batch_shapes, batches = _plan(z, meta, name)
    ar = np.array([h / w for h, w in meta["shapes"]], np.float64)
    assert np.array_equal(order, np.argsort(ar))                 # the reference's call on this host
    assert np.array_equal(batch_shapes, z[f"{name}_batch_shapes"])
    assert len(batches) == c["n_batches"]
    for b, batch in enumerate(batches):
        paths = z[f"{name}_paths_{b}"].tolist()
        assert sorted(batch.indices) == sorted(paths)            # ties are permuted within one batch only
        ref_t, ref_s = z[f"{name}_targets_{b}"], z[f"{name}_shapes_{b}"]
        assert batch.targets.dtype == np.float32 and len(batch.targets) == len(ref_t)
        for pos, i in enumerate(batch.indices):
            rpos = paths.index(i)
            assert np.array_equal(_rows(batch.targets, pos), _rows(ref_t, rpos)), (b, i)
            (h0, w0), ((gh, gw), (pw, ph)) = batch.shapes[pos]
            assert np.array_equal(np.array([h0, w0, gh, gw, pw, ph], np.float64), ref_s[rpos]), (b, i)
        if c["single_cls"] and len(batch.targets):
            assert (batch.targets[:, 1] == 0).all()


@pytest.mark.parametrize("name", ["main", "single_cls", "big_batch"])
def test_restated_batch_images_match_reference(name):
    z, meta = _cases()
    _, batch_shapes, batches = _plan(z, meta, name)
    for b, batch in enumerate(batches):
        imgs = RV.val_batch_images([z[f"{name}_cache_{i}"] for i in batch.indices], batch_shapes[b])
        paths = z[f"{name}_paths_{b}"].tolist()
        ref = z[f"{name}_img_{b}"]
        assert imgs.shape == ref.shape
        for pos, i in enumerate(batch.indices):
            assert np.array_equal(imgs[pos], ref[paths.index(i)]), (b, i)


def test_plan_batch_shape_branches_and_short_batches():
    z, meta = _cases()
    _, bs_main, batches = _plan(z, meta, "main")
    assert [len(b.indices) for b in batches] == [4, 4, 4, 1]               # 4 does not divide 13
    kinds = {("landscape" if h < w else "portrait" if h > w else "square") for h, w in bs_main.tolist()}
    assert kinds == {"landscape", "portrait", "square"}
    _, _, batches = _plan(z, meta, "big_batch")
    assert len(batches) == 1 and len(batches[0].indices) == 13              # batch size 32 > n
