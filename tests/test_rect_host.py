"""CPU: `--rect` training batches (LoadImagesAndLabels(augment=True, rect=True)).  The plan (rect_plan: order, batch index, batch shapes),
the restatement's items (oracle/restate_rect.py getitem_rect) and the host half of DetRectLoader (draws, letterbox and warp geometry,
labels) against the reference's own batches (tests/golden/rect_cases.npz, oracle/make_golden_rect.py); the DDP order against torch's
DistributedSampler; a batch of mixed shapes raises."""
import json
import os
import random

import numpy as np
import pytest
import torch

from oracle import restate_augment as ra
from oracle import restate_rect as rr

GOLD = os.path.join(os.path.dirname(__file__), "golden")
CASES = ["scratch", "stress", "flipud", "identity"]


def _golden():
    g = np.load(os.path.join(GOLD, "rect_cases.npz"))
    return g, json.loads(bytes(g["meta_json"]).decode())


def _source(g, meta, name):
    n = len(meta["shapes"])
    c = meta["cases"][name]
    return ra.Source([g[f"src_{k}"] for k in range(n)], [g[f"labels_{k}"] for k in range(n)], c["img_size"], c["hyp"])


class _HostCache:
    """what DetRectLoader reads from a DeviceImageCache(augment=True), without a device (pointers are placeholders)"""

    def __init__(self, src, shapes0):
        self.img_size, self.n, self.labels, self.augment = src.img_size, src.n, src.labels, True
        self.shapes0 = [tuple(s) for s in shapes0]
        self.shapes = [im.shape[:2] for im in src.cache]

    def ptr(self, i):
        return 4096 * (i + 1)


def _loader(g, meta, name):
    from multiyolov5_b200.utils.datasets import DetRectLoader
    c = meta["cases"][name]
    src = _source(g, meta, name)
    return src, DetRectLoader(_HostCache(src, meta["shapes"]), c["hyp"], c["batch_size"])


def _batches(n, bs):
    return [list(range(k, min(k + bs, n))) for k in range(0, n, bs)]


@pytest.mark.parametrize("name", CASES)
def test_plan_matches_reference(name):
    from multiyolov5_b200.utils.datasets import rect_plan
    g, meta = _golden()
    c = meta["cases"][name]
    order, bi, shapes = rect_plan(meta["shapes"], c["img_size"], c["batch_size"], 32, 0.0)
    assert np.array_equal(order, g[f"{name}_order"]) and np.array_equal(shapes, g[f"{name}_batch_shapes"])
    assert np.array_equal(bi, np.arange(len(order)) // c["batch_size"])
    r_order, r_bi, r_shapes = rr.rect_batch_shapes(meta["shapes"], c["img_size"], c["batch_size"])
    assert np.array_equal(order, r_order) and np.array_equal(bi, r_bi) and np.array_equal(shapes, r_shapes)
    _, loader = _loader(g, meta, name)
    assert np.array_equal(loader.order, order) and np.array_equal(loader.batch, bi) and np.array_equal(loader.batch_shapes, shapes)
    assert len(loader) == c["n_batches"]


def test_fixtures_cover_every_batch_kind():
    g, meta = _golden()
    ar = np.array([h / w for h, w in meta["shapes"]])
    assert len(np.unique(ar)) == len(ar)                              # no ties: the order does not depend on the CPU
    for name in CASES:
        c = meta["cases"][name]
        order, bs = g[f"{name}_order"], c["batch_size"]
        kinds = []
        for pos in _batches(len(order), bs):
            a = ar[order[pos]]
            kinds.append("landscape" if a.max() < 1 else "portrait" if a.min() > 1 else "mixed")
        assert kinds[:3] == ["landscape", "mixed", "portrait"] and len(order) % bs, (name, kinds)
        assert g[f"{name}_batch_shapes"][1].tolist() == [c["img_size"] // 32 * 32 + (32 if c["img_size"] % 32 else 0)] * 2
    hyps = {n: meta["cases"][n]["hyp"] for n in CASES}
    assert hyps["stress"]["degrees"] == 10 and hyps["stress"]["shear"] == 5 and hyps["flipud"]["flipud"] == 1
    assert all(hyps["identity"][k] == 0 for k in ("translate", "scale", "degrees", "shear"))
    assert any(meta["cases"][n]["img_size"] % 32 for n in CASES)      # the letterbox up-scales too


@pytest.mark.parametrize("name", CASES)
def test_restatement_matches_reference_batches(name):
    g, meta = _golden()
    c = meta["cases"][name]
    src = _source(g, meta, name)
    order, shapes = g[f"{name}_order"], g[f"{name}_batch_shapes"]
    random.seed(c["seed"])
    np.random.seed(c["seed"])
    for b, pos in enumerate(_batches(len(order), c["batch_size"])):
        items = [rr.getitem_rect(src, int(order[p]), shapes[b]) for p in pos]
        img = np.stack([i for i, _ in items])
        ref = g[f"{name}_img_{b}"]
        assert img.shape == ref.shape and np.array_equal(img, ref), (name, b, int((img != ref).sum()))
        t = np.concatenate([np.concatenate((np.full((len(lab), 1), k, np.float32), lab), 1) for k, (_, lab) in enumerate(items)])
        assert np.array_equal(t, g[f"{name}_targets_{b}"]), (name, b)
    assert random.random() == c["next_random"] and float(np.random.random()) == c["next_np"], "random number consumption differs"


@pytest.mark.parametrize("name", CASES)
def test_host_draws_geometry_and_labels_match_reference(name):
    """DetRectLoader.item (host half of the device path): the reference's targets and draws over the whole epoch; per item the warp's
    inverse matrix is the restatement's and its one tile is the letterboxed image inside the batch shape"""
    from multiyolov5_b200.utils.datasets import letterbox_geometry
    g, meta = _golden()
    c = meta["cases"][name]
    src, loader = _loader(g, meta, name)
    loader.aug._resized = lambda index, nh, nw: 1 << 40                # the letterbox's up-scaling resize is a device launch
    random.seed(c["seed"])
    np.random.seed(c["seed"])
    resized = 0
    for b, pos in enumerate(_batches(loader.n, c["batch_size"])):
        shape = loader.batch_shapes[b]
        labs = []
        for k, p in enumerate(pos):
            index = int(loader.order[p])
            r_state = random.getstate()
            M, out_w, out_h, _ = ra.affine_params(int(shape[0]), int(shape[1]), (0, 0), c["hyp"])
            random.setstate(r_state)
            it, lab = loader.item(p)
            assert (out_h, out_w) == tuple(int(v) for v in shape)
            w = it.warp[0]
            assert it.n_warps == 1 and w.n_tiles == 1 and list(w.minv) == list(ra.invert_affine(M[:2])), (name, b, k)
            (nw, nh), _, _, (top, _, left, _) = letterbox_geometry(src.cache[index].shape[:2], shape, auto=False, scaleup=True)
            assert list(w.rect[0]) == [left, top, left + nw, top + nh] and list(w.off[0]) == [left, top] and w.src_w[0] == nw
            resized += (nh, nw) != src.cache[index].shape[:2]
            assert w.src[0] == (1 << 40 if (nh, nw) != src.cache[index].shape[:2] else 4096 * (index + 1))
            labs.append(np.concatenate((np.full((len(lab), 1), k, np.float32), lab), 1))
        assert np.array_equal(np.concatenate(labs), g[f"{name}_targets_{b}"]), (name, b)
    assert (resized > 0) == (c["img_size"] % 32 != 0), resized
    assert random.random() == c["next_random"] and float(np.random.random()) == c["next_np"], "random number consumption differs"


def test_order_of_tied_aspect_ratios_is_this_hosts_argsort():
    from multiyolov5_b200.utils.datasets import rect_plan
    rs = np.random.RandomState(0)
    shapes0 = [[(1024, 2048), (720, 1280), (600, 600), (900, 600)][k] for k in rs.randint(0, 4, 50)]
    order, bi, shapes = rect_plan(shapes0, 1024, 8)
    ar = np.array([h / w for h, w in shapes0], np.float64)
    assert np.array_equal(order, ar.argsort()) and len(shapes) == 7
    assert [1024 // 2, 1024] in shapes.tolist()                       # Cityscapes 2048 x 1024 at 1024: 512 x 1024


@pytest.mark.parametrize("world_size", [2, 3, 8])
def test_ddp_order_is_distributed_samplers(world_size):
    from torch.utils.data import DistributedSampler
    g, meta = _golden()
    _, loader = _loader(g, meta, "scratch")
    for epoch in (0, 1, 5):
        for rank in range(world_size):
            sampler = DistributedSampler(range(loader.n), num_replicas=world_size, rank=rank, shuffle=True, seed=0)
            sampler.set_epoch(epoch)
            assert loader.epoch_positions(epoch, rank, world_size) == list(sampler), (epoch, rank, world_size)
    with pytest.raises(ValueError):
        loader.epoch_positions(0, world_size, world_size)


def test_batch_of_mixed_shapes_raises():
    g, meta = _golden()
    _, loader = _loader(g, meta, "scratch")
    state = random.getstate()
    with pytest.raises(ValueError, match="torch.stack"):
        loader([0, loader.n - 1])
    assert random.getstate() == state                                 # refused before any draw
    with pytest.raises(ValueError):
        loader([loader.n])
    assert loader.shape_of([0, 1, 2]).tolist() == loader.batch_shapes[0].tolist()


def test_loader_needs_the_training_cache():
    from multiyolov5_b200.utils.datasets import DetRectLoader
    g, meta = _golden()
    src = _source(g, meta, "scratch")
    cache = _HostCache(src, meta["shapes"])
    cache.augment = False
    with pytest.raises(ValueError, match="augment=True"):
        DetRectLoader(cache, meta["cases"]["scratch"]["hyp"], 3)


def test_val_plan_keeps_its_batches():
    """det_val_plan takes its order and shapes from rect_plan; the validation arithmetic (pad 0.5) is unchanged"""
    from multiyolov5_b200.utils.datasets import det_val_plan, rect_plan
    g, meta = _golden()
    shapes0 = [tuple(s) for s in meta["shapes"]]
    labels = [g[f"labels_{k}"] for k in range(len(shapes0))]
    order, shapes, batches = det_val_plan(shapes0, shapes0, labels, 96, 3)
    r_order, _, r_shapes = rr.rect_batch_shapes(shapes0, 96, 3, 32, 0.5)
    assert np.array_equal(order, r_order) and np.array_equal(shapes, r_shapes) and len(batches) == len(shapes)
    assert np.array_equal(rect_plan(shapes0, 96, 3, 32, 0.5)[2], shapes)
    assert torch.equal(torch.as_tensor(shapes), torch.as_tensor(r_shapes))


def test_single_cls_zeroes_the_class_and_nothing_else():
    """single_cls (the reference sets every label's class to 0 at construction): the same draws, boxes and filtering, class 0"""
    from multiyolov5_b200.utils.datasets import DetRectLoader
    g, meta = _golden()
    c = meta["cases"]["stress"]
    src, loader = _loader(g, meta, "stress")
    one = DetRectLoader(_HostCache(src, meta["shapes"]), c["hyp"], c["batch_size"], single_cls=True)
    for p in range(loader.n):
        random.seed(p)
        np.random.seed(p)
        _, want = loader.item(p)
        random.seed(p)
        np.random.seed(p)
        _, got = one.item(p)
        assert np.array_equal(got[:, 1:], want[:, 1:]) and (got[:, 0] == 0).all(), p
    assert all(len(lb) and lb[:, 0].any() for lb in src.labels[:3])     # the source classes are untouched
