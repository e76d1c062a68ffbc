"""Host: the numpy restatement of --image-weights (oracle/restate_image_weights.py), which fixes the device kernels' arithmetic and
order, against the reference's own results (tests/golden/image_weights_cases.npz), numpy's summation order against numpy itself, the
C-ABI exports, and the DDP broadcast of ImageWeights.draw over gloo."""
import ctypes as C
import os
import random
import socket

import numpy as np
import pytest
import torch

from oracle import restate_image_weights as riw

GOLD = os.path.join(os.path.dirname(__file__), "golden")
NAMES = ["nc1_single", "nc5", "nc10_city", "nc80", "nc130", "all_maps_one", "n1"]


def _cases():
    return riw.load_cases(os.path.join(GOLD, "image_weights_cases.npz"))


def test_fixture_has_every_case():
    cases, aug_meta, aug = _cases()
    assert set(NAMES) <= set(cases) and {"aug_mosaic", "aug_single"} <= set(aug_meta)
    assert {c["nc"] for c in cases.values()} >= {1, 5, 10, 80, 130}
    assert cases["all_maps_one"]["errors"] == ["Total of weights must be greater than zero"]
    assert cases["n1"]["n"] == 1 and cases["nc10_city"]["n"] == 2975
    assert all(cases[k]["epochs"] == 2 for k in ("nc5", "nc10_city", "nc80"))
    assert (np.concatenate(cases["nc1_single"]["labels"])[:, 0] == 0).all()
    assert (cases["nc5"]["e0_cw"] == 0).any()                                     # maps at 1.0: zero class weight
    assert any(len(x) == 0 for x in cases["nc5"]["labels"])                      # images without labels


def test_augmented_items_sources_are_augment_fixtures():
    """the augmented cases were made from make_golden_augment.sources(), which augment_cases.npz holds: the GPU tests read them there"""
    from oracle import make_golden_augment as mga
    a = np.load(os.path.join(GOLD, "augment_cases.npz"))
    imgs, labels = mga.sources()
    assert all(np.array_equal(im, a[f"src_{k}"]) and np.array_equal(lb, a[f"labels_{k}"])
               for k, (im, lb) in enumerate(zip(imgs, labels)))


@pytest.mark.parametrize("name", NAMES)
def test_restatement_equals_reference(name):
    c = _cases()[0][name]
    nc, labels = c["nc"], c["labels"]
    cwt = riw.class_weights(labels, nc)
    assert np.array_equal(cwt.view(np.int64), c["class_weights"].view(np.int64))
    random.seed(c["seed"])
    np.random.seed(c["seed"])
    for e in range(c["epochs"]):
        cw = riw.epoch_cw(cwt * nc, c[f"e{e}_maps"])
        assert np.array_equal(cw.view(np.int64), c[f"e{e}_cw"].view(np.int64)), e
        iw = riw.image_weights(labels, nc, cw)
        assert np.array_equal(iw.view(np.int64), c[f"e{e}_iw"].view(np.int64)), e
        if c["errors"][e] is None:
            idx, _, _ = riw.choices(iw, random)
            assert np.array_equal(idx, c[f"e{e}_indices"]), e
            empty = np.array([len(x) == 0 for x in labels])
            assert not empty[idx].any()                                          # an image without labels is never drawn
        else:
            with pytest.raises(ValueError, match=c["errors"][e]):
                riw.choices(iw, random)
    assert random.random() == c["next_random"] and float(np.random.random()) == c["next_np"]


def test_choices_equals_random_choices():
    rs = np.random.default_rng(0)
    w = rs.lognormal(0, 2, 5000) * (rs.random(5000) < 0.8)
    random.seed(5)
    want = random.choices(range(len(w)), weights=w, k=len(w))
    after = random.random()
    random.seed(5)
    idx, cum, total = riw.choices(w, random)
    assert idx.tolist() == want and random.random() == after
    assert total == cum[-1] and np.array_equal(cum, np.cumsum(w))


@pytest.mark.parametrize("nc", [1, 2, 7, 8, 9, 10, 16, 80, 127, 128, 129, 300])
def test_numpy_sum_order(nc):
    """np.add.reduce over the contiguous last axis: the pairwise sum of all nc values (from -0.0 below 8) added to 0.0.  Taking the
    first element as the initial value instead differs from numpy for every nc >= 7 on these inputs"""
    rs = np.random.default_rng(nc)
    a = rs.lognormal(0.0, 3.0, (4000, nc)) * (rs.random((4000, nc)) < 0.7)
    want = np.add.reduce(a, axis=1)
    assert np.array_equal(riw.numpy_sum_rows(a), want)
    assert all(riw.numpy_sum(r) == np.add.reduce(r) for r in a[:200])
    first = a[:, 0] + (riw.pairwise_rows(a[:, 1:]) if nc > 1 else 0.0)
    assert nc < 7 or not np.array_equal(first, want)


def test_numpy_sum_order_at_coco_scale():
    """the reference's (class_weights.reshape(1, nc) * class_counts).sum(1) over 118 287 images and 80 classes"""
    rs = np.random.default_rng(1)
    counts = rs.poisson(0.09, (118_287, 80))
    cw = rs.lognormal(0.0, 1.0, 80) * (rs.random(80) < 0.9)
    assert np.array_equal(riw.numpy_sum_rows(cw.reshape(1, 80) * counts), (cw.reshape(1, 80) * counts).sum(1))


def test_new_symbols_are_exported():
    from multiyolov5_b200 import _lib
    L = _lib.lib()
    for name in ("myolo_class_weights", "myolo_image_weights", "myolo_weighted_draw"):
        assert name in _lib.EXPORTS and hasattr(L, name)
    p = C.c_void_p(16)                                         # never dereferenced: the arguments are refused first
    assert L.myolo_class_weights(p, 1, _lib.IW_NC_MAX + 1, p, p, p, None) == -1
    assert b"1024" in L.myolo_last_error()
    assert L.myolo_image_weights(p, p, 1, p, 0, p, p, None) == -1
    assert L.myolo_weighted_draw(p, p, 0, p, p, p, p, None) == -1


def test_epoch_positions():
    from torch.utils.data import DistributedSampler

    from multiyolov5_b200.utils.datasets import ImageWeights
    iwts = ImageWeights(_StandInAug(_labels(37)))
    assert iwts.epoch_positions() == list(range(37))
    for rank in range(3):
        s = DistributedSampler(range(37), num_replicas=3, rank=rank, shuffle=True, seed=0)
        s.set_epoch(4)
        assert iwts.epoch_positions(4, rank, 3) == list(s)


class _StandInAug:
    """what ImageWeights reads of a DetAugmenter: n, cache.labels and the indices it sets"""

    def __init__(self, labels):
        self.n, self.indices = len(labels), range(len(labels))
        self.cache = type("Cache", (), {"labels": labels})()


def _labels(n, nc=7, seed=0):
    rs = np.random.RandomState(seed)
    out = []
    for _ in range(n):
        k = rs.randint(0, 4)
        lb = np.zeros((k, 5), np.float32)
        lb[:, 0] = rs.randint(0, nc, k)
        out.append(lb)
    return out


def _restated_draw(self, cw):
    """ImageWeights._draw on the host (the restatement), for a CPU-only rank 0"""
    state = random.getstate()
    iw = riw.image_weights(self.aug.cache.labels, len(cw), cw)
    buf = torch.zeros(self.n + 1, dtype=torch.int32)
    try:
        buf[:self.n] = torch.from_numpy(riw.choices(iw, random)[0])
    except ValueError:
        buf[self.n] = 2
    return buf, state


def _free_port():
    s = socket.socket(); s.bind(("127.0.0.1", 0)); p = s.getsockname()[1]; s.close(); return p


def _worker(rank, world, port, ret):
    import torch.distributed as dist

    from multiyolov5_b200.utils.datasets import ImageWeights
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    ImageWeights._draw = _restated_draw
    nc = 7
    aug = _StandInAug(_labels(50, nc))
    iwts = ImageWeights(aug)
    cwm = riw.class_weights(aug.cache.labels, nc) * nc
    random.seed(11 + rank)                                       # different streams: rank 1 must not use its own
    before = random.getstate()
    idx = iwts.draw(torch.from_numpy(cwm), np.linspace(0, 0.5, nc), rank=rank)
    ret[f"idx{rank}"], ret[f"aug{rank}"] = idx, list(aug.indices)
    ret[f"untouched{rank}"] = random.getstate() == before
    try:
        iwts.draw(cwm, np.ones(nc), rank=rank)                   # every class weight zero: rank 0 raises, rank 1 raises with it
    except ValueError as e:
        ret[f"err{rank}"] = str(e)
    ret[f"restored{rank}"] = random.getstate() == before if rank else None
    dist.destroy_process_group()


def test_draw_broadcast_gloo():
    import torch.multiprocessing as mp
    mgr = mp.Manager(); ret = mgr.dict(); port = _free_port()
    mp.spawn(_worker, args=(2, port, ret), nprocs=2, join=True)
    nc = 7
    labels = _labels(50, nc)
    random.seed(11)
    want, _, _ = riw.epoch_indices(labels, riw.class_weights(labels, nc) * nc, np.linspace(0, 0.5, nc), random)
    assert ret["idx0"] == want.tolist() == ret["idx1"] == ret["aug1"] == ret["aug0"]
    assert not ret["untouched0"] and ret["untouched1"]           # rank 1 consumed no draws
    assert ret["err0"] == ret["err1"] == "Total of weights must be greater than zero"
    assert ret["restored1"]
