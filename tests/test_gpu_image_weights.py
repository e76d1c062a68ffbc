"""GPU: --image-weights on the device (csrc/image_weights.cu, utils.general.labels_to_class_weights / labels_to_image_weights,
utils.datasets.ImageWeights) against the reference's own results (tests/golden/image_weights_cases.npz) and, at COCO scale, against the
numpy restatement (oracle/restate_image_weights.py).  Weights are compared as float64 bits, draws as indices and the next draws."""
import os
import random

import numpy as np
import pytest
import torch

from oracle import restate_image_weights as riw

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden")
NAMES = ["nc1_single", "nc5", "nc10_city", "nc80", "nc130", "all_maps_one", "n1"]


def _cases():
    return riw.load_cases(os.path.join(GOLD, "image_weights_cases.npz"))


def _bits(a):
    return np.ascontiguousarray(a, np.float64).view(np.int64)


class _Aug:
    """what ImageWeights reads of a DetAugmenter, for label-only cases"""

    def __init__(self, labels):
        self.n, self.indices = len(labels), range(len(labels))
        self.cache = type("Cache", (), {"labels": labels})()


@pytest.mark.parametrize("name", NAMES)
def test_device_equals_reference(name):
    from multiyolov5_b200.utils.datasets import ImageWeights
    from multiyolov5_b200.utils.general import labels_to_class_weights, labels_to_image_weights
    c = _cases()[0][name]
    nc, labels = c["nc"], c["labels"]
    cwt = labels_to_class_weights(labels, nc)
    assert cwt.dtype == torch.float64 and cwt.is_cuda
    assert np.array_equal(_bits(cwt.cpu().numpy()), _bits(c["class_weights"]))
    model_cw = cwt.to("cuda") * nc
    aug = _Aug(labels)
    iwts = ImageWeights(aug)
    random.seed(c["seed"])
    np.random.seed(c["seed"])
    for e in range(c["epochs"]):
        iw = labels_to_image_weights(labels, nc=nc, class_weights=c[f"e{e}_cw"])
        assert isinstance(iw, np.ndarray) and np.array_equal(_bits(iw), _bits(c[f"e{e}_iw"])), e
        if c["errors"][e] is None:
            idx = iwts.draw(model_cw, c[f"e{e}_maps"])
            assert idx == c[f"e{e}_indices"].tolist() and aug.indices == idx, e
        else:
            state = random.getstate()
            with pytest.raises(ValueError, match=c["errors"][e]):
                iwts.draw(model_cw, c[f"e{e}_maps"])
            assert random.getstate() == state
    assert random.random() == c["next_random"] and float(np.random.random()) == c["next_np"]


def test_coco_scale_equals_restatement():
    """118 287 images, 80 classes, about 7 labels per image, random maps with a few classes at 1.0; two epochs"""
    from multiyolov5_b200.utils.datasets import ImageWeights
    from multiyolov5_b200.utils.general import labels_to_class_weights
    rs = np.random.RandomState(0)
    n, nc = 118_287, 80
    k = rs.poisson(7.3, n) * (rs.random_sample(n) > 0.01)
    cls = rs.randint(0, nc, k.sum()).astype(np.float32)
    offs = np.concatenate([[0], np.cumsum(k)])
    labels = [np.stack([cls[offs[i]:offs[i + 1]]] + [np.full(k[i], 0.5, np.float32)] * 4, 1) for i in range(n)]
    cwt = labels_to_class_weights(labels, nc)
    want_cwt = riw.class_weights(labels, nc)
    assert np.array_equal(_bits(cwt.cpu().numpy()), _bits(want_cwt))
    iwts = ImageWeights(_Aug(labels))
    for epoch in range(2):
        maps = rs.uniform(0, 0.95, nc)
        maps[rs.choice(nc, 4, replace=False)] = 1.0
        random.seed(epoch)
        want, _, _ = riw.epoch_indices(labels, want_cwt * nc, maps, random)
        after = random.random()
        random.seed(epoch)
        assert iwts.draw(cwt * nc, maps) == want.tolist()
        assert random.random() == after


def test_weighted_draw_kernel_equals_accumulate_and_bisect():
    """myolo_weighted_draw alone: the cumulative sums are itertools.accumulate's, the total cum[-1] + 0.0, the draws bisect_right's"""
    from multiyolov5_b200 import _lib
    rs = np.random.default_rng(3)
    for n in (1, 2, 4095, 4096, 4097, 50_001):
        w = rs.lognormal(0, 2, n) * (rs.random(n) < 0.7)
        w[-1] = w[-1] or 1.0
        u = rs.random(n)
        rng = type("R", (), {"it": iter(u.tolist())})()
        rng.random = lambda: next(rng.it)
        want, want_cum, want_total = riw.choices(w, rng)
        wd, ud = torch.from_numpy(w).cuda(), torch.from_numpy(u).cuda()
        cum = torch.empty(n, dtype=torch.float64, device="cuda")
        total = torch.empty(1, dtype=torch.float64, device="cuda")
        idx = torch.empty(n, dtype=torch.int32, device="cuda")
        status = torch.zeros(1, dtype=torch.int32, device="cuda")
        _lib.check(_lib.lib().myolo_weighted_draw(_lib.ptr(wd), _lib.ptr(ud), n, _lib.ptr(cum), _lib.ptr(total), _lib.ptr(idx),
                                                  _lib.ptr(status), _lib.stream_ptr()))
        assert int(status.item()) == 0
        assert np.array_equal(_bits(cum.cpu().numpy()), _bits(want_cum)) and float(total.item()) == want_total
        assert np.array_equal(idx.cpu().numpy(), want), n


@pytest.mark.parametrize("w,msg", [(np.zeros(5), "greater than zero"), (np.array([1.0, -2.0, 0.5]), "greater than zero"),
                                   (np.array([1.0, np.inf, 2.0]), "must be finite"), (np.array([1.0, np.nan]), "must be finite")])
def test_total_errors_are_random_choices_errors(w, msg):
    from multiyolov5_b200 import _lib
    from multiyolov5_b200.utils.general import iw_status_error
    with pytest.raises(ValueError, match=msg):
        random.choices(range(len(w)), weights=w, k=len(w))
    n = len(w)
    wd, ud = torch.from_numpy(w).cuda(), torch.full((n,), 0.5, dtype=torch.float64, device="cuda")
    cum, total = torch.empty(n, dtype=torch.float64, device="cuda"), torch.empty(1, dtype=torch.float64, device="cuda")
    idx, status = torch.full((n,), -7, dtype=torch.int32, device="cuda"), torch.zeros(1, dtype=torch.int32, device="cuda")
    _lib.check(_lib.lib().myolo_weighted_draw(_lib.ptr(wd), _lib.ptr(ud), n, _lib.ptr(cum), _lib.ptr(total), _lib.ptr(idx),
                                              _lib.ptr(status), _lib.stream_ptr()))
    with pytest.raises(ValueError, match=msg):
        raise iw_status_error(int(status.item()))
    assert (idx.cpu() == -7).all()                                 # nothing drawn


def test_bad_classes_and_nc_bound_raise():
    from multiyolov5_b200 import _lib
    from multiyolov5_b200.utils.general import labels_to_class_weights, labels_to_image_weights
    bad = [np.array([[1, .5, .5, .1, .1], [7, .5, .5, .1, .1]], np.float32)]
    with pytest.raises(ValueError, match="outside"):
        labels_to_class_weights(bad, 5)
    with pytest.raises(ValueError, match="outside"):
        labels_to_image_weights(bad, 5, np.ones(5))
    neg = [np.array([[-1, .5, .5, .1, .1]], np.float32)]
    with pytest.raises(ValueError, match="outside"):
        labels_to_image_weights(neg, 5, np.ones(5))
    frac = [np.array([[-0.5, .5, .5, .1, .1], [4.9, .5, .5, .1, .1]], np.float32)]   # astype(int): 0 and 4
    assert labels_to_image_weights(frac, 5, np.arange(5.0))[0] == 4.0
    with pytest.raises(ValueError, match="nc"):
        labels_to_class_weights(bad, _lib.IW_NC_MAX + 1)


def _aug_sources():
    """the augmented items' sources: augment_cases.npz's (make_golden_augment.sources()), with the images that have no labels here"""
    import json
    a = np.load(os.path.join(GOLD, "augment_cases.npz"))
    g = np.load(os.path.join(GOLD, "image_weights_cases.npz"))
    meta = json.loads(bytes(g["meta_json"]).decode())
    n = meta["aug_sources"]
    labels = [np.zeros((0, 5), np.float32) if k in meta["aug_empty"] else a[f"labels_{k}"].copy() for k in range(n)]
    return [a[f"src_{k}"] for k in range(n)], labels


def _aug_setup(name):
    from multiyolov5_b200.utils.datasets import DetAugmenter, DeviceImageCache, ImageWeights
    from multiyolov5_b200.utils.general import labels_to_class_weights
    _, meta, g = _cases()
    m = meta[name]
    srcs, labels = _aug_sources()
    aug = DetAugmenter(DeviceImageCache(srcs, m["img_size"], labels), m["hyp"])
    iwts = ImageWeights(aug)
    return m, g, aug, iwts, labels_to_class_weights(labels, m["nc"]).cuda() * m["nc"]


@pytest.mark.parametrize("name", ["aug_mosaic", "aug_single"])
def test_batches_under_drawn_indices_equal_reference_items(name):
    """the reference's __getitem__ over its drawn indices (mosaic partners from the drawn list, mixup from range(n)) against
    ImageWeights(aug)(positions): images, labels and the next draws"""
    m, g, aug, iwts, model_cw = _aug_setup(name)
    random.seed(m["seed"])
    np.random.seed(m["seed"])
    idx = iwts.draw(model_cw, np.array(m["maps"]))
    assert idx == g[f"{name}_indices"].tolist()
    positions = iwts.epoch_positions()[:m["items"]]
    imgs, targets = iwts(positions)
    assert random.random() == m["next_random"] and float(np.random.random()) == m["next_np"]
    t = targets.cpu().numpy()
    for b, p in enumerate(positions):
        assert np.array_equal(imgs[b].cpu().numpy(), g[f"{name}_img_{p}"]), (name, p)
        assert np.array_equal(t[t[:, 0] == b][:, 1:], g[f"{name}_lab_{p}"]), (name, p)


def test_trainer_step_and_quad_on_image_weighted_batches():
    from multiyolov5_b200.models.yolo import Model
    from multiyolov5_b200.train import Trainer, scale_hyp
    from multiyolov5_b200.utils.datasets import DetAugmenter, DeviceImageCache, ImageWeights, collate_quad
    from multiyolov5_b200.utils.general import labels_to_class_weights
    from oracle import synth
    yml = "yolov5s_city_seg.yaml"
    cfg = synth.load_cfg(yml)
    model = Model(yml)
    model.load_state_dict(synth.synth_state_dict(synth.load_manifest("s_psp"), cfg, seed=1, gain=1.0))
    model.cuda().train()
    hyp = dict(lr0=0.01, momentum=0.937, weight_decay=5e-4, box=0.05, cls=0.5, cls_pw=1.0, obj=1.0, obj_pw=1.0, anchor_t=4.0, fl_gamma=0.0)
    B, s, nc = 2, 256, cfg["nc"]
    tr = Trainer(model, scale_hyp(hyp, nl=3, nc=nc, imgsz=s, total_batch_size=B), batch_size=B, init_scale=2.0 ** 10)
    srcs, labels = _aug_sources()
    for lb in labels:
        lb[:, 0] = lb[:, 0] % nc
    aug = DetAugmenter(DeviceImageCache(srcs, s, labels),
                       dict(hsv_h=0.015, hsv_s=0.7, hsv_v=0.4, degrees=0.0, translate=0.1, scale=0.5, shear=0.0, perspective=0.0,
                            flipud=0.0, fliplr=0.5, mosaic=1.0, mixup=0.0))
    iwts = ImageWeights(aug)
    random.seed(0)
    np.random.seed(0)
    iwts.draw(labels_to_class_weights(labels, nc).cuda() * nc, np.zeros(nc))
    segimgs = synth.synth_image(B, s, s, seed=2).cuda()
    mask = torch.from_numpy(np.random.RandomState(1).randint(-1, 19, (B, s, s)).astype(np.int64)).cuda()
    imgs, targets = iwts(iwts.epoch_positions()[:B])
    items, segloss = tr.step(imgs.float() / 255.0, targets, segimgs, mask)
    assert torch.isfinite(items).all() and torch.isfinite(segloss).all()
    q_imgs, q_t = collate_quad(*iwts(iwts.epoch_positions()[:4]))
    assert q_imgs.shape == (1, 3, 2 * s, 2 * s) and q_t.shape[1] == 6


def test_nccl_broadcast_at_one_rank():
    import socket

    import torch.distributed as dist

    from multiyolov5_b200.utils.datasets import ImageWeights
    from multiyolov5_b200.utils.general import labels_to_class_weights
    c = _cases()[0]["nc5"]
    sk = socket.socket(); sk.bind(("127.0.0.1", 0)); port = sk.getsockname()[1]; sk.close()
    dist.init_process_group("nccl", init_method=f"tcp://127.0.0.1:{port}", rank=0, world_size=1)
    try:
        iwts = ImageWeights(_Aug(c["labels"]))
        model_cw = labels_to_class_weights(c["labels"], c["nc"]) * c["nc"]
        random.seed(c["seed"])
        assert iwts.draw(model_cw, c["e0_maps"], rank=0) == c["e0_indices"].tolist()
    finally:
        dist.destroy_process_group()
