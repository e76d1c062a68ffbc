"""GPU: detection training batches built on the device (DeviceImageCache + DetAugmenter) against the reference's own items
(tests/golden/augment_cases.npz) and against the numpy restatement (oracle/restate_augment.py) at full size.  Integer work: bit exact."""
import json
import os
import random

import numpy as np
import pytest
import torch

from oracle import restate_augment as ra

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden")


def _golden():
    g = np.load(os.path.join(GOLD, "augment_cases.npz"))
    return g, json.loads(bytes(g["meta_json"]).decode())


def _labels_of(targets, b):
    t = targets.cpu().numpy()
    return t[t[:, 0] == b][:, 1:]


@pytest.mark.parametrize("name", ["scratch", "stress", "mixup", "flipud", "single"])
def test_device_batch_matches_reference_fixtures(name):
    from multiyolov5_b200.utils.datasets import DetAugmenter, DeviceImageCache
    g, meta = _golden()
    c = meta["cases"][name]
    n = len(meta["shapes"])
    cache = DeviceImageCache([g[f"src_{k}"] for k in range(n)], c["img_size"], [g[f"labels_{k}"] for k in range(n)])
    for i in range(n):                           # stored for one size; the items pin the other
        key = f"cache{c['img_size']}_{i}"
        assert key not in g.files or np.array_equal(cache.image(i).cpu().numpy(), g[key]), (name, i)
    aug = DetAugmenter(cache, c["hyp"])
    random.seed(c["seed"])
    np.random.seed(c["seed"])
    imgs, targets = aug(c["items"])
    assert random.random() == c["next_random"] and float(np.random.random()) == c["next_np"]
    assert imgs.dtype == torch.uint8 and targets.dtype == torch.float32 and targets.is_cuda
    for b, i in enumerate(c["items"]):
        got = imgs[b].cpu().numpy()
        ref = g[f"{name}_img_{i}"]
        assert np.array_equal(got, ref), (name, i, int((got != ref).sum()))
        assert np.array_equal(_labels_of(targets, b), g[f"{name}_lab_{i}"]), (name, i)


def _sources(rs, n, big):
    shapes = [(512, 1024), (1024, 512), (300, 200), (120, 90), (700, 900), (256, 256)] if big else [(200, 300), (64, 48), (480, 640)]
    imgs, labels = [], []
    for k in range(n):
        h, w = shapes[k % len(shapes)]
        yy, xx = np.mgrid[0:h, 0:w]
        base = np.stack([xx * 255 // w, yy * 255 // h, (xx ^ yy) & 255], -1)
        imgs.append(np.clip(base + rs.randint(-40, 41, (h, w, 3)), 0, 255).astype(np.uint8))
        m = rs.randint(0, 6)
        lb = np.zeros((m, 5), np.float32)
        lb[:, 0] = rs.randint(0, 10, m)
        lb[:, 3:5] = rs.uniform(0.02, 0.5, (m, 2))
        lb[:, 1:3] = rs.uniform(0.1, 0.9, (m, 2))
        labels.append(lb)
    return imgs, labels


EXTREME_HYPS = [
    dict(degrees=10.0, translate=0.1, scale=0.5, shear=5.0, mixup=1.0),
    dict(degrees=10.0, translate=0.25, scale=0.5, shear=0.0, mixup=0.0, flipud=0.5),
    dict(degrees=0.0, translate=0.0, scale=0.0, shear=0.0, mixup=0.5),
    dict(degrees=10.0, translate=0.1, scale=0.5, shear=2.0, mosaic=0.0),
]


@pytest.mark.parametrize("s,n_items", [(640, 16), (1024, 16)])
def test_device_batch_matches_restatement_full_size(s, n_items):
    """full-size items under extreme draws (rotation to 10 deg, scale 0.5-1.5, translate at its limits, tiles smaller than a canvas
    quadrant, mixup, the non-mosaic branch): the device batch equals the restatement; the float outputs equal uint8 / 255 on the GPU"""
    from multiyolov5_b200.utils.datasets import DetAugmenter, DeviceImageCache
    rs = np.random.RandomState(s)
    imgs0, labels0 = _sources(rs, 6, big=True)
    cache = DeviceImageCache(imgs0, s, labels0)
    per_hyp = n_items // len(EXTREME_HYPS)
    for h, over in enumerate(EXTREME_HYPS):
        hyp = dict(ra_scratch(), **over)
        src = ra.Source(imgs0, labels0, s, hyp)
        for i in range(cache.n):
            assert np.array_equal(cache.image(i).cpu().numpy(), src.cache[i])
        idx = [int(v) for v in rs.randint(0, cache.n, per_hyp)]
        seed = 1000 * s + h
        random.seed(seed)
        np.random.seed(seed)
        want = [ra.getitem(src, i) for i in idx]
        aug = DetAugmenter(cache, hyp)
        for dtype in (torch.uint8, torch.float16, torch.float32):
            random.seed(seed)
            np.random.seed(seed)
            imgs, targets = aug(idx, out_dtype=dtype)
            for b, (wi, wl) in enumerate(want):
                ref = torch.from_numpy(wi).cuda()
                if dtype == torch.uint8:
                    assert torch.equal(imgs[b], ref), (s, h, b, int((imgs[b] != ref).sum()))
                else:
                    assert torch.equal(imgs[b], ref.to(dtype) / 255.0 if dtype == torch.float16 else ref.float() / 255.0), (s, h, b, dtype)
                assert np.array_equal(_labels_of(targets, b), wl), (s, h, b)


def ra_scratch():
    return dict(hsv_h=0.015, hsv_s=0.7, hsv_v=0.4, degrees=0.0, translate=0.1, scale=0.5, shear=0.0, perspective=0.0, flipud=0.0,
                fliplr=0.5, mosaic=1.0, mixup=0.0)


def test_item_does_not_depend_on_batch_neighbours():
    from multiyolov5_b200.utils.datasets import DetAugmenter, DeviceImageCache
    rs = np.random.RandomState(5)
    imgs0, labels0 = _sources(rs, 3, big=False)
    cache = DeviceImageCache(imgs0, 256, labels0)
    aug = DetAugmenter(cache, dict(ra_scratch(), mixup=0.5, degrees=5.0))
    random.seed(3)
    np.random.seed(3)
    batch, tb = aug([0, 1, 2, 1])
    random.seed(3)
    np.random.seed(3)
    for b, i in enumerate([0, 1, 2, 1]):
        one, t1 = aug([i])
        assert torch.equal(one[0], batch[b])
        assert np.array_equal(_labels_of(t1, 0), _labels_of(tb, b))


def test_unsupported_settings_raise_on_device():
    from multiyolov5_b200.utils.datasets import DetAugmenter, DeviceImageCache
    img = np.zeros((64, 64, 3), np.uint8)
    with pytest.raises(NotImplementedError):
        DeviceImageCache([img], 64, [np.zeros((0, 5), np.float32)], segments=[[np.zeros((4, 2), np.float32)]])
    cache = DeviceImageCache([img], 64)
    with pytest.raises(NotImplementedError):
        DetAugmenter(cache, dict(ra_scratch(), perspective=0.0005))


def test_trainer_step_on_device_batches():
    """one Trainer.step (det pass + seg pass + optimiser) fed by DetAugmenter gives finite losses"""
    from multiyolov5_b200.models.yolo import Model
    from multiyolov5_b200.train import Trainer, scale_hyp
    from multiyolov5_b200.utils.datasets import DetAugmenter, DeviceImageCache
    from oracle import synth
    yml = "yolov5s_city_seg.yaml"
    cfg = synth.load_cfg(yml)
    model = Model(yml)
    model.load_state_dict(synth.synth_state_dict(synth.load_manifest("s_psp"), cfg, seed=1, gain=1.0))
    model.cuda().train()
    hyp = dict(lr0=0.01, momentum=0.937, weight_decay=5e-4, box=0.05, cls=0.5, cls_pw=1.0, obj=1.0, obj_pw=1.0, anchor_t=4.0, fl_gamma=0.0)
    B, s = 2, 256
    tr = Trainer(model, scale_hyp(hyp, nl=3, nc=cfg["nc"], imgsz=s, total_batch_size=B), batch_size=B, init_scale=2.0 ** 10)
    rs = np.random.RandomState(1)
    imgs0, labels0 = _sources(rs, 3, big=False)
    for lb in labels0:
        lb[:, 0] = lb[:, 0] % cfg["nc"]
    aug = DetAugmenter(DeviceImageCache(imgs0, s, labels0), ra_scratch())
    random.seed(0)
    np.random.seed(0)
    segimgs = synth.synth_image(B, s, s, seed=2).cuda()
    mask = torch.from_numpy(rs.randint(-1, 19, (B, s, s)).astype(np.int64)).cuda()
    for _ in range(2):
        imgs, targets = aug([0, 1], out_dtype=torch.float32)
        items, segloss = tr.step(imgs, targets, segimgs, mask)
        assert torch.isfinite(items).all() and torch.isfinite(segloss).all()
