"""GPU: `--rect` training batches built on the device (DeviceImageCache + DetRectLoader) against the reference's own batches
(tests/golden/rect_cases.npz) and against the numpy restatement (oracle/restate_rect.py getitem_rect) at full size, bit exact; and
Trainer steps over several rect shapes on one reserved workspace against the same steps on private plans (the bar of
test_gpu_multiscale.py)."""
import json
import os
import random

import numpy as np
import pytest
import torch

from oracle import restate_augment as ra
from oracle import restate_rect as rr
from oracle import synth
from tests.test_gpu_multiscale import HYP, _assert_within, _model

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden")
CASES = ["scratch", "stress", "flipud", "identity"]


def _golden():
    g = np.load(os.path.join(GOLD, "rect_cases.npz"))
    return g, json.loads(bytes(g["meta_json"]).decode())


def _scratch():
    return dict(hsv_h=0.015, hsv_s=0.7, hsv_v=0.4, degrees=0.0, translate=0.1, scale=0.5, shear=0.0, perspective=0.0, flipud=0.0,
                fliplr=0.5, mosaic=1.0, mixup=0.0)


@pytest.mark.parametrize("name", CASES)
def test_device_batches_match_reference_fixtures(name):
    from multiyolov5_b200.utils.datasets import DetRectLoader, DeviceImageCache
    g, meta = _golden()
    c = meta["cases"][name]
    n = len(meta["shapes"])
    cache = DeviceImageCache([g[f"src_{k}"] for k in range(n)], c["img_size"], [g[f"labels_{k}"] for k in range(n)])
    loader = DetRectLoader(cache, c["hyp"], c["batch_size"])
    assert np.array_equal(loader.order, g[f"{name}_order"]) and np.array_equal(loader.batch_shapes, g[f"{name}_batch_shapes"])
    random.seed(c["seed"])
    np.random.seed(c["seed"])
    ref8 = []
    for b, (imgs, targets) in enumerate(loader):
        ref = g[f"{name}_img_{b}"]
        assert imgs.dtype == torch.uint8 and targets.dtype == torch.float32 and targets.is_cuda
        got = imgs.cpu().numpy()
        assert got.shape == ref.shape and np.array_equal(got, ref), (name, b, int((got != ref).sum()) if got.shape == ref.shape else got.shape)
        assert np.array_equal(targets.cpu().numpy(), g[f"{name}_targets_{b}"]), (name, b)
        ref8.append(imgs)
    assert b + 1 == c["n_batches"]
    assert random.random() == c["next_random"] and float(np.random.random()) == c["next_np"]
    for dtype in (torch.float16, torch.float32):
        random.seed(c["seed"])
        np.random.seed(c["seed"])
        for b, (imgs, _) in enumerate(loader.batches(out_dtype=dtype)):
            want = ref8[b].to(dtype) / 255.0 if dtype == torch.float16 else ref8[b].float() / 255.0
            assert imgs.dtype == dtype and torch.equal(imgs, want), (name, b, dtype)


def _frames(rs, shapes):
    imgs, labels = [], []
    for h, w in shapes:
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
    dict(degrees=10.0, translate=0.25, scale=0.5, shear=5.0, flipud=0.5),
    dict(degrees=0.0, translate=0.0, scale=0.0, shear=0.0),
]
FULL = {  # name -> (frame shapes, img_size, batch size, expected batch shapes)
    "cityscapes": ([(1024, 2048)] * 5, 1024, 4, [[512, 1024]] * 2),
    "bdd": ([(720, 1280)] * 3, 1024, 4, [[576, 1024]]),
    "mixed": ([(480, 640), (640, 480), (600, 600), (300, 700), (700, 350)], 640, 2, [[480, 640], [640, 640], [640, 320]]),
}


@pytest.mark.parametrize("name", list(FULL))
def test_device_batches_match_restatement_full_size(name):
    """full-size rect batches under extreme draws (rotation to 10 deg, shear 5, scale 0.5-1.5, translate at its limits, flipud, and the
    identity hyp where the reference skips the warp): the device batch equals the restatement on this host"""
    from multiyolov5_b200.utils.datasets import DetRectLoader, DeviceImageCache
    shapes, s, bs, want_shapes = FULL[name]
    rs = np.random.RandomState(len(name))
    imgs0, labels0 = _frames(rs, shapes)
    cache = DeviceImageCache(imgs0, s, labels0)
    for h, over in enumerate(EXTREME_HYPS):
        hyp = dict(_scratch(), **over)
        loader = DetRectLoader(cache, hyp, bs)
        assert loader.batch_shapes.tolist() == want_shapes
        src = ra.Source(imgs0, labels0, s, hyp)
        seed = 100 * len(name) + h
        random.seed(seed)
        np.random.seed(seed)
        want = [[rr.getitem_rect(src, int(loader.order[p]), loader.batch_shapes[loader.batch[p]]) for p in range(k, min(k + bs, cache.n))]
                for k in range(0, cache.n, bs)]
        random.seed(seed)
        np.random.seed(seed)
        for b, (imgs, targets) in enumerate(loader):
            t = targets.cpu().numpy()
            for k, (wi, wl) in enumerate(want[b]):
                ref = torch.from_numpy(wi).cuda()
                assert torch.equal(imgs[k], ref), (name, h, b, k, int((imgs[k] != ref).sum()))
                assert np.array_equal(t[t[:, 0] == k][:, 1:], wl), (name, h, b, k)


# ---- train steps over rect shapes on one reserved workspace ------------------------------------------------------------------------
B = 4
SEQ = [(B, 512, 1024), (B, 1024, 576), (B, 576, 1024), (2, 512, 1024), (B, 640, 1024)]    # three+ shapes, a partial batch, a return


def _batch(n, H, W, nc, seed):
    rs = np.random.RandomState(seed)
    imgs = synth.synth_image(n, H, W, seed=seed).cuda().half()
    t = np.zeros((6 * n, 6), np.float32)
    t[:, 0] = np.arange(6 * n) % n; t[:, 1] = rs.randint(0, nc, 6 * n)
    t[:, 2:4] = rs.uniform(0.1, 0.9, (6 * n, 2)); t[:, 4:6] = rs.uniform(0.05, 0.3, (6 * n, 2))
    return imgs, torch.from_numpy(t).cuda()


def _run(shared):
    from multiyolov5_b200.train import Trainer, scale_hyp
    model, cfg = _model()
    shapes = sorted({(H, W) for _, H, W in SEQ})
    tr = Trainer(model, scale_hyp(HYP, nl=3, nc=cfg["nc"], imgsz=1024, total_batch_size=B), batch_size=B, init_scale=2.0 ** 10,
                 det_shapes=shapes if shared else None)
    eng = model.engine()
    rs = np.random.RandomState(7)
    segimgs = synth.synth_image(B, 256, 512, seed=7).cuda()
    segtargets = torch.from_numpy(rs.randint(-1, 19, (B, 256, 512)).astype(np.int64)).cuda()
    out = []
    for k, (n, H, W) in enumerate(SEQ):
        if shared and k:                                    # another shape's data in every byte: fp16 NaN patterns
            eng._arenas[0].ws.fill_(0xFF)
            eng._arenas[0].gws.fill_(0xFF)
        imgs, targets = _batch(n, H, W, cfg["nc"], seed=k)
        items, segloss = tr.step(imgs, targets, segimgs, segtargets)
        out.append([float(v) for v in items] + [float(segloss)])
    torch.cuda.synchronize()
    det = {key: p for key, p in eng.plans.items() if key[0] == "train" and len(key) == 4}
    assert set(det) == {("train", n, H, W) for n, H, W in SEQ}
    if shared:
        assert all(p.arena is eng._arenas[0] for p in det.values())
        assert tr.det_train_shapes() == shapes
    else:
        assert all(p.arena is None for p in det.values())
    state = {k: v.detach().float().cpu().clone() for k, v in model.state_dict().items()}
    del tr, model, eng, det
    torch.cuda.empty_cache()
    return np.array(out), state


def test_rect_steps_on_one_reserved_workspace_equal_private_plans():
    privates = [_run(False) for _ in range(4)]
    _assert_within(_run(True), privates, "rect shapes 512x1024 -> 1024x576 -> 576x1024 -> 2 x 512x1024 -> 640x1024, poisoned between")


def test_rect_with_multiscale_reserves_and_runs_the_cityscapes_shape():
    from multiyolov5_b200.train import MultiScale, Trainer, scale_hyp
    from multiyolov5_b200.utils.datasets import DetRectLoader, DeviceImageCache
    model, cfg = _model()
    rs = np.random.RandomState(3)
    imgs0, labels0 = _frames(rs, [(1024, 2048)] * 4)
    for lb in labels0:
        lb[:, 0] = lb[:, 0] % cfg["nc"]
    loader = DetRectLoader(DeviceImageCache(imgs0, 1024, labels0), _scratch(), B)
    assert loader.batch_shapes.tolist() == [[512, 1024]]
    ms = MultiScale(1024)
    tr = Trainer(model, scale_hyp(HYP, nl=3, nc=cfg["nc"], imgsz=1024, total_batch_size=B), batch_size=B, init_scale=2.0 ** 10,
                 multi_scale=ms, det_shapes=loader.batch_shapes)
    eng = model.engine()
    arena = eng._arenas[0]
    assert tr.det_train_shapes() == ms.shapes((512, 1024)) and (512, 1024) in tr.det_train_shapes()
    segimgs = synth.synth_image(B, 256, 512, seed=1).cuda()
    segtargets = torch.from_numpy(rs.randint(-1, 19, (B, 256, 512)).astype(np.int64)).cuda()
    random.seed(0); np.random.seed(0)
    seen = set()
    for sz in (1024, 512, 1536, 800):                          # the batch's own size, the smallest, the largest, one between
        imgs, targets = next(iter(loader))
        imgs = ms(imgs, torch.float16, rng=_Fixed(sz))
        seen.add(tuple(imgs.shape[2:]))
        items, segloss = tr.step(imgs, targets, segimgs, segtargets)
        assert torch.isfinite(items).all() and torch.isfinite(segloss).all()
    torch.cuda.synchronize()
    assert seen == {(512, 1024), (256, 512), (768, 1536), (416, 800)}, seen
    det = [p for key, p in eng.plans.items() if key[0] == "train" and len(key) == 4]
    assert len(det) == 4 and all(p.arena is arena for p in det) and eng._arenas[0] is arena
    print(f"\nrect 512x1024 + multi-scale: {len(tr.det_train_shapes())} reserved shapes, shared pair {arena.capacity / 1e9:.2f} GB")


class _Fixed:
    def __init__(self, v):
        self.v = v

    def randrange(self, a, b):
        assert a <= self.v < b
        return self.v
