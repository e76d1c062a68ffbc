"""GPU: mode='val' segmentation batches built on the device (SegAugmenter.val, train.SegValBatches) against the reference's own items
(tests/golden/seg_val_cases.npz) and the numpy restatement (oracle/restate_seg_val.py) at full size, bit exact; seg_validation and fit
over SegValBatches."""
import json
import os
import random

import numpy as np
import pytest
import torch

from oracle import restate_seg_val as rv

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden")


def _golden():
    g = np.load(os.path.join(GOLD, "seg_val_cases.npz"))
    return g, json.loads(bytes(g["meta_json"]).decode())["cases"]


def _kinds(c):
    return ["trainid" if c["loader"] == "citysbdd" and f.endswith("jpg") else "cityscapes" for f in c["files"]]


@pytest.mark.parametrize("name", ["citys", "citys_c63", "citysbdd"])
def test_device_batch_matches_reference_fixtures(name):
    """every item of a case in ONE batch of mixed source sizes and mask maps; float32 bit for bit, float16 = that rounded, uint8 = the
    bytes; no `random` or torch draw consumed"""
    from multiyolov5_b200.utils.datasets import DeviceSegCache, SegAugmenter
    g, cases = _golden()
    c = cases[name]
    cache = DeviceSegCache([g[f"src_{si}"] for si, _ in c["sources"]], [g[f"mask_{mi}"] for _, mi in c["sources"]], mask_map=_kinds(c))
    aug = SegAugmenter(cache, base_size=1024, preset="citysbdd")
    idx = list(range(len(c["files"])))
    crop = c["crop_size"]
    random.seed(c["seed"])
    torch.manual_seed(c["seed"])
    out = {dt: aug.val(idx, crop, out_dtype=dt) for dt in (torch.float32, torch.float16, torch.uint8)}
    assert random.random() == c["next_random"] and float(torch.rand(1)) == c["next_torch"]
    imgs, labels = out[torch.float32]
    assert imgs.shape == (len(idx), 3, crop, crop) and labels.shape == (len(idx), crop, crop)
    assert imgs.dtype == torch.float32 and labels.dtype == torch.int64 and imgs.is_cuda and labels.is_cuda
    for j in idx:
        v = torch.from_numpy(g[f"{name}_img_{j}"]).cuda()
        ref = torch.from_numpy(g[f"{name}_img_{j}"].astype(np.float32) / np.float32(255)).cuda()      # ToTensor's true division
        lab = torch.from_numpy(g[f"{name}_lab_{j}"].astype(np.int64)).cuda()
        assert torch.equal(imgs[j], ref), (name, j, int((imgs[j] != ref).sum()))
        assert torch.equal(out[torch.float16][0][j], ref.half()) and torch.equal(out[torch.uint8][0][j], v), (name, j)
        for dt in out:
            assert torch.equal(out[dt][1][j], lab), (name, j, dt)


def _full_size_sources():
    """two 2048x1024 Cityscapes-style sources (label ids and 255) and two 1280x720 BDD-style ones (train ids and 255)"""
    r = np.random.RandomState(11)
    imgs, masks, kinds = [], [], []
    for k, (h, w) in enumerate([(1024, 2048), (720, 1280), (1024, 2048), (720, 1280)]):
        yy, xx = np.mgrid[0:h, 0:w]
        base = np.stack([xx * 255 // (w - 1), yy * 255 // (h - 1), (xx ^ yy) & 255], -1)
        img = np.clip(base + r.randint(-50, 51, (h, w, 3)), 0, 255).astype(np.uint8)
        img[100:300, 200:700] = r.randint(0, 256, 3)
        ids = np.concatenate([np.arange(34 if w == 2048 else 19), [255]])
        imgs.append(img)
        masks.append(r.choice(ids, (h, w)).astype(np.uint8))
        kinds.append("cityscapes" if w == 2048 else "trainid")
    return imgs, masks, kinds


def test_mixed_full_size_batch_matches_restatement():
    """train_citysbdd.py's validation batch: 2048x1024 .png-mapped and 1280x720 .jpg-mapped sources at crop 512, in one batch"""
    from multiyolov5_b200.utils.datasets import DeviceSegCache, SegAugmenter
    imgs0, masks0, kinds = _full_size_sources()
    aug = SegAugmenter(DeviceSegCache(imgs0, masks0, mask_map=kinds), base_size=1024, preset="citysbdd")
    order = [0, 1, 3, 2]
    imgs, labels = aug.val(order, 512)
    u8, _ = aug.val(order, 512, out_dtype=torch.uint8)
    assert imgs.shape == (4, 3, 512, 512) and labels.shape == (4, 512, 512)
    for b, i in enumerate(order):
        want, wl = rv.val_item(imgs0[i], masks0[i], rv.mask_lut(kinds[i]), 512)
        ref = torch.from_numpy(want).cuda()
        assert torch.equal(imgs[b], ref), (b, int((imgs[b] != ref).sum()))
        assert torch.equal(u8[b], torch.round(ref * 255).to(torch.uint8)), b
        assert torch.equal(labels[b], torch.from_numpy(wl).cuda()), b
    assert bool((labels[1] == -1).any()) and bool((labels[0] == -1).any())


def test_item_does_not_depend_on_batch_neighbours():
    from multiyolov5_b200.utils.datasets import DeviceSegCache, SegAugmenter
    r = np.random.RandomState(3)
    shapes = [(300, 500), (480, 256), (128, 700), (200, 200), (90, 160)]
    imgs = [r.randint(0, 256, (h, w, 3)).astype(np.uint8) for h, w in shapes]
    masks = [r.randint(0, 34, (h, w)).astype(np.uint8) for h, w in shapes]
    aug = SegAugmenter(DeviceSegCache(imgs, masks, mask_map=["cityscapes", "trainid"] * 2 + ["cityscapes"]), preset="citysbdd")
    order = [0, 1, 2, 3, 4, 1, 0]
    batch, lb = aug.val(order, 96)
    for b, i in enumerate(order):
        one, l1 = aug.val([i], 96)
        assert torch.equal(one[0], batch[b]) and torch.equal(l1[0], lb[b]), b


def _val_set():
    """five sources of four sizes (one mixed batch per pair), Cityscapes- and BDD-mapped"""
    r = np.random.RandomState(5)
    shapes = [(256, 512), (144, 256), (256, 512), (200, 150), (100, 300)]
    imgs, masks, kinds = [], [], []
    for k, (h, w) in enumerate(shapes):
        yy, xx = np.mgrid[0:h, 0:w]
        imgs.append(np.clip(np.stack([xx * 255 // (w - 1), yy * 255 // (h - 1), (xx * yy) & 255], -1) + r.randint(-30, 31, (h, w, 3)),
                            0, 255).astype(np.uint8))
        kinds.append("trainid" if k % 2 else "cityscapes")
        ids = np.concatenate([np.arange(19 if k % 2 else 34), [255]])
        masks.append(np.kron(r.choice(ids, (h // 8 + 1, w // 8 + 1)), np.ones((8, 8), np.int64))[:h, :w].astype(np.uint8))
    return imgs, masks, kinds


def _restated_batches(imgs, masks, kinds, batch_size, crop):
    out = []
    for k in range(0, len(imgs), batch_size):
        items = [rv.val_item(imgs[i], masks[i], rv.mask_lut(kinds[i]), crop) for i in range(k, min(k + batch_size, len(imgs)))]
        out.append((torch.from_numpy(np.stack([a for a, _ in items])).cuda(), torch.from_numpy(np.stack([b for _, b in items])).cuda()))
    return out


def test_seg_validation_over_val_batches():
    """seg_validation over SegValBatches(mode='val') returns the mIoU it returns over the restated batches, uploaded"""
    from multiyolov5_b200.test import seg_validation
    from multiyolov5_b200.train import SegValBatches
    from multiyolov5_b200.utils.datasets import DeviceSegCache, SegAugmenter
    from tests.test_gpu_train_loop import psp_model
    model, _ = psp_model()
    imgs, masks, kinds = _val_set()
    sv = SegValBatches(SegAugmenter(DeviceSegCache(imgs, masks, mask_map=kinds), preset="citysbdd"), 2, mode="val", crop_size=128)
    n_segcls = model.model[-2].c_out
    got = seg_validation(model, n_segcls, sv, "cuda")
    want = seg_validation(model, n_segcls, _restated_batches(imgs, masks, kinds, 2, 128), "cuda")
    again = seg_validation(model, n_segcls, sv, "cuda")
    assert isinstance(got, np.float64) and got == want == again, (got, want, again)
    assert len(sv) == 3


def test_fit_validates_every_epoch_over_val_batches(tmp_path, monkeypatch):
    """a two-epoch fit with segval_loader=SegValBatches(mode='val'): seg_validation runs at both epochs over every batch (the loader is
    iterated again), best_fitness is fitness2 of the results and that mIoU, and results.txt does not carry the mIoU"""
    import multiyolov5_b200.test as T
    from multiyolov5_b200.train import SegValBatches, fit
    from multiyolov5_b200.utils.datasets import DeviceSegCache, SegAugmenter
    from multiyolov5_b200.utils.metrics import fitness2
    from multiyolov5_b200.utils.torch_utils import ModelEMA
    from multiyolov5_b200.models.experimental import load_checkpoint
    from tests.test_gpu_train_loop import HYP, Cycle, make_batches, opt_, psp_model
    model, cfg = psp_model()
    det, seg = make_batches(cfg["nc"])
    imgs, masks, kinds = _val_set()
    sv = SegValBatches(SegAugmenter(DeviceSegCache(imgs, masks, mask_map=kinds), preset="citysbdd"), 2, mode="val", crop_size=128)
    built, mious, orig = [], [], T.seg_validation

    def recording(model, n_segcls, valloader, device, half_precision=True):
        assert valloader is sv
        n = [0]

        def counted():
            for batch in valloader:
                n[0] += 1
                yield batch
        m = orig(model, n_segcls, counted(), device, half_precision)
        built.append(n[0])
        mious.append(m)
        return m
    monkeypatch.setattr(T, "seg_validation", recording)
    ema = ModelEMA(model)
    results = fit(model, HYP, opt_(epochs=2), Cycle(det, 3), Cycle(seg, 3), segval_loader=sv, save_dir=tmp_path, ema=ema,
                  init_scale=2.0 ** 10)
    assert built == [3, 3] and len(mious) == 2 and all(m > 0 for m in mious), (built, mious)
    assert orig(ema.ema, model.model[-2].c_out, sv, "cuda") == mious[-1]             # the EMA has not changed since the last pass
    fis = [fitness2(np.array(results).reshape(1, -1), m) for m in mious]
    ck = load_checkpoint(str(tmp_path / "weights" / "last.pt"))
    best = max([0.0] + [float(np.max(f)) for f in fis])
    assert float(np.max(ck["best_fitness"])) == best
    lines = (tmp_path / "results.txt").read_text().splitlines()
    assert len(lines) == 2 and all(len(line.split()) == 16 for line in lines)
    assert all([float(v) for v in line.split()[-7:]] == [0.0] * 7 for line in lines)
