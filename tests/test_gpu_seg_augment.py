"""GPU: segmentation training batches built on the device (DeviceSegCache + SegAugmenter) against the reference's own items
(tests/golden/seg_augment_cases.npz) and against the numpy restatement (oracle/restate_seg.py) at full size.  Bit exact, no tolerance."""
import itertools
import json
import os
import random

import numpy as np
import pytest
import torch

from oracle import restate_seg as rs

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden")


def _golden():
    g = np.load(os.path.join(GOLD, "seg_augment_cases.npz"))
    return g, json.loads(bytes(g["meta_json"]).decode())["cases"]


def _fixture_cache(g, c):
    from multiyolov5_b200.utils.datasets import DeviceSegCache
    kinds = ["cityscapes" if c["loader"] == "citys" or (c["loader"] == "citysbdd" and f.endswith("png")) else "trainid" for f in c["files"]]
    return DeviceSegCache([g[f"src_{si}"] for si, _ in c["sources"]], [g[f"mask_{mi}"] for _, mi in c["sources"]], mask_map=kinds)


@pytest.mark.parametrize("name", ["citys", "citysbdd", "custom"])
def test_device_batch_matches_reference_fixtures(name):
    from multiyolov5_b200.utils.datasets import SegAugmenter
    g, cases = _golden()
    c = cases[name]
    aug = SegAugmenter(_fixture_cache(g, c), base_size=c["base_size"], crop_size=tuple(c["crop_size"]), preset=c["loader"])
    random.seed(c["seed"])
    torch.manual_seed(c["seed"])
    imgs, labels = aug(c["items"])
    assert random.random() == c["next_random"] and float(torch.rand(1)) == c["next_torch"]
    assert imgs.dtype == torch.float32 and labels.dtype == torch.int64 and imgs.is_cuda and labels.is_cuda
    for j in range(len(c["items"])):
        ref = torch.from_numpy(g[f"{name}_img_{j}"].astype(np.float32) / np.float32(255)).cuda()
        assert torch.equal(imgs[j], ref), (name, j, int((imgs[j] != ref).sum()))
        assert torch.equal(labels[j], torch.from_numpy(g[f"{name}_lab_{j}"].astype(np.int64)).cuda()), (name, j)


def test_testval_matches_reference_fixtures():
    from multiyolov5_b200.utils.datasets import SegAugmenter
    g, cases = _golden()
    c = cases["testval"]
    aug = SegAugmenter(_fixture_cache(g, c), base_size=c["base_size"], crop_size=tuple(c["crop_size"]), preset="citys")
    for j, i in enumerate(c["items"]):
        imgs, labels = aug.testval([i])
        ref = torch.from_numpy(g[f"testval_img_{j}"].astype(np.float32) / np.float32(255)).cuda()
        assert torch.equal(imgs[0], ref) and torch.equal(labels[0], torch.from_numpy(g[f"testval_lab_{j}"].astype(np.int64)).cuda()), j


def _big_sources(n):
    rs_ = np.random.RandomState(7)
    imgs, masks = [], []
    for k in range(n):
        yy, xx = np.mgrid[0:1024, 0:2048]
        base = np.stack([xx * 255 // 2047, yy * 255 // 1023, (xx ^ yy) & 255], -1)
        imgs.append(np.clip(base + rs_.randint(-60, 61, (1024, 2048, 3)), 0, 255).astype(np.uint8))
        imgs[-1][100:300, 200:900] = rs_.randint(0, 256, 3)       # a flat block: grey / saturated edge cases
        imgs[-1][400:500, 0:600] = 255
        masks.append(rs_.choice(np.concatenate([np.arange(34), [255]]), (1024, 2048)).astype(np.uint8))
    return imgs, masks


# full-size geometries: (flip, ow, oh, x1, y1) - long side 672 (padded both ways, ~7 taps), 3072 (2 taps, crop at the far corner),
# identity (one-tap tables), and the mirror with up- and down-scaling
GEOMS = [(True, 672, 336, 0, 0), (False, 3072, 1536, 2048, 1024), (False, 2048, 1024, 517, 311), (True, 3072, 1536, 1, 777),
         (True, 1536, 768, 512, 256), (False, 1024, 512, 0, 0)]


def _forced_params():
    """24 items: every jitter order once, brightness / contrast / saturation on both sides of 1, hue wrapping both ways"""
    out = []
    for k, order in enumerate(itertools.permutations(range(4))):
        flip, ow, oh, x1, y1 = GEOMS[k % len(GEOMS)]
        f = [float(np.float32(v)) for v in ([0.55, 1.45][k % 2], [0.55, 1.45][(k // 2) % 2], [0.6, 1.45][(k // 4) % 2],
                                             [-0.5, 0.5, -0.15, 0.15, 0.0039, -0.0039][k % 6])]
        if k == 23:
            f[1] = None                                              # a preset without contrast: no mean to accumulate
        out.append(dict(flip=flip, ow=ow, oh=oh, x1=x1, y1=y1, order=list(order), factors=f))
    return out


def test_device_batch_matches_restatement_full_size():
    from multiyolov5_b200.utils.datasets import DeviceSegCache, SegAugmenter
    imgs0, masks0 = _big_sources(2)
    cache = DeviceSegCache(imgs0, masks0, mask_map="cityscapes")
    aug = SegAugmenter(cache, base_size=1024, crop_size=(1024, 512), preset="citys")
    params = _forced_params()
    idx = [k % 2 for k in range(len(params))]
    lut = rs.mask_lut("cityscapes")
    crops = {}
    outs = {dt: aug.build(idx, params, out_dtype=dt) for dt in (torch.uint8, torch.float16, torch.float32)}
    for b, (i, p) in enumerate(zip(idx, params)):
        key = (i, p["flip"], p["ow"], p["oh"], p["x1"], p["y1"])
        if key not in crops:
            crops[key] = rs.crop_of(imgs0[i], masks0[i], p, (1024, 512))
        im, m = crops[key]
        want = rs.color_jitter(im, p["order"], p["factors"])
        ref_u8 = torch.from_numpy(np.ascontiguousarray(want.transpose(2, 0, 1))).cuda()
        ref_f32 = torch.from_numpy(rs.to_tensor(want)).cuda()
        assert torch.equal(outs[torch.uint8][0][b], ref_u8), (b, p, int((outs[torch.uint8][0][b] != ref_u8).sum()))
        assert torch.equal(outs[torch.float32][0][b], ref_f32), b
        assert torch.equal(outs[torch.float16][0][b], ref_f32.half()), b
        for dt in outs:
            assert torch.equal(outs[dt][1][b], torch.from_numpy(lut[m]).cuda()), (b, dt)


def test_item_does_not_depend_on_batch_neighbours():
    from multiyolov5_b200.utils.datasets import DeviceSegCache, SegAugmenter
    r = np.random.RandomState(3)
    shapes = [(300, 500), (480, 256), (128, 700)]
    imgs = [r.randint(0, 256, (h, w, 3)).astype(np.uint8) for h, w in shapes]
    masks = [r.randint(0, 34, (h, w)).astype(np.uint8) for h, w in shapes]
    aug = SegAugmenter(DeviceSegCache(imgs, masks), base_size=256, crop_size=(256, 128), preset="citys")
    order = [0, 1, 2, 1, 0]
    random.seed(5)
    torch.manual_seed(5)
    batch, lb = aug(order)
    random.seed(5)
    torch.manual_seed(5)
    for b, i in enumerate(order):
        one, l1 = aug([i])
        assert torch.equal(one[0], batch[b]) and torch.equal(l1[0], lb[b]), b


def test_testval_full_size():
    from multiyolov5_b200.utils.datasets import DeviceSegCache, SegAugmenter
    imgs0, masks0 = _big_sources(1)
    aug = SegAugmenter(DeviceSegCache(imgs0 * 2, masks0 * 2), base_size=1024, preset="citys")
    imgs, labels = aug.testval([0, 1])
    want, wl = rs.testval_item(imgs0[0], masks0[0], rs.mask_lut("cityscapes"), 1024)
    assert imgs.shape == (2, 3, 512, 1024) and labels.shape == (2, 1024, 2048)
    for b in range(2):
        assert torch.equal(imgs[b], torch.from_numpy(want).cuda()) and torch.equal(labels[b], torch.from_numpy(wl).cuda())


def test_trainer_step_on_device_batches():
    """one Trainer.step fed by DetAugmenter (det batch) and SegAugmenter (seg batch) gives finite losses"""
    from multiyolov5_b200.models.yolo import Model
    from multiyolov5_b200.train import Trainer, scale_hyp
    from multiyolov5_b200.utils.datasets import DetAugmenter, DeviceImageCache, DeviceSegCache, SegAugmenter
    from oracle import synth
    yml = "yolov5s_city_seg.yaml"
    cfg = synth.load_cfg(yml)
    model = Model(yml)
    model.load_state_dict(synth.synth_state_dict(synth.load_manifest("s_psp"), cfg, seed=1, gain=1.0))
    model.cuda().train()
    hyp = dict(lr0=0.01, momentum=0.937, weight_decay=5e-4, box=0.05, cls=0.5, cls_pw=1.0, obj=1.0, obj_pw=1.0, anchor_t=4.0, fl_gamma=0.0)
    B, s = 2, 256
    tr = Trainer(model, scale_hyp(hyp, nl=3, nc=cfg["nc"], imgsz=s, total_batch_size=B), batch_size=B, init_scale=2.0 ** 10)
    r = np.random.RandomState(1)
    det_imgs = [r.randint(0, 256, (200, 300, 3)).astype(np.uint8) for _ in range(2)]
    det_labels = [np.array([[k % cfg["nc"], 0.5, 0.5, 0.3, 0.2]], np.float32) for k in range(2)]
    det = DetAugmenter(DeviceImageCache(det_imgs, s, det_labels), dict(hsv_h=0.015, hsv_s=0.7, hsv_v=0.4, degrees=0.0, translate=0.1,
                                                                       scale=0.5, shear=0.0, perspective=0.0, flipud=0.0, fliplr=0.5,
                                                                       mosaic=1.0, mixup=0.0))
    seg_imgs = [r.randint(0, 256, (256, 512, 3)).astype(np.uint8) for _ in range(2)]
    seg_masks = [r.randint(0, 34, (256, 512)).astype(np.uint8) for _ in range(2)]
    seg = SegAugmenter(DeviceSegCache(seg_imgs, seg_masks), base_size=s, crop_size=(s, s), preset="citys")
    random.seed(0)
    np.random.seed(0)
    torch.manual_seed(0)
    for _ in range(2):
        imgs, targets = det([0, 1], out_dtype=torch.float32)
        segimgs, segtargets = seg([0, 1])
        items, segloss = tr.step(imgs, targets, segimgs, segtargets)
        assert torch.isfinite(items).all() and torch.isfinite(segloss).all()
