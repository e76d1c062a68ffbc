#!/usr/bin/env python
"""Benchmark of the device-side mode='val' segmentation batches (SegAugmenter.val through train.SegValBatches, csrc/augment_seg.cu)
against the reference's PIL item on the host.

    python tools/bench_seg_val.py [--steps K] [--warmup W] [--batch B]

Workload: train_citysbdd.py's validation, B = 4 at crop 512 over 8 sources in the device cache, 2048x1024 (Cityscapes, label-id masks)
and 1280x720 (BDD100k, train-id masks) alternating, so every batch mixes both sizes.  Prints ONE JSON line:
  * launch: myolo_augment_seg alone over one uploaded batch (CUDA events over K batches);
  * batches: SegValBatches iterated end to end (geometry, Pillow tables, one pinned upload, the launch), to a device synchronise;
  * validation: test.seg_validation of s/PSP (synthetic weights, fp16) over SegValBatches and over the same batches built beforehand,
    so that the difference is what building the batches adds to a validation pass;
  * host_reference_1core: the reference's item (`_val_sync_transform`'s PIL resizes and centre crop, ToTensor, the mask map) through
    PIL + torchvision on one core, recorded as unavailable when those libraries are not installed;
and the card's name, power limit and clocks read next to the measurement.  Writes nothing to disk.
"""
import argparse
import ctypes as C
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from bench_seg_augment import gpu_state  # noqa: E402

CROP = 512


def sources(n, seed=0):
    rs = np.random.RandomState(seed)
    imgs, masks, kinds = [], [], []
    for k in range(n):
        h, w = (1024, 2048) if k % 2 == 0 else (720, 1280)
        yy, xx = np.mgrid[0:h, 0:w]
        base = np.stack([xx * 255 // (w - 1), yy * 255 // (h - 1), (xx ^ yy) & 255], -1)
        imgs.append(np.clip(base + rs.randint(-40, 41, (h, w, 3)), 0, 255).astype(np.uint8))
        ids = np.concatenate([np.arange(34 if k % 2 == 0 else 19), [255]])
        masks.append(rs.choice(ids, (h, w)).astype(np.uint8))
        kinds.append("cityscapes" if k % 2 == 0 else "trainid")
    return imgs, masks, kinds


def host_item(img, mask, kind):
    """one mode='val' item as the reference builds it: `_val_sync_transform` through PIL, ToTensor, the item's mask map"""
    from PIL import Image
    from torchvision import transforms
    img, mask = Image.fromarray(img), Image.fromarray(mask)
    w, h = img.size
    if w > h:
        oh = CROP
        ow = int(1.0 * w * oh / h)
    else:
        ow = CROP
        oh = int(1.0 * h * ow / w)
    img, mask = img.resize((ow, oh), Image.BILINEAR), mask.resize((ow, oh), Image.NEAREST)
    w, h = img.size
    x1, y1 = int(round((w - CROP) / 2.)), int(round((h - CROP) / 2.))
    img, mask = img.crop((x1, y1, x1 + CROP, y1 + CROP)), mask.crop((x1, y1, x1 + CROP, y1 + CROP))
    if kind == "cityscapes":
        m = np.array(mask).astype("int32")
        m[m == 255] = 0
        key = np.array([-1] * 8 + [0, 1, -1, -1, 2, 3, 4, -1, -1, -1, 5, -1, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15, -1, -1, 16, 17, 18])
        lab = torch.from_numpy(key[np.digitize(m.ravel(), np.arange(-1, 34), right=True)].reshape(m.shape)).long()
    else:
        lab = torch.from_numpy(np.array(mask)).long()
        lab[lab == 255] = -1
    return transforms.ToTensor()(img), lab


def host_rate(imgs, masks, kinds, n_items):
    try:
        import PIL  # noqa: F401
        import torchvision  # noqa: F401
    except ImportError as e:
        return {"unavailable": f"{type(e).__name__}: {e}"[:200]}
    torch.set_num_threads(1)
    host_item(imgs[0], masks[0], kinds[0])
    t0 = time.perf_counter()
    for k in range(n_items):
        host_item(imgs[k % len(imgs)], masks[k % len(imgs)], kinds[k % len(imgs)])
    dt = time.perf_counter() - t0
    torch.set_num_threads(max(1, len(os.sched_getaffinity(0))))
    return {"items": n_items, "ms_per_item": 1e3 * dt / n_items, "ms_per_batch": 1e3 * dt / n_items * 4, "img_per_s": n_items / dt}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--batch", type=int, default=4)
    ap.add_argument("--passes", type=int, default=10)
    ap.add_argument("--host-items", type=int, default=16)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_seg_val needs a CUDA device")
    from multiyolov5_b200 import _lib, synth
    from multiyolov5_b200.models.yolo import Model
    from multiyolov5_b200.test import seg_validation
    from multiyolov5_b200.train import SegValBatches
    from multiyolov5_b200.utils.datasets import DeviceSegCache, SegAugmenter
    imgs, masks, kinds = sources(8)
    aug = SegAugmenter(DeviceSegCache(imgs, masks, mask_map=kinds), preset="citysbdd")
    B = a.batch
    sv = SegValBatches(aug, B, mode="val", crop_size=CROP)
    rec = {"workload": dict(batch=B, sources="2048x1024 and 1280x720 alternating", crop=CROP, batches_per_pass=len(sv))}

    # the launch alone, re-run over one uploaded batch
    aug.val(list(range(B)), CROP)
    host, dev, scratch = aug._keep
    isz = C.sizeof(_lib.SegItem)
    out = torch.empty((B, 3, CROP, CROP), dtype=torch.float32, device="cuda")
    labels = torch.empty((B, CROP, CROP), dtype=torch.int64, device="cuda")
    L = _lib.lib()

    def launch():
        _lib.check(L.myolo_augment_seg(C.c_void_p(dev.data_ptr()), B, CROP, CROP, CROP, CROP, C.c_void_p(dev.data_ptr() + B * isz),
                                       _lib.ptr(scratch), _lib.ptr(out), _lib.F32, _lib.ptr(labels), _lib.stream_ptr()))
    for _ in range(a.warmup):
        launch()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(a.steps):
        launch()
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / a.steps
    rec["launch"] = {"ms_per_batch": ms, "us_per_img": 1e3 * ms / B, "img_per_s": 1e3 * B / ms, "batches": a.steps}

    # SegValBatches end to end, to a synchronise
    n_pass = max(1, a.steps // len(sv))
    for _ in range(max(1, a.warmup // len(sv))):
        for _b in sv:
            pass
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(n_pass):
        for _b in sv:
            pass
    torch.cuda.synchronize()
    dt = (time.perf_counter() - t0) / (n_pass * len(sv))
    rec["batches"] = {"ms_per_batch": 1e3 * dt, "img_per_s": B / dt, "batches": n_pass * len(sv)}

    # a validation pass of s/PSP over the device batches, and over the same batches built beforehand
    yml = "yolov5s_city_seg.yaml"
    cfg = synth.load_cfg(yml)
    model = Model(yml)
    model.load_state_dict(synth.synth_state_dict(synth.load_manifest("s_psp"), cfg, seed=1))
    model.cuda()
    n_segcls = model.model[-2].c_out
    built = [(x.clone(), y.clone()) for x, y in sv]
    arms = {"over_SegValBatches": sv, "over_prebuilt_batches": built}
    times = {k: [] for k in arms}
    for k, loader in arms.items():                                 # warm-up: plans and graphs of both batch shapes
        seg_validation(model, n_segcls, loader, "cuda")
    for _ in range(a.passes):                                      # alternate the arms
        for k, loader in arms.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            seg_validation(model, n_segcls, loader, "cuda")        # reads the counters back: ends in a synchronise
            times[k].append(1e3 * (time.perf_counter() - t0) / len(sv))
    rec["validation"] = {k: {"ms_per_batch_median": float(np.median(v)), "ms_per_batch_min": float(np.min(v)), "passes": a.passes}
                         for k, v in times.items()}
    rec["host_reference_1core"] = host_rate(imgs, masks, kinds, a.host_items)
    rec["gpu"] = gpu_state()
    print(json.dumps(rec))


if __name__ == "__main__":
    main()
