#!/usr/bin/env python
"""Benchmark of the device-side segmentation training batches (SegAugmenter, csrc/augment_seg.cu) against the reference's host loader.

    python tools/bench_seg_augment.py [--steps K] [--warmup W] [--batch B]

Workload: B = 4 items of 2048x1024 sources (Cityscapes' size), base_size 1024, crop (1024, 512), the `citys` preset.  Prints ONE JSON
line: the two kernels alone (CUDA events over K batches of fixed parameters), the builder end to end (host draws + tables + parameter
upload + kernels, to a device synchronise) and the reference's operations through PIL + torchvision (mirror, resize, pad, crop,
ColorJitter, ToTensor, mask mapping) on one core and on every core of this host - recorded as unavailable when those libraries are not
installed - plus the card's name and power limit read next to the measurement.  Writes nothing to disk.
"""
import argparse
import json
import os
import random
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402


def gpu_state(gpu_index=0):
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader,nounits", "-i", str(gpu_index)],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        name, power_w, sm, sm_max = [v.strip() for v in out.split(",")]
        return {"name": name, "power_limit_w": float(power_w), "sm_mhz": float(sm), "sm_max_mhz": float(sm_max)}
    except Exception as e:
        return {"name": torch.cuda.get_device_name(gpu_index), "unavailable": f"{type(e).__name__}: {e}"[:200]}


def sources(n, seed=0):
    rs = np.random.RandomState(seed)
    yy, xx = np.mgrid[0:1024, 0:2048]
    base = np.stack([xx * 255 // 2047, yy * 255 // 1023, (xx ^ yy) & 255], -1)
    imgs = [np.clip(base + rs.randint(-40, 41, (1024, 2048, 3)), 0, 255).astype(np.uint8) for _ in range(n)]
    masks = [rs.randint(0, 34, (1024, 2048)).astype(np.uint8) for _ in range(n)]
    return imgs, masks


_HOST = {}


def _host_init(imgs, masks):
    _HOST["imgs"], _HOST["masks"] = imgs, masks


def _host_item(k):
    """one item of the reference's mode='train' path through PIL + torchvision (`_sync_transform` with a uniform long side in
    [672, 3072] standing in for get_long_size, ColorJitter, ToTensor, the Cityscapes mask map)"""
    from PIL import Image, ImageOps
    from torchvision import transforms
    torch.set_num_threads(1)
    img, mask = Image.fromarray(_HOST["imgs"][k % len(_HOST["imgs"])]), Image.fromarray(_HOST["masks"][k % len(_HOST["masks"])])
    if random.random() < 0.5:
        img, mask = img.transpose(Image.FLIP_LEFT_RIGHT), mask.transpose(Image.FLIP_LEFT_RIGHT)
    long_size = random.randint(21, 96) * 32
    w, h = img.size
    ow, oh = long_size, int(1.0 * h * long_size / w + 0.5)
    img, mask = img.resize((ow, oh), Image.BILINEAR), mask.resize((ow, oh), Image.NEAREST)
    if ow < 1024 or oh < 512:
        padh, padw = max(512 - oh, 0), max(1024 - ow, 0)
        img, mask = ImageOps.expand(img, border=(0, 0, padw, padh), fill=0), ImageOps.expand(mask, border=(0, 0, padw, padh), fill=255)
    w, h = img.size
    x1, y1 = random.randint(0, w - 1024), random.randint(0, h - 512)
    img, mask = img.crop((x1, y1, x1 + 1024, y1 + 512)), mask.crop((x1, y1, x1 + 1024, y1 + 512))
    t = transforms.Compose([transforms.ColorJitter(0.45, 0.45, 0.45, 0.15), transforms.ToTensor()])
    m = np.array(mask).astype("int32")
    m[m == 255] = 0
    key = np.array([-1] * 8 + [0, 1, -1, -1, 2, 3, 4, -1, -1, -1, 5, -1, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15, -1, -1, 16, 17, 18])
    lab = torch.from_numpy(key[np.digitize(m.ravel(), np.arange(-1, 34), right=True)].reshape(m.shape)).long()
    return t(img).shape, lab.shape


def host_rate(imgs, masks, n_items, workers):
    try:
        import PIL  # noqa: F401
        import torchvision  # noqa: F401
    except ImportError as e:
        return {"unavailable": f"{type(e).__name__}: {e}"[:200]}
    if workers == 1:
        _host_init(imgs, masks)
        t0 = time.perf_counter()
        for k in range(n_items):
            _host_item(k)
        dt = time.perf_counter() - t0
    else:
        import multiprocessing as mp
        ctx = mp.get_context("fork")
        with ctx.Pool(workers, initializer=_host_init, initargs=(imgs, masks)) as pool:
            pool.map(_host_item, range(workers))                      # warm-up: imports in every worker
            t0 = time.perf_counter()
            pool.map(_host_item, range(n_items), chunksize=1)
            dt = time.perf_counter() - t0
    return {"workers": workers, "items": n_items, "ms_per_item": 1e3 * dt / n_items * workers if workers > 1 else 1e3 * dt / n_items,
            "img_per_s": n_items / dt}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--batch", type=int, default=4)
    ap.add_argument("--host-items", type=int, default=24)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_seg_augment needs a CUDA device")
    from multiyolov5_b200.utils.datasets import DeviceSegCache, SegAugmenter
    imgs, masks = sources(8)
    cache = DeviceSegCache(imgs, masks, mask_map="cityscapes")
    aug = SegAugmenter(cache, base_size=1024, crop_size=(1024, 512), preset="citys")
    B = a.batch
    rec = {"workload": dict(batch=B, source="2048x1024", base_size=1024, crop="1024x512", preset="citys")}
    random.seed(0)
    torch.manual_seed(0)
    # kernels alone: fixed parameters, the launches re-run over the same uploaded items (their contrast sums keep accumulating, which
    # changes the output but not the work)
    idx = list(range(B))
    params = [aug.draw(i) for i in idx]
    aug.build(idx, params)
    host, dev, scratch = aug._keep
    from multiyolov5_b200 import _lib
    import ctypes as C
    isz = C.sizeof(_lib.SegItem)
    imgs_out = torch.empty((B, 3, 512, 1024), dtype=torch.float32, device="cuda")
    labels = torch.empty((B, 512, 1024), dtype=torch.int64, device="cuda")
    L = _lib.lib()

    def launch():
        _lib.check(L.myolo_augment_seg(C.c_void_p(dev.data_ptr()), B, 512, 1024, 512, 1024, C.c_void_p(dev.data_ptr() + B * isz),
                                       _lib.ptr(scratch), _lib.ptr(imgs_out), _lib.F32, _lib.ptr(labels), _lib.stream_ptr()))
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
    rec["kernels"] = {"ms_per_batch": ms, "us_per_img": 1e3 * ms / B, "img_per_s": 1e3 * B / ms, "batches": a.steps}
    # builder end to end: draws + tables + upload + kernels, to a synchronise
    rs = np.random.RandomState(1)
    for _ in range(a.warmup):
        aug([int(i) for i in rs.randint(0, cache.n, B)])
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(a.steps):
        aug([int(i) for i in rs.randint(0, cache.n, B)])
    torch.cuda.synchronize()
    dt = (time.perf_counter() - t0) / a.steps
    rec["builder"] = {"ms_per_batch": 1e3 * dt, "img_per_s": B / dt, "batches": a.steps}
    ncpu = len(os.sched_getaffinity(0))
    rec["host_reference_1core"] = host_rate(imgs, masks, a.host_items, 1)
    rec["host_reference_all_cores"] = host_rate(imgs, masks, max(a.host_items, 4 * ncpu), ncpu)
    rec["host_cores"] = ncpu
    rec["gpu"] = gpu_state()
    print(json.dumps(rec))


if __name__ == "__main__":
    main()
