#!/usr/bin/env python
"""Benchmark of the device-side detection training batches (DetAugmenter, csrc/augment.cu) against the reference's host loader.

    python tools/bench_augment.py [--steps K] [--warmup W] [--batch B] [--img-size S]

Prints ONE JSON line: the kernel alone (CUDA events over K launches), the builder end to end (host draws + labels + parameter upload +
kernel, to a device synchronise) and the reference's per-item arithmetic through cv2 on one core and on every core of this host, plus
the card's name, power limit and clocks read next to the measurement.  Writes nothing to disk.
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402


def gpu_state(gpu_index=0):
    """name, power limit and clocks of the card (a number is only worth something with them)"""
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader,nounits", "-i", str(gpu_index)],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        name, power_w, sm, sm_max = [v.strip() for v in out.split(",")]
        return {"name": name, "power_limit_w": float(power_w), "sm_mhz": float(sm), "sm_max_mhz": float(sm_max)}
    except Exception as e:
        return {"name": torch.cuda.get_device_name(gpu_index), "unavailable": f"{type(e).__name__}: {e}"[:200]}


AUG_HYP = dict(hsv_h=0.015, hsv_s=0.7, hsv_v=0.4, degrees=0.0, translate=0.1, scale=0.5, shear=0.0, perspective=0.0, flipud=0.0,
               fliplr=0.5, mosaic=1.0, mixup=0.0)      # reference data/hyp.scratch.yaml


def _host_augment_item(cache, labels, s, hyp, index, cv2):
    """the reference's per-item host arithmetic through cv2 (load_mosaic + random_perspective + augment_hsv + flips + CHW), for the
    host arm of the augment record; labels are left out (they are host work in both arms)"""
    import math
    import random
    yc, xc = [int(random.uniform(s // 2, 2 * s - s // 2)) for _ in range(2)]
    idx = [index] + random.choices(range(len(cache)), k=3)
    img4 = np.full((2 * s, 2 * s, 3), 114, dtype=np.uint8)
    for i, k in enumerate(idx):
        img = cache[k]
        h, w = img.shape[:2]
        if i == 0:
            x1a, y1a, x2a, y2a = max(xc - w, 0), max(yc - h, 0), xc, yc
            x1b, y1b, x2b, y2b = w - (x2a - x1a), h - (y2a - y1a), w, h
        elif i == 1:
            x1a, y1a, x2a, y2a = xc, max(yc - h, 0), min(xc + w, s * 2), yc
            x1b, y1b, x2b, y2b = 0, h - (y2a - y1a), min(w, x2a - x1a), h
        elif i == 2:
            x1a, y1a, x2a, y2a = max(xc - w, 0), yc, xc, min(s * 2, yc + h)
            x1b, y1b, x2b, y2b = w - (x2a - x1a), 0, w, min(y2a - y1a, h)
        else:
            x1a, y1a, x2a, y2a = xc, yc, min(xc + w, s * 2), min(s * 2, yc + h)
            x1b, y1b, x2b, y2b = 0, 0, min(w, x2a - x1a), min(y2a - y1a, h)
        img4[y1a:y2a, x1a:x2a] = img[y1b:y2b, x1b:x2b]
    C_ = np.eye(3); C_[0, 2] = C_[1, 2] = -s
    R = np.eye(3)
    R[:2] = cv2.getRotationMatrix2D(angle=random.uniform(-hyp["degrees"], hyp["degrees"]), center=(0, 0),
                                    scale=random.uniform(1 - hyp["scale"], 1 + hyp["scale"]))
    S = np.eye(3)
    S[0, 1] = math.tan(random.uniform(-hyp["shear"], hyp["shear"]) * math.pi / 180)
    S[1, 0] = math.tan(random.uniform(-hyp["shear"], hyp["shear"]) * math.pi / 180)
    T = np.eye(3)
    T[0, 2] = random.uniform(0.5 - hyp["translate"], 0.5 + hyp["translate"]) * s
    T[1, 2] = random.uniform(0.5 - hyp["translate"], 0.5 + hyp["translate"]) * s
    M = T @ S @ R @ C_
    img = cv2.warpAffine(img4, M[:2], dsize=(s, s), borderValue=(114, 114, 114))
    r = np.random.uniform(-1, 1, 3) * [hyp["hsv_h"], hyp["hsv_s"], hyp["hsv_v"]] + 1
    hue, sat, val = cv2.split(cv2.cvtColor(img, cv2.COLOR_BGR2HSV))
    x = np.arange(0, 256, dtype=np.int16)
    luts = ((x * r[0]) % 180).astype(np.uint8), np.clip(x * r[1], 0, 255).astype(np.uint8), np.clip(x * r[2], 0, 255).astype(np.uint8)
    hsv = cv2.merge((cv2.LUT(hue, luts[0]), cv2.LUT(sat, luts[1]), cv2.LUT(val, luts[2])))
    cv2.cvtColor(hsv, cv2.COLOR_HSV2BGR, dst=img)
    if random.random() < hyp["fliplr"]:
        img = np.fliplr(img)
    return np.ascontiguousarray(img[:, :, ::-1].transpose(2, 0, 1))


def augment_record(steps, warmup, B=16, s=1024):
    """device detection batches (DetAugmenter: mosaic + affine warp + HSV + flips, one kernel per batch) against the reference's host
    arithmetic through cv2 on one core and on every core of this host.  Sources: 8 Cityscapes-shaped 1024x512 images already in the
    device cache (no resize), hyp.scratch."""
    import random
    from concurrent.futures import ThreadPoolExecutor
    from multiyolov5_b200.utils.datasets import DetAugmenter, DeviceImageCache
    rs = np.random.RandomState(0)
    srcs = [rs.randint(0, 256, (512, 1024, 3), dtype=np.uint8) for _ in range(8)]
    labels = [np.array([[k % 10, 0.5, 0.5, 0.2, 0.3], [1, 0.1, 0.8, 0.1, 0.2]], np.float32) for k in range(8)]
    cache = DeviceImageCache(srcs, s, labels)
    aug = DetAugmenter(cache, AUG_HYP)
    random.seed(0)
    np.random.seed(0)
    idx = [int(i) for i in rs.randint(0, 8, B)]
    for _ in range(warmup):
        aug(idx)
    torch.cuda.synchronize()
    # device time of the kernel alone (parameters prepared once), CUDA events around `steps` launches
    from multiyolov5_b200 import _lib
    L = _lib.lib()
    items = (_lib.AugItem * B)()
    for b, i in enumerate(idx):
        items[b], _ = aug.item(i)
    dev_items = torch.frombuffer(bytearray(items), dtype=torch.uint8).cuda()
    out = torch.empty((B, 3, s, s), dtype=torch.uint8, device="cuda")
    sp = _lib.stream_ptr()
    for _ in range(warmup):
        _lib.check(L.myolo_augment_det_hw(_lib.ptr(dev_items), B, s, s, _lib.ptr(out), _lib.U8, sp))
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        _lib.check(L.myolo_augment_det_hw(_lib.ptr(dev_items), B, s, s, _lib.ptr(out), _lib.U8, sp))
    e1.record()
    torch.cuda.synchronize()
    kernel_ms = e0.elapsed_time(e1) / steps
    # builder end to end: host draws + labels + parameter upload + kernel, timed to a device synchronise
    t0 = time.perf_counter()
    for _ in range(steps):
        aug(idx)
    torch.cuda.synchronize()
    builder_ms = (time.perf_counter() - t0) * 1e3 / steps
    rec = {"B": B, "img_size": s, "sources": "8 x 1024x512 BGR uint8 in the device cache", "hyp": "hyp.scratch",
           "kernel_us_per_image": kernel_ms * 1e3 / B, "kernel_images_per_s": B / (kernel_ms * 1e-3),
           "builder_us_per_image": builder_ms * 1e3 / B, "builder_images_per_s": B / (builder_ms * 1e-3),
           "bytes_written_per_image": 3 * s * s,
           "kernel_hbm_gbs": 3 * s * s * B / (kernel_ms * 1e-3) / 1e9}
    try:
        import cv2
    except ImportError as e:
        rec["host"] = {"unavailable": str(e)}
        return rec
    n_host = max(4, B // 2)
    n_cores = os.cpu_count() or 1
    prev = cv2.getNumThreads()
    cv2.setNumThreads(1)
    try:
        _host_augment_item(srcs, labels, s, AUG_HYP, 0, cv2)
        t0 = time.perf_counter()
        for k in range(n_host):
            _host_augment_item(srcs, labels, s, AUG_HYP, k % 8, cv2)
        one_ms = (time.perf_counter() - t0) * 1e3 / n_host
        n_all = n_host * n_cores
        with ThreadPoolExecutor(max_workers=n_cores) as ex:
            list(ex.map(lambda k: _host_augment_item(srcs, labels, s, AUG_HYP, k % 8, cv2), range(n_cores)))
            t0 = time.perf_counter()
            list(ex.map(lambda k: _host_augment_item(srcs, labels, s, AUG_HYP, k % 8, cv2), range(n_all)))
            all_s = time.perf_counter() - t0
    finally:
        cv2.setNumThreads(prev)
    rec["host"] = {"ms_per_image_one_core": one_ms, "images_per_s_one_core": 1e3 / one_ms, "cores": n_cores,
                   "images_per_s_all_cores": n_all / all_s,
                   "note": "reference arithmetic through cv2 (cv2 single-threaded per call, one Python thread per core)"}
    return rec


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--img-size", type=int, default=1024)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_augment needs a CUDA device")
    rec = augment_record(args.steps, args.warmup, B=args.batch, s=args.img_size)
    rec["gpu"] = gpu_state(torch.cuda.current_device())
    print(json.dumps(rec), flush=True)


if __name__ == "__main__":
    main()
