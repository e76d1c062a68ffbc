#!/usr/bin/env python
"""Benchmark of the detection validation batches on the device (myolo_resize_area_u8, DeviceImageCache(augment=False), DetValLoader).

    python tools/bench_val_batches.py [--steps K] [--warmup W]

The workload is Cityscapes val as test() sees it during training: 500 synthetic 2048x1024 frames, img_size 1024, batch 32, which gives
the batch shape 544x1056.  Prints ONE JSON line with the card's name, power limit and clocks read next to the measurement:
  area_us_{shape}          myolo_resize_area_u8 of one frame, CUDA events over K (>= 200) launches, and its GB/s from source +
                           destination bytes; shapes 2048x1024->640x320, 1280x720->1024x576, 1920x1080->640x360
  cv2_area_ms_{shape}      cv2.resize(INTER_AREA) of the same frame on one host core
  cv2_cache_ms_500         the reference's cache build resize: ThreadPool(8) over 500 frames 2048x1024->1024x512 (decoding excluded)
  cache_ms_500             DeviceImageCache(augment=False) of the 500 device-resident frames, to a device synchronise
  loader_us_per_image      one full DetValLoader pass over the 500 images, to a device synchronise
  ref_item_us_per_image    the reference's per-item host work for the same pass: copyMakeBorder, BGR->RGB transpose, torch.stack,
                           pinned host-to-device copy (one host thread)
  test_ms_500_{loader,prebuilt}  test() end to end with the s/PSP model in half precision, fed by DetValLoader or by the same batches
                           built beforehand on the device, alternating in this process (best of the repeats)
Writes nothing to disk.
"""
import argparse
import json
import os
import sys
import time
from multiprocessing.pool import ThreadPool

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from tools.bench_augment import gpu_state  # noqa: E402

AREA_SHAPES = [((1024, 2048), (320, 640)), ((720, 1280), (576, 1024)), ((1080, 1920), (360, 640))]


def _tag(hw0, hw):
    return f"{hw0[1]}x{hw0[0]}_{hw[1]}x{hw[0]}"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--images", type=int, default=500)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_val_batches needs a CUDA device")
    steps = max(args.steps, 200)
    from multiyolov5_b200 import _lib
    from multiyolov5_b200.utils.datasets import DetValLoader, DeviceImageCache
    L = _lib.lib()
    try:
        import cv2
        cv2.setNumThreads(1)
    except ImportError:
        cv2 = None
    rec = {"gpu": gpu_state(), "images": args.images, "img_size": 1024, "batch_size": 32, "host_cpus": os.cpu_count()}
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    g = torch.Generator(device="cuda").manual_seed(0)

    # ---- the area resize kernel alone, and cv2 on one core
    for hw0, hw in AREA_SHAPES:
        src = torch.randint(0, 256, hw0 + (3,), dtype=torch.uint8, device="cuda", generator=g)
        dst = torch.empty(hw + (3,), dtype=torch.uint8, device="cuda")
        args_ = (_lib.ptr(src), hw0[0], hw0[1], _lib.ptr(dst), hw[0], hw[1], _lib.stream_ptr())
        for _ in range(args.warmup):
            _lib.check(L.myolo_resize_area_u8(*args_))
        torch.cuda.synchronize()
        ev0.record()
        for _ in range(steps):
            L.myolo_resize_area_u8(*args_)
        ev1.record()
        torch.cuda.synchronize()
        us = ev0.elapsed_time(ev1) * 1e3 / steps
        rec[f"area_us_{_tag(hw0, hw)}"] = us
        rec[f"area_gbps_{_tag(hw0, hw)}"] = (src.numel() + dst.numel()) / (us * 1e-6) / 1e9
        if cv2 is not None:
            h_src = src.cpu().numpy()
            times = []
            for _ in range(10):
                t0 = time.perf_counter()
                cv2.resize(h_src, (hw[1], hw[0]), interpolation=cv2.INTER_AREA)
                times.append(time.perf_counter() - t0)
            rec[f"cv2_area_ms_{_tag(hw0, hw)}"] = float(np.median(times) * 1e3)

    # ---- the validation cache and loader over the Cityscapes val workload
    n = args.images
    distinct = [torch.randint(0, 256, (1024, 2048, 3), dtype=torch.uint8, device="cuda", generator=g) for _ in range(8)]
    frames = [distinct[i % 8] for i in range(n)]
    rs = np.random.RandomState(0)
    labels = []
    for _ in range(n):
        k = rs.randint(5, 25)
        lb = np.zeros((k, 5), np.float32)
        lb[:, 0] = rs.randint(0, 10, k)
        lb[:, 1:3] = rs.uniform(0.1, 0.9, (k, 2))
        lb[:, 3:5] = rs.uniform(0.02, 0.2, (k, 2))
        labels.append(lb)
    DeviceImageCache(frames[:8], 1024, labels[:8], augment=False)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    cache = DeviceImageCache(frames, 1024, labels, augment=False)
    torch.cuda.synchronize()
    rec["cache_ms_500"] = (time.perf_counter() - t0) * 1e3
    if cv2 is not None:
        h_frames = [f.cpu().numpy() for f in distinct]
        cv2.setNumThreads(0)                       # the reference's default: cv2's own threading inside each of the 8 workers
        with ThreadPool(8) as pool:
            t0 = time.perf_counter()
            list(pool.imap(lambda i: cv2.resize(h_frames[i % 8], (1024, 512), interpolation=cv2.INTER_AREA), range(n)))
            rec["cv2_cache_ms_500"] = (time.perf_counter() - t0) * 1e3
        cv2.setNumThreads(1)
    loader = DetValLoader(cache, 32)
    rec["batch_shapes"] = sorted({tuple(s) for s in loader.batch_shapes.tolist()})
    for _ in loader:
        pass
    times = []
    for _ in range(3):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in loader:
            pass
        torch.cuda.synchronize()
        times.append(time.perf_counter() - t0)
    rec["loader_us_per_image"] = float(min(times) * 1e6 / n)

    # ---- the reference's per-item host work for the same pass (letterbox is a copyMakeBorder here: r = 1)
    if cv2 is not None:
        cached = [cache.image(i).cpu().numpy() for i in range(8)]
        torch.set_num_threads(1)
        times = []
        for _ in range(2):
            t0 = time.perf_counter()
            for b, batch in enumerate(loader.batches):
                H, W = loader.batch_shapes[b].tolist()
                items = []
                for i, geom in zip(batch.indices, batch.geoms):
                    top, bottom, left, right = geom[3]
                    img = cv2.copyMakeBorder(cached[i % 8], top, bottom, left, right, cv2.BORDER_CONSTANT, value=(114, 114, 114))
                    items.append(torch.from_numpy(np.ascontiguousarray(img[:, :, ::-1].transpose(2, 0, 1))))
                x = torch.stack(items, 0).pin_memory().to("cuda", non_blocking=True)
            torch.cuda.synchronize()
            times.append(time.perf_counter() - t0)
            del x
        rec["ref_item_us_per_image"] = float(min(times) * 1e6 / n)

    # ---- test() fed by the loader and by pre-built device batches, alternating
    from multiyolov5_b200.models.yolo import Model
    from multiyolov5_b200.test import test
    from oracle import synth
    yml = "yolov5s_city_seg.yaml"
    cfg = synth.load_cfg(yml)
    model = Model(yml)
    model.load_state_dict(synth.synth_state_dict(synth.load_manifest("s_psp"), cfg, seed=1))
    model.cuda().eval()
    prebuilt = [(i.clone(), t, p, s) for i, t, p, s in loader]
    data = {"nc": cfg["nc"]}
    test(data, model=model, dataloader=prebuilt, plots=False)                 # warm-up: plans for both batch sizes
    res = {}
    times = {"loader": [], "prebuilt": []}
    for _ in range(3):
        for name, dl in (("loader", loader), ("prebuilt", prebuilt)):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            res[name] = test(data, model=model, dataloader=dl, plots=False)[0]
            times[name].append(time.perf_counter() - t0)
    for name, v in times.items():
        rec[f"test_ms_500_{name}"] = float(min(v) * 1e3)
        rec[f"test_ms_500_{name}_all"] = [float(x * 1e3) for x in v]
    rec["test_same_result"] = bool(res["loader"] == res["prebuilt"])
    rec["gpu_after"] = gpu_state()
    print(json.dumps(rec), flush=True)


if __name__ == "__main__":
    main()
