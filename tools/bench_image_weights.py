#!/usr/bin/env python
"""Benchmark of --image-weights on the device (csrc/image_weights.cu, utils.datasets.ImageWeights).

    python tools/bench_image_weights.py [--launches L]

Prints ONE JSON line with the card's name, power limit and clocks read in the same run, for synthetic label sets at Cityscapes scale
(2 975 images, 10 classes, about 6 labels per image) and COCO scale (118 287 images, 80 classes, about 7.3 labels per image):
  class_weights_us    myolo_class_weights on uploaded labels (count kernel + weights kernel), CUDA events over L launches, per launch
  image_weights_us    myolo_image_weights, the same way
  weighted_draw_us    myolo_weighted_draw (the sequential scan + the bisect kernel), the same way
  draw_ms             one whole ImageWeights.draw on a host clock ending in a synchronise: cw on the host, n random() draws, the upload
                      of the uniforms, the kernels and the read-back of the indices (median and min of 10)
  cpu_ms              the reference's formulation on one CPU core: labels_to_class_weights (per-class bincount of the concatenated
                      labels, 1 / count, / sum), labels_to_image_weights (one bincount per image, (cw * counts).sum(1)) and
                      random.choices(range(n), weights=iw, k=n), each the median of 5 runs
"""
import argparse
import json
import os
import random
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from tools.bench_augment import gpu_state  # noqa: E402

SIZES = {"cityscapes": (2975, 10, 6.0), "coco": (118_287, 80, 7.3)}


def synth(n, nc, per, seed=0):
    rs = np.random.RandomState(seed)
    k = rs.poisson(per, n)
    labels = []
    for i in range(n):
        lb = np.full((k[i], 5), 0.5, np.float32)
        lb[:, 0] = rs.randint(0, nc, k[i])
        labels.append(lb)
    return labels


def _events(fn, launches):
    fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(launches):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return round(e0.elapsed_time(e1) * 1e3 / launches, 2)


def _median_ms(fn, runs):
    ts = []
    for _ in range(runs):
        t0 = time.perf_counter()
        fn()
        ts.append((time.perf_counter() - t0) * 1e3)
    return ts


def cpu_reference(labels, nc, cw):
    """the reference's three steps, on the host, one core"""
    def class_weights():
        c = np.bincount(np.concatenate(labels, 0)[:, 0].astype(int), minlength=nc)
        c[c == 0] = 1
        w = 1 / c
        return w / w.sum()

    def image_weights():
        counts = np.array([np.bincount(x[:, 0].astype(int), minlength=nc) for x in labels])
        return (cw.reshape(1, nc) * counts).sum(1)

    iw = image_weights()
    return {"class_weights": round(float(np.median(_median_ms(class_weights, 5))), 2),
            "image_weights": round(float(np.median(_median_ms(image_weights, 5))), 2),
            "random_choices": round(float(np.median(_median_ms(lambda: random.choices(range(len(labels)), weights=iw, k=len(labels)),
                                                                 5))), 2)}


def one_size(tag, launches):
    from multiyolov5_b200 import _lib
    from multiyolov5_b200.utils.datasets import ImageWeights
    from multiyolov5_b200.utils.general import device_image_weights, label_classes, labels_to_class_weights
    n, nc, per = SIZES[tag]
    labels = synth(n, nc, per)
    L, sp = _lib.lib(), _lib.stream_ptr()
    cls, offsets = label_classes(labels)
    status = torch.zeros(1, dtype=torch.int32, device="cuda")
    counts = torch.empty(nc, dtype=torch.int64, device="cuda")
    w = torch.empty(nc, dtype=torch.float64, device="cuda")
    cw_model = labels_to_class_weights(labels, nc) * nc
    maps = np.random.RandomState(1).uniform(0, 0.9, nc)
    cw = cw_model.cpu().numpy() * (1 - maps) ** 2 / nc
    iw = device_image_weights(cls, offsets, cw, status)
    u = torch.rand(n, dtype=torch.float64, device="cuda")
    cum = torch.empty(n, dtype=torch.float64, device="cuda")
    total = torch.empty(1, dtype=torch.float64, device="cuda")
    idx = torch.empty(n, dtype=torch.int32, device="cuda")
    cwd = torch.from_numpy(cw).cuda()
    rec = {"images": n, "nc": nc, "labels": int(cls.numel())}
    rec["class_weights_us"] = _events(lambda: _lib.check(L.myolo_class_weights(_lib.ptr(cls), cls.numel(), nc, _lib.ptr(counts),
                                                                               _lib.ptr(w), _lib.ptr(status), sp)), launches)
    rec["image_weights_us"] = _events(lambda: _lib.check(L.myolo_image_weights(_lib.ptr(cls), _lib.ptr(offsets), n, _lib.ptr(cwd), nc,
                                                                               _lib.ptr(iw), _lib.ptr(status), sp)), launches)
    rec["weighted_draw_us"] = _events(lambda: _lib.check(L.myolo_weighted_draw(_lib.ptr(iw), _lib.ptr(u), n, _lib.ptr(cum),
                                                                               _lib.ptr(total), _lib.ptr(idx), _lib.ptr(status), sp)),
                                      launches)
    assert int(status.item()) == 0

    class _Aug:
        def __init__(self):
            self.n, self.indices = n, range(n)
            self.cache = type("Cache", (), {"labels": labels})()
    iwts = ImageWeights(_Aug())
    iwts.draw(cw_model, maps)                                      # uploads the labels once, warms the kernels

    def whole():
        iwts.draw(cw_model, maps)
        torch.cuda.synchronize()
    ts = _median_ms(whole, 10)
    rec["draw_ms"] = {"median": round(float(np.median(ts)), 3), "min": round(float(np.min(ts)), 3), "n": len(ts)}
    rec["cpu_ms"] = cpu_reference(labels, nc, cw)
    return rec


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=200)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_image_weights needs a GPU"
    torch.set_num_threads(1)
    rec = {"bench": "image_weights", "gpu": gpu_state()}
    for tag in SIZES:
        rec[tag] = one_size(tag, args.launches)
        print(f"{tag}: {json.dumps(rec[tag])}", file=sys.stderr, flush=True)
    rec["gpu_after"] = gpu_state()
    print(json.dumps(rec))


if __name__ == "__main__":
    main()
