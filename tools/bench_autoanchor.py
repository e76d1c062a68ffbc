#!/usr/bin/env python
"""Benchmark of the reference's autoanchor on the device (utils.autoanchor: kmean_anchors with gen=1000, myolo_kmeans, myolo_anchor_evolve).

    python tools/bench_autoanchor.py [--repeats R]

Prints ONE JSON line with the card's name, power limit and clocks read next to the measurement, for synthetic label sets of ~60 k
(Cityscapes scale) and ~790 k (COCO scale) labels at img_size 1024 (oracle.restate_autoanchor.synth_dataset):
  host_draws_ms   the 1000 generations' mutation factors drawn on the host (numpy, the reference's loop)
  kmeans_ms       kmeans(wh / s, 9, iter=30) on the device (myolo_kmeans, all 30 restarts in one launch), CUDA events around
                  kmeans_restarts: the launch plus its input copies and the one read-back (median and min of R)
  evolve_ms       myolo_anchor_evolve over the filtered labels, CUDA events around the one cooperative launch (median and min of R)
  end_to_end_ms   kmean_anchors(dataset, n=9, img_size=1024, gen=1000, verbose=False) on a host clock ending in a synchronise
The reference's times on a CPU (8 torch threads) are quoted from its measurement, not re-run here: 10.5 s (3.8 s of it k-means) at 59 793
labels and 121 s (42 s k-means) at 791 794 labels.  So are scipy's kmeans times on the H100 box's CPU, from the same call before it moved
to the device: 5.2 s at 59 802 labels and 76 s at 789 336.
"""
import argparse
import contextlib
import io
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from tools.bench_augment import gpu_state  # noqa: E402

CITY = [(12, 30), (25, 60), (40, 25), (90, 55), (200, 120), (8, 8), (30, 80), (150, 300)]
SIZES = {"60k": (600, 100), "790k": (7900, 100)}
QUOTED_CPU_S = {"60k": {"labels": 59793, "total_s": 10.5, "kmeans_s": 3.8}, "790k": {"labels": 791794, "total_s": 121.0, "kmeans_s": 42.0}}
QUOTED_SCIPY_S = {"60k": 5.2, "790k": 76.0}
IMG, N, GEN = 1024, 9, 1000


class _Dataset:
    def __init__(self, shapes, labels):
        self.shapes, self.labels = shapes, labels


def _timed(fn, repeats):
    """CUDA event times (ms) of fn() over `repeats` calls, and its last result"""
    ts = []
    for _ in range(repeats):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        out = fn()
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    return ts, out


def _stats(ts, nd=3):
    return {"median": round(float(np.median(ts)), nd), "min": round(float(np.min(ts)), nd), "n": len(ts)}


def one_size(tag, repeats):
    from multiyolov5_b200.utils import autoanchor as aa
    from oracle import restate_autoanchor as ra
    n_img, per = SIZES[tag]
    shapes0, labels = ra.synth_dataset(17, n_img, per, CITY, spread=0.45, shapes=((1024, 2048), (720, 1280), (480, 640)))
    ds = _Dataset(ra.shapes_wh(shapes0), labels)
    wh0 = ra.label_wh(ds.shapes, labels, IMG)
    wh = wh0[(wh0 >= 2.0).any(1)]
    print(f"{tag}: {len(wh0)} labels", file=sys.stderr, flush=True)
    np.random.seed(0)
    t0 = time.perf_counter()
    V = aa.draw_mutations(GEN, (N, 2))
    draws_ms = (time.perf_counter() - t0) * 1e3
    s = wh.std(0)
    obs = wh / s
    idx = np.stack([np.random.choice(len(obs), N, replace=False) for _ in range(30)])
    aa.kmeans_restarts(obs, idx[:2])                               # warm-up: module load, allocator
    km, (books, _, iters, best) = _timed(lambda: aa.kmeans_restarts(obs, idx), repeats)
    print(f"{tag}: kmeans {np.median(km):.1f} ms", file=sys.stderr, flush=True)
    k = ra.sort_by_area(books[best] * s)
    wh_d = torch.tensor(wh, dtype=torch.float32).cuda()
    aa.evolve(wh_d, k, V[:10], 0.25)
    ev, out = _timed(lambda: aa.evolve(wh_d, k, V, 0.25), repeats)
    e2e = []
    for r in range(3):
        np.random.seed(r)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        with contextlib.redirect_stdout(io.StringIO()):
            aa.kmean_anchors(ds, n=N, img_size=IMG, thr=4.0, gen=GEN, verbose=False)
        torch.cuda.synchronize()
        e2e.append((time.perf_counter() - t0) * 1e3)
    # both event windows include the host->device copies of the inputs and the device->host reads of the results
    return {"labels": int(len(wh0)), "labels_filtered": int(len(wh)), "host_draws_ms": round(draws_ms, 2), "kmeans_ms": _stats(km),
            "kmeans_lloyd_iterations": {"max": int(iters.max()), "sum": int(iters.sum())}, "evolve_ms": _stats(ev),
            "evolve_us_per_generation": round(float(np.median(ev)) * 1e3 / GEN, 2), "accepted": out[4],
            "end_to_end_ms": _stats(e2e, 1), "scipy_kmeans_quoted_s": QUOTED_SCIPY_S[tag], "reference_cpu_quoted": QUOTED_CPU_S[tag]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=10)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_autoanchor needs a GPU"
    rec = {"bench": "autoanchor", "gpu": gpu_state(), "n": N, "img_size": IMG, "gen": GEN}
    for tag in SIZES:
        rec[tag] = one_size(tag, args.repeats)
        print(f"{tag}: {json.dumps(rec[tag])}", file=sys.stderr, flush=True)
    rec["gpu_after"] = gpu_state()
    print(json.dumps(rec))


if __name__ == "__main__":
    main()
