#!/usr/bin/env python
"""Benchmark of the class-weighted CE and the focal seg loss in the fused pass (myolo_plan_backward_seg_loss) against the mean CE
(myolo_plan_backward_seg_ce).

    python tools/bench_segloss.py [--steps K] [--warmup W]

Prints ONE JSON line with the card's name, power limit and clocks read next to the measurement:
  fused_kernels  device time per call of the seg loss kernels (CE: count_valid, seg_ce_pixel, seg_ce_gather, seg_ce_finalize; weighted /
                 focal: seg_wf_pixel, seg_wf_finalize, seg_ce_gather) at the s/PSP seg shape: 4 images, 19 classes, 64 x 128 logits ->
                 512 x 1024, from torch.profiler over K calls of each arm, the arms alternating: CE, weighted CE (19 class weights),
                 focal (gamma 2, the same weights).
  seg_pass       the whole seg pass of Trainer.backward_seg on the fused path (train forward + loss + backward through the network), CUDA
                 events per call, the arms alternating in blocks; median and min in ms.
Synthetic weights, images and labels (labels uniform in [-1, 19): ~5 % ignored).
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from tools.bench_augment import gpu_state  # noqa: E402
from tools.bench_ohem import B, H, NC, W, _labels, _model  # noqa: E402

LOSS_KERNELS = ("count_valid", "seg_ce_pixel", "seg_ce_gather", "seg_ce_finalize", "seg_wf_")
CALL_START = ("count_valid", "seg_wf_pixel")


def _arms():
    w = torch.from_numpy(np.random.RandomState(0).uniform(0.5, 1.5, NC).astype(np.float32)).cuda()
    return {"ce": None, "weighted_ce": (w, 0.0), "focal": (w, 2.0)}


def _call(eng, x, labels, arm):
    _, _, plan = eng.train_forward(x, want_seg=False)
    if arm is None:
        return eng.train_backward_seg_ce(plan, labels)
    return eng.train_backward_seg_loss(plan, labels, arm[0], arm[1])


def fused_kernels(model, steps, warmup):
    from oracle import synth
    eng = model.engine()
    x = synth.synth_image(B, H, W, seed=5).cuda()
    labels = _labels()
    arms = _arms()
    for _ in range(warmup):
        for a in arms.values():
            _call(eng, x, labels, a)
    torch.cuda.synchronize()
    per_arm = {k: 0.0 for k in arms}
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(steps):
            for a in arms.values():
                _call(eng, x, labels, a)
        torch.cuda.synchronize()
    # kernels are attributed to the arm by launch order: the loss kernels of one call run back to back between its forward and backward
    evs = sorted((e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA), key=lambda e: e.time_range.start)
    names = list(arms)
    call_i = -1
    for e in evs:
        if any(k in e.name for k in CALL_START):
            call_i += 1
        if call_i >= 0 and any(k in e.name for k in LOSS_KERNELS):
            per_arm[names[call_i % len(names)]] += e.time_range.elapsed_us()
    assert call_i + 1 == steps * len(arms), (call_i + 1, steps * len(arms))
    losses = {k: float(_call(eng, x, labels, a)) for k, a in arms.items()}
    return {k: round(v / steps, 2) for k, v in per_arm.items()}, losses


def seg_pass(model, steps, warmup):
    from oracle import synth
    eng = model.engine()
    x = synth.synth_image(B, H, W, seed=2).cuda()
    labels = _labels()
    arms = _arms()
    times = {k: [] for k in arms}
    for _ in range(warmup):
        for a in arms.values():
            _call(eng, x, labels, a)
    block = 5
    for _ in range(max(1, steps // block)):
        for name, a in arms.items():
            for _ in range(block):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                _call(eng, x, labels, a)
                e1.record()
                torch.cuda.synchronize()
                times[name].append(e0.elapsed_time(e1))
    return {k: {"median_ms": round(float(np.median(ts)), 3), "min_ms": round(float(np.min(ts)), 3), "n": len(ts)} for k, ts in times.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_segloss needs a GPU"
    model, _ = _model()
    kernels_us, losses = fused_kernels(model, args.steps, args.warmup)
    rec = {"bench": "segloss", "gpu": gpu_state(), "shape": [B, NC, H // 8, W // 8, H, W],
           "fused_kernels_us_per_call": kernels_us, "fused_losses": losses, "seg_pass": seg_pass(model, args.steps, args.warmup)}
    ce = rec["seg_pass"]["ce"]["median_ms"]
    rec["seg_pass_over_ce"] = {k: round(v["median_ms"] / ce, 4) for k, v in rec["seg_pass"].items()}
    rec["gpu_after"] = gpu_state()
    print(json.dumps(rec))


if __name__ == "__main__":
    main()
