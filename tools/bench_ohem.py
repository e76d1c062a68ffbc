#!/usr/bin/env python
"""Benchmark of the reference's OhemCELoss on the device (Trainer(seg_loss=OhemCELoss(0.7)), myolo_plan_backward_seg_ohem).

    python tools/bench_ohem.py [--steps K] [--warmup W]

Prints ONE JSON line with the card's name, power limit and clocks read next to the measurement:
  fused_kernels  device time per call of the fused seg loss kernels (count_valid, seg_ce_pixel, the OHEM selection, seg_ce_gather,
                 finalize) at the s/PSP seg shape: 4 images, 19 classes, 64 x 128 logits -> 512 x 1024, from torch.profiler over K calls
                 of each arm, the arms alternating: CE, OHEM on the threshold branch (thresh 0.7) and OHEM on the top-k branch.
  reference      the reference's formulation on the same card and logits: F.interpolate(x8, align_corners=True) + OhemCELoss.forward_once
                 (CE reduction='none', threshold, .numel() host reads, topk, mean) + backward, CUDA events over K calls per branch.
  trainer_step   Trainer.step of 4 det + 4 seg images of 512 x 1024 (s/PSP, fused seg loss), with SegmentationLosses and with
                 OhemCELoss(0.7), CUDA events per step, the arms alternating in blocks; median and min in ms.
Synthetic weights, images, targets and labels (labels uniform in [-1, 19): ~5 % ignored).
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402

from tools.bench_augment import gpu_state  # noqa: E402
from tools.bench_optim import CFGS, HYP  # noqa: E402

B, H, W, NC = 4, 512, 1024, 19
LOSS_KERNELS = ("count_valid", "seg_ce_pixel", "seg_ce_gather", "seg_ce_finalize", "ohem_")


def _model():
    from multiyolov5_b200.models.yolo import Model
    from oracle import synth
    cfg = synth.load_cfg(CFGS["s_psp"])
    model = Model(CFGS["s_psp"])
    model.load_state_dict(synth.synth_state_dict(synth.load_manifest("s_psp"), cfg, seed=1, gain=1.0))
    return model.cuda().train(), cfg


def _labels(seed=3):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.randint(-1, NC, (B, H, W), device="cuda", generator=g)


def fused_kernels(model, steps, warmup):
    from multiyolov5_b200.utils.loss import ohem_thresh_t
    from oracle import synth
    eng = model.engine()
    x = synth.synth_image(B, H, W, seed=5).cuda()
    labels = _labels()
    arms = {"ce": None, "ohem_threshold": ohem_thresh_t(0.7), "ohem_topk": 1e30}

    def call(th):
        _, _, plan = eng.train_forward(x, want_seg=False)
        if th is None:
            return eng.train_backward_seg_ce(plan, labels)
        return eng.train_backward_seg_ohem(plan, labels, th)

    for _ in range(warmup):
        for th in arms.values():
            call(th)
    torch.cuda.synchronize()
    per_arm = {k: 0.0 for k in arms}
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(steps):
            for name, th in arms.items():
                with torch.profiler.record_function(f"arm_{name}"):
                    call(th)
        torch.cuda.synchronize()
    # kernels are attributed to the arm by launch order: the loss kernels of one call run back to back between its forward and backward
    evs = sorted((e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA), key=lambda e: e.time_range.start)
    names = list(arms)
    call_i, in_loss = -1, False
    for e in evs:
        is_loss = any(k in e.name for k in LOSS_KERNELS)
        if is_loss and "count_valid" in e.name:
            call_i += 1
        if is_loss and call_i >= 0:
            per_arm[names[call_i % len(names)]] += e.time_range.elapsed_us()
    losses = {k: float(call(th)) for k, th in arms.items()}
    return {k: round(v / steps, 2) for k, v in per_arm.items()}, losses


def reference(model, steps, warmup):
    from multiyolov5_b200 import _lib
    from multiyolov5_b200.utils.loss import ohem_thresh_t
    from oracle import synth
    eng = model.engine()
    x = synth.synth_image(B, H, W, seed=5).cuda()
    _, _, plan = eng.train_forward(x, want_seg=False)
    v = [o.in_ for o in plan.pb.ops if o.kind == _lib.OP_SEG_UPSAMPLE][0]
    lo = eng.read_view(v, plan)[:, :NC].contiguous()
    labels = _labels()
    crit = torch.nn.CrossEntropyLoss(ignore_index=-1, reduction="none")
    out = {}
    for name, thresh in (("threshold", torch.tensor(ohem_thresh_t(0.7), device="cuda")), ("topk", torch.tensor(1e30, device="cuda"))):
        def once():
            p = lo.clone().requires_grad_(True)
            up = F.interpolate(p, (H, W), mode="bilinear", align_corners=True)
            n_min = int(labels[labels != -1].numel() // 16)
            loss = crit(up, labels).view(-1)
            hard = loss[loss > thresh]
            if hard.numel() < n_min:
                hard, _ = loss.topk(n_min)
            torch.mean(hard).backward()
        for _ in range(warmup):
            once()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record()
        for _ in range(steps):
            once()
        e1.record()
        torch.cuda.synchronize()
        out[name] = round(e0.elapsed_time(e1) * 1000 / steps, 1)
    return out


def trainer_step(model, cfg, steps, warmup):
    from multiyolov5_b200.train import Trainer, scale_hyp
    from multiyolov5_b200.utils.loss import OhemCELoss
    from oracle import synth
    tr = Trainer(model, scale_hyp(HYP, nl=3, nc=cfg["nc"], imgsz=W, total_batch_size=B), batch_size=B, init_scale=2.0 ** 10)
    ohem = OhemCELoss(0.7)
    imgs = synth.synth_image(B, H, W, seed=1).cuda()
    segimgs = synth.synth_image(B, H, W, seed=2).cuda()
    rs = np.random.RandomState(0)
    t = np.zeros((3 * B, 6), np.float32)
    t[:, 0] = np.repeat(np.arange(B), 3); t[:, 1] = rs.randint(0, cfg["nc"], 3 * B)
    t[:, 2:4] = rs.uniform(0.1, 0.9, (3 * B, 2)); t[:, 4:6] = rs.uniform(0.05, 0.4, (3 * B, 2))
    targets = torch.from_numpy(t).cuda()
    labels = _labels()
    times = {"ce": [], "ohem": []}
    for _ in range(warmup):
        for arm in times:
            tr.ohem = ohem if arm == "ohem" else None
            tr.step(imgs, targets, segimgs, labels)
    block = 5
    for _ in range(max(1, steps // block)):
        for arm, ts in times.items():
            tr.ohem = ohem if arm == "ohem" else None
            for _ in range(block):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                tr.step(imgs, targets, segimgs, labels)
                e1.record()
                torch.cuda.synchronize()
                ts.append(e0.elapsed_time(e1))
    return {arm: {"median_ms": round(float(np.median(ts)), 3), "min_ms": round(float(np.min(ts)), 3), "n": len(ts)}
            for arm, ts in times.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_ohem needs a GPU"
    model, cfg = _model()
    kernels_us, losses = fused_kernels(model, args.steps, args.warmup)
    rec = {"bench": "ohem", "gpu": gpu_state(), "shape": [B, NC, H // 8, W // 8, H, W],
           "fused_kernels_us_per_call": kernels_us, "fused_losses": losses,
           "reference_fwd_bwd_us": reference(model, args.steps, args.warmup),
           "trainer_step": trainer_step(model, cfg, args.steps, args.warmup)}
    rec["ohem_step_over_ce"] = round(rec["trainer_step"]["ohem"]["median_ms"] / rec["trainer_step"]["ce"]["median_ms"], 4)
    rec["gpu_after"] = gpu_state()
    print(json.dumps(rec))


if __name__ == "__main__":
    main()
