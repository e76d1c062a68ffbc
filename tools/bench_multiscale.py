#!/usr/bin/env python
"""Benchmark of --multi-scale training (reference train.py:354-359): the rescale kernel, train steps through the det lane's shared
workspace, and a multi-scale run.

    python tools/bench_multiscale.py [--steps K] [--warmup W]

Prints ONE JSON line with the card's name, power limit and clocks read next to the measurement:
  rescale_us_{s}        myolo_resize_bilinear of a B=4 uint8 1024x1024 batch to s x s (fp16 out), CUDA events over K (>= 200) launches
  interpolate_us_{s}    the reference's `F.interpolate(imgs.float() / 255.0, ...)` of the same batch on the same card (both launches)
  step_arms             Trainer.step (s/PSP, B=4, seg batch 4 x 512 x 1024) through the shared workspace and through private plans,
                        the two trainers alternating step by step, median and min over K/10 steps per arm, SM clock before / after
                        each arm.  Arms 512, 1024, 1536 hold one size; alt_1504_1536 changes size (and the shared workspace's owner)
                        every step; 512_again repeats the first arm last
  owner_change_zero_ms_1536  the zeroing of the 1536 plan's workspace prefix on a change of owner, CUDA events over 50 memsets
  run_*                 a K-step multi-scale run at imgsz 1024 fed by synthetic uint8 det batches: mean step time and det img/s after
                        every size has been seen once, the first step at each size (plan creation + in-order warm-up), peak memory allocated
                        through torch, and device memory in use (driver) before the run and with all 34 plans alive
Writes nothing to disk.
"""
import argparse
import gc
import json
import os
import random
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402

from tools.bench_augment import gpu_state  # noqa: E402

B = 4
HYP = dict(lr0=0.01, momentum=0.937, weight_decay=5e-4, box=0.05, cls=0.5, cls_pw=1.0, obj=1.0, obj_pw=1.0, anchor_t=4.0, fl_gamma=0.0)


def _trainer(shared):
    from multiyolov5_b200.models.yolo import Model
    from multiyolov5_b200.train import MultiScale, Trainer, scale_hyp
    from oracle import synth
    yml = "yolov5s_city_seg.yaml"
    cfg = synth.load_cfg(yml)
    model = Model(yml)
    model.load_state_dict(synth.synth_state_dict(synth.load_manifest("s_psp"), cfg, seed=1, gain=1.0))
    model.cuda().train()
    tr = Trainer(model, scale_hyp(HYP, nl=3, nc=cfg["nc"], imgsz=1024, total_batch_size=B), batch_size=B, init_scale=2.0 ** 10,
                 multi_scale=MultiScale(1024) if shared else None)
    return tr, cfg["nc"]


def _targets(nc, seed):
    rs = np.random.RandomState(seed)
    t = np.zeros((40, 6), np.float32)
    t[:, 0] = rs.randint(0, B, 40); t[:, 1] = rs.randint(0, nc, 40)
    t[:, 2:4] = rs.uniform(0.1, 0.9, (40, 2)); t[:, 4:6] = rs.uniform(0.02, 0.3, (40, 2))
    return torch.from_numpy(t).cuda()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_multiscale needs a CUDA device")
    steps = max(args.steps, 200)
    from multiyolov5_b200.train import resize_bilinear
    rec = {"gpu": gpu_state(), "batch": B, "imgsz": 1024}
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    g = torch.Generator(device="cuda").manual_seed(0)
    x8 = torch.randint(0, 256, (B, 3, 1024, 1024), dtype=torch.uint8, device="cuda", generator=g)

    def timed(fn):
        for _ in range(args.warmup):
            fn()
        torch.cuda.synchronize()
        ev0.record()
        for _ in range(steps):
            fn()
        ev1.record()
        torch.cuda.synchronize()
        return ev0.elapsed_time(ev1) * 1e3 / steps

    for s in (512, 1056, 1536):
        rec[f"rescale_us_{s}"] = timed(lambda: resize_bilinear(x8, (s, s), torch.float16))
        rec[f"interpolate_us_{s}"] = timed(lambda: F.interpolate(x8.float() / 255.0, size=[s, s], mode="bilinear", align_corners=False))

    # ---- one step through the shared workspace vs a private plan, the two trainers alternating step by step.  Each arm holds one size
    # (the shared workspace keeps its owner: no zeroing inside the timed steps) except `alt`, which changes size every step (the shared
    # workspace changes owner every step and zeroes the new owner's prefix).  512 runs first and again last; the SM clock is read around
    # every arm.
    seg = torch.rand((B, 3, 512, 1024), device="cuda", generator=g)
    segt = torch.randint(-1, 19, (B, 512, 1024), device="cuda", generator=g)
    trs = {"shared": _trainer(True), "private": _trainer(False)}
    n = max(steps // 10, 10)
    arms = []
    for name, sizes in (("512", [512]), ("1024", [1024]), ("1536", [1536]), ("alt_1504_1536", [1504, 1536]), ("512_again", [512])):
        batches = [resize_bilinear(x8, (s, s), torch.float16) for s in sizes]
        times = {k: [] for k in trs}
        clock_before = gpu_state().get("sm_mhz")
        for i in range(n + 3):
            imgs = batches[i % len(batches)]
            for k, (tr, nc) in trs.items():
                t = _targets(nc, i)
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                tr.step(imgs, t, seg, segt)
                torch.cuda.synchronize()
                if i >= 3:
                    times[k].append(time.perf_counter() - t0)
        arm = {"arm": name, "sm_mhz_before": clock_before, "sm_mhz_after": gpu_state().get("sm_mhz")}
        for k, v in times.items():
            arm[f"{k}_ms_median"] = float(np.median(v) * 1e3)
            arm[f"{k}_ms_min"] = float(np.min(v) * 1e3)
        arms.append(arm)
    rec["step_arms"] = arms
    # the zeroing of a change of owner on its own: the 1536 plan's workspace prefix, CUDA events over 50 memsets
    eng = trs["shared"][0].model.engine()
    arena = eng._arenas[0]
    wb = eng.plans[("train", B, 1536, 1536)].pb.workspace_bytes
    torch.cuda.synchronize()
    ev0.record()
    for _ in range(50):
        arena.ws[:wb].zero_()
    ev1.record()
    torch.cuda.synchronize()
    rec["owner_change_zero_ms_1536"] = ev0.elapsed_time(ev1) / 50
    rec["owner_change_zero_bytes_1536"] = int(wb)
    del trs, eng, arena
    gc.collect()
    torch.cuda.empty_cache()

    # ---- a multi-scale run (device memory in use is read through the driver: it includes what the plans allocate themselves)
    torch.cuda.reset_peak_memory_stats()
    free, total = torch.cuda.mem_get_info()
    rec["run_device_used_before_gb"] = (total - free) / 1e9
    tr, nc = _trainer(True)
    ms = tr.multi_scale
    draws = random.Random(0)
    first_use, seen, run = {}, set(), []
    for i in range(steps):
        imgs = ms(x8, torch.float16, rng=draws)
        hw = tuple(imgs.shape[2:])
        t = _targets(nc, i)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        tr.step(imgs, t, seg, segt)
        torch.cuda.synchronize()
        dt = time.perf_counter() - t0
        if hw not in seen:
            seen.add(hw)
            first_use[hw[0]] = dt * 1e3
        else:
            run.append(dt)
    rec["run_steps"] = steps
    rec["run_sizes_seen"] = len(seen)
    rec["run_step_ms_mean"] = float(np.mean(run) * 1e3)
    rec["run_img_per_s"] = float(B / np.mean(run))
    rec["run_first_use_ms"] = {str(k): round(v, 1) for k, v in sorted(first_use.items())}
    rec["run_peak_allocated_gb"] = torch.cuda.max_memory_allocated() / 1e9
    free, total = torch.cuda.mem_get_info()
    rec["run_device_used_gb"] = (total - free) / 1e9                   # 33 det plans + the seg plan alive
    rec["run_det_plans"] = sum(1 for key in tr.model.engine().plans if key[0] == "train" and len(key) == 4)
    rec["gpu_after"] = gpu_state()
    print(json.dumps(rec), flush=True)


if __name__ == "__main__":
    main()
