#!/usr/bin/env python
"""Benchmark of the EMA update (`myolo_ema_update` behind utils.torch_utils.ModelEMA, the reference's `ema.update(model)`).

    python tools/bench_ema.py [--steps K] [--warmup W]

Prints ONE JSON line with the card's name, power limit and clocks read next to the measurement:
  kernels.<cfg>.<fp32|fp16>  the launch alone over every floating-point entry of s/PSP and m/Lab, with an fp32 EMA and with the fp16 EMA
                             that the reference's validation leaves (test.py:124): CUDA events over K launches; bytes per launch (fp32
                             EMA: v read + written, m read = 12 B per element; fp16 EMA: 8 B) and the floor at the data sheet's 3.35 TB/s
                             (H100 SXM, 700 W), which is a floor, not an expectation
  update.<cfg>               wall time of one ModelEMA.update(model) followed by torch.cuda.synchronize(), median and min over K, fp32
                             EMA: this path; the previous CUDA path (two foreach ops over both state_dict()s, torch's rounding); the
                             reference's per-entry loop (utils/torch_utils.py:296-300)
  step                       Trainer.step at accumulate=1 (s/PSP, 4 det + 4 seg images of 512 x 1024) without and with ema=ModelEMA,
                             two trainers alternating step by step, median and min over K/5 steps each
Synthetic weights, images and targets; writes nothing to disk.
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from tools.bench_augment import gpu_state  # noqa: E402
from tools.bench_optim import CFGS, HBM_TBS, HYP, _events  # noqa: E402


def _model(yml, train=True):
    from multiyolov5_b200.models.yolo import Model
    from oracle import synth
    cfg = synth.load_cfg(yml)
    model = Model(yml)
    tag = "s_psp" if yml == CFGS["s_psp"] else "m_lab"
    model.load_state_dict(synth.synth_state_dict(synth.load_manifest(tag), cfg, seed=1, gain=1.0))
    model.cuda()
    model.train(train)
    return model, cfg


def foreach_update(ema, model):
    """the previous CUDA path: both state_dict()s per update and two foreach ops (torch's FMA rounding on the second)"""
    with torch.no_grad():
        ema.updates += 1
        d = ema.decay(ema.updates)
        msd = model.state_dict()
        mine, theirs = [], []
        for k, v in ema.ema.state_dict().items():
            if v.dtype.is_floating_point:
                mine.append(v)
                theirs.append(msd[k].detach())
        torch._foreach_mul_(mine, d)
        torch._foreach_add_(mine, theirs, alpha=1.0 - d)


def reference_update(ema, model):
    """reference utils/torch_utils.py:290-300"""
    with torch.no_grad():
        ema.updates += 1
        d = ema.decay(ema.updates)
        msd = model.state_dict()
        for k, v in ema.ema.state_dict().items():
            if v.dtype.is_floating_point:
                v *= d
                v += (1. - d) * msd[k].detach()


def _wall(fn, steps, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(steps):
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        ts.append(time.perf_counter() - t0)
    return {"ms_median": float(np.median(ts) * 1e3), "ms_min": float(np.min(ts) * 1e3)}


def bench_kernels(yml, steps, warmup):
    from multiyolov5_b200 import _lib
    from multiyolov5_b200.utils.torch_utils import ModelEMA, ema_entries
    model, _ = _model(yml)
    ema = ModelEMA(model)
    ema.updates = 100_000
    L, sp = _lib.lib(), _lib.stream_ptr()
    rec = {}
    for name in ("fp32", "fp16"):
        if name == "fp16":
            ema.ema.half()
        table, n_chunks = ema.table(model)
        n = sum(v.numel() for _, v, _ in ema_entries(ema.ema, model))
        bpe = 12 if name == "fp32" else 8

        def launch():
            _lib.check(L.myolo_ema_update(_lib.ptr(table), n_chunks, 0.9999, sp))

        us = _events(launch, steps, warmup)
        rec[name] = {"us": us, "elements": n, "chunks": n_chunks, "bytes": n * bpe, "tb_per_s": n * bpe / (us * 1e-6) / 1e12,
                     "floor_us_at_3_35_tbs": n * bpe / (HBM_TBS * 1e12) * 1e6}
    rec["entries"] = len(ema_entries(ema.ema, model))
    return rec


def bench_update(yml, steps, warmup):
    from multiyolov5_b200.utils.torch_utils import ModelEMA
    model, _ = _model(yml)
    rec = {}
    for name, fn in (("device", lambda e: e.update(model)), ("foreach", lambda e: foreach_update(e, model)),
                     ("reference_loop", lambda e: reference_update(e, model))):
        ema = ModelEMA(model)
        rec[name] = _wall(lambda: fn(ema), steps, warmup)
    return rec


def _trainer(ema):
    from multiyolov5_b200.train import Trainer, scale_hyp
    from multiyolov5_b200.utils.torch_utils import ModelEMA
    model, cfg = _model(CFGS["s_psp"])
    return Trainer(model, scale_hyp(HYP, nl=3, nc=cfg["nc"], imgsz=1024, total_batch_size=4), batch_size=4, init_scale=2.0 ** 10,
                   ema=ModelEMA(model) if ema else None), cfg["nc"]


def bench_steps(steps, warmup):
    from oracle import synth
    B, H, W = 4, 512, 1024
    trs = {}
    for name in ("no_ema", "ema"):
        trs[name], nc = _trainer(name == "ema")
    rs = np.random.RandomState(0)
    t = np.zeros((40, 6), np.float32)
    t[:, 0] = rs.randint(0, B, 40); t[:, 1] = rs.randint(0, nc, 40)
    t[:, 2:4] = rs.uniform(0.1, 0.9, (40, 2)); t[:, 4:6] = rs.uniform(0.02, 0.3, (40, 2))
    t = torch.from_numpy(t).cuda()
    imgs, seg = synth.synth_image(B, H, W, seed=1).cuda(), synth.synth_image(B, H, W, seed=2).cuda()
    segt = torch.from_numpy(rs.randint(-1, 19, (B, H, W)).astype(np.int64)).cuda()
    for _ in range(warmup):
        for tr in trs.values():
            tr.step(imgs, t, seg, segt)
    torch.cuda.synchronize()
    clock_before = gpu_state().get("sm_mhz")
    times = {k: [] for k in trs}
    n = max(steps // 5, 10)
    for _ in range(n):
        for k, tr in trs.items():
            t0 = time.perf_counter()
            tr.step(imgs, t, seg, segt)
            torch.cuda.synchronize()
            times[k].append(time.perf_counter() - t0)
    rec = {"B_det": B, "B_seg": B, "H": H, "W": W, "accumulate": 1, "steps_per_arm": n, "sm_mhz_before": clock_before,
           "sm_mhz_after": gpu_state().get("sm_mhz")}
    for k, v in times.items():
        rec[f"{k}_ms_median"] = float(np.median(v) * 1e3)
        rec[f"{k}_ms_min"] = float(np.min(v) * 1e3)
    assert trs["ema"].ema.updates == warmup + n
    return rec


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=10)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_ema.py measures on the GPU; no CUDA device is visible")
    rec = {"gpu": gpu_state(), "kernels": {}, "update": {}}
    for cfg, yml in CFGS.items():
        rec["kernels"][cfg] = bench_kernels(yml, args.steps, args.warmup)
        rec["update"][cfg] = bench_update(yml, max(args.steps // 4, 10), args.warmup)
    rec["step"] = bench_steps(args.steps, args.warmup)
    rec["gpu_after"] = gpu_state()
    print(json.dumps(rec), flush=True)


if __name__ == "__main__":
    main()
