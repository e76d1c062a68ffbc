#!/usr/bin/env python
"""Benchmark of the optimiser step: `myolo_adam_step` (the reference's --adam) next to `myolo_sgd_step` and torch's own Adam.

    python tools/bench_optim.py [--steps K] [--warmup W]

Prints ONE JSON line with the card's name, power limit and clocks read next to the measurement:
  kernels.<cfg>           at the flat buffer size of s/PSP and m/Lab (every parameter, 16-byte aligned, as the Trainer lays them out):
                          myolo_adam_step and myolo_sgd_step alone, CUDA events over K launches; bytes moved per launch (Adam: p, g,
                          exp_avg, exp_avg_sq read and written + 1 group byte = 33 B per element; SGD: p, g, momentum = 25 B) over the time,
                          and the share of the data sheet's 3.35 TB/s (H100 SXM, 700 W) that this is
  kernels.<cfg>.torch_adam_us
                          torch.optim.Adam (default foreach implementation) behind torch.amp.GradScaler over per-parameter tensors of the
                          same model: scaler.step (unscale + inf check + host sync + Adam) + scaler.update + zero_grad, CUDA events over K
  step                    Trainer.step (s/PSP, 4 det + 4 seg images of 512 x 1024) with optimizer="sgd" and "adam", two trainers
                          alternating step by step, median and min over K/5 steps each
Synthetic weights, images and targets; writes nothing to disk.
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

from tools.bench_augment import gpu_state  # noqa: E402

HBM_TBS = 3.35
HYP = dict(lr0=0.01, momentum=0.937, weight_decay=5e-4, box=0.05, cls=0.5, cls_pw=1.0, obj=1.0, obj_pw=1.0, anchor_t=4.0, fl_gamma=0.0)
CFGS = {"s_psp": "yolov5s_city_seg.yaml", "m_lab": "yolov5m_city_seg_lab.yaml"}


def _events(fn, steps, warmup):
    for _ in range(warmup):
        fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(steps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1e3 / steps                                    # us per call


def bench_kernels(yml, steps, warmup):
    from multiyolov5_b200 import _lib
    from multiyolov5_b200.engine import flat_offsets
    from multiyolov5_b200.models.yolo import Model
    from multiyolov5_b200.train import parameter_groups
    model = Model(yml)
    params = [p for p in model.parameters() if p.requires_grad]
    offsets, n = flat_offsets(params)
    grp = parameter_groups(model)
    group = torch.ones(n, dtype=torch.uint8)
    for p, o in zip(params, offsets):
        group[o:o + p.numel()] = grp[id(p)]
    group = group.cuda()
    gen = torch.Generator(device="cuda").manual_seed(0)
    p, g = torch.randn(n, device="cuda", generator=gen), torch.randn(n, device="cuda", generator=gen)
    m, v = torch.zeros(n, device="cuda"), torch.zeros(n, device="cuda")
    steps_dev = torch.zeros((), dtype=torch.int32, device="cuda")
    inv = torch.full((), 1.0 / 1024, device="cuda")
    found = torch.zeros(1, dtype=torch.int32, device="cuda")
    L, sp = _lib.lib(), _lib.stream_ptr()
    lr_d, lr_f, wd = (C.c_double * 3)(0.01, 0.01, 0.01), (C.c_float * 3)(0.01, 0.01, 0.01), (C.c_float * 3)(0.0, 5e-4, 0.0)

    def adam():
        _lib.check(L.myolo_adam_step(_lib.ptr(p), _lib.ptr(g), _lib.ptr(m), _lib.ptr(v), _lib.ptr(group), n, lr_d, wd, 3, 0.937, 0.999, 1e-8,
                                     _lib.ptr(steps_dev), _lib.ptr(inv), _lib.ptr(found), 1, sp))

    def sgd():
        _lib.check(L.myolo_sgd_step(_lib.ptr(p), _lib.ptr(g), _lib.ptr(m), _lib.ptr(group), n, lr_f, wd, 3, 0.937, 1, _lib.ptr(inv),
                                    _lib.ptr(found), 1, sp))

    rec = {"n": n, "tensors": len(params)}
    for name, fn, bpe in (("adam", adam, 33), ("sgd", sgd, 25)):
        us = _events(fn, steps, warmup)
        tbs = n * bpe / (us * 1e-6) / 1e12
        rec[name] = {"us": us, "bytes": n * bpe, "tb_per_s": tbs, "share_of_3_35_tbs": tbs / HBM_TBS}
    rec["adam"]["floor_us_at_3_35_tbs"] = n * 33 / (HBM_TBS * 1e12) * 1e6

    # torch's Adam + GradScaler over per-parameter tensors of the same shapes and groups
    from multiyolov5_b200.train import reference_param_groups
    tp = [[torch.randn(q.shape, device="cuda", generator=gen).requires_grad_(True) for q in pg] for pg in reference_param_groups(model)]
    opt = torch.optim.Adam([{"params": tp[0]}], lr=0.01, betas=(0.937, 0.999))
    opt.add_param_group({"params": tp[1], "weight_decay": 5e-4})
    opt.add_param_group({"params": tp[2]})
    for q in (q for pg in tp for q in pg):
        q.grad = torch.randn(q.shape, device="cuda", generator=gen)
    scaler = torch.amp.GradScaler("cuda", init_scale=1024.0)
    scaler.scale(torch.ones((), device="cuda"))

    def torch_adam():
        scaler.step(opt)
        scaler.update()
        opt.zero_grad(set_to_none=False)

    rec["torch_adam_us"] = _events(torch_adam, steps, warmup)
    return rec


def _trainer(optimizer):
    from multiyolov5_b200.models.yolo import Model
    from multiyolov5_b200.train import Trainer, scale_hyp
    from oracle import synth
    yml = CFGS["s_psp"]
    cfg = synth.load_cfg(yml)
    model = Model(yml)
    model.load_state_dict(synth.synth_state_dict(synth.load_manifest("s_psp"), cfg, seed=1, gain=1.0))
    model.cuda().train()
    return Trainer(model, scale_hyp(HYP, nl=3, nc=cfg["nc"], imgsz=1024, total_batch_size=4), batch_size=4, init_scale=2.0 ** 10,
                   optimizer=optimizer), cfg["nc"]


def bench_steps(steps, warmup):
    from oracle import synth
    B, H, W = 4, 512, 1024
    trs = {}
    for name in ("sgd", "adam"):
        trs[name], nc = _trainer(name)
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
    rec = {"B_det": B, "B_seg": B, "H": H, "W": W, "steps_per_arm": n, "sm_mhz_before": clock_before, "sm_mhz_after": gpu_state().get("sm_mhz")}
    for k, v in times.items():
        rec[f"{k}_ms_median"] = float(np.median(v) * 1e3)
        rec[f"{k}_ms_min"] = float(np.min(v) * 1e3)
    rec["adam_extra_memory_mb"] = trs["adam"].flat.exp_avg_sq.numel() * 4 / 1e6
    return rec


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=10)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_optim.py measures on the GPU; no CUDA device is visible")
    rec = {"gpu": gpu_state(), "kernels": {}}
    for cfg, yml in CFGS.items():
        rec["kernels"][cfg] = bench_kernels(yml, args.steps, args.warmup)
    rec["step"] = bench_steps(args.steps, args.warmup)
    rec["gpu_after"] = gpu_state()
    print(json.dumps(rec), flush=True)


if __name__ == "__main__":
    main()
