#!/usr/bin/env python
"""Benchmark of synchronised BatchNorm in the train plans (the reference's --sync-bn, myolo_plan_set_bn_sync).

    python tools/bench_sync_bn.py [--steps K] [--warmup W]                    # one GPU
    torchrun --nproc-per-node N tools/bench_sync_bn.py [--steps K] [--warmup W]  # N GPUs

Prints ONE JSON line (rank 0) with the card's name, power limit and clocks read next to the measurement:
  one_gpu   s/PSP train forward + backward of 4 images at 512 x 1024 with fixed cotangents: the plain plan (CUDA-graph replay) and the
            same plan synchronised through a one-rank NCCL process group (in-order launches plus one all-gather per BN layer in the forward
            and one all-reduce per BN layer in the backward).  CUDA events over K iterations each, the two arms alternating in blocks.
  trainer   (torchrun, N > 1) Trainer.step of 4 det + 4 seg images of 512 x 1024 per GPU with the plain model and with
            torch.nn.SyncBatchNorm.convert_sync_batchnorm(model), median and min over K steps each, host clock around a synchronise.
  exchanges collectives and bytes per train forward + full backward, counted from the plan: each BN layer all-gathers one record of
            (4 + 2C) fp32 words per rank and all-reduces 2C fp32 words.
Synthetic weights, images and targets.  The one-rank process group uses a file store in a temporary directory.
"""
import argparse
import json
import os
import sys
import tempfile
import time
from datetime import timedelta

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402

from tools.bench_augment import gpu_state  # noqa: E402
from tools.bench_optim import CFGS, HYP  # noqa: E402


def _model(convert=False):
    from multiyolov5_b200.models.yolo import Model
    from oracle import synth
    cfg = synth.load_cfg(CFGS["s_psp"])
    model = Model(CFGS["s_psp"])
    model.load_state_dict(synth.synth_state_dict(synth.load_manifest("s_psp"), cfg, seed=1, gain=1.0))
    if convert:
        model = torch.nn.SyncBatchNorm.convert_sync_batchnorm(model)
    return model.cuda().train(), cfg


def exchanges(plan, world):
    from multiyolov5_b200 import _lib
    cs = [o.in_.c for o in plan.pb.ops if o.kind == _lib.OP_BN_ACT]
    fwd = sum(world * (4 + 2 * c) * 4 for c in cs)
    bwd = sum(2 * c * 4 for c in cs)
    return {"bn_layers": len(cs), "allgathers": len(cs), "allgather_bytes_received": fwd, "allreduces": len(cs), "allreduce_bytes": bwd}


def one_gpu(steps, warmup):
    from multiyolov5_b200.parallel import nccl_comm_ptr
    B, H, W = 4, 512, 1024
    from oracle import synth
    x = synth.synth_image(B, H, W, seed=5).cuda()
    gen = torch.Generator().manual_seed(11)
    Rs = [(torch.randn((B, 3, H // s, W // s, 15), generator=gen) * 4.0).cuda() for s in (8, 16, 32)]
    S = (torch.randn((B, 19, H, W), generator=gen) * 0.05).cuda()
    arms = {}
    for name in ("plain", "sync_nccl_1rank"):
        model, _ = _model()
        eng = model.engine()
        p = eng.train_plan_for(B, H, W)
        eng.ensure_flat_grads()
        eng.prepare_train_plan(p)
        if name != "plain":
            dist.all_reduce(torch.zeros(1, device="cuda"))
            eng.set_bn_sync(p, comm=nccl_comm_ptr())
        arms[name] = (model, eng, p)

    def it(arm):
        model, eng, p = arms[arm]
        raws, seg, plan = eng.train_forward(x, want_seg=True)
        eng.train_backward(plan, Rs, S)

    res = {k: [] for k in arms}
    for name in arms:
        for _ in range(warmup):
            it(name)
    torch.cuda.synchronize()
    block = max(1, steps // 5)
    for _ in range(5):
        for name in arms:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(block):
                it(name)
            e1.record()
            e1.synchronize()
            res[name].append(e0.elapsed_time(e1) / block)
    out = {k: {"ms_median": float(np.median(v)), "ms_min": float(np.min(v)), "blocks": len(v), "iters_per_block": block} for k, v in res.items()}
    out["exchanges_per_forward_backward"] = exchanges(arms["sync_nccl_1rank"][2], 1)
    return out


def trainer(steps, warmup, rank, world):
    from multiyolov5_b200.train import Trainer, scale_hyp
    from oracle import synth
    B, H, W = 4, 512, 1024
    rs = np.random.RandomState(rank)
    imgs = synth.synth_image(B, H, W, seed=1 + rank).cuda()
    segimgs = synth.synth_image(B, H, W, seed=100 + rank).cuda()
    t = np.zeros((40, 6), np.float32)
    t[:, 0] = rs.randint(0, B, 40); t[:, 1] = rs.randint(0, 10, 40)
    t[:, 2:4] = rs.uniform(0.1, 0.9, (40, 2)); t[:, 4:6] = rs.uniform(0.05, 0.3, (40, 2))
    targets = torch.from_numpy(t).cuda()
    mask = torch.from_numpy(rs.randint(-1, 19, (B, H, W)).astype(np.int64)).cuda()
    out = {}
    for name, convert in (("plain", False), ("sync_bn", True)):
        model, cfg = _model(convert)
        tr = Trainer(model, scale_hyp(HYP, nl=3, nc=cfg["nc"], imgsz=W, total_batch_size=B * world), batch_size=B, world_size=world,
                     rank=rank, init_scale=2.0 ** 10)
        assert tr.sync_bn == convert
        for _ in range(warmup):
            tr.step(imgs, targets, segimgs, mask)
        ts = []
        for _ in range(steps):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            tr.step(imgs, targets, segimgs, mask)
            torch.cuda.synchronize()
            ts.append((time.perf_counter() - t0) * 1e3)
        out[name] = {"ms_median": float(np.median(ts)), "ms_min": float(np.min(ts)), "steps": steps}
        if convert:
            plan = model.engine().last_plan
            out["exchanges_per_forward_backward"] = exchanges(plan, world)
        del tr, model
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_sync_bn needs a CUDA device")
    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    torch.cuda.set_device(int(os.environ.get("LOCAL_RANK", "0")))
    rec = {"gpu": gpu_state(torch.cuda.current_device()), "world_size": world}
    if world > 1:
        dist.init_process_group("nccl", timeout=timedelta(seconds=300))
        rec["trainer"] = trainer(a.steps, a.warmup, rank, world)
    else:
        with tempfile.TemporaryDirectory() as tmp:
            dist.init_process_group("nccl", init_method="file://" + os.path.join(tmp, "store"), rank=0, world_size=1,
                                    timeout=timedelta(seconds=300))
            try:
                rec["one_gpu"] = one_gpu(a.steps, a.warmup)
            finally:
                dist.destroy_process_group()
    if world > 1:
        dist.destroy_process_group()
    if rank == 0:
        print(json.dumps(rec))


if __name__ == "__main__":
    main()
