#!/usr/bin/env python
"""Benchmark of what --evolve's anchor counts cost on the device (s/PSP, 4 images of 512 x 1024, synthetic weights and targets).

    python tools/bench_evolve.py [--iters N]

Prints ONE JSON line with the card's name, power limit and clocks read in the same run:
  det_loss_ms     the detection loss forward + backward at na = 3, 4 and 10 (80 targets): the fused loss (myolo_det_loss, four launches)
                  and the torch formulation replayed as one CUDA graph (what the Trainer runs for hyps the fused loss does not take, such
                  as cls_pw != 1), CUDA events over N calls, the two alternated call by call within one process (median and min per call)
  step_ms         Trainer.step (det + seg pass, SGD) at na = 3 and 10, host clock around N steps ending in a synchronise (per step)
  generation_ms   the fixed cost of one generation before its training iterations, on a host clock ending in synchronises: Model build
                  and upload, check_anchors on placeholder anchors (k-means and 1000 generations), Trainer construction, and the first
                  step (train plans, arenas, weight packs, graph capture) less a steady step
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

CFG = "yolov5s_city_seg.yaml"
B, H, W = 4, 512, 1024
HYP = dict(lr0=0.0015, lrf=0.2, momentum=0.937, weight_decay=5e-4, warmup_epochs=3.0, warmup_momentum=0.8, warmup_bias_lr=0.1, box=0.05,
           cls=0.5, cls_pw=1.0, obj=1.0, obj_pw=1.0, anchor_t=4.0, fl_gamma=0.0)


def model_n(n):
    from multiyolov5_b200.models.yolo import Model
    from oracle import restate_evolve as rev
    from oracle import synth
    cfg = dict(synth.load_cfg(CFG), anchors=rev.anchor_table(n))
    model = Model(CFG, anchors=n)
    manifest = [[k, list(v.shape), str(v.dtype).replace("torch.", "")] for k, v in model.state_dict().items()]
    model.load_state_dict(synth.synth_state_dict(manifest, cfg, seed=1, gain=1.0))
    return model.cuda().train()


def targets(nt=80, seed=3):
    rs = np.random.RandomState(seed)
    t = np.zeros((nt, 6), np.float32)
    t[:, 0] = np.repeat(np.arange(B), nt // B); t[:, 1] = rs.randint(0, 10, nt)
    t[:, 2:4] = rs.uniform(0.1, 0.9, (nt, 2)); t[:, 4:6] = rs.uniform(0.02, 0.22, (nt, 2))
    return torch.from_numpy(t).cuda()


def trainer(model):
    from multiyolov5_b200.train import Trainer, scale_hyp
    return Trainer(model, scale_hyp(HYP, nl=3, nc=10, imgsz=W, total_batch_size=B), batch_size=B, init_scale=2.0 ** 10)


def det_loss(na, iters):
    """fused and graphed-torch loss, alternated call by call"""
    model = model_n(na)
    tr = trainer(model)
    det = model.model[-1]
    shapes = [(B, na, H // int(s), W // int(s), det.no) for s in det.stride.tolist()]
    gen = torch.Generator(device="cuda").manual_seed(5)
    p = [torch.randn(sh, device="cuda", generator=gen) for sh in shapes]
    tg = targets()
    st = tr._det_graph(shapes, 128, p[0].device)
    for q, s in zip(p, st.p):
        s.data.copy_(q)
    st.t.zero_()
    st.t[:tg.shape[0]].copy_(tg)
    fused = lambda: tr._fused_det(p, tg, mult=tr.det_mult(), scale=tr.scale)  # noqa: E731
    graph = st.graph.replay
    ts = {"fused": [], "torch_graph": []}
    for _ in range(5):
        fused(); graph()
    for _ in range(iters):
        for name, fn in (("fused", fused), ("torch_graph", graph)):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            fn()
            e1.record()
            torch.cuda.synchronize()
            ts[name].append(e0.elapsed_time(e1))
    return {k: {"median": round(float(np.median(v)), 4), "min": round(float(np.min(v)), 4)} for k, v in ts.items()}


def batches(n=4):
    from oracle import synth
    out = []
    for k in range(n):
        g = torch.Generator().manual_seed(k)
        out.append((synth.synth_image(B, H, W, seed=10 * k + 1).cuda(), targets(seed=k), synth.synth_image(B, H, W, seed=10 * k + 2).cuda(),
                    torch.randint(-1, 19, (B, H, W), generator=g).cuda()))
    return out


def step_time(tr, data, iters):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for i in range(iters):
        tr.step(*data[i % len(data)])
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3 / iters


def generation(na, data, iters):
    """the fixed cost of one generation, and the steady Trainer.step after it"""
    from multiyolov5_b200.models.yolo import Model
    from multiyolov5_b200.utils.autoanchor import check_anchors
    from multiyolov5_b200.utils.datasets import DeviceImageCache
    from oracle import restate_autoanchor as ra
    shapes0, labels = ra.synth_dataset(200, 40, 61, [(12, 30), (25, 60), (40, 25), (90, 55), (200, 120), (8, 8)], spread=0.35)
    cache = DeviceImageCache([np.zeros((h0, w0, 3), np.uint8) for h0, w0 in shapes0], 64, labels=labels)
    t = {}
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    model = Model(CFG, nc=10, anchors=na).cuda().train()
    torch.cuda.synchronize()
    t["model_ms"] = (time.perf_counter() - t0) * 1e3
    np.random.seed(0)
    t0 = time.perf_counter()
    with contextlib.redirect_stdout(io.StringIO()):
        check_anchors(cache, model, thr=4.0, imgsz=W)
    torch.cuda.synchronize()
    t["check_anchors_ms"] = (time.perf_counter() - t0) * 1e3
    t0 = time.perf_counter()
    tr = trainer(model)
    torch.cuda.synchronize()
    t["trainer_ms"] = (time.perf_counter() - t0) * 1e3
    first = step_time(tr, data, 1)
    steady = step_time(tr, data, iters)
    t["first_step_less_steady_ms"] = first - steady
    t["total_ms"] = t["model_ms"] + t["check_anchors_ms"] + t["trainer_ms"] + t["first_step_less_steady_ms"]
    return {k: round(v, 2) for k, v in t.items()}, steady


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_evolve needs a GPU"
    rec = {"bench": "evolve", "gpu": gpu_state(), "model": CFG, "batch": [B, 3, H, W], "targets": 80}
    rec["det_loss_ms"] = {}
    for na in (3, 4, 10):
        rec["det_loss_ms"][f"na{na}"] = det_loss(na, args.iters)
        print(f"det loss na={na}: {json.dumps(rec['det_loss_ms'][f'na{na}'])}", file=sys.stderr, flush=True)
    data = batches()
    rec["generation_ms"], rec["step_ms"] = {}, {}
    for na in (3, 10):
        gen_ms, steady = generation(na, data, args.iters)
        rec["generation_ms"][f"na{na}"] = gen_ms
        rec["step_ms"][f"na{na}"] = round(steady, 3)
        print(f"na={na}: step {steady:.2f} ms, generation {json.dumps(gen_ms)}", file=sys.stderr, flush=True)
    rec["gpu_after"] = gpu_state()
    print(json.dumps(rec))


if __name__ == "__main__":
    main()
