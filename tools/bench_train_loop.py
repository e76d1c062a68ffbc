#!/usr/bin/env python
"""What the epoch loop (train.fit) costs on top of the step: one epoch of N iterations through fit against the same batches through bare
Trainer.step calls, the two alternating, s/PSP with 4 det + 4 seg images of 512 x 1024.

    python tools/bench_train_loop.py [--iters N] [--warmup W] [--rounds R]

Each arm is timed from iteration W to the end of its N iterations, with a device synchronise at both ends; the fit arm's window includes
its log line every `log_interval` (50) iterations and excludes the epoch end (validation and checkpoints are off).  Prints ONE JSON line
with the median ms per iteration of each arm over R rounds and the card's name, power limit and clocks read in the same run.
Synthetic weights, images and targets; writes only under a temporary directory.
"""
import argparse
import json
import os
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from tools.bench_augment import gpu_state  # noqa: E402

HYP = dict(lr0=0.01, lrf=0.2, momentum=0.937, weight_decay=5e-4, warmup_epochs=3.0, warmup_momentum=0.8, warmup_bias_lr=0.1, box=0.05,
           cls=0.5, cls_pw=1.0, obj=1.0, obj_pw=1.0, anchor_t=4.0, fl_gamma=0.0)
B, H, W = 4, 512, 1024


def _model():
    from multiyolov5_b200.models.yolo import Model
    from oracle import synth
    cfg = synth.load_cfg("yolov5s_city_seg.yaml")
    model = Model("yolov5s_city_seg.yaml")
    model.load_state_dict(synth.synth_state_dict(synth.load_manifest("s_psp"), cfg, seed=1, gain=1.0))
    return model.cuda(), cfg


def _batches(nc, n=4):
    from oracle import synth
    rs = np.random.RandomState(0)
    det, seg = [], []
    for k in range(n):
        t = np.zeros((40, 6), np.float32)
        t[:, 0] = rs.randint(0, B, 40); t[:, 1] = rs.randint(0, nc, 40)
        t[:, 2:4] = rs.uniform(0.1, 0.9, (40, 2)); t[:, 4:6] = rs.uniform(0.02, 0.3, (40, 2))
        det.append((synth.synth_image(B, H, W, seed=10 * k + 1).cuda(), torch.from_numpy(t).cuda()))
        seg.append((synth.synth_image(B, H, W, seed=10 * k + 2).cuda(),
                    torch.from_numpy(rs.randint(-1, 19, (B, H, W)).astype(np.int64)).cuda()))
    return det, seg


class _Timed:
    """det_batches of N iterations cycling through `items`, stamping the clock (after a synchronise) at iteration W and at the end"""

    def __init__(self, items, n, w):
        self.items, self.n, self.w, self.t = items, n, w, {}

    def __len__(self):
        return self.n

    def __call__(self, epoch):
        for i in range(self.n):
            if i == self.w:
                torch.cuda.synchronize()
                self.t["start"] = time.perf_counter()
            yield self.items[i % len(self.items)]
        torch.cuda.synchronize()
        self.t["end"] = time.perf_counter()


def fit_arm(det, seg, n, w, tmp):
    import argparse as ap
    from multiyolov5_b200.train import fit
    model, _ = _model()
    opt = ap.Namespace(epochs=1, batch_size=B, img_size=[1024, 1024], linear_lr=False, adam=False, notest=True, nosave=True, evolve=True,
                       multi_scale=False, quad=False, single_cls=False, resume=False, global_rank=-1, world_size=1, label_smoothing=0.0,
                       weights="", cfg="")
    timed = _Timed(det, n, w)
    fit(model, HYP, opt, timed, lambda e: iter([seg[i % len(seg)] for i in range(n)]), save_dir=tmp, init_scale=2.0 ** 10)
    return (timed.t["end"] - timed.t["start"]) / (n - w)


def bare_arm(det, seg, n, w, nc):
    """the same steps by hand: the schedule's accumulate and ni, computed before the timed window"""
    from multiyolov5_b200.train import LRSchedule, Trainer, scale_hyp
    from multiyolov5_b200.utils.torch_utils import ModelEMA
    model, _ = _model()
    tr = Trainer(model, scale_hyp(HYP, nl=3, nc=nc, imgsz=1024, total_batch_size=B), B, accumulate=16, ema=ModelEMA(model),
                 init_scale=2.0 ** 10)
    sched = LRSchedule(HYP, 1, n, B)
    its = [sched.iteration(0, i) for i in range(n)]
    for i, it in enumerate(its):
        if i == w:
            torch.cuda.synchronize()
            t0 = time.perf_counter()
        tr.set_lr(*it.lr)
        tr.set_momentum(it.momentum)
        tr.accumulate = it.accumulate
        tr.step(*det[i % len(det)], *seg[i % len(seg)], ni=it.ni)
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) / (n - w)


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--iters", type=int, default=200)
    p.add_argument("--warmup", type=int, default=20)
    p.add_argument("--rounds", type=int, default=3)
    a = p.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_train_loop.py measures on the GPU; no CUDA device is visible")
    from oracle import synth
    nc = synth.load_cfg("yolov5s_city_seg.yaml")["nc"]
    det, seg = _batches(nc)
    rec = {"gpu": gpu_state(), "B_det": B, "B_seg": B, "H": H, "W": W, "iters": a.iters, "warmup": a.warmup, "rounds": a.rounds}
    fit_t, bare_t = [], []
    with tempfile.TemporaryDirectory() as tmp:
        for _ in range(a.rounds):
            fit_t.append(fit_arm(det, seg, a.iters, a.warmup, tmp))
            bare_t.append(bare_arm(det, seg, a.iters, a.warmup, nc))
    rec.update(fit_ms_per_iter_median=float(np.median(fit_t) * 1e3), bare_ms_per_iter_median=float(np.median(bare_t) * 1e3),
               fit_ms_per_iter=[t * 1e3 for t in fit_t], bare_ms_per_iter=[t * 1e3 for t in bare_t], gpu_after=gpu_state())
    print(json.dumps(rec), flush=True)


if __name__ == "__main__":
    main()
