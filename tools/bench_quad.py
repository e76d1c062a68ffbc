#!/usr/bin/env python
"""Benchmark of `--quad` training (utils.datasets.collate_quad, csrc/augment.cu myolo_collate_quad, Trainer(quad=True)).

    python tools/bench_quad.py [--steps K] [--warmup W]

Prints ONE JSON line with the card's name, power limit and clocks read next to the measurement:
  kernel            myolo_collate_quad alone on 16 x 3 x 1024^2 uint8 -> 4 x 3 x 2048^2, for uint8 / fp16 / fp32 outputs and three flag
                    patterns (all tiles, all upsamples, alternating), CUDA events over K launches; the HBM floor is the bytes the pattern
                    must read (3 B H W for tiles, a quarter of it for upsamples) plus the bytes written, at the data sheet's 3.35 TB/s
  collate_quad_ms   collate_quad(imgs, targets) end to end (draws, kernel, label selection with its one synchronisation), alternating flags
  host_collate_fn4  collate_fn4's operations on the same batch on the CPU (torch.cat of the tiles, F.interpolate + uint8 cast of the
                    upsampled items, torch.stack), on one thread (a DataLoader worker's) and on torch's default thread count
  step              Trainer.step (s/PSP, batch_size 8 at imgsz 1024, seg 8 x 512 x 1024): quad (2 x 2048^2 det images, loss x 4) against
                    no quad (8 x 1024^2 det images), two trainers alternating step by step, median and min over K/10 steps each
The images are random uint8 with 40 targets per batch.  Writes nothing to disk.
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
import torch.nn.functional as F  # noqa: E402

from tools.bench_augment import gpu_state  # noqa: E402
from tools.bench_rect import HYP, _model  # noqa: E402

HBM_BYTES_PER_S = 3.35e12        # H100 SXM data sheet


class _Cycle:
    """an rng whose random() cycles through the given values (one per quad)"""

    def __init__(self, values):
        self.values, self.k = list(values), 0

    def random(self):
        v = self.values[self.k % len(self.values)]
        self.k += 1
        return v


def _targets(B, nc, seed):
    rs = np.random.RandomState(seed)
    t = np.zeros((40, 6), np.float32)
    t[:, 0] = np.sort(rs.randint(0, B, 40)); t[:, 1] = rs.randint(0, nc, 40)
    t[:, 2:4] = rs.uniform(0.1, 0.9, (40, 2)); t[:, 4:6] = rs.uniform(0.02, 0.3, (40, 2))
    return torch.from_numpy(t).cuda()


def _host_collate(imgs, tile):
    """collate_fn4's pixel operations on CPU tensors (the labels are a few hundred bytes in both arms)"""
    out = []
    for q, t in enumerate(tile):
        i = 4 * q
        if not t:
            out.append(F.interpolate(imgs[i].float()[None], scale_factor=2., mode="bilinear", align_corners=False)[0].type(imgs[i].type()))
        else:
            out.append(torch.cat((torch.cat((imgs[i], imgs[i + 1]), 1), torch.cat((imgs[i + 2], imgs[i + 3]), 1)), 2))
    return torch.stack(out, 0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=10)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_quad needs a CUDA device")
    import ctypes as C

    from multiyolov5_b200 import _lib
    from multiyolov5_b200.train import Trainer, scale_hyp
    from multiyolov5_b200.utils.datasets import collate_quad
    steps = args.steps
    rec = {"gpu": gpu_state()}
    B, H, W = 16, 1024, 1024
    n = B // 4
    g = torch.Generator(device="cuda").manual_seed(0)
    imgs = torch.randint(0, 256, (B, 3, H, W), dtype=torch.uint8, device="cuda", generator=g)
    L, sp = _lib.lib(), _lib.stream_ptr()
    patterns = {"tile": [1] * n, "upsample": [0] * n, "alternating": [0, 1] * (n // 2)}
    rec["kernel"] = {"B": B, "in": [B, 3, H, W], "out": [n, 3, 2 * H, 2 * W]}
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for dtype in (torch.uint8, torch.float16, torch.float32):
        out = torch.empty((n, 3, 2 * H, 2 * W), dtype=dtype, device="cuda")
        es = out.element_size()
        for pname, tile in patterns.items():
            flags = (C.c_uint8 * n)(*tile)
            args_ = (_lib.ptr(imgs), B, H, W, flags, _lib.ptr(out), _lib.torch_dtype_code(dtype), sp)
            for _ in range(args.warmup):
                _lib.check(L.myolo_collate_quad(*args_))
            e0.record()
            for _ in range(steps):
                _lib.check(L.myolo_collate_quad(*args_))
            e1.record()
            torch.cuda.synchronize()
            us = e0.elapsed_time(e1) * 1e3 / steps
            read = sum(3 * (4 if t else 1) * H * W for t in tile)
            written = 12 * n * H * W * es
            floor_us = (read + written) / HBM_BYTES_PER_S * 1e6
            rec["kernel"][f"{str(dtype)[6:]}_{pname}"] = {"us": us, "bytes_read": read, "bytes_written": written, "floor_us": floor_us,
                                                          "floor_fraction": floor_us / us, "gb_per_s": (read + written) / us / 1e3}
        del out
    # ---- collate_quad end to end, alternating flags
    targets = _targets(B, 10, 0)
    rng = _Cycle([0.2, 0.7])
    for _ in range(args.warmup):
        collate_quad(imgs, targets, rng=rng)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(steps):
        collate_quad(imgs, targets, rng=rng)
    torch.cuda.synchronize()
    rec["collate_quad_ms"] = (time.perf_counter() - t0) * 1e3 / steps
    # ---- the reference's collate on the CPU
    cpu = imgs.cpu()
    tile = patterns["alternating"]
    prev = torch.get_num_threads()
    host = {"pattern": "alternating"}
    for label, threads in (("one_thread", 1), ("default_threads", prev)):
        torch.set_num_threads(threads)
        try:
            _host_collate(cpu, tile)
            k = 5
            t0 = time.perf_counter()
            for _ in range(k):
                _host_collate(cpu, tile)
            host[f"{label}_ms"] = (time.perf_counter() - t0) * 1e3 / k
            host[f"{label}_threads"] = threads
        finally:
            torch.set_num_threads(prev)
    rec["host_collate_fn4"] = host
    del cpu, imgs
    torch.cuda.empty_cache()
    # ---- Trainer.step with and without quad, alternating
    SB, s = 8, 1024
    trs = {}
    for quad in (True, False):
        model, nc = _model()
        trs[quad] = Trainer(model, scale_hyp(HYP, nl=3, nc=nc, imgsz=s, total_batch_size=SB), batch_size=SB, init_scale=2.0 ** 10,
                            quad=quad)
    items = torch.randint(0, 256, (SB, 3, s, s), dtype=torch.uint8, device="cuda", generator=g)
    seg = torch.rand((SB, 3, 512, 1024), device="cuda", generator=g)
    segt = torch.randint(-1, 19, (SB, 512, 1024), device="cuda", generator=g)
    nsteps = max(steps // 10, 10)
    times = {True: [], False: []}
    clock_before = gpu_state().get("sm_mhz")
    rng = _Cycle([0.2, 0.7])
    for i in range(nsteps + 3):
        for quad, tr in trs.items():
            t = _targets(SB, nc, i)
            if quad:
                det, t = collate_quad(items, t, rng=rng, out_dtype=torch.float16)
            else:
                det = items.half() / 255.0
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            tr.step(det, t, seg, segt)
            torch.cuda.synchronize()
            if i >= 3:
                times[quad].append(time.perf_counter() - t0)
    rec["step"] = {"batch_size": SB, "det_quad": [SB // 4, 3, 2 * s, 2 * s], "det_plain": [SB, 3, s, s], "seg": [SB, 3, 512, 1024],
                   "steps_per_arm": nsteps, "sm_mhz_before": clock_before, "sm_mhz_after": gpu_state().get("sm_mhz")}
    for quad, v in times.items():
        k = "quad" if quad else "plain"
        rec["step"][f"{k}_ms_median"] = float(np.median(v) * 1e3)
        rec["step"][f"{k}_ms_min"] = float(np.min(v) * 1e3)
    rec["gpu_after"] = gpu_state()
    print(json.dumps(rec), flush=True)


if __name__ == "__main__":
    main()
