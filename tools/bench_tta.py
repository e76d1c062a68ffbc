#!/usr/bin/env python
"""Benchmark of test-time augmentation, Model.forward(augment=True), on s/PSP at 16 x 3 x 512 x 1024 fp16 (BASELINE config 2).

    python tools/bench_tta.py [--rounds R] [--iters N]

Every arm is its forward followed by non_max_suppression(0.25, 0.45) and the seg argmax (the fused seg_argmax=True output):
  plain     one forward, augment=False
  tta       augment=True: scale_img kernels, det-only plans for the scaled passes, de-scale / de-flip inside the Detect decodes
  torch     the reference's loop composed in torch: flip / interpolate / pad, three plain forwards, `/= si`, the de-flip and torch.cat
  tta_full  augment=True with full plans (seg head included) for the scaled passes: the A/B of the det-only plans
Every shape is warmed first; the arms alternate within each round, each timed with CUDA events over N iterations; the medians of R
rounds are printed (ms per iteration) in ONE JSON line with the card's name, power limit and clocks.  Also printed: the workspace bytes
of each plan the arms use and their fp16 weight-pack bytes, estimated from the conv shapes (Co and Ci rounded up to 16).
Writes nothing to disk.
"""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from tools.bench_augment import gpu_state  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--batch", type=int, default=16)
    a = ap.parse_args()
    from multiyolov5_b200 import synth
    from multiyolov5_b200.models.yolo import Model
    from multiyolov5_b200.utils.general import non_max_suppression
    from multiyolov5_b200.utils.torch_utils import tta_passes
    from oracle import restate_tta
    assert torch.cuda.is_available(), "bench_tta needs a CUDA device"
    yml = "yolov5s_city_seg.yaml"
    cfg = synth.load_cfg(yml)
    model = Model(yml)
    model.load_state_dict(synth.synth_state_dict(synth.load_manifest("s_psp"), cfg, seed=1))
    model.cuda().eval()
    eng = model.engine()
    B, H, W = a.batch, 512, 1024
    x = synth.synth_image(B, H, W, seed=0).cuda().half()

    def post(z, amax):
        return non_max_suppression(z, 0.25, 0.45), amax

    def plain():
        out = model(x, seg_argmax=True)
        return post(out[0][0], out[2])

    def tta():
        out = model(x, augment=True, seg_argmax=True)
        return post(out[0][0], out[2])

    def tta_full():
        out = eng.forward_augment(x, seg_argmax=True, det_only_scaled=False)
        return post(out[0][0], out[2])

    def torch_composed():
        amax = []

        def z_of(xi):
            out = model(xi, seg_argmax=True)
            if not amax:
                amax.append(out[2])          # pass 0's, the one detect.py keeps
            return out[0][0]
        return post(restate_tta.tta(z_of, x, gs=32), amax[0])

    arms = {"plain": plain, "tta": tta, "torch": torch_composed, "tta_full": tta_full}
    with torch.no_grad():
        for f in arms.values():              # every plan built, warmed and captured
            for _ in range(3):
                f()
        torch.cuda.synchronize()
        times = {k: [] for k in arms}
        for _ in range(a.rounds):
            for k, f in arms.items():
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(a.iters):
                    f()
                e1.record()
                e1.synchronize()
                times[k].append(e0.elapsed_time(e1) / a.iters)
    med = {k: statistics.median(v) for k, v in times.items()}
    rec = {"bench": "tta", "model": "s_psp", "shape": [B, 3, H, W], "dtype": "fp16", "rounds": a.rounds, "iters": a.iters,
           "ms": {k: round(v, 3) for k, v in med.items()},
           "ms_spread": {k: [round(min(v), 3), round(max(v), 3)] for k, v in times.items()},
           "tta_over_plain": round(med["tta"] / med["plain"], 3), "torch_over_tta": round(med["torch"] / med["tta"], 3),
           "tta_full_over_tta": round(med["tta_full"] / med["tta"], 3)}

    def pack_bytes(p):
        return sum(((s.conv.out_channels + 15) // 16 * 16) * s.conv.kernel_size[0] ** 2 * ((s.conv.in_channels + 15) // 16 * 16) * 2
                   for s in p.pb.slots)
    plans = {}
    for k, (_, _, _, (hp, wp)) in enumerate(tta_passes(H, W, 32)):
        for key in ((B, hp, wp), ("det", B, hp, wp)):
            if key in eng.plans:
                p = eng.plans[key]
                plans["x".join(str(v) for v in key)] = {"workspace_bytes": int(p.pb.workspace_bytes), "weight_pack_bytes_est": pack_bytes(p)}
    rec["plans"] = plans
    rec["gpu"] = gpu_state()
    print(json.dumps(rec))


if __name__ == "__main__":
    main()
