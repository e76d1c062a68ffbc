#!/usr/bin/env python
"""Benchmark of autoShape (multiyolov5_b200/models/common.py) against the reference's host path, on 16 mixed frames (720p, 1080p and
portrait 1080x1920, RGB uint8) at size 640 with s/PSP synth weights:

    python tools/bench_autoshape.py [--rounds R] [--size S]

Arms, alternating within one call (R timed rounds each after warm-up):
  device  one autoShape call: pinned staging copy, myolo_letterbox_items, forward, NMS, myolo_scale_boxes, myolo_seg_crop_upsample_argmax
  host    the reference's models/common.py:655-667: per-image cv2 letterbox (cv2.resize + copyMakeBorder), np.stack, transpose, upload,
          `.float() / 255.`, then the same forward and non_max_suppression (its row counts read back)
Per arm the medians of the pre-process (up to the batch x on the device) and of the whole call, from CUDA events (the host work in
between shows up in them: the stream is idle while the host prepares).  Prints ONE JSON line with the card's name and power limit.
"""
import argparse
import contextlib
import io
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import cv2  # noqa: E402
import numpy as np  # noqa: E402
import torch  # noqa: E402

from tools.bench_detect import gpu_state  # noqa: E402


def frames16(seed=0):
    rng = np.random.default_rng(seed)
    shapes = [(720, 1280), (1080, 1920), (1920, 1080)] * 5 + [(720, 1280)]
    out = []
    for h, w in shapes:
        yy, xx = np.mgrid[0:h, 0:w].astype(np.float32)
        img = np.stack([128 + 90 * np.sin(rng.uniform(0.002, 0.02) * yy + c) * np.cos(rng.uniform(0.002, 0.02) * xx) for c in range(3)], 2)
        img += rng.normal(0, 12, img.shape).astype(np.float32)
        out.append(np.clip(img, 0, 255).astype(np.uint8))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--size", type=int, default=640)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_autoshape needs a CUDA device"
    torch.cuda.set_device(0)
    from multiyolov5_b200.models.common import autoshape_inputs
    from multiyolov5_b200.models.yolo import Model
    from multiyolov5_b200.utils.datasets import letterbox_geometry
    from multiyolov5_b200.utils.general import non_max_suppression
    from oracle import synth

    yml = "yolov5s_city_seg.yaml"
    cfg = synth.load_cfg(yml)
    net = Model(yml)
    net.load_state_dict(synth.synth_state_dict(synth.load_manifest("s_psp"), cfg, seed=1))
    net.cuda().eval()
    with contextlib.redirect_stdout(io.StringIO()):
        shaped = net.autoshape()
    imgs = frames16()
    dev = torch.device("cuda", 0)

    def device_call():
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
        ev[0].record()
        d = shaped(imgs, size=args.size)
        ev[1].record()
        ev[1].synchronize()
        return d._times[0].elapsed_time(d._times[1]), ev[0].elapsed_time(ev[1])

    def host_call():
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
        ev[0].record()
        ims, _, _, shape1 = autoshape_inputs(imgs, args.size, 32)
        x = []
        for im in ims:
            (rw, rh), _, _, (top, bottom, left, right) = letterbox_geometry(im.shape[:2], shape1, auto=False)
            r = cv2.resize(im, (rw, rh), interpolation=cv2.INTER_LINEAR) if im.shape[1::-1] != (rw, rh) else im
            x.append(cv2.copyMakeBorder(r, top, bottom, left, right, cv2.BORDER_CONSTANT, value=(114, 114, 114)))
        x = np.ascontiguousarray(np.stack(x, 0).transpose((0, 3, 1, 2)))
        x = torch.from_numpy(x).to(dev).float() / 255.
        ev[1].record()
        with torch.no_grad():
            y = net(x)[0][0]
            non_max_suppression(y, shaped.conf, shaped.iou)
        ev[2].record()
        ev[2].synchronize()
        return ev[0].elapsed_time(ev[1]), ev[0].elapsed_time(ev[2])

    for _ in range(args.warmup):
        device_call()
        host_call()
    res = {"device": [], "host": []}
    for _ in range(args.rounds):
        res["device"].append(device_call())
        res["host"].append(host_call())
    line = {"bench": "autoshape", "frames": len(imgs), "size": args.size, "rounds": args.rounds, "gpu": gpu_state(0)}
    for arm, v in res.items():
        line[f"{arm}_preprocess_ms"] = round(statistics.median(a for a, _ in v), 3)
        line[f"{arm}_call_ms"] = round(statistics.median(b for _, b in v), 3)
    print(json.dumps(line))


if __name__ == "__main__":
    main()
