#!/usr/bin/env python
"""Benchmark of detect() (multiyolov5_b200/detect.py) against the per-frame composition of the public functions the reference's
detect.py loop is made of, on synthetic 1024x2048 frames at --img-size 1024 with s/PSP synth weights:

    python tools/bench_detect.py [--frames N] [--batch-size B] [--rounds R] [--out DIR]

Two modes: `--submit --nosave` (the Cityscapes submission run) and saving images (boxes, mask, blend, --save-txt).  Per mode and arm
two frame rates: the device pipeline (CUDA events from the first upload to the last device-to-host copy, the host writes replaced by a
wait for the copies) and end to end (host clock, PNG encoding and the txt writes included).  The driver and the composition alternate
within one call, R rounds each.  Prints ONE JSON line with the card's name and power limit read next to the measurement.  Writes its
files under a temporary directory (or --out), never into the tree.
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time
from argparse import Namespace

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import cv2  # noqa: E402
import numpy as np  # noqa: E402
import torch  # noqa: E402


def gpu_state(gpu_index=0):
    q = "name,power.limit,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader,nounits", "-i", str(gpu_index)],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        name, power_w, sm_max = [v.strip() for v in out.split(",")]
        return {"name": name, "power_limit_w": float(power_w), "max_sm_clock_mhz": float(sm_max)}
    except Exception as e:  # noqa: BLE001
        return {"name": torch.cuda.get_device_name(0), "nvidia_smi_error": str(e)}


def synth_frames(n, h, w, seed=0):
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float32)
    out = []
    for _ in range(n):
        img = np.empty((h, w, 3), np.float32)
        for c in range(3):
            fy, fx = rng.uniform(0.002, 0.02, 2)
            img[..., c] = 128 + 90 * np.sin(fy * yy + rng.uniform(0, 6.28)) * np.cos(fx * xx)
        img += rng.normal(0, 12, img.shape).astype(np.float32)
        out.append(np.clip(img, 0, 255).astype(np.uint8))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=48)
    ap.add_argument("--batch-size", type=int, default=16)
    ap.add_argument("--img-size", type=int, default=1024)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--conf-thres", type=float, default=0.25)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_detect needs a CUDA device"
    torch.cuda.set_device(0)
    from multiyolov5_b200 import detect as D
    from multiyolov5_b200.models.yolo import Model
    from multiyolov5_b200.utils.datasets import preprocess
    from multiyolov5_b200.utils.general import non_max_suppression, scale_coords, seg_argmax, seg_overlay, trainid2id, xyxy2xywh
    from multiyolov5_b200.utils.plots import plot_one_box
    from oracle import synth

    yml = "yolov5s_city_seg.yaml"
    cfg = synth.load_cfg(yml)
    model = Model(yml)
    model.load_state_dict(synth.synth_state_dict(synth.load_manifest("s_psp"), cfg, seed=1))
    model.cuda().eval()
    names = model.names
    base = synth_frames(4, 1024, 2048)
    frames = [(f"/frames/f_{i:04d}.png", base[i % len(base)]) for i in range(args.frames)]
    colors = [[int(v) for v in np.random.default_rng(1).integers(0, 255, 3)] for _ in names]

    class DeviceOnly(D.Postprocess):
        """the driver's stage with the host writes replaced by a wait for the copies: the device pipeline alone"""

        def _write(self, done, dev, host, *rest):
            done.synchronize()

    def opt_for(mode, root, tag):
        save = mode == "save"
        return Namespace(weights=None, source="", img_size=args.img_size, conf_thres=args.conf_thres, iou_thres=0.45, device="",
                         view_img=False, save_txt=save, save_conf=save, nosave=not save, classes=None, agnostic_nms=False, augment=False,
                         update=False, project=root, name=tag, exist_ok=False, save_as_video=False, submit=True, batch_size=args.batch_size)

    def driver_device(opt):
        save_dir, save_img = D.prepare(opt)
        post = DeviceOnly(opt, save_dir, names, colors, save_img)
        dev0 = torch.device("cuda", 0)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        with torch.no_grad():
            for paths, fr in D.batches(frames, opt.batch_size):
                dev, host = D.upload(fr, dev0)
                img = preprocess(dev, opt.img_size, stride=32, half=False)[0]
                out = model(img)
                post(paths, dev, img.shape[2:], out[0][0], out[1], host_frames=host)
        post.close()
        torch.cuda.current_stream().wait_stream(post.side)
        e1.record()
        e1.synchronize()
        return e0.elapsed_time(e1) / 1e3

    def driver_e2e(opt):
        t = time.perf_counter()
        D.detect(opt, dataset=frames, model=model)
        return time.perf_counter() - t

    def compose(opt, write):
        """the reference's per-frame loop over the public functions; write=False keeps only the device work and the copies back"""
        save_dir, save_img = D.prepare(opt)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t = time.perf_counter()
        e0.record()
        with torch.no_grad():
            for path, im0 in frames:
                im0 = im0.copy()
                stem = os.path.basename(path)[:-4]
                img = preprocess(im0, opt.img_size, stride=32, half=False)[0]
                out = model(img)
                det = non_max_suppression(out[0][0], opt.conf_thres, opt.iou_thres)[0].cpu()
                gn = torch.tensor(im0.shape)[[1, 0, 1, 0]]
                if len(det):
                    det[:, :4] = scale_coords(img.shape[2:], det[:, :4], im0.shape).round()
                    if write:
                        for *xyxy, conf, cls in reversed(det):
                            if opt.save_txt:
                                xywh = (xyxy2xywh(torch.tensor(xyxy).view(1, 4)) / gn).view(-1).tolist()
                                line = (cls, *xywh, conf)
                                with open(str(save_dir / "labels" / stem) + ".txt", "a") as f:
                                    f.write(("%g " * len(line)).rstrip() % line + "\n")
                            if save_img:
                                plot_one_box(xyxy, im0, label=f"{names[int(cls)]} {conf:.2f}", color=colors[int(cls)], line_thickness=3)
                cls_map = seg_argmax(out[1], im0.shape[:2])[0]
                ids = trainid2id(cls_map).cpu().numpy()
                if save_img:
                    mask = seg_overlay(cls_map, torch.from_numpy(im0).cuda())[0].cpu().numpy()
                    if write:
                        cv2.imwrite(str(save_dir / f"{stem}.png"), im0)
                        cv2.imwrite(str(save_dir / f"{stem}_mask.png"), mask)
                        cv2.imwrite(str(save_dir / f"{stem}_dst.png"), cv2.addWeighted(mask, 0.4, im0, 0.6, 0))
                if write:
                    cv2.imwrite(str(save_dir) + f"/results/{stem}_pred.png", ids)
        e1.record()
        e1.synchronize()
        return e0.elapsed_time(e1) / 1e3 if not write else time.perf_counter() - t

    res = {}
    with tempfile.TemporaryDirectory() as tmp:
        root = args.out or tmp
        k = 0
        for mode in ("submit_nosave", "save"):
            arms = {"driver_device": lambda o: driver_device(o), "driver_e2e": driver_e2e, "compose_device": lambda o: compose(o, False),
                    "compose_e2e": lambda o: compose(o, True)}
            times = {a: [] for a in arms}
            for a, fn in arms.items():                 # warm-up: every shape and batch size once
                fn(opt_for(mode, root, f"w{k}"))
                k += 1
            for _ in range(args.rounds):
                for a, fn in arms.items():
                    times[a].append(fn(opt_for(mode, root, f"r{k}")))
                    k += 1
            res[mode] = {a: {"frames_per_s": args.frames / min(v), "s_per_run": [round(x, 4) for x in v]} for a, v in times.items()}
    line = {"bench": "detect", "frames": args.frames, "frame_hw": [1024, 2048], "img_size": args.img_size, "batch_size": args.batch_size,
            "weights": "s_psp synth (seed 1)", "conf_thres": args.conf_thres, "gpu": gpu_state(), "results": res,
            "note": "device = CUDA events to the last device-to-host copy (driver) or the last .cpu() (composition); e2e = host clock "
                    "with every file written; PNG encoding runs on one writer thread"}
    print(json.dumps(line))


if __name__ == "__main__":
    main()
