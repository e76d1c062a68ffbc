#!/usr/bin/env python
"""Benchmark of `--rect` training (DetRectLoader, csrc/augment.cu at H x W, Trainer(det_shapes=...)).

    python tools/bench_rect.py [--steps K] [--warmup W]

Prints ONE JSON line with the card's name, power limit and clocks read next to the measurement:
  kernel_us_per_image     myolo_augment_det_hw alone at B = 16 and 512 x 1024 (uint8 out), CUDA events over K launches
  loader_us_per_image     DetRectLoader(positions) end to end (host draws + labels + parameter upload + kernel), to a device synchronise
  host                    the reference's per-item arithmetic through cv2 on one core (letterbox + warpAffine + augment_hsv + flips + CHW)
  step                    Trainer.step (s/PSP, 4 det + 4 seg images of 512 x 1024) with a rect 512 x 1024 det batch and with a 1024 x 1024
                          mosaic batch, two trainers alternating step by step, median and min over K/10 steps each
  cityscapes_rect_ms      Cityscapes rect (512 x 1024) + --multi-scale at imgsz 1024, B = 16: the reserved shapes, the shared pair's size and
                          the device memory in use (driver) before and with every reserved plan created and prepared
  random_ar_640_ms        random aspect ratios at img_size 640, batch 16, 2000 images, rect + multi-scale: the same, plans prepared
                          until 120 s or 8 GB free remain (how many were made is reported)
The sources are synthetic: 16 Cityscapes-shaped 2048 x 1024 BGR frames (cached at 1024 x 512), hyp.scratch.  Writes nothing to disk.
"""
import argparse
import gc
import json
import math
import os
import random
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from tools.bench_augment import AUG_HYP, gpu_state  # noqa: E402

HYP = dict(lr0=0.01, momentum=0.937, weight_decay=5e-4, box=0.05, cls=0.5, cls_pw=1.0, obj=1.0, obj_pw=1.0, anchor_t=4.0, fl_gamma=0.0)


def _host_rect_item(img, shape, hyp, cv2):
    """the reference's per-item host arithmetic through cv2 for rect=True (letterbox to the batch shape, random_perspective at that size,
    augment_hsv, flips, CHW); labels are left out (host work in both arms)"""
    h, w = img.shape[:2]
    r = min(shape[0] / h, shape[1] / w)
    nw, nh = int(round(w * r)), int(round(h * r))
    if (nw, nh) != (w, h):
        img = cv2.resize(img, (nw, nh), interpolation=cv2.INTER_LINEAR)
    dw, dh = (shape[1] - nw) / 2, (shape[0] - nh) / 2
    img = cv2.copyMakeBorder(img, int(round(dh - 0.1)), int(round(dh + 0.1)), int(round(dw - 0.1)), int(round(dw + 0.1)),
                             cv2.BORDER_CONSTANT, value=(114, 114, 114))
    H, W = img.shape[:2]
    C_ = np.eye(3); C_[0, 2], C_[1, 2] = -W / 2, -H / 2
    R = np.eye(3)
    R[:2] = cv2.getRotationMatrix2D(angle=random.uniform(-hyp["degrees"], hyp["degrees"]), center=(0, 0),
                                    scale=random.uniform(1 - hyp["scale"], 1 + hyp["scale"]))
    S = np.eye(3)
    S[0, 1] = math.tan(random.uniform(-hyp["shear"], hyp["shear"]) * math.pi / 180)
    S[1, 0] = math.tan(random.uniform(-hyp["shear"], hyp["shear"]) * math.pi / 180)
    T = np.eye(3)
    T[0, 2] = random.uniform(0.5 - hyp["translate"], 0.5 + hyp["translate"]) * W
    T[1, 2] = random.uniform(0.5 - hyp["translate"], 0.5 + hyp["translate"]) * H
    M = T @ S @ R @ C_
    img = cv2.warpAffine(img, M[:2], dsize=(W, H), borderValue=(114, 114, 114))
    g = np.random.uniform(-1, 1, 3) * [hyp["hsv_h"], hyp["hsv_s"], hyp["hsv_v"]] + 1
    hue, sat, val = cv2.split(cv2.cvtColor(img, cv2.COLOR_BGR2HSV))
    x = np.arange(0, 256, dtype=np.int16)
    luts = ((x * g[0]) % 180).astype(np.uint8), np.clip(x * g[1], 0, 255).astype(np.uint8), np.clip(x * g[2], 0, 255).astype(np.uint8)
    img = cv2.cvtColor(cv2.merge((cv2.LUT(hue, luts[0]), cv2.LUT(sat, luts[1]), cv2.LUT(val, luts[2]))), cv2.COLOR_HSV2BGR)
    if random.random() < hyp["fliplr"]:
        img = np.fliplr(img)
    return np.ascontiguousarray(img[:, :, ::-1].transpose(2, 0, 1))


def _model():
    from multiyolov5_b200.models.yolo import Model
    from oracle import synth
    yml = "yolov5s_city_seg.yaml"
    cfg = synth.load_cfg(yml)
    model = Model(yml)
    model.load_state_dict(synth.synth_state_dict(synth.load_manifest("s_psp"), cfg, seed=1, gain=1.0))
    return model.cuda().train(), cfg["nc"]


def _trainer(B, imgsz, **kw):
    from multiyolov5_b200.train import Trainer, scale_hyp
    model, nc = _model()
    return Trainer(model, scale_hyp(HYP, nl=3, nc=nc, imgsz=imgsz, total_batch_size=B), batch_size=B, init_scale=2.0 ** 10, **kw), nc


def _targets(B, nc, seed):
    rs = np.random.RandomState(seed)
    t = np.zeros((40, 6), np.float32)
    t[:, 0] = rs.randint(0, B, 40); t[:, 1] = rs.randint(0, nc, 40)
    t[:, 2:4] = rs.uniform(0.1, 0.9, (40, 2)); t[:, 4:6] = rs.uniform(0.02, 0.3, (40, 2))
    return torch.from_numpy(t).cuda()


def _used_gb():
    free, total = torch.cuda.mem_get_info()
    return (total - free) / 1e9


def _reserve_record(tr, B, budget_s):
    """reserved shapes, the shared pair, and the device memory (driver, whole card) with the reserved plans created and prepared
    (weight packs, parameter and gradient pointers: what a plan holds besides the shared pair), until budget_s or 8 GB free"""
    eng = tr.model.engine()
    shapes = tr.det_train_shapes()
    rec = {"reserved_shapes": len(shapes), "shared_pair_gb": eng._arenas[0].capacity * 2 / 1e9, "device_used_gb_before_plans": _used_gb()}
    t0, made = time.perf_counter(), 0
    for H, W in sorted(shapes, key=lambda hw: -hw[0] * hw[1]):
        if time.perf_counter() - t0 > budget_s or torch.cuda.mem_get_info()[0] < 8e9:
            break
        eng.prepare_train_plan(eng.train_plan_for(B, H, W))
        made += 1
    torch.cuda.synchronize()
    rec.update(plans_prepared=made, device_used_gb_with_plans=_used_gb(), seconds_to_prepare=time.perf_counter() - t0)
    rec["gb_per_plan"] = (rec["device_used_gb_with_plans"] - rec["device_used_gb_before_plans"]) / max(made, 1)
    return rec


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=10)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_rect needs a CUDA device")
    from multiyolov5_b200 import _lib
    from multiyolov5_b200.train import MultiScale
    from multiyolov5_b200.utils.datasets import DetAugmenter, DetRectLoader, DeviceImageCache
    steps = args.steps
    rec = {"gpu": gpu_state()}
    B, s = 16, 1024
    rs = np.random.RandomState(0)
    frames = [rs.randint(0, 256, (1024, 2048, 3), dtype=np.uint8) for _ in range(B)]
    labels = [np.array([[k % 10, 0.5, 0.5, 0.2, 0.3], [1, 0.1, 0.8, 0.1, 0.2]], np.float32) for k in range(B)]
    cache = DeviceImageCache(frames, s, labels)
    loader = DetRectLoader(cache, AUG_HYP, B)
    assert loader.batch_shapes.tolist() == [[512, 1024]]
    random.seed(0)
    np.random.seed(0)
    pos = list(range(B))
    for _ in range(args.warmup):
        loader(pos)
    torch.cuda.synchronize()
    # ---- the kernel alone, parameters prepared once
    L, sp = _lib.lib(), _lib.stream_ptr()
    items = (_lib.AugItem * B)(*[loader.item(p)[0] for p in pos])
    dev_items = torch.frombuffer(bytearray(items), dtype=torch.uint8).cuda()
    out = torch.empty((B, 3, 512, 1024), dtype=torch.uint8, device="cuda")
    for _ in range(args.warmup):
        _lib.check(L.myolo_augment_det_hw(_lib.ptr(dev_items), B, 512, 1024, _lib.ptr(out), _lib.U8, sp))
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        _lib.check(L.myolo_augment_det_hw(_lib.ptr(dev_items), B, 512, 1024, _lib.ptr(out), _lib.U8, sp))
    e1.record()
    torch.cuda.synchronize()
    kernel_ms = e0.elapsed_time(e1) / steps
    # ---- the loader end to end
    t0 = time.perf_counter()
    for _ in range(steps):
        loader(pos)
    torch.cuda.synchronize()
    loader_ms = (time.perf_counter() - t0) * 1e3 / steps
    rec.update(B=B, shape=[512, 1024], sources="16 x 2048x1024 BGR uint8, cached at 1024x512", hyp="hyp.scratch",
               kernel_us_per_image=kernel_ms * 1e3 / B, kernel_images_per_s=B / (kernel_ms * 1e-3),
               kernel_hbm_gbs=3 * 512 * 1024 * B / (kernel_ms * 1e-3) / 1e9,
               loader_us_per_image=loader_ms * 1e3 / B, loader_images_per_s=B / (loader_ms * 1e-3))
    try:
        import cv2
        cached = [cache.image(i).cpu().numpy() for i in range(B)]
        prev = cv2.getNumThreads()
        cv2.setNumThreads(1)
        try:
            _host_rect_item(cached[0], (512, 1024), AUG_HYP, cv2)
            n_host = 32
            t0 = time.perf_counter()
            for k in range(n_host):
                _host_rect_item(cached[k % B], (512, 1024), AUG_HYP, cv2)
            one_ms = (time.perf_counter() - t0) * 1e3 / n_host
        finally:
            cv2.setNumThreads(prev)
        rec["host"] = {"ms_per_image_one_core": one_ms, "images_per_s_one_core": 1e3 / one_ms}
    except ImportError as e:
        rec["host"] = {"not measured": str(e)}
    del items, dev_items, out
    # ---- Trainer.step: rect 512 x 1024 against a 1024 x 1024 mosaic batch, alternating
    SB = 4
    rect = DetRectLoader(cache, AUG_HYP, SB)
    square = DetAugmenter(DeviceImageCache([f[:512, :1024] for f in frames[:8]], s, labels[:8]), AUG_HYP)
    trs = {"rect_512x1024": _trainer(SB, s, det_shapes=rect.batch_shapes), "mosaic_1024x1024": _trainer(SB, s)}
    g = torch.Generator(device="cuda").manual_seed(0)
    seg = torch.rand((SB, 3, 512, 1024), device="cuda", generator=g)
    segt = torch.randint(-1, 19, (SB, 512, 1024), device="cuda", generator=g)
    n = max(steps // 10, 10)
    times = {k: [] for k in trs}
    clock_before = gpu_state().get("sm_mhz")
    for i in range(n + 3):
        for k, (tr, nc) in trs.items():
            imgs, _ = rect(list(range(SB)), torch.float16) if k.startswith("rect") else square(list(range(SB)), torch.float16)
            t = _targets(SB, nc, i)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            tr.step(imgs, t, seg, segt)
            torch.cuda.synchronize()
            if i >= 3:
                times[k].append(time.perf_counter() - t0)
    rec["step"] = {"B_det": SB, "B_seg": SB, "steps_per_arm": n, "sm_mhz_before": clock_before, "sm_mhz_after": gpu_state().get("sm_mhz")}
    for k, v in times.items():
        rec["step"][f"{k}_ms_median"] = float(np.median(v) * 1e3)
        rec["step"][f"{k}_ms_min"] = float(np.min(v) * 1e3)
    del trs, rect, square
    gc.collect()
    torch.cuda.empty_cache()
    # ---- reserved shapes and device memory: Cityscapes rect + multi-scale at 1024, then random aspect ratios at 640
    tr, _ = _trainer(B, s, multi_scale=MultiScale(s), det_shapes=loader.batch_shapes)
    rec["cityscapes_rect_ms"] = _reserve_record(tr, B, budget_s=600)
    del tr
    gc.collect()
    torch.cuda.empty_cache()
    from multiyolov5_b200.utils.datasets import rect_plan
    ar_rs = np.random.RandomState(1)
    shapes0 = [(int(h), int(w)) for h, w in zip(ar_rs.randint(200, 1200, 2000), ar_rs.randint(200, 1200, 2000))]
    _, _, bshapes = rect_plan(shapes0, 640, B)
    tr, _ = _trainer(B, 640, multi_scale=MultiScale(640), det_shapes=bshapes)
    rec["random_ar_640_ms"] = dict(_reserve_record(tr, B, budget_s=120), images=2000, batches=len(bshapes),
                                   distinct_batch_shapes=len({tuple(v) for v in bshapes.tolist()}))
    rec["gpu_after"] = gpu_state()
    print(json.dumps(rec), flush=True)


if __name__ == "__main__":
    main()
