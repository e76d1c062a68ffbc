#!/usr/bin/env python
"""Benchmark of the device-side validation statistics (utils.metrics.DetectionStats, csrc/metrics.cu) and of test().

    python tools/bench_val.py [--steps K] [--warmup W]

Prints ONE JSON line with the card's name, power limit and clocks read next to the measurement:
  match_us_per_image     myolo_det_match (batches of 32 images, 300 rows and 20 labels each), CUDA events over K launches
  ap_ms_{500,5000}       myolo_det_ap over 500 / 5 000 images x up to 300 predictions, CUDA events over K calls
  stats_ms_{500,5000}    DetectionStats end to end: every update + compute to host results, host clock
  ref_ms_500             the reference's statistics arithmetic on the same 500 images: the test.py:182-265 loop as torch ops on this GPU
                         (ref_match_ms_500) plus ap_per_class in numpy on one host core (ref_ap_ms_500)
  test_ms_500            test() end to end with the s/PSP model, 500 synthetic uint8 images at 544x1056 (2048x1024 frames at imgsz
                         1024, pad 0.5, stride 32), batch 32, half precision
Writes nothing to disk.
"""
import argparse
import json
import os
import sys
import time
import warnings

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from tools.bench_augment import gpu_state  # noqa: E402


def synth_batch(rs, B, nc=10, nl=20, max_det=300, hw=(544, 1056)):
    H, W = hw
    shapes, tg = [], []
    dets = np.zeros((B, max_det, 6), np.float32)
    counts = np.full(B, max_det, np.int32)
    for si in range(B):
        shapes.append(((1024, 2048), ((0.5, 0.5), (0.0, 16.0))))
        lab = np.zeros((nl, 6), np.float32)
        lab[:, 0] = si
        lab[:, 1] = rs.randint(0, nc, nl)
        lab[:, 2:4] = rs.uniform(0.05, 0.95, (nl, 2))
        lab[:, 4:6] = rs.uniform(0.02, 0.3, (nl, 2))
        tg.append(lab)
        t = lab[rs.randint(nl, size=max_det)]
        x, y, w, h = t[:, 2] * W, t[:, 3] * H, t[:, 4] * W, t[:, 5] * H
        j = rs.normal(0, 0.15, (max_det, 4)).astype(np.float32)
        x, y, w, h = x + j[:, 0] * w, y + j[:, 1] * h, w * (1 + j[:, 2]), h * (1 + j[:, 3])
        cls = np.where(rs.rand(max_det) < 0.85, t[:, 1], rs.randint(0, nc, max_det))
        conf = -np.sort(-rs.uniform(0.001, 1, max_det).astype(np.float32))
        dets[si] = np.stack([x - w / 2, y - h / 2, x + w / 2, y + h / 2, conf, cls], 1)
    return dets, counts, np.concatenate(tg, 0), shapes


def ref_match_torch(dets, counts, targets, hw, shapes, device):
    """test.py:175,182-265 as the reference runs it, on `device` (per image and class: nonzero, box_iou, max, .item())"""
    from multiyolov5_b200.utils.general import box_iou, scale_coords, xywh2xyxy
    iouv = torch.linspace(0.5, 0.95, 10).to(device)
    targets = targets.clone()
    height, width = hw
    targets[:, 2:] *= torch.Tensor([width, height, width, height]).to(device)
    stats = []
    for si in range(dets.shape[0]):
        pred = dets[si, :int(counts[si])]
        labels = targets[targets[:, 0] == si, 1:]
        nl = len(labels)
        tcls = labels[:, 0].tolist() if nl else []
        predn = pred.clone()
        scale_coords(hw, predn[:, :4], shapes[si][0], shapes[si][1])
        correct = torch.zeros(pred.shape[0], 10, dtype=torch.bool, device=device)
        if nl:
            detected = []
            tcls_tensor = labels[:, 0]
            tbox = xywh2xyxy(labels[:, 1:5])
            scale_coords(hw, tbox, shapes[si][0], shapes[si][1])
            for cls in torch.unique(tcls_tensor):
                ti = (cls == tcls_tensor).nonzero(as_tuple=False).view(-1)
                pi = (cls == pred[:, 5]).nonzero(as_tuple=False).view(-1)
                if pi.shape[0]:
                    ious, i = box_iou(predn[pi, :4], tbox[ti]).max(1)
                    detected_set = set()
                    for j in (ious > iouv[0]).nonzero(as_tuple=False):
                        d = ti[i[j]]
                        if d.item() not in detected_set:
                            detected_set.add(d.item())
                            detected.append(d)
                            correct[pi[j]] = ious[j] > iouv
                            if len(detected) == nl:
                                break
        stats.append((correct.cpu(), pred[:, 4].cpu(), pred[:, 5].cpu(), tcls))
    return stats


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_val needs a CUDA device"
    from multiyolov5_b200 import _lib
    from multiyolov5_b200.utils.metrics import DetectionStats, _run_ap
    from oracle import restate_val as R
    dev = torch.device("cuda")
    rs = np.random.RandomState(0)
    hw = (544, 1056)
    host = [synth_batch(rs, 32) for _ in range(157)]               # 5 024 images
    batches = [(torch.from_numpy(d).to(dev), torch.from_numpy(c).to(dev), torch.from_numpy(t).to(dev), s) for d, c, t, s in host]
    rec = {"gpu": gpu_state(), "images_per_batch": 32, "rows_per_image": 300, "labels_per_image": 20, "classes": 10}
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)

    # match kernel alone
    st = DetectionStats(max_det=300, capacity=32)
    d, c, t, s = batches[0]
    for _ in range(args.warmup):
        st.seen = 0
        st.update(d, c, t, hw, s)
    torch.cuda.synchronize()
    ev0.record()
    for _ in range(args.steps):
        st.seen = 0
        st.update(d, c, t, hw, s)
    ev1.record()
    torch.cuda.synchronize()
    rec["match_us_per_image"] = ev0.elapsed_time(ev1) * 1e3 / (args.steps * 32)

    for n_img in (500, 5000):
        nb = (n_img + 31) // 32
        st = DetectionStats(max_det=300, capacity=nb * 32)
        for d, c, t, s in batches[:nb]:
            st.update(d, c, t, hw, s)
        n = st.seen
        for _ in range(args.warmup):
            _run_ap(st.correct, st.conf, st.cls, st.rows, n, 300, 10, st.tcount)
        torch.cuda.synchronize()
        ev0.record()
        for _ in range(args.steps):
            _run_ap(st.correct, st.conf, st.cls, st.rows, n, 300, 10, st.tcount)
        ev1.record()
        torch.cuda.synchronize()
        rec[f"ap_ms_{n_img}"] = ev0.elapsed_time(ev1) / args.steps
        rec[f"ap_images_{n_img}"] = n
        times = []
        for _ in range(max(3, args.steps // 10)):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            st2 = DetectionStats(max_det=300, capacity=nb * 32)
            for d, c, t, s in batches[:nb]:
                st2.update(d, c, t, hw, s)
            out = st2.compute(10)
            times.append(time.perf_counter() - t0)
        rec[f"stats_ms_{n_img}"] = float(np.median(times) * 1e3)
        rec[f"map50_{n_img}"] = float(out[2][:, 0].mean())

    # the reference's arithmetic on the same first 512 images
    torch.set_num_threads(1)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    stats = []
    for d, c, t, s in batches[:16]:
        stats += ref_match_torch(d, c.cpu(), t, hw, s, dev)
    t1 = time.perf_counter()
    cat = [np.concatenate([np.asarray(x) for x in col], 0) for col in zip(*stats)]
    t2 = time.perf_counter()
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        R.ap_per_class(*cat)
    t3 = time.perf_counter()
    rec["ref_match_ms_500"] = (t1 - t0) * 1e3
    rec["ref_ap_ms_500"] = (t3 - t2) * 1e3
    rec["ref_ms_500"] = (t3 - t0) * 1e3

    # test() end to end with the s/PSP model
    from multiyolov5_b200.models.yolo import Model
    from multiyolov5_b200.test import test
    from oracle import synth
    yml = "yolov5s_city_seg.yaml"
    cfg = synth.load_cfg(yml)
    model = Model(yml)
    model.load_state_dict(synth.synth_state_dict(synth.load_manifest("s_psp"), cfg, seed=1))
    model.cuda().eval()
    g = torch.Generator().manual_seed(0)
    loader = []
    for b in range(0, 500, 32):
        B = min(32, 500 - b)
        img = torch.randint(0, 256, (B, 3, 544, 1056), dtype=torch.uint8, generator=g).to(dev)
        _, _, tg, shapes = host[b // 32]
        tg = torch.from_numpy(tg[tg[:, 0] < B]).to(dev)
        loader.append((img, tg, [""] * B, shapes[:B]))
    test({"nc": cfg["nc"]}, model=model, dataloader=loader[:2], plots=False)       # warm-up: plans for both batch sizes
    test({"nc": cfg["nc"]}, model=model, dataloader=loader[-1:], plots=False)
    times = []
    for _ in range(2):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        res, _, t = test({"nc": cfg["nc"]}, model=model, dataloader=loader, plots=False)
        times.append(time.perf_counter() - t0)
    rec["test_ms_500"] = float(min(times) * 1e3)
    rec["test_forward_nms_ms_per_image"] = [float(v) for v in t[:3]]
    rec["gpu_after"] = gpu_state()
    print(json.dumps(rec), flush=True)
    _lib.lib()


if __name__ == "__main__":
    main()
