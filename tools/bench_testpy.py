"""Times the two device pieces behind test.py's --save-hybrid and plots options on one GPU, with CUDA events, as medians over
alternating rounds, and prints ONE JSON line with the card's name and power limit:

  nms        non_max_suppression at B = 32 over z of 1024x512 inputs (32 256 rows) and of their TTA (71 316 rows), nc 8, multi-label at
             conf 0.001: the plain kernel against myolo_nms_labels with 0, 20 and 200 labels per image
  confusion  ConfusionMatrix.update over a batch of 32 images (300 NMS rows, 100 labels each, nc 10) against the per-image torch
             composition of process_batch that test.py runs (torch.where, box_iou, the two sorts and the counting loops)

    python tools/bench_testpy.py [--rounds 15 --warmup 3]
"""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from tools.bench_detect import gpu_state  # noqa: E402


def timed(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b)


def torch_process_batch(matrix, detections, labels, nc, conf=0.25, iou_thres=0.45):
    """the fork's process_batch statements on device tensors (its numpy part on the host)"""
    from multiyolov5_b200.utils.general import box_iou
    detections = detections[detections[:, 4] > conf]
    gt_classes = labels[:, 0].int()
    detection_classes = detections[:, 5].int()
    iou = box_iou(labels[:, 1:], detections[:, :4])
    x = torch.where(iou > iou_thres)
    if x[0].shape[0]:
        matches = torch.cat((torch.stack(x, 1), iou[x[0], x[1]][:, None]), 1).cpu().numpy()
        if x[0].shape[0] > 1:
            matches = matches[matches[:, 2].argsort()[::-1]]
            matches = matches[np.unique(matches[:, 1], return_index=True)[1]]
            matches = matches[matches[:, 2].argsort()[::-1]]
            matches = matches[np.unique(matches[:, 0], return_index=True)[1]]
    else:
        matches = np.zeros((0, 3))
    n = matches.shape[0] > 0
    m0, m1, _ = matches.transpose().astype(np.int16)
    gt_classes, detection_classes = gt_classes.cpu().numpy(), detection_classes.cpu().numpy()
    for i, gc in enumerate(gt_classes):
        j = m0 == i
        if n and sum(j) == 1:
            matrix[gc, detection_classes[m1[j]]] += 1
        else:
            matrix[nc, gc] += 1
    if n:
        for i, dc in enumerate(detection_classes):
            if not any(m1 == i):
                matrix[dc, nc] += 1


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=15)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    from multiyolov5_b200.utils.general import NmsLabels, non_max_suppression
    from multiyolov5_b200.utils.metrics import ConfusionMatrix
    torch.cuda.set_device(0)
    line = {"bench": "testpy", "rounds": args.rounds, "gpu": gpu_state(0)}
    B, nc = 32, 8
    for A in (32256, 71316):
        g = torch.Generator(device="cuda").manual_seed(A)
        z = torch.rand((B, A, 5 + nc), device="cuda", generator=g)
        z[..., :2] *= 1024
        z[..., 2:4] = z[..., 2:4] * 120 + 2
        z[..., 4] = z[..., 4] ** 3
        arms = {"plain": lambda: non_max_suppression(z, 0.001, 0.6, multi_label=True, return_padded=True)}
        for k in (0, 20, 200):
            rs = np.random.RandomState(k)
            rows = np.zeros((B * k, 5), np.float32)
            rows[:, 0] = rs.randint(0, nc, B * k)
            rows[:, 1:3], rows[:, 3:5] = rs.uniform(0, 1024, (B * k, 2)), rs.uniform(2, 120, (B * k, 2))
            lab = NmsLabels(torch.from_numpy(rows).cuda(), torch.arange(0, B * k + 1, max(k, 1), dtype=torch.int32).cuda()[:B + 1]
                            if k else torch.zeros(B + 1, dtype=torch.int32, device="cuda"), k)
            arms[f"labels{k}"] = (lambda lab=lab: non_max_suppression(z, 0.001, 0.6, multi_label=True, labels=lab, return_padded=True))
        res = {a: [] for a in arms}
        for r in range(args.warmup + args.rounds):
            for a, fn in arms.items():
                t = timed(fn)
                if r >= args.warmup:
                    res[a].append(t)
        for a, v in res.items():
            line[f"nms_A{A}_{a}_ms"] = round(statistics.median(v), 3)
    # confusion matrix
    nc, H, W, B = 10, 512, 1024, 32
    rs = np.random.RandomState(0)
    tg, dets = [], torch.zeros((B, 300, 6))
    for b in range(B):
        lab = np.zeros((100, 6), np.float32)
        lab[:, 0], lab[:, 1] = b, rs.randint(0, nc, 100)
        lab[:, 2:4], lab[:, 4:6] = rs.uniform(0.05, 0.95, (100, 2)), rs.uniform(0.02, 0.2, (100, 2))
        tg.append(lab)
        src = rs.randint(0, 100, 300)
        c = lab[src, 2:6] * np.float32([W, H, W, H]) + rs.uniform(-6, 6, (300, 4)).astype(np.float32)
        dets[b, :, :2], dets[b, :, 2:4] = torch.from_numpy(c[:, :2] - c[:, 2:] / 2), torch.from_numpy(c[:, :2] + c[:, 2:] / 2)
        dets[b, :, 4] = torch.from_numpy(np.sort(rs.uniform(0.01, 1, 300))[::-1].copy())
        dets[b, :, 5] = torch.from_numpy(np.where(rs.rand(300) < 0.7, lab[src, 1], rs.randint(0, nc, 300)).astype(np.float32))
    targets = torch.from_numpy(np.concatenate(tg)).cuda()
    dets, counts = dets.cuda(), torch.full((B,), 300, dtype=torch.int32, device="cuda")
    shapes = [((H, W), ((1.0, 1.0), (0.0, 0.0)))] * B
    cm = ConfusionMatrix(nc)
    labn = []
    for b in range(B):
        t = targets[targets[:, 0] == b, 1:].clone()
        t[:, 1:] *= torch.tensor([W, H, W, H], device="cuda")
        xy = torch.cat([t[:, 1:3] - t[:, 3:5] / 2, t[:, 1:3] + t[:, 3:5] / 2], 1)
        labn.append(torch.cat([t[:, :1], xy], 1))
    ref = np.zeros((nc + 1, nc + 1))
    arms = {"device": lambda: cm.update(dets, counts, targets, (H, W), shapes),
            "torch": lambda: [torch_process_batch(ref, dets[b], labn[b], nc) for b in range(B)]}
    res = {a: [] for a in arms}
    for r in range(args.warmup + args.rounds):
        for a, fn in arms.items():
            t = timed(fn)
            if r >= args.warmup:
                res[a].append(t)
    for a, v in res.items():
        line[f"confusion_{a}_ms"] = round(statistics.median(v), 3)
    print(json.dumps(line))


if __name__ == "__main__":
    main()
