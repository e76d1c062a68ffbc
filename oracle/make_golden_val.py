"""TEST INFRASTRUCTURE - generates tests/golden/val_cases.npz by running the UNMODIFIED reference's test.test() (test.py:77-340) on the
CPU, with a stand-in model whose forward returns crafted `z` tensors and a list dataloader of collate_fn tuples.

    MYOLO_REFERENCE_ROOT=<checkout> python oracle/make_golden_val.py

`ap_per_class` is wrapped in the imported test module's namespace (its source is untouched) to record its inputs (correct, conf, pcls,
tcls) and outputs.  The file holds, per case: every batch's z, network input size, targets and shapes (as (h0, w0, gain_h, gain_w, padw,
padh) rows), the recorded ap_per_class call (if test() made one) and test()'s return value.  Cases:
  main       nc 3, two batches: rect shapes with gains 0.416 / 1.04 / 0.5 and half-pixel pads; one target per IoU probe, whose
             prediction's native-space IoU is exactly each iouv or one float32 ulp either side (22 of the 30 values have such a box
             within the search; the others are left out); boxes clipped at the borders; zero-area
             boxes (NaN IoU, which wins the max and never matches); two predictions with the same best target where the second one's
             second-best target is free (it stays incorrect); an image with labels and no predictions, and one with predictions only
  single_cls nc 1 (single_cls=True), one class in z and targets
  no_tp      nc 3, no prediction overlaps a target (the `stats[0].any()` branch: maps all equal map)
Confidences are distinct within each case, so the reference's unstable argsort has no ties to break.
"""
import json
import os
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
from oracle import ref_shims, restate_val as R  # noqa: E402

GOLD = os.path.join(HERE, "..", "tests", "golden")
A = 160          # rows of z per image


class Case:
    def __init__(self, nc, seed):
        self.nc = nc
        self.rs = np.random.RandomState(seed)
        self.batches = []
        self.used_conf = set()

    def conf(self):
        while True:
            c = np.float32(self.rs.uniform(0.05, 0.99))
            if float(c) not in self.used_conf:
                self.used_conf.add(float(c))
                return c

    def batch(self, hw, shapes):
        b = dict(hw=hw, shapes=shapes, preds=[[] for _ in shapes], labels=[[] for _ in shapes])
        self.batches.append(b)
        return b


def net_xywh(box, shape):
    """native xyxy -> approximate network-space xywh (float32)"""
    g, (pw, ph) = shape[1][0][0], shape[1][1]
    x1, y1, x2, y2 = (box[0] * g + pw, box[1] * g + ph, box[2] * g + pw, box[3] * g + ph)
    return np.float32([(x1 + x2) / 2, (y1 + y2) / 2, x2 - x1, y2 - y1])


def add_label(b, si, cls, box):
    """native xyxy box -> normalised [cls, x, y, w, h] label"""
    x, y, w, h = net_xywh(box, b["shapes"][si])
    H, W = b["hw"]
    b["labels"][si].append([cls, x / W, y / H, w / W, h / H])


def add_pred(c, b, si, cls, xywh, conf=None):
    b["preds"][si].append((np.float32(xywh), cls, c.conf() if conf is None else np.float32(conf)))


def probe(b, si, cls, want):
    """network xywh of a prediction whose native IoU with the image's last label is exactly `want` (or None): the prediction has the
    label's y and size and slides right in x; bisection on consecutive float32 centres, then a local scan"""
    H, W = b["hw"]
    g = R.geometry(b["hw"], b["shapes"][si])
    lab = np.float32([b["labels"][si][-1]])
    tb = R.target_boxes(lab, (H, W), g)
    x, y, w, h = lab[0, 1] * W, lab[0, 2] * H, lab[0, 3] * W, lab[0, 4] * H
    x, y, w, h = np.float32(x), np.float32(y), np.float32(w), np.float32(h)

    def iou_of(xs):
        xs = np.asarray(xs, np.float32)
        n = len(xs)
        pb = np.stack([xs - w / np.float32(2), np.full(n, y - h / np.float32(2), np.float32), xs + w / np.float32(2),
                       np.full(n, y + h / np.float32(2), np.float32)], 1).astype(np.float32)
        return R.box_iou(R._scale_clip(pb, g), tb)[:, 0]

    w0, h0 = w, h
    for dw in range(1024):                   # sizes a few float32 ulps apart until a centre gives the IoU exactly
        w = (np.float32(w0).view(np.int32) + np.int32(dw % 64)).view(np.float32)
        h = (np.float32(h0).view(np.int32) + np.int32(dw // 64)).view(np.float32)
        lo, hi = int(np.float32(x).view(np.int32)), int(np.float32(x + w).view(np.int32))
        while hi - lo > 1:                   # iou decreases from 1 (lo) to 0 (hi)
            mid = (lo + hi) // 2
            if iou_of([np.int32(mid).view(np.float32)])[0] > want:
                lo = mid
            else:
                hi = mid
        xs = np.arange(lo - 400, lo + 400, dtype=np.int64).astype(np.int32).view(np.float32)
        hit = np.flatnonzero(iou_of(xs) == want)
        if len(hit):
            return np.float32([xs[hit[0]], y, w, h])
    return None


def build_main():
    c = Case(3, 1)
    sh0 = [((600, 1000), ((0.416, 0.416), (0.5, 3.5))), ((230, 400), ((1.04, 1.04), (0.0, 8.4))), ((600, 1000), ((0.416, 0.416), (0.0, 3.0))),
           ((480, 800), ((0.52, 0.52), (0.0, 3.2))), ((480, 800), ((0.52, 0.52), (0.0, 3.2)))]
    b = c.batch((256, 416), sh0)
    # image 0: IoU probes at each iouv and one ulp either side, each against its own target, spread over a grid
    hits = 0
    k = 0
    for v in R.IOUV:
        for want in (np.nextafter(v, np.float32(0)), v, np.nextafter(v, np.float32(2))):
            cls = k % 2
            col, row = k % 6, k // 6
            box = [20 + col * 160, 20 + row * 115, 20 + col * 160 + 70, 20 + row * 115 + 60]
            add_label(b, 0, cls, box)
            p = probe(b, 0, cls, want)
            if p is not None:
                add_pred(c, b, 0, cls, p)
                hits += 1
            k += 1
    print("iou probes hit exactly:", hits, "of", k)
    # image 1: border clipping and zero-area boxes (class 2); gain 1.04
    add_label(b, 1, 2, [0, 50, 60, 110])
    add_pred(c, b, 1, 2, net_xywh([-12, 52, 58, 112], sh0[1]))                    # clipped at the left border, matches
    add_label(b, 1, 2, [200, 100, 200, 100])                                        # zero-area target
    add_pred(c, b, 1, 2, net_xywh([150, 150, 150, 150], sh0[1]))                    # zero-area prediction: NaN IoU wins, no match
    add_label(b, 1, 1, [330, 170, 400, 230])
    add_pred(c, b, 1, 1, net_xywh([335, 175, 420, 245], sh0[1]))                    # clipped at the right and bottom borders
    add_pred(c, b, 1, 1, net_xywh([420, 20, 440, 60], sh0[1]))                      # outside the frame: clipped to zero width
    add_label(b, 1, 0, [100, 20, 160, 80])
    add_pred(c, b, 1, 0, net_xywh([102, 22, 161, 79], sh0[1]))
    # image 2: two predictions with the same best target; the second's second-best target is free but it stays incorrect
    add_label(b, 2, 0, [100, 100, 200, 200])                                        # T1
    add_label(b, 2, 0, [100, 120, 200, 230])                                        # T2
    add_pred(c, b, 2, 0, net_xywh([100, 100, 200, 160], sh0[2]), conf=0.97)         # A: T1
    add_pred(c, b, 2, 0, net_xywh([100, 140, 200, 200], sh0[2]), conf=0.96)         # B: best T1 (taken), T2 second
    add_label(b, 2, 1, [500, 300, 600, 420])
    for j in range(6):
        add_pred(c, b, 2, 1, net_xywh([500 + 8 * j, 300 + 5 * j, 600 + 8 * j, 420 + 5 * j], sh0[2]))
    # image 3: labels, no predictions; image 4: predictions, no labels
    add_label(b, 3, 0, [10, 10, 100, 100])
    add_label(b, 3, 2, [300, 200, 400, 260])
    for j in range(5):
        add_pred(c, b, 4, j % 3, net_xywh([50 + 120 * j, 40, 150 + 120 * j, 140], sh0[4]))
    # batch 2: jittered predictions around random labels
    sh1 = [((480, 640), ((0.5, 0.5), (0.0, 40.0))), ((320, 320), ((1.0, 1.0), (0.0, 0.0))), ((500, 375), ((0.64, 0.64), (40.0, 0.0)))]
    b = c.batch((320, 320), sh1)
    for si, shp in enumerate(sh1):
        h0, w0 = shp[0]
        for _ in range(8):
            cls = int(c.rs.randint(3))
            bw, bh = c.rs.uniform(20, w0 / 3), c.rs.uniform(20, h0 / 3)
            x1, y1 = c.rs.uniform(-10, w0 - bw + 10), c.rs.uniform(-10, h0 - bh + 10)
            add_label(b, si, cls, [x1, y1, x1 + bw, y1 + bh])
            for _ in range(c.rs.randint(0, 4)):
                j = c.rs.normal(0, 0.12, 4) * [bw, bh, bw, bh]
                pc = cls if c.rs.rand() < 0.8 else int(c.rs.randint(3))
                add_pred(c, b, si, pc, net_xywh([x1 + j[0], y1 + j[1], x1 + bw + j[2], y1 + bh + j[3]], shp))
        for _ in range(4):
            x1, y1 = c.rs.uniform(0, w0 - 40), c.rs.uniform(0, h0 - 40)
            add_pred(c, b, si, int(c.rs.randint(3)), net_xywh([x1, y1, x1 + 40, y1 + 30], shp))
    return c


def build_single_cls():
    c = Case(1, 2)
    shapes = [((600, 1000), ((0.416, 0.416), (0.5, 3.5)))] * 4
    b = c.batch((256, 416), shapes)
    for si in range(4):
        for _ in range(5):
            bw, bh = c.rs.uniform(30, 200), c.rs.uniform(30, 150)
            x1, y1 = c.rs.uniform(0, 1000 - bw), c.rs.uniform(0, 600 - bh)
            add_label(b, si, 0, [x1, y1, x1 + bw, y1 + bh])
            for _ in range(c.rs.randint(0, 3)):
                j = c.rs.normal(0, 0.1, 4) * [bw, bh, bw, bh]
                add_pred(c, b, si, 0, net_xywh([x1 + j[0], y1 + j[1], x1 + bw + j[2], y1 + bh + j[3]], shapes[si]))
    return c


def build_no_tp():
    c = Case(3, 3)
    shapes = [((600, 1000), ((0.416, 0.416), (0.0, 3.0)))] * 3
    b = c.batch((256, 416), shapes)
    for si in range(3):
        add_label(b, si, si, [10, 10, 100, 100])
        add_pred(c, b, si, si, net_xywh([500, 300, 600, 400], shapes[si]))
        add_pred(c, b, si, (si + 1) % 3, net_xywh([12, 12, 100, 100], shapes[si]))
    return c


def tensors(c, b):
    """z (B, A, 5+nc) with one class per prediction row (cls prob 1, obj = conf) and collate_fn targets (n, 6)"""
    B = len(b["shapes"])
    z = np.zeros((B, A, 5 + c.nc), np.float32)
    z[:, :, 2:4] = 8.0
    for si, rows in enumerate(b["preds"]):
        assert len(rows) <= A
        for k, (xywh, cls, conf) in enumerate(rows):
            z[si, k, :4] = xywh
            z[si, k, 4] = conf
            z[si, k, 5 + cls] = 1.0
    t = [[si] + list(l) for si, ls in enumerate(b["labels"]) for l in ls]
    targets = np.array(t, np.float32).reshape(-1, 6)
    shp = np.array([[s[0][0], s[0][1], s[1][0][0], s[1][0][1], s[1][1][0], s[1][1][1]] for s in b["shapes"]], np.float64)
    return z, targets, shp


def run(ref_test, torch, c, single_cls):
    import torch.nn as nn
    zs = [tensors(c, b) for b in c.batches]

    class StandIn(nn.Module):
        def __init__(self):
            super().__init__()
            self.w = nn.Parameter(torch.zeros(1))
            self.names = [f"c{i}" for i in range(c.nc)]
            self.k = 0

        def forward(self, img, augment=False):
            z = torch.from_numpy(zs[self.k][0].copy())
            self.k += 1
            return [(z, None), None]

    loader = []
    for b, (z, t, _) in zip(c.batches, zs):
        H, W = b["hw"]
        loader.append((torch.zeros((len(b["shapes"]), 3, H, W), dtype=torch.uint8), torch.from_numpy(t.copy()),
                       [f"im{i}.jpg" for i in range(len(b["shapes"]))], b["shapes"]))
    calls = []
    orig = ref_test.ap_per_class

    def recording(tp, conf, pred_cls, target_cls, **kw):
        out = orig(tp, conf, pred_cls, target_cls, **kw)
        calls.append(((tp.copy(), conf.copy(), pred_cls.copy(), np.asarray(target_cls).copy()), out))
        return out

    ref_test.ap_per_class = recording
    try:
        with tempfile.TemporaryDirectory() as tmp:
            data = {"nc": c.nc, "val": tmp, "names": [f"c{i}" for i in range(c.nc)]}
            res, maps, _ = ref_test.test(data, batch_size=32, model=StandIn(), dataloader=loader, plots=False, single_cls=single_cls,
                                         compute_loss=None, half_precision=True)
    finally:
        ref_test.ap_per_class = orig
    return zs, calls, res, maps


def main():
    import torch
    ref_shims.import_reference()
    import test as ref_test      # the reference's test.py (sys.path set by import_reference)
    out, meta = {}, {}
    for name, builder, single in (("main", build_main, False), ("single_cls", build_single_cls, True), ("no_tp", build_no_tp, False)):
        c = builder()
        zs, calls, res, maps = run(ref_test, torch, c, single)
        for bi, (b, (z, t, shp)) in enumerate(zip(c.batches, zs)):
            out[f"{name}_z_{bi}"], out[f"{name}_targets_{bi}"], out[f"{name}_shapes_{bi}"] = z, t, shp
        assert len(calls) <= 1
        if calls:
            (tp, conf, pcls, tcls), (p, r, ap, f1, ap_class) = calls[0]
            for k, v in dict(correct=tp, conf=conf, pcls=pcls, tcls=tcls, p=p, r=r, ap=ap, f1=f1, ap_class=ap_class).items():
                out[f"{name}_{k}"] = np.asarray(v)
        out[f"{name}_results"] = np.array(res, np.float64)
        out[f"{name}_maps"] = np.asarray(maps, np.float64)
        meta[name] = dict(nc=c.nc, single_cls=single, hw=[list(b["hw"]) for b in c.batches], n_batches=len(c.batches), ap_called=bool(calls))
        print(name, "results", res, "TP rows", int(calls[0][0][0].any(1).sum()) if calls else 0)
    out["meta_json"] = np.frombuffer(json.dumps(meta).encode(), dtype=np.uint8)
    path = os.path.join(GOLD, "val_cases.npz")
    np.savez_compressed(path, **out)
    print("val cases", os.path.getsize(path) / 1e6, "MB")


if __name__ == "__main__":
    main()
