"""GPU: detection validation statistics on the device (DetectionStats, ap_per_class, test) against the unmodified reference's test()
(tests/golden/val_cases.npz) and the numpy restatement (oracle/restate_val.py) at full size, and seg_validation against the host formula.
Bit exact, no tolerance."""
import json
import os

import numpy as np
import pytest
import torch

from oracle import restate_val as R

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden", "val_cases.npz")


def _cases():
    z = np.load(GOLD)
    return z, json.loads(bytes(z["meta_json"]).decode())


def _shapes(rows):
    return [((int(s[0]), int(s[1])), ((float(s[2]), float(s[3])), (float(s[4]), float(s[5])))) for s in rows]


class StandIn(torch.nn.Module):
    """a model whose forward returns the fixture's z tensors in turn"""

    def __init__(self, zs, nc):
        super().__init__()
        self.w = torch.nn.Parameter(torch.zeros(1, device="cuda"))
        self.names = [f"c{i}" for i in range(nc)]
        self.zs, self.k = zs, 0

    def forward(self, img, augment=False):
        z = self.zs[self.k]
        self.k += 1
        return [(z, None), None]


@pytest.mark.parametrize("name", ["main", "single_cls", "no_tp"])
def test_fixture_statistics_bit_exact(name):
    from multiyolov5_b200.test import test
    from multiyolov5_b200.utils.general import non_max_suppression
    from multiyolov5_b200.utils.metrics import DetectionStats
    z, meta = _cases()
    m = meta[name]
    st = DetectionStats(max_det=300, capacity=2)                 # grows while the batches arrive
    zs, loader = [], []
    for bi in range(m["n_batches"]):
        zz = torch.from_numpy(z[f"{name}_z_{bi}"]).cuda()
        tg = torch.from_numpy(z[f"{name}_targets_{bi}"])
        shp = _shapes(z[f"{name}_shapes_{bi}"])
        dets, cnt = non_max_suppression(zz, 0.001, 0.6, multi_label=True, return_padded=True)
        st.update(dets, cnt, tg if bi % 2 else tg.cuda(), tuple(m["hw"][bi]), shp)
        zs.append(zz)
        H, W = m["hw"][bi]
        loader.append((torch.zeros((len(shp), 3, H, W), dtype=torch.uint8), tg, [f"im{i}.jpg" for i in range(len(shp))], shp))
    p, r, ap, f1, ap_class, nt, seen = st.compute(m["nc"])
    assert seen == sum(len(z[f"{name}_shapes_{bi}"]) for bi in range(m["n_batches"]))
    if m["ap_called"]:
        correct, conf, pcls = st.correct_rows()
        assert np.array_equal(correct, z[f"{name}_correct"])
        assert np.array_equal(conf, z[f"{name}_conf"]) and np.array_equal(pcls, z[f"{name}_pcls"])
        for k, v in dict(p=p, r=r, ap=ap, f1=f1, ap_class=ap_class).items():
            ref = z[f"{name}_{k}"]
            assert v.dtype == ref.dtype and np.array_equal(v, ref), k
        assert np.array_equal(nt, np.bincount(z[f"{name}_tcls"].astype(np.int64), minlength=m["nc"]))
    else:
        assert len(ap_class) == 0 and p == 0.
    res, maps, t = test({"nc": m["nc"]}, model=StandIn(zs, m["nc"]), dataloader=loader, plots=False, single_cls=m["single_cls"],
                        half_precision=False)
    assert np.array_equal(np.array(res[:4], np.float64), z[f"{name}_results"][:4]) and list(res[4:]) == [0.0, 0.0, 0.0]
    assert np.array_equal(maps, z[f"{name}_maps"])
    assert len(t) == 6 and all(v >= 0 for v in t[:3])


def synth_batch(rs, B, nc=10, nl=20, max_det=300, hw=(320, 512), ties=False):
    """padded NMS-like rows jittered around random labels plus edge cases: clipped boxes, zero-area boxes, duplicate hits"""
    H, W = hw
    shapes, tg = [], []
    dets = np.zeros((B, max_det, 6), np.float32)
    counts = np.zeros(B, np.int32)
    for si in range(B):
        h0, w0 = int(rs.randint(200, 900)), int(rs.randint(300, 1400))
        gain = min(H / h0, W / w0)
        padw, padh = (W - w0 * gain) / 2, (H - h0 * gain) / 2
        shapes.append(((h0, w0), ((gain, gain), (padw, padh))))
        n_l = int(rs.randint(0, nl + 1))
        lab = np.zeros((n_l, 6), np.float32)
        lab[:, 0] = si
        lab[:, 1] = rs.randint(0, nc, n_l)
        lab[:, 2:4] = rs.uniform(0.0, 1.0, (n_l, 2))
        lab[:, 4:6] = rs.uniform(0.0, 0.4, (n_l, 2))
        lab[rs.rand(n_l) < 0.05, 4:6] = 0.0                         # zero-area targets
        tg.append(lab)
        n = int(rs.randint(0, max_det + 1)) if rs.rand() > 0.1 else 0
        rows = np.zeros((n, 6), np.float32)
        for k in range(n):
            if n_l and rs.rand() < 0.7:
                t = lab[rs.randint(n_l)]
                x, y, w, h = t[2] * W, t[3] * H, t[4] * W, t[5] * H
                j = rs.normal(0, 0.15, 4)
                x, y, w, h = x + j[0] * w, y + j[1] * h, w * (1 + j[2]), h * (1 + j[3])
                c = t[1] if rs.rand() < 0.85 else rs.randint(nc)
            else:
                x, y, w, h = rs.uniform(-20, W + 20), rs.uniform(-20, H + 20), rs.uniform(0, W / 3), rs.uniform(0, H / 3)
                c = rs.randint(nc)
            if rs.rand() < 0.03:
                w = h = 0.0
            rows[k] = [x - w / 2, y - h / 2, x + w / 2, y + h / 2, 0.0, c]
        conf = rs.uniform(0.001, 1.0, n).astype(np.float32)
        if ties:
            conf = np.round(conf * 50) / np.float32(50) + np.float32(0.001)
        rows[:, 4] = -np.sort(-conf)
        dets[si, :n] = rows
        counts[si] = n
    return dets, counts, np.concatenate(tg, 0), shapes


def restated(batches, hw, nc=10):
    stats = []
    for dets, counts, tg, shapes in batches:
        for si in range(len(shapes)):
            d = dets[si, :counts[si]]
            labels = tg[tg[:, 0] == si, 1:]
            g = R.geometry(hw, shapes[si])
            if len(d) == 0:
                if len(labels):
                    stats.append((np.zeros((0, 10), bool), np.zeros(0, np.float32), np.zeros(0, np.float32), labels[:, 0]))
                continue
            stats.append((R.match_image(d, labels, hw, g), d[:, 4], d[:, 5], labels[:, 0]))
    return [np.concatenate(x, 0) for x in zip(*stats)]


def device_stats(batches, hw, nc=10):
    from multiyolov5_b200.utils.metrics import DetectionStats
    st = DetectionStats(max_det=300)
    for dets, counts, tg, shapes in batches:
        st.update(torch.from_numpy(dets).cuda(), torch.from_numpy(counts).cuda(), torch.from_numpy(tg).cuda(), hw, shapes)
    return st, st.compute(nc)


@pytest.mark.parametrize("n_images,ties", [(500, False), (500, True), (5000, False)])
def test_full_size_against_restatement(n_images, ties):
    rs = np.random.RandomState(n_images + ties)
    hw = (320, 512)
    batches = [synth_batch(rs, min(32, n_images - b), hw=hw, ties=ties) for b in range(0, n_images, 32)]
    st, (p, r, ap, f1, ap_class, nt, seen) = device_stats(batches, hw)
    ref = restated(batches, hw)
    correct, conf, pcls = st.correct_rows()
    assert np.array_equal(correct, ref[0]) and np.array_equal(conf, ref[1]) and np.array_equal(pcls, ref[2])
    rp, rr, rap, rf1, rcls = R.ap_per_class(*ref)
    for a, b in ((p, rp), (r, rr), (ap, rap), (f1, rf1), (ap_class, rcls)):
        assert np.array_equal(a, b)
    assert np.array_equal(nt, np.bincount(ref[3].astype(np.int64), minlength=10)) and seen == n_images


def test_batch_independence():
    rs = np.random.RandomState(3)
    hw = (320, 512)
    dets, counts, tg, shapes = synth_batch(rs, 64, hw=hw)
    outs = []
    for bs in (1, 7, 32):
        batches = []
        for b in range(0, 64, bs):
            sel = (tg[:, 0] >= b) & (tg[:, 0] < b + bs)
            t = tg[sel].copy()
            t[:, 0] -= b
            batches.append((dets[b:b + bs], counts[b:b + bs], t, shapes[b:b + bs]))
        outs.append(device_stats(batches, hw))
    for st, res in outs[1:]:
        assert np.array_equal(st.correct_rows()[0], outs[0][0].correct_rows()[0])
        for a, b in zip(res[:5], outs[0][1][:5]):
            assert np.array_equal(a, b)


def test_ap_per_class_host_inputs():
    from multiyolov5_b200.utils.metrics import ap_per_class
    rs = np.random.RandomState(4)
    for n, ncol in ((1, 10), (700, 10), (20000, 1), (3000, 16)):
        tp = rs.rand(n, ncol) < np.linspace(0.7, 0.1, ncol)
        conf = rs.uniform(0, 1, n).astype(np.float32)
        pcls = rs.randint(0, 5, n).astype(np.float64)
        tcls = rs.randint(0, 6, 300).astype(np.float64)
        out = ap_per_class(tp, conf, pcls, tcls)
        ref = R.ap_per_class(tp, conf, pcls, tcls)
        for a, b in zip(out, ref):
            assert np.array_equal(a, b)
        out_t = ap_per_class(torch.from_numpy(tp), torch.from_numpy(conf), torch.from_numpy(pcls), torch.from_numpy(tcls))
        for a, b in zip(out_t, ref):
            assert np.array_equal(a, b)


def test_out_of_range_class_raises():
    from multiyolov5_b200.utils.metrics import DetectionStats
    st = DetectionStats(max_det=300)
    dets = torch.zeros((1, 300, 6), device="cuda")
    cnt = torch.zeros(1, dtype=torch.int32, device="cuda")
    st.update(dets, cnt, torch.tensor([[0, 2.5, 0.5, 0.5, 0.1, 0.1]]), (64, 64), [((64, 64), None)])
    with pytest.raises(ValueError):
        st.compute(3)
    st = DetectionStats(max_det=300)
    st.update(dets, cnt, torch.tensor([[0, 3, 0.5, 0.5, 0.1, 0.1]]), (64, 64), [((64, 64), None)])
    with pytest.raises(ValueError):
        st.compute(3)
    st.compute(4)


def _psp_model():
    from multiyolov5_b200.models.yolo import Model
    from oracle import synth
    yml = "yolov5s_city_seg.yaml"
    cfg = synth.load_cfg(yml)
    model = Model(yml)
    model.load_state_dict(synth.synth_state_dict(synth.load_manifest("s_psp"), cfg, seed=1))
    return model.cuda().eval(), cfg


def test_test_with_model_half():
    from multiyolov5_b200.test import test
    from multiyolov5_b200.train import scale_hyp
    from multiyolov5_b200.utils.general import non_max_suppression
    from multiyolov5_b200.utils.loss import FusedComputeLoss
    model, cfg = _psp_model()
    hyp = dict(lr0=0.01, momentum=0.937, weight_decay=5e-4, box=0.05, cls=0.5, cls_pw=1.0, obj=1.0, obj_pw=1.0, anchor_t=4.0, fl_gamma=0.0)
    model.hyp, model.gr = scale_hyp(hyp, nl=3, nc=cfg["nc"], imgsz=256, total_batch_size=4), 1.0
    g = torch.Generator().manual_seed(0)
    H, W = 256, 320
    loader = []
    model.half()
    for b in range(3):
        img = torch.randint(0, 256, (4, 3, H, W), dtype=torch.uint8, generator=g)
        shapes = [((H * 2, W * 2), ((0.5, 0.5), (0.0, 0.0)))] * 4
        with torch.no_grad():
            out = model(img.cuda().half() / 255.0)[0][0]
        dets = non_max_suppression(out, 0.001, 0.6, multi_label=True)
        tg = []
        for si, d in enumerate(dets):            # labels near some of the model's own boxes, so that some predictions are correct
            d = d[:12].cpu().numpy()
            xywh = np.stack([(d[:, 0] + d[:, 2]) / 2 / W, (d[:, 1] + d[:, 3]) / 2 / H, (d[:, 2] - d[:, 0]) / W, (d[:, 3] - d[:, 1]) / H], 1)
            tg.append(np.concatenate([np.full((len(d), 1), si), d[:, 5:6], xywh * np.float32(1.02)], 1))
        loader.append((img, torch.from_numpy(np.concatenate(tg, 0).astype(np.float32)), [""] * 4, shapes))
    model.float()
    res, maps, t = test({"nc": cfg["nc"]}, model=model, dataloader=loader, plots=False, compute_loss=FusedComputeLoss(model))
    assert next(model.parameters()).dtype == torch.float32 and len(res) == 7 and maps.shape == (cfg["nc"],) and len(t) == 6
    assert all(np.isfinite(v) for v in res[4:]) and res[4] > 0
    # the restated statistics of the same NMS rows (the model in half mode, as test() runs it)
    model.half()
    batches = []
    for img, tg, _, shapes in loader:
        with torch.no_grad():
            out = model(img.cuda().half() / 255.0)[0][0]
        d, c = non_max_suppression(out, 0.001, 0.6, multi_label=True, return_padded=True)
        batches.append((d.cpu().numpy(), c.cpu().numpy(), tg.numpy(), shapes))
    model.float()
    ref = R.test_statistics(_restated_stats(batches, (H, W)), cfg["nc"])
    assert ref["map50"] > 0
    assert np.array_equal(np.array(res[:4], np.float64), np.array([ref["mp"], ref["mr"], ref["map50"], ref["map"]], np.float64))
    assert np.array_equal(maps, ref["maps"])


def _restated_stats(batches, hw):
    stats = []
    for dets, counts, tg, shapes in batches:
        for si in range(len(shapes)):
            d = dets[si, :counts[si]]
            labels = tg[tg[:, 0] == si, 1:]
            if len(d) == 0:
                if len(labels):
                    stats.append((np.zeros((0, 10), bool), np.zeros(0, np.float32), np.zeros(0, np.float32), labels[:, 0]))
                continue
            stats.append((R.match_image(d, labels, hw, R.geometry(hw, shapes[si])), d[:, 4], d[:, 5], labels[:, 0]))
    return stats


def test_seg_validation_matches_host_formula():
    from multiyolov5_b200.test import seg_validation
    from multiyolov5_b200.utils.datasets import DeviceSegCache, SegAugmenter
    from multiyolov5_b200.utils.metrics import seg_eval_batch
    rs = np.random.RandomState(5)
    imgs = [rs.randint(0, 256, (256, 512, 3)).astype(np.uint8) for _ in range(3)]
    masks = [rs.choice(np.concatenate([np.arange(34), [255]]), (256, 512)).astype(np.uint8) for _ in range(3)]
    aug = SegAugmenter(DeviceSegCache(imgs, masks, mask_map="cityscapes"), base_size=256, crop_size=(256, 128), preset="citys")
    loader = [aug.testval([i]) for i in range(3)]
    model, _ = _psp_model()
    miou = seg_validation(model, 19, loader, torch.device("cuda"))
    assert isinstance(miou, np.float64)
    model.half()
    tot_i, tot_u = 0, 0
    for image, target in loader:
        with torch.no_grad():
            seg = model(image.half())[1]
        _, _, inter, union = seg_eval_batch(seg, target, 19)
        tot_i, tot_u = tot_i + inter, tot_u + union
    model.float()
    assert miou == (1.0 * tot_i / (np.spacing(1) + tot_u)).mean()
