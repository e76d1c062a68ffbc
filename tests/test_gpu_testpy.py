"""GPU: the --save-hybrid NMS (myolo_nms_labels) and the confusion matrix (myolo_confusion_update) against the unmodified reference
(tests/golden/testpy_cases.npz, oracle/make_golden_testpy.py), against the plain NMS kernel over z with the labels appended as rows,
and against the numpy restatement of process_batch (oracle/restate_confusion.py); test()'s new options against the composition of
the public functions.  Bit exact, no tolerance."""
import json
import os

import numpy as np
import pytest
import torch

from oracle import restate_confusion as RC
from tests.test_testpy_host import GOLD, nms_case

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("name", [str(n) for n in GOLD["nms_names"]])
def test_hybrid_nms_fixture(name):
    from multiyolov5_b200.utils.general import NmsLabels, non_max_suppression
    z, nc, kw, labels, outs = nms_case(name)
    zc = torch.from_numpy(z).cuda()
    got = non_max_suppression(zc, labels=[torch.from_numpy(l).cuda() for l in labels], **kw)
    for g, o in zip(got, outs):
        assert np.array_equal(g.cpu().numpy(), o)
    lab = NmsLabels.from_list(labels, nc, "cuda")
    dets, cnt = non_max_suppression(zc, labels=lab, return_padded=True, **kw)
    lab.check()
    for b, o in enumerate(outs):
        assert int(cnt[b]) == len(o) and np.array_equal(dets[b, :len(o)].cpu().numpy(), o)


def _appended(z, labels, nc):
    """z with each image's labels as rows A .. A + k_b - 1 (obj 1, one-hot), padded with obj 0 rows to a common length"""
    B, A, no = z.shape
    kmax = max(len(l) for l in labels)
    out = torch.zeros((B, A + kmax, no), device=z.device)
    out[:, :A] = z
    for b, l in enumerate(labels):
        if len(l):
            out[b, A:A + len(l)] = torch.from_numpy(RC.label_rows(l, nc)).cuda()
    return out


@pytest.mark.parametrize("A", [32256, 71316])
@pytest.mark.parametrize("kw", [dict(conf_thres=0.001, iou_thres=0.6, multi_label=True), dict(conf_thres=0.25, iou_thres=0.45),
                                dict(conf_thres=0.001, iou_thres=0.6, multi_label=True, classes=[1, 3, 5], agnostic=True)])
def test_hybrid_nms_equals_appended_rows(A, kw):
    from multiyolov5_b200.utils.general import NmsLabels, non_max_suppression
    B, nc = 32, 8
    g = torch.Generator(device="cuda").manual_seed(A + int(kw["conf_thres"] * 100))
    z = torch.rand((B, A, 5 + nc), device="cuda", generator=g)
    z[..., :2] *= 1024
    z[..., 2:4] = z[..., 2:4] * 120 + 2
    z[..., 4] = z[..., 4] ** 3
    rs = np.random.RandomState(A)
    labels = []
    for b in range(B):
        k = [0, 200, 1][b % 3] if b else 0
        k = rs.randint(0, 201) if b >= 3 else k
        l = np.zeros((k, 5), np.float32)
        l[:, 0] = rs.randint(0, nc, k)
        l[:, 1:3] = rs.uniform(0, 1024, (k, 2))
        l[:, 3:5] = rs.uniform(2, 120, (k, 2))
        if k > 2:
            l[1] = l[0]                                            # a duplicate label
            src = z[b, rs.randint(A)].cpu().numpy()                # a label on a prediction
            l[2, 1:5] = src[:4]
        labels.append(l)
    ref_d, ref_c = non_max_suppression(_appended(z, labels, nc), return_padded=True, **kw)
    got_d, got_c = non_max_suppression(z, labels=NmsLabels.from_list(labels, nc, "cuda"), return_padded=True, **kw)
    assert torch.equal(got_c, ref_c)
    for b in range(B):
        n = int(ref_c[b])
        assert torch.equal(got_d[b, :n], ref_d[b, :n]), b


def test_hybrid_nms_bad_class_and_conf1():
    from multiyolov5_b200.utils.general import NmsLabels, non_max_suppression
    z = torch.rand((2, 500, 8), device="cuda")
    lab = NmsLabels(torch.tensor([[1., 5, 5, 4, 4], [3., 9, 9, 4, 4]], device="cuda"), torch.tensor([0, 1, 2], device="cuda"), 2)
    non_max_suppression(z, 0.1, 0.5, labels=lab, return_padded=True)
    with pytest.raises(ValueError, match="class"):
        lab.check()
    with pytest.raises(ValueError):
        non_max_suppression(z, labels=[np.float32([[3, 5, 5, 4, 4]]), np.zeros((0, 5), np.float32)])
    out = non_max_suppression(z * 0.5, 1.0, 0.5, labels=[np.float32([[1, 5, 5, 4, 4]]), np.zeros((0, 5), np.float32)])
    assert all(len(o) == 0 for o in out)


@pytest.mark.parametrize("name", [str(n) for n in GOLD["cm_names"]])
def test_confusion_fixture(name):
    from multiyolov5_b200.utils.metrics import ConfusionMatrix
    n, nc = (int(v) for v in GOLD[f"cm_{name}_n"])
    cm = ConfusionMatrix(nc)
    for k in range(n):
        cm.process_batch(torch.from_numpy(GOLD[f"cm_{name}_det{k}"]).cuda(), torch.from_numpy(GOLD[f"cm_{name}_lab{k}"]).cuda())
        assert np.array_equal(cm.matrix, GOLD[f"cm_{name}_matrix{k}"]), k


def _native(dets, targets, hw, shapes):
    """test.py:194-195,223-224 with the public host functions: per image native-space predn and labelsn"""
    from multiyolov5_b200.utils.general import scale_coords, xywh2xyxy
    H, W = hw
    out = []
    for si, d in enumerate(dets):
        lab = targets[targets[:, 0] == si, 1:].clone()
        lab[:, 1:] *= torch.tensor([W, H, W, H], dtype=torch.float32)
        predn = d.cpu().clone()
        scale_coords((H, W), predn[:, :4], shapes[si][0], shapes[si][1])
        tbox = xywh2xyxy(lab[:, 1:5])
        scale_coords((H, W), tbox, shapes[si][0], shapes[si][1])
        out.append((predn.numpy(), torch.cat([lab[:, :1], tbox], 1).numpy()))
    return out


@pytest.mark.parametrize("nc", [10, 80])
def test_confusion_update_random(nc):
    from multiyolov5_b200.utils.metrics import ConfusionMatrix
    rs = np.random.RandomState(nc)
    cm = ConfusionMatrix(nc)
    ref = np.zeros((nc + 1, nc + 1))
    for batch in range(3):
        B, H, W, max_det = 8, 384, 640, 300
        shapes = [((int(h0), int(w0)), ((g, g), (float(pw), float(ph))))
                  for h0, w0, g, pw, ph in zip(rs.randint(200, 800, B), rs.randint(300, 1200, B), rs.uniform(0.4, 1.2, B),
                                               rs.uniform(0, 40, B), rs.uniform(0, 30, B))]
        tg, dets, counts = [], torch.zeros((B, max_det, 6)), torch.zeros(B, dtype=torch.int32)
        for b in range(B):
            nl = [0, 100, 5][b % 3] if b < 3 else rs.randint(0, 101)
            n = [300, 0, 300][b % 3] if b < 3 else rs.randint(0, 301)
            lab = np.zeros((nl, 6), np.float32)
            lab[:, 0], lab[:, 1] = b, rs.randint(0, nc, nl)
            lab[:, 2:4] = rs.uniform(0.05, 0.95, (nl, 2))
            lab[:, 4:6] = rs.uniform(0.02, 0.3, (nl, 2))
            tg.append(lab)
            src = rs.randint(0, max(nl, 1), n)
            c = lab[src, 2:6] * np.float32([W, H, W, H]) if nl else rs.uniform(10, 300, (n, 4)).astype(np.float32)
            c = c + rs.uniform(-8, 8, (n, 4)).astype(np.float32)
            d = np.zeros((n, 6), np.float32)
            d[:, :2], d[:, 2:4] = c[:, :2] - c[:, 2:4] / 2, c[:, :2] + c[:, 2:4] / 2
            d[:, 4] = np.sort(rs.uniform(0.01, 1, n))[::-1]
            d[:, 5] = np.where(rs.rand(n) < 0.7, lab[src, 1] if nl else 0, rs.randint(0, nc, n))
            dets[b, :n] = torch.from_numpy(d)
            counts[b] = n
        targets = torch.from_numpy(np.concatenate(tg))
        cm.update(dets.cuda(), counts.cuda(), targets.cuda(), (H, W), shapes)
        for (predn, labn) in _native([dets[b, :counts[b]] for b in range(B)], targets, (H, W), shapes):
            if len(labn) and len(predn):
                RC.process_batch(ref, predn, labn, nc)
        assert np.array_equal(cm.matrix, ref), batch
    assert ref[:nc, :nc].trace() > 0 and ref[nc].sum() > 0 and ref[:, nc].sum() > 0


class StandIn(torch.nn.Module):
    """a model whose forward returns given z tensors in turn"""

    def __init__(self, zs, nc):
        super().__init__()
        self.w = torch.nn.Parameter(torch.zeros(1, device="cuda"))
        self.names = [f"c{i}" for i in range(nc)]
        self.zs, self.k, self.augment = zs, 0, []

    def forward(self, img, augment=False):
        self.augment.append(augment)
        z = self.zs[self.k]
        self.k += 1
        return [(z, None), None]


def _val_case():
    from tests.test_gpu_val import _cases, _shapes
    z, meta = _cases()
    m = meta["main"]
    zs, loader = [], []
    for bi in range(m["n_batches"]):
        zs.append(torch.from_numpy(z[f"main_z_{bi}"]).cuda())
        tg = torch.from_numpy(z[f"main_targets_{bi}"])
        shp = _shapes(z[f"main_shapes_{bi}"])
        H, W = m["hw"][bi]
        loader.append((torch.zeros((len(shp), 3, H, W), dtype=torch.uint8), tg, [f"{bi}{i}.jpg" if i else f"im{bi}.jpg"
                                                                                     for i in range(len(shp))], shp))
    return zs, loader, m


def test_test_flags_against_composition(tmp_path, monkeypatch):
    from multiyolov5_b200 import test as T
    from multiyolov5_b200.utils.general import NmsLabels, non_max_suppression, xyxy2xywh
    from multiyolov5_b200.utils.metrics import DetectionStats
    zs, loader, m = _val_case()
    nc = m["nc"]
    seen = {}
    monkeypatch.setattr(T.ConfusionMatrix, "plot", lambda self, save_dir="", names=(): seen.setdefault("m", self.matrix))
    model = StandIn(zs, nc)
    res = T.test({"nc": nc}, weights="best.pt", model=model, dataloader=loader, save_dir=tmp_path, save_txt=True, save_conf=True,
                 save_json=True, save_hybrid=True, plots=True, augment=True, half_precision=False, is_coco=True)
    assert model.augment == [True] * len(zs)
    # the composition: list-form NMS with labels, DetectionStats, per-image native rows, the reference's statements on the host
    st = DetectionStats()
    ref = np.zeros((nc + 1, nc + 1))
    jdict, txt = [], {}
    coco91 = T.coco80_to_coco91_class()
    for z, (img, tg, paths, shapes) in zip(zs, loader):
        H, W = img.shape[2:]
        lb = tg.clone()
        lb[:, 2:] *= torch.tensor([W, H, W, H], dtype=torch.float32)
        out = non_max_suppression(z, 0.001, 0.6, multi_label=True, labels=[lb[lb[:, 0] == i, 1:] for i in range(len(paths))])
        d, c = torch.zeros((len(paths), 300, 6), device="cuda"), torch.tensor([len(o) for o in out], dtype=torch.int32)
        for i, o in enumerate(out):
            d[i, :len(o)] = o
        st.update(d, c.cuda(), tg, (H, W), shapes)
        for si, (predn, labn) in enumerate(_native(out, tg, (H, W), shapes)):
            if not len(predn):
                continue
            from pathlib import Path
            stem = Path(paths[si]).stem
            gn = torch.tensor(shapes[si][0])[[1, 0, 1, 0]]
            for *xyxy, conf, cls in predn.tolist():
                xywh = (xyxy2xywh(torch.tensor(xyxy).view(1, 4)) / gn).view(-1).tolist()
                line = (cls, *xywh, conf)
                txt[stem] = txt.get(stem, "") + ("%g " * len(line)).rstrip() % line + "\n"
            box = xyxy2xywh(torch.from_numpy(predn[:, :4]))
            box[:, :2] -= box[:, 2:] / 2
            image_id = int(stem) if stem.isnumeric() else stem
            for p, b in zip(out[si].tolist(), box.tolist()):
                jdict.append({"image_id": image_id, "category_id": coco91[int(p[5])], "bbox": [round(x, 3) for x in b],
                              "score": round(p[4], 5)})
            if len(labn):
                RC.process_batch(ref, predn, labn, nc)
    p, r, ap, f1, ap_class, nt, nseen = st.compute(nc)
    ap50, ap = ap[:, 0], ap.mean(1)
    assert res[0][:4] == (p.mean(), r.mean(), ap50.mean(), ap.mean())
    assert np.array_equal(seen["m"], ref)
    files = sorted(os.listdir(tmp_path / "labels"))
    assert files == sorted(f"{k}.txt" for k in txt)
    for k, v in txt.items():
        assert (tmp_path / "labels" / f"{k}.txt").read_text() == v
    assert (tmp_path / "best_predictions.json").read_text() == json.dumps(jdict)
    with pytest.raises(ValueError):
        T.test({"nc": nc}, model=StandIn(zs, nc), dataloader=loader, augment=True, compute_loss=lambda *a: None, plots=False)


@pytest.mark.parametrize("name", [str(n) for n in GOLD["run_names"]])
def test_test_options_match_reference(name, tmp_path, monkeypatch, capsys):
    """test() with each option set reproduces the unmodified reference's run over the same z (oracle/make_golden_testpy.py RUN_CASES):
    every file under save_dir byte for byte, stdout, the returned results and maps, and the matrix handed to plot().  The header row
    the reference shows in its tqdm bar on stderr is printed to stdout here, so stdout is compared after it."""
    from multiyolov5_b200 import test as T
    from oracle.make_golden_testpy import RUN_CASES, run_paths, val_main
    kw = dict(RUN_CASES[name])
    batches, hws, nc = val_main(kw.pop("case", "main"))
    loader = [(torch.zeros((len(shp), 3, H, W), dtype=torch.uint8), torch.from_numpy(t.copy()), run_paths(bi, len(shp)), shp)
              for bi, ((z, t, shp), (H, W)) in enumerate(zip(batches, hws))]
    seen = {}
    monkeypatch.setattr(T.ConfusionMatrix, "plot", lambda self, save_dir="", names=(): seen.setdefault("m", self.matrix))
    save_dir = tmp_path / "exp"
    save_dir.mkdir()
    capsys.readouterr()
    res, maps, _ = T.test({"nc": nc}, model=StandIn([torch.from_numpy(z).cuda() for z, _, _ in batches], nc), dataloader=loader,
                          save_dir=save_dir, half_precision=True, **{"plots": False, **kw})
    out = capsys.readouterr().out.split("\n", 1)[1].replace(str(save_dir), "<save_dir>")
    p = f"run_{name}_"
    assert out == bytes(GOLD[p + "stdout"]).decode()
    assert np.array_equal(np.array(res, np.float64), GOLD[p + "results"])
    assert np.array_equal(np.asarray(maps, np.float64), GOLD[p + "maps"])
    want = [str(f) for f in GOLD[p + "files"]]
    got = sorted(str(f.relative_to(save_dir)) for f in save_dir.rglob("*") if f.is_file())
    assert got == want
    for k, f in enumerate(want):
        assert (save_dir / f).read_bytes() == bytes(GOLD[p + f"file{k}"]), f
    if p + "matrix" in GOLD:
        assert np.array_equal(seen["m"], GOLD[p + "matrix"])
    else:
        assert "m" not in seen


def test_confusion_plot_and_errors(tmp_path):
    """plot() draws nothing without seaborn and matplotlib, but a bad class id still raises before the drawing; limits raise"""
    from multiyolov5_b200.utils.metrics import ConfusionMatrix
    cm = ConfusionMatrix(2)
    cm.process_batch(torch.tensor([[0., 0, 10, 10, 0.9, 1]]), torch.tensor([[1., 0, 0, 10, 10]]))
    cm.plot(save_dir=tmp_path)
    try:
        import matplotlib  # noqa: F401
        import seaborn  # noqa: F401
    except ImportError:
        assert not (tmp_path / "confusion_matrix.png").exists()
    cm.process_batch(torch.tensor([[0., 0, 10, 10, 0.9, 1]]), torch.tensor([[2., 0, 0, 10, 10]]))
    with pytest.raises(ValueError, match="label class"):
        cm.plot(save_dir=tmp_path)
    with pytest.raises(ValueError):
        ConfusionMatrix(2).process_batch(torch.zeros((1025, 6)), torch.zeros((1, 5)))


def test_hybrid_nms_label_count_bound():
    """an image with more labels than max_labels sets the count bit, also when max_labels is 0"""
    from multiyolov5_b200.utils.general import NmsLabels, non_max_suppression
    z = torch.rand((2, 300, 8), device="cuda")
    rows = torch.tensor([[1., 5, 5, 4, 4], [2., 9, 9, 4, 4]], device="cuda")
    for bound in (0, 1):
        lab = NmsLabels(rows, torch.tensor([0, 2, 2], device="cuda"), bound)
        non_max_suppression(z, 0.1, 0.5, labels=lab, return_padded=True)
        with pytest.raises(ValueError, match="max_labels"):
            lab.check()
