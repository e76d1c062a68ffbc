"""TEST INFRASTRUCTURE - generates tests/golden/testpy_cases.npz by running the UNMODIFIED reference's
`non_max_suppression(..., labels=lb)` (utils/general.py:421-509, the autolabelling of test.py --save-hybrid) and the fork's
`ConfusionMatrix.process_batch` (utils/metrics.py:115-162) on the CPU (through oracle/ref_shims.py).

    MYOLO_REFERENCE_ROOT=<checkout> python oracle/make_golden_testpy.py

z is not stored: every case rebuilds it from its seed with `make_z` (numpy's RandomState, so the bytes are the same everywhere).
NMS cases (`nms_<k>_*`): the settings, the per-image labels (k, 5) [cls, x, y, w, h] in pixels, and the reference's rows per image.
  multi      nc 4, multi-label at conf 0.001: labels coinciding with predictions, duplicate labels, an image whose z has no candidate
             but has labels, an image without labels
  best       the same z and labels, best class at conf 0.25
  classes    multi-label with classes=[0, 2]
  nc1        nc 1 (multi-label off, as at :440)
  conf1      conf_thres 1.0: the labels drop out as well
  maxnms     nc 4 at obj 1 with distinct class scores: 32 000 candidates plus one label, more than max_nms = 30 000
Candidate scores are distinct within an image (re-drawn otherwise), so the reference's unstable sorts have no ties to break.  The
labels' score 1.0 ties among labels; below max_nms torchvision's stable sort keeps their order, above it the reference's unstable
argsort would not, so the max_nms case has a single label.
Confusion cases (`cm_<k>_*`): a sequence of process_batch calls (detections (N, 6) and labels (M, 5) per call) and the matrix after
each call.  They put IoU exactly at 0.45 and conf exactly at 0.25 and one float32 ulp either side, one label claimed by several
detections and one detection overlapping several labels, no matches, all detections below conf, and random images whose IoUs above
the threshold are distinct.
test() cases (`run_<k>_*`): the unmodified reference's test() with a stand-in model whose forward returns the stored z of the `main`
case of tests/golden/val_cases.npz (two batches, nc 3; `hybrid` takes the `single_cls` case, see below), over a list loader of its targets and shapes with the paths `RUN_PATHS`
(numeric and non-numeric stems), once per option set in `RUN_CASES`.  Recorded: every file written under save_dir (name and bytes),
stdout with save_dir written as <save_dir>, the returned (mp, mr, map50, map, *loss) and maps, and, with plots, the matrix handed to
ConfusionMatrix.plot.  The recording wraps names in the imported test module's namespace (its source is untouched): ConfusionMatrix
by a subclass whose plot() keeps the matrix, ap_per_class with plot=False (the PR curves need the real matplotlib), plot_images by a
no-op.  The reference only makes save_dir/labels for a run that loads its own model, so the generator makes it for save_txt.
With --save-hybrid every label becomes a row of conf 1.0, so rows of one class tie in ap_per_class, whose np.argsort is not stable; the
`main` case has a zero-area target whose label row is not correct (NaN IoU), which makes the tie order matter.  The `hybrid` run uses the
`single_cls` case, whose label rows are all correct, so any order of the ties gives the same statistics.
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
from oracle import ref_shims  # noqa: E402

GOLD = os.path.join(HERE, "..", "tests", "golden")


def make_z(seed, B, A, nc, distinct=False):
    """(B, A, 5 + nc) float32 predictions in a 512 x 512 input.  distinct: obj 1 and class scores distinct multiples of 2^-16."""
    rs = np.random.RandomState(seed)
    z = np.zeros((B, A, 5 + nc), np.float32)
    z[..., 0:2] = rs.uniform(0, 512, (B, A, 2))
    z[..., 2:4] = rs.uniform(4, 96, (B, A, 2))
    if distinct:
        z[..., 4] = 1.0
        for b in range(B):
            z[b, :, 5:] = ((rs.permutation(65000)[:A * nc] + 100) / 65536.0).reshape(A, nc)
    else:
        z[..., 4] = rs.uniform(0, 1, (B, A)) ** 2
        z[..., 5:] = rs.uniform(0, 1, (B, A, nc))
    return z


def scores_distinct(z, conf):
    for b in range(z.shape[0]):
        s = (z[b, :, 5:] * z[b, :, 4:5])[z[b, :, 4] > conf].reshape(-1)
        s = s[s > conf]
        if len(np.unique(s)) != len(s):
            return False
    return True


def nms_cases():
    """(name, seed, B, A, nc, distinct, kwargs, label builder)"""
    def labels_mixed(z, nc, rs):
        # image 0: two labels on predicted boxes (one duplicated), two free; image 1: z emptied, labels only; image 2: none
        lb = []
        zi = z[0]
        top = np.argsort(-(zi[:, 4] * zi[:, 5:].max(1)))[:2]
        l0 = [[float(np.argmax(zi[i, 5:])), *zi[i, :4]] for i in top]
        l0.append(list(l0[0]))
        l0 += [[float(rs.randint(nc)), *rs.uniform(20, 480, 2), *rs.uniform(8, 64, 2)] for _ in range(2)]
        lb.append(np.float32(l0))
        lb.append(np.float32([[float(rs.randint(nc)), *rs.uniform(20, 480, 2), *rs.uniform(8, 64, 2)] for _ in range(3)]))
        lb.append(np.zeros((0, 5), np.float32))
        return lb
    return [
        ("multi", 11, 3, 400, 4, False, dict(conf_thres=0.001, iou_thres=0.6, multi_label=True), labels_mixed),
        ("best", 11, 3, 400, 4, False, dict(conf_thres=0.25, iou_thres=0.45, multi_label=False), labels_mixed),
        ("classes", 11, 3, 400, 4, False, dict(conf_thres=0.001, iou_thres=0.6, multi_label=True, classes=[0, 2]), labels_mixed),
        ("nc1", 12, 3, 400, 1, False, dict(conf_thres=0.001, iou_thres=0.6, multi_label=True), labels_mixed),
        ("conf1", 11, 3, 400, 4, False, dict(conf_thres=1.0, iou_thres=0.6, multi_label=True), labels_mixed),
        ("maxnms", 13, 1, 8000, 4, True, dict(conf_thres=0.001, iou_thres=0.6, multi_label=True),
         lambda z, nc, rs: [np.float32([[3, 300, 200, 30, 50]])]),
    ]


def ulp_boxes(target):
    """(label side L, det width w) float32 with label [0, 0, L, 100] and det [0, 0, w, 100]: IoU == target under fp32 box_iou"""
    f = np.float32
    for L in range(100, 400):
        L = f(L)
        w = f(L * f(0.45))
        for _ in range(64):
            w = np.nextafter(w, f(0), dtype=f)
        for _ in range(128):
            inter = w * f(100.0)
            iou = inter / (L * f(100.0) + inter - inter)
            if iou == target:
                return L, w
            w = np.nextafter(w, f(1000), dtype=f)
    raise RuntimeError("no box for", target)


def cm_cases(rs):
    f = np.float32
    t45 = f(0.45)
    lo, hi = np.nextafter(t45, f(0)), np.nextafter(t45, f(1))
    c25 = f(0.25)
    clo, chi = np.nextafter(c25, f(0)), np.nextafter(c25, f(1))
    seqs = {}
    # IoU at the threshold: one label per class-1 image, det widths giving IoU = 0.45 - ulp, 0.45, 0.45 + ulp; conf at 0.25 +- ulp
    calls = []
    for k, iou in enumerate((lo, t45, hi)):
        L, w = ulp_boxes(iou)
        calls.append((np.float32([[0, 0, w, 100, 0.9, 1]]), np.float32([[1, 0, 0, L, 100]])))
    for c in (clo, c25, chi):
        calls.append((np.float32([[0, 0, 100, 100, c, 2], [200, 200, 260, 260, 0.8, 0]]), np.float32([[2, 0, 0, 100, 100], [0, 300, 300, 350, 350]])))
    seqs["edges"] = calls
    # one label claimed by several detections (distinct IoUs), and one detection overlapping several labels
    seqs["claims"] = [
        (np.float32([[0, 0, 100, 100, 0.9, 0], [0, 0, 90, 100, 0.8, 1], [0, 0, 80, 100, 0.7, 2], [500, 500, 600, 600, 0.6, 1]]),
         np.float32([[0, 0, 0, 100, 100], [2, 400, 400, 450, 450]])),
        (np.float32([[0, 0, 100, 100, 0.9, 1]]),
         np.float32([[1, 0, 0, 95, 100], [0, 0, 0, 90, 100], [2, 0, 0, 100, 85]])),
        (np.float32([[0, 0, 100, 100, 0.9, 1], [0, 0, 96, 100, 0.5, 0]]),
         np.float32([[1, 0, 0, 95, 100], [0, 0, 0, 90, 100]])),
    ]
    seqs["nomatch"] = [(np.float32([[0, 0, 10, 10, 0.9, 0], [50, 50, 60, 60, 0.5, 1]]), np.float32([[0, 100, 100, 150, 150], [2, 300, 0, 330, 40]]))]
    seqs["belowconf"] = [(np.float32([[0, 0, 100, 100, 0.2, 0], [0, 0, 100, 100, 0.25, 1]]), np.float32([[0, 0, 0, 100, 100], [1, 5, 5, 100, 100]]))]
    # random images: nc 5, up to 40 labels / 60 detections clustered so that many pairs pass 0.45
    calls = []
    while len(calls) < 12:
        nl, nd = rs.randint(0, 40), rs.randint(0, 60)
        lab = np.zeros((nl, 5), np.float32)
        lab[:, 0] = rs.randint(0, 5, nl)
        xy = rs.uniform(0, 400, (nl, 2)).astype(np.float32)
        lab[:, 1:3], lab[:, 3:5] = xy, xy + rs.uniform(10, 80, (nl, 2)).astype(np.float32)
        det = np.zeros((nd, 6), np.float32)
        src = rs.randint(0, max(nl, 1), nd)
        base = lab[src, 1:5] if nl else rs.uniform(0, 400, (nd, 4)).astype(np.float32)
        det[:, :4] = base + rs.uniform(-12, 12, (nd, 4)).astype(np.float32)
        det[:, 4] = rs.uniform(0.05, 1.0, nd)
        det[:, 5] = rs.randint(0, 5, nd)
        if nd and nl and not iou_distinct(det, lab):
            continue
        calls.append((det, lab))
    seqs["random"] = calls
    return seqs


def iou_distinct(det, lab):
    import torch
    import utils.general as G
    d = torch.from_numpy(det)
    d = d[d[:, 4] > 0.25]
    iou = G.box_iou(torch.from_numpy(lab[:, 1:]), d[:, :4]).numpy()
    rows_ok = all(len(np.unique(r[r > np.float32(0.45)])) == (r > np.float32(0.45)).sum() for r in iou)
    cols_ok = all(len(np.unique(c[c > np.float32(0.45)])) == (c > np.float32(0.45)).sum() for c in iou.T)
    return rows_ok and cols_ok


RUN_CASES = {
    "txt_conf": dict(save_txt=True, save_conf=True),
    "txt": dict(save_txt=True),
    "hybrid": dict(save_hybrid=True, case="single_cls"),
    "json": dict(save_json=True, weights="runs/best.pt"),
    "json_coco": dict(save_json=True, is_coco=True, weights=["last.pt", "best.pt"]),
    "plots": dict(plots=True),
}


def run_paths(bi, n):
    return [f"data/{bi}{i}.jpg" if i % 2 else f"data/im{bi}_{i}.png" for i in range(n)]


def val_main(case="main"):
    """a case of tests/golden/val_cases.npz: [(z, targets, shapes)], (H, W) per batch, nc"""
    import json
    g = np.load(os.path.join(GOLD, "val_cases.npz"))
    meta = json.loads(bytes(g["meta_json"]).decode())[case]
    shapes = lambda rows: [((int(r[0]), int(r[1])), ((float(r[2]), float(r[3])), (float(r[4]), float(r[5])))) for r in rows]  # noqa: E731
    batches = [(g[f"{case}_z_{bi}"], g[f"{case}_targets_{bi}"], shapes(g[f"{case}_shapes_{bi}"])) for bi in range(meta["n_batches"])]
    return batches, [tuple(hw) for hw in meta["hw"]], meta["nc"]


def run_test(ref_test, torch, kw):
    import contextlib
    import io
    import tempfile
    import torch.nn as nn
    kw = dict(kw)
    batches, hws, nc = val_main(kw.pop("case", "main"))

    class StandIn(nn.Module):
        def __init__(self):
            super().__init__()
            self.w = nn.Parameter(torch.zeros(1))
            self.names = [f"c{i}" for i in range(nc)]
            self.k = 0

        def forward(self, img, augment=False):
            z = torch.from_numpy(batches[self.k][0].copy())
            self.k += 1
            return [(z, None), None]

    loader = [(torch.zeros((len(shp), 3, H, W), dtype=torch.uint8), torch.from_numpy(t.copy()), run_paths(bi, len(shp)), shp)
              for bi, ((z, t, shp), (H, W)) in enumerate(zip(batches, hws))]
    seen = {}

    class Recording(ref_test.ConfusionMatrix):
        def plot(self, save_dir="", names=()):
            seen["matrix"] = self.matrix.copy()

    saved = ref_test.ConfusionMatrix, ref_test.ap_per_class, ref_test.plot_images
    orig_ap = ref_test.ap_per_class
    ref_test.ConfusionMatrix = Recording
    ref_test.ap_per_class = lambda *a, **k: orig_ap(*a, **{**k, "plot": False})
    ref_test.plot_images = lambda *a, **k: None
    try:
        with tempfile.TemporaryDirectory() as tmp:
            save_dir = os.path.join(tmp, "exp")
            os.makedirs(os.path.join(save_dir, "labels") if kw.get("save_txt") else save_dir)
            buf = io.StringIO()
            with contextlib.redirect_stdout(buf):
                res, maps, _ = ref_test.test({"nc": nc}, batch_size=32, model=StandIn(), dataloader=loader, save_dir=ref_test.Path(save_dir),
                                             compute_loss=None, half_precision=True, **{"plots": False, **kw})
            files = {}
            for root, _, names in os.walk(save_dir):
                for n in names:
                    f = os.path.join(root, n)
                    with open(f, "rb") as fh:
                        files[os.path.relpath(f, save_dir)] = fh.read()
    finally:
        ref_test.ConfusionMatrix, ref_test.ap_per_class, ref_test.plot_images = saved
    return files, buf.getvalue().replace(save_dir, "<save_dir>"), np.array(res, np.float64), np.asarray(maps, np.float64), seen.get("matrix")


def main():
    if not ref_shims.reference_available():
        raise SystemExit("set MYOLO_REFERENCE_ROOT to the reference checkout")
    np.int = int                      # the reference uses the removed alias
    _, G = ref_shims.import_reference()
    import torch
    import utils.metrics as M
    out = {}
    names = []
    for name, seed, B, A, nc, distinct, kw, mk in nms_cases():
        s = seed
        while True:
            z = make_z(s, B, A, nc, distinct)
            if scores_distinct(z, kw["conf_thres"]):
                break
            s += 1000
        rs = np.random.RandomState(s)
        if name != "maxnms":
            z[1, :, 4] = 0.0                            # image 1: no candidates, labels only
        lb = mk(z, nc, rs)
        res = G.non_max_suppression(torch.from_numpy(z.copy()), labels=[torch.from_numpy(l) for l in lb], **kw)
        names.append(name)
        p = f"nms_{name}_"
        out[p + "z"] = np.array([s, B, A, nc, int(distinct), int(name != "maxnms")], np.int64)
        out[p + "kw"] = np.array([kw["conf_thres"], kw["iou_thres"], float(kw["multi_label"])], np.float64)
        out[p + "classes"] = np.array(kw.get("classes", []), np.int64)
        for b in range(B):
            out[p + f"labels{b}"] = lb[b]
            out[p + f"out{b}"] = res[b].numpy().astype(np.float32)
        print(name, [len(r) for r in res])
    out["nms_names"] = np.array(names)
    rs = np.random.RandomState(5)
    seqs = cm_cases(rs)
    for name, calls in seqs.items():
        nc = 5 if name == "random" else 3
        cm = M.ConfusionMatrix(nc=nc)
        p = f"cm_{name}_"
        out[p + "n"] = np.array([len(calls), nc], np.int64)
        for k, (det, lab) in enumerate(calls):
            cm.process_batch(torch.from_numpy(det), torch.from_numpy(lab))
            out[p + f"det{k}"], out[p + f"lab{k}"] = det, lab
            out[p + f"matrix{k}"] = cm.matrix.copy()
        print(name, cm.matrix.sum())
    out["cm_names"] = np.array(list(seqs))
    import test as ref_test      # the reference's test.py (sys.path set by import_reference)
    for name, kw in RUN_CASES.items():
        files, stdout, res, maps, matrix = run_test(ref_test, torch, kw)
        p = f"run_{name}_"
        out[p + "files"] = np.array(sorted(files))
        for k, f in enumerate(sorted(files)):
            out[p + f"file{k}"] = np.frombuffer(files[f], np.uint8)
        out[p + "stdout"] = np.frombuffer(stdout.encode(), np.uint8)
        out[p + "results"], out[p + "maps"] = res, maps
        if matrix is not None:
            out[p + "matrix"] = matrix
        print(name, sorted(files), res[:4])
    out["run_names"] = np.array(list(RUN_CASES))
    path = os.path.join(GOLD, "testpy_cases.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
