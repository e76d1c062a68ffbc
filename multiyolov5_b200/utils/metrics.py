"""Segmentation validation metrics behind the reference's names (utils/metrics.py:234-275), computed on the GPU: the class map never
leaves the device, only 2 + 3*nclass counters do (SURVEY.md section 8f rank 2).

    batch_pix_accuracy(output, target)                -> (pixel_correct, pixel_labeled)
    batch_intersection_union(output, target, nclass)  -> (area_inter[nclass], area_union[nclass])
    seg_eval_batch(seg, target, nclass)               -> all four from the model's seg output (any resolution): the x8 bilinear upsample,
                                                         the argmax and the counters run without materialising full-resolution logits
`output`: (B,C,H,W) CUDA logits; `target`: (B,H,W) integer labels, -1 = ignore.
"""
import numpy as np
import torch

from .. import _lib
from .general import seg_argmax


def _counters(pred: torch.Tensor, target: torch.Tensor, nclass: int) -> np.ndarray:
    assert pred.is_cuda and pred.dtype in (torch.uint8, torch.int64) and pred.shape == target.shape
    tgt = target.to(device=pred.device, dtype=torch.int64).contiguous()
    out = torch.zeros(2 + 3 * nclass, dtype=torch.int64, device=pred.device)
    _lib.check(_lib.lib().myolo_seg_metrics(_lib.ptr(pred.contiguous()), _lib.torch_dtype_code(pred.dtype), _lib.ptr(tgt), pred.numel(), nclass,
                                            _lib.ptr(out), _lib.stream_ptr()))
    return out.cpu().numpy()


def _class_map(output: torch.Tensor, hw) -> torch.Tensor:
    return seg_argmax(output, tuple(hw), out_dtype=torch.uint8 if output.shape[1] <= 256 else torch.int64)


def seg_eval_batch(seg, target, nclass):
    """(pixel_correct, pixel_labeled, area_inter, area_union) like test.py:33-41 (`eval_batch`) for one batch"""
    c = _counters(_class_map(seg, target.shape[-2:]), target, nclass)
    inter, pred_a, lab_a = c[2:2 + nclass], c[2 + nclass:2 + 2 * nclass], c[2 + 2 * nclass:]
    return int(c[0]), int(c[1]), inter.copy(), pred_a + lab_a - inter


def batch_pix_accuracy(output, target):
    correct, labeled, _, _ = seg_eval_batch(output, target, output.shape[1])
    assert correct <= labeled, "Correct area should be smaller than Labeled"
    return correct, labeled


def batch_intersection_union(output, target, nclass):
    _, _, inter, union = seg_eval_batch(output, target, nclass)
    assert (inter <= union).all(), "Intersection area should be smaller than Union area"
    return inter, union


# ---- detection statistics (reference test.py:182-282, utils/metrics.py:12-112) on the device ----
# DetectionStats matches each image's NMS rows to its labels in one launch per batch (`myolo_det_match`) and keeps the results in a device
# stats store; `compute` runs ap_per_class over the whole store (`myolo_det_ap`: compaction, stable radix sort by (class, descending conf),
# cumulative sums, envelopes, np.interp and np.trapz in float64) and copies only per-class rows back.  Tied confidences within one class
# keep (image, row) order; the reference's np.argsort(-conf) is not stable, so the two agree whenever tied predictions of one class have
# identical `correct` rows.
_PX = np.linspace(0, 1, 1000)      # utils/metrics.py:47
_X101 = np.linspace(0, 1, 101)     # utils/metrics.py:106
_dev_tables = {}


def _tables(device):
    key = str(device)
    if key not in _dev_tables:
        _dev_tables[key] = (torch.from_numpy(_PX).to(device), torch.from_numpy(_X101).to(device),
                            torch.linspace(0.5, 0.95, 10).to(device))
    return _dev_tables[key]


def fitness(x):
    # Model fitness as a weighted combination of metrics (reference utils/metrics.py:12-15)
    w = [0.0, 0.0, 0.1, 0.9]  # weights for [P, R, mAP@0.5, mAP@0.5:0.95]
    return (x[:, :4] * w).sum(1)


def fitness2(x, mIoU):
    # reference utils/metrics.py:17-22: weights for [P, R, mAP@0.5, mAP@0.5:0.95, mIoU]
    w = [0.0, 0.0, 0.1, 0.2, 0.7]
    x_m = np.expand_dims(np.append(x[:, :4], mIoU), 0)
    return (x_m * w).sum(1)


def pack_geometry(img_hw, shapes):
    """(B, 5) float32 rows (h0, w0, gain, padw, padh) from collate_fn shapes[si] = ((h0, w0), ((h/h0, w/w0), (padw, padh))); a None
    ratio_pad is derived from the network input size as scale_coords does (reference utils/general.py:319-331).  The Python floats are
    rounded to float32 as torch rounds them when they meet a float32 tensor."""
    rows = []
    for (h0, w0), ratio_pad in shapes:
        if ratio_pad is None:
            gain = min(img_hw[0] / h0, img_hw[1] / w0)
            pad = (img_hw[1] - w0 * gain) / 2, (img_hw[0] - h0 * gain) / 2
        else:
            gain, pad = ratio_pad[0][0], ratio_pad[1]
        rows.append([float(h0), float(w0), float(gain), float(pad[0]), float(pad[1])])
    return np.array(rows, np.float64).astype(np.float32).reshape(-1, 5)


def _to_device(a, device, dtype):
    """host array / tensor -> device tensor without waiting for the device (pinned staging)"""
    t = a if isinstance(a, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(a))
    t = t.to(dtype=dtype).contiguous()
    if t.device.type == "cpu":
        return t.pin_memory().to(device, non_blocking=True)
    return t.to(device)


def _check_error(err, tcount, nc):
    if err & _lib.DET_ERR_TARGET_CLASS:
        raise ValueError("target class ids must be integers in [0, 256)")
    if err & _lib.DET_ERR_PRED_CLASS:
        raise ValueError("prediction class ids must be integers in [0, 256)")
    if err & _lib.DET_ERR_LABELS:
        raise ValueError("an image has more than 1024 targets")
    if nc is not None and tcount[nc:].any():
        raise ValueError(f"target class ids must be in [0, {nc})")


def _run_ap(correct, conf, cls, rows, n_images, max_det, ncol, tcount):
    """myolo_det_ap over a store -> (any, ap (nu, ncol), p (nu, 1000), r (nu, 1000)) on the host, nu = classes with targets"""
    L = _lib.lib()
    dev = correct.device
    px, x101, _ = _tables(dev)
    need = int(L.myolo_det_ap_workspace_bytes(n_images, max_det, ncol))
    ws = torch.empty(need, dtype=torch.uint8, device=dev)
    out_ap = torch.empty((256, ncol), dtype=torch.float64, device=dev)
    out_p = torch.empty((256, 1000), dtype=torch.float64, device=dev)
    out_r = torch.empty((256, 1000), dtype=torch.float64, device=dev)
    info = torch.zeros(2, dtype=torch.int32, device=dev)
    _lib.check(L.myolo_det_ap(_lib.ptr(correct), _lib.ptr(conf), _lib.ptr(cls), _lib.ptr(rows), n_images, max_det, ncol, _lib.ptr(tcount),
                              _lib.ptr(px), _lib.ptr(x101), _lib.ptr(out_ap), _lib.ptr(out_p), _lib.ptr(out_r), _lib.ptr(info), _lib.ptr(ws),
                              need, _lib.stream_ptr()))
    return info, out_ap, out_p, out_r


def _select(classes, out_ap, out_p, out_r):
    """ap_per_class's tail (utils/metrics.py:76-84) on the host: F1 and the index of its maximum mean"""
    nu = len(classes)
    ap, p, r = (t[:nu].cpu().numpy() for t in (out_ap, out_p, out_r))
    f1 = 2 * p * r / (p + r + 1e-16)
    i = f1.mean(0).argmax()
    return p[:, i], r[:, i], ap, f1[:, i], classes.astype("int32")


class DetectionStats:
    """Device stats store of a validation pass: one slot per (image, NMS row) holding the 10 `correct` bits (uint16), conf (fp32) and the
    class (uint8), each image's row count, and per-class target counts.  Slots are padded to `max_det` per image (7 B each plus 4 B per
    image); the store doubles when it fills.

        update(dets, counts, targets, img_hw, shapes)   one launch on the current stream, no synchronisation
        compute(nc) -> p, r, ap, f1, ap_class, nt, seen  what test.py:275-282 derives (p, r, f1 are 0. and ap, ap_class empty when no
                                                         prediction is correct at any IoU, nt then torch.zeros(1), as there)

    dets, counts: non_max_suppression(..., return_padded=True); targets: collate_fn's (n, 6) [image, class, x, y, w, h] normalised, on
    the host or the device; img_hw: the network input (height, width); shapes: collate_fn's per-image shapes."""

    def __init__(self, max_det=300, device="cuda", capacity=64):
        if not 0 < max_det <= 1024:
            raise ValueError("max_det must be in [1, 1024]")
        self.max_det, self.device, self.seen = int(max_det), torch.device(device), 0
        self.tcount = torch.zeros(256, dtype=torch.int64, device=self.device)
        self.err = torch.zeros(1, dtype=torch.int32, device=self.device)
        self._alloc(max(1, int(capacity)))

    def _alloc(self, cap):
        n = cap * self.max_det
        new = (torch.zeros(n, dtype=torch.int16, device=self.device), torch.zeros(n, dtype=torch.float32, device=self.device),
               torch.zeros(n, dtype=torch.uint8, device=self.device), torch.zeros(cap, dtype=torch.int32, device=self.device))
        if hasattr(self, "correct"):
            m = self.seen * self.max_det
            for dst, src, k in zip(new, (self.correct, self.conf, self.cls, self.rows), (m, m, m, self.seen)):
                dst[:k].copy_(src[:k])
        self.correct, self.conf, self.cls, self.rows = new
        self.capacity = cap

    def update(self, dets, counts, targets, img_hw, shapes):
        B, max_det, six = dets.shape
        if max_det != self.max_det or six != 6:
            raise ValueError(f"dets must be (B, {self.max_det}, 6) padded NMS rows")
        if len(shapes) != B:
            raise ValueError("one shapes entry per image")
        if not dets.is_cuda:
            raise _lib.MyoloError("DetectionStats.update needs the device NMS output")
        if self.seen + B > self.capacity:
            cap = self.capacity
            while cap < self.seen + B:
                cap *= 2
            self._alloc(cap)
        geom = _to_device(pack_geometry(img_hw, shapes), dets.device, torch.float32)
        tg = _to_device(targets, dets.device, torch.float32).reshape(-1, 6)
        dets = dets.float().contiguous()
        counts = counts.to(torch.int32).contiguous()
        iouv = _tables(dets.device)[2]
        _lib.check(_lib.lib().myolo_det_match(_lib.ptr(dets), _lib.ptr(counts), B, max_det, _lib.ptr(tg), int(tg.shape[0]), int(img_hw[0]),
                                              int(img_hw[1]), _lib.ptr(geom), _lib.ptr(iouv), self.seen, _lib.ptr(self.correct),
                                              _lib.ptr(self.conf), _lib.ptr(self.cls), _lib.ptr(self.rows), _lib.ptr(self.tcount),
                                              _lib.ptr(self.err), _lib.stream_ptr()))
        self.seen += B

    def correct_rows(self):
        """(correct (n, 10) bool, conf, pcls) of every stored prediction in (image, row) order: the reference's concatenated stats[0:3]"""
        rows = self.rows[:self.seen].cpu().numpy()
        c = self.correct[:self.seen * self.max_det].view(self.seen, self.max_det).cpu().numpy().astype(np.uint16)
        conf = self.conf[:self.seen * self.max_det].view(self.seen, self.max_det).cpu().numpy()
        cls = self.cls[:self.seen * self.max_det].view(self.seen, self.max_det).cpu().numpy()
        keep = np.arange(self.max_det)[None, :] < rows[:, None]
        bits = (c[keep][:, None] >> np.arange(10, dtype=np.uint16)) & 1
        return bits.astype(bool), conf[keep], cls[keep].astype(np.float32)

    def compute(self, nc):
        if not 0 < nc <= 256:
            raise ValueError("nc must be in [1, 256]")
        if self.seen == 0:
            return 0., 0., [], 0., [], torch.zeros(1), 0
        info, out_ap, out_p, out_r = _run_ap(self.correct, self.conf, self.cls, self.rows, self.seen, self.max_det, 10, self.tcount)
        head = torch.cat([self.err.long(), info.long(), self.tcount]).cpu().numpy()     # the one synchronisation before the rows
        err, any_tp, tcount = int(head[0]), bool(head[1]), head[3:]
        _check_error(err, tcount, nc)
        if not any_tp:
            return 0., 0., [], 0., [], torch.zeros(1), self.seen
        classes = np.flatnonzero(tcount)
        p, r, ap, f1, ap_class = _select(classes, out_ap, out_p, out_r)
        return p, r, ap, f1, ap_class, tcount[:nc].astype(np.int64), self.seen


class ConfusionMatrix:
    """The fork's ConfusionMatrix (utils/metrics.py:115-187) with the counters on the device: one `myolo_confusion_update` launch per call,
    int64 counts read once by `.matrix`.  Row = true class, column = predicted class (the fork's order, the transpose of upstream
    YOLOv5); row nc holds unmatched labels (background FP), column nc unmatched detections (background FN).  Exactly equal IoUs are
    broken towards the lower label index, then the lower detection row (the fork's unstable argsort leaves them open).

        process_batch(detections, labels)                one image: (N, 6) [x1, y1, x2, y2, conf, cls], (M, 5) [cls, x1, y1, x2, y2]
        update(dets, counts, targets, img_hw, shapes)    a batch of padded NMS rows with DetectionStats.update's arguments; only images
                                                         with labels and rows count, as test.py:189-192 and :233-241 call process_batch
        matrix                                           float64 (nc + 1, nc + 1) numpy array (synchronises); a fresh copy of the
                                                         device counters on every read, not the fork's mutable attribute
        print(), plot(save_dir, names)                   plot() draws confusion_matrix.png only when seaborn and matplotlib import

    One image holds at most 1024 detections and 1024 labels (the fork takes any number); process_batch raises ValueError above
    that, and update() reports more than 1024 labels in one image when `.matrix` is read."""

    def __init__(self, nc, conf=0.25, iou_thres=0.45, device="cuda"):
        self.nc, self.conf, self.iou_thres = int(nc), conf, iou_thres
        self.device = torch.device(device)
        self.counts = torch.zeros((self.nc + 1, self.nc + 1), dtype=torch.int64, device=self.device)
        self.err = torch.zeros(1, dtype=torch.int32, device=self.device)

    def _launch(self, dets, counts, B, max_det, targets, H, W, geom, require_rows):
        tg = targets.reshape(-1, 6)
        _lib.check(_lib.lib().myolo_confusion_update(_lib.ptr(dets), _lib.ptr(counts), B, max_det, _lib.ptr(tg) if tg.numel() else None,
                                                     int(tg.shape[0]), int(H), int(W), _lib.ptr(geom), self.nc, float(self.conf),
                                                     float(self.iou_thres), int(require_rows), _lib.ptr(self.counts), _lib.ptr(self.err),
                                                     _lib.stream_ptr()))

    def process_batch(self, detections, labels):
        d = _to_device(detections, self.device, torch.float32).reshape(-1, 6)
        lb = _to_device(labels, self.device, torch.float32).reshape(-1, 5)
        n = d.shape[0]
        if n > 1024 or lb.shape[0] > 1024:
            raise ValueError("ConfusionMatrix.process_batch takes at most 1024 detections and 1024 labels per image")
        dets = d if n else torch.zeros((1, 6), device=self.device)
        cnt = torch.tensor([n], dtype=torch.int32).pin_memory().to(self.device, non_blocking=True)
        tg = torch.cat([torch.zeros((lb.shape[0], 1), device=self.device), lb], 1).contiguous()
        self._launch(dets.contiguous(), cnt, 1, max(n, 1), tg, 0, 0, None, 0)

    def update(self, dets, counts, targets, img_hw, shapes):
        B, max_det, six = dets.shape
        if six != 6 or len(shapes) != B:
            raise ValueError("dets must be (B, max_det, 6) padded NMS rows with one shapes entry per image")
        if not dets.is_cuda:
            raise _lib.MyoloError("ConfusionMatrix.update needs the device NMS output")
        geom = _to_device(pack_geometry(img_hw, shapes), dets.device, torch.float32)
        tg = _to_device(targets, dets.device, torch.float32).reshape(-1, 6)
        self._launch(dets.float().contiguous(), counts.to(torch.int32).contiguous(), B, max_det, tg, img_hw[0], img_hw[1], geom, 1)

    @property
    def matrix(self):
        head = torch.cat([self.err.long(), self.counts.reshape(-1)]).cpu().numpy()
        err = int(head[0])
        if err & _lib.DET_ERR_TARGET_CLASS:
            raise ValueError(f"label class ids must be integers in [0, {self.nc})")
        if err & _lib.DET_ERR_PRED_CLASS:
            raise ValueError(f"detection class ids must be integers in [0, {self.nc})")
        if err & _lib.DET_ERR_LABELS:
            raise ValueError("an image has more than 1024 labels")
        return head[1:].reshape(self.nc + 1, self.nc + 1).astype(np.float64)

    def plot(self, save_dir="", names=()):
        """the fork's plot: any failure of the drawing, a missing seaborn or matplotlib included, draws nothing.  A bad class id in the
        counted batches still raises: the matrix is read before the drawing starts."""
        matrix = self.matrix
        try:
            import matplotlib
            matplotlib.use("Agg")
            import matplotlib.pyplot as plt
            import seaborn as sn
            from pathlib import Path

            array = matrix / (matrix.sum(0).reshape(1, self.nc + 1) + 1E-6)  # normalize
            array[array < 0.005] = np.nan  # don't annotate (would appear as 0.00)
            fig = plt.figure(figsize=(12, 9), tight_layout=True)
            sn.set(font_scale=1.0 if self.nc < 50 else 0.8)
            labels = (0 < len(names) < 99) and len(names) == self.nc
            sn.heatmap(array, annot=self.nc < 30, annot_kws={"size": 8}, cmap="Blues", fmt=".2f", square=True,
                       xticklabels=list(names) + ["background FP"] if labels else "auto",
                       yticklabels=list(names) + ["background FN"] if labels else "auto").set_facecolor((1, 1, 1))
            fig.axes[0].set_xlabel("True")
            fig.axes[0].set_ylabel("Predicted")
            fig.savefig(Path(save_dir) / "confusion_matrix.png", dpi=250)
            plt.close(fig)
        except Exception:
            pass

    def print(self):
        m = self.matrix
        for i in range(self.nc + 1):
            print(" ".join(map(str, m[i])))


def _class_ids(a, what):
    a = np.asarray(a.cpu().numpy() if isinstance(a, torch.Tensor) else a).reshape(-1)
    if len(a) and not (np.all(a >= 0) and np.all(a < 256) and np.all(a == np.floor(a))):
        raise ValueError(f"{what} must be integers in [0, 256)")
    return a


def ap_per_class(tp, conf, pred_cls, target_cls, plot=False, save_dir=".", names=()):
    """reference utils/metrics.py:24-84 on the device (numpy or torch inputs): returns p, r, ap, f1, unique classes (int32).  Predictions of
    one class with equal conf are taken in input order (the reference's argsort is not stable).  conf must be exact in float32."""
    if plot:
        raise NotImplementedError("ap_per_class(plot=True): the PR / F1 curve plots are not built")
    tp = np.asarray(tp.cpu().numpy() if isinstance(tp, torch.Tensor) else tp)
    tp = tp.reshape(len(tp), -1).astype(bool)
    conf_in = np.asarray(conf.cpu().numpy() if isinstance(conf, torch.Tensor) else conf).reshape(-1)
    conf32 = conf_in.astype(np.float32)
    if not np.array_equal(conf32.astype(conf_in.dtype), conf_in):
        raise ValueError("conf must be exactly representable in float32")
    pred_cls = _class_ids(pred_cls, "pred_cls")
    target_cls = _class_ids(target_cls, "target_cls")
    n, ncol = tp.shape
    if not 1 <= ncol <= 16:
        raise ValueError("tp must have 1 to 16 columns")
    dev = torch.device("cuda")
    classes = np.unique(target_cls)
    tcount = np.bincount(target_cls.astype(np.int64), minlength=256)
    bits = (tp.astype(np.uint16) << np.arange(ncol, dtype=np.uint16)).sum(1).astype(np.uint16) if n else np.zeros(0, np.uint16)
    m = max(n, 1)
    correct = torch.zeros(m, dtype=torch.int16, device=dev)
    cf = torch.zeros(m, dtype=torch.float32, device=dev)
    cl = torch.zeros(m, dtype=torch.uint8, device=dev)
    if n:
        correct[:n] = torch.from_numpy(bits.view(np.int16)).to(dev)
        cf[:n] = torch.from_numpy(conf32).to(dev)
        cl[:n] = torch.from_numpy(pred_cls.astype(np.uint8)).to(dev)
    rows = torch.tensor([n], dtype=torch.int32, device=dev)
    _, out_ap, out_p, out_r = _run_ap(correct, cf, cl, rows, 1, m, ncol, torch.from_numpy(tcount).to(dev))
    return _select(classes, out_ap, out_p, out_r)
