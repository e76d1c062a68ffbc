"""Restatement of the reference's detection validation statistics, in numpy, written from the reference's rules rather than copied.

    match_image(pred, labels, hw, geom, iouv)    -> correct (n, 10) bool    test.py:175,183-265 for one image
    ap_per_class(tp, conf, pred_cls, target_cls) -> p, r, ap, f1, classes  utils/metrics.py:24-84 (curves from `ap_curves`)
    interp(x, xp, fp, left, right)               -> np.interp as numpy computes it
    pairwise_sum(a)                              -> np.add.reduce's pairwise order for a 1-D float64 array

All float32 work is single numpy operations on float32 arrays (one rounding each, no fused multiply-add); all float64 work likewise.
`ap_per_class` orders predictions by a STABLE descending sort of conf, so tied confidences keep their input order (the reference's
np.argsort(-conf) is not stable; the two agree whenever tied predictions of one class have identical `tp` rows).
"""
import numpy as np

IOUV = np.linspace(0.5, 0.95, 10).astype(np.float32)     # == torch.linspace(0.5, 0.95, 10) in float32 (checked by the tests)
PX = np.linspace(0, 1, 1000)                               # utils/metrics.py:47
X101 = np.linspace(0, 1, 101)                              # utils/metrics.py:106
f32 = np.float32


def geometry(img_hw, shape):
    """(h0, w0, gain, padw, padh) as float32 from the loader's shapes[si] = ((h0, w0), ((h/h0, w/w0), (padw, padh))) or ((h0, w0), None)
    (scale_coords, utils/general.py:319-331: Python floats, rounded to float32 when they meet a float32 tensor)"""
    (h0, w0), ratio_pad = shape
    if ratio_pad is None:
        gain = min(img_hw[0] / h0, img_hw[1] / w0)
        pad = (img_hw[1] - w0 * gain) / 2, (img_hw[0] - h0 * gain) / 2
    else:
        gain, pad = ratio_pad[0][0], ratio_pad[1]
    return np.array([h0, w0, gain, pad[0], pad[1]], dtype=np.float64).astype(np.float32)


def _scale_clip(b, g):
    """scale_coords with ratio_pad + clip_coords on float32 xyxy rows (a copy)"""
    b = b.astype(np.float32).copy()
    b[:, [0, 2]] = b[:, [0, 2]] - g[3]
    b[:, [1, 3]] = b[:, [1, 3]] - g[4]
    b[:, :4] = b[:, :4] / g[2]
    b[:, [0, 2]] = np.minimum(np.maximum(b[:, [0, 2]], f32(0)), g[1])
    b[:, [1, 3]] = np.minimum(np.maximum(b[:, [1, 3]], f32(0)), g[0])
    return b


def target_boxes(labels, hw, g):
    """labels (nl, 5) [cls, x, y, w, h] normalised -> native-space xyxy float32 (test.py:175,238-239)"""
    h, w = hw
    t = labels[:, 1:5].astype(np.float32) * np.array([w, h, w, h], np.float32)
    xy = np.empty_like(t)
    xy[:, 0] = t[:, 0] - t[:, 2] / f32(2)
    xy[:, 1] = t[:, 1] - t[:, 3] / f32(2)
    xy[:, 2] = t[:, 0] + t[:, 2] / f32(2)
    xy[:, 3] = t[:, 1] + t[:, 3] / f32(2)
    return _scale_clip(xy, g)


def box_iou(a, b):
    """(N,4) x (M,4) float32 -> (N,M): inter / ((area1 + area2) - inter); 0/0 gives NaN"""
    area1 = (a[:, 2] - a[:, 0]) * (a[:, 3] - a[:, 1])
    area2 = (b[:, 2] - b[:, 0]) * (b[:, 3] - b[:, 1])
    iw = np.maximum(np.minimum(a[:, None, 2], b[None, :, 2]) - np.maximum(a[:, None, 0], b[None, :, 0]), f32(0))
    ih = np.maximum(np.minimum(a[:, None, 3], b[None, :, 3]) - np.maximum(a[:, None, 1], b[None, :, 1]), f32(0))
    inter = iw * ih
    with np.errstate(invalid="ignore", divide="ignore"):
        return inter / ((area1[:, None] + area2[None, :]) - inter)


def first_max(v):
    """torch.max(dim) on one row: the first NaN if any, else the first maximum"""
    nan = np.flatnonzero(np.isnan(v))
    k = int(nan[0]) if len(nan) else int(np.argmax(v))
    return v[k], k


def match_image(pred, labels, hw, g, iouv=IOUV):
    """pred (n,6) float32 NMS rows, labels (nl,5) [cls,x,y,w,h] normalised -> correct (n, len(iouv)) bool.
    For each prediction in row order: its best target among the targets of its class (torch max semantics); it takes that target
    if the IoU exceeds iouv[0] and the target is still free; a prediction whose best target is taken stays incorrect."""
    n = len(pred)
    correct = np.zeros((n, len(iouv)), bool)
    if n == 0 or len(labels) == 0:
        return correct
    pbox = _scale_clip(pred[:, :4], g)
    tbox = target_boxes(labels, hw, g)
    iou = box_iou(pbox, tbox)
    taken = set()
    for k in range(n):
        same = np.flatnonzero(labels[:, 0] == pred[k, 5])
        if not len(same):
            continue
        v, j = first_max(iou[k, same])
        if v > iouv[0] and same[j] not in taken:
            taken.add(same[j])
            correct[k] = v > iouv
    return correct


def interp(x, xp, fp, left=None, right=None):
    """np.interp: j = (number of xp <= x) - 1; left below xp[0], right above xp[-1]; fp[j] at the last index or where xp[j] == x;
    otherwise slope * (x - xp[j]) + fp[j] with slope = (fp[j+1] - fp[j]) / (xp[j+1] - xp[j])"""
    x, xp, fp = (np.asarray(a, np.float64) for a in (x, xp, fp))
    left = fp[0] if left is None else float(left)
    right = fp[-1] if right is None else float(right)
    j = np.searchsorted(xp, x, side="right") - 1
    out = np.empty(x.shape, np.float64)
    lo, hi = j < 0, x > xp[-1]
    last = ~lo & ~hi & (j == len(xp) - 1)
    mid = ~lo & ~hi & ~last
    out[lo], out[hi], out[last] = left, right, fp[-1]
    jm, xm = j[mid], x[mid]
    exact = xp[jm] == xm
    jn = np.minimum(jm + 1, len(xp) - 1)
    with np.errstate(invalid="ignore", divide="ignore"):
        slope = (fp[jn] - fp[jm]) / (xp[jn] - xp[jm])
        val = slope * (xm - xp[jm]) + fp[jm]
    out[mid] = np.where(exact, fp[jm], val)
    return out


def pairwise_sum(a):
    """numpy's pairwise summation of a contiguous float64 array (umath loops: 8 accumulators below 128 elements, halving above)"""
    a = np.asarray(a, np.float64)
    n = len(a)
    if n < 8:
        res = 0.0
        for v in a:
            res += v
        return res
    if n <= 128:
        r = a[:8].copy()
        m = n - n % 8
        for i in range(8, m, 8):
            r += a[i:i + 8]
        res = ((r[0] + r[1]) + (r[2] + r[3])) + ((r[4] + r[5]) + (r[6] + r[7]))
        for i in range(m, n):
            res += a[i]
        return res
    n2 = n // 2
    n2 -= n2 % 8
    return pairwise_sum(a[:n2]) + pairwise_sum(a[n2:])


def trapz(y, x):
    d = np.diff(x)
    return 0.0 + pairwise_sum(d * (y[1:] + y[:-1]) / 2.0)


def compute_ap(recall, precision):
    mrec = np.concatenate(([0.0], recall, [recall[-1] + 0.01]))
    mpre = np.concatenate(([1.0], precision, [0.0]))
    env = np.maximum.accumulate(mpre[::-1])[::-1]
    return trapz(interp(X101, mrec, env), X101)


def ap_curves(tp, conf, pred_cls, target_cls):
    """(classes, ap (nc,k), p (nc,1000), r (nc,1000)) of ap_per_class before its F1 selection"""
    tp = np.asarray(tp).astype(bool)
    if tp.ndim == 1:
        tp = tp[:, None]
    conf = np.asarray(conf)
    pred_cls = np.asarray(pred_cls)
    target_cls = np.asarray(target_cls)
    order = np.argsort(-conf, kind="stable")
    tp, conf, pred_cls = tp[order], conf[order], pred_cls[order]
    classes = np.unique(target_cls)
    nc = len(classes)
    ap, p, r = np.zeros((nc, tp.shape[1])), np.zeros((nc, 1000)), np.zeros((nc, 1000))
    for ci, c in enumerate(classes):
        i = pred_cls == c
        n_l = (target_cls == c).sum()
        n_p = i.sum()
        if n_p == 0 or n_l == 0:
            continue
        tpc = tp[i].astype(np.int64).cumsum(0)
        fpc = (1 - tp[i].astype(np.int64)).cumsum(0)
        recall = tpc / (n_l + 1e-16)
        precision = tpc / (tpc + fpc)
        xc = -conf[i]
        r[ci] = interp(-PX, xc, recall[:, 0], left=0)
        p[ci] = interp(-PX, xc, precision[:, 0], left=1)
        for j in range(tp.shape[1]):
            ap[ci, j] = compute_ap(recall[:, j], precision[:, j])
    return classes, ap, p, r


def ap_per_class(tp, conf, pred_cls, target_cls):
    classes, ap, p, r = ap_curves(tp, conf, pred_cls, target_cls)
    f1 = 2 * p * r / (p + r + 1e-16)
    i = f1.mean(0).argmax()
    return p[:, i], r[:, i], ap, f1[:, i], classes.astype("int32")


def test_statistics(stats, nc):
    """test.py:275-282 + :337-339 from per-image (correct, conf, pcls, tcls) tuples -> (mp, mr, map50, map, maps, p, r, ap, f1, ap_class, nt)"""
    stats = [np.concatenate(x, 0) for x in zip(*stats)]
    p, r, f1, mp, mr, map50, map_ = 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0
    ap, ap_class = [], []
    if len(stats) and stats[0].any():
        p, r, ap, f1, ap_class = ap_per_class(*stats)
        ap50, ap = ap[:, 0], ap.mean(1)
        mp, mr, map50, map_ = p.mean(), r.mean(), ap50.mean(), ap.mean()
        nt = np.bincount(stats[3].astype(np.int64), minlength=nc)
    else:
        nt = np.zeros(1)
    maps = np.zeros(nc) + map_
    for i, c in enumerate(ap_class):
        maps[c] = ap[i]
    return dict(mp=mp, mr=mr, map50=map50, map=map_, maps=maps, p=p, r=r, ap=ap, f1=f1, ap_class=ap_class, nt=nt)
