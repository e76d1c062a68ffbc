"""TEST INFRASTRUCTURE - the fork's ConfusionMatrix.process_batch (utils/metrics.py:115-162) restated in numpy float32, and the
apriori-label rows of non_max_suppression(labels=...) (utils/general.py:448-455) as plain candidate rows.

process_batch keeps the fork's steps: conf filter, box_iou(labels, detections) in fp32, pairs with IoU > iou_thres, each detection's
best label, then each label's best detection.  The fork breaks exact IoU ties with numpy's unstable argsort; this restatement takes the
lower label index, then the lower detection index, as the device kernel does, so the two agree on every input without exact ties.
"""
import numpy as np


def box_iou(box1, box2):
    """general.box_iou in float32: (N, 4) x (M, 4) -> (N, M)"""
    b1, b2 = np.asarray(box1, np.float32), np.asarray(box2, np.float32)
    a1 = (b1[:, 2] - b1[:, 0]) * (b1[:, 3] - b1[:, 1])
    a2 = (b2[:, 2] - b2[:, 0]) * (b2[:, 3] - b2[:, 1])
    wh = np.minimum(b1[:, None, 2:], b2[None, :, 2:]) - np.maximum(b1[:, None, :2], b2[None, :, :2])
    inter = np.maximum(wh, np.float32(0)).prod(2, dtype=np.float32)
    return (inter / (a1[:, None] + a2[None, :] - inter)).astype(np.float32)


def process_batch(matrix, detections, labels, nc, conf=0.25, iou_thres=0.45):
    """adds one image to `matrix` ((nc + 1, nc + 1) float64, row = true class); detections (N, 6), labels (M, 5) [cls, x1, y1, x2, y2]"""
    det = np.asarray(detections, np.float32).reshape(-1, 6)
    lab = np.asarray(labels, np.float32).reshape(-1, 5)
    det = det[det[:, 4] > np.float32(conf)]
    gc = lab[:, 0].astype(np.int64)
    dc = det[:, 5].astype(np.int64)
    iou = box_iou(lab[:, 1:], det[:, :4])
    ok = iou > np.float32(iou_thres)
    best_lab = np.full(len(det), -1)
    for j in range(len(det)):
        ks = np.flatnonzero(ok[:, j])
        if len(ks):
            best_lab[j] = ks[np.argmax(iou[ks, j])]            # first maximum: the lower label index
    match = np.full(len(lab), -1)
    for i in range(len(lab)):
        js = np.flatnonzero(best_lab == i)
        if len(js):
            match[i] = js[np.argmax(iou[i, js])]
    n = (match >= 0).any()
    for i, g in enumerate(gc):
        if match[i] >= 0:
            matrix[g, dc[match[i]]] += 1
        else:
            matrix[nc, g] += 1
    if n:
        matched = set(match[match >= 0].tolist())
        for j, d in enumerate(dc):
            if j not in matched:
                matrix[d, nc] += 1
    return matrix


def label_rows(labels, nc):
    """(k, 5) [cls, x, y, w, h] apriori labels -> (k, 5 + nc) candidate rows: box, obj 1.0, one-hot class"""
    lab = np.asarray(labels, np.float32).reshape(-1, 5)
    v = np.zeros((len(lab), nc + 5), np.float32)
    v[:, :4] = lab[:, 1:5]
    v[:, 4] = 1.0
    v[np.arange(len(lab)), lab[:, 0].astype(np.int64) + 5] = 1.0
    return v
