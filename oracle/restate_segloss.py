"""Restatement of the reference's class-weighted CE and SegFocalLoss in numpy fp64, pinned to the reference by
tests/golden/segloss_cases.npz (oracle/make_golden_segloss.py).

With t' = t on valid pixels and 0 on ignored ones (the reference's `target * (target != ignore_index)`), p = softmax(z, 1), N = B*H*W
and a_i = w[t_i] on valid pixels, 0 on ignored ones:

    SegmentationLosses(weight=w)  (reference utils/loss.py:221-244):  A = sum a CE / sum a;  BiSe: A(out) + 1.5 aux_w A(aux16) + 0.5 aux_w A(aux32)
    SegFocalLoss(gamma, alpha=w, reduction)  (:279-297):               loss = A * F
        'mean': A = sum a CE / sum a,  F = sum_all (1 - p_t')^gamma / N
        'sum':  A = sum a CE,          F = sum_all (1 - p_t')^gamma        (the CE inside takes the outer reduction)

    d loss / d z_i = (c1 a_i + c2 gamma (1 - p_t')^(gamma-1) p_t') (p_i - e_t'),
        c1 = F / sum a (mean) or F (sum),   c2 = A / N (mean) or A (sum),   c2 = 0 for gamma = 0 (torch's pow backward of a zero exponent)

the formulation the library's kernels compute (csrc/train.cu, seg_wf_* / seg_focal_nchw_*).
"""
import json

import numpy as np


def load_cases(path):
    """tests/golden/segloss_cases.npz as {cases: [{name, kind, gamma, reduction, ignore_index, aux_weight, weight (or None), labels,
    logits [..], loss, grad [..]}]} with numpy arrays"""
    g = np.load(path)
    meta = json.loads(bytes(g["meta_json"]).decode())
    for c in meta["cases"]:
        n = c["name"]
        c["labels"] = g[f"{n}_labels"]
        c["loss"] = g[f"{n}_loss"]
        c["weight"] = g[f"{n}_weight"] if c["has_weight"] else None
        c["logits"] = [g[f"{n}_logits_{i}"] for i in range(c["n_outputs"])]
        c["grad"] = [g[f"{n}_grad_{i}"] for i in range(c["n_outputs"])]
    return meta


def focal(z, t, weight=None, gamma=0.0, ignore_index=-1, reduction="mean"):
    """(loss, d loss / d z) of SegFocalLoss(gamma, alpha=weight, ignore_index, reduction) in fp64; gamma = 0 with 'mean' is
    CrossEntropyLoss(weight=weight, ignore_index=ignore_index).  Labels outside [0, C) other than ignore_index count as ignored."""
    z = np.asarray(z, np.float64)
    t = np.asarray(t)
    B, C, H, W = z.shape
    valid = (t != ignore_index) & (t >= 0) & (t < C)
    tp = np.where(valid, t, 0)
    m = z.max(1, keepdims=True)
    e = np.exp(z - m)
    s = e.sum(1, keepdims=True)
    p = e / s
    ce = -np.take_along_axis(z - m - np.log(s), tp[:, None], 1)[:, 0]
    pt = np.take_along_axis(p, tp[:, None], 1)[:, 0]
    w = np.ones(C) if weight is None else np.asarray(weight, np.float64)
    a = np.where(valid, w[tp], 0.0)
    n = float(t.size)
    s_wl, s_w = float((a * ce).sum()), float(a.sum())
    with np.errstate(divide="ignore", invalid="ignore"):
        s_f = n if gamma == 0 else float(((1.0 - pt) ** gamma).sum())
        if reduction == "mean":
            A = s_wl / s_w if s_w else np.nan
            F = s_f / n
            c1 = F / s_w if s_w else 0.0
            c2 = 0.0 if gamma == 0 else A / n
        elif reduction == "sum":
            A, F = s_wl, s_f
            c1, c2 = F, (0.0 if gamma == 0 else A)
        else:
            raise ValueError(reduction)
        b = np.zeros_like(pt) if gamma == 0 else gamma * (1.0 - pt) ** (gamma - 1.0) * pt
        k = c1 * a + c2 * b
        onehot = np.moveaxis(np.eye(C)[tp], -1, 1)
        grad = np.where((k == 0)[:, None], 0.0, k[:, None] * (p - onehot))
    return A * F, grad


def seg_losses(preds, t, weight, aux_weight=None, ignore_index=-1):
    """SegmentationLosses(weight=weight, ignore_index)(*preds, t): one output, or BiSe's three with aux_num=2"""
    if aux_weight is None:
        return focal(preds[0], t, weight, 0.0, ignore_index)
    coef = [1.0, aux_weight * 1.5, aux_weight / 2.0]
    parts = [focal(p, t, weight, 0.0, ignore_index) for p in preds]
    return sum(c * l for c, (l, _) in zip(coef, parts)), [c * g for c, (_, g) in zip(coef, parts)]


def case_value(c):
    """(loss, [grads]) of a fixture case"""
    if c["kind"] == "wce":
        loss, grads = seg_losses(c["logits"], c["labels"], c["weight"], c["aux_weight"], c["ignore_index"])
        return loss, grads if isinstance(grads, list) else [grads]
    loss, grad = focal(c["logits"][0], c["labels"], c["weight"], c["gamma"], c["ignore_index"], c["reduction"])
    return loss, [grad]
