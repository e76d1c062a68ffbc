"""Restatement of the reference's OhemCELoss (reference utils/loss.py:303-328), pinned to the reference by tests/golden/ohem_cases.npz
(oracle/make_golden_ohem.py), and a numpy model of the library's device-side selection (csrc/train.cu, ohem_*_kernel).

forward_once(preds, labels):
    n_min = count(labels != ignore_index) // 16
    loss  = CrossEntropyLoss(ignore_index, reduction='none')(preds, labels).view(-1)       # ignored pixels: 0
    hard  = loss[loss > -log(thresh)]                                                      # -log in fp32
    if hard.numel() < n_min: hard = loss.topk(n_min)                                       # ignored pixels take part with 0
    return mean(hard)                                                                      # n_min = 0 and nothing hard: NaN

torch.topk leaves the order of equal values unspecified; here, as on the device, the lowest flat indices are taken first.
"""
import json

import numpy as np
import torch
import torch.nn.functional as F

CHUNK = 4096                     # pixels per block of the device's tie count (kOhemChunk)
PER_THREAD = CHUNK // 256        # pixels per thread of the device's cut kernel


def load_cases(path):
    """tests/golden/ohem_cases.npz as {thresh_t, margin, cases: [{name, thresh, ignore_index, aux, aux_weight, labels, logits [..],
    loss, grad [..]}]} with CPU torch tensors"""
    g = np.load(path)
    meta = json.loads(bytes(g["meta_json"]).decode())
    for c in meta["cases"]:
        n = c["name"]
        c["labels"] = torch.from_numpy(g[f"{n}_labels"])
        c["loss"] = torch.from_numpy(g[f"{n}_loss"])
        c["logits"] = [torch.from_numpy(g[f"{n}_logits_{i}"]) for i in range(c["n_outputs"])]
        c["grad"] = [torch.from_numpy(g[f"{n}_grad_{i}"]) for i in range(c["n_outputs"])]
    return meta


def thresh_t(thresh: float) -> float:
    """-log(thresh) in fp32, as the reference's constructor computes it"""
    return float(-torch.log(torch.tensor(thresh, dtype=torch.float32)))


def topk_mask(loss: torch.Tensor, k: int) -> torch.Tensor:
    """boolean mask of the k largest values of a 1-D tensor, ties taken in ascending index order"""
    mask = torch.zeros(loss.numel(), dtype=torch.bool, device=loss.device)
    if k:
        mask[torch.sort(-loss, stable=True).indices[:k]] = True
    return mask


def forward_once(preds: torch.Tensor, labels: torch.Tensor, thresh: float, ignore_index: int = -1) -> torch.Tensor:
    n_min = int((labels != ignore_index).sum()) // 16
    loss = F.cross_entropy(preds, labels, ignore_index=ignore_index, reduction="none").view(-1)
    taken = loss > thresh_t(thresh)
    if int(taken.sum()) < n_min:
        taken = topk_mask(loss.detach(), n_min)
    return loss[taken].mean()


def ohem_loss(preds, labels, thresh: float, ignore_index: int = -1, aux: bool = False, aux_weight=(0.15, 0.05)) -> torch.Tensor:
    """OhemCELoss(thresh, ignore_index, aux, aux_weight)(preds, labels)"""
    if not aux:
        return forward_once(preds, labels, thresh, ignore_index)
    return (forward_once(preds[0], labels, thresh, ignore_index) + aux_weight[0] * forward_once(preds[1], labels, thresh, ignore_index)
            + aux_weight[1] * forward_once(preds[2], labels, thresh, ignore_index))


# ---- the device selection, step by step ------------------------------------------------------------------------------------------
def keys(v: np.ndarray) -> np.ndarray:
    """order-preserving uint32 keys of float32 values; -0.0 takes +0.0's key"""
    u = np.ascontiguousarray(v, np.float32).view(np.uint32).copy()
    u[u == 0x80000000] = 0
    return np.where(u & 0x80000000, ~u, u | 0x80000000).astype(np.uint32)


def radix_kth(k32: np.ndarray, k: int):
    """the k-th largest key (k >= 1) by four 8-bit digit passes: (key, how many of the pixels equal to it are taken, how many there are)"""
    prefix, mask = 0, 0
    for p in range(4):
        shift = 24 - 8 * p
        cand = k32[(k32 & np.uint32(mask)) == prefix]
        hist = np.bincount((cand >> shift) & 255, minlength=256)
        incl = np.cumsum(hist[::-1])                          # digits in descending order
        j = int(np.argmax(incl >= k))
        d = 255 - j
        k -= int(incl[j] - hist[d])
        prefix |= d << shift
        mask |= 255 << shift
    return prefix, k, int(hist[d])


def tie_cut(k32: np.ndarray, kth: int, need: int) -> int:
    """flat index of the need-th pixel (in index order) whose key is kth: per-chunk counts, then one chunk in runs of PER_THREAD"""
    tied = (k32 == kth).astype(np.int64)
    counts = np.add.reduceat(tied, np.arange(0, tied.size, CHUNK))
    incl = np.cumsum(counts)
    c = int(np.argmax(incl >= need))
    r = need - int(incl[c] - counts[c])
    runs = tied[c * CHUNK:(c + 1) * CHUNK]
    run_counts = np.add.reduceat(runs, np.arange(0, runs.size, PER_THREAD))
    run_incl = np.cumsum(run_counts)
    t = int(np.argmax(run_incl >= r))
    left = r - int(run_incl[t] - run_counts[t])
    pos = np.flatnonzero(runs[t * PER_THREAD:(t + 1) * PER_THREAD])[left - 1]
    return c * CHUNK + t * PER_THREAD + int(pos)


def select_topk(v: np.ndarray, k: int) -> np.ndarray:
    """mask of the k largest values as the device selects them"""
    mask = np.zeros(v.size, bool)
    if k == 0:
        return mask
    k32 = keys(v)
    kth, need, tie_total = radix_kth(k32, k)
    cut = v.size if tie_total == need else tie_cut(k32, kth, need)
    idx = np.arange(v.size)
    return (k32 > kth) | ((k32 == kth) & (idx <= cut))


def select(v: np.ndarray, n_valid: int, th: float):
    """(mask, denominator) of the device selection over per-pixel losses v (float32) with n_valid valid pixels"""
    n_min = n_valid // 16
    hard = v > np.float32(th)
    if int(hard.sum()) >= n_min:
        return hard, int(hard.sum())
    return select_topk(v, n_min), n_min
