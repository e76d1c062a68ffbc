"""Restatement of scipy.cluster.vq.kmeans(obs, k, iter, thresh) for an int k and (n, 2) float64 obs, in numpy, in the order of the
library's device kernel (csrc/kmeans.cu); pinned to scipy by tests/golden/kmeans_cases.npz (oracle/make_golden_kmeans.py).

1. Draws.  Every restart's start is numpy.random's global `choice(n, k, replace=False)` (scipy's `_kpoints`); nothing between two draws
   reads the generator, so all `iter` draws are made up front.
2. vq.  dist2 = (c0 - x0)^2 + (c1 - x1)^2 per code in code order, each operation rounded (no fused multiply-add); the code is the first j
   with the smallest dist2 (strict <); the distance is sqrt(dist2), correctly rounded.
3. Mean distortion.  numpy's pairwise sum over the n distances, then / n.  Below 8 elements a sequential sum from 0; at 8 to 128 eight
   strided accumulators combined as ((r0+r1)+(r2+r3))+((r4+r5)+(r6+r7)), then the remainder sequentially; above 128 a split at
   n2 = n//2 - (n//2) % 8 and left + right.  The split points depend on n only.
4. Cluster means.  Per cluster the per-feature sum runs sequentially in observation order (scipy's `_vq.update_cluster_means`), then is
   divided by the member count; clusters without members are dropped and the survivors renumbered in order.
5. Loop.  diff = |prev - cur| of consecutive means from prev = inf, iterating while diff > thresh; then one more vq with the final book
   gives the restart's distortion (scipy >= 1.17).  The winner is the first restart with dist < best (strict, from inf).
"""
import json

import numpy as np

LEAF = 128                                # numpy's PW_BLOCKSIZE


def pairwise_leaves(n):
    """the leaves (start, length) of numpy's pairwise sum over n elements, in order"""
    out = []

    def rec(s, m):
        if m <= LEAF:
            out.append((s, m))
            return
        h = m // 2
        h -= h % 8
        rec(s, h)
        rec(s + h, m - h)

    rec(0, n)
    return out


def _leaf_sums(a, leaves):
    """each leaf's partial as numpy forms it; leaves of one length are done together (the same operations, element by element)"""
    out = np.empty(len(leaves))
    starts = np.array([s for s, _ in leaves], dtype=np.int64)
    lens = np.array([m for _, m in leaves], dtype=np.int64)
    for m in np.unique(lens):
        sel = np.nonzero(lens == m)[0]
        blk = a[starts[sel, None] + np.arange(m)[None]]       # (leaves, m)
        if m < 8:
            res = np.zeros(len(sel))
            for i in range(m):
                res = res + blk[:, i]
        else:
            r = blk[:, :8].copy()
            i = 8
            while i < m - m % 8:
                r = r + blk[:, i:i + 8]
                i += 8
            res = ((r[:, 0] + r[:, 1]) + (r[:, 2] + r[:, 3])) + ((r[:, 4] + r[:, 5]) + (r[:, 6] + r[:, 7]))
            for j in range(i, m):
                res = res + blk[:, j]
        out[sel] = res
    return out


def pairwise_sum(a):
    """numpy's pairwise sum of a 1-D float64 array: the leaf partials combined along the recursion's own tree"""
    a = np.ascontiguousarray(a, dtype=np.float64)
    leaves = pairwise_leaves(len(a))
    part = iter(_leaf_sums(a, leaves).tolist())

    def rec(m):
        if m <= LEAF:
            return next(part)
        h = m // 2
        h -= h % 8
        left = rec(h)
        return left + rec(m - h)

    return rec(len(a))


def pairwise_mean(a):
    return np.float64(pairwise_sum(a) / len(a))


def vq(obs, book):
    """(codes, distances) of rule 2"""
    best = np.full(len(obs), np.inf)
    code = np.zeros(len(obs), dtype=np.int64)
    for j in range(len(book)):
        a = book[j, 0] - obs[:, 0]
        b = book[j, 1] - obs[:, 1]
        d2 = a * a + b * b
        m = d2 < best
        code[m] = j
        best[m] = d2[m]
    return code, np.sqrt(best)


def cluster_means(obs, code, k):
    """rule 4: the new book (members' sequential sums / counts, empty clusters dropped)"""
    sums = np.zeros((k, 2))
    np.add.at(sums, code, obs)
    cnt = np.bincount(code, minlength=k)
    live = cnt > 0
    return sums[live] / cnt[live, None]


def kmeans_one(obs, book, thresh=1e-5):
    """one restart from the book `book`: (final book, distortion, Lloyd iterations)"""
    prev, diff, it = np.inf, np.inf, 0
    while diff > thresh:
        code, dist = vq(obs, book)
        cur = pairwise_mean(dist)
        it += 1
        book = cluster_means(obs, code, len(book))
        diff = abs(prev - cur)
        prev = cur
    _, dist = vq(obs, book)
    return book, pairwise_mean(dist), it


def draw_starts(n, k, iters, npr=np.random):
    """every restart's start indices (iters, k), drawn as scipy's `_kpoints` draws them"""
    return np.stack([npr.choice(n, k, replace=False) for _ in range(iters)])


def kmeans(obs, k, iter=20, thresh=1e-5):
    """scipy.cluster.vq.kmeans(obs, k, iter, thresh) for an int k: (book, distortion, per-restart [(book, distortion, iterations)])"""
    obs = np.asarray(obs, dtype=np.float64)
    if not np.isfinite(obs).all():
        raise ValueError("array must not contain infs or NaNs")
    if iter < 1:
        raise ValueError(f"iter must be at least 1, got {iter}")
    if k < 1:
        raise ValueError(f"Asked for {k} clusters.")
    idx = draw_starts(len(obs), k, iter)
    runs = [kmeans_one(obs, obs[i], thresh) for i in idx]
    best, best_dist = None, np.inf
    for book, dist, _ in runs:
        if dist < best_dist:
            best, best_dist = book, dist
    return best, best_dist, runs


# ---- fixtures ------------------------------------------------------------------------------------------------------------------------
def case_obs(c):
    """a fixture case's observations: its stored points, or kmean_anchors' whitened `wh / s` of a seeded synthetic label set
    (oracle.restate_autoanchor.synth_dataset + label_wh, filtered to sides >= 2 px), optionally rounded to whole pixels and cut to the
    first `take` labels"""
    if "points" in c:
        return np.asarray(c["points"], dtype=np.float64)
    from oracle import restate_autoanchor as ra
    d = c["data"]
    shapes0, labels = ra.synth_dataset(**d["synth"])
    wh0 = ra.label_wh(ra.shapes_wh(shapes0), labels, d["img_size"])
    wh = wh0[(wh0 >= 2.0).any(1)]
    if d.get("round"):
        wh = np.round(wh)
    if d.get("take"):
        wh = wh[:d["take"]]
    return wh / wh.std(0)


def load_cases(path):
    """tests/golden/kmeans_cases.npz as a list of case dicts (meta from JSON, arrays as numpy); each case's per-restart books as a list"""
    g = np.load(path)
    meta = json.loads(bytes(g["meta_json"]).decode())
    for c in meta["cases"]:
        pre = c["name"] + "_"
        for key in g.files:
            if key.startswith(pre):
                c[key[len(pre):]] = g[key]
        c["run_books"] = np.split(c["run_books_flat"], np.cumsum(c["run_k"])[:-1])
    return meta["cases"]
