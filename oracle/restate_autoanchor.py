"""Restatement of the reference's autoanchor (utils/autoanchor.py:23-160) in numpy, in the arithmetic of the library's device kernels
(csrc/autoanchor.cu), pinned to the reference by tests/golden/autoanchor_cases.npz (oracle/make_golden_autoanchor.py); and the seeded
synthetic label sets the fixtures are built from.

ratio metric (the reference's `metric`), computed in the dtype torch promotes to (fp64 as soon as either operand is fp64):
    r    = wh[:, None] / k[None]                       # correctly rounded divide
    x    = min(r, 1 / r).min(2)                        # torch's `1. / r` is r.reciprocal() * 1.: a correctly rounded reciprocal
    best = x.max(1)
    comparisons with 1 / thr in that same dtype (the Python float cast to it)

fitness of the evolution (anchor_fitness, fp32):
    term = best if best > fp32(1 / thr) else 0
    S    = sum of the terms in fp64                    # exact: see below
    f    = fp32(S) / fp32(n)                           # torch's CPU mean divides its sum by n

With anchor_t <= 16 every non-zero term is an fp32 value in (1/16, 1], i.e. an integer multiple of 2^-27, so a sum of fewer than 2^26
of them is an integer below 2^53 times 2^-27: fp64 holds it exactly whatever the order of the additions.  Torch's own fp32 cascade sum
rounds on the way and may differ from fp32(S) by a few ulp; the fixture generator only keeps seeds where that cannot change a decision.
"""
import json

import numpy as np

MP, SIGMA = 0.9, 0.1            # mutation probability and sigma of the reference's evolution


# ---- seeded synthetic label sets ----------------------------------------------------------------------------------------------------
def synth_dataset(seed, n_img, per_img, clusters, spread=0.3, tiny=0.0, shapes=((256, 512), (180, 320), (120, 160), (300, 300))):
    """(shapes0 [(h0, w0)], labels [(m, 5) float32 class, x, y, w, h normalised]) drawn from numpy's Generator(seed) only (never the global
    state).  Box sizes are log-normal around `clusters` ((w, h) pixels at a long side of 640) with `spread`; a `tiny` share is 0.5-3 px."""
    rng = np.random.default_rng(seed)
    shapes0 = [tuple(int(v) for v in shapes[i]) for i in rng.integers(0, len(shapes), n_img)]
    cl = np.asarray(clusters, dtype=np.float64)
    labels = []
    for h0, w0 in shapes0:
        m = int(rng.poisson(per_img))
        c = cl[rng.integers(0, len(cl), m)]
        px = c * np.exp(rng.normal(0.0, spread, (m, 2)))
        small = rng.random(m) < tiny
        px[small] = rng.uniform(0.5, 3.0, (int(small.sum()), 2))
        scale = 640.0 / max(h0, w0)
        wn = np.clip(px[:, 0] / (w0 * scale), 1e-4, 1.0)
        hn = np.clip(px[:, 1] / (h0 * scale), 1e-4, 1.0)
        l = np.stack([rng.integers(0, 8, m).astype(np.float64), rng.random(m), rng.random(m), wn, hn], 1)
        labels.append(l.astype(np.float32))
    return shapes0, labels


def shapes_wh(shapes0):
    """the reference dataset's `shapes`: (n, 2) float64 [w, h]"""
    return np.array([(w0, h0) for h0, w0 in shapes0], dtype=np.float64).reshape(-1, 2)


def label_wh(shapes, labels, img_size, scale=None):
    """the reference's label wh in pixels (float64): shapes rescaled to a long side of img_size, times the optional per-image scale"""
    s = img_size * shapes / shapes.max(1, keepdims=True)
    if scale is not None:
        s = s * scale
    return np.concatenate([l[:, 3:5] * v for v, l in zip(s, labels)])


# ---- the arithmetic ------------------------------------------------------------------------------------------------------------------
def ratio_metric(wh, k):
    dt = np.result_type(wh.dtype, k.dtype)
    r = wh.astype(dt)[:, None] / k.astype(dt)[None]
    with np.errstate(divide="ignore"):                          # a zero side: r = 0, 1 / r = inf, x = 0
        x = np.minimum(r, dt.type(1) / r).min(2)
    return x, x.max(1)


def metric_stats(wh, k, thr):
    """what myolo_anchor_metric returns: counts of best > thr and x > thr, and the fp64 sums of x, best and x over thr (thr = 1 / anchor_t,
    compared in the metric's dtype)"""
    x, best = ratio_metric(wh, k)
    t = x.dtype.type(thr)
    return dict(n_best=int((best > t).sum()), n_x=int((x > t).sum()), sum_x=float(x.astype(np.float64).sum()),
                sum_best=float(best.astype(np.float64).sum()), sum_x_above=float(x[x > t].astype(np.float64).sum()))


def fitness(wh32, k, thr):
    """anchor_fitness(k) with the exact fp64 sum: fp32"""
    _, best = ratio_metric(wh32, np.asarray(k, dtype=np.float64).astype(np.float32))
    term = np.where(best > np.float32(thr), best, np.float32(0))
    return np.float32(np.float32(term.astype(np.float64).sum()) / np.float32(wh32.shape[0]))


def draw_mutations(gen, sh, npr=np.random):
    """the reference's gen mutation factors (gen, *sh), drawn from numpy's global state exactly as its loop draws them"""
    out = np.empty((gen,) + tuple(sh), dtype=np.float64)
    for g in range(gen):
        v = np.ones(sh)
        while (v == 1).all():
            v = ((npr.random(sh) < MP) * npr.random() * npr.randn(*sh) * SIGMA + 1).clip(0.3, 3.0)
        out[g] = v
    return out


def evolve(wh32, k0, V, thr):
    """the evolution over pre-drawn factors V: (k, f, per-generation fg, accepted count)"""
    k = np.asarray(k0, dtype=np.float64)
    f = fitness(wh32, k, thr)
    fgs = np.empty(len(V), dtype=np.float32)
    acc = 0
    for g, v in enumerate(V):
        kg = np.maximum(k * v, 2.0)
        fg = fgs[g] = fitness(wh32, kg, thr)
        if fg > f:
            f, k = fg, kg
            acc += 1
    return k, f, fgs, acc


def sort_by_area(k):
    return k[np.argsort(k.prod(1))]


def kmean_anchors(shapes, labels, n, img_size, thr, gen):
    """kmean_anchors over a loaded dataset (thr = anchor_t): the k-means k (sorted), the evolved k (sorted) and the evolution record"""
    from scipy.cluster.vq import kmeans
    t = 1.0 / thr
    wh0 = label_wh(shapes, labels, img_size)
    wh = wh0[(wh0 >= 2.0).any(1)]
    s = wh.std(0)
    k, _ = kmeans(wh / s, n, iter=30)
    assert len(k) == n
    k = sort_by_area(k * s)
    V = draw_mutations(gen, k.shape)
    kf, f, fgs, acc = evolve(wh.astype(np.float32), k, V, t)
    return dict(k_kmeans=k, k=sort_by_area(kf), f=f, fg=fgs, accepted=acc, n_small=int((wh0 < 3.0).any(1).sum()), n_wh=len(wh))


def check_anchors(shapes, labels, anchor_grid, stride, thr, imgsz):
    """check_anchors over a loaded dataset with Detect buffers anchor_grid (nl, 1, na, 1, 1, 2) fp32 and stride (nl,) fp32: a dict with the
    reference's decisions and the buffers after the call (fp32 numpy)"""
    t = 1.0 / thr
    scale = np.random.uniform(0.9, 1.1, size=(shapes.shape[0], 1))
    wh = label_wh(shapes, labels, imgsz, scale).astype(np.float32)
    n = np.float32(wh.shape[0])
    anchors = anchor_grid.reshape(-1, 2).astype(np.float32)
    st = metric_stats(wh, anchors, t)
    out = dict(bpr=np.float32(np.float32(st["n_best"]) / n), aat=np.float32(np.float32(st["n_x"]) / n), replaced=False, flipped=False,
               anchor_grid=anchor_grid.astype(np.float32).copy(), anchors=None)
    if out["bpr"] < 0.98:
        km = kmean_anchors(shapes, labels, anchor_grid[0].size // 2 * anchor_grid.shape[0], imgsz, thr, 1000)
        out.update(km)
        st2 = metric_stats(wh, km["k"], t)
        out["new_bpr"] = np.float32(np.float32(st2["n_best"]) / n)
        if out["new_bpr"] > out["bpr"]:
            a = km["k"].astype(np.float32)
            ag = a.reshape(anchor_grid.shape)
            an = a.reshape(anchor_grid.shape[0], -1, 2) / stride.astype(np.float32).reshape(-1, 1, 1)
            area = ag.prod(-1).reshape(-1)
            if np.sign(area[-1] - area[0]) != np.sign(stride[-1] - stride[0]):
                ag, an = ag[::-1].copy(), an[::-1].copy()
                out["flipped"] = True
            out.update(replaced=True, anchor_grid=ag, anchors=an)
    return out


# ---- fixtures ------------------------------------------------------------------------------------------------------------------------
def load_cases(path):
    """tests/golden/autoanchor_cases.npz as a list of case dicts (meta from JSON, arrays as numpy)"""
    g = np.load(path)
    meta = json.loads(bytes(g["meta_json"]).decode())
    for c in meta["cases"]:
        pre = c["name"] + "_"
        for key in g.files:
            if key.startswith(pre):
                c[key[len(pre):]] = g[key]
    return meta["cases"]


def case_dataset(c):
    """(shapes0, labels) of a fixture case, re-drawn from its seed"""
    return synth_dataset(**c["data"])
