"""TEST INFRASTRUCTURE - the numpy restatement of `--image-weights` (reference train.py:255,305-316, utils/general.py:216-240) that fixes
the device kernels' arithmetic and order (csrc/image_weights.cu, DESIGN.md section 3c):

    class_weights(labels, nc)        labels_to_class_weights: exact counts, empty bins -> 1, 1 / count, / numpy's sum over nc
    image_weights(labels, nc, cw)    labels_to_image_weights: per image sum over nc of cw * count, in numpy's order
    epoch_cw(class_weights, maps)    train.py's `cw = model.class_weights.cpu().numpy() * (1 - maps) ** 2 / nc`
    choices(iw, rng)                 random.choices(range(n), weights=iw, k=n): sequential cumulative sums, total = cum[-1] + 0.0, its
                                     ValueErrors before any draw, then bisect_right(cum, random() * total, 0, n - 1) per draw
    epoch_indices(...)               the whole per-epoch block at rank -1 / 0

numpy's np.add.reduce over a contiguous axis of m values is `0.0 + pairwise(a)`: below 8 values a sequential sum from -0.0, up to 128
eight strided accumulators combined as ((r0 + r1) + (r2 + r3)) + ((r4 + r5) + (r6 + r7)) and then the rest in order, above that a split
at n2 = m // 2 - (m // 2) % 8.  tests/test_image_weights_host.py proves it against numpy itself.
"""
import bisect
import hashlib
import itertools
import json

import numpy as np

LEAF = 128


def pairwise_rows(a):
    """numpy's pairwise sum along the last axis of a 2-D float64 array, row by row (each step is one fp64 operation on every row)"""
    a = np.asarray(a, np.float64)
    m = a.shape[1]
    if m < 8:
        res = np.full(a.shape[0], -0.0)
        for i in range(m):
            res = res + a[:, i]
        return res
    if m <= LEAF:
        r = [a[:, j].copy() for j in range(8)]
        i = 8
        while i < m - m % 8:
            for j in range(8):
                r[j] = r[j] + a[:, i + j]
            i += 8
        res = ((r[0] + r[1]) + (r[2] + r[3])) + ((r[4] + r[5]) + (r[6] + r[7]))
        for i in range(i, m):
            res = res + a[:, i]
        return res
    h = m // 2
    h -= h % 8
    return pairwise_rows(a[:, :h]) + pairwise_rows(a[:, h:])


def numpy_sum_rows(a):
    """np.add.reduce(a, axis=-1) of a 2-D float64 array: the pairwise sum added to the reduction's initial 0.0"""
    return 0.0 + pairwise_rows(a)


def numpy_sum(a):
    return np.float64(numpy_sum_rows(np.asarray(a, np.float64)[None])[0])


def class_column(labels):
    """the float32 class column of every label, concatenated, and each image's [start, end) in it (n + 1 int64)"""
    cols = [np.asarray(x, np.float32).reshape(-1, 5)[:, 0] for x in labels]
    offsets = np.zeros(len(cols) + 1, np.int64)
    offsets[1:] = np.cumsum([len(c) for c in cols])
    return (np.concatenate(cols) if cols else np.zeros(0, np.float32)), offsets


def class_weights(labels, nc):
    cls, _ = class_column(labels)
    counts = np.bincount(cls.astype(np.int64), minlength=nc)
    assert len(counts) == nc, "a class outside [0, nc)"
    w = 1.0 / np.where(counts == 0, 1, counts).astype(np.float64)
    return w / numpy_sum(w)


def image_weights(labels, nc, cw):
    cls, offsets = class_column(labels)
    n = len(offsets) - 1
    img = np.repeat(np.arange(n), np.diff(offsets))
    c = cls.astype(np.int64)
    assert ((c >= 0) & (c < nc)).all(), "a class outside [0, nc)"
    counts = np.bincount(img * nc + c, minlength=n * nc).reshape(n, nc)
    return numpy_sum_rows(np.asarray(cw, np.float64).reshape(1, nc) * counts.astype(np.float64))


def epoch_cw(class_weights, maps):
    """train.py:309: the model's class weights (labels_to_class_weights * nc) scaled by (1 - maps) ** 2 / nc"""
    cw = np.asarray(class_weights, np.float64)
    return cw * (1 - np.asarray(maps, np.float64)) ** 2 / len(cw)


def cumulative(w):
    return np.array(list(itertools.accumulate(float(v) for v in w)), np.float64)


def choices(w, rng):
    """random.choices(range(n), weights=w, k=n) with `rng.random` as the source: (indices int32, cumulative sums, total)"""
    cum = cumulative(w)
    n = len(cum)
    total = float(cum[-1]) + 0.0
    if total <= 0.0:
        raise ValueError("Total of weights must be greater than zero")
    if not np.isfinite(total):
        raise ValueError("Total of weights must be finite")
    cl = cum.tolist()
    idx = np.array([bisect.bisect_right(cl, rng.random() * total, 0, n - 1) for _ in range(n)], np.int32)
    return idx, cum, total


def epoch_indices(labels, class_weights, maps, rng):
    """the per-epoch block of train.py:305-316 at rank -1 / 0: (indices, cw, iw)"""
    cw = epoch_cw(class_weights, maps)
    iw = image_weights(labels, len(cw), cw)
    idx, _, _ = choices(iw, rng)
    return idx, cw, iw


def synth_labels(seed, n, nc, per_image, empty=0.0, frac=False, single=False):
    """the fixtures' synthetic (k, 5) float32 label sets, regenerated from their seed: Poisson(per_image) labels per image, a share
    `empty` of images without labels, classes in [0, nc) (with fractions of .25 / .5 / .75 when `frac`: astype(int) truncates them), and
    for `single` classes drawn from 10 then zeroed as LoadImagesAndLabels(single_cls=True) does"""
    rs = np.random.RandomState(seed)
    labels = []
    for _ in range(n):
        k = 0 if rs.random_sample() < empty else rs.poisson(per_image)
        lb = np.zeros((k, 5), np.float32)
        lb[:, 0] = rs.randint(0, 10 if single else nc, k) + (rs.choice([0.0, 0.25, 0.5, 0.75], k) if frac else 0.0)
        lb[:, 1:3] = rs.uniform(0.1, 0.9, (k, 2))
        lb[:, 3:5] = rs.uniform(0.02, 0.3, (k, 2))
        if single:
            lb[:, 0] = 0
        labels.append(lb)
    return labels


def labels_digest(labels):
    """sha256 of the concatenated labels and each image's label count: pins regenerated label sets to the ones the fixtures were made of"""
    h = hashlib.sha256(np.ascontiguousarray(np.concatenate(labels, 0), np.float32).tobytes())
    h.update(np.array([len(x) for x in labels], np.int64).tobytes())
    return h.hexdigest()


def load_cases(path):
    """tests/golden/image_weights_cases.npz -> ({name: dict}, {aug case: meta}, {aug key: array}).  A case holds its labels (regenerated
    from the stored spec and checked against the stored digest), nc, the class weights, and per epoch maps / cw / iw / indices (or the
    error message), with the seeds and the next draws"""
    g = np.load(path)
    meta = json.loads(bytes(g["meta_json"]).decode())
    cases = {}
    for name, m in meta["cases"].items():
        labels = synth_labels(**m["labels_spec"])
        assert labels_digest(labels) == m["labels_sha256"], f"{name}: regenerated labels differ from the fixture's"
        c = dict(m, labels=labels, class_weights=g[f"{name}_class_weights"])
        for e in range(m["epochs"]):
            for k in ("maps", "cw", "iw", "indices"):
                key = f"{name}_e{e}_{k}"
                if key in g.files:
                    c[f"e{e}_{k}"] = g[key]
        cases[name] = c
    aug = {k: g[k] for k in g.files if k.startswith("aug_")}
    return cases, meta.get("aug", {}), aug
