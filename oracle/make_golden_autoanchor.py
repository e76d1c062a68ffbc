"""TEST INFRASTRUCTURE - generates tests/golden/autoanchor_cases.npz from the UNMODIFIED reference's check_anchors / kmean_anchors
(utils/autoanchor.py:23-160) on the CPU:

    MYOLO_REFERENCE_ROOT=<checkout> python oracle/make_golden_autoanchor.py

(oracle.restate_autoanchor.load_cases reads it back.)

Each case seeds `random`, `numpy.random` and torch, then calls the reference on a reference-style dataset (`shapes` (n, 2) float64 [w, h],
float32 `labels`) drawn by oracle.restate_autoanchor.synth_dataset from a seed (the labels are not stored: the case keeps the draw's
arguments and a digest), and on a stand-in Detect with the case's anchors and strides.  It stores the printed lines, the k-means result, the
returned / written anchors, the Detect buffers after the call, bpr / aat / new_bpr, the next draws of `random` and `numpy.random`, and the
fitness torch computed in every generation.

The reference is observed, not changed: its module-level `kmeans` is wrapped to record the result and numpy's state right after it (the
mutation draws start there); the generations are then replayed here with the reference's own torch formulation of anchor_fitness over the
recorded draws, and the replay must land on the anchors the reference returned.

Seed rule.  Torch's fp32 `mean` over many values uses a cascade sum whose rounding depends on the CPU's vector width and thread count, so
the reference's fitness is not reproducible bit for bit across machines; the library sums exactly in fp64 instead (see the restatement's
docstring).  A seed is rejected when any generation has torch's fg and the running best f within 8 fp32 ulp of each other but unequal:
there, a last-bit difference could flip an acceptance.  Torch's fg equal to f counts as such a near tie too, unless the exact sums are
equal as well (an exact tie: equal terms, equal sums on every machine).  The restatement must then reproduce the reference's decisions,
which is asserted.  Such near ties are common (a generation whose one random scale is tiny barely moves the anchors), so most seeds are
rejected; the restatement screens them first, before the reference's slower run.
"""
import argparse
import contextlib
import hashlib
import io
import json
import os
import random
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
from oracle import ref_shims  # noqa: E402
from oracle import restate_autoanchor as ra  # noqa: E402

GOLD = os.path.join(HERE, "..", "tests", "golden")
COCO = [[10, 13, 16, 30, 33, 23], [30, 61, 62, 45, 59, 119], [116, 90, 156, 198, 373, 326]]
POOR = [[4, 5, 5, 4, 6, 6], [7, 8, 8, 7, 9, 9], [10, 11, 11, 10, 12, 12]]
CITY = [(12, 30), (25, 60), (40, 25), (90, 55), (200, 120), (8, 8)]
ULP_MARGIN = 8


class _Detect:
    """what check_anchors reads of Detect: anchors, anchor_grid, stride"""

    def __init__(self, anchors, stride):
        a = torch.tensor(anchors).float().view(len(anchors), -1, 2)
        self.stride = torch.tensor(stride, dtype=torch.float32)
        self.anchors = a / self.stride.view(-1, 1, 1)
        self.anchor_grid = a.clone().view(len(anchors), 1, -1, 1, 1, 2)


class _Model:
    def __init__(self, det):
        self.model = [det]


class _Dataset:
    def __init__(self, shapes0, labels):
        self.shapes = ra.shapes_wh(shapes0)
        self.labels = labels


def digest(labels):
    h = hashlib.sha256()
    for l in labels:
        h.update(np.ascontiguousarray(l).tobytes())
    return h.hexdigest()


def torch_fitness(wh, k, thr):
    """the reference's anchor_fitness, restated in its own torch ops"""
    r = wh[:, None] / torch.tensor(k, dtype=torch.float32)[None]
    best = torch.min(r, 1. / r).min(2)[0].max(1)[0]
    return (best * (best > thr).float()).mean()


def _near(a, b, exact_tie):
    """fg and f within ULP_MARGIN fp32 ulp, unless they are an exact tie (equal terms give equal sums on every machine)"""
    a, b = np.float32(a), np.float32(b)
    return abs(a - b) <= ULP_MARGIN * np.spacing(max(a, b)) and not (a == b and exact_tie)


def prescreen(shapes0, labels, thr, imgsz, n, gen):
    """the restatement's evolution has no generation within ULP_MARGIN + 2 ulp of its running best (torch's sum is a few ulp from the
    exact one), so the costly reference run is only made for seeds that can pass; numpy's global state is consumed"""
    km = ra.kmean_anchors(ra.shapes_wh(shapes0), labels, n, imgsz, thr, gen)
    wh0 = ra.label_wh(ra.shapes_wh(shapes0), labels, imgsz)
    wh32 = wh0[(wh0 >= 2.0).any(1)].astype(np.float32)
    f = ra.fitness(wh32, km["k_kmeans"], 1.0 / thr)
    for fg in km["fg"]:
        if fg != f and abs(fg - f) <= (ULP_MARGIN + 2) * np.spacing(max(fg, f)):
            return False
        f = max(f, fg)
    return True


def replay(rec, thr, gen):
    """the reference's generations over its recorded draws, with torch's fitness and the exact one side by side: (torch fg per
    generation, exact fg per generation, final k, near tie found, final torch f, accepted count).  The draws must end in the state numpy
    was in when the reference returned."""
    np.random.set_state(rec["state"])
    V = ra.draw_mutations(gen, rec["k"].shape)
    after = np.random.get_state()
    assert all(np.array_equal(a, b) if isinstance(a, np.ndarray) else a == b for a, b in zip(after, rec["post"])), "replay drew differently"
    wh = torch.tensor(rec["wh"], dtype=torch.float32)
    wh32 = wh.numpy()
    t = 1.0 / thr
    k = rec["k"]
    f, fe = torch_fitness(wh, k, t), ra.fitness(wh32, k, t)
    fgs, fges, near, acc = np.empty(gen, np.float32), np.empty(gen, np.float32), False, 0
    for g in range(gen):
        kg = (k.copy() * V[g]).clip(min=2.0)
        fg, fge = torch_fitness(wh, kg, t), ra.fitness(wh32, kg, t)
        fgs[g], fges[g] = float(fg), fge
        near |= _near(float(fg), float(f), fge == fe)
        if fg > f:
            f, fe, k = fg, fge, kg.copy()
            acc += 1
    return fgs, fges, ra.sort_by_area(k), near, float(f), acc


def run_case(name, ref, data, anchors=COCO, stride=(8.0, 16.0, 32.0), thr=4.0, imgsz=640, call="check", n=9, gen=1000, verbose=False,
             seed=0, want=None, tries=80):
    """first seed from `seed` whose run satisfies the seed rule (and `want`: 'fit' / 'replace' / 'keep' / 'flip', checked on the
    restatement before the reference runs)"""
    for s in range(seed, seed + tries):
        d = dict(data, seed=data["seed"] + s - seed)
        shapes0, labels = ra.synth_dataset(**d)
        ds = _Dataset(shapes0, labels)
        if want is not None:
            np.random.seed(s)
            det = _Detect(anchors, stride)
            o = ra.check_anchors(ds.shapes, labels, det.anchor_grid.numpy(), det.stride.numpy(), thr, imgsz)
            got = "fit" if o["bpr"] >= 0.98 else ("flip" if o["flipped"] else "replace") if o["replaced"] else "keep"
            if got != want:
                print(f"{name}: seed {s} gives {got}, not {want}")
                continue
        if want != "fit":
            np.random.seed(s)
            if call == "check":
                np.random.uniform(0.9, 1.1, size=(len(shapes0), 1))
            if not prescreen(shapes0, labels, thr, imgsz, n if call == "kmean" else len(anchors) * len(anchors[0]) // 2,
                             gen if call == "kmean" else 1000):
                print(f"{name}: seed {s} has a near tie in the restatement; next seed")
                continue
        rec = {}
        real = ref.kmeans

        def kmeans(obs, k, **kw):
            out = real(obs, k, **kw)
            rec["state"] = np.random.get_state()
            rec["k_white"] = out[0].copy()
            return out

        random.seed(s); np.random.seed(s); torch.manual_seed(s)
        det = _Detect(anchors, stride)
        ag0, an0 = det.anchor_grid.clone(), det.anchors.clone()
        buf = io.StringIO()
        ref.kmeans = kmeans
        try:
            with contextlib.redirect_stdout(buf):
                if call == "check":
                    ref.check_anchors(ds, _Model(det), thr=thr, imgsz=imgsz)
                    ret = None
                else:
                    ret = ref.kmean_anchors(ds, n=n, img_size=imgsz, thr=thr, gen=gen, verbose=verbose)
        finally:
            ref.kmeans = real
        rec["post"] = np.random.get_state()
        next_py = np.array([random.random(), random.random()])
        next_np = np.random.random(4)
        arrays = dict(anchor_grid0=ag0.numpy(), anchors0=an0.numpy(), anchor_grid1=det.anchor_grid.numpy().copy(),
                      anchors1=det.anchors.numpy().copy(), next_py=next_py, next_np=next_np)
        meta = dict(name=name, data=d, thr=thr, imgsz=imgsz, stride=list(stride), call=call, n=n, gen=gen, verbose=verbose, seed=s,
                    stdout=buf.getvalue(), digest=digest(labels), evolved="state" in rec)
        if "state" in rec:
            # the filtered wh and the sorted k-means k, recomputed with the reference's statements
            wh0 = ra.label_wh(ds.shapes, labels, imgsz)
            wh = wh0[(wh0 >= 2.0).any(1)]
            rec["wh"] = wh
            rec["k"] = ra.sort_by_area(rec["k_white"] * wh.std(0))
            g = gen if call == "kmean" else 1000
            fgs, fges, k_end, near, f_end, acc = replay(rec, thr, g)
            if near:
                print(f"{name}: seed {s} has a near tie between torch's fg and f; next seed")
                continue
            # the restatement (exact fp64 sums) takes the same decisions
            np.random.set_state(rec["state"])
            k_r, f_r, fg_r, acc_r = ra.evolve(wh.astype(np.float32), rec["k"], ra.draw_mutations(g, rec["k"].shape), 1.0 / thr)
            assert np.array_equal(ra.sort_by_area(k_r), k_end) and acc_r == acc and np.array_equal(fg_r, fges), \
                f"{name}: the restatement's evolution differs from the reference's"
            arrays.update(k_kmeans=rec["k"], k=k_end, fg_torch=fgs, fg_exact=fg_r)
            meta.update(accepted=int(acc), f_torch=f_end, f_exact=float(f_r))
            if ret is not None:
                assert np.array_equal(ret, k_end), f"{name}: replay does not reproduce the returned anchors"
        if ret is not None:
            arrays["returned"] = np.asarray(ret)
        print(f"{name}: seed {s}, {sum(len(l) for l in labels)} labels, evolved={meta['evolved']}")
        return meta, arrays
    print(f"{name}: no seed in {tries} gives the case; skipped")
    return None


def main():
    argp = argparse.ArgumentParser()
    argp.add_argument("--out", default=os.path.join(GOLD, "autoanchor_cases.npz"))
    args = argp.parse_args()
    ref_shims.import_reference()
    import utils.autoanchor as ref                         # the reference's (sys.path set by import_reference)
    base = dict(n_img=40, per_img=50, clusters=CITY, spread=0.35)
    specs = [
        ("fit", dict(data=dict(base, seed=11, clusters=[(10, 13), (16, 30), (33, 23), (30, 61), (62, 45), (59, 119), (116, 90),
                                                        (156, 198)], spread=0.2), want="fit", seed=100)),
        ("replace", dict(data=dict(base, seed=21), anchors=POOR, want="replace", seed=200)),
        ("flip", dict(data=dict(base, seed=31), anchors=POOR, stride=(32.0, 16.0, 8.0), want="flip", seed=300)),
        ("tiny", dict(data=dict(base, seed=41, tiny=0.15), anchors=POOR, want="replace", seed=400)),
        ("thr291", dict(data=dict(base, seed=51), anchors=POOR, thr=2.91, imgsz=1024, want="replace", seed=500)),
        ("keep", dict(data=dict(base, seed=61, clusters=[(8, 40), (40, 8), (20, 20), (300, 300)], spread=0.6),
                      anchors=[[8, 40, 40, 8, 20, 20], [8, 40, 40, 8, 20, 20], [300, 300, 60, 300, 300, 60]], want="keep", seed=600,
                      tries=30)),
        ("large", dict(data=dict(n_img=200, per_img=100, clusters=CITY, spread=0.4, seed=71, tiny=0.02), anchors=POOR, imgsz=1024,
                       want="replace", seed=700)),
        ("kmean_verbose", dict(data=dict(base, seed=81), call="kmean", n=9, gen=300, verbose=True, seed=800)),
    ]
    arrays, meta = {}, []
    for name, kw in specs:
        out = run_case(name, ref, **kw)
        if out is None:
            continue
        m, a = out
        meta.append(m)
        for k, v in a.items():
            arrays[f"{name}_{k}"] = v
    arrays["meta_json"] = np.frombuffer(json.dumps(dict(ulp_margin=ULP_MARGIN, cases=meta)).encode(), np.uint8)
    np.savez_compressed(args.out, **arrays)
    print("wrote", args.out, os.path.getsize(args.out), "bytes")


if __name__ == "__main__":
    main()
