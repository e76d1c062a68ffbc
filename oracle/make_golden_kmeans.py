"""TEST INFRASTRUCTURE - generates tests/golden/kmeans_cases.npz from scipy.cluster.vq.kmeans itself (scipy >= 1.17, whose `_kmeans`
returns the mean of one more vq with the final book) on the CPU:

    python oracle/make_golden_kmeans.py

(oracle.restate_kmeans.load_cases reads it back.)

Each case seeds `numpy.random`, calls `kmeans(obs, k, iter=iters)` and records the returned book and distortion and the next four
`numpy.random.random` values.  It then re-seeds, draws the same starts as scipy's `_kpoints` does and runs scipy's `_kmeans` from each,
recording every restart's book, distortion and Lloyd iteration count (calls of `_vq.update_cluster_means`).  Observations are
kmean_anchors' whitened `wh / s` of a seeded synthetic label set (oracle.restate_autoanchor.synth_dataset + label_wh; the case keeps the
draw's arguments, not the points), or a few stored points for the tiny cases.
"""
import argparse
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
from oracle import restate_kmeans as rk  # noqa: E402

GOLD = os.path.join(HERE, "..", "tests", "golden")
CITY = [(12, 30), (25, 60), (40, 25), (90, 55), (200, 120), (8, 8)]
CITY8 = CITY + [(30, 80), (150, 300)]
BIG_SHAPES = ((1024, 2048), (720, 1280), (480, 640))


class _Counted:
    """scipy's _vq module with update_cluster_means counted"""

    def __init__(self, mod):
        self.mod, self.calls = mod, 0

    def __getattr__(self, name):
        return getattr(self.mod, name)

    def update_cluster_means(self, *a):
        self.calls += 1
        return self.mod.update_cluster_means(*a)


def run_case(name, k, iters, seed, thresh=1e-5, data=None, points=None):
    from scipy.cluster.vq import _vq_impl, kmeans
    c = dict(name=name, k=k, iter=iters, seed=seed, thresh=thresh)
    if points is not None:
        c["points"] = np.asarray(points, dtype=np.float64).tolist()
    else:
        c["data"] = data
    obs = rk.case_obs(c)
    np.random.seed(seed)
    book, dist = kmeans(obs, k, iter=iters, thresh=thresh)
    next_np = np.random.random(4)
    np.random.seed(seed)
    starts = rk.draw_starts(len(obs), k, iters)
    real = _vq_impl._vq
    books, dists, its = [], [], []
    try:
        for idx in starts:
            _vq_impl._vq = cnt = _Counted(real)
            b, d = _vq_impl._kmeans(obs, obs[idx], thresh=thresh)
            books.append(np.asarray(b))
            dists.append(float(d))
            its.append(cnt.calls)
    finally:
        _vq_impl._vq = real
    win = min(range(iters), key=lambda r: (dists[r], r))
    assert np.array_equal(books[win], book) and dists[win] == dist, f"{name}: the restarts do not reproduce scipy's winner"
    c.update(n=len(obs), best=win, dist=float(dist))
    arrays = dict(book=np.asarray(book), next_np=next_np, starts=starts, run_k=np.array([len(b) for b in books], np.int64),
                  run_books_flat=np.concatenate(books), run_dists=np.array(dists), run_iters=np.array(its, np.int64))
    print(f"{name}: n = {len(obs)}, k' = {len(book)}, dist = {dist!r}, restart k' {sorted(set(arrays['run_k'].tolist()))}, "
          f"iterations {min(its)}-{max(its)}", flush=True)
    return c, arrays


def main():
    argp = argparse.ArgumentParser()
    argp.add_argument("--out", default=os.path.join(GOLD, "kmeans_cases.npz"))
    argp.add_argument("--no-coco", action="store_true", help="skip the ~790 k label case (about a minute of scipy)")
    args = argp.parse_args()
    city = dict(n_img=60, per_img=50, clusters=CITY, spread=0.35)
    specs = [
        ("city", dict(k=9, iters=30, seed=1, data=dict(synth=dict(city, seed=3), img_size=640))),
        # rounded to whole pixels at a small size: duplicate starts, clusters dropped
        ("dup", dict(k=9, iters=30, seed=2, data=dict(synth=dict(city, seed=5, n_img=30), img_size=96, round=True))),
        ("few_distinct", dict(k=9, iters=10, seed=3, points=[[1.0, 2.0], [3.0, 1.5], [0.5, 0.5], [2.0, 2.0], [4.0, 4.0]] * 8)),
        ("n5", dict(k=3, iters=10, seed=4, points=[[0.3, 1.2], [2.5, 0.7], [1.1, 1.9], [0.2, 0.4], [3.3, 2.8]])),
        ("n127", dict(k=9, iters=20, seed=5, data=dict(synth=dict(city, seed=7), img_size=640, take=127))),
        ("n128", dict(k=9, iters=20, seed=6, data=dict(synth=dict(city, seed=7), img_size=640, take=128))),
        ("n129", dict(k=9, iters=20, seed=7, data=dict(synth=dict(city, seed=7), img_size=640, take=129))),
        ("n8191", dict(k=9, iters=20, seed=8, data=dict(synth=dict(city, seed=9, n_img=200), img_size=1024, take=8191))),
        ("n8192", dict(k=9, iters=20, seed=9, data=dict(synth=dict(city, seed=9, n_img=200), img_size=1024, take=8192))),
        ("n8193", dict(k=9, iters=20, seed=10, data=dict(synth=dict(city, seed=9, n_img=200), img_size=1024, take=8193))),
        ("k32", dict(k=32, iters=8, seed=11, data=dict(synth=dict(city, seed=13), img_size=640))),
    ]
    if not args.no_coco:
        specs.append(("coco", dict(k=9, iters=30, seed=12, data=dict(synth=dict(seed=17, n_img=7900, per_img=100, clusters=CITY8, spread=0.45,
                                                                              shapes=BIG_SHAPES), img_size=1024))))
    arrays, meta = {}, []
    for name, kw in specs:
        m, a = run_case(name, **kw)
        meta.append(m)
        for key, v in a.items():
            arrays[f"{name}_{key}"] = v
    arrays["meta_json"] = np.frombuffer(json.dumps(dict(cases=meta)).encode(), np.uint8)
    np.savez_compressed(args.out, **arrays)
    print("wrote", args.out, os.path.getsize(args.out), "bytes")


if __name__ == "__main__":
    main()
