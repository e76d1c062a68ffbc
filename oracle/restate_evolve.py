"""TEST INFRASTRUCTURE - the reference's --evolve loop (train.py:637-717) and print_mutation (utils/general.py:528-556) restated for the
host tests, written from their statements rather than from multiyolov5_b200.train.evolve, plus the stub training run and frozen clock that
oracle/make_golden_evolve.py drives the unmodified reference with (tests/golden/evolve_cases.json).

    generation(hyp, evolve_txt, now, rng)      the hyp one generation trains with (parent draw, mutation, limits)
    record(hyp, results, evolve_txt, yaml_file) print_mutation's files
    run(hyp, results_fn, generations, ...)     both, generation after generation; returns the hyp of every generation
"""
import bisect
import itertools
import os
import random

import numpy as np

META = [("lr0", 1, 1e-5, 1e-1), ("lrf", 1, 0.01, 1.0), ("momentum", 0.3, 0.6, 0.98), ("weight_decay", 1, 0.0, 0.001),
        ("warmup_epochs", 1, 0.0, 5.0), ("warmup_momentum", 1, 0.0, 0.95), ("warmup_bias_lr", 1, 0.0, 0.2), ("box", 1, 0.02, 0.2),
        ("cls", 1, 0.2, 4.0), ("cls_pw", 1, 0.5, 2.0), ("obj", 1, 0.2, 4.0), ("obj_pw", 1, 0.5, 2.0), ("iou_t", 0, 0.1, 0.7),
        ("anchor_t", 1, 2.0, 8.0), ("anchors", 2, 2.0, 10.0), ("fl_gamma", 0, 0.0, 2.0), ("hsv_h", 1, 0.0, 0.1), ("hsv_s", 1, 0.0, 0.9),
        ("hsv_v", 1, 0.0, 0.9), ("degrees", 1, 0.0, 45.0), ("translate", 1, 0.0, 0.9), ("scale", 1, 0.0, 0.9), ("shear", 1, 0.0, 10.0),
        ("perspective", 0, 0.0, 0.001), ("flipud", 1, 0.0, 1.0), ("fliplr", 0, 0.0, 1.0), ("mosaic", 1, 0.0, 1.0), ("mixup", 1, 0.0, 1.0)]

# data/hyp.scratch.yaml of the reference with its commented `anchors: 3` line enabled
HYP_SCRATCH = dict(lr0=0.0015, lrf=0.2, momentum=0.937, weight_decay=0.0005, warmup_epochs=3.0, warmup_momentum=0.8, warmup_bias_lr=0.1,
                   box=0.05, cls=0.5, cls_pw=1.0, obj=1.0, obj_pw=1.0, iou_t=0.2, anchor_t=4.0, anchors=3, fl_gamma=0.0, hsv_h=0.015,
                   hsv_s=0.7, hsv_v=0.4, degrees=0.0, translate=0.1, scale=0.5, shear=0.0, perspective=0.0, flipud=0.0, fliplr=0.5,
                   mosaic=1.0, mixup=0.0)

CLOCK0 = 1_700_000_000


def clock(calls):
    """the frozen wall clock of the fixtures: a function of how many training runs have started"""
    return CLOCK0 + 3607 * calls + 0.25


def stub_results(hyp, seed, zero=False):
    """7 training results (P, R, mAP@.5, mAP@.5:.95, 3 val losses) as a seeded function of the hyp; zero=True: mAP 0, as an untrained
    model scores"""
    key = sum(int(round(v * 1e5)) * (i + 1) for i, v in enumerate(hyp.values()))
    rs = np.random.RandomState((seed * 1_000_003 + key) % 2 ** 32)
    p, r = rs.uniform(0.0, 1.0, 2)
    m50 = 0.0 if zero else rs.uniform(0.0, 0.8)
    m = 0.0 if zero else m50 * rs.uniform(0.3, 0.7)
    return (float(p), float(r), float(m50), float(m), *[float(v) for v in rs.uniform(0.01, 0.2, 3)])


def fitness(x):
    return (x[:, :4] * [0.0, 0.0, 0.1, 0.9]).sum(1)


def choices38(n, weights, rng):
    cum = list(itertools.accumulate(weights))
    return bisect.bisect(cum, rng.random() * (cum[-1] + 0.0), 0, n - 1)


def generation(hyp, evolve_txt, now, rng=random):
    hyp = dict(hyp)
    if os.path.exists(evolve_txt):
        x = np.loadtxt(evolve_txt, ndmin=2)
        n = min(5, len(x))
        x = x[np.argsort(-fitness(x))][:n]
        f = fitness(x)
        x = x[choices38(n, f - f.min(), rng)]
        np.random.seed(int(now))
        gains = np.array([m[1] for m in META])
        v = np.ones(len(META))
        while (v == 1).all():
            v = (gains * (np.random.random(len(META)) < 0.8) * np.random.randn(len(META)) * np.random.random() * 0.2 + 1).clip(0.3, 3.0)
        for i, k in enumerate(hyp):
            hyp[k] = float(x[7 + i] * v[i])
    for k, _, lo, hi in META:
        hyp[k] = round(min(max(hyp[k], lo), hi), 5)
    return hyp


def record(hyp, results, evolve_txt, yaml_file):
    import yaml
    with open(evolve_txt, "a") as f:
        f.write("".join("%10.4g" % r for r in results) + "".join("%10.3g" % v for v in hyp.values()) + "\n")
    x = np.unique(np.loadtxt(evolve_txt, ndmin=2), axis=0)
    x = x[np.argsort(-fitness(x))]
    np.savetxt(evolve_txt, x, "%10.3g")
    best = {k: float(x[0, 7 + i]) for i, k in enumerate(hyp)}
    with open(yaml_file, "w") as f:
        f.write("# Hyperparameter Evolution Results\n# Generations: %g\n# Metrics: " % len(x) + "".join("%10.4g" % r for r in x[0, :7]) + "\n\n")
        yaml.dump(best, f, sort_keys=False)


def run(hyp, results_fn, generations, evolve_txt, yaml_file, calls0=0, rng=random):
    """the hyps of `generations` generations; results_fn(hyp, k) gives generation k's results; the clock reads clock(calls0 + k)"""
    hyps = []
    for k in range(generations):
        hyp = generation(hyp, evolve_txt, clock(calls0 + k), rng)
        hyps.append(dict(hyp))
        record(hyp, results_fn(dict(hyp), k), evolve_txt, yaml_file)
    return hyps


def anchor_table(n, lo=6.0, hi=420.0):
    """n anchors per level (3 levels) in pixels, as a yaml lists them: sizes spaced geometrically from lo to hi over the 3n anchors, in
    increasing area with the level (stride 8, 16, 32), aspect ratios cycling through 1, 2, 1/2 - what autoanchor leaves after replacing the
    placeholders of Model(cfg, anchors=n)"""
    s = np.geomspace(lo, hi, 3 * n)
    ar = [1.0, 2.0, 0.5]
    wh = [(round(float(v * np.sqrt(ar[j % 3])), 1), round(float(v / np.sqrt(ar[j % 3])), 1)) for j, v in enumerate(s)]
    return [[c for w, h in wh[l * n:(l + 1) * n] for c in (w, h)] for l in range(3)]


LOSS_SHAPE = (2, 64, 128)           # B, H, W of the anchor-count loss fixtures (tests/golden/anchor_count_cases.npz)


def loss_predictions(na, no=15):
    """the head outputs the anchor-count loss fixtures evaluate ComputeLoss on, drawn from a seed (they are not stored), and the random
    state the fixture's targets were drawn from next"""
    B, H, W = LOSS_SHAPE
    rs = np.random.RandomState(100 + na)
    return [rs.normal(0, 1.0, (B, na, H // s, W // s, no)).astype(np.float32) for s in (8, 16, 32)], rs
