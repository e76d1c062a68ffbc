"""CPU: the --multi-scale draw (reference train.py:354-359) against tests/golden/multiscale_cases.npz (oracle/make_golden_multiscale.py
executes the reference's statements), and the host side of the shared train workspace of the det lane."""
import os
import random

import numpy as np
import pytest

from multiyolov5_b200.train import MultiScale

GOLD = os.path.join(os.path.dirname(__file__), "golden", "multiscale_cases.npz")


def _cases():
    g = np.load(GOLD)
    for k in range(int(g["n_cases"][0])):
        seed, imgsz, gs, H, W = (int(v) for v in g[f"case{k}_meta"])
        yield seed, imgsz, gs, (H, W), g[f"case{k}_same"], g[f"case{k}_ns"], float(g[f"case{k}_next"][0])


def test_size_equals_reference_draw_for_draw_and_consumes_the_same_stream():
    n = 0
    for seed, imgsz, gs, shape, same, ns, nxt in _cases():
        ms = MultiScale(imgsz, gs)
        rng = random.Random(seed)
        for i in range(len(same)):
            got = ms.size(shape, rng)
            if same[i]:
                assert got is None, (seed, i, got)
            else:
                assert got == [int(v) for v in ns[i]], (seed, i, got, ns[i])
        assert rng.random() == nxt, seed
        n += 1
    assert n >= 7


def test_size_draws_from_the_global_random_by_default():
    ms = MultiScale(1024)
    random.seed(11)
    a = [ms.size((1024, 1024)) for _ in range(50)]
    rng = random.Random(11)
    assert a == [ms.size((1024, 1024), rng) for _ in range(50)]


def test_shapes_is_exactly_the_set_the_draw_reaches():
    for seed, imgsz, gs, shape, same, ns, _ in _cases():
        reached = {tuple(int(v) for v in r) for r in ns}
        assert set(MultiScale(imgsz, gs).shapes(shape)) == reached, (seed, shape)
    s = MultiScale(1024).shapes((1024, 1024))
    assert s == [(v, v) for v in range(512, 1537, 32)] and len(s) == 33


def test_non_integral_bounds_raise_like_python_311_randrange():
    with pytest.raises(ValueError):
        MultiScale(641)


def test_shared_workspace_capacity_is_the_largest_shape_and_holds_every_buffer():
    from multiyolov5_b200.engine import shared_train_plans
    from multiyolov5_b200.models.yolo import Model
    model = Model("yolov5s_city_seg.yaml")
    shapes = MultiScale(1024).shapes((1024, 1024))
    pbs, cap = shared_train_plans(model, 4, shapes)
    assert cap == 3_047_912_448
    assert cap == max(pb.workspace_bytes for pb in pbs.values()) == pbs[(1536, 1536)].workspace_bytes
    # the private workspaces of the 33 shapes would not fit an 80 GB card twice over (activations + gradients)
    assert 2 * sum(pb.workspace_bytes for pb in pbs.values()) > 80e9
    es = {0: 2, 1: 4}                                       # plan.py dtypes: F16, F32
    for (H, W), pb in pbs.items():
        assert pb.workspace_bytes <= cap
        for b in pb.bufs:
            size = 4 * b.h * b.w * b.c * es[b.dtype]
            assert 0 <= b.offset and b.offset % 256 == 0 and b.offset + size <= pb.workspace_bytes, (H, W, b)
