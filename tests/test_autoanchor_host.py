"""CPU: the reference's autoanchor.  The numpy restatement of the device arithmetic (oracle/restate_autoanchor.py) against every case the
reference computed (tests/golden/autoanchor_cases.npz, oracle/make_golden_autoanchor.py): Detect buffers bit for bit, decisions, the
per-generation fitness, and the state of `random` / `numpy.random` afterwards.  Pins of the torch details the kernels restate, the order
independence of the exact fp64 sum, and the host-side argument errors of utils.autoanchor."""
import os
import random
from fractions import Fraction

import numpy as np
import pytest
import torch

from oracle import restate_autoanchor as ra

GOLD = os.path.join(os.path.dirname(__file__), "golden")


def _cases():
    return ra.load_cases(os.path.join(GOLD, "autoanchor_cases.npz"))


def _digest(labels):
    import hashlib
    h = hashlib.sha256()
    for l in labels:
        h.update(np.ascontiguousarray(l).tobytes())
    return h.hexdigest()


def test_fixture_covers_the_cases():
    names = {c["name"] for c in _cases()}
    assert {"fit", "replace", "flip", "tiny", "thr291", "large", "kmean_verbose"} <= names
    by = {c["name"]: c for c in _cases()}
    assert "New anchors saved" in by["flip"]["stdout"] and "Reversing anchor order" in by["flip"]["stdout"]
    assert "Extremely small objects" in by["tiny"]["stdout"]
    assert not by["fit"]["evolved"] and "Attempting" not in by["fit"]["stdout"]
    assert sum(len(l) for l in ra.case_dataset(by["large"])[1]) > 15000
    if "keep" in by:
        assert "Original anchors better" in by["keep"]["stdout"]


@pytest.mark.parametrize("name", ["fit", "replace", "flip", "tiny", "thr291", "large", "kmean_verbose"])
def test_restatement_reproduces_the_reference(name):
    cases = {c["name"]: c for c in _cases()}
    if name not in cases:
        pytest.skip(f"the fixture has no {name} case (no seed produced it)")
    c = cases[name]
    shapes0, labels = ra.case_dataset(c)
    assert _digest(labels) == c["digest"], "the seeded label draw changed"
    shapes = ra.shapes_wh(shapes0)
    random.seed(c["seed"]); np.random.seed(c["seed"])
    if c["call"] == "check":
        out = ra.check_anchors(shapes, labels, c["anchor_grid0"], np.array(c["stride"], np.float32), c["thr"], c["imgsz"])
        assert np.array_equal(out["anchor_grid"], c["anchor_grid1"])
        if out["replaced"]:
            assert np.array_equal(out["anchors"], c["anchors1"])
        else:
            assert np.array_equal(c["anchors1"], c["anchors0"])
        assert out["replaced"] == ("New anchors saved" in c["stdout"])
        assert out["flipped"] == ("Reversing anchor order" in c["stdout"])
        line = f"anchors/target = {float(out['aat']):.2f}, Best Possible Recall (BPR) = {float(out['bpr']):.4f}"
        assert line in c["stdout"]
    else:
        out = ra.kmean_anchors(shapes, labels, c["n"], c["imgsz"], c["thr"], c["gen"])
        assert np.array_equal(out["k"], c["returned"])
    if c["evolved"]:
        assert np.array_equal(out["k_kmeans"], c["k_kmeans"])
        assert np.array_equal(out["k"], c["k"])
        assert np.array_equal(out["fg"], c["fg_exact"])
        assert out["accepted"] == c["accepted"]
        # the exact fitness stays within a few ulp of torch's cascade sum
        assert np.all(np.abs(out["fg"] - c["fg_torch"]) <= 4 * np.spacing(c["fg_torch"]))
    assert np.array_equal(np.array([random.random(), random.random()]), c["next_py"])
    assert np.array_equal(np.random.random(4), c["next_np"])


def test_product_draws_are_the_restatements():
    from multiyolov5_b200.utils.autoanchor import draw_mutations
    np.random.seed(5)
    a = draw_mutations(300, (9, 2))
    sa = np.random.get_state()
    np.random.seed(5)
    b = ra.draw_mutations(300, (9, 2))
    sb = np.random.get_state()
    assert np.array_equal(a, b) and np.array_equal(sa[1], sb[1]) and sa[2] == sb[2]
    assert not np.any(np.all(a == 1, axis=(1, 2)))


def test_colorstr_prefix():
    from multiyolov5_b200.utils.autoanchor import colorstr
    assert colorstr("autoanchor: ") == "\033[34m\033[1mautoanchor: \033[0m"


# ---- pins of the torch arithmetic the kernels restate ------------------------------------------------------------------------------
def test_torch_rtruediv_is_a_correctly_rounded_reciprocal():
    g = torch.Generator().manual_seed(0)
    for dt, npdt in ((torch.float32, np.float32), (torch.float64, np.float64)):
        r = (torch.rand(200000, generator=g, dtype=torch.float64) * 50 + 1e-3).to(dt)
        assert torch.equal(1. / r, r.reciprocal())
        assert np.array_equal((1. / r).numpy(), npdt(1) / r.numpy())


def test_torch_fp32_cast_of_float64_anchors_rounds_to_nearest():
    k = np.random.default_rng(1).uniform(2, 400, (1000, 2))
    assert np.array_equal(torch.tensor(k, dtype=torch.float32).numpy(), k.astype(np.float32))


def test_comparisons_run_in_the_tensor_dtype():
    thr = 1. / 2.91
    t32 = np.float32(thr)
    assert float(t32) > thr                                   # fp32(1 / 2.91) lies above the double
    x = torch.tensor([float(t32)], dtype=torch.float32)
    assert not bool(x > thr)                                  # fp32 comparison: equal, not greater
    assert bool(x.double() > thr)                             # fp64 comparison: greater


def test_fp32_over_float64_numpy_promotes_to_float64():
    wh = torch.rand(5, 2)
    k = np.array([[10., 13.], [16., 30.]])
    r = wh[:, None] / k[None]
    assert r.dtype == torch.float64
    assert (torch.min(r, 1. / r).min(2)[0] > 0.25).dtype == torch.bool


def test_torch_cpu_mean_divides_its_sum_by_n():
    """integer-valued fp32 (an exact sum S): the mean is fp32(S) / fp32(n), not fp32(S) * fp32(1 / n)"""
    g = torch.Generator().manual_seed(0)
    differing = 0
    for n in range(3, 6000, 7):
        t = torch.randint(0, 2, (n,), generator=g).float()
        S = np.float32(t.sum().item())
        div, mul = np.float32(S / np.float32(n)), np.float32(S * np.float32(1.0 / n))
        assert np.float32(t.mean().item()) == div
        differing += div != mul
    assert differing > 50                                     # the two scalings do differ on these cases


def test_exact_sum_is_order_independent():
    """terms of the fitness (fp32 in (1/16, 1] or 0) sum exactly in fp64: any order, any chunking, equal to the rational sum"""
    rng = np.random.default_rng(3)
    n = 200000
    best = rng.uniform(0.0, 1.0, n).astype(np.float32)
    best[rng.random(n) < 0.01] = 1.0
    term = np.where(best > np.float32(1 / 16), best, np.float32(0)).astype(np.float64)
    ref = float(sum(Fraction(float(v)) for v in term[:5000]))
    assert float(np.sum(term[:5000])) == ref
    s0 = np.sum(term)
    for seed in range(4):
        p = np.random.default_rng(seed).permutation(n)
        assert np.sum(term[p]) == s0
        acc = 0.0
        for q in np.array_split(term[p], 1 + seed * 37)[::-1]:      # per-CTA partials, added in any order
            acc += float(np.sum(q))
        assert acc == s0
        seq = 0.0
        for v in term[p][:20000]:
            seq += v
        assert seq == np.sum(term[p][:20000])


def test_restated_fitness_matches_torch_within_a_few_ulp():
    shapes0, labels = ra.synth_dataset(9, 30, 60, [(12, 30), (40, 25), (90, 55)])
    wh0 = ra.label_wh(ra.shapes_wh(shapes0), labels, 640)
    wh32 = wh0[(wh0 >= 2).any(1)].astype(np.float32)
    k = np.array([[8, 20], [12, 30], [30, 20], [40, 25], [60, 40], [90, 55], [120, 80], [200, 120], [300, 200]], np.float64)
    r = torch.from_numpy(wh32)[:, None] / torch.tensor(k, dtype=torch.float32)[None]
    best = torch.min(r, 1. / r).min(2)[0].max(1)[0]
    f_t = np.float32((best * (best > 0.25).float()).mean().item())
    f_e = ra.fitness(wh32, k, 0.25)
    assert abs(f_t - f_e) <= 4 * np.spacing(f_e)


# ---- argument errors ------------------------------------------------------------------------------------------------------------------
def test_a_path_raises_not_implemented():
    from multiyolov5_b200.utils import autoanchor as aa
    with pytest.raises(NotImplementedError):
        aa.kmean_anchors("./data/coco128.yaml")
    with pytest.raises(NotImplementedError):
        aa.dataset_shapes_labels("train.txt")


def test_a_dataset_without_shapes_and_labels_raises():
    from multiyolov5_b200.utils import autoanchor as aa
    with pytest.raises(TypeError):
        aa.dataset_shapes_labels(object())


def test_reference_style_dataset_shapes():
    from multiyolov5_b200.utils import autoanchor as aa

    class D:
        shapes = [[640, 480], [320, 320]]
        labels = [np.zeros((0, 5), np.float32)] * 2
    s, l = aa.dataset_shapes_labels(D())
    assert s.dtype == np.float64 and s.shape == (2, 2) and l is D.labels
