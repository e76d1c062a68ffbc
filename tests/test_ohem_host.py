"""CPU: the reference's OhemCELoss.  The restatement (oracle/restate_ohem.py) against every case the reference computed
(tests/golden/ohem_cases.npz, oracle/make_golden_ohem.py); the numpy model of the device selection (order-preserving keys, four digit
passes, the tie cutoff) against a sort on adversarial vectors; and the ValueErrors of OhemCELoss and of Trainer(seg_loss=)."""
import os

import numpy as np
import pytest
import torch

from oracle import restate_ohem as ro

GOLD = os.path.join(os.path.dirname(__file__), "golden")


def _cases():
    return ro.load_cases(os.path.join(GOLD, "ohem_cases.npz"))


def test_restatement_reproduces_the_reference_cases():
    g = _cases()
    assert g["thresh_t"] == ro.thresh_t(0.7)
    for c in g["cases"]:
        ps = [p.clone().requires_grad_(True) for p in c["logits"]]
        loss = ro.ohem_loss(ps if c["aux"] else ps[0], c["labels"], c["thresh"], c["ignore_index"], c["aux"], c["aux_weight"])
        loss.backward()
        if c["name"] == "all_ignored":
            assert torch.isnan(loss) and torch.isnan(c["loss"])
        else:
            torch.testing.assert_close(loss.detach(), c["loss"], rtol=1e-6, atol=0)
        for p, gr in zip(ps, c["grad"]):
            torch.testing.assert_close(p.grad, gr, rtol=1e-6, atol=1e-9)


def _branch(logits, labels, th):
    loss = torch.nn.functional.cross_entropy(logits, labels, ignore_index=-1, reduction="none").view(-1).numpy()
    n_valid = int((labels != -1).sum())
    mask, denom = ro.select(loss, n_valid, th)
    return ("threshold" if int((loss > np.float32(th)).sum()) >= n_valid // 16 else "topk"), mask, denom, loss


def test_the_cases_cover_both_branches_and_the_model_selects_what_the_reference_averages():
    g = _cases()
    th = g["thresh_t"]
    seen = {}
    for c in g["cases"]:
        for p, gr in zip(c["logits"], c["grad"]):
            branch, mask, denom, loss = _branch(p, c["labels"], th)
            seen.setdefault(c["name"], []).append(branch)
            rows = (gr.permute(0, 2, 3, 1).reshape(-1, gr.shape[1]) != 0).any(1).numpy()
            valid = (c["labels"] != -1).view(-1).numpy()
            np.testing.assert_array_equal(rows, mask & valid)         # taken ignored pixels have no gradient
    assert seen["threshold"] == ["threshold"] and seen["topk"] == ["topk"] and seen["nmin0"] == ["threshold"]
    assert sorted(set(seen["aux"])) == ["threshold", "topk"]


def _sorted_topk(v, k):
    mask = np.zeros(v.size, bool)
    mask[np.argsort(-v.astype(np.float64), kind="stable")[:k]] = True      # float64: -0.0 and +0.0 compare equal, ties keep index order
    return mask


def _adversarial():
    r = np.random.default_rng(7)
    n = 3 * ro.CHUNK + 123
    yield "all_equal", np.full(n, 1.25, np.float32)
    v = r.random(n, dtype=np.float32)
    v[r.choice(n, 700, replace=False)] = np.float32(0.5)
    yield "many_ties", v
    z = np.zeros(n, np.float32)
    z[r.choice(n, n // 3, replace=False)] = np.float32(-0.0)
    z[r.choice(n, 50, replace=False)] = -np.float32(1e-7) * r.random(50, dtype=np.float32)
    z[r.choice(n, 40, replace=False)] = r.random(40, dtype=np.float32)
    yield "zeros_negzeros_tiny_negatives", z
    w = r.standard_normal(n).astype(np.float32) * np.float32(3)
    w[r.choice(n, 300, replace=False)] = np.float32(np.inf)
    w[r.choice(n, 300, replace=False)] = -np.float32(2.0)
    yield "mixed_signs", w
    d = np.repeat(r.random(40, dtype=np.float32), (n + 39) // 40)[:n]              # long runs of equal values across chunks
    yield "runs", d


@pytest.mark.parametrize("name,v", list(_adversarial()), ids=[n for n, _ in _adversarial()])
def test_device_selection_model_matches_a_sort(name, v):
    n = v.size
    for k in sorted({0, 1, 2, 17, 700, 701, n // 16, n // 3, ro.CHUNK, ro.CHUNK + 1, n - 1, n}):
        got = ro.select_topk(v, k)
        assert got.sum() == k, (name, k)
        np.testing.assert_array_equal(got, _sorted_topk(v, k), err_msg=f"{name} k={k}")


def test_key_map_orders_floats():
    v = np.array([-np.inf, -3.0, -1e-30, -0.0, 0.0, 1e-45, 1e-30, 0.7, 3.0, np.inf], np.float32)
    k = ro.keys(v)
    assert k[3] == k[4]                                                          # -0.0 == +0.0
    assert all(int(a) < int(b) for i, (a, b) in enumerate(zip(k[:-1], k[1:])) if i != 3)


def test_threshold_branch_and_denominators():
    v = np.array([0.1, 0.5, 0.9, 0.0, 2.0] * 20, np.float32)
    mask, denom = ro.select(v, 100, 0.4)                                         # 60 hard >= n_min 6
    np.testing.assert_array_equal(mask, v > np.float32(0.4))
    assert denom == 60
    mask, denom = ro.select(v, 100, 5.0)                                         # none hard: the 6 largest
    assert denom == 6 and mask.sum() == 6 and (v[mask] == 2.0).all()
    mask, denom = ro.select(v, 15, 5.0)                                          # n_min 0, nothing hard: 0 / 0
    assert denom == 0 and not mask.any()


@pytest.mark.parametrize("thresh", [0.0, -0.5, 1.0001, 2.0, float("nan")])
def test_ohem_rejects_thresholds_outside_0_1(thresh):
    from multiyolov5_b200.utils.loss import OhemCELoss
    with pytest.raises(ValueError):
        OhemCELoss(thresh)


def test_ohem_defaults_and_cpu_tensors():
    from multiyolov5_b200.utils.loss import OhemCELoss
    m = OhemCELoss()
    assert m.thresh_t == ro.thresh_t(0.5) and m.ignore_index == -1 and not m.aux and m.aux_weight == [0.15, 0.05]
    assert OhemCELoss(1.0).thresh_t == 0.0
    with pytest.raises(ValueError):
        m(torch.zeros(1, 3, 4, 4), torch.zeros(1, 4, 4, dtype=torch.long))
    with pytest.raises(ValueError):
        OhemCELoss(0.7, aux=True)([torch.zeros(1, 3, 4, 4)], torch.zeros(1, 4, 4, dtype=torch.long))


@pytest.mark.parametrize("yml,loss_kw", [("yolov5s_city_seg.yaml", dict(aux=True)), ("yolov5s_city_seg_bise.yaml", dict(aux=False)),
                                         ("yolov5s_city_seg.yaml", None)])
def test_trainer_rejects_a_seg_loss_that_does_not_fit_the_head(yml, loss_kw):
    from multiyolov5_b200.models.yolo import Model
    from multiyolov5_b200.train import Trainer
    from multiyolov5_b200.utils.loss import OhemCELoss, SegmentationLosses
    seg_loss = SegmentationLosses() if loss_kw is None else OhemCELoss(0.7, **loss_kw)
    with pytest.raises(ValueError):
        Trainer(Model(yml), {}, 4, seg_loss=seg_loss)
