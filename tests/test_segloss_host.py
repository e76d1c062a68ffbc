"""CPU: the reference's class-weighted CE and SegFocalLoss.  The fp64 restatement (oracle/restate_segloss.py) against every case the
reference computed (tests/golden/segloss_cases.npz, oracle/make_golden_segloss.py); the generator's inputs against the committed file;
the argument errors of SegFocalLoss; and the ValueErrors of Trainer(seg_loss=) for the weighted CE and the focal loss."""
import os

import numpy as np
import pytest
import torch

from oracle import make_golden_segloss as mg
from oracle import restate_segloss as rs

GOLD = os.path.join(os.path.dirname(__file__), "golden")
PATH = os.path.join(GOLD, "segloss_cases.npz")


def _cases():
    return rs.load_cases(PATH)["cases"]


def test_the_cases_cover_what_the_reference_offers():
    cs = {c["name"]: c for c in _cases()}
    focal = [c for c in cs.values() if c["kind"] == "focal"]
    assert {c["gamma"] for c in focal} == {0.0, 0.5, 1.5, 2.0}
    assert {c["reduction"] for c in focal} == {"mean", "sum"}
    assert {c["has_weight"] for c in focal} == {True, False}
    assert cs["wce_bise"]["n_outputs"] == 3 and cs["focal_g2_2cls"]["logits"][0].shape[1] == 2
    assert (cs["wce_all_ignored"]["labels"] == -1).all() and (cs["focal_g2_alpha_all_ignored"]["labels"] == -1).all()


def test_restatement_reproduces_the_reference_cases():
    for c in _cases():
        loss, grads = rs.case_value(c)
        ref = float(c["loss"])
        if np.isnan(ref):
            assert np.isnan(loss), c["name"]
        else:
            assert abs(loss - ref) <= 2e-6 * abs(ref), (c["name"], loss, ref)
        for g, gr in zip(grads, c["grad"]):
            fin = np.isfinite(gr)
            np.testing.assert_array_equal(np.isfinite(g), fin, err_msg=c["name"])
            assert np.abs(g[fin] - gr[fin]).max(initial=0.0) <= 1e-5 * np.abs(gr[fin]).max(initial=1.0) + 1e-9, c["name"]


def test_the_edge_cases_behave_as_the_reference():
    cs = {c["name"]: c for c in _cases()}
    # every pixel ignored: NaN loss; zero gradients for the weighted CE, NaN for the focal loss (A = NaN enters every pixel's gradient)
    assert np.isnan(cs["wce_all_ignored"]["loss"]) and (cs["wce_all_ignored"]["grad"][0] == 0).all()
    assert np.isnan(cs["focal_g2_alpha_all_ignored"]["loss"]) and np.isnan(cs["focal_g2_alpha_all_ignored"]["grad"][0]).all()
    # the saturated pixel with gamma < 1: a finite loss, that pixel's gradient non-finite, every other pixel's finite
    c = cs["focal_g05_alpha_saturated"]
    g = c["grad"][0]
    assert np.isfinite(c["loss"])
    bad = ~np.isfinite(g).all(1)
    assert bad.sum() == 1 and bad[0, 1, 2]
    # the default ignore_index -100 is honoured
    assert (cs["focal_g2_default_ignore"]["labels"] == -100).any()


def test_generator_reproduces_the_committed_inputs():
    g = np.load(PATH)
    drawn = mg.draw_inputs()
    assert [s[0] for s, *_ in drawn] == [c["name"] for c in _cases()]
    for spec, logits, labels, weight in drawn:
        n = spec[0]
        np.testing.assert_array_equal(labels.numpy(), g[f"{n}_labels"])
        for i, x in enumerate(logits):
            np.testing.assert_array_equal(x.numpy(), g[f"{n}_logits_{i}"])
        if weight is None:
            assert f"{n}_weight" not in g.files
        else:
            np.testing.assert_array_equal(weight.numpy(), g[f"{n}_weight"])


def test_generator_reproduces_the_committed_file_from_the_reference(tmp_path):
    from oracle import ref_shims
    if not ref_shims.reference_available():
        pytest.skip("MYOLO_REFERENCE_ROOT does not name a reference checkout")
    import subprocess
    import sys
    out = tmp_path / "segloss_cases.npz"
    subprocess.run([sys.executable, mg.__file__, "--out", str(out)], check=True, capture_output=True)
    a, b = np.load(out), np.load(PATH)
    assert sorted(a.files) == sorted(b.files)
    for k in a.files:
        np.testing.assert_array_equal(a[k], b[k], err_msg=k)


def test_focal_loss_arguments():
    from multiyolov5_b200.utils.loss import SegFocalLoss
    m = SegFocalLoss()
    assert m.gamma == 2.0 and m.weight is None and m.ignore_index == -100 and m.reduction == "mean"
    with pytest.raises(NotImplementedError, match="broadcast"):
        SegFocalLoss(reduction="none")
    with pytest.raises(ValueError):
        SegFocalLoss(reduction="avg")
    for gamma in (-1.0, float("nan"), float("inf")):
        with pytest.raises(ValueError):
            SegFocalLoss(gamma=gamma)
    with pytest.raises(ValueError):                                      # CPU tensors: the loss runs in the library's kernels
        m(torch.zeros(1, 3, 4, 4), torch.zeros(1, 4, 4, dtype=torch.long))
    w = SegFocalLoss(alpha=[1.0, 2.0, 0.5]).weight
    assert w.dtype == torch.float32 and w.tolist() == [1.0, 2.0, 0.5]


def _two_class_model():
    from multiyolov5_b200.models.yolo import Model
    from oracle import synth
    cfg = synth.load_cfg("yolov5s_city_seg.yaml")
    cfg["nc"], cfg["n_segcls"] = 1, 2
    return Model(cfg)


W19 = [1.0] * 19


@pytest.mark.parametrize("yml,make", [
    ("yolov5s_city_seg_bise.yaml", lambda L: L.SegFocalLoss(gamma=2, ignore_index=-1)),                # no aux in SegFocalLoss
    ("yolov5s_city_seg.yaml", lambda L: L.SegFocalLoss(gamma=2, ignore_index=-1, reduction="sum")),
    ("yolov5s_city_seg.yaml", lambda L: L.SegFocalLoss(gamma=2)),                                       # ignore_index -100
    ("yolov5s_city_seg.yaml", lambda L: L.SegFocalLoss(gamma=2, alpha=[1.0] * 18, ignore_index=-1)),    # wrong length
    ("yolov5s_city_seg.yaml", lambda L: L.SegmentationLosses(weight=torch.ones(20))),
    ("yolov5s_city_seg.yaml", lambda L: L.SegmentationLosses(weight=torch.tensor(W19), ignore_index=255)),
    ("yolov5s_city_seg.yaml", lambda L: L.SegmentationLosses(aux=True, weight=torch.tensor(W19))),       # aux on a plain head
    ("yolov5s_city_seg_bise.yaml", lambda L: L.SegmentationLosses(weight=torch.tensor(W19))),            # no aux on BiSe
    ("yolov5s_city_seg_bise.yaml", lambda L: L.SegmentationLosses(aux=True, aux_num=1, weight=torch.tensor(W19))),
    ("yolov5s_city_seg.yaml", lambda L: torch.nn.CrossEntropyLoss()),
], ids=["focal_bise", "focal_sum", "focal_ignore", "focal_alpha_len", "wce_len", "wce_ignore", "wce_aux_plain", "wce_bise_no_aux",
        "wce_bise_aux_num1", "other_module"])
def test_trainer_rejects_a_weighted_or_focal_loss_that_does_not_fit(yml, make):
    from multiyolov5_b200.models.yolo import Model
    from multiyolov5_b200.train import Trainer
    from multiyolov5_b200.utils import loss as L
    with pytest.raises(ValueError):
        Trainer(Model(yml), {}, 4, seg_loss=make(L))


def test_trainer_rejects_unweighted_segmentation_losses_naming_the_default():
    from multiyolov5_b200.models.yolo import Model
    from multiyolov5_b200.train import Trainer
    from multiyolov5_b200.utils.loss import SegmentationLosses
    with pytest.raises(ValueError, match="seg_loss=None"):
        Trainer(Model("yolov5s_city_seg.yaml"), {}, 4, seg_loss=SegmentationLosses())


def test_trainer_takes_the_losses_that_fit_up_to_the_device_check():
    """the checks pass for these; the CPU model then stops at the Trainer's model.cuda() assertion"""
    from multiyolov5_b200.models.yolo import Model
    from multiyolov5_b200.train import Trainer
    from multiyolov5_b200.utils import loss as L
    for model, seg_loss in [(Model("yolov5s_city_seg.yaml"), L.SegmentationLosses(weight=torch.tensor(W19))),
                            (Model("yolov5s_city_seg_bise.yaml"), L.SegmentationLosses(aux=True, aux_num=2, weight=torch.tensor(W19))),
                            (Model("yolov5s_city_seg.yaml"), L.SegFocalLoss(gamma=2, alpha=W19, ignore_index=-1)),
                            (_two_class_model(), L.SegFocalLoss(gamma=2, ignore_index=-1))]:
        with pytest.raises(AssertionError, match="cuda"):
            Trainer(model, {}, 4, seg_loss=seg_loss)
