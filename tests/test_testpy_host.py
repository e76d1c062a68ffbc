"""Host checks of the --save-hybrid NMS and the confusion matrix: the restatements in oracle/restate_confusion.py against the reference
fixture tests/golden/testpy_cases.npz (oracle/make_golden_testpy.py), the label packing, and test()'s argument checks."""
import os

import numpy as np
import pytest
import torch

from oracle import restate, restate_confusion as RC
from oracle.make_golden_testpy import make_z

GOLD = np.load(os.path.join(os.path.dirname(__file__), "golden", "testpy_cases.npz"))


def nms_case(name):
    s, B, A, nc, distinct, empty1 = (int(v) for v in GOLD[f"nms_{name}_z"])
    z = make_z(s, B, A, nc, bool(distinct))
    if empty1:
        z[1, :, 4] = 0.0
    ct, it, ml = GOLD[f"nms_{name}_kw"]
    cls = GOLD[f"nms_{name}_classes"]
    kw = dict(conf_thres=float(ct), iou_thres=float(it), multi_label=bool(ml), classes=[int(c) for c in cls] if len(cls) else None)
    labels = [GOLD[f"nms_{name}_labels{b}"] for b in range(B)]
    outs = [GOLD[f"nms_{name}_out{b}"] for b in range(B)]
    return z, nc, kw, labels, outs


@pytest.mark.parametrize("name", [str(n) for n in GOLD["nms_names"]])
def test_label_rows_are_appended_candidates(name):
    """below conf 1 the reference's autolabelling NMS equals the plain NMS over z with the labels appended as rows"""
    z, nc, kw, labels, outs = nms_case(name)
    if kw["conf_thres"] >= 1:
        assert all(len(o) == 0 for o in outs)
        return
    for b in range(len(labels)):
        zz = np.concatenate([z[b], RC.label_rows(labels[b], nc)])[None]
        assert np.array_equal(restate.non_max_suppression(zz, **kw)[0], outs[b])


@pytest.mark.parametrize("name", [str(n) for n in GOLD["cm_names"]])
def test_confusion_restatement(name):
    n, nc = (int(v) for v in GOLD[f"cm_{name}_n"])
    m = np.zeros((nc + 1, nc + 1))
    for k in range(n):
        RC.process_batch(m, GOLD[f"cm_{name}_det{k}"], GOLD[f"cm_{name}_lab{k}"], nc)
        assert np.array_equal(m, GOLD[f"cm_{name}_matrix{k}"]), k


def test_confusion_edges_in_fixture():
    """the edge sequence really sits on the thresholds: 0.45 - ulp and 0.45 do not match, 0.45 + ulp does; conf likewise"""
    m = [GOLD[f"cm_edges_matrix{k}"] for k in range(6)]
    assert m[0][3, 1] == 1 and m[1][3, 1] == 2 and m[2][1, 1] == 1
    assert m[3][2, 2] == 0 and m[4][2, 2] == 0 and m[5][2, 2] == 1


def test_pack_labels_from_targets():
    from multiyolov5_b200.utils.general import NmsLabels
    t = torch.tensor([[1, 2, .5, .5, .1, .2], [0, 1, .25, .5, .5, .5], [1, 0, .75, .25, .2, .2], [3, 1, .1, .1, .1, .1]])
    lab = NmsLabels.from_targets(t, 4, (64, 128))
    assert lab.offsets.tolist() == [0, 1, 3, 3, 4]
    assert lab.max_labels == 4
    want = torch.cat([t[[1, 0, 2, 3], 1:2], t[[1, 0, 2, 3], 2:] * torch.tensor([128., 64., 128., 64.])], 1)
    assert torch.equal(lab.rows, want)


def test_pack_labels_from_list_checks_classes():
    from multiyolov5_b200.utils.general import NmsLabels
    lab = NmsLabels.from_list([np.float32([[1, 5, 5, 2, 2]]), np.zeros((0, 5), np.float32), np.float32([[0, 1, 1, 1, 1], [2, 3, 3, 1, 1]])],
                              3, "cpu")
    assert lab.offsets.tolist() == [0, 1, 1, 3] and lab.max_labels == 2
    with pytest.raises(ValueError):
        NmsLabels.from_list([np.float32([[3, 5, 5, 2, 2]])], 3, "cpu")
    with pytest.raises(ValueError):
        NmsLabels.from_list([np.float32([[-1, 5, 5, 2, 2]])], 3, "cpu")


def test_test_refuses_before_anything_else():
    from multiyolov5_b200.test import test
    m = torch.nn.Linear(1, 1)
    with pytest.raises(NotImplementedError, match="weights"):
        test({"nc": 1}, model=None, dataloader=[])
    for kw in (dict(save_json=True), dict(save_hybrid=True), dict(augment=True), dict(plots=True)):
        with pytest.raises(NotImplementedError, match="CPU"):
            test({"nc": 1}, model=m, dataloader=[], **kw)
    with pytest.raises(NotImplementedError, match="W&B"):
        test({"nc": 1}, model=m, dataloader=[], wandb_logger=object())
