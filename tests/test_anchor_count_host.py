"""Models built with an anchor count, on the host: `Model(cfg, anchors=n)` and a yaml with `anchors: n` against the unmodified reference's
Model (tests/golden/anchor_count_cases.npz, oracle/make_golden_anchor_counts.py) - state-dict keys and shapes, the anchors buffers, the
Detect biases and yaml['anchors'] - and the torch ComputeLoss at na = 4 and 10 against the reference's."""
import json
import os

import numpy as np
import pytest
import torch

from oracle import restate_evolve as rev
from oracle import synth

GOLD = os.path.join(os.path.dirname(__file__), "golden")
CFG = "yolov5s_city_seg.yaml"


def _fixture():
    return np.load(os.path.join(GOLD, "anchor_count_cases.npz"))


def _model_recording_biases(monkeypatch, **kw):
    """Model(CFG, **kw) and the Detect biases _initialize_biases started from"""
    from multiyolov5_b200.models.yolo import Model
    pre = {}
    real = Model._initialize_biases

    def observed(self, cf=None):
        pre["b"] = [mi.bias.detach().clone() for mi in self.model[-1].m]
        return real(self, cf)
    monkeypatch.setattr(Model, "_initialize_biases", observed)
    torch.manual_seed(0)
    m = Model(**kw)
    return m, pre["b"]


@pytest.mark.parametrize("n", [2, 2.5, 3.5, 4, 10])
@pytest.mark.parametrize("via", ["argument", "yaml"])
def test_model_with_an_anchor_count_matches_the_reference(n, via, monkeypatch):
    g = _fixture()
    tag = f"model_{n}".replace(".", "p")
    if via == "argument":
        m, b0 = _model_recording_biases(monkeypatch, cfg=CFG, anchors=n)
    else:
        m, b0 = _model_recording_biases(monkeypatch, cfg=dict(synth.load_cfg(CFG), anchors=round(n)))
    det = m.model[-1]
    keys = json.loads(bytes(g[f"{tag}_keys_json"]).decode())
    assert [[k, list(v.shape)] for k, v in m.state_dict().items()] == keys
    assert det.na == round(n) and m.yaml["anchors"] == int(g[f"{tag}_yaml_anchors"]) and isinstance(m.yaml["anchors"], int)
    assert np.array_equal(det.stride.numpy(), g[f"{tag}_stride"])
    assert np.array_equal(det.anchors.numpy(), g[f"{tag}_anchors"])
    assert np.array_equal(det.anchor_grid.numpy(), g[f"{tag}_anchor_grid"])
    for i, mi in enumerate(det.m):
        # the conv initialisation draws differ from the reference's module order; what _initialize_biases adds must not
        got = mi.bias.detach().numpy() - b0[i].numpy()
        exp = g[f"{tag}_bias{i}"] - g[f"{tag}_bias_init{i}"]
        assert np.allclose(got, exp, rtol=0, atol=1e-6), i


def test_an_anchor_count_survives_a_checkpoint_round_trip(tmp_path):
    """yaml['anchors'] stays the int in a saved model, and the loaded model has the count's buffers"""
    from multiyolov5_b200.models.experimental import attempt_load
    from multiyolov5_b200.models.yolo import Model
    m = Model(CFG, anchors=4)
    m.model[-1].anchor_grid.mul_(1.5)
    path = str(tmp_path / "w.pt")
    torch.save({"model": m.half(), "epoch": -1}, path)
    back = attempt_load(path, map_location="cpu")
    assert back.yaml["anchors"] == 4 and back.model[-1].na == 4
    assert torch.equal(back.model[-1].anchor_grid.float(), m.model[-1].anchor_grid.float())


@pytest.mark.parametrize("na", [4, 10])
def test_det_loss_at_more_anchors_matches_the_reference(na):
    """the torch ComputeLoss (the yardstick of the fused loss) at na = 4 and 10: loss, items and gradients (fp32 tolerance 1e-5)"""
    from multiyolov5_b200.models.yolo import Model
    from multiyolov5_b200.utils.loss import ComputeLoss
    g = _fixture()
    tag = f"loss{na}"
    model = Model(CFG, anchors=na)
    model.hyp, model.gr = json.loads(bytes(g["loss_hyp_json"]).decode()), 1.0
    model.model[-1].anchors[:] = torch.from_numpy(g[f"{tag}_anchors"])
    crit = ComputeLoss(model)
    p = [torch.from_numpy(q).requires_grad_(True) for q in rev.loss_predictions(na)[0]]
    loss, items = crit(p, torch.from_numpy(g[f"{tag}_targets"]))
    loss.backward()
    ref = float(g[f"{tag}_loss"][0])
    assert abs(float(loss.detach()) - ref) <= 1e-5 * abs(ref)
    assert np.allclose(items.numpy(), g[f"{tag}_items"], rtol=1e-5, atol=1e-6)
    for i in range(3):
        r = g[f"{tag}_g{i}"]
        assert np.abs(p[i].grad.numpy() - r).max() <= 1e-5 * np.abs(r).max()
