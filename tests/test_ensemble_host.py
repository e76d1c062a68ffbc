"""CPU: model ensembles' host side (models.experimental.Ensemble, attempt_load of several weights): what attempt_load returns and prints
for reference-written checkpoints, every refusal before any launch, and myolo_seg_ensemble without a device."""
import ctypes as C
import os

import pytest
import torch

from multiyolov5_b200 import _lib
from multiyolov5_b200.models.experimental import Ensemble, attempt_load
from multiyolov5_b200.models.yolo import Model
from oracle import synth

CKPTS = [os.path.join(synth.GOLDEN_DIR, f) for f in ("ref_ckpt_tiny.pt", "ref_ckpt_tiny_syncbn.pt")]


def test_attempt_load_one_checkpoint_is_the_model(capsys):
    for w in (CKPTS[0], [CKPTS[0]]):
        m = attempt_load(w, map_location="cpu")
        assert type(m) is Model and not m.training
    assert "Ensemble" not in capsys.readouterr().out


def test_attempt_load_several_checkpoints_is_an_ensemble(capsys):
    e = attempt_load(CKPTS, map_location="cpu")
    assert type(e) is Ensemble and len(e) == 2 and all(type(m) is Model and not m.training for m in e)
    assert capsys.readouterr().out == f"Ensemble created with {CKPTS}\n\n"        # reference models/experimental.py:129
    assert e.names is e[-1].names and e.stride is e[-1].stride                    # the last member's, as in the reference
    assert e.names == [f"cls{i}" for i in range(10)] and e.stride.tolist() == [8.0, 16.0, 32.0]


@pytest.fixture(scope="module")
def small():
    return Model("yolov5s_city_seg.yaml").eval()


def _ens(*models):
    e = Ensemble()
    for m in models:
        e.append(m)
    return e.eval()


def test_refuses_mismatched_members(small):
    cfg = synth.load_cfg("yolov5s_city_seg.yaml")
    with pytest.raises(ValueError, match=r"member 1 has Detect.no \(5 \+ nc\) 10, member 0 has 15"):
        _ens(small, Model(cfg, nc=5).eval()).check_members()
    cfg["n_segcls"] = 7
    with pytest.raises(ValueError, match="member 1 has seg classes 7, member 0 has 19"):
        _ens(small, Model(cfg).eval()).check_members()
    other = Model("yolov5s_city_seg.yaml").eval()
    other.model[-1].stride = torch.tensor([8.0, 16.0, 64.0])
    with pytest.raises(ValueError, match="member 1 has Detect.stride"):
        _ens(small, other).check_members()
    other = Model("yolov5s_city_seg_bise.yaml").eval().half()
    with pytest.raises(ValueError, match="member 1 has parameter dtype torch.float16, member 0 has torch.float32"):
        _ens(small, other).check_members()
    with pytest.raises(ValueError, match="9 members; the device path takes 1 to 8"):
        _ens(*[small] * 9).check_members()
    _ens(*[small] * 8).check_members()
    with pytest.raises(ValueError, match="member 0 is a Conv2d, not a Model"):
        _ens(torch.nn.Conv2d(3, 3, 1), small).check_members()


def test_attempt_load_checks_members(tmp_path):
    ck = torch.load(CKPTS[0], map_location="cpu", weights_only=False, pickle_module=__import__(
        "multiyolov5_b200.models.experimental", fromlist=["x"])._RefPickleModule)
    ck["model"].model[-1].stride = torch.tensor([8.0, 16.0, 64.0])
    bad = tmp_path / "bad.pt"
    torch.save(ck, bad)
    with pytest.raises(ValueError, match="member 1 has Detect.stride"):
        attempt_load([CKPTS[0], str(bad)], map_location="cpu")


def test_refuses_train_mode_and_profile(small):
    x = torch.zeros(1, 3, 64, 64)
    e = _ens(small, small)
    with pytest.raises(ValueError, match="profile=True"):
        e(x, profile=True)
    e.train()
    with pytest.raises(RuntimeError, match="eval mode"):
        e(x)
    e.eval()
    small.train()
    try:
        with pytest.raises(RuntimeError, match="eval mode"):
            e(x)
    finally:
        small.eval()


def test_test_refuses_compute_loss_with_an_ensemble(small):
    from multiyolov5_b200 import test as T
    with pytest.raises(ValueError, match="compute_loss"):
        T.test({"nc": 10}, model=_ens(small, small), dataloader=[], compute_loss=lambda *a: None)


@pytest.mark.skipif(torch.cuda.is_available(), reason="host buffers where the library expects device memory")
def test_entry_point_without_device():
    L = _lib.lib()
    buf = C.create_string_buffer(1 << 12)
    P = C.addressof(buf)
    plans = (C.c_void_p * 9)(*[P] * 9)
    assert L.myolo_nms(None, 1, 1, 6, 0.25, 0.45, None, 0, 0, 0, 1, 1, 0.0, None, None, None, 0, None) == -1
    other = L.myolo_last_error()
    assert L.myolo_seg_ensemble(plans, 2, P, _lib.F16, None, None) == -3                  # MYOLO_E_NODEVICE
    msg = L.myolo_last_error()
    assert msg and msg != other, msg
    assert L.myolo_seg_ensemble(plans, 2, None, _lib.F16, P, None) == -3
    assert L.myolo_seg_ensemble(plans, 9, P, _lib.F16, None, None) == -1                  # more than MYOLO_ENSEMBLE_MAX
    assert L.myolo_seg_ensemble(plans, 0, P, _lib.F16, None, None) == -1
    assert L.myolo_seg_ensemble(plans, 2, None, _lib.F16, None, None) == -1               # no output
    assert L.myolo_seg_ensemble(plans, 2, P, _lib.U8, None, None) == -1


# ---- the reference's ensemble (tests/golden/ensemble_cases.npz, oracle/make_golden_ensemble.py) ---------------------------------------
GOLD = os.path.join(synth.GOLDEN_DIR, "ensemble_cases.npz")


@pytest.mark.parametrize("k", [0, 1])
def test_restated_ensemble_matches_reference(k):
    import numpy as np
    from oracle import restate_ensemble
    g = np.load(GOLD)
    x = restate_ensemble.fixture_input(g, k)
    z, seg, ids = restate_ensemble.model_forward_ensemble(restate_ensemble.fixture_members(g), x)
    rows, idx = g[f"case{k}_rows"], g[f"case{k}_seg_idx"]
    per_member = z.shape[1] // 3
    assert z.shape[1] == 3 * per_member and rows[-1] < z.shape[1] <= rows[-1] + 13
    rel = lambda a, b: float(np.abs(a - b).max() / np.abs(b).max())       # noqa: E731
    assert rel(z.numpy()[:, rows], g[f"case{k}_z"]) < 2e-4            # the tolerance of test_oracle_golden.py for z (fp32 CPU both sides)
    assert rel(seg.numpy().reshape(-1)[idx], g[f"case{k}_seg"]) < 2e-4
    assert (ids.numpy() == g[f"case{k}_ids"]).mean() > 0.999
