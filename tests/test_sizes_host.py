"""Host: the l and x city-seg configs (yolov5{l,x}_city_seg{,_lab,_bise,_base}.yaml) build the reference's graph - state_dict keys, shapes
and parameter count equal the manifests the unmodified reference wrote (oracle/make_golden_sizes.py) - their fixtures are present, and the
fp32 restatement (oracle/restate.py), which the GPU tests use as the truth at tensor-core sizes, reproduces the reference's outputs."""
import os

import numpy as np
import pytest
import torch

from oracle import restate, synth

HEADS = {"psp": "", "lab": "_lab", "bise": "_bise", "base": "_base"}
SIZES = {"l": (1.0, 1.0), "x": (1.33, 1.25)}
CASES = [(f"{s}_{h}", f"yolov5{s}_city_seg{suffix}.yaml") for s in SIZES for h, suffix in HEADS.items()]
# millions of parameters, printed by the reference's own Model (oracle/make_golden_sizes.py)
PARAMS_M = {"l_psp": 49.36, "l_lab": 51.72, "l_bise": 49.51, "l_base": 50.29, "x_psp": 91.49, "x_lab": 100.84, "x_bise": 90.92,
            "x_base": 93.93}


@pytest.mark.parametrize("tag,yml", CASES)
def test_config_builds_the_reference_graph(tag, yml):
    from multiyolov5_b200.models.yolo import Model
    cfg = synth.load_cfg(yml)
    s16 = synth.load_cfg(yml.replace(f"yolov5{tag[0]}_", "yolov5s_"))
    assert (cfg["depth_multiple"], cfg["width_multiple"]) == SIZES[tag[0]]
    assert {k: v for k, v in cfg.items() if not k.endswith("_multiple")} == {k: v for k, v in s16.items() if not k.endswith("_multiple")}
    torch.manual_seed(0)
    model = Model(yml)
    sd = model.state_dict()
    manifest = synth.load_manifest(tag)
    assert [k for k, _, _ in manifest] == list(sd)
    for k, shape, dt in manifest:
        assert list(sd[k].shape) == shape and str(sd[k].dtype) == f"torch.{dt}", k
    n = sum(p.numel() for p in model.parameters())
    g = np.load(os.path.join(synth.GOLDEN_DIR, f"net_{tag}.npz"))
    assert n == int(g["n_params"]) and round(n / 1e6, 2) == PARAMS_M[tag], (n, int(g["n_params"]))
    model.load_state_dict(synth.synth_state_dict(manifest, cfg, seed=1))


def test_fixtures_cover_every_head_and_size():
    for tag, _ in CASES:
        path = os.path.join(synth.GOLDEN_DIR, f"net_{tag}.npz")
        g = np.load(path)
        B, H, W = (int(v) for v in g["shape"])
        assert (B, H, W) == (1, 64, 128), tag
        assert g["z"].shape == (1, 3 * (8 * 16 + 4 * 8 + 2 * 4), 15), tag
        assert g["seg_lowres"].shape[:2] == (1, 19) and g["seg_argmax"].shape == (1, H, W), tag
        assert {"raw0", "raw1", "raw2", "layer9", "layer23"} <= set(g.files), tag
        # the synthetic weights keep every activation of the fp32 reference (at 1 x 256 x 512) far inside fp16 range
        assert 1.0 < float(g["act_absmax"]) < 64.0, (tag, float(g["act_absmax"]))
        assert os.path.getsize(path) < 128e3, tag


@pytest.mark.parametrize("tag,yml", CASES)
def test_restatement_matches_reference(tag, yml):
    """fp32 CPU both sides: differences are only BN-fold order and kernel choice (raw and taps are stored as fp16)"""
    cfg = synth.load_cfg(yml)
    g = np.load(os.path.join(synth.GOLDEN_DIR, f"net_{tag}.npz"))
    B, H, W = (int(v) for v in g["shape"])
    out = restate.model_forward(cfg, synth.synth_state_dict(synth.load_manifest(tag), cfg, seed=1), synth.synth_image(B, H, W, seed=int(g["seed"])),
                                keep=(9, 23))
    rel = lambda a, b: float(np.abs(a - b).max() / np.abs(b).max())     # noqa: E731
    assert rel(out["z"].numpy(), g["z"]) < 2e-4
    assert rel(out["seg_lowres"].numpy(), g["seg_lowres"]) < 2e-4
    for i in range(3):
        assert rel(out["raw"][i].numpy(), g[f"raw{i}"].astype(np.float32)) < 2e-3
    for i in (9, 23):
        assert rel(out["layers"][i].numpy(), g[f"layer{i}"].astype(np.float32)) < 2e-3


def test_l_checkpoint_loads_by_attempt_load(tmp_path):
    """a checkpoint of an l model, saved as the reference's train.py saves it (the pickled Model in half precision), loads through
    attempt_load with the same weights"""
    from multiyolov5_b200.models.experimental import attempt_load
    from multiyolov5_b200.models.yolo import Model
    yml = "yolov5l_city_seg.yaml"
    model = Model(yml)
    model.load_state_dict(synth.synth_state_dict(synth.load_manifest("l_psp"), synth.load_cfg(yml), seed=1))
    model.names = [f"cls{i}" for i in range(10)]
    path = str(tmp_path / "l.pt")
    torch.save({"epoch": 0, "model": model.half(), "ema": None}, path)
    loaded = attempt_load(path, map_location="cpu")
    assert loaded.yaml["width_multiple"] == 1.0 and loaded.names == model.names
    w = dict(loaded.named_parameters())["model.9.cv3.conv.weight"]     # the last C3 of the backbone: 1024 outputs
    assert w.dtype == torch.float32 and w.shape[0] == 1024
