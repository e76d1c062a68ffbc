"""CPU: test-time augmentation's host side against tests/golden/tta_cases.npz (the reference's own scale_img and forward_once,
oracle/make_golden_tta.py): the pass geometry of the product, the restated scale_img and the restated augmented forward."""
import os

import numpy as np
import pytest
import torch

from multiyolov5_b200.utils.torch_utils import scale_img_shapes, tta_passes
from oracle import restate_tta, synth

GOLD = os.path.join(synth.GOLDEN_DIR, "tta_cases.npz")


@pytest.fixture(scope="module")
def g():
    return np.load(GOLD)


def relmax(a, b):
    a = np.asarray(a, np.float64); b = np.asarray(b, np.float64)
    return float(np.abs(a - b).max() / (np.abs(b).max() + 1e-30))


def test_pass_geometry_matches_reference_scale_img_shapes(g):
    for (h, w, r, same), shape in zip(g["sweep_args"], g["sweep_shape"]):
        _, out = scale_img_shapes(int(h), int(w), float(r), bool(same), 32)
        assert list(out) == list(shape), (h, w, r, same)
    for h, w in {(int(a[0]), int(a[1])) for a in g["sweep_args"]}:
        for si, flip, resized, padded in tta_passes(h, w, 32):
            assert scale_img_shapes(h, w, si, False, 32) == (resized, padded) and flip == (si == 0.83)


def test_pass_geometry_at_baseline_shape():
    """16 x 3 x 512 x 1024: pass 1 resizes to 424 x 849 and pads to 448 x 864, pass 2 resizes to 343 x 686 and pads to 352 x 704; with
    three anchors per cell that is 32 256 + 23 814 + 15 246 = 71 316 rows per image"""
    p = tta_passes(512, 1024, 32)
    assert [q[2:] for q in p] == [((512, 1024), (512, 1024)), ((424, 849), (448, 864)), ((343, 686), (352, 704))]
    rows = [3 * sum((h // s) * (w // s) for s in (8, 16, 32)) for _, _, _, (h, w) in p]
    assert rows == [32256, 23814, 15246] and sum(rows) == 71316


def test_restated_scale_img_bit_exact(g):
    x = torch.from_numpy(g["si_x"])
    for j in range(int(g["n_si"])):
        r, same, flip = g[f"si{j}_args"]
        y = restate_tta.scale_img(x.flip(3) if flip else x, float(r), same_shape=bool(same), gs=32)
        assert np.array_equal(y.numpy(), g[f"si{j}_out"]), (r, same, flip)


@pytest.mark.parametrize("k", [0, 1])
def test_restated_tta_matches_reference(g, k):
    B, H, W = (int(v) for v in g[f"case{k}_shape"])
    x = synth.synth_image(B, H, W, seed=int(g[f"case{k}_seed"]))
    assert x.double().sum().item() == pytest.approx(float(g[f"case{k}_x_sum"]), rel=1e-12)
    cfg = synth.load_cfg("yolov5s_city_seg.yaml")
    sd = synth.synth_state_dict(synth.load_manifest("s_psp"), cfg, seed=1)
    z = restate_tta.model_forward_tta(cfg, sd, x)
    rows = g[f"case{k}_rows"]                                # the fixture keeps a fixed sample of z's rows
    assert z.shape[:2] == (B, 18396) and rows[-1] < z.shape[1] <= rows[-1] + 13
    zs = z.numpy()[:, rows]
    assert zs.shape == g[f"case{k}_z"].shape
    assert relmax(zs, g[f"case{k}_z"]) < 2e-4                # the tolerance of test_oracle_golden.py for z (fp32 CPU both sides)
