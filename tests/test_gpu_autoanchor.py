"""H100: the reference's autoanchor on the device.  check_anchors / kmean_anchors on a DeviceImageCache against every case the reference
computed (tests/golden/autoanchor_cases.npz): printed lines, Detect buffers and the state of `random` / `numpy.random` afterwards, bit for
bit.  myolo_anchor_evolve against the numpy restatement (per-generation fitness bit for bit) at n = 1, n not a multiple of the block size
and ~300 k labels; run-to-run identity; the argument checks; and the two consumers of the Detect buffers: an inference plan built before
check_anchors decodes with the new anchors, and a Trainer built before it computes the det loss with them."""
import contextlib
import io
import os
import random

import numpy as np
import pytest
import torch

from oracle import restate_autoanchor as ra
from oracle import synth

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden")


class _Detect:
    """the Detect buffers check_anchors reads and writes, on the GPU"""

    def __init__(self, anchor_grid, stride):
        self.stride = torch.tensor(stride, dtype=torch.float32)
        self.anchor_grid = torch.from_numpy(anchor_grid.copy()).cuda()
        self.anchors = (self.anchor_grid.view(len(stride), -1, 2) / self.stride.cuda().view(-1, 1, 1)).contiguous()


class _Model:
    def __init__(self, det):
        self.model = [det]


def _cache(shapes0, labels):
    from multiyolov5_b200.utils.datasets import DeviceImageCache
    imgs = [np.zeros((h0, w0, 3), np.uint8) for h0, w0 in shapes0]
    return DeviceImageCache(imgs, 64, labels=labels)


def _run(c, det=None):
    from multiyolov5_b200.utils import autoanchor as aa
    shapes0, labels = ra.case_dataset(c)
    cache = _cache(shapes0, labels)
    random.seed(c["seed"]); np.random.seed(c["seed"]); torch.manual_seed(c["seed"])
    buf = io.StringIO()
    with contextlib.redirect_stdout(buf):
        if c["call"] == "check":
            aa.check_anchors(cache, _Model(det), thr=c["thr"], imgsz=c["imgsz"])
            ret = None
        else:
            ret = aa.kmean_anchors(cache, n=c["n"], img_size=c["imgsz"], thr=c["thr"], gen=c["gen"], verbose=c["verbose"])
    return buf.getvalue(), ret


@pytest.mark.parametrize("name", ["fit", "replace", "flip", "tiny", "thr291", "large", "kmean_verbose"])
def test_matches_the_reference_case(name):
    cases = {c["name"]: c for c in ra.load_cases(os.path.join(GOLD, "autoanchor_cases.npz"))}
    if name not in cases:
        pytest.skip(f"the fixture has no {name} case (no seed produced it)")
    c = cases[name]
    det = _Detect(c["anchor_grid0"], c["stride"]) if c["call"] == "check" else None
    out, ret = _run(c, det)
    assert out == c["stdout"]
    if det is not None:
        assert np.array_equal(det.anchor_grid.cpu().numpy(), c["anchor_grid1"])
        assert np.array_equal(det.anchors.cpu().numpy(), c["anchors1"])
    else:
        assert np.array_equal(ret, c["returned"])
    assert np.array_equal(np.array([random.random(), random.random()]), c["next_py"])
    assert np.array_equal(np.random.random(4), c["next_np"])


def _labels(n, seed):
    rng = np.random.default_rng(seed)
    c = np.array([[12, 30], [25, 60], [40, 25], [90, 55], [200, 120], [8, 8]], np.float64)
    wh = c[rng.integers(0, len(c), n)] * np.exp(rng.normal(0, 0.4, (n, 2)))
    wh[rng.random(n) < 0.02] = 0.0                                  # zero-size sides: r = 0, 1 / r = inf
    return np.maximum(wh, 0).astype(np.float32)


K0 = np.array([[9, 9], [13, 29], [26, 58], [39, 26], [60, 40], [88, 56], [120, 90], [198, 121], [300, 250]], np.float64)


@pytest.mark.parametrize("n,gen,thr", [(1, 50, 4.0), (1000, 300, 4.0), (257, 200, 2.91), (300_000, 200, 4.0)])
def test_evolve_matches_the_restatement(n, gen, thr):
    from multiyolov5_b200.utils import autoanchor as aa
    wh = _labels(n, n)
    np.random.seed(n)
    V = ra.draw_mutations(gen, K0.shape)
    k, f0, f, fg, acc = aa.evolve(torch.from_numpy(wh).cuda(), K0, V, 1.0 / thr)
    k_r, f_r, fg_r, acc_r = ra.evolve(wh, K0, V, 1.0 / thr)
    assert f0 == ra.fitness(wh, K0, 1.0 / thr)
    assert np.array_equal(fg, fg_r) and np.array_equal(k, k_r) and f == f_r and acc == acc_r
    if n > 1:
        assert acc > 0


def test_metric_matches_the_restatement_in_both_dtypes():
    from multiyolov5_b200.utils import autoanchor as aa
    wh = _labels(100_000, 7)
    t = 1.0 / 2.91
    for k in (K0, K0.astype(np.float32)):
        got = aa.anchor_metric(torch.from_numpy(wh).cuda(), k if k.dtype == np.float64 else torch.from_numpy(k).cuda(), t)
        exp = ra.metric_stats(wh, k, t)
        assert got["n_best"] == exp["n_best"] and got["n_x"] == exp["n_x"], (got, exp)
        for key in ("sum_x", "sum_best", "sum_x_above"):
            assert abs(got[key] - exp[key]) <= 1e-12 * exp[key]


def test_two_runs_are_identical():
    from multiyolov5_b200.utils import autoanchor as aa
    wh = torch.from_numpy(_labels(300_000, 3)).cuda()
    np.random.seed(1)
    V = ra.draw_mutations(100, K0.shape)
    a, b = aa.evolve(wh, K0, V, 0.25), aa.evolve(wh, K0, V, 0.25)
    assert np.array_equal(a[0], b[0]) and np.array_equal(a[3], b[3]) and a[1:3] == b[1:3] and a[4] == b[4]
    assert aa.anchor_metric(wh, K0, 0.25) == aa.anchor_metric(wh, K0, 0.25)


def test_evolve_refuses_what_the_exact_sum_does_not_cover():
    from multiyolov5_b200 import _lib
    from multiyolov5_b200.utils import autoanchor as aa
    wh = torch.from_numpy(_labels(100, 1)).cuda()
    V = np.ones((1, 9, 2))
    with pytest.raises(_lib.MyoloError, match="anchor_t <= 16"):
        aa.evolve(wh, K0, V, 1.0 / 17.0)
    with pytest.raises(_lib.MyoloError):
        aa.evolve(wh, np.ones((33, 2)), np.ones((1, 33, 2)), 0.25)


def _model():
    from multiyolov5_b200.models.yolo import Model
    yml = "yolov5s_city_seg.yaml"
    cfg = synth.load_cfg(yml)
    sd = synth.synth_state_dict(synth.load_manifest("s_psp"), cfg, seed=1)
    model = Model(yml)
    model.load_state_dict(sd)
    return model.cuda(), cfg


def _small_object_cache():
    """labels far smaller than the yaml's anchors: BPR < 0.98, new anchors replace them"""
    shapes0, labels = ra.synth_dataset(5, 40, 40, [(3, 9), (5, 4), (6, 14), (10, 8)], spread=0.3)
    return _cache(shapes0, labels)


def _check(model, cache):
    from multiyolov5_b200.utils import autoanchor as aa
    np.random.seed(0)
    with contextlib.redirect_stdout(io.StringIO()) as buf:
        aa.check_anchors(cache, model, thr=4.0, imgsz=640)
    assert "New anchors saved" in buf.getvalue()


def test_inference_plan_built_before_check_anchors_decodes_with_the_new_anchors():
    from multiyolov5_b200.models.yolo import Model
    model, _ = _model()
    model.eval()
    x = synth.synth_image(1, 128, 256, seed=0).cuda()
    (z0, _), _ = model(x)                                   # the plan exists and holds the yaml's anchors
    old = model.model[-1].anchor_grid.clone()
    _check(model, _small_object_cache())
    assert not torch.equal(model.model[-1].anchor_grid, old)
    (z1, _), _ = model(x)
    fresh = Model("yolov5s_city_seg.yaml")
    fresh.load_state_dict(model.state_dict())               # anchors and anchor_grid are buffers: the new ones
    fresh.cuda().eval()
    (z2, _), _ = fresh(x)
    torch.cuda.synchronize()
    assert torch.equal(z1, z2)
    assert not torch.equal(z0, z1)


def test_trainer_built_before_check_anchors_uses_the_new_anchors():
    from multiyolov5_b200.train import Trainer, scale_hyp
    hyp = dict(lr0=0.01, momentum=0.937, weight_decay=5e-4, box=0.05, cls=0.5, cls_pw=1.0, obj=1.0, obj_pw=1.0, anchor_t=4.0, fl_gamma=0.0)
    B, H, W = 2, 128, 256
    rs = np.random.RandomState(0)
    t = np.zeros((4 * B, 6), np.float32)
    t[:, 0] = np.repeat(np.arange(B), 4); t[:, 1] = rs.randint(0, 10, 4 * B)
    t[:, 2:4] = rs.uniform(0.2, 0.8, (4 * B, 2)); t[:, 4:6] = rs.uniform(0.01, 0.05, (4 * B, 2))
    imgs, targets = synth.synth_image(B, H, W, seed=1).cuda(), torch.from_numpy(t).cuda()
    cache = _small_object_cache()

    def trainer(model, cfg):
        return Trainer(model, scale_hyp(hyp, nl=3, nc=cfg["nc"], imgsz=256, total_batch_size=B), batch_size=B, accumulate=1000,
                       init_scale=2.0 ** 10)

    m1, cfg = _model()
    tr1 = trainer(m1, cfg)
    before = tr1.backward_det(imgs, targets).clone()        # the fused loss has read the yaml's anchors
    _check(m1, cache)
    after = [tr1.backward_det(imgs, targets).clone() for _ in range(2)]
    m2, _ = _model()
    _check(m2, cache)
    assert torch.equal(m1.model[-1].anchors, m2.model[-1].anchors)
    tr2 = trainer(m2, cfg)
    fresh = [tr2.backward_det(imgs, targets).clone() for _ in range(2)]
    torch.cuda.synchronize()
    # the yardstick is the run-to-run spread of the train forward (fp32 atomics in its BatchNorm statistics), floored at 1e-3 relative
    spread = torch.maximum((after[0] - after[1]).abs(), (fresh[0] - fresh[1]).abs())
    tol = torch.maximum(3 * spread, 1e-3 * fresh[0].abs())
    assert bool(((after[0] - fresh[0]).abs() <= tol).all()), (after, fresh)
    assert float(((before - fresh[0]).abs() / tol).max()) > 10, (before, fresh)     # the anchors did change the loss
