"""GPU: test-time augmentation, Model.forward(augment=True) (reference models/yolo.py:274-289 with forward_once(xi)[0][0]).

The device path (utils.torch_utils.scale_img in one launch, det-only plans for the scaled passes, de-scale and de-flip inside the Detect
decodes) against torch composing the reference's loop on CUDA over this library's plain forwards, bit for bit; and against the reference's
fp32 CPU fixture (tests/golden/tta_cases.npz) within the error caps of tests/test_gpu_parity.py and its torch-fp16 yardstick rule."""
import math
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from multiyolov5_b200 import _lib
from oracle import restate, restate_tta, synth

pytestmark = pytest.mark.gpu

YML = "yolov5s_city_seg.yaml"
GOLD = os.path.join(synth.GOLDEN_DIR, "tta_cases.npz")
# tests/test_gpu_parity.py CAPS: boxes (pixels for boxes up to 256 px, relative to the box size for all) and scores against the fp32 reference
CAPS = {"box_px_max_le256": 15.0, "box_rel_max": 0.11, "score_abs_max": 2.2e-2}


def build(anchors=None):
    from multiyolov5_b200.models.yolo import Model
    if anchors is not None:
        return Model(YML, anchors=anchors).cuda().eval()
    cfg = synth.load_cfg(YML)
    sd = synth.synth_state_dict(synth.load_manifest("s_psp"), cfg, seed=1)
    m = Model(YML)
    m.load_state_dict(sd)
    return m.cuda().eval()


@pytest.fixture(scope="module")
def model():
    return build()


def torch_tta(model, x):
    """the reference's loop composed in torch on CUDA (flip, interpolate, pad, de-scale, cat) over this library's plain forwards"""
    return restate_tta.tta(lambda xi: model(xi)[0][0], x, gs=32)


def box_score_errors(z, zr):
    z = z.float().cpu().numpy().astype(np.float64); zr = zr.astype(np.float64)
    d = np.abs(z[..., :4] - zr[..., :4]).max(-1)
    size = np.maximum(zr[..., 2], zr[..., 3])
    return {"box_px_max_le256": float(d[size <= 256.0].max()), "box_rel_max": float((d / np.maximum(size, 8.0)).max()),
            "score_abs_max": float(np.abs(z[..., 4:] - zr[..., 4:]).max())}


# ---- scale_img ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", [torch.float16, torch.float32])
@pytest.mark.parametrize("ratio,same_shape,flip", [(0.83, False, True), (0.83, False, False), (0.67, False, False), (0.67, False, True),
                                                   (0.83, True, False), (1.3, False, False), (1.3, True, True), (1.0, False, True)])
@pytest.mark.parametrize("shape", [(2, 3, 200, 330), (1, 3, 512, 1024)])
def test_scale_img_bit_exact_with_torch(dtype, ratio, same_shape, flip, shape):
    from multiyolov5_b200.utils.torch_utils import scale_img
    g = torch.Generator(device="cuda").manual_seed(1)
    x = torch.rand(shape, device="cuda", generator=g).to(dtype)
    ours = scale_img(x, ratio, same_shape=same_shape, gs=32, flip_lr=flip)
    xf = x.flip(3) if flip else x
    h, w = shape[2:]
    if ratio == 1.0:
        ref = xf
    else:
        s = (int(h * ratio), int(w * ratio))
        ho, wo = (h, w) if same_shape else [math.ceil(v * ratio / 32) * 32 for v in (h, w)]
        ref = F.pad(F.interpolate(xf, size=s, mode="bilinear", align_corners=False), [0, wo - s[1], 0, ho - s[0]], value=0.447)
    assert ours.dtype == dtype and ours.shape == ref.shape
    assert torch.equal(ours, ref)


def test_scale_img_ratio_one_returns_the_input(model):
    from multiyolov5_b200.utils.torch_utils import scale_img
    x = torch.rand((1, 3, 64, 64), device="cuda")
    assert scale_img(x, 1.0) is x


# ---- the augmented forward ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("B,H,W,dtype", [(2, 256, 512, torch.float32), (2, 256, 512, torch.float16), (1, 320, 416, torch.float32),
                                         (1, 320, 416, torch.float16), (16, 512, 1024, torch.float16), (1, 512, 1024, torch.float32)])
def test_tta_bit_exact_with_torch_composition(model, B, H, W, dtype):
    x = synth.synth_image(B, H, W, seed=7).cuda().to(dtype)
    out = model(x, augment=True)
    (z, none), seg = out
    assert none is None and z.dtype == torch.float32
    ref = torch_tta(model, x)
    assert z.shape == ref.shape
    assert torch.equal(z, ref)
    plain = model(x)
    assert torch.equal(seg, plain[1])                      # pass 0's seg, that of augment=False
    z2, seg2, amax = model(x, augment=True, seg_argmax=True)
    assert z2[1] is None and seg2 is None and torch.equal(z2[0], z)
    assert torch.equal(amax, model(x, seg_argmax=True)[2])


def test_tta_rows_at_baseline_shape(model):
    x = synth.synth_image(1, 512, 1024, seed=0).cuda().half()
    z = model(x, augment=True)[0][0]
    assert z.shape == (1, 71316, 15)


def test_tta_anchor_count_4():
    m = build(anchors=4)
    x = synth.synth_image(2, 256, 512, seed=3).cuda()
    z = m(x, augment=True)[0][0]
    assert z.shape[1] == sum(4 * (h // s) * (w // s) for (h, w) in ((256, 512), (224, 448), (192, 352)) for s in (8, 16, 32))
    assert torch.equal(z, torch_tta(m, x))


def test_det_only_plans_match_full_plans(model):
    """the scaled passes on plans without the seg head give the z of the full plans of the same shapes, bit for bit"""
    eng = model.engine()
    for dtype in (torch.float16, torch.float32):
        x = synth.synth_image(2, 320, 416, seed=5).cuda().to(dtype)
        a = eng.forward_augment(x)[0][0]
        b = eng.forward_augment(x, det_only_scaled=False)[0][0]
        assert torch.equal(a, b)
    full, det = eng.plans[(2, 224, 288)], eng.plans[("det", 2, 224, 288)]
    assert not any(o.kind == _lib.OP_SEG_UPSAMPLE for o in det.pb.ops)
    assert det.pb.det_rows == full.pb.det_rows and len(det.pb.ops) < len(full.pb.ops)


def test_alternating_plain_and_tta_calls(model):
    """plain and augmented calls on the same plans give unchanged outputs, build no plan and capture no graph again"""
    x = synth.synth_image(1, 256, 512, seed=11).cuda().half()
    (z0, _), s0 = model(x)
    zt0, st0 = model(x, augment=True)
    model(x); model(x, augment=True)                       # every plan warm and captured
    torch.cuda.synchronize()
    plans = dict(model.engine().plans)
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CPU, torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(3):
            (z1, _), s1 = model(x)
            zt1, st1 = model(x, augment=True)
            assert torch.equal(z1, z0) and torch.equal(s1, s0) and torch.equal(zt1[0], zt0[0]) and torch.equal(st1, st0)
        torch.cuda.synchronize()
    assert model.engine().plans == plans
    names = [e.name for e in prof.events()]
    if not any("GraphLaunch" in n for n in names):
        pytest.skip("the profiler does not see the library's CUDA runtime calls")
    assert not any("BeginCapture" in n or "GraphInstantiate" in n for n in names), sorted({n for n in names if "Graph" in n or "Capture" in n})


def test_detect_and_test_call_sites(model):
    """detect.py:144-149 and test.py:167 as written, with non_max_suppression on the 71 316-row z"""
    from multiyolov5_b200.utils.general import non_max_suppression
    img = synth.synth_image(2, 512, 1024, seed=2).cuda().half()
    with torch.no_grad():
        out = model(img, augment=True)
        pred = out[0][0]
        seg = out[1]
        pred = non_max_suppression(pred, 0.25, 0.45)
    assert out[0][0].shape == (2, 71316, 15) and seg.shape == (2, model.model[-2].c_out, 512, 1024)
    ref = restate.non_max_suppression(out[0][0].float().cpu().numpy(), 0.25, 0.45)
    assert len(pred) == 2 and all(np.array_equal(d.cpu().numpy(), r) for d, r in zip(pred, ref))
    out, train_out = model(img, augment=True)[0]
    assert train_out is None and out.shape == (2, 71316, 15)


def test_ema_model_tta(model):
    from multiyolov5_b200.utils.torch_utils import ModelEMA
    ema = ModelEMA(model)
    x = synth.synth_image(1, 320, 416, seed=9).cuda()
    assert torch.equal(ema.ema(x, augment=True)[0][0], model(x, augment=True)[0][0])


@pytest.mark.parametrize("k", [0, 1])
def test_tta_vs_reference_fixture(model, k):
    g = np.load(GOLD)
    B, H, W = (int(v) for v in g[f"case{k}_shape"])
    x = synth.synth_image(B, H, W, seed=int(g[f"case{k}_seed"]))
    assert x.double().sum().item() == pytest.approx(float(g[f"case{k}_x_sum"]), rel=1e-12)
    zr, rows = g[f"case{k}_z"], torch.from_numpy(g[f"case{k}_rows"])      # the fixture keeps a fixed sample of z's rows
    ours = box_score_errors(model(x.cuda(), augment=True)[0][0][:, rows.cuda()], zr)
    cfg = synth.load_cfg(YML)
    sd = synth.synth_state_dict(synth.load_manifest("s_psp"), cfg, seed=1)
    sdc = {key: v.cuda() for key, v in sd.items()}
    yard = box_score_errors(restate_tta.model_forward_tta(cfg, sdc, x.cuda(), half=True)[:, rows.cuda()], zr)
    print("ours", ours, "torch fp16", yard)
    for key, cap in CAPS.items():
        assert ours[key] <= cap, (key, ours[key])
        assert ours[key] <= 1.25 * yard[key] + 1e-3, (key, ours[key], yard[key])


def test_error_cases(model):
    x = synth.synth_image(1, 64, 64, seed=0).cuda()
    with pytest.raises(ValueError, match="profile"):
        model(x, augment=True, profile=True)
    with pytest.raises(TypeError, match="fp16 or fp32"):
        model((x * 255).to(torch.uint8), augment=True)
    with pytest.raises(_lib.MyoloError, match="CUDA"):
        model(x.cpu(), augment=True)
    model.train()
    try:
        with pytest.raises(RuntimeError, match="eval mode"):
            model(x, augment=True)
    finally:
        model.eval()
