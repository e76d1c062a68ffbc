"""GPU: the l and x city-seg models (yolov5{l,x}_city_seg{,_lab,_bise,_base}.yaml) on the device.
  - inference against the unmodified reference's fp32 fixtures (oracle/make_golden_sizes.py) at 1 x 64 x 128, and against the fp32
    restatement at 1 x 256 x 512, where every backbone / neck / head conv runs on the wgmma kernel: no further away than torch's fp16 +
    cuDNN run of the same graph (the rule of test_gpu_parity.py), detections after NMS and the seg class ids included;
  - a route census of every l / x plan: each forward conv on the wgmma kernel unless its s sibling leaves the same op elsewhere, and the
    backward routes, with SPP.cv2's data gradient (4 c_ = 2048 / 2560 output channels) on the wgmma kernel;
  - that data gradient on its own against fp64;
  - training: forward and backward against the fp32 autograd oracle, no further away than torch autocast (the rule of
    test_gpu_train.py), and Trainer.step on l / PSP and on x / BiSe (the three-output aux path)."""
import ctypes as C
import os
from collections import defaultdict

import numpy as np
import pytest
import torch

from oracle import restate, synth
from tests.test_gpu_conv_backward import DGRAD, LIMIT_DGRAD, WGRAD, census_ops, check, describe, print_worst, run
from tests.test_gpu_parity import build, errors_vs_fixture, rel
from tests.test_gpu_train import amp_yardstick, dropout_mask_of, oracle_train, rel_f, setup

pytestmark = pytest.mark.gpu

HEADS = {"psp": "", "lab": "_lab", "bise": "_bise", "base": "_base"}
CONFIGS = {f"{s}_{h}": f"yolov5{s}_city_seg{suffix}.yaml" for s in ("l", "x") for h, suffix in HEADS.items()}


# ---- inference parity ------------------------------------------------------------------------------------------------------------
def nms_recall(d_ref, d):
    """share of the rows of d_ref (x1,y1,x2,y2,conf,cls) that d holds with the same class and a box within max(2 px, 3 % of its size)"""
    if len(d_ref) == 0:
        return 1.0
    used = np.zeros(len(d), bool)
    hit = 0
    for r in d_ref:
        cand = np.where((d[:, 5] == r[5]) & ~used)[0]
        if not len(cand):
            continue
        j = cand[np.abs(d[cand, :4] - r[None, :4]).max(1).argmin()]
        if np.abs(d[j, :4] - r[:4]).max() <= max(2.0, 0.03 * float(max(r[2] - r[0], r[3] - r[1]))):
            used[j] = True
            hit += 1
    return hit / len(d_ref)


def check_forward(tag, x, g):
    """our forward of x against the truth g (z, raw0..2, seg_lowres, seg_argmax, layer9, layer23): no further away than torch's fp16 run
    of the same graph x 1.25 (test_gpu_parity.py's rule), the detections after NMS and the seg class ids included"""
    yml = CONFIGS[tag]
    model, cfg, sd = build(tag, yml)
    (z, raws), seg = model(x.cuda())
    torch.cuda.synchronize()
    ours = errors_vs_fixture(z, raws, seg, g)
    y = restate.model_forward(cfg, {k: v.cuda() for k, v in sd.items()}, x.cuda(), half=True)
    torch.cuda.synchronize()
    yard = errors_vs_fixture(y["z"], y["raw"], y["seg"], g)
    d_ref = restate.non_max_suppression(g["z"], 0.25, 0.45)[0]
    ours["nms_recall"] = nms_recall(d_ref, restate.non_max_suppression(z.float().cpu().numpy(), 0.25, 0.45)[0])
    yard["nms_recall"] = nms_recall(d_ref, restate.non_max_suppression(y["z"].float().cpu().numpy(), 0.25, 0.45)[0])
    print(f"\n[{tag} {tuple(x.shape)}] {len(d_ref)} reference detections\n  ours  vs fp32: {ours}\n  torch fp16 vs fp32: {yard}")
    for k in ("raw0", "raw1", "raw2", "seg"):
        assert ours[k] <= 1.25 * yard[k] + 2e-4, (k, ours[k], yard[k])
    for k in ("box_px_max_le256", "box_rel_max", "score_abs_max"):
        assert ours[k] <= 1.25 * yard[k] + 1e-3, (k, ours[k], yard[k])
    assert ours["cls_agree"] >= yard["cls_agree"] - 4e-3, (ours["cls_agree"], yard["cls_agree"])
    assert len(d_ref) > 0 and ours["nms_recall"] >= yard["nms_recall"] - 0.02, (ours["nms_recall"], yard["nms_recall"])
    # taps: P5 features of the backbone and the neck
    m2, _, _ = build(tag, yml, sd)
    m2.engine().noalias = True
    m2(x.cuda())
    for i in (9, 23):
        got = m2.engine().read_view(m2.engine().last_plan.pb.layer_views[i]).cpu().numpy()
        e = rel(got, np.asarray(g[f"layer{i}"], np.float32))
        print(f"  layer {i} tap: {e:.2e}")
        assert e <= 2e-2, (i, e)


@pytest.mark.parametrize("tag", list(CONFIGS))
def test_forward_vs_reference_fixture(tag):
    """at the fixture's 1 x 64 x 128 (maps below P3 on the CUDA-core kernel) against the unmodified reference"""
    g = np.load(os.path.join(synth.GOLDEN_DIR, f"net_{tag}.npz"))
    B, H, W = (int(v) for v in g["shape"])
    x = synth.synth_image(B, H, W, seed=int(g["seed"]))
    assert abs(float(x.double().sum()) - float(g["x_sum"])) < 1e-6 * float(g["x_sum"])
    check_forward(tag, x, g)


@pytest.mark.parametrize("tag", list(CONFIGS))
def test_forward_at_tensor_core_sizes(tag):
    """at 1 x 256 x 512, where every backbone / neck / head conv runs on the wgmma kernel, against the fp32 restatement on this GPU
    (TF32 off), which tests/test_sizes_host.py pins to the reference's fixtures"""
    cfg = synth.load_cfg(CONFIGS[tag])
    sd = synth.synth_state_dict(synth.load_manifest(tag), cfg, seed=1)
    x = synth.synth_image(1, 256, 512, seed=3)
    flags = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    try:
        with torch.no_grad():
            t = restate.model_forward(cfg, {k: v.cuda() for k, v in sd.items()}, x.cuda(), keep=(9, 23))
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = flags
    g = {"z": t["z"].cpu().numpy(), "seg_lowres": t["seg_lowres"].cpu().numpy(),
         "seg_argmax": t["seg"].argmax(1).cpu().numpy().astype(np.uint8)}
    for i in range(3):
        g[f"raw{i}"] = t["raw"][i].cpu().numpy()
    for i in (9, 23):
        g[f"layer{i}"] = t["layers"][i].cpu().numpy()
    check_forward(tag, x, g)


# ---- route census ----------------------------------------------------------------------------------------------------------------
def forward_routes(yml, B, H, W, train):
    """{op key: wgmma?} for every conv op of the plan; the key (layer tag, kernel, stride, output map) names the same op in the s, l and x
    plans of one head"""
    from multiyolov5_b200 import _lib as L
    from multiyolov5_b200.engine import CompiledPlan
    from multiyolov5_b200.models.yolo import Model
    torch.manual_seed(0)
    model = Model(yml).cuda()
    model.train(train)
    plan = CompiledPlan(model, B, H, W, train=train)
    plan.upload_weights()
    routes, kinds = {}, defaultdict(int)
    info = (C.c_int32 * 12)()
    for i, o in enumerate(plan.pb.ops):
        if o.kind != L.OP_CONV:
            continue
        L.check(L.lib().myolo_plan_conv_info(plan.handle, i, info))
        key = (o.tag, o.k, o.stride, o.out.h, o.out.w)
        routes[key] = routes.get(key, True) and bool(info[0])
        kinds["wgmma" if info[0] else "simt"] += 1
        if info[0]:
            kinds[f"wgmma BN={info[3]} kc={info[10]}{' resident' if info[6] else ''}{' strip' if info[5] else ''} {info[11]} cta/SM"] += 1
    del plan, model
    torch.cuda.empty_cache()
    return routes, kinds


CENSUS = [(16, 512, 1024, False), (4, 512, 1024, True)]     # the bench's inference batch and the Trainer's per-GPU slice


@pytest.mark.parametrize("tag", list(CONFIGS))
def test_forward_route_census(tag):
    yml = CONFIGS[tag]
    for B, H, W, train in CENSUS:
        routes, kinds = forward_routes(yml, B, H, W, train)
        s_routes, _ = forward_routes(yml.replace(f"yolov5{tag[0]}_", "yolov5s_"), B, H, W, train)
        print(f"\n[{tag} {'train' if train else 'infer'} {B}x{H}x{W}] " + ", ".join(f"{k}: {v}" for k, v in sorted(kinds.items())))
        off = sorted(k for k, tc in routes.items() if not tc)
        print(f"  off the wgmma kernel: {off}")
        assert all(not s_routes.get(k, True) for k in off), [k for k in off if s_routes.get(k, True)]


@pytest.mark.parametrize("tag", ["l_psp", "x_bise"])
def test_backward_route_census(tag):
    """every conv op of the train plan at the Trainer's 4 x 512 x 1024 slice: the train plan's backward entry at the op's geometry and
    slice layout against fp64, the routes printed, and SPP.cv2's data gradient on the wgmma kernel"""
    B, H, W = 4, 512, 1024
    fails, count, spp = [], defaultdict(int), []
    for i, wo, a in census_ops(CONFIGS[tag], B, H, W):
        info, err, ok = run(**a)
        fails += check(f"{tag} op {i}", info, err, ok)
        count[f"dgrad {DGRAD[info[0]]}"] += 1
        count[f"wgrad {WGRAD[info[1]]}"] += 1
        if info[1] == 2:
            count[f"wgrad mma.sync ci={a['ci']} co={a['co']}"] += 1
        if a["ci"] in (2048, 2560) and a["k"] == 1:
            spp.append((i, info))
        torch.cuda.empty_cache()
    print(f"\n[{tag} train {B}x{H}x{W}] " + ", ".join(f"{k}: {v}" for k, v in sorted(count.items())))
    for i, info in spp:
        print(f"  SPP.cv2 (op {i}): {describe(info)}")
    print_worst()
    assert not fails, "\n".join(fails[:30])
    assert len(spp) == 1 and spp[0][1][0] == 2, spp


# ---- SPP.cv2's data gradient in isolation ------------------------------------------------------------------------------------------
SPP_CASES = {  # (B, H, W, 4 c_ = the data gradient's output channels, c2)
    "l_512x1024": (4, 16, 32, 2048, 1024),
    "x_512x1024": (4, 16, 32, 2560, 1280),
    "x_rect_416x736": (4, 13, 23, 2560, 1280),
}


@pytest.mark.parametrize("name", list(SPP_CASES))
def test_spp_cv2_data_gradient_on_wgmma(name):
    B, H, W, ci, co = SPP_CASES[name]
    info, err, ok = run(B=B, H=H, W=W, ci=ci, co=co, x_off=8, gin_off=8, dy_off=24, seed=len(name))
    print(f"\n[{name}] {describe(info)}\n[{name}] " + "  ".join(f"{k} {v:.2e}" for k, v in err.items()))
    assert info[0] == 2 and info[3] == 64 and info[4] == 128 and info[13] == ci // 128, describe(info)
    assert err["dgrad"] <= LIMIT_DGRAD["wgmma"], err
    fails = check(name, info, err, ok)
    assert not fails, "\n".join(fails)


# ---- training ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("tag", ["l_psp", "x_bise"])
def test_train_forward_and_backward_match_autograd_oracle(tag):
    """test_gpu_train.py's parity bar at 2 x 128 x 256: forward per output and gradients (median and worst) no further from the fp32
    autograd oracle than torch autocast x 1.25.  Its absolute bounds (forward 0.10, gradients 0.25 / 0.40, cosine 0.95) were set for s and
    m: at l / x depth torch autocast itself is further away (H100: forward up to 0.20 (l) and 0.56 (x) relative Frobenius), so here they
    are printed, and the yardstick alone decides"""
    B, H, W = 2, 128, 256
    model, cfg, sd, x = setup(tag, CONFIGS[tag], B=B, H=H, W=W)
    torch.set_num_threads(min(32, os.cpu_count() or 1))
    gen = torch.Generator().manual_seed(11)
    raws, seg = model(x.cuda())
    segs = seg if isinstance(seg, list) else [seg]
    assert len(segs) == (3 if tag.endswith("bise") else 1)
    Rs = [torch.randn(r.shape, generator=gen) * 4.0 for r in raws]
    S = [torch.randn(g.shape, generator=gen) * 0.05 for g in segs]
    loss = sum((r * R.cuda()).sum() for r, R in zip(raws, Rs)) + sum((g * Sk.cuda()).sum() for g, Sk in zip(segs, S))
    loss.backward()
    torch.cuda.synchronize()
    dmask = dropout_mask_of(model)
    o_raw, o_seg, sdg = oracle_train(cfg, sd, x, Rs, S, dmask)
    amp_fwd, amp_grd = amp_yardstick(cfg, sd, x, Rs, S, o_raw, o_seg, sdg, dmask)
    ours_fwd = [rel_f(a.detach().cpu(), b.detach()) for a, b in zip(list(raws) + segs, list(o_raw) + list(o_seg))]
    print("\n[%s] train forward rel err: ours %s | torch autocast %s" % (tag, np.round(ours_fwd, 4), np.round(amp_fwd, 4)))
    assert all(o <= 1.25 * a + 2e-3 for o, a in zip(ours_fwd, amp_fwd)), (ours_fwd, amp_fwd)
    errs, coss = {}, {}
    for name, p in model.named_parameters():
        g_ref = sdg[name].grad
        assert p.grad is not None and g_ref is not None, name
        if g_ref.norm() < 1e-8:
            continue
        g = p.grad.detach().cpu()
        errs[name] = rel_f(g, g_ref)
        coss[name] = float((g.double().flatten() @ g_ref.double().flatten()) / (g.double().norm() * g_ref.double().norm()))
    worst = max(errs.items(), key=lambda kv: kv[1])
    med, amp_med = float(np.median(list(errs.values()))), float(np.median(list(amp_grd.values())))
    print("[%s] gradient rel err: ours median %.3e max %.3e (%s) | torch autocast median %.3e max %.3e; min cosine %.4f"
          % (tag, med, worst[1], worst[0], amp_med, max(amp_grd.values()), min(coss.values())))
    assert worst[1] <= 1.25 * max(amp_grd.values()), (worst, max(amp_grd.values()))
    assert med <= 1.25 * amp_med, (med, amp_med)
    assert errs["model.25.m.0.bias"] < 1e-5


@pytest.mark.parametrize("tag", ["l_psp", "x_bise"])
def test_trainer_step(tag):
    """det pass + seg pass + SGD on one fixed batch (reference train.py:363-401): finite losses that fall and a loss scale that settles"""
    from multiyolov5_b200.train import Trainer, scale_hyp
    B, H, W = 2, 128, 256
    model, cfg, _, _ = setup(tag, CONFIGS[tag], B=B, H=H, W=W)
    hyp = dict(lr0=0.01, momentum=0.937, weight_decay=5e-4, box=0.05, cls=0.5, cls_pw=1.0, obj=1.0, obj_pw=1.0, anchor_t=4.0, fl_gamma=0.0)
    tr = Trainer(model, scale_hyp(hyp, nl=3, nc=cfg["nc"], imgsz=W, total_batch_size=2 * B), batch_size=B, init_scale=2.0 ** 10)
    assert tr.n_seg_outputs == (3 if tag.endswith("bise") else 1)
    rs = np.random.RandomState(0)
    imgs = synth.synth_image(B, H, W, seed=1).cuda()
    segimgs = synth.synth_image(B, H, W, seed=2).cuda()
    t = np.zeros((12, 6), np.float32)
    t[:, 0] = rs.randint(0, B, 12); t[:, 1] = rs.randint(0, cfg["nc"], 12)
    t[:, 2:4] = rs.uniform(0.1, 0.9, (12, 2)); t[:, 4:6] = rs.uniform(0.05, 0.4, (12, 2))
    targets = torch.from_numpy(t).cuda()
    mask = torch.from_numpy(rs.randint(-1, 19, (B, 1, H // 8, W // 8)).astype(np.int64)).cuda()
    mask = mask.repeat_interleave(8, 2).repeat_interleave(8, 3)[:, 0].contiguous()
    hist = []
    for _ in range(30):
        items, segloss = tr.step(imgs, targets, segimgs, mask)
        hist.append((float(items[3]), float(segloss)))
    print(f"\n[{tag}] loss (det, seg): first {hist[0]} last {hist[-1]}, scale {float(tr.scale):.0f}")
    assert all(np.isfinite(h).all() for h in hist)
    assert hist[-1][0] < 0.8 * hist[0][0] and hist[-1][1] < 0.85 * hist[0][1], (hist[0], hist[-1])
    assert float(tr.scale) >= 1.0
