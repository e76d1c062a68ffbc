"""H100: the reference's OhemCELoss on the device.  utils.loss.OhemCELoss against the reference's cases (tests/golden/ohem_cases.npz);
exact ties at the k-th value; the fused upsample + CE + OHEM pass of the train plan against torch on the same low-resolution logits, with
the branch switching between calls on one plan, eagerly and under graph replay; Trainer steps with seg_loss=OhemCELoss on s/PSP (fused)
and s/BiSe (autograd, aux=True)."""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import restate_ohem as ro
from oracle import synth

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden")


def rel_f(a, b):
    a = a.double(); b = b.double()
    return float((a - b).norm() / (b.norm() + 1e-30))


def setup(tag="s_psp", yml="yolov5s_city_seg.yaml", B=4, H=128, W=256):
    from multiyolov5_b200.models.yolo import Model
    cfg = synth.load_cfg(yml)
    sd = synth.synth_state_dict(synth.load_manifest(tag), cfg, seed=1, gain=1.0)
    model = Model(yml)
    model.load_state_dict(sd)
    model.cuda().train()
    return model, cfg, synth.synth_image(B, H, W, seed=5)


def test_module_matches_the_reference_cases():
    from multiyolov5_b200.utils.loss import OhemCELoss
    g = ro.load_cases(os.path.join(GOLD, "ohem_cases.npz"))
    for c in g["cases"]:
        crit = OhemCELoss(c["thresh"], c["ignore_index"], c["aux"], c["aux_weight"])
        ps = [p.cuda().requires_grad_(True) for p in c["logits"]]
        labels = c["labels"].cuda()
        loss = crit(ps if c["aux"] else ps[0], labels)
        (loss * 3.0).backward()
        torch.cuda.synchronize()
        if c["name"] == "all_ignored":
            assert torch.isnan(loss) and all(float(p.grad.abs().sum()) == 0.0 for p in ps)
            continue
        loss = loss.detach()
        assert abs(float(loss) - float(c["loss"])) <= 1e-5 * abs(float(c["loss"])), (c["name"], float(loss), float(c["loss"]))
        for p, gr in zip(ps, c["grad"]):
            assert rel_f(p.grad.cpu() / 3.0, gr) < 1e-4, c["name"]


def test_exact_ties_take_the_lowest_indices():
    """hundreds of pixels share the n_min-th CE: exactly n_min gradient rows are non-zero, the tied ones taken are the lowest flat indices"""
    from multiyolov5_b200.utils.loss import OhemCELoss
    B, C, H, W = 2, 7, 64, 96
    g = torch.Generator().manual_seed(3)
    proto = torch.randn(C, generator=g)
    xl = proto.repeat(B * H * W, 1)                                         # every pixel the same logits ...
    labels = torch.zeros(B * H * W, dtype=torch.long)                       # ... and the same label: one CE value everywhere
    hi = torch.rand(B * H * W, generator=g) < 0.01                          # ~120 pixels with a larger CE (label 1, made unlikely)
    labels[hi] = 1
    xl[hi, 1] -= 4.0
    labels[torch.rand(B * H * W, generator=g) < 0.05] = -1
    x = xl.view(B, H, W, C).permute(0, 3, 1, 2).contiguous()
    labels = labels.view(B, H, W)
    crit = OhemCELoss(0.7)
    crit.thresh_t = 50.0                                                    # nothing is hard: the top-k branch
    xc, lc = x.cuda().requires_grad_(True), labels.cuda()
    loss = crit(xc, lc)
    loss.backward()
    n_min = int((labels != -1).sum()) // 16
    per = F.cross_entropy(x, labels, ignore_index=-1, reduction="none").view(-1)
    mask = ro.topk_mask(per, n_min)
    rows = (xc.grad.permute(0, 2, 3, 1).reshape(-1, C) != 0).any(1).cpu()
    kth = torch.sort(per, descending=True).values[n_min - 1]
    assert int((per == kth).sum()) > 200 and int(rows.sum()) == n_min
    assert torch.equal(rows, mask)
    ref = per.topk(n_min).values.mean()
    assert abs(float(loss.detach()) - float(ref)) <= 1e-5 * float(ref)


def _margin_ok(vals, boundary, rel=1e-5):
    return bool(((vals - boundary).abs() > rel * abs(boundary)).all())


def test_fused_ohem_matches_torch_on_the_same_logits_and_switches_branch():
    """the fused pass (myolo_plan_backward_seg_ohem) against F.interpolate(align_corners=True) + the restated OHEM on the SAME low-res
    logits: loss to 1e-5, d loss / d logits to 1e-4 relative.  The branch alternates from call to call on one plan: top-k (thresh_t above
    every CE) and threshold (thresh_t in a gap of the CEs); the seeded labels are chosen so that no CE lies within 1e-5 of the boundary."""
    from multiyolov5_b200 import _lib
    model, cfg, x = setup(B=2)
    eng = model.engine()
    _, _, plan = eng.train_forward(x.cuda(), want_seg=False)
    v = [o.in_ for o in plan.pb.ops if o.kind == _lib.OP_SEG_UPSAMPLE][0]
    lo = eng.read_view(v, plan)[:, :19].clone()
    up = F.interpolate(lo, (128, 256), mode="bilinear", align_corners=True)
    for seed in range(50):                                                   # labels: ~4 % valid pixels, the rest ignored
        rs = np.random.RandomState(seed)
        labels = torch.from_numpy(np.where(rs.rand(2, 128, 256) < 0.04, rs.randint(0, 19, (2, 128, 256)), -1).astype(np.int64)).cuda()
        per = F.cross_entropy(up, labels, ignore_index=-1, reduction="none").view(-1)
        valid = per[labels.view(-1) != -1]
        n_min = valid.numel() // 16
        srt = torch.sort(per, descending=True).values
        kth = srt[n_min - 1]
        others = torch.cat((srt[:n_min - 1], srt[n_min:]))
        vs = torch.sort(valid).values
        gaps = vs[1:] - vs[:-1]
        mid = slice(valid.numel() // 4, valid.numel() // 2)                 # hard count between 1/2 and 3/4 of the valid: >= n_min
        j = int(torch.argmax(gaps[mid])) + valid.numel() // 4
        th_gap = float((vs[j] + vs[j + 1]) / 2)
        if _margin_ok(others, kth) and _margin_ok(valid, th_gap):
            break
    else:
        pytest.fail("no seeded labels keep the margins")
    th_top = float(per.max()) * 2 + 1.0
    for it, th in enumerate([th_top, th_gap, th_top, th_gap]):              # eager, warm, then replays of the plan's graphs
        model.zero_grad(set_to_none=False)
        _, _, plan = eng.train_forward(x.cuda(), want_seg=False)
        scale = torch.full((), 8.0, device="cuda")
        loss = eng.train_backward_seg_ohem(plan, labels, th, factor=0.5, scale=scale)
        lo = eng.read_view(v, plan).clone().requires_grad_(True)
        dlo = eng.read_grad_view(v, plan)
        upg = F.interpolate(lo[:, :19], (128, 256), mode="bilinear", align_corners=True)
        pl = F.cross_entropy(upg, labels, ignore_index=-1, reduction="none").view(-1)
        taken = pl.detach() > th
        if int(taken.sum()) < n_min:
            taken = ro.topk_mask(pl.detach(), n_min)
        assert (it % 2 == 0) == (int((pl.detach() > th).sum()) < n_min)
        ref = pl[taken].mean()
        (ref * 0.5 * 8.0).backward()
        torch.cuda.synchronize()
        assert abs(float(loss) - float(ref)) < 1e-5 * abs(float(ref)), (it, float(loss), float(ref))
        assert rel_f(dlo[:, :19].cpu(), lo.grad[:, :19].cpu()) < 1e-4, it
    # nothing valid: n_min = 0 and no hard pixel -> NaN loss, no gradient
    model.zero_grad(set_to_none=False)
    _, _, plan = eng.train_forward(x.cuda(), want_seg=False)
    loss = eng.train_backward_seg_ohem(plan, torch.full_like(labels, -1), th_gap)
    assert torch.isnan(loss) and float(dict(model.named_parameters())["model.24.out.3.weight"].grad.abs().sum()) == 0.0


def test_module_under_graph_replay_switches_branch():
    """myolo_seg_ohem_loss / _backward captured once in a CUDA graph: replays with new logits take either branch"""
    from multiyolov5_b200.utils.loss import OhemCELoss
    B, C, H, W = 2, 19, 64, 128
    crit = OhemCELoss(0.7)
    x = torch.zeros(B, C, H, W, device="cuda", requires_grad=True)
    labels = torch.randint(0, C, (B, H, W), device="cuda", generator=torch.Generator("cuda").manual_seed(1))
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(2):
            x.grad = None
            crit(x, labels).backward()
    torch.cuda.current_stream().wait_stream(side)
    x.grad = None
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        loss = crit(x, labels)
        loss.backward()
    oh = F.one_hot(labels, C).permute(0, 3, 1, 2).float()
    th = ro.thresh_t(0.7)
    n_min = labels.numel() // 16
    for it, bias in enumerate([0.0, 9.0, 0.0, 9.0]):                        # plain randn logits: threshold; strong label bias: top-k
        for seed in range(100 * it, 100 * it + 100):                        # seeded logits with every CE away from the boundary
            xn = torch.randn(B, C, H, W, device="cuda", generator=torch.Generator("cuda").manual_seed(seed)) + bias * oh
            per = F.cross_entropy(xn, labels, reduction="none").view(-1)
            srt = torch.sort(per, descending=True).values
            if _margin_ok(per, th) and _margin_ok(torch.cat((srt[:n_min - 1], srt[n_min:])), srt[n_min - 1]):
                break
        else:
            pytest.fail("no seeded logits keep the margins")
        with torch.no_grad():
            x.copy_(xn)
        graph.replay()
        xr = x.detach().clone().requires_grad_(True)
        ref = ro.forward_once(xr, labels, 0.7)
        ref.backward()
        torch.cuda.synchronize()
        assert (it % 2 == 1) == (int((per > th).sum()) < n_min)
        assert abs(float(loss) - float(ref)) < 1e-5 * float(ref), it
        assert rel_f(x.grad.cpu(), xr.grad.cpu()) < 1e-4, it


def _det_batch(cfg, B, H, W, seed=0):
    rs = np.random.RandomState(seed)
    t = np.zeros((3 * B, 6), np.float32)
    t[:, 0] = np.repeat(np.arange(B), 3); t[:, 1] = rs.randint(0, cfg["nc"], 3 * B)
    t[:, 2:4] = rs.uniform(0.1, 0.9, (3 * B, 2)); t[:, 4:6] = rs.uniform(0.05, 0.4, (3 * B, 2))
    return synth.synth_image(B, H, W, seed=seed + 1).cuda(), torch.from_numpy(t).cuda()


HYP = dict(lr0=0.01, momentum=0.937, weight_decay=5e-4, box=0.05, cls=0.5, cls_pw=1.0, obj=1.0, obj_pw=1.0, anchor_t=4.0, fl_gamma=0.0)


def test_trainer_psp_fused_ohem_step_matches_the_module_on_autograd_outputs():
    """one Trainer.step of s/PSP with seg_loss=OhemCELoss(0.7) through the fused pass (concurrent passes) against the same step through
    OhemCELoss on Model.forward's outputs (autograd, sequential passes).  The yardstick is each path's own run-to-run spread (the fp32
    atomics of the BN statistics and the weight gradients change the last bits from run to run, and these synthetic weights amplify
    them), with 1e-4 relative for the gradients and 1e-5 for the loss as the floor."""
    from multiyolov5_b200.train import Trainer, scale_hyp
    from multiyolov5_b200.utils.loss import OhemCELoss
    model, cfg, _ = setup(B=4)
    tr = Trainer(model, scale_hyp(HYP, nl=3, nc=cfg["nc"], imgsz=256, total_batch_size=4), batch_size=4, accumulate=1000,
                 init_scale=2.0 ** 10, seg_loss=OhemCELoss(0.7))
    assert tr.fused_seg and tr.ohem is not None
    imgs, targets = _det_batch(cfg, 4, 128, 256)
    segimgs = synth.synth_image(4, 128, 256, seed=9).cuda()
    rs = np.random.RandomState(4)
    mask = torch.from_numpy(rs.randint(-1, 19, (4, 128, 256)).astype(np.int64)).cuda()
    runs = []
    for fused in (True, False, False, True):                 # accumulate=1000: no optimizer step, every run sees the same weights
        tr.fused_seg = fused                                 # False: the same step through OhemCELoss on Model.forward's outputs
        tr.flat.grad.zero_()
        _, segloss = tr.step(imgs, targets, segimgs, mask)
        runs.append((float(segloss), tr.flat.grad.clone().cpu()))
    (lf, gf), (la, ga), (la2, ga2), (lf2, gf2) = runs
    assert all(np.isfinite(v[0]) for v in runs)
    g_spread = max(rel_f(ga2, ga), rel_f(gf2, gf))
    l_spread = max(abs(la2 - la), abs(lf2 - lf))
    assert rel_f(gf, ga) <= max(3 * g_spread, 1e-4), (rel_f(gf, ga), g_spread)
    assert abs(lf - la) <= max(3 * l_spread, 1e-5 * abs(la)), (lf, la, l_spread)


def test_trainer_bise_aux_ohem_step():
    from multiyolov5_b200.train import Trainer, scale_hyp
    from multiyolov5_b200.utils.loss import OhemCELoss
    model, cfg, _ = setup("s_bise", "yolov5s_city_seg_bise.yaml", B=2)
    tr = Trainer(model, scale_hyp(HYP, nl=3, nc=cfg["nc"], imgsz=256, total_batch_size=2), batch_size=2, init_scale=2.0 ** 10,
                 seg_loss=OhemCELoss(0.7, aux=True, aux_weight=[0.15, 0.1]))
    assert not tr.fused_seg and tr.n_seg_outputs == 3
    segimgs = synth.synth_image(2, 128, 256, seed=9).cuda()
    rs = np.random.RandomState(0)
    mask = torch.from_numpy(rs.randint(-1, 19, (2, 128, 256)).astype(np.int64)).cuda()
    model.zero_grad(set_to_none=False)
    segloss = tr.backward_seg(segimgs, mask)
    torch.cuda.synchronize()
    named = dict(model.named_parameters())
    assert np.isfinite(float(segloss)) and float(segloss) > 0
    for k in ("model.24.out.2.weight", "model.24.aux16.1.weight", "model.24.aux32.1.weight"):
        assert float(named[k].grad.abs().sum()) > 0, k
    assert float(named["model.25.m.0.weight"].grad.abs().sum()) == 0.0    # the seg pass leaves the det head untouched
    imgs, targets = _det_batch(cfg, 2, 128, 256)
    hist = [float(tr.step(imgs, targets, segimgs, mask)[1]) for _ in range(3)]
    assert np.isfinite(hist).all()
