"""H100: the reference's class-weighted CE and SegFocalLoss on the device.  utils.loss.SegFocalLoss (and the weighted CE through the same
kernels) against the reference's cases (tests/golden/segloss_cases.npz); the fused upsample + weighted / focal pass of the train plan
against torch in fp64 on the same low-resolution logits, eagerly and under graph replay on one plan; Trainer steps with the weighted CE
and the focal loss on s/PSP (fused against autograd), s/BiSe (weighted CE with aux) and a 2-class head (focal, autograd)."""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import restate_segloss as rs
from oracle import synth

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden")
HYP = dict(lr0=0.01, momentum=0.937, weight_decay=5e-4, box=0.05, cls=0.5, cls_pw=1.0, obj=1.0, obj_pw=1.0, anchor_t=4.0, fl_gamma=0.0)


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


def class_weights(n, seed=0):
    return torch.from_numpy(np.random.RandomState(seed).uniform(0.5, 1.5, n).astype(np.float32))


def torch_focal(z, t, w, gamma, ignore_index=-1):
    """the reference's SegFocalLoss(gamma, alpha=w, ignore_index, 'mean') formula in torch (gamma = 0: CrossEntropyLoss(weight=w))"""
    ce = F.cross_entropy(z, t, weight=w, ignore_index=ignore_index)
    tp = t * (t != ignore_index).long()
    pt = torch.gather(F.softmax(z, 1), 1, tp.unsqueeze(1))
    return (torch.pow(1 - pt, gamma) * ce).mean()


def test_module_matches_the_reference_cases():
    from multiyolov5_b200.utils.loss import SegFocalLoss, seg_focal_loss
    for c in rs.load_cases(os.path.join(GOLD, "segloss_cases.npz"))["cases"]:
        w = None if c["weight"] is None else torch.from_numpy(c["weight"])
        ps = [torch.from_numpy(p).cuda().requires_grad_(True) for p in c["logits"]]
        labels = torch.from_numpy(c["labels"]).cuda()
        if c["kind"] == "focal":
            loss = SegFocalLoss(c["gamma"], w, c["ignore_index"], c["reduction"]).cuda()(ps[0], labels)
        else:                                                                 # the weighted CE as the Trainer computes it
            parts = [seg_focal_loss(p, labels, w, 0.0, c["ignore_index"]) for p in ps]
            aw = c["aux_weight"]
            loss = parts[0] if aw is None else parts[0] + aw * 1.5 * parts[1] + aw / 2.0 * parts[2]
        (loss * 3.0).backward()
        torch.cuda.synchronize()
        ref, got = float(c["loss"]), float(loss.detach())
        if np.isnan(ref):
            assert np.isnan(got), c["name"]
        else:
            assert abs(got - ref) <= 1e-5 * abs(ref), (c["name"], got, ref)
        for p, gr in zip(ps, c["grad"]):
            g = p.grad.cpu().numpy() / 3.0
            fin = np.isfinite(gr)
            np.testing.assert_array_equal(np.isfinite(g), fin, err_msg=c["name"])
            if fin.any():
                assert rel_f(torch.from_numpy(g[fin]), torch.from_numpy(gr[fin])) < 1e-4, c["name"]


def test_fused_pass_matches_torch_on_the_same_logits():
    """the fused pass (myolo_plan_backward_seg_loss) against F.interpolate(align_corners=True) + the reference's formula in fp64 on the SAME
    low-res logits, for gamma in {0, 2} x weights on / off: loss to 1e-5, d loss / d logits to 1e-4 relative.  The four settings run twice
    on one plan: the first calls eagerly, the later ones under the plan's graph replay."""
    from multiyolov5_b200 import _lib
    model, cfg, x = setup(B=2)
    eng = model.engine()
    rng = np.random.RandomState(3)
    labels = torch.from_numpy(np.where(rng.rand(2, 128, 256) < 0.7, rng.randint(0, 19, (2, 128, 256)), -1).astype(np.int64)).cuda()
    w = class_weights(19).cuda()
    _, _, plan = eng.train_forward(x.cuda(), want_seg=False)
    v = [o.in_ for o in plan.pb.ops if o.kind == _lib.OP_SEG_UPSAMPLE][0]
    for it, (gamma, wt) in enumerate([(0.0, None), (0.0, w), (2.0, None), (2.0, w)] * 2):
        model.zero_grad(set_to_none=False)
        _, _, plan = eng.train_forward(x.cuda(), want_seg=False)
        scale = torch.full((), 8.0, device="cuda")
        loss = eng.train_backward_seg_loss(plan, labels, wt, gamma, factor=0.5, scale=scale)
        lo = eng.read_view(v, plan).double().clone().requires_grad_(True)
        dlo = eng.read_grad_view(v, plan)
        up = F.interpolate(lo[:, :19], (128, 256), mode="bilinear", align_corners=True)
        ref = torch_focal(up, labels, None if wt is None else wt.double(), gamma)
        (ref * 0.5 * 8.0).backward()
        torch.cuda.synchronize()
        ref = float(ref.detach())
        assert abs(float(loss) - ref) < 1e-5 * abs(ref), (it, float(loss), ref)
        assert rel_f(dlo[:, :19].cpu(), lo.grad[:, :19].cpu()) < 1e-4, it
    # nothing valid: NaN loss; the weighted CE leaves no gradient, as the reference's
    model.zero_grad(set_to_none=False)
    _, _, plan = eng.train_forward(x.cuda(), want_seg=False)
    loss = eng.train_backward_seg_loss(plan, torch.full_like(labels, -1), w, 0.0)
    assert torch.isnan(loss) and float(dict(model.named_parameters())["model.24.out.3.weight"].grad.abs().sum()) == 0.0


def _det_batch(cfg, B, H, W, seed=0):
    rng = np.random.RandomState(seed)
    t = np.zeros((3 * B, 6), np.float32)
    t[:, 0] = np.repeat(np.arange(B), 3); t[:, 1] = rng.randint(0, cfg["nc"], 3 * B)
    t[:, 2:4] = rng.uniform(0.1, 0.9, (3 * B, 2)); t[:, 4:6] = rng.uniform(0.05, 0.4, (3 * B, 2))
    return synth.synth_image(B, H, W, seed=seed + 1).cuda(), torch.from_numpy(t).cuda()


@pytest.mark.parametrize("kind", ["focal", "weighted_ce"])
def test_trainer_psp_fused_step_matches_the_module_on_autograd_outputs(kind):
    """Trainer.step of s/PSP through the fused pass (concurrent passes) against the same step through the library's loss kernels on
    Model.forward's outputs (autograd, sequential passes).  The same step repeated on one path moves the loss by ~1e-4 relative and the
    gradients by ~10 % (the fp32 atomics of the BN statistics and the weight gradients, amplified by these synthetic weights), so the
    yardstick is that spread: four runs per path, alternating, and the median distance between a fused and an autograd run may be at
    most 3x the median distance between two runs of the noisier path (floors: 1e-5 relative for the loss, 1e-4 for the gradients).  With
    one pair of runs per path the comparison would fail by chance: when all three distances come from one distribution, the cross distance
    exceeds 3x the larger within-path one in several percent of runs.  The head's dropout is off: every forward draws a new mask,
    which would add the masks' spread to both sides."""
    from multiyolov5_b200.train import Trainer, scale_hyp
    from multiyolov5_b200.utils.loss import SegFocalLoss, SegmentationLosses
    model, cfg, _ = setup(B=4)
    for m in model.modules():
        if isinstance(m, torch.nn.Dropout):
            m.p = 0.0
    w = class_weights(19)
    seg_loss = SegFocalLoss(gamma=2, alpha=w, ignore_index=-1) if kind == "focal" else SegmentationLosses(ignore_index=-1, weight=w)
    tr = Trainer(model, scale_hyp(HYP, nl=3, nc=cfg["nc"], imgsz=256, total_batch_size=4), batch_size=4, accumulate=1000,
                 init_scale=2.0 ** 10, seg_loss=seg_loss)
    assert tr.fused_seg and tr.seg_wf is not None and tr.seg_wf[0].is_cuda
    imgs, targets = _det_batch(cfg, 4, 128, 256)
    segimgs = synth.synth_image(4, 128, 256, seed=9).cuda()
    rng = np.random.RandomState(4)
    mask = torch.from_numpy(rng.randint(-1, 19, (4, 128, 256)).astype(np.int64)).cuda()
    runs = {True: [], False: []}
    for fused in (True, False, False, True) * 2:              # accumulate=1000: no optimizer step, every run sees the same weights
        tr.fused_seg = fused
        tr.flat.grad.zero_()
        _, segloss = tr.step(imgs, targets, segimgs, mask)
        runs[fused].append((float(segloss), tr.flat.grad.clone().cpu()))
    assert all(np.isfinite(l) for rs in runs.values() for l, _ in rs)

    def median_dist(pairs, d):
        return float(np.median([d(a, b) for a, b in pairs]))

    within = [[(a, b) for i, a in enumerate(rs) for b in rs[i + 1:]] for rs in runs.values()]
    cross = [(a, b) for a in runs[True] for b in runs[False]]
    la = float(np.mean([l for l, _ in runs[False]]))
    dl, dg = (lambda a, b: abs(a[0] - b[0])), (lambda a, b: rel_f(a[1], b[1]))
    l_within, l_cross = max(median_dist(w, dl) for w in within), median_dist(cross, dl)    # the noisier path's spread
    g_within, g_cross = max(median_dist(w, dg) for w in within), median_dist(cross, dg)
    assert g_cross <= max(3 * g_within, 1e-4), (g_cross, g_within)
    assert l_cross <= max(3 * l_within, 1e-5 * abs(la)), (l_cross, l_within, la)


def test_trainer_bise_weighted_ce_step():
    from multiyolov5_b200.train import Trainer, scale_hyp
    from multiyolov5_b200.utils.loss import SegmentationLosses
    model, cfg, _ = setup("s_bise", "yolov5s_city_seg_bise.yaml", B=2)
    seg_loss = SegmentationLosses(nclass=19, aux=True, aux_num=2, aux_weight=0.1, ignore_index=-1, weight=class_weights(19))
    tr = Trainer(model, scale_hyp(HYP, nl=3, nc=cfg["nc"], imgsz=256, total_batch_size=2), batch_size=2, init_scale=2.0 ** 10,
                 seg_loss=seg_loss)
    assert not tr.fused_seg and tr.n_seg_outputs == 3
    segimgs = synth.synth_image(2, 128, 256, seed=9).cuda()
    rng = np.random.RandomState(0)
    mask = torch.from_numpy(rng.randint(-1, 19, (2, 128, 256)).astype(np.int64)).cuda()
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


def test_trainer_two_class_head_focal_step():
    """the custom dataset's head (nc=1, n_segcls=2, from the s/PSP yaml): SegFocalLoss(gamma=2, ignore_index=-1) through autograd"""
    from multiyolov5_b200.models.yolo import Model
    from multiyolov5_b200.train import Trainer, scale_hyp
    from multiyolov5_b200.utils.loss import SegFocalLoss
    cfg = synth.load_cfg("yolov5s_city_seg.yaml")
    cfg["nc"], cfg["n_segcls"] = 1, 2
    model = Model(cfg)
    manifest = [[k, list(t.shape), str(t.dtype).replace("torch.", "")] for k, t in model.state_dict().items()]
    model.load_state_dict(synth.synth_state_dict(manifest, cfg, seed=1, gain=1.0))
    model.cuda().train()
    crit = SegFocalLoss(gamma=2, ignore_index=-1)
    tr = Trainer(model, scale_hyp(HYP, nl=3, nc=1, imgsz=256, total_batch_size=2), batch_size=2, init_scale=2.0 ** 10, seg_loss=crit)
    assert not tr.fused_seg and model.model[-2].c_out == 2
    segimgs = synth.synth_image(2, 128, 256, seed=9).cuda()
    rng = np.random.RandomState(1)
    mask = torch.from_numpy(rng.randint(-1, 2, (2, 128, 256)).astype(np.int64)).cuda()
    model.zero_grad(set_to_none=False)
    segloss = tr.backward_seg(segimgs, mask)
    torch.cuda.synchronize()
    assert np.isfinite(float(segloss)) and float(segloss) > 0
    assert float(dict(model.named_parameters())["model.24.out.3.weight"].grad.abs().sum()) > 0
    imgs, targets = _det_batch(cfg, 2, 128, 256)
    hist = [float(tr.step(imgs, targets, segimgs, mask)[1]) for _ in range(3)]
    assert np.isfinite(hist).all()
