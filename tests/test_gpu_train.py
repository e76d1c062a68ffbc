"""GPU: training row (SURVEY.md section 8 a13) - train-mode forward (batch-statistics BatchNorm) and the hand-written backward against
torch.autograd on the oracle's fp32 restatement of the same graph (oracle.restate.model_forward_train).  fp16 activation / gradient
storage: tolerances are relative Frobenius errors per tensor."""
import numpy as np
import pytest
import torch

from oracle import restate, synth

pytestmark = pytest.mark.gpu


def rel_f(a, b):
    a = a.double(); b = b.double()
    return float((a - b).norm() / (b.norm() + 1e-30))


def setup(tag="s_psp", yml="yolov5s_city_seg.yaml", B=4, H=128, W=256):
    from multiyolov5_b200.models.yolo import Model
    cfg = synth.load_cfg(yml)
    sd = synth.synth_state_dict(synth.load_manifest(tag), cfg, seed=1, gain=1.0)   # contractive weights: well-conditioned gradients
    model = Model(yml)
    model.load_state_dict(sd)
    model.cuda().train()
    x = synth.synth_image(B, H, W, seed=5)
    return model, cfg, sd, x


def oracle_train(cfg, sd, x, Rs, S, dropout_mask=None):
    sdg = {k: (v.clone().requires_grad_(True) if v.is_floating_point() and "running" not in k and "anchor" not in k else v.clone())
           for k, v in sd.items()}
    raw, seg = restate.model_forward_train(cfg, sdg, x, dropout_mask)
    segs = seg if isinstance(seg, list) else [seg]
    loss = sum((r * R).sum() for r, R in zip(raw, Rs)) + sum((g * Sk).sum() for g, Sk in zip(segs, S))
    loss.backward()
    return raw, segs, sdg


def dropout_mask_of(model):
    """the keep mask our last train forward applied (Base head): read back so that the oracle can apply the same one"""
    from multiyolov5_b200 import _lib
    eng = model.engine()
    ops = [o for o in eng.last_plan.pb.ops if o.kind == _lib.OP_DROPOUT]
    if not ops:
        return None
    xin, xout = eng.read_view(ops[0].in_), eng.read_view(ops[0].out)
    keep = ((xout != 0) | (xin == 0)).float()
    frac = float(keep.mean())
    assert 0.88 < frac < 0.92, frac                                   # Bernoulli(0.9)
    assert torch.allclose(xout, xin * keep / 0.9, rtol=2e-3, atol=1e-6)   # kept values scaled by 1/(1-p) (fp16 rounding)
    return keep.cpu()


def amp_yardstick(cfg, sd, x, Rs, S, ref_raw, ref_seg, ref_sdg, dropout_mask=None):
    """the SAME restated graph through torch's fp16 autocast on the GPU - what the reference's `amp.autocast` training computes
    (train.py:363) - measured against the fp32 oracle: the error level an fp16-storage path is entitled to."""
    sda = {k: (v.detach().clone().cuda().requires_grad_(True) if v.requires_grad else v.detach().clone().cuda()) for k, v in ref_sdg.items()}
    with torch.autocast("cuda", dtype=torch.float16):
        araw, aseg = restate.model_forward_train(cfg, sda, x.cuda(), None if dropout_mask is None else dropout_mask.cuda())
    asegs = aseg if isinstance(aseg, list) else [aseg]
    loss = sum((r.float() * R.cuda()).sum() for r, R in zip(araw, Rs)) + sum((g.float() * Sk.cuda()).sum() for g, Sk in zip(asegs, S))
    loss.backward()
    fwd = [rel_f(a.detach().float().cpu(), b.detach()) for a, b in zip(list(araw) + asegs, list(ref_raw) + list(ref_seg))]
    grd = {n: rel_f(v.grad.float().cpu(), ref_sdg[n].grad) for n, v in sda.items()
           if v.requires_grad and ref_sdg[n].grad is not None and ref_sdg[n].grad.norm() > 1e-8}
    return fwd, grd


TRAIN_CASES = {"s_psp": "yolov5s_city_seg.yaml", "m_lab": "yolov5m_city_seg_lab.yaml", "s_base": "yolov5s_city_seg_base.yaml",
               "s_bise": "yolov5s_city_seg_bise.yaml"}


# (tag, B, H, W): the four heads at 128x256, and BASELINE.json configs[3]'s per-GPU slice (4 x 3 x 512 x 1024, every conv on the wgmma
# kernels, the bench's weights) for the flagship model
PARITY_CASES = [("s_psp", 4, 128, 256), ("m_lab", 2, 128, 256), ("s_base", 2, 128, 256), ("s_bise", 2, 128, 256), ("s_psp", 4, 512, 1024)]


@pytest.mark.parametrize("tag,B,H,W", PARITY_CASES)
def test_train_forward_and_backward_match_autograd_oracle(tag, B, H, W):
    """Parity bar for fp16-storage training: against the fp32 autograd oracle our forward / gradients must be (a) no further away than
    torch's own fp16 autocast of the same graph (x1.25 slack for run-to-run noise; forward per output, gradient median and worst) and
    (b) within loose absolute sanity bounds: forward 0.10 relative Frobenius, gradients median 0.25 / worst 0.40, cosine >= 0.95 on
    every parameter (a wrong formula in any op shows up as cosine << 0.9 downstream of it).  (Deep BN networks amplify
    fp16 rounding noise - max-pool argmax flips in SPP alone double the error upstream of it; tools/train_diag.py prints the
    per-layer picture.  Ours and torch autocast sit at the same level, a few 1e-2.)"""
    model, cfg, sd, x = setup(tag, TRAIN_CASES[tag], B=B, H=H, W=W)
    torch.set_num_threads(min(32, __import__("os").cpu_count() or 1))       # the fp32 autograd oracle runs on the host
    gen = torch.Generator().manual_seed(11)
    out = model(x.cuda())
    raws, seg = out
    segs = seg if isinstance(seg, list) else [seg]          # BiSe: [out, aux16, aux32] (reference models/yolo.py:86)
    assert len(segs) == (3 if tag == "s_bise" else 1)
    assert len(raws) == 3 and raws[0].shape == (x.shape[0], 3, H // 8, W // 8, 15)
    assert all(g.shape == (x.shape[0], 19, H, W) and g.requires_grad for g in segs)
    Rs = [torch.randn(r.shape, generator=gen) * 4.0 for r in raws]
    S = [torch.randn(g.shape, generator=gen) * 0.05 for g in segs]
    loss = sum((r * R.cuda()).sum() for r, R in zip(raws, Rs)) + sum((g * Sk.cuda()).sum() for g, Sk in zip(segs, S))
    loss.backward()
    torch.cuda.synchronize()
    dmask = dropout_mask_of(model)
    assert (dmask is not None) == (tag in ("s_base", "s_bise"))
    o_raw, o_seg, sdg = oracle_train(cfg, sd, x, Rs, S, dmask)
    amp_fwd, amp_grd = amp_yardstick(cfg, sd, x, Rs, S, o_raw, o_seg, sdg, dmask)
    ours_fwd = [rel_f(a.detach().cpu(), b.detach()) for a, b in zip(list(raws) + segs, list(o_raw) + list(o_seg))]
    print("\ntrain forward rel err: ours %s | torch autocast %s" % (np.round(ours_fwd, 4), np.round(amp_fwd, 4)))
    assert max(ours_fwd) < 0.10, ours_fwd
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
    worst = sorted(errs.items(), key=lambda kv: -kv[1])[:5]
    med, amp_med = float(np.median(list(errs.values()))), float(np.median(list(amp_grd.values())))
    print("gradient rel err: ours median %.3e max %.3e | torch autocast median %.3e max %.3e; worst %s"
          % (med, worst[0][1], amp_med, max(amp_grd.values()), [(k, round(v, 4)) for k, v in worst]))
    assert len(errs) > 150
    assert med < 0.25 and worst[0][1] < 0.40 and min(coss.values()) > 0.95, (med, worst, min(coss.values()))
    assert worst[0][1] <= 1.25 * max(amp_grd.values()), (worst, max(amp_grd.values()))
    assert med <= 1.25 * amp_med, (med, amp_med)
    # biases of the fp32 heads see the fp32 gradient: exact up to summation order
    assert errs["model.25.m.0.bias"] < 1e-5
    if tag == "s_psp":
        assert errs["model.24.out.3.bias"] < 1e-5


def test_running_stats_and_accumulation():
    model, cfg, sd, x = setup(B=2, H=64, W=128)
    bn0 = model.model[0].conv.bn
    rm0 = bn0.running_mean.clone()
    out = model(x.cuda())
    (out[1].sum() * 1e-3).backward()
    g1 = model.model[-2].out[3].weight.grad.clone() if hasattr(model.model[-2], "out") else None
    gb1 = {n: p.grad.clone() for n, p in model.named_parameters() if n.endswith("m.0.bias") or n.endswith("out.3.bias")}
    # running_mean <- (1-m)*old + m*batch_mean   (reference utils/torch_utils.py:150-152 momentum 0.03)
    xs = x[..., ::2, ::2], x[..., 1::2, ::2], x[..., ::2, 1::2], x[..., 1::2, 1::2]
    u = torch.nn.functional.conv2d(torch.cat(xs, 1), sd["model.0.conv.conv.weight"], None, 1, 1)
    want = 0.97 * rm0.cpu() + 0.03 * u.mean((0, 2, 3))
    assert rel_f(bn0.running_mean.cpu(), want) < 2e-2
    assert int(bn0.num_batches_tracked) == 1
    # a second forward/backward ACCUMULATES into .grad (det pass + seg pass of one iteration, train.py:371,392).  The head bias
    # gradients depend only on the seed gradient, so they double exactly; deeper gradients double up to fp16 run-to-run noise
    # (atomics reorder sums -> fp16 roundings flip -> the two passes decorrelate at the noise floor of the pipeline).
    out = model(x.cuda())
    (out[1].sum() * 1e-3).backward()
    for n, g in gb1.items():
        p = dict(model.named_parameters())[n]
        if g.norm() > 0:
            assert rel_f(p.grad.cpu(), 2 * g.cpu()) < 1e-5, n
    g_a = model.model[1].conv.weight.grad
    assert g_a.abs().sum() > 0
    # det-only backward leaves the seg head untouched (ops with an all-zero output gradient are skipped) and vice versa
    model.zero_grad(set_to_none=False)
    out = model(x.cuda())
    out[0][1].sum().backward()
    named = dict(model.named_parameters())
    assert float(named["model.24.out.3.weight"].grad.abs().sum()) == 0.0
    assert float(named["model.25.m.1.weight"].grad.abs().sum()) > 0 and float(named["model.25.m.0.weight"].grad.abs().sum()) == 0.0
    assert float(named["model.1.conv.weight"].grad.abs().sum()) > 0


def test_sgd_step_matches_torch_optim():
    """myolo_sgd_step == torch.optim.SGD(momentum, nesterov=True) with the reference's three parameter groups (train.py:108-126),
    including unscale, overflow skip and zero_grad; fp32 tolerance 1e-6 relative."""
    import ctypes as C
    from multiyolov5_b200 import _lib
    L = _lib.lib()
    n = 100003
    g = torch.Generator(device="cuda").manual_seed(3)
    p = torch.randn(n, device="cuda", generator=g)
    grad = torch.randn(n, device="cuda", generator=g) * 64.0
    group = torch.randint(0, 3, (n,), device="cuda", generator=g).to(torch.uint8)
    lr, wd, mom = [0.01, 0.02, 0.03], [0.0, 5e-4, 0.0], 0.937
    ref_p = [p[group == k].clone().requires_grad_(True) for k in range(3)]
    opt = torch.optim.SGD([{"params": [ref_p[k]], "lr": lr[k], "weight_decay": wd[k]} for k in range(3)], lr=0.1, momentum=mom, nesterov=True)
    buf = torch.zeros_like(p)
    inv = torch.full((), 1.0 / 64.0, device="cuda")
    found = torch.zeros(1, dtype=torch.int32, device="cuda")
    sp = _lib.stream_ptr()
    for it in range(3):
        gi = grad * (it + 1)
        for k in range(3):
            ref_p[k].grad = (gi[group == k] / 64.0).clone()
        opt.step()
        gg = gi.clone()
        _lib.check(L.myolo_grads_check_finite(_lib.ptr(gg), n, _lib.ptr(found), sp))
        _lib.check(L.myolo_sgd_step(_lib.ptr(p), _lib.ptr(gg), _lib.ptr(buf), _lib.ptr(group), n, (C.c_float * 3)(*lr), (C.c_float * 3)(*wd), 3,
                                    mom, 1, _lib.ptr(inv), _lib.ptr(found), 1, sp))
        assert int(found) == 0 and float(gg.abs().sum()) == 0.0
        for k in range(3):
            assert rel_f(p[group == k].cpu(), ref_p[k].detach().cpu()) < 1e-6
    # overflow: the step is skipped, gradients still cleared
    before = p.clone()
    gg = grad.clone(); gg[12345] = float("inf")
    _lib.check(L.myolo_grads_check_finite(_lib.ptr(gg), n, _lib.ptr(found), sp))
    _lib.check(L.myolo_sgd_step(_lib.ptr(p), _lib.ptr(gg), _lib.ptr(buf), _lib.ptr(group), n, (C.c_float * 3)(*lr), (C.c_float * 3)(*wd), 3,
                                mom, 1, _lib.ptr(inv), _lib.ptr(found), 1, sp))
    assert int(found) == 1 and torch.equal(p, before) and float(gg.abs().sum()) == 0.0


def test_trainer_overfits_a_fixed_batch():
    """end to end: det pass + seg pass + optimiser (reference train.py:363-401) on one fixed synthetic batch; the loss must fall and
    the loss scale must settle (no persistent overflow)."""
    from multiyolov5_b200.train import Trainer, scale_hyp
    import yaml, os
    model, cfg, sd, _ = setup(B=2, H=128, W=256)
    hyp = dict(lr0=0.01, momentum=0.937, weight_decay=5e-4, box=0.05, cls=0.5, cls_pw=1.0, obj=1.0, obj_pw=1.0, anchor_t=4.0, fl_gamma=0.0)
    hyp = scale_hyp(hyp, nl=3, nc=cfg["nc"], imgsz=256, total_batch_size=4)
    B = 2
    tr = Trainer(model, hyp, batch_size=B, init_scale=2.0 ** 10)
    rs = np.random.RandomState(0)
    imgs = synth.synth_image(B, 128, 256, seed=1).cuda()
    segimgs = synth.synth_image(B, 128, 256, seed=2).cuda()
    t = np.zeros((12, 6), np.float32)
    t[:, 0] = rs.randint(0, B, 12); t[:, 1] = rs.randint(0, cfg["nc"], 12)
    t[:, 2:4] = rs.uniform(0.1, 0.9, (12, 2)); t[:, 4:6] = rs.uniform(0.05, 0.4, (12, 2))
    targets = torch.from_numpy(t).cuda()
    mask = torch.from_numpy(rs.randint(-1, 19, (B, 1, 16, 32)).astype(np.int64)).cuda()
    mask = mask.repeat_interleave(8, 2).repeat_interleave(8, 3)[:, 0].contiguous()     # blocky labels: learnable
    hist = []
    for it in range(40):
        items, segloss = tr.step(imgs, targets, segimgs, mask)
        hist.append((float(items[3]), float(segloss)))
    print("\nloss history (det, seg): first %s last %s scale %.0f" % (hist[0], hist[-1], float(tr.scale)))
    assert all(np.isfinite(h).all() for h in hist)
    assert hist[-1][0] < 0.8 * hist[0][0] and hist[-1][1] < 0.8 * hist[0][1], (hist[0], hist[-1])
    assert float(tr.scale) >= 1.0


WGRAD_SHAPES = [  # B, H, W, ci, co, k, stride, dil
    (2, 32, 64, 64, 64, 1, 1, 1), (2, 32, 64, 128, 256, 1, 1, 1), (1, 64, 128, 64, 128, 3, 1, 1), (2, 32, 32, 128, 64, 3, 1, 1),
    (2, 64, 64, 64, 128, 3, 2, 1), (1, 32, 64, 64, 64, 3, 1, 2), (1, 32, 64, 192, 48, 1, 1, 1), (2, 16, 128, 256, 256, 3, 1, 1),
    (1, 48, 80, 64, 96, 3, 1, 3), (2, 64, 128, 32, 64, 3, 2, 1), (1, 64, 128, 32, 32, 3, 1, 1), (1, 64, 64, 16, 32, 3, 1, 1),
    (2, 32, 64, 32, 32, 1, 1, 1),
]


@pytest.mark.parametrize("path", [0, 1])
@pytest.mark.parametrize("shape", WGRAD_SHAPES, ids=[f"w{i}" for i in range(len(WGRAD_SHAPES))])
def test_conv_wgrad_kernels_match_torch(shape, path):
    """per-op: dW of one conv from fp16 NHWC x / dy, both kernels (0: mma.sync, 1: wgmma MN-major) against torch's conv weight
    gradient in fp64 on the same fp16-rounded inputs; tolerance 2e-3 relative Frobenius (fp32 accumulation order only)."""
    from multiyolov5_b200 import _lib
    B, H, W, ci, co, k, stride, dil = shape
    g = torch.Generator().manual_seed(sum(shape))
    x = torch.randn((B, ci, H, W), generator=g).half()
    pad = dil * (k // 2)
    Ho = (H + 2 * pad - dil * (k - 1) - 1) // stride + 1
    Wo = (W + 2 * pad - dil * (k - 1) - 1) // stride + 1
    dy = torch.randn((B, co, Ho, Wo), generator=g).half()
    w = torch.zeros((co, ci, k, k), dtype=torch.float64, requires_grad=True)
    y = torch.nn.functional.conv2d(x.double(), w, None, stride, pad, dil)
    (y * dy.double()).sum().backward()
    xd = x.permute(0, 2, 3, 1).contiguous().cuda()
    dyd = dy.permute(0, 2, 3, 1).contiguous().cuda()
    dW = torch.ones((co, ci, k, k), dtype=torch.float32, device="cuda")       # accumulate-into semantics: starts at 1
    _lib.check(_lib.lib().myolo_conv_wgrad(_lib.ptr(xd), _lib.ptr(dyd), B, H, W, ci, co, k, stride, dil, _lib.ptr(dW), path, _lib.stream_ptr()))
    torch.cuda.synchronize()
    err = rel_f((dW - 1.0).cpu(), w.grad)
    assert err < 2e-3, err


def test_graphed_det_loss_equals_eager_path():
    """Trainer(graph_loss=True) replays ComputeLoss forward+backward as one CUDA graph on static buffers, targets zero-padded to a
    multiple of 64 rows.  On identical head outputs the replayed graph must give the eager loss items and d loss / d head outputs
    (same torch kernels: 1e-6), for several target counts incl. none; and the det pass must leave the seg head untouched."""
    from multiyolov5_b200.train import Trainer, scale_hyp
    model, cfg, sd, _ = setup(B=2, H=128, W=256)
    hyp = dict(lr0=0.01, momentum=0.937, weight_decay=5e-4, box=0.05, cls=0.5, cls_pw=1.0, obj=1.0, obj_pw=1.0, anchor_t=4.0, fl_gamma=0.0)
    hyp = scale_hyp(hyp, nl=3, nc=cfg["nc"], imgsz=256, total_batch_size=4)
    tr = Trainer(model, hyp, batch_size=2, init_scale=64.0, graph_loss=True)
    shapes = [(2, 3, 16, 32, 15), (2, 3, 8, 16, 15), (2, 3, 4, 8, 15)]
    st = tr._det_graph(shapes, 64, torch.device("cuda"))
    rs = np.random.RandomState(0)
    gen = torch.Generator(device="cuda").manual_seed(4)
    for nt in (9, 0, 64, 9):
        ps = [torch.randn(sh, device="cuda", generator=gen) for sh in shapes]
        t = np.zeros((nt, 6), np.float32)
        if nt:
            t[:, 0] = rs.randint(0, 2, nt); t[:, 1] = rs.randint(0, cfg["nc"], nt)
            t[:, 2:4] = rs.uniform(0.05, 0.95, (nt, 2)); t[:, 4:6] = rs.uniform(0.03, 0.5, (nt, 2))
        tt = torch.from_numpy(t).cuda()
        with torch.no_grad():
            for q, v in zip(st.p, ps):
                q.copy_(v)
            st.t.zero_()
            if nt:
                st.t[:nt].copy_(tt)
        st.graph.replay()
        pe = [v.clone().requires_grad_(True) for v in ps]
        loss, items = tr._det_loss_scaled(pe, tt)
        loss.backward()
        torch.cuda.synchronize()
        assert torch.allclose(st.items, items, rtol=1e-6, atol=1e-7), (nt, st.items, items)
        for q, e in zip(st.p, pe):
            assert rel_f(q.grad.cpu(), e.grad.cpu()) < 1e-6, nt
    # end to end through the network: second call replays the captured graphs (network and loss)
    imgs = synth.synth_image(2, 128, 256, seed=1).cuda()
    for _ in range(2):
        model.zero_grad(set_to_none=False)
        items = tr.backward_det(imgs, tt)
    torch.cuda.synchronize()
    named = dict(model.named_parameters())
    assert torch.isfinite(items).all() and float(named["model.25.m.0.weight"].grad.abs().sum()) > 0
    assert float(named["model.24.out.3.weight"].grad.abs().sum()) == 0.0      # det pass leaves the seg head untouched


def test_fused_seg_ce_matches_torch_on_the_same_logits():
    """SURVEY 8f-3: CE(ignore -1) of the x8 bilinear upsample, forward + backward from the low-resolution logits in one kernel.  On the
    SAME low-res logits torch gives (interpolate -> cross_entropy -> autograd): loss to 1e-5, d loss / d logits to 1e-4 relative."""
    from multiyolov5_b200 import _lib
    model, cfg, sd, x = setup(B=2, H=128, W=256)
    eng = model.engine()
    rs = np.random.RandomState(5)
    labels = torch.from_numpy(rs.randint(-1, 19, (2, 128, 256)).astype(np.int64)).cuda()
    labels[0, :40] = -1                                               # a block of ignored pixels
    for it in range(3):                                               # eager, warm, graph replay
        model.zero_grad(set_to_none=False)
        _, _, plan = eng.train_forward(x.cuda(), want_seg=False)
        scale = torch.full((), 8.0, device="cuda")
        loss = eng.train_backward_seg_ce(plan, labels, factor=0.5, scale=scale)
        v = [o.in_ for o in plan.pb.ops if o.kind == _lib.OP_SEG_UPSAMPLE][0]
        lo = eng.read_view(v, plan).clone().requires_grad_(True)
        dlo = eng.read_grad_view(v, plan)
        up = torch.nn.functional.interpolate(lo[:, :19], (128, 256), mode="bilinear", align_corners=True)
        ref = torch.nn.functional.cross_entropy(up, labels, ignore_index=-1)
        (ref * 0.5 * 8.0).backward()
        torch.cuda.synchronize()
        assert abs(float(loss) - float(ref)) < 1e-5 * max(1.0, abs(float(ref))), (it, float(loss), float(ref))
        assert rel_f(dlo[:, :19].cpu(), lo.grad[:, :19].cpu()) < 1e-4, it
        named = dict(model.named_parameters())
        assert float(named["model.24.out.3.weight"].grad.abs().sum()) > 0 and float(named["model.25.m.0.weight"].grad.abs().sum()) == 0.0
    # all labels ignored: zero loss, zero gradients, no NaN
    model.zero_grad(set_to_none=False)
    _, _, plan = eng.train_forward(x.cuda(), want_seg=False)
    loss = eng.train_backward_seg_ce(plan, torch.full_like(labels, -1))
    assert float(loss) == 0.0 and float(dict(model.named_parameters())["model.24.out.3.weight"].grad.abs().sum()) == 0.0


def test_trainer_bise_head_three_outputs():
    """BiSe in train mode returns [out, aux16, aux32]; the step uses SegmentationLosses(aux=True, aux_num=2) (reference train.py:387-388)"""
    from multiyolov5_b200.train import Trainer, scale_hyp
    model, cfg, sd, _ = setup("s_bise", "yolov5s_city_seg_bise.yaml", B=2, H=128, W=256)
    hyp = dict(lr0=0.01, momentum=0.937, weight_decay=5e-4, box=0.05, cls=0.5, cls_pw=1.0, obj=1.0, obj_pw=1.0, anchor_t=4.0, fl_gamma=0.0)
    tr = Trainer(model, scale_hyp(hyp, nl=3, nc=cfg["nc"], imgsz=256, total_batch_size=4), batch_size=2, init_scale=2.0 ** 10)
    assert tr.n_seg_outputs == 3
    rs = np.random.RandomState(0)
    imgs = synth.synth_image(2, 128, 256, seed=1).cuda()
    t = np.zeros((6, 6), np.float32)
    t[:, 0] = rs.randint(0, 2, 6); t[:, 1] = rs.randint(0, cfg["nc"], 6)
    t[:, 2:4] = rs.uniform(0.1, 0.9, (6, 2)); t[:, 4:6] = rs.uniform(0.05, 0.4, (6, 2))
    mask = torch.from_numpy(rs.randint(-1, 19, (2, 1, 16, 32)).astype(np.int64)).cuda().repeat_interleave(8, 2).repeat_interleave(8, 3)[:, 0].contiguous()
    hist = [tr.step(imgs, torch.from_numpy(t).cuda(), imgs, mask) for _ in range(25)]
    first, last = float(hist[0][1]), float(hist[-1][1])
    assert np.isfinite([float(h[1]) for h in hist]).all() and last < 0.85 * first, (first, last)
    named = dict(model.named_parameters())
    assert float(named["model.24.aux16.1.weight"].abs().sum()) > 0


def test_backward_of_a_stale_forward_is_refused():
    """one plan = one activation workspace per (B,H,W): forward, forward, backward would silently use the second forward's activations for
    the first output's gradients.  The engine counts train forwards per plan and refuses the stale backward (reference order is forward,
    backward, forward, backward - train.py:364-392)."""
    from multiyolov5_b200 import _lib
    model, cfg, sd, x = setup(B=2, H=64, W=128)
    xa, xb = x.cuda(), (x * 0.5).cuda()
    p1 = model(xa)
    p2 = model(xb)
    with pytest.raises(_lib.MyoloError, match="stale"):
        (p1[1].float().sum() + p2[1].float().sum()).backward()
    p3 = model(xa)                      # the regular order still works afterwards
    p3[1].float().sum().backward()
    torch.cuda.synchronize()
    g = model.model[0].conv.conv.weight.grad
    assert g is not None and torch.isfinite(g).all() and float(g.abs().sum()) > 0


def test_eval_after_train_forward_uses_updated_running_statistics():
    """a train-mode forward moves running_mean / running_var through raw pointers: the inference plans' BN-folded weights must be re-packed"""
    model, cfg, sd, x = setup(B=2, H=64, W=128)
    xc = x.cuda()
    model.eval()
    (z0, _), _ = model(xc)
    model.train()
    model(xc)
    model.eval()
    (z1, _), _ = model(xc)
    torch.cuda.synchronize()
    sd1 = {k: v.detach().cpu().clone() for k, v in model.state_dict().items()}
    fresh, _, _, _ = setup(B=2, H=64, W=128)
    fresh.load_state_dict(sd1)
    fresh.cuda().eval()
    (z2, _), _ = fresh(xc)
    torch.cuda.synchronize()
    assert not torch.equal(z0, z1)                                  # statistics moved ...
    assert torch.equal(z1, z2)                                      # ... and the cached inference plan saw them


@pytest.mark.parametrize("name", ["a", "empty", "edge"])
def test_fused_det_loss_matches_reference_fixture(name):
    """`myolo_det_loss` (csrc/detloss.cu: target assignment, CIoU / BCE losses and THEIR GRADIENTS in four launches) against the fixtures written
    by the unmodified reference's ComputeLoss + autograd (tests/golden/loss_cases.npz: loss items and d loss / d p_i)"""
    import json, os
    from multiyolov5_b200.models.yolo import Model
    from multiyolov5_b200.utils.loss import FusedComputeLoss
    g = np.load(os.path.join(synth.GOLDEN_DIR, "loss_cases.npz"))
    hyp = json.loads(bytes(g["hyp_json"]).decode())
    model = Model("yolov5s_city_seg.yaml")
    model.hyp, model.gr = hyp, 1.0
    crit = FusedComputeLoss(model)
    assert crit.supported
    p = [torch.from_numpy(g[f"{name}_p{i}"]).cuda().contiguous() for i in range(3)]
    grads, items = crit(p, torch.from_numpy(g[f"{name}_targets"]).cuda())
    torch.cuda.synchronize()
    assert np.allclose(items.cpu().numpy(), g[f"{name}_items"], rtol=2e-5, atol=1e-6), (items.cpu().numpy(), g[f"{name}_items"])
    for i in range(3):
        ref = g[f"{name}_g{i}"]
        err = np.abs(grads[i].cpu().numpy() - ref).max() / np.abs(ref).max()
        assert err <= 2e-5, (i, err)


def test_fused_det_loss_matches_torch_formulation_at_bench_shapes():
    """the shapes of the train step (4 x 3 x 64x128 / 32x64 / 16x32, 80 boxes with duplicate cells) incl. loss scale and multiplier"""
    from multiyolov5_b200.models.yolo import Model
    from multiyolov5_b200.train import scale_hyp
    from multiyolov5_b200.utils.loss import ComputeLoss, FusedComputeLoss
    model = Model("yolov5s_city_seg.yaml").cuda()
    hyp = dict(lr0=0.0015, momentum=0.937, weight_decay=5e-4, box=0.05, cls=0.5, cls_pw=1.0, obj=1.0, obj_pw=1.0, anchor_t=4.0, fl_gamma=0.0)
    model.hyp, model.gr = scale_hyp(hyp, nl=3, nc=10, imgsz=1024, total_batch_size=32), 1.0
    gen = torch.Generator(device="cuda").manual_seed(5)
    B = 4
    p = [torch.randn((B, 3, 512 // s, 1024 // s, 15), device="cuda", generator=gen).requires_grad_(True) for s in (8, 16, 32)]
    rs = np.random.RandomState(3)
    t = np.zeros((80 + 16, 6), np.float32)                       # 16 all-zero padding rows: never match
    t[:80, 0] = np.repeat(np.arange(B), 20); t[:80, 1] = rs.randint(0, 10, 80)
    t[:80, 2:4] = rs.uniform(0.1, 0.9, (80, 2)); t[:80, 4:6] = rs.uniform(0.02, 0.22, (80, 2))
    t[10:14, 2:6] = t[10, 2:6]                                   # identical boxes in one image: several candidates share cells
    t[10:14, 0] = t[10, 0]
    tg = torch.from_numpy(t).cuda()
    scale = torch.full((), 1024.0, device="cuda")
    loss, items = ComputeLoss(model)(p, tg)
    (loss * 8 * 0.6 * scale).backward()
    grads, fitems = FusedComputeLoss(model)([q.detach() for q in p], tg, mult=8 * 0.6, scale=scale)
    torch.cuda.synchronize()
    assert torch.allclose(fitems, items, rtol=2e-5, atol=1e-6), (fitems, items)
    for q, gq in zip(p, grads):
        err = float((gq - q.grad).abs().max() / q.grad.abs().max())
        assert err <= 5e-5, err


def test_grouped_weight_repack_equals_per_slot_packs(monkeypatch):
    """after an in-place parameter update every fp16 copy (forward packs and the flipped / transposed data-gradient packs) is rewritten by
    ONE launch (myolo_plan_repack_weights); the result must equal the per-slot pack kernels' (MYOLO_REPACK=0)"""
    from multiyolov5_b200 import _lib

    def two_steps(repack):
        monkeypatch.setenv("MYOLO_REPACK", "1" if repack else "0")
        model, cfg, sd, x = setup(B=2, H=128, W=256)
        xc = x.cuda()
        out = model(xc)
        (out[1].float().square().mean() + sum(r.float().square().mean() for r in out[0])).backward()
        with torch.no_grad():
            for i, p in enumerate(model.parameters()):
                p.mul_(1.0 + 0.01 * ((i % 5) - 2))           # in place: same tensors, new values
                p.grad.zero_()
        out = model(xc)
        (out[1].float().square().mean() + sum(r.float().square().mean() for r in out[0])).backward()
        torch.cuda.synchronize()
        return ([r.detach().float().cpu() for r in out[0]] + [out[1].detach().float().cpu()],
                {k: p.grad.detach().cpu().clone() for k, p in model.named_parameters()})

    o1, g1 = two_steps(True)
    o0, g0 = two_steps(False)
    o0b, g0b = two_steps(False)
    # batch statistics and parameter gradients are reduced with fp32 atomics and tiny maps (2x4 pixels at P5 here) amplify the summation
    # order: the yardstick is the run-to-run spread of the per-slot path itself; a wrong pack is an O(1) error
    noise_o = max(rel_f(a, b) for a, b in zip(o0b, o0))
    diff_o = max(rel_f(a, b) for a, b in zip(o1, o0))

    def gdiff(ga, gb):
        # median over the parameter tensors of the relative Frobenius difference: single ill-conditioned tensors (BatchNorm over a 2x4 map)
        # swing by tens of percent from run to run, a wrong data-gradient pack corrupts every gradient upstream of it
        return float(np.median([rel_f(ga[k], gb[k]) for k in gb]))
    noise_g, diff_g = gdiff(g0b, g0), gdiff(g1, g0)
    print(f"\nrepack vs per-slot: outputs {diff_o:.2e} (run-to-run {noise_o:.2e}), gradients (median rel.) {diff_g:.2e} (run-to-run {noise_g:.2e})")
    assert diff_o <= max(3 * noise_o, 1e-3), (diff_o, noise_o)
    assert diff_g <= max(3 * noise_g, 5e-3), (diff_g, noise_g)


def test_concurrent_forwards_keep_the_reference_order_of_running_statistics():
    """Trainer(concurrent_forwards=True) runs the seg forward next to the det forward; the seg plan defers its BatchNorm running-statistics
    update and applies it after the det forward.  running_mean / running_var / num_batches_tracked and the stepped parameters must equal
    the strictly sequential schedule's (reference train.py:364-398: det forward+backward, seg forward+backward, optimizer.step)."""
    from multiyolov5_b200.train import Trainer, scale_hyp
    B = 2
    rs = np.random.RandomState(0)
    imgs = synth.synth_image(B, 128, 256, seed=1).cuda()
    segimgs = synth.synth_image(B, 128, 256, seed=2).cuda()
    t = np.zeros((12, 6), np.float32)
    t[:, 0] = rs.randint(0, B, 12); t[:, 1] = rs.randint(0, 15, 12)
    t[:, 2:4] = rs.uniform(0.1, 0.9, (12, 2)); t[:, 4:6] = rs.uniform(0.05, 0.4, (12, 2))
    targets = torch.from_numpy(t).cuda()
    mask = torch.from_numpy(rs.randint(-1, 19, (B, 128, 256)).astype(np.int64)).cuda()

    def run(**kw):
        model, cfg, sd, _ = setup(B=B, H=128, W=256)
        hyp = dict(lr0=0.01, momentum=0.937, weight_decay=5e-4, box=0.05, cls=0.5, cls_pw=1.0, obj=1.0, obj_pw=1.0, anchor_t=4.0, fl_gamma=0.0)
        hyp = scale_hyp(hyp, nl=3, nc=cfg["nc"], imgsz=256, total_batch_size=4)
        tr = Trainer(model, hyp, batch_size=B, init_scale=2.0 ** 10, **kw)
        items, segloss = tr.step(imgs, targets, segimgs, mask)
        torch.cuda.synchronize()
        first = ({k: v.detach().float().cpu().clone() for k, v in model.state_dict().items() if "running_" in k or "num_batches" in k},
                 [float(v) for v in items])
        for _ in range(2):                                   # the schedule keeps working step after step
            items, segloss = tr.step(imgs, targets, segimgs, mask)
        torch.cuda.synchronize()
        nbt = [int(v) for k, v in model.state_dict().items() if k.endswith("num_batches_tracked")]
        assert all(np.isfinite(float(v)) for v in items) and np.isfinite(float(segloss))
        return first, nbt

    # compared after ONE step: from the second step on the two schedules legitimately differ (the seg pass draws its dropout masks from its
    # own plan's counter in the concurrent schedule), the first step's forward statistics do not depend on any mask
    (sa, la), na = run(concurrent_forwards=True)
    (sb, lb), nb = run(overlap_passes=False)
    (sc, lc), _ = run(overlap_passes=False)                  # run-to-run spread of the sequential schedule (fp32 atomics in the batch sums)
    assert set(na) == set(nb) == {6}, (set(na), set(nb))     # 3 steps x (det batch + seg batch)

    def spread(x, y):
        return max(float((x[k] - y[k]).abs().max()) / (float(y[k].abs().max()) + 1e-12) for k in y if "running_" in k)
    noise, diff = spread(sc, sb), spread(sa, sb)
    print(f"\nrunning statistics after one step, concurrent vs sequential: {diff:.2e} (sequential run to run: {noise:.2e})")
    for k in sb:
        if k.endswith("num_batches_tracked"):
            assert int(sa[k]) == int(sb[k]) == 2, k
    assert diff <= max(3 * noise, 1e-5), (diff, noise)
    assert max(abs(x - y) for x, y in zip(la, lb)) <= max(3 * max(abs(x - y) for x, y in zip(lc, lb)), 1e-4 * abs(lb[3])), (la, lb, lc)
