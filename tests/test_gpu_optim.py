"""GPU: the reference's --adam (myolo_adam_step, Trainer(optimizer="adam")) bit for bit against torch.optim.Adam behind torch.amp.GradScaler,
and the optimiser state in torch's format (Trainer.state_dict / load_state_dict): resume, and the state of a torch optimizer built as the
reference builds it, in both directions."""
import ctypes as C
import io

import numpy as np
import pytest
import torch

from oracle import synth

pytestmark = pytest.mark.gpu
BETAS = (0.937, 0.999)


def adam_launch(p, g, m, v, group, lr, wd, steps, inv, found, betas=BETAS):
    from multiyolov5_b200 import _lib
    _lib.check(_lib.lib().myolo_adam_step(_lib.ptr(p), _lib.ptr(g), _lib.ptr(m), _lib.ptr(v), _lib.ptr(group), p.numel(),
                                          (C.c_double * 3)(*lr), (C.c_float * 3)(*wd), 3, betas[0], betas[1], 1e-8, _lib.ptr(steps),
                                          _lib.ptr(inv), _lib.ptr(found), 1, _lib.stream_ptr()))


def check_finite(g, found):
    from multiyolov5_b200 import _lib
    _lib.check(_lib.lib().myolo_grads_check_finite(_lib.ptr(g), g.numel(), _lib.ptr(found), _lib.stream_ptr()))


@pytest.mark.parametrize("betas", [BETAS, (0.3, 0.99)], ids=["hyp", "beta1_below_half"])
def test_adam_step_is_bit_identical_to_torch_adam_with_grad_scaler(betas):
    """n odd (a tail after the float4 body), three interleaved groups with their own lr and weight decay, lr changing every step as in
    warm-up (doubles that fp32 does not hold), loss scale 2^6: after every step parameters, exp_avg and exp_avg_sq equal torch's bit for
    bit.  A step with an inf gradient moves nothing, clears the gradients and does not advance the step count; GradScaler then halves its
    scale and the steps after it match again.  beta1 = 0.3 makes the lerp weight 1 - beta1 >= 0.5: torch's lerp takes its other branch."""
    n = 100003
    gen = torch.Generator(device="cuda").manual_seed(11)
    p = torch.randn(n, device="cuda", generator=gen)
    group = torch.randint(0, 3, (n,), device="cuda", generator=gen).to(torch.uint8)
    wd = [0.0, 5e-4, 1e-2]
    ref_p = [p[group == k].clone().requires_grad_(True) for k in range(3)]
    opt = torch.optim.Adam([{"params": [ref_p[k]], "weight_decay": wd[k]} for k in range(3)], lr=0.01, betas=betas)
    scaler = torch.amp.GradScaler("cuda", init_scale=64.0, growth_interval=1000)
    scaler.scale(torch.ones((), device="cuda"))                                   # creates the scaler's scale tensor
    m, v = torch.zeros_like(p), torch.zeros_like(p)
    steps = torch.zeros((), dtype=torch.int32, device="cuda")
    found = torch.zeros(1, dtype=torch.int32, device="cuda")
    for it in range(9):
        lr = [0.01 * (it + 1) / 7.0, 0.013 * (it + 2) / 9.0, 0.1 - 0.09 * it / 11.0]
        for k in range(3):
            opt.param_groups[k]["lr"] = lr[k]
        s = scaler.get_scale()
        g = torch.randn(n, device="cuda", generator=gen) * (0.1 * s * (it + 1))
        g[::97] = 0.0                                                            # exact zero gradients
        if it == 4:
            g[4321] = float("inf")
        for k in range(3):
            ref_p[k].grad = g[group == k].clone()
        before = [t.clone() for t in (p, m, v)]
        scaler.step(opt)
        scaler.update()
        gg = g.clone()
        inv = torch.full((), 1.0 / s, device="cuda")
        check_finite(gg, found)
        adam_launch(p, gg, m, v, group, lr, wd, steps, inv, found, betas)
        steps += (found[0] == 0).to(torch.int32)
        assert float(gg.abs().sum()) == 0.0
        if it == 4:
            assert int(found) == 1 and all(torch.equal(a, b) for a, b in zip((p, m, v), before))
            assert int(steps) == 4 and int(opt.state[ref_p[0]]["step"]) == 4
        else:
            assert int(found) == 0
        for k in range(3):
            st = opt.state[ref_p[k]]
            assert int(st["step"]) == int(steps)
            sel = group == k
            for mine, ref, name in ((p, ref_p[k].detach(), "param"), (m, st["exp_avg"], "exp_avg"), (v, st["exp_avg_sq"], "exp_avg_sq")):
                d = (mine[sel] != ref).sum()
                assert int(d) == 0, f"step {it} group {k} {name}: {int(d)} elements differ"


@pytest.mark.parametrize("lr", [0.01, 0.001, 0.0123456789012345])
def test_bias_corrections_equal_pythons_up_to_a_million_steps(lr):
    """for every step count k = 1 .. 10^6 the device's double bias corrections 1 - beta^k equal Python's bit for bit (CUDA's pow against
    glibc's, at the hyp betas), so every lr gives torch's scalars: (lr / bc1) * -1 and bc2 ** 0.5 are correctly rounded in both.  The fp32
    step size and bc2_sqrt are compared as well, at three lr values."""
    from multiyolov5_b200 import _lib
    K = 10 ** 6
    ks = torch.arange(1, K + 1, dtype=torch.int32, device="cuda")
    ss, bs = torch.empty(K, device="cuda"), torch.empty(K, device="cuda")
    bc1, bc2 = torch.empty(K, dtype=torch.float64, device="cuda"), torch.empty(K, dtype=torch.float64, device="cuda")
    _lib.check(_lib.lib().myolo_adam_scalars(_lib.ptr(ks), K, lr, BETAS[0], BETAS[1], _lib.ptr(ss), _lib.ptr(bs), _lib.ptr(bc1), _lib.ptr(bc2),
                                             _lib.stream_ptr()))
    b1, b2 = BETAS
    ref_bc1 = np.array([1 - b1 ** float(k) for k in range(1, K + 1)], np.float64)
    ref_bc2 = np.array([1 - b2 ** float(k) for k in range(1, K + 1)], np.float64)
    d1 = np.flatnonzero(bc1.cpu().numpy().view(np.int64) != ref_bc1.view(np.int64))
    d2 = np.flatnonzero(bc2.cpu().numpy().view(np.int64) != ref_bc2.view(np.int64))
    assert d1.size == 0 and d2.size == 0, (d1.size, d1[:10] + 1, d2.size, d2[:10] + 1)
    ref_ss = np.array([(lr / (1 - b1 ** float(k))) * -1 for k in range(1, K + 1)], np.float64).astype(np.float32)
    ref_bs = np.array([(1 - b2 ** float(k)) ** 0.5 for k in range(1, K + 1)], np.float64).astype(np.float32)
    d_ss = np.flatnonzero(ss.cpu().numpy() != ref_ss)
    d_bs = np.flatnonzero(bs.cpu().numpy() != ref_bs)
    assert d_ss.size == 0 and d_bs.size == 0, (d_ss[:10] + 1, d_bs[:10] + 1)


def make_trainer(optimizer, seed=1, **kw):
    from multiyolov5_b200.models.yolo import Model
    from multiyolov5_b200.train import Trainer, scale_hyp
    yml = "yolov5s_city_seg.yaml"
    cfg = synth.load_cfg(yml)
    sd = synth.synth_state_dict(synth.load_manifest("s_psp"), cfg, seed=seed, gain=1.0)
    model = Model(yml)
    model.load_state_dict(sd)
    model.cuda().train()
    hyp = dict(lr0=0.01, momentum=0.937, weight_decay=5e-4, box=0.05, cls=0.5, cls_pw=1.0, obj=1.0, obj_pw=1.0, anchor_t=4.0, fl_gamma=0.0)
    hyp = scale_hyp(hyp, nl=3, nc=cfg["nc"], imgsz=256, total_batch_size=4)
    return Trainer(model, hyp, batch_size=2, init_scale=2.0 ** 10, optimizer=optimizer, **kw), cfg


def batch(cfg, B=2, seed=0):
    rs = np.random.RandomState(seed)
    imgs = synth.synth_image(B, 128, 256, seed=seed + 1).cuda()
    segimgs = synth.synth_image(B, 128, 256, seed=seed + 2).cuda()
    t = np.zeros((12, 6), np.float32)
    t[:, 0] = rs.randint(0, B, 12); t[:, 1] = rs.randint(0, cfg["nc"], 12)
    t[:, 2:4] = rs.uniform(0.1, 0.9, (12, 2)); t[:, 4:6] = rs.uniform(0.05, 0.4, (12, 2))
    mask = torch.from_numpy(rs.randint(-1, 19, (B, 1, 16, 32)).astype(np.int64)).cuda()
    mask = mask.repeat_interleave(8, 2).repeat_interleave(8, 3)[:, 0].contiguous()
    return imgs, torch.from_numpy(t).cuda(), segimgs, mask


def torch_adam_like(tr):
    """torch.optim.Adam + GradScaler over copies of the trainer's parameters, grouped as the reference groups them"""
    from multiyolov5_b200.train import reference_param_groups
    pgs = reference_param_groups(tr.model)
    copies = [[p.detach().clone().requires_grad_(True) for p in pg] for pg in pgs]
    opt = torch.optim.Adam([{"params": c, "lr": tr.lr[k], "weight_decay": tr.wd[k]} for k, c in enumerate(copies)], lr=0.01,
                           betas=tr.betas, eps=tr.eps)
    scaler = torch.amp.GradScaler("cuda", init_scale=float(tr.scale), growth_interval=tr.growth_interval)
    scaler.scale(torch.ones((), device="cuda"))
    return pgs, copies, opt, scaler


def test_trainer_adam_step_equals_torch_adam_on_the_trainers_gradient():
    """Trainer(optimizer="adam", accumulate=2) on s/PSP at 2x128x256: the first step() leaves the flat gradient of the det + seg passes
    (scaled) in place; torch's Adam + GradScaler applied to that gradient gives the parameters the trainer's optimizer_step gives, bit for
    bit, over two steps with the lr changed in between (set_lr)"""
    tr, cfg = make_trainer("adam", accumulate=2)
    pgs, copies, opt, scaler = torch_adam_like(tr)
    with pytest.raises(ValueError):
        tr.set_momentum(0.8)
    for it in range(2):
        if it:
            tr.set_lr(0.002, 0.003, 0.05)
            for k in range(3):
                opt.param_groups[k]["lr"] = tr.lr[k]
        tr.step(*batch(cfg, seed=it))                                           # ni odd: backward only
        assert tr.ni % 2 == 1
        for pg, cg in zip(pgs, copies):
            for p, c in zip(pg, cg):
                c.grad = p.grad.detach().clone()
        assert float(tr.flat.grad.abs().sum()) > 0
        tr.ni += 1
        tr.optimizer_step()
        scaler.step(opt)
        scaler.update()
        assert int(tr.found_inf) == 0 and int(tr.steps) == it + 1
        for pg, cg in zip(pgs, copies):
            for p, c in zip(pg, cg):
                assert torch.equal(p.detach(), c.detach())
                st = opt.state[c]
                o = (p.data_ptr() - tr.flat.param.data_ptr()) // 4
                assert torch.equal(tr.flat.momentum[o:o + p.numel()].view_as(p), st["exp_avg"])
                assert torch.equal(tr.flat.exp_avg_sq[o:o + p.numel()].view_as(p), st["exp_avg_sq"])


def same(a, b, path="sd"):
    """equal values AND types, recursively; tensors equal in dtype, shape, device and every bit"""
    assert type(a) is type(b), (path, type(a), type(b))
    if isinstance(a, torch.Tensor):
        assert a.dtype == b.dtype and a.shape == b.shape and a.device == b.device and torch.equal(a, b), path
    elif isinstance(a, dict):
        assert list(a.keys()) == list(b.keys()), (path, list(a.keys()), list(b.keys()))
        for k in a:
            same(a[k], b[k], f"{path}[{k!r}]")
    elif isinstance(a, (list, tuple)):
        assert len(a) == len(b), path
        for i, (x, y) in enumerate(zip(a, b)):
            same(x, y, f"{path}[{i}]")
    else:
        assert a == b, (path, a, b)


@pytest.mark.parametrize("optimizer", ["sgd", "adam"])
def test_resume_restores_the_optimizer_state_bit_for_bit(optimizer):
    """train three steps, torch.save the state_dict, build a fresh model + Trainer from the saved model weights and load it: the flat
    optimiser buffers and the step count equal the originals, state_dict() returns the loaded dict, and one optimizer_step on the same
    fixed gradient gives identical parameters in both trainers.  (Whole train steps are not compared: the parameter gradients are
    accumulated atomically, so two runs of a step differ in the last bits.)"""
    tr, cfg = make_trainer(optimizer)
    assert tr.state_dict()["state"] == {}                                      # torch has no state before the first step
    for it in range(3):
        tr.step(*batch(cfg, seed=it))
    tr.set_lr(0.004, 0.005, 0.03)
    buf = io.BytesIO()
    torch.save({"model": tr.model.state_dict(), "optimizer": tr.state_dict()}, buf)
    buf.seek(0)
    ck = torch.load(buf, map_location="cpu")
    sd = ck["optimizer"]
    assert len(sd["state"]) == sum(1 for p in tr.model.parameters()) == 229
    tr2, _ = make_trainer(optimizer, seed=7)
    tr2.model.load_state_dict(ck["model"])         # copies into the parameters, i.e. into the flat buffer they view
    tr2.load_state_dict(sd)
    assert torch.equal(tr2.flat.param, tr.flat.param) and tr2.lr == tr.lr and int(tr.steps) == 3
    # torch's SGD state has no step count: a loaded SGD trainer only knows that state exists
    assert int(tr2.steps) == (3 if optimizer == "adam" else 1)
    for name, b in tr._state_buffers().items():
        assert torch.equal(tr2._state_buffers()[name], b), name
    back = tr2.state_dict()                        # CUDA state tensors, as torch's own optimizer over CUDA parameters keeps them
    same(back, {"state": {i: {k: t if k == "step" else t.cuda() for k, t in st.items()} for i, st in sd["state"].items()},
                "param_groups": sd["param_groups"]})
    tr2.scale.copy_(tr.scale)                     # the loss scale is not part of the optimiser state
    g = torch.randn(tr.flat.n, device="cuda", generator=torch.Generator(device="cuda").manual_seed(5)) * float(tr.scale) * 1e-3
    for t in (tr, tr2):
        t.flat.grad.copy_(g)
        t.optimizer_step()
    assert torch.equal(tr.flat.param, tr2.flat.param)
    for name, b in tr._state_buffers().items():
        assert torch.equal(tr2._state_buffers()[name], b), name


def reference_optimizer(optimizer, model, hyp):
    """torch's optimizer over `model` built as reference train.py:119-137 and :145 build it (groups, betas / nesterov, LambdaLR's
    initial_lr)"""
    from multiyolov5_b200.train import reference_param_groups
    pg0, pg1, pg2 = reference_param_groups(model)
    if optimizer == "adam":
        opt = torch.optim.Adam(pg0, lr=hyp["lr0"], betas=(hyp["momentum"], 0.999))
    else:
        opt = torch.optim.SGD(pg0, lr=hyp["lr0"], momentum=hyp["momentum"], nesterov=True)
    opt.add_param_group({"params": pg1, "weight_decay": hyp["weight_decay"]})
    opt.add_param_group({"params": pg2})
    torch.optim.lr_scheduler.LambdaLR(opt, lr_lambda=lambda x: 1.0)
    return opt


@pytest.mark.parametrize("optimizer", ["sgd", "adam"])
def test_torch_optimizer_state_continues_here_and_back(optimizer):
    """a torch optimizer built as the reference builds it takes three steps (warm-up lr and momentum) on a copy of the model; its
    state_dict() loads into a Trainer, whose state_dict() returns it, and one step on a fixed gradient in both gives the same parameters
    (Adam: bit for bit; SGD: myolo_sgd_step, bounded as tests/test_gpu_train.py bounds it).  The trainer's dict then loads back into the
    torch optimizer, which takes a second step equal to the trainer's."""
    import copy
    tr, cfg = make_trainer(optimizer)
    ref_model = copy.deepcopy(tr.model)
    opt = reference_optimizer(optimizer, ref_model, tr.hyp)
    params = [p for p in ref_model.parameters()]
    gen = torch.Generator(device="cuda").manual_seed(4)
    for it in range(3):
        for j, x in enumerate(opt.param_groups):
            x["lr"] = float(np.interp(it, [0, 10], [0.1 if j == 2 else 0.0, 0.01]))
            if "momentum" in x:
                x["momentum"] = np.interp(it, [0, 10], [0.8, 0.937])
        for p in params:
            p.grad = torch.randn(p.shape, device="cuda", generator=gen) * 1e-2
        opt.step()
    sd = copy.deepcopy(opt.state_dict())
    tr.model.load_state_dict(ref_model.state_dict())
    tr.load_state_dict(sd)
    same(tr.state_dict(), sd)
    scaler = torch.amp.GradScaler("cuda", init_scale=float(tr.scale))
    scaler.scale(torch.ones((), device="cuda"))
    for rnd in range(2):
        if rnd:
            opt.load_state_dict(tr.state_dict())
        g = torch.randn(tr.flat.n, device="cuda", generator=gen) * float(tr.scale) * 1e-2
        tr.flat.grad.copy_(g)
        for p, q in zip(tr.model.parameters(), params):
            q.grad = p.grad.detach().clone()
        tr.optimizer_step()
        scaler.step(opt)
        scaler.update()
        for p, q in zip(tr.model.parameters(), params):
            if optimizer == "adam":
                assert torch.equal(p.detach(), q.detach())
            else:
                assert float((p.detach() - q.detach()).abs().max()) <= 1e-6 * max(float(q.detach().abs().max()), 1e-6)
