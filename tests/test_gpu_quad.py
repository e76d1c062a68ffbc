"""GPU: `--quad` batches built on the device (DetAugmenter / DetRectLoader + collate_quad) against the reference's own batches
(tests/golden/quad_cases.npz) and against the numpy restatement (oracle/restate_quad.py) at full size, bit exact; quads independent of
their neighbours on both kernel paths; and Trainer(quad=True): finite steps, the x4 det loss of the fused loss against the torch
formulation, and quad with multi_scale and det_shapes on one reserved workspace."""
import json
import os
import random

import numpy as np
import pytest
import torch

from oracle import restate_quad as rq
from oracle import synth
from tests.test_gpu_multiscale import HYP, _model

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden")
CASES = ["mosaic", "mixup", "rect"]


def _golden():
    g = np.load(os.path.join(GOLD, "quad_cases.npz"))
    return g, json.loads(bytes(g["meta_json"]).decode())


def _state(g, name, b):
    r = random.Random()
    r.setstate((3, tuple(int(v) for v in g[f"{name}_state_{b}"]), None))
    return r


class _Draws:
    """an rng whose random() returns the given values"""

    def __init__(self, values):
        self.values = list(values)

    def random(self):
        return self.values.pop(0)


@pytest.mark.parametrize("name", CASES)
def test_device_batches_match_reference_fixtures(name):
    from multiyolov5_b200.utils.datasets import DetAugmenter, DetRectLoader, DeviceImageCache, collate_quad
    g, meta = _golden()
    c = meta["cases"][name]
    n = len(meta["shapes"])
    cache = DeviceImageCache([g[f"src_{k}"] for k in range(n)], c["img_size"], [g[f"labels_{k}"] for k in range(n)])
    if c["rect"]:
        loader = DetRectLoader(cache, c["hyp"], c["batch_size"])
        assert np.array_equal(loader.order, g[f"{name}_order"]) and np.array_equal(loader.batch_shapes, g[f"{name}_batch_shapes"])
    else:
        loader = DetAugmenter(cache, c["hyp"])
    random.seed(c["seed"])
    np.random.seed(c["seed"])
    for b in range(c["n_batches"]):
        imgs, targets = loader(range(8 * b, min(8 * b + 8, n)))
        assert torch.equal(imgs.cpu(), torch.from_numpy(g[f"{name}_items_{b}"])), (name, b)
        assert np.array_equal(targets.cpu().numpy(), g[f"{name}_targets_{b}"]), (name, b)
        img4, t4 = collate_quad(imgs, targets)
        ref = g[f"{name}_img4_{b}"]
        assert img4.dtype == torch.uint8 and t4.dtype == torch.float32 and img4.is_cuda and t4.is_cuda
        got = img4.cpu().numpy()
        assert got.shape == ref.shape and np.array_equal(got, ref), (name, b, int((got != ref).sum()) if got.shape == ref.shape else got.shape)
        assert np.array_equal(t4.cpu().numpy(), g[f"{name}_targets4_{b}"]), (name, b)
        st, nst = random.getstate(), np.random.get_state()          # peek at the next draws, then go on from where the reference did
        assert random.random() == c["next_random"][b] and float(np.random.random()) == c["next_np"][b], (name, b)
        random.setstate(st)
        np.random.set_state(nst)
        for dtype in (torch.float16, torch.float32):
            f4, ft4 = collate_quad(imgs, targets, rng=_state(g, name, b), out_dtype=dtype)
            want = img4.to(dtype) / 255.0 if dtype == torch.float16 else img4.float() / 255.0
            assert f4.dtype == dtype and torch.equal(f4, want), (name, b, dtype)
            assert torch.equal(ft4, t4)
    assert any(sum(c["tiles"], [])) and not all(sum(c["tiles"], []))


def _frames(rs, shapes):
    imgs, labels = [], []
    for h, w in shapes:
        yy, xx = np.mgrid[0:h, 0:w]
        base = np.stack([xx * 255 // w, yy * 255 // h, (xx ^ yy) & 255], -1)
        imgs.append(np.clip(base + rs.randint(-40, 41, (h, w, 3)), 0, 255).astype(np.uint8))
        m = rs.randint(1, 6)
        lb = np.zeros((m, 5), np.float32)
        lb[:, 0] = rs.randint(0, 10, m)
        lb[:, 3:5] = rs.uniform(0.05, 0.4, (m, 2))
        lb[:, 1:3] = rs.uniform(0.2, 0.8, (m, 2))
        labels.append(lb)
    return imgs, labels


def _scratch():
    return dict(hsv_h=0.015, hsv_s=0.7, hsv_v=0.4, degrees=5.0, translate=0.1, scale=0.5, shear=2.0, perspective=0.0, flipud=0.5,
                fliplr=0.5, mosaic=1.0, mixup=0.3)


def test_full_size_cityscapes_batches_equal_restatement():
    """16 Cityscapes-shaped items at imgsz 1024: mosaic 16 x 1024^2 -> 4 x 2048^2 and rect 16 x 512x1024 -> 4 x 1024x2048, with both
    branches, equal to the restatement on the device's own items"""
    from multiyolov5_b200.utils.datasets import DetAugmenter, DetRectLoader, DeviceImageCache, collate_quad
    rs = np.random.RandomState(11)
    imgs0, labels0 = _frames(rs, [(1024, 2048)] * 4)
    cache = DeviceImageCache(imgs0 * 4, 1024, labels0 * 4)
    random.seed(5)
    np.random.seed(5)
    draws = [0.2, 0.7, 0.49, 0.5]                                    # upsample, tile, upsample, tile (0.5 tiles: `< 0.5` upsamples)
    for loader, hw in ((DetAugmenter(cache, _scratch()), (1024, 1024)), (DetRectLoader(cache, _scratch(), 16), (512, 1024))):
        imgs, targets = loader(range(16))
        assert tuple(imgs.shape) == (16, 3) + hw
        img4, t4 = collate_quad(imgs, targets, rng=_Draws(draws))
        want_img, want_t = rq.collate_quad_np(imgs.cpu().numpy(), targets.cpu().numpy(), _Draws(draws))
        assert tuple(img4.shape) == (4, 3, 2 * hw[0], 2 * hw[1])
        got = img4.cpu().numpy()
        assert np.array_equal(got, want_img), (hw, int((got != want_img).sum()))
        assert np.array_equal(t4.cpu().numpy(), want_t), hw


@pytest.mark.parametrize("hw", [(37, 50), (1, 3), (40, 72), (64, 32)])      # any-W kernel, then the 8-pixel one
def test_each_quad_is_independent_of_its_neighbours(hw):
    from multiyolov5_b200.utils.datasets import collate_quad
    h, w = hw
    g = torch.Generator(device="cuda").manual_seed(h * 100 + w)
    imgs = torch.randint(0, 256, (14, 3, h, w), dtype=torch.uint8, device="cuda", generator=g)
    rs = np.random.RandomState(h + w)
    t = np.zeros((28, 6), np.float32)
    t[:, 0] = np.arange(28) % 14
    t[:, 1] = rs.randint(0, 10, 28)
    t[:, 2:] = rs.uniform(0.05, 0.95, (28, 4))
    targets = torch.from_numpy(t[np.argsort(t[:, 0], kind="stable")]).cuda()
    draws = [0.9, 0.1, 0.6]
    for dtype in (torch.uint8, torch.float16, torch.float32):
        full, tf = collate_quad(imgs, targets, rng=_Draws(draws), out_dtype=dtype)
        assert tuple(full.shape) == (3, 3, 2 * h, 2 * w)
        poisoned = imgs.clone()
        poisoned[12:] = 255 - poisoned[12:]                          # the dropped items are never read
        assert torch.equal(collate_quad(poisoned, targets, rng=_Draws(draws), out_dtype=dtype)[0], full)
        for q, d in enumerate(draws):
            sel = (targets[:, 0] >= 4 * q) & (targets[:, 0] < 4 * q + 4)
            tq = targets[sel].clone()
            tq[:, 0] -= 4 * q
            one, t1 = collate_quad(imgs[4 * q:4 * q + 4], tq, rng=_Draws([d]), out_dtype=dtype)
            assert torch.equal(one[0], full[q]), (hw, dtype, q)
            assert torch.equal(t1[:, 1:], tf[tf[:, 0] == q][:, 1:]), (hw, q)
        if dtype == torch.uint8:
            want, want_t = rq.collate_quad_np(imgs.cpu().numpy(), targets.cpu().numpy(), _Draws(draws))
            assert np.array_equal(full.cpu().numpy(), want) and np.array_equal(tf.cpu().numpy(), want_t), hw


def test_fewer_than_four_images_raise():
    from multiyolov5_b200.train import Trainer
    from multiyolov5_b200.utils.datasets import collate_quad
    imgs = torch.zeros((3, 3, 16, 16), dtype=torch.uint8, device="cuda")
    with pytest.raises(ValueError):
        collate_quad(imgs, torch.zeros((0, 6), device="cuda"))
    model, cfg = _model()
    with pytest.raises(ValueError):
        Trainer(model, HYP, batch_size=3, quad=True)


# ---- Trainer(quad=True) ------------------------------------------------------------------------------------------------------------
def _quad_batch(n_items, h, w, nc, seed, rng, dtype=torch.float16):
    from multiyolov5_b200.utils.datasets import collate_quad
    rs = np.random.RandomState(seed)
    g = torch.Generator(device="cuda").manual_seed(seed)
    imgs = torch.randint(0, 256, (n_items, 3, h, w), dtype=torch.uint8, device="cuda", generator=g)
    t = np.zeros((3 * n_items, 6), np.float32)
    t[:, 0] = np.repeat(np.arange(n_items), 3); t[:, 1] = rs.randint(0, nc, 3 * n_items)
    t[:, 2:4] = rs.uniform(0.1, 0.9, (3 * n_items, 2)); t[:, 4:6] = rs.uniform(0.05, 0.4, (3 * n_items, 2))
    return collate_quad(imgs, torch.from_numpy(t).cuda(), rng=rng, out_dtype=dtype)


def _seg(B, nc_seg=19, seed=7):
    rs = np.random.RandomState(seed)
    return (synth.synth_image(B, 128, 256, seed=seed).cuda(),
            torch.from_numpy(rs.randint(-1, nc_seg, (B, 128, 256)).astype(np.int64)).cuda())


def test_trainer_quad_steps_and_x4_det_loss():
    from multiyolov5_b200.train import Trainer, scale_hyp
    from multiyolov5_b200.utils.loss import FusedComputeLoss
    model, cfg = _model()
    B = 8
    hyp = scale_hyp(HYP, nl=3, nc=cfg["nc"], imgsz=256, total_batch_size=B)
    tr = Trainer(model, hyp, batch_size=B, init_scale=2.0 ** 10, quad=True)
    assert tr._fused_det.supported and tr.det_mult() == 4. * 0.6
    segimgs, segtargets = _seg(B)
    for k, draws in enumerate(([0.2, 0.8], [0.7, 0.6], [0.1, 0.3])):
        imgs, targets = _quad_batch(B, 128, 256, cfg["nc"], k, _Draws(draws))
        assert tuple(imgs.shape) == (2, 3, 256, 512)
        items, segloss = tr.step(imgs, targets, segimgs, segtargets)
        assert torch.isfinite(items).all() and torch.isfinite(segloss).all(), k
    torch.cuda.synchronize()
    # the fused loss at the Trainer's multiplier against the torch formulation with the x4 (the bar of
    # test_gpu_train.py::test_fused_det_loss_matches_torch_formulation_at_bench_shapes)
    gen = torch.Generator(device="cuda").manual_seed(5)
    p = [torch.randn((2, 3, 256 // s, 512 // s, cfg["nc"] + 5), device="cuda", generator=gen).requires_grad_(True) for s in (8, 16, 32)]
    _, targets = _quad_batch(B, 128, 256, cfg["nc"], 9, _Draws([0.9, 0.9]))
    loss, items = tr._det_loss_scaled(p, targets)
    loss.backward()
    plain = Trainer.__new__(Trainer)
    plain.__dict__.update(tr.__dict__, quad=False)
    q0 = [v.detach().clone().requires_grad_(True) for v in p]
    loss0, _ = plain._det_loss_scaled(q0, targets)
    assert torch.allclose(loss.detach(), loss0.detach() * 4., rtol=1e-6, atol=0)
    grads, fitems = FusedComputeLoss(model)([q.detach() for q in p], targets, mult=tr.det_mult(), scale=tr.scale)
    torch.cuda.synchronize()
    assert torch.allclose(fitems, items, rtol=2e-5, atol=1e-6), (fitems, items)
    for q, gq in zip(p, grads):
        err = float((gq - q.grad).abs().max() / q.grad.abs().max())
        assert err <= 5e-5, err


def test_trainer_quad_graphed_det_loss_for_unfused_hyps():
    """positive weights take the torch formulation as a captured graph; its key holds quad, and the replay equals the eager x4 loss"""
    from multiyolov5_b200.train import Trainer, scale_hyp
    model, cfg = _model()
    B = 8
    hyp = scale_hyp(dict(HYP, cls_pw=0.631, obj_pw=0.911), nl=3, nc=cfg["nc"], imgsz=256, total_batch_size=B)
    tr = Trainer(model, hyp, batch_size=B, init_scale=2.0 ** 10, quad=True)
    assert not tr._fused_det.supported
    shapes = [(2, 3, 256 // s, 512 // s, cfg["nc"] + 5) for s in (8, 16, 32)]
    st = tr._det_graph(shapes, 64, torch.device("cuda"))
    tr.quad = False
    assert tr._det_graph(shapes, 64, torch.device("cuda")) is not st          # quad is part of the key
    tr.quad = True
    gen = torch.Generator(device="cuda").manual_seed(3)
    ps = [torch.randn(sh, device="cuda", generator=gen) for sh in shapes]
    _, targets = _quad_batch(B, 128, 256, cfg["nc"], 4, _Draws([0.9, 0.1]))
    nt = targets.shape[0]
    with torch.no_grad():
        for q, v in zip(st.p, ps):
            q.copy_(v)
        st.t.zero_()
        st.t[:nt].copy_(targets)
    st.graph.replay()
    pe = [v.clone().requires_grad_(True) for v in ps]
    loss, items = tr._det_loss_scaled(pe, targets)
    loss.backward()
    torch.cuda.synchronize()
    assert torch.allclose(st.items, items, rtol=1e-6, atol=1e-7)
    for q, e in zip(st.p, pe):
        assert float((q.grad - e.grad).norm() / e.grad.norm()) < 1e-6
    segimgs, segtargets = _seg(B)
    imgs, targets = _quad_batch(B, 128, 256, cfg["nc"], 5, _Draws([0.2, 0.8]))
    items, segloss = tr.step(imgs, targets, segimgs, segtargets)
    torch.cuda.synchronize()
    assert torch.isfinite(items).all() and torch.isfinite(segloss).all()


class _Fixed:
    def __init__(self, v):
        self.v = v

    def randrange(self, a, b):
        assert a <= self.v < b
        return self.v


def test_quad_with_multiscale_and_det_shapes_runs_every_size_on_one_workspace():
    from multiyolov5_b200.train import MultiScale, Trainer, scale_hyp
    model, cfg = _model()
    B = 8
    hyp = scale_hyp(HYP, nl=3, nc=cfg["nc"], imgsz=256, total_batch_size=B)
    ms = MultiScale(256)
    det_shapes = [(128, 256), (256, 128)]
    tr = Trainer(model, hyp, batch_size=B, init_scale=2.0 ** 10, multi_scale=ms, det_shapes=det_shapes, quad=True)
    want = sorted(set(ms.shapes((256, 512))) | set(ms.shapes((512, 256))))
    assert tr.det_train_shapes() == want and tr._ms_batches == {2}
    eng = model.engine()
    arena = eng._arenas[0]
    assert {k for k in eng._reserved if k[1] == 2} == {("train", 2, H, W) for H, W in want}
    segimgs, segtargets = _seg(B)
    seen = set()
    for k, (h, w) in enumerate(det_shapes):
        imgs4, targets = _quad_batch(B, h, w, cfg["nc"], 20 + k, _Draws([0.3, 0.8]), dtype=torch.uint8)
        for sz in sorted({v // 32 * 32 for v in range(ms.lo, ms.hi)}):
            imgs = ms(imgs4, torch.float16, rng=_Fixed(sz))
            seen.add(tuple(imgs.shape[2:]))
            items, segloss = tr.step(imgs, targets, segimgs, segtargets)
            assert torch.isfinite(items).all() and torch.isfinite(segloss).all(), (h, w, sz)
    torch.cuda.synchronize()
    assert seen == set(want), sorted(set(want) ^ seen)
    det = [p for key, p in eng.plans.items() if key[0] == "train" and len(key) == 4 and key[1] == 2]
    assert len(det) == len(want) and all(p.arena is arena for p in det) and eng._arenas[0] is arena
    # multi_scale alone: the square (2S, 2S) batch's sizes
    model2, _ = _model()
    tr2 = Trainer(model2, hyp, batch_size=B, init_scale=2.0 ** 10, multi_scale=ms, quad=True)
    assert tr2.det_train_shapes() == ms.shapes((512, 512))
