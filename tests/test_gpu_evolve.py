"""H100: models with 2 to 10 anchors per level, as `Model(cfg, anchors=n)` and --evolve's `anchors` hyp build them, on every device path -
the inference plan and NMS, the train plan's forward and backward, the fused detection loss, autoanchor on the placeholder anchors - and
train.evolve end to end: three generations of fit on s/PSP with a frozen clock, each generation's hyp against the host restatement, and
nothing of a finished generation left on the device."""
import argparse
import contextlib
import gc
import io
import json
import os
import random
import time
import weakref
from copy import deepcopy

import numpy as np
import pytest
import torch

from oracle import restate, synth
from oracle import restate_autoanchor as ra
from oracle import restate_evolve as rev

pytestmark = pytest.mark.gpu
CFG = "yolov5s_city_seg.yaml"
GOLD = os.path.join(os.path.dirname(__file__), "golden")


def model_n(n, gain=None):
    """Model(CFG, anchors=n) with synthetic weights and the anchors autoanchor could leave (rev.anchor_table(n)); its cfg and state dict
    for the restatement"""
    from multiyolov5_b200.models.yolo import Model
    cfg = dict(synth.load_cfg(CFG), anchors=rev.anchor_table(n))
    model = Model(CFG, anchors=n)
    manifest = [[k, list(v.shape), str(v.dtype).replace("torch.", "")] for k, v in model.state_dict().items()]
    sd = synth.synth_state_dict(manifest, cfg, seed=1, gain=gain)
    model.load_state_dict(sd)
    return model.cuda(), cfg, sd


def rel(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return float((a - b).abs().max() / (b.abs().max() + 1e-30))


@pytest.mark.parametrize("n", [2, 4, 10])
def test_inference_and_nms_at_an_anchor_count(n):
    """z / raws / seg against the restatement within smoke()'s and the parity tests' tolerances; NMS rows equal to the restatement's on
    the same z (na * sum(ny * nx) rows)"""
    from multiyolov5_b200.utils.general import non_max_suppression
    model, cfg, sd = model_n(n)
    model.eval()
    B, H, W = 2, 128, 256
    x = synth.synth_image(B, H, W, seed=0)
    (z, raws), seg = model(x.cuda())
    torch.cuda.synchronize()
    assert z.shape == (B, n * sum((H // s) * (W // s) for s in (8, 16, 32)), 15)
    assert [tuple(r.shape) for r in raws] == [(B, n, H // s, W // s, 15) for s in (8, 16, 32)]
    q = restate.model_forward(cfg, sd, x, quantised=True)
    assert rel(seg, q["seg"]) < 4e-3 and rel(z, q["z"]) < 2e-2, (rel(seg, q["seg"]), rel(z, q["z"]))
    for r, qr in zip(raws, q["raw"]):
        assert rel(r, qr) < 6e-3
    dets = non_max_suppression(z, 0.25, 0.45)
    ref = restate.non_max_suppression(z.cpu().numpy(), 0.25, 0.45)
    assert all(np.array_equal(d.cpu().numpy(), r) for d, r in zip(dets, ref))


@pytest.mark.parametrize("n", [2, 4, 10])
def test_train_forward_and_backward_at_an_anchor_count(n):
    """the train plan (Detect convs of Co = n * 15) against the fp32 autograd oracle, with test_gpu_train's bars: no further than torch's
    fp16 autocast of the same graph, and the fp32 Detect biases exact up to summation order"""
    from tests.test_gpu_train import amp_yardstick, oracle_train, rel_f
    model, cfg, sd = model_n(n, gain=1.0)
    model.train()
    B, H, W = 2, 128, 256
    x = synth.synth_image(B, H, W, seed=5)
    torch.set_num_threads(min(32, os.cpu_count() or 1))
    gen = torch.Generator().manual_seed(11)
    raws, seg = model(x.cuda())
    assert [tuple(r.shape) for r in raws] == [(B, n, H // s, W // s, 15) for s in (8, 16, 32)]
    Rs = [torch.randn(r.shape, generator=gen) * 4.0 for r in raws]
    S = [torch.randn(seg.shape, generator=gen) * 0.05]
    (sum((r * R.cuda()).sum() for r, R in zip(raws, Rs)) + (seg * S[0].cuda()).sum()).backward()
    torch.cuda.synchronize()
    o_raw, o_seg, sdg = oracle_train(cfg, sd, x, Rs, S)
    amp_fwd, amp_grd = amp_yardstick(cfg, sd, x, Rs, S, o_raw, o_seg, sdg)
    ours_fwd = [rel_f(a.detach().cpu(), b.detach()) for a, b in zip(list(raws) + [seg], list(o_raw) + list(o_seg))]
    assert max(ours_fwd) < 0.10 and all(o <= 1.25 * a + 2e-3 for o, a in zip(ours_fwd, amp_fwd)), (ours_fwd, amp_fwd)
    errs, coss = {}, {}
    for name, p in model.named_parameters():
        g_ref = sdg[name].grad
        if g_ref is None or g_ref.norm() < 1e-8:
            continue
        g = p.grad.detach().cpu()
        errs[name] = rel_f(g, g_ref)
        coss[name] = float((g.double().flatten() @ g_ref.double().flatten()) / (g.double().norm() * g_ref.double().norm()))
    med, amp_med = float(np.median(list(errs.values()))), float(np.median(list(amp_grd.values())))
    assert med < 0.25 and max(errs.values()) < 0.40 and min(coss.values()) > 0.95, (med, max(errs.values()), min(coss.values()))
    assert max(errs.values()) <= 1.25 * max(amp_grd.values()) and med <= 1.25 * amp_med, (med, amp_med)
    for i in range(3):
        assert errs[f"model.25.m.{i}.bias"] < 1e-5 and coss[f"model.25.m.{i}.weight"] > 0.99


def _fixture():
    return np.load(os.path.join(GOLD, "anchor_count_cases.npz"))


@pytest.mark.parametrize("na", [4, 10])
def test_fused_det_loss_at_more_anchors_matches_the_reference(na):
    from multiyolov5_b200.models.yolo import Model
    from multiyolov5_b200.utils.loss import FusedComputeLoss
    g = _fixture()
    tag = f"loss{na}"
    model = Model(CFG, anchors=na)
    model.hyp, model.gr = json.loads(bytes(g["loss_hyp_json"]).decode()), 1.0
    model.model[-1].anchors[:] = torch.from_numpy(g[f"{tag}_anchors"])
    crit = FusedComputeLoss(model)
    assert crit.supported
    p = [torch.from_numpy(q).cuda().contiguous() for q in rev.loss_predictions(na)[0]]
    grads, items = crit(p, torch.from_numpy(g[f"{tag}_targets"]).cuda())
    torch.cuda.synchronize()
    assert np.allclose(items.cpu().numpy(), g[f"{tag}_items"], rtol=2e-5, atol=1e-6), (items.cpu().numpy(), g[f"{tag}_items"])
    for i in range(3):
        ref = g[f"{tag}_g{i}"]
        assert np.abs(grads[i].cpu().numpy() - ref).max() / np.abs(ref).max() <= 2e-5, i


@pytest.mark.parametrize("na", [4, 10])
def test_fused_det_loss_at_more_anchors_matches_torch_at_bench_shapes(na):
    """4 x na x 64x128 / 32x64 / 16x32 with 80 boxes (duplicate cells, padding rows), loss scale and multiplier; and the Trainer takes
    the fused loss at this anchor count with cls_pw = obj_pw = 1"""
    from multiyolov5_b200.train import Trainer, scale_hyp
    from multiyolov5_b200.utils.loss import ComputeLoss, FusedComputeLoss
    model, _, _ = model_n(na)
    hyp = dict(lr0=0.0015, momentum=0.937, weight_decay=5e-4, box=0.05, cls=0.5, cls_pw=1.0, obj=1.0, obj_pw=1.0, anchor_t=4.0, fl_gamma=0.0)
    model.hyp, model.gr = scale_hyp(hyp, nl=3, nc=10, imgsz=1024, total_batch_size=32), 1.0
    gen = torch.Generator(device="cuda").manual_seed(5)
    B = 4
    p = [torch.randn((B, na, 512 // s, 1024 // s, 15), device="cuda", generator=gen).requires_grad_(True) for s in (8, 16, 32)]
    rs = np.random.RandomState(3)
    t = np.zeros((80 + 16, 6), np.float32)
    t[:80, 0] = np.repeat(np.arange(B), 20); t[:80, 1] = rs.randint(0, 10, 80)
    t[:80, 2:4] = rs.uniform(0.1, 0.9, (80, 2)); t[:80, 4:6] = rs.uniform(0.02, 0.22, (80, 2))
    t[10:14, 2:6] = t[10, 2:6]
    t[10:14, 0] = t[10, 0]
    tg = torch.from_numpy(t).cuda()
    scale = torch.full((), 1024.0, device="cuda")
    loss, items = ComputeLoss(model)(p, tg)
    (loss * 8 * 0.6 * scale).backward()
    grads, fitems = FusedComputeLoss(model)([q.detach() for q in p], tg, mult=8 * 0.6, scale=scale)
    torch.cuda.synchronize()
    assert torch.allclose(fitems, items, rtol=2e-5, atol=1e-6), (fitems, items)
    for q, gq in zip(p, grads):
        assert float((gq - q.grad).abs().max() / q.grad.abs().max()) <= 5e-5
    tr = Trainer(model, scale_hyp(hyp, nl=3, nc=10, imgsz=256, total_batch_size=2), batch_size=2, accumulate=1000, init_scale=2.0 ** 10)
    assert tr._fused_det.supported


def test_fused_det_loss_refuses_more_than_ten_anchors():
    from multiyolov5_b200 import _lib
    from multiyolov5_b200.models.yolo import Model
    from multiyolov5_b200.utils.loss import FusedComputeLoss
    model = Model(CFG, anchors=11)
    model.hyp, model.gr = dict(box=0.05, cls=0.5, obj=1.0, anchor_t=4.0), 1.0
    assert not FusedComputeLoss(model).supported
    p = [torch.zeros((1, 11, 8 // s, 8 // s, 15), device="cuda") for s in (1, 2, 4)]
    crit = FusedComputeLoss(model)
    crit.supported = True
    with pytest.raises(_lib.MyoloError, match="bad arguments"):
        crit(p, torch.zeros((0, 6), device="cuda"))


def _cache(shapes0, labels, augment=True, img_size=64):
    from multiyolov5_b200.utils.datasets import DeviceImageCache
    return DeviceImageCache([np.zeros((h0, w0, 3), np.uint8) for h0, w0 in shapes0], img_size, labels=labels, augment=augment)


@pytest.mark.parametrize("n", [2, 4, 10])
def test_check_anchors_on_placeholder_anchors(n):
    """check_anchors on the placeholders of Model(cfg, anchors=n) (one anchor 0 wide: ratios inf and 0) against the reference's run:
    printed lines, the Detect buffers and the state of random / numpy.random afterwards"""
    from multiyolov5_b200.models.yolo import Model
    from multiyolov5_b200.utils import autoanchor as aa
    cases = {c["name"]: c for c in ra.load_cases(os.path.join(GOLD, "autoanchor_placeholder_cases.npz"))}
    if f"placeholder{n}" not in cases:
        pytest.skip(f"the fixture has no placeholder{n} case (no seed produced it)")
    c = cases[f"placeholder{n}"]
    model = Model(CFG, anchors=n).cuda()
    det = model.model[-1]
    assert np.array_equal(det.anchor_grid.cpu().numpy(), c["anchor_grid0"]) and np.array_equal(det.anchors.cpu().numpy(), c["anchors0"])
    shapes0, labels = ra.case_dataset(c)
    cache = _cache(shapes0, labels)
    random.seed(c["seed"]); np.random.seed(c["seed"]); torch.manual_seed(c["seed"])
    with contextlib.redirect_stdout(io.StringIO()) as buf:
        aa.check_anchors(cache, model, thr=c["thr"], imgsz=c["imgsz"])
    assert buf.getvalue() == c["stdout"]
    assert np.array_equal(det.anchor_grid.cpu().numpy(), c["anchor_grid1"])
    assert np.array_equal(det.anchors.cpu().numpy(), c["anchors1"])
    assert np.array_equal(np.array([random.random(), random.random()]), c["next_py"])
    assert np.array_equal(np.random.random(4), c["next_np"])


# ---- evolve end to end ----
B, H, W = 2, 128, 256


def _frames(n, seed, nc=10, per_img=40):
    rs = np.random.RandomState(seed)
    imgs = [rs.randint(0, 256, (H, W, 3)).astype(np.uint8) for _ in range(n)]
    labels = []
    for _ in range(n):
        l = np.zeros((per_img, 5), np.float32)
        l[:, 0] = rs.randint(0, nc, per_img)
        l[:, 1:3] = rs.uniform(0.15, 0.85, (per_img, 2))
        l[:, 3:5] = rs.uniform(0.03, 0.3, (per_img, 2))
        labels.append(l)
    return imgs, labels


def test_evolve_three_generations_end_to_end(tmp_path, monkeypatch):
    """three generations of one epoch each (2 + 2 images of 128 x 256, notest: the final test over a DetValLoader) through the
    train_fn of the README: every generation's hyp equals the restatement's given the earlier results, Detect.na follows the `anchors`
    hyp, evolve.txt has the reference's layout, and generation 1's Model, Engine and Trainer are gone and its device memory is free while
    generation 3 runs"""
    import multiyolov5_b200.train as TR
    from multiyolov5_b200.models.yolo import Model
    from multiyolov5_b200.train import DetEpochBatches, evolve, fit
    from multiyolov5_b200.utils.autoanchor import check_anchors
    from multiyolov5_b200.utils.datasets import DetAugmenter, DetValLoader, DeviceImageCache
    from tests.test_gpu_train_loop import psp_model
    imgs, labels = _frames(2, 0)
    cache = DeviceImageCache(imgs, 256, labels=labels)
    val = DetValLoader(DeviceImageCache(imgs, 256, labels=labels, augment=False), B)
    gen = torch.Generator().manual_seed(3)
    seg = [(torch.rand((B, 3, H, W), generator=gen).cuda(), torch.randint(-1, 19, (B, H, W), generator=gen).cuda())]
    start, _ = psp_model()
    weights = str(tmp_path / "start.pt")
    torch.save({"epoch": -1, "best_fitness": 0.0, "training_results": None, "model": deepcopy(start).half(), "ema": None, "updates": 0,
                "optimizer": None, "wandb_id": None}, weights)
    del start

    trainers = []

    class Recorded(TR.Trainer):
        def __init__(self, *a, **k):
            super().__init__(*a, **k)
            trainers.append(weakref.ref(self))
    monkeypatch.setattr(TR, "Trainer", Recorded)

    refs, results, nas, mem = [], [], [], {}

    def settled_memory():
        """device memory in use between generations; NMS keeps one workspace sized by its last call's row count (na * sum ny * nx),
        which is not a generation's and is dropped here"""
        from multiyolov5_b200.utils import general
        general._ws_cache.clear()
        gc.collect()
        torch.cuda.synchronize()
        return torch.cuda.memory_allocated()

    def train_fn(hyp, opt):
        k = len(results)
        if k == 1:
            mem["after1"] = settled_memory()
        if k == 2:
            gc.collect()
            assert all(r() is None for r in refs[0]), [r() is None for r in refs[0]]
        model = Model(CFG, nc=10, anchors=hyp.get("anchors")).cuda()
        model.names = [str(i) for i in range(10)]
        with contextlib.redirect_stdout(io.StringIO()):
            check_anchors(cache, model, thr=hyp["anchor_t"], imgsz=256)
        nas.append(model.model[-1].na)
        r = fit(model, hyp, opt, DetEpochBatches(DetAugmenter(cache, hyp), B), lambda epoch: iter(seg), test_loader=val,
                save_dir=tmp_path / f"gen{k}", init_scale=2.0 ** 10)
        refs.append((weakref.ref(model), weakref.ref(model.engine()), trainers[-1]))
        results.append(tuple(float(v) for v in r))
        return r

    clock = lambda: rev.clock(len(results))                                       # noqa: E731
    monkeypatch.setattr(time, "time", clock)
    monkeypatch.chdir(tmp_path)
    opt = argparse.Namespace(epochs=1, batch_size=B, img_size=[256, 256], linear_lr=False, adam=False, notest=False, nosave=False,
                             evolve=True, multi_scale=False, quad=False, single_cls=False, resume=False, global_rank=-1, local_rank=-1,
                             world_size=1, label_smoothing=0.0, weights=weights, cfg="", save_dir=str(tmp_path / "run"))
    os.makedirs(opt.save_dir)
    random.seed(7)
    hyps = []
    real_fn = train_fn

    def recording_fn(hyp, o):
        hyps.append(dict(hyp))
        return real_fn(hyp, o)
    evolve(dict(rev.HYP_SCRATCH), opt, recording_fn, generations=3, evolve_txt="evolve.txt")
    after3 = settled_memory()
    assert after3 <= mem["after1"], (after3, mem["after1"])
    assert opt.notest and opt.nosave and len(hyps) == 3
    assert nas == [round(h["anchors"]) for h in hyps]

    random.seed(7)
    os.makedirs("replay")
    exp = rev.run(dict(rev.HYP_SCRATCH), lambda h, k: results[k], 3, "replay/evolve.txt", "replay/hyp.yaml")
    assert hyps == exp
    assert (tmp_path / "evolve.txt").read_text() == (tmp_path / "replay" / "evolve.txt").read_text()
    rows = (tmp_path / "evolve.txt").read_text().splitlines()
    x = np.loadtxt(tmp_path / "evolve.txt", ndmin=2)
    assert 1 <= len(rows) <= 3 and x.shape[1] == 7 + len(rev.HYP_SCRATCH)
    assert rows == [" ".join("%10.3g" % v for v in row) for row in x]            # np.savetxt(fmt='%10.3g'): 35 fields, one space apart
    # print_mutation sorts the rows it reads back (the earlier generations' at '%10.3g', the last one's results at '%10.4g') by fitness
    # and only then saves every row at '%10.3g', which can swap the order of near-tied fitness values: restore the last generation's
    # results to what the sort saw, and the rows are in descending fitness exactly
    seen = [float("%10.4g" % v) for v in results[-1]]
    (last,) = [i for i, row in enumerate(x) if row[:7].tolist() == [float("%10.3g" % v) for v in seen]]
    x[last, :7] = seen
    f = (x[:, :4] * [0.0, 0.0, 0.1, 0.9]).sum(1)
    assert (np.diff(f) <= 0).all(), f
    assert (tmp_path / "run" / "hyp_evolved.yaml").read_text().startswith("# Hyperparameter Evolution Results\n# Generations: ")
