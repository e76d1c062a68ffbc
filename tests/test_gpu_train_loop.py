"""train.fit on the GPU: s/PSP at 2 + 2 images of 128 x 256, synthetic weights, frames and targets.  The schedule the loop hands the
Trainer past the 800-iteration warm-up, the loop's calls against a hand-written sequence, checkpoints and resume, and no host
synchronisation between two log points."""
import argparse
import os

import numpy as np
import pytest
import torch

from oracle import synth

pytestmark = pytest.mark.gpu

CFG = "yolov5s_city_seg.yaml"
HYP = dict(lr0=0.01, lrf=0.2, momentum=0.937, weight_decay=5e-4, warmup_epochs=3.0, warmup_momentum=0.8, warmup_bias_lr=0.1, box=0.05,
           cls=0.5, cls_pw=1.0, obj=1.0, obj_pw=1.0, anchor_t=4.0, fl_gamma=0.0)
B, H, W = 2, 128, 256


def psp_model():
    from multiyolov5_b200.models.yolo import Model
    cfg = synth.load_cfg(CFG)
    sd = synth.synth_state_dict(synth.load_manifest("s_psp"), cfg, seed=1, gain=1.0)
    torch.manual_seed(0)
    model = Model(CFG)
    model.load_state_dict(sd)
    return model.cuda(), cfg


def make_batches(nc, n=4, seed=0):
    rs = np.random.RandomState(seed)
    det, seg = [], []
    for k in range(n):
        t = np.zeros((12, 6), np.float32)
        t[:, 0] = rs.randint(0, B, 12); t[:, 1] = rs.randint(0, nc, 12)
        t[:, 2:4] = rs.uniform(0.1, 0.9, (12, 2)); t[:, 4:6] = rs.uniform(0.05, 0.4, (12, 2))
        mask = torch.from_numpy(rs.randint(-1, 19, (B, 1, 16, 32)).astype(np.int64)).cuda()
        mask = mask.repeat_interleave(8, 2).repeat_interleave(8, 3)[:, 0].contiguous()
        det.append((synth.synth_image(B, H, W, seed=10 * k + 1).cuda(), torch.from_numpy(t).cuda()))
        seg.append((synth.synth_image(B, H, W, seed=10 * k + 2).cuda(), mask))
    return det, seg


class Cycle:
    """nb batches per epoch, cycling through a few device batches; `before(epoch, i)` runs before batch i is handed out"""

    def __init__(self, items, nb, before=None):
        self.items, self.nb, self.before = items, nb, before

    def __len__(self):
        return self.nb

    def __call__(self, epoch):
        for i in range(self.nb):
            if self.before is not None:
                self.before(epoch, i)
            yield self.items[i % len(self.items)]
        if self.before is not None:
            self.before(epoch, None)


def opt_(**kw):
    o = dict(epochs=1, batch_size=B, img_size=[256, 256], linear_lr=False, adam=False, notest=False, nosave=False, evolve=False,
             multi_scale=False, quad=False, single_cls=False, resume=False, global_rank=-1, world_size=1, label_smoothing=0.0,
             weights="", cfg="")
    o.update(kw)
    return argparse.Namespace(**o)


@pytest.fixture
def recording(monkeypatch):
    """Trainer whose instances and step calls are recorded: (ni, lr, momentum, accumulate, batch ids, loss items, seg loss)"""
    import multiyolov5_b200.train as TR
    rec = {"trainers": [], "calls": []}

    class Recorded(TR.Trainer):
        def __init__(self, *a, **k):
            super().__init__(*a, **k)
            rec["trainers"].append(self)

        def step(self, imgs, targets, segimgs, segtargets, ni=None):
            if "on_first_step" in rec and not rec["calls"]:
                rec["on_first_step"](self)
            items, segloss = super().step(imgs, targets, segimgs, segtargets, ni=ni)
            rec["calls"].append((ni, tuple(self.lr), self.momentum, self.accumulate, id(imgs), id(segimgs), items, segloss))
            return items, segloss

    monkeypatch.setattr(TR, "Trainer", Recorded)
    return rec


def tiny_val(nc):
    g = torch.Generator().manual_seed(5)
    det = []
    for _ in range(2):
        t = torch.rand((6, 6), generator=g)
        t[:, 0] = torch.arange(6) % B
        t[:, 1] = torch.randint(0, nc, (6,), generator=g).float()
        t[:, 4:6] = t[:, 4:6] * 0.3 + 0.05
        det.append((torch.randint(0, 256, (B, 3, H, W), dtype=torch.uint8, generator=g), t, [""] * B,
                    [((H, W), ((1.0, 1.0), (0.0, 0.0)))] * B))
    seg = [(torch.rand((B, 3, H, W), generator=g).cuda(), torch.randint(-1, 19, (B, H, W), generator=g).cuda()) for _ in range(2)]
    return det, seg


def test_a_run_past_the_warm_up_follows_the_schedule(tmp_path, recording):
    """9 epochs of 100 iterations (warm-up: 800): every (lr, momentum, accumulate, step) handed to the Trainer is the schedule's, the
    device step counter equals the optimizer steps the schedule predicts, and the losses are finite"""
    from multiyolov5_b200.train import LRSchedule, fit
    model, cfg = psp_model()
    det, seg = make_batches(cfg["nc"])
    nb, epochs = 100, 9
    fit(model, HYP, opt_(epochs=epochs, nosave=True, evolve=True), Cycle(det, nb), Cycle(seg, nb), save_dir=tmp_path, log_interval=100,
        init_scale=2.0 ** 10)
    sched = LRSchedule(HYP, epochs, nb, B)
    calls = recording["calls"]
    assert len(calls) == nb * epochs
    predicted = 0
    for k, c in enumerate(calls):
        e, i = divmod(k, nb)
        it = sched.iteration(e, i)
        assert c[0] == it.ni and c[1] == it.lr and c[2] == it.momentum and c[3] == it.accumulate, (k, c[:4], it)
        predicted += it.step
        if i == nb - 1:
            sched.step()
    assert sched.nw == 800 and calls[-1][3] == 64 // B
    tr = recording["trainers"][0]
    assert int(tr.steps) == predicted
    items = torch.stack([c[6] for c in calls])
    segs = torch.stack([c[7].reshape(()) for c in calls])
    assert bool(torch.isfinite(items).all()) and bool(torch.isfinite(segs).all())


def _states(tr, ema):
    f = tr.flat
    return [f.param.clone(), f.momentum.clone()] + [v.detach().clone() for v in ema.ema.state_dict().values() if v.dtype.is_floating_point]


def test_the_loop_adds_nothing_to_the_step(tmp_path, recording):
    """fit's first 12 iterations against a hand-written sequence of set_lr / set_momentum / accumulate / Trainer.step(ni=...) over the
    same batches: the same calls with the same arguments, and parameters, momentum and EMA within the run-to-run spread of the
    hand-written sequence itself (the backward adds gradients with fp32 atomics, so two runs of one sequence may differ in the last bits)"""
    from multiyolov5_b200.train import LRSchedule, Trainer, fit, scale_hyp
    from multiyolov5_b200.utils.torch_utils import ModelEMA
    K = 12
    model, cfg = psp_model()
    det, seg = make_batches(cfg["nc"])
    fit(model, HYP, opt_(nosave=True, evolve=True), Cycle(det, K), Cycle(seg, K), save_dir=tmp_path, init_scale=2.0 ** 10)
    tr_fit = recording["trainers"][0]
    fit_calls = [c[:4] + (c[4] - id(det[0][0]),) for c in recording["calls"]]
    torch.cuda.synchronize()
    got = _states(tr_fit, tr_fit.ema)
    Trainer = Trainer.__mro__[1]                   # the unrecorded class
    runs = []
    for _ in range(2):
        m, _ = psp_model()
        ema = ModelEMA(m)
        m.half().float()
        tr = Trainer(m, scale_hyp(HYP, nl=3, nc=cfg["nc"], imgsz=256, total_batch_size=B), B, accumulate=32, ema=ema, init_scale=2.0 ** 10)
        sched = LRSchedule(HYP, 1, K, B)
        calls = []
        for i in range(K):
            it = sched.iteration(0, i)
            tr.set_lr(*it.lr)
            tr.set_momentum(it.momentum)
            tr.accumulate = it.accumulate
            tr.step(*det[i % len(det)], *seg[i % len(seg)], ni=it.ni)
            calls.append((it.ni, it.lr, it.momentum, it.accumulate, id(det[i % len(det)][0]) - id(det[0][0])))
        assert calls == fit_calls
        torch.cuda.synchronize()
        runs.append(_states(tr, ema))
    for a, b, c in zip(got, runs[0], runs[1]):
        spread = float((b - c).abs().max())
        assert float((a - b).abs().max()) <= 4 * spread + 1e-7, (float((a - b).abs().max()), spread)


def test_checkpoints_and_resume(tmp_path, recording, monkeypatch):
    """last.pt / best.pt carry the golden reference checkpoint's keys and value types and load with attempt_load; resuming from the
    last.pt of epoch 1 restores moments, step count, initial_lr, the EMA and its updates, best_fitness, results.txt and start_epoch, and
    the first resumed iteration gets the uninterrupted run's lr"""
    from multiyolov5_b200.models.experimental import attempt_load, load_checkpoint
    from multiyolov5_b200.train import fit
    golden = load_checkpoint(os.path.join(synth.GOLDEN_DIR, "ref_ckpt_tiny.pt"))
    model, cfg = psp_model()
    det, seg = make_batches(cfg["nc"])
    vdet, vseg = tiny_val(cfg["nc"])
    nb = 6
    saved, orig = {}, torch.save

    def save(obj, f):
        orig(obj, f)
        if str(f).endswith("last.pt"):
            orig(obj, str(tmp_path / f"epoch{obj['epoch']}.pt"))
            saved[obj["epoch"]] = str(tmp_path / f"epoch{obj['epoch']}.pt")
    monkeypatch.setattr(torch, "save", save)
    run_a = tmp_path / "a"
    fit(model, HYP, opt_(epochs=3), Cycle(det, nb), Cycle(seg, nb), test_loader=vdet, segval_loader=vseg, save_dir=run_a,
        init_scale=2.0 ** 10)
    calls_a = list(recording["calls"])
    for name in ("last.pt", "best.pt"):
        ck = load_checkpoint(str(run_a / "weights" / name))
        assert list(ck) == list(golden)
        for k, v in golden.items():
            if k == "best_fitness":                          # 0.0 until fitness2 first exceeds it, then fitness2's (1,) array
                assert isinstance(ck[k], (float, np.ndarray))
            elif v is not None:
                assert type(ck[k]) is type(v), k
        assert type(ck["ema"]) is type(golden["model"]) and isinstance(ck["optimizer"], dict) and ck["wandb_id"] is None
        assert next(ck["model"].parameters()).dtype == torch.float16 and next(ck["ema"].parameters()).dtype == torch.float16
        m = attempt_load(str(run_a / "weights" / name), map_location="cuda")
        with torch.no_grad():
            out = m(synth.synth_image(1, H, W, seed=3).cuda())
        assert torch.isfinite(out[1]).all()

    ck1 = load_checkpoint(saved[1], map_location="cuda")
    recording["calls"].clear()
    restored = {}

    def on_first_step(tr):
        restored["sd"] = tr.state_dict()
        restored["ema"] = {k: v.clone() for k, v in tr.ema.ema.state_dict().items()}
        restored["updates"] = tr.ema.updates
        restored["results"] = (tmp_path / "b" / "results.txt").read_text()
    recording["on_first_step"] = on_first_step
    model_b, _ = psp_model()
    fit(model_b, HYP, opt_(epochs=3, resume=True, weights=saved[1]), Cycle(det, nb), Cycle(seg, nb), test_loader=vdet,
        segval_loader=vseg, save_dir=tmp_path / "b", init_scale=2.0 ** 10)
    sd, ref = restored["sd"], ck1["optimizer"]
    # every group setting but lr and momentum, which the first iteration's warm-up has set already (checked below)
    strip = lambda gs: [{k: v for k, v in g.items() if k not in ("lr", "momentum")} for g in gs]          # noqa: E731
    assert strip(sd["param_groups"]) == strip(ref["param_groups"])
    assert sorted(sd["state"]) == sorted(ref["state"])
    assert all(torch.equal(sd["state"][j]["momentum_buffer"], ref["state"][j]["momentum_buffer"]) for j in ref["state"])
    esd = ck1["ema"].float().state_dict()
    assert all(torch.equal(restored["ema"][k], v) for k, v in esd.items() if v.dtype.is_floating_point)
    assert restored["updates"] == ck1["updates"]
    assert restored["results"] == ck1["training_results"]
    first = recording["calls"][0]
    assert first[0] == 2 * nb                                               # start_epoch 2
    a_at = [c for c in calls_a if c[0] == 2 * nb][0]
    assert first[1] == a_at[1] and first[2] == a_at[2] and first[3] == a_at[3]
    ck_b = load_checkpoint(str(tmp_path / "b" / "weights" / "last.pt"))
    assert ck_b["training_results"].startswith(ck1["training_results"]) and ck_b["epoch"] == 2
    assert float(np.max(ck_b["best_fitness"])) >= float(np.max(ck1["best_fitness"]))
    assert ck_b["updates"] == ck1["updates"] + sum(1 for c in recording["calls"] if c[0] % c[3] == 0)


def test_no_host_synchronisation_between_log_points(tmp_path, recording):
    """epoch 1 of a run with log_interval 5 under torch.cuda.set_sync_debug_mode('error') for every iteration that does not end at a
    log point (epoch 0 builds the plans and tables, which may synchronise)"""
    from multiyolov5_b200.train import fit
    model, cfg = psp_model()
    det, seg = make_batches(cfg["nc"])
    nb, L = 20, 5
    checked = []

    def before(epoch, i):
        if epoch >= 1 and i is not None and (i + 1) % L:
            torch.cuda.set_sync_debug_mode("error")
            checked.append(i)
        else:
            torch.cuda.set_sync_debug_mode("default")
    try:
        fit(model, HYP, opt_(epochs=2, nosave=True, evolve=True), Cycle(det, nb, before), Cycle(seg, nb), save_dir=tmp_path,
            log_interval=L, init_scale=2.0 ** 10)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    assert len(checked) == nb - nb // L
