"""The epoch loop of reference train.py without a GPU: LRSchedule against oracle/restate_loop.py (torch's real LambdaLR), fit's
bookkeeping over a fake Trainer and fake validators, and the seg epoch order of SegEpochBatches."""
import argparse

import numpy as np
import pytest
import torch
import torch.nn as nn

from oracle import restate_loop as R

# the schedule keys of the reference's data/hyp.scratch.yaml and data/hyp.finetune.yaml
SCRATCH = dict(lr0=0.0015, lrf=0.2, momentum=0.937, weight_decay=0.0005, warmup_epochs=3.0, warmup_momentum=0.8, warmup_bias_lr=0.1)
FINETUNE = dict(lr0=0.0032, lrf=0.12, momentum=0.843, weight_decay=0.00036, warmup_epochs=2.0, warmup_momentum=0.5, warmup_bias_lr=0.05)
HYPS = {"scratch": SCRATCH, "finetune": FINETUNE}
# (nb, epochs): warm-up of 800 iterations ending mid-epoch (800 / 7), nb * warmup_epochs below 800, and above it (3 * 300 = 900)
RUNS = [(7, 118), (100, 10), (300, 5)]


def schedule_records(sched, epochs, nb, skip=(), start_epoch=0):
    out = []
    for epoch in range(start_epoch, epochs):
        for i in range(nb):
            if (epoch, i) in skip:
                continue
            it = sched.iteration(epoch, i)
            out.append((epoch, i, it.ni, list(it.lr), it.momentum, it.accumulate, it.step))
        sched.step()
    return out


def assert_same(mine, ref):
    assert len(mine) == len(ref)
    for a, b in zip(mine, ref):
        assert a[:3] == b[:3]
        ctx = (a[:3], a[3:], b[3:])
        assert all(type(x) is float for x in a[3]), ctx
        assert [x.hex() for x in a[3]] == [float(x).hex() for x in b[3]], ctx            # bit for bit
        assert (a[4] is None) == (b[4] is None), ctx
        if a[4] is not None:
            assert float(a[4]).hex() == float(b[4]).hex(), ctx
        assert a[5] == b[5] and a[6] == b[6], ctx


@pytest.mark.parametrize("nb,epochs", RUNS, ids=[f"nb{nb}" for nb, _ in RUNS])
@pytest.mark.parametrize("tbs", [16, 18, 64])
@pytest.mark.parametrize("adam", [False, True], ids=["sgd", "adam"])
@pytest.mark.parametrize("linear", [False, True], ids=["cos", "linear"])
@pytest.mark.parametrize("hyp", sorted(HYPS))
def test_schedule_equals_the_references_statements(hyp, linear, adam, tbs, nb, epochs):
    from multiyolov5_b200.train import LRSchedule
    h = HYPS[hyp]
    ref = R.run(h, epochs, nb, tbs, linear_lr=linear, adam=adam)
    sched = LRSchedule(h, epochs, nb, tbs, linear_lr=linear, optimizer="adam" if adam else "sgd")
    mine = schedule_records(sched, epochs, nb)
    assert_same(mine, ref)
    assert sched.nw < len(mine)                                  # the run goes past the warm-up


@pytest.mark.parametrize("start_epoch,resume_epochs", [(1, 6), (5, 6), (5, 3)], ids=["start1", "start5", "finetune_extension"])
@pytest.mark.parametrize("adam", [False, True], ids=["sgd", "adam"])
@pytest.mark.parametrize("linear", [False, True], ids=["cos", "linear"])
def test_resumed_schedule_equals_the_references(start_epoch, resume_epochs, adam, linear):
    """a run of 6 epochs of 300 batches, checkpointed after epoch start_epoch - 1 and resumed with `resume_epochs` (3 < start_epoch:
    the fine-tune extension to 3 + 4 epochs); batches skipped on both sides of the warm-up's end"""
    from multiyolov5_b200.train import LRSchedule
    nb, tbs = 300, 18
    skip = {(2, 199), (2, 200), (3, 5)}                          # ni 799, 800 (= nw: the warm-up's last iteration) and 905
    saved = {}
    R.run(SCRATCH, 6, nb, tbs, linear_lr=linear, adam=adam, skip=skip, on_epoch_end=lambda e, sd: saved.__setitem__(e, sd))
    sd = saved[start_epoch - 1]
    ref = R.run(SCRATCH, resume_epochs, nb, tbs, linear_lr=linear, adam=adam, start_epoch=start_epoch, optimizer_state=sd, skip=skip)
    sched = LRSchedule(SCRATCH, resume_epochs, nb, tbs, linear_lr=linear, optimizer="adam" if adam else "sgd", start_epoch=start_epoch,
                       param_groups=sd["param_groups"])
    assert sched.epochs == (resume_epochs + start_epoch - 1 if resume_epochs < start_epoch else resume_epochs)
    assert sched.last_epoch == start_epoch - 1
    mine = schedule_records(sched, sched.epochs, nb, skip, start_epoch)
    assert mine and mine[0][0] == start_epoch
    assert_same(mine, ref)


def test_start_epoch_zero_equals_a_fresh_run_with_skips():
    from multiyolov5_b200.train import LRSchedule
    skip = {(0, 0), (2, 199), (2, 200)}
    ref = R.run(SCRATCH, 4, 300, 16, skip=skip)
    assert_same(schedule_records(LRSchedule(SCRATCH, 4, 300, 16, start_epoch=0), 4, 300, skip), ref)


# ---- fit's bookkeeping ------------------------------------------------------------------------------------------------------------
class _Head(nn.Module):
    def __init__(self, nc=3, nl=3):
        super().__init__()
        self.nc, self.nl = nc, nl
        self.conv = nn.Conv2d(3, 4, 1)


class _SegHead(nn.Module):
    def __init__(self):
        super().__init__()
        self.c_out = 19
        self.bn = nn.BatchNorm2d(4)


class FakeModel(nn.Module):
    def __init__(self):
        super().__init__()
        self.model = nn.Sequential(_SegHead(), _Head())
        self.stride = torch.tensor([8., 16., 32.])
        self.names = ["a", "b", "c"]


class FakeTrainer:
    """records what fit hands the step; returns loss items derived from ni, so the running means are predictable"""
    log = []

    def __init__(self, model, hyp, batch_size, world_size=1, rank=-1, accumulate=1, optimizer="sgd", ema=None, quad=False,
                 multi_scale=None, **kw):
        self.model, self.hyp, self.batch_size, self.accumulate, self.optimizer = model, hyp, batch_size, accumulate, optimizer
        self.lr, self.momentum, self.compute_loss = [hyp["lr0"]] * 3, hyp["momentum"], object()
        self.steps = 0
        FakeTrainer.log = []
        FakeTrainer.instance = self

    def set_lr(self, a, b, c):
        self.lr = [a, b, c]

    def set_momentum(self, m):
        self.momentum = m

    def step(self, imgs, targets, segimgs, segtargets, ni=None):
        stepped = ni % self.accumulate == 0
        self.steps += stepped
        FakeTrainer.log.append((ni, tuple(self.lr), self.momentum, self.accumulate, stepped, len(imgs), len(segimgs)))
        return loss_items(ni), torch.tensor(0.25 * (ni % 5))

    def state_dict(self):
        return {"state": {}, "param_groups": [{"lr": lr, "momentum": self.momentum, "initial_lr": self.hyp["lr0"], "params": [k]}
                                              for k, lr in enumerate(self.lr)]}


def loss_items(ni):
    return torch.tensor([0.01 * (ni % 7), 0.02, 0.003 * (ni % 3), 0.5], dtype=torch.float32)


class Batches:
    """sizes[epoch][i] = images in batch i"""

    def __init__(self, sizes, seg=False):
        self.sizes, self.seg = sizes, seg

    def __len__(self):
        return len(self.sizes(0))

    def __call__(self, epoch):
        for b in self.sizes(epoch):
            x = torch.zeros((b, 3, 32, 64))
            yield (x, torch.zeros((b, 16, 32), dtype=torch.int64)) if self.seg else (x, torch.zeros((2 * b, 6)))


def _opt(**kw):
    o = dict(epochs=3, batch_size=4, img_size=[64, 64], linear_lr=False, adam=False, notest=False, nosave=False, evolve=False,
             multi_scale=False, quad=False, single_cls=False, resume=False, global_rank=-1, world_size=1, label_smoothing=0.0,
             weights="", cfg="")
    o.update(kw)
    return argparse.Namespace(**o)


HYP = dict(SCRATCH, box=0.05, cls=0.5, obj=1.0)


@pytest.fixture
def fake_env(monkeypatch):
    import multiyolov5_b200.test as T
    import multiyolov5_b200.train as TR
    calls = {"seg": [], "test": []}

    # fit validates after the epoch's scheduler step, which advanced calls["epoch"]
    def seg_validation(model, n_segcls, valloader, device, half_precision=True):
        calls["seg"].append(calls["epoch"] - 1)
        return calls["miou"](calls["epoch"] - 1)

    def test(data, batch_size=32, imgsz=640, model=None, single_cls=False, dataloader=None, save_dir=None, verbose=False, plots=True,
             compute_loss=None, **kw):
        assert plots is False and model is not None and compute_loss is FakeTrainer.instance.compute_loss
        calls["test"].append(calls["epoch"] - 1)
        return calls["results"](calls["epoch"] - 1), np.zeros(data["nc"]), (0, 0, 0)

    monkeypatch.setattr(TR, "Trainer", FakeTrainer)
    monkeypatch.setattr(T, "seg_validation", seg_validation)
    monkeypatch.setattr(T, "test", test)
    orig_step = TR.LRSchedule.step

    def step(self):
        calls["epoch"] += 1
        orig_step(self)
    monkeypatch.setattr(TR.LRSchedule, "step", step)
    return calls


def _fit(tmp_path, calls, opt, det, seg, start=0, miou=lambda e: 0.5, results=lambda e: (0.1, 0.2, 0.3, 0.4, 0.01, 0.02, 0.03)):
    from multiyolov5_b200.train import fit
    calls.update(epoch=start, miou=miou, results=results)
    return fit(FakeModel(), HYP, opt, det, seg, test_loader=[], segval_loader=[], save_dir=tmp_path, log_interval=2)


def test_skipped_batches_still_count_and_epochs_run_min_of_both_loaders(tmp_path, fake_env):
    """det batch 1 holds one image and seg batch 3 holds one image: both iterations are skipped, ni keeps counting them; the seg loader
    has 5 batches, the det loader 6 (nb), so an epoch trains min(6, 5) minus the skipped ones, and ni = i + 6 * epoch"""
    det = Batches(lambda e: [4, 1, 4, 4, 4, 4])
    seg = Batches(lambda e: [4, 4, 4, 1, 4], seg=True)
    _fit(tmp_path, fake_env, _opt(epochs=2), det, seg)
    nis = [r[0] for r in FakeTrainer.log]
    assert nis == [0, 2, 4, 6, 8, 10]
    from multiyolov5_b200.train import LRSchedule
    sched = LRSchedule(SCRATCH, 2, 6, 4)
    for r in FakeTrainer.log:
        e, i = divmod(r[0], 6)
        it = sched.iteration(e, i)
        assert r[1:5] == (it.lr, it.momentum, it.accumulate, it.step)
        if i == 4:
            sched.step()


def _fi(results, miou):
    from multiyolov5_b200.utils.metrics import fitness2
    return fitness2(np.array(results).reshape(1, -1), miou)


def test_validation_cadence_best_and_results_lines(tmp_path, fake_env):
    """42 epochs: seg validation on epoch 0 and on every epoch with epochs - epoch < 40 (3 .. 41), mIoU 0 on epochs 1 and 2; test every
    epoch; best.pt is the last epoch whose fitness2 reached the best; results.txt holds the reference's format applied to the numbers"""
    from multiyolov5_b200.models.experimental import load_checkpoint
    epochs = 42
    det = Batches(lambda e: [4, 4, 4])
    seg = Batches(lambda e: [4, 4, 4], seg=True)
    miou = lambda e: [0.3, 0.9, 0.9, 0.2, 0.95][e] if e < 5 else 0.1       # noqa: E731
    res = lambda e: (0.5, 0.5, 0.1 * (e % 3), 0.05, 0.1, 0.2, 0.3)          # noqa: E731
    out = _fit(tmp_path, fake_env, _opt(epochs=epochs), det, seg, miou=miou, results=res)
    assert fake_env["seg"] == [0] + list(range(3, epochs))
    assert fake_env["test"] == list(range(epochs))
    assert out == res(epochs - 1)
    fis = [_fi(res(e), miou(e) if e in fake_env["seg"] else 0) for e in range(epochs)]
    best_e = max(e for e in range(epochs) if fis[e] == max(fis))
    best = load_checkpoint(str(tmp_path / "weights" / "best.pt"))
    last = load_checkpoint(str(tmp_path / "weights" / "last.pt"))
    assert best["epoch"] == best_e == 4 and last["epoch"] == epochs - 1
    assert last["best_fitness"] == max(fis) and isinstance(last["best_fitness"], np.ndarray)
    lines = (tmp_path / "results.txt").read_text().splitlines()
    assert last["training_results"] == (tmp_path / "results.txt").read_text()
    assert len(lines) == epochs
    for e, line in enumerate(lines):
        nis = [e * 3 + i for i in range(3)]
        mloss, mseg = torch.zeros(4), torch.zeros(1)
        for i, ni in enumerate(nis):
            mloss = (mloss * i + loss_items(ni)) / (i + 1)
            mseg = (mseg * i + torch.tensor(0.25 * (ni % 5)) / 4) / (i + 1)
        s = ("%10s" * 2 + "%10.4g" * 7) % ("%g/%g" % (e, epochs - 1), "0G", *mloss, mseg, 8, 64)
        assert line == s + "%10.4g" * 7 % res(e)


@pytest.mark.parametrize("flags,saved", [({}, "every"), ({"nosave": True}, "final"), ({"nosave": True, "evolve": True}, "none"),
                                         ({"notest": True}, "every")], ids=["default", "nosave", "nosave_evolve", "notest"])
def test_notest_and_save_rules(tmp_path, fake_env, monkeypatch, flags, saved):
    from multiyolov5_b200.models.experimental import load_checkpoint
    det = Batches(lambda e: [4, 4])
    seg = Batches(lambda e: [4, 4], seg=True)
    written, orig = [], torch.save
    monkeypatch.setattr(torch, "save", lambda obj, f: (written.append((obj["epoch"], str(f)[-7:])), orig(obj, f)))
    out = _fit(tmp_path, fake_env, _opt(epochs=3, **flags), det, seg)
    assert fake_env["test"] == ([2] if flags.get("notest") else [0, 1, 2])
    lasts = [e for e, f in written if f == "last.pt"]
    assert lasts == {"every": [0, 1, 2], "final": [2], "none": []}[saved]
    assert (tmp_path / "weights" / "last.pt").exists() == (saved != "none")
    if flags.get("notest"):
        assert out == (0.1, 0.2, 0.3, 0.4, 0.01, 0.02, 0.03)
    if saved != "none":
        ck = load_checkpoint(str(tmp_path / "weights" / "last.pt"))
        assert list(ck) == ["epoch", "best_fitness", "training_results", "model", "ema", "updates", "optimizer", "wandb_id"]


@pytest.mark.parametrize("flag", ["bucket", "entity", "upload_dataset", "data"])
def test_flags_the_loop_cannot_honour_raise(tmp_path, fake_env, flag):
    with pytest.raises(NotImplementedError, match=flag):
        _fit(tmp_path, fake_env, _opt(**{flag: "x"}), Batches(lambda e: [4]), Batches(lambda e: [4], seg=True))


# ---- the seg epoch order ----------------------------------------------------------------------------------------------------------
class _FakeSegAug:
    """records the indices of each batch and draws ColorJitter's torch.randperm(4) per item, as SegAugmenter.draw does"""

    def __init__(self, n):
        self.cache = argparse.Namespace(n=n)
        self.batches, self.perms = [], []

    def __call__(self, indices, out_dtype):
        self.batches.append(list(indices))
        self.perms += [torch.randperm(4).tolist() for _ in indices]
        return indices


@pytest.mark.parametrize("drop_last", [False, True])
def test_seg_epoch_order_is_the_dataloaders(drop_last):
    from multiyolov5_b200.train import SegEpochBatches
    n, B = 23, 4
    aug = _FakeSegAug(n)
    sb = SegEpochBatches(aug, B, drop_last=drop_last)
    torch.manual_seed(7)
    for epoch in range(3):
        list(sb(epoch))
    torch.manual_seed(7)
    ref_batches, ref_perms = [], []
    for epoch in range(3):
        for idx in torch.utils.data.DataLoader(range(n), batch_size=B, shuffle=True, drop_last=drop_last):
            ref_batches.append(idx.tolist())
            ref_perms += [torch.randperm(4).tolist() for _ in idx]
    assert aug.batches == ref_batches and aug.perms == ref_perms
    assert len(sb) == (n // B if drop_last else -(-n // B)) == len(ref_batches) // 3
