"""GPU: synchronised BatchNorm in the train plans (the reference's --sync-bn, train.py:190-193; torch.nn.SyncBatchNorm semantics,
oracle/restate_sync_bn.py).  One-GPU rank emulation (myolo_plan_set_bn_sync with image groups) runs the multi-rank arithmetic through the
real executor wiring and must equal BatchNorm over the whole batch; a one-rank NCCL process group runs the real exchanges and must leave
every result as the unsynchronised plan computes it.

Batch statistics and parameter gradients are reduced with fp32 atomics, so two runs of the same plan may differ in the last bits.  The
yardstick of every comparison is that run-to-run spread of the plain plan, measured in the same test: "bit identical" below means
identical whenever the plain plan repeats itself bit for bit, and within its own spread otherwise."""
import os

import numpy as np
import pytest
import torch
import torch.multiprocessing as mp

from oracle import synth

pytestmark = pytest.mark.gpu

CASES = {"s_psp": "yolov5s_city_seg.yaml", "m_lab": "yolov5m_city_seg_lab.yaml"}


def rel_f(a, b):
    a = a.double(); b = b.double()
    return float((a - b).norm() / (b.norm() + 1e-30))


def make_model(tag, sync_layers=False):
    from multiyolov5_b200.models.yolo import Model
    cfg = synth.load_cfg(CASES[tag])
    sd = synth.synth_state_dict(synth.load_manifest(tag), cfg, seed=1, gain=1.0)
    model = Model(CASES[tag])
    model.load_state_dict(sd)
    if sync_layers:
        model = torch.nn.SyncBatchNorm.convert_sync_batchnorm(model)
    return model.cuda().train(), cfg, sd


def train_pass(model, x, Rs, S, comm=None, rank_images=None):
    """one train forward + backward with the fixed cotangents; the plan's BatchNorm synchronised as given.  Head outputs, gradients and
    running statistics on the host."""
    eng = model.engine()
    B, _, H, W = x.shape
    p = eng.train_plan_for(B, H, W)
    eng.ensure_flat_grads()
    eng.prepare_train_plan(p)
    if comm is not None or rank_images is not None:
        eng.set_bn_sync(p, comm=comm, rank_images=rank_images)
    raws, seg = model(x)
    segs = seg if isinstance(seg, list) else [seg]
    loss = sum((r * R).sum() for r, R in zip(raws, Rs)) + sum((g * Sk).sum() for g, Sk in zip(segs, S))
    loss.backward()
    torch.cuda.synchronize()
    return {"out": [t.detach().float().cpu() for t in list(raws) + segs],
            "grad": {n: q.grad.detach().cpu().clone() for n, q in model.named_parameters()},
            "running": {k: v.detach().float().cpu().clone() for k, v in model.state_dict().items() if "running_" in k},
            "nbt": {k: int(v) for k, v in model.state_dict().items() if k.endswith("num_batches_tracked")}}


def probes(B, H, W, tag, seed=11):
    gen = torch.Generator().manual_seed(seed)
    shapes = [(B, 3, H // s, W // s, 15) for s in (8, 16, 32)]
    Rs = [(torch.randn(sh, generator=gen) * 4.0).cuda() for sh in shapes]
    S = [(torch.randn((B, 19, H, W), generator=gen) * 0.05).cuda()]
    return Rs, S


def spread(a, b):
    """(outputs: max rel. Frobenius, gradients: median rel. Frobenius, running statistics: max rel. max-abs) of run a against run b"""
    o = max(rel_f(x, y) for x, y in zip(a["out"], b["out"]))
    g = float(np.median([rel_f(a["grad"][k], v) for k, v in b["grad"].items() if v.norm() > 1e-8]))
    r = max(float((a["running"][k] - v).abs().max()) / (float(v.abs().max()) + 1e-12) for k, v in b["running"].items())
    return np.array([o, g, r])


def assert_identical_up_to_repeat(diff, noise, what):
    for d, n, name in zip(diff, noise, ("outputs", "gradients", "running statistics")):
        if n == 0.0:
            assert d == 0.0, (what, name, d)
        else:
            assert d <= 3 * n, (what, name, d, n)


@pytest.mark.parametrize("tag", list(CASES))
def test_rank_emulation_equals_whole_batch_batch_norm(tag):
    """B = 4 split into emulated ranks of [2, 2] and [3, 1] images: global count, statistics combined over the groups, backward sums
    summed over the groups.  Torch's SyncBatchNorm over those ranks is BatchNorm over the whole batch, i.e. the plain plan.  [4] is the
    plain plan launch for launch."""
    B, H, W = 4, 128, 256
    x = synth.synth_image(B, H, W, seed=5).cuda()
    Rs, S = probes(B, H, W, tag)
    plain = train_pass(make_model(tag)[0], x, Rs, S)
    noise = spread(train_pass(make_model(tag)[0], x, Rs, S), plain)
    for groups in ([2, 2], [3, 1], [4]):
        model = make_model(tag)[0]
        run = train_pass(model, x, Rs, S, rank_images=groups)
        assert model.engine().last_plan.bn_sync == ("ranks", tuple(groups))
        assert run["nbt"] == plain["nbt"] and set(run["nbt"].values()) == {1}
        diff = spread(run, plain)
        print(f"\n{tag} {groups}: outputs / gradients / running stats {np.round(diff, 8)} (plain run to run {np.round(noise, 8)})")
        if groups == [4]:
            assert_identical_up_to_repeat(diff, noise, groups)
        else:   # another summation order of the statistics (shift value and partial sums per group): fp32 rounding, amplified downstream
            assert diff[0] <= max(3 * noise[0], 2e-3) and diff[1] <= max(3 * noise[1], 1e-2) and diff[2] <= max(3 * noise[2], 1e-4), \
                (groups, diff, noise)


@pytest.mark.parametrize("tag", list(CASES))
def test_rank_emulation_of_the_golden_batch_matches_the_reference(tag):
    """the reference's own train-mode Model + autograd on two images (tests/golden/train_<tag>.npz, oracle/make_golden.py gen_train) is
    what SyncBatchNorm over two ranks of one image each computes.  With rank_images = [1, 1] the plan is as far from the reference as the
    plain plan on the same batch (fp16 storage; BatchNorm over the 2 x 3 map of P5 amplifies its rounding), within the train parity
    tests' sanity bounds (gradient norms median 0.25 / worst 0.40), and its running statistics match"""
    from oracle.digest import train_probe_tensors
    g = np.load(os.path.join(synth.GOLDEN_DIR, f"train_{tag}.npz"))
    x = synth.synth_image(2, 64, 96, seed=5).cuda()
    shapes_raw = [tuple(g[f"raw{i}"].shape) for i in range(3)]
    Rs, Ss = train_probe_tensors(shapes_raw, [(2, 19, 64, 96)])

    def errors(run):
        fwd = max(rel_f(run["out"][i], torch.from_numpy(g[f"raw{i}"])) for i in range(3))
        grd = [abs(float(run["grad"][str(n)].double().norm()) - d[0]) / max(d[0], 1e-12) for n, d in zip(g["grad_names"], g["grad_digest"])]
        return fwd, grd
    plain_fwd, plain_grd = errors(train_pass(make_model(tag)[0], x, [r.cuda() for r in Rs], [s.cuda() for s in Ss]))
    run = train_pass(make_model(tag)[0], x, [r.cuda() for r in Rs], [s.cuda() for s in Ss], rank_images=[1, 1])
    fwd, errs = errors(run)
    print(f"\n{tag} [1, 1] vs reference: forward {fwd:.3e} (plain plan {plain_fwd:.3e}), gradient norms median {np.median(errs):.3e} "
          f"worst {max(errs):.3e} (plain plan {np.median(plain_grd):.3e} / {max(plain_grd):.3e})")
    assert fwd <= 1.5 * plain_fwd + 1e-2, (fwd, plain_fwd)
    assert float(np.median(errs)) <= 1.5 * float(np.median(plain_grd)) + 1e-2, (np.median(errs), np.median(plain_grd))
    assert len(errs) > 150 and float(np.median(errs)) < 0.25 and max(errs) < 0.40, (float(np.median(errs)), max(errs))
    off = 0
    for n in [str(v) for v in g["bn_names"]]:
        rm, rv = run["running"][n + ".running_mean"], run["running"][n + ".running_var"]
        c = rm.numel()
        assert np.allclose(rm.numpy(), g["bn_mean"][off:off + c], rtol=2e-2, atol=2e-3), n
        assert np.allclose(rv.numpy(), g["bn_var"][off:off + c], rtol=2e-2, atol=2e-3), n
        off += c
    assert off == g["bn_mean"].size


def _one_rank_nccl_worker(rank, store, ret):
    import torch.distributed as dist
    from datetime import timedelta
    torch.cuda.set_device(0)
    dist.init_process_group("nccl", init_method="file://" + store, rank=0, world_size=1, timeout=timedelta(seconds=120),
                            device_id=torch.device("cuda", 0))
    try:
        from multiyolov5_b200.parallel import bn_sync_group, nccl_comm_ptr
        dist.all_reduce(torch.zeros(1, device="cuda"))           # torch creates the communicator at the first collective
        comm = nccl_comm_ptr()
        assert comm is not None
        B, H, W = 4, 128, 256
        x = synth.synth_image(B, H, W, seed=5).cuda()
        Rs, S = probes(B, H, W, "s_psp")
        plain = train_pass(make_model("s_psp")[0], x, Rs, S)
        noise = spread(train_pass(make_model("s_psp")[0], x, Rs, S), plain)
        model = make_model("s_psp")[0]
        runs = [train_pass(model, x, Rs, S, comm=comm)]
        model.zero_grad(set_to_none=False)
        runs.append(train_pass(model, x, Rs, S))                  # second step on the same (eager) plan, running statistics moved twice
        conv = make_model("s_psp", sync_layers=True)[0]          # torch at world size 1: no exchange, plain BatchNorm
        ret["converted_group"] = bn_sync_group([m for m in conv.modules() if isinstance(m, torch.nn.SyncBatchNorm)]) is None
        ret["bn_sync"] = model.engine().last_plan.bn_sync[0]
        ret["diff"], ret["noise"] = spread(runs[0], plain).tolist(), noise.tolist()
        ret["finite"] = all(bool(torch.isfinite(t).all()) for t in runs[1]["out"])
        ret["nbt"] = sorted(set(runs[1]["nbt"].values()))
    finally:
        dist.destroy_process_group()


def test_one_rank_nccl_exchange_leaves_the_plan_unchanged(tmp_path):
    """a real NCCL process group of one rank (file store: no host or port involved): the plan all-gathers one record per BN layer and
    all-reduces the backward sums over it.  Forward, backward and running statistics are the unsynchronised plan's."""
    ctx = mp.get_context("spawn")
    ret = ctx.Manager().dict()
    pc = mp.start_processes(_one_rank_nccl_worker, args=(str(tmp_path / "store"), ret), nprocs=1, join=False, start_method="spawn")
    done = pc.join(timeout=900)
    if not done:
        for p in pc.processes:
            p.terminate()
    assert done and pc.processes[0].exitcode == 0, dict(ret)
    print(f"\none-rank NCCL vs plain: {np.round(ret['diff'], 8)} (plain run to run {np.round(ret['noise'], 8)})")
    assert ret["bn_sync"] == "nccl" and ret["converted_group"] and ret["finite"] and ret["nbt"] == [2]
    assert_identical_up_to_repeat(ret["diff"], ret["noise"], "one-rank NCCL")


def test_converted_model_at_world_size_one_trains_and_infers_like_the_plain_model():
    """without a process group, SyncBatchNorm is F.batch_norm (torch's need_sync): a Trainer step of a converted model equals the plain
    model's; inference folds SyncBatchNorm like BatchNorm2d, bit for bit, also for a reference checkpoint of a --sync-bn run"""
    from multiyolov5_b200.models.experimental import attempt_load
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

    def step(convert):
        model, cfg, _ = make_model("s_psp", sync_layers=convert)
        hyp = dict(lr0=0.01, momentum=0.937, weight_decay=5e-4, box=0.05, cls=0.5, cls_pw=1.0, obj=1.0, obj_pw=1.0, anchor_t=4.0, fl_gamma=0.0)
        tr = Trainer(model, scale_hyp(hyp, nl=3, nc=cfg["nc"], imgsz=256, total_batch_size=4), batch_size=B, init_scale=2.0 ** 10)
        assert not tr.sync_bn
        items, segloss = tr.step(imgs, targets, segimgs, mask)
        torch.cuda.synchronize()
        return {"out": [items.float().cpu(), segloss.float().cpu().view(1)],
                "grad": {n: q.detach().cpu().clone() for n, q in model.named_parameters()},          # the stepped parameters
                "running": {k: v.detach().float().cpu().clone() for k, v in model.state_dict().items() if "running_" in k}}
    plain = step(False)
    noise = spread(step(False), plain)
    diff = spread(step(True), plain)
    print(f"\nTrainer.step converted vs plain: {np.round(diff, 8)} (plain run to run {np.round(noise, 8)})")
    assert_identical_up_to_repeat(diff, noise, "converted Trainer.step")

    from multiyolov5_b200.models.yolo import Model
    x = synth.synth_image(1, 64, 64, seed=5).cuda()
    sync_m = attempt_load(os.path.join(synth.GOLDEN_DIR, "ref_ckpt_tiny_syncbn.pt")).cuda()
    assert any(isinstance(m, torch.nn.SyncBatchNorm) for m in sync_m.modules())
    plain_m = Model(sync_m.yaml)                                  # the same weights with plain BatchNorm2d
    plain_m.load_state_dict(sync_m.state_dict())
    plain_m = plain_m.cuda().eval()
    assert not any(isinstance(m, torch.nn.SyncBatchNorm) for m in plain_m.modules())
    with torch.no_grad():
        (za, _), sa = plain_m(x)
        (zb, _), sb = sync_m(x)
    assert torch.equal(za, zb) and torch.equal(sa, sb)
    a, b = make_model("s_psp")[0].eval(), make_model("s_psp", sync_layers=True)[0].eval()
    x = synth.synth_image(2, 128, 256, seed=3).cuda()
    with torch.no_grad():
        (za, _), sa = a(x)
        (zb, _), sb = b(x)
    assert torch.equal(za, zb) and torch.equal(sa, sb)


def test_converting_after_the_train_plans_were_built_raises():
    """convert_sync_batchnorm replaces the BatchNorm modules; a train plan built from the old ones must not keep training with them"""
    from multiyolov5_b200 import _lib
    model = make_model("s_psp")[0]
    x = synth.synth_image(2, 64, 128, seed=5).cuda()
    out = model(x)
    (out[1].sum() * 1e-3).backward()
    torch.nn.SyncBatchNorm.convert_sync_batchnorm(model)
    with pytest.raises(_lib.MyoloError, match="BatchNorm layers were replaced"):
        model(x)


def test_rank_emulation_rejects_bad_groups():
    from multiyolov5_b200 import _lib
    model = make_model("s_psp")[0]
    eng = model.engine()
    p = eng.train_plan_for(4, 64, 128)
    for groups in ([2, 1], [4, 0], [1, 1, 1, 2]):
        with pytest.raises(_lib.MyoloError):
            eng.set_bn_sync(p, rank_images=groups)
    eng.set_bn_sync(p, rank_images=[1, 3])
    with pytest.raises(_lib.MyoloError, match="synchronises"):
        eng.set_defer_running(p)


def _two_rank_worker(rank, store, ret):
    import torch.distributed as dist
    from datetime import timedelta
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", init_method="file://" + store, rank=rank, world_size=2, timeout=timedelta(seconds=120),
                            device_id=torch.device("cuda", rank))
    try:
        B, H, W = 4, 128, 256
        x = synth.synth_image(B, H, W, seed=5).cuda()
        Rs, S = probes(B, H, W, "s_psp")
        sl = slice(2 * rank, 2 * rank + 2)
        model = make_model("s_psp", sync_layers=True)[0]          # Engine.prepare_train_plan hands the group's communicator over
        run = train_pass(model, x[sl].contiguous(), [r[sl].contiguous() for r in Rs], [s[sl].contiguous() for s in S])
        assert model.engine().last_plan.bn_sync[0] == "nccl"
        for _ in range(2):
            model.zero_grad(set_to_none=False)
            last = train_pass(model, x[sl].contiguous(), [r[sl].contiguous() for r in Rs], [s[sl].contiguous() for s in S])
        ret[rank] = {"out": run["out"], "grad": run["grad"], "running": run["running"], "running_last": last["running"]}
    finally:
        dist.destroy_process_group()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_two_nccl_ranks_equal_the_rank_emulation_of_the_whole_batch(tmp_path):
    """two processes, half of the batch each, a converted model: outputs, summed gradients and running statistics against one process
    emulating the same two ranks over the whole batch; running statistics identical across the ranks after several steps"""
    ctx = mp.get_context("spawn")
    ret = ctx.Manager().dict()
    pc = mp.start_processes(_two_rank_worker, args=(str(tmp_path / "store"), ret), nprocs=2, join=False, start_method="spawn")
    done = False
    for _ in range(2):
        done = pc.join(timeout=900)
        if done:
            break
    if not done:
        for p in pc.processes:
            p.terminate()
    assert done and all(p.exitcode == 0 for p in pc.processes)
    B, H, W = 4, 128, 256
    x = synth.synth_image(B, H, W, seed=5).cuda()
    Rs, S = probes(B, H, W, "s_psp")
    emu = train_pass(make_model("s_psp")[0], x, Rs, S, rank_images=[2, 2])
    r0, r1 = ret[0], ret[1]
    both = {"out": [torch.cat([a, b]) for a, b in zip(r0["out"], r1["out"])],
            "grad": {k: r0["grad"][k] + r1["grad"][k] for k in r0["grad"]}, "running": r0["running"]}
    diff = spread(both, emu)
    print(f"\ntwo NCCL ranks vs rank emulation: {np.round(diff, 8)}")
    assert diff[0] <= 2e-3 and diff[1] <= 1e-2 and diff[2] <= 1e-4, diff
    assert all(torch.equal(r0["running_last"][k], r1["running_last"][k]) for k in r0["running_last"])
