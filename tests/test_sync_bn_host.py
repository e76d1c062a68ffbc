"""CPU: the semantics of the reference's --sync-bn (train.py:190-193, torch.nn.SyncBatchNorm) as the train plans implement them.
The fp64 restatement (oracle/restate_sync_bn.py) against torch's BatchNorm over the concatenated batch; the decision which process group
the train plans synchronise over (parallel.bn_sync_group); the optimizer's parameter groups of a converted model; a reference checkpoint
written by a --sync-bn run (tests/golden/ref_ckpt_tiny_syncbn.pt, oracle/make_golden_syncbn.py)."""
import os

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp
import torch.nn as nn
import torch.nn.functional as F

from oracle import restate, synth
from oracle.restate_sync_bn import sync_bn_backward, sync_bn_forward


@pytest.mark.parametrize("images", [[3], [2, 1], [1, 3, 2, 1]])
def test_restatement_equals_batch_norm_over_the_whole_batch(images):
    """per-rank batches of unequal size: outputs, input gradients, summed d weight / d bias and running statistics are those of
    F.batch_norm + autograd over the concatenation, which is what SyncBatchNorm computes"""
    g = torch.Generator().manual_seed(3)
    C, H, W = 6, 5, 7
    xs = [torch.randn(b, C, H, W, generator=g, dtype=torch.float64) * 2 + 5 for b in images]
    dys = [torch.randn(b, C, H, W, generator=g, dtype=torch.float64) for b in images]
    w = torch.rand(C, generator=g, dtype=torch.float64) + 0.5
    b = torch.randn(C, generator=g, dtype=torch.float64)
    rm0, rv0 = torch.randn(C, generator=g, dtype=torch.float64), torch.rand(C, generator=g, dtype=torch.float64) + 0.5
    ys, ctx, rm, rv = sync_bn_forward(xs, w, b, rm0, rv0)
    dxs, dws, dbs = sync_bn_backward(dys, ctx)

    x = torch.cat(xs).requires_grad_(True)
    wr, br = w.clone().requires_grad_(True), b.clone().requires_grad_(True)
    rm_t, rv_t = rm0.clone(), rv0.clone()
    y = F.batch_norm(x, rm_t, rv_t, wr, br, training=True, momentum=0.03, eps=1e-3)
    y.backward(torch.cat(dys))
    tol = dict(rtol=1e-10, atol=1e-10)
    assert torch.allclose(torch.cat(ys), y.detach(), **tol)
    assert torch.allclose(torch.cat(dxs), x.grad, **tol)
    assert torch.allclose(sum(dws), wr.grad, **tol) and torch.allclose(sum(dbs), br.grad, **tol)
    assert torch.allclose(rm, rm_t, **tol) and torch.allclose(rv, rv_t, **tol)


def _tiny_model():
    from multiyolov5_b200.models.yolo import Model
    cfg = synth.load_cfg("yolov5s_city_seg.yaml")
    cfg["width_multiple"] = 0.25
    torch.manual_seed(0)
    return Model(cfg)


def _bns(model):
    return [m for m in model.modules() if isinstance(m, nn.modules.batchnorm._BatchNorm)]


def test_decision_without_dist_is_local_and_rejects_a_mix():
    from multiyolov5_b200.parallel import bn_sync_group
    assert not (dist.is_available() and dist.is_initialized())
    model = _tiny_model()
    assert bn_sync_group(_bns(model)) is None                                   # plain BatchNorm
    conv = nn.SyncBatchNorm.convert_sync_batchnorm(model)
    assert bn_sync_group(_bns(conv)) is None                                    # torch: no process group, no exchange
    bns = _bns(conv)
    mixed = bns[:3] + [nn.BatchNorm2d(bns[3].num_features)] + bns[4:]
    with pytest.raises(ValueError, match="SyncBatchNorm"):
        bn_sync_group(mixed)
    a, b = nn.SyncBatchNorm(8, process_group=object()), nn.SyncBatchNorm(8)
    with pytest.raises(ValueError, match="different process groups"):
        bn_sync_group([a, b])


def _decision_worker(rank, world, init, ret):
    dist.init_process_group("gloo", init_method=init, rank=rank, world_size=world)
    try:
        from multiyolov5_b200.parallel import bn_sync_group
        bns = _bns(nn.SyncBatchNorm.convert_sync_batchnorm(_tiny_model()))
        try:
            ret[rank] = ("group", bn_sync_group(bns) is not None)
        except ValueError as e:
            ret[rank] = ("ValueError", str(e))
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("world", [1, 2])
def test_decision_over_gloo(world, tmp_path):
    """world size 1: no exchange (torch's need_sync); world size 2 over gloo: ValueError, the library exchanges over NCCL only"""
    ret = mp.Manager().dict()
    init = "file://" + os.path.join(str(tmp_path), "store")
    ctx = mp.start_processes(_decision_worker, args=(world, init, ret), nprocs=world, join=False, start_method="spawn")
    for _ in range(world):                     # join(timeout) returns when one process ends
        if ctx.join(timeout=300):
            break
    for p in ctx.processes:
        if p.is_alive():
            p.terminate()
    assert len(ret) == world and all(ctx.processes[r].exitcode == 0 for r in range(world)), dict(ret)
    for r in range(world):
        if world == 1:
            assert ret[r] == ("group", False)
        else:
            assert ret[r][0] == "ValueError" and "gloo" in ret[r][1] and "NCCL" in ret[r][1]


def test_parameter_groups_and_optimizer_numbering_survive_conversion():
    """the reference builds its optimizer before convert_sync_batchnorm (train.py:108-137 vs :190-193): a Trainer built after the
    conversion must number the parameters as that optimizer does"""
    from multiyolov5_b200.train import default_param_groups, optimizer_state_dict, parameter_groups, reference_param_groups
    model = _tiny_model()
    before = [[id(p) for p in pg] for pg in reference_param_groups(model)]
    groups_before = parameter_groups(model)
    n = sum((p.numel() + 3) // 4 * 4 for p in model.parameters())
    buf = {"momentum_buffer": torch.arange(n, dtype=torch.float32)}
    hyp = {"lr0": 0.01, "momentum": 0.937, "weight_decay": 5e-4}
    sd_before = optimizer_state_dict(model, "sgd", default_param_groups("sgd", hyp), 1, buf)
    conv = nn.SyncBatchNorm.convert_sync_batchnorm(model)
    assert sum(isinstance(m, nn.SyncBatchNorm) for m in conv.modules()) == len(before[0]) > 0
    assert [[id(p) for p in pg] for pg in reference_param_groups(conv)] == before
    assert parameter_groups(conv) == groups_before
    sd_after = optimizer_state_dict(conv, "sgd", default_param_groups("sgd", hyp), 1, buf)
    assert sd_after["param_groups"] == sd_before["param_groups"]
    assert sd_after["state"].keys() == sd_before["state"].keys()
    assert all(torch.equal(sd_after["state"][k]["momentum_buffer"], sd_before["state"][k]["momentum_buffer"]) for k in sd_before["state"])


def test_attempt_load_of_a_sync_bn_checkpoint_matches_reference_output():
    """ckpt['model'] of a --sync-bn run pickles SyncBatchNorm modules; attempt_load resolves them, and the weights reproduce what the
    reference's loading recipe computed from the same file (oracle/make_golden_syncbn.py)"""
    from multiyolov5_b200.models.experimental import attempt_load
    from multiyolov5_b200.models.yolo import Model
    from multiyolov5_b200.plan import build_plan
    m = attempt_load(os.path.join(synth.GOLDEN_DIR, "ref_ckpt_tiny_syncbn.pt"), map_location="cpu")
    g = np.load(os.path.join(synth.GOLDEN_DIR, "ref_ckpt_tiny_syncbn_out.npz"))
    assert isinstance(m, Model) and not m.training and next(m.parameters()).dtype == torch.float32
    assert sum(isinstance(x, nn.SyncBatchNorm) for x in m.modules()) == int(g["n_sync"]) == 73
    assert list(m.names) == list(g["names"]) and np.array_equal(m.stride.numpy(), g["stride"])
    assert len(build_plan(m, 1, 64, 64).ops) == len(build_plan(Model(m.yaml), 1, 64, 64).ops)
    sd = {k: v.float() for k, v in m.state_dict().items()}
    out = restate.model_forward(dict(m.yaml), sd, synth.synth_image(1, 64, 64, seed=5))
    seg = out["seg"][:, :, ::2, ::2]
    assert float((seg - torch.from_numpy(g["seg_sub"])).abs().max()) < 1e-5 * max(1.0, float(np.abs(g["seg_sub"]).max()))
    assert float((out["z"] - torch.from_numpy(g["z"])).abs().max()) < 1e-5 * float(np.abs(g["z"]).max())
