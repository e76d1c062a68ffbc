"""CPU: the mapping between the reference's optimizer state dict (torch's `optimizer.state_dict()`, what its checkpoints hold in
ckpt['optimizer']) and the Trainer's flat buffers (multiyolov5_b200.train: reference_param_groups, optimizer_state_dict,
optimizer_state_from_dict).  The yardstick is a real torch optimizer built over the model as reference train.py:119-145 builds it."""
import copy

import pytest
import torch
import torch.nn as nn

CONFIGS = ["yolov5s_city_seg.yaml", "yolov5s_city_seg_base.yaml", "yolov5s_city_seg_bise.yaml", "yolov5s_city_seg_lab.yaml",
           "yolov5m_city_seg_lab.yaml"]
HYP = dict(lr0=0.01, momentum=0.937, weight_decay=5e-4)


def model_of(yml="yolov5s_city_seg.yaml", seed=0):
    from multiyolov5_b200.models.yolo import Model
    torch.manual_seed(seed)
    return Model(yml)


def reference_optimizer(kind, model, hyp=HYP):
    """torch.optim.SGD(nesterov) / Adam over pg0, + pg1 with weight decay, + pg2, and LambdaLR (train.py:119-145)"""
    pg0, pg1, pg2 = [], [], []
    for _, v in model.named_modules():                                        # the reference's loop, independent of the code under test
        if hasattr(v, "bias") and isinstance(v.bias, nn.Parameter):
            pg2.append(v.bias)
        if isinstance(v, nn.BatchNorm2d):
            pg0.append(v.weight)
        elif hasattr(v, "weight") and isinstance(v.weight, nn.Parameter):
            pg1.append(v.weight)
    if kind == "adam":
        opt = torch.optim.Adam(pg0, lr=hyp["lr0"], betas=(hyp["momentum"], 0.999))
    else:
        opt = torch.optim.SGD(pg0, lr=hyp["lr0"], momentum=hyp["momentum"], nesterov=True)
    opt.add_param_group({"params": pg1, "weight_decay": hyp["weight_decay"]})
    opt.add_param_group({"params": pg2})
    torch.optim.lr_scheduler.LambdaLR(opt, lr_lambda=lambda x: 1.0)
    return opt


def trained_state(kind, model, steps=2):
    opt = reference_optimizer(kind, model)
    g = torch.Generator().manual_seed(1)
    for it in range(steps):
        for j, x in enumerate(opt.param_groups):                               # warm-up as train.py:348-352 sets it
            x["lr"] = float(0.1 - 0.01 * it if j == 2 else 0.001 * (it + 1))
            if "momentum" in x:
                x["momentum"] = 0.8 + 0.05 * it
        for p in model.parameters():
            p.grad = torch.randn(p.shape, generator=g)
        opt.step()
    return opt, copy.deepcopy(opt.state_dict())


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


@pytest.mark.parametrize("yml", CONFIGS)
def test_reference_groups_cover_every_parameter_once_in_the_references_index_order(yml):
    from multiyolov5_b200.train import reference_param_groups
    model = model_of(yml)
    pgs = reference_param_groups(model)
    ids = [id(p) for pg in pgs for p in pg]
    assert len(ids) == len(set(ids)) == len(list(model.parameters()))
    opt = reference_optimizer("sgd", model)
    assert [[id(p) for p in g["params"]] for g in opt.param_groups] == [[id(p) for p in pg] for pg in pgs]
    names = {id(p): n for n, p in model.named_parameters()}
    bn = {id(m.weight) for m in model.modules() if isinstance(m, nn.BatchNorm2d)}
    assert all(id(p) in bn for p in pgs[0])
    assert all(names[id(p)].endswith(".weight") and id(p) not in bn for p in pgs[1])
    assert all(names[id(p)].endswith(".bias") for p in pgs[2])
    if yml == "yolov5s_city_seg.yaml":
        assert [len(pg) for pg in pgs] == [73, 79, 77]


@pytest.mark.parametrize("kind", ["sgd", "adam"])
def test_state_dict_to_flat_buffers_and_back_is_bit_exact(kind):
    """a real torch optimizer's state dict -> flat buffers (each parameter's slice holds its state) -> state dict: identical, including
    the param_groups' values, key order and initial_lr, and Adam's step tensors (CPU float32 scalars)"""
    from multiyolov5_b200.engine import flat_offsets
    from multiyolov5_b200.train import OPTIMIZER_STATE, optimizer_state_dict, optimizer_state_from_dict
    model = model_of()
    opt, sd = trained_state(kind, model)
    groups, steps, bufs = optimizer_state_from_dict(model, kind, sd)
    assert steps == (2 if kind == "adam" else 1)
    params = list(model.parameters())
    offsets, n = flat_offsets(params)
    for p, o in zip(params, offsets):
        for name in OPTIMIZER_STATE[kind]:
            assert torch.equal(bufs[name][o:o + p.numel()].view_as(p), opt.state[p][name])
    back = optimizer_state_dict(model, kind, groups, steps, bufs)
    same(back, sd)
    if kind == "adam":
        st = back["state"][0]["step"]
        assert st.dtype == torch.float32 and st.device.type == "cpu" and st.dim() == 0
    # before the first step torch has no state: an empty dict maps to zero buffers and back
    fresh = reference_optimizer(kind, model_of()).state_dict()
    g0, s0, b0 = optimizer_state_from_dict(model, kind, fresh)
    assert s0 == 0 and all(float(b.abs().sum()) == 0 for b in b0.values())
    same(optimizer_state_dict(model, kind, g0, s0, b0), fresh)


def test_invalid_state_dicts_raise_value_error():
    from multiyolov5_b200.train import optimizer_state_from_dict
    model = model_of()
    _, sgd = trained_state("sgd", model_of())
    _, adam = trained_state("adam", model_of())
    with pytest.raises(ValueError, match="sgd"):
        optimizer_state_from_dict(model, "adam", sgd)                            # kind mismatch, both ways
    with pytest.raises(ValueError, match="adam"):
        optimizer_state_from_dict(model, "sgd", adam)
    bad = copy.deepcopy(adam)
    bad["param_groups"][1]["params"] = bad["param_groups"][1]["params"][:-1]
    with pytest.raises(ValueError, match="group sizes"):
        optimizer_state_from_dict(model, "adam", bad)
    other = model_of("yolov5m_city_seg_lab.yaml")                               # the dict of another model
    with pytest.raises(ValueError, match="group sizes"):
        optimizer_state_from_dict(other, "sgd", sgd)
    bad = copy.deepcopy(sgd)
    bad["state"][80]["momentum_buffer"] = bad["state"][80]["momentum_buffer"].reshape(-1)
    with pytest.raises(ValueError, match="shape"):
        optimizer_state_from_dict(model, "sgd", bad)
    bad = copy.deepcopy(adam)
    bad["state"][100]["exp_avg_sq"] = torch.zeros(3)
    with pytest.raises(ValueError, match="shape"):
        optimizer_state_from_dict(model, "adam", bad)
    bad = copy.deepcopy(adam)
    bad["state"][7]["step"] = torch.tensor(3.0)
    with pytest.raises(ValueError, match="step counts differ"):
        optimizer_state_from_dict(model, "adam", bad)
    bad = copy.deepcopy(sgd)
    del bad["state"][3]
    with pytest.raises(ValueError, match="state for"):
        optimizer_state_from_dict(model, "sgd", bad)
    bad = copy.deepcopy(sgd)
    for g in bad["param_groups"]:
        g["nesterov"] = False
    with pytest.raises(ValueError, match="nesterov"):
        optimizer_state_from_dict(model, "sgd", bad)
    bad = copy.deepcopy(adam)
    bad["param_groups"][2]["betas"] = (0.9, 0.999)
    with pytest.raises(ValueError, match="betas"):
        optimizer_state_from_dict(model, "adam", bad)


@pytest.mark.parametrize("kind", ["sgd", "adam"])
def test_param_group_keys_are_those_of_the_installed_torch(kind):
    """the groups a Trainer writes before any checkpoint was loaded: a real torch optimizer's keys, defaults and values (after LambdaLR)"""
    from multiyolov5_b200.train import default_param_groups
    groups = default_param_groups(kind, HYP)
    ref = reference_optimizer(kind, model_of()).state_dict()["param_groups"]
    same(groups, [{k: v for k, v in g.items() if k != "params"} for g in ref])
    for g in groups:
        assert "initial_lr" in g and g["initial_lr"] == HYP["lr0"]
    with pytest.raises(ValueError):
        default_param_groups("rmsprop", HYP)


def test_frozen_parameters_are_refused():
    """the reference numbers frozen parameters in its groups; the flat buffers do not hold them: a clear ValueError, not a KeyError"""
    from multiyolov5_b200.train import default_param_groups, optimizer_state_dict, optimizer_state_from_dict
    model = model_of()
    _, sd = trained_state("sgd", model_of())
    next(model.parameters()).requires_grad_(False)
    with pytest.raises(ValueError, match="frozen"):
        optimizer_state_from_dict(model, "sgd", sd)
    with pytest.raises(ValueError, match="frozen"):
        optimizer_state_dict(model, "sgd", default_param_groups("sgd", HYP), 0, {})


GOLD = __import__("os").path.join(__import__("os").path.dirname(__file__), "golden", "optim_cases.pt")


@pytest.mark.parametrize("kind", ["sgd", "adam"])
def test_reference_run_numbers_parameters_as_this_model_does(kind):
    """tests/golden/optim_cases.pt (oracle/make_golden_optim.py: the unmodified reference's train.train() for one CPU epoch): the names of
    each group of the optimizer it built, in index order, equal this model's reference_param_groups; every state entry of its last.pt
    has the keys torch writes and this model's parameter shape at that index; its param_groups (values and Python / numpy types) pass
    through the flat conversion unchanged; Adam's steps are equal CPU float32 scalars"""
    from multiyolov5_b200.train import OPTIMIZER_STATE, optimizer_state_dict, optimizer_state_from_dict, reference_param_groups
    case = torch.load(GOLD, map_location="cpu", weights_only=False)[kind]
    model = model_of()
    names = {id(p): n for n, p in model.named_parameters()}
    pgs = reference_param_groups(model)
    assert [[names[id(p)] for p in pg] for pg in pgs] == case["names"]
    assert sorted(n for g in case["names"] for n in g) == sorted(names.values())
    params = [p for pg in pgs for p in pg]
    assert sorted(case["state"]) == list(range(len(params)))
    for i, p in enumerate(params):
        st = case["state"][i]
        assert list(st) == (["step"] if kind == "adam" else []) + list(OPTIMIZER_STATE[kind])
        for k in OPTIMIZER_STATE[kind]:
            assert st[k]["shape"] == tuple(p.shape) and st[k]["dtype"] == "torch.float32", (i, k)
        if kind == "adam":
            assert st["step"]["value"].dtype == torch.float32 and st["step"]["value"].dim() == 0
            assert float(st["step"]["value"]) == float(case["state"][0]["step"]["value"]) >= 1
    sd = {"state": {}, "param_groups": case["param_groups"]}
    groups, steps, bufs = optimizer_state_from_dict(model, kind, sd)
    same(optimizer_state_dict(model, kind, groups, steps, bufs), sd)
