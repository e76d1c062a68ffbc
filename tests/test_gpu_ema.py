"""GPU: the device ModelEMA (myolo_ema_update behind utils.torch_utils.ModelEMA) bit for bit against the reference's per-entry statements
`v *= d; v += (1. - d) * msd[k]` (utils/torch_utils.py:297-300) run by torch on the card, in fp32 and after the reference's ema.half();
the replay of tests/golden/ema_cases.pt; the Trainer's update after every optimizer step; and evaluation of the EMA, whose anchors move."""
import copy
import os

import numpy as np
import pytest
import torch

from oracle import make_golden_ema as G
from oracle import synth

pytestmark = pytest.mark.gpu
HYP = dict(lr0=0.01, momentum=0.937, weight_decay=5e-4, box=0.05, cls=0.5, cls_pw=1.0, obj=1.0, obj_pw=1.0, anchor_t=4.0, fl_gamma=0.0)


def reference_update(ema_sd, msd, d):
    """the reference's loop over the EMA's floating-point entries, as torch runs it on the card"""
    with torch.no_grad():
        for k, v in ema_sd.items():
            if v.dtype.is_floating_point:
                v *= d
                v += (1. - d) * msd[k].detach()


def launch(segments, d):
    from multiyolov5_b200 import _lib
    from multiyolov5_b200.utils.torch_utils import ema_chunks
    chunks = ema_chunks([(v.data_ptr(), s.data_ptr(), v.numel(), _lib.torch_dtype_code(v.dtype)) for v, s in segments])
    arr = (_lib.EmaChunk * len(chunks))(*[_lib.EmaChunk(*c) for c in chunks])
    table = torch.frombuffer(bytearray(arr), dtype=torch.uint8).cuda()
    _lib.check(_lib.lib().myolo_ema_update(_lib.ptr(table), len(chunks), d, _lib.stream_ptr()))
    torch.cuda.synchronize()


@pytest.mark.parametrize("dtype", [torch.float32, torch.float16], ids=["fp32", "fp16"])
def test_kernel_is_bit_identical_to_the_references_statements(dtype):
    """odd sizes (1 element, every n % 4, around the chunk size), a segment 1 element off its allocation (the element-by-element path)
    and one aligned; at every update count of the decay ramp the fp32 / fp16 EMA equals torch's three statements bit for bit"""
    from multiyolov5_b200.utils.torch_utils import ModelEMA
    decay = ModelEMA(torch.nn.Linear(1, 1)).decay
    gen = torch.Generator(device="cuda").manual_seed(3)
    sizes = [1, 2, 3, 5, 7, 8191, 8192, 8193, 100003]
    base = [torch.randn(n + 1, device="cuda", generator=gen).to(dtype) * 4 for n in sizes]
    emas = [b[1:] if i % 2 else b[:-1] for i, b in enumerate(base)]            # odd ones: 2 / 4 bytes off the allocation
    srcs = [torch.randn(n + 1, device="cuda", generator=gen)[int(i % 3 == 2):][:n] for i, n in enumerate(sizes)]
    refs = [e.clone() for e in emas]
    for updates in (1, 2, 7, 500, 2000, 3000, 10 ** 5, 10 ** 6):
        d = decay(updates)
        for s in srcs:
            s.add_(torch.randn(s.shape, device="cuda", generator=gen) * 0.1)
        launch(list(zip(emas, srcs)), d)
        reference_update({str(i): r for i, r in enumerate(refs)}, {str(i): s for i, s in enumerate(srcs)}, d)
        for n, e, r in zip(sizes, emas, refs):
            assert torch.equal(e, r), (updates, n, int((e != r).sum()))


def psp_model(seed=1, gain=None):
    from multiyolov5_b200.models.yolo import Model
    cfg = synth.load_cfg(G.CFG)
    sd = synth.synth_state_dict(synth.load_manifest("s_psp"), cfg, seed=seed, **({} if gain is None else {"gain": gain}))
    torch.manual_seed(0)
    model = Model(G.CFG)
    model.load_state_dict(sd)
    return model.cuda(), cfg


def test_replay_of_the_references_ema_life():
    """tests/golden/ema_cases.pt: fp32 updates, ema.half() and fp16 updates, .float(), jumps along the decay ramp, a checkpoint resume.
    The device ModelEMA gives every entry's SHA-256 of the reference after every update, its d, its dtypes and its final anchors."""
    from multiyolov5_b200.utils.torch_utils import ModelEMA
    cases = torch.load(os.path.join(G.GOLD, "ema_cases.pt"), weights_only=False)
    model, _ = psp_model()
    model.train()
    msd = model.state_dict()
    keys = G.averaged_keys(msd)
    assert keys == cases["keys"]
    base = {k: msd[k].detach().cpu().clone() for k in keys}
    bad = []

    def on_update(i, ema, d):
        assert next(ema.ema.parameters()).is_cuda and ema._table is not None          # the device path ran
        assert d == float(cases["d"][i])
        esd = ema.ema.state_dict()
        assert str(esd[keys[0]].dtype) == cases["ema_dtypes"][i]
        for j, k in enumerate(keys):
            if G.digest(esd[k]) != bytes(cases["digests"][i, j]):
                bad.append((i, k))

    ema = G.replay(ModelEMA, model, base, keys, on_update)
    assert not bad, (len(bad), bad[:10])
    assert ema.updates == cases["updates"]
    esd = ema.ema.state_dict()
    for k, v in cases["anchors"].items():
        assert torch.equal(esd[k].cpu(), v), k


def trainer_batch(cfg, B=2, seed=0):
    rs = np.random.RandomState(seed)
    imgs = synth.synth_image(B, 128, 256, seed=seed + 1).cuda()
    segimgs = synth.synth_image(B, 128, 256, seed=seed + 2).cuda()
    t = np.zeros((12, 6), np.float32)
    t[:, 0] = rs.randint(0, B, 12); t[:, 1] = rs.randint(0, cfg["nc"], 12)
    t[:, 2:4] = rs.uniform(0.1, 0.9, (12, 2)); t[:, 4:6] = rs.uniform(0.05, 0.4, (12, 2))
    mask = torch.from_numpy(rs.randint(-1, 19, (B, 1, 16, 32)).astype(np.int64)).cuda()
    mask = mask.repeat_interleave(8, 2).repeat_interleave(8, 3)[:, 0].contiguous()
    return imgs, torch.from_numpy(t).cuda(), segimgs, mask


def floating(sd):
    return {k: v.detach().clone() for k, v in sd.items() if v.dtype.is_floating_point}


@pytest.mark.parametrize("built", ["before_trainer", "after_trainer"])
def test_trainer_updates_the_ema_after_every_optimizer_step(built):
    """Trainer(accumulate=2, ema=...) over eight iterations, one of whose optimizer steps overflows (a loss scale of 2^40 puts inf in the
    fp16 gradients) and is skipped: ema.updates counts all four optimizer steps, the skipped one too, and after each the EMA equals the
    reference's statements applied to a torch copy fed with the trainer model's state_dict() at that point.  Built before the Trainer, the
    EMA has already updated once with its table on the model's own tensors; the Trainer then moves the parameters into its flat buffer."""
    from multiyolov5_b200.train import Trainer, scale_hyp
    from multiyolov5_b200.utils.torch_utils import ModelEMA
    model, cfg = psp_model(gain=1.0)
    model.train()
    hyp = scale_hyp(HYP, nl=3, nc=cfg["nc"], imgsz=256, total_batch_size=4)
    ema = ref = None
    if built == "before_trainer":
        ema = ModelEMA(model)
        ref = floating(ema.ema.state_dict())
        ema.update(model)
        reference_update(ref, model.state_dict(), ema.decay(1))
    tr = Trainer(model, hyp, batch_size=2, accumulate=2, init_scale=2.0 ** 10, ema=ema)
    if ema is None:
        ema = tr.ema = ModelEMA(model)
        ref = floating(ema.ema.state_dict())
    n0 = ema.updates
    for it in range(8):
        if it == 4:
            tr.scale.fill_(2.0 ** 40)
        tr.step(*trainer_batch(cfg, seed=it))
        if tr.ni % 2:
            assert ema.updates == n0 + it // 2
            continue
        torch.cuda.synchronize()
        assert ema.updates == n0 + (it + 1) // 2
        if it == 5:
            assert int(tr.found_inf) == 1 and float(tr.scale) == 2.0 ** 39
            tr.scale.fill_(2.0 ** 10)
        else:
            assert int(tr.found_inf) == 0
        reference_update(ref, tr.model.state_dict(), ema.decay(ema.updates))
        esd = ema.ema.state_dict()
        for k, v in ref.items():
            assert torch.equal(esd[k], v), (it, k)
    assert ema.updates == n0 + 4


def seg_loader(B=2, H=128, W=256, n=2):
    g = torch.Generator().manual_seed(4)
    return [(torch.rand((B, 3, H, W), generator=g).cuda(), torch.randint(-1, 19, (B, H, W), generator=g).cuda()) for _ in range(n)]


def det_loader(nc, B=2, H=128, W=256, n=2):
    g = torch.Generator().manual_seed(5)
    out = []
    for _ in range(n):
        img = torch.randint(0, 256, (B, 3, H, W), dtype=torch.uint8, generator=g)
        t = torch.rand((6, 6), generator=g)
        t[:, 0] = torch.arange(6) % B
        t[:, 1] = torch.randint(0, nc, (6,), generator=g).float()
        t[:, 4:6] = t[:, 4:6] * 0.3 + 0.05
        out.append((img, t, [""] * B, [((H, W), ((1.0, 1.0), (0.0, 0.0)))] * B))
    return out


def forward_equal(a, b, x):
    with torch.no_grad():
        (za, ra), sa = a(x)
        (zb, rb), sb = b(x)
    assert torch.equal(za, zb) and all(torch.equal(p, q) for p, q in zip(ra, rb)) and torch.equal(sa, sb)


def test_evaluating_the_ema_follows_its_anchors():
    """the reference's epoch on rank 0: updates, seg_validation(ema.ema) (leaves it fp16), fp16 updates, test(ema.ema) (half, then float),
    fp32 updates.  Validation leaves the EMA where the reference's half() / float() leave a torch copy, updates in between match the
    reference's statements in fp16 and fp32, and after the anchors have moved ema.ema(x) gives bit for bit the z, raws and seg of a fresh
    deepcopy, whose plan takes its anchors from anchor_grid when it is built."""
    from multiyolov5_b200.test import seg_validation, test
    from multiyolov5_b200.utils.torch_utils import ModelEMA
    model, cfg = psp_model()
    model.train()
    msd = model.state_dict()
    keys = G.averaged_keys(msd)
    base = {k: msd[k].detach().cpu().clone() for k in keys}
    ema = ModelEMA(model)
    ema.updates = 99_990                                       # late in the ramp: fp16 updates freeze most entries, fp32 ones move them
    ref = floating(ema.ema.state_dict())
    x = synth.synth_image(2, 128, 256, seed=9).cuda()
    anchors0 = ema.ema.model[-1].anchor_grid.clone()
    i = 0

    def updates(n):
        nonlocal i
        for _ in range(n):
            G.set_source_state(model, base, keys, i)
            ema.update(model)
            reference_update(ref, model.state_dict(), ema.decay(ema.updates))
            i += 1
        esd = ema.ema.state_dict()
        for k, v in ref.items():
            assert torch.equal(esd[k], v), k

    with torch.no_grad():
        ema.ema(x)                                             # the first evaluation builds the plan with today's anchors
    updates(3)
    seg_validation(ema.ema, 19, seg_loader(), torch.device("cuda"))
    ref = {k: v.half() for k, v in ref.items()}                # test.py:124 model.half(); seg_validation does not go back to fp32
    assert all(torch.equal(ema.ema.state_dict()[k], v) for k, v in ref.items())
    updates(3)
    test({"nc": cfg["nc"]}, model=ema.ema, dataloader=det_loader(cfg["nc"]), plots=False)
    ref = {k: v.half().float() for k, v in ref.items()}        # test.py:45 half() (already fp16), test.py:333 float()
    assert next(ema.ema.parameters()).dtype == torch.float32
    assert all(torch.equal(ema.ema.state_dict()[k], v) for k, v in ref.items())
    updates(20)
    assert not torch.equal(ema.ema.model[-1].anchor_grid, anchors0)          # the averaging arithmetic has moved the anchors
    forward_equal(ema.ema, copy.deepcopy(ema.ema), x)
    ema.ema.half()
    forward_equal(ema.ema, copy.deepcopy(ema.ema), x.half())
