"""GPU: every op of an inference plan checked on its own.  One forward of a model through a plan that gives every buffer private memory
(Engine.noalias; the same op list as the default plan, only the offsets differ); then each op's stored output is compared with an fp64
restatement of that op fed with the fp16 / fp32 tensors the plan itself stored as its inputs.  Upstream error does not accumulate, so the
limits sit near fp16 storage rounding, where the whole-network tests (test_gpu_model.py, test_gpu_parity.py) have to absorb ~60 layers
of it.

Two patterns overwrite a view after an op has read it: the last bottleneck of a fused C3 writes the cv1 half of the [cv1 | cv2] buffer,
and FFM's CHANNEL_SCALE scales the convblk output in place.  Such values are read from a second plan that runs a prefix of the same op
list on the same buffers and offsets (the forward has no atomics: the prefix writes the same bytes).

The second test runs the default (liveness-packed) plan against the private-buffer plan: every output must be bit-identical."""
import copy
import ctypes as C
import math
from collections import defaultdict
from types import SimpleNamespace

import pytest
import torch
import torch.nn.functional as F

from oracle import synth
from tests import test_gpu_train_layers as TL

pytestmark = pytest.mark.gpu

YAML = dict(TL.YAML, m_psp="yolov5m_city_seg.yaml")
U16 = TL.U16

# Limits, calibrated on an H100 80GB HBM3 (700 W power limit) over the nine cases below: each is about 4x the worst value observed
# there.  fp16 outputs: (|ours - ref| - U16 |ref|) / max|ref| (what is left after the one fp16 rounding of the stored value; 0 for the
# ops that move values or round once); fp32 outputs: |ours - ref| / max|ref|.  CONV_F32 are the convs with fp32 outputs (Detect heads, seg
# classifier, FFM attention), which get no rounding allowance.
# Worst values there: CONV 2.3e-6 (m_psp bench), CONV_F32 2.5e-6 (s_base), BILINEAR 4.6e-7 (416x736), REGION_SUM 7.5e-8, REGION_COMBINE
# 2.3e-7, CHANNEL_SCALE 6.5e-10, DETECT_DECODE 2.5e-7, SEG_UPSAMPLE 1.7e-6 (s_base); INPUT_FOCUS, SPP_POOL, UPSAMPLE_NEAREST, ADD and
# BROADCAST exactly 0.
LIMIT = {"INPUT_FOCUS": 0.0, "CONV": 1e-5, "CONV_F32": 1e-5, "UPSAMPLE_NEAREST": 0.0, "SPP_POOL": 0.0, "BILINEAR": 2e-6, "REGION_SUM": 3e-7,
         "REGION_COMBINE": 1e-6, "CHANNEL_SCALE": 3e-9, "ADD": 0.0, "BROADCAST": 0.0, "DETECT_DECODE": 1e-6, "SEG_UPSAMPLE": 7e-6}


# ---- the plan and its execution order --------------------------------------------------------------------------------------------
def base_view(v):
    """the pixel-pair alias of layer 0 seen as its base buffer"""
    from multiyolov5_b200.plan import V
    return V(v.buf.alias_of, 0, v.buf.alias_of.c) if v.buf.alias_of is not None else v


def written_view(op):
    from multiyolov5_b200 import _lib as L
    return op.in_ if op.kind == L.OP_CHANNEL_SCALE else op.out   # CHANNEL_SCALE scales its input in place


def exec_positions(pb):
    """plan index of the launch that runs each op: a group member runs in its head's launch"""
    from multiyolov5_b200 import _lib as L
    pos, head = [], -1
    for i, o in enumerate(pb.ops):
        if o.flags & L.OP_GROUP_HEAD:
            head = i
        pos.append(head if o.flags & L.OP_GROUP_MEMBER else i)
    return pos


def overlap(a, b):
    a, b = base_view(a), base_view(b)
    return a.buf is b.buf and a.c_off < b.c_off + b.c and b.c_off < a.c_off + a.c


def value_sources(pb):
    """for every (op, role) whose stored value is overwritten later in the forward: the length of the op-list prefix after which the
    workspace holds the value the op saw (role "in0" / "in1": its inputs, before it ran; "out": its output, after it ran)"""
    from multiyolov5_b200 import _lib as L
    pos = exec_positions(pb)
    writes = [(j, w) for j, o in enumerate(pb.ops) if (w := written_view(o)) is not None]

    def prefix(v, t_incl):               # ops up to the last writer of v at or before exec position t_incl, a whole group included
        n = 1 + max(j for j, w in writes if pos[j] <= t_incl and overlap(v, w))
        while n < len(pb.ops) and pb.ops[n].flags & L.OP_GROUP_MEMBER:
            n += 1
        return n
    src = {}
    for i, op in enumerate(pb.ops):
        for r, v in (("in0", op.in_), ("in1", op.in2)):
            if v is not None and any(pos[j] >= pos[i] and overlap(v, w) for j, w in writes):
                src[(i, r)] = (v, prefix(v, pos[i] - 1))
        w = written_view(op)
        if w is not None and any(pos[j] > pos[i] and overlap(w, ww) for j, ww in writes):
            src[(i, "out")] = (w, prefix(w, pos[i]))
    return src


def same_plan(a, b):
    """the two host plans differ in buffer offsets only"""
    def vk(v):
        return None if v is None else (v.buf.id, v.c_off, v.c)

    def sk(s):
        c = s.conv
        parts = (c.a, c.b) if hasattr(c, "a") else ((c.base,) if hasattr(c, "base") else (c,))
        bn = s.bn
        bns = () if bn is None else ((bn.a, bn.b) if hasattr(bn, "a") else (bn,))
        return type(c).__name__, tuple(map(id, parts)), tuple(map(id, bns)), s.name
    assert len(a.ops) == len(b.ops) and len(a.bufs) == len(b.bufs) and list(a.extra) == list(b.extra)
    assert [(x.id, x.h, x.w, x.c, x.dtype, x.alias_of and x.alias_of.id) for x in a.bufs] == \
           [(x.id, x.h, x.w, x.c, x.dtype, x.alias_of and x.alias_of.id) for x in b.bufs]
    for i, (p, q) in enumerate(zip(a.ops, b.ops)):
        assert (p.kind, vk(p.in_), vk(p.in2), vk(p.out), p.k, p.stride, p.dil, p.act, p.flags, p.slot, list(p.aux), list(p.faux)) == \
               (q.kind, vk(q.in_), vk(q.in2), vk(q.out), q.k, q.stride, q.dil, q.act, q.flags, q.slot, list(q.aux), list(q.faux)), i
    assert [sk(s) for s in a.slots] == [sk(s) for s in b.slots]


def conv_info(plan, i):
    from multiyolov5_b200 import _lib
    info = (C.c_int32 * 12)()
    _lib.check(_lib.lib().myolo_plan_conv_info(plan.handle, i, info))
    return list(info)


# ---- running a plan ----------------------------------------------------------------------------------------------------------------
def make_model(tag, bench_weights, half):
    from multiyolov5_b200.models.yolo import Model
    if bench_weights:
        import bench
        yml, _, sd = bench.make_weights(tag)
    else:
        yml = YAML[tag]
        sd = synth.synth_state_dict(synth.load_manifest(tag), synth.load_cfg(yml), seed=1)
    m = Model(yml)
    m.load_state_dict(sd)
    m.cuda().eval()
    return m.half() if half else m


def make_input(B, H, W, xtype):
    if xtype == "u8":
        return torch.randint(0, 256, (B, 3, H, W), dtype=torch.uint8, generator=torch.Generator().manual_seed(5)).cuda()
    x = synth.synth_image(B, H, W, seed=5)
    return (x.half() if xtype == "fp16" else x).cuda()


def forward(eng, plan, x):
    """one myolo_plan_forward writing z, the three raw, the seg logits AND the fused argmax (Engine.forward returns one of the last two)"""
    from multiyolov5_b200 import _lib
    model = eng.model
    B, _, H, W = x.shape
    det, seg_head = model.model[-1], model.model[-2]
    eng._upload_if_stale(plan)
    dev = x.device
    z = torch.empty((B, sum(plan.pb.det_rows), det.no), dtype=torch.float32, device=dev)
    raws = [torch.empty((B, det.na, o.in_.h, o.in_.w, det.no), dtype=torch.float32, device=dev)
            for o in plan.pb.ops if o.kind == _lib.OP_DETECT_DECODE]
    half = x.dtype == torch.float16 or next(model.parameters()).dtype == torch.float16
    seg = torch.empty((B, seg_head.c_out, H, W), dtype=torch.float16 if half else torch.float32, device=dev)
    amax = torch.empty((B, H, W), dtype=torch.int64, device=dev)
    raw_ptrs = (C.c_void_p * 3)(*[_lib.ptr(r) for r in raws])
    _lib.check(_lib.lib().myolo_plan_forward(plan.handle, _lib.ptr(x), _lib.torch_dtype_code(x.dtype), _lib.ptr(z), raw_ptrs, _lib.ptr(seg),
                                             _lib.torch_dtype_code(seg.dtype), _lib.ptr(amax), _lib.stream_ptr()))
    return SimpleNamespace(z=z, raws=raws, seg=seg, amax=amax)


def engine_plan(model, B, H, W, noalias, pb=None):
    from multiyolov5_b200.engine import CompiledPlan, Engine
    eng = Engine(model)
    eng.noalias = noalias
    plan = CompiledPlan(model, B, H, W, noalias=noalias, pb=pb)
    eng.plans[(B, H, W)] = plan
    return eng, plan


def run_case(tag, B, H, W, xtype, bench_weights=False):
    """the noalias plan's forward, the default plan's op list and conv routes, and the pre-overwrite values from prefix plans"""
    from multiyolov5_b200 import _lib as L
    half = xtype == "fp16" and bench_weights
    model = make_model(tag, bench_weights, half)
    x = make_input(B, H, W, xtype)
    eng, plan = engine_plan(model, B, H, W, noalias=True)
    out = forward(eng, plan, x)
    deng, dplan = engine_plan(model, B, H, W, noalias=False)
    forward(deng, dplan, x)
    pb = plan.pb
    same_plan(pb, dplan.pb)
    routes = {i: conv_info(plan, i) for i, o in enumerate(pb.ops) if o.kind == L.OP_CONV}
    assert routes == {i: conv_info(dplan, i) for i in routes}
    del deng, dplan
    src = value_sources(pb)
    pre = {}
    for n in sorted({n for _, n in src.values()}):
        ppb = copy.copy(pb)                # the first n ops on the same buffers, offsets, weight slots and tables
        ppb.ops = pb.ops[:n]
        peng, pplan = engine_plan(model, B, H, W, noalias=True, pb=ppb)
        forward(peng, pplan, x)
        for key, (v, m) in src.items():
            if m == n:
                pre[key] = peng.read_view(v, pplan)
        del peng, pplan
    torch.cuda.synchronize()
    return SimpleNamespace(tag=tag, model=model, eng=eng, plan=plan, pb=pb, x=x, out=out, B=B, H=H, W=W, routes=routes, src=src, pre=pre,
                           served=set())


def stored(st, i, role, v):
    """fp64 value of view v as op i saw it (role "in0" / "in1") or left it ("out")"""
    if (i, role) in st.src:
        st.served.add((i, role))
        return st.pre[(i, role)].double()
    return st.eng.read_view(v, st.plan).double()


# ---- fp64 restatements --------------------------------------------------------------------------------------------------------------
def act(z, a):
    from multiyolov5_b200._lib import ACT_SIGMOID, ACT_SILU
    return z * torch.sigmoid(z) if a == ACT_SILU else (torch.sigmoid(z) if a == ACT_SIGMOID else z)


FOLD_REL = 2.0 ** -20      # relative error bound of the pack's fp32 BN fold (w * (gamma / sqrtf(var + eps)): three fp32 roundings)


def conv_ref(st, op, x, res, mutant=None):
    """reference Conv.fuseforward: BN folded in fp64 with the slot's eps, the folded weight rounded to fp16 (the pack), bias, act, then the
    residual.  The fused C3 cv1+cv2 is its two reference convs, each with its own BN; layer 0 on pixel pairs is the reference 3x3 conv.
    Returns (reference, allowance): the pack folds in fp32, so a folded weight within FOLD_REL of an fp16 rounding boundary may round
    either way (~2e-4 of the weights); the allowance bounds what that can move each output, sum |x| |w_up - w_down| over those weights
    times the largest slope of the activation."""
    from multiyolov5_b200._lib import ACT_SIGMOID, ACT_SILU
    from multiyolov5_b200.plan import _CatConv, _PairedConv
    s = st.pb.slots[op.slot]
    if isinstance(s.conv, _CatConv):
        parts = [(s.conv.a, s.bn.a), (s.conv.b, s.bn.b)]
    elif isinstance(s.conv, _PairedConv):
        parts = [(s.conv.base, s.bn.a)]
    else:
        parts = [(s.conv, s.bn)]
    ys, allow = [], []
    for conv, bn in parts:
        w = conv.weight.detach().double()
        b = conv.bias.detach().double() if conv.bias is not None else torch.zeros(w.shape[0], dtype=torch.float64, device=w.device)
        if bn is not None:
            eps = 1e-5 if mutant == "eps" else bn.eps
            g = bn.weight.detach().double() / torch.sqrt(bn.running_var.detach().double() + eps)
            w = w * g.view(-1, 1, 1, 1)
            b = bn.bias.detach().double() - bn.running_mean.detach().double() * g + b * g
        xs = x[:, :conv.in_channels]
        ys.append(F.conv2d(xs, w.half().double(), b, conv.stride, conv.padding, conv.dilation))
        dw = ((w * (1 + FOLD_REL)).half().double() - (w * (1 - FOLD_REL)).half().double()).abs()
        allow.append(F.conv2d(xs.abs(), dw, None, conv.stride, conv.padding, conv.dilation))
    y, a = torch.cat(ys, 1), torch.cat(allow, 1)
    a = a * (1.1 if op.act == ACT_SILU else (0.25 if op.act == ACT_SIGMOID else 1.0))     # max |SiLU'| = 1.0998, max |sigmoid'| = 1/4
    if res is not None and mutant == "residual":        # residual added before the activation
        return act(y + res, op.act), a
    y = act(y, op.act)
    return (y + res if res is not None else y), a


def decode_ref(st, raws, mutant=None):
    """reference Detect.forward (eval) from the returned raw: xy = (2 sigma - 0.5 + grid) stride, wh = (2 sigma)^2 anchor_grid, rest sigma"""
    det = st.model.model[-1]
    zs = []
    for lvl, r in enumerate(raws):
        s = torch.sigmoid(r.double())
        ny, nx = r.shape[2], r.shape[3]
        yv, xv = torch.meshgrid(torch.arange(ny, device=r.device), torch.arange(nx, device=r.device), indexing="ij")
        grid = torch.stack((xv, yv), 2).view(1, 1, ny, nx, 2).double()
        off = 0.0 if mutant == "grid" else 0.5
        xy = (s[..., 0:2] * 2.0 - off + grid) * float(det.stride[lvl])
        wh = (s[..., 2:4] * 2.0) ** 2 * det.anchor_grid[lvl].double()
        zs.append(torch.cat((xy, wh, s[..., 4:]), -1).view(r.shape[0], -1, r.shape[-1]))
    return torch.cat(zs, 1)


def err16(ours, ref, allow=0.0):
    return float(((ours - ref).abs() - U16 * ref.abs() - allow).clamp_min(0).max()) / max(float(ref.abs().max()), 1e-30)


def err32(ours, ref, allow=0.0):
    return float(((ours - ref).abs() - allow).clamp_min(0).max()) / max(float(ref.abs().max()), 1e-30)


def op_errors(st, mutant=None):
    """(op index, kind, error) for every op of the plan"""
    from multiyolov5_b200 import _lib as L
    from multiyolov5_b200.plan import _PairedConv
    names = TL.kind_names()
    ns = SimpleNamespace(pb=st.pb)
    errs = []
    for i, op in enumerate(st.pb.ops):
        kind = names[op.kind]
        if op.kind == L.OP_INPUT_FOCUS:            # to_unit (uint8 / 255 in fp32), one fp16 rounding; channels 12..15 exactly 0
            x = st.x.float() / 255.0 if st.x.dtype == torch.uint8 else st.x.float()
            x = x.half().double()
            ref = torch.cat([x[..., ::2, ::2], x[..., 1::2, ::2], x[..., ::2, 1::2], x[..., 1::2, 1::2]], 1)
            ours = stored(st, i, "out", op.out)
            assert float(ours[:, 12:].abs().max()) == 0.0, i
            errs.append((i, kind, err16(ours[:, :12], ref)))
            continue
        if op.kind == L.OP_DETECT_DECODE:          # raw: the head conv's output permuted, bit for bit; z: all levels at once below
            na, no = op.aux[1], op.aux[2]
            head = st.eng.read_view(op.in_, st.plan)[:, :na * no]
            perm = head.reshape(st.B, na, no, op.in_.h, op.in_.w).permute(0, 1, 3, 4, 2)
            assert torch.equal(st.out.raws[op.aux[0]], perm), f"op {i}: raw[{op.aux[0]}] is not the head conv's output"
            continue
        if op.kind == L.OP_SEG_UPSAMPLE:
            errs.append((i, kind, seg_check(st, op, mutant)))
            continue
        if op.kind == L.OP_CONV:
            conv = st.pb.slots[op.slot].conv
            if isinstance(conv, _PairedConv):      # read through the base buffers, not the pixel-pair aliases
                x = stored(st, i, "in0", base_view(op.in_))
                ours = stored(st, i, "out", base_view(op.out))
            else:
                x = stored(st, i, "in0", op.in_)
                ours = stored(st, i, "out", op.out)
            res = stored(st, i, "in1", op.in2) if op.in2 is not None else None
            with torch.no_grad():
                ref, allow = conv_ref(st, op, x, res, mutant)
            ours = ours[:, :ref.shape[1]]
            f32 = op.out.buf.dtype == L.F32
            errs.append((i, "CONV_F32" if f32 else "CONV", (err32 if f32 else err16)(ours, ref, allow)))
            continue
        ins = [stored(st, i, r, v) for r, v in (("in0", op.in_), ("in1", op.in2)) if v is not None]
        if op.kind == L.OP_CHANNEL_SCALE:          # FFM: feat * att + feat, in place, one rounding
            f, a = ins[0], ins[1][:, :op.in_.c]
            ref = f * a if mutant == "scale" else f * a + f
            ours = stored(st, i, "out", op.in_)
        else:
            if op.kind == L.OP_BILINEAR and mutant == "bilinear":
                ref = F.interpolate(ins[0], (op.out.h, op.out.w), mode="bilinear", align_corners=False)
            else:
                ref = TL.restate(ns, i, op, ins, {})
            ours = stored(st, i, "out", op.out)[:, :ref.shape[1]]
        f32 = written_view(op).buf.dtype == L.F32
        errs.append((i, kind, (err32 if f32 else err16)(ours, ref)))
    # z against the restatement from the returned raw: every level's rows and its row offset at once; each column group (xy, wh, sigma)
    # relative to its own largest value, so that the pixel-sized xy do not hide an error in the probabilities
    with torch.no_grad():
        zr = decode_ref(st, st.out.raws, mutant)
    z = st.out.z.double()
    assert z.shape == zr.shape
    di = max(err32(z[..., a:b], zr[..., a:b]) for a, b in ((0, 2), (2, 4), (4, z.shape[-1])))
    errs.append((len(st.pb.ops), "DETECT_DECODE", di))
    # REGION_SUM + REGION_COMBINE together are adaptive_avg_pool2d of the pooled map
    for i, op in enumerate(st.pb.ops):
        if op.kind == L.OP_REGION_COMBINE:
            srcop = [(j, o) for j, o in enumerate(st.pb.ops) if o.kind == L.OP_REGION_SUM and o.out.buf is op.in_.buf][0]
            x = stored(st, srcop[0], "in0", srcop[1].in_)
            with torch.no_grad():
                pooled = TL.restate(ns, -1, op, [TL.restate(ns, -1, srcop[1], [x], {})], {})
            ref = F.adaptive_avg_pool2d(x, (op.out.h, op.out.w))
            assert float((pooled - ref).abs().max()) <= 1e-12 * max(1.0, float(ref.abs().max())), i
    return errs


def seg_check(st, op, mutant=None):
    """seg logits against an fp64 align_corners bilinear upsample of the stored low-resolution logits (image by image); the fused argmax
    against the argmax of that reference wherever its two best classes are further apart than the limit allows either to move"""
    n = op.aux[0]
    lo = st.eng.read_view(op.in_, st.plan)[:, :n].double()
    f16 = st.out.seg.dtype == torch.float16
    scale = float(lo.abs().max())          # >= max |ref|: the interpolation is convex
    worst, top, checked = 0.0, 0.0, 0
    margin = 2.0 * max(LIMIT["SEG_UPSAMPLE"], 1e-6) * scale + (2 * U16 * scale if f16 else 0.0)
    for b in range(st.B):
        ref = F.interpolate(lo[b:b + 1], (st.H, st.W), mode="bilinear", align_corners=True)[0]
        d = (st.out.seg[b].double() - ref).abs()
        if f16:
            d = d - U16 * ref.abs()
        worst = max(worst, float(d.max()))
        top = max(top, float(ref.abs().max()))
        t2 = ref.topk(2, dim=0)
        sure = (t2.values[0] - t2.values[1]) > margin
        bad = (st.out.amax[b] != t2.indices[0]) & sure
        assert not bool(bad.any()), f"fused argmax differs from the reference at {int(bad.sum())} clear pixels of image {b}"
        checked += int(sure.sum())
    st.argmax_checked = checked / (st.B * st.H * st.W)
    return max(worst, 0.0) / top


# ---- coverage -------------------------------------------------------------------------------------------------------------------------
def coverage(st):
    from multiyolov5_b200 import _lib as L
    from multiyolov5_b200.plan import _CatConv, _PairedConv
    c = defaultdict(int)
    for i, o in enumerate(st.pb.ops):
        if o.kind == L.OP_CONV:
            info = st.routes[i]
            conv = st.pb.slots[o.slot].conv
            if info[0]:
                c["wgmma"] += 1
                c["wgmma resident" if info[6] else "wgmma streamed"] += 1
                c["wgmma strip"] += info[5] == 1
                c[f"wgmma BN={info[3]}"] += 1
                c["wgmma fp32 out"] += o.out.buf.dtype == L.F32
                c["wgmma 2 CTA/SM"] += info[11] == 2
            else:
                c["simt"] += 1
            c["fp32-input conv"] += o.in_.buf.dtype == L.F32
            c["residual from a slice"] += o.in2 is not None and o.in2.buf.c != o.in2.c
            c["pixel-pair layer 0"] += isinstance(conv, _PairedConv)
            c["fused C3 cv1+cv2"] += isinstance(conv, _CatConv)
        if o.flags & L.OP_GROUP_HEAD:
            c[f"grouped {TL.kind_names()[o.kind]}"] += 1
    return dict(sorted(c.items()))


CASES = {  # id: (model, B, H, W, input, bench weights + model.half(), MYOLO_FORCE_SIMT)
    "s_psp_bench": ("s_psp", 16, 512, 1024, "fp16", True, False),    # bench.py's default workload
    "m_psp_bench": ("m_psp", 8, 512, 1024, "fp16", True, False),     # bench.py's m batch
    "s_psp": ("s_psp", 2, 256, 512, "fp32", False, False),
    "s_psp_u8": ("s_psp", 1, 256, 512, "u8", False, False),          # uint8 frames, converted by the first kernel
    "s_psp_416x736": ("s_psp", 2, 416, 736, "fp32", False, False),   # ragged tiles, overlapping adaptive bins
    "s_psp_simt": ("s_psp", 2, 256, 512, "fp32", False, True),       # every conv on the CUDA-core kernel
    "m_lab": ("m_lab", 2, 256, 512, "fp32", False, False),
    "s_bise": ("s_bise", 2, 256, 512, "fp32", False, False),
    "s_base": ("s_base", 1, 512, 1024, "fp32", False, False),
}


def assert_coverage(name, st, cov, simt):
    from multiyolov5_b200 import _lib as L
    from multiyolov5_b200.plan import adaptive_bins
    assert cov["pixel-pair layer 0"] == 1 and cov["fused C3 cv1+cv2"] >= 8 and cov["residual from a slice"] >= 1, cov
    if simt:
        assert cov.get("wgmma", 0) == 0 and cov["simt"] >= 60, cov
    else:
        assert cov["wgmma resident"] >= 1 and cov["wgmma streamed"] >= 1 and cov["wgmma strip"] >= 1, cov
        assert sum(1 for k in cov if k.startswith("wgmma BN=")) >= 2 and cov["wgmma fp32 out"] >= 1, cov
    if st.tag in ("s_psp", "m_psp"):
        assert cov["grouped CONV"] >= 1 and cov["grouped BILINEAR"] >= 1 and cov["grouped REGION_COMBINE"] >= 1, cov
    if st.tag in ("s_psp", "m_psp", "m_lab", "s_bise"):      # FFM: attention convs on fp32 inputs, CHANNEL_SCALE in place
        assert cov["fp32-input conv"] >= 2 and any(o.kind == L.OP_CHANNEL_SCALE for o in st.pb.ops), cov
    if name == "s_psp_416x736":
        pooled = [(src.in_.h, src.in_.w, o.out.h) for o in st.pb.ops if o.kind == L.OP_REGION_COMBINE
                  for src in st.pb.ops if src.kind == L.OP_REGION_SUM and src.out.buf is o.in_.buf]
        assert any(a[1] > b[0] for h, w, k in pooled for n in (h, w) for a, b in zip(adaptive_bins(n, k), adaptive_bins(n, k)[1:]))
        assert any(b.w % 8 for b in st.pb.bufs)               # maps whose rows end inside a tile


def check_case(st):
    """per-kind worst value against the limit; returns the failures"""
    errs = op_errors(st)
    worst = defaultdict(float)
    fails = []
    for i, kind, e in errs:
        worst[kind] = max(worst[kind], e)
        if e > LIMIT[kind]:
            fails.append(f"op {i} {kind}: {e:.3e} > {LIMIT[kind]:.1e}")
    print(TL.fmt_table("worst per op kind (fp16 outputs: (|err| - fp16 rounding) / max|ref|; fp32 outputs: |err| / max|ref|):",
                       [(k, f"{v:.2e}", f"{LIMIT[k]:.0e}") for k, v in sorted(worst.items())]))
    return fails


@pytest.mark.parametrize("name", list(CASES))
def test_every_inference_op_matches_its_fp64_restatement(name, monkeypatch):
    tag, B, H, W, xtype, bench_weights, simt = CASES[name]
    monkeypatch.setenv("MYOLO_FORCE_SIMT", "1" if simt else "0")
    torch.manual_seed(0)
    st = run_case(tag, B, H, W, xtype, bench_weights)
    fails = check_case(st)
    cov = coverage(st)
    print(f"[{name}] coverage: {cov}")
    print(f"[{name}] values overwritten in place, read from prefix plans: {len(st.src)} "
          f"({sorted({TL.kind_names()[st.pb.ops[i].kind] + ':' + r for i, r in st.src})}); "
          f"fused argmax checked at {100 * st.argmax_checked:.1f} % of the pixels")
    assert st.served == set(st.src), set(st.src) - st.served
    assert st.src, "no view is overwritten in place: the fused C3 and FFM patterns are gone"
    assert_coverage(name, st, cov, simt)
    assert not fails, "\n".join(fails[:20])


MUTANTS = {"eps": "CONV", "residual": "CONV", "bilinear": "BILINEAR", "grid": "DETECT_DECODE", "scale": "CHANNEL_SCALE"}


def test_layer_checks_catch_wrong_restatements(monkeypatch):
    """the limits discriminate: with one deliberately wrong restatement its op kind must miss the limit by at least 10x - the BN fold with
    eps 1e-5 instead of the slot's 1e-3, the residual added before SiLU, bilinear with align_corners=False, z without the -0.5 grid
    offset, and CHANNEL_SCALE as feat * att"""
    monkeypatch.setenv("MYOLO_FORCE_SIMT", "0")
    torch.manual_seed(0)
    st = run_case("s_psp", 2, 256, 512, "fp32")
    print()
    missed = {}
    for mutant, kind in MUTANTS.items():
        worst = max(e for _, k, e in op_errors(st, mutant) if k == kind)
        missed[mutant] = worst / LIMIT[kind] if LIMIT[kind] else (math.inf if worst > 0 else 0.0)
        print(f"mutant {mutant:<9} ({kind}): worst op {worst:.2e}, {missed[mutant]:.0f}x its limit")
    assert all(v >= 10 for v in missed.values()), missed


# ---- packed workspace against private buffers --------------------------------------------------------------------------------------------
PACK_CASES = {f"{t}_2x256x512": (t, 2, 256, 512, "fp32", False) for t in YAML} | {"s_psp_bench": ("s_psp", 16, 512, 1024, "fp16", True)}


@pytest.mark.parametrize("name", list(PACK_CASES))
def test_packed_workspace_matches_private_buffers(name, monkeypatch):
    """the liveness-packed plan and the plan with private buffers return the same bits: z, the three raw, the seg logits and the fused
    argmax, on the first (eager) call and on the second (CUDA-graph replay)"""
    tag, B, H, W, xtype, bench_weights = PACK_CASES[name]
    monkeypatch.setenv("MYOLO_FORCE_SIMT", "0")
    model = make_model(tag, bench_weights, bench_weights)
    x = make_input(B, H, W, xtype)
    pe, pp = engine_plan(model, B, H, W, noalias=False)
    ne, npl = engine_plan(model, B, H, W, noalias=True)
    assert pp.pb.workspace_bytes < npl.pb.workspace_bytes
    for call in ("eager", "graph replay"):
        a, b = forward(pe, pp, x), forward(ne, npl, x)
        torch.cuda.synchronize()
        for what in ("z", "seg", "amax"):
            assert torch.equal(getattr(a, what), getattr(b, what)), (call, what)
        for lvl, (ra, rb) in enumerate(zip(a.raws, b.raws)):
            assert torch.equal(ra, rb), (call, f"raw[{lvl}]")
