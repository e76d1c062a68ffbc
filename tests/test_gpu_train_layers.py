"""GPU: every op of a train plan checked on its own.  One train forward and backward of a model; then each op's stored output is compared
with an fp64 restatement of that op (the semantics of oracle/restate.py) fed with the fp16 / fp32 tensors the plan itself stored, and each
buffer's gradient with the sum, over the ops that read it, of autograd through the same restatements seeded with those ops' stored output
gradients.  Upstream error does not accumulate, so the limits sit near fp16 storage rounding, where the end-to-end parity test
(test_gpu_train.py) has to allow for a deep BN network amplifying fp16 noise.

Train plans never alias buffers (plan.build_plan), so every activation and its twin in the gradient workspace is still readable after the
backward.  The parameter gradients and the running statistics are checked against fp64 references from the same stored tensors."""
import math
from collections import defaultdict
from types import SimpleNamespace

import pytest
import torch
import torch.nn.functional as F

from oracle import synth

pytestmark = pytest.mark.gpu

YAML = {"s_psp": "yolov5s_city_seg.yaml", "m_lab": "yolov5m_city_seg_lab.yaml", "s_base": "yolov5s_city_seg_base.yaml",
        "s_bise": "yolov5s_city_seg_bise.yaml"}
U16 = 2.0 ** -11            # fp16 unit roundoff: one rounding of a stored value

# Limits, calibrated on an H100 80GB HBM3 (400 W power limit) over the eight cases below: each is about 4x the worst value observed
# there, so that a kernel wrong by a fraction of a percent fails.
# Forward: (|ours - ref| - U16 |ref|) / max|ref|, elementwise: what is left after one fp16 rounding of the stored output (fp32
# accumulation order; 0 for the ops that move or compare values exactly).
FWD_TOL = {"CONV": 6e-6, "BN_ACT": 4e-6, "ACT": 0.0, "ADD": 0.0, "BROADCAST": 0.0, "CHANNEL_SCALE_OOP": 1e-8, "UPSAMPLE_NEAREST": 0.0,
           "BILINEAR": 4e-6, "SPP_POOL": 0.0, "REGION_SUM": 0.0, "REGION_COMBINE": 2e-8, "DROPOUT": 1e-8, "INPUT_FOCUS": 0.0,
           "SEG_UPSAMPLE": 8e-6, "DETECT_DECODE": 0.0}
# Backward, per gradient buffer: (relative Frobenius error, max |ours - ref| / max |ref|).  A buffer read by several ops gets the loosest
# limit of their kinds.  fp16 gradient buffers take one rounding per accumulation step (~3e-4 relative); fp32 ones almost none.
BWD_TOL = {"CONV": (1.4e-3, 2.5e-3), "BN_ACT": (1.1e-3, 2e-3), "ACT": (3e-7, 5e-7), "ADD": (1.2e-3, 2e-3), "BROADCAST": (8e-4, 1e-3),
           "CHANNEL_SCALE_OOP": (1.2e-3, 2.2e-3), "UPSAMPLE_NEAREST": (1.1e-3, 1.6e-3), "BILINEAR": (9e-4, 1.7e-3), "SPP_POOL": (1.1e-3, 1.7e-3),
           "REGION_SUM": (1.2e-3, 2.5e-3), "REGION_COMBINE": (2.5e-7, 5e-7), "DROPOUT": (8e-4, 1.2e-3), "SEG_UPSAMPLE": (1.4e-5, 2e-5),
           "DETECT_DECODE": (0.0, 0.0)}
# parameter gradients (relative Frobenius) and running statistics (max error over momentum x max |batch statistic|)
PARAM_TOL = {"conv.weight": 9e-4, "conv.bias": 1.4e-6, "bn.weight": 1e-5, "bn.bias": 7.5e-4, "running_mean": 2e-5, "running_var": 2e-5}


def kind_names():
    from multiyolov5_b200 import _lib
    return {getattr(_lib, n): n[3:] for n in dir(_lib) if n.startswith("OP_") and n not in ("OP_GROUP_HEAD", "OP_GROUP_MEMBER")}


# ---- the plan's view of the model ---------------------------------------------------------------------------------------------
def dgrad_routes(pb, B, force_simt=False):
    """conv_backward's routing (csrc/plan.cu), restated: for every conv op that computes a data gradient, (op index, path, kc, stride,
    dilation) with path "small" (conv_small_dgrad_kernel), "wgmma" (conv_tc) or "simt" (conv_simt), kc the wgmma K chunk"""
    from multiyolov5_b200._lib import F32, OP_CONV, OP_INPUT_FOCUS
    focus = {o.out.buf.id for o in pb.ops if o.kind == OP_INPUT_FOCUS}
    routes = []
    for i, o in enumerate(pb.ops):
        if o.kind != OP_CONV or o.in_.buf.id in focus:
            continue
        conv = pb.slots[o.slot].conv
        ci, co = conv.in_channels, conv.out_channels
        cpad = (co + 15) // 16 * 16
        kc = 64 if cpad % 64 == 0 else (32 if cpad % 32 == 0 else 16)
        if o.in_.buf.dtype == F32 or B * o.out.h * o.out.w <= 1024 or o.out.h * o.out.w < 128:
            path = "small"
        else:
            # the data-gradient conv: input = dY (zero-stuffed for stride 2, cast for fp32 heads) with cpad channels, output += grad(in)
            dy_ctot = cpad if (o.out.buf.dtype == F32 or o.stride == 2) else o.out.buf.c
            ok = (o.k in (1, 3) and dy_ctot % 8 == 0 and ci % 16 == 0 and o.in_.buf.c % 8 == 0 and o.in_.w >= 8 and o.in_.h >= 2
                  and o.in_.h * o.in_.w >= 128 and cpad * 4 + 512 <= 8192 and (ci + 15) // 16 * 16 * 4 + 512 <= 8192)
            path = "wgmma" if ok and not force_simt else "simt"
        routes.append((i, path, kc, o.stride, o.dil))
    return routes


def train_step(tag, B, H, W, image="synth"):
    """one train forward + backward through the engine, seeded like test_gpu_train.py (d loss / d raw = 4 N(0,1), d loss / d seg = 0.05 N(0,1))"""
    from multiyolov5_b200.models.yolo import Model
    cfg = synth.load_cfg(YAML[tag])
    sd = synth.synth_state_dict(synth.load_manifest(tag), cfg, seed=1, gain=1.0)
    model = Model(YAML[tag])
    model.load_state_dict(sd)
    model.cuda().train()
    if image == "flat":
        # flat content (letterbox padding, sky, road) gives tied maxima in the SPP windows.  Channels whose mean is >100x their spread need
        # more than the image: a 3x3 conv's zero padding alone makes the border pixels of a flat map spread (mean/std stays below ~50
        # here).  Layer 1's BN bias is raised by 100, so the 1x1 convs of the C3 after it (no padding) see inputs of mean ~100, spread ~1.
        x = 0.5 + 0.002 * torch.randn((B, 3, H, W), generator=torch.Generator().manual_seed(5))
        with torch.no_grad():
            model.model[1].bn.bias += 100.0
    else:
        x = synth.synth_image(B, H, W, seed=5)
    run0 = {id(m): (m.running_mean.detach().clone(), m.running_var.detach().clone()) for m in model.modules() if isinstance(m, torch.nn.BatchNorm2d)}
    eng = model.engine()
    raws, seg, plan = eng.train_forward(x.cuda())
    segs = seg if isinstance(seg, list) else [seg]
    gen = torch.Generator().manual_seed(11)
    # a flat map has a tiny batch std, so its BN backward multiplies the gradient by a large 1/std: the seeds are scaled down like a loss
    # scaler would, to keep the fp16 gradient buffers of the first layers in range
    seed_scale = 2.0 ** -6 if image == "flat" else 1.0
    R = [(torch.randn(r.shape, generator=gen) * 4.0 * seed_scale).cuda() for r in raws]
    S = [(torch.randn(g.shape, generator=gen) * 0.05 * seed_scale).cuda() for g in segs]
    eng.train_backward(plan, R, S)
    torch.cuda.synchronize()
    return SimpleNamespace(model=model, eng=eng, plan=plan, pb=plan.pb, x=x.cuda(), raws=raws, segs=segs, R=R, S=S, run0=run0, B=B, H=H, W=W,
                           cache={}, gcache={})


def read(st, v, grad=False):
    """a view of the plan's activation (or gradient) workspace as (B, C, H, W) fp64"""
    key = (v.buf.id, v.c_off, v.c)
    cache = st.gcache if grad else st.cache
    if key not in cache:
        cache[key] = (st.eng.read_grad_view(v, st.plan) if grad else st.eng.read_view(v, st.plan)).double()
    return cache[key]


# ---- fp64 restatements, one per op kind (oracle/restate.py) -------------------------------------------------------------------
def wrong_grad(right, wrong):
    """the value of `right` with the gradient of `wrong`: the mutants of the sensitivity test change only the backward"""
    return right.detach() + (wrong - wrong.detach())


def act(z, a, mutant=None):
    from multiyolov5_b200._lib import ACT_SIGMOID, ACT_SILU
    if a == ACT_SILU:                                    # nn.SiLU (mutant "silu": d/dz = sigmoid(z) instead of s (1 + z (1 - s)))
        s = torch.sigmoid(z)
        return z * (s.detach() if mutant == "silu" else s)
    if a == ACT_SIGMOID:
        return torch.sigmoid(z)
    return z


def op_params(st, op):
    """fp64 leaves of the master parameters an op reads, keyed by the model tensor they stand for"""
    from multiyolov5_b200._lib import OP_BN_ACT, OP_CONV
    if op.kind == OP_CONV:
        conv = st.pb.slots[op.slot].conv
        ts = {"w": ("conv.weight", conv.weight)} | ({"b": ("conv.bias", conv.bias)} if conv.bias is not None else {})
    elif op.kind == OP_BN_ACT:
        bn = st.pb.bn_slots[op.aux[0]]
        ts = {"g": ("bn.weight", bn.weight), "b": ("bn.bias", bn.bias)}
    else:
        return {}, {}
    return {k: t.detach().double().requires_grad_(True) for k, (_, t) in ts.items()}, ts


def restate(st, i, op, ins, prm, mutant=None):
    from multiyolov5_b200 import _lib as L
    x, k = ins[0], op.kind
    if k == L.OP_CONV:        # raw conv (train mode: BN is its own op) on the first ci channels; the kernels multiply fp16 weight packs
        conv = st.pb.slots[op.slot].conv
        w = prm["w"]
        wq = w + (w.detach().float().half().double() - w.detach())
        xs, pad = x[:, :conv.in_channels], op.dil * (op.k // 2)
        y = F.conv2d(xs, wq, prm.get("b"), op.stride, pad, op.dil)
        if mutant == "unflipped" and op.k == 3:          # data gradient with the 3x3 kernel not flipped
            y = wrong_grad(y, F.conv2d(xs, wq.flip(2, 3), prm.get("b"), op.stride, pad, op.dil))
        return y
    if k == L.OP_BN_ACT:      # F.batch_norm(training=True): batch statistics of the stored u, biased variance, the slot's eps
        bn = st.pb.bn_slots[op.aux[0]]
        mean, var = x.mean((0, 2, 3), keepdim=True), x.var((0, 2, 3), unbiased=False, keepdim=True)
        if mutant == "bn":                               # BN backward without its two mean terms
            mean, var = mean.detach(), var.detach()
        z = (x - mean) / torch.sqrt(var + bn.eps) * prm["g"].view(1, -1, 1, 1) + prm["b"].view(1, -1, 1, 1)
        y = act(z, op.act, mutant)
        return y + ins[1] if len(ins) > 1 else y
    if k == L.OP_ACT:
        return act(x, op.act, mutant)
    if k == L.OP_ADD:
        return x + ins[1]
    if k == L.OP_BROADCAST:
        return x.expand(-1, -1, op.out.h, op.out.w)
    if k == L.OP_CHANNEL_SCALE_OOP:                      # FFM: feat * att + feat
        return x * (1.0 + ins[1])
    if k == L.OP_UPSAMPLE_NEAREST:
        y = x.repeat_interleave(2, 2).repeat_interleave(2, 3)
        if mutant == "nearest":                          # adjoint that takes one pixel of the four
            m = torch.zeros_like(y)
            m[..., ::2, ::2] = 1.0
            y = wrong_grad(y, y * m)
        return y
    if k == L.OP_BILINEAR:
        y = F.interpolate(x, (op.out.h, op.out.w), mode="bilinear", align_corners=True)
        if mutant == "bilinear":
            y = wrong_grad(y, F.interpolate(x, (op.out.h, op.out.w), mode="bilinear", align_corners=False))
        return y
    if k == L.OP_SPP_POOL:    # SPP: max pools 5, 9, 13 (stride 1, -inf padding) of the same input into three slices
        return torch.cat([F.max_pool2d(x, kk, 1, kk // 2) for kk in (5, 9, 13)], 1)
    if k == L.OP_REGION_SUM:  # atom sums over the cells of the plan's y / x edge tables
        ex = st.pb.extra
        ys, xs = ex[op.aux[0]:op.aux[0] + op.aux[1] + 1], ex[op.aux[2]:op.aux[2] + op.aux[3] + 1]
        rows = torch.stack([x[:, :, a:b].sum(2) for a, b in zip(ys[:-1], ys[1:])], 2)
        return torch.stack([rows[..., a:b].sum(3) for a, b in zip(xs[:-1], xs[1:])], 3)
    if k == L.OP_REGION_COMBINE:   # bin = sum of its atoms / pixel count, table rows [ay0, ay1, ax0, ax1, count]
        t = st.pb.extra[op.aux[0]:op.aux[0] + 5 * op.aux[1]]
        bins = [x[:, :, t[5 * j]:t[5 * j + 1], t[5 * j + 2]:t[5 * j + 3]].sum((2, 3)) / t[5 * j + 4] for j in range(op.aux[1])]
        return torch.stack(bins, 2).view(x.shape[0], x.shape[1], op.out.h, op.out.w)
    if k == L.OP_DROPOUT:
        return x * st.keep[i] / (1.0 - op.faux[0])
    if k == L.OP_SEG_UPSAMPLE:
        return F.interpolate(x[:, :op.aux[0]], (st.H, st.W), mode="bilinear", align_corners=True)
    if k == L.OP_DETECT_DECODE:    # raw x_i (B, na, ny, nx, no) = conv output channels a*no + o
        na, no = op.aux[1], op.aux[2]
        return x[:, :na * no].reshape(x.shape[0], na, no, x.shape[2], x.shape[3]).permute(0, 1, 3, 4, 2)
    raise AssertionError(f"op {i}: no restatement of kind {k}")


def stored_out(st, op, grad=False):
    """what the plan computed for op (grad: the final gradient of its output): caller-owned outputs for the two seed ops"""
    from multiyolov5_b200 import _lib as L
    if op.kind == L.OP_SEG_UPSAMPLE:
        return (st.S if grad else st.segs)[op.aux[1]].double()
    if op.kind == L.OP_DETECT_DECODE:
        return (st.R if grad else st.raws)[op.aux[0]].double()
    return read(st, op.out, grad)


def op_inputs(op):
    return [v for v in (op.in_, op.in2) if v is not None]


# ---- the checks --------------------------------------------------------------------------------------------------------------
def forward_check(st):
    """per op: max over elements of (|ours - ref| - U16 |ref|) / max |ref|; also fills st.keep (dropout masks) and st.exclude"""
    from multiyolov5_b200 import _lib as L
    names = kind_names()
    st.keep, st.exclude, st.bn_u = {}, {}, {}
    errs = []
    for i, op in enumerate(st.pb.ops):
        if op.kind == L.OP_INPUT_FOCUS:   # space-to-depth of the fp16-rounded input (reference Focus), zero channels 12..15
            x = st.x.half().double()
            ref = torch.cat([x[..., ::2, ::2], x[..., 1::2, ::2], x[..., ::2, 1::2], x[..., 1::2, 1::2], torch.zeros_like(x[..., ::2, ::2][:, :1].expand(-1, 4, -1, -1))], 1)
            ours = read(st, op.out)
        else:
            ins = [read(st, v) for v in op_inputs(op)]
            if op.kind == L.OP_DROPOUT:   # the keep mask the kernel applied, read back; an element whose input is 0 has no readable mask
                out = read(st, op.out)
                st.keep[i] = ((out != 0) | (ins[0] == 0)).double()
                st.exclude[op.in_.buf.id] = (op.in_, ins[0] == 0)
                frac = float(st.keep[i].mean())
                assert abs(frac - (1.0 - op.faux[0])) < 0.01, (i, frac)
            if op.kind == L.OP_BN_ACT:
                st.bn_u[i] = ins[0]
            prm, _ = op_params(st, op)
            with torch.no_grad():
                ref = restate(st, i, op, ins, prm)
            ours = stored_out(st, op)[:, :ref.shape[1]] if op.kind != L.OP_DETECT_DECODE else stored_out(st, op)
        assert ours.shape == ref.shape, (i, names[op.kind], ours.shape, ref.shape)
        scale = float(ref.abs().max())
        e = float(((ours - ref).abs() - U16 * ref.abs()).clamp_min(0).max()) / max(scale, 1e-30)
        errs.append((i, names[op.kind], e))
    # REGION_SUM + REGION_COMBINE together are adaptive_avg_pool2d of the pooled map (the plan's bin tables against ATen's index math)
    for op in st.pb.ops:
        if op.kind == L.OP_REGION_COMBINE:
            src = [o for o in st.pb.ops if o.kind == L.OP_REGION_SUM and o.out.buf is op.in_.buf][0]
            x = read(st, src.in_)
            with torch.no_grad():
                pooled = restate(st, -1, op, [restate(st, -1, src, [x], {})], {})
            ref = F.adaptive_avg_pool2d(x, (op.out.h, op.out.w))
            assert float((pooled - ref).abs().max()) <= 1e-12 * max(1.0, float(ref.abs().max())), op.out.h
    return errs


def backward_check(st, mutant=None):
    """autograd of every op's restatement, seeded with the op's final output gradient from the plan; contributions summed per buffer
    and channel slice and compared with the gradient workspace.  Returns per-buffer errors, the kinds that read each buffer, and the
    fp64 parameter gradients"""
    from multiyolov5_b200 import _lib as L
    from multiyolov5_b200.plan import V
    names = kind_names()
    acc, readers = {}, defaultdict(set)
    pgrad = {}
    for i, op in enumerate(st.pb.ops):
        if op.kind == L.OP_INPUT_FOCUS:
            continue
        views = op_inputs(op)
        leaves = [read(st, v).clone().requires_grad_(True) for v in views]
        prm, ts = op_params(st, op)
        y = restate(st, i, op, leaves, prm, mutant)
        gy = stored_out(st, op, grad=True)
        if op.kind != L.OP_DETECT_DECODE:
            gy = gy[:, :y.shape[1]]
        gs = torch.autograd.grad(y, leaves + list(prm.values()), gy, allow_unused=True)
        for v, g in zip(views, gs[:len(views)]):
            readers[v.buf.id].add(names[op.kind])
            if v.buf.id not in acc:
                acc[v.buf.id] = (v.buf, torch.zeros((st.B, v.buf.c, v.buf.h, v.buf.w), dtype=torch.float64, device=st.x.device))
            if g is not None:
                acc[v.buf.id][1][:, v.c_off:v.c_off + v.c] += g
        for key, g in zip(prm, gs[len(views):]):
            kind, t = ts[key]
            # a BN parameter gradient is a sum over pixels that can cancel (the next BN removes the mean of the gradient): measured against
            # one fp16 rounding of the output gradient it sums when that is larger
            floor = U16 * float(gy.norm()) if op.kind == L.OP_BN_ACT else 0.0
            pgrad[id(t)] = (kind, t, pgrad[id(t)][2] + g if id(t) in pgrad else g, floor)
    focus = {o.out.buf.id for o in st.pb.ops if o.kind == L.OP_INPUT_FOCUS}
    errs = []
    for bid, (buf, ref) in acc.items():
        if bid in focus:                 # the input conversion's buffer gets no data gradient
            continue
        ours = read(st, V(buf, 0, buf.c), grad=True)
        if bid in st.exclude:            # dropout inputs that are exactly 0: the keep mask is not readable there
            v, amb = st.exclude[bid]
            m = torch.ones_like(ref, dtype=torch.bool)
            m[:, v.c_off:v.c_off + v.c] = ~amb
            ours, ref = ours * m, ref * m
        rn, rmax = float(ref.norm()), float(ref.abs().max())
        d = ours - ref
        if rn == 0:
            assert float(d.abs().max()) == 0, f"buffer {bid} (read by {sorted(readers[bid])}): zero reference gradient, ours {float(d.abs().max())}"
            continue
        errs.append((bid, sorted(readers[bid]), float(d.norm()) / rn, float(d.abs().max()) / rmax))
    return errs, pgrad


def param_check(st, pgrad):
    """per conv slot / BN slot: relative Frobenius error of .grad against the fp64 sums; running statistics after the forward"""
    from multiyolov5_b200 import _lib as L
    rows = []
    for kind, t, g, floor in pgrad.values():
        if float(g.norm()) == 0:
            continue
        rows.append((kind, float((t.grad.double() - g).norm()) / max(float(g.norm()), floor)))
    for i, op in enumerate(st.pb.ops):
        if op.kind != L.OP_BN_ACT:
            continue
        bn, u = st.pb.bn_slots[op.aux[0]], st.bn_u[i]
        m, n = bn.momentum, u.numel() // u.shape[1]
        mean, var = u.mean((0, 2, 3)), u.var((0, 2, 3), unbiased=False)
        rm0, rv0 = [t.double() for t in st.run0[id(bn)]]
        for kind, ours, ref, stat in (("running_mean", bn.running_mean, (1 - m) * rm0 + m * mean, torch.maximum(mean.abs(), var.sqrt())),
                                      ("running_var", bn.running_var, (1 - m) * rv0 + m * var * n / max(n - 1, 1), var)):
            # four fp32 roundings of the update itself, then relative to the momentum-scaled batch statistic
            d = ((ours.double() - ref).abs() - 2.0 ** -22 * ref.abs()).clamp_min(0)
            rows.append((kind, float(d.max()) / (m * float(stat.max()))))
    return rows


def fmt_table(title, rows):
    lines = [title]
    for k, v, lim in rows:
        lines.append(f"  {k:<20} {v}  (limit {lim})")
    return "\n".join(lines)


def check_all(st):
    """runs the three checks, prints the per-kind table, returns the failures"""
    fwd = forward_check(st)
    bwd, pgrad = backward_check(st)
    prm = param_check(st, pgrad)
    fails = []
    worst_f = defaultdict(float)
    for i, kind, e in fwd:
        worst_f[kind] = max(worst_f[kind], e)
        if e > FWD_TOL[kind]:
            fails.append(f"forward op {i} {kind}: {e:.3e} > {FWD_TOL[kind]:.1e}")
    worst_b = defaultdict(lambda: [0.0, 0.0])
    for bid, kinds, ef, em in bwd:
        lf, lm = max(BWD_TOL[k][0] for k in kinds), max(BWD_TOL[k][1] for k in kinds)
        for k in kinds:
            worst_b[k][0], worst_b[k][1] = max(worst_b[k][0], ef), max(worst_b[k][1], em)
        if ef > lf or em > lm:
            fails.append(f"gradient of buffer {bid} (read by {'+'.join(kinds)}): rel {ef:.3e} (limit {lf:.1e}), max {em:.3e} (limit {lm:.1e})")
    worst_p = defaultdict(float)
    for kind, e in prm:
        worst_p[kind] = max(worst_p[kind], e)
        if e > PARAM_TOL[kind]:
            fails.append(f"{kind}: {e:.3e} > {PARAM_TOL[kind]:.1e}")
    print(fmt_table("forward, worst (|err| - fp16 rounding) / max|ref| per op kind:",
                    [(k, f"{v:.2e}", f"{FWD_TOL[k]:.0e}") for k, v in sorted(worst_f.items())]))
    print(fmt_table("backward, worst per gradient buffer by the kinds that read it (rel. Frobenius, max/max):",
                    [(k, f"{v[0]:.2e} {v[1]:.2e}", f"{BWD_TOL[k][0]:.0e} {BWD_TOL[k][1]:.0e}") for k, v in sorted(worst_b.items())]))
    print(fmt_table("parameters, worst per kind:", [(k, f"{v:.2e}", f"{PARAM_TOL[k]:.0e}") for k, v in sorted(worst_p.items())]))
    return fails, bwd


# ---- cases -------------------------------------------------------------------------------------------------------------------
CASES = {  # id: (model, B, H, W, image, MYOLO_FORCE_SIMT)
    "s_psp": ("s_psp", 2, 256, 512, "synth", False),                # mixed data-gradient paths
    "m_lab": ("m_lab", 4, 256, 512, "synth", False),                # kc = 16 wgmma data gradients, ASPP dilations on wgmma
    "s_bise": ("s_bise", 2, 256, 512, "synth", False),              # dropout, ADD, BROADCAST, three seg seeds
    "s_base": ("s_base", 2, 256, 512, "synth", False),              # dropout, C3SPP in the head
    "s_psp_416x736": ("s_psp", 2, 416, 736, "synth", False),        # P32 13 x 23: overlapping adaptive bins, non-integer bilinear ratios
    "s_psp_512x1024": ("s_psp", 4, 512, 1024, "synth", False),      # the benchmark's per-GPU slice
    "s_psp_simt": ("s_psp", 2, 256, 512, "synth", True),            # data gradients on the CUDA-core conv kernel
    "s_psp_flat": ("s_psp", 2, 256, 512, "flat", False),            # mean >> spread channels, tied SPP maxima
}


def assert_coverage(name, st, simt):
    """each case hits what it claims: the data-gradient routes (counted by path, kc, stride, dilation) and the op kinds"""
    from multiyolov5_b200 import _lib as L
    pb = st.pb
    routes = dgrad_routes(pb, st.B, simt)
    count = defaultdict(int)
    for _, path, kc, s, d in routes:
        count[path] += 1
        if path == "wgmma":
            count[f"wgmma kc={kc}"] += 1
            count[f"wgmma s={s}"] += 1
            count[f"wgmma d={d}"] += 1
    kinds = defaultdict(int)
    for o in pb.ops:
        kinds[kind_names()[o.kind]] += 1
    print(f"\n[{name}] data-gradient convs: {dict(sorted(count.items()))}")
    print(f"[{name}] ops: {dict(sorted(kinds.items()))}")
    if name == "s_psp":
        assert count["small"] >= 10 and count["wgmma"] >= 5 and count["wgmma s=2"] >= 1
    if name == "m_lab":
        assert count["wgmma kc=16"] >= 10 and all(count[f"wgmma d={d}"] >= 1 for d in (3, 6, 9))
    if name == "s_bise":
        assert kinds["DROPOUT"] >= 1 and kinds["ADD"] >= 1 and kinds["BROADCAST"] >= 1 and kinds["SEG_UPSAMPLE"] == 3
    if name == "s_base":
        head_spp = [o for o in pb.ops if o.kind == L.OP_SPP_POOL and "SegMaskBase" in o.tag]
        assert kinds["DROPOUT"] >= 1 and len(head_spp) == 1
    if name == "s_psp_416x736":
        from multiyolov5_b200.plan import adaptive_bins
        assert any((b.h, b.w) == (13, 23) for b in pb.bufs)
        pooled = [(src.in_.h, src.in_.w, o.out.h) for o in pb.ops if o.kind == L.OP_REGION_COMBINE
                  for src in pb.ops if src.kind == L.OP_REGION_SUM and src.out.buf is o.in_.buf]
        overlap = [(h, w, k) for h, w, k in pooled for n in (h, w) if any(a[1] > b[0] for a, b in zip(adaptive_bins(n, k), adaptive_bins(n, k)[1:]))]
        print(f"[{name}] adaptive pools with overlapping bins (map h, w, bins): {sorted(set(overlap))}")
        assert overlap
        ratios = [((o.in_.h - 1) / (o.out.h - 1), (o.in_.w - 1) / (o.out.w - 1)) for o in pb.ops if o.kind == L.OP_BILINEAR and o.out.h > 1]
        assert any(r != int(r) for rr in ratios for r in rr)
    if name == "s_psp_512x1024":
        assert count["small"] == 6 and count["wgmma"] == len(routes) - 6
    if name == "s_psp_simt":
        assert count["wgmma"] == 0 and count["simt"] >= 20
    if name == "s_psp_flat":
        ratio = max(float((u.mean((0, 2, 3)).abs() / u.std((0, 2, 3)).clamp_min(1e-30)).max()) for u in st.bn_u.values())
        spp = [o for o in pb.ops if o.kind == L.OP_SPP_POOL][0]
        x = read(st, spp.in_)
        mx = F.max_pool2d(x, 5, 1, 2)
        xp = F.pad(x, (2, 2, 2, 2), value=-math.inf)
        hits = sum((xp[..., dy:dy + x.shape[2], dx:dx + x.shape[3]] == mx).int() for dy in range(5) for dx in range(5))
        ties = int((hits > 1).sum())
        print(f"[{name}] largest channel mean/std at a BN input: {ratio:.0f}; 5x5 SPP windows with a tied maximum: {ties}")
        assert ratio > 100 and ties >= 50


@pytest.mark.parametrize("name", list(CASES))
def test_every_train_op_matches_its_fp64_restatement(name, monkeypatch):
    """forward of every op against its restatement on the op's own stored inputs; backward of every buffer against autograd of the
    restatements of the ops that read it; parameter gradients and running statistics against fp64 references"""
    tag, B, H, W, image, simt = CASES[name]
    monkeypatch.setenv("MYOLO_FORCE_SIMT", "1" if simt else "0")
    torch.manual_seed(0)
    st = train_step(tag, B, H, W, image)
    fails, _ = check_all(st)
    assert_coverage(name, st, simt)
    assert not fails, "\n".join(fails[:20])


MUTANTS = {"bn": "BN_ACT", "bilinear": "BILINEAR", "unflipped": "CONV", "nearest": "UPSAMPLE_NEAREST", "silu": "BN_ACT"}


def test_layer_checks_catch_wrong_backward_formulas(monkeypatch):
    """the backward limits discriminate: with one deliberately wrong restatement the buffers its op kind feeds must miss their limit by
    at least 10x - BN backward without its mean terms, the bilinear adjoint with align_corners=False, the data gradient with an unflipped
    3x3 kernel, a nearest adjoint that takes one pixel of four, and sigmoid(z) as the SiLU derivative"""
    monkeypatch.setenv("MYOLO_FORCE_SIMT", "0")
    torch.manual_seed(0)
    st = train_step("s_psp", 2, 256, 512)
    forward_check(st)
    print()
    for mutant, kind in MUTANTS.items():
        errs, _ = backward_check(st, mutant)
        over = max(max(ef / max(BWD_TOL[k][0] for k in kinds), em / max(BWD_TOL[k][1] for k in kinds))
                   for _, kinds, ef, em in errs if kind in kinds)
        print(f"mutant {mutant:<10} ({kind}): worst buffer at {over:.0f}x its limit")
        assert over >= 10, (mutant, over)
