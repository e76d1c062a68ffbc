"""CPU: host-side logic - state_dict key parity of the shells, planner invariants (liveness packing, concat elimination,
dependency-safe aliasing), C-ABI library loads and exports every symbol declared in include/myolo.h (no compute calls)."""
import os
import re

import pytest
import torch

from oracle import synth

NETS = {"s_psp": "yolov5s_city_seg.yaml", "m_lab": "yolov5m_city_seg_lab.yaml", "s_bise": "yolov5s_city_seg_bise.yaml",
        "s_base": "yolov5s_city_seg_base.yaml", "m_psp": "yolov5m_city_seg.yaml"}
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("tag", list(NETS))
def test_state_dict_keys_match_reference_manifest(tag):
    from multiyolov5_b200.models.yolo import Model
    m = Model(NETS[tag])
    man = synth.load_manifest(tag)
    sd = m.state_dict()
    assert [k for k, _, _ in man] == list(sd.keys())
    assert all(list(sd[k].shape) == s for k, s, _ in man)
    assert m.stride.tolist() == [8.0, 16.0, 32.0]
    m.load_state_dict(synth.synth_state_dict(man, synth.load_cfg(NETS[tag]), seed=1))
    for mod in m.modules():
        if type(mod) is torch.nn.BatchNorm2d:
            assert mod.eps == 1e-3 and mod.momentum == 0.03   # reference utils/torch_utils.py:150-152


def test_model_surface():
    from multiyolov5_b200.models.yolo import Detect, Model
    m = Model("yolov5s_city_seg.yaml")
    det = m.model[-1]
    assert isinstance(det, Detect) and (det.nl, det.na, det.nc, det.no) == (3, 3, 10, 15)
    assert m.save == sorted(m.save[:-1]) + [24] and 24 in m.save
    assert m.names == [str(i) for i in range(10)]
    assert m.fuse() is m
    with pytest.raises(Exception):
        m.model[1](torch.zeros(1, 32, 8, 8))       # shells hold parameters only: no eager fallback
    m.train()
    with pytest.raises(Exception):                 # train mode exists, but only on CUDA tensors: no CPU path
        m(torch.zeros(1, 3, 64, 64))


@pytest.mark.parametrize("tag,B,H,W", [("s_psp", 16, 512, 1024), ("m_lab", 8, 512, 1024), ("s_bise", 2, 256, 256), ("s_base", 1, 64, 96)])
def test_planner_op_and_buffer_invariants(tag, B, H, W):
    from multiyolov5_b200 import _lib
    from multiyolov5_b200.models.yolo import Model
    from multiyolov5_b200.plan import build_plan
    pb = build_plan(Model(NETS[tag]), B, H, W)
    n = len(pb.ops)
    aliases = [b for b in pb.bufs if b.alias_of is not None]
    for b in aliases:       # pixel-pair views (layer 0): same bytes, same total size, another (w, c) factorisation
        assert b.offset == b.alias_of.offset and b.nbytes(B) == b.alias_of.nbytes(B) and b.h == b.alias_of.h
    used = [b for b in pb.bufs if b.first >= 0 and b.alias_of is None]
    # liveness packing never overlaps two simultaneously-live buffers, and beats the unpacked footprint
    for i, a in enumerate(used):
        assert a.offset % 256 == 0 and a.offset + a.nbytes(B) <= pb.workspace_bytes
        for b in used[i + 1:]:
            if not (a.last < b.first or b.last < a.first):
                assert a.offset + a.nbytes(B) <= b.offset or b.offset + b.nbytes(B) <= a.offset, (a, b)
    assert pb.workspace_bytes < sum(b.nbytes(B) for b in used)
    # every conv reads exactly the (16-padded) input channels it was packed for; outputs land in slices (no concat copies)
    kinds = [o.kind for o in pb.ops]
    assert kinds.count(_lib.OP_INPUT_FOCUS) == 1   # layer 0: space-to-depth + conv
    assert kinds.count(_lib.OP_DETECT_DECODE) == 3 and kinds.count(_lib.OP_SEG_UPSAMPLE) == 1
    for o in pb.ops:
        if o.kind == _lib.OP_CONV:
            c = pb.slots[o.slot].conv
            assert o.in_.c == (c.in_channels + 15) // 16 * 16
            assert o.out.buf.dtype == _lib.F32 or o.out.c == c.out_channels
    # buffers read by the ops that run after the CUDA graph stay live to the end
    for o in pb.ops:
        if o.kind in (_lib.OP_DETECT_DECODE, _lib.OP_SEG_UPSAMPLE):
            assert o.in_.buf.last > n
    assert sum(pb.det_rows) == 3 * ((H // 8) * (W // 8) + (H // 16) * (W // 16) + (H // 32) * (W // 32))


def execution_intervals(pb):
    """[first, last] execution position of every base buffer of an inference plan, in the order the executor runs the ops: INPUT_FOCUS
    first, a group member in its head's launch, DETECT_DECODE and SEG_UPSAMPLE after the captured graph (csrc/plan.cu myolo_plan_forward)"""
    from multiyolov5_b200 import _lib
    n = len(pb.ops)
    pos, head = [], -1
    for i, o in enumerate(pb.ops):
        if o.flags & _lib.OP_GROUP_HEAD:
            head = i
        if o.kind == _lib.OP_INPUT_FOCUS:
            pos.append(-1)
        elif o.kind in (_lib.OP_DETECT_DECODE, _lib.OP_SEG_UPSAMPLE):
            pos.append(n)
        else:
            pos.append(head if o.flags & _lib.OP_GROUP_MEMBER else i)
    live = {}
    for o, p in zip(pb.ops, pos):
        for v in (o.in_, o.in2, o.out):
            if v is not None:
                b = v.buf.alias_of or v.buf
                f, l = live.get(b.id, (p, p))
                live[b.id] = (min(f, p), max(l, p))
    return pos, live


@pytest.mark.parametrize("tag", list(NETS))
def test_workspace_packing_respects_execution_order(tag):
    """buffers that share workspace bytes are never live at the same time in EXECUTION order (which differs from plan order: group
    members run in their head's launch, the caller-output ops after the graph), and no member of a grouped launch writes what another
    member of the same launch reads"""
    from multiyolov5_b200 import _lib
    from multiyolov5_b200.models.yolo import Model
    from multiyolov5_b200.plan import build_plan
    model = Model(NETS[tag])
    for B in (1, 2, 16):
        for H, W in ((128, 256), (256, 512), (416, 736), (512, 1024), (640, 640)):
            pb = build_plan(model, B, H, W)
            pos, live = execution_intervals(pb)
            bufs = {b.id: b for b in pb.bufs if b.alias_of is None and b.id in live}
            spans = sorted((b.offset, b.offset + b.nbytes(B), b.id) for b in bufs.values())
            for i, (o0, e0, a) in enumerate(spans):
                for o1, e1, b in spans[i + 1:]:
                    if o1 >= e0:
                        break
                    (fa, la), (fb, lb) = live[a], live[b]
                    assert la < fb or lb < fa, (B, H, W, f"buffers {a} and {b} share bytes and are live together: {live[a]} {live[b]}")
            for h in (i for i, o in enumerate(pb.ops) if o.flags & _lib.OP_GROUP_HEAD):
                members = pb.ops[h:h + pb.ops[h].aux[7]]
                for j, m in enumerate(members):
                    for k, r in enumerate(members):
                        for v in (r.in_, r.in2):
                            if j == k or v is None:
                                continue
                            wb, vb = m.out.buf.alias_of or m.out.buf, v.buf.alias_of or v.buf
                            same = wb is vb and m.out.c_off < v.c_off + v.c and v.c_off < m.out.c_off + m.out.c
                            apart = wb is not vb and (wb.offset + wb.nbytes(B) <= vb.offset or vb.offset + vb.nbytes(B) <= wb.offset)
                            assert not same and (wb is vb or apart), (B, H, W, h, j, k)


def test_adaptive_bins_match_torch():
    from multiyolov5_b200.plan import adaptive_bins
    import torch.nn.functional as F
    for n_in, k in [(64, 6), (64, 3), (128, 6), (8, 3), (12, 6), (7, 2), (5, 5)]:
        x = torch.arange(n_in, dtype=torch.float32).view(1, 1, 1, n_in)
        ref = F.adaptive_avg_pool2d(x, (1, k)).view(-1)
        mine = torch.tensor([sum(range(a, b)) / (b - a) for a, b in adaptive_bins(n_in, k)])
        assert torch.allclose(ref, mine)


def test_cabi_library_exports_header_symbols():
    from multiyolov5_b200 import _lib
    L = _lib.lib()                       # raises if the .so is missing: build() must have run
    hdr = open(os.path.join(ROOT, "include", "myolo.h")).read()
    declared = sorted(set(re.findall(r"\b(myolo_[a-z0-9_]+)\s*\(", hdr)))
    assert len(declared) >= 15
    for name in declared:
        assert hasattr(L, name), f"{name} declared in include/myolo.h but not exported"
    assert sorted(_lib.EXPORTS) == declared
    assert L.myolo_abi_version() == 1
    # no device here: entry points must fail loudly, not fall back
    if not torch.cuda.is_available():
        import ctypes as C
        h = C.c_void_p()
        ops = (_lib.Op * 1)(); bufs = (_lib.BufDesc * 1)()
        rc = L.myolo_plan_create(ops, 1, bufs, 1, None, 0, 1, 64, 64, 256, 0, C.byref(h))
        assert rc != 0 and len(L.myolo_last_error()) > 0


def test_product_never_imports_oracle():
    pkg = os.path.join(ROOT, "multiyolov5_b200")
    for dp, _, fs in os.walk(pkg):
        for f in fs:
            if f.endswith((".py", ".cu", ".cuh", ".h")):
                src = open(os.path.join(dp, f)).read()
                assert "oracle" not in src.replace("the oracle", "").replace("use the oracle for CPU numbers", ""), os.path.join(dp, f)


def test_letterbox_geometry_host_logic_matches_restatement():
    """the product's shape arithmetic for the device letterbox (resized size, padding, offsets) against the restatement of reference
    utils/datasets.py:818-845 over many frame shapes / options (importing the product module needs no GPU)"""
    import numpy as np
    from multiyolov5_b200.utils.datasets import letterbox_geometry
    from oracle import restate
    rs = np.random.RandomState(0)
    for _ in range(300):
        shape = (int(rs.randint(17, 2200)), int(rs.randint(17, 2200)))
        new_shape = int(rs.choice([320, 512, 640, 1024])) if rs.rand() < 0.5 else (int(rs.randint(2, 40)) * 32, int(rs.randint(2, 40)) * 32)
        kw = dict(auto=bool(rs.rand() < 0.5), scaleFill=bool(rs.rand() < 0.2), scaleup=bool(rs.rand() < 0.7), stride=int(rs.choice([32, 64])))
        a = letterbox_geometry(shape, new_shape, **kw)
        b = restate.letterbox_geometry(shape, new_shape, **kw)
        assert a[0] == b[0] and a[3] == b[3] and np.allclose(a[1], b[1]) and np.allclose(a[2], b[2]), (shape, new_shape, kw)


def test_trainer_parameter_groups_follow_reference_rules():
    """pg0 = BatchNorm weights (no decay), pg1 = other weights (decay), pg2 = biases (reference train.py:108-116)"""
    from multiyolov5_b200.models.yolo import Model
    from multiyolov5_b200.train import parameter_groups, scale_hyp
    import torch.nn as nn
    model = Model("yolov5s_city_seg.yaml")
    grp = parameter_groups(model)
    named = dict(model.named_parameters())
    assert len(grp) == len(named) == 229                          # SURVEY 8 a13: 229 gradient tensors for s/PSP
    bn_weights = {id(m.weight) for m in model.modules() if isinstance(m, nn.BatchNorm2d)}
    assert len(bn_weights) > 60
    for name, p in named.items():
        g = grp[id(p)]
        if name.endswith(".bias"):
            assert g == 2, name
        elif id(p) in bn_weights:
            assert g == 0, name
        else:
            assert g == 1 and p.dim() == 4, name           # conv weights
    h = scale_hyp(dict(weight_decay=5e-4, box=0.05, cls=0.5, obj=1.0), nl=3, nc=10, imgsz=1024, total_batch_size=32)
    assert abs(h["weight_decay"] - 5e-4 * 32 * 2 / 64) < 1e-12 and abs(h["cls"] - 0.5 * 10 / 80) < 1e-12 and abs(h["obj"] - (1024 / 640) ** 2) < 1e-12


def test_train_plans_build_for_every_head_and_only_use_differentiable_ops():
    """planner, train=True: all five shipped configs lower to op kinds that the backward walk implements (csrc/plan.cu: backward_walk),
    nothing aliases, BiSe exposes its three seg outputs with indices 0/1/2 and the Base / BiSe dropout becomes an op"""
    from multiyolov5_b200 import _lib, plan as P
    from multiyolov5_b200.models.yolo import Model
    differentiable = {_lib.OP_CONV, _lib.OP_BN_ACT, _lib.OP_ACT, _lib.OP_DROPOUT, _lib.OP_CHANNEL_SCALE_OOP, _lib.OP_UPSAMPLE_NEAREST,
                      _lib.OP_BILINEAR, _lib.OP_SPP_POOL, _lib.OP_REGION_COMBINE, _lib.OP_REGION_SUM, _lib.OP_ADD, _lib.OP_BROADCAST}
    seeds = {_lib.OP_INPUT_FOCUS, _lib.OP_DETECT_DECODE, _lib.OP_SEG_UPSAMPLE}
    for yml, n_seg, n_drop in (("yolov5s_city_seg.yaml", 1, 0), ("yolov5m_city_seg_lab.yaml", 1, 0), ("yolov5s_city_seg_base.yaml", 1, 1),
                               ("yolov5s_city_seg_bise.yaml", 3, 1), ("yolov5m_city_seg.yaml", 1, 0)):
        pb = P.build_plan(Model(yml), 2, 128, 256, train=True)
        kinds = [o.kind for o in pb.ops]
        assert set(kinds) <= differentiable | seeds, (yml, set(kinds) - differentiable - seeds)
        segs = [o for o in pb.ops if o.kind == _lib.OP_SEG_UPSAMPLE]
        assert sorted(o.aux[1] for o in segs) == list(range(n_seg)), yml
        assert kinds.count(_lib.OP_DROPOUT) == n_drop and kinds.count(_lib.OP_DETECT_DECODE) == 3, yml
        assert len(pb.bn_slots) == kinds.count(_lib.OP_BN_ACT) > 60, yml
        # train plans keep every buffer: no two buffers share workspace bytes
        spans = sorted((b.offset, b.offset + 2 * b.h * b.w * b.c * (1 if b.dtype == _lib.F16 else 2) * 2) for b in pb.bufs)
        assert all(a[1] <= b[0] for a, b in zip(spans, spans[1:])), yml
        # eval plans of the same model have a single seg output and no train-only ops
        pe = P.build_plan(Model(yml), 2, 128, 256)
        ke = [o.kind for o in pe.ops]
        assert ke.count(_lib.OP_SEG_UPSAMPLE) == 1 and not ({_lib.OP_BN_ACT, _lib.OP_DROPOUT, _lib.OP_ACT} & set(ke)), yml


def test_c3_pair_fusion_plan(monkeypatch):
    """the two 1x1 convs of a C3 that read the same input become one conv with concatenated output channels (default; MYOLO_FUSE_C3=0
    restores one launch per reference Conv module)"""
    import torch
    from multiyolov5_b200 import _lib, plan as P
    from multiyolov5_b200.models.yolo import Model
    model = Model("yolov5s_city_seg.yaml")
    monkeypatch.setenv("MYOLO_FUSE_C3", "0")
    base = P.build_plan(model, 1, 64, 64)
    monkeypatch.delenv("MYOLO_FUSE_C3")
    fused = P.build_plan(model, 1, 64, 64)
    n_base = sum(o.kind == _lib.OP_CONV for o in base.ops)
    n_fused = sum(o.kind == _lib.OP_CONV for o in fused.ops)
    assert n_base == 79 and n_fused == 71                                       # 8 C3 blocks
    merged = [s for s in fused.slots if s.name == "c3.cv1+cv2"]
    c3 = model.model[2]
    assert torch.equal(merged[0].conv.weight, torch.cat([c3.cv1.conv.weight, c3.cv2.conv.weight], 0))
    assert torch.equal(merged[0].bn.running_var, torch.cat([c3.cv1.bn.running_var, c3.cv2.bn.running_var], 0))
    assert len(P.build_plan(model, 1, 64, 64, train=True).ops) > len(base.ops)          # train plans are never fused


def test_inference_plan_always_lowers_detect_before_the_seg_head():
    """execution order is a planner decision: the Detect layer (yaml index 25) is lowered before the seg head (24) it follows - neither reads
    the other - so that the captured graph ends with the seg classifier conv; train plans keep the yaml order"""
    from multiyolov5_b200 import _lib, plan as P
    from multiyolov5_b200.models.yolo import Model
    model = Model("yolov5s_city_seg.yaml")

    def first_last(pb):
        det = [i for i, o in enumerate(pb.ops) if o.tag.startswith("L25:")]
        seg = [i for i, o in enumerate(pb.ops) if o.tag.startswith("L24:")]
        return det, seg
    det, seg = first_last(P.build_plan(model, 1, 64, 128))
    assert det and seg and max(det) < min(seg)
    det, seg = first_last(P.build_plan(model, 1, 64, 128, train=True))
    assert max(seg) < min(det)
    # the ops reading caller-owned outputs keep their inputs alive to the end of the plan
    pb = P.build_plan(model, 1, 64, 128)
    for o in pb.ops:
        if o.kind in (_lib.OP_DETECT_DECODE, _lib.OP_SEG_UPSAMPLE):
            assert o.in_.buf.last > len(pb.ops)


def test_global_average_pool_is_split_into_atoms():
    """AdaptiveAvgPool2d(1) of the FFM attention: one bin per image would be one CTA per image; the planner cuts it into 16 x 4 atoms whose
    fp32 sums the combine step adds up (REGION_SUM aux = [ybounds, ny, xbounds, nx])"""
    from multiyolov5_b200 import _lib, plan as P
    from multiyolov5_b200.models.yolo import Model
    pb = P.build_plan(Model("yolov5s_city_seg.yaml"), 2, 512, 1024)
    sums = [o for o in pb.ops if o.kind == _lib.OP_REGION_SUM]
    assert len(sums) == 2                                                        # the pooling pyramid and the FFM global pool
    ny, nx = sums[-1].aux[1], sums[-1].aux[3]
    assert (ny, nx) == (16, 4)
    ys = pb.extra[sums[-1].aux[0]: sums[-1].aux[0] + ny + 1]
    xs = pb.extra[sums[-1].aux[2]: sums[-1].aux[2] + nx + 1]
    assert ys[0] == 0 and ys[-1] == 64 and xs[0] == 0 and xs[-1] == 128 and list(ys) == sorted(set(ys)) and list(xs) == sorted(set(xs))
