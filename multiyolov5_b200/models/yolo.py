"""`Model(cfg).forward` of the reference (reference models/yolo.py:233-370) on a compiled sm_90a layer plan.

Surface kept from the reference: Model(cfg='*.yaml' | dict, ch=3, nc=None, anchors=None), .forward(x) ->
eval `[(z, [x0,x1,x2]), seg]`, .fuse(), .stride, .names, .yaml, .save, .model[-1] (Detect with nl/na/nc/no/anchors/
anchor_grid/stride), state_dict() keys (tests/golden/manifest_*.json).  The seg heads and Detect are parameter shells like
models/common.py; all arithmetic runs in libmyolo_sm90a.so.
"""
import math
import os
from copy import deepcopy

import torch
import torch.nn as nn

from .common import (ASPP, C3, C3SPP, FFM, RFB2, SPP, Bottleneck, Concat, Conv, Focus, PyramidPooling, _PlanOnly)  # noqa: F401

_CFG_DIR = os.path.dirname(os.path.abspath(__file__))


def make_divisible(x, divisor):  # reference utils/general.py:176-178
    return math.ceil(x / divisor) * divisor


def _bilinear(scale):
    return nn.Upsample(scale_factor=scale, mode="bilinear", align_corners=True)


class SegMaskPSP(_PlanOnly):  # reference models/yolo.py:149-186
    def __init__(self, n_segcls=19, n=1, c_hid=256, shortcut=False, ch=()):
        super().__init__()
        self.c_in8, self.c_in16, self.c_in32, self.c_out, self.c_hid = ch[0], ch[1], ch[2], n_segcls, c_hid
        self.out = nn.Sequential(RFB2(c_hid * 3, c_hid, d=[2, 3], map_reduce=6), PyramidPooling(c_hid, k=[1, 2, 3, 6]),
                                 FFM(c_hid * 2, c_hid, k=3, is_cat=False), nn.Conv2d(c_hid, self.c_out, kernel_size=1, padding=0),
                                 _bilinear(8))
        self.m8 = nn.Sequential(Conv(self.c_in8, c_hid, k=1))
        self.m32 = nn.Sequential(Conv(self.c_in32, c_hid, k=1), _bilinear(4))
        self.m16 = nn.Sequential(Conv(self.c_in16, c_hid, k=1), _bilinear(2))


class SegMaskLab(_PlanOnly):  # reference models/yolo.py:93-124
    def __init__(self, n_segcls=19, n=1, c_hid=256, shortcut=False, ch=()):
        super().__init__()
        self.c_detail, self.c_in16, self.c_out, self.c_hid = ch[0], ch[1], n_segcls, c_hid
        self.detail = nn.Sequential(Conv(self.c_detail, 48, k=1), Conv(48, 48, k=3))
        self.encoder = nn.Sequential(Conv(self.c_in16, c_hid * 2, k=1),
                                     ASPP(c_hid * 2, 256, d=[3, 6, 9], has_globel=False, map_reduce=5 - n), _bilinear(2))
        self.decoder = nn.Sequential(FFM(256 + 48, 256, k=1, is_cat=True), Conv(256, c_hid, k=3),
                                     nn.Conv2d(c_hid, self.c_out, kernel_size=1, padding=0), _bilinear(8))


class SegMaskBiSe(_PlanOnly):  # reference models/yolo.py:30-86
    def __init__(self, n_segcls=19, n=1, c_hid=256, shortcut=False, ch=()):
        super().__init__()
        self.c_in8, self.c_in16, self.c_in32, self.c_out = ch[0], ch[1], ch[2], n_segcls
        self.m8 = nn.Sequential(Conv(self.c_in8, 128, k=1, s=1))
        self.m16 = nn.Sequential(RFB2(self.c_in16, 128, map_reduce=4, d=[2, 3], has_globel=False))
        self.m32 = nn.Sequential(RFB2(self.c_in32, 128, map_reduce=8, d=[2, 3], has_globel=True))
        self.up16 = nn.Sequential(Conv(128, 128, 3), _bilinear(2))
        self.up32 = nn.Sequential(Conv(128, 128, 3), _bilinear(2))
        self.out = nn.Sequential(FFM(256, 256, k=3), nn.Dropout(0.1), nn.Conv2d(256, self.c_out, kernel_size=1, padding=0), _bilinear(8))
        self.aux16 = nn.Sequential(Conv(128, 128, 3), nn.Conv2d(128, self.c_out, kernel_size=1), _bilinear(8))
        self.aux32 = nn.Sequential(Conv(128, 128, 3), nn.Conv2d(128, self.c_out, kernel_size=1), _bilinear(16))


class SegMaskBase(_PlanOnly):  # reference models/yolo.py:129-146
    def __init__(self, n_segcls=19, n=1, c_hid=256, shortcut=False, ch=()):
        super().__init__()
        self.c_in, self.c_out = ch[0], n_segcls
        self.m = nn.Sequential(C3(c1=self.c_in, c2=c_hid, n=n, shortcut=shortcut, g=1, e=0.5),
                               C3SPP(c1=c_hid, c2=int(c_hid * 1.5), k=(5, 9, 13), g=1, e=0.5), nn.Dropout(0.1, True),
                               nn.Conv2d(int(c_hid * 1.5), self.c_out, kernel_size=(3, 3), stride=(1, 1), padding=(1, 1), groups=1,
                                         bias=False), _bilinear(8))


class Detect(_PlanOnly):  # reference models/yolo.py:189-230
    stride = None
    export = False

    def __init__(self, nc=80, anchors=(), ch=()):
        super().__init__()
        self.nc, self.no, self.nl, self.na = nc, nc + 5, len(anchors), len(anchors[0]) // 2
        a = torch.tensor(anchors).float().view(self.nl, -1, 2)
        self.register_buffer("anchors", a)
        self.register_buffer("anchor_grid", a.clone().view(self.nl, 1, -1, 1, 1, 2))
        self.m = nn.ModuleList(nn.Conv2d(x, self.no * self.na, 1) for x in ch)


_MODULES = dict(Conv=Conv, C3=C3, SPP=SPP, Focus=Focus, Concat=Concat, Detect=Detect, SegMaskPSP=SegMaskPSP, SegMaskLab=SegMaskLab,
                SegMaskBiSe=SegMaskBiSe, SegMaskBase=SegMaskBase)
_MODULES["nn.Upsample"] = nn.Upsample
_SEG_HEADS = (SegMaskPSP, SegMaskLab, SegMaskBiSe, SegMaskBase)


def parse_model(d, ch):
    """yaml dict -> (nn.Sequential, savelist); channel/depth scaling rules of reference models/yolo.py:373-429."""
    anchors, nc, gd, gw, n_segcls = d["anchors"], d["nc"], d["depth_multiple"], d["width_multiple"], d["n_segcls"]
    na = (len(anchors[0]) // 2) if isinstance(anchors, list) else anchors
    no = na * (nc + 5)
    names = dict(nc=nc, anchors=anchors, n_segcls=n_segcls)
    layers, save, c2 = [], [], ch[-1]
    for i, (f, n, mname, args) in enumerate(d["backbone"] + d["head"]):
        if mname not in _MODULES:
            raise NotImplementedError(f"module '{mname}' is not on the *_city_seg hot path (SURVEY.md section 8)")
        m = _MODULES[mname]
        args = [names[a] if isinstance(a, str) and a in names else (None if a == "None" else (False if a == "False" else (True if a == "True" else a)))
                for a in args]
        n = max(round(n * gd), 1) if n > 1 else n
        if m in (Conv, SPP, Focus, C3):
            c1, c2 = ch[f], args[0]
            if c2 != no:
                c2 = make_divisible(c2 * gw, 8)
            args = [c1, c2, *args[1:]]
            if m is C3:
                args.insert(2, n)
                n = 1
        elif m is Concat:
            c2 = sum(ch[x] for x in f)
        elif m is Detect:
            args.append([ch[x] for x in f])
            if isinstance(args[1], int):  # an anchor count: placeholder anchors that autoanchor replaces (reference models/yolo.py:405-406)
                args[1] = [list(range(args[1] * 2))] * len(f)
        elif m in _SEG_HEADS:
            args[1] = max(round(args[1] * gd), 1) if args[1] > 1 else args[1]
            args[2] = make_divisible(args[2] * gw, 8)
            args.append([ch[x] for x in f])
        else:
            c2 = ch[f]
        m_ = nn.Sequential(*[m(*args) for _ in range(n)]) if n > 1 else m(*args)
        m_.i, m_.f, m_.type = i, f, mname if mname.startswith("nn.") else f"models.common.{mname}" if m not in (Detect, *_SEG_HEADS) else mname
        m_.np = sum(x.numel() for x in m_.parameters())
        save.extend(x % i for x in ([f] if isinstance(f, int) else f) if x != -1)
        layers.append(m_)
        if i == 0:
            ch = []
        ch.append(c2)
    return nn.Sequential(*layers), sorted(save)


class Model(nn.Module):
    def __init__(self, cfg="yolov5s_city_seg.yaml", ch=3, nc=None, anchors=None):
        super().__init__()
        if isinstance(cfg, dict):
            self.yaml = deepcopy(cfg)
        else:
            import yaml
            path = cfg if os.path.isfile(cfg) else os.path.join(_CFG_DIR, os.path.basename(cfg))
            self.yaml_file = os.path.basename(path)
            with open(path) as f:
                self.yaml = yaml.safe_load(f)
        ch = self.yaml["ch"] = self.yaml.get("ch", ch)
        if nc and nc != self.yaml["nc"]:
            self.yaml["nc"] = nc
        if anchors:
            self.yaml["anchors"] = round(anchors)
        self.model, self.save = parse_model(deepcopy(self.yaml), ch=[ch])
        self.save.append(24)  # seg layer is always kept (reference models/yolo.py:253)
        self.names = [str(i) for i in range(self.yaml["nc"])]
        m = self.model[-1]
        if isinstance(m, Detect):
            # the reference infers strides from a dry-run forward (models/yolo.py:260-261); the graph's strides are static
            m.stride = torch.tensor(self._static_strides(m))
            m.anchors /= m.stride.view(-1, 1, 1)
            # check_anchor_order (reference utils/autoanchor.py:12-20)
            a = m.anchor_grid.prod(-1).view(-1)
            if (a[-1] - a[0]).sign() != (m.stride[-1] - m.stride[0]).sign():
                m.anchors[:] = m.anchors.flip(0)
                m.anchor_grid[:] = m.anchor_grid.flip(0)
            self.stride = m.stride
            self._initialize_biases()
        for mod in self.modules():  # reference utils/torch_utils.py:145-154
            if type(mod) is nn.BatchNorm2d:
                mod.eps, mod.momentum = 1e-3, 0.03
        self._engine = None

    # ---- reference helpers -----------------------------------------------------------------------------------------
    def _static_strides(self, det):
        from ..plan import infer_strides
        s = infer_strides(self)
        return [float(s[j]) for j in det.f]

    def _initialize_biases(self, cf=None):  # reference models/yolo.py:318-326
        m = self.model[-1]
        for mi, s in zip(m.m, m.stride):
            b = mi.bias.view(m.na, -1)
            b.data[:, 4] += math.log(8 / (640 / s) ** 2)
            b.data[:, 5:] += math.log(0.6 / (m.nc - 0.99)) if cf is None else torch.log(cf / cf.sum())
            mi.bias = torch.nn.Parameter(b.view(-1), requires_grad=True)

    def fuse(self):
        """BN folding happens inside the plan's weight packing (myolo_plan_set_conv_weights); module structure and
        state_dict keys stay those of the un-fused reference model.  Kept for `attempt_load(...).fuse().eval()` call sites."""
        self.invalidate_weights()
        return self

    def info(self, verbose=False, img_size=640):
        n_p = sum(x.numel() for x in self.parameters())
        print(f"Model Summary: {len(list(self.modules()))} layers, {n_p} parameters")

    # ---- plan / engine ---------------------------------------------------------------------------------------------
    def invalidate_weights(self):
        """parameters or buffers were written where torch's version counters do not see it (raw pointers: the Trainer's fused optimiser,
        ModelEMA.update; new storage: _apply, load_state_dict): every compiled plan re-packs its weights before its next launch"""
        if getattr(self, "_engine", None) is not None:
            self._engine.param_epoch += 1

    def tensors_moved(self):
        """parameters / buffers may have new storage or dtype (_apply, load_state_dict, the Trainer's flat buffers): bumps the counter
        that tables of raw pointers into them (ModelEMA's device table) compare against"""
        self._tensor_epoch = getattr(self, "_tensor_epoch", 0) + 1

    def load_state_dict(self, *a, **k):
        r = super().load_state_dict(*a, **k)
        self.invalidate_weights()
        self.tensors_moved()
        return r

    def _apply(self, fn, *a, **k):
        r = super()._apply(fn, *a, **k)
        self.invalidate_weights()
        self.tensors_moved()
        return r

    # ---- pickling / deepcopy (reference train.py:485 `deepcopy(model).half()`, utils/torch_utils.py:282 ModelEMA, torch.save of the
    # whole module): the compiled plans hold device handles and are rebuilt lazily, they never travel with the module ----
    def __getstate__(self):
        d = dict(self.__dict__)
        d["_engine"] = None
        return d

    def __setstate__(self, state):
        super().__setstate__(state)
        object.__setattr__(self, "_engine", None)

    def engine(self):
        if getattr(self, "_engine", None) is None:
            from ..engine import Engine
            object.__setattr__(self, "_engine", Engine(self))
        return self._engine

    def forward(self, x, augment=False, profile=False, seg_argmax=False):
        """eval: `[(z, [x0,x1,x2]), seg]` like reference models/yolo.py:225,316.  `seg_argmax=True` additionally returns the
        fused upsample+argmax class map (B,H,W) int64 as a third element and skips materialising logits."""
        if augment:
            raise NotImplementedError("TTA (augment=True) is broken in the reference fork itself (SURVEY.md section 2 #18)")
        if self.training:
            # train mode: `[[x0,x1,x2], seg]` with batch-statistics BatchNorm and a hand-written backward behind torch.autograd
            # (reference models/yolo.py:225,316; train.py:363-392).  All four heads; BiSe returns seg = [out, aux16, aux32] (models/yolo.py:86).
            from ..engine import train_forward
            return train_forward(self, x)
        if profile:
            # reference models/yolo.py:300-309 prints ms per top-level layer; here: device time of every op of the plan (CUDA events around
            # each op, eager launches), summed per yaml layer
            eng = self.engine()
            out = eng.forward(x, seg_argmax=seg_argmax, profile=True)
            per_layer = {}
            for o, ms in zip(eng.last_plan.pb.ops, eng.last_profile):
                per_layer[o.tag] = per_layer.get(o.tag, 0.0) + ms
            for tag, ms in per_layer.items():
                print(f"{ms:10.3f} ms  {tag}")
            print(f"{sum(per_layer.values()):10.3f} ms  total (device time, {len(eng.last_profile)} kernels)")
            return out
        return self.engine().forward(x, seg_argmax=seg_argmax)
