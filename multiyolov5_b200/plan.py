"""Host-side planner: lowers the module tree built by models.yolo.parse_model to the flat op list that
libmyolo_sm90a.so replays (include/myolo.h `myolo_op`), i.e. the compiled form of Model.forward_once
(reference models/yolo.py:293-316).

Design points
  * activations are NHWC fp16; every tensor is a *view* (buffer, channel offset, channels).  torch.cat never runs:
    producers write straight into channel slices of the consumer's concat buffer (C3, SPP, yaml Concat layers, PSP / RFB2 /
    PyramidPooling / FFM concatenations).
  * buffers are liveness-packed into one workspace (first-fit over [first-def, last-use] intervals).
  * aux[] conventions per op kind are documented next to each emit_* helper.
"""
import math
import os
import struct
from dataclasses import dataclass, field
from typing import Dict, List, Optional, Sequence

import torch
import torch.nn as nn

from . import _lib
from ._lib import (ACT_NONE, ACT_SIGMOID, ACT_SILU, F16, F32, OP_ADD, OP_BILINEAR, OP_BROADCAST, OP_CHANNEL_SCALE, OP_CONV,
                   OP_ACT, OP_BN_ACT, OP_CHANNEL_SCALE_OOP, OP_DROPOUT, OP_DETECT_DECODE, OP_INPUT_FOCUS, OP_REGION_COMBINE, OP_REGION_SUM, OP_SEG_UPSAMPLE, OP_SPP_POOL,
                   OP_UPSAMPLE_NEAREST)
from .models import common as cm


@dataclass
class Buf:
    id: int
    h: int
    w: int
    c: int
    dtype: int = F16
    first: int = -1
    last: int = -1
    offset: int = 0
    alias_of: Optional["Buf"] = None    # same memory seen with another (w, c) factorisation of the pixel row (pixel-pair views)

    def nbytes(self, B):
        return B * self.h * self.w * self.c * (2 if self.dtype == F16 else 4)


@dataclass
class V:
    """channel slice of a buffer"""
    buf: Buf
    c_off: int
    c: int

    @property
    def h(self):
        return self.buf.h

    @property
    def w(self):
        return self.buf.w

    def sub(self, off, c):
        assert off + c <= self.c
        return V(self.buf, self.c_off + off, c)


@dataclass
class WeightSlot:
    conv: nn.Conv2d
    bn: Optional[nn.BatchNorm2d]
    name: str = ""


@dataclass
class OpRec:
    kind: int
    in_: Optional[V] = None
    in2: Optional[V] = None
    out: Optional[V] = None
    k: int = 1
    stride: int = 1
    dil: int = 1
    act: int = ACT_NONE
    flags: int = 0
    slot: int = -1
    aux: List[int] = field(default_factory=lambda: [0] * 8)
    faux: List[float] = field(default_factory=lambda: [0.0] * 4)
    tag: str = ""


class _CatConv:
    """two convolutions of the same input as one: duck-types the nn.Conv2d attributes the planner / weight upload read"""

    def __init__(self, a: nn.Conv2d, b: nn.Conv2d):
        assert (a.kernel_size, a.stride, a.dilation, a.padding, a.groups, a.in_channels) == \
               (b.kernel_size, b.stride, b.dilation, b.padding, b.groups, b.in_channels) and a.bias is None and b.bias is None
        self.a, self.b = a, b
        self.kernel_size, self.stride, self.dilation, self.padding, self.groups = a.kernel_size, a.stride, a.dilation, a.padding, a.groups
        self.in_channels, self.out_channels, self.bias = a.in_channels, a.out_channels + b.out_channels, None

    @property
    def weight(self):
        return torch.cat([self.a.weight.detach(), self.b.weight.detach()], 0)


class _PairedConv:
    """A 3x3 stride-1 conv on C_in (<= 16, zero padded to 16) channels restated on PIXEL PAIRS: the NHWC input (H, W, 16) is the same memory as
    (H, W/2, 32) and the output (H, W, Co) the same as (H, W/2, 2 Co).  Output pair j = pixels (2j, 2j+1) needs input pixels 2j-1 .. 2j+2 =
    pairs j-1, j, j+1, so the restated conv is again 3x3 / stride 1 / pad 1 with
        W'[p_out*Co + co, p_in*16 + ci, ky, pt] = W[co, ci, ky, kx],  kx = 2*(pt-1) + p_in - p_out + 1  (zero where kx is outside 0..2).
    Same arithmetic (the extra products are exact zeros), but the implicit-GEMM kernel sees 64-byte instead of 32-byte pixel rows, half as
    many of them, and N = 2 Co: the first layer is bound by the TMA's per-row cost (one request per 32-byte row)."""

    def __init__(self, conv: nn.Conv2d):
        assert conv.kernel_size == (3, 3) and conv.stride == (1, 1) and conv.dilation == (1, 1) and conv.padding == (1, 1)
        assert conv.groups == 1 and conv.bias is None and conv.in_channels <= 16
        self.base = conv
        self.kernel_size, self.stride, self.dilation, self.padding, self.groups = (3, 3), (1, 1), (1, 1), (1, 1), 1
        self.in_channels, self.out_channels, self.bias = 32, 2 * conv.out_channels, None

    @property
    def weight(self):
        w = self.base.weight.detach()
        co, ci = w.shape[0], w.shape[1]
        out = torch.zeros((2 * co, 32, 3, 3), dtype=w.dtype, device=w.device)
        for p_out in range(2):
            for p_in in range(2):
                for pt in range(3):
                    kx = 2 * (pt - 1) + p_in - p_out + 1
                    if 0 <= kx <= 2:
                        out[p_out * co:(p_out + 1) * co, p_in * 16:p_in * 16 + ci, :, pt] = w[:, :, :, kx]
        return out


def conv_algorithmic_flops(conv, B: int, out_view) -> float:
    """2 x MACs of the REFERENCE convolution behind a plan conv op (SURVEY.md section 8d accounting): restated convs (_PairedConv) count what
    the reference layer computes, not the zero-padded products"""
    if isinstance(conv, _PairedConv):
        b = conv.base
        return 2.0 * B * out_view.h * (out_view.w * 2) * b.out_channels * b.in_channels * 9
    return 2.0 * B * out_view.h * out_view.w * conv.out_channels * conv.in_channels * conv.kernel_size[0] * conv.kernel_size[1]


class _CatBN:
    def __init__(self, a: nn.BatchNorm2d, b: nn.BatchNorm2d):
        assert a.eps == b.eps
        self.a, self.b, self.eps, self.num_features = a, b, a.eps, a.num_features + b.num_features

    def _cat(self, name):
        return torch.cat([getattr(self.a, name).detach(), getattr(self.b, name).detach()], 0)

    weight = property(lambda self: self._cat("weight"))
    bias = property(lambda self: self._cat("bias"))
    running_mean = property(lambda self: self._cat("running_mean"))
    running_var = property(lambda self: self._cat("running_var"))


def adaptive_bins(n_in: int, k: int):
    """AdaptiveAvgPool2d bin edges: start=floor(i*n/k), end=ceil((i+1)*n/k)  (ATen adaptive pooling index math)."""
    return [(math.floor(i * n_in / k), math.ceil((i + 1) * n_in / k)) for i in range(k)]


class PlanBuilder:
    def __init__(self, B: int, H: int, W: int, train: bool = False):
        self.B, self.H, self.W = B, H, W
        self.train = train                      # train mode: raw conv -> batch-stat BN + act ops, nothing in place, no aliasing
        # cv1 and cv2 of a C3 read the same input: ONE launch with concatenated output channels (one read of the input)
        self.fuse_c3 = os.environ.get("MYOLO_FUSE_C3", "1") == "1"
        self.bn_slots: List[nn.BatchNorm2d] = []
        self.bufs: List[Buf] = []
        self.ops: List[OpRec] = []
        self.slots: List[WeightSlot] = []
        self.extra: List[int] = []
        self.tag = ""

    # ---- bookkeeping ----
    def new_buf(self, h, w, c, dtype=F16) -> V:
        b = Buf(len(self.bufs), h, w, c, dtype)
        self.bufs.append(b)
        return V(b, 0, c)

    def _touch(self, v: Optional[V], idx: int):
        if v is None:
            return
        for b in (v.buf, v.buf.alias_of):
            if b is None:
                continue
            if b.first < 0:
                b.first = idx
            b.last = idx

    def alias_buf(self, base: Buf, h, w, c) -> V:
        """another (w, c) factorisation of the same NHWC memory"""
        assert base.alias_of is None and h * w * c == base.h * base.w * base.c and base.dtype == F16
        b = Buf(len(self.bufs), h, w, c, base.dtype, alias_of=base)
        self.bufs.append(b)
        return V(b, 0, c)

    def emit(self, rec: OpRec):
        idx = len(self.ops)
        rec.tag = rec.tag or self.tag
        for v in (rec.in_, rec.in2, rec.out):
            self._touch(v, idx)
        self.ops.append(rec)
        return rec

    def add_extra(self, ints: Sequence[int]) -> int:
        off = len(self.extra)
        self.extra.extend(int(x) for x in ints)
        return off

    def add_extra_floats(self, fl: Sequence[float]) -> int:
        return self.add_extra(struct.unpack(f"{len(fl)}i", struct.pack(f"{len(fl)}f", *fl)))

    # ---- primitive emitters ----
    def conv(self, x: V, conv: nn.Conv2d, bn: Optional[nn.BatchNorm2d], act: int, dst: Optional[V] = None,
             residual: Optional[V] = None, out_dtype=F16, name="") -> V:
        """OP_CONV. in2 = residual.  Geometry from the nn.Conv2d (square kernels, symmetric stride/dilation only)."""
        k, s, d = conv.kernel_size[0], conv.stride[0], conv.dilation[0]
        assert conv.kernel_size[0] == conv.kernel_size[1] and conv.groups == 1
        assert conv.padding[0] == d * (k // 2), "only 'same'-style padding is on the path"
        ho = (x.h + 2 * d * (k // 2) - d * (k - 1) - 1) // s + 1
        wo = (x.w + 2 * d * (k // 2) - d * (k - 1) - 1) // s + 1
        co = conv.out_channels
        if dst is None:
            if out_dtype == F32:   # fp32 NHWC head outputs are padded to a multiple of 16 channels (full-row stores)
                dst = self.new_buf(ho, wo, (co + 15) // 16 * 16, F32)
            else:
                dst = self.new_buf(ho, wo, co, F16)
        assert dst.h == ho and dst.w == wo, (dst.h, dst.w, ho, wo)
        assert x.c == (conv.in_channels + 15) // 16 * 16, f"{name}: input view {x.c}ch vs conv {conv.in_channels}ch"
        slot = len(self.slots)
        self.slots.append(WeightSlot(conv, bn, name))
        self.emit(OpRec(OP_CONV, x, residual, dst, k, s, d, act, 0, slot))
        return dst

    def bn_act(self, u: V, bn: nn.BatchNorm2d, act: int, dst: Optional[V], residual: Optional[V]) -> V:
        """OP_BN_ACT (train mode): y = act(BN_batchstats(u)) (+ residual); aux[0] = bn slot."""
        dst = dst or self.new_buf(u.h, u.w, u.c)
        rec = OpRec(OP_BN_ACT, u, residual, dst, act=act)
        rec.aux[0] = len(self.bn_slots)
        self.bn_slots.append(bn)
        self.emit(rec)
        return dst

    def Conv(self, m: cm.Conv, x: V, dst=None, residual=None) -> V:
        act = ACT_SILU if isinstance(m.act, nn.SiLU) else ACT_NONE
        assert isinstance(m.act, (nn.SiLU, nn.Identity)), "only SiLU / identity activations are on the path"
        if self.train:
            u = self.conv(x, m.conv, None, ACT_NONE)
            return self.bn_act(u, m.bn, act, dst, residual)
        return self.conv(x, m.conv, m.bn, act, dst, residual)

    def dilated(self, seq: nn.Sequential, x: V, dst=None) -> V:
        if self.train:
            return self.bn_act(self.conv(x, seq[0], None, ACT_NONE), seq[1], ACT_SILU, dst, None)
        return self.conv(x, seq[0], seq[1], ACT_SILU, dst)

    def bilinear(self, x: V, h, w, dst: Optional[V] = None) -> V:
        dst = dst or self.new_buf(h, w, x.c)
        assert dst.h == h and dst.w == w and dst.c == x.c
        self.emit(OpRec(OP_BILINEAR, x, None, dst))
        return dst

    def nearest2x(self, x: V, dst: Optional[V] = None) -> V:
        dst = dst or self.new_buf(2 * x.h, 2 * x.w, x.c)
        self.emit(OpRec(OP_UPSAMPLE_NEAREST, x, None, dst))
        return dst

    def pool_pyramid(self, x: V, ks: Sequence[int], out_dtype=F16) -> List[V]:
        """AdaptiveAvgPool2d(k) for each k via one atom pass + one combine per level.
        REGION_SUM aux = [ybounds_off, ny, xbounds_off, nx];  REGION_COMBINE aux = [bins_off, nbins, atoms_nx]."""
        ys = sorted({e for k in ks for be in adaptive_bins(x.h, k) for e in be})
        xs = sorted({e for k in ks for be in adaptive_bins(x.w, k) for e in be})
        if len(ys) == 2 and x.h >= 16:      # a single huge bin (global pool): split into 16 x 4 tiles for parallelism (one CTA per atom)
            ys = sorted(set(list(range(0, x.h, max(1, x.h // 16))) + [x.h]))
            if len(xs) == 2 and x.w >= 32:
                xs = sorted(set(list(range(0, x.w, max(1, x.w // 4))) + [x.w]))
        ny, nx = len(ys) - 1, len(xs) - 1
        atoms = self.new_buf(ny, nx, x.c, F32)
        rec = OpRec(OP_REGION_SUM, x, None, atoms)
        rec.aux[0], rec.aux[1], rec.aux[2], rec.aux[3] = self.add_extra(ys), ny, self.add_extra(xs), nx
        self.emit(rec)
        outs = []
        for k in ks:
            by, bx = adaptive_bins(x.h, k), adaptive_bins(x.w, k)
            table = []
            for (y0, y1) in by:
                for (x0, x1) in bx:
                    table += [ys.index(y0), ys.index(y1), xs.index(x0), xs.index(x1), (y1 - y0) * (x1 - x0)]
            o = self.new_buf(k, k, x.c, out_dtype)
            rec = OpRec(OP_REGION_COMBINE, atoms, None, o)
            rec.aux[0], rec.aux[1], rec.aux[2] = self.add_extra(table), k * k, nx
            self.emit(rec)
            outs.append(o)
        return outs

    # ---- reference blocks ----
    def Bottleneck(self, m: cm.Bottleneck, x: V, dst=None) -> V:
        h = self.Conv(m.cv1, x)
        return self.Conv(m.cv2, h, dst, residual=x if m.add else None)

    def C3(self, m: cm.C3, x: V, dst=None) -> V:
        c_ = m.cv1.conv.out_channels
        n = len(m.m)
        if self.fuse_c3 and not self.train and n >= 1:
            # cv1 and cv2 read the same input, so they run as ONE 1x1 conv with concatenated output channels writing [cv1_out | cv2_out];
            # the last bottleneck then overwrites the (by then dead) cv1 half with the m-chain output, which is exactly the concat cv3
            # reads.  One launch and one read of x less per C3; no kernel change (tests/test_gpu_model.py::test_c3_cv1_cv2_fusion...).
            both = self.new_buf(x.h, x.w, 2 * c_)
            self.conv(x, _CatConv(m.cv1.conv, m.cv2.conv), _CatBN(m.cv1.bn, m.cv2.bn), ACT_SILU, both, name="c3.cv1+cv2")
            y = both.sub(0, c_)
            for i, bt in enumerate(m.m):
                y = self.Bottleneck(bt, y, both.sub(0, c_) if i == n - 1 else None)
            return self.Conv(m.cv3, both, dst)
        cat = self.new_buf(x.h, x.w, 2 * c_)
        y = self.Conv(m.cv1, x, cat.sub(0, c_) if n == 0 else None)
        for i, bt in enumerate(m.m):
            y = self.Bottleneck(bt, y, cat.sub(0, c_) if i == n - 1 else None)
        self.Conv(m.cv2, x, cat.sub(c_, c_))
        return self.Conv(m.cv3, cat, dst)

    def SPP(self, m: cm.SPP, x: V, dst=None) -> V:
        assert tuple(m.k) == (5, 9, 13), "SPP kernel pyramid other than (5,9,13) is not on the path"
        c_ = m.cv1.conv.out_channels
        cat = self.new_buf(x.h, x.w, 4 * c_)
        self.Conv(m.cv1, x, cat.sub(0, c_))
        rec = OpRec(OP_SPP_POOL, cat.sub(0, c_), None, cat.sub(c_, c_))   # aux = [n_cascade, kernel]; writes 3 slices
        rec.aux[0], rec.aux[1] = 3, 5
        rec.out = cat.sub(c_, 3 * c_)
        self.emit(rec)
        return self.Conv(m.cv2, cat, dst)

    def C3SPP(self, m: cm.C3SPP, x: V, dst=None) -> V:
        c_ = m.cv1.conv.out_channels
        c_spp = m.m.cv2.conv.out_channels
        cat = self.new_buf(x.h, x.w, c_spp + c_)
        self.SPP(m.m, self.Conv(m.cv1, x), cat.sub(0, c_spp))
        self.Conv(m.cv2, x, cat.sub(c_spp, c_))
        return self.Conv(m.cv3, cat, dst)

    def Focus(self, m: cm.Focus, dst=None) -> V:
        conv = m.conv.conv
        assert conv.in_channels == 12
        s2d = self.new_buf(self.H // 2, self.W // 2, 16)
        self.emit(OpRec(OP_INPUT_FOCUS, None, None, s2d))
        if (not self.train and dst is None and conv.kernel_size == (3, 3) and conv.stride == (1, 1) and isinstance(m.conv.act, nn.SiLU)
                and (self.W // 2) % 2 == 0):
            # layer 0 on pixel pairs (_PairedConv): same memory, 64-byte rows, N = 2 Co
            out = self.new_buf(self.H // 2, self.W // 2, conv.out_channels)
            x2 = self.alias_buf(s2d.buf, self.H // 2, self.W // 4, 32)
            y2 = self.alias_buf(out.buf, self.H // 2, self.W // 4, 2 * conv.out_channels)
            self.conv(x2, _PairedConv(conv), _CatBN(m.conv.bn, m.conv.bn), ACT_SILU, y2, name="focus.conv(pixel pairs)")
            self._touch(out, len(self.ops) - 1)
            return out
        return self.Conv(m.conv, s2d, dst)

    def RFB2(self, m: cm.RFB2, x: V, dst=None) -> V:
        ip = m.branch3[0].conv.out_channels
        nb = 5 if m.has_globel else 4
        cat = self.new_buf(x.h, x.w, nb * ip)
        self.Conv(m.branch3[0], x, cat.sub(3 * ip, ip))
        x0 = self.Conv(m.branch0[1], self.Conv(m.branch0[0], x), cat.sub(0, ip))
        x1 = self.dilated(m.branch1, x0, cat.sub(ip, ip))
        x2 = self.dilated(m.branch2, x1, cat.sub(2 * ip, ip))
        if m.has_globel:
            g = self.pool_pyramid(x2, [1])[0]
            g = self.Conv(m.branch4[1], g)
            self.emit(OpRec(OP_BROADCAST, g, None, cat.sub(4 * ip, ip)))
        return self.Conv(m.ConvLinear, cat, dst)

    def ASPP(self, m: cm.ASPP, x: V, dst=None) -> V:
        assert not m.has_globel, "ASPP(has_globel=True) is not used by the shipped heads"
        hid = m.hid
        cat = self.new_buf(x.h, x.w, 4 * hid)
        self.Conv(m.branch0[0], x, cat.sub(0, hid))
        for i, br in enumerate((m.branch1, m.branch2, m.branch3)):
            self.dilated(br, x, cat.sub((i + 1) * hid, hid))
        return self.Conv(m.ConvLinear, cat, dst)

    def group(self, first: int, n: int):
        """ops[first : first+n] (same kind, emitted back to back) run as ONE launch (include/myolo.h MYOLO_OP_GROUP_*)"""
        if n < 2 or n > 4 or self.train:
            return
        kinds = {o.kind for o in self.ops[first:first + n]}
        assert len(kinds) == 1 and first + n <= len(self.ops)
        self.ops[first].flags |= _lib.OP_GROUP_HEAD
        self.ops[first].aux[7] = n
        for o in self.ops[first + 1:first + n]:
            o.flags |= _lib.OP_GROUP_MEMBER

    def PyramidPooling(self, m: cm.PyramidPooling, x_in_cat: V, cat: V) -> V:
        """x_in_cat is slice 0 of `cat` (2C channels); fills slices 1..4 and returns cat.  The four levels run level-parallel: one launch
        each for the bin averages, the four 1x1 convs on the pooled bins and the four upsamplings (12 tiny kernels -> 3)."""
        C = x_in_cat.c
        n0 = len(self.ops)
        pooled = self.pool_pyramid(x_in_cat, m.k)             # REGION_SUM + one REGION_COMBINE per level
        self.group(n0 + 1, len(pooled))
        n1 = len(self.ops)
        feats = [self.Conv(conv, p) for p, conv in zip(pooled, (m.conv1, m.conv2, m.conv3, m.conv4))]
        if not self.train and all(p.h * p.w < 128 for p in pooled):          # all four are CUDA-core convs (maps below one 128-pixel tile)
            self.group(n1, len(feats))
        n2 = len(self.ops)
        for i, f in enumerate(feats):
            self.bilinear(f, x_in_cat.h, x_in_cat.w, cat.sub(C + i * (C // 4), C // 4))
        self.group(n2, len(feats))
        return cat

    def FFM(self, m: cm.FFM, x: V, dst=None) -> V:
        feat = self.Conv(m.convblk, x, dst)
        gap = self.pool_pyramid(feat, [1], out_dtype=F32)[0]
        if self.train:   # keep pre-activations and the unscaled feature map for the backward pass
            p1 = self.conv(gap, m.channel_attention[1], None, ACT_NONE, out_dtype=F32, name="ffm.att1")
            a1 = self.new_buf(1, 1, p1.c, F32)
            self.emit(OpRec(OP_ACT, p1, None, a1, act=ACT_SILU))
            p2 = self.conv(a1, m.channel_attention[3], None, ACT_NONE, out_dtype=F32, name="ffm.att2")
            a2 = self.new_buf(1, 1, p2.c, F32)
            self.emit(OpRec(OP_ACT, p2, None, a2, act=ACT_SIGMOID))
            out = self.new_buf(feat.h, feat.w, feat.c)
            self.emit(OpRec(OP_CHANNEL_SCALE_OOP, feat, a2.sub(0, feat.c), out))
            return out
        a = self.conv(gap, m.channel_attention[1], None, ACT_SILU, out_dtype=F32, name="ffm.att1")
        a = self.conv(a, m.channel_attention[3], None, ACT_SIGMOID, out_dtype=F32, name="ffm.att2")
        self.emit(OpRec(OP_CHANNEL_SCALE, feat, a.sub(0, feat.c), None))
        return feat

    def classifier(self, conv: nn.Conv2d, x: V, n_cls: int, out_index: int = 0):
        lo = self.conv(x, conv, None, ACT_NONE, out_dtype=F32, name="seg.classifier")
        rec = OpRec(OP_SEG_UPSAMPLE, lo, None, None)   # aux = [n_cls, output index (0 main; 1, 2: BiSe aux heads in train mode)]
        rec.aux[0] = n_cls
        rec.aux[1] = out_index
        self.emit(rec)
        return lo

    # ---- seg heads ----
    def SegMaskPSP(self, m, xs: List[V]):
        ch = m.c_hid
        h, w = xs[0].h, xs[0].w
        cat3 = self.new_buf(h, w, 3 * ch)
        self.Conv(m.m8[0], xs[0], cat3.sub(0, ch))
        self.bilinear(self.Conv(m.m16[0], xs[1]), h, w, cat3.sub(ch, ch))
        self.bilinear(self.Conv(m.m32[0], xs[2]), h, w, cat3.sub(2 * ch, ch))
        ppm_cat = self.new_buf(h, w, 2 * ch)
        y = self.RFB2(m.out[0], cat3, ppm_cat.sub(0, ch))
        self.PyramidPooling(m.out[1], y, ppm_cat)
        y = self.FFM(m.out[2], ppm_cat)
        return self.classifier(m.out[3], y, m.c_out)

    def SegMaskLab(self, m, xs: List[V]):
        h, w = xs[0].h, xs[0].w
        cat = self.new_buf(h, w, 48 + 256)
        e = self.ASPP(m.encoder[1], self.Conv(m.encoder[0], xs[1]))
        self.Conv(m.detail[1], self.Conv(m.detail[0], xs[0]), cat.sub(0, 48))
        self.bilinear(e, h, w, cat.sub(48, 256))
        y = self.FFM(m.decoder[0], cat)
        y = self.Conv(m.decoder[1], y)
        return self.classifier(m.decoder[2], y, m.c_out)

    def SegMaskBiSe(self, m, xs: List[V]):
        h, w = xs[0].h, xs[0].w
        f3 = self.RFB2(m.m32[0], xs[2])
        f3 = self.bilinear(self.Conv(m.up32[0], f3), xs[1].h, xs[1].w)
        f2 = self.RFB2(m.m16[0], xs[1])
        s = self.new_buf(f2.h, f2.w, f2.c)
        self.emit(OpRec(OP_ADD, f2, f3, s))
        cat = self.new_buf(h, w, 256)
        self.Conv(m.m8[0], xs[0], cat.sub(0, 128))
        f2 = self.bilinear(self.Conv(m.up16[0], s), h, w, cat.sub(128, 128))
        y = self.FFM(m.out[0], cat)
        y = self.dropout(m.out[1], y)                  # nn.Dropout(0.1), reference models/yolo.py:65
        lo = self.classifier(m.out[2], y, m.c_out)
        if self.train:                                 # auxiliary heads, training only (reference models/yolo.py:70-79,86)
            self.classifier(m.aux16[1], self.Conv(m.aux16[0], f2), m.c_out, out_index=1)
            self.classifier(m.aux32[1], self.Conv(m.aux32[0], f3), m.c_out, out_index=2)
        return lo

    def dropout(self, m: nn.Dropout, x: V) -> V:
        """nn.Dropout: identity in eval; in train mode OP_DROPOUT (faux[0] = p, aux[0] = per-op salt of the mask hash)"""
        if not self.train or m.p <= 0:
            return x
        out = self.new_buf(x.h, x.w, x.c)
        rec = OpRec(OP_DROPOUT, x, None, out)
        rec.aux[0] = len(self.ops) + 1
        rec.faux[0] = float(m.p)
        self.emit(rec)
        return out

    def SegMaskBase(self, m, xs: List[V]):
        y = self.C3(m.m[0], xs[0])
        y = self.C3SPP(m.m[1], y)
        y = self.dropout(m.m[2], y)                    # nn.Dropout(0.1, True), reference models/yolo.py:140
        return self.classifier(m.m[3], y, m.c_out)

    # ---- Detect ----
    def Detect(self, m, xs: List[V]):
        """DETECT_DECODE aux = [level, na, no, z_row_offset, z_rows_total, anchors_off(extra, 2*na float bits)]; faux[0]=stride."""
        rows = [m.na * v.h * v.w for v in xs]
        total, off = sum(rows), 0
        for i, v in enumerate(xs):
            raw = self.conv(v, m.m[i], None, ACT_NONE, out_dtype=F32, name=f"detect.m.{i}")
            rec = OpRec(OP_DETECT_DECODE, raw, None, None)
            anchors_px = [float(a) for a in m.anchor_grid[i].view(-1).tolist()]
            rec.aux[0:6] = [i, m.na, m.no, off, total, self.add_extra_floats(anchors_px)]
            rec.faux[0] = float(m.stride[i])
            self.emit(rec)
            off += rows[i]
        return rows


# ------------------------------------------------------------------------------------------------
def _layer_meta(model):
    """static (channels, stride) per yaml layer, without running anything."""
    from .models import yolo as Y
    ch, st = [], []
    for m in model.model:
        f = m.f
        src = (len(ch) - 1 if f == -1 else f) if isinstance(f, int) else [len(ch) - 1 if j == -1 else j for j in f]
        mod = m
        if type(m) is nn.Sequential:
            raise NotImplementedError("depth-repeated nn.Sequential layers are not on the shipped *_city_seg path")
        if isinstance(mod, cm.Focus):
            c, s = mod.conv.conv.out_channels, 2
        elif isinstance(mod, cm.Conv):
            c, s = mod.conv.out_channels, st[src] * mod.conv.stride[0]
        elif isinstance(mod, cm.C3):
            c, s = mod.cv3.conv.out_channels, st[src]
        elif isinstance(mod, cm.SPP):
            c, s = mod.cv2.conv.out_channels, st[src]
        elif isinstance(mod, nn.Upsample):
            c, s = ch[src], st[src] / 2
        elif isinstance(mod, cm.Concat):
            c, s = sum(ch[j] for j in src), st[src[0]]
        else:  # seg head / Detect
            c, s = 0, 0
        ch.append(c)
        st.append(s)
    return ch, st


def infer_strides(model):
    return _layer_meta(model)[1]


def build_plan(model, B: int, H: int, W: int, noalias: bool = False, train: bool = False, seg: bool = True) -> PlanBuilder:
    """Lowers model.model (yaml layers) for a fixed input shape (train=True: batch-stat BN ops, everything kept for backward).
    seg=False (inference only): without the seg head's ops, for the scaled passes of test-time augmentation, whose seg output nobody
    reads (reference models/yolo.py:274-289 keeps the Detect output only); every other op is lowered as in the full plan."""
    from .models import yolo as Y
    assert H % 32 == 0 and W % 32 == 0, "input H, W must be multiples of the max stride 32 (reference check_img_size)"
    assert seg or not train, "a train plan keeps the seg head"
    seg_types = (Y.SegMaskPSP, Y.SegMaskLab, Y.SegMaskBiSe, Y.SegMaskBase)
    pb = PlanBuilder(B, H, W, train=train)
    noalias = noalias or train
    ch, st = _layer_meta(model)
    layers = list(model.model)
    n = len(layers)
    absf = lambda i, f: (i - 1 if f == -1 else f)  # noqa: E731
    # where does each layer's output go?  (first Concat that consumes it gets it written in place)
    cat_of: Dict[int, tuple] = {}
    cat_buf: Dict[int, V] = {}
    for j, m in enumerate(layers):
        if isinstance(m, cm.Concat):
            off = 0
            for f in m.f:
                src = absf(j, f)
                if src in cat_of:
                    raise NotImplementedError(f"layer {src} feeds two Concat layers; a copy op would be needed")
                cat_of[src] = (j, off)
                off += ch[src]

    def dst_for(i):
        if i not in cat_of:
            return None
        j, off = cat_of[i]
        if j not in cat_buf:
            s = int(st[j])
            cat_buf[j] = pb.new_buf(H // s, W // s, ch[j])
        return cat_buf[j].sub(off, ch[i])

    outs: List[Optional[V]] = [None] * n
    # execution order = yaml order, except that an inference plan lowers the Detect layer BEFORE the seg head it follows (neither reads the
    # other): the graph then ends with the seg classifier conv and the x8 seg upsample - the longest caller-output kernel, run after the
    # graph - no longer waits behind the three Detect convs
    order = list(range(n))
    if not train:
        for i in range(1, n):
            if isinstance(layers[i], Y.Detect) and isinstance(layers[i - 1], seg_types) and \
                    all(absf(i, j) < i - 1 for j in ([layers[i].f] if isinstance(layers[i].f, int) else layers[i].f)):
                order[i - 1], order[i] = i, i - 1
    if not seg:
        order = [i for i in order if not isinstance(layers[i], seg_types)]
    for i in order:
        m = layers[i]
        pb.tag = f"L{i}:{type(m).__name__}"
        f = m.f
        x = None
        if isinstance(f, int):
            x = outs[absf(i, f)] if i > 0 else None
        else:
            x = [outs[absf(i, j)] for j in f]
        dst = dst_for(i)
        if isinstance(m, cm.Focus):
            y = pb.Focus(m, dst)
        elif isinstance(m, cm.Conv):
            y = pb.Conv(m, x, dst)
        elif isinstance(m, cm.C3):
            y = pb.C3(m, x, dst)
        elif isinstance(m, cm.SPP):
            y = pb.SPP(m, x, dst)
        elif isinstance(m, nn.Upsample):
            assert m.mode == "nearest" and float(m.scale_factor) == 2.0
            y = pb.nearest2x(x, dst)
        elif isinstance(m, cm.Concat):
            y = cat_buf[i]
            for v in x:
                assert v.buf is y.buf, "concat input was not produced in place"
        elif isinstance(m, Y.SegMaskPSP):
            y = pb.SegMaskPSP(m, x)
        elif isinstance(m, Y.SegMaskLab):
            y = pb.SegMaskLab(m, x)
        elif isinstance(m, Y.SegMaskBiSe):
            y = pb.SegMaskBiSe(m, x)
        elif isinstance(m, Y.SegMaskBase):
            y = pb.SegMaskBase(m, x)
        elif isinstance(m, Y.Detect):
            pb.det_rows = pb.Detect(m, x)
            y = None
        else:
            raise NotImplementedError(f"layer {i}: {type(m).__name__} (a depth-repeated nn.Sequential of Conv is not on the shipped path)")
        outs[i] = y
        # keep saved layers alive until their last consumer: extend liveness at consumption time (done by emit/_touch)
    pb.layer_views = outs
    # the executor replays all internal ops as one CUDA graph and runs the ops that touch caller-owned tensors afterwards:
    # whatever those read must stay live until the end of the plan
    for rec in pb.ops:
        if rec.kind in (OP_DETECT_DECODE, OP_SEG_UPSAMPLE) and rec.in_ is not None:
            rec.in_.buf.last = len(pb.ops) + 1
    assign_offsets(pb, noalias=noalias)
    return pb


def assign_offsets(pb: PlanBuilder, align: int = 256, noalias: bool = False):
    """first-fit packing of [first,last] live intervals (ops run sequentially on one stream, so disjoint lifetimes may alias)."""
    placed = []  # (offset, size, first, last)
    order = sorted((b for b in pb.bufs if b.first >= 0 and b.alias_of is None), key=lambda b: (-b.nbytes(pb.B), b.first))
    total = 0
    for b in order:
        size = (b.nbytes(pb.B) + align - 1) // align * align
        busy = sorted((o, s) for (o, s, f, l) in placed if noalias or not (l < b.first or f > b.last))
        off = 0
        for (o, s) in busy:
            if off + size <= o:
                break
            off = max(off, o + s)
        b.offset = off
        placed.append((off, size, b.first, b.last))
        total = max(total, off + size)
    for b in pb.bufs:
        if b.alias_of is not None:
            b.offset = b.alias_of.offset
        elif b.first < 0:
            b.offset = 0
    pb.workspace_bytes = max(total, align)
    return pb.workspace_bytes


def to_ctypes(pb: PlanBuilder):
    ops = (_lib.Op * len(pb.ops))()
    for o, r in zip(ops, pb.ops):
        o.kind = r.kind
        for name, v in (("in_", r.in_), ("in2", r.in2), ("out", r.out)):
            cv = getattr(o, name)
            if v is None:
                cv.buf, cv.c_off, cv.c = -1, 0, 0
            else:
                cv.buf, cv.c_off, cv.c = v.buf.id, v.c_off, v.c
        o.k, o.stride, o.dil, o.act, o.flags, o.weight_slot = r.k, r.stride, r.dil, r.act, r.flags, r.slot
        for i in range(8):
            o.aux[i] = int(r.aux[i])
        for i in range(4):
            o.faux[i] = float(r.faux[i])
    bufs = (_lib.BufDesc * len(pb.bufs))()
    for d, b in zip(bufs, pb.bufs):
        d.h, d.w, d.c, d.dtype, d.offset = b.h, b.w, b.c, b.dtype, b.offset
    import ctypes as C
    extra = (C.c_int32 * max(1, len(pb.extra)))(*pb.extra)
    return ops, bufs, extra
