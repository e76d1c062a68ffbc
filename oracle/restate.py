"""TEST INFRASTRUCTURE (the oracle) — a CPU restatement of the reference's joint det+seg forward path and
post-process.  NOT product code: only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline /
`--impl reference` arm may import this module.  The product (multiyolov5_b200/) never does.

Parity status: PINNED.  The reference ships no golden vectors (SURVEY.md §4), so this restatement is
pinned by (a) oracle/make_golden.py, which runs the UNMODIFIED reference in the build container and
commits its outputs under tests/golden/, and (b) tests/test_oracle_golden.py, which checks this file
against those fixtures on every CPU test run.

Floating-point work is restated with torch fp32 CPU ops (the reference's own substrate); index work
(NMS ordering / suppression, class-id argmax) is restated in numpy so its order of operations is explicit.

Every function cites the reference file:line it follows (paths relative to the reference root).
`state_dict` keys are the reference's own (e.g. ``model.2.m.0.cv1.conv.weight``).

A `q` hook (default identity) is applied wherever the CUDA path rounds to fp16 storage, so that
`quantised=True` gives an "fp16-storage emulation" of the same graph for tight kernel-level checks.
"""
import math
from typing import Callable, Dict, List, Optional, Sequence

import numpy as np
import torch
import torch.nn.functional as F

BN_MOMENTUM = 0.03  # reference utils/torch_utils.py:151
BN_EPS = 1e-3  # reference utils/torch_utils.py:150 (initialize_weights sets eps=1e-3 on every BN instance)


def make_divisible(x, divisor):
    # reference utils/general.py:176-178
    return math.ceil(x / divisor) * divisor


def _ident(t):
    return t


def q16(t: torch.Tensor) -> torch.Tensor:
    """fp16 storage rounding used by the fp16-emulation mode."""
    return t.to(torch.float16).to(torch.float32)


class Ctx:
    def __init__(self, sd: Dict[str, torch.Tensor], quantised: bool = False, train: bool = False, half: bool = False):
        # half: the reference's CUDA configuration (detect.py:96-103,136): `model.fuse()` folds BN in fp32, `model.half()` rounds the
        # folded weights / biases to fp16, activations are fp16 tensors end to end (torch fp16 kernels, cuDNN convolutions)
        self.half = half
        self.train = train   # train mode: BatchNorm uses batch statistics (reference train.py runs model.train()); tensors keep autograd
        self.sd = sd if train else {k: v.detach().to(torch.float32) if v.is_floating_point() else v for k, v in sd.items()}
        self.quantised = quantised
        self.q: Callable = q16 if quantised else _ident
        self.taps: Dict[str, torch.Tensor] = {}  # optional named intermediates


# ---------------------------------------------------------------------------------------------
# building blocks
# ---------------------------------------------------------------------------------------------
def _bn_affine(cx: Ctx, p: str):
    # eval-mode BatchNorm as a per-channel affine; reference utils/torch_utils.py:182-202 (fuse algebra)
    g, b = cx.sd[p + ".weight"], cx.sd[p + ".bias"]
    m, v = cx.sd[p + ".running_mean"], cx.sd[p + ".running_var"]
    scale = g / torch.sqrt(v + BN_EPS)
    return scale, b - m * scale


def conv_bn_act(cx: Ctx, x, wkey: str, bnp: Optional[str], k: int, s: int = 1, d: int = 1, act: bool = True,
                bias_key: Optional[str] = None, residual=None):
    """`Conv.forward` = act(bn(conv(x)))  (reference models/common.py:42-43); pad = k//2 (autopad :22-26),
    dilated bare branches use padding=dilation (models/common.py:482,487,243-253)."""
    w = cx.sd[wkey]
    pad = d * (k // 2)
    if bnp is not None and cx.train:
        y = F.conv2d(x, w, None, s, pad, d)
        if getattr(cx, "new_running", None) is not None:
            # nn.BatchNorm2d's running-statistics update in train mode: momentum 0.03 (reference utils/torch_utils.py:150-152), batch mean and
            # UNBIASED batch variance
            with torch.no_grad():
                n = y.numel() // y.shape[1]
                bm, bv = y.mean((0, 2, 3)), y.var((0, 2, 3), unbiased=False)
                cx.new_running[bnp] = ((1 - BN_MOMENTUM) * cx.sd[bnp + ".running_mean"] + BN_MOMENTUM * bm,
                                       (1 - BN_MOMENTUM) * cx.sd[bnp + ".running_var"] + BN_MOMENTUM * bv * n / max(n - 1, 1))
        y = F.batch_norm(y, None, None, cx.sd[bnp + ".weight"], cx.sd[bnp + ".bias"], training=True, momentum=0.0, eps=BN_EPS)
        if act:
            y = y * torch.sigmoid(y)
        return y if residual is None else residual + y
    if getattr(cx, "half", False):
        if bnp is not None:
            scale, shift = _bn_affine(cx, bnp)
            y = F.conv2d(x, (w * scale.view(-1, 1, 1, 1)).half(), shift.half(), s, pad, d)
        else:
            y = F.conv2d(x, w.half(), cx.sd[bias_key].half() if bias_key is not None else None, s, pad, d)
        if act:
            y = F.silu(y)
        return y if residual is None else residual + y
    if bnp is not None:
        scale, shift = _bn_affine(cx, bnp)
        if cx.quantised:  # fold BN into fp16 weights exactly like the CUDA pack kernel
            w = q16(w * scale.view(-1, 1, 1, 1))
            y = F.conv2d(x, w, None, s, pad, d) + shift.view(1, -1, 1, 1)
        else:
            y = F.conv2d(x, w, None, s, pad, d)
            y = y * scale.view(1, -1, 1, 1) + shift.view(1, -1, 1, 1)
    else:
        if cx.quantised:
            w = q16(w)
        y = F.conv2d(x, w, None, s, pad, d)
        if bias_key is not None:
            y = y + cx.sd[bias_key].view(1, -1, 1, 1)
    if act:
        y = y * torch.sigmoid(y)  # nn.SiLU
    if residual is not None:
        y = residual + y  # Bottleneck shortcut, reference models/common.py:105
    return y


def Conv(cx, p, x, k=1, s=1, residual=None, quant_out=True):
    y = conv_bn_act(cx, x, p + ".conv.weight", p + ".bn", k, s, residual=residual)
    return cx.q(y) if quant_out else y


def bare_conv_bn_silu(cx, p, x, d):
    # nn.Sequential(Conv2d(k3, dilation d, bias False), BatchNorm2d, SiLU): reference models/common.py:481-490
    return cx.q(conv_bn_act(cx, x, p + ".0.weight", p + ".1", 3, 1, d))


def Bottleneck(cx, p, x, shortcut):
    # reference models/common.py:95-105 (c1 == c2 always holds inside C3 because e=1.0, :135)
    h = Conv(cx, p + ".cv1", x, 1)
    return Conv(cx, p + ".cv2", h, 3, residual=x if shortcut else None)


def C3(cx, p, x, n, shortcut):
    # reference models/common.py:127-139
    y = Conv(cx, p + ".cv1", x, 1)
    for i in range(n):
        y = Bottleneck(cx, f"{p}.m.{i}", y, shortcut)
    return Conv(cx, p + ".cv3", torch.cat((y, Conv(cx, p + ".cv2", x, 1)), 1), 1)


def SPP(cx, p, x, ks=(5, 9, 13)):
    # reference models/common.py:163-174
    x = Conv(cx, p + ".cv1", x, 1)
    return Conv(cx, p + ".cv2", torch.cat([x] + [F.max_pool2d(x, k, 1, k // 2) for k in ks], 1), 1)


def C3SPP(cx, p, x):
    # reference models/common.py:142-152
    return Conv(cx, p + ".cv3", torch.cat((SPP(cx, p + ".m", Conv(cx, p + ".cv1", x, 1)), Conv(cx, p + ".cv2", x, 1)), 1), 1)


def Focus(cx, p, x):
    # reference models/common.py:542-551: space-to-depth (order [::2,::2],[1::2,::2],[::2,1::2],[1::2,1::2]) then Conv k3
    x = cx.q(x)
    return Conv(cx, p + ".conv", torch.cat([x[..., ::2, ::2], x[..., 1::2, ::2], x[..., ::2, 1::2], x[..., 1::2, 1::2]], 1), 3)


def bilinear(cx, x, size=None, scale=None):
    # nn.Upsample(mode='bilinear', align_corners=True) / F.interpolate(..., align_corners=True)
    if size is None:
        size = (x.shape[2] * scale, x.shape[3] * scale)
    return F.interpolate(x, size, mode="bilinear", align_corners=True)


def RFB2(cx, p, x, d=(2, 3), has_globel=False):
    # reference models/common.py:470-511
    x3 = Conv(cx, p + ".branch3.0", x, 1)
    x0 = Conv(cx, p + ".branch0.1", Conv(cx, p + ".branch0.0", x, 1), 3)
    x1 = bare_conv_bn_silu(cx, p + ".branch1", x0, d[0])
    x2 = bare_conv_bn_silu(cx, p + ".branch2", x1, d[1])
    feats = [x0, x1, x2, x3]
    if has_globel:
        g = Conv(cx, p + ".branch4.1", cx.q(F.adaptive_avg_pool2d(x2, 1)), 1)
        feats.append(F.interpolate(g, (x.shape[2], x.shape[3]), mode="nearest"))
    return Conv(cx, p + ".ConvLinear", torch.cat(feats, 1), 1)


def ASPP(cx, p, x, d=(3, 6, 9)):
    # reference models/common.py:233-275 (has_globel=False is the only shipped use, models/yolo.py:109)
    x0 = Conv(cx, p + ".branch0.0", x, 1)
    xs = [x0] + [bare_conv_bn_silu(cx, f"{p}.branch{i + 1}", x, d[i]) for i in range(3)]
    return Conv(cx, p + ".ConvLinear", torch.cat(xs, 1), 1)


def PyramidPooling(cx, p, x, ks=(1, 2, 3, 6)):
    # reference models/common.py:514-539
    h, w = x.shape[2:]
    feats = [x]
    for i, k in enumerate(ks):
        pooled = cx.q(F.adaptive_avg_pool2d(x, k))
        feats.append(cx.q(bilinear(cx, Conv(cx, f"{p}.conv{i + 1}", pooled, 1), (h, w))))
    return torch.cat(feats, 1)


def FFM(cx, p, x, k):
    # reference models/common.py:210-230 ; x is already concatenated when is_cat
    feat = Conv(cx, p + ".convblk", x, k)
    a = F.adaptive_avg_pool2d(feat, 1)
    wa, wb = cx.sd[p + ".channel_attention.1.weight"], cx.sd[p + ".channel_attention.3.weight"]
    a = F.conv2d(a, wa.to(a.dtype))
    a = a * torch.sigmoid(a)
    a = torch.sigmoid(F.conv2d(a, wb.to(a.dtype)))
    return cx.q(feat * a + feat)


# ---------------------------------------------------------------------------------------------
# segmentation heads (return logits at input resolution, i.e. after the final x8 bilinear)
# ---------------------------------------------------------------------------------------------
def _classifier(cx, p, x, k=1, bias=True):
    return conv_bn_act(cx, x, p + ".weight", None, k, act=False, bias_key=(p + ".bias") if bias else None)


def SegMaskPSP(cx, p, xs, c_hid):
    # reference models/yolo.py:149-186
    f8 = Conv(cx, p + ".m8.0", xs[0], 1)
    f16 = cx.q(bilinear(cx, Conv(cx, p + ".m16.0", xs[1], 1), scale=2))
    f32 = cx.q(bilinear(cx, Conv(cx, p + ".m32.0", xs[2], 1), scale=4))
    y = RFB2(cx, p + ".out.0", torch.cat([f8, f16, f32], 1), d=(2, 3))
    y = PyramidPooling(cx, p + ".out.1", y)
    y = FFM(cx, p + ".out.2", y, 3)
    lo = _classifier(cx, p + ".out.3", y)
    cx.taps["seg_lowres"] = lo
    return bilinear(cx, lo, scale=8)


def SegMaskLab(cx, p, xs, c_hid, n):
    # reference models/yolo.py:93-124
    e = Conv(cx, p + ".encoder.0", xs[1], 1)
    e = ASPP(cx, p + ".encoder.1", e, d=(3, 6, 9))
    e = cx.q(bilinear(cx, e, scale=2))
    dt = Conv(cx, p + ".detail.1", Conv(cx, p + ".detail.0", xs[0], 1), 3)
    y = FFM(cx, p + ".decoder.0", torch.cat([dt, e], 1), 1)
    y = Conv(cx, p + ".decoder.1", y, 3)
    lo = _classifier(cx, p + ".decoder.2", y)
    cx.taps["seg_lowres"] = lo
    return bilinear(cx, lo, scale=8)


def SegMaskBiSe(cx, p, xs):
    # reference models/yolo.py:30-86 (eval: returns self.out(feat1); train: [out, aux16(feat2), aux32(feat3)])
    f3 = RFB2(cx, p + ".m32.0", xs[2], d=(2, 3), has_globel=True)
    f3 = cx.q(bilinear(cx, Conv(cx, p + ".up32.0", f3, 3), scale=2))
    f2 = cx.q(RFB2(cx, p + ".m16.0", xs[1], d=(2, 3)) + f3)
    f2 = cx.q(bilinear(cx, Conv(cx, p + ".up16.0", f2, 3), scale=2))
    y = FFM(cx, p + ".out.0", torch.cat([Conv(cx, p + ".m8.0", xs[0], 1), f2], 1), 3)
    if getattr(cx, "dropout_mask", None) is not None:     # out.1 = nn.Dropout(0.1), active in train mode; keep mask is an input
        y = y * cx.dropout_mask / (1.0 - 0.1)
    lo = _classifier(cx, p + ".out.2", y)
    cx.taps["seg_lowres"] = lo
    out = bilinear(cx, lo, scale=8)
    if not getattr(cx, "train", False):
        return out
    a16 = bilinear(cx, _classifier(cx, p + ".aux16.1", Conv(cx, p + ".aux16.0", f2, 3)), scale=8)      # models/yolo.py:70-74
    a32 = bilinear(cx, _classifier(cx, p + ".aux32.1", Conv(cx, p + ".aux32.0", f3, 3)), scale=16)     # models/yolo.py:75-79
    return [out, a16, a32]


def SegMaskBase(cx, p, xs, n, shortcut):
    # reference models/yolo.py:129-146
    y = C3(cx, p + ".m.0", xs[0], n, shortcut)
    y = C3SPP(cx, p + ".m.1", y)
    if getattr(cx, "dropout_mask", None) is not None:     # m.2 = nn.Dropout(0.1, True) (reference models/yolo.py:140): active in train mode;
        y = y * cx.dropout_mask / (1.0 - 0.1)             # the keep mask is an INPUT here (torch's RNG stream is not part of the parity contract)
    lo = _classifier(cx, p + ".m.3", y, k=3, bias=False)
    cx.taps["seg_lowres"] = lo
    return bilinear(cx, lo, scale=8)


# ---------------------------------------------------------------------------------------------
# Detect
# ---------------------------------------------------------------------------------------------
def Detect(cx, p, xs, nc, anchors_px: Sequence[Sequence[float]], strides: Sequence[float]):
    """reference models/yolo.py:206-225 (eval branch).  `anchors_px` are the yaml anchors in pixels
    (== anchor_grid buffer); returns (z (B,sumA,no), [x_i (B,na,ny,nx,no)])."""
    no = nc + 5
    z, raw = [], []
    for i, x in enumerate(xs):
        y = conv_bn_act(cx, x, f"{p}.m.{i}.weight", None, 1, act=False, bias_key=f"{p}.m.{i}.bias")
        bs, _, ny, nx = y.shape
        na = y.shape[1] // no
        y = y.view(bs, na, no, ny, nx).permute(0, 1, 3, 4, 2).contiguous()
        raw.append(y)
        s = y.sigmoid()
        yv, xv = torch.meshgrid([torch.arange(ny, device=y.device), torch.arange(nx, device=y.device)], indexing="ij")
        grid = torch.stack((xv, yv), 2).view(1, 1, ny, nx, 2).float()          # `_make_grid` result: fp32 even under model.half()
        ag = torch.tensor(anchors_px[i], dtype=torch.float32, device=y.device).view(1, na, 1, 1, 2).to(y.dtype)   # buffer: follows .half()
        s[..., 0:2] = (s[..., 0:2] * 2.0 - 0.5 + grid) * strides[i]
        s[..., 2:4] = (s[..., 2:4] * 2) ** 2 * ag
        z.append(s.view(bs, -1, no))
    return torch.cat(z, 1), raw


# ---------------------------------------------------------------------------------------------
# whole model
# ---------------------------------------------------------------------------------------------
def parse_cfg(cfg: dict):
    """Channel / depth bookkeeping of reference models/yolo.py:373-429 (parse_model), restated for the
    module kinds the shipped *_city_seg.yaml files use."""
    gd, gw = cfg["depth_multiple"], cfg["width_multiple"]
    nc, nseg = cfg["nc"], cfg["n_segcls"]
    anchors = cfg["anchors"]
    na = len(anchors[0]) // 2
    no = na * (nc + 5)
    ch = [cfg.get("ch", 3)]
    layers = []
    for i, (f, n, m, args) in enumerate(cfg["backbone"] + cfg["head"]):
        args = [nseg if a == "n_segcls" else nc if a == "nc" else anchors if a == "anchors" else
                (None if a == "None" else (False if a == "False" else a)) for a in args]
        n = max(round(n * gd), 1) if n > 1 else n
        spec = {"i": i, "f": f, "type": m}
        if m in ("Conv", "Focus", "SPP", "C3"):
            c1, c2 = ch[f], args[0]
            if c2 != no:
                c2 = make_divisible(c2 * gw, 8)
            spec.update(c1=c1, c2=c2)
            if m == "Conv":
                spec.update(k=args[1] if len(args) > 1 else 1, s=args[2] if len(args) > 2 else 1)
            elif m == "Focus":
                spec.update(k=args[1] if len(args) > 1 else 1)
            elif m == "SPP":
                spec.update(ks=tuple(args[1]))
            else:
                spec.update(n=n, shortcut=args[1] if len(args) > 1 else True)
        elif m == "nn.Upsample":
            c2 = ch[f]
            spec.update(scale=args[1], mode=args[2])
        elif m == "Concat":
            c2 = sum(ch[x] for x in f)
        elif m == "Detect":
            c2 = None
            spec.update(nc=nc, anchors=anchors, ch=[ch[x] for x in f])
        elif m.startswith("SegMask"):
            n_ = max(round(args[1] * gd), 1) if args[1] > 1 else args[1]
            c2 = ch[f[0]] if False else None
            spec.update(n_segcls=args[0], n=n_, c_hid=make_divisible(args[2] * gw, 8), shortcut=args[3],
                        ch=[ch[x] for x in f])
        else:
            raise NotImplementedError(m)
        layers.append(spec)
        if i == 0:
            ch = []
        ch.append(c2)
    return layers


def model_forward(cfg: dict, sd: Dict[str, torch.Tensor], x: torch.Tensor, quantised: bool = False,
                  keep: Sequence[int] = (), half: bool = False):
    """`Model.forward_once` (reference models/yolo.py:293-316) in eval mode.
    Returns dict(z, raw=[x0,x1,x2], seg, seg_lowres, layers={i: tensor}).
    half=True (CUDA tensors): the same graph the way the reference runs it on a GPU - BN folded in fp32, weights and activations fp16,
    torch/cuDNN kernels (detect.py:96-103) - the precision yardstick of the GPU parity tests and the `reference-gpu` bench arm."""
    cx = Ctx(sd, quantised, half=half)
    layers = parse_cfg(cfg)
    ys: List[Optional[torch.Tensor]] = []
    x = x.to(torch.float16 if half else torch.float32)
    if half:
        assert x.is_cuda and not quantised, "half=True is the torch fp16 CUDA yardstick (the reference's own GPU configuration)"
    det = seg = None
    strides = []
    with torch.no_grad():
        for sp in layers:
            i, f, t = sp["i"], sp["f"], sp["type"]
            p = f"model.{i}"
            inp = x if f == -1 else (ys[f] if isinstance(f, int) else [x if j == -1 else ys[j] for j in f])
            if t == "Focus":
                x = Focus(cx, p, inp)
            elif t == "Conv":
                x = Conv(cx, p, inp, sp["k"], sp["s"])
            elif t == "C3":
                x = C3(cx, p, inp, sp["n"], sp["shortcut"])
            elif t == "SPP":
                x = SPP(cx, p, inp, sp["ks"])
            elif t == "nn.Upsample":
                x = F.interpolate(inp, scale_factor=sp["scale"], mode=sp["mode"])
            elif t == "Concat":
                x = torch.cat(inp, 1)
            elif t == "SegMaskPSP":
                x = seg = SegMaskPSP(cx, p, inp, sp["c_hid"])
            elif t == "SegMaskLab":
                x = seg = SegMaskLab(cx, p, inp, sp["c_hid"], sp["n"])
            elif t == "SegMaskBiSe":
                x = seg = SegMaskBiSe(cx, p, inp)
            elif t == "SegMaskBase":
                x = seg = SegMaskBase(cx, p, inp, sp["n"], sp["shortcut"])
            elif t == "Detect":
                H = ys[0].shape[2] * 2
                strides = [H / a.shape[2] for a in inp]
                anchors_px = [[(a[2 * j], a[2 * j + 1]) for j in range(len(a) // 2)] for a in sp["anchors"]]
                det = Detect(cx, p, inp, sp["nc"], anchors_px, strides)
                x = det
            ys.append(x)
    out = dict(z=det[0], raw=det[1], seg=seg, seg_lowres=cx.taps.get("seg_lowres"),
               layers={i: ys[i] for i in keep})
    return out


# ---------------------------------------------------------------------------------------------
# post-process: NMS (index work -> numpy, explicit op order) and seg argmax
# ---------------------------------------------------------------------------------------------
def nms_greedy(boxes: np.ndarray, scores: np.ndarray, iou_thres: float) -> np.ndarray:
    """torchvision.ops.nms (0.26.0 CPU kernel; third-party, un-vendored — call site reference
    utils/general.py:493).  Published algorithm, restated: candidates are visited in STABLE descending score
    order; j is suppressed by a kept i iff inter/(area_i+area_j-inter) > thr with every operation in fp32;
    returns kept ORIGINAL indices (int64) in visiting order.  NaN IoU (zero areas) never suppresses."""
    boxes = np.ascontiguousarray(boxes, dtype=np.float32)
    scores = np.asarray(scores, dtype=np.float32)
    n = boxes.shape[0]
    if n == 0:
        return np.zeros((0,), np.int64)
    order = np.argsort(-scores, kind="stable")
    x1, y1, x2, y2 = (boxes[order, k] for k in range(4))
    areas = ((x2 - x1) * (y2 - y1)).astype(np.float32)
    suppressed = np.zeros(n, bool)
    keep = []
    thr = np.float32(iou_thres)
    with np.errstate(invalid="ignore", divide="ignore"):
        for i in range(n):
            if suppressed[i]:
                continue
            keep.append(order[i])
            if i + 1 == n:
                break
            xx1 = np.maximum(x1[i], x1[i + 1:])
            yy1 = np.maximum(y1[i], y1[i + 1:])
            xx2 = np.minimum(x2[i], x2[i + 1:])
            yy2 = np.minimum(y2[i], y2[i + 1:])
            w = np.maximum(np.float32(0), (xx2 - xx1).astype(np.float32))
            h = np.maximum(np.float32(0), (yy2 - yy1).astype(np.float32))
            inter = (w * h).astype(np.float32)
            ovr = inter / ((areas[i] + areas[i + 1:]).astype(np.float32) - inter).astype(np.float32)
            suppressed[i + 1:] |= ovr > thr
    return np.asarray(keep, np.int64)


def non_max_suppression(prediction: np.ndarray, conf_thres=0.25, iou_thres=0.45, classes=None, agnostic=False,
                        multi_label=False, max_det=300, max_nms=30000, max_wh=4096) -> List[np.ndarray]:
    """reference utils/general.py:421-509, restated in numpy fp32 (labels=() and merge=False, the shipped
    settings; the 10 s wall-clock bail-out :505-507 is not restated).  Returns list of (n,6) fp32."""
    pred = np.asarray(prediction, dtype=np.float32)
    nc = pred.shape[2] - 5
    multi_label = multi_label and nc > 1
    ct = np.float32(conf_thres)
    out = []
    for x in pred:
        x = x[x[:, 4] > ct].copy()                                   # :430,446
        if not x.shape[0]:
            out.append(np.zeros((0, 6), np.float32)); continue
        x[:, 5:] = (x[:, 5:] * x[:, 4:5]).astype(np.float32)         # :462
        half_w = (x[:, 2] / np.float32(2)).astype(np.float32)
        half_h = (x[:, 3] / np.float32(2)).astype(np.float32)
        box = np.stack([x[:, 0] - half_w, x[:, 1] - half_h, x[:, 0] + half_w, x[:, 1] + half_h], 1).astype(np.float32)  # :265-272
        if multi_label:                                              # :468-470
            i, j = np.nonzero(x[:, 5:] > ct)
            x = np.concatenate([box[i], x[i, j + 5, None], j[:, None].astype(np.float32)], 1)
        else:                                                        # :471-473
            j = x[:, 5:].argmax(1)
            conf = x[np.arange(x.shape[0]), j + 5]
            x = np.concatenate([box, conf[:, None], j[:, None].astype(np.float32)], 1)[conf > ct]
        if classes is not None:                                      # :476-477
            x = x[np.isin(x[:, 5], np.asarray(classes, np.float32))]
        n = x.shape[0]
        if not n:
            out.append(np.zeros((0, 6), np.float32)); continue
        if n > max_nms:                                              # :487-488
            x = x[np.argsort(-x[:, 4], kind="stable")[:max_nms]]
        c = x[:, 5:6] * np.float32(0 if agnostic else max_wh)        # :491
        keep = nms_greedy((x[:, :4] + c).astype(np.float32), x[:, 4], iou_thres)[:max_det]  # :492-495
        out.append(x[keep].astype(np.float32))
    return out


def bilinear_align_corners_np(x: np.ndarray, out_hw) -> np.ndarray:
    """ATen upsample_bilinear2d(align_corners=True) restated in numpy fp32: scale=(in-1)/(out-1) (0 if out==1),
    src=scale*dst, i0=floor(src), i1=i0+(i0<in-1), l1=src-i0, l0=1-l1,
    out = lh0*(lw0*a + lw1*b) + lh1*(lw0*c + lw1*d).   x: (...,h,w) -> (...,H,W)."""
    x = np.asarray(x, np.float32)
    h, w = x.shape[-2:]
    H, W = out_hw

    def axis(n_in, n_out):
        scale = np.float32(n_in - 1) / np.float32(n_out - 1) if n_out > 1 else np.float32(0)
        src = (scale * np.arange(n_out, dtype=np.float32)).astype(np.float32)
        i0 = np.minimum(src.astype(np.int64), n_in - 1)
        i1 = i0 + (i0 < n_in - 1)
        l1 = (src - i0.astype(np.float32)).astype(np.float32)
        l0 = (np.float32(1) - l1).astype(np.float32)
        return i0, i1, l0, l1

    y0, y1, ly0, ly1 = axis(h, H)
    x0, x1, lx0, lx1 = axis(w, W)
    top = (lx0 * x[..., y0, :][..., x0] + lx1 * x[..., y0, :][..., x1]).astype(np.float32)
    bot = (lx0 * x[..., y1, :][..., x0] + lx1 * x[..., y1, :][..., x1]).astype(np.float32)
    return (ly0[:, None] * top + ly1[:, None] * bot).astype(np.float32)


def seg_postprocess(seg: np.ndarray, out_hw) -> np.ndarray:
    """reference detect.py:191-193: F.interpolate(seg,(H0,W0),'bilinear',align_corners=True) then
    `.max(axis=0)[1]` (first maximum wins) per image.  seg: (B,C,h,w) -> (B,H0,W0) int64."""
    up = bilinear_align_corners_np(seg, out_hw)
    return up.argmax(axis=1).astype(np.int64)


def model_forward_train(cfg: dict, sd: Dict[str, torch.Tensor], x: torch.Tensor, dropout_mask: Optional[torch.Tensor] = None,
                        new_running: Optional[dict] = None):
    """`Model.forward` in TRAIN mode (reference models/yolo.py:225,316): returns ([x0,x1,x2] raw head outputs, seg logits) with autograd
    history, so tests can compare hand-written gradients with torch.autograd on the restated graph.  `sd` tensors that should receive
    gradients must be leaf tensors with requires_grad=True.  `new_running`: optional dict that receives {bn prefix: (running_mean,
    running_var)} as nn.BatchNorm2d would leave them after this forward.  Pinned against the reference's own train-mode Model + autograd
    by tests/golden/train_*.npz (tests/test_oracle_golden.py)."""
    cx = Ctx(sd, quantised=False, train=True)
    cx.new_running = new_running
    cx.dropout_mask = dropout_mask      # (B,C,h,w) keep mask of the Base head's dropout, or None = identity
    layers = parse_cfg(cfg)
    ys: List[Optional[torch.Tensor]] = []
    x = x.to(torch.float32)
    raw = seg = None
    for sp in layers:
        i, f, t = sp["i"], sp["f"], sp["type"]
        p = f"model.{i}"
        inp = x if f == -1 else (ys[f] if isinstance(f, int) else [x if j == -1 else ys[j] for j in f])
        if t == "Focus":
            x = Focus(cx, p, inp)
        elif t == "Conv":
            x = Conv(cx, p, inp, sp["k"], sp["s"])
        elif t == "C3":
            x = C3(cx, p, inp, sp["n"], sp["shortcut"])
        elif t == "SPP":
            x = SPP(cx, p, inp, sp["ks"])
        elif t == "nn.Upsample":
            x = F.interpolate(inp, scale_factor=sp["scale"], mode=sp["mode"])
        elif t == "Concat":
            x = torch.cat(inp, 1)
        elif t == "SegMaskPSP":
            x = seg = SegMaskPSP(cx, p, inp, sp["c_hid"])
        elif t == "SegMaskLab":
            x = seg = SegMaskLab(cx, p, inp, sp["c_hid"], sp["n"])
        elif t == "SegMaskBase":
            x = seg = SegMaskBase(cx, p, inp, sp["n"], sp["shortcut"])
        elif t == "SegMaskBiSe":
            x = seg = SegMaskBiSe(cx, p, inp)          # train mode: [out, aux16, aux32]
        elif t == "Detect":
            raw = []
            no = sp["nc"] + 5
            for li, xi in enumerate(inp):
                y = conv_bn_act(cx, xi, f"{p}.m.{li}.weight", None, 1, act=False, bias_key=f"{p}.m.{li}.bias")
                bs, _, ny, nx = y.shape
                raw.append(y.view(bs, y.shape[1] // no, no, ny, nx).permute(0, 1, 3, 4, 2).contiguous())
            x = raw
        else:
            raise NotImplementedError(t)
        ys.append(x)
    return raw, seg


# ------------------------------------------------------------------------------------------------
# training losses (SURVEY.md section 8 row a13) - plain restatement, per-target Python loops; small cases only
# ------------------------------------------------------------------------------------------------
DET_LOSS_MUTANTS = ("ties", "half_le", "gt_ge", "unclamped", "first_wins", "alpha_grad", "balance", "gr", "cp_cn")


def ciou_xywh(pb: torch.Tensor, tb: torch.Tensor, eps: float = 1e-7, mutant: Optional[str] = None) -> torch.Tensor:
    """bbox_iou(box1.T, box2, x1y1x2y2=False, CIoU=True) of reference utils/general.py:343-380 for (n,4) xywh boxes.  torch.min / torch.max
    split the gradient evenly between equal arguments; mutant 'ties' gives all of it to the prediction's edge, 'alpha_grad' differentiates
    through alpha."""
    mn, mx = torch.min, torch.max
    if mutant == "ties":
        mn = lambda a, b: torch.where(a <= b, a, b)   # noqa: E731
        mx = lambda a, b: torch.where(a >= b, a, b)   # noqa: E731
    px1, px2 = pb[:, 0] - pb[:, 2] / 2, pb[:, 0] + pb[:, 2] / 2
    py1, py2 = pb[:, 1] - pb[:, 3] / 2, pb[:, 1] + pb[:, 3] / 2
    tx1, tx2 = tb[:, 0] - tb[:, 2] / 2, tb[:, 0] + tb[:, 2] / 2
    ty1, ty2 = tb[:, 1] - tb[:, 3] / 2, tb[:, 1] + tb[:, 3] / 2
    inter = (mn(px2, tx2) - mx(px1, tx1)).clamp(0) * (mn(py2, ty2) - mx(py1, ty1)).clamp(0)                                # :358-359
    w1, h1 = px2 - px1, py2 - py1 + eps                                                                                    # :362
    w2, h2 = tx2 - tx1, ty2 - ty1 + eps                                                                                    # :363
    union = w1 * h1 + w2 * h2 - inter + eps
    iou = inter / union
    cw = mx(px2, tx2) - mn(px1, tx1)
    ch = mx(py2, ty2) - mn(py1, ty1)
    c2 = cw ** 2 + ch ** 2 + eps
    rho2 = ((tx1 + tx2 - px1 - px2) ** 2 + (ty1 + ty2 - py1 - py2) ** 2) / 4
    v = (4 / math.pi ** 2) * torch.pow(torch.atan(w2 / h2) - torch.atan(w1 / h1), 2)
    with torch.set_grad_enabled(mutant == "alpha_grad" and torch.is_grad_enabled()):
        alpha = v / (v - iou + (1 + eps))                                                                                  # :378-379
    return iou - (rho2 / c2 + v * alpha)


def _near(v, mutant: Optional[str] = None) -> bool:
    """the neighbouring cell on this side is the nearer one: v % 1 < 0.5 and v > 1 (reference utils/loss.py:193-194); mutants 'half_le' and
    'gt_ge' make either comparison inclusive"""
    half = v % 1.0 <= 0.5 if mutant == "half_le" else v % 1.0 < 0.5
    inside = v >= 1.0 if mutant == "gt_ge" else v > 1.0
    return bool(half and inside)


def build_targets_loop(shapes, targets: np.ndarray, anchors: np.ndarray, anchor_t: float, mutant: Optional[str] = None):
    """ComputeLoss.build_targets (reference utils/loss.py:164-217) as explicit loops.  shapes[i] = (ny, nx); anchors (nl, na, 2) in grid
    units.  Returns per level a list of (img, anchor, gj, gi, tbox(4), cls, cand) in the reference's candidate order: the 5 offsets
    (centre, x-1, y-1, x+1, y+1) outermost, then anchors, then targets; cand = (offset * na + anchor) * nt + target numbers them in that
    order.  Mutant 'unclamped' takes the box offset relative to the unclamped cell; 'half_le' and 'gt_ge' are those of _near."""
    out = []
    nt, na = len(targets), anchors.shape[1]
    offs = np.array([[0, 0], [1, 0], [0, 1], [-1, 0], [0, -1]], np.float32) * np.float32(0.5)
    for i, (ny, nx) in enumerate(shapes):
        gain = np.array([nx, ny], np.float32)
        kept = []     # (anchor index, target index, scaled target row)
        for a in range(na):
            for ti, t in enumerate(targets):
                gxy = t[2:4] * gain
                gwh = t[4:6] * gain
                r = gwh / anchors[i, a]
                if max(np.maximum(r, np.float32(1.0) / r)) < anchor_t:                         # :185-186
                    kept.append((a, ti, int(t[0]), int(t[1]), gxy.astype(np.float32), gwh.astype(np.float32)))
        rows = []
        for k in range(5):
            for (a, ti, img, cls, gxy, gwh) in kept:
                gxi = gain - gxy
                if k == 0:
                    sel = True
                elif k == 1:
                    sel = _near(gxy[0], mutant)                                                # j  :193
                elif k == 2:
                    sel = _near(gxy[1], mutant)                                                # k
                elif k == 3:
                    sel = _near(gxi[0], mutant)                                                # l  :194
                else:
                    sel = _near(gxi[1], mutant)                                                # m
                if not sel:
                    continue
                gij = (gxy - offs[k]).astype(np.int64)                                         # .long() truncation :206
                gi = int(min(max(gij[0], 0), nx - 1))
                gj = int(min(max(gij[1], 0), ny - 1))
                # gj/gi are VIEWS of gij and clamp_ is in place (:211), so the box offset (:212) is relative to the CLAMPED cell
                ci = gij if mutant == "unclamped" else np.array([gi, gj])
                tb = np.concatenate([gxy - ci.astype(np.float32), gwh]).astype(np.float32)
                rows.append((img, a, gj, gi, tb, cls, (k * na + a) * nt + ti))
        out.append(rows)
    return out


def bce_logits(x: torch.Tensor, t: torch.Tensor) -> torch.Tensor:
    """nn.BCEWithLogitsLoss(pos_weight=1) elementwise, ATen's formula.  Its autograd gradient is sigmoid(x) - t everywhere, as the
    loss's own backward; that of max(x, 0) - x t + log1p(exp(-|x|)) is 1 - t at x = 0, where clamp and abs meet their kinks."""
    return (1 - t) * x - F.logsigmoid(x)


def compute_det_loss(p: List[torch.Tensor], targets: np.ndarray, anchors: np.ndarray, hyp: dict, nc: int, gr: float = 1.0,
                     assignment: bool = False, mutant: Optional[str] = None):
    """ComputeLoss.__call__ (reference utils/loss.py:115-162), fl_gamma = 0, label smoothing from hyp.  p[i]: (B, na, ny, nx, 5+nc),
    any number of levels.  The decisions are the reference's float32 ones (build_targets_loop); the arithmetic is in the dtype of p, so
    float64 p makes this the fp64 yardstick of the fused loss.  Returns (loss * batch, items[lbox, lobj, lcls, loss]) and, with
    assignment=True, per level (number of valid candidates, (B, na, ny, nx) int64 array of the last valid candidate of every cell or -1,
    the objectness targets).
    `mutant` (one of DET_LOSS_MUTANTS) makes it deliberately wrong in one place, for tests that show their limits catch such errors:
    'first_wins' lets the first candidate of a cell set its objectness target, 'balance' takes the other branch of the per-level
    balance lookup, 'gr' ignores gr, 'cp_cn' swaps the smoothed class targets; the others are those of ciou_xywh and build_targets_loop."""
    eps_ls = hyp.get("label_smoothing", 0.0)
    cp, cn = 1.0 - 0.5 * eps_ls, 0.5 * eps_ls
    if mutant == "cp_cn":
        cp, cn = cn, cp
    if mutant == "gr":
        gr = 1.0
    nl = len(p)
    balance = {3: [4.0, 1.0, 0.4]}.get(nl, [4.0, 1.0, 0.25, 0.06, 0.02])                                      # :104
    if mutant == "balance":
        balance = [4.0, 1.0, 0.25, 0.06, 0.02] if nl == 3 else [4.0, 1.0, 0.4]
    shapes = [(pi.shape[2], pi.shape[3]) for pi in p]
    cand = build_targets_loop(shapes, targets, anchors, hyp["anchor_t"], mutant)
    dt = p[0].dtype
    lbox = torch.zeros(1, dtype=dt); lobj = torch.zeros(1, dtype=dt); lcls = torch.zeros(1, dtype=dt)
    assigned = []
    for i, pi in enumerate(p):
        tobj = torch.zeros(pi.shape[:4], dtype=dt)
        winner = np.full(pi.shape[:4], -1, np.int64)
        rows = cand[i]
        if rows:
            b = torch.tensor([r[0] for r in rows]); a = torch.tensor([r[1] for r in rows])
            gj = torch.tensor([r[2] for r in rows]); gi = torch.tensor([r[3] for r in rows])
            tb = torch.from_numpy(np.stack([r[4] for r in rows]))
            tc = torch.tensor([r[5] for r in rows])
            ps = pi[b, a, gj, gi]
            pxy = ps[:, :2].sigmoid() * 2.0 - 0.5
            pwh = (ps[:, 2:4].sigmoid() * 2) ** 2 * torch.from_numpy(anchors[i])[a]
            iou = ciou_xywh(torch.cat((pxy, pwh), 1), tb, mutant=mutant)
            lbox = lbox + (1.0 - iou).mean()
            vals = (1.0 - gr) + gr * iou.detach().clamp(0)
            order = range(len(rows)) if mutant != "first_wins" else reversed(range(len(rows)))
            for r in order:                                # sequential writes: the last candidate of a cell wins (CPU index_put_)
                tobj[b[r], a[r], gj[r], gi[r]] = vals[r]
                winner[rows[r][0], rows[r][1], rows[r][2], rows[r][3]] = rows[r][6]
            if nc > 1:
                t = torch.full_like(ps[:, 5:], cn)
                t[torch.arange(len(rows)), tc] = cp
                lcls = lcls + bce_logits(ps[:, 5:], t).mean()
        lobj = lobj + bce_logits(pi[..., 4], tobj).mean() * balance[i]
        assigned.append((len(rows), winner, tobj))
    lbox = lbox * hyp["box"]; lobj = lobj * hyp["obj"]; lcls = lcls * hyp["cls"]
    loss = lbox + lobj + lcls
    out = loss * p[0].shape[0], torch.cat((lbox, lobj, lcls, loss)).detach()
    return (*out, assigned) if assignment else out


def seg_ce_loss(seg: torch.Tensor, mask: torch.Tensor) -> torch.Tensor:
    """SegmentationLosses.forward without aux (reference utils/loss.py:235-237) == CrossEntropyLoss(ignore_index=-1), mean over valid"""
    return F.cross_entropy(seg, mask, ignore_index=-1)


# ------------------------------------------------------------------------------------------------
# pre-process (SURVEY.md section 8f rank 1): letterbox + BGR->RGB + HWC->CHW  (reference utils/datasets.py:818-848, :185-189)
# The arithmetic lives in a third-party dependency that is not part of the reference tree: OpenCV `cv2.resize(..., INTER_LINEAR)` and
# `cv2.copyMakeBorder` (requirements.txt: opencv-python>=4.1.2; 4.13.0 installed).  Its published 8-bit algorithm (imgproc/resize.cpp)
# is restated here and pinned against cv2 itself through the fixtures (tests/golden/letterbox_cases.npz, generated by running the
# reference's own `letterbox`).
# ------------------------------------------------------------------------------------------------
def _cv_lin_coeffs(dst: int, src: int):
    """source index / fraction per destination index: fx = float((d + 0.5) * scale - 0.5) with scale = 1 / (dst / src) in double"""
    scale = 1.0 / (float(dst) / float(src))
    d = np.arange(dst, dtype=np.float64)
    f = ((d + 0.5) * scale - 0.5).astype(np.float32)
    s = np.floor(f).astype(np.int32)
    return s, (f - s.astype(np.float32)).astype(np.float32)


def cv2_resize_linear_u8(img: np.ndarray, dw: int, dh: int) -> np.ndarray:
    """cv2.resize(img, (dw, dh), interpolation=cv2.INTER_LINEAR) for uint8 HWC images, bit for bit:
    * exact 2x down-scaling is routed to the INTER_AREA fast path: (a + b + c + d + 2) >> 2;
    * otherwise 11-bit fixed point: coefficients saturate_cast<short>(w * 2048) (round half to even), horizontal pass in int32,
      vertical pass ((b0 * (S0 >> 4)) >> 16) + ((b1 * (S1 >> 4)) >> 16) + 2) >> 2; x indices clamp with fx = 0 at both borders,
      y rows clamp."""
    sh, sw = img.shape[:2]
    sx_, sy_ = 1.0 / (dw / sw), 1.0 / (dh / sh)
    eps = np.finfo(np.float64).eps
    if abs(sx_ - 2) < eps and abs(sy_ - 2) < eps:
        a = img.astype(np.int32)
        return ((a[0::2, 0::2] + a[0::2, 1::2] + a[1::2, 0::2] + a[1::2, 1::2] + 2) >> 2).astype(np.uint8)
    sx, fx = _cv_lin_coeffs(dw, sw)
    lo = sx < 0
    fx = np.where(lo, np.float32(0), fx); sx = np.where(lo, 0, sx)
    hi = sx >= sw - 1
    fx = np.where(hi, np.float32(0), fx); sx = np.where(hi, sw - 1, sx)
    a0 = np.rint((np.float32(1) - fx) * np.float32(2048)).astype(np.int32)
    a1 = np.rint(fx * np.float32(2048)).astype(np.int32)
    sx1 = np.minimum(sx + 1, sw - 1)
    sy, fy = _cv_lin_coeffs(dh, sh)
    b0 = np.rint((np.float32(1) - fy) * np.float32(2048)).astype(np.int32)
    b1 = np.rint(fy * np.float32(2048)).astype(np.int32)
    y0, y1 = np.clip(sy, 0, sh - 1), np.clip(sy + 1, 0, sh - 1)
    s = img.astype(np.int32)
    hz = s[:, sx] * a0[None, :, None] + s[:, sx1] * a1[None, :, None]
    out = (((b0[:, None, None] * (hz[y0] >> 4)) >> 16) + ((b1[:, None, None] * (hz[y1] >> 4)) >> 16) + 2) >> 2
    return out.astype(np.uint8)


def letterbox_geometry(shape, new_shape=(640, 640), auto=True, scaleFill=False, scaleup=True, stride=32):
    """the host arithmetic of reference utils/datasets.py:818-845: returns (new_unpad (w,h), ratio (w,h), (dw,dh), (top,bottom,left,right))"""
    if isinstance(new_shape, int):
        new_shape = (new_shape, new_shape)
    r = min(new_shape[0] / shape[0], new_shape[1] / shape[1])
    if not scaleup:
        r = min(r, 1.0)
    ratio = r, r
    new_unpad = int(round(shape[1] * r)), int(round(shape[0] * r))
    dw, dh = new_shape[1] - new_unpad[0], new_shape[0] - new_unpad[1]
    if auto:
        dw, dh = np.mod(dw, stride), np.mod(dh, stride)
    elif scaleFill:
        dw, dh = 0.0, 0.0
        new_unpad = (new_shape[1], new_shape[0])
        ratio = new_shape[1] / shape[1], new_shape[0] / shape[0]
    dw /= 2
    dh /= 2
    top, bottom = int(round(dh - 0.1)), int(round(dh + 0.1))
    left, right = int(round(dw - 0.1)), int(round(dw + 0.1))
    return new_unpad, ratio, (dw, dh), (top, bottom, left, right)


def letterbox_np(img: np.ndarray, new_shape=(640, 640), color=(114, 114, 114), auto=True, scaleFill=False, scaleup=True, stride=32):
    """reference utils/datasets.py:818-848 `letterbox` (uint8 HWC in, padded uint8 HWC out, ratio, (dw, dh))"""
    shape = img.shape[:2]
    new_unpad, ratio, (dw, dh), (top, bottom, left, right) = letterbox_geometry(shape, new_shape, auto, scaleFill, scaleup, stride)
    if shape[::-1] != new_unpad:
        img = cv2_resize_linear_u8(img, new_unpad[0], new_unpad[1])
    out = np.empty((img.shape[0] + top + bottom, img.shape[1] + left + right, 3), np.uint8)
    out[...] = np.array(color, np.uint8)
    out[top:top + img.shape[0], left:left + img.shape[1]] = img
    return out, ratio, (dw, dh)


def preprocess_np(img0: np.ndarray, img_size=640, stride=32) -> np.ndarray:
    """LoadImages.__next__ (reference utils/datasets.py:185-189): letterbox, BGR->RGB, HWC->CHW; uint8 (3,H,W)"""
    img = letterbox_np(img0, img_size, stride=stride)[0]
    return np.ascontiguousarray(img[:, :, ::-1].transpose(2, 0, 1))


# ------------------------------------------------------------------------------------------------
# seg output consumers (SURVEY.md section 8f rank 2)
# ------------------------------------------------------------------------------------------------
def label2image_np(pred: np.ndarray, colormap: np.ndarray) -> np.ndarray:
    """detect.py:69-72 (also trainid2id :74-77): palette look-up, (H,W) class ids -> (H,W,ch) uint8"""
    return np.asarray(colormap, np.uint8)[pred.astype(np.int32), :]


def add_weighted_u8(a: np.ndarray, alpha: float, b: np.ndarray, beta: float) -> np.ndarray:
    """cv2.addWeighted(a, alpha, b, beta, 0) for uint8 (detect.py:194): fp32 products and sum, round half to even, saturate"""
    r = a.astype(np.float32) * np.float32(alpha) + b.astype(np.float32) * np.float32(beta)
    return np.clip(np.rint(r), 0, 255).astype(np.uint8)


def seg_metrics_np(output: np.ndarray, target: np.ndarray, nclass: int):
    """batch_pix_accuracy + batch_intersection_union (reference utils/metrics.py:234-275) on (B,C,H,W) logits and (B,H,W) labels with
    -1 = ignore: returns (pixel_correct, pixel_labeled, area_inter[nclass], area_union[nclass])"""
    predict = output.argmax(1).astype(np.int64) + 1          # torch.max(output, 1): first maximum wins, like numpy
    tgt = target.astype(np.int64) + 1
    labeled = int((tgt > 0).sum())
    correct = int(((predict == tgt) * (tgt > 0)).sum())
    predict = predict * (tgt > 0)
    inter = predict * (predict == tgt)
    area_inter, _ = np.histogram(inter, bins=nclass, range=(1, nclass))
    area_pred, _ = np.histogram(predict, bins=nclass, range=(1, nclass))
    area_lab, _ = np.histogram(tgt, bins=nclass, range=(1, nclass))
    return correct, labeled, area_inter.astype(np.int64), (area_pred + area_lab - area_inter).astype(np.int64)
