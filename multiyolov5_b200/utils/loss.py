"""Training losses behind the reference's surface: `ComputeLoss(model)(p, targets)` (reference utils/loss.py:89-217),
`SegmentationLosses` (:221-262), `SegFocalLoss` (:279-297) and `OhemCELoss` (:303-328).  They consume the train-mode outputs of `Model.forward` ([x_i (B,na,ny,nx,5+nc)] and seg logits)
and, through torch.autograd, seed the hand-written backward of the network (engine._TrainFunction).

Design notes (not a transcription of the reference):
  * target assignment is computed for the FULL candidate grid (5 offsets x na anchors x nt targets) with a validity mask instead of
    boolean-filtered tensors, so no tensor shape depends on device data: no host synchronisation, CUDA-graph friendly;
  * the objectness target scatter resolves duplicate cells deterministically (the LAST candidate in the reference's candidate order
    wins - what the reference's CPU `index_put_` does; on CUDA the reference is nondeterministic there);
  * the box offset is relative to the CLAMPED cell, as in the reference (its `gj.clamp_` acts in place on a view of `gij`,
    utils/loss.py:211-212).
Parity: tests/ (test_det_loss_product_matches_reference) against fixtures generated from the unmodified reference.
"""
import math

import torch
import torch.nn as nn
import torch.nn.functional as F


def smooth_BCE(eps=0.1):
    """positive / negative BCE targets under label smoothing (reference utils/loss.py:11-13)"""
    return 1.0 - 0.5 * eps, 0.5 * eps


def _bce_with_logits(x, t, pos_weight=1.0):
    """elementwise nn.BCEWithLogitsLoss: pw*t*softplus(-x) + (1-t)*softplus(x)"""
    sp_neg = F.softplus(-x)
    if pos_weight == 1.0:
        return (1.0 - t) * x + sp_neg
    return (1.0 - t) * (x + sp_neg) + pos_weight * t * sp_neg


def _focal(loss, x, t, gamma, alpha=0.25):
    """FocalLoss wrapper of the reference (utils/loss.py:33-60): modulate the elementwise BCE"""
    pr = torch.sigmoid(x)
    p_t = t * pr + (1 - t) * (1 - pr)
    return loss * (t * alpha + (1 - t) * (1 - alpha)) * (1.0 - p_t) ** gamma


def ciou(pb, tb, eps=1e-7):
    """Complete-IoU of xywh boxes, last dim 4, broadcastable (reference utils/general.py:343-380 with x1y1x2y2=False, CIoU=True)"""
    px, py, pw, ph = pb.unbind(-1)
    tx, ty, tw, th = tb.unbind(-1)
    px1, px2, py1, py2 = px - pw / 2, px + pw / 2, py - ph / 2, py + ph / 2
    tx1, tx2, ty1, ty2 = tx - tw / 2, tx + tw / 2, ty - th / 2, ty + th / 2
    inter = (torch.min(px2, tx2) - torch.max(px1, tx1)).clamp(0) * (torch.min(py2, ty2) - torch.max(py1, ty1)).clamp(0)
    w1, h1 = px2 - px1, py2 - py1 + eps
    w2, h2 = tx2 - tx1, ty2 - ty1 + eps
    union = w1 * h1 + w2 * h2 - inter + eps
    iou = inter / union
    cw = torch.max(px2, tx2) - torch.min(px1, tx1)
    ch = torch.max(py2, ty2) - torch.min(py1, ty1)
    c2 = cw ** 2 + ch ** 2 + eps
    rho2 = ((tx1 + tx2 - px1 - px2) ** 2 + (ty1 + ty2 - py1 - py2) ** 2) / 4
    v = (4 / math.pi ** 2) * (torch.atan(w2 / h2) - torch.atan(w1 / h1)) ** 2
    with torch.no_grad():
        alpha = v / (v - iou + (1 + eps))
    return iou - (rho2 / c2 + v * alpha)


class ComputeLoss:
    """Detection loss: CIoU box + BCE objectness (target = IoU) + BCE class, per-level balance 4/1/0.4."""

    def __init__(self, model, autobalance=False):
        m = model.module if hasattr(model, "module") else model
        h = m.hyp
        det = m.model[-1]
        self.hyp, self.gr, self.autobalance = h, float(getattr(m, "gr", 1.0)), autobalance
        self.cp, self.cn = smooth_BCE(eps=h.get("label_smoothing", 0.0))
        self.gamma = float(h.get("fl_gamma", 0.0))
        self.cls_pw, self.obj_pw = float(h.get("cls_pw", 1.0)), float(h.get("obj_pw", 1.0))
        self.na, self.nc, self.nl, self.anchors = det.na, det.nc, det.nl, det.anchors
        self.balance = {3: [4.0, 1.0, 0.4]}.get(det.nl, [4.0, 1.0, 0.25, 0.06, 0.02])
        self.ssi = list(det.stride).index(16) if autobalance else 0
        self._cache = {}        # device constants (built once per grid shape: nothing is uploaded from the host inside __call__, which
                                # keeps the loss capturable in a CUDA graph)

    def _consts(self, dev, ny, nx, i):
        key = (str(dev), ny, nx, i)
        c = self._cache.get(key)
        if c is None:
            c = dict(gain=torch.tensor([nx, ny], device=dev, dtype=torch.float32),
                     off=torch.tensor([[0, 0], [1, 0], [0, 1], [-1, 0], [0, -1]], device=dev, dtype=torch.float32) * 0.5,
                     anchors=self.anchors[i].to(dev).float().clone())
            self._cache[key] = c
        return c

    def _elem(self, x, t, pw):
        loss = _bce_with_logits(x, t, pw)
        return _focal(loss, x, t, self.gamma) if self.gamma > 0 else loss

    def assign(self, shape, targets, anchors, consts=None):
        """Candidate grid for one level.  shape = (ny, nx); targets (nt,6) [img, cls, x, y, w, h] normalised; anchors (na,2) grid units.
        Returns dict of (5,na,nt)-shaped tensors: valid, b, a, gj, gi, tbox (…,4), cls."""
        ny, nx = shape
        dev = targets.device
        nt, na = targets.shape[0], anchors.shape[0]
        gain = consts["gain"] if consts else torch.tensor([nx, ny], device=dev, dtype=torch.float32)
        gxy = targets[:, 2:4] * gain
        gwh = targets[:, 4:6] * gain
        r = gwh[None] / anchors[:, None]                                        # (na,nt,2)
        match = torch.max(r, 1.0 / r).amax(2) < self.hyp["anchor_t"]            # (na,nt)
        gxi = gain - gxy
        near_lo = (gxy % 1.0 < 0.5) & (gxy > 1.0)                               # neighbour on the low side in x / y
        near_hi = (gxi % 1.0 < 0.5) & (gxi > 1.0)
        sel = torch.stack((torch.ones(nt, dtype=torch.bool, device=dev), near_lo[:, 0], near_lo[:, 1], near_hi[:, 0], near_hi[:, 1]))
        off = consts["off"] if consts else torch.tensor([[0, 0], [1, 0], [0, 1], [-1, 0], [0, -1]], device=dev, dtype=torch.float32) * 0.5
        cell = (gxy[None] - off[:, None]).long()                                # (5,nt,2) truncation toward zero
        gi = cell[..., 0].clamp(0, nx - 1)
        gj = cell[..., 1].clamp(0, ny - 1)
        txy = gxy[None] - torch.stack((gi, gj), -1).float()
        full = (5, na, nt)
        return dict(valid=(sel[:, None] & match[None]),
                    b=targets[:, 0].long()[None, None].expand(full), cls=targets[:, 1].long()[None, None].expand(full),
                    a=torch.arange(na, device=dev)[None, :, None].expand(full),
                    gj=gj[:, None].expand(full), gi=gi[:, None].expand(full),
                    tbox=torch.cat((txy, gwh[None].expand(5, nt, 2)), -1)[:, None].expand(5, na, nt, 4))

    def __call__(self, p, targets):
        dev = targets.device
        targets = targets.float()
        nt = targets.shape[0]
        lbox = torch.zeros(1, device=dev)
        lobj = torch.zeros(1, device=dev)
        lcls = torch.zeros(1, device=dev)
        for i, pi in enumerate(p):
            pi = pi.float()
            B, na, ny, nx, _ = pi.shape
            n_cells = B * na * ny * nx
            tobj = torch.zeros(n_cells, device=dev)
            if nt:
                k = self._consts(dev, ny, nx, i)
                anchors = k["anchors"]
                c = self.assign((ny, nx), targets, anchors, k)
                valid = c["valid"]
                vf = valid.float()
                n = vf.sum()
                denom = n.clamp(min=1.0)
                ps = pi[c["b"], c["a"], c["gj"], c["gi"]]                       # (5,na,nt,no)
                pxy = ps[..., :2].sigmoid() * 2.0 - 0.5
                pwh = (ps[..., 2:4].sigmoid() * 2.0) ** 2 * anchors[None, :, None]
                iou = ciou(torch.cat((pxy, pwh), -1), c["tbox"])
                lbox = lbox + ((1.0 - iou) * vf).sum() / denom
                # objectness targets; the last valid candidate of a cell wins
                flat = ((c["b"] * na + c["a"]) * ny + c["gj"]) * nx + c["gi"]
                flat = torch.where(valid, flat, torch.full_like(flat, n_cells)).reshape(-1)
                order = torch.arange(flat.numel(), device=dev)
                winner = torch.full((n_cells + 1,), -1, device=dev, dtype=torch.long).scatter_reduce(0, flat, order, "amax", include_self=True)
                vals = ((1.0 - self.gr) + self.gr * iou.detach().clamp(0)).reshape(-1)
                w = winner[:n_cells]
                tobj = torch.where(w >= 0, vals[w.clamp(min=0)], tobj)
                if self.nc > 1:
                    t = torch.full_like(ps[..., 5:], self.cn)
                    t.scatter_(-1, c["cls"][..., None], self.cp)
                    lcls = lcls + (self._elem(ps[..., 5:], t, self.cls_pw) * vf[..., None]).sum() / (denom * self.nc)
            obji = self._elem(pi[..., 4].reshape(-1), tobj, self.obj_pw).mean()
            lobj = lobj + obji * self.balance[i]
            if self.autobalance:
                self.balance[i] = self.balance[i] * 0.9999 + 0.0001 / obji.detach().item()
        if self.autobalance:
            self.balance = [x / self.balance[self.ssi] for x in self.balance]
        lbox = lbox * self.hyp["box"]
        lobj = lobj * self.hyp["obj"]
        lcls = lcls * self.hyp["cls"]
        bs = p[0].shape[0]
        loss = lbox + lobj + lcls
        return loss * bs, torch.cat((lbox, lobj, lcls, loss)).detach()


class FusedComputeLoss:
    """`ComputeLoss` forward + backward in four launches of libmyolo_sm90a (`myolo_det_loss`, csrc/detloss.cu): same arithmetic as the class
    above (which is the yardstick of tests/test_gpu_train.py::test_fused_det_loss_matches_torch_formulation and the fallback for focal loss /
    positive weights / autobalance).  `__call__(p, targets, mult, scale)` returns (grads [d loss / d p_i], loss_items); the gradient is that of
    `ComputeLoss(...)(p, targets)[0] * mult / batch * scale` with the batch factor already inside, i.e. of `loss * mult_after_bs * scale`."""

    def __init__(self, model):
        from .. import _lib
        self.ref = ComputeLoss(model)
        r = self.ref
        self.supported = (r.gamma == 0.0 and r.cls_pw == 1.0 and r.obj_pw == 1.0 and not r.autobalance and r.nl <= 3
                          and r.na <= _lib.DET_LOSS_NA_MAX)
        self._ws = None

    def __call__(self, p, targets, mult=1.0, scale=None):
        import ctypes as C
        from .. import _lib
        r = self.ref
        assert self.supported and all(t.is_cuda and t.dtype == torch.float32 and t.is_contiguous() for t in p)
        B, na, _, _, no = p[0].shape
        nl = len(p)
        ny = (C.c_int32 * nl)(*[int(t.shape[2]) for t in p])
        nx = (C.c_int32 * nl)(*[int(t.shape[3]) for t in p])
        L = _lib.lib()
        need = int(L.myolo_det_loss_workspace_bytes(B, na, nl, ny, nx))
        if self._ws is None or self._ws.numel() < need:
            self._ws = torch.empty(need, dtype=torch.uint8, device=p[0].device)
        targets = targets.float().contiguous()
        dp = [torch.empty_like(t) for t in p]
        items = torch.empty(4, dtype=torch.float32, device=p[0].device)
        vp = C.c_void_p
        # the anchors are a device buffer of the Detect layer: read them back ONCE (a .tolist() per step is a host-device synchronisation
        # in the middle of the step - it kept the host from running ahead of the GPU)
        akey = (r.anchors.data_ptr(), r.anchors._version)
        if getattr(self, "_anchors_key", None) != akey:
            self._anchors_host = [float(v) for v in r.anchors.reshape(-1).tolist()]
            self._anchors_key = akey
        anchors = (C.c_float * (nl * na * 2))(*self._anchors_host)
        balance = (C.c_float * nl)(*[float(b) for b in r.balance])
        _lib.check(L.myolo_det_loss((vp * nl)(*[_lib.ptr(t) for t in p]), (vp * nl)(*[_lib.ptr(t) for t in dp]), _lib.ptr(targets),
                                    int(targets.shape[0]), B, na, no, nl, ny, nx, anchors, balance, float(r.hyp["box"]), float(r.hyp["obj"]),
                                    float(r.hyp["cls"]), float(r.hyp["anchor_t"]), float(r.gr), float(r.cp), float(r.cn), float(mult) * B,
                                    _lib.ptr(scale), _lib.ptr(items), _lib.ptr(self._ws), need, _lib.stream_ptr()))
        return dp, items


class SegmentationLosses(nn.CrossEntropyLoss):
    """2-D cross entropy over (B,C,H,W) logits with ignore_index=-1; with aux=True the BiSe head's auxiliary outputs are weighted
    1 : 1.5*aux_weight : 0.5*aux_weight (aux_num=2) or 1 : aux_weight (aux_num=1), as reference utils/loss.py:235-249."""

    def __init__(self, se_loss=False, se_weight=0.2, nclass=-1, aux_num=2, aux=False, aux_weight=0.1, weight=None, ignore_index=-1):
        super().__init__(weight, None, ignore_index)
        if se_loss:
            raise NotImplementedError("se_loss is unused (and broken) in the reference; not provided")
        self.aux, self.aux_num, self.aux_weight, self.nclass = aux, aux_num, aux_weight, nclass

    def forward(self, *inputs):
        ce = super().forward
        if not self.aux:
            pred, target = inputs
            return ce(pred, target)
        *preds, target = inputs
        if self.aux_num == 2:
            p1, p2, p3 = preds
            return ce(p1, target) + self.aux_weight * 1.5 * ce(p2, target) + self.aux_weight / 2.0 * ce(p3, target)
        assert self.aux_num == 1
        p1, p2 = preds
        return ce(p1, target) + self.aux_weight * ce(p2, target)


def ohem_thresh_t(thresh):
    """-log(thresh) as the reference's OhemCELoss computes it: in fp32 by torch (utils/loss.py:306).  ValueError outside (0, 1]: above 1
    the threshold is negative and the reference would average the ignored pixels (CE 0) into the loss."""
    thresh = float(thresh)
    if not 0.0 < thresh <= 1.0:
        raise ValueError(f"OhemCELoss: thresh must lie in (0, 1], got {thresh}")
    return float(-torch.log(torch.tensor(thresh, dtype=torch.float32)))


class _OhemCE(torch.autograd.Function):
    """OhemCELoss.forward_once on the library (myolo_seg_ohem_loss / _backward): the selection stays on the device between the passes"""

    @staticmethod
    def forward(ctx, pred, labels, thresh_t, ignore_index):
        from .. import _lib
        B, Cc, H, W = pred.shape
        L = _lib.lib()
        need = int(L.myolo_seg_ohem_loss_workspace_bytes(B, H, W))
        ws = torch.empty(need, dtype=torch.uint8, device=pred.device)
        loss = torch.empty((), dtype=torch.float32, device=pred.device)
        _lib.check(L.myolo_seg_ohem_loss(_lib.ptr(pred), _lib.ptr(labels), B, Cc, H, W, int(ignore_index), float(thresh_t), _lib.ptr(loss),
                                         _lib.ptr(ws), need, _lib.stream_ptr()))
        ctx.save_for_backward(pred, labels)
        ctx.ws, ctx.ignore_index = ws, int(ignore_index)
        return loss

    @staticmethod
    def backward(ctx, grad_out):
        from .. import _lib
        pred, labels = ctx.saved_tensors
        B, Cc, H, W = pred.shape
        g = grad_out.float().contiguous()
        dx = torch.empty_like(pred)
        _lib.check(_lib.lib().myolo_seg_ohem_loss_backward(_lib.ptr(pred), _lib.ptr(labels), B, Cc, H, W, ctx.ignore_index, _lib.ptr(g),
                                                           _lib.ptr(dx), _lib.ptr(ctx.ws), ctx.ws.numel(), _lib.stream_ptr()))
        return dx, None, None, None


class OhemCELoss(nn.Module):
    """The reference's OhemCELoss (utils/loss.py:303-328): per pixel CE(ignore_index); the pixels with CE > -log(thresh), or the
    (valid pixels // 16) largest CEs when fewer are that hard, averaged.  With aux=True, preds is [out, aux16, aux32] (the BiSe head) and the
    loss is f(out) + aux_weight[0] * f(aux16) + aux_weight[1] * f(aux32).  The reference's train.py:285-288 suggests thresh=0.7, aux=False
    for the PSP, Lab and Base heads and thresh=0.7, aux=True, aux_weight=[0.15, 0.1] for BiSe.

    Forward and backward are library kernels over (B, C, H, W) fp32 CUDA logits and (B, H, W) int64 CUDA labels, with no host
    synchronisation: the selection (hard count, branch, the k-th largest CE by radix select) stays on the device.  Among pixels tied at the
    k-th largest CE the lowest flat indices are taken (torch.topk leaves that order unspecified).  n_min = 0 with no hard pixel gives NaN and
    zero gradients, as the reference does.  Labels outside [0, C) other than ignore_index count as ignored (torch would raise)."""

    def __init__(self, thresh=0.5, ignore_index=-1, aux=False, aux_weight=(0.15, 0.05)):
        super().__init__()
        self.thresh_t = ohem_thresh_t(thresh)
        self.ignore_index, self.aux, self.aux_weight = int(ignore_index), bool(aux), [float(w) for w in aux_weight]
        if self.aux and len(self.aux_weight) != 2:
            raise ValueError(f"OhemCELoss: aux=True takes two aux weights, got {aux_weight}")

    def forward_once(self, pred, labels):
        if not (isinstance(pred, torch.Tensor) and pred.is_cuda and pred.dtype == torch.float32 and pred.dim() == 4):
            raise ValueError("OhemCELoss: expected (B, C, H, W) float32 CUDA logits")
        if not (isinstance(labels, torch.Tensor) and labels.is_cuda and labels.dtype == torch.int64 and labels.device == pred.device
                and tuple(labels.shape) == (pred.shape[0], pred.shape[2], pred.shape[3])):
            raise ValueError(f"OhemCELoss: expected (B, H, W) = {(pred.shape[0], pred.shape[2], pred.shape[3])} int64 CUDA labels on the "
                             "logits' device")
        return _OhemCE.apply(pred.contiguous(), labels.contiguous(), self.thresh_t, self.ignore_index)

    def forward(self, preds, labels):
        if not self.aux:
            return self.forward_once(preds, labels)
        if not isinstance(preds, (list, tuple)) or len(preds) != 3:
            raise ValueError("OhemCELoss(aux=True): preds must be the list [out, aux16, aux32]")
        return (self.forward_once(preds[0], labels) + self.aux_weight[0] * self.forward_once(preds[1], labels)
                + self.aux_weight[1] * self.forward_once(preds[2], labels))


class _SegFocal(torch.autograd.Function):
    """SegFocalLoss.forward on the library (myolo_seg_focal_loss / _backward): the loss's coefficients stay on the device between the
    passes"""

    @staticmethod
    def forward(ctx, pred, labels, weight, gamma, ignore_index, reduction):
        from .. import _lib
        B, Cc, H, W = pred.shape
        L = _lib.lib()
        need = int(L.myolo_seg_focal_loss_workspace_bytes())
        ws = torch.empty(need, dtype=torch.uint8, device=pred.device)
        loss = torch.empty((), dtype=torch.float32, device=pred.device)
        red = _lib.REDUCTION_SUM if reduction == "sum" else _lib.REDUCTION_MEAN
        _lib.check(L.myolo_seg_focal_loss(_lib.ptr(pred), _lib.ptr(labels), B, Cc, H, W, int(ignore_index), _lib.ptr(weight), float(gamma),
                                          red, _lib.ptr(loss), _lib.ptr(ws), need, _lib.stream_ptr()))
        ctx.save_for_backward(pred, labels)
        ctx.ws, ctx.weight, ctx.gamma, ctx.ignore_index = ws, weight, float(gamma), int(ignore_index)
        return loss

    @staticmethod
    def backward(ctx, grad_out):
        from .. import _lib
        pred, labels = ctx.saved_tensors
        B, Cc, H, W = pred.shape
        g = grad_out.float().contiguous()
        dx = torch.empty_like(pred)
        _lib.check(_lib.lib().myolo_seg_focal_loss_backward(_lib.ptr(pred), _lib.ptr(labels), B, Cc, H, W, ctx.ignore_index,
                                                            _lib.ptr(ctx.weight), ctx.gamma, _lib.ptr(g), _lib.ptr(dx), _lib.ptr(ctx.ws),
                                                            ctx.ws.numel(), _lib.stream_ptr()))
        return dx, None, None, None, None, None


def seg_focal_loss(pred, labels, weight=None, gamma=0.0, ignore_index=-1, reduction="mean", who="SegFocalLoss"):
    """SegFocalLoss's value on the library, differentiable in pred: (B, C, H, W) fp32 CUDA logits, (B, H, W) int64 CUDA labels, weight
    None or C values.  gamma = 0 with reduction 'mean' is CrossEntropyLoss(weight=weight, ignore_index=ignore_index)."""
    if not (isinstance(pred, torch.Tensor) and pred.is_cuda and pred.dtype == torch.float32 and pred.dim() == 4):
        raise ValueError(f"{who}: expected (B, C, H, W) float32 CUDA logits")
    if not (isinstance(labels, torch.Tensor) and labels.is_cuda and labels.dtype == torch.int64 and labels.device == pred.device
            and tuple(labels.shape) == (pred.shape[0], pred.shape[2], pred.shape[3])):
        raise ValueError(f"{who}: expected (B, H, W) = {(pred.shape[0], pred.shape[2], pred.shape[3])} int64 CUDA labels on the "
                         "logits' device")
    if weight is not None:
        if weight.numel() != pred.shape[1]:
            raise ValueError(f"{who}: {weight.numel()} class weights for {pred.shape[1]} classes")
        weight = weight.to(device=pred.device, dtype=torch.float32).contiguous()
    return _SegFocal.apply(pred.contiguous(), labels.contiguous(), weight, float(gamma), int(ignore_index), reduction)


class SegFocalLoss(nn.Module):
    """The reference's SegFocalLoss (utils/loss.py:279-297): with t' = the label on valid pixels and 0 on ignored ones (the reference's
    `target * (target != ignore_index)`) and p = softmax(input, 1),
        loss = reduce((1 - p_t')^gamma) * CrossEntropyLoss(weight=alpha, ignore_index, reduction)(input, target)
    where both reductions are `reduction` (the reference overwrites the CE's): 'mean' gives the alpha-weighted mean CE times the mean of
    (1 - p_t')^gamma over every pixel, ignored ones included; 'sum' the weighted CE sum times the sum.  'none' would broadcast the
    (B, 1, H, W) focal factor against the (B, H, W) CE into (B, B, H, W) and is not provided (NotImplementedError).

    Forward and backward are library kernels over (B, C, H, W) fp32 CUDA logits of any class count and (B, H, W) int64 CUDA labels, with no
    host synchronisation.  Labels outside [0, C) other than ignore_index count as ignored (torch would raise).  With gamma < 1 a pixel whose
    p_t' rounds to 1 has an infinite (1 - p_t')^(gamma - 1): its gradient is NaN, as the reference's autograd gives.  A batch with no valid
    pixel gives a NaN loss, as the reference does."""

    def __init__(self, gamma=2, alpha=None, ignore_index=-100, reduction="mean"):
        super().__init__()
        if reduction == "none":
            raise NotImplementedError("SegFocalLoss(reduction='none'): the reference broadcasts the (B, 1, H, W) focal factor against the "
                                      "(B, H, W) cross entropy into a (B, B, H, W) loss; use 'mean' or 'sum'")
        if reduction not in ("mean", "sum"):
            raise ValueError(f"SegFocalLoss: {reduction!r} is not a valid value for reduction")
        gamma = float(gamma)
        if not (math.isfinite(gamma) and gamma >= 0.0):
            raise ValueError(f"SegFocalLoss: gamma must be finite and >= 0, got {gamma}")
        self.gamma, self.ignore_index, self.reduction = gamma, int(ignore_index), reduction
        self.register_buffer("weight", None if alpha is None else torch.as_tensor(alpha, dtype=torch.float32).reshape(-1).clone())

    def forward(self, input_, target):
        return seg_focal_loss(input_, target, self.weight, self.gamma, self.ignore_index, self.reduction)
