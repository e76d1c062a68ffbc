"""Training losses behind the reference's surface: `ComputeLoss(model)(p, targets)` (reference utils/loss.py:89-217) and
`SegmentationLosses` (:221-262).  They consume the train-mode outputs of `Model.forward` ([x_i (B,na,ny,nx,5+nc)] and seg logits)
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
        self.ref = ComputeLoss(model)
        r = self.ref
        self.supported = (r.gamma == 0.0 and r.cls_pw == 1.0 and r.obj_pw == 1.0 and not r.autobalance and r.nl <= 3 and r.na <= 3)
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
