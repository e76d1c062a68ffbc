"""Runtime glue between the nn.Module shells and libmyolo_sm90a.so: compiles one plan per input shape, uploads
(BN-folded, fp16-packed) weights, allocates caller-owned output tensors and launches the plan on the current stream."""
import os
import ctypes as C
from typing import Dict, Tuple

import torch

from . import _lib
from .plan import build_plan, to_ctypes


class CompiledPlan:
    def __init__(self, model, B, H, W, noalias=False, train=False):
        self.train = train
        self.pb = build_plan(model, B, H, W, noalias=noalias, train=train)
        self.ops, self.bufs, self.extra = to_ctypes(self.pb)
        L = _lib.lib()
        h = C.c_void_p()
        _lib.check(L.myolo_plan_create(self.ops, len(self.pb.ops), self.bufs, len(self.pb.bufs), self.extra, len(self.pb.extra),
                                       B, H, W, int(self.pb.workspace_bytes), len(self.pb.slots), C.byref(h)))
        self.handle = h
        self.B, self.H, self.W = B, H, W
        self.weights_uploaded = False
        self.weights_registered = None       # pointer signature of the tensors the library holds (myolo_plan_repack_weights)

    def __del__(self):
        try:
            if getattr(self, "handle", None):
                _lib.lib().myolo_plan_destroy(self.handle)
                self.handle = None
        except Exception:
            pass

    def _pointer_signature(self):
        sig = []
        for s in self.pb.slots:
            for t in (s.conv.weight, s.conv.bias) + ((s.bn.weight, s.bn.bias, s.bn.running_mean, s.bn.running_var) if s.bn is not None else ()):
                sig.append(0 if t is None else (t.data_ptr() if t.dtype == torch.float32 and t.is_contiguous() else -1))
        return tuple(sig)

    def upload_weights(self):
        L = _lib.lib()
        sp = _lib.stream_ptr()
        # same fp32 tensors as at the last full upload (in-place optimiser updates): every pack of the plan in one launch
        sig = self._pointer_signature()
        if self.weights_registered == sig and -1 not in sig and os.environ.get("MYOLO_REPACK", "1") != "0":
            _lib.check(L.myolo_plan_repack_weights(self.handle, sp))
            self.weights_uploaded = True
            return
        keep = []

        def f32(t):
            if t is None:
                return None
            t = t.detach()
            if t.dtype != torch.float32 or not t.is_contiguous():
                t = t.float().contiguous()
            assert t.is_cuda, "model parameters must live on the CUDA device (model.cuda())"
            keep.append(t)
            return t

        for i, s in enumerate(self.pb.slots):
            w = f32(s.conv.weight)
            bias = f32(s.conv.bias)
            if s.bn is not None:
                g, b, m, v = f32(s.bn.weight), f32(s.bn.bias), f32(s.bn.running_mean), f32(s.bn.running_var)
                eps = float(s.bn.eps)
            else:
                g = b = m = v = None
                eps = 0.0
            co, ci, k = w.shape[0], w.shape[1], w.shape[2]
            _lib.check(L.myolo_plan_set_conv_weights(self.handle, i, _lib.ptr(w), co, ci, k, _lib.ptr(g), _lib.ptr(b), _lib.ptr(m),
                                                     _lib.ptr(v), eps, _lib.ptr(bias), sp))
        self.weights_uploaded = True
        self.weights_registered = sig


class Engine:
    def __init__(self, model):
        self.model = model
        self.plans: Dict[Tuple[int, int, int], CompiledPlan] = {}
        self.weights_dirty = True
        self.last_plan = None
        self.noalias = False   # debug: give every buffer private memory so intermediate views stay readable after forward

    def plan_for(self, B, H, W) -> CompiledPlan:
        key = (B, H, W)
        if key not in self.plans:
            self.plans[key] = CompiledPlan(self.model, B, H, W, self.noalias)
        p = self.plans[key]
        ver = sum(q._version for q in self.model.parameters()) + sum(q._version for q in self.model.buffers())
        if getattr(self, "_infer_version", None) != ver:      # in-place edits of parameters / buffers bump torch's version counters
            self._infer_version = ver
            self.weights_dirty = True
        if self.weights_dirty:
            for q in self.plans.values():
                q.weights_uploaded = False
            self.weights_dirty = False
        if not p.weights_uploaded:
            p.upload_weights()
        self.last_plan = p
        return p

    def forward(self, x: torch.Tensor, seg_argmax=False, want_seg=True, want_raw=True, profile=False):
        if not x.is_cuda:
            raise _lib.MyoloError("Model.forward needs a CUDA tensor: multiyolov5_b200 has no CPU path (use the oracle for CPU numbers)")
        assert x.dim() == 4 and x.shape[1] == 3, "expected (B,3,H,W)"
        x = x.contiguous()
        B, _, H, W = x.shape
        p = self.plan_for(B, H, W)
        det = self.model.model[-1]
        seg_head = self.model.model[-2]
        rows = p.pb.det_rows
        dev = x.device
        z = torch.empty((B, sum(rows), det.no), dtype=torch.float32, device=dev)
        raws = []
        for i, v in enumerate([o.in_ for o in p.pb.ops if o.kind == _lib.OP_DETECT_DECODE]):
            raws.append(torch.empty((B, det.na, v.h, v.w, det.no), dtype=torch.float32, device=dev) if want_raw else None)
        # like the reference: fp16 in (or model.half(), detect.py:96-103) -> fp16 seg logits; otherwise fp32
        half_model = next(self.model.parameters()).dtype == torch.float16
        seg_dt = torch.float16 if (x.dtype == torch.float16 or half_model) else torch.float32
        seg = torch.empty((B, seg_head.c_out, H, W), dtype=seg_dt, device=dev) if (want_seg and not seg_argmax) else None
        amax = torch.empty((B, H, W), dtype=torch.int64, device=dev) if seg_argmax else None
        raw_ptrs = (C.c_void_p * 3)(*[_lib.ptr(r) for r in raws])
        L = _lib.lib()
        args = (p.handle, _lib.ptr(x), _lib.torch_dtype_code(x.dtype), _lib.ptr(z), raw_ptrs if want_raw else None, _lib.ptr(seg),
                _lib.torch_dtype_code(seg_dt), _lib.ptr(amax))
        if profile:
            ms = (C.c_float * len(p.pb.ops))()
            _lib.check(L.myolo_plan_profile(*args, ms, _lib.stream_ptr()))
            self.last_profile = list(ms)
        else:
            _lib.check(L.myolo_plan_forward(*args, _lib.stream_ptr()))
        out = [(z, raws), seg]
        if seg_argmax:
            out.append(amax)
        return out

    # ---- training (SURVEY.md section 8 row a13) -----------------------------------------------------------------------
    def train_plan_for(self, B, H, W, lane=0) -> CompiledPlan:
        """lane: independent train plans of the same shape (own activation / gradient workspaces) so that the two passes of a training step
        can be in flight at the same time (train.Trainer overlap_passes)"""
        key = ("train", B, H, W) if lane == 0 else ("train", B, H, W, lane)
        if key not in self.plans:
            self.plans[key] = CompiledPlan(self.model, B, H, W, train=True)
        return self.plans[key]

    def ensure_flat_grads(self):
        """every parameter's .grad is a view into ONE flat fp32 buffer (what the data-parallel all-reduce moves, reference
        train.py:243-245 DDP semantics) that the backward kernels accumulate into."""
        params = [p for p in self.model.parameters() if p.requires_grad]
        self._train_params = params
        if getattr(self, "_flat_grad", None) is not None and all(p.grad is not None and p.grad.data_ptr() == g.data_ptr()
                                                                  for p, g in zip(params, self._grad_views)):
            return self._flat_grad
        for p in params:
            assert p.dtype == torch.float32 and p.is_cuda, "training keeps fp32 master parameters on the GPU"
        # every tensor starts on a 16-byte boundary (vector loads / vector reductions in the kernels); the gaps stay zero
        self._flat_offsets, off = [], 0
        for p in params:
            self._flat_offsets.append(off)
            off += (p.numel() + 3) // 4 * 4
        n = off
        old = [p.grad for p in params]
        self._flat_grad = torch.zeros(n, dtype=torch.float32, device=params[0].device)
        self._grad_views = []
        for p, g, off in zip(params, old, self._flat_offsets):
            v = self._flat_grad[off:off + p.numel()].view_as(p)
            if g is not None:
                v.copy_(g)
            p.grad = v
            self._grad_views.append(v)
        return self._flat_grad

    def prepare_train_plan(self, p):
        """seed, fp16 weight packs and parameter / gradient pointers of a train plan for the current parameter values (idempotent; the
        Trainer calls it ahead of time on the side stream for the seg pass)"""
        L = _lib.lib()
        sp = _lib.stream_ptr()
        params = self._train_params
        if not getattr(p, "_seed_set", False):       # dropout masks follow torch's global seed (one hash stream per plan)
            _lib.check(L.myolo_plan_set_seed(p.handle, C.c_uint64(torch.initial_seed() & 0xFFFFFFFFFFFFFFFF)))
            p._seed_set = True
        # re-pack the fp16 weights only when the parameters changed (in-place torch updates bump _version; Trainer's fused optimiser
        # writes through raw pointers and sets weights_dirty)
        ver = sum(q._version for q in params)
        if self.weights_dirty:
            self._dirty_epoch = getattr(self, "_dirty_epoch", 0) + 1      # the fused optimiser wrote through raw pointers
            self.weights_dirty = False
            for q in self.plans.values():        # every plan (inference ones too) holds packed copies of the old values
                q.weights_uploaded = False
        sig_w = (ver, getattr(self, "_dirty_epoch", 0))
        if getattr(p, "_w_version", None) != sig_w:
            p.weights_uploaded = False
        if not p.weights_uploaded:
            p.upload_weights()                   # fp16, K-major, no BN folding
            p._w_version = sig_w
        sig = (self._flat_grad.data_ptr(), params[0].data_ptr(), params[-1].data_ptr(), len(params))
        if getattr(p, "_ptr_sig", None) != sig:  # (re)register parameter / gradient pointers only when they moved
            for i, s in enumerate(p.pb.slots):
                _lib.check(L.myolo_plan_set_conv_grad(p.handle, i, _lib.ptr(s.conv.weight.grad), _lib.ptr(s.conv.bias.grad if s.conv.bias is not None else None)))
            for i, bn in enumerate(p.pb.bn_slots):
                _lib.check(L.myolo_plan_set_bn(p.handle, i, bn.num_features, _lib.ptr(bn.weight), _lib.ptr(bn.bias), _lib.ptr(bn.running_mean),
                                               _lib.ptr(bn.running_var), _lib.ptr(bn.weight.grad), _lib.ptr(bn.bias.grad), float(bn.momentum), float(bn.eps)))
            p._ptr_sig = sig
            p._nbt = [bn.num_batches_tracked for bn in p.pb.bn_slots]

    def train_forward(self, x: torch.Tensor, out_raws=None, want_seg=True, lane=0):
        """out_raws: optional list of three preallocated (B,na,ny,nx,no) fp32 tensors to write the head outputs into (static buffers of a
        captured loss graph); want_seg=False skips the full-resolution logits (the det pass never reads them)."""
        assert x.is_cuda and x.dim() == 4, "expected a CUDA (B,3,H,W) tensor"
        x = x.contiguous()
        B, _, H, W = x.shape
        p = self.train_plan_for(B, H, W, lane)
        self.ensure_flat_grads()
        self.prepare_train_plan(p)
        L = _lib.lib()
        sp = _lib.stream_ptr()
        if not getattr(p, "_defer_running", False):      # a deferring plan counts its batch in apply_running
            torch._foreach_add_(p._nbt, 1)
        det, seg_head = self.model.model[-1], self.model.model[-2]
        dec = [o.in_ for o in p.pb.ops if o.kind == _lib.OP_DETECT_DECODE]
        shapes = [(B, det.na, v.h, v.w, det.no) for v in dec]
        if out_raws is not None:
            assert all(tuple(r.shape) == sh and r.dtype == torch.float32 and r.is_contiguous() for r, sh in zip(out_raws, shapes))
            raws = list(out_raws)
        else:
            raws = [torch.empty(sh, dtype=torch.float32, device=x.device) for sh in shapes]
        n_seg = sum(1 for o in p.pb.ops if o.kind == _lib.OP_SEG_UPSAMPLE)        # 3 for the BiSe head (main + two aux outputs)
        segs = [torch.empty((B, seg_head.c_out, H, W), dtype=torch.float32, device=x.device) if want_seg else None for _ in range(n_seg)]
        raw_ptrs = (C.c_void_p * 3)(*[_lib.ptr(r) for r in raws])
        seg_ptrs = (C.c_void_p * 3)(*[_lib.ptr(segs[k]) if k < n_seg else None for k in range(3)])
        _lib.check(L.myolo_plan_train_forward_multi(p.handle, _lib.ptr(x), _lib.torch_dtype_code(x.dtype), raw_ptrs, seg_ptrs, sp))
        # activations / batch statistics / dropout step of THIS forward live in the plan's single workspace: a backward is only valid
        # for the most recent train forward of the plan (the reference's order forward, backward, forward, backward - train.py:364-392)
        p.fwd_generation = getattr(p, "fwd_generation", 0) + 1
        # running_mean / running_var moved (raw pointers): every inference plan's BN-folded weights are stale now
        for q in self.plans.values():
            if not q.train:
                q.weights_uploaded = False
        self.last_plan = p
        return raws, (segs[0] if n_seg == 1 else segs), p

    def set_defer_running(self, plan, on=True):
        """a deferring train plan leaves running_mean / running_var / num_batches_tracked alone in its forward (apply_running moves them):
        lets the seg pass's forward run next to the det pass's while the statistics still move in the reference's order"""
        if getattr(plan, "_defer_running", False) != bool(on):
            _lib.check(_lib.lib().myolo_plan_set_defer_running(plan.handle, int(bool(on))))
            plan._defer_running = bool(on)

    def apply_running(self, plan):
        _lib.check(_lib.lib().myolo_plan_apply_running(plan.handle, _lib.stream_ptr()))
        torch._foreach_add_(plan._nbt, 1)

    def _check_generation(self, plan, generation):
        if generation is not None and generation != getattr(plan, "fwd_generation", 0):
            raise _lib.MyoloError("backward of a stale train-mode forward: another forward of the same (B,H,W) ran in between and overwrote the "
                                  "saved activations (one outstanding forward per shape; run forward, backward, forward, backward like "
                                  "reference train.py:364-392)")

    def train_backward(self, plan, grad_raws, grad_seg, generation=None):
        """grad_seg: one tensor / None, or a list of up to three (BiSe: main, aux16, aux32)"""
        self._check_generation(plan, generation)
        gr = [g.float().contiguous() if g is not None else None for g in grad_raws]
        gsl = list(grad_seg) if isinstance(grad_seg, (list, tuple)) else [grad_seg]
        gsl = [g.float().contiguous() if g is not None else None for g in gsl] + [None] * (3 - len(gsl))
        ptrs = (C.c_void_p * 3)(*[_lib.ptr(g) for g in gr])
        sptrs = (C.c_void_p * 3)(*[_lib.ptr(g) for g in gsl])
        _lib.check(_lib.lib().myolo_plan_backward_multi(plan.handle, ptrs, sptrs, _lib.stream_ptr()))

    def train_backward_seg_ce(self, plan, labels, factor=1.0, scale=None, ignore_index=-1):
        """fused seg loss + backward (SURVEY.md section 8f rank 3): mean CE(ignore_index) of the upsampled logits of the last train forward
        against `labels` (B,H,W) int64; gradients scaled by factor * scale (device scalar tensor).  Returns the mean CE (device scalar)."""
        assert labels.is_cuda and labels.dtype == torch.int64 and tuple(labels.shape) == (plan.B, plan.H, plan.W)
        loss = torch.empty((), dtype=torch.float32, device=labels.device)
        _lib.check(_lib.lib().myolo_plan_backward_seg_ce(plan.handle, _lib.ptr(labels.contiguous()), int(ignore_index), float(factor),
                                                         _lib.ptr(scale), _lib.ptr(loss), _lib.stream_ptr()))
        return loss

    def read_grad_view(self, v, plan=None):
        """debug: NHWC slice of the gradient workspace -> (B,C,H,W) fp32 torch tensor"""
        p = plan or self.last_plan
        out = torch.empty((p.B, v.c, v.h, v.w), dtype=torch.float32, device="cuda")
        _lib.check(_lib.lib().myolo_plan_read_grad_view(p.handle, _lib.View(v.buf.id, v.c_off, v.c), _lib.ptr(out), _lib.stream_ptr()))
        return out

    def launches(self):
        return int(_lib.lib().myolo_plan_last_launch_count(self.last_plan.handle)) if self.last_plan else 0

    def read_view(self, v, plan=None):
        """debug: NHWC slice -> (B,C,H,W) fp32 torch tensor"""
        p = plan or self.last_plan
        out = torch.empty((p.B, v.c, v.h, v.w), dtype=torch.float32, device="cuda")
        _lib.check(_lib.lib().myolo_plan_read_view(p.handle, _lib.View(v.buf.id, v.c_off, v.c), _lib.ptr(out), _lib.stream_ptr()))
        return out


class _TrainFunction(torch.autograd.Function):
    """Glue to torch.autograd: the losses (reference utils/loss.py) stay in PyTorch and seed the hand-written backward."""

    @staticmethod
    def forward(ctx, anchor, engine, x):
        ctx.set_materialize_grads(False)
        raws, seg, plan = engine.train_forward(x)
        ctx.engine, ctx.plan, ctx.generation = engine, plan, plan.fwd_generation
        segs = seg if isinstance(seg, list) else [seg]
        return (*raws, *segs)

    @staticmethod
    def backward(ctx, g0, g1, g2, *gsegs):
        ctx.engine.train_backward(ctx.plan, [g0, g1, g2], list(gsegs), generation=ctx.generation)   # parameter gradients are accumulated into the flat .grad buffer
        return None, None, None


def train_forward(model, x):
    eng = model.engine()
    if not hasattr(eng, "_anchor"):
        eng._anchor = torch.zeros((), device=x.device, requires_grad=True)
    out = _TrainFunction.apply(eng._anchor, eng, x)
    return [list(out[:3]), out[3] if len(out) == 4 else list(out[3:])]     # BiSe: seg = [out, aux16, aux32] (models/yolo.py:86)
