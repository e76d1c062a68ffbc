"""Runtime glue between the nn.Module shells and libmyolo_sm90a.so: compiles one plan per input shape, uploads
(BN-folded, fp16-packed) weights, allocates caller-owned output tensors and launches the plan on the current stream."""
import os
import ctypes as C
from typing import Dict, Tuple

import numpy as np
import torch

from . import _lib
from .plan import build_plan, to_ctypes


def shared_train_plans(model, B, shapes):
    """host train plans for batches of B images at each (H, W) of `shapes`, and the workspace capacity they need when they share one
    (the largest of their workspaces; every buffer of every plan lies inside its own plan's workspace_bytes)"""
    pbs = {(int(h), int(w)): build_plan(model, B, int(h), int(w), train=True) for h, w in shapes}
    return pbs, max([int(pb.workspace_bytes) for pb in pbs.values()], default=0)


def flat_offsets(params):
    """(offsets, total) of the parameters in the flat parameter / gradient / optimiser buffers: back to back in the given order, every
    tensor starting on a 16-byte boundary (vector loads / vector reductions in the kernels); the gaps stay zero"""
    offsets, off = [], 0
    for p in params:
        offsets.append(off)
        off += (p.numel() + 3) // 4 * 4
    return offsets, off


class TrainArena:
    """One activation workspace and one gradient workspace shared by the train plans of one lane (Engine.reserve_train_shapes).

    The plans bake the workspace address into their tensor maps and captured graphs, so the pair is allocated once, at its final size,
    before the first plan binds to it, and never moves.  Plans of one lane run one after another on one stream; `owner` is the plan whose
    forward wrote the activations last, `generation` counts the forwards (a backward is valid only for the arena's latest forward)."""

    def __init__(self, capacity, device):
        self.capacity = int(capacity)
        self.ws = torch.zeros(self.capacity, dtype=torch.uint8, device=device)
        self.gws = torch.zeros(self.capacity, dtype=torch.uint8, device=device)
        self.owner = None
        self.generation = 0

    def claim(self, plan):
        """called before `plan`'s forward, on the stream it runs on.  A plan reads some bytes of its workspace it never writes as zeros (the
        zero-padded input channels and the padded fp32 head channels, plan.py); another shape's plan may have written anything there, so
        the plan's whole workspace prefix is zeroed when the arena changes hands - the state a private workspace has after creation."""
        if self.owner is not None and self.owner is not plan:
            self.ws[:plan.pb.workspace_bytes].zero_()
        self.owner = plan
        self.generation += 1
        return self.generation


class CompiledPlan:
    def __init__(self, model, B, H, W, noalias=False, train=False, arena=None, pb=None, seg=True):
        """arena: a TrainArena the (train) plan binds to instead of allocating private workspaces; pb: its already-built host plan;
        seg=False: an inference plan without the seg head (build_plan)"""
        self.train = train
        self.pb = pb if pb is not None else build_plan(model, B, H, W, noalias=noalias, train=train, seg=seg)
        self.ops, self.bufs, self.extra = to_ctypes(self.pb)
        self.arena = arena                   # keeps the shared workspaces alive as long as the plan
        L = _lib.lib()
        h = C.c_void_p()
        args = (self.ops, len(self.pb.ops), self.bufs, len(self.pb.bufs), self.extra, len(self.pb.extra), B, H, W,
                int(self.pb.workspace_bytes), len(self.pb.slots))
        if arena is None:
            _lib.check(L.myolo_plan_create(*args, C.byref(h)))
        else:
            _lib.check(L.myolo_plan_create_shared(*args, _lib.ptr(arena.ws), _lib.ptr(arena.gws), arena.capacity, C.byref(h)))
        self.handle = h
        self.B, self.H, self.W = B, H, W
        self.weights_key = None              # Engine.weights_key() when the fp16 packs were last uploaded: stale when it differs
        self.weights_registered = None       # pointer signature of the tensors the library holds (myolo_plan_repack_weights)
        # train plans only (Engine.prepare_train_plan / train_forward)
        self._seed_set = False
        self._ptr_sig = None                 # parameter / gradient pointers registered with the library
        self._nbt = []                       # num_batches_tracked of the BatchNorm slots
        self._defer_running = False          # Engine.set_defer_running
        self._bn_owners = None               # (parent's _modules, name, module) of every BatchNorm slot, bound by the first prepare
        self.bn_sync = None                  # Engine.set_bn_sync: None (local statistics), ("nccl", comm) or ("ranks", images per rank)
        self.fwd_generation = 0              # train forwards of this plan (or of its arena): a backward is valid for the latest only

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
        self.weights_registered = sig

    def refresh_anchors(self, det):
        """rewrites each DETECT_DECODE op's anchors (pixels, in the plan's extra table since the plan was built) from det.anchor_grid as it
        is now, in place: an EMA averages anchor_grid with every other floating-point entry (reference utils/torch_utils.py:297-300), so
        its values move between validations.  fp16 after model.half(): the same values the plan would take from a fresh build."""
        L, sp = _lib.lib(), _lib.stream_ptr()
        ag = det.anchor_grid.detach().to(dtype=torch.float32).contiguous()     # (nl, 1, na, 1, 1, 2)
        for o in self.pb.ops:
            if o.kind == _lib.OP_DETECT_DECODE:
                level, na, off = o.aux[0], o.aux[1], o.aux[5]
                src = ag[level].reshape(-1)
                assert src.numel() == 2 * na
                _lib.check(L.myolo_plan_set_extra(self.handle, off, _lib.ptr(src), 2 * na, sp))


class Engine:
    def __init__(self, model):
        self.model = model
        self.plans: Dict[Tuple[int, ...], CompiledPlan] = {}
        self.param_epoch = 0   # writes to parameters / buffers that torch's version counters do not see (Model.invalidate_weights)
        self.stats_epoch = 0   # train forwards: they move the BatchNorm running statistics through raw pointers
        self.last_plan = None
        self.last_profile = None
        self.noalias = False   # debug: give every buffer private memory so intermediate views stay readable after forward
        self._reserved = {}    # train plan key -> (TrainArena, host plan) (reserve_train_shapes)
        self._arenas = {}      # lane -> TrainArena
        self._train_params = []
        self._flat_grad = None
        self._flat_offsets = []
        self._grad_views = []
        self._anchor = None    # autograd input of _TrainFunction

    def weights_key(self, train):
        """what a plan's fp16 weight packs were made from; a plan re-packs before its next launch when the key differs from the one of its
        last upload.  Inference packs fold BatchNorm, so every parameter and buffer counts, the running statistics included; train packs
        do not fold it, so only the trainable parameters count (running statistics moving between optimiser steps repack nothing)."""
        if train:
            return sum(q._version for q in self._train_params), self.param_epoch
        ver = sum(q._version for q in self.model.parameters()) + sum(q._version for q in self.model.buffers())
        return ver, self.param_epoch, self.stats_epoch

    def _upload_if_stale(self, p):
        key = self.weights_key(p.train)
        if p.weights_key != key:
            p.upload_weights()                   # train plans: fp16, K-major, no BN folding
            if not p.train:
                p.refresh_anchors(self.model.model[-1])
            p.weights_key = key

    def plan_for(self, B, H, W, seg=True) -> CompiledPlan:
        """the inference plan of (B, H, W); seg=False: the one without the seg head (test-time augmentation's scaled passes)"""
        key = (B, H, W) if seg else ("det", B, H, W)
        if key not in self.plans:
            self.plans[key] = CompiledPlan(self.model, B, H, W, self.noalias, seg=seg)
        p = self.plans[key]
        self._upload_if_stale(p)
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

    def forward_augment(self, x: torch.Tensor, seg_argmax=False, det_only_scaled=True):
        """test-time augmentation, reference models/yolo.py:274-289 (Model.forward(augment=True)) with the fork's missing index restored
        (`forward_once(xi)[0][0]`): `[(z, None), seg]`, plus the argmax map with seg_argmax=True.  z (B, rows of the three passes, no) fp32
        holds, per image, pass 0's rows, then pass 1's (x.flip(3) scaled by 0.83), then pass 2's (scaled by 0.67), their boxes de-scaled
        and pass 1's x mirrored back, each pass's Detect decodes writing straight into its slice.  seg / argmax are pass 0's, those of
        augment=False; the scaled passes run plans without the seg head (det_only_scaled=False: the full plans, for comparison).  Every
        launch goes to the current stream; nothing synchronises with the host."""
        x = self._augment_input(x)
        B, _, H, W = x.shape
        det = self.model.model[-1]
        rows = self.augment_rows(H, W)
        dev = x.device
        z = torch.empty((B, rows, det.no), dtype=torch.float32, device=dev)
        seg_dt = self.seg_dtype(x)
        seg_head = self.model.model[-2]
        seg = torch.empty((B, seg_head.c_out, H, W), dtype=seg_dt, device=dev) if not seg_argmax else None
        amax = torch.empty((B, H, W), dtype=torch.int64, device=dev) if seg_argmax else None
        self.augment_passes(x, z, 0, seg, seg_dt, amax, det_only_scaled)
        out = [(z, None), seg]
        if seg_argmax:
            out.append(amax)
        return out

    @staticmethod
    def _augment_input(x):
        if not x.is_cuda:
            raise _lib.MyoloError("Model.forward(augment=True) needs a CUDA tensor: multiyolov5_b200 has no CPU path")
        if x.dtype not in (torch.float16, torch.float32):
            raise TypeError(f"Model.forward(augment=True) takes fp16 or fp32 input scaled to [0, 1] (detect.py divides by 255 first), "
                            f"not {x.dtype}")
        assert x.dim() == 4 and x.shape[1] == 3, "expected (B,3,H,W)"
        return x.contiguous()

    def seg_dtype(self, x):
        """like the reference: fp16 in (or model.half(), detect.py:96-103) -> fp16 seg logits; otherwise fp32"""
        half_model = next(self.model.parameters()).dtype == torch.float16
        return torch.float16 if (x.dtype == torch.float16 or half_model) else torch.float32

    def plain_rows(self, H, W):
        """z rows per image of a plain forward at (H, W)"""
        det = self.model.model[-1]
        return sum(det.na * (H // int(s)) * (W // int(s)) for s in det.stride)

    def augment_rows(self, H, W):
        """z rows per image of a test-time augmentation forward at (H, W): the three passes' rows"""
        from .utils.torch_utils import tta_passes
        gs = int(self.model.model[-1].stride.max())
        return sum(self.plain_rows(hp, wp) for _, _, _, (hp, wp) in tta_passes(H, W, gs))

    def augment_passes(self, x, z, z_off, seg, seg_dt, amax, det_only_scaled=True):
        """forward_augment's three passes over contiguous x, writing this model's rows from row z_off of z (B, rows, no) on, and pass 0's
        seg / argmax (both may be None: the pass-0 plan then keeps its low-res logits for myolo_seg_ensemble)"""
        from .utils.torch_utils import scale_img, tta_passes
        B, _, H, W = x.shape
        det = self.model.model[-1]
        gs = int(det.stride.max())
        passes = tta_passes(H, W, gs)
        offs = [z_off]
        for _, _, _, (hp, wp) in passes:
            offs.append(offs[-1] + self.plain_rows(hp, wp))
        L, sp = _lib.lib(), _lib.stream_ptr()
        # each pass's plan is looked up (and on first use built) right before its launches, so that this host work overlaps the
        # previous pass on the device
        for k, (si, flip, _, (hp, wp)) in enumerate(passes):
            p = self.plan_for(B, hp, wp, seg=(k == 0 or not det_only_scaled))
            assert sum(p.pb.det_rows) == offs[k + 1] - offs[k]
            if k == 0:
                self.last_plan = p
            xi = x if k == 0 else scale_img(x, si, gs=gs, flip_lr=flip)
            inv = float(np.float32(1.0) / np.float32(si))          # `yi[..., :4] /= si`: ATen multiplies by the fp32 reciprocal
            _lib.check(L.myolo_plan_forward_pass(p.handle, _lib.ptr(xi), _lib.torch_dtype_code(xi.dtype), _lib.ptr(z), z.shape[1], offs[k],
                                                 inv, W if flip else 0, _lib.ptr(seg if k == 0 else None), _lib.torch_dtype_code(seg_dt),
                                                 _lib.ptr(amax if k == 0 else None), sp))

    # ---- training (SURVEY.md section 8 row a13) -----------------------------------------------------------------------
    def train_plan_for(self, B, H, W, lane=0) -> CompiledPlan:
        """lane: independent train plans of the same shape (own activation / gradient workspaces) so that the two passes of a training step
        can be in flight at the same time (train.Trainer: the seg pass runs on lane 1)"""
        key = ("train", B, H, W) if lane == 0 else ("train", B, H, W, lane)
        if key not in self.plans:
            arena, pb = self._reserved.get(key, (None, None))
            self.plans[key] = CompiledPlan(self.model, B, H, W, train=True, arena=arena, pb=pb)
        return self.plans[key]

    def reserve_train_shapes(self, B, shapes, lane=0):
        """Train plans for batches of B images at each (H, W) of `shapes` on `lane` share ONE activation and ONE gradient workspace sized
        for the largest of them (--multi-scale, reference train.py:354-359: 33 sizes at imgsz 1024 would need ~97 GB of private
        workspaces; the shared pair needs 6.1 GB).  Builds the host plans now, allocates and zeroes the pair once; the device plans are
        created on first use.  A lane keeps its pair for good: more shapes may be reserved later if they fit, a larger reservation raises
        (the existing plans bake in the address).  Returns the TrainArena."""
        shapes = sorted({(int(h), int(w)) for h, w in shapes})
        if not shapes:
            raise ValueError("reserve_train_shapes: no shapes")
        keys = {hw: (("train", B) + hw if lane == 0 else ("train", B) + hw + (lane,)) for hw in shapes}
        arena = self._arenas.get(lane)
        pbs, need = shared_train_plans(self.model, B, [hw for hw in shapes
                                                       if arena is None or self._reserved.get(keys[hw], (None,))[0] is not arena])
        if arena is None:
            arena = TrainArena(need, next(self.model.parameters()).device)
            self._arenas[lane] = arena
        elif need > arena.capacity:
            raise _lib.MyoloError(f"lane {lane} already has a shared train workspace of {arena.capacity} bytes and the new shapes need {need}: "
                                  "it cannot grow under the plans bound to it; reserve every shape (the largest first) before training")
        for hw, pb in pbs.items():
            self.plans.pop(keys[hw], None)           # a private plan of this shape is rebuilt on the shared workspaces
            self._reserved[keys[hw]] = (arena, pb)
        return arena

    def ensure_flat_grads(self):
        """every parameter's .grad is a view into ONE flat fp32 buffer (what the data-parallel all-reduce moves, reference
        train.py:243-245 DDP semantics) that the backward kernels accumulate into."""
        params = [p for p in self.model.parameters() if p.requires_grad]
        self._train_params = params
        if self._flat_grad is not None and all(p.grad is not None and p.grad.data_ptr() == g.data_ptr()
                                                                  for p, g in zip(params, self._grad_views)):
            return self._flat_grad
        for p in params:
            assert p.dtype == torch.float32 and p.is_cuda, "training keeps fp32 master parameters on the GPU"
        self._flat_offsets, n = flat_offsets(params)
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
        """seed, fp16 weight packs and parameter / gradient pointers of a train plan for the current parameter values (idempotent)"""
        L = _lib.lib()
        params = self._train_params
        if not p._seed_set:                      # dropout masks follow torch's global seed (one hash stream per plan)
            _lib.check(L.myolo_plan_set_seed(p.handle, C.c_uint64(torch.initial_seed() & 0xFFFFFFFFFFFFFFFF)))
            p._seed_set = True
        if p._bn_owners is None:
            self._bind_bn_sync(p)
        elif any(d.get(name) is not bn for d, name, bn in p._bn_owners):
            raise _lib.MyoloError(self._BN_CHANGED)
        self._upload_if_stale(p)
        sig = (self._flat_grad.data_ptr(), params[0].data_ptr(), params[-1].data_ptr(), len(params))
        if p._ptr_sig != sig:                    # (re)register parameter / gradient pointers only when they moved
            for i, s in enumerate(p.pb.slots):
                _lib.check(L.myolo_plan_set_conv_grad(p.handle, i, _lib.ptr(s.conv.weight.grad), _lib.ptr(s.conv.bias.grad if s.conv.bias is not None else None)))
            for i, bn in enumerate(p.pb.bn_slots):
                _lib.check(L.myolo_plan_set_bn(p.handle, i, bn.num_features, _lib.ptr(bn.weight), _lib.ptr(bn.bias), _lib.ptr(bn.running_mean),
                                               _lib.ptr(bn.running_var), _lib.ptr(bn.weight.grad), _lib.ptr(bn.bias.grad), float(bn.momentum), float(bn.eps)))
            p._ptr_sig = sig
            p._nbt = [bn.num_batches_tracked for bn in p.pb.bn_slots]

    _BN_CHANGED = ("the model's BatchNorm layers were replaced after its train plans were built (torch.nn.SyncBatchNorm."
                   "convert_sync_batchnorm?): those plans would normalise with the old layers' semantics.  Convert the model before its "
                   "first train forward and before building a Trainer, as reference train.py:190-193 does")

    def _bind_bn_sync(self, p):
        """first prepare of train plan p: remembers where each of its BatchNorm layers sits in the model (a layer replaced later raises
        instead of training with the old semantics) and, for SyncBatchNorm layers that synchronise (parallel.bn_sync_group), hands the
        group's NCCL communicator to the plan"""
        from .parallel import bn_sync_group, nccl_comm_ptr
        owners = {id(c): (m._modules, name) for m in self.model.modules() for name, c in m._modules.items()}
        if any(id(bn) not in owners for bn in p.pb.bn_slots):
            raise _lib.MyoloError(self._BN_CHANGED)
        group = bn_sync_group(p.pb.bn_slots)
        if group is not None:
            import torch.distributed as dist
            dev = torch.device("cuda", torch.cuda.current_device())
            comm = nccl_comm_ptr(group, dev)
            if comm is None:                     # torch creates the group's communicator at its first collective
                dist.all_reduce(torch.zeros(1, device=dev), group=group)
                comm = nccl_comm_ptr(group, dev)
            if comm is None:
                raise _lib.MyoloError("SyncBatchNorm: the process group has no NCCL communicator the library can use")
            self.set_bn_sync(p, comm=comm)
        p._bn_owners = [owners[id(bn)] + (bn,) for bn in p.pb.bn_slots]

    def set_bn_sync(self, plan, comm=None, rank_images=None):
        """synchronised BatchNorm for train plan `plan` (myolo_plan_set_bn_sync): comm = a raw ncclComm_t (parallel.nccl_comm_ptr), or
        rank_images = the images of each emulated rank (one-GPU rank emulation: the plan's batch split into consecutive groups); neither:
        local statistics.  The plan then runs without CUDA-graph replay."""
        imgs = None if rank_images is None else (C.c_int32 * len(rank_images))(*[int(n) for n in rank_images])
        _lib.check(_lib.lib().myolo_plan_set_bn_sync(plan.handle, C.c_void_p(comm) if comm else None, imgs,
                                                     0 if rank_images is None else len(rank_images)))
        plan.bn_sync = ("nccl", comm) if comm else (("ranks", tuple(int(n) for n in rank_images)) if rank_images is not None else None)

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
        if not p._defer_running:                         # a deferring plan counts its batch in apply_running
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
        gen = p.arena.claim(p) if p.arena is not None else None
        _lib.check(L.myolo_plan_train_forward_multi(p.handle, _lib.ptr(x), _lib.torch_dtype_code(x.dtype), raw_ptrs, seg_ptrs, sp))
        # activations / batch statistics / dropout step of THIS forward live in the plan's single workspace: a backward is only valid
        # for the most recent train forward of the plan (the reference's order forward, backward, forward, backward - train.py:364-392);
        # plans on a shared workspace: for the most recent train forward of ANY plan bound to it
        p.fwd_generation = gen if gen is not None else p.fwd_generation + 1
        self.stats_epoch += 1                            # running_mean / running_var moved: inference packs are stale
        self.last_plan = p
        return raws, (segs[0] if n_seg == 1 else segs), p

    def set_defer_running(self, plan):
        """from now on `plan`'s forwards leave running_mean / running_var / num_batches_tracked alone (apply_running moves them): lets the
        seg pass's forward run next to the det pass's while the statistics still move in the reference's order"""
        if not plan._defer_running:
            _lib.check(_lib.lib().myolo_plan_set_defer_running(plan.handle, 1))
            plan._defer_running = True

    def apply_running(self, plan):
        _lib.check(_lib.lib().myolo_plan_apply_running(plan.handle, _lib.stream_ptr()))
        torch._foreach_add_(plan._nbt, 1)

    def _check_generation(self, plan, generation):
        a = plan.arena
        if a is not None and (a.owner is not plan or (generation is not None and generation != a.generation)):
            raise _lib.MyoloError(f"backward of a stale train-mode forward: another train forward ran on the shared workspace of "
                                  f"({plan.B},{plan.H},{plan.W}) after it and overwrote the saved activations (one outstanding forward per "
                                  "lane; run forward, backward, forward, backward like reference train.py:364-392)")
        if generation is not None and generation != plan.fwd_generation:
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
        self._check_generation(plan, None)
        loss = torch.empty((), dtype=torch.float32, device=labels.device)
        _lib.check(_lib.lib().myolo_plan_backward_seg_ce(plan.handle, _lib.ptr(labels.contiguous()), int(ignore_index), float(factor),
                                                         _lib.ptr(scale), _lib.ptr(loss), _lib.stream_ptr()))
        return loss

    def train_backward_seg_ohem(self, plan, labels, thresh_t, factor=1.0, scale=None, ignore_index=-1):
        """train_backward_seg_ce with the reference's OhemCELoss in place of the mean CE (myolo_plan_backward_seg_ohem): the pixels whose
        CE exceeds thresh_t (= -log(thresh), utils.loss.OhemCELoss.thresh_t), or the (valid pixels // 16) largest when fewer are hard, chosen
        on the device.  Returns the OHEM loss (device scalar)."""
        assert labels.is_cuda and labels.dtype == torch.int64 and tuple(labels.shape) == (plan.B, plan.H, plan.W)
        self._check_generation(plan, None)
        loss = torch.empty((), dtype=torch.float32, device=labels.device)
        _lib.check(_lib.lib().myolo_plan_backward_seg_ohem(plan.handle, _lib.ptr(labels.contiguous()), int(ignore_index), float(thresh_t),
                                                           float(factor), _lib.ptr(scale), _lib.ptr(loss), _lib.stream_ptr()))
        return loss

    def train_backward_seg_loss(self, plan, labels, weights=None, gamma=0.0, factor=1.0, scale=None, ignore_index=-1):
        """train_backward_seg_ce with the class-weighted CE / focal loss in place of the mean CE (myolo_plan_backward_seg_loss):
        SegFocalLoss(gamma, alpha=weights, reduction='mean'), which with gamma = 0 is CrossEntropyLoss(weight=weights).  weights: None or
        an (n_segcls,) fp32 CUDA tensor, read by the kernels at their launch.  Returns the loss (device scalar)."""
        assert labels.is_cuda and labels.dtype == torch.int64 and tuple(labels.shape) == (plan.B, plan.H, plan.W)
        assert weights is None or (weights.is_cuda and weights.dtype == torch.float32 and weights.is_contiguous())
        self._check_generation(plan, None)
        loss = torch.empty((), dtype=torch.float32, device=labels.device)
        _lib.check(_lib.lib().myolo_plan_backward_seg_loss(plan.handle, _lib.ptr(labels.contiguous()), int(ignore_index), _lib.ptr(weights),
                                                           float(gamma), float(factor), _lib.ptr(scale), _lib.ptr(loss),
                                                           _lib.stream_ptr()))
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


def forward_ensemble(members, x: torch.Tensor, augment=False, seg_argmax=False):
    """Ensemble.forward in eval mode (models.experimental.Ensemble): `[(z, None), seg]`, plus the argmax map with seg_argmax=True.
    z (B, the members' rows, no) fp32 holds member 0's rows, then member 1's, ..., each member's Detect decodes writing straight into its
    slice (augment=True: each member's block is its forward_augment rows).  seg is the mean of the members' plain seg logits in the dtype
    one member returns, and the argmax map that of the fp32 mean: one myolo_seg_ensemble launch over the low-res logits the members'
    passes leave in their plans, with no full-size map per member.  The members were checked to agree (Ensemble.check_members).  Every
    launch goes to the current stream; nothing synchronises with the host."""
    if augment:
        x = Engine._augment_input(x)
    else:
        if not x.is_cuda:
            raise _lib.MyoloError("Ensemble.forward needs a CUDA tensor: multiyolov5_b200 has no CPU path (use the oracle for CPU numbers)")
        assert x.dim() == 4 and x.shape[1] == 3, "expected (B,3,H,W)"
        x = x.contiguous()
    B, _, H, W = x.shape
    engines = [m.engine() for m in members]
    rows = [e.augment_rows(H, W) if augment else e.plain_rows(H, W) for e in engines]
    offs = np.cumsum([0] + rows).tolist()
    dev = x.device
    z = torch.empty((B, offs[-1], members[0].model[-1].no), dtype=torch.float32, device=dev)
    seg_dt = engines[0].seg_dtype(x)
    L, sp = _lib.lib(), _lib.stream_ptr()
    plans = []
    for e, off, n in zip(engines, offs, rows):
        if augment:
            e.augment_passes(x, z, off, None, seg_dt, None)
            p = e.plans[(B, H, W)]                   # pass 0's plan: the plain one, with the seg head
        else:
            p = e.plan_for(B, H, W)                  # looked up right before its launches, as forward_augment does
            assert sum(p.pb.det_rows) == n
            _lib.check(L.myolo_plan_forward_pass(p.handle, _lib.ptr(x), _lib.torch_dtype_code(x.dtype), _lib.ptr(z), offs[-1], off, 1.0,
                                                 0, None, _lib.torch_dtype_code(seg_dt), None, sp))
        plans.append(p.handle)
    seg = torch.empty((B, members[0].model[-2].c_out, H, W), dtype=seg_dt, device=dev) if not seg_argmax else None
    amax = torch.empty((B, H, W), dtype=torch.int64, device=dev) if seg_argmax else None
    _lib.check(L.myolo_seg_ensemble((C.c_void_p * len(plans))(*[h.value for h in plans]), len(plans), _lib.ptr(seg),
                                    _lib.torch_dtype_code(seg_dt), _lib.ptr(amax), sp))
    out = [(z, None), seg]
    if seg_argmax:
        out.append(amax)
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
    if eng._anchor is None:
        eng._anchor = torch.zeros((), device=x.device, requires_grad=True)
    out = _TrainFunction.apply(eng._anchor, eng, x)
    return [list(out[:3]), out[3] if len(out) == 4 else list(out[3:])]     # BiSe: seg = [out, aux16, aux32] (models/yolo.py:86)
