"""One training iteration of the joint det+seg model, mirroring the step glue of reference train.py:363-401:

    det forward -> ComputeLoss x world_size x detgain -> scaled backward          (train.py:364-371)
    seg forward -> SegmentationLosses x batch_size x seggain -> scaled backward   (train.py:381-392; gradients ACCUMULATE)
    every `accumulate` iterations: ONE all-reduce of the flat gradient buffer (the reference's DDP reducer, train.py:243-245),
    GradScaler-style finite check, SGD(momentum, nesterov) with the three parameter groups of train.py:108-126, zero_grad.

What is GPU-native here: forward/backward are the hand-written kernels behind `Model.forward` (engine._TrainFunction); all
parameters, gradients and momentum buffers live in three FLAT fp32 buffers, so the collective is a single NCCL call over one
contiguous 31 MB region and the optimiser is a single HBM-bound launch (`myolo_sgd_step`) that also unscales, skips on overflow and
clears the gradients.  `torch.distributed` is plumbing only (process group + all_reduce on the flat buffer).

Out of scope (the reference's outer loop, not the hot path): data loading, LR schedule / warm-up (call `set_lr` / `set_momentum`),
EMA, checkpointing, plotting, DDP buffer broadcast.
"""
import os
import ctypes as C

import torch
import torch.nn as nn

from . import _lib
from .parallel import allreduce_flat_grads
from .utils.loss import ComputeLoss, FusedComputeLoss, SegmentationLosses


def scale_hyp(hyp: dict, nl: int, nc: int, imgsz: int, total_batch_size: int, nbs: int = 64, label_smoothing: float = 0.0) -> dict:
    """hyper-parameter scalings of reference train.py:102-104 (weight decay) and :248-251 (loss gains)"""
    h = dict(hyp)
    accumulate = max(round(nbs / total_batch_size), 1)
    h["weight_decay"] = hyp["weight_decay"] * total_batch_size * accumulate / nbs
    h["box"] = hyp["box"] * 3.0 / nl
    h["cls"] = hyp["cls"] * nc / 80.0 * 3.0 / nl
    h["obj"] = hyp["obj"] * (imgsz / 640) ** 2 * 3.0 / nl
    h["label_smoothing"] = label_smoothing
    return h


def parameter_groups(model: nn.Module):
    """{id(param): group} with group 0 = BatchNorm weights (no decay), 1 = other weights (decay), 2 = biases (reference train.py:108-116)"""
    grp = {}
    for _, m in model.named_modules():
        b = getattr(m, "bias", None)
        if isinstance(b, nn.Parameter):
            grp[id(b)] = 2
        w = getattr(m, "weight", None)
        if isinstance(m, nn.BatchNorm2d):
            grp[id(m.weight)] = 0
        elif isinstance(w, nn.Parameter):
            grp[id(w)] = 1
    return grp


class FlatState:
    """Parameters, gradients and momentum of a model as three flat fp32 CUDA buffers; `p.data` / `p.grad` become views."""

    def __init__(self, model: nn.Module):
        self.params = [p for p in model.parameters() if p.requires_grad]
        assert self.params and all(p.is_cuda and p.dtype == torch.float32 for p in self.params), "fp32 master parameters on the GPU"
        dev = self.params[0].device
        self.grad = model.engine().ensure_flat_grads()          # defines the (16-byte aligned) offsets shared by all three buffers
        self.offsets = list(model.engine()._flat_offsets)
        n = self.grad.numel()
        self.n = n
        self.param = torch.zeros(n, dtype=torch.float32, device=dev)
        self.momentum = torch.zeros(n, dtype=torch.float32, device=dev)
        self.group = torch.ones(n, dtype=torch.uint8, device=dev)
        groups = parameter_groups(model)
        for p, off in zip(self.params, self.offsets):
            k = p.numel()
            self.param[off:off + k].copy_(p.data.reshape(-1))
            p.data = self.param[off:off + k].view_as(p)
            self.group[off:off + k] = groups.get(id(p), 1)

    def check_views(self, model):
        """cheap guard: someone re-assigned parameters (.half(), load_state_dict with assign, .to()) -> views are stale"""
        p0, p1 = self.params[0], self.params[-1]
        ok = p0.data_ptr() == self.param.data_ptr() and p1.data_ptr() == self.param.data_ptr() + 4 * self.offsets[-1]
        g = model.engine().ensure_flat_grads()
        if not ok or g.data_ptr() != self.grad.data_ptr():
            raise RuntimeError("model parameters / gradients no longer alias the flat training buffers; rebuild the Trainer")


class Trainer:
    """`Trainer(model, hyp, batch_size).step(imgs, targets, segimgs, segtargets)`; hyp already scaled (see scale_hyp)."""

    def __init__(self, model, hyp, batch_size, world_size=1, rank=-1, accumulate=1, detgain=0.6, seggain=0.35, init_scale=2.0 ** 16,
                 growth_interval=2000, process_group=None, graph_loss=True, fused_seg_loss=True, overlap_passes=True, fused_det_loss=True,
                 concurrent_forwards=None):
        assert next(model.parameters()).is_cuda, "model.cuda() first"
        self.model, self.hyp, self.batch_size = model, hyp, batch_size
        self.world_size, self.rank, self.accumulate, self.pg = world_size, rank, accumulate, process_group
        self.detgain, self.seggain = detgain, seggain          # train.py:290
        model.hyp, model.gr = hyp, getattr(model, "gr", 1.0)
        model.train()
        self.compute_loss = ComputeLoss(model)
        # detection loss forward + backward as four launches of the library (csrc/detloss.cu) instead of ~760 torch kernels; the torch
        # formulation stays for focal loss / positive weights / autobalance and is what the tests compare it with
        self._fused_det = FusedComputeLoss(model) if fused_det_loss else None
        self.fused_det_loss = bool(fused_det_loss) and self._fused_det.supported
        self.n_seg_outputs = 3 if type(model.model[-2]).__name__ == "SegMaskBiSe" else 1
        # BiSe returns [out, aux16, aux32]: loss1 + 1.5*aux_weight*loss2 + 0.5*aux_weight*loss3 (reference train.py:387-388, utils/loss.py:239-244)
        self.compute_seg_loss = SegmentationLosses(ignore_index=-1, aux=self.n_seg_outputs == 3, aux_num=2)
        self.flat = FlatState(model)
        dev = self.flat.param.device
        self.lr = [hyp["lr0"]] * 3
        self.wd = [0.0, hyp["weight_decay"], 0.0]
        self.momentum = hyp["momentum"]
        self.scale = torch.full((), float(init_scale), device=dev)
        self.growth_tracker = torch.zeros((), dtype=torch.int32, device=dev)
        self.growth_interval = growth_interval
        self.found_inf = torch.zeros(1, dtype=torch.int32, device=dev)
        self.inv_scale = torch.ones((), device=dev)
        self.ni = 0
        self.graph_loss = graph_loss        # replay the detection loss (forward + autograd backward, ~700 tiny kernels) as ONE CUDA graph
        self._det_graphs = {}
        self.fused_seg_loss = fused_seg_loss  # CE + x8 upsample forward/backward in one kernel, no full-resolution logits (plain heads only)
        # overlap_passes: the seg pass runs on its own train plan and stream.  Its forward starts when the det FORWARD has finished (BatchNorm
        # running statistics are then updated in the reference's order, det batch first: train.py:364,381), so the seg forward/backward
        # overlaps the det loss + backward; parameter gradients of both passes add up atomically in the one flat buffer.  At 4 images per
        # pass the kernels are launch/latency bound and each pass alone leaves most of the 132 SMs idle.
        self.overlap_passes = bool(overlap_passes) and (graph_loss or fused_det_loss)
        self._s_seg = torch.cuda.Stream() if self.overlap_passes else None
        if concurrent_forwards is None:
            concurrent_forwards = os.environ.get("MYOLO_CONCURRENT_FWD", "1") != "0"
        self.concurrent_forwards = bool(concurrent_forwards) and self.overlap_passes
        self._ev_detfwd, self._ev_start, self._ev_seg = torch.cuda.Event(), torch.cuda.Event(), torch.cuda.Event()

    def set_lr(self, lr_bn, lr_weight, lr_bias):
        self.lr = [float(lr_bn), float(lr_weight), float(lr_bias)]

    def set_momentum(self, m):
        self.momentum = float(m)

    # ---- the two passes --------------------------------------------------------------------------------------------
    def _det_loss_scaled(self, p, targets):
        loss, items = self.compute_loss(p, targets)
        if self.rank != -1:
            loss = loss * self.world_size                                         # train.py:367-368
        return loss * self.detgain * self.scale, items

    def _det_graph(self, shapes, nt_pad, dev):
        """static inputs (head outputs, padded targets) -> static outputs (d loss / d head outputs, loss items), captured once per
        (grid shapes, padded target count).  Padding rows are all-zero targets: zero width/height never matches an anchor."""
        # every scalar the captured kernels bake in is part of the key: changing hyp / gains / gr / autobalance state re-captures
        cl = self.compute_loss
        key = (tuple(shapes), nt_pad, self.detgain, self.world_size, self.rank, float(getattr(self.model, "gr", 1.0)),
               tuple(sorted((k, float(v)) for k, v in self.hyp.items() if isinstance(v, (int, float)))),
               tuple(float(b) for b in getattr(cl, "balance", ())), bool(getattr(cl, "autobalance", False)))
        st = self._det_graphs.get(key)
        if st is not None:
            return st

        class _St:
            pass
        st = _St()
        st.p = [torch.zeros(sh, dtype=torch.float32, device=dev, requires_grad=True) for sh in shapes]
        st.t = torch.zeros((nt_pad, 6), dtype=torch.float32, device=dev)
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):                                             # warm-up off the capture stream (allocator, cuBLAS-free)
            for _ in range(2):
                for q in st.p:
                    q.grad = None
                loss, _ = self._det_loss_scaled(st.p, st.t)
                loss.backward()
        torch.cuda.current_stream().wait_stream(side)
        for q in st.p:
            q.grad = None
        st.graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(st.graph):
            loss, st.items = self._det_loss_scaled(st.p, st.t)
            loss.backward()
        self._det_graphs[key] = st
        return st

    def backward_det(self, imgs, targets):
        if self.fused_det_loss:
            eng = self.model.engine()
            raws, _, plan = eng.train_forward(imgs, want_seg=False)
            self._ev_detfwd.record(torch.cuda.current_stream())
            mult = (self.world_size if self.rank != -1 else 1) * self.detgain              # train.py:367-368 and :290
            grads, items = self._fused_det(raws, targets, mult=mult, scale=self.scale)
            eng.train_backward(plan, grads, None)
            return items
        if not self.graph_loss:
            pred = self.model(imgs)                                               # train mode: [[x0,x1,x2], seg]
            loss, items = self._det_loss_scaled(pred[0], targets)
            loss.backward()
            return items
        eng = self.model.engine()
        B, _, H, W = imgs.shape
        det = self.model.model[-1]
        shapes = [(B, det.na, H // int(s), W // int(s), det.no) for s in det.stride.tolist()]
        nt = targets.shape[0]
        nt_pad = max(64, (nt + 63) // 64 * 64)
        st = self._det_graph(shapes, nt_pad, imgs.device)
        st.t.zero_()
        if nt:
            st.t[:nt].copy_(targets)
        _, _, plan = eng.train_forward(imgs, out_raws=st.p, want_seg=False)       # head outputs land in the graph's static inputs
        self._ev_detfwd.record(torch.cuda.current_stream())
        st.graph.replay()
        eng.train_backward(plan, [q.grad for q in st.p], None)
        return st.items.clone()                                                   # the static tensor is overwritten by the next replay

    def backward_seg(self, segimgs, segtargets, lane=0):
        # the fused kernels are instantiated for 19 (Cityscapes) and 32 classes; any other n_segcls takes the autograd path below
        if self.fused_seg_loss and self.n_seg_outputs == 1 and self.model.model[-2].c_out in (19, 32):
            eng = self.model.engine()
            _, _, plan = eng.train_forward(segimgs, want_seg=False, lane=lane)
            loss = eng.train_backward_seg_ce(plan, segtargets, factor=self.batch_size * self.seggain, scale=self.scale)
            return loss * (self.batch_size * self.seggain)
        pred = self.model(segimgs)
        outs = pred[1] if isinstance(pred[1], list) else [pred[1]]
        segloss = self.compute_seg_loss(*outs, segtargets) * self.batch_size * self.seggain   # train.py:385-391
        (segloss * self.scale).backward()
        return segloss.detach()

    # ---- reduce + optimiser ------------------------------------------------------------------------------------------
    def allreduce(self):
        if self.world_size > 1:
            world = allreduce_flat_grads(self.flat.grad, group=self.pg)
            assert world == self.world_size, f"process group has {world} ranks, Trainer was built for {self.world_size}"

    def optimizer_step(self):
        f = self.flat
        f.check_views(self.model)
        self.allreduce()
        L, sp = _lib.lib(), _lib.stream_ptr()
        torch.reciprocal(self.scale * float(self.world_size), out=self.inv_scale)  # DDP averages: sum / world_size
        _lib.check(L.myolo_grads_check_finite(_lib.ptr(f.grad), f.n, _lib.ptr(self.found_inf), sp))
        lr = (C.c_float * 3)(*self.lr)
        wd = (C.c_float * 3)(*self.wd)
        _lib.check(L.myolo_sgd_step(_lib.ptr(f.param), _lib.ptr(f.grad), _lib.ptr(f.momentum), _lib.ptr(f.group), f.n, lr, wd, 3,
                                    float(self.momentum), 1, _lib.ptr(self.inv_scale), _lib.ptr(self.found_inf), 1, sp))
        # amp.GradScaler.update: halve on overflow, double after growth_interval clean steps (device-side, no host sync)
        bad = self.found_inf[0] != 0
        tracker = torch.where(bad, torch.zeros_like(self.growth_tracker), self.growth_tracker + 1)
        grow = tracker >= self.growth_interval
        self.scale.copy_(torch.where(bad, self.scale * 0.5, torch.where(grow, self.scale * 2.0, self.scale)))   # in place: graphs read it
        self.growth_tracker.copy_(torch.where(grow, torch.zeros_like(tracker), tracker))
        self.model.engine().weights_dirty = True

    def step(self, imgs, targets, segimgs, segtargets):
        """one iteration (train.py:363-401).  Returns (det loss items [lbox,lobj,lcls,loss], seg loss) as device tensors."""
        fused_seg = self.fused_seg_loss and self.n_seg_outputs == 1 and self.model.model[-2].c_out in (19, 32)
        if self.overlap_passes and fused_seg:
            main = torch.cuda.current_stream()
            self._ev_start.record(main)
            # the seg pass runs on its own train plan and stream.  Its forward starts with the det forward (both are chains of small
            # launches at 4 images: two chains fill the machine better than one); its BatchNorm running statistics are deferred and
            # applied after the det forward, i.e. in the reference's order (train.py:364 det batch, :385 seg batch)
            with torch.cuda.stream(self._s_seg):
                self._s_seg.wait_event(self._ev_start)
                eng = self.model.engine()
                B, _, H, W = segimgs.shape
                eng.ensure_flat_grads()
                plan = eng.train_plan_for(B, H, W, lane=1)
                eng.set_defer_running(plan, self.concurrent_forwards)
                eng.prepare_train_plan(plan)
                if self.concurrent_forwards:
                    eng.train_forward(segimgs, want_seg=False, lane=1)
            items = self.backward_det(imgs, targets)                 # records _ev_detfwd right after the det forward
            with torch.cuda.stream(self._s_seg):
                self._s_seg.wait_event(self._ev_detfwd)
                if self.concurrent_forwards:
                    eng.apply_running(plan)
                    segloss = eng.train_backward_seg_ce(plan, segtargets, factor=self.batch_size * self.seggain, scale=self.scale)
                    segloss = segloss * (self.batch_size * self.seggain)
                else:                                                # forward after the det forward, overlapping the det backward
                    segloss = self.backward_seg(segimgs, segtargets, lane=1)
                self._ev_seg.record(self._s_seg)
            main.wait_event(self._ev_seg)
            segimgs.record_stream(self._s_seg); segtargets.record_stream(self._s_seg)
        else:
            items = self.backward_det(imgs, targets)
            segloss = self.backward_seg(segimgs, segtargets)
        self.ni += 1
        if self.ni % self.accumulate == 0:
            self.optimizer_step()
        return items, segloss
