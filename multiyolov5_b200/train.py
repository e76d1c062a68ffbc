"""One training iteration of the joint det+seg model, mirroring the step glue of reference train.py:363-401:

    det forward -> ComputeLoss x world_size x detgain -> scaled backward          (train.py:364-371)
    seg forward -> SegmentationLosses x batch_size x seggain -> scaled backward   (train.py:381-392; gradients ACCUMULATE)
    every `accumulate` iterations: ONE all-reduce of the flat gradient buffer (the reference's DDP reducer, train.py:243-245),
    GradScaler-style finite check, SGD(momentum, nesterov) with the three parameter groups of train.py:108-126, zero_grad.

What is GPU-native here: forward/backward are the hand-written kernels behind `Model.forward` (engine._TrainFunction); all
parameters, gradients and momentum buffers live in three FLAT fp32 buffers, so the collective is a single NCCL call over one
contiguous 31 MB region and the optimiser is a single HBM-bound launch (`myolo_sgd_step`) that also unscales, skips on overflow and
clears the gradients.  `torch.distributed` is plumbing only (process group + all_reduce on the flat buffer).

`Trainer(..., optimizer="adam")` is the reference's `--adam` (train.py:128-137): torch.optim.Adam with the same three groups, one
more flat buffer for the second moment and one launch (`myolo_adam_step`).  `Trainer.state_dict()` / `load_state_dict()` convert the flat
optimiser buffers to and from torch's `optimizer.state_dict()` format, which is what the reference's checkpoints hold in
`ckpt['optimizer']` (train.py:482-494, restored at :155-160).

`Trainer(..., ema=ModelEMA(model))` is the reference's `ema.update(model)` after every optimizer step (train.py:401), including a step
skipped for overflow: one launch (`myolo_ema_update`) over every floating-point entry of the model, bit-identical with the reference's
per-entry statements.  Pass it on rank -1 / 0 and None elsewhere, as train.py:151 builds it.

`Trainer(..., seg_loss=OhemCELoss(0.7))` trains with the reference's OHEM segmentation loss (train.py:285-288) in place of
SegmentationLosses; `seg_loss=SegmentationLosses(weight=w)` with its class-weighted CE (train.py:269-282), and
`seg_loss=SegFocalLoss(gamma=2, ignore_index=-1)` with its focal loss (train_custom.py:284).

`Trainer(..., quad=True)` is the reference's `--quad`: det batches from `utils.datasets.collate_quad` (collate_fn4) and the det loss x 4
(train.py:368-369).

A model converted with torch.nn.SyncBatchNorm.convert_sync_batchnorm (the reference's --sync-bn, train.py:190-193) trains with
BatchNorm statistics exchanged across the ranks of its NCCL process group inside the train plans (Engine.set_bn_sync); the two passes of a
step then run one after the other.  At world size 1, or without torch.distributed, it trains exactly like the plain model, as torch does.

`fit(model, hyp, opt, det_batches, seg_batches, ...)` is the reference's epoch loop (train.py:44-543) around the step: `LRSchedule` (warm-up,
LambdaLR, momentum, accumulation), the validation cadence, fitness2 and best.pt, results.txt, last.pt / best.pt and resume.
`DetEpochBatches` / `SegEpochBatches` give each epoch's batches from the device loaders in the reference's order, and `SegValBatches` the
seg validation batches (mode='val' or 'testval') for `fit(..., segval_loader=)`.

`evolve(hyp, opt, train_fn)` is the reference's --evolve (train.py:637-717): generations of `train_fn` (a training run such as `fit`),
each with hyper-parameters mutated from the best earlier results in evolve.txt.

Out of scope: loading and decoding data files, plotting, W&B / TensorBoard, --bucket, DDP buffer broadcast.
"""
import collections
import math
import random
import time
import ctypes as C

import numpy as np
import torch
import torch.nn as nn

from . import _lib
from .engine import flat_offsets
from .parallel import allreduce_flat_grads, bn_sync_group
from .utils.general import init_seeds, one_cycle
from .utils.loss import FusedComputeLoss, OhemCELoss, SegFocalLoss, SegmentationLosses, seg_focal_loss


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


def reference_param_groups(model: nn.Module):
    """[pg0, pg1, pg2] = BatchNorm weights (no decay), other weights (decay), biases, each in named_modules() order, as reference
    train.py:119-126 builds them.  The reference's optimizer numbers its parameters in this order (pg0, then pg1, then pg2), which is
    neither model.parameters() order nor the flat buffers' order."""
    pg0, pg1, pg2 = [], [], []
    for _, m in model.named_modules():
        b = getattr(m, "bias", None)
        if isinstance(b, nn.Parameter):
            pg2.append(b)
        w = getattr(m, "weight", None)
        if isinstance(m, nn.modules.batchnorm._BatchNorm):     # nn.BatchNorm2d, and nn.SyncBatchNorm after convert_sync_batchnorm
            pg0.append(m.weight)
        elif isinstance(w, nn.Parameter):
            pg1.append(w)
    return [pg0, pg1, pg2]


def parameter_groups(model: nn.Module):
    """{id(param): group} with group 0 = BatchNorm weights (no decay), 1 = other weights (decay), 2 = biases (reference train.py:108-116)"""
    return {id(p): k for k, pg in enumerate(reference_param_groups(model)) for p in pg}


# ---- optimiser state in torch's format ---------------------------------------------------------------------------------------------
OPTIMIZER_STATE = {"sgd": ("momentum_buffer",), "adam": ("exp_avg", "exp_avg_sq")}     # per-parameter state tensors, in torch's order


def default_param_groups(optimizer: str, hyp: dict):
    """the three param_groups entries (without 'params') of the reference's optimizer when it writes its first checkpoint: the keys and
    defaults of torch.optim.SGD(nesterov=True) / torch.optim.Adam under the installed torch, built as train.py:128-137 builds them
    (pg1 with hyp['weight_decay']), plus the 'initial_lr' = hyp['lr0'] that its LambdaLR adds"""
    ps = [torch.zeros(1) for _ in range(3)]
    if optimizer == "sgd":
        opt = torch.optim.SGD(ps[:1], lr=hyp["lr0"], momentum=hyp["momentum"], nesterov=True)
    elif optimizer == "adam":
        opt = torch.optim.Adam(ps[:1], lr=hyp["lr0"], betas=(hyp["momentum"], 0.999))
    else:
        raise ValueError(f"optimizer must be 'sgd' or 'adam', got {optimizer!r}")
    opt.add_param_group({"params": ps[1:2], "weight_decay": hyp["weight_decay"]})
    opt.add_param_group({"params": ps[2:]})
    return [dict({k: v for k, v in g.items() if k != "params"}, initial_lr=hyp["lr0"]) for g in opt.param_groups]


def _flat_slices(model):
    """{id(param): (offset, numel)} of the parameters in the flat buffers (engine.flat_offsets over model.parameters()), and n.
    The flat buffers hold trainable parameters only, while the reference's groups (and so its state dict's indices) also number frozen
    ones (its `freeze` list, train.py:106-112): a model with frozen parameters is refused."""
    params = list(model.parameters())
    frozen = [n for n, p in model.named_parameters() if not p.requires_grad]
    if frozen:
        raise ValueError(f"optimizer state of a model with frozen parameters is not supported: {frozen[:3]}{' ...' if len(frozen) > 3 else ''}")
    offsets, n = flat_offsets(params)
    return {id(p): (o, p.numel()) for p, o in zip(params, offsets)}, n


def optimizer_state_dict(model, optimizer: str, groups, steps: int, buffers):
    """torch's `optimizer.state_dict()` of the reference's optimizer over `model`, from flat buffers.
    groups: the three groups' settings (dicts without 'params'); steps: optimiser steps taken that were not skipped (0: torch has no
    state yet); buffers: {state name: flat fp32 tensor (CPU or CUDA)} laid out as the Trainer's flat buffers.  State tensors are copies on
    the buffers' device; Adam's 'step' is a CPU float32 scalar, as torch keeps it (capturable=False)."""
    slices, _ = _flat_slices(model)
    state, param_groups, i = {}, [], 0
    for g, ps in zip(groups, reference_param_groups(model)):
        ids = list(range(i, i + len(ps)))
        i += len(ps)
        if steps:
            for j, p in zip(ids, ps):
                o, k = slices[id(p)]
                st = {"step": torch.tensor(float(steps), dtype=torch.float32)} if optimizer == "adam" else {}
                for name in OPTIMIZER_STATE[optimizer]:
                    st[name] = buffers[name][o:o + k].view_as(p).clone()
                state[j] = st
        param_groups.append(dict(g, params=ids))
    return {"state": state, "param_groups": param_groups}


def optimizer_kind(sd) -> str:
    """'sgd' or 'adam' from the keys of a state dict's param_groups"""
    groups = sd.get("param_groups") if isinstance(sd, dict) else None
    if not groups:
        raise ValueError("not an optimizer state dict: no param_groups")
    if all("betas" in g for g in groups):
        return "adam"
    if all("momentum" in g and "nesterov" in g for g in groups):
        return "sgd"
    raise ValueError("optimizer state dict is neither torch.optim.SGD's nor torch.optim.Adam's")


def _check_same(groups, key):
    vals = [g[key] for g in groups]
    if any(v != vals[0] for v in vals[1:]):
        raise ValueError(f"the flat optimiser step takes one {key!r} for all groups, the state dict has {vals}")


def optimizer_state_from_dict(model, optimizer: str, sd, device=None):
    """inverse of optimizer_state_dict: (groups, steps, buffers) from torch's state dict of the reference's optimizer over `model` (e.g. a
    reference checkpoint's ckpt['optimizer'], tensors on any device).  groups keep every key of the dict's groups; buffers are new flat fp32
    tensors on `device`, zero where the dict has no state; steps is Adam's step count, for SGD 1 when the dict has state, else 0.
    Raises ValueError when the optimizer kind is not `optimizer`, the group sizes differ from the model's, a state tensor has the wrong
    shape, state is missing for some parameters, the Adam step counts differ, or a setting is one the flat step does not implement."""
    kind = optimizer_kind(sd)
    if kind != optimizer:
        raise ValueError(f"the state dict is {kind}'s, this optimizer is {optimizer}")
    groups = sd["param_groups"]
    pgs = reference_param_groups(model)
    if [len(g["params"]) for g in groups] != [len(pg) for pg in pgs]:
        raise ValueError(f"parameter group sizes {[len(g['params']) for g in groups]} != the model's {[len(pg) for pg in pgs]}")
    if optimizer == "sgd":
        if not all(g["nesterov"] and g.get("dampening", 0) == 0 and not g.get("maximize", False) for g in groups):
            raise ValueError("only SGD(nesterov=True, dampening=0, maximize=False) is implemented")
        _check_same(groups, "momentum")
    else:
        if any(g.get("amsgrad", False) or g.get("maximize", False) or g.get("decoupled_weight_decay", False) for g in groups):
            raise ValueError("only Adam(amsgrad=False, maximize=False, decoupled_weight_decay=False) is implemented")
        _check_same(groups, "betas")
        _check_same(groups, "eps")
    slices, n = _flat_slices(model)
    buffers = {name: torch.zeros(n, dtype=torch.float32, device=device) for name in OPTIMIZER_STATE[optimizer]}
    state, seen, steps = sd.get("state", {}), 0, set()
    for g, ps in zip(groups, pgs):
        for j, p in zip(g["params"], ps):
            st = state.get(j)
            if st is None:
                continue
            seen += 1
            o, k = slices[id(p)]
            for name in OPTIMIZER_STATE[optimizer]:
                t = st.get(name)
                if not isinstance(t, torch.Tensor) or tuple(t.shape) != tuple(p.shape):
                    raise ValueError(f"state {j} {name!r}: expected a tensor of shape {tuple(p.shape)}, got "
                                     f"{tuple(t.shape) if isinstance(t, torch.Tensor) else type(t).__name__}")
                buffers[name][o:o + k].copy_(t.reshape(-1))
            if optimizer == "adam":
                steps.add(float(st["step"]))
    if seen not in (0, sum(len(pg) for pg in pgs)):
        raise ValueError(f"the state dict has state for {seen} of {sum(len(pg) for pg in pgs)} parameters")
    if len(steps) > 1:
        raise ValueError(f"Adam step counts differ between parameters: {sorted(steps)}")
    nsteps = (int(steps.pop()) if optimizer == "adam" else 1) if seen else 0
    return [{k: v for k, v in g.items() if k != "params"} for g in groups], nsteps, buffers


class FlatState:
    """Parameters, gradients and momentum of a model as three flat fp32 CUDA buffers; `p.data` / `p.grad` become views.  With adam,
    `momentum` is Adam's first moment (exp_avg) and a fourth buffer, `exp_avg_sq`, holds the second."""

    def __init__(self, model: nn.Module, adam: bool = False):
        self.params = [p for p in model.parameters() if p.requires_grad]
        assert self.params and all(p.is_cuda and p.dtype == torch.float32 for p in self.params), "fp32 master parameters on the GPU"
        dev = self.params[0].device
        self.grad = model.engine().ensure_flat_grads()          # defines the (16-byte aligned) offsets shared by all three buffers
        self.offsets = list(model.engine()._flat_offsets)
        n = self.grad.numel()
        self.n = n
        self.param = torch.zeros(n, dtype=torch.float32, device=dev)
        self.momentum = torch.zeros(n, dtype=torch.float32, device=dev)
        self.exp_avg_sq = torch.zeros(n, dtype=torch.float32, device=dev) if adam else None
        self.group = torch.ones(n, dtype=torch.uint8, device=dev)
        groups = parameter_groups(model)
        for p, off in zip(self.params, self.offsets):
            k = p.numel()
            self.param[off:off + k].copy_(p.data.reshape(-1))
            p.data = self.param[off:off + k].view_as(p)
            self.group[off:off + k] = groups.get(id(p), 1)
        if hasattr(model, "tensors_moved"):
            model.tensors_moved()                                 # a ModelEMA built before the Trainer re-reads the new addresses

    def check_views(self, model):
        """cheap guard: someone re-assigned parameters (.half(), load_state_dict with assign, .to()) -> views are stale"""
        p0, p1 = self.params[0], self.params[-1]
        ok = p0.data_ptr() == self.param.data_ptr() and p1.data_ptr() == self.param.data_ptr() + 4 * self.offsets[-1]
        g = model.engine().ensure_flat_grads()
        if not ok or g.data_ptr() != self.grad.data_ptr():
            raise RuntimeError("model parameters / gradients no longer alias the flat training buffers; rebuild the Trainer")


class MultiScale:
    """--multi-scale (reference train.py:354-359): each iteration rescales the det batch so that its long side is a random multiple of gs
    in [imgsz/2, imgsz*3/2], with torch's bilinear (align_corners=False) interpolation, before the forward.

        sz = random.randrange(imgsz * 0.5, imgsz * 1.5 + gs) // gs * gs
        sf = sz / max(imgs.shape[2:])
        if sf != 1: ns = [math.ceil(x * sf / gs) * gs for x in imgs.shape[2:]]; imgs = F.interpolate(imgs, size=ns, ...)

    The reference passes float bounds to randrange, which Python 3.12 rejects; the draw here takes int() of the two bounds, which
    consumes the `random` stream exactly as Python <= 3.11 did with integral floats (istart + _randbelow(width)).  Only the det batch is
    rescaled: the seg batch, hyp['obj'] (scaled by imgsz) and the normalised targets stay as they are."""

    def __init__(self, imgsz, gs=32):
        self.imgsz, self.gs = int(imgsz), int(gs)
        lo, hi = imgsz * 0.5, imgsz * 1.5 + gs
        if lo != int(lo) or hi != int(hi):                   # what randrange of Python <= 3.11 raised for non-integral floats
            raise ValueError(f"non-integer bounds {lo}, {hi} for randrange()")
        self.lo, self.hi = int(lo), int(hi)

    def _ns(self, sz, shape):
        sf = sz / max(shape)
        if sf == 1:
            return None
        return [math.ceil(x * sf / self.gs) * self.gs for x in shape]

    def size(self, shape, rng=random):
        """one draw: the new (H, W) as a list, or None when the batch keeps its size (sf == 1)"""
        sz = rng.randrange(self.lo, self.hi) // self.gs * self.gs
        return self._ns(sz, tuple(int(x) for x in shape))

    def shapes(self, shape):
        """every (H, W) a batch of `shape` can have after a draw, ascending: the rescaled sizes, and `shape` itself when a draw can keep it"""
        shape = tuple(int(x) for x in shape)
        out = set()
        for sz in {v // self.gs * self.gs for v in range(self.lo, self.hi)}:
            ns = self._ns(sz, shape)
            out.add(shape if ns is None else tuple(ns))
        return sorted(out)

    def __call__(self, imgs, out_dtype=torch.float16, rng=random):
        """draws once and rescales the (B, C, H, W) det batch on the device (uint8 / fp16 / fp32 in; uint8 is converted as
        imgs.float() / 255.0 first).  fp16 out is the fp32 result rounded to nearest, which is what the train plan's input conversion does
        to fp32 input.  When the draw keeps the size, a float batch of the requested dtype comes back as it is, without a launch."""
        if out_dtype not in (torch.float16, torch.float32):
            raise ValueError(f"MultiScale: out_dtype must be float16 or float32, got {out_dtype}")
        if imgs.dtype not in (torch.uint8, torch.float16, torch.float32) or imgs.dim() != 4 or not imgs.is_cuda:
            raise ValueError("MultiScale: expected a CUDA (B, C, H, W) uint8 / float16 / float32 tensor")
        ns = self.size(imgs.shape[2:], rng)
        if ns is None and imgs.dtype == out_dtype:
            return imgs
        return resize_bilinear(imgs, imgs.shape[2:] if ns is None else ns, out_dtype)


def resize_bilinear(x, size, out_dtype=torch.float32):
    """F.interpolate(x, size, mode='bilinear', align_corners=False) of a CUDA NCHW tensor on the library's kernel, bit exact with torch's
    for fp32 input; uint8 input is converted as x.float() / 255.0 first; fp16 out = the fp32 result rounded to nearest"""
    x = x.contiguous()
    B, Cc, H, W = x.shape
    Ho, Wo = int(size[0]), int(size[1])
    out = torch.empty((B, Cc, Ho, Wo), dtype=out_dtype, device=x.device)
    _lib.check(_lib.lib().myolo_resize_bilinear(_lib.ptr(x), _lib.torch_dtype_code(x.dtype), B, Cc, H, W, _lib.ptr(out),
                                                _lib.torch_dtype_code(out_dtype), Ho, Wo, _lib.stream_ptr()))
    return out


def _check_weighted_seg_loss(seg_loss, n_seg_outputs, n_segcls):
    """ValueError unless a SegmentationLosses / SegFocalLoss seg_loss fits the head and the loop (ignore_index -1, the segtargets'
    marker); returns its class weights (None: unit weights).  Other losses pass through with None."""
    if isinstance(seg_loss, SegmentationLosses):
        name = "SegmentationLosses"
        if seg_loss.weight is None:
            raise ValueError("seg_loss=SegmentationLosses() without weight is the default loss: pass seg_loss=None for it")
        bise = n_seg_outputs == 3
        if seg_loss.aux != bise or (bise and seg_loss.aux_num != 2):
            raise ValueError(f"SegmentationLosses(aux={seg_loss.aux}, aux_num={seg_loss.aux_num}) does not fit a seg head with "
                             f"{n_seg_outputs} output(s): aux=True, aux_num=2 is for the BiSe head's [out, aux16, aux32] only")
        weight = seg_loss.weight
    elif isinstance(seg_loss, SegFocalLoss):
        name = "SegFocalLoss"
        if n_seg_outputs != 1:
            raise ValueError("SegFocalLoss has no auxiliary outputs: it does not fit the BiSe head's [out, aux16, aux32]")
        if seg_loss.reduction != "mean":
            raise ValueError(f"SegFocalLoss(reduction={seg_loss.reduction!r}): the training loop takes reduction='mean'")
        weight = seg_loss.weight
    else:
        return None
    if seg_loss.ignore_index != -1:
        raise ValueError(f"{name}(ignore_index={seg_loss.ignore_index}): the seg targets mark ignored pixels with -1; pass ignore_index=-1")
    if weight is not None and weight.numel() != n_segcls:
        raise ValueError(f"{name}: {weight.numel()} class weights for a seg head of {n_segcls} classes")
    return weight


class Trainer:
    """`Trainer(model, hyp, batch_size).step(imgs, targets, segimgs, segtargets)`; hyp already scaled (see scale_hyp)."""

    def __init__(self, model, hyp, batch_size, world_size=1, rank=-1, accumulate=1, detgain=0.6, seggain=0.35, init_scale=2.0 ** 16,
                 growth_interval=2000, process_group=None, multi_scale=None, det_shapes=None, optimizer="sgd", ema=None, quad=False,
                 seg_loss=None):
        """multi_scale: a MultiScale.  The det lane's train plans for every size it can draw from an imgsz x imgsz batch are reserved on
        one shared workspace (Engine.reserve_train_shapes); rescale each det batch with `multi_scale(imgs)` before `step`, as the reference
        does before its forward (train.py:354-359).  A det batch of fewer images (the loader's partial last batch) reserves its sizes on
        the same workspace the first time it comes; a batch of more images than batch_size does not fit it and raises MyoloError.
        det_shapes: the (H, W) shapes of the det batches (--rect: DetRectLoader.batch_shapes).  Their train plans are reserved on that one
        shared workspace instead of a private pair per shape; with multi_scale, every size it can draw from each of them.
        optimizer: "sgd" (torch.optim.SGD(momentum=hyp['momentum'], nesterov=True)) or "adam" (the reference's --adam:
        torch.optim.Adam(betas=(hyp['momentum'], 0.999), eps=1e-8)), both over the reference's three groups.  Adam keeps its second
        moment in one more flat fp32 buffer: 4 bytes per parameter element (31 MB for s/PSP, 94 MB for m/Lab).
        ema: a utils.torch_utils.ModelEMA of this model (built before or after the Trainer), updated on the main stream right after every
        optimizer step, when both passes have joined and the seg pass's deferred BatchNorm statistics are applied.
        quad: the reference's --quad.  Det batches come from utils.datasets.collate_quad: batch_size // 4 images of twice the loader's
        height and width, and the det loss is multiplied by 4 (train.py:368-369).  The reserved det plans (multi_scale / det_shapes) are
        for batch_size // 4 images at the doubled shapes, with multi_scale every size it can draw from them.  The seg pass and its
        batch_size factor are unchanged (train.py:385).  The reference's loop skips a det batch of one image (train.py:338), so with quad
        a per-GPU batch_size below 8 never trains; the Trainer steps whatever it is given.
        seg_loss: None (SegmentationLosses, as the reference's default), a utils.loss.OhemCELoss, a SegmentationLosses with `weight` set
        (n_segcls class weights: the class-weighted CE of train.py:269-282) or a utils.loss.SegFocalLoss (train_custom.py:284), multiplied
        by batch_size * seggain like the default (train.py:385-391).  On a plain head with 19 or 32 classes it runs in the fused upsample +
        CE kernels; on any other head through autograd on the model's full-resolution outputs, in the library's loss kernels.  The class
        weights are uploaded once, here.  ValueError for a loss that does not fit: an aux that does not match the head (aux=True, and
        aux_num=2 for SegmentationLosses, for BiSe's three outputs only), SegFocalLoss on BiSe (it has no aux), a SegFocalLoss reduction
        other than 'mean', a weight vector whose length is not n_segcls, an ignore_index other than -1, and SegmentationLosses without
        weight (the default: pass seg_loss=None)."""
        if optimizer not in OPTIMIZER_STATE:
            raise ValueError(f"optimizer must be 'sgd' or 'adam', got {optimizer!r}")
        if quad and batch_size < 4:
            raise ValueError(f"quad: a batch of {batch_size} images has no quad (collate_fn4 needs at least 4)")
        if seg_loss is not None and not isinstance(seg_loss, (OhemCELoss, SegmentationLosses, SegFocalLoss)):
            raise ValueError("seg_loss must be None or a utils.loss.OhemCELoss, SegmentationLosses(weight=...) or SegFocalLoss, got "
                             f"{type(seg_loss).__name__}")
        n_seg_outputs = 3 if type(model.model[-2]).__name__ == "SegMaskBiSe" else 1
        if isinstance(seg_loss, OhemCELoss) and seg_loss.aux != (n_seg_outputs == 3):
            raise ValueError(f"OhemCELoss(aux={seg_loss.aux}) does not fit a seg head with {n_seg_outputs} output(s): aux=True is for "
                             "the BiSe head's [out, aux16, aux32]")
        seg_weight = _check_weighted_seg_loss(seg_loss, n_seg_outputs, model.model[-2].c_out)
        assert next(model.parameters()).is_cuda, "model.cuda() first"
        self.model, self.hyp, self.batch_size = model, hyp, batch_size
        self.world_size, self.rank, self.accumulate, self.pg = world_size, rank, accumulate, process_group
        self.detgain, self.seggain = detgain, seggain          # train.py:290
        self.quad = bool(quad)
        model.hyp, model.gr = hyp, getattr(model, "gr", 1.0)
        model.train()
        # detection loss forward + backward as four launches of the library (csrc/detloss.cu) instead of ~760 torch kernels.  Focal loss /
        # positive weights / autobalance take the torch formulation (compute_loss), replayed as one captured CUDA graph (_det_graph)
        self._fused_det = FusedComputeLoss(model)
        self.compute_loss = self._fused_det.ref
        self.n_seg_outputs = n_seg_outputs
        # BiSe returns [out, aux16, aux32]: loss1 + 1.5*aux_weight*loss2 + 0.5*aux_weight*loss3 (reference train.py:387-388, utils/loss.py:239-244)
        self.compute_seg_loss = SegmentationLosses(ignore_index=-1, aux=self.n_seg_outputs == 3, aux_num=2)
        self.ohem = seg_loss if isinstance(seg_loss, OhemCELoss) else None     # an OhemCELoss in place of compute_seg_loss, or None
        # the class-weighted CE / focal loss in place of compute_seg_loss (SegFocalLoss with gamma = 0 is the weighted CE): its weights,
        # uploaded once, and gamma; None for the other losses
        self.seg_wf = None
        if isinstance(seg_loss, (SegmentationLosses, SegFocalLoss)):
            gamma = seg_loss.gamma if isinstance(seg_loss, SegFocalLoss) else 0.0
            w = None if seg_weight is None else seg_weight.detach().to(device=next(model.parameters()).device, dtype=torch.float32).contiguous()
            aux_weight = float(seg_loss.aux_weight) if isinstance(seg_loss, SegmentationLosses) and seg_loss.aux else None
            self.seg_wf = (w, float(gamma), aux_weight)
        # seg CE + x8 upsample forward / backward in one kernel, no full-resolution logits: plain heads with 19 (Cityscapes) or 32 classes,
        # the instantiations in csrc/train.cu; other heads take autograd
        self.fused_seg = self.n_seg_outputs == 1 and model.model[-2].c_out in (19, 32)
        self.optimizer = optimizer
        self.ema = ema
        self.flat = FlatState(model, adam=optimizer == "adam")
        dev = self.flat.param.device
        self.lr = [hyp["lr0"]] * 3
        self.momentum = hyp["momentum"]
        self.betas, self.eps = (hyp["momentum"], 0.999), 1e-8                # train.py:129; used by "adam" only
        self.param_groups = default_param_groups(optimizer, hyp)            # every other key of the groups, for state_dict()
        self.wd = [g["weight_decay"] for g in self.param_groups]             # 0, hyp['weight_decay'], 0
        # optimiser steps taken that were not skipped, counted on the device (Adam's bias corrections; whether torch would have state)
        self.steps = torch.zeros((), dtype=torch.int32, device=dev)
        self.scale = torch.full((), float(init_scale), device=dev)
        self.growth_tracker = torch.zeros((), dtype=torch.int32, device=dev)
        self.growth_interval = growth_interval
        self.found_inf = torch.zeros(1, dtype=torch.int32, device=dev)
        self.inv_scale = torch.ones((), device=dev)
        self.ni = 0
        self._det_graphs = {}
        # SyncBatchNorm layers that synchronise (torch.distributed initialised, more than one rank): the train plans exchange their
        # statistics over NCCL, and the two passes run one after the other, so that every rank issues the exchanges in one order on one
        # communicator (_passes_concurrent would interleave two streams of them differently on each rank)
        self.sync_bn = bn_sync_group([m for m in model.modules() if isinstance(m, nn.modules.batchnorm._BatchNorm)]) is not None
        self._s_seg = torch.cuda.Stream() if self.fused_seg else None          # the seg pass of _passes_concurrent
        self._ev_detfwd, self._ev_start, self._ev_seg = torch.cuda.Event(), torch.cuda.Event(), torch.cuda.Event()
        self.multi_scale = multi_scale
        self.det_shapes = None if det_shapes is None else sorted({(int(h), int(w)) for h, w in det_shapes})
        self._ms_batches = set()
        if multi_scale is not None or det_shapes is not None:
            self._reserve_det(batch_size // 4 if self.quad else batch_size)

    def det_train_shapes(self):
        """every (H, W) the det lane's shared workspace holds plans for"""
        ms = self.multi_scale
        base = self.det_shapes if self.det_shapes is not None else [(ms.imgsz, ms.imgsz)]
        if self.quad:
            base = [(2 * h, 2 * w) for h, w in base]
        return base if ms is None else sorted({hw for shape in base for hw in ms.shapes(shape)})

    def _reserve_det(self, B):
        self.model.engine().reserve_train_shapes(B, self.det_train_shapes(), lane=0)
        self._ms_batches.add(B)

    def set_lr(self, lr_bn, lr_weight, lr_bias):
        self.lr = [float(lr_bn), float(lr_weight), float(lr_bias)]

    def set_momentum(self, m):
        if self.optimizer == "adam":
            raise ValueError("Adam's groups have no 'momentum': the reference's warm-up (train.py:351-352) leaves beta1 at hyp['momentum']")
        self.momentum = float(m)

    # ---- optimiser state in torch's format (reference checkpoints' ckpt['optimizer']) ----------------------------------------------
    def _state_buffers(self):
        f = self.flat
        return {"momentum_buffer": f.momentum} if self.optimizer == "sgd" else {"exp_avg": f.momentum, "exp_avg_sq": f.exp_avg_sq}

    def state_dict(self):
        """`optimizer.state_dict()` of the reference's optimizer (SGD or --adam) over this model, as its checkpoints hold it; state tensors
        are CUDA copies.  Synchronises with the device (reads the step counter)."""
        key = {"momentum": self.momentum} if self.optimizer == "sgd" else {"betas": self.betas, "eps": self.eps}
        groups = [dict(g, lr=lr, weight_decay=wd, **key) for g, lr, wd in zip(self.param_groups, self.lr, self.wd)]
        return optimizer_state_dict(self.model, self.optimizer, groups, int(self.steps), self._state_buffers())

    def load_state_dict(self, sd):
        """restores a state_dict() of this class or a reference checkpoint's ckpt['optimizer'] (tensors on any device): the moments, the step
        count and each group's lr, weight decay and momentum / betas.  The loss scale is not touched (the reference does not save its
        GradScaler).  ValueError when the dict does not fit this optimizer and model (see optimizer_state_from_dict)."""
        groups, steps, bufs = optimizer_state_from_dict(self.model, self.optimizer, sd, device=self.flat.param.device)
        for name, dst in self._state_buffers().items():
            dst.copy_(bufs[name])
        self.steps.fill_(steps)
        self.param_groups = groups
        self.lr = [g["lr"] for g in groups]
        self.wd = [g["weight_decay"] for g in groups]
        if self.optimizer == "sgd":
            self.momentum = groups[0]["momentum"]
        else:
            self.betas, self.eps = groups[0]["betas"], groups[0]["eps"]

    # ---- the two passes --------------------------------------------------------------------------------------------
    def _det_loss_scaled(self, p, targets):
        loss, items = self.compute_loss(p, targets)
        if self.rank != -1:
            loss = loss * self.world_size                                         # train.py:367-368
        if self.quad:
            loss = loss * 4.                                                      # train.py:368-369
        return loss * self.detgain * self.scale, items

    def det_mult(self):
        """the fused det loss's multiplier: world_size under DDP, 4 with quad, detgain (train.py:367-370 and :290)"""
        return (self.world_size if self.rank != -1 else 1) * (4. if self.quad else 1) * self.detgain

    def _det_graph(self, shapes, nt_pad, dev):
        """static inputs (head outputs, padded targets) -> static outputs (d loss / d head outputs, loss items), captured once per
        (grid shapes, padded target count).  Padding rows are all-zero targets: zero width/height never matches an anchor."""
        # every scalar the captured kernels bake in is part of the key: changing hyp / gains / gr / autobalance state re-captures
        cl = self.compute_loss
        key = (tuple(shapes), nt_pad, self.detgain, self.world_size, self.rank, self.quad, float(getattr(self.model, "gr", 1.0)),
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
        eng = self.model.engine()
        if self._fused_det.supported:
            raws, _, plan = eng.train_forward(imgs, want_seg=False)
            self._ev_detfwd.record(torch.cuda.current_stream())
            grads, items = self._fused_det(raws, targets, mult=self.det_mult(), scale=self.scale)
            eng.train_backward(plan, grads, None)
            return items
        # the torch formulation: forward + autograd backward (~700 tiny kernels) replayed as ONE CUDA graph
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

    def _seg_ce_backward(self, plan, segtargets):
        f = self.batch_size * self.seggain                                                   # train.py:385-391
        eng = self.model.engine()
        if self.ohem is not None:
            return eng.train_backward_seg_ohem(plan, segtargets, self.ohem.thresh_t, factor=f, scale=self.scale,
                                               ignore_index=self.ohem.ignore_index) * f
        if self.seg_wf is not None:
            w, gamma, _ = self.seg_wf
            return eng.train_backward_seg_loss(plan, segtargets, w, gamma, factor=f, scale=self.scale) * f
        return eng.train_backward_seg_ce(plan, segtargets, factor=f, scale=self.scale) * f

    def backward_seg(self, segimgs, segtargets):
        if self.fused_seg:
            _, _, plan = self.model.engine().train_forward(segimgs, want_seg=False)
            return self._seg_ce_backward(plan, segtargets)
        pred = self.model(segimgs)
        if self.ohem is not None:
            loss = self.ohem(pred[1], segtargets)                   # the reference's call: the output, or the list of BiSe's three
        elif self.seg_wf is not None:
            w, gamma, aux_weight = self.seg_wf
            outs = pred[1] if isinstance(pred[1], list) else [pred[1]]
            parts = [seg_focal_loss(o, segtargets, w, gamma) for o in outs]
            # BiSe: loss1 + 1.5 * aux_weight * loss2 + 0.5 * aux_weight * loss3 (reference utils/loss.py:239-244)
            loss = parts[0] if len(parts) == 1 else parts[0] + aux_weight * 1.5 * parts[1] + aux_weight / 2.0 * parts[2]
        else:
            outs = pred[1] if isinstance(pred[1], list) else [pred[1]]
            loss = self.compute_seg_loss(*outs, segtargets)
        segloss = loss * self.batch_size * self.seggain                                     # train.py:385-391
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
        wd = (C.c_float * 3)(*self.wd)
        if self.optimizer == "adam":
            lr = (C.c_double * 3)(*self.lr)
            _lib.check(L.myolo_adam_step(_lib.ptr(f.param), _lib.ptr(f.grad), _lib.ptr(f.momentum), _lib.ptr(f.exp_avg_sq), _lib.ptr(f.group),
                                         f.n, lr, wd, 3, float(self.betas[0]), float(self.betas[1]), float(self.eps), _lib.ptr(self.steps),
                                         _lib.ptr(self.inv_scale), _lib.ptr(self.found_inf), 1, sp))
        else:
            lr = (C.c_float * 3)(*self.lr)
            _lib.check(L.myolo_sgd_step(_lib.ptr(f.param), _lib.ptr(f.grad), _lib.ptr(f.momentum), _lib.ptr(f.group), f.n, lr, wd, 3,
                                        float(self.momentum), 1, _lib.ptr(self.inv_scale), _lib.ptr(self.found_inf), 1, sp))
        # amp.GradScaler.update: halve on overflow, double after growth_interval clean steps (device-side, no host sync)
        bad = self.found_inf[0] != 0
        self.steps.add_((~bad).to(torch.int32))                               # after the launch: every block read the old count
        tracker = torch.where(bad, torch.zeros_like(self.growth_tracker), self.growth_tracker + 1)
        grow = tracker >= self.growth_interval
        self.scale.copy_(torch.where(bad, self.scale * 0.5, torch.where(grow, self.scale * 2.0, self.scale)))   # in place: graphs read it
        self.growth_tracker.copy_(torch.where(grow, torch.zeros_like(tracker), tracker))
        self.model.invalidate_weights()            # the step wrote the parameters through raw pointers
        if self.ema is not None:
            self.ema.update(self.model)            # train.py:401: every step, a skipped one too (reads parameters and BN buffers)

    def _passes_sequential(self, imgs, targets, segimgs, segtargets):
        return self.backward_det(imgs, targets), self.backward_seg(segimgs, segtargets)

    def _passes_concurrent(self, imgs, targets, segimgs, segtargets):
        """the seg pass on its own train plan (lane 1) and stream.  At 4 images per pass every kernel is small and each pass alone is a
        latency-bound chain that leaves most of the 132 SMs idle, so both forwards start together.  The seg plan defers its BatchNorm
        running statistics and applies them after the det forward, i.e. in the reference's order (train.py:364 det batch, :385 seg batch);
        the two backwards overlap too, their parameter gradients add up atomically in the one flat buffer."""
        eng = self.model.engine()
        main = torch.cuda.current_stream()
        self._ev_start.record(main)
        with torch.cuda.stream(self._s_seg):
            self._s_seg.wait_event(self._ev_start)
            B, _, H, W = segimgs.shape
            plan = eng.train_plan_for(B, H, W, lane=1)
            eng.set_defer_running(plan)
            eng.train_forward(segimgs, want_seg=False, lane=1)
        items = self.backward_det(imgs, targets)                 # records _ev_detfwd right after the det forward
        with torch.cuda.stream(self._s_seg):
            self._s_seg.wait_event(self._ev_detfwd)
            eng.apply_running(plan)
            segloss = self._seg_ce_backward(plan, segtargets)
            self._ev_seg.record(self._s_seg)
        main.wait_event(self._ev_seg)
        segimgs.record_stream(self._s_seg); segtargets.record_stream(self._s_seg)
        return items, segloss

    def step(self, imgs, targets, segimgs, segtargets, ni=None):
        """one iteration (train.py:363-401).  Returns (det loss items [lbox,lobj,lcls,loss], seg loss) as device tensors.
        ni: the reference's iteration number (train.py:341, which also counts skipped batches); when given, the optimizer steps when
        ni % self.accumulate == 0 (train.py:396), else every `accumulate` calls of this method."""
        if self._ms_batches and imgs.shape[0] not in self._ms_batches:
            self._reserve_det(int(imgs.shape[0]))               # host plans only: the shared workspace is already there
        # autograd's seg pass runs Model.forward: lane 0.  Synchronised BatchNorm: one stream of collectives, det pass then seg pass
        passes = self._passes_concurrent if self.fused_seg and not self.sync_bn else self._passes_sequential
        items, segloss = passes(imgs, targets, segimgs, segtargets)
        self.ni += 1
        if (self.ni if ni is None else ni) % self.accumulate == 0:
            self.optimizer_step()
        return items, segloss


# ---- the epoch loop (reference train.py:44-543) ---------------------------------------------------------------------------------------
NBS = 64                # nominal batch size (train.py:115)
WARMUP_MIN = 800        # least number of warm-up iterations (train.py:260: this fork's 800; upstream YOLOv5 uses 1000)
EMA_ATTRS = ("yaml", "nc", "hyp", "gr", "names", "stride", "class_weights")         # ema.update_attr's include list (train.py:433)

Iteration = collections.namedtuple("Iteration", "ni lr momentum accumulate step")


class LRSchedule:
    """The learning rates, momentum and gradient accumulation of reference train.py, per iteration and per epoch:

        nw = max(round(hyp['warmup_epochs'] * nb), 800)                                  (train.py:260; nb counts det batches)
        while ni <= nw (ni = i + nb * epoch):                                            (train.py:344-352)
            accumulate = max(1, interp(ni, [0, nw], [1, floor(64 / total_batch_size)]).round())
            lr[j]      = interp(ni, [0, nw], [hyp['warmup_bias_lr'] if j == 2 else 0.0, initial_lr[j] * lf(epoch)])
            momentum   = interp(ni, [0, nw], [hyp['warmup_momentum'], hyp['momentum']])  (SGD only: Adam's groups have no 'momentum')
        after each epoch: lr[j] = lr0 * lf(epoch + 1)                                    (LambdaLR.step, train.py:428)

    with lf = one_cycle(1, lrf, epochs), or the linear ramp of --linear-lr (train.py:143-147).  Outside the warm-up every value stays where
    the last warm-up iteration (or the last epoch end) left it; `accumulate` starts at max(round(64 / total_batch_size), 1) (train.py:116),
    which is also what weight decay is scaled for, and the warm-up ends it at floor(64 / total_batch_size).  The floats are numpy's
    float64 interp and torch LambdaLR's `base_lr * lf(epoch)`, computed by the same operations in the same order.

    Resume (start_epoch > 0): pass the checkpoint optimizer's `param_groups`; lr, momentum and initial_lr come from them, as
    optimizer.load_state_dict sets them (train.py:157-158), and the epoch count is extended when fine-tuning past the end (train.py:174-177).
    The cosine lf keeps the epoch count it was built with, the linear one reads the extended count when called, as the reference's
    closure over `epochs` does.

    `iteration(epoch, i)` is called for each batch that trains (not for the batches of one image the loop skips) and returns
    Iteration(ni, (lr_bn, lr_weight, lr_bias), momentum (None for Adam), accumulate, step: whether the optimizer steps).  `step()` is the
    epoch end.  `state_dict()` is the schedule's state: the epoch count, last_epoch, lr, momentum, initial_lr, accumulate."""

    def __init__(self, hyp, epochs, nb, total_batch_size, linear_lr=False, optimizer="sgd", start_epoch=0, param_groups=None, nbs=NBS):
        if optimizer not in OPTIMIZER_STATE:
            raise ValueError(f"optimizer must be 'sgd' or 'adam', got {optimizer!r}")
        if nb < 1:
            raise ValueError(f"an epoch of {nb} det batches has no iteration")
        h = self.hyp = dict(hyp)
        self.nb, self.nbs, self.total_batch_size, self.sgd = int(nb), nbs, total_batch_size, optimizer == "sgd"
        self.epochs = epochs + start_epoch - 1 if start_epoch > 0 and epochs < start_epoch else epochs
        if linear_lr:
            n = self.epochs
            self.lf = lambda x: (1 - x / (n - 1)) * (1.0 - h["lrf"]) + h["lrf"]
        else:
            self.lf = one_cycle(1, h["lrf"], epochs)
        self.nw = max(round(h["warmup_epochs"] * self.nb), WARMUP_MIN)
        self.base_lrs = [h["lr0"]] * 3                       # LambdaLR's, from the groups' lr when it was built: this run's lr0
        self.last_epoch = start_epoch - 1
        self.accumulate = max(round(nbs / total_batch_size), 1)
        if param_groups is None:
            self.initial_lr = list(self.base_lrs)
            self.lr = [b * self.lf(0) for b in self.base_lrs]           # LambdaLR's first step, in its constructor
            self.momentum = h["momentum"] if self.sgd else None
        else:
            if len(param_groups) != 3:
                raise ValueError(f"expected the reference's three parameter groups, got {len(param_groups)}")
            self.initial_lr = [g.get("initial_lr", h["lr0"]) for g in param_groups]
            self.lr = [g["lr"] for g in param_groups]
            self.momentum = param_groups[0]["momentum"] if self.sgd else None

    def iteration(self, epoch, i):
        ni = i + self.nb * epoch
        if ni <= self.nw:
            xi = [0, self.nw]
            self.accumulate = int(max(1, np.interp(ni, xi, [1, math.floor(self.nbs / self.total_batch_size)]).round()))
            self.lr = [float(np.interp(ni, xi, [self.hyp["warmup_bias_lr"] if j == 2 else 0.0, self.initial_lr[j] * self.lf(epoch)]))
                       for j in range(3)]
            if self.sgd:
                self.momentum = float(np.interp(ni, xi, [self.hyp["warmup_momentum"], self.hyp["momentum"]]))
        return Iteration(ni, tuple(self.lr), self.momentum, self.accumulate, ni % self.accumulate == 0)

    def step(self):
        self.last_epoch += 1
        self.lr = [b * self.lf(self.last_epoch) for b in self.base_lrs]

    def state_dict(self):
        return {"epochs": self.epochs, "last_epoch": self.last_epoch, "lr": list(self.lr), "momentum": self.momentum,
                "initial_lr": list(self.initial_lr), "accumulate": self.accumulate}


class DetEpochBatches:
    """`det_batches` for fit: `batches(epoch)` iterates one epoch's det batches as the reference's train loader yields them.

    source: a utils.datasets.DetAugmenter (the square mosaic loader), DetRectLoader (--rect) or ImageWeights (--image-weights); each
    builds the batch of a list of dataset positions.  Positions run 0 .. n-1 in order at rank -1 (the loader has no sampler), and are
    DistributedSampler's (utils.datasets.distributed_positions, seed 0, set_epoch(epoch)) under DDP; a batch is a run of `batch_size`
    of them, the last one partial.  With ImageWeights, `ImageWeights.draw(class_weights, maps, rank, group)` runs when the epoch's
    iterable is made (train.py:305-316), with `maps` the per-class mAP fit stores in `self.maps` after each test() (zeros before).
    quad: each uint8 batch goes through utils.datasets.collate_quad (collate_fn4).  Batches are built when they are asked for, so the
    random draws come in the reference's order when fit zips them with the seg batches."""

    def __init__(self, source, batch_size, rank=-1, world_size=1, quad=False, class_weights=None, group=None, out_dtype=torch.float32):
        from .utils.datasets import ImageWeights
        self.image_weights = isinstance(source, ImageWeights)
        if self.image_weights and class_weights is None:
            raise ValueError("DetEpochBatches: ImageWeights needs the model's class weights (labels_to_class_weights(labels, nc) * nc)")
        self.source, self.batch_size, self.rank, self.world_size = source, int(batch_size), rank, world_size
        self.quad, self.class_weights, self.group, self.out_dtype = bool(quad), class_weights, group, out_dtype
        self.n = source.n
        self.maps = None

    def positions(self, epoch):
        from .utils.datasets import distributed_positions
        return list(range(self.n)) if self.rank == -1 else distributed_positions(self.n, epoch, self.rank, self.world_size)

    def __len__(self):
        n = self.n if self.rank == -1 else math.ceil(self.n / self.world_size)
        return math.ceil(n / self.batch_size)

    def __call__(self, epoch):
        if self.image_weights:
            cw = self.class_weights
            self.source.draw(cw, np.zeros(len(cw)) if self.maps is None else self.maps, self.rank, self.group)
        return self._batches(self.positions(epoch))

    def _batches(self, positions):
        from .utils.datasets import collate_quad
        for k in range(0, len(positions), self.batch_size):
            chunk = positions[k:k + self.batch_size]
            if self.quad:
                yield collate_quad(*self.source(chunk, torch.uint8), out_dtype=self.out_dtype)
            else:
                yield self.source(chunk, self.out_dtype)


class SegEpochBatches:
    """`seg_batches` for fit: one epoch's seg batches from a utils.datasets.SegAugmenter in the order of the reference's
    DataLoader(shuffle=True, drop_last=...) (SegmentationDataset.get_*_loader: drop_last=False for get_citys_loader, True for the
    citysbdd and custom loaders).  The order is torch's own: a DataLoader over range(n) with those settings, iterated by index batches,
    so its RandomSampler draws from torch's default generator exactly when the reference's does (the loader's base seed when the epoch's
    iterator is made, the permutation's seed at its first batch), before the items' ColorJitter draws."""

    def __init__(self, aug, batch_size, drop_last=False, out_dtype=torch.float32):
        self.aug, self.batch_size, self.drop_last, self.out_dtype = aug, int(batch_size), bool(drop_last), out_dtype
        self.n = aug.cache.n

    def __len__(self):
        return self.n // self.batch_size if self.drop_last else math.ceil(self.n / self.batch_size)

    def order(self):
        """the epoch's index batches (an iterator of int64 tensors), made now"""
        return iter(torch.utils.data.DataLoader(range(self.n), batch_size=self.batch_size, shuffle=True, drop_last=self.drop_last))

    def __call__(self, epoch):
        return (self.aug(idx.tolist(), self.out_dtype) for idx in self.order())


class SegValBatches:
    """`segval_loader` for fit and `valloader` for test.seg_validation: the seg validation batches of a utils.datasets.SegAugmenter in the
    order of the reference's DataLoader(shuffle=False, drop_last=False) (SegmentationDataset.get_*_loader with a mode other than
    'train'): items 0 .. n-1 in runs of `batch_size`, the last one partial.  Iterable again for every validation pass; each batch is
    built when it is asked for, so a pass holds one batch at a time.

    mode='val': `aug.val(chunk, crop_size)`, train_citysbdd.py's validation (batch 4, int crop_size 512 over City+BDD sources of
    different sizes).  mode='testval': `aug.testval(chunk)`, that of train.py (batch 4, base_size 1024) and of train_custom.py (batch 1,
    base_size imgsz), at the augmenter's base_size; crop_size is unused, as in the reference.  The items of a testval batch must share
    their source size, as default_collate requires: a batch that does not raises ValueError here, before any batch is built."""

    def __init__(self, aug, batch_size, mode="val", crop_size=None, out_dtype=torch.float32):
        from .utils.datasets import seg_val_crop
        if mode not in ("val", "testval"):
            raise ValueError(f"SegValBatches: mode must be 'val' or 'testval', got {mode!r}")
        if int(batch_size) < 1:
            raise ValueError(f"SegValBatches: batch_size must be positive, got {batch_size}")
        if out_dtype not in (torch.uint8, torch.float16, torch.float32):
            raise ValueError(f"SegValBatches: out_dtype must be uint8, float16 or float32, got {out_dtype}")
        self.aug, self.batch_size, self.mode, self.out_dtype = aug, int(batch_size), mode, out_dtype
        self.n = aug.cache.n
        self.crop_size = seg_val_crop(crop_size) if mode == "val" else crop_size
        if mode == "testval":
            for chunk in self.chunks():
                shapes = sorted({aug.cache.shapes[i] for i in chunk})
                if len(shapes) != 1:
                    raise ValueError(f"SegValBatches: testval batch of items {chunk[0]}..{chunk[-1]} mixes source sizes {shapes}, which "
                                     "default_collate cannot stack (mode='val' crops them to one size)")

    def __len__(self):
        return math.ceil(self.n / self.batch_size)

    def chunks(self):
        """the index batches, in order"""
        return [list(range(k, min(k + self.batch_size, self.n))) for k in range(0, self.n, self.batch_size)]

    def __iter__(self):
        for chunk in self.chunks():
            if self.mode == "val":
                yield self.aug.val(chunk, self.crop_size, self.out_dtype)
            else:
                yield self.aug.testval(chunk, self.out_dtype)


def _unsupported_flags(opt):
    """NotImplementedError naming the first flag of `opt` the loop cannot honour"""
    for name, on in (("bucket", getattr(opt, "bucket", "")), ("entity", getattr(opt, "entity", None)),
                     ("upload_dataset", getattr(opt, "upload_dataset", False)), ("data", isinstance(getattr(opt, "data", None), str))):
        if on:
            raise NotImplementedError(f"fit: --{name} is not built (W&B, gsutil uploads and loading a data yaml are not part of the loop)")


def _load_start(path, model, hyp, opt, device):
    """the checkpoint of train.py:86-95 and :152-177 (this loop's or the reference's): loads its model weights into `model` and returns it"""
    from .models.experimental import load_checkpoint
    ckpt = load_checkpoint(path, map_location=device)
    exclude = ["anchor"] if (getattr(opt, "cfg", "") or hyp.get("anchors")) and not opt.resume else []
    msd = model.state_dict()
    sd = {k: v for k, v in ckpt["model"].float().state_dict().items()
          if k in msd and not any(x in k for x in exclude) and v.shape == msd[k].shape}          # intersect_dicts
    model.load_state_dict(sd, strict=False)
    return ckpt


def fit(model, hyp, opt, det_batches, seg_batches, *, test_loader=None, segval_loader=None, save_dir, ema=None, log_interval=50,
        **trainer_kwargs):
    """The training run of reference train.py:train() (train.py:44-543) over device batches; returns `results` as it does:
    (P, R, mAP@.5, mAP@.5:.95, val box, obj, cls loss) of the last test().

    model: a CUDA models.yolo.Model (fp32) with `names` set, built as train.py:86-98 builds it; hyp: the unscaled hyper-parameters (this
    scales weight decay and the loss gains as train.py:116-117 and :248-251 do).  opt: an argparse.Namespace with the reference's flag
    names: epochs, batch_size (total), img_size ([train, test]), linear_lr, adam, notest, nosave, evolve, multi_scale, quad, single_cls,
    resume, global_rank, world_size, label_smoothing, and `weights` (a .pt to start from, or '') and `cfg` as train.py reads them.
    det_batches(epoch) / seg_batches(epoch): that epoch's iterables of (imgs, targets, ...) and (segimgs, segtargets) device batches,
    with len(det_batches) = nb; DetEpochBatches / SegEpochBatches build them from the device loaders in the reference's order.  Det images
    are float (B, 3, H, W) = uint8 / 255, or uint8 under multi_scale.  test_loader: DetValLoader batches for test.test (None: no test,
    results stay zeros); segval_loader: an iterable of seg validation batches for test.seg_validation, iterated again at every
    validation (SegValBatches, mode='val' or 'testval'; None: mIoU 0).  save_dir: results.txt and
    weights/last.pt, best.pt go there.  ema: a ModelEMA of `model` (built here on rank -1 / 0 when None).  trainer_kwargs go to Trainer
    (seg_loss, process_group, det_shapes, ...).

    Per run: init_seeds(2 + rank); the EMA; the start checkpoint (opt.weights ending in .pt): model weights, optimizer state and
    best_fitness, EMA and its update count, results.txt, start_epoch, and the fine-tune extension of the epoch count; then, when not
    resuming, model.half().float() (train.py:225); the Trainer and the LRSchedule.  Per iteration (train.py:335-410): batches of one
    image are skipped but still counted in `i`; the schedule goes to Trainer.set_lr / set_momentum / accumulate; MultiScale rescales the
    det batch under multi_scale; Trainer.step(..., ni=ni).  The running mean losses stay on the device and are read and printed every
    `log_interval` iterations and at the epoch end only, where the reference formats them every iteration (a host synchronisation per
    step).  Per epoch (train.py:426-500): the schedule's step, ema.update_attr, seg_validation on ema.ema when epoch % 10 == 0 or
    epochs - epoch < 40 (mIoU 0 otherwise), test.test(model=ema.ema) unless notest and always on the final epoch, fitness2 and
    best_fitness, the results.txt line in the reference's format, and last.pt / best.pt with the reference's keys unless nosave (the
    final epoch saves unless evolve).

    Deviations: test() runs with plots=False on the final epoch too (plots are not built); autoanchor (train.py:223-224) is the caller's,
    before fit; no W&B, TensorBoard or --bucket (NotImplementedError), no data yaml (opt.data must not be a path), no strip_optimizer or
    COCO re-test after the last epoch.  Reproducibility: a seeded run's batches equal the reference's only under --workers 0, since
    DataLoader worker processes draw from `random` / `numpy.random` streams of their own; and torch's default generator, which the seg
    order and ColorJitter draw from, has also served the reference's model initialisation before its first epoch."""
    from copy import deepcopy
    from pathlib import Path
    from . import test as _test
    from .utils.metrics import fitness2
    from .utils.torch_utils import ModelEMA

    _unsupported_flags(opt)
    save_dir = Path(save_dir)
    wdir = save_dir / "weights"
    wdir.mkdir(parents=True, exist_ok=True)
    last, best, results_file = wdir / "last.pt", wdir / "best.pt", save_dir / "results.txt"
    rank, world_size = getattr(opt, "global_rank", -1), getattr(opt, "world_size", 1)
    total_batch_size = opt.batch_size
    batch_size = total_batch_size // world_size if rank != -1 else total_batch_size
    epochs = opt.epochs
    device = next(model.parameters()).device
    init_seeds(2 + rank)

    det = model.model[-1]
    nc = 1 if opt.single_cls else int(det.nc)
    nl = det.nl
    gs = max(int(model.stride.max()), 32)
    imgsz, imgsz_test = (list(opt.img_size) * 2)[:2]
    if imgsz % gs or imgsz_test % gs:
        raise ValueError(f"image sizes {imgsz}, {imgsz_test} must be multiples of the grid size {gs}")

    weights = getattr(opt, "weights", "") or ""
    if isinstance(opt.resume, str):
        weights = opt.resume
    ckpt = _load_start(weights, model, hyp, opt, device) if weights.endswith(".pt") else None
    if ema is None and rank in (-1, 0):
        ema = ModelEMA(model)                                                      # train.py:151
    start_epoch, best_fitness = 0, 0.0
    if ckpt is not None:
        if ckpt.get("optimizer") is not None:
            best_fitness = ckpt["best_fitness"]
        if ema is not None and ckpt.get("ema") is not None:
            ema.ema.load_state_dict(ckpt["ema"].float().state_dict())
            ema.updates = ckpt["updates"]
        if ckpt.get("training_results") is not None:
            results_file.write_text(ckpt["training_results"])
        start_epoch = ckpt["epoch"] + 1
        if opt.resume and start_epoch <= 0:
            raise ValueError(f"{weights} training to {epochs} epochs is finished, nothing to resume")
    if rank in (-1, 0) and not opt.resume:
        model.half().float()                                                       # train.py:225: pre-reduce anchor precision

    h = scale_hyp(hyp, nl=nl, nc=nc, imgsz=imgsz, total_batch_size=total_batch_size, nbs=NBS, label_smoothing=opt.label_smoothing)
    nb = len(det_batches)
    optimizer = "adam" if opt.adam else "sgd"
    groups = ckpt["optimizer"]["param_groups"] if ckpt is not None and ckpt.get("optimizer") is not None else None
    sched = LRSchedule(hyp, epochs, nb, total_batch_size, linear_lr=opt.linear_lr, optimizer=optimizer, start_epoch=start_epoch,
                       param_groups=groups)
    epochs = sched.epochs
    multi_scale = MultiScale(imgsz, gs) if opt.multi_scale else None
    tr = Trainer(model, h, batch_size, world_size=world_size, rank=rank, accumulate=sched.accumulate, optimizer=optimizer, ema=ema,
                 quad=opt.quad, multi_scale=multi_scale, **trainer_kwargs)
    if groups is not None:
        tr.load_state_dict(ckpt["optimizer"])
    del ckpt
    model.nc = nc
    cl = tr.compute_loss

    results = (0, 0, 0, 0, 0, 0, 0)
    maps = np.zeros(nc)
    for epoch in range(start_epoch, epochs):
        mIoU = 0
        model.train()
        mloss = torch.zeros(4, device=device)
        msegloss = torch.zeros(1, device=device)
        s = None
        for (i, det_batch), (_, seg_batch) in zip(enumerate(det_batches(epoch)), enumerate(seg_batches(epoch))):
            imgs, targets = det_batch[0], det_batch[1]
            segimgs, segtargets = seg_batch[0], seg_batch[1]
            if len(imgs) == 1 or len(segimgs) == 1:                               # train.py:338-339
                continue
            it = sched.iteration(epoch, i)
            tr.set_lr(*it.lr)
            if it.momentum is not None:
                tr.set_momentum(it.momentum)
            tr.accumulate = it.accumulate
            if multi_scale is not None:
                imgs = multi_scale(imgs)
            elif not imgs.is_floating_point():
                raise ValueError("fit: det images must be float (uint8 / 255) unless multi_scale converts them")
            loss_items, segloss = tr.step(imgs, targets, segimgs, segtargets, ni=it.ni)
            if rank in (-1, 0):
                mloss = (mloss * i + loss_items) / (i + 1)
                msegloss = (msegloss * i + segloss.detach() / total_batch_size) / (i + 1)
                s = (epoch, targets.shape[0], imgs.shape[-1])
                if (i + 1) % log_interval == 0:
                    print(_progress(epoch, epochs, mloss, msegloss, *s[1:]), flush=True)
        sched.step()                                                               # train.py:428
        tr.set_lr(*sched.lr)

        if rank in (-1, 0):
            if s is None:
                raise ValueError(f"epoch {epoch} trained no batch")
            line = _progress(epoch, epochs, mloss, msegloss, *s[1:])
            print(line, flush=True)
            ema.update_attr(model, include=EMA_ATTRS)
            if epoch % 10 == 0 or (epochs - epoch) < 40:
                if segval_loader is not None:
                    mIoU = _test.seg_validation(model=ema.ema, valloader=segval_loader, device=device, n_segcls=model.model[-2].c_out,
                                                half_precision=True)
            final_epoch = epoch + 1 == epochs
            if (not opt.notest or final_epoch) and test_loader is not None:
                results, maps, _ = _test.test({"nc": nc}, batch_size=batch_size * 2, imgsz=imgsz_test, model=ema.ema,
                                              single_cls=opt.single_cls, dataloader=test_loader, save_dir=save_dir,
                                              verbose=nc < 50 and final_epoch, plots=False, compute_loss=cl)
                if hasattr(det_batches, "maps"):
                    det_batches.maps = maps
            with open(results_file, "a") as f:
                f.write(line + "%10.4g" * 7 % results + "\n")                     # train.py:456-457
            fi = fitness2(np.array(results).reshape(1, -1), mIoU)
            if fi > best_fitness:
                best_fitness = fi
            if (not opt.nosave) or (final_epoch and not opt.evolve):
                ckpt = {"epoch": epoch,
                        "best_fitness": best_fitness,
                        "training_results": results_file.read_text(),
                        "model": deepcopy(model).half(),
                        "ema": deepcopy(ema.ema).half(),
                        "updates": ema.updates,
                        "optimizer": tr.state_dict(),
                        "wandb_id": None}
                torch.save(ckpt, last)
                if best_fitness == fi:
                    torch.save(ckpt, best)
                del ckpt
    return results


def _progress(epoch, epochs, mloss, msegloss, n_targets, imgshape):
    """the progress line of train.py:407-409 (reads the device means: a host synchronisation)"""
    mem = "%.3gG" % (torch.cuda.memory_reserved() / 1E9 if torch.cuda.is_available() else 0)
    return ("%10s" * 2 + "%10.4g" * 7) % ("%g/%g" % (epoch, epochs - 1), mem, *mloss.tolist(), *msegloss.tolist(), n_targets, imgshape)


# --evolve's mutation metadata (reference train.py:640-667): key -> (mutation gain 0-1, lower limit, upper limit), in the reference's order
EVOLVE_META = {"lr0": (1, 1e-5, 1e-1), "lrf": (1, 0.01, 1.0), "momentum": (0.3, 0.6, 0.98), "weight_decay": (1, 0.0, 0.001),
               "warmup_epochs": (1, 0.0, 5.0), "warmup_momentum": (1, 0.0, 0.95), "warmup_bias_lr": (1, 0.0, 0.2), "box": (1, 0.02, 0.2),
               "cls": (1, 0.2, 4.0), "cls_pw": (1, 0.5, 2.0), "obj": (1, 0.2, 4.0), "obj_pw": (1, 0.5, 2.0), "iou_t": (0, 0.1, 0.7),
               "anchor_t": (1, 2.0, 8.0), "anchors": (2, 2.0, 10.0), "fl_gamma": (0, 0.0, 2.0), "hsv_h": (1, 0.0, 0.1),
               "hsv_s": (1, 0.0, 0.9), "hsv_v": (1, 0.0, 0.9), "degrees": (1, 0.0, 45.0), "translate": (1, 0.0, 0.9), "scale": (1, 0.0, 0.9),
               "shear": (1, 0.0, 10.0), "perspective": (0, 0.0, 0.001), "flipud": (1, 0.0, 1.0), "fliplr": (0, 0.0, 1.0),
               "mosaic": (1, 0.0, 1.0), "mixup": (1, 0.0, 1.0)}


def choice_py38(n, weights, rng=random):
    """`random.choices(range(n), weights=weights)[0]` as Python 3.8 computes it, the version the reference ran on: one rng.random()
    scaled by the weights' total and a bisection of their running sums up to n - 1.  A total of zero (one earlier result, or tied
    fitness) gives n - 1, where Python 3.9+ raises ValueError; with a positive total both versions give the same index."""
    import bisect
    import itertools
    cum = list(itertools.accumulate(weights))
    if len(cum) != n:
        raise ValueError("The number of weights does not match the population")
    total = cum[-1] + 0.0
    return bisect.bisect(cum, rng.random() * total, 0, n - 1)


def evolve(hyp, opt, train_fn, generations=300, evolve_txt="evolve.txt"):
    """The reference's hyper-parameter evolution (train.py:637-717) around `results = train_fn(hyp.copy(), opt)`, a training run that
    returns the 7 results of `fit` (P, R, mAP@.5, mAP@.5:.95, val box, obj, cls loss).  `hyp` holds exactly the keys of EVOLVE_META, in its
    order (the mutation indexes evolve.txt's columns by hyp's key order), `anchors` included; it is updated in place.

    Per generation: when `evolve_txt` exists (a previous generation, or an earlier run to resume), the parent is drawn from its top
    min(5, n) rows by utils.metrics.fitness with weights fitness - min through the global `random` (choice_py38), and mutated with
    numpy.random seeded from int(time.time()) until a factor differs from 1; then every value is clipped to EVOLVE_META's limits and
    rounded to 5 decimals, train_fn runs, and utils.general.print_mutation appends the result to `evolve_txt` and writes
    save_dir/hyp_evolved.yaml.  Sets opt.notest = opt.nosave = True; DDP (opt.global_rank or opt.local_rank other than -1) is refused.
    Returns the path of hyp_evolved.yaml.  Nothing of a generation stays referenced here once train_fn returns."""
    from pathlib import Path
    from .utils.general import print_mutation
    from .utils.metrics import fitness
    if "anchors" not in hyp:
        raise KeyError("anchors", "--evolve mutates hyp['anchors']: enable the commented line '# anchors: 3' of the hyp file")
    if list(hyp) != list(EVOLVE_META):
        raise ValueError(f"--evolve needs the hyp keys {list(EVOLVE_META)} in this order, got {list(hyp)}")
    if getattr(opt, "global_rank", -1) != -1 or getattr(opt, "local_rank", -1) != -1:
        raise ValueError("DDP mode not implemented for --evolve")
    opt.notest, opt.nosave = True, True
    yaml_file = Path(opt.save_dir) / "hyp_evolved.yaml"
    evolve_txt = Path(evolve_txt)
    g = np.array([m[0] for m in EVOLVE_META.values()])              # gains 0-1
    ng = len(EVOLVE_META)
    for _ in range(generations):
        if evolve_txt.exists():
            x = np.loadtxt(evolve_txt, ndmin=2)
            n = min(5, len(x))                                        # number of previous results to consider
            x = x[np.argsort(-fitness(x))][:n]
            w = fitness(x) - fitness(x).min()
            x = x[choice_py38(n, w)]
            mp, s = 0.8, 0.2                                          # mutation probability, sigma
            npr = np.random
            npr.seed(int(time.time()))
            v = np.ones(ng)
            while all(v == 1):                                        # mutate until a change occurs
                v = (g * (npr.random(ng) < mp) * npr.randn(ng) * npr.random() * s + 1).clip(0.3, 3.0)
            for i, k in enumerate(hyp.keys()):
                hyp[k] = float(x[i + 7] * v[i])
        for k, (_, lo, hi) in EVOLVE_META.items():
            hyp[k] = round(min(max(hyp[k], lo), hi), 5)
        results = train_fn(hyp.copy(), opt)
        print_mutation(hyp.copy(), results, yaml_file, evolve_txt)
    print(f"Hyperparameter evolution complete. Best results saved as: {yaml_file}\n"
          f"Command to train a new model with these hyperparameters: $ python train.py --hyp {yaml_file}")
    return yaml_file
