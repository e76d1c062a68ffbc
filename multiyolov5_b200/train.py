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

Out of scope (the reference's outer loop, not the hot path): data loading, LR schedule / warm-up (call `set_lr` / `set_momentum`),
writing checkpoint files, plotting, DDP buffer broadcast.
"""
import math
import random
import ctypes as C

import torch
import torch.nn as nn

from . import _lib
from .engine import flat_offsets
from .parallel import allreduce_flat_grads, bn_sync_group
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

    def step(self, imgs, targets, segimgs, segtargets):
        """one iteration (train.py:363-401).  Returns (det loss items [lbox,lobj,lcls,loss], seg loss) as device tensors."""
        if self._ms_batches and imgs.shape[0] not in self._ms_batches:
            self._reserve_det(int(imgs.shape[0]))               # host plans only: the shared workspace is already there
        # autograd's seg pass runs Model.forward: lane 0.  Synchronised BatchNorm: one stream of collectives, det pass then seg pass
        passes = self._passes_concurrent if self.fused_seg and not self.sync_bn else self._passes_sequential
        items, segloss = passes(imgs, targets, segimgs, segtargets)
        self.ni += 1
        if self.ni % self.accumulate == 0:
            self.optimizer_step()
        return items, segloss
