"""Step-glue helpers the reference's train.py touches around the hot path (reference utils/torch_utils.py)."""
import math
from copy import deepcopy

import torch

from .. import _lib


def scale_img_shapes(h, w, ratio=1.0, same_shape=False, gs=32):
    """((resized h, w), (output h, w)) of reference utils/torch_utils.py:248-258 scale_img, with its host arithmetic: int(h * ratio) for
    the resize, math.ceil(h * ratio / gs) * gs for the padded output unless same_shape keeps (h, w).  ratio 1.0 returns the image as is."""
    if ratio == 1.0:
        return (h, w), (h, w)
    s = (int(h * ratio), int(w * ratio))
    if not same_shape:
        h, w = [math.ceil(x * ratio / gs) * gs for x in (h, w)]
    return s, (h, w)


TTA_SCALES, TTA_FLIPS = (1, 0.83, 0.67), (False, True, False)      # reference models/yolo.py:276-277: flips None, 3 (left-right), None


def tta_passes(h, w, gs=32):
    """[(scale, left-right flip, (resized h, w), (input h, w))] of the three passes of test-time augmentation on an (h, w) input"""
    return [(si, fi) + scale_img_shapes(h, w, si, gs=gs) for si, fi in zip(TTA_SCALES, TTA_FLIPS)]


def scale_img(img, ratio=1.0, same_shape=False, gs=32, flip_lr=False):
    """reference utils/torch_utils.py:248-258 on the device (myolo_scale_img, one launch): F.interpolate(img, bilinear,
    align_corners=False) to int(h * ratio) x int(w * ratio), then F.pad on the right and bottom with 0.447 to a multiple of gs (or back
    to (h, w) with same_shape).  flip_lr=True scales img.flip(3) instead.  img: (B, C, H, W) fp16 or fp32 CUDA; ratio 1.0 without
    flip_lr returns img itself, as the reference does."""
    if not img.is_cuda:
        raise _lib.MyoloError("scale_img needs a CUDA tensor: multiyolov5_b200 has no CPU path")
    if img.dtype not in (torch.float16, torch.float32):
        raise TypeError(f"scale_img takes fp16 or fp32 images, not {img.dtype}")
    if ratio == 1.0 and not flip_lr:
        return img
    h, w = img.shape[2:]
    (ho, wo), (hp, wp) = scale_img_shapes(h, w, ratio, same_shape, gs)
    img = img.contiguous()
    out = torch.empty((img.shape[0], img.shape[1], hp, wp), dtype=img.dtype, device=img.device)
    pad = float(torch.tensor(0.447, dtype=img.dtype))          # the value F.pad fills in: 0.447 rounded to the image's dtype
    _lib.check(_lib.lib().myolo_scale_img(_lib.ptr(img), _lib.torch_dtype_code(img.dtype), img.shape[0], img.shape[1], h, w, _lib.ptr(out),
                                          ho, wo, hp, wp, int(flip_lr), pad, _lib.stream_ptr()))
    return out


def is_parallel(model):
    return type(model) in (torch.nn.parallel.DataParallel, torch.nn.parallel.DistributedDataParallel)


def ema_entries(ema_model, model):
    """[(key, EMA tensor, source tensor)] of the entries ModelEMA.update averages: every floating-point entry of the EMA's state_dict, in
    its order (num_batches_tracked and other integer entries are left alone, as in the reference).  Raises ValueError when an entry has no
    counterpart in `model`, the counterpart is not fp32 or has another shape, an EMA entry is neither fp32 nor fp16, a tensor is not
    contiguous, or the two live on different devices."""
    msd = model.state_dict()
    out = []
    for k, v in ema_model.state_dict().items():
        if not v.dtype.is_floating_point:
            continue
        m = msd.get(k)
        if m is None:
            raise ValueError(f"EMA entry {k!r} has no counterpart in the model")
        if m.dtype != torch.float32:
            raise ValueError(f"EMA source {k!r} is {m.dtype}: the model being averaged keeps fp32 entries")
        if v.dtype not in (torch.float32, torch.float16):
            raise ValueError(f"EMA entry {k!r} is {v.dtype}: the device EMA averages into fp32 or fp16")
        if tuple(v.shape) != tuple(m.shape):
            raise ValueError(f"EMA entry {k!r} has shape {tuple(v.shape)}, the model's has {tuple(m.shape)}")
        if v.device != m.device:
            raise ValueError(f"EMA entry {k!r} is on {v.device}, the model's on {m.device}")
        if not (v.is_contiguous() and m.is_contiguous()):
            raise ValueError(f"EMA entry {k!r}: non-contiguous tensors are not averaged")
        out.append((k, v, m.detach()))
    return out


def ema_chunks(segments, chunk=_lib.EMA_CHUNK):
    """segments: [(ema address, source address, n, dtype code _lib.F32 / _lib.F16)] -> the myolo_ema_update work table as tuples of the same
    form: each segment cut at multiples of `chunk` elements (a multiple of 4, so every piece keeps its segment's 16-byte alignment).
    Empty segments give no chunk."""
    assert chunk % 4 == 0 and chunk > 0
    out = []
    for ema, src, n, dt in segments:
        es = 4 if dt == _lib.F32 else 2
        for o in range(0, n, chunk):
            out.append((ema + o * es, src + o * 4, min(chunk, n - o), dt))
    return out


def _tensor_epoch(m):
    return getattr(m, "_tensor_epoch", 0)


class ModelEMA:
    """reference utils/torch_utils.py:270-304: exponential moving average of everything in the state_dict (parameters AND BN
    buffers), decay ramped by the update count.

    On CUDA one update is one launch (myolo_ema_update) over a device table of every floating-point entry, bit-identical with the
    reference's `v *= d; v += (1. - d) * msd[k]` in fp32 and, after the reference's `ema.half()` in validation, in fp16.  The table is
    built on the first update and rebuilt only when a pointer or dtype in it may have changed: the EMA or the model went through `_apply`
    (.half(), .float(), .to()) or load_state_dict, or the Trainer moved the model's parameters into its flat buffers.
    On the CPU the average is ONE multi-tensor lerp over all floating-point entries (torch's foreach rounding)."""

    def __init__(self, model, decay=0.9999, updates=0):
        self.ema = deepcopy(model.module if is_parallel(model) else model).eval()   # Model.__getstate__ drops the compiled plans
        self.updates = updates
        self.decay = lambda x: decay * (1 - math.exp(-x / 2000))
        for p in self.ema.parameters():
            p.requires_grad_(False)
        self._table = None

    def __getstate__(self):
        d = dict(self.__dict__)
        d["_table"] = None            # raw device pointers into this EMA: a copy builds its own
        return d

    def table(self, model):
        """(device chunk table, number of chunks) for averaging `model` (the training model, unwrapped) into the EMA; built when needed.
        It is reused while both modules and their pointer epochs (models.yolo.Model.tensors_moved) are the same and, as a cheap guard
        against `p.data = ...`, the first and last parameter of each side still have the addresses they had when it was built."""
        key = (id(self.ema), _tensor_epoch(self.ema), id(model), _tensor_epoch(model))
        t = getattr(self, "_table", None)
        if t is not None and t[0] == key and all(p.data_ptr() == a for p, a in t[3]):
            return t[1], t[2]
        entries = ema_entries(self.ema, model)
        segs = [(v.data_ptr(), s.data_ptr(), v.numel(), _lib.torch_dtype_code(v.dtype)) for _, v, s in entries]
        chunks = ema_chunks(segs)
        if not chunks:
            raise ValueError("ModelEMA: the model has no floating-point entries to average")
        arr = (_lib.EmaChunk * len(chunks))(*[_lib.EmaChunk(*c) for c in chunks])
        host = torch.frombuffer(bytearray(arr), dtype=torch.uint8).pin_memory()
        dev = host.to(entries[0][1].device, non_blocking=True)
        guard = []
        for mod in (self.ema, model):
            ps = list(mod.parameters())
            guard += [(p, p.data_ptr()) for p in ps[:1] + ps[-1:]]
        # the entries stay referenced with the table: memory it points into is not handed out again while it may be used
        self._table = (key, dev, len(chunks), guard, entries)
        return dev, len(chunks)

    def update(self, model):
        m = model.module if is_parallel(model) else model
        with torch.no_grad():
            self.updates += 1
            d = self.decay(self.updates)
            p0 = next(self.ema.parameters(), None)
            if p0 is not None and p0.is_cuda:
                table, n = self.table(m)
                _lib.check(_lib.lib().myolo_ema_update(_lib.ptr(table), n, d, _lib.stream_ptr()))
            else:
                msd = m.state_dict()
                mine, theirs = [], []
                for k, v in self.ema.state_dict().items():
                    if v.dtype.is_floating_point:
                        mine.append(v)
                        theirs.append(msd[k].detach())
                torch._foreach_mul_(mine, d)
                torch._foreach_add_(mine, theirs, alpha=1.0 - d)
        if hasattr(self.ema, "invalidate_weights"):
            self.ema.invalidate_weights()      # the EMA copy's packed fp16 weights are stale now

    def update_attr(self, model, include=(), exclude=("process_group", "reducer")):
        for k, v in model.__dict__.items():
            if (len(include) and k not in include) or k.startswith("_") or k in exclude:
                continue
            setattr(self.ema, k, v)
