"""Checkpoint loading behind the reference's names (reference models/experimental.py:95-134).

`attempt_load(weights)` accepts what the reference's `train.py:482-494` writes: a dict whose 'model' / 'ema' entry is a whole pickled
`nn.Module` in half precision.  Checkpoints written by the REFERENCE name its classes (`models.yolo.Model`, `models.common.Conv`, ...);
they are resolved to this package's parameter shells while unpickling (same sub-module names -> same `state_dict()` keys), and the few
constructor arguments the reference does not keep as attributes are recovered from the sub-modules (`_compat_fixup`).
"""
import pickle

import torch
import torch.nn as nn

from . import common as _common
from . import yolo as _yolo

_REMAP = {"models.yolo": _yolo, "models.common": _common, "models.experimental": None}


class _RefUnpickler(pickle.Unpickler):
    """resolves the reference's module paths to this package (only classes that exist here; anything else is an error, not a guess)"""

    def find_class(self, module, name):
        if module in _REMAP:
            mod = _REMAP[module] or __import__(__name__, fromlist=["x"])
            if not hasattr(mod, name):
                raise pickle.UnpicklingError(f"checkpoint needs {module}.{name}, which is not on the *_city_seg hot path (SURVEY.md section 8)")
            return getattr(mod, name)
        return super().find_class(module, name)


class _RefPickleModule:
    """`pickle_module` for torch.load"""
    __name__ = "multiyolov5_b200.models.experimental._RefPickleModule"
    Unpickler = _RefUnpickler
    load = staticmethod(lambda f, **k: _RefUnpickler(f, **k).load())
    loads = staticmethod(pickle.loads)
    dumps = staticmethod(pickle.dumps)
    dump = staticmethod(pickle.dump)
    HIGHEST_PROTOCOL = pickle.HIGHEST_PROTOCOL
    PickleError, UnpicklingError, PicklingError = pickle.PickleError, pickle.UnpicklingError, pickle.PicklingError


def load_checkpoint(path, map_location=None):
    """torch.load of a reference-style checkpoint dict (whole pickled modules -> weights_only=False) with the class remap"""
    return torch.load(path, map_location=map_location, weights_only=False, pickle_module=_RefPickleModule)


def _compat_fixup(model):
    """attributes the planner reads that the reference's modules do not store (they are constructor arguments there)"""
    for m in model.modules():
        d = m.__dict__
        if isinstance(m, _common.SPP) and "k" not in d:
            m.k = tuple(int(p.kernel_size) for p in m.m)
        elif isinstance(m, _common.PyramidPooling) and "k" not in d:
            m.k = tuple(int(p.output_size if isinstance(p.output_size, int) else p.output_size[0]) for p in (m.pool1, m.pool2, m.pool3, m.pool4))
        elif isinstance(m, _common.RFB2) and "d" not in d:
            m.d = (int(m.branch1[0].dilation[0]), int(m.branch2[0].dilation[0]))
        elif isinstance(m, _common.ASPP) and "d" not in d:
            m.d = tuple(int(b[0].dilation[0]) for b in (m.branch1, m.branch2, m.branch3))
        elif isinstance(m, _common.FFM) and "k" not in d:
            m.k = int(m.convblk.conv.kernel_size[0])
        elif isinstance(m, _yolo.SegMaskPSP) and "c_hid" not in d:
            m.c_hid = int(m.m8[0].conv.out_channels)
        elif isinstance(m, _yolo.SegMaskLab) and "c_hid" not in d:
            m.c_hid = int(m.decoder[1].conv.out_channels)
        elif isinstance(m, _yolo.SegMaskLab) and "c_detail" not in d:
            m.c_detail = int(m.detail[0].conv.in_channels)
        if isinstance(m, nn.BatchNorm2d):   # eps / momentum are plain attributes and travel with the pickle; nothing to do
            pass
    if isinstance(model, _yolo.Model):
        object.__setattr__(model, "_engine", None)
    return model


class Ensemble(nn.ModuleList):
    """reference models/experimental.py:98-110: several models on one input.  In eval mode forward returns what Model.forward returns,
    `[(z, None), seg]` (plus the argmax map with seg_argmax=True): z concatenates the members' decoded predictions along the anchor axis
    (the reference's "nms ensemble" with the fork's missing index restored, `module(x, augment)[0][0]`), and seg is the mean of the
    members' seg logits (the reference's commented "mean ensemble" applied to the seg output; the fork defines none).  On the device:
    engine.forward_ensemble."""

    def check_members(self):
        """raises ValueError unless the members can share one output: the same Detect.no, seg classes, Detect.stride, device and parameter
        dtype, and at most MYOLO_ENSEMBLE_MAX of them.  Runs once per member list and dtype / device state."""
        from .. import _lib
        for k, m in enumerate(self):
            if not isinstance(m, _yolo.Model):
                raise ValueError(f"Ensemble member {k} is a {type(m).__name__}, not a Model")
        params = [next(m.parameters()) for m in self]
        key = tuple((id(m), p.dtype, p.device) for m, p in zip(self, params))
        if getattr(self, "_checked", None) == key:
            return
        if not 1 <= len(self) <= _lib.ENSEMBLE_MAX:
            raise ValueError(f"Ensemble: {len(self)} members; the device path takes 1 to {_lib.ENSEMBLE_MAX}")

        def props(m, p):
            det, seg = m.model[-1], m.model[-2]
            return {"Detect.no (5 + nc)": int(det.no), "seg classes": int(seg.c_out), "Detect.stride": [float(s) for s in det.stride],
                    "device": p.device, "parameter dtype": p.dtype}
        first = props(self[0], params[0])
        for k, (m, p) in enumerate(zip(self, params)):
            for name, v in props(m, p).items():
                if v != first[name]:
                    raise ValueError(f"Ensemble member {k} has {name} {v}, member 0 has {first[name]}: members must agree to share one output")
        self._checked = key

    def forward(self, x, augment=False, profile=False, seg_argmax=False):
        if self.training or any(m.training for m in self):
            raise RuntimeError("Ensemble.forward needs eval mode: the members' decoded predictions are concatenated, which a train-mode "
                               "forward does not produce (call ensemble.eval())")
        if profile:
            raise ValueError("Ensemble.forward: profile=True profiles one plain Model forward; it cannot be combined with an ensemble")
        self.check_members()
        from ..engine import forward_ensemble
        return forward_ensemble(list(self), x, augment=augment, seg_argmax=seg_argmax)


def attempt_load(weights, map_location=None):
    """reference models/experimental.py:113-134.  Returns the model (or an Ensemble) in fp32, `.fuse().eval()`-ed.  An Ensemble's members
    are checked (Ensemble.check_members) here, so mismatched checkpoints fail before any input is read."""
    model = Ensemble()
    for w in weights if isinstance(weights, (list, tuple)) else [weights]:
        ckpt = load_checkpoint(w, map_location=map_location)
        m = ckpt["ema" if ckpt.get("ema") else "model"]
        model.append(_compat_fixup(m).float().fuse().eval())
    if len(model) == 1:
        return model[-1]
    print('Ensemble created with %s\n' % (weights,))
    for k in ("names", "stride"):
        setattr(model, k, getattr(model[-1], k))
    model.check_members()
    return model
