"""TEST/BENCH INFRASTRUCTURE — the reference's detect.py job (reference detect.py:134-149,191-193) on the host CPU, built
from the oracle restatement.  Used only by bench.py's `cpu_baseline` leg and `--impl reference` arm (the Python reference
itself cannot travel to the GPU box).  Same substrate as the reference: torch fp32 CPU ops, torchvision.ops.nms when
importable (that IS the reference's NMS backend, utils/general.py:493), else the numpy greedy restatement.
"""
import time

import numpy as np
import torch
import torch.nn.functional as F

from . import restate

try:
    import torchvision
    _tv_nms = torchvision.ops.nms
except Exception:  # pragma: no cover
    _tv_nms = None


def nms_torch(prediction: torch.Tensor, conf_thres=0.25, iou_thres=0.45, max_det=300, max_nms=30000, max_wh=4096):
    """reference utils/general.py:421-509 (best-class branch) with torch ops + torchvision.ops.nms, as the reference runs it."""
    if _tv_nms is None:
        return [torch.from_numpy(o) for o in restate.non_max_suppression(prediction.numpy(), conf_thres, iou_thres)]
    out = []
    for x in prediction:
        x = x[x[:, 4] > conf_thres]
        if not x.shape[0]:
            out.append(torch.zeros((0, 6))); continue
        x[:, 5:] *= x[:, 4:5]
        box = x[:, :4].clone()
        box[:, 0] = x[:, 0] - x[:, 2] / 2; box[:, 1] = x[:, 1] - x[:, 3] / 2
        box[:, 2] = x[:, 0] + x[:, 2] / 2; box[:, 3] = x[:, 1] + x[:, 3] / 2
        conf, j = x[:, 5:].max(1, keepdim=True)
        x = torch.cat((box, conf, j.float()), 1)[conf.view(-1) > conf_thres]
        if not x.shape[0]:
            out.append(torch.zeros((0, 6))); continue
        if x.shape[0] > max_nms:
            x = x[x[:, 4].argsort(descending=True)[:max_nms]]
        c = x[:, 5:6] * max_wh
        i = _tv_nms(x[:, :4] + c, x[:, 4], iou_thres)[:max_det]
        out.append(x[i])
    return out


class CpuPipeline:
    def __init__(self, cfg, sd, threads=None):
        self.cfg, self.sd = cfg, sd
        if threads:
            torch.set_num_threads(threads)
        self.threads = torch.get_num_threads()

    def __call__(self, x: torch.Tensor, conf=0.25, iou=0.45):
        """x: (B,3,H,W) float in [0,1] (CPU).  Returns (dets list, class map (B,H,W) int64, timings dict)."""
        t0 = time.perf_counter()
        out = restate.model_forward(self.cfg, self.sd, x)
        t1 = time.perf_counter()
        dets = nms_torch(out["z"].clone(), conf, iou)
        t2 = time.perf_counter()
        H, W = x.shape[2:]
        cls = torch.stack([F.interpolate(out["seg"][b:b + 1], (H, W), mode="bilinear", align_corners=True)[0].max(0)[1]
                           for b in range(x.shape[0])])
        t3 = time.perf_counter()
        return dets, cls, dict(model=t1 - t0, nms=t2 - t1, segpost=t3 - t2)


class ReferencePipeline:
    """The UNMODIFIED reference tree (MYOLO_REFERENCE_ROOT or `baseline/_ref`, whichever exists) imported through
    oracle/ref_shims.py and driven exactly like detect.py:144-148,191-193.  The tree cannot travel to the GPU box (it is not an installable
    package: `pip install <reference checkout>` fails with "Neither 'setup.py' nor 'pyproject.toml' found", DESIGN.md), so this class is what
    bench.py uses in the build container and CpuPipeline (the port) is what it uses where the tree is absent."""

    def __init__(self, cfg, sd, threads=None):
        import copy
        from . import ref_shims
        ref_yolo, ref_general = ref_shims.import_reference()
        if threads:
            torch.set_num_threads(threads)
        self.threads = torch.get_num_threads()
        torch.manual_seed(0)
        self.model = ref_yolo.Model(copy.deepcopy(cfg))
        self.model.load_state_dict(sd)
        self.model.fuse().eval()
        self.nms = ref_general.non_max_suppression

    def __call__(self, x: torch.Tensor, conf=0.25, iou=0.45):
        with torch.no_grad():
            t0 = time.perf_counter()
            out = self.model(x)
            t1 = time.perf_counter()
            dets = self.nms(out[0][0], conf, iou)
            t2 = time.perf_counter()
            H, W = x.shape[2:]
            seg = out[1]
            cls = torch.stack([F.interpolate(seg[b:b + 1], (H, W), mode="bilinear", align_corners=True)[0].max(0)[1] for b in range(x.shape[0])])
            t3 = time.perf_counter()
        return dets, cls, dict(model=t1 - t0, nms=t2 - t1, segpost=t3 - t2)


def reference_root():
    """first existing location of the unmodified reference tree, or None"""
    import os
    here = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    for cand in (os.environ.get("MYOLO_REFERENCE_ROOT"), os.path.join(here, "baseline", "_ref")):
        if cand and os.path.isfile(os.path.join(cand, "models", "yolo.py")):
            return cand
    return None


def make_cpu_pipeline(cfg, sd, threads=None):
    """(pipeline, kind): the unmodified reference when its tree is present, the port otherwise"""
    root = reference_root()
    if root is not None:
        import os
        os.environ["MYOLO_REFERENCE_ROOT"] = root
        from . import ref_shims
        ref_shims.REF_ROOT = root
        try:
            return ReferencePipeline(cfg, sd, threads), "reference"
        except Exception:       # an incomplete tree: fall back to the port rather than fail the bench
            pass
    return CpuPipeline(cfg, sd, threads), "port"
