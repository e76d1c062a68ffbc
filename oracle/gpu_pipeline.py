"""BENCH INFRASTRUCTURE - the reference's OWN GPU path as a baseline on the same GPU (BASELINE.md section 3 "secondary, honest comparison"):
PyTorch fp16 + cuDNN with `cudnn.benchmark = True` (reference detect.py:96-103,115-124,144-148,191-193) for the detect.py job, and an
`amp.autocast` step (reference train.py:363-401) for training.  The graph is the oracle restatement run on CUDA tensors (the reference tree
itself cannot travel to the GPU box); when the unmodified tree is present (build container) the module builds the real reference `Model`.
None of this is the product: bench.py reports it beside our numbers as `reference_gpu`."""
import time

import torch
import torch.nn.functional as F

from . import restate
from .cpu_pipeline import nms_torch, reference_root


class TorchHalfPipeline:
    """detect.py job on the GPU with torch kernels: half model, half input"""

    def __init__(self, cfg, sd, device="cuda"):
        torch.backends.cudnn.benchmark = True                       # detect.py:124
        self.cfg = cfg
        self.kind = "port (oracle restatement on torch CUDA fp16 + cuDNN)"
        self.model = None
        root = reference_root()
        if root is not None:
            try:
                import copy
                from . import ref_shims
                ref_shims.REF_ROOT = root
                ref_yolo, ref_general = ref_shims.import_reference()
                m = ref_yolo.Model(copy.deepcopy(cfg))
                m.load_state_dict(sd)
                self.model = m.fuse().eval().to(device).half()       # detect.py:99-103
                self.ref_nms = ref_general.non_max_suppression
                self.kind = "reference (unmodified tree, model.half(), cudnn.benchmark)"
            except Exception:
                self.model = None
        self.sd = {k: v.to(device) for k, v in sd.items()}

    @torch.no_grad()
    def __call__(self, x_half, conf=0.25, iou=0.45):
        """x_half: (B,3,H,W) fp16 CUDA.  Returns (dets, class map)."""
        H, W = x_half.shape[2:]
        if self.model is not None:
            out = self.model(x_half)
            z, seg = out[0][0], out[1]
            dets = self.ref_nms(z, conf, iou)
        else:
            o = restate.model_forward(self.cfg, self.sd, x_half, half=True)
            z, seg = o["z"], o["seg"]
            dets = nms_torch(z.float(), conf, iou)
        # detect.py:191-193, per image as the reference does
        cls = torch.stack([F.interpolate(seg[b:b + 1], (H, W), mode="bilinear", align_corners=True)[0].max(0)[1] for b in range(seg.shape[0])])
        return dets, cls


class TorchAutocastTrainStep:
    """train.py:363-401 with torch kernels: autocast forward of the train-mode graph, the torch loss modules, GradScaler, SGD(nesterov)"""

    def __init__(self, cfg, sd, loss_model, hyp, batch_size, detgain=0.6, seggain=0.35, device="cuda"):
        from multiyolov5_b200.utils.loss import ComputeLoss, SegmentationLosses
        torch.backends.cudnn.benchmark = True
        self.cfg, self.bs, self.detgain, self.seggain = cfg, batch_size, detgain, seggain
        self.sd = {}
        params = []
        for k, v in sd.items():
            t = v.to(device).clone()
            if v.is_floating_point() and "running" not in k and "anchor" not in k:
                t.requires_grad_(True)
                params.append(t)
            self.sd[k] = t
        loss_model.hyp, loss_model.gr = hyp, 1.0
        self.det_loss = ComputeLoss(loss_model)
        self.seg_loss = SegmentationLosses(ignore_index=-1)
        self.opt = torch.optim.SGD(params, lr=hyp["lr0"], momentum=hyp["momentum"], nesterov=True, weight_decay=hyp["weight_decay"])
        self.scaler = torch.amp.GradScaler("cuda", init_scale=2.0 ** 10)

    def step(self, imgs, targets, segimgs, segtargets):
        with torch.autocast("cuda", dtype=torch.float16):
            raws, _ = restate.model_forward_train(self.cfg, self.sd, imgs)
            loss, _ = self.det_loss([r.float() for r in raws], targets)
        self.scaler.scale(loss * self.detgain).backward()
        with torch.autocast("cuda", dtype=torch.float16):
            _, seg = restate.model_forward_train(self.cfg, self.sd, segimgs)
            segloss = self.seg_loss(seg.float(), segtargets) * self.bs * self.seggain
        self.scaler.scale(segloss).backward()
        self.scaler.step(self.opt)
        self.scaler.update()
        self.opt.zero_grad(set_to_none=True)
        return loss.detach(), segloss.detach()
