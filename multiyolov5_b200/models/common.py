"""Parameter-holding shells of the reference's building blocks (reference models/common.py).

The classes keep the reference's constructor signatures and sub-module names so that `state_dict()` keys are
identical (tests/golden/manifest_*.json) and reference checkpoints' tensors load unchanged.  They contain NO arithmetic:
compute happens in the compiled layer plan (multiyolov5_b200/plan.py -> libmyolo_sm90a.so) driven by Model.forward.
Calling a block's forward() directly raises - there is deliberately no eager PyTorch path.

autoShape / Detections (reference models/common.py:605-752) wrap a Model for in-memory inputs; see autoShape.
"""
import math
from pathlib import Path

import numpy as np
import torch
import torch.nn as nn

from ..utils.datasets import LETTERBOX_ITEM, letterbox_geometry, letterbox_item_table, letterbox_items
from ..utils.general import (SEG_CROP_ITEM, increment_path, non_max_suppression, scale_boxes, scale_coords_geometry, seg_crop_argmax,
                             seg_crop_item_table)


class _PlanOnly(nn.Module):
    def forward(self, *a, **k):
        raise RuntimeError(f"{type(self).__name__} holds parameters only; run it through models.yolo.Model.forward "
                           "(compiled sm_90a plan). There is no eager PyTorch fallback.")


def autopad(k, p=None):  # reference models/common.py:22-26
    return (k // 2 if isinstance(k, int) else [x // 2 for x in k]) if p is None else p


class Conv(_PlanOnly):
    """Conv2d(bias=False) + BatchNorm2d + SiLU   (reference models/common.py:33-46)"""

    def __init__(self, c1, c2, k=1, s=1, p=None, g=1, act=True):
        super().__init__()
        assert g == 1, "grouped convolutions are not on the shipped *_city_seg path"
        self.conv = nn.Conv2d(c1, c2, k, s, autopad(k, p), groups=g, bias=False)
        self.bn = nn.BatchNorm2d(c2)
        self.act = nn.SiLU() if act is True else (act if isinstance(act, nn.Module) else nn.Identity())


class Bottleneck(_PlanOnly):  # reference models/common.py:95-105
    def __init__(self, c1, c2, shortcut=True, g=1, e=0.5):
        super().__init__()
        c_ = int(c2 * e)
        self.cv1, self.cv2 = Conv(c1, c_, 1, 1), Conv(c_, c2, 3, 1, g=g)
        self.add = shortcut and c1 == c2


class C3(_PlanOnly):  # reference models/common.py:127-139
    def __init__(self, c1, c2, n=1, shortcut=True, g=1, e=0.5):
        super().__init__()
        c_ = int(c2 * e)
        self.cv1, self.cv2, self.cv3 = Conv(c1, c_, 1, 1), Conv(c1, c_, 1, 1), Conv(2 * c_, c2, 1)
        self.m = nn.Sequential(*[Bottleneck(c_, c_, shortcut, g, e=1.0) for _ in range(n)])


class SPP(_PlanOnly):  # reference models/common.py:163-174
    def __init__(self, c1, c2, k=(5, 9, 13)):
        super().__init__()
        c_ = c1 // 2
        self.cv1, self.cv2 = Conv(c1, c_, 1, 1), Conv(c_ * (len(k) + 1), c2, 1, 1)
        self.m = nn.ModuleList([nn.MaxPool2d(kernel_size=x, stride=1, padding=x // 2) for x in k])
        self.k = tuple(k)


class C3SPP(_PlanOnly):  # reference models/common.py:142-152
    def __init__(self, c1, c2, k=(5, 9, 13), g=1, e=0.5):
        super().__init__()
        c_ = int(c1 * e)
        self.cv1, self.cv2, self.cv3 = Conv(c1, c_, 1, 1), Conv(c1, c_, 1, 1), Conv(c_ + int(c_ * 1.5), c2, 1)
        self.m = SPP(c_, int(c_ * 1.5), k=k)


class Focus(_PlanOnly):  # reference models/common.py:542-551
    def __init__(self, c1, c2, k=1, s=1, p=None, g=1, act=True):
        super().__init__()
        self.conv = Conv(c1 * 4, c2, k, s, p, g, act)


class Concat(_PlanOnly):  # reference models/common.py:582-589
    def __init__(self, dimension=1):
        super().__init__()
        self.d = dimension


def _dilated(c1, c2, d):  # bare Conv2d + BN + SiLU branch (reference models/common.py:481-490, 243-257)
    return nn.Sequential(nn.Conv2d(c1, c2, kernel_size=3, stride=1, padding=d, dilation=d, bias=False), nn.BatchNorm2d(c2), nn.SiLU())


class FFM(_PlanOnly):  # reference models/common.py:210-230
    def __init__(self, in_chan, out_chan, reduction=1, is_cat=True, k=1):
        super().__init__()
        self.convblk = Conv(in_chan, out_chan, k=k, s=1, p=None)
        self.channel_attention = nn.Sequential(
            nn.AdaptiveAvgPool2d(1), nn.Conv2d(out_chan, out_chan // reduction, 1, 1, 0, bias=False), nn.SiLU(inplace=True),
            nn.Conv2d(out_chan // reduction, out_chan, 1, 1, 0, bias=False), nn.Sigmoid())
        self.is_cat = is_cat
        self.k = k


class ASPP(_PlanOnly):  # reference models/common.py:233-275
    def __init__(self, in_planes, out_planes, d=(3, 6, 9), has_globel=True, map_reduce=4):
        super().__init__()
        self.has_globel, self.hid, self.d = has_globel, in_planes // map_reduce, tuple(d)
        self.branch0 = nn.Sequential(Conv(in_planes, self.hid, k=1, s=1))
        self.branch1, self.branch2, self.branch3 = (_dilated(in_planes, self.hid, x) for x in d)
        if has_globel:
            self.branch4 = nn.Sequential(nn.AdaptiveAvgPool2d(1), Conv(in_planes, self.hid, k=1))
        self.ConvLinear = Conv(int((5 if has_globel else 4) * self.hid), out_planes, k=1, s=1)


class RFB2(_PlanOnly):  # reference models/common.py:470-511
    def __init__(self, in_planes, out_planes, map_reduce=4, d=(2, 3), has_globel=False):
        super().__init__()
        self.out_channels, self.has_globel, self.d = out_planes, has_globel, tuple(d)
        ip = in_planes // map_reduce
        self.branch0 = nn.Sequential(Conv(in_planes, ip, k=1, s=1), Conv(ip, ip, k=3, s=1))
        self.branch1, self.branch2 = _dilated(ip, ip, d[0]), _dilated(ip, ip, d[1])
        self.branch3 = nn.Sequential(Conv(in_planes, ip, k=1, s=1))
        if has_globel:
            self.branch4 = nn.Sequential(nn.AdaptiveAvgPool2d(1), Conv(ip, ip, k=1))
        self.ConvLinear = Conv(int((5 if has_globel else 4) * ip), out_planes, k=1, s=1)


class PyramidPooling(_PlanOnly):  # reference models/common.py:514-539
    def __init__(self, in_channels, k=(1, 2, 3, 6)):
        super().__init__()
        self.k = tuple(k)
        self.pool1, self.pool2, self.pool3, self.pool4 = (nn.AdaptiveAvgPool2d(x) for x in k)
        oc = in_channels // 4
        self.conv1, self.conv2, self.conv3, self.conv4 = (Conv(in_channels, oc, k=1) for _ in range(4))


# ---- autoShape (reference models/common.py:605-752) ----
def color_list():
    """reference utils/plots.py:29-34: matplotlib's ten TABLEAU_COLORS as (r, g, b), written out (matplotlib is not a dependency)"""
    hexes = ("1f77b4", "ff7f0e", "2ca02c", "d62728", "9467bd", "8c564b", "e377c2", "7f7f7f", "bcbd22", "17becf")
    return [tuple(int(h[i:i + 2], 16) for i in (0, 2, 4)) for h in hexes]


def autoshape_inputs(imgs, size=640, stride=32):
    """reference models/common.py:637-654: the inputs as 3-channel uint8 HWC arrays (paths and PIL images read, CHW when shape[0] < 5
    transposed, grayscale tiled, a 4th channel cut), their `files` names, shape0 [(h0, w0)] and the shared inference shape1 [H, W]"""
    from PIL import Image
    n, imgs = (len(imgs), imgs) if isinstance(imgs, list) else (1, [imgs])
    out, shape0, shape1, files = [], [], [], []
    for i, im in enumerate(imgs):
        f = f"image{i}"
        if isinstance(im, str):
            if im.startswith("http"):
                raise NotImplementedError("autoShape: URL inputs are not built (there is no network access); pass a file path or an array")
            im, f = np.asarray(Image.open(im)), im
        elif isinstance(im, Image.Image):
            im, f = np.asarray(im), getattr(im, "filename", f) or f
        files.append(Path(f).with_suffix(".jpg").name)
        im = np.asarray(im)
        if im.dtype != np.uint8:
            raise ValueError(f"autoShape: image {i} is {im.dtype}; the device letterbox takes uint8 pixels (the reference's cv2 path)")
        if im.shape[0] < 5:
            im = im.transpose((1, 2, 0))
        im = im[:, :, :3] if im.ndim == 3 else np.tile(im[:, :, None], 3)
        s = im.shape[:2]
        shape0.append(s)
        g = size / max(s)
        shape1.append([y * g for y in s])
        out.append(im)
    shape1 = [int(math.ceil(x / stride) * stride) for x in np.stack(shape1, 0).max(0)]     # make_divisible
    return out, files, shape0, shape1


class AutoShapeStage:
    """the device side of one autoShape call, from ONE pinned host-to-device copy: the packed sources, the letterbox and seg-crop item
    tables and the scale_coords geometry (views of one device buffer)"""

    def __init__(self, imgs, shape0, shape1, device, pinned=None):
        B = len(imgs)
        windows, offs = [], []
        for h0, w0 in shape0:
            (rw, rh), _, _, (top, _, left, _) = letterbox_geometry((h0, w0), shape1, auto=False)
            windows.append((top, left, rh, rw))
        align = lambda v: (v + 63) // 64 * 64      # noqa: E731
        o_seg = align(B * LETTERBOX_ITEM.itemsize)
        o_geom = align(o_seg + B * SEG_CROP_ITEM.itemsize)
        end = align(o_geom + B * 20)
        for h0, w0 in shape0:
            offs.append(end)
            end = align(end + h0 * w0 * 3)
        if pinned is None or pinned.numel() < end:
            pinned = torch.empty(end, dtype=torch.uint8, pin_memory=True)
        self.pinned = pinned
        host = pinned.numpy()
        host[:B * LETTERBOX_ITEM.itemsize] = letterbox_item_table(shape0, shape1, offs).view(np.uint8)
        host[o_seg:o_seg + B * SEG_CROP_ITEM.itemsize] = seg_crop_item_table(windows, shape0).view(np.uint8)
        geom = np.stack([scale_coords_geometry(shape1, s) for s in shape0])
        host[o_geom:o_geom + B * 20] = geom.view(np.uint8).reshape(-1)
        for im, off, (h0, w0) in zip(imgs, offs, shape0):
            host[off:off + h0 * w0 * 3].reshape(h0, w0, 3)[...] = im
        self.buf = torch.empty(end, dtype=torch.uint8, device=device)
        self.buf.copy_(pinned[:end], non_blocking=True)
        self.B, self.shape0, self.shape1 = B, list(shape0), list(shape1)
        self.lb_items = self.buf[:B * LETTERBOX_ITEM.itemsize]
        self.seg_items = self.buf[o_seg:o_seg + B * SEG_CROP_ITEM.itemsize]
        self.geom = self.buf[o_geom:o_geom + B * 20].view(torch.float32).view(B, 5)

    def letterbox(self, dtype=torch.float32):
        """(B,3,H,W) letterboxed batch, one launch"""
        return letterbox_items(self.buf, self.lb_items, self.B, self.shape1, dtype)


class autoShape(nn.Module):
    """reference models/common.py:605-672: a Model for cv2 / numpy / PIL / file-path / torch inputs, with pre-process and NMS.

        results = model([im1, im2, im3], size=640)        # HWC uint8 RGB arrays of any sizes, CHW, grayscale, RGBA, PIL, paths
        results.print(); results.xyxy[0]; results.render(); results.seg[0]

    One call is one pinned staging copy of every source and table, one letterbox launch for the ragged batch (myolo_letterbox_items),
    one forward (its `[0][0]`: the fork's `[0]` is the tuple (z, train_out) of this multi-task model), non_max_suppression, one launch
    that scales every image's rows to it and writes the normalised forms (myolo_scale_boxes) and one that makes every image's class
    map (myolo_seg_crop_upsample_argmax).  The NMS row counts are the only device-to-host read; the results stay on the device.
    Timings are CUDA events, read when printed.  A torch.Tensor goes straight to the model.  Not built: URL inputs, inputs that are not
    uint8 (the reference resizes those with cv2's float path)."""
    conf = 0.25     # NMS confidence threshold
    iou = 0.45      # NMS IoU threshold
    classes = None  # (optional list) filter by class

    def __init__(self, model):
        super().__init__()
        self.model = model.eval()
        self._pinned = None

    def autoshape(self):
        print("autoShape already enabled, skipping... ")
        return self

    @torch.no_grad()
    def forward(self, imgs, size=640, augment=False, profile=False):
        p = next(self.model.parameters())
        if isinstance(imgs, torch.Tensor):
            return self.model(imgs.to(p.device).type_as(p), augment, profile)
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
        ev[0].record()
        imgs, files, shape0, shape1 = autoshape_inputs(imgs, size, int(self.stride.max()))
        st = self.stage(imgs, shape0, shape1, p.device)
        x = st.letterbox(p.dtype)
        ev[1].record()
        y = self.model(x, augment, profile)
        ev[2].record()
        return self.postprocess(imgs, files, st, x.shape, y[0][0], y[1], ev)

    def stage(self, imgs, shape0, shape1, device):
        """the call's one host-to-device copy (AutoShapeStage); the pinned buffer is kept for the next call"""
        st = AutoShapeStage(imgs, shape0, shape1, device, self._pinned)
        self._pinned = st.pinned
        return st

    def postprocess(self, imgs, files, st, shape, z, seg, ev):
        """NMS of z, boxes to image space and the class maps of seg for the staged batch `st`: Detections.  ev: four CUDA events, the
        first three recorded (start, after the pre-process, after the forward); the fourth is recorded here"""
        rows, cnt = non_max_suppression(z, conf_thres=self.conf, iou_thres=self.iou, classes=self.classes, return_padded=True)
        xywh, xyxyn, xywhn = scale_boxes(rows, cnt, st.geom)
        maps = seg_crop_argmax(seg, st.seg_items, st.shape0)
        ev[3].record()
        counts = cnt.tolist()
        cut = lambda t: [t[i, :counts[i]] for i in range(st.B)]      # noqa: E731
        return Detections(imgs, cut(rows), files, ev, self.names, shape, xywh=cut(xywh), xyxyn=cut(xyxyn), xywhn=cut(xywhn), seg=maps)


class Detections:
    """reference models/common.py:675-752: the results of one autoShape call.  imgs (the RGB arrays), pred = xyxy (per image (n, 6)
    [x1, y1, x2, y2, conf, cls] in its pixels, on the device), xywh, xyxyn, xywhn, n, t (ms per image: pre-process, inference, NMS),
    s (the inference BCHW shape), names, files; and seg, this port's addition: per image its (h0, w0) uint8 class map on the device."""

    def __init__(self, imgs, pred, files, times=None, names=None, shape=None, xywh=None, xyxyn=None, xywhn=None, seg=None):
        self.imgs = imgs
        self.pred = pred
        self.names = names
        self.files = files
        self.xyxy = pred
        self.xywh, self.xyxyn, self.xywhn = xywh, xyxyn, xywhn
        self.seg = seg
        self.n = len(self.pred)
        self._times, self._t = times, None
        self.s = shape

    @property
    def t(self):
        if self._t is None:
            ev = self._times
            ev[-1].synchronize()
            self._t = tuple(ev[i].elapsed_time(ev[i + 1]) / self.n for i in range(3))
        return self._t

    def display(self, pprint=False, show=False, save=False, render=False, save_dir=""):
        from PIL import Image
        from ..utils.plots import plot_one_box
        colors = color_list()
        for i, (img, pred) in enumerate(zip(self.imgs, self.pred)):
            line = f"image {i + 1}/{len(self.pred)}: {img.shape[0]}x{img.shape[1]} "
            pred = pred.cpu()
            for c in pred[:, -1].unique():
                n = int((pred[:, -1] == c).sum())
                line += f"{n} {self.names[int(c)]}{'s' * (n > 1)}, "
            if save or render:
                if not (img.flags.writeable and img.flags.c_contiguous):
                    img = self.imgs[i] = np.array(img, order="C")   # cv2 draws only on a writable, contiguous array
                for *box, conf, cls in pred.tolist():
                    plot_one_box(box, img, label=f"{self.names[int(cls)]} {conf:.2f}", color=colors[int(cls) % 10])
            img = Image.fromarray(img.astype(np.uint8)) if isinstance(img, np.ndarray) else img
            if pprint:
                print(line.rstrip(", "))
            if save:
                f = self.files[i]
                img.save(Path(save_dir) / f)
                print(f"{'Saved' * (i == 0)} {f}", end="," if i < self.n - 1 else f" to {save_dir}\n")
            if render:
                self.imgs[i] = np.asarray(img)

    def print(self):
        self.display(pprint=True)
        print(f"Speed: %.1fms pre-process, %.1fms inference, %.1fms NMS per image at shape {tuple(self.s)}" % self.t)

    def show(self):
        raise NotImplementedError("Detections.show(): there is no display here; use render() or save()")

    def save(self, save_dir="runs/hub/exp"):
        save_dir = increment_path(save_dir, exist_ok=save_dir != "runs/hub/exp")
        Path(save_dir).mkdir(parents=True, exist_ok=True)
        self.display(save=True, save_dir=save_dir)

    def render(self):
        self.display(render=True)
        return self.imgs

    def pandas(self):
        raise NotImplementedError("Detections.pandas(): pandas is not a dependency; use xyxy / xywh / xyxyn / xywhn")

    def tolist(self):
        """one Detections per image, its lists popped to single items, as the reference's tolist (models/common.py:743-749) - which
        passes `names` where the file names go (and the shape as the times), so its items have no names and cannot print: here
        each keeps its file name, the names, the shape and the call's per-image times"""
        x = [Detections([self.imgs[i]], [self.pred[i]], [self.files[i]], None, self.names, self.s, xywh=[self.xywh[i]],
                        xyxyn=[self.xyxyn[i]], xywhn=[self.xywhn[i]], seg=[self.seg[i]]) for i in range(self.n)]
        for d in x:
            d._t = self.t
            for k in ["imgs", "pred", "xyxy", "xyxyn", "xywh", "xywhn", "seg"]:
                setattr(d, k, getattr(d, k)[0])
        return x

    def __len__(self):
        return self.n
