"""Parameter-holding shells of the reference's building blocks (reference models/common.py).

The classes keep the reference's constructor signatures and sub-module names so that `state_dict()` keys are
identical (tests/golden/manifest_*.json) and reference checkpoints' tensors load unchanged.  They contain NO arithmetic:
compute happens in the compiled layer plan (multiyolov5_b200/plan.py -> libmyolo_sm90a.so) driven by Model.forward.
Calling a block's forward() directly raises - there is deliberately no eager PyTorch path.
"""
import torch.nn as nn


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
