"""Device-side pre-process behind the reference's names (SURVEY.md section 8f rank 1):

    letterbox(img, new_shape, color, auto, scaleFill, scaleup, stride) -> (img, ratio, (dw, dh))     reference utils/datasets.py:818-848
    preprocess(img0, img_size, stride, half)  -> (1|B,3,H,W) float tensor in [0,1]                     :185-189 + detect.py:135-137
    DeviceImageCache(images, img_size, labels) / DetAugmenter(cache, hyp)(indices) -> (imgs, targets)   :518-599 (augment=True)

`img` is a uint8 HWC BGR frame (numpy array or torch tensor; a CPU input is uploaded as uint8 - 4x less than the fp32 the reference
ships to the GPU); the resize (OpenCV's 8-bit INTER_LINEAR arithmetic, bit exact), the 114 border, the channel swap, the transpose and
the /255 run in ONE kernel of libmyolo_sm90a.  The host only does the reference's shape arithmetic.
"""
import ctypes as C
import math
import random

import numpy as np
import torch

from .. import _lib


def letterbox_geometry(shape, new_shape=(640, 640), auto=True, scaleFill=False, scaleup=True, stride=32):
    """host arithmetic of the reference's letterbox: ((new_w, new_h), ratio, (dw, dh), (top, bottom, left, right))"""
    if isinstance(new_shape, int):
        new_shape = (new_shape, new_shape)
    r = min(new_shape[0] / shape[0], new_shape[1] / shape[1])
    if not scaleup:
        r = min(r, 1.0)
    ratio = r, r
    new_unpad = int(round(shape[1] * r)), int(round(shape[0] * r))
    dw, dh = new_shape[1] - new_unpad[0], new_shape[0] - new_unpad[1]
    if auto:
        dw, dh = np.mod(dw, stride), np.mod(dh, stride)
    elif scaleFill:
        dw, dh = 0.0, 0.0
        new_unpad = (new_shape[1], new_shape[0])
        ratio = new_shape[1] / shape[1], new_shape[0] / shape[0]
    dw /= 2
    dh /= 2
    top, bottom = int(round(dh - 0.1)), int(round(dh + 0.1))
    left, right = int(round(dw - 0.1)), int(round(dw + 0.1))
    return new_unpad, ratio, (dw, dh), (top, bottom, left, right)


def _as_device_frames(img):
    t = torch.from_numpy(np.ascontiguousarray(img)) if isinstance(img, np.ndarray) else img
    assert t.dtype == torch.uint8 and t.dim() in (3, 4) and t.shape[-1] == 3, "expected uint8 (H,W,3) or (B,H,W,3) BGR frames"
    if not t.is_cuda:
        t = t.pin_memory().cuda(non_blocking=True) if torch.cuda.is_available() else t
    if not t.is_cuda:
        raise _lib.MyoloError("letterbox needs a CUDA device: multiyolov5_b200 has no CPU path")
    return t.contiguous()


def _run(frames, geom, color, out_dtype, chw, swap_rb):
    batched = frames.dim() == 4
    f4 = frames if batched else frames[None]
    B, H0, W0, _ = f4.shape
    (rw, rh), _, _, (top, bottom, left, right) = geom
    H, W = rh + top + bottom, rw + left + right
    shape = (B, 3, H, W) if chw else (B, H, W, 3)
    out = torch.empty(shape, dtype=out_dtype, device=frames.device)
    pad = (C.c_int32 * 3)(*[int(c) for c in color])
    _lib.check(_lib.lib().myolo_letterbox(_lib.ptr(f4), B, H0, W0, rw, rh, top, left, H, W, pad, _lib.ptr(out), _lib.torch_dtype_code(out_dtype),
                                          int(chw), int(swap_rb), _lib.stream_ptr()))
    return out if batched else out[0]


def letterbox(img, new_shape=(640, 640), color=(114, 114, 114), auto=True, scaleFill=False, scaleup=True, stride=32):
    """Resize and pad while meeting stride-multiple constraints; returns (uint8 HWC frame on the GPU, ratio, (dw, dh))"""
    frames = _as_device_frames(img)
    geom = letterbox_geometry(tuple(frames.shape[-3:-1]), new_shape, auto, scaleFill, scaleup, stride)
    return _run(frames, geom, color, torch.uint8, chw=False, swap_rb=False), geom[1], geom[2]


def preprocess(img0, img_size=640, stride=32, half=True, color=(114, 114, 114), auto=True):
    """LoadImages.__next__ + the conversion at the top of detect.py's loop in one kernel: BGR uint8 frame(s) -> RGB (B,3,H,W) fp16/fp32
    in [0,1], letterboxed to `img_size`.  Returns (tensor, ratio, (dw, dh))."""
    frames = _as_device_frames(img0)
    geom = letterbox_geometry(tuple(frames.shape[-3:-1]), img_size, auto, False, True, stride)
    out = _run(frames, geom, color, torch.float16 if half else torch.float32, chw=True, swap_rb=True)
    return (out if out.dim() == 4 else out[None]), geom[1], geom[2]


# ------------------------------------------------------------------------------------------------
# detection training batches (reference utils/datasets.py:518-599 LoadImagesAndLabels.__getitem__ + collate_fn, augment=True)
# ------------------------------------------------------------------------------------------------
def _xywhn2xyxy(x, w, h, padw, padh):   # reference utils/general.py:275-282 (numpy, keeps the input dtype)
    y = np.copy(x)
    y[:, 0] = w * (x[:, 0] - x[:, 2] / 2) + padw
    y[:, 1] = h * (x[:, 1] - x[:, 3] / 2) + padh
    y[:, 2] = w * (x[:, 0] + x[:, 2] / 2) + padw
    y[:, 3] = h * (x[:, 1] + x[:, 3] / 2) + padh
    return y


def _xyxy2xywh(x):                      # reference utils/general.py:255-262 (numpy)
    y = np.copy(x)
    y[:, 0] = (x[:, 0] + x[:, 2]) / 2
    y[:, 1] = (x[:, 1] + x[:, 3]) / 2
    y[:, 2] = x[:, 2] - x[:, 0]
    y[:, 3] = x[:, 3] - x[:, 1]
    return y


class DeviceImageCache:
    """The reference's `cache_images` on the device: each decoded uint8 HWC BGR frame is resized so that its long side is `img_size`
    (`load_image`, cv2.resize INTER_LINEAR as with augment=True; exact 2x down-scaling takes OpenCV's area path) by a bit-exact kernel and
    kept in ONE device arena (`offsets` / `shapes` index it).  `labels[i]`: (n, 5) [class, x, y, w, h] normalised, stored as float32 like
    the reference's label cache.  Decoding (cv2.imread) stays with the caller."""

    def __init__(self, images, img_size, labels=None, segments=None):
        if segments is not None and any(len(s) for s in segments):
            raise NotImplementedError("DeviceImageCache: polygon label segments are not supported (boxes only)")
        if not torch.cuda.is_available():
            raise _lib.MyoloError("DeviceImageCache needs a CUDA device: multiyolov5_b200 has no CPU path")
        self.img_size, self.n = int(img_size), len(images)
        self.shapes0, self.shapes, self.offsets = [], [], []
        total = 0
        for im in images:
            assert im.dtype in (np.uint8, torch.uint8) and im.ndim == 3 and im.shape[2] == 3, "expected uint8 (H,W,3) BGR frames"
            h0, w0 = int(im.shape[0]), int(im.shape[1])
            r = self.img_size / max(h0, w0)
            h, w = (int(h0 * r), int(w0 * r)) if r != 1 else (h0, w0)
            self.shapes0.append((h0, w0)); self.shapes.append((h, w)); self.offsets.append(total)
            total += h * w * 3
        self.arena = torch.empty(max(total, 1), dtype=torch.uint8, device="cuda")
        L, sp = _lib.lib(), _lib.stream_ptr()
        for im, (h0, w0), (h, w), off in zip(images, self.shapes0, self.shapes, self.offsets):
            src = _as_device_frames(im)
            _lib.check(L.myolo_resize_u8(_lib.ptr(src), h0, w0, C.c_void_p(self.arena.data_ptr() + off), h, w, sp))
        self.labels = [np.array(l, dtype=np.float32).reshape(-1, 5) for l in labels] if labels is not None else \
            [np.zeros((0, 5), np.float32) for _ in range(self.n)]
        assert len(self.labels) == self.n

    def image(self, i):
        """cached image i as a (h, w, 3) uint8 view of the arena"""
        h, w = self.shapes[i]
        return self.arena[self.offsets[i]:self.offsets[i] + h * w * 3].view(h, w, 3)

    def ptr(self, i):
        return self.arena.data_ptr() + self.offsets[i]


class DetAugmenter:
    """Detection training batches on the device: `DetAugmenter(cache, hyp)(indices)` returns what
    `collate_fn([dataset[i] for i in indices])` returns for a LoadImagesAndLabels(augment=True, rect=False) dataset - uint8 (B,3,s,s) RGB
    images (or float16/float32 = value / 255, as the training loop's `imgs.float() / 255`) and (n, 6) [image, class, x, y, w, h] float32
    targets, both on the GPU.

    The random parameters are drawn on the host from Python `random` and `numpy.random` in exactly the order and number of calls of
    the reference (mosaic choice, mosaic centre and partners, random_perspective, mixup, HSV gains, flips), so a seeded run gives the
    reference's batch bit for bit.  Labels are transformed on the host with the reference's numpy formulas; the pixels (mosaic, affine
    warp, mixup, HSV, flips, BGR->RGB / CHW) are one kernel launch per batch on the current stream, without a device synchronisation.
    Not built (raises): perspective != 0 (warpPerspective), label segments, the 9-image mosaic and the quad collate."""

    def __init__(self, cache, hyp, stride=32, mosaic9=False, quad=False):
        if float(hyp.get("perspective", 0.0)) != 0.0:
            raise NotImplementedError("DetAugmenter: hyp['perspective'] != 0 needs cv2.warpPerspective, which is not built (affine only)")
        if mosaic9:
            raise NotImplementedError("DetAugmenter: load_mosaic9 (9-image mosaic) is not built")
        if quad:
            raise NotImplementedError("DetAugmenter: the quad collate (collate_fn4) is not built")
        self.cache, self.hyp, self.stride = cache, dict(hyp), stride
        self.img_size, self.n = cache.img_size, cache.n
        self.indices = range(self.n)
        self.mosaic_border = [-self.img_size // 2, -self.img_size // 2]
        self._keep = []

    # ---- random_perspective (reference :851-937), affine only
    def _perspective(self, img_h, img_w, targets, border=(0, 0)):
        hyp = self.hyp
        height, width = img_h + border[0] * 2, img_w + border[1] * 2
        C_ = np.eye(3)
        C_[0, 2], C_[1, 2] = -img_w / 2, -img_h / 2
        P = np.eye(3)
        p = hyp["perspective"]
        P[2, 0], P[2, 1] = random.uniform(-p, p), random.uniform(-p, p)
        R = np.eye(3)
        a = random.uniform(-hyp["degrees"], hyp["degrees"])
        s = random.uniform(1 - hyp["scale"], 1 + hyp["scale"])
        ang = a * (math.pi / 180)                  # cv2.getRotationMatrix2D(center=(0, 0), angle=a, scale=s), restated
        alpha, beta = math.cos(ang) * s, math.sin(ang) * s
        R[0] = alpha, beta, (1 - alpha) * 0.0 - beta * 0.0
        R[1] = -beta, alpha, beta * 0.0 + (1 - alpha) * 0.0
        S = np.eye(3)
        S[0, 1] = math.tan(random.uniform(-hyp["shear"], hyp["shear"]) * math.pi / 180)
        S[1, 0] = math.tan(random.uniform(-hyp["shear"], hyp["shear"]) * math.pi / 180)
        T = np.eye(3)
        T[0, 2] = random.uniform(0.5 - hyp["translate"], 0.5 + hyp["translate"]) * width
        T[1, 2] = random.uniform(0.5 - hyp["translate"], 0.5 + hyp["translate"]) * height
        M = T @ S @ R @ P @ C_
        assert (height, width) == (self.img_size, self.img_size)
        n = len(targets)
        if n:
            xy = np.ones((n * 4, 3))
            xy[:, :2] = targets[:, [1, 2, 3, 4, 1, 4, 3, 2]].reshape(n * 4, 2)
            xy = (xy @ M.T)[:, :2].reshape(n, 8)
            x, y = xy[:, [0, 2, 4, 6]], xy[:, [1, 3, 5, 7]]
            new = np.concatenate((x.min(1), y.min(1), x.max(1), y.max(1))).reshape(4, n).T
            new[:, [0, 2]] = new[:, [0, 2]].clip(0, width)
            new[:, [1, 3]] = new[:, [1, 3]].clip(0, height)
            box1, box2 = targets[:, 1:5].T * s, new.T          # box_candidates(wh_thr=2, ar_thr=20, area_thr=0.1)
            w1, h1 = box1[2] - box1[0], box1[3] - box1[1]
            w2, h2 = box2[2] - box2[0], box2[3] - box2[1]
            ar = np.maximum(w2 / (h2 + 1e-16), h2 / (w2 + 1e-16))
            i = (w2 > 2) & (h2 > 2) & (w2 * h2 / (w1 * h1 + 1e-16) > 0.1) & (ar < 20)
            targets = targets[i]
            targets[:, 1:5] = new[i]
        return M, targets

    @staticmethod
    def _warp(tiles, M):
        """myolo_aug_warp of a canvas made of `tiles` [(src pointer, src width, x1a, y1a, x2a, y2a, padw, padh)]; M inverted as
        cv2.warpAffine inverts it (double)"""
        w = _lib.AugWarp()
        for t, (p, sw, x1, y1, x2, y2, pw, ph) in enumerate(tiles):
            w.src[t] = p
            w.rect[t][:] = [x1, y1, x2, y2]
            w.off[t][:] = [pw, ph]
            w.src_w[t] = sw
        w.n_tiles = len(tiles)
        m = [float(v) for v in M[:2].reshape(-1)]
        D = m[0] * m[4] - m[1] * m[3]
        D = 1.0 / D if D != 0 else 0.0
        i0, i1, i3, i4 = m[4] * D, m[1] * -D, m[3] * -D, m[0] * D
        w.minv[:] = [i0, i1, -i0 * m[2] - i1 * m[5], i3, i4, -i3 * m[2] - i4 * m[5]]
        return w

    # ---- load_mosaic (reference :671-724)
    def _mosaic(self, index):
        s, cache = self.img_size, self.cache
        yc, xc = [int(random.uniform(-x, 2 * s + x)) for x in self.mosaic_border]
        indices = [index] + random.choices(self.indices, k=3)
        tiles, labels4 = [], []
        for i, index in enumerate(indices):
            h, w = cache.shapes[index]
            if i == 0:
                x1a, y1a, x2a, y2a = max(xc - w, 0), max(yc - h, 0), xc, yc
                x1b, y1b = w - (x2a - x1a), h - (y2a - y1a)
            elif i == 1:
                x1a, y1a, x2a, y2a = xc, max(yc - h, 0), min(xc + w, s * 2), yc
                x1b, y1b = 0, h - (y2a - y1a)
            elif i == 2:
                x1a, y1a, x2a, y2a = max(xc - w, 0), yc, xc, min(s * 2, yc + h)
                x1b, y1b = w - (x2a - x1a), 0
            else:
                x1a, y1a, x2a, y2a = xc, yc, min(xc + w, s * 2), min(s * 2, yc + h)
                x1b, y1b = 0, 0
            padw, padh = x1a - x1b, y1a - y1b
            tiles.append((cache.ptr(index), w, x1a, y1a, x2a, y2a, padw, padh))
            labels = cache.labels[index].copy()
            if labels.size:
                labels[:, 1:] = _xywhn2xyxy(labels[:, 1:], w, h, padw, padh)
            labels4.append(labels)
        labels4 = np.concatenate(labels4, 0)
        np.clip(labels4[:, 1:], 0, 2 * s, out=labels4[:, 1:])
        M, labels4 = self._perspective(2 * s, 2 * s, labels4, border=self.mosaic_border)
        return self._warp(tiles, M), labels4

    # ---- letterbox(auto=False, scaleup=True) + random_perspective(border=0) (reference :536-557)
    def _single(self, index):
        s, cache = self.img_size, self.cache
        h, w = cache.shapes[index]
        (nw, nh), ratio, (dw, dh), (top, bottom, left, right) = letterbox_geometry((h, w), s, auto=False, scaleup=True)
        if (w, h) != (nw, nh):
            img = torch.empty((nh, nw, 3), dtype=torch.uint8, device="cuda")
            _lib.check(_lib.lib().myolo_resize_u8(C.c_void_p(cache.ptr(index)), h, w, _lib.ptr(img), nh, nw, _lib.stream_ptr()))
            self._keep.append(img)
            p = img.data_ptr()
        else:
            p = cache.ptr(index)
        labels = cache.labels[index].copy()
        if labels.size:
            labels[:, 1:] = _xywhn2xyxy(labels[:, 1:], ratio[0] * w, ratio[1] * h, dw, dh)
        M, labels = self._perspective(nh + top + bottom, nw + left + right, labels)
        return self._warp([(p, nw, left, top, left + nw, top + nh, left, top)], M), labels

    def item(self, index):
        """parameters (myolo_aug_item) and final labels (n, 5) of dataset[index]; consumes the random draws of one __getitem__"""
        hyp, s = self.hyp, self.img_size
        it = _lib.AugItem()
        if random.random() < hyp["mosaic"]:
            it.warp[0], labels = self._mosaic(index)
            it.n_warps = 1
            if random.random() < hyp["mixup"]:
                it.warp[1], labels2 = self._mosaic(random.randint(0, self.n - 1))
                r = np.random.beta(8.0, 8.0)
                it.mix_r, it.mix_q, it.n_warps = float(r), float(1 - r), 2
                labels = np.concatenate((labels, labels2), 0)
        else:
            it.warp[0], labels = self._single(index)
            it.n_warps = 1
        g = np.random.uniform(-1, 1, 3) * [hyp["hsv_h"], hyp["hsv_s"], hyp["hsv_v"]] + 1     # augment_hsv (reference :646-657)
        x = np.arange(0, 256, dtype=np.int16)
        luts = (((x * g[0]) % 180).astype(np.uint8), np.clip(x * g[1], 0, 255).astype(np.uint8), np.clip(x * g[2], 0, 255).astype(np.uint8))
        for c in range(3):
            C.memmove(C.addressof(it.lut[c]), np.ascontiguousarray(luts[c]).ctypes.data, 256)
        nL = len(labels)
        if nL:
            labels[:, 1:5] = _xyxy2xywh(labels[:, 1:5])
            labels[:, [2, 4]] /= s
            labels[:, [1, 3]] /= s
        if random.random() < hyp["flipud"]:
            it.flipud = 1
            if nL:
                labels[:, 2] = 1 - labels[:, 2]
        if random.random() < hyp["fliplr"]:
            it.fliplr = 1
            if nL:
                labels[:, 1] = 1 - labels[:, 1]
        return it, labels

    def __call__(self, indices, out_dtype=torch.uint8):
        """one batch: (imgs (B,3,s,s) of out_dtype, targets (n,6) float32), both on the current CUDA device / stream"""
        self._keep = []
        B, s = len(indices), self.img_size
        items = (_lib.AugItem * B)()
        targets = []
        for b, index in enumerate(indices):
            items[b], labels = self.item(index)
            t = torch.zeros((len(labels), 6))
            t[:, 0] = b
            if len(labels):
                t[:, 1:] = torch.from_numpy(labels)
            targets.append(t)
        host = torch.frombuffer(bytearray(items), dtype=torch.uint8).pin_memory()
        dev_items = host.cuda(non_blocking=True)
        imgs = torch.empty((B, 3, s, s), dtype=out_dtype, device="cuda")
        _lib.check(_lib.lib().myolo_augment_det(_lib.ptr(dev_items), B, s, _lib.ptr(imgs), _lib.torch_dtype_code(out_dtype), _lib.stream_ptr()))
        targets = torch.cat(targets, 0).pin_memory().cuda(non_blocking=True)
        self._keep = [dev_items] + self._keep
        return imgs, targets
