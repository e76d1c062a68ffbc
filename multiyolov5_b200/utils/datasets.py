"""Device-side pre-process behind the reference's names (SURVEY.md section 8f rank 1):

    letterbox(img, new_shape, color, auto, scaleFill, scaleup, stride) -> (img, ratio, (dw, dh))     reference utils/datasets.py:818-848
    preprocess(img0, img_size, stride, half)  -> (1|B,3,H,W) float tensor in [0,1]                     :185-189 + detect.py:135-137
    DeviceImageCache(images, img_size, labels) / DetAugmenter(cache, hyp)(indices) -> (imgs, targets)   :518-599 (augment=True)
    DeviceImageCache(images, img_size, labels) / DetRectLoader(cache, hyp, batch_size)(positions) -> (imgs, targets), iterable
                                                                             :347-439 + :518-599 (augment=True, rect=True: --rect)
    collate_quad(imgs, targets) -> (imgs4, targets4)                               :602-625 collate_fn4 (--quad) over either batch
    ImageWeights(DetAugmenter(...)).draw(class_weights, maps) -> indices, then (...)(positions) -> (imgs, targets)
                                                                    train.py:305-316 --image-weights + :519 index = self.indices[index]
    DeviceImageCache(images, img_size, labels, augment=False) / DetValLoader(cache, batch_size) -> iterable of (imgs, targets, paths,
        shapes) for test(data, model=m, dataloader=DetValLoader(cache, 32))                          :347-452 + :518-599 (rect=True)
    DeviceSegCache(images, masks, mask_map) / SegAugmenter(cache, base_size, crop_size, preset)(indices) -> (segimgs, segtargets)
                                                                             SegmentationDataset.py:118-151 + ColorJitter + ToTensor
    SegAugmenter(...).val(indices, crop_size) / .testval(indices) -> (segimgs, segtargets)      :96-116 (mode='val') / :81-94 (testval)

`img` is a uint8 HWC BGR frame (numpy array or torch tensor; a CPU input is uploaded as uint8 - 4x less than the fp32 the reference
ships to the GPU); the resize (OpenCV's 8-bit INTER_LINEAR arithmetic, bit exact), the 114 border, the channel swap, the transpose and
the /255 run in ONE kernel of libmyolo_sm90a.  The host only does the reference's shape arithmetic.
"""
import ctypes as C
import functools
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


# ---- autoShape's ragged batch (reference models/common.py:655-658; csrc/preprocess.cu letterbox_items_kernel) ----
# include/myolo.h myolo_letterbox_item
LETTERBOX_ITEM = np.dtype([("offset", "<i8"), ("scale_x", "<f8"), ("scale_y", "<f8"), ("H0", "<i4"), ("W0", "<i4"), ("mode", "<i4"),
                           ("rw", "<i4"), ("rh", "<i4"), ("top", "<i4"), ("left", "<i4"), ("reserved", "<i4")])


def resize_geometry(H0, W0, rh, rw):
    """cv2.resize's INTER_LINEAR set-up for (H0, W0) -> (rh, rw), as csrc/resize.cuh resize_geom computes it: (scale_x, scale_y, mode),
    scales 1 / (dst / src) in double, mode 0 copy, 1 bilinear, 2 exact 2x down-scale (cv2 takes its area path there)"""
    sx, sy = 1.0 / (rw / W0), 1.0 / (rh / H0)
    eps = 2.220446049250313e-16
    mode = 0 if (rw == W0 and rh == H0) else 2 if (abs(sx - 2.0) < eps and abs(sy - 2.0) < eps) else 1
    return sx, sy, mode


def letterbox_item_table(shapes0, shape1, offsets):
    """the myolo_letterbox_item table of letterbox(im, new_shape=shape1, auto=False) for images of shapes0 (h0, w0) whose HWC sources
    start at byte `offsets` of the packed buffer"""
    t = np.zeros(len(shapes0), LETTERBOX_ITEM)
    for k, ((h0, w0), off) in enumerate(zip(shapes0, offsets)):
        (rw, rh), _, _, (top, _, left, _) = letterbox_geometry((h0, w0), shape1, auto=False)
        sx, sy, mode = resize_geometry(h0, w0, rh, rw)
        t[k] = (off, sx, sy, h0, w0, mode, rw, rh, top, left, 0)
    return t


def letterbox_items(src, items, B, shape1, out_dtype=torch.float32):
    """B packed RGB uint8 sources letterboxed to shape1 (H, W) in one launch: (B,3,H,W) uint8, or fp16 / fp32 value / 255.  src: the
    CUDA uint8 buffer holding the sources; items: CUDA uint8 bytes of the letterbox_item_table"""
    if not (src.is_cuda and items.is_cuda and src.dtype == torch.uint8 and items.numel() == B * LETTERBOX_ITEM.itemsize):
        raise _lib.MyoloError("letterbox_items needs CUDA uint8 sources and a CUDA table of B items")
    out = torch.empty((B, 3, int(shape1[0]), int(shape1[1])), dtype=out_dtype, device=src.device)
    _lib.check(_lib.lib().myolo_letterbox_items(_lib.ptr(src), _lib.ptr(items), B, out.shape[2], out.shape[3], _lib.ptr(out),
                                                _lib.torch_dtype_code(out_dtype), _lib.stream_ptr()))
    return out


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
    (`load_image`) by a bit-exact kernel and kept in ONE device arena (`offsets` / `shapes` index it).  `augment` is the dataset's flag:
    True (training) resizes with cv2.resize INTER_LINEAR (exact 2x down-scaling takes OpenCV's area path); False (validation) shrinks with
    INTER_AREA and grows with INTER_LINEAR, as load_image does.  `labels[i]`: (n, 5) [class, x, y, w, h] normalised, stored as float32
    like the reference's label cache.  Decoding (cv2.imread) stays with the caller."""

    def __init__(self, images, img_size, labels=None, segments=None, augment=True):
        if segments is not None and any(len(s) for s in segments):
            raise NotImplementedError("DeviceImageCache: polygon label segments are not supported (boxes only)")
        if not torch.cuda.is_available():
            raise _lib.MyoloError("DeviceImageCache needs a CUDA device: multiyolov5_b200 has no CPU path")
        self.img_size, self.n, self.augment = int(img_size), len(images), bool(augment)
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
            shrink = not self.augment and self.img_size < max(h0, w0)         # load_image: INTER_AREA if r < 1 and not augment
            resize = L.myolo_resize_area_u8 if shrink else L.myolo_resize_u8
            _lib.check(resize(_lib.ptr(src), h0, w0, C.c_void_p(self.arena.data_ptr() + off), h, w, sp))
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
    `--quad` is a collate step over the drawn batch, as in the reference: pass this batch (uint8) to `collate_quad`.
    Not built (raises): perspective != 0 (warpPerspective), label segments, the 9-image mosaic, and `quad=True` here."""

    def __init__(self, cache, hyp, stride=32, mosaic9=False, quad=False):
        if float(hyp.get("perspective", 0.0)) != 0.0:
            raise NotImplementedError("DetAugmenter: hyp['perspective'] != 0 needs cv2.warpPerspective, which is not built (affine only)")
        if mosaic9:
            raise NotImplementedError("DetAugmenter: load_mosaic9 (9-image mosaic) is not built")
        if quad:
            raise NotImplementedError("DetAugmenter: quad is a collate step, not a dataset option: pass the uint8 batch to "
                                      "utils.datasets.collate_quad (collate_fn4)")
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
    def _single(self, index, shape):
        """`shape`: img_size (int), or a rect batch's [h, w] row of batch_shapes (numpy ints, as the reference passes it: ratio and pad
        come out as numpy float64)"""
        cache = self.cache
        h, w = cache.shapes[index]
        (nw, nh), ratio, (dw, dh), (top, bottom, left, right) = letterbox_geometry((h, w), shape, auto=False, scaleup=True)
        p = self._resized(index, nh, nw) if (w, h) != (nw, nh) else cache.ptr(index)
        labels = cache.labels[index].copy()
        if labels.size:
            labels[:, 1:] = _xywhn2xyxy(labels[:, 1:], ratio[0] * w, ratio[1] * h, dw, dh)
        M, labels = self._perspective(nh + top + bottom, nw + left + right, labels)
        return self._warp([(p, nw, left, top, left + nw, top + nh, left, top)], M), labels

    def _resized(self, index, nh, nw):
        """device pointer of cached image `index` resized to nw x nh (letterbox's cv2.resize INTER_LINEAR), kept until the next batch"""
        h, w = self.cache.shapes[index]
        img = torch.empty((nh, nw, 3), dtype=torch.uint8, device="cuda")
        _lib.check(_lib.lib().myolo_resize_u8(C.c_void_p(self.cache.ptr(index)), h, w, _lib.ptr(img), nh, nw, _lib.stream_ptr()))
        self._keep.append(img)
        return img.data_ptr()

    def item(self, index, shape=None):
        """parameters (myolo_aug_item) and final labels (n, 5) of dataset[index]; consumes the random draws of one __getitem__.  `shape`:
        None for the square dataset (rect=False), or the item's rect batch shape [h, w] (rect=True: no mosaic draw, no mixup)"""
        hyp = self.hyp
        H, W = (self.img_size, self.img_size) if shape is None else (int(shape[0]), int(shape[1]))    # img.shape[:2] at :563-564
        it = _lib.AugItem()
        if shape is not None:
            it.warp[0], labels = self._single(index, shape)
            it.n_warps = 1
        elif random.random() < hyp["mosaic"]:
            it.warp[0], labels = self._mosaic(index)
            it.n_warps = 1
            if random.random() < hyp["mixup"]:
                it.warp[1], labels2 = self._mosaic(random.randint(0, self.n - 1))
                r = np.random.beta(8.0, 8.0)
                it.mix_r, it.mix_q, it.n_warps = float(r), float(1 - r), 2
                labels = np.concatenate((labels, labels2), 0)
        else:
            it.warp[0], labels = self._single(index, self.img_size)
            it.n_warps = 1
        g = np.random.uniform(-1, 1, 3) * [hyp["hsv_h"], hyp["hsv_s"], hyp["hsv_v"]] + 1     # augment_hsv (reference :646-657)
        x = np.arange(0, 256, dtype=np.int16)
        luts = (((x * g[0]) % 180).astype(np.uint8), np.clip(x * g[1], 0, 255).astype(np.uint8), np.clip(x * g[2], 0, 255).astype(np.uint8))
        for c in range(3):
            C.memmove(C.addressof(it.lut[c]), np.ascontiguousarray(luts[c]).ctypes.data, 256)
        nL = len(labels)
        if nL:
            labels[:, 1:5] = _xyxy2xywh(labels[:, 1:5])
            labels[:, [2, 4]] /= H
            labels[:, [1, 3]] /= W
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
        return self.launch([self.item(index) for index in indices], self.img_size, self.img_size, out_dtype)

    def launch(self, items_labels, H, W, out_dtype=torch.uint8):
        """the batch of drawn items [(myolo_aug_item, (n, 5) labels)] at H x W: one pinned copy of the items, one kernel, the targets"""
        B = len(items_labels)
        items = (_lib.AugItem * B)()
        targets = []
        for b, (it, labels) in enumerate(items_labels):
            items[b] = it
            t = torch.zeros((len(labels), 6))
            t[:, 0] = b
            if len(labels):
                t[:, 1:] = torch.from_numpy(labels)
            targets.append(t)
        host = torch.frombuffer(bytearray(items), dtype=torch.uint8).pin_memory()
        dev_items = host.cuda(non_blocking=True)
        imgs = torch.empty((B, 3, H, W), dtype=out_dtype, device="cuda")
        _lib.check(_lib.lib().myolo_augment_det_hw(_lib.ptr(dev_items), B, H, W, _lib.ptr(imgs), _lib.torch_dtype_code(out_dtype),
                                                   _lib.stream_ptr()))
        targets = torch.cat(targets, 0).pin_memory().cuda(non_blocking=True)
        self._keep = [dev_items] + self._keep
        return imgs, targets


# ------------------------------------------------------------------------------------------------
# detection validation batches (reference utils/datasets.py:347-452 + :518-599 LoadImagesAndLabels(augment=False, rect=True) + collate_fn,
# as create_dataloader builds it for test(): train.py:207-210)
# ------------------------------------------------------------------------------------------------
class ValBatch:
    """one rect validation batch planned on the host: source indices, letterbox geometry per item ((new_w, new_h), ratio, (dw, dh),
    (top, bottom, left, right)), the (n, 6) float32 targets and collate_fn's `shapes` tuple"""

    def __init__(self, indices, geoms, targets, shapes):
        self.indices, self.geoms, self.targets, self.shapes = indices, geoms, targets, shapes


def rect_plan(shapes0, img_size, batch_size, stride=32, pad=0.0):
    """The rect arithmetic of the reference's LoadImagesAndLabels.__init__ (:410-439) over the original (h0, w0) `shapes0`: returns
    (order, bi, batch_shapes).  `order` is the aspect-ratio sort (the reference's `irect`: numpy's default argsort kind, not stable, so
    the order of equal aspect ratios depends on the host CPU), `bi` the batch index of each sorted position and `batch_shapes` the
    (nb, 2) [h, w] int letterbox shapes."""
    n = len(shapes0)
    if n == 0:
        raise ValueError("rect_plan: no images")
    s = np.array([(w0, h0) for h0, w0 in shapes0], dtype=np.float64)         # the reference's self.shapes: wh
    ar = s[:, 1] / s[:, 0]
    order = ar.argsort()
    ar = ar[order]
    bi = np.floor(np.arange(n) / batch_size).astype(int)
    nb = bi[-1] + 1
    bshapes = [[1, 1]] * nb
    for i in range(nb):
        ari = ar[bi == i]
        mini, maxi = ari.min(), ari.max()
        if maxi < 1:
            bshapes[i] = [maxi, 1]
        elif mini > 1:
            bshapes[i] = [1, 1 / mini]
    return order, bi, np.ceil(np.array(bshapes) * img_size / stride + pad).astype(int) * stride


def det_val_plan(shapes0, shapes, labels, img_size, batch_size, stride=32, pad=0.5, single_cls=False):
    """The host arithmetic of the reference's rect validation dataset over cached images, in its statements and dtypes: `shapes0` are the
    original (h0, w0), `shapes` the cached (h, w), `labels` (n, 5) float32 normalised [class, x, y, w, h].  Returns (order, batch_shapes,
    [ValBatch]): `order` and `batch_shapes` as rect_plan gives them."""
    order, bi, batch_shapes = rect_plan(shapes0, img_size, batch_size, stride, pad)
    nb = len(batch_shapes)
    batches = []
    for b in range(nb):
        shape = batch_shapes[b]                  # a numpy row, as the reference passes it: ratio and pad come out as numpy float64
        indices, geoms, targets, shp = [], [], [], []
        for pos, j in enumerate(np.flatnonzero(bi == b)):
            index = int(order[j])
            (h0, w0), (h, w) = shapes0[index], shapes[index]
            geom = letterbox_geometry((h, w), shape, auto=False, scaleup=False)
            ratio, pd = geom[1], geom[2]
            lab = np.array(labels[index], dtype=np.float32).reshape(-1, 5)
            if single_cls:
                lab[:, 0] = 0
            if lab.size:
                lab[:, 1:] = _xywhn2xyxy(lab[:, 1:], ratio[0] * w, ratio[1] * h, pd[0], pd[1])
            nL = len(lab)
            if nL:
                lab[:, 1:5] = _xyxy2xywh(lab[:, 1:5])
                lab[:, [2, 4]] /= int(shape[0])
                lab[:, [1, 3]] /= int(shape[1])
            t = np.zeros((nL, 6), np.float32)
            t[:, 0] = pos
            t[:, 1:] = lab
            indices.append(index)
            geoms.append(geom)
            targets.append(t)
            shp.append(((h0, w0), ((h / h0, w / w0), pd)))
        batches.append(ValBatch(tuple(indices), geoms, np.concatenate(targets, 0), tuple(shp)))
    return order, batch_shapes, batches


class DetValLoader:
    """Detection validation batches on the device: the reference's `create_dataloader(path, imgsz, batch_size, gs, opt, rect=True,
    pad=pad)` (a LoadImagesAndLabels with augment=False, rect=True, and collate_fn) over a DeviceImageCache built with augment=False.
    Feeds `test.test(data, model=m, dataloader=DetValLoader(cache, 32))`; `batch_size` is the dataset's (train.py passes batch_size * 2).

    Iterating yields one (img uint8 (B, 3, H, W) RGB, targets (n, 6) float32, paths, shapes) per batch in loader order, images and
    targets on the device; `paths` are the source indices and `shapes` collate_fn's ((h0, w0), ((h / h0, w / w0), (dw, dh))) per item.
    The order, batch shapes, letterbox geometry and labels are planned once at construction (det_val_plan) and every batch's targets
    uploaded once: the batches are deterministic, so iterating does no label work and no host-to-device copy.  Each item is one
    myolo_letterbox launch (114 border, BGR -> RGB, CHW) into its slice of the batch, on the current stream, without a synchronisation."""

    def __init__(self, cache, batch_size, stride=32, pad=0.5, single_cls=False):
        if cache.augment:
            raise ValueError("DetValLoader: the cache must be built with augment=False (load_image's INTER_AREA validation resize)")
        self.cache, self.batch_size, self.stride, self.pad = cache, int(batch_size), int(stride), pad
        self.order, self.batch_shapes, self.batches = det_val_plan(cache.shapes0, cache.shapes, cache.labels, cache.img_size,
                                                                   self.batch_size, self.stride, pad, single_cls)
        self.targets = [torch.from_numpy(b.targets).cuda() for b in self.batches]

    def __len__(self):
        return len(self.batches)

    def __iter__(self):
        L, sp, cache = _lib.lib(), _lib.stream_ptr(), self.cache
        color = (C.c_int32 * 3)(114, 114, 114)
        for (H, W), batch, targets in zip(self.batch_shapes.tolist(), self.batches, self.targets):
            imgs = torch.empty((len(batch.indices), 3, H, W), dtype=torch.uint8, device="cuda")
            for k, (i, geom) in enumerate(zip(batch.indices, batch.geoms)):
                (rw, rh), _, _, (top, _, left, _) = geom
                h, w = cache.shapes[i]
                _lib.check(L.myolo_letterbox(C.c_void_p(cache.ptr(i)), 1, h, w, rw, rh, top, left, H, W, color,
                                             C.c_void_p(imgs.data_ptr() + k * 3 * H * W), _lib.U8, 1, 1, sp))
            yield imgs, targets, batch.indices, batch.shapes


def distributed_positions(n, epoch, rank, world_size, seed=0):
    """rank's positions of one epoch over a dataset of n under DistributedSampler(dataset, shuffle=True, seed=seed) after
    set_epoch(epoch): randperm from a generator seeded with seed + epoch, padded with its own head to a multiple of world_size, then every
    world_size-th from rank"""
    if not 0 <= rank < world_size:
        raise ValueError(f"rank {rank} outside world size {world_size}")
    g = torch.Generator()
    g.manual_seed(seed + epoch)
    idx = torch.randperm(n, generator=g).tolist()
    total = math.ceil(n / world_size) * world_size
    pad = total - len(idx)
    idx += (idx * math.ceil(pad / len(idx)))[:pad] if pad else []
    return idx[rank:total:world_size]


# ------------------------------------------------------------------------------------------------
# rect training batches (reference train.py:196-198 create_dataloader(..., augment=True, rect=opt.rect): LoadImagesAndLabels with
# augment=True, rect=True (:347-439, __getitem__ :518-592 without mosaic) + collate_fn)
# ------------------------------------------------------------------------------------------------
class DetRectLoader:
    """Detection training batches of `--rect` on the device, over a DeviceImageCache built with augment=True (INTER_LINEAR cache).

    The dataset is sorted by aspect ratio and every run of `batch_size` sorted positions shares one letterbox shape, as the reference
    plans it (rect_plan): `order` (position -> source index, the reference's `irect`), `batch` (position -> batch index) and
    `batch_shapes` ((nb, 2) [h, w]).  `loader(positions)` builds the batch of those sorted positions: per item the reference's draws in
    its order and number (random_perspective, augment_hsv, flipud, fliplr: no mosaic draw and no mixup under rect), the labels on the
    host with its numpy formulas, the pixels (letterbox to the batch shape, affine warp at that size, HSV, flips, BGR->RGB, CHW) in one
    myolo_augment_det_hw launch.  Positions whose batch shapes differ raise ValueError, as collate_fn's torch.stack does.

    Iterating yields the batches of consecutive positions (no sampler: rank -1), the partial last batch included.  `epoch_positions`
    gives one rank's positions under DDP (DistributedSampler(dataset) with shuffle, seed 0, set_epoch(epoch)); its batches are runs of
    `batch_size` of them, and any run that mixes shapes raises, as it does in the reference."""

    def __init__(self, cache, hyp, batch_size, stride=32, pad=0.0, single_cls=False):
        if not cache.augment:
            raise ValueError("DetRectLoader: the cache must be built with augment=True (load_image's INTER_LINEAR training resize)")
        self.aug = DetAugmenter(cache, hyp, stride)
        self.cache, self.batch_size, self.single_cls = cache, int(batch_size), bool(single_cls)
        self.order, self.batch, self.batch_shapes = rect_plan(cache.shapes0, cache.img_size, self.batch_size, stride, pad)
        self.n = cache.n

    def __len__(self):
        return len(self.batch_shapes)

    def shape_of(self, positions):
        """the batch shape [h, w] shared by `positions`; ValueError if they differ"""
        shapes = {tuple(int(v) for v in self.batch_shapes[self.batch[p]]) for p in positions}
        if len(shapes) != 1:
            raise ValueError(f"DetRectLoader: positions {list(positions)} have different batch shapes {sorted(shapes)}: collate_fn's "
                             "torch.stack cannot stack them")
        return self.batch_shapes[self.batch[positions[0]]]

    def item(self, position):
        """(myolo_aug_item, (n, 5) float32 labels) of dataset[position]; consumes the reference's draws of one item"""
        it, labels = self.aug.item(int(self.order[position]), self.batch_shapes[self.batch[position]])
        if self.single_cls:
            labels[:, 0] = 0
        return it, labels

    def __call__(self, positions, out_dtype=torch.uint8):
        """the batch of sorted `positions`: (imgs (B, 3, h, w) of out_dtype, targets (n, 6) float32), both on the current CUDA device /
        stream; float outputs are uint8 / 255 as the training loop's imgs.float() / 255"""
        positions = [int(p) for p in positions]
        if not positions or min(positions) < 0 or max(positions) >= self.n:
            raise ValueError(f"DetRectLoader: positions must be in [0, {self.n}), got {positions}")
        H, W = (int(v) for v in self.shape_of(positions))
        self.aug._keep = []
        return self.aug.launch([self.item(p) for p in positions], H, W, out_dtype)

    def epoch_positions(self, epoch, rank, world_size, seed=0):
        """rank's positions of one epoch under DistributedSampler(dataset, shuffle=True, seed=seed) after set_epoch(epoch)"""
        return distributed_positions(self.n, epoch, rank, world_size, seed)

    def batches(self, positions=None, out_dtype=torch.uint8):
        """the batches of runs of batch_size `positions` (default: every position in order), the last one partial"""
        positions = list(range(self.n)) if positions is None else list(positions)
        for k in range(0, len(positions), self.batch_size):
            yield self(positions[k:k + self.batch_size], out_dtype)

    def __iter__(self):
        return self.batches()


# ------------------------------------------------------------------------------------------------
# image-weighted training batches (reference train.py:255,305-316 --image-weights; utils/datasets.py:354,519,677)
# ------------------------------------------------------------------------------------------------
class ImageWeights:
    """`--image-weights` over a DetAugmenter: once per epoch, `draw(model_class_weights, maps, rank, group)` is the reference's
    train.py:305-316 block and sets the indices its dataset then reads.  Batches are `aug([iwts.indices[p] for p in positions])`, or
    `iwts(positions)`, with `positions` from `epoch_positions`: sequential at rank -1 (a plain DataLoader), DistributedSampler(shuffle=True,
    seed=0) after set_epoch(epoch) under DDP.  `collate_quad` and `train.MultiScale` apply to these batches unchanged.  The reference turns
    `--rect` off under `--image-weights` (its dataset's rect = False), so the square DetAugmenter batches are the ones it trains on.

    `model_class_weights` is train.py:255's `labels_to_class_weights(dataset.labels, nc).to(device) * nc` (utils.general), `maps` the
    float64 per-class mAP of the last test() (np.zeros(nc) before the first).  On rank -1 / 0, `draw`:
      - computes `cw = model_class_weights * (1 - maps) ** 2 / nc` with numpy on the host, as the reference does (nc values);
      - computes labels_to_image_weights for it on the device (myolo_image_weights), over labels uploaded at the first draw;
      - draws n `random.random()` values in the reference's order and runs random.choices(range(n), weights=iw, k=n) on the device
        (myolo_weighted_draw), bit for bit; when the total weight is not positive and finite it raises random.choices' ValueError and
        leaves `random` where it was, as random.choices does.
    Under DDP (rank >= 0, `group` an initialised process group) rank 0 broadcasts the int32 indices and a status word (NCCL: from the
    device), and the other ranks draw nothing and raise rank 0's ValueError if it had one.  Every rank then reads the indices back once
    and sets `aug.indices` to them, so DetAugmenter's mosaic partners (`random.choices(self.indices, k=3)`) come from the drawn list, as
    in the reference; mixup's `random.randint(0, n - 1)` does not.  The cache's labels are the dataset's: for `--single-cls` build it
    from labels whose class column is zeroed, as LoadImagesAndLabels(single_cls=True) does, with nc = 1."""

    def __init__(self, aug):
        self.aug, self.n = aug, aug.n
        self.indices = list(range(self.n))
        self._labels = None

    def _draw(self, cw):
        """the device work of rank -1 / 0: (int32 (n + 1) device tensor of the indices and the status word, `random`'s state before
        the draws)"""
        from .general import device_image_weights, label_classes
        if self._labels is None:
            self._labels = label_classes(self.aug.cache.labels)
        cls, offsets = self._labels
        n, dev = self.n, cls.device
        buf = torch.zeros(n + 1, dtype=torch.int32, device=dev)
        status = buf[n:]
        iw = device_image_weights(cls, offsets, cw, status)
        state = random.getstate()
        u = torch.tensor([random.random() for _ in range(n)], dtype=torch.float64).to(dev)
        cum = torch.empty(n, dtype=torch.float64, device=dev)
        total = torch.empty(1, dtype=torch.float64, device=dev)
        _lib.check(_lib.lib().myolo_weighted_draw(_lib.ptr(iw), _lib.ptr(u), n, _lib.ptr(cum), _lib.ptr(total), _lib.ptr(buf),
                                                  _lib.ptr(status), _lib.stream_ptr()))
        return buf, state

    def draw(self, class_weights, maps, rank=-1, group=None):
        """one epoch's drawn indices (a list of n ints), also set as `self.indices` and `aug.indices`"""
        state = None
        if rank in (-1, 0):
            cwm = class_weights.detach().cpu().numpy() if isinstance(class_weights, torch.Tensor) else np.asarray(class_weights)
            nc = len(cwm)
            cw = cwm * (1 - maps) ** 2 / nc
            buf, state = self._draw(cw)
        if rank != -1:
            import torch.distributed as dist
            nccl = dist.get_backend(group) == "nccl"
            dev = torch.device("cuda", torch.cuda.current_device()) if nccl else torch.device("cpu")
            buf = buf.to(dev) if rank == 0 else torch.zeros(self.n + 1, dtype=torch.int32, device=dev)
            dist.broadcast(buf, 0, group=group)
        host = buf.cpu().numpy()
        status = int(host[self.n])
        if status:
            from .general import iw_status_error
            if state is not None:
                random.setstate(state)
            raise iw_status_error(status)
        self.indices = host[:self.n].tolist()
        self.aug.indices = self.indices
        return self.indices

    def epoch_positions(self, epoch=0, rank=-1, world_size=1, seed=0):
        """rank's dataset positions of one epoch: 0 .. n-1 at rank -1, else DistributedSampler's (distributed_positions)"""
        return list(range(self.n)) if rank == -1 else distributed_positions(self.n, epoch, rank, world_size, seed)

    def __call__(self, positions, out_dtype=torch.uint8):
        """the batch of dataset `positions`: aug([indices[p] for p in positions])"""
        return self.aug([self.indices[int(p)] for p in positions], out_dtype)


# ------------------------------------------------------------------------------------------------
# quad training batches (reference train.py:197-199 create_dataloader(..., quad=opt.quad): LoadImagesAndLabels.collate_fn4, :602-625)
# ------------------------------------------------------------------------------------------------
_QUAD_HO = (0., 0, 0, 1, 0, 0)      # collate_fn4's ho, wo and s
_QUAD_WO = (0., 0, 1, 0, 0, 0)
_QUAD_S = (1, 1, .5, .5, .5, .5)


def collate_quad(imgs, targets, rng=random, out_dtype=torch.uint8):
    """`--quad`'s collate_fn4 over one drawn batch on the device: `imgs` uint8 (B, 3, h, w) and `targets` (n, 6) float32 [image, class,
    x, y, w, h] as DetAugmenter(...)(indices), DetRectLoader(...)(positions) or its iterator give them, both on the GPU.  Returns (imgs4
    (B // 4, 3, 2h, 2w) of out_dtype, targets4 (m, 6) float32) on the device; float outputs are uint8 / 255 as the training loop's
    imgs.float() / 255.

    One `rng.random()` per quad, in quad order, as the reference draws them after the whole batch: below 0.5 the quad is item 4q
    bilinearly up-scaled x2 (F.interpolate(..., scale_factor=2.) truncated to uint8) with its labels unchanged, and items 4q+1 .. 4q+3 are
    dropped; otherwise the 2x2 tile of the four items (4q top left, 4q+1 bottom left, 4q+2 top right, 4q+3 bottom right) with their labels
    shifted and halved by the reference's float32 operations in its order.  Items past 4 * (B // 4) are dropped.  The pixels are one
    myolo_collate_quad launch on the current stream; selecting the kept label rows synchronises with the device once, because their
    number is known only there.  ValueError for fewer than 4 images, as collate_fn4's torch.stack([]) fails on them."""
    if not (isinstance(imgs, torch.Tensor) and imgs.is_cuda and imgs.dtype == torch.uint8 and imgs.dim() == 4 and imgs.shape[1] == 3):
        raise ValueError("collate_quad: imgs must be a CUDA uint8 (B, 3, h, w) tensor")
    if not (isinstance(targets, torch.Tensor) and targets.is_cuda and targets.dtype == torch.float32 and targets.dim() == 2
            and targets.shape[1] == 6):
        raise ValueError("collate_quad: targets must be a CUDA float32 (n, 6) tensor")
    if out_dtype not in (torch.uint8, torch.float16, torch.float32):
        raise ValueError(f"collate_quad: out_dtype must be uint8, float16 or float32, got {out_dtype}")
    B, _, h, w = imgs.shape
    n = B // 4
    if n == 0:
        raise ValueError(f"collate_quad: a batch of {B} images has no quad (collate_fn4 needs at least 4)")
    tile = [rng.random() >= 0.5 for _ in range(n)]
    imgs = imgs.contiguous()
    out = torch.empty((n, 3, 2 * h, 2 * w), dtype=out_dtype, device=imgs.device)
    flags = (C.c_uint8 * n)(*tile)
    _lib.check(_lib.lib().myolo_collate_quad(_lib.ptr(imgs), B, h, w, flags, _lib.ptr(out), _lib.torch_dtype_code(out_dtype),
                                             _lib.stream_ptr()))
    host = torch.tensor(_QUAD_HO + _QUAD_WO + _QUAD_S + tuple(float(v) for v in tile) + (0.0,), dtype=torch.float32).pin_memory()
    dev = host.to(targets.device, non_blocking=True)             # one upload, no synchronisation
    ho, wo, s, tile_q = dev[0:6], dev[6:12], dev[12:18], dev[18:] != 0
    item = targets[:, 0].long()
    q, k = item // 4, item % 4
    t_row = tile_q[q.clamp(max=n)]                               # rows of items past the last quad index the False sentinel
    keep = (q < n) & (t_row | (k == 0))
    t, q, k, t_row = targets[keep], q[keep], k[keep], t_row[keep]
    # label[i], label[i+1] + ho, label[i+2] + wo, label[i+3] + ho + wo, each then * s; the first item takes no addition
    shifted = t + ho * ((k == 1) | (k == 3))[:, None] + wo * ((k == 2) | (k == 3))[:, None]
    tiled = torch.where((k == 0)[:, None], t, shifted) * s
    t = torch.where(t_row[:, None], tiled, t)
    t[:, 0] = q.float()
    return out, t


# ------------------------------------------------------------------------------------------------
# segmentation training batches (reference SegmentationDataset.py:118-151 _sync_transform, :182-189 / :219-222 _mask_transform,
# :81-94 _testval_img_transform, and the loader functions' ColorJitter + ToTensor, :458-531)
# ------------------------------------------------------------------------------------------------
# Cityscapes label id -> train id (the reference's `_key` at np.digitize(id, range(-1, 34), right=True) = id + 1)
_CITYSCAPES_KEY = np.array([-1, -1, -1, -1, -1, -1, -1, -1, 0, 1, -1, -1, 2, 3, 4, -1, -1, -1, 5, -1, 6, 7, 8, 9, 10, 11, 12, 13, 14,
                            15, -1, -1, 16, 17, 18])
_INVALID = -2

# the reference's get_citys_loader / get_citysbdd_loader / get_custom_loader: ColorJitter(b, c, s, h), get_long_size(low, high, std), crop
SEG_PRESETS = {
    "citys": dict(brightness=0.45, contrast=0.45, saturation=0.45, hue=0.15, low=0.65, high=3.0, std=25, crop_size=(1024, 512)),
    "citysbdd": dict(brightness=0.4, contrast=0.4, saturation=0.4, hue=0.05, low=0.65, high=2.0, std=40, crop_size=(1024, 512)),
    "custom": dict(brightness=0.4, contrast=0.4, saturation=0.4, hue=0.0, low=0.75, high=1.5, std=35, crop_size=None),   # (base, base)
}


def seg_mask_lut(kind):
    """256-entry int64 label map of a uint8 mask: 'cityscapes' is `_class_to_index` (255 -> 0, then id -> trainId; ids 34..254 are not
    in the reference's mapping and are marked -2), 'trainid' maps 255 -> -1 and keeps every other value"""
    lut = np.full(256, _INVALID, np.int64)
    if kind == "cityscapes":
        lut[:34] = _CITYSCAPES_KEY[1:]
        lut[255] = _CITYSCAPES_KEY[1]
    elif kind == "trainid":
        lut[:] = np.arange(256)
        lut[255] = -1
    else:
        raise ValueError(f"mask_map: expected 'cityscapes' or 'trainid', got {kind!r}")
    return lut


def _norm_pdf(x, mean, std):
    """scipy.stats.norm.pdf(x, mean, std), computed as scipy computes it (tests/test_seg_augment_host.py pins it ==)"""
    y = (np.asarray(x, np.float64) - mean) / std
    return np.exp(-y ** 2 / 2.0) / np.sqrt(2 * np.pi) / std


@functools.lru_cache(128)
def range_and_prob(base_size, low=0.5, high=3.0, std=25):
    """the reference's range_and_prob (SegmentationDataset.py:25-35): long-side candidates / 32 and their cumulative probabilities"""
    lo = math.ceil((base_size * low) / 32)
    hi = math.ceil((base_size * high) / 32)
    mean = math.ceil(base_size / 32) - 4
    x = np.array(list(range(lo, hi + 1)))
    p = _norm_pdf(x, mean, std)
    p = p / p.sum()
    return x, np.cumsum(p)


@functools.lru_cache(256)
def _bilinear_table(in_size, out_size):
    """Pillow's bilinear precompute_coeffs + normalize_coeffs_8bpc for an axis in_size -> out_size, as int32 rows {xmin, taps, k[0..K)}
    (22 fraction bits).  An unchanged axis is a one-tap identity, which equals Pillow's skipped pass."""
    if in_size == out_size:
        t = np.zeros((out_size, 3), np.int32)
        t[:, 0], t[:, 1], t[:, 2] = np.arange(out_size), 1, 1 << 22
        return t
    scale = float(in_size) / out_size
    filterscale = max(scale, 1.0)
    support = filterscale
    ksize = int(math.ceil(support)) * 2 + 1
    center = (np.arange(out_size) + 0.5) * scale
    xmin = np.maximum((center - support + 0.5).astype(np.int64), 0)
    xmax = np.minimum((center + support + 0.5).astype(np.int64), in_size) - xmin
    w = np.zeros((out_size, ksize))
    ww = np.zeros(out_size)
    for x in range(ksize):                                   # Pillow's loop order: ww accumulates tap by tap
        t = np.abs((x + xmin - center + 0.5) * (1.0 / filterscale))
        w[:, x] = np.where(x < xmax, np.where(t < 1.0, 1.0 - t, 0.0), 0.0)
        ww = ww + w[:, x]
    k = np.where(ww[:, None] != 0.0, w / np.where(ww == 0.0, 1.0, ww)[:, None], w)
    kk = np.where(k < 0, (-0.5 + k * (1 << 22)).astype(np.int64), (0.5 + k * (1 << 22)).astype(np.int64))
    t = np.zeros((out_size, ksize + 2), np.int32)
    t[:, 0], t[:, 1], t[:, 2:] = xmin, xmax, np.where(np.arange(ksize) < xmax[:, None], kk, 0)
    return t


@functools.lru_cache(256)
def _nearest_index(in_size, out_size):
    """source index per output position of Pillow's NEAREST resize (ImagingScaleAffine: xo = a/2, then xo += a, in double)"""
    a = float(in_size) / out_size
    idx = np.empty(out_size, np.int32)
    xo = a * 0.5
    for x in range(out_size):
        idx[x] = -1 if xo < 0.0 else int(xo)
        xo += a
    return idx


def _crop_rows(table, start, n, pad):
    """rows start..start+n of an axis table, `pad` (taps 0 / index -1) beyond its end"""
    out = np.empty((n,) + table.shape[1:], np.int32)
    m = max(0, min(n, len(table) - start))
    out[:m] = table[start:start + m]
    out[m:] = pad
    return out


class DeviceSegCache:
    """Decoded segmentation sources on the device: uint8 (H, W, 3) RGB frames as PIL's `convert('RGB')` decodes them and uint8 (H, W)
    masks as `np.array(Image.open(mask))` reads them, kept at native resolution (no resize at cache time) in ONE device arena.  Decoding
    stays with the caller.  The arena holds 4 bytes per source pixel: Cityscapes train (2975 frames of 2048x1024) is about 25 GB.

    `mask_map` is 'cityscapes' (the reference's `_class_to_index`: 255 -> 0, then label id -> train id), 'trainid' (255 -> -1, every other
    value kept: BDD100k and custom data), or a list with one of those per item (City+BDD, whose .png items are Cityscapes ids and .jpg
    items train ids).  Masks are validated on the host before upload: a 'cityscapes' mask holding a value outside the reference's mapping
    (34..254) raises ValueError, as the reference's assert fails on it."""

    def __init__(self, images, masks, mask_map="cityscapes"):
        if len(images) != len(masks):
            raise ValueError(f"DeviceSegCache: {len(images)} images but {len(masks)} masks")
        self.n = len(images)
        kinds = [mask_map] * self.n if isinstance(mask_map, str) else list(mask_map)
        if len(kinds) != self.n:
            raise ValueError(f"DeviceSegCache: mask_map has {len(kinds)} entries for {self.n} items")
        self.luts = [seg_mask_lut(k) for k in kinds]
        self.shapes, self.img_off, self.mask_off = [], [], []
        total = 0
        host = []
        for i, (im, m) in enumerate(zip(images, masks)):
            im = im.cpu().numpy() if isinstance(im, torch.Tensor) else np.asarray(im)
            m = m.cpu().numpy() if isinstance(m, torch.Tensor) else np.asarray(m)
            if im.dtype != np.uint8 or im.ndim != 3 or im.shape[2] != 3:
                raise ValueError(f"DeviceSegCache: image {i} must be uint8 (H, W, 3) RGB, got {im.dtype} {im.shape}")
            if m.dtype != np.uint8 or m.shape != im.shape[:2]:
                raise ValueError(f"DeviceSegCache: mask {i} must be uint8 {im.shape[:2]}, got {m.dtype} {m.shape}")
            bad = np.flatnonzero((self.luts[i][np.flatnonzero(np.bincount(m.ravel(), minlength=256))] == _INVALID))
            if bad.size:
                vals = np.flatnonzero(np.bincount(m.ravel(), minlength=256))[bad]
                raise ValueError(f"DeviceSegCache: mask {i} holds values {vals.tolist()} outside the {kinds[i]} mapping")
            h, w = im.shape[:2]
            self.shapes.append((h, w))
            self.img_off.append(total)
            self.mask_off.append(total + h * w * 3)
            total += h * w * 4
            host.append((im, m))
        if not torch.cuda.is_available():
            raise _lib.MyoloError("DeviceSegCache needs a CUDA device: multiyolov5_b200 has no CPU path")
        self.arena = torch.empty(max(total, 1), dtype=torch.uint8, device="cuda")
        for (im, m), io, mo in zip(host, self.img_off, self.mask_off):
            self.arena[io:mo].copy_(torch.from_numpy(np.ascontiguousarray(im)).view(-1))
            self.arena[mo:mo + m.size].copy_(torch.from_numpy(np.ascontiguousarray(m)).view(-1))

    def image(self, i):
        h, w = self.shapes[i]
        return self.arena[self.img_off[i]:self.img_off[i] + h * w * 3].view(h, w, 3)

    def mask(self, i):
        h, w = self.shapes[i]
        return self.arena[self.mask_off[i]:self.mask_off[i] + h * w].view(h, w)


class SegAugmenter:
    """Segmentation training batches on the device: `SegAugmenter(cache, base_size, crop_size, preset)(indices)` returns what
    `default_collate([dataset[i] for i in indices])` returns for the reference's mode='train' datasets (CitySegmentation,
    CityBddSegmentation, CustomSegmentation with the transforms of their loader functions): float32 (B, 3, h, w) images = uint8 / 255 as
    ToTensor divides (or uint8 / float16 = that float32 rounded) and int64 (B, h, w) labels with -1 = ignore, both on the GPU; (w, h) is
    `crop_size`.

    `preset` is 'citys', 'citysbdd' or 'custom' (SEG_PRESETS: jitter factors, long-side sampling low / high / std, crop); explicit
    arguments override it.  The random parameters are drawn on the host in exactly the reference's order and number: `random.random()`
    (mirror), `random.choices` (long side), `random.randint` (x1, then y1), then ColorJitter.get_params on torch's CPU generator
    (`torch.randperm(4)` and one `uniform_` per enabled factor).  Under the same seeds, with items taken in sequence (num_workers=0), the
    batch equals the reference's bit for bit.  The pixels are two kernel launches per batch on the current stream, after one pinned
    host-to-device copy of the parameters, without a device synchronisation.

    `testval(indices)` gives the reference's mode='testval' items and `val(indices, crop_size)` its mode='val' items
    (`_val_sync_transform`, with the int crop_size that train_citysbdd.py passes; the loaders' default tuple crop_size makes the
    reference raise TypeError there)."""

    def __init__(self, cache, base_size=1024, crop_size=None, preset="citys", brightness=None, contrast=None, saturation=None, hue=None,
                 low=None, high=None, std=None):
        if preset not in SEG_PRESETS:
            raise ValueError(f"SegAugmenter: preset must be one of {sorted(SEG_PRESETS)}, got {preset!r}")
        p = dict(SEG_PRESETS[preset])
        for k, v in dict(brightness=brightness, contrast=contrast, saturation=saturation, hue=hue, low=low, high=high, std=std).items():
            if v is not None:
                p[k] = v
        self.cache, self.base_size = cache, int(base_size)
        crop = crop_size if crop_size is not None else p["crop_size"] or (self.base_size, self.base_size)
        self.crop_size = (int(crop[0]), int(crop[1]))
        self.low, self.high, self.std = p["low"], p["high"], p["std"]

        def rng(v, center, clip):                        # ColorJitter._check_input for a number
            lo, hi = center - float(v), center + float(v)
            if clip:
                lo = max(lo, 0.0)
            return None if lo == hi == center else (float(lo), float(hi))
        if not 0.0 <= float(p["hue"]) <= 0.5:
            raise ValueError("SegAugmenter: hue must be in [0, 0.5]")
        self.jitter_ranges = (rng(p["brightness"], 1, True), rng(p["contrast"], 1, True), rng(p["saturation"], 1, True),
                              rng(p["hue"], 0, False))
        self._keep = []

    def draw(self, index):
        """the random parameters of dataset[index] (mode='train'), consuming the reference's draws"""
        h, w = self.cache.shapes[index]
        flip = random.random() < 0.5
        x, cum_p = range_and_prob(self.base_size, self.low, self.high, self.std)
        long_size = random.choices(population=x, cum_weights=cum_p, k=1)[0] * 32
        if h > w:
            oh = long_size
            ow = int(1.0 * w * long_size / h + 0.5)
        else:
            ow = long_size
            oh = int(1.0 * h * long_size / w + 0.5)
        cw, ch = self.crop_size
        x1 = random.randint(0, max(ow, cw) - cw)
        y1 = random.randint(0, max(oh, ch) - ch)
        order = torch.randperm(4).tolist()
        factors = [None if r is None else float(torch.empty(1).uniform_(r[0], r[1])) for r in self.jitter_ranges]
        return dict(flip=flip, ow=int(ow), oh=int(oh), x1=x1, y1=y1, order=order, factors=factors)

    @staticmethod
    def _item(cache, index, flip, ow, oh, x1, y1, w, h, mw, mh, order, factors, tables, mask_size=None):
        """one myolo_seg_item: the image resized to (ow, oh), the mask to `mask_size` (default (ow, oh)), both cropped at (x1, y1) to
        (w, h) / (mw, mh); appends its tables (int32 arrays) to `tables` [(offset, array)]"""
        H0, W0 = cache.shapes[index]
        it = _lib.SegItem()
        it.img, it.mask = cache.arena.data_ptr() + cache.img_off[index], cache.arena.data_ptr() + cache.mask_off[index]
        it.H0, it.W0, it.flip = H0, W0, int(bool(flip))
        tx, ty = _bilinear_table(W0, ow), _bilinear_table(H0, oh)
        it.kx, it.ky = tx.shape[1] - 2, ty.shape[1] - 2
        mow, moh = mask_size or (ow, oh)
        parts = [_crop_rows(tx, x1, w, 0), _crop_rows(ty, y1, h, 0), _crop_rows(_nearest_index(W0, mow), x1, mw, -1),
                 _crop_rows(_nearest_index(H0, moh), y1, mh, -1)]
        off = tables[-1][0] + tables[-1][1].size if tables else 0
        offs = []
        for a in parts:
            offs.append(off)
            tables.append((off, a))
            off += a.size
        it.col, it.row, it.mcol, it.mrow = offs
        ops = [k for k in order if factors[k] is not None]
        it.order[:] = ops + [-1] * (4 - len(ops))
        it.factor[:] = [0.0 if f is None else f for f in factors[:3]]
        it.hue_shift = int(np.int32(factors[3] * 255).astype(np.uint8)) if factors[3] is not None else 0   # adjust_hue's uint8 shift
        it.lut[:] = cache.luts[index].astype(np.int32).tolist()
        return it

    def _launch(self, items, tables, B, h, w, mh, mw, out_dtype):
        isz = C.sizeof(_lib.SegItem)
        n_tab = sum(a.size for _, a in tables)
        host = torch.empty(B * isz + 4 * n_tab, dtype=torch.uint8).pin_memory()
        C.memmove(host.data_ptr(), C.addressof(items), B * isz)
        tab = host[B * isz:].view(torch.int32).numpy()
        for off, a in tables:
            tab[off:off + a.size] = a.ravel()
        dev = host.cuda(non_blocking=True)
        imgs = torch.empty((B, 3, h, w), dtype=out_dtype, device="cuda")
        labels = torch.empty((B, mh, mw), dtype=torch.int64, device="cuda")
        scratch = torch.empty(B * h * w * 3, dtype=torch.uint8, device="cuda")
        _lib.check(_lib.lib().myolo_augment_seg(C.c_void_p(dev.data_ptr()), B, h, w, mh, mw, C.c_void_p(dev.data_ptr() + B * isz),
                                                _lib.ptr(scratch), _lib.ptr(imgs), _lib.torch_dtype_code(out_dtype), _lib.ptr(labels),
                                                _lib.stream_ptr()))
        self._keep = [host, dev, scratch]
        return imgs, labels

    def build(self, indices, params, out_dtype=torch.float32):
        """the batch of `indices` from drawn (or chosen) parameters, one dict per item as `draw` returns them"""
        if out_dtype not in (torch.uint8, torch.float16, torch.float32):
            raise ValueError(f"SegAugmenter: out_dtype must be uint8, float16 or float32, got {out_dtype}")
        cw, ch = self.crop_size
        B = len(indices)
        items, tables = (_lib.SegItem * B)(), []
        for b, (i, p) in enumerate(zip(indices, params)):
            ow, oh, x1, y1 = int(p["ow"]), int(p["oh"]), int(p["x1"]), int(p["y1"])
            if ow <= 0 or oh <= 0 or not 0 <= x1 <= max(ow, cw) - cw or not 0 <= y1 <= max(oh, ch) - ch:
                raise ValueError(f"SegAugmenter: item {b}: crop ({x1}, {y1}) of {cw}x{ch} outside the padded {ow}x{oh} image")
            items[b] = self._item(self.cache, i, p["flip"], ow, oh, x1, y1, cw, ch, cw, ch, p["order"], p["factors"], tables)
        return self._launch(items, tables, B, ch, cw, ch, cw, out_dtype)

    def __call__(self, indices, out_dtype=torch.float32):
        """one mode='train' batch: (images (B, 3, h, w) of out_dtype, labels (B, h, w) int64) on the current CUDA device / stream"""
        params = [self.draw(i) for i in indices]
        return self.build(indices, params, out_dtype)

    def testval(self, indices, out_dtype=torch.float32):
        """mode='testval' items (`_testval_img_transform` + ToTensor, `_mask_transform` at native size): (images (B, 3, oh, ow), labels
        (B, H, W) int64), the long side resized to make_divisible(base_size, 32) and the short side to a multiple of 32 by Pillow's
        bilinear resize.  The items of one call must share their source size, as default_collate requires."""
        shapes = {self.cache.shapes[i] for i in indices}
        if len(shapes) != 1:
            raise ValueError(f"SegAugmenter.testval: items of one batch must share a source size, got {sorted(shapes)}")
        H0, W0 = shapes.pop()
        outlong = math.ceil(self.base_size / 32) * 32
        if W0 > H0:
            ow, oh = outlong, math.ceil(int(1.0 * H0 * outlong / W0) / 32) * 32
        else:
            oh, ow = outlong, math.ceil(int(1.0 * W0 * outlong / H0) / 32) * 32
        B = len(indices)
        items, tables = (_lib.SegItem * B)(), []
        for b, i in enumerate(indices):
            items[b] = self._item(self.cache, i, False, ow, oh, 0, 0, ow, oh, W0, H0, [], [None] * 4, tables, mask_size=(W0, H0))
        return self._launch(items, tables, B, oh, ow, H0, W0, out_dtype)

    def val(self, indices, crop_size, out_dtype=torch.float32):
        """mode='val' items (`_val_sync_transform` + ToTensor, the item's mask map): (images (B, 3, c, c), labels (B, c, c) int64) with
        c = crop_size.  Each item's short side is resized to c by Pillow's bilinear resize (the mask by NEAREST) and the c x c centre
        crop taken (seg_val_geometry), so sources of different sizes share a batch.  Draws nothing from `random` or torch."""
        c = seg_val_crop(crop_size)
        if out_dtype not in (torch.uint8, torch.float16, torch.float32):
            raise ValueError(f"SegAugmenter: out_dtype must be uint8, float16 or float32, got {out_dtype}")
        B = len(indices)
        items, tables = (_lib.SegItem * B)(), []
        for b, i in enumerate(indices):
            H0, W0 = self.cache.shapes[i]
            ow, oh, x1, y1 = seg_val_geometry(W0, H0, c)
            items[b] = self._item(self.cache, i, False, ow, oh, x1, y1, c, c, c, c, [], [None] * 4, tables)
        return self._launch(items, tables, B, c, c, c, c, out_dtype)


def seg_val_crop(crop_size):
    """the int crop_size of mode='val'; a tuple (the default of get_citys_loader / get_citysbdd_loader, and what get_custom_loader always
    passes) raises ValueError, where the reference's `_val_sync_transform` raises TypeError multiplying the tuple"""
    if isinstance(crop_size, (tuple, list)):
        raise ValueError(f"mode='val' needs an int crop_size, got {crop_size!r}: the reference's _val_sync_transform raises TypeError "
                         "on a tuple crop_size (the default of get_citys_loader / get_citysbdd_loader and what get_custom_loader passes)")
    if isinstance(crop_size, bool) or not isinstance(crop_size, (int, np.integer)) or crop_size <= 0:
        raise ValueError(f"mode='val' needs a positive int crop_size, got {crop_size!r}")
    return int(crop_size)


def seg_val_geometry(w, h, crop):
    """(ow, oh, x1, y1) of the reference's `_val_sync_transform` (SegmentationDataset.py:96-116) for a w x h source: the short side
    resized to `crop` and the long side to int(1.0 * long * crop / short) (a square goes the portrait way), then the crop x crop centre
    crop at int(round((ow - crop) / 2.)), Python's round half to even, and the same for y1"""
    if w > h:
        oh = crop
        ow = int(1.0 * w * oh / h)
    else:
        ow = crop
        oh = int(1.0 * h * ow / w)
    return ow, oh, int(round((ow - crop) / 2.)), int(round((oh - crop) / 2.))
