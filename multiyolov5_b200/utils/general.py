"""Post-process of the hot path behind the reference's names (reference utils/general.py, detect.py:191-193)."""
import ctypes as C
import math

import numpy as np
import torch

from .. import _lib

_ws_cache = {}


def xywh2xyxy(x):  # reference utils/general.py:265-272 (host-side helper kept for callers; NMS does this on the device)
    y = x.clone()
    y[:, 0] = x[:, 0] - x[:, 2] / 2
    y[:, 1] = x[:, 1] - x[:, 3] / 2
    y[:, 2] = x[:, 0] + x[:, 2] / 2
    y[:, 3] = x[:, 1] + x[:, 3] / 2
    return y


def xyxy2xywh(x):  # reference utils/general.py:254-262
    y = x.clone()
    y[:, 0] = (x[:, 0] + x[:, 2]) / 2
    y[:, 1] = (x[:, 1] + x[:, 3]) / 2
    y[:, 2] = x[:, 2] - x[:, 0]
    y[:, 3] = x[:, 3] - x[:, 1]
    return y


def clip_coords(boxes, img_shape):
    """in place, like the reference (utils/general.py:334-340): xyxy boxes clipped to (height, width)"""
    boxes[:, 0].clamp_(0, img_shape[1])
    boxes[:, 1].clamp_(0, img_shape[0])
    boxes[:, 2].clamp_(0, img_shape[1])
    boxes[:, 3].clamp_(0, img_shape[0])


def scale_coords(img1_shape, coords, img0_shape, ratio_pad=None):
    """xyxy boxes from the letterboxed network input back to the original frame, IN PLACE on the caller's tensor (reference
    utils/general.py:319-331, called on NMS output rows at detect.py:169; the rows returned by non_max_suppression are ordinary
    writable tensors for exactly this reason)."""
    if ratio_pad is None:
        gain = min(img1_shape[0] / img0_shape[0], img1_shape[1] / img0_shape[1])
        pad = (img1_shape[1] - img0_shape[1] * gain) / 2, (img1_shape[0] - img0_shape[0] * gain) / 2
    else:
        gain, pad = ratio_pad[0][0], ratio_pad[1]
    coords[:, [0, 2]] -= pad[0]
    coords[:, [1, 3]] -= pad[1]
    coords[:, :4] /= gain
    clip_coords(coords, img0_shape)
    return coords


def box_iou(box1, box2):
    """(N,4) x (M,4) xyxy -> (N,M) IoU (reference utils/general.py:388-410)"""
    area1 = (box1[:, 2] - box1[:, 0]) * (box1[:, 3] - box1[:, 1])
    area2 = (box2[:, 2] - box2[:, 0]) * (box2[:, 3] - box2[:, 1])
    inter = (torch.min(box1[:, None, 2:], box2[:, 2:]) - torch.max(box1[:, None, :2], box2[:, :2])).clamp(0).prod(2)
    return inter / (area1[:, None] + area2 - inter)


# ---- --image-weights (reference utils/general.py:216-240, train.py:255,305-316; csrc/image_weights.cu) ----
_IW_ERRORS = ((_lib.IW_BAD_CLASS, "labels_to_image_weights: a label's class is outside [0, nc)"),
              (_lib.IW_TOTAL_NONPOS, "Total of weights must be greater than zero"),      # random.choices' own messages
              (_lib.IW_TOTAL_NONFINITE, "Total of weights must be finite"))


def iw_status_error(status):
    """the ValueError for a nonzero image-weights status word (a bad class first, as bincount raises before random.choices)"""
    return next(ValueError(msg) for bit, msg in _IW_ERRORS if status & bit)


def label_classes(labels, device=None):
    """the float32 class column of every image's (k, 5) labels, concatenated, and each image's [start, end) in it ((n + 1) int64), both
    uploaded to the device once"""
    cols = [np.asarray(x, np.float32).reshape(-1, 5)[:, 0] for x in labels]
    offsets = np.zeros(len(cols) + 1, np.int64)
    np.cumsum([len(c) for c in cols], out=offsets[1:])
    dev = device or torch.device("cuda", torch.cuda.current_device())
    cls = torch.from_numpy(np.concatenate(cols) if cols else np.zeros(0, np.float32)).to(dev)
    return cls, torch.from_numpy(offsets).to(dev)


def _nc(nc):
    if not 1 <= int(nc) <= _lib.IW_NC_MAX:
        raise ValueError(f"nc = {nc}: image weights are built for 1 <= nc <= {_lib.IW_NC_MAX}")
    return int(nc)


def labels_to_class_weights(labels, nc=80):
    """the reference's labels_to_class_weights on the device, bit for bit: inverse class frequencies (empty classes count 1), normalised
    by numpy's sum over nc.  Returns a float64 CUDA tensor of nc (the reference returns a CPU one; train.py moves it with `.to(device)`
    and multiplies it by nc).  A class outside [0, nc) raises ValueError.  Reads one status word back."""
    if labels[0] is None:
        return torch.Tensor()
    nc = _nc(nc)
    cls, _ = label_classes(labels)
    counts = torch.empty(nc, dtype=torch.int64, device=cls.device)
    w = torch.empty(nc, dtype=torch.float64, device=cls.device)
    status = torch.zeros(1, dtype=torch.int32, device=cls.device)
    _lib.check(_lib.lib().myolo_class_weights(_lib.ptr(cls), cls.numel(), nc, _lib.ptr(counts), _lib.ptr(w), _lib.ptr(status),
                                              _lib.stream_ptr()))
    if int(status.item()):
        raise iw_status_error(int(status.item()))
    return w


def device_image_weights(cls, offsets, cw, status):
    """myolo_image_weights over uploaded labels (label_classes) for the nc class weights `cw` (float64 numpy): a float64 CUDA tensor of
    the n image weights; a bad class ORs the status word"""
    cw = np.ascontiguousarray(cw, np.float64)
    nc = _nc(cw.size)
    n = offsets.numel() - 1
    cw_d = torch.from_numpy(cw).to(cls.device)
    iw = torch.empty(n, dtype=torch.float64, device=cls.device)
    _lib.check(_lib.lib().myolo_image_weights(_lib.ptr(cls), _lib.ptr(offsets), n, _lib.ptr(cw_d), nc, _lib.ptr(iw), _lib.ptr(status),
                                              _lib.stream_ptr()))
    return iw


def labels_to_image_weights(labels, nc=80, class_weights=np.ones(80)):
    """the reference's labels_to_image_weights on the device, bit for bit: per image, the sum over nc of class_weights * its label count
    per class, in numpy's order.  Returns a float64 numpy array of len(labels).  A class outside [0, nc) raises ValueError."""
    cw = np.asarray(class_weights, np.float64).reshape(nc)
    cls, offsets = label_classes(labels)
    status = torch.zeros(1, dtype=torch.int32, device=cls.device)
    iw = device_image_weights(cls, offsets, cw, status)
    if int(status.item()):
        raise iw_status_error(int(status.item()))
    return iw.cpu().numpy()


def strip_optimizer(f="best.pt", s=""):
    """reference utils/general.py:512-525: finalise a training checkpoint - EMA becomes the model, optimiser state dropped, fp16, frozen"""
    import os
    from ..models.experimental import load_checkpoint
    x = load_checkpoint(f, map_location=torch.device("cpu"))
    if x.get("ema"):
        x["model"] = x["ema"]
    for k in ("optimizer", "training_results", "wandb_id", "ema", "updates"):
        x[k] = None
    x["epoch"] = -1
    x["model"].half()
    for p in x["model"].parameters():
        p.requires_grad = False
    torch.save(x, s or f)
    mb = os.path.getsize(s or f) / 1e6
    print(f"Optimizer stripped from {f},{(' saved as %s,' % s) if s else ''} {mb:.1f}MB")


def init_seeds(seed=0):
    """reference utils/general.py:39-43 with torch_utils.init_torch_seeds: seeds `random`, `numpy.random` and torch's default generator;
    seed 0 asks cuDNN for determinism, any other seed for its benchmark mode"""
    import random
    random.seed(seed)
    np.random.seed(seed)
    torch.manual_seed(seed)
    torch.backends.cudnn.benchmark, torch.backends.cudnn.deterministic = (False, True) if seed == 0 else (True, False)


def print_mutation(hyp, results, yaml_file="hyp_evolved.yaml", evolve_txt="evolve.txt"):
    """--evolve's record of one generation (reference utils/general.py:528-556, without the gsutil bucket): prints the hyp and the 7
    results, appends them to evolve_txt, rewrites it as its unique rows sorted by fitness ('%10.3g'), and writes the best row's
    hyper-parameters to yaml_file under a header with the generation count and its results"""
    import yaml
    from .metrics import fitness
    a = "%10s" * len(hyp) % tuple(hyp.keys())
    b = "%10.3g" * len(hyp) % tuple(hyp.values())
    c = "%10.4g" * len(results) % tuple(results)
    print("\n%s\n%s\nEvolved fitness: %s\n" % (a, b, c))
    with open(evolve_txt, "a") as f:
        f.write(c + b + "\n")
    x = np.unique(np.loadtxt(evolve_txt, ndmin=2), axis=0)
    x = x[np.argsort(-fitness(x))]
    np.savetxt(evolve_txt, x, "%10.3g")
    for i, k in enumerate(hyp.keys()):
        hyp[k] = float(x[0, i + 7])
    with open(yaml_file, "w") as f:
        best = tuple(x[0, :7])
        f.write("# Hyperparameter Evolution Results\n# Generations: %g\n# Metrics: " % len(x) + "%10.4g" * len(best) % best + "\n\n")
        yaml.dump(hyp, f, sort_keys=False)


def one_cycle(y1=0.0, y2=1.0, steps=100):
    """the cosine ramp from y1 at x = 0 to y2 at x = steps of reference utils/general.py:186-188, its operations in its order so that
    every float is the reference's"""
    def f(x):
        return ((1 - math.cos(x * math.pi / steps)) / 2) * (y2 - y1) + y1
    return f


def coco80_to_coco91_class():
    """COCO category ids (1..90 with the ten ids the 2017 detection set leaves unused) of the 80 contiguous class indices"""
    return [i for i in range(1, 91) if i not in (12, 26, 29, 30, 45, 66, 68, 69, 71, 83)]


class NmsLabels:
    """Apriori labels for non_max_suppression(labels=...) packed for the device (utils/general.py:448-455, test.py --save-hybrid).

        rows      (n, 5) fp32 [cls, x, y, w, h] in network-input pixels, image b's rows at rows[offsets[b]:offsets[b + 1]]
        offsets   (B + 1) int32
        max_labels  a bound on any image's label count (n is always one)
        err       (1,) int32 device word the NMS ORs MYOLO_NMS_ERR_* bits into; check() reads it

    `from_targets` builds it from collate_fn targets on the device without a host round trip, as test.py:175-176 does."""

    def __init__(self, rows, offsets, max_labels, err=None):
        self.rows = rows.float().contiguous()
        self.offsets = offsets.to(torch.int32).contiguous()
        self.max_labels = int(max_labels)
        self.err = err if err is not None else torch.zeros(1, dtype=torch.int32, device=self.rows.device)

    @classmethod
    def from_targets(cls, targets, batch_size, img_hw, err=None):
        """test.py:175-176: targets (n, 6) [image, class, x, y, w, h] normalised, scaled to pixels by (w, h) in fp32; each image's rows
        keep their order (targets[targets[:, 0] == i, 1:])"""
        t = targets.float().reshape(-1, 6)
        height, width = img_hw
        scale = torch.tensor([1.0, width, height, width, height], dtype=torch.float32, device=t.device)
        img, order = torch.sort(t[:, 0], stable=True)
        rows = t[order, 1:] * scale
        offsets = torch.searchsorted(img.contiguous(), torch.arange(batch_size + 1, dtype=torch.float32, device=t.device))
        return cls(rows, offsets, t.shape[0], err)

    @classmethod
    def from_list(cls, labels, nc, device):
        """the reference's per-image list of (k, 5) [cls, x, y, w, h] tensors; class ids are checked on the host (an id outside [0, nc)
        is an index error in the reference)"""
        ls = [torch.as_tensor(l, dtype=torch.float32).reshape(-1, 5) for l in labels]
        rows = torch.cat(ls).to(device) if ls else torch.zeros((0, 5), device=device)
        c = rows[:, 0].cpu()
        if len(c) and not bool(((c > -1) & (c < nc)).all()):
            raise ValueError(f"label class ids must be in [0, {nc})")
        sizes = [len(l) for l in ls]
        offsets = torch.tensor(np.concatenate([[0], np.cumsum(sizes)]), dtype=torch.int32).to(device)
        return cls(rows, offsets, max(sizes, default=0))

    def check(self):
        """reads the error word (one synchronisation) and raises on a bad label"""
        check_nms_labels_error(int(self.err.item()))


def check_nms_labels_error(e):
    """raises for the MYOLO_NMS_ERR_* bits of a myolo_nms_labels error word"""
    if e & _lib.NMS_ERR_LABEL_CLASS:
        raise ValueError("a label class id is outside [0, nc)")
    if e & _lib.NMS_ERR_LABEL_COUNT:
        raise ValueError("an image has more labels than max_labels")


def non_max_suppression(prediction, conf_thres=0.25, iou_thres=0.45, classes=None, agnostic=False, multi_label=False, labels=(),
                        max_det=300, return_padded=False):
    """reference utils/general.py:421-509.  prediction: (B,A,5+nc) fp32 CUDA.  Returns list[(n,6)] like the reference
    ([x1,y1,x2,y2,conf,cls], descending conf, <=300 rows).  `labels`: the reference's per-image list of (k, 5) [cls, x, y, w, h] apriori
    labels (autolabelling), or an NmsLabels; with an NmsLabels and return_padded its error word is left to the caller's check()."""
    if not prediction.is_cuda:
        raise _lib.MyoloError("non_max_suppression needs a CUDA tensor: there is no CPU path in multiyolov5_b200")
    pred = prediction.float().contiguous()
    B, A, no = pred.shape
    L = _lib.lib()
    ml = bool(multi_label) and (no - 5) > 1
    lab = None
    if isinstance(labels, NmsLabels):
        lab = labels
    elif labels is not None and len(labels):
        if len(labels) != B:
            raise ValueError("labels: one (k, 5) entry per image")
        lab = NmsLabels.from_list(labels, no - 5, pred.device)
    if lab is not None:
        if lab.offsets.numel() != B + 1:
            raise ValueError("labels: offsets must have B + 1 entries")
        nbytes = int(L.myolo_nms_labels_workspace_bytes(B, A, no, int(ml), lab.max_labels))
    else:
        nbytes = int(L.myolo_nms_workspace_bytes(B, A, no, int(ml)))
    key = (pred.device, nbytes)
    ws = _ws_cache.get(key)
    if ws is None:
        _ws_cache.clear()
        ws = _ws_cache[key] = torch.empty(nbytes, dtype=torch.uint8, device=pred.device)
    out = torch.zeros((B, max_det, 6), dtype=torch.float32, device=pred.device)
    cnt = torch.empty((B,), dtype=torch.int32, device=pred.device)
    cls_t = torch.tensor(list(classes), dtype=torch.int32, device=pred.device) if classes is not None else None
    if lab is None:
        _lib.check(L.myolo_nms(_lib.ptr(pred), B, A, no, float(conf_thres), float(iou_thres), _lib.ptr(cls_t),
                               0 if cls_t is None else cls_t.numel(), int(bool(agnostic)), int(ml), int(max_det), 30000, 4096.0,
                               _lib.ptr(out), _lib.ptr(cnt), _lib.ptr(ws), nbytes, _lib.stream_ptr()))
    else:
        _lib.check(L.myolo_nms_labels(_lib.ptr(pred), B, A, no, float(conf_thres), float(iou_thres), _lib.ptr(cls_t),
                                      0 if cls_t is None else cls_t.numel(), int(bool(agnostic)), int(ml), int(max_det), 30000, 4096.0,
                                      _lib.ptr(lab.rows) if lab.rows.numel() else None, _lib.ptr(lab.offsets), lab.max_labels,
                                      _lib.ptr(lab.err), _lib.ptr(out), _lib.ptr(cnt), _lib.ptr(ws), nbytes, _lib.stream_ptr()))
    if return_padded:
        return out, cnt
    if lab is not None:
        lab.check()
    counts = cnt.tolist()  # the one device->host sync, like the reference's shape checks (utils/general.py:458,484)
    return [out[b, :counts[b]] for b in range(B)]


def seg_argmax(seg, out_hw=None, out_dtype=torch.int64):
    """detect.py:191-193: F.interpolate(seg,(H0,W0),bilinear,align_corners=True) then argmax over classes, fused.
    seg: (B,C,h,w) fp32/fp16 CUDA -> (B,H0,W0) int64 (or uint8)."""
    if not seg.is_cuda:
        raise _lib.MyoloError("seg_argmax needs a CUDA tensor")
    seg = seg.contiguous()
    B, Cc, h, w = seg.shape
    H, W = out_hw if out_hw is not None else (h, w)
    out = torch.empty((B, H, W), dtype=out_dtype, device=seg.device)
    _lib.check(_lib.lib().myolo_seg_upsample_argmax(_lib.ptr(seg), _lib.torch_dtype_code(seg.dtype), B, Cc, h, w, H, W, _lib.ptr(out),
                                                    _lib.torch_dtype_code(out_dtype), _lib.stream_ptr()))
    return out


def bilinear_align_corners(seg, out_hw):
    seg = seg.float().contiguous()
    B, Cc, h, w = seg.shape
    out = torch.empty((B, Cc, out_hw[0], out_hw[1]), dtype=torch.float32, device=seg.device)
    _lib.check(_lib.lib().myolo_bilinear_nchw(_lib.ptr(seg), B, Cc, h, w, out_hw[0], out_hw[1], _lib.ptr(out), _lib.stream_ptr()))
    return out


# ---- seg output consumers (SURVEY.md section 8f rank 2; reference detect.py:69-77,193-194,206) ----
# standard Cityscapes trainId palette (RGB) and trainId -> labelId table, the data of detect.py:19-61
Cityscapes_COLORMAP = [[128, 64, 128], [244, 35, 232], [70, 70, 70], [102, 102, 156], [190, 153, 153], [153, 153, 153], [250, 170, 30],
                       [220, 220, 0], [107, 142, 35], [152, 251, 152], [0, 130, 180], [220, 20, 60], [255, 0, 0], [0, 0, 142], [0, 0, 70],
                       [0, 60, 100], [0, 80, 100], [0, 0, 230], [119, 11, 32]]
Cityscapes_IDMAP = [[7], [8], [11], [12], [13], [17], [19], [20], [21], [22], [23], [24], [25], [26], [27], [28], [31], [32], [33]]
_lut_cache = {}


def _lut(table, device):
    key = (id(table), str(device))
    if key not in _lut_cache:
        _lut_cache[key] = torch.tensor(table, dtype=torch.uint8, device=device).contiguous()
    return _lut_cache[key]


def _lut_call(pred, table, reverse, image=None, alpha=0.0, beta=0.0, want_out=True, table2=None):
    assert pred.is_cuda and pred.dtype in (torch.uint8, torch.int64), "class map: CUDA uint8 / int64 tensor"
    pred = pred.contiguous()
    lut = _lut(table, pred.device)
    n_entries, ch = lut.shape
    out = torch.empty(tuple(pred.shape) + (ch,), dtype=torch.uint8, device=pred.device) if want_out else None
    blend = None
    if image is not None:
        image = image.contiguous()
        assert image.dtype == torch.uint8 and tuple(image.shape) == tuple(pred.shape) + (ch,) and image.is_cuda
        blend = torch.empty_like(image)
    lut2 = out2 = None
    if table2 is not None:
        lut2 = _lut(table2, pred.device)
        assert lut2.shape[0] == n_entries, "the second table needs as many entries as the first"
        out2 = torch.empty(tuple(pred.shape) + (lut2.shape[1],), dtype=torch.uint8, device=pred.device)
    _lib.check(_lib.lib().myolo_seg_lut_blend(_lib.ptr(pred), _lib.torch_dtype_code(pred.dtype), pred.numel(), _lib.ptr(lut), n_entries, ch,
                                              int(reverse), _lib.ptr(out), _lib.ptr(image), float(alpha), float(beta), _lib.ptr(blend),
                                              _lib.ptr(lut2), 0 if lut2 is None else lut2.shape[1], _lib.ptr(out2), _lib.stream_ptr()))
    return (out, blend) if table2 is None else (out, blend, out2)


def label2image(pred, COLORMAP=Cityscapes_COLORMAP):
    """class ids (H,W) -> (H,W,3) uint8 colours (reference detect.py:69-72), on the device"""
    return _lut_call(pred, COLORMAP, False)[0]


def trainid2id(pred, IDMAP=Cityscapes_IDMAP):
    """trainIds -> Cityscapes label ids (H,W,1) uint8 (reference detect.py:74-77), on the device"""
    return _lut_call(pred, IDMAP, False)[0]


def seg_products(pred, im0=None, mask=True, ids=False, COLORMAP=Cityscapes_COLORMAP, IDMAP=Cityscapes_IDMAP, alpha=0.4, beta=0.6):
    """detect.py:193-194,206 in one pass over the class map: the BGR `mask`, the blend cv2.addWeighted(mask, alpha, im0, beta, 0) when
    im0 is given and the trainid2id label `ids` (H,W,1), each only when asked for.  pred: (..., H, W) uint8 / int64 class map, im0:
    (..., H, W, 3) uint8 BGR frames, both on the GPU.  Returns (mask, dst, ids), None for each product not asked for."""
    if not (mask or im0 is not None or ids):
        raise ValueError("seg_products: ask for at least one of mask, blend (im0) and ids")
    out = _lut_call(pred, COLORMAP, True, image=im0, alpha=alpha, beta=beta, want_out=mask, table2=IDMAP if ids else None)
    return out if ids else out + (None,)


def seg_overlay(pred, im0, COLORMAP=Cityscapes_COLORMAP, alpha=0.4, beta=0.6):
    """detect.py:193-194 in one kernel: mask = label2image(pred)[:, :, ::-1] (BGR) and dst = cv2.addWeighted(mask, alpha, im0, beta, 0).
    pred: (H,W) class map, im0: (H,W,3) uint8 BGR frame, both on the GPU.  Returns (mask, dst)."""
    return _lut_call(pred, COLORMAP, True, image=im0, alpha=alpha, beta=beta)


# ---- detect.py (reference utils/general.py:123-128,594-604; detect.py:166-177) ----
def check_img_size(img_size, s=32):
    """reference utils/general.py:123-128: img_size rounded up to a multiple of the stride s, with the reference's warning"""
    from ..models.yolo import make_divisible
    new_size = make_divisible(img_size, int(s))
    if new_size != img_size:
        print("WARNING: --img-size %g must be multiple of max stride %g, updating to %g" % (img_size, s, new_size))
    return new_size


def increment_path(path, exist_ok=True, sep=""):
    """reference utils/general.py:594-604: runs/exp stays runs/exp when it is free (or exist_ok), else runs/exp{sep}N for one more than
    the largest N already there (2 when there is none)"""
    import glob
    import re
    from pathlib import Path
    path = Path(path)
    if (path.exists() and exist_ok) or (not path.exists()):
        return str(path)
    dirs = glob.glob(f"{path}{sep}*")
    matches = [re.search(rf"%s{sep}(\d+)" % path.stem, d) for d in dirs]
    i = [int(m.groups()[0]) for m in matches if m]
    n = max(i) + 1 if i else 2
    return f"{path}{sep}{n}"


def scale_coords_geometry(img1_shape, img0_shape):
    """the Python scalars of scale_coords(img1_shape, ., img0_shape) (float64, the reference's order) rounded to fp32 as torch's CPU
    kernels round a scalar operand: float32 (B=1, 5) row {pad_x, pad_y, gain, w0, h0} of myolo_detect_boxes"""
    gain = min(img1_shape[0] / img0_shape[0], img1_shape[1] / img0_shape[1])
    pad = (img1_shape[1] - img0_shape[1] * gain) / 2, (img1_shape[0] - img0_shape[0] * gain) / 2
    return np.array([pad[0], pad[1], gain, img0_shape[1], img0_shape[0]], np.float32)


def detect_boxes(rows, counts, geom, nc=None, xywhn=False):
    """detect.py:166-177 for a batch in one launch: rows (B, max_det, 6) fp32 CUDA padded NMS rows (non_max_suppression(...,
    return_padded=True)) and counts (B,) int32 -> rows[b, :counts[b], :4] = scale_coords(...).round() IN PLACE, bit for bit torch's CPU
    fp32.  geom: (B, 5) fp32 rows of scale_coords_geometry (host or device).  Returns (xywhn, class_counts): the (B, max_det, 4)
    normalised xywh of --save-txt when xywhn, the (B, nc) int32 per-class row counts of the printed line when nc is given; None otherwise."""
    if not (rows.is_cuda and rows.dtype == torch.float32 and rows.is_contiguous() and rows.dim() == 3 and rows.shape[2] == 6):
        raise _lib.MyoloError("detect_boxes needs contiguous (B, max_det, 6) fp32 CUDA rows")
    B, max_det, _ = rows.shape
    counts = counts.to(device=rows.device, dtype=torch.int32).contiguous()
    geom = torch.as_tensor(geom, dtype=torch.float32).reshape(B, 5).to(rows.device, non_blocking=True).contiguous()
    wh = torch.empty((B, max_det, 4), dtype=torch.float32, device=rows.device) if xywhn else None
    cc = torch.empty((B, int(nc)), dtype=torch.int32, device=rows.device) if nc is not None else None
    _lib.check(_lib.lib().myolo_detect_boxes(_lib.ptr(rows), _lib.ptr(counts), B, max_det, _lib.ptr(geom), 0 if nc is None else int(nc),
                                             _lib.ptr(wh), _lib.ptr(cc), _lib.stream_ptr()))
    return wh, cc


# ---- autoShape (reference models/common.py:661-672,680-688) ----
# include/myolo.h myolo_seg_crop_item
SEG_CROP_ITEM = np.dtype([("offset", "<i8"), ("top", "<i4"), ("left", "<i4"), ("rh", "<i4"), ("rw", "<i4"), ("h0", "<i4"), ("w0", "<i4")])


def scale_boxes(rows, counts, geom):
    """autoShape's `scale_coords(shape1, y[i][:, :4], shape0[i])` for a batch in one launch: rows (B, max_det, 6) fp32 CUDA padded NMS
    rows (non_max_suppression(..., return_padded=True)), rows[b, :counts[b], :4] scaled IN PLACE without rounding, bit for bit torch's
    CPU fp32.  geom: (B, 5) fp32 rows of scale_coords_geometry (host or device).  Returns Detections' (xywh, xyxyn, xywhn) as
    (B, max_det, 6) fp32 tensors, valid for the same rows."""
    if not (rows.is_cuda and rows.dtype == torch.float32 and rows.is_contiguous() and rows.dim() == 3 and rows.shape[2] == 6):
        raise _lib.MyoloError("scale_boxes needs contiguous (B, max_det, 6) fp32 CUDA rows")
    B, max_det, _ = rows.shape
    counts = counts.to(device=rows.device, dtype=torch.int32).contiguous()
    geom = torch.as_tensor(geom, dtype=torch.float32).reshape(B, 5).to(rows.device, non_blocking=True).contiguous()
    xywh, xyxyn, xywhn = (torch.empty_like(rows) for _ in range(3))
    _lib.check(_lib.lib().myolo_scale_boxes(_lib.ptr(rows), _lib.ptr(counts), B, max_det, _lib.ptr(geom), _lib.ptr(xywh), _lib.ptr(xyxyn),
                                            _lib.ptr(xywhn), _lib.stream_ptr()))
    return xywh, xyxyn, xywhn


def seg_crop_item_table(windows, shapes0):
    """the myolo_seg_crop_item table: windows (top, left, rh, rw) of the letterboxed images, shapes0 (h0, w0) the class map sizes, packed
    one after the other"""
    t = np.zeros(len(shapes0), SEG_CROP_ITEM)
    off = 0
    for k, ((top, left, rh, rw), (h0, w0)) in enumerate(zip(windows, shapes0)):
        t[k] = (off, top, left, rh, rw, h0, w0)
        off += h0 * w0
    return t


def seg_crop_argmax(seg, items, shapes0):
    """autoShape's class maps in one launch: for image i, F.interpolate(seg[i:i+1, :, top:top+rh, left:left+rw], shapes0[i], 'bilinear',
    align_corners=True).argmax(1) as a uint8 (h0, w0) CUDA tensor, all views of one packed buffer.  seg: (B,C,H,W) fp32 / fp16 CUDA
    logits; items: CUDA uint8 bytes of the seg_crop_item_table (its windows must lie inside H x W)."""
    if not (seg.is_cuda and items.is_cuda and seg.dim() == 4 and items.numel() == seg.shape[0] * SEG_CROP_ITEM.itemsize):
        raise _lib.MyoloError("seg_crop_argmax needs (B,C,H,W) CUDA logits and a CUDA table of B items")
    seg = seg.contiguous()
    B, Cc, H, W = seg.shape
    sizes = [int(h) * int(w) for h, w in shapes0]
    out = torch.empty(sum(sizes), dtype=torch.uint8, device=seg.device)
    _lib.check(_lib.lib().myolo_seg_crop_upsample_argmax(_lib.ptr(seg), _lib.torch_dtype_code(seg.dtype), B, Cc, H, W, _lib.ptr(items),
                                                         max(sizes), _lib.ptr(out), _lib.stream_ptr()))
    return [m.view(int(h), int(w)) for m, (h, w) in zip(out.split(sizes), shapes0)]
