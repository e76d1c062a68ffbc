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


def non_max_suppression(prediction, conf_thres=0.25, iou_thres=0.45, classes=None, agnostic=False, multi_label=False, labels=(),
                        max_det=300, return_padded=False):
    """reference utils/general.py:421-509.  prediction: (B,A,5+nc) fp32 CUDA.  Returns list[(n,6)] like the reference
    ([x1,y1,x2,y2,conf,cls], descending conf, <=300 rows).  `labels` (auto-labelling apriori boxes) is not on the hot path."""
    if labels:
        raise NotImplementedError("non_max_suppression(labels=...) (autolabelling) is out of scope (SURVEY.md section 8)")
    if not prediction.is_cuda:
        raise _lib.MyoloError("non_max_suppression needs a CUDA tensor: there is no CPU path in multiyolov5_b200")
    pred = prediction.float().contiguous()
    B, A, no = pred.shape
    L = _lib.lib()
    ml = bool(multi_label) and (no - 5) > 1
    nbytes = int(L.myolo_nms_workspace_bytes(B, A, no, int(ml)))
    key = (pred.device, nbytes)
    ws = _ws_cache.get(key)
    if ws is None:
        _ws_cache.clear()
        ws = _ws_cache[key] = torch.empty(nbytes, dtype=torch.uint8, device=pred.device)
    out = torch.zeros((B, max_det, 6), dtype=torch.float32, device=pred.device)
    cnt = torch.empty((B,), dtype=torch.int32, device=pred.device)
    cls_t = torch.tensor(list(classes), dtype=torch.int32, device=pred.device) if classes is not None else None
    _lib.check(L.myolo_nms(_lib.ptr(pred), B, A, no, float(conf_thres), float(iou_thres), _lib.ptr(cls_t),
                           0 if cls_t is None else cls_t.numel(), int(bool(agnostic)), int(ml), int(max_det), 30000, 4096.0,
                           _lib.ptr(out), _lib.ptr(cnt), _lib.ptr(ws), nbytes, _lib.stream_ptr()))
    if return_padded:
        return out, cnt
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


def _lut_call(pred, table, reverse, image=None, alpha=0.0, beta=0.0, want_out=True):
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
    _lib.check(_lib.lib().myolo_seg_lut_blend(_lib.ptr(pred), _lib.torch_dtype_code(pred.dtype), pred.numel(), _lib.ptr(lut), n_entries, ch,
                                              int(reverse), _lib.ptr(out), _lib.ptr(image), float(alpha), float(beta), _lib.ptr(blend),
                                              _lib.stream_ptr()))
    return out, blend


def label2image(pred, COLORMAP=Cityscapes_COLORMAP):
    """class ids (H,W) -> (H,W,3) uint8 colours (reference detect.py:69-72), on the device"""
    return _lut_call(pred, COLORMAP, False)[0]


def trainid2id(pred, IDMAP=Cityscapes_IDMAP):
    """trainIds -> Cityscapes label ids (H,W,1) uint8 (reference detect.py:74-77), on the device"""
    return _lut_call(pred, IDMAP, False)[0]


def seg_overlay(pred, im0, COLORMAP=Cityscapes_COLORMAP, alpha=0.4, beta=0.6):
    """detect.py:193-194 in one kernel: mask = label2image(pred)[:, :, ::-1] (BGR) and dst = cv2.addWeighted(mask, alpha, im0, beta, 0).
    pred: (H,W) class map, im0: (H,W,3) uint8 BGR frame, both on the GPU.  Returns (mask, dst)."""
    return _lut_call(pred, COLORMAP, True, image=im0, alpha=alpha, beta=beta)
