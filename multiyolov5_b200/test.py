"""Validation passes behind the reference's names (reference test.py): `test` (the training path of test.py:77-340) and `seg_validation`
(test.py:31-65).  A pass stays on the device from the uint8 batch to a few per-class numbers: per batch one forward, one NMS and one
matching launch (utils.metrics.DetectionStats), with no host synchronisation; ap_per_class runs once at the end.

The reference validates in fp16 on CUDA (its z, NMS rows and box_iou are half tensors); this model keeps z in fp32, so the statistics
equal the reference's fp32 statistics of the same predictions, which is what its test() computes on a CPU device.

The batches can come from the device as well: `test(data, model=m, dataloader=DetValLoader(cache, 32), plots=False)` with
`cache = utils.datasets.DeviceImageCache(frames, imgsz, labels, augment=False)` is the reference's rect validation loader of
train.py:207-210 (`create_dataloader(..., rect=True, pad=0.5)`), bit exact with it.
"""
from pathlib import Path

import numpy as np
import torch

from . import _lib
from .utils.general import non_max_suppression
from .utils.metrics import DetectionStats, _class_map


def test(data, weights=None, batch_size=32, imgsz=640, conf_thres=0.001, iou_thres=0.6, save_json=False, single_cls=False, augment=False,
         verbose=False, model=None, dataloader=None, save_dir=Path(""), save_txt=False, save_hybrid=False, save_conf=False, plots=True,
         wandb_logger=None, compute_loss=None, half_precision=True, is_coco=False):
    """Returns ((mp, mr, map50, map, *loss), maps, t) like the reference.  `dataloader` yields collate_fn tuples
    (img uint8 (B,3,H,W), targets (n,6), paths, shapes) on the host or the device.  Prints the `all` row (and per-class rows with
    verbose).  t = (forward, NMS, total) ms per image from CUDA events, then (imgsz, imgsz, batch_size)."""
    if model is None:
        raise NotImplementedError("test(model=None): loading weights and data files is not built; pass model= and dataloader=")
    for flag, name in ((save_json, "save_json"), (save_txt, "save_txt"), (save_hybrid, "save_hybrid"), (augment, "augment"),
                       (plots, "plots (the confusion matrix and plots)"), (wandb_logger, "a W&B logger")):
        if flag:
            raise NotImplementedError(f"test({name}) is not built")
    if dataloader is None:
        raise ValueError("test() needs a dataloader of collate_fn batches")
    device = next(model.parameters()).device
    half = device.type != "cpu" and half_precision
    if half:
        model.half()
    model.eval()
    if isinstance(data, str):
        import yaml
        with open(data) as f:
            data = yaml.load(f, Loader=yaml.SafeLoader)
    nc = 1 if single_cls else int(data["nc"])
    m = model.module if hasattr(model, "module") else model
    names = {k: v for k, v in enumerate(m.names)}
    s = ("%20s" + "%12s" * 6) % ("Class", "Images", "Labels", "P", "R", "mAP@.5", "mAP@.5:.95")
    print(s)
    p, r, f1, mp, mr, map50, map = 0., 0., 0., 0., 0., 0., 0.
    loss = torch.zeros(3, device=device)
    stats = DetectionStats(max_det=300, device=device)
    events = []
    nbatches = 0
    for img, targets, paths, shapes in dataloader:
        nbatches += 1
        img = img.to(device, non_blocking=True)
        img = img.half() if half else img.float()
        img /= 255.0
        targets = targets.to(device)
        nb, _, height, width = img.shape
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
        with torch.no_grad():
            ev[0].record()
            out, train_out = model(img, augment=augment)[0]
            ev[1].record()
            if compute_loss:
                loss += compute_loss([x.float().contiguous() for x in train_out], targets)[1][:3]
            ev[2].record()
            dets, counts = non_max_suppression(out, conf_thres=conf_thres, iou_thres=iou_thres, multi_label=True, return_padded=True)
            ev.append(torch.cuda.Event(enable_timing=True))
            ev[3].record()
        stats.update(dets, counts, targets, (height, width), shapes)
        events.append(ev)

    p, r, ap, f1, ap_class, nt, seen = stats.compute(nc)       # synchronises once
    t0 = sum(e[0].elapsed_time(e[1]) for e in events) / 1e3
    t1 = sum(e[2].elapsed_time(e[3]) for e in events) / 1e3
    if len(ap_class):
        ap50, ap = ap[:, 0], ap.mean(1)
        mp, mr, map50, map = p.mean(), r.mean(), ap50.mean(), ap.mean()

    pf = "%20s" + "%12i" * 2 + "%12.3g" * 4
    print(pf % ("all", seen, nt.sum(), mp, mr, map50, map))
    if verbose and nc > 1 and seen:
        for i, c in enumerate(ap_class):
            print(pf % (names[c], seen, nt[c], p[i], r[i], ap50[i], ap[i]))
    t = tuple(x / max(seen, 1) * 1E3 for x in (t0, t1, t0 + t1)) + (imgsz, imgsz, batch_size)
    model.float()
    maps = np.zeros(nc) + map
    for i, c in enumerate(ap_class):
        maps[c] = ap[i]
    return (mp, mr, map50, map, *(loss.cpu() / max(nbatches, 1)).tolist()), maps, t


def seg_validation(model, n_segcls, valloader, device, half_precision=True):
    """reference test.py:31-65: mIoU = (inter / (np.spacing(1) + union)).mean() over the whole loader, in float64.  The batches'
    counters (myolo_seg_metrics) accumulate in one device buffer and are read once."""
    device = torch.device(device)
    half = device.type != "cpu" and half_precision
    if half:
        model.half()
    model.eval()
    counters = torch.zeros(2 + 3 * n_segcls, dtype=torch.int64, device=device)
    L = _lib.lib()
    for image, target in valloader:
        image = image.to(device, non_blocking=True)
        image = image.half() if half else image.float()
        with torch.no_grad():
            seg = model(image)[1]
            tgt = target.to(device=device, dtype=torch.int64, non_blocking=True).contiguous()
            pred = _class_map(seg, tgt.shape[-2:]).contiguous()
            _lib.check(L.myolo_seg_metrics(_lib.ptr(pred), _lib.torch_dtype_code(pred.dtype), _lib.ptr(tgt), pred.numel(), n_segcls,
                                           _lib.ptr(counters), _lib.stream_ptr()))
    c = counters.cpu().numpy()
    inter, pred_a, lab_a = c[2:2 + n_segcls], c[2 + n_segcls:2 + 2 * n_segcls], c[2 + 2 * n_segcls:]
    union = pred_a + lab_a - inter
    IoU = 1.0 * inter / (np.spacing(1) + union)
    return IoU.mean()
