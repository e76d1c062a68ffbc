"""Validation passes behind the reference's names (reference test.py): `test` (the training path of test.py:77-340) and `seg_validation`
(test.py:31-65).  A pass stays on the device from the uint8 batch to a few per-class numbers: per batch one forward, one NMS and one
matching launch (utils.metrics.DetectionStats), with no host synchronisation; ap_per_class runs once at the end.

The reference validates in fp16 on CUDA (its z, NMS rows and box_iou are half tensors); this model keeps z in fp32, so the statistics
equal the reference's fp32 statistics of the same predictions, which is what its test() computes on a CPU device.

The batches can come from the device as well: `test(data, model=m, dataloader=DetValLoader(cache, 32), plots=False)` with
`cache = utils.datasets.DeviceImageCache(frames, imgsz, labels, augment=False)` is the reference's rect validation loader of
train.py:207-210 (`create_dataloader(..., rect=True, pad=0.5)`), bit exact with it.

test()'s options, as the reference's test.py has them:
  augment      the TTA forward (model(img, augment=True)[0] is (z, None), so compute_loss cannot go with it)
  model        a Model or an Ensemble (models.experimental.attempt_load of several weights: its [0] is (z, None) too, so compute_loss
               cannot go with it; model.half() reaches every member)
  save_hybrid  the labels join each image's NMS candidates (non_max_suppression with an NmsLabels, myolo_nms_labels), so the
               statistics include them, as in the reference
  plots        the confusion matrix (utils.metrics.ConfusionMatrix, one myolo_confusion_update launch per batch) and its plot();
               the batch mosaics and PR curves are not drawn
  save_txt, save_conf, save_json
               labels/<stem>.txt and <weights stem>_predictions.json, from native-space rows (myolo_scale_boxes on a copy of the NMS
               rows); the rows are copied to the host once per batch, only when one of these is set
"""
import json
from pathlib import Path

import numpy as np
import torch

from . import _lib
from .models.experimental import Ensemble
from .utils.general import NmsLabels, check_nms_labels_error, coco80_to_coco91_class, non_max_suppression, scale_boxes
from .utils.metrics import ConfusionMatrix, DetectionStats, _class_map, pack_geometry


def _write_rows(rows, xywh, xywhn, counts, paths, shapes, save_dir, save_txt, save_conf, save_json, is_coco, coco91, jdict):
    """test.py:197-205 (labels/<stem>.txt) and :220-229 (the JSON records) for one batch of host rows: rows are the native-space
    predn, xywh / xywhn their xyxy2xywh and its division by (w0, h0, w0, h0), all float32 as in the reference"""
    for si in range(len(counts)):
        n = int(counts[si])
        if n == 0:
            continue
        path = Path(paths[si])
        if save_txt:
            with open(save_dir / "labels" / (path.stem + ".txt"), "a") as f:
                for k in range(n):
                    cls, conf = float(rows[si, k, 5]), float(rows[si, k, 4])
                    wh = [float(v) for v in xywhn[si, k, :4]]
                    line = (cls, *wh, conf) if save_conf else (cls, *wh)
                    f.write(("%g " * len(line)).rstrip() % line + "\n")
        if save_json:
            image_id = int(path.stem) if path.stem.isnumeric() else path.stem
            box = xywh[si, :n, :4].copy()
            box[:, :2] -= box[:, 2:] / np.float32(2)       # xy center to top-left corner, in float32
            for k in range(n):
                c = int(rows[si, k, 5])
                jdict.append({"image_id": image_id, "category_id": coco91[c] if is_coco else c,
                              "bbox": [round(float(x), 3) for x in box[k]], "score": round(float(rows[si, k, 4]), 5)})


def test(data, weights=None, batch_size=32, imgsz=640, conf_thres=0.001, iou_thres=0.6, save_json=False, single_cls=False, augment=False,
         verbose=False, model=None, dataloader=None, save_dir=Path(""), save_txt=False, save_hybrid=False, save_conf=False, plots=True,
         wandb_logger=None, compute_loss=None, half_precision=True, is_coco=False):
    """Returns ((mp, mr, map50, map, *loss), maps, t) like the reference.  `dataloader` yields collate_fn tuples
    (img uint8 (B,3,H,W), targets (n,6), paths, shapes) on the host or the device.  Prints the `all` row (and per-class rows with
    verbose).  t = (forward, NMS, total) ms per image from CUDA events, then (imgsz, imgsz, batch_size).  The module docstring lists
    the options; files go to save_dir."""
    if model is None:
        raise NotImplementedError("test(model=None): loading weights and data files is not built; pass model= and dataloader=")
    if wandb_logger:
        raise NotImplementedError("test(wandb_logger=...): W&B logging is not built")
    if compute_loss and isinstance(model, Ensemble):
        raise ValueError("test(model=Ensemble) returns no training outputs (model(img)[0] is (z, None)), so compute_loss cannot be "
                         "evaluated with it")
    if next(model.parameters()).device.type != "cuda":
        raise NotImplementedError("test() on a CPU model: there is no CPU path; move the model to the GPU")
    if augment and compute_loss:
        raise ValueError("test(augment=True) returns no training outputs, so compute_loss cannot be evaluated with it")
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
    save_dir = Path(save_dir)
    if save_txt:
        (save_dir / "labels").mkdir(parents=True, exist_ok=True)
    confusion_matrix = ConfusionMatrix(nc=nc, device=device) if plots else None
    hybrid_err = torch.zeros(1, dtype=torch.int32, device=device) if save_hybrid else None
    coco91 = coco80_to_coco91_class()
    jdict = []
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
            lb = NmsLabels.from_targets(targets, nb, (height, width), err=hybrid_err) if save_hybrid else ()
            dets, counts = non_max_suppression(out, conf_thres=conf_thres, iou_thres=iou_thres, labels=lb, multi_label=True,
                                               return_padded=True)
            ev.append(torch.cuda.Event(enable_timing=True))
            ev[3].record()
        stats.update(dets, counts, targets, (height, width), shapes)
        if plots:
            confusion_matrix.update(dets, counts, targets, (height, width), shapes)
        if save_txt or save_json:
            geom = pack_geometry((height, width), shapes)[:, [3, 4, 2, 1, 0]]      # (padw, padh, gain, w0, h0)
            rows = dets.clone()
            xywh, _, xywhn = scale_boxes(rows, counts, geom)
            host = torch.stack([rows, xywh, xywhn]).cpu().numpy()
            _write_rows(host[0], host[1], host[2], counts.cpu().numpy(), paths, shapes, save_dir, save_txt, save_conf, save_json, is_coco,
                        coco91, jdict)
        events.append(ev)

    p, r, ap, f1, ap_class, nt, seen = stats.compute(nc)       # synchronises once
    if save_hybrid:
        check_nms_labels_error(int(hybrid_err.item()))
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
    if plots:
        confusion_matrix.plot(save_dir=save_dir, names=list(names.values()))
    if save_json and len(jdict):
        w = Path(weights[0] if isinstance(weights, list) else weights).stem if weights is not None else ""
        pred_json = str(save_dir / f"{w}_predictions.json")
        print("\nEvaluating pycocotools mAP... saving %s..." % pred_json)
        with open(pred_json, "w") as f:
            json.dump(jdict, f)
        try:
            from pycocotools.coco import COCO  # noqa: F401
            raise NotImplementedError("pycocotools evaluation is not built")
        except Exception as e:
            print(f"pycocotools unable to run: {e}")
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
