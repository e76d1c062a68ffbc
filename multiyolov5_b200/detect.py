"""The reference's detect.py (reference detect.py:79-233) on the device, batched:

    from multiyolov5_b200.detect import detect, LoadImages
    detect(opt)                      # opt: argparse.Namespace of the flags below (batch_size defaults to 16)
    detect(opt, dataset=frames)      # frames: iterable of (path, im0), im0 a decoded BGR uint8 (H0, W0, 3) numpy array or CUDA tensor
    python -m multiyolov5_b200.detect --weights w.pt --source dir --img-size 1024 --submit --nosave

Decoding stays on the host (cv2.imread).  Consecutive frames of one shape go through one preprocess, one forward and one NMS of up to
`batch_size` frames; a new shape closes the batch.  Per batch, on the device: myolo_detect_boxes scales every frame's NMS rows to the frame
in place (scale_coords(...).round()) and writes the --save-txt xywh and the per-class counts of the printed line; seg_argmax makes the uint8
class map at frame size and one myolo_seg_lut_blend pass writes the BGR mask, the 0.4/0.6 blend of the undrawn frame and the trainid2id
ids the flags ask for.  Device-to-host copies into pinned buffers run on a side stream; a writer thread draws the boxes (cv2, as the
reference), re-blends only the rectangles the drawing touched, and writes the PNGs, the txt labels and the video, so the GPU runs ahead
of PNG encoding.  Every file and printed line is the reference's, whatever the batch size, with the reference's z run in fp32 (its CPU
path); the per-frame time printed is the batch's forward + NMS device time over its frames.

Not built (NotImplementedError): --view-img, --update, webcams, streams, URLs and video files (there is no video decoding).
"""
import argparse
import glob
import os
import queue
import threading
import time
from pathlib import Path

import cv2
import numpy as np
import torch

from .models.experimental import attempt_load
from .utils.datasets import preprocess
from .utils.general import (check_img_size, detect_boxes, increment_path, non_max_suppression, scale_coords_geometry, seg_argmax,
                            seg_products)
from .utils.plots import box_extent, plot_one_box, reblend

img_formats = ['bmp', 'jpg', 'jpeg', 'png', 'tif', 'tiff', 'dng', 'webp', 'mpo']     # reference utils/datasets.py:29-30
vid_formats = ['mov', 'avi', 'mp4', 'mpg', 'mpeg', 'm4v', 'wmv', 'mkv']


class LoadImages:
    """reference utils/datasets.py:122-191 for image files: the files of a path, directory or glob, sorted, with an image suffix, decoded
    by cv2.imread on the host.  Yields (path, im0); `nf` and `count` as the reference's, for the 'image k/n path: ' prefix."""

    def __init__(self, path, img_size=640, stride=32):
        p = str(Path(path).absolute())
        if '*' in p:
            files = sorted(glob.glob(p, recursive=True))
        elif os.path.isdir(p):
            files = sorted(glob.glob(os.path.join(p, '*.*')))
        elif os.path.isfile(p):
            files = [p]
        else:
            raise Exception(f'ERROR: {p} does not exist')
        images = [x for x in files if x.split('.')[-1].lower() in img_formats]
        videos = [x for x in files if x.split('.')[-1].lower() in vid_formats]
        if videos:
            raise NotImplementedError(f"detect: video files ({videos[0]}) are not built: there is no video decoding")
        self.img_size, self.stride = img_size, stride
        self.files, self.nf, self.mode = images, len(images), 'image'
        assert self.nf > 0, f'No images or videos found in {p}. Supported formats are:\nimages: {img_formats}\nvideos: {vid_formats}'

    def __len__(self):
        return self.nf

    def __iter__(self):
        for self.count, path in enumerate(self.files, 1):
            img0 = cv2.imread(path)
            assert img0 is not None, 'Image Not Found ' + path
            yield path, img0


def _refuse(opt):
    source = str(opt.source)
    for flag, name in (("view_img", "--view-img"), ("update", "--update")):
        if getattr(opt, flag, False):
            raise NotImplementedError(f"detect {name} is not built")
    if source.isnumeric():
        raise NotImplementedError("detect --source <webcam index>: webcams are not built")
    if source.endswith('.txt'):
        raise NotImplementedError("detect --source <streams .txt>: streams are not built")
    if source.lower().startswith(('rtsp://', 'rtmp://', 'http://', 'https://')):
        raise NotImplementedError("detect --source <URL>: URLs are not built")
    if str(getattr(opt, "device", "")).lower() == "cpu":
        raise NotImplementedError("detect --device cpu: multiyolov5_b200 runs on the GPU only")


class Postprocess:
    """the stage of detect() after the forward, one call per batch: __call__(paths, frames, img_hw, z, seg) enqueues the device work and the
    copies and returns without a synchronisation; close() waits for the writer and releases the video.  frames: (B, H0, W0, 3) uint8 CUDA
    tensor, host_frames the same frames on the host when the caller has them (else they are copied back when boxes are drawn).  z / seg
    are the model's out[0][0] and out[1] for the letterboxed batch of height-width img_hw."""

    def __init__(self, opt, save_dir, names, colors, save_img, nf=None, queue_depth=3):
        self.opt, self.save_dir, self.names, self.colors, self.save_img, self.nf = opt, Path(save_dir), list(names), colors, save_img, nf
        self.save_txt, self.save_conf = bool(opt.save_txt), bool(opt.save_conf)
        self.submit, self.save_as_video = bool(opt.submit), bool(opt.save_as_video)
        self.sub_dir = str(self.save_dir) + "/results/"
        self.side = torch.cuda.Stream()
        self.count = 0
        self.s_writer = None
        self.error = None
        self.q = queue.Queue(maxsize=queue_depth)
        self.thread = threading.Thread(target=self._run, daemon=True)
        self.thread.start()

    # ---- device side (caller's thread, current stream) ----
    def __call__(self, paths, frames, img_hw, z, seg, host_frames=None, events=None):
        opt = self.opt
        B, H0, W0, _ = frames.shape
        rows, cnt = non_max_suppression(z, opt.conf_thres, opt.iou_thres, classes=opt.classes, agnostic=opt.agnostic_nms, return_padded=True)
        if events is not None:
            events[1].record()
        draw = self.save_img
        geom = np.tile(scale_coords_geometry(tuple(img_hw), (H0, W0)), (B, 1))
        xywhn, cc = detect_boxes(rows, cnt, torch.from_numpy(geom).pin_memory(), nc=len(self.names), xywhn=self.save_txt)
        want_dst = draw or self.save_as_video
        mask = dst = ids = None
        if draw or want_dst or self.submit:
            cls = seg_argmax(seg, (H0, W0), out_dtype=torch.uint8)
            mask, dst, ids = seg_products(cls, frames if want_dst else None, mask=draw, ids=self.submit)
        dev = {"cnt": cnt, "cc": cc}
        if self.save_txt or draw:
            dev["rows"] = rows
        if self.save_txt:
            dev["xywhn"] = xywhn
        for k, v in (("mask", mask), ("dst", dst), ("ids", ids)):
            if v is not None:
                dev[k] = v
        if draw and host_frames is None:
            dev["frames"] = frames
        done = torch.cuda.Event()
        self.side.wait_stream(torch.cuda.current_stream())
        host = {}
        with torch.cuda.stream(self.side):
            for k, v in dev.items():
                host[k] = torch.empty(v.shape, dtype=v.dtype, pin_memory=True)
                host[k].copy_(v, non_blocking=True)
            done.record(self.side)
        names = [str(p) for p in paths]
        first = self.count
        self.count += B
        self._put((done, dev, host, names, host_frames, tuple(int(v) for v in img_hw), events, first))

    def _put(self, item):
        while True:
            if self.error is not None:
                raise self.error
            try:
                self.q.put(item, timeout=0.5)
                return
            except queue.Full:
                continue

    def close(self):
        self.q.put(None)
        self.thread.join()
        if self.s_writer is not None:
            self.s_writer.release()
        if self.error is not None:
            raise self.error

    # ---- host side (writer thread) ----
    def _run(self):
        while True:
            item = self.q.get()
            if item is None:
                return
            if self.error is not None:
                continue
            try:
                self._write(*item)
            except BaseException as e:   # re-raised in the caller's thread
                self.error = e

    def _write(self, done, dev, host, paths, host_frames, img_hw, events, first):
        done.synchronize()
        del dev                                             # the device buffers may be reused once the copies are done
        h = {k: v.numpy() for k, v in host.items()}
        dt = events[0].elapsed_time(events[1]) / 1e3 / len(paths) if events is not None else 0.0
        for i, path in enumerate(paths):
            p = Path(path)
            s = f'image {first + i + 1}/{self.nf} {path}: ' if self.nf else ''
            s += frame_string(img_hw, h["cc"][i], self.names)
            n = int(h["cnt"][i])
            im0 = None
            if self.save_img:
                im0 = np.array(host_frames[i] if host_frames is not None else h["frames"][i])
            rects = []
            if n and (self.save_txt or self.save_img):
                det = h["rows"][i, :n]
                if self.save_txt:
                    with open(str(self.save_dir / 'labels' / p.stem) + '.txt', 'a') as f:
                        f.write(txt_lines(det, h["xywhn"][i, :n], self.save_conf))
                if self.save_img:
                    for xyxy, conf, cls in zip(det[::-1, :4], det[::-1, 4], det[::-1, 5]):
                        label = f'{self.names[int(cls)]} {float(conf):.2f}'
                        plot_one_box(xyxy, im0, label=label, color=self.colors[int(cls)], line_thickness=3)
                        rects += box_extent(xyxy, im0.shape, label=label, line_thickness=3)
            print(f'{s}Done. ({dt:.5f}s)')
            dst = h["dst"][i] if "dst" in h else None
            if dst is not None and rects:
                dst = reblend(np.array(dst), h["mask"][i], im0, rects)
            if self.submit:
                sub_path = (self.sub_dir + str(p.name))[:-4] + "_pred.png"
                cv2.imwrite(sub_path, h["ids"][i])
            if self.save_img:
                save_path = str(self.save_dir / p.name)
                cv2.imwrite(save_path, im0)
                cv2.imwrite(save_path[:-4] + "_mask" + save_path[-4:], h["mask"][i])
                cv2.imwrite(save_path[:-4] + "_dst" + save_path[-4:], dst)
            if self.save_as_video:
                if self.s_writer is None:
                    self.s_writer = cv2.VideoWriter(str(self.save_dir) + "out.mp4", cv2.VideoWriter_fourcc(*'mp4v'), 30,
                                                    (dst.shape[1], dst.shape[0]))
                self.s_writer.write(dst)


def frame_string(img_hw, class_counts, names):
    """detect.py:164,172-174: 'HxW ' of the network input, then 'n name' for each class present, in class order, plural with an s"""
    s = '%gx%g ' % tuple(img_hw)
    for c in np.flatnonzero(class_counts):
        n = int(class_counts[c])
        s += f"{n} {names[int(c)]}{'s' * (n > 1)}, "
    return s


def txt_lines(det, xywhn, save_conf):
    """detect.py:177-181 for one frame: its --save-txt lines, last row first as `reversed(det)`.  det: (n, 6) fp32 rows in frame space,
    xywhn: their (n, 4) fp32 normalised xywh"""
    out = []
    for j in range(len(det) - 1, -1, -1):
        xywh = [float(v) for v in xywhn[j]]
        line = (float(det[j, 5]), *xywh, float(det[j, 4])) if save_conf else (float(det[j, 5]), *xywh)
        out.append(('%g ' * len(line)).rstrip() % line + '\n')
    return ''.join(out)


def batches(dataset, batch_size):
    """consecutive (path, im0) of one shape, up to batch_size at a time: lists of paths and frames"""
    paths, frames = [], []
    for path, im0 in dataset:
        if frames and (len(frames) == batch_size or tuple(im0.shape) != tuple(frames[0].shape)):
            yield paths, frames
            paths, frames = [], []
        paths.append(path)
        frames.append(im0)
    if frames:
        yield paths, frames


def upload(frames, device):
    """a batch of decoded frames as one (B, H0, W0, 3) uint8 CUDA tensor, and the host frames (None when they came as CUDA tensors)"""
    if all(isinstance(f, torch.Tensor) and f.is_cuda for f in frames):
        return torch.stack([f.to(device) for f in frames]), None
    host = [f.cpu().numpy() if isinstance(f, torch.Tensor) else np.asarray(f) for f in frames]
    for f in host:
        if f.dtype != np.uint8 or f.ndim != 3 or f.shape[2] != 3:
            raise ValueError(f"detect: frames are decoded BGR uint8 (H0, W0, 3) arrays, got {f.dtype} {f.shape}")
    return torch.from_numpy(np.stack(host)).pin_memory().to(device, non_blocking=True), host


def prepare(opt):
    """detect.py:80-89: refuses what is not built, makes save_dir (and labels/, results/); returns (save_dir, save_img)"""
    _refuse(opt)
    save_img = not opt.nosave
    save_dir = Path(increment_path(Path(opt.project) / opt.name, exist_ok=opt.exist_ok))
    (save_dir / 'labels' if opt.save_txt else save_dir).mkdir(parents=True, exist_ok=True)
    if opt.submit:
        sub_dir = str(save_dir) + "/results/"
        if not os.path.exists(sub_dir):
            os.mkdir(sub_dir)
    return save_dir, save_img


def finish(opt, save_dir, save_img, t0):
    """detect.py:227-232: the closing lines"""
    if opt.save_txt or save_img:
        s = f"\n{len(list(save_dir.glob('labels/*.txt')))} labels saved to {save_dir / 'labels'}" if opt.save_txt else ''
        print(f"Results saved to {save_dir}{s}")
    print(f'Done. ({time.time() - t0:.3f}s)')


def detect(opt, dataset=None, model=None):
    """reference detect.py:79-233 on the device.  opt: the reference's flags (argparse.Namespace; batch_size defaults to 16).  dataset:
    an iterable of (path, im0) to run instead of LoadImages(opt.source); model: an already loaded model instead of attempt_load(opt.weights).
    Returns save_dir."""
    save_dir, save_img = prepare(opt)
    device = torch.device("cuda", torch.cuda.current_device())
    if model is None:
        model = attempt_load(opt.weights, map_location=device)
    model.to(device).eval()
    stride = int(model.stride.max())
    imgsz = check_img_size(opt.img_size, s=stride)
    if dataset is None:
        dataset = LoadImages(opt.source, img_size=imgsz, stride=stride)
    names = model.module.names if hasattr(model, 'module') else model.names
    colors = [[np.random.randint(0, 255) for _ in range(3)] for _ in names]
    post = Postprocess(opt, save_dir, names, colors, save_img, nf=getattr(dataset, "nf", None))
    t0 = time.time()
    try:
        with torch.no_grad():
            for paths, frames in batches(dataset, int(getattr(opt, "batch_size", 16) or 16)):
                dev, host = upload(frames, device)
                img = preprocess(dev, imgsz, stride=stride, half=False)[0]
                ev = (torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True))
                ev[0].record()
                out = model(img, augment=opt.augment)
                post(paths, dev, img.shape[2:], out[0][0], out[1], host_frames=host, events=ev)
    finally:
        post.close()
    finish(opt, save_dir, save_img, t0)
    return save_dir


def parse_opt(argv=None):
    parser = argparse.ArgumentParser()
    parser.add_argument('--weights', nargs='+', type=str, default='yolov5s.pt', help='model.pt path(s)')
    parser.add_argument('--source', type=str, default='data/images', help='source')
    parser.add_argument('--img-size', type=int, default=640, help='inference size (pixels)')
    parser.add_argument('--conf-thres', type=float, default=0.25, help='object confidence threshold')
    parser.add_argument('--iou-thres', type=float, default=0.45, help='IOU threshold for NMS')
    parser.add_argument('--device', default='', help='cuda device, i.e. 0')
    parser.add_argument('--view-img', action='store_true', help='display results (not built)')
    parser.add_argument('--save-txt', action='store_true', help='save results to *.txt')
    parser.add_argument('--save-conf', action='store_true', help='save confidences in --save-txt labels')
    parser.add_argument('--nosave', action='store_true', help='do not save images/videos')
    parser.add_argument('--classes', nargs='+', type=int, help='filter by class: --class 0, or --class 0 2 3')
    parser.add_argument('--agnostic-nms', action='store_true', help='class-agnostic NMS')
    parser.add_argument('--augment', action='store_true', help='augmented inference')
    parser.add_argument('--update', action='store_true', help='update all models (not built)')
    parser.add_argument('--project', default='runs/detect', help='save results to project/name')
    parser.add_argument('--name', default='exp', help='save results to project/name')
    parser.add_argument('--exist-ok', action='store_true', help='existing project/name ok, do not increment')
    parser.add_argument('--save-as-video', action='store_true', help='save same size images as a video')
    parser.add_argument('--submit', action='store_true', help='get submit file in folder submit')
    parser.add_argument('--batch-size', type=int, default=16, help='frames of one shape per forward')
    return parser.parse_args(argv)


if __name__ == '__main__':
    opt = parse_opt()
    print(opt)
    if opt.device and not str(opt.device).lower() == "cpu":
        torch.cuda.set_device(int(str(opt.device).split(",")[0]))
    detect(opt)
