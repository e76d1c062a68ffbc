"""TEST INFRASTRUCTURE - generates tests/golden/detect_cases.npz by running the UNMODIFIED reference's detect() (MYOLO_REFERENCE_ROOT,
imported through oracle/ref_shims.py) on the CPU, in fp32:

    MYOLO_REFERENCE_ROOT=<checkout> python oracle/make_golden_detect.py

The module's own `detect()` is called with its global `opt` set (its `__main__` is never run: it would check and install requirements).
Settings: tests/golden/ref_ckpt_tiny.pt, --img-size 256, --save-txt --save-conf --submit --save-as-video, numpy.random seeded with SEED,
over FRAMES written as PNGs to a temporary folder: two frames of one shape and one whose letterbox padding is split unevenly (a
fractional pad in scale_coords).  cv2.imwrite and cv2.VideoWriter are wrapped to record what the reference hands them, and a forward
hook records the model's out[0][0] (z) and its seg logits.  Stored:
  frame{k} / name{k}        the decoded BGR frame and its file name
  z{k}                      z (1, A, 5+nc) fp32 with every row zeroed whose objectness, or whose best objectness x class score, is not
                            above CONF: NMS drops those rows before anything else, so the detections are unchanged, and the fixture compresses
  seglow{k}                 the seg head's logits before its final x8 bilinear (align_corners=True) upsample; the generator checks that
                            torch's CPU F.interpolate of them is bit for bit the seg the reference used, so tests rebuild seg from them
  colors                    the reference's per-class box colours (numpy.random after the seed)
  img{k} / mask{k} / dst{k} / ids{k}   the arrays the reference wrote: frame with boxes, BGR mask, blend, Cityscapes label ids
  video{k}                  the frames handed to the out.mp4 writer, video_size its (w, h)
  txt{k}                    the bytes of labels/<stem>.txt
  stdout                    the lines printed by detect(), the temporary folder replaced by <dir> and timings by <t>
"""
import contextlib
import io
import os
import re
import sys
import tempfile
from argparse import Namespace

import cv2
import numpy as np
import torch
import torch.nn.functional as F

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
from oracle import ref_shims  # noqa: E402

GOLD = os.path.join(HERE, "..", "tests", "golden")
SEED = 3
IMG_SIZE = 256
CONF, IOU = 0.0012, 0.45
FRAMES = [("a_000.png", 160, 320, 1), ("a_001.png", 160, 320, 2), ("b_000.png", 150, 230, 3)]     # (name, H0, W0, seed)


def synth_frame(h, w, seed):
    """a smooth BGR frame with a few flat rectangles: it compresses, and the tiny model still fires on it"""
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float64)
    img = np.empty((h, w, 3), np.float64)
    for c in range(3):
        fy, fx, ph = rng.uniform(0.01, 0.06, 2).tolist() + [rng.uniform(0, 6.28)]
        img[..., c] = 128 + 100 * np.sin(fy * yy + ph) * np.cos(fx * xx)
    for _ in range(6):
        y0, x0 = int(rng.integers(0, h - 20)), int(rng.integers(0, w - 20))
        img[y0:y0 + int(rng.integers(10, 60)), x0:x0 + int(rng.integers(10, 80))] = rng.integers(0, 256, 3)
    return np.clip(np.rint(img), 0, 255).astype(np.uint8)


def main():
    if not ref_shims.reference_available():
        raise SystemExit("set MYOLO_REFERENCE_ROOT to a reference checkout")
    ref_shims.import_reference()
    import detect as ref_detect                 # the reference's detect.py, on sys.path after import_reference

    out = {}
    with tempfile.TemporaryDirectory() as tmp:
        src = os.path.join(tmp, "src")
        os.makedirs(src)
        for k, (name, h, w, seed) in enumerate(FRAMES):
            f = synth_frame(h, w, seed)
            cv2.imwrite(os.path.join(src, name), f)
            out[f"frame{k}"], out[f"name{k}"] = f, np.array(name)

        recorded = {"z": [], "seglow": [], "imwrite": {}, "video": [], "video_size": None}
        load = ref_detect.attempt_load

        def attempt_load(*a, **kw):
            torch_load = torch.load     # the reference predates torch's weights_only default; its checkpoint pickles whole modules
            torch.load = lambda *la, **lk: torch_load(*la, **{**lk, "weights_only": False})
            try:
                model = load(*a, **kw)
            finally:
                torch.load = torch_load
            up = model.model[-2].out[-1]        # SegMaskPSP.out's final nn.Upsample(scale_factor=8, bilinear, align_corners=True)
            assert isinstance(up, torch.nn.Upsample)
            cap = {}
            up.register_forward_hook(lambda m, i, o: cap.update(low=i[0].detach().clone(), seg=o.detach().clone()))

            def hook(m, i, o):
                z, seg = o[0][0].detach().clone(), o[1].detach().clone()
                assert torch.equal(seg, cap["seg"])
                re_seg = F.interpolate(cap["low"], scale_factor=8, mode="bilinear", align_corners=True)
                assert torch.equal(re_seg, seg), "the seg head's upsample is not reproducible from its input"
                recorded["z"].append(z)
                recorded["seglow"].append(cap["low"])
            model.register_forward_hook(hook)
            return model

        imwrite = cv2.imwrite

        def rec_imwrite(path, arr, *a):
            recorded["imwrite"][os.path.relpath(path, tmp)] = np.array(arr, copy=True)
            return imwrite(path, arr, *a)

        class RecWriter:
            def __init__(self, path, fourcc, fps, size):
                recorded["video_size"] = (os.path.relpath(path, tmp), fps, size)

            def write(self, frame):
                recorded["video"].append(np.array(frame, copy=True))

            def release(self):
                pass

        ref_detect.attempt_load = attempt_load
        ref_detect.cv2.imwrite = rec_imwrite
        video_writer = ref_detect.cv2.VideoWriter
        ref_detect.cv2.VideoWriter = RecWriter
        ref_detect.opt = Namespace(weights=os.path.join(GOLD, "ref_ckpt_tiny.pt"), source=src, img_size=IMG_SIZE, conf_thres=CONF,
                                   iou_thres=IOU, device="cpu", view_img=False, save_txt=True, save_conf=True, nosave=False, classes=None,
                                   agnostic_nms=False, augment=False, update=False, project=tmp, name="exp", exist_ok=False,
                                   save_as_video=True, submit=True)
        np.random.seed(SEED)
        buf = io.StringIO()
        try:
            with contextlib.redirect_stdout(buf), torch.no_grad():
                ref_detect.detect()
        finally:
            ref_detect.cv2.imwrite, ref_detect.cv2.VideoWriter = imwrite, video_writer
        np.random.seed(SEED)
        out["colors"] = np.array([[np.random.randint(0, 255) for _ in range(3)] for _ in range(10)], np.int64)

        lines = buf.getvalue().replace(tmp, "<dir>").splitlines()
        lines = [re.sub(r"Done\. \([0-9.]+s\)", "Done. (<t>s)", s) for s in lines if not s.startswith("Fusing layers")]
        out["stdout"] = np.array("\n".join(lines))
        print("\n".join(lines))
        wr = recorded["imwrite"]
        for k, (name, h, w, seed) in enumerate(FRAMES):
            stem = name[:-4]
            z = recorded["z"][k]
            keep = (z[..., 4] > CONF) & ((z[..., 5:] * z[..., 4:5]).amax(-1) > CONF)
            z = torch.where(keep[..., None], z, torch.zeros_like(z))
            out[f"z{k}"], out[f"seglow{k}"] = z.numpy(), recorded["seglow"][k].numpy()
            out[f"img{k}"] = wr[f"exp/{name}"]
            out[f"mask{k}"] = wr[f"exp/{stem}_mask.png"]
            out[f"dst{k}"] = wr[f"exp/{stem}_dst.png"]
            out[f"ids{k}"] = wr[f"exp/results/{stem}_pred.png"]
            out[f"video{k}"] = recorded["video"][k]
            with open(os.path.join(tmp, "exp", "labels", stem + ".txt"), "rb") as f:
                out[f"txt{k}"] = np.frombuffer(f.read(), np.uint8)
            n = out[f"txt{k}"].tobytes().count(b"\n")
            print(f"{name}: {n} boxes, {int(keep.sum())} candidate rows")
            assert 5 <= n <= 50, "tune CONF: every frame should keep 5-50 boxes"
        assert sorted(wr) == sorted([f"exp/{n[:-4]}{s}.png" for n, *_ in FRAMES for s in ("", "_mask", "_dst")] +
                                    [f"exp/results/{n[:-4]}_pred.png" for n, *_ in FRAMES])
        vpath, fps, size = recorded["video_size"]
        assert vpath == "expout.mp4" and fps == 30, recorded["video_size"]
        out["video_size"] = np.array(size, np.int64)
        out["n_frames"] = np.int64(len(FRAMES))
        out["settings"] = np.array([IMG_SIZE, CONF, IOU, SEED], np.float64)
    os.makedirs(GOLD, exist_ok=True)
    path = os.path.join(GOLD, "detect_cases.npz")
    np.savez_compressed(path, **out)
    print(f"wrote {path}: {os.path.getsize(path) / 1e6:.2f} MB")


if __name__ == "__main__":
    main()
