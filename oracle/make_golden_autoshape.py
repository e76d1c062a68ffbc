"""TEST INFRASTRUCTURE - generates tests/golden/autoshape_cases.npz by running the UNMODIFIED reference's autoShape (models/common.py:605-752,
MYOLO_REFERENCE_ROOT, imported through oracle/ref_shims.py) on the CPU, in fp32:

    MYOLO_REFERENCE_ROOT=<checkout> python oracle/make_golden_autoshape.py

The model is tests/golden/ref_ckpt_tiny.pt through the reference's attempt_load and Model.autoshape().  The fork's autoShape indexes
`self.model(x)[0]`, which in this multi-task model is the tuple (z, train_out); the wrapped model returns [z] instead, the `[0][0]` the
port uses (as for --augment), and records x, z and the seg head's logits before its final x8 bilinear (align_corners=True) upsample.
matplotlib is absent, so color_list()'s TABLEAU_COLORS are given to the shim.  The reference's render() draws with cv2 on the arrays it
holds, which for PIL / path inputs (read-only), CHW and RGBA inputs (strided views) cv2 refuses; they are replaced by writable contiguous
copies first, as the port does.  Calls (CALLS): five mixed inputs at size 160 (an exact 2x down-scale, a CHW array, a grayscale up-scale,
an RGBA PIL image, a file path; uneven pad splits) and a batch of one at size 192.  The inputs are not stored: make_input rebuilds each
from its kind, size and seed.  Stored per call c:
  c{c}_kind{k} / c{c}_hw{k} / c{c}_seed{k}   the input's kind, (H0, W0) and seed, and its array's CRC-32 (c{c}_crc{k}), which tests
  c{c}_crc{k} / c{c}_name{k}                 compare with the rebuilt input; for a path the file name
  c{c}_size, c{c}_shape1, c{c}_files         forward's size, the inference shape1 and Detections.files
  c{c}_x                                     the letterboxed batch as uint8 (the generator checks that the reference's x is exactly its /255.)
  c{c}_z                                     z (B, A, 5+nc) fp32, rows zeroed that NMS drops first (as detect_cases.npz does)
  c{c}_seglow                                the seg head's logits before the x8 upsample (torch's CPU F.interpolate of them is checked to be the seg)
  c{c}_{xyxy,xywh,xyxyn,xywhn}{k}            Detections' per-image tensors
  c{c}_render{k}                             the render() arrays
  c{c}_stdout                                the lines of print(), the timings replaced by <t>
"""
import contextlib
import io
import os
import re
import sys
import tempfile
import types
import zlib

import numpy as np
import torch
import torch.nn.functional as F
from PIL import Image

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
from oracle import ref_shims  # noqa: E402
from oracle.make_golden_detect import synth_frame  # noqa: E402

GOLD = os.path.join(HERE, "..", "tests", "golden")
CONF, IOU = 0.0012, 0.45
TABLEAU = {"tab:blue": "#1f77b4", "tab:orange": "#ff7f0e", "tab:green": "#2ca02c", "tab:red": "#d62728", "tab:purple": "#9467bd",
           "tab:brown": "#8c564b", "tab:pink": "#e377c2", "tab:gray": "#7f7f7f", "tab:olive": "#bcbd22", "tab:cyan": "#17becf"}
# (kind, (H0, W0), seed, file name for paths); kinds: hwc, chw (given as (3, H0, W0)), gray, pil_rgba, path
CALLS = [(160, [("hwc", (240, 320), 21, None), ("chw", (90, 140), 22, None), ("gray", (61, 127), 23, None),
                ("pil_rgba", (125, 75), 24, None), ("path", (60, 45), 25, "e_004.png")]),
         (192, [("hwc", (130, 170), 26, None)])]


def make_input(kind, hw, seed):
    """the array of one input, as stored: HWC RGB uint8, (3, H, W) for chw, (H, W) for gray, (H, W, 4) for pil_rgba"""
    rgb = synth_frame(*hw, seed)[:, :, ::-1].copy()
    if kind == "chw":
        return np.ascontiguousarray(rgb.transpose(2, 0, 1))
    if kind == "gray":
        return np.ascontiguousarray(rgb[:, :, 1])
    if kind == "pil_rgba":
        return np.concatenate([rgb, np.full(hw + (1,), 200, np.uint8)], 2)
    return rgb


def as_given(kind, arr, name, folder):
    """what the caller hands autoShape for one stored input"""
    if kind == "pil_rgba":
        return Image.fromarray(arr, "RGBA")
    if kind == "path":
        path = os.path.join(folder, name)
        Image.fromarray(arr).save(path)
        return path
    return arr.copy()


def main():
    if not ref_shims.reference_available():
        raise SystemExit("set MYOLO_REFERENCE_ROOT to a reference checkout")
    ref_shims.import_reference()
    sys.modules["matplotlib"].colors = types.SimpleNamespace(TABLEAU_COLORS=TABLEAU)
    from models.experimental import attempt_load            # the reference's, on sys.path after import_reference

    torch_load = torch.load     # the reference predates torch's weights_only default; its checkpoint pickles whole modules
    torch.load = lambda *la, **lk: torch_load(*la, **{**lk, "weights_only": False})
    try:
        model = attempt_load(os.path.join(GOLD, "ref_ckpt_tiny.pt"), map_location="cpu")
    finally:
        torch.load = torch_load
    up = model.model[-2].out[-1]        # SegMaskPSP.out's final nn.Upsample(scale_factor=8, bilinear, align_corners=True)
    assert isinstance(up, torch.nn.Upsample)
    cap = {}
    up.register_forward_hook(lambda m, i, o: cap.update(low=i[0].detach().clone(), seg=o.detach().clone()))

    class ZOnly(torch.nn.Module):
        def __init__(self, m):
            super().__init__()
            self.m = m

        def forward(self, x, augment=False, profile=False):
            out = self.m(x, augment, profile)
            assert torch.equal(out[1], cap["seg"])
            re_seg = F.interpolate(cap["low"], scale_factor=8, mode="bilinear", align_corners=True)
            assert torch.equal(re_seg, out[1]), "the seg head's upsample is not reproducible from its input"
            cap.update(x=x.clone(), z=out[0][0].clone())
            return [out[0][0]]

    with contextlib.redirect_stdout(io.StringIO()):
        shaped = model.autoshape()
    shaped.model = ZOnly(model)
    shaped.conf, shaped.iou = CONF, IOU

    out = {}
    with tempfile.TemporaryDirectory() as tmp:
        for c, (size, items) in enumerate(CALLS):
            inputs = []
            for k, (kind, hw, seed, name) in enumerate(items):
                arr = make_input(kind, hw, seed)
                out[f"c{c}_kind{k}"], out[f"c{c}_hw{k}"], out[f"c{c}_seed{k}"] = np.array(kind), np.array(hw, np.int64), np.int64(seed)
                out[f"c{c}_crc{k}"] = np.int64(zlib.crc32(arr.tobytes()))
                if name:
                    out[f"c{c}_name{k}"] = np.array(name)
                inputs.append(as_given(kind, arr, name, tmp))
            with torch.no_grad():
                res = shaped(inputs, size=size)
            x = cap["x"]
            x8 = torch.round(x * 255).to(torch.uint8)
            assert torch.equal(x8.float() / 255., x), "x is not uint8 / 255."
            z = cap["z"]
            keep = (z[..., 4] > CONF) & ((z[..., 5:] * z[..., 4:5]).amax(-1) > CONF)
            out[f"c{c}_z"] = torch.where(keep[..., None], z, torch.zeros_like(z)).numpy()
            out[f"c{c}_x"], out[f"c{c}_seglow"] = x8.numpy(), cap["low"].numpy()
            out[f"c{c}_size"], out[f"c{c}_shape1"] = np.int64(size), np.array(x.shape[2:], np.int64)
            out[f"c{c}_files"] = np.array(res.files)
            for k in range(res.n):
                for a in ("xyxy", "xywh", "xyxyn", "xywhn"):
                    out[f"c{c}_{a}{k}"] = getattr(res, a)[k].numpy()
                print(f"call {c} image {k}: {len(res.pred[k])} boxes, {int(keep[k].sum())} candidate rows, files {res.files[k]}")
                assert 3 <= len(res.pred[k]) <= 60, "tune CONF: every image should keep a few boxes"
            buf = io.StringIO()
            with contextlib.redirect_stdout(buf):
                res.print()
            lines = [re.sub(r"[0-9.]+ms", "<t>ms", s) for s in buf.getvalue().splitlines()]
            out[f"c{c}_stdout"] = np.array("\n".join(lines))
            print("\n".join(lines))
            res.imgs = [np.array(im, order="C") for im in res.imgs]
            for k, im in enumerate(res.render()):
                out[f"c{c}_render{k}"] = np.array(im)
    out["settings"] = np.array([CONF, IOU], np.float64)
    path = os.path.join(GOLD, "autoshape_cases.npz")
    np.savez_compressed(path, **out)
    print(f"wrote {path}: {os.path.getsize(path) / 1e6:.2f} MB")


if __name__ == "__main__":
    main()
