"""GPU: detect() (multiyolov5_b200/detect.py, reference detect.py:79-233).

- Fixture replay: the post-process stage fed the reference's own z and seg (tests/golden/detect_cases.npz, oracle/make_golden_detect.py)
  writes every file and prints every line the reference did, byte for byte.
- myolo_detect_boxes against torch's CPU statements of detect.py:169,178 over random geometries, clip edges and exact .5 ties.
- End to end at batch sizes 1, 3 and 16 over mixed frame shapes, and with --classes, --agnostic-nms and --augment: every file equals the
  per-frame composition of the public functions (preprocess -> Model -> non_max_suppression -> scale_coords(...).round() on host copies
  of the rows -> seg_argmax -> seg_overlay / trainid2id -> cv2)."""
import os
import re
import time
from argparse import Namespace

import cv2
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from multiyolov5_b200 import detect as D
from multiyolov5_b200.utils.general import (detect_boxes, non_max_suppression, scale_coords, scale_coords_geometry, seg_argmax, seg_overlay,
                                            trainid2id, xyxy2xywh)
from multiyolov5_b200.utils.datasets import preprocess
from multiyolov5_b200.utils.plots import plot_one_box
from oracle import synth

pytestmark = pytest.mark.gpu

GOLD = os.path.join(synth.GOLDEN_DIR, "detect_cases.npz")
CKPT = os.path.join(synth.GOLDEN_DIR, "ref_ckpt_tiny.pt")
NAMES = [f"cls{i}" for i in range(10)]
CONF, IOU = 0.0012, 0.45


def _opt(tmp, **kw):
    o = dict(weights=CKPT, source=str(tmp), img_size=256, conf_thres=CONF, iou_thres=IOU, device="", view_img=False, save_txt=True,
             save_conf=True, nosave=False, classes=None, agnostic_nms=False, augment=False, update=False, project=str(tmp), name="exp",
             exist_ok=False, save_as_video=True, submit=True, batch_size=16)
    o.update(kw)
    return Namespace(**o)


class _VideoRec:
    frames, opened = [], []

    def __init__(self, path, fourcc, fps, size):
        _VideoRec.opened.append((path, fps, tuple(size)))

    def write(self, f):
        _VideoRec.frames.append(np.array(f, copy=True))

    def release(self):
        pass


@pytest.fixture
def video(monkeypatch):
    _VideoRec.frames, _VideoRec.opened = [], []
    monkeypatch.setattr(D.cv2, "VideoWriter", _VideoRec)
    return _VideoRec


def _read(path):
    a = cv2.imread(str(path), cv2.IMREAD_UNCHANGED)
    assert a is not None, path
    return a


def test_fixture_replay(tmp_path, capsys, video):
    g = np.load(GOLD)
    n = int(g["n_frames"])
    src = tmp_path / "src"
    src.mkdir()
    paths = [str(src / str(g[f"name{k}"])) for k in range(n)]
    opt = _opt(tmp_path)
    colors = [[int(v) for v in c] for c in g["colors"]]
    save_dir, save_img = D.prepare(opt)
    post = D.Postprocess(opt, save_dir, NAMES, colors, save_img, nf=n)
    t0 = time.time()
    for ks in ([0, 1], [2]):
        frames = [g[f"frame{k}"] for k in ks]
        z = torch.cat([torch.from_numpy(g[f"z{k}"]) for k in ks]).cuda()
        seg = torch.cat([F.interpolate(torch.from_numpy(g[f"seglow{k}"]), scale_factor=8, mode="bilinear", align_corners=True) for k in ks])
        post([paths[k] for k in ks], torch.from_numpy(np.stack(frames)).cuda(), seg.shape[2:], z, seg.cuda(), host_frames=frames)
    post.close()
    D.finish(opt, save_dir, save_img, t0)
    out = capsys.readouterr().out.replace(str(tmp_path), "<dir>")
    out = re.sub(r"Done\. \([0-9.]+s\)", "Done. (<t>s)", out)
    assert out.splitlines() == str(g["stdout"]).splitlines()
    exp = tmp_path / "exp"
    for k in range(n):
        stem = str(g[f"name{k}"])[:-4]
        np.testing.assert_array_equal(_read(exp / f"{stem}.png"), g[f"img{k}"])
        np.testing.assert_array_equal(_read(exp / f"{stem}_mask.png"), g[f"mask{k}"])
        np.testing.assert_array_equal(_read(exp / f"{stem}_dst.png"), g[f"dst{k}"])
        np.testing.assert_array_equal(_read(exp / "results" / f"{stem}_pred.png"), g[f"ids{k}"].reshape(g[f"ids{k}"].shape[:2]))
        assert (exp / "labels" / f"{stem}.txt").read_bytes() == g[f"txt{k}"].tobytes()
        np.testing.assert_array_equal(video.frames[k], g[f"video{k}"])
    assert video.opened == [(str(exp) + "out.mp4", 30, tuple(int(v) for v in g["video_size"]))]


def test_box_kernel_matches_torch_cpu():
    rng = np.random.default_rng(0)
    for trial in range(40):
        B, max_det, nc = int(rng.integers(1, 9)), 300, int(rng.integers(1, 40))
        geoms, hw0 = [], []
        rows = np.zeros((B, max_det, 6), np.float32)
        counts = rng.integers(0, max_det + 1, B).astype(np.int32)
        counts[0] = max_det
        for b in range(B):
            if trial % 4 == 0:          # gains of exactly 0.5, 1 and 2, so that .5 lands exactly on ties
                h0, w0 = [(128, 256), (256, 512), (512, 1024)][b % 3]
                hw = (256, 512)
            else:
                h0, w0 = int(rng.integers(16, 2500)), int(rng.integers(16, 2500))
                hw = (int(rng.integers(1, 60)) * 32, int(rng.integers(1, 60)) * 32)
            geoms.append(scale_coords_geometry(hw, (h0, w0)))
            hw0.append((hw, (h0, w0)))
            n = int(counts[b])
            big = max(hw)
            r = rng.uniform(-0.2 * big, 1.2 * big, (n, 4)).astype(np.float32)
            ties = rng.random((n, 4)) < 0.4
            r[ties] = (np.floor(r[ties]) + 0.5).astype(np.float32)
            edge = rng.random((n, 4)) < 0.1
            r[edge] = np.float32(0.0)
            rows[b, :n, :4] = r
            rows[b, :n, 4] = rng.random(n).astype(np.float32)
            rows[b, :n, 5] = rng.integers(0, nc, n).astype(np.float32)
            rows[b, n:] = rng.random((max_det - n, 6)).astype(np.float32) * 100    # past the count: untouched
        d = torch.from_numpy(rows).cuda()
        wh, cc = detect_boxes(d, torch.from_numpy(counts).cuda(), np.stack(geoms), nc=nc, xywhn=True)
        got, wh, cc = d.cpu().numpy(), wh.cpu().numpy(), cc.cpu().numpy()
        for b, (hw, (h0, w0)) in enumerate(hw0):
            n = int(counts[b])
            det = torch.from_numpy(rows[b, :n].copy())
            det[:, :4] = scale_coords(hw, det[:, :4], (h0, w0, 3)).round()
            np.testing.assert_array_equal(got[b, :n], det.numpy())
            np.testing.assert_array_equal(got[b, n:], rows[b, n:])
            gn = torch.tensor((h0, w0, 3))[[1, 0, 1, 0]]
            for j in range(n):
                ref = (xyxy2xywh(torch.tensor(list(det[j, :4])).view(1, 4)) / gn).view(-1).numpy()
                np.testing.assert_array_equal(wh[b, j], ref)
            np.testing.assert_array_equal(cc[b], np.bincount(rows[b, :n, 5].astype(np.int64), minlength=nc))


# ---- end to end ----
SHAPES = [(160, 320)] * 4 + [(150, 230)] * 2 + [(160, 320)] * 3 + [(97, 203)] + [(150, 230)] * 5


def _frames():
    from oracle.make_golden_detect import synth_frame
    return [(f"/data/f_{i:03d}.png", synth_frame(h, w, 10 + i)) for i, (h, w) in enumerate(SHAPES)]


def _compose(model, opt, frames, colors):
    """the per-frame reference loop composed of this library's public functions"""
    files, txt, lines, video = {}, {}, [], []
    for path, im0 in frames:
        stem = os.path.basename(path)[:-4]
        im0 = im0.copy()
        img = preprocess(im0, opt.img_size, stride=32, half=False)[0]
        out = model(img, augment=opt.augment)
        det = non_max_suppression(out[0][0], opt.conf_thres, opt.iou_thres, classes=opt.classes, agnostic=opt.agnostic_nms)[0].cpu()
        s = "%gx%g " % img.shape[2:]
        gn = torch.tensor(im0.shape)[[1, 0, 1, 0]]
        if len(det):
            det[:, :4] = scale_coords(img.shape[2:], det[:, :4], im0.shape).round()
            for c in det[:, -1].unique():
                n = (det[:, -1] == c).sum()
                s += f"{n} {NAMES[int(c)]}{'s' * (n > 1)}, "
            for *xyxy, conf, cls in reversed(det):
                if opt.save_txt:
                    xywh = (xyxy2xywh(torch.tensor(xyxy).view(1, 4)) / gn).view(-1).tolist()
                    line = (cls, *xywh, conf) if opt.save_conf else (cls, *xywh)
                    txt[stem] = txt.get(stem, "") + ("%g " * len(line)).rstrip() % line + "\n"
                if not opt.nosave:
                    plot_one_box(xyxy, im0, label=f"{NAMES[int(cls)]} {conf:.2f}", color=colors[int(cls)], line_thickness=3)
        lines.append(s)
        cls_map = seg_argmax(out[1], im0.shape[:2])[0]
        mask = seg_overlay(cls_map, torch.from_numpy(im0).cuda())[0].cpu().numpy()
        dst = cv2.addWeighted(mask, 0.4, im0, 0.6, 0)
        if opt.submit:
            files[f"results/{stem}_pred.png"] = trainid2id(cls_map).cpu().numpy()[..., 0]
        if not opt.nosave:
            files[f"{stem}.png"], files[f"{stem}_mask.png"], files[f"{stem}_dst.png"] = im0, mask, dst
        video.append(dst)
    return files, txt, lines, video


@pytest.fixture(scope="module")
def model():
    from multiyolov5_b200.models.experimental import attempt_load
    return attempt_load(CKPT).cuda().eval()


def _run_and_compare(tmp_path, capsys, video, model, frames, **kw):
    opt = _opt(tmp_path, **kw)
    np.random.seed(5)
    colors = [[np.random.randint(0, 255) for _ in range(3)] for _ in NAMES]
    files, txt, lines, vid = _compose(model, opt, frames, colors)
    capsys.readouterr()
    np.random.seed(5)
    save_dir = D.detect(opt, dataset=frames, model=model)
    out = capsys.readouterr().out.splitlines()
    assert [s.rsplit("Done. (", 1)[0] for s in out[:len(frames)]] == lines
    assert out[-1].startswith("Done. (")
    for rel, a in files.items():
        np.testing.assert_array_equal(_read(save_dir / rel), a, err_msg=rel)
    written = {str(p.relative_to(save_dir)) for p in save_dir.rglob("*.png")}
    assert written == set(files)
    got_txt = {p.stem: p.read_text() for p in (save_dir / "labels").glob("*.txt")} if opt.save_txt else {}
    assert got_txt == txt
    if opt.save_as_video:
        assert len(video.frames) == len(vid)
        for a, b in zip(video.frames, vid):
            np.testing.assert_array_equal(a, b)
    return txt


@pytest.mark.parametrize("bs", [1, 3, 16])
def test_end_to_end_batch_sizes(tmp_path, capsys, video, model, bs):
    frames = _frames()
    txt = _run_and_compare(tmp_path, capsys, video, model, frames, batch_size=bs)
    assert len(txt) == len(frames)


def test_end_to_end_cuda_frames_submit_nosave(tmp_path, capsys, video, model):
    frames = [(p, torch.from_numpy(f).cuda()) for p, f in _frames()]
    opt = _opt(tmp_path, nosave=True, save_txt=False, save_as_video=False, batch_size=4)
    save_dir = D.detect(opt, dataset=frames, model=model)
    host = [(p, f.cpu().numpy()) for p, f in frames]
    files, _, lines, _ = _compose(model, opt, host, None)
    out = capsys.readouterr().out.splitlines()
    assert [s.rsplit("Done. (", 1)[0] for s in out[-len(frames) - 1:-1]] == lines
    assert {str(p.relative_to(save_dir)) for p in save_dir.rglob("*") if p.is_file()} == set(files)
    for rel, a in files.items():
        np.testing.assert_array_equal(_read(save_dir / rel), a, err_msg=rel)


@pytest.mark.parametrize("kw", [dict(classes=[3, 7]), dict(agnostic_nms=True), dict(augment=True)], ids=["classes", "agnostic", "augment"])
def test_end_to_end_flags(tmp_path, capsys, video, model, kw):
    _run_and_compare(tmp_path, capsys, video, model, _frames()[:8], batch_size=3, **kw)


def test_load_images_end_to_end(tmp_path, capsys, video, model):
    src = tmp_path / "src"
    src.mkdir()
    frames = _frames()[:5]
    for p, f in frames:
        cv2.imwrite(str(src / os.path.basename(p)), f)
    opt = _opt(tmp_path, source=str(src), save_as_video=False, batch_size=2)
    save_dir = D.detect(opt, model=model)
    out = capsys.readouterr().out.splitlines()
    for i, (p, _) in enumerate(frames):
        assert out[i].startswith(f"image {i + 1}/5 {src / os.path.basename(p)}: ")
    assert out[-2] == f"Results saved to {save_dir}\n5 labels saved to {save_dir / 'labels'}".splitlines()[-1]
