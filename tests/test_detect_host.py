"""Host side of detect() (multiyolov5_b200/detect.py, reference detect.py): LoadImages' file order, increment_path, the printed line and
--save-txt formatting against the reference's output in tests/golden/detect_cases.npz (oracle/make_golden_detect.py), the re-blend of
the drawn rectangles against a full cv2.addWeighted, and the flags that are not built."""
import os
from argparse import Namespace

import cv2
import numpy as np
import pytest
import torch

from multiyolov5_b200 import detect as D
from multiyolov5_b200.utils.general import increment_path, scale_coords, xyxy2xywh
from multiyolov5_b200.utils.plots import box_extent, plot_one_box, reblend
from oracle import restate, synth

GOLD = os.path.join(synth.GOLDEN_DIR, "detect_cases.npz")
NAMES = [f"cls{i}" for i in range(10)]


def test_load_images_order(tmp_path):
    names = ["b.png", "a.JPG", "c.txt", "a.png", "10.bmp", "2.webp", "x.tif", "noext", "d.jpeg"]
    img = np.full((4, 6, 3), 7, np.uint8)
    for n in names:
        if n.endswith(("png", "JPG", "bmp", "webp", "tif", "jpeg")):
            cv2.imwrite(str(tmp_path / n), img) if not n.endswith("JPG") else cv2.imwrite(str(tmp_path / "tmp.jpg"), img)
            if n.endswith("JPG"):
                os.rename(tmp_path / "tmp.jpg", tmp_path / n)
        else:
            (tmp_path / n).write_text("x")
    ds = D.LoadImages(str(tmp_path), 64, 32)
    expect = sorted(str(tmp_path / n) for n in names if n.split(".")[-1].lower() in D.img_formats)
    assert ds.files == expect and ds.nf == len(expect)
    got = list(ds)
    assert [p for p, _ in got] == expect and all(im.shape == (4, 6, 3) for _, im in got)
    assert D.LoadImages(str(tmp_path / "*.png"), 64).files == [str(tmp_path / "a.png"), str(tmp_path / "b.png")]
    assert D.LoadImages(str(tmp_path / "b.png"), 64).files == [str(tmp_path / "b.png")]
    with pytest.raises(Exception, match="does not exist"):
        D.LoadImages(str(tmp_path / "missing"), 64)
    (tmp_path / "clip.mp4").write_bytes(b"")
    with pytest.raises(NotImplementedError, match="video"):
        D.LoadImages(str(tmp_path), 64)


def test_increment_path(tmp_path):
    p = tmp_path / "exp"
    assert increment_path(p) == str(p)
    p.mkdir()
    assert increment_path(p, exist_ok=True) == str(p)
    assert increment_path(p, exist_ok=False) == str(tmp_path / "exp2")
    (tmp_path / "exp7").mkdir()
    (tmp_path / "expx").mkdir()
    assert increment_path(p, exist_ok=False) == str(tmp_path / "exp8")
    assert increment_path(p, exist_ok=False, sep="_") == str(tmp_path / "exp_2")


def _fixture_rows(g, k):
    """the reference's rows of frame k, restated on the host: numpy NMS of the fixture's z, then the torch CPU statements of
    detect.py:169,178"""
    img_size, conf, iou, _ = g["settings"]
    h0, w0 = g[f"frame{k}"].shape[:2]
    z = g[f"z{k}"]
    det = torch.from_numpy(restate.non_max_suppression(z, float(conf), float(iou))[0].copy())
    hw = (128, 256) if h0 == 160 else (192, 256)
    det[:, :4] = scale_coords(hw, det[:, :4], (h0, w0)).round()
    gn = torch.tensor((h0, w0, 3))[[1, 0, 1, 0]]
    xywhn = torch.cat([(xyxy2xywh(r[:4].view(1, 4)) / gn) for r in det]) if len(det) else torch.zeros((0, 4))
    return hw, det.numpy(), xywhn.numpy()


def test_printed_lines_and_txt_from_fixture():
    g = np.load(GOLD)
    lines = str(g["stdout"]).splitlines()
    n = int(g["n_frames"])
    for k in range(n):
        hw, det, xywhn = _fixture_rows(g, k)
        cc = np.bincount(det[:, 5].astype(np.int64), minlength=10)
        s = D.frame_string(hw, cc, NAMES)
        assert lines[k].endswith(": " + s + "Done. (<t>s)"), (lines[k], s)
        assert D.txt_lines(det, xywhn, True).encode() == g[f"txt{k}"].tobytes()
        short = D.txt_lines(det, xywhn, False).splitlines()
        assert [" ".join(x.split()[:5]) for x in g[f"txt{k}"].tobytes().decode().splitlines()] == short


def _random_case(rng, h, w):
    im0 = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
    mask = np.array(synth_palette(), np.uint8)[rng.integers(0, 19, (h, w))]
    boxes = []
    for _ in range(int(rng.integers(1, 12))):
        x1, x2 = sorted(rng.integers(-20, w + 20, 2))
        y1, y2 = sorted(rng.integers(-20, h + 20, 2))
        boxes.append((np.float32(np.clip(x1, 0, w)), np.float32(np.clip(y1, 0, h)), np.float32(np.clip(x2, 0, w)), np.float32(np.clip(y2, 0, h)),
                      float(rng.uniform(0, 1)), int(rng.integers(0, 10))))
    return im0, mask, boxes


def synth_palette():
    from multiyolov5_b200.utils.general import Cityscapes_COLORMAP
    return [c[::-1] for c in Cityscapes_COLORMAP]


@pytest.mark.parametrize("seed", range(12))
def test_dst_reblend_equals_full_blend(seed):
    rng = np.random.default_rng(seed)
    h, w = [(60, 90), (200, 320), (33, 517), (480, 640)][seed % 4]
    im0, mask, boxes = _random_case(rng, h, w)
    dst = cv2.addWeighted(mask, 0.4, im0, 0.6, 0)         # the device blends the undrawn frame (bit exact with this)
    drawn = im0.copy()
    rects = []
    names = ["person", "traffic light", "pg", "x", "bicycle", "q", "jy", "WWWWWWWW", "car", "g"]
    colors = [[int(v) for v in rng.integers(0, 255, 3)] for _ in names]
    for x1, y1, x2, y2, conf, c in boxes:
        label = f"{names[c]} {conf:.2f}"
        plot_one_box((x1, y1, x2, y2), drawn, label=label, color=colors[c], line_thickness=3)
        rects += box_extent((x1, y1, x2, y2), drawn.shape, label=label, line_thickness=3)
    changed = np.any(drawn != im0, axis=2)
    covered = np.zeros_like(changed)
    for a, b, c, d in rects:
        covered[a:b, c:d] = True
    assert not (changed & ~covered).any(), "drawing touched a pixel outside the extents"
    np.testing.assert_array_equal(reblend(dst.copy(), mask, drawn, rects), cv2.addWeighted(mask, 0.4, drawn, 0.6, 0))


def _opt(tmp_path, **kw):
    o = dict(weights="w.pt", source=str(tmp_path), img_size=256, conf_thres=0.25, iou_thres=0.45, device="", view_img=False,
             save_txt=False, save_conf=False, nosave=False, classes=None, agnostic_nms=False, augment=False, update=False,
             project=str(tmp_path / "runs"), name="exp", exist_ok=False, save_as_video=False, submit=False, batch_size=16)
    o.update(kw)
    return Namespace(**o)


@pytest.mark.parametrize("kw,match", [({"view_img": True}, "--view-img"), ({"update": True}, "--update"), ({"source": "0"}, "webcam"),
                                      ({"source": "streams.txt"}, "streams"), ({"source": "rtsp://host/x"}, "URL"),
                                      ({"source": "https://host/x.jpg"}, "URL"), ({"device": "cpu"}, "--device cpu")])
def test_refused_flags(tmp_path, kw, match):
    with pytest.raises(NotImplementedError, match=match):
        D.detect(_opt(tmp_path, **kw))
    assert not (tmp_path / "runs").exists()


def test_cli_flags():
    opt = D.parse_opt(["--weights", "a.pt", "--source", "d", "--img-size", "1024", "--submit", "--nosave", "--classes", "0", "2",
                       "--save-as-video", "--batch-size", "4"])
    assert opt.weights == ["a.pt"] and opt.img_size == 1024 and opt.submit and opt.nosave and opt.classes == [0, 2]
    assert opt.save_as_video and opt.batch_size == 4 and opt.project == "runs/detect" and opt.name == "exp"
