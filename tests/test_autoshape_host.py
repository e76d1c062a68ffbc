"""Host side of autoShape / Detections (multiyolov5_b200/models/common.py, reference models/common.py:605-752) against
tests/golden/autoshape_cases.npz (oracle/make_golden_autoshape.py): input normalisation, files, shape1 and each item's letterbox geometry
(a host cv2 letterbox with the table's numbers gives the reference's x), the printed lines and render() of Detections, tolist, and the
refusals.  No GPU."""
import os
import zlib

import cv2
import numpy as np
import pytest
import torch
from PIL import Image

from multiyolov5_b200.models.common import Detections, autoshape_inputs
from multiyolov5_b200.utils.datasets import LETTERBOX_ITEM, letterbox_item_table
from multiyolov5_b200.utils.general import SEG_CROP_ITEM, seg_crop_item_table
from oracle import synth
from oracle.make_golden_autoshape import make_input

GOLD = os.path.join(synth.GOLDEN_DIR, "autoshape_cases.npz")
NAMES = [f"cls{i}" for i in range(10)]


def _calls():
    g = np.load(GOLD)
    return g, sorted({int(k[1:k.index("_")]) for k in g.files if k.startswith("c")})


def given_inputs(g, c, folder):
    """the inputs of fixture call c as the reference was handed them, rebuilt from their kind, size and seed"""
    out, k = [], 0
    while f"c{c}_kind{k}" in g:
        kind = str(g[f"c{c}_kind{k}"])
        arr = make_input(kind, tuple(int(v) for v in g[f"c{c}_hw{k}"]), int(g[f"c{c}_seed{k}"]))
        assert zlib.crc32(arr.tobytes()) == int(g[f"c{c}_crc{k}"]), f"call {c} input {k} is not the one the fixture was made from"
        if kind == "pil_rgba":
            out.append(Image.fromarray(arr, "RGBA"))
        elif kind == "path":
            path = os.path.join(str(folder), str(g[f"c{c}_name{k}"]))
            Image.fromarray(arr).save(path)
            out.append(path)
        else:
            out.append(arr)
        k += 1
    return out


def test_item_sizes_match_the_c_structs():
    assert LETTERBOX_ITEM.itemsize == 56 and SEG_CROP_ITEM.itemsize == 32       # include/myolo.h


def test_inputs_files_shape1_and_geometry(tmp_path):
    g, calls = _calls()
    for c in calls:
        imgs, files, shape0, shape1 = autoshape_inputs(given_inputs(g, c, tmp_path), int(g[f"c{c}_size"]), 32)
        assert files == list(g[f"c{c}_files"])
        assert shape1 == list(g[f"c{c}_shape1"])
        x = g[f"c{c}_x"]
        assert all(im.dtype == np.uint8 and im.ndim == 3 and im.shape[2] == 3 for im in imgs)
        table = letterbox_item_table(shape0, shape1, [0] * len(imgs))
        for k, (im, it) in enumerate(zip(imgs, table)):
            assert (it["H0"], it["W0"]) == im.shape[:2] == tuple(shape0[k])
            r = cv2.resize(np.ascontiguousarray(im), (int(it["rw"]), int(it["rh"])), interpolation=cv2.INTER_LINEAR)
            H, W = shape1
            lb = cv2.copyMakeBorder(r, int(it["top"]), H - it["rh"] - it["top"], int(it["left"]), W - it["rw"] - it["left"],
                                    cv2.BORDER_CONSTANT, value=(114, 114, 114))
            np.testing.assert_array_equal(lb.transpose(2, 0, 1), x[k], err_msg=f"call {c} item {k}")
    # the cases the fixture is built to cover
    imgs, _, shape0, shape1 = autoshape_inputs(given_inputs(g, 0, tmp_path), int(g["c0_size"]), 32)
    t = letterbox_item_table(shape0, shape1, [0] * len(imgs))
    assert t["mode"][0] == 2 and t["scale_x"][0] == 2.0                       # exact 2x down-scale: cv2's area path
    assert (t["rh"] > t["H0"]).any()                                            # an up-scale
    uneven = [(H - rh - top) != top for H, rh, top in zip([shape1[0]] * len(t), t["rh"], t["top"])]
    assert any(uneven)
    assert len(autoshape_inputs(given_inputs(g, 1, tmp_path), int(g["c1_size"]), 32)[0]) == 1


def test_normalisation_kinds(tmp_path):
    rgb = np.arange(40 * 60 * 3, dtype=np.uint8).reshape(40, 60, 3)
    chw = np.ascontiguousarray(rgb.transpose(2, 0, 1))
    rgba = np.concatenate([rgb, np.zeros((40, 60, 1), np.uint8)], 2)
    path = str(tmp_path / "p.png")
    Image.fromarray(rgb).save(path)
    imgs, files, shape0, shape1 = autoshape_inputs([rgb, chw, rgb[:, :, 0], Image.fromarray(rgba, "RGBA"), path], 64, 32)
    for im in (imgs[0], imgs[1], imgs[3], imgs[4]):
        np.testing.assert_array_equal(im, rgb)
    np.testing.assert_array_equal(imgs[2], np.repeat(rgb[:, :, :1], 3, 2))
    assert files == ["image0.jpg", "image1.jpg", "image2.jpg", "image3.jpg", "p.jpg"]
    assert shape0 == [(40, 60)] * 5 and shape1 == [64, 64]
    one = autoshape_inputs(rgb, 640, 32)          # a single image, not in a list
    assert one[1] == ["image0.jpg"] and one[3] == [448, 640]


def test_refusals():
    with pytest.raises(NotImplementedError):
        autoshape_inputs(["https://example.com/a.jpg"], 640, 32)
    with pytest.raises(ValueError):
        autoshape_inputs([np.zeros((64, 64, 3))], 640, 32)
    d = Detections([np.zeros((8, 8, 3), np.uint8)], [torch.zeros(0, 6)], ["image0.jpg"], None, NAMES, (1, 3, 32, 32))
    with pytest.raises(NotImplementedError):
        d.show()
    with pytest.raises(NotImplementedError):
        d.pandas()


def _fixture_detections(g, c, tmp_path):
    imgs, files, shape0, shape1 = autoshape_inputs(given_inputs(g, c, tmp_path), int(g[f"c{c}_size"]), 32)
    n = len(imgs)
    get = lambda a: [torch.from_numpy(g[f"c{c}_{a}{k}"]) for k in range(n)]     # noqa: E731
    d = Detections(imgs, get("xyxy"), files, None, NAMES, (n, 3, *shape1), xywh=get("xywh"), xyxyn=get("xyxyn"), xywhn=get("xywhn"),
                   seg=[None] * n)
    d._t = (1.0, 2.0, 3.0)
    return d


def test_print_and_render_match_reference(tmp_path, capsys):
    g, calls = _calls()
    for c in calls:
        d = _fixture_detections(g, c, tmp_path)
        capsys.readouterr()
        d.print()
        lines = capsys.readouterr().out.splitlines()
        ref = str(g[f"c{c}_stdout"]).splitlines()
        assert lines[:-1] == ref[:-1]
        assert lines[-1].replace("1.0ms", "<t>ms").replace("2.0ms", "<t>ms").replace("3.0ms", "<t>ms") == ref[-1]
        for k, im in enumerate(d.render()):
            np.testing.assert_array_equal(im, g[f"c{c}_render{k}"], err_msg=f"call {c} image {k}")
        assert len(d) == d.n == len(d.files)


def test_tolist_keeps_files_names_and_times(tmp_path, capsys):
    g, _ = _calls()
    d = _fixture_detections(g, 0, tmp_path)
    items = d.tolist()
    assert len(items) == d.n
    for k, it in enumerate(items):
        assert it.files == [d.files[k]] and it.names == NAMES and it.t == d.t and it.s == d.s
        assert torch.equal(it.pred, d.pred[k]) and torch.equal(it.xywhn, d.xywhn[k]) and it.imgs is d.imgs[k]


def test_save_writes_files(tmp_path, capsys):
    g, _ = _calls()
    d = _fixture_detections(g, 1, tmp_path)
    d.save(str(tmp_path / "hub"))
    out = capsys.readouterr().out
    assert (tmp_path / "hub" / "image0.jpg").is_file()
    assert out == f"Saved image0.jpg to {tmp_path / 'hub'}\n"


def test_seg_crop_table_packs_maps():
    t = seg_crop_item_table([(1, 2, 30, 40), (0, 0, 10, 20)], [(7, 9), (5, 3)])
    assert list(t["offset"]) == [0, 63] and list(t["h0"]) == [7, 5] and list(t["rw"]) == [40, 20]
