"""GPU: autoShape (multiyolov5_b200/models/common.py, reference models/common.py:605-752) and its three kernels.

- myolo_letterbox_items: the reference's x (tests/golden/autoshape_cases.npz) bit for bit as uint8, fp32 and fp16, over mixed sizes,
  an exact 2x down-scale, up-scales, uneven pads and a batch of one.
- The post stage fed the reference's z and seg gives its xyxy, xywh, xyxyn, xywhn, render() arrays and printed lines.
- myolo_scale_boxes against torch's CPU statements over random geometries and at the clip edges.
- myolo_seg_crop_upsample_argmax against the torch composition: bit exact on fp32 (CPU torch), on fp16 only near-ties may differ.
- End to end, custom(ref_ckpt_tiny.pt)(imgs) equals the per-image composition of the public functions; tensor inputs and
  Model.autoshape()'s attributes."""
import os
import re

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from multiyolov5_b200.hub import custom
from multiyolov5_b200.models.common import autoShape, autoshape_inputs
from multiyolov5_b200.utils.datasets import letterbox, letterbox_geometry
from multiyolov5_b200.utils.general import (non_max_suppression, scale_boxes, scale_coords, scale_coords_geometry, seg_argmax,
                                            seg_crop_argmax, seg_crop_item_table, xyxy2xywh)
from oracle import synth
from tests.test_autoshape_host import given_inputs

pytestmark = pytest.mark.gpu

GOLD = os.path.join(synth.GOLDEN_DIR, "autoshape_cases.npz")
CKPT = os.path.join(synth.GOLDEN_DIR, "ref_ckpt_tiny.pt")
CONF, IOU = 0.0012, 0.45
CALLS = (0, 1)


@pytest.fixture(scope="module")
def model():
    m = custom(CKPT)
    m.conf, m.iou = CONF, IOU
    return m


def _staged(model, g, c, tmp_path):
    imgs, files, shape0, shape1 = autoshape_inputs(given_inputs(g, c, tmp_path), int(g[f"c{c}_size"]), 32)
    return imgs, files, model.stage(imgs, shape0, shape1, torch.device("cuda"))


@pytest.mark.parametrize("c", CALLS)
def test_letterbox_items_bit_exact(model, tmp_path, c):
    g = np.load(GOLD)
    _, _, st = _staged(model, g, c, tmp_path)
    x8 = torch.from_numpy(g[f"c{c}_x"])
    assert torch.equal(st.letterbox(torch.uint8).cpu(), x8)
    assert torch.equal(st.letterbox(torch.float32).cpu(), x8.float() / 255.)        # the reference's x (checked by the generator)
    assert torch.equal(st.letterbox(torch.float16).cpu(), x8.half() / 255.)        # `.type_as(p) / 255.` with a half p


def _events():
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
    for e in ev[:3]:
        e.record()
    return ev


@pytest.mark.parametrize("c", CALLS)
def test_post_stage_replays_reference(model, tmp_path, capsys, c):
    g = np.load(GOLD)
    imgs, files, st = _staged(model, g, c, tmp_path)
    z = torch.from_numpy(g[f"c{c}_z"]).cuda()
    seg = F.interpolate(torch.from_numpy(g[f"c{c}_seglow"]), scale_factor=8, mode="bilinear", align_corners=True).cuda()
    d = model.postprocess(imgs, files, st, torch.Size((len(imgs), 3, *st.shape1)), z, seg, _events())
    for k in range(d.n):
        for a in ("xyxy", "xywh", "xyxyn", "xywhn"):
            np.testing.assert_array_equal(getattr(d, a)[k].cpu().numpy(), g[f"c{c}_{a}{k}"], err_msg=f"{a} {k}")
    assert d.files == list(g[f"c{c}_files"])
    capsys.readouterr()
    d.print()
    out = [re.sub(r"[0-9.]+ms", "<t>ms", s) for s in capsys.readouterr().out.splitlines()]
    assert out == str(g[f"c{c}_stdout"]).splitlines()
    for k, im in enumerate(d.render()):
        np.testing.assert_array_equal(im, g[f"c{c}_render{k}"])


def test_scale_boxes_matches_torch_cpu():
    rng = np.random.default_rng(0)
    for trial in range(40):
        B, max_det = int(rng.integers(1, 9)), 300
        counts = rng.integers(0, max_det + 1, B).astype(np.int32)
        counts[0] = max_det
        rows = rng.random((B, max_det, 6)).astype(np.float32) * 100
        geoms, hw0 = [], []
        for b in range(B):
            if trial % 4 == 0:          # gains of exactly 2 and 0.5
                (h0, w0), hw = ((128, 256) if b % 2 else (512, 1024)), (256, 512)
            else:
                h0, w0 = int(rng.integers(16, 2500)), int(rng.integers(16, 2500))
                hw = (int(rng.integers(1, 60)) * 32, int(rng.integers(1, 60)) * 32)
            geoms.append(scale_coords_geometry(hw, (h0, w0)))
            hw0.append((hw, (h0, w0)))
            n, big = int(counts[b]), max(hw)
            r = rng.uniform(-0.2 * big, 1.2 * big, (n, 4)).astype(np.float32)
            edge = rng.random((n, 4)) < 0.15        # exactly on the pad, so the clip edge 0 is hit exactly
            pad = np.array([geoms[-1][0], geoms[-1][1]] * 2, np.float32)
            r[edge] = np.broadcast_to(pad, r.shape)[edge]
            rows[b, :n, :4] = r
            rows[b, :n, 5] = rng.integers(0, 10, n).astype(np.float32)
        d = torch.from_numpy(rows).cuda()
        xywh, xyxyn, xywhn = (t.cpu().numpy() for t in scale_boxes(d, torch.from_numpy(counts).cuda(), np.stack(geoms)))
        got = d.cpu().numpy()
        for b, (hw, (h0, w0)) in enumerate(hw0):
            n = int(counts[b])
            y = torch.from_numpy(rows[b, :n].copy())
            scale_coords(hw, y[:, :4], (h0, w0, 3))
            gn = torch.tensor([w0, h0, w0, h0, 1., 1.])
            np.testing.assert_array_equal(got[b, :n], y.numpy())
            np.testing.assert_array_equal(got[b, n:], rows[b, n:])
            np.testing.assert_array_equal(xywh[b, :n], xyxy2xywh(y).numpy())
            np.testing.assert_array_equal(xyxyn[b, :n], (y / gn).numpy())
            np.testing.assert_array_equal(xywhn[b, :n], (xyxy2xywh(y) / gn).numpy())
            if n:
                assert (got[b, :n, [0, 2]] <= w0).all() and (got[b, :n, :4] >= 0).all()


def _windows(rng, B, H, W):
    wins, shapes0 = [], []
    for _ in range(B):
        rh, rw = int(rng.integers(1, H + 1)), int(rng.integers(1, W + 1))
        top, left = int(rng.integers(0, H - rh + 1)), int(rng.integers(0, W - rw + 1))
        wins.append((top, left, rh, rw))
        shapes0.append((int(rng.integers(1, 300)), int(rng.integers(1, 300))))
    wins[0] = (0, 0, H, W)
    shapes0[-1] = (1, 1)
    return wins, shapes0


def test_seg_crop_argmax_fp32_bit_exact_with_torch():
    rng = np.random.default_rng(1)
    for B, C, H, W in [(3, 19, 64, 96), (1, 5, 32, 32), (6, 19, 40, 24)]:
        seg = torch.from_numpy(rng.normal(0, 2, (B, C, H, W)).astype(np.float32))
        seg[0, 3] = seg[0, 1]                       # exact ties: the lowest class id wins
        wins, shapes0 = _windows(rng, B, H, W)
        items = torch.from_numpy(seg_crop_item_table(wins, shapes0).view(np.uint8)).cuda()
        maps = seg_crop_argmax(seg.cuda(), items, shapes0)
        for i, ((top, left, rh, rw), hw) in enumerate(zip(wins, shapes0)):
            ref = F.interpolate(seg[i:i + 1, :, top:top + rh, left:left + rw], hw, mode="bilinear", align_corners=True).argmax(1)[0]
            assert maps[i].dtype == torch.uint8 and tuple(maps[i].shape) == hw
            assert torch.equal(maps[i].cpu().long(), ref), (B, C, H, W, i)


def test_seg_crop_argmax_fp16_differs_only_at_near_ties():
    rng = np.random.default_rng(2)
    B, C, H, W = 4, 19, 48, 64
    seg = (torch.from_numpy(rng.normal(0, 3, (B, C, H, W)).astype(np.float32))).half().cuda()
    wins, shapes0 = _windows(rng, B, H, W)
    items = torch.from_numpy(seg_crop_item_table(wins, shapes0).view(np.uint8)).cuda()
    maps = seg_crop_argmax(seg, items, shapes0)
    agree, total = 0, 0
    for i, ((top, left, rh, rw), hw) in enumerate(zip(wins, shapes0)):
        up = F.interpolate(seg[i:i + 1, :, top:top + rh, left:left + rw], hw, mode="bilinear", align_corners=True)[0].float()
        ref = up.argmax(0)
        top2 = up.topk(min(2, C), dim=0).values
        close = (top2[0] - top2[1]) <= 2e-2 * top2[0].abs().clamp_min(1.0)
        same = maps[i].long() == ref
        assert bool((same | close).all()), "disagreement away from an fp16 near-tie"
        agree, total = agree + int(same.sum()), total + same.numel()
    assert agree / total > 0.995


def _composition(m, imgs, size):
    """the per-image reference call composed of this library's public functions"""
    net = m.model
    ims, files, shape0, shape1 = autoshape_inputs(imgs, size, 32)
    out = []
    for im, s0 in zip(ims, shape0):
        lb = letterbox(np.ascontiguousarray(im), new_shape=shape1, auto=False)[0]
        x = (lb.permute(2, 0, 1)[None].cpu().float() / 255.).cuda()
        y = net(x)
        det = non_max_suppression(y[0][0], CONF, IOU)[0].cpu()
        scale_coords(shape1, det[:, :4], s0)
        gn = torch.tensor([s0[1], s0[0], s0[1], s0[0], 1., 1.])
        (rw, rh), _, _, (top, _, left, _) = letterbox_geometry(s0, shape1, auto=False)
        crop = y[1][:, :, top:top + rh, left:left + rw].contiguous()
        out.append((det, xyxy2xywh(det), det / gn, xyxy2xywh(det) / gn, seg_argmax(crop, s0, out_dtype=torch.uint8)[0].cpu()))
    return files, out


def test_end_to_end_equals_composition(model, tmp_path, capsys):
    g = np.load(GOLD)
    rng = np.random.default_rng(4)
    extra = [rng.integers(0, 256, (h, w, 3), dtype=np.uint8) for h, w in [(61, 333), (240, 180), (128, 128)]]
    for imgs, size in [(given_inputs(g, 0, tmp_path) + extra, 256), (given_inputs(g, 1, tmp_path), 192), (extra[1], 320)]:
        files, ref = _composition(model, imgs if isinstance(imgs, list) else [imgs], size)
        d = model(imgs, size=size)
        assert d.files == files and d.n == len(ref)
        for k, r in enumerate(ref):
            for a, b in zip((d.xyxy[k], d.xywh[k], d.xyxyn[k], d.xywhn[k], d.seg[k]), r):
                assert torch.equal(a.cpu(), b), k
        assert all(t >= 0 for t in d.t)
        d.print()
        assert capsys.readouterr().out.splitlines()[-1].startswith("Speed: ")


def test_tensor_input_and_autoshape_attributes(capsys):
    from multiyolov5_b200.models.experimental import attempt_load
    net = attempt_load(CKPT).cuda()
    m = net.autoshape()
    assert capsys.readouterr().out == "Adding autoShape... \n"
    assert isinstance(m, autoShape) and m.autoshape() is m
    assert m.names == net.names and m.yaml == net.yaml and torch.equal(m.stride, net.stride)
    x = torch.rand(2, 3, 128, 160).cuda()
    y, ref = m(x), net(x)
    assert torch.equal(y[0][0], ref[0][0]) and torch.equal(y[1], ref[1])
