"""GPU: detection validation batches on the device (DeviceImageCache(augment=False), DetValLoader, myolo_resize_area_u8) against the
unmodified reference's rect loader (tests/golden/val_batch_cases.npz) and the numpy restatement (oracle/restate_val_batches.py) at full
size, and test() fed by the loader against test() fed by host-built batches.  Bit exact, no tolerance.  Items are compared keyed by
source index: numpy's argsort permutes equal aspect ratios in a CPU-dependent order."""
import ctypes as C
import json
import os

import numpy as np
import pytest
import torch

from oracle import restate_val_batches as RV

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden", "val_batch_cases.npz")


def _cases():
    z = np.load(GOLD)
    meta = json.loads(bytes(z["meta_json"]).decode())
    n = len(meta["shapes"])
    return z, meta, [z[f"src_{k}"] for k in range(n)], [z[f"labels_{k}"] for k in range(n)]


def _area_dev(img, W, H):
    from multiyolov5_b200 import _lib
    src = torch.from_numpy(img).cuda()
    dst = torch.empty((H, W, 3), dtype=torch.uint8, device="cuda")
    _lib.check(_lib.lib().myolo_resize_area_u8(_lib.ptr(src), img.shape[0], img.shape[1], _lib.ptr(dst), H, W, _lib.stream_ptr()))
    return dst.cpu().numpy()


@pytest.mark.parametrize("name", ["main", "single_cls", "big_batch"])
def test_cache_matches_reference(name):
    from multiyolov5_b200.utils.datasets import DeviceImageCache
    z, meta, srcs, labels = _cases()
    cache = DeviceImageCache(srcs, meta["cases"][name]["img_size"], labels, augment=False)
    assert cache.augment is False
    for k in range(len(srcs)):
        assert np.array_equal(cache.image(k).cpu().numpy(), z[f"{name}_cache_{k}"]), k


@pytest.mark.parametrize("name", ["main", "single_cls", "big_batch"])
def test_loader_matches_reference(name):
    from multiyolov5_b200.utils.datasets import DetValLoader, DeviceImageCache
    z, meta, srcs, labels = _cases()
    c = meta["cases"][name]
    loader = DetValLoader(DeviceImageCache(srcs, c["img_size"], labels, augment=False), c["batch_size"], single_cls=c["single_cls"])
    assert len(loader) == c["n_batches"] and np.array_equal(loader.batch_shapes, z[f"{name}_batch_shapes"])
    ar = np.array([h / w for h, w in meta["shapes"]], np.float64)
    assert np.array_equal(loader.order, np.argsort(ar))
    for b, (img, targets, paths, shapes) in enumerate(loader):
        assert img.is_cuda and targets.is_cuda and img.dtype == torch.uint8 and targets.dtype == torch.float32
        ref_paths = z[f"{name}_paths_{b}"].tolist()
        ref_img, ref_t, ref_s = z[f"{name}_img_{b}"], z[f"{name}_targets_{b}"], z[f"{name}_shapes_{b}"]
        img, targets = img.cpu().numpy(), targets.cpu().numpy()
        assert img.shape == ref_img.shape and sorted(paths) == sorted(ref_paths) and len(targets) == len(ref_t)
        for pos, i in enumerate(paths):
            rpos = ref_paths.index(i)
            assert np.array_equal(img[pos], ref_img[rpos]), (b, i)
            assert np.array_equal(targets[targets[:, 0] == pos, 1:], ref_t[ref_t[:, 0] == rpos, 1:]), (b, i)
            (h0, w0), ((gh, gw), (pw, ph)) = shapes[pos]
            assert np.array_equal(np.array([h0, w0, gh, gw, pw, ph], np.float64), ref_s[rpos]), (b, i)


@pytest.mark.parametrize("H0,W0,H,W", [(1024, 2048, 320, 640), (1024, 2048, 512, 1024), (720, 1280, 576, 1024), (720, 1280, 360, 640),
                                       (1080, 1920, 360, 640), (1080, 1920, 1080, 1920), (1081, 1921, 363, 641), (517, 333, 101, 97),
                                       (37, 41, 36, 1), (41, 1, 7, 1), (64, 96, 21, 1)])
def test_area_resize_full_size(H0, W0, H, W):
    rs = np.random.RandomState(H0 * 7 + W)
    img = rs.randint(0, 256, (H0, W0, 3)).astype(np.uint8)
    assert np.array_equal(_area_dev(img, W, H), RV.cv2_resize_area_u8(img, W, H)), RV.area_path(H0, W0, H, W)


def test_area_resize_rejects_upscaling():
    from multiyolov5_b200 import _lib
    L = _lib.lib()
    src = torch.zeros((32, 48, 3), dtype=torch.uint8, device="cuda")
    dst = torch.zeros((64, 64, 3), dtype=torch.uint8, device="cuda")
    for H, W in ((33, 48), (32, 49), (64, 64)):
        assert L.myolo_resize_area_u8(_lib.ptr(src), 32, 48, _lib.ptr(dst), H, W, _lib.stream_ptr()) == -1   # MYOLO_E_INVALID
    assert b"down-scaling" in L.myolo_last_error()


def test_loader_rejects_training_cache_and_repeats():
    from multiyolov5_b200.utils.datasets import DetValLoader, DeviceImageCache
    z, meta, srcs, labels = _cases()
    with pytest.raises(ValueError):
        DetValLoader(DeviceImageCache(srcs[:3], 64, labels[:3]), 2)
    loader = DetValLoader(DeviceImageCache(srcs, 96, labels, augment=False), 4)
    first = [(i.cpu(), t.cpu(), p, s) for i, t, p, s in loader]
    second = [(i.cpu(), t.cpu(), p, s) for i, t, p, s in loader]
    assert len(first) == len(second) == len(loader)
    for a, b in zip(first, second):
        assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1]) and a[2] == b[2] and a[3] == b[3]


def _psp_model():
    from multiyolov5_b200.models.yolo import Model
    from oracle import synth
    yml = "yolov5s_city_seg.yaml"
    cfg = synth.load_cfg(yml)
    model = Model(yml)
    model.load_state_dict(synth.synth_state_dict(synth.load_manifest("s_psp"), cfg, seed=1))
    return model.cuda().eval(), cfg


def test_test_fed_by_loader_equals_host_batches():
    from multiyolov5_b200.test import test
    from multiyolov5_b200.utils.datasets import DetValLoader, DeviceImageCache
    from multiyolov5_b200.utils.general import non_max_suppression
    model, cfg = _psp_model()
    rs = np.random.RandomState(7)
    sizes = [(360, 640), (400, 300), (256, 256), (300, 540), (512, 1024), (150, 200), (700, 420)]
    imgs = [np.kron(rs.randint(0, 256, (h // 9 + 1, w // 9 + 1, 3)), np.ones((9, 9, 1), np.int64))[:h, :w].astype(np.uint8)
            for h, w in sizes]
    s = 256
    cache = DeviceImageCache(imgs, s, augment=False)
    model.half()
    labels = [np.zeros((0, 5), np.float32) for _ in imgs]      # labels near some of the model's own boxes: some predictions are correct
    for img, _, paths, shapes in DetValLoader(cache, 3):
        with torch.no_grad():
            out = model(img.half() / 255.0)[0][0]
        for pos, (d, i) in enumerate(zip(non_max_suppression(out, 0.001, 0.6, multi_label=True), paths)):
            d = d[:10].cpu().numpy().astype(np.float64)
            (h0, w0), ((gh, gw), (pw, ph)) = shapes[pos]
            h, w = h0 * gh, w0 * gw
            xc, yc = ((d[:, 0] + d[:, 2]) / 2 - pw) / w, ((d[:, 1] + d[:, 3]) / 2 - ph) / h
            bw, bh = (d[:, 2] - d[:, 0]) / w, (d[:, 3] - d[:, 1]) / h
            labels[i] = np.clip(np.stack([d[:, 5], xc, yc, bw * 1.02, bh * 1.02], 1), 0, 1).astype(np.float32)
            labels[i][:, 0] = d[:, 5]
    model.float()
    cache.labels = labels
    loader = DetValLoader(cache, 3)
    host = []
    cached = [RV.load_image_val(im, s) for im in imgs]
    for b, batch in enumerate(loader.batches):
        host.append((torch.from_numpy(RV.val_batch_images([cached[i] for i in batch.indices], loader.batch_shapes[b])),
                     torch.from_numpy(batch.targets), batch.indices, batch.shapes))
    for (di, dt, _, _), (hi, ht, _, _) in zip(loader, host):
        assert torch.equal(di.cpu(), hi) and torch.equal(dt.cpu(), ht)
    res_dev, maps_dev, _ = test({"nc": cfg["nc"]}, model=model, dataloader=loader, plots=False)
    res_host, maps_host, _ = test({"nc": cfg["nc"]}, model=model, dataloader=host, plots=False)
    assert res_dev[2] > 0
    assert res_dev == res_host and np.array_equal(maps_dev, maps_host)
