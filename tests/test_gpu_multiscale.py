"""GPU: --multi-scale training (reference train.py:354-359).  The rescale kernel against torch's F.interpolate on the same card, bit for
bit; train steps through the det lane's shared workspace against the same steps through private plans (bar: the private plans' own
run-to-run spread over several runs, the idea of
test_gpu_train.py::test_concurrent_passes_keep_the_reference_order_of_running_statistics); the stale-backward and capacity checks; and a 40-step multi-scale run at imgsz 1024 fed by the device batch builders."""
import ctypes as C
import random

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import synth

pytestmark = pytest.mark.gpu

SIZES = list(range(512, 1537, 32))


def _resize(x, size, out_dtype):
    from multiyolov5_b200.train import resize_bilinear
    return resize_bilinear(x, size, out_dtype)


def _torch_ref(x, size):
    xf = x.float() / 255.0 if x.dtype == torch.uint8 else x
    return F.interpolate(xf, size=list(size), mode="bilinear", align_corners=False)


def _check(x, size):
    ref = _torch_ref(x, size)
    for dt in (torch.float32, torch.float16):
        out = _resize(x, size, dt)
        want = ref if dt == torch.float32 else ref.half()
        assert out.dtype == dt and out.shape == want.shape
        assert torch.equal(out, want), (tuple(x.shape), size, dt, float((out.float() - want.float()).abs().max()))


def test_rescale_equals_torch_from_1024_to_every_multiscale_size():
    g = torch.Generator(device="cuda").manual_seed(0)
    x8 = torch.randint(0, 256, (4, 3, 1024, 1024), dtype=torch.uint8, device="cuda", generator=g)
    x32 = torch.rand((4, 3, 1024, 1024), device="cuda", generator=g)
    for s in SIZES:
        _check(x8, (s, s))
        _check(x32, (s, s))


@pytest.mark.parametrize("H,W", [(512, 1024), (1024, 2048), (1000, 1000)])
def test_rescale_equals_torch_non_square_and_non_integral_ratios(H, W):
    from multiyolov5_b200.train import MultiScale
    g = torch.Generator(device="cuda").manual_seed(H + W)
    x8 = torch.randint(0, 256, (4, 3, H, W), dtype=torch.uint8, device="cuda", generator=g)
    x32 = torch.rand((4, 3, H, W), device="cuda", generator=g)
    sizes = [s for s in MultiScale(1024).shapes((H, W)) if s != (H, W)] + [(H + 7, W - 5), (H // 3 + 1, W // 7 + 3)]
    for size in sizes:
        _check(x8, size)
        _check(x32, size)
    x16 = x32.half()                                      # fp16 source: torch's half kernel
    for size in sizes[:6]:
        assert torch.equal(_resize(x16, size, torch.float16), F.interpolate(x16, size=list(size), mode="bilinear", align_corners=False))


def test_rescale_edge_cases_one_pixel_wide():
    g = torch.Generator(device="cuda").manual_seed(3)
    x8 = torch.randint(0, 256, (2, 3, 37, 1), dtype=torch.uint8, device="cuda", generator=g)
    for size in [(64, 1), (64, 32), (5, 3), (37, 1), (1, 1)]:
        _check(x8, size)
        _check(x8.transpose(2, 3).contiguous(), size[::-1])
    _check(torch.rand((1, 3, 1, 1), device="cuda", generator=g), (32, 64))


class _Fixed:
    def __init__(self, v):
        self.v = v

    def randrange(self, a, b):
        assert a <= self.v < b
        return self.v


def test_same_size_draw_returns_without_a_launch():
    from multiyolov5_b200.train import MultiScale
    ms = MultiScale(1024)
    x16 = torch.rand((4, 3, 1024, 1024), device="cuda").half()
    assert ms(x16, torch.float16, rng=_Fixed(1024)) is x16
    x8 = torch.randint(0, 256, (4, 3, 1024, 1024), dtype=torch.uint8, device="cuda")
    assert torch.equal(ms(x8, torch.float16, rng=_Fixed(1024)), (x8.float() / 255.0).half())    # still the /255 conversion
    assert torch.equal(ms(x8, torch.float32, rng=_Fixed(1030)), x8.float() / 255.0)             # 1030 // 32 * 32 == 1024
    out = ms(x8, torch.float32, rng=_Fixed(1536))
    assert out.shape == (4, 3, 1536, 1536) and torch.equal(out, _torch_ref(x8, (1536, 1536)))


# ---- train steps through the shared workspace ---------------------------------------------------------------------------------------
HYP = dict(lr0=0.01, momentum=0.937, weight_decay=5e-4, box=0.05, cls=0.5, cls_pw=1.0, obj=1.0, obj_pw=1.0, anchor_t=4.0, fl_gamma=0.0)
B = 4


def _model():
    from multiyolov5_b200.models.yolo import Model
    yml = "yolov5s_city_seg.yaml"
    cfg = synth.load_cfg(yml)
    model = Model(yml)
    model.load_state_dict(synth.synth_state_dict(synth.load_manifest("s_psp"), cfg, seed=1, gain=1.0))
    return model.cuda().train(), cfg


def _trainer(shared):
    from multiyolov5_b200.train import MultiScale, Trainer, scale_hyp
    model, cfg = _model()
    tr = Trainer(model, scale_hyp(HYP, nl=3, nc=cfg["nc"], imgsz=1024, total_batch_size=B), batch_size=B, init_scale=2.0 ** 10,
                 multi_scale=MultiScale(1024) if shared else None)
    return model, cfg, tr


def _batch(s, nc, seed):
    rs = np.random.RandomState(seed)
    imgs = synth.synth_image(B, s, s, seed=seed).cuda().half()
    t = np.zeros((24, 6), np.float32)
    t[:, 0] = rs.randint(0, B, 24); t[:, 1] = rs.randint(0, nc, 24)
    t[:, 2:4] = rs.uniform(0.1, 0.9, (24, 2)); t[:, 4:6] = rs.uniform(0.05, 0.3, (24, 2))
    return imgs, torch.from_numpy(t).cuda()


def _seg_batch(seed):
    rs = np.random.RandomState(seed)
    return synth.synth_image(B, 256, 512, seed=seed).cuda(), torch.from_numpy(rs.randint(-1, 19, (B, 256, 512)).astype(np.int64)).cuda()


def _run(shared, sizes, poison=False):
    model, cfg, tr = _trainer(shared)
    eng = model.engine()
    out = []
    segimgs, segtargets = _seg_batch(7)
    for k, s in enumerate(sizes):
        if poison and k:                                 # another shape's data in every byte: fp16 NaN patterns
            a = eng._arenas[0]
            a.ws.fill_(0xFF)
            a.gws.fill_(0xFF)
        imgs, targets = _batch(s, cfg["nc"], seed=s)
        items, segloss = tr.step(imgs, targets, segimgs, segtargets)
        out.append([float(v) for v in items] + [float(segloss)])
    torch.cuda.synchronize()
    state = {k: v.detach().float().cpu().clone() for k, v in model.state_dict().items()}
    plans = [p for key, p in eng.plans.items() if key[0] == "train" and len(key) == 4]
    assert all((p.arena is not None) == shared for p in plans)
    del tr, model, eng, plans
    torch.cuda.empty_cache()
    return np.array(out), state


def _spread(a, b):
    items = float(np.max(np.abs(a[0] - b[0]) / (np.abs(b[0]) + 1e-12)))
    stats = max(float((a[1][k] - b[1][k]).abs().max()) / (float(b[1][k].abs().max()) + 1e-12) for k in b[1] if "running_" in k)
    params = max(float((a[1][k] - b[1][k]).norm()) / (float(b[1][k].norm()) + 1e-12) for k in b[1]
                 if "running_" not in k and "num_batches" not in k and b[1][k].is_floating_point())
    return np.array([items, stats, params])


N_PRIVATE = 4


def _assert_within(shared, privates, what):
    """shared: one run through the shared workspace; privates: N_PRIVATE runs of the same steps through private plans.  The batch
    statistics and parameter gradients are summed with fp32 atomics, so the private runs differ among themselves.  Their spread is the
    largest distance between any two of them (per metric, over all pairs); the shared run's distance is its median distance to the
    private runs.  The metrics are maxima over many tensors, so every distance between two runs lands close to the same value: a run that
    behaves like one more private run comes out at 0.3 - 1.5 x the envelope (measured on the H100 over five repeats of the four tests),
    hence the factor 2.  A wrong workspace (stale or NaN bytes) gives O(1) differences."""
    pairs = [(i, j) for i in range(len(privates)) for j in range(len(privates)) if i != j]
    noise = np.max([_spread(privates[i], privates[j]) for i, j in pairs], axis=0)
    diff = np.median([_spread(shared, p) for p in privates], axis=0)
    print(f"\n{what}: shared vs private (items, running stats, parameters) {diff} (private envelope over {len(privates)} runs {noise})")
    assert np.isfinite(shared[0]).all()
    p0 = privates[0]
    for k in p0[1]:
        if k.endswith("num_batches_tracked"):
            assert int(shared[1][k]) == int(p0[1][k]), k
    floor = np.array([1e-4, 1e-5, 1e-6])
    assert (diff <= np.maximum(2 * noise, floor)).all(), (diff, noise)


@pytest.mark.parametrize("s", [512, 1024, 1536])
def test_step_through_shared_workspace_equals_private_plan(s):
    privates = [_run(False, [s]) for _ in range(N_PRIVATE)]
    _assert_within(_run(True, [s]), privates, f"one step at {s}")


def test_interleaved_shapes_over_a_poisoned_workspace_stay_exact():
    seq = [640, 1536, 640]
    privates = [_run(False, seq) for _ in range(N_PRIVATE)]
    _assert_within(_run(True, seq, poison=True), privates, "640 -> 1536 -> 640, workspace filled with 0xFF before each switch")


def test_backward_of_a_stale_forward_raises_before_launching():
    from multiyolov5_b200 import _lib
    model, cfg, tr = _trainer(True)
    eng = model.engine()
    xa, _ = _batch(512, cfg["nc"], 1)
    xb, _ = _batch(544, cfg["nc"], 2)
    raws_a, _, pa = eng.train_forward(xa, want_seg=False)
    gen_a = pa.fwd_generation
    raws_b, _, pb = eng.train_forward(xb, want_seg=False)
    assert pa.arena is pb.arena is not None
    with pytest.raises(_lib.MyoloError, match="stale"):
        eng.train_backward(pa, [torch.zeros_like(r) for r in raws_a], None, generation=gen_a)
    with pytest.raises(_lib.MyoloError, match="stale"):
        eng.train_backward(pa, [torch.zeros_like(r) for r in raws_a], None)
    eng.train_backward(pb, [torch.zeros_like(r) for r in raws_b], None, generation=pb.fwd_generation)   # the latest one is fine
    torch.cuda.synchronize()


def test_create_refuses_a_plan_larger_than_the_shared_workspace():
    from multiyolov5_b200 import _lib
    from multiyolov5_b200.plan import build_plan, to_ctypes
    model, _ = _model()
    pb = build_plan(model, B, 1536, 1536, train=True)
    ops, bufs, extra = to_ctypes(pb)
    ws = torch.zeros(1 << 20, dtype=torch.uint8, device="cuda")
    h = C.c_void_p()
    rc = _lib.lib().myolo_plan_create_shared(ops, len(pb.ops), bufs, len(pb.bufs), extra, len(pb.extra), B, 1536, 1536,
                                             int(pb.workspace_bytes), len(pb.slots), _lib.ptr(ws), _lib.ptr(ws), int(pb.workspace_bytes) - 256,
                                             C.byref(h))
    assert rc == -1 and not h.value                       # MYOLO_E_INVALID, no plan
    assert "workspace" in _lib.lib().myolo_last_error().decode()
    eng = model.engine()
    eng.reserve_train_shapes(B, [(512, 512)])
    with pytest.raises(_lib.MyoloError, match="cannot grow"):
        eng.reserve_train_shapes(B, [(1024, 1024)])      # the lane's workspace never moves under its plans
    eng.reserve_train_shapes(B, [(480, 480)])             # smaller shapes may join


def test_partial_last_batch_shares_the_reserved_workspace():
    """a det batch of fewer images than batch_size (the loader's last batch) binds to the same workspace, not to private ones"""
    model, cfg, tr = _trainer(True)
    eng = model.engine()
    a = eng._arenas[0]
    segimgs, segtargets = _seg_batch(5)
    for n, s in ((B, 1024), (2, 544), (B, 544), (2, 1536)):
        imgs, targets = _batch(s, cfg["nc"], seed=s)
        imgs, targets = imgs[:n].contiguous(), targets[targets[:, 0] < n].contiguous()
        items, segloss = tr.step(imgs, targets, segimgs, segtargets)
    torch.cuda.synchronize()
    assert torch.isfinite(items).all() and torch.isfinite(segloss).all()
    det = {key: p for key, p in eng.plans.items() if key[0] == "train" and len(key) == 4}
    assert set(det) == {("train", B, 1024, 1024), ("train", 2, 544, 544), ("train", B, 544, 544), ("train", 2, 1536, 1536)}
    assert all(p.arena is a for p in det.values()) and eng._arenas[0] is a


def test_every_multiscale_shape_runs_on_one_workspace_that_never_moves():
    model, cfg, tr = _trainer(True)
    eng = model.engine()
    a = eng._arenas[0]
    ptrs = (a.ws.data_ptr(), a.gws.data_ptr(), a.capacity)
    assert a.capacity == 3_047_912_448
    segimgs, segtargets = _seg_batch(3)
    for s in SIZES:
        imgs, targets = _batch(s, cfg["nc"], seed=s)
        items, segloss = tr.step(imgs, targets, segimgs, segtargets)
    torch.cuda.synchronize()
    assert torch.isfinite(items).all() and torch.isfinite(segloss).all()
    assert (eng._arenas[0].ws.data_ptr(), eng._arenas[0].gws.data_ptr(), eng._arenas[0].capacity) == ptrs
    det_plans = [p for key, p in eng.plans.items() if key[0] == "train" and len(key) == 4]
    assert len(det_plans) == 33 and all(p.arena is a for p in det_plans)
    print(f"\n33 det plans + seg plan: {torch.cuda.max_memory_allocated() / 1e9:.1f} GB peak allocated by torch, "
          f"{(torch.cuda.mem_get_info()[1] - torch.cuda.mem_get_info()[0]) / 1e9:.1f} GB in use on the card")


def test_forty_step_multiscale_run_on_device_batches():
    from multiyolov5_b200.utils.datasets import DetAugmenter, DeviceImageCache, DeviceSegCache, SegAugmenter
    model, cfg, tr = _trainer(True)
    ms = tr.multi_scale
    r = np.random.RandomState(1)
    det_imgs = [r.randint(0, 256, (600, 800, 3)).astype(np.uint8) for _ in range(4)]
    det_labels = [np.array([[k % cfg["nc"], 0.5, 0.5, 0.3, 0.2], [(k + 3) % cfg["nc"], 0.3, 0.6, 0.1, 0.2]], np.float32) for k in range(4)]
    det = DetAugmenter(DeviceImageCache(det_imgs, 1024, det_labels), dict(hsv_h=0.015, hsv_s=0.7, hsv_v=0.4, degrees=0.0, translate=0.1,
                                                                          scale=0.5, shear=0.0, perspective=0.0, flipud=0.0, fliplr=0.5,
                                                                          mosaic=1.0, mixup=0.0))
    seg_imgs = [r.randint(0, 256, (512, 1024, 3)).astype(np.uint8) for _ in range(4)]
    seg_masks = [r.randint(0, 34, (512, 1024)).astype(np.uint8) for _ in range(4)]
    seg = SegAugmenter(DeviceSegCache(seg_imgs, seg_masks), base_size=1024, crop_size=(1024, 512), preset="citys")
    random.seed(0); np.random.seed(0); torch.manual_seed(0)
    draws = random.Random(0)                              # the sizes' own stream: 40 draws reach 24 sizes, 512 and 1536 among them
    seen, losses = set(), []
    for _ in range(40):
        imgs, targets = det([0, 1, 2, 3], out_dtype=torch.uint8)
        imgs = ms(imgs, torch.float16, rng=draws)
        seen.add(tuple(imgs.shape[2:]))
        segimgs, segtargets = seg([0, 1, 2, 3])
        items, segloss = tr.step(imgs, targets, segimgs, segtargets)
        losses.append(torch.cat((items, segloss.reshape(1))))
    torch.cuda.synchronize()
    assert torch.isfinite(torch.stack(losses)).all()
    nbt = {int(v) for k, v in model.state_dict().items() if k.endswith("num_batches_tracked")}
    assert nbt == {80}, nbt                               # 40 steps x (det batch + seg batch)
    assert (1536, 1536) in seen and (512, 512) in seen and len(seen) >= 10, sorted(seen)
