"""GPU: model ensembles, Ensemble.forward (reference models/experimental.py:98-110 with the missing index restored and the seg mean).

The device path (each member's passes writing its z slice, one myolo_seg_ensemble launch for the seg) against torch composing the
ensemble over this library's single-model forwards on the card, bit for bit: z = cat of the members' z, seg = the mean of the members'
seg logits as `torch.stack(...).mean(0)` computes it, the class map its argmax.  Then detect() and test() over ensembles against the
same composition behind their public functions."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from multiyolov5_b200 import _lib
from multiyolov5_b200.models.experimental import Ensemble, attempt_load
from oracle import restate, restate_ensemble, synth
from tests.test_gpu_parity import CAPS
from tests.test_gpu_sizes import nms_recall
from tests.test_gpu_detect import NAMES, _compose, _frames, _opt, _read, video  # noqa: F401  (video: fixture)

pytestmark = pytest.mark.gpu

SPECS = {"s_psp": ("yolov5s_city_seg.yaml", 1), "s_bise": ("yolov5s_city_seg_bise.yaml", 2), "m_psp": ("yolov5m_city_seg.yaml", 3),
         "m_lab": ("yolov5m_city_seg_lab.yaml", 4), "s_base": ("yolov5s_city_seg_base.yaml", 5)}
SETS = {1: ["s_psp"], 2: ["s_psp", "m_psp"], 3: ["s_psp", "s_bise", "m_psp"], 5: ["s_psp", "s_bise", "m_psp", "m_lab", "s_base"]}
CKPTS = [os.path.join(synth.GOLDEN_DIR, f) for f in ("ref_ckpt_tiny.pt", "ref_ckpt_tiny_syncbn.pt")]


def build(tag):
    from multiyolov5_b200.models.yolo import Model
    yml, seed = SPECS[tag]
    m = Model(yml)
    m.load_state_dict(synth.synth_state_dict(synth.load_manifest(tag), synth.load_cfg(yml), seed=seed))
    return m.cuda().eval()


@pytest.fixture(scope="module")
def members():
    return {tag: build(tag) for tag in SPECS}


def compose(models, x, augment=False):
    """the definition: torch over the members' own forwards"""
    outs = [m(x, augment=augment) for m in models]
    z = torch.cat([o[0][0] for o in outs], 1)
    plain = outs if not augment else [m(x) for m in models]
    mean = torch.stack([o[1].float() for o in plain]).mean(0)
    return z, mean.to(plain[0][1].dtype), mean.argmax(1)


def ensemble(models):
    e = Ensemble()
    for m in models:
        e.append(m)
    return e.eval()


@pytest.mark.parametrize("K", sorted(SETS))
@pytest.mark.parametrize("shape", [(1, 512, 1024), (2, 128, 192)], ids=["512x1024", "4px"])
@pytest.mark.parametrize("dtype", [torch.float16, torch.float32])
def test_forward_equals_composition(members, K, shape, dtype):
    models = [members[t] for t in SETS[K]]
    B, H, W = shape
    x = synth.synth_image(B, H, W, seed=K).cuda().to(dtype)
    z0, seg0, amax0 = compose(models, x)
    e = ensemble(models)
    (z, none), seg = e(x)
    assert none is None and seg.dtype == seg0.dtype == dtype
    assert torch.equal(z, z0)
    assert torch.equal(seg, seg0)
    (z2, _), seg2, amax = e(x, seg_argmax=True)
    assert seg2 is None and torch.equal(z2, z0) and torch.equal(amax, amax0)


@pytest.mark.parametrize("K", [2, 3])
def test_augment_equals_composition(members, K):
    models = [members[t] for t in SETS[K]]
    x = synth.synth_image(2, 256, 512, seed=7).cuda().half()
    z0, seg0, amax0 = compose(models, x, augment=True)
    e = ensemble(models)
    (z, _), seg = e(x, augment=True)
    assert torch.equal(z, z0) and torch.equal(seg, seg0)
    (z, _), _, amax = e(x, augment=True, seg_argmax=True)
    assert torch.equal(z, z0) and torch.equal(amax, amax0)


def test_same_member_twice(members):
    """one Model listed twice shares its plan: the second pass rewrites the same logits, and the result is still the composition"""
    m = members["s_psp"]
    x = synth.synth_image(1, 256, 512, seed=3).cuda()
    z0, seg0, _ = compose([m, m, members["s_bise"]], x)
    (z, _), seg = ensemble([m, m, members["s_bise"]])(x)
    assert torch.equal(z, z0) and torch.equal(seg, seg0)


@pytest.mark.parametrize("K", [4, 5])
def test_forward_equals_composition_past_32bit_offsets(members, K):
    """16 x 19 x 512 x 1024 fp32 maps: four or five of them stacked span more than 2^31 bytes, so torch reduces the member axis in parts
    ((m0 + m1) + (m2 + m3) at K = 4, (m0 + m1) + ((m2 + m3) + m4) at K = 5) and the kernel must group its sums the same way"""
    models = [members[t] for t in SETS[5][:K]]
    assert K * 16 * 19 * 512 * 1024 * 4 > 2 ** 31
    x = torch.rand((16, 3, 512, 1024), device="cuda", generator=torch.Generator(device="cuda").manual_seed(K))
    z0, seg0, amax0 = compose(models, x)
    (z, _), seg = ensemble(models)(x)
    assert seg.dtype == torch.float32 and torch.equal(z, z0) and torch.equal(seg, seg0)
    del seg, seg0
    _, _, amax = ensemble(models)(x, seg_argmax=True)
    assert torch.equal(amax, amax0)
    del z, z0, amax, amax0
    torch.cuda.empty_cache()


GOLD = os.path.join(synth.GOLDEN_DIR, "ensemble_cases.npz")


def _errors(z, seg, ids, g, k):
    """distances of an ensemble's outputs from the reference's fp32 ensemble on the fixture's samples"""
    zr, zs = g[f"case{k}_z"].astype(np.float64), z.float().cpu().numpy()[:, g[f"case{k}_rows"]].astype(np.float64)
    d = np.abs(zs[..., :4] - zr[..., :4]).max(-1)
    size = np.maximum(zr[..., 2], zr[..., 3])
    sr = g[f"case{k}_seg"].astype(np.float64)
    ss = seg.float().cpu().numpy().reshape(-1)[g[f"case{k}_seg_idx"]].astype(np.float64)
    d_ref = restate.non_max_suppression(g[f"case{k}_z"], 0.25, 0.45)
    d_got = restate.non_max_suppression(zs.astype(np.float32), 0.25, 0.45)
    return {"box_px_max_le256": float(d[size <= 256.0].max(initial=0.0)), "box_rel_max": float((d / np.maximum(size, 8.0)).max()),
            "score_abs_max": float(np.abs(zs[..., 4:] - zr[..., 4:]).max()), "seg": float(np.abs(ss - sr).max() / np.abs(sr).max()),
            "ids_agree": float((ids.cpu().numpy() == g[f"case{k}_ids"]).mean()),
            "nms_recall": float(np.mean([nms_recall(r, o) for r, o in zip(d_ref, d_got)])), "n_ref_dets": sum(len(r) for r in d_ref)}


@pytest.mark.parametrize("k", [0, 1])
def test_parity_with_reference_fixture(k):
    """the ensemble on the card against the reference's own fp32 ensemble (oracle/make_golden_ensemble.py, three mixed-head members): no
    further away than torch's fp16 run of the same ensemble x 1.25 (tests/test_gpu_parity.py's rule), the NMS rows of the sampled z and
    the seg class ids included"""
    g = np.load(GOLD)
    x = restate_ensemble.fixture_input(g, k).cuda()
    members_sd = restate_ensemble.fixture_members(g)
    from multiyolov5_b200.models.yolo import Model
    models = []
    for (tag, yml, seed), (cfg, sd) in zip(g["members"], members_sd):
        m = Model(str(yml))
        m.load_state_dict(sd)
        models.append(m.cuda().eval())
    e = ensemble(models)
    (z, _), seg = e(x)
    _, _, ids = e(x, seg_argmax=True)
    ours = _errors(z, seg, ids, g, k)
    yz, yseg, yids = restate_ensemble.model_forward_ensemble([(cfg, {n: t.cuda() for n, t in sd.items()}) for cfg, sd in members_sd], x,
                                                             half=True)
    yard = _errors(yz, yseg, yids, g, k)
    print(f"\n[ensemble case {k}] ours vs fp32: {ours}\n  torch fp16 vs fp32: {yard}")
    assert z.shape[1] == 3 * (z.shape[1] // 3) and yz.shape == z.shape
    assert ours["seg"] <= 1.25 * yard["seg"] + 2e-4, (ours["seg"], yard["seg"])
    for key in ("box_px_max_le256", "box_rel_max", "score_abs_max"):
        assert ours[key] <= CAPS[key], (key, ours[key])
        if key != "box_rel_max" or k > 0:
            assert ours[key] <= 1.25 * yard[key] + 1e-3, (key, ours[key], yard[key])
    # at 1 x 64 x 128 the relative box error is that of sub-pixel errors on boxes of at most 8 px (the 8 px floor of its denominator):
    # the members' own forwards, whose rows z holds bit for bit, measured 0.022 against torch fp16's 0.015 there.  That size is on the
    # CUDA-core conv kernel, where tests/test_gpu_parity.py bounds each model by its absolute caps; at 1 x 256 x 512 the x 1.25 rule holds
    assert ours["ids_agree"] >= yard["ids_agree"] - 4e-3, (ours["ids_agree"], yard["ids_agree"])
    assert ours["n_ref_dets"] > 0 and ours["nms_recall"] >= yard["nms_recall"] - 0.02, (ours["nms_recall"], yard["nms_recall"])


def _edge_width(K, ncls, optin):
    """the widest W (a multiple of 32) whose K staged source rows fit in `optin` bytes, and the next multiple of 32"""
    fits = lambda W: K * ncls * ((W // 8 + 2) | 1) * 4 <= optin   # noqa: E731  (myolo_seg_ensemble's bound)
    W = 32
    while fits(W + 32):
        W += 32
    return W, W + 32


def test_kernel_at_shared_memory_edge(members):
    models = [members[t] for t in SETS[5]]
    optin = torch.cuda.get_device_properties(0).shared_memory_per_block_optin
    W, W_over = _edge_width(5, 19, optin)
    assert 5 * 19 * ((W // 8 + 2) | 1) * 4 > 48 * 1024          # the launch opts in past the default 48 KB
    x = synth.synth_image(1, 64, W, seed=11).cuda()
    z0, seg0, amax0 = compose(models, x)
    (z, _), seg = ensemble(models)(x)
    assert torch.equal(z, z0) and torch.equal(seg, seg0)
    _, _, amax = ensemble(models)(x, seg_argmax=True)
    assert torch.equal(amax, amax0)
    x = synth.synth_image(1, 64, W_over, seed=11).cuda()
    with pytest.raises(_lib.MyoloError, match="shared memory"):
        ensemble(models)(x)


def test_entry_point_refuses_mismatched_plans(members):
    e = ensemble([members["s_psp"], members["m_psp"]])
    e(synth.synth_image(1, 128, 256, seed=1).cuda())
    a = members["s_psp"].engine().plans[(1, 128, 256)]
    members["m_psp"](synth.synth_image(1, 128, 320, seed=1).cuda())
    b = members["m_psp"].engine().plans[(1, 128, 320)]
    L = _lib.lib()
    seg = torch.empty((1, 19, 128, 256), device="cuda")
    plans = (C.c_void_p * 2)(a.handle.value, b.handle.value)
    assert L.myolo_seg_ensemble(plans, 2, _lib.ptr(seg), _lib.F32, None, _lib.stream_ptr()) == -1
    assert b"member 1" in L.myolo_last_error()
    plans = (C.c_void_p * 9)(*([a.handle.value] * 9))
    assert L.myolo_seg_ensemble(plans, 9, _lib.ptr(seg), _lib.F32, None, _lib.stream_ptr()) == -1


def test_no_host_synchronisation(members):
    models = [members[t] for t in SETS[3]]
    e = ensemble(models)
    x = synth.synth_image(2, 256, 512, seed=5).cuda().half()
    e(x), e(x, augment=True), e(x, seg_argmax=True)              # plans built, weights packed
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        for kw in (dict(), dict(augment=True), dict(seg_argmax=True)):
            e(x, **kw)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    torch.cuda.synchronize()


class Composed(torch.nn.Module):
    """a stand-in whose forward is the composition over the members"""

    def __init__(self, models, names=None):
        super().__init__()
        self.m = torch.nn.ModuleList(models)
        self.names = names

    def forward(self, x, augment=False):
        z, seg, _ = compose(list(self.m), x, augment=augment)
        return [(z, None), seg]


@pytest.fixture(scope="module")
def ckpt_ensemble():
    return attempt_load(CKPTS).cuda().eval()


@pytest.mark.parametrize("augment", [False, True], ids=["plain", "augment"])
def test_detect_two_weights_equals_composition(tmp_path, capsys, video, ckpt_ensemble, augment):  # noqa: F811
    from multiyolov5_b200 import detect as D
    frames = _frames()[:6]
    opt = _opt(tmp_path, augment=augment, batch_size=3, weights=CKPTS)
    np.random.seed(5)
    colors = [[np.random.randint(0, 255) for _ in range(3)] for _ in NAMES]
    files, txt, lines, vid = _compose(Composed(list(ckpt_ensemble)), opt, frames, colors)
    capsys.readouterr()
    np.random.seed(5)
    save_dir = D.detect(opt, dataset=frames)                     # attempt_load(opt.weights): the two checkpoints
    out = capsys.readouterr().out.splitlines()
    assert out[0].startswith("Ensemble created with ")
    assert [s.rsplit("Done. (", 1)[0] for s in out[2:2 + len(frames)]] == lines
    for rel, a in files.items():
        np.testing.assert_array_equal(_read(save_dir / rel), a, err_msg=rel)
    assert {str(p.relative_to(save_dir)) for p in save_dir.rglob("*.png")} == set(files)
    assert {p.stem: p.read_text() for p in (save_dir / "labels").glob("*.txt")} == txt
    assert len(video.frames) == len(vid) and all(np.array_equal(a, b) for a, b in zip(video.frames, vid))


def _loader(seed=0):
    from tests.test_gpu_val import _cases, _shapes
    z, meta = _cases()
    m = meta["main"]
    g = torch.Generator().manual_seed(seed)
    loader = []
    for bi in range(m["n_batches"]):
        shp = _shapes(z[f"main_shapes_{bi}"])
        H, W = m["hw"][bi]
        img = torch.randint(0, 256, (len(shp), 3, H, W), dtype=torch.uint8, generator=g)
        loader.append((img, torch.from_numpy(z[f"main_targets_{bi}"]), [f"im{bi}_{i}.jpg" for i in range(len(shp))], shp))
    return loader


def test_test_with_ensemble_equals_composition(members, tmp_path):
    from multiyolov5_b200 import test as T
    models = [build("s_psp"), build("s_bise")]
    names = [f"c{i}" for i in range(10)]
    loader = _loader()
    e = ensemble(models)
    e.names = names
    seen = []
    e.register_forward_pre_hook(lambda mod, args: seen.append(next(mod[1].parameters()).dtype))
    kw = dict(plots=False, conf_thres=0.1, save_txt=True, save_conf=True)
    got = T.test({"nc": 10}, model=e, dataloader=loader, save_dir=tmp_path / "e", **kw)
    assert seen and set(seen) == {torch.float16}                   # model.half() reached every member
    ref = T.test({"nc": 10}, model=Composed(models, names), dataloader=loader, save_dir=tmp_path / "c", **kw)
    assert got[0] == ref[0] and np.array_equal(got[1], ref[1])
    txt = {p.name: p.read_text() for p in (tmp_path / "e" / "labels").glob("*.txt")}
    assert txt and txt == {p.name: p.read_text() for p in (tmp_path / "c" / "labels").glob("*.txt")}
    with pytest.raises(ValueError, match="compute_loss"):
        T.test({"nc": 10}, model=e, dataloader=loader, compute_loss=lambda *a: None)
    g = torch.Generator().manual_seed(1)
    seg_loader = [(img.cuda().float() / 255.0, torch.randint(0, 19, (img.shape[0], img.shape[2], img.shape[3]), generator=g).cuda())
                  for img, _, _, _ in loader[:1]]
    got = T.seg_validation(e, 19, seg_loader, "cuda")
    ref = T.seg_validation(Composed(models), 19, seg_loader, "cuda")
    assert got == ref
