"""CPU tests of the validation statistics: the numpy restatement (oracle/restate_val.py) against the unmodified reference's fixtures
(tests/golden/val_cases.npz, oracle/make_golden_val.py) and against np.interp / np.trapz, plus the host logic of utils.metrics and test."""
import json
import os
import warnings

import numpy as np
import pytest
import torch

from oracle import restate_val as R

GOLD = os.path.join(os.path.dirname(__file__), "golden", "val_cases.npz")


def _cases():
    z = np.load(GOLD)
    return z, json.loads(bytes(z["meta_json"]).decode())


def restated_case(z, name, meta):
    """per-image (correct, conf, pcls, tcls) from the reference's CPU NMS rows of the fixture z, through the restated matching"""
    from oracle import restate
    stats = []
    for bi in range(meta["n_batches"]):
        zz, tg, shp = z[f"{name}_z_{bi}"], z[f"{name}_targets_{bi}"], z[f"{name}_shapes_{bi}"]
        hw = meta["hw"][bi]
        dets = restate.non_max_suppression(zz, 0.001, 0.6, multi_label=True)
        for si, d in enumerate(dets):
            d = np.asarray(d, np.float32)
            labels = tg[tg[:, 0] == si, 1:]
            s = shp[si]
            g = R.geometry(hw, ((s[0], s[1]), ((s[2], s[3]), (s[4], s[5]))))
            if len(d) == 0:
                if len(labels):
                    stats.append((np.zeros((0, 10), bool), np.zeros(0, np.float32), np.zeros(0, np.float32), labels[:, 0]))
                continue
            stats.append((R.match_image(d, labels, hw, g), d[:, 4], d[:, 5], labels[:, 0]))
    return stats


def test_iouv_table():
    assert np.array_equal(R.IOUV, torch.linspace(0.5, 0.95, 10).numpy())


@pytest.mark.parametrize("name", ["main", "single_cls", "no_tp"])
def test_restatement_equals_reference_fixtures(name):
    z, meta = _cases()
    m = meta[name]
    stats = restated_case(z, name, m)
    if m["ap_called"]:
        cat = [np.concatenate(x, 0) for x in zip(*stats)]
        assert np.array_equal(cat[0], z[f"{name}_correct"])
        assert np.array_equal(cat[1], z[f"{name}_conf"]) and np.array_equal(cat[2], z[f"{name}_pcls"])
        assert np.array_equal(cat[3], z[f"{name}_tcls"])
        p, r, ap, f1, cls = R.ap_per_class(z[f"{name}_correct"], z[f"{name}_conf"], z[f"{name}_pcls"], z[f"{name}_tcls"])
        for k, v in dict(p=p, r=r, ap=ap, f1=f1, ap_class=cls).items():
            assert np.array_equal(v, z[f"{name}_{k}"]), k
    res = R.test_statistics(stats, m["nc"])
    assert np.array_equal(np.array([res["mp"], res["mr"], res["map50"], res["map"]]), z[f"{name}_results"][:4])
    assert np.array_equal(res["maps"], z[f"{name}_maps"])


def test_fixture_covers_edge_cases():
    z, meta = _cases()
    c = z["main_correct"]
    assert c.any() and not c.all() and len(np.unique(c.sum(1))) >= 8       # rows cut at most of the thresholds
    assert not z["no_tp_results"][:4].any() and "no_tp_correct" not in z.files
    for name in ("main", "single_cls"):
        conf, pcls = z[f"{name}_conf"], z[f"{name}_pcls"]
        for c_ in np.unique(pcls):
            v = conf[pcls == c_]
            assert len(np.unique(v)) == len(v)           # no within-class ties


def test_interp_and_pairwise_equal_numpy():
    rs = np.random.RandomState(0)
    for _ in range(500):
        n = rs.randint(1, 80)
        xp = np.sort(rs.choice(rs.rand(rs.randint(1, n + 1)), n))      # repeated values
        fp = rs.rand(n)
        x = rs.rand(300) * 1.4 - 0.2
        x[:20] = rs.choice(xp, 20)
        for left, right in ((None, None), (0.0, None), (1.0, 0.5)):
            assert np.array_equal(np.interp(x, xp, fp, left=left, right=right), R.interp(x, xp, fp, left=left, right=right))
        y = rs.rand(101)
        with warnings.catch_warnings():
            warnings.simplefilter("ignore", DeprecationWarning)
            assert np.trapz(y, R.X101) == R.trapz(y, R.X101)
        a = rs.randn(rs.randint(1, 400))
        assert np.add.reduce(a) == R.pairwise_sum(a)


def test_ap_per_class_restatement_equals_reference_formula():
    """the loop-form restatement against the reference's ap_per_class formulas written with numpy's own interp / trapz"""
    rs = np.random.RandomState(1)
    for _ in range(40):
        n = rs.randint(1, 400)
        tp = rs.rand(n, 10) < np.linspace(0.8, 0.1, 10)
        conf = rs.permutation(np.linspace(0.01, 0.99, n).astype(np.float32))
        pcls = rs.randint(0, 4, n).astype(np.float32)
        tcls = rs.randint(0, 4, rs.randint(1, 200)).astype(np.float32)
        classes, ap, p, r = R.ap_curves(tp, conf, pcls, tcls)
        i = np.argsort(-conf)
        for ci, c in enumerate(classes):
            m = pcls[i] == c
            nl = (tcls == c).sum()
            if not m.any():
                continue
            tpc = tp[i][m].cumsum(0)
            fpc = (1 - tp[i][m]).cumsum(0)
            rec, pre = tpc / (nl + 1e-16), tpc / (tpc + fpc)
            assert np.array_equal(r[ci], np.interp(-R.PX, -conf[i][m], rec[:, 0], left=0))
            assert np.array_equal(p[ci], np.interp(-R.PX, -conf[i][m], pre[:, 0], left=1))
            for j in range(10):
                mrec = np.concatenate(([0.], rec[:, j], [rec[-1, j] + 0.01]))
                mpre = np.flip(np.maximum.accumulate(np.flip(np.concatenate(([1.], pre[:, j], [0.])))))
                with warnings.catch_warnings():
                    warnings.simplefilter("ignore", DeprecationWarning)
                    assert ap[ci, j] == np.trapz(np.interp(R.X101, mrec, mpre), R.X101)


def test_pack_geometry():
    from multiyolov5_b200.utils.metrics import pack_geometry
    g = pack_geometry((256, 416), [((600, 1000), ((0.416, 0.416), (0.5, 3.5))), ((480, 640), None)])
    assert g.dtype == np.float32 and g.shape == (2, 5)
    assert np.array_equal(g[0], np.float32([600, 1000, 0.416, 0.5, 3.5]))
    gain = min(256 / 480, 416 / 640)
    assert np.array_equal(g[1], np.float32([480, 640, gain, (416 - 640 * gain) / 2, (256 - 480 * gain) / 2]))
    assert np.array_equal(g[0], R.geometry((256, 416), ((600, 1000), ((0.416, 0.416), (0.5, 3.5)))))


def test_fitness():
    from multiyolov5_b200.utils.metrics import fitness, fitness2
    x = np.array([[0.5, 0.4, 0.3, 0.2, 1.0, 2.0]])
    assert np.allclose(fitness(x), 0.1 * 0.3 + 0.9 * 0.2)
    assert np.allclose(fitness2(x, 0.6), 0.1 * 0.3 + 0.2 * 0.2 + 0.7 * 0.6)


def test_error_word_raises():
    from multiyolov5_b200 import _lib
    from multiyolov5_b200.utils.metrics import _check_error
    t = np.zeros(256, np.int64)
    for bit in (_lib.DET_ERR_TARGET_CLASS, _lib.DET_ERR_PRED_CLASS, _lib.DET_ERR_LABELS):
        with pytest.raises(ValueError):
            _check_error(bit, t, 3)
    _check_error(0, t, 3)
    t[3] = 1
    with pytest.raises(ValueError):
        _check_error(0, t, 3)


def test_ap_per_class_argument_checks():
    from multiyolov5_b200.utils.metrics import ap_per_class
    tp, conf = np.ones((2, 10), bool), np.float32([0.9, 0.8])
    with pytest.raises(NotImplementedError):
        ap_per_class(tp, conf, [0, 0], [0], plot=True)
    with pytest.raises(ValueError):
        ap_per_class(tp, conf, [0, 0.5], [0])
    with pytest.raises(ValueError):
        ap_per_class(tp, conf, [0, 0], [-1])
    with pytest.raises(ValueError):
        ap_per_class(tp, np.array([0.9, 0.1]), [0, 0], [0])       # float64 conf not exact in float32


def test_stats_store_growth_and_checks():
    from multiyolov5_b200.utils.metrics import DetectionStats
    s = DetectionStats(max_det=4, device="cpu", capacity=2)
    s.correct[:8] = torch.arange(8, dtype=torch.int16)
    s.rows[:2] = torch.tensor([3, 4], dtype=torch.int32)
    s.seen = 2
    s._alloc(8)
    assert s.capacity == 8 and s.correct.numel() == 32 and torch.equal(s.correct[:8], torch.arange(8, dtype=torch.int16))
    assert torch.equal(s.rows[:2], torch.tensor([3, 4], dtype=torch.int32)) and not s.rows[2:].any()
    with pytest.raises(ValueError):
        DetectionStats(max_det=2000, device="cpu")
    with pytest.raises(ValueError):
        s.update(torch.zeros(1, 5, 6), torch.zeros(1), torch.zeros(0, 6), (32, 32), [((32, 32), None)])
    with pytest.raises(ValueError):
        s.compute(0)


def test_unsupported_test_options_raise():
    from multiyolov5_b200.test import test
    m = torch.nn.Linear(1, 1)
    with pytest.raises(NotImplementedError):
        test({"nc": 1}, model=None, dataloader=[])
    for kw in (dict(save_json=True), dict(save_txt=True), dict(save_hybrid=True), dict(augment=True), dict(plots=True),
               dict(wandb_logger=object())):
        with pytest.raises(NotImplementedError):
            test({"nc": 1}, model=m, dataloader=[], **{"plots": False, **kw})
