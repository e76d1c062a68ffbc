"""H100: scipy's k-means on the device (utils.autoanchor.kmeans, myolo_kmeans) against scipy's own results on every fixture case
(tests/golden/kmeans_cases.npz, the ~790 k label case included): the book, k', the distortion, every restart's book, distortion and
Lloyd iteration count, and the state of `numpy.random` afterwards, bit for bit.  Run-to-run identity, the iteration cap and argument
checks as clean errors, and kmean_anchors without scipy."""
import contextlib
import io
import os
import random

import numpy as np
import pytest
import torch

from oracle import restate_autoanchor as ra
from oracle import restate_kmeans as rk

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden")
NAMES = ["city", "dup", "few_distinct", "n5", "n127", "n128", "n129", "n8191", "n8192", "n8193", "k32", "coco"]


@pytest.fixture(scope="module")
def cases():
    return {c["name"]: c for c in rk.load_cases(os.path.join(GOLD, "kmeans_cases.npz"))}


@pytest.mark.parametrize("name", NAMES)
def test_matches_scipy(cases, name):
    from multiyolov5_b200.utils import autoanchor as aa
    c = cases[name]
    obs = rk.case_obs(c)
    np.random.seed(c["seed"])
    book, dist = aa.kmeans(obs, c["k"], iter=c["iter"], thresh=c["thresh"])
    assert np.array_equal(np.random.random(4), c["next_np"])
    assert book.dtype == np.float64 and len(book) == len(c["book"])
    assert np.array_equal(book, c["book"]) and dist == c["dist"]
    books, dists, iters, best = aa.kmeans_restarts(obs, c["starts"], c["thresh"])
    assert best == c["best"]
    assert np.array_equal(iters, c["run_iters"])
    assert np.array_equal(dists, c["run_dists"])
    for r in range(c["iter"]):
        assert np.array_equal(books[r], c["run_books"][r]), r


def test_two_runs_are_identical(cases):
    from multiyolov5_b200.utils import autoanchor as aa
    c = cases["n8193"]
    obs = rk.case_obs(c)
    a, b = aa.kmeans_restarts(obs, c["starts"], c["thresh"]), aa.kmeans_restarts(obs, c["starts"], c["thresh"])
    assert all(np.array_equal(x, y) for x, y in zip(a[0], b[0]))
    assert np.array_equal(a[1], b[1]) and np.array_equal(a[2], b[2]) and a[3] == b[3]


def test_iteration_cap_raises(cases):
    from multiyolov5_b200 import _lib
    from multiyolov5_b200.utils import autoanchor as aa
    c = cases["city"]
    obs = rk.case_obs(c)
    with pytest.raises(_lib.MyoloError, match="still moving after 3"):
        aa.kmeans_restarts(obs, c["starts"], c["thresh"], max_iter=3)
    books, dists, _, best = aa.kmeans_restarts(obs, c["starts"], c["thresh"])       # the device is fine afterwards
    assert np.array_equal(books[best], c["book"]) and dists[best] == c["dist"]


def test_argument_checks(cases):
    from multiyolov5_b200 import _lib
    from multiyolov5_b200.utils import autoanchor as aa
    obs = rk.case_obs(cases["city"])
    with pytest.raises(_lib.MyoloError, match="k = 33"):
        aa.kmeans_restarts(obs, np.arange(33)[None], 1e-5)
    with pytest.raises(_lib.MyoloError, match="d = 3"):
        aa.kmeans_restarts(np.ones((100, 3)), np.arange(9)[None], 1e-5)
    with pytest.raises(_lib.MyoloError, match="start indices"):
        aa.kmeans_restarts(obs, np.array([[0, 1, len(obs)]]), 1e-5)
    with pytest.raises(_lib.MyoloError, match="restarts"):
        aa.kmeans_restarts(obs, np.zeros((1000, 2), np.int64), 1e-5)     # more restarts than co-resident CTAs


class _Dataset:
    def __init__(self, shapes, labels):
        self.shapes, self.labels = shapes, labels


def _no_scipy(monkeypatch):
    import scipy.cluster.vq

    def boom(*a, **kw):
        raise AssertionError("scipy's kmeans called")
    monkeypatch.setattr(scipy.cluster.vq, "kmeans", boom)


def test_kmean_anchors_without_scipy(monkeypatch):
    """the reference's recorded kmean_anchors case (tests/golden/autoanchor_cases.npz): printed lines, anchors and RNG state"""
    from multiyolov5_b200.utils import autoanchor as aa
    _no_scipy(monkeypatch)
    c = {c["name"]: c for c in ra.load_cases(os.path.join(GOLD, "autoanchor_cases.npz"))}["kmean_verbose"]
    shapes0, labels = ra.case_dataset(c)
    random.seed(c["seed"]); np.random.seed(c["seed"]); torch.manual_seed(c["seed"])
    buf = io.StringIO()
    with contextlib.redirect_stdout(buf):
        ret = aa.kmean_anchors(_Dataset(ra.shapes_wh(shapes0), labels), n=c["n"], img_size=c["imgsz"], thr=c["thr"], gen=c["gen"],
                               verbose=c["verbose"])
    assert buf.getvalue() == c["stdout"]
    assert np.array_equal(ret, c["returned"])
    assert np.array_equal(np.random.random(4), c["next_np"])


def test_kmean_anchors_fewer_distinct_sizes_than_anchors(monkeypatch):
    """three box sizes on one image shape, nine anchors: k-means returns fewer codes and kmean_anchors fails as the reference does"""
    from multiyolov5_b200.utils import autoanchor as aa
    _no_scipy(monkeypatch)
    shapes0, labels = ra.synth_dataset(4, 20, 30, [(20, 40), (60, 30), (100, 120)], spread=0.0, shapes=((320, 640),))
    np.random.seed(0)
    buf = io.StringIO()
    with contextlib.redirect_stdout(buf), pytest.raises(AssertionError):
        aa.kmean_anchors(_Dataset(ra.shapes_wh(shapes0), labels), n=9, img_size=640, thr=4.0, gen=10, verbose=False)
    assert "ERROR: scipy.cluster.vq.kmeans requested 9 points but returned only" in buf.getvalue()
