"""Host: the numpy restatement of scipy's k-means (oracle/restate_kmeans.py), which fixes the device kernel's arithmetic and order, against
scipy's own results (tests/golden/kmeans_cases.npz) and against scipy's and numpy's pieces one by one: the pairwise mean, the sequential
cluster sums, the final vq (rule 5), the draws and the error messages of utils.autoanchor.kmeans."""
import os

import numpy as np
import pytest

from oracle import restate_kmeans as rk

GOLD = os.path.join(os.path.dirname(__file__), "golden")
SMALL = ["city", "dup", "few_distinct", "n5", "n127", "n128", "n129", "n8191", "n8192", "n8193", "k32"]


def _cases():
    return {c["name"]: c for c in rk.load_cases(os.path.join(GOLD, "kmeans_cases.npz"))}


def test_fixture_has_every_case():
    cases = _cases()
    assert set(SMALL) | {"coco"} <= set(cases)
    assert any(len(b) < cases["dup"]["k"] for b in cases["dup"]["run_books"])          # scipy dropped a cluster
    assert len(cases["few_distinct"]["book"]) < cases["few_distinct"]["k"]              # kmean_anchors' len(k) != n path
    assert cases["coco"]["n"] > 700_000


@pytest.mark.parametrize("name", SMALL)
def test_restatement_equals_scipy(name):
    c = _cases()[name]
    obs = rk.case_obs(c)
    assert len(obs) == c["n"]
    np.random.seed(c["seed"])
    book, dist, runs = rk.kmeans(obs, c["k"], iter=c["iter"], thresh=c["thresh"])
    assert np.array_equal(book, c["book"]) and dist == c["dist"]
    assert np.array_equal(np.random.random(4), c["next_np"])
    for r, (b, d, it) in enumerate(runs):
        assert np.array_equal(b, c["run_books"][r]) and d == c["run_dists"][r] and it == c["run_iters"][r], r


@pytest.mark.parametrize("n", list(range(1, 300)) + [8191, 8192, 8193, 20_000, 100_003])
def test_pairwise_mean_equals_numpy(n):
    a = np.random.default_rng(n).lognormal(0.0, 1.0, n)
    assert rk.pairwise_mean(a) == np.mean(a)


def test_leaves_cover_the_array_in_order():
    for n in (1, 7, 8, 128, 129, 1000, 8193, 790_001):
        leaves = rk.pairwise_leaves(n)
        assert leaves[0][0] == 0 and all(s + m == t for (s, m), (t, _) in zip(leaves, leaves[1:]))
        assert sum(m for _, m in leaves) == n and all(m <= rk.LEAF for _, m in leaves)


def test_sequential_sums_equal_update_cluster_means():
    from scipy.cluster.vq import _vq_impl
    rng = np.random.default_rng(1)
    obs = rng.lognormal(0.0, 1.0, (50_000, 2))
    code = rng.integers(0, 9, len(obs)).astype(np.int32)
    code[code == 4] = 3                                              # an empty cluster
    mine = rk.cluster_means(obs, code.astype(np.int64), 9)
    ref, has = _vq_impl._vq.update_cluster_means(obs, code, 9)
    assert np.array_equal(mine, ref[has])


def test_vq_equals_scipy():
    from scipy.cluster.vq import vq
    rng = np.random.default_rng(2)
    obs = rng.lognormal(0.0, 1.0, (20_000, 2))
    book = np.concatenate([obs[:8], obs[3:4]])                       # a duplicate code: the first one wins
    code, dist = rk.vq(obs, book)
    c_ref, d_ref = vq(obs, book)
    assert np.array_equal(code, c_ref) and np.array_equal(dist, d_ref)
    assert not (code == 8).any()


def test_distortion_is_the_mean_of_a_final_vq():
    """scipy >= 1.17: _kmeans returns the mean of one more vq with the final book, not the last in-loop mean (the vq of the book before
    the last update), which differs on some restarts"""
    from scipy.cluster.vq import _vq_impl
    c = _cases()["city"]
    obs = rk.case_obs(c)
    differs = 0
    for idx in c["starts"][:10]:
        book, dist, _ = rk.kmeans_one(obs, obs[idx], c["thresh"])
        ref_book, ref_dist = _vq_impl._kmeans(obs, obs[idx], thresh=c["thresh"])
        assert np.array_equal(book, ref_book) and dist == ref_dist
        assert dist == rk.pairwise_mean(rk.vq(obs, book)[1])
        prev, diff, b = np.inf, np.inf, obs[idx]
        while diff > c["thresh"]:
            code, d = rk.vq(obs, b)
            cur = rk.pairwise_mean(d)
            b = rk.cluster_means(obs, code, len(b))
            diff, prev = abs(prev - cur), cur
        differs += prev != dist
    assert differs > 0


def test_draws_equal_scipy_kpoints():
    from scipy.cluster.vq import _vq_impl
    np.random.seed(3)
    mine = rk.draw_starts(1000, 9, 5)
    np.random.seed(3)
    ref = [np.asarray(_vq_impl._kpoints(np.arange(1000.0)[:, None], 9, np.random.mtrand._rand, np)).ravel() for _ in range(5)]
    assert np.array_equal(mine, np.stack(ref).astype(mine.dtype))


def _scipy_error(*a, **kw):
    from scipy.cluster.vq import kmeans
    with pytest.raises(ValueError) as e:
        kmeans(*a, **kw)
    return str(e.value)


@pytest.mark.parametrize("obs,k,kw", [
    (np.ones((5, 2)), 9, {}),                                        # n < k: numpy's choice raises, as in scipy
    (np.array([[1.0, np.nan], [2.0, 3.0]]), 1, {}),
    (np.array([[1.0, np.inf], [2.0, 3.0]]), 1, {}),
    (np.ones((5, 2)), 0, {}),
    (np.ones((5, 2)), 2, {"iter": 0}),
])
def test_errors_equal_scipys(obs, k, kw):
    """raised on the host before any launch, so no device is needed; the generator ends where scipy leaves it"""
    from multiyolov5_b200.utils import autoanchor as aa
    np.random.seed(0)
    msg = _scipy_error(obs, k, **kw)
    after = np.random.random()
    np.random.seed(0)
    with pytest.raises(ValueError) as e:
        aa.kmeans(obs, k, **kw)
    assert str(e.value) == msg
    assert np.random.random() == after


def test_new_symbols_are_exported():
    from multiyolov5_b200 import _lib
    L = _lib.lib()
    for name in ("myolo_kmeans", "myolo_kmeans_workspace_bytes"):
        assert name in _lib.EXPORTS and hasattr(L, name)
    assert L.myolo_kmeans_workspace_bytes(0, 9, 30) == -1
    assert L.myolo_kmeans_workspace_bytes(1000, 9, 30) > 30 * 1000
