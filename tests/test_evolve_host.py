"""--evolve on the host: multiyolov5_b200.train.evolve with a stub training run against the unmodified reference's evolve block
(tests/golden/evolve_cases.json, oracle/make_golden_evolve.py): every generation's hyp, evolve.txt and hyp_evolved.yaml byte for byte and
the printed lines, from scratch, at mAP 0 throughout and resuming from an existing evolve.txt of tied rows; the restatement against the
same fixture; and the hyps and options the loop refuses."""
import argparse
import json
import os
import random
import time

import numpy as np
import pytest

from oracle import restate_evolve as rev

GOLD = os.path.join(os.path.dirname(__file__), "golden")


def _cases():
    with open(os.path.join(GOLD, "evolve_cases.json")) as f:
        return {c["name"]: c for c in json.load(f)["cases"]}


CASES = _cases()


def _opt(**kw):
    o = dict(global_rank=-1, local_rank=-1, save_dir="run", notest=False, nosave=False)
    o.update(kw)
    return argparse.Namespace(**o)


@pytest.mark.parametrize("name", sorted(CASES))
def test_evolve_matches_the_reference(name, tmp_path, monkeypatch, capsys):
    from multiyolov5_b200.train import evolve
    c = CASES[name]
    monkeypatch.chdir(tmp_path)
    os.makedirs("run")
    if c["pre"] is not None:
        (tmp_path / "evolve.txt").write_text(c["pre"])
    calls = []

    def train_fn(hyp, opt):
        assert opt.notest and opt.nosave
        calls.append(dict(hyp))
        return rev.stub_results(hyp, c["seed"], c["zero"])

    monkeypatch.setattr(time, "time", lambda: rev.clock(len(calls)))
    random.seed(c["seed"])
    hyp = dict(rev.HYP_SCRATCH)
    opt = _opt()
    capsys.readouterr()
    assert str(evolve(hyp, opt, train_fn, generations=c["generations"])) == os.path.join("run", "hyp_evolved.yaml")
    assert capsys.readouterr().out == c["stdout"]
    assert len(calls) == len(c["hyps"])
    for k, (got, exp) in enumerate(zip(calls, c["hyps"])):
        assert list(got) == list(exp) and got == exp, k
    assert (tmp_path / "evolve.txt").read_text() == c["evolve_txt"]
    assert (tmp_path / "run" / "hyp_evolved.yaml").read_text() == c["hyp_evolved"]
    assert random.random() == c["next_random"]                  # one draw of the global `random` per generation with a parent


@pytest.mark.parametrize("name", sorted(CASES))
def test_restatement_matches_the_reference(name, tmp_path):
    c = CASES[name]
    txt, yml = str(tmp_path / "evolve.txt"), str(tmp_path / "hyp_evolved.yaml")
    if c["pre"] is not None:
        (tmp_path / "evolve.txt").write_text(c["pre"])
    random.seed(c["seed"])
    hyps = rev.run(dict(rev.HYP_SCRATCH), lambda h, k: rev.stub_results(h, c["seed"], c["zero"]), c["generations"], txt, yml)
    assert hyps == c["hyps"]
    assert (tmp_path / "evolve.txt").read_text() == c["evolve_txt"]
    assert (tmp_path / "hyp_evolved.yaml").read_text() == c["hyp_evolved"]


def test_the_fixture_covers_tied_parents():
    """a zero total weight (one row, or the top rows tied) happens in the fixture's cases: the draw then takes the last of the top rows"""
    assert CASES["resume_one"]["pre"].count("\n") == 1
    assert CASES["zero_map"]["zero"] and CASES["resume_tied"]["pre"].count("\n") == 3


def test_choice_matches_python_where_the_total_is_positive():
    from multiyolov5_b200.train import choice_py38
    rs = np.random.RandomState(0)
    for n in (1, 2, 5):
        for _ in range(50):
            w = rs.uniform(0, 1, n) * (rs.uniform(size=n) < 0.7)
            if w.sum() <= 0:
                continue
            random.seed(n)
            a = random.choices(range(n), weights=w)[0]
            random.seed(n)
            assert choice_py38(n, w) == a


def test_choice_takes_the_last_index_at_a_zero_total():
    from multiyolov5_b200.train import choice_py38
    random.seed(5)
    after = (random.random(), random.random())
    random.seed(5)
    assert choice_py38(4, np.zeros(4)) == 3
    assert random.random() == after[1]                          # one draw made


def test_the_shipped_hyp_without_anchors_raises_key_error(tmp_path):
    from multiyolov5_b200.train import evolve
    hyp = {k: v for k, v in rev.HYP_SCRATCH.items() if k != "anchors"}
    with pytest.raises(KeyError) as e:
        evolve(hyp, _opt(save_dir=str(tmp_path)), lambda h, o: pytest.fail("trained"), evolve_txt=str(tmp_path / "evolve.txt"))
    assert e.value.args[0] == "anchors" and "anchors: 3" in str(e.value)


def test_out_of_order_or_extra_keys_are_refused(tmp_path):
    from multiyolov5_b200.train import evolve
    keys = list(rev.HYP_SCRATCH)
    swapped = {k: rev.HYP_SCRATCH[k] for k in [keys[1], keys[0], *keys[2:]]}
    extra = dict(rev.HYP_SCRATCH, label_smoothing=0.0)
    for hyp in (swapped, extra):
        with pytest.raises(ValueError, match="in this order"):
            evolve(hyp, _opt(save_dir=str(tmp_path)), lambda h, o: pytest.fail("trained"), evolve_txt=str(tmp_path / "evolve.txt"))


@pytest.mark.parametrize("rank", [dict(global_rank=0), dict(local_rank=0)])
def test_ddp_is_refused(rank, tmp_path):
    from multiyolov5_b200.train import evolve
    with pytest.raises(ValueError, match="DDP"):
        evolve(dict(rev.HYP_SCRATCH), _opt(save_dir=str(tmp_path), **rank), lambda h, o: pytest.fail("trained"),
               evolve_txt=str(tmp_path / "evolve.txt"))


def test_meta_is_the_reference_order_and_limits():
    from multiyolov5_b200.train import EVOLVE_META
    assert [(k, *v) for k, v in EVOLVE_META.items()] == rev.META
