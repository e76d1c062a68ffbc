"""TEST INFRASTRUCTURE - generates tests/golden/evolve_cases.json from the UNMODIFIED reference's --evolve block (train.py:637-717), its
print_mutation (utils/general.py:528-556) and fitness (utils/metrics.py:12-15) on the CPU:

    MYOLO_REFERENCE_ROOT=<checkout> python oracle/make_golden_evolve.py

The evolve block is read from the reference's train.py at generation time and executed in memory (it lives under `if __name__ ==
'__main__'`); three statements are changed in that text: the generation count (300 -> the case's), and the `random` / `time` modules it
sees, which are stand-ins: `random.choices` with Python 3.8's semantics (the reference's NGC 21.03 image runs 3.8: a zero total weight gives
the last index after one `random()` draw, where 3.9+ raises) over the global `random` stream, and a frozen clock (oracle.restate_evolve.
clock: a function of how many training runs have started).  `train` is oracle.restate_evolve.stub_results; `plot_evolution` does nothing.
Each case records the hyp every `train` call received, and the final evolve.txt and hyp_evolved.yaml text.
"""
import contextlib
import io
import json
import os
import random
import sys
import tempfile
import textwrap
import types
from pathlib import Path

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
from oracle import ref_shims  # noqa: E402
from oracle import restate_evolve as rev  # noqa: E402

GOLD = os.path.join(HERE, "..", "tests", "golden")


def evolve_block(generations):
    src = open(os.path.join(ref_shims.REF_ROOT, "train.py")).read().splitlines()
    start = next(i for i, l in enumerate(src) if "# Evolve hyperparameters (optional)" in l)
    end = next(i for i, l in enumerate(src) if "Command to train a new model with these hyperparameters" in l)
    body = textwrap.dedent("\n".join(src[start + 2:end + 1]))          # the `else:` branch's statements
    assert body.count("range(300)") == 1
    return body.replace("range(300)", f"range({generations})")


class _Random38:
    """the `random` module as the evolve block uses it, with Python 3.8's choices()"""

    @staticmethod
    def choices(population, weights=None, *, cum_weights=None, k=1):
        import bisect
        import itertools
        assert cum_weights is None and weights is not None
        cum = list(itertools.accumulate(weights))
        total = cum[-1] + 0.0
        return [population[bisect.bisect(cum, random.random() * total, 0, len(population) - 1)] for _ in range(k)]


def run_case(name, ref_general, ref_metrics, generations, seed, zero=False, pre=None):
    calls = []

    def train(hyp, opt, device):
        calls.append(dict(hyp))
        return rev.stub_results(hyp, seed, zero)

    clock = types.SimpleNamespace(time=lambda: rev.clock(len(calls)))
    hyp = dict(rev.HYP_SCRATCH)
    opt = types.SimpleNamespace(local_rank=-1, save_dir="run", bucket="", notest=False, nosave=False)
    cwd = os.getcwd()
    with tempfile.TemporaryDirectory() as d:
        os.chdir(d)
        try:
            os.makedirs("run")
            if pre is not None:
                Path("evolve.txt").write_text(pre)
            random.seed(seed)
            ns = dict(meta=None, opt=opt, hyp=hyp, device="cpu", train=train, print_mutation=ref_general.print_mutation,
                      fitness=ref_metrics.fitness, plot_evolution=lambda f: None, Path=Path, np=np, random=_Random38, time=clock,
                      os=os)
            out = io.StringIO()
            with contextlib.redirect_stdout(out):
                exec(compile(evolve_block(generations), "reference:train.py (evolve block)", "exec"), ns)
            case = dict(name=name, generations=generations, seed=seed, zero=zero, pre=pre, hyps=calls,
                        evolve_txt=Path("evolve.txt").read_text(), hyp_evolved=Path("run/hyp_evolved.yaml").read_text(),
                        stdout=out.getvalue(), next_random=random.random())
        finally:
            os.chdir(cwd)
    print(name, generations, "generations; best row", case["evolve_txt"].splitlines()[0][:60])
    return case


def tied_rows(n, seed):
    """an evolve.txt of n rows whose fitness ties (equal mAPs, different P / R and hyps), as print_mutation writes it"""
    rs = np.random.RandomState(seed)
    rows = []
    for _ in range(n):
        hyp = {k: v * rs.uniform(0.8, 1.2) for k, v in rev.HYP_SCRATCH.items()}
        res = (rs.uniform(), rs.uniform(), 0.25, 0.125, *rs.uniform(0.01, 0.2, 3))
        rows.append("".join("%10.4g" % r for r in res) + "".join("%10.3g" % v for v in hyp.values()))
    return "\n".join(rows) + "\n"


def main():
    ref_shims.import_reference()
    import utils.general as ref_general                    # the reference's (sys.path set by import_reference)
    import utils.metrics as ref_metrics
    cases = [run_case("fresh", ref_general, ref_metrics, 20, seed=1),
             run_case("zero_map", ref_general, ref_metrics, 6, seed=2, zero=True),
             run_case("resume_tied", ref_general, ref_metrics, 5, seed=3, pre=tied_rows(3, 3)),
             run_case("resume_one", ref_general, ref_metrics, 4, seed=4, pre=tied_rows(1, 4))]
    out = os.path.join(GOLD, "evolve_cases.json")
    with open(out, "w") as f:
        json.dump(dict(clock0=rev.CLOCK0, hyp=rev.HYP_SCRATCH, cases=cases), f, indent=1)
    print("wrote", out, os.path.getsize(out), "bytes")


if __name__ == "__main__":
    main()
