"""TEST INFRASTRUCTURE - generates tests/golden/multiscale_cases.npz by executing the reference's --multi-scale statements
(train.py:354-359), read from the reference tree at generation time:

    MYOLO_REFERENCE_ROOT=<checkout> python oracle/make_golden_multiscale.py

The statements pass float bounds to random.randrange, which Python 3.12 rejects with TypeError.  They run here with a `random` whose
randrange turns integral floats into ints first and refuses others, which is what randrange did on Python <= 3.11; the stream it consumes
is the same.  `imgs` is a stand-in with the batch's shape, `F.interpolate` records the size it is asked for.

Per case (seed, imgsz, gs, input shape): 2 000 draws of sz, whether sf == 1, and ns (the input shape when sf == 1), plus the next
random() of the generator after the draws (so that a restatement can show it consumed the stream exactly as the reference did).
"""
import os
import random
import re
import sys
import textwrap

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
from oracle import ref_shims  # noqa: E402

GOLD = os.path.join(HERE, "..", "tests", "golden")
N_DRAWS = 2000
CASES = [  # (seed, imgsz, gs, (H, W))
    (0, 640, 32, (640, 640)), (1, 640, 32, (384, 640)), (2, 640, 32, (640, 352)),
    (3, 1024, 32, (1024, 1024)), (4, 1024, 32, (512, 1024)), (5, 1024, 32, (1000, 1000)), (6, 1024, 32, (1024, 2048)),
]


class Py311Random(random.Random):
    """randrange as Python <= 3.11 accepted it: integral floats are used as ints (non-integral ones raise ValueError)"""

    def randrange(self, start, stop=None, step=1):
        def idx(v):
            if isinstance(v, float):
                if v != int(v):
                    raise ValueError("non-integer arg for randrange()")
                return int(v)
            return v
        return super().randrange(idx(start), None if stop is None else idx(stop), idx(step))


def reference_statements():
    src = open(os.path.join(ref_shims.REF_ROOT, "train.py"), encoding="utf-8").read().splitlines()
    start = next(i for i, ln in enumerate(src) if ln.strip().startswith("if opt.multi_scale:"))
    body = []
    indent = len(src[start]) - len(src[start].lstrip())
    for ln in src[start + 1:]:
        if ln.strip() and len(ln) - len(ln.lstrip()) <= indent:
            break
        body.append(re.sub(r"\s+#.*$", "", ln))           # drop trailing comments
    text = textwrap.dedent("\n".join(body)).strip("\n")
    assert "random.randrange(imgsz * 0.5, imgsz * 1.5 + gs)" in text and "F.interpolate" in text, text
    return text


def main():
    if not ref_shims.reference_available():
        raise SystemExit("set MYOLO_REFERENCE_ROOT to a reference checkout")
    code = compile(reference_statements(), "reference train.py:355-359", "exec")
    out = {}
    for k, (seed, imgsz, gs, shape) in enumerate(CASES):
        rng = Py311Random(seed)

        class Imgs:
            pass

        class F:
            @staticmethod
            def interpolate(x, size, mode, align_corners):
                assert mode == "bilinear" and align_corners is False
                ns_seen.append(list(size))
                return x
        sz_out, same, ns_out = [], [], []
        for _ in range(N_DRAWS):
            imgs = Imgs()
            imgs.shape = (4, 3) + shape
            ns_seen = []
            env = {"random": rng, "math": __import__("math"), "imgs": imgs, "imgsz": imgsz, "gs": gs, "F": F}
            exec(code, env)
            sz_out.append(env["sz"])
            same.append(env["sf"] == 1)
            ns_out.append(ns_seen[0] if ns_seen else list(shape))
            assert (len(ns_seen) == 0) == (env["sf"] == 1)
        out[f"case{k}_meta"] = np.array([seed, imgsz, gs, shape[0], shape[1]], np.int64)
        out[f"case{k}_sz"] = np.array(sz_out, np.int64)
        out[f"case{k}_same"] = np.array(same, bool)
        out[f"case{k}_ns"] = np.array(ns_out, np.int64)
        out[f"case{k}_next"] = np.array([rng.random()], np.float64)
    out["n_cases"] = np.array([len(CASES)], np.int64)
    os.makedirs(GOLD, exist_ok=True)
    np.savez_compressed(os.path.join(GOLD, "multiscale_cases.npz"), **out)
    print(f"wrote {len(CASES)} cases x {N_DRAWS} draws")


if __name__ == "__main__":
    main()
