"""TEST INFRASTRUCTURE — import-only shims so the UNMODIFIED reference (a checkout named by
MYOLO_REFERENCE_ROOT) can be imported on a CPU machine to generate fixtures (it is not an installable package).

Only oracle/make_golden.py and oracle/check_restatement.py use this module.  Nothing in the product
(multiyolov5_b200/), bench.py's default arm, or the `-m gpu` tests may import it.

What is stubbed (none of it touches arithmetic; see SURVEY.md §8c):
  * `onnx`, `onnx.external_data_helper`   — stray import at reference models/yolo.py:8
  * `matplotlib`, `matplotlib.pyplot`, `seaborn` — plotting imports at reference utils/plots.py:11-25
"""
import importlib.machinery as _im
import os
import sys
import types

REF_ROOT = os.environ.get("MYOLO_REFERENCE_ROOT", "")


def reference_available() -> bool:
    return os.path.isfile(os.path.join(REF_ROOT, "models", "yolo.py"))


def install_shims():
    for name in ("onnx", "onnx.external_data_helper", "matplotlib", "matplotlib.pyplot", "seaborn"):
        if name in sys.modules:
            continue
        m = types.ModuleType(name)
        m.__spec__ = _im.ModuleSpec(name, None)
        m.__path__ = []
        sys.modules[name] = m
    sys.modules["matplotlib"].rc = lambda *a, **k: None
    sys.modules["matplotlib"].use = lambda *a, **k: None
    sys.modules["matplotlib"].pyplot = sys.modules["matplotlib.pyplot"]
    sys.modules["onnx"].external_data_helper = sys.modules["onnx.external_data_helper"]


def import_reference():
    """Returns (models.yolo, utils.general) of the reference.  Changes sys.path (not cwd)."""
    if not reference_available():
        raise RuntimeError(f"reference tree not found at {REF_ROOT}")
    install_shims()
    # the reference's packages are called `models` and `utils`; make sure ours are not shadowing
    for k in [k for k in sys.modules if k == "models" or k.startswith("models.") or k == "utils" or k.startswith("utils.")]:
        del sys.modules[k]
    if REF_ROOT not in sys.path:
        sys.path.insert(0, REF_ROOT)
    import models.yolo as ref_yolo  # noqa
    import utils.general as ref_general  # noqa
    return ref_yolo, ref_general
