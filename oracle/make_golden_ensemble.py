"""TEST INFRASTRUCTURE - generates tests/golden/ensemble_cases.npz by running the UNMODIFIED reference (MYOLO_REFERENCE_ROOT, imported
through oracle/ref_shims.py) on the CPU, in fp32:

    MYOLO_REFERENCE_ROOT=<checkout> python oracle/make_golden_ensemble.py

Three members of different heads and sizes that share nc 10, 19 seg classes and the strides: s/PSP seed 1, s/BiSe seed 2 and m/PSP seed 3
(synthetic weights from the manifests).  Each is the reference's own Model, `.fuse().eval()` as attempt_load leaves it; the fork's
Ensemble.forward cannot run (oracle/restate_ensemble.py says why), so the members' `forward_once` outputs are combined by
restate_ensemble.ensemble, the fork's loop with the index restored and the seg mean.  Stored, with no weights:
  members                       (tag, yaml, seed) of each member
  case{k}_seed / _shape / _x_sum  the synth.synth_image input of each case (re-created by the tests from the seed)
  case{k}_rows / case{k}_z        every ROW_STEP-th row of the ensemble's z (all columns, fp32) and those rows' indices
  case{k}_seg_idx / case{k}_seg   every SEG_STEP-th element of the flattened mean seg logits (fp32) and their flat indices
  case{k}_ids                     the argmax of the mean seg (B, H, W) uint8
"""
import copy
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
from oracle import ref_shims, restate_ensemble, synth  # noqa: E402

GOLD = os.path.join(HERE, "..", "tests", "golden")
MEMBERS = [("s_psp", "yolov5s_city_seg.yaml", 1), ("s_bise", "yolov5s_city_seg_bise.yaml", 2), ("m_psp", "yolov5m_city_seg.yaml", 3)]
CASES = [(2, 64, 128, 3), (1, 256, 512, 4)]                      # (B, H, W, seed)
ROW_STEP = 13                # prime: the sample does not follow the row layout's powers of two (anchor, y, x of each level)
SEG_STEP = 97


def main():
    if not ref_shims.reference_available():
        raise SystemExit("set MYOLO_REFERENCE_ROOT to a reference checkout")
    ref_yolo, _ = ref_shims.import_reference()
    models = []
    for tag, yml, seed in MEMBERS:
        cfg = synth.load_cfg(yml)
        torch.manual_seed(0)
        m = ref_yolo.Model(copy.deepcopy(cfg))
        m.load_state_dict(synth.synth_state_dict(synth.load_manifest(tag), cfg, seed=seed))
        models.append(m.float().fuse().eval())
    out = {"members": np.array([[t, y, str(s)] for t, y, s in MEMBERS])}
    for k, (B, H, W, seed) in enumerate(CASES):
        x = synth.synth_image(B, H, W, seed=seed)
        with torch.no_grad():
            z, seg, ids = restate_ensemble.ensemble([m.forward_once(x) for m in models])
        out[f"case{k}_seed"] = np.int64(seed)
        out[f"case{k}_shape"] = np.array([B, H, W], np.int64)
        out[f"case{k}_x_sum"] = np.float64(x.double().sum().item())
        rows = np.arange(0, z.shape[1], ROW_STEP, dtype=np.int64)
        out[f"case{k}_rows"] = rows
        out[f"case{k}_z"] = z.numpy().astype(np.float32)[:, rows]
        idx = np.arange(0, seg.numel(), SEG_STEP, dtype=np.int64)
        out[f"case{k}_seg_idx"] = idx
        out[f"case{k}_seg"] = seg.numpy().astype(np.float32).reshape(-1)[idx]
        out[f"case{k}_ids"] = ids.numpy().astype(np.uint8)
        print(f"case {k}: x {tuple(x.shape)} -> z {tuple(z.shape)} ({len(rows)} rows kept), seg {tuple(seg.shape)} ({len(idx)} values kept)")
    out["n_cases"] = np.int64(len(CASES))
    os.makedirs(GOLD, exist_ok=True)
    path = os.path.join(GOLD, "ensemble_cases.npz")
    np.savez_compressed(path, **out)
    print(f"wrote {path}: {os.path.getsize(path) / 1e6:.2f} MB")


if __name__ == "__main__":
    main()
