"""TEST INFRASTRUCTURE - generates tests/golden/tta_cases.npz by running the UNMODIFIED reference (MYOLO_REFERENCE_ROOT, imported through
oracle/ref_shims.py) on the CPU:

    MYOLO_REFERENCE_ROOT=<checkout> python oracle/make_golden_tta.py

The reference's own `scale_img` and `Model.forward_once` run inside the augment loop of oracle/restate_tta.py (the fork's loop itself
cannot de-scale the pair forward_once returns; restate_tta.py says why).  Stored, with no weights (they are re-synthesised from the
manifest and seed 1, s/PSP):
  case{k}_seed / _shape / _x_sum  the synth.synth_image input of each forward case (re-created by the tests from the seed)
  case{k}_rows / case{k}_z         every ROW_STEP-th row of its augmented z (all columns, fp32), and those rows' indices: the whole z of
                                   both cases would make the fixture megabytes of incompressible floats
  si_x                             a small random fp32 input of scale_img
  si{j}_args / si{j}_out           (ratio, same_shape, flip) and the reference's scale_img(x.flip(3) if flip else x, ratio, same_shape)
  sweep_args / sweep_shape         (h, w, ratio, same_shape) and the (h, w) of the reference's scale_img output
"""
import copy
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
from oracle import ref_shims, restate_tta, synth  # noqa: E402

GOLD = os.path.join(HERE, "..", "tests", "golden")
CASES = [(2, 256, 512, 3), (1, 320, 416, 4)]                     # (B, H, W, seed)
ROW_STEP = 13                # prime: the sample does not follow the row layout's powers of two (anchor, y, x of each level)
SI_ARGS = [(0.83, False, False), (0.83, False, True), (0.67, False, False), (0.67, False, True), (0.83, True, False), (1.3, False, False),
           (1.3, True, True)]
SWEEP_HW = [(h, w) for h in (32, 64, 96, 200, 256, 320, 384, 416, 512, 640, 720, 1024) for w in (32, 100, 416, 512, 640, 1024, 1280, 2048)]
SWEEP_R = [(0.83, False), (0.67, False), (0.5, False), (1.2, False), (0.83, True), (0.67, True)]


def main():
    if not ref_shims.reference_available():
        raise SystemExit("set MYOLO_REFERENCE_ROOT to a reference checkout")
    ref_yolo, _ = ref_shims.import_reference()
    import utils.torch_utils as ref_tu          # the reference's, on sys.path after import_reference

    out = {}
    cfg = synth.load_cfg("yolov5s_city_seg.yaml")
    torch.manual_seed(0)
    model = ref_yolo.Model(copy.deepcopy(cfg))
    model.load_state_dict(synth.synth_state_dict(synth.load_manifest("s_psp"), cfg, seed=1))
    model.fuse().eval()
    gs = int(model.stride.max())
    assert gs == 32
    for k, (B, H, W, seed) in enumerate(CASES):
        x = synth.synth_image(B, H, W, seed=seed)
        width = x.shape[-1]
        zs = []
        with torch.no_grad():
            for si, mirror in restate_tta.PASSES:
                xi = ref_tu.scale_img(x.flip(3) if mirror else x, si, gs=gs)
                yi = model.forward_once(xi)[0][0]
                yi[..., :4] /= si
                if mirror:
                    yi[..., 0] = width - yi[..., 0]
                zs.append(yi)
        z = torch.cat(zs, 1)
        out[f"case{k}_seed"] = np.int64(seed)
        out[f"case{k}_shape"] = np.array([B, H, W], np.int64)
        out[f"case{k}_x_sum"] = np.float64(x.double().sum().item())
        rows = np.arange(0, z.shape[1], ROW_STEP, dtype=np.int64)
        out[f"case{k}_rows"] = rows
        out[f"case{k}_z"] = z.numpy().astype(np.float32)[:, rows]
        print(f"case {k}: x {tuple(x.shape)} -> z {tuple(z.shape)}, {len(rows)} rows kept")
    g = torch.Generator().manual_seed(0)
    x = torch.rand((1, 3, 23, 37), generator=g, dtype=torch.float32)
    out["si_x"] = x.numpy()
    for j, (r, same, flip) in enumerate(SI_ARGS):
        out[f"si{j}_args"] = np.array([r, same, flip], np.float64)
        out[f"si{j}_out"] = ref_tu.scale_img(x.flip(3) if flip else x, r, same_shape=same, gs=gs).numpy()
    args, shapes = [], []
    for h, w in SWEEP_HW:
        t = torch.zeros((1, 1, h, w))
        for r, same in SWEEP_R:
            args.append([h, w, r, same])
            shapes.append(list(ref_tu.scale_img(t, r, same_shape=same, gs=gs).shape[-2:]))
    out["sweep_args"] = np.array(args, np.float64)
    out["sweep_shape"] = np.array(shapes, np.int64)
    out["n_cases"], out["n_si"] = np.int64(len(CASES)), np.int64(len(SI_ARGS))
    os.makedirs(GOLD, exist_ok=True)
    path = os.path.join(GOLD, "tta_cases.npz")
    np.savez_compressed(path, **out)
    print(f"wrote {path}: {os.path.getsize(path) / 1e6:.2f} MB")


if __name__ == "__main__":
    main()
