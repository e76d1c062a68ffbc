"""TEST INFRASTRUCTURE - generates tests/golden/segloss_cases.npz from the UNMODIFIED reference's `SegFocalLoss` (utils/loss.py:279-297)
and `SegmentationLosses(weight=...)` (:221-244) on the CPU:

    MYOLO_REFERENCE_ROOT=<checkout> python oracle/make_golden_segloss.py

(tests/golden/segloss_cases.npz, compressed; oracle.restate_segloss.load_cases reads it back.)

Each case is B=2 images of logits at 6 x 8 (19 classes, or 2 for the custom dataset's head) with ~15 % of the labels ignored; it stores
the logits, the labels, the class weights (a seeded draw in [0.5, 1.5], not the reference's Cityscapes vector, which train.py leaves
commented out), the constructor arguments, the loss and d loss / d logits (autograd through the reference).  Cases: the weighted CE; BiSe's
three outputs with aux_num=2 and weights; SegFocalLoss with gamma in {0, 0.5, 1.5, 2}, alpha on and off, reduction 'mean' and 'sum'; the
reference's default ignore_index -100; a 2-class head; every pixel ignored (weighted CE and focal); and one valid pixel saturated (its
label's logit 200 above the others, so p_t = 1 in fp32) with gamma = 0.5, where (1 - p_t)^(gamma - 1) is infinite.

`draw_inputs()` needs no reference: tests/test_segloss_host.py regenerates every input from it and compares with the committed file.
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))

GOLD = os.path.join(HERE, "..", "tests", "golden")
B, NC, H, W = 2, 19, 6, 8

# name, kind ('wce': SegmentationLosses(weight), 'focal': SegFocalLoss), gamma, alpha/weight on, reduction, ignore_index, extra
SPECS = [
    ("wce", "wce", 0.0, True, "mean", -1, {}),
    ("wce_bise", "wce", 0.0, True, "mean", -1, dict(aux_weight=0.1)),
    ("focal_g0_alpha", "focal", 0.0, True, "mean", -1, {}),
    ("focal_g05_alpha", "focal", 0.5, True, "mean", -1, {}),
    ("focal_g15_alpha", "focal", 1.5, True, "mean", -1, {}),
    ("focal_g2_alpha", "focal", 2.0, True, "mean", -1, {}),
    ("focal_g2", "focal", 2.0, False, "mean", -1, {}),
    ("focal_g05", "focal", 0.5, False, "mean", -1, {}),
    ("focal_g0_alpha_sum", "focal", 0.0, True, "sum", -1, {}),
    ("focal_g15_sum", "focal", 1.5, False, "sum", -1, {}),
    ("focal_g2_alpha_sum", "focal", 2.0, True, "sum", -1, {}),
    ("focal_g2_default_ignore", "focal", 2.0, False, "mean", -100, {}),
    ("focal_g2_2cls", "focal", 2.0, False, "mean", -1, dict(nc=2)),
    ("wce_all_ignored", "wce", 0.0, True, "mean", -1, dict(valid_frac=0.0)),
    ("focal_g2_alpha_all_ignored", "focal", 2.0, True, "mean", -1, dict(valid_frac=0.0)),
    ("focal_g05_alpha_saturated", "focal", 0.5, True, "mean", -1, dict(saturate=True)),
]


def draw_inputs():
    """[(spec, logits [..], labels, weight or None)] for SPECS, seeded per case"""
    out = []
    for k, spec in enumerate(SPECS):
        name, kind, gamma, has_w, red, ign, extra = spec
        nc = extra.get("nc", NC)
        g = torch.Generator().manual_seed(2000 + k)
        labels = torch.randint(0, nc, (B, H, W), generator=g)
        labels[torch.rand((B, H, W), generator=g) >= extra.get("valid_frac", 0.85)] = ign
        n_out = 3 if "aux_weight" in extra else 1
        logits = [(torch.randn((B, nc, H, W), generator=g) * 2.0).contiguous() for _ in range(n_out)]
        weight = (torch.rand(nc, generator=g) + 0.5) if has_w else None
        if extra.get("saturate"):
            labels[0, 1, 2] = 3                                      # one valid pixel whose label's probability rounds to 1
            logits[0][0, :, 1, 2] = 0.0
            logits[0][0, 3, 1, 2] = 200.0
        out.append((spec, logits, labels, weight))
    return out


def run_reference(ref_loss, spec, logits, labels, weight):
    name, kind, gamma, has_w, red, ign, extra = spec
    if kind == "wce":
        if "aux_weight" in extra:
            crit = ref_loss.SegmentationLosses(nclass=NC, aux=True, aux_num=2, aux_weight=extra["aux_weight"], ignore_index=ign, weight=weight)
        else:
            crit = ref_loss.SegmentationLosses(aux=False, ignore_index=ign, weight=weight)
    else:
        crit = ref_loss.SegFocalLoss(gamma=gamma, alpha=weight, ignore_index=ign, reduction=red)
    ps = [x.clone().requires_grad_(True) for x in logits]
    loss = crit(*ps, labels)
    loss.backward()
    print(f"{name}: loss {float(loss.detach())!r}")
    return loss.detach(), [p.grad.detach().clone() for p in ps]


def main():
    argp = argparse.ArgumentParser()
    argp.add_argument("--out", default=os.path.join(GOLD, "segloss_cases.npz"))
    args = argp.parse_args()
    from oracle import ref_shims
    ref_shims.import_reference()
    import utils.loss as ref_loss                            # the reference's (sys.path set by import_reference)
    arrays, meta = {}, []
    for spec, logits, labels, weight in draw_inputs():
        name, kind, gamma, has_w, red, ign, extra = spec
        loss, grads = run_reference(ref_loss, spec, logits, labels, weight)
        arrays[f"{name}_labels"] = labels.numpy()
        arrays[f"{name}_loss"] = loss.numpy()
        if weight is not None:
            arrays[f"{name}_weight"] = weight.numpy()
        for i, (x, gr) in enumerate(zip(logits, grads)):
            arrays[f"{name}_logits_{i}"] = x.numpy()
            arrays[f"{name}_grad_{i}"] = gr.numpy()
        meta.append(dict(name=name, kind=kind, gamma=gamma, has_weight=has_w, reduction=red, ignore_index=ign,
                         aux_weight=extra.get("aux_weight"), n_outputs=len(logits)))
    arrays["meta_json"] = np.frombuffer(json.dumps(dict(cases=meta)).encode(), np.uint8)
    np.savez_compressed(args.out, **arrays)
    print("wrote", args.out, os.path.getsize(args.out), "bytes")


if __name__ == "__main__":
    main()
