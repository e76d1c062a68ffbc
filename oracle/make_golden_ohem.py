"""TEST INFRASTRUCTURE - generates tests/golden/ohem_cases.npz from the UNMODIFIED reference's `OhemCELoss` (utils/loss.py:303-328) on
the CPU:

    MYOLO_REFERENCE_ROOT=<checkout> python oracle/make_golden_ohem.py

(tests/golden/ohem_cases.npz, compressed; oracle.restate_ohem.load_cases reads it back.)

The reference's constructor moves its threshold to the GPU (`-torch.log(torch.tensor(thresh)).cuda()`).  This machine-independent
generator replaces `torch.Tensor.cuda` by the identity for the duration of the constructor call only, so the threshold stays the same
fp32 CPU scalar; nothing else of the reference is touched.

Each case is B=2 images of 19-class logits at 8 x 16 with labels in [0, 19) or -1 (ignored); it stores the logits, the labels, the
constructor arguments, the loss and d loss / d logits (autograd through the reference).  Cases: the threshold branch, the top-k branch,
fewer than 16 valid pixels with some hard ones (n_min = 0), every pixel ignored (NaN loss, zero gradient), and aux=True with
aux_weight [0.15, 0.1] over three outputs, one on each branch.  Every pixel's CE lies at least MARGIN (relative) away from -log(thresh)
and from the n_min-th largest CE, so that a last-bit difference in a per-pixel CE cannot change the selection; a case whose seeded draw
does not satisfy that is redrawn with the next seed.
"""
import argparse
import json
import os
import sys

import numpy as np
import torch
import torch.nn.functional as F

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
from oracle import ref_shims  # noqa: E402
from oracle.restate_ohem import thresh_t  # noqa: E402

GOLD = os.path.join(HERE, "..", "tests", "golden")
B, NC, H, W = 2, 19, 8, 16
THRESH = 0.7
MARGIN = 1e-3


def draw(seed, easy_bias, hard_frac, valid_frac=0.9, n_valid=None):
    """logits: randn, plus easy_bias on the label's class for all but a hard_frac share of the pixels; labels with 1 - valid_frac ignored
    (or exactly n_valid valid pixels)"""
    g = torch.Generator().manual_seed(seed)
    labels = torch.randint(0, NC, (B, H, W), generator=g)
    if n_valid is None:
        labels[torch.rand((B, H, W), generator=g) > valid_frac] = -1
    else:
        keep = torch.randperm(B * H * W, generator=g)[:n_valid]
        flat = torch.full((B * H * W,), -1, dtype=torch.long)
        flat[keep] = labels.view(-1)[keep]
        labels = flat.view(B, H, W)
    logits = torch.randn((B, NC, H, W), generator=g) * 1.5
    easy = (torch.rand((B, H, W), generator=g) >= hard_frac) & (labels >= 0)
    bias = F.one_hot(labels.clamp(min=0), NC).permute(0, 3, 1, 2).float() * easy[:, None] * easy_bias
    return (logits + bias).contiguous(), labels


def margins_ok(logits, labels, th):
    loss = F.cross_entropy(logits, labels, ignore_index=-1, reduction="none").view(-1)
    valid = (labels != -1).view(-1)
    lv = loss[valid]
    if lv.numel() and ((lv - th).abs() < MARGIN * th).any():
        return False
    n_min = int(valid.sum()) // 16
    if int((loss > th).sum()) < n_min:
        kth = torch.sort(loss, descending=True).values[n_min - 1]
        others = loss[(loss != kth)]
        if ((others - kth).abs() < MARGIN * kth.abs()).any() or int((loss == kth).sum()) != 1:
            return False
    return True


def case(name, ref_cls, spec, aux=False, aux_weight=(0.15, 0.05)):
    """spec: one draw() kwargs (or three, aux); the first seed from 1000 whose draws all keep the margins"""
    th = thresh_t(THRESH)
    specs = spec if aux else [spec]
    seed = 1000
    while True:
        drawn = [draw(seed + 17 * i, **s) for i, s in enumerate(specs)]
        labels = drawn[0][1]
        outs = [d[0] for d in drawn]
        if all(margins_ok(o, labels, th) for o in outs):
            break
        seed += 1
    orig = torch.Tensor.cuda
    torch.Tensor.cuda = lambda self, *a, **k: self          # the reference's constructor only: see the module docstring
    try:
        crit = ref_cls(thresh=THRESH, ignore_index=-1, aux=aux, aux_weight=list(aux_weight)) if aux else ref_cls(thresh=THRESH, ignore_index=-1)
    finally:
        torch.Tensor.cuda = orig
    ps = [o.clone().requires_grad_(True) for o in outs]
    loss = crit(ps if aux else ps[0], labels)
    loss.backward()
    print(f"{name}: seed {seed} loss {float(loss.detach())!r}")
    return dict(name=name, thresh=THRESH, ignore_index=-1, aux=aux, aux_weight=list(aux_weight), seed=seed, labels=labels,
                logits=[o.detach() for o in outs], loss=loss.detach(), grad=[p.grad.detach().clone() for p in ps])


def main():
    argp = argparse.ArgumentParser()
    argp.add_argument("--out", default=os.path.join(GOLD, "ohem_cases.npz"))
    args = argp.parse_args()
    ref_shims.import_reference()
    import utils.loss as ref_loss                            # the reference's (sys.path set by import_reference)
    R = ref_loss.OhemCELoss
    cases = [
        case("threshold", R, dict(easy_bias=0.0, hard_frac=1.0)),
        case("topk", R, dict(easy_bias=9.0, hard_frac=0.02)),
        case("nmin0", R, dict(easy_bias=0.0, hard_frac=1.0, n_valid=12)),
        case("all_ignored", R, dict(easy_bias=0.0, hard_frac=1.0, n_valid=0)),
        case("aux", R, [dict(easy_bias=9.0, hard_frac=0.02), dict(easy_bias=0.0, hard_frac=1.0), dict(easy_bias=6.0, hard_frac=0.2)],
             aux=True, aux_weight=(0.15, 0.1)),
    ]
    arrays, meta = {}, []
    for c in cases:
        n = c["name"]
        arrays[f"{n}_labels"] = c["labels"].numpy()
        arrays[f"{n}_loss"] = c["loss"].numpy()
        for i, (x, g) in enumerate(zip(c["logits"], c["grad"])):
            arrays[f"{n}_logits_{i}"] = x.numpy()
            arrays[f"{n}_grad_{i}"] = g.numpy()
        meta.append({k: c[k] for k in ("name", "thresh", "ignore_index", "aux", "aux_weight", "seed")} | {"n_outputs": len(c["logits"])})
    arrays["meta_json"] = np.frombuffer(json.dumps(dict(thresh_t=thresh_t(THRESH), margin=MARGIN, cases=meta)).encode(), np.uint8)
    np.savez_compressed(args.out, **arrays)
    print("wrote", args.out, os.path.getsize(args.out), "bytes")


if __name__ == "__main__":
    main()
