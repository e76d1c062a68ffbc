"""Restatement of a model ensemble (reference models/experimental.py:98-110, `Ensemble.forward`) over `restate.model_forward`.

The fork's loop appends `module(x, augment)[0]`, which in this fork is the pair (z, raw list), and then `torch.cat`s those pairs, which
fails; the loop restated here takes z, `module(x, augment)[0][0]`, and concatenates the members' z along the rows (the reference's "nms
ensemble").  The seg output is the mean of the members' seg logits, `torch.stack(segs).mean(0)` (the reference's commented "mean
ensemble" of models/experimental.py:108 applied to the seg output, which the fork does not define), and the class map its argmax.
"""
import torch

from oracle import restate, synth


def ensemble(outs):
    """outs: each member's forward_once output [(z, raw), seg] -> (z, mean seg, argmax of the mean)"""
    z = torch.cat([o[0][0] for o in outs], 1)
    mean = torch.stack([o[1].float() for o in outs]).mean(0)
    return z, mean.to(outs[0][1].dtype), mean.argmax(1)


def model_forward_ensemble(members, x: torch.Tensor, half: bool = False):
    """members: [(cfg, state_dict)] -> (z, seg, argmax) of the ensemble: fp32 on the CPU, or (half=True, CUDA input and weights) the torch
    fp16 yardstick of restate.model_forward"""
    outs = []
    for cfg, sd in members:
        y = restate.model_forward(cfg, sd, x, half=half)
        outs.append([(y["z"], y["raw"]), y["seg"]])
    return ensemble(outs)


def fixture_members(g):
    """[(cfg, state_dict)] of the members of tests/golden/ensemble_cases.npz (synthetic weights from the manifests and seeds)"""
    return [(synth.load_cfg(yml), synth.synth_state_dict(synth.load_manifest(tag), synth.load_cfg(yml), seed=int(seed)))
            for tag, yml, seed in g["members"]]


def fixture_input(g, k):
    """the input of case k of tests/golden/ensemble_cases.npz, checked against the stored sum"""
    B, H, W = (int(v) for v in g[f"case{k}_shape"])
    x = synth.synth_image(B, H, W, seed=int(g[f"case{k}_seed"]))
    s = float(g[f"case{k}_x_sum"])
    assert abs(x.double().sum().item() - s) <= 1e-12 * abs(s), "synth.synth_image no longer reproduces the fixture's input"
    return x
