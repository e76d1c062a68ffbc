"""Deterministic synthetic weights / inputs (there is no network for real checkpoints or datasets): used by bench.py, the tools and -
through the re-export in the checker package - by the golden-fixture generator and the tests, so that every parity run hands the SAME
synthetic `state_dict` (reference key names, from tests/golden/manifest_*.json) to the reference, its CPU restatement and the CUDA path.  numpy's legacy RandomState is frozen across versions, so the
values are reproducible on the GPU box without shipping 31 MB of weights.

BN statistics are randomised on purpose (reference defaults 0/1/1/0 would make BN folding trivial,
SURVEY.md §8c "Weights").
"""
import gzip
import json
import os
from typing import Dict, List

import numpy as np
import torch

GOLDEN_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests", "golden")
CFG_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "models")


def load_cfg(name: str) -> dict:
    import yaml
    with open(os.path.join(CFG_DIR, name)) as f:
        return yaml.safe_load(f)


def load_manifest(tag: str) -> List[list]:
    path = os.path.join(GOLDEN_DIR, f"manifest_{tag}.json")
    if not os.path.isfile(path):      # the l / x manifests are stored compressed
        with gzip.open(path + ".gz", "rt") as f:
            return json.load(f)
    with open(path) as f:
        return json.load(f)


def synth_state_dict(manifest: List[list], cfg: dict, seed: int = 1, gain: float = None) -> Dict[str, torch.Tensor]:
    """manifest: [[key, shape, dtype_str], ...] in the reference's state_dict order."""
    if gain is None:  # near-critical gains keep activations O(1..10) through ~60 layers (calibrated, see DESIGN.md).  The deeper l / x
        # C3 stacks amplify faster: at 1.9 their largest activation is 2e4 (l) and 1e6 (x); at 1.6 / 1.4 it is 11 / 10
        w = cfg["width_multiple"]
        gain = 2.0 if w <= 0.5 else (1.9 if w <= 0.75 else (1.6 if w <= 1.0 else 1.4))
    rs = np.random.RandomState(seed)
    sd = {}
    strides = [8.0, 16.0, 32.0]
    for key, shape, dt in manifest:
        shape = tuple(shape)
        if key.endswith("num_batches_tracked"):
            v = np.zeros(shape, np.int64)
        elif key.endswith(".anchors"):
            a = np.asarray(cfg["anchors"], np.float32).reshape(len(cfg["anchors"]), -1, 2)
            v = a / np.asarray(strides, np.float32).reshape(-1, 1, 1)
        elif key.endswith(".anchor_grid"):
            v = np.asarray(cfg["anchors"], np.float32).reshape(len(cfg["anchors"]), 1, -1, 1, 1, 2)
        elif key.endswith("running_var"):
            v = rs.uniform(0.5, 1.5, shape)
        elif key.endswith("running_mean"):
            v = rs.normal(0.0, 0.1, shape)
        elif len(shape) == 4:
            fan_in = shape[1] * shape[2] * shape[3]
            v = rs.normal(0.0, np.sqrt(gain / fan_in), shape)
        elif key.endswith("bn.weight") or (len(shape) == 1 and key.split(".")[-2].isdigit() and key.endswith(".weight")):
            v = rs.uniform(0.8, 1.2, shape)       # BN gamma (Conv.bn.weight, or bare nn.Sequential BN '.1.weight')
        elif key.endswith("bn.bias") or (len(shape) == 1 and key.endswith(".1.bias")):
            v = rs.normal(0.0, 0.1, shape)        # BN beta
        elif key.endswith(".bias"):
            v = rs.normal(0.0, 0.5, shape)        # Conv2d bias of Detect / seg classifier
        else:
            raise KeyError(f"synth: unclassified key {key} {shape}")
        t = torch.from_numpy(np.asarray(v).astype(np.int64 if dt == "int64" else np.float32))
        sd[key] = t.reshape(shape)
    return sd


def synth_image(b: int, h: int, w: int, seed: int = 0) -> torch.Tensor:
    rs = np.random.RandomState(seed)
    return torch.from_numpy(rs.uniform(0.0, 1.0, (b, 3, h, w)).astype(np.float32))


def synth_predictions(b: int, n: int, nc: int = 10, seed: int = 0, W: float = 1024.0, H: float = 512.0) -> np.ndarray:
    """SURVEY.md §8d config 5: cxcy~U([0,W]x[0,H]), wh~U(4,104), obj~U(0.3,1), cls~U(0,1)."""
    rs = np.random.RandomState(seed)
    p = np.empty((b, n, 5 + nc), np.float32)
    p[..., 0] = rs.uniform(0, W, (b, n))
    p[..., 1] = rs.uniform(0, H, (b, n))
    p[..., 2:4] = rs.uniform(4, 104, (b, n, 2))
    p[..., 4] = rs.uniform(0.3, 1.0, (b, n))
    p[..., 5:] = rs.uniform(0, 1, (b, n, nc))
    return p
