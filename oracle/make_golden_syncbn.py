"""TEST INFRASTRUCTURE — writes tests/golden/ref_ckpt_tiny_syncbn.pt: the checkpoint the reference's train.py:482-494 writes from a
`--sync-bn` run (train.py:190-193 `torch.nn.SyncBatchNorm.convert_sync_batchnorm(model)`), whose pickled `ckpt['model']` holds
SyncBatchNorm modules, and tests/golden/ref_ckpt_tiny_syncbn_out.npz: what the reference's own loading recipe
(`ckpt['model'].float().fuse().eval()`, models/experimental.py:119) computes from it.  The UNMODIFIED reference model is converted, then
saved as train.py does.  Runs on the CPU: in eval mode SyncBatchNorm is F.batch_norm.

    python oracle/make_golden_syncbn.py     # needs MYOLO_REFERENCE_ROOT

The weights follow make_golden.py gen_ckpt's recipe (same seeds, same draws per module) on a narrow yolov5s_city_seg (gen_ckpt's
quarter width, every Conv / C3 / SPP / Focus argument capped at 128 channels and the PSP head's hidden width at 128: 32 channels at most
in the backbone), so the fixture stays near half a megabyte while keeping all 73 BatchNorm layers.  The generator asserts that the
unconverted model computes the same outputs: the conversion changes the modules' class, nothing they compute in eval mode.
"""
import copy
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
from oracle import ref_shims, synth  # noqa: E402
from oracle.make_golden import GOLD, build_reference_model  # noqa: E402

CAP = 128


def narrow_cfg():
    cfg = synth.load_cfg("yolov5s_city_seg.yaml")
    cfg["width_multiple"] = 0.25
    for part in ("backbone", "head"):
        for row in cfg[part]:
            if row[2] in ("Conv", "C3", "SPP", "Focus"):
                row[3][0] = min(row[3][0], CAP)
            elif row[2] == "SegMaskPSP":
                row[3][2] = min(row[3][2], CAP)
    return cfg


def _load_and_run(path, x):
    m = torch.load(path, weights_only=False)["model"].float().fuse().eval()     # the reference's own loading recipe
    with torch.no_grad():
        (z, raw), seg = m(x)
    return z, raw, seg


def gen_ckpt_syncbn(ref_yolo):
    import tempfile
    cfg = narrow_cfg()
    torch.manual_seed(7)
    model = build_reference_model(ref_yolo, cfg)
    g = torch.Generator().manual_seed(11)
    with torch.no_grad():                      # gen_ckpt's weight recipe
        for m in model.modules():
            if isinstance(m, torch.nn.BatchNorm2d):
                m.running_mean.copy_(torch.randn(m.running_mean.shape, generator=g) * 0.1)
                m.running_var.copy_(torch.rand(m.running_var.shape, generator=g) + 0.5)
                m.weight.copy_(torch.rand(m.weight.shape, generator=g) * 0.4 + 0.8)
                m.bias.copy_(torch.randn(m.bias.shape, generator=g) * 0.1)
            elif isinstance(m, torch.nn.Conv2d):
                fan_in = m.weight.shape[1] * m.weight.shape[2] * m.weight.shape[3]
                m.weight.copy_(torch.randn(m.weight.shape, generator=g) * (2.0 / fan_in) ** 0.5)
    model.names = [f"cls{i}" for i in range(cfg["nc"])]
    n_bn = sum(isinstance(m, torch.nn.BatchNorm2d) for m in model.modules())
    x = synth.synth_image(1, 64, 64, seed=5)
    with tempfile.TemporaryDirectory() as tmp:                       # the same weights with plain BatchNorm, for the assertion below
        plain = os.path.join(tmp, "plain.pt")
        torch.save({"model": copy.deepcopy(model).half()}, plain)
        z0, raw0, seg0 = _load_and_run(plain, x)
    model = torch.nn.SyncBatchNorm.convert_sync_batchnorm(model)
    n_sync = sum(isinstance(m, torch.nn.SyncBatchNorm) for m in model.modules())
    assert n_sync == n_bn > 0 and not any(type(m) is torch.nn.BatchNorm2d for m in model.modules())
    ckpt = {"epoch": 3, "best_fitness": 0.5, "training_results": "synthetic", "model": copy.deepcopy(model).half(), "ema": None, "updates": 0,
            "optimizer": None, "wandb_id": None}
    path = os.path.join(GOLD, "ref_ckpt_tiny_syncbn.pt")
    torch.save(ckpt, path)
    z, raw, seg = _load_and_run(path, x)
    assert torch.equal(z, z0) and torch.equal(raw[0], raw0[0]) and torch.equal(seg, seg0)
    np.savez_compressed(os.path.join(GOLD, "ref_ckpt_tiny_syncbn_out.npz"), z=z.numpy(), seg_sub=seg[:, :, ::2, ::2].numpy(),
                        names=np.array(model.names), stride=model.stride.numpy(), n_sync=np.array(n_sync))
    print("ckpt (SyncBatchNorm)", os.path.getsize(path) / 1e6, "MB,", n_sync, "SyncBatchNorm layers;", z.shape, seg.shape)


if __name__ == "__main__":
    ref_yolo, _ = ref_shims.import_reference()
    gen_ckpt_syncbn(ref_yolo)
