"""TEST INFRASTRUCTURE - generates tests/golden/ema_cases.pt by driving the UNMODIFIED reference's `ModelEMA` (utils/torch_utils.py:270-304)
and `Model` (models/yolo.py) on the CPU:

    MYOLO_REFERENCE_ROOT=<checkout> python oracle/make_golden_ema.py

The model is yolov5s_city_seg.yaml loaded with `synth.synth_state_dict(manifest_s_psp, seed=1)`.  Before every update the training
model's floating-point entries, all but the two anchor buffers, are set to `base + 0.01 * randn` with the generator seeded by
`state_seed(i, j)` (i: the update's ordinal, j: the entry's index among the floating-point keys); `set_source_state` does it for the
reference here and for the CUDA path in the tests, bit for bit.  SEQUENCE is the reference's EMA life in training:

  * fp32 updates;
  * `ema.ema.half()` (what test.py:124 seg_validation does to the EMA), then fp16 updates, as in a --notest epoch;
  * `.float()` (test.py:333, the end of test()), then fp32 updates;
  * jumps of `ema.updates` that sample the decay ramp near 0, around 2000 and beyond 10^5;
  * a resume as train.py:151,162-164 and :485-486 do it: ckpt['ema'] = deepcopy(ema.ema).half(), a new ModelEMA(model),
    ema.ema.load_state_dict(ckpt['ema'].float().state_dict()), ema.updates = ckpt['updates'], then more updates.

The file holds the averaged keys in order with their dtypes before the first update, the `d` of every update (Python doubles), the
SHA-256 of every averaged entry after every update (uint8 [updates, keys, 32]), the EMA's dtype after every update, and the final
`anchors` / `anchor_grid` in full.
"""
import argparse
import copy
import hashlib
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
from oracle import ref_shims  # noqa: E402

GOLD = os.path.join(HERE, "..", "tests", "golden")
CFG = "yolov5s_city_seg.yaml"
NOISE = 0.01

# ("update", n): n updates; ("half",) / ("float",): the EMA's dtype; ("jump", k): ema.updates = k; ("resume",): checkpoint round trip
SEQUENCE = [("update", 3), ("half",), ("update", 3), ("float",), ("update", 2),
            ("jump", 1997), ("update", 3), ("half",), ("update", 2), ("float",),
            ("jump", 99998), ("update", 2), ("half",), ("update", 2), ("float",),
            ("resume",), ("update", 3)]


def state_seed(i: int, j: int) -> int:
    return 1_000_003 * (i + 1) + j


def averaged_keys(sd):
    return [k for k, v in sd.items() if v.dtype.is_floating_point]


def set_source_state(model, base, keys, i):
    """the training model's state before update number i (0-based): base + NOISE * randn for every averaged key but the anchors, in place
    (the model's tensors keep their storage).  base: {key: CPU fp32 tensor}."""
    import torch
    sd = model.state_dict()
    with torch.no_grad():
        for j, k in enumerate(keys):
            if k.endswith(".anchors") or k.endswith(".anchor_grid"):
                continue
            g = torch.Generator().manual_seed(state_seed(i, j))
            v = base[k] + NOISE * torch.randn(base[k].shape, generator=g, dtype=torch.float32)
            sd[k].copy_(v)


def digest(t) -> bytes:
    return hashlib.sha256(t.detach().cpu().contiguous().numpy().tobytes()).digest()


def replay(ema_cls, model, base, keys, on_update):
    """drives SEQUENCE: ema_cls(model) first, then the steps; on_update(i, ema, d) after every update.  Returns the last ModelEMA."""
    ema = ema_cls(model)
    i = 0
    for step in SEQUENCE:
        if step[0] == "update":
            for _ in range(step[1]):
                set_source_state(model, base, keys, i)
                ema.update(model)
                on_update(i, ema, ema.decay(ema.updates))
                i += 1
        elif step[0] == "half":
            ema.ema.half()
        elif step[0] == "float":
            ema.ema.float()
        elif step[0] == "jump":
            ema.updates = step[1]
        elif step[0] == "resume":
            ckpt = {"ema": copy.deepcopy(ema.ema).half(), "updates": ema.updates}
            ema = ema_cls(model)
            ema.ema.load_state_dict(ckpt["ema"].float().state_dict())
            ema.updates = ckpt["updates"]
        else:
            raise ValueError(step)
    return ema


def n_updates():
    return sum(s[1] for s in SEQUENCE if s[0] == "update")


def main():
    argp = argparse.ArgumentParser()
    argp.add_argument("--out", default=os.path.join(GOLD, "ema_cases.pt"))
    args = argp.parse_args()
    import torch
    from oracle import synth
    ref_yolo, _ = ref_shims.import_reference()
    import utils.torch_utils as ref_tu                      # the reference's (sys.path set by import_reference)
    torch.set_num_threads(min(16, os.cpu_count() or 1))
    cfg = synth.load_cfg(CFG)
    sd = synth.synth_state_dict(synth.load_manifest("s_psp"), cfg, seed=1)
    cwd = os.getcwd()
    os.chdir(ref_shims.REF_ROOT)
    try:
        torch.manual_seed(0)
        model = ref_yolo.Model(copy.deepcopy(cfg))
    finally:
        os.chdir(cwd)
    model.load_state_dict(sd)
    model.train()
    msd = model.state_dict()
    keys = averaged_keys(msd)
    base = {k: msd[k].detach().clone() for k in keys}
    dtypes = [str(msd[k].dtype) for k in keys]
    ds, digests, ema_dtypes = [], [], []

    def on_update(i, ema, d):
        esd = ema.ema.state_dict()
        assert averaged_keys(esd) == keys
        ds.append(float(d))
        digests.append(np.frombuffer(b"".join(digest(esd[k]) for k in keys), np.uint8).reshape(len(keys), 32))
        ema_dtypes.append(str(esd[keys[0]].dtype))
        print(f"update {i}: updates={ema.updates} d={d!r} {ema_dtypes[-1]}")

    ema = replay(ref_tu.ModelEMA, model, base, keys, on_update)
    esd = ema.ema.state_dict()
    out = dict(cfg=CFG, seed=1, noise=NOISE, sequence=SEQUENCE, keys=keys, dtypes=dtypes, d=np.asarray(ds, np.float64),
               updates=ema.updates, digests=np.stack(digests), ema_dtypes=ema_dtypes,
               anchors={k: esd[k].detach().clone() for k in keys if k.endswith(".anchors") or k.endswith(".anchor_grid")})
    assert len(ds) == n_updates()
    torch.save(out, args.out)
    print("wrote", args.out, os.path.getsize(args.out), "bytes")


if __name__ == "__main__":
    main()
