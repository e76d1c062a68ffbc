"""TEST INFRASTRUCTURE — generates the l / x fixtures in tests/golden/ by running the UNMODIFIED reference (a checkout named by
MYOLO_REFERENCE_ROOT, imported through oracle/ref_shims.py) on a CPU machine.  The reference builds its city-seg graph at any
depth / width multiple (models/yolo.py parse_model) but ships no l / x city-seg yaml: the yamls of multiyolov5_b200/models are the s
graphs at the upstream yolov5l (1.0 / 1.0) and yolov5x (1.33 / 1.25) multiples, and the reference's own `Model` is built from them.

    MYOLO_REFERENCE_ROOT=... python oracle/make_golden_sizes.py

Fixtures (weights are NOT stored — they are re-synthesised from the manifest + seed, as for make_golden.py):
  manifest_<tag>.json.gz  reference state_dict keys / shapes / dtypes (gzip: the l / x key lists are 40 - 50 KB of JSON each)
  net_<tag>.npz           Model.forward (eval, fused) at 1 x 3 x 64 x 128: z (fp32), raw x_i (fp16, with their fp32 max |.|), the
                          low-resolution seg logits (fp32), the argmax of the upsampled seg, taps of layers 9 and 23 (fp16), and the largest
                          |activation| of any layer at 1 x 3 x 256 x 512.  The input is re-created from its seed by the tests (its sum is
                          stored as a checksum).  At this size the maps below P3 are too small for the wgmma kernel; the GPU tests check
                          the tensor-core sizes against the fp32 restatement, which these fixtures pin to the reference.
"""
import gzip
import json
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
from oracle import ref_shims, synth  # noqa: E402
from oracle.make_golden import build_reference_model  # noqa: E402

GOLD = os.path.join(HERE, "..", "tests", "golden")

# tag -> yaml in multiyolov5_b200/models
SIZE_CASES = {
    "l_psp": "yolov5l_city_seg.yaml", "l_lab": "yolov5l_city_seg_lab.yaml", "l_bise": "yolov5l_city_seg_bise.yaml",
    "l_base": "yolov5l_city_seg_base.yaml",
    "x_psp": "yolov5x_city_seg.yaml", "x_lab": "yolov5x_city_seg_lab.yaml", "x_bise": "yolov5x_city_seg_bise.yaml",
    "x_base": "yolov5x_city_seg_base.yaml",
}
B, H, W, SEED = 1, 64, 128, 3
H_RANGE, W_RANGE = 256, 512      # the activation-range check runs at the size the GPU tests use
TAPS = (9, 23)
FP16_MAX = 65504.0


def gen(ref_yolo, tag, yml):
    cfg = synth.load_cfg(yml)
    torch.manual_seed(0)
    model = build_reference_model(ref_yolo, cfg)
    sd0 = model.state_dict()
    manifest = [[k, list(v.shape), str(v.dtype).replace("torch.", "")] for k, v in sd0.items()]
    with gzip.open(os.path.join(GOLD, f"manifest_{tag}.json.gz"), "wt") as f:
        json.dump(manifest, f)
    n_params = sum(p.numel() for p in model.parameters())
    sd = synth.synth_state_dict(manifest, cfg, seed=1)
    for k in sd:   # anchor buffers must equal what the reference itself computed
        if k.endswith(".anchors") or k.endswith(".anchor_grid"):
            assert torch.allclose(sd[k], sd0[k]), k
    model.load_state_dict(sd)
    model.fuse().eval()
    x = synth.synth_image(B, H, W, seed=SEED)
    feats, lowres, absmax = {}, {}, {}

    def tap(i):
        def hook(m, a, o):
            outs = o if isinstance(o, (list, tuple)) else [o]
            absmax[i] = max(absmax.get(i, 0.0), max(float(t.abs().max()) for t in outs if torch.is_tensor(t)))
            if i in TAPS:
                feats[i] = o.detach().clone()
        return hook
    hooks = [model.model[i].register_forward_hook(tap(i)) for i in range(len(model.model) - 1)]
    seg_head = model.model[24]
    seq = seg_head.out if hasattr(seg_head, "out") else (seg_head.decoder if hasattr(seg_head, "decoder") else seg_head.m)
    hooks.append(seq[-1].register_forward_hook(lambda m, a, o: lowres.__setitem__("x", a[0].detach().clone())))
    with torch.no_grad():
        model(synth.synth_image(1, H_RANGE, W_RANGE, seed=SEED))
        # the synthetic weights must keep every activation well inside fp16 range, or the GPU parity tests would compare overflowed tensors
        worst = max(absmax.values())
        worst_layer = max(absmax, key=absmax.get)
        (z, raw), seg = model(x)
    for h in hooks:
        h.remove()
    assert worst < FP16_MAX / 16, (tag, worst, absmax)
    arrs = dict(x_sum=np.float64(x.double().sum().item()), z=z.numpy(), seg_lowres=lowres["x"].numpy(),
                seg_argmax=seg.argmax(1).numpy().astype(np.uint8), seed=np.int64(SEED), shape=np.array([B, H, W]),
                n_params=np.int64(n_params), act_absmax=np.float32(worst))
    for i, r in enumerate(raw):
        arrs[f"raw{i}"] = r.numpy().astype(np.float16)
        arrs[f"raw{i}_absmax"] = np.float32(r.abs().max().item())
    for i, t in feats.items():
        arrs[f"layer{i}"] = t.numpy().astype(np.float16)
    path = os.path.join(GOLD, f"net_{tag}.npz")
    np.savez_compressed(path, **arrs)
    print(f"{tag}: {n_params / 1e6:.2f} M parameters, largest |activation| {worst:.1f} (layer {worst_layer}), "
          f"z |max| {float(z.abs().max()):.1f}, {os.path.getsize(path) / 1e6:.2f} MB")


if __name__ == "__main__":
    os.makedirs(GOLD, exist_ok=True)
    ref_yolo, _ = ref_shims.import_reference()
    torch.set_num_threads(min(32, os.cpu_count() or 1))
    only = set(sys.argv[1:])
    for tag, yml in SIZE_CASES.items():
        if not only or tag in only:
            gen(ref_yolo, tag, yml)
