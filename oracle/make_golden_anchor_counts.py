"""TEST INFRASTRUCTURE - fixtures of models built with an anchor count (`Model(cfg, anchors=n)`, `hyp['anchors']` under --evolve), from
the UNMODIFIED reference on the CPU:

    MYOLO_REFERENCE_ROOT=<checkout> python oracle/make_golden_anchor_counts.py

tests/golden/anchor_count_cases.npz
    model_<n>_*       Model(yolov5s_city_seg, anchors=n) for n in 2, 2.5, 3.5, 4, 10 (torch.manual_seed(0)): the state-dict keys and
                      shapes, the anchors / anchor_grid buffers, the Detect biases before and after
                      _initialize_biases, yaml['anchors'] and the strides
    loss<na>_*        ComputeLoss (utils/loss.py:89-217, through make_golden.load_reference_loss) of that model at na = 4 and 10, its
                      anchors set to oracle.restate_evolve.anchor_table(na) as autoanchor would leave them: the loss, loss items and
                      d loss / d p on seeded predictions (restate_evolve.loss_predictions: drawn from the seed again by the tests, not stored) and
                      targets (B = 2, 64 x 128, data/hyp.scratch.yaml scaled as train.py does)
tests/golden/autoanchor_placeholder_cases.npz
    check_anchors (utils/autoanchor.py:23-68) on the placeholders of Model(cfg, anchors=n) for n = 2, 4 and 10 (3n anchors, one of them
    0 wide), in the format of autoanchor_cases.npz (oracle/make_golden_autoanchor.run_case)
"""
import json
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
from oracle import make_golden, make_golden_autoanchor, ref_shims, synth  # noqa: E402
from oracle.restate_evolve import LOSS_SHAPE, anchor_table, loss_predictions  # noqa: E402

GOLD = os.path.join(HERE, "..", "tests", "golden")
CFG = "yolov5s_city_seg.yaml"
MODEL_COUNTS = (2, 2.5, 3.5, 4, 10)


def ref_model(ref_yolo, n):
    torch.manual_seed(0)
    return ref_yolo.Model(synth.load_cfg(CFG), anchors=n)


def gen_models(ref_yolo, arrays):
    pre = {}
    real = ref_yolo.Model._initialize_biases

    def observed(self, cf=None):                           # records the Detect biases _initialize_biases starts from
        pre["b"] = [mi.bias.detach().clone() for mi in self.model[-1].m]
        return real(self, cf)
    for n in MODEL_COUNTS:
        ref_yolo.Model._initialize_biases = observed
        try:
            m = ref_model(ref_yolo, n)
        finally:
            ref_yolo.Model._initialize_biases = real
        det = m.model[-1]
        tag = f"model_{n}".replace(".", "p")
        sd = m.state_dict()
        arrays[f"{tag}_keys_json"] = np.frombuffer(json.dumps([[k, list(v.shape)] for k, v in sd.items()]).encode(), np.uint8)
        arrays[f"{tag}_anchors"] = det.anchors.numpy().copy()
        arrays[f"{tag}_anchor_grid"] = det.anchor_grid.numpy().copy()
        arrays[f"{tag}_stride"] = det.stride.numpy().copy()
        arrays[f"{tag}_yaml_anchors"] = np.array(m.yaml["anchors"])
        for i, mi in enumerate(det.m):
            arrays[f"{tag}_bias{i}"] = mi.bias.detach().numpy().copy()
            arrays[f"{tag}_bias_init{i}"] = pre["b"][i].numpy()
        print(tag, "na", det.na, "yaml anchors", m.yaml["anchors"], "keys", len(sd))


def gen_loss(ref_yolo, arrays):
    ref_loss = make_golden.load_reference_loss()
    cfg = synth.load_cfg(CFG)
    hyp = make_golden.loss_hyp(nl=3, nc=cfg["nc"], imgsz=256)
    arrays["loss_hyp_json"] = np.frombuffer(json.dumps(hyp).encode(), np.uint8)
    for na in (4, 10):
        model = ref_model(ref_yolo, na)
        model.hyp, model.gr, model.nc = hyp, 1.0, cfg["nc"]
        det = model.model[-1]
        a = torch.tensor(anchor_table(na), dtype=torch.float32).view(3, na, 2)
        det.anchors[:] = a / det.stride.view(-1, 1, 1)
        det.anchor_grid[:] = a.view(3, 1, na, 1, 1, 2)
        crit = ref_loss.ComputeLoss(model)
        B, nt = LOSS_SHAPE[0], 24
        p, rs = loss_predictions(na, det.no)
        p = [torch.from_numpy(q).requires_grad_(True) for q in p]
        t = np.zeros((nt, 6), np.float32)
        t[:, 0] = rs.randint(0, B, nt)
        t[:, 1] = rs.randint(0, cfg["nc"], nt)
        t[:, 2:4] = rs.uniform(0.02, 0.98, (nt, 2))
        t[:, 4:6] = rs.uniform(0.02, 0.5, (nt, 2))
        loss, items = crit(p, torch.from_numpy(t))
        loss.backward()
        tag = f"loss{na}"
        arrays[f"{tag}_anchors"] = det.anchors.numpy().copy()
        arrays[f"{tag}_targets"] = t
        for i in range(3):
            arrays[f"{tag}_g{i}"] = p[i].grad.numpy()
        arrays[f"{tag}_loss"] = loss.detach().numpy()
        arrays[f"{tag}_items"] = items.numpy()
        print(tag, "loss", float(loss.detach()), "items", items.tolist())


def gen_autoanchor():
    import utils.autoanchor as ref                        # the reference's (sys.path set by import_reference)
    base = dict(n_img=40, per_img=50, clusters=make_golden_autoanchor.CITY, spread=0.35)
    arrays, meta = {}, []
    for k, n in enumerate((2, 4, 10)):
        out = make_golden_autoanchor.run_case(f"placeholder{n}", ref, dict(base, seed=91 + k), anchors=[list(range(2 * n))] * 3,
                                              seed=900 + 100 * k)
        if out is None:
            continue
        m, a = out
        meta.append(m)
        for key, v in a.items():
            arrays[f"placeholder{n}_{key}"] = v
    arrays["meta_json"] = np.frombuffer(json.dumps(dict(ulp_margin=make_golden_autoanchor.ULP_MARGIN, cases=meta)).encode(), np.uint8)
    out = os.path.join(GOLD, "autoanchor_placeholder_cases.npz")
    np.savez_compressed(out, **arrays)
    print("wrote", out, os.path.getsize(out), "bytes")


def main():
    ref_yolo, _ = ref_shims.import_reference()
    arrays = {}
    gen_models(ref_yolo, arrays)
    gen_loss(ref_yolo, arrays)
    out = os.path.join(GOLD, "anchor_count_cases.npz")
    np.savez_compressed(out, **arrays)
    print("wrote", out, os.path.getsize(out), "bytes")
    gen_autoanchor()


if __name__ == "__main__":
    main()
