"""Measurements of model ensembles (models.experimental.Ensemble) on one GPU, B x 3 x 512 x 1024 fp16 with synthetic weights, for the
member sets s/PSP + m/PSP and s/PSP x 3 (seeds 1, 2, 3).  Every arm is followed by NMS(0.25, 0.45) and the seg argmax:
  - ensemble: Ensemble.forward (each member's passes into one z, one myolo_seg_ensemble launch for the mean seg);
  - composition: torch over the members' own forwards, torch.cat of the z's and torch.stack(seg).mean(0);
  - members: each member's plain forward with its own NMS and seg argmax, one after another (K single-model inferences);
  - ensemble_augment / composition_augment: the same with augment=True.
Arms alternate within each round; the figures are medians over rounds of CUDA-event times.  Also detect.py's frames/s with --submit
--nosave over the two reference-written test checkpoints against the first alone (wall clock around detect(), synchronised).  The
card's name and power limit are read in the same run.

    python tools/bench_ensemble.py [--rounds 5] [--steps 10] [--batch 16] [--out FILE]

Prints ONE JSON line (and writes it to --out).
"""
import argparse
import json
import os
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402
from tools.bench_train import timed_steps  # noqa: E402

H, W = 512, 1024
SETS = {"s_psp+m_psp": [("s_psp", "yolov5s_city_seg.yaml", 1), ("m_psp", "yolov5m_city_seg.yaml", 1)],
        "s_psp x3": [("s_psp", "yolov5s_city_seg.yaml", s) for s in (1, 2, 3)]}


def member(tag, yml, seed):
    """synthetic weights with bench.py's objectness-bias shift, so that NMS sees O(100) candidates per image, not thousands"""
    from multiyolov5_b200 import synth
    from multiyolov5_b200.models.yolo import Model
    cfg = synth.load_cfg(yml)
    sd = synth.synth_state_dict(synth.load_manifest(tag), cfg, seed=seed)
    for lvl in range(3):
        sd[f"model.25.m.{lvl}.bias"].view(-1, cfg["nc"] + 5)[:, 4] -= 10.0
    m = Model(yml)
    m.load_state_dict(sd)
    return m.cuda().eval().half()


def arms(name, B, steps, rounds):
    from multiyolov5_b200.models.experimental import Ensemble
    from multiyolov5_b200.utils.general import non_max_suppression, seg_argmax
    models = [member(*spec) for spec in SETS[name]]
    e = Ensemble()
    for m in models:
        e.append(m)
    e.eval()
    gen = torch.Generator(device="cuda").manual_seed(99)
    xs = [torch.rand((B, 3, H, W), device="cuda", generator=gen).half() for _ in range(2)]

    def post(z, seg):
        non_max_suppression(z, 0.25, 0.45, return_padded=True)
        seg_argmax(seg, (H, W))

    def composition(x, augment):
        outs = [m(x, augment=augment) for m in models]
        z = torch.cat([o[0][0] for o in outs], 1)
        seg = torch.stack([o[1].float() for o in outs]).mean(0).to(outs[0][1].dtype)
        return z, seg

    def run_members(x):
        for m in models:
            (z, _), seg = m(x)
            post(z, seg)

    def post_out(o):
        post(o[0][0], o[1])

    fns = {"ensemble": lambda i: post_out(e(xs[i % 2])),
           "composition": lambda i: post(*composition(xs[i % 2], False)),
           "members": lambda i: run_members(xs[i % 2]),
           "ensemble_augment": lambda i: post_out(e(xs[i % 2], augment=True)),
           "composition_augment": lambda i: post(*composition(xs[i % 2], True))}
    for f in fns.values():
        for i in range(3):
            f(i)
    ms = {k: [] for k in fns}
    for _ in range(rounds):
        for k, f in fns.items():
            ms[k].append(timed_steps(f, steps, 1) / steps)
    # the same outputs on one input: the ensemble against the composition (bit for bit by construction; reported, not assumed)
    (z, _), seg = e(xs[0])
    z0, seg0 = composition(xs[0], False)
    rec = {"workload": f"{'+'.join(s[0] + '/seed' + str(s[2]) for s in SETS[name])}, {B}x3x{H}x{W} fp16, + NMS(0.25, 0.45) + seg argmax",
           "equal_to_composition": bool(torch.equal(z, z0) and torch.equal(seg, seg0))}
    for k, v in ms.items():
        med = float(np.median(v))
        rec[k] = {"ms_per_step": med, "images_per_s": B / (med * 1e-3), "rounds_ms": [round(t, 2) for t in v]}
    rec["ensemble_minus_members_ms"] = rec["ensemble"]["ms_per_step"] - rec["members"]["ms_per_step"]
    rec["composition_minus_ensemble_ms"] = rec["composition"]["ms_per_step"] - rec["ensemble"]["ms_per_step"]
    del models, e, xs
    torch.cuda.empty_cache()
    return rec


def detect_fps(n_frames, rounds):
    """detect.py --submit --nosave over n_frames synthetic 1024 x 2048 frames at --img-size 1024, two weights against one"""
    from argparse import Namespace

    from multiyolov5_b200 import detect as D
    from multiyolov5_b200 import synth
    from multiyolov5_b200.models.experimental import attempt_load
    ckpts = [os.path.join(synth.GOLDEN_DIR, f) for f in ("ref_ckpt_tiny.pt", "ref_ckpt_tiny_syncbn.pt")]
    rs = np.random.RandomState(3)
    frames = [(f"/data/f_{i:03d}.png", torch.from_numpy(rs.randint(0, 256, (1024, 2048, 3), dtype=np.uint8)).cuda())
              for i in range(n_frames)]
    out = {}
    with tempfile.TemporaryDirectory() as tmp:
        runs = {"one_weight": attempt_load(ckpts[0]).cuda().eval(), "two_weights": attempt_load(ckpts).cuda().eval()}
        for name, model in runs.items():
            out[name] = []
        for r in range(rounds + 1):
            for name, model in runs.items():
                opt = Namespace(weights=ckpts, source="", img_size=1024, conf_thres=0.25, iou_thres=0.45, device="", view_img=False,
                                save_txt=False, save_conf=False, nosave=True, classes=None, agnostic_nms=False, augment=False,
                                update=False, project=tmp, name=f"{name}_{r}", exist_ok=True, save_as_video=False, submit=True,
                                batch_size=16)
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                D.detect(opt, dataset=frames, model=model)
                torch.cuda.synchronize()
                if r:                                     # round 0 builds the plans
                    out[name].append(n_frames / (time.perf_counter() - t0))
    return {k: {"frames_per_s": float(np.median(v)), "rounds": [round(x, 1) for x in v]} for k, v in out.items()} | {
        "workload": f"detect() --submit --nosave, {n_frames} frames 1024x2048 uint8 on the device, --img-size 1024, batch 16, "
                    "the reference-written test checkpoints (tests/golden/ref_ckpt_tiny*.pt)"}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--frames", type=int, default=64)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    torch.cuda.set_device(0)
    line = {"gpu": bench.gpu_state(0), "arms": {}}
    for name in SETS:
        line["arms"][name] = arms(name, args.batch, args.steps, args.rounds)
    line["detect"] = detect_fps(args.frames, args.rounds)
    line["gpu_after"] = bench.gpu_state(0)
    s = json.dumps(line)
    print(s, flush=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(s + "\n")


if __name__ == "__main__":
    main()
