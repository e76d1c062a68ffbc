"""Measurements of the l and x city-seg models (yolov5{l,x}_city_seg.yaml, PSP head) on one GPU:
  - inference images/s at B x 3 x 512 x 1024 fp16 (Model.forward + NMS(0.25, 0.45) + seg argmax, as bench.py's headline step), against the
    same job through torch fp16 + cuDNN on the same graph (oracle/gpu_pipeline.py), in alternating rounds;
  - the Trainer.step time at 4 det + 4 seg images of 3 x 512 x 1024 (tools/bench_train.py's workload);
  - SPP.cv2's data gradient (4 c_ = 2048 / 2560 output channels) on the wgmma kernel against the CUDA-core kernel it ran on before, kernel
    time from torch.profiler on the same seeded inputs, and the difference of the two results.
Every shape is warmed up; the figures are medians over rounds.  The card's name and power limit are read in the same run.

    python tools/bench_sizes.py [--rounds 5] [--steps 10] [--batch 16] [--out FILE]

Prints ONE JSON line (and writes it to --out).
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402
from tools.bench_train import timed_steps  # noqa: E402

H, W = 512, 1024
MODELS = {"l_psp": "yolov5l_city_seg.yaml", "x_psp": "yolov5x_city_seg.yaml"}


def weights(tag):
    """the synthetic weights, with bench.py's objectness-bias shift so that NMS sees O(100) candidates per image, not thousands"""
    from multiyolov5_b200 import synth
    yml = MODELS[tag]
    cfg = synth.load_cfg(yml)
    sd = synth.synth_state_dict(synth.load_manifest(tag), cfg, seed=1)
    for lvl in range(3):
        sd[f"model.25.m.{lvl}.bias"].view(-1, cfg["nc"] + 5)[:, 4] -= 10.0
    return yml, cfg, sd


def infer(tag, B, steps, rounds):
    from multiyolov5_b200.models.yolo import Model
    from multiyolov5_b200.utils.general import non_max_suppression, seg_argmax
    from oracle.gpu_pipeline import TorchHalfPipeline
    yml, cfg, sd = weights(tag)
    model = Model(yml)
    model.load_state_dict(sd)
    model.cuda().eval().half()
    ref = TorchHalfPipeline(cfg, sd)
    gen = torch.Generator(device="cuda").manual_seed(99)
    xs = [torch.rand((B, 3, H, W), device="cuda", generator=gen).half() for _ in range(4)]
    n_det = []

    def ours(i):
        (z, _), seg = model(xs[i % 4])
        det, cnt = non_max_suppression(z, 0.25, 0.45, return_padded=True)
        seg_argmax(seg, (H, W))
        if i == 0:
            n_det.append(cnt)

    def torch_ref(i):
        ref(xs[i % 4])
    for i in range(3):
        ours(i)
        torch_ref(i)
    ms = {"ours": [], "torch": []}
    for _ in range(rounds):
        ms["ours"].append(timed_steps(ours, steps, 1) / steps)
        ms["torch"].append(timed_steps(torch_ref, steps, 1) / steps)
    rec = {"workload": f"{yml} inference, {B}x3x{H}x{W} fp16: Model.forward + NMS(0.25, 0.45) + seg argmax", "batch": B}
    for k, v in ms.items():
        med = float(np.median(v))
        rec[k] = {"ms_per_step": med, "images_per_s": B / (med * 1e-3), "rounds_ms": [round(t, 2) for t in v]}
    rec["torch"]["kind"] = ref.kind
    rec["speedup"] = rec["ours"]["images_per_s"] / rec["torch"]["images_per_s"]
    rec["detections_per_image"] = float(n_det[-1].float().mean()) if n_det else None
    del model, ref, xs
    torch.cuda.empty_cache()
    return rec


def train(tag, steps, rounds, B=4):
    from multiyolov5_b200 import synth
    from multiyolov5_b200.models.yolo import Model
    from multiyolov5_b200.train import Trainer, scale_hyp
    yml = MODELS[tag]
    cfg = synth.load_cfg(yml)
    model = Model(yml)
    model.load_state_dict(synth.synth_state_dict(synth.load_manifest(tag), cfg, seed=1, gain=1.0))
    model.cuda().train()
    hyp = dict(lr0=0.0015, momentum=0.937, weight_decay=5e-4, box=0.05, cls=0.5, cls_pw=1.0, obj=1.0, obj_pw=1.0, anchor_t=4.0, fl_gamma=0.0)
    tr = Trainer(model, scale_hyp(hyp, nl=3, nc=cfg["nc"], imgsz=W, total_batch_size=B), batch_size=B, init_scale=2.0 ** 10)
    gen = torch.Generator(device="cuda").manual_seed(77)
    imgs = [torch.rand((B, 3, H, W), device="cuda", generator=gen) for _ in range(3)]
    segimgs = [torch.rand((B, 3, H, W), device="cuda", generator=gen) for _ in range(3)]
    rs = np.random.RandomState(5)
    tg = []
    for _ in range(3):
        t = np.zeros((20 * B, 6), np.float32)
        t[:, 0] = np.repeat(np.arange(B), 20); t[:, 1] = rs.randint(0, 10, 20 * B)
        t[:, 2:4] = rs.uniform(0.1, 0.9, (20 * B, 2)); t[:, 4:6] = rs.uniform(0.02, 0.22, (20 * B, 2))
        tg.append(torch.from_numpy(t).cuda())
    masks = [torch.randint(-1, 19, (B, H, W), device="cuda", generator=gen) for _ in range(3)]
    last = []

    def step(i):
        last[:] = tr.step(imgs[i % 3], tg[i % 3], segimgs[i % 3], masks[i % 3])
    for i in range(3):
        step(i)
    ms = [timed_steps(step, steps, 1) / steps for _ in range(rounds)]
    med = float(np.median(ms))
    rec = {"workload": f"{yml} Trainer.step, {B} det + {B} seg images 3x{H}x{W}, 20 boxes/img", "ms_per_step": med,
           "images_per_s": 2 * B / (med * 1e-3), "rounds_ms": [round(t, 2) for t in ms], "max_memory_allocated_gb": torch.cuda.max_memory_allocated() / 1e9,
           "last_losses": {"det": [float(v) for v in last[0]], "seg": float(last[1])}, "loss_scale": float(tr.scale)}
    del model, tr
    torch.cuda.empty_cache()
    return rec


def spp_dgrad(B, Hm, Wm, ci, co, reps):
    """SPP.cv2's backward on its train-plan geometry (B x Hm x Wm, fp16 NHWC), data gradient on the wgmma kernel (route 0) and on the
    CUDA-core kernel (route CONV_BWD_SIMT), same inputs and prior; kernel times from the profiler, medians over the launches"""
    from torch.profiler import ProfilerActivity, profile

    from multiyolov5_b200 import _lib, ops
    g = torch.Generator(device="cuda").manual_seed(ci)
    x = torch.randn((B, Hm, Wm, ci), generator=g, device="cuda").half()
    dy = torch.randn((B, Hm, Wm, co), generator=g, device="cuda").half()
    w = torch.randn((co, ci, 1, 1), generator=g, device="cuda") / co ** 0.5
    prior = torch.randn((B, Hm, Wm, ci), generator=g, device="cuda").half()
    out, times, launches = {}, {}, {}
    for name, route, kernel in (("wgmma", 0, "conv_tc_kernel"), ("simt", _lib.CONV_BWD_SIMT, "conv_simt_kernel")):
        dW = torch.zeros_like(w)
        gin = prior.clone()
        info = ops.conv_backward(x, w, dy, dW, gin=gin, route=route)
        assert info[0] == (2 if route == 0 else 3), info
        out[name] = gin.double() - prior.double()
        for _ in range(2):
            ops.conv_backward(x, w, dy, torch.zeros_like(w), gin=prior.clone(), route=route)
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(reps):
                ops.conv_backward(x, w, dy, dW, gin=gin, route=route)
            torch.cuda.synchronize()
        ts = [e.device_time for e in prof.events() if kernel in e.name]
        launches[name] = len(ts)
        times[name] = float(np.median(ts)) * 1e-3 if ts else float("nan")    # ms
    d = (out["wgmma"] - out["simt"]).abs()
    ulp = prior.double().abs().add(out["simt"].abs()).clamp_min(2.0 ** -14) * 2.0 ** -10   # one fp16 ulp of the stored sum (upper bound)
    flops = 2.0 * B * Hm * Wm * ci * co
    return {"shape": f"B={B} {Hm}x{Wm}, dY {co} -> grad(in) {ci} channels, 1x1", "wgmma_ms": times["wgmma"], "simt_ms": times["simt"],
            "speedup": times["simt"] / times["wgmma"], "timed_launches": launches, "wgmma_tflops": flops / (times["wgmma"] * 1e-3) / 1e12,
            "max_abs_diff": float(d.max()), "max_diff_in_fp16_ulps": float((d / ulp).max()),
            "share_of_elements_differing": float((d > 0).double().mean()), "max_abs_grad": float(out["simt"].abs().max())}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    torch.cuda.set_device(0)
    line = {"gpu": bench.gpu_state(0), "infer": {}, "train": {}, "spp_cv2_dgrad": {}}
    for tag in MODELS:
        line["infer"][tag] = infer(tag, args.batch, args.steps, args.rounds)
        line["train"][tag] = train(tag, args.steps, args.rounds)
    for tag, (ci, co) in {"l_psp": (2048, 1024), "x_psp": (2560, 1280)}.items():
        line["spp_cv2_dgrad"][tag] = [spp_dgrad(B, 16, 32, ci, co, 20) for B in (4, 16)]
    line["gpu_after"] = bench.gpu_state(0)
    s = json.dumps(line)
    print(s, flush=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(s + "\n")


if __name__ == "__main__":
    main()
