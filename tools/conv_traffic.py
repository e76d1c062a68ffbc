"""Per-launch operand traffic of the wgmma conv kernel against its measured time.

Reads the `#conv` table that `bench.py --profile-ops` prints to stderr and, from each launch's shape and tiling (`myolo_plan_conv_info`),
computes the bytes the kernel moves from L2 into shared memory: A (activation boxes or strips) and B (weights), the number of TMA pixel
rows, and the launch's HBM floor (input + output activations and weights once, fp16, at 3.35 TB/s, or the FLOPs at 989 TFLOP/s if
larger; residual reads are not counted).  Prints one row per launch and the totals.

    python tools/conv_traffic.py bench_stderr.txt [--batch 16]
"""
import argparse
import re

HBM_BPS, TC_FLOPS = 3.35e12, 989e12
LINE = re.compile(r"^#conv\s+(\d+)\s+(\S+)\s+(\d+)->(\d+) k(\d)s(\d)d(\d+) @(\d+)x(\d+)\s+\[([^\]]*)\]\s+([\d.]+) us")


def choose_tile(w, h):   # conv_tc.cu choose_tile
    best = None
    t = 128
    while t >= 8:
        tiles = -(-w // t) * -(-h // (128 // t))
        if best is None or tiles < best[0]:
            best = (tiles, t, 128 // t)
        t //= 2
    return best[1], best[2]


def launch_traffic(ci, co, k, stride, dil, ho, wo, info, batch):
    _, grid, _, bn, _, strip, resident, _, tiles, ntn, kc, _ = info
    ci_pad = -(-ci // kc) * kc
    cblocks, taps = ci_pad // kc, k * k
    tw, th = choose_tile(wo, ho)
    if strip:
        sw = tw + 2 * dil
        a_rows = 3 * cblocks * sw * th
    else:
        a_rows = taps * cblocks * 128
    a = tiles * a_rows * kc * 2
    pack = taps * ci_pad * bn * 2
    b = grid * pack if resident else tiles * pack
    flops = 2.0 * batch * ho * wo * co * ci * taps
    hbm = batch * (ho * stride) * (wo * stride) * ci * 2 + batch * ho * wo * co * 2 + co * ci * taps * 2
    return a, b, tiles * a_rows, max(hbm / HBM_BPS, flops / TC_FLOPS)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("profile")
    ap.add_argument("--batch", type=int, default=16)
    args = ap.parse_args()
    tot = [0.0] * 5
    print(f"{'op':>3} {'layer':14s} {'shape':24s} {'path':6s} {'us':>7} {'A MB':>7} {'B MB':>7} {'rows M':>7} {'floor us':>8} "
          f"{'L2->SM TB/s':>11} {'x floor':>7}")
    for line in open(args.profile):
        m = LINE.match(line)
        if not m:
            continue
        info = [int(v) for v in m.group(10).split(",")]
        if not info[0]:
            continue
        op, tag = int(m.group(1)), m.group(2)
        ci, co, k, s, d, ho, wo = (int(m.group(i)) for i in range(3, 10))
        us = float(m.group(11))
        a, b, rows, floor = launch_traffic(ci, co, k, s, d, ho, wo, info, args.batch)
        path = ("S" if info[5] else "T") + ("R" if info[6] else "-")
        print(f"{op:3d} {tag:14s} {f'{ci}->{co} k{k}s{s}d{d} @{ho}x{wo}':24s} {path:6s} {us:7.1f} {a / 1e6:7.1f} {b / 1e6:7.1f} "
              f"{rows / 1e6:7.2f} {floor * 1e6:8.1f} {(a + b) / (us * 1e-6) / 1e12:11.2f} {us / (floor * 1e6):7.2f}")
        for i, v in enumerate((us, a, b, rows, floor * 1e6)):
            tot[i] += v
    print(f"total: {tot[0]:.1f} us, A {tot[1] / 1e9:.2f} GB, B {tot[2] / 1e9:.2f} GB, {tot[3] / 1e6:.1f} M rows, floors {tot[4]:.1f} us")
    print("path: T = one TMA box per tap, S = one strip per filter row; R = resident weights, - = streamed")


if __name__ == "__main__":
    main()
