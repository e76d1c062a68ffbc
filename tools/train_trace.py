"""CUPTI timeline of ONE training step (tools/bench_train.make_workload): wall, busy time per stream, union coverage, kernels ranked by total
device time.  Usage: python tools/train_trace.py [--out DIR]   (full per-kernel listing: DIR/train_trace_full.txt, default a temporary
directory)"""
import collections, json, os, sys, tempfile
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from tools.bench_train import make_workload
wl = make_workload(1, 0, 4)
tr, NROT = wl["tr"], wl["NROT"]
def step(i):
    k = i % NROT
    return tr.step(wl["imgs"][k], wl["tg"][k], wl["segimgs"][k], wl["masks"][k])
for i in range(5):
    step(i)
torch.cuda.synchronize()
from torch.profiler import profile, ProfilerActivity
with profile(activities=[ProfilerActivity.CUDA, ProfilerActivity.CPU]) as prof:
    for i in range(4):          # back to back (no synchronisation): the CPU runs ahead as it does in training; step 2 of 4 is analysed
        step(i)
    torch.cuda.synchronize()
f = tempfile.mktemp(suffix=".json")
prof.export_chrome_trace(f)
ev = [e for e in json.load(open(f))["traceEvents"] if e.get("cat") == "kernel"]
ev.sort(key=lambda e: e["ts"])
# a step ends with its sgd_step_kernel: cut there
ends = [i for i, e in enumerate(ev) if "sgd_step_kernel" in e["name"]]
assert len(ends) >= 3, len(ends)
t_lo = ev[ends[1]]["ts"] + ev[ends[1]]["dur"]
t_hi = ev[ends[2]]["ts"] + ev[ends[2]]["dur"]
st = [e for e in ev if t_lo <= e["ts"] < t_hi]
t0 = t_lo; end = t_hi
iv = sorted((e["ts"], e["ts"] + e["dur"]) for e in st)
cov, cs, ce = 0.0, iv[0][0], iv[0][1]
for a, b in iv[1:]:
    if a > ce:
        cov += ce - cs; cs, ce = a, b
    else:
        ce = max(ce, b)
cov += ce - cs
print(f"# one step: {len(st)} kernels, wall {end - t0:.0f} us, sum of durations {sum(e['dur'] for e in st):.0f} us, union {cov:.0f} us, idle {end - t0 - cov:.0f} us")
busy = collections.Counter()
for e in st:
    busy[e["args"].get("stream")] += e["dur"]
print("# busy us per stream:", dict(sorted(((k, round(v)) for k, v in busy.items()), key=lambda kv: -kv[1])[:12]))
agg = collections.defaultdict(lambda: [0, 0.0])
for e in st:
    n = e["name"].replace("myolo::", "").replace("void ", "").split("(")[0][:70]
    agg[n][0] += 1; agg[n][1] += e["dur"]
for n, (c, t) in sorted(agg.items(), key=lambda kv: -kv[1][1])[:28]:
    print(f"{t:9.1f} us {c:5d}x  {n}")
# phase markers: first / last kernel of each stream
for s in list(busy)[:6]:
    ks = [e for e in st if e["args"].get("stream") == s]
    print(f"# stream {s}: {len(ks)} kernels from {ks[0]['ts'] - t0:.0f} to {ks[-1]['ts'] + ks[-1]['dur'] - t0:.0f} us")

# concurrency profile: per 0.5 ms bucket, kernel-time / wall-time (> 1 means kernels of different streams overlap) and the dominant kernels
B = 500.0
nb = int((end - t0) / B) + 1
load = [0.0] * nb
names = [collections.Counter() for _ in range(nb)]
for e in st:
    a, b = e["ts"] - t0, e["ts"] - t0 + e["dur"]
    k = int(a / B)
    while a < b and k < nb:
        hi = min(b, (k + 1) * B)
        load[k] += hi - a
        names[k][e["name"].replace("myolo::", "").replace("void ", "").split("(")[0].split("<")[0][:22]] += hi - a
        a = hi; k += 1
print("# bucket(ms)  kernel-time/wall  top kernels")
for k in range(nb):
    print(f"{k * B / 1000:6.1f}  {load[k] / B:5.2f}  " + ", ".join(f"{n}:{t:.0f}" for n, t in names[k].most_common(3)))

print("# individual launches of selected kernels (start us, duration us, grid):")
for e in st:
    if any(k in e["name"] for k in ("conv_simt", "spp_bwd", "seg_ce", "zero_stuff")):
        print(f"{e['ts'] - t0:9.0f} {e['dur']:7.1f} grid{e['args'].get('grid')} {e['name'].replace('myolo::', '')[:60]}")

# the whole step, one line per kernel (start us, duration us, stream, name): <out>/train_trace_full.txt
out_dir = sys.argv[sys.argv.index("--out") + 1] if "--out" in sys.argv else tempfile.mkdtemp(prefix="train_trace_")
os.makedirs(out_dir, exist_ok=True)
print(f"# full listing: {os.path.join(out_dir, 'train_trace_full.txt')}")
with open(os.path.join(out_dir, "train_trace_full.txt"), "w") as fh:
    for e in st:
        fh.write(f"{e['ts'] - t0:9.1f} {e['dur']:7.1f} s{e['args'].get('stream')} grid{e['args'].get('grid')} "
                 f"{e['name'].replace('myolo::', '').replace('void ', '')[:90]}\n")
