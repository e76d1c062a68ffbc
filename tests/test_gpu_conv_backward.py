"""GPU: the backward of one conv on its own - data, weight and bias gradients - through the train plan's own routing and launches
(ops.conv_backward -> csrc/plan.cu conv_backward_views, the function the plan's backward walk calls), against autograd of F.conv2d in
fp64 on the values each kernel actually reads:
  - weights: the wgmma and CUDA-core data gradients multiply the fp16 pack of the flipped weights, the small route the fp32 masters;
  - dY: an fp32 head gradient is cast to fp16 before the data and weight gradients of the tensor-core routes, never before the bias
    gradient, and not at all on the small route.
Every gradient is accumulated into a nonzero prior, every view is a channel slice of a wider buffer, and every word outside the slices
(other channels, pixel rows past the map) holds an fp16 / fp32 NaN that must survive.  Each case asserts the route it was built for, so a
silent fall-back fails.  The census runs the same entry at the exact geometry and slice layout of every conv op of two train plans at
three input shapes."""
from collections import defaultdict

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

U16 = 2.0 ** -11            # fp16 unit roundoff: one rounding of a stored value
NAN16 = 0x7E01              # fp16 NaN bit pattern of the words no kernel may write
NAN32 = 0x7FC01234          # fp32 NaN bit pattern
PAD_ROWS = 16               # pixel rows past the map in every buffer
DGRAD = {0: "none", 1: "small", 2: "wgmma", 3: "simt"}
WGRAD = {1: "small", 2: "mma.sync", 3: "wgmma direct", 4: "wgmma packed"}

# Limits, calibrated on an H100 80GB HBM3 (700 W power limit) over the cases and the census below: each is about 4x the worst value
# observed there, which fp32 accumulation order explains (sums of up to ~10^6 products; no route needs more).
#   data gradient (fp16 / fp32 grad(in) = prior + gradient): max over elements of (|ours - ref| - U16 |ref|) / max |ref|, i.e. what is
#     left after the one rounding of the stored sum.  Worst: small 7.2e-7, wgmma 2.2e-6 (census), simt 5.9e-8.
#   weight gradient (fp32 dW = prior + gradient): relative Frobenius error and max |err| / max |ref| of the gradient.  Worst (Frobenius,
#     max): small 5.8e-7, 1.3e-6; mma.sync 2.7e-6, 2.9e-6; wgmma direct 9.6e-7, 1.2e-6; wgmma packed 7.3e-6, 7.8e-6 (census: the long
#     row slabs of the 512 x 1024 plans).
#   bias gradient: max |err| / max |ref| of the gradient.  Worst: from fp32 dY 6.0e-7, from fp16 dY 2.4e-7.
LIMIT_DGRAD = {"small": 3e-6, "wgmma": 1e-5, "simt": 2.5e-7}
LIMIT_WGRAD = {"small": (2.5e-6, 5e-6), "mma.sync": (1.2e-5, 1.2e-5), "wgmma direct": (4e-6, 5e-6), "wgmma packed": (3e-5, 3e-5)}
LIMIT_BIAS = {"fp32": 2.5e-6, "fp16": 1e-6}

WORST = defaultdict(float)      # measure -> worst value seen in this session (printed next to its limit)


def ceil16(n):
    return (n + 15) // 16 * 16


# ---- buffers -----------------------------------------------------------------------------------------------------------------------
def sentinel_buffer(B, H, W, ctot, dtype):
    """an NHWC buffer of B*H*W pixels + PAD_ROWS more, every word a NaN; returns (whole flat buffer, (B,H,W,ctot) view of the map)"""
    if dtype == torch.float16:
        flat = torch.full((B * H * W + PAD_ROWS, ctot), NAN16, dtype=torch.int16, device="cuda").view(torch.float16)
    else:
        flat = torch.full((B * H * W + PAD_ROWS, ctot), NAN32, dtype=torch.int32, device="cuda").view(torch.float32)
    return flat, flat[:B * H * W].view(B, H, W, ctot)


def put(view, off, vals_nchw, width):
    """channels [off, off + width) of the view = the values (NCHW, C <= width), zero above C"""
    C = vals_nchw.shape[1]
    view[..., off:off + C] = vals_nchw.permute(0, 2, 3, 1).to(view.dtype)
    if width > C:
        view[..., off + C:off + width] = 0


def get(view, off, C):
    return view[..., off:off + C].permute(0, 3, 1, 2).double()


def untouched(flat, view, off, width):
    """every word of the buffer outside channels [off, off + width) of the map still holds the sentinel"""
    bits = flat.view(torch.int16 if flat.dtype == torch.float16 else torch.int32)
    s = NAN16 if flat.dtype == torch.float16 else NAN32
    npix = view.shape[0] * view.shape[1] * view.shape[2]
    return bool((bits[:npix, :off] == s).all() and (bits[:npix, off + width:] == s).all() and (bits[npix:] == s).all())


# ---- one run of the entry and its fp64 reference ---------------------------------------------------------------------------------
def run(B, H, W, ci, co, k=1, s=1, d=1, x_dt=torch.float16, dy_dt=torch.float16, dgrad=True, bias=False, x_off=0, dy_off=0, gin_off=0,
        x_ctot=None, dy_ctot=None, route=0, seed=0, mutant=None):
    """runs ops.conv_backward once on random data and returns (info, errors, sentinels intact); errors = {measure: value}"""
    from multiyolov5_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(seed)
    pad = d * (k // 2)
    Ho, Wo = (H + 2 * pad - d * (k - 1) - 1) // s + 1, (W + 2 * pad - d * (k - 1) - 1) // s + 1
    xc, dyc = ceil16(ci), (ceil16(co) if dy_dt == torch.float32 else co)
    x_ctot = x_ctot or max(x_off, gin_off) + xc + 8
    dy_ctot = dy_ctot or dy_off + dyc + 8
    xflat, xv = sentinel_buffer(B, H, W, x_ctot, x_dt)
    dflat, dv = sentinel_buffer(B, Ho, Wo, dy_ctot, dy_dt)
    x = torch.randn((B, ci, H, W), generator=g, device="cuda").to(x_dt)
    dy = torch.randn((B, co, Ho, Wo), generator=g, device="cuda").to(dy_dt)
    w = torch.randn((co, ci, k, k), generator=g, device="cuda") / (co * k * k) ** 0.5
    put(xv, x_off, x, xc)
    put(dv, dy_off, dy, dyc)
    x0, d0 = xflat.clone(), dflat.clone()

    # priors of the accumulated gradients, at the gradients' own scale (w is scaled so that grad(in) is about N(0, 1))
    gflat = gv = None
    if dgrad:
        gflat, gv = sentinel_buffer(B, H, W, x_ctot, x_dt)
        prior = torch.randn((B, ci, H, W), generator=g, device="cuda").to(x_dt)
        put(gv, gin_off, prior, ci)
        nan = torch.tensor([NAN16 if x_dt == F16 else NAN32], dtype=torch.int16 if x_dt == F16 else torch.int32, device="cuda")
        gv[..., gin_off + ci:gin_off + xc] = nan.view(x_dt)
    npix = B * Ho * Wo
    w_prior = torch.randn((co, ci, k, k), generator=g, device="cuda") * npix ** 0.5 / 2
    dW = w_prior.clone()
    db_prior = torch.randn((co,), generator=g, device="cuda") * npix ** 0.5 if bias else None
    db = db_prior.clone() if bias else None

    info = ops.conv_backward(xv, w, dv, dW, gin=gv, dbias=db, x_off=x_off, dy_off=dy_off, gin_off=gin_off, stride=s, dil=d, route=route)
    torch.cuda.synchronize()

    # fp64 gradients of the values the kernels of the route taken read: the small route reads the fp32 masters and dY as stored; the
    # tensor-core and CUDA-core routes the fp16 weight pack and fp16 dY (an fp32 head gradient cast once); the bias always dY as stored
    x64, dy64 = x.double(), dy.double()
    dy_mm = dy64 if info[1] == 1 or mutant == "head_unrounded" else dy.half().double()
    gx = gw = gb = None
    if dgrad:
        xr = x64.clone().requires_grad_(True)
        w_dg = w.double() if info[0] == 1 else w.half().double()
        if mutant == "unflipped":
            w_dg = w_dg.flip(2, 3)
        F.conv2d(xr, w_dg, None, s, pad, d).backward(dy64 if info[0] == 1 else dy_mm)
        gx = xr.grad
    wr = torch.zeros((co, ci, k, k), dtype=torch.float64, device="cuda", requires_grad=True)
    F.conv2d(x64, wr, None, s, pad, d).backward(dy_mm)
    gw = wr.grad
    if mutant == "row_missing":
        gw = gw.clone()
        gw[:, :, 0, :] = 0
    if bias:
        gb = (dy.half().double() if mutant == "bias_from_fp16" else dy64).sum((0, 2, 3))

    err = {}
    ok = bool(torch.equal(xflat.view(torch.uint8), x0.view(torch.uint8)) and torch.equal(dflat.view(torch.uint8), d0.view(torch.uint8)))
    if dgrad:
        ref = (gx if mutant == "prior_dropped" else prior.double() + gx)
        ours = get(gv, gin_off, ci)
        e = ((ours - ref).abs() - U16 * ref.abs()).clamp_min(0).max() / ref.abs().max()
        err["dgrad"] = float(e)
        ok = ok and untouched(gflat, gv, gin_off, ci)
    ew = dW.double() - w_prior.double() - gw
    err["wgrad_frob"] = float(ew.norm() / gw.norm())
    err["wgrad_max"] = float(ew.abs().max() / gw.abs().max())
    if bias:
        err["bias"] = float((db.double() - db_prior.double() - gb).abs().max() / gb.abs().max())
    return info, err, ok


def over_limit(info, err):
    """each measured error over its route's limit (NaN stays NaN: a NaN read fails)"""
    r = {}
    if "dgrad" in err:
        r["dgrad"] = err["dgrad"] / LIMIT_DGRAD[DGRAD[info[0]]]
    lf, lm = LIMIT_WGRAD[WGRAD[info[1]]]
    r["wgrad"] = max(err["wgrad_frob"] / lf, err["wgrad_max"] / lm) if err["wgrad_frob"] == err["wgrad_frob"] else float("nan")
    if "bias" in err:
        r["bias"] = err["bias"] / LIMIT_BIAS["fp32" if info[2] == 1 else "fp16"]
    return r


def record(info, err):
    if "dgrad" in err:
        key = f"dgrad {DGRAD[info[0]]}"
        WORST[key] = max(WORST[key], err["dgrad"])
    for m in ("wgrad_frob", "wgrad_max"):
        key = f"{m} {WGRAD[info[1]]}"
        WORST[key] = max(WORST[key], err[m])
    if "bias" in err:
        key = f"bias {'fp32' if info[2] == 1 else 'fp16'}"
        WORST[key] = max(WORST[key], err["bias"])


def limit_of(key):
    kind, route = key.split(" ", 1)
    if kind == "dgrad":
        return LIMIT_DGRAD[route]
    if kind == "bias":
        return LIMIT_BIAS[route]
    return LIMIT_WGRAD[route][0 if kind == "wgrad_frob" else 1]


def print_worst():
    print("\nworst error per route so far (limit):")
    for key in sorted(WORST):
        print(f"  {key:<26} {WORST[key]:.2e}  ({limit_of(key):.1e})")


def describe(info):
    s = f"dgrad {DGRAD[info[0]]}"
    if info[0] == 2:
        s += f" kc={info[3]} BN={info[4]} ctas/SM={info[5]} resident={info[6]} strip={info[7]} n_tiles={info[13]} n_pad={info[14]}"
    s += f" | wgrad {WGRAD[info[1]]}"
    if info[1] >= 3:
        s += f" Kc={info[8]} N={info[9]} slabs={info[10]}x{info[11]} rows of {info[12]}"
    if info[2]:
        s += f" | bias from {'fp32' if info[2] == 1 else 'fp16'}"
    return s


def check(name, info, err, ok):
    """the stored-result checks shared by the cases and the census: errors within the route's limits, sentinels intact, and the wgmma
    data gradient's N tiles inside its padded pack"""
    record(info, err)
    over = over_limit(info, err)
    fails = [f"{name}: {k} at {v:.2f}x its limit ({err})" for k, v in over.items() if not v <= 1.0]
    if not ok:
        fails.append(f"{name}: a word outside the views was written")
    if info[0] == 2 and not info[13] * info[4] <= info[14]:
        fails.append(f"{name}: data-gradient N tiles {info[13]} x {info[4]} past the pack's {info[14]} channels")
    return fails


# ---- cases: the edges of every route ---------------------------------------------------------------------------------------------
F16, F32 = torch.float16, torch.float32
OFFS = (0, 8, 24)
CASES = {
    # id: (geometry and dtypes, expected info slots {slot: value})
    # wgmma weight gradient: Kc 64 / 32 / 16, N 16 / 32 / 64 / 128, Co <= 64 and 96, direct and packed, stride 2, dilation, slabs
    "wg_kc64_n128_direct": (dict(B=2, H=32, W=64, ci=128, co=64), {0: 2, 1: 3, 8: 64, 9: 128, 3: 64, 5: 1, 7: 0}),
    "wg_kc32_n64_co96": (dict(B=2, H=24, W=96, ci=64, co=96, k=3), {0: 2, 1: 4, 8: 32, 9: 64, 3: 32}),
    "wg_kc16_n16_ci12": (dict(B=2, H=40, W=80, ci=12, co=32, k=3, dgrad=False), {0: 0, 1: 4, 8: 16, 9: 16}),
    "wg_n16_direct": (dict(B=2, H=16, W=64, ci=16, co=64), {1: 3, 8: 64, 9: 16}),
    "wg_n32_s2": (dict(B=2, H=64, W=128, ci=32, co=64, k=3, s=2), {0: 2, 1: 4, 8: 64, 9: 32}),
    "wg_d2": (dict(B=1, H=48, W=64, ci=64, co=64, k=3, d=2), {0: 2, 1: 4, 9: 64}),
    "wg_d3_ragged_slabs": (dict(B=1, H=37, W=64, ci=64, co=64, k=3, d=3), {0: 2, 1: 4, 8: 64}),
    "wg_d6_co128": (dict(B=2, H=30, W=64, ci=128, co=128, k=3, d=6), {0: 2, 1: 4, 9: 64}),
    "wg_npix_2048": (dict(B=1, H=32, W=64, ci=64, co=32), {1: 3}),
    "wg_co96_n128": (dict(B=2, H=16, W=128, ci=256, co=96), {1: 3, 9: 128, 3: 32}),
    # mma.sync weight gradient: ci 48 / 96, Co % 64 != 0, Wo % 16 != 0 with B Ho Wo % 32 != 0, stride 2, dilation, x at c_off 8
    "mma_npix_2032": (dict(B=1, H=127, W=16, ci=64, co=32), {1: 2, 0: 2}),
    "mma_ci48_co96": (dict(B=2, H=40, W=80, ci=48, co=96, k=3), {1: 2, 0: 2, 3: 32, 4: 48}),
    "mma_ci96_ragged": (dict(B=2, H=23, W=46, ci=96, co=80), {1: 2, 0: 2, 3: 16, 4: 96}),
    "mma_s2_slice": (dict(B=2, H=46, W=92, ci=64, co=128, k=3, s=2, x_off=8, gin_off=24), {1: 2, 0: 2, 3: 64}),
    "mma_ci48_d3": (dict(B=2, H=30, W=60, ci=48, co=48, k=3, d=3), {1: 2, 0: 2, 3: 16}),
    "mma_forced": (dict(B=2, H=32, W=64, ci=128, co=64, route=2), {1: 2, 0: 2}),
    # small route (both gradients): fp32 x, PPM bins, the B Ho Wo <= 1024 and Ho Wo < 128 thresholds, 3x3 on a 2x2 map
    "small_ffm_fc_f32": (dict(B=4, H=1, W=1, ci=256, co=256, x_dt=F32, dy_dt=F32, bias=True), {0: 1, 1: 1, 2: 1}),
    "small_ppm1_f32": (dict(B=4, H=1, W=1, ci=512, co=128, x_dt=F32), {0: 1, 1: 1}),
    "small_ppm2": (dict(B=4, H=2, W=2, ci=512, co=128), {0: 1, 1: 1}),
    "small_ppm3_f32": (dict(B=4, H=3, W=3, ci=512, co=128, x_dt=F32), {0: 1, 1: 1}),
    "small_ppm6": (dict(B=4, H=6, W=6, ci=512, co=128), {0: 1, 1: 1}),
    "small_npix_1024": (dict(B=8, H=8, W=16, ci=64, co=64, k=3), {0: 1, 1: 1}),
    "tc_npix_1025": (dict(B=1, H=25, W=41, ci=64, co=64, k=3), {0: 2, 1: 2}),
    "small_hw_127": (dict(B=9, H=1, W=127, ci=32, co=32, k=3), {0: 1, 1: 1}),
    "tc_hw_128": (dict(B=9, H=8, W=16, ci=32, co=32, k=3), {0: 2, 1: 2, 3: 32}),
    "small_3x3_on_2x2": (dict(B=4, H=2, W=2, ci=64, co=64, k=3), {0: 1, 1: 1}),
    "small_head_f32": (dict(B=2, H=8, W=16, ci=128, co=57, dy_dt=F32, bias=True), {0: 1, 1: 1, 2: 1}),
    # wgmma data gradient: BN from ci > 128, two CTAs per SM with strip mode, fp32 dY at stride 2 (cast, then zero-stuffed), dilation 9
    "dg_ci192": (dict(B=2, H=32, W=64, ci=192, co=64), {0: 2, 3: 64, 4: 96}),
    "dg_spp_cv2": (dict(B=4, H=16, W=32, ci=1024, co=512), {0: 2, 3: 64, 4: 128, 13: 8}),
    "dg_two_cta_strip": (dict(B=4, H=128, W=256, ci=64, co=64, k=3), {0: 2, 5: 2, 7: 1}),
    "dg_s2_f32_dy": (dict(B=2, H=64, W=128, ci=64, co=45, k=3, s=2, dy_dt=F32, bias=True), {0: 2, 1: 4, 2: 1, 3: 16}),
    "dg_d9": (dict(B=2, H=40, W=80, ci=128, co=48, k=3, d=9), {0: 2, 1: 4, 3: 16, 8: 16}),
    "dg_ragged_map": (dict(B=2, H=37, W=75, ci=64, co=64, k=3), {0: 2, 1: 2}),
    # CUDA-core data gradient: forced, and ci % 16 != 0 (the residual of the wgmma kernel needs Co % 16 == 0)
    "simt_forced": (dict(B=1, H=48, W=64, ci=64, co=64, k=3, d=2, route=1), {0: 3, 1: 4}),
    "simt_ci24": (dict(B=2, H=32, W=64, ci=24, co=64, k=3), {0: 3, 1: 4, 9: 32}),
    # bias gradient: Detect heads at nc 10 and 14 (fp32 dY, Co 45 / 57), fp16 dY in a view wider than Co
    "bias_head45": (dict(B=2, H=32, W=64, ci=128, co=45, dy_dt=F32, bias=True), {0: 2, 1: 3, 2: 1, 3: 16}),
    "bias_head57": (dict(B=2, H=16, W=64, ci=256, co=57, dy_dt=F32, bias=True), {0: 2, 1: 3, 2: 1}),
    "bias_f16_slice": (dict(B=2, H=32, W=64, ci=64, co=64, bias=True, dy_off=24, dy_ctot=128), {2: 2}),
    # wgmma weight gradient of layer 0 at the --multi-scale widths 64 n + 32 (Wo = 272): steps of 16 output pixels, and with 16 input
    # channels such a step is 512 bytes of X per tap, less than its 1024-byte aligned slot
    "wg_ms_wo272_s1": (dict(B=2, H=16, W=272, ci=16, co=32, k=3, dgrad=False), {0: 0, 1: 4, 8: 16}),
    "wg_ms_wo272_s2": (dict(B=2, H=32, W=544, ci=16, co=32, k=3, s=2, dgrad=False), {0: 0, 1: 4, 8: 16}),
}

# (B, H, W, ci, co, k, stride, dil): weight gradients on both tensor-core kernels, each shape at 2048 or more output pixels
WGRAD_SHAPES = [
    (2, 32, 64, 64, 64, 1, 1, 1), (2, 32, 64, 128, 256, 1, 1, 1), (1, 64, 128, 64, 128, 3, 1, 1), (2, 32, 32, 128, 64, 3, 1, 1),
    (2, 64, 64, 64, 128, 3, 2, 1), (1, 32, 64, 64, 64, 3, 1, 2), (1, 32, 64, 192, 48, 1, 1, 1), (2, 16, 128, 256, 256, 3, 1, 1),
    (1, 48, 80, 64, 96, 3, 1, 3), (2, 64, 128, 32, 64, 3, 2, 1), (1, 64, 128, 32, 32, 3, 1, 1), (1, 64, 64, 16, 32, 3, 1, 1),
    (2, 32, 64, 32, 32, 1, 1, 1),
]


def wgrad_cases():
    """WGRAD_SHAPES on the mma.sync kernel (route 2: MYOLO_CONV_BWD_NO_WGRAD_TC) and on the wgmma kernel, which accumulates straight into
    dW for a 1x1 conv whose channels need no padding and through its packed buffer otherwise (conv_wgrad_packed_bytes)"""
    out = {}
    for i, (B, H, W, ci, co, k, s, d) in enumerate(WGRAD_SHAPES):
        geo = dict(B=B, H=H, W=W, ci=ci, co=co, k=k, s=s, d=d, dgrad=False)
        out[f"wgrad_mma_w{i}"] = (dict(geo, route=2), {0: 0, 1: 2})
        out[f"wgrad_wgmma_w{i}"] = (geo, {0: 0, 1: 3 if k == 1 and ci % 16 == 0 else 4})
    return out


CASES.update(wgrad_cases())


def case_args(name):
    geo, _ = CASES[name]
    i = list(CASES).index(name)
    a = dict(x_off=OFFS[i % 3], gin_off=OFFS[(i + 1) % 3], dy_off=OFFS[(i + 2) % 3], seed=i)
    a.update(geo)
    return a


@pytest.mark.parametrize("name", list(CASES))
def test_conv_backward_matches_fp64(name):
    """one conv's data, weight and bias gradients on the route the case was built for, accumulated into priors, through channel slices"""
    a = case_args(name)
    info, err, ok = run(**a)
    print(f"\n[{name}] {describe(info)}\n[{name}] " + "  ".join(f"{k} {v:.2e}" for k, v in err.items()))
    want = CASES[name][1]
    got = {s: info[s] for s in want}
    assert got == want, f"route: expected slots {want}, got {got} ({describe(info)})"
    if name == "wg_d3_ragged_slabs":
        assert info[12] % info[11] != 0, "the last row slab should be short"
    if name == "wg_npix_2048":
        assert a["B"] * a["H"] * a["W"] == 2048
    fails = check(name, info, err, ok)
    print_worst()
    assert not fails, "\n".join(fails)


# ---- census: every conv op of the train plans ------------------------------------------------------------------------------------
CENSUS_SHAPES = [(4, 512, 1024), (2, 416, 736), (2, 544, 1088)]   # the bench slice, a --rect shape, a --multi-scale size 64 n + 32
CENSUS_MODELS = {"s_psp": "yolov5s_city_seg.yaml", "m_lab": "yolov5m_city_seg_lab.yaml"}


def census_ops(yml, B, H, W):
    """(op index, output width, geometry kwargs of run()) for every conv op of the train plan"""
    from multiyolov5_b200 import _lib as L
    from multiyolov5_b200.models.yolo import Model
    from multiyolov5_b200.plan import build_plan
    pb = build_plan(Model(yml), B, H, W, train=True)
    focus = {o.out.buf.id for o in pb.ops if o.kind == L.OP_INPUT_FOCUS}
    dt = {L.F16: torch.float16, L.F32: torch.float32}
    out = []
    for i, o in enumerate(pb.ops):
        if o.kind != L.OP_CONV:
            continue
        conv = pb.slots[o.slot].conv
        ci, co = conv.in_channels, conv.out_channels
        dy_dt = dt[o.out.buf.dtype]
        assert o.in_.c == ceil16(ci) and o.out.c == (ceil16(co) if dy_dt == torch.float32 else co), (i, o.in_.c, o.out.c, ci, co)
        out.append((i, o.out.w, dict(B=B, H=o.in_.h, W=o.in_.w, ci=ci, co=co, k=o.k, s=o.stride, d=o.dil, x_dt=dt[o.in_.buf.dtype], dy_dt=dy_dt,
                            dgrad=o.in_.buf.id not in focus, bias=conv.bias is not None, x_off=o.in_.c_off, x_ctot=o.in_.buf.c,
                            gin_off=o.in_.c_off, dy_off=o.out.c_off, dy_ctot=o.out.buf.c, seed=i)))
    return out


def test_conv_backward_census_of_the_train_plans():
    """every conv op of the s_psp and m_lab train plans at the bench slice, a --rect shape and a --multi-scale size: the entry at the op's
    geometry and slice layout, against fp64; prints the routes per plan and asserts that the census reaches the edges it claims"""
    fails, total = [], defaultdict(int)
    for tag, yml in CENSUS_MODELS.items():
        for B, H, W in CENSUS_SHAPES:
            count = defaultdict(int)
            for i, wo, a in census_ops(yml, B, H, W):
                info, err, ok = run(**a)
                fails += check(f"{tag} {H}x{W} op {i}", info, err, ok)
                count[f"dgrad {DGRAD[info[0]]}"] += 1
                count[f"wgrad {WGRAD[info[1]]}"] += 1
                if info[0] == 2:
                    count[f"dgrad wgmma kc={info[3]}"] += 1
                    count[f"dgrad wgmma {info[5]} cta/SM"] += 1
                if info[1] >= 3:
                    count[f"wgrad wgmma Kc={info[8]}"] += 1
                if info[1] == 2 and wo % 16 != 0:
                    count["wgrad mma.sync ragged width"] += 1
                if info[2]:
                    count[f"bias from {'fp32' if info[2] == 1 else 'fp16'}"] += 1
                count["ops"] += 1
            print(f"\n[{tag} {B}x{H}x{W}] " + ", ".join(f"{k}: {v}" for k, v in sorted(count.items())))
            for k, v in count.items():
                total[k] += v
    print_worst()
    assert not fails, "\n".join(fails[:30])
    assert total["wgrad mma.sync ragged width"] >= 1
    assert total["wgrad wgmma Kc=16"] >= 1
    assert total["dgrad wgmma 2 cta/SM"] >= 1


# ---- sensitivity ---------------------------------------------------------------------------------------------------------------
MUTANTS = {  # wrong reference: (case it runs on, the measure it must push 10x past its limit)
    "unflipped": ("wg_kc32_n64_co96", "dgrad"),           # the 3x3 kernel not flipped in the data gradient
    "head_unrounded": ("bias_head45", "wgrad"),           # the fp32 head gradient not rounded to fp16 before the tensor cores
    "prior_dropped": ("mma_ci48_co96", "dgrad"),          # grad(in) without its prior
    "row_missing": ("wg_kc32_n64_co96", "wgrad"),         # one filter row missing from the weight gradient
    "bias_from_fp16": ("bias_head45", "bias"),            # the bias summed from the fp16 cast of an fp32 head gradient
}


def test_conv_backward_limits_catch_wrong_references():
    """the limits discriminate: each deliberately wrong reference misses its limit by at least 10x"""
    print()
    for mutant, (case, measure) in MUTANTS.items():
        info, err, _ = run(**case_args(case), mutant=mutant)
        over = over_limit(info, err)[measure]
        print(f"mutant {mutant:<15} on {case:<20}: {measure} at {over:.0f}x its limit")
        assert over >= 10, (mutant, over, err)
