"""GPU: the forward of one conv on its own, through the plan's own routing and launches (ops.conv_forward -> csrc/plan.cu
conv_forward_views, the function the plan's prepare_conv calls), against F.conv2d in fp64 on the values the kernels actually read:
  - the fp16 input (or the fp32 input of the CUDA-core kernel);
  - the fp16 weight pack: with BatchNorm, the pack's fold restated in fp32 in pack_weights_kernel's operation order (w * (gamma / sqrt(var
    + eps)); beta - gamma mean / sqrt(var + eps) + bias gamma / sqrt(var + eps); IEEE sqrt and division on both sides), then rounded to
    fp16; without it, weights that fp16 holds exactly;
  - the fp32 bias; then the exact activation in fp64 and the residual added before the single rounding of the stored output.
Every view is a channel slice of a wider buffer, and every word outside the slices (other channels, the padding channels of an fp32 head
buffer, pixel rows past the map) holds an fp16 / fp32 NaN that must survive; the input and a separate residual buffer must come back
unchanged.  Each case asserts the route it was built for, so a silent fall-back fails; across the cases every instantiation of
conv_tc_kernel<KC, BN, RES, CTAS_PER_SM> that conv_tc_launch can dispatch runs.  A case may launch a twin on the same inputs that must
give the same output bit for bit: the streamed-weight layout with one A box per tap (path 3: the same MMAs in the same K order, so any
difference is a layout or synchronisation bug of the resident weights, the strip or the second CTA), or the residual aliasing the
output instead of a separate buffer.  The census runs the entry at the exact geometry and slice layout of every conv op of two inference
plans at two shapes and two train plans, and asserts that it routes and tiles each one as the plan does; one more test pins which convs
of the s/PSP forward keep their weights resident and take the strip."""
from collections import defaultdict

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

U16 = 2.0 ** -11            # fp16 unit roundoff: one rounding of a stored value
NAN16 = 0x7E01              # fp16 NaN bit pattern of the words no kernel may write
NAN32 = 0x7FC01234          # fp32 NaN bit pattern
PAD_PIX = 256               # pixels past the map in every buffer, beyond 16 map rows (the tallest tile is 8 x 16)
F16, F32 = torch.float16, torch.float32
NONE, SILU, SIGMOID = 0, 1, 2

# Limits, the metric of test_gpu_infer_layers.py: fp16 outputs max over elements of (|ours - ref| - U16 |ref|) / max |ref| (what is left
# after the one rounding of the stored value), fp32 outputs max |ours - ref| / max |ref|.  Calibrated on an H100 80GB HBM3 (700 W power
# limit) over the cases and the census below, each about 4x the worst value observed there.  Worst: fp16 wgmma 1.5e-5 (census: a 3x3
# 512-channel layer of m_lab at 16 x 512 x 1024, where the tensor cores' fp32 sums run over K = 4608 products of random weights), fp16
# simt 3.4e-6, fp32 wgmma 1.2e-6, fp32 simt 2.5e-7.
LIMIT = {"fp16": 6e-5, "fp32": 5e-6}

WORST = defaultdict(float)      # "dtype route" -> worst value seen in this session


def ceil16(n):
    return (n + 15) // 16 * 16


def out_hw(H, W, k, s, d):
    pad = d * (k // 2)
    return (H + 2 * pad - d * (k - 1) - 1) // s + 1, (W + 2 * pad - d * (k - 1) - 1) // s + 1


# ---- buffers -----------------------------------------------------------------------------------------------------------------------
def sentinel_buffer(B, H, W, ctot, dtype):
    """an NHWC buffer of B*H*W pixels + 16*W + PAD_PIX more, every word a NaN; returns (whole flat buffer, (B,H,W,ctot) view of the map)"""
    n = B * H * W + 16 * W + PAD_PIX
    if dtype == F16:
        flat = torch.full((n, ctot), NAN16, dtype=torch.int16, device="cuda").view(F16)
    else:
        flat = torch.full((n, ctot), NAN32, dtype=torch.int32, device="cuda").view(F32)
    return flat, flat[:B * H * W].view(B, H, W, ctot)


def untouched(flat, npix, off, width):
    """every word of the buffer outside channels [off, off + width) of the map still holds the sentinel"""
    bits = flat.view(torch.int16 if flat.dtype == F16 else torch.int32)
    s = NAN16 if flat.dtype == F16 else NAN32
    return bool((bits[:npix, :off] == s).all() and (bits[:npix, off + width:] == s).all() and (bits[npix:] == s).all())


def same_bits(a, b):
    return torch.equal(a.view(torch.uint8), b.view(torch.uint8))


# ---- the reference ---------------------------------------------------------------------------------------------------------------------
def pack_ref(w, bn, bias, eps):
    """the fp16 weights and fp32 bias of pack_weights_kernel (csrc/conv_simt.cu), restated in fp32 in its operation order"""
    w = w.cpu()
    co = w.shape[0]
    if bn is None:
        return w.half(), (bias.cpu() if bias is not None else torch.zeros(co))
    g, b, m, v = [t.cpu() for t in bn]
    sd = torch.sqrt(v + torch.tensor(eps, dtype=F32))
    wp = (w * (g / sd).view(-1, 1, 1, 1)).half()
    bp = b - (g * m) / sd
    if bias is not None:
        bp = bp + (bias.cpu() * g) / sd
    return wp, bp


def act64(z, a):
    return z * torch.sigmoid(z) if a == SILU else (torch.sigmoid(z) if a == SIGMOID else z)


def conv64(x64, wp, bp, k, s, d, act):
    """act(conv(x, wp) + bp) in fp64 on NCHW x64"""
    return act64(F.conv2d(x64, wp.double().cuda(), bp.double().cuda(), s, d * (k // 2), d), act)


# ---- one run of the entry and its fp64 reference ---------------------------------------------------------------------------------
def run(B, H, W, ci, co, k=1, s=1, d=1, x_dt=F16, y_dt=F16, act=SILU, res=None, bn=True, bias=True, x_off=0, y_off=0, r_off=0,
        x_ctot=None, y_ctot=None, r_ctot=None, path=0, seed=0, images=None, res_cancel=False, mutant=None, twin=None):
    """runs ops.conv_forward once on random data; returns (info, {dtype: error, "change": mutant's relative change}, sentinels intact,
    twin).  res: None, "sep" (own buffer) or "alias" (the output slice itself); images: the images compared (default all).  twin: None,
    "path3" (the same inputs again on path 3) or "alias" (again on the same path, with res "sep", the residual in the output slice); twin
    is then (the twin's info, both output buffers bit-identical), else None"""
    from multiyolov5_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(seed)
    Ho, Wo = out_hw(H, W, k, s, d)
    xc = ceil16(ci)
    x_ctot = x_ctot or x_off + xc + 8
    y_ctot = y_ctot or y_off + (ceil16(co) if y_dt == F32 else co) + 8
    xflat, xv = sentinel_buffer(B, H, W, x_ctot, x_dt)
    yflat, yv = sentinel_buffer(B, Ho, Wo, y_ctot, y_dt)
    xv[..., x_off:x_off + ci] = torch.randn((B, H, W, ci), generator=g, device="cuda").to(x_dt)
    xv[..., x_off + ci:x_off + xc] = 0
    w = torch.randn((co, ci, k, k), generator=g, device="cuda") / (ci * k * k) ** 0.5
    bnp = None
    if bn:
        bnp = [torch.rand((co,), generator=g, device="cuda") * 0.4 + 0.8, torch.randn((co,), generator=g, device="cuda") * 0.1,
               torch.randn((co,), generator=g, device="cuda") * 0.1, torch.rand((co,), generator=g, device="cuda") + 0.5]
    else:
        w = w.half().float()
    bvec = torch.randn((co,), generator=g, device="cuda") * 0.1 if bias else None
    eps = 1e-3
    wp, bp = pack_ref(w, bnp, bvec, eps)
    imgs = list(range(B)) if images is None else images
    x64 = xv[imgs, :, :, x_off:x_off + ci].permute(0, 3, 1, 2).double()

    rflat = rbuf = None
    if res is not None:
        rv_vals = torch.randn((B, Ho, Wo, co), generator=g, device="cuda")
        if res_cancel:          # the residual cancels the conv's output up to a tenth: the output's rounding is then what matters
            rv_vals = -conv64(x64, wp, bp, k, s, d, act).permute(0, 2, 3, 1).float() + 0.1 * rv_vals
        if res == "alias":
            r_off, r_ctot, rbuf = y_off, y_ctot, yv
            rbuf[..., r_off:r_off + co] = rv_vals.half()
        else:
            r_ctot = r_ctot or r_off + co + 8
            rflat, rbuf = sentinel_buffer(B, Ho, Wo, r_ctot, F16)
            rbuf[..., r_off:r_off + co] = rv_vals.half()
        r64 = rbuf[imgs, :, :, r_off:r_off + co].permute(0, 3, 1, 2).double()
    x0 = xflat.clone()
    r0 = rflat.clone() if rflat is not None else None

    info = ops.conv_forward(xv, w, yv, bn=bnp, bias=bvec, residual=rbuf, x_off=x_off, y_off=y_off, res_off=r_off, stride=s, dil=d, act=act,
                            path=path, eps=eps)
    if twin is not None:
        assert twin == "path3" or res == "sep", (twin, res)
        yflat2, yv2 = sentinel_buffer(B, Ho, Wo, y_ctot, y_dt)
        rbuf2, r_off2 = rbuf, r_off
        if res == "alias" or twin == "alias":
            yv2[..., y_off:y_off + co] = rv_vals.half()
            rbuf2, r_off2 = yv2, y_off
        twin_info = ops.conv_forward(xv, w, yv2, bn=bnp, bias=bvec, residual=rbuf2, x_off=x_off, y_off=y_off, res_off=r_off2, stride=s,
                                     dil=d, act=act, path=3 if twin == "path3" else path, eps=eps)
    torch.cuda.synchronize()

    ok = same_bits(xflat, x0) and (r0 is None or same_bits(rflat, r0)) and untouched(yflat, B * Ho * Wo, y_off, co)
    twin = None if twin is None else (twin_info, same_bits(yflat, yflat2))
    with torch.no_grad():
        ref = conv64(x64, wp, bp, k, s, d, act)
        if res is not None:
            ref = ref + r64
        ours = yv[imgs, :, :, y_off:y_off + co].permute(0, 3, 1, 2).double()
        err = {}
        if mutant is not None:
            bad = wrong_reference(mutant, x64, w, bnp, bvec, eps, wp, bp, k, s, d, act, r64 if res is not None else None)
            err["change"] = float((bad - ref).norm() / ref.norm())
            ref = bad
        scale = float(ref.abs().max())
        if y_dt == F16:
            err["fp16"] = float(((ours - ref).abs() - U16 * ref.abs()).clamp_min(0).max()) / scale
        else:
            err["fp32"] = float((ours - ref).abs().max()) / scale
    return info, err, ok, twin


def wrong_reference(mutant, x64, w, bnp, bvec, eps, wp, bp, k, s, d, act, r64):
    """the reference restated wrongly on purpose (test_conv_forward_limits_catch_wrong_references)"""
    if mutant == "bf16":                     # the folded weights rounded to bf16 instead of fp16
        wf = w.cpu() if bnp is None else (w.cpu() * (bnp[0].cpu() / torch.sqrt(bnp[3].cpu() + torch.tensor(eps))).view(-1, 1, 1, 1))
        wp = wf.bfloat16()
    elif mutant == "tap":                    # one filter tap's weights scaled by 1 + 2^-9
        wp = wp.double().clone()
        wp[:, :, 0, 0] *= 1 + 2.0 ** -9
    elif mutant == "bias":                   # one channel's bias off by 1e-3 max |bias|
        bp = bp.clone()
        bp[bp.shape[0] // 2] += 1e-3 * float(bp.abs().max())
    y = None
    if mutant == "replicate":                # the right border padded with the edge column instead of zeros
        p = d * (k // 2)
        xp = F.pad(F.pad(x64, (0, p, 0, 0), mode="replicate"), (p, 0, p, p))
        y = act64(F.conv2d(xp, wp.double().cuda(), bp.double().cuda(), s, 0, d), act)
    if y is None:
        y = act64(F.conv2d(x64, wp.double().cuda(), bp.double().cuda(), s, d * (k // 2), d), act)
    if r64 is None:
        return y
    if mutant == "rounded_before_residual":  # the conv's output rounded to fp16 before the residual is added
        return y.half().double() + r64
    return y + r64


def record(info, err):
    for m in ("fp16", "fp32"):
        if m in err:
            key = f"{m} {'wgmma' if info[0] else 'simt'}"
            WORST[key] = max(WORST[key], err[m])


def print_worst():
    print("\nworst error per output type and route so far (limit):")
    for key in sorted(WORST):
        print(f"  {key:<12} {WORST[key]:.2e}  ({LIMIT[key.split()[0]]:.0e})")


def describe(info):
    if not info[0]:
        return "simt"
    return (f"wgmma kc={info[10]} BN={info[3]} ctas/SM={info[11]} resident={info[6]} strip={info[5]} stages={info[4]} grid={info[1]} "
            f"tiles={info[8]} n_tiles={info[9]} smem={info[2]}")


def check(name, info, err, ok):
    """the stored-result checks shared by the cases and the census"""
    record(info, err)
    fails = [f"{name}: {m} error {err[m]:.2e} over its limit {LIMIT[m]:.0e}" for m in ("fp16", "fp32") if m in err and not err[m] <= LIMIT[m]]
    if not ok:
        fails.append(f"{name}: a word outside the output slice, of the input or of the residual buffer was written")
    return fails


# ---- cases ---------------------------------------------------------------------------------------------------------------------------
OFFS = (0, 8, 24)
SLOT = dict(tc=0, grid=1, smem=2, BN=3, stages=4, strip=5, resident=6, tiles=8, n_tiles=9, kc=10, ctas=11)


def tile_geometry(tw):
    """the smallest map (W, H) on which choose_tile (csrc/conv_tc.cu) picks tile width tw, ragged in x and in y.  Tile width 8 is picked
    only for maps exactly 8 wide (on a wider map 16-wide tiles cover it in as few tiles, and ties go to the wider tile): ragged in y only.
    Tile width 128 is one row tall: ragged in x only."""
    def choose(W, H):
        best = None
        for t in (128, 64, 32, 16, 8):
            n = -(-W // t) * -(-H // (128 // t))
            if best is None or n < best[0]:
                best = (n, t)
        return best[1]
    cands = [(W * H, W, H) for W in range(8, 400) for H in range(3, 200)
             if choose(W, H) == tw and (W % tw or tw == 8) and (H % (128 // tw) or tw == 128) and W * H >= 128]
    _, W, H = min(cands)
    return W, H, -(-W // tw) * -(-H // (128 // tw))


def coverage_cases():
    """one case per (KC, BN, RES, CTAS_PER_SM) instantiation: BN = Co, KC from the input channels (12 -> kc 16 on a zero-padded 16,
    48 -> 16, 32 / 96 -> 32, 64 / 128 -> 64); one CTA per SM on a map of fewer tiles than SMs, two on a map of 140 tiles with resident
    weights.  The residual instantiations take fp16 outputs; the others alternate fp16 and fp32 outputs and the three activations."""
    CI = {16: (12, 48), 32: (32, 96), 64: (64, 128)}
    out = {}
    for kc, cis in CI.items():
        for res in (False, True):
            for j, bn in enumerate(range(16, 129, 16)):
                geo = dict(B=1, H=20, W=44, ci=cis[(j + res) % 2], co=bn, k=3 if j % 2 == 0 else 1, act=(NONE, SILU, SIGMOID)[j % 3],
                           res="sep" if res else None, y_dt=F32 if not res and j % 2 else F16)
                out[f"cov_kc{kc}_bn{bn}{'_res' if res else ''}_1cta"] = (geo, dict(tc=1, kc=kc, BN=bn, ctas=1))
            for j, bn in enumerate((16, 32, 48, 64)):
                ci, k = (cis[0], 3) if not res else (cis[1], 1)
                geo = dict(B=1, H=140, W=128, ci=ci, co=bn, k=k, act=(SILU, NONE, SIGMOID)[j % 3], res="alias" if res and j % 2 else
                           ("sep" if res else None), y_dt=F32 if not res and j % 2 else F16)
                out[f"cov_kc{kc}_bn{bn}{'_res' if res else ''}_2cta"] = (geo, dict(tc=1, kc=kc, BN=bn, ctas=2, resident=1, strip=int(k == 3)))
    return out


def tile_cases():
    """every tile width choose_tile can pick, each on a map ragged in x and in y"""
    out = {}
    for j, tw in enumerate((8, 16, 32, 64, 128)):
        W, H, tiles = tile_geometry(tw)
        out[f"tw{tw}_ragged_{W}x{H}"] = (dict(B=2, H=H, W=W, ci=32, co=48, k=3, res="sep" if j % 2 else None),
                                        dict(tc=1, tiles=2 * tiles, BN=48))
    return out


CASES = {
    **coverage_cases(),
    **tile_cases(),
    # stride 2 through the four parity maps: ragged output, two N tiles, the fp32 head layout
    "s2_ragged": (dict(B=2, H=50, W=86, ci=32, co=64, k=3, s=2), dict(tc=1, BN=64, strip=0)),
    "s2_two_n_tiles": (dict(B=2, H=64, W=128, ci=64, co=256, k=3, s=2, res="sep"), dict(tc=1, n_tiles=2, strip=0)),
    "s2_kc16_f32": (dict(B=1, H=34, W=68, ci=48, co=45, k=3, s=2, y_dt=F32, act=NONE), dict(tc=1, kc=16, BN=48)),
    # dilation with and without the strip: strip at tw 64 / 128, at four channel blocks, at tw + 2 dil = 256 and just past it
    "d2_strip": (dict(B=1, H=32, W=64, ci=64, co=64, k=3, d=2), dict(tc=1, strip=1)),
    "d3_strip_res": (dict(B=1, H=12, W=128, ci=64, co=64, k=3, d=3, res="alias"), dict(tc=1, strip=1)),
    "d6_no_strip_tw32": (dict(B=2, H=30, W=40, ci=64, co=64, k=3, d=6), dict(tc=1, strip=0)),
    "d6_streamed": (dict(B=1, H=16, W=128, ci=256, co=128, k=3, d=6), dict(tc=1, strip=0, resident=0)),
    "strip_cblocks4": (dict(B=2, H=3, W=100, ci=256, co=16, k=3), dict(tc=1, strip=1, kc=64, resident=1)),
    "strip_cblocks5_none": (dict(B=2, H=3, W=100, ci=320, co=16, k=3), dict(tc=1, strip=0, kc=64, resident=1)),
    "strip_w256_d64": (dict(B=2, H=3, W=100, ci=16, co=32, k=3, d=64), dict(tc=1, strip=1)),
    "strip_w258_d65": (dict(B=2, H=3, W=100, ci=16, co=32, k=3, d=65), dict(tc=1, strip=0, resident=1)),
    # weight residency at the pack limit (121 KB): 1x1 480 -> 128 just under, 496 -> 128 just over
    "resident_120k": (dict(B=2, H=32, W=64, ci=480, co=128), dict(tc=1, resident=1, BN=128)),
    "streamed_124k": (dict(B=2, H=32, W=64, ci=496, co=128, res="sep"), dict(tc=1, resident=0, BN=128)),
    # waves: fewer tiles than SMs, between one and two waves, many; grid % n_tiles_n on the resident path
    "tiles_lt_sms": (dict(B=3, H=8, W=16, ci=64, co=64), dict(tc=1, tiles=3)),
    "tiles_1_to_2_waves": (dict(B=1, H=200, W=128, ci=64, co=96), dict(tc=1, tiles=200, ctas=1)),
    "tiles_many_waves": (dict(B=4, H=96, W=256, ci=32, co=32, k=3, res="sep"), dict(tc=1, tiles=768, ctas=2)),
    "grid_mod_n_tiles": (dict(B=1, H=40, W=128, ci=16, co=640, y_dt=F32, act=SIGMOID), dict(tc=1, resident=1, n_tiles=10, BN=64, grid=260)),
    # epilogue: BN 80 / 112 / 48-with-a-tail layouts, fp32 heads with odd channel counts (the last channel stored alone) in slices
    "co160_bn80": (dict(B=2, H=16, W=64, ci=64, co=160, res="sep"), dict(tc=1, BN=80, n_tiles=2)),
    "co224_bn112": (dict(B=2, H=16, W=64, ci=64, co=224, y_dt=F32, act=SIGMOID), dict(tc=1, BN=112, n_tiles=2)),
    "co144_bn48": (dict(B=2, H=16, W=64, ci=64, co=144), dict(tc=1, BN=48, n_tiles=3)),
    "co40_bn48_f16": (dict(B=2, H=24, W=40, ci=32, co=40, k=3, act=NONE), dict(tc=1, BN=48)),
    "co40_bn48_f32": (dict(B=2, H=24, W=40, ci=32, co=40, k=3, y_dt=F32, act=SILU), dict(tc=1, BN=48)),
    "head45_f32_off8": (dict(B=2, H=32, W=64, ci=128, co=45, y_dt=F32, act=NONE, bn=False, y_off=8), dict(tc=1, BN=48)),
    "head19_f32_off24": (dict(B=2, H=32, W=64, ci=128, co=19, y_dt=F32, act=NONE, bn=False, y_off=24), dict(tc=1, BN=32)),
    "head57_f32_off0": (dict(B=2, H=16, W=64, ci=256, co=57, y_dt=F32, act=SIGMOID, y_off=0), dict(tc=1, BN=64)),
    "head255_f32_off8": (dict(B=1, H=16, W=32, ci=256, co=255, y_dt=F32, act=NONE, bn=False, y_off=8), dict(tc=1, BN=128, n_tiles=2)),
    # CUDA-core kernel (path 2, and path 0 where the wgmma kernel does not take the op): fp32 input slices, tiny maps, co % 8 != 0
    "simt_f32_in": (dict(B=4, H=1, W=1, ci=256, co=256, x_dt=F32, y_dt=F32, act=SILU, bias=False, bn=False), dict(tc=0)),
    "simt_f32_in_slice": (dict(B=2, H=6, W=6, ci=128, co=64, x_dt=F32, y_dt=F32, act=SIGMOID, x_off=8), dict(tc=0)),
    "simt_f32_in_3x3": (dict(B=2, H=16, W=32, ci=64, co=48, k=3, x_dt=F32, act=SILU), dict(tc=0)),
    "simt_forced_3x3": (dict(B=2, H=24, W=40, ci=64, co=64, k=3, d=2, res="sep", path=2), dict(tc=0)),
    "simt_forced_s2": (dict(B=1, H=32, W=64, ci=32, co=48, k=3, s=2, y_dt=F32, path=2), dict(tc=0)),
    "simt_forced_alias": (dict(B=2, H=16, W=32, ci=128, co=64, res="alias", path=2), dict(tc=0)),
    "simt_co20": (dict(B=2, H=16, W=32, ci=32, co=20, k=3), dict(tc=0)),
    "simt_tiny_map": (dict(B=4, H=4, W=8, ci=64, co=64, k=3, res="sep"), dict(tc=0)),
}

# (B, H, W, ci, co, k, stride, dil, residual): layer classes of the s and m models, and layers at bench scale
LAYERS = [
    (2, 32, 64, 64, 64, 1, 1, 1, False),      # plain 1x1, SW128
    (1, 64, 128, 128, 128, 1, 1, 1, False),
    (2, 16, 32, 512, 256, 1, 1, 1, False),    # 2 N tiles, 8 K stages
    (1, 16, 32, 1024, 512, 1, 1, 1, False),   # SPP.cv2 class
    (2, 64, 64, 16, 32, 3, 1, 1, False),      # Focus conv class: kc=16 (SW32), 9 taps
    (2, 32, 64, 32, 32, 3, 1, 1, True),       # Bottleneck.cv2 + residual, kc=32 (SW64)
    (1, 32, 64, 64, 64, 3, 1, 1, True),
    (1, 16, 32, 128, 128, 3, 1, 1, False),
    (2, 64, 128, 32, 64, 3, 2, 1, False),     # stride-2 parity maps
    (1, 32, 64, 64, 128, 3, 2, 1, False),
    (1, 32, 64, 64, 64, 3, 1, 2, False),      # dilated (RFB2 branch1/2)
    (1, 32, 64, 64, 64, 3, 1, 3, False),
    (1, 16, 32, 256, 128, 3, 1, 6, False),    # ASPP-like dilation
    (1, 24, 40, 64, 64, 3, 1, 1, False),      # W, H not multiples of the tile -> OOB zero fill / clipped stores
    (1, 16, 12, 64, 48, 1, 1, 1, False),      # box wider than the map, Co=48 (m model)
    (1, 32, 32, 48, 96, 3, 1, 1, False),      # kc=16 with Ci=48, Co=96
    (1, 16, 32, 192, 192, 1, 1, 1, False),    # Co=192 -> BN=96 x 2
    (3, 8, 16, 64, 64, 1, 1, 1, False),       # exactly one tile per image
    (2, 16, 128, 64, 64, 3, 1, 1, False),     # full-row tiles (tw=128)
    (1, 12, 128, 64, 64, 3, 1, 2, True),      # full-row tiles + dilation 2 + residual
    (1, 8, 128, 64, 64, 3, 1, 3, False),      # full-row tiles + dilation 3
    (1, 8, 256, 256, 128, 3, 1, 1, False),    # 4 channel blocks, W=256 (2 tiles per row)
    (2, 16, 256, 32, 32, 3, 1, 1, True),      # 64-byte rows (kc=32) + residual (L2 bottleneck class)
    (2, 16, 512, 16, 32, 3, 1, 1, False),     # 32-byte rows (kc=16): Focus conv class
    (1, 8, 128, 48, 96, 3, 1, 2, False),      # kc=16 x 3 channel blocks, dilation 2
    (16, 64, 256, 32, 32, 3, 1, 1, True),     # many full-row tiles + residual
    (16, 128, 256, 16, 32, 3, 1, 1, False),   # many full-row tiles, 32-byte rows (Focus conv at scale)
    (8, 37, 512, 32, 32, 3, 1, 1, False),     # ragged image height (Ho = 37)
    (16, 64, 256, 32, 32, 1, 1, 1, False),    # many tiles, BN=32
    (8, 64, 128, 64, 64, 1, 1, 1, True),      # many tiles + residual
    # layers at bench scale (more tiles than SMs: the persistent CTAs take several tiles each)
    (16, 32, 64, 128, 128, 3, 1, 1, True),    # P4 bottleneck 3x3, residual
    (16, 64, 128, 64, 64, 3, 1, 2, False),    # dilation 2, 1024 tiles
    (16, 64, 128, 128, 256, 3, 2, 1, False),  # stride 2, two N tiles
    (16, 32, 64, 128, 80, 3, 1, 1, False),    # N tile of 80 channels
    (6, 64, 128, 256, 128, 3, 1, 1, False),   # FFM class: 4 channel blocks, 384 tiles
]
STREAMED = [s for s in LAYERS if s[0] >= 6 and s[5] == 3][-5:] + [(16, 32, 64, 256, 128, 1, 1, 1, False), (2, 32, 64, 64, 64, 1, 1, 1, False)]

# (B, H, W, ci, co, k, stride, dil, residual): resident weights and strip loads on path 1, each against its streamed twin
REUSE = [
    (2, 64, 64, 16, 32, 3, 1, 1, False),      # kc = 16 (32-byte rows)
    (1, 32, 32, 48, 96, 3, 1, 1, False),      # kc = 16, three channel blocks
    (2, 32, 256, 32, 32, 3, 1, 1, True),      # kc = 32, tw = 128, residual
    (1, 32, 64, 64, 64, 3, 1, 2, False),      # kc = 64, tw = 64 (th = 2), dilation 2
    (1, 32, 64, 64, 64, 3, 1, 3, True),       # dilation 3 + residual
    (1, 12, 128, 64, 64, 3, 1, 2, True),      # tw = 128, dilation 2 + residual
    (1, 24, 40, 64, 64, 3, 1, 1, False),      # ragged right edge and height
    (8, 37, 512, 32, 32, 3, 1, 1, False),     # ragged height, many tiles
    (3, 8, 16, 64, 64, 1, 1, 1, False),       # fewer tiles than SMs
    (2, 16, 32, 512, 256, 1, 1, 1, False),    # Co = 256: two N tiles
    (4, 32, 64, 128, 256, 1, 1, 1, True),     # two N tiles + residual
    (2, 16, 32, 192, 192, 1, 1, 1, False),    # BN = 96 x 2
    (2, 32, 64, 480, 128, 1, 1, 1, False),    # pack 120 KB: just under the residency limit
    (2, 32, 64, 496, 128, 1, 1, 1, False),    # pack 124 KB: just over (streamed on both paths)
    (16, 64, 128, 32, 64, 3, 2, 1, False),    # stride 2, resident
    (16, 64, 128, 64, 128, 3, 2, 1, False),   # stride 2, 144 KB pack (streamed)
    # bench-scale layers of the s/PSP forward (batch 16 at 512x1024)
    (16, 256, 256, 32, 64, 3, 1, 1, False),   # layer 0 on pixel pairs
    (16, 128, 256, 32, 32, 3, 1, 1, True),    # C3 bottleneck 3x3 32->32 + residual
    (16, 128, 256, 32, 32, 1, 1, 1, False),
    (16, 64, 128, 64, 64, 3, 1, 1, True),     # C3 bottleneck 3x3 64->64 + residual
    (16, 64, 128, 64, 64, 3, 1, 2, False),    # SegMaskPSP dilated 3x3
    (16, 32, 64, 128, 128, 3, 1, 1, True),
    (16, 16, 32, 256, 512, 1, 1, 1, False),   # four N tiles, resident
    (6, 64, 128, 256, 128, 3, 1, 1, False),   # FFM 3x3 256->128 (576 KB pack: streamed)
]

# (B, H, W, ci, co, k, stride, residual, BN at two CTAs): two CTAs per SM beyond the narrow 1x1 layers, including Co = 128 / 256 layers
# that take BN = 64 N tiles to admit the second CTA; every map is ragged in x (a tile width that does not divide the map's)
TWO_CTA = [
    (4, 37, 250, 32, 64, 3, 1, False, 64),    # 3x3 strip (layer 0 class)
    (4, 21, 250, 32, 32, 3, 1, True, 32),     # 3x3 strip + residual (C3 bottleneck class)
    (8, 64, 252, 32, 64, 3, 2, False, 64),    # 3x3 stride 2, per-tap boxes
    (8, 40, 250, 64, 64, 1, 1, True, 64),     # 1x1 + residual
    (8, 32, 120, 256, 128, 1, 1, False, 64),  # Co = 128: BN 128 -> 64
    (8, 16, 100, 256, 256, 1, 1, False, 64),  # Co = 256: BN 128 -> 64, tw = 8 over width 100
]

# (B, H, W, ci, co, k, residual): the fp16 epilogue transposes each quad's accumulator words so that a lane stores the 8 channels of one
# group as one 16-byte vector (a transposition error shows as gross mismatches); slices at channel 8, the smallest offset it allows
EPILOGUE = [
    (2, 37, 45, 32, 64, 3, False),     # ragged right edge and bottom (tiles reach past the map)
    (1, 20, 70, 16, 48, 1, False),     # BN = 48: a last block of two 8-channel groups
    (3, 11, 136, 64, 32, 1, False),    # tw = 128 over a ragged width
    (16, 64, 128, 64, 64, 1, False),   # 1x1 at BN = 64 over many tiles (two CTAs per SM)
    (2, 16, 32, 128, 256, 1, False),   # two N tiles
    (2, 33, 40, 64, 64, 3, True),      # residual, ragged map
    (4, 32, 64, 128, 256, 1, True),    # residual, two N tiles
]


def shape_list_cases():
    """LAYERS on the CUDA-core kernel (path 2) and the wgmma kernel (path 1), STREAMED on path 3; REUSE on path 1 with a path-3 twin;
    TWO_CTA on path 1 into a slice at channel 8 with a path-3 twin, and with a residual also against its aliasing twin; EPILOGUE on path 1
    without BatchNorm into a slice at channel 8, and with a residual also against its aliasing twin"""
    out = {}
    for path, kind, shapes in ((2, "simt", LAYERS), (1, "tc", LAYERS), (3, "streamed", STREAMED)):
        for i, (B, H, W, ci, co, k, s, d, res) in enumerate(shapes):
            out[f"layer_{kind}_{i}"] = (dict(B=B, H=H, W=W, ci=ci, co=co, k=k, s=s, d=d, res="sep" if res else None, path=path),
                                        dict(tc=int(path != 2)))
    for B, H, W, ci, co, k, s, d, res in REUSE:
        out[f"reuse_{ci}-{co}-k{k}s{s}d{d}-{B}x{H}x{W}{'-res' if res else ''}"] = (
            dict(B=B, H=H, W=W, ci=ci, co=co, k=k, s=s, d=d, res="sep" if res else None, path=1, twin="path3"), dict(tc=1))
    for B, H, W, ci, co, k, s, res, bn in TWO_CTA:
        geo = dict(B=B, H=H, W=W, ci=ci, co=co, k=k, s=s, res="sep" if res else None, bn=False, y_off=8, path=1)
        want = dict(tc=1, resident=1, ctas=2, BN=bn, strip=int(k == 3 and s == 1))
        name = f"two_cta_{ci}-{co}-k{k}s{s}-{B}x{H}x{W}{'-res' if res else ''}"
        out[name] = (dict(geo, twin="path3"), want)
        if res:
            out[name + "_alias"] = (dict(geo, twin="alias"), want)
    for B, H, W, ci, co, k, res in EPILOGUE:
        geo = dict(B=B, H=H, W=W, ci=ci, co=co, k=k, res="sep" if res else None, bn=False, y_off=8, path=1)
        name = f"epilogue_{ci}-{co}-k{k}-{B}x{H}x{W}{'-res' if res else ''}"
        out[name] = (geo, dict(tc=1))
        if res:
            out[name + "_alias"] = (dict(geo, twin="alias"), dict(tc=1))
    return out


CASES.update(shape_list_cases())


def case_args(name):
    geo, _ = CASES[name]
    i = list(CASES).index(name)
    a = dict(x_off=OFFS[i % 3], y_off=OFFS[(i + 1) % 3], r_off=OFFS[(i + 2) % 3], seed=i)
    a.update(geo)
    return a


_RESULTS = {}


def result(name):
    """the case's run, once per session (the coverage test reuses the cases' launches)"""
    if name not in _RESULTS:
        a = case_args(name)
        _RESULTS[name] = (a, *run(**a))
    return _RESULTS[name]


@pytest.mark.parametrize("name", list(CASES))
def test_conv_forward_matches_fp64(name):
    """one conv on the route the case was built for, through channel slices, against fp64 (a NaN or an infinity fails it); a twin
    matches it bit for bit: a path-3 twin on streamed weights at one CTA per SM, an aliasing twin on the same route"""
    a, info, err, ok, twin = result(name)
    print(f"\n[{name}] {describe(info)}\n[{name}] " + "  ".join(f"{k} {v:.2e}" for k, v in err.items()))
    want = CASES[name][1]
    got = {k: info[SLOT[k]] for k in want}
    assert got == want, f"route: expected {want}, got {got} ({describe(info)})"
    fails = check(name, info, err, ok)
    print_worst()
    assert not fails, "\n".join(fails)
    if twin is not None:
        twin_info, same = twin
        print(f"[{name}] {a['twin']} twin: {describe(twin_info)}")
        if a["twin"] == "path3":
            got = {k: twin_info[SLOT[k]] for k in ("tc", "resident", "strip", "ctas")}
            assert got == dict(tc=1, resident=0, strip=0, ctas=1), f"path-3 twin: {describe(twin_info)}"
        else:
            assert twin_info == info, f"aliasing twin routed {describe(twin_info)}"
        assert same, f"the {a['twin']} twin's output buffer differs from the launch's"


def test_conv_forward_reaches_every_instantiation():
    """the cases launch every conv_tc_kernel<KC, BN, RES, CTAS_PER_SM> conv_tc_launch dispatches: KC 16 / 32 / 64, BN 16 .. 128, with and
    without a residual, at one CTA per SM and, for BN <= 64 (kTwoCtaMaxBN), at two.  None is unreachable under conv_tc_prepare's rules."""
    want = {(kc, bn, res, ctas) for kc in (16, 32, 64) for bn in range(16, 129, 16) for res in (0, 1) for ctas in ((1, 2) if bn <= 64 else (1,))}
    assert len(want) == 72
    reached = defaultdict(list)
    for name in CASES:
        a, info = result(name)[:2]
        if info[0]:
            reached[(info[10], info[3], int(a.get("res") is not None), info[11])].append(name)
    missing = sorted(want - set(reached))
    print(f"\n{len(set(reached) & want)} of {len(want)} instantiations reached; missing: {missing}")
    assert not missing
    assert set(reached) <= want, sorted(set(reached) - want)


# ---- census: every conv op of the plans ----------------------------------------------------------------------------------------------
CENSUS = [  # (model tag, yaml, B, H, W, train)
    ("s_psp", "yolov5s_city_seg.yaml", 16, 512, 1024, False),
    ("s_psp", "yolov5s_city_seg.yaml", 2, 416, 736, False),
    ("m_lab", "yolov5m_city_seg_lab.yaml", 16, 512, 1024, False),
    ("m_lab", "yolov5m_city_seg_lab.yaml", 2, 416, 736, False),
    ("s_psp", "yolov5s_city_seg.yaml", 4, 512, 1024, True),
    ("m_lab", "yolov5m_city_seg_lab.yaml", 4, 512, 1024, True),
]
DT = {0: F16, 1: F32}


def census_ops(yml, B, H, W, train):
    """(op index, the plan's info slots, run() arguments at the op's geometry and slice layout) for every conv op of the plan"""
    import ctypes as C

    from multiyolov5_b200 import _lib as L
    from multiyolov5_b200.engine import CompiledPlan
    from multiyolov5_b200.models.yolo import Model
    torch.manual_seed(0)
    model = Model(yml).cuda()
    model.train(train)
    plan = CompiledPlan(model, B, H, W, train=train)
    plan.upload_weights()
    out = []
    for i, o in enumerate(plan.pb.ops):
        if o.kind != L.OP_CONV:
            continue
        info = (C.c_int32 * 12)()
        L.check(L.lib().myolo_plan_conv_info(plan.handle, i, info))
        s = plan.pb.slots[o.slot]
        co, ci, k = s.conv.weight.shape[0], s.conv.weight.shape[1], s.conv.weight.shape[2]
        assert o.in_.c == ceil16(ci) and k == o.k, (i, o.in_.c, ci)
        res = None
        a = dict(B=B, H=o.in_.h, W=o.in_.w, ci=ci, co=co, k=o.k, s=o.stride, d=o.dil, x_dt=DT[o.in_.buf.dtype], y_dt=DT[o.out.buf.dtype],
                 act=o.act, bn=s.bn is not None, bias=s.conv.bias is not None, x_off=o.in_.c_off, x_ctot=o.in_.buf.c, y_off=o.out.c_off,
                 y_ctot=o.out.buf.c, seed=i, images=[0, B - 1])
        if o.in2 is not None:
            if o.in2.buf is o.out.buf and o.in2.c_off == o.out.c_off:
                res = "alias"
            else:
                res = "sep"
                a.update(r_off=o.in2.c_off, r_ctot=o.in2.buf.c)
        a["res"] = res
        out.append((i, list(info), a))
    del plan
    return out


def test_conv_forward_census_of_the_plans(monkeypatch):
    """every conv op of the s_psp and m_lab inference plans at 16 x 512 x 1024 and 2 x 416 x 736 and of their train plans at 4 x 512 x
    1024: the entry at the op's geometry and slice layout routes and tiles it as the plan does (all 12 info slots equal), and matches fp64
    on the first and the last image (the last holds the tail tiles)"""
    monkeypatch.setenv("MYOLO_FORCE_SIMT", "0")
    fails, total = [], defaultdict(int)
    for tag, yml, B, H, W, train in CENSUS:
        count = defaultdict(int)
        for i, plan_info, a in census_ops(yml, B, H, W, train):
            info, err, ok, _ = run(**a)
            name = f"{tag} {'train ' if train else ''}{B}x{H}x{W} op {i}"
            if info != plan_info:
                fails.append(f"{name}: entry routed {info}, the plan {plan_info}")
            fails += check(name, info, err, ok)
            count["wgmma" if info[0] else "simt"] += 1
            if info[0]:
                count[f"wgmma {info[11]} cta/SM"] += 1
                count["wgmma strip"] += info[5]
                count["wgmma fp32 out"] += a["y_dt"] == F32
                count["wgmma residual"] += a["res"] is not None
            count["input slice"] += a["x_ctot"] != ceil16(a["ci"])
            count["ops"] += 1
            torch.cuda.empty_cache()
        print(f"\n[{tag} {'train' if train else 'infer'} {B}x{H}x{W}] " + ", ".join(f"{k}: {v}" for k, v in sorted(count.items())))
        for k, v in count.items():
            total[k] += v
    print_worst()
    assert not fails, "\n".join(fails[:30])
    assert total["wgmma 2 cta/SM"] >= 1 and total["wgmma strip"] >= 1 and total["wgmma fp32 out"] >= 1 and total["input slice"] >= 1, total


SMEM_BUDGET = 227 * 1024
RESIDENT_LIMIT = SMEM_BUDGET - (1024 + 8192 + 1024) - 6 * 128 * 64 * 2   # misc + six A stages (conv_tc.cu)


def test_spsp_plan_reuse_paths():
    import ctypes as C
    from multiyolov5_b200 import _lib, synth
    from multiyolov5_b200.models.yolo import Model
    yml = "yolov5s_city_seg.yaml"
    sd = synth.synth_state_dict(synth.load_manifest("s_psp"), synth.load_cfg(yml), seed=1)
    model = Model(yml)
    model.load_state_dict(sd)
    model.cuda().eval().half()
    model(torch.zeros(16, 3, 512, 1024, dtype=torch.float16, device="cuda"))
    torch.cuda.synchronize()
    plan = model.engine().last_plan
    info = (C.c_int32 * 12)()
    n_tc = n_res = n_strip = 0
    for i, o in enumerate(plan.pb.ops):
        if o.kind != _lib.OP_CONV:
            continue
        _lib.check(_lib.lib().myolo_plan_conv_info(plan.handle, i, info))
        if not info[0]:
            continue
        n_tc += 1
        s = plan.pb.slots[o.slot].conv
        k, bn, kc, ntn, grid = s.kernel_size[0], info[3], info[10], info[9], info[1]
        ci_pad = (s.in_channels + kc - 1) // kc * kc
        pack = (k * k * ci_pad * bn * 2 + 1023) // 1024 * 1024
        expect = pack <= RESIDENT_LIMIT
        assert info[6] == int(expect), f"op {i} {o.tag} {s.in_channels}->{s.out_channels} k{k}: pack {pack} B, resident {info[6]}"
        if info[6]:
            assert grid % ntn == 0, f"op {i}: grid {grid} is not a multiple of {ntn} N tiles"
        strip = bool(info[6]) and k == 3 and s.stride[0] == 1 and o.out.w >= 64 and ci_pad // kc <= 4
        assert info[5] == int(strip), f"op {i} {o.tag} {s.in_channels}->{s.out_channels} k{k} @{o.out.h}x{o.out.w}: strip {info[5]}"
        n_res += info[6]
        n_strip += info[5]
    # streamed: the 22 packs over 120 KB (3x3 with 64+ input channels and 1x1 with 512+ input channels, at BN = 128).
    # strip: layer 0, the C3 bottleneck 3x3 layers at 128x256 and 64x128, and the three SegMaskPSP 3x3 64->64 layers
    assert (n_tc, n_res, n_strip) == (65, 43, 9)


# ---- sensitivity ---------------------------------------------------------------------------------------------------------------
MUTANT_CASES = {  # wrong reference: the case it runs on
    "bf16": dict(B=2, H=24, W=40, ci=64, co=64, k=3, bn=True, act=SILU),
    "tap": dict(B=2, H=24, W=40, ci=64, co=64, k=3, bn=False, act=NONE, y_dt=F32),
    "bias": dict(B=2, H=24, W=40, ci=64, co=64, k=1, bn=True, act=SILU, y_dt=F32),
    "replicate": dict(B=1, H=16, W=4096, ci=16, co=16, k=3, bn=False, act=NONE),
    "rounded_before_residual": dict(B=2, H=24, W=40, ci=64, co=64, k=3, bn=True, act=SILU, res="sep", res_cancel=True),
}


def test_conv_forward_limits_catch_wrong_references():
    """the limits discriminate: each deliberately wrong reference moves the output by less than 1 % (relative Frobenius norm) and still
    misses its limit by at least 10x"""
    print()
    for mutant, a in MUTANT_CASES.items():
        info, err, _, _ = run(**a, mutant=mutant)
        m = "fp16" if a.get("y_dt", F16) == F16 else "fp32"
        over = err[m] / LIMIT[m]
        print(f"mutant {mutant:<24} ({describe(info)}): changes the output by {100 * err['change']:.3f} %, {m} error at {over:.0f}x its limit")
        assert info[0] == 1, mutant
        assert err["change"] < 0.01, (mutant, err)
        assert over >= 10, (mutant, over, err)
