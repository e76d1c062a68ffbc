"""GPU: the wgmma conv kernel at two CTAs per SM beyond the narrow 1x1 layers: 3x3 strip layers with and without a residual, 3x3 stride 2,
1x1 with a residual (also aliasing the output, as the data-gradient convs use it), and Co = 128 / 256 layers that take BN = 64 N tiles
to admit the second CTA.  Each shape must launch at two CTAs per SM (slot 11 of the launch report), match the streamed-weight one-CTA
launch of the same op (path 3, BN from Co alone) bit for bit, match an fp64 conv on the values the kernel reads (test_gpu_conv_forward.py), and leave pixels past a ragged map untouched."""
import pytest
import torch

from tests.test_gpu_conv_forward import LIMIT, SILU, U16, conv64, pack_ref

pytestmark = pytest.mark.gpu

SENTINEL = -12345   # int16 bit pattern of the untouched fp16 words (a negative NaN)
C_OFF = 8           # the slice starts 8 channels into the buffer

# (B, H, W, Ci, Co, k, stride, residual, BN at two CTAs); every map is ragged in x (a tile width that does not divide the map's)
SHAPES = [
    (4, 37, 250, 32, 64, 3, 1, False, 64),    # 3x3 strip (layer 0 class)
    (4, 21, 250, 32, 32, 3, 1, True, 32),     # 3x3 strip + residual (C3 bottleneck class)
    (8, 64, 252, 32, 64, 3, 2, False, 64),    # 3x3 stride 2, per-tap boxes
    (8, 40, 250, 64, 64, 1, 1, True, 64),     # 1x1 + residual
    (8, 32, 120, 256, 128, 1, 1, False, 64),  # Co = 128: BN 128 -> 64
    (8, 16, 100, 256, 256, 1, 1, False, 64),  # Co = 256: BN 128 -> 64, tw = 8 over width 100
]
IDS = [f"{s[3]}-{s[4]}-k{s[5]}s{s[6]}-{s[0]}x{s[1]}x{s[2]}{'-res' if s[7] else ''}" for s in SHAPES]


def _inputs(shape):
    B, H, W, Ci, Co, k, s, res, _ = shape
    g = torch.Generator().manual_seed(3000 + SHAPES.index(shape))
    x = torch.randn(B, H, W, Ci, generator=g).half().cuda()
    w = (torch.randn(Co, Ci, k, k, generator=g) * (2.0 / (Ci * k * k)) ** 0.5).cuda()
    bias = (torch.randn(Co, generator=g) * 0.1).cuda()
    Ho, Wo = (H - 1) // s + 1, (W - 1) // s + 1
    r = torch.randn(B, Ho, Wo, Co, generator=g).half().cuda() if res else None
    return x, w, bias, r


def _reference(x, w, bias, r, s):
    """fp64 on the values the kernel reads: the fp16 pack of w, the fp32 bias, an exact SiLU, the residual before the output's rounding"""
    wp, bp = pack_ref(w, None, bias, 0.0)
    y = conv64(x.permute(0, 3, 1, 2).double(), wp, bp, w.shape[-1], s, 1, SILU).permute(0, 2, 3, 1)
    return y + r.double() if r is not None else y


@pytest.mark.parametrize("shape", SHAPES, ids=IDS)
def test_two_cta_matches_one_cta_and_torch(shape):
    from multiyolov5_b200 import ops
    B, H, W, Ci, Co, k, s, res, bn = shape
    x, w, bias, r = _inputs(shape)
    Ho, Wo = (H - 1) // s + 1, (W - 1) // s + 1
    ctot = C_OFF + Co + 16
    n_pix = B * Ho * Wo
    pad_pix = 16 * Wo + 256                # room for every row a tile could reach past the last image
    buf = torch.full((n_pix + pad_pix, ctot), SENTINEL, dtype=torch.int16, device="cuda")
    out = buf[:n_pix].view(torch.float16).view(B, Ho, Wo, ctot)[..., C_OFF:C_OFF + Co]
    info1, info3 = [], []
    ops.conv_bn_silu(x, w, None, bias=bias, stride=s, residual=r, path=1, out=out, info=info1)
    y3 = ops.conv_bn_silu(x, w, None, bias=bias, stride=s, residual=r, path=3, info=info3)
    torch.cuda.synchronize()
    assert info1[0] == 1 and info1[6] == 1, f"{shape}: not a resident-weight wgmma launch: {info1}"
    assert info1[11] == 2, f"{shape}: {info1[11]} CTAs per SM"
    assert info1[3] == bn, f"{shape}: BN {info1[3]}"
    assert info1[5] == int(k == 3 and s == 1), f"{shape}: strip {info1[5]}"
    assert info3[11] == 1 and info3[6] == 0, f"{shape}: path 3 {info3}"
    assert (buf[:, :C_OFF] == SENTINEL).all(), "channels before the slice were written"
    assert (buf[:, C_OFF + Co:] == SENTINEL).all(), "channels after the slice were written"
    assert (buf[n_pix:] == SENTINEL).all(), "pixels past the map were written"
    assert torch.equal(out.contiguous().view(torch.int16), y3.view(torch.int16)), \
        f"{shape}: {(out != y3).sum().item()} outputs differ from the one-CTA launch"
    ref = _reference(x, w, bias, r, s)
    y = out.double()
    err = float(((y - ref).abs() - U16 * ref.abs()).clamp_min(0).max()) / float(ref.abs().max())
    assert err <= LIMIT["fp16"], f"{shape}: error {err:.3g} over the limit {LIMIT['fp16']:.0e} (test_gpu_conv_forward.py)"


@pytest.mark.parametrize("shape", [s for s in SHAPES if s[7]], ids=[i for i, s in zip(IDS, SHAPES) if s[7]])
def test_two_cta_residual_aliasing_output(shape):
    from multiyolov5_b200 import ops
    x, w, bias, r = _inputs(shape)
    s = shape[6]
    y_sep = ops.conv_bn_silu(x, w, None, bias=bias, stride=s, residual=r, path=3)
    y_alias = r.clone()
    info = []
    ops.conv_bn_silu(x, w, None, bias=bias, stride=s, residual=y_alias, path=1, out=y_alias, info=info)
    torch.cuda.synchronize()
    assert info[11] == 2
    assert torch.equal(y_alias.view(torch.int16), y_sep.view(torch.int16))
