"""GPU: the wgmma conv kernel's fp16 epilogue, which transposes each quad's accumulator words so that a lane stores the 8 channels of one
group as one 16-byte vector.  The output goes into a channel slice of a buffer filled with a sentinel: channels outside the slice and
pixels past the map must keep the sentinel, the slice must match an fp64 conv on the values the kernel reads (test_gpu_conv_forward.py) (a transposition error shows as gross mismatches),
and a residual that aliases the output must give what a separate residual buffer gives."""
import pytest
import torch

from tests.test_gpu_conv_forward import LIMIT, SILU, U16, conv64, pack_ref

pytestmark = pytest.mark.gpu

SENTINEL = -12345   # int16 bit pattern of the untouched fp16 words (a negative NaN)
C_OFF = 8           # the slice starts 8 channels into the buffer (16 bytes: the smallest offset the vector stores allow)

# (B, H, W, Ci, Co, k, residual)
SHAPES = [
    (2, 37, 45, 32, 64, 3, False),     # ragged right edge and bottom (tiles reach past the map)
    (1, 20, 70, 16, 48, 1, False),     # BN = 48: a last block of two 8-channel groups
    (3, 11, 136, 64, 32, 1, False),    # tw = 128 over a ragged width
    (16, 64, 128, 64, 64, 1, False),   # 1x1 at BN = 64 over many tiles (two CTAs per SM)
    (2, 16, 32, 128, 256, 1, False),   # two N tiles
    (2, 33, 40, 64, 64, 3, True),      # residual, ragged map
    (4, 32, 64, 128, 256, 1, True),    # residual, two N tiles
]


def _inputs(shape):
    B, H, W, Ci, Co, k, res = shape
    g = torch.Generator().manual_seed(2000 + SHAPES.index(shape))
    x = torch.randn(B, H, W, Ci, generator=g).half().cuda()
    w = (torch.randn(Co, Ci, k, k, generator=g) * (2.0 / (Ci * k * k)) ** 0.5).cuda()
    bias = (torch.randn(Co, generator=g) * 0.1).cuda()
    r = torch.randn(B, H, W, Co, generator=g).half().cuda() if res else None
    return x, w, bias, r


def _reference(x, w, bias, r):
    """fp64 on the values the kernel reads: the fp16 pack of w, the fp32 bias, an exact SiLU, the residual before the output's rounding"""
    wp, bp = pack_ref(w, None, bias, 0.0)
    y = conv64(x.permute(0, 3, 1, 2).double(), wp, bp, w.shape[-1], 1, 1, SILU).permute(0, 2, 3, 1)
    return y + r.double() if r is not None else y


@pytest.mark.parametrize("shape", SHAPES, ids=[f"{s[3]}-{s[4]}-k{s[5]}-{s[0]}x{s[1]}x{s[2]}{'-res' if s[6] else ''}" for s in SHAPES])
def test_epilogue_slice_and_values(shape):
    from multiyolov5_b200 import ops
    B, H, W, Ci, Co, k, res = shape
    x, w, bias, r = _inputs(shape)
    ctot = C_OFF + Co + 16
    n_pix = B * H * W
    pad_pix = 16 * W + 256                 # room for every row a tile could reach past the last image
    buf = torch.full((n_pix + pad_pix, ctot), SENTINEL, dtype=torch.int16, device="cuda")
    out = buf[:n_pix].view(torch.float16).view(B, H, W, ctot)[..., C_OFF:C_OFF + Co]
    ops.conv_bn_silu(x, w, None, bias=bias, residual=r, path=1, out=out)
    torch.cuda.synchronize()
    assert (buf[:, :C_OFF] == SENTINEL).all(), "channels before the slice were written"
    assert (buf[:, C_OFF + Co:] == SENTINEL).all(), "channels after the slice were written"
    assert (buf[n_pix:] == SENTINEL).all(), "pixels past the map were written"
    y = out.double()
    ref = _reference(x, w, bias, r)
    err = float(((y - ref).abs() - U16 * ref.abs()).clamp_min(0).max()) / float(ref.abs().max())
    assert err <= LIMIT["fp16"], f"{shape}: error {err:.3g} over the limit {LIMIT['fp16']:.0e} (test_gpu_conv_forward.py)"


@pytest.mark.parametrize("shape", [s for s in SHAPES if s[6]], ids=lambda s: f"{s[3]}-{s[4]}-k{s[5]}-{s[0]}x{s[1]}x{s[2]}")
def test_epilogue_residual_aliasing_output(shape):
    from multiyolov5_b200 import ops
    x, w, bias, r = _inputs(shape)
    y_sep = ops.conv_bn_silu(x, w, None, bias=bias, residual=r, path=1)
    y_alias = r.clone()
    ops.conv_bn_silu(x, w, None, bias=bias, residual=y_alias, path=1, out=y_alias)
    torch.cuda.synchronize()
    assert torch.equal(y_alias.view(torch.int16), y_sep.view(torch.int16))
