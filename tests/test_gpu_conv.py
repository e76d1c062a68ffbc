"""GPU: the fused Conv+BN+SiLU(+residual) kernels (wgmma path and CUDA-core path) against a torch fp32 restatement of
Conv.fuseforward (reference models/common.py:45-46, BN fold utils/torch_utils.py:182-202) on identical fp16-rounded inputs.
Tolerance: |err| <= 2e-3 * max|ref| + fp16 output rounding (the kernels accumulate in fp32; only the sum order differs)."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

# (B, H, W, Ci, Co, k, stride, dil, residual)
SHAPES = [
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


def torch_ref(x_nhwc, w, bn, stride, dil, residual, eps=1e-3):
    x = x_nhwc.float().permute(0, 3, 1, 2).cpu()
    g, b, m, v = [t.cpu() for t in bn]
    scale = g / torch.sqrt(v + eps)
    wf = (w.cpu() * scale.view(-1, 1, 1, 1)).half().float()      # the pack kernel rounds folded weights to fp16
    k = w.shape[2]
    y = F.conv2d(x, wf, None, stride, dil * (k // 2), dil) + (b - m * scale).view(1, -1, 1, 1)
    y = y * torch.sigmoid(y)
    if residual is not None:
        y = y + residual.float().permute(0, 3, 1, 2).cpu()
    return y.permute(0, 2, 3, 1).contiguous()


# path 2: CUDA-core kernel, 1: wgmma kernel with the planner's tiling rules, 3: the same wgmma kernel through the standalone path-3 entry
PAIR_SHAPES = [s for s in SHAPES if s[0] >= 6 and s[5] == 3][-5:] + [(16, 32, 64, 256, 128, 1, 1, 1, False), (2, 32, 64, 64, 64, 1, 1, 1, False)]


@pytest.mark.parametrize("path,shape", [(p, s) for p in (2, 1) for s in SHAPES] + [(3, s) for s in PAIR_SHAPES],
                         ids=[f"{'simt' if p == 2 else 'tc'}-{i}" for p in (2, 1) for i in range(len(SHAPES))]
                         + [f"pair-{i}" for i in range(len(PAIR_SHAPES))])
def test_conv_bn_silu(shape, path):
    from multiyolov5_b200 import ops
    B, H, W, Ci, Co, k, s, d, res = shape
    gsd = torch.Generator().manual_seed(hash(shape) % (2 ** 31))
    x = torch.randn(B, H, W, Ci, generator=gsd).half().cuda()
    w = (torch.randn(Co, Ci, k, k, generator=gsd) * (2.0 / (Ci * k * k)) ** 0.5).cuda()
    bn = [torch.rand(Co, generator=gsd) * 0.4 + 0.8, torch.randn(Co, generator=gsd) * 0.1, torch.randn(Co, generator=gsd) * 0.1,
          torch.rand(Co, generator=gsd) + 0.5]
    bn = [t.cuda() for t in bn]
    Ho = (H + 2 * d * (k // 2) - d * (k - 1) - 1) // s + 1
    Wo = (W + 2 * d * (k // 2) - d * (k - 1) - 1) // s + 1
    r = torch.randn(B, Ho, Wo, Co, generator=gsd).half().cuda() if res else None
    y = ops.conv_bn_silu(x, w, bn, stride=s, dil=d, residual=r, path=path)
    torch.cuda.synchronize()
    ref = torch_ref(x, w, bn, s, d, r)
    err = (y.float().cpu() - ref).abs().max().item()
    tol = 2e-3 * ref.abs().max().item() + 1e-3
    assert err <= tol, f"path={path} shape={shape}: max err {err:.4g} > {tol:.4g}"
