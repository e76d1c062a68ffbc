"""GPU: the wgmma conv kernel with resident weights, strip A loads for 3x3 stride-1 layers and the residual loads issued ahead of the
epilogue (path 1) against the same kernel with streamed weights and one A box per tap (path 3), bit for bit: both paths run the same
MMAs in the same K order, so any difference is a layout or synchronisation bug.  Also pins which launches of the s/PSP forward keep
their weights resident and take the strip, so that a silent fallback fails here."""
import pytest
import torch

pytestmark = pytest.mark.gpu

SMEM_BUDGET = 227 * 1024
RESIDENT_LIMIT = SMEM_BUDGET - (1024 + 8192 + 1024) - 6 * 128 * 64 * 2   # misc + six A stages (conv_tc.cu)

# (B, H, W, Ci, Co, k, stride, dil, residual)
SHAPES = [
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


@pytest.mark.parametrize("shape", SHAPES, ids=[f"{s[3]}-{s[4]}-k{s[5]}s{s[6]}d{s[7]}-{s[0]}x{s[1]}x{s[2]}{'-res' if s[8] else ''}"
                                                for s in SHAPES])
def test_reuse_matches_streamed_bit_for_bit(shape):
    from multiyolov5_b200 import ops
    B, H, W, Ci, Co, k, s, d, res = shape
    g = torch.Generator().manual_seed(1000 + SHAPES.index(shape))
    x = torch.randn(B, H, W, Ci, generator=g).half().cuda()
    w = (torch.randn(Co, Ci, k, k, generator=g) * (2.0 / (Ci * k * k)) ** 0.5).cuda()
    bn = [torch.rand(Co, generator=g) * 0.4 + 0.8, torch.randn(Co, generator=g) * 0.1, torch.randn(Co, generator=g) * 0.1,
          torch.rand(Co, generator=g) + 0.5]
    bn = [t.cuda() for t in bn]
    Ho = (H + 2 * d * (k // 2) - d * (k - 1) - 1) // s + 1
    Wo = (W + 2 * d * (k // 2) - d * (k - 1) - 1) // s + 1
    r = torch.randn(B, Ho, Wo, Co, generator=g).half().cuda() if res else None
    y1 = ops.conv_bn_silu(x, w, bn, stride=s, dil=d, residual=r, path=1)
    y3 = ops.conv_bn_silu(x, w, bn, stride=s, dil=d, residual=r, path=3)
    torch.cuda.synchronize()
    assert torch.isfinite(y3.float()).all()
    assert torch.equal(y1.view(torch.int16), y3.view(torch.int16)), \
        f"{shape}: {(y1 != y3).sum().item()} outputs differ, max {(y1.float() - y3.float()).abs().max().item():.4g}"


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
