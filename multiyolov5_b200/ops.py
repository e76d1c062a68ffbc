"""Per-op entry points of libmyolo_sm90a.so (kernel-level parity tests, ncu captures)."""
import ctypes

import torch

from . import _lib


def conv_bn_silu(x_nhwc: torch.Tensor, w: torch.Tensor, bn=None, bias=None, stride=1, dil=1, act=_lib.ACT_SILU, residual=None, path=0,
                 eps=1e-3, out=None, info=None):
    """x_nhwc: (B,H,W,Ci) fp16 CUDA; w: (Co,Ci,k,k) fp32 CUDA; bn: (gamma,beta,mean,var) fp32 or None.
    path: 0 auto, 1 wgmma (tensor cores), 2 CUDA-core, 3 wgmma with streamed weights (the reference layout for path 1's weight
    residency: same MMAs, same K order, bit-identical results).  out: optional (B,Ho,Wo,Co) fp16 channel slice of an NHWC buffer
    (out = buf[..., c0:c0 + Co]) to write into; it may be the residual itself.  info: optional list that receives the launch's
    routing, the 12 slots of myolo_plan_conv_info (slot 3 BN, slot 11 CTAs per SM).  Returns (B,Ho,Wo,Co) fp16."""
    assert x_nhwc.is_cuda and x_nhwc.dtype == torch.float16 and x_nhwc.is_contiguous()
    B, H, W, Ci = x_nhwc.shape
    Co, _, k, _ = w.shape
    pad = dil * (k // 2)
    Ho = (H + 2 * pad - dil * (k - 1) - 1) // stride + 1
    Wo = (W + 2 * pad - dil * (k - 1) - 1) // stride + 1
    if out is None:
        y = torch.empty((B, Ho, Wo, Co), dtype=torch.float16, device=x_nhwc.device)
    else:
        y = out
        ctot = y.stride(2)
        assert y.shape == (B, Ho, Wo, Co) and y.dtype == torch.float16 and y.stride() == (Ho * Wo * ctot, Wo * ctot, ctot, 1)
    w = w.float().contiguous()
    g = b = m = v = None
    if bn is not None:
        g, b, m, v = [t.float().contiguous() for t in bn]
    bias = bias.float().contiguous() if bias is not None else None
    if residual is not None:
        assert residual.shape == y.shape and residual.dtype == torch.float16 and residual.is_contiguous()
    slots = (ctypes.c_int32 * 12)()
    _lib.check(_lib.lib().myolo_conv_bn_silu_info(_lib.ptr(x_nhwc), B, H, W, Ci, _lib.ptr(w), Co, k, stride, dil, _lib.ptr(g),
                                                  _lib.ptr(b), _lib.ptr(m), _lib.ptr(v), float(eps), _lib.ptr(bias), int(act),
                                                  _lib.ptr(residual), _lib.ptr(y), y.stride(2), int(path), slots, _lib.stream_ptr()))
    if info is not None:
        info[:] = list(slots)
    return y
