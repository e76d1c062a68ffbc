"""Per-op entry points of libmyolo_sm90a.so (kernel-level parity tests, ncu captures)."""
import ctypes

import torch

from . import _lib


def conv_forward(x, w, y, bn=None, bias=None, residual=None, x_off=0, y_off=0, res_off=0, stride=1, dil=1, act=_lib.ACT_SILU, path=0,
                 eps=1e-3):
    """The plan's forward of one conv (csrc/plan.cu conv_forward_views) on channel slices of NHWC CUDA buffers.
    x: (B,H,W,ctot) fp16 / fp32 buffer whose channels [x_off, x_off + ci16) are the input (ci16: ci rounded up to 16, zero padding);
    y: (B,Ho,Wo,ctot) fp16 / fp32 buffer, y[..., y_off:y_off + co] = act(conv + bias) (+ residual[..., res_off:res_off + co]); residual:
    None or an fp16 (B,Ho,Wo,ctot) buffer, y itself allowed.  w: (co,ci,k,k) fp32 masters; bn: (gamma,beta,mean,var) fp32 folded in with
    eps, or None; bias: (co,) fp32 or None.  path: 0 as the plan, 1 wgmma, 2 CUDA-core, 3 wgmma with streamed weights.  Returns the 12 info
    slots of myolo_plan_conv_info: the route taken and its tiling."""
    for t in (x, y, residual):
        assert t is None or (t.is_cuda and t.is_contiguous() and t.dim() == 4 and t.dtype in (torch.float16, torch.float32))
    assert residual is None or (residual.dtype == torch.float16 and residual.shape[:3] == y.shape[:3])
    co, ci, k, _ = w.shape
    B, H, W = x.shape[:3]
    w = w.float().contiguous()
    g = b = m = v = None
    if bn is not None:
        g, b, m, v = [t.float().contiguous() for t in bn]
    bias = bias.float().contiguous() if bias is not None else None
    slots = (ctypes.c_int32 * 12)()
    _lib.check(_lib.lib().myolo_conv_forward(_lib.ptr(x), _lib.torch_dtype_code(x.dtype), B, H, W, x.shape[3], x_off, _lib.ptr(y),
                                             _lib.torch_dtype_code(y.dtype), y.shape[3], y_off, _lib.ptr(residual),
                                             residual.shape[3] if residual is not None else 0, res_off, _lib.ptr(w), co, ci, k, stride, dil,
                                             _lib.ptr(g), _lib.ptr(b), _lib.ptr(m), _lib.ptr(v), float(eps), _lib.ptr(bias), int(act), int(path),
                                             slots, _lib.stream_ptr()))
    return list(slots)


def conv_backward(x, w, dy, dW, gin=None, dbias=None, x_off=0, dy_off=0, gin_off=0, stride=1, dil=1, route=0):
    """The train plan's backward of one conv (csrc/plan.cu conv_backward_views) on channel slices of NHWC CUDA buffers.
    x: (B,H,W,ctot) fp16 / fp32 buffer whose channels [x_off, x_off + ci16) are the input (ci16: ci rounded up to 16, zero padding);
    dy: (B,Ho,Wo,ctot) buffer holding dL/dy at [dy_off, dy_off + co) in fp16, or at [dy_off, dy_off + co16) in fp32 (zero padding);
    gin: None or x's twin buffer, grad(in) += at [gin_off, gin_off + ci16); w: (co,ci,k,k) fp32 master weights; dW (same shape) and
    dbias (co,) fp32 are accumulated into.  route: 0 as the plan, or _lib.CONV_BWD_* bits.  Returns the 16 info slots of
    myolo_conv_backward (include/myolo.h): the routes taken and their tiling."""
    B, H, W, _ = x.shape
    co, ci, k, _ = w.shape
    for t in (x, dy, gin):
        assert t is None or (t.is_cuda and t.is_contiguous() and t.dtype in (torch.float16, torch.float32))
    pad = dil * (k // 2)
    Ho, Wo = (H + 2 * pad - dil * (k - 1) - 1) // stride + 1, (W + 2 * pad - dil * (k - 1) - 1) // stride + 1
    assert dy.shape[:3] == (B, Ho, Wo), (dy.shape, (B, Ho, Wo))
    assert gin is None or (gin.shape == x.shape and gin.dtype == x.dtype)
    assert w.dtype == dW.dtype == torch.float32 and w.is_contiguous() and dW.is_contiguous() and dW.shape == w.shape
    assert dbias is None or (dbias.dtype == torch.float32 and dbias.shape == (co,))
    slots = (ctypes.c_int32 * 16)()
    _lib.check(_lib.lib().myolo_conv_backward(_lib.ptr(x), _lib.torch_dtype_code(x.dtype), B, H, W, x.shape[3], x_off, _lib.ptr(dy),
                                              _lib.torch_dtype_code(dy.dtype), dy.shape[3], dy_off, _lib.ptr(gin), x.shape[3], gin_off,
                                              _lib.ptr(w), co, ci, k, stride, dil, _lib.ptr(dW), _lib.ptr(dbias), int(route), slots,
                                              _lib.stream_ptr()))
    return list(slots)
