"""Depthwise 3x3 convolution on the CUDA-core kernels of csrc/dwconv.cu (torchvision mobilenet_v2's groups == C layers
behind reference pytorch/bts.py:297-300): NHWC fp32, pad 1, stride 1 or 2, no bias, C % 4 == 0.

  fwd    y = dw(pre(x)), pre = relu6(x*scale + shift) (a BatchNorm + ReLU6 folded into the staging of the input window),
         optionally with the BatchNorm statistics of y or the eval-mode epilogue relu6(y*scale + shift)
  dgrad  dx from dy (stride 2: only the taps that land, no zero-stuffed dy)
  wgrad  dW from (x, dy), the prologue recomputed from the raw x
"""
import torch

from . import _lib
from .conv import _nhwc_view
from .ops import _ptr, _stream


def eligible(conv):
    """True for an nn.Conv2d the kernels take: depthwise 3x3, pad 1, dilation 1, stride 1 or 2, no bias, C % 4 == 0"""
    C = conv.in_channels
    return (conv.groups == C and conv.out_channels == C and C % 4 == 0 and tuple(conv.kernel_size) == (3, 3)
            and tuple(conv.padding) == (1, 1) and tuple(conv.dilation) == (1, 1) and conv.stride[0] == conv.stride[1]
            and conv.stride[0] in (1, 2) and conv.bias is None and conv.padding_mode == "zeros")


def _quad_view(t):
    """NHWC view whose pixel rows start on 16-byte boundaries (one copy when t is not laid out that way)"""
    t, ts = _nhwc_view(t)
    if ts % 4 or t.data_ptr() % 16:
        t = t.contiguous(memory_format=torch.channels_last)
        ts = t.shape[1]
    return t, ts


def _out_hw(H, W, stride):
    return (H - 1) // stride + 1, (W - 1) // stride + 1


def fwd(x, weight, stride, pre=None, post=None, stats=False):
    """y = dw(pre(x)) [-> relu6(y*post[0] + post[1])]; pre = (scale, shift) of a BatchNorm followed by ReLU6.
    Returns y, or (y, sums) with sums = fp64 [2, C] (sum, sum of squares of y) when `stats`."""
    x, xs = _quad_view(x)
    B, C, H, W = x.shape
    Ho, Wo = _out_hw(H, W, stride)
    y = torch.empty((B, C, Ho, Wo), device=x.device, dtype=torch.float32, memory_format=torch.channels_last)
    L = _lib.lib()
    sums = ws = None
    if stats:
        sums = torch.empty((2, C), device=x.device, dtype=torch.float64)
        n = L.bts_dw3x3_fwd_workspace_floats(B, H, W, C, stride)
        if n < 0:
            _lib.check(int(n), "bts_dw3x3_fwd_workspace_floats")
        ws = torch.empty(n, device=x.device, dtype=torch.float32)
    psc, psh = (pre[0].contiguous(), pre[1].contiguous()) if pre is not None else (None, None)
    esc, esh = (post[0].contiguous(), post[1].contiguous()) if post is not None else (None, None)
    s = weight.stride()
    _lib.check(L.bts_dw3x3_fwd(_ptr(x), xs, B, H, W, C, stride, _ptr(weight), s[0], s[2], s[3], _ptr(psc), _ptr(psh),
                               _ptr(esc), _ptr(esh), _ptr(y), C, _ptr(sums[0]) if stats else None,
                               _ptr(sums[1]) if stats else None, _ptr(ws), _stream()), "bts_dw3x3_fwd")
    _lib.count(2 if stats else 1)
    return (y, sums) if stats else y


def dgrad(dy, weight, stride, H, W):
    """dx (B, C, H, W) of the depthwise conv whose input was H x W"""
    dy, dys = _quad_view(dy)
    B, C = dy.shape[:2]
    dx = torch.empty((B, C, H, W), device=dy.device, dtype=torch.float32, memory_format=torch.channels_last)
    s = weight.stride()
    _lib.check(_lib.lib().bts_dw3x3_dgrad(_ptr(dy), dys, B, H, W, C, stride, _ptr(weight), s[0], s[2], s[3], _ptr(dx), C,
                                          _stream()), "bts_dw3x3_dgrad")
    _lib.count()
    return dx


def wgrad(x, dy, weight, stride, pre=None):
    """dW, shaped and strided like `weight`; pre = (scale, shift) recomputes relu6(x*scale + shift) from the raw x"""
    x, xs = _quad_view(x)
    dy, dys = _quad_view(dy)
    B, C, H, W = x.shape
    L = _lib.lib()
    n = L.bts_dw3x3_wgrad_workspace_floats(B, H, W, C, stride)
    if n < 0:
        _lib.check(int(n), "bts_dw3x3_wgrad_workspace_floats")
    ws = torch.empty(n, device=x.device, dtype=torch.float32)
    gw = torch.empty_strided(tuple(weight.shape), tuple(weight.stride()), device=x.device, dtype=torch.float32)
    psc, psh = (pre[0].contiguous(), pre[1].contiguous()) if pre is not None else (None, None)
    s = weight.stride()
    _lib.check(L.bts_dw3x3_wgrad(_ptr(x), xs, _ptr(dy), dys, B, H, W, C, stride, _ptr(psc), _ptr(psh), _ptr(ws), _ptr(gw),
                                 s[0], s[2], s[3], _stream()), "bts_dw3x3_wgrad")
    _lib.count(2)
    return gw


class _DwConv(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, weight, stride):
        ctx.stride = stride
        ctx.save_for_backward(x, weight)
        return fwd(x, weight, stride)

    @staticmethod
    def backward(ctx, gy):
        x, weight = ctx.saved_tensors
        gx = dgrad(gy, weight, ctx.stride, x.shape[2], x.shape[3]) if ctx.needs_input_grad[0] else None
        gw = wgrad(x, gy, weight, ctx.stride) if ctx.needs_input_grad[1] else None
        return gx, gw, None


def conv(x, weight, stride):
    """a plain depthwise 3x3 / pad 1 convolution with autograd, all three passes on the kernels above"""
    return _DwConv.apply(x, weight, int(stride))
