"""Concat-free, BN-fused DenseNet dense block (the encoder of the K16 / N4 configs: torchvision `_DenseBlock`, i.e. the
`[BN -> ReLU -> 1x1 conv -> BN -> ReLU -> 3x3 conv -> concat]` chain of reference pytorch/bts.py:268-320 / SURVEY a11).

The reference (torch-eager) runs, per dense layer, a `cat` of all previous features, two BatchNorm kernels, two ReLU
kernels and two cuDNN convs forward, and the mirror image plus one `add` per consumer of every feature backward
(SURVEY 2.4: 104 cat, 1068 add kernels per step).  Here one autograd Function owns the whole block:

  forward   one NHWC slab holds every feature; each layer's 3x3 conv writes its 48 channels straight into its slice.
            Batch statistics of a feature are reduced ONCE, when it is produced (every later BN re-reads the same
            channel: same mean/var, different gamma/beta).  BN-apply + ReLU never run as kernels -- they are the
            A-operand prologue of the consuming wgmma conv (scale/shift per channel).
  backward  one gradient slab accumulates the concat fan-out in place (the BN+ReLU backward kernel writes `+=` into
            its channel range), dgrad / wgrad run on the tensor-core engine with the same fused prologue.

Parameters and buffers stay the torchvision modules' own (names, shapes, running-stat semantics: momentum, unbiased
running variance, num_batches_tracked), so checkpoints and bts_main.set_misc's name-based freezing are unaffected.
"""
import os

import torch

from . import _lib, conv, glue
from .ops import _ptr, _stream

EPI_STATS = True   # BatchNorm batch statistics reduced in the producing conv's epilogue (csrc/conv_tc.cu)


def _view(t):
    t2, s = conv._nhwc_view(t)
    if t2 is not t:
        raise ValueError("fused BN ops need NHWC-in-memory tensors")
    return t, s


# One-pass norm1 backward of a dense layer: the sums-independent part of dx is accumulated into the gradient slab by the
# reduce pass itself, the per-channel affine remainder is summed over layers in K and applied to each growth slice right
# before that slice is consumed (bts_bn_relu_bwd_fused / bts_bn_bwd_correct).  BTS_B200_BN_ONEPASS=0 -> reduce + apply.
BN_ONEPASS = os.environ.get("BTS_B200_BN_ONEPASS", "1") == "1"


def bn_relu_backward_onepass(x, g, st, out, K):
    """out += [y>0]*scale*g ; K += (k0, k1) (K None: frozen statistics); returns (S1, S2) fp64 [2,C]"""
    x, xs = _view(x)
    g, gs = _view(g)
    out, os_ = _view(out)
    B, C, H, W = x.shape
    M = B * H * W
    S = torch.empty((2, C), device=x.device, dtype=torch.float64)
    _lib.check(_lib.lib().bts_bn_relu_bwd_fused(_ptr(x), xs, _ptr(g), gs, M, C, _ptr(st[0]), _ptr(st[1]), _ptr(st[2]),
                                                _ptr(st[3]), _ptr(S[0]), _ptr(S[1]), _ptr(out), os_,
                                                _ptr(K[0]) if K is not None else None,
                                                _ptr(K[1]) if K is not None else None, _stream()), "bts_bn_relu_bwd_fused")
    _lib.count(2 if K is not None else 1)
    return S


def bn_backward_correct(x, K, out):
    """out += K[1]*x + K[0] per channel (the deferred remainder of the one-pass BatchNorm backward)"""
    x, xs = _view(x)
    out, os_ = _view(out)
    B, C, H, W = x.shape
    _lib.check(_lib.lib().bts_bn_bwd_correct(_ptr(x), xs, B * H * W, C, _ptr(K[0]), _ptr(K[1]), _ptr(out), os_, _stream()),
               "bts_bn_bwd_correct")
    _lib.count()


# BatchNorm-backward sums reduced in the dgrad epilogue (bts_conv_fwd with x_bn / bn_st) instead of a separate pass.  The
# epilogue already paces the short-K dgrads, and the fused form adds strided reads of x and of the per-channel parameters
# to it, so the separate streaming reduce pass is the default; the fused form stays available (and tested) for long-K
# layers.
EPI_BNBWD = os.environ.get("BTS_B200_EPI_BNBWD", "0") == "1"


def bn_relu_backward_from_sums(x, g, st, S, use_stats, out, accumulate):
    """the apply half of glue.bn_backward(act=1) when S = (S1, S2) already came out of the dgrad epilogue"""
    x, xs = _view(x)
    g, gs = _view(g)
    out, os_ = _view(out)
    B, C, H, W = x.shape
    M = B * H * W
    L = _lib.lib()
    coef = None
    if use_stats:
        coef = torch.empty((2, C), device=x.device, dtype=torch.float32)
        _lib.check(L.bts_bn_bwd_coef(_ptr(S[0]), _ptr(S[1]), M, C, _ptr(st[0]), _ptr(st[2]), _ptr(st[3]), _ptr(coef), _stream()),
                   "bts_bn_bwd_coef")
    _lib.check(L.bts_bn_bwd_apply(_ptr(x), xs, _ptr(g), gs, M, C, _ptr(st[0]), _ptr(st[1]), _ptr(coef), 1, _ptr(out), os_,
                                  int(accumulate), _stream()), "bts_bn_bwd_apply")
    _lib.count(2)
    return S


def dgrad_bn_relu_backward(gy, weight, padding, dilation, x_bn, st, use_stats, out=None, accumulate=False):
    """d/dx_bn of conv(relu(bn(x_bn))) given gy = d/d(conv output): dgrad on the engine with the BatchNorm-backward sums
    reduced in its epilogue, then one streaming apply pass.  Returns (dx, S) with S = (dbeta, dgamma) as fp64 [2,C]."""
    KH = weight.shape[2]
    C = weight.shape[1]
    S = torch.zeros((2, C), device=gy.device, dtype=torch.float64)
    g_a = conv.conv2d_tc(gy, weight, 1, dilation * (KH - 1) - padding, dilation, transpose_flip=True, stats=S,
                         bn_bwd=(x_bn, st, True))
    if out is None:
        out = g_a
    bn_relu_backward_from_sums(x_bn, g_a, st, S, use_stats, out, accumulate)
    return out, S


class _DenseBlockFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, block, training, *params):
        layers = list(block.children())
        B, C0, H, W = x.shape
        growth = layers[0].conv2.out_channels
        Ct = C0 + growth * len(layers)
        n = B * H * W
        slab = torch.empty((B, Ct, H, W), device=x.device, dtype=torch.float32, memory_format=torch.channels_last)
        slab[:, :C0].copy_(x)
        sums = torch.empty((2, Ct), device=x.device, dtype=torch.float64)
        if training:
            sums[:, :C0] = glue.bn_stats(slab[:, :C0])
        saved_b, saved_st = [], []
        C = C0
        # the zeroed [2, C] accumulators of the epilogue statistics of every layer, carved out of ONE zero fill
        zoff = [0]
        zbuf = torch.zeros(2 * sum(params[6 * li + 2].shape[0] + growth for li in range(len(layers))), device=x.device,
                           dtype=torch.float64) if training else None

        def zeros2(c):
            v = zbuf[zoff[0]:zoff[0] + 2 * c].view(2, c)
            zoff[0] += 2 * c
            return v

        for li, layer in enumerate(layers):
            w1, w2 = params[6 * li + 2], params[6 * li + 5]
            bn1, bn2 = layer.norm1, layer.norm2
            st1 = glue.bn_finalize(sums[:, :C] if training else None, n, bn1, bn1.weight, bn1.bias, training)
            epi = training and EPI_STATS and w1.shape[0] <= 256 and growth <= 256
            sb = zeros2(w1.shape[0]) if epi else None
            b = conv.conv2d_tc(slab[:, :C], w1, 1, 0, 1, pre_scale=st1[0], pre_shift=st1[1], pre_relu=True, stats=sb)
            st2 = glue.bn_finalize((sb if epi else glue.bn_stats(b)) if training else None, n, bn2, bn2.weight, bn2.bias,
                                   training)
            more = training and li + 1 < len(layers)
            sn = zeros2(growth) if (epi and more) else None
            conv.conv2d_tc(b, w2, 1, 1, 1, pre_scale=st2[0], pre_shift=st2[1], pre_relu=True, out=slab[:, C:C + growth],
                           stats=sn)
            if more:
                sums[:, C:C + growth] = sn if sn is not None else glue.bn_stats(slab[:, C:C + growth])
            saved_b.append(b)
            saved_st += [st1, st2]
            C += growth
        ctx.block, ctx.training, ctx.C0, ctx.growth = block, training, C0, growth
        ctx.nl = len(layers)
        ctx.save_for_backward(slab, *saved_b, *saved_st, *params)
        return slab

    @staticmethod
    def backward(ctx, gout):
        nl, C0, growth, training = ctx.nl, ctx.C0, ctx.growth, ctx.training
        sv = ctx.saved_tensors
        slab = sv[0]
        bs = sv[1:1 + nl]
        sts = sv[1 + nl:1 + 3 * nl]
        params = sv[1 + 3 * nl:]
        G = gout.clone(memory_format=torch.channels_last)      # owned: the concat fan-out accumulates into it in place
        grads = [None] * len(params)
        need = ctx.needs_input_grad[3:]
        onepass = BN_ONEPASS and not EPI_BNBWD
        K = torch.zeros((2, slab.shape[1]), device=slab.device, dtype=torch.float64) if (onepass and training) else None
        for li in reversed(range(nl)):
            C = C0 + growth * li
            g1, b1, w1, g2, b2, w2 = params[6 * li:6 * li + 6]
            st1, st2 = sts[2 * li], sts[2 * li + 1]
            b = bs[li]
            g_out = G[:, C:C + growth]
            if K is not None and li + 1 < nl:
                # every later layer read these channels: their deferred k1*x + k0 terms land now, before g_out is used
                bn_backward_correct(slab[:, C:C + growth], K[:, C:C + growth], g_out)
            # ---- conv2 (3x3) backward
            if need[6 * li + 5]:
                grads[6 * li + 5] = conv.wgrad_tc(b, g_out, w2.shape, w2.stride(), 1, 1, 1, pre_scale=st2[0],
                                                  pre_shift=st2[1], pre_relu=True)
            if EPI_BNBWD:
                g_a2, S = dgrad_bn_relu_backward(g_out, w2, 1, 1, b, st2, training)        # sums in the dgrad epilogue
            else:
                g_a2 = conv.conv2d_tc(g_out, w2, 1, 1, 1, transpose_flip=True)
                # ---- norm2 + relu2 backward (in place on g_a2)
                _, S = glue.bn_backward(b, g_a2, st2, training, 1, out=g_a2)
            if need[6 * li + 3]:
                grads[6 * li + 3] = S[1].float()
            if need[6 * li + 4]:
                grads[6 * li + 4] = S[0].float()
            # ---- conv1 (1x1) backward
            xin = slab[:, :C]
            if need[6 * li + 2]:
                grads[6 * li + 2] = conv.wgrad_tc(xin, g_a2, w1.shape, w1.stride(), 1, 0, 1, pre_scale=st1[0],
                                                  pre_shift=st1[1], pre_relu=True)
            # ---- norm1 + relu1 backward, accumulated into the gradient slab (the concat fan-out)
            if EPI_BNBWD:
                _, S = dgrad_bn_relu_backward(g_a2, w1, 0, 1, xin, st1, training, out=G[:, :C], accumulate=True)
            else:
                g_a1 = conv.conv2d_tc(g_a2, w1, 1, 0, 1, transpose_flip=True)
                if onepass:
                    S = bn_relu_backward_onepass(xin, g_a1, st1, G[:, :C], K)
                else:
                    _, S = glue.bn_backward(xin, g_a1, st1, training, 1, out=G[:, :C], accumulate=True)
            if need[6 * li + 0]:
                grads[6 * li + 0] = S[1].float()
            if need[6 * li + 1]:
                grads[6 * li + 1] = S[0].float()
        if K is not None and ctx.needs_input_grad[0]:
            bn_backward_correct(slab[:, :C0], K[:, :C0], G[:, :C0])
        gx = G[:, :C0] if ctx.needs_input_grad[0] else None
        return (gx, None, None) + tuple(grads)


def dense_block_forward(block, x):
    """drop-in for torchvision `_DenseBlock.forward` (returns the concatenated feature slab)"""
    params = []
    for layer in block.children():
        params += [layer.norm1.weight, layer.norm1.bias, layer.conv1.weight, layer.norm2.weight, layer.norm2.bias,
                   layer.conv2.weight]
    return _DenseBlockFn.apply(x, block, block.training, *params)


def dense_block_eligible(block, x):
    if not (x.is_cuda and x.dtype == torch.float32 and x.dim() == 4):
        return False
    for layer in block.children():
        ok = (hasattr(layer, "norm1") and hasattr(layer, "conv2") and layer.conv1.kernel_size == (1, 1)
              and layer.conv2.kernel_size == (3, 3) and layer.conv2.padding == (1, 1) and layer.conv1.bias is None
              and layer.conv2.bias is None and float(getattr(layer, "drop_rate", 0.0)) == 0.0
              and layer.norm1.affine and layer.norm2.affine and layer.norm1.track_running_stats
              and layer.norm2.track_running_stats)
        if not ok:
            return False
        if layer.norm1.training != block.training or layer.norm2.training != block.training:
            return False          # e.g. bn_init_as_tf froze some BNs: keep the unfused path
    return True
