"""Composable fused autograd units for the BTS decoder and the encoder's non-dense-block stages (SURVEY 8a rows a5-a10,
a11 transitions/stem).  The reference (torch-eager, pytorch/bts.py:196-266) runs every BatchNorm, ReLU, ELU, nearest
up-sample and torch.cat as its own ATen/cuDNN kernel, forward and backward; here they are either folded into the wgmma
conv engine (ELU in the epilogue, ReLU / BN-apply + ReLU in the A-operand prologue, the x2 up-sample in the im2col map) or
run as one of the streaming NHWC kernels of csrc/elem.cu / csrc/bn.cu:

  conv_act       y = act(conv(pre_relu?(up2?(x))))        upconv (bts.py:69-80), iconvs (:156-192), reduction chains (:83-108)
  bn_act         y = BN(x) [ReLU | ReLU6]                  decoder BNs (:154-182), torchvision norm0(+relu0) / norm5,
                                                           mobilenet_v2's stem and last Conv2dNormActivation
  bn_relu_conv   y = conv(ReLU(BN(x)))                     atrous_conv halves (:51-66), DenseNet transitions
  cat_nhwc       channel concat into a 16-byte-aligned slab (the nine torch.cat of bts.forward); backward = views
  avgpool2       2x2 average pool of the transitions
  inverted_residual  one torchvision InvertedResidual (mobilenet_v2, bts.py:297-300) as a single Function: 1x1 expand
                 with BN1 statistics from the engine epilogue, depthwise 3x3 with BN1 + ReLU6 in its prologue and BN2
                 statistics in its epilogue (csrc/dwconv.cu), BN2 + ReLU6, 1x1 project, BN3 [+ residual]

Each unit is a torch.autograd.Function whose backward launches our kernels too (ELU', BN reductions, wgrad / dgrad on
the engine, 2x2 gradient fold of the up-sample).  Parameters stay the nn.Modules' own, BatchNorm running statistics are
updated with nn.BatchNorm2d semantics (momentum, unbiased variance, num_batches_tracked).
"""
import torch

from . import _lib, conv
from .ops import _ptr, _stream


def eligible(x):
    return x.is_cuda and x.dtype == torch.float32 and x.dim() == 4


def _nhwc(t):
    """(tensor, pixel stride) with NHWC memory; converts (one copy) when the layout is something else"""
    return conv._nhwc_view(t)


def _new(B, C, H, W, dev):
    return torch.empty((B, C, H, W), device=dev, dtype=torch.float32, memory_format=torch.channels_last)


# ------------------------------------------------------------------------------------------------ raw kernel wrappers
def bn_stats(x):
    x, xs = _nhwc(x)
    B, C, H, W = x.shape
    out = torch.empty((2, C), device=x.device, dtype=torch.float64)
    _lib.check(_lib.lib().bts_bn_stats(_ptr(x), xs, B * H * W, C, _ptr(out[0]), _ptr(out[1]), _stream()), "bts_bn_stats")
    _lib.count()
    return out


def bn_finalize(sums, n, bn, gamma, beta, training):
    """(scale, shift, mean, invstd) as a [4,C] tensor; in training also the module's running-stat update"""
    C = bn.num_features
    out = torch.empty((4, C), device=bn.running_mean.device if bn.running_mean is not None else gamma.device,
                      dtype=torch.float32)
    L = _lib.lib()
    g = gamma.detach() if gamma is not None else None
    b = beta.detach() if beta is not None else None
    if training:
        track = bn.track_running_stats and bn.running_mean is not None
        mom = bn.momentum if bn.momentum is not None else 0.1
        nbt = bn.num_batches_tracked if (track and bn.num_batches_tracked is not None) else None
        _lib.check(L.bts_bn_finalize_track(_ptr(sums[0]), _ptr(sums[1]), n, C, _ptr(g), _ptr(b), float(bn.eps), float(mom),
                                           _ptr(bn.running_mean) if track else None, _ptr(bn.running_var) if track else None,
                                           _ptr(nbt), _ptr(out[0]), _ptr(out[1]), _ptr(out[2]), _ptr(out[3]), _stream()),
                   "bts_bn_finalize_track")
    else:
        _lib.check(L.bts_bn_fold(C, _ptr(g), _ptr(b), float(bn.eps), _ptr(bn.running_mean), _ptr(bn.running_var),
                                 _ptr(out[0]), _ptr(out[1]), _ptr(out[2]), _ptr(out[3]), _stream()), "bts_bn_fold")
    _lib.count()
    return out


def bn_uses_batch_stats(bn):
    """nn.BatchNorm2d: batch statistics in train mode, or whenever no running statistics are tracked"""
    return bn.training or bn.running_mean is None


def bn_backward(x, g, st, use_stats, act, out=None, accumulate=False):
    """d/dx of act(bn(x)) given g = d/d(output), activation code `act`: 0 none, 1 ReLU, 2 ReLU6 (a bool is 0 / 1);
    returns (dx, S) with S = (dbeta, dgamma) as fp64 [2,C]"""
    x, xs = _nhwc(x)
    g, gs = _nhwc(g)
    B, C, H, W = x.shape
    if out is None:
        out = _new(B, C, H, W, x.device)
    o2, os_ = _nhwc(out)
    if o2 is not out:
        raise ValueError("bn_backward: out must be NHWC in memory")
    M = B * H * W
    L = _lib.lib()
    S = torch.empty((2, C), device=x.device, dtype=torch.float64)
    coef = torch.empty((2, C), device=x.device, dtype=torch.float32)
    _lib.check(L.bts_bn_bwd_reduce(_ptr(x), xs, _ptr(g), gs, M, C, _ptr(st[0]), _ptr(st[1]), _ptr(st[2]), _ptr(st[3]),
                                   int(act), _ptr(S[0]), _ptr(S[1]), _ptr(coef), _stream()), "bts_bn_bwd_reduce")
    _lib.check(L.bts_bn_bwd_apply(_ptr(x), xs, _ptr(g), gs, M, C, _ptr(st[0]), _ptr(st[1]),
                                  _ptr(coef) if use_stats else None, int(act), _ptr(out), os_, int(accumulate), _stream()),
               "bts_bn_bwd_apply")
    _lib.count(3)
    return out, S


def copy_channels(src, dst, accumulate=False):
    s, ss = _nhwc(src)
    d, ds = _nhwc(dst)
    if d is not dst:
        raise ValueError("copy_channels: dst must be NHWC in memory")
    B, C, H, W = s.shape
    _lib.check(_lib.lib().bts_copy_channels(_ptr(s), ss, B * H * W, C, _ptr(d), ds, int(accumulate), _stream()),
               "bts_copy_channels")
    _lib.count()


# ------------------------------------------------------------------------------------------------ conv (+ pre / act)
class _ConvAct(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, weight, padding, dilation, pre_relu, up, act):
        y = conv.conv2d_tc(x, weight, 1, padding, dilation, pre_relu=pre_relu, upsample2=up, act=act)
        ctx.cfg = (padding, dilation, pre_relu, up, act)
        ctx.save_for_backward(x, weight, y if act == "elu" else None)
        return y

    @staticmethod
    def backward(ctx, gy):
        x, weight, y = ctx.saved_tensors
        padding, dilation, pre_relu, up, act = ctx.cfg
        L = _lib.lib()
        g, gs = _nhwc(gy)
        B, Co, Ho, Wo = g.shape
        if act == "elu":
            ge = _new(B, Co, Ho, Wo, g.device)
            y2, ys = _nhwc(y)
            _lib.check(L.bts_elu_bwd(_ptr(g), gs, _ptr(y2), ys, B * Ho * Wo, Co, _ptr(ge), Co, _stream()), "bts_elu_bwd")
            _lib.count()
            g = ge
        elif act is not None:
            raise RuntimeError("conv_act backward supports act in (None, 'elu')")
        gx = gw = None
        KH = weight.shape[2]
        if ctx.needs_input_grad[1]:
            gw = conv.wgrad_tc(x, g, weight.shape, weight.stride(), 1, padding, dilation, pre_relu=pre_relu, upsample2=up)
        if ctx.needs_input_grad[0]:
            Ci = weight.shape[1]
            out = None
            if Ci % 4:        # keep the gradient's pixel rows 16-byte aligned (concat3 = 225, concat2 = 161 channels)
                Hf, Wf = (2 * x.shape[2], 2 * x.shape[3]) if up else (x.shape[2], x.shape[3])
                out = _new(x.shape[0], (Ci + 3) // 4 * 4, Hf, Wf, g.device)[:, :Ci]
            full = conv.conv2d_tc(g, weight, 1, dilation * (KH - 1) - padding, dilation, transpose_flip=True, out=out)
            if up:
                x2, xs = _nhwc(x)
                Bx, Ci, Hs, Ws = x2.shape
                gx = _new(Bx, Ci, Hs, Ws, g.device)
                full, fs = _nhwc(full)
                _lib.check(L.bts_upsample2_sum(_ptr(full), fs, Bx, Hs, Ws, Ci, _ptr(x2) if pre_relu else None, xs,
                                               _ptr(gx), Ci, _stream()), "bts_upsample2_sum")
                _lib.count()
            elif pre_relu:
                gx = torch.where(x > 0, full, torch.zeros((), device=full.device))
            else:
                gx = full
        return gx, gw, None, None, None, None, None


def conv_act(x, weight, padding=0, dilation=1, pre_relu=False, up=False, act=None):
    """act(conv2d(pre_relu ? relu(x) : x, nearest-x2 up-sampled when `up`)), stride 1, all three GEMMs on the engine"""
    return _ConvAct.apply(x, weight, int(padding), int(dilation), bool(pre_relu), bool(up), act)


# ------------------------------------------------------------------------------------------------ BatchNorm (+ ReLU)
class _BnAct(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, gamma, beta, bn, act):
        x, xs = _nhwc(x)
        B, C, H, W = x.shape
        n = B * H * W
        batch = bn_uses_batch_stats(bn)
        st = bn_finalize(bn_stats(x) if batch else None, n, bn, gamma, beta, batch)
        y = _new(B, C, H, W, x.device)
        _lib.check(_lib.lib().bts_bn_apply(_ptr(x), xs, n, C, _ptr(st[0]), _ptr(st[1]), act, _ptr(y), C, _stream()),
                   "bts_bn_apply")
        _lib.count()
        ctx.cfg = (batch, act)
        ctx.save_for_backward(x, st)
        return y

    @staticmethod
    def backward(ctx, gy):
        x, st = ctx.saved_tensors
        batch, act = ctx.cfg
        gx, S = bn_backward(x, gy, st, batch, act)
        return (gx if ctx.needs_input_grad[0] else None, S[1].float() if ctx.needs_input_grad[1] else None,
                S[0].float() if ctx.needs_input_grad[2] else None, None, None)


ACT_CODES = {None: 0, "relu": 1, "relu6": 2}


def bn_act(x, bn, relu=False, act=None):
    """nn.BatchNorm2d `bn` applied to x (batch statistics + running-stat update in train mode, folded running
    statistics in eval mode), followed by the activation `act` (None, "relu" or "relu6") -- 3 streaming kernels forward,
    3 backward.  `relu=True` is the older spelling of act="relu" that the ResNet / DenseNet callers use."""
    if relu and act not in (None, "relu"):
        raise ValueError("bn_act: relu=True contradicts act=%r" % (act,))
    return _BnAct.apply(x, bn.weight, bn.bias, bn, ACT_CODES["relu" if relu else act])


# ------------------------------------------------------------------------------------------------ BN -> ReLU -> conv
class _BnReluConv(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, gamma, beta, weight, bn, padding, dilation):
        x, _ = _nhwc(x)
        B, C, H, W = x.shape
        n = B * H * W
        batch = bn_uses_batch_stats(bn)
        st = bn_finalize(bn_stats(x) if batch else None, n, bn, gamma, beta, batch)
        y = conv.conv2d_tc(x, weight, 1, padding, dilation, pre_scale=st[0], pre_shift=st[1], pre_relu=True)
        ctx.cfg = (padding, dilation, batch)
        ctx.save_for_backward(x, weight, st)
        return y

    @staticmethod
    def backward(ctx, gy):
        x, weight, st = ctx.saved_tensors
        padding, dilation, batch = ctx.cfg
        KH = weight.shape[2]
        gw = None
        if ctx.needs_input_grad[3]:
            gw = conv.wgrad_tc(x, gy, weight.shape, weight.stride(), 1, padding, dilation, pre_scale=st[0], pre_shift=st[1],
                               pre_relu=True)
        from . import fused
        if fused.EPI_BNBWD:
            gx, S = fused.dgrad_bn_relu_backward(gy, weight, padding, dilation, x, st, batch)   # sums in the dgrad epilogue
        else:
            g_a = conv.conv2d_tc(gy, weight, 1, dilation * (KH - 1) - padding, dilation, transpose_flip=True)
            gx, S = bn_backward(x, g_a, st, batch, True, out=g_a)          # in place on the dgrad result
        return (gx if ctx.needs_input_grad[0] else None, S[1].float() if ctx.needs_input_grad[1] else None,
                S[0].float() if ctx.needs_input_grad[2] else None, gw, None, None, None)


def bn_relu_conv(x, bn, weight, padding=0, dilation=1):
    """conv2d(relu(bn(x))): the normalisation + ReLU run inside the conv's A-operand prologue (never materialised)"""
    return _BnReluConv.apply(x, bn.weight, bn.bias, weight, bn, int(padding), int(dilation))


# ------------------------------------------------------------------------------------------------ concat
class _CatNHWC(torch.autograd.Function):
    @staticmethod
    def forward(ctx, *ts):
        B, _, H, W = ts[0].shape
        cs = [int(t.shape[1]) for t in ts]
        C = sum(cs)
        Cp = (C + 3) // 4 * 4
        slab = _new(B, Cp, H, W, ts[0].device)
        off = 0
        for t, c in zip(ts, cs):
            copy_channels(t, slab[:, off:off + c])
            off += c
        if Cp != C:
            _lib.check(_lib.lib().bts_zero_channels(_ptr(slab), Cp, B * H * W, C, Cp, _stream()), "bts_zero_channels")
            _lib.count()
        ctx.cs = cs
        return slab[:, :C] if Cp != C else slab

    @staticmethod
    def backward(ctx, g):
        out, off = [], 0
        for i, c in enumerate(ctx.cs):
            out.append(g[:, off:off + c] if ctx.needs_input_grad[i] else None)
            off += c
        return tuple(out)


def cat_nhwc(tensors):
    """torch.cat(tensors, 1) into a fresh NHWC slab whose pixel rows are 16-byte aligned (zero channels appended when the
    channel sum is not a multiple of 4: concat3 = 225, concat2 = 161); backward hands out channel-slice views"""
    return _CatNHWC.apply(*tensors)


# ------------------------------------------------------------------------------------------------ 2x2 average pool
class _AvgPool2(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x):
        x, xs = _nhwc(x)
        B, C, H, W = x.shape
        if H % 2 or W % 2:
            raise ValueError("avgpool2 needs even spatial dims")
        y = _new(B, C, H // 2, W // 2, x.device)
        _lib.check(_lib.lib().bts_avgpool2_fwd(_ptr(x), xs, B, H // 2, W // 2, C, _ptr(y), C, _stream()), "bts_avgpool2_fwd")
        _lib.count()
        return y

    @staticmethod
    def backward(ctx, g):
        g, gs = _nhwc(g)
        B, C, Ho, Wo = g.shape
        gx = _new(B, C, 2 * Ho, 2 * Wo, g.device)
        _lib.check(_lib.lib().bts_avgpool2_bwd(_ptr(g), gs, B, Ho, Wo, C, _ptr(gx), C, _stream()), "bts_avgpool2_bwd")
        _lib.count()
        return gx


def avgpool2(x):
    return _AvgPool2.apply(x)


# ------------------------------------------------------------------------------------------------ ResNet / ResNeXt glue
class _MaxPool3s2(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x):
        x, xs = _nhwc(x)
        B, C, H, W = x.shape
        Ho, Wo = (H - 1) // 2 + 1, (W - 1) // 2 + 1
        y = _new(B, C, Ho, Wo, x.device)
        arg = torch.empty(B * Ho * Wo * C, device=x.device, dtype=torch.uint8)
        _lib.check(_lib.lib().bts_maxpool3s2_fwd(_ptr(x), xs, B, H, W, C, _ptr(y), C, _ptr(arg), _stream()), "bts_maxpool3s2_fwd")
        _lib.count()
        ctx.shape = (B, C, H, W)
        ctx.save_for_backward(arg)
        return y

    @staticmethod
    def backward(ctx, g):
        (arg,) = ctx.saved_tensors
        B, C, H, W = ctx.shape
        g, gs = _nhwc(g)
        gx = _new(B, C, H, W, g.device)
        _lib.check(_lib.lib().bts_maxpool3s2_bwd(_ptr(g), gs, _ptr(arg), B, H, W, C, _ptr(gx), C, _stream()), "bts_maxpool3s2_bwd")
        _lib.count()
        return gx


def maxpool3s2(x):
    """3x3 / stride 2 / pad 1 max-pool (torchvision densenet `pool0`, resnet `maxpool`) on our NHWC kernels"""
    return _MaxPool3s2.apply(x)


class _BnAddRelu(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, res, gamma, beta, bn):
        x, xs = _nhwc(x)
        res, rs = _nhwc(res)
        B, C, H, W = x.shape
        n = B * H * W
        batch = bn_uses_batch_stats(bn)
        st = bn_finalize(bn_stats(x) if batch else None, n, bn, gamma, beta, batch)
        y = _new(B, C, H, W, x.device)
        _lib.check(_lib.lib().bts_bn_add_relu(_ptr(x), xs, n, C, _ptr(st[0]), _ptr(st[1]), _ptr(res), rs, _ptr(y), C, _stream()),
                   "bts_bn_add_relu")
        _lib.count()
        ctx.batch = batch
        ctx.save_for_backward(x, st, y)
        return y

    @staticmethod
    def backward(ctx, gy):
        x, st, y = ctx.saved_tensors
        g, gs = _nhwc(gy)
        B, C, H, W = y.shape
        gm = _new(B, C, H, W, y.device)
        _lib.check(_lib.lib().bts_relu_bwd(_ptr(g), gs, _ptr(y), C, B * H * W, C, _ptr(gm), C, _stream()), "bts_relu_bwd")
        _lib.count()
        gx, S = bn_backward(x, gm, st, ctx.batch, False)
        return (gx if ctx.needs_input_grad[0] else None, gm if ctx.needs_input_grad[1] else None,
                S[1].float() if ctx.needs_input_grad[2] else None, S[0].float() if ctx.needs_input_grad[3] else None, None)


def bn_add_relu(x, res, bn):
    """relu(bn(x) + res): the tail of a torchvision Bottleneck, one streaming kernel after the statistics"""
    return _BnAddRelu.apply(x, res, bn.weight, bn.bias, bn)


# ------------------------------------------------------------------------------------------------ MobileNetV2 glue
def _bn_apply(x, st, act, res=None):
    """act(x*st[0] + st[1]) [+ res] into a fresh NHWC tensor (bts_bn_apply / bts_bn_add)"""
    x, xs = _nhwc(x)
    B, C, H, W = x.shape
    y = _new(B, C, H, W, x.device)
    L = _lib.lib()
    if res is None:
        _lib.check(L.bts_bn_apply(_ptr(x), xs, B * H * W, C, _ptr(st[0]), _ptr(st[1]), int(act), _ptr(y), C, _stream()),
                   "bts_bn_apply")
    else:
        r, rs = _nhwc(res)
        _lib.check(L.bts_bn_add(_ptr(x), xs, B * H * W, C, _ptr(st[0]), _ptr(st[1]), _ptr(r), rs, _ptr(y), C, _stream()),
                   "bts_bn_add")
    _lib.count()
    return y


def _stats_buffer(C, dev):
    return torch.zeros((2, C), device=dev, dtype=torch.float64)


class _InvertedResidual(torch.autograd.Function):
    """torchvision InvertedResidual [1x1 -> BN1 -> ReLU6 ->] dw 3x3 -> BN2 -> ReLU6 -> 1x1 -> BN3 [+ x]"""

    @staticmethod
    def forward(ctx, x, w1, g1, b1, w2, g2, b2, w3, g3, b3, bns, stride, res, fuse_eval):
        from . import dwconv
        bn1, bn2, bn3 = bns
        x, _ = _nhwc(x)
        B, _, H, W = x.shape
        Ho, Wo = (H - 1) // stride + 1, (W - 1) // stride + 1
        y1 = st1 = pre = None
        t1 = False
        if w1 is not None:                          # expand 1x1 on the engine, BN1 statistics from its epilogue
            t1 = bn_uses_batch_stats(bn1)
            s1 = _stats_buffer(w1.shape[0], x.device) if t1 else None
            y1 = conv.conv2d_tc(x, w1, stats=s1)
            st1 = bn_finalize(s1, B * H * W, bn1, g1, b1, t1)
            pre = (st1[0], st1[1])
        dw_in = x if y1 is None else y1
        t2 = bn_uses_batch_stats(bn2)
        y2 = None
        if t2:                                      # depthwise with the BN1 + ReLU6 prologue and BN2 statistics epilogue
            y2, s2 = dwconv.fwd(dw_in, w2, stride, pre=pre, stats=True)
            st2 = bn_finalize(s2, B * Ho * Wo, bn2, g2, b2, True)
            a2 = _bn_apply(y2, st2, 2)
        else:
            st2 = bn_finalize(None, B * Ho * Wo, bn2, g2, b2, False)
            if fuse_eval:                           # no backward follows: relu6(bn2(.)) from the folded statistics
                a2 = dwconv.fwd(dw_in, w2, stride, pre=pre, post=(st2[0], st2[1]))   # in the epilogue
            else:                                   # the backward needs the BN2 input y2
                y2 = dwconv.fwd(dw_in, w2, stride, pre=pre)
                a2 = _bn_apply(y2, st2, 2)
        t3 = bn_uses_batch_stats(bn3)
        s3 = _stats_buffer(w3.shape[0], x.device) if t3 else None
        y3 = conv.conv2d_tc(a2, w3, stats=s3)
        st3 = bn_finalize(s3, B * Ho * Wo, bn3, g3, b3, t3)
        out = _bn_apply(y3, st3, 0, x if res else None)
        ctx.cfg = (stride, res, t1, t2, t3, H, W)
        ctx.save_for_backward(x, w1, w2, w3, y1, st1, y2, st2, a2, y3, st3)
        return out

    @staticmethod
    def backward(ctx, gy):
        from . import dwconv
        x, w1, w2, w3, y1, st1, y2, st2, a2, y3, st3 = ctx.saved_tensors
        stride, res, t1, t2, t3, H, W = ctx.cfg
        need = ctx.needs_input_grad
        g, _ = _nhwc(gy)
        gx = gw1 = gw2 = gw3 = G1 = G2 = G3 = None
        need_a1 = need[0] or any(need[1:4])               # the gradient has to reach the depthwise input
        need_y2 = need_a1 or any(need[4:7])
        g_y3, G3 = bn_backward(y3, g, st3, t3, 0)
        if need[7]:
            gw3 = conv.wgrad_tc(a2, g_y3, w3.shape, w3.stride())
        if need_y2:
            g_a2 = conv.conv2d_tc(g_y3, w3, 1, 0, 1, transpose_flip=True)
            g_y2, G2 = bn_backward(y2, g_a2, st2, t2, 2, out=g_a2)
            dw_in = x if y1 is None else y1
            pre = None if st1 is None else (st1[0], st1[1])
            if need[4]:
                gw2 = dwconv.wgrad(dw_in, g_y2, w2, stride, pre=pre)
            if need_a1:
                g_a1 = dwconv.dgrad(g_y2, w2, stride, H, W)
                if w1 is None:
                    gx = g_a1
                else:
                    g_y1, G1 = bn_backward(y1, g_a1, st1, t1, 2, out=g_a1)
                    if need[1]:
                        gw1 = conv.wgrad_tc(x, g_y1, w1.shape, w1.stride())
                    if need[0]:
                        gx = conv.conv2d_tc(g_y1, w1, 1, 0, 1, transpose_flip=True)
        if need[0] and res:
            if gx is None:
                gx = g.clone(memory_format=torch.channels_last)
            else:
                copy_channels(g, gx, accumulate=True)     # residual branch: dx += dy
        dg = lambda G, i: G[1].float() if need[i] and G is not None else None
        db = lambda G, i: G[0].float() if need[i] and G is not None else None
        return (gx if need[0] else None, gw1, dg(G1, 2), db(G1, 3), gw2, dg(G2, 5), db(G2, 6), gw3, dg(G3, 8), db(G3, 9),
                None, None, None, None)


def inverted_residual(x, block):
    """torchvision InvertedResidual `block` (re-classed by model.adopt_convs) applied to x as one autograd Function"""
    layers = list(block.conv)
    if len(layers) == 4:
        expand, dw, proj, bn3 = layers
        w1, g1, b1, bn1 = expand[0].weight, expand[1].weight, expand[1].bias, expand[1]
    else:
        dw, proj, bn3 = layers
        w1 = g1 = b1 = bn1 = None
    bn2 = dw[1]
    # BN2 on folded running statistics can run as the depthwise conv's epilogue only when no backward follows.  That is
    # decided here: inside the Function, needs_input_grad reflects requires_grad alone and ignores no_grad / inference_mode.
    fuse_eval = not bn_uses_batch_stats(bn2) and not (
        torch.is_grad_enabled() and (x.requires_grad or any(p.requires_grad for p in block.parameters())))
    return _InvertedResidual.apply(x, w1, g1, b1, dw[0].weight, bn2.weight, bn2.bias, proj.weight, bn3.weight, bn3.bias,
                                   (bn1, bn2, bn3), int(dw[0].stride[0]), bool(block.use_res_connect), fuse_eval)
