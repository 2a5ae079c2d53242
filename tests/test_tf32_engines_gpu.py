"""GPU checks of the single-pass TF32 kernels (conv_tf32_kernel, wgrad_tf32_kernel, wgrad2_tf32_kernel) against fp64 CPU
references.  Every template instantiation runs at least once, and torch.profiler confirms the kernel and its template
arguments.  The bar is that of the engine's fast-mode tests: 1e-5 < err < 5e-3 of the output scale.  The lower bound
shows that one product ran, not three."""
import ctypes

import pytest
import torch
import torch.nn.functional as F

from engine_checks import Op, kernels, nhwc_slice, ran, rel_err

pytestmark = pytest.mark.gpu

LO, HI = 1e-5, 5e-3
TF32 = r"wgrad2?_tf32_kernel|conv_tf32_kernel"


def _L():
    from bts_b200 import _lib
    return _lib.lib()


def _profiled(fn):
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        out = fn()
        torch.cuda.synchronize()
    return out, kernels(prof, TF32), kernels(prof)


def _bar(e):
    assert LO < e < HI, e


# ------------------------------------------------------------------------------------------------ forward / dgrad
@pytest.mark.parametrize("vec", [True, False])
@pytest.mark.parametrize("mode", [0, 1, 2])
@pytest.mark.parametrize("pre", [0, 1, 2, 3])
def test_conv_every_instantiation(pre, mode, vec):
    """conv_tf32_kernel<PRE, UP, VEC>: pre-op none / ReLU / affine / affine + ReLU, source as is / x2 up-sampled /
    zero-stuffed (the dgrad of a stride-2 3x3 conv, transposed operator), 16-byte or scalar loads (x as a slice of a
    slab with pixel stride 71); Cin = 68, Cout = 40"""
    from bts_b200 import conv
    g = torch.Generator().manual_seed(10 * pre + 3 * mode + vec)
    Cin, Cout, Hs, Ws = 68, 40, 9, 11
    x = torch.randn(2, Cin, Hs, Ws, generator=g)
    scale = (torch.rand(Cin, generator=g) + 0.5).cuda() if pre & 2 else None
    shift = (torch.randn(Cin, generator=g) * 0.3).cuda() if pre & 2 else None
    relu = bool(pre & 1)
    if mode == 2:     # layer weight (Cin, Cout, 3, 3): its input had Cout channels at (2 Hs - 1) x (2 Ws - 1)
        w = torch.randn(Cin, Cout, 3, 3, generator=g) / (Cin * 9) ** 0.5
        out_hw = (2 * Hs - 1, 2 * Ws - 1)
        op = Op(w, 1, 1, 1, scale, shift, relu, mode=2, out_hw=out_hw, transpose_flip=True)
        kw = dict(transpose_flip=True, zero_stuff_out=out_hw)
        args = (1, 1, 1)
    else:
        w = torch.randn(Cout, Cin, 3, 3, generator=g) / (Cin * 9) ** 0.5
        op = Op(w, 1, 1, 1, scale, shift, relu, mode=mode)
        kw = dict(upsample2=mode == 1)
        args = (1, 1, 1)
    xc = nhwc_slice(x, None if vec else 71)
    y, ks, parity = _profiled(lambda: conv.conv2d_tc(xc, w.cuda(), *args, pre_scale=scale, pre_shift=shift, pre_relu=relu,
                                                     precision=1, **kw))
    assert ran(ks, "conv_tf32_kernel", (pre, mode, vec)) and not parity, (ks, parity)
    _bar(rel_err(y, op.full(x)))


def test_conv_epilogue_statistics_and_grouped_operator():
    """BatchNorm statistics from the epilogue (fp64 sums of the kernel's own output, two n-tiles of 96) and the
    block-diagonal operator of a ResNeXt 3x3 (32 groups of 8)"""
    from bts_b200 import conv
    g = torch.Generator().manual_seed(7)
    x = torch.randn(2, 64, 12, 14, generator=g)
    w = torch.randn(192, 64, 3, 3, generator=g) / 24
    st = torch.zeros(2, 192, dtype=torch.float64, device="cuda")
    y, ks, _ = _profiled(lambda: conv.conv2d_tc(nhwc_slice(x), w.cuda(), 1, 1, 1, stats=st, precision=1))
    assert ran(ks, "conv_tf32_kernel", (0, 0, 1))
    _bar(rel_err(y, Op(w, 1, 1, 1).full(x)))
    yd = y.double()
    s1, s2 = yd.sum((0, 2, 3)), (yd * yd).sum((0, 2, 3))
    # the per-warp column sums are fp32 before the fp64 partials: the bar of tests/test_conv_prologue_stats_gpu.py
    assert float((st[0] - s1).abs().max()) <= 1e-5 * float(yd.abs().sum((0, 2, 3)).max())
    assert float((st[1] - s2).abs().max()) <= 1e-5 * float((yd * yd).sum((0, 2, 3)).max())

    xg = torch.randn(2, 256, 8, 10, generator=g)
    wg = torch.randn(256, 8, 3, 3, generator=g) / (8 * 9) ** 0.5
    yg, ks, _ = _profiled(lambda: conv.conv2d_tc(nhwc_slice(xg), wg.cuda(), 1, 1, 1, groups=32, precision=1))
    assert ran(ks, "conv_tf32_kernel", (0, 0, 1))
    _bar(rel_err(yg, F.conv2d(xg.double(), wg.double(), None, 1, 1, 1, 32)))


def test_conv_mode_setting_reaches_the_kernel():
    """precision=None follows set_precision; explicit 0 / 1 keep their meaning whatever the mode"""
    import bts_b200
    from bts_b200 import conv
    g = torch.Generator().manual_seed(9)
    x = nhwc_slice(torch.randn(1, 32, 10, 10, generator=g))
    w = (torch.randn(48, 32, 3, 3, generator=g) / 17).cuda()
    prev = bts_b200.set_precision("tf32")
    try:
        y1, ks1, p1 = _profiled(lambda: conv.conv2d_tc(x, w, 1, 1, 1))
        y0, ks0, p0 = _profiled(lambda: conv.conv2d_tc(x, w, 1, 1, 1, precision=0))
    finally:
        bts_b200.set_precision(prev)
    y2, ks2, p2 = _profiled(lambda: conv.conv2d_tc(x, w, 1, 1, 1, precision=1))
    assert ran(ks1, "conv_tf32_kernel") and ran(p0, "conv_tc_kernel") and ran(ks2, "conv_tf32_kernel")
    assert not ks0 and not p1
    assert torch.equal(y1, y2) and not torch.equal(y0, y1)


# ------------------------------------------------------------------------------------------------ weight gradient
def _wgrad_case(B, Cin, Hs, Ws, Cout, k, pre=0, up=False, seed=0):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, Cin, Hs, Ws, generator=g)
    scale = torch.rand(Cin, generator=g) + 0.5 if pre & 2 else None
    shift = torch.randn(Cin, generator=g) * 0.3 if pre & 2 else None
    xd = x.double()
    if pre & 2:
        xd = xd * scale.double().view(1, -1, 1, 1) + shift.double().view(1, -1, 1, 1)
    if pre & 1:
        xd = F.relu(xd)
    if up:
        xd = F.interpolate(xd, scale_factor=2, mode="nearest")
    wd = torch.zeros(Cout, Cin, k, k, dtype=torch.float64, requires_grad=True)
    y = F.conv2d(xd, wd, None, 1, k // 2, 1)
    gy = torch.randn(y.shape, generator=g)
    y.backward(gy.double())
    return x, gy, scale, shift, wd.grad


def _route(min_pixels, tma=1):
    L = _L()
    L.bts_wgrad2_set_min_pixels(min_pixels)
    L.bts_wgrad2_set_tma(tma)


@pytest.fixture
def restore_routing():
    yield
    _route(-1, 1)


def _wgrad(x, gy, scale, shift, pre, up, k, x_width=None):
    from bts_b200 import conv
    Cout, Cin = gy.shape[1], x.shape[1]
    xc, gc = nhwc_slice(x, x_width), nhwc_slice(gy)
    sc = scale.cuda() if scale is not None else None
    sh = shift.cuda() if shift is not None else None
    return _profiled(lambda: conv.wgrad_tc(xc, gc, (Cout, Cin, k, k), (Cin * k * k, k * k, k, 1), 1, k // 2, 1, sc, sh,
                                           bool(pre & 1), up, precision=1))


@pytest.mark.parametrize("vec", [True, False])
@pytest.mark.parametrize("up", [False, True])
@pytest.mark.parametrize("pre", [0, 1, 2, 3])
def test_tap_in_grid_wgrad_every_instantiation(restore_routing, pre, up, vec):
    """wgrad_tf32_kernel<PRE, UP, VEC>, every layer forced onto the tap-in-grid kernel; Cin = 70 read from a slab of
    72 channels (16-byte loads) or 71 (scalar loads)"""
    _route(1 << 40)
    x, gy, sc, sh, ref = _wgrad_case(2, 70, 6, 9, 72, 3, pre, up, seed=100 + 10 * pre + up)
    dw, ks, parity = _wgrad(x, gy, sc, sh, pre, up, 3, 72 if vec else 71)
    assert ran(ks, "wgrad_tf32_kernel", (pre, up, vec)) and not parity, (ks, parity)
    _bar(rel_err(dw, ref))


@pytest.mark.parametrize("path", ["tma_ring", "loads_vec", "loads_scalar"])
@pytest.mark.parametrize("up", [False, True])
@pytest.mark.parametrize("pre", [0, 1, 2, 3])
def test_shifted_dy_wgrad_every_instantiation(restore_routing, pre, up, path):
    """wgrad2_tf32_kernel<PRE, UP, VEC, TMA>: the landing ring (vector loads only) and the load path with 16-byte or
    scalar loads, every layer of 3x3 with Cout <= 64 forced onto the shifted-dY kernel"""
    _route(0, 1 if path == "tma_ring" else 0)
    x, gy, sc, sh, ref = _wgrad_case(2, 72, 7, 10, 40, 3, pre, up, seed=200 + 10 * pre + up)
    vec = path != "loads_scalar"
    dw, ks, parity = _wgrad(x, gy, sc, sh, pre, up, 3, None if vec else 73)
    assert ran(ks, "wgrad2_tf32_kernel", (pre, up, vec, path == "tma_ring")) and not parity, (ks, parity)
    _bar(rel_err(dw, ref))


@pytest.mark.parametrize("route", ["tap_in_grid", "shifted_dy"])
def test_split_k_wgrad_matches_an_explicit_call_bitwise(restore_routing, route):
    """conv.wgrad_tc at the plan's split and the explicit-split ABI call at that split give bit-identical dW; the
    plan splits this 4096-pixel reduction on the full grid"""
    from bts_b200 import _lib, conv
    from bts_b200.ops import _ptr, _stream
    _route(1 << 40 if route == "tap_in_grid" else 0)
    x, gy, _, _, ref = _wgrad_case(1, 64, 64, 64, 48, 3, seed=48)
    xc, gc = nhwc_slice(x), nhwc_slice(gy)
    L = _L()
    sp, wsf = ctypes.c_int(0), ctypes.c_longlong(0)
    _lib.check(L.bts_conv_wgrad_plan(1, 64, 64, 64, 48, 3, 3, 1, ctypes.byref(sp), ctypes.byref(wsf)), "plan")
    ws = torch.full((wsf.value,), float("nan"), device="cuda")
    dw = torch.empty(48, 64, 3, 3, device="cuda")

    def explicit():
        _lib.check(L.bts_conv_wgrad(_ptr(xc), 64, 1, 64, 64, 0, 64, 3, 3, 1, 1, 1, None, None, 0, _ptr(gc), 48, 48, _ptr(ws),
                                    sp.value, _ptr(dw), 576, 9, 3, 1, 1, _stream()), "bts_conv_wgrad")
        return dw
    _, ks, _ = _profiled(explicit)
    gw = conv.wgrad_tc(xc, gc, (48, 64, 3, 3), (576, 9, 3, 1), 1, 1, 1, precision=1)
    torch.cuda.synchronize()
    assert ran(ks, "wgrad_tf32_kernel" if route == "tap_in_grid" else "wgrad2_tf32_kernel")
    assert torch.equal(gw, dw)
    _bar(rel_err(dw, ref))


def test_grouped_wgrad():
    """bts_conv_wgrad_grouped (ResNeXt 3x3, 32 groups of 8) on wgrad_tf32_kernel<0, false, true>"""
    from bts_b200 import conv
    g = torch.Generator().manual_seed(600)
    x = torch.randn(2, 256, 8, 10, generator=g)
    gy = torch.randn(2, 256, 8, 10, generator=g)
    wd = torch.zeros(256, 8, 3, 3, dtype=torch.float64, requires_grad=True)
    F.conv2d(x.double(), wd, None, 1, 1, 1, 32).backward(gy.double())
    dw, ks, _ = _profiled(lambda: conv.wgrad_grouped_tc(nhwc_slice(x), nhwc_slice(gy), (256, 8, 3, 3), (72, 9, 3, 1), 1, 1,
                                                        1, precision=1))
    assert ran(ks, "wgrad_tf32_kernel", (0, False, True))
    _bar(rel_err(dw, wd.grad))
