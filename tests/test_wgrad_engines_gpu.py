"""GPU parity of the two weight-gradient kernels against torch fp64 autograd on the CPU, at the 2e-5 output-scale bar of
tests/test_conv_gpu.py: the tap-in-grid kernel (wgrad_tc_kernel, csrc/wgrad_tc.cu) and the shifted-dY kernel
(wgrad2_tc_kernel, csrc/wgrad2_tc.cu), with the routing between them forced, plus the grouped (block-diagonal) path.

Every call goes through the C ABI with an explicit split count.  The split-K workspace is exactly
splitK * taps * Cin * Cout floats and filled with NaN, so a partial the kernel never writes turns into NaN in dW; dW is a
strided view inside a larger NaN-filled buffer, so a write outside the view shows as a lost guard.  Each call records
the kernels it launched (torch.profiler), and the tests assert which template instantiation ran.  The pixels one CTA
reduces stay at or below about 2k, where 3xTF32 meets the bar without the K-length allowance of test_conv_gpu.py: the
tensor cores' fp32 accumulator truncates on every step, and one CTA reducing 3256 pixels of ReLU'd activations (the split
case below at split 1, on a 2x37x44 map) measured 2.3e-5 on an H100."""
import ctypes
import os

import pytest
import torch
import torch.nn.functional as F

from engine_checks import check_written, guarded, kernels, nan, nhwc_slice, ran

pytestmark = pytest.mark.gpu

TOL = 2e-5
KP = 32                 # pixels per k-block of wgrad_tc_kernel
SPLIT_PX = 16           # split-K ranges of wgrad2_tc_kernel are whole multiples of this many pixels


def _L():
    from bts_b200 import _lib
    return _lib.lib()


def _route(tap_in_grid, tma=1):
    L = _L()
    L.bts_wgrad2_set_min_pixels(1 << 40 if tap_in_grid else 0)
    L.bts_wgrad2_set_tma(tma)


def _capped_grid():
    """BTS_B200_SM_LIMIT (read with atoi by csrc/util.cu) caps the library's grids below this GPU's SM count"""
    lim = int(os.environ.get("BTS_B200_SM_LIMIT") or 0)
    return 0 < lim < torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count


def _restore():
    L = _L()
    L.bts_wgrad2_set_min_pixels(-1)
    L.bts_wgrad2_set_tma(1)


@pytest.fixture
def tap_in_grid():
    """every layer on wgrad_tc_kernel, whatever its size and width"""
    _route(True)
    yield "tap_in_grid"
    _restore()


@pytest.fixture(params=["tma_ring", "global_loads"])
def shifted_dy(request):
    """eligible layers (3x3 with Cout <= 64, 1x1 with 64 < Cout <= 256) on wgrad2_tc_kernel at any map size, with the
    operands staged through the TMA landing ring where the shape allows it, or loaded by the producers"""
    _route(False, 1 if request.param == "tma_ring" else 0)
    yield request.param
    _restore()


@pytest.fixture(params=["tap_in_grid", "shifted_dy_tma", "shifted_dy_global"])
def route(request):
    _route(request.param == "tap_in_grid", 0 if request.param == "shifted_dy_global" else 1)
    yield request.param
    _restore()


# --------------------------------------------------------------------------------------------------------------- helpers
def _weight_strides(Cout, Cin, k, layout):
    if layout == "contiguous":
        return (Cin * k * k, k * k, k, 1)
    if layout == "channels_last":
        return torch.empty(Cout, Cin, k, k).contiguous(memory_format=torch.channels_last).stride()
    if layout == "transposed":             # (Cin, Cout, k, k) in memory: s_co < s_ci
        return (k * k, Cout * k * k, k, 1)
    if layout == "pitched":                # rows of the output channel padded by 7 floats: guards between the rows
        return (Cin * k * k + 7, k * k, k, 1)
    raise ValueError(layout)


def _nhwc(t):
    """(pixel stride) of a (B,C,H,W) NHWC-in-memory tensor, asserting the engine will read it in place"""
    from bts_b200 import conv
    v, s = conv._nhwc_view(t)
    assert v.data_ptr() == t.data_ptr()
    return s


def wgrad(x, gy, k, stride=1, pad=0, dil=1, scale=None, shift=None, relu=False, up=False, split=None, precision=0,
          layout="contiguous"):
    """bts_conv_wgrad with an explicit split count (None: the plan's), marshalled as conv.wgrad_tc does, on a NaN-filled
    workspace of exactly the planned size and a guarded dW view.  Returns (dW, split, launched wgrad kernels)."""
    from bts_b200 import _lib
    from bts_b200.ops import _ptr, _stream
    L = _L()
    xs, gs = _nhwc(x), _nhwc(gy)
    B, Cin, Hs, Ws = x.shape
    _, Cout, Ho, Wo = gy.shape
    if split is None:
        sp, wsf = ctypes.c_int(0), ctypes.c_longlong(0)
        _lib.check(L.bts_conv_wgrad_plan(B, Ho, Wo, Cin, Cout, k, k, stride, ctypes.byref(sp), ctypes.byref(wsf)),
                   "bts_conv_wgrad_plan")
        split = sp.value
        assert wsf.value == split * k * k * Cin * Cout
    ws = nan(split * k * k * Cin * Cout)
    s = _weight_strides(Cout, Cin, k, layout)
    dw, buf, inside = guarded((Cout, Cin, k, k), s)
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        rc = L.bts_conv_wgrad(_ptr(x), xs, B, Hs, Ws, int(up), Cin, k, k, stride, pad, dil, _ptr(scale), _ptr(shift),
                              int(relu), _ptr(gy), gs, Cout, _ptr(ws), split, _ptr(dw), s[0], s[1], s[2], s[3],
                              int(precision), _stream())
        _lib.check(rc, "bts_conv_wgrad")
        torch.cuda.synchronize()
    check_written(dw, buf, inside)
    return dw, split, kernels(prof)


class Case:
    """seeded fp32 inputs of one layer and the fp64 CPU reference of its weight gradient: pre-op (affine for pre & 2,
    ReLU for pre & 1), nearest x2 up-sample, conv2d, autograd"""

    def __init__(self, B, Cin, Hs, Ws, Cout, k, stride=1, pad=None, dil=1, pre=0, up=False, seed=0):
        g = torch.Generator().manual_seed(seed)
        self.k, self.stride, self.dil, self.pre, self.up = k, stride, dil, pre, up
        self.pad = dil * (k // 2) if pad is None else pad
        self.x = torch.randn(B, Cin, Hs, Ws, generator=g)
        self.scale = torch.rand(Cin, generator=g) + 0.5 if pre & 2 else None
        self.shift = torch.randn(Cin, generator=g) * 0.3 if pre & 2 else None
        xd = self.x.double()
        if pre & 2:
            xd = xd * self.scale.double().view(1, -1, 1, 1) + self.shift.double().view(1, -1, 1, 1)
        if pre & 1:
            xd = F.relu(xd)
        if up:
            xd = F.interpolate(xd, scale_factor=2, mode="nearest")
        wd = torch.zeros(Cout, Cin, k, k, dtype=torch.float64, requires_grad=True)
        y = F.conv2d(xd, wd, None, stride, self.pad, dil)
        self.gy = torch.randn(y.shape, generator=g)
        y.backward(self.gy.double())
        self.ref = wd.grad

    def run(self, x_width=None, x_off=0, dy_width=None, dy_off=0, **kw):
        x, gy = nhwc_slice(self.x, x_width, x_off), nhwc_slice(self.gy, dy_width, dy_off)
        sc = self.scale.cuda() if self.scale is not None else None
        sh = self.shift.cuda() if self.shift is not None else None
        return wgrad(x, gy, self.k, self.stride, self.pad, self.dil, sc, sh, bool(self.pre & 1), self.up, **kw)

    def err(self, dw):
        return float((dw.detach().cpu().double() - self.ref).abs().max() / self.ref.abs().max())


# ------------------------------------------------------------------------------------------- tap-in-grid kernel (wgrad_tc)
@pytest.mark.parametrize("load", ["vec", "x_stride", "dy_offset"])
@pytest.mark.parametrize("up", [False, True])
@pytest.mark.parametrize("pre", [0, 1, 2, 3])
def test_tap_in_grid_every_instantiation(tap_in_grid, pre, up, load):
    """wgrad_tc_kernel<PRE, UP, VEC>: all 16 instantiations.  PRE 0 none / 1 ReLU (the decoder upconvs) / 2 affine / 3
    affine + ReLU, padding applied after the pre-op; UP reads x through the nearest x2 up-sample.  The scalar-load path
    (VEC = false) is reached two ways: x as a channel slice of a slab whose pixel stride (71) is not a multiple of 4, and
    dY as the slice at channel offset 1 of a slab (base not 16-byte aligned).  Cin = 70 leaves a half-filled 4-channel
    unit and a partial 128-channel tile; Cout = 72 gives two 48-wide tiles, the second 24 channels live."""
    c = Case(2, 70, 6, 9, 72, 3, pre=pre, up=up, seed=100 + 10 * pre + up)
    kw = {"vec": dict(x_width=72), "x_stride": dict(x_width=71), "dy_offset": dict(x_width=72, dy_width=76, dy_off=1)}[load]
    dw, _, ks = c.run(**kw)
    assert ran(ks, "wgrad_tc_kernel", (pre, up, load == "vec")), ks
    assert c.err(dw) < TOL


@pytest.mark.parametrize("Cout,k", [(16, 3), (24, 3), (48, 3), (64, 3), (80, 3), (96, 3), (112, 3), (128, 3), (192, 3),
                                    (256, 3), (512, 3), (1056, 1)])
def test_tap_in_grid_output_tile_widths(tap_in_grid, Cout, k):
    """every n-tile width (16, 32, 48, 64) and tile count of wgrad_n_tile: 80 and 96 are two 48-wide tiles whose second
    32-channel dY chunk reaches into the next tile's channels, 112 two 64-wide tiles with a 48-channel tail, 512 eight
    tiles; the 1x1 layer with Cout = 1056 runs 17 tiles of 64, the last one half live"""
    c = Case(1, 40, 9, 13, Cout, k, seed=Cout + k)
    dw, _, ks = c.run()
    assert ran(ks, "wgrad_tc_kernel", (0, False, True)), ks
    assert c.err(dw) < TOL


DECODER = [
    # name, B, Cin, Hs, Ws, Cout, dil, up, pre   (3x3, 'same' padding; the DenseNet-161 decoder at num_features 512)
    ("upconv5", 1, 2208, 6, 11, 512, 1, True, 1),
    ("conv5", 1, 896, 12, 22, 512, 1, False, 0),
    ("upconv4", 1, 512, 12, 22, 256, 1, True, 0),
    ("conv4", 1, 448, 24, 44, 256, 1, False, 0),
    ("daspp_12", 2, 256, 10, 20, 128, 12, False, 3),
    ("daspp_24", 2, 256, 10, 20, 128, 24, False, 3),
    ("daspp_conv", 1, 896, 24, 44, 128, 1, False, 0),
    ("conv3", 2, 225, 12, 22, 128, 1, False, 0),
    ("conv2", 2, 161, 16, 24, 64, 1, False, 0),
]


@pytest.mark.parametrize("name,B,Cin,Hs,Ws,Cout,dil,up,pre", DECODER, ids=[d[0] for d in DECODER])
def test_tap_in_grid_decoder_layers(tap_in_grid, name, B, Cin, Hs, Ws, Cout, dil, up, pre):
    """the decoder's wide 3x3 layers at their real channel counts on small maps: upconv5 reads its 2208-channel source
    through the ReLU-only pre-op and the x2 up-sample (18 input-channel tiles x 8 output tiles), the daspp convs take
    the BatchNorm + ReLU pre-op at dilations larger than the map (whole taps in the padding), conv3 and conv2 have odd
    Cin (scalar loads).  conv2 runs on the shifted-dY kernel in production; here it is forced onto this one."""
    c = Case(B, Cin, Hs, Ws, Cout, 3, dil=dil, pre=pre, up=up, seed=Cin + Cout + dil)
    dw, _, ks = c.run()
    assert ran(ks, "wgrad_tc_kernel", (pre, up, Cin % 4 == 0)), ks
    assert c.err(dw) < TOL


@pytest.mark.parametrize("B,Cin,H,W,Cout,k,pad", [(2, 64, 13, 15, 96, 3, 1), (2, 3, 40, 48, 96, 7, 3)])
def test_tap_in_grid_stride2(tap_in_grid, B, Cin, H, W, Cout, k, pad):
    """stride 2: a 3x3 conv on an odd-sized input (the last input row and column are read by one tap only) and the 7x7
    stem with Cin = 3 (49 taps in the grid, one partial 4-channel unit, scalar loads)"""
    c = Case(B, Cin, H, W, Cout, k, stride=2, pad=pad, seed=k + Cin)
    dw, _, ks = c.run()
    assert ran(ks, "wgrad_tc_kernel", (0,)), ks
    assert c.err(dw) < TOL


@pytest.mark.parametrize("pad,dil", [(0, 1), (3, 1), (5, 2)])
def test_tap_in_grid_padding_not_same(tap_in_grid, pad, dil):
    """padding other than dil * (k // 2): Hout != Hin, so a tap's input window is shifted against the output grid;
    pad > dil leaves output rows whose every tap but one reads padding"""
    c = Case(2, 48, 10, 13, 40, 3, pad=pad, dil=dil, pre=3, seed=pad + 10 * dil)
    dw, _, ks = c.run()
    assert ran(ks, "wgrad_tc_kernel", (3, False, True)), ks
    assert c.err(dw) < TOL


SPLIT_CASE = dict(B=2, Cin=96, Hs=23, Ws=33, Cout=64, k=3)       # 1518 output pixels: KBp = 48 k-blocks of 32
KBP = -(-2 * 23 * 33 // KP)


@pytest.mark.parametrize("split", [1, 2, 3, 7, KBP, KBP + 3])
def test_tap_in_grid_forced_split(tap_in_grid, split):
    """split-K counts the plan never picks for this shape: 7 leaves the last range short (48 = 6 x 7 + 6), KBp gives
    one k-block per CTA and KBp + 3 leaves three trailing splits with no k-block, whose partials must still be written
    (as zeros) into the NaN-filled workspace.  A split-K result is bit-reproducible: fixed summation order."""
    c = Case(**SPLIT_CASE, pre=3, seed=7)
    dw, sp, ks = c.run(split=split)
    assert sp == split and ran(ks, "wgrad_tc_kernel", (3, False, True)), ks
    assert c.err(dw) < TOL
    if split > 1:
        dw2, _, _ = c.run(split=split)
        assert torch.equal(dw, dw2)


@pytest.mark.parametrize("layout", ["channels_last", "transposed", "pitched"])
def test_weight_gradient_written_through_strides(tap_in_grid, layout):
    """the reduce kernel writes dW through (s_co, s_ci, s_kh, s_kw): a channels_last weight, a transposed pair
    (s_co < s_ci) and rows with a pitch, whose gaps must keep their NaN; split 3 so the reduce sums several partials"""
    c = Case(2, 40, 9, 11, 24, 3, seed=3)
    dw, _, _ = c.run(split=3, layout=layout)
    assert c.err(dw) < TOL


def test_precision_flag_reaches_both_kernels(route):
    """precision = 1 (single-pass TF32) reaches the kernel: measurably less exact than parity mode, yet bounded"""
    c = Case(1, 128, 16, 16, 48, 3, seed=5)
    d3, _, ks = c.run()
    d1, _, ks1 = c.run(precision=1)
    name = "wgrad_tc_kernel" if route == "tap_in_grid" else "wgrad2_tc_kernel"
    assert ran(ks, name) and ran(ks1, name), ks
    e3, e1 = c.err(d3), c.err(d1)
    assert e3 < TOL and 1e-5 < e1 < 5e-3, (e3, e1)


@pytest.mark.parametrize("k,Cout", [(3, 48), (3, 512), (1, 136)])
def test_production_wgrad_matches_explicit_split_bitwise(route, k, Cout):
    """conv.wgrad_tc (the plan's split, torch.empty workspace) and the explicit-split ABI call at that split give
    bit-identical dW, on whichever kernel the routing picks; 4096 output pixels so the plan splits the reduction on the
    full grid.  On a grid capped by BTS_B200_SM_LIMIT the plan may keep one split, and one CTA reducing all 4096 pixels
    is past the ~2k where 3xTF32 meets the bar (see above): there the claim is bit-identity alone."""
    from bts_b200 import conv
    c = Case(1, 64, 64, 64, Cout, k, seed=k * Cout)
    dw, sp, ks = c.run()
    assert sp > 1 or _capped_grid()
    if sp > 1:
        assert c.err(dw) < TOL
    x, gy = nhwc_slice(c.x), nhwc_slice(c.gy)
    gw = conv.wgrad_tc(x, gy, (Cout, 64, k, k), (64 * k * k, k * k, k, 1), 1, c.pad, 1)
    torch.cuda.synchronize()
    assert torch.equal(gw, dw)
    if route == "tap_in_grid":
        assert ran(ks, "wgrad_tc_kernel")


# ---------------------------------------------------------------------------------------- shifted-dY kernel (wgrad2_tc)
@pytest.mark.parametrize("up", [False, True])
@pytest.mark.parametrize("pre", [1, 2])
def test_shifted_dy_pre_ops(shifted_dy, pre, up):
    """wgrad2_tc_kernel<PRE = 1 | 2, UP, VEC, TMA>: the ReLU-only and affine-only pre-ops, with and without the x2
    up-sample (TMA ring: dY segments through the ring, the up-sampled x through the load path); Cout = 40 leaves the
    third 16-channel co-group half live, Cin = 72 a partial 64-channel tile"""
    c = Case(2, 72, 7, 10, 40, 3, pre=pre, up=up, seed=200 + 10 * pre + up)
    dw, _, ks = c.run()
    assert ran(ks, "wgrad2_tc_kernel", (pre, up, True, shifted_dy == "tma_ring")), ks
    assert c.err(dw) < TOL


@pytest.mark.parametrize("pre", [0, 3])
def test_shifted_dy_unaligned_dy_slice(shifted_dy, pre):
    """dY as the slice at channel offset 1 of a wider slab: base not 16-byte aligned, so the scalar-load path (VEC =
    false) runs even where the TMA ring is enabled"""
    c = Case(2, 36, 9, 12, 32, 3, pre=pre, seed=300 + pre)
    dw, _, ks = c.run(dy_width=36, dy_off=1)
    assert ran(ks, "wgrad2_tc_kernel", (pre, False, False, False)), ks
    assert c.err(dw) < TOL


@pytest.mark.parametrize("Cout", [65, 136, 250])
def test_shifted_dy_pointwise_uneven_co_groups(shifted_dy, Cout):
    """1x1 layers with 64 < Cout <= 256 on the single-tap mapping: 65 is one 80-wide co-group with 15 dead columns, 136
    two groups of 80 / 56 live channels, 250 two 128-wide groups, the second with 122 live (odd Cout: scalar dY loads)"""
    c = Case(2, 100, 8, 11, Cout, 1, pre=3, seed=Cout)
    dw, _, ks = c.run()
    assert ran(ks, "wgrad2_tc_kernel", (3,)), ks
    assert c.err(dw) < TOL


@pytest.mark.parametrize("pad", [0, 2])
def test_shifted_dy_padding_not_same(shifted_dy, pad):
    """3x3 at dil = 1 with pad 0 (Hout = Hin - 2) or pad 2 (Hout = Hin + 2): the dY shift of a tap no longer maps the
    input grid onto the output grid, so these shapes skip the landing ring and use the load path"""
    c = Case(2, 64, 11, 13, 48, 3, pad=pad, pre=3, seed=400 + pad)
    dw, _, ks = c.run()
    assert ran(ks, "wgrad2_tc_kernel", (3, False, True, False)), ks
    assert c.err(dw) < TOL


@pytest.mark.parametrize("k,Cout,B,H,W", [(3, 48, 1, 7, 9), (3, 64, 2, 12, 14), (1, 136, 2, 12, 14)])
def test_shifted_dy_splits_beyond_pixels(shifted_dy, k, Cout, B, H, W):
    """splitK = ceil(Mq / 16) + 3: every split owns one 16-pixel block and the last three own no pixel at all; their
    CTAs run no k-block, and their partials must still be written as zeros into the NaN-filled workspace"""
    c = Case(B, 40, H, W, Cout, k, pre=1, seed=500 + Cout)
    split = -(-B * H * W // SPLIT_PX) + 3
    dw, sp, ks = c.run(split=split)
    assert sp == split and ran(ks, "wgrad2_tc_kernel", (1,)), ks
    assert c.err(dw) < TOL


# --------------------------------------------------------------------------------------------- grouped (block-diagonal)
@pytest.mark.parametrize("split", [1, 3, 8])
def test_grouped_forced_split_with_empty_splits(split):
    """bts_conv_wgrad_grouped (ResNeXt 3x3, 32 groups of 8, 128-wide diagonal windows) with forced split counts: 160
    output pixels are 5 k-blocks, so split 3 leaves the last range short and split 8 three ranges empty; every
    [split][tap][width][128] partial must be written before the grouped reduce extracts the diagonal blocks"""
    from bts_b200 import _lib
    from bts_b200.ops import _ptr, _stream
    L = _L()
    width, cpg, B, H, W = 256, 8, 2, 8, 10
    g = torch.Generator().manual_seed(600 + split)
    x = torch.randn(B, width, H, W, generator=g)
    gy = torch.randn(B, width, H, W, generator=g)
    wd = torch.zeros(width, cpg, 3, 3, dtype=torch.float64, requires_grad=True)
    F.conv2d(x.double(), wd, None, 1, 1, 1, width // cpg).backward(gy.double())
    xc, gc = nhwc_slice(x), nhwc_slice(gy)
    ws = nan(split * 9 * width * 128)
    s = (cpg * 9, 9, 3, 1)
    dw, buf, inside = guarded((width, cpg, 3, 3), s)
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        rc = L.bts_conv_wgrad_grouped(_ptr(xc), width, B, H, W, width, cpg, 3, 3, 1, 1, 1, _ptr(gc), width, _ptr(ws), split,
                                      _ptr(dw), s[0], s[1], s[2], s[3], 0, _stream())
        _lib.check(rc, "bts_conv_wgrad_grouped")
        torch.cuda.synchronize()
    assert ran(kernels(prof), "wgrad_tc_kernel", (0, False, True))
    check_written(dw, buf, inside)
    assert float((dw.cpu().double() - wd.grad).abs().max() / wd.grad.abs().max()) < TOL
