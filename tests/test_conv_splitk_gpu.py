"""GPU parity of the split-K mode of the forward / dgrad engine (csrc/conv_tc.cu: conv_tc_kernel / conv_tf32_kernel with
CTAs per (split, tile group) writing raw partial tile sums to a workspace, then conv_splitk_reduce_kernel adding them in a
fixed order and applying the activation) against fp64 on the CPU, at the 2e-5 output-scale bar of test_conv_engine_gpu.py.

Every call forces a split count through conv2d_tc(splits=n) and writes into a channel slice of a NaN-filled NHWC slab
inside a NaN-filled buffer (the view must come back finite, everything else NaN); torch.profiler confirms that the conv
kernel ran with the expected template arguments and that the reduce kernel ran after it."""
import pytest
import torch

import engine_checks as E
from engine_checks import Op

pytestmark = pytest.mark.gpu

TOL = 2e-5
REDUCE = "conv_splitk_reduce_kernel"


def _G():
    return torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count


def _cl(t):
    return t.cuda().contiguous(memory_format=torch.channels_last)


def _w(Cout, Cin, k, g):
    return torch.randn(Cout, Cin, k, k, generator=g) / (Cin * k * k) ** 0.5


def run(op, x, splits, width=None, off=1, precision=None, kernel="conv_tc_kernel"):
    """op on the GPU through conv.conv2d_tc(splits=splits) into a guarded channel slice [off, off + Cout): the output
    view and the engine kernels recorded, after asserting that `kernel` ran once and the reduce kernel once"""
    from bts_b200 import conv
    B, _, Hs, Ws = x.shape
    Ho, Wo = op.out_size(Hs, Ws)
    Cout = op.w.shape[0]
    y, buf, inside = E.guarded_nhwc(B, Cout, Ho, Wo, width, off)
    sc = op.scale.cuda() if op.scale is not None else None
    sh = op.shift.cuda() if op.shift is not None else None
    w = op.weight.cuda()
    conv.pack_weights(w, op.transpose_flip, op.groups)
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        conv.conv2d_tc(x, w, op.stride, op.pad, op.dil, sc, sh, op.relu, op.mode == 1, op.act, out=y,
                       transpose_flip=op.transpose_flip, groups=op.groups, precision=precision,
                       zero_stuff_out=op.out_hw if op.mode == 2 else None, splits=splits)
        torch.cuda.synchronize()
    E.check_written(y, buf, inside)
    names = [e.name for e in prof.events()]
    ks = E.kernels(prof, "conv_tc_kernel|conv_tf32_kernel")
    if ks:           # CUPTI now and then records no kernel of a region this short (engine_checks.ran)
        assert [n for n, _ in ks] == [kernel], ks
        assert sum(REDUCE in n for n in names) == 1, names
    return y, ks


def _plan(op, x, splits):
    from bts_b200 import conv
    B, Cin, Hs, Ws = x.shape
    Ho, Wo = op.out_size(Hs, Ws)
    k = op.w.shape[2]
    return conv.splitk_plan(B, Ho, Wo, 0, Cin, k, k, op.w.shape[0], splits)[0]


# ------------------------------------------------------------------------------------- every <PRE, UP, VEC>, 2 / 3 splits
@pytest.mark.parametrize("splits", [2, 3])
@pytest.mark.parametrize("load", ["vec", "x_stride", "x_offset"])
@pytest.mark.parametrize("up", [0, 1, 2])
@pytest.mark.parametrize("pre", [0, 1, 2, 3])
def test_every_instantiation_split(pre, up, load, splits):
    """conv_tc_kernel<PRE, UP, VEC> in split mode.  Cin = 86 (a half-filled channel quad) at 3x3 is 25 k-blocks: 2 splits
    of 13 and 3 of 9, so a range starts in the middle of a tap and the last one runs 1 or 2 k-blocks past KB (padding that
    must add zeros).  The map is about 0.4 tiles per SM: with 3 splits each CTA of the grid (a third of the SMs per split)
    walks one or two tiles.  The output goes to a 16-byte aligned slice (the reduce kernel's vector stores) with 2 splits
    and to an odd channel offset with 3."""
    G = _G()
    B, Cin, Cout, W = 1, 86, 40, 58
    H = E.walk_rows(G, 1, B, W, even=True, target=0.4)
    Hs, Ws = (H, W) if up == 0 else (H // 2, W // 2)
    g = torch.Generator().manual_seed(2000 + 100 * pre + 10 * up + len(load) + splits)
    x = torch.randn(B, Cin, Hs, Ws, generator=g)
    sc, sh = (torch.rand(Cin, generator=g) + 0.5, torch.randn(Cin, generator=g) * 0.3) if pre & 2 else (None, None)
    op = Op(_w(Cout, Cin, 3, g), pad=1, scale=sc, shift=sh, relu=bool(pre & 1), mode=up,
            out_hw=(H, W) if up == 2 else None)
    width, off = {"vec": (88, 0), "x_stride": (87, 0), "x_offset": (88, 1)}[load]
    xd = E.nhwc_slice(x, width, off)
    assert E.kblocks(Cin, 3) == 25 and _plan(op, xd, splits) == splits
    y, ks = run(op, xd, splits, *((Cout + 8, 4) if splits == 2 else (Cout + 5, 3)))
    if ks:
        assert ks[0][1] == (pre, up, load == "vec"), ks
    assert E.rel_err(y, op.full(x)) < TOL


@pytest.mark.parametrize("act", ["elu", "sigmoid"])
def test_activation_in_the_reduce(act):
    """ELU / sigmoid are applied once, to the sum of the splits, by the reduce kernel"""
    g = torch.Generator().manual_seed(31 if act == "elu" else 32)
    x = torch.randn(1, 64, 30, 41, generator=g)
    op = Op(_w(48, 64, 3, g), pad=1, act=act)
    y, _ = run(op, _cl(x), 3)
    assert E.rel_err(y, op.full(x)) < TOL


def test_grouped_operator_split():
    """ResNeXt 3x3 block-diagonal operator (32 groups of 8, window 128, two n-tiles) with 3 splits of its 36 k-blocks"""
    g = torch.Generator().manual_seed(41)
    x = torch.randn(1, 256, 17, 23, generator=g)
    op = Op(_w(256, 8, 3, g), pad=1, groups=32)
    y, _ = run(op, _cl(x), 3)
    assert E.rel_err(y, op.full(x)) < TOL


def test_dgrad_split_with_dilation():
    """the transposed, tap-flipped operator of a dilated 3x3 (a DASPP layer's dgrad), 4 splits"""
    g = torch.Generator().manual_seed(43)
    x = torch.randn(1, 128, 26, 34, generator=g)
    op = Op(_w(128, 96, 3, g), pad=6, dil=6, transpose_flip=True)
    y, _ = run(op, _cl(x), 4)
    assert E.rel_err(y, op.full(x)) < TOL


def test_tiles_outnumber_the_split_grid():
    """5 n-tiles of 112, about 0.9 tiles per SM and 3 splits: each split gets a third of the SMs, so its CTAs walk two or
    three tiles and the n-tile changes along a walk"""
    G = _G()
    g = torch.Generator().manual_seed(47)
    W = 29
    H = E.walk_rows(G, 5, 1, W, target=0.9)
    x = torch.randn(1, 96, H, W, generator=g)
    op = Op(_w(560, 96, 3, g), pad=1)
    tiles = -(-H * W // E.BLOCK_M) * 5
    assert tiles > 2 * (G // 3)
    y, _ = run(op, _cl(x), 3)
    assert E.rel_err(y, op.full(x)) < TOL


def test_single_pass_tf32_split():
    """conv_tf32_kernel in split mode at the bar of test_tf32_engines_gpu.py (1e-5 < err < 5e-3: one product ran)"""
    g = torch.Generator().manual_seed(53)
    x = torch.randn(1, 68, 30, 41, generator=g)
    sc, sh = torch.rand(68, generator=g) + 0.5, torch.randn(68, generator=g) * 0.3
    op = Op(_w(40, 68, 3, g), pad=1, scale=sc, shift=sh, relu=True)
    y, ks = run(op, _cl(x), 2, precision=1, kernel="conv_tf32_kernel")
    if ks:
        assert ks[0][1] == (3, 0, 1), ks
    assert 1e-5 < E.rel_err(y, op.full(x)) < 5e-3


def test_split_is_bit_reproducible():
    """the splits are added in a fixed order: two runs give the same bits"""
    g = torch.Generator().manual_seed(59)
    x = _cl(torch.randn(1, 256, 26, 34, generator=g))
    op = Op(_w(128, 256, 3, g), pad=1, act="elu")
    a, _ = run(op, x, 4)
    b, _ = run(op, x, 4)
    assert torch.equal(a, b)


def test_split_rejects_epilogue_reductions():
    """split mode has no statistics and no BatchNorm-backward epilogue: forcing it with either raises"""
    from bts_b200 import conv
    g = torch.Generator().manual_seed(61)
    x = _cl(torch.randn(1, 64, 12, 14, generator=g))
    w = _w(48, 64, 3, g).cuda()
    st = torch.zeros((2, 48), device="cuda", dtype=torch.float64)
    with pytest.raises(ValueError, match="BTS_EINVAL"):
        conv.conv2d_tc(x, w, 1, 1, 1, stats=st, splits=2)
    xb = _cl(torch.randn(1, 48, 12, 14, generator=g))              # the dgrad of a 48 -> 64 layer writes 48 channels
    bst = torch.ones((4, 48), device="cuda")
    with pytest.raises(ValueError, match="BatchNorm-backward"):
        conv.conv2d_tc(x, _w(64, 48, 3, g).cuda(), 1, 1, 1, transpose_flip=True, stats=torch.zeros_like(st),
                       bn_bwd=(xb, bst, True), splits=2)
    y = conv.conv2d_tc(x, w, 1, 1, 1, stats=st, splits=1)      # 1: the plain launch, statistics included
    torch.cuda.synchronize()
    assert bool(torch.isfinite(y).all()) and bool(st.abs().sum() > 0)


def test_inference_scope_gates_the_split():
    """conv2d_tc splits a launch that fills at most half the SMs only inside conv.inference() and without statistics;
    the result agrees with the unsplit launch at the bar"""
    from bts_b200 import conv
    g = torch.Generator().manual_seed(67)
    x = _cl(torch.randn(1, 512, 26, 34, generator=g))
    w = _w(256, 512, 3, g).cuda()

    def profiled(fn):
        torch.cuda.synchronize()
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            y = fn()
            torch.cuda.synchronize()
        return y, sum(REDUCE in e.name for e in prof.events()), len(E.kernels(prof, "conv_tc_kernel"))

    y0, r0, _ = profiled(lambda: conv.conv2d_tc(x, w, 1, 1, 1, act="elu"))
    with conv.inference():
        y1, r1, k1 = profiled(lambda: conv.conv2d_tc(x, w, 1, 1, 1, act="elu"))
        st = torch.zeros((2, 256), device="cuda", dtype=torch.float64)
        _, r2, _ = profiled(lambda: conv.conv2d_tc(x, w, 1, 1, 1, stats=st))
    assert r0 == 0 and r2 == 0
    if k1:
        assert r1 == 1
    assert float((y1 - y0).abs().max() / y0.abs().max()) < TOL
