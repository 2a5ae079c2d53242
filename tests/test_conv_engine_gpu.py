"""GPU parity of the forward / dgrad engine (conv_tc_kernel, csrc/conv_tc.cu) against fp64 on the CPU, at the 2e-5
output-scale bar of tests/test_conv_gpu.py: every <PRE, UP, VEC> instantiation, persistent walks in which every CTA runs
two or three tiles, the K16 layers of the DenseNet-161 encoder and the decoder with a reference sampled on every m-tile,
and the same launches on a capped SM grid (BTS_B200_SM_LIMIT).

The kernel is persistent: its grid is min(tiles, SMs) and CTA b runs tiles b, b + G, b + 2G, ...  What changes from a
CTA's second tile on (the producers' tile cursor, the consumers' tile sum, the stage ring's phases, the epilogue
statistics' flushes, the n-tile when n_tiles does not divide G) is reached only by launches with more tiles than SMs.

Every call writes into a channel slice of a NaN-filled NHWC slab with guard channels on both sides, inside a NaN-filled
buffer: the view must come back finite and everything else NaN.  Each call is profiled (torch.profiler) and the test
asserts which instantiation ran.  The reference (engine_checks.Op) is F.conv2d in fp64 of pre(x) after the nearest
up-sample or zero-stuffing; on the large maps it is computed at sampled output pixels, three in every 128-pixel m-tile in
the engine's pixel order, the partial last tile included, so that one wrong tile cannot hide."""
import os
import subprocess
import sys
import time

import pytest
import torch

import engine_checks as E
from engine_checks import Op

pytestmark = pytest.mark.gpu

TOL = 2e-5
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
WORST = {}          # group -> worst error measured, printed at the end of the module


@pytest.fixture(scope="module", autouse=True)
def _report_worst_errors():
    yield
    for group, (err, where) in sorted(WORST.items()):
        print("\n%-24s worst error %.3g (%s)" % (group, err, where), end="")
    print()


def _record(group, where, err, tol=TOL):
    if err > WORST.get(group, (-1.0, ""))[0]:
        WORST[group] = (err, where)
    assert err < tol, "%s: error %.3g (bar %.3g)" % (where, err, tol)


def _G():
    return torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count


def _cl(t):
    return t.cuda().contiguous(memory_format=torch.channels_last)


def _bn(C, g):
    return torch.rand(C, generator=g) + 0.5, torch.randn(C, generator=g) * 0.3


def _w(Cout, Cin, k, g):
    return torch.randn(Cout, Cin, k, k, generator=g) / (Cin * k * k) ** 0.5


def run(op, x, stats=False, bn_bwd=None, width=None, off=1):
    """op on the GPU through conv.conv2d_tc into a guarded channel slice [off, off + Cout) of a NaN-filled slab:
    (output view, fp64 [2, Cout] statistics or None, the conv_tc_kernel launches recorded)"""
    from bts_b200 import conv
    B, _, Hs, Ws = x.shape
    Ho, Wo = op.out_size(Hs, Ws)
    Cout = op.w.shape[0]
    y, buf, inside = E.guarded_nhwc(B, Cout, Ho, Wo, width, off)
    st = torch.zeros((2, Cout), device="cuda", dtype=torch.float64) if stats or bn_bwd is not None else None
    sc = op.scale.cuda() if op.scale is not None else None
    sh = op.shift.cuda() if op.shift is not None else None
    w = op.weight.cuda()
    conv.pack_weights(w, op.transpose_flip, op.groups)          # packed (and cached) outside the profiled region
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        conv.conv2d_tc(x, w, op.stride, op.pad, op.dil, sc, sh, op.relu, op.mode == 1, op.act, out=y,
                       transpose_flip=op.transpose_flip, stats=st, groups=op.groups,
                       zero_stuff_out=op.out_hw if op.mode == 2 else None, bn_bwd=bn_bwd)
        torch.cuda.synchronize()
    E.check_written(y, buf, inside)
    ks = E.kernels(prof, "conv_tc_kernel")
    if ks:
        print("ran conv_tc_kernel<%s>" % ", ".join(map(str, ks[0][1])))
    return y, st, ks


def _check_sums(got, terms, what):
    """fp64 per-channel sums from the epilogue against the fp64 sums of the terms (B, C, H, W), at the output bar
    applied to the sum of the terms' magnitudes"""
    ref = terms.sum((0, 2, 3), dtype=torch.float64).cpu()
    scale = terms.abs().sum((0, 2, 3), dtype=torch.float64).cpu().clamp_min(1e-30)
    err = float(((got.cpu() - ref).abs() / scale).max())
    _record("statistics", what, err)


# ------------------------------------------------------------------------------------ A. every <PRE, UP, VEC> (24)
@pytest.mark.parametrize("load", ["vec", "x_stride", "x_offset"])
@pytest.mark.parametrize("up", [0, 1, 2])
@pytest.mark.parametrize("pre", [0, 1, 2, 3])
def test_every_instantiation(pre, up, load):
    """conv_tc_kernel<PRE, UP, VEC>: PRE 0 none / 1 ReLU / 2 affine / 3 affine + ReLU, padding applied after the pre-op;
    UP 0 the source as is / 1 the nearest x2 up-sample / 2 the zero-stuffed x2 expansion (the dgrad of a stride-2 conv).
    With a pre-op and UP 2 the reference is zero_stuff(pre(x)): the kernel masks the stuffed zeros after the pre-op, so
    they stay zero whatever the affine shift.  The scalar-load path (VEC = false) is reached with a source slab whose
    pixel stride (71) is not a multiple of 4 and with the source at channel offset 1 (base not 16-byte aligned).
    Cin = 70 leaves a half-filled 16-byte unit; the map has about 2.5 tiles per SM, so every CTA walks 2 or 3 tiles."""
    G = _G()
    B, Cin, Cout, W = 2, 70, 40, 58
    H = E.walk_rows(G, 1, B, W, even=True)
    Hs, Ws = (H, W) if up == 0 else (H // 2, W // 2)
    g = torch.Generator().manual_seed(1000 + 100 * pre + 10 * up + len(load))
    x = torch.randn(B, Cin, Hs, Ws, generator=g)
    sc, sh = _bn(Cin, g) if pre & 2 else (None, None)
    op = Op(_w(Cout, Cin, 3, g), pad=1, scale=sc, shift=sh, relu=bool(pre & 1), mode=up,
            out_hw=(H, W) if up == 2 else None)
    width, off = {"vec": (72, 0), "x_stride": (71, 0), "x_offset": (72, 1)}[load]
    xd = E.nhwc_slice(x, width, off)
    y, _, ks = run(op, xd)
    assert E.ran(ks, "conv_tc_kernel", (pre, up, load == "vec")), ks
    _record("A instantiations", "pre %d up %d %s" % (pre, up, load), E.rel_err(y, op.full(x)))


# --------------------------------------------------------------------------------------------- B. persistent walks
def make_walk(name, G, variant=None):
    """seeded inputs of one persistent-walk case (engine_checks.WALKS), sized for G SMs:
    (shape, op, x on the GPU, run() keywords, expected <PRE, UP, VEC>, bn_bwd reference inputs or None)"""
    s = E.walk_shape(name, G)
    B, Cin, H, W, Cout, k = s["B"], s["Cin"], s["H"], s["W"], s["Cout"], s["k"]
    g = torch.Generator().manual_seed(sum(map(ord, name)) + (7 if variant else 0))
    kw, bnb = {}, None
    if name in ("kb1_stats", "kb_odd", "kb_even", "nt_coprime", "nt_divides", "odd_slice", "ring3"):
        pre = {"kb1_stats": 3, "kb_odd": 0, "kb_even": 1, "nt_coprime": 3, "nt_divides": 2, "odd_slice": 3, "ring3": 3}[name]
        sc, sh = _bn(Cin, g) if pre & 2 else (None, None)
        op = Op(_w(Cout, Cin, k, g), pad=k // 2, scale=sc, shift=sh, relu=bool(pre & 1))
        x = torch.randn(B, Cin, H, W, generator=g)
        kw["stats"] = name not in ("kb_even", "odd_slice")
        if name == "odd_slice":
            kw.update(width=Cout + 5, off=3)          # odd pixel stride and offset: the epilogue's scalar stores
        expect = (pre, 0, 1)
    elif name == "bnbwd":                             # dgrad of a 3x3 layer Cout -> Cin
        op = Op(_w(Cin, Cout, k, g), pad=1, transpose_flip=True)
        x = torch.randn(B, Cin, H, W, generator=g)
        xb = torch.randn(B, Cout, H, W, generator=g)
        sc, sh = _bn(Cout, g)
        mu, istd = torch.randn(Cout, generator=g) * 0.1, torch.rand(Cout, generator=g) + 0.5
        bnb = (xb, torch.stack([sc, sh, mu, istd]), variant == "relu")
        kw["bn_bwd"] = (_cl(xb), bnb[1].cuda().contiguous(), bnb[2])
        expect = (0, 0, 1)
    elif name == "zero_stuffed":                      # dgrad of a stride-2 3x3 layer Cout -> Cin, input H x W
        op = Op(_w(Cin, Cout, k, g), pad=1, transpose_flip=True, mode=2, out_hw=(H, W))
        x = torch.randn(B, Cin, (H - 1) // 2 + 1, (W - 1) // 2 + 1, generator=g)
        expect = (0, 2, 1)
    elif name == "grouped":                           # ResNeXt 3x3: 32 groups of 8 channels
        op = Op(_w(Cout, 8, k, g), pad=1, groups=Cin // 8)
        x = torch.randn(B, Cin, H, W, generator=g)
        expect = (0, 0, 1)
    else:                                             # "act"
        op = Op(_w(Cout, Cin, k, g), pad=1, act=variant)
        x = torch.randn(B, Cin, H, W, generator=g)
        expect = (0, 0, 1)
    return s, op, x, kw, expect, bnb


WALK_RUNS = [("kb1_stats", None), ("kb_odd", None), ("kb_even", None), ("nt_coprime", None), ("nt_divides", None),
             ("bnbwd", "relu"), ("bnbwd", "no_relu"), ("zero_stuffed", None), ("grouped", None), ("act", "elu"),
             ("act", "sigmoid"), ("odd_slice", None), ("ring3", None)]


def _walk_properties(name, s, G):
    assert s["tiles"] > G and s["tiles"] % G and s["M"] % E.BLOCK_M, s     # 2-3 tiles per CTA, unequal walks
    if name == "kb1_stats":
        assert s["KB"] == 1
    if name == "kb_odd":
        assert s["KB"] > 1 and s["KB"] % 2 == 1
    if name == "kb_even":
        assert s["KB"] % 2 == 0
    if name == "nt_coprime":
        assert s["n_tiles"] > 1 and E.coprime(s["n_tiles"], G), s
    if name == "nt_divides":
        assert s["n_tiles"] > 1 and G % s["n_tiles"] == 0, s
    if name == "grouped":
        assert s["n_tiles"] == 2
    if name == "ring3":
        assert E.ring_stages(s["Cin"], s["n_tile"], True, True) == 3


@pytest.mark.parametrize("name,variant", WALK_RUNS, ids=["%s-%s" % r if r[1] else r[0] for r in WALK_RUNS])
def test_persistent_walk(name, variant):
    """About 2.5 tiles per SM, a tile count that is not a multiple of the SM count (CTAs walk 2 or 3 tiles) and a
    partial last m-tile: KB = 1 (each producer group fills whole tiles in turn), odd KB (the group filling k-block 0
    alternates from tile to tile) and even KB; 5 n-tiles of 112 (coprime with the SM count: the n-tile changes along a
    walk) and 2 of 96 (it stays); the epilogue statistics flushed once per CTA (one n-tile) and after every tile
    (several); the BatchNorm-backward epilogue with and without its ReLU mask; a zero-stuffed stride-2 dgrad; a
    grouped operator with two 128-wide n-tiles; ELU and sigmoid; an output at an odd channel offset (scalar stores); the
    3-stage smem ring (affine pre-op over 2300 channels, statistics, 128-wide tiles)."""
    G = _G()
    s, op, x, kw, expect, bnb = make_walk(name, G, variant)
    _walk_properties(name, s, G)
    xg = _cl(x)
    y, st, ks = run(op, xg, **kw)
    assert E.ran(ks, "conv_tc_kernel", expect), ks
    where = name + ("-" + variant if variant else "")
    if name == "ring3":                               # 2300-channel source: the reference is sampled
        m = E.sample_pixels(s["M"], 3, seed=1)
        _record("B walks", where, E.rel_err(E.pixels_of(y, m), op.sample(xg, m)))
        _check_sums(st[0], y, where + " sum")
        _check_sums(st[1], y.square(), where + " sum of squares")
        return
    ref = op.full(x)
    _record("B walks", where, E.rel_err(y, ref))
    if bnb is not None:
        xb, bst, relu = bnb
        xd, c = xb.double(), lambda v: v.double().view(1, -1, 1, 1)
        gm = ref * ((xd * c(bst[0]) + c(bst[1]) > 0) if relu else 1)
        _check_sums(st[0], gm, where + " S1")
        _check_sums(st[1], gm * ((xd - c(bst[2])) * c(bst[3])), where + " S2")
    elif st is not None:
        _check_sums(st[0], ref, where + " sum")
        _check_sums(st[1], ref * ref, where + " sum of squares")


# ------------------------------------------------------------------------------------- C. K16 layers, sampled reference
K16 = ["stem", "db1_conv1", "db1_conv2", "db1_dgrad", "upconv1", "conv1"]


@pytest.mark.parametrize("layer", K16)
def test_k16_layer_sampled(layer):
    """The K16 shapes of tools/conv_layers.py (352 x 704 input) with the pre-ops, statistics and outputs of fused.py and
    model.py: the DenseNet-161 stem 7x7/2 3 -> 96 (pixel stride 3: VEC = false, 7744 tiles); dense block 1, layer 4:
    conv1 1x1 240 -> 192 reading the block's 384-channel slab through the BatchNorm + ReLU prologue, with statistics;
    conv2 3x3 192 -> 48 with the prologue and statistics, written into channels [240, 288) of the slab; the dgrad of
    that 3x3 (48 -> 192); the decoder's upconv1 (64 -> 32, x2 up-sample, ELU) and conv1 (36 -> 32, ELU) at B = 8 to stay
    under 1.5 GB.  The output is checked at three pixels of every m-tile; the statistics against the fp64 sums of the
    output, which is verified on every tile."""
    g = torch.Generator().manual_seed(sum(map(ord, layer)))
    kw, stats = dict(width=None, off=2), False
    if layer == "stem":
        x = _cl(torch.randn(16, 3, 352, 704, generator=g))
        op = Op(_w(96, 3, 7, g), stride=2, pad=3)
        kw.update(width=100)
    elif layer == "db1_conv1":
        slab = _cl(torch.randn(16, 384, 88, 176, generator=g))
        x = slab[:, :240]
        sc, sh = _bn(240, g)
        op = Op(_w(192, 240, 1, g), scale=sc, shift=sh, relu=True)
        stats, kw["width"] = True, 196
    elif layer == "db1_conv2":
        x = _cl(torch.randn(16, 192, 88, 176, generator=g))
        sc, sh = _bn(192, g)
        op = Op(_w(48, 192, 3, g), pad=1, scale=sc, shift=sh, relu=True)
        stats, kw = True, dict(width=384, off=240)
    elif layer == "db1_dgrad":
        x = _cl(torch.randn(16, 48, 88, 176, generator=g))
        op = Op(_w(48, 192, 3, g), pad=1, transpose_flip=True)
        kw["width"] = 196
    elif layer == "upconv1":
        x = _cl(torch.randn(8, 64, 176, 352, generator=g))
        op = Op(_w(32, 64, 3, g), pad=1, mode=1, act="elu")
        kw["width"] = 36
    else:
        x = _cl(torch.randn(8, 36, 352, 704, generator=g))
        op = Op(_w(32, 36, 3, g), pad=1, act="elu")
        kw["width"] = 36
    y, st, ks = run(op, x, stats=stats, **kw)
    assert E.ran(ks, "conv_tc_kernel", (op.pre, op.mode, layer != "stem")), ks
    B, Cout, Ho, Wo = y.shape
    m = E.sample_pixels(B * Ho * Wo, 3, seed=2)
    K = x.shape[1] * op.w.shape[2] ** 2
    _record("C K16 sampled", layer, E.rel_err(E.pixels_of(y, m), op.sample(x, m)), max(TOL, 8e-9 * K))
    if stats:
        _check_sums(st[0], y, layer + " sum")
        _check_sums(st[1], y.square(), layer + " sum of squares")


# ------------------------------------------------------------------------------------------------ D. capped SM grid
def walk_outputs():
    """every persistent-walk run, sized for this device's SM count: name -> (output, statistics or None) on the CPU"""
    G = _G()
    out = {}
    for name, variant in WALK_RUNS:
        s, op, x, kw, _, _ = make_walk(name, G, variant)
        y, st, _ = run(op, _cl(x), **kw)
        out["%s-%s" % (name, variant)] = (y.cpu(), None if st is None else st.cpu())
    return out


def _python():
    return [sys.executable] + (["-s"] if sys.flags.no_user_site else [])


def _capped(cap, args, timeout):
    env = dict(os.environ, BTS_B200_SM_LIMIT=str(cap))
    t0 = time.time()
    r = subprocess.run(_python() + args, cwd=ROOT, env=env, capture_output=True, text=True, timeout=timeout)
    print("BTS_B200_SM_LIMIT=%d: %s ... exit %d in %.0f s" % (cap, " ".join(args[:3]), r.returncode, time.time() - t0))
    if r.returncode:
        print(r.stdout[-20000:], r.stderr[-5000:])
    assert r.returncode == 0, "the run under BTS_B200_SM_LIMIT=%d failed (its output is printed above)" % cap
    return r


@pytest.mark.skipif("BTS_B200_SM_LIMIT" in os.environ, reason="already under a capped SM grid")
def test_capped_sm_grid(tmp_path):
    """BTS_B200_SM_LIMIT caps the grid of every persistent or grid-capped kernel; the library reads it once per process,
    so this runs subprocesses.  (1) The persistent-walk runs at the full grid, at 7 SMs and at 1 (one CTA walks every
    tile): a tile's arithmetic does not depend on the CTA that runs it, so the outputs are bit-identical; the
    statistics sum per-CTA fp64 partials with atomics in a varying order and agree to 1e-12 of each quantity's largest
    channel.  (2) Under 7 SMs, the parity tests of the kernels whose grids, split plans or workspaces read the SM
    count: this file, both wgrad kernels, the single-output-channel and CUDA-core pointwise kernels, the depthwise
    kernels."""
    full = walk_outputs()
    for cap in (7, 1):
        path = str(tmp_path / ("walks_%d.pt" % cap))
        code = ("import sys, torch; sys.path.insert(0, 'tests'); import test_conv_engine_gpu as t; "
                "torch.save(t.walk_outputs(), sys.argv[1])")
        _capped(cap, ["-c", code, path], 900)
        capped = torch.load(path)
        assert capped.keys() == full.keys()
        for key, (y, st) in full.items():
            yc, stc = capped[key]
            assert torch.equal(y, yc), "%s: output differs at BTS_B200_SM_LIMIT=%d" % (key, cap)
            if st is not None:          # relative to each quantity's largest channel: a sum may nearly cancel
                assert float(((stc - st).abs() / st.abs().amax(1, keepdim=True)).max()) < 1e-12, (key, cap)
    _capped(7, ["-m", "pytest", "-q", "-p", "no:cacheprovider",
                "tests/test_conv_engine_gpu.py", "tests/test_wgrad_engines_gpu.py",
                "tests/test_conv_gpu.py::test_single_output_channel_head_kernels",
                "tests/test_conv_gpu.py::test_pointwise_forward_and_dgrad_cuda_core_kernel",
                "tests/test_conv_gpu.py::test_pointwise_wgrad_cuda_core_kernel",
                "tests/test_conv_gpu.py::test_wgrad_pointwise_wide_tile_on_shifted_dy_kernel",
                "tests/test_mobilenet_gpu.py::test_depthwise_kernels_vs_fp64",
                "tests/test_mobilenet_gpu.py::test_depthwise_kernels_read_channel_slices",
                "tests/test_mobilenet_gpu.py::test_depthwise_statistics_are_bit_reproducible",
                "tests/test_mobilenet_gpu.py::test_depthwise_kernels_walk_several_tiles_per_cta"], 2400)
