"""CPU checks of what tests/test_conv_engine_gpu.py stands on: its sampled fp64 reference equals F.conv2d (and the
zero-stuffed source equals the input gradient of a stride-2 conv), the sampled pixels cover every m-tile, the
persistent-walk shapes meet their tile-count, k-block and n-tile conditions on an H100 SXM (132 SMs) and an H100 PCIe
(114), with the library's own n-tile plan and packed-operator sizes, and the 3-stage smem ring case lies where the plan
gives 3 stages.  No GPU: the library's host-side planning functions load without one."""
import pytest
import torch
import torch.nn.functional as F

import engine_checks as E
from engine_checks import Op

SM_COUNTS = [132, 114]


def _case(pre, mode, seed, transpose_flip=False, stride=1, dil=1):
    g = torch.Generator().manual_seed(seed)
    Cin, Cout, k = 6, 5, 3
    x = torch.randn(2, Cin, 5, 7, generator=g)
    sc, sh = (torch.rand(Cin, generator=g) + 0.5, torch.randn(Cin, generator=g)) if pre & 2 else (None, None)
    w = torch.randn(Cin, Cout, k, k, generator=g) if transpose_flip else torch.randn(Cout, Cin, k, k, generator=g)
    return x, Op(w, stride=stride, pad=dil, dil=dil, scale=sc, shift=sh, relu=bool(pre & 1), mode=mode,
                 out_hw=(9, 13) if mode == 2 else None, transpose_flip=transpose_flip)


@pytest.mark.parametrize("mode", [0, 1, 2])
@pytest.mark.parametrize("pre", [0, 1, 2, 3])
def test_sampled_reference_equals_conv2d(pre, mode):
    """every output pixel through Op.sample == F.conv2d of pre(x) after the up-sample / zero-stuffing; with a shift the
    stuffed zeros of mode 2 stay zero (pre-op first, then the expansion)"""
    x, op = _case(pre, mode, 10 * pre + mode)
    s = op.pre_op(x)
    if mode == 1:
        s = F.interpolate(s, scale_factor=2, mode="nearest")
    elif mode == 2:
        s = torch.zeros(2, 6, 10, 14, dtype=torch.float64)
        s[:, :, ::2, ::2] = op.pre_op(x)
    ref = F.conv2d(s, op.w.double(), None, 1, 1, 1)
    if mode == 2:
        ref = ref[:, :, :9, :13]
    full = op.full(x)
    assert full.shape == ref.shape and torch.allclose(full, ref, rtol=0, atol=1e-12)
    M = ref.shape[0] * ref.shape[2] * ref.shape[3]
    got = op.sample(x, torch.arange(M), chunk=37)
    assert torch.allclose(got, ref.permute(0, 2, 3, 1).reshape(M, -1), rtol=0, atol=1e-12)
    if mode == 2 and pre == 2:          # the pre-op applied after the stuffing would turn the stuffed zeros into shifts
        z = torch.zeros(2, 6, 10, 14)
        z[:, :, ::2, ::2] = x
        assert not torch.allclose(F.conv2d(op.pre_op(z), op.w.double(), None, 1, 1, 1)[:, :, :9, :13], ref)


@pytest.mark.parametrize("stride,dil", [(2, 1), (1, 2)])
def test_sampled_reference_strided_dilated_and_grouped(stride, dil):
    x, op = _case(3, 0, 40 + stride + dil, stride=stride, dil=dil)
    M = op.full(x).numel() // 5
    ref = op.full(x)
    assert ref.shape[2:] == F.conv2d(x, op.w, None, stride, dil, dil).shape[2:]
    got = op.sample(x, torch.arange(M), chunk=11)
    assert torch.allclose(got, ref.permute(0, 2, 3, 1).reshape(M, -1), rtol=0, atol=1e-12)
    g = torch.Generator().manual_seed(5)
    xg, wg = torch.randn(1, 16, 6, 5, generator=g), torch.randn(16, 4, 3, 3, generator=g)
    opg = Op(wg, pad=1, groups=4)
    ref = F.conv2d(xg.double(), wg.double(), None, 1, 1, 1, 4)
    assert torch.allclose(opg.full(xg), ref, rtol=0, atol=1e-12)
    assert torch.allclose(opg.sample(xg, torch.arange(30)), ref.permute(0, 2, 3, 1).reshape(30, -1), rtol=0, atol=1e-12)


def test_zero_stuffed_dgrad_is_the_input_gradient_of_a_stride2_conv():
    """mode 2 with the transposed, tap-flipped operator at pad' = dil * (k - 1) - pad is dL/dx of a stride-2 conv, for
    an even and an odd input size"""
    g = torch.Generator().manual_seed(3)
    w = torch.randn(5, 6, 3, 3, generator=g, dtype=torch.float64)
    for H, W in ((10, 14), (9, 13)):
        Ho, Wo = (H - 1) // 2 + 1, (W - 1) // 2 + 1
        gy = torch.randn(2, 5, Ho, Wo, generator=g)
        op = Op(w, pad=1, mode=2, out_hw=(H, W), transpose_flip=True)
        ref = torch.nn.grad.conv2d_input((2, 6, H, W), w, gy.double(), 2, 1)
        assert torch.allclose(op.full(gy), ref, rtol=0, atol=1e-12)


def test_sampled_pixels_cover_every_m_tile():
    for M in (128 * 7, 128 * 7 + 1, 128 * 7 + 77, 5):
        m = E.sample_pixels(M, 3, seed=M)
        assert int(m.max()) == M - 1 and int(m.min()) == 0
        per_tile = torch.bincount(m // E.BLOCK_M)
        live = (M - torch.arange(per_tile.numel()) * E.BLOCK_M).clamp(max=E.BLOCK_M)
        assert per_tile.numel() == -(-M // E.BLOCK_M) and bool((per_tile >= live.clamp(max=2)).all())
    y = torch.arange(2 * 3 * 4 * 5, dtype=torch.float32).view(2, 3, 4, 5)
    m = torch.tensor([0, 7, 39])
    assert torch.equal(E.pixels_of(y, m), y.permute(0, 2, 3, 1).reshape(40, 3)[m])


@pytest.mark.parametrize("G", SM_COUNTS)
@pytest.mark.parametrize("name", list(E.WALKS))
def test_walk_shapes(name, G):
    """about 2.5 tiles per SM, not a multiple of G, a partial last m-tile; the n-tile plan and the k-block count agree
    with the library's packed-operator size"""
    from bts_b200 import _lib
    L = _lib.lib()
    s = E.walk_shape(name, G)
    assert s["M"] % E.BLOCK_M and s["tiles"] % G and 2.2 * G <= s["tiles"] <= 2.8 * G, s
    if name == "grouped":
        assert L.bts_conv_group_n_tile(L.bts_conv_group_window(s["Cin"], 8)) == s["n_tile"] == 128
        packed = L.bts_conv_packed_floats_grouped(s["Cin"], 8, s["k"], s["k"])
    else:
        assert L.bts_conv_n_tile(s["Cout"]) == s["n_tile"]
        packed = L.bts_conv_packed_floats(s["Cout"], s["Cin"], s["k"], s["k"])
    assert packed == s["n_tiles"] * s["KB"] * 2 * s["n_tile"] * 32
    want = {"kb1_stats": lambda: s["KB"] == 1,
            "kb_odd": lambda: s["KB"] > 1 and s["KB"] % 2 == 1,
            "kb_even": lambda: s["KB"] % 2 == 0,
            "nt_coprime": lambda: s["n_tiles"] == 5 and s["n_tile"] == 112 and E.coprime(s["n_tiles"], G),
            "nt_divides": lambda: s["n_tiles"] == 2 and s["n_tile"] == 96 and G % s["n_tiles"] == 0,
            "grouped": lambda: s["n_tiles"] == 2,
            "ring3": lambda: 2273 <= s["Cin"] <= 4096 and s["n_tile"] == 128}.get(name, lambda: True)
    assert want(), s


@pytest.mark.parametrize("G", SM_COUNTS)
def test_instantiation_map_walks_two_or_three_tiles(G):
    H = E.walk_rows(G, 1, 2, 58, even=True)
    M = 2 * H * 58
    tiles = -(-M // E.BLOCK_M)
    assert H % 2 == 0 and M % E.BLOCK_M and tiles % G and 2 * G < tiles < 3 * G


def test_three_stage_ring_needs_statistics_an_affine_pre_op_and_2273_to_4096_channels():
    """conv_fwd_impl's smem plan at 128-wide tiles: 3 stages only with the statistics partials and a staged scale / shift
    of more than 71 32-channel chunks; the pre-op is limited to 4096 input channels"""
    Cin = E.WALKS["ring3"]["Cin"]
    assert 2273 <= Cin <= 4096 and E.ring_stages(Cin, 128, True, True) == 3
    assert E.ring_stages(2272, 128, True, True) == 4 and E.ring_stages(2273, 128, True, True) == 3
    assert E.ring_stages(4096, 128, True, True) == 3
    assert E.ring_stages(4096, 128, False, True) == 4 and E.ring_stages(4096, 112, True, True) == 4
