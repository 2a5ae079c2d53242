"""GPU parity of the conv engine's wide output tiles (n-tiles of 80..128 channels, bts_conv_n_tile) against torch fp64 on
the CPU, at the 2e-5 output-scale bar of tests/test_conv_gpu.py: forward and dgrad widths, the BatchNorm/ReLU pre-op with
padding, the folded x2 up-sample, the zero-stuffed source of a stride-2 dgrad, channel tails, channel slices of wider slabs,
the epilogue statistics and the BatchNorm-backward epilogue, fast mode, a grouped operator with a 128-wide window, and a
launch with fewer tiles than SMs."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

WIDTHS = [80, 96, 112, 128, 192, 200, 448]


def _cl(t):
    return t.cuda().contiguous(memory_format=torch.channels_last)


def _err(got, ref):
    return float((got.detach().cpu().double() - ref).abs().max() / ref.abs().max().clamp_min(1e-30))


def _bn(C, g):
    return torch.rand(C, generator=g) + 0.5, torch.randn(C, generator=g) * 0.3


@pytest.mark.parametrize("Cout", WIDTHS)
@pytest.mark.parametrize("k,up", [(3, False), (1, False), (3, True)])
def test_wide_forward_with_pre_op(Cout, k, up):
    """affine + ReLU pre-op (padding applied after it), optionally with the x2 up-sample folded into the address map"""
    from bts_b200 import conv
    g = torch.Generator().manual_seed(Cout + 10 * k + up)
    Cin = 68                                   # 17 channel quads: a partial last k-block
    x = torch.randn(2, Cin, 7, 9, generator=g)
    w = torch.randn(Cout, Cin, k, k, generator=g) / (Cin * k * k) ** 0.5
    sc, sh = _bn(Cin, g)
    xd = F.relu(x.double() * sc.double().view(1, -1, 1, 1) + sh.double().view(1, -1, 1, 1))
    if up:
        xd = F.interpolate(xd, scale_factor=2, mode="nearest")
    ref = F.conv2d(xd, w.double(), None, 1, k // 2, 1)
    y = conv.conv2d_tc(_cl(x), w.cuda(), 1, k // 2, 1, sc.cuda(), sh.cuda(), True, up)
    torch.cuda.synchronize()
    assert _err(y, ref) < 2e-5


@pytest.mark.parametrize("Cin", WIDTHS)
def test_wide_dgrad(Cin):
    """the input gradient of a 3x3 conv: the output width is the layer's Cin"""
    from bts_b200 import conv
    g = torch.Generator().manual_seed(Cin)
    Cout = 48
    w = torch.randn(Cout, Cin, 3, 3, generator=g) / (Cout * 9) ** 0.5
    gy = torch.randn(2, Cout, 8, 10, generator=g)
    ref = F.conv_transpose2d(gy.double(), w.double(), None, 1, 1)
    y = conv.conv2d_tc(_cl(gy), w.cuda(), 1, 1, 1, transpose_flip=True)
    torch.cuda.synchronize()
    assert _err(y, ref) < 2e-5


@pytest.mark.parametrize("Cin,Cout", [(96, 30), (200, 13), (112, 64)])
def test_wide_dgrad_of_stride2_conv_zero_stuffed_source(Cin, Cout):
    """source_mode 2 (odd coordinates of the virtual source are zeros) with a channel tail on the K side (Cout % 4 != 0)"""
    from bts_b200 import conv
    g = torch.Generator().manual_seed(Cin + Cout)
    w = torch.randn(Cout, Cin, 3, 3, generator=g) / (Cout * 9) ** 0.5
    H, W = 9, 13
    gy = torch.randn(2, Cout, 5, 7, generator=g)
    ref = F.conv_transpose2d(gy.double(), w.double(), None, 2, 1, output_padding=0)
    assert ref.shape[-2:] == (H, W)
    y = conv.conv2d_tc(_cl(gy), w.cuda(), 1, 1, 1, transpose_flip=True, zero_stuff_out=(H, W))
    torch.cuda.synchronize()
    assert _err(y, ref) < 2e-5


@pytest.mark.parametrize("Cout", [96, 128, 200])
def test_wide_channel_tail_scalar_loads(Cout):
    """Cin % 4 != 0 with an odd pixel stride (4-byte copies) and with a 16-byte aligned stride (partial 16-byte copies)"""
    from bts_b200 import conv
    g = torch.Generator().manual_seed(Cout)
    for Cin, slab in ((37, 37), (37, 40)):
        xs = torch.randn(2, slab, 6, 11, generator=g)
        x = _cl(xs)[:, :Cin]
        w = torch.randn(Cout, Cin, 3, 3, generator=g) / (Cin * 9) ** 0.5
        ref = F.conv2d(xs[:, :Cin].double(), w.double(), None, 1, 1, 1)
        y = conv.conv2d_tc(x, w.cuda(), 1, 1, 1)
        torch.cuda.synchronize()
        assert _err(y, ref) < 2e-5, (Cin, slab)


def test_wide_tiles_read_and_write_channel_slices():
    from bts_b200 import conv
    g = torch.Generator().manual_seed(7)
    slab = _cl(torch.randn(2, 256, 7, 9, generator=g))
    w = (torch.randn(192, 96, 3, 3, generator=g) / 30).cuda()
    out = torch.zeros(2, 448, 7, 9, device="cuda").contiguous(memory_format=torch.channels_last)
    conv.conv2d_tc(slab[:, 64:160], w, 1, 1, 1, out=out[:, 128:320])
    torch.cuda.synchronize()
    ref = F.conv2d(slab[:, 64:160].double().cpu(), w.double().cpu(), None, 1, 1, 1)
    assert _err(out[:, 128:320], ref) < 2e-5
    assert float(out[:, :128].abs().sum()) == 0 and float(out[:, 320:].abs().sum()) == 0


@pytest.mark.parametrize("Cout", [96, 128, 192, 448])
def test_wide_epilogue_statistics(Cout):
    """per-channel sum / sum of squares from the epilogue, with one n-tile (96, 128) and with several (192, 448)"""
    from bts_b200 import conv
    g = torch.Generator().manual_seed(Cout + 1)
    x = _cl(torch.randn(3, 64, 9, 14, generator=g))
    w = (torch.randn(Cout, 64, 3, 3, generator=g) / 24).cuda()
    st = torch.zeros((2, Cout), device="cuda", dtype=torch.float64)
    y = conv.conv2d_tc(x, w, 1, 1, 1, stats=st)
    y0 = conv.conv2d_tc(x, w, 1, 1, 1)
    assert torch.equal(y, y0)
    ref = F.conv2d(x.double().cpu(), w.double().cpu(), None, 1, 1, 1)
    assert _err(y, ref) < 2e-5
    yd = y.double()
    s1, s2 = yd.sum((0, 2, 3)), (yd * yd).sum((0, 2, 3))
    assert (st[0] - s1).abs().max() <= 1e-5 * s2.sqrt().max()
    assert ((st[1] - s2).abs() / s2).max() < 1e-5


@pytest.mark.parametrize("C", [128, 192])
def test_wide_batchnorm_backward_epilogue(C):
    """dgrad whose epilogue also reduces the BatchNorm(+ReLU) backward sums of the layer in front of the conv"""
    from bts_b200 import conv
    g = torch.Generator().manual_seed(C + 2)
    Cout = 48
    w = torch.randn(Cout, C, 3, 3, generator=g) / (Cout * 9) ** 0.5
    gy = torch.randn(2, Cout, 8, 9, generator=g)
    xb = torch.randn(2, C, 8, 9, generator=g)
    sc, sh = _bn(C, g)
    mu, istd = torch.randn(C, generator=g) * 0.1, torch.rand(C, generator=g) + 0.5
    st = torch.stack([sc, sh, mu, istd]).cuda().contiguous()
    sums = torch.zeros((2, C), device="cuda", dtype=torch.float64)
    y = conv.conv2d_tc(_cl(gy), w.cuda(), 1, 1, 1, transpose_flip=True, stats=sums, bn_bwd=(_cl(xb), st, True))
    torch.cuda.synchronize()
    ref = F.conv_transpose2d(gy.double(), w.double(), None, 1, 1)
    assert _err(y, ref) < 2e-5
    xd = xb.double()
    mask = (xd * sc.double().view(1, -1, 1, 1) + sh.double().view(1, -1, 1, 1)) > 0
    gm = y.double().cpu() * mask
    s1 = gm.sum((0, 2, 3))
    t2 = gm * ((xd - mu.double().view(1, -1, 1, 1)) * istd.double().view(1, -1, 1, 1))
    s2 = t2.sum((0, 2, 3))
    assert (sums[0].cpu() - s1).abs().max() <= 1e-5 * gm.abs().sum((0, 2, 3)).max()
    assert (sums[1].cpu() - s2).abs().max() <= 1e-5 * t2.abs().sum((0, 2, 3)).max()


@pytest.mark.parametrize("Cout", [128, 192])
def test_wide_fast_mode_is_labelled_and_less_exact(Cout):
    from bts_b200 import conv
    g = torch.Generator().manual_seed(Cout + 5)
    x = torch.randn(1, 128, 16, 16, generator=g)
    w = torch.randn(Cout, 128, 3, 3, generator=g) / 34
    ref = F.conv2d(x.double(), w.double(), None, 1, 1, 1)
    xc = _cl(x)
    e3 = _err(conv.conv2d_tc(xc, w.cuda(), 1, 1, 1), ref)
    e1 = _err(conv.conv2d_tc(xc, w.cuda(), 1, 1, 1, precision=1), ref)
    assert e3 < 2e-5 and 1e-5 < e1 < 5e-3


def test_grouped_operator_with_a_128_wide_window():
    """ResNeXt-style grouped 3x3 (32 groups x 8): one 128-wide n-tile per diagonal block"""
    from bts_b200 import _lib, conv
    assert _lib.lib().bts_conv_group_n_tile(128) == 128
    g = torch.Generator().manual_seed(11)
    width, cpg = 256, 8
    x = torch.randn(2, width, 8, 10, generator=g)
    w = torch.randn(width, cpg, 3, 3, generator=g) / (cpg * 9) ** 0.5
    ref = F.conv2d(x.double(), w.double(), None, 1, 1, 1, width // cpg)
    y = conv.conv2d_tc(_cl(x), w.cuda(), 1, 1, 1, groups=width // cpg)
    torch.cuda.synchronize()
    assert _err(y, ref) < 2e-5


def test_wide_launch_with_fewer_tiles_than_sms():
    """the dense-block-4 1x1 shape: 31 m-tiles x 2 n-tiles of 96 on a GPU with more SMs than tiles"""
    from bts_b200 import conv
    g = torch.Generator().manual_seed(13)
    Cin = 416
    x = torch.randn(16, Cin, 11, 22, generator=g)
    w = torch.randn(192, Cin, 1, 1, generator=g) / Cin ** 0.5
    sc, sh = _bn(Cin, g)
    xd = F.relu(x.double() * sc.double().view(1, -1, 1, 1) + sh.double().view(1, -1, 1, 1))
    ref = F.conv2d(xd, w.double())
    y = conv.conv2d_tc(_cl(x), w.cuda(), 1, 0, 1, sc.cuda(), sh.cuda(), True)
    torch.cuda.synchronize()
    assert _err(y, ref) < 2e-5
