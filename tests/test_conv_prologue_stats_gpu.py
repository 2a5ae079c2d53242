"""GPU parity of the conv engine's forward with the fused BatchNorm/ReLU prologue and statistics epilogue, and of its dgrad,
against torch fp64 on the CPU.  Same checker and tolerance as tests/test_conv_gpu.py: 1x1 and multi-tap layers, atrous
dilations, channel tails, wide tiles, and a source that is a channel slice of a wider slab."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("B,Cin,H,W,Cout,k,pad,dil,pre", [
    (2, 64, 12, 20, 48, 1, 0, 1, False),       # 1x1, M tail (480 px)
    (1, 32, 16, 16, 16, 3, 1, 1, False),       # 3x3, exact 2 tiles, one k-block per tap
    (2, 192, 9, 11, 48, 3, 1, 1, True),        # dense-layer 3x3 with the BN+ReLU prologue
    (1, 256, 11, 22, 128, 3, 3, 3, True),      # atrous d=3
    (1, 64, 11, 22, 32, 3, 12, 12, False),     # atrous d=12
    (3, 128, 7, 9, 64, 3, 1, 1, False),        # tiles straddle rows and images
    (1, 96, 12, 16, 256, 3, 1, 1, False),      # 256-wide tile
    (1, 32, 20, 24, 16, 7, 3, 1, False),       # 49 taps (more than the 32-bit tap mask covers)
    (1, 256, 6, 8, 256, 1, 0, 1, True),        # 1x1 with prologue, 256-wide tile
    (2, 96, 10, 14, 192, 1, 0, 1, True),       # dense 1x1
    (2, 36, 10, 12, 64, 3, 1, 1, True),        # prologue over 9 channel quads: a partial last k-block
    (1, 3, 20, 24, 64, 7, 3, 1, False),        # 7x7 stem over 3 channels: 4-byte copies (pixel stride 3)
])
def test_conv_fwd_dgrad_prologue_stats(B, Cin, H, W, Cout, k, pad, dil, pre):
    from bts_b200 import conv
    g = torch.Generator().manual_seed(Cin + Cout + k + dil)
    x = torch.randn(B, Cin, H, W, generator=g)
    w = torch.randn(Cout, Cin, k, k, generator=g) / (Cin * k * k) ** 0.5
    sc = sh = None
    xd = x.double()
    if pre:
        sc, sh = torch.rand(Cin, generator=g) + 0.5, torch.randn(Cin, generator=g) * 0.3
        xd = F.relu(xd * sc.double().view(1, -1, 1, 1) + sh.double().view(1, -1, 1, 1))
    ref = F.conv2d(xd, w.double(), None, 1, pad, dil)
    xc = x.cuda().contiguous(memory_format=torch.channels_last)
    st = torch.zeros(2, Cout, device="cuda", dtype=torch.float64)
    y = conv.conv2d_tc(xc, w.cuda(), 1, pad, dil, pre_scale=sc.cuda() if pre else None, pre_shift=sh.cuda() if pre else None,
                       pre_relu=pre, stats=st)
    torch.cuda.synchronize()
    assert float((y.cpu().double() - ref).abs().max() / ref.abs().max()) < 2e-5
    assert torch.allclose(st[0].cpu(), ref.sum((0, 2, 3)), rtol=1e-4, atol=1e-3)
    # dgrad = the same engine over the transposed, tap-flipped operator (its K channels are the layer's Cout)
    gy = torch.randn(ref.shape, generator=g)
    gref = torch.nn.grad.conv2d_input(x.shape, w.double(), gy.double(), 1, pad, dil)
    gx = conv.conv2d_tc(gy.cuda().contiguous(memory_format=torch.channels_last), w.cuda(), 1, dil * (k - 1) - pad, dil,
                        transpose_flip=True)
    torch.cuda.synchronize()
    assert float((gx.cpu().double() - gref).abs().max() / gref.abs().max()) < 2e-5


def test_conv_reads_a_channel_slice_of_a_slab_and_feeds_the_stats_epilogue():
    from bts_b200 import conv
    g = torch.Generator().manual_seed(5)
    slab = torch.randn(2, 160, 9, 13, generator=g).cuda().contiguous(memory_format=torch.channels_last)
    x = slab[:, 32:128]                                        # 96 channels at offset 32 of a 160-channel slab
    w = (torch.randn(48, 96, 3, 3, generator=g) / 30).cuda()
    ref = F.conv2d(x.double().cpu(), w.double().cpu(), None, 1, 1, 1)
    st = torch.zeros(2, 48, device="cuda", dtype=torch.float64)
    y = conv.conv2d_tc(x, w, 1, 1, 1, stats=st)
    torch.cuda.synchronize()
    assert float((y.cpu().double() - ref).abs().max() / ref.abs().max()) < 2e-5
    assert torch.allclose(st[0].cpu(), ref.sum((0, 2, 3)), rtol=1e-4, atol=1e-3)
    assert torch.allclose(st[1].cpu(), (ref * ref).sum((0, 2, 3)), rtol=1e-4, atol=1e-3)
