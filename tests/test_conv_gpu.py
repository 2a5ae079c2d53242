"""GPU parity tests of the wgmma implicit-GEMM conv engine through the C-ABI.
Checker: torch fp64 conv2d on the CPU (the engine is a floating-point kernel; tolerance stated per test:
3xTF32 parity mode must match fp32-grade, <= 2e-5 of the output scale; the reference's own fp32 noise is ~1e-6)."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


def ref_conv(x, w, stride, pad, dil, scale=None, shift=None, relu=False, up=False, act=None):
    x = x.double()
    if scale is not None:
        x = x * scale.double().view(1, -1, 1, 1) + shift.double().view(1, -1, 1, 1)
    if relu:
        x = F.relu(x)
    if up:
        x = F.interpolate(x, scale_factor=2, mode="nearest")
    y = F.conv2d(x, w.double(), None, stride, pad, dil)
    if act == "elu":
        y = F.elu(y)
    elif act == "sigmoid":
        y = torch.sigmoid(y)
    return y


CASES = [
    # B, Cin, H, W, Cout, k, stride, pad, dil
    (2, 64, 12, 20, 48, 1, 1, 0, 1),        # dense-layer 1x1, M tail (480 px), N=48
    (1, 32, 16, 16, 16, 3, 1, 1, 1),        # 3x3, exact 2 tiles
    (2, 192, 9, 11, 48, 3, 1, 1, 1),        # dense-layer 3x3
    (1, 256, 11, 22, 128, 3, 1, 3, 3),      # atrous d=3
    (1, 64, 11, 22, 32, 3, 1, 12, 12),      # atrous d=12 (> map height on one axis)
    (1, 256, 6, 8, 256, 1, 1, 0, 1),        # two N tiles
    (1, 36, 10, 12, 32, 3, 1, 1, 1),        # Cin tail (36 = 32 + 4)
    (1, 225, 6, 7, 128, 3, 1, 1, 1),        # odd Cin -> scalar loads (pixel stride not a multiple of 4)
    (1, 8, 9, 9, 3, 1, 1, 0, 1),            # Cout = 3 (plane_params)
    (2, 32, 8, 8, 1, 3, 1, 1, 1),           # Cout = 1 (get_depth)
    (1, 2208, 3, 5, 64, 3, 1, 1, 1),        # long K (upconv5-like)
    (1, 3, 20, 24, 96, 7, 2, 3, 1),         # stem conv0 7x7 / 2
]


@pytest.mark.parametrize("B,Cin,H,W,Cout,k,stride,pad,dil", CASES)
def test_conv_parity_3xtf32(B, Cin, H, W, Cout, k, stride, pad, dil):
    from bts_b200 import conv
    g = torch.Generator().manual_seed(Cin * 7 + Cout)
    x = torch.randn(B, Cin, H, W, generator=g)
    w = torch.randn(Cout, Cin, k, k, generator=g) / (Cin * k * k) ** 0.5
    ref = ref_conv(x, w, stride, pad, dil)
    y = conv.conv2d_tc(x.cuda().contiguous(memory_format=torch.channels_last), w.cuda(), stride, pad, dil)
    torch.cuda.synchronize()
    assert y.shape == ref.shape
    err = (y.cpu().double() - ref).abs().max() / ref.abs().max()
    # fp32-grade: 2e-5 of the output scale; the tensor core's fp32 accumulator truncates (rounds toward zero) on
    # every accumulation step, a systematic ~2^-26 relative shrink per K=8 step that shows for very long reductions
    # (K = 9*2208 = 19872 -> 1.2e-4, measured) -- still two orders below single-pass TF32 (~3e-3).
    K = Cin * k * k
    tol = max(2e-5, 8e-9 * K)
    assert err < tol, "rel-to-scale error %.3g (tol %.3g)" % (err, tol)


def test_conv_fused_pre_affine_relu_upsample_elu():
    """upconv (bts.py:76-80) with a folded BN+ReLU on its input: nearest x2 folded into the address map."""
    from bts_b200 import conv
    g = torch.Generator().manual_seed(3)
    x = torch.randn(2, 64, 7, 9, generator=g)
    w = torch.randn(32, 64, 3, 3, generator=g) / 24
    sc, sh = torch.rand(64, generator=g) + 0.5, torch.randn(64, generator=g) * 0.3
    ref = ref_conv(x, w, 1, 1, 1, sc, sh, True, True, "elu")
    y = conv.conv2d_tc(x.cuda().contiguous(memory_format=torch.channels_last), w.cuda(), 1, 1, 1, sc.cuda(), sh.cuda(),
                       True, True, "elu")
    err = (y.cpu().double() - ref).abs().max() / ref.abs().max()
    assert err < 2e-5


def test_conv_writes_into_channel_slice_and_reads_from_slice():
    """concat-free dataflow: read a channel slice of a slab, write into a slice of another slab."""
    from bts_b200 import conv
    g = torch.Generator().manual_seed(4)
    slab = torch.randn(1, 96, 8, 8, generator=g).cuda().contiguous(memory_format=torch.channels_last)
    w = torch.randn(48, 64, 1, 1, generator=g).cuda() / 8
    out = torch.zeros(1, 128, 8, 8, device="cuda").contiguous(memory_format=torch.channels_last)
    conv.conv2d_tc(slab[:, :64], w, out=out[:, 64:112])
    ref = ref_conv(slab[:, :64].cpu(), w.cpu(), 1, 0, 1)
    assert (out[:, 64:112].cpu().double() - ref).abs().max() / ref.abs().max() < 2e-5
    assert float(out[:, :64].abs().sum()) == 0 and float(out[:, 112:].abs().sum()) == 0


def test_conv_fast_mode_is_labelled_and_less_exact():
    from bts_b200 import conv
    g = torch.Generator().manual_seed(5)
    x = torch.randn(1, 128, 16, 16, generator=g)
    w = torch.randn(64, 128, 3, 3, generator=g) / 34
    ref = ref_conv(x, w, 1, 1, 1)
    xc = x.cuda().contiguous(memory_format=torch.channels_last)
    e3 = (conv.conv2d_tc(xc, w.cuda(), 1, 1, 1).cpu().double() - ref).abs().max() / ref.abs().max()
    e1 = (conv.conv2d_tc(xc, w.cuda(), 1, 1, 1, precision=1).cpu().double() - ref).abs().max() / ref.abs().max()
    assert e3 < 2e-5 and 1e-5 < e1 < 5e-3


@pytest.mark.parametrize("k,pad,dil", [(1, 0, 1), (3, 1, 1), (3, 6, 6)])
def test_conv_autograd_dgrad_on_engine(k, pad, dil):
    from bts_b200 import conv
    g = torch.Generator().manual_seed(k + dil)
    x = torch.randn(2, 64, 10, 12, generator=g)
    w = torch.randn(48, 64, k, k, generator=g) / (64 * k * k) ** 0.5
    gy = torch.randn(2, 48, 10, 12, generator=g)
    xd, wd = x.double().requires_grad_(True), w.double().requires_grad_(True)
    F.conv2d(xd, wd, None, 1, pad, dil).backward(gy.double())
    xc = x.cuda().contiguous(memory_format=torch.channels_last).requires_grad_(True)
    wc = w.cuda().requires_grad_(True)
    conv.conv2d(xc, wc, 1, pad, dil).backward(gy.cuda())
    assert (xc.grad.cpu().double() - xd.grad).abs().max() / xd.grad.abs().max() < 2e-5
    assert (wc.grad.cpu().double() - wd.grad).abs().max() / wd.grad.abs().max() < 1e-4


@pytest.mark.parametrize("C,K,sig", [(32, 3, True), (8, 1, True), (32, 3, False), (64, 3, False), (16, 1, False)])
def test_single_output_channel_head_kernels(C, K, sig):
    """get_depth (3x3 32->1 + sigmoid) / reduc1x1.final (1x1 8->1 + sigmoid): CUDA-core streaming kernels, fp32 FMA --
    fwd, dgrad and wgrad vs torch fp64."""
    from bts_b200 import conv
    g = torch.Generator().manual_seed(C + K)
    x = torch.randn(2, C, 13, 17, generator=g)
    w = torch.randn(1, C, K, K, generator=g) / (C * K * K) ** 0.5
    gy = torch.randn(2, 1, 13, 17, generator=g)
    xd, wd = x.double().requires_grad_(True), w.double().requires_grad_(True)
    yd = F.conv2d(xd, wd, None, 1, K // 2)
    if sig:
        yd = torch.sigmoid(yd)
    yd.backward(gy.double())
    xc = x.cuda().contiguous(memory_format=torch.channels_last).requires_grad_(True)
    wc = w.cuda().requires_grad_(True)
    y = conv.conv_c1(xc, wc, sigmoid=sig)
    y.backward(gy.cuda())
    assert (y.detach().cpu().double() - yd.detach()).abs().max() < 1e-5
    assert (xc.grad.cpu().double() - xd.grad).abs().max() / xd.grad.abs().max() < 1e-5
    assert (wc.grad.cpu().double() - wd.grad).abs().max() / wd.grad.abs().max() < 1e-5


@pytest.fixture(params=["tma_ring", "global_loads", "auto_small_map"])
def w2_mode(request):
    """routes small test shapes to the shifted-dY kernel (its production threshold is 12k pixels) with the operands staged
    through the TMA landing ring or loaded by the producers; 'auto_small_map' leaves the production routing (wgrad_tc)"""
    from bts_b200 import _lib
    L = _lib.lib()
    if request.param != "auto_small_map":
        L.bts_wgrad2_set_min_pixels(0)
        L.bts_wgrad2_set_tma(1 if request.param == "tma_ring" else 0)
    yield request.param
    L.bts_wgrad2_set_min_pixels(-1)
    L.bts_wgrad2_set_tma(1)


@pytest.mark.parametrize("Cin,Cout,H,W,dil,up,pre", [(192, 48, 9, 11, 1, False, True), (36, 32, 10, 13, 1, False, False),
                                                     (64, 32, 6, 7, 1, True, False), (161, 64, 8, 9, 1, False, False),
                                                     (40, 24, 7, 5, 3, False, True), (192, 48, 16, 32, 1, False, True),
                                                     (64, 32, 5, 8, 1, True, True), (128, 64, 12, 16, 1, True, False),
                                                     (36, 32, 33, 47, 1, False, False)])
def test_wgrad_narrow_output_shifted_dy_kernel(w2_mode, Cin, Cout, H, W, dil, up, pre):
    """Cout <= 64, 3x3: the all-taps-in-one-CTA wgrad (wgrad2_tc.cu) incl. fused BN+ReLU prologue, nearest-x2
    up-sampling, dilation, odd channel counts (scalar-load path), k-blocks that straddle image rows and images -- vs torch
    fp64 autograd."""
    from bts_b200 import conv
    g = torch.Generator().manual_seed(Cin + Cout)
    x = torch.randn(2, Cin, H, W, generator=g)
    w = torch.randn(Cout, Cin, 3, 3, generator=g) / (Cin * 9) ** 0.5
    sc = torch.rand(Cin, generator=g) + 0.5
    sh = torch.randn(Cin, generator=g) * 0.3
    Ho, Wo = (2 * H, 2 * W) if up else (H, W)
    gy = torch.randn(2, Cout, Ho, Wo, generator=g)
    xd = x.double()
    if pre:
        xd = F.relu(xd * sc.double().view(1, -1, 1, 1) + sh.double().view(1, -1, 1, 1))
    if up:
        xd = F.interpolate(xd, scale_factor=2, mode="nearest")
    wd = w.double().requires_grad_(True)
    F.conv2d(xd, wd, None, 1, dil, dil).backward(gy.double())
    xc = x.cuda().contiguous(memory_format=torch.channels_last)
    gw = conv.wgrad_tc(xc, gy.cuda().contiguous(memory_format=torch.channels_last), w.shape, w.stride(), 1, dil, dil,
                       pre_scale=sc.cuda() if pre else None, pre_shift=sh.cuda() if pre else None, pre_relu=pre,
                       upsample2=up)
    err = (gw.cpu().double() - wd.grad).abs().max() / wd.grad.abs().max()
    assert err < 2e-5, err


@pytest.mark.parametrize("Cin,Cout,H,W,pre", [(240, 192, 9, 14, True), (96, 128, 16, 16, False), (300, 192, 7, 9, True),
                                               (64, 256, 8, 8, False), (130, 80, 5, 7, True), (2064, 192, 6, 11, True)])
def test_wgrad_pointwise_wide_tile_on_shifted_dy_kernel(w2_mode, Cin, Cout, H, W, pre):
    """1x1 layers with 64 < Cout <= 256 (dense-layer conv1, transitions, decoder reductions): one <= 256-wide output tile per
    CTA on wgrad2_tc.cu (single-tap unit mapping), TMA ring / global loads / production routing -- vs torch fp64."""
    from bts_b200 import conv
    g = torch.Generator().manual_seed(Cin * 7 + Cout)
    x = torch.randn(3, Cin, H, W, generator=g)
    gy = torch.randn(3, Cout, H, W, generator=g)
    sc = torch.rand(Cin, generator=g) + 0.5
    sh = torch.randn(Cin, generator=g) * 0.3
    xd = x.double()
    if pre:
        xd = F.relu(xd * sc.double().view(1, -1, 1, 1) + sh.double().view(1, -1, 1, 1))
    ref = torch.einsum("bohw,bihw->oi", gy.double(), xd).reshape(Cout, Cin, 1, 1)
    xc = x.cuda().contiguous(memory_format=torch.channels_last)
    gw = conv.wgrad_tc(xc, gy.cuda().contiguous(memory_format=torch.channels_last), (Cout, Cin, 1, 1), (Cin, 1, 1, 1), 1, 0, 1,
                       pre_scale=sc.cuda() if pre else None, pre_shift=sh.cuda() if pre else None, pre_relu=pre)
    err = (gw.cpu().double() - ref).abs().max() / ref.abs().max()
    assert err < 2e-5, err


@pytest.mark.parametrize("Cin,Cout,act", [(32, 16, "elu"), (16, 8, "elu"), (8, 3, None), (64, 32, "elu"), (64, 12, None),
                                           (8, 1, "sigmoid"), (16, 64, None), (32, 64, "elu")])
def test_pointwise_forward_and_dgrad_cuda_core_kernel(Cin, Cout, act, monkeypatch):
    """narrow 1x1 layers of the reduction heads: forward (+ELU / sigmoid) and dgrad on the HBM-bound CUDA-core kernel
    (bts_conv_pw_fwd) vs fp64, NHWC tensors, channel slices of wider slabs as input and output"""
    from bts_b200 import conv
    monkeypatch.setattr(conv, "PW_MIN_PIXELS", 0)
    g = torch.Generator().manual_seed(31 + Cin + Cout)
    slab = torch.randn(3, Cin + 8, 17, 23, generator=g).cuda().contiguous(memory_format=torch.channels_last)
    x = slab[:, 4:4 + Cin]
    w = (torch.randn(Cout, Cin, 1, 1, generator=g) / Cin ** 0.5).cuda()
    before = len(conv.trace_log) if conv.TRACE else None
    y = conv.conv2d_tc(x, w, 1, 0, 1, act=act)
    ref = F.conv2d(x.double().cpu(), w.double().cpu())
    if act == "elu":
        ref = F.elu(ref)
    elif act == "sigmoid":
        ref = torch.sigmoid(ref)
    assert y.shape == ref.shape and y.is_contiguous(memory_format=torch.channels_last)
    assert (y.cpu().double() - ref).abs().max() / ref.abs().max() < 1e-5
    # into a channel slice of a wider output slab
    oslab = torch.zeros(3, Cout + 4, 17, 23).cuda().contiguous(memory_format=torch.channels_last)
    conv.conv2d_tc(x, w, 1, 0, 1, act=act, out=oslab[:, :Cout])
    assert torch.equal(oslab[:, :Cout], y) and float(oslab[:, Cout:].abs().sum()) == 0.0
    # dgrad = the transposed operator
    gy = torch.randn(3, Cout, 17, 23, generator=g).cuda().contiguous(memory_format=torch.channels_last)
    gx = conv.conv2d_tc(gy, w, 1, 0, 1, transpose_flip=True)
    gref = F.conv_transpose2d(gy.double().cpu(), w.double().cpu())
    assert gx.shape == gref.shape
    assert (gx.cpu().double() - gref).abs().max() / gref.abs().max() < 1e-5
    assert before is None or len(conv.trace_log) > before


@pytest.mark.parametrize("Cin,Cout", [(32, 16), (16, 8), (8, 3), (64, 32), (64, 12), (8, 1)])
def test_pointwise_wgrad_cuda_core_kernel(Cin, Cout, monkeypatch):
    """narrow 1x1 layers of the reduction heads: dW on the HBM-bound CUDA-core kernel (csrc/pointwise.cu) vs fp64"""
    from bts_b200 import _lib, conv
    monkeypatch.setattr(conv, "PW_MIN_PIXELS", 0)
    assert _lib.lib().bts_conv_pw_wgrad_eligible(Cin, Cout)
    g = torch.Generator().manual_seed(11)
    x = torch.randn(3, Cin, 17, 23, generator=g)
    gy = torch.randn(3, Cout, 17, 23, generator=g)
    ref = torch.einsum("bohw,bihw->oi", gy.double(), x.double()).reshape(Cout, Cin, 1, 1)
    xc = x.cuda().contiguous(memory_format=torch.channels_last)
    for gyc in (gy.cuda().contiguous(memory_format=torch.channels_last), gy.cuda()):      # NHWC and NCHW upstream grads
        before = len(conv.trace_log)
        gw = conv.wgrad_tc(xc, gyc, (Cout, Cin, 1, 1), (Cin, 1, 1, 1), 1, 0, 1)
        err = (gw.cpu().double() - ref).abs().max() / ref.abs().max()
        assert err < 1e-5, float(err)
    # a channel slice of a wider slab as the activation operand
    slab = torch.randn(3, Cin + 8, 17, 23, generator=g).cuda().contiguous(memory_format=torch.channels_last)
    gw = conv.wgrad_tc(slab[:, 4:4 + Cin], gy.cuda(), (Cout, Cin, 1, 1), (Cin, 1, 1, 1), 1, 0, 1)
    ref2 = torch.einsum("bohw,bihw->oi", gy.double(), slab[:, 4:4 + Cin].cpu().double()).reshape(Cout, Cin, 1, 1)
    assert (gw.cpu().double() - ref2).abs().max() / ref2.abs().max() < 1e-5


@pytest.mark.parametrize("Cin,Cout,k,H,W,act", [(40, 48, 3, 13, 21, None), (96, 192, 1, 9, 14, None), (36, 32, 3, 20, 28, None),
                                                 (64, 256, 1, 8, 8, None)])
def test_conv_epilogue_batch_statistics(Cin, Cout, k, H, W, act):
    """per-channel sum / sum of squares of the conv output reduced in the epilogue (bts_conv_fwd with stat_sum /
    stat_sumsq) == a separate pass"""
    from bts_b200 import conv
    g = torch.Generator().manual_seed(21)
    x = torch.randn(3, Cin, H, W, generator=g).cuda().contiguous(memory_format=torch.channels_last)
    w = (torch.randn(Cout, Cin, k, k, generator=g) / (Cin * k * k) ** 0.5).cuda()
    st = torch.zeros((2, Cout), device="cuda", dtype=torch.float64)
    y = conv.conv2d_tc(x, w, 1, k // 2, 1, act=act, stats=st)
    y0 = conv.conv2d_tc(x, w, 1, k // 2, 1, act=act)
    assert torch.equal(y, y0)
    yd = y.double()
    s1, s2 = yd.sum((0, 2, 3)), (yd * yd).sum((0, 2, 3))
    assert (st[0] - s1).abs().max() <= 1e-5 * s2.sqrt().max()
    assert ((st[1] - s2).abs() / s2).max() < 1e-5
