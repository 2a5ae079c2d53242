"""GPU parity tests of the ResNet / ResNeXt encoder pieces (reference pytorch/bts.py:282-296 via torchvision.models.resnet):
grouped 3x3 convolution as a block-diagonal tensor-core operator (forward, dgrad, wgrad), the dgrad of stride-2 convolutions
(zero-stuffed source), the stem max-pool and the bottleneck tail relu(bn(x) + identity).
Checker: torch fp64 on the CPU; tolerance 2e-5 of the output scale (fp32-grade, as tests/test_conv_gpu.py)."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


def _cl(t):
    return t.cuda().contiguous(memory_format=torch.channels_last)


def _err(got, ref):
    return float((got.detach().cpu().double() - ref).abs().max() / ref.abs().max().clamp_min(1e-30))


GROUPED = [
    # B, width, cpg, H, W, stride
    (2, 128, 4, 9, 11, 1),       # resnext50 layer1 (32 groups x 4)
    (1, 256, 8, 8, 12, 1),       # resnext101 32x8d layer1, two diagonal blocks
    (2, 256, 8, 10, 14, 2),      # stride-2 grouped 3x3 (first block of layer2..4)
    (1, 512, 16, 5, 7, 1),
    (1, 128, 64, 6, 6, 1),       # wide groups (resnext101 layer4: 64 channels per group)
]


@pytest.mark.parametrize("B,width,cpg,H,W,stride", GROUPED)
def test_grouped_conv_fwd_dgrad_wgrad(B, width, cpg, H, W, stride):
    from bts_b200 import conv
    groups = width // cpg
    g = torch.Generator().manual_seed(width + cpg + stride)
    x = torch.randn(B, width, H, W, generator=g)
    w = torch.randn(width, cpg, 3, 3, generator=g) / (cpg * 9) ** 0.5
    xd = x.double().requires_grad_(True)
    wd = w.double().requires_grad_(True)
    ref = F.conv2d(xd, wd, None, stride, 1, 1, groups)
    gy = torch.randn(ref.shape, generator=g)
    ref.backward(gy.double())
    xc = _cl(x).requires_grad_(True)
    wc = w.cuda().requires_grad_(True)
    y = conv.conv2d(xc, wc, stride, 1, 1, groups)
    assert y.shape == ref.shape
    assert _err(y, ref.detach()) < 2e-5
    y.backward(_cl(gy))
    torch.cuda.synchronize()
    assert _err(xc.grad, xd.grad) < 2e-5
    assert wc.grad.shape == w.shape
    assert _err(wc.grad, wd.grad) < 2e-5


STRIDED = [
    # B, Cin, H, W, Cout, k, pad
    (2, 64, 12, 16, 128, 1, 0),      # resnet downsample 1x1 / 2
    (1, 96, 10, 14, 64, 3, 1),       # 3x3 / 2 (resnet50 conv2 of a stage's first block)
    (1, 32, 9, 13, 48, 3, 1),        # odd input size: (9,13) -> (5,7)
    (1, 256, 8, 8, 512, 1, 0),
]


@pytest.mark.parametrize("B,Cin,H,W,Cout,k,pad", STRIDED)
def test_stride2_conv_all_three_gemms(B, Cin, H, W, Cout, k, pad):
    from bts_b200 import conv
    g = torch.Generator().manual_seed(Cin + Cout + k)
    x = torch.randn(B, Cin, H, W, generator=g)
    w = torch.randn(Cout, Cin, k, k, generator=g) / (Cin * k * k) ** 0.5
    xd = x.double().requires_grad_(True)
    wd = w.double().requires_grad_(True)
    ref = F.conv2d(xd, wd, None, 2, pad)
    gy = torch.randn(ref.shape, generator=g)
    ref.backward(gy.double())
    xc = _cl(x).requires_grad_(True)
    wc = w.cuda().requires_grad_(True)
    y = conv.conv2d(xc, wc, 2, pad, 1)
    assert _err(y, ref.detach()) < 2e-5
    y.backward(_cl(gy))
    torch.cuda.synchronize()
    assert xc.grad.shape == x.shape
    assert _err(xc.grad, xd.grad) < 2e-5
    assert _err(wc.grad, wd.grad) < 2e-5


@pytest.mark.parametrize("B,C,H,W", [(2, 64, 12, 16), (1, 96, 11, 13), (1, 6, 7, 9)])
def test_maxpool3s2_fwd_bwd(B, C, H, W):
    from bts_b200 import glue
    g = torch.Generator().manual_seed(C + H)
    x = torch.randn(B, C, H, W, generator=g)
    x[0, 0, :3, :3] = 1.5                                     # ties: the first maximum in scan order takes the gradient
    xd = x.double().requires_grad_(True)
    ref = F.max_pool2d(xd, 3, 2, 1)
    gy = torch.randn(ref.shape, generator=g)
    ref.backward(gy.double())
    xc = _cl(x).requires_grad_(True)
    y = glue.maxpool3s2(xc)
    assert torch.equal(y.detach().cpu(), ref.detach().float())          # selection: bit-exact
    y.backward(_cl(gy))
    torch.cuda.synchronize()
    assert torch.allclose(xc.grad.cpu().double(), xd.grad, rtol=0, atol=1e-6)


@pytest.mark.parametrize("train", [True, False])
def test_bn_add_relu_tail(train):
    from bts_b200 import glue
    g = torch.Generator().manual_seed(11)
    B, C, H, W = 2, 64, 9, 10
    x = torch.randn(B, C, H, W, generator=g) * 2 + 0.3
    res = torch.randn(B, C, H, W, generator=g)
    bn_ref = torch.nn.BatchNorm2d(C).double()
    bn = torch.nn.BatchNorm2d(C)
    with torch.no_grad():
        bn_ref.weight.copy_(torch.rand(C, generator=g) + 0.5)
        bn_ref.bias.copy_(torch.randn(C, generator=g) * 0.2)
        bn_ref.running_mean.copy_(torch.randn(C, generator=g) * 0.1)
        bn_ref.running_var.copy_(torch.rand(C, generator=g) + 0.5)
    bn.load_state_dict({k: (v.float() if v.is_floating_point() else v) for k, v in bn_ref.state_dict().items()})
    bn.cuda()
    bn_ref.train(train)
    bn.train(train)
    xd, rd = x.double().requires_grad_(True), res.double().requires_grad_(True)
    ref = F.relu(bn_ref(xd) + rd)
    gy = torch.randn(ref.shape, generator=g)
    ref.backward(gy.double())
    xc, rc = _cl(x).requires_grad_(True), _cl(res).requires_grad_(True)
    y = glue.bn_add_relu(xc, rc, bn)
    assert _err(y, ref.detach()) < 1e-5
    y.backward(_cl(gy))
    torch.cuda.synchronize()
    assert _err(xc.grad, xd.grad) < 2e-5
    assert _err(rc.grad, rd.grad) < 1e-6
    assert _err(bn.weight.grad, bn_ref.weight.grad) < 2e-5
    assert _err(bn.bias.grad, bn_ref.bias.grad) < 2e-5
    if train:
        assert torch.allclose(bn.running_var.cpu().double(), bn_ref.running_var, rtol=1e-5)
        assert int(bn.num_batches_tracked) == int(bn_ref.num_batches_tracked)
