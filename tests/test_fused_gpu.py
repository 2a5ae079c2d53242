"""GPU parity of the fused, concat-free DenseNet block (bts_b200/fused.py) against torchvision's own _DenseBlock
(the reference's encoder arithmetic) in fp64 on the CPU: outputs, input gradient, every parameter gradient and the
BatchNorm running statistics."""
import copy

import pytest
import torch

pytestmark = pytest.mark.gpu


def _block(C0, L, growth=48, bn_size=4):
    from torchvision.models.densenet import _DenseBlock
    torch.manual_seed(0)
    blk = _DenseBlock(L, C0, bn_size, growth, 0.0)
    g = torch.Generator().manual_seed(1)
    with torch.no_grad():
        for m in blk.modules():
            if isinstance(m, torch.nn.BatchNorm2d):
                m.weight.copy_(torch.rand(m.weight.shape, generator=g) + 0.5)
                m.bias.copy_(torch.randn(m.bias.shape, generator=g) * 0.2)
    return blk


@pytest.fixture(params=["onepass", "reduce_apply", "epilogue"],
                ids=["bn_one_pass_deferred_affine", "bn_reduce_then_apply", "bn_sums_in_dgrad_epilogue"])
def epi_bnbwd(request):
    """the three forms of the dense-layer BatchNorm backward: one streaming pass with the per-channel affine remainder
    deferred (default, bts_bn_relu_bwd_fused + bts_bn_bwd_correct), reduce pass + apply pass, and the sums reduced in the
    dgrad epilogue (bts_conv_fwd with x_bn / bn_st)"""
    from bts_b200 import fused
    prev = fused.EPI_BNBWD, fused.BN_ONEPASS
    fused.EPI_BNBWD = request.param == "epilogue"
    fused.BN_ONEPASS = request.param == "onepass"
    yield request.param
    fused.EPI_BNBWD, fused.BN_ONEPASS = prev


@pytest.mark.parametrize("mode", ["train", "eval"])
@pytest.mark.parametrize("C0,L,H,W", [(96, 3, 12, 20), (64, 2, 9, 7), (208, 2, 6, 10)])
def test_dense_block_matches_torchvision(epi_bnbwd, mode, C0, L, H, W):
    from bts_b200 import model as M
    ref = _block(C0, L).double()
    ours = copy.deepcopy(ref).float()
    M.adopt_convs(ours)
    assert type(ours).__name__ == "DenseBlockTC"
    ours.cuda()
    getattr(ref, mode)()
    getattr(ours, mode)()
    g = torch.Generator().manual_seed(2)
    x = torch.randn(2, C0, H, W, generator=g)
    gy = torch.randn(2, C0 + 48 * L, H, W, generator=g)
    xr = x.double().requires_grad_(True)
    yr = ref(xr)
    yr.backward(gy.double())
    xo = x.cuda().contiguous(memory_format=torch.channels_last).requires_grad_(True)
    yo = ours(xo)
    yo.backward(gy.cuda())
    scale = yr.abs().max()
    assert (yo.detach().cpu().double() - yr.detach()).abs().max() / scale < 2e-5
    assert (xo.grad.cpu().double() - xr.grad).abs().max() / xr.grad.abs().max() < 2e-4
    pr = dict(ref.named_parameters())
    for k, p in ours.named_parameters():
        a, b = p.grad.cpu().double(), pr[k].grad
        assert (a - b).abs().max() / b.abs().max().clamp_min(1e-12) < 5e-4, k
    br = dict(ref.named_buffers())
    for k, b in ours.named_buffers():
        if b.dtype.is_floating_point:
            assert (b.cpu().double() - br[k]).abs().max() < 1e-5, k
        else:
            assert int(b) == int(br[k]), k
