"""GPU tests of the native MobileNetV2 path: the depthwise 3x3 kernels (csrc/dwconv.cu), the fused InvertedResidual Function
and the whole mobilenetv2_bts model.  The checker is torch fp64 on the CPU; the kernel and block bar is 2e-5 of the output
scale, as in test_resnet_gpu.py and test_wgrad_engines_gpu.py."""
import glob
import os
import re
import types

import pytest
import torch
import torch.nn.functional as F

import bts_oracle as O
from conftest import ROOT
from test_model_gpu import check_outputs

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
TOL = 2e-5


def close(got, want, what, tol=TOL):
    got = got.detach().double().cpu()
    want = want.detach().double()
    scale = float(want.abs().max()) or 1.0
    err = float((got - want).abs().max())
    assert err <= tol * scale, "%s: max abs err %.3g > %.1g x scale %.3g" % (what, err, tol, scale)


def nhwc(t):
    return t.float().to(DEV).contiguous(memory_format=torch.channels_last)


def bn_pre(C, g):
    """scale / shift that send a visible fraction of x*scale + shift (x ~ N(0,1)) below 0 and above 6"""
    return torch.rand(C, generator=g, dtype=torch.float64) * 3 + 1.5, torch.rand(C, generator=g, dtype=torch.float64) * 4 - 1


# ---------------------------------------------------------------------------------------------- kernel parity
@pytest.mark.parametrize("C,B", [(32, 1), (96, 2), (144, 1), (384, 2), (960, 1)])
@pytest.mark.parametrize("stride", [1, 2])
@pytest.mark.parametrize("pre", [False, True])
def test_depthwise_kernels_vs_fp64(C, B, stride, pre):
    from bts_b200 import dwconv
    g = torch.Generator().manual_seed(C * 10 + stride + 3 * pre)
    H, W = 9, 13
    x = torch.randn(B, C, H, W, generator=g, dtype=torch.float64)
    w = torch.randn(C, 1, 3, 3, generator=g, dtype=torch.float64) / 3
    sc, sh = bn_pre(C, g)
    a = (x * sc.view(1, -1, 1, 1) + sh.view(1, -1, 1, 1)).clamp(0, 6) if pre else x
    if pre:
        assert float((a == 0).double().mean()) > 0.05 and float((a == 6).double().mean()) > 0.05
    xr = x.clone().requires_grad_(True)
    wr = w.clone().requires_grad_(True)
    ar = (xr * sc.view(1, -1, 1, 1) + sh.view(1, -1, 1, 1)).clamp(0, 6) if pre else xr
    yr = F.conv2d(ar, wr, stride=stride, padding=1, groups=C)
    gy = torch.randn(yr.shape, generator=g, dtype=torch.float64)
    yr.backward(gy)
    prep = (sc.float().to(DEV), sh.float().to(DEV)) if pre else None
    wd = w.float().to(DEV)
    y, sums = dwconv.fwd(nhwc(x), wd, stride, pre=prep, stats=True)
    close(y, yr, "fwd")
    yd = yr.detach()
    s_ref = yd.sum(dim=(0, 2, 3))
    q_ref = (yd * yd).sum(dim=(0, 2, 3))
    close(sums[0], s_ref, "sum", tol=1e-5 * float(yd.abs().sum(dim=(0, 2, 3)).max()) / float(s_ref.abs().max()))
    close(sums[1], q_ref, "sum of squares")
    # dgrad of the conv alone (the prologue's backward is the BatchNorm kernels' job), wgrad with the prologue
    dx = dwconv.dgrad(nhwc(gy), wd, stride, H, W)
    at = a.clone().requires_grad_(True)
    F.conv2d(at, w, stride=stride, padding=1, groups=C).backward(gy)
    close(dx, at.grad, "dgrad")
    dw = dwconv.wgrad(nhwc(x), nhwc(gy), wd, stride, pre=prep)
    close(dw, wr.grad, "wgrad")
    # eval epilogue: relu6(y*s2 + h2)
    s2, h2 = bn_pre(C, g)
    ye = dwconv.fwd(nhwc(x), wd, stride, pre=prep, post=(s2.float().to(DEV), h2.float().to(DEV)))
    close(ye, (yd * s2.view(1, -1, 1, 1) + h2.view(1, -1, 1, 1)).clamp(0, 6), "eval epilogue")


def test_depthwise_kernels_read_channel_slices():
    from bts_b200 import dwconv
    g = torch.Generator().manual_seed(7)
    C, B, H, W = 96, 2, 11, 9
    slab = torch.randn(B, C + 8, H, W, generator=g, dtype=torch.float64)
    x = slab[:, 4:4 + C]
    w = torch.randn(C, 1, 3, 3, generator=g, dtype=torch.float64)
    sc, sh = bn_pre(C, g)
    for stride in (1, 2):
        a = (x * sc.view(1, -1, 1, 1) + sh.view(1, -1, 1, 1)).clamp(0, 6)
        yr = F.conv2d(a, w, stride=stride, padding=1, groups=C)
        gy_slab = torch.randn(B, C + 4, yr.shape[2], yr.shape[3], generator=g, dtype=torch.float64)
        gy = gy_slab[:, 4:]
        xs = nhwc(slab)[:, 4:4 + C]                   # pixel stride C + 8, 16-byte aligned channel offset
        gys = nhwc(gy_slab)[:, 4:]
        assert xs.stride(3) == C + 8
        prep = (sc.float().to(DEV), sh.float().to(DEV))
        close(dwconv.fwd(xs, w.float().to(DEV), stride, pre=prep), yr, "fwd slice s%d" % stride)
        ar = a.clone().requires_grad_(True)
        wr = w.clone().requires_grad_(True)
        F.conv2d(ar, wr, stride=stride, padding=1, groups=C).backward(gy)
        close(dwconv.dgrad(gys, w.float().to(DEV), stride, H, W), ar.grad, "dgrad slice s%d" % stride)
        close(dwconv.wgrad(xs, gys, w.float().to(DEV), stride, pre=prep), wr.grad, "wgrad slice s%d" % stride)


def test_depthwise_statistics_are_bit_reproducible():
    from bts_b200 import dwconv
    g = torch.Generator().manual_seed(3)
    x = nhwc(torch.randn(2, 144, 56, 88, generator=g))
    w = torch.randn(144, 1, 3, 3, generator=g).to(DEV)
    gy = nhwc(torch.randn(2, 144, 56, 88, generator=g))
    a = [dwconv.fwd(x, w, 1, stats=True) for _ in range(2)]
    assert torch.equal(a[0][0], a[1][0]) and torch.equal(a[0][1], a[1][1])
    assert torch.equal(dwconv.wgrad(x, gy, w, 1), dwconv.wgrad(x, gy, w, 1))


@pytest.mark.parametrize("C,B,H,W,stride", [(32, 8, 176, 352, 1), (96, 8, 176, 352, 2)])
def test_depthwise_kernels_walk_several_tiles_per_cta(C, B, H, W, stride):
    """batch-16-sized maps: each CTA walks several tiles (the staged-window barrier, fp32 runs over up to 32 tiles, the
    multi-tile wgrad accumulation), which the small shapes above never reach"""
    from bts_b200 import _lib, dwconv
    TH, TW = (8, 16) if stride == 1 else (4, 16)
    Ho, Wo = (H - 1) // stride + 1, (W - 1) // stride + 1
    ntiles = B * -(-Ho // TH) * -(-Wo // TW)
    slices = _lib.lib().bts_dw3x3_fwd_workspace_floats(B, H, W, C, stride) // (4 * C)
    assert 0 < slices and 2 * slices < ntiles, (slices, ntiles)
    g = torch.Generator().manual_seed(11 + stride)
    x = torch.randn(B, C, H, W, generator=g, dtype=torch.float64)
    w = torch.randn(C, 1, 3, 3, generator=g, dtype=torch.float64) / 3
    sc, sh = bn_pre(C, g)
    xr = x.clone().requires_grad_(True)
    wr = w.clone().requires_grad_(True)
    ar = (xr * sc.view(1, -1, 1, 1) + sh.view(1, -1, 1, 1)).clamp(0, 6)
    yr = F.conv2d(ar, wr, stride=stride, padding=1, groups=C)
    gy = torch.randn(yr.shape, generator=g, dtype=torch.float64)
    yr.backward(gy)
    prep = (sc.float().to(DEV), sh.float().to(DEV))
    wd = w.float().to(DEV)
    y, sums = dwconv.fwd(nhwc(x), wd, stride, pre=prep, stats=True)
    yd = yr.detach()
    close(y, yd, "fwd")
    s_ref = yd.sum(dim=(0, 2, 3))
    close(sums[0], s_ref, "sum", tol=1e-5 * float(yd.abs().sum(dim=(0, 2, 3)).max()) / float(s_ref.abs().max()))
    close(sums[1], (yd * yd).sum(dim=(0, 2, 3)), "sum of squares")
    close(dwconv.wgrad(nhwc(x), nhwc(gy), wd, stride, pre=prep), wr.grad, "wgrad")
    at = ar.detach().clone().requires_grad_(True)
    F.conv2d(at, w, stride=stride, padding=1, groups=C).backward(gy)
    close(dwconv.dgrad(nhwc(gy), wd, stride, H, W), at.grad, "dgrad")


# ---------------------------------------------------------------------------------------------- block parity
def _randomise_bns(m, g):
    for bn in m.modules():
        if isinstance(bn, torch.nn.BatchNorm2d):
            C = bn.num_features
            dt = bn.weight.dtype
            bn.weight.data = torch.rand(C, generator=g, dtype=dt) + 0.5
            bn.bias.data = torch.rand(C, generator=g, dtype=dt) - 0.5
            bn.running_mean.data = torch.randn(C, generator=g, dtype=dt) * 0.2
            bn.running_var.data = torch.rand(C, generator=g, dtype=dt) + 0.5


@pytest.mark.parametrize("inp,oup,stride,t", [(24, 24, 1, 6), (24, 32, 2, 6), (32, 16, 1, 1)],
                         ids=["residual", "stride2", "expand1"])
@pytest.mark.parametrize("mode", ["train", "eval"])
def test_inverted_residual_block_vs_torchvision_fp64(inp, oup, stride, t, mode):
    from torchvision.models.mobilenetv2 import InvertedResidual
    from bts_b200 import model as M
    g = torch.Generator().manual_seed(inp + oup + stride + t)
    torch.manual_seed(0)
    ref = InvertedResidual(inp, oup, stride, t).double()
    _randomise_bns(ref, g)
    ours = torch.nn.Sequential(InvertedResidual(inp, oup, stride, t))
    ours[0].load_state_dict(ref.state_dict())
    M.adopt_convs(ours)
    assert type(ours[0]).__name__ == "InvertedResidualTC"
    ours.to(DEV)
    getattr(ref, mode)()
    getattr(ours, mode)()
    B, H, W = 2, 15, 21
    x = torch.randn(B, inp, H, W, generator=g, dtype=torch.float64)
    xr = x.clone().requires_grad_(True)
    yr = ref(xr)
    gy = torch.randn(yr.shape, generator=g, dtype=torch.float64)
    yr.backward(gy)
    xo = nhwc(x).requires_grad_(True)
    y = ours(xo)
    close(y, yr, "output")
    y.backward(nhwc(gy))
    close(xo.grad, xr.grad, "input gradient")
    po = dict(ours[0].named_parameters())
    for k, p in ref.named_parameters():
        close(po[k].grad, p.grad, "grad " + k)
    bo = dict(ours[0].named_buffers())
    for k, b in ref.named_buffers():
        if b.is_floating_point():
            close(bo[k], b, "buffer " + k, tol=1e-5)
        else:
            assert int(bo[k]) == int(b), k


@pytest.mark.parametrize("inp,oup,stride,t", [(24, 24, 1, 6), (24, 32, 2, 6), (32, 16, 1, 1)],
                         ids=["residual", "stride2", "expand1"])
def test_inverted_residual_eval_under_no_grad_fuses_bn2(inp, oup, stride, t, monkeypatch):
    """the bts_test.py path: eval mode under no_grad with parameters that still require grad.  relu6(bn2(.)) must come
    out of the depthwise conv's epilogue (no y2, no separate BN-apply pass) and match torchvision in fp64"""
    from torchvision.models.mobilenetv2 import InvertedResidual
    from bts_b200 import dwconv, model as M
    g = torch.Generator().manual_seed(100 + inp + oup + stride + t)
    torch.manual_seed(0)
    ref = InvertedResidual(inp, oup, stride, t).double()
    _randomise_bns(ref, g)
    ours = torch.nn.Sequential(InvertedResidual(inp, oup, stride, t))
    ours[0].load_state_dict(ref.state_dict())
    M.adopt_convs(ours)
    ours.to(DEV).eval()
    ref.eval()
    assert all(p.requires_grad for p in ours.parameters())
    calls = []
    real = dwconv.fwd

    def spy(*a, **k):
        calls.append(k.get("post") is not None)
        return real(*a, **k)

    monkeypatch.setattr(dwconv, "fwd", spy)
    x = torch.randn(2, inp, 15, 21, generator=g, dtype=torch.float64)
    with torch.no_grad():
        y = ours(nhwc(x))
        yr = ref(x)
    close(y, yr, "output")
    assert calls == [True]
    with torch.inference_mode():
        close(ours(nhwc(x)), yr, "output (inference_mode)")
    assert calls == [True, True]
    # with autograd recording, the unfused branch keeps y2 for the backward
    ours(nhwc(x)).sum().backward()
    assert calls == [True, True, False]


# ---------------------------------------------------------------------------------------------- whole model
def _mobilenet(dev=DEV):
    import bts
    torch.manual_seed(0)
    p = types.SimpleNamespace(encoder="mobilenetv2_bts", max_depth=80.0, dataset="kitti", bts_size=512, pretrained=False)
    m = bts.BtsModel(p)
    m.decoder.apply(bts.weights_init_xavier)
    return m


@pytest.mark.parametrize("mode", ["eval", "train"])
def test_mobilenet_k16_shape_vs_oracle(mode):
    import bts
    m = _mobilenet()
    orc = O.OracleModel("mobilenetv2_bts", 80.0, "kitti", 512)
    orc.load_state_dict(m.state_dict())
    m.to(DEV)
    getattr(m, mode)()
    getattr(orc, mode)()
    H, W = 352, 704
    g = torch.Generator().manual_seed(1)
    x = torch.randn(1, 3, H, W, generator=g)
    focal = torch.full((1,), 715.0873)
    with torch.no_grad():
        out = m(x.to(DEV), focal.to(DEV))
        ref = orc(x, focal)
    check_outputs(out, ref)
    if mode == "train":
        gt = torch.rand(1, 1, H, W, generator=g) * 80
        mask = gt > 1.0
        loss = bts.silog_loss(0.85)(out[4], gt.to(DEV), mask.to(DEV))
        lref = O.silog(ref[4], gt, mask, 0.85)
        assert abs(float(loss) - float(lref)) < 1e-3 * abs(float(lref))
        sd, sr = m.state_dict(), orc.state_dict()
        for k in sd:
            if k.endswith("running_var"):
                close(sd[k], sr[k], k, tol=1e-4)
            elif k.endswith("running_mean"):     # often ~0 (a conv of a zero-mean BatchNorm output): scale by the std
                std = float(sr[k[:-4] + "var"].sqrt().max())
                assert float((sd[k].cpu().double() - sr[k].double()).abs().max()) <= 1e-4 * std, k


def _batch(B=2, H=96, W=128, seed=5):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, 3, H, W, generator=g).to(DEV)
    gt = (torch.rand(B, 1, H, W, generator=g) * 80).to(DEV)
    focal = torch.full((B,), 715.0873, device=DEV)
    return x, focal, gt


def test_mobilenet_training_steps_are_bit_reproducible():
    import bts
    x, focal, gt = _batch()
    crit = bts.silog_loss(0.85)

    def step():
        m = _mobilenet().to(DEV).train()
        out = m(x, focal)
        crit(out[4], gt, gt > 1.0).backward()
        return [o.detach().clone() for o in out], {k: q.grad.clone() for k, q in m.named_parameters() if q.grad is not None}

    (oa, ga), (ob, gb) = step(), step()
    for u, v in zip(oa, ob):
        assert torch.equal(u, v)
    assert ga.keys() == gb.keys() and len(ga) == len(list(_mobilenet().parameters()))
    for k in ga:
        assert torch.equal(ga[k], gb[k]), k


def test_mobilenet_graphed_step_matches_eager_bit_for_bit():
    import bts
    from bts_b200.graph import GraphedTrainStep
    x, focal, gt = _batch(seed=6)
    crit = bts.silog_loss(0.85)
    m = _mobilenet().to(DEV).train()
    loss_fn = lambda out, g: crit(out[4], g, g > 1.0)
    step = GraphedTrainStep(m, loss_fn, ((x, focal), (gt,)))
    loss_g = step((x, focal), (gt,)).clone()
    torch.cuda.synchronize()
    params = [p for p in m.parameters() if p.requires_grad]
    grads_g = [p.grad.clone() for p in params]
    static = [p.grad for p in params]
    for p in params:
        p.grad = None
    loss_e = loss_fn(m(x, focal), gt)
    loss_e.backward()
    assert torch.equal(loss_g, loss_e.detach())
    for p, gg in zip(params, grads_g):
        assert torch.equal(p.grad, gg)
    for p, s in zip(params, static):
        p.grad = s


def _kernel_names(prof):
    names = set()
    for e in prof.events():
        if e.device_type == torch.autograd.DeviceType.CUDA:
            names.add(e.name)
    return names


def _library_kernels():
    stems = set()
    for f in glob.glob(os.path.join(ROOT, "bts_b200", "csrc", "*.cu")):
        src = open(f).read()
        stems.update(re.findall(r"__global__\s+void\s+(?:__launch_bounds__\([^)]*\)\s+)?(\w+)\s*\(", src))
    return stems


def test_mobilenet_step_runs_no_foreign_kernels():
    import bts
    from torch.profiler import ProfilerActivity, profile
    x, focal, gt = _batch()
    crit = bts.silog_loss(0.85)

    def kernels(enc):
        p = types.SimpleNamespace(encoder=enc, max_depth=80.0, dataset="kitti", bts_size=512, pretrained=False)
        torch.manual_seed(0)
        m = bts.BtsModel(p).to(DEV).train()
        crit(m(x, focal)[4], gt, gt > 1.0).backward()          # warm-up: packing, allocator, module loads
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            m.zero_grad(set_to_none=True)
            crit(m(x, focal)[4], gt, gt > 1.0).backward()
            torch.cuda.synchronize()
        return _kernel_names(prof)

    mob, dense = kernels("mobilenetv2_bts"), kernels("densenet121_bts")
    assert any("dw3x3_fwd_kernel" in k for k in mob) and any("dw3x3_wgrad_kernel" in k for k in mob)
    banned = [k for k in mob if re.search(r"cudnn|batch_norm|hardtanh|xmma|convolve|cutlass|depthwise", k, re.I)]
    assert not banned, "library kernels in the MobileNetV2 step: %s" % banned[:8]
    ours = _library_kernels()
    foreign = [k for k in mob - dense if not any(re.search(r"\b%s\b" % s, k) for s in ours)]
    assert not foreign, "kernels of the MobileNetV2 step that are neither libbts_b200.so's nor in a DenseNet step: %s" % \
        foreign[:8]
