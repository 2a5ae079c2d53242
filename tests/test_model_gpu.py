"""GPU parity tests of the module surface: decoder vs the reference's golden outputs, whole model vs the
oracle restatement on identical inputs and an identical state_dict (bar: <=1e-3 relative on fp32 depth)."""
import types

import numpy as np
import pytest
import torch

import bts_oracle as O

pytestmark = pytest.mark.gpu


def rel_err(a, b):
    """relative error with the denominator floored at 1e-3 of the map's typical magnitude"""
    a, b = a.double(), b.double()
    return (a - b).abs() / b.abs().clamp_min(1e-3 * b.abs().median())


def check_outputs(got, want, tol=1e-3):
    for i, (a, b) in enumerate(zip(got, want)):
        a, b = a.detach().cpu(), torch.as_tensor(b)
        assert a.shape == b.shape
        e = rel_err(a, b)
        if i < 3:
            # LPG maps: pixels whose plane denominator is ~0 (|depth| far above the map's scale) amplify any
            # ulp of difference without bound (SURVEY Q4, 8c hazard (i)); they are excluded, the rest must hold.
            ok = b.abs() < 20 * b.abs().median()
            assert ok.double().mean() > 0.98
            e = e[ok]
            # the amplification is continuous in the denominator, so a handful of the remaining pixels still sit at
            # 1.0-1.2e-3 on the deep ResNet/ResNeXt encoders: 99.9% of the pixels must meet the tolerance and none may
            # exceed 2x.  The final depth (the quantity the 1e-3 bar is stated on) and the 1x1 reduction keep the strict
            # max below.
            assert torch.quantile(e.flatten()[:: max(1, e.numel() // 4000000)], 0.999) < tol, \
                "output %d: 99.9%% rel err %.3g" % (i, torch.quantile(e.flatten(), 0.999))
            assert e.max() < 2 * tol, "output %d: max rel err %.3g" % (i, e.max())
            continue
        assert e.max() < tol, "output %d: max rel err %.3g" % (i, e.max())


@pytest.mark.parametrize("dataset", ["kitti", "nyu"])
@pytest.mark.parametrize("mode", ["eval", "train"])
def test_decoder_vs_reference_golden(golden, dataset, mode):
    import bts
    g = golden("decoder_" + dataset)
    md = float(g["max_depth"])
    dec = bts.bts(types.SimpleNamespace(max_depth=md, dataset=dataset), [int(c) for c in g["feat_channels"]], 128)
    dec.load_state_dict({k[3:]: torch.from_numpy(v) for k, v in g.items() if k.startswith("sd.")})
    dec.cuda()
    getattr(dec, mode)()
    feats = [torch.from_numpy(g["feat%d" % i]).cuda() for i in range(5)]
    with torch.no_grad():
        out = dec(feats, torch.from_numpy(g["focal"]).cuda())
    check_outputs(out, [g["%s_out%d" % (mode, i)] for i in range(5)])
    if mode == "train":        # running-stat update semantics (momentum 0.01, unbiased var) -- state_dict parity
        sd = dec.state_dict()
        for k, v in g.items():
            if k.startswith("sd_after."):
                np.testing.assert_allclose(sd[k[9:]].cpu().numpy(), v, rtol=1e-4, atol=1e-6)


@pytest.mark.parametrize("enc,mode,B", [("densenet121_bts", "eval", 1), ("densenet121_bts", "train", 2),
                                         ("densenet161_bts", "train", 2), ("resnext50_bts", "train", 2),
                                         ("resnext101_bts", "train", 2), ("resnet50_bts", "eval", 1),
                                         ("mobilenetv2_bts", "eval", 1), ("mobilenetv2_bts", "train", 2)])
def test_full_model_forward_backward_vs_oracle(enc, mode, B):
    import bts
    torch.manual_seed(0)
    p = types.SimpleNamespace(encoder=enc, max_depth=10.0, dataset="nyu", bts_size=512)
    m = bts.BtsModel(p)
    m.decoder.apply(bts.weights_init_xavier)
    orc = O.OracleModel(enc, 10.0, "nyu", 512)
    orc.load_state_dict(m.state_dict())
    m.cuda()
    getattr(m, mode)()
    getattr(orc, mode)()
    H, W = 96, 128
    x = torch.randn(B, 3, H, W, generator=torch.Generator().manual_seed(1))
    focal = torch.full((B,), 518.8579)
    gt = torch.rand(B, 1, H, W, generator=torch.Generator().manual_seed(2)) * 10
    mask = gt > 0.1
    if mode == "eval":
        with torch.no_grad():
            check_outputs(m(x.cuda(), focal.cuda()), orc(x, focal))
        return
    out = m(x.cuda(), focal.cuda())
    ref = orc(x, focal)
    check_outputs(out, [r.detach() for r in ref])            # 1e-3 relative, the bar of north_star, train-mode BN included
    loss = bts.silog_loss(0.85)(out[4], gt.cuda(), mask.cuda())
    lref = O.silog(ref[4], gt, mask, 0.85)
    assert abs(float(loss.detach()) - float(lref.detach())) < 1e-3 * abs(float(lref.detach()))
    loss.backward()
    lref.backward()
    # Gradients of a random-init, batch-stat-BN network are ill-conditioned: the reference's own fp32 arithmetic is
    # only accurate to ~1e-2 on some tensors.  Measure both against an fp64 run of the oracle and require ours to be
    # as accurate as the fp32 reference (x4 slack + 2e-3 floor) -- that is the parity that means something here.
    orc64 = O.OracleModel(enc, 10.0, "nyu", 512).double()
    orc64.load_state_dict({k: v.double() if v.is_floating_point() else v for k, v in m.state_dict().items()})
    orc64.train()
    r64 = orc64(x.double(), focal.double())
    O.silog(r64[4], gt.double(), mask, 0.85).backward()
    g64 = {k: p_.grad for k, p_ in orc64.named_parameters()}
    gm = dict(m.named_parameters())
    go = dict(orc.named_parameters())
    worst_ours = worst_ref = 0.0
    for k, b in g64.items():
        if b is None:
            assert gm[k].grad is None or float(gm[k].grad.abs().sum()) == 0.0
            continue
        den = b.norm().clamp_min(1e-20)
        worst_ours = max(worst_ours, float((gm[k].grad.cpu().double() - b).norm() / den))
        worst_ref = max(worst_ref, float((go[k].grad.double() - b).norm() / den))
    assert worst_ours < 4 * worst_ref + 2e-3, "worst per-tensor gradient error vs fp64: ours %.3g, fp32 reference %.3g" % (
        worst_ours, worst_ref)



# ---- the BASELINE.json shapes themselves (SURVEY 8d): T1 = DenseNet-121 416x544 B=1 eval (configs[0]); K16 / N4 spatial
#      sizes with DenseNet-161 (44x88 maps under dilation 18/24, 11x22 deepest features), B=1 so the CPU oracle finishes
#      in seconds.  Train mode uses batch statistics (over H x W of the single image).
@pytest.mark.parametrize("enc,H,W,dataset,md,focal,mode", [
    ("densenet121_bts", 416, 544, "nyu", 10.0, 518.8579, "eval"),     # T1
    ("densenet161_bts", 352, 704, "kitti", 80.0, 721.5377, "train"),  # K16 shape
    ("densenet161_bts", 416, 544, "nyu", 10.0, 518.8579, "train"),    # N4 shape
    ("densenet161_bts", 352, 704, "kitti", 80.0, 721.5377, "eval"),
])
def test_full_model_at_baseline_shapes_vs_oracle(enc, H, W, dataset, md, focal, mode):
    import bts
    torch.manual_seed(0)
    p = types.SimpleNamespace(encoder=enc, max_depth=md, dataset=dataset, bts_size=512)
    m = bts.BtsModel(p)
    m.decoder.apply(bts.weights_init_xavier)
    orc = O.OracleModel(enc, md, dataset, 512)
    orc.load_state_dict(m.state_dict())
    m.cuda()
    getattr(m, mode)()
    getattr(orc, mode)()
    x = torch.randn(1, 3, H, W, generator=torch.Generator().manual_seed(0))
    f = torch.full((1,), focal, dtype=torch.float64)
    with torch.no_grad():
        got = m(x.cuda(), f.cuda())
        want = orc(x, f)
    assert all(o.shape == (1, 1, H, W) and o.dtype == torch.float32 for o in got)
    check_outputs(got, want)
    if mode == "train":           # running statistics after the step: state_dict parity at the real shape
        sd, so = m.state_dict(), orc.state_dict()
        for k in ("decoder.bn5.running_var", "decoder.bn2.running_mean", "decoder.daspp_24.atrous_conv.first_bn.running_var"):
            np.testing.assert_allclose(sd[k].cpu().numpy(), so[k].numpy(), rtol=2e-4, atol=1e-6)
