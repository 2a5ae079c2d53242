"""The whole model in single-pass TF32 mode (bts_b200.set_precision("tf32")): accuracy against the fp64 oracle, a
training step, isolation from the default mode, CUDA-graph capture and the routing of the CUDA-core heads."""
import types

import pytest
import torch

import bts_oracle as O

pytestmark = pytest.mark.gpu

ENCODERS = ["densenet121_bts", "densenet161_bts", "resnet50_bts", "resnet101_bts", "resnext50_bts", "resnext101_bts",
            "mobilenetv2_bts"]
PARITY_KERNELS = ("conv_tc_kernel", "wgrad_tc_kernel", "wgrad2_tc_kernel")
TF32_KERNELS = ("conv_tf32_kernel", "wgrad_tf32_kernel", "wgrad2_tf32_kernel")


class mode:
    """with mode("tf32"): ... -- restores the previous mode on exit"""

    def __init__(self, m):
        self.m = m

    def __enter__(self):
        import bts_b200
        self.prev = bts_b200.set_precision(self.m)

    def __exit__(self, *exc):
        import bts_b200
        bts_b200.set_precision(self.prev)


def _model(enc, seed=0):
    import bts
    torch.manual_seed(seed)
    m = bts.BtsModel(types.SimpleNamespace(encoder=enc, max_depth=10.0, dataset="nyu", bts_size=512))
    m.decoder.apply(bts.weights_init_xavier)
    return m


def _calibrate(m, x, focal):
    """running BatchNorm statistics set to those of one batch (momentum 1), as a trained network's would be: with the
    initial statistics (mean 0, variance 1) a deep random-init network in eval mode does not normalise its activations,
    and its depth depends on every rounding of the encoder (ResNet-101: 3.5e-3 from fp32 rounding alone)"""
    bns = [mod for mod in m.modules() if isinstance(mod, torch.nn.modules.batchnorm._BatchNorm)]
    for bn in bns:
        bn.momentum = 1.0
    m.train()
    with torch.no_grad():
        m(x, focal)
    for bn in bns:
        bn.momentum = 0.1
    m.eval()


def _batch(B, H, W, seed=1):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, 3, H, W, generator=g)
    focal = torch.full((B,), 518.8579)
    gt = torch.rand(B, 1, H, W, generator=g) * 10
    return x, focal, gt


def _rel(a, b):
    """normwise relative error ||a - b|| / ||b||"""
    a, b = a.detach().cpu().double(), b.detach().cpu().double()
    return float((a - b).norm() / b.norm())


@pytest.mark.parametrize("enc", ENCODERS)
def test_eval_forward_against_the_fp64_oracle(enc):
    """final depth within 1e-1 (normwise relative) of the fp64 oracle, and at least 10x less exact than the fp32-mode
    depth; BatchNorm statistics calibrated on the batch (in fp32 mode) first.  Measured on an H100: 7.2e-3 (DenseNet-121
    and -161), 1.3e-2 (ResNeXt-50), 1.7e-2 (ResNet-50), 3.2e-2 (MobileNetV2), 3.4e-2 (ResNet-101), 4.7e-2 (ResNeXt-101);
    fp32 mode 1.5e-5 to 9.9e-5.  The deep random-init encoders amplify the per-layer TF32 rounding; the bar leaves a 2x
    margin over the worst of them."""
    m = _model(enc).cuda()
    x, focal, _ = _batch(1, 96, 128)
    _calibrate(m, x.cuda(), focal.cuda())
    orc = O.OracleModel(enc, 10.0, "nyu", 512).double()
    orc.load_state_dict({k: v.double() if v.is_floating_point() else v for k, v in m.state_dict().items()})
    orc.eval()
    with torch.no_grad():
        ref = orc(x.double(), focal.double())[4]
        d32 = m(x.cuda(), focal.cuda())[4].clone()
        with mode("tf32"):
            d1 = m(x.cuda(), focal.cuda())[4].clone()
    e1, e32 = _rel(d1, ref), _rel(d32, ref)
    print("%s eval depth vs fp64 oracle: tf32 %.3g, fp32 %.3g" % (enc, e1, e32))
    assert e1 < 1e-1, (e1, e32)
    assert not torch.equal(d1, d32) and e1 > 10 * e32, (e1, e32)


def test_densenet121_train_step():
    """One training step of DenseNet-121 (B = 2, 96 x 128, train-mode BatchNorm) in TF32 mode: finite loss and
    gradients, and a loss within 1e-3 relative of the fp64 oracle's.  Measured on an H100: 7.0e-5, so the bar leaves a
    14x margin."""
    import bts
    m = _model("densenet121_bts")
    orc = O.OracleModel("densenet121_bts", 10.0, "nyu", 512).double()
    orc.load_state_dict({k: v.double() if v.is_floating_point() else v for k, v in m.state_dict().items()})
    m.cuda().train()
    orc.train()
    x, focal, gt = _batch(2, 96, 128)
    mask = gt > 0.1
    with mode("tf32"):
        out = m(x.cuda(), focal.cuda())
        loss = bts.silog_loss(0.85)(out[4], gt.cuda(), mask.cuda())
        loss.backward()
    lref = float(O.silog(orc(x.double(), focal.double())[4], gt.double(), mask, 0.85).detach())
    assert torch.isfinite(loss.detach()).all()
    grads = [p.grad for p in m.parameters() if p.requires_grad and p.grad is not None]
    assert grads and all(bool(torch.isfinite(g).all()) for g in grads)
    e = abs(float(loss.detach()) - lref) / abs(lref)
    print("tf32 train-step loss %.6f, fp64 oracle %.6f, relative %.3g" % (float(loss.detach()), lref, e))
    assert e < 1e-3, e


def test_modes_are_isolated():
    """fp32 -> tf32 -> fp32 on the same inputs: the two fp32 results are bit-identical, the tf32 one differs"""
    m = _model("densenet121_bts").cuda().eval()
    x, focal, _ = _batch(1, 96, 128)
    with torch.no_grad():
        a = m(x.cuda(), focal.cuda())[4].clone()
        with mode("tf32"):
            b = m(x.cuda(), focal.cuda())[4].clone()
        c = m(x.cuda(), focal.cuda())[4].clone()
    assert torch.equal(a, c) and not torch.equal(a, b)


def _tc_kernels(fn):
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    names = [e.name for e in prof.events()]
    return ({k for k in PARITY_KERNELS if any(k + "<" in n or k + "I" in n for n in names)},
            {k for k in TF32_KERNELS if any(k + "<" in n or k + "I" in n for n in names)})


def test_graph_captured_in_tf32_mode():
    """A GraphedTrainStep captured in TF32 mode matches an eager TF32 step bit for bit, launches only the single-pass
    tensor-core kernels, keeps replaying TF32 after the mode is switched back, and two replays are bit-identical"""
    import bts
    from bts_b200.graph import GraphedTrainStep
    m = _model("densenet121_bts").cuda().train()
    x, focal, gt = (t.cuda() for t in _batch(2, 96, 128, seed=6))
    crit = bts.silog_loss(0.85)
    loss_fn = lambda out, g: crit(out[4], g, g > 1.0)
    params = [p for p in m.parameters() if p.requires_grad]
    with mode("tf32"):
        step = GraphedTrainStep(m, loss_fn, ((x, focal), (gt,)))
    parity, tf32 = _tc_kernels(lambda: step((x, focal), (gt,)))          # replayed with the default mode active
    assert not parity and tf32 == set(TF32_KERNELS), (parity, tf32)
    loss_g = step((x, focal), (gt,)).clone()
    torch.cuda.synchronize()
    grads_g = [p.grad.clone() for p in params]
    loss_g2 = step((x, focal), (gt,)).clone()
    torch.cuda.synchronize()
    assert torch.equal(loss_g, loss_g2) and all(torch.equal(p.grad, g) for p, g in zip(params, grads_g))
    for p in params:
        p.grad = None
    with mode("tf32"):
        loss_e = loss_fn(m(x, focal), gt)
        loss_e.backward()
    assert torch.equal(loss_g, loss_e.detach())
    assert all(torch.equal(p.grad, g) for p, g in zip(params, grads_g))


def test_cuda_core_heads_keep_their_routing():
    """In both modes the reduction heads run the CUDA-core kernels (bts_conv_pw_* for the narrow 1x1 layers at
    >= 200k pixels, bts_conv_c1_* for Cout = 1) and every engine call has the same shape: only the numerics of the
    tensor-core engine follow the mode"""
    import bts
    from bts_b200 import conv
    m = _model("densenet121_bts").cuda().train()
    x, focal, gt = (t.cuda() for t in _batch(2, 352, 288, seed=3))    # 2 x 352 x 288 = 202752 full-resolution pixels
    calls = {}
    for md in ("fp32", "tf32"):
        with mode(md):
            conv.set_trace(True)
            try:
                m.zero_grad(set_to_none=True)
                bts.silog_loss(0.85)(m(x, focal)[4], gt, gt > 1.0).backward()
                torch.cuda.synchronize()
                calls[md] = sorted((k, d) for k, d, _, _, _ in conv.trace_log)
            finally:
                conv.set_trace(False)
    kinds = {k for k, _ in calls["tf32"]}
    assert {"pwfwd", "pwwgrad", "c1fwd", "c1wgrad"} <= kinds, kinds
    assert calls["tf32"] == calls["fp32"]
