"""Batch-1 inference on the GPU: the eval forward with split-K engine launches (BtsModel.forward enters conv.inference()
when no backward can follow) against the oracle at the 1e-3 bar of test_model_gpu.check_outputs, training launches
without split-K, and bts_b200.graph.GraphedInference: the forward captured as one CUDA graph replays bit-identical to the
eager forward, also while BatchNorm running statistics, weights (an AdamW step) and the state_dict change under it."""
import types

import pytest
import torch

import bts_oracle as O
from test_model_gpu import check_outputs

pytestmark = pytest.mark.gpu


def _model(enc):
    import bts
    torch.manual_seed(0)
    p = types.SimpleNamespace(encoder=enc, max_depth=10.0, dataset="nyu", bts_size=512)
    m = bts.BtsModel(p)
    m.decoder.apply(bts.weights_init_xavier)
    return m


def _same(a, b):
    return all(torch.equal(u, v) for u, v in zip(a, b))


REDUCE = "conv_splitk_reduce_kernel"


def _reduces(fn):
    """(fn(), number of split-K reduce launches in it)"""
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        out = fn()
        torch.cuda.synchronize()
    return out, sum(REDUCE in e.name for e in prof.events())


@pytest.mark.parametrize("enc,H,W", [("densenet121_bts", 416, 544),        # T1
                                     ("densenet161_bts", 480, 640),        # NYU test split (bts_test.py)
                                     ("densenet121_bts", 96, 128), ("densenet161_bts", 96, 128),
                                     ("resnext50_bts", 96, 128), ("mobilenetv2_bts", 96, 128)])
def test_batch1_eval_forward_splits_and_matches_oracle(enc, H, W):
    m = _model(enc)
    orc = O.OracleModel(enc, 10.0, "nyu", 512)
    orc.load_state_dict(m.state_dict())
    m.cuda().eval()
    orc.eval()
    x = torch.randn(1, 3, H, W, generator=torch.Generator().manual_seed(1))
    f = torch.full((1,), 518.8579)
    with torch.no_grad():
        got, n = _reduces(lambda: m(x.cuda(), f.cuda()))
        want = orc(x, f)
    assert n > 0, "no split-K launch in the batch-1 eval forward"
    check_outputs(got, want)


def test_training_step_launches_no_split():
    """forward + backward of a train step: no launch enters the inference scope, although these small maps have few
    tiles; the same model in eval mode with grad enabled (a backward may follow) does not split either"""
    import bts
    m = _model("densenet121_bts").cuda().train()
    x = torch.randn(2, 3, 64, 96, generator=torch.Generator().manual_seed(3)).cuda()
    f = torch.full((2,), 518.8579).cuda()
    gt = torch.rand(2, 1, 64, 96, generator=torch.Generator().manual_seed(4)).cuda() * 10

    def step():
        out = m(x, f)
        bts.silog_loss(0.85)(out[4], gt, gt > 0.1).backward()

    _, n = _reduces(step)
    assert n == 0
    m.eval()
    _, n = _reduces(lambda: m(x, f)[4].sum().backward())
    assert n == 0
    with torch.no_grad():
        _, n = _reduces(lambda: m(x, f))
    assert n > 0


def test_graphed_t1_forward_matches_eager_and_oracle():
    """T1: DenseNet-121, one 416 x 544 image, eval forward"""
    from bts_b200.graph import GraphedInference
    m = _model("densenet121_bts")
    orc = O.OracleModel("densenet121_bts", 10.0, "nyu", 512)
    orc.load_state_dict(m.state_dict())
    m.cuda().eval()
    orc.eval()
    x = torch.randn(1, 3, 416, 544, generator=torch.Generator().manual_seed(1))
    f = torch.full((1,), 518.8579)
    gi = GraphedInference(m, x.cuda(), f.cuda())
    got = [t.clone() for t in gi(x.cuda(), f.cuda())]
    with torch.no_grad():
        eager = m(x.cuda(), f.cuda())
        want = orc(x, f)
    assert _same(got, eager)
    check_outputs(got, want)


def test_graphed_inference_follows_weight_and_statistics_changes():
    import bts
    from bts_b200.graph import GraphedInference
    m = _model("densenet121_bts").cuda().eval()
    g = torch.Generator().manual_seed(5)
    x = torch.randn(1, 3, 96, 128, generator=g).cuda()
    f = torch.full((1,), 518.8579).cuda()
    gi = GraphedInference(m, x, f)
    assert gi.launches_per_replay > 0

    def eager():
        with torch.no_grad():
            return [t.clone() for t in m(x, f)]

    def graphed():
        return [t.clone() for t in gi(x, f)]

    g0 = graphed()
    assert _same(eager(), g0)
    x2 = torch.randn(1, 3, 96, 128, generator=g).cuda()         # a new input through the static buffer
    with torch.no_grad():
        e2 = [t.clone() for t in m(x2, f)]
    assert _same(e2, [t.clone() for t in gi(x2, f)])

    # a train-mode forward moves the BatchNorm running statistics only: folded inside the graph, seen by the replay
    m.train()
    with torch.no_grad():
        m(x2 * 2 + 1, f)
    m.eval()
    g1 = graphed()
    assert not _same(g0, g1) and _same(eager(), g1)

    # an AdamW step (plus the running statistics of its train forward): the packed operators are re-packed in place
    opt = torch.optim.AdamW(m.parameters(), lr=1e-3)
    m.train()
    gt = torch.rand(2, 1, 96, 128, generator=g).cuda() * 10
    out = m(torch.cat([x, x2]), f.repeat(2))
    bts.silog_loss(0.85)(out[4], gt, gt > 0.1).backward()
    opt.step()
    m.eval()
    e3 = eager()                                   # the eager forward packs the new weights into buffers of its own
    g3 = graphed()
    assert not _same(g1, g3) and _same(e3, g3)

    # load_state_dict copies into the same storage
    m.load_state_dict(_model("densenet121_bts").state_dict())
    g4 = graphed()
    assert not _same(g3, g4) and _same(eager(), g4)

    # another input shape, or a parameter whose storage was replaced, cannot be replayed
    with pytest.raises(ValueError, match="captured for"):
        gi(torch.zeros(1, 3, 64, 128, device="cuda"), f)
    w = m.decoder.conv5[0].weight
    w.data = w.data.clone()
    with pytest.raises(RuntimeError, match="capture a new GraphedInference"):
        gi(x, f)


def test_graphed_inference_needs_eval_mode():
    from bts_b200.graph import GraphedInference
    m = _model("mobilenetv2_bts").cuda().train()
    with pytest.raises(ValueError, match="model.eval"):
        GraphedInference(m, torch.zeros(1, 3, 64, 96, device="cuda"), torch.ones(1, device="cuda"))
