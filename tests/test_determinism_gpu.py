"""A training step of the engine is bit-reproducible run to run: every reduction either has a fixed order (warp butterflies,
per-warp shared-memory partials, split-K partial buffers summed by a second kernel) or is accumulated in fp64
(tools/determinism_probe.py reports the worst difference between two identical steps)."""
import types

import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("enc", ["densenet121_bts", "resnext50_bts"])
def test_two_identical_training_steps_give_identical_gradients(enc, monkeypatch):
    monkeypatch.setenv("BTS_B200_PRETRAINED", "0")
    import bts
    dev = torch.device("cuda", 0)
    p = types.SimpleNamespace(encoder=enc, max_depth=10.0, dataset="nyu", bts_size=512, pretrained=False)
    g = torch.Generator().manual_seed(5)
    x = torch.randn(2, 3, 96, 128, generator=g).to(dev)
    gt = (torch.rand(2, 1, 96, 128, generator=g) * 10).to(dev)
    focal = torch.full((2,), 518.8579, device=dev)
    crit = bts.silog_loss(0.85)

    def step():
        torch.manual_seed(0)
        m = bts.BtsModel(p)
        m.decoder.apply(bts.weights_init_xavier)
        m = m.to(dev).train()
        out = m(x, focal)
        crit(out[4], gt, gt > 0.1).backward()
        return [o.detach().clone() for o in out], {k: q.grad.clone() for k, q in m.named_parameters() if q.grad is not None}

    (oa, ga), (ob, gb) = step(), step()
    for u, v in zip(oa, ob):
        assert torch.equal(u, v)
    assert ga.keys() == gb.keys()
    for k in ga:
        assert torch.equal(ga[k], gb[k]), k
