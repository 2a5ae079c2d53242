"""Worker of tests/test_multigpu_gpu.py (one process per GPU, launched by torch.distributed.run).
Checks, for the data-parallel path of the reference (DistributedDataParallel(find_unused_parameters=True), bts_main.py:352):
  (1) gradients after DDP's NCCL all-reduce == mean over ranks of the gradients each rank computes alone on its shard;
  (2) BatchNorm running statistics entering a forward pass equal rank 0's (DDP broadcast_buffers), although every rank
      normalises with its own batch statistics (no SyncBN, SURVEY Q9)."""
import os
import sys
import types

import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    dist.init_process_group("nccl", device_id=dev)
    import bts
    enc = sys.argv[1] if len(sys.argv) > 1 else "densenet121_bts"
    p = types.SimpleNamespace(encoder=enc, max_depth=10.0, dataset="nyu", bts_size=512, pretrained=False)

    def build():
        torch.manual_seed(0)
        m = bts.BtsModel(p)
        m.decoder.apply(bts.weights_init_xavier)
        return m.to(dev).train()

    solo, par = build(), build()
    ddp = torch.nn.parallel.DistributedDataParallel(par, device_ids=[local], find_unused_parameters=True)
    g = torch.Generator().manual_seed(100 + rank)                # every rank its own shard
    x = torch.randn(2, 3, 128, 160, generator=g).to(dev)
    gt = (torch.rand(2, 1, 128, 160, generator=g) * 10).to(dev)
    focal = torch.full((2,), 518.8579, device=dev)
    crit = bts.silog_loss(0.85)
    crit(solo(x, focal)[4], gt, gt > 0.1).backward()
    crit(ddp(x, focal)[4], gt, gt > 0.1).backward()
    # `solo` and `par` run the same arithmetic on the same shard; the engine is bit-reproducible run to run
    # (tools/determinism_probe.py: every reduction has a fixed order or runs in fp64), so what remains between them is the
    # all-reduce itself: NCCL's ring sum of the world's gradients in fp32 vs this test's own all_reduce + divide.
    worst, errs = 0.0, []
    for (k, a), (_, b) in zip(solo.named_parameters(), par.named_parameters()):
        if a.grad is None:
            assert b.grad is None or float(b.grad.abs().sum()) == 0.0, k
            continue
        mean = a.grad.clone()
        dist.all_reduce(mean)
        mean /= world
        err = float((b.grad - mean).norm() / mean.norm().clamp_min(1e-20))
        worst = max(worst, err)
        errs.append(err)
        assert err < 1e-5, "%s: DDP gradient differs from the mean of the per-shard gradients by %.3g" % (k, err)
    # (1b) the native schedule of bench.py -- bts_b200.dist.FlatGradReducer -- produces the same averaged gradients
    from bts_b200 import dist as D
    flat_m = build()
    red = D.FlatGradReducer(flat_m.parameters())
    crit(flat_m(x, focal)[4], gt, gt > 0.1).backward()
    red.reduce()
    for (k, a), (_, b) in zip(flat_m.named_parameters(), par.named_parameters()):
        if b.grad is None:
            continue
        err = float((a.grad - b.grad).norm() / b.grad.norm().clamp_min(1e-20))
        assert err < 1e-5, "%s: flat reducer vs DDP %.3g" % (k, err)
    bb = D.FlatBufferBroadcaster(flat_m)
    bb.broadcast(0)
    fb = (flat_m.encoder.base_model.norm0 if hasattr(flat_m.encoder.base_model, "norm0") else flat_m.encoder.base_model.bn1)
    chk = fb.running_var.clone()
    dist.broadcast(chk, 0)
    assert torch.equal(chk, fb.running_var)
    # buffers: after step 1 each rank holds its own running statistics; the next forward starts from rank 0's
    bn = par.encoder.base_model.norm0 if hasattr(par.encoder.base_model, "norm0") else par.encoder.base_model.bn1
    mine = bn.running_mean.clone()
    r0 = mine.clone()
    dist.broadcast(r0, 0)
    seen = {}
    def grab(_module, _args):                    # (a pre-hook's return value replaces the inputs: return None)
        seen.setdefault("rm", bn.running_mean.clone())

    h = par.register_forward_pre_hook(grab)
    with torch.no_grad():
        ddp(x, focal)
    h.remove()
    assert torch.equal(seen["rm"], r0), "buffers entering the forward pass differ from rank 0's"
    if world > 1 and rank > 0:
        assert not torch.equal(mine, r0), "per-rank batch statistics expected to differ before the broadcast"
    dist.barrier()
    if rank == 0:
        print("DIST_OK worst_grad_err=%.3g world=%d" % (worst, world))
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
