"""Data-parallel plumbing for the hot path (SURVEY 8e): one process per GPU, batch sharding, ONE collective per
step -- a mean all-reduce of the gradient vector -- plus the rank-0 broadcast of BatchNorm buffers that the reference
gets from DistributedDataParallel (bts_main.py:352: C1 + C3 in SURVEY 2.5).

The drop-in boundary is the module, so an unchanged bts_main.py keeps using torch's DDP.  `FlatGradReducer` +
`FlatBufferBroadcaster` are the native alternative that bench.py uses for N > 1 (`--reducer flat`, the default;
`--reducer ddp` runs torch's DDP exactly as bts_main.py does): one all-reduce over a single flat buffer after backward.  Works with the gloo backend on CPU tensors, which is how
tests/test_dist_cpu.py covers it.
"""
import torch
import torch.distributed as dist


def shard_batch(tensors, rank, world):
    """contiguous batch shards, like DistributedSampler + bts_main.py:351 (global batch / ngpus per rank)"""
    out = []
    for t in tensors:
        n = t.shape[0]
        if n % world:
            raise ValueError("global batch %d is not divisible by world size %d" % (n, world))
        per = n // world
        out.append(t[rank * per:(rank + 1) * per])
    return out


class FlatGradReducer:
    """ONE mean all-reduce of the whole gradient vector per step over a single persistent flat fp32 buffer.

    DDP buckets the 187 MB (DenseNet-161) gradient into 25 MB pieces and overlaps their all-reduces with the backward
    pass; every conv kernel here is a persistent one-CTA-per-SM grid, so NCCL's reduction kernels cannot run beside
    them and the "overlap" serialises piecemeal.  The schedule is therefore the simple one:
    finish backward, gather the gradients into the flat buffer with one multi-tensor copy, one NCCL all-reduce (AVG),
    and let the optimizer read the flat views.  Parameters without a gradient contribute zeros (like DDP with
    find_unused_parameters=True, bts_main.py:352).  Works with gloo on CPU tensors (tests/test_dist_cpu.py)."""

    def __init__(self, params, group=None):
        self.params = [p for p in params if p.requires_grad]
        self.group = group
        n = sum(p.numel() for p in self.params)
        dev = self.params[0].device if self.params else torch.device("cpu")
        self.flat = torch.zeros(n, device=dev, dtype=torch.float32)
        self.views = []
        o = 0
        for p in self.params:
            self.views.append(self.flat[o:o + p.numel()].view_as(p))
            o += p.numel()

    @torch.no_grad()
    def reduce(self, inplace=False):
        """inplace=False: afterwards p.grad IS the reduced flat view (no copy back).  inplace=True: the averaged values are
        copied back into the existing .grad tensors -- for static gradients of a CUDA-graphed step (bts_b200.graph)."""
        world = dist.get_world_size(self.group)
        src, dst, missing = [], [], []
        for p, v in zip(self.params, self.views):
            if p.grad is None:
                missing.append(v)
            elif p.grad.data_ptr() != v.data_ptr():
                src.append(p.grad)
                dst.append(v)
        if missing:
            torch._foreach_zero_(missing)
        if dst:
            torch._foreach_copy_(dst, src)                   # one multi-tensor kernel, not one launch per parameter
        avg = self.flat.is_cuda                              # NCCL averages in the collective; gloo has no AVG
        dist.all_reduce(self.flat, op=dist.ReduceOp.AVG if avg else dist.ReduceOp.SUM, group=self.group)
        if not avg:
            self.flat.div_(world)
        if inplace and dst:
            torch._foreach_copy_(src, dst)
            for p, v in zip(self.params, self.views):
                if p.grad is None:
                    p.grad = v
            return
        for p, v in zip(self.params, self.views):
            p.grad = v                                       # the optimizer reads the reduced flat buffer in place


class FlatBufferBroadcaster:
    """rank-0 BatchNorm running statistics to every rank (DDP's broadcast_buffers, C3 in SURVEY 2.5) as ONE broadcast of
    a flat staging buffer per dtype instead of one collective per buffer (DenseNet-161: 525 buffers, 0.93 MB)."""

    def __init__(self, module, group=None):
        self.group = group
        by = {}
        for b in module.buffers():
            by.setdefault(b.dtype, []).append(b)
        self.sets = []
        for dt, bufs in by.items():
            flat = torch.empty(sum(b.numel() for b in bufs), device=bufs[0].device, dtype=dt)
            views, o = [], 0
            for b in bufs:
                views.append(flat[o:o + b.numel()].view_as(b))
                o += b.numel()
            self.sets.append((flat, bufs, views))

    @torch.no_grad()
    def broadcast(self, src=0):
        rank = dist.get_rank(self.group)
        for flat, bufs, views in self.sets:
            if rank == src:
                torch._foreach_copy_(views, bufs)
            dist.broadcast(flat, src=src, group=self.group)
            if rank != src:
                torch._foreach_copy_(bufs, views)


@torch.no_grad()
def broadcast_buffers(module, src=0, group=None):
    """one-shot form of FlatBufferBroadcaster (builds the staging buffers on every call)"""
    FlatBufferBroadcaster(module, group).broadcast(src)
