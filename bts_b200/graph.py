"""CUDA-graph capture of the training step's forward + loss + backward (north star: "CUDA streams and graphs instead of a
tracing compiler"; SURVEY section 7 step 8).

The step launches ~2000 kernels through ctypes plus the Python of ~1100 autograd nodes; once the kernels are fast that host
work -- not the GPU -- sets the step time (and at 8 processes per node the launch paths contend).  Everything on the path is
capturable: no host synchronisation, allocations through torch's caching allocator (graph-private pool), BatchNorm running
statistics and `num_batches_tracked` updated by device ops, packed conv operators re-written IN PLACE by
bts_b200.optim.FusedAdamW after each step.  One replay = one step's forward + loss + backward; the gradients land in static
`.grad` tensors that the (eager) collective and optimizer step then read.

The numeric mode of the tensor-core engine (bts_b200.set_precision) is resolved when each launch is enqueued, so a graph
replays the mode it was captured in, whatever the mode is at replay time.  Capture a new GraphedTrainStep after switching.
"""
import torch


class GraphedTrainStep:
    def __init__(self, model, loss_fn, example, warmup=3):
        """model: nn.Module in train mode; loss_fn(outputs, *targets) -> scalar; example = (inputs tuple, targets tuple) of
        CUDA tensors with the shapes of every later step (static shapes: one batch size, one resolution)."""
        inputs, targets = example
        self.inputs = [t.clone() for t in inputs]
        self.targets = [t.clone() for t in targets]
        self.model = model
        params = [p for p in model.parameters() if p.requires_grad]
        cur = torch.cuda.current_stream()
        side = torch.cuda.Stream()
        side.wait_stream(cur)
        with torch.cuda.stream(side):                      # warm-up off the capturing stream (torch.cuda.graphs recipe)
            for _ in range(warmup):
                for p in params:
                    p.grad = None
                loss_fn(model(*self.inputs), *self.targets).backward()
        cur.wait_stream(side)
        torch.cuda.synchronize()
        for p in params:
            p.grad = None
        from . import _lib
        l0 = _lib.launches
        self.graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(self.graph):
            self.loss = loss_fn(model(*self.inputs), *self.targets)
            self.loss.backward()
        self.launches_per_replay = _lib.launches - l0       # native launches recorded into the graph
        self.params = params

    def __call__(self, inputs, targets):
        """copies the batch into the graph's static buffers (device->device, or host->device when given pinned host
        tensors), replays, returns the (static) loss tensor; gradients are in p.grad of every trainable parameter"""
        from . import _lib
        for dst, src in zip(self.inputs, inputs):
            if dst.data_ptr() != src.data_ptr():
                dst.copy_(src, non_blocking=True)
        for dst, src in zip(self.targets, targets):
            if dst.data_ptr() != src.data_ptr():
                dst.copy_(src, non_blocking=True)
        self.graph.replay()
        _lib.count(self.launches_per_replay)
        return self.loss
