"""CUDA-graph capture of the training step's forward + loss + backward (north star: "CUDA streams and graphs instead of a
tracing compiler"; SURVEY section 7 step 8).

The step launches ~2000 kernels through ctypes plus the Python of ~1100 autograd nodes; once the kernels are fast that host
work -- not the GPU -- sets the step time (and at 8 processes per node the launch paths contend).  Everything on the path is
capturable: no host synchronisation, allocations through torch's caching allocator (graph-private pool), BatchNorm running
statistics and `num_batches_tracked` updated by device ops, packed conv operators re-written IN PLACE by
bts_b200.optim.FusedAdamW after each step.  One replay = one step's forward + loss + backward; the gradients land in static
`.grad` tensors that the (eager) collective and optimizer step then read.

GraphedInference does the same for the batch-1 eval forward (bts_test.py, online eval): one replay = one model(x, focal)
in eval mode under no_grad (split-K engine launches included, conv.inference()), several hundred native launches without
their Python and ctypes cost.

The numeric mode of the tensor-core engine (bts_b200.set_precision) is resolved when each launch is enqueued, so a graph
replays the mode it was captured in, whatever the mode is at replay time.  Capture a new graph after switching.
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


class GraphedInference:
    """model(x, focal) of an eval-mode model under torch.no_grad(), captured for one input shape into one CUDA graph.

    __call__(x, focal) copies the inputs into the graph's static buffers, replays and returns the graph's static 5-tuple of
    outputs: the next call overwrites it, so clone what has to outlive it.  The graph replays the precision mode
    (bts_b200.set_precision) it was captured in.

    Weights may change between calls (online eval during training: optimizer steps, load_state_dict): BatchNorm running
    statistics are folded inside the graph and the CUDA-core kernels read the parameters themselves, so replays see
    their current values; the engine reads packed operators, which are re-packed in place (one launch) before a replay
    when a parameter's version counter moved.  In-place writes through `.data` do not move it: call
    bts_b200.conv.invalidate_packed() after those.  A parameter or buffer whose storage was replaced (`p.data = ...`,
    `.to()`) cannot be followed by the graph: the call raises and a new capture is needed."""

    def __init__(self, model, x, focal, warmup=2):
        from . import _lib, conv
        if model.training:
            raise ValueError("GraphedInference captures the eval forward: call model.eval() first")
        self.model = model
        self.x = x.clone()
        self.focal = focal.clone()
        cur = torch.cuda.current_stream()
        side = torch.cuda.Stream()
        side.wait_stream(cur)
        with torch.no_grad():
            with torch.cuda.stream(side):                  # warm-up off the capturing stream: packs every operator
                for _ in range(warmup):
                    model(self.x, self.focal)
            cur.wait_stream(side)
            torch.cuda.synchronize()
            l0 = _lib.launches
            self.graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(self.graph):
                self.out = model(self.x, self.focal)
        self.launches_per_replay = _lib.launches - l0
        self.params = list(model.parameters())
        self.tensors = [(t, t.data_ptr()) for t in self.params + list(model.buffers())]
        self.versions = [p._version for p in self.params]
        self.operators = conv.cached_operators(self.params)

    def _refresh(self):
        from . import conv
        for t, ptr in self.tensors:
            if t.data_ptr() != ptr:
                raise RuntimeError("GraphedInference: a parameter or buffer of the model was re-allocated since the capture "
                                   "(its storage moved); capture a new GraphedInference")
        versions = [p._version for p in self.params]
        if conv.restore_operators(self.operators) or versions != self.versions:
            conv.repack_cached()
            self.versions = versions

    def __call__(self, x, focal):
        from . import _lib
        if x.shape != self.x.shape or focal.shape != self.focal.shape:
            raise ValueError("GraphedInference was captured for x %s, focal %s; got %s, %s" % (
                tuple(self.x.shape), tuple(self.focal.shape), tuple(x.shape), tuple(focal.shape)))
        self._refresh()
        if x.data_ptr() != self.x.data_ptr():
            self.x.copy_(x, non_blocking=True)
        if focal.data_ptr() != self.focal.data_ptr():
            self.focal.copy_(focal, non_blocking=True)
        self.graph.replay()
        _lib.count(self.launches_per_replay)
        return self.out
