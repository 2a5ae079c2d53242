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

Eval graphs (set_eval_graphs / BTS_B200_EVAL_GRAPH=1, off by default) bring GraphedInference to code that only calls
model(x, focal), such as the unmodified bts_test.py and bts_main.py --do_online_eval: BtsModel.forward hands an eval
forward under no_grad to eval_forward(), which serves it from a small per-model cache of GraphedInference objects.
"""
import collections
import os
import weakref

import torch

EVAL_GRAPH_KEYS = 4        # input signatures a model's cache holds (captured or seen once), least recently used out first


def _switch_from_env():
    value = os.environ.get("BTS_B200_EVAL_GRAPH", "0")
    if value not in ("0", "1"):
        raise ValueError("BTS_B200_EVAL_GRAPH: expected 0 or 1, got %r" % value)
    return value == "1"


_eval_graphs = _switch_from_env()
_caches = weakref.WeakSet()          # every model's _EvalGraphCache, so that switching off frees their graphs
_stats = {"captures": 0, "replays": 0, "evictions": 0, "recaptures": 0}
_capturing = 0                       # GraphedInference warm-up or capture in progress: its forwards run the eager body


def set_eval_graphs(on):
    """Turns the eval-graph cache on or off for every BtsModel and returns the previous setting.  Off (the default, unless
    BTS_B200_EVAL_GRAPH=1) also frees every graph captured so far.

    While on, an eval-mode BtsModel (not a DataParallel replica) called under no_grad with a CUDA fp32 4-D input, outside
    a CUDA graph capture, runs eager the first time it sees an input signature (the shapes and dtypes of x and focal, the
    device, the precision mode), captures a GraphedInference the second time and replays it from then on.  Each model
    keeps EVAL_GRAPH_KEYS signatures; the least recently used one is dropped, with its graph and the graph's memory pool.
    Outputs are fresh clones of the graph's, bit-identical to the eager forward's.

    What a driver accepts with it: each captured signature keeps a private memory pool; in-place writes through `.data`
    are seen only after bts_b200.conv.invalidate_packed(); forward hooks on the model's modules do not run on replays.  A
    graph whose parameters or buffers were re-allocated (`p.data = ...`, `model.to(...)`) is captured again."""
    global _eval_graphs
    if on not in (True, False):
        raise ValueError("set_eval_graphs: expected True or False, got %r" % (on,))
    prev, _eval_graphs = _eval_graphs, bool(on)
    if not _eval_graphs:
        for cache in list(_caches):
            cache.entries.clear()
    return prev


def get_eval_graphs():
    return _eval_graphs


def eval_graph_stats():
    """process-wide counts of the eval-graph caches: captures, replays, evictions (captured graphs dropped to make room)
    and recaptures (graphs dropped because the model's storage moved)"""
    return dict(_stats)


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
    `.to()`) cannot be followed by the graph: the call raises and a new capture is needed.

    `capture_error_mode` is torch.cuda.graph's: "thread_local" lets other threads of the process (a DataLoader's
    pin-memory thread) make CUDA calls while the capture runs."""

    def __init__(self, model, x, focal, warmup=2, capture_error_mode="global"):
        global _capturing
        from . import _lib, conv
        if model.training:
            raise ValueError("GraphedInference captures the eval forward: call model.eval() first")
        self.model = model
        self.x = x.clone()
        self.focal = focal.clone()
        cur = torch.cuda.current_stream()
        side = torch.cuda.Stream()
        side.wait_stream(cur)
        _capturing += 1
        try:
            with torch.no_grad():
                with torch.cuda.stream(side):              # warm-up off the capturing stream: packs every operator
                    for _ in range(warmup):
                        model(self.x, self.focal)
                cur.wait_stream(side)
                torch.cuda.synchronize()
                l0 = _lib.launches
                self.graph = torch.cuda.CUDAGraph()
                with torch.cuda.graph(self.graph, capture_error_mode=capture_error_mode):
                    self.out = model(self.x, self.focal)
        finally:
            _capturing -= 1
        self.launches_per_replay = _lib.launches - l0
        self.params = list(model.parameters())
        self.tensors = [(t, t.data_ptr()) for t in self.params + list(model.buffers())]
        self.versions = [p._version for p in self.params]
        self.operators = conv.cached_operators(self.params)

    def _refresh(self):
        """False when a parameter or buffer was re-allocated since the capture; otherwise re-packs moved weights, True"""
        from . import conv
        for t, ptr in self.tensors:
            if t.data_ptr() != ptr:
                return False
        versions = [p._version for p in self.params]
        if conv.restore_operators(self.operators) or versions != self.versions:
            conv.repack_cached()
            self.versions = versions
        return True

    def replay(self, x, focal):
        """__call__, except that a re-allocated parameter or buffer returns None instead of raising"""
        from . import _lib
        if x.shape != self.x.shape or focal.shape != self.focal.shape:
            raise ValueError("GraphedInference was captured for x %s, focal %s; got %s, %s" % (
                tuple(self.x.shape), tuple(self.focal.shape), tuple(x.shape), tuple(focal.shape)))
        if not self._refresh():
            return None
        if x.data_ptr() != self.x.data_ptr():
            self.x.copy_(x, non_blocking=True)
        if focal.data_ptr() != self.focal.data_ptr():
            self.focal.copy_(focal, non_blocking=True)
        self.graph.replay()
        _lib.count(self.launches_per_replay)
        return self.out

    def __call__(self, x, focal):
        out = self.replay(x, focal)
        if out is None:
            raise RuntimeError("GraphedInference: a parameter or buffer of the model was re-allocated since the capture "
                               "(its storage moved); capture a new GraphedInference")
        return out


class _EvalGraphCache:
    """One model's eval graphs: input signature -> GraphedInference, or None for a signature seen once.  A copy or an
    unpickled model starts with an empty cache (graphs can be neither copied nor pickled)."""

    def __init__(self):
        self.entries = collections.OrderedDict()
        _caches.add(self)

    def __deepcopy__(self, memo):
        return _EvalGraphCache()

    def __reduce__(self):
        return _EvalGraphCache, ()


def eval_forward(model, x, focal):
    """BtsModel.forward's eval forward (no backward can follow) from the model's eval-graph cache (set_eval_graphs), or
    None when the caller is to run the eager forward: the cache is off or does not apply, or the signature is new."""
    from . import _lib, conv
    if not (_eval_graphs and not _capturing and not model.training and x.is_cuda and x.dtype == torch.float32
            and x.dim() == 4 and isinstance(focal, torch.Tensor) and not model.__dict__.get("_is_replica", False)
            and not conv.TRACE and not conv.SYNC_DEBUG and not torch.cuda.is_current_stream_capturing()):
        return None
    cache = model.__dict__.get("_eval_graph_cache")
    if cache is None:
        cache = model._eval_graph_cache = _EvalGraphCache()
    # conv.SPLITK (switched by tools and tests) is recorded into the graph like the precision mode
    key = (tuple(x.shape), x.dtype, x.device, tuple(focal.shape), focal.dtype, focal.device, conv.get_precision(),
           conv.SPLITK)
    entries = cache.entries
    if key not in entries:
        entries[key] = None
        if len(entries) > EVAL_GRAPH_KEYS:
            if entries.popitem(last=False)[1] is not None:
                _stats["evictions"] += 1
        return None
    entries.move_to_end(key)
    graphed = entries[key]
    out = None if graphed is None else graphed.replay(x, focal)
    if out is None:
        if graphed is not None:
            _stats["recaptures"] += 1
            entries[key] = graphed = None          # frees the stale graph and its pool before the new capture
        graphed = entries[key] = GraphedInference(model, x, focal, capture_error_mode="thread_local")
        _lib.count(-graphed.launches_per_replay)   # recorded by the capture, not run
        _stats["captures"] += 1
        out = graphed.replay(x, focal)
    _stats["replays"] += 1
    return tuple(t.clone() for t in out)
