"""Host side of the wgmma implicit-GEMM convolution engine (csrc/conv_tc.cu, C-ABI bts_conv_*).

Activations are NHWC in memory: torch tensors of logical shape (B,C,H,W) in `channels_last` format, so the same
tensor is understood by the rest of torch (cat, BatchNorm, autograd) without transposes.  Weights keep the
reference's (Cout,Cin,kh,kw) parameter layout (checkpoint wire format) and are re-packed into the engine's
pre-split, pre-swizzled tile stream whenever the parameter's version counter changes (i.e. once per optimizer step).

Numeric mode of the tensor-core engine (set_precision / BTS_B200_PRECISION): "fp32" (default) runs every GEMM as 3xTF32,
fp32-grade; "tf32" runs the single-pass TF32 kernels, one product per MMA.  Only the engine's forward, dgrad and wgrad
follow the mode; the CUDA-core kernels (narrow 1x1 and Cout = 1 heads, depthwise, BatchNorm, LPG, loss, optimizer) and
the library-conv fallback compute in fp32 either way, and their routing does not depend on it.
"""
import contextlib
import ctypes
import weakref

import torch

from . import _lib
from .ops import _need_cuda, _ptr, _stream

ACT = {None: 0, "none": 0, "elu": 1, "sigmoid": 2}
import os as _os

PW_FWD = _os.environ.get("BTS_B200_PW_FWD", "1") == "1"      # CUDA-core forward / dgrad for the same layers
PW_WGRAD = True                                               # CUDA-core wgrad for narrow 1x1 layers (csrc/pointwise.cu)
PW_MIN_PIXELS = 200000                                        # below this the tensor-core path is already short
TRACE = _os.environ.get("BTS_B200_TRACE", "0") == "1"     # per-call CUDA-event timing, aggregated by shape
trace_log = []
SPLITK = True                 # split-K forward launches inside inference(); tools and tests turn it off to compare
_inference_depth = 0
_splitk_plans = {}            # (device, launch geometry, requested splits) -> (splits, workspace floats)


@contextlib.contextmanager
def inference():
    """Scope in which no backward pass follows the forward launches: conv2d_tc may then cut a launch whose tiles fill at
    most half the SMs (batch-1 maps) into split-K ranges, whose partial sums a second kernel adds.  BtsModel.forward enters
    it under torch.no_grad() or when nothing requires grad; enter it directly when calling the engine below the model.
    Launches with epilogue statistics or BatchNorm-backward sums (training) never split, inside the scope or not."""
    global _inference_depth
    _inference_depth += 1
    try:
        yield
    finally:
        _inference_depth -= 1


def splitk_plan(B, Hout, Wout, kwin, Cin, KH, KW, Cout, splits=0):
    """(splits, workspace floats) of a forward / dgrad engine launch on the current device: splits = 0 asks for the engine's
    choice (1: no split), n > 0 forces n (reduced so that no split is empty)"""
    key = (torch.cuda.current_device(), B, Hout, Wout, kwin, Cin, KH, KW, Cout, splits)
    plan = _splitk_plans.get(key)
    if plan is None:
        n, wsf = ctypes.c_int(int(splits)), ctypes.c_longlong(0)
        _lib.check(_lib.lib().bts_conv_fwd_splitk_plan(B, Hout, Wout, kwin, Cin, KH, KW, Cout, ctypes.byref(n),
                                                        ctypes.byref(wsf)), "bts_conv_fwd_splitk_plan")
        plan = _splitk_plans[key] = (n.value, wsf.value)
    return plan


PRECISIONS = {"fp32": 0, "tf32": 1}       # mode -> the `precision` argument of the C ABI


def _check_mode(mode, what):
    if not isinstance(mode, str) or mode not in PRECISIONS:
        raise ValueError("%s: unknown precision mode %r (expected one of %s)" % (what, mode, ", ".join(sorted(PRECISIONS))))
    return mode


_precision = _check_mode(_os.environ.get("BTS_B200_PRECISION", "fp32"), "BTS_B200_PRECISION")


def set_precision(mode):
    """Selects the numeric mode of every later tensor-core engine launch -- forward, dgrad and wgrad of the whole model:
    "fp32" (the default: 3xTF32, fp32-grade) or "tf32" (single-pass TF32: faster, about 1e-3 relative per layer).
    Returns the previous mode, so that a caller can restore it.  The mode is read when a launch is enqueued: a captured
    CUDA graph (bts_b200.graph.GraphedTrainStep) keeps replaying the mode it was captured in."""
    global _precision
    prev, _precision = _precision, _check_mode(mode, "set_precision")
    return prev


def get_precision():
    return _precision


def _engine_precision(precision):
    """the C ABI's `precision` of an engine call: explicit 0 / 1, or None = the current mode"""
    return PRECISIONS[_precision] if precision is None else int(precision)


def set_trace(on):
    """bench.py / tools: CUDA events around every engine call (measurement only; never on in the timed region)"""
    global TRACE
    TRACE = bool(on)
    del trace_log[:]


SYNC_DEBUG = _os.environ.get("BTS_B200_SYNC", "0") == "1"    # bring-up: synchronize after every engine call, name the failing one


def _traced(kind, desc, fn, flops=0.0):
    if SYNC_DEBUG:
        out = fn()
        try:
            torch.cuda.synchronize()
        except Exception as e:
            print("BTS_B200_SYNC: engine call failed: %s %s (%s)" % (kind, desc, str(e).splitlines()[0]), flush=True)
            raise
        return out
    if not TRACE:
        return fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    out = fn()
    e1.record()
    trace_log.append((kind, desc, flops, e0, e1))
    return out


def trace_report():
    """[(total ms, calls, (kind, desc), total nominal FLOPs)] sorted by time"""
    torch.cuda.synchronize()
    agg = {}
    for kind, desc, flops, e0, e1 in trace_log:
        k = (kind, desc)
        t, n, f = agg.get(k, (0.0, 0, 0.0))
        agg[k] = (t + e0.elapsed_time(e1), n + 1, f + flops)
    return sorted(((t, n, k, f) for k, (t, n, f) in agg.items()), reverse=True)


if _os.environ.get("BTS_B200_W2_TMA") is not None:         # 0: narrow-output wgrad producers load from global memory
    _lib.lib().bts_wgrad2_set_tma(int(_os.environ["BTS_B200_W2_TMA"]))

_pack_cache = {}   # id(weight) -> (weakref, version, data_ptr, transpose) -> packed tensor


def invalidate_packed():
    """Drops every cached packed operator.  The cache is keyed on the parameter's version counter, which in-place writes
    through `.data` (apex / multi-tensor optimizers, manual EMA swaps, some checkpoint loaders) do not bump: call this
    after such a write (torch.optim.* and load_state_dict bump the counter and need nothing)."""
    _pack_cache.clear()


_multi_plan = None          # (signature, device descriptor table, total) of the last repack_cached()


def repack_cached():
    """Re-packs EVERY cached operator (forward and transposed, dense and grouped) in ONE launch and marks the cache
    entries current -- called by bts_b200.optim.FusedAdamW after its step, so the next forward pass finds every operator
    ready instead of issuing one pack launch per conv layer (394 per step for DenseNet-161 + decoder)."""
    global _multi_plan
    import numpy as np
    live = [(k, e) for k, e in _pack_cache.items() if e[0]() is not None]
    if not live:
        return 0
    L = _lib.lib()
    sig = tuple((k, e[0]().data_ptr(), e[3].data_ptr(), tuple(e[0]().stride())) for k, e in live)
    if _multi_plan is None or _multi_plan[0] != sig:
        dt = np.dtype([("w", "<u8"), ("wpack", "<u8"), ("s_co", "<i8"), ("s_ci", "<i8"), ("s_kh", "<i8"), ("s_kw", "<i8"),
                       ("start", "<i8"), ("Cout", "<i4"), ("Cin", "<i4"), ("KH", "<i4"), ("KW", "<i4"), ("tf", "<i4"),
                       ("n_tile", "<i4"), ("n_tiles", "<i4"), ("kwin", "<i4"), ("cpg", "<i4"), ("pad", "<i4")])
        assert dt.itemsize == 96
        tab = np.zeros(len(live), dtype=dt)
        start = 0
        for i, ((wid, tf), (ref, ver, ptr, packed, groups)) in enumerate(live):
            w = ref()
            Cout, Cin, KH, KW = w.shape
            st = w.stride()
            if groups > 1:
                kwin = group_window(Cout, Cin)
                n_tile = L.bts_conv_group_n_tile(kwin)
                n_tiles, cpg, ci_tot = Cout // n_tile, Cin, Cout
            else:
                rows = Cin if tf else Cout
                n_tile = L.bts_conv_n_tile(rows)
                n_tiles, kwin, cpg, ci_tot = (rows + n_tile - 1) // n_tile, 0, 1, Cin
            tab[i] = (w.data_ptr(), packed.data_ptr(), st[0], st[1], st[2], st[3], start, Cout, ci_tot, KH, KW, int(tf),
                      n_tile, n_tiles, kwin, cpg, 0)
            start += packed.numel() // 2
        dev = live[0][1][3].device
        _multi_plan = (sig, torch.from_numpy(tab.view(np.uint8)).to(dev), start, dev)
    _, table, total, dev = _multi_plan
    with torch.cuda.device(dev):
        _lib.check(L.bts_conv_pack_weights_multi(_ptr(table), len(live), total, _stream()), "bts_conv_pack_weights_multi")
    _lib.count()
    for k, (ref, ver, ptr, packed, groups) in live:
        w = ref()
        _pack_cache[k] = (ref, w._version, w.data_ptr(), packed, groups)
    return len(live)


def cached_operators(params):
    """the cache entries [(key, entry)] of the packed operators of `params` -- the buffers a CUDA graph captured over
    these parameters reads (bts_b200.graph.GraphedInference keeps them)"""
    ids = {id(p) for p in params}
    return [(k, e) for k, e in _pack_cache.items() if k[0] in ids and e[0]() is not None]


def restore_operators(entries):
    """Puts the packed operators `entries` (from cached_operators) back into the cache wherever a later pack_weights
    replaced them or invalidate_packed() dropped them, marked stale, so that the next repack_cached() rewrites those very
    buffers in place.  Returns True if any was put back.

    The cache is shared by eager forwards and captured graphs: a buffer that an eager pack_weights made after the weights
    changed is dropped here (freed once no pending work uses it), and eager forwards then read the graph's buffers, which
    repack_cached() keeps current.  repack_cached() rewrites every live cached operator, of every model, in its one
    launch -- not only the graph's."""
    put = False
    for k, (ref, ver, ptr, packed, groups) in entries:
        cur = _pack_cache.get(k)
        if cur is None or cur[3] is not packed:
            _pack_cache[k] = (ref, -1, ptr, packed, groups)
            put = True
    return put


def group_window(width, cpg):
    return _lib.lib().bts_conv_group_window(int(width), int(cpg))


def pack_weights(weight, transpose_flip=False, groups=1):
    """(Cout,Cin/groups,KH,KW) fp32 parameter -> packed operator.  Cached on the tensor's version counter."""
    _need_cuda(weight)
    key = (id(weight), bool(transpose_flip))
    ent = _pack_cache.get(key)
    w = weight.detach()
    if ent is not None:
        ref, ver, ptr, packed, _ = ent
        if ref() is weight and ver == weight._version and ptr == w.data_ptr():
            return packed
    Cout, Cin, KH, KW = w.shape
    rows, kch = (Cin, Cout) if transpose_flip else (Cout, Cin)
    L = _lib.lib()
    s = w.stride()
    if groups > 1:
        if not group_window(Cout, Cin):
            raise ValueError("grouped conv %s with %d groups is not supported by the block-diagonal engine path" % (tuple(w.shape), groups))
        packed = torch.empty(L.bts_conv_packed_floats_grouped(Cout, Cin, KH, KW), device=w.device, dtype=torch.float32)
        with torch.cuda.device(w.device):
            _lib.check(L.bts_conv_pack_weights_grouped(_ptr(w), s[0], s[1], s[2], s[3], Cout, Cin, KH, KW,
                                                       int(transpose_flip), _ptr(packed), _stream()),
                       "bts_conv_pack_weights_grouped")
    else:
        packed = torch.empty(L.bts_conv_packed_floats(rows, kch, KH, KW), device=w.device, dtype=torch.float32)
        with torch.cuda.device(w.device):
            _lib.check(L.bts_conv_pack_weights(_ptr(w), s[0], s[1], s[2], s[3], Cout, Cin, KH, KW, int(transpose_flip),
                                               _ptr(packed), _stream()), "bts_conv_pack_weights")
    _lib.count()
    _pack_cache[key] = (weakref.ref(weight), weight._version, w.data_ptr(), packed, int(groups))
    if len(_pack_cache) > 4096:
        for k in [k for k, v in _pack_cache.items() if v[0]() is None]:
            del _pack_cache[k]
    return packed


def _nhwc_view(x):
    """(ptr tensor, pixel stride) of a (B,C,H,W) tensor whose memory is NHWC (channels_last, possibly a channel
    slice of a wider slab).  Anything else is converted (one copy)."""
    B, C, H, W = x.shape
    sb, sc, sh, sw = x.stride()
    ok = (sc == 1 or C == 1) and sh == W * sw and sb == H * sh and sw >= C
    if not ok:
        x = x.contiguous(memory_format=torch.channels_last)
        sb, sc, sh, sw = x.stride()
        if C == 1:               # channels_last of a 1-channel tensor keeps NCHW strides; pixel stride is 1
            sw = 1
    return x, sw


def conv2d_tc(x, weight, stride=1, padding=0, dilation=1, pre_scale=None, pre_shift=None, pre_relu=False,
              upsample2=False, act=None, out=None, precision=None, packed=None, cout=None, transpose_flip=False,
              stats=None, groups=1, zero_stuff_out=None, bn_bwd=None, splits=None):
    """Runs the engine.  x: (B,Cin,Hs,Ws) NHWC-in-memory fp32 CUDA.  Returns (B,Cout,Hout,Wout) channels_last.
    `out` may be a pre-allocated channels_last tensor or a channel slice of one (concat-free writes).
    `stats`: a ZEROED fp64 [2, Cout] tensor that receives per-channel (sum, sum of squares) of the output, reduced in the
    conv epilogue (any Cout: the partials are flushed per n-tile) -- the BatchNorm batch statistics of the tensor being
    produced.
    `bn_bwd=(x_bn, st, relu)` (with a zeroed `stats`): the output is the gradient w.r.t. [relu](bn(x_bn)); the epilogue also
    reduces the BatchNorm-backward sums S1 = sum g*mask, S2 = sum g*mask*xhat into stats[0], stats[1] (st = [4,C] from
    bn_finalize) -- the separate reduce pass over (x, g) disappears.
    `groups` > 1: block-diagonal operator (ResNeXt 3x3).  `zero_stuff_out=(H,W)`: x is the gradient of a stride-2 layer
    whose input was HxW -- the source is read as its zero-stuffed x2 expansion (use with transpose_flip, stride 1).
    `precision`: None = the mode of set_precision, 0 = 3xTF32, 1 = single-pass TF32 on the engine (an explicit 1 also
    keeps the layer off the CUDA-core 1x1 kernel, which is fp32 in every mode).
    Inside `inference()` a launch without `stats` / `bn_bwd` runs split-K when the engine's plan says so.  `splits` (tests)
    forces a split count on the engine path: 1 never splits, n > 1 always does (and rejects `stats` / `bn_bwd`)."""
    _need_cuda(x, weight)
    if x.dtype != torch.float32:
        raise TypeError("conv2d_tc computes in fp32 (3xTF32 on wgmma); got %s" % x.dtype)
    x, xs = _nhwc_view(x)
    B, Cin, Hs, Ws = x.shape
    Co, Ci, KH, KW = weight.shape
    kwin = 0
    if groups > 1:
        kwin = group_window(Co, Ci)
        if not kwin:
            raise ValueError("unsupported grouped conv %s" % (tuple(weight.shape),))
        Ci = Co                              # block diagonal: both sides carry the full width
    elif transpose_flip:
        Co, Ci = Ci, Co
    if Ci != Cin:
        raise ValueError("weight expects %d input channels, got %d" % (Ci, Cin))
    if (PW_FWD and KH == 1 and KW == 1 and stride == 1 and padding == 0 and groups == 1 and not upsample2
            and zero_stuff_out is None and pre_scale is None and not pre_relu and stats is None and bn_bwd is None
            and precision in (None, 0) and packed is None and splits is None and act in ACT and B * Hs * Ws >= PW_MIN_PIXELS
            and xs % 4 == 0 and x.data_ptr() % 16 == 0 and _lib.lib().bts_conv_pw_fwd_eligible(Cin, Co)):
        # narrow 1x1 layers of the reduction heads (forward and dgrad): HBM-bound CUDA-core kernel (csrc/pointwise.cu)
        if out is None:
            out = torch.empty((B, Co, Hs, Ws), device=x.device, dtype=torch.float32, memory_format=torch.channels_last)
            os_ = Co
        else:
            if tuple(out.shape) != (B, Co, Hs, Ws):
                raise ValueError("out has shape %s, expected %s" % (tuple(out.shape), (B, Co, Hs, Ws)))
            o2, os_ = _nhwc_view(out)
            if o2 is not out:
                raise ValueError("out must be NHWC in memory")
        ws = weight.stride()
        s_out, s_in = (ws[1], ws[0]) if transpose_flip else (ws[0], ws[1])
        with torch.cuda.device(x.device):
            rc = _traced("pwdgrad" if transpose_flip else "pwfwd", "%dx%dx%d %d->%d k1" % (B, Hs, Ws, Cin, Co),
                         lambda: _lib.lib().bts_conv_pw_fwd(_ptr(x), xs, B * Hs * Ws, Cin, _ptr(weight), s_out, s_in, Co,
                                                            ACT[act], _ptr(out), os_, _stream()),
                         2.0 * B * Hs * Ws * Co * Cin)
        _lib.check(rc, "bts_conv_pw_fwd")
        _lib.count()
        return out
    precision = _engine_precision(precision)
    if packed is None:
        packed = pack_weights(weight, transpose_flip, groups)
    if zero_stuff_out is not None:
        mode = 2
        Hout, Wout = int(zero_stuff_out[0]), int(zero_stuff_out[1])
        if stride != 1 or upsample2:
            raise ValueError("zero_stuff_out needs stride 1 and no up-sample")
    else:
        mode = 1 if upsample2 else 0
        Hin, Win = (2 * Hs, 2 * Ws) if upsample2 else (Hs, Ws)
        Hout = (Hin + 2 * padding - dilation * (KH - 1) - 1) // stride + 1
        Wout = (Win + 2 * padding - dilation * (KW - 1) - 1) // stride + 1
    if out is None:
        out = torch.empty((B, Co, Hout, Wout), device=x.device, dtype=torch.float32,
                          memory_format=torch.channels_last)
        os_ = Co
    else:
        if tuple(out.shape) != (B, Co, Hout, Wout):
            raise ValueError("out has shape %s, expected %s" % (tuple(out.shape), (B, Co, Hout, Wout)))
        o2, os_ = _nhwc_view(out)
        if o2 is not out:
            raise ValueError("out must be NHWC in memory")
    if pre_scale is not None:
        pre_scale = pre_scale.contiguous()
        pre_shift = pre_shift.contiguous()
    if stats is not None and (stats.dtype != torch.float64 or tuple(stats.shape) != (2, Co) or not stats.is_contiguous()):
        raise ValueError("stats must be a contiguous fp64 [2, Cout] tensor")
    nsplit, ws = 1, None
    if splits is not None or (SPLITK and _inference_depth > 0 and stats is None and bn_bwd is None):
        if bn_bwd is not None and splits > 1:
            raise ValueError("split-K launches have no BatchNorm-backward epilogue")
        with torch.cuda.device(x.device):
            nsplit, wsf = splitk_plan(B, Hout, Wout, kwin, Cin, KH, KW, Co, 0 if splits is None else int(splits))
        if nsplit > 1:
            ws = torch.empty(wsf, device=x.device, dtype=torch.float32)
    xb = st = None
    xbs = relu = 0
    if bn_bwd is not None:
        xb, st, relu = bn_bwd
        xb, xbs = _nhwc_view(xb)
        if stats is None or act is not None or pre_scale is not None or pre_relu or tuple(xb.shape) != (B, Co, Hout, Wout) \
                or tuple(st.shape) != (4, Co) or not st.is_contiguous():
            raise ValueError("bn_bwd needs zeroed stats, no act / pre-op, x_bn shaped like the output and st = [4, Cout]")
    st0 = _ptr(stats[0]) if stats is not None else None
    st1 = _ptr(stats[1]) if stats is not None else None
    with torch.cuda.device(x.device):
        rc = _traced("dgrad" if transpose_flip else "fwd",
                     "%dx%dx%d %d->%d k%d d%d s%d%s%s%s%s" % (B, Hs, Ws, Cin, Co, KH, dilation, stride,
                                                             " up" if upsample2 else (" zs" if mode == 2 else ""),
                                                             " g%d" % groups if groups > 1 else "",
                                                             " sk%d" % nsplit if ws is not None else "",
                                                             " bnb" if bn_bwd is not None else ""),
                     lambda: _lib.lib().bts_conv_fwd(_ptr(x), xs, B, Hs, Ws, mode, Hout if mode == 2 else 0,
                                                     Wout if mode == 2 else 0, kwin, Cin, KH, KW, stride, padding, dilation,
                                                     _ptr(packed), Co, _ptr(pre_scale), _ptr(pre_shift), int(pre_relu),
                                                     _ptr(out), os_, ACT[act], int(precision), st0, st1, _ptr(xb), xbs,
                                                     _ptr(st), int(bool(relu)), nsplit, _ptr(ws), _stream()),
                     2.0 * B * Hout * Wout * Co * (Cin // groups) * KH * KW / (4.0 if mode == 2 else 1.0))
    _lib.check(rc, "bts_conv_fwd")
    _lib.count(2 if ws is not None else 1)
    return out


def wgrad_grouped_tc(x, gy, weight_shape, weight_strides, stride=1, padding=0, dilation=1, precision=None):
    """dW of a grouped (block-diagonal) 3x3 conv: weight (width, cpg, KH, KW).  precision: as conv2d_tc"""
    _need_cuda(x, gy)
    x, xs = _nhwc_view(x)
    gy, gs = _nhwc_view(gy)
    B, width, Hs, Ws = x.shape
    _, cpg, KH, KW = weight_shape
    L = _lib.lib()
    split = ctypes.c_int(0)
    wsf = ctypes.c_longlong(0)
    _lib.check(L.bts_conv_wgrad_grouped_plan(B, gy.shape[2], gy.shape[3], width, cpg, KH, KW, ctypes.byref(split),
                                             ctypes.byref(wsf)), "bts_conv_wgrad_grouped_plan")
    ws = torch.empty(wsf.value, device=x.device, dtype=torch.float32)
    gw = torch.empty_strided(tuple(weight_shape), tuple(weight_strides), device=x.device, dtype=torch.float32)
    s = weight_strides
    with torch.cuda.device(x.device):
        rc = _traced("wgrad", "%dx%dx%d %d->%d k%d d%d s%d g%d" % (B, Hs, Ws, width, width, KH, dilation, stride, width // cpg),
                     lambda: L.bts_conv_wgrad_grouped(_ptr(x), xs, B, Hs, Ws, width, cpg, KH, KW, stride, padding, dilation,
                                                      _ptr(gy), gs, _ptr(ws), split.value, _ptr(gw), s[0], s[1], s[2], s[3],
                                                      _engine_precision(precision), _stream()),
                     2.0 * B * gy.shape[2] * gy.shape[3] * width * cpg * KH * KW)
    _lib.check(rc, "bts_conv_wgrad_grouped")
    _lib.count(2)
    return gw


def wgrad_tc(x, gy, weight_shape, weight_strides, stride=1, padding=0, dilation=1, pre_scale=None, pre_shift=None,
             pre_relu=False, upsample2=False, precision=None):
    """dW (shaped/strided like the weight parameter) on the wgmma engine.  precision: as conv2d_tc"""
    _need_cuda(x, gy)
    x, xs = _nhwc_view(x)
    gy, gs = _nhwc_view(gy)
    B, Cin, Hs, Ws = x.shape
    Cout, _, KH, KW = weight_shape
    L = _lib.lib()
    if (PW_WGRAD and KH == 1 and KW == 1 and stride == 1 and padding == 0 and pre_scale is None and not pre_relu
            and not upsample2 and precision in (None, 0) and B * Hs * Ws >= PW_MIN_PIXELS and L.bts_conv_pw_wgrad_eligible(Cin, Cout)):
        # narrow 1x1 layers of the reduction heads: HBM-bound CUDA-core kernel (csrc/pointwise.cu)
        ws = torch.empty(L.bts_conv_pw_wgrad_workspace_floats(Cin, Cout), device=x.device, dtype=torch.float32)
        gw = torch.empty_strided(tuple(weight_shape), tuple(weight_strides), device=x.device, dtype=torch.float32)
        with torch.cuda.device(x.device):
            rc = _traced("pwwgrad", "%dx%dx%d %d->%d k1" % (B, Hs, Ws, Cin, Cout),
                         lambda: L.bts_conv_pw_wgrad(_ptr(x), xs, _ptr(gy), gs, B * Hs * Ws, Cin, Cout, _ptr(ws), _ptr(gw),
                                                     weight_strides[0], weight_strides[1], _stream()),
                         2.0 * B * Hs * Ws * Cout * Cin)
        _lib.check(rc, "bts_conv_pw_wgrad")
        _lib.count(2)
        return gw
    precision = _engine_precision(precision)
    split = ctypes.c_int(0)
    wsf = ctypes.c_longlong(0)
    _lib.check(L.bts_conv_wgrad_plan(B, gy.shape[2], gy.shape[3], Cin, Cout, KH, KW, stride, ctypes.byref(split), ctypes.byref(wsf)),
               "bts_conv_wgrad_plan")
    ws = torch.empty(wsf.value, device=x.device, dtype=torch.float32)
    gw = torch.empty_strided(tuple(weight_shape), tuple(weight_strides), device=x.device, dtype=torch.float32)
    s = weight_strides
    if pre_scale is not None:
        pre_scale, pre_shift = pre_scale.contiguous(), pre_shift.contiguous()
    with torch.cuda.device(x.device):
        rc = _traced("wgrad", "%dx%dx%d %d->%d k%d d%d s%d%s" % (B, Hs, Ws, Cin, Cout, KH, dilation, stride,
                                                                  " up" if upsample2 else ""),
                     lambda: L.bts_conv_wgrad(_ptr(x), xs, B, Hs, Ws, int(upsample2), Cin, KH, KW, stride, padding,
                                              dilation, _ptr(pre_scale), _ptr(pre_shift), int(pre_relu), _ptr(gy), gs,
                                              Cout, _ptr(ws), split.value, _ptr(gw), s[0], s[1], s[2], s[3],
                                              int(precision), _stream()),
                     2.0 * B * gy.shape[2] * gy.shape[3] * Cout * Cin * KH * KW)
    _lib.check(rc, "bts_conv_wgrad")
    _lib.count(2)
    return gw


class _ConvTC(torch.autograd.Function):
    """Plain convolution (no fused pre/post ops) with autograd, all three GEMMs on the wgmma engine: forward,
    dgrad (the same kernel over the transposed, tap-flipped packed operator; a stride-2 layer's dgrad reads dY as its
    zero-stuffed expansion) and wgrad (operands transposed to K-major on their way into shared memory).  groups > 1: block-diagonal operator (ResNeXt)."""

    @staticmethod
    def forward(ctx, x, weight, stride, padding, dilation, groups):
        y = conv2d_tc(x, weight, stride, padding, dilation, groups=groups)
        ctx.save_for_backward(x, weight)
        ctx.cfg = (stride, padding, dilation, groups)
        return y

    @staticmethod
    def backward(ctx, gy):
        x, weight = ctx.saved_tensors
        stride, padding, dilation, groups = ctx.cfg
        gx = gw = None
        KH = weight.shape[2]
        if ctx.needs_input_grad[0]:
            padT = dilation * (KH - 1) - padding
            if stride == 1:
                gx = conv2d_tc(gy, weight, 1, padT, dilation, transpose_flip=True, groups=groups)
            elif stride == 2 and padT >= 0:
                gx = conv2d_tc(gy, weight, 1, padT, dilation, transpose_flip=True, groups=groups,
                               zero_stuff_out=(x.shape[2], x.shape[3]))
            else:
                raise NotImplementedError("conv dgrad on the engine: stride %d / padding %d not covered (BTS encoders use "
                                          "stride 1 and 2 only)" % (stride, padding))
        if ctx.needs_input_grad[1]:
            if groups > 1:
                gw = wgrad_grouped_tc(x, gy, weight.shape, weight.stride(), stride, padding, dilation)
            else:
                gw = wgrad_tc(x, gy, weight.shape, weight.stride(), stride, padding, dilation)
        return gx, gw, None, None, None, None


def conv2d(x, weight, stride=1, padding=0, dilation=1, groups=1):
    return _ConvTC.apply(x, weight, stride, padding, dilation, groups)


# ---------------------------------------------------------------------------- single-output-channel heads
C1_CHANNELS = (8, 16, 32, 64, 128)


def c1_eligible(weight, stride, padding, dilation):
    co, ci, kh, kw = weight.shape
    return (co == 1 and kh == kw and kh in (1, 3) and stride == 1 and dilation == 1 and padding == kh // 2
            and ci in C1_CHANNELS)


class _ConvC1(torch.autograd.Function):
    """Cout = 1 convolution (+ optional fused sigmoid) on the HBM-bound CUDA-core kernels (csrc/thin.cu)."""

    @staticmethod
    def forward(ctx, x, weight, sigmoid):
        _need_cuda(x, weight)
        x, xs = _nhwc_view(x)
        if xs % 4 != 0 or x.data_ptr() % 16 != 0:
            x = x.contiguous(memory_format=torch.channels_last)
            xs = x.shape[1]
        B, C, H, W = x.shape
        K = weight.shape[2]
        y = torch.empty((B, 1, H, W), device=x.device, dtype=torch.float32)
        s = weight.stride()
        with torch.cuda.device(x.device):
            rc = _traced("c1fwd", "%dx%dx%d %d->1 k%d" % (B, H, W, C, K),
                         lambda: _lib.lib().bts_conv_c1_fwd(_ptr(x), xs, B, H, W, C, K, _ptr(weight), s[1], s[2], s[3],
                                                            2 if sigmoid else 0, _ptr(y), _stream()))
        _lib.check(rc, "bts_conv_c1_fwd")
        _lib.count()
        ctx.save_for_backward(x, weight, y if sigmoid else None)
        ctx.xs = xs
        return y

    @staticmethod
    def backward(ctx, gy):
        x, weight, sig = ctx.saved_tensors
        B, C, H, W = x.shape
        K = weight.shape[2]
        gy = gy.contiguous()
        s = weight.stride()
        L = _lib.lib()
        gx = gw = None
        with torch.cuda.device(x.device):
            if ctx.needs_input_grad[0]:
                gx = torch.empty((B, C, H, W), device=x.device, dtype=torch.float32, memory_format=torch.channels_last)
                rc = _traced("c1dgrad", "%dx%dx%d 1->%d k%d" % (B, H, W, C, K),
                             lambda: L.bts_conv_c1_dgrad(_ptr(gy), _ptr(sig), B, H, W, C, K, _ptr(weight), s[1], s[2], s[3],
                                                         _ptr(gx), C, _stream()))
                _lib.check(rc, "bts_conv_c1_dgrad")
                _lib.count()
            if ctx.needs_input_grad[1]:
                ws = torch.empty(L.bts_conv_c1_workspace_floats(C, K), device=x.device, dtype=torch.float32)
                gw = torch.empty_strided(tuple(weight.shape), tuple(s), device=x.device, dtype=torch.float32)
                rc = _traced("c1wgrad", "%dx%dx%d %d->1 k%d" % (B, H, W, C, K),
                             lambda: L.bts_conv_c1_wgrad(_ptr(x), ctx.xs, _ptr(gy), _ptr(sig), B, H, W, C, K, _ptr(ws),
                                                         _ptr(gw), s[1], s[2], s[3], _stream()))
                _lib.check(rc, "bts_conv_c1_wgrad")
                _lib.count(2)
        return gx, gw, None


def conv_c1(x, weight, sigmoid=False):
    return _ConvC1.apply(x, weight, bool(sigmoid))
