"""Batch-1 eval forward throughput (bts_test.py / online eval) with split-K engine launches on and off, eager and as a
captured CUDA graph (bts_b200.graph.GraphedInference).

  python tools/infer_step.py [--shapes T1,NYU,KITTI] [--steps 30] [--warmup 5] [--rounds 3] [--kernels]

Shapes: T1 = DenseNet-121 at 416 x 544 (bench.py --config T1), NYU = DenseNet-161 at 480 x 640 (NYU test split), KITTI =
DenseNet-161 at 352 x 1216 (the KB crop of the KITTI test split); random-init weights, a seeded input.  Split-K is switched
through conv.SPLITK in this one process (one graph is captured per setting); the four variants (split-K on / off, eager /
graphed) alternate over --rounds rounds, each round times --steps forwards after --warmup with CUDA events around the loop
(one synchronize at its end), and the reported img/s is the median round.  Native launches per forward come from
bts_b200._lib.launches.  The final depth maps with split-K on and off must agree at the model bar (1e-3 of the map's
largest value) and each graph's outputs must equal the eager ones bit for bit.  --kernels adds a separate profiled eager
forward per setting (torch.profiler, CUDA activity): the summed duration of every kernel (the GPU's busy time per forward,
against which the eager and graphed times show the host's share), of the engine's conv_tc_kernel / conv_tf32_kernel and
of conv_splitk_reduce_kernel.  The card's name, power limit and max SM clock are read in the same run.  One JSON line per
result."""
import argparse
import json
import os
import subprocess
import sys
import types

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SHAPES = {"T1": ("densenet121_bts", 416, 544, "nyu", 10.0, 518.8579),
          "NYU": ("densenet161_bts", 480, 640, "nyu", 10.0, 518.8579),
          "KITTI": ("densenet161_bts", 352, 1216, "kitti", 80.0, 721.5377)}


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clk = [s.strip() for s in out.split(",")]
        return {"gpu": name, "power_limit": power, "max_sm_clock": clk}
    except Exception as e:                       # the numbers are still printed, the card is reported unknown
        return {"gpu": "unknown (%s)" % type(e).__name__}


def median(xs):
    xs = sorted(xs)
    return xs[len(xs) // 2] if len(xs) % 2 else 0.5 * (xs[len(xs) // 2 - 1] + xs[len(xs) // 2])


def build(torch, shape):
    import bts
    enc, H, W, dataset, md, focal = SHAPES[shape]
    torch.manual_seed(0)
    p = types.SimpleNamespace(encoder=enc, max_depth=md, dataset=dataset, bts_size=512, pretrained=False)
    m = bts.BtsModel(p)
    m.decoder.apply(bts.weights_init_xavier)
    m.cuda().eval()
    g = torch.Generator().manual_seed(1)
    x = torch.randn(1, 3, H, W, generator=g).cuda()
    f = torch.full((1,), focal).cuda()
    return m, x, f


def timed(torch, fn, steps, warmup):
    for _ in range(warmup):
        fn()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    for _ in range(steps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / steps


def measure(torch, shape, args):
    from bts_b200 import _lib, conv
    from bts_b200.graph import GraphedInference
    m, x, f = build(torch, shape)
    res = {}
    for on in (True, False):
        conv.SPLITK = on
        with torch.no_grad():
            m(x, f)
            torch.cuda.synchronize()
            l0 = _lib.launches
            eager_out = [t.clone() for t in m(x, f)]
            launches = _lib.launches - l0
        gi = GraphedInference(m, x, f)            # captures the current setting
        same = all(torch.equal(a, b) for a, b in zip(eager_out, gi(x, f)))
        res[on] = dict(gi=gi, depth=eager_out[4], launches=launches, same=same, eager_ms=[], graph_ms=[])
    for r in range(args.rounds):
        for on in ((True, False) if r % 2 == 0 else (False, True)):
            conv.SPLITK = on
            gi = res[on]["gi"]
            with torch.no_grad():
                res[on]["eager_ms"].append(timed(torch, lambda: m(x, f), args.steps, args.warmup))
            res[on]["graph_ms"].append(timed(torch, lambda: gi(x, f), args.steps, args.warmup))
    conv.SPLITK = True
    d_on, d_off = res[True]["depth"].double(), res[False]["depth"].double()
    depth_rel = float((d_on - d_off).abs().max() / d_off.abs().max())
    out = []
    for on in (True, False):
        r = res[on]
        e, g = median(r["eager_ms"]), median(r["graph_ms"])
        out.append({"what": "batch-1 eval forward", "shape": shape, "encoder": SHAPES[shape][0],
                    "HxW": "%dx%d" % SHAPES[shape][1:3], "splitk": on, "native_launches_per_forward": r["launches"],
                    "graph_launches_per_replay": r["gi"].launches_per_replay,
                    "eager_ms": round(e, 3), "eager_img_per_s": round(1000.0 / e, 2),
                    "eager_ms_rounds": [round(t, 3) for t in r["eager_ms"]],
                    "graph_ms": round(g, 3), "graph_img_per_s": round(1000.0 / g, 2),
                    "graph_ms_rounds": [round(t, 3) for t in r["graph_ms"]],
                    "graph_equals_eager": r["same"], "depth_rel_diff_splitk_on_off": depth_rel,
                    "depth_within_1e-3": depth_rel < 1e-3})
    if args.kernels:
        for on in (True, False):
            conv.SPLITK = on
            out.append(kernel_times(torch, shape, m, x, f, on))
        conv.SPLITK = True
    return out


def kernel_times(torch, shape, m, x, f, on):
    from torch.profiler import ProfilerActivity, profile
    with torch.no_grad():
        m(x, f)
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            m(x, f)
            torch.cuda.synchronize()
    t = {"all": [0.0, 0], "conv": [0.0, 0], "reduce": [0.0, 0]}
    for e in prof.events():
        if e.device_type != torch.autograd.DeviceType.CUDA:
            continue
        d = (e.time_range.end - e.time_range.start) / 1000.0
        keys = ["all"]
        if "conv_tc_kernel" in e.name or "conv_tf32_kernel" in e.name:
            keys.append("conv")
        elif "conv_splitk_reduce_kernel" in e.name:
            keys.append("reduce")
        for k in keys:
            t[k][0] += d
            t[k][1] += 1
    return {"what": "kernel time per batch-1 eval forward (profiled, eager)", "shape": shape, "splitk": on,
            "all_kernels_ms": round(t["all"][0], 3), "kernels": t["all"][1],
            "conv_engine_ms": round(t["conv"][0], 3), "conv_engine_launches": t["conv"][1],
            "reduce_ms": round(t["reduce"][0], 3), "reduce_launches": t["reduce"][1]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", default="T1,NYU,KITTI")
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--kernels", action="store_true")
    args = ap.parse_args()
    shapes = args.shapes.split(",")
    for s in shapes:
        if s not in SHAPES:
            ap.error("unknown shape %r (expected %s)" % (s, ", ".join(SHAPES)))
    sys.path.insert(0, ROOT)
    os.environ.setdefault("BTS_B200_PRETRAINED", "0")
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("infer_step.py measures on a GPU; none is visible")
    info = card()
    for s in shapes:
        for r in measure(torch, s, args):
            r.update(info)
            print(json.dumps(r), flush=True)


if __name__ == "__main__":
    main()
