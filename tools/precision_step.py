"""Time the K16 training step in both numeric modes of the tensor-core engine: fp32 (3xTF32, the default) and tf32
(single-pass TF32, bts_b200.set_precision("tf32")).

  python tools/precision_step.py [--rounds 3] [--steps 10] [--warmup 3] [--kernels]

The step is bench.py's K16 step: DenseNet-161, 352x704 KITTI, batch 16, random-init weights, frozen like
bench.freeze_like_set_misc, GraphedTrainStep (forward + silog + backward in one CUDA graph) + FusedAdamW.  One graph is
captured per mode (each replays the mode it was captured in), both on the same model, and the modes alternate in one
process: --rounds rounds of --steps steps per mode after --warmup steps, each step timed with CUDA events.  Printed per
mode: the median ms/step and img/s over every timed step.  --kernels adds a separate profiled run: one eager training step
per mode under torch.profiler (CUDA activity), with the time of each tensor-core kernel family (conv_*: forward and dgrad,
wgrad_*: tap-in-grid weight gradient, wgrad2_*: shifted-dY weight gradient).  The card's name, power limit and maximum SM
clock are read in the same run (nvidia-smi --query-gpu, read only).  One JSON line per result.
"""
import argparse
import json
import os
import re
import subprocess
import sys
import types

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FAMILIES = (("wgrad2", r"wgrad2_(tc|tf32)_kernel"), ("wgrad", r"wgrad_(tc|tf32)_kernel"), ("conv", r"conv_(tc|tf32)_kernel"))


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


def setup(torch):
    import bench
    import bts
    cfg = bench.CONFIGS["K16"]
    dev = torch.device("cuda", 0)
    torch.manual_seed(0)
    p = types.SimpleNamespace(encoder=cfg["encoder"], max_depth=cfg["max_depth"], dataset=cfg["dataset"], bts_size=512,
                              pretrained=False)
    model = bts.BtsModel(p).train()
    model.decoder.apply(bts.weights_init_xavier)
    bench.freeze_like_set_misc(model)
    model.to(dev)
    crit = bts.silog_loss(0.85)
    img, focal, gt = bench.synth_batch(cfg, cfg["B"], 1, dev)
    loss_fn = lambda out, g: crit(out[4], g, g > cfg["thr"])
    return cfg, model, loss_fn, (img, focal), (gt,)


def step_times(torch, rounds, steps, warmup):
    import bench
    import bts_b200
    from bts_b200.graph import GraphedTrainStep
    cfg, model, loss_fn, inputs, targets = setup(torch)
    opt = bench.make_optimizer(model, torch, fused=True)
    graphs = {}
    for mode in ("fp32", "tf32"):
        prev = bts_b200.set_precision(mode)
        try:
            graphs[mode] = GraphedTrainStep(model, loss_fn, (inputs, targets))
        finally:
            bts_b200.set_precision(prev)
    times = {"fp32": [], "tf32": []}
    losses = {}

    def run(mode, n, keep):
        for _ in range(n):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            loss = graphs[mode](inputs, targets)
            opt.step()
            b.record()
            torch.cuda.synchronize()
            if keep:
                times[mode].append(a.elapsed_time(b))
            losses[mode] = float(loss)

    for mode in ("fp32", "tf32"):
        run(mode, warmup, False)
    for _ in range(rounds):
        for mode in ("fp32", "tf32"):
            run(mode, steps, True)
    out = {}
    for mode in ("fp32", "tf32"):
        ms = median(times[mode])
        out[mode] = {"ms_per_step": round(ms, 2), "img_per_s": round(cfg["B"] * 1000.0 / ms, 1),
                     "min_ms": round(min(times[mode]), 2), "max_ms": round(max(times[mode]), 2),
                     "steps": len(times[mode]), "last_loss": losses[mode]}
    return out


def kernel_times(torch):
    import bts_b200
    cfg, model, loss_fn, inputs, targets = setup(torch)
    out = {}
    for mode in ("fp32", "tf32", "fp32", "tf32"):         # the first pass of each mode warms up; the second is kept
        prev = bts_b200.set_precision(mode)
        try:
            model.zero_grad(set_to_none=True)
            torch.cuda.synchronize()
            with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
                loss_fn(model(*inputs), *targets).backward()
                torch.cuda.synchronize()
        finally:
            bts_b200.set_precision(prev)
        fam = {name: [0.0, 0] for name, _ in FAMILIES}
        for e in prof.events():
            if e.device_type != torch.autograd.DeviceType.CUDA:
                continue
            for name, pat in FAMILIES:
                if re.search(pat, e.name):
                    fam[name][0] += e.device_time_total / 1000.0
                    fam[name][1] += 1
                    break
        out[mode] = {name: {"ms": round(t, 2), "launches": n} for name, (t, n) in fam.items()}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--kernels", action="store_true", help="also a profiled eager step per mode: time per kernel family")
    args = ap.parse_args()
    sys.path.insert(0, ROOT)
    import torch
    if not torch.cuda.is_available():
        sys.exit("tools/precision_step.py measures on a CUDA device; none is available")
    info = card()
    res = step_times(torch, args.rounds, args.steps, args.warmup)
    res["tf32_speedup"] = round(res["fp32"]["ms_per_step"] / res["tf32"]["ms_per_step"], 3)
    print(json.dumps(dict(info, metric="K16 step (graph + FusedAdamW), median over alternating rounds", **res)), flush=True)
    if args.kernels:
        print(json.dumps(dict(info, metric="K16 eager step, tensor-core kernel time per family (torch.profiler)",
                              **kernel_times(torch))), flush=True)


if __name__ == "__main__":
    main()
