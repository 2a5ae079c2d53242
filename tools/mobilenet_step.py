"""Time the MobileNetV2 training step at the K16 shape (352x704 KITTI, batch 16) and the depthwise kernels inside it.

  python tools/mobilenet_step.py [--root TREE] [--steps 10] [--warmup 3] [--kernels]

The step is bench.py's: GraphedTrainStep (forward + silog + backward in one CUDA graph) + FusedAdamW, random-init weights,
bench.py's synthetic KITTI batch.  Step time = median over --steps steps of CUDA events after --warmup steps.  --root runs
the same measurement against another checkout of the project (for example the parent commit), whose `bts` and bench.py are
imported instead of this tree's.  --kernels adds a separate profiled run: one eager training step of the same model under
torch.profiler (CUDA activity), from which each depthwise layer's forward (BN1 + ReLU6 prologue, BN2 statistics and their
second pass), dgrad and wgrad (with its second pass) kernel time is read, with its achieved bandwidth from the algorithmic
bytes 4*C*(B*H*W + B*Ho*Wo) (each pass reads one tensor and reads or writes the other once).  The card's name and
power limit are read in the same run and printed with the numbers.  One JSON line per result.
"""
import argparse
import json
import os
import subprocess
import sys
import types

HBM_TBS = 3.35          # H100 SXM data sheet, HBM3


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


def step_time(torch, root, steps, warmup):
    import bench
    import bts
    from bts_b200.graph import GraphedTrainStep
    cfg = dict(bench.CONFIGS["K16"], encoder="mobilenetv2_bts")
    dev = torch.device("cuda", 0)
    torch.manual_seed(0)
    p = types.SimpleNamespace(encoder=cfg["encoder"], max_depth=cfg["max_depth"], dataset=cfg["dataset"], bts_size=512,
                              pretrained=False)
    model = bts.BtsModel(p).train()
    model.decoder.apply(bts.weights_init_xavier)
    bench.freeze_like_set_misc(model)
    model.to(dev)
    opt = bench.make_optimizer(model, torch, fused=True)
    crit = bts.silog_loss(0.85)
    img, focal, gt = bench.synth_batch(cfg, cfg["B"], 1, dev)
    graphed = GraphedTrainStep(model, lambda out, g: crit(out[4], g, g > cfg["thr"]), ((img, focal), (gt,)))
    times = []
    for i in range(warmup + steps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        loss = graphed((img, focal), (gt,))
        opt.step()
        b.record()
        torch.cuda.synchronize()
        if i >= warmup:
            times.append(a.elapsed_time(b))
    ms = median(times)
    r = {"what": "mobilenetv2_bts K16-shape train step (graph + FusedAdamW)", "root": root, "B": cfg["B"],
         "median_ms": round(ms, 3), "img_per_s": round(cfg["B"] * 1000.0 / ms, 2),
         "spread_ms": [round(min(times), 3), round(max(times), 3)], "loss": float(loss)}
    return r, model, (lambda out, g: crit(out[4], g, g > cfg["thr"])), (img, focal, gt)


def depthwise_layers(B=16, H=352, W=704):
    """(C, H, W, stride) of the 17 depthwise layers of mobilenet_v2().features at the input size"""
    import torchvision
    f = torchvision.models.mobilenet_v2().features
    h, w = (H - 1) // 2 + 1, (W - 1) // 2 + 1          # after the 3x3/2 stem
    out = []
    for blk in list(f)[1:18]:
        dw = blk.conv[-3][0]
        s = dw.stride[0]
        out.append((dw.in_channels, h, w, s))
        h, w = (h - 1) // s + 1, (w - 1) // s + 1
    return out


def kernel_times(torch, model, loss_fn, batch, B=16):
    """Depthwise kernel durations from torch.profiler CUDA activity over one eager training step of the timed model (a
    separate run: the step timing above is taken without the profiler).  In launch order the step runs, per layer, the
    forward (fwd kernel + statistics pass) from features.1 to features.17, then per layer from features.17 down to
    features.1 the wgrad (kernel + fixed-order sum) and the dgrad (the forward kernel over flipped taps at stride 1, the
    gather kernel at stride 2)."""
    from torch.profiler import ProfilerActivity, profile
    img, focal, gt = batch
    for _ in range(2):                                  # eager warm-up: allocator, packed operators
        model.zero_grad(set_to_none=True)
        loss_fn(model(img, focal), gt).backward()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        model.zero_grad(set_to_none=True)
        loss_fn(model(img, focal), gt).backward()
        torch.cuda.synchronize()
    ev = sorted((e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA
                 and ("dw3x3_" in e.name or "dw_colsum" in e.name)), key=lambda e: e.time_range.start)
    dur = [(e.name, e.time_range.end - e.time_range.start) for e in ev]
    layers = depthwise_layers(B)
    n = len(layers)
    if len(dur) != 5 * n:
        raise SystemExit("expected %d depthwise kernels in the step, profiled %d" % (5 * n, len(dur)))
    t = {}
    for i in range(n):                                  # forward, features.1 .. features.17
        (k0, d0), (k1, d1) = dur[2 * i], dur[2 * i + 1]
        assert "dw3x3_fwd_kernel" in k0 and "dw_colsum_kernel<0>" in k1, (k0, k1)
        t[(i, "fwd")] = d0 + d1
    for j in range(n):                                  # backward, features.17 .. features.1
        i = n - 1 - j
        (k0, d0), (k1, d1), (k2, d2) = dur[2 * n + 3 * j: 2 * n + 3 * j + 3]
        assert "dw3x3_wgrad_kernel" in k0 and "dw_colsum_kernel<1>" in k1 and ("dw3x3_fwd_kernel<1, false>" in k2 or
                                                                               "dw3x3_dgrad_s2_kernel" in k2), (k0, k1, k2)
        t[(i, "wgrad")] = d0 + d1
        t[(i, "dgrad")] = d2
    res = []
    for i, (C, H, W, s) in enumerate(layers):
        Ho, Wo = (H - 1) // s + 1, (W - 1) // s + 1
        nbytes = 4.0 * C * (B * H * W + B * Ho * Wo)
        for name in ("fwd", "dgrad", "wgrad"):
            us = t[(i, name)]
            gbs = nbytes / us / 1e3
            res.append({"layer": "features.%d" % (i + 1), "pass": name, "C": C, "in": [H, W], "stride": s,
                        "us": round(us, 1), "GB_s": round(gbs, 1), "hbm_share": round(gbs / (HBM_TBS * 1e3), 3)})
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--root", default=os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--kernels", action="store_true")
    args = ap.parse_args()
    root = os.path.abspath(args.root)
    sys.path.insert(0, root)
    os.environ.setdefault("BTS_B200_PRETRAINED", "0")
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("mobilenet_step.py measures on a GPU; none is visible")
    info = card()
    r, model, loss_fn, batch = step_time(torch, root, args.steps, args.warmup)
    r.update(info)
    print(json.dumps(r), flush=True)
    if args.kernels:
        for k in kernel_times(torch, model, loss_fn, batch):
            k.update(info)
            print(json.dumps(k), flush=True)


if __name__ == "__main__":
    main()
