"""Measures the batched PNG decoder (ops.decode_png; csrc/png.cu) against Pillow on one host thread.

Inputs are seeded KITTI-like frames, encoded by Pillow at its defaults: a 375x1242 RGB frame (a smooth field plus noise)
and a sparse 16-bit depth frame of the same size.  The compression ratio is reported, since the decode rate depends on the
content.  Results:
  pillow     decode + the KB fixed crop per sample, one host thread
  kernel     png_inflate_kernel and png_unfilter_kernel alone, CUDA events over many launches, B = 4, 16, 64
  e2e        ops.decode_png wall time (parse + CRC, H2D, both kernels, status read), B = 4, 16, 64
  overlap    the K16 GraphedTrainStep step time alone and with the next batch's 16 RGB + 16 depth PNGs decoded on a side
             stream during each step, alternated in one process
The card's name and power limit are read in the same run.  One JSON line per result.

    python tools/png_decode.py [--iters 20] [--steps 20]
"""
import argparse
import io
import json
import os
import subprocess
import sys
import time
import types

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

H, W = 375, 1242


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


def frames(n):
    """n seeded (rgb, depth) PNG pairs, Pillow defaults"""
    import numpy as np
    from PIL import Image
    out = []
    yy, xx = np.mgrid[0:H, 0:W]
    for i in range(n):
        rng = np.random.RandomState(i)
        field = 128 + 60 * np.sin(yy / (40.0 + i) + i)[..., None] + 50 * np.cos(xx / (90.0 + i))[..., None]
        img = np.clip(field + rng.normal(0, 6, (H, W, 3)), 0, 255).astype(np.uint8)
        dep = ((yy * 40 + xx * 3 + 2000) * (rng.uniform(size=(H, W)) < 0.05)).astype(np.uint16)
        pair = []
        for a in (img, dep):
            buf = io.BytesIO()
            Image.fromarray(a).save(buf, format="PNG")
            pair.append(buf.getvalue())
        out.append(tuple(pair))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--steps", type=int, default=20)
    a = ap.parse_args()
    import numpy as np
    import torch
    from PIL import Image
    from bts_b200 import _lib, data, ops

    info = card()
    pairs = frames(64)
    box = data.fixed_crop_box("kitti", True, H, W)
    for k, name, bpp in ((0, "rgb8", 3), (1, "gray16", 2)):
        raw = H * (1 + W * bpp)
        comp = float(np.mean([len(p[k]) for p in pairs]))
        t = []
        for p in pairs[:16]:
            t0 = time.perf_counter()
            data.fixed_crop(np.asarray(Image.open(io.BytesIO(p[k]))), "kitti", True)
            t.append(time.perf_counter() - t0)
        print(json.dumps(dict(info, what="pillow decode + KB crop, one host thread", format=name, frame=[H, W],
                              compression_ratio=round(raw / comp, 2), png_bytes=int(comp), ms_per_sample=round(median(t) * 1e3, 3))),
              flush=True)

    dev = torch.device("cuda", 0)
    L = _lib.lib()
    for k, name, bpp in ((0, "rgb8", 3), (1, "gray16", 2)):
        for B in (4, 16, 64):
            blobs = [p[k] for p in pairs[:B]]
            parsed = [data.parse_png(b) for b in blobs]
            streams = b"".join(p[4] for p in parsed)
            meta = np.zeros((B, 8), np.int64)
            so = ro = 0
            for i, p in enumerate(parsed):
                meta[i] = (so, len(p[4]), ro, H, W, box[0], box[1], 0)
                so += len(p[4])
                ro += H * (1 + W * bpp)
            src = torch.frombuffer(bytearray(streams), dtype=torch.uint8).to(dev)
            meta_d = torch.from_numpy(meta).to(dev)
            rawb = torch.empty(ro, dtype=torch.uint8, device=dev)
            work = torch.empty(2 * B, dtype=torch.int32, device=dev)
            out = torch.empty(B * box[2] * box[3] * bpp, dtype=torch.uint8, device=dev)
            st = torch.cuda.current_stream().cuda_stream

            def inflate():
                _lib.check(L.bts_png_inflate(src.data_ptr(), meta_d.data_ptr(), B, bpp, rawb.data_ptr(),
                                             work[B:].data_ptr(), work[:B].data_ptr(), st), "inflate")

            def unfilter():
                _lib.check(L.bts_png_unfilter(rawb.data_ptr(), meta_d.data_ptr(), work[B:].data_ptr(), B, bpp, box[2],
                                              box[3], out.data_ptr(), work[:B].data_ptr(), st), "unfilter")

            inflate()
            unfilter()
            torch.cuda.synchronize()
            assert int(work[:B].abs().sum()) == 0
            times = {}
            for kname, fn in (("png_inflate_kernel", inflate), ("png_unfilter_kernel", unfilter)):
                ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
                ev[0].record()
                for _ in range(a.iters):
                    fn()
                ev[1].record()
                torch.cuda.synchronize()
                times[kname] = ev[0].elapsed_time(ev[1]) / a.iters
            e2e = []
            for _ in range(a.iters):
                t0 = time.perf_counter()
                ops.decode_png(blobs, [box[:2]] * B, box[2:])
                e2e.append(time.perf_counter() - t0)
            ms = median(e2e) * 1e3
            out_mb = B * box[2] * box[3] * bpp / 1e6
            print(json.dumps(dict(info, what="decode_png", format=name, B=B,
                                  inflate_ms=round(times["png_inflate_kernel"], 3),
                                  unfilter_ms=round(times["png_unfilter_kernel"], 3), e2e_ms=round(ms, 3),
                                  e2e_img_per_s=round(B * 1e3 / ms, 1), e2e_out_MB_per_s=round(out_mb * 1e3 / ms, 1),
                                  kernels_img_per_s=round(B * 1e3 / (times["png_inflate_kernel"] + times["png_unfilter_kernel"]), 1))),
                  flush=True)

    # interference with training: K16 step alone vs with the next batch decoded on a side stream
    import bench
    import bts
    from bts_b200.graph import GraphedTrainStep
    cfg = bench.CONFIGS["K16"]
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
    side = torch.cuda.Stream()
    rgb, dep = [q[0] for q in pairs[:16]], [q[1] for q in pairs[:16]]
    res = {"alone": [], "with_decode": []}
    for i in range(3 + 2 * a.steps):
        mode = "alone" if i % 2 == 0 else "with_decode"
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
        ev[0].record()
        graphed((img, focal), (gt,))
        opt.step()
        ev[1].record()
        if mode == "with_decode":
            with torch.cuda.stream(side):
                ops.decode_png(rgb, [box[:2]] * 16, box[2:])
                ops.decode_png(dep, [box[:2]] * 16, box[2:])
        torch.cuda.synchronize()
        if i >= 3:
            res[mode].append(ev[0].elapsed_time(ev[1]))
    print(json.dumps(dict(info, what="K16 train step with the next batch decoded on a side stream", encoder=cfg["encoder"],
                          B=cfg["B"], alone_ms=round(median(res["alone"]), 3),
                          with_decode_ms=round(median(res["with_decode"]), 3), steps_each=len(res["alone"]))), flush=True)


if __name__ == "__main__":
    main()
