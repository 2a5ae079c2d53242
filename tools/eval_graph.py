"""Batch-1 eval forward in the loop of the unmodified bts_test.py / bts_main.py --do_online_eval, with eval graphs
(bts_b200.set_eval_graphs, BTS_B200_EVAL_GRAPH=1) off and on.

  python tools/eval_graph.py [--shapes T1,NYU,KITTI] [--images 50] [--warmup 5] [--rounds 3]

Shapes as tools/infer_step.py: T1 = DenseNet-121 at 416 x 544, NYU = DenseNet-161 at 480 x 640, KITTI = DenseNet-161 at
352 x 1216; random-init weights.  Per image, as the scripts do: image.cuda() and focal.cuda() of host tensors (focal in
float64, as the reference loader gives it), model(image, focal) under no_grad, .cpu() of the depth map, which waits for
the GPU.  A round times --images such images (cycling over four seeded ones) on the host clock after --warmup untimed
ones; rounds alternate off and on (switching off frees the graphs, so every on round captures again in its warm-up), and
the reported time is the median round.  Also reported: the eval-graph counters over the on rounds, the peak allocated
memory the first capture adds (torch.cuda.max_memory_allocated after it, minus the peak of the eager forwards before
it), the memory the captured graph keeps reserved (torch.cuda.memory_reserved after and before it, each after
empty_cache), and whether the depth maps with the switch on and off are bit-identical.  The card's name, power limit and
max SM clock are read in the same run.  One JSON line per shape."""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
from infer_step import SHAPES, build, card, median  # noqa: E402

MB = float(1 << 20)


def script_loop(torch, m, images, focal, n):
    """n images of the scripts' loop; returns (ms per image, the depth maps of the first len(images) images)"""
    depths = []
    t0 = time.perf_counter()
    with torch.no_grad():
        for i in range(n):
            out = m(images[i % len(images)].cuda(), focal.cuda())
            depth = out[4].cpu()
            if i < len(images):
                depths.append(depth)
    return 1000.0 * (time.perf_counter() - t0) / n, depths


def measure(torch, shape, args):
    import bts_b200
    from bts_b200 import graph
    m, _, _ = build(torch, shape)
    enc, H, W, _, _, focal = SHAPES[shape]
    g = torch.Generator().manual_seed(1)
    images = [torch.randn(1, 3, H, W, generator=g) for _ in range(4)]
    f = torch.tensor([focal], dtype=torch.float64)

    # memory of the first capture: eager forwards set the peak, then the second call of the signature captures
    bts_b200.set_eval_graphs(False)
    script_loop(torch, m, images, f, 2)
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    script_loop(torch, m, images, f, 2)
    torch.cuda.empty_cache()
    peak0, reserved0 = torch.cuda.max_memory_allocated(), torch.cuda.memory_reserved()
    bts_b200.set_eval_graphs(True)
    s0 = graph.eval_graph_stats()
    script_loop(torch, m, images, f, 2)
    torch.cuda.synchronize()
    peak1 = torch.cuda.max_memory_allocated()
    torch.cuda.empty_cache()
    reserved1 = torch.cuda.memory_reserved()
    assert graph.eval_graph_stats()["captures"] == s0["captures"] + 1

    res = {False: {"ms": [], "depth": None}, True: {"ms": [], "depth": None}}
    s0 = graph.eval_graph_stats()
    for r in range(args.rounds):
        for on in ((False, True) if r % 2 == 0 else (True, False)):
            bts_b200.set_eval_graphs(on)
            script_loop(torch, m, images, f, args.warmup)
            ms, depths = script_loop(torch, m, images, f, args.images)
            res[on]["ms"].append(ms)
            res[on]["depth"] = depths
    s1 = graph.eval_graph_stats()
    bts_b200.set_eval_graphs(False)
    same = all(torch.equal(a, b) for a, b in zip(res[False]["depth"], res[True]["depth"]))
    off, on = median(res[False]["ms"]), median(res[True]["ms"])
    return {"what": "batch-1 eval forward, script loop", "shape": shape, "encoder": enc, "HxW": "%dx%d" % (H, W),
            "images_per_round": args.images,
            "off_ms_per_img": round(off, 3), "off_img_per_s": round(1000.0 / off, 2),
            "off_ms_rounds": [round(t, 3) for t in res[False]["ms"]],
            "on_ms_per_img": round(on, 3), "on_img_per_s": round(1000.0 / on, 2),
            "on_ms_rounds": [round(t, 3) for t in res[True]["ms"]],
            "speedup": round(off / on, 2),
            "captures": s1["captures"] - s0["captures"], "replays": s1["replays"] - s0["replays"],
            "capture_peak_alloc_added_mb": round((peak1 - peak0) / MB, 1),
            "graph_reserved_mb": round((reserved1 - reserved0) / MB, 1),
            "depth_equal_on_off": same}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", default="T1,NYU,KITTI")
    ap.add_argument("--images", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    shapes = args.shapes.split(",")
    for s in shapes:
        if s not in SHAPES:
            ap.error("unknown shape %r (expected %s)" % (s, ", ".join(SHAPES)))
    if args.warmup < 2:
        ap.error("--warmup must be at least 2: the second call of a signature captures its graph")
    sys.path.insert(0, ROOT)
    os.environ.setdefault("BTS_B200_PRETRAINED", "0")
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("eval_graph.py measures on a GPU; none is visible")
    info = card()
    for s in shapes:
        r = measure(torch, s, args)
        r.update(info)
        print(json.dumps(r), flush=True)
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
