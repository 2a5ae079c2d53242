"""GPU training transform with and without the random rotation (bts_input_prep / bts_input_prep_rotated, csrc/io.cu),
against the reference loader's CPU transform per sample.

  python tools/input_prep_rotate.py [--iters 200] [--rounds 5] [--cpu-samples 20] [--out FILE]

GPU: batches at the recipes' shapes -- KITTI B = 4 and 16 (352 x 1216 after the KB crop -> 352 x 704 crop) and NYU B = 4 and
16 (427 x 565 after its crop -> 416 x 544) -- with seeded frames and 16-bit depth, half the samples flipped and half
augmented, one angle per sample within the recipe's degree (eigen 1.0, nyu 2.5).  The two kernels are launched through the
C ABI on preallocated buffers and alternate over --rounds rounds; each round times --iters launches with CUDA events (one
synchronize at the end) and the reported time is the median round.  Algorithmic bytes per output pixel: 3 (image read) +
2 (depth read) + 12 (fp32 image write) + 4 (fp32 depth write); the bilinear 2x2 neighbourhoods overlap between neighbouring
pixels, so rotation adds no algorithmic traffic.  The share of peak is those bytes at the H100 SXM data sheet's 3.35 TB/s
over the kernel time.  The rotated output is checked against the unrotated one at angle 0 (bit-identical) before timing.

CPU: the unmodified reference loader (oracle/_ref/bts_dataloader.py, when `make -C oracle` placed it there), one process,
one torch thread, as `--num_threads 1` runs it: DataLoadPreprocess.__getitem__ (train, rotation on) per sample on a
synthetic PNG set in a temporary directory, the PNG decode (+ fixed crop) alone, and the two PIL rotates alone.
The card's name and power limit and the host's core count are read in the same run.  One JSON line per result."""
import argparse
import ctypes
import json
import os
import random
import shutil
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM_BYTES_PER_S = 3.35e12
BYTES_PER_PIXEL = 3 + 2 + 12 + 4
# name: (dataset, frame Hs, Ws, crop H, W, depth divisor, recipe degree)
SHAPES = {"kitti": ("kitti", 352, 1216, 352, 704, 256.0, 1.0), "nyu": ("nyu", 427, 565, 416, 544, 1000.0, 2.5)}
RAW = {"kitti": (375, 1242), "nyu": (480, 640)}


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clk = [s.strip() for s in out.split(",")]
        return {"gpu": name, "power_limit": power, "max_sm_clock": clk}
    except Exception as e:                       # the numbers are still printed, the card is reported unknown
        return {"gpu": "unknown (%s)" % type(e).__name__}


def cores():
    return {"cpu_count": os.cpu_count(), "cpu_affinity": len(os.sched_getaffinity(0))}


def median(xs):
    xs = sorted(xs)
    return xs[len(xs) // 2] if len(xs) % 2 else 0.5 * (xs[len(xs) // 2 - 1] + xs[len(xs) // 2])


def gpu_rows(iters, rounds):
    import numpy as np
    import torch
    from bts_b200 import _lib, data, ops
    if not torch.cuda.is_available():
        raise SystemExit("the GPU measurement needs a CUDA device")
    L = _lib.lib()
    ptr = ctypes.c_void_p
    rows = []
    for name, B in (("kitti", 4), ("kitti", 16), ("nyu", 4), ("nyu", 16)):
        dataset, Hs, Ws, H, W, div, degree = SHAPES[name]
        rng = np.random.RandomState(B)
        img = torch.from_numpy(rng.randint(0, 256, (B, Hs, Ws, 3)).astype(np.uint8)).cuda()
        dep = torch.from_numpy(rng.randint(0, 65536, (B, Hs, Ws)).astype(np.int16)).cuda().view(torch.uint16)
        par = torch.from_numpy(np.array([[rng.randint(0, Hs - H + 1), rng.randint(0, Ws - W + 1), b % 2, (b // 2) % 2,
                                          1.05, 0.95, 0.92, 1.03, 1.08] for b in range(B)], dtype=np.float32)).cuda()
        angles = list(rng.uniform(-degree, degree, B))
        affine = torch.tensor([data.rotate_affine(a, Ws, Hs) for a in angles], dtype=torch.float64).cuda()
        out = torch.empty((B, H, W, 3), device="cuda")
        dout = torch.empty((B, H, W), device="cuda")
        stream = ptr(torch.cuda.current_stream().cuda_stream)

        def launch(aff):
            rc = L.bts_input_prep_rotated(ptr(img.data_ptr()), Hs, Ws, ptr(dep.data_ptr()), div, ptr(par.data_ptr()), aff, B,
                                          H, W, ptr(out.data_ptr()), 3, ptr(dout.data_ptr()), stream)
            if rc != 0:
                raise RuntimeError("bts_input_prep_rotated returned %d" % rc)

        # angle 0 through the rotated kernel must equal the unrotated kernel
        i0, d0 = ops.input_prep(img, par, (H, W), dep, div)
        i1, d1 = ops.input_prep(img, par, (H, W), dep, div, angles=[0.0] * B)
        assert torch.equal(i0, i1) and torch.equal(d0, d1), "angle 0 differs from the unrotated transform"
        variants = {"plain": None, "rotated": ptr(affine.data_ptr())}
        times = {k: [] for k in variants}
        for k, aff in variants.items():                    # warm-up
            for _ in range(10):
                launch(aff)
        torch.cuda.synchronize()
        for _ in range(rounds):
            for k, aff in variants.items():
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(iters):
                    launch(aff)
                e1.record()
                e1.synchronize()
                times[k].append(e0.elapsed_time(e1) / iters * 1e3)      # us per launch
        nbytes = B * H * W * BYTES_PER_PIXEL
        for k in variants:
            t = median(times[k])
            rows.append({"kind": "gpu", "shape": name, "B": B, "frame": [Hs, Ws], "crop": [H, W], "variant": k,
                         "us_per_batch": round(t, 2), "spread_us": [round(min(times[k]), 2), round(max(times[k]), 2)],
                         "samples_per_s": round(B / (t * 1e-6)), "alg_bytes": nbytes,
                         "hbm_share": round(nbytes / HBM_BYTES_PER_S / (t * 1e-6), 3)})
    return rows


def cpu_rows(samples):
    import numpy as np
    import torch
    from PIL import Image
    ref = os.path.join(ROOT, "oracle", "_ref")
    if not os.path.isfile(os.path.join(ref, "bts_dataloader.py")):
        return [{"kind": "cpu", "note": "not measured: oracle/_ref/bts_dataloader.py is absent"}]
    sys.path.insert(0, ref)
    import bts_dataloader as R
    import types
    torch.set_num_threads(1)
    rows = []
    tmp = tempfile.mkdtemp(prefix="input_prep_rotate_")
    try:
        for name in ("kitti", "nyu"):
            dataset, Hs, Ws, H, W, div, degree = SHAPES[name]
            h, w = RAW[name]
            rng = np.random.RandomState(0)
            yy, xx = np.mgrid[0:h, 0:w].astype(np.float32)
            lines = []
            for i in range(4):
                img = np.stack([xx / w * 255, yy / h * 255, rng.uniform(0, 255, (h, w))], -1).astype(np.uint8)
                dep = ((1.0 + 4.0 * yy / h + 0.5 * np.sin(xx / 40.0 + i)) * div).astype(np.uint16)
                Image.fromarray(img).save(os.path.join(tmp, "%s_%d_img.png" % (name, i)))
                Image.fromarray(dep).save(os.path.join(tmp, "%s_%d_dep.png" % (name, i)))
                lines.append("%s_%d_img.png %s_%d_dep.png 518.8579" % (name, i, name, i))
            flist = os.path.join(tmp, name + ".txt")
            with open(flist, "w") as f:
                f.write("\n".join(lines) + "\n")
            args = types.SimpleNamespace(dataset=dataset, use_right=False, data_path=tmp + "/", gt_path=tmp + "/",
                                         filenames_file=flist, do_kb_crop=name == "kitti", do_random_rotate=True,
                                         degree=degree, input_height=H, input_width=W)
            ds = R.DataLoadPreprocess(args, "train", transform=R.preprocessing_transforms("train"))
            random.seed(0)
            np.random.seed(0)
            ds[0]
            t0 = time.perf_counter()
            for i in range(samples):
                ds[i % len(lines)]
            t_item = (time.perf_counter() - t0) / samples

            def decoded(i):
                a, b = Image.open(os.path.join(tmp, "%s_%d_img.png" % (name, i))), \
                    Image.open(os.path.join(tmp, "%s_%d_dep.png" % (name, i)))
                if name == "kitti":
                    box = ((w - 1216) // 2, h - 352, (w - 1216) // 2 + 1216, h)
                else:
                    box = (43, 45, 608, 472)
                return a.crop(box), b.crop(box)

            t0 = time.perf_counter()
            frames = [decoded(i % len(lines)) for i in range(samples)]
            for a, b in frames:
                a.load()
                b.load()
            t_dec = (time.perf_counter() - t0) / samples
            t0 = time.perf_counter()
            for a, b in frames:
                angle = (random.random() - 0.5) * 2 * degree
                ds.rotate_image(a, angle)
                ds.rotate_image(b, angle, flag=Image.NEAREST)
            t_rot = (time.perf_counter() - t0) / samples
            rows.append(dict({"kind": "cpu", "shape": name, "raw": [h, w], "crop": [H, W], "samples": samples,
                              "getitem_ms": round(t_item * 1e3, 2), "decode_crop_ms": round(t_dec * 1e3, 2),
                              "rotate_ms": round(t_rot * 1e3, 2),
                              "getitem_samples_per_s": round(1.0 / t_item, 1)}, **cores()))
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--cpu-samples", type=int, default=20)
    ap.add_argument("--out", default=None, help="also append the JSON lines to this file")
    a = ap.parse_args()
    rows = [dict({"kind": "card"}, **card(), **cores())] + gpu_rows(a.iters, a.rounds) + cpu_rows(a.cpu_samples)
    for r in rows:
        print(json.dumps(r), flush=True)
    if a.out:
        with open(a.out, "a") as f:
            for r in rows:
                f.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
