"""TEST INFRASTRUCTURE ONLY -- generates tests/golden/*.npz by running the UNMODIFIED reference
(/root/reference/pytorch/bts.py through oracle/ref_shim.py) on seeded inputs, on the CPU, fp32.

Run in the build container (the reference is mounted there, not on the GPU box):
    python oracle/make_golden.py
The committed fixtures are what pins oracle/bts_oracle.py and the CUDA path to the reference.
"""
import os
import sys
import types

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from ref_shim import load_reference  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests", "golden")


PART_BYTES = 900 * 1024      # fixture files stay below 1 MB: larger sets are split into NAME.npz + NAME.partK.npz


def save_split(name, d):
    """np.savez_compressed of d as NAME.npz, spilling arrays into NAME.part1.npz, ... (tests/conftest.py merges them).
    Part files of an earlier, larger set are removed first so that the loader never merges stale arrays."""
    import glob
    for old in glob.glob(os.path.join(OUT, name + ".part*.npz")):
        os.remove(old)
    parts, cur, size = [], {}, 0
    for k, v in d.items():
        if cur and size + v.nbytes > PART_BYTES:
            parts.append(cur)
            cur, size = {}, 0
        cur[k] = v
        size += v.nbytes
    parts.append(cur)
    for i, part in enumerate(parts):
        np.savez_compressed(os.path.join(OUT, name + (".part%d" % i if i else "") + ".npz"), **part)


def head_planes(B, h, w, max_depth, gen):
    """Plane coefficients through the real head parametrisation (BASELINE.md LPG-u inputs)."""
    z = torch.randn(B, 3, h, w, generator=gen)
    th = torch.sigmoid(z[:, 0]) * np.pi / 3
    ph = torch.sigmoid(z[:, 1]) * np.pi * 2
    d = torch.sigmoid(z[:, 2]) * max_depth
    return torch.stack([torch.sin(th) * torch.cos(ph), torch.sin(th) * torch.sin(ph), torch.cos(th), d], 1).contiguous()


# cases of tests/test_io_oracle.py: the inputs are regenerated there from the same seeds, only the reference's answers are stored
IO_DATASETS = ("nyu", "kitti")
IO_SEEDS = 6
# (B, h, w, r, seed) of tests/test_oracle_properties.py: drawn once from its hypothesis strategy's ranges
LPG_SHAPES = [(1, 1, 1, 2, 0), (1, 6, 7, 8, 1), (3, 1, 7, 4, 2), (2, 5, 3, 2, 3), (3, 6, 1, 8, 4), (1, 3, 4, 4, 5),
              (2, 2, 6, 8, 6), (3, 4, 5, 2, 999983), (2, 6, 7, 4, 123456), (1, 5, 2, 8, 777), (3, 3, 3, 2, 42), (2, 1, 4, 4, 10 ** 6)]
# encoders of tests/test_oracle.py::test_oracle_model_vs_live_reference_full_model
FULL_MODELS = ("densenet121_bts", "resnext50_bts", "mobilenetv2_bts")


def io_reference(R):
    """The reference's compute_errors (bts_main.py, extracted by ast: the script parses argv at import) and its training
    transform (bts_dataloader.py random_crop / train_preprocess / ToTensor) on the seeded inputs of test_io_oracle.py."""
    import ast
    import random
    from ref_shim import REFERENCE_DIR
    d = {}
    src = open(os.path.join(REFERENCE_DIR, "bts_main.py")).read()
    fn = [n for n in ast.parse(src).body if isinstance(n, ast.FunctionDef) and n.name == "compute_errors"][0]
    ns = {"np": np}
    exec(compile(ast.Module([fn], []), "bts_main.compute_errors", "exec"), ns)
    rng = np.random.RandomState(0)
    gt = rng.uniform(0.5, 70, 5000).astype(np.float32)
    pred = (gt * rng.uniform(0.6, 1.6, 5000)).astype(np.float32)
    d["compute_errors"] = np.array(ns["compute_errors"](gt, pred), dtype=np.float64)
    sys.path.insert(0, REFERENCE_DIR)
    import importlib
    D = importlib.import_module("bts_dataloader")
    for dataset in IO_DATASETS:
        ds = D.DataLoadPreprocess.__new__(D.DataLoadPreprocess)
        ds.args = types.SimpleNamespace(dataset=dataset)
        rng = np.random.RandomState(1)
        img_u8 = rng.randint(0, 256, (40, 56, 3)).astype(np.uint8)
        dep_u16 = rng.randint(0, 60000, (40, 56)).astype(np.uint16)
        div = 1000.0 if dataset == "nyu" else 256.0
        for seed in range(IO_SEEDS):
            random.seed(seed)
            np.random.seed(seed)
            image = np.asarray(img_u8, dtype=np.float32) / 255.0
            depth = np.expand_dims(np.asarray(dep_u16, dtype=np.float32), 2) / div
            ci, cd = ds.random_crop(image, depth, 32, 32)
            ri, rd = ds.train_preprocess(ci, cd)
            sample = D.ToTensor("train")({"image": ri, "depth": rd, "focal": 1.0})
            d["%s_%d_image" % (dataset, seed)] = sample["image"].numpy()
            d["%s_%d_depth" % (dataset, seed)] = sample["depth"].numpy()
    np.savez_compressed(os.path.join(OUT, "io_reference.npz"), **d)


def lpg_shapes(R):
    """local_planar_guidance of the reference on the planes tests/conftest.py:head_planes draws for LPG_SHAPES."""
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests"))
    from conftest import head_planes as planes
    d = {"shapes": np.array(LPG_SHAPES, dtype=np.int64)}
    for i, (B, h, w, r, seed) in enumerate(LPG_SHAPES):
        plane = planes(B, h, w, 10.0, seed=seed)
        want = R.local_planar_guidance(r)(plane, torch.full((B,), 518.8579))
        d["depth%d" % i] = (want.squeeze(1) if want.dim() == 4 else want).numpy()
    np.savez_compressed(os.path.join(OUT, "lpg_shapes.npz"), **d)


def full_models(R):
    """The reference BtsModel with the weights the oracle model draws under torch.manual_seed(0) (so that the test can
    rebuild them without the reference), eval and train mode, on the seeded inputs of test_oracle.py."""
    import bts_oracle as O
    d = {}
    for enc in FULL_MODELS:
        p = types.SimpleNamespace(encoder=enc, max_depth=10.0, dataset="nyu", bts_size=512)
        torch.manual_seed(0)
        orc = O.OracleModel(enc, 10.0, "nyu", 512)
        ref = R.BtsModel(p)
        ref.load_state_dict(orc.state_dict(), strict=True)
        x = torch.randn(1, 3, 64, 96, generator=torch.Generator().manual_seed(1))
        focal = torch.tensor([518.8579])
        for mode in ("eval", "train"):
            getattr(ref, mode)()
            if mode == "train":
                x = torch.cat([x, x.flip(3)], 0)
                focal = torch.tensor([518.8579, 518.8579])
            with torch.no_grad():
                outs = ref(x, focal)
            d.update({"%s_%s_out%d" % (enc, mode, i): o.numpy() for i, o in enumerate(outs)})
    np.savez_compressed(os.path.join(OUT, "full_models.npz"), **d)


def main():
    os.makedirs(OUT, exist_ok=True)
    R = load_reference()
    torch.set_num_threads(4)
    if len(sys.argv) > 1:                  # named fixture sets only, e.g. `make_golden.py io_reference full_models`
        for name in sys.argv[1:]:
            globals()[name](R)
        return

    # ---- LPG: forward + autograd gradient, r = 2, 4, 8 (pytorch/bts.py:124-146)
    for r in (2, 4, 8):
        gen = torch.Generator().manual_seed(100 + r)
        plane = head_planes(2, 5, 6, 10.0, gen).requires_grad_(True)
        mod = R.local_planar_guidance(r)
        depth = mod(plane, torch.tensor([518.8579, 518.8579]))
        dy = torch.randn(depth.shape, generator=gen)
        depth.backward(dy)
        np.savez_compressed(os.path.join(OUT, "lpg_r%d.npz" % r), plane=plane.detach().numpy(),
                            depth=depth.detach().numpy(), dy=dy.numpy(), dplane=plane.grad.numpy())

    # ---- reduction_1x1 (non-final and final) (pytorch/bts.py:83-122)
    gen = torch.Generator().manual_seed(7)
    torch.manual_seed(7)
    for final in (False, True):
        mod = R.reduction_1x1(32, 16, 10.0, is_final=final)
        x = torch.randn(2, 32, 6, 7, generator=gen)
        y = mod(x)
        d = {"x": x.numpy(), "y": y.detach().numpy()}
        d.update({"sd." + k: v.numpy() for k, v in mod.state_dict().items()})
        np.savez_compressed(os.path.join(OUT, "reduc_%s.npz" % ("final" if final else "plane")), **d)

    # ---- silog_loss forward + autograd gradient (pytorch/bts.py:41-48)
    gen = torch.Generator().manual_seed(11)
    est = (torch.rand(2, 1, 16, 24, generator=gen) * 79 + 1).requires_grad_(True)
    gt = torch.rand(2, 1, 16, 24, generator=gen) * 80
    gt = torch.where(torch.rand(2, 1, 16, 24, generator=gen) < 0.3, gt, torch.zeros_like(gt))
    mask = gt > 1.0
    loss = R.silog_loss(0.85).forward(est, gt, mask)
    loss.backward()
    np.savez_compressed(os.path.join(OUT, "silog.npz"), est=est.detach().numpy(), gt=gt.numpy(),
                        mask=mask.numpy(), loss=loss.detach().numpy(), dest=est.grad.numpy())

    # ---- whole decoder `bts` (pytorch/bts.py:148-266), small widths, eval and train mode
    feat = [8, 8, 16, 24, 40]
    for dataset, max_depth in (("kitti", 80.0), ("nyu", 10.0)):
        torch.manual_seed(3)
        params = types.SimpleNamespace(max_depth=max_depth, dataset=dataset)
        dec = R.bts(params, feat, num_features=128)
        dec.apply(R.weights_init_xavier)
        gen = torch.Generator().manual_seed(5)
        with torch.no_grad():      # non-trivial BN affine / running stats
            for m in dec.modules():
                if isinstance(m, torch.nn.BatchNorm2d):
                    m.weight.copy_(torch.rand(m.weight.shape, generator=gen) + 0.5)
                    m.bias.copy_(torch.randn(m.bias.shape, generator=gen) * 0.1)
                    m.running_mean.copy_(torch.randn(m.bias.shape, generator=gen) * 0.1)
                    m.running_var.copy_(torch.rand(m.bias.shape, generator=gen) + 0.5)
        H = W = 64
        B = 2
        feats = [torch.randn(B, feat[i], H >> (i + 1), W >> (i + 1), generator=gen) for i in range(5)]
        focal = torch.tensor([721.5377, 707.0912])
        d = {"focal": focal.numpy(), "feat_channels": np.array(feat), "num_features": np.array(128),
             "max_depth": np.array(max_depth)}
        d.update({"feat%d" % i: f.numpy() for i, f in enumerate(feats)})
        d.update({"sd." + k: v.clone().numpy() for k, v in dec.state_dict().items()})
        dec.eval()
        with torch.no_grad():
            outs = dec(feats, focal)
        d.update({"eval_out%d" % i: o.numpy() for i, o in enumerate(outs)})
        dec.train()
        with torch.no_grad():
            outs = dec(feats, focal)
        d.update({"train_out%d" % i: o.numpy() for i, o in enumerate(outs)})
        d.update({"sd_after." + k: v.numpy() for k, v in dec.state_dict().items() if "running" in k})
        save_split("decoder_%s" % dataset, d)
    io_reference(R)
    lpg_shapes(R)
    full_models(R)
    print("golden fixtures written to", os.path.abspath(OUT))
    for f in sorted(os.listdir(OUT)):
        print("  %-24s %8d bytes" % (f, os.path.getsize(os.path.join(OUT, f))))


if __name__ == "__main__":
    main()
