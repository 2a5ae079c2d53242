"""GPU tests of ops.decode_png (csrc/png.cu): bit-identical with Pillow's decode (np.asarray(Image.open(f))) and the
reference's fixed crops, on Pillow-encoded files and on the tests' own encoder (every filter type, every zlib strategy,
IDAT split into small chunks); chained into the GPU input transform; malformed streams reported per image."""
import io
import os

import numpy as np
import pytest
import torch
from PIL import Image

import io_rotate_oracle as RO
import png_testutil as PT
from bts_b200 import data

pytestmark = pytest.mark.gpu


def _pil_png(arr, **kw):
    buf = io.BytesIO()
    Image.fromarray(arr).save(buf, format="PNG", **kw)
    return buf.getvalue()


def _pil(blob):
    return np.asarray(Image.open(io.BytesIO(blob)))


def _decode(blobs, origins=None, out_hw=None):
    from bts_b200 import ops
    return ops.decode_png(blobs, origins, out_hw).cpu().numpy()


def _frame(kind, H, W, seed):
    rng = np.random.RandomState(seed)
    yy, xx = np.mgrid[0:H, 0:W]
    if kind == "rgb":
        base = (np.sin(yy / 9.0)[..., None] * 50 + np.cos(xx / 13.0)[..., None] * 50 + 128) + rng.randint(-8, 9, (H, W, 3))
        return np.clip(base, 0, 255).astype(np.uint8)
    dep = (rng.uniform(size=(H, W)) < 0.3) * (yy * 97 + xx * 31 + rng.randint(0, 200, (H, W)))
    return (dep % 65536).astype(np.uint16)


@pytest.mark.parametrize("kind", ["rgb", "gray16"])
@pytest.mark.parametrize("hw", [(1, 1), (7, 5), (64, 3), (375, 1242)])
def test_pillow_encoded(kind, hw):
    H, W = hw
    arr = _frame(kind, H, W, H + W)
    blobs = [_pil_png(arr, compress_level=lv) for lv in (0, 1, 6, 9)] + [_pil_png(arr, optimize=True)]
    got = _decode(blobs)
    for i, b in enumerate(blobs):
        np.testing.assert_array_equal(got[i], _pil(b), err_msg="blob %d" % i)


@pytest.mark.parametrize("kind", ["rgb", "gray16"])
def test_own_encoder_filters_strategies_chunks(kind):
    H, W = 37, 29
    arr = _frame(kind, H, W, 9)
    blobs = [PT.encode_png(arr, filters=f) for f in range(5)] + [PT.encode_png(arr, filters="mix", seed=s) for s in (1, 2)]
    blobs += [PT.encode_png(arr, filters="mix", strategy=s, level=lv) for s in PT.STRATEGIES for lv in (1, 9)]
    blobs += [PT.encode_png(arr, filters="mix", idat_chunk=c) for c in (1, 7)]
    got = _decode(blobs)
    for i, b in enumerate(blobs):
        np.testing.assert_array_equal(got[i], _pil(b), err_msg="blob %d" % i)
        np.testing.assert_array_equal(got[i], arr, err_msg="blob %d" % i)


KITTI_SIZES = [(375, 1242), (376, 1241), (370, 1224), (374, 1238), (370, 1226)]


@pytest.mark.parametrize("kind", ["rgb", "gray16"])
def test_mixed_size_kitti_batch_with_kb_crop(kind):
    blobs = [_pil_png(_frame(kind, h, w, i)) for i, (h, w) in enumerate(KITTI_SIZES)]
    boxes = [data.fixed_crop_box("kitti", True, h, w) for h, w in KITTI_SIZES]
    got = _decode(blobs, [b[:2] for b in boxes], boxes[0][2:])
    want = np.stack([data.fixed_crop(_pil(b), "kitti", True) for b in blobs])
    np.testing.assert_array_equal(got, want)


def test_nyu_depth_with_nyu_box():
    blobs = [_pil_png(_frame("gray16", 480, 640, s)) for s in range(3)]
    y0, x0, Hc, Wc = data.fixed_crop_box("nyu", False, 480, 640)
    got = _decode(blobs, [(y0, x0)] * 3, (Hc, Wc))
    np.testing.assert_array_equal(got, np.stack([data.fixed_crop(_pil(b), "nyu", False) for b in blobs]))


def test_decode_chained_into_input_prep():
    from bts_b200 import ops
    rgb = [_pil_png(_frame("rgb", 375, 1242, s)) for s in range(2)]
    dep = [_pil_png(_frame("gray16", 375, 1242, s + 5)) for s in range(2)]
    box = data.fixed_crop_box("kitti", True, 375, 1242)
    img_d = ops.decode_png(rgb, [box[:2]] * 2, box[2:])
    dep_d = ops.decode_png(dep, [box[:2]] * 2, box[2:])
    img_p = torch.from_numpy(np.stack([data.fixed_crop(_pil(b), "kitti", True) for b in rgb])).cuda()
    dep_p = torch.from_numpy(np.stack([data.fixed_crop(_pil(b), "kitti", True) for b in dep]).view(np.int16)).cuda()
    par = torch.tensor([[0, 5, 1, 1, 1.05, 0.95, 0.9, 1.0, 1.1], [10, 400, 0, 0, 1, 1, 1, 1, 1]], device="cuda")
    for angles in (None, [0.7, -1.0]):
        a = ops.input_prep(img_d, par, (320, 704), dep_d, 256.0, angles=angles)
        b = ops.input_prep(img_p, par, (320, 704), dep_p.view(torch.uint16), 256.0, angles=angles)
        for x, y in zip(a, b):
            assert torch.equal(x, y)


@pytest.mark.skipif(not os.path.isfile(RO.REF_LOADER), reason="reference loader not available (`make -C oracle` copies it "
                                                             "into oracle/_ref)")
@pytest.mark.parametrize("dataset", ["kitti", "nyu"])
def test_decode_then_transform_reproduces_reference_loader(dataset, tmp_path):
    """DataLoadPreprocess.__getitem__ (train, rotation on) against file bytes -> draw_train_sample -> decode_png with the
    fixed_crop_box window -> input_prep_rotated, on the same seeds"""
    import random
    from bts_b200 import ops
    mod = RO.reference_loader()
    root = str(tmp_path) + "/"
    lines = RO.make_dataset(root, dataset)
    _, (H, W), div, _ = RO.CASES[dataset]
    args = RO.reference_args(root, dataset)
    for seed in range(4):
        idx = seed % len(lines)
        want_i, want_d = RO.reference_sample(mod, args, idx, seed)
        random.seed(seed)
        np.random.seed(seed)
        f = lines[idx].split()
        w, h = Image.open(os.path.join(root, f[0])).size
        y0, x0, Hc, Wc = data.fixed_crop_box(dataset, args.do_kb_crop, h, w)
        params, angle, right = data.draw_train_sample(dataset, (Hc, Wc), (H, W), True, args.degree, args.use_right)
        names = (f[3], f[4]) if right else (f[0], f[1])
        blobs = [open(os.path.join(root, n), "rb").read() for n in names]
        img = ops.decode_png(blobs[:1], [(y0, x0)], (Hc, Wc))
        dep = ops.decode_png(blobs[1:], [(y0, x0)], (Hc, Wc))
        gi, gd = ops.input_prep(img, torch.from_numpy(params[None]).cuda(), (H, W), dep, div, angles=[angle])
        np.testing.assert_array_equal(gd.cpu().numpy()[0], want_d, err_msg="seed %d" % seed)
        np.testing.assert_allclose(gi.cpu().numpy()[0], want_i, rtol=2e-6, atol=2e-6, err_msg="seed %d" % seed)


REASONS = {1: "truncated stream", 2: "bad zlib header", 5: "distance too far back", 7: "Adler-32 mismatch",
           8: "bad filter type"}


@pytest.mark.parametrize("name", sorted(PT.malformed_cases()))
def test_malformed_stream_names_image_and_reason(name):
    blob, H, W, status = PT.malformed_cases()[name]
    good = [_pil_png(_frame("rgb", H, W, s)) for s in range(3)]
    with pytest.raises(ValueError, match="image 2: %s" % REASONS[status]):
        _decode(good[:2] + [blob] + good[2:])
    got = _decode(good)   # nothing is left behind: the next batch decodes
    np.testing.assert_array_equal(got, np.stack([_pil(b) for b in good]))


def test_non_default_stream():
    from bts_b200 import ops
    blobs = [_pil_png(_frame("rgb", 64, 96, s)) for s in range(4)]
    want = _decode(blobs)
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        got = ops.decode_png(blobs)
    s.synchronize()
    np.testing.assert_array_equal(got.cpu().numpy(), want)
