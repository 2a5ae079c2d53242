"""GPU parity of the rotated input transform (bts_input_prep_rotated, csrc/io.cu) against tests/io_rotate_oracle.py (itself
pinned to Pillow's Image.rotate and to the reference loader by tests/test_io_rotate_cpu.py).  The rotated depth is
bit-exact; the image is exact through the /255 value (the byte PIL's rotate leaves) and within test_io_gpu.py's tolerance
after the float steps (powf)."""
import os

import numpy as np
import pytest
import torch

import io_rotate_oracle as RO
from bts_b200 import data

pytestmark = pytest.mark.gpu

MEAN = np.array([0.485, 0.456, 0.406], dtype=np.float32)[:, None, None]
STD = np.array([0.229, 0.224, 0.225], dtype=np.float32)[:, None, None]


def _frames(B, Hs, Ws, seed):
    rng = np.random.RandomState(seed)
    img = rng.randint(0, 256, (B, Hs, Ws, 3)).astype(np.uint8)
    dep = rng.randint(1, 65536, (B, Hs, Ws)).astype(np.uint16)
    dep[rng.uniform(size=dep.shape) < 0.3] = 0
    return img, dep


def _params(rows):
    """rows of (y0, x0, flip, augment); augment rows get gamma / brightness / colours of the loader's ranges"""
    rng = np.random.RandomState(len(rows))
    return np.array([[y0, x0, fl, au, rng.uniform(0.9, 1.1), rng.uniform(0.75, 1.25), *rng.uniform(0.9, 1.1, 3)]
                     for y0, x0, fl, au in rows], dtype=np.float32)


def _run(img, dep, par, H, W, div, angles):
    from bts_b200 import ops
    gi, gd = ops.input_prep(torch.from_numpy(img).cuda(), torch.from_numpy(par).cuda(), (H, W),
                            torch.from_numpy(dep.view(np.int16)).cuda().view(torch.uint16), div, angles=angles)
    torch.cuda.synchronize()
    return gi.cpu().numpy(), gd.cpu().numpy()


def _check(img, dep, par, H, W, div, angles):
    gi, gd = _run(img, dep, par, H, W, div, angles)
    Hs, Ws = img.shape[1:3]
    for b in range(img.shape[0]):
        co = data.rotate_affine(angles[b], Ws, Hs)
        args = (int(par[b, 0]), int(par[b, 1]), H, W, par[b, 2] > 0.5, par[b, 3] > 0.5, par[b, 4], par[b, 5], par[b, 6:9])
        wi, wd = RO.input_prep(img[b], dep[b], div, *args, coeffs=co)
        msg = "sample %d angle %g" % (b, angles[b])
        np.testing.assert_array_equal(gd[b], wd, err_msg=msg)
        np.testing.assert_allclose(gi[b], wi, rtol=2e-6, atol=2e-6, err_msg=msg)
        if par[b, 3] < 0.5:
            # no augmentation: the output is (byte/255 - mean)/std, so the bytes the rotation produced can be read back
            want = RO.input_prep(img[b], None, div, *args[:5], False, 1.0, 1.0, np.ones(3), coeffs=co)[0]
            got_u8 = np.rint((gi[b] * STD + MEAN) * 255.0).astype(np.int64)
            want_u8 = np.rint((want * STD + MEAN) * 255.0).astype(np.int64)
            np.testing.assert_array_equal(got_u8, want_u8, err_msg=msg)


@pytest.mark.parametrize("shape,div,angles", [
    ((352, 1216, 352, 704), 256.0, [1.0, -0.63, 0.25, -1.0]),        # KITTI after the KB crop, eigen recipe degree 1.0
    ((427, 565, 416, 544), 1000.0, [2.5, -2.5, 1.37, -0.08]),        # NYU after its crop, nyu recipe degree 2.5
])
def test_rotated_input_prep_matches_oracle(shape, div, angles):
    Hs, Ws, H, W = shape
    img, dep = _frames(4, Hs, Ws, Hs)
    # per-sample angles, flip and augment mixed, crops at the frame's corners (where the fill shows) and inside
    par = _params([(0, 0, 0, 0), (Hs - H, Ws - W, 1, 0), (Hs - H, 0, 0, 1), ((Hs - H) // 2, Ws - W - 5, 1, 1)])
    _check(img, dep, par, H, W, div, angles)


@pytest.mark.parametrize("angles", [[30.0, -45.0, 90.0, 180.0], [-30.0, 45.0, 270.0, 359.5]])
def test_large_angles_fill_and_clamp(angles):
    Hs, Ws, H, W = 96, 160, 64, 112
    img, dep = _frames(4, Hs, Ws, 11)
    par = _params([(0, 0, 0, 0), (Hs - H, Ws - W, 1, 0), (7, 13, 0, 1), (Hs - H, 0, 1, 1)])
    _check(img, dep, par, H, W, 256.0, angles)


@pytest.mark.parametrize("shape", [(351, 1215, 351, 703), (427, 565, 415, 543), (37, 53, 37, 53)])
def test_odd_frame_sizes(shape):
    Hs, Ws, H, W = shape
    img, dep = _frames(3, Hs, Ws, Ws)
    par = _params([(0, 0, 1, 0), (Hs - H, Ws - W, 0, 1), ((Hs - H) // 2, (Ws - W) // 2, 1, 1)])
    _check(img, dep, par, H, W, 1000.0, [0.91, -2.5, 17.3])


def test_angle_zero_is_bit_identical_to_the_unrotated_transform():
    Hs, Ws, H, W = 427, 565, 416, 544
    img, dep = _frames(4, Hs, Ws, 5)
    par = _params([(0, 0, 0, 0), (Hs - H, Ws - W, 1, 0), (2, 9, 0, 1), (Hs - H, 0, 1, 1)])
    plain_i, plain_d = _run(img, dep, par, H, W, 1000.0, None)
    for angles in ([0.0] * 4, [360.0, -360.0, 0.0, 720.0]):
        gi, gd = _run(img, dep, par, H, W, 1000.0, angles)
        assert np.array_equal(gi.view(np.int32), plain_i.view(np.int32))
        assert np.array_equal(gd.view(np.int32), plain_d.view(np.int32))


def test_angles_are_validated():
    from bts_b200 import ops
    img = torch.zeros((2, 8, 8, 3), dtype=torch.uint8, device="cuda")
    par = torch.zeros((2, 9), device="cuda")
    with pytest.raises(ValueError, match="one angle per sample"):
        ops.input_prep(img, par, (4, 4), angles=[1.0])
    with pytest.raises(ValueError, match="finite"):
        ops.input_prep(img, par, (4, 4), angles=[1.0, float("nan")])
    gi, _ = ops.input_prep(img, par, (4, 4), angles=torch.tensor([1.0, -1.0]))
    assert gi.shape == (2, 3, 4, 4)


# ------------------------------------------------------------------ seeded end-to-end against the reference loader
@pytest.mark.skipif(not os.path.isfile(RO.REF_LOADER), reason="reference loader not available (`make -C oracle` copies it "
                                                             "into oracle/_ref)")
@pytest.mark.parametrize("dataset", ["kitti", "nyu"])
def test_gpu_transform_reproduces_reference_loader(dataset, tmp_path):
    """DataLoadPreprocess.__getitem__ (train, rotation on) against fixed_crop + draw_train_sample + ops.input_prep, on the
    same seeds: sample['depth'] bit for bit, sample['image'] within the float tolerance"""
    mod = RO.reference_loader()
    root = str(tmp_path) + "/"
    lines = RO.make_dataset(root, dataset)
    _, (H, W), div, _ = RO.CASES[dataset]
    for degree, seeds in ((None, range(4)), (30.0, range(4, 6))):
        args = RO.reference_args(root, dataset, degree)
        for seed in seeds:
            idx = seed % len(lines)
            want_i, want_d = RO.reference_sample(mod, args, idx, seed)
            img, dep, params, angle, _ = RO.our_sample(args, lines[idx], seed)
            gi, gd = _run(img[None].copy(), dep[None].copy(), params[None], H, W, div, [angle])
            np.testing.assert_array_equal(gd[0], want_d, err_msg="seed %d" % seed)
            np.testing.assert_allclose(gi[0], want_i, rtol=2e-6, atol=2e-6, err_msg="seed %d" % seed)
