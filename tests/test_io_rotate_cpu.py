"""CPU: the host side of the rotated GPU input transform, pinned to Pillow and to the reference loader.

  * bts_b200.data.rotate_affine equals, bit for bit, the matrix Image.rotate hands to Image.transform;
  * io_rotate_oracle (the checker of bts_input_prep_rotated) equals Image.rotate bit for bit: bilinear on RGB frames, nearest
    on 16-bit depth read back from a PNG (mode I;16, as the loader opens KITTI / NYU ground truth);
  * with `random` / `np.random` seeded, data.fixed_crop + data.draw_train_sample + the oracle reproduce the unmodified
    reference DataLoadPreprocess.__getitem__ (train mode, rotation on), when oracle/_ref holds the reference loader."""
import ctypes
import io
import os

import numpy as np
import pytest
from PIL import Image

import io_rotate_oracle as RO
from bts_b200 import data

ANGLES = [0.3, -0.3, 1.0, -1.0, 2.5, -2.5, 0.0, 360.0, -360.0, 90.0, 180.0, 30.0]
SIZES = [(1216, 352), (565, 427), (1215, 351)]         # PIL (w, h): KITTI after the KB crop, NYU after its crop, odd


def _bits(v):
    return np.array(v, dtype=np.float64).view(np.int64).tolist()


@pytest.mark.parametrize("w,h", SIZES)
def test_rotate_affine_is_the_matrix_pillow_passes_to_transform(w, h, monkeypatch):
    captured = []
    transform = Image.Image.transform

    def spy(self, size, method, data_=None, *args, **kwargs):
        captured.append(list(data_))
        return transform(self, size, method, data_, *args, **kwargs)

    monkeypatch.setattr(Image.Image, "transform", spy)
    im = Image.new("L", (w, h))
    for angle in ANGLES:
        captured.clear()
        im.rotate(angle, resample=Image.BILINEAR)
        if not captured:
            # Pillow's fast paths (copy / transpose) skip transform; an explicit default centre forces the affine path,
            # which builds the matrix with the same expressions
            im.rotate(angle, resample=Image.BILINEAR, center=(w / 2, h / 2))
        assert len(captured) == 1
        assert _bits(data.rotate_affine(angle, w, h)) == _bits(captured[0]), angle


def test_rotate_affine_at_zero_is_the_identity_and_rejects_non_finite_angles():
    for angle in (0.0, 360.0, -360.0, 720.0):
        a, b, c, d, e, f = data.rotate_affine(angle, 1215, 351)
        assert (a, b, c, d, e, f) == (1.0, 0.0, 0.0, 0.0, 1.0, 0.0)
    for bad in (float("nan"), float("inf")):
        with pytest.raises(ValueError):
            data.rotate_affine(bad, 10, 10)


def _png_u16(a):
    buf = io.BytesIO()
    Image.fromarray(a).save(buf, format="PNG")
    buf.seek(0)
    im = Image.open(buf)
    im.load()
    return im


@pytest.mark.parametrize("hw", [(352, 1216), (427, 565), (351, 1215), (64, 64)])
def test_oracle_matches_pillow_rotate_bit_for_bit(hw):
    h, w = hw
    rng = np.random.RandomState(h + w)
    img = rng.randint(0, 256, (h, w, 3)).astype(np.uint8)
    dep = rng.randint(0, 65536, (h, w)).astype(np.uint16)
    dep[rng.uniform(size=(h, w)) < 0.5] = 0                  # sparse, as KITTI ground truth
    dpil = _png_u16(dep)
    assert dpil.mode == "I;16"
    ipil = Image.fromarray(img)
    for angle in (0.73, -0.41, 2.5, -2.5, 1.0, 17.3, 30.0, -45.0, 0.0, 90.0, 180.0, 270.0):
        co = data.rotate_affine(angle, w, h)
        np.testing.assert_array_equal(RO.rotate_bilinear_u8(img, co),
                                      np.asarray(ipil.rotate(angle, resample=Image.BILINEAR)), err_msg=str(angle))
        np.testing.assert_array_equal(RO.rotate_nearest(dep, co),
                                      np.asarray(dpil.rotate(angle, resample=Image.NEAREST)), err_msg=str(angle))


def test_fixed_crop_is_the_reference_crop_boxes():
    rng = np.random.RandomState(0)
    kitti = rng.randint(0, 256, (375, 1242, 3)).astype(np.uint8)
    want = np.asarray(Image.fromarray(kitti).crop((13, 23, 13 + 1216, 23 + 352)))
    np.testing.assert_array_equal(data.fixed_crop(kitti, "kitti", do_kb_crop=True), want)
    assert data.fixed_crop(kitti, "kitti").shape == kitti.shape
    nyu = rng.randint(0, 65536, (480, 640)).astype(np.uint16)
    np.testing.assert_array_equal(data.fixed_crop(nyu, "nyu"), np.asarray(_png_u16(nyu).crop((43, 45, 608, 472))))
    with pytest.raises(ValueError):
        data.fixed_crop(kitti[:351], "kitti", do_kb_crop=True)
    with pytest.raises(ValueError):
        data.fixed_crop(nyu[:, :600], "nyu")
    with pytest.raises(ValueError):
        data.draw_train_sample("nyu", (427, 565), (428, 544))


def test_rotated_entry_point_refuses_bad_arguments():
    from bts_b200 import _lib
    L = _lib.lib()
    EINVAL = -1
    p = ctypes.c_void_p(1 << 20)          # fake device address: every call below must return before it launches
    ok = dict(img=p, Hs=8, Ws=8, dep=None, div=1000.0, params=p, affine=p, B=1, H=4, W=4, out=p, os=3, dout=None)

    def call(**kw):
        a = dict(ok, **kw)
        return L.bts_input_prep_rotated(a["img"], a["Hs"], a["Ws"], a["dep"], a["div"], a["params"], a["affine"], a["B"],
                                        a["H"], a["W"], a["out"], a["os"], a["dout"], None)

    for bad in (dict(img=None), dict(params=None), dict(out=None), dict(B=0), dict(H=0), dict(W=-1), dict(Hs=3),
                dict(Ws=3), dict(os=2), dict(dep=p), dict(dep=p, dout=p, div=0.0)):
        assert call(**bad) == EINVAL, bad


# ------------------------------------------------------------------ seeded end-to-end against the reference loader
@pytest.mark.skipif(not os.path.isfile(RO.REF_LOADER), reason="reference loader not available (`make -C oracle` copies it "
                                                           "into oracle/_ref)")
@pytest.mark.parametrize("dataset", ["kitti", "nyu"])
def test_seeded_draws_and_oracle_reproduce_reference_loader(dataset, tmp_path):
    mod = RO.reference_loader()
    root = str(tmp_path)
    lines = RO.make_dataset(root, dataset)
    _, (H, W), div, _ = RO.CASES[dataset]
    seen_right = set()
    for degree, seeds in ((None, range(4)), (30.0, range(4, 6))):       # the recipe's degree, and large angles (fill)
        args = RO.reference_args(root + "/", dataset, degree)
        for seed in seeds:
            idx = seed % len(lines)
            want_i, want_d = RO.reference_sample(mod, args, idx, seed)
            img, dep, params, angle, right = RO.our_sample(args, lines[idx], seed)
            assert angle != 0.0
            seen_right.add(right)
            got_i, got_d = RO.input_prep(img, dep, div, int(params[0]), int(params[1]), H, W, params[2] > 0.5,
                                         params[3] > 0.5, params[4], params[5], params[6:9],
                                         data.rotate_affine(angle, img.shape[1], img.shape[0]))
            np.testing.assert_allclose(got_i, want_i, rtol=1e-6, atol=1e-6)
            np.testing.assert_array_equal(got_d, want_d)
    assert seen_right == ({False, True} if dataset == "kitti" else {False})
