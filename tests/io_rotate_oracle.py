"""TEST INFRASTRUCTURE ONLY -- float64 numpy restatement of Pillow's affine resampling as Image.rotate uses it
(pytorch/bts_dataloader.py:124-125,187-189): bilinear for the RGB frame, nearest for the 16-bit depth.  The checker of the
rotated variant of bts_input_prep (csrc/io.cu); pinned to Image.rotate bit for bit by tests/test_io_rotate_cpu.py.

Coefficients (a..f) map output pixel (x, y) to the source point X = a*(x+.5) + b*(y+.5) + c, Y = d*(x+.5) + e*(y+.5) + f,
evaluated left to right in float64 with every product and sum rounded on its own (numpy does not fuse them).
  bilinear  0 unless 0 <= X < Ws and 0 <= Y < Hs; X -= .5, Y -= .5, x0 = floor X, y0 = floor Y, dx = X-x0, dy = Y-y0;
            columns x0, x0+1 and row y0 clamped to the frame; v1 = p(y0,x0) + (p(y0,x0+1) - p(y0,x0))*dx, v2 the same on
            row y0+1 when that row is inside the frame, else v1; v = v1 + (v2-v1)*dy; the byte is v truncated.
  nearest   xs = X < 0 ? -1 : int(X), ys likewise; 0 outside the frame, else the source value.
"""
import importlib.util
import os
import random
import sys
from types import SimpleNamespace

import numpy as np
from PIL import Image

import io_oracle as IO
from bts_b200 import data


def _source_points(coeffs, Hs, Ws):
    a, b, c, d, e, f = (np.float64(v) for v in coeffs)
    yi, xi = np.mgrid[0:Hs, 0:Ws].astype(np.float64)
    xi += 0.5
    yi += 0.5
    return (a * xi + b * yi) + c, (d * xi + e * yi) + f


def rotate_bilinear_u8(frame, coeffs):
    """Image.rotate(angle, resample=BILINEAR) of an (Hs,Ws,3) uint8 frame, coeffs = bts_b200.data.rotate_affine(angle)"""
    Hs, Ws = frame.shape[:2]
    X, Y = _source_points(coeffs, Hs, Ws)
    inside = (X >= 0) & (X < Ws) & (Y >= 0) & (Y < Hs)
    X = X - 0.5
    Y = Y - 0.5
    x0 = np.floor(X).astype(np.int64)
    y0 = np.floor(Y).astype(np.int64)
    dx = (X - x0)[..., None]
    dy = (Y - y0)[..., None]
    xa, xb = np.clip(x0, 0, Ws - 1), np.clip(x0 + 1, 0, Ws - 1)
    ya = np.clip(y0, 0, Hs - 1)
    p = frame.astype(np.int64)
    v1 = p[ya, xa] + (p[ya, xb] - p[ya, xa]) * dx
    y1 = y0 + 1
    row1 = (y1 >= 0) & (y1 < Hs)
    yb = np.clip(y1, 0, Hs - 1)
    v2 = np.where(row1[..., None], p[yb, xa] + (p[yb, xb] - p[yb, xa]) * dx, v1)
    v = v1 + (v2 - v1) * dy
    out = np.trunc(v).astype(np.uint8)
    out[~inside] = 0
    return out


def rotate_nearest(frame, coeffs):
    """Image.rotate(angle, resample=NEAREST) of an (Hs,Ws) frame (the uint16 depth, mode I;16)"""
    Hs, Ws = frame.shape[:2]
    X, Y = _source_points(coeffs, Hs, Ws)
    xs = np.where(X < 0, -1, np.trunc(np.maximum(X, -1.0))).astype(np.int64)
    ys = np.where(Y < 0, -1, np.trunc(np.maximum(Y, -1.0))).astype(np.int64)
    inside = (xs >= 0) & (xs < Ws) & (ys >= 0) & (ys < Hs)
    out = frame[np.clip(ys, 0, Hs - 1), np.clip(xs, 0, Ws - 1)]
    out[~inside] = 0
    return out


def input_prep(img_u8, depth_u16, depth_div, y0, x0, H, W, flip, augment, gamma, brightness, colors, coeffs=None):
    """io_oracle.input_prep after the reference's rotation of the whole (fixed-cropped) frame (bts_dataloader.py:122-125)"""
    if coeffs is not None:
        img_u8 = rotate_bilinear_u8(img_u8, coeffs)
        if depth_u16 is not None:
            depth_u16 = rotate_nearest(depth_u16, coeffs)
    return IO.input_prep(img_u8, depth_u16, depth_div, y0, x0, H, W, flip, augment, gamma, brightness, colors)


# ------------------------------------------------------------------ seeded samples of the reference loader
# The unmodified pytorch/bts_dataloader.py (copied into oracle/_ref by `make -C oracle`, absent elsewhere) and the host side
# of the GPU transform (bts_b200.data) on the same synthetic PNG set and the same seeds.
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_DIR = os.path.join(ROOT, "oracle", "_ref")
REF_LOADER = os.path.join(REF_DIR, "bts_dataloader.py")


def reference_loader():
    """the unmodified pytorch/bts_dataloader.py that `make -C oracle` copies into oracle/_ref, or None"""
    if not os.path.isfile(REF_LOADER):
        return None
    sys.path.insert(0, REF_DIR)
    try:
        spec = importlib.util.spec_from_file_location("_ref_bts_dataloader", REF_LOADER)
        mod = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(mod)
    finally:
        sys.path.remove(REF_DIR)
    return mod


CASES = {
    # dataset: (raw frame h, w), (input_height, input_width), depth scale, degree (the recipes': eigen 1.0, nyu 2.5)
    "kitti": ((375, 1242), (352, 704), 256.0, 1.0),
    "nyu": ((480, 640), (416, 544), 1000.0, 2.5),
}


def make_dataset(root, dataset, n=2):
    """n synthetic samples as the loader reads them: RGB PNG + 16-bit depth PNG (left and right camera for KITTI), and the
    file list `image depth focal [right_image right_depth]`"""
    (h, w), _, _, _ = CASES[dataset]
    rng = np.random.RandomState(7)
    lines = []
    for i in range(n):
        names = []
        for cam in ("l", "r"):
            img = rng.randint(0, 256, (h, w, 3)).astype(np.uint8)
            dep = rng.randint(1, 65536, (h, w)).astype(np.uint16)
            dep[rng.uniform(size=(h, w)) < 0.3] = 0
            Image.fromarray(img).save(os.path.join(root, "%s_%d_img.png" % (cam, i)))
            Image.fromarray(dep).save(os.path.join(root, "%s_%d_dep.png" % (cam, i)))
            names.append(("%s_%d_img.png" % (cam, i), "%s_%d_dep.png" % (cam, i)))
        lines.append("%s %s 721.5377 %s %s" % (names[0][0], names[0][1], names[1][0], names[1][1]))
    with open(os.path.join(root, "files.txt"), "w") as f:
        f.write("\n".join(lines) + "\n")
    return lines


def reference_args(root, dataset, degree=None):
    _, (H, W), _, deg = CASES[dataset]
    return SimpleNamespace(dataset=dataset, use_right=dataset == "kitti", data_path=root, gt_path=root,
                           filenames_file=os.path.join(root, "files.txt"), do_kb_crop=dataset == "kitti",
                           do_random_rotate=True, degree=deg if degree is None else degree, input_height=H, input_width=W)


def our_sample(args, line, seed):
    """the GPU transform's inputs for one sample, drawn and laid out on the host: the fixed-cropped uint8 / uint16 frames,
    the params row and the rotation angle (what ops.input_prep takes), from the same seeds as the reference"""
    random.seed(seed)
    np.random.seed(seed)
    f = line.split()
    _, (H, W), _, _ = CASES[args.dataset]
    w, h = Image.open(os.path.join(args.data_path, f[0])).size
    frame_hw = data.fixed_crop(np.empty((h, w), np.uint8), args.dataset, args.do_kb_crop).shape
    params, angle, right = data.draw_train_sample(args.dataset, frame_hw, (H, W), args.do_random_rotate, args.degree,
                                                  args.use_right)
    img_name, dep_name = (f[3], f[4]) if right else (f[0], f[1])
    img = data.fixed_crop(np.asarray(Image.open(os.path.join(args.data_path, img_name))), args.dataset, args.do_kb_crop)
    dep = data.fixed_crop(np.asarray(Image.open(os.path.join(args.gt_path, dep_name))), args.dataset, args.do_kb_crop)
    return img, dep, params, angle, right


def reference_sample(mod, args, idx, seed):
    """DataLoadPreprocess(args, 'train')[idx] of the reference loader module `mod`, from `seed`: (image, depth)"""
    random.seed(seed)
    np.random.seed(seed)
    ds = mod.DataLoadPreprocess(args, "train", transform=mod.preprocessing_transforms("train"))
    s = ds[idx]
    return s["image"].numpy(), s["depth"].numpy()
