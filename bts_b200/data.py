"""Host side of the GPU training transform (ops.input_prep): the reference loader's random decisions and geometry, drawn
and laid out on the CPU so that a seeded run reproduces DataLoadPreprocess.__getitem__ (train mode) of
pytorch/bts_dataloader.py:94-138 sample for sample.

  fixed_crop          the KB crop (:109-115) and NYU's blank-border crop (:118-120) as slices of decoded frames
  rotate_affine       the six inverse-map coefficients Pillow's Image.rotate hands to Image.transform (:187-189)
  draw_train_sample   one sample's random draws in the reference's call order -> (params row, angle, use_right)

Decoding stays on the CPU with PIL, as in the reference.  Everything here is plain Python / numpy; the sampling itself runs
in bts_input_prep_rotated (csrc/io.cu).
"""
import math
import random

import numpy as np

KB_HW = (352, 1216)
NYU_BOX = (43, 45, 608, 472)        # PIL box (left, upper, right, lower)


def fixed_crop(frame, dataset, do_kb_crop=False):
    """The reference's fixed crops, applied to a decoded (H,W) or (H,W,C) array, in its order: the KB crop when
    `do_kb_crop`, then NYU's (43, 45, 608, 472) box when `dataset == 'nyu'`.  The result is the frame that gets rotated:
    PIL rotates the cropped image about its own centre and fills outside its own bounds."""
    frame = np.asarray(frame)
    if do_kb_crop:
        height, width = frame.shape[:2]
        if height < KB_HW[0] or width < KB_HW[1]:
            raise ValueError("KB crop needs a frame of at least %dx%d, got %dx%d" % (*KB_HW, height, width))
        top_margin = int(height - 352)
        left_margin = int((width - 1216) / 2)
        frame = frame[top_margin:top_margin + 352, left_margin:left_margin + 1216]
    if dataset == "nyu":
        left, upper, right, lower = NYU_BOX
        if frame.shape[0] < lower or frame.shape[1] < right:
            raise ValueError("NYU crop needs a frame of at least %dx%d, got %dx%d" % (lower, right, *frame.shape[:2]))
        frame = frame[upper:lower, left:right]
    return frame


def rotate_affine(angle, w, h):
    """The inverse map (a, b, c, d, e, f) that Image.rotate(angle) of a w x h image passes to Image.transform: output
    pixel (x, y) samples the source at (a*(x+.5) + b*(y+.5) + c, d*(x+.5) + e*(y+.5) + f).  Pillow's own expressions,
    in its order (PIL/Image.py, Image.rotate, no centre / translate / expand).  Where Pillow takes a fast path instead
    (angle % 360 in 0, 180, or 90 / 270 on a square image) these coefficients are exact integers and half-integers, and
    sampling with them gives the same pixels."""
    angle = float(angle)
    if not math.isfinite(angle):
        raise ValueError("rotation angle must be finite, got %r" % angle)
    angle = angle % 360.0
    center = (w / 2, h / 2)
    angle = -math.radians(angle)
    matrix = [
        round(math.cos(angle), 15),
        round(math.sin(angle), 15),
        0.0,
        round(-math.sin(angle), 15),
        round(math.cos(angle), 15),
        0.0,
    ]

    def transform(x, y, matrix):
        a, b, c, d, e, f = matrix
        return a * x + b * y + c, d * x + e * y + f

    matrix[2], matrix[5] = transform(-center[0], -center[1], matrix)
    matrix[2] += center[0]
    matrix[5] += center[1]
    return matrix


def draw_train_sample(dataset, frame_hw, out_hw, do_random_rotate=False, degree=2.5, use_right=False):
    """One training sample's random decisions, drawn from the global `random` / `np.random` states in the order
    DataLoadPreprocess.__getitem__ consumes them (bts_dataloader.py:99,123,196-197,204,210,218-229):
    use_right (KITTI with use_right only), the rotation angle (when rotating), crop x then y, flip, augment, and when
    augmenting gamma, brightness (0.75-1.25 for NYU, 0.9-1.1 otherwise) and the three np.random colours.

    frame_hw is the (height, width) of the frame after the fixed crops (the frame that is rotated and then randomly
    cropped); out_hw is (input_height, input_width).  Returns (params, angle, use_right): params is the (9,) float32 row
    of ops.input_prep (y0, x0, flip, augment, gamma, brightness, colour r, g, b), angle is in degrees (0.0 when not
    rotating), use_right says whether to load the right camera's files (kitti only)."""
    Hs, Ws = frame_hw
    H, W = out_hw
    if Hs < H or Ws < W:
        raise ValueError("the crop %dx%d does not fit the frame %dx%d" % (H, W, Hs, Ws))
    right = dataset == "kitti" and use_right is True and random.random() > 0.5
    angle = 0.0
    if do_random_rotate is True:
        angle = (random.random() - 0.5) * 2 * degree
    x = random.randint(0, Ws - W)
    y = random.randint(0, Hs - H)
    do_flip = random.random()
    do_augment = random.random()
    gamma = brightness = 1.0
    colors = np.ones(3)
    if do_augment > 0.5:
        gamma = random.uniform(0.9, 1.1)
        if dataset == "nyu":
            brightness = random.uniform(0.75, 1.25)
        else:
            brightness = random.uniform(0.9, 1.1)
        colors = np.random.uniform(0.9, 1.1, size=3)
    params = np.array([y, x, do_flip > 0.5, do_augment > 0.5, gamma, brightness, *colors], dtype=np.float32)
    return params, angle, right
