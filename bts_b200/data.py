"""Host side of the GPU training transform (ops.input_prep): the reference loader's random decisions and geometry, drawn
and laid out on the CPU so that a seeded run reproduces DataLoadPreprocess.__getitem__ (train mode) of
pytorch/bts_dataloader.py:94-138 sample for sample.

  fixed_crop_box      the KB crop (:109-115) and NYU's blank-border crop (:118-120) as one window (y0, x0, Hc, Wc)
  fixed_crop          that window as a slice of a decoded frame
  parse_png           the PNG container checks of ops.decode_png (signature, chunk CRCs, IHDR / IEND, the formats the
                      device decoder takes) and the file's zlib stream
  rotate_affine       the six inverse-map coefficients Pillow's Image.rotate hands to Image.transform (:187-189)
  draw_train_sample   one sample's random draws in the reference's call order -> (params row, angle, use_right)

Everything here is plain Python / numpy; the sampling itself runs in bts_input_prep_rotated (csrc/io.cu) and the decoding
of the training PNGs in bts_png_inflate / bts_png_unfilter (csrc/png.cu).
"""
import math
import random
import struct
import zlib

import numpy as np

KB_HW = (352, 1216)
NYU_BOX = (43, 45, 608, 472)        # PIL box (left, upper, right, lower)


def fixed_crop_box(dataset, do_kb_crop, h, w):
    """The reference's fixed crops of an h x w frame as one window (y0, x0, Hc, Wc), in its order: the KB crop when
    `do_kb_crop`, then NYU's (43, 45, 608, 472) box when `dataset == 'nyu'`."""
    y0, x0, Hc, Wc = 0, 0, h, w
    if do_kb_crop:
        if h < KB_HW[0] or w < KB_HW[1]:
            raise ValueError("KB crop needs a frame of at least %dx%d, got %dx%d" % (*KB_HW, h, w))
        y0, x0, Hc, Wc = int(h - 352), int((w - 1216) / 2), 352, 1216
    if dataset == "nyu":
        left, upper, right, lower = NYU_BOX
        if Hc < lower or Wc < right:
            raise ValueError("NYU crop needs a frame of at least %dx%d, got %dx%d" % (lower, right, Hc, Wc))
        y0, x0, Hc, Wc = y0 + upper, x0 + left, lower - upper, right - left
    return y0, x0, Hc, Wc


def fixed_crop(frame, dataset, do_kb_crop=False):
    """The reference's fixed crops (fixed_crop_box) applied to a decoded (H,W) or (H,W,C) array.  The result is the frame
    that gets rotated: PIL rotates the cropped image about its own centre and fills outside its own bounds."""
    frame = np.asarray(frame)
    y0, x0, Hc, Wc = fixed_crop_box(dataset, do_kb_crop, *frame.shape[:2])
    return frame[y0:y0 + Hc, x0:x0 + Wc]


# ------------------------------------------------------------------ PNG container (ops.decode_png)
PNG_SIGNATURE = b"\x89PNG\r\n\x1a\n"
PNG_MAX_ROW_BYTES = 16384          # BTS_PNG_MAX_ROW_BYTES: bts_png_unfilter keeps two rows in shared memory
PNG_MAX_RAW_BYTES = 1 << 28        # per image, height * (1 + width * bpp)
# (colour type, bit depth) -> (format name, bytes per pixel) of the formats the device decoder takes
PNG_FORMATS = {(2, 8): ("RGB8", 3), (0, 16): ("Gray16", 2)}
_COLOUR_TYPES = {0: "grayscale", 2: "RGB", 3: "palette", 4: "grayscale+alpha", 6: "RGBA"}


def parse_png(blob):
    """Checks one PNG file's container and returns (format, bpp, height, width, zlib stream).

    Checked: the signature; the chunk walk, every chunk's CRC-32; IHDR first, IEND present, at least one IDAT; a format
    the device decoder takes (8-bit RGB or 16-bit grayscale, non-interlaced).  Everything else raises ValueError naming
    what is wrong.  The IDAT payloads are concatenated into the file's one zlib stream."""
    b = memoryview(blob).cast("B")
    if bytes(b[:8]) != PNG_SIGNATURE:
        raise ValueError("not a PNG file: bad signature")
    pos, ihdr, idat, iend = 8, None, [], False
    while pos < len(b):
        if pos + 12 > len(b):
            raise ValueError("truncated PNG chunk at byte %d" % pos)
        length, ctype = struct.unpack(">I4s", b[pos:pos + 8])
        end = pos + 12 + length
        if length > 0x7fffffff or end > len(b):
            raise ValueError("truncated PNG chunk %r at byte %d" % (ctype, pos))
        body = b[pos + 8:pos + 8 + length]
        (crc,) = struct.unpack(">I", b[end - 4:end])
        if zlib.crc32(body, zlib.crc32(ctype)) != crc:
            raise ValueError("CRC mismatch in PNG chunk %r at byte %d" % (ctype.decode("latin-1"), pos))
        if ihdr is None and ctype != b"IHDR":
            raise ValueError("PNG chunk IHDR must come first, found %r" % ctype.decode("latin-1"))
        if ctype == b"IHDR":
            if ihdr is not None or length != 13:
                raise ValueError("malformed PNG IHDR chunk")
            ihdr = struct.unpack(">IIBBBBB", body)
        elif ctype == b"IDAT":
            idat.append(body)
        elif ctype == b"IEND":
            iend = True
            break
        pos = end
    if ihdr is None:
        raise ValueError("PNG has no IHDR chunk")
    if not iend:
        raise ValueError("PNG has no IEND chunk")
    width, height, depth, colour, compression, filt, interlace = ihdr
    if width == 0 or height == 0:
        raise ValueError("PNG has zero width or height (%dx%d)" % (width, height))
    if compression != 0 or filt != 0:
        raise ValueError("PNG compression method %d / filter method %d is not defined" % (compression, filt))
    if (colour, depth) not in PNG_FORMATS:
        raise ValueError("unsupported PNG format: %d-bit %s (the decoder takes 8-bit RGB and 16-bit grayscale)"
                         % (depth, _COLOUR_TYPES.get(colour, "colour type %d" % colour)))
    if interlace != 0:
        raise ValueError("unsupported PNG format: Adam7 interlaced")
    name, bpp = PNG_FORMATS[(colour, depth)]
    if width * bpp > PNG_MAX_ROW_BYTES:
        raise ValueError("PNG rows of %d bytes are wider than the decoder's %d" % (width * bpp, PNG_MAX_ROW_BYTES))
    if height * (1 + width * bpp) > PNG_MAX_RAW_BYTES:
        raise ValueError("PNG of %dx%d is larger than the decoder's %d decompressed bytes" % (height, width,
                                                                                              PNG_MAX_RAW_BYTES))
    if not idat:
        raise ValueError("PNG has no IDAT chunk")
    return name, bpp, height, width, b"".join(idat)


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
