"""CPU tests of the batched PNG decoder (no GPU): the host container parser and crop box (bts_b200.data), the decode core
(csrc/png_core.cuh) built serially with AddressSanitizer / UBSan against zlib and a numpy unfilter, and the kernels'
resources in the built library."""
import io
import os
import random
import re
import shutil
import subprocess
import zlib

import numpy as np
import pytest
from PIL import Image

import png_testutil as PT
from bts_b200 import data

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "bts_b200", "libbts_b200.so")


def _rgb_png(H=4, W=3):
    return PT.encode_png(np.random.RandomState(0).randint(0, 256, (H, W, 3)).astype(np.uint8))


def _chunks(blob):
    out, pos = [], 8
    while pos < len(blob):
        n = int.from_bytes(blob[pos:pos + 4], "big")
        out.append((blob[pos + 4:pos + 8], blob[pos + 8:pos + 8 + n]))
        pos += 12 + n
    return out


def _rebuild(chunks):
    return b"\x89PNG\r\n\x1a\n" + b"".join(PT._chunk(k, b) for k, b in chunks)


# ------------------------------------------------------------------ container parser
def test_parser_accepts_the_two_formats():
    name, bpp, h, w, z = data.parse_png(_rgb_png(4, 3))
    assert (name, bpp, h, w) == ("RGB8", 3, 4, 3) and len(zlib.decompress(z)) == 4 * (1 + 9)
    buf = io.BytesIO()
    Image.fromarray(np.arange(12, dtype=np.uint16).reshape(3, 4) * 5000).save(buf, format="PNG")
    assert data.parse_png(buf.getvalue())[:4] == ("Gray16", 2, 3, 4)


@pytest.mark.parametrize("mutate,match", [
    (lambda b: b"\x89PNG\r\n\x1a\x00" + b[8:], "signature"),
    (lambda b: b[:20] + bytes([b[20] ^ 1]) + b[21:], "CRC mismatch"),
    (lambda b: _rebuild([c for c in _chunks(b) if c[0] != b"IHDR"]), "IHDR"),
    (lambda b: _rebuild([c for c in _chunks(b) if c[0] != b"IEND"]), "IEND"),
    (lambda b: _rebuild([c for c in _chunks(b) if c[0] != b"IDAT"]), "IDAT"),
    (lambda b: b[:-6], "truncated"),
])
def test_parser_rejects_broken_containers(mutate, match):
    with pytest.raises(ValueError, match=match):
        data.parse_png(mutate(_rgb_png()))


def _with_ihdr(w, h, depth, colour, interlace=0):
    chunks = _chunks(_rgb_png())
    chunks[0] = (b"IHDR", PT.struct.pack(">IIBBBBB", w, h, depth, colour, 0, 0, interlace))
    return _rebuild(chunks)


@pytest.mark.parametrize("depth,colour,interlace,match", [
    (8, 3, 0, "palette"), (8, 6, 0, "RGBA"), (8, 4, 0, "alpha"), (8, 0, 0, "8-bit grayscale"), (16, 2, 0, "16-bit RGB"),
    (8, 2, 1, "Adam7"), (1, 0, 0, "1-bit grayscale"),
])
def test_parser_names_unsupported_formats(depth, colour, interlace, match):
    with pytest.raises(ValueError, match=match):
        data.parse_png(_with_ihdr(3, 4, depth, colour, interlace))


@pytest.mark.parametrize("w,h", [(0, 4), (3, 0)])
def test_parser_rejects_zero_size(w, h):
    with pytest.raises(ValueError, match="zero width or height"):
        data.parse_png(_with_ihdr(w, h, 8, 2))


def test_parser_rejects_rows_wider_than_the_unfilter_holds():
    with pytest.raises(ValueError, match="wider"):
        data.parse_png(_with_ihdr(data.PNG_MAX_ROW_BYTES // 3 + 1, 2, 8, 2))


def test_decode_png_validates_the_batch_before_cuda():
    from bts_b200 import ops
    gray = PT.encode_png(np.zeros((4, 3), np.uint16))
    with pytest.raises(ValueError, match="one format per call"):
        ops.decode_png([_rgb_png(), gray])
    with pytest.raises(ValueError, match="same size"):
        ops.decode_png([_rgb_png(4, 3), _rgb_png(5, 3)])
    with pytest.raises(ValueError, match="image 1: the crop"):
        ops.decode_png([_rgb_png(4, 3), _rgb_png(4, 3)], origins=[(0, 0), (1, 1)], out_hw=(4, 2))
    with pytest.raises(ValueError, match="outside"):
        ops.decode_png([_rgb_png(4, 3)], origins=[(0, 0)], out_hw=(0, 3))
    with pytest.raises(ValueError, match="one \\(y0, x0\\) per image"):
        ops.decode_png([_rgb_png(4, 3)], origins=[(0, 0), (0, 0)], out_hw=(1, 1))


@pytest.mark.parametrize("h,w", [(375, 1242), (376, 1241), (370, 1224), (374, 1238), (370, 1226)])
def test_fixed_crop_box_matches_fixed_crop_kitti(h, w):
    frame = np.arange(h * w, dtype=np.int64).reshape(h, w)
    y0, x0, Hc, Wc = data.fixed_crop_box("kitti", True, h, w)
    np.testing.assert_array_equal(frame[y0:y0 + Hc, x0:x0 + Wc], data.fixed_crop(frame, "kitti", True))
    assert (Hc, Wc) == (352, 1216)
    assert data.fixed_crop_box("kitti", False, h, w) == (0, 0, h, w)


def test_fixed_crop_box_matches_fixed_crop_nyu():
    frame = np.arange(480 * 640, dtype=np.int64).reshape(480, 640)
    y0, x0, Hc, Wc = data.fixed_crop_box("nyu", False, 480, 640)
    assert (y0, x0, Hc, Wc) == (45, 43, 427, 565)
    np.testing.assert_array_equal(frame[y0:y0 + Hc, x0:x0 + Wc], data.fixed_crop(frame, "nyu", False))
    with pytest.raises(ValueError, match="KB crop"):
        data.fixed_crop_box("kitti", True, 300, 1242)


# ------------------------------------------------------------------ the decode core under sanitizers
@pytest.fixture(scope="module")
def harness(tmp_path_factory):
    if shutil.which("g++") is None:
        pytest.skip("g++ not found")
    return PT.build_harness(str(tmp_path_factory.mktemp("png_harness")))


def _zlib_result(stream, expected_len):
    """zlib's verdict: the stream decodes to its end (Adler-32 checked) with exactly expected_len bytes"""
    try:
        d = zlib.decompressobj()
        out = d.decompress(stream)
    except zlib.error:
        return None
    return out if d.eof and len(out) == expected_len else None


def _payloads():
    rng = np.random.RandomState(1)
    yy, xx = np.mgrid[0:40, 0:57]
    smooth = ((np.sin(yy / 7.0) + np.cos(xx / 5.0)) * 60 + 128)[..., None] + rng.randint(0, 6, (40, 57, 3))
    img = np.clip(smooth, 0, 255).astype(np.uint8)
    dep = (rng.uniform(size=(23, 31)) < 0.2) * rng.randint(1, 65536, (23, 31))
    return {
        "rgb_mix": PT.scanlines(img, np.random.RandomState(2).randint(0, 5, 40)),
        "gray16_sparse": PT.scanlines(dep.astype(np.uint16), [0] * 23),
        "rgb_1x1": PT.scanlines(np.array([[[1, 2, 3]]], np.uint8), [0]),
        "gray16_2x3": PT.scanlines(np.arange(6, dtype=np.uint16).reshape(2, 3) * 9999, [1, 4]),
        "text": b"".join(b"row %d of a repetitive payload; " % (i % 17) for i in range(300)),
        "random": rng.randint(0, 256, 3000).astype(np.uint8).tobytes(),
    }


def _streams():
    cases = []
    for pname, p in _payloads().items():
        for level in range(10):
            for sname in PT.STRATEGIES:
                for wbits in range(9, 16):
                    co = zlib.compressobj(level, zlib.DEFLATED, wbits, 8, PT.STRATEGIES[sname])
                    cases.append(("%s/l%d/%s/w%d" % (pname, level, sname, wbits), co.compress(p) + co.flush(), p))
        # empty stored blocks from sync / full flushes, trailing bytes after the Adler-32
        co = zlib.compressobj(6)
        z = co.compress(p[:len(p) // 2]) + co.flush(zlib.Z_SYNC_FLUSH) + co.flush(zlib.Z_FULL_FLUSH)
        z += co.compress(p[len(p) // 2:]) + co.flush(zlib.Z_SYNC_FLUSH) + co.flush()
        cases.append(("%s/flushes" % pname, z, p))
        cases.append(("%s/trailing" % pname, zlib.compress(p, 9) + b"\x00garbage after the stream", p))
    # a stream of nothing but an empty final stored block, for an empty output
    cases.append(("empty_stored", b"\x78\x01\x01\x00\x00\xff\xff\x00\x00\x00\x01", b""))
    return cases


def test_core_inflate_matches_zlib(harness):
    cases = _streams()
    assert len(cases) > 2000
    res = PT.run_harness(harness, [(0, z, len(p), 0) for _, z, p in cases])
    for (name, z, p), (st, out) in zip(cases, res):
        assert st == 0, "%s: status %d" % (name, st)
        assert out == p, name


def test_core_unfilter_matches_numpy(harness):
    rng = np.random.RandomState(4)
    recs, want = [], []
    for bpp, arr in ((3, rng.randint(0, 256, (9, 13, 3)).astype(np.uint8)),
                     (2, rng.randint(0, 65536, (9, 11)).astype(np.uint16))):
        H, W = arr.shape[:2]
        expect = arr.astype(">u2").view(np.uint8).reshape(H, -1) if bpp == 2 else arr.reshape(H, -1)
        for filters in [[f] * H for f in range(5)] + [list(rng.randint(0, 5, H)) for _ in range(4)]:
            raw = PT.scanlines(arr, filters)
            ref = PT.unfilter_reference(raw, H, W, bpp)
            np.testing.assert_array_equal(ref, expect)
            recs.append((1, raw, H, W * 16 + bpp))
            want.append(expect.tobytes())
        bad = bytearray(PT.scanlines(arr, [0] * H))
        bad[(W * bpp + 1) * 3] = 5
        assert PT.unfilter_reference(bytes(bad), H, W, bpp) is None
        recs.append((1, bytes(bad), H, W * 16 + bpp))
        want.append(None)
    for (st, out), w in zip(PT.run_harness(harness, recs), want):
        if w is None:
            assert st == 8
        else:
            assert st == 0 and out == w


def _mutations(n, seed=5):
    rng = random.Random(seed)
    p = _payloads()
    fixed = zlib.compressobj(6, zlib.DEFLATED, 15, 8, zlib.Z_FIXED)
    bases = [zlib.compress(p["rgb_mix"], 6), zlib.compress(p["text"], 9), zlib.compress(p["gray16_sparse"], 1),
             fixed.compress(p["text"]) + fixed.flush(), zlib.compress(p["random"], 0)]
    sizes = [len(p["rgb_mix"]), len(p["text"]), len(p["gray16_sparse"]), len(p["text"]), len(p["random"])]
    out = []
    for i in range(n):
        k = i % len(bases)
        z = bytearray(bases[k])
        kind = rng.randrange(4)
        if kind == 0:
            z = z[:rng.randrange(len(z))]
        elif kind == 1:
            for _ in range(rng.randint(1, 3)):
                j = rng.randrange(len(z) * 8)
                z[j // 8] ^= 1 << (j % 8)
        elif kind == 2:
            for _ in range(rng.randint(1, 4)):
                z[rng.randrange(len(z))] = rng.randrange(256)
        else:
            j = rng.randrange(2)
            z[j] = rng.randrange(256)
            if rng.random() < 0.5:   # keep FCHECK valid so the edit reaches CM / CINFO / FDICT
                z[1] = (z[1] & 0xe0) | (31 - ((z[0] << 8) | (z[1] & 0xe0)) % 31) % 31
        out.append((bytes(z), sizes[k]))
    return out


def test_core_agrees_with_zlib_on_mutated_streams(harness):
    muts = _mutations(2400)
    res = PT.run_harness(harness, [(0, z, n, 0) for z, n in muts])
    n_ok = 0
    for i, ((z, n), (st, out)) in enumerate(zip(muts, res)):
        want = _zlib_result(z, n)
        if want is None:
            assert st != 0, "mutation %d: zlib fails, the core accepts" % i
        else:
            n_ok += 1
            assert st == 0 and out == want, "mutation %d: zlib decodes, the core returns status %d" % (i, st)
    assert 0 < n_ok < len(muts)


def test_core_on_the_malformed_inputs_of_the_gpu_tests(harness):
    for name, (blob, H, W, want) in PT.malformed_cases().items():
        _, bpp, h, w, z = data.parse_png(blob)
        st, raw = PT.run_harness(harness, [(0, z, H * (1 + W * bpp), 0)])[0]
        if want == 8:   # inflates cleanly; the row filter is what is wrong
            assert st == 0
            st = PT.run_harness(harness, [(1, raw, H, W * 16 + bpp)])[0][0]
        assert st == want, name


# ------------------------------------------------------------------ resources
def test_png_kernels_have_no_stack_frame():
    if not os.path.isfile(LIB):
        pytest.skip("libbts_b200.so is not built")
    exe = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.isfile(exe):
        pytest.skip("cuobjdump not found")
    out = subprocess.run([exe, "-res-usage", LIB], capture_output=True, text=True, check=True).stdout
    res, name = {}, None
    for line in out.splitlines():
        m = re.match(r"\s*Function (\S+):", line)
        if m:
            name = m.group(1)
            continue
        m = re.search(r"REG:(\d+) STACK:(\d+)", line)
        if m and name:
            for k in ("png_inflate_kernel", "png_unfilter_kernel"):
                if k in name:
                    res[k] = (int(m.group(1)), int(m.group(2)))
        name = None
    assert set(res) == {"png_inflate_kernel", "png_unfilter_kernel"}, res
    assert all(stack == 0 for _, stack in res.values()), res
