"""TEST INFRASTRUCTURE ONLY -- a small PNG encoder that chooses each row's filter type, the zlib strategy and the IDAT chunking
(Pillow never writes the Average filter), a numpy row unfilter, and the serial host build of the decode core
(bts_b200/csrc/png_core.cuh) under AddressSanitizer / UBSan as a subprocess."""
import os
import struct
import subprocess
import zlib

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
STRATEGIES = {"default": zlib.Z_DEFAULT_STRATEGY, "filtered": zlib.Z_FILTERED, "huffman_only": zlib.Z_HUFFMAN_ONLY,
              "rle": zlib.Z_RLE, "fixed": zlib.Z_FIXED}


def _paeth(a, b, c):
    p = a + b - c
    pa, pb, pc = np.abs(p - a), np.abs(p - b), np.abs(p - c)
    return np.where((pa <= pb) & (pa <= pc), a, np.where(pb <= pc, b, c))


def scanlines(arr, filters):
    """arr: (H, W, 3) uint8 or (H, W) uint16 -> filtered scanlines bytes (big-endian 16-bit samples)"""
    if arr.dtype == np.uint16:
        rows, bpp = arr.astype(">u2").view(np.uint8).reshape(arr.shape[0], -1), 2
    else:
        rows, bpp = arr.reshape(arr.shape[0], -1), 3
    x = rows.astype(np.int32)
    H, n = x.shape
    a = np.zeros_like(x)
    a[:, bpp:] = x[:, :-bpp]
    b = np.zeros_like(x)
    b[1:] = x[:-1]
    c = np.zeros_like(x)
    c[1:, bpp:] = x[:-1, :-bpp]
    pred = {0: np.zeros_like(x), 1: a, 2: b, 3: (a + b) >> 1, 4: _paeth(a, b, c)}
    out = np.empty((H, n + 1), dtype=np.uint8)
    for r in range(H):
        f = int(filters[r])
        out[r, 0] = f
        out[r, 1:] = ((x[r] - pred[f][r]) & 255).astype(np.uint8)
    return out.tobytes()


def _chunk(kind, body):
    return struct.pack(">I", len(body)) + kind + body + struct.pack(">I", zlib.crc32(body, zlib.crc32(kind)))


def encode_png(arr, filters=None, level=6, strategy="default", idat_chunk=None, wbits=15, seed=0):
    """filters: None (all 0), an int for every row, 'mix' (a seeded per-row mix of 0-4) or a per-row sequence.
    idat_chunk: None for one IDAT, else the payload size of each IDAT chunk."""
    H, W = arr.shape[:2]
    if filters is None:
        filters = 0
    if isinstance(filters, str):
        filters = np.random.RandomState(seed).randint(0, 5, H)
    elif np.isscalar(filters):
        filters = [int(filters)] * H
    colour, depth = (2, 8) if arr.dtype == np.uint8 else (0, 16)
    co = zlib.compressobj(level, zlib.DEFLATED, wbits, 8, STRATEGIES[strategy])
    z = co.compress(scanlines(arr, filters)) + co.flush()
    parts = [z] if idat_chunk is None else [z[i:i + idat_chunk] for i in range(0, len(z), idat_chunk)]
    return (b"\x89PNG\r\n\x1a\n" + _chunk(b"IHDR", struct.pack(">IIBBBBB", W, H, depth, colour, 0, 0, 0))
            + b"".join(_chunk(b"IDAT", p) for p in parts) + _chunk(b"IEND", b""))


def unfilter_reference(raw, H, W, bpp):
    """numpy restatement of the PNG row unfilter (filters 0-4): raw scanlines -> (H, W*bpp) uint8, or None on a filter > 4"""
    n = W * bpp
    rows = np.frombuffer(raw, dtype=np.uint8).reshape(H, n + 1).astype(np.int32)
    out = np.zeros((H, n), dtype=np.int32)
    prev = np.zeros(n, dtype=np.int32)
    for r in range(H):
        f, x = rows[r, 0], rows[r, 1:]
        if f > 4:
            return None
        if f == 0:
            cur = x.copy()
        elif f == 1:
            cur = np.cumsum(x.reshape(W, bpp), axis=0).reshape(-1) & 255
        elif f == 2:
            cur = (x + prev) & 255
        else:
            cur = x.copy()
            for j in range(n):
                a = cur[j - bpp] if j >= bpp else 0
                c = prev[j - bpp] if j >= bpp else 0
                cur[j] = (x[j] + ((a + prev[j]) >> 1 if f == 3 else int(_paeth(a, prev[j], c)))) & 255
        out[r] = cur
        prev = cur
    return out.astype(np.uint8)


# ------------------------------------------------------------------ the core's serial host build, sanitized
HARNESS = r'''
#include <cstdio>
#include <cstring>
#include <vector>
#include "png_core.cuh"

// serial executor: writes into a buffer of exactly the expected size and trusts the commands, as the GPU executor does
struct Exec {
    const uint8_t *src;
    uint8_t *out;
    uint32_t pos = 0;
    void literal(uint8_t b) { out[pos++] = b; }
    void match(uint32_t len, uint32_t d) { for (uint32_t k = 0; k < len; ++k, ++pos) out[pos] = out[pos - d]; }
    void stored(uint32_t at, uint32_t len) { memcpy(out + pos, src + at, len); pos += len; }
};

static bool rd(void *p, size_t n) { return fread(p, 1, n, stdin) == n; }

int main() {
    // records: u32 mode (0 inflate, 1 unfilter), u32 len, u32 a, u32 b, payload[len]
    //   inflate:  a = expected size;  out: i32 status, u32 n, bytes[n]
    //   unfilter: a = height, b = width * 16 + bpp;  out: i32 status, u32 n, bytes[n]
    uint32_t hdr[4];
    while (rd(hdr, sizeof hdr)) {
        uint8_t *in = new uint8_t[hdr[1] ? hdr[1] : 1];
        if (hdr[1] && !rd(in, hdr[1])) return 2;
        int st;
        uint32_t n = 0;
        uint8_t *out = nullptr;
        if (hdr[0] == 0) {
            out = new uint8_t[hdr[2] ? hdr[2] : 1];
            Exec ex{in, out};
            uint32_t adler;
            st = bts_png::inflate_serial(in, hdr[1], hdr[2], ex, adler);
            if (!st && bts_png::adler32(out, hdr[2]) != adler) st = BTS_PNG_ADLER_MISMATCH;
            n = st ? 0 : hdr[2];
        } else {
            const int H = (int)hdr[2], W = (int)(hdr[3] >> 4), bpp = (int)(hdr[3] & 15), rb = W * bpp;
            out = new uint8_t[(size_t)H * rb + 1];
            std::vector<uint8_t> zero(rb, 0);
            st = BTS_PNG_OK;
            for (int r = 0; r < H && !st; ++r) {
                uint8_t *cur = out + (size_t)r * rb;
                memcpy(cur, in + (size_t)r * (rb + 1) + 1, rb);
                st = bts_png::unfilter_row(in[(size_t)r * (rb + 1)], cur, r ? cur - rb : zero.data(), rb, bpp);
            }
            n = st ? 0 : (uint32_t)(H * rb);
        }
        fwrite(&st, 4, 1, stdout);
        fwrite(&n, 4, 1, stdout);
        if (n) fwrite(out, 1, n, stdout);
        delete[] in;
        delete[] out;
    }
    return 0;
}
'''


def build_harness(tmpdir):
    src = os.path.join(tmpdir, "png_harness.cpp")
    exe = os.path.join(tmpdir, "png_harness")
    with open(src, "w") as f:
        f.write(HARNESS)
    subprocess.run(["g++", "-std=c++17", "-O1", "-g", "-fsanitize=address,undefined", "-fno-sanitize-recover=all",
                    "-fno-omit-frame-pointer", "-I", os.path.join(ROOT, "bts_b200", "csrc"), src, "-o", exe],
                   check=True, capture_output=True)
    return exe


def run_harness(exe, records):
    """records: (mode, payload, a, b) -> [(status, bytes)]; fails on any sanitizer report"""
    blob = b"".join(struct.pack("<4I", m, len(p), a, b) + p for m, p, a, b in records)
    env = dict(os.environ, ASAN_OPTIONS="detect_leaks=1:abort_on_error=0", UBSAN_OPTIONS="print_stacktrace=1")
    r = subprocess.run([exe], input=blob, capture_output=True, env=env)
    err = r.stderr.decode(errors="replace")
    assert r.returncode == 0 and "Sanitizer" not in err and "runtime error" not in err, err[-4000:]
    out, pos, res = r.stdout, 0, []
    for _ in records:
        st, n = struct.unpack_from("<iI", out, pos)
        res.append((st, out[pos + 8:pos + 8 + n]))
        pos += 8 + n
    assert pos == len(out)
    return res


def _bits_lsb(fields):
    """(value, nbits, msb_first) fields -> bytes, DEFLATE bit order (Huffman codes are written MSB first)"""
    acc = n = 0
    for v, k, msb in fields:
        if msb:
            v = int(format(v, "0%db" % k)[::-1], 2)
        acc |= v << n
        n += k
    return acc.to_bytes((n + 7) // 8, "little")


def png_from_stream(stream, H, W, bpp=3):
    colour, depth = (2, 8) if bpp == 3 else (0, 16)
    return (b"\x89PNG\r\n\x1a\n" + _chunk(b"IHDR", struct.pack(">IIBBBBB", W, H, depth, colour, 0, 0, 0))
            + _chunk(b"IDAT", stream) + _chunk(b"IEND", b""))


def malformed_cases():
    """name -> (PNG bytes, height, width, expected BTS_PNG_* status).  Every one is valid at the container level; the
    CPU tests run their zlib streams through the sanitized core, the GPU tests through decode_png."""
    H, W = 6, 5
    arr = np.random.RandomState(3).randint(0, 256, (H, W, 3)).astype(np.uint8)
    raw = scanlines(arr, [0, 1, 2, 3, 4, 1])
    z = zlib.compress(raw, 6)
    bad_filter = bytearray(raw)
    bad_filter[(W * 3 + 1) * 2] = 5
    # fixed-Huffman block whose first symbol is a match: length 3 (code 257 = 0000001), distance code 0 (distance 1)
    far = b"\x78\x9c" + _bits_lsb([(1, 1, False), (1, 2, False), (1, 7, True), (0, 5, True), (0, 7, True)]) + b"\0\0\0\1"
    return {
        "truncated": (png_from_stream(z[:len(z) // 2], H, W), H, W, 1),
        "adler": (png_from_stream(z[:-1] + bytes([z[-1] ^ 1]), H, W), H, W, 7),
        "filter5": (png_from_stream(zlib.compress(bytes(bad_filter)), H, W), H, W, 8),
        "zlib_header": (png_from_stream(b"\x79" + z[1:], H, W), H, W, 2),
        "distance": (png_from_stream(far, H, W), H, W, 5),
    }
