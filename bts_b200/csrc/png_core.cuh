// Decode core of the batched PNG decoder (csrc/png.cu): the zlib container (RFC 1950), DEFLATE (RFC 1951) and the PNG row
// unfilter, written once as __host__ __device__ code so that the GPU kernels and a serial host build share every
// validation.  Plain C++17; compiles under nvcc and g++ (the CPU tests build it with -fsanitize=address,undefined).
//
// The decoder never writes output itself.  It hands an emitter three commands, literal bytes, matches (length,
// distance) and stored runs (offset into the compressed stream, length), after it has checked them:
//   - a match's distance is <= the bytes produced so far;
//   - the output never grows past the expected size;
//   - a stored run lies inside the input.
// An executor can therefore copy without bounds checks of its own.  Malformed input only ever returns a BTS_PNG_* status.
//
// Huffman tables follow zlib's inflate_table: a root table indexed by the next `root` bits, whose entries are either a
// leaf {symbol, code length} or a link to a sub-table for the codes longer than `root`.  The code-length rules are zlib's
// (see table_plan); a code that passes them fits the zlib bounds ENOUGH_LENS (852, root 9) and ENOUGH_DISTS (592, root 6).
#pragma once

#include <stdint.h>

#include "../../include/bts_b200.h"

#if defined(__CUDACC__)
#define BTS_PNG_HD __host__ __device__ __forceinline__
#else
#define BTS_PNG_HD inline
#endif

namespace bts_png {

constexpr int CLEN_ROOT = 7, LITLEN_ROOT = 9, DIST_ROOT = 6;
constexpr int CLEN_ENOUGH = 128, LITLEN_ENOUGH = 852, DIST_ENOUGH = 592;
constexpr int KIND_CLEN = 0, KIND_LITLEN = 1, KIND_DIST = 2;

// table entry: 0 = no code; leaf = (len << 16) | symbol (len 1..15); link = 0x80000000 | (sub-table bits << 16) | offset
BTS_PNG_HD uint32_t leaf(int sym, int len) { return ((uint32_t)len << 16) | (uint32_t)sym; }

BTS_PNG_HD uint32_t reverse_bits(uint32_t v, int n) {
    uint32_t r = 0;
    for (int i = 0; i < n; ++i) {
        r = (r << 1) | (v & 1u);
        v >>= 1;
    }
    return r;
}

// LSB-first bit reader over [p, p + n).  Never loads outside the span; a read past its end fails.
struct BitReader {
    const uint8_t *p;
    uint32_t n, pos;   // pos: next byte to load into buf
    uint64_t buf;
    int cnt;           // valid bits in buf

    BTS_PNG_HD void init(const uint8_t *src, uint32_t len) {
        p = src;
        n = len;
        pos = 0;
        buf = 0;
        cnt = 0;
    }
    BTS_PNG_HD void fill() {
        while (cnt <= 56 && pos < n) {
            buf |= (uint64_t)p[pos++] << cnt;
            cnt += 8;
        }
    }
    BTS_PNG_HD bool bits(int k, uint32_t &v) {
        if (cnt < k) {
            fill();
            if (cnt < k) return false;
        }
        v = (uint32_t)(buf & ((1ull << k) - 1));
        buf >>= k;
        cnt -= k;
        return true;
    }
    BTS_PNG_HD void align() {
        const int r = cnt & 7;
        buf >>= r;
        cnt -= r;
    }
    // after align(): offset of the next unread byte
    BTS_PNG_HD uint32_t byte_pos() const { return pos - (uint32_t)(cnt >> 3); }
    BTS_PNG_HD void seek(uint32_t b) {
        pos = b;
        buf = 0;
        cnt = 0;
    }
};

// Decodes one symbol through a table built by build_table.  Near the end of the input the bits past it read as zeros;
// the code is accepted only when its own length fits the bits that exist.
BTS_PNG_HD int decode_sym(BitReader &br, const uint32_t *t, int root, int &sym) {
    if (br.cnt < 15) br.fill();
    uint32_t e = t[br.buf & ((1u << root) - 1)];
    if (e >> 31) e = t[(e & 0xffffu) + ((uint32_t)(br.buf >> root) & ((1u << ((e >> 16) & 15)) - 1))];
    const int len = (int)((e >> 16) & 15);
    if (len == 0) return BTS_PNG_BAD_CODE_TABLE;
    if (len > br.cnt) return BTS_PNG_TRUNCATED;
    br.buf >>= len;
    br.cnt -= len;
    sym = (int)(e & 0xffffu);
    return BTS_PNG_OK;
}

// Code-length counts -> canonical layout, with zlib's acceptance rules (inflate_table):
//   over-subscribed: error;  incomplete: error for the code-length code, and for the literal/length and distance codes
//   unless the code is a single code of length 1;  no codes at all: accepted for the distance code only.
// offs[len] = index of the first code of that length in (length, symbol) order; first[len] = its canonical code.
struct Plan {
    uint16_t count[16];
    uint16_t offs[16];
    uint32_t first[16];
    int max;
};

BTS_PNG_HD int table_plan(Plan &pl, int kind) {
    pl.count[0] = 0;
    int max = 15;
    while (max >= 1 && pl.count[max] == 0) --max;
    pl.max = max;
    if (max == 0) return kind == KIND_DIST ? BTS_PNG_OK : BTS_PNG_BAD_CODE_TABLE;
    int left = 1;
    for (int len = 1; len <= 15; ++len) {
        left <<= 1;
        left -= pl.count[len];
        if (left < 0) return BTS_PNG_BAD_CODE_TABLE;
    }
    if (left > 0 && (kind == KIND_CLEN || max != 1)) return BTS_PNG_BAD_CODE_TABLE;
    pl.offs[0] = pl.offs[1] = 0;
    for (int len = 1; len < 15; ++len) pl.offs[len + 1] = (uint16_t)(pl.offs[len] + pl.count[len]);
    uint32_t code = 0;
    pl.first[0] = 0;
    for (int len = 1; len <= 15; ++len) {
        code = (code + pl.count[len - 1]) << 1;
        pl.first[len] = code;
    }
    return BTS_PNG_OK;
}

// Root-table entries of the code at sorted index i (symbol sym, length len <= root).
BTS_PNG_HD void fill_short(uint32_t *t, int root, const Plan &pl, int i, int sym, int len) {
    const uint32_t code = pl.first[len] + (uint32_t)(i - pl.offs[len]);
    const uint32_t e = leaf(sym, len);
    for (uint32_t j = reverse_bits(code, len); j < (1u << root); j += 1u << len) t[j] = e;
}

// Codes longer than root, in sorted order from index i0 to n_codes: sub-tables sized as zlib sizes them, one per distinct
// root prefix.  Returns BTS_PNG_BAD_CODE_TABLE if the tables would outgrow cap entries.
BTS_PNG_HD int fill_long(uint32_t *t, int root, int cap, const Plan &pl, const uint16_t *sorted, const uint8_t *lens,
                         int i0, int n_codes) {
    uint32_t next = 1u << root, base = 0, prefix = 0xffffffffu;
    int sub = 0;
    for (int i = i0; i < n_codes; ++i) {
        const int sym = sorted[i], len = lens[sym];
        const uint32_t code = pl.first[len] + (uint32_t)(i - pl.offs[len]);
        const int drop = len - root;
        if ((code >> drop) != prefix) {
            prefix = code >> drop;
            // codes not yet placed: of this length, from index i on; of every longer length, all of them
            int curr = drop, l = len, left = 1 << curr;
            while (l < pl.max) {
                left -= l == len ? pl.count[len] - (i - pl.offs[len]) : pl.count[l];
                if (left <= 0) break;
                ++curr;
                ++l;
                left <<= 1;
            }
            if (next + (1u << curr) > (uint32_t)cap) return BTS_PNG_BAD_CODE_TABLE;
            base = next;
            sub = curr;
            next += 1u << curr;
            t[reverse_bits(prefix, root)] = 0x80000000u | ((uint32_t)sub << 16) | base;
        }
        const uint32_t e = leaf(sym, len);
        for (uint32_t j = reverse_bits(code & ((1u << drop) - 1), drop); j < (1u << sub); j += 1u << drop) t[base + j] = e;
    }
    return BTS_PNG_OK;
}

// Serial table build: lens[0..n) -> t (cap entries).  `sorted` is scratch of n entries.
BTS_PNG_HD int build_table(const uint8_t *lens, int n, uint32_t *t, int root, int cap, int kind, uint16_t *sorted) {
    Plan pl;
    for (int l = 0; l < 16; ++l) pl.count[l] = 0;
    for (int s = 0; s < n; ++s) ++pl.count[lens[s]];
    const int st = table_plan(pl, kind);
    if (st) return st;
    for (int j = 0; j < cap; ++j) t[j] = 0;
    uint16_t at[16];
    for (int l = 0; l < 16; ++l) at[l] = pl.offs[l];
    for (int s = 0; s < n; ++s)
        if (lens[s]) sorted[at[lens[s]]++] = (uint16_t)s;
    int n_short = 0, n_codes = 0;
    for (int l = 1; l <= 15; ++l) {
        n_codes += pl.count[l];
        if (l <= root) n_short += pl.count[l];
    }
    for (int i = 0; i < n_short; ++i) fill_short(t, root, pl, i, sorted[i], lens[sorted[i]]);
    return fill_long(t, root, cap, pl, sorted, lens, n_short, n_codes);
}

// RFC 1950 header: CM = 8, CINFO <= 7, FCHECK, no preset dictionary
BTS_PNG_HD int zlib_header(BitReader &br) {
    uint32_t cmf, flg;
    if (!br.bits(8, cmf) || !br.bits(8, flg)) return BTS_PNG_TRUNCATED;
    if ((cmf & 15) != 8 || (cmf >> 4) > 7 || ((cmf << 8) | flg) % 31 != 0 || (flg & 0x20)) return BTS_PNG_BAD_ZLIB_HEADER;
    return BTS_PNG_OK;
}

BTS_PNG_HD int block_header(BitReader &br, uint32_t &final, uint32_t &type) {
    if (!br.bits(1, final) || !br.bits(2, type)) return BTS_PNG_TRUNCATED;
    return type == 3 ? BTS_PNG_BAD_BLOCK : BTS_PNG_OK;
}

// Stored block after its 3 header bits: LEN / NLEN, then LEN bytes emitted as one stored run.
template <class Emit>
BTS_PNG_HD int stored_block(BitReader &br, uint32_t expected, uint32_t &produced, Emit &emit) {
    br.align();
    uint32_t len, nlen;
    if (!br.bits(16, len) || !br.bits(16, nlen)) return BTS_PNG_TRUNCATED;
    if (len != (~nlen & 0xffffu)) return BTS_PNG_BAD_BLOCK;
    const uint32_t at = br.byte_pos();
    if (len > br.n - at) return BTS_PNG_TRUNCATED;
    if (len > expected - produced) return BTS_PNG_BAD_SIZE;
    if (len) emit.stored(at, len);
    produced += len;
    br.seek(at + len);
    return BTS_PNG_OK;
}

// Dynamic block header after its 3 header bits: the code-length code, then HLIT + HDIST code lengths into lens[0..320).
// The code-length table is built by `build(lens, n, table, root, cap, kind)` (serial here, warp-cooperative on the GPU).
// Only a caller with `writer` set stores into lens (on the GPU all lanes of a warp run this in step and lane 0 writes).
// The code-length code's lengths go to lens[0..19) first and are overwritten by the decoded lengths.
BTS_PNG_HD int clen_order(int i) {   // 16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15, 5 bits each
    constexpr uint64_t lo = 16ull | 17ull << 5 | 18ull << 10 | 0ull << 15 | 8ull << 20 | 7ull << 25 | 9ull << 30 |
                            6ull << 35 | 10ull << 40 | 5ull << 45 | 11ull << 50 | 4ull << 55;
    constexpr uint64_t hi = 12ull | 3ull << 5 | 13ull << 10 | 2ull << 15 | 14ull << 20 | 1ull << 25 | 15ull << 30;
    return (int)((i < 12 ? lo >> (5 * i) : hi >> (5 * (i - 12))) & 31);
}

template <class Build>
BTS_PNG_HD int dynamic_lengths(BitReader &br, uint8_t *lens, uint32_t *clen_table, int &hlit, int &hdist, bool writer,
                               Build &build) {
    uint32_t a, b, c;
    if (!br.bits(5, a) || !br.bits(5, b) || !br.bits(4, c)) return BTS_PNG_TRUNCATED;
    hlit = (int)a + 257;
    hdist = (int)b + 1;
    const int hclen = (int)c + 4;
    if (hlit > 286 || hdist > 30) return BTS_PNG_BAD_CODE_TABLE;
    for (int i = 0; i < 19; ++i) {
        uint32_t v = 0;
        if (i < hclen && !br.bits(3, v)) return BTS_PNG_TRUNCATED;
        if (writer) lens[clen_order(i)] = (uint8_t)v;
    }
    int st = build(lens, 19, clen_table, CLEN_ROOT, CLEN_ENOUGH, KIND_CLEN);
    if (st) return st;
    const int total = hlit + hdist;
    int prev = -1;
    for (int i = 0; i < total;) {
        int sym;
        st = decode_sym(br, clen_table, CLEN_ROOT, sym);
        if (st) return st;
        if (sym < 16) {
            if (writer) lens[i] = (uint8_t)sym;
            prev = sym;
            ++i;
            continue;
        }
        uint32_t r;
        int val = 0, rep;
        if (sym == 16) {
            if (prev < 0) return BTS_PNG_BAD_CODE_TABLE;
            if (!br.bits(2, r)) return BTS_PNG_TRUNCATED;
            val = prev;
            rep = 3 + (int)r;
        } else if (sym == 17) {
            if (!br.bits(3, r)) return BTS_PNG_TRUNCATED;
            rep = 3 + (int)r;
        } else {
            if (!br.bits(7, r)) return BTS_PNG_TRUNCATED;
            rep = 11 + (int)r;
        }
        if (rep > total - i) return BTS_PNG_BAD_CODE_TABLE;
        for (int k = 0; k < rep; ++k)
            if (writer) lens[i + k] = (uint8_t)val;
        prev = val;
        i += rep;
    }
    return BTS_PNG_OK;
}

// The fixed code of block type 1 (RFC 1951 3.2.6): lens[0..288) literal/length, lens[288..320) distance.
BTS_PNG_HD uint8_t fixed_len(int i) {
    if (i >= 288) return 5;
    return i < 144 ? 8 : i < 256 ? 9 : i < 280 ? 7 : 8;
}

// Literal/length and distance symbols of one Huffman block up to its end-of-block code.
template <class Emit>
BTS_PNG_HD int huffman_block(BitReader &br, const uint32_t *lit, const uint32_t *dist, uint32_t expected,
                             uint32_t &produced, Emit &emit) {
    for (;;) {
        int sym;
        int st = decode_sym(br, lit, LITLEN_ROOT, sym);
        if (st) return st;
        if (sym < 256) {
            if (produced >= expected) return BTS_PNG_BAD_SIZE;
            emit.literal((uint8_t)sym);
            ++produced;
            continue;
        }
        if (sym == 256) return BTS_PNG_OK;
        sym -= 257;
        if (sym >= 29) return BTS_PNG_BAD_CODE_TABLE;   // length symbols 286, 287
        // length base / extra bits of RFC 1951 3.2.5, in closed form: 3..10 (0 extra), then 4 codes per extra bit, 258
        const int lx = sym < 8 || sym == 28 ? 0 : (sym >> 2) - 1;
        const uint32_t lb = sym < 8 ? 3 + sym : sym == 28 ? 258 : ((4u + (sym & 3)) << lx) + 3;
        uint32_t e, len, d;
        if (!br.bits(lx, e)) return BTS_PNG_TRUNCATED;
        len = lb + e;
        st = decode_sym(br, dist, DIST_ROOT, sym);
        if (st) return st;
        if (sym >= 30) return BTS_PNG_BAD_CODE_TABLE;   // distance symbols 30, 31
        const int dx = sym < 4 ? 0 : (sym >> 1) - 1;   // distances 1..4 (0 extra), then 2 codes per extra bit
        if (!br.bits(dx, e)) return BTS_PNG_TRUNCATED;
        d = (sym < 4 ? 1u + sym : ((2u + (sym & 1)) << dx) + 1) + e;
        if (d > produced) return BTS_PNG_DISTANCE_TOO_FAR;
        if (len > expected - produced) return BTS_PNG_BAD_SIZE;
        emit.match(len, d);
        produced += len;
    }
}

// After the final block: the big-endian Adler-32 on the next byte boundary; the decompressed size must be exact.
// Bytes after the Adler-32 are ignored.
BTS_PNG_HD int trailer(BitReader &br, uint32_t expected, uint32_t produced, uint32_t &adler) {
    br.align();
    adler = 0;
    for (int i = 0; i < 4; ++i) {
        uint32_t v;
        if (!br.bits(8, v)) return BTS_PNG_TRUNCATED;
        adler = (adler << 8) | v;
    }
    return produced == expected ? BTS_PNG_OK : BTS_PNG_BAD_SIZE;
}

struct SerialBuild {
    uint16_t sorted[320];
    BTS_PNG_HD int operator()(const uint8_t *lens, int n, uint32_t *t, int root, int cap, int kind) {
        return build_table(lens, n, t, root, cap, kind, sorted);
    }
};

// Whole zlib stream, serially: the host build of the decoder.  adler receives the stream's stored Adler-32 (the caller
// checks it against the output).
template <class Emit>
inline int inflate_serial(const uint8_t *src, uint32_t n, uint32_t expected, Emit &emit, uint32_t &adler) {
    BitReader br;
    br.init(src, n);
    uint32_t lit[LITLEN_ENOUGH], dist[DIST_ENOUGH], clen[CLEN_ENOUGH];
    uint8_t lens[320];
    SerialBuild build;
    uint32_t produced = 0;
    int st = zlib_header(br);
    if (st) return st;
    for (;;) {
        uint32_t final, type;
        st = block_header(br, final, type);
        if (st) return st;
        if (type == 0) {
            st = stored_block(br, expected, produced, emit);
        } else {
            int hlit = 288, hdist = 32;
            if (type == 1) {
                for (int i = 0; i < 320; ++i) lens[i] = fixed_len(i);
            } else {
                st = dynamic_lengths(br, lens, clen, hlit, hdist, true, build);
                if (!st && lens[256] == 0) st = BTS_PNG_BAD_CODE_TABLE;   // no end-of-block code
            }
            if (!st) st = build(lens, hlit, lit, LITLEN_ROOT, LITLEN_ENOUGH, KIND_LITLEN);
            if (!st) st = build(lens + hlit, hdist, dist, DIST_ROOT, DIST_ENOUGH, KIND_DIST);
            if (!st) st = huffman_block(br, lit, dist, expected, produced, emit);
        }
        if (st) return st;
        if (final) break;
    }
    return trailer(br, expected, produced, adler);
}

BTS_PNG_HD uint32_t adler32(const uint8_t *d, uint64_t n) {
    uint32_t a = 1, b = 0;
    for (uint64_t i = 0; i < n; ++i) {
        a = (a + d[i]) % 65521u;
        b = (b + a) % 65521u;
    }
    return (b << 16) | a;
}

// ------------------------------------------------------------------------------------------------ row unfilter
BTS_PNG_HD uint8_t paeth(int a, int b, int c) {
    const int p = a + b - c;
    const int pa = p > a ? p - a : a - p, pb = p > b ? p - b : b - p, pc = p > c ? p - c : c - p;
    return (uint8_t)(pa <= pb && pa <= pc ? a : pb <= pc ? b : c);
}

// Average (3) or Paeth (4) on byte lane `lane` (0 <= lane < bpp) of a row: cur holds the filtered bytes and receives the
// reconstructed ones; prev is the reconstructed previous row (zeros above the first row).  The lane is serial: each byte
// needs its left neighbour's result.
BTS_PNG_HD void unfilter_lane(int filter, uint8_t *cur, const uint8_t *prev, int rowbytes, int bpp, int lane) {
    int a = 0, c = 0;
    for (int j = lane; j < rowbytes; j += bpp) {
        const int b = prev[j];
        const uint8_t x = (uint8_t)(cur[j] + (filter == 3 ? (uint8_t)((a + b) >> 1) : paeth(a, b, c)));
        cur[j] = x;
        a = x;
        c = b;
    }
}

// One row, serially (host build).  Returns BTS_PNG_BAD_FILTER for a filter byte > 4.
BTS_PNG_HD int unfilter_row(int filter, uint8_t *cur, const uint8_t *prev, int rowbytes, int bpp) {
    switch (filter) {
    case 0: return BTS_PNG_OK;
    case 1:
        for (int j = bpp; j < rowbytes; ++j) cur[j] = (uint8_t)(cur[j] + cur[j - bpp]);
        return BTS_PNG_OK;
    case 2:
        for (int j = 0; j < rowbytes; ++j) cur[j] = (uint8_t)(cur[j] + prev[j]);
        return BTS_PNG_OK;
    case 3:
    case 4:
        for (int lane = 0; lane < bpp; ++lane) unfilter_lane(filter, cur, prev, rowbytes, bpp, lane);
        return BTS_PNG_OK;
    default: return BTS_PNG_BAD_FILTER;
    }
}

}  // namespace bts_png
