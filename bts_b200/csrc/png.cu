// Batched PNG decode on the device (bts_png_inflate, bts_png_unfilter; ops.decode_png), sm_90a.
//
//  png_inflate_kernel   one CTA (two warps) per zlib stream.  Decoding a stream is serial, so the parallelism is the batch;
//                       inside a CTA the two warps overlap.  Warp 0 parses block headers and builds the Huffman tables in
//                       shared memory together; then its lane 0 decodes the block's symbols through the shared core
//                       (png_core.cuh) into a command ring in shared memory.  Warp 1 executes the commands into the raw
//                       (still filtered) scanlines in global memory, 32 lanes per literal run, match or stored run.  The
//                       hand-off is a pair of shared-memory counters with release / acquire ordering; no block-wide
//                       barrier sits inside the symbol loop.
//  png_unfilter_kernel  one CTA per image, rows in order, previous and current row in shared memory: filters None and Up
//                       on all threads, Sub as a per-byte-lane prefix sum mod 256, Average and Paeth serially on `bpp`
//                       threads (each byte needs its left neighbour).  Each image writes only its crop window into the
//                       batched output, 16-bit samples byte-swapped to native order.  The same pass checks the stream's
//                       Adler-32 over the raw bytes.
#include <cuda/atomic>

#include "common.cuh"
#include "png_core.cuh"

namespace {

using namespace bts_png;

constexpr int INFLATE_THREADS = 64;
constexpr int RING = 256;       // commands in flight
constexpr int LITRING = 4096;   // literal bytes in flight
constexpr int LITRUN = 1024;    // longest literal run per command (< LITRING, so a pending run never blocks the ring)
constexpr uint32_t CMD_LIT = 0u << 30, CMD_MATCH = 1u << 30, CMD_STORED = 2u << 30, CMD_END = 3u << 30;
constexpr long long MAX_RAW = 1ll << 28;   // per image: keeps the unfilter's 64-bit Adler-32 partial sums exact

struct InflateShared {
    uint32_t lit[LITLEN_ENOUGH];
    uint32_t dist[DIST_ENOUGH];
    uint32_t clen[CLEN_ENOUGH];
    Plan plan;
    uint16_t at[16];
    uint16_t sorted[320];
    uint8_t lens[320];
    int table_status;
    uint2 ring[RING];   // x = kind | length, y = literal-ring offset (LIT), distance (MATCH) or source offset (STORED)
    uint8_t litring[LITRING];
    unsigned head, tail, lit_done;
};

using block_counter = cuda::atomic_ref<unsigned, cuda::thread_scope_block>;

// Huffman table build by the 32 lanes of warp 0: counting and placing the code lengths with __match_any_sync, filling the
// root table in parallel; the rules (table_plan) and the sub-tables (fill_long) are the core's, on lane 0.
struct WarpBuild {
    InflateShared *s;
    int lane;
    __device__ int operator()(const uint8_t *lens, int n, uint32_t *t, int root, int cap, int kind) {
        Plan &pl = s->plan;
        __syncwarp();   // lens may have been written by lane 0 alone
        if (lane < 16) pl.count[lane] = 0;
        for (int j = lane; j < cap; j += 32) t[j] = 0;
        __syncwarp();
        for (int c = 0; c < n; c += 32) {
            const int len = c + lane < n ? lens[c + lane] : 0;
            const unsigned grp = __match_any_sync(0xffffffffu, len);
            if (lane == 31 - __clz(grp)) pl.count[len] += __popc(grp);   // count[0] is not used
            __syncwarp();
        }
        if (lane == 0) s->table_status = table_plan(pl, kind);
        __syncwarp();
        int st = s->table_status;
        if (st || pl.max == 0) return st;
        if (lane < 16) s->at[lane] = pl.offs[lane];
        __syncwarp();
        for (int c = 0; c < n; c += 32) {
            const int len = c + lane < n ? lens[c + lane] : 0;
            const unsigned grp = __match_any_sync(0xffffffffu, len);
            if (len) s->sorted[s->at[len] + __popc(grp & ((1u << lane) - 1))] = (uint16_t)(c + lane);
            __syncwarp();
            if (len && lane == 31 - __clz(grp)) s->at[len] += __popc(grp);
            __syncwarp();
        }
        const int n_short = pl.offs[root + 1], n_codes = pl.offs[15] + pl.count[15];
        for (int i = lane; i < n_short; i += 32) fill_short(t, root, pl, i, s->sorted[i], lens[s->sorted[i]]);
        __syncwarp();
        if (lane == 0) s->table_status = fill_long(t, root, cap, pl, s->sorted, lens, n_short, n_codes);
        __syncwarp();
        return s->table_status;
    }
};

// Producer side of the command ring (lane 0 of warp 0).  Consecutive literals are collected into one run.
struct RingEmit {
    InflateShared *s;
    unsigned head, tail_seen, lit_head, lit_seen, run;
    __device__ void push(uint32_t x, uint32_t y) {
        if (head - tail_seen >= (unsigned)RING) {
            block_counter tail(s->tail);
            do tail_seen = tail.load(cuda::memory_order_acquire);
            while (head - tail_seen >= (unsigned)RING);
        }
        s->ring[head % RING] = make_uint2(x, y);
        ++head;
        block_counter(s->head).store(head, cuda::memory_order_release);
    }
    __device__ void flush() {
        if (run) push(CMD_LIT | run, lit_head - run);
        run = 0;
    }
    __device__ void literal(uint8_t b) {
        if (lit_head - lit_seen >= (unsigned)LITRING) {
            block_counter done(s->lit_done);
            do lit_seen = done.load(cuda::memory_order_acquire);
            while (lit_head - lit_seen >= (unsigned)LITRING);
        }
        s->litring[lit_head % LITRING] = b;
        ++lit_head;
        if (++run == (unsigned)LITRUN) flush();
    }
    __device__ void match(uint32_t len, uint32_t dist) {
        flush();
        push(CMD_MATCH | len, dist);
    }
    __device__ void stored(uint32_t at, uint32_t len) {
        flush();
        push(CMD_STORED | len, at);
    }
};

// Consumer (warp 1): commands in order into out.  The core has checked every command, so the copies need no bounds tests.
__device__ void execute_commands(InflateShared *s, const uint8_t *src, uint8_t *out, int lane) {
    block_counter head(s->head);
    unsigned tail = 0;
    uint32_t pos = 0;
    for (;;) {
        unsigned h;
        while ((h = head.load(cuda::memory_order_acquire)) == tail) {
        }
        for (; tail != h; ++tail) {
            const uint2 c = s->ring[tail % RING];
            const uint32_t kind = c.x & 0xc0000000u, len = c.x & 0x3fffffffu;
            if (kind == CMD_END) return;
            if (kind == CMD_LIT) {
                for (uint32_t k = lane; k < len; k += 32) out[pos + k] = s->litring[(c.y + k) % LITRING];
            } else if (kind == CMD_STORED) {
                for (uint32_t k = lane; k < len; k += 32) out[pos + k] = src[c.y + k];
            } else if (c.y >= 32) {
                // each 32-byte step reads bytes written before it
                for (uint32_t k0 = 0; k0 < len; k0 += 32) {
                    if (k0 + lane < len) out[pos + k0 + lane] = out[pos + k0 + lane - c.y];
                    __syncwarp();
                }
            } else {
                // a short distance repeats the last c.y bytes: copy with that period, from bytes before pos only
                for (uint32_t k = lane; k < len; k += 32) out[pos + k] = out[pos - c.y + k % c.y];
            }
            pos += len;
            __syncwarp();
            if (lane == 0) {
                block_counter(s->tail).store(tail + 1, cuda::memory_order_release);
                if (kind == CMD_LIT) block_counter(s->lit_done).store(c.y + len, cuda::memory_order_release);
            }
        }
    }
}

// meta row: src offset, src length, raw offset, height, width, crop y0, crop x0, (unused)
__global__ void __launch_bounds__(INFLATE_THREADS) png_inflate_kernel(const uint8_t *src, const long long *__restrict__ meta,
                                                                      int bpp, uint8_t *raw, unsigned *__restrict__ adler_out,
                                                                      int *__restrict__ status) {
    __shared__ InflateShared s;
    const int img = blockIdx.x, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const long long *m = meta + (long long)img * 8;
    const long long H = m[3], W = m[4], expected_ll = H * (1 + W * bpp);
    const bool sane = m[0] >= 0 && m[1] >= 0 && m[1] <= 0xffffffffll && m[2] >= 0 && H > 0 && W > 0 && expected_ll <= MAX_RAW;
    if (!sane) {   // uniform over the CTA; the host never sends such a row
        if (threadIdx.x == 0) status[img] = BTS_PNG_BAD_SIZE;
        return;
    }
    const uint8_t *in = src + m[0];
    const uint32_t expected = (uint32_t)expected_ll;
    if (threadIdx.x == 0) s.head = s.tail = s.lit_done = 0;
    __syncthreads();
    if (warp == 1) {
        execute_commands(&s, in, raw + m[2], lane);
        return;
    }
    BitReader br;
    br.init(in, (uint32_t)m[1]);
    WarpBuild build{&s, lane};
    RingEmit emit{&s, 0, 0, 0, 0, 0};
    uint32_t produced = 0, adler = 0;
    int st = zlib_header(br);
    while (!st) {
        uint32_t final, type;
        st = block_header(br, final, type);
        if (st) break;
        if (type == 0) {
            if (lane == 0) st = stored_block(br, expected, produced, emit);
        } else {
            int hlit = 288, hdist = 32;
            if (type == 1) {
                for (int i = lane; i < 320; i += 32) s.lens[i] = fixed_len(i);
            } else {
                st = dynamic_lengths(br, s.lens, s.clen, hlit, hdist, lane == 0, build);
                __syncwarp();
                if (!st && s.lens[256] == 0) st = BTS_PNG_BAD_CODE_TABLE;   // no end-of-block code
            }
            if (!st) st = build(s.lens, hlit, s.lit, LITLEN_ROOT, LITLEN_ENOUGH, KIND_LITLEN);
            if (!st) st = build(s.lens + hlit, hdist, s.dist, DIST_ROOT, DIST_ENOUGH, KIND_DIST);
            if (!st && lane == 0) st = huffman_block(br, s.lit, s.dist, expected, produced, emit);
        }
        // after a stored or Huffman block lane 0 holds the reader's state
        __syncwarp();
        st = __shfl_sync(0xffffffffu, st, 0);
        produced = __shfl_sync(0xffffffffu, produced, 0);
        br.pos = __shfl_sync(0xffffffffu, br.pos, 0);
        br.cnt = __shfl_sync(0xffffffffu, br.cnt, 0);
        br.buf = __shfl_sync(0xffffffffu, (unsigned long long)br.buf, 0);
        if (final) break;
    }
    if (!st) st = trailer(br, expected, produced, adler);
    if (lane == 0) {
        emit.flush();
        emit.push(CMD_END, 0);
        status[img] = st;
        adler_out[img] = adler;
    }
}

constexpr int UNFILTER_THREADS = 256;

// Block-wide exclusive scan of per-thread words under per-byte addition mod 256 (__vadd4); returns this thread's prefix.
__device__ uint32_t block_scan_vadd4(uint32_t v, uint32_t *warp_tot) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    uint32_t inc = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const uint32_t u = __shfl_up_sync(0xffffffffu, inc, o);
        if (lane >= o) inc = __vadd4(inc, u);
    }
    if (lane == 31) warp_tot[warp] = inc;
    __syncthreads();
    uint32_t base = 0;
    for (int w = 0; w < warp; ++w) base = __vadd4(base, warp_tot[w]);
    __syncthreads();
    return __vadd4(base, __vsub4(inc, v));
}

__device__ __forceinline__ uint32_t load_px(const uint8_t *p, int bpp) {
    return bpp == 3 ? (uint32_t)p[0] | (uint32_t)p[1] << 8 | (uint32_t)p[2] << 16 : (uint32_t)p[0] | (uint32_t)p[1] << 8;
}

__global__ void __launch_bounds__(UNFILTER_THREADS) png_unfilter_kernel(const uint8_t *__restrict__ raw,
                                                                        const long long *__restrict__ meta,
                                                                        const unsigned *__restrict__ adler, int bpp, int out_h,
                                                                        int out_w, uint8_t *__restrict__ out,
                                                                        int *__restrict__ status) {
    __shared__ __align__(16) uint8_t rows[2][BTS_PNG_MAX_ROW_BYTES];
    __shared__ uint32_t warp_tot[UNFILTER_THREADS / 32];
    __shared__ unsigned long long red[2][UNFILTER_THREADS / 32];
    const int img = blockIdx.x, tid = threadIdx.x;
    if (status[img] != BTS_PNG_OK) return;
    const long long *m = meta + (long long)img * 8;
    const long long H = m[3], W = m[4], y0 = m[5], x0 = m[6];
    if (W * bpp > BTS_PNG_MAX_ROW_BYTES || y0 < 0 || x0 < 0 || y0 + out_h > H || x0 + out_w > W) {
        if (tid == 0) status[img] = BTS_PNG_BAD_SIZE;   // the host never sends such a row
        return;
    }
    const int rowbytes = (int)W * bpp, stride = rowbytes + 1;
    const uint8_t *src = raw + m[2];
    uint8_t *prev = rows[0], *cur = rows[1];
    for (int j = tid; j < rowbytes; j += UNFILTER_THREADS) prev[j] = 0;
    unsigned long long sd = 0, sid = 0;   // Adler-32 partials: sum of bytes, sum of position * byte
    const int seg = ((int)W + UNFILTER_THREADS - 1) / UNFILTER_THREADS;
    for (int r = 0; r < (int)H; ++r) {
        const uint8_t *row = src + (long long)r * stride;
        const unsigned long long at = (unsigned long long)r * stride;
        const int f = row[0];
        if (tid == 0) {
            sd += f;
            sid += at * f;
        }
        if (f > 4) {
            if (tid == 0) status[img] = BTS_PNG_BAD_FILTER;
            return;
        }
        for (int j = tid; j < rowbytes; j += UNFILTER_THREADS) {
            const uint8_t v = row[1 + j];
            cur[j] = v;
            sd += v;
            sid += (at + 1 + j) * v;
        }
        __syncthreads();
        if (f == 2) {
            for (int j = tid; j < rowbytes; j += UNFILTER_THREADS) cur[j] = (uint8_t)(cur[j] + prev[j]);
        } else if (f == 1) {
            // Sub: pixel p = its filtered bytes + pixel p-1, per byte lane; pixels packed in words, summed with __vadd4
            const int p0 = min(tid * seg, (int)W), p1 = min(p0 + seg, (int)W);
            uint32_t tot = 0;
            for (int p = p0; p < p1; ++p) tot = __vadd4(tot, load_px(cur + p * bpp, bpp));
            uint32_t acc = block_scan_vadd4(tot, warp_tot);
            for (int p = p0; p < p1; ++p) {
                acc = __vadd4(acc, load_px(cur + p * bpp, bpp));
                for (int k = 0; k < bpp; ++k) cur[p * bpp + k] = (uint8_t)(acc >> (8 * k));
            }
        } else if (f >= 3 && tid < bpp) {
            unfilter_lane(f, cur, prev, rowbytes, bpp, tid);
        }
        __syncthreads();
        if (r >= y0 && r < y0 + out_h) {
            const long long orow = (long long)img * out_h + (r - y0);
            if (bpp == 3) {
                uint8_t *dst = out + orow * out_w * 3;
                const uint8_t *s = cur + x0 * 3;
                for (int j = tid; j < out_w * 3; j += UNFILTER_THREADS) dst[j] = s[j];
            } else {
                uint16_t *dst = reinterpret_cast<uint16_t *>(out) + orow * out_w;
                const uint8_t *s = cur + x0 * 2;
                for (int j = tid; j < out_w; j += UNFILTER_THREADS) dst[j] = (uint16_t)(s[2 * j] << 8 | s[2 * j + 1]);
            }
        }
        uint8_t *t = prev;
        prev = cur;
        cur = t;
    }
    // Adler-32 of n bytes d_i: a = 1 + sum d_i, b = n + n * sum d_i - sum i * d_i (mod 65521)
    const int lane = tid & 31, warp = tid >> 5;
    for (int o = 16; o > 0; o >>= 1) {
        sd += __shfl_xor_sync(0xffffffffu, sd, o);
        sid += __shfl_xor_sync(0xffffffffu, sid, o);
    }
    if (lane == 0) {
        red[0][warp] = sd;
        red[1][warp] = sid;
    }
    __syncthreads();
    if (tid == 0) {
        unsigned long long d = 0, id = 0;
        for (int w = 0; w < UNFILTER_THREADS / 32; ++w) {
            d += red[0][w];
            id += red[1][w];
        }
        const unsigned long long M = 65521, n = (unsigned long long)H * stride % M;
        const unsigned long long a = (1 + d) % M, b = (n + n * (d % M) + M - id % M) % M;
        if ((unsigned)(b << 16 | a) != adler[img]) status[img] = BTS_PNG_ADLER_MISMATCH;
    }
}

}  // namespace

extern "C" int bts_png_inflate(const unsigned char *src, const long long *meta, int n, int bpp, unsigned char *raw,
                               unsigned int *adler, int *status, void *stream) {
    if (!src || !meta || !raw || !adler || !status || n <= 0 || (bpp != 2 && bpp != 3)) return BTS_EINVAL;
    png_inflate_kernel<<<n, INFLATE_THREADS, 0, (cudaStream_t)stream>>>(src, meta, bpp, raw, adler, status);
    BTS_LAUNCH_CHECK();
    return 0;
}

extern "C" int bts_png_unfilter(const unsigned char *raw, const long long *meta, const unsigned int *adler, int n, int bpp,
                                int out_h, int out_w, void *out, int *status, void *stream) {
    if (!raw || !meta || !adler || !out || !status || n <= 0 || (bpp != 2 && bpp != 3) || out_h <= 0 || out_w <= 0)
        return BTS_EINVAL;
    png_unfilter_kernel<<<n, UNFILTER_THREADS, 0, (cudaStream_t)stream>>>(raw, meta, adler, bpp, out_h, out_w,
                                                                          (uint8_t *)out, status);
    BTS_LAUNCH_CHECK();
    return 0;
}
