// wgrad for narrow-output 3x3 convolutions (Cout <= 64: the DenseNet 3x3 dense-layer convs 192->48 and the full- /
// half-resolution decoder convs conv1/upconv1/conv2/upconv2) and for 1x1 layers with 64 < Cout <= 256, on the Hopper
// tensor cores (wgmma, register accumulators), 3xTF32 -- "shifted dY" formulation.
//
//   dW[co, ci, tap] = sum_q  x~[q, ci] * dY[q - off(tap), co]            q = INPUT pixel, off(tap) = tap*dil - pad
//
// wgrad_tc.cu puts the tap in the grid, so the activation tile -- the expensive operand: loads, BN/ReLU pre-op, hi/lo
// split, shared-memory writes per k-block -- is produced once per tap.  Here ONE CTA owns all taps of a (64 ci, cg co)
// block: per k-block of 16 input pixels the activation tile is produced once and multiplied against the shifted dY tiles
// of every tap, packed densely along N (tap t owns the N slots [t*ncol, (t+1)*ncol)), so that wgmma of width
// taps*ncol <= 144 covers them all; two consumer warpgroups split those columns (<= 40 accumulator registers per thread).
// Operand tiles are K-major (pixels contiguous per channel row) in 8 x 16-byte core matrices, written by the producers;
// deterministic split-K partial layout as wgrad_tc.cu.
//
// Operand staging: the shifted dY windows of a k-block overlap -- they are KH row segments of 16 + (KW-1)*dil consecutive
// output pixels.  With TMA = true a loader lane copies the raw fp32 segments (and the raw x tile unless it is read through
// the nearest-neighbour up-sample) into a small landing ring, several k-blocks ahead (cp.async.bulk.tensor.2d, no swizzle,
// zero fill past the tensor ends); the producers then read shared memory, apply the border masks / pre-op, split hi/lo
// and write the operand tiles.
#include <cuda.h>

#include <cstring>
#include <type_traits>

#include "tc_common.cuh"

using namespace tc;

namespace {

constexpr int BLOCK_CI = 64;                 // input channels per CTA = the M of one consumer warpgroup
constexpr int X_CHUNKS = BLOCK_CI / 32;      // 32-channel chunks of the activation tile
constexpr int KP = 16;                       // input pixels per k-block (2 k-groups of 8)
constexpr uint32_t CORE_SBO = 4 * 128 + 16;  // one 8-row group of a k-block: 4 core matrices along K + a bank pad
constexpr int A_BYTES = BLOCK_CI / 8 * CORE_SBO;   // hi or lo
constexpr int MAX_TAPS = 9;
constexpr int MAX_NT = 144;                  // widest packed N (taps * ncol), split between the two consumer warpgroups
constexpr int MAX_STAGES = 4;
constexpr int CONSUMER_THREADS = 256;       // two warpgroups, each owns about half of the packed N columns
constexpr int LOADER_WARP = CONSUMER_THREADS / 32;
constexpr int GROUPS = 3;                    // producer groups of 128 threads: group g owns the dY taps t == g (mod 3)
constexpr int PRODUCERS = 128 * GROUPS;
constexpr int NUM_THREADS = CONSUMER_THREADS + 32 + PRODUCERS;
constexpr int SMEM_BUDGET = 224 * 1024;
constexpr int MAX_RING = 4;                  // landing-ring slots (TMA staging)
constexpr int X_RAW_BYTES = KP * BLOCK_CI * 4;   // raw x tile of a k-block: 4 KB

struct W2Params {
    const float *x; long long xs;
    int B, Hs, Ws, up, Cin;
    int KH, KW, pad, dil;
    const float *pre_scale, *pre_shift;
    const float *dy; long long dys;
    int Cout, Hout, Wout, Hin, Win;
    int cg, nb;              // output channels per CTA (multiple of 16) and their 32-channel chunks
    int nchunks;             // 32-row chunks of the tap-packed dY tile: ceil(taps*cg/32)
    float *part;             // [splitK][taps][Cin][Cout]
    int splitK, kb_per_split, KBq;
    int Mq;                  // B*Hin*Win input pixels
    int stages, stage_bytes, precision;
    // TMA landing ring (TMA = true): slot = [raw x tile (unless up) | KH segments of segw pixels x cg channels]
    int ring, slot_bytes, seg_bytes, segw, tox_max, slot_tx;
};

template <int PRE, bool UP, bool VEC, bool TMA>
__global__ void __launch_bounds__(NUM_THREADS, 1) wgrad2_tc_kernel(const W2Params p, const __grid_constant__ CUtensorMap tmx,
                                                                   const __grid_constant__ CUtensorMap tmd) {
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;
    uint8_t *sm = smem_raw + (base - smem_u32(smem_raw));
    const int taps = p.KH * p.KW;
    const int S = p.stages;
    const uint32_t ring_off = (uint32_t)S * (uint32_t)p.stage_bytes;
    const uint32_t pre_off = ring_off + (TMA ? (uint32_t)p.ring * (uint32_t)p.slot_bytes : 0u);
    float *s_scale = reinterpret_cast<float *>(sm + pre_off);
    float *s_shift = s_scale + BLOCK_CI;
    const uint32_t bar0 = base + pre_off + 2 * BLOCK_CI * 4;
    auto full = [&](int s) { return bar0 + 8u * s; };
    auto empty = [&](int s) { return bar0 + 8u * (MAX_STAGES + s); };
    auto rfull = [&](int j) { return bar0 + 8u * (2 * MAX_STAGES + j); };
    auto rempty = [&](int j) { return bar0 + 8u * (2 * MAX_STAGES + MAX_RING + j); };
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int ci_tile = blockIdx.x, cgi = blockIdx.y, split = blockIdx.z;
    const int co0 = cgi * p.cg;
    const int ncol = min(p.cg, ((p.Cout - co0 + 15) >> 4) << 4);     // live columns of this CTA (multiple of 16)
    const int nb = p.nb;
    // dY operand: the taps are packed DENSELY along N -- tap t owns the N rows [t*ncol, (t+1)*ncol) of one tile of
    // ceil(taps*ncol/32) 32-row chunks -- so that a single wgmma multiplies the activation tile against all taps at once.
    // hi and lo tiles follow each other.
    const int n_total = taps * ncol;
    const uint32_t b_half = (uint32_t)p.nchunks * 4u * CORE_SBO;
    const int kb0 = split * p.kb_per_split;
    int kb1 = kb0 + p.kb_per_split;
    if (kb1 > p.KBq) kb1 = p.KBq;
    const int nkb = kb1 > kb0 ? kb1 - kb0 : 0;

    if (threadIdx.x == 0) {
        for (int s = 0; s < MAX_STAGES; ++s) {
            mbar_init(full(s), PRODUCERS);
            mbar_init(empty(s), CONSUMER_THREADS);
        }
        for (int j = 0; j < MAX_RING; ++j) {
            mbar_init(rfull(j), 1);
            mbar_init(rempty(j), PRODUCERS);
        }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    if (PRE >= 2) {
        for (int c = threadIdx.x; c < BLOCK_CI; c += NUM_THREADS) {
            const int ch = ci_tile * BLOCK_CI + c;
            s_scale[c] = ch < p.Cin ? p.pre_scale[ch] : 0.f;
            s_shift[c] = ch < p.Cin ? p.pre_shift[ch] : 0.f;
        }
    }
    // zero every operand stage once: dead channel chunks / dead units are never written afterwards
    for (int i = threadIdx.x; i < S * p.stage_bytes / 16; i += NUM_THREADS) st_shared_v4(base + i * 16, 0.f, 0.f, 0.f, 0.f);
    fence_proxy_async();
    __syncthreads();

    if (warp == LOADER_WARP) {
        // ---- loader: one lane keeps the landing ring `ring` k-blocks ahead of the producers
        if (TMA && lane == 0) {
            if (!UP) tma_prefetch_desc(&tmx);
            tma_prefetch_desc(&tmd);
            int j = 0;
            uint32_t ph = 0;
            for (int it = 0; it < nkb; ++it) {
                mbar_wait(rempty(j), ph ^ 1);
                const uint32_t dst = base + ring_off + (uint32_t)j * (uint32_t)p.slot_bytes;
                const int q0 = (kb0 + it) * KP;
                mbar_arrive_expect_tx(rfull(j), (uint32_t)p.slot_tx);
                uint32_t seg = dst;
                if (!UP) {
                    tma_tile_2d(dst, &tmx, ci_tile * BLOCK_CI, q0, rfull(j));
                    seg += X_RAW_BYTES;
                }
                for (int ky = 0; ky < p.KH; ++ky)     // output pixels q - (ky*dil - pad)*W - tox, tox <= tox_max
                    tma_tile_2d(seg + (uint32_t)ky * (uint32_t)p.seg_bytes, &tmd, co0,
                                q0 - (ky * p.dil - p.pad) * p.Wout - p.tox_max, rfull(j));
                if (++j == p.ring) { j = 0; ph ^= 1; }
            }
        }
    } else if (warp < LOADER_WARP) {
        // ---- consumer warpgroups: rows = the 64 input channels; warpgroup wg owns the packed columns [n0, n0 + N) of
        //      all taps x ncol (n0 = 0 | the first half rounded up to 16); 3xTF32 per k8 step, small cross terms first;
        //      a stage is released as soon as its wgmma group has completed
        const int wg = warp >> 2;
        const int n_half = (n_total + 31) / 32 * 16;
        const int n0 = wg ? n_half : 0, n_mine = wg ? n_total - n_half : n_half;
        auto consume = [&](auto NT) {
            constexpr int N = decltype(NT)::value;
            float acc[N > 0 ? N / 2 : 1];
#pragma unroll
            for (int i = 0; i < (N > 0 ? N / 2 : 1); ++i) acc[i] = 0.f;
            const bool single = p.precision != 0;
            int s = 0;
            uint32_t ph = 0;
            for (int it = 0; it < nkb; ++it) {
                mbar_wait(full(s), ph);
                wgmma_fence();
                const uint32_t a_hi = base + (uint32_t)s * (uint32_t)p.stage_bytes, a_lo = a_hi + A_BYTES;
                const uint32_t b_hi = a_hi + 2 * A_BYTES + (uint32_t)(n0 >> 3) * CORE_SBO, b_lo = b_hi + b_half;
                if constexpr (N > 0) {
#pragma unroll
                    for (int kg = 0; kg < KP / 8; ++kg) {
                        const uint32_t ko = (uint32_t)kg * 256u;
                        const uint64_t dah = make_desc_core(a_hi + ko, 128, CORE_SBO), dal = make_desc_core(a_lo + ko, 128, CORE_SBO);
                        const uint64_t dbh = make_desc_core(b_hi + ko, 128, CORE_SBO), dbl = make_desc_core(b_lo + ko, 128, CORE_SBO);
                        const uint32_t accumulate = (it | kg) != 0;
                        if (single) {
                            Wgmma<N>::mma(acc, dah, dbh, accumulate);
                        } else {
                            Wgmma<N>::mma(acc, dal, dbh, accumulate);
                            Wgmma<N>::mma(acc, dah, dbl, 1);
                            Wgmma<N>::mma(acc, dah, dbh, 1);
                        }
                    }
                }
                wgmma_commit();
                wgmma_wait<0>();
                mbar_arrive(empty(s));
                if (++s == S) { s = 0; ph ^= 1; }
            }
            wgmma_wait<0>();
            wgmma_fence_operands(acc);
            if (N == 0) return;
            // ---- epilogue: accumulator row = input channel, column n = tap (n / ncol), output channel co0 + n % ncol
            const bool ovec = (p.Cout & 1) == 0 && ((((uintptr_t)p.part) & 7) == 0) && ((co0 & 1) == 0);
#pragma unroll
            for (int i = 0; i < 2; ++i) {
                const int ci = ci_tile * BLOCK_CI + (warp & 3) * 16 + (lane >> 2) + 8 * i;
                if (ci >= p.Cin) continue;
#pragma unroll
                for (int j = 0; j < (N > 0 ? N / 8 : 0); ++j) {
                    const int n = n0 + 8 * j + (lane & 3) * 2;
                    if (n >= n0 + n_mine) continue;
                    const int t = n / ncol, cc = n - t * ncol;
                    float *dst = p.part + (((long long)split * taps + t) * p.Cin + ci) * p.Cout + co0 + cc;
                    const float v0 = acc[4 * j + 2 * i], v1 = acc[4 * j + 2 * i + 1];
                    if (ovec && co0 + cc + 1 < p.Cout) {
                        *reinterpret_cast<float2 *>(dst) = make_float2(v0, v1);
                    } else {
                        if (co0 + cc < p.Cout) dst[0] = v0;
                        if (co0 + cc + 1 < p.Cout) dst[1] = v1;
                    }
                }
            }
        };
        switch (n_mine) {
            case 0: consume(std::integral_constant<int, 0>()); break;       // nothing to multiply: only releases stages
            case 16: consume(std::integral_constant<int, 16>()); break;
            case 32: consume(std::integral_constant<int, 32>()); break;
            case 48: consume(std::integral_constant<int, 48>()); break;
            case 64: consume(std::integral_constant<int, 64>()); break;
            default: consume(std::integral_constant<int, 80>()); break;
        }
    } else {
        // 12 producer warps in GROUPS = 3 groups of 128 threads.  Group q owns the x chunk q (if any) and the dY taps
        // t == q (mod 3): at most 1 + 6 sixteen-byte units per thread.
        const int pt = threadIdx.x - (CONSUMER_THREADS + 32);   // 0..PRODUCERS-1
        const int unit = pt & 7;                   // 16-byte unit of the 128-byte row
        const int row = (pt >> 3) & 15;            // pixel row of the 16-pixel k-block
        const int half = pt >> 7;                  // group 0..2: A chunk `half` (< X_CHUNKS);  dY: taps t == half (mod 3)
        const bool xq = half < X_CHUNKS;
        constexpr bool AFF = PRE >= 2;
        constexpr bool RELU = (PRE & 1) != 0;
        // K-major core-matrix tiles: element (row n, pixel k) at (n / 8) * CORE_SBO + (k / 4) * 128 + (n % 8) * 16 + (k % 4) * 4;
        // a thread's 4 consecutive channels of one pixel are 4 scalar stores 16 bytes apart
        auto core_off = [&](int n) {
            return (uint32_t)(n >> 3) * CORE_SBO + (uint32_t)(row >> 2) * 128u + (uint32_t)(n & 7) * 16u + (uint32_t)(row & 3) * 4u;
        };
        const int xs = (int)p.xs, dys = (int)p.dys;
        const int cbx = ci_tile * BLOCK_CI + half * 32 + unit * 4;    // first x channel of this thread (chunk `half`)
        const int cbd = co0 + unit * 4;                               // first dY channel (chunk 0)
        const float *__restrict__ xg = p.x;
        const float *__restrict__ dg = p.dy;
        float sc[1][4], sh[1][4];
        if (AFF) {
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                sc[0][e] = xq ? s_scale[half * 32 + unit * 4 + e] : 0.f;
                sh[0][e] = xq ? s_shift[half * 32 + unit * 4 + e] : 0.f;
            }
        }
        // input-pixel coordinates of this thread's row, advanced by 16 pixels per k-block (no divisions in the loop)
        int qx, qy, qb;
        {
            const int q = kb0 * KP + row;
            qx = q % p.Win;
            const int r = q / p.Win;
            qy = r % p.Hin;
            qb = r / p.Hin;
        }
        constexpr int NBU = 6;                     // dY units per thread per k-block: <= 3 taps x 2 chunks
        constexpr int NAU = 1;                     // x units per thread per k-block
        // Unit slots (j, ch), j = 0..2, ch = 0..1.  Multi-tap layers: tap t = half + 3j, 32-channel chunk ch of <= 2.
        // Single-tap (1x1) layers: tap 0, chunk half + 3*(2j + ch) of <= 4 (an output tile up to 128 channels wide).
        const bool single = taps == 1;
        auto unit_tap = [&](int j) { return single ? 0 : half + GROUPS * j; };
        auto unit_chunk = [&](int j, int ch) { return single ? half + GROUPS * (2 * j + ch) : ch; };
        // tap offsets of this thread's taps, computed once: no divisions in the k-loop
        int toy[NBU / 2], tox[NBU / 2], tky[NBU / 2];
#pragma unroll
        for (int j = 0; j < NBU / 2; ++j) {
            const int t = unit_tap(j);
            const int ky = t / p.KW, kx = t - ky * p.KW;
            toy[j] = ky * p.dil - p.pad;
            tox[j] = kx * p.dil - p.pad;
            tky[j] = ky < p.KH ? ky : 0;
        }
        // shared-memory offsets of this thread's dY units in the densely packed tile: N slot = t*ncol + channel
        uint32_t boff[NBU];
        bool blive[NBU];
#pragma unroll
        for (int j = 0; j < NBU / 2; ++j)
#pragma unroll
            for (int ch = 0; ch < 2; ++ch) {
                const int t = unit_tap(j), cc = unit_chunk(j, ch);
                const int c = unit * 4 + cc * 32;                         // channel within this CTA's group
                const int n = t * ncol + c;
                blive[j * 2 + ch] = t < taps && cc < nb && c < ncol;
                boff[j * 2 + ch] = core_off(n);
            }
        struct Cursor { int qx, qy, qb; };
        Cursor cur = {qx, qy, qb};
        auto advance = [&](Cursor &c) {
            c.qx += KP;
            while (c.qx >= p.Win) {
                c.qx -= p.Win;
                if (++c.qy == p.Hin) { c.qy = 0; ++c.qb; }
            }
        };
        // ---- x~ tile through the load path: this thread's pixel, channels of its chunk
        auto load_x = [&](int it, const Cursor &c_, F4(&va)[NAU], bool &okx) {
            const int q = (kb0 + it) * KP + row;
            okx = q < p.Mq;
            const int sy = UP ? (c_.qy >> 1) : c_.qy, sx = UP ? (c_.qx >> 1) : c_.qx;
            const int xoff = ((c_.qb * p.Hs + sy) * p.Ws + sx) * xs;
#pragma unroll
            for (int ch = 0; ch < NAU; ++ch) {
                const int c = cbx + ch * 32;
                const bool live = xq && okx && c < p.Cin;
                if (VEC) {
                    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
                    if (live) v = __ldg(reinterpret_cast<const float4 *>(xg + xoff + c));
                    if (c + 3 >= p.Cin) {
                        if (c + 1 >= p.Cin) v.y = 0.f;
                        if (c + 2 >= p.Cin) v.z = 0.f;
                        v.w = 0.f;
                    }
                    va[ch].v[0] = v.x; va[ch].v[1] = v.y; va[ch].v[2] = v.z; va[ch].v[3] = v.w;
                } else {
#pragma unroll
                    for (int e = 0; e < 4; ++e) {
                        float v = 0.f;
                        if (live && c + e < p.Cin) v = __ldg(xg + xoff + c + e);
                        va[ch].v[e] = v;
                    }
                }
            }
        };
        // ---- shifted dY tiles through the load path: taps t = half, half+4, ...; output pixel (qy - dy_t, qx - dx_t)
        auto load_d = [&](const Cursor &c_, bool okx, F4(&vb)[NBU]) {
#pragma unroll
            for (int j = 0; j < NBU / 2; ++j) {
                const int t = unit_tap(j);
                const int py = c_.qy - toy[j], px = c_.qx - tox[j];
                const bool okd = okx && t < taps && (unsigned)py < (unsigned)p.Hout && (unsigned)px < (unsigned)p.Wout;
                const int doff = ((c_.qb * p.Hout + py) * p.Wout + px) * dys;
#pragma unroll
                for (int ch = 0; ch < 2; ++ch) {
                    const int c = cbd + unit_chunk(j, ch) * 32;
                    const bool live = okd && blive[j * 2 + ch] && c < p.Cout;
                    F4 &dst = vb[j * 2 + ch];
                    if (VEC) {
                        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
                        if (live) v = __ldg(reinterpret_cast<const float4 *>(dg + doff + c));
                        if (c + 3 >= p.Cout) {
                            if (c + 1 >= p.Cout) v.y = 0.f;
                            if (c + 2 >= p.Cout) v.z = 0.f;
                            v.w = 0.f;
                        }
                        dst.v[0] = v.x; dst.v[1] = v.y; dst.v[2] = v.z; dst.v[3] = v.w;
                    } else {
#pragma unroll
                        for (int e = 0; e < 4; ++e) {
                            float v = 0.f;
                            if (live && c + e < p.Cout) v = __ldg(dg + doff + c + e);
                            dst.v[e] = v;
                        }
                    }
                }
            }
        };
        auto load = [&](int it, F4(&va)[NAU], F4(&vb)[NBU], bool &okx) {
            load_x(it, cur, va, okx);
            load_d(cur, okx, vb);
            advance(cur);
        };
        // ---- the same operands out of a landing-ring slot (TMA): raw x tile [16 px][128 ch], then KH segments [segw px][cg ch]
        auto ring_read = [&](int it, uint32_t slot, F4(&va)[NAU], F4(&vb)[NBU], bool &okx) {
            const int q = (kb0 + it) * KP + row;
            okx = q < p.Mq;
            uint32_t segb = slot;
            if (!UP) {
                float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
                if (xq) v = ld_shared_v4(slot + (uint32_t)((row * BLOCK_CI + half * 32 + unit * 4) * 4));
                va[0].v[0] = v.x; va[0].v[1] = v.y; va[0].v[2] = v.z; va[0].v[3] = v.w;    // channels >= Cin, pixels >= Mq: zero fill
                segb += X_RAW_BYTES;
            }
#pragma unroll
            for (int j = 0; j < NBU / 2; ++j) {
                const int t = unit_tap(j);
                const int py = cur.qy - toy[j], px = cur.qx - tox[j];
                const bool okd = okx && t < taps && (unsigned)py < (unsigned)p.Hout && (unsigned)px < (unsigned)p.Wout;
                const uint32_t rowb = segb + (uint32_t)tky[j] * (uint32_t)p.seg_bytes +
                                      (uint32_t)((row + p.tox_max - tox[j]) * p.cg + unit * 4) * 4u;
#pragma unroll
                for (int ch = 0; ch < 2; ++ch) {
                    F4 &dst = vb[j * 2 + ch];
                    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
                    if (okd && blive[j * 2 + ch]) v = ld_shared_v4(rowb + (uint32_t)unit_chunk(j, ch) * 128u);
                    dst.v[0] = v.x; dst.v[1] = v.y; dst.v[2] = v.z; dst.v[3] = v.w;
                }
            }
            advance(cur);
        };
        auto split_store = [&](uint32_t hi_addr, uint32_t lo_addr, const F4 &v) {
            float hi[4], lo[4];
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const float a = v.v[e];
                const float hh = __uint_as_float((__float_as_uint(a) + 0x1000u) & 0xffffe000u);
                hi[e] = hh;
                lo[e] = a - hh;
            }
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                st_shared_f32(hi_addr + 16u * e, hi[e]);
                st_shared_f32(lo_addr + 16u * e, lo[e]);
            }
        };
        int st_s = 0;
        uint32_t st_ph = 0;
        auto store = [&](int it, F4(&va)[NAU], F4(&vb)[NBU], bool okx) {
            const int s = st_s;
            const uint32_t ph = st_ph;
            if (++st_s == S) { st_s = 0; st_ph ^= 1; }
            if (PRE != 0) {
#pragma unroll
                for (int ch = 0; ch < NAU; ++ch)
#pragma unroll
                    for (int e = 0; e < 4; ++e) {
                        float a = va[ch].v[e];
                        if (AFF) {
                            a = fmaf(a, sc[ch][e], sh[ch][e]);
                            if (RELU) a = fmaxf(a, 0.f);
                            a = okx ? a : 0.f;
                        } else {
                            a = fmaxf(a, 0.f);
                        }
                        va[ch].v[e] = a;
                    }
            }
            mbar_wait(empty(s), ph ^ 1);
            const uint32_t a_hi = base + (uint32_t)s * (uint32_t)p.stage_bytes, a_lo = a_hi + A_BYTES;
            const uint32_t b_hi = a_hi + 2 * A_BYTES, b_lo = b_hi + b_half;
            if (xq) {
                const uint32_t o = core_off(half * 32 + unit * 4);
                split_store(a_hi + o, a_lo + o, va[0]);
            }
#pragma unroll
            for (int j = 0; j < NBU; ++j)
                if (blive[j]) split_store(b_hi + boff[j], b_lo + boff[j], vb[j]);
            fence_proxy_async();
            mbar_arrive(full(s));
        };
        if constexpr (!TMA) {
            F4 a0[NAU], a1[NAU], b0[NBU], b1[NBU];
            bool k0 = false, k1 = false;
            int it = 0;
            if (it < nkb) load(it, a0, b0, k0);
            for (; it < nkb; it += 2) {
                const bool more = it + 1 < nkb;
                if (more) load(it + 1, a1, b1, k1);
                store(it, a0, b0, k0);
                if (more) {
                    if (it + 2 < nkb) load(it + 2, a0, b0, k0);
                    store(it + 1, a1, b1, k1);
                }
            }
        } else {
            // consume the landing ring; an up-sampled x still comes through the load path, one k-block ahead (own cursor)
            F4 xc[NAU], xn[NAU], va[NAU], vb[NBU];
            bool kc = false, kn = false, okx = false;
            Cursor pre = cur;
            if (UP && nkb > 0) { load_x(0, pre, xc, kc); advance(pre); }
            int rj = 0;
            uint32_t rph = 0;
            for (int it = 0; it < nkb; ++it) {
                if (UP && it + 1 < nkb) { load_x(it + 1, pre, xn, kn); advance(pre); }
                mbar_wait(rfull(rj), rph);
                ring_read(it, base + ring_off + (uint32_t)rj * (uint32_t)p.slot_bytes, va, vb, okx);
                mbar_arrive(rempty(rj));               // the slot's values are in registers: the loader may refill it
                if (++rj == p.ring) { rj = 0; rph ^= 1; }
                if (UP) {
                    store(it, xc, vb, okx);
#pragma unroll
                    for (int ch = 0; ch < NAU; ++ch) xc[ch] = xn[ch];
                    kc = kn;
                } else {
                    store(it, va, vb, okx);
                }
            }
        }
    }
}

}  // namespace

// co-group width for the shifted-dY kernel: multiple of 16, taps*cg <= MAX_NT accumulator columns, groups as even as possible
int bts_wgrad2_cg(int Cout, int taps) {
    int cap = (MAX_NT / taps) / 16 * 16;
    if (taps == 1) {
        if (cap > 128) cap = 128;              // 1x1: output tiles up to 128 channels wide
    } else if (cap > 48) {
        cap = 48;
    }
    if (cap < 16) return 0;
    const int groups = (Cout + cap - 1) / cap;
    int cg = ((Cout + groups - 1) / groups + 15) / 16 * 16;
    if (cg > cap) cg = cap;
    return cg;
}

// used on maps of at least 12k pixels (down to the 22x44 maps of DenseNet block 3 at batch 16) with >= 8 k-blocks per
// split-K CTA; smaller maps stay on the tap-in-grid kernel
static long long g_w2_min_pixels = 12000;
static int g_w2_pointwise = 1;               // 1x1 layers (64 < Cout <= 256) on this kernel too
extern "C" int bts_wgrad2_set_pointwise(int on) { g_w2_pointwise = on ? 1 : 0; return 0; }
static int g_w2_min_kb = 8;                  // fewest 16-pixel k-blocks a split-K CTA gets
extern "C" int bts_wgrad2_set_min_pixels(long long n) { g_w2_min_pixels = n < 0 ? 12000 : n; return 0; }
extern "C" int bts_wgrad2_set_min_kblocks(int n) { g_w2_min_kb = n < 1 ? 8 : n; return 0; }

bool bts_wgrad2_eligible(int Cout, int KH, int KW, int stride, long long Mq) {
    const int taps = KH * KW;
    if (stride != 1 || Mq < g_w2_min_pixels || taps > MAX_TAPS || bts_wgrad2_cg(Cout, taps) <= 0) return false;
    if (taps == 1) return g_w2_pointwise && Cout > 64 && Cout <= 256;   // 1x1 layers with 64 < Cout <= 256
    return Cout <= 64;
}

void bts_wgrad2_plan(int B, int Hin, int Win, int Cin, int Cout, int KH, int KW, int *splitK) {
    const int taps = KH * KW;
    const int cg = bts_wgrad2_cg(Cout, taps);
    const long long Mq = (long long)B * Hin * Win;
    const long long KBq = (Mq + KP - 1) / KP;
    const long long tiles = (long long)((Cin + BLOCK_CI - 1) / BLOCK_CI) * ((Cout + cg - 1) / cg);
    const int sms = bts_num_sms();
    long long max_split = (KBq + g_w2_min_kb - 1) / g_w2_min_kb;
    if (max_split < 1) max_split = 1;
    if (max_split > 512) max_split = 512;
    long long split = 1;
    double best = -1.0;
    for (long long sp = 1; sp <= max_split; ++sp) {
        const long long ctas = tiles * sp;
        const long long waves = (ctas + sms - 1) / sms;
        if (waves > 2 && sp > 1) break;
        const double eff = (double)ctas / (double)(waves * sms);
        if (eff > best + 1e-9) { best = eff; split = sp; }      // ties -> fewer splits: less partial traffic for the reduce
    }
    *splitK = (int)split;
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *, const cuuint64_t *,
                                  const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn encode_tiled_fn() {
    static EncodeTiledFn fn = nullptr;
    static bool tried = false;
    if (!tried) {
        tried = true;
        void *ptr = nullptr;
        cudaDriverEntryPointQueryResult qres;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &qres) == cudaSuccess &&
            qres == cudaDriverEntryPointSuccess)
            fn = reinterpret_cast<EncodeTiledFn>(ptr);
    }
    return fn;
}

// [pixels][channels] fp32 view with a pixel stride (channel slices of slabs are fine); box = box_c channels x box_p pixels
static bool make_rows_map(CUtensorMap *map, const float *base, long long pixel_stride, int channels, long long pixels, int box_c,
                          int box_p) {
    EncodeTiledFn fn = encode_tiled_fn();
    if (!fn || box_c > 256 || box_p > 256) return false;
    const cuuint64_t gdim[2] = {(cuuint64_t)channels, (cuuint64_t)pixels};
    const cuuint64_t gstr[1] = {(cuuint64_t)pixel_stride * 4};
    const cuuint32_t box[2] = {(cuuint32_t)box_c, (cuuint32_t)box_p};
    const cuuint32_t estr[2] = {1, 1};
    return fn(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<float *>(base), gdim, gstr, box, estr,
              CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
              CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

static int g_w2_tma = 1;       // 1 (default): landing ring where eligible; 0: producers load from global memory
extern "C" int bts_wgrad2_set_tma(int on) { g_w2_tma = on ? 1 : 0; return 0; }

int bts_wgrad2_launch(const float *x, long long xs, int B, int Hs, int Ws, int up, int Cin, int KH, int KW, int pad,
                      int dil, const float *pre_scale, const float *pre_shift, int pre_relu, const float *dy,
                      long long dys, int Cout, int Hout, int Wout, float *workspace, int splitK, int precision,
                      cudaStream_t st) {
    W2Params p;
    const int taps = KH * KW;
    p.x = x; p.xs = xs; p.B = B; p.Hs = Hs; p.Ws = Ws; p.up = up; p.Cin = Cin;
    p.KH = KH; p.KW = KW; p.pad = pad; p.dil = dil;
    p.pre_scale = pre_scale; p.pre_shift = pre_shift;
    p.dy = dy; p.dys = dys; p.Cout = Cout; p.Hout = Hout; p.Wout = Wout;
    p.Hin = up ? 2 * Hs : Hs; p.Win = up ? 2 * Ws : Ws;
    p.cg = bts_wgrad2_cg(Cout, taps);
    p.nb = (p.cg + 31) / 32;
    p.part = workspace; p.splitK = splitK;
    const long long Mq = (long long)B * p.Hin * p.Win;
    if (Mq > 0x7ffffff0LL) return BTS_EINVAL;
    p.Mq = (int)Mq;
    p.KBq = (int)((Mq + KP - 1) / KP);
    p.kb_per_split = (p.KBq + splitK - 1) / splitK;
    p.nchunks = (taps * p.cg + 31) / 32;
    p.stage_bytes = 2 * A_BYTES + 2 * p.nchunks * 4 * (int)CORE_SBO;
    p.stages = SMEM_BUDGET / p.stage_bytes;
    if (p.stages > MAX_STAGES) p.stages = MAX_STAGES;
    if (p.stages < 2) return BTS_EINVAL;
    p.precision = precision;
    const int pre = (pre_scale ? 2 : 0) | (pre_relu ? 1 : 0);
    const bool vec = bts_aligned16(x) && (xs % 4 == 0) && bts_aligned16(dy) && (dys % 4 == 0);
    // ---- landing ring (TMA): 'same' convolutions with <= 3 kernel rows; 3 operand stages if >= 3 ring slots still fit, else 2
    CUtensorMap tmx, tmd;
    memset(&tmx, 0, sizeof(tmx));
    memset(&tmd, 0, sizeof(tmd));
    bool tma = false;
    p.ring = p.slot_bytes = p.seg_bytes = p.segw = p.tox_max = p.slot_tx = 0;
    if (g_w2_tma && vec && KH <= 3 && Hout == p.Hin && Wout == p.Win) {
        p.segw = KP + (KW - 1) * dil;
        p.tox_max = (KW - 1) * dil - pad;
        p.seg_bytes = (p.segw * p.cg * 4 + 127) / 128 * 128;
        p.slot_bytes = (up ? 0 : X_RAW_BYTES) + KH * p.seg_bytes;
        p.slot_tx = (up ? 0 : X_RAW_BYTES) + KH * p.segw * p.cg * 4;
        int st_try = p.stages > 3 ? 3 : p.stages;
        for (; st_try >= 2 && !tma; --st_try) {
            const int ring = (SMEM_BUDGET - st_try * p.stage_bytes) / p.slot_bytes;
            if (ring >= 3 || (st_try == 2 && ring >= 2)) {
                p.stages = st_try;
                p.ring = ring > MAX_RING ? MAX_RING : ring;
                tma = true;
            }
        }
        if (tma && p.segw <= 256)
            tma = make_rows_map(&tmd, dy, dys, Cout, (long long)B * Hout * Wout, p.cg, p.segw) &&
                  (up || make_rows_map(&tmx, x, xs, Cin, Mq, BLOCK_CI, KP));
        else
            tma = false;
        if (!tma) {
            p.ring = 0;
            p.stages = SMEM_BUDGET / p.stage_bytes > MAX_STAGES ? MAX_STAGES : SMEM_BUDGET / p.stage_bytes;
        }
    }
    const int smem = p.stages * p.stage_bytes + p.ring * p.slot_bytes + 2 * BLOCK_CI * 4 + 256 + 1024;
    dim3 grid((Cin + BLOCK_CI - 1) / BLOCK_CI, (Cout + p.cg - 1) / p.cg, splitK);
    cudaError_t err = cudaSuccess;
#define BTS_LAUNCH(PRE, UP, VEC, TMA)                                                                                 \
    do {                                                                                                              \
        static int attr_smem_[BTS_MAX_DEVICES] = {}; int &attr_smem = attr_smem_[bts_cur_device()];                   \
        if (attr_smem < smem) {                                                                                       \
            err = cudaFuncSetAttribute(wgrad2_tc_kernel<PRE, UP, VEC, TMA>, cudaFuncAttributeMaxDynamicSharedMemorySize, \
                                       SMEM_BUDGET + 2 * BLOCK_CI * 4 + 256 + 1024);                                  \
            if (err != cudaSuccess) return (int)err;                                                                  \
            attr_smem = SMEM_BUDGET + 2 * BLOCK_CI * 4 + 256 + 1024;                                                  \
        }                                                                                                             \
        wgrad2_tc_kernel<PRE, UP, VEC, TMA><<<grid, NUM_THREADS, smem, st>>>(p, tmx, tmd);                            \
    } while (0)
#define BTS_DISPATCH_UV(PRE)                                                                     \
    do {                                                                                         \
        if (tma) { if (p.up) BTS_LAUNCH(PRE, true, true, true); else BTS_LAUNCH(PRE, false, true, true); } \
        else if (p.up) { if (vec) BTS_LAUNCH(PRE, true, true, false); else BTS_LAUNCH(PRE, true, false, false); }   \
        else { if (vec) BTS_LAUNCH(PRE, false, true, false); else BTS_LAUNCH(PRE, false, false, false); }      \
    } while (0)
    switch (pre) {
        case 0: BTS_DISPATCH_UV(0); break;
        case 1: BTS_DISPATCH_UV(1); break;
        case 2: BTS_DISPATCH_UV(2); break;
        default: BTS_DISPATCH_UV(3); break;
    }
#undef BTS_DISPATCH_UV
#undef BTS_LAUNCH
    BTS_LAUNCH_CHECK();
    return 0;
}
