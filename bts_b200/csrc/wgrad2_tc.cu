// wgrad for narrow-output 3x3 convolutions (Cout <= 64: the DenseNet 3x3 dense-layer convs 192->48 and the full- /
// half-resolution decoder convs conv1/upconv1/conv2/upconv2) and for 1x1 layers with 64 < Cout <= 256, on the Hopper
// tensor cores (wgmma, register accumulators), 3xTF32 -- "shifted dY" formulation.
//
//   dW[co, ci, tap] = sum_q  x~[q, ci] * dY[q - off(tap), co]            q = INPUT pixel, off(tap) = tap*dil - pad
//
// wgrad_tc.cu puts the tap in the grid, so the activation tile -- the expensive operand: loads, BN/ReLU pre-op, hi/lo
// split, shared-memory writes per k-block -- is produced once per tap.  Here ONE CTA owns all taps of a (64 ci, cg co)
// block: per k-block of 32 input pixels the activation tile is produced once and multiplied against the shifted dY tiles
// of every tap, packed densely along N (tap t owns the N slots [t*ncol, (t+1)*ncol)), so that wgmma of width
// taps*ncol <= 144 covers them all; two consumer warpgroups split those columns (<= 40 accumulator registers per thread).
//   A = x: staged once per k-block as fp32 in its NHWC order ([pixel][64 channels], pre-op and zero padding applied);
//       every consumer thread loads its tf32 fragments from it, splits them into hi/lo in registers and issues
//       register-A wgmma.
//   B = dY: K-major (pixels contiguous per column) hi/lo tiles of 8 x 16-byte core matrices, transposed by the producers.
// Deterministic split-K partial layout as wgrad_tc.cu; split-K ranges are whole multiples of 16 pixels.
// 512 threads (16 warps, 128 registers per thread): 2 consumer warpgroups + 2 producer warpgroups.
// Single-pass TF32 (precision=1, opt-in) runs wgrad2_tf32_kernel, the same body compiled for one product: one dY tile
// (hi) per stage and A_hi*B_hi per k8 step.
//
// Operand staging: the shifted dY windows of a k-block overlap -- they are KH row segments of 32 + (KW-1)*dil consecutive
// output pixels.  With TMA = true one producer lane copies the raw fp32 segments (and the raw x tile unless it is read
// through the nearest-neighbour up-sample) into a small landing ring, `ring` k-blocks ahead (cp.async.bulk.tensor.2d, no
// swizzle, zero fill past the tensor ends); the producers then read shared memory, apply the border masks / pre-op and
// write the operand tiles.
#include <cuda.h>

#include <cstring>
#include <type_traits>

#include "tc_common.cuh"

using namespace tc;

namespace {

constexpr int BLOCK_CI = 64;                 // input channels per CTA = the M of one consumer warpgroup
constexpr int KP = 32;                       // input pixels per k-block (4 k8 steps)
constexpr int SPLIT_PX = 16;                 // split-K ranges are whole multiples of this many pixels (bts_wgrad2_plan)
constexpr uint32_t CORE_SBO = KP / 4 * 128 + 16;   // one 8-column group of a k-block: 8 core matrices along K + a bank pad
constexpr int X_ROW_BYTES = BLOCK_CI * 4;    // one pixel of the x tile: 64 fp32 channels
constexpr int X_BYTES = KP * X_ROW_BYTES;    // x tile of a k-block (stage and landing ring): 8 KB
constexpr int MAX_TAPS = 9;
constexpr int MAX_NT = 144;                  // widest packed N (taps * ncol), split between the two consumer warpgroups
constexpr int MAX_CHUNKS = (MAX_NT + 31) / 32;   // 32-column chunks of the packed dY tile
constexpr int MAX_STAGES = 4;
constexpr int CONSUMER_THREADS = 256;       // two warpgroups, each owns about half of the packed N columns
constexpr int PRODUCERS = 256;
constexpr int NUM_THREADS = CONSUMER_THREADS + PRODUCERS;
constexpr int SMEM_BUDGET = 224 * 1024;
constexpr int MAX_RING = 4;                  // landing-ring slots (TMA staging)

struct W2Params {
    const float *x; long long xs;
    int B, Hs, Ws, up, Cin;
    int KH, KW, pad, dil;
    const float *pre_scale, *pre_shift;
    const float *dy; long long dys;
    int Cout, Hout, Wout, Hin, Win;
    int cg;                  // output channels per CTA (multiple of 16)
    float *part;             // [splitK][taps][Cin][Cout]
    int splitK, px_per_split;
    int Mq;                  // B*Hin*Win input pixels
    int stages, stage_bytes, b_half;   // stage = [x X_BYTES | dY hi b_half | dY lo b_half] (single pass: no lo)
    // TMA landing ring (TMA = true): slot = [raw x tile (unless up) | KH segments of segw pixels x cg channels]
    int ring, slot_bytes, seg_bytes, segw, tox_max, slot_tx;
};

// SINGLE: single-pass TF32 (wgrad2_tf32_kernel) instead of 3xTF32 (wgrad2_tc_kernel)
template <int PRE, bool UP, bool VEC, bool TMA, bool SINGLE>
__device__ __forceinline__ void wgrad2_body(const W2Params &p, const CUtensorMap &tmx, const CUtensorMap &tmd) {
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;
    uint8_t *sm = smem_raw + (base - smem_u32(smem_raw));
    const int taps = p.KH * p.KW;
    const int S = p.stages;
    const uint32_t stage_bytes = (uint32_t)p.stage_bytes;
    const uint32_t ring_off = (uint32_t)S * stage_bytes;
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
    // dY operand: the taps are packed DENSELY along N -- tap t owns the N columns [t*ncol, (t+1)*ncol) -- so that a single
    // wgmma multiplies the activation tile against all taps at once.  hi and lo tiles follow each other.
    const int n_total = taps * ncol;
    const int q_begin = split * p.px_per_split;                      // this CTA's input pixels [q_begin, q_end)
    const int q_end = min(q_begin + p.px_per_split, p.Mq);
    const int nkb = q_end > q_begin ? (q_end - q_begin + KP - 1) / KP : 0;

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
    // (no zero fill of the stages: the producers write every byte of a stage that is read, dead channels as zeros)
    __syncthreads();

    if (warp < CONSUMER_THREADS / 32) {
        // ---- consumer warpgroups: rows = the 64 input channels; warpgroup wg owns the packed columns [n0, n0 + N) of
        //      all taps x ncol (n0 = 0 | the first half rounded up to 16).  Per k-block every thread loads its A fragments
        //      from the fp32 x tile, splits them into hi/lo in registers and issues per k8 step A_lo*B_hi, A_hi*B_lo,
        //      A_hi*B_hi (small cross terms first); a stage is released as soon as its wgmma group has completed
        const int wg = warp >> 2;
        const int n_half = (n_total + 31) / 32 * 16;
        const int n0 = wg ? n_half : 0, n_mine = wg ? n_total - n_half : n_half;
        // A fragment of k8 step k (wgmma_tf32.cuh): rows = channels c, c + 8 with c = 16 (warp % 4) + lane / 4, columns =
        // pixels 8k + q, 8k + q + 4 with q = lane % 4.  Pixel r of the x tile is the 256-byte row r (64 banks: a multiple
        // of 32), its 16-byte chunk u (channels 4u..4u+3) stored at chunk u ^ 2 (r % 4).  The 8 channels of one load span
        // chunks u0, u0 + 1 (u0 = 4 (warp % 4), so u0 % 8 is 0 or 4); XOR-ing 2q into bits 1-2 sends the 4 pixels to the
        // 4 distinct pairs of chunks mod 8, so the 8 channels x 4 pixels hit 32 distinct banks.  r % 4 == q for every
        // fragment of the thread, and chunk(c + 8) = chunk(c) ^ 2 (c % 16 < 8), so channel c + 8 sits at byte offset aF ^ 32.
        const int q = lane & 3;
        const int c = (warp & 3) * 16 + (lane >> 2);
        const uint32_t aF = (uint32_t)q * X_ROW_BYTES + ((uint32_t)((c >> 2) ^ (2 * q)) << 4) + (uint32_t)(c & 3) * 4u;
        auto consume = [&](auto NT) {
            constexpr int N = decltype(NT)::value;
            float acc[N > 0 ? N / 2 : 1];
#pragma unroll
            for (int i = 0; i < (N > 0 ? N / 2 : 1); ++i) acc[i] = 0.f;
            int s = 0;
            uint32_t ph = 0;
            for (int it = 0; it < nkb; ++it) {
                mbar_wait(full(s), ph);
                if constexpr (N > 0) {
                    const uint32_t st = base + (uint32_t)s * stage_bytes;
                    if constexpr (SINGLE) {
                        uint32_t hi[KP / 8][4];
#pragma unroll
                        for (int k = 0; k < KP / 8; ++k) {
#pragma unroll
                            for (int j = 0; j < 4; ++j) {              // j: row + 8 (j & 1), column + 4 (j >> 1)
                                const uint32_t x = ld_shared_u32(st + (aF ^ (32u * (j & 1))) + (uint32_t)(8 * k + 4 * (j >> 1)) * X_ROW_BYTES);
                                hi[k][j] = __float_as_uint(round_tf32(__uint_as_float(x)));
                            }
                        }
                        const uint32_t b_hi = st + X_BYTES + (uint32_t)(n0 >> 3) * CORE_SBO;
                        wgmma_fence();
#pragma unroll
                        for (int k = 0; k < KP / 8; ++k) {
                            const uint64_t dbh = make_desc_core(b_hi + (uint32_t)k * 256u, 128, CORE_SBO);
                            Wgmma<N>::mma_rs(acc, hi[k], dbh, (it | k) != 0);
                        }
                        wgmma_commit();
                        wgmma_wait<0>();
                        wgmma_fence_operands(acc);
#pragma unroll
                        for (int k = 0; k < KP / 8; ++k) wgmma_fence_operands(hi[k]);
                    } else {
                        uint32_t hi[KP / 8][4], lo[KP / 8][4];
#pragma unroll
                        for (int k = 0; k < KP / 8; ++k) {
#pragma unroll
                            for (int j = 0; j < 4; ++j) {              // j: row + 8 (j & 1), column + 4 (j >> 1)
                                const uint32_t x = ld_shared_u32(st + (aF ^ (32u * (j & 1))) + (uint32_t)(8 * k + 4 * (j >> 1)) * X_ROW_BYTES);
                                float h, l;
                                split_tf32(__uint_as_float(x), h, l);
                                hi[k][j] = __float_as_uint(h);
                                lo[k][j] = __float_as_uint(l);
                            }
                        }
                        const uint32_t b_hi = st + X_BYTES + (uint32_t)(n0 >> 3) * CORE_SBO, b_lo = b_hi + (uint32_t)p.b_half;
                        wgmma_fence();
#pragma unroll
                        for (int k = 0; k < KP / 8; ++k) {
                            const uint32_t ko = (uint32_t)k * 256u;
                            const uint64_t dbh = make_desc_core(b_hi + ko, 128, CORE_SBO), dbl = make_desc_core(b_lo + ko, 128, CORE_SBO);
                            const uint32_t accumulate = (it | k) != 0;
                            Wgmma<N>::mma_rs(acc, lo[k], dbh, accumulate);
                            Wgmma<N>::mma_rs(acc, hi[k], dbl, 1);
                            Wgmma<N>::mma_rs(acc, hi[k], dbh, 1);
                        }
                        wgmma_commit();
                        wgmma_wait<0>();
                        wgmma_fence_operands(acc);
#pragma unroll
                        for (int k = 0; k < KP / 8; ++k) {
                            wgmma_fence_operands(hi[k]);
                            wgmma_fence_operands(lo[k]);
                        }
                    }
                }
                mbar_arrive(empty(s));
                if (++s == S) { s = 0; ph ^= 1; }
            }
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
        // ---- producers: 8 warps.  Thread pt owns pixel row r = pt / 8 of every k-block and the 4-channel unit ul = pt % 8
        //      of each 32-channel chunk: the x channels 4 ul and 32 + 4 ul, and the packed dY columns n = 32 ch + 4 ul of
        //      every chunk with n < taps * ncol (tap n / ncol, output channel co0 + n % ncol).  A warp covers 4 pixels x 8 units.
        const int pt = threadIdx.x - CONSUMER_THREADS;
        const int ul = pt & 7;
        const int row = pt >> 3;
        constexpr bool AFF = PRE >= 2;
        constexpr bool RELU = (PRE & 1) != 0;
        // x tile: the unit's 16 bytes go to chunk ul ^ 2 (row % 4) of the pixel's 256-byte row (chunk + 8 for the second
        // unit).  Each 8-lane phase of a 128-bit store writes the 8 chunks of one pixel, which the XOR only permutes: no
        // bank conflict.
        const uint32_t xoff = (uint32_t)row * X_ROW_BYTES + ((uint32_t)(ul ^ (2 * (row & 3))) << 4);
        // dY tiles, K-major core matrices: element (column n, pixel k) at (n / 8) * CORE_SBO + (k / 4) * 128 + (n % 8) * 16 +
        // (k % 4) * 4, a unit = 4 scalar stores 16 bytes apart.  In 32-bit words CORE_SBO = 260 = 4 (mod 32) and a 4-pixel
        // group is 32 words, so the bank is 4 ((n / 8) + (n % 8)) + k % 4 (mod 32).  A warp's 8 units of one chunk give
        // (n / 8) + (n % 8) = 4 ch + ul / 2 + 4 (ul % 2) + e, 8 distinct values mod 8, and its 4 pixels distinct k % 4: each
        // scalar store hits 32 distinct banks.
        auto core_off = [&](int n) {
            return (uint32_t)(n >> 3) * CORE_SBO + (uint32_t)(row >> 2) * 128u + (uint32_t)(n & 7) * 16u + (uint32_t)(row & 3) * 4u;
        };
        const int xs = (int)p.xs, dys = (int)p.dys;
        const int cbx = ci_tile * BLOCK_CI + ul * 4;                  // first x channel of this thread's first unit
        const float *__restrict__ xg = p.x;
        const float *__restrict__ dg = p.dy;
        // The pre-op's scale / shift stay in 16 registers, except on the scalar-load path (VEC = false), which holds four
        // times the loads in flight: it reads them from shared memory at each use and so stays within 128 registers
        // without spills (the same values: the same results).
        constexpr bool AFF_REGS = AFF && VEC;
        float sc[2][4], sh[2][4];
        if (AFF_REGS) {
#pragma unroll
            for (int h = 0; h < 2; ++h)
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    sc[h][e] = s_scale[h * 32 + ul * 4 + e];          // 0 beyond Cin
                    sh[h][e] = s_shift[h * 32 + ul * 4 + e];
                }
        }
        // this thread's dY units, computed once (no divisions in the k-loop): tap offsets, channel within the group,
        // shared-memory offset in the packed tile and in a landing-ring slot
        int toy[MAX_CHUNKS], tox[MAX_CHUNKS], ucol[MAX_CHUNKS];
        uint32_t boff[MAX_CHUNKS], roff[MAX_CHUNKS];
        bool blive[MAX_CHUNKS];
#pragma unroll
        for (int ch = 0; ch < MAX_CHUNKS; ++ch) {
            const int n = ch * 32 + ul * 4;
            blive[ch] = n < n_total;
            const int t = blive[ch] ? n / ncol : 0;
            const int ky = t / p.KW, kx = t - ky * p.KW;
            toy[ch] = ky * p.dil - p.pad;
            tox[ch] = kx * p.dil - p.pad;
            ucol[ch] = n - t * ncol;
            boff[ch] = core_off(n);
            roff[ch] = (uint32_t)ky * (uint32_t)p.seg_bytes + (uint32_t)((row + p.tox_max - tox[ch]) * p.cg + ucol[ch]) * 4u;
        }
        // input-pixel coordinates of this thread's row, advanced by KP pixels per k-block (no divisions in the loop)
        struct Cursor { int qx, qy, qb; };
        Cursor cur;
        {
            const int q = q_begin + row;
            cur.qx = q % p.Win;
            const int r = q / p.Win;
            cur.qy = r % p.Hin;
            cur.qb = r / p.Hin;
        }
        auto advance = [&](Cursor &c) {
            c.qx += KP;
            while (c.qx >= p.Win) {
                c.qx -= p.Win;
                if (++c.qy == p.Hin) { c.qy = 0; ++c.qb; }
            }
        };
        auto pixel_ok = [&](int it) { return q_begin + it * KP + row < q_end; };
        // ---- x~ tile through the load path: this thread's pixel, its two 4-channel units
        auto load_x = [&](int it, const Cursor &c_, F4(&va)[2], bool &okx) {
            okx = pixel_ok(it);
            const int sy = UP ? (c_.qy >> 1) : c_.qy, sx = UP ? (c_.qx >> 1) : c_.qx;
            const int xo = ((c_.qb * p.Hs + sy) * p.Ws + sx) * xs;
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int c = cbx + h * 32;
                const bool live = okx && c < p.Cin;
                if (VEC) {
                    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
                    if (live) v = __ldg(reinterpret_cast<const float4 *>(xg + xo + c));
                    if (c + 3 >= p.Cin) {
                        if (c + 1 >= p.Cin) v.y = 0.f;
                        if (c + 2 >= p.Cin) v.z = 0.f;
                        v.w = 0.f;
                    }
                    va[h].v[0] = v.x; va[h].v[1] = v.y; va[h].v[2] = v.z; va[h].v[3] = v.w;
                } else {
#pragma unroll
                    for (int e = 0; e < 4; ++e) {
                        float v = 0.f;
                        if (live && c + e < p.Cin) v = __ldg(xg + xo + c + e);
                        va[h].v[e] = v;
                    }
                }
            }
        };
        // ---- shifted dY units through the load path: output pixel (qy - toy, qx - tox) of the unit's tap
        auto load_d = [&](const Cursor &c_, bool okx, F4(&vb)[MAX_CHUNKS]) {
#pragma unroll
            for (int ch = 0; ch < MAX_CHUNKS; ++ch) {
                const int py = c_.qy - toy[ch], px = c_.qx - tox[ch];
                const bool okd = okx && blive[ch] && (unsigned)py < (unsigned)p.Hout && (unsigned)px < (unsigned)p.Wout;
                const int doff = ((c_.qb * p.Hout + py) * p.Wout + px) * dys;
                const int c = co0 + ucol[ch];
                const bool live = okd && c < p.Cout;
                F4 &dst = vb[ch];
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
        };
        auto load = [&](int it, F4(&va)[2], F4(&vb)[MAX_CHUNKS], bool &okx) {
            load_x(it, cur, va, okx);
            load_d(cur, okx, vb);
            advance(cur);
        };
        // ---- the same operands out of a landing-ring slot (TMA): raw x tile [32 px][64 ch], then KH segments [segw px][cg ch]
        auto ring_read = [&](int it, uint32_t slot, F4(&va)[2], F4(&vb)[MAX_CHUNKS], bool &okx) {
            okx = pixel_ok(it);
            uint32_t segb = slot;
            if (!UP) {
#pragma unroll
                for (int h = 0; h < 2; ++h) {   // channels >= Cin and pixels >= Mq arrive as zeros (TMA zero fill)
                    const float4 v = ld_shared_v4(slot + (uint32_t)(row * X_ROW_BYTES + (h * 32 + ul * 4) * 4));
                    va[h].v[0] = v.x; va[h].v[1] = v.y; va[h].v[2] = v.z; va[h].v[3] = v.w;
                }
                segb += X_BYTES;
            }
#pragma unroll
            for (int ch = 0; ch < MAX_CHUNKS; ++ch) {
                const int py = cur.qy - toy[ch], px = cur.qx - tox[ch];
                const bool okd = okx && blive[ch] && (unsigned)py < (unsigned)p.Hout && (unsigned)px < (unsigned)p.Wout;
                float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
                if (okd) v = ld_shared_v4(segb + roff[ch]);
                vb[ch].v[0] = v.x; vb[ch].v[1] = v.y; vb[ch].v[2] = v.z; vb[ch].v[3] = v.w;
            }
            advance(cur);
        };
        int st_s = 0;
        uint32_t st_ph = 0;
        auto store = [&](F4(&va)[2], F4(&vb)[MAX_CHUNKS], bool okx) {
            const int s = st_s;
            const uint32_t ph = st_ph;
            if (++st_s == S) { st_s = 0; st_ph ^= 1; }
#pragma unroll
            for (int h = 0; h < 2; ++h)
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    float a = va[h].v[e];
                    if (AFF_REGS) a = fmaf(a, sc[h][e], sh[h][e]);
                    else if (AFF) a = fmaf(a, s_scale[h * 32 + ul * 4 + e], s_shift[h * 32 + ul * 4 + e]);
                    if (RELU) a = fmaxf(a, 0.f);
                    va[h].v[e] = okx ? a : 0.f;        // pixels past this CTA's range (zero padding after the pre-op)
                }
            mbar_wait(empty(s), ph ^ 1);
            const uint32_t st = base + (uint32_t)s * stage_bytes;
#pragma unroll
            for (int h = 0; h < 2; ++h)
                st_shared_v4(st + xoff + 128u * h, va[h].v[0], va[h].v[1], va[h].v[2], va[h].v[3]);
            const uint32_t b_hi = st + X_BYTES, b_lo = b_hi + (uint32_t)p.b_half;
#pragma unroll
            for (int ch = 0; ch < MAX_CHUNKS; ++ch) {
                if (!blive[ch]) continue;
                if constexpr (SINGLE) {
#pragma unroll
                    for (int e = 0; e < 4; ++e) st_shared_f32(b_hi + boff[ch] + 16u * e, round_tf32(vb[ch].v[e]));
                } else {
                    float hi[4], lo[4];
#pragma unroll
                    for (int e = 0; e < 4; ++e) split_tf32(vb[ch].v[e], hi[e], lo[e]);
#pragma unroll
                    for (int e = 0; e < 4; ++e) {
                        st_shared_f32(b_hi + boff[ch] + 16u * e, hi[e]);
                        st_shared_f32(b_lo + boff[ch] + 16u * e, lo[e]);
                    }
                }
            }
            fence_proxy_async();                       // generic-proxy dY writes -> visible to wgmma (async proxy)
            mbar_arrive(full(s));
        };
        if constexpr (!TMA) {
            F4 a0[2], a1[2], b0[MAX_CHUNKS], b1[MAX_CHUNKS];
            bool k0 = false, k1 = false;
            int it = 0;
            if (it < nkb) load(it, a0, b0, k0);
            for (; it < nkb; it += 2) {
                const bool more = it + 1 < nkb;
                if (more) load(it + 1, a1, b1, k1);
                store(a0, b0, k0);
                if (more) {
                    if (it + 2 < nkb) load(it + 2, a0, b0, k0);
                    store(a1, b1, k1);
                }
            }
        } else {
            // landing ring: producer thread 0 fills slot j with k-block `it` and refills it with k-block it + ring as soon
            // as every producer has released it.  An up-sampled x still comes through the load path, one k-block ahead.
            auto issue = [&](int it, int j) {
                const uint32_t dst = base + ring_off + (uint32_t)j * (uint32_t)p.slot_bytes;
                const int q0 = q_begin + it * KP;
                mbar_arrive_expect_tx(rfull(j), (uint32_t)p.slot_tx);
                uint32_t seg = dst;
                if (!UP) {
                    tma_tile_2d(dst, &tmx, ci_tile * BLOCK_CI, q0, rfull(j));
                    seg += X_BYTES;
                }
                for (int ky = 0; ky < p.KH; ++ky)     // output pixels q - (ky*dil - pad)*W - tox, tox <= tox_max
                    tma_tile_2d(seg + (uint32_t)ky * (uint32_t)p.seg_bytes, &tmd, co0,
                                q0 - (ky * p.dil - p.pad) * p.Wout - p.tox_max, rfull(j));
            };
            if (pt == 0) {
                if (!UP) tma_prefetch_desc(&tmx);
                tma_prefetch_desc(&tmd);
                for (int it = 0; it < nkb && it < p.ring; ++it) issue(it, it);
            }
            F4 xc[2], xn[2], va[2], vb[MAX_CHUNKS];
            bool kc = false, kn = false, okx = false;
            Cursor pre = cur;
            if (UP && nkb > 0) { load_x(0, pre, xc, kc); advance(pre); }
            int rj = 0;
            uint32_t rph = 0;
            for (int it = 0; it < nkb; ++it) {
                if (UP && it + 1 < nkb) { load_x(it + 1, pre, xn, kn); advance(pre); }
                mbar_wait(rfull(rj), rph);
                ring_read(it, base + ring_off + (uint32_t)rj * (uint32_t)p.slot_bytes, va, vb, okx);
                mbar_arrive(rempty(rj));               // the slot's values are in registers
                if (pt == 0 && it + p.ring < nkb) {
                    mbar_wait(rempty(rj), rph);
                    issue(it + p.ring, rj);
                }
                if (++rj == p.ring) { rj = 0; rph ^= 1; }
                if (UP) {
                    store(xc, vb, okx);
#pragma unroll
                    for (int h = 0; h < 2; ++h) xc[h] = xn[h];
                    kc = kn;
                } else {
                    store(va, vb, okx);
                }
            }
        }
    }
}

template <int PRE, bool UP, bool VEC, bool TMA>
__global__ void __launch_bounds__(NUM_THREADS, 1) wgrad2_tc_kernel(const W2Params p, const __grid_constant__ CUtensorMap tmx,
                                                                   const __grid_constant__ CUtensorMap tmd) {
    wgrad2_body<PRE, UP, VEC, TMA, false>(p, tmx, tmd);
}

template <int PRE, bool UP, bool VEC, bool TMA>
__global__ void __launch_bounds__(NUM_THREADS, 1) wgrad2_tf32_kernel(const W2Params p, const __grid_constant__ CUtensorMap tmx,
                                                                     const __grid_constant__ CUtensorMap tmd) {
    wgrad2_body<PRE, UP, VEC, TMA, true>(p, tmx, tmd);
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

// used on maps of at least 12k pixels (down to the 22x44 maps of DenseNet block 3 at batch 16) with >= 8 blocks of 16
// pixels per split-K CTA; smaller maps stay on the tap-in-grid kernel
static long long g_w2_min_pixels = 12000;
static int g_w2_pointwise = 1;               // 1x1 layers (64 < Cout <= 256) on this kernel too
extern "C" int bts_wgrad2_set_pointwise(int on) { g_w2_pointwise = on ? 1 : 0; return 0; }
static int g_w2_min_kb = 8;                  // fewest 16-pixel blocks (SPLIT_PX) a split-K CTA gets
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
    const long long KBq = (Mq + SPLIT_PX - 1) / SPLIT_PX;
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
    p.part = workspace; p.splitK = splitK;
    const long long Mq = (long long)B * p.Hin * p.Win;
    if (Mq > 0x7ffffff0LL) return BTS_EINVAL;
    p.Mq = (int)Mq;
    const int blocks = (int)((Mq + SPLIT_PX - 1) / SPLIT_PX);
    p.px_per_split = (blocks + splitK - 1) / splitK * SPLIT_PX;
    p.b_half = taps * p.cg / 8 * (int)CORE_SBO;
    p.stage_bytes = (X_BYTES + (precision ? 1 : 2) * p.b_half + 127) / 128 * 128;   // ring slots stay 128-byte aligned
    p.stages = SMEM_BUDGET / p.stage_bytes;
    if (p.stages > MAX_STAGES) p.stages = MAX_STAGES;
    if (p.stages < 2) return BTS_EINVAL;
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
        p.slot_bytes = (up ? 0 : X_BYTES) + KH * p.seg_bytes;
        p.slot_tx = (up ? 0 : X_BYTES) + KH * p.segw * p.cg * 4;
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
#define BTS_LAUNCH(KERNEL, PRE, UP, VEC, TMA)                                                                         \
    do {                                                                                                              \
        static int attr_smem_[BTS_MAX_DEVICES] = {}; int &attr_smem = attr_smem_[bts_cur_device()];                   \
        if (attr_smem < smem) {                                                                                       \
            err = cudaFuncSetAttribute(KERNEL<PRE, UP, VEC, TMA>, cudaFuncAttributeMaxDynamicSharedMemorySize,        \
                                       SMEM_BUDGET + 2 * BLOCK_CI * 4 + 256 + 1024);                                  \
            if (err != cudaSuccess) return (int)err;                                                                  \
            attr_smem = SMEM_BUDGET + 2 * BLOCK_CI * 4 + 256 + 1024;                                                  \
        }                                                                                                             \
        KERNEL<PRE, UP, VEC, TMA><<<grid, NUM_THREADS, smem, st>>>(p, tmx, tmd);                                      \
    } while (0)
#define BTS_DISPATCH_UV(KERNEL, PRE)                                                                                  \
    do {                                                                                                              \
        if (tma) { if (p.up) BTS_LAUNCH(KERNEL, PRE, true, true, true); else BTS_LAUNCH(KERNEL, PRE, false, true, true); } \
        else if (p.up) { if (vec) BTS_LAUNCH(KERNEL, PRE, true, true, false); else BTS_LAUNCH(KERNEL, PRE, true, false, false); } \
        else { if (vec) BTS_LAUNCH(KERNEL, PRE, false, true, false); else BTS_LAUNCH(KERNEL, PRE, false, false, false); } \
    } while (0)
#define BTS_DISPATCH(KERNEL)                                                                                          \
    do {                                                                                                              \
        switch (pre) {                                                                                                \
            case 0: BTS_DISPATCH_UV(KERNEL, 0); break;                                                                \
            case 1: BTS_DISPATCH_UV(KERNEL, 1); break;                                                                \
            case 2: BTS_DISPATCH_UV(KERNEL, 2); break;                                                                \
            default: BTS_DISPATCH_UV(KERNEL, 3); break;                                                               \
        }                                                                                                             \
    } while (0)
    if (precision) BTS_DISPATCH(wgrad2_tf32_kernel);
    else BTS_DISPATCH(wgrad2_tc_kernel);
#undef BTS_DISPATCH
#undef BTS_DISPATCH_UV
#undef BTS_LAUNCH
    BTS_LAUNCH_CHECK();
    return 0;
}
