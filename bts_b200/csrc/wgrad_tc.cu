// Weight-gradient (wgrad) of the implicit-GEMM convolution on the Hopper tensor cores (wgmma), sm_90a, 3xTF32.
//
//   dW[co, ci, tap] = sum_p  dY[p, co] * pre(x[p (+) tap, ci])            (same pre / (+) as conv_tc.cu)
//
// GEMM view per (tap, split):  M = 128 input channels (two consumer warpgroups of 64), N = n_tile <= 64 output channels,
// K = output pixels.  Both operands live in memory as [pixel][channel] (NHWC), i.e. the reduction index is the slow one.
//   A = x: staged once per k-block as fp32 in its NHWC order ([pixel][channel], pre-op and zero padding applied); every
//       consumer thread loads its tf32 fragments from it, splits them into hi/lo in registers and issues register-A wgmma.
//   B = dY: tf32 wgmma reads shared-memory operands K-major only, so the producers transpose dY on its way into shared
//       memory, split into hi/lo tiles of 8 x 16-byte core matrices (no swizzle).
// grid = (ceil(Cin/128), n_tiles(Cout), taps * splitK); each CTA reduces its pixel range into fp32 register accumulators
// and writes a partial; a second, deterministic kernel sums the splitK partials into the (Cout,Cin,KH,KW)-strided gradient.
// 512 threads (16 warps, 128 registers per thread): 2 consumer warpgroups + 2 producer warpgroups (x tile / dY tile),
// 2-6 operand stages.
// Single-pass TF32 (precision=1, opt-in) runs wgrad_tf32_kernel, the same body compiled for one product: the dY producers
// write only the hi tile, a stage is x + dY hi, and the consumers issue A_hi*B_hi per k8 step (A rounded as hi is).
#include <cstdlib>
#include <type_traits>

#include "tc_common.cuh"

using namespace tc;

namespace {

constexpr int BLOCK_CI = 128;
constexpr int BLOCK_KP = 32;                 // pixels per k-block
constexpr int MAX_N = 64;                    // output channels per CTA tile (register accumulator of the consumers)
constexpr int MAX_STAGES = 6;
constexpr int SMEM_LIMIT = 232448;
constexpr uint32_t CORE_SBO = 8 * 128 + 16;  // one 8-channel group of a k-block: 8 core matrices along K + a bank pad
constexpr int X_ROW_BYTES = BLOCK_CI * 4;    // one pixel of the x tile: 128 fp32 channels
constexpr int X_BYTES = BLOCK_KP * X_ROW_BYTES;
constexpr int CONSUMER_THREADS = 256;
constexpr int GROUP_THREADS = 128;
constexpr int NUM_THREADS = CONSUMER_THREADS + 2 * GROUP_THREADS;

struct WgradParams {
    const float *x; long long xs;
    int B, Hs, Ws, up, Cin;
    int KH, KW, stride, pad, dil;
    const float *pre_scale, *pre_shift; int pre_relu;
    const float *dy; long long dys;
    int Cout, Hout, Wout;
    int n_tile;
    int kwin;                // grouped (block-diagonal) layer: only the n-tiles inside the diagonal block ci_tile exist
    float *part;             // [splitK][taps][Cin][Cout]   (grouped: [splitK][taps][Cin][kwin])
    int splitK, kb_per_split, KBp;
    int M;
    int x_vec, dy_vec;
    int stages, stage_bytes;     // operand ring: [x X_BYTES | dY hi b_bytes | dY lo b_bytes] per stage (single pass: no lo)
    int b_bytes;
    FastDiv fd_wout, fd_hout;
};


// SINGLE: single-pass TF32 (wgrad_tf32_kernel) instead of 3xTF32 (wgrad_tc_kernel)
template <int PRE, bool UP, bool VEC, bool SINGLE>
__device__ __forceinline__ void wgrad_body(const WgradParams &p) {
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;
    uint8_t *sm = smem_raw + (base - smem_u32(smem_raw));
    const int S = p.stages;
    const uint32_t stage_bytes = (uint32_t)p.stage_bytes;
    const uint32_t pre_off = (uint32_t)S * stage_bytes;
    const uint32_t bar_off = pre_off + 2 * BLOCK_CI * 4;
    float *s_scale = reinterpret_cast<float *>(sm + pre_off);
    float *s_shift = s_scale + BLOCK_CI;
    const uint32_t bar0 = base + bar_off;
    auto full = [&](int s) { return bar0 + 8u * s; };
    auto empty = [&](int s) { return bar0 + 8u * (MAX_STAGES + s); };

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int nt = blockIdx.y;
    const int n_tile = p.n_tile;
    const int ci_tile = p.kwin ? nt * n_tile / BLOCK_CI : blockIdx.x;
    const int tap = blockIdx.z / p.splitK, split = blockIdx.z % p.splitK;
    const int kb0 = split * p.kb_per_split;
    int kb1 = kb0 + p.kb_per_split;
    if (kb1 > p.KBp) kb1 = p.KBp;
    const int nkb = kb1 > kb0 ? kb1 - kb0 : 0;

    if (threadIdx.x == 0) {
        for (int s = 0; s < S; ++s) {
            mbar_init(full(s), 2 * GROUP_THREADS);      // both producer groups (x tile + dY tile) arrive
            mbar_init(empty(s), CONSUMER_THREADS);
        }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    if (p.pre_scale) {
        for (int c = threadIdx.x; c < BLOCK_CI; c += NUM_THREADS) {
            const int ch = ci_tile * BLOCK_CI + c;
            s_scale[c] = ch < p.Cin ? p.pre_scale[ch] : 0.f;
            s_shift[c] = ch < p.Cin ? p.pre_shift[ch] : 0.f;
        }
    }
    // (no zero fill of the stages: the producers write every byte of a stage that is read, dead channels as zeros)
    __syncthreads();

    if (warp < CONSUMER_THREADS / 32) {
        // ---- consumers: two warpgroups, input channels [64 wg, 64 wg + 64) of the tile.  Per k-block every thread loads
        //      its A fragments from the fp32 x tile, splits them into hi/lo in registers (split_tf32) and issues per k8 step
        //      A_lo*B_hi, A_hi*B_lo, A_hi*B_hi (small cross terms first), B hi/lo from shared memory; a stage is released as
        //      soon as its wgmma group has completed (the other warpgroup keeps the tensor cores busy meanwhile)
        const int wg = warp >> 2;
        const uint32_t b_off = X_BYTES;
        const uint32_t bl_off = b_off + (uint32_t)p.b_bytes;
        // A fragment of k8 step k (wgmma_tf32.cuh): rows = channels c, c + 8 with c = 64 wg + 16 (warp % 4) + lane / 4,
        // columns = pixels 8k + q, 8k + q + 4 with q = lane % 4.  Pixel r of the x tile is the 512-byte row r, its 16-byte
        // chunk u (channels 4u..4u+3) stored at chunk u ^ 2 (r % 4): the 8 channels x 4 pixels of one fragment load hit 32
        // distinct banks.  r % 4 == q for every fragment of the thread, and chunk(c + 8) = chunk(c) ^ 2 (c % 16 < 8), so
        // channel c + 8 sits at byte offset aF ^ 32.
        const int q = lane & 3;
        const int c = wg * 64 + (warp & 3) * 16 + (lane >> 2);
        const uint32_t aF = (uint32_t)q * X_ROW_BYTES + ((uint32_t)((c >> 2) ^ (2 * q)) << 4) + (uint32_t)(c & 3) * 4u;
        auto consume = [&](auto NT) {
            constexpr int N = decltype(NT)::value;
            float acc[N / 2];
#pragma unroll
            for (int i = 0; i < N / 2; ++i) acc[i] = 0.f;
            int s = 0;
            uint32_t ph = 0;
            for (int it = 0; it < nkb; ++it) {
                mbar_wait(full(s), ph);
                const uint32_t st = base + (uint32_t)s * stage_bytes;
                if constexpr (SINGLE) {
                    uint32_t hi[BLOCK_KP / 8][4];
#pragma unroll
                    for (int k = 0; k < BLOCK_KP / 8; ++k) {
#pragma unroll
                        for (int j = 0; j < 4; ++j) {                  // j: row + 8 (j & 1), column + 4 (j >> 1)
                            const uint32_t x = ld_shared_u32(st + (aF ^ (32u * (j & 1))) + (uint32_t)(8 * k + 4 * (j >> 1)) * X_ROW_BYTES);
                            hi[k][j] = __float_as_uint(round_tf32(__uint_as_float(x)));
                        }
                    }
                    wgmma_fence();
#pragma unroll
                    for (int k = 0; k < BLOCK_KP / 8; ++k) {
                        const uint64_t dbh = make_desc_core(st + b_off + (uint32_t)k * 256u, 128, CORE_SBO);
                        Wgmma<N>::mma_rs(acc, hi[k], dbh, (it | k) != 0);
                    }
                    wgmma_commit();
                    wgmma_wait<0>();
                    wgmma_fence_operands(acc);
#pragma unroll
                    for (int k = 0; k < BLOCK_KP / 8; ++k) wgmma_fence_operands(hi[k]);
                } else {
                    uint32_t hi[BLOCK_KP / 8][4], lo[BLOCK_KP / 8][4];
#pragma unroll
                    for (int k = 0; k < BLOCK_KP / 8; ++k) {
#pragma unroll
                        for (int j = 0; j < 4; ++j) {                  // j: row + 8 (j & 1), column + 4 (j >> 1)
                            const uint32_t x = ld_shared_u32(st + (aF ^ (32u * (j & 1))) + (uint32_t)(8 * k + 4 * (j >> 1)) * X_ROW_BYTES);
                            float h, l;
                            split_tf32(__uint_as_float(x), h, l);
                            hi[k][j] = __float_as_uint(h);
                            lo[k][j] = __float_as_uint(l);
                        }
                    }
                    wgmma_fence();
#pragma unroll
                    for (int k = 0; k < BLOCK_KP / 8; ++k) {
                        const uint32_t ko = (uint32_t)k * 256u;
                        const uint64_t dbh = make_desc_core(st + b_off + ko, 128, CORE_SBO), dbl = make_desc_core(st + bl_off + ko, 128, CORE_SBO);
                        const uint32_t accumulate = (it | k) != 0;
                        Wgmma<N>::mma_rs(acc, lo[k], dbh, accumulate);
                        Wgmma<N>::mma_rs(acc, hi[k], dbl, 1);
                        Wgmma<N>::mma_rs(acc, hi[k], dbh, 1);
                    }
                    wgmma_commit();
                    wgmma_wait<0>();
                    wgmma_fence_operands(acc);
#pragma unroll
                    for (int k = 0; k < BLOCK_KP / 8; ++k) {
                        wgmma_fence_operands(hi[k]);
                        wgmma_fence_operands(lo[k]);
                    }
                }
                mbar_arrive(empty(s));
                if (++s == S) { s = 0; ph ^= 1; }
            }
            // ---- epilogue: accumulator row = input channel, column = output channel; partial [split][tap][ci][co]
            const int taps = p.KH * p.KW;
            const bool ovec = (p.Cout & 1) == 0 && ((((uintptr_t)p.part) & 7) == 0) && (n_tile & 1) == 0;
#pragma unroll
            for (int i = 0; i < 2; ++i) {
                const int ci = ci_tile * BLOCK_CI + wg * 64 + (warp & 3) * 16 + (lane >> 2) + 8 * i;
                if (ci >= p.Cin) continue;
                float *prow = p.kwin ? p.part + (((long long)split * taps + tap) * p.Cin + ci) * p.kwin + (nt * n_tile) % p.kwin
                                     : p.part + (((long long)split * taps + tap) * p.Cin + ci) * p.Cout + (long long)nt * n_tile;
                const int ccap = p.kwin ? n_tile : p.Cout - nt * n_tile;     // live columns of this tile
#pragma unroll
                for (int j = 0; j < N / 8; ++j) {
                    const int col = 8 * j + (lane & 3) * 2;
                    const float v0 = acc[4 * j + 2 * i], v1 = acc[4 * j + 2 * i + 1];
                    if (ovec && col + 1 < ccap) {
                        *reinterpret_cast<float2 *>(prow + col) = make_float2(v0, v1);
                    } else {
                        if (col < ccap) prow[col] = v0;
                        if (col + 1 < ccap) prow[col + 1] = v1;
                    }
                }
            }
        };
        switch (n_tile) {
            case 16: consume(std::integral_constant<int, 16>()); break;
            case 32: consume(std::integral_constant<int, 32>()); break;
            case 48: consume(std::integral_constant<int, 48>()); break;
            default: consume(std::integral_constant<int, 64>()); break;
        }
    } else {
        // ---- producers: group 0 (warps 8..11) stages the x tiles, group 1 (warps 12..15) the dY tiles; each keeps the
        //      global loads of its next k-block in flight while it stores the current one (register ping-pong)
        const int pt = threadIdx.x - CONSUMER_THREADS;
        const int grp = pt / GROUP_THREADS;
        const int t = pt % GROUP_THREADS;
        constexpr bool AFF = PRE >= 2;
        constexpr bool RELU = (PRE & 1) != 0;

        if (grp == 0) {
            // ------------------------------ x tiles (A operand), fp32 [pixel][channel] --------------------------------
            // Thread t owns the 4-channel unit u = t % 32 of pixel rows r0 + 4 i (i = 0..7, r0 = t / 32): a warp reads one
            // pixel's 512 contiguous bytes per row and writes them with one 128-bit shared store per lane (the chunk
            // swizzle u ^ 2 r0 permutes chunks within aligned groups of 8: conflict-free).
            constexpr int NR = BLOCK_KP / 4;           // rows per thread per k-block
            const int u = t & 31, r0 = t >> 5;
            const uint32_t xoff = (uint32_t)r0 * X_ROW_BYTES + ((uint32_t)(u ^ (2 * r0)) << 4);   // + 4 i rows
            const int Hin = UP ? 2 * p.Hs : p.Hs, Win = UP ? 2 * p.Ws : p.Ws;
            const int dyo = (tap / p.KW) * p.dil - p.pad, dxo = (tap % p.KW) * p.dil - p.pad;
            const int xs = (int)p.xs;
            const int c = ci_tile * BLOCK_CI + u * 4;  // first input channel of the unit
            float sc[4], sh[4];
            if (AFF) {
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    sc[e] = s_scale[u * 4 + e];        // 0 beyond Cin
                    sh[e] = s_shift[u * 4 + e];
                }
            }
            const float *__restrict__ xg = p.x;
            auto load_x = [&](int it, F4(&v)[NR], uint32_t &mask) {
                const int m0 = (kb0 + it) * BLOCK_KP + r0;
                uint32_t mk = 0;
#pragma unroll
                for (int i = 0; i < NR; ++i) {
                    const int m = m0 + 4 * i;
                    const uint32_t qo = fdiv((uint32_t)m, p.fd_wout);
                    const uint32_t b = fdiv(qo, p.fd_hout);
                    const int ox = m - (int)qo * p.Wout, oy = (int)qo - (int)b * p.Hout;
                    const int yy = oy * p.stride + dyo, xx = ox * p.stride + dxo;
                    const bool ok = m < p.M && (unsigned)yy < (unsigned)Hin && (unsigned)xx < (unsigned)Win;
                    mk |= (ok ? 1u : 0u) << i;
                    const int sy = UP ? (yy >> 1) : yy, sx = UP ? (xx >> 1) : xx;
                    const int off = (((int)b * p.Hs + sy) * p.Ws + sx) * xs + c;
                    const bool live = ok && c < p.Cin;
                    if (VEC) {
                        float4 q4 = make_float4(0.f, 0.f, 0.f, 0.f);
                        if (live) q4 = __ldg(reinterpret_cast<const float4 *>(xg + off));
                        if (c + 3 >= p.Cin) {          // channel tail of a 16-byte-padded row
                            if (c + 1 >= p.Cin) q4.y = 0.f;
                            if (c + 2 >= p.Cin) q4.z = 0.f;
                            q4.w = 0.f;
                        }
                        v[i].v[0] = q4.x; v[i].v[1] = q4.y; v[i].v[2] = q4.z; v[i].v[3] = q4.w;
                    } else {
#pragma unroll
                        for (int e = 0; e < 4; ++e) {
                            float q1 = 0.f;
                            if (live && c + e < p.Cin) q1 = __ldg(xg + off + e);
                            v[i].v[e] = q1;
                        }
                    }
                }
                mask = mk;
            };
            int xs_s = 0;
            uint32_t xs_ph = 0;
            auto store_x = [&](F4(&v)[NR], uint32_t mask) {
                if (PRE != 0) {
#pragma unroll
                    for (int i = 0; i < NR; ++i)
#pragma unroll
                        for (int e = 0; e < 4; ++e) {
                            float a = v[i].v[e];
                            if (AFF) {
                                a = fmaf(a, sc[e], sh[e]);
                                if (RELU) a = fmaxf(a, 0.f);
                                a = ((mask >> i) & 1u) ? a : 0.f;     // zero padding is applied after the pre-op
                            } else {
                                a = fmaxf(a, 0.f);
                            }
                            v[i].v[e] = a;
                        }
                }
                mbar_wait(empty(xs_s), xs_ph ^ 1);
                const uint32_t dst = base + (uint32_t)xs_s * stage_bytes + xoff;
#pragma unroll
                for (int i = 0; i < NR; ++i)
                    st_shared_v4(dst + (uint32_t)(4 * i) * X_ROW_BYTES, v[i].v[0], v[i].v[1], v[i].v[2], v[i].v[3]);
                mbar_arrive(full(xs_s));               // the consumers read x with generic loads: no proxy fence
                if (++xs_s == S) { xs_s = 0; xs_ph ^= 1; }
            };
            F4 va[NR], vb[NR];
            uint32_t ma = 0, mb = 0;
            int it = 0;
            if (it < nkb) load_x(it, va, ma);
            for (; it < nkb; it += 2) {
                const bool more = it + 1 < nkb;
                if (more) load_x(it + 1, vb, mb);
                store_x(va, ma);
                if (more) {
                    if (it + 2 < nkb) load_x(it + 2, va, ma);
                    store_x(vb, mb);
                }
            }
        } else {
            // ------------------------------ dY tiles (B operand): ceil(n_tile/32) <= 2 chunks of output channels ---
            // Thread t owns the 4-channel unit `unit` = t % 8 of each chunk in pixel rows r0 and r0 + 16 (r0 = t / 8).
            // K-major core-matrix tiles: element (row = channel, k = pixel) at (row / 8) * CORE_SBO + (k / 4) * 128 +
            // (row % 8) * 16 + (k % 4) * 4.  A unit is 4 scalar stores, which the 16-byte pad of CORE_SBO spreads over all
            // 32 banks across the warp.
            const int unit = t & 7, r0 = t >> 3;
            const uint32_t roff = (uint32_t)(unit >> 1) * CORE_SBO + (uint32_t)(r0 >> 2) * 128u + (uint32_t)(unit & 1) * 64u +
                                  (uint32_t)(r0 & 3) * 4u;   // + chunk * 4 CORE_SBO + h * 512 for row r0 + 16 h
            const int dys = (int)p.dys;
            const int nchunk = (n_tile + 31) >> 5;
            const int cb = nt * n_tile + unit * 4;
            const float *__restrict__ dg = p.dy;
            constexpr int NU = 4;                      // v[2 h + chunk]
            auto load_d = [&](int it, F4(&v)[NU]) {
                const int kb = kb0 + it;
#pragma unroll
                for (int i = 0; i < NU; ++i) {
                    const int h = i >> 1, chunk = i & 1;
                    const int m = kb * BLOCK_KP + r0 + 16 * h;
                    const int c = cb + chunk * 32;
                    const bool live = chunk < nchunk && m < p.M && c < p.Cout;
                    if (VEC) {
                        float4 q4 = make_float4(0.f, 0.f, 0.f, 0.f);
                        if (live) q4 = __ldg(reinterpret_cast<const float4 *>(dg + m * dys + c));
                        if (c + 3 >= p.Cout) {
                            if (c + 1 >= p.Cout) q4.y = 0.f;
                            if (c + 2 >= p.Cout) q4.z = 0.f;
                            q4.w = 0.f;
                        }
                        v[i].v[0] = q4.x; v[i].v[1] = q4.y; v[i].v[2] = q4.z; v[i].v[3] = q4.w;
                    } else {
#pragma unroll
                        for (int e = 0; e < 4; ++e) {
                            float q1 = 0.f;
                            if (live && c + e < p.Cout) q1 = __ldg(dg + m * dys + c + e);
                            v[i].v[e] = q1;
                        }
                    }
                }
            };
            int ds_s = 0;
            uint32_t ds_ph = 0;
            auto store_d = [&](F4(&v)[NU]) {
                mbar_wait(empty(ds_s), ds_ph ^ 1);
                const uint32_t t_hi = base + (uint32_t)ds_s * stage_bytes + X_BYTES + roff;
                const uint32_t t_lo = t_hi + (uint32_t)p.b_bytes;
#pragma unroll
                for (int i = 0; i < NU; ++i) {
                    const int h = i >> 1, chunk = i & 1;
                    if (chunk < nchunk) {
                        const uint32_t o = (uint32_t)chunk * 4u * CORE_SBO + (uint32_t)h * 512u;
                        if constexpr (SINGLE) {
#pragma unroll
                            for (int e = 0; e < 4; ++e) st_shared_f32(t_hi + o + 16u * e, round_tf32(v[i].v[e]));
                        } else {
                            float hi[4], lo[4];
#pragma unroll
                            for (int e = 0; e < 4; ++e) split_tf32(v[i].v[e], hi[e], lo[e]);
#pragma unroll
                            for (int e = 0; e < 4; ++e) {
                                st_shared_f32(t_hi + o + 16u * e, hi[e]);
                                st_shared_f32(t_lo + o + 16u * e, lo[e]);
                            }
                        }
                    }
                }
                fence_proxy_async();                   // generic-proxy writes -> visible to wgmma (async proxy)
                mbar_arrive(full(ds_s));
                if (++ds_s == S) { ds_s = 0; ds_ph ^= 1; }
            };
            F4 va[NU], vb[NU];
            int it = 0;
            if (it < nkb) load_d(it, va);
            for (; it < nkb; it += 2) {
                const bool more = it + 1 < nkb;
                if (more) load_d(it + 1, vb);
                store_d(va);
                if (more) {
                    if (it + 2 < nkb) load_d(it + 2, va);
                    store_d(vb);
                }
            }
        }
    }
}

template <int PRE, bool UP, bool VEC>
__global__ void __launch_bounds__(NUM_THREADS, 1) wgrad_tc_kernel(const WgradParams p) {
    wgrad_body<PRE, UP, VEC, false>(p);
}

template <int PRE, bool UP, bool VEC>
__global__ void __launch_bounds__(NUM_THREADS, 1) wgrad_tf32_kernel(const WgradParams p) {
    wgrad_body<PRE, UP, VEC, true>(p);
}

// dW[co,ci,kh,kw] (arbitrary strides) = sum_split part[split][tap][ci][co]; fixed summation order -> deterministic
__global__ void __launch_bounds__(256) wgrad_reduce_kernel(const float *__restrict__ part, int splitK, int taps, int Cin,
                                                           int Cout, int KW, float *__restrict__ dw, long long s_co,
                                                           long long s_ci, long long s_kh, long long s_kw) {
    const long long per = (long long)taps * Cin * Cout;
    for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < per;
         idx += (long long)gridDim.x * blockDim.x) {
        float acc = 0.f;
        for (int s = 0; s < splitK; ++s) acc += part[(long long)s * per + idx];
        const int co = (int)(idx % Cout);
        const long long t = idx / Cout;
        const int ci = (int)(t % Cin);
        const int tap = (int)(t / Cin);
        dw[co * s_co + ci * s_ci + (tap / KW) * s_kh + (tap % KW) * s_kw] = acc;
    }
}

// grouped layers: dW[co, ci_local, kh, kw] = sum_split part[split][tap][ci = (co / cpg) * cpg + ci_local][co % kwin]
__global__ void __launch_bounds__(256) wgrad_reduce_grouped_kernel(const float *__restrict__ part, int splitK, int taps,
                                                                   int width, int kwin, int cpg, int KW,
                                                                   float *__restrict__ dw, long long s_co, long long s_ci,
                                                                   long long s_kh, long long s_kw) {
    const long long per = (long long)taps * width * kwin;          // one split of the partial buffer
    const long long total = (long long)taps * width * cpg;
    for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
         idx += (long long)gridDim.x * blockDim.x) {
        const int cl = (int)(idx % cpg);
        const long long t = idx / cpg;
        const int co = (int)(t % width);
        const int tap = (int)(t / width);
        const int ci = (co / cpg) * cpg + cl;
        const long long src = ((long long)tap * width + ci) * kwin + (co % kwin);
        float acc = 0.f;
        for (int s = 0; s < splitK; ++s) acc += part[(long long)s * per + src];
        dw[co * s_co + cl * s_ci + (tap / KW) * s_kh + (tap % KW) * s_kw] = acc;
    }
}

}  // namespace

// N tile of the wgrad kernels: <= MAX_N output channels per CTA (the consumers' register accumulator)
static int wgrad_n_tile(int Cout) {
    const int cap = MAX_N;
    int n = (Cout + 15) / 16 * 16;
    if (n > cap) {
        const int tiles = (n + cap - 1) / cap;
        n = ((Cout + tiles - 1) / tiles + 15) / 16 * 16;
    }
    return n;
}


// narrow-output 3x3 layers use the shifted-dY kernel (wgrad2_tc.cu)
bool bts_wgrad2_eligible(int Cout, int KH, int KW, int stride, long long Mq);
void bts_wgrad2_plan(int B, int Hin, int Win, int Cin, int Cout, int KH, int KW, int *splitK);
int bts_wgrad2_launch(const float *x, long long xs, int B, int Hs, int Ws, int up, int Cin, int KH, int KW, int pad,
                      int dil, const float *pre_scale, const float *pre_shift, int pre_relu, const float *dy,
                      long long dys, int Cout, int Hout, int Wout, float *workspace, int splitK, int precision,
                      cudaStream_t st);

extern "C" int bts_conv_wgrad_plan(int B, int Hout, int Wout, int Cin, int Cout, int KH, int KW, int stride,
                                   int *splitK_out, long long *workspace_floats) {
    if (!splitK_out || !workspace_floats || B < 1 || Hout < 1 || Wout < 1 || Cin < 1 || Cout < 1 || stride < 1) return BTS_EINVAL;
    if (bts_wgrad2_eligible(Cout, KH, KW, stride, (long long)B * Hout * Wout)) {
        int sp = 1;
        bts_wgrad2_plan(B, Hout, Wout, Cin, Cout, KH, KW, &sp);
        *splitK_out = sp;
        *workspace_floats = (long long)sp * KH * KW * (long long)Cin * Cout;
        return 0;
    }
    const long long M = (long long)B * Hout * Wout;
    const long long KBp = (M + BLOCK_KP - 1) / BLOCK_KP;
    const int n_tile = wgrad_n_tile(Cout);
    const long long tiles = (long long)((Cin + BLOCK_CI - 1) / BLOCK_CI) * ((Cout + n_tile - 1) / n_tile) * KH * KW;
    const int sms = bts_num_sms();
    // split-K so that the CTA count fills whole waves of the SMs (a grid of 1.5 waves wastes a third of the
    // time in a 1-CTA tail): among splits giving <= 4 waves pick the best wave efficiency, ties -> more CTAs
    long long max_split = (KBp + 15) / 16;                    // at least 16 k-blocks (512 px) per CTA
    if (max_split < 1) max_split = 1;
    if (max_split > 64) max_split = 64;
    long long split = 1;
    double best = -1.0;
    for (long long sp = 1; sp <= max_split; ++sp) {
        const long long ctas = tiles * sp;
        const long long waves = (ctas + sms - 1) / sms;
        if (waves > 4 && sp > 1) break;
        const double eff = (double)ctas / (double)(waves * sms);
        if (eff >= best - 1e-9) { best = eff; split = sp; }
    }
    *splitK_out = (int)split;
    *workspace_floats = split * KH * KW * (long long)Cin * Cout;
    return 0;
}

extern "C" int bts_conv_wgrad(const float *x, long long x_pixel_stride, int B, int Hs, int Ws, int upsample2, int Cin,
                              int KH, int KW, int stride, int pad, int dil, const float *pre_scale,
                              const float *pre_shift, int pre_relu, const float *dy, long long dy_pixel_stride, int Cout,
                              float *workspace, int splitK, float *dw, long long s_co, long long s_ci, long long s_kh,
                              long long s_kw, int precision, void *stream) {
    if (!x || !dy || !workspace || !dw || B < 1 || Hs < 1 || Ws < 1 || Cin < 1 || Cout < 1 || KH < 1 || KW < 1 ||
        stride < 1 || pad < 0 || dil < 1 || splitK < 1)
        return BTS_EINVAL;
    if ((pre_scale == nullptr) != (pre_shift == nullptr)) return BTS_EINVAL;
    WgradParams p;
    p.x = x; p.xs = x_pixel_stride; p.B = B; p.Hs = Hs; p.Ws = Ws; p.up = upsample2 ? 1 : 0; p.Cin = Cin;
    p.KH = KH; p.KW = KW; p.stride = stride; p.pad = pad; p.dil = dil;
    p.pre_scale = pre_scale; p.pre_shift = pre_shift; p.pre_relu = pre_relu ? 1 : 0;
    p.dy = dy; p.dys = dy_pixel_stride; p.Cout = Cout;
    const int Hin = p.up ? 2 * Hs : Hs, Win = p.up ? 2 * Ws : Ws;
    p.Hout = (Hin + 2 * pad - dil * (KH - 1) - 1) / stride + 1;
    p.Wout = (Win + 2 * pad - dil * (KW - 1) - 1) / stride + 1;
    const long long M = (long long)B * p.Hout * p.Wout;
    if (p.Hout < 1 || p.Wout < 1 || M > 0x7ffffff0LL) return BTS_EINVAL;
    if ((long long)B * Hs * Ws * x_pixel_stride >= 0x7fffffffLL || M * dy_pixel_stride >= 0x7fffffffLL) return BTS_EINVAL;
    p.M = (int)M;
    p.n_tile = wgrad_n_tile(Cout);
    p.kwin = 0;
    p.part = workspace; p.splitK = splitK;
    p.KBp = (int)((M + BLOCK_KP - 1) / BLOCK_KP);
    p.kb_per_split = (p.KBp + splitK - 1) / splitK;
    p.x_vec = bts_aligned16(x) && (x_pixel_stride % 4 == 0);
    p.dy_vec = bts_aligned16(dy) && (dy_pixel_stride % 4 == 0);
    p.fd_wout = make_fastdiv((uint32_t)p.Wout);
    p.fd_hout = make_fastdiv((uint32_t)p.Hout);
    const int taps = KH * KW;
    if (bts_wgrad2_eligible(Cout, KH, KW, stride, M)) {
        int rc2 = bts_wgrad2_launch(x, x_pixel_stride, B, Hs, Ws, p.up, Cin, KH, KW, pad, dil, pre_scale, pre_shift,
                                    p.pre_relu, dy, dy_pixel_stride, Cout, p.Hout, p.Wout, workspace, splitK, precision,
                                    (cudaStream_t)stream);
        if (rc2) return rc2;
        const long long per2 = (long long)taps * Cin * Cout;
        long long g2 = (per2 + 255) / 256;
        const long long cap2 = (long long)bts_num_sms() * 16;
        if (g2 > cap2) g2 = cap2;
        wgrad_reduce_kernel<<<(int)g2, 256, 0, (cudaStream_t)stream>>>(workspace, splitK, taps, Cin, Cout, KW, dw, s_co, s_ci,
                                                                      s_kh, s_kw);
        BTS_LAUNCH_CHECK();
        return 0;
    }
    {
        const int nchunk = (p.n_tile + 31) / 32;
        p.b_bytes = nchunk * 4 * (int)CORE_SBO;
        p.stage_bytes = X_BYTES + (precision ? 1 : 2) * p.b_bytes;
        p.stages = (SMEM_LIMIT - 1024 - 2 * BLOCK_CI * 4 - 256) / p.stage_bytes;
        if (p.stages > MAX_STAGES) p.stages = MAX_STAGES;
        if (p.stages < 2) return BTS_EINVAL;
    }
    const int smem = p.stages * p.stage_bytes + 2 * BLOCK_CI * 4 + 256 + 1024;
    dim3 grid((Cin + BLOCK_CI - 1) / BLOCK_CI, (Cout + p.n_tile - 1) / p.n_tile, taps * splitK);
    if (grid.z > 65535) return BTS_EINVAL;
    cudaStream_t st = (cudaStream_t)stream;
    const int pre = (pre_scale ? 2 : 0) | (p.pre_relu ? 1 : 0);
    const bool vec = p.x_vec && p.dy_vec;   // aligned bases + pixel strides % 4 == 0 (channel tails masked in-kernel)
    cudaError_t err = cudaSuccess;
#define BTS_LAUNCH(KERNEL, PRE, UP, VEC)                                                                            \
    do {                                                                                                            \
        static bool attr_set_[BTS_MAX_DEVICES] = {}; bool &attr_set = attr_set_[bts_cur_device()];                  \
        if (!attr_set) {                                                                                            \
            err = cudaFuncSetAttribute(KERNEL<PRE, UP, VEC>, cudaFuncAttributeMaxDynamicSharedMemorySize,           \
                                       SMEM_LIMIT);                                                                 \
            if (err != cudaSuccess) return (int)err;                                                                \
            attr_set = true;                                                                                        \
        }                                                                                                           \
        KERNEL<PRE, UP, VEC><<<grid, NUM_THREADS, smem, st>>>(p);                                                   \
    } while (0)
#define BTS_DISPATCH_UV(KERNEL, PRE)                                                                                \
    do {                                                                                                            \
        if (p.up) { if (vec) BTS_LAUNCH(KERNEL, PRE, true, true); else BTS_LAUNCH(KERNEL, PRE, true, false); }      \
        else { if (vec) BTS_LAUNCH(KERNEL, PRE, false, true); else BTS_LAUNCH(KERNEL, PRE, false, false); }         \
    } while (0)
#define BTS_DISPATCH(KERNEL)                                                                                        \
    do {                                                                                                            \
        switch (pre) {                                                                                              \
            case 0: BTS_DISPATCH_UV(KERNEL, 0); break;                                                              \
            case 1: BTS_DISPATCH_UV(KERNEL, 1); break;                                                              \
            case 2: BTS_DISPATCH_UV(KERNEL, 2); break;                                                              \
            default: BTS_DISPATCH_UV(KERNEL, 3); break;                                                             \
        }                                                                                                           \
    } while (0)
    if (precision) BTS_DISPATCH(wgrad_tf32_kernel);
    else BTS_DISPATCH(wgrad_tc_kernel);
#undef BTS_DISPATCH
#undef BTS_DISPATCH_UV
#undef BTS_LAUNCH
    BTS_LAUNCH_CHECK();
    const long long per = (long long)taps * Cin * Cout;
    long long g = (per + 255) / 256;
    const long long cap = (long long)bts_num_sms() * 16;
    if (g > cap) g = cap;
    wgrad_reduce_kernel<<<(int)g, 256, 0, st>>>(workspace, splitK, taps, Cin, Cout, KW, dw, s_co, s_ci, s_kh, s_kw);
    BTS_LAUNCH_CHECK();
    return 0;
}

// ------------------------------------------------------------------------------------------- grouped (block-diagonal) wgrad
// ResNeXt 3x3 convs (pytorch/bts.py:291-296 via torchvision, 32 groups): x and dy carry `width` channels each, w is
// (width, cpg, KH, KW).  Only the diagonal 128 x 128 channel blocks are computed (one CTA per block, tap and split),
// the reduce kernel extracts every group's cpg x cpg sub-block.  Requires bts_conv_group_window(width, cpg) == 128.
extern "C" int bts_conv_group_window(int width, int cpg);

static long long wgrad_grouped_split(long long M, int width, int taps) {
    const long long KBp = (M + BLOCK_KP - 1) / BLOCK_KP;
    const long long tiles = (long long)(width / MAX_N) * taps;       // CTAs per split: the grid of bts_conv_wgrad_grouped
    const int sms = bts_num_sms();
    long long max_split = (KBp + 15) / 16;
    if (max_split < 1) max_split = 1;
    if (max_split > 64) max_split = 64;
    long long split = 1;
    double best = -1.0;
    for (long long sp = 1; sp <= max_split; ++sp) {
        const long long ctas = tiles * sp;
        const long long waves = (ctas + sms - 1) / sms;
        if (waves > 4 && sp > 1) break;
        const double eff = (double)ctas / (double)(waves * sms);
        if (eff >= best - 1e-9) { best = eff; split = sp; }
    }
    return split;
}

extern "C" int bts_conv_wgrad_grouped_plan(int B, int Hout, int Wout, int width, int cpg, int KH, int KW, int *splitK_out,
                                           long long *workspace_floats) {
    if (!splitK_out || !workspace_floats || B < 1 || Hout < 1 || Wout < 1 || KH < 1 || KW < 1) return BTS_EINVAL;
    if (bts_conv_group_window(width, cpg) != 128) return BTS_EINVAL;
    const long long split = wgrad_grouped_split((long long)B * Hout * Wout, width, KH * KW);
    *splitK_out = (int)split;
    *workspace_floats = split * KH * KW * (long long)width * 128;
    return 0;
}

extern "C" int bts_conv_wgrad_grouped(const float *x, long long x_pixel_stride, int B, int Hs, int Ws, int width, int cpg,
                                      int KH, int KW, int stride, int pad, int dil, const float *dy,
                                      long long dy_pixel_stride, float *workspace, int splitK, float *dw, long long s_co,
                                      long long s_ci, long long s_kh, long long s_kw, int precision, void *stream) {
    if (!x || !dy || !workspace || !dw || B < 1 || Hs < 1 || Ws < 1 || KH < 1 || KW < 1 || stride < 1 || pad < 0 || dil < 1 ||
        splitK < 1)
        return BTS_EINVAL;
    if (bts_conv_group_window(width, cpg) != 128) return BTS_EINVAL;
    WgradParams p;
    p.x = x; p.xs = x_pixel_stride; p.B = B; p.Hs = Hs; p.Ws = Ws; p.up = 0; p.Cin = width;
    p.KH = KH; p.KW = KW; p.stride = stride; p.pad = pad; p.dil = dil;
    p.pre_scale = nullptr; p.pre_shift = nullptr; p.pre_relu = 0;
    p.dy = dy; p.dys = dy_pixel_stride; p.Cout = width;
    p.Hout = (Hs + 2 * pad - dil * (KH - 1) - 1) / stride + 1;
    p.Wout = (Ws + 2 * pad - dil * (KW - 1) - 1) / stride + 1;
    const long long M = (long long)B * p.Hout * p.Wout;
    if (p.Hout < 1 || p.Wout < 1 || M > 0x7ffffff0LL) return BTS_EINVAL;
    if ((long long)B * Hs * Ws * x_pixel_stride >= 0x7fffffffLL || M * dy_pixel_stride >= 0x7fffffffLL) return BTS_EINVAL;
    p.M = (int)M;
    p.n_tile = MAX_N; p.kwin = 128;
    p.part = workspace; p.splitK = splitK;
    p.KBp = (int)((M + BLOCK_KP - 1) / BLOCK_KP);
    p.kb_per_split = (p.KBp + splitK - 1) / splitK;
    p.x_vec = bts_aligned16(x) && (x_pixel_stride % 4 == 0);
    p.dy_vec = bts_aligned16(dy) && (dy_pixel_stride % 4 == 0);
    p.fd_wout = make_fastdiv((uint32_t)p.Wout);
    p.fd_hout = make_fastdiv((uint32_t)p.Hout);
    const int taps = KH * KW;
    p.b_bytes = 2 * 4 * (int)CORE_SBO;
    p.stage_bytes = X_BYTES + (precision ? 1 : 2) * p.b_bytes;
    p.stages = (SMEM_LIMIT - 1024 - 2 * BLOCK_CI * 4 - 256) / p.stage_bytes;
    if (p.stages > MAX_STAGES) p.stages = MAX_STAGES;
    const int smem = p.stages * p.stage_bytes + 2 * BLOCK_CI * 4 + 256 + 1024;
    dim3 grid(1, width / MAX_N, taps * splitK);
    if (grid.z > 65535) return BTS_EINVAL;
    cudaStream_t st = (cudaStream_t)stream;
    cudaError_t err = cudaSuccess;
    const bool vec = p.x_vec && p.dy_vec;
#define BTS_LAUNCH_G(KERNEL, VEC)                                                                                    \
    do {                                                                                                             \
        static bool attr_set_[BTS_MAX_DEVICES] = {};                                                                 \
        bool &attr_set = attr_set_[bts_cur_device()];                                                                \
        if (!attr_set) {                                                                                             \
            err = cudaFuncSetAttribute(KERNEL<0, false, VEC>, cudaFuncAttributeMaxDynamicSharedMemorySize,           \
                                       SMEM_LIMIT);                                                                  \
            if (err != cudaSuccess) return (int)err;                                                                 \
            attr_set = true;                                                                                         \
        }                                                                                                            \
        KERNEL<0, false, VEC><<<grid, NUM_THREADS, smem, st>>>(p);                                                   \
    } while (0)
    if (precision) { if (vec) BTS_LAUNCH_G(wgrad_tf32_kernel, true); else BTS_LAUNCH_G(wgrad_tf32_kernel, false); }
    else { if (vec) BTS_LAUNCH_G(wgrad_tc_kernel, true); else BTS_LAUNCH_G(wgrad_tc_kernel, false); }
#undef BTS_LAUNCH_G
    BTS_LAUNCH_CHECK();
    const long long total = (long long)taps * width * cpg;
    long long g = (total + 255) / 256;
    const long long cap = (long long)bts_num_sms() * 16;
    if (g > cap) g = cap;
    wgrad_reduce_grouped_kernel<<<(int)g, 256, 0, st>>>(workspace, splitK, taps, width, 128, cpg, KW, dw, s_co, s_ci, s_kh, s_kw);
    BTS_LAUNCH_CHECK();
    return 0;
}
