// Weight-gradient (wgrad) of the implicit-GEMM convolution on the Hopper tensor cores (wgmma), sm_90a, 3xTF32.
//
//   dW[co, ci, tap] = sum_p  dY[p, co] * pre(x[p (+) tap, ci])            (same pre / (+) as conv_tc.cu)
//
// GEMM view per (tap, split):  M = 128 input channels (two consumer warpgroups of 64), N = n_tile <= 64 output channels,
// K = output pixels.  Both operands live in memory as [pixel][channel] (NHWC), i.e. the reduction index is the slow one,
// while tf32 wgmma reads only K-major operands: the producers transpose on their way into shared memory, writing
// [channel][pixel] tiles of 8 x 16-byte core matrices (no swizzle).
// grid = (ceil(Cin/128), n_tiles(Cout), taps * splitK); each CTA reduces its pixel range into fp32 register accumulators
// and writes a partial; a second, deterministic kernel sums the splitK partials into the (Cout,Cin,KH,KW)-strided gradient.
// 768 threads: 2 consumer warpgroups + 2 producer groups of 8 warps (x tile / dY tile), 2-4 operand stages.
#include <cstdlib>
#include <type_traits>

#include "tc_common.cuh"

using namespace tc;

namespace {

constexpr int BLOCK_CI = 128;
constexpr int BLOCK_KP = 32;                 // pixels per k-block
constexpr int MAX_N = 64;                    // output channels per CTA tile (register accumulator of the consumers)
constexpr int MAX_STAGES = 4;
constexpr int SMEM_LIMIT = 232448;
constexpr uint32_t CORE_SBO = 8 * 128 + 16;  // one 8-channel group of a k-block: 8 core matrices along K + a bank pad
constexpr int A_BYTES = 16 * CORE_SBO;       // 128 channels (hi or lo)
constexpr int CONSUMER_THREADS = 256;
constexpr int GROUP_THREADS = 256;
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
    int x_vec, dy_vec, precision;
    int stages, stage_bytes;     // operand ring: [A hi | A lo | dY hi b_bytes | dY lo b_bytes] per stage
    int b_bytes;
};


template <int PRE, bool UP, bool VEC>
__global__ void __launch_bounds__(NUM_THREADS, 1) wgrad_tc_kernel(const WgradParams p) {
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
    // channel chunks beyond the last live input / output channel are never produced: zero every stage once
    for (int i = threadIdx.x; i < S * stage_bytes / 16; i += NUM_THREADS) st_shared_v4(base + i * 16, 0.f, 0.f, 0.f, 0.f);
    fence_proxy_async();
    __syncthreads();

    if (warp < CONSUMER_THREADS / 32) {
        // ---- consumers: two warpgroups, input channels [64 wg, 64 wg + 64) of the tile; 3xTF32 per k8 step, small
        //      cross terms first; a stage is released as soon as its wgmma group has completed (the other warpgroup keeps
        //      the tensor cores busy meanwhile)
        const int wg = warp >> 2;
        const uint32_t b_off = 2 * A_BYTES;
        const uint32_t bl_off = b_off + (uint32_t)p.b_bytes;
        auto consume = [&](auto NT) {
            constexpr int N = decltype(NT)::value;
            float acc[N / 2];
#pragma unroll
            for (int i = 0; i < N / 2; ++i) acc[i] = 0.f;
            int s = 0;
            uint32_t ph = 0;
            for (int it = 0; it < nkb; ++it) {
                mbar_wait(full(s), ph);
                wgmma_fence();
                const uint32_t st = base + (uint32_t)s * stage_bytes;
                const uint32_t a_hi = st + (uint32_t)wg * 8u * CORE_SBO;
#pragma unroll
                for (int kg = 0; kg < BLOCK_KP / 8; ++kg) {
                    const uint32_t ko = (uint32_t)kg * 256u;
                    const uint64_t dah = make_desc_core(a_hi + ko, 128, CORE_SBO), dal = make_desc_core(a_hi + A_BYTES + ko, 128, CORE_SBO);
                    const uint64_t dbh = make_desc_core(st + b_off + ko, 128, CORE_SBO), dbl = make_desc_core(st + bl_off + ko, 128, CORE_SBO);
                    const uint32_t accumulate = (it | kg) != 0;
                    if (p.precision != 0) {
                        Wgmma<N>::mma(acc, dah, dbh, accumulate);
                    } else {
                        Wgmma<N>::mma(acc, dal, dbh, accumulate);
                        Wgmma<N>::mma(acc, dah, dbl, 1);
                        Wgmma<N>::mma(acc, dah, dbh, 1);
                    }
                }
                wgmma_commit();
                wgmma_wait<0>();
                mbar_arrive(empty(s));
                if (++s == S) { s = 0; ph ^= 1; }
            }
            wgmma_wait<0>();
            wgmma_fence_operands(acc);
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
        // 8 warps per group (round 1 ran 4 with two pixel rows per thread: ~9 cycles between a warp's instructions at
        // 2.5 warps per scheduler made the producers, not the tensor pipe, set the k-block time): one pixel row of the
        // 32-pixel k-block per thread, 4 sixteen-byte units (one per 32-channel chunk).
        const int pt = threadIdx.x - CONSUMER_THREADS;
        const int grp = pt >> 8;                   // group 0 produces the x (A) tiles, group 1 the dY (B) tiles
        const int t = pt & 255;
        const int unit = t & 7;                    // 16-byte unit of the 128-byte row
        const int r0 = t >> 3;                     // pixel row r0 of the 32-pixel k-block
        constexpr bool AFF = PRE >= 2;
        constexpr bool RELU = (PRE & 1) != 0;
        constexpr int NU = 4;                      // units per thread per k-block
        // K-major core-matrix tiles: element (row = channel, k = pixel) at (row / 8) * CORE_SBO + (k / 4) * 128 +
        // (row % 8) * 16 + (k % 4) * 4.  A thread holds 4 consecutive channels of one pixel: 4 scalar stores, which the
        // 16-byte pad of CORE_SBO spreads over all 32 banks across the warp.
        uint32_t roff[NU];
#pragma unroll
        for (int i = 0; i < NU; ++i)
            roff[i] = (uint32_t)(i * 4 + (unit >> 1)) * CORE_SBO + (uint32_t)(r0 >> 2) * 128u + (uint32_t)(unit & 1) * 64u +
                      (uint32_t)(r0 & 3) * 4u;

        // hi/lo split + swizzled stores of up to 8 units (4 chunks x 2 rows); only `nlive` chunks are written
        // (the A regions were zeroed once, so dead channel chunks stay zero)
        auto split_store = [&](uint32_t t_hi, uint32_t t_lo, F4(&v)[NU], int nlive) {
#pragma unroll
            for (int i = 0; i < NU; ++i) {
                if (i < nlive) {
                    float hi[4], lo[4];
#pragma unroll
                    for (int e = 0; e < 4; ++e) {
                        const float a = v[i].v[e];
                        const float hh = __uint_as_float((__float_as_uint(a) + 0x1000u) & 0xffffe000u);
                        hi[e] = hh;
                        lo[e] = a - hh;
                    }
#pragma unroll
                    for (int e = 0; e < 4; ++e) {
                        st_shared_f32(t_hi + roff[i] + 16u * e, hi[e]);
                        st_shared_f32(t_lo + roff[i] + 16u * e, lo[e]);
                    }
                }
            }
        };

        if (grp == 0) {
            // ------------------------------ x tiles (A operand): 4 chunks of 32 input channels ------------------
            const int Hin = UP ? 2 * p.Hs : p.Hs, Win = UP ? 2 * p.Ws : p.Ws;
            const int dyo = (tap / p.KW) * p.dil - p.pad, dxo = (tap % p.KW) * p.dil - p.pad;
            const int xs = (int)p.xs;
            const int cb = ci_tile * BLOCK_CI + unit * 4;
            int nlive = (p.Cin - ci_tile * BLOCK_CI + 31) >> 5;      // chunks that hold real channels
            if (nlive > 4) nlive = 4;
            float sc[4][4], sh[4][4];
            if (AFF) {
#pragma unroll
                for (int ch = 0; ch < 4; ++ch)
#pragma unroll
                    for (int e = 0; e < 4; ++e) {
                        sc[ch][e] = s_scale[ch * 32 + unit * 4 + e];
                        sh[ch][e] = s_shift[ch * 32 + unit * 4 + e];
                    }
            }
            const float *__restrict__ xg = p.x;
            // output-pixel coordinates of this thread's two rows, advanced by 32 pixels per k-block (no divisions)
            int px[1], py[1], pb[1];
#pragma unroll
            for (int h = 0; h < 1; ++h) {
                const int m = kb0 * BLOCK_KP + r0;
                px[h] = m % p.Wout;
                const int q = m / p.Wout;
                py[h] = q % p.Hout;
                pb[h] = q / p.Hout;
            }
            auto load_x = [&](int it, F4(&v)[NU], uint32_t &mask) {
                const int kb = kb0 + it;
                int off[1];
                bool ok[1];
#pragma unroll
                for (int h = 0; h < 1; ++h) {
                    const int m = kb * BLOCK_KP + r0;
                    const int yy = py[h] * p.stride + dyo, xx = px[h] * p.stride + dxo;
                    ok[h] = m < p.M && (unsigned)yy < (unsigned)Hin && (unsigned)xx < (unsigned)Win;
                    const int sy = UP ? (yy >> 1) : yy, sx = UP ? (xx >> 1) : xx;
                    off[h] = ((pb[h] * p.Hs + sy) * p.Ws + sx) * xs + cb;
                    px[h] += BLOCK_KP;
                    while (px[h] >= p.Wout) {
                        px[h] -= p.Wout;
                        if (++py[h] == p.Hout) { py[h] = 0; ++pb[h]; }
                    }
                }
                mask = ok[0] ? 1u : 0u;
#pragma unroll
                for (int i = 0; i < NU; ++i) {
                    const int h = 0, chunk = i;
                    const int c = cb + chunk * 32;
                    const bool live = chunk < nlive && ok[h] && c < p.Cin;
                    if (VEC) {
                        float4 q4 = make_float4(0.f, 0.f, 0.f, 0.f);
                        if (live) q4 = __ldg(reinterpret_cast<const float4 *>(xg + off[h] + chunk * 32));
                        if (c + 3 >= p.Cin) {        // channel tail of a 16-byte-padded row
                            if (c + 1 >= p.Cin) q4.y = 0.f;
                            if (c + 2 >= p.Cin) q4.z = 0.f;
                            q4.w = 0.f;
                        }
                        v[i].v[0] = q4.x; v[i].v[1] = q4.y; v[i].v[2] = q4.z; v[i].v[3] = q4.w;
                    } else {
#pragma unroll
                        for (int e = 0; e < 4; ++e) {
                            float q1 = 0.f;
                            if (live && c + e < p.Cin) q1 = __ldg(xg + off[h] + chunk * 32 + e);
                            v[i].v[e] = q1;
                        }
                    }
                }
            };
            int xs_s = 0;
            uint32_t xs_ph = 0;
            auto store_x = [&](int it, F4(&v)[NU], uint32_t mask) {
                const int s = xs_s;
                const uint32_t ph = xs_ph;
                if (++xs_s == S) { xs_s = 0; xs_ph ^= 1; }
                if (PRE != 0) {
#pragma unroll
                    for (int i = 0; i < NU; ++i)
#pragma unroll
                        for (int e = 0; e < 4; ++e) {
                            float a = v[i].v[e];
                            if (AFF) {
                                a = fmaf(a, sc[i][e], sh[i][e]);
                                if (RELU) a = fmaxf(a, 0.f);
                                a = (mask & 1u) ? a : 0.f;
                            } else {
                                a = fmaxf(a, 0.f);
                            }
                            v[i].v[e] = a;
                        }
                }
                mbar_wait(empty(s), ph ^ 1);
                const uint32_t t_hi = base + (uint32_t)s * stage_bytes;
                split_store(t_hi, t_hi + A_BYTES, v, nlive);
                fence_proxy_async();
                mbar_arrive(full(s));
            };
            F4 va[NU], vb[NU];
            uint32_t ma = 0, mb = 0;
            int it = 0;
            if (it < nkb) load_x(it, va, ma);
            for (; it < nkb; it += 2) {
                const bool more = it + 1 < nkb;
                if (more) load_x(it + 1, vb, mb);
                store_x(it, va, ma);
                if (more) {
                    if (it + 2 < nkb) load_x(it + 2, va, ma);
                    store_x(it + 1, vb, mb);
                }
            }
        } else {
            // ------------------------------ dY tiles (B operand): ceil(n_tile/32) <= 2 chunks of output channels ---
            const int dys = (int)p.dys;
            const int nchunk = (n_tile + 31) >> 5;
            const int cb = nt * n_tile + unit * 4;
            const float *__restrict__ dg = p.dy;
            auto load_d = [&](int it, F4(&v)[NU]) {
                const int kb = kb0 + it;
#pragma unroll
                for (int i = 0; i < NU; ++i) {
                    const int chunk = i;
                    const int m = kb * BLOCK_KP + r0;
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
                const int s = ds_s;
                mbar_wait(empty(s), ds_ph ^ 1);
                const uint32_t t_hi = base + (uint32_t)s * stage_bytes + 2 * A_BYTES;
                split_store(t_hi, t_hi + (uint32_t)p.b_bytes, v, nchunk);
                fence_proxy_async();
                mbar_arrive(full(s));
                if (++ds_s == S) { ds_s = 0; ds_ph ^= 1; }
            };
            F4 va[NU], vb[NU];
            const int nj = nkb;
            int it = 0;
            if (it < nj) load_d(it, va);
            for (; it < nj; it += 2) {
                const bool more = it + 1 < nj;
                if (more) load_d(it + 1, vb);
                store_d(va);
                if (more) {
                    if (it + 2 < nj) load_d(it + 2, va);
                    store_d(vb);
                }
            }
        }

    }
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
    p.precision = precision;
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
        p.stage_bytes = 2 * A_BYTES + 2 * p.b_bytes;
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
#define BTS_LAUNCH(PRE, UP, VEC)                                                                                    \
    do {                                                                                                            \
        static bool attr_set_[BTS_MAX_DEVICES] = {}; bool &attr_set = attr_set_[bts_cur_device()];                                                                             \
        if (!attr_set) {                                                                                            \
            err = cudaFuncSetAttribute(wgrad_tc_kernel<PRE, UP, VEC>, cudaFuncAttributeMaxDynamicSharedMemorySize,  \
                                       SMEM_LIMIT);                                                                 \
            if (err != cudaSuccess) return (int)err;                                                                \
            attr_set = true;                                                                                        \
        }                                                                                                           \
        wgrad_tc_kernel<PRE, UP, VEC><<<grid, NUM_THREADS, smem, st>>>(p);                                          \
    } while (0)
#define BTS_DISPATCH_UV(PRE)                                                                     \
    do {                                                                                         \
        if (p.up) { if (vec) BTS_LAUNCH(PRE, true, true); else BTS_LAUNCH(PRE, true, false); }   \
        else { if (vec) BTS_LAUNCH(PRE, false, true); else BTS_LAUNCH(PRE, false, false); }      \
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
    p.precision = precision;
    const int taps = KH * KW;
    p.b_bytes = 2 * 4 * (int)CORE_SBO;
    p.stage_bytes = 2 * A_BYTES + 2 * p.b_bytes;
    p.stages = (SMEM_LIMIT - 1024 - 2 * BLOCK_CI * 4 - 256) / p.stage_bytes;
    if (p.stages > MAX_STAGES) p.stages = MAX_STAGES;
    const int smem = p.stages * p.stage_bytes + 2 * BLOCK_CI * 4 + 256 + 1024;
    dim3 grid(1, width / MAX_N, taps * splitK);
    if (grid.z > 65535) return BTS_EINVAL;
    cudaStream_t st = (cudaStream_t)stream;
    cudaError_t err = cudaSuccess;
    const bool vec = p.x_vec && p.dy_vec;
#define BTS_LAUNCH_G(VEC)                                                                                            \
    do {                                                                                                             \
        static bool attr_set_[BTS_MAX_DEVICES] = {};                                                                 \
        bool &attr_set = attr_set_[bts_cur_device()];                                                                \
        if (!attr_set) {                                                                                             \
            err = cudaFuncSetAttribute(wgrad_tc_kernel<0, false, VEC>, cudaFuncAttributeMaxDynamicSharedMemorySize,  \
                                       SMEM_LIMIT);                                                                  \
            if (err != cudaSuccess) return (int)err;                                                                 \
            attr_set = true;                                                                                         \
        }                                                                                                            \
        wgrad_tc_kernel<0, false, VEC><<<grid, NUM_THREADS, smem, st>>>(p);                                          \
    } while (0)
    if (vec) BTS_LAUNCH_G(true); else BTS_LAUNCH_G(false);
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
