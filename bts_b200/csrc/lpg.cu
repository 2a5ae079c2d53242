// Local planar guidance (LPG) plane-to-depth up-sample, forward + backward, sm_90a.
//
// Replaces: pytorch/bts.py:124-146 (local_planar_guidance.forward + its autograd backward, ~15-25
// full-resolution ATen passes) and tensorflow/custom_layer/local_planar_guidance.cu:33-72 / 95-150.
//
// HBM-bound streaming kernels (algorithmic traffic: fwd 4*(1+4/r^2) B/px, bwd 4*(1+8/r^2) B/px):
//   * one lane owns a float4 of 4 consecutive output columns and walks the r rows of its patch row,
//     so every warp-level LDG/STG.128 covers 512 contiguous bytes of one output row;
//   * plane coefficients are read once per patch (16 B), never re-read per pixel;
//   * backward reduces the r x r tile in registers; for r = 8 the two lanes that share a patch
//     combine with one warp shuffle -- no atomics, no global read-modify-write, deterministic;
//   * the index grid u,v = ((k mod r) - (r-1)/2)/r is compile-time exact (dyadic) for r = 2,4,8 and
//     the denominator is evaluated as ((n1*u) + (n2*v)) + n3 with un-contracted mul/add, which makes
//     the forward bit-identical to the reference's fp32 arithmetic (pytorch/bts.py:146).
#include "common.cuh"

namespace {

template <int R>
__device__ __forceinline__ float grid_at(int k) {   // exact for power-of-two R
    return ((float)k - (float)(R - 1) * 0.5f) / (float)R;
}
__device__ __forceinline__ float grid_rt(int k, int r) {   // custom_layer/local_planar_guidance.cc:100-101
    return ((float)k - (float)(r - 1.0f) / 2.0f) / (float)r;
}

#define BTS_SRC_HEAD 2 /* internal: `plane` is the (B,3,h,w) output of reduc.plane_params (pytorch/bts.py:98) */

struct HeadVals {   // everything the head tail computes for one patch (pytorch/bts.py:112-120, 223-226)
    float s0, s1, s2, st, ct, sp, cp, nrm;
    float4 eq;      // (n^1, n^2, n^3, dist)
};

__device__ __forceinline__ float sigmoidf_(float x) { return 1.0f / (1.0f + expf(-x)); }

__device__ __forceinline__ HeadVals head_eval(float c0, float c1, float c2, float max_depth) {
    HeadVals v;
    v.s0 = sigmoidf_(c0); v.s1 = sigmoidf_(c1); v.s2 = sigmoidf_(c2);
    const float theta = __fdiv_rn(__fmul_rn(v.s0, 3.14159274101257324f), 3.0f);   // sigmoid * math.pi / 3
    const float phi = __fmul_rn(__fmul_rn(v.s1, 3.14159274101257324f), 2.0f);     // sigmoid * math.pi * 2
    sincosf(theta, &v.st, &v.ct);
    sincosf(phi, &v.sp, &v.cp);
    const float n1 = __fmul_rn(v.st, v.cp), n2 = __fmul_rn(v.st, v.sp), n3 = v.ct;
    v.nrm = fmaxf(sqrtf(__fadd_rn(__fadd_rn(__fmul_rn(n1, n1), __fmul_rn(n2, n2)), __fmul_rn(n3, n3))), 1e-12f);
    v.eq = make_float4(__fdiv_rn(n1, v.nrm), __fdiv_rn(n2, v.nrm), __fdiv_rn(n3, v.nrm), __fmul_rn(v.s2, max_depth));
    return v;
}

struct PlaneSrc {
    const float *p;      // plane (NCHW / NHWC) or c3 (HEAD)
    float *plane_out;    // HEAD only: optional (B,4,h,w) copy of the plane equation
    float max_depth;     // HEAD only
};

template <int LAYOUT>
__device__ __forceinline__ float4 load_plane(const PlaneSrc &src, int b, int i, int j, int h, int w, bool writer) {
    if (LAYOUT == BTS_LAYOUT_NHWC) {
        return __ldg(reinterpret_cast<const float4 *>(src.p) + ((size_t)b * h + i) * w + j);
    } else if (LAYOUT == BTS_LAYOUT_NCHW) {
        const size_t hw = (size_t)h * w;
        const float *p = src.p + (size_t)b * 4 * hw + (size_t)i * w + j;
        return make_float4(__ldg(p), __ldg(p + hw), __ldg(p + 2 * hw), __ldg(p + 3 * hw));
    } else {
        const size_t hw = (size_t)h * w;
        const float *p = src.p + (size_t)b * 3 * hw + (size_t)i * w + j;
        const HeadVals v = head_eval(__ldg(p), __ldg(p + hw), __ldg(p + 2 * hw), src.max_depth);
        if (writer && src.plane_out) {
            float *q = src.plane_out + (size_t)b * 4 * hw + (size_t)i * w + j;
            q[0] = v.eq.x; q[hw] = v.eq.y; q[2 * hw] = v.eq.z; q[3 * hw] = v.eq.w;
        }
        return v.eq;
    }
}

template <int LAYOUT>
__device__ __forceinline__ void store_plane(float *__restrict__ dplane, const PlaneSrc &src, int b, int i, int j, int h,
                                            int w, float4 g) {
    if (LAYOUT == BTS_LAYOUT_NHWC) {
        reinterpret_cast<float4 *>(dplane)[((size_t)b * h + i) * w + j] = g;
    } else if (LAYOUT == BTS_LAYOUT_NCHW) {
        const size_t hw = (size_t)h * w;
        float *p = dplane + (size_t)b * 4 * hw + (size_t)i * w + j;
        p[0] = g.x; p[hw] = g.y; p[2 * hw] = g.z; p[3 * hw] = g.w;
    } else {
        // chain rule through normalize -> (sin,cos) -> sigmoid, back to the 3 conv channels
        const size_t hw = (size_t)h * w;
        const float *p = src.p + (size_t)b * 3 * hw + (size_t)i * w + j;
        const HeadVals v = head_eval(__ldg(p), __ldg(p + hw), __ldg(p + 2 * hw), src.max_depth);
        const float dot = g.x * v.eq.x + g.y * v.eq.y + g.z * v.eq.z;
        const float inv = 1.0f / v.nrm;
        const float d1 = (g.x - v.eq.x * dot) * inv, d2 = (g.y - v.eq.y * dot) * inv, d3 = (g.z - v.eq.z * dot) * inv;
        const float dth = d1 * v.ct * v.cp + d2 * v.ct * v.sp - d3 * v.st;
        const float dph = -d1 * v.st * v.sp + d2 * v.st * v.cp;
        float *q = dplane + (size_t)b * 3 * hw + (size_t)i * w + j;
        q[0] = dth * (3.14159274101257324f / 3.0f) * v.s0 * (1.0f - v.s0);
        q[hw] = dph * (3.14159274101257324f * 2.0f) * v.s1 * (1.0f - v.s1);
        q[2 * hw] = g.w * src.max_depth * v.s2 * (1.0f - v.s2);
    }
}

__device__ __forceinline__ float lpg_den(float n1, float n2, float n3, float u, float v) {
    return __fadd_rn(__fadd_rn(__fmul_rn(n1, u), __fmul_rn(n2, v)), n3);
}

// ------------------------------------------------------------------------------------------ forward
// FUSED = false: depth only.  FUSED = true: scaled = depth/max_depth (+ optional ds = scaled[::R/2, ::R/2]).
template <int R, int LAYOUT, bool FUSED>
__global__ void __launch_bounds__(256) lpg_fwd_vec(const PlaneSrc plane, float *__restrict__ depth,
                                                   float *__restrict__ scaled, float *__restrict__ ds,
                                                   float max_depth, int B, int h, int w) {
    constexpr int NP = (R == 2) ? 2 : 1;   // patches per lane
    constexpr int CPP = 4 / NP;            // columns per patch within the float4
    constexpr int S = (R >= 4) ? R / 2 : 1;
    const unsigned W = w * R, H = h * R, Wq = W >> 2;
    const unsigned total = (unsigned)B * h * Wq;
    const unsigned idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= total) return;
    const unsigned xq = idx % Wq;
    const unsigned t = idx / Wq;
    const unsigned i = t % h, b = t / h;
    const unsigned j0 = (R == 2) ? 2 * xq : (4 * xq) / R;
    const unsigned c0 = (R == 2) ? 0 : (4 * xq) % R;

    float n1u[4], n2[NP], n3[NP], n4[NP];
#pragma unroll
    for (int p = 0; p < NP; ++p) {
        const float4 pl = load_plane<LAYOUT>(plane, b, i, j0 + p, h, w, c0 == 0);
        n2[p] = pl.y; n3[p] = pl.z; n4[p] = pl.w;
#pragma unroll
        for (int c = 0; c < CPP; ++c) n1u[p * CPP + c] = __fmul_rn(pl.x, grid_at<R>(c0 + c));
    }
    const size_t row0 = ((size_t)b * H + (size_t)i * R) * W + 4 * (size_t)xq;
#pragma unroll
    for (int k = 0; k < R; ++k) {
        const float v = grid_at<R>(k);
        float d[4];
#pragma unroll
        for (int c = 0; c < 4; ++c) {
            const int p = c / CPP;
            const float den = __fadd_rn(__fadd_rn(n1u[c], __fmul_rn(n2[p], v)), n3[p]);
            d[c] = __fdiv_rn(n4[p], den);
        }
        const size_t off = row0 + (size_t)k * W;
        if (!FUSED) {
            *reinterpret_cast<float4 *>(depth + off) = make_float4(d[0], d[1], d[2], d[3]);
        } else {
#pragma unroll
            for (int c = 0; c < 4; ++c) d[c] = __fdiv_rn(d[c], max_depth);
            *reinterpret_cast<float4 *>(scaled + off) = make_float4(d[0], d[1], d[2], d[3]);
            if (R >= 4 && (k % S) == 0 && ds) {
                // nearest down-sample by S (Q14): rows k = 0, S; columns 4*xq + c with c % S == 0
                const unsigned Ws = W / S, Hs = H / S;
                float *q = ds + ((size_t)b * Hs + (i * R + k) / S) * Ws + (4 * xq) / S;
                if (S == 4) q[0] = d[0];
                else { q[0] = d[0]; q[1] = d[2]; }
            }
        }
    }
}

// any r (1 or even per the TF shape function, .cc:36-44; odd values work too), any alignment
template <int LAYOUT>
__global__ void __launch_bounds__(256) lpg_fwd_generic(const PlaneSrc plane, float *__restrict__ depth,
                                                       float *__restrict__ scaled, float *__restrict__ ds,
                                                       float max_depth, int S, int B, int h, int w, int r) {
    const int W = w * r, H = h * r;
    const long long total = (long long)B * H * W;
    for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
         idx += (long long)gridDim.x * blockDim.x) {
        const int x = (int)(idx % W);
        const long long t = idx / W;
        const int y = (int)(t % H), b = (int)(t / H);
        const float4 pl = load_plane<LAYOUT>(plane, b, y / r, x / r, h, w, (x % r == 0) && (y % r == 0));
        const float d = __fdiv_rn(pl.w, lpg_den(pl.x, pl.y, pl.z, grid_rt(x % r, r), grid_rt(y % r, r)));
        if (depth) depth[idx] = d;
        if (scaled || ds) {
            const float s = __fdiv_rn(d, max_depth);
            if (scaled) scaled[idx] = s;
            if (ds && (y % S == 0) && (x % S == 0)) ds[((size_t)b * (H / S) + y / S) * (W / S) + x / S] = s;
        }
    }
}

// ------------------------------------------------------------------------------------------ backward
// FUSED = false: dY = d_depth.
// FUSED = true : dY = (d_scaled + [y%S==0 && x%S==0] d_ds[y/S, x/S]) / max_depth with S = R/2 (d_ds optional).
// Every global load of the tile is issued before the first use (R independent 16-byte loads per lane in flight);
// per pixel: den (2 FADD), one MUFU reciprocal, q = dY/den, pp = dY/den^2, three running sums.  The u / v / n4
// factors are pulled out of the pixel loop: column sums carry u, row sums carry v.
template <int R, int LAYOUT, bool FUSED>
__global__ void __launch_bounds__(256) lpg_bwd_vec(const float *__restrict__ d_depth, const float *__restrict__ d_scaled,
                                                   const float *__restrict__ d_ds, float max_depth,
                                                   const PlaneSrc plane, float *__restrict__ dplane,
                                                   int B, int h, int w, int tf_compat) {
    constexpr int NP = (R == 2) ? 2 : 1;
    constexpr int CPP = 4 / NP;
    constexpr int LPP = (R >= 4) ? R / 4 : 1;   // lanes that share one patch (r=8: 2)
    constexpr int S = (R >= 4) ? R / 2 : 1;
    const unsigned W = w * R, H = h * R, Wq = W >> 2;
    const unsigned total = (unsigned)B * h * Wq;
    const unsigned idx = blockIdx.x * blockDim.x + threadIdx.x;
    const bool active = idx < total;            // inactive lanes still take part in the shuffle
    const unsigned idc = active ? idx : 0;
    const unsigned xq = idc % Wq;
    const unsigned t = idc / Wq;
    const unsigned i = t % h, b = t / h;
    const unsigned j0 = (R == 2) ? 2 * xq : (4 * xq) / R;
    const unsigned c0 = (R == 2) ? 0 : (4 * xq) % R;

    float g[NP][4];
#pragma unroll
    for (int p = 0; p < NP; ++p) g[p][0] = g[p][1] = g[p][2] = g[p][3] = 0.f;

    if (active) {
        const size_t row0 = ((size_t)b * H + (size_t)i * R) * W + 4 * (size_t)xq;
        const float *src = FUSED ? d_scaled : d_depth;
        float4 dy4[R];
#pragma unroll
        for (int k = 0; k < R; ++k) dy4[k] = __ldg(reinterpret_cast<const float4 *>(src + row0 + (size_t)k * W));
        float e0 = 0.f, e1 = 0.f, e2 = 0.f, e3 = 0.f;   // d_ds contributions: rows 0 and S; columns 0 (and 2)
        if (FUSED && R >= 4 && d_ds) {
            const unsigned Ws = W / S, Hs = H / S;
            const float *q = d_ds + ((size_t)b * Hs + (i * R) / S) * Ws + (4 * xq) / S;
            e0 = __ldg(q);
            e2 = __ldg(q + Ws);
            if (S == 2) { e1 = __ldg(q + 1); e3 = __ldg(q + Ws + 1); }
        }
        float4 pl[NP];
#pragma unroll
        for (int p = 0; p < NP; ++p) pl[p] = load_plane<LAYOUT>(plane, b, i, j0 + p, h, w, false);
        float dy[R][4];
#pragma unroll
        for (int k = 0; k < R; ++k) { dy[k][0] = dy4[k].x; dy[k][1] = dy4[k].y; dy[k][2] = dy4[k].z; dy[k][3] = dy4[k].w; }
        if (FUSED) {
            if (R >= 4) {
                dy[0][0] += e0; dy[S][0] += e2;
                if (S == 2) { dy[0][2] += e1; dy[S][2] += e3; }
            }
            const float inv_md = 1.0f / max_depth;
#pragma unroll
            for (int k = 0; k < R; ++k)
#pragma unroll
                for (int c = 0; c < 4; ++c) dy[k][c] *= inv_md;
        }
        float n1u[4];
#pragma unroll
        for (int c = 0; c < 4; ++c) n1u[c] = __fmul_rn(pl[c / CPP].x, grid_at<R>(c0 + (c % CPP)));
        float colsum[4] = {0.f, 0.f, 0.f, 0.f};   // sum over rows of pp, per column
        float vsum[NP], qsum[NP];
#pragma unroll
        for (int p = 0; p < NP; ++p) vsum[p] = qsum[p] = 0.f;
#pragma unroll
        for (int k = 0; k < R; ++k) {
            const float v = grid_at<R>(k);
            float rowsum[NP];
#pragma unroll
            for (int p = 0; p < NP; ++p) rowsum[p] = 0.f;
#pragma unroll
            for (int c = 0; c < 4; ++c) {
                const int p = c / CPP;
                const float den = __fadd_rn(__fadd_rn(n1u[c], __fmul_rn(pl[p].y, v)), pl[p].z);
                float inv;
                asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(inv) : "f"(den));
                const float q = dy[k][c] * inv;       // dY/den
                const float pp = q * inv;             // dY/den^2
                colsum[c] += pp;
                rowsum[p] += pp;
                qsum[p] += q;
            }
#pragma unroll
            for (int p = 0; p < NP; ++p) vsum[p] = fmaf(v, rowsum[p], vsum[p]);
        }
#pragma unroll
        for (int p = 0; p < NP; ++p) {
            float us = 0.f, ps = 0.f;
#pragma unroll
            for (int c = 0; c < CPP; ++c) {
                us = fmaf(grid_at<R>(c0 + c), colsum[p * CPP + c], us);
                ps += colsum[p * CPP + c];
            }
            const float sc = tf_compat ? 1.0f : pl[p].w;   // true gradient carries n4 (SURVEY Q5)
            g[p][0] = -sc * us;
            g[p][1] = -sc * vsum[p];
            g[p][2] = -sc * ps;
            g[p][3] = qsum[p];
        }
    }
    if (LPP > 1) {
#pragma unroll
        for (int m = 1; m < LPP; m <<= 1)
#pragma unroll
            for (int q = 0; q < 4; ++q) g[0][q] += __shfl_xor_sync(0xffffffffu, g[0][q], m);
    }
    if (!active) return;
    if (LPP > 1 && (xq % LPP) != 0) return;
#pragma unroll
    for (int p = 0; p < NP; ++p)
        store_plane<LAYOUT>(dplane, plane, b, i, j0 + p, h, w, make_float4(g[p][0], g[p][1], g[p][2], g[p][3]));
}

template <int LAYOUT>
__global__ void __launch_bounds__(256) lpg_bwd_generic(const float *__restrict__ d_depth, const float *__restrict__ d_scaled,
                                                       const float *__restrict__ d_ds, float max_depth, int S,
                                                       const PlaneSrc plane, float *__restrict__ dplane,
                                                       int B, int h, int w, int r, int tf_compat) {
    const int W = w * r, H = h * r;
    const long long total = (long long)B * h * w;
    for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
         idx += (long long)gridDim.x * blockDim.x) {
        const int j = (int)(idx % w);
        const long long t = idx / w;
        const int i = (int)(t % h), b = (int)(t / h);
        const float4 pl = load_plane<LAYOUT>(plane, b, i, j, h, w, false);
        float g0 = 0.f, g1 = 0.f, g2 = 0.f, g3 = 0.f;
        for (int a = 0; a < r; ++a)
            for (int c = 0; c < r; ++c) {
                const int y = i * r + a, x = j * r + c;
                const size_t off = ((size_t)b * H + y) * W + x;
                float dy = 0.f;
                if (d_scaled) dy = d_scaled[off];
                if (d_ds && (y % S == 0) && (x % S == 0)) dy += d_ds[((size_t)b * (H / S) + y / S) * (W / S) + x / S];
                if (d_scaled || d_ds) dy = __fdiv_rn(dy, max_depth);
                if (d_depth) dy += d_depth[off];
                const float u = grid_rt(c, r), v = grid_rt(a, r);
                const float inv = __frcp_rn(lpg_den(pl.x, pl.y, pl.z, u, v));
                const float q = dy * inv;
                float pp = q * inv;
                if (!tf_compat) pp *= pl.w;
                g0 -= pp * u; g1 -= pp * v; g2 -= pp; g3 += q;
            }
        store_plane<LAYOUT>(dplane, plane, b, i, j, h, w, make_float4(g0, g1, g2, g3));
    }
}

bool fast_ok(int r, int w, int layout, const void *a, const void *b, const void *c, const void *d) {
    if (r != 2 && r != 4 && r != 8) return false;
    if ((w * r) % 4 != 0) return false;
    if (!bts_aligned16(a) || !bts_aligned16(b) || !bts_aligned16(c)) return false;
    if (layout == BTS_LAYOUT_NHWC && !bts_aligned16(d)) return false;
    return true;
}

template <int LAYOUT>
int launch_fwd(const PlaneSrc plane, float *depth, float *scaled, float *ds, float max_depth, int S, int B, int h,
               int w, int r, cudaStream_t st) {
    const long long total = (long long)B * h * (w * r / 4);
    // vector kernels: depth only, or scaled (+ ds with stride r/2) only; everything else -> generic kernel
    const bool plain = depth && !scaled && !ds;
    const bool fused = !depth && scaled && (!ds || (r >= 4 && S == r / 2));
    if (fast_ok(r, w, LAYOUT, depth, scaled, nullptr, plane.p) && (plain || fused) && total < 0x7fffffffLL) {
        const int grid = bts_ceil_div(total, 256);
#define BTS_FWD(RR)                                                                                                \
    if (plain) lpg_fwd_vec<RR, LAYOUT, false><<<grid, 256, 0, st>>>(plane, depth, scaled, ds, max_depth, B, h, w); \
    else lpg_fwd_vec<RR, LAYOUT, true><<<grid, 256, 0, st>>>(plane, depth, scaled, ds, max_depth, B, h, w);
        if (r == 2) { BTS_FWD(2) } else if (r == 4) { BTS_FWD(4) } else { BTS_FWD(8) }
#undef BTS_FWD
    } else {
        const long long npx = (long long)B * h * r * w * r;
        long long grid = (npx + 255) / 256;
        const long long cap = (long long)bts_num_sms() * 16;
        if (grid > cap) grid = cap;
        lpg_fwd_generic<LAYOUT><<<(int)grid, 256, 0, st>>>(plane, depth, scaled, ds, max_depth, S, B, h, w, r);
    }
    BTS_LAUNCH_CHECK();
    return 0;
}

template <int LAYOUT>
int launch_bwd(const float *d_depth, const float *d_scaled, const float *d_ds, float max_depth, int S,
               const PlaneSrc plane, float *dplane, int B, int h, int w, int r, int tfc, cudaStream_t st) {
    const long long total = (long long)B * h * (w * r / 4);
    const bool plain = d_depth && !d_scaled && !d_ds;
    const bool fused = !d_depth && d_scaled && (!d_ds || (r >= 4 && S == r / 2));
    if (fast_ok(r, w, LAYOUT, d_depth, d_scaled, LAYOUT == BTS_LAYOUT_NHWC ? (const void *)dplane : nullptr, plane.p) &&
        (plain || fused) && total < 0x7fffffffLL) {
        const int grid = bts_ceil_div(total, 256);
#define BTS_BWD(RR)                                                                                              \
    if (plain) lpg_bwd_vec<RR, LAYOUT, false><<<grid, 256, 0, st>>>(d_depth, d_scaled, d_ds, max_depth, plane,   \
                                                                    dplane, B, h, w, tfc);                       \
    else lpg_bwd_vec<RR, LAYOUT, true><<<grid, 256, 0, st>>>(d_depth, d_scaled, d_ds, max_depth, plane, dplane, \
                                                             B, h, w, tfc);
        if (r == 2) { BTS_BWD(2) } else if (r == 4) { BTS_BWD(4) } else { BTS_BWD(8) }
#undef BTS_BWD
    } else {
        const long long npatch = (long long)B * h * w;
        long long grid = (npatch + 255) / 256;
        const long long cap = (long long)bts_num_sms() * 16;
        if (grid > cap) grid = cap;
        lpg_bwd_generic<LAYOUT><<<(int)grid, 256, 0, st>>>(d_depth, d_scaled, d_ds, max_depth, S, plane, dplane, B, h, w, r, tfc);
    }
    BTS_LAUNCH_CHECK();
    return 0;
}

int check_common(const void *plane, int B, int h, int w, int r, int layout) {
    if (B < 0 || h < 0 || w < 0) return BTS_EINVAL;
    if (!plane && (long long)B * h * w != 0) return BTS_EINVAL;   // an empty tensor may legitimately be null
    if (r < 1 || (r > 1 && (r % 2) != 0)) return BTS_EINVAL;   // "Upratio should be multiple of 2 or 1" (.cc:36-44)
    if (layout != BTS_LAYOUT_NCHW && layout != BTS_LAYOUT_NHWC) return BTS_EINVAL;
    return 0;
}

}  // namespace

extern "C" int bts_lpg_fwd(const float *plane, float *depth, int B, int h, int w, int r, int layout, void *stream) {
    int rc = check_common(plane, B, h, w, r, layout);
    if (rc) return rc;
    if ((long long)B * h * w == 0) return 0;   // empty input: nothing to do (TF op allocates an empty output)
    if (!depth) return BTS_EINVAL;
    cudaStream_t st = (cudaStream_t)stream;
    const PlaneSrc src{plane, nullptr, 0.f};
    return layout == BTS_LAYOUT_NCHW ? launch_fwd<BTS_LAYOUT_NCHW>(src, depth, nullptr, nullptr, 1.f, 1, B, h, w, r, st)
                                     : launch_fwd<BTS_LAYOUT_NHWC>(src, depth, nullptr, nullptr, 1.f, 1, B, h, w, r, st);
}

extern "C" int bts_lpg_bwd(const float *dy, const float *plane, float *dplane, int B, int h, int w, int r, int layout,
                           int tf_compat, void *stream) {
    int rc = check_common(plane, B, h, w, r, layout);
    if (rc) return rc;
    if ((long long)B * h * w == 0) return 0;
    if (!dy || !dplane) return BTS_EINVAL;
    cudaStream_t st = (cudaStream_t)stream;
    const PlaneSrc src{plane, nullptr, 0.f};
    return layout == BTS_LAYOUT_NCHW
               ? launch_bwd<BTS_LAYOUT_NCHW>(dy, nullptr, nullptr, 1.f, 1, src, dplane, B, h, w, r, tf_compat, st)
               : launch_bwd<BTS_LAYOUT_NHWC>(dy, nullptr, nullptr, 1.f, 1, src, dplane, B, h, w, r, tf_compat, st);
}

// ---- fused plane-coefficient head tail + LPG (pytorch/bts.py:112-120 + 223-229) -------------------
extern "C" int bts_plane_head_fwd(const float *c3, float *plane_out, float *scaled, float *ds, float max_depth,
                                  int ds_stride, int B, int h, int w, int r, void *stream) {
    int rc = check_common(c3, B, h, w, r, BTS_LAYOUT_NCHW);
    if (rc) return rc;
    if (!scaled || !(max_depth > 0.f)) return BTS_EINVAL;
    if (ds && (ds_stride < 1 || (h * r) % ds_stride || (w * r) % ds_stride)) return BTS_EINVAL;
    if ((long long)B * h * w == 0) return 0;
    const PlaneSrc src{c3, plane_out, max_depth};
    return launch_fwd<BTS_SRC_HEAD>(src, nullptr, scaled, ds, max_depth, ds ? ds_stride : 1, B, h, w, r,
                                    (cudaStream_t)stream);
}

extern "C" int bts_plane_head_bwd(const float *d_scaled, const float *d_ds, const float *c3, float *dc3,
                                  float max_depth, int ds_stride, int B, int h, int w, int r, void *stream) {
    int rc = check_common(c3, B, h, w, r, BTS_LAYOUT_NCHW);
    if (rc) return rc;
    if (!dc3 || (!d_scaled && !d_ds) || !(max_depth > 0.f)) return BTS_EINVAL;
    if (d_ds && (ds_stride < 1 || (h * r) % ds_stride || (w * r) % ds_stride)) return BTS_EINVAL;
    if ((long long)B * h * w == 0) return 0;
    const PlaneSrc src{c3, nullptr, max_depth};
    return launch_bwd<BTS_SRC_HEAD>(nullptr, d_scaled, d_ds, max_depth, d_ds ? ds_stride : 1, src, dc3, B, h, w, r, 0,
                                    (cudaStream_t)stream);
}

// ---- host-pointer plugin form (TF-op surface: LocalPlanarGuidanceOp / GradOp ::Compute) ----------
namespace {
struct DevBuf {
    void *p = nullptr;
    cudaError_t alloc(size_t n) { return cudaMalloc(&p, n ? n : 16); }
    ~DevBuf() { if (p) cudaFree(p); }
};
}  // namespace

extern "C" int bts_lpg_fwd_h(const float *plane_host, float *depth_host, int B, int h, int w, int r, int layout) {
    if (!plane_host || !depth_host) return BTS_EINVAL;
    int rc = check_common(plane_host, B, h, w, r, layout);
    if (rc) return rc;
    const size_t np = (size_t)B * h * w * 4 * sizeof(float), nd = (size_t)B * h * r * w * r * sizeof(float);
    if (nd == 0) return 0;
    DevBuf dp, dd;
    cudaError_t e;
    if ((e = dp.alloc(np)) != cudaSuccess || (e = dd.alloc(nd)) != cudaSuccess) return (int)e;
    if ((e = cudaMemcpyAsync(dp.p, plane_host, np, cudaMemcpyHostToDevice, 0)) != cudaSuccess) return (int)e;
    rc = bts_lpg_fwd((const float *)dp.p, (float *)dd.p, B, h, w, r, layout, nullptr);
    if (rc) return rc;
    if ((e = cudaMemcpyAsync(depth_host, dd.p, nd, cudaMemcpyDeviceToHost, 0)) != cudaSuccess) return (int)e;
    return (int)cudaStreamSynchronize(0);
}

extern "C" int bts_lpg_bwd_h(const float *dy_host, const float *plane_host, float *dplane_host, int B, int h, int w,
                             int r, int layout, int tf_compat) {
    if (!dy_host || !plane_host || !dplane_host) return BTS_EINVAL;
    int rc = check_common(plane_host, B, h, w, r, layout);
    if (rc) return rc;
    const size_t np = (size_t)B * h * w * 4 * sizeof(float), nd = (size_t)B * h * r * w * r * sizeof(float);
    if (nd == 0) return 0;
    DevBuf dp, dd, dg;
    cudaError_t e;
    if ((e = dp.alloc(np)) != cudaSuccess || (e = dd.alloc(nd)) != cudaSuccess || (e = dg.alloc(np)) != cudaSuccess)
        return (int)e;
    if ((e = cudaMemcpyAsync(dp.p, plane_host, np, cudaMemcpyHostToDevice, 0)) != cudaSuccess) return (int)e;
    if ((e = cudaMemcpyAsync(dd.p, dy_host, nd, cudaMemcpyHostToDevice, 0)) != cudaSuccess) return (int)e;
    rc = bts_lpg_bwd((const float *)dd.p, (const float *)dp.p, (float *)dg.p, B, h, w, r, layout, tf_compat, nullptr);
    if (rc) return rc;
    if ((e = cudaMemcpyAsync(dplane_host, dg.p, np, cudaMemcpyDeviceToHost, 0)) != cudaSuccess) return (int)e;
    return (int)cudaStreamSynchronize(0);
}
