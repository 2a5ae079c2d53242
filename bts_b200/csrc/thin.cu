// Single-output-channel convolutions (Cout = 1) as HBM-bound CUDA-core kernels, sm_90a.
//
// Replaces, for the two 1-channel heads of the BTS decoder -- `get_depth` (3x3, 32->1, + Sigmoid; reference
// pytorch/bts.py:193-194,262) and `reduc1x1.reduc.final` (1x1, 8->1, + Sigmoid; bts.py:94-96) -- the cuDNN conv /
// sigmoid / their backward kernels.  With one output channel there is no GEMM: a tensor-core tile would carry a single
// live column, so these are written as streaming kernels (SURVEY 7 "Cout 1/3 heads are better as CUDA-core GEMV").
//
// Layout: x NHWC (pixel stride xs), C in {8,16,32,64,128}; LPP = C/4 lanes share one pixel, each lane owning 4
// channels (one 16-byte load per tap, so a warp instruction reads 32/LPP full pixel rows -- coalesced).
//   fwd  : y[p]      = act( sum_tap sum_c x[p+tap][c] * w[tap][c] )               act: none | sigmoid
//   dgrad: dx[p][c]  = sum_tap g[p-tap] * w[tap][c]                                g = dy * s(1-s) if sigmoid
//   wgrad: dw[tap][c]= sum_p   g[p] * x[p+tap][c]        per-block partials + a fixed-order second pass (deterministic)
#include "common.cuh"

namespace {

constexpr int MAXC = 128;
constexpr int MAXTAPS = 9;

struct ThinParams {
    const float *x; long long xs;
    int B, H, W, C, K;            // stride 1, dilation 1, pad = K/2
    const float *w; long long s_ci, s_kh, s_kw;
    const float *dy;              // (B,H,W) upstream gradient            (backward)
    const float *s;               // (B,H,W) saved sigmoid output or null (backward)
    float *y;                     // (B,H,W) output                        (forward)
    float *dx; long long dxs;     // NHWC gradient wrt x                   (dgrad)
    float *part;                  // [gridDim.x][K*K*C] partials           (wgrad)
    int act;
};

__device__ __forceinline__ float geff(const ThinParams &p, size_t idx) {
    const float g = __ldg(p.dy + idx);
    if (!p.s) return g;
    const float s = __ldg(p.s + idx);
    return g * s * (1.0f - s);
}

__device__ __forceinline__ void load_w(const ThinParams &p, float *sw) {
    const int taps = p.K * p.K;
    for (int i = threadIdx.x; i < taps * p.C; i += blockDim.x) {
        const int tap = i / p.C, c = i - tap * p.C;
        sw[i] = p.w[c * p.s_ci + (tap / p.K) * p.s_kh + (tap % p.K) * p.s_kw];
    }
    __syncthreads();
}

template <int LPP>
__global__ void __launch_bounds__(256) thin_fwd(const ThinParams p) {
    __shared__ __align__(16) float sw[MAXTAPS * MAXC];
    load_w(p, sw);
    const int lane = threadIdx.x & 31;
    const int u = lane % LPP, slot = lane / LPP;
    constexpr int PPW = 32 / LPP;                       // pixels per warp-iteration
    const long long npix = (long long)p.B * p.H * p.W;
    const long long ngroups = (npix + PPW - 1) / PPW;
    const long long warp0 = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const long long nwarps = ((long long)gridDim.x * blockDim.x) >> 5;
    const int pad = p.K / 2;
    for (long long g = warp0; g < ngroups; g += nwarps) {
        const long long pix = g * PPW + slot;
        float acc = 0.f;
        if (pix < npix) {
            const int x = (int)(pix % p.W);
            const long long q = pix / p.W;
            const int y = (int)(q % p.H);
            const long long b = q / p.H;
            for (int ky = 0; ky < p.K; ++ky) {
                const int yy = y + ky - pad;
                if ((unsigned)yy >= (unsigned)p.H) continue;
                for (int kx = 0; kx < p.K; ++kx) {
                    const int xx = x + kx - pad;
                    if ((unsigned)xx >= (unsigned)p.W) continue;
                    const float4 v = __ldg(reinterpret_cast<const float4 *>(p.x + ((b * p.H + yy) * p.W + xx) * p.xs) + u);
                    const float4 wv = *reinterpret_cast<const float4 *>(sw + (ky * p.K + kx) * p.C + 4 * u);
                    acc = fmaf(v.x, wv.x, acc); acc = fmaf(v.y, wv.y, acc);
                    acc = fmaf(v.z, wv.z, acc); acc = fmaf(v.w, wv.w, acc);
                }
            }
        }
#pragma unroll
        for (int m = 1; m < LPP; m <<= 1) acc += __shfl_xor_sync(0xffffffffu, acc, m);
        if (u == 0 && pix < npix) {
            if (p.act == 2) acc = 1.0f / (1.0f + expf(-acc));
            p.y[pix] = acc;
        }
    }
}

template <int LPP>
__global__ void __launch_bounds__(256) thin_dgrad(const ThinParams p) {
    __shared__ __align__(16) float sw[MAXTAPS * MAXC];
    load_w(p, sw);
    const int lane = threadIdx.x & 31;
    const int u = lane % LPP, slot = lane / LPP;
    constexpr int PPW = 32 / LPP;
    const long long npix = (long long)p.B * p.H * p.W;
    const long long ngroups = (npix + PPW - 1) / PPW;
    const long long warp0 = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const long long nwarps = ((long long)gridDim.x * blockDim.x) >> 5;
    const int pad = p.K / 2;
    for (long long g = warp0; g < ngroups; g += nwarps) {
        const long long pix = g * PPW + slot;
        if (pix >= npix) continue;
        const int x = (int)(pix % p.W);
        const long long q = pix / p.W;
        const int y = (int)(q % p.H);
        const long long b = q / p.H;
        float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
        // dx[p] = sum_tap g[p - (tap - pad)] * w[tap]   (the output pixel that saw p through tap (ky,kx))
        for (int ky = 0; ky < p.K; ++ky) {
            const int yy = y - (ky - pad);
            if ((unsigned)yy >= (unsigned)p.H) continue;
            for (int kx = 0; kx < p.K; ++kx) {
                const int xx = x - (kx - pad);
                if ((unsigned)xx >= (unsigned)p.W) continue;
                const float gv = geff(p, (size_t)((b * p.H + yy) * p.W + xx));
                const float4 wv = *reinterpret_cast<const float4 *>(sw + (ky * p.K + kx) * p.C + 4 * u);
                acc.x = fmaf(gv, wv.x, acc.x); acc.y = fmaf(gv, wv.y, acc.y);
                acc.z = fmaf(gv, wv.z, acc.z); acc.w = fmaf(gv, wv.w, acc.w);
            }
        }
        *(reinterpret_cast<float4 *>(p.dx + pix * p.dxs) + u) = acc;
    }
}

template <int LPP, int K>
__global__ void __launch_bounds__(256) thin_wgrad(const ThinParams p) {
    constexpr int TAPS = K * K;
    constexpr int PPW = 32 / LPP;
    constexpr int PAD = K / 2;
    __shared__ float red[8][TAPS * 4 * LPP];            // per-warp results: [tap][channel]
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int u = lane % LPP, slot = lane / LPP;
    const long long npix = (long long)p.B * p.H * p.W;
    const long long ngroups = (npix + PPW - 1) / PPW;
    const long long warp0 = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const long long nwarps = ((long long)gridDim.x * blockDim.x) >> 5;
    float4 acc[TAPS];
#pragma unroll
    for (int t = 0; t < TAPS; ++t) acc[t] = make_float4(0.f, 0.f, 0.f, 0.f);
    for (long long g = warp0; g < ngroups; g += nwarps) {
        const long long pix = g * PPW + slot;
        if (pix >= npix) continue;
        const int x = (int)(pix % p.W);
        const long long q = pix / p.W;
        const int y = (int)(q % p.H);
        const long long b = q / p.H;
        const float gv = geff(p, (size_t)pix);
#pragma unroll
        for (int ky = 0; ky < K; ++ky) {
            const int yy = y + ky - PAD;
#pragma unroll
            for (int kx = 0; kx < K; ++kx) {
                const int xx = x + kx - PAD;
                if ((unsigned)yy < (unsigned)p.H && (unsigned)xx < (unsigned)p.W) {
                    const float4 v = __ldg(reinterpret_cast<const float4 *>(p.x + ((b * p.H + yy) * p.W + xx) * p.xs) + u);
                    float4 &a = acc[ky * K + kx];
                    a.x = fmaf(gv, v.x, a.x); a.y = fmaf(gv, v.y, a.y);
                    a.z = fmaf(gv, v.z, a.z); a.w = fmaf(gv, v.w, a.w);
                }
            }
        }
    }
    // reduce the PPW pixel slots of the warp, then the 8 warps of the block (fixed order -> deterministic)
#pragma unroll
    for (int t = 0; t < TAPS; ++t) {
#pragma unroll
        for (int m = LPP; m < 32; m <<= 1) {
            acc[t].x += __shfl_xor_sync(0xffffffffu, acc[t].x, m);
            acc[t].y += __shfl_xor_sync(0xffffffffu, acc[t].y, m);
            acc[t].z += __shfl_xor_sync(0xffffffffu, acc[t].z, m);
            acc[t].w += __shfl_xor_sync(0xffffffffu, acc[t].w, m);
        }
        if (slot == 0) {
            float *r = &red[warp][t * 4 * LPP + 4 * u];
            r[0] = acc[t].x; r[1] = acc[t].y; r[2] = acc[t].z; r[3] = acc[t].w;
        }
    }
    __syncthreads();
    const int n = TAPS * 4 * LPP;
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
        float sum = 0.f;
#pragma unroll
        for (int wv = 0; wv < 8; ++wv) sum += red[wv][i];
        p.part[(size_t)blockIdx.x * n + i] = sum;
    }
}

// ---- 3x3 variants with vertical register reuse (round 2).  The per-pixel kernels above issue 9 sixteen-byte loads, 64-bit
// index arithmetic and a bounds test per tap and pixel; at 352x704x32 that, not HBM, set the time (0.83 / 0.67 / 0.85 ms
// per K16 step against ~0.1 ms of traffic).  Here a lane group owns a COLUMN RUN of R pixels: the 3 x (R+2) input window
// is loaded once (2.4x fewer loads for R = 8), row validity is warp-uniform, the weights of the lane's 4 channels sit in
// registers, and R accumulators give the FMA pipe independent chains.
constexpr int RUN = 8;

struct RunIndex { int x, y0, b; bool live; };

template <int LPP>
__device__ __forceinline__ RunIndex run_index(const ThinParams &p, long long work, int slot) {
    constexpr int PPW = 32 / LPP;
    const int xgroups = (p.W + PPW - 1) / PPW, strips = (p.H + RUN - 1) / RUN;
    RunIndex r;
    const int xg = (int)(work % xgroups);
    const long long t = work / xgroups;
    r.x = xg * PPW + slot;
    r.y0 = (int)(t % strips) * RUN;
    r.b = (int)(t / strips);
    r.live = r.x < p.W;
    return r;
}

template <int LPP>
__global__ void __launch_bounds__(256) thin_fwd3(const ThinParams p) {
    __shared__ __align__(16) float sw[MAXTAPS * MAXC];
    load_w(p, sw);
    const int lane = threadIdx.x & 31;
    const int u = lane % LPP, slot = lane / LPP;
    constexpr int PPW = 32 / LPP;
    float4 w[9];
#pragma unroll
    for (int t = 0; t < 9; ++t) w[t] = *reinterpret_cast<const float4 *>(sw + t * p.C + 4 * u);
    const long long nwork = (long long)p.B * ((p.H + RUN - 1) / RUN) * ((p.W + PPW - 1) / PPW);
    const long long warp0 = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const long long nwarps = ((long long)gridDim.x * blockDim.x) >> 5;
    for (long long work = warp0; work < nwork; work += nwarps) {
        const RunIndex ri = run_index<LPP>(p, work, slot);
        float acc[RUN];
#pragma unroll
        for (int r = 0; r < RUN; ++r) acc[r] = 0.f;
        const float *base = p.x + ((long long)ri.b * p.H * p.W) * p.xs + 4 * u;
#pragma unroll
        for (int r = -1; r <= RUN; ++r) {                       // input row y0 + r feeds output rows r - ky + 1
            const int yy = ri.y0 + r;
            if ((unsigned)yy >= (unsigned)p.H) continue;        // warp-uniform
#pragma unroll
            for (int kx = 0; kx < 3; ++kx) {
                const int xx = ri.x + kx - 1;
                float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
                if (ri.live && (unsigned)xx < (unsigned)p.W)
                    v = __ldg(reinterpret_cast<const float4 *>(base + ((long long)yy * p.W + xx) * p.xs));
#pragma unroll
                for (int ky = 0; ky < 3; ++ky) {
                    const int ro = r - ky + 1;
                    if (ro >= 0 && ro < RUN) {
                        const float4 wv = w[ky * 3 + kx];
                        float a = acc[ro];
                        a = fmaf(v.x, wv.x, a); a = fmaf(v.y, wv.y, a); a = fmaf(v.z, wv.z, a); a = fmaf(v.w, wv.w, a);
                        acc[ro] = a;
                    }
                }
            }
        }
#pragma unroll
        for (int r = 0; r < RUN; ++r) {
            float a = acc[r];
#pragma unroll
            for (int m = 1; m < LPP; m <<= 1) a += __shfl_xor_sync(0xffffffffu, a, m);
            if (u == 0 && ri.live && ri.y0 + r < p.H) {
                if (p.act == 2) a = 1.0f / (1.0f + expf(-a));
                p.y[((long long)ri.b * p.H + ri.y0 + r) * p.W + ri.x] = a;
            }
        }
    }
}

// the 3 x (RUN+2) window of effective upstream gradients around a column run: win[r + 1][kx] = g(y0 + r, x + kx - 1)
template <int LPP>
__device__ __forceinline__ void load_gwin(const ThinParams &p, const RunIndex &ri, float (&win)[RUN + 2][3]) {
#pragma unroll
    for (int r = -1; r <= RUN; ++r) {
        const int yy = ri.y0 + r;
#pragma unroll
        for (int kx = 0; kx < 3; ++kx) {
            const int xx = ri.x + kx - 1;
            float gv = 0.f;
            if (ri.live && (unsigned)yy < (unsigned)p.H && (unsigned)xx < (unsigned)p.W)
                gv = geff(p, (size_t)(((long long)ri.b * p.H + yy) * p.W + xx));
            win[r + 1][kx] = gv;
        }
    }
}

template <int LPP>
__global__ void __launch_bounds__(256) thin_dgrad3(const ThinParams p) {
    __shared__ __align__(16) float sw[MAXTAPS * MAXC];
    load_w(p, sw);
    const int lane = threadIdx.x & 31;
    const int u = lane % LPP, slot = lane / LPP;
    constexpr int PPW = 32 / LPP;
    float4 w[9];
#pragma unroll
    for (int t = 0; t < 9; ++t) w[t] = *reinterpret_cast<const float4 *>(sw + t * p.C + 4 * u);
    const long long nwork = (long long)p.B * ((p.H + RUN - 1) / RUN) * ((p.W + PPW - 1) / PPW);
    const long long warp0 = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const long long nwarps = ((long long)gridDim.x * blockDim.x) >> 5;
    for (long long work = warp0; work < nwork; work += nwarps) {
        const RunIndex ri = run_index<LPP>(p, work, slot);
        float win[RUN + 2][3];
        load_gwin<LPP>(p, ri, win);
#pragma unroll
        for (int r = 0; r < RUN; ++r) {
            // dx[y][x] = sum_tap g[y - (ky - 1)][x - (kx - 1)] * w[tap]
            float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
            for (int ky = 0; ky < 3; ++ky)
#pragma unroll
                for (int kx = 0; kx < 3; ++kx) {
                    const float gv = win[r - (ky - 1) + 1][2 - kx];
                    const float4 wv = w[ky * 3 + kx];
                    acc.x = fmaf(gv, wv.x, acc.x); acc.y = fmaf(gv, wv.y, acc.y);
                    acc.z = fmaf(gv, wv.z, acc.z); acc.w = fmaf(gv, wv.w, acc.w);
                }
            if (ri.live && ri.y0 + r < p.H)
                *(reinterpret_cast<float4 *>(p.dx + (((long long)ri.b * p.H + ri.y0 + r) * p.W + ri.x) * p.dxs) + u) = acc;
        }
    }
}

template <int LPP>
__global__ void __launch_bounds__(256) thin_wgrad3(const ThinParams p) {
    constexpr int TAPS = 9;
    constexpr int PPW = 32 / LPP;
    __shared__ float red[8][TAPS * 4 * LPP];            // per-warp results: [tap][channel]
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int u = lane % LPP, slot = lane / LPP;
    const long long nwork = (long long)p.B * ((p.H + RUN - 1) / RUN) * ((p.W + PPW - 1) / PPW);
    const long long warp0 = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const long long nwarps = ((long long)gridDim.x * blockDim.x) >> 5;
    float4 acc[TAPS];
#pragma unroll
    for (int t = 0; t < TAPS; ++t) acc[t] = make_float4(0.f, 0.f, 0.f, 0.f);
    for (long long work = warp0; work < nwork; work += nwarps) {
        const RunIndex ri = run_index<LPP>(p, work, slot);
        float win[RUN + 2][3];
        load_gwin<LPP>(p, ri, win);
        const float *base = p.x + ((long long)ri.b * p.H * p.W) * p.xs + 4 * u;
#pragma unroll
        for (int r = 0; r < RUN; ++r) {
            // dw[tap] += x[q] * g[q - off(tap)],  q = (y0 + r, x): each input pixel is read once
            float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
            if (ri.live && ri.y0 + r < p.H)
                v = __ldg(reinterpret_cast<const float4 *>(base + ((long long)(ri.y0 + r) * p.W + ri.x) * p.xs));
#pragma unroll
            for (int ky = 0; ky < 3; ++ky)
#pragma unroll
                for (int kx = 0; kx < 3; ++kx) {
                    const float gv = win[r - (ky - 1) + 1][2 - kx];
                    float4 &a = acc[ky * 3 + kx];
                    a.x = fmaf(gv, v.x, a.x); a.y = fmaf(gv, v.y, a.y);
                    a.z = fmaf(gv, v.z, a.z); a.w = fmaf(gv, v.w, a.w);
                }
        }
    }
#pragma unroll
    for (int t = 0; t < TAPS; ++t) {
#pragma unroll
        for (int m = LPP; m < 32; m <<= 1) {
            acc[t].x += __shfl_xor_sync(0xffffffffu, acc[t].x, m);
            acc[t].y += __shfl_xor_sync(0xffffffffu, acc[t].y, m);
            acc[t].z += __shfl_xor_sync(0xffffffffu, acc[t].z, m);
            acc[t].w += __shfl_xor_sync(0xffffffffu, acc[t].w, m);
        }
        if (slot == 0) {
            float *r = &red[warp][t * 4 * LPP + 4 * u];
            r[0] = acc[t].x; r[1] = acc[t].y; r[2] = acc[t].z; r[3] = acc[t].w;
        }
    }
    __syncthreads();
    const int n = TAPS * 4 * LPP;
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
        float sum = 0.f;
#pragma unroll
        for (int wv = 0; wv < 8; ++wv) sum += red[wv][i];
        p.part[(size_t)blockIdx.x * n + i] = sum;
    }
}

__global__ void thin_wgrad_reduce(const float *__restrict__ part, int nblocks, int C, int K, float *__restrict__ dw,
                                  long long s_ci, long long s_kh, long long s_kw) {
    const int n = K * K * C;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        float sum = 0.f;
        for (int b = 0; b < nblocks; ++b) sum += part[(size_t)b * n + i];
        const int tap = i / C, c = i - tap * C;
        dw[c * s_ci + (tap / K) * s_kh + (tap % K) * s_kw] = sum;
    }
}

int lpp_of(int C) { return (C == 8 || C == 16 || C == 32 || C == 64 || C == 128) ? C / 4 : 0; }

int grid_for(long long npix, int lpp) {
    const long long groups = (npix + (32 / lpp) - 1) / (32 / lpp);
    long long blocks = (groups + 7) / 8;
    const long long cap = (long long)bts_num_sms() * 8;
    if (blocks > cap) blocks = cap;
    if (blocks < 1) blocks = 1;
    return (int)blocks;
}

int grid_for_runs(int B, int H, int W, int lpp) {
    const int ppw = 32 / lpp;
    const long long work = (long long)B * ((H + RUN - 1) / RUN) * ((W + ppw - 1) / ppw);
    long long blocks = (work + 7) / 8;
    const long long cap = (long long)bts_num_sms() * 8;
    if (blocks > cap) blocks = cap;
    if (blocks < 1) blocks = 1;
    return (int)blocks;
}

int check(const float *x, long long xs, int B, int H, int W, int C, int K) {
    if (!x || B < 0 || H < 1 || W < 1 || (K != 1 && K != 3) || !lpp_of(C)) return BTS_EINVAL;
    if (!bts_aligned16(x) || (xs % 4) != 0) return BTS_EALIGN;
    return 0;
}

}  // namespace

#define BTS_THIN_DISPATCH(KERNEL, ...)                         \
    switch (lpp_of(C)) {                                       \
        case 2: KERNEL<2> __VA_ARGS__; break;                  \
        case 4: KERNEL<4> __VA_ARGS__; break;                  \
        case 8: KERNEL<8> __VA_ARGS__; break;                  \
        case 16: KERNEL<16> __VA_ARGS__; break;                \
        default: KERNEL<32> __VA_ARGS__; break;                \
    }

extern "C" int bts_conv_c1_workspace_floats(int C, int K) { return bts_num_sms() * 8 * K * K * C; }

extern "C" int bts_conv_c1_fwd(const float *x, long long x_pixel_stride, int B, int H, int W, int C, int K,
                               const float *w, long long s_ci, long long s_kh, long long s_kw, int act, float *y,
                               void *stream) {
    int rc = check(x, x_pixel_stride, B, H, W, C, K);
    if (rc) return rc;
    if (!w || !y || (act != 0 && act != 2)) return BTS_EINVAL;
    if (B == 0) return 0;
    ThinParams p{};
    p.x = x; p.xs = x_pixel_stride; p.B = B; p.H = H; p.W = W; p.C = C; p.K = K;
    p.w = w; p.s_ci = s_ci; p.s_kh = s_kh; p.s_kw = s_kw; p.y = y; p.act = act;
    cudaStream_t st = (cudaStream_t)stream;
    if (K == 3 && C <= 64 && H >= RUN) {
        const int grid3 = grid_for_runs(B, H, W, lpp_of(C));
        BTS_THIN_DISPATCH(thin_fwd3, <<<grid3, 256, 0, st>>>(p))
        BTS_LAUNCH_CHECK();
        return 0;
    }
    const int grid = grid_for((long long)B * H * W, lpp_of(C));
    BTS_THIN_DISPATCH(thin_fwd, <<<grid, 256, 0, st>>>(p))
    BTS_LAUNCH_CHECK();
    return 0;
}

extern "C" int bts_conv_c1_dgrad(const float *dy, const float *sig, int B, int H, int W, int C, int K, const float *w,
                                 long long s_ci, long long s_kh, long long s_kw, float *dx, long long dx_pixel_stride,
                                 void *stream) {
    if (!dy || !w || !dx || B < 0 || H < 1 || W < 1 || (K != 1 && K != 3) || !lpp_of(C)) return BTS_EINVAL;
    if (!bts_aligned16(dx) || (dx_pixel_stride % 4) != 0) return BTS_EALIGN;
    if (B == 0) return 0;
    ThinParams p{};
    p.B = B; p.H = H; p.W = W; p.C = C; p.K = K; p.w = w; p.s_ci = s_ci; p.s_kh = s_kh; p.s_kw = s_kw;
    p.dy = dy; p.s = sig; p.dx = dx; p.dxs = dx_pixel_stride;
    cudaStream_t st = (cudaStream_t)stream;
    if (K == 3 && C <= 64 && H >= RUN) {
        const int grid3 = grid_for_runs(B, H, W, lpp_of(C));
        BTS_THIN_DISPATCH(thin_dgrad3, <<<grid3, 256, 0, st>>>(p))
        BTS_LAUNCH_CHECK();
        return 0;
    }
    const int grid = grid_for((long long)B * H * W, lpp_of(C));
    BTS_THIN_DISPATCH(thin_dgrad, <<<grid, 256, 0, st>>>(p))
    BTS_LAUNCH_CHECK();
    return 0;
}

extern "C" int bts_conv_c1_wgrad(const float *x, long long x_pixel_stride, const float *dy, const float *sig, int B,
                                 int H, int W, int C, int K, float *workspace, float *dw, long long s_ci,
                                 long long s_kh, long long s_kw, void *stream) {
    int rc = check(x, x_pixel_stride, B, H, W, C, K);
    if (rc) return rc;
    if (!dy || !workspace || !dw || B < 1) return BTS_EINVAL;
    ThinParams p{};
    p.x = x; p.xs = x_pixel_stride; p.B = B; p.H = H; p.W = W; p.C = C; p.K = K;
    p.dy = dy; p.s = sig; p.part = workspace;
    const int lpp = lpp_of(C);
    const bool runs = K == 3 && C <= 64 && H >= RUN;
    const int grid = runs ? grid_for_runs(B, H, W, lpp) : grid_for((long long)B * H * W, lpp);
    cudaStream_t st = (cudaStream_t)stream;
#define BTS_WG(L)                                                             \
    if (K == 1) thin_wgrad<L, 1><<<grid, 256, 0, st>>>(p);                    \
    else if (runs) thin_wgrad3<L><<<grid, 256, 0, st>>>(p);                   \
    else thin_wgrad<L, 3><<<grid, 256, 0, st>>>(p);
    switch (lpp) {
        case 2: BTS_WG(2) break;
        case 4: BTS_WG(4) break;
        case 8: BTS_WG(8) break;
        case 16: BTS_WG(16) break;
        default: BTS_WG(32) break;
    }
#undef BTS_WG
    BTS_LAUNCH_CHECK();
    thin_wgrad_reduce<<<(K * K * C + 127) / 128, 128, 0, st>>>(workspace, grid, C, K, dw, s_ci, s_kh, s_kw);
    BTS_LAUNCH_CHECK();
    return 0;
}
