// Depthwise 3x3 convolution of the MobileNetV2 inverted-residual blocks (torchvision mobilenet_v2 `features[1..17]`,
// the `mobilenetv2_bts` encoder of reference pytorch/bts.py:297-300), NHWC fp32, pad 1, stride 1 or 2, C % 4 == 0, on
// CUDA cores.  The layer does 9 FMAs per output element, so it is bound by HBM, not by arithmetic.
//
// Tiling (forward and wgrad).  A 256-thread CTA owns 32 channels (8 quads of 16 bytes) and a TH x TW output tile.  Each
// thread owns one channel quad and RW consecutive outputs of one tile row.  The input window of the tile, with its halo,
// is staged once in shared memory as 16-byte NHWC granules: 8 adjacent threads read the 128 contiguous bytes of a
// pixel's channel group.  Granules outside the image are zero.  The optional BatchNorm + ReLU6 prologue is applied
// while staging, so once per input element and not once per tap read.  The padding stays zero after the prologue,
// because the reference pads the activated tensor.  Each thread keeps its 9 x 4 weights in registers and loads one
// window row of (RW-1)*S+3 columns per kernel row, so every column it loads serves several outputs.
//
// Determinism.  A CTA walks a fixed set of tiles (tile = slice + k * nslices, at most DW_MAX_TILES of them).  Per-thread
// fp32 runs over those tiles are combined across the CTA's threads in fp64 in a fixed order.  The per-CTA partials go to
// the caller's workspace, and a second kernel sums them in a fixed order.  The forward's BatchNorm statistics and the
// wgrad both work this way, so the results are bit-reproducible.
#include "common.cuh"

namespace {

constexpr int DW_CQ = 8;                  // channel quads per CTA
constexpr int DW_NW = 32;                 // pixel workers per CTA
constexpr int DW_NT = DW_CQ * DW_NW;      // threads per CTA
constexpr int DW_MAX_TILES = 32;          // tiles per CTA at most: bounds the fp32 runs of the partial sums

template <int S>
struct DwTile;
template <>
struct DwTile<1> {
    static constexpr int TH = 8, SEG = 4, RW = 4;   // 8 rows x 4 segments of 4 outputs: a 8 x 16 tile
};
template <>
struct DwTile<2> {
    static constexpr int TH = 4, SEG = 8, RW = 2;   // 4 rows x 8 segments of 2 outputs: a 4 x 16 tile
};

template <int S>
struct DwGeom {
    static constexpr int TH = DwTile<S>::TH, SEG = DwTile<S>::SEG, RW = DwTile<S>::RW, TW = SEG * RW;
    static constexpr int IH = (TH - 1) * S + 3, IW = (TW - 1) * S + 3;   // staged window with its halo
    static constexpr int RC = (RW - 1) * S + 3;                           // window columns one thread reads per row
};

struct DwShape {
    int B, H, W, C, Ho, Wo, tiles_y, tiles_x;
    long long ntiles;
};

__device__ __forceinline__ float relu6f(float v) { return fminf(fmaxf(v, 0.f), 6.f); }

__device__ __forceinline__ float4 fma4(float4 a, float4 b, float4 c) {
    return make_float4(fmaf(a.x, b.x, c.x), fmaf(a.y, b.y, c.y), fmaf(a.z, b.z, c.z), fmaf(a.w, b.w, c.w));
}

__device__ __forceinline__ float4 affine_relu6(float4 v, float4 s, float4 h) {
    return make_float4(relu6f(fmaf(v.x, s.x, h.x)), relu6f(fmaf(v.y, s.y, h.y)), relu6f(fmaf(v.z, s.z, h.z)),
                       relu6f(fmaf(v.w, s.w, h.w)));
}

__device__ __forceinline__ float4 load_quad(const float *__restrict__ p, int c, long long sc) {
    return make_float4(__ldg(p + (long long)c * sc), __ldg(p + (long long)(c + 1) * sc), __ldg(p + (long long)(c + 2) * sc),
                       __ldg(p + (long long)(c + 3) * sc));
}

// stages the (IH x IW) window whose top-left input pixel is (iy0, ix0) for channels [c0, c0 + 32), applying the prologue
template <int S, bool PRE>
__device__ __forceinline__ void dw_stage(float4 *sm, const float *__restrict__ x, long long xs, const DwShape &d, int b, int iy0,
                                         int ix0, int c0, float4 psc, float4 psh) {
    using G = DwGeom<S>;
    const int q = threadIdx.x % DW_CQ;
    const int c = c0 + 4 * q;
    for (int p = threadIdx.x / DW_CQ; p < G::IH * G::IW; p += DW_NW) {
        const int iy = iy0 + p / G::IW, ix = ix0 + p % G::IW;
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (c < d.C && iy >= 0 && iy < d.H && ix >= 0 && ix < d.W) {
            v = __ldg(reinterpret_cast<const float4 *>(x + (((long long)b * d.H + iy) * d.W + ix) * xs + c));
            if (PRE) v = affine_relu6(v, psc, psh);
        }
        sm[p * DW_CQ + q] = v;
    }
}

__device__ __forceinline__ void tile_origin(const DwShape &d, long long tile, int TH, int TW, int &b, int &oy0, int &ox0) {
    const long long per_img = (long long)d.tiles_y * d.tiles_x;
    b = (int)(tile / per_img);
    const int r = (int)(tile - (long long)b * per_img);
    oy0 = (r / d.tiles_x) * TH;
    ox0 = (r % d.tiles_x) * TW;
}

// y = dw(pre(x)) [-> relu6(y*post_scale + post_shift)];  part[slice][0:C] / [C:2C] = fp64 (sum, sum of squares) of y
template <int S, bool PRE>
__global__ void __launch_bounds__(DW_NT) dw3x3_fwd_kernel(const float *__restrict__ x, long long xs, const DwShape d,
                                                          const float *__restrict__ w, long long s_c, long long s_kh,
                                                          long long s_kw, const float *__restrict__ pre_scale,
                                                          const float *__restrict__ pre_shift,
                                                          const float *__restrict__ post_scale,
                                                          const float *__restrict__ post_shift, float *__restrict__ y,
                                                          long long ys, double *__restrict__ part) {
    using G = DwGeom<S>;
    __shared__ float4 sm[G::IH * G::IW * DW_CQ];
    __shared__ float red[2][DW_NW][DW_CQ * 4];
    const int q = threadIdx.x % DW_CQ, wk = threadIdx.x / DW_CQ;
    const int row = wk / G::SEG, seg = wk % G::SEG;
    const int c0 = blockIdx.y * DW_CQ * 4, c = c0 + 4 * q;
    const bool cok = c < d.C;
    float4 wr[9], psc = make_float4(0.f, 0.f, 0.f, 0.f), psh = psc, esc = psc, esh = psc;
#pragma unroll
    for (int t = 0; t < 9; ++t)
        wr[t] = cok ? load_quad(w + (t / 3) * s_kh + (t % 3) * s_kw, c, s_c) : make_float4(0.f, 0.f, 0.f, 0.f);
    if (PRE && cok) {
        psc = __ldg(reinterpret_cast<const float4 *>(pre_scale + c));
        psh = __ldg(reinterpret_cast<const float4 *>(pre_shift + c));
    }
    if (post_scale && cok) {
        esc = __ldg(reinterpret_cast<const float4 *>(post_scale + c));
        esh = __ldg(reinterpret_cast<const float4 *>(post_shift + c));
    }
    float4 s1 = make_float4(0.f, 0.f, 0.f, 0.f), s2 = s1;
    for (long long tile = blockIdx.x; tile < d.ntiles; tile += gridDim.x) {
        int b, oy0, ox0;
        tile_origin(d, tile, G::TH, G::TW, b, oy0, ox0);
        __syncthreads();                                   // the previous tile's window is no longer read
        dw_stage<S, PRE>(sm, x, xs, d, b, oy0 * S - 1, ox0 * S - 1, c0, psc, psh);
        __syncthreads();
        float4 acc[G::RW];
#pragma unroll
        for (int j = 0; j < G::RW; ++j) acc[j] = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
        for (int kh = 0; kh < 3; ++kh) {
            const float4 *src = sm + ((row * S + kh) * G::IW + seg * G::RW * S) * DW_CQ + q;
            float4 in[G::RC];
#pragma unroll
            for (int k = 0; k < G::RC; ++k) in[k] = src[k * DW_CQ];
#pragma unroll
            for (int j = 0; j < G::RW; ++j)
#pragma unroll
                for (int kw = 0; kw < 3; ++kw) acc[j] = fma4(in[j * S + kw], wr[kh * 3 + kw], acc[j]);
        }
        const int oy = oy0 + row;
        if (cok && oy < d.Ho) {
#pragma unroll
            for (int j = 0; j < G::RW; ++j) {
                const int ox = ox0 + seg * G::RW + j;
                if (ox < d.Wo) {
                    float4 v = acc[j];
                    if (part) {
                        s1.x += v.x; s1.y += v.y; s1.z += v.z; s1.w += v.w;
                        s2 = fma4(v, v, s2);
                    }
                    if (post_scale) v = affine_relu6(v, esc, esh);
                    *reinterpret_cast<float4 *>(y + (((long long)b * d.Ho + oy) * d.Wo + ox) * ys + c) = v;
                }
            }
        }
    }
    if (!part) return;
    *reinterpret_cast<float4 *>(&red[0][wk][4 * q]) = s1;
    *reinterpret_cast<float4 *>(&red[1][wk][4 * q]) = s2;
    __syncthreads();
    if (threadIdx.x < DW_CQ * 4 && c0 + (int)threadIdx.x < d.C) {
        double a = 0.0, a2 = 0.0;
        for (int k = 0; k < DW_NW; ++k) {
            a += (double)red[0][k][threadIdx.x];
            a2 += (double)red[1][k][threadIdx.x];
        }
        double *o = part + (long long)blockIdx.x * 2 * d.C + c0 + threadIdx.x;
        o[0] = a;
        o[d.C] = a2;
    }
}

// dW partials: part[slice][c][tap] = sum over the slice's tiles of dy[o, c] * pre(x)[o*S + tap - 1, c]
template <int S, bool PRE>
__global__ void __launch_bounds__(DW_NT) dw3x3_wgrad_kernel(const float *__restrict__ x, long long xs,
                                                            const float *__restrict__ dy, long long dys, const DwShape d,
                                                            const float *__restrict__ pre_scale,
                                                            const float *__restrict__ pre_shift, double *__restrict__ part) {
    using G = DwGeom<S>;
    __shared__ float4 sm[G::IH * G::IW * DW_CQ];
    __shared__ float red[DW_NW][DW_CQ * 4];
    const int q = threadIdx.x % DW_CQ, wk = threadIdx.x / DW_CQ;
    const int row = wk / G::SEG, seg = wk % G::SEG;
    const int c0 = blockIdx.y * DW_CQ * 4, c = c0 + 4 * q;
    const bool cok = c < d.C;
    float4 psc = make_float4(0.f, 0.f, 0.f, 0.f), psh = psc;
    if (PRE && cok) {
        psc = __ldg(reinterpret_cast<const float4 *>(pre_scale + c));
        psh = __ldg(reinterpret_cast<const float4 *>(pre_shift + c));
    }
    float4 acc[9];
#pragma unroll
    for (int t = 0; t < 9; ++t) acc[t] = make_float4(0.f, 0.f, 0.f, 0.f);
    for (long long tile = blockIdx.x; tile < d.ntiles; tile += gridDim.x) {
        int b, oy0, ox0;
        tile_origin(d, tile, G::TH, G::TW, b, oy0, ox0);
        __syncthreads();
        dw_stage<S, PRE>(sm, x, xs, d, b, oy0 * S - 1, ox0 * S - 1, c0, psc, psh);
        float4 g[G::RW];
        const int oy = oy0 + row;
#pragma unroll
        for (int j = 0; j < G::RW; ++j) {
            const int ox = ox0 + seg * G::RW + j;
            g[j] = (cok && oy < d.Ho && ox < d.Wo)
                       ? __ldg(reinterpret_cast<const float4 *>(dy + (((long long)b * d.Ho + oy) * d.Wo + ox) * dys + c))
                       : make_float4(0.f, 0.f, 0.f, 0.f);
        }
        __syncthreads();
#pragma unroll
        for (int kh = 0; kh < 3; ++kh) {
            const float4 *src = sm + ((row * S + kh) * G::IW + seg * G::RW * S) * DW_CQ + q;
            float4 in[G::RC];
#pragma unroll
            for (int k = 0; k < G::RC; ++k) in[k] = src[k * DW_CQ];
#pragma unroll
            for (int kw = 0; kw < 3; ++kw)
#pragma unroll
                for (int j = 0; j < G::RW; ++j) acc[kh * 3 + kw] = fma4(g[j], in[j * S + kw], acc[kh * 3 + kw]);
        }
    }
    // threads -> fp64 per (channel, tap) in a fixed order, one tap at a time through `red`
#pragma unroll
    for (int t = 0; t < 9; ++t) {
        __syncthreads();
        *reinterpret_cast<float4 *>(&red[wk][4 * q]) = acc[t];
        __syncthreads();
        if (threadIdx.x < DW_CQ * 4 && c0 + (int)threadIdx.x < d.C) {
            double a = 0.0;
            for (int k = 0; k < DW_NW; ++k) a += (double)red[k][threadIdx.x];
            part[((long long)blockIdx.x * d.C + c0 + threadIdx.x) * 9 + t] = a;
        }
    }
}

// stride-2 dgrad: dx[i] = sum over the taps that land, dy[(i + 1 - tap) / 2] * w[tap] -- no zero-stuffed dy
__global__ void __launch_bounds__(DW_NT) dw3x3_dgrad_s2_kernel(const float *__restrict__ dy, long long dys, const DwShape d,
                                                               const float *__restrict__ w, long long s_c, long long s_kh,
                                                               long long s_kw, float *__restrict__ dx, long long dxs) {
    const int q = threadIdx.x % DW_CQ, wk = threadIdx.x / DW_CQ;
    const int c = blockIdx.y * DW_CQ * 4 + 4 * q;
    if (c >= d.C) return;
    float4 wr[9];
#pragma unroll
    for (int t = 0; t < 9; ++t) wr[t] = load_quad(w + (t / 3) * s_kh + (t % 3) * s_kw, c, s_c);
    const long long npix = (long long)d.B * d.H * d.W;
    for (long long p = (long long)blockIdx.x * DW_NW + wk; p < npix; p += (long long)gridDim.x * DW_NW) {
        const int ix = (int)(p % d.W);
        const long long t2 = p / d.W;
        const int iy = (int)(t2 % d.H), b = (int)(t2 / d.H);
        float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
        // tap kh lands when iy + 1 - kh is even: kh = 1 for even iy, kh in {0, 2} for odd iy (likewise kw)
#pragma unroll
        for (int kh = 0; kh < 3; ++kh) {
            const int ty = iy + 1 - kh;
            if ((ty & 1) || ty < 0 || (ty >> 1) >= d.Ho) continue;
#pragma unroll
            for (int kw = 0; kw < 3; ++kw) {
                const int tx = ix + 1 - kw;
                if ((tx & 1) || tx < 0 || (tx >> 1) >= d.Wo) continue;
                const float4 g = __ldg(
                    reinterpret_cast<const float4 *>(dy + (((long long)b * d.Ho + (ty >> 1)) * d.Wo + (tx >> 1)) * dys + c));
                acc = fma4(g, wr[kh * 3 + kw], acc);
            }
        }
        *reinterpret_cast<float4 *>(dx + p * dxs + c) = acc;
    }
}

// second pass: column sums of part[rows][cols] in a fixed order.  A block covers 32 columns with 8 row slices; slice k
// adds rows k, k+8, ... and the slices are added in order.  MODE 0: statistics (cols = 2C -> sum | sumsq);
// MODE 1: wgrad (cols = 9C, column c*9 + tap -> dw[c*s_c + kh*s_kh + kw*s_kw]).
template <int MODE>
__global__ void __launch_bounds__(256) dw_colsum_kernel(const double *__restrict__ part, int rows, int cols, int C,
                                                        double *__restrict__ sum, double *__restrict__ sumsq,
                                                        float *__restrict__ dw, long long s_c, long long s_kh, long long s_kw) {
    __shared__ double red[8][32];
    const int lc = threadIdx.x % 32, sl = threadIdx.x / 32;
    const int col = blockIdx.x * 32 + lc;
    double a = 0.0;
    if (col < cols)
        for (int r = sl; r < rows; r += 8) a += part[(long long)r * cols + col];
    red[sl][lc] = a;
    __syncthreads();
    if (sl != 0 || col >= cols) return;
    double t = 0.0;
#pragma unroll
    for (int k = 0; k < 8; ++k) t += red[k][lc];
    if (MODE == 0) {
        if (col < C) sum[col] = t;
        else sumsq[col - C] = t;
    } else {
        const int c = col / 9, tap = col % 9;
        dw[(long long)c * s_c + (tap / 3) * s_kh + (tap % 3) * s_kw] = (float)t;
    }
}

template <int S>
DwShape dw_shape(int B, int H, int W, int C) {
    using G = DwGeom<S>;
    DwShape d;
    d.B = B; d.H = H; d.W = W; d.C = C;
    d.Ho = (H - 1) / S + 1;
    d.Wo = (W - 1) / S + 1;
    d.tiles_y = bts_ceil_div(d.Ho, G::TH);
    d.tiles_x = bts_ceil_div(d.Wo, G::TW);
    d.ntiles = (long long)B * d.tiles_y * d.tiles_x;
    return d;
}

DwShape dw_shape_s(int stride, int B, int H, int W, int C) {
    return stride == 1 ? dw_shape<1>(B, H, W, C) : dw_shape<2>(B, H, W, C);
}

int dw_cgroups(int C) { return bts_ceil_div(C, DW_CQ * 4); }

// CTAs along the tile axis: enough for ~8 CTAs per SM over all channel groups, and at most DW_MAX_TILES tiles each
long long dw_slices(const DwShape &d) {
    long long n = ((long long)bts_num_sms() * 8 + dw_cgroups(d.C) - 1) / dw_cgroups(d.C);
    const long long lo = (d.ntiles + DW_MAX_TILES - 1) / DW_MAX_TILES;
    if (n < lo) n = lo;
    if (n > d.ntiles) n = d.ntiles;
    return n;
}

bool dw_args_ok(int B, int H, int W, int C, int stride) {
    return B >= 1 && H >= 1 && W >= 1 && C >= 4 && C % 4 == 0 && (stride == 1 || stride == 2);
}

bool quad_ok(const void *p, long long pixel_stride) { return p && bts_aligned16(p) && pixel_stride % 4 == 0 && pixel_stride > 0; }

template <int S, bool PRE>
int launch_fwd(const float *x, long long xs, const DwShape &d, const float *w, long long s_c, long long s_kh, long long s_kw,
               const float *pre_scale, const float *pre_shift, const float *post_scale, const float *post_shift, float *y,
               long long ys, double *part, long long nslices, cudaStream_t st) {
    dim3 grid((unsigned)nslices, (unsigned)dw_cgroups(d.C));
    dw3x3_fwd_kernel<S, PRE><<<grid, DW_NT, 0, st>>>(x, xs, d, w, s_c, s_kh, s_kw, pre_scale, pre_shift, post_scale, post_shift, y,
                                                     ys, part);
    BTS_LAUNCH_CHECK();
    return 0;
}

int fwd_dispatch(const float *x, long long xs, const DwShape &d, int stride, const float *w, long long s_c, long long s_kh,
                 long long s_kw, const float *pre_scale, const float *pre_shift, const float *post_scale, const float *post_shift,
                 float *y, long long ys, double *part, long long nslices, cudaStream_t st) {
    const bool pre = pre_scale != nullptr;
    if (stride == 1)
        return pre ? launch_fwd<1, true>(x, xs, d, w, s_c, s_kh, s_kw, pre_scale, pre_shift, post_scale, post_shift, y, ys, part,
                                         nslices, st)
                   : launch_fwd<1, false>(x, xs, d, w, s_c, s_kh, s_kw, pre_scale, pre_shift, post_scale, post_shift, y, ys, part,
                                          nslices, st);
    return pre ? launch_fwd<2, true>(x, xs, d, w, s_c, s_kh, s_kw, pre_scale, pre_shift, post_scale, post_shift, y, ys, part,
                                     nslices, st)
               : launch_fwd<2, false>(x, xs, d, w, s_c, s_kh, s_kw, pre_scale, pre_shift, post_scale, post_shift, y, ys, part,
                                      nslices, st);
}

}  // namespace

extern "C" long long bts_dw3x3_fwd_workspace_floats(int B, int H, int W, int C, int stride) {
    if (!dw_args_ok(B, H, W, C, stride)) return BTS_EINVAL;
    return 2LL * dw_slices(dw_shape_s(stride, B, H, W, C)) * 2 * C;
}

extern "C" int bts_dw3x3_fwd(const float *x, long long x_pixel_stride, int B, int H, int W, int C, int stride, const float *w,
                             long long s_c, long long s_kh, long long s_kw, const float *pre_scale, const float *pre_shift,
                             const float *post_scale, const float *post_shift, float *y, long long y_pixel_stride,
                             double *stat_sum, double *stat_sumsq, float *workspace, void *stream) {
    if (!dw_args_ok(B, H, W, C, stride) || !w || !quad_ok(x, x_pixel_stride) || !quad_ok(y, y_pixel_stride)) return BTS_EINVAL;
    if ((pre_scale == nullptr) != (pre_shift == nullptr) || (post_scale == nullptr) != (post_shift == nullptr)) return BTS_EINVAL;
    if ((pre_scale && (!bts_aligned16(pre_scale) || !bts_aligned16(pre_shift))) ||
        (post_scale && (!bts_aligned16(post_scale) || !bts_aligned16(post_shift))))
        return BTS_EINVAL;
    const bool stats = stat_sum != nullptr;
    if (stats != (stat_sumsq != nullptr) || (stats && (!workspace || post_scale))) return BTS_EINVAL;
    const DwShape d = dw_shape_s(stride, B, H, W, C);
    const long long ns = dw_slices(d);
    cudaStream_t st = (cudaStream_t)stream;
    double *part = stats ? reinterpret_cast<double *>(workspace) : nullptr;
    if (stats && (((uintptr_t)part) & 7)) return BTS_EINVAL;
    int rc = fwd_dispatch(x, x_pixel_stride, d, stride, w, s_c, s_kh, s_kw, pre_scale, pre_shift, post_scale, post_shift, y,
                          y_pixel_stride, part, ns, st);
    if (rc || !stats) return rc;
    dw_colsum_kernel<0><<<bts_ceil_div(2 * C, 32), 256, 0, st>>>(part, (int)ns, 2 * C, C, stat_sum, stat_sumsq, nullptr, 0, 0, 0);
    BTS_LAUNCH_CHECK();
    return 0;
}

extern "C" int bts_dw3x3_dgrad(const float *dy, long long dy_pixel_stride, int B, int H, int W, int C, int stride, const float *w,
                               long long s_c, long long s_kh, long long s_kw, float *dx, long long dx_pixel_stride, void *stream) {
    if (!dw_args_ok(B, H, W, C, stride) || !w || !quad_ok(dy, dy_pixel_stride) || !quad_ok(dx, dx_pixel_stride)) return BTS_EINVAL;
    cudaStream_t st = (cudaStream_t)stream;
    if (stride == 1) {
        // the forward over flipped taps: w'[kh][kw] = w[2-kh][2-kw], read in place through negated strides
        const DwShape d = dw_shape<1>(B, H, W, C);
        return launch_fwd<1, false>(dy, dy_pixel_stride, d, w + 2 * s_kh + 2 * s_kw, s_c, -s_kh, -s_kw, nullptr, nullptr, nullptr,
                                    nullptr, dx, dx_pixel_stride, nullptr, dw_slices(d), st);
    }
    const DwShape d = dw_shape<2>(B, H, W, C);
    long long blocks = ((long long)B * H * W + DW_NW - 1) / DW_NW;
    const long long cap = ((long long)bts_num_sms() * 8 + dw_cgroups(C) - 1) / dw_cgroups(C);
    if (blocks > cap) blocks = cap;
    dw3x3_dgrad_s2_kernel<<<dim3((unsigned)blocks, (unsigned)dw_cgroups(C)), DW_NT, 0, st>>>(dy, dy_pixel_stride, d, w, s_c, s_kh,
                                                                                             s_kw, dx, dx_pixel_stride);
    BTS_LAUNCH_CHECK();
    return 0;
}

extern "C" long long bts_dw3x3_wgrad_workspace_floats(int B, int H, int W, int C, int stride) {
    if (!dw_args_ok(B, H, W, C, stride)) return BTS_EINVAL;
    return 2LL * dw_slices(dw_shape_s(stride, B, H, W, C)) * 9 * C;
}

extern "C" int bts_dw3x3_wgrad(const float *x, long long x_pixel_stride, const float *dy, long long dy_pixel_stride, int B, int H,
                               int W, int C, int stride, const float *pre_scale, const float *pre_shift, float *workspace,
                               float *dw, long long s_c, long long s_kh, long long s_kw, void *stream) {
    if (!dw_args_ok(B, H, W, C, stride) || !quad_ok(x, x_pixel_stride) || !quad_ok(dy, dy_pixel_stride) || !workspace || !dw)
        return BTS_EINVAL;
    if ((pre_scale == nullptr) != (pre_shift == nullptr)) return BTS_EINVAL;
    if (pre_scale && (!bts_aligned16(pre_scale) || !bts_aligned16(pre_shift))) return BTS_EINVAL;
    if (((uintptr_t)workspace) & 7) return BTS_EINVAL;
    const DwShape d = dw_shape_s(stride, B, H, W, C);
    const long long ns = dw_slices(d);
    double *part = reinterpret_cast<double *>(workspace);
    cudaStream_t st = (cudaStream_t)stream;
    dim3 grid((unsigned)ns, (unsigned)dw_cgroups(C));
    if (stride == 1) {
        if (pre_scale) dw3x3_wgrad_kernel<1, true><<<grid, DW_NT, 0, st>>>(x, x_pixel_stride, dy, dy_pixel_stride, d, pre_scale, pre_shift, part);
        else dw3x3_wgrad_kernel<1, false><<<grid, DW_NT, 0, st>>>(x, x_pixel_stride, dy, dy_pixel_stride, d, nullptr, nullptr, part);
    } else {
        if (pre_scale) dw3x3_wgrad_kernel<2, true><<<grid, DW_NT, 0, st>>>(x, x_pixel_stride, dy, dy_pixel_stride, d, pre_scale, pre_shift, part);
        else dw3x3_wgrad_kernel<2, false><<<grid, DW_NT, 0, st>>>(x, x_pixel_stride, dy, dy_pixel_stride, d, nullptr, nullptr, part);
    }
    BTS_LAUNCH_CHECK();
    dw_colsum_kernel<1><<<bts_ceil_div(9 * C, 32), 256, 0, st>>>(part, (int)ns, 9 * C, C, nullptr, nullptr, dw, s_c, s_kh, s_kw);
    BTS_LAUNCH_CHECK();
    return 0;
}
