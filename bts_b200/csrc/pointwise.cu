// Weight gradient of the narrow 1x1 convolutions of the reduction heads (reference pytorch/bts.py:83-108:
// reduc1x1 32->16->8 at full resolution, reduc2x2 64->32->16->8->3 at half resolution, ...) as an HBM-bound CUDA-core
// kernel, sm_90a.
//
//   dW[co, ci] = sum_p dY[p, co] * x[p, ci]            Cin in {8,16,32,64}, Cout <= 32, NHWC operands
//
// On the tensor-core wgrad these layers fill 32 (or 8) of the 128 rows and 16 (or 3) of the columns of a tile and still
// pay the full operand-staging pipeline, while the layer itself is HBM-bound.
// Here a lane owns one (or two) input channels of one pixel slot and keeps all Cout accumulators in registers:
// the x row of a pixel is one coalesced load, the dY row a broadcast load; pixel slots of a warp, warps of a block and
// blocks are combined in a fixed order (shuffles, shared memory, a second pass over per-block partials) -> deterministic.
#include "common.cuh"

namespace {

constexpr int PW_THREADS = 256;
constexpr int PW_MAXCO = 32;

struct PwParams {
    const float *x; long long xs;
    const float *dy; long long dys;
    long long M;
    int Cin, Cout;
    float *part;              // [gridDim.x][Cin][Cout]
};

// CL = lanes per pixel (min(Cin, 32)), R = channels per lane (Cin / CL), CO = Cout rounded up to a multiple of 4
template <int CL, int R, int CO>
__global__ void __launch_bounds__(PW_THREADS) pw_wgrad_kernel(const PwParams p) {
    constexpr int PP = 32 / CL;                            // pixel slots per warp iteration
    __shared__ float red[PW_THREADS / 64][CL * R * CO];     // <= 4 x 2048 floats = 32 KB
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int ci = lane % CL, slot = lane / CL;
    float acc[R][CO];
#pragma unroll
    for (int r = 0; r < R; ++r)
#pragma unroll
        for (int c = 0; c < CO; ++c) acc[r][c] = 0.f;
    const long long nwarps = (long long)gridDim.x * (PW_THREADS / 32);
    const long long w0 = (long long)blockIdx.x * (PW_THREADS / 32) + warp;
    const bool dvec = ((p.dys & 3) == 0) && ((((uintptr_t)p.dy) & 15) == 0) && (p.Cout % 4 == 0);
    for (long long pix = w0 * PP + slot; pix < p.M; pix += nwarps * PP) {
        float xv[R];
#pragma unroll
        for (int r = 0; r < R; ++r) xv[r] = __ldg(p.x + pix * p.xs + ci + r * CL);
        float g[CO];
        const float *drow = p.dy + pix * p.dys;
        if (dvec) {
#pragma unroll
            for (int c = 0; c < CO; c += 4) {
                if (c < p.Cout) {
                    const float4 q = __ldg(reinterpret_cast<const float4 *>(drow + c));
                    g[c] = q.x; g[c + 1] = q.y; g[c + 2] = q.z; g[c + 3] = q.w;
                } else {
                    g[c] = g[c + 1] = g[c + 2] = g[c + 3] = 0.f;
                }
            }
        } else {
#pragma unroll
            for (int c = 0; c < CO; ++c) g[c] = c < p.Cout ? __ldg(drow + c) : 0.f;
        }
#pragma unroll
        for (int r = 0; r < R; ++r)
#pragma unroll
            for (int c = 0; c < CO; ++c) acc[r][c] = fmaf(xv[r], g[c], acc[r][c]);
    }
    // pixel slots of the warp (lane bits above log2 CL), fixed butterfly order
#pragma unroll
    for (int m = CL; m < 32; m <<= 1)
#pragma unroll
        for (int r = 0; r < R; ++r)
#pragma unroll
            for (int c = 0; c < CO; ++c) acc[r][c] += __shfl_xor_sync(0xffffffffu, acc[r][c], m);
    // warps of the block: the upper four park their sums, the lower four add them to their own and park the result
    constexpr int HW = PW_THREADS / 64;
    if (slot == 0 && warp >= HW) {
#pragma unroll
        for (int r = 0; r < R; ++r)
#pragma unroll
            for (int c = 0; c < CO; ++c) red[warp - HW][(ci + r * CL) * CO + c] = acc[r][c];
    }
    __syncthreads();
    if (slot == 0 && warp < HW) {
#pragma unroll
        for (int r = 0; r < R; ++r)
#pragma unroll
            for (int c = 0; c < CO; ++c) red[warp][(ci + r * CL) * CO + c] += acc[r][c];
    }
    __syncthreads();
    const int n = CL * R * CO;
    for (int i = threadIdx.x; i < n; i += PW_THREADS) {
        float sum = 0.f;
#pragma unroll
        for (int wv = 0; wv < HW; ++wv) sum += red[wv][i];
        const int c = i % CO, cin = i / CO;
        if (c < p.Cout) p.part[((size_t)blockIdx.x * p.Cin + cin) * p.Cout + c] = sum;
    }
}

__global__ void pw_wgrad_reduce(const float *__restrict__ part, int nblocks, int Cin, int Cout, float *__restrict__ dw,
                                long long s_co, long long s_ci) {
    const int n = Cin * Cout;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        float sum = 0.f;
        for (int b = 0; b < nblocks; ++b) sum += part[(size_t)b * n + i];
        const int ci = i / Cout, co = i - ci * Cout;
        dw[co * s_co + ci * s_ci] = sum;
    }
}

int pw_grid() { return bts_num_sms() * 4; }

}  // namespace

extern "C" int bts_conv_pw_wgrad_eligible(int Cin, int Cout) {
    return (Cin == 8 || Cin == 16 || Cin == 32 || Cin == 64) && Cout >= 1 && Cout <= PW_MAXCO;
}

extern "C" long long bts_conv_pw_wgrad_workspace_floats(int Cin, int Cout) { return (long long)pw_grid() * Cin * Cout; }

extern "C" int bts_conv_pw_wgrad(const float *x, long long x_pixel_stride, const float *dy, long long dy_pixel_stride,
                                 long long M, int Cin, int Cout, float *workspace, float *dw, long long s_co,
                                 long long s_ci, void *stream) {
    if (!x || !dy || !workspace || !dw || M < 1 || !bts_conv_pw_wgrad_eligible(Cin, Cout)) return BTS_EINVAL;
    PwParams p;
    p.x = x; p.xs = x_pixel_stride; p.dy = dy; p.dys = dy_pixel_stride; p.M = M; p.Cin = Cin; p.Cout = Cout;
    p.part = workspace;
    const int grid = pw_grid();
    cudaStream_t st = (cudaStream_t)stream;
    const int co4 = (Cout + 3) / 4 * 4;
#define BTS_PW(CL, R)                                                                                   \
    switch (co4) {                                                                                      \
        case 4: pw_wgrad_kernel<CL, R, 4><<<grid, PW_THREADS, 0, st>>>(p); break;                       \
        case 8: pw_wgrad_kernel<CL, R, 8><<<grid, PW_THREADS, 0, st>>>(p); break;                       \
        case 12: case 16: pw_wgrad_kernel<CL, R, 16><<<grid, PW_THREADS, 0, st>>>(p); break;            \
        default: pw_wgrad_kernel<CL, R, 32><<<grid, PW_THREADS, 0, st>>>(p); break;                     \
    }
    switch (Cin) {
        case 8: BTS_PW(8, 1) break;
        case 16: BTS_PW(16, 1) break;
        case 32: BTS_PW(32, 1) break;
        default: BTS_PW(32, 2) break;
    }
#undef BTS_PW
    BTS_LAUNCH_CHECK();
    pw_wgrad_reduce<<<(Cin * Cout + 127) / 128, 128, 0, st>>>(workspace, grid, Cin, Cout, dw, s_co, s_ci);
    BTS_LAUNCH_CHECK();
    return 0;
}

// ------------------------------------------------------------------------------------------------------------------
// Forward / dgrad of the same narrow 1x1 layers.  These are HBM-bound (e.g. 32->16 at 352x704x16): on the tensor engine a
// 128x16 output tile leaves the MMA nearly idle while the full operand-staging pipeline still runs.  Here:
//   out[p, co] = act( sum_ci x[p, ci] * W[co, ci] )        dgrad: the same with W read transposed (x := dY)
// A thread owns one pixel and one group of 4 output channels (the groups of a pixel are adjacent lanes, so the x row of a
// pixel is a broadcast load and a warp writes 512 contiguous bytes); x sits in registers, the (transposed, zero-padded)
// weights in shared memory as float4 rows.  HBM-bound: 4*(Cin + Cout) bytes per pixel.
namespace {

constexpr int PWF_MAXCI = 64, PWF_MAXCO = 64;

struct PwfParams {
    const float *x; long long xs;
    long long M;
    const float *w; long long s_out, s_in;   // W[out, in] element strides (dgrad passes them swapped)
    int Cout, act;                            // act: 0 none, 1 ELU, 2 sigmoid
    float *out; long long os;
    int ncog, lg;                             // output-channel groups of 4 (padded to a power of two = 1 << lg)
};

template <int CIN>
__global__ void __launch_bounds__(256) pw_fwd_kernel(const PwfParams p) {
    __shared__ __align__(16) float sw[CIN * PWF_MAXCO];          // [ci][co padded to 4 << lg]
    const int cop = 4 << p.lg;
    for (int i = threadIdx.x; i < CIN * cop; i += blockDim.x) {
        const int ci = i / cop, co = i - ci * cop;
        sw[i] = co < p.Cout ? p.w[co * p.s_out + ci * p.s_in] : 0.f;
    }
    __syncthreads();
    const int cog = (int)threadIdx.x & ((1 << p.lg) - 1);
    const long long ppb = 256 >> p.lg;                            // pixels per block iteration
    const bool ovec = ((p.os & 3) == 0) && ((((uintptr_t)p.out) & 15) == 0) && ((p.Cout & 3) == 0);
    for (long long m = (long long)blockIdx.x * ppb + ((int)threadIdx.x >> p.lg); m < p.M; m += (long long)gridDim.x * ppb) {
        float xv[CIN];
        const float4 *xr = reinterpret_cast<const float4 *>(p.x + m * p.xs);
#pragma unroll
        for (int j = 0; j < CIN / 4; ++j) {
            const float4 v = __ldg(xr + j);
            xv[4 * j] = v.x; xv[4 * j + 1] = v.y; xv[4 * j + 2] = v.z; xv[4 * j + 3] = v.w;
        }
        if (cog >= p.ncog) continue;
        float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
        const float4 *wr = reinterpret_cast<const float4 *>(sw) + cog;
#pragma unroll
        for (int ci = 0; ci < CIN; ++ci) {
            const float4 wv = wr[ci << p.lg];
            acc.x = fmaf(xv[ci], wv.x, acc.x); acc.y = fmaf(xv[ci], wv.y, acc.y);
            acc.z = fmaf(xv[ci], wv.z, acc.z); acc.w = fmaf(xv[ci], wv.w, acc.w);
        }
        float r[4] = {acc.x, acc.y, acc.z, acc.w};
        if (p.act == 1) {
#pragma unroll
            for (int e = 0; e < 4; ++e) r[e] = r[e] > 0.f ? r[e] : expm1f(r[e]);
        } else if (p.act == 2) {
#pragma unroll
            for (int e = 0; e < 4; ++e) r[e] = 1.0f / (1.0f + expf(-r[e]));
        }
        float *o = p.out + m * p.os + cog * 4;
        if (ovec) {
            *reinterpret_cast<float4 *>(o) = make_float4(r[0], r[1], r[2], r[3]);
        } else {
#pragma unroll
            for (int e = 0; e < 4; ++e)
                if (cog * 4 + e < p.Cout) o[e] = r[e];
        }
    }
}

}  // namespace

extern "C" int bts_conv_pw_fwd_eligible(int Cin, int Cout) {
    return (Cin == 8 || Cin == 16 || Cin == 32 || Cin == 64) && Cout >= 1 && Cout <= PWF_MAXCO;
}

// x: [M pixels][Cin] with pixel stride; w: element strides of W[out, in] (for dgrad pass the conv weight's (s_ci, s_co));
// act: 0 none, 1 ELU, 2 sigmoid; out: [M][Cout] with pixel stride
extern "C" int bts_conv_pw_fwd(const float *x, long long x_pixel_stride, long long M, int Cin, const float *w, long long s_out,
                               long long s_in, int Cout, int act, float *out, long long out_pixel_stride, void *stream) {
    if (!x || !w || !out || M < 1 || !bts_conv_pw_fwd_eligible(Cin, Cout) || act < 0 || act > 2) return BTS_EINVAL;
    if (!bts_aligned16(x) || (x_pixel_stride & 3)) return BTS_EALIGN;
    PwfParams p;
    p.x = x; p.xs = x_pixel_stride; p.M = M; p.w = w; p.s_out = s_out; p.s_in = s_in; p.Cout = Cout; p.act = act;
    p.out = out; p.os = out_pixel_stride;
    p.ncog = (Cout + 3) / 4;
    p.lg = 0;
    while ((1 << p.lg) < p.ncog) ++p.lg;
    const long long ppb = 256 >> p.lg;
    long long grid = (M + ppb - 1) / ppb;
    const long long cap = (long long)bts_num_sms() * 8;
    if (grid > cap) grid = cap;
    cudaStream_t st = (cudaStream_t)stream;
    switch (Cin) {
        case 8: pw_fwd_kernel<8><<<(int)grid, 256, 0, st>>>(p); break;
        case 16: pw_fwd_kernel<16><<<(int)grid, 256, 0, st>>>(p); break;
        case 32: pw_fwd_kernel<32><<<(int)grid, 256, 0, st>>>(p); break;
        default: pw_fwd_kernel<64><<<(int)grid, 256, 0, st>>>(p); break;
    }
    BTS_LAUNCH_CHECK();
    return 0;
}

