// Scale-invariant log loss (silog_loss, pytorch/bts.py:41-48) forward + backward, sm_90a.
//
// The reference compacts est/gt with a boolean-mask index (nonzero + gather, twice), then runs ~8 small
// ATen kernels; backward scatters back.  Here: ONE streaming pass reduces (sum d, sum d^2, N) over the
// masked pixels (8 B/px + 1 B/px mask), a 1-thread finalize writes the loss, and ONE elementwise pass
// writes d loss / d est (12 B/px).  Cross-block accumulation is fp64 so the result does not depend on
// the block schedule at fp32 resolution.
#include "common.cuh"

namespace {

__device__ __forceinline__ void acc_one(float e, float g, unsigned m, float &s1, float &s2, float &cnt) {
    if (m) {
        const float d = logf(e) - logf(g);
        s1 += d;
        s2 = fmaf(d, d, s2);
        cnt += 1.f;
    }
}

__global__ void __launch_bounds__(256) silog_reduce(const float *__restrict__ est, const float *__restrict__ gt,
                                                    const uint8_t *__restrict__ mask, long long n, int vec_ok,
                                                    double *__restrict__ ws) {
    float s1 = 0.f, s2 = 0.f, cnt = 0.f;
    const long long tid = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long nthreads = (long long)gridDim.x * blockDim.x;
    long long done = 0;
    if (vec_ok) {
        const long long nq = n >> 2;
        const float4 *e4 = reinterpret_cast<const float4 *>(est);
        const float4 *g4 = reinterpret_cast<const float4 *>(gt);
        const uchar4 *m4 = reinterpret_cast<const uchar4 *>(mask);
        for (long long q = tid; q < nq; q += nthreads) {
            const float4 e = __ldg(e4 + q);
            const float4 g = __ldg(g4 + q);
            const uchar4 m = __ldg(m4 + q);
            acc_one(e.x, g.x, m.x, s1, s2, cnt);
            acc_one(e.y, g.y, m.y, s1, s2, cnt);
            acc_one(e.z, g.z, m.z, s1, s2, cnt);
            acc_one(e.w, g.w, m.w, s1, s2, cnt);
        }
        done = nq << 2;
    }
    for (long long i = done + tid; i < n; i += nthreads) acc_one(est[i], gt[i], mask[i], s1, s2, cnt);

    double a = s1, b = s2, c = cnt;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        a += __shfl_xor_sync(0xffffffffu, a, o);
        b += __shfl_xor_sync(0xffffffffu, b, o);
        c += __shfl_xor_sync(0xffffffffu, c, o);
    }
    __shared__ double sm[3][8];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (lane == 0) { sm[0][warp] = a; sm[1][warp] = b; sm[2][warp] = c; }
    __syncthreads();
    if (warp == 0) {
        a = lane < 8 ? sm[0][lane] : 0.0;
        b = lane < 8 ? sm[1][lane] : 0.0;
        c = lane < 8 ? sm[2][lane] : 0.0;
#pragma unroll
        for (int o = 4; o > 0; o >>= 1) {
            a += __shfl_xor_sync(0xffffffffu, a, o);
            b += __shfl_xor_sync(0xffffffffu, b, o);
            c += __shfl_xor_sync(0xffffffffu, c, o);
        }
        if (lane == 0) {
            atomicAdd(ws + 0, a);
            atomicAdd(ws + 1, b);
            atomicAdd(ws + 2, c);
        }
    }
}

__global__ void silog_finalize(const double *__restrict__ ws, float lambda, float *__restrict__ loss) {
    const double n = ws[2];
    const double m1 = ws[0] / n, m2 = ws[1] / n;   // n == 0 -> NaN, like mean() of an empty tensor
    loss[0] = (float)(sqrt(m2 - (double)lambda * m1 * m1) * 10.0);
}

__global__ void __launch_bounds__(256) silog_grad(const float *__restrict__ est, const float *__restrict__ gt,
                                                  const uint8_t *__restrict__ mask, long long n, int vec_ok,
                                                  float lambda, const double *__restrict__ ws,
                                                  const float *__restrict__ gout, float *__restrict__ dest) {
    const double nn = ws[2];
    const double m1 = ws[0] / nn, m2 = ws[1] / nn;
    const double S = m2 - (double)lambda * m1 * m1;
    const float coef = (float)((double)gout[0] * 10.0 / (sqrt(S) * nn));
    const float lm1 = (float)((double)lambda * m1);
    const long long tid = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long nthreads = (long long)gridDim.x * blockDim.x;
    long long done = 0;
    auto one = [&](float e, float g, unsigned m) -> float {
        return m ? coef * ((logf(e) - logf(g)) - lm1) / e : 0.f;
    };
    if (vec_ok) {
        const long long nq = n >> 2;
        const float4 *e4 = reinterpret_cast<const float4 *>(est);
        const float4 *g4 = reinterpret_cast<const float4 *>(gt);
        const uchar4 *m4 = reinterpret_cast<const uchar4 *>(mask);
        float4 *o4 = reinterpret_cast<float4 *>(dest);
        for (long long q = tid; q < nq; q += nthreads) {
            const float4 e = __ldg(e4 + q);
            const float4 g = __ldg(g4 + q);
            const uchar4 m = __ldg(m4 + q);
            o4[q] = make_float4(one(e.x, g.x, m.x), one(e.y, g.y, m.y), one(e.z, g.z, m.z), one(e.w, g.w, m.w));
        }
        done = nq << 2;
    }
    for (long long i = done + tid; i < n; i += nthreads) dest[i] = one(est[i], gt[i], mask[i]);
}

int stream_grid(long long n) {
    long long g = (n / 4 + 255) / 256;
    const long long cap = (long long)bts_num_sms() * 8;
    if (g > cap) g = cap;
    if (g < 1) g = 1;
    return (int)g;
}

}  // namespace

extern "C" int bts_silog_fwd(const float *est, const float *gt, const uint8_t *mask, long long n, float lambda,
                             double *ws, float *loss, void *stream) {
    if (!est || !gt || !mask || !ws || !loss || n < 0) return BTS_EINVAL;
    cudaStream_t st = (cudaStream_t)stream;
    cudaError_t e = cudaMemsetAsync(ws, 0, 4 * sizeof(double), st);
    if (e != cudaSuccess) return (int)e;
    const int vec_ok = bts_aligned16(est) && bts_aligned16(gt) && ((((uintptr_t)mask) & 3u) == 0);
    if (n > 0) {
        silog_reduce<<<stream_grid(n), 256, 0, st>>>(est, gt, mask, n, vec_ok, ws);
        BTS_LAUNCH_CHECK();
    }
    silog_finalize<<<1, 1, 0, st>>>(ws, lambda, loss);
    BTS_LAUNCH_CHECK();
    return 0;
}

extern "C" int bts_silog_bwd(const float *est, const float *gt, const uint8_t *mask, long long n, float lambda,
                             const double *ws, const float *gout, float *dest, void *stream) {
    if (!est || !gt || !mask || !ws || !gout || !dest || n < 0) return BTS_EINVAL;
    if (n == 0) return 0;
    cudaStream_t st = (cudaStream_t)stream;
    const int vec_ok = bts_aligned16(est) && bts_aligned16(gt) && bts_aligned16(dest) && ((((uintptr_t)mask) & 3u) == 0);
    silog_grad<<<stream_grid(n), 256, 0, st>>>(est, gt, mask, n, vec_ok, lambda, ws, gout, dest);
    BTS_LAUNCH_CHECK();
    return 0;
}
