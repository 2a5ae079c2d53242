// The data formats on either side of the hot path (SURVEY 8f ranks 2 and 3), sm_90a, HBM-bound streaming kernels.
//
//  bts_input_prep   the per-sample input transform of the reference loader, after decoding, fused with the H2D hand-off:
//                   uint8 HWC frame (+ uint16 depth PNG) -> random crop -> horizontal flip -> gamma / brightness / colour
//                   augmentation with clip -> ImageNet mean/std normalisation -> fp32 NHWC image (the layout the conv
//                   engine reads) and fp32 depth in metres.  Reference: pytorch/bts_dataloader.py:128-140 (scaling
//                   /255, /1000 | /256, random_crop), :202-235 (train_preprocess, augment_image), :244-249 (ToTensor +
//                   Normalize); the random decisions (crop origin, flip, gamma, brightness, colours) stay on the host
//                   and arrive as one 9-float parameter row per sample.
//  bts_eval_errors  online-eval post-processing + the nine depth metrics of one image in one pass: clamp / inf / nan
//                   handling of the prediction, validity mask min < gt < max, optional crop rectangle, then
//                   silog, abs_rel, log10, rms, sq_rel, log_rms, d1, d2, d3.  Reference: pytorch/bts_main.py:144-165
//                   (compute_errors), :275-296 (clamps + masks); utils/eval_with_pngs.py:50-72.
//  bts_depth_to_u16 the PNG wire format of bts_test.py:179-185: uint16(depth * scale), scale 256 (KITTI) / 1000 (NYU).
#include <cmath>

#include "common.cuh"

namespace {

constexpr int TPB = 256;

__host__ inline int io_grid(long long items) {
    long long grid = (items + TPB - 1) / TPB;
    const long long cap = (long long)bts_num_sms() * 16;
    if (grid > cap) grid = cap;
    if (grid < 1) grid = 1;
    return (int)grid;
}

// params row (9 floats per sample): y0, x0 (crop origin in the source frame), flip (0/1), augment (0/1), gamma, brightness,
// colour[3].  out image: NHWC fp32 with pixel stride os (>= 3); depth out: (B,H,W) fp32.
__global__ void __launch_bounds__(TPB) input_prep_kernel(const unsigned char *__restrict__ img, int Hs, int Ws,
                                                         const unsigned short *__restrict__ dep, float depth_div,
                                                         const float *__restrict__ params, int B, int H, int W,
                                                         float *__restrict__ out, long long os, float *__restrict__ dout) {
    const float mean[3] = {0.485f, 0.456f, 0.406f}, stdv[3] = {0.229f, 0.224f, 0.225f};
    const long long total = (long long)B * H * W;
    for (long long idx = (long long)blockIdx.x * TPB + threadIdx.x; idx < total; idx += (long long)gridDim.x * TPB) {
        const int x = (int)(idx % W);
        const long long t = idx / W;
        const int y = (int)(t % H), b = (int)(t / H);
        const float *pr = params + b * 9;
        const int y0 = (int)pr[0], x0 = (int)pr[1];
        const bool flip = pr[2] > 0.5f, aug = pr[3] > 0.5f;
        const int sx = x0 + (flip ? (W - 1 - x) : x), sy = y0 + y;       // flip acts on the CROPPED frame (dataloader.py:205-207)
        const unsigned char *px = img + (((long long)b * Hs + sy) * Ws + sx) * 3;
        float o[3];
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            float v = (float)px[c] / 255.0f;                             // np.asarray(image, float32) / 255.0
            if (aug) {
                v = powf(v, pr[4]);                                      // image ** gamma
                v = v * pr[5];                                           // * brightness
                v = v * pr[6 + c];                                       // *= colour image
                v = fminf(fmaxf(v, 0.f), 1.f);                           // np.clip(., 0, 1)
            }
            o[c] = (v - mean[c]) / stdv[c];                              // transforms.Normalize
        }
        float *op = out + idx * os;
        op[0] = o[0]; op[1] = o[1]; op[2] = o[2];
        if (dep) dout[idx] = (float)dep[((long long)b * Hs + sy) * Ws + sx] / depth_div;
    }
}

// sums: [0] n, [1] sum err, [2] sum err^2 (err = ln pred - ln gt), [3] sum |gt-pred|/gt, [4] sum |log10 pred - log10 gt|,
//       [5] sum (gt-pred)^2, [6] sum (gt-pred)^2/gt, [7..9] counts thresh < 1.25^k
__global__ void __launch_bounds__(TPB) eval_reduce_kernel(const float *__restrict__ pred, const float *__restrict__ gt, int H,
                                                          int W, float dmin, float dmax, int cy0, int cy1, int cx0, int cx1,
                                                          double *__restrict__ sums) {
    double acc[10] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0};
    const long long total = (long long)H * W;
    for (long long idx = (long long)blockIdx.x * TPB + threadIdx.x; idx < total; idx += (long long)gridDim.x * TPB) {
        const int x = (int)(idx % W), y = (int)(idx / W);
        const float g = gt[idx];
        float p = pred[idx];
        // bts_main.py:275-278, in this order: < min -> min; > max -> max; inf -> max; nan -> min
        if (p < dmin) p = dmin;
        if (p > dmax) p = dmax;
        if (isinf(p)) p = dmax;
        if (p != p) p = dmin;
        const bool ok = g > dmin && g < dmax && y >= cy0 && y < cy1 && x >= cx0 && x < cx1;
        if (!ok) continue;
        const double gd = g, pd = p;
        const float th = fmaxf(g / p, p / g);                          // fp32, as the numpy reference
        const double err = log(pd) - log(gd), d = gd - pd;
        acc[0] += 1.0;
        acc[1] += err;
        acc[2] += err * err;
        acc[3] += fabs(d) / gd;
        acc[4] += fabs(log10(pd) - log10(gd));
        acc[5] += d * d;
        acc[6] += d * d / gd;
        acc[7] += th < 1.25f ? 1.0 : 0.0;
        acc[8] += th < 1.5625f ? 1.0 : 0.0;
        acc[9] += th < 1.953125f ? 1.0 : 0.0;
    }
    __shared__ double red[TPB / 32][10];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int k = 0; k < 10; ++k) {
        double v = acc[k];
        for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
        if (lane == 0) red[warp][k] = v;
    }
    __syncthreads();
    if (threadIdx.x < 10) {
        double v = 0.0;
        for (int w = 0; w < TPB / 32; ++w) v += red[w][threadIdx.x];
        atomicAdd(sums + threadIdx.x, v);
    }
}

// out[9] = silog, abs_rel, log10, rms, sq_rel, log_rms, d1, d2, d3 (the order of eval_metrics, bts_main.py:141); out[9] = n
__global__ void eval_finalize_kernel(const double *__restrict__ s, float *__restrict__ out) {
    const double n = s[0];
    const double m1 = s[1] / n, m2 = s[2] / n;
    out[0] = (float)(sqrt(m2 - m1 * m1) * 100.0);
    out[1] = (float)(s[3] / n);
    out[2] = (float)(s[4] / n);
    out[3] = (float)sqrt(s[5] / n);
    out[4] = (float)(s[6] / n);
    out[5] = (float)sqrt(m2);              // log_rms: (ln gt - ln pred)^2 == err^2
    out[6] = (float)(s[7] / n);
    out[7] = (float)(s[8] / n);
    out[8] = (float)(s[9] / n);
    out[9] = (float)n;
}

__global__ void __launch_bounds__(TPB) depth_to_u16_kernel(const float *__restrict__ d, float scale, long long n,
                                                           unsigned short *__restrict__ out) {
    for (long long i = (long long)blockIdx.x * TPB + threadIdx.x; i < n; i += (long long)gridDim.x * TPB) {
        const float v = d[i] * scale;
        // numpy float32 -> uint16 astype: C conversion (truncation toward zero) and wrap modulo 2^16 for in-range ints
        const long long q = (long long)v;
        out[i] = (unsigned short)(q & 0xffff);
    }
}

}  // namespace

extern "C" int bts_input_prep(const unsigned char *img_u8, int Hs, int Ws, const unsigned short *depth_u16, float depth_div,
                              const float *params, int B, int H, int W, float *image_out, long long out_pixel_stride,
                              float *depth_out, void *stream) {
    if (!img_u8 || !params || !image_out || B < 1 || H < 1 || W < 1 || Hs < H || Ws < W || out_pixel_stride < 3) return BTS_EINVAL;
    if (depth_u16 && (!depth_out || depth_div <= 0.f)) return BTS_EINVAL;
    input_prep_kernel<<<io_grid((long long)B * H * W), TPB, 0, (cudaStream_t)stream>>>(img_u8, Hs, Ws, depth_u16, depth_div, params,
                                                                                       B, H, W, image_out, out_pixel_stride,
                                                                                       depth_out);
    BTS_LAUNCH_CHECK();
    return 0;
}

// workspace: 10 doubles; metrics_out: 10 floats (9 metrics + the number of valid pixels).  crop = [y0, y1) x [x0, x1).
extern "C" int bts_eval_errors(const float *pred, const float *gt, int H, int W, float min_depth, float max_depth, int crop_y0,
                               int crop_y1, int crop_x0, int crop_x1, double *workspace, float *metrics_out, void *stream) {
    if (!pred || !gt || !workspace || !metrics_out || H < 1 || W < 1) return BTS_EINVAL;
    cudaStream_t st = (cudaStream_t)stream;
    cudaError_t e = cudaMemsetAsync(workspace, 0, 10 * sizeof(double), st);
    if (e != cudaSuccess) return (int)e;
    eval_reduce_kernel<<<io_grid((long long)H * W), TPB, 0, st>>>(pred, gt, H, W, min_depth, max_depth, crop_y0, crop_y1, crop_x0,
                                                                 crop_x1, workspace);
    BTS_LAUNCH_CHECK();
    eval_finalize_kernel<<<1, 1, 0, st>>>(workspace, metrics_out);
    BTS_LAUNCH_CHECK();
    return 0;
}

extern "C" int bts_depth_to_u16(const float *depth, float scale, long long n, unsigned short *out, void *stream) {
    if (!depth || !out || n < 1) return BTS_EINVAL;
    depth_to_u16_kernel<<<io_grid(n), TPB, 0, (cudaStream_t)stream>>>(depth, scale, n, out);
    BTS_LAUNCH_CHECK();
    return 0;
}
