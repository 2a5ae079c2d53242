// Fused multi-tensor AdamW (decoupled weight decay) -- the optimizer step of the reference training loop
// (pytorch/bts_main.py:371-373 torch.optim.AdamW over two parameter groups, :456-460 poly learning rate), sm_90a,
// HBM-bound: every parameter of the model in ONE launch instead of torch's ~10 foreach kernels per group.
//
// Per element, in the operation order of torch's own multi-tensor implementation (torch/optim/adam.py _multi_tensor_adam)
// so that results agree to an ulp:
//   p  = p * (1 - lr*wd)
//   m  = m + (1-b1) * (g - m)                      (_foreach_lerp_)
//   v  = v * b2;  v = v + (1-b2) * g * g           (_foreach_mul_, _foreach_addcmul_)
//   d  = sqrt(v) / sqrt(1 - b2^t) + eps
//   p  = p + (-lr / (1 - b1^t)) * (m / d)          (_foreach_addcdiv_)
// The per-group scalars are computed on the host in double and rounded to fp32 exactly as torch's python-scalar overloads do.
// Algorithmic bytes: 16 B read + 12 B written per parameter.
#include "common.cuh"

namespace {

constexpr int TPB = 256;
constexpr int CHUNK = 4096;            // elements per block-iteration
constexpr int MAX_GROUPS = 8;

struct AdamGroups {
    float decay[MAX_GROUPS];           // 1 - lr*wd
    float w1[MAX_GROUPS];              // 1 - beta1
    float b2[MAX_GROUPS];              // beta2
    float w2[MAX_GROUPS];              // 1 - beta2
    float bc2_sqrt[MAX_GROUPS];        // sqrt(1 - beta2^t)
    float eps[MAX_GROUPS];
    float neg_step[MAX_GROUPS];        // -lr / (1 - beta1^t)
};

// tensor table: 4 pointer arrays [n] (param, grad, exp_avg, exp_avg_sq), numel[n], group[n]; chunk table: tensor id + offset
__global__ void __launch_bounds__(TPB) adamw_multi_kernel(const long long *__restrict__ ptrs, const long long *__restrict__ numel,
                                                          const int *__restrict__ group, int n,
                                                          const int *__restrict__ chunk_tensor,
                                                          const long long *__restrict__ chunk_off, int n_chunks,
                                                          const AdamGroups G) {
    for (int ch = blockIdx.x; ch < n_chunks; ch += gridDim.x) {
        const int t = chunk_tensor[ch];
        const long long off = chunk_off[ch];
        float *__restrict__ p = reinterpret_cast<float *>(ptrs[t]) + off;
        const float *__restrict__ g = reinterpret_cast<const float *>(ptrs[n + t]) + off;
        float *__restrict__ m = reinterpret_cast<float *>(ptrs[2 * n + t]) + off;
        float *__restrict__ v = reinterpret_cast<float *>(ptrs[3 * n + t]) + off;
        long long cnt = numel[t] - off;
        if (cnt > CHUNK) cnt = CHUNK;
        const int gi = group[t];
        const float decay = G.decay[gi], w1 = G.w1[gi], b2 = G.b2[gi], w2 = G.w2[gi], bs = G.bc2_sqrt[gi], eps = G.eps[gi],
                    ns = G.neg_step[gi];
        auto upd = [&](float &pp, float gg, float &mm, float &vv) {
            pp = __fmul_rn(pp, decay);
            mm = fmaf(w1, gg - mm, mm);
            vv = __fmul_rn(vv, b2);
            vv = fmaf(__fmul_rn(w2, gg), gg, vv);
            const float d = __fadd_rn(__fdiv_rn(__fsqrt_rn(vv), bs), eps);
            pp = fmaf(ns, __fdiv_rn(mm, d), pp);
        };
        const bool vec = ((((uintptr_t)p) | ((uintptr_t)g) | ((uintptr_t)m) | ((uintptr_t)v)) & 15u) == 0;
        if (vec) {
            const int n4 = (int)(cnt >> 2);
            for (int i = threadIdx.x; i < n4; i += TPB) {
                float4 P = reinterpret_cast<float4 *>(p)[i];
                const float4 Gd = __ldg(reinterpret_cast<const float4 *>(g) + i);
                float4 M = reinterpret_cast<float4 *>(m)[i];
                float4 V = reinterpret_cast<float4 *>(v)[i];
                upd(P.x, Gd.x, M.x, V.x);
                upd(P.y, Gd.y, M.y, V.y);
                upd(P.z, Gd.z, M.z, V.z);
                upd(P.w, Gd.w, M.w, V.w);
                reinterpret_cast<float4 *>(p)[i] = P;
                reinterpret_cast<float4 *>(m)[i] = M;
                reinterpret_cast<float4 *>(v)[i] = V;
            }
            for (int i = (n4 << 2) + threadIdx.x; i < cnt; i += TPB) upd(p[i], g[i], m[i], v[i]);
        } else {
            for (int i = threadIdx.x; i < cnt; i += TPB) upd(p[i], g[i], m[i], v[i]);
        }
    }
}

}  // namespace

extern "C" int bts_adamw_chunk(void) { return CHUNK; }

// ptrs: device int64 [4*n] = param | grad | exp_avg | exp_avg_sq addresses; numel: device int64 [n]; group: device int32 [n]
// (index into the n_groups scalar sets); chunk_tensor / chunk_off: device tables of the bts_adamw_chunk()-element pieces.
// scalars: host float [7 * n_groups] = decay | 1-beta1 | beta2 | 1-beta2 | sqrt(1-beta2^t) | eps | -lr/(1-beta1^t), group-major
// within each of the seven blocks.
extern "C" int bts_adamw_multi(const long long *ptrs, const long long *numel, const int *group, int n, const int *chunk_tensor,
                               const long long *chunk_off, int n_chunks, const float *scalars, int n_groups, void *stream) {
    if (!ptrs || !numel || !group || !chunk_tensor || !chunk_off || !scalars || n < 1 || n_chunks < 1 || n_groups < 1 ||
        n_groups > MAX_GROUPS)
        return BTS_EINVAL;
    AdamGroups G;
    for (int i = 0; i < n_groups; ++i) {
        G.decay[i] = scalars[0 * n_groups + i];
        G.w1[i] = scalars[1 * n_groups + i];
        G.b2[i] = scalars[2 * n_groups + i];
        G.w2[i] = scalars[3 * n_groups + i];
        G.bc2_sqrt[i] = scalars[4 * n_groups + i];
        G.eps[i] = scalars[5 * n_groups + i];
        G.neg_step[i] = scalars[6 * n_groups + i];
    }
    int grid = n_chunks;
    const int cap = bts_num_sms() * 16;
    if (grid > cap) grid = cap;
    adamw_multi_kernel<<<grid, TPB, 0, (cudaStream_t)stream>>>(ptrs, numel, group, n, chunk_tensor, chunk_off, n_chunks, G);
    BTS_LAUNCH_CHECK();
    return 0;
}
