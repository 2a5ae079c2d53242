// Implicit-GEMM convolution on the Hopper tensor cores (wgmma, register accumulators), sm_90a, parity-grade 3xTF32.
//
// Replaces the cuDNN convolution (+ separate BN-apply / ReLU / ELU / nearest-upsample ATen kernels) behind every
// 1x1 / 3x3 / dilated conv of the BTS decoder and the torchvision encoder (reference pytorch/bts.py:51-80,153-194).
//
//   out[p, co] = act( sum_{tap, ci}  pre(x[p (+) tap, ci]) * w[co, ci, tap] )         NHWC activations
//       pre  = optional per-input-channel affine (a folded BatchNorm: x*scale+shift) and/or ReLU, applied to the
//              A operand on its way into shared memory; zero padding is applied AFTER pre (as conv2d pads the
//              normalised tensor);  (+) includes stride, dilation and an optional nearest x2 up-sample of the source
//              (upconv, bts.py:77) which is folded into the address map -- the 4x tensor is never materialised.
//       act  = none | ELU | sigmoid, fused in the epilogue.
//
// GEMM view: M = B*Hout*Wout pixels (128 per CTA tile: two warpgroups of 64 rows), N = Cout (<= 64 per tile: the
// k-block accumulator and the tile sum of a 64 x 64 tile are 64 registers per thread), K = the dense sequence of 16-byte channel quads,
// tap-major, in blocks of 32 fp32 (one 128-byte swizzled row per pixel).
// Precision: fp32 operands are split x = hi + lo with hi = rna_tf32(x), lo = rna_tf32(x - hi) and the tile
// accumulates  A_lo*B_hi + A_hi*B_lo + A_hi*B_hi  with tf32 wgmma into fp32 register accumulators (error
// ~2^-21 per product: fp32-grade, SURVEY Appendix F); every k-block's tensor-core sum is added into the tile sum with
// round-to-nearest fp32 adds.
// Single-pass TF32 is available as an explicitly labelled fast mode (precision=1) and is NOT used for parity.
//
// Persistent kernel: grid = min(#tiles, #SMs); every CTA walks tiles blockIdx.x, +gridDim.x, ... with the smem stage
// ring and all warp roles running continuously across tile boundaries (the loader and producers fill the stages of tile
// t+1 while the consumers run the epilogue of tile t; no per-tile launch or pipeline-fill cost).
// Warp roles (288 + 128 G threads, 1 CTA/SM):
//   warps 0..7  : two consumer warpgroups -- wgmma on the staged operands, then the epilogue from the accumulator
//                 registers: activation, NHWC stores, optional BatchNorm batch statistics of the output;
//   warp 8      : weight loader -- one thread streams pre-packed, pre-split, pre-swizzled weight tiles with 1-D bulk
//                 async copies (cp.async.bulk) completing on an mbarrier (and, in TMA mode, the im2col activation tile);
//   warps 9..   : G producer groups (alternating k-blocks): coalesced 128-bit global loads of the activation
//                 tile (8 lanes cover one pixel's 128 B), pre-op + hi/lo split in registers, swizzled 128-bit
//                 shared stores of both halves, fence.proxy.async, mbarrier arrive.
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <type_traits>

#include <cuda.h>

#include "tc_common.cuh"

namespace {

constexpr int BLOCK_M = 128;
constexpr int BLOCK_K = 32;                 // fp32 elements per k-block = one 128-byte row
constexpr int MAX_N = 64;                   // output channels per tile (two register accumulators per consumer thread)
constexpr int A_TILE_BYTES = BLOCK_M * 128; // 16 KB (hi or lo)
constexpr int CONSUMER_THREADS = 256;       // two warpgroups
constexpr int LOADER_WARP = CONSUMER_THREADS / 32;
constexpr int PRODUCER_THREADS = 128;       // per group
constexpr int FOUR_GROUPS_MAX_N = 48;       // widest tile run with four producer groups
constexpr int MAX_CIN_SMEM = 4096;          // pre-op scale/shift staged in smem (32 KB at most)

struct ConvParams {
    const float *x;          // NHWC source, pixel stride xs floats
    long long xs;
    int B, Hs, Ws;           // source dims (before the optional x2 up-sample)
    int up;                  // 1: nearest x2 up-sample folded in (conv sees 2Hs x 2Ws); 2: zero-stuffed x2 (the dgrad of a
                             //    stride-2 convolution: only even coordinates of the Hv x Wv virtual source are live)
    int Hv, Wv;              // virtual source dims seen by the conv (= Hs,Ws | 2Hs,2Ws | the stride-2 layer's input size)
    int Cin;                 // K channels per tap of ONE n-tile (grouped: the channel window, else all input channels)
    int kwin;                // grouped / block-diagonal: output channels c read the input-channel window
                             //    [c / kwin * kwin, + kwin) (n_tile divides kwin); 0 = dense
    int KH, KW, stride, pad, dil;
    const float *wpack;      // packed weights (see pack kernel)
    int n_tile, n_tiles, Cout;
    const float *pre_scale;  // [Cin] or null
    const float *pre_shift;  // [Cin] or null
    int pre_relu;
    float *out;              // NHWC, pixel stride os floats (may be a channel slice of a wider slab)
    long long os;
    int Hout, Wout;
    int act;                 // 0 none, 1 ELU, 2 sigmoid
    int precision;           // 0: 3xTF32 (parity), 1: 1xTF32 (fast, labelled)
    int vec_ok;              // 16-byte aligned rows -> float4 loads
    long long M;             // B*Hout*Wout
    int m_tiles, total_tiles;
    int KC;                  // ceil(Cin/32)
    int CQ;                  // ceil(Cin/4): 16-byte channel quads per tap (dense-K order, see the pack kernel)
    int KB;                  // ceil(KH*KW*CQ / 8) k-blocks
    tc::FastDiv fd_cq, fd_kw;
    double *stat_sum, *stat_sumsq;   // optional per-output-channel sum / sum of squares of the (activated) output
    // BatchNorm-backward reduction fused into a dgrad's epilogue (bnb_x != null): the tile being written is g = dL/d relu(bn(x));
    // stat_sum[c] += sum_p g*[bn(x)>0],  stat_sumsq[c] += sum_p g*[bn(x)>0]*xhat   (bts_bn_relu_bwd_reduce without its pass)
    int chunk_major;         // K order: k-block kb = (chunk kb / taps, tap kb % taps) -- consecutive k-blocks re-read the SAME
                             // pixels' lines shifted by one tap, so they hit in L1 instead of going to L2 nine times
    int tma_adj;             // TMA mode: base-pixel coordinate = out*stride - tma_adj (the bounding box's lower corner)
    tc::FastDiv fd_taps;     // chunk-major: kb -> (kb / taps, kb % taps)
    tc::FastDiv fd_kc;       // TMA mode: k-block -> (tap, 32-channel chunk) = (kb / KC, kb % KC)
    const float *bnb_x; long long bnb_xs;
    const float *bnb_st;             // [4][Cout]: scale, shift, mean, invstd
    int bnb_relu;
    int stages, stage_bytes; // smem ring: as many (A hi/lo + B hi/lo) stages as fit
    tc::FastDiv fd_wout, fd_hout, fd_ntiles;
};

using namespace tc;

// ------------------------------------------------------------------------------------------- weight packing
// wpack layout: [n_tiles][KB][2 (hi,lo)][n_tile rows][32 floats], each row 128 B with the 16-byte chunk index
// XOR-ed by (row & 7) -- exactly the shared-memory image of a K-major SWIZZLE_128B tile, so one contiguous bulk
// copy per k-block lands it.
// K order ("dense K"): the K axis is the sequence of 16-byte channel quads, tap-major: quad g = tap * CQ + c4 with
// CQ = ceil(Kch / 4); k-block kb holds quads 8 kb .. 8 kb + 7.  A tap therefore costs ceil4(Kch) K-slots instead of
// ceil32(Kch): conv1 (Cin 36) 11 k-blocks instead of 18, the 3x3 dgrad of the dense layers (48) 14 instead of 18,
// the 7x7 stem (Cin 3) 7 instead of 49.  Identical to the per-tap 32-channel chunking whenever Kch % 32 == 0.
// transpose_flip=1 packs the dgrad operator: rows = ci, k = (flipped tap, co).
__device__ __forceinline__ void pack_one(const float *__restrict__ w, long long s_co, long long s_ci, long long s_kh,
                                         long long s_kw, int Cout, int Cin, int KH, int KW, int transpose_flip,
                                         float *__restrict__ wpack, int n_tile, int kwin, int cpg, int flags,
                                         long long idx) {
    // grouped (kwin > 0): Cin == Cout == total width, w is (width, cpg, KH, KW); rows = all channels, the K channels of
    // n-tile nt are the window of kwin channels that holds its rows (n_tile divides kwin) and entries outside the row's
    // group are zero (block diagonal)
    const int Nrows = transpose_flip ? Cin : Cout;    // GEMM N
    const int Kch = kwin ? kwin : (transpose_flip ? Cout : Cin);      // GEMM K channels per tap
    const int CQ = (Kch + 3) / 4;
    const int taps = KH * KW;
    const int KB = (taps * CQ + 7) / 8;
    const int kk = (int)(idx & 31);
    long long t = idx >> 5;
    const int n = (int)(t % n_tile);
    t /= n_tile;
    const int kb = (int)(t % KB);
    const int nt = (int)(t / KB);
    const int g = kb * 8 + (kk >> 2);
    int tap = g / CQ;
    int ch = (g - tap * CQ) * 4 + (kk & 3);
    if (flags & 1) {                      // chunk-major K order (Kch % 32 == 0): k-block = (32-channel chunk, tap), taps innermost
        tap = kb % taps;
        ch = (kb / taps) * 32 + kk;
    }
    const int row = nt * n_tile + n;
    float val = 0.f;
    if (row < Nrows && tap < taps && ch < Kch) {
        int kh = tap / KW, kw = tap % KW;
        long long off;
        bool live = true;
        int kc = ch, rr = row;            // K channel / row index into w's (co, ci) axes
        if (kwin) {
            const int kglob = nt * n_tile / kwin * kwin + ch;     // global channel on the K side
            live = (kglob / cpg) == (row / cpg);
            if (transpose_flip) { kc = kglob; rr = row % cpg; }   // w[co = kglob][ci_local = row % cpg]
            else { kc = kglob % cpg; }                            // w[co = row][ci_local = kglob % cpg]
        }
        if (transpose_flip) {
            kh = KH - 1 - kh; kw = KW - 1 - kw;
            off = (long long)kc * s_co + (long long)rr * s_ci + kh * s_kh + kw * s_kw;
        } else {
            off = (long long)rr * s_co + (long long)kc * s_ci + kh * s_kh + kw * s_kw;
        }
        if (live) val = w[off];
    }
    const float hi = rna_tf32(val);
    const float lo = rna_tf32(val - hi);
    const size_t tile = ((size_t)nt * KB + kb) * 2 * (size_t)n_tile * 32;
    const size_t in_tile = (size_t)n * 32 + (size_t)(((kk >> 2) ^ (n & 7)) << 2) + (kk & 3);
    wpack[tile + in_tile] = hi;
    wpack[tile + (size_t)n_tile * 32 + in_tile] = lo;
}

__global__ void __launch_bounds__(256) pack_weights_kernel(const float *__restrict__ w, long long s_co, long long s_ci,
                                                           long long s_kh, long long s_kw, int Cout, int Cin, int KH,
                                                           int KW, int transpose_flip, float *__restrict__ wpack,
                                                           int n_tile, int n_tiles, int kwin, int cpg, int flags) {
    const int Kch = kwin ? kwin : (transpose_flip ? Cout : Cin);
    const int KB = (KH * KW * ((Kch + 3) / 4) + 7) / 8;
    const long long total = (long long)n_tiles * KB * n_tile * 32;
    for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
         idx += (long long)gridDim.x * blockDim.x)
        pack_one(w, s_co, s_ci, s_kh, s_kw, Cout, Cin, KH, KW, transpose_flip, wpack, n_tile, kwin, cpg, flags, idx);
}

// every packed operator of a model in ONE launch (after an optimizer step: 394 launches -> 1 for DenseNet-161 + decoder)
struct PackDesc {
    const float *w;
    float *wpack;
    long long s_co, s_ci, s_kh, s_kw;
    long long start;                     // first global index of this operator (prefix sum of packed_floats / 2)
    int Cout, Cin, KH, KW, transpose_flip, n_tile, n_tiles, kwin, cpg, flags;   // flags bit 0: chunk-major K order
};
static_assert(sizeof(PackDesc) == 96, "PackDesc layout is mirrored by bts_b200/conv.py");

__global__ void __launch_bounds__(256) pack_weights_multi_kernel(const PackDesc *__restrict__ d, int n, long long total) {
    for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
         idx += (long long)gridDim.x * blockDim.x) {
        int lo = 0, hi = n - 1;                                    // last descriptor with start <= idx
        while (lo < hi) {
            const int mid = (lo + hi + 1) >> 1;
            if (d[mid].start <= idx) lo = mid; else hi = mid - 1;
        }
        const PackDesc &q = d[lo];
        pack_one(q.w, q.s_co, q.s_ci, q.s_kh, q.s_kw, q.Cout, q.Cin, q.KH, q.KW, q.transpose_flip, q.wpack, q.n_tile, q.kwin,
                 q.cpg, q.flags, idx - q.start);
    }
}

// ------------------------------------------------------------------------------------------- main kernel
// dynamic smem, 1024-byte aligned base:
//   [S stages][A_hi 16K | A_lo 16K | B_hi n_tile*128 | B_lo n_tile*128]   S = as many stages as fit (2..MAX_STAGES)
//   [pre-op scale[KC*32], shift[KC*32]]  (PRE >= 2 only)   [mbarriers]   [epilogue statistics partials]
constexpr int MAX_STAGES = 6;
constexpr int SMEM_LIMIT = 232448;          // 227 KB opt-in maximum per CTA
constexpr int BAR_BYTES = 256;
// per-CTA partial sums of the epilogue statistics: fp64, one private set per consumer warp ([8][2][n_tile]) -- no atomics
// inside the CTA and a fixed accumulation order, so a training step is reproducible run to run
constexpr int STAT_SETS = CONSUMER_THREADS / 32;

// PRE: 0 none, 1 ReLU, 2 affine, 3 affine + ReLU (compile-time so the per-element producer code carries no dead ops)
// UP : nearest x2 up-sample folded into the address map;  VEC: 16-byte aligned rows (float4 loads)
//
// Index arithmetic: every k-block -> (tile, tap, channel chunk, stage, phase) mapping is carried in incrementally updated
// counters, and the per-tile pixel decode uses multiply-shift division by host-precomputed constants (FastDiv).
// TMA = true: the activation tile is staged by the Tensor Memory Accelerator (one cp.async.bulk.tensor im2col load per
// k-block lands 128 pixels x 32 channels, swizzled, zero-filled where the filter tap falls into the padding) and is used
// AS IS as the A_hi operand (the tensor core reads the top 19 bits of each fp32 word); the producer warps only derive
// A_lo = x - trunc_tf32(x) from shared memory (and apply the BN/ReLU pre-op in place) -- no global loads, no address /
// bounds arithmetic, one shared store instead of two.  K is enumerated per tap in 32-channel chunks (identical to the
// dense-quad order whenever the K channels are a multiple of 32, which the host requires), stride 1, no up-sample.
// G: producer groups (4 warps each).  G = 2 keeps one k-block of register prefetch per thread (two F4[8] buffers); G = 4
// (narrow-N layers with >= 4 stages) drops the second buffer and lets the other groups' work hide a group's load latency.
template <int PRE, int UP, bool VEC, bool TMA, int G>
__global__ void __launch_bounds__(CONSUMER_THREADS + 32 + 128 * G, 1) conv_tc_kernel(const ConvParams p,
                                                                                      const __grid_constant__ CUtensorMap tmap) {
    constexpr int NUM_THREADS = CONSUMER_THREADS + 32 + 128 * G;
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    // dynamic smem base is only guaranteed 16-byte aligned: round up to 1024 (SWIZZLE_128B atoms)
    const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;
    uint8_t *sm = smem_raw + (base - smem_u32(smem_raw));
    const int S = p.stages;
    const uint32_t stage_bytes = (uint32_t)p.stage_bytes;
    const uint32_t pre_off = (uint32_t)S * stage_bytes;
    float *s_scale = reinterpret_cast<float *>(sm + pre_off);
    float *s_shift = s_scale + p.KC * 32;
    const uint32_t bar_off = pre_off + (PRE >= 2 ? (uint32_t)p.KC * 32u * 8u : 0u);
    // bars: [0..MS) full (128 producer arrivals [+ the weight loader's expect_tx arrival and its bytes]), [MS..2MS) raw
    // (TMA mode: the activation tile and the weights land there), [2MS..3MS) empty (one arrival per consumer warp)
    const uint32_t bar0 = base + bar_off;
    auto full_a = [&](int s) { return bar0 + 8u * s; };
    auto raw = [&](int s) { return bar0 + 8u * (MAX_STAGES + s); };
    auto full_b = [&](int s) { return TMA ? raw(s) : full_a(s); };
    auto empty = [&](int s) { return bar0 + 8u * (2 * MAX_STAGES + s); };
    double *s_stat = reinterpret_cast<double *>(sm + bar_off + BAR_BYTES);    // [8 warps][2][n_tile], only when p.stat_sum

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int n_tile = p.n_tile;
    const int KB = p.KB;
    if (p.stat_sum)
        for (int i = threadIdx.x; i < STAT_SETS * 2 * n_tile; i += NUM_THREADS) s_stat[i] = 0.0;
    // tiles of this CTA: blockIdx.x, blockIdx.x + gridDim.x, ...   (tile -> m_tile = tile / n_tiles, nt = tile % n_tiles)
    const int my_tiles = (p.total_tiles - (int)blockIdx.x + (int)gridDim.x - 1) / (int)gridDim.x;
    const int total_kb = my_tiles * KB;          // host guarantees < 2^31

    if (threadIdx.x == 0) {
        for (int s = 0; s < S; ++s) {
            mbar_init(full_a(s), TMA ? PRODUCER_THREADS : PRODUCER_THREADS + 1);
            mbar_init(raw(s), 1);
            mbar_init(empty(s), CONSUMER_THREADS / 32);
        }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    if (PRE >= 2) {
        for (int c = threadIdx.x; c < p.KC * 32; c += NUM_THREADS) {
            s_scale[c] = c < p.Cin ? p.pre_scale[c] : 0.f;
            s_shift[c] = c < p.Cin ? p.pre_shift[c] : 0.f;
        }
    }
    __syncthreads();

    if (warp == LOADER_WARP) {
        // ===================== weight loader =====================
        if (lane == 0) {
            const uint32_t bytes = 2u * (uint32_t)n_tile * 128u;
            if (TMA) tma_prefetch_desc(&tmap);
            int s = 0;
            uint32_t ph = 0;
            for (int ti = 0; ti < my_tiles; ++ti) {
                const int tile = (int)blockIdx.x + ti * (int)gridDim.x;
                const uint32_t m_tile = fdiv((uint32_t)tile, p.fd_ntiles);
                const int nt = tile - (int)m_tile * p.n_tiles;
                const uint8_t *src = reinterpret_cast<const uint8_t *>(p.wpack) + (size_t)nt * KB * bytes;
                const int win0 = p.kwin ? nt * n_tile / p.kwin * p.kwin : 0;     // grouped: first channel of the K window
                int tw = 0, th = 0, tn = 0;
                if (TMA) {                         // first output pixel of the tile -> base-pixel coordinate of the im2col walk
                    const uint32_t m0 = m_tile * BLOCK_M;
                    const uint32_t q = fdiv(m0, p.fd_wout);
                    const uint32_t b = fdiv(q, p.fd_hout);
                    tw = (int)(m0 - q * (uint32_t)p.Wout) - p.tma_adj;
                    th = (int)(q - b * (uint32_t)p.Hout) - p.tma_adj;
                    tn = (int)b;
                }
                int tap = 0, kc = 0;               // k-block -> (tap, chunk), advanced incrementally
                for (int kb = 0; kb < KB; ++kb) {
                    mbar_wait_sleep(empty(s), ph ^ 1);
                    if (TMA) {
                        mbar_arrive_expect_tx(raw(s), bytes + (uint32_t)A_TILE_BYTES);
                        const int ky = (int)fdiv((uint32_t)tap, p.fd_kw), kx = tap - ky * p.KW;
                        tma_im2col_4d(base + (uint32_t)s * stage_bytes, &tmap, win0 + kc * 32, tw, th, tn, raw(s),
                                      (uint16_t)(kx * p.dil), (uint16_t)(ky * p.dil));
                        if (++kc == p.KC) { kc = 0; ++tap; }
                    } else {
                        mbar_arrive_expect_tx(full_b(s), bytes);
                    }
                    bulk_copy_g2s(base + (uint32_t)s * stage_bytes + 2 * A_TILE_BYTES, src + (size_t)kb * bytes, bytes, full_b(s));
                    if (++s == S) { s = 0; ph ^= 1; }
                }
            }
        }
    } else if (warp > LOADER_WARP) {
        // ===================== activation producers (G groups x 4 warps) =====================
        const int pt = threadIdx.x - (CONSUMER_THREADS + 32);
        const int grp = pt >> 7;                   // producer group: global k-blocks gk == grp (mod G)
        const int t = pt & 127;
        const int chunk = t & 7;                   // 16-byte chunk of the 128-byte row
        const int r0 = t >> 3;                     // rows r0 + 16*i, i = 0..7  (row & 7 == r0 & 7 for all of them)
        const int Hin = p.Hv, Win = p.Wv;
        const int xs = (int)p.xs;                  // host guarantees the source has < 2^31 elements
        const int KW = p.KW, dil = p.dil, Cin = p.Cin, Ws = p.Ws;
        const int taps = p.KH * p.KW;
        constexpr bool AFF = PRE >= 2;
        constexpr bool RELU = (PRE & 1) != 0;
        const float *__restrict__ xg = p.x;
        // swizzled byte offset of (row r0 + 16 i, chunk) inside a tile = roff0 + i * 2048
        const uint32_t roff0 = (uint32_t)r0 * 128u + (uint32_t)((chunk ^ (r0 & 7)) << 4);
        if constexpr (TMA) {
            // ---- lo-producers: the raw tile is already in shared memory (TMA); derive A_lo (and the pre-op) in place
            const bool need_mask = AFF && taps > 1;        // zero padding is applied AFTER the BatchNorm/ReLU pre-op
            int oyt[8], oxt[8];
            int ti = 0, kb = grp, cur = -1;
            while (kb >= KB) { kb -= KB; ++ti; }
            int s_t = grp;
            uint32_t ph_t = 0;
            const int mine_t = (total_kb - grp + 1) >> 1;
            for (int it = 0; it < mine_t; ++it) {
                int tap = 0, kc = kb;
                if (taps > 1) { tap = (int)fdiv((uint32_t)kb, p.fd_kc); kc = kb - tap * p.KC; }
                const int c = kc * 32 + chunk * 4;
                uint32_t live = 0xffu;
                if (need_mask) {
                    if (ti != cur) {
                        cur = ti;
                        const int tile = (int)blockIdx.x + ti * (int)gridDim.x;
                        const uint32_t m_base = fdiv((uint32_t)tile, p.fd_ntiles) * BLOCK_M + (uint32_t)r0;
#pragma unroll
                        for (int i = 0; i < 8; ++i) {
                            const uint32_t m = m_base + 16u * i;
                            const uint32_t q = fdiv(m, p.fd_wout);
                            const uint32_t b = fdiv(q, p.fd_hout);
                            oxt[i] = (int)(m - q * (uint32_t)p.Wout) - p.pad;
                            oyt[i] = (int)(q - b * (uint32_t)p.Hout) - p.pad;
                        }
                    }
                    const int ky = (int)fdiv((uint32_t)tap, p.fd_kw), kx = tap - ky * KW;
                    live = 0;
#pragma unroll
                    for (int i = 0; i < 8; ++i)
                        live |= (((unsigned)(oyt[i] + ky * dil) < (unsigned)Hin && (unsigned)(oxt[i] + kx * dil) < (unsigned)Win) ? 1u : 0u) << i;
                }
                float sc[4] = {1.f, 1.f, 1.f, 1.f}, sh[4] = {0.f, 0.f, 0.f, 0.f};
                if (AFF) {
                    const float4 a4 = *reinterpret_cast<const float4 *>(s_scale + c);
                    const float4 b4 = *reinterpret_cast<const float4 *>(s_shift + c);
                    sc[0] = a4.x; sc[1] = a4.y; sc[2] = a4.z; sc[3] = a4.w;
                    sh[0] = b4.x; sh[1] = b4.y; sh[2] = b4.z; sh[3] = b4.w;
                }
                const uint32_t a_hi = base + (uint32_t)s_t * stage_bytes + roff0;
                const uint32_t a_lo = a_hi + A_TILE_BYTES;
                // First make sure the PREVIOUS use of this stage was consumed (what the loader waited for before re-arming
                // raw): a parity wait only tells adjacent phases apart, and a group that runs ahead of the other group's
                // k-block on the same stage would otherwise see the phase before last as "complete" and read a stale tile.
                mbar_wait(empty(s_t), ph_t ^ 1);
                mbar_wait(raw(s_t), ph_t);
#pragma unroll
                for (int i = 0; i < 8; ++i) {
                    const float4 q4 = ld_shared_v4(a_hi + (uint32_t)i * 2048u);
                    float v[4] = {q4.x, q4.y, q4.z, q4.w}, lo[4];
#pragma unroll
                    for (int e = 0; e < 4; ++e) {
                        float a = v[e];
                        if (AFF) {
                            a = fmaf(a, sc[e], sh[e]);              // scale/shift are 0 beyond Cin
                            if (RELU) a = fmaxf(a, 0.f);
                            a = ((live >> i) & 1u) ? a : 0.f;
                        } else if (RELU) {
                            a = fmaxf(a, 0.f);
                        }
                        v[e] = a;
                        lo[e] = a - __uint_as_float(__float_as_uint(a) & 0xffffe000u);   // exact; hi = what the tensor core reads
                    }
                    if (PRE != 0) st_shared_v4(a_hi + (uint32_t)i * 2048u, v[0], v[1], v[2], v[3]);
                    st_shared_v4(a_lo + (uint32_t)i * 2048u, lo[0], lo[1], lo[2], lo[3]);
                }
                fence_proxy_async();
                mbar_arrive(full_a(s_t));
                s_t += 2;
                if (s_t >= S) { s_t -= S; ph_t ^= 1; }
                kb += 2;
                while (kb >= KB) { kb -= KB; ++ti; }
            }
        } else {
        // ---- LOAD cursor: (tile iteration, k-block in tile) of the next k-block this group loads; this lane's channel
        //      quad of that k-block is g = 8 kb + chunk -> (tap, quad in tap) by multiply-shift division
        int oy[8], ox[8], rowoff[8];
        int l_ti = 0, l_kb = grp, cur_ti = -1;      // (KB may be smaller than G)
        while (l_kb >= KB) { l_kb -= KB; ++l_ti; }
        auto set_tile = [&](int ti) {
            cur_ti = ti;
            const int tile = (int)blockIdx.x + ti * (int)gridDim.x;
            const uint32_t m_tile = fdiv((uint32_t)tile, p.fd_ntiles);
            const uint32_t m_base = m_tile * BLOCK_M + (uint32_t)r0;
            const int nt = tile - (int)m_tile * p.n_tiles;
            const int cwin = p.kwin ? nt * p.n_tile / p.kwin * p.kwin : 0;     // first input channel of this n-tile's window
#pragma unroll
            for (int i = 0; i < 8; ++i) {
                const uint32_t m = m_base + 16u * i;
                if ((long long)m < p.M) {
                    const uint32_t q = fdiv(m, p.fd_wout);
                    const int x = (int)(m - q * (uint32_t)p.Wout);
                    const uint32_t b = fdiv(q, p.fd_hout);
                    const int y = (int)(q - b * (uint32_t)p.Hout);
                    oy[i] = y * p.stride - p.pad;
                    ox[i] = x * p.stride - p.pad;
                    rowoff[i] = (int)b * p.Hs * Ws * xs + (UP ? 0 : (oy[i] * Ws + ox[i]) * xs) + cwin;
                } else {
                    oy[i] = ox[i] = -0x40000000;   // never in bounds
                    rowoff[i] = 0;
                }
            }
        };
        // ---- load phase: this lane's 8 x 16-byte global loads of one k-block (predicated, branch-free)
        auto load_kb = [&](F4(&v)[8], uint32_t &mask, int &c_out) {
            if (l_ti != cur_ti) set_tile(l_ti);
            uint32_t g = (uint32_t)(l_kb * 8 + chunk);
            uint32_t tap = fdiv(g, p.fd_cq);
            if (p.chunk_major) {                   // (chunk, tap) order: one tap per k-block, the chunk advances every `taps` k-blocks
                const uint32_t kc = fdiv((uint32_t)l_kb, p.fd_taps);
                tap = (uint32_t)l_kb - kc * (uint32_t)taps;
                g = tap * (uint32_t)p.CQ + kc * 8u + (uint32_t)chunk;
            }
            const uint32_t ky = fdiv(tap, p.fd_kw);
            const int kx = (int)(tap - ky * (uint32_t)KW);
            const int dy = (int)ky * dil, dx = kx * dil;
            const bool cok = (int)tap < taps;      // quads past the last tap pad the final k-block
            const int c = cok ? (int)(g - tap * (uint32_t)p.CQ) * 4 : 0;   // first channel of this lane's 16-byte unit
            c_out = c;
            const int tapoff = UP ? c : (dy * Ws + dx) * xs + c;
            uint32_t mk = 0;
#pragma unroll
            for (int i = 0; i < 8; ++i) {
                const int yy = oy[i] + dy, xx = ox[i] + dx;
                bool ok = cok && (unsigned)yy < (unsigned)Hin && (unsigned)xx < (unsigned)Win;
                if (UP == 2) ok = ok && (((yy | xx) & 1) == 0);          // zero-stuffed source: odd coordinates are zeros
                mk |= (ok ? 1u : 0u) << i;
                int off;
                if (UP) off = rowoff[i] + ((yy >> 1) * Ws + (xx >> 1)) * xs + tapoff;
                else off = rowoff[i] + tapoff;
                if (VEC) {
                    float4 q = make_float4(0.f, 0.f, 0.f, 0.f);
                    if (ok) q = __ldg(reinterpret_cast<const float4 *>(xg + off));
                    v[i].v[0] = q.x; v[i].v[1] = q.y; v[i].v[2] = q.z; v[i].v[3] = q.w;
                } else {
#pragma unroll
                    for (int e = 0; e < 4; ++e) {
                        float q = 0.f;
                        if (ok && c + e < Cin) q = __ldg(xg + off + e);
                        v[i].v[e] = q;
                    }
                }
            }
            mask = mk;
            l_kb += G;
            while (l_kb >= KB) { l_kb -= KB; ++l_ti; }
        };
        // ---- store phase: wait for the stage, pre-op + hi/lo split in registers, swizzled 128-bit stores, publish.
        //      hi = fp32 rounded to tf32 (round-half-away on the 13 dropped bits, 2 integer ops); lo = x - hi is
        //      exact in fp32 and the tensor core reads its top 19 bits (error <= 2^-21 |x|).
        int s_s = grp;                             // stage of this group's next store (S >= 2)
        uint32_t s_ph = 0;
        while (s_s >= S) { s_s -= S; s_ph ^= 1; }
        auto store_kb = [&](F4(&v)[8], uint32_t mask, const int c) {
            const uint32_t a_hi = base + (uint32_t)s_s * stage_bytes + roff0;
            const uint32_t a_lo = a_hi + A_TILE_BYTES;
            const uint32_t bar_full = full_a(s_s);
            mbar_wait(empty(s_s), s_ph ^ 1);
            s_s += G;
            while (s_s >= S) { s_s -= S; s_ph ^= 1; }
            float sc[4], sh[4];
            if (AFF) {
                const float4 a4 = *reinterpret_cast<const float4 *>(s_scale + c);
                const float4 b4 = *reinterpret_cast<const float4 *>(s_shift + c);
                sc[0] = a4.x; sc[1] = a4.y; sc[2] = a4.z; sc[3] = a4.w;
                sh[0] = b4.x; sh[1] = b4.y; sh[2] = b4.z; sh[3] = b4.w;
            }
            if (VEC && c < Cin && c + 3 >= Cin) {
                // channel tail (Cin % 4 != 0, rows padded to 16 B): the float4 read past Cin -- zero those lanes
#pragma unroll
                for (int i = 0; i < 8; ++i)
#pragma unroll
                    for (int e = 1; e < 4; ++e)
                        if (c + e >= Cin) v[i].v[e] = 0.f;
            }
            // hi = fp32 rounded to tf32 (round-half-away on the 13 dropped bits, 2 integer ops); lo = x - hi is exact in fp32
            // and the tensor core reads its top 19 bits.  (Truncating instead of rounding saves one op per element but
            // makes lo one-signed: the dropped lo*lo term and lo's own truncation then add up coherently over K -- measured
            // 2-3x the error, past the 2e-5 bar of tests/test_conv_gpu.py -- so the rounding stays.  A per-tile tap-mask +
            // select-free interior path was also measured: more registers -> spills, fwd 27 -> 34 ms per K16 step.)
#pragma unroll
            for (int i = 0; i < 8; ++i) {
                const bool live = (mask >> i) & 1u;
                float hi[4], lo[4];
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    float a = v[i].v[e];
                    if (AFF) {
                        a = fmaf(a, sc[e], sh[e]);              // scale/shift are 0 beyond Cin
                        if (RELU) a = fmaxf(a, 0.f);
                        a = live ? a : 0.f;                     // zero padding is applied after the pre-op
                    } else if (RELU) {
                        a = fmaxf(a, 0.f);                      // padded lanes were loaded as 0
                    }
                    const float h = __uint_as_float((__float_as_uint(a) + 0x1000u) & 0xffffe000u);
                    hi[e] = h;
                    lo[e] = a - h;
                }
                st_shared_v4(a_hi + (uint32_t)i * 2048u, hi[0], hi[1], hi[2], hi[3]);
                st_shared_v4(a_lo + (uint32_t)i * 2048u, lo[0], lo[1], lo[2], lo[3]);
            }
            fence_proxy_async();               // generic-proxy writes -> visible to the tensor-core (async) proxy
            mbar_arrive(bar_full);
        };
        // ---- software pipeline (register ping-pong): the loads of this group's next k-block -- possibly of the next
        //      tile -- are in flight while the current one is transformed and stored
        const int mine = total_kb > grp ? (total_kb - grp + G - 1) / G : 0;   // k-blocks of this group
        if constexpr (G == 2) {
            F4 va[8], vb[8];
            uint32_t ma = 0, mb = 0;
            int ca = 0, cb = 0;
            int issued = 0;
            if (issued < mine) { load_kb(va, ma, ca); ++issued; }
            for (int done = 0; done < mine; done += 2) {
                if (issued < mine) { load_kb(vb, mb, cb); ++issued; }
                store_kb(va, ma, ca);
                if (done + 1 < mine) {
                    if (issued < mine) { load_kb(va, ma, ca); ++issued; }
                    store_kb(vb, mb, cb);
                }
            }
        } else {
            F4 va[8];
            uint32_t ma = 0;
            int ca = 0;
            for (int done = 0; done < mine; ++done) {
                load_kb(va, ma, ca);
                store_kb(va, ma, ca);
            }
        }
        }   // !TMA
    } else {
        // ===================== consumers: two warpgroups, rows [64 wg, 64 wg + 64) of every 128-pixel tile =========
        // 3xTF32: per k8 step A_lo*B_hi, A_hi*B_lo, A_hi*B_hi (small cross terms first).  The tensor cores accumulate one
        // k-block (4 k8 steps x 3 products) into `acc`; it is then added into the fp32 tile sum `tot` with round-to-nearest
        // adds, which keeps the accumulation error of long-K layers at the level of a plain fp32 sum.  The stage is handed
        // back to the loader / producers as soon as its wgmma group has completed.
        const int wg = warp >> 2;
        const int row = wg * 64 + (warp & 3) * 16 + (lane >> 2);     // rows row and row + 8 of the tile
        const int cq = (lane & 3) * 2;                               // columns 8 j + cq, 8 j + cq + 1
        const bool ovec = ((p.os & 1) == 0) && ((((uintptr_t)p.out) & 7) == 0);
        const bool single = p.precision != 0;
        auto consume = [&](auto NT) {
            constexpr int N = decltype(NT)::value;
            constexpr int R = N / 2;
            float acc[R], tot[R];
            const uint64_t dA0 = make_desc(base + (uint32_t)wg * (64u * 128u));      // A_hi of stage 0, this warpgroup's rows
            const uint64_t oAlo = (uint64_t)(A_TILE_BYTES >> 4);
            const uint64_t oBhi = (uint64_t)((2 * A_TILE_BYTES - wg * 64 * 128) >> 4);
            const uint64_t oBlo = oBhi + (uint64_t)((N * 128) >> 4), stage_step = (uint64_t)(stage_bytes >> 4);
            int s = 0;
            uint32_t ph = 0;
            uint64_t d = dA0;
            for (int ti = 0; ti < my_tiles; ++ti) {
                const int tile = (int)blockIdx.x + ti * (int)gridDim.x;
                const int m_tile = (int)fdiv((uint32_t)tile, p.fd_ntiles), nt = tile - m_tile * p.n_tiles;
#pragma unroll
                for (int i = 0; i < R; ++i) tot[i] = 0.f;
                for (int kb = 0; kb < KB; ++kb) {
                    mbar_wait(full_a(s), ph);
                    wgmma_fence();
                    const uint64_t dah = d, dal = d + oAlo, dbh = d + oBhi, dbl = d + oBlo;
#pragma unroll
                    for (int k = 0; k < BLOCK_K / 8; ++k) {
                        const uint32_t accumulate = k != 0;
                        if (single) {
                            Wgmma<N>::mma(acc, dah + 2 * k, dbh + 2 * k, accumulate);
                        } else {
                            Wgmma<N>::mma(acc, dal + 2 * k, dbh + 2 * k, accumulate);
                            Wgmma<N>::mma(acc, dah + 2 * k, dbl + 2 * k, 1);
                            Wgmma<N>::mma(acc, dah + 2 * k, dbh + 2 * k, 1);
                        }
                    }
                    wgmma_commit();
                    wgmma_wait<0>();
                    wgmma_fence_operands(acc);
                    __syncwarp();
                    if (lane == 0) mbar_arrive(empty(s));
#pragma unroll
                    for (int i = 0; i < R; ++i) tot[i] += acc[i];
                    d += stage_step;
                    if (++s == S) { s = 0; ph ^= 1; d = dA0; }
                }

                // ---- epilogue straight from the accumulator registers
                const long long m0 = (long long)m_tile * BLOCK_M + row, m1 = m0 + 8;
                float *orow0 = p.out + (m0 < p.M ? m0 : 0) * p.os + (long long)nt * n_tile;
                float *orow1 = p.out + (m1 < p.M ? m1 : 0) * p.os + (long long)nt * n_tile;
#pragma unroll
                for (int j = 0; j < N / 8; ++j) {
                    const int col = 8 * j + cq;
                    const int cabs = nt * n_tile + col;
#pragma unroll
                    for (int i = 0; i < 2; ++i) {
                        float o[2];
#pragma unroll
                        for (int c = 0; c < 2; ++c) {
                            float a = tot[4 * j + 2 * i + c];
                            if (p.act == 1) a = a > 0.f ? a : expm1f(a);
                            else if (p.act == 2) a = 1.0f / (1.0f + expf(-a));
                            o[c] = a;
                        }
                        if ((i ? m1 : m0) < p.M) {
                            float *orow = i ? orow1 : orow0;
                            if (ovec && cabs + 1 < p.Cout) {
                                *reinterpret_cast<float2 *>(orow + col) = make_float2(o[0], o[1]);
                            } else {
                                if (cabs < p.Cout) orow[col] = o[0];
                                if (cabs + 1 < p.Cout) orow[col + 1] = o[1];
                            }
                        }
                    }
                }
                if (p.stat_sum) {
                    // BatchNorm batch statistics of the tensor being produced (bts_bn_stats fused into its producer): column
                    // sums over the warp's 16 rows by a butterfly over the 8 row lanes, then per-warp fp64 partials per CTA.
                    // (host guarantees act == none here: the statistics are those of the raw conv output)
                    // With bnb_x set the two quantities are instead the BatchNorm-BACKWARD sums of the gradient tile.
#pragma unroll
                    for (int j = 0; j < N / 8; ++j) {
                        const int col = 8 * j + cq;
                        const int cabs = nt * n_tile + col;
#pragma unroll
                        for (int c = 0; c < 2; ++c) {
                            float s1 = 0.f, s2 = 0.f;
                            const int ch = cabs + c;
#pragma unroll
                            for (int i = 0; i < 2; ++i) {
                                const long long m = i ? m1 : m0;
                                if (m < p.M && ch < p.Cout) {
                                    const float g = tot[4 * j + 2 * i + c];
                                    if (p.bnb_x) {
                                        const float xv = __ldg(p.bnb_x + m * p.bnb_xs + ch);
                                        const float sc = __ldg(p.bnb_st + ch), sh = __ldg(p.bnb_st + p.Cout + ch);
                                        const float mu = __ldg(p.bnb_st + 2 * p.Cout + ch), is = __ldg(p.bnb_st + 3 * p.Cout + ch);
                                        const float y = fmaf(xv, sc, sh);
                                        const float gm = (!p.bnb_relu || y > 0.f) ? g : 0.f;
                                        s1 += gm;
                                        s2 += gm * ((xv - mu) * is);
                                    } else {
                                        s1 += g;
                                        s2 += g * g;
                                    }
                                }
                            }
#pragma unroll
                            for (int w = 4; w <= 16; w <<= 1) {
                                s1 += __shfl_xor_sync(0xffffffffu, s1, w);
                                s2 += __shfl_xor_sync(0xffffffffu, s2, w);
                            }
                            if (lane < 4 && ch < p.Cout) {                 // this (warp, lane) owns the slot: plain adds
                                double *mine = s_stat + (size_t)warp * 2 * n_tile;
                                mine[col + c] += (double)s1;
                                mine[n_tile + col + c] += (double)s2;
                            }
                        }
                    }
                }
                if (p.stat_sum && p.n_tiles > 1) {
                    // several N tiles per layer: the per-CTA partials belong to THIS tile's channel range -- flush them
                    // before the next tile (consumer warps only)
                    asm volatile("bar.sync 1, %0;" ::"n"(CONSUMER_THREADS) : "memory");
                    for (int c = (int)threadIdx.x; c < n_tile; c += CONSUMER_THREADS) {
                        const int ch = nt * n_tile + c;
                        double t1 = 0.0, t2 = 0.0;
                        for (int w = 0; w < STAT_SETS; ++w) {                // fixed order over the consumer warps
                            t1 += s_stat[(size_t)w * 2 * n_tile + c];
                            t2 += s_stat[(size_t)w * 2 * n_tile + n_tile + c];
                            s_stat[(size_t)w * 2 * n_tile + c] = 0.0;
                            s_stat[(size_t)w * 2 * n_tile + n_tile + c] = 0.0;
                        }
                        if (ch < p.Cout) {
                            atomicAdd(p.stat_sum + ch, t1);
                            atomicAdd(p.stat_sumsq + ch, t2);
                        }
                    }
                    asm volatile("bar.sync 1, %0;" ::"n"(CONSUMER_THREADS) : "memory");
                }
            }
        };
        switch (n_tile) {
            case 16: consume(std::integral_constant<int, 16>()); break;
            case 32: consume(std::integral_constant<int, 32>()); break;
            case 48: consume(std::integral_constant<int, 48>()); break;
            default:
                if constexpr (G == 2) consume(std::integral_constant<int, 64>());   // four groups run n_tile <= 48 only
                break;
        }
        if (p.stat_sum && p.n_tiles == 1) {
            asm volatile("bar.sync 1, %0;" ::"n"(CONSUMER_THREADS) : "memory");
            for (int c = (int)threadIdx.x; c < p.Cout; c += CONSUMER_THREADS) {
                double t1 = 0.0, t2 = 0.0;
                for (int w = 0; w < STAT_SETS; ++w) {                    // fixed order over the consumer warps
                    t1 += s_stat[(size_t)w * 2 * n_tile + c];
                    t2 += s_stat[(size_t)w * 2 * n_tile + n_tile + c];
                }
                atomicAdd(p.stat_sum + c, t1);
                atomicAdd(p.stat_sumsq + c, t2);
            }
        }
    }
}


}  // namespace

// ------------------------------------------------------------------------------------------- C ABI
extern "C" int bts_conv_n_tile(int Cout) {
    int n = (Cout + 15) / 16 * 16;
    if (n > MAX_N) {
        // split into equal tiles <= MAX_N, multiples of 16
        const int tiles = (n + MAX_N - 1) / MAX_N;
        n = ((Cout + tiles - 1) / tiles + 15) / 16 * 16;
    }
    return n;
}

extern "C" long long bts_conv_packed_floats(int n_rows, int k_channels, int KH, int KW) {
    const int n_tile = bts_conv_n_tile(n_rows);
    const int n_tiles = (n_rows + n_tile - 1) / n_tile;
    const int CQ = (k_channels + 3) / 4;
    const int KB = (KH * KW * CQ + 7) / 8;
    return (long long)n_tiles * KB * 2 * n_tile * 32;
}

extern "C" int bts_conv_pack_weights(const float *w, long long s_co, long long s_ci, long long s_kh, long long s_kw,
                                     int Cout, int Cin, int KH, int KW, int transpose_flip, int flags, float *wpack,
                                     void *stream) {
    if (!w || !wpack || Cout < 1 || Cin < 1 || KH < 1 || KW < 1) return BTS_EINVAL;
    if ((flags & 1) && ((transpose_flip ? Cout : Cin) % 32)) return BTS_EINVAL;      // chunk-major needs whole 32-channel chunks
    if (!bts_aligned16(wpack)) return BTS_EALIGN;
    const int rows = transpose_flip ? Cin : Cout;
    const int n_tile = bts_conv_n_tile(rows);
    const int n_tiles = (rows + n_tile - 1) / n_tile;
    const long long total = bts_conv_packed_floats(rows, transpose_flip ? Cout : Cin, KH, KW) / 2;
    long long grid = (total + 255) / 256;
    const long long cap = (long long)bts_num_sms() * 16;
    if (grid > cap) grid = cap;
    pack_weights_kernel<<<(int)grid, 256, 0, (cudaStream_t)stream>>>(w, s_co, s_ci, s_kh, s_kw, Cout, Cin, KH, KW,
                                                                    transpose_flip, wpack, n_tile, n_tiles, 0, 1, flags);
    BTS_LAUNCH_CHECK();
    return 0;
}

// Grouped convolution whose groups tile a 128-wide diagonal block (ResNeXt 3x3: width % kwin == 0, kwin % cpg == 0):
// w is (width, cpg, KH, KW); the packed operator has width/n_tile n-tiles of n_tile = bts_conv_group_n_tile(kwin) rows,
// each over the K window of kwin channels that holds its rows -- zeros outside the row's group.  Run with
// bts_conv_fwd_ex(kwin = bts_conv_group_window(width, cpg)).
extern "C" int bts_conv_group_window(int width, int cpg) {
    if (width < 1 || cpg < 1 || width % cpg) return 0;
    int k = 128;
    if (width % k || k % cpg) {
        // narrower windows for widths that are not multiples of 128: the largest multiple of lcm(16, cpg) dividing width
        k = 0;
        for (int c = 16; c <= 256 && c <= width; c += 16)
            if (width % c == 0 && c % cpg == 0) k = c;
    }
    return k;
}

// n-tile width of a grouped operator: the widest multiple of 16 <= MAX_N that divides the window
extern "C" int bts_conv_group_n_tile(int kwin) {
    if (kwin < 16 || kwin % 16) return 0;
    int n = MAX_N;
    while (kwin % n) n -= 16;
    return n;
}

extern "C" long long bts_conv_packed_floats_grouped(int width, int cpg, int KH, int KW) {
    const int kwin = bts_conv_group_window(width, cpg);
    if (!kwin) return 0;
    const int CQ = kwin / 4;
    const int KB = (KH * KW * CQ + 7) / 8;
    const int nt = bts_conv_group_n_tile(kwin);
    return (long long)(width / nt) * KB * 2 * nt * 32;
}

extern "C" int bts_conv_pack_weights_grouped(const float *w, long long s_co, long long s_ci, long long s_kh, long long s_kw,
                                             int width, int cpg, int KH, int KW, int transpose_flip, int flags,
                                             float *wpack, void *stream) {
    if (!w || !wpack || KH < 1 || KW < 1) return BTS_EINVAL;
    const int kwin = bts_conv_group_window(width, cpg);
    if (!kwin) return BTS_EINVAL;
    if (!bts_aligned16(wpack)) return BTS_EALIGN;
    const long long total = bts_conv_packed_floats_grouped(width, cpg, KH, KW) / 2;
    long long grid = (total + 255) / 256;
    const long long cap = (long long)bts_num_sms() * 16;
    if (grid > cap) grid = cap;
    pack_weights_kernel<<<(int)grid, 256, 0, (cudaStream_t)stream>>>(w, s_co, s_ci, s_kh, s_kw, width, width, KH, KW,
                                                                    transpose_flip, wpack, bts_conv_group_n_tile(kwin),
                                                                    width / bts_conv_group_n_tile(kwin), kwin, cpg, flags);
    BTS_LAUNCH_CHECK();
    return 0;
}

// ---- TMA tensor map of the NHWC activation tensor, im2col mode (cuTensorMapEncodeIm2col through the runtime's driver
//      entry-point query: no link-time dependency on libcuda)
static int g_producer_groups = 0;   // 0 / 4: four groups where the ring has >= 4 stages, 2: always two
static int g_tma_mode = 0;      // 0 off, 1 on, 2 on with base-pixel coordinates NOT shifted by the lower corner, 3 on + strict

typedef CUresult (*EncodeIm2colFn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *, const cuuint64_t *,
                                   const int *, const int *, cuuint32_t, cuuint32_t, const cuuint32_t *, CUtensorMapInterleave,
                                   CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeIm2colFn encode_im2col_fn() {
    static EncodeIm2colFn fn = nullptr;
    static bool tried = false;
    if (!tried) {
        tried = true;
        void *ptr = nullptr;
        cudaDriverEntryPointQueryResult qres;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeIm2col", &ptr, cudaEnableDefault, &qres) == cudaSuccess &&
            qres == cudaDriverEntryPointSuccess)
            fn = reinterpret_cast<EncodeIm2colFn>(ptr);
    }
    return fn;
}

// x: NHWC fp32, pixel stride xs floats (a channel slice of a wider slab is fine), C channels visible to the loads
static int make_im2col_map(CUtensorMap *map, const float *x, long long xs, int B, int H, int W, int C, int KH, int KW, int pad,
                           int dil) {
    EncodeIm2colFn fn = encode_im2col_fn();
    if (!fn) return BTS_EINVAL;
    const cuuint64_t gdim[4] = {(cuuint64_t)C, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)B};
    const cuuint64_t gstr[3] = {(cuuint64_t)xs * 4, (cuuint64_t)xs * 4 * W, (cuuint64_t)xs * 4 * W * H};
    const int lower[2] = {-pad, -pad};                                        // bounding box lower corner (W, H)
    const int upper[2] = {pad - dil * (KW - 1), pad - dil * (KH - 1)};        // upper corner: last base pixel = last output pixel
    const cuuint32_t estr[4] = {1, 1, 1, 1};
    const CUresult r = fn(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, const_cast<float *>(x), gdim, gstr, lower, upper,
                          /*channelsPerPixel=*/32, /*pixelsPerColumn=*/BLOCK_M, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                          CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    return r == CUDA_SUCCESS ? 0 : 700 + (int)r;
}

// 0: activation tiles loaded by the producer warps (LDG); 1: staged by TMA where eligible; 2: bring-up variant of 1
extern "C" int bts_conv_set_tma(int mode) {
    if (mode < 0 || mode > 3) return BTS_EINVAL;
    g_tma_mode = mode;
    return 0;
}
extern "C" int bts_conv_get_tma(void) { return g_tma_mode; }
extern "C" int bts_conv_set_producer_groups(int g) {
    if (g != 0 && g != 2 && g != 4) return BTS_EINVAL;
    g_producer_groups = g;
    return 0;
}


struct BnBwdArgs {
    const float *x; long long xs; const float *st; int relu;
};

static int conv_fwd_impl(const float *x, long long x_pixel_stride, int B, int Hs, int Ws, int upsample2, int out_h,
                         int out_w, int kwin, int Cin,
                         int KH, int KW, int stride, int pad, int dil, const float *wpack, int Cout,
                         const float *pre_scale, const float *pre_shift, int pre_relu, float *out,
                         long long out_pixel_stride, int act, int precision, double *stat_sum, double *stat_sumsq,
                         void *stream, const BnBwdArgs *bnb = nullptr, int flags = 0) {
    if (!x || !wpack || !out || B < 0 || Hs < 1 || Ws < 1 || Cin < 1 || Cout < 1 || KH < 1 || KW < 1 || stride < 1 ||
        pad < 0 || dil < 1)
        return BTS_EINVAL;
    if ((pre_scale == nullptr) != (pre_shift == nullptr)) return BTS_EINVAL;
    if (pre_scale && Cin > MAX_CIN_SMEM) return BTS_EINVAL;
    if (act < 0 || act > 2 || precision < 0 || precision > 1) return BTS_EINVAL;
    if (upsample2 < 0 || upsample2 > 2 || kwin < 0) return BTS_EINVAL;
    if (upsample2 == 2 && (stride != 1 || out_h < 1 || out_w < 1)) return BTS_EINVAL;
    if (kwin && (pre_scale || Cin % kwin || Cout % kwin)) return BTS_EINVAL;   // whole windows; no pre-op on grouped convs
    if (!bts_aligned16(wpack)) return BTS_EALIGN;
    if (B == 0) return 0;
    if ((long long)B * Hs * Ws * x_pixel_stride >= 0x7fffffffLL) return BTS_EINVAL;   // 32-bit element offsets
    ConvParams p;
    p.x = x; p.xs = x_pixel_stride; p.B = B; p.Hs = Hs; p.Ws = Ws; p.up = upsample2; p.Cin = kwin ? kwin : Cin;
    p.kwin = kwin;
    p.KH = KH; p.KW = KW; p.stride = stride; p.pad = pad; p.dil = dil;
    p.wpack = wpack; p.Cout = Cout;
    if (kwin % 16) return BTS_EINVAL;
    p.n_tile = kwin ? bts_conv_group_n_tile(kwin) : bts_conv_n_tile(Cout);
    p.n_tiles = (Cout + p.n_tile - 1) / p.n_tile;
    p.pre_scale = pre_scale; p.pre_shift = pre_shift; p.pre_relu = pre_relu ? 1 : 0;
    p.out = out; p.os = out_pixel_stride; p.act = act; p.precision = precision;
    p.stat_sum = stat_sum; p.stat_sumsq = stat_sumsq;
    if ((stat_sum == nullptr) != (stat_sumsq == nullptr)) return BTS_EINVAL;
    p.bnb_x = nullptr; p.bnb_xs = 0; p.bnb_st = nullptr; p.bnb_relu = 0;
    if (bnb) {
        if (!bnb->x || !bnb->st || !stat_sum || act != 0) return BTS_EINVAL;
        p.bnb_x = bnb->x; p.bnb_xs = bnb->xs; p.bnb_st = bnb->st; p.bnb_relu = bnb->relu ? 1 : 0;
    }
    if (stat_sum && act != 0) return BTS_EINVAL;                        // statistics of the raw conv output only
    const int Hin = p.up ? 2 * Hs : Hs, Win = p.up ? 2 * Ws : Ws;
    p.Hv = Hin; p.Wv = Win;      // mode 2: live source coordinates are the even ones below 2Hs x 2Ws, zeros everywhere else
    p.Hout = p.up == 2 ? out_h : (Hin + 2 * pad - dil * (KH - 1) - 1) / stride + 1;
    p.Wout = p.up == 2 ? out_w : (Win + 2 * pad - dil * (KW - 1) - 1) / stride + 1;
    if (p.Hout < 1 || p.Wout < 1) return BTS_EINVAL;
    p.M = (long long)B * p.Hout * p.Wout;
    p.KC = (p.Cin + 31) / 32;
    p.CQ = (p.Cin + 3) / 4;
    p.KB = (KH * KW * p.CQ + 7) / 8;
    p.fd_cq = make_fastdiv((uint32_t)p.CQ);
    p.fd_kw = make_fastdiv((uint32_t)KW);
    p.vec_ok = bts_aligned16(x) && (x_pixel_stride % 4 == 0);
    const long long m_tiles = (p.M + BLOCK_M - 1) / BLOCK_M;
    if (m_tiles * p.n_tiles * (long long)p.KB > 0x7fffffffLL || p.M + BLOCK_M >= 0x7fffffffLL) return BTS_EINVAL;
    p.m_tiles = (int)m_tiles;
    p.total_tiles = (int)(m_tiles * p.n_tiles);
    p.fd_wout = make_fastdiv((uint32_t)p.Wout);
    p.fd_hout = make_fastdiv((uint32_t)p.Hout);
    p.fd_ntiles = make_fastdiv((uint32_t)p.n_tiles);
    const int pre = (pre_scale ? 2 : 0) | (p.pre_relu ? 1 : 0);
    // shared-memory plan: stage = A hi/lo (2 x 16 KB) + B hi/lo (2 x n_tile x 128 B); as many stages as fit
    p.stage_bytes = 2 * A_TILE_BYTES + 2 * p.n_tile * 128;
    const int pre_bytes = pre >= 2 ? p.KC * 32 * 8 : 0;
    const int stat_bytes = stat_sum ? STAT_SETS * 2 * p.n_tile * 8 : 0;
    p.stages = (SMEM_LIMIT - 1024 - BAR_BYTES - pre_bytes - stat_bytes) / p.stage_bytes;
    if (p.stages > MAX_STAGES) p.stages = MAX_STAGES;
    if (p.stages < 2) return BTS_EINVAL;
    p.chunk_major = (flags & 1) ? 1 : 0;
    if (p.chunk_major && ((p.Cin % 32) || p.up)) return BTS_EINVAL;
    if (p.chunk_major && p.stages > 3) p.stages = 3;   // leave most of the SM's 228 KB to L1: consecutive k-blocks of a chunk
                                                        // re-read the same pixels' lines shifted by one tap
    const int smem = p.stages * p.stage_bytes + pre_bytes + BAR_BYTES + stat_bytes + 1024;
    const int sms = bts_num_sms();
    dim3 grid((unsigned)(p.total_tiles < sms ? p.total_tiles : sms));
    const bool vec = p.vec_ok;      // aligned base + pixel stride % 4 == 0 (a channel tail is masked in-kernel)
    cudaError_t err = cudaSuccess;
    // ---- TMA-staged activation tiles (see the kernel's TMA template parameter): stride-1, non-up-sampled layers whose K
    //      channels are a multiple of 32 (dense-quad K order == per-tap 32-channel chunks) and whose rows are 16-byte aligned
    CUtensorMap tmap;
    memset(&tmap, 0, sizeof(tmap));
    bool use_tma = false;
    p.tma_adj = 0;
    p.fd_taps = make_fastdiv((uint32_t)(KH * KW));
    p.fd_kc = make_fastdiv((uint32_t)p.KC);
    if (g_tma_mode != 0 && !p.chunk_major && p.up == 0 && stride == 1 && p.vec_ok && (p.Cin % 32) == 0 && pad <= 127 &&
        dil * (KH - 1) - pad <= 128 && dil * (KW - 1) - pad <= 128 && dil * (KH - 1) <= 255 && dil * (KW - 1) <= 255) {
        const int rc = make_im2col_map(&tmap, x, x_pixel_stride, B, Hs, Ws, kwin ? Cin : p.Cin, KH, KW, pad, dil);
        if (rc == 0) {
            use_tma = true;
            p.tma_adj = g_tma_mode == 2 ? 0 : pad;      // mode 2: alternative coordinate convention (bring-up switch)
        } else if (g_tma_mode == 3) {
            return rc;                                   // forced: report why the map could not be built
        }
    }
    // four producer groups on the narrow layers (n_tile <= 48), where producing the activation tile, not the tensor
    // cores, sets the k-block time; the 800-thread CTA leaves no registers for a wider accumulator
    const bool four = !use_tma && p.stages >= 4 && p.n_tile <= FOUR_GROUPS_MAX_N && g_producer_groups != 2;
#define BTS_LAUNCH_G(PRE, UP, VEC, TMA, G)                                                                         \
    do {                                                                                                           \
        static bool attr_set_[BTS_MAX_DEVICES] = {};                                                               \
        bool &attr_set = attr_set_[bts_cur_device()];                                                              \
        if (!attr_set) {                                                                                           \
            err = cudaFuncSetAttribute(conv_tc_kernel<PRE, UP, VEC, TMA, G>, cudaFuncAttributeMaxDynamicSharedMemorySize, \
                                       SMEM_LIMIT);                                                                \
            if (err != cudaSuccess) return (int)err;                                                               \
            attr_set = true;                                                                                       \
        }                                                                                                          \
        conv_tc_kernel<PRE, UP, VEC, TMA, G><<<grid, CONSUMER_THREADS + 32 + 128 * G, smem, (cudaStream_t)stream>>>(p, tmap);         \
    } while (0)
#define BTS_LAUNCH(PRE, UP, VEC, TMA)                                                                              \
    do {                                                                                                           \
        if (four && VEC && !TMA) BTS_LAUNCH_G(PRE, UP, true, false, 4);                                            \
        else BTS_LAUNCH_G(PRE, UP, VEC, TMA, 2);                                                                   \
    } while (0)
#define BTS_DISPATCH_UV(PRE)                                  \
    do {                                                      \
        if (use_tma) BTS_LAUNCH(PRE, 0, true, true);                                                            \
        else if (p.up == 2) { if (vec) BTS_LAUNCH(PRE, 2, true, false); else BTS_LAUNCH(PRE, 2, false, false); }    \
        else if (p.up) { if (vec) BTS_LAUNCH(PRE, 1, true, false); else BTS_LAUNCH(PRE, 1, false, false); }    \
        else { if (vec) BTS_LAUNCH(PRE, 0, true, false); else BTS_LAUNCH(PRE, 0, false, false); }              \
    } while (0)
    switch (pre) {
        case 0: BTS_DISPATCH_UV(0); break;
        case 1: BTS_DISPATCH_UV(1); break;
        case 2: BTS_DISPATCH_UV(2); break;
        default: BTS_DISPATCH_UV(3); break;
    }
#undef BTS_DISPATCH_UV
#undef BTS_LAUNCH
#undef BTS_LAUNCH_G
    BTS_LAUNCH_CHECK();
    return 0;
}

extern "C" int bts_conv_fwd(const float *x, long long x_pixel_stride, int B, int Hs, int Ws, int upsample2, int Cin,
                            int KH, int KW, int stride, int pad, int dil, const float *wpack, int Cout,
                            const float *pre_scale, const float *pre_shift, int pre_relu, float *out,
                            long long out_pixel_stride, int act, int precision, void *stream) {
    return conv_fwd_impl(x, x_pixel_stride, B, Hs, Ws, upsample2 ? 1 : 0, 0, 0, 0, Cin, KH, KW, stride, pad, dil, wpack, Cout,
                         pre_scale, pre_shift, pre_relu, out, out_pixel_stride, act, precision, nullptr, nullptr, stream);
}

extern "C" int bts_conv_fwd_stats(const float *x, long long x_pixel_stride, int B, int Hs, int Ws, int upsample2, int Cin,
                                  int KH, int KW, int stride, int pad, int dil, const float *wpack, int Cout,
                                  const float *pre_scale, const float *pre_shift, int pre_relu, float *out,
                                  long long out_pixel_stride, int act, int precision, double *stat_sum,
                                  double *stat_sumsq, void *stream) {
    if (!stat_sum || !stat_sumsq) return BTS_EINVAL;
    return conv_fwd_impl(x, x_pixel_stride, B, Hs, Ws, upsample2 ? 1 : 0, 0, 0, 0, Cin, KH, KW, stride, pad, dil, wpack, Cout,
                         pre_scale, pre_shift, pre_relu, out, out_pixel_stride, act, precision, stat_sum, stat_sumsq, stream);
}

// General entry point: everything bts_conv_fwd does, plus
//   source_mode 2: the source is the zero-stuffed x2 expansion of x (value at (2i,2j) = x[i,j], zeros elsewhere) and the
//       output has the given out_h x out_w -- with the transposed, tap-flipped packed operator and pad' = dil*(K-1) - pad
//       this is the input gradient of a STRIDE-2 convolution whose input was out_h x out_w (ResNet / ResNeXt stages,
//       pytorch/bts.py:282-296 via torchvision); call with stride = 1;
//   kwin > 0: block-diagonal ("grouped") operator: output channels [nt*kwin, (nt+1)*kwin) only see input channels
//       [nt*kwin, (nt+1)*kwin) (ResNeXt 3x3 convs, 32 groups: groups are packed kwin/cpg to a 128-wide diagonal block,
//       see bts_conv_pack_weights_grouped); Cin and Cout are the layer's total channel counts.
extern "C" int bts_conv_fwd_ex(const float *x, long long x_pixel_stride, int B, int Hs, int Ws, int source_mode, int out_h,
                               int out_w, int kwin, int Cin, int KH, int KW, int stride, int pad, int dil,
                               const float *wpack, int Cout, const float *pre_scale, const float *pre_shift, int pre_relu,
                               float *out, long long out_pixel_stride, int act, int precision, double *stat_sum,
                               double *stat_sumsq, int flags, void *stream) {
    return conv_fwd_impl(x, x_pixel_stride, B, Hs, Ws, source_mode, out_h, out_w, kwin, Cin, KH, KW, stride, pad, dil, wpack,
                         Cout, pre_scale, pre_shift, pre_relu, out, out_pixel_stride, act, precision, stat_sum, stat_sumsq,
                         stream, nullptr, flags);
}

// descs: device array of n PackDesc (layout above; built by the host side once per model), total = sum of packed_floats / 2
extern "C" int bts_conv_pack_weights_multi(const void *descs, int n, long long total, void *stream) {
    if (!descs || n < 1 || total < 1) return BTS_EINVAL;
    long long grid = (total + 255) / 256;
    const long long cap = (long long)bts_num_sms() * 16;
    if (grid > cap) grid = cap;
    pack_weights_multi_kernel<<<(int)grid, 256, 0, (cudaStream_t)stream>>>(reinterpret_cast<const PackDesc *>(descs), n, total);
    BTS_LAUNCH_CHECK();
    return 0;
}

// dgrad whose epilogue also reduces the BatchNorm(+ReLU) backward sums of the layer in front of the conv: the tile written
// is g = dL/d[relu](bn(x_bn)); S1[c] += sum_p g*mask, S2[c] += sum_p g*mask*xhat with mask = [bn(x)>0] (relu) or 1,
// xhat = (x - mean)*invstd.  x_bn: the BatchNorm INPUT at the output's pixels/channels (NHWC, pixel stride x_bn_stride),
// bn_st: [4][Cout] = scale, shift, mean, invstd (bts_bn_finalize layout).  S1/S2 must be zeroed.  Replaces the separate
// bts_bn_relu_bwd_reduce pass over (x, g) -- 174 launches and two full tensor reads per DenseNet-161 step.
extern "C" int bts_conv_fwd_bnbwd(const float *x, long long x_pixel_stride, int B, int Hs, int Ws, int source_mode, int out_h,
                                  int out_w, int kwin, int Cin, int KH, int KW, int stride, int pad, int dil,
                                  const float *wpack, int Cout, float *out, long long out_pixel_stride, int precision,
                                  const float *x_bn, long long x_bn_stride, const float *bn_st, int relu, double *S1,
                                  double *S2, int flags, void *stream) {
    BnBwdArgs a{x_bn, x_bn_stride, bn_st, relu};
    return conv_fwd_impl(x, x_pixel_stride, B, Hs, Ws, source_mode, out_h, out_w, kwin, Cin, KH, KW, stride, pad, dil, wpack,
                         Cout, nullptr, nullptr, 0, out, out_pixel_stride, 0, precision, S1, S2, stream, &a, flags);
}
