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
// GEMM view: M = B*Hout*Wout pixels (128 per CTA tile: two warpgroups of 64 rows), N = Cout (<= 128 per tile, equal
// tiles in multiples of 16: the k-block accumulator and the tile sum of a 64 x 128 warpgroup tile are 128 registers per
// thread), K = the dense sequence of 16-byte channel quads, tap-major, in blocks of 32 fp32 (one 128-byte swizzled row per
// pixel).
// Precision: fp32 operands are split x = hi + lo with hi = x rounded to tf32, lo = x - hi and the tile accumulates
// A_lo*B_hi + A_hi*B_lo + A_hi*B_hi  with tf32 wgmma into fp32 register accumulators (error ~2^-21 per product:
// fp32-grade, SURVEY Appendix F); every k-block's tensor-core sum is added into the tile sum with round-to-nearest fp32
// adds.  The weights are split once, when they are packed; the activations are split by the consumers in registers.
// Single-pass TF32 (precision=1, opt-in) runs conv_tf32_kernel, the same body compiled for one product: A and B_hi
// only, A_hi*B_hi per k8 step.  Its stage is A + B_hi (the producers' bulk copy fetches only the hi half of each packed
// k-block), so more stages fit; the k-block order, the tile sum and the epilogue are those of conv_tc_kernel.
//
// Persistent kernel: grid = min(#tiles, #SMs); every CTA walks tiles blockIdx.x, +gridDim.x, ... with the smem stage
// ring and all warp roles running continuously across tile boundaries (the producers fill the stages of tile t+1 while
// the consumers run the epilogue of tile t; no per-tile launch or pipeline-fill cost).
// Warp roles (512 threads = 16 warps launched with 128 registers per thread, 1 CTA/SM; setmaxnreg then moves registers
// from the producers, which keep 80, to the consumers, which get 176):
//   warps 0..7  : two consumer warpgroups -- per k-block, each thread loads its A fragments (fp32) from the swizzled tile,
//                 splits them into hi/lo in registers and issues register-A wgmma against the B hi/lo tiles in shared
//                 memory; then the epilogue from the accumulator registers: activation, NHWC stores, optional BatchNorm
//                 batch statistics of the output;
//   warps 8..15 : two producer groups (alternating k-blocks).  One lane of the group filling a k-block streams its
//                 pre-packed, pre-split, pre-swizzled weight tile with a 1-D bulk async copy (cp.async.bulk) completing on
//                 the stage's mbarrier; the group's threads copy the activation tile from global memory straight into its
//                 swizzled slots with 16-byte cp.async (8 lanes cover one pixel's 128 B; padding is zero-filled), whose
//                 completion is their arrival on the stage's mbarrier; with a BatchNorm / ReLU pre-op they wait for the
//                 copies and apply it in place first.
// Staging A as fp32 and splitting it in the consumers keeps shared-memory traffic per k-block at one A tile written and
// read once (A from shared memory through descriptors would be read by each of the three products).
#include <cstdio>
#include <cstdlib>
#include <type_traits>

#include "tc_common.cuh"

namespace {

constexpr int BLOCK_M = 128;
constexpr int BLOCK_K = 32;                 // fp32 elements per k-block = one 128-byte row
constexpr int MAX_N = 128;                  // output channels per tile (two register accumulators per consumer thread)
constexpr int A_TILE_BYTES = BLOCK_M * 128; // 16 KB of fp32 activations
constexpr int CONSUMER_THREADS = 256;       // two warpgroups
constexpr int PRODUCER_THREADS = 128;       // per group
constexpr int NUM_THREADS = CONSUMER_THREADS + 2 * PRODUCER_THREADS;   // 16 warps: 128 registers per thread
// registers per thread after the warpgroups' reallocation (setmaxnreg): the producers hand theirs to the consumers, whose
// k-block accumulator, tile sum and A fragments are 64 + 64 + 32 registers at N = 128
constexpr int PRODUCER_REGS = 80;
constexpr int CONSUMER_REGS = 176;
static_assert(CONSUMER_THREADS * CONSUMER_REGS + 2 * PRODUCER_THREADS * PRODUCER_REGS <= NUM_THREADS * 128,
              "the reallocation must fit the registers the CTA was launched with");
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
    int vec_ok;              // 16-byte aligned rows -> float4 loads
    long long M;             // B*Hout*Wout
    int m_tiles, total_tiles;
    int KC;                  // ceil(Cin/32): 32-channel chunks of the pre-op scale/shift staged in smem
    int CQ;                  // ceil(Cin/4): 16-byte channel quads per tap (dense-K order, see the pack kernel)
    int KB;                  // ceil(KH*KW*CQ / 8) k-blocks
    tc::FastDiv fd_cq, fd_kw;
    double *stat_sum, *stat_sumsq;   // optional per-output-channel sum / sum of squares of the (activated) output
    // BatchNorm-backward reduction fused into a dgrad's epilogue (bnb_x != null): the tile being written is g = dL/d relu(bn(x));
    // stat_sum[c] += sum_p g*[bn(x)>0],  stat_sumsq[c] += sum_p g*[bn(x)>0]*xhat   (bts_bn_bwd_reduce without its pass)
    const float *bnb_x; long long bnb_xs;
    const float *bnb_st;             // [4][Cout]: scale, shift, mean, invstd
    int bnb_relu;
    int stages, stage_bytes; // smem ring: as many (A + B hi/lo, single pass: A + B hi) stages as fit
    tc::FastDiv fd_wout, fd_hout, fd_ntiles;
    // split-K: the grid is splits x vgrid CTAs; CTA b runs split s = b / vgrid over tiles b - s * vgrid, + vgrid, ... and
    // streams the kb_split k-blocks [s * kb_split, (s + 1) * kb_split) of each; its epilogue stores the raw tile sum at
    // out + s * split_stride (the workspace).  The last split's k-blocks past KB lie past the last tap: their A tile is
    // zero-filled like any quad past the last tap and their weight tile index is clamped to w_last (finite values times
    // zeros leave the tile sum unchanged).  Without split-K: splits = 1, vgrid = the grid, kb_split = KB, split_stride = 0.
    int splits, kb_split, vgrid, w_last;
    long long split_stride;
    tc::FastDiv fd_vgrid;
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
                                         float *__restrict__ wpack, int n_tile, int kwin, int cpg, long long idx) {
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
    const int tap = g / CQ;
    const int ch = (g - tap * CQ) * 4 + (kk & 3);
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
                                                           int n_tile, int n_tiles, int kwin, int cpg) {
    const int Kch = kwin ? kwin : (transpose_flip ? Cout : Cin);
    const int KB = (KH * KW * ((Kch + 3) / 4) + 7) / 8;
    const long long total = (long long)n_tiles * KB * n_tile * 32;
    for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
         idx += (long long)gridDim.x * blockDim.x)
        pack_one(w, s_co, s_ci, s_kh, s_kw, Cout, Cin, KH, KW, transpose_flip, wpack, n_tile, kwin, cpg, idx);
}

// every packed operator of a model in ONE launch (after an optimizer step: 394 launches -> 1 for DenseNet-161 + decoder)
struct PackDesc {
    const float *w;
    float *wpack;
    long long s_co, s_ci, s_kh, s_kw;
    long long start;                     // first global index of this operator (prefix sum of packed_floats / 2)
    int Cout, Cin, KH, KW, transpose_flip, n_tile, n_tiles, kwin, cpg;
    int pad_;                            // explicit padding (written as 0)
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
                 q.cpg, idx - q.start);
    }
}

// ------------------------------------------------------------------------------------------- main kernel
// dynamic smem, 1024-byte aligned base:
//   [S stages][A 16K | B_hi n_tile*128 | B_lo n_tile*128]   S = as many stages as fit (2..MAX_STAGES)
//   (single pass: [A 16K | B_hi n_tile*128] per stage)
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
// SINGLE: single-pass TF32 (conv_tf32_kernel) instead of 3xTF32 (conv_tc_kernel).
template <int PRE, int UP, bool VEC, bool SINGLE>
__device__ __forceinline__ void conv_body(const ConvParams &p) {
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
    // bars: [0..MS) full (the filling group's 128 producer arrivals + its expect_tx arrival for the weight bytes),
    // [MS..2MS) spare, [2MS..3MS) empty (one arrival per consumer warp).  The spare set is initialised like the others:
    // without those instructions ptxas places the consumers' k-block loops 208 bytes earlier, and that placement measured
    // 2-7 % slower on the wide-tile dgrad layers (H100 SXM, 700 W), with identical loop bodies.
    const uint32_t bar0 = base + bar_off;
    auto full = [&](int s) { return bar0 + 8u * s; };
    auto spare = [&](int s) { return bar0 + 8u * (MAX_STAGES + s); };
    auto empty = [&](int s) { return bar0 + 8u * (2 * MAX_STAGES + s); };
    double *s_stat = reinterpret_cast<double *>(sm + bar_off + BAR_BYTES);    // [8 warps][2][n_tile], only when p.stat_sum

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int n_tile = p.n_tile;
    const int KB = p.KB;
    if (p.stat_sum)
        for (int i = threadIdx.x; i < STAT_SETS * 2 * n_tile; i += NUM_THREADS) s_stat[i] = 0.0;
    // tiles of this CTA: t0, t0 + vgrid, ...   (tile -> m_tile = tile / n_tiles, nt = tile % n_tiles), all of split s.
    // s and t0 are recomputed from %ctaid where they are used (volatile: not hoisted), so they hold no register across
    // the k-block loops, where the producers have none to spare.
    auto cta_split = [&]() {
        uint32_t b;
        asm volatile("mov.u32 %0, %%ctaid.x;" : "=r"(b));
        return (int)fdiv(b, p.fd_vgrid);
    };
    auto cta_tile0 = [&]() {
        uint32_t b;
        asm volatile("mov.u32 %0, %%ctaid.x;" : "=r"(b));
        return (int)b - (int)fdiv(b, p.fd_vgrid) * p.vgrid;
    };
    const int my_tiles = (p.total_tiles - cta_tile0() + p.vgrid - 1) / p.vgrid;

    if (threadIdx.x == 0) {
        for (int s = 0; s < S; ++s) {
            mbar_init(full(s), PRODUCER_THREADS + 1);
            mbar_init(spare(s), 1);
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

    if (threadIdx.x >= CONSUMER_THREADS) {
        // ===================== producers (two groups x 4 warps, alternating k-blocks) =====================
        setmaxnreg_dec<PRODUCER_REGS>();
        // The group that fills a k-block also stages its weight tile: right after the stage has been released, one lane
        // issues the 1-D bulk async copy (cp.async.bulk) of the pre-packed, pre-split, pre-swizzled B hi/lo rows,
        // completing on an mbarrier.
        const int total_kb = my_tiles * p.kb_split;        // host guarantees < 2^31
        const int pt = threadIdx.x - CONSUMER_THREADS;
        const int grp = pt / PRODUCER_THREADS;     // producer group: global k-blocks gk == grp (mod 2)
        const int t = pt % PRODUCER_THREADS;
        const bool issuer = t == 0;
        const uint32_t wstride = 2u * (uint32_t)n_tile * 128u;           // one packed k-block: [hi | lo] rows
        const uint32_t wbytes = SINGLE ? wstride / 2u : wstride;          // single pass: the hi half only
        const uint8_t *wsrc = reinterpret_cast<const uint8_t *>(p.wpack);
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
        const int gq0 = chunk + 8 * p.kb_split * cta_split();    // this lane's channel quad in the split's first k-block
        // ---- cursor: (tile iteration, k-block in tile) of the next k-block this group fills; this lane's channel quad of
        //      that k-block is g = 8 kb + chunk -> (tap, quad in tap) by multiply-shift division
        // oyx[i]: the row's top-left source coordinate, (oy << 16) | (ox & 0xffff) -- one register per row instead of two
        // (host: |coordinates| < 2^14)
        int oyx[8], rowoff[8];
        // l_kb counts the k-blocks of the split (kb_split per tile); cur_w = the weight tile of the split's first k-block
        int l_ti = 0, l_kb = grp, cur_ti = -1, cur_w = 0;       // (kb_split may be 1)
        while (l_kb >= p.kb_split) { l_kb -= p.kb_split; ++l_ti; }
        auto set_tile = [&](int ti) {
            cur_ti = ti;
            const int tile = cta_tile0() + ti * p.vgrid;
            const uint32_t m_tile = fdiv((uint32_t)tile, p.fd_ntiles);
            const uint32_t m_base = m_tile * BLOCK_M + (uint32_t)r0;
            const int nt = tile - (int)m_tile * p.n_tiles;
            cur_w = nt * KB + p.kb_split * cta_split();
            const int cwin = p.kwin ? nt * p.n_tile / p.kwin * p.kwin : 0;     // first input channel of this n-tile's window
#pragma unroll
            for (int i = 0; i < 8; ++i) {
                const uint32_t m = m_base + 16u * i;
                if ((long long)m < p.M) {
                    const uint32_t q = fdiv(m, p.fd_wout);
                    const int x = (int)(m - q * (uint32_t)p.Wout);
                    const uint32_t b = fdiv(q, p.fd_hout);
                    const int y = (int)(q - b * (uint32_t)p.Hout);
                    const int oy = y * p.stride - p.pad, ox = x * p.stride - p.pad;
                    oyx[i] = (int)(((uint32_t)oy << 16) | ((uint32_t)ox & 0xffffu));
                    rowoff[i] = (int)b * p.Hs * Ws * xs + (UP ? 0 : (oy * Ws + ox) * xs) + cwin;
                } else {
                    oyx[i] = (int)0xc000c000u;     // (-0x4000, -0x4000): never in bounds
                    rowoff[i] = 0;
                }
            }
        };
        // ---- pre-op of a landed k-block, in place (this thread's own 8 slots): BatchNorm-apply and/or ReLU; rows in the
        //      padding (mask bit clear) are re-zeroed, because the padding is applied after the pre-op
        auto pre_op = [&](const uint32_t a_st, const uint32_t mask, const int c) {
            float sc[4] = {1.f, 1.f, 1.f, 1.f}, sh[4] = {0.f, 0.f, 0.f, 0.f};
            if (AFF) {
                const float4 a4 = *reinterpret_cast<const float4 *>(s_scale + c);
                const float4 b4 = *reinterpret_cast<const float4 *>(s_shift + c);
                sc[0] = a4.x; sc[1] = a4.y; sc[2] = a4.z; sc[3] = a4.w;
                sh[0] = b4.x; sh[1] = b4.y; sh[2] = b4.z; sh[3] = b4.w;
            }
#pragma unroll
            for (int i = 0; i < 8; ++i) {
                const float4 q4 = ld_shared_v4(a_st + (uint32_t)i * 2048u);
                float v[4] = {q4.x, q4.y, q4.z, q4.w};
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    float a = v[e];
                    if (AFF) {
                        a = fmaf(a, sc[e], sh[e]);              // scale/shift are 0 beyond Cin
                        if (RELU) a = fmaxf(a, 0.f);
                        a = ((mask >> i) & 1u) ? a : 0.f;
                    } else if (RELU) {
                        a = fmaxf(a, 0.f);                      // padded rows landed as zeros
                    }
                    v[e] = a;
                }
                st_shared_v4(a_st + (uint32_t)i * 2048u, v[0], v[1], v[2], v[3]);
            }
        };
        // ---- per k-block: wait for the stage, stage its weights, then one asynchronous copy (cp.async, LDGSTS) per
        //      (row, chunk) from global memory straight into the row's swizzled slot.  Padding, rows past M, quads past
        //      the last tap and the odd coordinates of the zero-stuffed source copy 0 bytes (zero-filled); the Cin % 4
        //      tail copies the live channels only.  Without a pre-op the copies' completion is the thread's arrival on
        //      the stage's full barrier, so a producer never waits for its own loads and runs ahead as far as the ring
        //      allows.  With a pre-op the thread waits for the copies of its PREVIOUS k-block (one k-block of copies
        //      stays in flight; needs S >= 3, else it waits for the current one), transforms them in place and arrives.
        int s_s = grp;                             // stage of this group's next k-block (S >= 2)
        uint32_t s_ph = 0;
        int pend_s = -1;                           // pre-op: stage of the k-block whose copies are in flight (-1: none)
        uint32_t pend_mask = 0;
        int pend_c = 0;
        auto publish_pending = [&]() {
            pre_op(base + (uint32_t)pend_s * stage_bytes + roff0, pend_mask, pend_c);
            mbar_arrive(full(pend_s));
        };
        const int mine = total_kb > grp ? (total_kb - grp + 1) / 2 : 0;   // k-blocks of this group
#pragma unroll 1
        for (int it = 0; it < mine; ++it) {
            if (l_ti != cur_ti) set_tile(l_ti);
            const int w = min(cur_w + l_kb, p.w_last);   // the k-block's weight tile in wpack (host guarantees < 2^31)
            const uint32_t g = (uint32_t)(l_kb * 8 + gq0);
            const uint32_t tap = fdiv(g, p.fd_cq);
            const uint32_t ky = fdiv(tap, p.fd_kw);
            const int kx = (int)(tap - ky * (uint32_t)KW);
            const int dy = (int)ky * dil, dx = kx * dil;
            const bool cok = (int)tap < taps;      // quads past the last tap pad the final k-block
            const int c = cok ? (int)(g - tap * (uint32_t)p.CQ) * 4 : 0;   // first channel of this lane's 16-byte unit
            const int tapoff = UP ? c : (dy * Ws + dx) * xs + c;
            const uint32_t vbytes = c + 4 <= Cin ? 16u : (uint32_t)(Cin - c) * 4u;
            const uint32_t stage = base + (uint32_t)s_s * stage_bytes;
            const uint32_t a_st = stage + roff0;
            const uint32_t bar_full = full(s_s);
            mbar_wait(empty(s_s), s_ph ^ 1);
            if (issuer) {
                mbar_arrive_expect_tx(bar_full, wbytes);
                bulk_copy_g2s(stage + A_TILE_BYTES, wsrc + (size_t)w * wstride, wbytes, bar_full);
            }
            uint32_t mk = 0;
#pragma unroll
            for (int i = 0; i < 8; ++i) {
                const int yy = (oyx[i] >> 16) + dy, xx = (int)(short)(oyx[i] & 0xffff) + dx;
                bool ok = cok && (unsigned)yy < (unsigned)Hin && (unsigned)xx < (unsigned)Win;
                if (UP == 2) ok = ok && (((yy | xx) & 1) == 0);          // zero-stuffed source: odd coordinates are zeros
                mk |= (ok ? 1u : 0u) << i;
                int off;
                if (UP) off = rowoff[i] + ((yy >> 1) * Ws + (xx >> 1)) * xs + tapoff;
                else off = rowoff[i] + tapoff;
                const uint32_t dst = a_st + (uint32_t)i * 2048u;
                if (VEC) {
                    cp_async16(dst, ok ? xg + off : xg, ok ? vbytes : 0u);
                } else {
#pragma unroll
                    for (int e = 0; e < 4; ++e) {
                        const bool oke = ok && c + e < Cin;
                        cp_async4(dst + 4u * e, oke ? xg + off + e : xg, oke ? 4u : 0u);
                    }
                }
            }
            if constexpr (PRE == 0) {
                cp_async_mbar_arrive(bar_full);
            } else {
                cp_async_commit();
                if (pend_s >= 0) {
                    cp_async_wait_dyn(1);
                    publish_pending();
                }
                pend_s = s_s; pend_mask = mk; pend_c = c;
                if (S < 3) {                       // the group's next stage may be the one still waiting to be published
                    cp_async_wait_dyn(0);
                    publish_pending();
                    pend_s = -1;
                }
            }
            s_s += 2;
            if (s_s >= S) { s_s -= S; s_ph ^= 1; }
            l_kb += 2;
            while (l_kb >= p.kb_split) { l_kb -= p.kb_split; ++l_ti; }
        }
        if (PRE != 0 && pend_s >= 0) {
            cp_async_wait_dyn(0);
            publish_pending();
        }
    } else {
        // ===================== consumers: two warpgroups, rows [64 wg, 64 wg + 64) of every 128-pixel tile =========
        setmaxnreg_inc<CONSUMER_REGS>();
        // 3xTF32: every thread loads its A fragments of the k-block from the swizzled fp32 tile and splits them in
        // registers: hi = x rounded to tf32 (round-half-away on the 13 dropped bits, 2 integer ops), lo = x - hi, exact in
        // fp32 (the tensor core reads its top 19 bits: error <= 2^-21 |x|).  (Truncating instead of rounding saves one op
        // but makes lo one-signed: the dropped lo*lo term and lo's own truncation then add up coherently over K -- measured
        // 2-3x the error, past the 2e-5 bar of tests/test_conv_gpu.py -- so the rounding stays.)
        // Per k8 step A_lo*B_hi, A_hi*B_lo, A_hi*B_hi (small cross terms first), A from registers, B from shared memory.
        // The tensor cores accumulate one k-block (4 k8 steps x 3 products) into `acc`; it is then added into the fp32
        // tile sum `tot` with round-to-nearest adds, which keeps the accumulation error of long-K layers at the level of a
        // plain fp32 sum.  The stage is handed back to the producers as soon as its wgmma group has completed.
        // Single pass: A rounded like hi above, one product A_hi*B_hi per k8 step, the same k-block sums.
        const int wg = warp >> 2;
        const int row = wg * 64 + (warp & 3) * 16 + (lane >> 2);     // rows row and row + 8 of the tile
        const bool ovec = ((p.os & 1) == 0) && ((((uintptr_t)p.out) & 7) == 0);
        auto consume = [&](auto NT) {
            constexpr int N = decltype(NT)::value;
            constexpr int R = N / 2;
            float acc[R], tot[R];
            // A fragment of k8 step k (wgmma_tf32.cuh): (row, 8k + q), (row + 8, 8k + q), (row, 8k + q + 4),
            // (row + 8, 8k + q + 4) with q = lane % 4.  16-byte chunk c of a row sits at chunk c ^ (row & 7) of its
            // 128-byte line (SWIZZLE_128B), the same for row + 8; the chunk bits of aF hold row & 7, so the address of
            // chunk c is aF ^ (c << 4)
            const uint32_t aF0 = base + (uint32_t)row * 128u + ((uint32_t)(row & 7) << 4) + (threadIdx.x & 3u) * 4u;
            const uint64_t dB0 = make_desc(base + A_TILE_BYTES);                              // B_hi of stage 0
            const uint64_t oBlo = (uint64_t)((N * 128) >> 4), stage_step = (uint64_t)(stage_bytes >> 4);
            int s = 0;
            uint32_t ph = 0;
            uint32_t aF = aF0;
            uint64_t d = dB0;
            for (int ti = 0; ti < my_tiles; ++ti) {
                const int tile = cta_tile0() + ti * p.vgrid;
                const int m_tile = (int)fdiv((uint32_t)tile, p.fd_ntiles), nt = tile - m_tile * p.n_tiles;
#pragma unroll
                for (int i = 0; i < R; ++i) tot[i] = 0.f;
                for (int kb = 0; kb < p.kb_split; ++kb) {
                    mbar_wait_no_trap(full(s), ph);
                    if constexpr (SINGLE) {
                        uint32_t hi[BLOCK_K / 8][4];
#pragma unroll
                        for (int k = 0; k < BLOCK_K / 8; ++k) {
#pragma unroll
                            for (int j = 0; j < 4; ++j) {                  // j: row + 8 (j & 1), column + 4 (j >> 1)
                                const uint32_t x = ld_shared_u32((aF ^ (uint32_t)(32 * k + 16 * (j >> 1))) + 1024u * (j & 1));
                                hi[k][j] = __float_as_uint(round_tf32(__uint_as_float(x)));
                            }
                        }
                        wgmma_fence();
#pragma unroll
                        for (int k = 0; k < BLOCK_K / 8; ++k) Wgmma<N>::mma_rs(acc, hi[k], d + 2 * k, k != 0);
                        wgmma_commit();
                        wgmma_wait<0>();
                        wgmma_fence_operands(acc);
#pragma unroll
                        for (int k = 0; k < BLOCK_K / 8; ++k) wgmma_fence_operands(hi[k]);
                    } else {
                        uint32_t hi[BLOCK_K / 8][4], lo[BLOCK_K / 8][4];
#pragma unroll
                        for (int k = 0; k < BLOCK_K / 8; ++k) {
#pragma unroll
                            for (int j = 0; j < 4; ++j) {                  // j: row + 8 (j & 1), column + 4 (j >> 1)
                                const uint32_t x = ld_shared_u32((aF ^ (uint32_t)(32 * k + 16 * (j >> 1))) + 1024u * (j & 1));
                                float h, l;
                                split_tf32(__uint_as_float(x), h, l);
                                hi[k][j] = __float_as_uint(h);
                                lo[k][j] = __float_as_uint(l);
                            }
                        }
                        wgmma_fence();
#pragma unroll
                        for (int k = 0; k < BLOCK_K / 8; ++k) {
                            const uint64_t dbh = d + 2 * k, dbl = dbh + oBlo;
                            Wgmma<N>::mma_rs(acc, lo[k], dbh, k != 0);
                            Wgmma<N>::mma_rs(acc, hi[k], dbl, 1);
                            Wgmma<N>::mma_rs(acc, hi[k], dbh, 1);
                        }
                        wgmma_commit();
                        wgmma_wait<0>();
                        wgmma_fence_operands(acc);
#pragma unroll
                        for (int k = 0; k < BLOCK_K / 8; ++k) {
                            wgmma_fence_operands(hi[k]);
                            wgmma_fence_operands(lo[k]);
                        }
                    }
                    __syncwarp();
                    if (lane == 0) mbar_arrive(empty(s));
#pragma unroll
                    for (int i = 0; i < R; ++i) tot[i] += acc[i];
                    d += stage_step;
                    aF += stage_bytes;
                    if (++s == S) { s = 0; ph ^= 1; d = dB0; aF = aF0; }
                }

                // ---- epilogue straight from the accumulator registers.  Its inputs are re-read per tile through an empty
                //      asm: left loop-invariant, the per-column indices and addresses derived from them (dozens of values)
                //      are computed before the tile loop and spill across the k-block loop.
                int cq = ((int)threadIdx.x & 3) * 2, Cout = p.Cout;      // columns 8 j + cq, 8 j + cq + 1
                const float *bnb_x = p.bnb_x, *bnb_st = p.bnb_st;
                asm volatile("" : "+r"(cq), "+r"(Cout), "+l"(bnb_x), "+l"(bnb_st));
                const long long m0 = (long long)m_tile * BLOCK_M + row, m1 = m0 + 8;
                float *out = p.out + cta_split() * p.split_stride;       // split-K: this split's slice of the workspace
                float *orow0 = out + (m0 < p.M ? m0 : 0) * p.os + (long long)nt * n_tile;
                float *orow1 = out + (m1 < p.M ? m1 : 0) * p.os + (long long)nt * n_tile;
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
                            if (ovec && cabs + 1 < Cout) {
                                *reinterpret_cast<float2 *>(orow + col) = make_float2(o[0], o[1]);
                            } else {
                                if (cabs < Cout) orow[col] = o[0];
                                if (cabs + 1 < Cout) orow[col + 1] = o[1];
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
                                if (m < p.M && ch < Cout) {
                                    const float g = tot[4 * j + 2 * i + c];
                                    if (bnb_x) {
                                        const float xv = __ldg(bnb_x + m * p.bnb_xs + ch);
                                        const float sc = __ldg(bnb_st + ch), sh = __ldg(bnb_st + Cout + ch);
                                        const float mu = __ldg(bnb_st + 2 * Cout + ch), is = __ldg(bnb_st + 3 * Cout + ch);
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
                            if (lane < 4 && ch < Cout) {                 // this (warp, lane) owns the slot: plain adds
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
            case 64: consume(std::integral_constant<int, 64>()); break;
            case 80: consume(std::integral_constant<int, 80>()); break;
            case 96: consume(std::integral_constant<int, 96>()); break;
            case 112: consume(std::integral_constant<int, 112>()); break;
            default: consume(std::integral_constant<int, 128>()); break;
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

template <int PRE, int UP, bool VEC>
__global__ void __launch_bounds__(NUM_THREADS, 1) conv_tc_kernel(const ConvParams p) {
    conv_body<PRE, UP, VEC, false>(p);
}

template <int PRE, int UP, bool VEC>
__global__ void __launch_bounds__(NUM_THREADS, 1) conv_tf32_kernel(const ConvParams p) {
    conv_body<PRE, UP, VEC, true>(p);
}

__device__ __forceinline__ float splitk_act(float a, int act) {      // the activations of conv_body's epilogue
    if (act == 1) return a > 0.f ? a : expm1f(a);
    if (act == 2) return 1.0f / (1.0f + expf(-a));
    return a;
}

// Split-K reduction: out[m, c] = act(part[0][m][c] + part[1][m][c] + ...) for c < Cout, the splits added in a fixed order
// (bit-reproducible run to run); part is [splits][M][Cpad] with Cpad = Cout rounded up to 4, out is NHWC at pixel stride
// os (a channel slice of a wider slab is fine).  One thread per 16-byte channel quad of a pixel; n = M * Cpad / 4 < 2^31.
// 256-thread blocks; the grid stride is written with the literal block size (with blockDim.x ptxas keeps it on a stack
// frame).
__global__ void __launch_bounds__(256) conv_splitk_reduce_kernel(const float *__restrict__ part, int splits,
                                                                 long long split_stride, int n, int Cout, int Cpad, int act,
                                                                 float *__restrict__ out, long long os, int vec) {
    const int CQ = Cpad >> 2;
    for (int i = (int)blockIdx.x * 256 + (int)threadIdx.x; i < n; i += (int)gridDim.x * 256) {
        const int m = i / CQ, c = (i - m * CQ) * 4;
        const float *src = part + (long long)m * Cpad + c;
        float4 a = __ldg(reinterpret_cast<const float4 *>(src));
        for (int s = 1; s < splits; ++s) {
            const float4 b = __ldg(reinterpret_cast<const float4 *>(src + s * split_stride));
            a.x += b.x; a.y += b.y; a.z += b.z; a.w += b.w;
        }
        a.x = splitk_act(a.x, act); a.y = splitk_act(a.y, act); a.z = splitk_act(a.z, act); a.w = splitk_act(a.w, act);
        float *dst = out + (long long)m * os + c;
        if (vec && c + 4 <= Cout) {
            *reinterpret_cast<float4 *>(dst) = a;
        } else {
            dst[0] = a.x;
            if (c + 1 < Cout) dst[1] = a.y;
            if (c + 2 < Cout) dst[2] = a.z;
            if (c + 3 < Cout) dst[3] = a.w;
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
                                     int Cout, int Cin, int KH, int KW, int transpose_flip, float *wpack, void *stream) {
    if (!w || !wpack || Cout < 1 || Cin < 1 || KH < 1 || KW < 1) return BTS_EINVAL;
    if (!bts_aligned16(wpack)) return BTS_EALIGN;
    const int rows = transpose_flip ? Cin : Cout;
    const int n_tile = bts_conv_n_tile(rows);
    const int n_tiles = (rows + n_tile - 1) / n_tile;
    const long long total = bts_conv_packed_floats(rows, transpose_flip ? Cout : Cin, KH, KW) / 2;
    long long grid = (total + 255) / 256;
    const long long cap = (long long)bts_num_sms() * 16;
    if (grid > cap) grid = cap;
    pack_weights_kernel<<<(int)grid, 256, 0, (cudaStream_t)stream>>>(w, s_co, s_ci, s_kh, s_kw, Cout, Cin, KH, KW,
                                                                    transpose_flip, wpack, n_tile, n_tiles, 0, 1);
    BTS_LAUNCH_CHECK();
    return 0;
}

// Grouped convolution whose groups tile a 128-wide diagonal block (ResNeXt 3x3: width % kwin == 0, kwin % cpg == 0):
// w is (width, cpg, KH, KW); the packed operator has width/n_tile n-tiles of n_tile = bts_conv_group_n_tile(kwin) rows,
// each over the K window of kwin channels that holds its rows -- zeros outside the row's group.  Run with
// bts_conv_fwd(kwin = bts_conv_group_window(width, cpg)).
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
                                             int width, int cpg, int KH, int KW, int transpose_flip, float *wpack,
                                             void *stream) {
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
                                                                    width / bts_conv_group_n_tile(kwin), kwin, cpg);
    BTS_LAUNCH_CHECK();
    return 0;
}

// Forward / dgrad entry point (see bts_b200.h).  Split mode (workspace != NULL): the conv kernel writes raw partial tile
// sums into `workspace` ([splits][M][Cpad]), conv_splitk_reduce_kernel adds them and applies the activation into out.
// Every check of an argument combination comes before the first CUDA runtime call (bts_num_sms).
extern "C" int bts_conv_fwd(const float *x, long long x_pixel_stride, int B, int Hs, int Ws, int source_mode, int out_h,
                            int out_w, int kwin, int Cin, int KH, int KW, int stride, int pad, int dil, const float *wpack,
                            int Cout, const float *pre_scale, const float *pre_shift, int pre_relu, float *out,
                            long long out_pixel_stride, int act, int precision, double *stat_sum, double *stat_sumsq,
                            const float *x_bn, long long x_bn_stride, const float *bn_st, int relu, int splits,
                            float *workspace, void *stream) {
    if (!x || !wpack || !out || B < 0 || Hs < 1 || Ws < 1 || Cin < 1 || Cout < 1 || KH < 1 || KW < 1 || stride < 1 ||
        pad < 0 || dil < 1)
        return BTS_EINVAL;
    if ((pre_scale == nullptr) != (pre_shift == nullptr)) return BTS_EINVAL;
    if (pre_scale && Cin > MAX_CIN_SMEM) return BTS_EINVAL;
    if (act < 0 || act > 2 || precision < 0 || precision > 1) return BTS_EINVAL;
    if (source_mode < 0 || source_mode > 2 || kwin < 0) return BTS_EINVAL;
    if (source_mode == 2 && (stride != 1 || out_h < 1 || out_w < 1)) return BTS_EINVAL;
    if (kwin && (pre_scale || Cin % kwin || Cout % kwin)) return BTS_EINVAL;   // whole windows; no pre-op on grouped convs
    if (!bts_aligned16(wpack)) return BTS_EALIGN;
    if ((stat_sum == nullptr) != (stat_sumsq == nullptr)) return BTS_EINVAL;
    if (stat_sum && act != 0) return BTS_EINVAL;                        // statistics of the raw conv output only
    const bool bnb = x_bn || bn_st;
    if (bnb && (!x_bn || !bn_st || !stat_sum)) return BTS_EINVAL;       // its sums go to stat_sum / stat_sumsq
    if (splits < 1 || (splits > 1 && !workspace)) return BTS_EINVAL;
    const bool split_mode = workspace != nullptr;
    if (split_mode && (stat_sum || bnb)) return BTS_EINVAL;             // raw sums: no epilogue reductions
    if (split_mode && !bts_aligned16(workspace)) return BTS_EALIGN;
    if (B == 0) return 0;
    if ((long long)B * Hs * Ws * x_pixel_stride >= 0x7fffffffLL) return BTS_EINVAL;   // 32-bit element offsets
    ConvParams p;
    p.x = x; p.xs = x_pixel_stride; p.B = B; p.Hs = Hs; p.Ws = Ws; p.up = source_mode; p.Cin = kwin ? kwin : Cin;
    p.kwin = kwin;
    p.KH = KH; p.KW = KW; p.stride = stride; p.pad = pad; p.dil = dil;
    p.wpack = wpack; p.Cout = Cout;
    if (kwin % 16) return BTS_EINVAL;
    p.n_tile = kwin ? bts_conv_group_n_tile(kwin) : bts_conv_n_tile(Cout);
    p.n_tiles = (Cout + p.n_tile - 1) / p.n_tile;
    p.pre_scale = pre_scale; p.pre_shift = pre_shift; p.pre_relu = pre_relu ? 1 : 0;
    p.out = out; p.os = out_pixel_stride; p.act = act;
    p.stat_sum = stat_sum; p.stat_sumsq = stat_sumsq;
    p.bnb_x = x_bn; p.bnb_xs = x_bn_stride; p.bnb_st = bn_st; p.bnb_relu = relu ? 1 : 0;
    const int Hin = p.up ? 2 * Hs : Hs, Win = p.up ? 2 * Ws : Ws;
    p.Hv = Hin; p.Wv = Win;      // mode 2: live source coordinates are the even ones below 2Hs x 2Ws, zeros everywhere else
    p.Hout = p.up == 2 ? out_h : (Hin + 2 * pad - dil * (KH - 1) - 1) / stride + 1;
    p.Wout = p.up == 2 ? out_w : (Win + 2 * pad - dil * (KW - 1) - 1) / stride + 1;
    if (p.Hout < 1 || p.Wout < 1) return BTS_EINVAL;
    // the producers keep a row's source coordinates as two 16-bit halves of one register
    if (Hin >= 0x4000 || Win >= 0x4000 || p.Hout >= 0x4000 || p.Wout >= 0x4000 || pad >= 0x4000 ||
        dil * (KH - 1) >= 0x4000 || dil * (KW - 1) >= 0x4000)
        return BTS_EINVAL;
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
    const int sms = bts_num_sms();
    // split-K: ranges of kb_split k-blocks (the last one padded past KB); a count that would leave a split empty is reduced
    p.kb_split = (p.KB + splits - 1) / splits;
    p.splits = split_mode ? (p.KB + p.kb_split - 1) / p.kb_split : 1;
    if (!split_mode) p.kb_split = p.KB;
    if (p.splits > sms) return BTS_EINVAL;
    p.vgrid = p.total_tiles < sms / p.splits ? p.total_tiles : sms / p.splits;
    p.fd_vgrid = make_fastdiv((uint32_t)p.vgrid);
    p.w_last = p.n_tiles * p.KB - 1;
    const int Cpad = (Cout + 3) / 4 * 4;
    p.split_stride = 0;
    if (split_mode) {
        if (p.M * (Cpad / 4) >= 0x7fffffffLL) return BTS_EINVAL;
        p.out = workspace; p.os = Cpad; p.act = 0; p.split_stride = p.M * Cpad;
    }
    p.fd_wout = make_fastdiv((uint32_t)p.Wout);
    p.fd_hout = make_fastdiv((uint32_t)p.Hout);
    p.fd_ntiles = make_fastdiv((uint32_t)p.n_tiles);
    const int pre = (pre_scale ? 2 : 0) | (p.pre_relu ? 1 : 0);
    // shared-memory plan: stage = A (16 KB) + B hi/lo (2 x n_tile x 128 B), single pass A + B hi; as many stages as fit
    p.stage_bytes = A_TILE_BYTES + (precision ? 1 : 2) * p.n_tile * 128;
    const int pre_bytes = pre >= 2 ? p.KC * 32 * 8 : 0;
    const int stat_bytes = stat_sum ? STAT_SETS * 2 * p.n_tile * 8 : 0;
    p.stages = (SMEM_LIMIT - 1024 - BAR_BYTES - pre_bytes - stat_bytes) / p.stage_bytes;
    if (p.stages > MAX_STAGES) p.stages = MAX_STAGES;
    if (p.stages < 2) return BTS_EINVAL;
    const int smem = p.stages * p.stage_bytes + pre_bytes + BAR_BYTES + stat_bytes + 1024;
    dim3 grid((unsigned)(p.vgrid * p.splits));
    const bool vec = p.vec_ok;      // aligned base + pixel stride % 4 == 0 (a channel tail is masked in-kernel)
    cudaError_t err = cudaSuccess;
#define BTS_LAUNCH(KERNEL, PRE, UP, VEC)                                                                           \
    do {                                                                                                           \
        static bool attr_set_[BTS_MAX_DEVICES] = {};                                                               \
        bool &attr_set = attr_set_[bts_cur_device()];                                                              \
        if (!attr_set) {                                                                                           \
            err = cudaFuncSetAttribute(KERNEL<PRE, UP, VEC>, cudaFuncAttributeMaxDynamicSharedMemorySize,          \
                                       SMEM_LIMIT);                                                                \
            if (err != cudaSuccess) return (int)err;                                                               \
            attr_set = true;                                                                                       \
        }                                                                                                          \
        KERNEL<PRE, UP, VEC><<<grid, NUM_THREADS, smem, (cudaStream_t)stream>>>(p);                                \
    } while (0)
#define BTS_DISPATCH_UV(KERNEL, PRE)                                                                               \
    do {                                                                                                           \
        if (p.up == 2) { if (vec) BTS_LAUNCH(KERNEL, PRE, 2, true); else BTS_LAUNCH(KERNEL, PRE, 2, false); }      \
        else if (p.up) { if (vec) BTS_LAUNCH(KERNEL, PRE, 1, true); else BTS_LAUNCH(KERNEL, PRE, 1, false); }      \
        else { if (vec) BTS_LAUNCH(KERNEL, PRE, 0, true); else BTS_LAUNCH(KERNEL, PRE, 0, false); }                \
    } while (0)
#define BTS_DISPATCH(KERNEL)                                                                                       \
    do {                                                                                                           \
        switch (pre) {                                                                                             \
            case 0: BTS_DISPATCH_UV(KERNEL, 0); break;                                                             \
            case 1: BTS_DISPATCH_UV(KERNEL, 1); break;                                                             \
            case 2: BTS_DISPATCH_UV(KERNEL, 2); break;                                                             \
            default: BTS_DISPATCH_UV(KERNEL, 3); break;                                                            \
        }                                                                                                          \
    } while (0)
    if (precision) BTS_DISPATCH(conv_tf32_kernel);
    else BTS_DISPATCH(conv_tc_kernel);
#undef BTS_DISPATCH
#undef BTS_DISPATCH_UV
#undef BTS_LAUNCH
    BTS_LAUNCH_CHECK();
    if (split_mode) {
        const int n = (int)(p.M * (Cpad / 4));
        int rgrid = (n + 255) / 256;
        if (rgrid > sms * 8) rgrid = sms * 8;
        const int vec = bts_aligned16(out) && out_pixel_stride % 4 == 0;
        conv_splitk_reduce_kernel<<<rgrid, 256, 0, (cudaStream_t)stream>>>(workspace, p.splits, p.split_stride, n, Cout,
                                                                           Cpad, act, out, out_pixel_stride, vec);
        BTS_LAUNCH_CHECK();
    }
    return 0;
}

// Split-K plan of a forward / dgrad launch (see bts_b200.h).  A launch splits only when its tiles fill at most half the SMs:
// splits = as many as keep tiles * splits within one wave of bts_num_sms() and every split at least SPLITK_MIN_KB k-blocks
// long (its padded tail included), so that each tile of a split streams more k-blocks than the deepest stage ring holds
// (MAX_STAGES) and its epilogue, which writes the partial tile sum, stays short next to its main loop.  *splits > 0 on
// entry forces that count instead.
constexpr int SPLITK_MIN_KB = 8;
static_assert(SPLITK_MIN_KB > MAX_STAGES, "a split must stream more k-blocks than the ring holds");

extern "C" int bts_conv_fwd_splitk_plan(int B, int Hout, int Wout, int kwin, int Cin, int KH, int KW, int Cout, int *splits,
                                        long long *workspace_floats) {
    if (!splits || !workspace_floats || B < 1 || Hout < 1 || Wout < 1 || kwin < 0 || kwin % 16 || Cin < 1 || Cout < 1 ||
        KH < 1 || KW < 1 || *splits < 0)
        return BTS_EINVAL;
    const int n_tile = kwin ? bts_conv_group_n_tile(kwin) : bts_conv_n_tile(Cout);
    if (!n_tile) return BTS_EINVAL;
    const long long n_tiles = (Cout + n_tile - 1) / n_tile;
    const long long M = (long long)B * Hout * Wout;
    const long long tiles = (M + BLOCK_M - 1) / BLOCK_M * n_tiles;
    const long long KB = ((long long)KH * KW * (((kwin ? kwin : Cin) + 3) / 4) + 7) / 8;
    const long long Cpad = (Cout + 3) / 4 * 4;
    const long long sms = bts_num_sms();
    long long s = *splits;
    if (s == 0) {
        s = 1;
        if (2 * tiles <= sms) {
            s = sms / tiles;
            if (s > KB / SPLITK_MIN_KB) s = KB / SPLITK_MIN_KB;
        }
        if (M * (Cpad / 4) >= 0x7fffffffLL) s = 1;
    }
    if (s > KB) s = KB;
    if (s > sms) s = sms;
    if (s > 1) s = (KB + (KB + s - 1) / s - 1) / ((KB + s - 1) / s);       // no empty split (as the launch counts them)
    if (s < 1) s = 1;
    *splits = (int)s;
    *workspace_floats = s > 1 ? s * M * Cpad : 0;
    return 0;
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
