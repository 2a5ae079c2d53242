// wgmma / mbarrier / bulk-copy / TMA PTX wrappers shared by the tensor-core kernels (sm_90a).
#pragma once
#include "common.cuh"
#include "wgmma_tf32.cuh"

namespace tc {

__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint32_t bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
    uint32_t ok = 0;
    uint32_t spins = 0;
    while (true) {
        asm volatile(
            "{\n\t.reg .pred p;\n\t"
            "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
            "selp.u32 %0, 1, 0, p;\n\t}"
            : "=r"(ok)
            : "r"(bar), "r"(parity)
            : "memory");
        if (ok) break;
        if (++spins > 200000000u) __trap();   // watchdog: a protocol bug must fail loudly, not hang the box
    }
}
// same protocol, for waits that are expected to be long (the weight loader waiting for a free stage): back off between
// polls so the spinning lane does not take issue slots from the producer warps.
__device__ __forceinline__ void mbar_wait_sleep(uint32_t bar, uint32_t parity) {
    uint32_t ok = 0;
    uint32_t spins = 0;
    while (true) {
        asm volatile(
            "{\n\t.reg .pred p;\n\t"
            "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
            "selp.u32 %0, 1, 0, p;\n\t}"
            : "=r"(ok)
            : "r"(bar), "r"(parity)
            : "memory");
        if (ok) break;
        __nanosleep(32);
        if (++spins > 50000000u) __trap();
    }
}
__device__ __forceinline__ void bulk_copy_g2s(uint32_t dst, const void *src, uint32_t bytes, uint32_t bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst),
                 "l"(src), "r"(bytes), "r"(bar)
                 : "memory");
}
// TMA im2col load (cp.async.bulk.tensor ... .im2col): `pixelsPerColumn` consecutive base pixels starting at
// tensor coordinate (w, h, n), each shifted by the filter offset (off_w, off_h), `channelsPerPixel` channels from c; pixels
// that fall outside the tensor (the convolution's zero padding) arrive as zeros.  Completes `bytes` on the mbarrier.
__device__ __forceinline__ void tma_im2col_4d(uint32_t dst, const void *tmap, int c, int w, int h, int n, uint32_t bar,
                                              uint16_t off_w, uint16_t off_h) {
    asm volatile(
        "cp.async.bulk.tensor.4d.shared::cluster.global.im2col.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4, %5}], [%6], "
        "{%7, %8};" ::"r"(dst),
        "l"(tmap), "r"(c), "r"(w), "r"(h), "r"(n), "r"(bar), "h"(off_w), "h"(off_h)
        : "memory");
}
// plain (tiled) 2-D tensor load: coordinates {c0 = innermost, c1}; out-of-range elements are zero-filled
__device__ __forceinline__ void tma_tile_2d(uint32_t dst, const void *tmap, int c0, int c1, uint32_t bar) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];" ::"r"(dst),
        "l"(tmap), "r"(c0), "r"(c1), "r"(bar)
        : "memory");
}
__device__ __forceinline__ void tma_prefetch_desc(const void *tmap) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(tmap) : "memory");
}
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// ---- warpgroup MMA (wgmma): ordering of the accumulator registers and of the asynchronous operand reads
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int PENDING>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(PENDING) : "memory"); }
// keeps the compiler from moving accumulator reads / writes across an in-flight wgmma
template <int R>
__device__ __forceinline__ void wgmma_fence_operands(float (&d)[R]) {
#pragma unroll
    for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// K-major, 128-byte swizzle shared-memory matrix descriptor (sm_90 wgmma): start>>4 | LBO (unused, 1) | SBO = 1024 B
// (8 rows x 128 B) | layout SWIZZLE_128B (=1 at bits [62,64)).  Tiles are 1024-byte aligned; one k8 step of tf32 = +32 B.
__device__ __forceinline__ uint64_t make_desc(uint32_t saddr) {
    return (uint64_t)((saddr >> 4) & 0x3FFFu) | (1ull << 16) | ((uint64_t)(1024 >> 4) << 32) | (1ull << 62);
}
// K-major, no swizzle ("interleaved" core matrices of 8 rows x 16 B stored as 128 contiguous bytes): LBO = byte stride
// between core matrices adjacent along K, SBO = byte stride between core matrices adjacent along M / N.
__device__ __forceinline__ uint64_t make_desc_core(uint32_t saddr, uint32_t lbo, uint32_t sbo) {
    return (uint64_t)((saddr >> 4) & 0x3FFFu) | ((uint64_t)((lbo >> 4) & 0x3FFFu) << 16) |
           ((uint64_t)((sbo >> 4) & 0x3FFFu) << 32);
}

__device__ __forceinline__ float rna_tf32(float x) {
    uint32_t r;
    asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
    return __uint_as_float(r);
}

struct __align__(16) F4 { float v[4]; };

// Division of n < 2^31 by a runtime constant d >= 1 as multiply-high + shift (the divisor's magic numbers are computed
// once on the host): with s = ceil(log2 d) and mul = ceil(2^(31+s) / d) the quotient is umulhi(n, mul) >> (s-1),
// exact for every n < 2^31.  Replaces the ~25-instruction I2F/MUFU.RCP/F2I sequences of `/` and `%`.
struct FastDiv {
    uint32_t mul, shr, d;
};
inline FastDiv make_fastdiv(uint32_t d) {
    FastDiv f;
    f.d = d;
    f.mul = 0;
    f.shr = 0;
    if (d > 1) {
        uint32_t s = 0;
        while ((1ull << s) < d) ++s;                        // s = ceil(log2 d) >= 1
        f.mul = (uint32_t)(((1ull << (31 + s)) + d - 1) / d);
        f.shr = s - 1;
    }
    return f;
}
__device__ __forceinline__ uint32_t fdiv(uint32_t n, const FastDiv &f) {
    return f.d == 1 ? n : (__umulhi(n, f.mul) >> f.shr);
}

// Ampere-style async copies (LDGSTS): 16-byte / 4-byte global -> shared with zero-fill when src_bytes == 0
__device__ __forceinline__ void cp_async16(uint32_t dst, const void *src, uint32_t src_bytes) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(src_bytes) : "memory");
}
__device__ __forceinline__ void cp_async4(uint32_t dst, const void *src, uint32_t src_bytes) {
    asm volatile("cp.async.ca.shared.global [%0], [%1], 4, %2;" ::"r"(dst), "l"(src), "r"(src_bytes) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
__device__ __forceinline__ void cp_async_wait_dyn(int pending) {   // wait until <= pending groups are in flight
    switch (pending) {
        case 0: asm volatile("cp.async.wait_group 0;" ::: "memory"); break;
        case 1: asm volatile("cp.async.wait_group 1;" ::: "memory"); break;
        case 2: asm volatile("cp.async.wait_group 2;" ::: "memory"); break;
        case 3: asm volatile("cp.async.wait_group 3;" ::: "memory"); break;
        case 4: asm volatile("cp.async.wait_group 4;" ::: "memory"); break;
        case 5: asm volatile("cp.async.wait_group 5;" ::: "memory"); break;
        case 6: asm volatile("cp.async.wait_group 6;" ::: "memory"); break;
        default: asm volatile("cp.async.wait_group 7;" ::: "memory"); break;
    }
}
__device__ __forceinline__ float4 ld_shared_v4(uint32_t addr) {
    float4 v;
    asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(addr) : "memory");
    return v;
}

__device__ __forceinline__ void st_shared_f32(uint32_t addr, float a) {
    asm volatile("st.shared.f32 [%0], %1;" ::"r"(addr), "f"(a) : "memory");
}
__device__ __forceinline__ void st_shared_v4(uint32_t addr, float a, float b, float c, float d) {
    asm volatile("st.shared.v4.f32 [%0], {%1, %2, %3, %4};" ::"r"(addr), "f"(a), "f"(b), "f"(c), "f"(d) : "memory");
}


}  // namespace tc
