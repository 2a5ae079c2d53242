// Shared helpers for the bts_b200 kernels (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/bts_b200.h"

#define BTS_LAUNCH_CHECK()                                   \
    do {                                                     \
        cudaError_t e__ = cudaGetLastError();                \
        if (e__ != cudaSuccess) return (int)e__;             \
    } while (0)

static inline bool bts_aligned16(const void *p) { return (((uintptr_t)p) & 15u) == 0; }

__host__ __device__ constexpr int bts_ceil_div(long long a, long long b) { return (int)((a + b - 1) / b); }

// number of SMs of the current device (cached); grids of persistent kernels are sized from it
int bts_num_sms();
// current device ordinal (mod BTS_MAX_DEVICES): key of per-device one-time setup (cudaFuncSetAttribute is per device)
constexpr int BTS_MAX_DEVICES = 64;
int bts_cur_device();
