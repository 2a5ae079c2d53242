// Library identification + device queries shared by all kernels.
#include <cstdio>
#include <cstdlib>
#include <cstring>

#include "common.cuh"

int bts_cur_device() {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0) dev = 0;
    return dev & (BTS_MAX_DEVICES - 1);
}

// SM count of the CURRENT device, cached per device ordinal (one process may drive several GPUs: nn.DataParallel,
// bts_main.py:357).  BTS_B200_SM_LIMIT=k caps the persistent grids at k SMs (leaves SMs to NCCL's kernels when a
// collective overlaps the backward pass; see bench.py / DESIGN 6).
int bts_num_sms() {
    static int cached[BTS_MAX_DEVICES] = {};
    static int limit = -1;
    const int dev = bts_cur_device();
    if (limit < 0) {
        const char *e = getenv("BTS_B200_SM_LIMIT");
        limit = e ? atoi(e) : 0;
    }
    if (!cached[dev]) {
        int n = 0;
        if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) n = 132;   // H100 SXM
        cached[dev] = n;
    }
    return (limit > 0 && limit < cached[dev]) ? limit : cached[dev];
}

extern "C" int bts_version(char *buf, int buflen) {
    static const char v[] = "bts_b200 0.1 (sm_90a; lpg, plane_head, silog, conv_tc)";
    if (buf && buflen > 0) {
        std::strncpy(buf, v, (size_t)buflen - 1);
        buf[buflen - 1] = 0;
    }
    return 90;
}

// zero n floats on the stream (grad_focal of the TF-op surface: `focal` never enters the LPG arithmetic, SURVEY Q1)
extern "C" int bts_fill_zero_f32(float *p, long long n, void *stream) {
    if (n < 0 || (n > 0 && !p)) return BTS_EINVAL;
    if (n == 0) return 0;
    const cudaError_t e = cudaMemsetAsync(p, 0, sizeof(float) * (size_t)n, (cudaStream_t)stream);
    return e == cudaSuccess ? 0 : (int)e;
}
