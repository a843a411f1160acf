// Shared helpers for libsdb200 (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/sdb200.h"

// every kernel launch of the library is followed by exactly one SDB_CHECK_LAUNCH: it also counts the launch
// (sdb_launch_count(), read by bench.py for its `gpu_launches` claim)
extern "C" void sdb_count_launch_(void);

#define SDB_CHECK_LAUNCH()                                   \
    do {                                                     \
        cudaError_t e__ = cudaGetLastError();                \
        if (e__ != cudaSuccess) return (int)e__;             \
        sdb_count_launch_();                                 \
    } while (0)

#define SDB_CUDA(call)                                       \
    do {                                                     \
        cudaError_t e__ = (call);                            \
        if (e__ != cudaSuccess) return (int)e__;             \
    } while (0)

static inline int sdb_num_sms() {
    int dev = 0, n = 132;
    if (cudaGetDevice(&dev) == cudaSuccess) cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
    return n > 0 ? n : 132;
}

template <typename T>
static inline T sdb_div_up(T a, T b) { return (a + b - 1) / b; }
