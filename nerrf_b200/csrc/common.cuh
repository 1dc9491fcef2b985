// Shared helpers for the nerrf_b200 C-ABI library (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdarg.h>
#include "../../include/nerrf_b200.h"

namespace nerrf {

void set_error(const char* fmt, ...);

#define NERRF_CHECK_CUDA(expr)                                                              \
    do {                                                                                    \
        cudaError_t _e = (expr);                                                            \
        if (_e != cudaSuccess) {                                                            \
            nerrf::set_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e),        \
                             __FILE__, __LINE__);                                           \
            return NERRF_ERR_CUDA;                                                          \
        }                                                                                   \
    } while (0)

#define NERRF_REQUIRE(cond, ...)                                                            \
    do {                                                                                    \
        if (!(cond)) {                                                                      \
            nerrf::set_error(__VA_ARGS__);                                                  \
            return NERRF_ERR_INVALID;                                                       \
        }                                                                                   \
    } while (0)

inline int launch_status(const char* what) {
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) {
        set_error("launch of %s failed: %s", what, cudaGetErrorString(e));
        return NERRF_ERR_CUDA;
    }
    return NERRF_OK;
}

int sm_count();   // cached per process (current device at first call)

// Raise `kernel`'s dynamic shared-memory limit on the current device to at least `bytes`.  The attribute is set once per
// (device, kernel) and again only when a larger size is asked for.  Returns NERRF_OK or NERRF_ERR_CUDA.
int set_max_dynamic_smem(const void* kernel, size_t bytes);

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

__device__ __forceinline__ float4 ldg4(const float* p) {
    return __ldg(reinterpret_cast<const float4*>(p));
}

}  // namespace nerrf
