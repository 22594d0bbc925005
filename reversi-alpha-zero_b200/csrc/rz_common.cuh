// rz_common.cuh -- error plumbing shared by the C-ABI translation units.
#pragma once
#include <cuda_runtime.h>
#include <stdarg.h>
#include <stdio.h>
#include "../../include/rz_engine.h"

namespace rz {

void set_error(const char* fmt, ...);  // thread-local message returned by rz_last_error()

#define RZ_CUDA_TRY(expr)                                                                      \
    do {                                                                                       \
        cudaError_t _e = (expr);                                                               \
        if (_e != cudaSuccess) {                                                               \
            rz::set_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), __FILE__, __LINE__); \
            return RZ_ECUDA;                                                                   \
        }                                                                                      \
    } while (0)

#define RZ_REQUIRE(cond, ...)        \
    do {                             \
        if (!(cond)) {               \
            rz::set_error(__VA_ARGS__); \
            return RZ_EINVAL;        \
        }                            \
    } while (0)

#define RZ_TRY(expr)             \
    do {                         \
        int _r = (expr);         \
        if (_r != RZ_OK) return _r; \
    } while (0)

// Launch-error check: catches bad configurations synchronously; asynchronous faults surface at the
// next synchronising call and are reported there.
#define RZ_LAUNCH_CHECK() RZ_CUDA_TRY(cudaGetLastError())

inline int num_sms() {
    static int sms = 0;
    if (!sms) {
        int dev = 0;
        cudaGetDevice(&dev);
        cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
        if (sms <= 0) sms = 132;
    }
    return sms;
}

}  // namespace rz
