// Shared host-side helpers for libirn_b200.so: error reporting and launch checks.
#pragma once
#include <cuda_runtime.h>
#include <cstdarg>
#include <cstdio>

#include "../../include/irn_b200.h"

namespace irn {

enum { kOk = 0, kBadArg = -1, kCudaError = -2, kWorkspace = -3, kUnsupported = -4 };

char* last_error_buf();             // thread-local, 512 bytes
int fail(int code, const char* fmt, ...);
int& launch_counter();              // thread-local count of kernels launched by the last API call
long long& total_launch_counter();  // thread-local, never reset: bench.py's gpu_launches

inline int check_cuda(cudaError_t e, const char* what) {
    if (e == cudaSuccess) return kOk;
    return fail(kCudaError, "%s: %s", what, cudaGetErrorString(e));
}

#define IRN_CUDA(call)                                            \
    do {                                                          \
        int _rc = ::irn::check_cuda((call), #call);               \
        if (_rc != 0) return _rc;                                 \
    } while (0)

#define IRN_LAUNCH_CHECK(name)                                    \
    do {                                                          \
        ::irn::launch_counter()++;                                \
        ::irn::total_launch_counter()++;                          \
        int _rc = ::irn::check_cuda(cudaGetLastError(), name);    \
        if (_rc != 0) return _rc;                                 \
    } while (0)

inline size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

// true when p is device (or managed) memory of the CUDA runtime
inline bool is_device_ptr(const void* p) {
    cudaPointerAttributes a;
    if (cudaPointerGetAttributes(&a, p) != cudaSuccess) {
        cudaGetLastError();
        return false;
    }
    return a.type == cudaMemoryTypeDevice || a.type == cudaMemoryTypeManaged;
}

// cudaFuncSetAttribute and the SM count belong to the CURRENT device: launch helpers keep one flag / value per device so that a
// process driving several GPUs (one host thread each) configures every one of them.
struct DeviceOnce {
    bool done[64] = {};
    int n_sm[64] = {};
    // slot of the current device (a device index beyond the table shares slot 63 and is simply configured again on every call)
    int slot() const {
        int dev = 0;
        cudaGetDevice(&dev);
        return dev >= 0 && dev < 63 ? dev : 63;
    }
    bool need(int s) const { return s == 63 || !done[s]; }
};

}  // namespace irn
