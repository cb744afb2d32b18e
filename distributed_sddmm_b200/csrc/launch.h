// launch.h -- helpers shared by the translation units of libhnh_b200.so: error reporting, the grid policy of the
// grid-stride kernels, the one kernel-launch path, and the scratch allocations of the setup and plan entry points.
#pragma once
#include <algorithm>
#include <cstdarg>
#include <cstdint>
#include <cuda_runtime.h>

#include "hnh_b200.h"

#define HNH_STR2(x) #x
#define HNH_STR(x) HNH_STR2(x)

namespace hnh {
// Record a failure description for hnh_last_error_string() and return `code`.
int set_error(int code, const char *fmt, ...);
// HNH_OK, or HNH_E_CUDA with the CUDA error text recorded.
int check_cuda(cudaError_t e, const char *what);
// Add to the process-wide kernel-launch counter (hnh_launch_count()).
void count_launch(uint64_t n);
// Number of SMs of the current device (cached).
int device_sm_count(int *out);

// threads per CTA of every grid-stride kernel
constexpr int kBlock = 256;
// grid_for's per_sm: as many CTAs of the kernel as are resident on an SM at once
constexpr int kResident = 0;

// Grid of a grid-stride kernel: one CTA per `per_cta` work items, at least one, at most `per_sm` CTAs per SM (kResident:
// the kernel's occupancy at kBlock threads) and at most `max_ctas`.
template <typename K>
int grid_for(K kernel, int64_t work, int64_t per_cta, int *grid, int per_sm = kResident, int64_t max_ctas = INT64_MAX) {
    int sms = 0;
    int rc = device_sm_count(&sms);
    if (rc) return rc;
    if (per_sm == kResident) {
        cudaError_t e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, kBlock, 0);
        if (e != cudaSuccess) return check_cuda(e, "cudaOccupancyMaxActiveBlocksPerMultiprocessor");
        per_sm = std::max(per_sm, 1);
    }
    *grid = (int)std::max<int64_t>(1, std::min({(work + per_cta - 1) / per_cta, (int64_t)sms * per_sm, max_ctas}));
    return HNH_OK;
}

// Every kernel launch of the library: launch, count it for hnh_launch_count(), report a launch failure under `name`.
template <typename... Params, typename... Args>
int launch(void (*kernel)(Params...), dim3 grid, dim3 block, cudaStream_t st, const char *name, Args... args) {
    kernel<<<grid, block, 0, st>>>(args...);
    count_launch(1);
    return check_cuda(cudaGetLastError(), name);
}

// cudaMalloc'ed temporaries of one call, released on every exit path
struct Scratch {
    void *p[12] = {};
    int n = 0;
    cudaError_t get(void **out, size_t bytes) {
        cudaError_t e = cudaMalloc(out, std::max<size_t>(bytes, 256));
        if (e == cudaSuccess) p[n++] = *out;
        return e;
    }
    ~Scratch() { for (int i = 0; i < n; i++) cudaFree(p[i]); }
};

// radix-sort bits that hold every key up to max_value
inline int bits_for(uint64_t max_value) {
    int b = 1;
    while (b < 64 && (max_value >> b) != 0) b++;
    return b;
}
}  // namespace hnh
