// row_gather.cuh -- the pieces shared by the row-owning gather kernels of gatv2.cu and sparse_attention.cu: a group of
// G lanes owns one CSR row, gathered rows arrive in 128-bit loads, dots end in the group's xor-butterfly, and the grid
// is capped at the resident CTAs.  The load / store forms are those of kernels.cuh (not included here: it defines
// non-template kernels of c_abi.cu).  Gathers use the read-only path at the normal L2 policy; index and value streams
// do not allocate in L1.
#pragma once
#include <algorithm>
#include <cstdint>

#include "hnh_b200.h"
#include "launch.h"

namespace {

template <int VW>
__device__ __forceinline__ void ld_gather(double (&d)[VW], const double *p) {
    static_assert(VW == 2, "128-bit loads only");
    asm("ld.global.nc.L1::no_allocate.v2.f64 {%0,%1}, [%2];" : "=d"(d[0]), "=d"(d[1]) : "l"(p));
}
template <int VW>
__device__ __forceinline__ void ld_rw(double (&d)[VW], const double *p) {
    static_assert(VW == 2, "128-bit loads only");
    asm volatile("ld.global.L1::no_allocate.v2.f64 {%0,%1}, [%2];" : "=d"(d[0]), "=d"(d[1]) : "l"(p) : "memory");
}
template <int VW>
__device__ __forceinline__ void st_rw(double *p, const double (&d)[VW]) {
    static_assert(VW == 2, "128-bit stores only");
    asm volatile("st.global.L1::no_allocate.v2.f64 [%0], {%1,%2};" ::"l"(p), "d"(d[0]), "d"(d[1]) : "memory");
}
__device__ __forceinline__ int64_t ld_stream_i64(const int64_t *p) {
    int64_t v;
    asm volatile("ld.global.nc.L1::no_allocate.s64 %0, [%1];" : "=l"(v) : "l"(p));
    return v;
}
__device__ __forceinline__ double ld_stream_f64(const double *p) {
    double v;
    asm volatile("ld.global.nc.L1::no_allocate.f64 %0, [%1];" : "=d"(v) : "l"(p));
    return v;
}
template <int G>
__device__ __forceinline__ unsigned group_mask(int lane) {
    if constexpr (G == 32) {
        return 0xffffffffu;
    } else {
        return ((1u << G) - 1u) << (lane & ~(G - 1));
    }
}
// the sum over the group, the same bits on every lane of it
template <int G>
__device__ __forceinline__ double group_allreduce(double d, unsigned mask) {
#pragma unroll
    for (int o = G / 2; o > 0; o >>= 1) d += __shfl_xor_sync(mask, d, o, G);
    return d;
}

constexpr int kBlock = 256;

// grid for a grid-stride kernel: at most the CTAs resident at once, at most one per `per_cta` work items, at most `cap`
template <typename K>
int grid_for(K kernel, int64_t per_cta, int64_t work, int64_t cap, int *grid) {
    int sms = 0;
    int rc = hnh::device_sm_count(&sms);
    if (rc) return rc;
    int occ = 0;
    cudaError_t e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kernel, kBlock, 0);
    if (e != cudaSuccess) return hnh::check_cuda(e, "cudaOccupancyMaxActiveBlocksPerMultiprocessor");
    const int64_t need = (work + per_cta - 1) / per_cta;
    *grid = (int)std::max<int64_t>(1, std::min({need, (int64_t)sms * std::max(occ, 1), cap}));
    return HNH_OK;
}

bool aligned16(const void *p) { return ((uintptr_t)p & 15) == 0; }

// the width table of the fast kernels: R -> (G lanes per row, VW doubles per load, UN rows in flight), as
// HNH_DISPATCH_R in c_abi.cu
#define ROW_GATHER_DISPATCH(r, CALL)          \
    switch (r) {                              \
        case 4:   CALL(4, 2, 2, 2); break;    \
        case 8:   CALL(8, 4, 2, 4); break;    \
        case 16:  CALL(16, 8, 2, 4); break;   \
        case 32:  CALL(32, 16, 2, 4); break;  \
        case 64:  CALL(64, 32, 2, 4); break;  \
        case 128: CALL(128, 32, 2, 4); break; \
        case 256: CALL(256, 32, 2, 2); break; \
        default: break;                       \
    }

bool table_width(int r) { return r >= 4 && r <= 256 && (r & (r - 1)) == 0; }

}  // namespace
