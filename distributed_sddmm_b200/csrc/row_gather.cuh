// row_gather.cuh -- the device primitives of the row-owning gather kernels (kernels.cuh, gatv2.cu, sparse_attention.cu)
// and the warp reductions of the attention kernels: a group of G lanes owns one CSR row, gathered rows arrive in 128-bit
// loads, dots end in the group's xor-butterfly.  Gathers use the read-only path at the normal L2 policy (gathered
// factor rows are the only data with any reuse); index and value streams do not allocate in L1.
#pragma once
#include <cstdint>

#include "hnh_b200.h"
#include "launch.h"

namespace {

using hnh::kBlock;

template <int VW>
__device__ __forceinline__ void ld_gather(double (&d)[VW], const double *p) {
    static_assert(VW == 1 || VW == 2, "64- or 128-bit loads");
    if constexpr (VW == 2) {
        asm volatile("ld.global.nc.L1::no_allocate.v2.f64 {%0,%1}, [%2];" : "=d"(d[0]), "=d"(d[1]) : "l"(p));
    } else {
        d[0] = __ldg(p);
    }
}
// plain (coherent) vector load / store for read-modify-write of output rows
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
// coherent (non-.nc) streaming load: for `values`, which the same kernel overwrites
__device__ __forceinline__ double ld_rw_f64(const double *p) {
    double v;
    asm volatile("ld.global.L1::no_allocate.f64 %0, [%1];" : "=d"(v) : "l"(p) : "memory");
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
// the sum over the warp, on lane 0
__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) v += __shfl_down_sync(0xffffffffu, v, off);
    return v;
}

// the (max, count) pairs of max aggregation (graph_sage.cu) and max readout (graph_readout.cu): (m, c) absorbs one
// candidate x; the stored (z, n) absorbs another (m, c).  The larger maximum wins, equal maxima add their counts.
__device__ __forceinline__ void max_take(double &m, double &c, double x) {
    if (x > m) {
        m = x;
        c = 1.0;
    } else if (x == m) {
        c += 1.0;
    }
}
__device__ __forceinline__ void max_merge(double &z, double &n, double m, double c) {
    if (m > z) {
        z = m;
        n = c;
    } else if (m == z) {
        n += c;
    }
}

bool aligned16(const void *p) { return ((uintptr_t)p & 15) == 0; }

// The width table of the fast kernels: R -> (G lanes per row, VW doubles per vector load, UN rows in flight).
// 128-bit loads (VW = 2, the widest on sm_90) need 16-byte aligned operand rows.
#define HNH_DISPATCH_R(r, CALL, FALLBACK)     \
    switch (r) {                              \
        case 4:   CALL(4, 2, 2, 2); break;    \
        case 8:   CALL(8, 4, 2, 4); break;    \
        case 16:  CALL(16, 8, 2, 4); break;   \
        case 32:  CALL(32, 16, 2, 4); break;  \
        case 64:  CALL(64, 32, 2, 4); break;  \
        case 128: CALL(128, 32, 2, 4); break; \
        case 256: CALL(256, 32, 2, 2); break; \
        default: FALLBACK; break;             \
    }

bool table_width(int r) { return r >= 4 && r <= 256 && (r & (r - 1)) == 0; }

}  // namespace
