// gine.cu -- edge-ReLU aggregation (Distributed_Sparse::edgeReluAggregate, GINE's message ReLU(x_v + e_uv);
// include/hnh/gin.hpp) on one CSR block, its two gradients, and GIN's (1 + eps) combination.
//
// With u the stored row, v = col_idx of the block's entry i and E_i that entry's f-wide edge row (E + i lde):
//     step       A_u  += sum_i ReLU(X_v + E_i)                     (A order: A rides with the stored rows)
//     grad       dX_v += sum_i [X_v + E_i > 0] dA_u                (B order: X, dX stored; dA gathered)
//     edge_grad  dE_i  = [X_v + E_i > 0] dA_u                      (A order: dA stored; X gathered; written once)
// The mask is strict, as torch's relu backward: an entry with X_v + E_i == 0 passes no gradient.
// The fast kernels follow multi_aggregate_step_kernel (pna.cu): a group of G lanes owns one CSR row, a chunk of G
// column indices is read coalesced and broadcast by shuffles, gathered rows come in with 128-bit loads, UN rows in
// flight per lane.  The rows E_i of a chunk's entries are contiguous, so every lane reads its own slice of each beside
// the row it gathers: E is streamed once, coalesced, with an L2 evict-first policy so that it does not push the
// gathered rows, the only data with reuse, out of L2.  Sums run in stored order in registers, then one read-modify-write
// per row: the state may ride a ring and carry earlier blocks.  Widths 4..256 (powers of two) with 16-byte aligned
// operands and even leading dimensions take them; every other window takes the one-warp-per-row generic kernels.  Wider
// rows run as column windows of 256: every column is independent.  No atomics: repeated calls are bit-identical.
#include <cmath>

#include "row_gather.cuh"

namespace {

using hnh::grid_for;
using hnh::launch;
using hnh::set_error;

constexpr int kWindow = 256;  // the widest column window of one launch

// an L2 policy that evicts E's lines first: E is read once, the gathered rows are read by every row that has them
__device__ __forceinline__ uint64_t evict_first_policy() {
    uint64_t p;
    asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p));
    return p;
}
template <int VW>
__device__ __forceinline__ void ld_edge(double (&d)[VW], const double *p, uint64_t policy) {
    static_assert(VW == 2, "128-bit loads only");
    asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.v2.f64 {%0,%1}, [%2], %3;"
                 : "=d"(d[0]), "=d"(d[1])
                 : "l"(p), "l"(policy));
}
__device__ __forceinline__ double ld_edge1(const double *p, uint64_t policy) {
    double v;
    asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.f64 %0, [%1], %2;" : "=d"(v) : "l"(p), "l"(policy));
    return v;
}

__device__ __forceinline__ double relu(double s) { return s > 0.0 ? s : 0.0; }

// ---- fast row kernels ------------------------------------------------------------------------------------------------
template <int R, int G, int VW, int UN>
__global__ void __launch_bounds__(kBlock, 1)
edge_relu_step_kernel(const int64_t *__restrict__ rowStart, const int64_t *__restrict__ col_idx, int64_t rows,
                      const double *__restrict__ X, int64_t ldx, const double *__restrict__ E, int64_t lde, double *__restrict__ A,
                      int64_t lda) {
    constexpr int NV = R / (G * VW);
    static_assert(NV * G * VW == R, "R must equal NV*G*VW");
    const uint64_t pol = evict_first_policy();
    const int lane = threadIdx.x & 31;
    const int gl = lane & (G - 1);
    const unsigned gmask = group_mask<G>(lane);
    const int64_t ngroups = (int64_t)gridDim.x * (blockDim.x / G);
    for (int64_t row = (int64_t)blockIdx.x * (blockDim.x / G) + threadIdx.x / G; row < rows; row += ngroups) {
        const int64_t s = ld_stream_i64(rowStart + row);
        const int64_t e = ld_stream_i64(rowStart + row + 1);
        if (s == e) continue;  // nothing to add
        double acc[NV][VW];
#pragma unroll
        for (int v = 0; v < NV; v++)
#pragma unroll
            for (int w = 0; w < VW; w++) acc[v][w] = 0.0;
        for (int64_t j = s; j < e; j += G) {
            const int cnt = (e - j < G) ? (int)(e - j) : G;
            const int64_t mycol = gl < cnt ? ld_stream_i64(col_idx + j + gl) : 0;
            for (int k0 = 0; k0 < cnt; k0 += UN) {
                double y[UN][NV][VW], ev[UN][NV][VW];
#pragma unroll
                for (int u = 0; u < UN; u++) {
                    const int k = k0 + u;
                    const int64_t col = __shfl_sync(gmask, mycol, k < G ? k : G - 1, G);
#pragma unroll
                    for (int v = 0; v < NV; v++) {
                        if (k < cnt) {
                            ld_gather<VW>(y[u][v], X + col * ldx + (v * G + gl) * VW);
                            ld_edge<VW>(ev[u][v], E + (j + k) * lde + (v * G + gl) * VW, pol);
                        } else {
#pragma unroll
                            for (int w = 0; w < VW; w++) y[u][v][w] = ev[u][v][w] = 0.0;
                        }
                    }
                }
                // in stored order; padding slots past cnt add ReLU(0) = 0, which leaves the sums' bits as they are
#pragma unroll
                for (int u = 0; u < UN; u++)
#pragma unroll
                    for (int v = 0; v < NV; v++)
#pragma unroll
                        for (int w = 0; w < VW; w++) acc[v][w] += relu(y[u][v][w] + ev[u][v][w]);
            }
        }
#pragma unroll
        for (int v = 0; v < NV; v++) {
            double *p = A + row * lda + (v * G + gl) * VW;
            double o[VW];
            ld_rw<VW>(o, p);
#pragma unroll
            for (int w = 0; w < VW; w++) o[w] += acc[v][w];
            st_rw<VW>(p, o);
        }
    }
}

template <int R, int G, int VW, int UN>
__global__ void __launch_bounds__(kBlock, 1)
edge_relu_grad_kernel(const int64_t *__restrict__ rowStart, const int64_t *__restrict__ col_idx, int64_t rows,
                      const double *__restrict__ X, int64_t ldx, const double *__restrict__ E, int64_t lde,
                      const double *__restrict__ dA, int64_t ldda, double *__restrict__ dX, int64_t lddx) {
    constexpr int NV = R / (G * VW);
    static_assert(NV * G * VW == R, "R must equal NV*G*VW");
    const uint64_t pol = evict_first_policy();
    const int lane = threadIdx.x & 31;
    const int gl = lane & (G - 1);
    const unsigned gmask = group_mask<G>(lane);
    const int64_t ngroups = (int64_t)gridDim.x * (blockDim.x / G);
    for (int64_t row = (int64_t)blockIdx.x * (blockDim.x / G) + threadIdx.x / G; row < rows; row += ngroups) {
        const int64_t s = ld_stream_i64(rowStart + row);
        const int64_t e = ld_stream_i64(rowStart + row + 1);
        if (s == e) continue;
        double x[NV][VW], acc[NV][VW];
#pragma unroll
        for (int v = 0; v < NV; v++) {
            ld_gather<VW>(x[v], X + row * ldx + (v * G + gl) * VW);
#pragma unroll
            for (int w = 0; w < VW; w++) acc[v][w] = 0.0;
        }
        for (int64_t j = s; j < e; j += G) {
            const int cnt = (e - j < G) ? (int)(e - j) : G;
            const int64_t mycol = gl < cnt ? ld_stream_i64(col_idx + j + gl) : 0;
            for (int k0 = 0; k0 < cnt; k0 += UN) {
                double d[UN][NV][VW], ev[UN][NV][VW];
#pragma unroll
                for (int u = 0; u < UN; u++) {
                    const int k = k0 + u;
                    const int64_t col = __shfl_sync(gmask, mycol, k < G ? k : G - 1, G);
#pragma unroll
                    for (int v = 0; v < NV; v++) {
                        if (k < cnt) {
                            ld_gather<VW>(d[u][v], dA + col * ldda + (v * G + gl) * VW);
                            ld_edge<VW>(ev[u][v], E + (j + k) * lde + (v * G + gl) * VW, pol);
                        } else {
#pragma unroll
                            for (int w = 0; w < VW; w++) d[u][v][w] = ev[u][v][w] = 0.0;
                        }
                    }
                }
#pragma unroll
                for (int u = 0; u < UN; u++)
#pragma unroll
                    for (int v = 0; v < NV; v++)
#pragma unroll
                        for (int w = 0; w < VW; w++)
                            if (x[v][w] + ev[u][v][w] > 0.0) acc[v][w] += d[u][v][w];  // padding: d = 0
            }
        }
#pragma unroll
        for (int v = 0; v < NV; v++) {
            double *p = dX + row * lddx + (v * G + gl) * VW;
            double o[VW];
            ld_rw<VW>(o, p);
#pragma unroll
            for (int w = 0; w < VW; w++) o[w] += acc[v][w];
            st_rw<VW>(p, o);
        }
    }
}

template <int R, int G, int VW, int UN>
__global__ void __launch_bounds__(kBlock, 1)
edge_relu_edge_grad_kernel(const int64_t *__restrict__ rowStart, const int64_t *__restrict__ col_idx, int64_t rows,
                           const double *__restrict__ dA, int64_t ldda, const double *__restrict__ X, int64_t ldx,
                           const double *__restrict__ E, int64_t lde, double *__restrict__ dE, int64_t ldde) {
    constexpr int NV = R / (G * VW);
    static_assert(NV * G * VW == R, "R must equal NV*G*VW");
    const uint64_t pol = evict_first_policy();
    const int lane = threadIdx.x & 31;
    const int gl = lane & (G - 1);
    const unsigned gmask = group_mask<G>(lane);
    const int64_t ngroups = (int64_t)gridDim.x * (blockDim.x / G);
    for (int64_t row = (int64_t)blockIdx.x * (blockDim.x / G) + threadIdx.x / G; row < rows; row += ngroups) {
        const int64_t s = ld_stream_i64(rowStart + row);
        const int64_t e = ld_stream_i64(rowStart + row + 1);
        if (s == e) continue;
        double da[NV][VW];
#pragma unroll
        for (int v = 0; v < NV; v++) ld_gather<VW>(da[v], dA + row * ldda + (v * G + gl) * VW);
        for (int64_t j = s; j < e; j += G) {
            const int cnt = (e - j < G) ? (int)(e - j) : G;
            const int64_t mycol = gl < cnt ? ld_stream_i64(col_idx + j + gl) : 0;
            for (int k0 = 0; k0 < cnt; k0 += UN) {
                double y[UN][NV][VW], ev[UN][NV][VW];
#pragma unroll
                for (int u = 0; u < UN; u++) {
                    const int k = k0 + u;
                    const int64_t col = __shfl_sync(gmask, mycol, k < G ? k : G - 1, G);
                    if (k < cnt) {
#pragma unroll
                        for (int v = 0; v < NV; v++) {
                            ld_gather<VW>(y[u][v], X + col * ldx + (v * G + gl) * VW);
                            ld_edge<VW>(ev[u][v], E + (j + k) * lde + (v * G + gl) * VW, pol);
                        }
                    }
                }
#pragma unroll
                for (int u = 0; u < UN; u++)
                    if (k0 + u < cnt) {
#pragma unroll
                        for (int v = 0; v < NV; v++) {
                            double o[VW];
#pragma unroll
                            for (int w = 0; w < VW; w++) o[w] = y[u][v][w] + ev[u][v][w] > 0.0 ? da[v][w] : 0.0;
                            st_rw<VW>(dE + (j + k0 + u) * ldde + (v * G + gl) * VW, o);
                        }
                    }
            }
        }
    }
}

// ---- generic kernels: any window width up to 256, any leading dimension, any alignment; one warp per row ---------------
// Lane l owns columns l + 32 t (t < kS) of the row, width <= 32 kS.
template <int kS>
__global__ void __launch_bounds__(kBlock, 1)
edge_relu_step_generic_kernel(const int64_t *__restrict__ rowStart, const int64_t *__restrict__ col_idx, int64_t rows,
                              const double *__restrict__ X, int64_t ldx, const double *__restrict__ E, int64_t lde, int width,
                              double *__restrict__ A, int64_t lda) {
    const uint64_t pol = evict_first_policy();
    const int lane = threadIdx.x & 31;
    const int64_t warps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t row = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; row < rows; row += warps) {
        const int64_t s = rowStart[row], e = rowStart[row + 1];
        if (s == e) continue;
        double acc[kS];
#pragma unroll
        for (int t = 0; t < kS; t++) acc[t] = 0.0;
        for (int64_t j = s; j < e; j++) {
            const double *xr = X + col_idx[j] * ldx, *er = E + j * lde;
#pragma unroll
            for (int t = 0; t < kS; t++) {
                const int k = lane + 32 * t;
                if (k < width) acc[t] += relu(xr[k] + ld_edge1(er + k, pol));
            }
        }
#pragma unroll
        for (int t = 0; t < kS; t++) {
            const int k = lane + 32 * t;
            if (k < width) A[row * lda + k] += acc[t];
        }
    }
}

template <int kS>
__global__ void __launch_bounds__(kBlock, 1)
edge_relu_grad_generic_kernel(const int64_t *__restrict__ rowStart, const int64_t *__restrict__ col_idx, int64_t rows,
                              const double *__restrict__ X, int64_t ldx, const double *__restrict__ E, int64_t lde,
                              const double *__restrict__ dA, int64_t ldda, int width, double *__restrict__ dX, int64_t lddx) {
    const uint64_t pol = evict_first_policy();
    const int lane = threadIdx.x & 31;
    const int64_t warps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t row = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; row < rows; row += warps) {
        const int64_t s = rowStart[row], e = rowStart[row + 1];
        if (s == e) continue;
        double x[kS], acc[kS];
#pragma unroll
        for (int t = 0; t < kS; t++) {
            const int k = lane + 32 * t;
            x[t] = k < width ? X[row * ldx + k] : 0.0;
            acc[t] = 0.0;
        }
        for (int64_t j = s; j < e; j++) {
            const double *dr = dA + col_idx[j] * ldda, *er = E + j * lde;
#pragma unroll
            for (int t = 0; t < kS; t++) {
                const int k = lane + 32 * t;
                if (k < width && x[t] + ld_edge1(er + k, pol) > 0.0) acc[t] += dr[k];
            }
        }
#pragma unroll
        for (int t = 0; t < kS; t++) {
            const int k = lane + 32 * t;
            if (k < width) dX[row * lddx + k] += acc[t];
        }
    }
}

template <int kS>
__global__ void __launch_bounds__(kBlock, 1)
edge_relu_edge_grad_generic_kernel(const int64_t *__restrict__ rowStart, const int64_t *__restrict__ col_idx, int64_t rows,
                                   const double *__restrict__ dA, int64_t ldda, const double *__restrict__ X, int64_t ldx,
                                   const double *__restrict__ E, int64_t lde, int width, double *__restrict__ dE, int64_t ldde) {
    const uint64_t pol = evict_first_policy();
    const int lane = threadIdx.x & 31;
    const int64_t warps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t row = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; row < rows; row += warps) {
        const int64_t s = rowStart[row], e = rowStart[row + 1];
        if (s == e) continue;
        double da[kS];
#pragma unroll
        for (int t = 0; t < kS; t++) {
            const int k = lane + 32 * t;
            da[t] = k < width ? dA[row * ldda + k] : 0.0;
        }
        for (int64_t j = s; j < e; j++) {
            const double *xr = X + col_idx[j] * ldx, *er = E + j * lde;
#pragma unroll
            for (int t = 0; t < kS; t++) {
                const int k = lane + 32 * t;
                if (k < width) dE[j * ldde + k] = xr[k] + ld_edge1(er + k, pol) > 0.0 ? da[t] : 0.0;
            }
        }
    }
}

// ---- GIN's combination -----------------------------------------------------------------------------------------------
// H = M + (1 + eps) X over n elements, eps read on the device
__global__ void __launch_bounds__(kBlock, 1) gin_combine_kernel(double *__restrict__ H, const double *__restrict__ M,
                                                                const double *__restrict__ X, const double *__restrict__ eps,
                                                                int64_t n) {
    const double a = 1.0 + *eps;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) H[i] = fma(a, X[i], M[i]);
}

// dX = (1 + eps) dH over n elements; with `partial`, each CTA's share of sum dH X (fixed order) into partial[blockIdx.x]
__global__ void __launch_bounds__(kBlock, 1) gin_combine_grad_kernel(double *__restrict__ dX, double *__restrict__ partial,
                                                                     const double *__restrict__ dH, const double *__restrict__ X,
                                                                     const double *__restrict__ eps, int64_t n) {
    __shared__ double warp_sums[kBlock / 32];
    const double a = 1.0 + *eps;
    double acc = 0.0;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
        const double g = dH[i];
        dX[i] = a * g;
        if (partial) acc = fma(g, X[i], acc);
    }
    if (!partial) return;
    acc = group_allreduce<32>(acc, 0xffffffffu);
    if ((threadIdx.x & 31) == 0) warp_sums[threadIdx.x >> 5] = acc;
    __syncthreads();
    if (threadIdx.x == 0) {
        double t = 0.0;
        for (int w = 0; w < kBlock / 32; w++) t += warp_sums[w];
        partial[blockIdx.x] = t;
    }
}

__global__ void __launch_bounds__(kBlock, 1) gin_sum_partials_kernel(double *__restrict__ out, const double *__restrict__ partial, int n) {
    __shared__ double warp_sums[kBlock / 32];
    double acc = 0.0;
    for (int i = threadIdx.x; i < n; i += blockDim.x) acc += partial[i];
    acc = group_allreduce<32>(acc, 0xffffffffu);
    if ((threadIdx.x & 31) == 0) warp_sums[threadIdx.x >> 5] = acc;
    __syncthreads();
    if (threadIdx.x == 0) {
        double t = 0.0;
        for (int w = 0; w < kBlock / 32; w++) t += warp_sums[w];
        *out = t;
    }
}

// the one-warp-per-row instantiation for a window of width w <= 256
template <typename K>
K pick_generic(int w, K k1, K k2, K k4, K k8) {
    return w <= 32 ? k1 : w <= 64 ? k2 : w <= 128 ? k4 : k8;
}

// the checks every edge-ReLU entry point shares
int check_edge_relu(const char *who, int64_t rows, int64_t nnz, int f, std::initializer_list<int64_t> lds) {
    if (rows < 0 || nnz < 0) return set_error(HNH_E_INVALID, "%s: negative size", who);
    if (f < 1) return set_error(HNH_E_INVALID, "%s: f must be positive (got %d)", who, f);
    for (int64_t ld : lds)
        if (ld < f) return set_error(HNH_E_INVALID, "%s: a leading dimension is below f = %d", who, f);
    return HNH_OK;
}
bool even(std::initializer_list<int64_t> lds) {
    for (int64_t ld : lds)
        if (ld % 2 != 0) return false;
    return true;
}

}  // namespace

extern "C" {

int hnh_edge_relu_aggregate_step_f64(const int64_t *rowStart, const int64_t *col_idx, int64_t rows, int64_t nnz, const double *X,
                                     int64_t ldx, const double *E, int64_t lde, int f, double *A, int64_t lda, void *stream) {
    const char *who = "hnh_edge_relu_aggregate_step_f64";
    if (int rc = check_edge_relu(who, rows, nnz, f, {ldx, lde, lda})) return rc;
    if (rows == 0 || nnz == 0) return HNH_OK;
    if (!rowStart || !col_idx || !X || !E || !A) return set_error(HNH_E_INVALID, "%s: null pointer", who);
    if (A == X || A == E) return set_error(HNH_E_INVALID, "%s: A may not be an input", who);
    cudaStream_t st = (cudaStream_t)stream;
    int rc = HNH_OK;
    for (int c0 = 0; c0 < f && rc == HNH_OK; c0 += kWindow) {
        const int w = std::min(kWindow, f - c0);
        const double *Xw = X + c0, *Ew = E + c0;
        double *Aw = A + c0;
        int grid = 0;
        if (table_width(w) && aligned16(Xw) && aligned16(Ew) && aligned16(Aw) && even({ldx, lde, lda})) {
#define ES(RR, G, VW, UN)                                                                                                  \
    {                                                                                                                      \
        auto k = edge_relu_step_kernel<RR, G, VW, UN>;                                                                     \
        rc = grid_for(k, rows, kBlock / G, &grid);                                                                         \
        if (!rc) rc = launch(k, grid, kBlock, st, "edge_relu_step_kernel", rowStart, col_idx, rows, Xw, ldx, Ew, lde, Aw, lda); \
    }
            HNH_DISPATCH_R(w, ES, )
#undef ES
            continue;
        }
        auto k = pick_generic(w, edge_relu_step_generic_kernel<1>, edge_relu_step_generic_kernel<2>, edge_relu_step_generic_kernel<4>,
                              edge_relu_step_generic_kernel<8>);
        rc = grid_for(k, rows, kBlock / 32, &grid);
        if (!rc) rc = launch(k, grid, kBlock, st, "edge_relu_step_generic_kernel", rowStart, col_idx, rows, Xw, ldx, Ew, lde, w, Aw, lda);
    }
    return rc;
}

int hnh_edge_relu_aggregate_grad_f64(const int64_t *rowStart, const int64_t *col_idx, int64_t rows, int64_t nnz, const double *X,
                                     int64_t ldx, const double *E, int64_t lde, const double *dA, int64_t ldda, int f, double *dX,
                                     int64_t lddx, void *stream) {
    const char *who = "hnh_edge_relu_aggregate_grad_f64";
    if (int rc = check_edge_relu(who, rows, nnz, f, {ldx, lde, ldda, lddx})) return rc;
    if (rows == 0 || nnz == 0) return HNH_OK;
    if (!rowStart || !col_idx || !X || !E || !dA || !dX) return set_error(HNH_E_INVALID, "%s: null pointer", who);
    if (dX == X || dX == E || dX == dA) return set_error(HNH_E_INVALID, "%s: dX may not be an input", who);
    cudaStream_t st = (cudaStream_t)stream;
    int rc = HNH_OK;
    for (int c0 = 0; c0 < f && rc == HNH_OK; c0 += kWindow) {
        const int w = std::min(kWindow, f - c0);
        const double *Xw = X + c0, *Ew = E + c0, *dAw = dA + c0;
        double *dXw = dX + c0;
        int grid = 0;
        if (table_width(w) && aligned16(Xw) && aligned16(Ew) && aligned16(dAw) && aligned16(dXw) && even({ldx, lde, ldda, lddx})) {
#define EG(RR, G, VW, UN)                                                                                                  \
    {                                                                                                                      \
        auto k = edge_relu_grad_kernel<RR, G, VW, UN>;                                                                     \
        rc = grid_for(k, rows, kBlock / G, &grid);                                                                         \
        if (!rc)                                                                                                           \
            rc = launch(k, grid, kBlock, st, "edge_relu_grad_kernel", rowStart, col_idx, rows, Xw, ldx, Ew, lde, dAw, ldda, dXw, lddx); \
    }
            HNH_DISPATCH_R(w, EG, )
#undef EG
            continue;
        }
        auto k = pick_generic(w, edge_relu_grad_generic_kernel<1>, edge_relu_grad_generic_kernel<2>, edge_relu_grad_generic_kernel<4>,
                              edge_relu_grad_generic_kernel<8>);
        rc = grid_for(k, rows, kBlock / 32, &grid);
        if (!rc)
            rc = launch(k, grid, kBlock, st, "edge_relu_grad_generic_kernel", rowStart, col_idx, rows, Xw, ldx, Ew, lde, dAw, ldda, w, dXw,
                        lddx);
    }
    return rc;
}

int hnh_edge_relu_aggregate_edge_grad_f64(const int64_t *rowStart, const int64_t *col_idx, int64_t rows, int64_t nnz,
                                          const double *dA, int64_t ldda, const double *X, int64_t ldx, const double *E, int64_t lde,
                                          int f, double *dE, int64_t ldde, void *stream) {
    const char *who = "hnh_edge_relu_aggregate_edge_grad_f64";
    if (int rc = check_edge_relu(who, rows, nnz, f, {ldda, ldx, lde, ldde})) return rc;
    if (rows == 0 || nnz == 0) return HNH_OK;
    if (!rowStart || !col_idx || !dA || !X || !E || !dE) return set_error(HNH_E_INVALID, "%s: null pointer", who);
    if (dE == X || dE == E || dE == dA) return set_error(HNH_E_INVALID, "%s: dE may not be an input", who);
    cudaStream_t st = (cudaStream_t)stream;
    int rc = HNH_OK;
    for (int c0 = 0; c0 < f && rc == HNH_OK; c0 += kWindow) {
        const int w = std::min(kWindow, f - c0);
        const double *dAw = dA + c0, *Xw = X + c0, *Ew = E + c0;
        double *dEw = dE + c0;
        int grid = 0;
        if (table_width(w) && aligned16(dAw) && aligned16(Xw) && aligned16(Ew) && aligned16(dEw) && even({ldda, ldx, lde, ldde})) {
#define EE(RR, G, VW, UN)                                                                                                  \
    {                                                                                                                      \
        auto k = edge_relu_edge_grad_kernel<RR, G, VW, UN>;                                                                \
        rc = grid_for(k, rows, kBlock / G, &grid);                                                                         \
        if (!rc)                                                                                                           \
            rc = launch(k, grid, kBlock, st, "edge_relu_edge_grad_kernel", rowStart, col_idx, rows, dAw, ldda, Xw, ldx, Ew, lde, dEw, ldde); \
    }
            HNH_DISPATCH_R(w, EE, )
#undef EE
            continue;
        }
        auto k = pick_generic(w, edge_relu_edge_grad_generic_kernel<1>, edge_relu_edge_grad_generic_kernel<2>,
                              edge_relu_edge_grad_generic_kernel<4>, edge_relu_edge_grad_generic_kernel<8>);
        rc = grid_for(k, rows, kBlock / 32, &grid);
        if (!rc)
            rc = launch(k, grid, kBlock, st, "edge_relu_edge_grad_generic_kernel", rowStart, col_idx, rows, dAw, ldda, Xw, ldx, Ew, lde, w,
                        dEw, ldde);
    }
    return rc;
}

int hnh_gin_combine_f64(double *H, const double *M, const double *X, const double *eps, int64_t n, void *stream) {
    if (n < 0) return set_error(HNH_E_INVALID, "hnh_gin_combine_f64: negative size");
    if (n == 0) return HNH_OK;
    if (!H || !M || !X || !eps) return set_error(HNH_E_INVALID, "hnh_gin_combine_f64: null pointer");
    if (H == X) return set_error(HNH_E_INVALID, "hnh_gin_combine_f64: H may not be X");
    int grid = 0;
    int rc = grid_for(gin_combine_kernel, n, kBlock * 4, &grid);
    return rc ? rc : launch(gin_combine_kernel, grid, kBlock, (cudaStream_t)stream, "gin_combine_kernel", H, M, X, eps, n);
}

int hnh_gin_combine_grad_f64(double *dX, double *deps, const double *dH, const double *X, const double *eps, int64_t n, void *stream) {
    const char *who = "hnh_gin_combine_grad_f64";
    if (n < 0) return set_error(HNH_E_INVALID, "%s: negative size", who);
    cudaStream_t st = (cudaStream_t)stream;
    if (n == 0) return deps ? hnh::check_cuda(cudaMemsetAsync(deps, 0, sizeof(double), st), "cudaMemsetAsync") : HNH_OK;
    if (!dX || !dH || !eps || (deps && !X)) return set_error(HNH_E_INVALID, "%s: null pointer", who);
    if (dX == dH || dX == X) return set_error(HNH_E_INVALID, "%s: dX may not be an input", who);
    int grid = 0;
    int rc = grid_for(gin_combine_grad_kernel, n, kBlock * 4, &grid);
    if (rc) return rc;
    if (!deps) return launch(gin_combine_grad_kernel, grid, kBlock, st, "gin_combine_grad_kernel", dX, (double *)nullptr, dH, X, eps, n);
    // per-call scratch, stream-ordered; the grid, and so the order of the sum, depends on the device and n only
    double *partial = nullptr;
    rc = hnh::check_cuda(cudaMallocAsync((void **)&partial, sizeof(double) * (size_t)grid, st), "cudaMallocAsync");
    if (rc) return rc;
    rc = launch(gin_combine_grad_kernel, grid, kBlock, st, "gin_combine_grad_kernel", dX, partial, dH, X, eps, n);
    if (!rc) rc = launch(gin_sum_partials_kernel, 1, kBlock, st, "gin_sum_partials_kernel", deps, (const double *)partial, grid);
    cudaError_t e = cudaFreeAsync(partial, st);
    return rc ? rc : hnh::check_cuda(e, "cudaFreeAsync");
}

}  // extern "C"
