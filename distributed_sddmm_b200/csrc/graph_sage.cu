// graph_sage.cu -- max aggregation (Distributed_Sparse::maxAggregate, include/hnh/graph_sage.hpp) on one CSR block: the
// SpMM over the (max, .) semiring and its gradient.  With Y the gathered side (indexed by col_idx v) and the stored row u:
//     step:   (Z_u,k, C_u,k) = merge((Z_u,k, C_u,k), (max_v Y_v,k, #{v : Y_v,k == max}))      merge: larger max wins,
//                                                                                        equal maxima add their counts
//     grad:   dX_u,k += sum_v [X_u,k == Z_v,k] G_v,k            (B order: X's rows stored, [Z | G] gathered, G = dZ / C)
// The fast kernels follow link_bce_kernel (link_prediction.cu): a group of G lanes owns one CSR row; a chunk of G column
// indices is read coalesced and broadcast by shuffles; gathered rows come in with 128-bit loads, UN rows in flight per
// lane.  The step keeps the running (max, count) per column in registers and merges it into [Z | C] with one
// read-modify-write at the row end (the operand may ride a ring and carry the maxima of earlier blocks); the grad keeps
// X_u and the row's sum in registers and adds it to dX once at the row end.  The step has no floating-point sum at all
// (counts are small integers, exact in doubles); the grad sums in stored order.  Widths 4..256 (powers of two) with
// 16-byte aligned operands and even leading dimensions take them; every other window takes the one-warp-per-row generic
// kernel.  Wider rows run as column windows of 256: max is independent per column.  No atomics anywhere: repeated calls
// are bit-identical.
#include <cmath>

#include "row_gather.cuh"

namespace {

using hnh::grid_for;
using hnh::launch;
using hnh::set_error;

constexpr int kWindow = 256;  // the widest column window of one launch

// ---- fast row kernels ------------------------------------------------------------------------------------------------
template <int R, int G, int VW, int UN>
__global__ void __launch_bounds__(kBlock, 1)
max_aggregate_step_kernel(const int64_t *__restrict__ rowStart, const int64_t *__restrict__ col_idx, int64_t rows,
                          const double *__restrict__ X, int64_t ldx, double *__restrict__ Z, int64_t ldz,
                          double *__restrict__ C, int64_t ldc) {
    constexpr int NV = R / (G * VW);
    static_assert(NV * G * VW == R, "R must equal NV*G*VW");
    const int lane = threadIdx.x & 31;
    const int gl = lane & (G - 1);
    const unsigned gmask = group_mask<G>(lane);
    const int64_t ngroups = (int64_t)gridDim.x * (blockDim.x / G);
    for (int64_t row = (int64_t)blockIdx.x * (blockDim.x / G) + threadIdx.x / G; row < rows; row += ngroups) {
        const int64_t s = ld_stream_i64(rowStart + row);
        const int64_t e = ld_stream_i64(rowStart + row + 1);
        if (s == e) continue;  // nothing to merge
        double m[NV][VW], c[NV][VW];
#pragma unroll
        for (int v = 0; v < NV; v++)
#pragma unroll
            for (int w = 0; w < VW; w++) {
                m[v][w] = -INFINITY;
                c[v][w] = 0.0;
            }
        for (int64_t j = s; j < e; j += G) {
            const int cnt = (e - j < G) ? (int)(e - j) : G;
            const int64_t mycol = gl < cnt ? ld_stream_i64(col_idx + j + gl) : 0;
            for (int k0 = 0; k0 < cnt; k0 += UN) {
                double y[UN][NV][VW];
#pragma unroll
                for (int u = 0; u < UN; u++) {
                    const int k = k0 + u;
                    const int64_t col = __shfl_sync(gmask, mycol, k < G ? k : G - 1, G);
                    if (k < cnt) {
#pragma unroll
                        for (int v = 0; v < NV; v++) ld_gather<VW>(y[u][v], X + col * ldx + (v * G + gl) * VW);
                    } else {
#pragma unroll
                        for (int v = 0; v < NV; v++)
#pragma unroll
                            for (int w = 0; w < VW; w++) y[u][v][w] = -INFINITY;
                    }
                }
                // in stored order: which of tied +0.0 / -0.0 is kept depends on the order only
#pragma unroll
                for (int u = 0; u < UN; u++)
                    if (k0 + u < cnt) {
#pragma unroll
                        for (int v = 0; v < NV; v++)
#pragma unroll
                            for (int w = 0; w < VW; w++) max_take(m[v][w], c[v][w], y[u][v][w]);
                    }
            }
        }
#pragma unroll
        for (int v = 0; v < NV; v++) {
            double z[VW], n[VW];
            double *pz = Z + row * ldz + (v * G + gl) * VW, *pc = C + row * ldc + (v * G + gl) * VW;
            ld_rw<VW>(z, pz);
            ld_rw<VW>(n, pc);
#pragma unroll
            for (int w = 0; w < VW; w++) max_merge(z[w], n[w], m[v][w], c[v][w]);
            st_rw<VW>(pz, z);
            st_rw<VW>(pc, n);
        }
    }
}

template <int R, int G, int VW, int UN>
__global__ void __launch_bounds__(kBlock, 1)
max_aggregate_grad_kernel(const int64_t *__restrict__ rowStart, const int64_t *__restrict__ col_idx, int64_t rows,
                          const double *__restrict__ X, int64_t ldx, const double *__restrict__ Z, int64_t ldz,
                          const double *__restrict__ Gm, int64_t ldg, double *__restrict__ dX, int64_t lddx) {
    constexpr int NV = R / (G * VW);
    static_assert(NV * G * VW == R, "R must equal NV*G*VW");
    const int lane = threadIdx.x & 31;
    const int gl = lane & (G - 1);
    const unsigned gmask = group_mask<G>(lane);
    const int64_t ngroups = (int64_t)gridDim.x * (blockDim.x / G);
    for (int64_t row = (int64_t)blockIdx.x * (blockDim.x / G) + threadIdx.x / G; row < rows; row += ngroups) {
        const int64_t s = ld_stream_i64(rowStart + row);
        const int64_t e = ld_stream_i64(rowStart + row + 1);
        if (s == e) continue;  // nothing to add
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
                double z[UN][NV][VW], g[UN][NV][VW];
#pragma unroll
                for (int u = 0; u < UN; u++) {
                    const int k = k0 + u;
                    const int64_t col = __shfl_sync(gmask, mycol, k < G ? k : G - 1, G);
                    if (k < cnt) {
#pragma unroll
                        for (int v = 0; v < NV; v++) {
                            ld_gather<VW>(z[u][v], Z + col * ldz + (v * G + gl) * VW);
                            ld_gather<VW>(g[u][v], Gm + col * ldg + (v * G + gl) * VW);
                        }
                    } else {
#pragma unroll
                        for (int v = 0; v < NV; v++)
#pragma unroll
                            for (int w = 0; w < VW; w++) z[u][v][w] = g[u][v][w] = 0.0;
                    }
                }
#pragma unroll
                for (int u = 0; u < UN; u++)
                    if (k0 + u < cnt) {
#pragma unroll
                        for (int v = 0; v < NV; v++)
#pragma unroll
                            for (int w = 0; w < VW; w++)
                                if (x[v][w] == z[u][v][w]) acc[v][w] += g[u][v][w];
                    }
            }
        }
#pragma unroll
        for (int v = 0; v < NV; v++) {
            double o[VW];
            double *p = dX + row * lddx + (v * G + gl) * VW;
            ld_rw<VW>(o, p);
#pragma unroll
            for (int w = 0; w < VW; w++) o[w] += acc[v][w];
            st_rw<VW>(p, o);
        }
    }
}

// ---- generic kernels: any window width up to 256, any leading dimension, any alignment; one warp per row ---------------
// Lane l keeps columns l + 32 t (t < kS) of the row's state in registers, f <= 32 kS.
template <int kS>
__global__ void __launch_bounds__(kBlock, 1)
max_aggregate_step_generic_kernel(const int64_t *__restrict__ rowStart, const int64_t *__restrict__ col_idx, int64_t rows,
                                  const double *__restrict__ X, int64_t ldx, int f, double *__restrict__ Z, int64_t ldz,
                                  double *__restrict__ C, int64_t ldc) {
    const int lane = threadIdx.x & 31;
    const int64_t warps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t row = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; row < rows; row += warps) {
        const int64_t s = rowStart[row], e = rowStart[row + 1];
        if (s == e) continue;
        double m[kS], c[kS];
#pragma unroll
        for (int t = 0; t < kS; t++) {
            m[t] = -INFINITY;
            c[t] = 0.0;
        }
        for (int64_t j = s; j < e; j++) {
            const double *yr = X + col_idx[j] * ldx;
#pragma unroll
            for (int t = 0; t < kS; t++)
                if (lane + 32 * t < f) max_take(m[t], c[t], yr[lane + 32 * t]);
        }
#pragma unroll
        for (int t = 0; t < kS; t++) {
            const int k = lane + 32 * t;
            if (k < f) {
                double z = Z[row * ldz + k], n = C[row * ldc + k];
                max_merge(z, n, m[t], c[t]);
                Z[row * ldz + k] = z;
                C[row * ldc + k] = n;
            }
        }
    }
}

template <int kS>
__global__ void __launch_bounds__(kBlock, 1)
max_aggregate_grad_generic_kernel(const int64_t *__restrict__ rowStart, const int64_t *__restrict__ col_idx, int64_t rows,
                                  const double *__restrict__ X, int64_t ldx, const double *__restrict__ Z, int64_t ldz,
                                  const double *__restrict__ Gm, int64_t ldg, int f, double *__restrict__ dX, int64_t lddx) {
    const int lane = threadIdx.x & 31;
    const int64_t warps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t row = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; row < rows; row += warps) {
        const int64_t s = rowStart[row], e = rowStart[row + 1];
        if (s == e) continue;
        double x[kS], acc[kS];
#pragma unroll
        for (int t = 0; t < kS; t++) {
            const int k = lane + 32 * t;
            x[t] = k < f ? X[row * ldx + k] : 0.0;
            acc[t] = 0.0;
        }
        for (int64_t j = s; j < e; j++) {
            const int64_t col = col_idx[j];
#pragma unroll
            for (int t = 0; t < kS; t++) {
                const int k = lane + 32 * t;
                if (k < f && x[t] == Z[col * ldz + k]) acc[t] += Gm[col * ldg + k];
            }
        }
#pragma unroll
        for (int t = 0; t < kS; t++)
            if (lane + 32 * t < f) dX[row * lddx + lane + 32 * t] += acc[t];
    }
}

// ---- elementwise ----------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kBlock, 1) max_aggregate_finish_kernel(double *__restrict__ Z, const double *__restrict__ C, int64_t n) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride)
        if (C[i] == 0.0) Z[i] = 0.0;
}

__global__ void __launch_bounds__(kBlock, 1) max_aggregate_grad_scale_kernel(double *G, const double *dZ, const double *__restrict__ C,
                                                                             int64_t n) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
        const double c = C[i];
        G[i] = c == 0.0 ? 0.0 : dZ[i] / c;
    }
}

// the one-warp-per-row instantiation for a window of width f <= 256
template <typename K>
K pick_generic(int f, K k1, K k2, K k4, K k8) {
    return f <= 32 ? k1 : f <= 64 ? k2 : f <= 128 ? k4 : k8;
}

}  // namespace

extern "C" {

int hnh_max_aggregate_step_f64(const int64_t *rowStart, const int64_t *col_idx, int64_t rows, int64_t nnz, const double *X,
                               int64_t ldx, int f, double *Z, int64_t ldz, double *C, int64_t ldc, void *stream) {
    const char *who = "hnh_max_aggregate_step_f64";
    if (rows < 0 || nnz < 0) return set_error(HNH_E_INVALID, "%s: negative size", who);
    if (f < 1) return set_error(HNH_E_INVALID, "%s: f must be positive (got %d)", who, f);
    if (ldx < f || ldz < f || ldc < f) return set_error(HNH_E_INVALID, "%s: a leading dimension is below f = %d", who, f);
    if (rows == 0 || nnz == 0) return HNH_OK;
    if (!rowStart || !col_idx || !X || !Z || !C) return set_error(HNH_E_INVALID, "%s: null pointer", who);
    if (Z == X || C == X) return set_error(HNH_E_INVALID, "%s: an output may not be the input", who);
    if (Z == C) return set_error(HNH_E_INVALID, "%s: Z and C must be distinct", who);
    cudaStream_t st = (cudaStream_t)stream;
    int rc = HNH_OK;
    for (int c0 = 0; c0 < f && rc == HNH_OK; c0 += kWindow) {
        const int w = std::min(kWindow, f - c0);
        const double *Xw = X + c0;
        double *Zw = Z + c0, *Cw = C + c0;
        int grid = 0;
        if (table_width(w) && aligned16(Xw) && aligned16(Zw) && aligned16(Cw) && ldx % 2 == 0 && ldz % 2 == 0 && ldc % 2 == 0) {
#define MS(RR, G, VW, UN)                                                                                                  \
    {                                                                                                                      \
        auto k = max_aggregate_step_kernel<RR, G, VW, UN>;                                                                 \
        rc = grid_for(k, rows, kBlock / G, &grid);                                                                         \
        if (!rc) rc = launch(k, grid, kBlock, st, "max_aggregate_step_kernel", rowStart, col_idx, rows, Xw, ldx, Zw, ldz, Cw, ldc); \
    }
            HNH_DISPATCH_R(w, MS, )
#undef MS
            continue;
        }
        auto k = pick_generic(w, max_aggregate_step_generic_kernel<1>, max_aggregate_step_generic_kernel<2>,
                              max_aggregate_step_generic_kernel<4>, max_aggregate_step_generic_kernel<8>);
        rc = grid_for(k, rows, kBlock / 32, &grid);
        if (!rc) rc = launch(k, grid, kBlock, st, "max_aggregate_step_generic_kernel", rowStart, col_idx, rows, Xw, ldx, w, Zw, ldz, Cw, ldc);
    }
    return rc;
}

int hnh_max_aggregate_finish_f64(double *Z, const double *C, int64_t n, void *stream) {
    if (n < 0) return set_error(HNH_E_INVALID, "hnh_max_aggregate_finish_f64: negative size");
    if (n == 0) return HNH_OK;
    if (!Z || !C) return set_error(HNH_E_INVALID, "hnh_max_aggregate_finish_f64: null pointer");
    if ((const double *)Z == C) return set_error(HNH_E_INVALID, "hnh_max_aggregate_finish_f64: Z and C must be distinct");
    int grid = 0;
    int rc = grid_for(max_aggregate_finish_kernel, n, kBlock * 4, &grid);
    return rc ? rc : launch(max_aggregate_finish_kernel, grid, kBlock, (cudaStream_t)stream, "max_aggregate_finish_kernel", Z, C, n);
}

int hnh_max_aggregate_grad_scale_f64(double *G, const double *dZ, const double *C, int64_t n, void *stream) {
    if (n < 0) return set_error(HNH_E_INVALID, "hnh_max_aggregate_grad_scale_f64: negative size");
    if (n == 0) return HNH_OK;
    if (!G || !dZ || !C) return set_error(HNH_E_INVALID, "hnh_max_aggregate_grad_scale_f64: null pointer");
    if ((const double *)G == C) return set_error(HNH_E_INVALID, "hnh_max_aggregate_grad_scale_f64: G may not be C");
    int grid = 0;
    int rc = grid_for(max_aggregate_grad_scale_kernel, n, kBlock * 4, &grid);
    return rc ? rc
              : launch(max_aggregate_grad_scale_kernel, grid, kBlock, (cudaStream_t)stream, "max_aggregate_grad_scale_kernel", G, dZ,
                       C, n);
}

int hnh_max_aggregate_grad_f64(const int64_t *rowStart, const int64_t *col_idx, int64_t rows, int64_t nnz, const double *X,
                               int64_t ldx, const double *Z, int64_t ldz, const double *G, int64_t ldg, int f, double *dX,
                               int64_t lddx, void *stream) {
    const char *who = "hnh_max_aggregate_grad_f64";
    if (rows < 0 || nnz < 0) return set_error(HNH_E_INVALID, "%s: negative size", who);
    if (f < 1) return set_error(HNH_E_INVALID, "%s: f must be positive (got %d)", who, f);
    if (ldx < f || ldz < f || ldg < f || lddx < f) return set_error(HNH_E_INVALID, "%s: a leading dimension is below f = %d", who, f);
    if (rows == 0 || nnz == 0) return HNH_OK;
    if (!rowStart || !col_idx || !X || !Z || !G || !dX) return set_error(HNH_E_INVALID, "%s: null pointer", who);
    if (dX == X || dX == Z || dX == G) return set_error(HNH_E_INVALID, "%s: dX may not be an input", who);
    cudaStream_t st = (cudaStream_t)stream;
    int rc = HNH_OK;
    for (int c0 = 0; c0 < f && rc == HNH_OK; c0 += kWindow) {
        const int w = std::min(kWindow, f - c0);
        const double *Xw = X + c0, *Zw = Z + c0, *Gw = G + c0;
        double *dXw = dX + c0;
        int grid = 0;
        if (table_width(w) && aligned16(Xw) && aligned16(Zw) && aligned16(Gw) && aligned16(dXw) && ldx % 2 == 0 && ldz % 2 == 0 &&
            ldg % 2 == 0 && lddx % 2 == 0) {
#define MG(RR, G_, VW, UN)                                                                                                 \
    {                                                                                                                      \
        auto k = max_aggregate_grad_kernel<RR, G_, VW, UN>;                                                                \
        rc = grid_for(k, rows, kBlock / G_, &grid);                                                                        \
        if (!rc)                                                                                                           \
            rc = launch(k, grid, kBlock, st, "max_aggregate_grad_kernel", rowStart, col_idx, rows, Xw, ldx, Zw, ldz, Gw, ldg, dXw, lddx); \
    }
            HNH_DISPATCH_R(w, MG, )
#undef MG
            continue;
        }
        auto k = pick_generic(w, max_aggregate_grad_generic_kernel<1>, max_aggregate_grad_generic_kernel<2>,
                              max_aggregate_grad_generic_kernel<4>, max_aggregate_grad_generic_kernel<8>);
        rc = grid_for(k, rows, kBlock / 32, &grid);
        if (!rc)
            rc = launch(k, grid, kBlock, st, "max_aggregate_grad_generic_kernel", rowStart, col_idx, rows, Xw, ldx, Zw, ldz, Gw, ldg, w,
                        dXw, lddx);
    }
    return rc;
}

}  // extern "C"
