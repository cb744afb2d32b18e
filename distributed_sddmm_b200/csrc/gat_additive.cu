// gat_additive.cu -- the device operations of additive graph attention (GAT::set_attention("additive"), Velickovic
// et al. 2018) beyond the SDDMM / SpMM path and the edge softmax: per head, with P = X W (n x d, row-major),
//     s = P a1, t = P a2                    node scalars, one read of P           (node_scalars_kernel)
//     x_uv = LeakyReLU(s_u + t_v)            edge scores from node scalars         (edge_scores_kernel)
//     dP += ds a1^T + dt a2^T                the backward's rank-2 row update      (rank2_update_kernel)
// The row and column sums of the backward's edge gradient are hnh_edge_sum_f64 (edge_softmax.cu).
//
// The two row kernels run one warp per row: lanes stride the row in 16-byte pairs (scalars when a row or a vector is
// not 16-byte aligned), and a row's dot products end in a fixed shuffle tree.  No floating-point atomics: repeated
// calls give bit-identical results.
#include <algorithm>
#include <cstdint>

#include "hnh_b200.h"
#include "launch.h"

namespace {

using hnh::check_cuda;
using hnh::count_launch;
using hnh::set_error;

constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;

int grid_for(int64_t work_items, int64_t per_block, int *grid) {
    int sms = 0;
    int rc = hnh::device_sm_count(&sms);
    if (rc) return rc;
    const int64_t want = (work_items + per_block - 1) / per_block;
    *grid = (int)std::max<int64_t>(1, std::min<int64_t>(want, (int64_t)sms * 16));
    return HNH_OK;
}

bool aligned16(const void *p) { return ((uintptr_t)p & 15) == 0; }

__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) v += __shfl_down_sync(0xffffffffu, v, off);
    return v;
}

// s[i] = <P[i, :], a1>, t[i] = <P[i, :], a2>.  P is read once, with streaming loads; a1 and a2 stay in L1.
template <bool kPairs>
__global__ void __launch_bounds__(kThreads)
node_scalars_kernel(double *__restrict__ s, double *__restrict__ t, const double *__restrict__ P, const double *__restrict__ a1,
                    const double *__restrict__ a2, int64_t n, int64_t d) {
    const int lane = threadIdx.x & 31;
    const int64_t warps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t i = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; i < n; i += warps) {
        double x = 0.0, y = 0.0;
        if (kPairs) {
            const double2 *row = reinterpret_cast<const double2 *>(P + i * d);
            const double2 *u = reinterpret_cast<const double2 *>(a1), *w = reinterpret_cast<const double2 *>(a2);
            for (int64_t k = lane; k < d / 2; k += 32) {
                const double2 v = __ldcs(row + k), uk = __ldg(u + k), wk = __ldg(w + k);
                x = fma(v.x, uk.x, x);
                x = fma(v.y, uk.y, x);
                y = fma(v.x, wk.x, y);
                y = fma(v.y, wk.y, y);
            }
        } else {
            const double *row = P + i * d;
            for (int64_t k = lane; k < d; k += 32) {
                const double v = __ldcs(row + k);
                x = fma(v, __ldg(a1 + k), x);
                y = fma(v, __ldg(a2 + k), y);
            }
        }
        x = warp_sum(x);
        y = warp_sum(y);
        if (lane == 0) {
            s[i] = x;
            t[i] = y;
        }
    }
}

// out[k] = LeakyReLU(s[row_key[k]] + t[col_key[k]]) (as leaky_relu_kernel), or its derivative: 1 where the argument
// is > 0, alpha elsewhere (as leaky_relu_grad_kernel)
template <bool kDerivative>
__global__ void edge_scores_kernel(double *__restrict__ out, const double *__restrict__ s, const double *__restrict__ t,
                                   const int32_t *__restrict__ row_key, const int32_t *__restrict__ col_key, int64_t n, double alpha) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; k < n; k += stride) {
        const double x = s[row_key[k]] + t[col_key[k]];
        out[k] = kDerivative ? (x > 0.0 ? 1.0 : alpha) : fmax(x, 0.0) + fmin(x, 0.0) * alpha;
    }
}

// dP[i, :] += ds[i] a1 + dt[i] a2
template <bool kPairs>
__global__ void __launch_bounds__(kThreads)
rank2_update_kernel(double *__restrict__ dP, const double *__restrict__ ds, const double *__restrict__ dt,
                    const double *__restrict__ a1, const double *__restrict__ a2, int64_t n, int64_t d) {
    const int lane = threadIdx.x & 31;
    const int64_t warps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t i = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; i < n; i += warps) {
        const double x = ds[i], y = dt[i];
        if (kPairs) {
            double2 *row = reinterpret_cast<double2 *>(dP + i * d);
            const double2 *u = reinterpret_cast<const double2 *>(a1), *w = reinterpret_cast<const double2 *>(a2);
            for (int64_t k = lane; k < d / 2; k += 32) {
                double2 v = row[k];
                const double2 uk = __ldg(u + k), wk = __ldg(w + k);
                v.x += fma(x, uk.x, y * wk.x);
                v.y += fma(x, uk.y, y * wk.y);
                row[k] = v;
            }
        } else {
            double *row = dP + i * d;
            for (int64_t k = lane; k < d; k += 32) row[k] += fma(x, __ldg(a1 + k), y * __ldg(a2 + k));
        }
    }
}

}  // namespace

extern "C" {

int hnh_gat_node_scalars_f64(double *s, double *t, const double *P, const double *a1, const double *a2, int64_t n, int64_t d,
                             void *stream) {
    if (n < 0 || d < 0) return set_error(HNH_E_INVALID, "hnh_gat_node_scalars_f64: negative size");
    if (n == 0) return HNH_OK;
    if (!s || !t || (d > 0 && (!P || !a1 || !a2))) return set_error(HNH_E_INVALID, "hnh_gat_node_scalars_f64: null pointer");
    int grid;
    int rc = grid_for(n, kWarps, &grid);
    if (rc) return rc;
    cudaStream_t st = (cudaStream_t)stream;
    if (d % 2 == 0 && aligned16(P) && aligned16(a1) && aligned16(a2))
        node_scalars_kernel<true><<<grid, kThreads, 0, st>>>(s, t, P, a1, a2, n, d);
    else
        node_scalars_kernel<false><<<grid, kThreads, 0, st>>>(s, t, P, a1, a2, n, d);
    count_launch(1);
    return check_cuda(cudaGetLastError(), "node_scalars_kernel launch");
}

int hnh_gat_edge_scores_f64(double *out, const double *s, const double *t, const int32_t *row_key, const int32_t *col_key,
                            int64_t n, double alpha, int derivative, void *stream) {
    if (n < 0) return set_error(HNH_E_INVALID, "hnh_gat_edge_scores_f64: negative size");
    if (n == 0) return HNH_OK;
    if (!out || !s || !t || !row_key || !col_key) return set_error(HNH_E_INVALID, "hnh_gat_edge_scores_f64: null pointer");
    int grid;
    int rc = grid_for(n, kThreads * 4, &grid);
    if (rc) return rc;
    cudaStream_t st = (cudaStream_t)stream;
    if (derivative)
        edge_scores_kernel<true><<<grid, kThreads, 0, st>>>(out, s, t, row_key, col_key, n, alpha);
    else
        edge_scores_kernel<false><<<grid, kThreads, 0, st>>>(out, s, t, row_key, col_key, n, alpha);
    count_launch(1);
    return check_cuda(cudaGetLastError(), "edge_scores_kernel launch");
}

int hnh_gat_rank2_update_f64(double *dP, const double *ds, const double *dt, const double *a1, const double *a2, int64_t n,
                             int64_t d, void *stream) {
    if (n < 0 || d < 0) return set_error(HNH_E_INVALID, "hnh_gat_rank2_update_f64: negative size");
    if (n == 0 || d == 0) return HNH_OK;
    if (!dP || !ds || !dt || !a1 || !a2) return set_error(HNH_E_INVALID, "hnh_gat_rank2_update_f64: null pointer");
    int grid;
    int rc = grid_for(n, kWarps, &grid);
    if (rc) return rc;
    cudaStream_t st = (cudaStream_t)stream;
    if (d % 2 == 0 && aligned16(dP) && aligned16(a1) && aligned16(a2))
        rank2_update_kernel<true><<<grid, kThreads, 0, st>>>(dP, ds, dt, a1, a2, n, d);
    else
        rank2_update_kernel<false><<<grid, kThreads, 0, st>>>(dP, ds, dt, a1, a2, n, d);
    count_launch(1);
    return check_cuda(cudaGetLastError(), "rank2_update_kernel launch");
}

}  // extern "C"
