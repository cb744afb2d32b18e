// edge_softmax.cu -- the row softmax over the stored entries of S (Distributed_Sparse::edgeSoftmax): the step between
// an SDDMM and an SpMM in graph attention, alpha_uv = exp(x_uv - m_u) / s_u with m_u the row maximum and s_u the
// row sum of exp(x_uv - m_u), and its backward dx_uv = alpha_uv (dalpha_uv - t_u) with t_u = sum_v alpha_uv dalpha_uv.
//
// A value vector is in the order of the CSR blocks it belongs to (A and B orders differ, fusion-1 blocks are stored
// transposed), so the row reductions work through a plan built once per order (hnh_edge_softmax_plan): `perm`
// groups the entries by global row (a stable radix sort of their row keys), `row_start` delimits each row's run in
// it, and every run is cut into pieces of at most kPiece entries.  A reduction is two launches: one warp per piece
// (lanes stride the piece in a fixed order, then a fixed shuffle tree), then one warp per row over its pieces the
// same way.  Long rows are spread over many warps, short rows cost one warp, and the summation order is a function of
// the plan alone: no floating-point atomics, repeated calls give bit-identical results.  The elementwise steps run
// in the vector's own order.
#include <cub/cub.cuh>

#include <cmath>

#include "row_gather.cuh"

namespace {

using hnh::bits_for;
using hnh::check_cuda;
using hnh::grid_for;
using hnh::launch;
using hnh::Scratch;
using hnh::set_error;

constexpr int kCtasPerSm = 16;  // grid cap of every kernel here
constexpr int kPiece = 1024;    // entries of a row that one warp reduces

// (m, s) <- the (max, sum of exp(x - max)) of the union of two sets; (-inf, 0) is the empty set
__device__ __forceinline__ void ms_merge(double &m, double &s, double m2, double s2) {
    if (m2 == -INFINITY) return;
    if (m == -INFINITY) {
        m = m2;
        s = s2;
    } else if (m2 > m) {
        s = s * exp(m - m2) + s2;
        m = m2;
    } else {
        s += s2 * exp(m2 - m);
    }
}

__device__ __forceinline__ void ms_warp_reduce(double &m, double &s) {
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) {
        const double m2 = __shfl_down_sync(0xffffffffu, m, off), s2 = __shfl_down_sync(0xffffffffu, s, off);
        ms_merge(m, s, m2, s2);
    }
}

// the positions [lo, hi) in perm order of piece q
__device__ __forceinline__ void piece_range(int64_t q, const int32_t *row_start, const int32_t *piece_first,
                                            const int32_t *piece_row, int64_t *lo, int64_t *hi) {
    const int u = piece_row[q];
    *lo = (int64_t)row_start[u] + (q - (int64_t)piece_first[u]) * kPiece;
    *hi = min(*lo + kPiece, (int64_t)row_start[u + 1]);
}

// ---- plan ---------------------------------------------------------------------------------------------------
__global__ void keys_check_iota_kernel(const int32_t *__restrict__ keys, int64_t n, int64_t num_rows, int32_t *__restrict__ idx,
                                       int *bad) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
        if (keys[i] < 0 || keys[i] >= num_rows) *bad = 1;
        idx[i] = (int32_t)i;
    }
}

// row_start[u] = first position with sorted[p] >= u (u = 0 .. num_rows); count[u] = pieces of row u, count[num_rows] = 0
__global__ void row_start_kernel(const int32_t *__restrict__ sorted, int64_t n, int64_t num_rows, int32_t *__restrict__ row_start) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t u = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; u <= num_rows; u += stride) {
        int64_t lo = 0, hi = n;
        while (lo < hi) {
            const int64_t mid = (lo + hi) >> 1;
            if (sorted[mid] < u) lo = mid + 1; else hi = mid;
        }
        row_start[u] = (int32_t)lo;
    }
}

__global__ void piece_count_kernel(const int32_t *__restrict__ row_start, int64_t num_rows, int32_t *__restrict__ count) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t u = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; u <= num_rows; u += stride)
        count[u] = u < num_rows ? (row_start[u + 1] - row_start[u] + kPiece - 1) / kPiece : 0;
}

__global__ void piece_row_kernel(const int32_t *__restrict__ piece_first, int64_t num_rows, int32_t *__restrict__ piece_row) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t u = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; u < num_rows; u += stride)
        for (int32_t q = piece_first[u]; q < piece_first[u + 1]; q++) piece_row[q] = (int32_t)u;
}

__global__ void keys_from_index_kernel(int32_t *__restrict__ keys, const int64_t *__restrict__ idx, int64_t n, int64_t offset) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) keys[i] = (int32_t)(idx[i] + offset);
}

// ---- forward ------------------------------------------------------------------------------------------------
// one warp per piece: (max, sum of exp(x - max)) over x[perm[lo .. hi)].  A -inf entry (a masked edge) adds nothing:
// exp(v - m) would be NaN while the lane's running max is still -inf.
__global__ void piece_stats_kernel(const double *__restrict__ x, const int32_t *__restrict__ perm, const int32_t *__restrict__ row_start,
                                   const int32_t *__restrict__ piece_first, const int32_t *__restrict__ piece_row, int64_t num_pieces,
                                   double *__restrict__ piece_max, double *__restrict__ piece_sum) {
    const int lane = threadIdx.x & 31;
    const int64_t warps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t q = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; q < num_pieces; q += warps) {
        int64_t lo, hi;
        piece_range(q, row_start, piece_first, piece_row, &lo, &hi);
        double m = -INFINITY, s = 0.0;
        for (int64_t p = lo + lane; p < hi; p += 32) {
            const double v = x[perm[p]];
            if (v > m) {
                s = s * exp(m - v) + 1.0;
                m = v;
            } else if (v != -INFINITY) {
                s += exp(v - m);
            }
        }
        ms_warp_reduce(m, s);
        if (lane == 0) {
            piece_max[q] = m;
            piece_sum[q] = s;
        }
    }
}

// one warp per row: merge the row's pieces; rows without entries get (-inf, 0)
__global__ void row_stats_kernel(const int32_t *__restrict__ piece_first, int64_t num_rows, const double *__restrict__ piece_max,
                                 const double *__restrict__ piece_sum, double *__restrict__ row_max, double *__restrict__ row_sum) {
    const int lane = threadIdx.x & 31;
    const int64_t warps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t u = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; u < num_rows; u += warps) {
        double m = -INFINITY, s = 0.0;
        for (int64_t q = piece_first[u] + lane; q < piece_first[u + 1]; q += 32) ms_merge(m, s, piece_max[q], piece_sum[q]);
        ms_warp_reduce(m, s);
        if (lane == 0) {
            row_max[u] = m;
            row_sum[u] = s;
        }
    }
}

__global__ void rescale_kernel(double *__restrict__ row_sum, const double *__restrict__ local_max, const double *__restrict__ global_max,
                               int64_t num_rows) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t u = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; u < num_rows; u += stride) {
        const double ml = local_max[u];
        row_sum[u] = ml == -INFINITY ? 0.0 : row_sum[u] * exp(ml - global_max[u]);
    }
}

// alpha may alias x
__global__ void apply_kernel(double *alpha, const double *x, const int32_t *__restrict__ keys, int64_t n,
                             const double *__restrict__ row_max, const double *__restrict__ row_sum) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
        const int k = keys[i];
        alpha[i] = exp(x[i] - row_max[k]) / row_sum[k];
    }
}

// ---- backward -----------------------------------------------------------------------------------------------
__global__ void piece_dot_kernel(const double *__restrict__ a, const double *__restrict__ b, const int32_t *__restrict__ perm,
                                 const int32_t *__restrict__ row_start, const int32_t *__restrict__ piece_first,
                                 const int32_t *__restrict__ piece_row, int64_t num_pieces, double *__restrict__ piece_dot) {
    const int lane = threadIdx.x & 31;
    const int64_t warps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t q = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; q < num_pieces; q += warps) {
        int64_t lo, hi;
        piece_range(q, row_start, piece_first, piece_row, &lo, &hi);
        double t = 0.0;
        for (int64_t p = lo + lane; p < hi; p += 32) {
            const int32_t i = perm[p];
            t += a[i] * b[i];
        }
        t = warp_sum(t);
        if (lane == 0) piece_dot[q] = t;
    }
}

// piece_dot_kernel's order with one operand: the sum of x over each piece
__global__ void piece_sum_kernel(const double *__restrict__ x, const int32_t *__restrict__ perm, const int32_t *__restrict__ row_start,
                                 const int32_t *__restrict__ piece_first, const int32_t *__restrict__ piece_row, int64_t num_pieces,
                                 double *__restrict__ piece_val) {
    const int lane = threadIdx.x & 31;
    const int64_t warps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t q = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; q < num_pieces; q += warps) {
        int64_t lo, hi;
        piece_range(q, row_start, piece_first, piece_row, &lo, &hi);
        double t = 0.0;
        for (int64_t p = lo + lane; p < hi; p += 32) t += x[perm[p]];
        t = warp_sum(t);
        if (lane == 0) piece_val[q] = t;
    }
}

__global__ void row_sum_kernel(const int32_t *__restrict__ piece_first, int64_t num_rows, const double *__restrict__ piece_val,
                               double *__restrict__ row_val) {
    const int lane = threadIdx.x & 31;
    const int64_t warps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t u = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; u < num_rows; u += warps) {
        double t = 0.0;
        for (int64_t q = piece_first[u] + lane; q < piece_first[u + 1]; q += 32) t += piece_val[q];
        t = warp_sum(t);
        if (lane == 0) row_val[u] = t;
    }
}

// dx may alias grad
__global__ void backward_apply_kernel(double *dx, const double *__restrict__ alpha, const double *grad, const int32_t *__restrict__ keys,
                                      int64_t n, const double *__restrict__ row_dot) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) dx[i] = alpha[i] * (grad[i] - row_dot[keys[i]]);
}

int check_plan(const char *who, const int32_t *perm, const int32_t *row_start, const int32_t *piece_first, const int32_t *piece_row,
               int64_t num_rows, int64_t num_pieces) {
    if (num_rows < 0 || num_pieces < 0) return set_error(HNH_E_INVALID, "%s: negative size", who);
    if (num_rows > 0 && (!row_start || !piece_first)) return set_error(HNH_E_INVALID, "%s: null plan pointer", who);
    if (num_pieces > 0 && (!perm || !piece_row)) return set_error(HNH_E_INVALID, "%s: null plan pointer", who);
    return HNH_OK;
}

}  // namespace

extern "C" {

int hnh_edge_keys_from_index(int32_t *keys, const int64_t *idx, int64_t n, int64_t offset, void *stream) {
    if (n < 0) return set_error(HNH_E_INVALID, "hnh_edge_keys_from_index: negative size");
    if (n == 0) return HNH_OK;
    if (!keys || !idx) return set_error(HNH_E_INVALID, "hnh_edge_keys_from_index: null pointer");
    int grid = 0;
    int rc = grid_for(keys_from_index_kernel, n, kBlock * 4, &grid, kCtasPerSm);
    return rc ? rc : launch(keys_from_index_kernel, grid, kBlock, (cudaStream_t)stream, "keys_from_index_kernel", keys, idx, n, offset);
}

int64_t hnh_edge_softmax_piece_bound(int64_t n, int64_t num_rows) {
    if (n < 0 || num_rows < 0) return set_error(HNH_E_INVALID, "hnh_edge_softmax_piece_bound: negative size");
    // sum over non-empty rows of ceil(len / kPiece) <= (rows with entries) + ceil(n / kPiece)
    return std::min(n, num_rows) + (n + kPiece - 1) / kPiece;
}

int hnh_edge_softmax_plan(const int32_t *keys, int64_t n, int64_t num_rows, int32_t *perm, int32_t *row_start, int32_t *piece_first,
                          int32_t *piece_row, int64_t piece_capacity, int64_t *num_pieces, void *stream) {
    if (n < 0 || num_rows < 0 || piece_capacity < 0) return set_error(HNH_E_INVALID, "hnh_edge_softmax_plan: negative size");
    if (n > INT32_MAX || num_rows >= INT32_MAX)
        return set_error(HNH_E_INVALID, "hnh_edge_softmax_plan: %lld entries of %lld rows: both must be below 2^31 - 1",
                         (long long)n, (long long)num_rows);
    if (!num_pieces || !row_start || !piece_first) return set_error(HNH_E_INVALID, "hnh_edge_softmax_plan: null pointer");
    if (n > 0 && (!keys || !perm || !piece_row)) return set_error(HNH_E_INVALID, "hnh_edge_softmax_plan: null pointer");
    *num_pieces = 0;
    cudaStream_t st = (cudaStream_t)stream;
    const size_t offsets_bytes = sizeof(int32_t) * (size_t)(num_rows + 1);
    if (n == 0) {
        int rc = check_cuda(cudaMemsetAsync(row_start, 0, offsets_bytes, st), "cudaMemsetAsync");
        if (!rc) rc = check_cuda(cudaMemsetAsync(piece_first, 0, offsets_bytes, st), "cudaMemsetAsync");
        return rc;
    }
    Scratch s;
    int32_t *idx = nullptr, *sorted = nullptr, *count = nullptr;
    int *bad = nullptr;
    void *tmp = nullptr;
    size_t sort_bytes = 0, scan_bytes = 0;
    int rc = check_cuda(s.get((void **)&idx, sizeof(int32_t) * (size_t)n), "cudaMalloc");
    if (!rc) rc = check_cuda(s.get((void **)&sorted, sizeof(int32_t) * (size_t)n), "cudaMalloc");
    if (!rc) rc = check_cuda(s.get((void **)&count, offsets_bytes), "cudaMalloc");
    if (!rc) rc = check_cuda(s.get((void **)&bad, sizeof(int)), "cudaMalloc");
    if (!rc) rc = check_cuda(cudaMemsetAsync(bad, 0, sizeof(int), st), "cudaMemsetAsync");
    int grid = 0;
    if (!rc) rc = grid_for(keys_check_iota_kernel, n, kBlock * 4, &grid, kCtasPerSm);
    if (!rc) rc = launch(keys_check_iota_kernel, grid, kBlock, st, "keys_check_iota_kernel", keys, n, num_rows, idx, bad);
    if (rc) return rc;
    int host_bad = 0;
    rc = check_cuda(cudaMemcpyAsync(&host_bad, bad, sizeof(int), cudaMemcpyDeviceToHost, st), "cudaMemcpyAsync");
    if (!rc) rc = check_cuda(cudaStreamSynchronize(st), "cudaStreamSynchronize");
    if (rc) return rc;
    if (host_bad) return set_error(HNH_E_INVALID, "hnh_edge_softmax_plan: a key lies outside [0, %lld)", (long long)num_rows);

    const int end_bit = bits_for((uint64_t)std::max<int64_t>(num_rows - 1, 1));
    rc = check_cuda(cub::DeviceRadixSort::SortPairs(nullptr, sort_bytes, keys, sorted, idx, perm, (int)n, 0, end_bit, st), "cub sort size");
    if (!rc) rc = check_cuda(cub::DeviceScan::ExclusiveSum(nullptr, scan_bytes, count, piece_first, (int)(num_rows + 1), st), "cub scan size");
    if (!rc) rc = check_cuda(s.get(&tmp, std::max(sort_bytes, scan_bytes)), "cudaMalloc");
    if (!rc) rc = check_cuda(cub::DeviceRadixSort::SortPairs(tmp, sort_bytes, keys, sorted, idx, perm, (int)n, 0, end_bit, st), "cub sort");
    if (!rc) rc = grid_for(row_start_kernel, num_rows + 1, kBlock, &grid, kCtasPerSm);
    if (!rc) rc = launch(row_start_kernel, grid, kBlock, st, "row_start_kernel", sorted, n, num_rows, row_start);
    if (!rc) rc = launch(piece_count_kernel, grid, kBlock, st, "piece_count_kernel", row_start, num_rows, count);
    if (!rc) rc = check_cuda(cub::DeviceScan::ExclusiveSum(tmp, scan_bytes, count, piece_first, (int)(num_rows + 1), st), "cub scan");
    int32_t total = 0;
    if (!rc) rc = check_cuda(cudaMemcpyAsync(&total, piece_first + num_rows, sizeof(int32_t), cudaMemcpyDeviceToHost, st), "cudaMemcpyAsync");
    if (!rc) rc = check_cuda(cudaStreamSynchronize(st), "cudaStreamSynchronize");
    if (rc) return rc;
    if (total > piece_capacity)
        return set_error(HNH_E_INVALID, "hnh_edge_softmax_plan: %lld pieces, room for %lld", (long long)total, (long long)piece_capacity);
    rc = grid_for(piece_row_kernel, num_rows, kBlock, &grid, kCtasPerSm);
    if (!rc) rc = launch(piece_row_kernel, grid, kBlock, st, "piece_row_kernel", piece_first, num_rows, piece_row);
    if (!rc) rc = check_cuda(cudaStreamSynchronize(st), "cudaStreamSynchronize");  // the scratch is freed on return
    if (!rc) *num_pieces = total;
    return rc;
}

int hnh_edge_softmax_stats_f64(const double *x, const int32_t *perm, const int32_t *row_start, const int32_t *piece_first,
                               const int32_t *piece_row, int64_t num_rows, int64_t num_pieces, double *piece_max, double *piece_sum,
                               double *row_max, double *row_sum, void *stream) {
    int rc = check_plan("hnh_edge_softmax_stats_f64", perm, row_start, piece_first, piece_row, num_rows, num_pieces);
    if (rc) return rc;
    if (num_rows == 0) return HNH_OK;
    if (!row_max || !row_sum || (num_pieces > 0 && (!x || !piece_max || !piece_sum)))
        return set_error(HNH_E_INVALID, "hnh_edge_softmax_stats_f64: null pointer");
    cudaStream_t st = (cudaStream_t)stream;
    int grid = 0;
    if (num_pieces > 0) {
        rc = grid_for(piece_stats_kernel, num_pieces, kBlock / 32, &grid, kCtasPerSm);
        if (!rc)
            rc = launch(piece_stats_kernel, grid, kBlock, st, "piece_stats_kernel", x, perm, row_start, piece_first, piece_row, num_pieces,
                        piece_max, piece_sum);
        if (rc) return rc;
    }
    rc = grid_for(row_stats_kernel, num_rows, kBlock / 32, &grid, kCtasPerSm);
    return rc ? rc : launch(row_stats_kernel, grid, kBlock, st, "row_stats_kernel", piece_first, num_rows, piece_max, piece_sum, row_max,
                            row_sum);
}

int hnh_edge_softmax_rescale_f64(double *row_sum, const double *local_max, const double *global_max, int64_t num_rows, void *stream) {
    if (num_rows < 0) return set_error(HNH_E_INVALID, "hnh_edge_softmax_rescale_f64: negative size");
    if (num_rows == 0) return HNH_OK;
    if (!row_sum || !local_max || !global_max) return set_error(HNH_E_INVALID, "hnh_edge_softmax_rescale_f64: null pointer");
    int grid = 0;
    int rc = grid_for(rescale_kernel, num_rows, kBlock * 4, &grid, kCtasPerSm);
    return rc ? rc : launch(rescale_kernel, grid, kBlock, (cudaStream_t)stream, "rescale_kernel", row_sum, local_max, global_max, num_rows);
}

int hnh_edge_softmax_apply_f64(double *alpha, const double *x, const int32_t *keys, int64_t n, const double *row_max,
                               const double *row_sum, void *stream) {
    if (n < 0) return set_error(HNH_E_INVALID, "hnh_edge_softmax_apply_f64: negative size");
    if (n == 0) return HNH_OK;
    if (!alpha || !x || !keys || !row_max || !row_sum) return set_error(HNH_E_INVALID, "hnh_edge_softmax_apply_f64: null pointer");
    int grid = 0;
    int rc = grid_for(apply_kernel, n, kBlock * 4, &grid, kCtasPerSm);
    return rc ? rc : launch(apply_kernel, grid, kBlock, (cudaStream_t)stream, "apply_kernel", alpha, x, keys, n, row_max, row_sum);
}

int hnh_edge_softmax_dot_f64(const double *alpha, const double *grad, const int32_t *perm, const int32_t *row_start,
                             const int32_t *piece_first, const int32_t *piece_row, int64_t num_rows, int64_t num_pieces,
                             double *piece_dot, double *row_dot, void *stream) {
    int rc = check_plan("hnh_edge_softmax_dot_f64", perm, row_start, piece_first, piece_row, num_rows, num_pieces);
    if (rc) return rc;
    if (num_rows == 0) return HNH_OK;
    if (!row_dot || (num_pieces > 0 && (!alpha || !grad || !piece_dot)))
        return set_error(HNH_E_INVALID, "hnh_edge_softmax_dot_f64: null pointer");
    cudaStream_t st = (cudaStream_t)stream;
    int grid = 0;
    if (num_pieces > 0) {
        rc = grid_for(piece_dot_kernel, num_pieces, kBlock / 32, &grid, kCtasPerSm);
        if (!rc)
            rc = launch(piece_dot_kernel, grid, kBlock, st, "piece_dot_kernel", alpha, grad, perm, row_start, piece_first, piece_row,
                        num_pieces, piece_dot);
        if (rc) return rc;
    }
    rc = grid_for(row_sum_kernel, num_rows, kBlock / 32, &grid, kCtasPerSm);
    return rc ? rc : launch(row_sum_kernel, grid, kBlock, st, "row_sum_kernel", piece_first, num_rows, piece_dot, row_dot);
}

int hnh_edge_sum_f64(const double *x, const int32_t *perm, const int32_t *row_start, const int32_t *piece_first,
                     const int32_t *piece_row, int64_t num_rows, int64_t num_pieces, double *piece_sum, double *row_sum,
                     void *stream) {
    int rc = check_plan("hnh_edge_sum_f64", perm, row_start, piece_first, piece_row, num_rows, num_pieces);
    if (rc) return rc;
    if (num_rows == 0) return HNH_OK;
    if (!row_sum || (num_pieces > 0 && (!x || !piece_sum))) return set_error(HNH_E_INVALID, "hnh_edge_sum_f64: null pointer");
    cudaStream_t st = (cudaStream_t)stream;
    int grid = 0;
    if (num_pieces > 0) {
        rc = grid_for(piece_sum_kernel, num_pieces, kBlock / 32, &grid, kCtasPerSm);
        if (!rc)
            rc = launch(piece_sum_kernel, grid, kBlock, st, "piece_sum_kernel", x, perm, row_start, piece_first, piece_row, num_pieces,
                        piece_sum);
        if (rc) return rc;
    }
    rc = grid_for(row_sum_kernel, num_rows, kBlock / 32, &grid, kCtasPerSm);
    return rc ? rc : launch(row_sum_kernel, grid, kBlock, st, "row_sum_kernel", piece_first, num_rows, piece_sum, row_sum);
}

int hnh_edge_softmax_backward_f64(double *dx, const double *alpha, const double *grad, const int32_t *keys, int64_t n,
                                  const double *row_dot, void *stream) {
    if (n < 0) return set_error(HNH_E_INVALID, "hnh_edge_softmax_backward_f64: negative size");
    if (n == 0) return HNH_OK;
    if (!dx || !alpha || !grad || !keys || !row_dot) return set_error(HNH_E_INVALID, "hnh_edge_softmax_backward_f64: null pointer");
    int grid = 0;
    int rc = grid_for(backward_apply_kernel, n, kBlock * 4, &grid, kCtasPerSm);
    return rc ? rc : launch(backward_apply_kernel, grid, kBlock, (cudaStream_t)stream, "backward_apply_kernel", dx, alpha, grad, keys, n,
                            row_dot);
}

}  // extern "C"
