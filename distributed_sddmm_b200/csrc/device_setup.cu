// device_setup.cu -- device-side versions of the two host setup helpers (host_setup.cpp), exported through
// the C ABI: the seeded Erdos-Renyi tuple generator and the COO -> CSR conversion of one block.  They produce
// bit-identical output to the host versions (the generator is a pure function of (seed, row, k); the CSR
// order is "stored row ascending, input order within a row", i.e. a STABLE sort by stored row, which is what
// cub::DeviceRadixSort gives).  SURVEY.md section 8(f) rank 3: the host classes still build their blocks
// with the host path; these entry points are the building blocks of a device-resident setup.
#include <cub/cub.cuh>

#include "launch.h"
#include "mix64.cuh"

namespace {

using hnh::bits_for;
using hnh::check_cuda;
using hnh::grid_for;
using hnh::kBlock;
using hnh::launch;
using hnh::Scratch;
using hnh::set_error;

constexpr int kCtasPerSm = 8;  // grid cap of every grid-stride kernel here
constexpr int kMaxPerRow = 128;  // columns drawn per row that one thread sorts in local memory

// the sorted, de-duplicated column draws of one row; returns how many are left
__device__ inline int draw_row(uint64_t seed, uint64_t row, int per_row, uint64_t mask, uint64_t *tmp) {
    const uint64_t base = mix64(seed ^ (row * 0xD1342543DE82EF95ull));
    for (int k = 0; k < per_row; k++) {  // insertion sort while drawing
        const uint64_t x = mix64(base + (uint64_t)k) & mask;
        int j = k;
        while (j > 0 && tmp[j - 1] > x) { tmp[j] = tmp[j - 1]; j--; }
        tmp[j] = x;
    }
    int n = 0;
    for (int k = 0; k < per_row; k++)
        if (k == 0 || tmp[k] != tmp[k - 1]) tmp[n++] = tmp[k];
    return n;
}

__global__ void er_count_kernel(uint64_t seed, int64_t row_lo, int64_t nrows, int per_row, uint64_t mask, int64_t *counts) {
    uint64_t tmp[kMaxPerRow];
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < nrows; i += stride)
        counts[i] = draw_row(seed, (uint64_t)(row_lo + i), per_row, mask, tmp);
}

__global__ void er_write_kernel(uint64_t seed, int64_t row_lo, int64_t nrows, int per_row, uint64_t mask,
                                const int64_t *__restrict__ offsets, uint64_t *__restrict__ rows_out,
                                uint64_t *__restrict__ cols_out, double *__restrict__ vals_out) {
    uint64_t tmp[kMaxPerRow];
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < nrows; i += stride) {
        const int n = draw_row(seed, (uint64_t)(row_lo + i), per_row, mask, tmp);
        int64_t o = offsets[i];
        for (int k = 0; k < n; k++, o++) {
            rows_out[o] = (uint64_t)(row_lo + i);
            cols_out[o] = tmp[k];
            vals_out[o] = 1.0;
        }
    }
}

// key[i] = stored row of entry i, idx[i] = i; *bad is set when a coordinate lies outside the block
__global__ void csr_keys_kernel(const uint64_t *__restrict__ sr, const uint64_t *__restrict__ sc, int64_t nnz,
                                uint64_t out_rows, uint64_t out_cols, uint64_t *__restrict__ key, int64_t *__restrict__ idx,
                                int *bad) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < nnz; i += stride) {
        if (sr[i] >= out_rows || sc[i] >= out_cols) *bad = 1;
        key[i] = sr[i];
        idx[i] = i;
    }
}

__global__ void csr_gather_kernel(const uint64_t *__restrict__ sorted_key, const int64_t *__restrict__ sorted_idx,
                                  const uint64_t *__restrict__ sc, const double *__restrict__ v, int64_t nnz,
                                  int64_t *__restrict__ col_idx, int64_t *__restrict__ row_idx, double *__restrict__ values) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; p < nnz; p += stride) {
        const int64_t i = sorted_idx[p];
        col_idx[p] = (int64_t)sc[i];
        values[p] = v[i];
        if (row_idx) row_idx[p] = (int64_t)sorted_key[p];
    }
}

// rowStart[r] = first position p with sorted_key[p] >= r, for r = 0 .. out_rows (binary search per row)
__global__ void csr_row_start_kernel(const uint64_t *__restrict__ sorted_key, int64_t nnz, int64_t out_rows,
                                     int64_t *__restrict__ rowStart) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r <= out_rows; r += stride) {
        int64_t lo = 0, hi = nnz;
        while (lo < hi) {
            const int64_t mid = (lo + hi) >> 1;
            if (sorted_key[mid] < (uint64_t)r) lo = mid + 1; else hi = mid;
        }
        rowStart[r] = lo;
    }
}

// ---- device-resident tuple pipeline (SpmatLocal::redistribute_nonzeros and friends) -------------------------
// owner of tuple i from a (row block, column block) table that the host filled by calling the distribution's
// blockOwner() for every block pair (NonzeroDistribution::getOwner, reference SpmatLocal.hpp:45-52)
__global__ void tuple_owner_kernel(const uint64_t *__restrict__ r, const uint64_t *__restrict__ c, int64_t n, int transpose,
                                   uint64_t rows_in_block, uint64_t cols_in_block, const int *__restrict__ table,
                                   int64_t table_rows, int64_t table_cols, unsigned *__restrict__ owner,
                                   int64_t *__restrict__ idx, int *bad) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
        const uint64_t rb = (transpose ? c[i] : r[i]) / rows_in_block, cb = (transpose ? r[i] : c[i]) / cols_in_block;
        int o = 0;
        if (rb >= (uint64_t)table_rows || cb >= (uint64_t)table_cols) *bad = 1;
        else o = table[rb * (uint64_t)table_cols + cb];
        if (o < 0) { *bad = 1; o = 0; }
        owner[i] = (unsigned)o;
        idx[i] = i;
    }
}

__global__ void iota_kernel(int64_t *__restrict__ idx, int64_t n) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) idx[i] = i;
}

// out[p] = in[perm[p]] for the three tuple arrays; swap_rc exchanges the roles of r and c on the way
__global__ void tuple_gather_kernel(const uint64_t *__restrict__ r, const uint64_t *__restrict__ c, const double *__restrict__ v,
                                    const int64_t *__restrict__ perm, int64_t n, int swap_rc, uint64_t *__restrict__ r_out,
                                    uint64_t *__restrict__ c_out, double *__restrict__ v_out) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; p < n; p += stride) {
        const int64_t i = perm[p];
        r_out[p] = swap_rc ? c[i] : r[i];
        c_out[p] = swap_rc ? r[i] : c[i];
        v_out[p] = v[i];
    }
}

__global__ void key_gather_kernel(const uint64_t *__restrict__ key, const int64_t *__restrict__ perm, int64_t n,
                                  uint64_t *__restrict__ out) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; p < n; p += stride) out[p] = key[perm[p]];
}

__global__ void tuple_mod_kernel(uint64_t *__restrict__ r, uint64_t *__restrict__ c, int64_t n, uint64_t mod_r, uint64_t mod_c) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
        if (mod_r) r[i] %= mod_r;
        if (mod_c) c[i] %= mod_c;
    }
}

// starts[k] = first position with key[p] >= k * width (keys ascending), k = 0 .. divisions
template <typename K>
__global__ void lower_bounds_kernel(const K *__restrict__ key, int64_t n, uint64_t width, int divisions, int64_t *__restrict__ starts) {
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k > divisions) return;
    const uint64_t want = (uint64_t)k * width;
    int64_t lo = 0, hi = n;
    while (lo < hi) {
        const int64_t mid = (lo + hi) >> 1;
        if ((uint64_t)key[mid] < want) lo = mid + 1; else hi = mid;
    }
    starts[k] = lo;
}

}  // namespace

extern "C" {

int64_t hnh_er_generate_device(int logM, int nnz_per_row, uint64_t seed, int64_t row_lo, int64_t row_hi, uint64_t *rows_out,
                               uint64_t *cols_out, double *vals_out, int64_t capacity, void *stream) {
    if (logM < 0 || logM > 40 || nnz_per_row < 0 || nnz_per_row > kMaxPerRow || row_lo < 0 || row_hi < row_lo ||
        row_hi > ((int64_t)1 << logM))
        return set_error(HNH_E_INVALID, "hnh_er_generate_device: bad argument (nnz_per_row <= %d)", kMaxPerRow);
    const int64_t nrows = row_hi - row_lo;
    if (nrows == 0 || nnz_per_row == 0) return 0;
    if (nrows >= INT32_MAX) return set_error(HNH_E_INVALID, "hnh_er_generate_device: at most 2^31 - 2 rows per call");
    if (!rows_out || !cols_out || !vals_out) return set_error(HNH_E_INVALID, "hnh_er_generate_device: null output");
    cudaStream_t st = (cudaStream_t)stream;
    const uint64_t mask = ((uint64_t)1 << logM) - 1;
    Scratch s;
    int64_t *counts = nullptr, *offsets = nullptr;
    void *tmp = nullptr;
    size_t tmp_bytes = 0;
    int rc = check_cuda(s.get((void **)&counts, sizeof(int64_t) * (size_t)(nrows + 1)), "cudaMalloc");
    if (!rc) rc = check_cuda(s.get((void **)&offsets, sizeof(int64_t) * (size_t)(nrows + 1)), "cudaMalloc");
    int grid = 0;
    if (!rc) rc = grid_for(er_count_kernel, nrows, kBlock, &grid, kCtasPerSm);
    if (!rc) rc = launch(er_count_kernel, grid, kBlock, st, "er_count_kernel", seed, row_lo, nrows, nnz_per_row, mask, counts);
    if (!rc) rc = check_cuda(cudaMemsetAsync(counts + nrows, 0, sizeof(int64_t), st), "cudaMemsetAsync");
    if (rc) return rc;
    rc = check_cuda(cub::DeviceScan::ExclusiveSum(nullptr, tmp_bytes, counts, offsets, (int)(nrows + 1), st), "cub scan size");
    if (!rc) rc = check_cuda(s.get(&tmp, tmp_bytes), "cudaMalloc");
    if (!rc) rc = check_cuda(cub::DeviceScan::ExclusiveSum(tmp, tmp_bytes, counts, offsets, (int)(nrows + 1), st), "cub scan");
    if (rc) return rc;
    int64_t total = 0;
    rc = check_cuda(cudaMemcpyAsync(&total, offsets + nrows, sizeof(int64_t), cudaMemcpyDeviceToHost, st), "cudaMemcpyAsync");
    if (!rc) rc = check_cuda(cudaStreamSynchronize(st), "cudaStreamSynchronize");
    if (rc) return rc;
    if (total > capacity)
        return set_error(HNH_E_INVALID, "hnh_er_generate_device: capacity %lld < %lld", (long long)capacity, (long long)total);
    rc = launch(er_write_kernel, grid, kBlock, st, "er_write_kernel", seed, row_lo, nrows, nnz_per_row, mask, offsets, rows_out, cols_out,
                vals_out);
    if (!rc) rc = check_cuda(cudaStreamSynchronize(st), "cudaStreamSynchronize");  // the scratch is freed on return
    return rc ? rc : total;
}

int hnh_coo_to_csr_device(int64_t rows, int64_t cols, int64_t nnz, const uint64_t *r, const uint64_t *c, const double *v,
                          int transpose, int64_t *rowStart, int64_t *col_idx, int64_t *row_idx, double *values, void *stream) {
    if (rows < 0 || cols < 0 || nnz < 0 || !rowStart) return set_error(HNH_E_INVALID, "hnh_coo_to_csr_device: bad argument");
    if (nnz > 0 && (!r || !c || !v || !col_idx || !values)) return set_error(HNH_E_INVALID, "hnh_coo_to_csr_device: null pointer");
    if (nnz > INT32_MAX) return set_error(HNH_E_INVALID, "hnh_coo_to_csr_device: more than 2^31 - 1 entries in one block");
    cudaStream_t st = (cudaStream_t)stream;
    const int64_t out_rows = transpose ? cols : rows, out_cols = transpose ? rows : cols;
    const uint64_t *sr = transpose ? c : r, *sc = transpose ? r : c;
    if (nnz == 0) return check_cuda(cudaMemsetAsync(rowStart, 0, sizeof(int64_t) * (size_t)(out_rows + 1), st), "cudaMemsetAsync");
    Scratch s;
    uint64_t *key = nullptr, *key_sorted = nullptr;
    int64_t *idx = nullptr, *idx_sorted = nullptr;
    int *bad = nullptr;
    void *tmp = nullptr;
    size_t tmp_bytes = 0;
    int rc = check_cuda(s.get((void **)&key, sizeof(uint64_t) * (size_t)nnz), "cudaMalloc");
    if (!rc) rc = check_cuda(s.get((void **)&key_sorted, sizeof(uint64_t) * (size_t)nnz), "cudaMalloc");
    if (!rc) rc = check_cuda(s.get((void **)&idx, sizeof(int64_t) * (size_t)nnz), "cudaMalloc");
    if (!rc) rc = check_cuda(s.get((void **)&idx_sorted, sizeof(int64_t) * (size_t)nnz), "cudaMalloc");
    if (!rc) rc = check_cuda(s.get((void **)&bad, sizeof(int)), "cudaMalloc");
    if (!rc) rc = check_cuda(cudaMemsetAsync(bad, 0, sizeof(int), st), "cudaMemsetAsync");
    int grid = 0;
    if (!rc) rc = grid_for(csr_keys_kernel, nnz, kBlock, &grid, kCtasPerSm);
    if (!rc) rc = launch(csr_keys_kernel, grid, kBlock, st, "csr_keys_kernel", sr, sc, nnz, (uint64_t)out_rows, (uint64_t)out_cols, key, idx, bad);
    if (rc) return rc;
    int host_bad = 0;
    rc = check_cuda(cudaMemcpyAsync(&host_bad, bad, sizeof(int), cudaMemcpyDeviceToHost, st), "cudaMemcpyAsync");
    if (!rc) rc = check_cuda(cudaStreamSynchronize(st), "cudaStreamSynchronize");
    if (rc) return rc;
    if (host_bad)
        return set_error(HNH_E_INVALID, "hnh_coo_to_csr_device: a coordinate lies outside the %lld x %lld block",
                         (long long)rows, (long long)cols);
    const int end_bit = bits_for((uint64_t)std::max<int64_t>(out_rows - 1, 1));
    rc = check_cuda(cub::DeviceRadixSort::SortPairs(nullptr, tmp_bytes, key, key_sorted, idx, idx_sorted, (int)nnz, 0, end_bit, st),
                    "cub sort size");
    if (!rc) rc = check_cuda(s.get(&tmp, tmp_bytes), "cudaMalloc");
    if (!rc) rc = check_cuda(cub::DeviceRadixSort::SortPairs(tmp, tmp_bytes, key, key_sorted, idx, idx_sorted, (int)nnz, 0, end_bit, st),
                             "cub sort");
    if (!rc) rc = launch(csr_gather_kernel, grid, kBlock, st, "csr_gather_kernel", key_sorted, idx_sorted, sc, v, nnz, col_idx, row_idx, values);
    if (!rc) rc = grid_for(csr_row_start_kernel, out_rows + 1, kBlock, &grid, kCtasPerSm);
    if (!rc) rc = launch(csr_row_start_kernel, grid, kBlock, st, "csr_row_start_kernel", key_sorted, nnz, out_rows, rowStart);
    if (!rc) rc = check_cuda(cudaStreamSynchronize(st), "cudaStreamSynchronize");  // the scratch is freed on return
    return rc;
}

// ---- device-resident tuple pipeline ------------------------------------------------------------------------------
int hnh_tuples_bucket_by_owner_device(const uint64_t *r, const uint64_t *c, const double *v, int64_t n, int transpose,
                                      int64_t rows_in_block, int64_t cols_in_block, const int *owner_table_host,
                                      int64_t table_rows, int64_t table_cols, int nbuckets, uint64_t *r_out, uint64_t *c_out,
                                      double *v_out, int64_t *starts_host, void *stream) {
    if (n < 0 || nbuckets < 1 || rows_in_block < 1 || cols_in_block < 1 || table_rows < 1 || table_cols < 1 || !owner_table_host ||
        !starts_host)
        return set_error(HNH_E_INVALID, "hnh_tuples_bucket_by_owner_device: bad argument");
    if (n > INT32_MAX) return set_error(HNH_E_INVALID, "hnh_tuples_bucket_by_owner_device: more than 2^31 - 1 tuples");
    for (int b = 0; b <= nbuckets; b++) starts_host[b] = 0;
    if (n == 0) return HNH_OK;
    if (!r || !c || !v || !r_out || !c_out || !v_out) return set_error(HNH_E_INVALID, "hnh_tuples_bucket_by_owner_device: null pointer");
    cudaStream_t st = (cudaStream_t)stream;
    Scratch s;
    int *table = nullptr, *bad = nullptr;
    unsigned *owner = nullptr, *owner_sorted = nullptr;
    int64_t *idx = nullptr, *idx_sorted = nullptr, *starts = nullptr;
    void *tmp = nullptr;
    size_t tmp_bytes = 0;
    const size_t tb = sizeof(int) * (size_t)(table_rows * table_cols);
    int rc = check_cuda(s.get((void **)&table, tb), "cudaMalloc");
    if (!rc) rc = check_cuda(s.get((void **)&bad, sizeof(int)), "cudaMalloc");
    if (!rc) rc = check_cuda(s.get((void **)&owner, sizeof(unsigned) * (size_t)n), "cudaMalloc");
    if (!rc) rc = check_cuda(s.get((void **)&owner_sorted, sizeof(unsigned) * (size_t)n), "cudaMalloc");
    if (!rc) rc = check_cuda(s.get((void **)&idx, sizeof(int64_t) * (size_t)n), "cudaMalloc");
    if (!rc) rc = check_cuda(s.get((void **)&idx_sorted, sizeof(int64_t) * (size_t)n), "cudaMalloc");
    if (!rc) rc = check_cuda(s.get((void **)&starts, sizeof(int64_t) * (size_t)(nbuckets + 1)), "cudaMalloc");
    if (!rc) rc = check_cuda(cudaMemcpyAsync(table, owner_table_host, tb, cudaMemcpyHostToDevice, st), "cudaMemcpyAsync");
    if (!rc) rc = check_cuda(cudaMemsetAsync(bad, 0, sizeof(int), st), "cudaMemsetAsync");
    int grid = 0;
    if (!rc) rc = grid_for(tuple_owner_kernel, n, kBlock, &grid, kCtasPerSm);
    if (!rc)
        rc = launch(tuple_owner_kernel, grid, kBlock, st, "tuple_owner_kernel", r, c, n, transpose, (uint64_t)rows_in_block,
                    (uint64_t)cols_in_block, table, table_rows, table_cols, owner, idx, bad);
    if (rc) return rc;
    const int end_bit = bits_for((uint64_t)std::max(nbuckets - 1, 1));
    rc = check_cuda(cub::DeviceRadixSort::SortPairs(nullptr, tmp_bytes, owner, owner_sorted, idx, idx_sorted, (int)n, 0, end_bit, st),
                    "cub sort size");
    if (!rc) rc = check_cuda(s.get(&tmp, tmp_bytes), "cudaMalloc");
    if (!rc) rc = check_cuda(cub::DeviceRadixSort::SortPairs(tmp, tmp_bytes, owner, owner_sorted, idx, idx_sorted, (int)n, 0, end_bit, st),
                             "cub sort");
    if (!rc) rc = launch(tuple_gather_kernel, grid, kBlock, st, "tuple_gather_kernel", r, c, v, idx_sorted, n, transpose, r_out, c_out, v_out);
    if (!rc)
        rc = launch(lower_bounds_kernel<unsigned>, (nbuckets + 1 + kBlock - 1) / kBlock, kBlock, st, "lower_bounds_kernel", owner_sorted, n,
                    1, nbuckets, starts);
    int host_bad = 0;
    if (!rc) rc = check_cuda(cudaMemcpyAsync(&host_bad, bad, sizeof(int), cudaMemcpyDeviceToHost, st), "cudaMemcpyAsync");
    if (!rc) rc = check_cuda(cudaMemcpyAsync(starts_host, starts, sizeof(int64_t) * (size_t)(nbuckets + 1), cudaMemcpyDeviceToHost, st),
                             "cudaMemcpyAsync");
    if (!rc) rc = check_cuda(cudaStreamSynchronize(st), "cudaStreamSynchronize");
    if (rc) return rc;
    if (host_bad) return set_error(HNH_E_INVALID, "hnh_tuples_bucket_by_owner_device: a coordinate has no owner (outside the block table)");
    return HNH_OK;
}

int hnh_tuples_sort_colmajor_device(uint64_t *r, uint64_t *c, double *v, int64_t n, uint64_t max_r, uint64_t max_c, void *stream) {
    if (n < 0) return set_error(HNH_E_INVALID, "hnh_tuples_sort_colmajor_device: bad argument");
    if (n > INT32_MAX) return set_error(HNH_E_INVALID, "hnh_tuples_sort_colmajor_device: more than 2^31 - 1 tuples");
    if (n <= 1) return HNH_OK;
    if (!r || !c || !v) return set_error(HNH_E_INVALID, "hnh_tuples_sort_colmajor_device: null pointer");
    cudaStream_t st = (cudaStream_t)stream;
    Scratch s;
    uint64_t *key_a = nullptr, *key_b = nullptr, *r2 = nullptr, *c2 = nullptr;
    double *v2 = nullptr;
    int64_t *idx_a = nullptr, *idx_b = nullptr;
    void *tmp = nullptr;
    size_t tmp_bytes = 0, tb2 = 0;
    const size_t b8 = sizeof(uint64_t) * (size_t)n;
    int rc = check_cuda(s.get((void **)&key_a, b8), "cudaMalloc");
    if (!rc) rc = check_cuda(s.get((void **)&key_b, b8), "cudaMalloc");
    if (!rc) rc = check_cuda(s.get((void **)&idx_a, b8), "cudaMalloc");
    if (!rc) rc = check_cuda(s.get((void **)&idx_b, b8), "cudaMalloc");
    if (!rc) rc = check_cuda(s.get((void **)&r2, b8), "cudaMalloc");
    if (!rc) rc = check_cuda(s.get((void **)&c2, b8), "cudaMalloc");
    if (!rc) rc = check_cuda(s.get((void **)&v2, b8), "cudaMalloc");
    if (rc) return rc;
    const int bits_r = bits_for(std::max<uint64_t>(max_r, 1)), bits_c = bits_for(std::max<uint64_t>(max_c, 1));
    rc = check_cuda(cub::DeviceRadixSort::SortPairs(nullptr, tmp_bytes, key_a, key_b, idx_a, idx_b, (int)n, 0, bits_r, st), "cub sort size");
    if (!rc) rc = check_cuda(cub::DeviceRadixSort::SortPairs(nullptr, tb2, key_a, key_b, idx_a, idx_b, (int)n, 0, bits_c, st), "cub sort size");
    tmp_bytes = std::max(tmp_bytes, tb2);
    if (!rc) rc = check_cuda(s.get(&tmp, tmp_bytes), "cudaMalloc");
    if (rc) return rc;
    // LSD over the pair: stable by row first, then stable by column  =>  ordered by (column, row), ties in input order
    int grid = 0;
    rc = grid_for(iota_kernel, n, kBlock, &grid, kCtasPerSm);
    if (!rc) rc = launch(iota_kernel, grid, kBlock, st, "iota_kernel", idx_a, n);
    if (!rc) rc = check_cuda(cub::DeviceRadixSort::SortPairs(tmp, tmp_bytes, r, key_b, idx_a, idx_b, (int)n, 0, bits_r, st), "cub sort (rows)");
    if (!rc) rc = launch(key_gather_kernel, grid, kBlock, st, "key_gather_kernel", c, idx_b, n, key_a);
    if (!rc) rc = check_cuda(cub::DeviceRadixSort::SortPairs(tmp, tmp_bytes, key_a, key_b, idx_b, idx_a, (int)n, 0, bits_c, st), "cub sort (cols)");
    if (!rc) rc = launch(tuple_gather_kernel, grid, kBlock, st, "tuple_gather_kernel", r, c, v, idx_a, n, 0, r2, c2, v2);
    if (!rc) rc = check_cuda(cudaMemcpyAsync(r, r2, b8, cudaMemcpyDeviceToDevice, st), "cudaMemcpyAsync");
    if (!rc) rc = check_cuda(cudaMemcpyAsync(c, c2, b8, cudaMemcpyDeviceToDevice, st), "cudaMemcpyAsync");
    if (!rc) rc = check_cuda(cudaMemcpyAsync(v, v2, b8, cudaMemcpyDeviceToDevice, st), "cudaMemcpyAsync");
    if (!rc) rc = check_cuda(cudaStreamSynchronize(st), "cudaStreamSynchronize");
    return rc;
}

int hnh_tuples_mod_device(uint64_t *r, uint64_t *c, int64_t n, uint64_t mod_r, uint64_t mod_c, void *stream) {
    if (n < 0) return set_error(HNH_E_INVALID, "hnh_tuples_mod_device: bad argument");
    if (n == 0 || (mod_r == 0 && mod_c == 0)) return HNH_OK;
    if (!r || !c) return set_error(HNH_E_INVALID, "hnh_tuples_mod_device: null pointer");
    int grid = 0;
    int rc = grid_for(tuple_mod_kernel, n, kBlock, &grid, kCtasPerSm);
    return rc ? rc : launch(tuple_mod_kernel, grid, kBlock, (cudaStream_t)stream, "tuple_mod_kernel", r, c, n, mod_r, mod_c);
}

int hnh_tuples_block_starts_device(const uint64_t *c_sorted, int64_t n, uint64_t block_width, int divisions, int64_t *starts_host,
                                   void *stream) {
    if (n < 0 || divisions < 0 || block_width == 0 || !starts_host) return set_error(HNH_E_INVALID, "hnh_tuples_block_starts_device: bad argument");
    if (n == 0) {
        for (int k = 0; k <= divisions; k++) starts_host[k] = 0;
        return HNH_OK;
    }
    if (!c_sorted) return set_error(HNH_E_INVALID, "hnh_tuples_block_starts_device: null pointer");
    cudaStream_t st = (cudaStream_t)stream;
    Scratch s;
    int64_t *starts = nullptr;
    int rc = check_cuda(s.get((void **)&starts, sizeof(int64_t) * (size_t)(divisions + 1)), "cudaMalloc");
    if (!rc)
        rc = launch(lower_bounds_kernel<uint64_t>, (divisions + 1 + kBlock - 1) / kBlock, kBlock, st, "lower_bounds_kernel", c_sorted, n,
                    block_width, divisions, starts);
    if (!rc) rc = check_cuda(cudaMemcpyAsync(starts_host, starts, sizeof(int64_t) * (size_t)(divisions + 1), cudaMemcpyDeviceToHost, st), "cudaMemcpyAsync");
    if (!rc) rc = check_cuda(cudaStreamSynchronize(st), "cudaStreamSynchronize");
    return rc;
}

}  // extern "C"
