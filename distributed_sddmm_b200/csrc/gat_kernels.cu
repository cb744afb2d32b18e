// gat_kernels.cu -- the three device operations the GAT forward pass (include/hnh/gat.hpp; reference
// gat.hpp:84-113) needs beyond the SDDMM / SpMM path: LeakyReLU on an edge-value vector, ReLU of a head's
// output written into its column window of the layer output, and the dense projection X * W.
//
// The projection is this library's own fp64 GEMM (dgemm_dmma_kernel below): C = A B for a tall A (rows of the
// graph) and a small B (the head's weight matrix), on the fp64 tensor-core path (mma.sync m8n8k4, DMMA) with
// shared-memory tiles.  Hopper's wgmma has no fp64 kind, so mma.sync IS the fp64 tensor path on sm_90a.
//
// The backward pass (GAT::backwardPass) adds the two other products of a projection on the same DMMA tiling --
// dW = X^T dP (dgemm_tn_kernel, split over the long k and reduced in a fixed order) and dX += dP W^T
// (dgemm_nt_kernel) -- and the derivatives of the two activations.
#include "launch.h"

namespace {

using hnh::check_cuda;
using hnh::grid_for;
using hnh::kBlock;
using hnh::launch;
using hnh::set_error;

constexpr int kCtasPerSm = 8;  // grid cap of every grid-stride kernel here

// x -> max(x, 0) + alpha * min(x, 0)
__global__ void leaky_relu_kernel(double *__restrict__ dst, const double *__restrict__ src, int64_t n, double alpha) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
        const double x = src[i];
        dst[i] = fmax(x, 0.0) + fmin(x, 0.0) * alpha;
    }
}

// dst[i, col0 + j] = max(src[i, j], 0): dst has ld_dst columns, src is rows x cols, contiguous
__global__ void relu_cols_kernel(double *__restrict__ dst, int64_t ld_dst, int64_t col0, const double *__restrict__ src,
                                 int64_t rows, int64_t cols) {
    const int64_t n = rows * cols;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < n; t += stride) {
        const int64_t i = t / cols, j = t - i * cols;
        dst[i * ld_dst + col0 + j] = fmax(src[t], 0.0);
    }
}

// ---- fp64 GEMM on DMMA ---------------------------------------------------------------------------------
// C (m x n) = A (m x k) B (k x n), all row-major, contiguous.  CTA tile 64 x 64, 4 warps of 32 x 32 (4 x 4 DMMA tiles
// of 8 x 8), K in steps of 16 through shared memory.  Fragment layout of mma.m8n8k4.f64 (PTX ISA): with g = lane / 4,
// t = lane % 4:  A[g][t],  B[t][g],  C[g][2t], C[g][2t + 1].  The shared-memory row strides (20 and 68 doubles) put
// the 16 lanes of a half-warp on 16 different bank pairs for both fragment loads.  Edges are zero-filled on load and
// masked on store, so any m, n, k >= 1 works.
constexpr int GM = 64, GN = 64, GK = 16, GA_LD = GK + 4, GB_LD = GN + 4;

__device__ __forceinline__ void dmma_8x8x4(double &c0, double &c1, double a, double b) {
    asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};"
                 : "+d"(c0), "+d"(c1)
                 : "d"(a), "d"(b));
}

__global__ void __launch_bounds__(128)
dgemm_dmma_kernel(double *__restrict__ C, const double *__restrict__ A, const double *__restrict__ B, int64_t m, int n, int k) {
    __shared__ double As[GM][GA_LD];
    __shared__ double Bs[GK][GB_LD];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int g = lane >> 2, t = lane & 3;
    const int wr = (warp >> 1) * 32, wc = (warp & 1) * 32;  // this warp's 32 x 32 corner inside the CTA tile
    const int col_tiles = (n + GN - 1) / GN;
    const int64_t row_tiles = (m + GM - 1) / GM;
    for (int64_t tile = blockIdx.x; tile < row_tiles * col_tiles; tile += gridDim.x) {
        const int64_t row0 = (tile / col_tiles) * GM;
        const int col0 = (int)(tile % col_tiles) * GN;
        double acc[4][4][2];
#pragma unroll
        for (int i = 0; i < 4; i++)
#pragma unroll
            for (int j = 0; j < 4; j++) acc[i][j][0] = acc[i][j][1] = 0.0;
        for (int k0 = 0; k0 < k; k0 += GK) {
            __syncthreads();  // the previous K step has been consumed
            for (int e = threadIdx.x; e < GM * GK; e += 128) {
                const int r = e / GK, c = e % GK;
                const int64_t gr = row0 + r;
                As[r][c] = (gr < m && k0 + c < k) ? A[gr * k + k0 + c] : 0.0;
            }
            for (int e = threadIdx.x; e < GK * GN; e += 128) {
                const int r = e / GN, c = e % GN;
                Bs[r][c] = (k0 + r < k && col0 + c < n) ? B[(int64_t)(k0 + r) * n + col0 + c] : 0.0;
            }
            __syncthreads();
#pragma unroll
            for (int kk = 0; kk < GK; kk += 4) {
                double a[4], b[4];
#pragma unroll
                for (int i = 0; i < 4; i++) a[i] = As[wr + i * 8 + g][kk + t];
#pragma unroll
                for (int j = 0; j < 4; j++) b[j] = Bs[kk + t][wc + j * 8 + g];
#pragma unroll
                for (int i = 0; i < 4; i++)
#pragma unroll
                    for (int j = 0; j < 4; j++) dmma_8x8x4(acc[i][j][0], acc[i][j][1], a[i], b[j]);
            }
        }
#pragma unroll
        for (int i = 0; i < 4; i++) {
            const int64_t r = row0 + wr + i * 8 + g;
            if (r >= m) continue;
#pragma unroll
            for (int j = 0; j < 4; j++) {
                const int c = col0 + wc + j * 8 + 2 * t;
                if (c < n) C[r * n + c] = acc[i][j][0];
                if (c + 1 < n) C[r * n + c + 1] = acc[i][j][1];
            }
        }
    }
}

// ---- backward-pass elementwise kernels -----------------------------------------------------------------
// x -> 1 where x > 0, alpha elsewhere (the derivative of leaky_relu_kernel; alpha at 0, as torch's leaky_relu)
__global__ void leaky_relu_grad_kernel(double *__restrict__ dst, const double *__restrict__ src, int64_t n, double alpha) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) dst[i] = src[i] > 0.0 ? 1.0 : alpha;
}

// dst[i, j] = out[i, col0 + j] > 0 ? grad[i, col0 + j] : 0: dst is rows x cols, contiguous; grad and out have ld columns
__global__ void relu_cols_backward_kernel(double *__restrict__ dst, const double *__restrict__ grad, const double *__restrict__ out,
                                          int64_t ld, int64_t col0, int64_t rows, int64_t cols) {
    const int64_t n = rows * cols;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < n; t += stride) {
        const int64_t i = t / cols, j = t - i * cols;
        const int64_t s = i * ld + col0 + j;
        dst[t] = out[s] > 0.0 ? grad[s] : 0.0;
    }
}

// ---- weight-gradient GEMM: C (m x n) = A^T B, A k x m, B k x n, row-major -------------------------------
// The same CTA tile (64 x 64, 4 warps of 4 x 4 DMMA tiles) and fragment layout as dgemm_dmma_kernel, but both operands
// are K-major: a K step stages rows k0 .. k0 + 15 of A (64 columns) and of B (64 columns), each a coalesced run of 64
// doubles.  Both fragment loads read S[kk + t][x + g]; a row stride of 68 doubles (68 mod 16 = 4) puts the 16 lanes of
// a half-warp on 16 different bank pairs.  k is long (the local row count) and there are few output tiles, so
// blockIdx.y splits k: split s sums rows [s * chunk, (s + 1) * chunk) into its own m x n slice of `part` (or
// straight into C when there is one split); tn_reduce_kernel then adds the slices in split order.
constexpr int TN_LD = GM + 4;

__global__ void __launch_bounds__(128)
dgemm_tn_kernel(double *__restrict__ part, const double *__restrict__ A, const double *__restrict__ B, int m, int n, int64_t k,
                int64_t chunk) {
    __shared__ double As[GK][TN_LD];
    __shared__ double Bs[GK][TN_LD];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int g = lane >> 2, t = lane & 3;
    const int wr = (warp >> 1) * 32, wc = (warp & 1) * 32;
    const int col_tiles = (n + GN - 1) / GN;
    const int row0 = (int)(blockIdx.x / col_tiles) * GM;
    const int col0 = (int)(blockIdx.x % col_tiles) * GN;
    const int64_t k_lo = (int64_t)blockIdx.y * chunk;
    const int64_t k_hi = k_lo + chunk < k ? k_lo + chunk : k;
    double acc[4][4][2];
#pragma unroll
    for (int i = 0; i < 4; i++)
#pragma unroll
        for (int j = 0; j < 4; j++) acc[i][j][0] = acc[i][j][1] = 0.0;
    for (int64_t k0 = k_lo; k0 < k_hi; k0 += GK) {
        __syncthreads();
#pragma unroll
        for (int e = threadIdx.x; e < GK * GM; e += 128) {
            const int r = e / GM, c = e % GM;
            const int64_t kr = k0 + r;
            As[r][c] = (kr < k_hi && row0 + c < m) ? A[kr * m + row0 + c] : 0.0;
            Bs[r][c] = (kr < k_hi && col0 + c < n) ? B[kr * n + col0 + c] : 0.0;
        }
        __syncthreads();
#pragma unroll
        for (int kk = 0; kk < GK; kk += 4) {
            double a[4], b[4];
#pragma unroll
            for (int i = 0; i < 4; i++) a[i] = As[kk + t][wr + i * 8 + g];
#pragma unroll
            for (int j = 0; j < 4; j++) b[j] = Bs[kk + t][wc + j * 8 + g];
#pragma unroll
            for (int i = 0; i < 4; i++)
#pragma unroll
                for (int j = 0; j < 4; j++) dmma_8x8x4(acc[i][j][0], acc[i][j][1], a[i], b[j]);
        }
    }
    double *out = part + (int64_t)blockIdx.y * m * n;
#pragma unroll
    for (int i = 0; i < 4; i++) {
        const int r = row0 + wr + i * 8 + g;
        if (r >= m) continue;
#pragma unroll
        for (int j = 0; j < 4; j++) {
            const int c = col0 + wc + j * 8 + 2 * t;
            if (c < n) out[(int64_t)r * n + c] = acc[i][j][0];
            if (c + 1 < n) out[(int64_t)r * n + c + 1] = acc[i][j][1];
        }
    }
}

// C[i] = sum over s = 0 .. splits - 1 of part[s][i], always in that order (no atomics: bit-reproducible)
__global__ void tn_reduce_kernel(double *__restrict__ C, const double *__restrict__ part, int64_t mn, int64_t splits) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < mn; i += stride) {
        double s = part[i];
        for (int64_t q = 1; q < splits; q++) s += part[q * mn + i];
        C[i] = s;
    }
}

// How dgemm_tn_kernel splits k.  A function of the shape only (the workspace size is known without a device): about
// kTnTargetCtas CTAs in all, each split at least kTnMinChunk rows of k, the chunk a multiple of the K step.
constexpr int64_t kTnTargetCtas = 512, kTnMinChunk = 512;
void tn_plan(int64_t m, int64_t n, int64_t k, int64_t *splits, int64_t *chunk) {
    const int64_t tiles = ((m + GM - 1) / GM) * ((n + GN - 1) / GN);
    int64_t s = std::max<int64_t>(1, std::min((kTnTargetCtas + tiles - 1) / tiles, k / kTnMinChunk));
    int64_t c = (k + s - 1) / s;
    c = (c + GK - 1) / GK * GK;
    *chunk = c;
    *splits = (k + c - 1) / c;
}

// ---- input-gradient GEMM: C (m x n) (+)= A B^T, A m x k, B n x k, row-major ----------------------------
// dgemm_dmma_kernel's tiling with B staged like A (row = output column, 16 consecutive k): the B fragment B^T[t][g] is
// Bs[wc + j * 8 + g][kk + t], the same conflict-free pattern (stride 20) as the A fragment.
__global__ void __launch_bounds__(128)
dgemm_nt_kernel(double *__restrict__ C, const double *__restrict__ A, const double *__restrict__ B, int64_t m, int n, int k,
                int accumulate) {
    __shared__ double As[GM][GA_LD];
    __shared__ double Bs[GN][GA_LD];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int g = lane >> 2, t = lane & 3;
    const int wr = (warp >> 1) * 32, wc = (warp & 1) * 32;
    const int col_tiles = (n + GN - 1) / GN;
    const int64_t row_tiles = (m + GM - 1) / GM;
    for (int64_t tile = blockIdx.x; tile < row_tiles * col_tiles; tile += gridDim.x) {
        const int64_t row0 = (tile / col_tiles) * GM;
        const int col0 = (int)(tile % col_tiles) * GN;
        double acc[4][4][2];
#pragma unroll
        for (int i = 0; i < 4; i++)
#pragma unroll
            for (int j = 0; j < 4; j++) acc[i][j][0] = acc[i][j][1] = 0.0;
        for (int k0 = 0; k0 < k; k0 += GK) {
            __syncthreads();
#pragma unroll
            for (int e = threadIdx.x; e < GM * GK; e += 128) {
                const int r = e / GK, c = e % GK;
                const int64_t gr = row0 + r;
                As[r][c] = (gr < m && k0 + c < k) ? A[gr * k + k0 + c] : 0.0;
                Bs[r][c] = (col0 + r < n && k0 + c < k) ? B[(int64_t)(col0 + r) * k + k0 + c] : 0.0;
            }
            __syncthreads();
#pragma unroll
            for (int kk = 0; kk < GK; kk += 4) {
                double a[4], b[4];
#pragma unroll
                for (int i = 0; i < 4; i++) a[i] = As[wr + i * 8 + g][kk + t];
#pragma unroll
                for (int j = 0; j < 4; j++) b[j] = Bs[wc + j * 8 + g][kk + t];
#pragma unroll
                for (int i = 0; i < 4; i++)
#pragma unroll
                    for (int j = 0; j < 4; j++) dmma_8x8x4(acc[i][j][0], acc[i][j][1], a[i], b[j]);
            }
        }
#pragma unroll
        for (int i = 0; i < 4; i++) {
            const int64_t r = row0 + wr + i * 8 + g;
            if (r >= m) continue;
#pragma unroll
            for (int j = 0; j < 4; j++) {
                const int c = col0 + wc + j * 8 + 2 * t;
                double *p = C + r * n + c;
                if (c < n) p[0] = accumulate ? p[0] + acc[i][j][0] : acc[i][j][0];
                if (c + 1 < n) p[1] = accumulate ? p[1] + acc[i][j][1] : acc[i][j][1];
            }
        }
    }
}

}  // namespace

extern "C" {

int hnh_leaky_relu_f64(double *dst, const double *src, int64_t n, double alpha, void *stream) {
    if (n < 0) return set_error(HNH_E_INVALID, "hnh_leaky_relu_f64: negative size");
    if (n == 0) return HNH_OK;
    if (!dst || !src) return set_error(HNH_E_INVALID, "hnh_leaky_relu_f64: null pointer");
    int grid;
    int rc = grid_for(leaky_relu_kernel, n, kBlock * 4, &grid, kCtasPerSm);
    return rc ? rc : launch(leaky_relu_kernel, grid, kBlock, (cudaStream_t)stream, "leaky_relu_kernel", dst, src, n, alpha);
}

int hnh_relu_cols_f64(double *dst, int64_t ld_dst, int64_t col0, const double *src, int64_t rows, int64_t cols, void *stream) {
    if (rows < 0 || cols < 0 || col0 < 0 || ld_dst < col0 + cols)
        return set_error(HNH_E_INVALID, "hnh_relu_cols_f64: column window [%lld, %lld) outside a row of %lld",
                         (long long)col0, (long long)(col0 + cols), (long long)ld_dst);
    if (rows == 0 || cols == 0) return HNH_OK;
    if (!dst || !src) return set_error(HNH_E_INVALID, "hnh_relu_cols_f64: null pointer");
    int grid;
    int rc = grid_for(relu_cols_kernel, rows * cols, kBlock * 4, &grid, kCtasPerSm);
    return rc ? rc : launch(relu_cols_kernel, grid, kBlock, (cudaStream_t)stream, "relu_cols_kernel", dst, ld_dst, col0, src, rows, cols);
}

int hnh_dgemm_f64(double *C, const double *A, const double *B, int64_t m, int64_t n, int64_t k, void *stream) {
    if (m < 0 || n < 0 || k < 0 || m > INT32_MAX || n > INT32_MAX || k > INT32_MAX)
        return set_error(HNH_E_INVALID, "hnh_dgemm_f64: bad shape %lld x %lld x %lld", (long long)m, (long long)n, (long long)k);
    if (m == 0 || n == 0) return HNH_OK;
    if (!C || (k > 0 && (!A || !B))) return set_error(HNH_E_INVALID, "hnh_dgemm_f64: null pointer");
    if (k == 0)
        return check_cuda(cudaMemsetAsync(C, 0, sizeof(double) * (size_t)(m * n), (cudaStream_t)stream), "cudaMemsetAsync");
    const int64_t tiles = ((m + GM - 1) / GM) * ((n + GN - 1) / GN);
    int grid;
    int rc = grid_for(dgemm_dmma_kernel, tiles, 1, &grid, kCtasPerSm);
    return rc ? rc : launch(dgemm_dmma_kernel, grid, 128, (cudaStream_t)stream, "dgemm_dmma_kernel", C, A, B, m, (int)n, (int)k);
}

int hnh_leaky_relu_grad_f64(double *dst, const double *src, int64_t n, double alpha, void *stream) {
    if (n < 0) return set_error(HNH_E_INVALID, "hnh_leaky_relu_grad_f64: negative size");
    if (n == 0) return HNH_OK;
    if (!dst || !src) return set_error(HNH_E_INVALID, "hnh_leaky_relu_grad_f64: null pointer");
    int grid;
    int rc = grid_for(leaky_relu_grad_kernel, n, kBlock * 4, &grid, kCtasPerSm);
    return rc ? rc : launch(leaky_relu_grad_kernel, grid, kBlock, (cudaStream_t)stream, "leaky_relu_grad_kernel", dst, src, n, alpha);
}

int hnh_relu_cols_backward_f64(double *dst, const double *grad, const double *out, int64_t ld, int64_t col0, int64_t rows,
                               int64_t cols, void *stream) {
    if (rows < 0 || cols < 0 || col0 < 0 || ld < col0 + cols)
        return set_error(HNH_E_INVALID, "hnh_relu_cols_backward_f64: column window [%lld, %lld) outside a row of %lld",
                         (long long)col0, (long long)(col0 + cols), (long long)ld);
    if (rows == 0 || cols == 0) return HNH_OK;
    if (!dst || !grad || !out) return set_error(HNH_E_INVALID, "hnh_relu_cols_backward_f64: null pointer");
    int grid;
    int rc = grid_for(relu_cols_backward_kernel, rows * cols, kBlock * 4, &grid, kCtasPerSm);
    return rc ? rc : launch(relu_cols_backward_kernel, grid, kBlock, (cudaStream_t)stream, "relu_cols_backward_kernel", dst, grad, out, ld, col0, rows, cols);
}

int64_t hnh_dgemm_tn_workspace_bytes(int64_t m, int64_t n, int64_t k) {
    // m, n: layer widths (one grid row of CTAs per 64 x 64 output tile); k: any row count
    if (m < 0 || n < 0 || k < 0 || m > (1 << 20) || n > (1 << 20))
        return set_error(HNH_E_INVALID, "hnh_dgemm_tn_workspace_bytes: bad shape %lld x %lld x %lld", (long long)m,
                         (long long)n, (long long)k);
    if (m == 0 || n == 0 || k == 0) return 0;
    int64_t splits, chunk;
    tn_plan(m, n, k, &splits, &chunk);
    return splits > 1 ? (int64_t)sizeof(double) * splits * m * n : 0;
}

int hnh_dgemm_tn_f64(double *C, const double *A, const double *B, int64_t m, int64_t n, int64_t k, void *workspace,
                     size_t workspace_bytes, void *stream) {
    const int64_t need = hnh_dgemm_tn_workspace_bytes(m, n, k);
    if (need < 0) return (int)need;
    if (m == 0 || n == 0) return HNH_OK;
    if (!C || (k > 0 && (!A || !B))) return set_error(HNH_E_INVALID, "hnh_dgemm_tn_f64: null pointer");
    if (need > 0 && (!workspace || workspace_bytes < (size_t)need))
        return set_error(HNH_E_INVALID, "hnh_dgemm_tn_f64: workspace of %zu bytes, %lld needed", workspace_bytes, (long long)need);
    if (k == 0)
        return check_cuda(cudaMemsetAsync(C, 0, sizeof(double) * (size_t)(m * n), (cudaStream_t)stream), "cudaMemsetAsync");
    int64_t splits, chunk;
    tn_plan(m, n, k, &splits, &chunk);
    const int64_t tiles = ((m + GM - 1) / GM) * ((n + GN - 1) / GN);
    double *part = splits > 1 ? (double *)workspace : C;
    int rc = launch(dgemm_tn_kernel, dim3((unsigned)tiles, (unsigned)splits), 128, (cudaStream_t)stream, "dgemm_tn_kernel", part, A, B,
                    (int)m, (int)n, k, chunk);
    if (rc || splits == 1) return rc;
    int grid;
    rc = grid_for(tn_reduce_kernel, m * n, kBlock * 4, &grid, kCtasPerSm);
    return rc ? rc : launch(tn_reduce_kernel, grid, kBlock, (cudaStream_t)stream, "tn_reduce_kernel", C, part, m * n, splits);
}

int hnh_dgemm_nt_f64(double *C, const double *A, const double *B, int64_t m, int64_t n, int64_t k, int accumulate, void *stream) {
    if (m < 0 || n < 0 || k < 0 || m > INT32_MAX || n > INT32_MAX || k > INT32_MAX)
        return set_error(HNH_E_INVALID, "hnh_dgemm_nt_f64: bad shape %lld x %lld x %lld", (long long)m, (long long)n, (long long)k);
    if (m == 0 || n == 0 || (k == 0 && accumulate)) return HNH_OK;
    if (!C || (k > 0 && (!A || !B))) return set_error(HNH_E_INVALID, "hnh_dgemm_nt_f64: null pointer");
    if (k == 0)
        return check_cuda(cudaMemsetAsync(C, 0, sizeof(double) * (size_t)(m * n), (cudaStream_t)stream), "cudaMemsetAsync");
    const int64_t tiles = ((m + GM - 1) / GM) * ((n + GN - 1) / GN);
    int grid;
    int rc = grid_for(dgemm_nt_kernel, tiles, 1, &grid, kCtasPerSm);
    return rc ? rc : launch(dgemm_nt_kernel, grid, 128, (cudaStream_t)stream, "dgemm_nt_kernel", C, A, B, m, (int)n, (int)k, accumulate ? 1 : 0);
}

}  // extern "C"
