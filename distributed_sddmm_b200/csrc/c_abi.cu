// c_abi.cu -- extern "C" layer of libhnh_b200.so: argument validation, kernel selection
// and launch for the entry points declared in include/hnh_b200.h.
#include "kernels.cuh"

#include <atomic>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <mutex>

namespace hnh {

static thread_local char g_err[512] = "";
static std::atomic<uint64_t> g_launches{0};

int set_error(int code, const char *fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
    return code;
}

void count_launch(uint64_t n) { g_launches.fetch_add(n, std::memory_order_relaxed); }

int check_cuda(cudaError_t e, const char *what) {
    if (e == cudaSuccess) return HNH_OK;
    return set_error(HNH_E_CUDA, "%s: %s", what, cudaGetErrorString(e));
}

// Per-device constants, looked up once.
struct DeviceInfo {
    int sm_count = 0;
    bool ok = false;
};
static DeviceInfo g_dev[64];
static std::mutex g_dev_mu;

int device_sm_count(int *out) {
    int dev = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e != cudaSuccess) return check_cuda(e, "cudaGetDevice");
    if (dev < 0 || dev >= 64) return set_error(HNH_E_CUDA, "device ordinal %d out of range", dev);
    if (!g_dev[dev].ok) {
        std::lock_guard<std::mutex> lk(g_dev_mu);
        int n = 0;
        e = cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
        if (e != cudaSuccess) return check_cuda(e, "cudaDeviceGetAttribute");
        g_dev[dev].sm_count = n;
        g_dev[dev].ok = true;
    }
    *out = g_dev[dev].sm_count;
    return HNH_OK;
}

// ------------------------------------------------------------------ K4 + row algebra -----
__global__ void fill_kernel(double *__restrict__ dst, int64_t n, double value) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride)
        dst[i] = value;
}

// uniform(-1, 1) from a counter-based hash of (seed, i): Eigen's setRandom() stand-in
__global__ void random_uniform_kernel(double *__restrict__ dst, int64_t n, uint64_t seed) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
        uint64_t z = seed + (uint64_t)i * 0x9E3779B97F4A7C15ull + 0x9E3779B97F4A7C15ull;
        z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
        z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
        z ^= z >> 31;
        dst[i] = (double)(z >> 11) * (2.0 / 9007199254740992.0) - 1.0;
    }
}

__global__ void hadamard_kernel(double *__restrict__ dst, const double *__restrict__ a,
                                const double *__restrict__ b, int64_t n) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride)
        dst[i] = a[i] * b[i];
}

__global__ void expand_row_idx_kernel(const int64_t *__restrict__ rowStart, int64_t rows,
                                      int64_t *__restrict__ row_idx) {
    const int lane = threadIdx.x & 31;
    const int64_t nwarps = (int64_t)gridDim.x * (blockDim.x >> 5);
    for (int64_t row = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); row < rows;
         row += nwarps) {
        const int64_t s = rowStart[row], e = rowStart[row + 1];
        for (int64_t j = s + lane; j < e; j += 32) row_idx[j] = row;
    }
}

__global__ void batch_dot_kernel(double *__restrict__ out, const double *__restrict__ A,
                                 const double *__restrict__ B, int64_t rows, int r) {
    const int lane = threadIdx.x & 31;
    const int64_t nwarps = (int64_t)gridDim.x * (blockDim.x >> 5);
    for (int64_t row = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); row < rows;
         row += nwarps) {
        double d = 0.0;
        for (int k = lane; k < r; k += 32)
            d = fma(A[row * (int64_t)r + k], B[row * (int64_t)r + k], d);
        d = group_allreduce<32>(d, 0xffffffffu);
        if (lane == 0) out[row] = d;
    }
}

__global__ void row_axpy_kernel(double *D, const double *C, double alpha,
                                const double *__restrict__ s, const double *M, int64_t rows,
                                int r) {
    const int64_t n = rows * (int64_t)r;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
        const double sc = s ? s[i / r] : 1.0;
        D[i] = (C ? C[i] : 0.0) + alpha * sc * M[i];
    }
}

__global__ void vec_quotient_kernel(double *out, const double *a, double ca, const double *b,
                                    double cb, int64_t n) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride)
        out[i] = b ? (a[i] + ca) / (b[i] + cb) : (a[i] + ca);
}

__global__ void axpby_kernel(double *dst, double alpha, const double *x, double beta,
                             const double *y, int64_t n) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride)
        dst[i] = alpha * x[i] + (y ? beta * y[i] : 0.0);
}

// Deterministic two-pass sum of squares (fingerprints and residuals must be bit-stable run to run): pass 1 leaves
// one partial per CTA (fixed grid-stride assignment, fixed shuffle tree), pass 2 -- one CTA -- adds the partials
// in a fixed order.  No atomics.
__global__ void squared_norm_partial_kernel(double *__restrict__ partial, const double *__restrict__ x, int64_t n) {
    __shared__ double warp_sums[8];
    double acc = 0.0;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride)
        acc = fma(x[i], x[i], acc);
    acc = group_allreduce<32>(acc, 0xffffffffu);
    if ((threadIdx.x & 31) == 0) warp_sums[threadIdx.x >> 5] = acc;
    __syncthreads();
    if (threadIdx.x == 0) {
        double t = 0.0;
        for (int w = 0; w < (int)(blockDim.x >> 5); w++) t += warp_sums[w];
        partial[blockIdx.x] = t;
    }
}

__global__ void sum_partials_kernel(double *__restrict__ out, const double *__restrict__ partial, int n) {
    __shared__ double warp_sums[8];
    double acc = 0.0;
    for (int i = threadIdx.x; i < n; i += blockDim.x) acc += partial[i];
    acc = group_allreduce<32>(acc, 0xffffffffu);
    if ((threadIdx.x & 31) == 0) warp_sums[threadIdx.x >> 5] = acc;
    __syncthreads();
    if (threadIdx.x == 0) {
        double t = 0.0;
        for (int w = 0; w < (int)(blockDim.x >> 5); w++) t += warp_sums[w];
        *out = t;
    }
}


// Narrow factors (r <= split_max_r()) use the split kernels.  Shape table:
// R -> (GK lanes across r, GN lanes across the row's nonzeros, VW, UN).
#define HNH_DISPATCH_SPLIT(r, CALL)            \
    switch (r) {                              \
        case 4:  CALL(4, 2, 8, 2, 4); break;   \
        case 8:  CALL(8, 4, 8, 2, 4); break;   \
        case 16: CALL(16, 8, 4, 2, 4); break;  \
        case 32: CALL(32, 16, 2, 2, 4); break; \
        default: break;                       \
    }

static int split_max_r() {
    static int v = -1;
    if (v < 0) {
        const char *e = getenv("HNH_SPLIT_MAX_R");
        v = e ? atoi(e) : 32;
    }
    return v;
}

// ---- TMA-staged kernels (HNH_FLAG_TMA_STAGE / HNH_FLAG_TMA_WARP; r in {128, 256}, 16-byte aligned operands) -----------
// Default choice between the TMA-staged and the direct-load row kernels: TMA staging for SDDMM at
// r = 128 and 256 and for the overwriting fused kernel at r = 256; the direct kernel for the fused
// kernel at r = 128, where the per-tile barrier makes the 8 warps of a CTA wait for the longest of
// their rows.  HNH_TMA=0 / 1 forces one or the other everywhere.
static bool tma_default(bool fused, int r, bool overwrite_out) {
    static int v = -2;
    if (v == -2) {
        const char *e = getenv("HNH_TMA");
        v = e ? (atoi(e) != 0 ? 1 : 0) : -1;
    }
    if (v >= 0) return v == 1;
    return fused ? (r == 256 && overwrite_out) : true;
}

// ---- the direct-load fused kernel of a table width ------------------------------------------------------------------
// fused_ring_kernel's shape at the widths where it runs (DESIGN.md section 3, chosen by a sweep at 2^20 rows x 32
// entries): UN rows per batch, S ring slots, CTAs per SM in its __launch_bounds__ -- all without spills, and the ring
// within the 48 KB of static shared memory of a CTA.  Every other width keeps fused_row_kernel (S = 0).
template <int R> struct FusedRing { static constexpr int UN = 0, S = 0, MINB = 0; };
template <> struct FusedRing<64> { static constexpr int UN = 2, S = 4, MINB = 3; };
template <> struct FusedRing<128> { static constexpr int UN = 2, S = 3, MINB = 3; };
template <> struct FusedRing<256> { static constexpr int UN = 1, S = 3, MINB = 2; };

using FusedKernel = decltype(&fused_row_kernel<4, 2, 2, 2, true, true>);
template <int R, int G, int VW, int UN>
static FusedKernel fused_direct_kernel(bool scale, bool bv, bool bo, const char **name) {
    using F = FusedRing<R>;
    if constexpr (F::S > 0) {
        *name = "fused_ring_kernel";
        return scale ? (bo ? fused_ring_kernel<R, F::UN, F::S, F::MINB, true, true, true>
                           : fused_ring_kernel<R, F::UN, F::S, F::MINB, true, false, true>)
             : bv   ? (bo ? fused_ring_kernel<R, F::UN, F::S, F::MINB, true, true> : fused_ring_kernel<R, F::UN, F::S, F::MINB, true, false>)
                    : (bo ? fused_ring_kernel<R, F::UN, F::S, F::MINB, false, true> : fused_ring_kernel<R, F::UN, F::S, F::MINB, false, false>);
    } else {
        *name = "fused_row_kernel";
        return scale ? (bo ? fused_row_kernel<R, G, VW, UN, true, true, true> : fused_row_kernel<R, G, VW, UN, true, false, true>)
             : bv   ? (bo ? fused_row_kernel<R, G, VW, UN, true, true> : fused_row_kernel<R, G, VW, UN, true, false>)
                    : (bo ? fused_row_kernel<R, G, VW, UN, false, true> : fused_row_kernel<R, G, VW, UN, false, false>);
    }
}

// the tile-staged (tma_row_kernel) or per-warp (tma_warp_kernel) instantiation for the overwrite flags
template <int R, bool FUSED>
auto tma_kernel(bool per_warp, bool bv, bool bo) {
    if (per_warp)
        return bv ? (bo ? tma_warp_kernel<R, 4, FUSED, true, true> : tma_warp_kernel<R, 4, FUSED, true, false>)
                  : (bo ? tma_warp_kernel<R, 4, FUSED, false, true> : tma_warp_kernel<R, 4, FUSED, false, false>);
    return bv ? (bo ? tma_row_kernel<R, 4, FUSED, true, true> : tma_row_kernel<R, 4, FUSED, true, false>)
              : (bo ? tma_row_kernel<R, 4, FUSED, false, true> : tma_row_kernel<R, 4, FUSED, false, false>);
}

static int validate_common(const void *a, const void *b, const void *c, int64_t rows,
                           int64_t nnz, int r, const char *who) {
    if (rows < 0 || nnz < 0) return set_error(HNH_E_INVALID, "%s: negative size", who);
    if (r <= 0) return set_error(HNH_E_INVALID, "%s: r must be positive (got %d)", who, r);
    if (rows == 0 || nnz == 0) return 1;  // successful no-op
    if (!a || !b || !c) return set_error(HNH_E_INVALID, "%s: null pointer", who);
    return HNH_OK;
}

}  // namespace hnh

using namespace hnh;

extern "C" {

int hnh_abi_version(void) { return 1; }

const char *hnh_build_info(void) {
    return "hnh_b200 sm_90a fp64 int64 (CUDA " HNH_STR(CUDART_VERSION) ")";
}

const char *hnh_last_error_string(void) { return g_err; }

uint64_t hnh_launch_count(void) { return g_launches.load(std::memory_order_relaxed); }

int hnh_sddmm_scaled_f64(const int64_t *rowStart, const int64_t *col_idx, double *values, int64_t rows,
                         int64_t nnz, const double *X, const double *Y, int r, int flags, const double *scale,
                         double *scaled_out, void *stream) {
    int v = validate_common(rowStart, col_idx, values, rows, nnz, r, "hnh_sddmm_f64");
    if (scaled_out && !scale) return set_error(HNH_E_INVALID, "hnh_sddmm_scaled_f64: scaled_out without scale");
    if (v < 0) return v;
    if (v == 1) return HNH_OK;
    if (!X || !Y) return set_error(HNH_E_INVALID, "hnh_sddmm_f64: null dense operand");
    cudaStream_t st = (cudaStream_t)stream;
    int grid = 0, rc = HNH_OK;
    const bool beta0 = (flags & HNH_FLAG_BETA0) != 0;
    const bool generic = (flags & HNH_FLAG_FORCE_GENERIC) || !aligned16(X) || !aligned16(Y) || !table_width(r);
    // The epilogue form needs a table kernel and distinct arrays (scale is read through the read-only path); otherwise
    // the product is one more elementwise pass after the plain SDDMM.
    if (scale && (generic || (const double *)scaled_out == scale || values == scale)) {
        rc = hnh_sddmm_scaled_f64(rowStart, col_idx, values, rows, nnz, X, Y, r, flags & ~HNH_FLAG_SCALE_VALUES, nullptr, nullptr, stream);
        if (rc) return rc;
        if (scaled_out && !(flags & HNH_FLAG_SCALE_VALUES)) return hnh_hadamard_f64(scaled_out, scale, values, nnz, stream);
        // the values take the product first: scaled_out may alias scale, so it receives a copy of them afterwards
        rc = hnh_hadamard_f64(values, scale, values, nnz, stream);
        if (rc || !scaled_out || scaled_out == values) return rc;
        return check_cuda(cudaMemcpyAsync(scaled_out, values, sizeof(double) * (size_t)nnz, cudaMemcpyDeviceToDevice, st),
                          "cudaMemcpyAsync");
    }
    const bool sv = (flags & HNH_FLAG_SCALE_VALUES) != 0;
    const bool warp = (flags & HNH_FLAG_TMA_WARP) != 0;
    if (!generic && (r == 128 || r == 256) &&
        (warp || (flags & HNH_FLAG_TMA_STAGE) || (tma_default(false, r, beta0) && !(flags & HNH_FLAG_FORCE_DIRECT)))) {
        auto k = r == 128 ? tma_kernel<128, false>(warp, beta0, false) : tma_kernel<256, false>(warp, beta0, false);
        rc = grid_for(k, rows, 8, &grid);
        return rc ? rc : launch(k, grid, kBlock, st, warp ? "tma_warp_kernel" : "tma_row_kernel", rowStart, col_idx, values, rows,
                                X, Y, nullptr, scale, scaled_out, sv);
    }
    if (generic) {
        if (beta0) {  // the any-r kernel accumulates: clear first
            rc = check_cuda(cudaMemsetAsync(values, 0, sizeof(double) * (size_t)nnz, st), "cudaMemsetAsync");
            if (rc) return rc;
        }
        rc = grid_for(sddmm_generic_kernel, rows, kBlock / 32, &grid);
        return rc ? rc : launch(sddmm_generic_kernel, grid, kBlock, st, "sddmm_generic_kernel", rowStart, col_idx, values, rows, X, Y, r);
    }
    decltype(&sddmm_row_kernel<4, 2, 2, 2, true>) k = nullptr;
    int64_t per_cta = 0;
    const char *name = "sddmm_split_kernel";
    if (r <= split_max_r() && r <= 32) {
#define SP(R, GK, GN, VW, UN)                                                                                    \
    {                                                                                                            \
        k = beta0 ? sddmm_split_kernel<R, GK, GN, VW, UN, true> : sddmm_split_kernel<R, GK, GN, VW, UN, false>;  \
        per_cta = kBlock / (GK * GN);                                                                            \
    }
        HNH_DISPATCH_SPLIT(r, SP)
#undef SP
    } else {
        name = "sddmm_row_kernel";
#define S4(R, G, VW, UN)                                                                         \
    {                                                                                            \
        k = beta0 ? sddmm_row_kernel<R, G, VW, UN, true> : sddmm_row_kernel<R, G, VW, UN, false>; \
        per_cta = kBlock / G;                                                                    \
    }
        HNH_DISPATCH_R(r, S4, )
#undef S4
    }
    rc = grid_for(k, rows, per_cta, &grid);
    return rc ? rc : launch(k, grid, kBlock, st, name, rowStart, col_idx, values, rows, X, Y, scale, scaled_out, sv);
}

int hnh_sddmm_f64(const int64_t *rowStart, const int64_t *col_idx, double *values, int64_t rows,
                  int64_t nnz, const double *X, const double *Y, int r, int flags, void *stream) {
    return hnh_sddmm_scaled_f64(rowStart, col_idx, values, rows, nnz, X, Y, r, flags, nullptr, nullptr, stream);
}

int hnh_sddmm_coo_f64(const int64_t *row_idx, const int64_t *col_idx, double *values,
                      int64_t nnz, const double *X, const double *Y, int r, int flags,
                      void *stream) {
    int v = validate_common(row_idx, col_idx, values, 1, nnz, r, "hnh_sddmm_coo_f64");
    if (v < 0) return v;
    if (v == 1) return HNH_OK;
    if (!X || !Y) return set_error(HNH_E_INVALID, "hnh_sddmm_coo_f64: null dense operand");
    cudaStream_t st = (cudaStream_t)stream;
    int grid = 0, rc = HNH_OK;
#define S4(R, G, VW, UN)                                                                                     \
    {                                                                                                        \
        auto k = sddmm_coo_kernel<R, G, VW, (UN > 2 ? 2 : UN)>;                                              \
        rc = grid_for(k, nnz, (int64_t)(kBlock / G) * G, &grid);                                             \
        if (!rc) rc = launch(k, grid, kBlock, st, "sddmm_coo_kernel", row_idx, col_idx, values, nnz, X, Y);  \
    }
#define SGEN                                                                                                 \
    {                                                                                                        \
        rc = grid_for(sddmm_coo_generic_kernel, nnz, kBlock / 32, &grid);                                    \
        if (!rc)                                                                                             \
            rc = launch(sddmm_coo_generic_kernel, grid, kBlock, st, "sddmm_coo_generic_kernel", row_idx,     \
                        col_idx, values, nnz, X, Y, r);                                                      \
    }
    if ((flags & HNH_FLAG_FORCE_GENERIC) || !aligned16(X) || !aligned16(Y)) {
        SGEN
    } else {
        HNH_DISPATCH_R(r, S4, SGEN)
    }
#undef S4
#undef SGEN
    return rc;
}

int hnh_spmm_f64(const int64_t *rowStart, const int64_t *col_idx, const double *values,
                 int64_t rows, int64_t nnz, const double *X, double *Y, int r, int flags,
                 void *stream) {
    int v = validate_common(rowStart, col_idx, values, rows, nnz, r, "hnh_spmm_f64");
    if (v < 0) return v;
    cudaStream_t st = (cudaStream_t)stream;
    if (v == 1) {
        // BETA0 == "zero the output first": an empty block still has to leave Y = 0
        if ((flags & HNH_FLAG_BETA0) && rows > 0) {
            if (!Y) return set_error(HNH_E_INVALID, "hnh_spmm_f64: null dense operand");
            return check_cuda(cudaMemsetAsync(Y, 0, sizeof(double) * (size_t)rows * r, st), "cudaMemsetAsync");
        }
        return HNH_OK;
    }
    if (!X || !Y) return set_error(HNH_E_INVALID, "hnh_spmm_f64: null dense operand");
    int grid = 0, rc = HNH_OK;
    const bool beta0 = (flags & HNH_FLAG_BETA0) != 0;
    if ((flags & HNH_FLAG_FORCE_GENERIC) || !aligned16(X) || !aligned16(Y) || !table_width(r)) {
        if (beta0) {
            rc = check_cuda(cudaMemsetAsync(Y, 0, sizeof(double) * (size_t)rows * r, st), "cudaMemsetAsync");
            if (rc) return rc;
        }
        rc = grid_for(spmm_generic_kernel, rows, kBlock / 32, &grid);
        return rc ? rc : launch(spmm_generic_kernel, grid, kBlock, st, "spmm_generic_kernel", rowStart, col_idx, values, rows, X, Y, r);
    }
    decltype(&spmm_row_kernel<4, 2, 2, 2, true>) k = nullptr;
    int64_t per_cta = 0;
    const char *name = "spmm_split_kernel";
    if (r <= split_max_r() && r <= 32) {
#define SP(R, GK, GN, VW, UN)                                                                                  \
    {                                                                                                          \
        k = beta0 ? spmm_split_kernel<R, GK, GN, VW, UN, true> : spmm_split_kernel<R, GK, GN, VW, UN, false>;  \
        per_cta = kBlock / (GK * GN);                                                                          \
    }
        HNH_DISPATCH_SPLIT(r, SP)
#undef SP
    } else {
        name = "spmm_row_kernel";
#define S4(R, G, VW, UN)                                                                       \
    {                                                                                          \
        k = beta0 ? spmm_row_kernel<R, G, VW, UN, true> : spmm_row_kernel<R, G, VW, UN, false>; \
        per_cta = kBlock / G;                                                                  \
    }
        HNH_DISPATCH_R(r, S4, )
#undef S4
    }
    rc = grid_for(k, rows, per_cta, &grid);
    return rc ? rc : launch(k, grid, kBlock, st, name, rowStart, col_idx, values, rows, X, Y);
}

int hnh_fused_scaled_f64(const int64_t *rowStart, const int64_t *col_idx, double *values, int64_t rows,
                         int64_t nnz, const double *X, const double *Y, double *Out, int r, int flags,
                         const double *scale, double *scaled_out, void *stream) {
    int v = validate_common(rowStart, col_idx, values, rows, nnz, r, "hnh_fused_f64");
    if (scaled_out && !scale) return set_error(HNH_E_INVALID, "hnh_fused_scaled_f64: scaled_out without scale");
    if (v < 0) return v;
    cudaStream_t st = (cudaStream_t)stream;
    if (v == 1) {
        // BETA0_OUT == "zero Out first": an empty block still has to leave Out = 0 (also in place, Out == X)
        if ((flags & (HNH_FLAG_BETA0 | HNH_FLAG_BETA0_OUT)) && rows > 0) {
            if (!Out) return set_error(HNH_E_INVALID, "hnh_fused_f64: null dense operand");
            return check_cuda(cudaMemsetAsync(Out, 0, sizeof(double) * (size_t)rows * r, st), "cudaMemsetAsync");
        }
        return HNH_OK;
    }
    if (!X || !Y || !Out) return set_error(HNH_E_INVALID, "hnh_fused_f64: null dense operand");
    int grid = 0, rc = HNH_OK;
    const bool bv = (flags & (HNH_FLAG_BETA0 | HNH_FLAG_BETA0_VALUES)) != 0;
    const bool bo = (flags & (HNH_FLAG_BETA0 | HNH_FLAG_BETA0_OUT)) != 0;
    if (X == Out && !bo)
        return set_error(HNH_E_INVALID, "hnh_fused_f64: Out may alias X only when Out is overwritten (BETA0_OUT)");
    const bool generic =
        (flags & HNH_FLAG_FORCE_GENERIC) || !aligned16(X) || !aligned16(Y) || !aligned16(Out) || !table_width(r);
    if (scale) {
        // the scaled epilogue exists in the first-visit form of the direct-load table kernels only
        if (!bv) return set_error(HNH_E_INVALID, "hnh_fused_scaled_f64: scale needs HNH_FLAG_BETA0_VALUES");
        if (generic)
            return set_error(HNH_E_INVALID, "hnh_fused_scaled_f64: scale needs a table width (4..256, power of two) and 16-byte "
                                            "aligned operands");
        if (values == scale || (const double *)scaled_out == scale)
            return set_error(HNH_E_INVALID, "hnh_fused_scaled_f64: scale must not alias values / scaled_out");
        flags = (flags | HNH_FLAG_FORCE_DIRECT) & ~(HNH_FLAG_TMA_STAGE | HNH_FLAG_TMA_WARP);
    }
    // in place (Out == X) is not offered with TMA staging: the next tile of X is prefetched while
    // the current one is still being written
    const bool warp = (flags & HNH_FLAG_TMA_WARP) != 0;
    if (!generic && (r == 128 || r == 256) && X != Out &&
        (warp || (flags & HNH_FLAG_TMA_STAGE) || (tma_default(true, r, bo) && !(flags & HNH_FLAG_FORCE_DIRECT)))) {
        auto k = r == 128 ? tma_kernel<128, true>(warp, bv, bo) : tma_kernel<256, true>(warp, bv, bo);
        rc = grid_for(k, rows, 8, &grid);
        return rc ? rc : launch(k, grid, kBlock, st, warp ? "tma_warp_kernel" : "tma_row_kernel", rowStart, col_idx, values, rows,
                                X, Y, Out, nullptr, nullptr, false);
    }
    if (generic) {
        if (X == Out)
            return set_error(HNH_E_INVALID, "hnh_fused_f64: in-place (Out == X) needs a table r "
                                            "(4..256, power of two) and 16-byte aligned operands");
        if (bv) rc = check_cuda(cudaMemsetAsync(values, 0, sizeof(double) * (size_t)nnz, st), "cudaMemsetAsync");
        if (!rc && bo) rc = check_cuda(cudaMemsetAsync(Out, 0, sizeof(double) * (size_t)rows * r, st), "cudaMemsetAsync");
        if (!rc) rc = grid_for(fused_generic_kernel, rows, kBlock / 32, &grid);
        return rc ? rc : launch(fused_generic_kernel, grid, kBlock, st, "fused_generic_kernel", rowStart, col_idx, values, rows, X, Y, Out, r);
    }
    // the scaled epilogue is a first-visit (BETA0_VALUES) form
    FusedKernel k = nullptr;
    int64_t per_cta = 0;
    const char *name = "fused_split_kernel";
    if (r <= split_max_r() && r <= 32) {
#define SP(R, GK, GN, VW, UN)                                                                                                \
    {                                                                                                                        \
        k = scale ? (bo ? fused_split_kernel<R, GK, GN, VW, UN, true, true, true> : fused_split_kernel<R, GK, GN, VW, UN, true, false, true>) \
            : bv  ? (bo ? fused_split_kernel<R, GK, GN, VW, UN, true, true> : fused_split_kernel<R, GK, GN, VW, UN, true, false>)             \
                  : (bo ? fused_split_kernel<R, GK, GN, VW, UN, false, true> : fused_split_kernel<R, GK, GN, VW, UN, false, false>);          \
        per_cta = kBlock / (GK * GN);                                                                                        \
    }
        HNH_DISPATCH_SPLIT(r, SP)
#undef SP
    } else {
#define S4(R, G, VW, UN)                                                    \
    {                                                                       \
        k = fused_direct_kernel<R, G, VW, UN>(scale != nullptr, bv, bo, &name); \
        per_cta = kBlock / G;                                               \
    }
        HNH_DISPATCH_R(r, S4, )
#undef S4
    }
    rc = grid_for(k, rows, per_cta, &grid);
    return rc ? rc : launch(k, grid, kBlock, st, name, rowStart, col_idx, values, rows, X, Y, Out, scale, scaled_out);
}

int hnh_fused_f64(const int64_t *rowStart, const int64_t *col_idx, double *values, int64_t rows,
                  int64_t nnz, const double *X, const double *Y, double *Out, int r, int flags,
                  void *stream) {
    return hnh_fused_scaled_f64(rowStart, col_idx, values, rows, nnz, X, Y, Out, r, flags, nullptr, nullptr, stream);
}

// ---- K4 + row algebra: one thread per element, kBlock * 4 elements per CTA ------------------------------------------
int hnh_fill_f64(double *dst, int64_t n, double value, void *stream) {
    if (n < 0) return set_error(HNH_E_INVALID, "hnh_fill_f64: negative size");
    if (n == 0) return HNH_OK;
    if (!dst) return set_error(HNH_E_INVALID, "hnh_fill_f64: null pointer");
    if (value == 0.0)
        return check_cuda(cudaMemsetAsync(dst, 0, sizeof(double) * (size_t)n, (cudaStream_t)stream), "cudaMemsetAsync");
    int grid;
    int rc = grid_for(fill_kernel, n, kBlock * 4, &grid);
    return rc ? rc : launch(fill_kernel, grid, kBlock, (cudaStream_t)stream, "fill_kernel", dst, n, value);
}

int hnh_random_uniform_f64(double *dst, int64_t n, uint64_t seed, void *stream) {
    if (n < 0) return set_error(HNH_E_INVALID, "hnh_random_uniform_f64: negative size");
    if (n == 0) return HNH_OK;
    if (!dst) return set_error(HNH_E_INVALID, "hnh_random_uniform_f64: null pointer");
    int grid;
    int rc = grid_for(random_uniform_kernel, n, kBlock * 4, &grid);
    return rc ? rc : launch(random_uniform_kernel, grid, kBlock, (cudaStream_t)stream, "random_uniform_kernel", dst, n, seed);
}

int hnh_hadamard_f64(double *dst, const double *a, const double *b, int64_t n, void *stream) {
    if (n < 0) return set_error(HNH_E_INVALID, "hnh_hadamard_f64: negative size");
    if (n == 0) return HNH_OK;
    if (!dst || !a || !b) return set_error(HNH_E_INVALID, "hnh_hadamard_f64: null pointer");
    int grid;
    int rc = grid_for(hadamard_kernel, n, kBlock * 4, &grid);
    return rc ? rc : launch(hadamard_kernel, grid, kBlock, (cudaStream_t)stream, "hadamard_kernel", dst, a, b, n);
}

int hnh_expand_row_idx(const int64_t *rowStart, int64_t rows, int64_t nnz, int64_t *row_idx,
                       void *stream) {
    if (rows < 0 || nnz < 0) return set_error(HNH_E_INVALID, "hnh_expand_row_idx: negative size");
    if (rows == 0 || nnz == 0) return HNH_OK;
    if (!rowStart || !row_idx) return set_error(HNH_E_INVALID, "hnh_expand_row_idx: null pointer");
    int grid;
    int rc = grid_for(expand_row_idx_kernel, rows, kBlock / 32, &grid);
    return rc ? rc : launch(expand_row_idx_kernel, grid, kBlock, (cudaStream_t)stream, "expand_row_idx_kernel", rowStart, rows, row_idx);
}

int hnh_batch_dot_f64(double *out, const double *A, const double *B, int64_t rows, int r,
                      void *stream) {
    if (rows < 0 || r <= 0) return set_error(HNH_E_INVALID, "hnh_batch_dot_f64: bad size");
    if (rows == 0) return HNH_OK;
    if (!out || !A || !B) return set_error(HNH_E_INVALID, "hnh_batch_dot_f64: null pointer");
    int grid;
    int rc = grid_for(batch_dot_kernel, rows, kBlock / 32, &grid);
    return rc ? rc : launch(batch_dot_kernel, grid, kBlock, (cudaStream_t)stream, "batch_dot_kernel", out, A, B, rows, r);
}

int hnh_row_axpy_f64(double *D, const double *C, double alpha, const double *s, const double *M,
                     int64_t rows, int r, void *stream) {
    if (rows < 0 || r <= 0) return set_error(HNH_E_INVALID, "hnh_row_axpy_f64: bad size");
    const int64_t n = rows * (int64_t)r;
    if (n == 0) return HNH_OK;
    if (!D || !M) return set_error(HNH_E_INVALID, "hnh_row_axpy_f64: null pointer");
    int grid;
    int rc = grid_for(row_axpy_kernel, n, kBlock * 4, &grid);
    return rc ? rc : launch(row_axpy_kernel, grid, kBlock, (cudaStream_t)stream, "row_axpy_kernel", D, C, alpha, s, M, rows, r);
}

int hnh_vec_quotient_f64(double *out, const double *a, double ca, const double *b, double cb,
                         int64_t n, void *stream) {
    if (n < 0) return set_error(HNH_E_INVALID, "hnh_vec_quotient_f64: negative size");
    if (n == 0) return HNH_OK;
    if (!out || !a) return set_error(HNH_E_INVALID, "hnh_vec_quotient_f64: null pointer");
    int grid;
    int rc = grid_for(vec_quotient_kernel, n, kBlock * 4, &grid);
    return rc ? rc : launch(vec_quotient_kernel, grid, kBlock, (cudaStream_t)stream, "vec_quotient_kernel", out, a, ca, b, cb, n);
}

int hnh_axpby_f64(double *dst, double alpha, const double *x, double beta, const double *y,
                  int64_t n, void *stream) {
    if (n < 0) return set_error(HNH_E_INVALID, "hnh_axpby_f64: negative size");
    if (n == 0) return HNH_OK;
    if (!dst || !x) return set_error(HNH_E_INVALID, "hnh_axpby_f64: null pointer");
    int grid;
    int rc = grid_for(axpby_kernel, n, kBlock * 4, &grid);
    return rc ? rc : launch(axpby_kernel, grid, kBlock, (cudaStream_t)stream, "axpby_kernel", dst, alpha, x, beta, y, n);
}

int hnh_squared_norm_f64(double *out, const double *x, int64_t n, void *stream) {
    if (!out) return set_error(HNH_E_INVALID, "hnh_squared_norm_f64: null pointer");
    if (n < 0) return set_error(HNH_E_INVALID, "hnh_squared_norm_f64: negative size");
    cudaStream_t st = (cudaStream_t)stream;
    if (n == 0) return check_cuda(cudaMemsetAsync(out, 0, sizeof(double), st), "cudaMemsetAsync");
    if (!x) return set_error(HNH_E_INVALID, "hnh_squared_norm_f64: null pointer");
    int grid;
    int rc = grid_for(squared_norm_partial_kernel, n, kBlock * 4, &grid);
    if (rc) return rc;
    // per-call scratch, stream-ordered: concurrent calls on different streams never share partials
    double *partial = nullptr;
    rc = check_cuda(cudaMallocAsync((void **)&partial, sizeof(double) * (size_t)grid, st), "cudaMallocAsync");
    if (rc) return rc;
    rc = launch(squared_norm_partial_kernel, grid, kBlock, st, "squared_norm_partial_kernel", partial, x, n);
    if (!rc) rc = launch(sum_partials_kernel, 1, kBlock, st, "sum_partials_kernel", out, partial, grid);
    cudaError_t e = cudaFreeAsync(partial, st);
    return rc ? rc : check_cuda(e, "cudaFreeAsync");
}

// ---- host-buffer block API --------------------------------------------------------------------
struct hnh_block {
    int64_t rows, cols, nnz;
    int r_max;
    int64_t *d_rowStart = nullptr, *d_col = nullptr;
    double *d_vals = nullptr, *d_X = nullptr, *d_Y = nullptr, *d_Out = nullptr;
};

void hnh_block_destroy(hnh_block_t *b) {
    if (!b) return;
    cudaFree(b->d_rowStart);
    cudaFree(b->d_col);
    cudaFree(b->d_vals);
    cudaFree(b->d_X);
    cudaFree(b->d_Y);
    cudaFree(b->d_Out);
    delete b;
}

int hnh_block_create_host(const int64_t *rowStart, const int64_t *col_idx, int64_t rows,
                          int64_t cols, int64_t nnz, int r_max, hnh_block_t **out) {
    if (!out || !rowStart || (nnz > 0 && !col_idx) || rows <= 0 || cols <= 0 || nnz < 0 || r_max <= 0)
        return set_error(HNH_E_INVALID, "hnh_block_create_host: bad argument");
    hnh_block *b = new hnh_block;
    b->rows = rows; b->cols = cols; b->nnz = nnz; b->r_max = r_max;
    const size_t nz = (size_t)(nnz > 0 ? nnz : 1);
    cudaError_t e = cudaSuccess;
    if (e == cudaSuccess) e = cudaMalloc(&b->d_rowStart, sizeof(int64_t) * (size_t)(rows + 1));
    if (e == cudaSuccess) e = cudaMalloc(&b->d_col, sizeof(int64_t) * nz);
    if (e == cudaSuccess) e = cudaMalloc(&b->d_vals, sizeof(double) * nz);
    if (e == cudaSuccess) e = cudaMalloc(&b->d_X, sizeof(double) * (size_t)rows * r_max);
    if (e == cudaSuccess) e = cudaMalloc(&b->d_Y, sizeof(double) * (size_t)cols * r_max);
    if (e == cudaSuccess) e = cudaMalloc(&b->d_Out, sizeof(double) * (size_t)rows * r_max);
    if (e == cudaSuccess)
        e = cudaMemcpy(b->d_rowStart, rowStart, sizeof(int64_t) * (size_t)(rows + 1), cudaMemcpyHostToDevice);
    if (e == cudaSuccess && nnz > 0)
        e = cudaMemcpy(b->d_col, col_idx, sizeof(int64_t) * (size_t)nnz, cudaMemcpyHostToDevice);
    if (e != cudaSuccess) {
        hnh_block_destroy(b);
        return set_error(e == cudaErrorMemoryAllocation ? HNH_E_ALLOC : HNH_E_CUDA,
                         "hnh_block_create_host: %s", cudaGetErrorString(e));
    }
    *out = b;
    return HNH_OK;
}

int hnh_block_run_host(hnh_block_t *b, int op, const double *X, const double *Y, double *values_io,
                       double *Out, int r, int run_flags, void *stream) {
    if (!b || !X || !Y || !values_io || r <= 0 || r > b->r_max || op < 0 || op > 2)
        return set_error(HNH_E_INVALID, "hnh_block_run_host: bad argument");
    if (op >= 1 && !Out) return set_error(HNH_E_INVALID, "hnh_block_run_host: Out is null");
    cudaStream_t st = (cudaStream_t)stream;
    cudaError_t e = cudaSuccess;
    const size_t xb = sizeof(double) * (size_t)b->rows * r, yb = sizeof(double) * (size_t)b->cols * r;
    const size_t vb = sizeof(double) * (size_t)b->nnz;
    // op 1 gathers Y by column and accumulates into Out (rows x r); X is unused there.
    if (op != 1) e = cudaMemcpyAsync(b->d_X, X, xb, cudaMemcpyHostToDevice, st);
    if (e == cudaSuccess) e = cudaMemcpyAsync(b->d_Y, Y, yb, cudaMemcpyHostToDevice, st);
    if (e == cudaSuccess && vb) {
        if (run_flags & HNH_RUN_ZERO_VALUES) e = cudaMemsetAsync(b->d_vals, 0, vb, st);
        else e = cudaMemcpyAsync(b->d_vals, values_io, vb, cudaMemcpyHostToDevice, st);
    }
    if (e == cudaSuccess && op >= 1) {
        if (run_flags & HNH_RUN_ZERO_OUT) e = cudaMemsetAsync(b->d_Out, 0, xb, st);
        else e = cudaMemcpyAsync(b->d_Out, Out, xb, cudaMemcpyHostToDevice, st);
    }
    if (e != cudaSuccess) return check_cuda(e, "hnh_block_run_host H2D");
    int rc = HNH_OK;
    if (op == 0)
        rc = hnh_sddmm_f64(b->d_rowStart, b->d_col, b->d_vals, b->rows, b->nnz, b->d_X, b->d_Y, r, 0, st);
    else if (op == 1)
        rc = hnh_spmm_f64(b->d_rowStart, b->d_col, b->d_vals, b->rows, b->nnz, b->d_Y, b->d_Out, r, 0, st);
    else
        rc = hnh_fused_f64(b->d_rowStart, b->d_col, b->d_vals, b->rows, b->nnz, b->d_X, b->d_Y, b->d_Out, r, 0, st);
    if (rc) return rc;
    if (op != 1 && vb) e = cudaMemcpyAsync(values_io, b->d_vals, vb, cudaMemcpyDeviceToHost, st);
    if (e == cudaSuccess && op >= 1) e = cudaMemcpyAsync(Out, b->d_Out, xb, cudaMemcpyDeviceToHost, st);
    if (e == cudaSuccess) e = cudaStreamSynchronize(st);
    return check_cuda(e, "hnh_block_run_host D2H");
}

}  // extern "C"
