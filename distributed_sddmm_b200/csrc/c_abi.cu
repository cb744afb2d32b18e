// c_abi.cu -- extern "C" layer of libhnh_b200.so: argument validation, kernel selection
// and launch for the entry points declared in include/hnh_b200.h.
#include "hnh_b200.h"
#include "kernels.cuh"
#include "launch.h"

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

// Grid for a grid-stride kernel: a whole number of resident CTAs per SM (multiple of the SM
// count), never more CTAs than there are work items.
template <typename K>
int grid_for(K kernel, int block, int64_t work_items_per_block_capacity, int64_t work_items,
             int *grid_out) {
    int sms = 0;
    int rc = device_sm_count(&sms);
    if (rc) return rc;
    int occ = 0;
    cudaError_t e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kernel, block, 0);
    if (e != cudaSuccess) return check_cuda(e, "cudaOccupancyMaxActiveBlocksPerMultiprocessor");
    if (occ < 1) occ = 1;
    int64_t need = (work_items + work_items_per_block_capacity - 1) / work_items_per_block_capacity;
    int64_t cap = (int64_t)sms * occ;
    int64_t g = need < cap ? need : cap;
    if (g < 1) g = 1;
    *grid_out = (int)g;
    return HNH_OK;
}

static inline bool aligned(const void *p, size_t a) { return ((uintptr_t)p & (a - 1)) == 0; }

constexpr int kBlock = 256;

// ---- templated launchers ------------------------------------------------------------------
template <int R, int G, int VW, int UN>
int launch_sddmm(const int64_t *rowStart, const int64_t *col_idx, double *values, int64_t rows,
                 const double *X, const double *Y, bool beta0, const double *scale, double *scaled_out, bool sv,
                 cudaStream_t st) {
    int grid;
    auto k = beta0 ? sddmm_row_kernel<R, G, VW, UN, true> : sddmm_row_kernel<R, G, VW, UN, false>;
    int rc = grid_for(k, kBlock, kBlock / G, rows, &grid);
    if (rc) return rc;
    k<<<grid, kBlock, 0, st>>>(rowStart, col_idx, values, rows, X, Y, scale, scaled_out, sv);
    count_launch(1);
    return check_cuda(cudaGetLastError(), "sddmm_row_kernel launch");
}
template <int R, int G, int VW, int UN>
int launch_spmm(const int64_t *rowStart, const int64_t *col_idx, const double *values,
                int64_t rows, const double *X, double *Y, bool beta0, cudaStream_t st) {
    int grid;
    auto k = beta0 ? spmm_row_kernel<R, G, VW, UN, true> : spmm_row_kernel<R, G, VW, UN, false>;
    int rc = grid_for(k, kBlock, kBlock / G, rows, &grid);
    if (rc) return rc;
    k<<<grid, kBlock, 0, st>>>(rowStart, col_idx, values, rows, X, Y);
    count_launch(1);
    return check_cuda(cudaGetLastError(), "spmm_row_kernel launch");
}
template <int R, int G, int VW, int UN>
int launch_fused(const int64_t *rowStart, const int64_t *col_idx, double *values, int64_t rows,
                 const double *X, const double *Y, double *Out, bool bv, bool bo, cudaStream_t st,
                 const double *scale = nullptr, double *scaled_out = nullptr) {
    int grid;
    auto k = bv ? (bo ? fused_row_kernel<R, G, VW, UN, true, true> : fused_row_kernel<R, G, VW, UN, true, false>)
                : (bo ? fused_row_kernel<R, G, VW, UN, false, true> : fused_row_kernel<R, G, VW, UN, false, false>);
    if (scale)  // scaled epilogue: first-visit form only (hnh_fused_scaled_f64 checks)
        k = bo ? fused_row_kernel<R, G, VW, UN, true, true, true> : fused_row_kernel<R, G, VW, UN, true, false, true>;
    int rc = grid_for(k, kBlock, kBlock / G, rows, &grid);
    if (rc) return rc;
    k<<<grid, kBlock, 0, st>>>(rowStart, col_idx, values, rows, X, Y, Out, scale, scaled_out);
    count_launch(1);
    return check_cuda(cudaGetLastError(), "fused_row_kernel launch");
}
template <int R, int G, int VW, int UN>
int launch_sddmm_coo(const int64_t *row_idx, const int64_t *col_idx, double *values,
                     int64_t nnz, const double *X, const double *Y, cudaStream_t st) {
    int grid;
    auto k = sddmm_coo_kernel<R, G, VW, UN>;
    int rc = grid_for(k, kBlock, (int64_t)(kBlock / G) * G, nnz, &grid);
    if (rc) return rc;
    k<<<grid, kBlock, 0, st>>>(row_idx, col_idx, values, nnz, X, Y);
    count_launch(1);
    return check_cuda(cudaGetLastError(), "sddmm_coo_kernel launch");
}

// ---- small-r ("split") launchers: G = GK*GN lanes per row ----------------------------------
template <int R, int GK, int GN, int VW, int UN>
int launch_sddmm_split(const int64_t *rowStart, const int64_t *col_idx, double *values,
                       int64_t rows, const double *X, const double *Y, bool beta0, const double *scale, double *scaled_out,
                       bool sv, cudaStream_t st) {
    int grid;
    auto k = beta0 ? sddmm_split_kernel<R, GK, GN, VW, UN, true> : sddmm_split_kernel<R, GK, GN, VW, UN, false>;
    int rc = grid_for(k, kBlock, kBlock / (GK * GN), rows, &grid);
    if (rc) return rc;
    k<<<grid, kBlock, 0, st>>>(rowStart, col_idx, values, rows, X, Y, scale, scaled_out, sv);
    count_launch(1);
    return check_cuda(cudaGetLastError(), "sddmm_split_kernel launch");
}
template <int R, int GK, int GN, int VW, int UN>
int launch_spmm_split(const int64_t *rowStart, const int64_t *col_idx, const double *values,
                      int64_t rows, const double *X, double *Y, bool beta0, cudaStream_t st) {
    int grid;
    auto k = beta0 ? spmm_split_kernel<R, GK, GN, VW, UN, true> : spmm_split_kernel<R, GK, GN, VW, UN, false>;
    int rc = grid_for(k, kBlock, kBlock / (GK * GN), rows, &grid);
    if (rc) return rc;
    k<<<grid, kBlock, 0, st>>>(rowStart, col_idx, values, rows, X, Y);
    count_launch(1);
    return check_cuda(cudaGetLastError(), "spmm_split_kernel launch");
}
template <int R, int GK, int GN, int VW, int UN>
int launch_fused_split(const int64_t *rowStart, const int64_t *col_idx, double *values,
                       int64_t rows, const double *X, const double *Y, double *Out, bool bv, bool bo,
                       cudaStream_t st, const double *scale = nullptr, double *scaled_out = nullptr) {
    int grid;
    auto k = bv ? (bo ? fused_split_kernel<R, GK, GN, VW, UN, true, true> : fused_split_kernel<R, GK, GN, VW, UN, true, false>)
                : (bo ? fused_split_kernel<R, GK, GN, VW, UN, false, true> : fused_split_kernel<R, GK, GN, VW, UN, false, false>);
    if (scale)
        k = bo ? fused_split_kernel<R, GK, GN, VW, UN, true, true, true> : fused_split_kernel<R, GK, GN, VW, UN, true, false, true>;
    int rc = grid_for(k, kBlock, kBlock / (GK * GN), rows, &grid);
    if (rc) return rc;
    k<<<grid, kBlock, 0, st>>>(rowStart, col_idx, values, rows, X, Y, Out, scale, scaled_out);
    count_launch(1);
    return check_cuda(cudaGetLastError(), "fused_split_kernel launch");
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

// ---- TMA-staged launchers (HNH_FLAG_TMA_STAGE; r in {128, 256}, 16-byte aligned operands) -----
template <int R, bool FUSED>
int launch_tma(const int64_t *rowStart, const int64_t *col_idx, double *values, int64_t rows, const double *X,
               const double *Y, double *Out, bool bv, bool bo, cudaStream_t st, const double *scale = nullptr,
               double *scaled_out = nullptr, bool sv = false) {
    int grid;
    auto k = bv ? (bo ? tma_row_kernel<R, 4, FUSED, true, true> : tma_row_kernel<R, 4, FUSED, true, false>)
                : (bo ? tma_row_kernel<R, 4, FUSED, false, true> : tma_row_kernel<R, 4, FUSED, false, false>);
    int rc = grid_for(k, kBlock, 8, rows, &grid);
    if (rc) return rc;
    k<<<grid, kBlock, 0, st>>>(rowStart, col_idx, values, rows, X, Y, Out, scale, scaled_out, sv);
    count_launch(1);
    return check_cuda(cudaGetLastError(), "tma_row_kernel launch");
}
// Default choice between the TMA-staged and the direct-load row kernels: TMA staging for SDDMM at
// r = 128 and 256 and for the overwriting fused kernel at r = 256; the direct kernel for the fused
// kernel at r = 128, where the per-tile barrier makes the 8 warps of a CTA wait for the longest of
// their rows.  HNH_TMA=0 / 1 forces one or the other everywhere.
template <int R, bool FUSED>
int launch_tma_warp(const int64_t *rowStart, const int64_t *col_idx, double *values, int64_t rows, const double *X,
                    const double *Y, double *Out, bool bv, bool bo, cudaStream_t st, const double *scale = nullptr,
                    double *scaled_out = nullptr, bool sv = false) {
    int grid;
    auto k = bv ? (bo ? tma_warp_kernel<R, 4, FUSED, true, true> : tma_warp_kernel<R, 4, FUSED, true, false>)
                : (bo ? tma_warp_kernel<R, 4, FUSED, false, true> : tma_warp_kernel<R, 4, FUSED, false, false>);
    int rc = grid_for(k, kBlock, 8, rows, &grid);
    if (rc) return rc;
    k<<<grid, kBlock, 0, st>>>(rowStart, col_idx, values, rows, X, Y, Out, scale, scaled_out, sv);
    count_launch(1);
    return check_cuda(cudaGetLastError(), "tma_warp_kernel launch");
}

static bool tma_default(bool fused, int r, bool overwrite_out) {
    static int v = -2;
    if (v == -2) {
        const char *e = getenv("HNH_TMA");
        v = e ? (atoi(e) != 0 ? 1 : 0) : -1;
    }
    if (v >= 0) return v == 1;
    return fused ? (r == 256 && overwrite_out) : true;
}

// Shape table: R -> (G lanes per row, VW doubles per vector load, UN rows in flight).
// 128-bit loads (VW=2, the widest on sm_90) need 16-byte aligned operand rows.
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
    int rc = HNH_OK;
    bool beta0 = (flags & HNH_FLAG_BETA0) != 0;
    const bool a16 = aligned(X, 16) && aligned(Y, 16);
#define S4(R, G, VW, UN) rc = launch_sddmm<R, G, VW, UN>(rowStart, col_idx, values, rows, X, Y, beta0, scale, scaled_out, sv, st)
#define SGEN                                                                                 \
    {                                                                                        \
        int grid;                                                                            \
        rc = grid_for(sddmm_generic_kernel, kBlock, kBlock / 32, rows, &grid);               \
        if (!rc) {                                                                           \
            sddmm_generic_kernel<<<grid, kBlock, 0, st>>>(rowStart, col_idx, values, rows, X, \
                                                          Y, r);                             \
            count_launch(1);                                                                 \
            rc = check_cuda(cudaGetLastError(), "sddmm_generic_kernel launch");              \
        }                                                                                    \
    }
    const bool table_r = r == 4 || r == 8 || r == 16 || r == 32 || r == 64 || r == 128 || r == 256;
    // The epilogue form needs a table kernel and distinct arrays (scale is read through the read-only path); otherwise
    // the product is one more elementwise pass after the plain SDDMM.
    if (scale && ((flags & HNH_FLAG_FORCE_GENERIC) || !a16 || !table_r || (const double *)scaled_out == scale || values == scale)) {
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
    if ((flags & HNH_FLAG_TMA_WARP) && a16 && (r == 128 || r == 256) && !(flags & HNH_FLAG_FORCE_GENERIC)) {
        return r == 128 ? launch_tma_warp<128, false>(rowStart, col_idx, values, rows, X, Y, nullptr, beta0, false, st, scale, scaled_out, sv)
                        : launch_tma_warp<256, false>(rowStart, col_idx, values, rows, X, Y, nullptr, beta0, false, st, scale, scaled_out, sv);
    }
    if (((flags & HNH_FLAG_TMA_STAGE) || (tma_default(false, r, beta0) && !(flags & HNH_FLAG_FORCE_DIRECT))) && a16 &&
        (r == 128 || r == 256) && !(flags & HNH_FLAG_FORCE_GENERIC)) {
        return r == 128 ? launch_tma<128, false>(rowStart, col_idx, values, rows, X, Y, nullptr, beta0, false, st, scale, scaled_out, sv)
                        : launch_tma<256, false>(rowStart, col_idx, values, rows, X, Y, nullptr, beta0, false, st, scale, scaled_out, sv);
    }
    if ((flags & HNH_FLAG_FORCE_GENERIC) || !a16 || !table_r) {
        if (beta0) {  // the any-r kernel accumulates: clear first
            rc = check_cuda(cudaMemsetAsync(values, 0, sizeof(double) * (size_t)nnz, st), "cudaMemsetAsync");
            if (rc) return rc;
        }
        SGEN
    } else if (r <= split_max_r() && r <= 32) {
#define SP(R, GK, GN, VW, UN) \
    rc = launch_sddmm_split<R, GK, GN, VW, UN>(rowStart, col_idx, values, rows, X, Y, beta0, scale, scaled_out, sv, st)
        HNH_DISPATCH_SPLIT(r, SP)
#undef SP
    } else {
        HNH_DISPATCH_R(r, S4, SGEN)
    }
#undef S4
#undef SGEN
    return rc;
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
    int rc = HNH_OK;
    const bool a16 = aligned(X, 16) && aligned(Y, 16);
#define S4(R, G, VW, UN) rc = launch_sddmm_coo<R, G, VW, (UN > 2 ? 2 : UN)>(row_idx, col_idx, values, nnz, X, Y, st)
#define SGEN                                                                                    \
    {                                                                                           \
        int grid;                                                                               \
        rc = grid_for(sddmm_coo_generic_kernel, kBlock, kBlock / 32, nnz, &grid);               \
        if (!rc) {                                                                              \
            sddmm_coo_generic_kernel<<<grid, kBlock, 0, st>>>(row_idx, col_idx, values, nnz, X, \
                                                              Y, r);                            \
            count_launch(1);                                                                    \
            rc = check_cuda(cudaGetLastError(), "sddmm_coo_generic_kernel launch");             \
        }                                                                                       \
    }
    if ((flags & HNH_FLAG_FORCE_GENERIC) || !a16) {
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
    int rc = HNH_OK;
    bool beta0 = (flags & HNH_FLAG_BETA0) != 0;
    const bool a16 = aligned(X, 16) && aligned(Y, 16);
#define S4(R, G, VW, UN) rc = launch_spmm<R, G, VW, UN>(rowStart, col_idx, values, rows, X, Y, beta0, st)
#define SGEN                                                                                \
    {                                                                                       \
        int grid;                                                                           \
        rc = grid_for(spmm_generic_kernel, kBlock, kBlock / 32, rows, &grid);               \
        if (!rc) {                                                                          \
            spmm_generic_kernel<<<grid, kBlock, 0, st>>>(rowStart, col_idx, values, rows, X, \
                                                         Y, r);                             \
            count_launch(1);                                                                \
            rc = check_cuda(cudaGetLastError(), "spmm_generic_kernel launch");              \
        }                                                                                   \
    }
    const bool table_r = r == 4 || r == 8 || r == 16 || r == 32 || r == 64 || r == 128 || r == 256;
    if ((flags & HNH_FLAG_FORCE_GENERIC) || !a16 || !table_r) {
        if (beta0) {
            rc = check_cuda(cudaMemsetAsync(Y, 0, sizeof(double) * (size_t)rows * r, st), "cudaMemsetAsync");
            if (rc) return rc;
        }
        SGEN
    } else if (r <= split_max_r() && r <= 32) {
#define SP(R, GK, GN, VW, UN) \
    rc = launch_spmm_split<R, GK, GN, VW, UN>(rowStart, col_idx, values, rows, X, Y, beta0, st)
        HNH_DISPATCH_SPLIT(r, SP)
#undef SP
    } else {
        HNH_DISPATCH_R(r, S4, SGEN)
    }
#undef S4
#undef SGEN
    return rc;
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
    int rc = HNH_OK;
    const bool bv = (flags & (HNH_FLAG_BETA0 | HNH_FLAG_BETA0_VALUES)) != 0;
    const bool bo = (flags & (HNH_FLAG_BETA0 | HNH_FLAG_BETA0_OUT)) != 0;
    if (X == Out && !bo)
        return set_error(HNH_E_INVALID, "hnh_fused_f64: Out may alias X only when Out is overwritten (BETA0_OUT)");
    const bool a16 = aligned(X, 16) && aligned(Y, 16) && aligned(Out, 16);
#define S4(R, G, VW, UN) \
    rc = launch_fused<R, G, VW, UN>(rowStart, col_idx, values, rows, X, Y, Out, bv, bo, st, scale, scaled_out)
#define SGEN                                                                                 \
    {                                                                                        \
        int grid;                                                                            \
        rc = grid_for(fused_generic_kernel, kBlock, kBlock / 32, rows, &grid);               \
        if (!rc) {                                                                           \
            fused_generic_kernel<<<grid, kBlock, 0, st>>>(rowStart, col_idx, values, rows, X, \
                                                          Y, Out, r);                        \
            count_launch(1);                                                                 \
            rc = check_cuda(cudaGetLastError(), "fused_generic_kernel launch");              \
        }                                                                                    \
    }
    const bool table_r = r == 4 || r == 8 || r == 16 || r == 32 || r == 64 || r == 128 || r == 256;
    if (scale) {
        // the scaled epilogue exists in the first-visit form of the direct-load table kernels only
        if (!bv) return set_error(HNH_E_INVALID, "hnh_fused_scaled_f64: scale needs HNH_FLAG_BETA0_VALUES");
        if (!a16 || !table_r || (flags & HNH_FLAG_FORCE_GENERIC))
            return set_error(HNH_E_INVALID, "hnh_fused_scaled_f64: scale needs a table width (4..256, power of two) and 16-byte "
                                            "aligned operands");
        if (values == scale || (const double *)scaled_out == scale)
            return set_error(HNH_E_INVALID, "hnh_fused_scaled_f64: scale must not alias values / scaled_out");
        flags = (flags | HNH_FLAG_FORCE_DIRECT) & ~(HNH_FLAG_TMA_STAGE | HNH_FLAG_TMA_WARP);
    }
    // in place (Out == X) is not offered with TMA staging: the next tile of X is prefetched while
    // the current one is still being written
    if ((flags & HNH_FLAG_TMA_WARP) && a16 && (r == 128 || r == 256) && X != Out && !(flags & HNH_FLAG_FORCE_GENERIC)) {
        return r == 128 ? launch_tma_warp<128, true>(rowStart, col_idx, values, rows, X, Y, Out, bv, bo, st)
                        : launch_tma_warp<256, true>(rowStart, col_idx, values, rows, X, Y, Out, bv, bo, st);
    }
    if (((flags & HNH_FLAG_TMA_STAGE) || (tma_default(true, r, bo) && !(flags & HNH_FLAG_FORCE_DIRECT))) && a16 &&
        (r == 128 || r == 256) && X != Out && !(flags & HNH_FLAG_FORCE_GENERIC)) {
        return r == 128 ? launch_tma<128, true>(rowStart, col_idx, values, rows, X, Y, Out, bv, bo, st)
                        : launch_tma<256, true>(rowStart, col_idx, values, rows, X, Y, Out, bv, bo, st);
    }
    if ((flags & HNH_FLAG_FORCE_GENERIC) || !a16 || !table_r) {
        if (X == Out)
            return set_error(HNH_E_INVALID, "hnh_fused_f64: in-place (Out == X) needs a table r "
                                            "(4..256, power of two) and 16-byte aligned operands");
        if (bv) rc = check_cuda(cudaMemsetAsync(values, 0, sizeof(double) * (size_t)nnz, st), "cudaMemsetAsync");
        if (!rc && bo) rc = check_cuda(cudaMemsetAsync(Out, 0, sizeof(double) * (size_t)rows * r, st), "cudaMemsetAsync");
        if (rc) return rc;
        SGEN
    } else if (r <= split_max_r() && r <= 32) {
#define SP(R, GK, GN, VW, UN) \
    rc = launch_fused_split<R, GK, GN, VW, UN>(rowStart, col_idx, values, rows, X, Y, Out, bv, bo, st, scale, scaled_out)
        HNH_DISPATCH_SPLIT(r, SP)
#undef SP
    } else {
        HNH_DISPATCH_R(r, S4, SGEN)
    }
#undef S4
#undef SGEN
    return rc;
}

int hnh_fused_f64(const int64_t *rowStart, const int64_t *col_idx, double *values, int64_t rows,
                  int64_t nnz, const double *X, const double *Y, double *Out, int r, int flags,
                  void *stream) {
    return hnh_fused_scaled_f64(rowStart, col_idx, values, rows, nnz, X, Y, Out, r, flags, nullptr, nullptr, stream);
}

// ---- K4 + row algebra -----------------------------------------------------------------------
#define HNH_ELEMENTWISE_LAUNCH(kernel, n, ...)                                       \
    do {                                                                             \
        if ((n) < 0) return set_error(HNH_E_INVALID, #kernel ": negative size");     \
        if ((n) == 0) return HNH_OK;                                                 \
        int grid;                                                                    \
        int rc_ = grid_for(kernel, kBlock, kBlock * 4, (n), &grid);                  \
        if (rc_) return rc_;                                                         \
        kernel<<<grid, kBlock, 0, (cudaStream_t)stream>>>(__VA_ARGS__);              \
        count_launch(1);                                                             \
        return check_cuda(cudaGetLastError(), #kernel " launch");                    \
    } while (0)

int hnh_fill_f64(double *dst, int64_t n, double value, void *stream) {
    if (n > 0 && !dst) return set_error(HNH_E_INVALID, "hnh_fill_f64: null pointer");
    if (n > 0 && value == 0.0)
        return check_cuda(cudaMemsetAsync(dst, 0, sizeof(double) * (size_t)n, (cudaStream_t)stream),
                          "cudaMemsetAsync");
    HNH_ELEMENTWISE_LAUNCH(fill_kernel, n, dst, n, value);
}

int hnh_random_uniform_f64(double *dst, int64_t n, uint64_t seed, void *stream) {
    if (n > 0 && !dst) return set_error(HNH_E_INVALID, "hnh_random_uniform_f64: null pointer");
    HNH_ELEMENTWISE_LAUNCH(random_uniform_kernel, n, dst, n, seed);
}

int hnh_hadamard_f64(double *dst, const double *a, const double *b, int64_t n, void *stream) {
    if (n > 0 && (!dst || !a || !b)) return set_error(HNH_E_INVALID, "hnh_hadamard_f64: null pointer");
    HNH_ELEMENTWISE_LAUNCH(hadamard_kernel, n, dst, a, b, n);
}

int hnh_expand_row_idx(const int64_t *rowStart, int64_t rows, int64_t nnz, int64_t *row_idx,
                       void *stream) {
    if (rows < 0 || nnz < 0) return set_error(HNH_E_INVALID, "hnh_expand_row_idx: negative size");
    if (rows == 0 || nnz == 0) return HNH_OK;
    if (!rowStart || !row_idx) return set_error(HNH_E_INVALID, "hnh_expand_row_idx: null pointer");
    int grid;
    int rc = grid_for(expand_row_idx_kernel, kBlock, kBlock / 32, rows, &grid);
    if (rc) return rc;
    expand_row_idx_kernel<<<grid, kBlock, 0, (cudaStream_t)stream>>>(rowStart, rows, row_idx);
    count_launch(1);
    return check_cuda(cudaGetLastError(), "expand_row_idx_kernel launch");
}

int hnh_batch_dot_f64(double *out, const double *A, const double *B, int64_t rows, int r,
                      void *stream) {
    if (rows < 0 || r <= 0) return set_error(HNH_E_INVALID, "hnh_batch_dot_f64: bad size");
    if (rows == 0) return HNH_OK;
    if (!out || !A || !B) return set_error(HNH_E_INVALID, "hnh_batch_dot_f64: null pointer");
    int grid;
    int rc = grid_for(batch_dot_kernel, kBlock, kBlock / 32, rows, &grid);
    if (rc) return rc;
    batch_dot_kernel<<<grid, kBlock, 0, (cudaStream_t)stream>>>(out, A, B, rows, r);
    count_launch(1);
    return check_cuda(cudaGetLastError(), "batch_dot_kernel launch");
}

int hnh_row_axpy_f64(double *D, const double *C, double alpha, const double *s, const double *M,
                     int64_t rows, int r, void *stream) {
    if (rows < 0 || r <= 0) return set_error(HNH_E_INVALID, "hnh_row_axpy_f64: bad size");
    const int64_t n = rows * (int64_t)r;
    if (n > 0 && (!D || !M)) return set_error(HNH_E_INVALID, "hnh_row_axpy_f64: null pointer");
    HNH_ELEMENTWISE_LAUNCH(row_axpy_kernel, n, D, C, alpha, s, M, rows, r);
}

int hnh_vec_quotient_f64(double *out, const double *a, double ca, const double *b, double cb,
                         int64_t n, void *stream) {
    if (n > 0 && (!out || !a)) return set_error(HNH_E_INVALID, "hnh_vec_quotient_f64: null pointer");
    HNH_ELEMENTWISE_LAUNCH(vec_quotient_kernel, n, out, a, ca, b, cb, n);
}

int hnh_axpby_f64(double *dst, double alpha, const double *x, double beta, const double *y,
                  int64_t n, void *stream) {
    if (n > 0 && (!dst || !x)) return set_error(HNH_E_INVALID, "hnh_axpby_f64: null pointer");
    HNH_ELEMENTWISE_LAUNCH(axpby_kernel, n, dst, alpha, x, beta, y, n);
}

int hnh_squared_norm_f64(double *out, const double *x, int64_t n, void *stream) {
    if (!out) return set_error(HNH_E_INVALID, "hnh_squared_norm_f64: null pointer");
    if (n < 0) return set_error(HNH_E_INVALID, "hnh_squared_norm_f64: negative size");
    cudaStream_t st = (cudaStream_t)stream;
    if (n == 0) return check_cuda(cudaMemsetAsync(out, 0, sizeof(double), st), "cudaMemsetAsync");
    if (!x) return set_error(HNH_E_INVALID, "hnh_squared_norm_f64: null pointer");
    int grid;
    int rc = grid_for(squared_norm_partial_kernel, kBlock, kBlock * 4, n, &grid);
    if (rc) return rc;
    // per-call scratch, stream-ordered: concurrent calls on different streams never share partials
    double *partial = nullptr;
    rc = check_cuda(cudaMallocAsync((void **)&partial, sizeof(double) * (size_t)grid, st), "cudaMallocAsync");
    if (rc) return rc;
    squared_norm_partial_kernel<<<grid, kBlock, 0, st>>>(partial, x, n);
    sum_partials_kernel<<<1, kBlock, 0, st>>>(out, partial, grid);
    count_launch(2);
    rc = check_cuda(cudaGetLastError(), "squared_norm launch");
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
