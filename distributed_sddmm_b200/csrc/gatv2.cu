// gatv2.cu -- the two sparse gathers of GATv2 attention (GAT::set_attention("gatv2"); Brody, Alon and Yahav 2022) on
// one CSR block.  With sigma = LeakyReLU(., alpha), R the row-side operand (indexed by the stored row) and Y the
// gathered side (indexed by col_idx), each row-major with its own leading dimension:
//     out[i]  = sum_k a[k] sigma(R[row(i), k] + Y[col_idx[i], k])                         (gatv2_scores_kernel)
//     dR[row] += a o sum_{i in row} g[i] sigma'(R[row] + Y[col_idx[i]])                   (gatv2_grad_kernel)
//     da      += sum_i g[i] sigma(R[row(i)] + Y[col_idx[i]])     per-CTA partials, then gatv2_da_reduce_kernel
// sigma'(z) = 1 where z > 0 and alpha elsewhere (hnh_leaky_relu_grad_f64's convention).
//
// The fast kernels follow the row kernels of kernels.cuh: a group of G lanes owns one CSR row and keeps R[row] and a
// in registers; a chunk of G (col, g) pairs is read coalesced and broadcast by shuffles; gathered Y rows come in with
// 128-bit loads, UN rows in flight per lane.  The score of an entry ends in the group's xor-butterfly; the gradient
// row is accumulated in registers and read-modify-written once.  The grid is capped at the resident CTAs and walked
// with a grid-stride loop.  Widths 4..256 (powers of two) with 16-byte aligned operands and even leading dimensions
// take these; every other case (any r >= 1, any leading dimension, any alignment) takes the one-warp-per-row generic
// kernels.  No floating-point atomics: two calls on the same device give bit-identical results.
#include "row_gather.cuh"

namespace {

using hnh::grid_for;
using hnh::kResident;
using hnh::launch;
using hnh::set_error;

// most CTAs a gradient launch uses (the da workspace holds one r-wide partial per CTA)
constexpr int64_t kMaxGradCtas = 2048;

__device__ __forceinline__ double leaky(double z, double alpha) { return z > 0.0 ? z : alpha * z; }
__device__ __forceinline__ double leaky_grad(double z, double alpha) { return z > 0.0 ? 1.0 : alpha; }

// ---- fast row kernels ----------------------------------------------------------------------------------------
template <int R, int G, int VW, int UN>
__global__ void __launch_bounds__(kBlock, 1)
gatv2_scores_kernel(const int64_t *__restrict__ rowStart, const int64_t *__restrict__ col_idx, int64_t rows,
                    const double *__restrict__ X, int64_t ldx, const double *__restrict__ Y, int64_t ldy,
                    const double *__restrict__ a, double alpha, double *__restrict__ out) {
    constexpr int NV = R / (G * VW);
    static_assert(NV * G * VW == R, "R must equal NV*G*VW");
    const int lane = threadIdx.x & 31;
    const int gl = lane & (G - 1);
    const unsigned gmask = group_mask<G>(lane);
    const int64_t ngroups = (int64_t)gridDim.x * (blockDim.x / G);
    double av[NV][VW];
#pragma unroll
    for (int v = 0; v < NV; v++) ld_gather<VW>(av[v], a + (v * G + gl) * VW);
    for (int64_t row = (int64_t)blockIdx.x * (blockDim.x / G) + threadIdx.x / G; row < rows; row += ngroups) {
        const int64_t s = ld_stream_i64(rowStart + row);
        const int64_t e = ld_stream_i64(rowStart + row + 1);
        if (s == e) continue;
        double x[NV][VW];
#pragma unroll
        for (int v = 0; v < NV; v++) ld_gather<VW>(x[v], X + row * ldx + (v * G + gl) * VW);
        for (int64_t j = s; j < e; j += G) {
            const int cnt = (e - j < G) ? (int)(e - j) : G;
            int64_t mycol = 0;
            if (gl < cnt) mycol = ld_stream_i64(col_idx + j + gl);
            double mine = 0.0;
            for (int k0 = 0; k0 < cnt; k0 += UN) {
                double y[UN][NV][VW];
#pragma unroll
                for (int u = 0; u < UN; u++) {
                    const int k = k0 + u;
                    const int64_t c = __shfl_sync(gmask, mycol, k < G ? k : G - 1, G);
                    if (k < cnt) {
#pragma unroll
                        for (int v = 0; v < NV; v++) ld_gather<VW>(y[u][v], Y + c * ldy + (v * G + gl) * VW);
                    } else {
#pragma unroll
                        for (int v = 0; v < NV; v++)
#pragma unroll
                            for (int w = 0; w < VW; w++) y[u][v][w] = 0.0;
                    }
                }
#pragma unroll
                for (int u = 0; u < UN; u++) {
                    double d = 0.0;
#pragma unroll
                    for (int v = 0; v < NV; v++)
#pragma unroll
                        for (int w = 0; w < VW; w++) d = fma(av[v][w], leaky(x[v][w] + y[u][v][w], alpha), d);
                    d = group_allreduce<G>(d, gmask);
                    if (gl == k0 + u) mine = d;
                }
            }
            if (gl < cnt) out[j + gl] = mine;
        }
    }
}

// DA: also the CTA's partial of da, written to part[blockIdx.x * R ..]: each group sums its rows in registers, then
// the groups are added in group order through shared memory
template <int R, int G, int VW, int UN, bool DA>
__global__ void __launch_bounds__(kBlock, 1)
gatv2_grad_kernel(const int64_t *__restrict__ rowStart, const int64_t *__restrict__ col_idx, const double *__restrict__ g,
                  int64_t rows, const double *__restrict__ X, int64_t ldx, const double *__restrict__ Y, int64_t ldy,
                  const double *__restrict__ a, double alpha, double *__restrict__ dX, int64_t lddx,
                  double *__restrict__ part) {
    constexpr int NV = R / (G * VW);
    static_assert(NV * G * VW == R, "R must equal NV*G*VW");
    constexpr int kGroups = kBlock / G;
    __shared__ double sh[DA ? kGroups * R : 1];
    const int lane = threadIdx.x & 31;
    const int gl = lane & (G - 1);
    const unsigned gmask = group_mask<G>(lane);
    const int64_t ngroups = (int64_t)gridDim.x * kGroups;
    double av[NV][VW], da[NV][VW];
#pragma unroll
    for (int v = 0; v < NV; v++) {
        ld_gather<VW>(av[v], a + (v * G + gl) * VW);
#pragma unroll
        for (int w = 0; w < VW; w++) da[v][w] = 0.0;
    }
    for (int64_t row = (int64_t)blockIdx.x * kGroups + threadIdx.x / G; row < rows; row += ngroups) {
        const int64_t s = ld_stream_i64(rowStart + row);
        const int64_t e = ld_stream_i64(rowStart + row + 1);
        if (s == e) continue;  // dX[row] += 0
        double x[NV][VW], acc[NV][VW];
#pragma unroll
        for (int v = 0; v < NV; v++) {
            ld_gather<VW>(x[v], X + row * ldx + (v * G + gl) * VW);
#pragma unroll
            for (int w = 0; w < VW; w++) acc[v][w] = 0.0;
        }
        for (int64_t j = s; j < e; j += G) {
            const int cnt = (e - j < G) ? (int)(e - j) : G;
            int64_t mycol = 0;
            double myg = 0.0;
            if (gl < cnt) {
                mycol = ld_stream_i64(col_idx + j + gl);
                myg = ld_stream_f64(g + j + gl);
            }
            for (int k0 = 0; k0 < cnt; k0 += UN) {
                double y[UN][NV][VW];
                double gv[UN];
#pragma unroll
                for (int u = 0; u < UN; u++) {
                    const int k = k0 + u;
                    const int src = k < G ? k : G - 1;
                    const int64_t c = __shfl_sync(gmask, mycol, src, G);
                    gv[u] = __shfl_sync(gmask, myg, src, G);
                    if (k < cnt) {
#pragma unroll
                        for (int v = 0; v < NV; v++) ld_gather<VW>(y[u][v], Y + c * ldy + (v * G + gl) * VW);
                    }
                }
#pragma unroll
                for (int u = 0; u < UN; u++) {
                    if (k0 + u < cnt) {
#pragma unroll
                        for (int v = 0; v < NV; v++)
#pragma unroll
                            for (int w = 0; w < VW; w++) {
                                const double z = x[v][w] + y[u][v][w];
                                acc[v][w] = fma(gv[u], leaky_grad(z, alpha), acc[v][w]);
                                if (DA) da[v][w] = fma(gv[u], leaky(z, alpha), da[v][w]);
                            }
                    }
                }
            }
        }
#pragma unroll
        for (int v = 0; v < NV; v++) {
            double o[VW];
            double *p = dX + row * lddx + (v * G + gl) * VW;
            ld_rw<VW>(o, p);
#pragma unroll
            for (int w = 0; w < VW; w++) o[w] = fma(av[v][w], acc[v][w], o[w]);
            st_rw<VW>(p, o);
        }
    }
    if (DA) {
        const int grp = threadIdx.x / G;
#pragma unroll
        for (int v = 0; v < NV; v++)
#pragma unroll
            for (int w = 0; w < VW; w++) sh[grp * R + (v * G + gl) * VW + w] = da[v][w];
        __syncthreads();
        for (int k = threadIdx.x; k < R; k += kBlock) {
            double t = sh[k];
            for (int q = 1; q < kGroups; q++) t += sh[q * R + k];
            part[(int64_t)blockIdx.x * R + k] = t;
        }
    }
}

// ---- generic kernels: any r, any leading dimension, any alignment; one warp per row ---------------------------
__global__ void __launch_bounds__(kBlock)
gatv2_scores_generic_kernel(const int64_t *__restrict__ rowStart, const int64_t *__restrict__ col_idx, int64_t rows,
                            const double *__restrict__ X, int64_t ldx, const double *__restrict__ Y, int64_t ldy,
                            const double *__restrict__ a, int r, double alpha, double *__restrict__ out) {
    const int lane = threadIdx.x & 31;
    const int64_t warps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t row = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; row < rows; row += warps) {
        const int64_t s = rowStart[row], e = rowStart[row + 1];
        for (int64_t j = s; j < e; j++) {
            const int64_t c = col_idx[j];
            double d = 0.0;
            for (int k = lane; k < r; k += 32) d = fma(a[k], leaky(X[row * ldx + k] + Y[c * ldy + k], alpha), d);
            d = group_allreduce<32>(d, 0xffffffffu);
            if (lane == 0) out[j] = d;
        }
    }
}

// Columns are taken 32 at a time (lane k of the warp owns column k0 + k), each a sweep over the warp's rows, so that
// a lane's share of da is one register.  part: as gatv2_grad_kernel (r doubles per CTA), when not null.
__global__ void __launch_bounds__(kBlock)
gatv2_grad_generic_kernel(const int64_t *__restrict__ rowStart, const int64_t *__restrict__ col_idx,
                          const double *__restrict__ g, int64_t rows, const double *__restrict__ X, int64_t ldx,
                          const double *__restrict__ Y, int64_t ldy, const double *__restrict__ a, int r, double alpha,
                          double *__restrict__ dX, int64_t lddx, double *__restrict__ part) {
    constexpr int kWarps = kBlock / 32;
    __shared__ double sh[kWarps][32];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int64_t warps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int k0 = 0; k0 < r; k0 += 32) {
        const int k = k0 + lane;
        const bool mine = k < r;
        const double ak = mine ? a[k] : 0.0;
        double da = 0.0;
        for (int64_t row = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; row < rows; row += warps) {
            const int64_t s = rowStart[row], e = rowStart[row + 1];
            if (s == e || !mine) continue;
            const double xk = X[row * ldx + k];
            double acc = 0.0;
            for (int64_t j = s; j < e; j++) {
                const double gj = g[j];
                const double z = xk + Y[col_idx[j] * ldy + k];
                acc = fma(gj, leaky_grad(z, alpha), acc);
                da = fma(gj, leaky(z, alpha), da);
            }
            dX[row * lddx + k] = fma(ak, acc, dX[row * lddx + k]);
        }
        if (part != nullptr) {
            sh[warp][lane] = da;
            __syncthreads();
            if (warp == 0) {
                double t = sh[0][lane];
                for (int q = 1; q < kWarps; q++) t += sh[q][lane];
                if (mine) part[(int64_t)blockIdx.x * r + k] = t;
            }
            __syncthreads();
        }
    }
}

// da[k] += sum over CTAs q = 0 .. ctas - 1 of part[q * r + k], always in that order
__global__ void gatv2_da_reduce_kernel(double *__restrict__ da, const double *__restrict__ part, int64_t ctas, int r) {
    for (int k = blockIdx.x * blockDim.x + threadIdx.x; k < r; k += gridDim.x * blockDim.x) {
        double t = part[k];
        for (int64_t q = 1; q < ctas; q++) t += part[q * r + k];
        da[k] += t;
    }
}

int check_block(const char *who, const int64_t *rowStart, const int64_t *col_idx, int64_t rows, int64_t nnz,
                const double *X, int64_t ldx, const double *Y, int64_t ldy, const double *a, int r) {
    if (rows < 0 || nnz < 0) return set_error(HNH_E_INVALID, "%s: negative size", who);
    if (r < 1) return set_error(HNH_E_INVALID, "%s: r must be positive (got %d)", who, r);
    if (ldx < r || ldy < r)
        return set_error(HNH_E_INVALID, "%s: leading dimensions %lld and %lld below r = %d", who, (long long)ldx,
                         (long long)ldy, r);
    if (rows == 0 || nnz == 0) return 1;  // successful no-op
    if (!rowStart || !col_idx || !X || !Y || !a) return set_error(HNH_E_INVALID, "%s: null pointer", who);
    return HNH_OK;
}

}  // namespace

extern "C" {

int hnh_gatv2_scores_f64(const int64_t *rowStart, const int64_t *col_idx, int64_t rows, int64_t nnz, const double *R,
                         int64_t ldr, const double *Y, int64_t ldy, const double *a, int r, double alpha, double *out,
                         void *stream) {
    int v = check_block("hnh_gatv2_scores_f64", rowStart, col_idx, rows, nnz, R, ldr, Y, ldy, a, r);
    if (v < 0) return v;
    if (v == 1) return HNH_OK;
    if (!out) return set_error(HNH_E_INVALID, "hnh_gatv2_scores_f64: null pointer");
    cudaStream_t st = (cudaStream_t)stream;
    int grid = 0, rc = HNH_OK;
    if (table_width(r) && aligned16(R) && aligned16(Y) && aligned16(a) && ldr % 2 == 0 && ldy % 2 == 0) {
#define SC(RR, G, VW, UN)                                                                                                  \
    {                                                                                                                      \
        auto k = gatv2_scores_kernel<RR, G, VW, UN>;                                                                       \
        rc = grid_for(k, rows, kBlock / G, &grid);                                                                         \
        if (!rc) rc = launch(k, grid, kBlock, st, "gatv2_scores_kernel", rowStart, col_idx, rows, R, ldr, Y, ldy, a, alpha, out); \
    }
        HNH_DISPATCH_R(r, SC, )
#undef SC
        return rc;
    }
    rc = grid_for(gatv2_scores_generic_kernel, rows, kBlock / 32, &grid);
    return rc ? rc : launch(gatv2_scores_generic_kernel, grid, kBlock, st, "gatv2_scores_generic_kernel", rowStart, col_idx, rows, R, ldr,
                            Y, ldy, a, r, alpha, out);
}

int64_t hnh_gatv2_grad_workspace_bytes(int64_t rows, int r) {
    if (rows < 0 || r < 1)
        return set_error(HNH_E_INVALID, "hnh_gatv2_grad_workspace_bytes: bad shape %lld x %d", (long long)rows, r);
    return std::min<int64_t>(rows, kMaxGradCtas) * r * (int64_t)sizeof(double);
}

int hnh_gatv2_grad_f64(const int64_t *rowStart, const int64_t *col_idx, const double *g, int64_t rows, int64_t nnz,
                       const double *R, int64_t ldr, const double *Y, int64_t ldy, const double *a, int r, double alpha,
                       double *dR, int64_t lddr, double *da, void *workspace, size_t workspace_bytes, void *stream) {
    int v = check_block("hnh_gatv2_grad_f64", rowStart, col_idx, rows, nnz, R, ldr, Y, ldy, a, r);
    if (v < 0) return v;
    if (lddr < r) return set_error(HNH_E_INVALID, "hnh_gatv2_grad_f64: leading dimension %lld of dR below r = %d", (long long)lddr, r);
    if (v == 1) return HNH_OK;
    if (!g || !dR) return set_error(HNH_E_INVALID, "hnh_gatv2_grad_f64: null pointer");
    const int64_t need = hnh_gatv2_grad_workspace_bytes(rows, r);
    if (da && (!workspace || workspace_bytes < (size_t)need))
        return set_error(HNH_E_INVALID, "hnh_gatv2_grad_f64: workspace of %zu bytes, %lld needed", workspace_bytes, (long long)need);
    cudaStream_t st = (cudaStream_t)stream;
    double *part = da ? (double *)workspace : nullptr;
    int ctas = 0, rc = HNH_OK;
    if (table_width(r) && aligned16(R) && aligned16(Y) && aligned16(a) && aligned16(dR) && ldr % 2 == 0 && ldy % 2 == 0 &&
        lddr % 2 == 0) {
#define GR(RR, G, VW, UN)                                                                                                  \
    {                                                                                                                      \
        auto k = part ? gatv2_grad_kernel<RR, G, VW, UN, true> : gatv2_grad_kernel<RR, G, VW, UN, false>;                  \
        rc = grid_for(k, rows, kBlock / G, &ctas, kResident, kMaxGradCtas);                                                \
        if (!rc)                                                                                                           \
            rc = launch(k, ctas, kBlock, st, "gatv2_grad_kernel", rowStart, col_idx, g, rows, R, ldr, Y, ldy, a, alpha, dR, lddr, part); \
    }
        HNH_DISPATCH_R(r, GR, )
#undef GR
    } else {
        rc = grid_for(gatv2_grad_generic_kernel, rows, kBlock / 32, &ctas, kResident, kMaxGradCtas);
        if (!rc)
            rc = launch(gatv2_grad_generic_kernel, ctas, kBlock, st, "gatv2_grad_generic_kernel", rowStart, col_idx, g, rows, R, ldr, Y,
                        ldy, a, r, alpha, dR, lddr, part);
    }
    if (rc || !da) return rc;
    return launch(gatv2_da_reduce_kernel, (r + kBlock - 1) / kBlock, kBlock, st, "gatv2_da_reduce_kernel", da, part, ctas, r);
}

}  // extern "C"
