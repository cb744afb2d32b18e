// link_prediction.cu -- the dot-product edge decoder of link prediction (Distributed_Sparse::linkLoss,
// include/hnh/training.hpp) on one CSR block.  With X the row side (indexed by the stored row u), Y the gathered side
// (indexed by col_idx v), each row-major with its own leading dimension, and the block's values y_uv the targets:
//     s_uv  = <X_u, Y_v>                                        scores[i]           (nullable: not written)
//     l_uv  = max(s, 0) - s y + log1p(exp(-|s|))                binary cross-entropy with logits, stable for any finite s
//     c_uv  = [(s > 0) == (y > 0.5)]
//     g_uv  = (sigmoid(s) - y) inv_count
//     dX_u += sum_v g_uv Y_v                                    (nullable)
//     stats[u, 0] += sum_v l_uv,  stats[u, 1] += sum_v c_uv     (nullable; leading dimension lds)
// The fast kernel follows the row kernels of gatv2.cu: a group of G lanes owns one CSR row and keeps X_u in registers;
// a chunk of G (col, y) pairs is read coalesced and broadcast by shuffles; gathered Y rows come in with 128-bit loads,
// UN rows in flight per lane.  The score ends in the group's xor-butterfly, so every lane of the group holds its bits;
// the epilogue (exp, log1p, a division) of a batch of UN entries runs once, entry u on lane u, and g comes back by
// shuffle.  g Y_v accumulates in registers in stored order, the row's loss and count per lane, and dX
// and stats are read, modified and written once at the row end (the operand they live in may ride a ring and
// accumulate across ring steps).  Widths 4..256 (powers of two) with 16-byte aligned operands and even leading
// dimensions take it; every other case takes the one-warp-per-row generic kernel.  No atomics anywhere: repeated calls
// are bit-identical.
#include <cmath>

#include "row_gather.cuh"

namespace {

using hnh::grid_for;
using hnh::launch;
using hnh::set_error;

struct Bce {
    double loss, correct, g;
};
__device__ __forceinline__ Bce bce(double s, double y, double inv_count) {
    const double e = exp(-fabs(s));                              // in (0, 1]: no overflow for any s
    const double sig = s >= 0.0 ? 1.0 / (1.0 + e) : e / (1.0 + e);  // sigmoid(s)
    return {fmax(s, 0.0) - s * y + log1p(e), (s > 0.0) == (y > 0.5) ? 1.0 : 0.0, (sig - y) * inv_count};
}

// ---- fast row kernel ---------------------------------------------------------------------------------------------
template <int R, int G, int VW, int UN>
__global__ void __launch_bounds__(kBlock, 1)
link_bce_kernel(const int64_t *__restrict__ rowStart, const int64_t *__restrict__ col_idx, const double *__restrict__ target,
                int64_t rows, const double *__restrict__ X, int64_t ldx, const double *__restrict__ Y, int64_t ldy,
                double inv_count, double *__restrict__ dX, int64_t lddx, double *__restrict__ stats, int64_t lds,
                double *__restrict__ scores) {
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
        double rl = 0.0, rc = 0.0;
        for (int64_t j = s; j < e; j += G) {
            const int cnt = (e - j < G) ? (int)(e - j) : G;
            int64_t mycol = 0;
            double myt = 0.0, mine = 0.0;
            if (gl < cnt) {
                mycol = ld_stream_i64(col_idx + j + gl);
                myt = ld_stream_f64(target + j + gl);
            }
            for (int k0 = 0; k0 < cnt; k0 += UN) {
                double y[UN][NV][VW];
                double tv[UN];
#pragma unroll
                for (int u = 0; u < UN; u++) {
                    const int k = k0 + u;
                    const int src = k < G ? k : G - 1;
                    const int64_t c = __shfl_sync(gmask, mycol, src, G);
                    tv[u] = __shfl_sync(gmask, myt, src, G);
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
                double dv[UN];
#pragma unroll
                for (int u = 0; u < UN; u++) {
                    double d = 0.0;
#pragma unroll
                    for (int v = 0; v < NV; v++)
#pragma unroll
                        for (int w = 0; w < VW; w++) d = fma(x[v][w], y[u][v][w], d);
                    dv[u] = group_allreduce<G>(d, gmask);
                    if (gl == k0 + u) mine = dv[u];
                }
                // the epilogue of entry k0 + u on lane u (and its copies on lanes u + UN, ..): one per batch, not UN
                const int mu = gl % UN;
                double dm = dv[0], tm = tv[0];
#pragma unroll
                for (int u = 1; u < UN; u++)
                    if (mu == u) {
                        dm = dv[u];
                        tm = tv[u];
                    }
                const Bce b = bce(dm, tm, inv_count);
                if (gl < UN && k0 + gl < cnt) {
                    rl += b.loss;
                    rc += b.correct;
                }
#pragma unroll
                for (int u = 0; u < UN; u++) {
                    const double gu = __shfl_sync(gmask, b.g, u, G);
                    if (k0 + u < cnt) {
#pragma unroll
                        for (int v = 0; v < NV; v++)
#pragma unroll
                            for (int w = 0; w < VW; w++) acc[v][w] = fma(gu, y[u][v][w], acc[v][w]);
                    }
                }
            }
            if (scores && gl < cnt) scores[j + gl] = mine;
        }
        if (dX) {
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
        if (stats) {
            // lane u holds the sums of the entries it took, in stored order; the butterfly adds them in a fixed order
            rl = group_allreduce<G>(rl, gmask);
            rc = group_allreduce<G>(rc, gmask);
            if (gl == 0) {
                stats[row * lds] += rl;
                stats[row * lds + 1] += rc;
            }
        }
    }
}

// ---- generic kernel: any r, any leading dimension, any alignment; one warp per row -------------------------------
// kS > 0: r <= 32 kS, lane l keeps columns l + 32 t (t < kS) of X_u and of the gradient row in registers, as the fast
// kernel does.  kS = 0: wider rows; X_u is reread per entry and g Y_v is added to dX_u entry by entry, in stored order.
template <int kS>
__global__ void __launch_bounds__(kBlock, 1)
link_bce_generic_kernel(const int64_t *__restrict__ rowStart, const int64_t *__restrict__ col_idx,
                        const double *__restrict__ target, int64_t rows, const double *__restrict__ X, int64_t ldx,
                        const double *__restrict__ Y, int64_t ldy, int r, double inv_count, double *__restrict__ dX,
                        int64_t lddx, double *__restrict__ stats, int64_t lds, double *__restrict__ scores) {
    constexpr int kR = kS > 0 ? kS : 1;
    const int lane = threadIdx.x & 31;
    const int64_t warps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t row = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; row < rows; row += warps) {
        const int64_t s = rowStart[row], e = rowStart[row + 1];
        if (s == e) continue;
        const double *xr = X + row * ldx;
        double x[kR], acc[kR];
#pragma unroll
        for (int t = 0; t < kR; t++) {
            const int k = lane + 32 * t;
            x[t] = kS > 0 && k < r ? xr[k] : 0.0;
            acc[t] = 0.0;
        }
        double rl = 0.0, rc = 0.0;
        for (int64_t j = s; j < e; j++) {
            const double *yr = Y + col_idx[j] * ldy;
            double d = 0.0;
            if constexpr (kS > 0) {
#pragma unroll
                for (int t = 0; t < kS; t++)
                    if (lane + 32 * t < r) d = fma(x[t], yr[lane + 32 * t], d);
            } else {
                for (int k = lane; k < r; k += 32) d = fma(xr[k], yr[k], d);
            }
            d = group_allreduce<32>(d, 0xffffffffu);
            const Bce b = bce(d, target[j], inv_count);
            rl += b.loss;
            rc += b.correct;
            if (scores && lane == 0) scores[j] = d;
            if (!dX) continue;
            if constexpr (kS > 0) {
#pragma unroll
                for (int t = 0; t < kS; t++)
                    if (lane + 32 * t < r) acc[t] = fma(b.g, yr[lane + 32 * t], acc[t]);
            } else {
                double *o = dX + row * lddx;
                for (int k = lane; k < r; k += 32) o[k] = fma(b.g, yr[k], o[k]);
            }
        }
        if constexpr (kS > 0) {
            if (dX) {
#pragma unroll
                for (int t = 0; t < kS; t++)
                    if (lane + 32 * t < r) dX[row * lddx + lane + 32 * t] += acc[t];
            }
        }
        if (stats && lane == 0) {
            stats[row * lds] += rl;
            stats[row * lds + 1] += rc;
        }
    }
}

// bad[0] += the number of y[i] that are not in [0, 1] (NaN and infinities included): one CTA, a fixed order
__global__ void __launch_bounds__(kBlock) link_target_check_kernel(double *__restrict__ bad, const double *__restrict__ y, int64_t n) {
    __shared__ double sh[kBlock / 32];
    double c = 0.0;
    for (int64_t i = threadIdx.x; i < n; i += kBlock) c += (y[i] >= 0.0 && y[i] <= 1.0) ? 0.0 : 1.0;
    c = group_allreduce<32>(c, 0xffffffffu);
    if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = c;
    __syncthreads();
    if (threadIdx.x == 0) {
        double t = 0.0;
        for (int w = 0; w < kBlock / 32; w++) t += sh[w];
        bad[0] += t;
    }
}

}  // namespace

extern "C" {

int hnh_link_bce_f64(const int64_t *rowStart, const int64_t *col_idx, const double *target, int64_t rows, int64_t nnz,
                     const double *X, int64_t ldx, const double *Y, int64_t ldy, int r, double inv_count, double *dX,
                     int64_t lddx, double *stats, int64_t lds, double *scores, void *stream) {
    const char *who = "hnh_link_bce_f64";
    if (rows < 0 || nnz < 0) return set_error(HNH_E_INVALID, "%s: negative size", who);
    if (r < 1) return set_error(HNH_E_INVALID, "%s: r must be positive (got %d)", who, r);
    if (ldx < r || ldy < r || (dX && lddx < r))
        return set_error(HNH_E_INVALID, "%s: a leading dimension is below r = %d", who, r);
    if (stats && lds < 2) return set_error(HNH_E_INVALID, "%s: the stats' leading dimension is below 2", who);
    if (!(inv_count >= 0.0) || !std::isfinite(inv_count)) return set_error(HNH_E_INVALID, "%s: inv_count must be finite and >= 0", who);
    if (rows == 0 || nnz == 0) return HNH_OK;
    if (!rowStart || !col_idx || !target || !X || !Y) return set_error(HNH_E_INVALID, "%s: null pointer", who);
    const void *outs[] = {dX, stats, scores};
    const void *ins[] = {X, Y, target};
    for (const void *o : outs)
        for (const void *i : ins)
            if (o && o == i) return set_error(HNH_E_INVALID, "%s: an output may not be an input", who);
    if ((dX && (dX == stats || dX == scores)) || (stats && stats == scores))
        return set_error(HNH_E_INVALID, "%s: the outputs must be distinct", who);
    cudaStream_t st = (cudaStream_t)stream;
    int grid = 0, rc = HNH_OK;
    if (table_width(r) && aligned16(X) && aligned16(Y) && ldx % 2 == 0 && ldy % 2 == 0 && (!dX || (aligned16(dX) && lddx % 2 == 0))) {
#define LB(RR, G, VW, UN)                                                                                                  \
    {                                                                                                                      \
        auto k = link_bce_kernel<RR, G, VW, UN>;                                                                           \
        rc = grid_for(k, rows, kBlock / G, &grid);                                                                         \
        if (!rc)                                                                                                           \
            rc = launch(k, grid, kBlock, st, "link_bce_kernel", rowStart, col_idx, target, rows, X, ldx, Y, ldy, inv_count, dX, \
                        lddx, stats, lds, scores);                                                                         \
    }
        HNH_DISPATCH_R(r, LB, )
#undef LB
        return rc;
    }
    auto k = r <= 32 ? link_bce_generic_kernel<1> : r <= 64 ? link_bce_generic_kernel<2> : r <= 128 ? link_bce_generic_kernel<4>
           : r <= 256 ? link_bce_generic_kernel<8> : link_bce_generic_kernel<0>;
    rc = grid_for(k, rows, kBlock / 32, &grid);
    return rc ? rc : launch(k, grid, kBlock, st, "link_bce_generic_kernel", rowStart, col_idx, target, rows, X, ldx, Y, ldy, r,
                            inv_count, dX, lddx, stats, lds, scores);
}

int hnh_link_target_check_f64(double *bad, const double *target, int64_t n, void *stream) {
    if (n < 0) return set_error(HNH_E_INVALID, "hnh_link_target_check_f64: negative size");
    if (!bad || (n > 0 && !target)) return set_error(HNH_E_INVALID, "hnh_link_target_check_f64: null pointer");
    if (n == 0) return HNH_OK;
    return launch(link_target_check_kernel, 1, kBlock, (cudaStream_t)stream, "link_target_check_kernel", bad, target, n);
}

}  // extern "C"
