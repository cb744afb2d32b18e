// pna.cu -- multi-statistic aggregation (Distributed_Sparse::multiAggregate, include/hnh/pna.hpp) on one CSR block, its
// gradient, and PNA's per-row combination of the statistics into aggregators and degree scalers.
//
// The state of a row is up to six f-wide windows, in the fixed order [S1 | S2 | MAX | CMAX | MIN | CMIN], of which the
// flags keep the moments (S1 = sum x, S2 = sum x^2), the maximum with its tie count and the minimum with its tie count:
//     step:   S1 += sum_v X_v,  S2 += sum_v X_v^2,  (MAX, CMAX) = merge(.., (max_v X_v, #ties)),  the same for MIN
//     grad:   dX_v += sum_u D1_u + 2 X_v sum_u D2_u + sum_u [X_v == MAX_u] GMAX_u + sum_u [X_v == MIN_u] GMIN_u
//             (B order: X's rows stored; D = [D1 | D2 | MAX | GMAX | MIN | GMIN] gathered, in the state's layout)
// The fast kernels follow max_aggregate_step_kernel (graph_sage.cu): a group of G lanes owns one CSR row, a chunk of G
// column indices is read coalesced and broadcast by shuffles, gathered rows come in with 128-bit loads, UN rows in
// flight per lane.  Every statistic is kept per column in registers and merged into the state with one read-modify-write
// at the row end, so the state may ride a ring and carry earlier blocks.  Sums run in stored order; extremes merge as
// max_merge does.  Widths 4..256 (powers of two) with 16-byte aligned windows and even leading dimensions take them;
// every other window takes the one-warp-per-row generic kernel.  Wider rows run as column windows of 256: every
// statistic is independent per column.  No atomics anywhere: repeated calls are bit-identical.
#include <cmath>

#include "row_gather.cuh"

namespace {

using hnh::grid_for;
using hnh::launch;
using hnh::set_error;

constexpr int kWindow = 256;  // the widest column window of one launch

__device__ __forceinline__ void min_take(double &m, double &c, double x) {
    if (x < m) {
        m = x;
        c = 1.0;
    } else if (x == m) {
        c += 1.0;
    }
}
__device__ __forceinline__ void min_merge(double &z, double &n, double m, double c) {
    if (m < z) {
        z = m;
        n = c;
    } else if (m == z) {
        n += c;
    }
}

// the column offsets of the windows within a row of the state, for the flags `which`
struct Windows {
    int64_t s1, s2, mx, cmx, mn, cmn;
    bool mom, has_max, has_min;
    __host__ __device__ Windows(int which, int64_t f) {
        mom = which & HNH_MULTI_MOMENTS;
        has_max = which & HNH_MULTI_MAX;
        has_min = which & HNH_MULTI_MIN;
        s1 = 0;
        s2 = f;
        mx = mom ? 2 * f : 0;
        cmx = mx + f;
        mn = mx + (has_max ? 2 * f : 0);
        cmn = mn + f;
    }
};

// ---- fast row kernels ------------------------------------------------------------------------------------------------
// the gradient gathers up to six windows per row; fewer rows in flight keep its registers below the spill line
template <int NVW, int UN>
__host__ __device__ constexpr int grad_un() {
    return NVW >= 8 ? 1 : NVW >= 4 ? (UN < 2 ? UN : 2) : UN;
}

template <int R, int G, int VW, int UN>
__global__ void __launch_bounds__(kBlock, 1)
multi_aggregate_step_kernel(const int64_t *__restrict__ rowStart, const int64_t *__restrict__ col_idx, int64_t rows,
                            const double *__restrict__ X, int64_t ldx, double *__restrict__ A, int64_t lda, int f, int which) {
    constexpr int NV = R / (G * VW);
    static_assert(NV * G * VW == R, "R must equal NV*G*VW");
    const Windows W(which, f);
    const int lane = threadIdx.x & 31;
    const int gl = lane & (G - 1);
    const unsigned gmask = group_mask<G>(lane);
    const int64_t ngroups = (int64_t)gridDim.x * (blockDim.x / G);
    for (int64_t row = (int64_t)blockIdx.x * (blockDim.x / G) + threadIdx.x / G; row < rows; row += ngroups) {
        const int64_t s = ld_stream_i64(rowStart + row);
        const int64_t e = ld_stream_i64(rowStart + row + 1);
        if (s == e) continue;  // nothing to merge
        double s1[NV][VW], s2[NV][VW], mx[NV][VW], cmx[NV][VW], mn[NV][VW], cmn[NV][VW];
#pragma unroll
        for (int v = 0; v < NV; v++)
#pragma unroll
            for (int w = 0; w < VW; w++) {
                s1[v][w] = s2[v][w] = cmx[v][w] = cmn[v][w] = 0.0;
                mx[v][w] = -INFINITY;
                mn[v][w] = INFINITY;
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
                            for (int w = 0; w < VW; w++) y[u][v][w] = 0.0;
                    }
                }
                // in stored order: the sums' rounding and which of tied +0.0 / -0.0 is kept depend on the order only
#pragma unroll
                for (int u = 0; u < UN; u++)
                    if (k0 + u < cnt) {
#pragma unroll
                        for (int v = 0; v < NV; v++)
#pragma unroll
                            for (int w = 0; w < VW; w++) {
                                const double x = y[u][v][w];
                                if (W.mom) {
                                    s1[v][w] += x;
                                    s2[v][w] = fma(x, x, s2[v][w]);
                                }
                                if (W.has_max) max_take(mx[v][w], cmx[v][w], x);
                                if (W.has_min) min_take(mn[v][w], cmn[v][w], x);
                            }
                    }
            }
        }
#pragma unroll
        for (int v = 0; v < NV; v++) {
            double *base = A + row * lda + (v * G + gl) * VW;
            double a[VW], b[VW];
            if (W.mom) {
                ld_rw<VW>(a, base + W.s1);
                ld_rw<VW>(b, base + W.s2);
#pragma unroll
                for (int w = 0; w < VW; w++) {
                    a[w] += s1[v][w];
                    b[w] += s2[v][w];
                }
                st_rw<VW>(base + W.s1, a);
                st_rw<VW>(base + W.s2, b);
            }
            if (W.has_max) {
                ld_rw<VW>(a, base + W.mx);
                ld_rw<VW>(b, base + W.cmx);
#pragma unroll
                for (int w = 0; w < VW; w++) max_merge(a[w], b[w], mx[v][w], cmx[v][w]);
                st_rw<VW>(base + W.mx, a);
                st_rw<VW>(base + W.cmx, b);
            }
            if (W.has_min) {
                ld_rw<VW>(a, base + W.mn);
                ld_rw<VW>(b, base + W.cmn);
#pragma unroll
                for (int w = 0; w < VW; w++) min_merge(a[w], b[w], mn[v][w], cmn[v][w]);
                st_rw<VW>(base + W.mn, a);
                st_rw<VW>(base + W.cmn, b);
            }
        }
    }
}

template <int R, int G, int VW, int UN_>
__global__ void __launch_bounds__(kBlock, 1)
multi_aggregate_grad_kernel(const int64_t *__restrict__ rowStart, const int64_t *__restrict__ col_idx, int64_t rows,
                            const double *__restrict__ X, int64_t ldx, const double *__restrict__ Dg, int64_t ldd, int f, int which,
                            double *__restrict__ dX, int64_t lddx) {
    constexpr int NV = R / (G * VW);
    static_assert(NV * G * VW == R, "R must equal NV*G*VW");
    constexpr int UN = grad_un<NV * VW, UN_>();
    const Windows W(which, f);
    const int lane = threadIdx.x & 31;
    const int gl = lane & (G - 1);
    const unsigned gmask = group_mask<G>(lane);
    const int64_t ngroups = (int64_t)gridDim.x * (blockDim.x / G);
    for (int64_t row = (int64_t)blockIdx.x * (blockDim.x / G) + threadIdx.x / G; row < rows; row += ngroups) {
        const int64_t s = ld_stream_i64(rowStart + row);
        const int64_t e = ld_stream_i64(rowStart + row + 1);
        if (s == e) continue;  // nothing to add
        double x[NV][VW], a1[NV][VW], a2[NV][VW], am[NV][VW], an[NV][VW];
#pragma unroll
        for (int v = 0; v < NV; v++) {
            ld_gather<VW>(x[v], X + row * ldx + (v * G + gl) * VW);
#pragma unroll
            for (int w = 0; w < VW; w++) a1[v][w] = a2[v][w] = am[v][w] = an[v][w] = 0.0;
        }
        for (int64_t j = s; j < e; j += G) {
            const int cnt = (e - j < G) ? (int)(e - j) : G;
            const int64_t mycol = gl < cnt ? ld_stream_i64(col_idx + j + gl) : 0;
            for (int k0 = 0; k0 < cnt; k0 += UN) {
                double d1[UN][NV][VW], d2[UN][NV][VW], zm[UN][NV][VW], gm[UN][NV][VW], zn[UN][NV][VW], gn[UN][NV][VW];
#pragma unroll
                for (int u = 0; u < UN; u++) {
                    const int k = k0 + u;
                    const int64_t col = __shfl_sync(gmask, mycol, k < G ? k : G - 1, G);
#pragma unroll
                    for (int v = 0; v < NV; v++) {
                        const double *p = Dg + col * ldd + (v * G + gl) * VW;
                        if (k < cnt && W.mom) {
                            ld_gather<VW>(d1[u][v], p + W.s1);
                            ld_gather<VW>(d2[u][v], p + W.s2);
                        } else {
#pragma unroll
                            for (int w = 0; w < VW; w++) d1[u][v][w] = d2[u][v][w] = 0.0;
                        }
                        if (k < cnt && W.has_max) {
                            ld_gather<VW>(zm[u][v], p + W.mx);
                            ld_gather<VW>(gm[u][v], p + W.cmx);
                        } else {
#pragma unroll
                            for (int w = 0; w < VW; w++) zm[u][v][w] = gm[u][v][w] = 0.0;
                        }
                        if (k < cnt && W.has_min) {
                            ld_gather<VW>(zn[u][v], p + W.mn);
                            ld_gather<VW>(gn[u][v], p + W.cmn);
                        } else {
#pragma unroll
                            for (int w = 0; w < VW; w++) zn[u][v][w] = gn[u][v][w] = 0.0;
                        }
                    }
                }
#pragma unroll
                for (int u = 0; u < UN; u++)
                    if (k0 + u < cnt) {
#pragma unroll
                        for (int v = 0; v < NV; v++)
#pragma unroll
                            for (int w = 0; w < VW; w++) {
                                a1[v][w] += d1[u][v][w];
                                a2[v][w] += d2[u][v][w];
                                if (W.has_max && x[v][w] == zm[u][v][w]) am[v][w] += gm[u][v][w];
                                if (W.has_min && x[v][w] == zn[u][v][w]) an[v][w] += gn[u][v][w];
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
            for (int w = 0; w < VW; w++) o[w] += ((a1[v][w] + 2.0 * x[v][w] * a2[v][w]) + am[v][w]) + an[v][w];
            st_rw<VW>(p, o);
        }
    }
}

// ---- generic kernels: any window width up to 256, any leading dimension, any alignment; one warp per row ---------------
// Lane l keeps columns l + 32 t (t < kS) of the row's state in registers, w <= 32 kS.
template <int kS>
__global__ void __launch_bounds__(kBlock, 1)
multi_aggregate_step_generic_kernel(const int64_t *__restrict__ rowStart, const int64_t *__restrict__ col_idx, int64_t rows,
                                    const double *__restrict__ X, int64_t ldx, int width, double *__restrict__ A, int64_t lda,
                                    int f, int which) {
    const Windows W(which, f);
    const int lane = threadIdx.x & 31;
    const int64_t warps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t row = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; row < rows; row += warps) {
        const int64_t s = rowStart[row], e = rowStart[row + 1];
        if (s == e) continue;
        double s1[kS], s2[kS], mx[kS], cmx[kS], mn[kS], cmn[kS];
#pragma unroll
        for (int t = 0; t < kS; t++) {
            s1[t] = s2[t] = cmx[t] = cmn[t] = 0.0;
            mx[t] = -INFINITY;
            mn[t] = INFINITY;
        }
        for (int64_t j = s; j < e; j++) {
            const double *yr = X + col_idx[j] * ldx;
#pragma unroll
            for (int t = 0; t < kS; t++)
                if (lane + 32 * t < width) {
                    const double x = yr[lane + 32 * t];
                    if (W.mom) {
                        s1[t] += x;
                        s2[t] = fma(x, x, s2[t]);
                    }
                    if (W.has_max) max_take(mx[t], cmx[t], x);
                    if (W.has_min) min_take(mn[t], cmn[t], x);
                }
        }
#pragma unroll
        for (int t = 0; t < kS; t++) {
            const int k = lane + 32 * t;
            if (k >= width) continue;
            double *base = A + row * lda + k;
            if (W.mom) {
                base[W.s1] += s1[t];
                base[W.s2] += s2[t];
            }
            if (W.has_max) {
                double z = base[W.mx], n = base[W.cmx];
                max_merge(z, n, mx[t], cmx[t]);
                base[W.mx] = z;
                base[W.cmx] = n;
            }
            if (W.has_min) {
                double z = base[W.mn], n = base[W.cmn];
                min_merge(z, n, mn[t], cmn[t]);
                base[W.mn] = z;
                base[W.cmn] = n;
            }
        }
    }
}

template <int kS>
__global__ void __launch_bounds__(kBlock, 1)
multi_aggregate_grad_generic_kernel(const int64_t *__restrict__ rowStart, const int64_t *__restrict__ col_idx, int64_t rows,
                                    const double *__restrict__ X, int64_t ldx, const double *__restrict__ Dg, int64_t ldd, int width,
                                    int f, int which, double *__restrict__ dX, int64_t lddx) {
    const Windows W(which, f);
    const int lane = threadIdx.x & 31;
    const int64_t warps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t row = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; row < rows; row += warps) {
        const int64_t s = rowStart[row], e = rowStart[row + 1];
        if (s == e) continue;
        double x[kS], a1[kS], a2[kS], am[kS], an[kS];
#pragma unroll
        for (int t = 0; t < kS; t++) {
            const int k = lane + 32 * t;
            x[t] = k < width ? X[row * ldx + k] : 0.0;
            a1[t] = a2[t] = am[t] = an[t] = 0.0;
        }
        for (int64_t j = s; j < e; j++) {
            const double *p = Dg + col_idx[j] * ldd;
#pragma unroll
            for (int t = 0; t < kS; t++) {
                const int k = lane + 32 * t;
                if (k >= width) continue;
                if (W.mom) {
                    a1[t] += p[W.s1 + k];
                    a2[t] += p[W.s2 + k];
                }
                if (W.has_max && x[t] == p[W.mx + k]) am[t] += p[W.cmx + k];
                if (W.has_min && x[t] == p[W.mn + k]) an[t] += p[W.cmn + k];
            }
        }
#pragma unroll
        for (int t = 0; t < kS; t++) {
            const int k = lane + 32 * t;
            if (k < width) dX[row * lddx + k] += ((a1[t] + 2.0 * x[t] * a2[t]) + am[t]) + an[t];
        }
    }
}

// ---- elementwise ----------------------------------------------------------------------------------------------------
// the extremes of rows without entries (count 0) become 0
__global__ void __launch_bounds__(kBlock, 1) multi_aggregate_finish_kernel(double *__restrict__ A, int64_t lda, int64_t rows, int f,
                                                                           int which) {
    const Windows W(which, f);
    const int64_t n = rows * f, stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
        double *p = A + (i / f) * lda + i % f;
        if (W.has_max && p[W.cmx] == 0.0) p[W.mx] = 0.0;
        if (W.has_min && p[W.cmn] == 0.0) p[W.mn] = 0.0;
    }
}

// D = [dA_S1 | dA_S2 | MAX | dA_MAX / CMAX | MIN | dA_MIN / CMIN] (0 where a count is 0)
__global__ void __launch_bounds__(kBlock, 1) multi_aggregate_grad_prep_kernel(const double *__restrict__ A, int64_t lda,
                                                                              const double *__restrict__ dA, int64_t ldda, int64_t rows,
                                                                              int f, int which, double *__restrict__ D, int64_t ldd) {
    const Windows W(which, f);
    const int64_t n = rows * f, stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
        const int64_t r = i / f, k = i % f;
        const double *a = A + r * lda + k, *da = dA + r * ldda + k;
        double *d = D + r * ldd + k;
        if (W.mom) {
            d[W.s1] = da[W.s1];
            d[W.s2] = da[W.s2];
        }
        if (W.has_max) {
            const double c = a[W.cmx];
            d[W.mx] = a[W.mx];
            d[W.cmx] = c == 0.0 ? 0.0 : da[W.mx] / c;
        }
        if (W.has_min) {
            const double c = a[W.cmn];
            d[W.mn] = a[W.mn];
            d[W.cmn] = c == 0.0 ? 0.0 : da[W.mn] / c;
        }
    }
}

// ---- PNA's aggregators and scalers -----------------------------------------------------------------------------------
// codes packed 4 bits each, the first in the lowest bits
__device__ __forceinline__ int code_at(unsigned packed, int i) { return (int)((packed >> (4 * i)) & 15u); }

constexpr double kStdEps = 1e-5;  // PyG's StdAggregation: sqrt(clamp(var, 1e-5)), 0 where that is <= sqrt(1e-5)

__device__ __forceinline__ double pna_scale(int code, double d, double lin, double lg) {
    const double dc = d < 1.0 ? 1.0 : d;  // PyG's degree(..).clamp(1)
    switch (code) {
        case HNH_PNA_AMPLIFICATION: return log(dc + 1.0) / lg;
        case HNH_PNA_ATTENUATION: return lg / log(dc + 1.0);
        case HNH_PNA_LINEAR: return dc / lin;
        case HNH_PNA_INVERSE_LINEAR: return lin / dc;
        default: return 1.0;
    }
}

// P[u] = [X_u | scale_s0(u) [agg_0 .. agg_A-1] | scale_s1(u) [..] | ..] for the aggregates of h_uv = c_u + z_v
__global__ void __launch_bounds__(kBlock, 1)
pna_combine_kernel(const double *__restrict__ X, int64_t ldx, const double *__restrict__ Cu, int64_t ldc, const double *__restrict__ A,
                   int64_t lda, int which, const double *__restrict__ deg, int64_t ldg, int64_t rows, int f, unsigned aggs, int n_aggs,
                   unsigned scalers, int n_scalers, double lin, double lg, double *__restrict__ P, int64_t ldp) {
    const Windows W(which, f);
    const int64_t n = rows * f, stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
        const int64_t r = i / f, k = i % f;
        const double *a = A + r * lda + k;
        const double d = deg[r * ldg], c = Cu[r * ldc + k];
        double *p = P + r * ldp + k;
        p[0] = X[r * ldx + k];
        double agg[6];  // fixed trip counts keep agg in registers
#pragma unroll
        for (int j = 0; j < 6; j++) {
            double v = 0.0;
            if (j < n_aggs && d > 0.0) {
                switch (code_at(aggs, j)) {
                    case HNH_PNA_MEAN: v = c + a[W.s1] / d; break;
                    case HNH_PNA_SUM: v = d * c + a[W.s1]; break;
                    case HNH_PNA_MIN: v = c + a[W.mn]; break;
                    case HNH_PNA_MAX: v = c + a[W.mx]; break;
                    default: {
                        const double m = a[W.s1] / d, var = a[W.s2] / d - m * m;
                        if (code_at(aggs, j) == HNH_PNA_VAR) {
                            v = var;
                        } else {
                            const double sd = sqrt(fmax(var, kStdEps));
                            v = sd <= sqrt(kStdEps) ? 0.0 : sd;
                        }
                    }
                }
            }
            agg[j] = v;
        }
        for (int s = 0; s < n_scalers; s++) {
            const double sc = pna_scale(code_at(scalers, s), d, lin, lg);
#pragma unroll
            for (int j = 0; j < 6; j++)
                if (j < n_aggs) p[(int64_t)(1 + s * n_aggs + j) * f] = sc * agg[j];
        }
    }
}

// dC and dA (the state's layout; the count windows 0) from dP, through the scalers and aggregators
__global__ void __launch_bounds__(kBlock, 1)
pna_combine_grad_kernel(const double *__restrict__ dP, int64_t lddp, const double *__restrict__ A, int64_t lda, int which,
                        const double *__restrict__ deg, int64_t ldg, int64_t rows, int f, unsigned aggs, int n_aggs, unsigned scalers,
                        int n_scalers, double lin, double lg, double *__restrict__ dC, int64_t lddc, double *__restrict__ dA,
                        int64_t ldda) {
    const Windows W(which, f);
    const int64_t n = rows * f, stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
        const int64_t r = i / f, k = i % f;
        const double *a = A + r * lda + k, *dp = dP + r * lddp + k;
        const double d = deg[r * ldg];
        double g1 = 0.0, g2 = 0.0, gmx = 0.0, gmn = 0.0, gc = 0.0;
        if (d > 0.0) {
            double sc[5];  // fixed trip counts keep sc in registers
#pragma unroll
            for (int s = 0; s < 5; s++) sc[s] = s < n_scalers ? pna_scale(code_at(scalers, s), d, lin, lg) : 0.0;
            const double m = W.mom ? a[W.s1] / d : 0.0, var = W.mom ? a[W.s2] / d - m * m : 0.0;
            for (int j = 0; j < n_aggs; j++) {
                double g = 0.0;
#pragma unroll
                for (int s = 0; s < 5; s++)
                    if (s < n_scalers) g += sc[s] * dp[(int64_t)(1 + s * n_aggs + j) * f];
                switch (code_at(aggs, j)) {
                    case HNH_PNA_MEAN:
                        g1 += g / d;
                        gc += g;
                        break;
                    case HNH_PNA_SUM:
                        g1 += g;
                        gc += d * g;
                        break;
                    case HNH_PNA_MIN:
                        gmn += g;
                        gc += g;
                        break;
                    case HNH_PNA_MAX:
                        gmx += g;
                        gc += g;
                        break;
                    default: {
                        double gv = g;  // dL/d var
                        if (code_at(aggs, j) == HNH_PNA_STD) {
                            const double sd = sqrt(fmax(var, kStdEps));
                            gv = sd <= sqrt(kStdEps) ? 0.0 : g / (2.0 * sd);
                        }
                        g2 += gv / d;
                        g1 -= 2.0 * m * gv / d;
                    }
                }
            }
        }
        dC[r * lddc + k] = gc;
        double *o = dA + r * ldda + k;
        if (W.mom) {
            o[W.s1] = g1;
            o[W.s2] = g2;
        }
        if (W.has_max) {
            o[W.mx] = gmx;
            o[W.cmx] = 0.0;
        }
        if (W.has_min) {
            o[W.mn] = gmn;
            o[W.cmn] = 0.0;
        }
    }
}

// the one-warp-per-row instantiation for a window of width w <= 256
template <typename K>
K pick_generic(int w, K k1, K k2, K k4, K k8) {
    return w <= 32 ? k1 : w <= 64 ? k2 : w <= 128 ? k4 : k8;
}

int check_which(const char *who, int which) {
    if (which < 1 || which > HNH_MULTI_ALL) return set_error(HNH_E_INVALID, "%s: which = %d selects no statistic or an unknown one", who, which);
    return HNH_OK;
}
// the state's width in columns
int64_t state_width(int which, int64_t f) {
    return 2 * f * (((which & HNH_MULTI_MOMENTS) != 0) + ((which & HNH_MULTI_MAX) != 0) + ((which & HNH_MULTI_MIN) != 0));
}
// every selected window of a state at column c0 is 16-byte aligned
bool windows_aligned(const double *A, int f, int which, int c0) {
    const Windows W(which, f);
    bool ok = true;
    if (W.mom) ok = ok && aligned16(A + c0 + W.s1) && aligned16(A + c0 + W.s2);
    if (W.has_max) ok = ok && aligned16(A + c0 + W.mx) && aligned16(A + c0 + W.cmx);
    if (W.has_min) ok = ok && aligned16(A + c0 + W.mn) && aligned16(A + c0 + W.cmn);
    return ok;
}

int check_codes(const char *who, unsigned packed, int n, int count) {
    if (n < 1 || n > count) return set_error(HNH_E_INVALID, "%s: %d codes, 1 to %d allowed", who, n, count);
    for (int i = 0; i < n; i++)
        if ((int)((packed >> (4 * i)) & 15u) >= count) return set_error(HNH_E_INVALID, "%s: unknown code at %d", who, i);
    return HNH_OK;
}

// every aggregator's statistic is in the state
int check_aggs_in_state(const char *who, unsigned aggs, int n_aggs, int which) {
    for (int i = 0; i < n_aggs; i++) {
        const int a = (int)((aggs >> (4 * i)) & 15u);
        const int need = a == HNH_PNA_MIN ? HNH_MULTI_MIN : a == HNH_PNA_MAX ? HNH_MULTI_MAX : HNH_MULTI_MOMENTS;
        if (!(which & need)) return set_error(HNH_E_INVALID, "%s: aggregator %d reads a statistic which = %d does not hold", who, i, which);
    }
    return HNH_OK;
}

}  // namespace

extern "C" {

int hnh_multi_aggregate_step_f64(const int64_t *rowStart, const int64_t *col_idx, int64_t rows, int64_t nnz, const double *X,
                                 int64_t ldx, int f, int which, double *A, int64_t lda, void *stream) {
    const char *who = "hnh_multi_aggregate_step_f64";
    if (rows < 0 || nnz < 0) return set_error(HNH_E_INVALID, "%s: negative size", who);
    if (f < 1) return set_error(HNH_E_INVALID, "%s: f must be positive (got %d)", who, f);
    if (int rc = check_which(who, which)) return rc;
    if (state_width(which, f) > INT32_MAX) return set_error(HNH_E_INVALID, "%s: the state is 2^31 columns or wider", who);
    if (ldx < f || lda < state_width(which, f)) return set_error(HNH_E_INVALID, "%s: a leading dimension is below its operand's width", who);
    if (rows == 0 || nnz == 0) return HNH_OK;
    if (!rowStart || !col_idx || !X || !A) return set_error(HNH_E_INVALID, "%s: null pointer", who);
    if (A == X) return set_error(HNH_E_INVALID, "%s: the state may not be the input", who);
    cudaStream_t st = (cudaStream_t)stream;
    int rc = HNH_OK;
    for (int c0 = 0; c0 < f && rc == HNH_OK; c0 += kWindow) {
        const int w = std::min(kWindow, f - c0);
        const double *Xw = X + c0;
        double *Aw = A + c0;
        int grid = 0;
        if (table_width(w) && aligned16(Xw) && windows_aligned(A, f, which, c0) && ldx % 2 == 0 && lda % 2 == 0) {
#define MS(RR, G, VW, UN)                                                                                                  \
    {                                                                                                                      \
        auto k = multi_aggregate_step_kernel<RR, G, VW, UN>;                                                               \
        rc = grid_for(k, rows, kBlock / G, &grid);                                                                         \
        if (!rc) rc = launch(k, grid, kBlock, st, "multi_aggregate_step_kernel", rowStart, col_idx, rows, Xw, ldx, Aw, lda, f, which); \
    }
            HNH_DISPATCH_R(w, MS, )
#undef MS
            continue;
        }
        auto k = pick_generic(w, multi_aggregate_step_generic_kernel<1>, multi_aggregate_step_generic_kernel<2>,
                              multi_aggregate_step_generic_kernel<4>, multi_aggregate_step_generic_kernel<8>);
        rc = grid_for(k, rows, kBlock / 32, &grid);
        if (!rc)
            rc = launch(k, grid, kBlock, st, "multi_aggregate_step_generic_kernel", rowStart, col_idx, rows, Xw, ldx, w, Aw, lda, f, which);
    }
    return rc;
}

int hnh_multi_aggregate_finish_f64(double *A, int64_t lda, int64_t rows, int f, int which, void *stream) {
    const char *who = "hnh_multi_aggregate_finish_f64";
    if (rows < 0 || f < 1) return set_error(HNH_E_INVALID, "%s: bad size", who);
    if (int rc = check_which(who, which)) return rc;
    if (lda < state_width(which, f)) return set_error(HNH_E_INVALID, "%s: lda is below the state's width", who);
    if (rows == 0 || !(which & (HNH_MULTI_MAX | HNH_MULTI_MIN))) return HNH_OK;
    if (!A) return set_error(HNH_E_INVALID, "%s: null pointer", who);
    int grid = 0;
    int rc = grid_for(multi_aggregate_finish_kernel, rows * f, kBlock * 4, &grid);
    return rc ? rc : launch(multi_aggregate_finish_kernel, grid, kBlock, (cudaStream_t)stream, "multi_aggregate_finish_kernel", A, lda, rows, f, which);
}

int hnh_multi_aggregate_grad_prep_f64(const double *A, int64_t lda, const double *dA, int64_t ldda, int64_t rows, int f, int which,
                                      double *D, int64_t ldd, void *stream) {
    const char *who = "hnh_multi_aggregate_grad_prep_f64";
    if (rows < 0 || f < 1) return set_error(HNH_E_INVALID, "%s: bad size", who);
    if (int rc = check_which(who, which)) return rc;
    const int64_t w = state_width(which, f);
    if (lda < w || ldda < w || ldd < w) return set_error(HNH_E_INVALID, "%s: a leading dimension is below the state's width", who);
    if (rows == 0) return HNH_OK;
    if (!A || !dA || !D) return set_error(HNH_E_INVALID, "%s: null pointer", who);
    if ((const double *)D == A || (const double *)D == dA) return set_error(HNH_E_INVALID, "%s: D may not be an input", who);
    int grid = 0;
    int rc = grid_for(multi_aggregate_grad_prep_kernel, rows * f, kBlock * 4, &grid);
    return rc ? rc
              : launch(multi_aggregate_grad_prep_kernel, grid, kBlock, (cudaStream_t)stream, "multi_aggregate_grad_prep_kernel", A, lda,
                       dA, ldda, rows, f, which, D, ldd);
}

int hnh_multi_aggregate_grad_f64(const int64_t *rowStart, const int64_t *col_idx, int64_t rows, int64_t nnz, const double *X,
                                 int64_t ldx, const double *D, int64_t ldd, int f, int which, double *dX, int64_t lddx, void *stream) {
    const char *who = "hnh_multi_aggregate_grad_f64";
    if (rows < 0 || nnz < 0) return set_error(HNH_E_INVALID, "%s: negative size", who);
    if (f < 1) return set_error(HNH_E_INVALID, "%s: f must be positive (got %d)", who, f);
    if (int rc = check_which(who, which)) return rc;
    if (state_width(which, f) > INT32_MAX) return set_error(HNH_E_INVALID, "%s: the state is 2^31 columns or wider", who);
    if (ldx < f || lddx < f || ldd < state_width(which, f))
        return set_error(HNH_E_INVALID, "%s: a leading dimension is below its operand's width", who);
    if (rows == 0 || nnz == 0) return HNH_OK;
    if (!rowStart || !col_idx || !X || !D || !dX) return set_error(HNH_E_INVALID, "%s: null pointer", who);
    if (dX == X || dX == D) return set_error(HNH_E_INVALID, "%s: dX may not be an input", who);
    cudaStream_t st = (cudaStream_t)stream;
    int rc = HNH_OK;
    for (int c0 = 0; c0 < f && rc == HNH_OK; c0 += kWindow) {
        const int w = std::min(kWindow, f - c0);
        const double *Xw = X + c0, *Dw = D + c0;
        double *dXw = dX + c0;
        int grid = 0;
        if (table_width(w) && aligned16(Xw) && aligned16(dXw) && windows_aligned(D, f, which, c0) && ldx % 2 == 0 && ldd % 2 == 0 &&
            lddx % 2 == 0) {
#define MG(RR, G_, VW, UN)                                                                                                 \
    {                                                                                                                      \
        auto k = multi_aggregate_grad_kernel<RR, G_, VW, UN>;                                                              \
        rc = grid_for(k, rows, kBlock / G_, &grid);                                                                        \
        if (!rc)                                                                                                           \
            rc = launch(k, grid, kBlock, st, "multi_aggregate_grad_kernel", rowStart, col_idx, rows, Xw, ldx, Dw, ldd, f, which, dXw, lddx); \
    }
            HNH_DISPATCH_R(w, MG, )
#undef MG
            continue;
        }
        auto k = pick_generic(w, multi_aggregate_grad_generic_kernel<1>, multi_aggregate_grad_generic_kernel<2>,
                              multi_aggregate_grad_generic_kernel<4>, multi_aggregate_grad_generic_kernel<8>);
        rc = grid_for(k, rows, kBlock / 32, &grid);
        if (!rc)
            rc = launch(k, grid, kBlock, st, "multi_aggregate_grad_generic_kernel", rowStart, col_idx, rows, Xw, ldx, Dw, ldd, w, f,
                        which, dXw, lddx);
    }
    return rc;
}

int hnh_pna_combine_f64(const double *X, int64_t ldx, const double *C, int64_t ldc, const double *A, int64_t lda, int which,
                        const double *deg, int64_t ldg, int64_t rows, int f, unsigned aggs, int n_aggs, unsigned scalers, int n_scalers,
                        double avg_deg_lin, double avg_deg_log, double *P, int64_t ldp, void *stream) {
    const char *who = "hnh_pna_combine_f64";
    if (rows < 0 || f < 1) return set_error(HNH_E_INVALID, "%s: bad size", who);
    if (int rc = check_which(who, which)) return rc;
    if (int rc = check_codes(who, aggs, n_aggs, 6)) return rc;
    if (int rc = check_codes(who, scalers, n_scalers, 5)) return rc;
    if (int rc = check_aggs_in_state(who, aggs, n_aggs, which)) return rc;
    const int64_t pw = ((int64_t)n_aggs * n_scalers + 1) * f;
    if (ldx < f || ldc < f || lda < state_width(which, f) || ldg < 1 || ldp < pw)
        return set_error(HNH_E_INVALID, "%s: a leading dimension is below its operand's width", who);
    if (rows == 0) return HNH_OK;
    if (!X || !C || !A || !deg || !P) return set_error(HNH_E_INVALID, "%s: null pointer", who);
    int grid = 0;
    int rc = grid_for(pna_combine_kernel, rows * f, kBlock * 4, &grid);
    return rc ? rc
              : launch(pna_combine_kernel, grid, kBlock, (cudaStream_t)stream, "pna_combine_kernel", X, ldx, C, ldc, A, lda, which, deg,
                       ldg, rows, f, aggs, n_aggs, scalers, n_scalers, avg_deg_lin, avg_deg_log, P, ldp);
}

int hnh_pna_combine_grad_f64(const double *dP, int64_t lddp, const double *A, int64_t lda, int which, const double *deg, int64_t ldg,
                             int64_t rows, int f, unsigned aggs, int n_aggs, unsigned scalers, int n_scalers, double avg_deg_lin,
                             double avg_deg_log, double *dC, int64_t lddc, double *dA, int64_t ldda, void *stream) {
    const char *who = "hnh_pna_combine_grad_f64";
    if (rows < 0 || f < 1) return set_error(HNH_E_INVALID, "%s: bad size", who);
    if (int rc = check_which(who, which)) return rc;
    if (int rc = check_codes(who, aggs, n_aggs, 6)) return rc;
    if (int rc = check_codes(who, scalers, n_scalers, 5)) return rc;
    if (int rc = check_aggs_in_state(who, aggs, n_aggs, which)) return rc;
    const int64_t pw = ((int64_t)n_aggs * n_scalers + 1) * f, w = state_width(which, f);
    if (lddp < pw || lda < w || ldda < w || ldg < 1 || lddc < f)
        return set_error(HNH_E_INVALID, "%s: a leading dimension is below its operand's width", who);
    if (rows == 0) return HNH_OK;
    if (!dP || !A || !deg || !dC || !dA) return set_error(HNH_E_INVALID, "%s: null pointer", who);
    int grid = 0;
    int rc = grid_for(pna_combine_grad_kernel, rows * f, kBlock * 4, &grid);
    return rc ? rc
              : launch(pna_combine_grad_kernel, grid, kBlock, (cudaStream_t)stream, "pna_combine_grad_kernel", dP, lddp, A, lda, which,
                       deg, ldg, rows, f, aggs, n_aggs, scalers, n_scalers, avg_deg_lin, avg_deg_log, dC, lddc, dA, ldda);
}

}  // extern "C"
