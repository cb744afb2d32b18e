// distmult.cu -- the DistMult edge decoder of relation-aware link prediction (Distributed_Sparse::distmultLoss,
// include/hnh/distmult.hpp) on one CSR block, and the reduction of its relation-table gradient.  With X the row side
// (indexed by the stored row u), Y the gathered side (indexed by col_idx v), D the R x r relation table, rho an entry's
// stored value read as a relation (an integer in [0, R); anything else contributes nothing) and y a constant target:
//     s   = sum_k X_u,k D_rho,k Y_v,k                              scores[i]           (nullable)
//     l   = max(s, 0) - s y + log1p(exp(-|s|)),  c = [(s > 0) == (y > 0.5)],  g = (sigmoid(s) - y) inv_count
//     dX_u += sum_v g (D_rho o Y_v)                                 (nullable)
//     stats[u, 0] += sum_v l,  stats[u, 1] += sum_v c               (nullable)
//     gout[i] = g                                                   (nullable; 0 for an entry that is no relation)
// The row kernels follow link_bce_kernel (link_prediction.cu): a group of G lanes owns one CSR row and keeps X_u in
// registers, gathered rows come in with 128-bit loads, UN rows in flight per lane, one epilogue per batch, sums in
// stored order and one read-modify-write of dX and stats per row.  D_rho is gathered per entry beside Y_v: D is small
// and read by every entry, so its lines get an L2 evict-last policy (and may stay in L1), while T's index and value
// streams, read once, get evict-first, so neither pushes D or the gathered rows out of L2.  Widths 4..256 (powers of
// two) with 16-byte aligned operands and even leading dimensions take them; every other case takes one warp per row.
//
// The relation-table gradient dD_rho = sum over the entries of relation rho of g (X_u o Y_v) runs on a grouping of a
// block's entries by relation (an hnh_edge_softmax_plan keyed by relation): one lane group per piece of at most
// HNH_EDGE_PIECE entries gathers X_u and Y_v of each and writes the piece's r-wide sum, then the pieces of each
// relation are summed column by column in plan order.  No atomics anywhere: repeated calls are bit-identical.
#include <cmath>

#include "row_gather.cuh"

namespace {

using hnh::grid_for;
using hnh::launch;
using hnh::set_error;

__device__ __forceinline__ uint64_t evict_first_policy() {
    uint64_t p;
    asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p));
    return p;
}
__device__ __forceinline__ uint64_t evict_last_policy() {
    uint64_t p;
    asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(p));
    return p;
}
// T's streams: read once, evicted first
__device__ __forceinline__ int64_t ld_first_i64(const int64_t *p, uint64_t policy) {
    int64_t v;
    asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.s64 %0, [%1], %2;" : "=l"(v) : "l"(p), "l"(policy));
    return v;
}
__device__ __forceinline__ double ld_first_f64(const double *p, uint64_t policy) {
    double v;
    asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.f64 %0, [%1], %2;" : "=d"(v) : "l"(p), "l"(policy));
    return v;
}
// D's rows: read by every entry, kept
template <int VW>
__device__ __forceinline__ void ld_table(double (&d)[VW], const double *p, uint64_t policy) {
    static_assert(VW == 2, "128-bit loads only");
    asm volatile("ld.global.nc.L2::cache_hint.v2.f64 {%0,%1}, [%2], %3;" : "=d"(d[0]), "=d"(d[1]) : "l"(p), "l"(policy));
}

__device__ __forceinline__ int relation_of(double v, int nrel) {
    return (v >= 0.0 && v < (double)nrel && v == trunc(v)) ? (int)v : nrel;
}

struct Bce {
    double loss, correct, g;
};
// link_prediction.cu's bce: the same formula, so that R = 1 with D = 1 gives linkLoss's bits
__device__ __forceinline__ Bce bce(double s, double y, double inv_count) {
    const double e = exp(-fabs(s));
    const double sig = s >= 0.0 ? 1.0 / (1.0 + e) : e / (1.0 + e);
    return {fmax(s, 0.0) - s * y + log1p(e), (s > 0.0) == (y > 0.5) ? 1.0 : 0.0, (sig - y) * inv_count};
}

struct BceArgs {
    const int64_t *rowStart, *col_idx;
    const double *rel;
    int64_t rows;
    int nrel;
    const double *X;
    int64_t ldx;
    const double *Y;
    int64_t ldy;
    const double *D;
    int64_t ldd;
    double target, inv_count;
    double *dX;
    int64_t lddx;
    double *stats;
    int64_t lds;
    double *scores, *gout;
};

// ---- fast row kernel ---------------------------------------------------------------------------------------------
template <int R, int G, int VW, int UN>
__global__ void __launch_bounds__(kBlock, 1) distmult_bce_kernel(const BceArgs a) {
    constexpr int NV = R / (G * VW);
    static_assert(NV * G * VW == R, "R must equal NV*G*VW");
    const uint64_t first = evict_first_policy(), last = evict_last_policy();
    const int lane = threadIdx.x & 31;
    const int gl = lane & (G - 1);
    const unsigned gmask = group_mask<G>(lane);
    const int64_t ngroups = (int64_t)gridDim.x * (blockDim.x / G);
    for (int64_t row = (int64_t)blockIdx.x * (blockDim.x / G) + threadIdx.x / G; row < a.rows; row += ngroups) {
        const int64_t s = ld_first_i64(a.rowStart + row, first);
        const int64_t e = ld_first_i64(a.rowStart + row + 1, first);
        if (s == e) continue;
        double x[NV][VW], acc[NV][VW];
#pragma unroll
        for (int v = 0; v < NV; v++) {
            ld_gather<VW>(x[v], a.X + row * a.ldx + (v * G + gl) * VW);
#pragma unroll
            for (int w = 0; w < VW; w++) acc[v][w] = 0.0;
        }
        double rl = 0.0, rc = 0.0;
        for (int64_t j = s; j < e; j += G) {
            const int cnt = (e - j < G) ? (int)(e - j) : G;
            int64_t mycol = 0;
            int myrel = a.nrel;
            double mine = 0.0;
            if (gl < cnt) {
                mycol = ld_first_i64(a.col_idx + j + gl, first);
                myrel = relation_of(ld_first_f64(a.rel + j + gl, first), a.nrel);
            }
            for (int k0 = 0; k0 < cnt; k0 += UN) {
                double y[UN][NV][VW], d[UN][NV][VW];
                bool on[UN];
#pragma unroll
                for (int u = 0; u < UN; u++) {
                    const int k = k0 + u;
                    const int src = k < G ? k : G - 1;
                    const int64_t c = __shfl_sync(gmask, mycol, src, G);
                    const int rho = __shfl_sync(gmask, myrel, src, G);
                    on[u] = k < cnt && rho < a.nrel;
                    if (on[u]) {
#pragma unroll
                        for (int v = 0; v < NV; v++) {
                            ld_gather<VW>(y[u][v], a.Y + c * a.ldy + (v * G + gl) * VW);
                            ld_table<VW>(d[u][v], a.D + rho * a.ldd + (v * G + gl) * VW, last);
                        }
                    } else {
#pragma unroll
                        for (int v = 0; v < NV; v++)
#pragma unroll
                            for (int w = 0; w < VW; w++) y[u][v][w] = d[u][v][w] = 0.0;
                    }
                }
                double dv[UN];
#pragma unroll
                for (int u = 0; u < UN; u++) {
                    double t = 0.0;
#pragma unroll
                    for (int v = 0; v < NV; v++)
#pragma unroll
                        for (int w = 0; w < VW; w++) t = fma(x[v][w] * d[u][v][w], y[u][v][w], t);
                    dv[u] = group_allreduce<G>(t, gmask);
                    if (gl == k0 + u) mine = dv[u];
                }
                // the epilogue of entry k0 + u on lane u (and its copies on lanes u + UN, ..)
                const int mu = gl % UN;
                double dm = dv[0];
                bool om = on[0];
#pragma unroll
                for (int u = 1; u < UN; u++)
                    if (mu == u) {
                        dm = dv[u];
                        om = on[u];
                    }
                const Bce b = bce(dm, a.target, a.inv_count);
                const double gm = om ? b.g : 0.0;
                if (gl < UN && k0 + gl < cnt) {
                    if (om) {
                        rl += b.loss;
                        rc += b.correct;
                    }
                    if (a.gout) a.gout[j + k0 + gl] = gm;
                }
#pragma unroll
                for (int u = 0; u < UN; u++) {
                    const double gu = __shfl_sync(gmask, gm, u, G);
                    if (on[u]) {
#pragma unroll
                        for (int v = 0; v < NV; v++)
#pragma unroll
                            for (int w = 0; w < VW; w++) acc[v][w] = fma(gu, d[u][v][w] * y[u][v][w], acc[v][w]);
                    }
                }
            }
            if (a.scores && gl < cnt) a.scores[j + gl] = mine;
        }
        if (a.dX) {
#pragma unroll
            for (int v = 0; v < NV; v++) {
                double o[VW];
                double *p = a.dX + row * a.lddx + (v * G + gl) * VW;
                ld_rw<VW>(o, p);
#pragma unroll
                for (int w = 0; w < VW; w++) o[w] += acc[v][w];
                st_rw<VW>(p, o);
            }
        }
        if (a.stats) {
            rl = group_allreduce<G>(rl, gmask);
            rc = group_allreduce<G>(rc, gmask);
            if (gl == 0) {
                a.stats[row * a.lds] += rl;
                a.stats[row * a.lds + 1] += rc;
            }
        }
    }
}

// ---- generic kernel: any r, any leading dimension, any alignment; one warp per row -------------------------------
// kS > 0: r <= 32 kS, lane l keeps columns l + 32 t of X_u and of the gradient row in registers.  kS = 0: wider rows;
// X_u is reread per entry and g (D_rho o Y_v) is added to dX_u entry by entry, in stored order.
template <int kS>
__global__ void __launch_bounds__(kBlock, 1) distmult_bce_generic_kernel(const BceArgs a, int r) {
    constexpr int kR = kS > 0 ? kS : 1;
    const int lane = threadIdx.x & 31;
    const int64_t warps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t row = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; row < a.rows; row += warps) {
        const int64_t s = a.rowStart[row], e = a.rowStart[row + 1];
        if (s == e) continue;
        const double *xr = a.X + row * a.ldx;
        double x[kR], acc[kR];
#pragma unroll
        for (int t = 0; t < kR; t++) {
            const int k = lane + 32 * t;
            x[t] = kS > 0 && k < r ? xr[k] : 0.0;
            acc[t] = 0.0;
        }
        double rl = 0.0, rc = 0.0;
        for (int64_t j = s; j < e; j++) {
            const int rho = relation_of(a.rel[j], a.nrel);
            if (rho == a.nrel) {
                if (lane == 0) {
                    if (a.scores) a.scores[j] = 0.0;
                    if (a.gout) a.gout[j] = 0.0;
                }
                continue;
            }
            const double *yr = a.Y + a.col_idx[j] * a.ldy, *dr = a.D + rho * a.ldd;
            double t = 0.0;
            if constexpr (kS > 0) {
#pragma unroll
                for (int q = 0; q < kS; q++)
                    if (lane + 32 * q < r) t = fma(x[q] * dr[lane + 32 * q], yr[lane + 32 * q], t);
            } else {
                for (int k = lane; k < r; k += 32) t = fma(xr[k] * dr[k], yr[k], t);
            }
            t = group_allreduce<32>(t, 0xffffffffu);
            const Bce b = bce(t, a.target, a.inv_count);
            rl += b.loss;
            rc += b.correct;
            if (lane == 0) {
                if (a.scores) a.scores[j] = t;
                if (a.gout) a.gout[j] = b.g;
            }
            if (!a.dX) continue;
            if constexpr (kS > 0) {
#pragma unroll
                for (int q = 0; q < kS; q++)
                    if (lane + 32 * q < r) acc[q] = fma(b.g, dr[lane + 32 * q] * yr[lane + 32 * q], acc[q]);
            } else {
                double *o = a.dX + row * a.lddx;
                for (int k = lane; k < r; k += 32) o[k] = fma(b.g, dr[k] * yr[k], o[k]);
            }
        }
        if constexpr (kS > 0) {
            if (a.dX) {
#pragma unroll
                for (int q = 0; q < kS; q++)
                    if (lane + 32 * q < r) a.dX[row * a.lddx + lane + 32 * q] += acc[q];
            }
        }
        if (a.stats && lane == 0) {
            a.stats[row * a.lds] += rl;
            a.stats[row * a.lds + 1] += rc;
        }
    }
}

// ---- relation-table gradient: one r-wide sum per piece of the relation grouping ----------------------------------
struct PieceArgs {
    const int32_t *perm, *key_start, *piece_first, *piece_key;
    int64_t pieces;
    int nrel;
    const int64_t *row_idx, *col_idx;
    const double *g;
    const double *X;
    int64_t ldx;
    const double *Y;
    int64_t ldy;
    double *partial;  // pieces x r
};

// the positions [lo, hi) in perm order of piece q, and its key
__device__ __forceinline__ int piece_range(const PieceArgs &a, int64_t q, int64_t *lo, int64_t *hi) {
    const int k = a.piece_key[q];
    *lo = (int64_t)a.key_start[k] + (q - (int64_t)a.piece_first[k]) * HNH_EDGE_PIECE;
    *hi = min(*lo + HNH_EDGE_PIECE, (int64_t)a.key_start[k + 1]);
    return k;
}

template <int R, int G, int VW, int UN>
__global__ void __launch_bounds__(kBlock, 1) distmult_piece_kernel(const PieceArgs a) {
    constexpr int NV = R / (G * VW);
    static_assert(NV * G * VW == R, "R must equal NV*G*VW");
    const uint64_t first = evict_first_policy();
    const int lane = threadIdx.x & 31;
    const int gl = lane & (G - 1);
    const unsigned gmask = group_mask<G>(lane);
    const int64_t ngroups = (int64_t)gridDim.x * (blockDim.x / G);
    for (int64_t q = (int64_t)blockIdx.x * (blockDim.x / G) + threadIdx.x / G; q < a.pieces; q += ngroups) {
        int64_t lo, hi;
        if (piece_range(a, q, &lo, &hi) == a.nrel) continue;  // the entries that are no relation
        double acc[NV][VW];
#pragma unroll
        for (int v = 0; v < NV; v++)
#pragma unroll
            for (int w = 0; w < VW; w++) acc[v][w] = 0.0;
        for (int64_t j = lo; j < hi; j += G) {
            const int cnt = (hi - j < G) ? (int)(hi - j) : G;
            int64_t myu = 0, myv = 0;
            double myg = 0.0;
            if (gl < cnt) {
                const int64_t i = a.perm[j + gl];
                myu = ld_first_i64(a.row_idx + i, first);
                myv = ld_first_i64(a.col_idx + i, first);
                myg = ld_first_f64(a.g + i, first);
            }
            for (int k0 = 0; k0 < cnt; k0 += UN) {
                double xu[UN][NV][VW], yv[UN][NV][VW], gk[UN];
#pragma unroll
                for (int u = 0; u < UN; u++) {
                    const int k = k0 + u;
                    const int src = k < G ? k : G - 1;
                    const int64_t ru = __shfl_sync(gmask, myu, src, G), cv = __shfl_sync(gmask, myv, src, G);
                    gk[u] = __shfl_sync(gmask, myg, src, G);
                    if (k < cnt) {
#pragma unroll
                        for (int v = 0; v < NV; v++) {
                            ld_gather<VW>(xu[u][v], a.X + ru * a.ldx + (v * G + gl) * VW);
                            ld_gather<VW>(yv[u][v], a.Y + cv * a.ldy + (v * G + gl) * VW);
                        }
                    }
                }
#pragma unroll
                for (int u = 0; u < UN; u++)
                    if (k0 + u < cnt) {
#pragma unroll
                        for (int v = 0; v < NV; v++)
#pragma unroll
                            for (int w = 0; w < VW; w++) acc[v][w] = fma(gk[u], xu[u][v][w] * yv[u][v][w], acc[v][w]);
                    }
            }
        }
#pragma unroll
        for (int v = 0; v < NV; v++) st_rw<VW>(a.partial + q * R + (v * G + gl) * VW, acc[v]);
    }
}

// one warp per piece; kS as in distmult_bce_generic_kernel (kS = 0: the partial row accumulates in memory)
template <int kS>
__global__ void __launch_bounds__(kBlock, 1) distmult_piece_generic_kernel(const PieceArgs a, int r) {
    constexpr int kR = kS > 0 ? kS : 1;
    const int lane = threadIdx.x & 31;
    const int64_t warps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t q = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; q < a.pieces; q += warps) {
        int64_t lo, hi;
        if (piece_range(a, q, &lo, &hi) == a.nrel) continue;
        double *out = a.partial + q * r;
        double acc[kR];
#pragma unroll
        for (int t = 0; t < kR; t++) acc[t] = 0.0;
        if constexpr (kS == 0)
            for (int k = lane; k < r; k += 32) out[k] = 0.0;
        for (int64_t j = lo; j < hi; j++) {
            const int64_t i = a.perm[j];
            const double *xr = a.X + a.row_idx[i] * a.ldx, *yr = a.Y + a.col_idx[i] * a.ldy;
            const double g = a.g[i];
            if constexpr (kS > 0) {
#pragma unroll
                for (int t = 0; t < kS; t++)
                    if (lane + 32 * t < r) acc[t] = fma(g, xr[lane + 32 * t] * yr[lane + 32 * t], acc[t]);
            } else {
                for (int k = lane; k < r; k += 32) out[k] = fma(g, xr[k] * yr[k], out[k]);
            }
        }
        if constexpr (kS > 0) {
#pragma unroll
            for (int t = 0; t < kS; t++)
                if (lane + 32 * t < r) out[lane + 32 * t] = acc[t];
        }
    }
}

// dD[k, c] += the sum of partial[q, c] over the pieces q of key k < nrel, in plan order: CTA (column tile, key); warp w
// takes the key's pieces w, w + 8, .. for the tile's 32 columns, then the 8 warp sums are added in warp order
constexpr int kSumWarps = kBlock / 32;
__global__ void __launch_bounds__(kBlock) distmult_key_sum_kernel(const int32_t *__restrict__ piece_first, const double *__restrict__ partial,
                                                                  int r, double *__restrict__ dD, int64_t ldd) {
    __shared__ double sh[kSumWarps][32];
    const int key = blockIdx.y, lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    const int col = blockIdx.x * 32 + lane;
    const int64_t q0 = piece_first[key], q1 = piece_first[key + 1];
    double t = 0.0;
    if (col < r)
        for (int64_t q = q0 + w; q < q1; q += kSumWarps) t += partial[q * r + col];
    sh[w][lane] = t;
    __syncthreads();
    if (w == 0 && col < r) {
        double s = 0.0;
#pragma unroll
        for (int i = 0; i < kSumWarps; i++) s += sh[i][lane];
        dD[(int64_t)key * ldd + col] += s;
    }
}

int launch_bce(const char *who, const BceArgs &a, int64_t nnz, int r, cudaStream_t st) {
    if (a.rows < 0 || nnz < 0) return set_error(HNH_E_INVALID, "%s: negative size", who);
    if (r < 1) return set_error(HNH_E_INVALID, "%s: r must be positive (got %d)", who, r);
    if (a.nrel < 1) return set_error(HNH_E_INVALID, "%s: the relation count must be positive (got %d)", who, a.nrel);
    if (a.ldx < r || a.ldy < r || a.ldd < r || (a.dX && a.lddx < r))
        return set_error(HNH_E_INVALID, "%s: a leading dimension is below r = %d", who, r);
    if (a.stats && a.lds < 2) return set_error(HNH_E_INVALID, "%s: the stats' leading dimension is below 2", who);
    if (!(a.inv_count >= 0.0) || !std::isfinite(a.inv_count))
        return set_error(HNH_E_INVALID, "%s: inv_count must be finite and >= 0", who);
    if (!(a.target >= 0.0 && a.target <= 1.0)) return set_error(HNH_E_INVALID, "%s: the target must lie in [0, 1]", who);
    if (a.rows == 0 || nnz == 0) return HNH_OK;
    if (!a.rowStart || !a.col_idx || !a.rel || !a.X || !a.Y || !a.D) return set_error(HNH_E_INVALID, "%s: null pointer", who);
    const void *outs[] = {a.dX, a.stats, a.scores, a.gout};
    const void *ins[] = {a.X, a.Y, a.D, a.rel};
    for (const void *o : outs)
        for (const void *i : ins)
            if (o && o == i) return set_error(HNH_E_INVALID, "%s: an output may not be an input", who);
    for (int i = 0; i < 4; i++)
        for (int k = i + 1; k < 4; k++)
            if (outs[i] && outs[i] == outs[k]) return set_error(HNH_E_INVALID, "%s: the outputs must be distinct", who);
    int grid = 0, rc = HNH_OK;
    if (table_width(r) && aligned16(a.X) && aligned16(a.Y) && aligned16(a.D) && a.ldx % 2 == 0 && a.ldy % 2 == 0 && a.ldd % 2 == 0 &&
        (!a.dX || (aligned16(a.dX) && a.lddx % 2 == 0))) {
#define DB(RR, G, VW, UN)                                                                   \
    {                                                                                       \
        auto k = distmult_bce_kernel<RR, G, VW, UN>;                                        \
        rc = grid_for(k, a.rows, kBlock / G, &grid);                                        \
        if (!rc) rc = launch(k, grid, kBlock, st, "distmult_bce_kernel", a);                \
    }
        HNH_DISPATCH_R(r, DB, )
#undef DB
        return rc;
    }
    auto k = r <= 32 ? distmult_bce_generic_kernel<1> : r <= 64 ? distmult_bce_generic_kernel<2> : r <= 128 ? distmult_bce_generic_kernel<4>
           : r <= 256 ? distmult_bce_generic_kernel<8> : distmult_bce_generic_kernel<0>;
    rc = grid_for(k, a.rows, kBlock / 32, &grid);
    return rc ? rc : launch(k, grid, kBlock, st, "distmult_bce_generic_kernel", a, r);
}

}  // namespace

extern "C" {

int hnh_distmult_bce_f64(const int64_t *rowStart, const int64_t *col_idx, const double *values, int64_t rows, int64_t nnz, int R,
                         const double *X, int64_t ldx, const double *Y, int64_t ldy, const double *D, int64_t ldd, int r,
                         double target, double inv_count, double *dX, int64_t lddx, double *stats, int64_t lds, double *scores,
                         double *g, void *stream) {
    return launch_bce("hnh_distmult_bce_f64",
                      {rowStart, col_idx, values, rows, R, X, ldx, Y, ldy, D, ldd, target, inv_count, dX, lddx, stats, lds, scores, g},
                      nnz, r, (cudaStream_t)stream);
}

int hnh_distmult_bce_grad_f64(const int64_t *rowStart, const int64_t *col_idx, const double *values, int64_t rows, int64_t nnz,
                              int R, const double *X, int64_t ldx, const double *Y, int64_t ldy, const double *D, int64_t ldd, int r,
                              double target, double inv_count, double *dX, int64_t lddx, void *stream) {
    if (!dX) return set_error(HNH_E_INVALID, "hnh_distmult_bce_grad_f64: null dX");
    return launch_bce("hnh_distmult_bce_grad_f64",
                      {rowStart, col_idx, values, rows, R, X, ldx, Y, ldy, D, ldd, target, inv_count, dX, lddx, nullptr, 2, nullptr,
                       nullptr},
                      nnz, r, (cudaStream_t)stream);
}

int hnh_distmult_relation_grad_f64(const int32_t *perm, const int32_t *key_start, const int32_t *piece_first, const int32_t *piece_key,
                                   int64_t num_pieces, int R, const int64_t *row_idx, const int64_t *col_idx, const double *g,
                                   const double *X, int64_t ldx, const double *Y, int64_t ldy, int r, double *partial, double *dD,
                                   int64_t ldd, void *stream) {
    const char *who = "hnh_distmult_relation_grad_f64";
    if (num_pieces < 0) return set_error(HNH_E_INVALID, "%s: negative size", who);
    if (r < 1 || R < 1) return set_error(HNH_E_INVALID, "%s: r and R must be positive (got %d, %d)", who, r, R);
    if (ldx < r || ldy < r || ldd < r) return set_error(HNH_E_INVALID, "%s: a leading dimension is below r = %d", who, r);
    if (num_pieces == 0) return HNH_OK;
    if (!perm || !key_start || !piece_first || !piece_key || !row_idx || !col_idx || !g || !X || !Y || !partial || !dD)
        return set_error(HNH_E_INVALID, "%s: null pointer", who);
    if (partial == X || partial == Y || partial == dD || dD == X || dD == Y || dD == g)
        return set_error(HNH_E_INVALID, "%s: an output may not be an input or another output", who);
    cudaStream_t st = (cudaStream_t)stream;
    const PieceArgs a{perm, key_start, piece_first, piece_key, num_pieces, R, row_idx, col_idx, g, X, ldx, Y, ldy, partial};
    int grid = 0, rc = HNH_OK;
    if (table_width(r) && aligned16(X) && aligned16(Y) && aligned16(partial) && ldx % 2 == 0 && ldy % 2 == 0) {
#define DP(RR, G, VW, UN)                                                                   \
    {                                                                                       \
        auto k = distmult_piece_kernel<RR, G, VW, UN>;                                      \
        rc = grid_for(k, num_pieces, kBlock / G, &grid);                                    \
        if (!rc) rc = launch(k, grid, kBlock, st, "distmult_piece_kernel", a);              \
    }
        HNH_DISPATCH_R(r, DP, )
#undef DP
    } else {
        auto k = r <= 32 ? distmult_piece_generic_kernel<1> : r <= 64 ? distmult_piece_generic_kernel<2>
               : r <= 128 ? distmult_piece_generic_kernel<4> : r <= 256 ? distmult_piece_generic_kernel<8> : distmult_piece_generic_kernel<0>;
        rc = grid_for(k, num_pieces, kBlock / 32, &grid);
        if (!rc) rc = launch(k, grid, kBlock, st, "distmult_piece_generic_kernel", a, r);
    }
    if (rc) return rc;
    const dim3 sum_grid((unsigned)((r + 31) / 32), (unsigned)R);
    return launch(distmult_key_sum_kernel, sum_grid, kBlock, st, "distmult_key_sum_kernel", piece_first, (const double *)partial, r, dD, ldd);
}

}  // extern "C"
