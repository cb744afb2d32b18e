// rgcn.cu -- relation-typed neighbour aggregation (Distributed_Sparse::relationalAggregate, include/hnh/rgcn.hpp) on one
// CSR block.  The block's stored value of an entry is its relation rho (an integer in [0, R)); with Y the gathered side
// (indexed by col_idx) and u the stored row:
//     aggregate:  A[u, rho f + k] += sum_{v : rel(u, v) = rho} X[v, k]         (A order: A's rows stored, X gathered)
//     grad:       dX[v, k]        += sum_u dA[u, rel(v, u) f + k]               (B order: X's rows stored, dA gathered)
// An entry whose value is not an integer in [0, R) (negative, >= R, fractional, infinite, NaN) contributes nothing and
// its gathered row is never read.
//
// The fast kernels follow max_aggregate_*_kernel (graph_sage.cu): a group of G lanes owns one CSR row; a chunk of G
// (column, value) pairs is read coalesced and broadcast by shuffles; gathered rows come in with 128-bit loads, UN rows in
// flight per lane.  The aggregate sweeps the relations present in the row in increasing order: each sweep gathers the
// row's entries of one relation (found by a ballot over the chunk, in stored order), sums them in registers and adds the
// sum to A's (row, relation) window with one read-modify-write, and finds the next relation as the smallest one above
// the current.  So every (row, relation) window with entries is read and written once per call, whatever the order of
// the entries, and a row's windows without entries are not touched (A may ride a ring and carry earlier blocks' sums).
// The sweeps re-read the row's index and value chunks (L1 / L2 hits; the first chunk stays in registers); the gathers,
// the bulk of the traffic, happen once per entry.  The grad is the accumulating SpMM with a per-entry column offset
// rel f in the gathered row: sums in registers in stored order, one read-modify-write of dX at the row end.  Widths
// 4..256 (powers of two) with 16-byte aligned operands, even leading dimensions and an even f take them; every other
// window takes the one-warp-per-row generic kernel.  Wider rows run as column windows of 256.  No atomics anywhere:
// repeated calls are bit-identical.
//
// With basis decomposition (Distributed_Sparse::basisAggregate) the entries are summed into one window per basis, with
// per-entry, per-basis coefficients, instead of one per relation; see "basis aggregation" below.
#include <cmath>

#include "row_gather.cuh"

namespace {

using hnh::grid_for;
using hnh::launch;
using hnh::set_error;

constexpr int kWindow = 256;  // the widest column window of one launch

// the relation of a stored value, or nrel for a value that is not an integer in [0, nrel)
__device__ __forceinline__ int relation_of(double v, int nrel) {
    return (v >= 0.0 && v < (double)nrel && v == trunc(v)) ? (int)v : nrel;
}
// the minimum over the group, on every lane of it
template <int G>
__device__ __forceinline__ int group_min(int x, unsigned mask) {
#pragma unroll
    for (int o = G / 2; o > 0; o >>= 1) x = min(x, __shfl_xor_sync(mask, x, o, G));
    return x;
}

// ---- fast row kernels ------------------------------------------------------------------------------------------------
// rstride: the distance between two relations' windows in A (the full f; the launch covers one column window of it)
template <int RW, int G, int VW, int UN>
__global__ void __launch_bounds__(kBlock, 1)
relational_aggregate_kernel(const int64_t *__restrict__ rowStart, const int64_t *__restrict__ col_idx,
                            const double *__restrict__ values, int64_t rows, const double *__restrict__ X, int64_t ldx,
                            int nrel, int64_t rstride, double *__restrict__ A, int64_t lda) {
    constexpr int NV = RW / (G * VW);
    static_assert(NV * G * VW == RW, "RW must equal NV*G*VW");
    const int lane = threadIdx.x & 31;
    const int gl = lane & (G - 1);
    const int gbase = lane & ~(G - 1);
    const unsigned gmask = group_mask<G>(lane);
    const int64_t ngroups = (int64_t)gridDim.x * (blockDim.x / G);
    for (int64_t row = (int64_t)blockIdx.x * (blockDim.x / G) + threadIdx.x / G; row < rows; row += ngroups) {
        const int64_t s = ld_stream_i64(rowStart + row);
        const int64_t e = ld_stream_i64(rowStart + row + 1);
        if (s == e) continue;  // nothing to add
        // the first chunk stays in registers across the sweeps
        const int cnt0 = (e - s < G) ? (int)(e - s) : G;
        const int64_t col0 = gl < cnt0 ? ld_stream_i64(col_idx + s + gl) : 0;
        const int rel0 = gl < cnt0 ? relation_of(__ldg(values + s + gl), nrel) : nrel;
        int cur = rel0;
        for (int64_t j = s + G; j < e; j += G)
            if (gl < e - j) cur = min(cur, relation_of(__ldg(values + j + gl), nrel));
        cur = group_min<G>(cur, gmask);
        while (cur < nrel) {
            double acc[NV][VW];
#pragma unroll
            for (int v = 0; v < NV; v++)
#pragma unroll
                for (int w = 0; w < VW; w++) acc[v][w] = 0.0;
            int nxt = nrel;
            for (int64_t j = s; j < e; j += G) {
                const int cnt = (e - j < G) ? (int)(e - j) : G;
                int64_t mycol = col0;
                int myrel = rel0;
                if (j != s) {
                    mycol = gl < cnt ? __ldg(col_idx + j + gl) : 0;
                    myrel = gl < cnt ? relation_of(__ldg(values + j + gl), nrel) : nrel;
                }
                if (myrel > cur) nxt = min(nxt, myrel);
                // the chunk's entries of relation `cur`, in stored order (lanes past cnt hold nrel)
                unsigned m = __ballot_sync(gmask, myrel == cur) >> gbase;
                while (m) {
                    const int nb = __popc(m) < UN ? __popc(m) : UN;
                    double y[UN][NV][VW];
#pragma unroll
                    for (int u = 0; u < UN; u++) {
                        const int k = m ? __ffs(m) - 1 : 0;
                        m &= m - 1;
                        const int64_t col = __shfl_sync(gmask, mycol, k, G);
                        if (u < nb) {
#pragma unroll
                            for (int v = 0; v < NV; v++) ld_gather<VW>(y[u][v], X + col * ldx + (v * G + gl) * VW);
                        } else {
#pragma unroll
                            for (int v = 0; v < NV; v++)
#pragma unroll
                                for (int w = 0; w < VW; w++) y[u][v][w] = 0.0;
                        }
                    }
#pragma unroll
                    for (int u = 0; u < UN; u++)
                        if (u < nb) {
#pragma unroll
                            for (int v = 0; v < NV; v++)
#pragma unroll
                                for (int w = 0; w < VW; w++) acc[v][w] += y[u][v][w];
                        }
                }
            }
#pragma unroll
            for (int v = 0; v < NV; v++) {
                double o[VW];
                double *p = A + row * lda + cur * rstride + (v * G + gl) * VW;
                ld_rw<VW>(o, p);
#pragma unroll
                for (int w = 0; w < VW; w++) o[w] += acc[v][w];
                st_rw<VW>(p, o);
            }
            cur = group_min<G>(nxt, gmask);
        }
    }
}

template <int RW, int G, int VW, int UN>
__global__ void __launch_bounds__(kBlock, 1)
relational_aggregate_grad_kernel(const int64_t *__restrict__ rowStart, const int64_t *__restrict__ col_idx,
                                 const double *__restrict__ values, int64_t rows, const double *__restrict__ dA, int64_t ldda,
                                 int nrel, int64_t rstride, double *__restrict__ dX, int64_t lddx) {
    constexpr int NV = RW / (G * VW);
    static_assert(NV * G * VW == RW, "RW must equal NV*G*VW");
    const int lane = threadIdx.x & 31;
    const int gl = lane & (G - 1);
    const unsigned gmask = group_mask<G>(lane);
    const int64_t ngroups = (int64_t)gridDim.x * (blockDim.x / G);
    for (int64_t row = (int64_t)blockIdx.x * (blockDim.x / G) + threadIdx.x / G; row < rows; row += ngroups) {
        const int64_t s = ld_stream_i64(rowStart + row);
        const int64_t e = ld_stream_i64(rowStart + row + 1);
        if (s == e) continue;  // nothing to add
        double acc[NV][VW];
#pragma unroll
        for (int v = 0; v < NV; v++)
#pragma unroll
            for (int w = 0; w < VW; w++) acc[v][w] = 0.0;
        for (int64_t j = s; j < e; j += G) {
            const int cnt = (e - j < G) ? (int)(e - j) : G;
            // the gathered row's window of this entry's relation, or -1 for an entry without a valid relation
            int64_t myoff = -1;
            if (gl < cnt) {
                const int rel = relation_of(ld_stream_f64(values + j + gl), nrel);
                if (rel < nrel) myoff = ld_stream_i64(col_idx + j + gl) * ldda + rel * rstride;
            }
            for (int k0 = 0; k0 < cnt; k0 += UN) {
                double y[UN][NV][VW];
                bool on[UN];
#pragma unroll
                for (int u = 0; u < UN; u++) {
                    const int k = k0 + u;
                    const int64_t off = __shfl_sync(gmask, myoff, k < G ? k : G - 1, G);
                    on[u] = k < cnt && off >= 0;
                    if (on[u]) {
#pragma unroll
                        for (int v = 0; v < NV; v++) ld_gather<VW>(y[u][v], dA + off + (v * G + gl) * VW);
                    } else {
#pragma unroll
                        for (int v = 0; v < NV; v++)
#pragma unroll
                            for (int w = 0; w < VW; w++) y[u][v][w] = 0.0;
                    }
                }
#pragma unroll
                for (int u = 0; u < UN; u++)
                    if (on[u]) {
#pragma unroll
                        for (int v = 0; v < NV; v++)
#pragma unroll
                            for (int w = 0; w < VW; w++) acc[v][w] += y[u][v][w];
                    }
            }
        }
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
}

// ---- generic kernels: any window width up to 256, any leading dimension, any alignment; one warp per row ---------------
// Lane l keeps columns l + 32 t (t < kS) of the row's sum in registers, f <= 32 kS.
template <int kS>
__global__ void __launch_bounds__(kBlock, 1)
relational_aggregate_generic_kernel(const int64_t *__restrict__ rowStart, const int64_t *__restrict__ col_idx,
                                    const double *__restrict__ values, int64_t rows, const double *__restrict__ X, int64_t ldx,
                                    int f, int nrel, int64_t rstride, double *__restrict__ A, int64_t lda) {
    const int lane = threadIdx.x & 31;
    const int64_t warps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t row = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; row < rows; row += warps) {
        const int64_t s = rowStart[row], e = rowStart[row + 1];
        if (s == e) continue;
        int cur = nrel;
        for (int64_t j = s + lane; j < e; j += 32) cur = min(cur, relation_of(values[j], nrel));
        cur = group_min<32>(cur, 0xffffffffu);
        while (cur < nrel) {
            double acc[kS];
#pragma unroll
            for (int t = 0; t < kS; t++) acc[t] = 0.0;
            int nxt = nrel;
            for (int64_t j0 = s; j0 < e; j0 += 32) {
                const int64_t j = j0 + lane;
                const int rel = j < e ? relation_of(values[j], nrel) : nrel;
                const int64_t col = j < e ? col_idx[j] : 0;
                if (rel > cur) nxt = min(nxt, rel);
                unsigned m = __ballot_sync(0xffffffffu, rel == cur);
                while (m) {
                    const int k = __ffs(m) - 1;
                    m &= m - 1;
                    const double *yr = X + __shfl_sync(0xffffffffu, col, k) * ldx;
#pragma unroll
                    for (int t = 0; t < kS; t++)
                        if (lane + 32 * t < f) acc[t] += yr[lane + 32 * t];
                }
            }
            double *o = A + row * lda + cur * rstride;
#pragma unroll
            for (int t = 0; t < kS; t++)
                if (lane + 32 * t < f) o[lane + 32 * t] += acc[t];
            cur = group_min<32>(nxt, 0xffffffffu);
        }
    }
}

template <int kS>
__global__ void __launch_bounds__(kBlock, 1)
relational_aggregate_grad_generic_kernel(const int64_t *__restrict__ rowStart, const int64_t *__restrict__ col_idx,
                                         const double *__restrict__ values, int64_t rows, const double *__restrict__ dA,
                                         int64_t ldda, int f, int nrel, int64_t rstride, double *__restrict__ dX, int64_t lddx) {
    const int lane = threadIdx.x & 31;
    const int64_t warps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t row = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; row < rows; row += warps) {
        const int64_t s = rowStart[row], e = rowStart[row + 1];
        if (s == e) continue;
        double acc[kS];
#pragma unroll
        for (int t = 0; t < kS; t++) acc[t] = 0.0;
        for (int64_t j = s; j < e; j++) {
            const int rel = relation_of(values[j], nrel);
            if (rel == nrel) continue;
            const double *yr = dA + col_idx[j] * ldda + rel * rstride;
#pragma unroll
            for (int t = 0; t < kS; t++)
                if (lane + 32 * t < f) acc[t] += yr[lane + 32 * t];
        }
#pragma unroll
        for (int t = 0; t < kS; t++)
            if (lane + 32 * t < f) dX[row * lddx + lane + 32 * t] += acc[t];
    }
}

// ---- per-window scale and the relation check -------------------------------------------------------------------------
// A[u, rho f + k] = C[u, rho] == 0 ? 0 : A[u, rho f + k] / C[u, rho]; one warp per row
__global__ void __launch_bounds__(kBlock, 1)
window_scale_kernel(double *__restrict__ A, int64_t lda, const double *__restrict__ C, int64_t ldc, int64_t n, int f, int nrel) {
    const int lane = threadIdx.x & 31;
    const int width = f * nrel;
    const int64_t warps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t row = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; row < n; row += warps) {
        double *a = A + row * lda;
        const double *c = C + row * ldc;
        for (int k = lane; k < width; k += 32) {
            const double cnt = c[k / f];
            a[k] = cnt == 0.0 ? 0.0 : a[k] / cnt;
        }
    }
}

// bad[0] += the number of v[i] that are not integers in [0, nrel) (NaN and infinities included): one CTA, a fixed order
__global__ void __launch_bounds__(kBlock) relation_check_kernel(double *__restrict__ bad, const double *__restrict__ v, int64_t n,
                                                                int nrel) {
    __shared__ double sh[kBlock / 32];
    double c = 0.0;
    for (int64_t i = threadIdx.x; i < n; i += kBlock) c += relation_of(v[i], nrel) < nrel ? 0.0 : 1.0;
    c = group_allreduce<32>(c, 0xffffffffu);
    if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = c;
    __syncthreads();
    if (threadIdx.x == 0) {
        double t = 0.0;
        for (int w = 0; w < kBlock / 32; w++) t += sh[w];
        bad[0] += t;
    }
}

// ---- basis aggregation (R-GCN with basis decomposition) --------------------------------------------------------------
// With comp the R x B coefficients (row-major) and w(u, rho) = scale[u, rho] (1 without a scale):
//     aggregate:  H[u, b f + k] += sum_{entries (v, rho) of row u} w(u, rho) comp[rho, b] X[v, k]     (A order)
//     grad:       dX[v, k] += sum_{entries (u, rho) of row v} w(u, rho) sum_b comp[rho, b] dH[u, b f + k]   (B order)
//                 P[b ldp + j] (= or +=) w(u, rho) <dH[u, b f .. b f + f), X[v, ..)> for entry j   (optional)
// The aggregate keeps up to NB bases' sums of the row in registers and gathers each entry's row once per chunk of NB
// bases; every H window of the chunk is read and written once per call.  The grad sums one basis at a time into one
// register row, gathering dH[u, b f ..] for UN entries at once, and reduces each entry's dot over the group for P.
// Entries that are not relations are skipped (their P is 0).  Column windows of 256 run as separate launches; the
// grad's P is written by the first window and added to by the others.

// the accumulator doubles per lane the fast aggregate keeps: NB = kBasisAcc / (RW / G) bases in registers
constexpr int kBasisAcc = 32;

template <int RW, int G, int VW, int UN, int NB>
__global__ void __launch_bounds__(kBlock, 1)
basis_aggregate_kernel(const int64_t *__restrict__ rowStart, const int64_t *__restrict__ col_idx, const double *__restrict__ values,
                       int64_t rows, const double *__restrict__ X, int64_t ldx, const double *scale, int64_t lds,
                       const double *__restrict__ comp, int nrel, int nbases, int64_t bstride, double *H, int64_t ldh) {
    constexpr int NV = RW / (G * VW);
    static_assert(NV * G * VW == RW, "RW must equal NV*G*VW");
    const int lane = threadIdx.x & 31;
    const int gl = lane & (G - 1);
    const int gbase = lane & ~(G - 1);
    const unsigned gmask = group_mask<G>(lane);
    const int64_t ngroups = (int64_t)gridDim.x * (blockDim.x / G);
    for (int64_t row = (int64_t)blockIdx.x * (blockDim.x / G) + threadIdx.x / G; row < rows; row += ngroups) {
        const int64_t s = ld_stream_i64(rowStart + row);
        const int64_t e = ld_stream_i64(rowStart + row + 1);
        if (s == e) continue;  // nothing to add
        for (int b0 = 0; b0 < nbases; b0 += NB) {
            const int nb = nbases - b0 < NB ? nbases - b0 : NB;
            double acc[NB][NV][VW];
#pragma unroll
            for (int b = 0; b < NB; b++)
#pragma unroll
                for (int v = 0; v < NV; v++)
#pragma unroll
                    for (int w = 0; w < VW; w++) acc[b][v][w] = 0.0;
            for (int64_t j = s; j < e; j += G) {
                const int cnt = (e - j < G) ? (int)(e - j) : G;
                int64_t mycol = 0;
                int myrel = nrel;
                double myw = 0.0;
                if (gl < cnt) {
                    myrel = relation_of(__ldg(values + j + gl), nrel);
                    if (myrel < nrel) {
                        mycol = __ldg(col_idx + j + gl);
                        myw = scale ? scale[row * lds + myrel] : 1.0;
                    }
                }
                // the chunk's entries that are relations, in stored order
                unsigned m = __ballot_sync(gmask, myrel < nrel) >> gbase;
                while (m) {
                    const int nt = __popc(m) < UN ? __popc(m) : UN;
                    double y[UN][NV][VW];
                    const double *cr[UN];
                    double wt[UN];
#pragma unroll
                    for (int u = 0; u < UN; u++) {
                        const int k = m ? __ffs(m) - 1 : 0;
                        m &= m - 1;
                        const int64_t col = __shfl_sync(gmask, mycol, k, G);
                        cr[u] = comp + (int64_t)__shfl_sync(gmask, myrel, k, G) * nbases + b0;
                        wt[u] = __shfl_sync(gmask, myw, k, G);
                        if (u < nt) {
#pragma unroll
                            for (int v = 0; v < NV; v++) ld_gather<VW>(y[u][v], X + col * ldx + (v * G + gl) * VW);
                        }
                    }
#pragma unroll
                    for (int u = 0; u < UN; u++)
                        if (u < nt) {
#pragma unroll
                            for (int b = 0; b < NB; b++)
                                if (b < nb) {
                                    const double c = wt[u] * __ldg(cr[u] + b);
#pragma unroll
                                    for (int v = 0; v < NV; v++)
#pragma unroll
                                        for (int w = 0; w < VW; w++) acc[b][v][w] = fma(c, y[u][v][w], acc[b][v][w]);
                                }
                        }
                }
            }
#pragma unroll
            for (int b = 0; b < NB; b++)
                if (b < nb) {
#pragma unroll
                    for (int v = 0; v < NV; v++) {
                        double o[VW];
                        double *p = H + row * ldh + (b0 + b) * bstride + (v * G + gl) * VW;
                        ld_rw<VW>(o, p);
#pragma unroll
                        for (int w = 0; w < VW; w++) o[w] += acc[b][v][w];
                        st_rw<VW>(p, o);
                    }
                }
        }
    }
}

template <int RW, int G, int VW, int UN>
__global__ void __launch_bounds__(kBlock, 1)
basis_aggregate_grad_kernel(const int64_t *__restrict__ rowStart, const int64_t *__restrict__ col_idx,
                            const double *__restrict__ values, int64_t rows, const double *__restrict__ dH, int64_t lddh,
                            const double *__restrict__ scale, int64_t lds, const double *__restrict__ comp, int nrel, int nbases,
                            int64_t bstride, const double *X, int64_t ldx, double *dX, int64_t lddx, double *P, int64_t ldp,
                            int p_add) {
    constexpr int NV = RW / (G * VW);
    static_assert(NV * G * VW == RW, "RW must equal NV*G*VW");
    const int lane = threadIdx.x & 31;
    const int gl = lane & (G - 1);
    const unsigned gmask = group_mask<G>(lane);
    const int64_t ngroups = (int64_t)gridDim.x * (blockDim.x / G);
    for (int64_t row = (int64_t)blockIdx.x * (blockDim.x / G) + threadIdx.x / G; row < rows; row += ngroups) {
        const int64_t s = ld_stream_i64(rowStart + row);
        const int64_t e = ld_stream_i64(rowStart + row + 1);
        if (s == e) continue;  // nothing to add
        double acc[NV][VW], x[NV][VW];
#pragma unroll
        for (int v = 0; v < NV; v++)
#pragma unroll
            for (int w = 0; w < VW; w++) acc[v][w] = x[v][w] = 0.0;
        if (P) {
#pragma unroll
            for (int v = 0; v < NV; v++) ld_gather<VW>(x[v], X + row * ldx + (v * G + gl) * VW);
        }
        for (int64_t j = s; j < e; j += G) {
            const int cnt = (e - j < G) ? (int)(e - j) : G;
            // this lane's entry: the gathered row's offset (-1 for an entry that is not a relation), its relation and weight
            int64_t myoff = -1;
            int myrel = 0;
            double myw = 0.0;
            if (gl < cnt) {
                const int rel = relation_of(ld_stream_f64(values + j + gl), nrel);
                if (rel < nrel) {
                    const int64_t u = ld_stream_i64(col_idx + j + gl);
                    myoff = u * lddh;
                    myrel = rel;
                    myw = scale ? __ldg(scale + u * lds + rel) : 1.0;
                }
            }
            for (int b = 0; b < nbases; b++) {
                double myp = 0.0;  // P of this lane's entry for basis b
                for (int k0 = 0; k0 < cnt; k0 += UN) {
                    double y[UN][NV][VW];
                    double c[UN], wt[UN];
                    bool on[UN];
#pragma unroll
                    for (int u = 0; u < UN; u++) {
                        const int k = k0 + u < G ? k0 + u : G - 1;
                        const int64_t off = __shfl_sync(gmask, myoff, k, G);
                        const int rel = __shfl_sync(gmask, myrel, k, G);
                        wt[u] = __shfl_sync(gmask, myw, k, G);
                        on[u] = k0 + u < cnt && off >= 0;
                        c[u] = 0.0;
                        if (on[u]) {
                            c[u] = wt[u] * __ldg(comp + (int64_t)rel * nbases + b);
#pragma unroll
                            for (int v = 0; v < NV; v++) ld_gather<VW>(y[u][v], dH + off + b * bstride + (v * G + gl) * VW);
                        }
                    }
#pragma unroll
                    for (int u = 0; u < UN; u++) {
                        double d = 0.0;
                        if (on[u]) {
#pragma unroll
                            for (int v = 0; v < NV; v++)
#pragma unroll
                                for (int w = 0; w < VW; w++) {
                                    acc[v][w] = fma(c[u], y[u][v][w], acc[v][w]);
                                    d = fma(y[u][v][w], x[v][w], d);
                                }
                        }
                        if (P && k0 + u < cnt) {
                            d = group_allreduce<G>(d, gmask) * wt[u];
                            if (gl == k0 + u) myp = d;
                        }
                    }
                }
                if (P && gl < cnt) {
                    double *q = P + b * ldp + j + gl;
                    *q = p_add ? *q + myp : myp;
                }
            }
        }
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
}

// one warp per row, any window width up to 256, leading dimension and alignment: lane l keeps columns l + 32 t (t < kS)
// of NB bases' sums
template <int kS, int NB>
__global__ void __launch_bounds__(kBlock, 1)
basis_aggregate_generic_kernel(const int64_t *__restrict__ rowStart, const int64_t *__restrict__ col_idx,
                               const double *__restrict__ values, int64_t rows, const double *__restrict__ X, int64_t ldx, int f,
                               const double *scale, int64_t lds, const double *__restrict__ comp, int nrel, int nbases,
                               int64_t bstride, double *H, int64_t ldh) {
    const int lane = threadIdx.x & 31;
    const int64_t warps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t row = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; row < rows; row += warps) {
        const int64_t s = rowStart[row], e = rowStart[row + 1];
        if (s == e) continue;
        for (int b0 = 0; b0 < nbases; b0 += NB) {
            const int nb = nbases - b0 < NB ? nbases - b0 : NB;
            double acc[NB][kS];
#pragma unroll
            for (int b = 0; b < NB; b++)
#pragma unroll
                for (int t = 0; t < kS; t++) acc[b][t] = 0.0;
            for (int64_t j = s; j < e; j++) {
                const int rel = relation_of(values[j], nrel);
                if (rel == nrel) continue;
                const double wt = scale ? scale[row * lds + rel] : 1.0;
                const double *yr = X + col_idx[j] * ldx;
                double y[kS];
#pragma unroll
                for (int t = 0; t < kS; t++) y[t] = lane + 32 * t < f ? yr[lane + 32 * t] : 0.0;
#pragma unroll
                for (int b = 0; b < NB; b++)
                    if (b < nb) {
                        const double c = wt * comp[(int64_t)rel * nbases + b0 + b];
#pragma unroll
                        for (int t = 0; t < kS; t++) acc[b][t] = fma(c, y[t], acc[b][t]);
                    }
            }
#pragma unroll
            for (int b = 0; b < NB; b++)
                if (b < nb) {
                    double *o = H + row * ldh + (b0 + b) * bstride;
#pragma unroll
                    for (int t = 0; t < kS; t++)
                        if (lane + 32 * t < f) o[lane + 32 * t] += acc[b][t];
                }
        }
    }
}

template <int kS>
__global__ void __launch_bounds__(kBlock, 1)
basis_aggregate_grad_generic_kernel(const int64_t *__restrict__ rowStart, const int64_t *__restrict__ col_idx,
                                    const double *__restrict__ values, int64_t rows, const double *__restrict__ dH, int64_t lddh,
                                    const double *__restrict__ scale, int64_t lds, const double *__restrict__ comp, int nrel,
                                    int nbases, int64_t bstride, const double *X, int64_t ldx, int f, double *dX, int64_t lddx,
                                    double *P, int64_t ldp, int p_add) {
    const int lane = threadIdx.x & 31;
    const int64_t warps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t row = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; row < rows; row += warps) {
        const int64_t s = rowStart[row], e = rowStart[row + 1];
        if (s == e) continue;
        double acc[kS], x[kS];
#pragma unroll
        for (int t = 0; t < kS; t++) {
            acc[t] = 0.0;
            x[t] = P && lane + 32 * t < f ? X[row * ldx + lane + 32 * t] : 0.0;
        }
        for (int64_t j = s; j < e; j++) {
            const int rel = relation_of(values[j], nrel);
            if (rel == nrel) {
                if (P && lane == 0 && !p_add)
                    for (int b = 0; b < nbases; b++) P[b * ldp + j] = 0.0;
                continue;
            }
            const int64_t u = col_idx[j];
            const double wt = scale ? scale[u * lds + rel] : 1.0;
            for (int b = 0; b < nbases; b++) {
                const double c = wt * comp[(int64_t)rel * nbases + b];
                const double *yr = dH + u * lddh + b * bstride;
                double d = 0.0;
#pragma unroll
                for (int t = 0; t < kS; t++)
                    if (lane + 32 * t < f) {
                        const double y = yr[lane + 32 * t];
                        acc[t] = fma(c, y, acc[t]);
                        d = fma(y, x[t], d);
                    }
                if (P) {
                    d = group_allreduce<32>(d, 0xffffffffu) * wt;
                    if (lane == 0) P[b * ldp + j] = p_add ? P[b * ldp + j] + d : d;
                }
            }
        }
#pragma unroll
        for (int t = 0; t < kS; t++)
            if (lane + 32 * t < f) dX[row * lddx + lane + 32 * t] += acc[t];
    }
}

// keys[i] = the relation of values[i], or nrel for a value that is not one
__global__ void __launch_bounds__(kBlock) relation_keys_kernel(int32_t *__restrict__ keys, const double *__restrict__ values, int64_t n,
                                                               int nrel) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
        keys[i] = relation_of(values[i], nrel);
}

// the shared argument checks of the two basis kernels; HNH_OK or the error
int check_basis(const char *who, int64_t rows, int64_t nnz, int f, int nrel, int nbases) {
    if (rows < 0 || nnz < 0) return set_error(HNH_E_INVALID, "%s: negative size", who);
    if (f < 1) return set_error(HNH_E_INVALID, "%s: f must be positive (got %d)", who, f);
    if (nrel < 1) return set_error(HNH_E_INVALID, "%s: the relation count must be positive (got %d)", who, nrel);
    if (nbases < 1) return set_error(HNH_E_INVALID, "%s: the basis count must be positive (got %d)", who, nbases);
    if ((int64_t)nbases * f > INT32_MAX || (int64_t)nrel * nbases > INT32_MAX)
        return set_error(HNH_E_INVALID, "%s: B f and R B must be below 2^31 (f = %d, R = %d, B = %d)", who, f, nrel, nbases);
    return HNH_OK;
}

// the one-warp-per-row instantiation for a window of width f <= 256
template <typename K>
K pick_generic(int f, K k1, K k2, K k4, K k8) {
    return f <= 32 ? k1 : f <= 64 ? k2 : f <= 128 ? k4 : k8;
}

// the shared argument checks of the two sparse kernels; HNH_OK or the error
int check_relational(const char *who, int64_t rows, int64_t nnz, int f, int nrel, int64_t ldy, int64_t ldo, bool y_is_wide) {
    if (rows < 0 || nnz < 0) return set_error(HNH_E_INVALID, "%s: negative size", who);
    if (f < 1) return set_error(HNH_E_INVALID, "%s: f must be positive (got %d)", who, f);
    if (nrel < 1) return set_error(HNH_E_INVALID, "%s: the relation count must be positive (got %d)", who, nrel);
    const int64_t wide = (int64_t)nrel * f;
    if (wide > INT32_MAX) return set_error(HNH_E_INVALID, "%s: R f = %lld must be below 2^31", who, (long long)wide);
    if (ldy < (y_is_wide ? wide : f) || ldo < (y_is_wide ? f : wide))
        return set_error(HNH_E_INVALID, "%s: a leading dimension is below its width (f = %d, R f = %lld)", who, f, (long long)wide);
    return HNH_OK;
}

}  // namespace

extern "C" {

int hnh_relational_aggregate_f64(const int64_t *rowStart, const int64_t *col_idx, const double *values, int64_t rows, int64_t nnz,
                                 const double *X, int64_t ldx, int f, int R, double *A, int64_t lda, void *stream) {
    const char *who = "hnh_relational_aggregate_f64";
    int rc = check_relational(who, rows, nnz, f, R, ldx, lda, false);
    if (rc) return rc;
    if (rows == 0 || nnz == 0) return HNH_OK;
    if (!rowStart || !col_idx || !values || !X || !A) return set_error(HNH_E_INVALID, "%s: null pointer", who);
    if (A == X || A == values) return set_error(HNH_E_INVALID, "%s: A may not be an input", who);
    cudaStream_t st = (cudaStream_t)stream;
    for (int c0 = 0; c0 < f && rc == HNH_OK; c0 += kWindow) {
        const int w = std::min(kWindow, f - c0);
        const double *Xw = X + c0;
        double *Aw = A + c0;
        int grid = 0;
        if (table_width(w) && aligned16(Xw) && aligned16(Aw) && ldx % 2 == 0 && lda % 2 == 0 && f % 2 == 0) {
#define RA(RR, G, VW, UN)                                                                                                  \
    {                                                                                                                      \
        auto k = relational_aggregate_kernel<RR, G, VW, UN>;                                                               \
        rc = grid_for(k, rows, kBlock / G, &grid);                                                                         \
        if (!rc)                                                                                                           \
            rc = launch(k, grid, kBlock, st, "relational_aggregate_kernel", rowStart, col_idx, values, rows, Xw, ldx, R,     \
                        (int64_t)f, Aw, lda);                                                                              \
    }
            HNH_DISPATCH_R(w, RA, )
#undef RA
            continue;
        }
        auto k = pick_generic(w, relational_aggregate_generic_kernel<1>, relational_aggregate_generic_kernel<2>,
                              relational_aggregate_generic_kernel<4>, relational_aggregate_generic_kernel<8>);
        rc = grid_for(k, rows, kBlock / 32, &grid);
        if (!rc)
            rc = launch(k, grid, kBlock, st, "relational_aggregate_generic_kernel", rowStart, col_idx, values, rows, Xw, ldx, w, R,
                        (int64_t)f, Aw, lda);
    }
    return rc;
}

int hnh_relational_aggregate_grad_f64(const int64_t *rowStart, const int64_t *col_idx, const double *values, int64_t rows,
                                      int64_t nnz, const double *dA, int64_t ldda, int f, int R, double *dX, int64_t lddx,
                                      void *stream) {
    const char *who = "hnh_relational_aggregate_grad_f64";
    int rc = check_relational(who, rows, nnz, f, R, ldda, lddx, true);
    if (rc) return rc;
    if (rows == 0 || nnz == 0) return HNH_OK;
    if (!rowStart || !col_idx || !values || !dA || !dX) return set_error(HNH_E_INVALID, "%s: null pointer", who);
    if (dX == dA || dX == values) return set_error(HNH_E_INVALID, "%s: dX may not be an input", who);
    cudaStream_t st = (cudaStream_t)stream;
    for (int c0 = 0; c0 < f && rc == HNH_OK; c0 += kWindow) {
        const int w = std::min(kWindow, f - c0);
        const double *dAw = dA + c0;
        double *dXw = dX + c0;
        int grid = 0;
        if (table_width(w) && aligned16(dAw) && aligned16(dXw) && ldda % 2 == 0 && lddx % 2 == 0 && f % 2 == 0) {
#define RG(RR, G, VW, UN)                                                                                                  \
    {                                                                                                                      \
        auto k = relational_aggregate_grad_kernel<RR, G, VW, UN>;                                                          \
        rc = grid_for(k, rows, kBlock / G, &grid);                                                                         \
        if (!rc)                                                                                                           \
            rc = launch(k, grid, kBlock, st, "relational_aggregate_grad_kernel", rowStart, col_idx, values, rows, dAw, ldda, R, \
                        (int64_t)f, dXw, lddx);                                                                            \
    }
            HNH_DISPATCH_R(w, RG, )
#undef RG
            continue;
        }
        auto k = pick_generic(w, relational_aggregate_grad_generic_kernel<1>, relational_aggregate_grad_generic_kernel<2>,
                              relational_aggregate_grad_generic_kernel<4>, relational_aggregate_grad_generic_kernel<8>);
        rc = grid_for(k, rows, kBlock / 32, &grid);
        if (!rc)
            rc = launch(k, grid, kBlock, st, "relational_aggregate_grad_generic_kernel", rowStart, col_idx, values, rows, dAw, ldda,
                        w, R, (int64_t)f, dXw, lddx);
    }
    return rc;
}

int hnh_window_scale_f64(double *A, int64_t lda, const double *C, int64_t ldc, int64_t n, int f, int R, void *stream) {
    const char *who = "hnh_window_scale_f64";
    if (n < 0) return set_error(HNH_E_INVALID, "%s: negative size", who);
    if (f < 1 || R < 1) return set_error(HNH_E_INVALID, "%s: f and R must be positive (got %d and %d)", who, f, R);
    if ((int64_t)R * f > INT32_MAX) return set_error(HNH_E_INVALID, "%s: R f must be below 2^31", who);
    if (lda < (int64_t)R * f || ldc < R) return set_error(HNH_E_INVALID, "%s: a leading dimension is below its width", who);
    if (n == 0) return HNH_OK;
    if (!A || !C) return set_error(HNH_E_INVALID, "%s: null pointer", who);
    if ((const double *)A == C) return set_error(HNH_E_INVALID, "%s: A may not be C", who);
    int grid = 0;
    int rc = grid_for(window_scale_kernel, n, kBlock / 32, &grid);
    return rc ? rc : launch(window_scale_kernel, grid, kBlock, (cudaStream_t)stream, "window_scale_kernel", A, lda, C, ldc, n, f, R);
}

int hnh_basis_aggregate_f64(const int64_t *rowStart, const int64_t *col_idx, const double *values, int64_t rows, int64_t nnz,
                            const double *X, int64_t ldx, int f, const double *scale, int64_t lds, const double *comp, int R, int B,
                            double *H, int64_t ldh, void *stream) {
    const char *who = "hnh_basis_aggregate_f64";
    int rc = check_basis(who, rows, nnz, f, R, B);
    if (rc) return rc;
    if (ldx < f || ldh < (int64_t)B * f || (scale && lds < R))
        return set_error(HNH_E_INVALID, "%s: a leading dimension is below its width (f = %d, B f = %lld, R = %d)", who, f,
                         (long long)B * f, R);
    if (rows == 0 || nnz == 0) return HNH_OK;
    if (!rowStart || !col_idx || !values || !X || !comp || !H) return set_error(HNH_E_INVALID, "%s: null pointer", who);
    if (H == X || H == values || H == comp || H == scale) return set_error(HNH_E_INVALID, "%s: H may not be an input", who);
    cudaStream_t st = (cudaStream_t)stream;
    for (int c0 = 0; c0 < f && rc == HNH_OK; c0 += kWindow) {
        const int w = std::min(kWindow, f - c0);
        const double *Xw = X + c0;
        double *Hw = H + c0;
        int grid = 0;
        if (table_width(w) && aligned16(Xw) && aligned16(Hw) && ldx % 2 == 0 && ldh % 2 == 0 && f % 2 == 0) {
            // the full register budget, or half of it when B fits there
#define BA(RR, G, VW, UN)                                                                                                  \
    {                                                                                                                      \
        constexpr int NF = kBasisAcc / ((RR) / (G));                                                                       \
        auto k = B <= NF / 2 ? basis_aggregate_kernel<RR, G, VW, UN, NF / 2> : basis_aggregate_kernel<RR, G, VW, UN, NF>;  \
        rc = grid_for(k, rows, kBlock / G, &grid);                                                                         \
        if (!rc)                                                                                                           \
            rc = launch(k, grid, kBlock, st, "basis_aggregate_kernel", rowStart, col_idx, values, rows, Xw, ldx, scale, lds, \
                        comp, R, B, (int64_t)f, Hw, ldh);                                                                  \
    }
            HNH_DISPATCH_R(w, BA, )
#undef BA
            continue;
        }
        auto k = pick_generic(w, basis_aggregate_generic_kernel<1, 16>, basis_aggregate_generic_kernel<2, 8>,
                              basis_aggregate_generic_kernel<4, 4>, basis_aggregate_generic_kernel<8, 2>);
        rc = grid_for(k, rows, kBlock / 32, &grid);
        if (!rc)
            rc = launch(k, grid, kBlock, st, "basis_aggregate_generic_kernel", rowStart, col_idx, values, rows, Xw, ldx, w, scale, lds,
                        comp, R, B, (int64_t)f, Hw, ldh);
    }
    return rc;
}

int hnh_basis_aggregate_grad_f64(const int64_t *rowStart, const int64_t *col_idx, const double *values, int64_t rows, int64_t nnz,
                                 const double *dH, int64_t lddh, const double *scale, int64_t lds, const double *comp, int R, int B,
                                 const double *X, int64_t ldx, int f, double *dX, int64_t lddx, double *products, int64_t ldp,
                                 void *stream) {
    const char *who = "hnh_basis_aggregate_grad_f64";
    int rc = check_basis(who, rows, nnz, f, R, B);
    if (rc) return rc;
    if (lddh < (int64_t)B * f || lddx < f || (scale && lds < R) || (products && (ldx < f || ldp < nnz)))
        return set_error(HNH_E_INVALID, "%s: a leading dimension is below its width (f = %d, B f = %lld, R = %d, nnz = %lld)", who, f,
                         (long long)B * f, R, (long long)nnz);
    if (rows == 0 || nnz == 0) return HNH_OK;
    if (!rowStart || !col_idx || !values || !dH || !comp || !dX || (products && !X))
        return set_error(HNH_E_INVALID, "%s: null pointer", who);
    for (const void *in : {(const void *)dH, (const void *)values, (const void *)comp, (const void *)scale, (const void *)X})
        if (in && (in == dX || in == products)) return set_error(HNH_E_INVALID, "%s: dX and the products may not be inputs", who);
    if ((const double *)dX == products) return set_error(HNH_E_INVALID, "%s: dX may not be the products", who);
    cudaStream_t st = (cudaStream_t)stream;
    for (int c0 = 0; c0 < f && rc == HNH_OK; c0 += kWindow) {
        const int w = std::min(kWindow, f - c0);
        const double *dHw = dH + c0, *Xw = products ? X + c0 : nullptr;
        double *dXw = dX + c0;
        const int p_add = c0 > 0;
        int grid = 0;
        if (table_width(w) && aligned16(dHw) && aligned16(dXw) && (!products || (aligned16(Xw) && ldx % 2 == 0)) && lddh % 2 == 0 &&
            lddx % 2 == 0 && f % 2 == 0) {
#define BG(RR, G, VW, UN)                                                                                                  \
    {                                                                                                                      \
        auto k = basis_aggregate_grad_kernel<RR, G, VW, UN>;                                                               \
        rc = grid_for(k, rows, kBlock / G, &grid);                                                                         \
        if (!rc)                                                                                                           \
            rc = launch(k, grid, kBlock, st, "basis_aggregate_grad_kernel", rowStart, col_idx, values, rows, dHw, lddh, scale, \
                        lds, comp, R, B, (int64_t)f, Xw, ldx, dXw, lddx, products, ldp, p_add);                            \
    }
            HNH_DISPATCH_R(w, BG, )
#undef BG
            continue;
        }
        auto k = pick_generic(w, basis_aggregate_grad_generic_kernel<1>, basis_aggregate_grad_generic_kernel<2>,
                              basis_aggregate_grad_generic_kernel<4>, basis_aggregate_grad_generic_kernel<8>);
        rc = grid_for(k, rows, kBlock / 32, &grid);
        if (!rc)
            rc = launch(k, grid, kBlock, st, "basis_aggregate_grad_generic_kernel", rowStart, col_idx, values, rows, dHw, lddh, scale,
                        lds, comp, R, B, (int64_t)f, Xw, ldx, w, dXw, lddx, products, ldp, p_add);
    }
    return rc;
}

int hnh_relation_keys(int32_t *keys, const double *values, int64_t n, int R, void *stream) {
    if (n < 0) return set_error(HNH_E_INVALID, "hnh_relation_keys: negative size");
    if (R < 1 || R == INT32_MAX) return set_error(HNH_E_INVALID, "hnh_relation_keys: the relation count must lie in [1, 2^31 - 1) (got %d)", R);
    if (n == 0) return HNH_OK;
    if (!keys || !values) return set_error(HNH_E_INVALID, "hnh_relation_keys: null pointer");
    int grid = 0;
    int rc = grid_for(relation_keys_kernel, n, kBlock * 4, &grid);
    return rc ? rc : launch(relation_keys_kernel, grid, kBlock, (cudaStream_t)stream, "relation_keys_kernel", keys, values, n, R);
}

int hnh_relation_check_f64(double *bad, const double *values, int64_t n, int R, void *stream) {
    if (n < 0) return set_error(HNH_E_INVALID, "hnh_relation_check_f64: negative size");
    if (R < 1) return set_error(HNH_E_INVALID, "hnh_relation_check_f64: the relation count must be positive (got %d)", R);
    if (!bad || (n > 0 && !values)) return set_error(HNH_E_INVALID, "hnh_relation_check_f64: null pointer");
    if (n == 0) return HNH_OK;
    return launch(relation_check_kernel, 1, kBlock, (cudaStream_t)stream, "relation_check_kernel", bad, values, n, R);
}

}  // extern "C"
