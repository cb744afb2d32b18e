// sparse_attention.cu -- fused sparse attention over the pattern of one CSR block (Distributed_Sparse::sparseAttention
// / sparseAttentionBackward).  With u the stored row, v = col_idx of an entry, sigma the scale, q, k, v, dz d-wide rows
// and L, t per-row scalars, every dense operand row-major with its own leading dimension:
//     x_uv = sigma <Q_u, K_v>,  alpha_uv = exp(x_uv - L_u),  dx_uv = alpha_uv (<dZ_u, V_v> - t_u)
//   step     (acc, m, s)_u  <- the online softmax of row u continued over the block's entries:
//              m' = max(m, max_v x_uv), acc' = e^(m - m') acc + sum_v e^(x_uv - m') V_v, s' = e^(m - m') s + sum_v e^(x_uv - m')
//   finish   Z_u = acc_u / s_u, L_u = m_u + log s_u (Z_u = 0, L_u = -inf where s_u = 0)
//   grad_q   dQ_u += sigma sum_v dx_uv K_v                                  (stored rows are query rows)
//   grad_kv  dK_v += sigma sum_u dx_uv Q_u,  dV_v += sum_u alpha_uv dZ_u     (stored rows are key rows)
//
// The fast kernels follow gatv2.cu: a group of G lanes owns one CSR row and keeps its row-side operands and
// accumulators in registers; a chunk of G column indices is read coalesced and broadcast by shuffles; gathered rows come
// in with 128-bit loads, UN rows in flight per lane; every dot ends in the group's xor-butterfly, which leaves the same
// bits on every lane.  The step kernel takes a chunk in two sweeps: the K rows and their scores, then one rescale of
// (acc, s) to the chunk's new maximum, then the V rows.  Widths 4..256 (powers of two) with 16-byte aligned d-wide
// operands and even leading dimensions take these; every other case takes the one-warp-per-row generic kernels.  No
// floating-point atomics: two calls on the same device give bit-identical results.
//
// Attention dropout (DROP = true; the *_dropout_f64 entry points): with D_uv the keep bit of entry (u, v) and
// w = 1 / (1 - p), the step adds D_uv w e^(x_uv - m') V_v to acc but every e^(x_uv - m') to s (L stays the
// log-sum-exp of all scores), and the gradients use dx_uv = alpha_uv (D_uv w <dZ_u, V_v> - t_u) and
// dV_v += sum_u D_uv w alpha_uv dZ_u.  D_uv is a hash of (seed, global u, global v) only (keep(), below), so the
// three passes, whatever their value order, block or ring step, see the same mask.  In the fast kernels the lane
// that loads entry k's column index hashes it and sends the bit along with what it already broadcasts: the sign of
// its weight (step) or its column index, complemented (gradients).  A dropped entry's V row (step), V row (grad_q)
// or dZ row (grad_kv) is not loaded.  The instantiations with DROP = false are the kernels without dropout.
//
// Additive score bias (BIAS = true; the *_bias_f64 entry points): x_uv = sigma <Q_u, K_v> + b_i for the block's entry
// i, and the gradient kernels add dx_i to db[i] when db is not null (dx_i is the bias gradient).  b = -inf masks an
// entry: it adds nothing to (acc, m, s), alpha = 0 (so dx = 0) even where L = -inf, and its V or dZ row is not
// loaded; a chunk whose entries are all masked leaves (acc, m, s) as they are, so a row masked throughout keeps s = 0
// and finishes with Z = 0, L = -inf.  In the fast kernels the lane that loads entry k's column index loads b_k: the
// step adds it to the lane's own score and sends a masked entry's weight with its sign bit set; the gradients
// broadcast it with one shuffle, send a masked entry's column index complemented, and lane k keeps dx_k and adds it
// to db[k] once per chunk.  The gradients compute x - L as (sigma <.,.> - L) + b, so a bias of zeros gives the bits
// of the kernels without bias.  The instantiations with BIAS = false are the kernels without bias.
//
// Edge features (EDGE = true; the *_edge_f64 entry points): entry i of the block reads a d-wide row E_i, added to the
// key and to the value: x_i = sigma <Q_u, K_v + E_i> (+ b_i), the step accumulates alpha_i (V_v + E_i), the gradients
// use g_i = <dZ_u, V_v + E_i>, dQ_u += sigma dx_i (K_v + E_i), and grad_q writes dE_i = sigma dx_i Q_u + D_i w
// alpha_i dZ_u (0 for a masked entry) once per entry when dE is not null.  The rows of a chunk's entries are
// contiguous: every lane loads its own slice of E_i beside the K (step sweep 1, grad_q) or Q (grad_kv) row it gathers,
// and adds it to the gathered row before any product, so E = 0 gives the bits of the kernels without E.  The step
// reads E_i twice, once per sweep; the first read allocates in L1 so that the second, a chunk later, hits a cache.
// grad_q writes the dE row from the Q_u and dZ_u it already holds, every lane its own slice.  The instantiations with
// EDGE = false are the kernels without edge features.
#include <cmath>

#include "mix64.cuh"
#include "row_gather.cuh"

namespace {

using hnh::grid_for;
using hnh::launch;
using hnh::set_error;

// The dropout of one call (include/hnh_b200.h): entry (u, v) is kept iff the high word of mix64(key ^ (u << 32 | v))
// is at least `threshold`, key = mix64(seed); u0 and v0 are the global S-row and S-column of the block's row and
// column 0.  The kernels without dropout receive it and do not read it.
struct Dropout {
    uint64_t key;
    int64_t u0, v0;
    double inv_keep;  // 1 / (1 - p)
    uint32_t threshold;
};

// The bias of one call: entry i of the block reads b[i]; the gradient kernels add dx_i to db[i] unless db is null.
// Passed after the Dropout, so the kernels without bias keep their parameter layout.
struct Bias {
    const double *b;
    double *db;
};

// The edge features of one call: entry i of the block reads E + i lde; grad_q writes dE_i to dE + i ldde unless dE
// is null.  Passed after the Bias, so the kernels without edge features keep their parameter layout.
struct Edge {
    const double *E;
    int64_t lde;
    double *dE;
    int64_t ldde;
};

// E_i's slice in the step's first sweep: read-only, allocating in L1 for the second sweep's read of the same row
template <int VW>
__device__ __forceinline__ void ld_edge(double (&d)[VW], const double *p) {
    static_assert(VW == 2, "128-bit loads only");
    asm volatile("ld.global.nc.v2.f64 {%0,%1}, [%2];" : "=d"(d[0]), "=d"(d[1]) : "l"(p));
}

__device__ __forceinline__ bool keep(const Dropout &dr, int64_t u, int64_t v) {
    return (uint32_t)(mix64(dr.key ^ ((uint64_t)u << 32 | (uint64_t)v)) >> 32) >= dr.threshold;
}

template <int G>
__device__ __forceinline__ double group_max(double d, unsigned mask) {
#pragma unroll
    for (int o = G / 2; o > 0; o >>= 1) d = fmax(d, __shfl_xor_sync(mask, d, o, G));
    return d;
}

// ---- fast row kernels ----------------------------------------------------------------------------------------
template <int R, int G, int VW, int UN, bool DROP, bool BIAS, bool EDGE>
__global__ void __launch_bounds__(kBlock, 1)
attn_step_kernel(const int64_t *__restrict__ rowStart, const int64_t *__restrict__ col_idx, int64_t rows,
                 const double *__restrict__ Q, int64_t ldq, const double *__restrict__ K, int64_t ldk,
                 const double *__restrict__ V, int64_t ldv, double scale, double *__restrict__ acc, int64_t ldacc,
                 double *__restrict__ m, int64_t ldm, double *__restrict__ s, int64_t lds, Dropout dr, Bias bs, Edge eg) {
    constexpr int NV = R / (G * VW);
    static_assert(NV * G * VW == R, "R must equal NV*G*VW");
    const int lane = threadIdx.x & 31;
    const int gl = lane & (G - 1);
    const unsigned gmask = group_mask<G>(lane);
    const int64_t ngroups = (int64_t)gridDim.x * (blockDim.x / G);
    for (int64_t row = (int64_t)blockIdx.x * (blockDim.x / G) + threadIdx.x / G; row < rows; row += ngroups) {
        const int64_t s0 = ld_stream_i64(rowStart + row);
        const int64_t e = ld_stream_i64(rowStart + row + 1);
        if (s0 == e) continue;
        double q[NV][VW], a[NV][VW];
#pragma unroll
        for (int v = 0; v < NV; v++) {
            ld_gather<VW>(q[v], Q + row * ldq + (v * G + gl) * VW);
            ld_rw<VW>(a[v], acc + row * ldacc + (v * G + gl) * VW);
        }
        double srow = s[row * lds];
        double mrow = srow == 0.0 ? -INFINITY : m[row * ldm];  // a row not started yet, whatever m holds
        for (int64_t j = s0; j < e; j += G) {
            const int cnt = (e - j < G) ? (int)(e - j) : G;
            int64_t mycol = 0;
            double mybias = 0.0;
            if (gl < cnt) {
                mycol = ld_stream_i64(col_idx + j + gl);
                if constexpr (BIAS) mybias = ld_stream_f64(bs.b + j + gl);
            }
            // sweep 1: the chunk's scores, entry k's on lane k
            double mine = -INFINITY;
            for (int k0 = 0; k0 < cnt; k0 += UN) {
                double y[UN][NV][VW];
#pragma unroll
                for (int u = 0; u < UN; u++) {
                    const int k = k0 + u;
                    const int64_t c = __shfl_sync(gmask, mycol, k < G ? k : G - 1, G);
                    if (k < cnt) {
#pragma unroll
                        for (int v = 0; v < NV; v++) ld_gather<VW>(y[u][v], K + c * ldk + (v * G + gl) * VW);
                        if constexpr (EDGE) {
#pragma unroll
                            for (int v = 0; v < NV; v++) {
                                double ev[VW];
                                ld_edge<VW>(ev, eg.E + (j + k) * eg.lde + (v * G + gl) * VW);
#pragma unroll
                                for (int w = 0; w < VW; w++) y[u][v][w] += ev[w];
                            }
                        }
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
                        for (int w = 0; w < VW; w++) d = fma(q[v][w], y[u][v][w], d);
                    d = group_allreduce<G>(d, gmask);
                    // padding slots past cnt (zero rows) must not enter the chunk's maximum
                    if (gl == k0 + u && k0 + u < cnt) mine = BIAS ? scale * d + mybias : scale * d;
                }
            }
            // one rescale to the chunk's maximum (exp(-inf) = 0 for a row's first chunk); a chunk whose entries are all
            // masked, with no earlier entry, has mnew = -inf and leaves the state as it is
            const double mnew = fmax(mrow, group_max<G>(mine, gmask));
            const double f = (BIAS && mnew == -INFINITY) ? 1.0 : exp(mrow - mnew);
#pragma unroll
            for (int v = 0; v < NV; v++)
#pragma unroll
                for (int w = 0; w < VW; w++) a[v][w] *= f;
            srow *= f;
            mrow = mnew;
            double pmine = gl < cnt ? exp(mine - mnew) : 0.0;
            // a dropped entry's weight travels with its sign bit set (-0.0 included): it counts in s, not in acc
            if constexpr (DROP)
                if (!keep(dr, dr.u0 + row, dr.v0 + mycol)) pmine = -pmine;
            // a masked entry's weight is -0.0: it counts in neither s nor acc
            if constexpr (BIAS)
                if (mine == -INFINITY) pmine = -0.0;
            // sweep 2: the V rows, weighted
            for (int k0 = 0; k0 < cnt; k0 += UN) {
                double y[UN][NV][VW];
                double pv[UN];
#pragma unroll
                for (int u = 0; u < UN; u++) {
                    const int k = k0 + u;
                    const int src = k < G ? k : G - 1;
                    const int64_t c = __shfl_sync(gmask, mycol, src, G);
                    pv[u] = __shfl_sync(gmask, pmine, src, G);
                    if (k < cnt && !((DROP || BIAS) && signbit(pv[u]))) {
#pragma unroll
                        for (int v = 0; v < NV; v++) ld_gather<VW>(y[u][v], V + c * ldv + (v * G + gl) * VW);
                        if constexpr (EDGE) {
#pragma unroll
                            for (int v = 0; v < NV; v++) {
                                double ev[VW];
                                ld_gather<VW>(ev, eg.E + (j + k) * eg.lde + (v * G + gl) * VW);
#pragma unroll
                                for (int w = 0; w < VW; w++) y[u][v][w] += ev[w];
                            }
                        }
                    }
                }
#pragma unroll
                for (int u = 0; u < UN; u++) {
                    if (k0 + u < cnt) {
                        if constexpr (DROP) {
                            if (!signbit(pv[u])) {
                                const double pw = pv[u] * dr.inv_keep;
#pragma unroll
                                for (int v = 0; v < NV; v++)
#pragma unroll
                                    for (int w = 0; w < VW; w++) a[v][w] = fma(pw, y[u][v][w], a[v][w]);
                            }
                            srow += fabs(pv[u]);
                        } else if constexpr (BIAS) {
                            if (!signbit(pv[u])) {
#pragma unroll
                                for (int v = 0; v < NV; v++)
#pragma unroll
                                    for (int w = 0; w < VW; w++) a[v][w] = fma(pv[u], y[u][v][w], a[v][w]);
                            }
                            srow += pv[u];
                        } else {
#pragma unroll
                            for (int v = 0; v < NV; v++)
#pragma unroll
                                for (int w = 0; w < VW; w++) a[v][w] = fma(pv[u], y[u][v][w], a[v][w]);
                            srow += pv[u];
                        }
                    }
                }
            }
        }
#pragma unroll
        for (int v = 0; v < NV; v++) st_rw<VW>(acc + row * ldacc + (v * G + gl) * VW, a[v]);
        if (gl == 0) {
            m[row * ldm] = mrow;
            s[row * lds] = srow;
        }
    }
}

template <int R, int G, int VW, int UN, bool DROP, bool BIAS, bool EDGE>
__global__ void __launch_bounds__(kBlock, 1)
attn_grad_q_kernel(const int64_t *__restrict__ rowStart, const int64_t *__restrict__ col_idx, int64_t rows,
                   const double *__restrict__ Q, int64_t ldq, const double *__restrict__ dZ, int64_t lddz,
                   const double *__restrict__ L, int64_t ldl, const double *__restrict__ t, int64_t ldt,
                   const double *__restrict__ K, int64_t ldk, const double *__restrict__ V, int64_t ldv, double scale,
                   double *__restrict__ dQ, int64_t lddq, Dropout dr, Bias bs, Edge eg) {
    constexpr int NV = R / (G * VW);
    static_assert(NV * G * VW == R, "R must equal NV*G*VW");
    const int lane = threadIdx.x & 31;
    const int gl = lane & (G - 1);
    const unsigned gmask = group_mask<G>(lane);
    const int64_t ngroups = (int64_t)gridDim.x * (blockDim.x / G);
    for (int64_t row = (int64_t)blockIdx.x * (blockDim.x / G) + threadIdx.x / G; row < rows; row += ngroups) {
        const int64_t s0 = ld_stream_i64(rowStart + row);
        const int64_t e = ld_stream_i64(rowStart + row + 1);
        if (s0 == e) continue;  // dQ[row] += 0
        double q[NV][VW], dz[NV][VW], a[NV][VW];
#pragma unroll
        for (int v = 0; v < NV; v++) {
            ld_gather<VW>(q[v], Q + row * ldq + (v * G + gl) * VW);
            ld_gather<VW>(dz[v], dZ + row * lddz + (v * G + gl) * VW);
#pragma unroll
            for (int w = 0; w < VW; w++) a[v][w] = 0.0;
        }
        const double Lr = L[row * ldl], tr = t[row * ldt];
        for (int64_t j = s0; j < e; j += G) {
            const int cnt = (e - j < G) ? (int)(e - j) : G;
            int64_t mycol = 0;
            double mybias = 0.0, mydx = 0.0;
            if (gl < cnt) {
                mycol = ld_stream_i64(col_idx + j + gl);
                if constexpr (BIAS) mybias = ld_stream_f64(bs.b + j + gl);
            }
            // a dropped entry's column index travels complemented (negative)
            if constexpr (DROP)
                if (!keep(dr, dr.u0 + row, dr.v0 + mycol)) mycol = ~mycol;
            // and so does a masked one's: it needs no V row either
            if constexpr (BIAS)
                if (mybias == -INFINITY && mycol >= 0) mycol = ~mycol;
            for (int k0 = 0; k0 < cnt; k0 += UN) {
                double yk[UN][NV][VW], yv[UN][NV][VW];
                double bu[UN];
                bool kept[UN];  // EDGE: D_i = 1 and not masked (the weight of dZ_u in dE_i is nonzero)
#pragma unroll
                for (int u = 0; u < UN; u++) {
                    const int k = k0 + u;
                    int64_t c = __shfl_sync(gmask, mycol, k < G ? k : G - 1, G);
                    if constexpr (BIAS) bu[u] = __shfl_sync(gmask, mybias, k < G ? k : G - 1, G);
                    const bool dropped = (DROP || BIAS) && c < 0;
                    if (dropped) c = ~c;
                    if constexpr (EDGE) kept[u] = !dropped;
                    if (k < cnt) {
#pragma unroll
                        for (int v = 0; v < NV; v++) {
                            ld_gather<VW>(yk[u][v], K + c * ldk + (v * G + gl) * VW);
                            // a dropped entry needs no <dZ_u, V_v>: a zero V row makes it 0
                            if (!dropped) {
                                ld_gather<VW>(yv[u][v], V + c * ldv + (v * G + gl) * VW);
                            } else {
#pragma unroll
                                for (int w = 0; w < VW; w++) yv[u][v][w] = 0.0;
                            }
                            if constexpr (EDGE) {
                                double ev[VW];
                                ld_gather<VW>(ev, eg.E + (j + k) * eg.lde + (v * G + gl) * VW);
#pragma unroll
                                for (int w = 0; w < VW; w++) {
                                    yk[u][v][w] += ev[w];
                                    if (!dropped) yv[u][v][w] += ev[w];
                                }
                            }
                        }
                    } else {
#pragma unroll
                        for (int v = 0; v < NV; v++)
#pragma unroll
                            for (int w = 0; w < VW; w++) yk[u][v][w] = yv[u][v][w] = 0.0;
                    }
                }
#pragma unroll
                for (int u = 0; u < UN; u++) {
                    double d1 = 0.0, d2 = 0.0;
#pragma unroll
                    for (int v = 0; v < NV; v++)
#pragma unroll
                        for (int w = 0; w < VW; w++) {
                            d1 = fma(q[v][w], yk[u][v][w], d1);
                            d2 = fma(dz[v][w], yv[u][v][w], d2);
                        }
                    d1 = group_allreduce<G>(d1, gmask);
                    d2 = group_allreduce<G>(d2, gmask);
                    if (k0 + u < cnt) {
                        double al;
                        if constexpr (BIAS) {
                            al = bu[u] == -INFINITY ? 0.0 : exp((scale * d1 - Lr) + bu[u]);
                        } else {
                            al = exp(scale * d1 - Lr);
                        }
                        const double dx = al * ((DROP ? dr.inv_keep * d2 : d2) - tr);
                        if (BIAS && gl == k0 + u) mydx = dx;
#pragma unroll
                        for (int v = 0; v < NV; v++)
#pragma unroll
                            for (int w = 0; w < VW; w++) a[v][w] = fma(dx, yk[u][v][w], a[v][w]);
                        if constexpr (EDGE) {
                            if (eg.dE != nullptr) {
                                // dE_i = sigma dx_i Q_u + D_i w alpha_i dZ_u
                                const double g = scale * dx, aw = kept[u] ? (DROP ? al * dr.inv_keep : al) : 0.0;
#pragma unroll
                                for (int v = 0; v < NV; v++) {
                                    double o[VW];
#pragma unroll
                                    for (int w = 0; w < VW; w++) o[w] = fma(g, q[v][w], aw * dz[v][w]);
                                    st_rw<VW>(eg.dE + (j + k0 + u) * eg.ldde + (v * G + gl) * VW, o);
                                }
                            }
                        }
                    }
                }
            }
            if constexpr (BIAS)
                if (bs.db != nullptr && gl < cnt) bs.db[j + gl] += mydx;
        }
#pragma unroll
        for (int v = 0; v < NV; v++) {
            double o[VW];
            double *p = dQ + row * lddq + (v * G + gl) * VW;
            ld_rw<VW>(o, p);
#pragma unroll
            for (int w = 0; w < VW; w++) o[w] = fma(scale, a[v][w], o[w]);
            st_rw<VW>(p, o);
        }
    }
}

template <int R, int G, int VW, int UN, bool DROP, bool BIAS, bool EDGE>
__global__ void __launch_bounds__(kBlock, 1)
attn_grad_kv_kernel(const int64_t *__restrict__ rowStart, const int64_t *__restrict__ col_idx, int64_t rows,
                    const double *__restrict__ K, int64_t ldk, const double *__restrict__ V, int64_t ldv,
                    const double *__restrict__ Q, int64_t ldq, const double *__restrict__ dZ, int64_t lddz,
                    const double *__restrict__ L, int64_t ldl, const double *__restrict__ t, int64_t ldt, double scale,
                    double *__restrict__ dK, int64_t lddk, double *__restrict__ dV, int64_t lddv, Dropout dr, Bias bs,
                    Edge eg) {
    constexpr int NV = R / (G * VW);
    static_assert(NV * G * VW == R, "R must equal NV*G*VW");
    const int lane = threadIdx.x & 31;
    const int gl = lane & (G - 1);
    const unsigned gmask = group_mask<G>(lane);
    const int64_t ngroups = (int64_t)gridDim.x * (blockDim.x / G);
    for (int64_t row = (int64_t)blockIdx.x * (blockDim.x / G) + threadIdx.x / G; row < rows; row += ngroups) {
        const int64_t s0 = ld_stream_i64(rowStart + row);
        const int64_t e = ld_stream_i64(rowStart + row + 1);
        if (s0 == e) continue;
        double kr[NV][VW], vr[NV][VW], ak[NV][VW], av[NV][VW];
#pragma unroll
        for (int v = 0; v < NV; v++) {
            ld_gather<VW>(kr[v], K + row * ldk + (v * G + gl) * VW);
            ld_gather<VW>(vr[v], V + row * ldv + (v * G + gl) * VW);
#pragma unroll
            for (int w = 0; w < VW; w++) ak[v][w] = av[v][w] = 0.0;
        }
        for (int64_t j = s0; j < e; j += G) {
            const int cnt = (e - j < G) ? (int)(e - j) : G;
            int64_t mycol = 0;
            double myL = 0.0, myt = 0.0, mybias = 0.0, mydx = 0.0;
            if (gl < cnt) {
                mycol = ld_stream_i64(col_idx + j + gl);
                if constexpr (BIAS) mybias = ld_stream_f64(bs.b + j + gl);
                myL = L[mycol * ldl];
                myt = t[mycol * ldt];
            }
            // a dropped entry's column index travels complemented (negative); here u = u0 + col_idx, v = v0 + row
            if constexpr (DROP)
                if (!keep(dr, dr.u0 + mycol, dr.v0 + row)) mycol = ~mycol;
            // and so does a masked one's: it needs no dZ row either
            if constexpr (BIAS)
                if (mybias == -INFINITY && mycol >= 0) mycol = ~mycol;
            for (int k0 = 0; k0 < cnt; k0 += UN) {
                double yq[UN][NV][VW], yd[UN][NV][VW], ye[UN][NV][VW];
                double Lu[UN], tu[UN], bu[UN];
#pragma unroll
                for (int u = 0; u < UN; u++) {
                    const int k = k0 + u;
                    const int src = k < G ? k : G - 1;
                    int64_t c = __shfl_sync(gmask, mycol, src, G);
                    Lu[u] = __shfl_sync(gmask, myL, src, G);
                    tu[u] = __shfl_sync(gmask, myt, src, G);
                    if constexpr (BIAS) bu[u] = __shfl_sync(gmask, mybias, src, G);
                    const bool dropped = (DROP || BIAS) && c < 0;
                    if (dropped) c = ~c;
                    if (k < cnt) {
#pragma unroll
                        for (int v = 0; v < NV; v++) {
                            ld_gather<VW>(yq[u][v], Q + c * ldq + (v * G + gl) * VW);
                            // a dropped entry adds nothing to dV and needs no <V_v, dZ_u>: a zero dZ row
                            if (!dropped) {
                                ld_gather<VW>(yd[u][v], dZ + c * lddz + (v * G + gl) * VW);
                            } else {
#pragma unroll
                                for (int w = 0; w < VW; w++) yd[u][v][w] = 0.0;
                            }
                            if constexpr (EDGE) ld_gather<VW>(ye[u][v], eg.E + (j + k) * eg.lde + (v * G + gl) * VW);
                        }
                    } else {
#pragma unroll
                        for (int v = 0; v < NV; v++)
#pragma unroll
                            for (int w = 0; w < VW; w++) yq[u][v][w] = yd[u][v][w] = 0.0;
                        if constexpr (EDGE)
#pragma unroll
                            for (int v = 0; v < NV; v++)
#pragma unroll
                                for (int w = 0; w < VW; w++) ye[u][v][w] = 0.0;
                    }
                }
#pragma unroll
                for (int u = 0; u < UN; u++) {
                    double d1 = 0.0, d2 = 0.0;
#pragma unroll
                    for (int v = 0; v < NV; v++)
#pragma unroll
                        for (int w = 0; w < VW; w++) {
                            if constexpr (EDGE) {
                                d1 = fma(kr[v][w] + ye[u][v][w], yq[u][v][w], d1);
                                d2 = fma(vr[v][w] + ye[u][v][w], yd[u][v][w], d2);
                            } else {
                                d1 = fma(kr[v][w], yq[u][v][w], d1);
                                d2 = fma(vr[v][w], yd[u][v][w], d2);
                            }
                        }
                    d1 = group_allreduce<G>(d1, gmask);
                    d2 = group_allreduce<G>(d2, gmask);
                    if (k0 + u < cnt) {
                        double al;
                        if constexpr (BIAS) {
                            al = bu[u] == -INFINITY ? 0.0 : exp((scale * d1 - Lu[u]) + bu[u]);
                        } else {
                            al = exp(scale * d1 - Lu[u]);
                        }
                        const double dx = al * ((DROP ? dr.inv_keep * d2 : d2) - tu[u]);
                        const double aw = DROP ? al * dr.inv_keep : al;
                        if (BIAS && gl == k0 + u) mydx = dx;
#pragma unroll
                        for (int v = 0; v < NV; v++)
#pragma unroll
                            for (int w = 0; w < VW; w++) {
                                ak[v][w] = fma(dx, yq[u][v][w], ak[v][w]);
                                av[v][w] = fma(aw, yd[u][v][w], av[v][w]);
                            }
                    }
                }
            }
            if constexpr (BIAS)
                if (bs.db != nullptr && gl < cnt) bs.db[j + gl] += mydx;
        }
#pragma unroll
        for (int v = 0; v < NV; v++) {
            double o[VW];
            double *p = dK + row * lddk + (v * G + gl) * VW;
            ld_rw<VW>(o, p);
#pragma unroll
            for (int w = 0; w < VW; w++) o[w] = fma(scale, ak[v][w], o[w]);
            st_rw<VW>(p, o);
            p = dV + row * lddv + (v * G + gl) * VW;
            ld_rw<VW>(o, p);
#pragma unroll
            for (int w = 0; w < VW; w++) o[w] += av[v][w];
            st_rw<VW>(p, o);
        }
    }
}

// ---- generic kernels: any d, any leading dimension, any alignment; one warp per row, entry by entry ----------------
__device__ __forceinline__ double warp_dot(const double *x, const double *y, int d, int lane) {
    double acc = 0.0;
    for (int k = lane; k < d; k += 32) acc = fma(x[k], y[k], acc);
    return group_allreduce<32>(acc, 0xffffffffu);
}
// <x, y + e>, with the bits of warp_dot(x, y) where e = 0
__device__ __forceinline__ double warp_dot_plus(const double *x, const double *y, const double *e, int d, int lane) {
    double acc = 0.0;
    for (int k = lane; k < d; k += 32) acc = fma(x[k], y[k] + e[k], acc);
    return group_allreduce<32>(acc, 0xffffffffu);
}

template <bool DROP, bool BIAS, bool EDGE>
__global__ void __launch_bounds__(kBlock)
attn_step_generic_kernel(const int64_t *__restrict__ rowStart, const int64_t *__restrict__ col_idx, int64_t rows, int d,
                         const double *__restrict__ Q, int64_t ldq, const double *__restrict__ K, int64_t ldk,
                         const double *__restrict__ V, int64_t ldv, double scale, double *__restrict__ acc,
                         int64_t ldacc, double *__restrict__ m, int64_t ldm, double *__restrict__ s, int64_t lds,
                         Dropout dr, Bias bs, Edge eg) {
    const int lane = threadIdx.x & 31;
    const int64_t warps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t row = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; row < rows; row += warps) {
        const int64_t s0 = rowStart[row], e = rowStart[row + 1];
        if (s0 == e) continue;
        double srow = s[row * lds];
        double mrow = srow == 0.0 ? -INFINITY : m[row * ldm];
        double *a = acc + row * ldacc;
        for (int64_t j = s0; j < e; j++) {
            const int64_t c = col_idx[j];
            const double *Ej = EDGE ? eg.E + j * eg.lde : nullptr;
            double x;
            if constexpr (BIAS) {
                if (bs.b[j] == -INFINITY) continue;  // masked: adds nothing
                x = scale * (EDGE ? warp_dot_plus(Q + row * ldq, K + c * ldk, Ej, d, lane)
                                  : warp_dot(Q + row * ldq, K + c * ldk, d, lane)) +
                    bs.b[j];
            } else {
                x = scale * (EDGE ? warp_dot_plus(Q + row * ldq, K + c * ldk, Ej, d, lane)
                                  : warp_dot(Q + row * ldq, K + c * ldk, d, lane));
            }
            const double mnew = fmax(mrow, x);
            const double f = exp(mrow - mnew), pj = exp(x - mnew);
            if (DROP && !keep(dr, dr.u0 + row, dr.v0 + c)) {
                for (int k = lane; k < d; k += 32) a[k] *= f;
            } else {
                const double pw = DROP ? pj * dr.inv_keep : pj;
                if constexpr (EDGE)
                    for (int k = lane; k < d; k += 32) a[k] = fma(pw, V[c * ldv + k] + Ej[k], a[k] * f);
                else
                    for (int k = lane; k < d; k += 32) a[k] = fma(pw, V[c * ldv + k], a[k] * f);
            }
            srow = fma(srow, f, pj);
            mrow = mnew;
        }
        if (lane == 0) {
            m[row * ldm] = mrow;
            s[row * lds] = srow;
        }
    }
}

template <bool DROP, bool BIAS, bool EDGE>
__global__ void __launch_bounds__(kBlock)
attn_grad_q_generic_kernel(const int64_t *__restrict__ rowStart, const int64_t *__restrict__ col_idx, int64_t rows, int d,
                           const double *__restrict__ Q, int64_t ldq, const double *__restrict__ dZ, int64_t lddz,
                           const double *__restrict__ L, int64_t ldl, const double *__restrict__ t, int64_t ldt,
                           const double *__restrict__ K, int64_t ldk, const double *__restrict__ V, int64_t ldv,
                           double scale, double *__restrict__ dQ, int64_t lddq, Dropout dr, Bias bs, Edge eg) {
    const int lane = threadIdx.x & 31;
    const int64_t warps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t row = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; row < rows; row += warps) {
        const int64_t s0 = rowStart[row], e = rowStart[row + 1];
        if (s0 == e) continue;
        const double Lr = L[row * ldl], tr = t[row * ldt];
        for (int64_t j = s0; j < e; j++) {
            const int64_t c = col_idx[j];
            if constexpr (EDGE) {
                const double *Ej = eg.E + j * eg.lde;
                double *dEj = eg.dE != nullptr ? eg.dE + j * eg.ldde : nullptr;
                const double bj = BIAS ? bs.b[j] : 0.0;
                if (BIAS && bj == -INFINITY) {  // masked: alpha = 0, dx = 0 (db[j] += 0), dE_j = 0
                    if (dEj != nullptr)
                        for (int k = lane; k < d; k += 32) dEj[k] = 0.0;
                    continue;
                }
                const double d1 = warp_dot_plus(Q + row * ldq, K + c * ldk, Ej, d, lane);
                const bool kept = !DROP || keep(dr, dr.u0 + row, dr.v0 + c);
                // D_j w <dZ_u, V_v + E_j>
                const double d2 = kept ? (DROP ? dr.inv_keep : 1.0) * warp_dot_plus(dZ + row * lddz, V + c * ldv, Ej, d, lane) : 0.0;
                // L and t read at their use, as in the bias instantiation
                const double al = BIAS ? exp((scale * d1 - L[row * ldl]) + bj) : exp(scale * d1 - L[row * ldl]);
                const double dx = al * (d2 - t[row * ldt]);
                if (BIAS && bs.db != nullptr && lane == 0) bs.db[j] += dx;
                const double g = scale * dx;
                if (dEj != nullptr) {
                    const double aw = kept ? (DROP ? al * dr.inv_keep : al) : 0.0;
                    for (int k = lane; k < d; k += 32) dEj[k] = fma(g, Q[row * ldq + k], aw * dZ[row * lddz + k]);
                }
                for (int k = lane; k < d; k += 32) dQ[row * lddq + k] = fma(g, K[c * ldk + k] + Ej[k], dQ[row * lddq + k]);
                continue;
            }
            double bj = 0.0;
            if constexpr (BIAS) {
                bj = bs.b[j];
                if (bj == -INFINITY) continue;  // masked: alpha = 0, dx = 0 (db[j] += 0)
            }
            const double d1 = warp_dot(Q + row * ldq, K + c * ldk, d, lane);
            double d2;  // D_uv w <dZ_u, V_v>
            if constexpr (DROP)
                d2 = keep(dr, dr.u0 + row, dr.v0 + c) ? dr.inv_keep * warp_dot(dZ + row * lddz, V + c * ldv, d, lane) : 0.0;
            else
                d2 = warp_dot(dZ + row * lddz, V + c * ldv, d, lane);
            double g;
            if constexpr (BIAS) {
                // L and t read at their use: held across the row, they spill in this instantiation
                const double dx = exp((scale * d1 - L[row * ldl]) + bj) * (d2 - t[row * ldt]);
                if (bs.db != nullptr && lane == 0) bs.db[j] += dx;
                g = scale * dx;
            } else {
                g = scale * (exp(scale * d1 - Lr) * (d2 - tr));
            }
            for (int k = lane; k < d; k += 32) dQ[row * lddq + k] = fma(g, K[c * ldk + k], dQ[row * lddq + k]);
        }
    }
}

template <bool DROP, bool BIAS, bool EDGE>
__global__ void __launch_bounds__(kBlock)
attn_grad_kv_generic_kernel(const int64_t *__restrict__ rowStart, const int64_t *__restrict__ col_idx, int64_t rows, int d,
                            const double *__restrict__ K, int64_t ldk, const double *__restrict__ V, int64_t ldv,
                            const double *__restrict__ Q, int64_t ldq, const double *__restrict__ dZ, int64_t lddz,
                            const double *__restrict__ L, int64_t ldl, const double *__restrict__ t, int64_t ldt,
                            double scale, double *__restrict__ dK, int64_t lddk, double *__restrict__ dV, int64_t lddv,
                            Dropout dr, Bias bs, Edge eg) {
    const int lane = threadIdx.x & 31;
    const int64_t warps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t row = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; row < rows; row += warps) {
        const int64_t s0 = rowStart[row], e = rowStart[row + 1];
        for (int64_t j = s0; j < e; j++) {
            const int64_t u = col_idx[j];
            if (BIAS && bs.b[j] == -INFINITY) continue;  // masked: alpha = 0, dx = 0 (db[j] += 0)
            const double *Ej = EDGE ? eg.E + j * eg.lde : nullptr;
            // <K_v + E_j, Q_u>
            const double d1 = EDGE ? warp_dot_plus(Q + u * ldq, K + row * ldk, Ej, d, lane) : warp_dot(K + row * ldk, Q + u * ldq, d, lane);
            // x_uv - L_u
            auto xl = [&] { return BIAS ? (scale * d1 - L[u * ldl]) + bs.b[j] : scale * d1 - L[u * ldl]; };
            if (DROP && !keep(dr, dr.u0 + u, dr.v0 + row)) {  // here the stored row is the key v
                const double dx = exp(xl()) * -t[u * ldt];
                if (BIAS && bs.db != nullptr && lane == 0) bs.db[j] += dx;
                const double g = scale * dx;
                for (int k = lane; k < d; k += 32) dK[row * lddk + k] = fma(g, Q[u * ldq + k], dK[row * lddk + k]);
                continue;
            }
            const double d2 = EDGE ? warp_dot_plus(dZ + u * lddz, V + row * ldv, Ej, d, lane) : warp_dot(V + row * ldv, dZ + u * lddz, d, lane);
            const double al = exp(xl());
            const double aw = DROP ? al * dr.inv_keep : al;
            const double dx = al * ((DROP ? dr.inv_keep * d2 : d2) - t[u * ldt]);
            if (BIAS && bs.db != nullptr && lane == 0) bs.db[j] += dx;
            const double g = scale * dx;
            for (int k = lane; k < d; k += 32) {
                dK[row * lddk + k] = fma(g, Q[u * ldq + k], dK[row * lddk + k]);
                dV[row * lddv + k] = fma(aw, dZ[u * lddz + k], dV[row * lddv + k]);
            }
        }
    }
}

// Z[row, k] = acc[row, k] / s[row]; L[row] = m[row] + log s[row].  Z may be acc and L may be m (same pointer and
// leading dimension): each element is read and written by the same thread.
__global__ void attn_finish_kernel(int64_t rows, int d, const double *acc, int64_t ldacc, const double *m, int64_t ldm,
                                   const double *s, int64_t lds, double *Z, int64_t ldz, double *L, int64_t ldl) {
    const int64_t n = rows * d;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t row = i / d;
        const int k = (int)(i - row * d);
        const double sr = s[row * lds];
        if (k == 0) L[row * ldl] = sr > 0.0 ? m[row * ldm] + log(sr) : -INFINITY;
        Z[row * ldz + k] = sr > 0.0 ? acc[row * ldacc + k] / sr : 0.0;
    }
}

// A d-wide row operand (vector) or a per-row scalar column (scalar): its pointer and leading dimension
struct Operand {
    const void *p;
    int64_t ld;
    bool vector;
};

// Validates one block call: 1 = successful no-op (no rows or no entries), HNH_OK = launch, < 0 = error
int check_call(const char *who, const int64_t *rowStart, const int64_t *col_idx, int64_t rows, int64_t nnz, int d,
               double scale, std::initializer_list<Operand> ops) {
    if (rows < 0 || nnz < 0) return set_error(HNH_E_INVALID, "%s: negative size", who);
    if (d < 1) return set_error(HNH_E_INVALID, "%s: d must be positive (got %d)", who, d);
    if (!std::isfinite(scale)) return set_error(HNH_E_INVALID, "%s: the scale must be finite", who);
    for (const Operand &o : ops)
        if (o.ld < (o.vector ? d : 1))
            return set_error(HNH_E_INVALID, "%s: leading dimension %lld below %d", who, (long long)o.ld, o.vector ? d : 1);
    if (rows == 0 || nnz == 0) return 1;
    if (!rowStart || !col_idx) return set_error(HNH_E_INVALID, "%s: null pointer", who);
    for (const Operand &o : ops)
        if (!o.p) return set_error(HNH_E_INVALID, "%s: null pointer", who);
    return HNH_OK;
}

// the fast kernels' condition: a table width, and every d-wide operand 16-byte aligned with an even leading dimension
bool fast_path(int d, std::initializer_list<Operand> ops) {
    if (!table_width(d)) return false;
    for (const Operand &o : ops)
        if (o.vector && (!aligned16(o.p) || o.ld % 2 != 0)) return false;
    return true;
}

// fast_path's condition on the edge operands: E and, when written, dE
bool edge_fast(const Edge &eg) {
    return aligned16(eg.E) && eg.lde % 2 == 0 && (eg.dE == nullptr || (aligned16(eg.dE) && eg.ldde % 2 == 0));
}

// The Dropout of a call: HNH_OK, or HNH_E_INVALID for p outside [0, 1) (NaN included) or a negative offset
int make_dropout(const char *who, double p, uint64_t seed, int64_t u0, int64_t v0, Dropout *dr) {
    if (!(p >= 0.0 && p < 1.0)) return set_error(HNH_E_INVALID, "%s: the dropout probability must lie in [0, 1) (got %g)", who, p);
    if (u0 < 0 || v0 < 0) return set_error(HNH_E_INVALID, "%s: negative row or column offset", who);
    const double T = std::ceil(p * 4294967296.0);  // p 2^32 is exact
    dr->threshold = T >= 4294967295.0 ? 0xffffffffu : (uint32_t)T;
    dr->key = mix64(seed);
    dr->u0 = u0;
    dr->v0 = v0;
    dr->inv_keep = 1.0 / (1.0 - p);
    return HNH_OK;
}

template <bool DROP, bool BIAS, bool EDGE>
int step(const char *who, const int64_t *rowStart, const int64_t *col_idx, int64_t rows, int64_t nnz, int d, const double *Q,
         int64_t ldq, const double *K, int64_t ldk, const double *V, int64_t ldv, double scale, double *acc, int64_t ldacc,
         double *m, int64_t ldm, double *s, int64_t lds, const Dropout &dr, const Bias &bs, const Edge &eg, void *stream) {
    const std::initializer_list<Operand> ops = {{Q, ldq, true}, {K, ldk, true},   {V, ldv, true},
                                                {acc, ldacc, true}, {m, ldm, false}, {s, lds, false}};
    int v = check_call(who, rowStart, col_idx, rows, nnz, d, scale, ops);
    if (v < 0) return v;
    if (v == 1) return HNH_OK;
    cudaStream_t st = (cudaStream_t)stream;
    int grid = 0, rc = HNH_OK;
    if (fast_path(d, ops) && (!EDGE || edge_fast(eg))) {
#define STEP(RR, G, VW, UN)                                                                                                \
    {                                                                                                                      \
        auto k = attn_step_kernel<RR, G, VW, UN, DROP, BIAS, EDGE>;                                                              \
        rc = grid_for(k, rows, kBlock / G, &grid);                                                                         \
        if (!rc)                                                                                                           \
            rc = launch(k, grid, kBlock, st, "attn_step_kernel", rowStart, col_idx, rows, Q, ldq, K, ldk, V, ldv, scale, acc, ldacc, m, \
                        ldm, s, lds, dr, bs, eg);                                                                              \
    }
        HNH_DISPATCH_R(d, STEP, )
#undef STEP
        return rc;
    }
    auto k = attn_step_generic_kernel<DROP, BIAS, EDGE>;
    rc = grid_for(k, rows, kBlock / 32, &grid);
    return rc ? rc : launch(k, grid, kBlock, st, "attn_step_generic_kernel", rowStart, col_idx, rows, d, Q, ldq, K, ldk, V, ldv,
                            scale, acc, ldacc, m, ldm, s, lds, dr, bs, eg);
}

template <bool DROP, bool BIAS, bool EDGE>
int grad_q(const char *who, const int64_t *rowStart, const int64_t *col_idx, int64_t rows, int64_t nnz, int d, const double *Q,
           int64_t ldq, const double *dZ, int64_t lddz, const double *L, int64_t ldl, const double *t, int64_t ldt,
           const double *K, int64_t ldk, const double *V, int64_t ldv, double scale, double *dQ, int64_t lddq,
           const Dropout &dr, const Bias &bs, const Edge &eg, void *stream) {
    const std::initializer_list<Operand> ops = {{Q, ldq, true}, {dZ, lddz, true}, {L, ldl, false}, {t, ldt, false},
                                                {K, ldk, true}, {V, ldv, true},   {dQ, lddq, true}};
    int v = check_call(who, rowStart, col_idx, rows, nnz, d, scale, ops);
    if (v < 0) return v;
    if (v == 1) return HNH_OK;
    cudaStream_t st = (cudaStream_t)stream;
    int grid = 0, rc = HNH_OK;
    if (fast_path(d, ops) && (!EDGE || edge_fast(eg))) {
#define GQ(RR, G, VW, UN)                                                                                                  \
    {                                                                                                                      \
        auto k = attn_grad_q_kernel<RR, G, VW, UN, DROP, BIAS, EDGE>;                                                            \
        rc = grid_for(k, rows, kBlock / G, &grid);                                                                         \
        if (!rc)                                                                                                           \
            rc = launch(k, grid, kBlock, st, "attn_grad_q_kernel", rowStart, col_idx, rows, Q, ldq, dZ, lddz, L, ldl, t, ldt, K, ldk, \
                        V, ldv, scale, dQ, lddq, dr, bs, eg);                                                                  \
    }
        HNH_DISPATCH_R(d, GQ, )
#undef GQ
        return rc;
    }
    auto k = attn_grad_q_generic_kernel<DROP, BIAS, EDGE>;
    rc = grid_for(k, rows, kBlock / 32, &grid);
    return rc ? rc : launch(k, grid, kBlock, st, "attn_grad_q_generic_kernel", rowStart, col_idx, rows, d, Q, ldq, dZ, lddz, L,
                            ldl, t, ldt, K, ldk, V, ldv, scale, dQ, lddq, dr, bs, eg);
}

template <bool DROP, bool BIAS, bool EDGE>
int grad_kv(const char *who, const int64_t *rowStart, const int64_t *col_idx, int64_t rows, int64_t nnz, int d, const double *K,
            int64_t ldk, const double *V, int64_t ldv, const double *Q, int64_t ldq, const double *dZ, int64_t lddz,
            const double *L, int64_t ldl, const double *t, int64_t ldt, double scale, double *dK, int64_t lddk, double *dV,
            int64_t lddv, const Dropout &dr, const Bias &bs, const Edge &eg, void *stream) {
    const std::initializer_list<Operand> ops = {{K, ldk, true},   {V, ldv, true},   {Q, ldq, true},   {dZ, lddz, true},
                                                {L, ldl, false},  {t, ldt, false},  {dK, lddk, true}, {dV, lddv, true}};
    int v = check_call(who, rowStart, col_idx, rows, nnz, d, scale, ops);
    if (v < 0) return v;
    if (v == 1) return HNH_OK;
    cudaStream_t st = (cudaStream_t)stream;
    int grid = 0, rc = HNH_OK;
    if (fast_path(d, ops) && (!EDGE || edge_fast(eg))) {
#define GKV(RR, G, VW, UN)                                                                                                 \
    {                                                                                                                      \
        auto k = attn_grad_kv_kernel<RR, G, VW, UN, DROP, BIAS, EDGE>;                                                           \
        rc = grid_for(k, rows, kBlock / G, &grid);                                                                         \
        if (!rc)                                                                                                           \
            rc = launch(k, grid, kBlock, st, "attn_grad_kv_kernel", rowStart, col_idx, rows, K, ldk, V, ldv, Q, ldq, dZ, lddz, L, \
                        ldl, t, ldt, scale, dK, lddk, dV, lddv, dr, bs, eg);                                                   \
    }
        HNH_DISPATCH_R(d, GKV, )
#undef GKV
        return rc;
    }
    auto k = attn_grad_kv_generic_kernel<DROP, BIAS, EDGE>;
    rc = grid_for(k, rows, kBlock / 32, &grid);
    return rc ? rc : launch(k, grid, kBlock, st, "attn_grad_kv_generic_kernel", rowStart, col_idx, rows, d, K, ldk, V, ldv, Q,
                            ldq, dZ, lddz, L, ldl, t, ldt, scale, dK, lddk, dV, lddv, dr, bs, eg);
}

// The Dropout of a bias call (p = 0: the kernels without dropout) with its bias checked: HNH_OK or HNH_E_INVALID
int make_bias_call(const char *who, double p, uint64_t seed, int64_t u0, int64_t v0, const double *bias, Dropout *dr) {
    const int rc = make_dropout(who, p, seed, u0, v0, dr);
    if (rc) return rc;
    if (!bias) return set_error(HNH_E_INVALID, "%s: null bias", who);
    return HNH_OK;
}

// The Dropout of an edge call (p = 0: the kernels without dropout) with its edge operands and nullable bias checked:
// HNH_OK or HNH_E_INVALID
int make_edge_call(const char *who, int d, double p, uint64_t seed, int64_t u0, int64_t v0, const double *bias,
                   const double *dbias, const Edge &eg, Dropout *dr) {
    const int rc = make_dropout(who, p, seed, u0, v0, dr);
    if (rc) return rc;
    if (dbias && !bias) return set_error(HNH_E_INVALID, "%s: dbias without a bias", who);
    if (!eg.E) return set_error(HNH_E_INVALID, "%s: null E", who);
    if (eg.lde < d) return set_error(HNH_E_INVALID, "%s: lde %lld below d = %d", who, (long long)eg.lde, d);
    if (eg.dE && eg.ldde < d) return set_error(HNH_E_INVALID, "%s: ldde %lld below d = %d", who, (long long)eg.ldde, d);
    if (eg.dE && (const double *)eg.dE == eg.E) return set_error(HNH_E_INVALID, "%s: dE is E", who);
    return HNH_OK;
}

// The (DROP, BIAS) instantiation with EDGE = true of an edge call: DROP iff p > 0, BIAS iff a bias is given
#define HNH_EDGE_CALL(FN, ...)                                                                                             \
    (p == 0.0 ? (bias ? FN<false, true, true>(__VA_ARGS__) : FN<false, false, true>(__VA_ARGS__))                        \
              : (bias ? FN<true, true, true>(__VA_ARGS__) : FN<true, false, true>(__VA_ARGS__)))

}  // namespace

extern "C" {

int hnh_sparse_attention_step_f64(const int64_t *rowStart, const int64_t *col_idx, int64_t rows, int64_t nnz, int d,
                                  const double *Q, int64_t ldq, const double *K, int64_t ldk, const double *V, int64_t ldv,
                                  double scale, double *acc, int64_t ldacc, double *m, int64_t ldm, double *s, int64_t lds,
                                  void *stream) {
    return step<false, false, false>("hnh_sparse_attention_step_f64", rowStart, col_idx, rows, nnz, d, Q, ldq, K, ldk, V, ldv, scale,
                              acc, ldacc, m, ldm, s, lds, Dropout{}, Bias{}, Edge{}, stream);
}

int hnh_sparse_attention_step_dropout_f64(const int64_t *rowStart, const int64_t *col_idx, int64_t rows, int64_t nnz, int d,
                                          const double *Q, int64_t ldq, const double *K, int64_t ldk, const double *V,
                                          int64_t ldv, double scale, double *acc, int64_t ldacc, double *m, int64_t ldm,
                                          double *s, int64_t lds, double p, uint64_t seed, int64_t u0, int64_t v0,
                                          void *stream) {
    const char *who = "hnh_sparse_attention_step_dropout_f64";
    Dropout dr;
    const int rc = make_dropout(who, p, seed, u0, v0, &dr);
    return rc ? rc : step<true, false, false>(who, rowStart, col_idx, rows, nnz, d, Q, ldq, K, ldk, V, ldv, scale, acc, ldacc, m, ldm, s,
                                       lds, dr, Bias{}, Edge{}, stream);
}

int hnh_sparse_attention_step_bias_f64(const int64_t *rowStart, const int64_t *col_idx, int64_t rows, int64_t nnz, int d,
                                       const double *Q, int64_t ldq, const double *K, int64_t ldk, const double *V, int64_t ldv,
                                       double scale, double *acc, int64_t ldacc, double *m, int64_t ldm, double *s, int64_t lds,
                                       double p, uint64_t seed, int64_t u0, int64_t v0, const double *bias, void *stream) {
    const char *who = "hnh_sparse_attention_step_bias_f64";
    Dropout dr;
    const int rc = make_bias_call(who, p, seed, u0, v0, bias, &dr);
    if (rc) return rc;
    const Bias bs{bias, nullptr};
    return p == 0.0 ? step<false, true, false>(who, rowStart, col_idx, rows, nnz, d, Q, ldq, K, ldk, V, ldv, scale, acc, ldacc, m, ldm, s,
                                        lds, dr, bs, Edge{}, stream)
                    : step<true, true, false>(who, rowStart, col_idx, rows, nnz, d, Q, ldq, K, ldk, V, ldv, scale, acc, ldacc, m, ldm, s,
                                       lds, dr, bs, Edge{}, stream);
}

int hnh_sparse_attention_finish_f64(int64_t rows, int d, const double *acc, int64_t ldacc, const double *m, int64_t ldm,
                                    const double *s, int64_t lds, double *Z, int64_t ldz, double *L, int64_t ldl,
                                    void *stream) {
    const char *who = "hnh_sparse_attention_finish_f64";
    if (rows < 0) return set_error(HNH_E_INVALID, "%s: negative size", who);
    if (d < 1) return set_error(HNH_E_INVALID, "%s: d must be positive (got %d)", who, d);
    if (ldacc < d || ldz < d || ldm < 1 || lds < 1 || ldl < 1)
        return set_error(HNH_E_INVALID, "%s: leading dimension below d = %d (rows) or 1 (scalars)", who, d);
    if (rows == 0) return HNH_OK;
    if (!acc || !m || !s || !Z || !L) return set_error(HNH_E_INVALID, "%s: null pointer", who);
    int grid = 0;
    int rc = grid_for(attn_finish_kernel, rows * d, kBlock, &grid);
    return rc ? rc : launch(attn_finish_kernel, grid, kBlock, (cudaStream_t)stream, "attn_finish_kernel", rows, d, acc, ldacc, m, ldm, s,
                            lds, Z, ldz, L, ldl);
}

int hnh_sparse_attention_grad_q_f64(const int64_t *rowStart, const int64_t *col_idx, int64_t rows, int64_t nnz, int d,
                                    const double *Q, int64_t ldq, const double *dZ, int64_t lddz, const double *L, int64_t ldl,
                                    const double *t, int64_t ldt, const double *K, int64_t ldk, const double *V, int64_t ldv,
                                    double scale, double *dQ, int64_t lddq, void *stream) {
    return grad_q<false, false, false>("hnh_sparse_attention_grad_q_f64", rowStart, col_idx, rows, nnz, d, Q, ldq, dZ, lddz, L, ldl, t,
                                ldt, K, ldk, V, ldv, scale, dQ, lddq, Dropout{}, Bias{}, Edge{}, stream);
}

int hnh_sparse_attention_grad_q_dropout_f64(const int64_t *rowStart, const int64_t *col_idx, int64_t rows, int64_t nnz, int d,
                                            const double *Q, int64_t ldq, const double *dZ, int64_t lddz, const double *L,
                                            int64_t ldl, const double *t, int64_t ldt, const double *K, int64_t ldk,
                                            const double *V, int64_t ldv, double scale, double *dQ, int64_t lddq, double p,
                                            uint64_t seed, int64_t u0, int64_t v0, void *stream) {
    const char *who = "hnh_sparse_attention_grad_q_dropout_f64";
    Dropout dr;
    const int rc = make_dropout(who, p, seed, u0, v0, &dr);
    return rc ? rc : grad_q<true, false, false>(who, rowStart, col_idx, rows, nnz, d, Q, ldq, dZ, lddz, L, ldl, t, ldt, K, ldk, V, ldv,
                                         scale, dQ, lddq, dr, Bias{}, Edge{}, stream);
}

int hnh_sparse_attention_grad_q_bias_f64(const int64_t *rowStart, const int64_t *col_idx, int64_t rows, int64_t nnz, int d,
                                         const double *Q, int64_t ldq, const double *dZ, int64_t lddz, const double *L,
                                         int64_t ldl, const double *t, int64_t ldt, const double *K, int64_t ldk,
                                         const double *V, int64_t ldv, double scale, double *dQ, int64_t lddq, double p,
                                         uint64_t seed, int64_t u0, int64_t v0, const double *bias, double *dbias,
                                         void *stream) {
    const char *who = "hnh_sparse_attention_grad_q_bias_f64";
    Dropout dr;
    const int rc = make_bias_call(who, p, seed, u0, v0, bias, &dr);
    if (rc) return rc;
    const Bias bs{bias, dbias};
    return p == 0.0 ? grad_q<false, true, false>(who, rowStart, col_idx, rows, nnz, d, Q, ldq, dZ, lddz, L, ldl, t, ldt, K, ldk, V, ldv,
                                          scale, dQ, lddq, dr, bs, Edge{}, stream)
                    : grad_q<true, true, false>(who, rowStart, col_idx, rows, nnz, d, Q, ldq, dZ, lddz, L, ldl, t, ldt, K, ldk, V, ldv,
                                         scale, dQ, lddq, dr, bs, Edge{}, stream);
}

int hnh_sparse_attention_grad_kv_f64(const int64_t *rowStart, const int64_t *col_idx, int64_t rows, int64_t nnz, int d,
                                     const double *K, int64_t ldk, const double *V, int64_t ldv, const double *Q, int64_t ldq,
                                     const double *dZ, int64_t lddz, const double *L, int64_t ldl, const double *t, int64_t ldt,
                                     double scale, double *dK, int64_t lddk, double *dV, int64_t lddv, void *stream) {
    return grad_kv<false, false, false>("hnh_sparse_attention_grad_kv_f64", rowStart, col_idx, rows, nnz, d, K, ldk, V, ldv, Q, ldq, dZ,
                                 lddz, L, ldl, t, ldt, scale, dK, lddk, dV, lddv, Dropout{}, Bias{}, Edge{}, stream);
}

int hnh_sparse_attention_grad_kv_dropout_f64(const int64_t *rowStart, const int64_t *col_idx, int64_t rows, int64_t nnz, int d,
                                             const double *K, int64_t ldk, const double *V, int64_t ldv, const double *Q,
                                             int64_t ldq, const double *dZ, int64_t lddz, const double *L, int64_t ldl,
                                             const double *t, int64_t ldt, double scale, double *dK, int64_t lddk, double *dV,
                                             int64_t lddv, double p, uint64_t seed, int64_t u0, int64_t v0, void *stream) {
    const char *who = "hnh_sparse_attention_grad_kv_dropout_f64";
    Dropout dr;
    const int rc = make_dropout(who, p, seed, u0, v0, &dr);
    return rc ? rc : grad_kv<true, false, false>(who, rowStart, col_idx, rows, nnz, d, K, ldk, V, ldv, Q, ldq, dZ, lddz, L, ldl, t, ldt,
                                          scale, dK, lddk, dV, lddv, dr, Bias{}, Edge{}, stream);
}

int hnh_sparse_attention_grad_kv_bias_f64(const int64_t *rowStart, const int64_t *col_idx, int64_t rows, int64_t nnz, int d,
                                          const double *K, int64_t ldk, const double *V, int64_t ldv, const double *Q,
                                          int64_t ldq, const double *dZ, int64_t lddz, const double *L, int64_t ldl,
                                          const double *t, int64_t ldt, double scale, double *dK, int64_t lddk, double *dV,
                                          int64_t lddv, double p, uint64_t seed, int64_t u0, int64_t v0, const double *bias,
                                          double *dbias, void *stream) {
    const char *who = "hnh_sparse_attention_grad_kv_bias_f64";
    Dropout dr;
    const int rc = make_bias_call(who, p, seed, u0, v0, bias, &dr);
    if (rc) return rc;
    const Bias bs{bias, dbias};
    return p == 0.0 ? grad_kv<false, true, false>(who, rowStart, col_idx, rows, nnz, d, K, ldk, V, ldv, Q, ldq, dZ, lddz, L, ldl, t, ldt,
                                           scale, dK, lddk, dV, lddv, dr, bs, Edge{}, stream)
                    : grad_kv<true, true, false>(who, rowStart, col_idx, rows, nnz, d, K, ldk, V, ldv, Q, ldq, dZ, lddz, L, ldl, t, ldt,
                                          scale, dK, lddk, dV, lddv, dr, bs, Edge{}, stream);
}

int hnh_sparse_attention_step_edge_f64(const int64_t *rowStart, const int64_t *col_idx, int64_t rows, int64_t nnz, int d,
                                       const double *Q, int64_t ldq, const double *K, int64_t ldk, const double *V, int64_t ldv,
                                       double scale, double *acc, int64_t ldacc, double *m, int64_t ldm, double *s, int64_t lds,
                                       double p, uint64_t seed, int64_t u0, int64_t v0, const double *bias, const double *E,
                                       int64_t lde, void *stream) {
    const char *who = "hnh_sparse_attention_step_edge_f64";
    const Edge eg{E, lde, nullptr, 0};
    Dropout dr;
    const int rc = make_edge_call(who, d, p, seed, u0, v0, bias, nullptr, eg, &dr);
    if (rc) return rc;
    const Bias bs{bias, nullptr};
    return HNH_EDGE_CALL(step, who, rowStart, col_idx, rows, nnz, d, Q, ldq, K, ldk, V, ldv, scale, acc, ldacc, m, ldm, s, lds,
                         dr, bs, eg, stream);
}

int hnh_sparse_attention_grad_q_edge_f64(const int64_t *rowStart, const int64_t *col_idx, int64_t rows, int64_t nnz, int d,
                                         const double *Q, int64_t ldq, const double *dZ, int64_t lddz, const double *L,
                                         int64_t ldl, const double *t, int64_t ldt, const double *K, int64_t ldk,
                                         const double *V, int64_t ldv, double scale, double *dQ, int64_t lddq, double p,
                                         uint64_t seed, int64_t u0, int64_t v0, const double *bias, double *dbias,
                                         const double *E, int64_t lde, double *dE, int64_t ldde, void *stream) {
    const char *who = "hnh_sparse_attention_grad_q_edge_f64";
    const Edge eg{E, lde, dE, ldde};
    Dropout dr;
    const int rc = make_edge_call(who, d, p, seed, u0, v0, bias, dbias, eg, &dr);
    if (rc) return rc;
    const Bias bs{bias, dbias};
    return HNH_EDGE_CALL(grad_q, who, rowStart, col_idx, rows, nnz, d, Q, ldq, dZ, lddz, L, ldl, t, ldt, K, ldk, V, ldv, scale,
                         dQ, lddq, dr, bs, eg, stream);
}

int hnh_sparse_attention_grad_kv_edge_f64(const int64_t *rowStart, const int64_t *col_idx, int64_t rows, int64_t nnz, int d,
                                          const double *K, int64_t ldk, const double *V, int64_t ldv, const double *Q,
                                          int64_t ldq, const double *dZ, int64_t lddz, const double *L, int64_t ldl,
                                          const double *t, int64_t ldt, double scale, double *dK, int64_t lddk, double *dV,
                                          int64_t lddv, double p, uint64_t seed, int64_t u0, int64_t v0, const double *bias,
                                          double *dbias, const double *E, int64_t lde, void *stream) {
    const char *who = "hnh_sparse_attention_grad_kv_edge_f64";
    const Edge eg{E, lde, nullptr, 0};
    Dropout dr;
    const int rc = make_edge_call(who, d, p, seed, u0, v0, bias, dbias, eg, &dr);
    if (rc) return rc;
    const Bias bs{bias, dbias};
    return HNH_EDGE_CALL(grad_kv, who, rowStart, col_idx, rows, nnz, d, K, ldk, V, ldv, Q, ldq, dZ, lddz, L, ldl, t, ldt, scale,
                         dK, lddk, dV, lddv, dr, bs, eg, stream);
}

}  // extern "C"
