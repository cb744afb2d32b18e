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
#include <cmath>

#include "row_gather.cuh"

namespace {

using hnh::grid_for;
using hnh::launch;
using hnh::set_error;

template <int G>
__device__ __forceinline__ double group_max(double d, unsigned mask) {
#pragma unroll
    for (int o = G / 2; o > 0; o >>= 1) d = fmax(d, __shfl_xor_sync(mask, d, o, G));
    return d;
}

// ---- fast row kernels ----------------------------------------------------------------------------------------
template <int R, int G, int VW, int UN>
__global__ void __launch_bounds__(kBlock, 1)
attn_step_kernel(const int64_t *__restrict__ rowStart, const int64_t *__restrict__ col_idx, int64_t rows,
                 const double *__restrict__ Q, int64_t ldq, const double *__restrict__ K, int64_t ldk,
                 const double *__restrict__ V, int64_t ldv, double scale, double *__restrict__ acc, int64_t ldacc,
                 double *__restrict__ m, int64_t ldm, double *__restrict__ s, int64_t lds) {
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
            if (gl < cnt) mycol = ld_stream_i64(col_idx + j + gl);
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
                    if (gl == k0 + u && k0 + u < cnt) mine = scale * d;
                }
            }
            // one rescale to the chunk's maximum (exp(-inf) = 0 for a row's first chunk)
            const double mnew = fmax(mrow, group_max<G>(mine, gmask));
            const double f = exp(mrow - mnew);
#pragma unroll
            for (int v = 0; v < NV; v++)
#pragma unroll
                for (int w = 0; w < VW; w++) a[v][w] *= f;
            srow *= f;
            mrow = mnew;
            const double pmine = gl < cnt ? exp(mine - mnew) : 0.0;
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
                    if (k < cnt) {
#pragma unroll
                        for (int v = 0; v < NV; v++) ld_gather<VW>(y[u][v], V + c * ldv + (v * G + gl) * VW);
                    }
                }
#pragma unroll
                for (int u = 0; u < UN; u++) {
                    if (k0 + u < cnt) {
#pragma unroll
                        for (int v = 0; v < NV; v++)
#pragma unroll
                            for (int w = 0; w < VW; w++) a[v][w] = fma(pv[u], y[u][v][w], a[v][w]);
                        srow += pv[u];
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

template <int R, int G, int VW, int UN>
__global__ void __launch_bounds__(kBlock, 1)
attn_grad_q_kernel(const int64_t *__restrict__ rowStart, const int64_t *__restrict__ col_idx, int64_t rows,
                   const double *__restrict__ Q, int64_t ldq, const double *__restrict__ dZ, int64_t lddz,
                   const double *__restrict__ L, int64_t ldl, const double *__restrict__ t, int64_t ldt,
                   const double *__restrict__ K, int64_t ldk, const double *__restrict__ V, int64_t ldv, double scale,
                   double *__restrict__ dQ, int64_t lddq) {
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
            if (gl < cnt) mycol = ld_stream_i64(col_idx + j + gl);
            for (int k0 = 0; k0 < cnt; k0 += UN) {
                double yk[UN][NV][VW], yv[UN][NV][VW];
#pragma unroll
                for (int u = 0; u < UN; u++) {
                    const int k = k0 + u;
                    const int64_t c = __shfl_sync(gmask, mycol, k < G ? k : G - 1, G);
                    if (k < cnt) {
#pragma unroll
                        for (int v = 0; v < NV; v++) {
                            ld_gather<VW>(yk[u][v], K + c * ldk + (v * G + gl) * VW);
                            ld_gather<VW>(yv[u][v], V + c * ldv + (v * G + gl) * VW);
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
                        const double dx = exp(scale * d1 - Lr) * (d2 - tr);
#pragma unroll
                        for (int v = 0; v < NV; v++)
#pragma unroll
                            for (int w = 0; w < VW; w++) a[v][w] = fma(dx, yk[u][v][w], a[v][w]);
                    }
                }
            }
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

template <int R, int G, int VW, int UN>
__global__ void __launch_bounds__(kBlock, 1)
attn_grad_kv_kernel(const int64_t *__restrict__ rowStart, const int64_t *__restrict__ col_idx, int64_t rows,
                    const double *__restrict__ K, int64_t ldk, const double *__restrict__ V, int64_t ldv,
                    const double *__restrict__ Q, int64_t ldq, const double *__restrict__ dZ, int64_t lddz,
                    const double *__restrict__ L, int64_t ldl, const double *__restrict__ t, int64_t ldt, double scale,
                    double *__restrict__ dK, int64_t lddk, double *__restrict__ dV, int64_t lddv) {
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
            double myL = 0.0, myt = 0.0;
            if (gl < cnt) {
                mycol = ld_stream_i64(col_idx + j + gl);
                myL = L[mycol * ldl];
                myt = t[mycol * ldt];
            }
            for (int k0 = 0; k0 < cnt; k0 += UN) {
                double yq[UN][NV][VW], yd[UN][NV][VW];
                double Lu[UN], tu[UN];
#pragma unroll
                for (int u = 0; u < UN; u++) {
                    const int k = k0 + u;
                    const int src = k < G ? k : G - 1;
                    const int64_t c = __shfl_sync(gmask, mycol, src, G);
                    Lu[u] = __shfl_sync(gmask, myL, src, G);
                    tu[u] = __shfl_sync(gmask, myt, src, G);
                    if (k < cnt) {
#pragma unroll
                        for (int v = 0; v < NV; v++) {
                            ld_gather<VW>(yq[u][v], Q + c * ldq + (v * G + gl) * VW);
                            ld_gather<VW>(yd[u][v], dZ + c * lddz + (v * G + gl) * VW);
                        }
                    } else {
#pragma unroll
                        for (int v = 0; v < NV; v++)
#pragma unroll
                            for (int w = 0; w < VW; w++) yq[u][v][w] = yd[u][v][w] = 0.0;
                    }
                }
#pragma unroll
                for (int u = 0; u < UN; u++) {
                    double d1 = 0.0, d2 = 0.0;
#pragma unroll
                    for (int v = 0; v < NV; v++)
#pragma unroll
                        for (int w = 0; w < VW; w++) {
                            d1 = fma(kr[v][w], yq[u][v][w], d1);
                            d2 = fma(vr[v][w], yd[u][v][w], d2);
                        }
                    d1 = group_allreduce<G>(d1, gmask);
                    d2 = group_allreduce<G>(d2, gmask);
                    if (k0 + u < cnt) {
                        const double al = exp(scale * d1 - Lu[u]);
                        const double dx = al * (d2 - tu[u]);
#pragma unroll
                        for (int v = 0; v < NV; v++)
#pragma unroll
                            for (int w = 0; w < VW; w++) {
                                ak[v][w] = fma(dx, yq[u][v][w], ak[v][w]);
                                av[v][w] = fma(al, yd[u][v][w], av[v][w]);
                            }
                    }
                }
            }
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

__global__ void __launch_bounds__(kBlock)
attn_step_generic_kernel(const int64_t *__restrict__ rowStart, const int64_t *__restrict__ col_idx, int64_t rows, int d,
                         const double *__restrict__ Q, int64_t ldq, const double *__restrict__ K, int64_t ldk,
                         const double *__restrict__ V, int64_t ldv, double scale, double *__restrict__ acc,
                         int64_t ldacc, double *__restrict__ m, int64_t ldm, double *__restrict__ s, int64_t lds) {
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
            const double x = scale * warp_dot(Q + row * ldq, K + c * ldk, d, lane);
            const double mnew = fmax(mrow, x);
            const double f = exp(mrow - mnew), pj = exp(x - mnew);
            for (int k = lane; k < d; k += 32) a[k] = fma(pj, V[c * ldv + k], a[k] * f);
            srow = fma(srow, f, pj);
            mrow = mnew;
        }
        if (lane == 0) {
            m[row * ldm] = mrow;
            s[row * lds] = srow;
        }
    }
}

__global__ void __launch_bounds__(kBlock)
attn_grad_q_generic_kernel(const int64_t *__restrict__ rowStart, const int64_t *__restrict__ col_idx, int64_t rows, int d,
                           const double *__restrict__ Q, int64_t ldq, const double *__restrict__ dZ, int64_t lddz,
                           const double *__restrict__ L, int64_t ldl, const double *__restrict__ t, int64_t ldt,
                           const double *__restrict__ K, int64_t ldk, const double *__restrict__ V, int64_t ldv,
                           double scale, double *__restrict__ dQ, int64_t lddq) {
    const int lane = threadIdx.x & 31;
    const int64_t warps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t row = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; row < rows; row += warps) {
        const int64_t s0 = rowStart[row], e = rowStart[row + 1];
        if (s0 == e) continue;
        const double Lr = L[row * ldl], tr = t[row * ldt];
        for (int64_t j = s0; j < e; j++) {
            const int64_t c = col_idx[j];
            const double d1 = warp_dot(Q + row * ldq, K + c * ldk, d, lane);
            const double d2 = warp_dot(dZ + row * lddz, V + c * ldv, d, lane);
            const double g = scale * (exp(scale * d1 - Lr) * (d2 - tr));
            for (int k = lane; k < d; k += 32) dQ[row * lddq + k] = fma(g, K[c * ldk + k], dQ[row * lddq + k]);
        }
    }
}

__global__ void __launch_bounds__(kBlock)
attn_grad_kv_generic_kernel(const int64_t *__restrict__ rowStart, const int64_t *__restrict__ col_idx, int64_t rows, int d,
                            const double *__restrict__ K, int64_t ldk, const double *__restrict__ V, int64_t ldv,
                            const double *__restrict__ Q, int64_t ldq, const double *__restrict__ dZ, int64_t lddz,
                            const double *__restrict__ L, int64_t ldl, const double *__restrict__ t, int64_t ldt,
                            double scale, double *__restrict__ dK, int64_t lddk, double *__restrict__ dV, int64_t lddv) {
    const int lane = threadIdx.x & 31;
    const int64_t warps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t row = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; row < rows; row += warps) {
        const int64_t s0 = rowStart[row], e = rowStart[row + 1];
        for (int64_t j = s0; j < e; j++) {
            const int64_t u = col_idx[j];
            const double d1 = warp_dot(K + row * ldk, Q + u * ldq, d, lane);
            const double d2 = warp_dot(V + row * ldv, dZ + u * lddz, d, lane);
            const double al = exp(scale * d1 - L[u * ldl]);
            const double g = scale * (al * (d2 - t[u * ldt]));
            for (int k = lane; k < d; k += 32) {
                dK[row * lddk + k] = fma(g, Q[u * ldq + k], dK[row * lddk + k]);
                dV[row * lddv + k] = fma(al, dZ[u * lddz + k], dV[row * lddv + k]);
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

}  // namespace

extern "C" {

int hnh_sparse_attention_step_f64(const int64_t *rowStart, const int64_t *col_idx, int64_t rows, int64_t nnz, int d,
                                  const double *Q, int64_t ldq, const double *K, int64_t ldk, const double *V, int64_t ldv,
                                  double scale, double *acc, int64_t ldacc, double *m, int64_t ldm, double *s, int64_t lds,
                                  void *stream) {
    const std::initializer_list<Operand> ops = {{Q, ldq, true}, {K, ldk, true},   {V, ldv, true},
                                                {acc, ldacc, true}, {m, ldm, false}, {s, lds, false}};
    int v = check_call("hnh_sparse_attention_step_f64", rowStart, col_idx, rows, nnz, d, scale, ops);
    if (v < 0) return v;
    if (v == 1) return HNH_OK;
    cudaStream_t st = (cudaStream_t)stream;
    int grid = 0, rc = HNH_OK;
    if (fast_path(d, ops)) {
#define STEP(RR, G, VW, UN)                                                                                                \
    {                                                                                                                      \
        auto k = attn_step_kernel<RR, G, VW, UN>;                                                                          \
        rc = grid_for(k, rows, kBlock / G, &grid);                                                                         \
        if (!rc)                                                                                                           \
            rc = launch(k, grid, kBlock, st, "attn_step_kernel", rowStart, col_idx, rows, Q, ldq, K, ldk, V, ldv, scale, acc, ldacc, m, \
                        ldm, s, lds);                                                                                      \
    }
        HNH_DISPATCH_R(d, STEP, )
#undef STEP
        return rc;
    }
    rc = grid_for(attn_step_generic_kernel, rows, kBlock / 32, &grid);
    return rc ? rc : launch(attn_step_generic_kernel, grid, kBlock, st, "attn_step_generic_kernel", rowStart, col_idx, rows, d, Q, ldq, K,
                            ldk, V, ldv, scale, acc, ldacc, m, ldm, s, lds);
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
    const std::initializer_list<Operand> ops = {{Q, ldq, true}, {dZ, lddz, true}, {L, ldl, false}, {t, ldt, false},
                                                {K, ldk, true}, {V, ldv, true},   {dQ, lddq, true}};
    int v = check_call("hnh_sparse_attention_grad_q_f64", rowStart, col_idx, rows, nnz, d, scale, ops);
    if (v < 0) return v;
    if (v == 1) return HNH_OK;
    cudaStream_t st = (cudaStream_t)stream;
    int grid = 0, rc = HNH_OK;
    if (fast_path(d, ops)) {
#define GQ(RR, G, VW, UN)                                                                                                  \
    {                                                                                                                      \
        auto k = attn_grad_q_kernel<RR, G, VW, UN>;                                                                        \
        rc = grid_for(k, rows, kBlock / G, &grid);                                                                         \
        if (!rc)                                                                                                           \
            rc = launch(k, grid, kBlock, st, "attn_grad_q_kernel", rowStart, col_idx, rows, Q, ldq, dZ, lddz, L, ldl, t, ldt, K, ldk, \
                        V, ldv, scale, dQ, lddq);                                                                          \
    }
        HNH_DISPATCH_R(d, GQ, )
#undef GQ
        return rc;
    }
    rc = grid_for(attn_grad_q_generic_kernel, rows, kBlock / 32, &grid);
    return rc ? rc : launch(attn_grad_q_generic_kernel, grid, kBlock, st, "attn_grad_q_generic_kernel", rowStart, col_idx, rows, d, Q, ldq,
                            dZ, lddz, L, ldl, t, ldt, K, ldk, V, ldv, scale, dQ, lddq);
}

int hnh_sparse_attention_grad_kv_f64(const int64_t *rowStart, const int64_t *col_idx, int64_t rows, int64_t nnz, int d,
                                     const double *K, int64_t ldk, const double *V, int64_t ldv, const double *Q, int64_t ldq,
                                     const double *dZ, int64_t lddz, const double *L, int64_t ldl, const double *t, int64_t ldt,
                                     double scale, double *dK, int64_t lddk, double *dV, int64_t lddv, void *stream) {
    const std::initializer_list<Operand> ops = {{K, ldk, true},   {V, ldv, true},   {Q, ldq, true},   {dZ, lddz, true},
                                                {L, ldl, false},  {t, ldt, false},  {dK, lddk, true}, {dV, lddv, true}};
    int v = check_call("hnh_sparse_attention_grad_kv_f64", rowStart, col_idx, rows, nnz, d, scale, ops);
    if (v < 0) return v;
    if (v == 1) return HNH_OK;
    cudaStream_t st = (cudaStream_t)stream;
    int grid = 0, rc = HNH_OK;
    if (fast_path(d, ops)) {
#define GKV(RR, G, VW, UN)                                                                                                 \
    {                                                                                                                      \
        auto k = attn_grad_kv_kernel<RR, G, VW, UN>;                                                                       \
        rc = grid_for(k, rows, kBlock / G, &grid);                                                                         \
        if (!rc)                                                                                                           \
            rc = launch(k, grid, kBlock, st, "attn_grad_kv_kernel", rowStart, col_idx, rows, K, ldk, V, ldv, Q, ldq, dZ, lddz, L, \
                        ldl, t, ldt, scale, dK, lddk, dV, lddv);                                                           \
    }
        HNH_DISPATCH_R(d, GKV, )
#undef GKV
        return rc;
    }
    rc = grid_for(attn_grad_kv_generic_kernel, rows, kBlock / 32, &grid);
    return rc ? rc : launch(attn_grad_kv_generic_kernel, grid, kBlock, st, "attn_grad_kv_generic_kernel", rowStart, col_idx, rows, d, K,
                            ldk, V, ldv, Q, ldq, dZ, lddz, L, ldl, t, ldt, scale, dK, lddk, dV, lddv);
}

}  // extern "C"
