// graph_transformer.cu -- the row-wise device operations of the graph transformer (include/hnh/graph_transformer.hpp)
// beyond the projections (hnh_dgemm_f64 and friends) and fused sparse attention.  All matrices are row-major n x r
// and contiguous; w_beta (nullable) holds 3r doubles [w1 | w2 | w3]:
//     X[i, :] += b                                            projection bias                 (row_bias_kernel)
//     s_i = <w1, M_i> + <w2, R_i> + <w3, M_i - R_i>,  beta_i = sigmoid(s_i)
//     Y_i = beta_i R_i + (1 - beta_i) M_i   (M_i + R_i without w_beta),  then ReLU when asked
//                                                             the gate forward                (gate_kernel)
// Backward, with dY = G, or G where Y > 0 after a ReLU, and ds_i = <dY_i, R_i - M_i> beta_i (1 - beta_i):
//     dM_i = (1 - beta_i) dY_i + ds_i (w1 + w3),  dR_i = beta_i dY_i + ds_i (w2 - w3)   (dM = dR = dY without w_beta)
//                                                             one row pass                    (gate_backward_kernel)
//     dw_beta = sum_i ds_i [M_i, R_i, M_i - R_i]              two stages: fixed row chunks     (gate_dw_partial_kernel)
//                                                             then the chunks in order         (gate_dw_final_kernel)
//
// The row kernels run one warp per row: lanes stride the row in 16-byte pairs when r is even and every row pointer is
// 16-byte aligned, in scalars otherwise, and a row's dot products end in the warp's xor butterfly, which leaves the
// same bits on every lane.  The dw_beta chunks depend on n only, never on the device, so repeated calls are
// bit-identical everywhere.  No floating-point atomics.
//
// The transformer block (ffn_ratio > 0) adds, on rows of width r (or h for the feed-forward hidden layer):
//     Z[i, :] = max(A[i, :] + b, 0)                           first FFN layer's bias and ReLU (row_bias_relu_kernel)
//     Y_i = gamma (x_i - mean_i) rstd_i + beta,  x = X + Res (Res nullable),  rstd_i = 1 / sqrt(var_i + eps)
//                                                             LayerNorm; (mean, rstd) per row   (layer_norm_kernel)
//     dX_i = rstd_i (g_i - mean(g_i) - xh_i mean(g_i xh_i)),  g = G gamma,  xh = (x - mean) rstd
//                                                             one row pass, dX overwritten or added to
//                                                                                       (layer_norm_backward_kernel)
//     dgamma = sum_i G_i xh_i,  dbeta = sum_i G_i              the dw_beta scheme: fixed row chunks
//                                                             (layer_norm_dw_partial_kernel), then gate_dw_final_kernel
// The LayerNorm kernels hold a row in registers (r <= 1536 forward, r <= 1024 backward), so it is read from HBM once; the
// variance is taken from the centred values.  Wider rows reread the row from L1 / L2 in every pass.
#include <cmath>

#include "row_regs.cuh"

namespace {

using hnh::grid_for;
using hnh::launch;
using hnh::set_error;

constexpr int kCtasPerSm = 16;         // grid cap of the row kernels
// register rows of the LayerNorm kernels up to r = 64 * this: the forward keeps one row (x), the backward two (G and
// xh), and ptxas spills the backward's at 24
constexpr int kLnWidest = 24, kLnBackwardWidest = 16;

__device__ __forceinline__ double sigmoid(double s) { return 1.0 / (1.0 + exp(-s)); }

// X[i, :] += b
template <bool kPairs>
__global__ void __launch_bounds__(kBlock) row_bias_kernel(double *__restrict__ X, const double *__restrict__ b, int64_t n, int64_t r) {
    const int lane = threadIdx.x & 31;
    const int64_t warps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t i = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; i < n; i += warps) {
        if (kPairs) {
            double2 *row = reinterpret_cast<double2 *>(X + i * r);
            const double2 *bb = reinterpret_cast<const double2 *>(b);
#pragma unroll 2  // ptxas spills 8 bytes at its default unroll of this loop
            for (int64_t k = lane; k < r / 2; k += 32) {
                const double2 v = row[k], c = __ldg(bb + k);
                row[k] = make_double2(v.x + c.x, v.y + c.y);
            }
        } else {
            double *row = X + i * r;
            for (int64_t k = lane; k < r; k += 32) row[k] += __ldg(b + k);
        }
    }
}

// s_i of row i: the gate's logit, the same bits on every lane
template <bool kPairs>
__device__ __forceinline__ double gate_logit(const double *m, const double *rr, const double *w, int64_t r, int lane) {
    double x = 0.0;
    if (kPairs) {
        const double2 *m2 = reinterpret_cast<const double2 *>(m), *r2 = reinterpret_cast<const double2 *>(rr);
        const double2 *w1 = reinterpret_cast<const double2 *>(w), *w2 = reinterpret_cast<const double2 *>(w + r),
                      *w3 = reinterpret_cast<const double2 *>(w + 2 * r);
        for (int64_t k = lane; k < r / 2; k += 32) {
            const double2 a = m2[k], c = r2[k], u = __ldg(w1 + k), v = __ldg(w2 + k), z = __ldg(w3 + k);
            x = fma(u.x, a.x, x);
            x = fma(v.x, c.x, x);
            x = fma(z.x, a.x - c.x, x);
            x = fma(u.y, a.y, x);
            x = fma(v.y, c.y, x);
            x = fma(z.y, a.y - c.y, x);
        }
    } else {
        for (int64_t k = lane; k < r; k += 32) {
            const double a = m[k], c = rr[k];
            x = fma(__ldg(w + k), a, x);
            x = fma(__ldg(w + r + k), c, x);
            x = fma(__ldg(w + 2 * r + k), a - c, x);
        }
    }
    return group_allreduce<32>(x, 0xffffffffu);
}

// Y = beta R + (1 - beta) M (M + R when !kBeta), ReLU when kRelu.  With the gate, the logit pass reads M and R
// through L1 and the combine pass rereads them there.
template <bool kPairs, bool kBeta, bool kRelu>
__global__ void __launch_bounds__(kBlock)
gate_kernel(double *__restrict__ Y, const double *__restrict__ M, const double *__restrict__ R, const double *__restrict__ w,
            int64_t n, int64_t r) {
    const int lane = threadIdx.x & 31;
    const int64_t warps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t i = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; i < n; i += warps) {
        const double *m = M + i * r, *rr = R + i * r;
        double beta = 0.0;
        if (kBeta) beta = sigmoid(gate_logit<kPairs>(m, rr, w, r, lane));
        auto combine = [&](double a, double c) {
            const double y = kBeta ? fma(beta, c, (1.0 - beta) * a) : a + c;
            return kRelu ? fmax(y, 0.0) : y;
        };
        if (kPairs) {
            const double2 *m2 = reinterpret_cast<const double2 *>(m), *r2 = reinterpret_cast<const double2 *>(rr);
            double2 *y2 = reinterpret_cast<double2 *>(Y + i * r);
            for (int64_t k = lane; k < r / 2; k += 32) {
                const double2 a = __ldcs(m2 + k), c = __ldcs(r2 + k);
                __stcs(y2 + k, make_double2(combine(a.x, c.x), combine(a.y, c.y)));
            }
        } else {
            double *y = Y + i * r;
            for (int64_t k = lane; k < r; k += 32) __stcs(y + k, combine(__ldcs(m + k), __ldcs(rr + k)));
        }
    }
}

// dM, dR (dR nullable without the gate) and ds_i (with the gate) of every row
template <bool kPairs, bool kBeta, bool kRelu>
__global__ void __launch_bounds__(kBlock)
gate_backward_kernel(double *__restrict__ dM, double *__restrict__ dR, double *__restrict__ ds_out, const double *__restrict__ G,
                     const double *__restrict__ Y, const double *__restrict__ M, const double *__restrict__ R,
                     const double *__restrict__ w, int64_t n, int64_t r) {
    const int lane = threadIdx.x & 31;
    const int64_t warps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t i = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; i < n; i += warps) {
        const double *g = G + i * r, *y = kRelu ? Y + i * r : nullptr, *m = M + i * r, *rr = R + i * r;
        auto dy = [&](double gk, double yk) { return kRelu ? (yk > 0.0 ? gk : 0.0) : gk; };
        double beta = 0.0, ds = 0.0;
        if (kBeta) {
            beta = sigmoid(gate_logit<kPairs>(m, rr, w, r, lane));
            double t = 0.0;
            if (kPairs) {
                const double2 *g2 = reinterpret_cast<const double2 *>(g), *y2 = reinterpret_cast<const double2 *>(y),
                              *m2 = reinterpret_cast<const double2 *>(m), *r2 = reinterpret_cast<const double2 *>(rr);
                for (int64_t k = lane; k < r / 2; k += 32) {
                    const double2 gk = g2[k], a = m2[k], c = r2[k];
                    double2 yk = make_double2(0.0, 0.0);
                    if (kRelu) yk = y2[k];
                    t = fma(dy(gk.x, yk.x), c.x - a.x, t);
                    t = fma(dy(gk.y, yk.y), c.y - a.y, t);
                }
            } else {
                for (int64_t k = lane; k < r; k += 32) t = fma(dy(g[k], kRelu ? y[k] : 0.0), rr[k] - m[k], t);
            }
            ds = group_allreduce<32>(t, 0xffffffffu) * beta * (1.0 - beta);
            if (lane == 0) ds_out[i] = ds;
        }
        if (kPairs) {
            const double2 *g2 = reinterpret_cast<const double2 *>(g), *y2 = reinterpret_cast<const double2 *>(y);
            double2 *dm2 = reinterpret_cast<double2 *>(dM + i * r), *dr2 = dR ? reinterpret_cast<double2 *>(dR + i * r) : nullptr;
            for (int64_t k = lane; k < r / 2; k += 32) {
                const double2 gk = __ldcs(g2 + k);
                double2 yk = make_double2(0.0, 0.0);
                if (kRelu) yk = __ldcs(y2 + k);
                const double ax = dy(gk.x, yk.x), ay = dy(gk.y, yk.y);
                if (kBeta) {
                    const double2 u = __ldg(reinterpret_cast<const double2 *>(w) + k),
                                  v = __ldg(reinterpret_cast<const double2 *>(w + r) + k),
                                  z = __ldg(reinterpret_cast<const double2 *>(w + 2 * r) + k);
                    __stcs(dm2 + k, make_double2(fma(ds, u.x + z.x, (1.0 - beta) * ax), fma(ds, u.y + z.y, (1.0 - beta) * ay)));
                    __stcs(dr2 + k, make_double2(fma(ds, v.x - z.x, beta * ax), fma(ds, v.y - z.y, beta * ay)));
                } else {
                    __stcs(dm2 + k, make_double2(ax, ay));
                    if (dr2) __stcs(dr2 + k, make_double2(ax, ay));
                }
            }
        } else {
            double *dm = dM + i * r, *dr = dR ? dR + i * r : nullptr;
            for (int64_t k = lane; k < r; k += 32) {
                const double a = dy(__ldcs(g + k), kRelu ? __ldcs(y + k) : 0.0);
                if (kBeta) {
                    const double u = __ldg(w + k), v = __ldg(w + r + k), z = __ldg(w + 2 * r + k);
                    __stcs(dm + k, fma(ds, u + z, (1.0 - beta) * a));
                    __stcs(dr + k, fma(ds, v - z, beta * a));
                } else {
                    __stcs(dm + k, a);
                    if (dr) __stcs(dr + k, a);
                }
            }
        }
    }
}

// partial[c, :] = sum over the rows of chunk c (in row order) of ds_i [M_i, R_i, M_i - R_i]; one thread per column,
// blockIdx.y the chunk
__global__ void __launch_bounds__(kBlock)
gate_dw_partial_kernel(double *__restrict__ partial, const double *__restrict__ ds, const double *__restrict__ M,
                       const double *__restrict__ R, int64_t n, int64_t r, int64_t chunk_rows) {
    const int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= r) return;
    const int64_t c = blockIdx.y, i0 = c * chunk_rows, i1 = n < i0 + chunk_rows ? n : i0 + chunk_rows;
    double a1 = 0.0, a2 = 0.0, a3 = 0.0;
    for (int64_t i = i0; i < i1; i++) {
        const double s = __ldg(ds + i), a = ld_stream_f64(M + i * r + k), b = ld_stream_f64(R + i * r + k);
        a1 = fma(s, a, a1);
        a2 = fma(s, b, a2);
        a3 = fma(s, a - b, a3);
    }
    double *out = partial + c * 3 * r;
    out[k] = a1;
    out[r + k] = a2;
    out[2 * r + k] = a3;
}

// ---- the transformer block (GraphTransformer with ffn_ratio > 0) ----------------------------------------------------
// Z[i, :] = max(A[i, :] + b, 0): the first feed-forward layer's bias and ReLU
template <bool kPairs>
__global__ void __launch_bounds__(kBlock)
row_bias_relu_kernel(double *__restrict__ Z, const double *__restrict__ A, const double *__restrict__ b, int64_t n, int64_t r) {
    const int lane = threadIdx.x & 31;
    const int64_t warps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t i = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; i < n; i += warps) {
        if (kPairs) {
            const double2 *a2 = reinterpret_cast<const double2 *>(A + i * r), *b2 = reinterpret_cast<const double2 *>(b);
            double2 *z2 = reinterpret_cast<double2 *>(Z + i * r);
#pragma unroll 2
            for (int64_t k = lane; k < r / 2; k += 32) {
                const double2 v = __ldcs(a2 + k), c = __ldg(b2 + k);
                z2[k] = make_double2(fmax(v.x + c.x, 0.0), fmax(v.y + c.y, 0.0));
            }
        } else {
            const double *a = A + i * r;
            double *z = Z + i * r;
            for (int64_t k = lane; k < r; k += 32) z[k] = fmax(__ldcs(a + k) + __ldg(b + k), 0.0);
        }
    }
}

// Y = gamma * (x - mean) * rstd + beta with x = X + Res (Res nullable), mean and rstd = 1 / sqrt(var + eps) of each
// row (biased variance, from the centred values), written to stats[2i], stats[2i + 1]
template <bool kPairs, int kN>
__global__ void __launch_bounds__(kBlock, 1)
layer_norm_kernel(double *__restrict__ Y, double *__restrict__ stats, const double *__restrict__ X, const double *__restrict__ Res,
                  const double *__restrict__ gamma, const double *__restrict__ beta, int64_t n, int64_t r, double eps) {
    const int lane = threadIdx.x & 31;
    const int64_t warps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    const double inv_r = 1.0 / (double)r;
    for (int64_t i = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; i < n; i += warps) {
        const double *x = X + i * r, *res = Res ? Res + i * r : nullptr;
        double *y = Y + i * r;
        double mean, rstd;
        if constexpr (kN > 0) {
            double v[2 * kN];
            ln_load<kPairs, kN>(v, x, res, r, lane);
            double s = 0.0;
#pragma unroll
            for (int j = 0; j < 2 * kN; j++) s += v[j];
            mean = group_allreduce<32>(s, 0xffffffffu) * inv_r;
            double q = 0.0;
#pragma unroll
            for (int j = 0; j < 2 * kN; j++) {
                const double c = v[j] - mean;
                if (ln_col<kPairs>(j, lane) < r) q = fma(c, c, q);
            }
            rstd = 1.0 / sqrt(group_allreduce<32>(q, 0xffffffffu) * inv_r + eps);
            if (kPairs) {
                const double2 *g2 = reinterpret_cast<const double2 *>(gamma), *b2 = reinterpret_cast<const double2 *>(beta);
                double2 *y2 = reinterpret_cast<double2 *>(y);
#pragma unroll
                for (int j = 0; j < kN; j++) {
                    const int64_t k = lane + 32 * j;
                    if (k < r / 2) {
                        const double2 g = __ldg(g2 + k), b = __ldg(b2 + k);
                        y2[k] = make_double2(fma((v[2 * j] - mean) * rstd, g.x, b.x), fma((v[2 * j + 1] - mean) * rstd, g.y, b.y));
                    }
                }
            } else {
#pragma unroll
                for (int j = 0; j < 2 * kN; j++) {
                    const int64_t k = lane + 32 * j;
                    if (k < r) y[k] = fma((v[j] - mean) * rstd, __ldg(gamma + k), __ldg(beta + k));
                }
            }
        } else {
            auto at = [&](int64_t k) { return res ? x[k] + res[k] : x[k]; };
            double s = 0.0;
            for (int64_t k = lane; k < r; k += 32) s += at(k);
            mean = group_allreduce<32>(s, 0xffffffffu) * inv_r;
            double q = 0.0;
            for (int64_t k = lane; k < r; k += 32) {
                const double c = at(k) - mean;
                q = fma(c, c, q);
            }
            rstd = 1.0 / sqrt(group_allreduce<32>(q, 0xffffffffu) * inv_r + eps);
            for (int64_t k = lane; k < r; k += 32) y[k] = fma((at(k) - mean) * rstd, __ldg(gamma + k), __ldg(beta + k));
        }
        if (lane == 0) {
            stats[2 * i] = mean;
            stats[2 * i + 1] = rstd;
        }
    }
}

// dX = rstd (g - mean(g) - xh mean(g xh)) with g = G gamma and xh = (X + Res - mean) rstd from stats; added to dX
// when accumulate.  kN as in layer_norm_kernel, for G and xh both.
template <bool kPairs, int kN>
__global__ void __launch_bounds__(kBlock, 1)
layer_norm_backward_kernel(double *__restrict__ dX, const double *__restrict__ G, const double *__restrict__ X,
                           const double *__restrict__ Res, const double *__restrict__ stats, const double *__restrict__ gamma,
                           int64_t n, int64_t r, int accumulate) {
    const int lane = threadIdx.x & 31;
    const int64_t warps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    const double inv_r = 1.0 / (double)r;
    for (int64_t i = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; i < n; i += warps) {
        const double *x = X + i * r, *res = Res ? Res + i * r : nullptr, *gr = G + i * r;
        double *dx = dX + i * r;
        const double mean = __ldg(stats + 2 * i), rstd = __ldg(stats + 2 * i + 1);
        auto out = [&](int64_t k, double v) { return accumulate ? dx[k] + v : v; };
        if constexpr (kN > 0) {
            constexpr int N = kN;
            double g[2 * N], xh[2 * N];
            ln_load<kPairs, N>(g, gr, nullptr, r, lane);
            ln_load<kPairs, N>(xh, x, res, r, lane);
            double s1 = 0.0, s2 = 0.0;
            if (kPairs) {
                const double2 *g2 = reinterpret_cast<const double2 *>(gamma);
#pragma unroll
                for (int j = 0; j < N; j++) {
                    const int64_t k = lane + 32 * j;
                    const double2 w = k < r / 2 ? __ldg(g2 + k) : make_double2(0.0, 0.0);
                    g[2 * j] *= w.x;
                    g[2 * j + 1] *= w.y;
                }
            } else {
#pragma unroll
                for (int j = 0; j < 2 * N; j++) {
                    const int64_t k = lane + 32 * j;
                    g[j] *= k < r ? __ldg(gamma + k) : 0.0;
                }
            }
#pragma unroll
            for (int j = 0; j < 2 * N; j++) {
                xh[j] = (xh[j] - mean) * rstd;
                s1 += g[j];
                s2 = fma(g[j], xh[j], s2);
            }
            const double m1 = group_allreduce<32>(s1, 0xffffffffu) * inv_r, m2 = group_allreduce<32>(s2, 0xffffffffu) * inv_r;
            if (kPairs) {
                double2 *d2 = reinterpret_cast<double2 *>(dx);
#pragma unroll
                for (int j = 0; j < N; j++) {
                    const int64_t k = lane + 32 * j;
                    if (k < r / 2) {
                        double2 v = make_double2(rstd * (g[2 * j] - m1 - xh[2 * j] * m2), rstd * (g[2 * j + 1] - m1 - xh[2 * j + 1] * m2));
                        if (accumulate) {
                            const double2 o = d2[k];
                            v = make_double2(o.x + v.x, o.y + v.y);
                        }
                        d2[k] = v;
                    }
                }
            } else {
#pragma unroll
                for (int j = 0; j < 2 * N; j++) {
                    const int64_t k = lane + 32 * j;
                    if (k < r) dx[k] = out(k, rstd * (g[j] - m1 - xh[j] * m2));
                }
            }
        } else {
            auto xhat = [&](int64_t k) { return ((res ? x[k] + res[k] : x[k]) - mean) * rstd; };
            double s1 = 0.0, s2 = 0.0;
            for (int64_t k = lane; k < r; k += 32) {
                const double gk = gr[k] * __ldg(gamma + k);
                s1 += gk;
                s2 = fma(gk, xhat(k), s2);
            }
            const double m1 = group_allreduce<32>(s1, 0xffffffffu) * inv_r, m2 = group_allreduce<32>(s2, 0xffffffffu) * inv_r;
            for (int64_t k = lane; k < r; k += 32) dx[k] = out(k, rstd * (gr[k] * __ldg(gamma + k) - m1 - xhat(k) * m2));
        }
    }
}

// partial[c, k] = sum over the rows of chunk c (in row order) of G_ik xh_ik, partial[chunks + c, k] = of G_ik; one
// thread per column, blockIdx.y the chunk.  The chunks are then summed in order by gate_dw_final_kernel.
__global__ void __launch_bounds__(kBlock)
layer_norm_dw_partial_kernel(double *__restrict__ partial, const double *__restrict__ G, const double *__restrict__ X,
                             const double *__restrict__ Res, const double *__restrict__ stats, int64_t n, int64_t r,
                             int64_t chunk_rows) {
    const int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= r) return;
    const int64_t c = blockIdx.y, i0 = c * chunk_rows, i1 = n < i0 + chunk_rows ? n : i0 + chunk_rows;
    double a1 = 0.0, a2 = 0.0;
    for (int64_t i = i0; i < i1; i++) {
        const double x = Res ? ld_stream_f64(X + i * r + k) + ld_stream_f64(Res + i * r + k) : ld_stream_f64(X + i * r + k);
        const double g = ld_stream_f64(G + i * r + k);
        a1 = fma(g, (x - __ldg(stats + 2 * i)) * __ldg(stats + 2 * i + 1), a1);
        a2 += g;
    }
    partial[c * r + k] = a1;
    partial[((int64_t)gridDim.y + c) * r + k] = a2;
}

template <bool kPairs>
auto layer_norm_for(int64_t r) {
    return pick_ln<kLnWidest>(r, layer_norm_kernel<kPairs, 1>, layer_norm_kernel<kPairs, 2>, layer_norm_kernel<kPairs, 4>,
                               layer_norm_kernel<kPairs, 8>, layer_norm_kernel<kPairs, 12>, layer_norm_kernel<kPairs, 16>,
                               layer_norm_kernel<kPairs, 24>, layer_norm_kernel<kPairs, 0>);
}
template <bool kPairs>
auto layer_norm_backward_for(int64_t r) {
    return pick_ln<kLnBackwardWidest>(
        r, layer_norm_backward_kernel<kPairs, 1>, layer_norm_backward_kernel<kPairs, 2>, layer_norm_backward_kernel<kPairs, 4>,
        layer_norm_backward_kernel<kPairs, 8>, layer_norm_backward_kernel<kPairs, 12>, layer_norm_backward_kernel<kPairs, 16>,
        layer_norm_backward_kernel<kPairs, 0>, layer_norm_backward_kernel<kPairs, 0>);  // past kLnBackwardWidest: kN = 0
}

template <bool kPairs, bool kBeta>
auto pick_gate(bool relu) {
    return relu ? gate_kernel<kPairs, kBeta, true> : gate_kernel<kPairs, kBeta, false>;
}
template <bool kPairs, bool kBeta>
auto pick_gate_backward(bool relu) {
    return relu ? gate_backward_kernel<kPairs, kBeta, true> : gate_backward_kernel<kPairs, kBeta, false>;
}

}  // namespace

extern "C" {

int hnh_row_bias_add_f64(double *X, const double *b, int64_t n, int64_t r, void *stream) {
    if (n < 0 || r < 0) return set_error(HNH_E_INVALID, "hnh_row_bias_add_f64: negative size");
    if (n == 0 || r == 0) return HNH_OK;
    if (!X || !b) return set_error(HNH_E_INVALID, "hnh_row_bias_add_f64: null pointer");
    auto k = r % 2 == 0 && aligned16(X) && aligned16(b) ? row_bias_kernel<true> : row_bias_kernel<false>;
    int grid;
    int rc = grid_for(k, n, kBlock / 32, &grid, kCtasPerSm);
    return rc ? rc : launch(k, grid, kBlock, (cudaStream_t)stream, "row_bias_kernel", X, b, n, r);
}

int hnh_gt_gate_f64(double *Y, const double *M, const double *R, const double *w_beta, int64_t n, int64_t r, int relu,
                    void *stream) {
    if (n < 0 || r < 0) return set_error(HNH_E_INVALID, "hnh_gt_gate_f64: negative size");
    if (n == 0 || r == 0) return HNH_OK;
    if (!Y || !M || !R) return set_error(HNH_E_INVALID, "hnh_gt_gate_f64: null pointer");
    if (Y == M || Y == R) return set_error(HNH_E_INVALID, "hnh_gt_gate_f64: Y may not be M or R");
    const bool pairs = r % 2 == 0 && aligned16(Y) && aligned16(M) && aligned16(R) && (!w_beta || aligned16(w_beta));
    auto k = w_beta ? (pairs ? pick_gate<true, true>(relu) : pick_gate<false, true>(relu))
                    : (pairs ? pick_gate<true, false>(relu) : pick_gate<false, false>(relu));
    int grid;
    int rc = grid_for(k, n, kBlock / 32, &grid, kCtasPerSm);
    return rc ? rc : launch(k, grid, kBlock, (cudaStream_t)stream, "gate_kernel", Y, M, R, w_beta, n, r);
}

int64_t hnh_gt_gate_backward_workspace_bytes(int64_t n, int64_t r) {
    if (n < 0 || r < 0) return set_error(HNH_E_INVALID, "hnh_gt_gate_backward_workspace_bytes: negative size");
    return (int64_t)sizeof(double) * (n + dw_chunks(n) * 3 * r);
}

int hnh_gt_gate_backward_f64(double *dM, double *dR, double *dw_beta, const double *G, const double *Y, const double *M,
                             const double *R, const double *w_beta, int64_t n, int64_t r, int relu, void *workspace,
                             size_t workspace_bytes, void *stream) {
    if (n < 0 || r < 0) return set_error(HNH_E_INVALID, "hnh_gt_gate_backward_f64: negative size");
    const bool beta = w_beta != nullptr;
    if (beta && !dw_beta) return set_error(HNH_E_INVALID, "hnh_gt_gate_backward_f64: the gate needs dw_beta");
    if (!beta && dw_beta) return set_error(HNH_E_INVALID, "hnh_gt_gate_backward_f64: dw_beta without the gate");
    if (r == 0) return HNH_OK;
    if (n == 0) {  // no rows: dw_beta = 0
        if (!beta) return HNH_OK;
        return hnh::check_cuda(cudaMemsetAsync(dw_beta, 0, sizeof(double) * 3 * (size_t)r, (cudaStream_t)stream), "dw_beta");
    }
    if (!dM || !G || !M || !R || (relu && !Y) || (beta && !dR))
        return set_error(HNH_E_INVALID, "hnh_gt_gate_backward_f64: null pointer");
    const double *ins[] = {G, relu ? Y : nullptr, M, R, w_beta};
    for (const double *o : {(const double *)dM, (const double *)dR, (const double *)dw_beta})
        for (const double *in : ins)
            if (o && o == in) return set_error(HNH_E_INVALID, "hnh_gt_gate_backward_f64: an output may not be an input");
    if (dR && dR == dM) return set_error(HNH_E_INVALID, "hnh_gt_gate_backward_f64: dM and dR are one matrix");
    const int64_t need = beta ? hnh_gt_gate_backward_workspace_bytes(n, r) : 0;
    if (beta && (!workspace || (int64_t)workspace_bytes < need))
        return set_error(HNH_E_INVALID, "hnh_gt_gate_backward_f64: the workspace needs %lld bytes", (long long)need);
    cudaStream_t st = (cudaStream_t)stream;
    const bool pairs = r % 2 == 0 && aligned16(dM) && (!dR || aligned16(dR)) && aligned16(G) && (!relu || aligned16(Y)) &&
                       aligned16(M) && aligned16(R) && (!beta || aligned16(w_beta));
    auto k = beta ? (pairs ? pick_gate_backward<true, true>(relu) : pick_gate_backward<false, true>(relu))
                  : (pairs ? pick_gate_backward<true, false>(relu) : pick_gate_backward<false, false>(relu));
    double *ds = beta ? (double *)workspace : nullptr;
    int grid;
    int rc = grid_for(k, n, kBlock / 32, &grid, kCtasPerSm);
    if (!rc) rc = launch(k, grid, kBlock, st, "gate_backward_kernel", dM, dR, ds, G, relu ? Y : nullptr, M, R, w_beta, n, r);
    if (rc || !beta) return rc;
    const int64_t chunks = dw_chunks(n), chunk_rows = (n + chunks - 1) / chunks;
    double *partial = ds + n;
    rc = launch(gate_dw_partial_kernel, dim3((unsigned)((r + kBlock - 1) / kBlock), (unsigned)chunks), kBlock, st,
                "gate_dw_partial_kernel", partial, (const double *)ds, M, R, n, r, chunk_rows);
    if (rc) return rc;
    rc = grid_for(gate_dw_final_kernel, 3 * r, kBlock, &grid, kCtasPerSm);
    return rc ? rc : launch(gate_dw_final_kernel, grid, kBlock, st, "gate_dw_final_kernel", dw_beta, (const double *)partial, chunks, 3 * r);
}

int hnh_row_bias_relu_f64(double *Z, const double *A, const double *b, int64_t n, int64_t r, void *stream) {
    if (n < 0 || r < 0) return set_error(HNH_E_INVALID, "hnh_row_bias_relu_f64: negative size");
    if (n == 0 || r == 0) return HNH_OK;
    if (!Z || !A || !b) return set_error(HNH_E_INVALID, "hnh_row_bias_relu_f64: null pointer");
    if (Z == A || Z == b) return set_error(HNH_E_INVALID, "hnh_row_bias_relu_f64: Z may not be A or b");
    auto k = r % 2 == 0 && aligned16(Z) && aligned16(A) && aligned16(b) ? row_bias_relu_kernel<true> : row_bias_relu_kernel<false>;
    int grid;
    int rc = grid_for(k, n, kBlock / 32, &grid, kCtasPerSm);
    return rc ? rc : launch(k, grid, kBlock, (cudaStream_t)stream, "row_bias_relu_kernel", Z, A, b, n, r);
}

int hnh_layer_norm_f64(double *Y, double *stats, const double *X, const double *Res, const double *gamma, const double *beta,
                       int64_t n, int64_t r, double eps, void *stream) {
    if (n < 0 || r < 0) return set_error(HNH_E_INVALID, "hnh_layer_norm_f64: negative size");
    if (!(eps > 0.0) || !std::isfinite(eps)) return set_error(HNH_E_INVALID, "hnh_layer_norm_f64: eps must be finite and > 0");
    if (n == 0 || r == 0) return HNH_OK;
    if (!Y || !stats || !X || !gamma || !beta) return set_error(HNH_E_INVALID, "hnh_layer_norm_f64: null pointer");
    for (const double *o : {(const double *)Y, (const double *)stats})
        for (const double *in : {X, Res, gamma, beta})
            if (o == in) return set_error(HNH_E_INVALID, "hnh_layer_norm_f64: an output may not be an input");
    if (Y == stats) return set_error(HNH_E_INVALID, "hnh_layer_norm_f64: Y and stats are one buffer");
    const bool pairs = r % 2 == 0 && aligned16(Y) && aligned16(X) && (!Res || aligned16(Res)) && aligned16(gamma) && aligned16(beta);
    auto k = pairs ? layer_norm_for<true>(r) : layer_norm_for<false>(r);
    int grid;
    int rc = grid_for(k, n, kBlock / 32, &grid);
    return rc ? rc : launch(k, grid, kBlock, (cudaStream_t)stream, "layer_norm_kernel", Y, stats, X, Res, gamma, beta, n, r, eps);
}

int64_t hnh_layer_norm_backward_workspace_bytes(int64_t n, int64_t r) {
    if (n < 0 || r < 0) return set_error(HNH_E_INVALID, "hnh_layer_norm_backward_workspace_bytes: negative size");
    return (int64_t)sizeof(double) * dw_chunks(n) * 2 * r;
}

int hnh_layer_norm_backward_f64(double *dX, double *dgamma, double *dbeta, const double *G, const double *X, const double *Res,
                                const double *stats, const double *gamma, int64_t n, int64_t r, int accumulate,
                                void *workspace, size_t workspace_bytes, void *stream) {
    if (n < 0 || r < 0) return set_error(HNH_E_INVALID, "hnh_layer_norm_backward_f64: negative size");
    if (r == 0) return HNH_OK;
    if (!dgamma || !dbeta) return set_error(HNH_E_INVALID, "hnh_layer_norm_backward_f64: null pointer");
    if (dgamma == dbeta) return set_error(HNH_E_INVALID, "hnh_layer_norm_backward_f64: dgamma and dbeta are one vector");
    cudaStream_t st = (cudaStream_t)stream;
    if (n == 0) {  // no rows: dgamma = dbeta = 0
        int rc = hnh::check_cuda(cudaMemsetAsync(dgamma, 0, sizeof(double) * (size_t)r, st), "dgamma");
        return rc ? rc : hnh::check_cuda(cudaMemsetAsync(dbeta, 0, sizeof(double) * (size_t)r, st), "dbeta");
    }
    if (!dX || !G || !X || !stats || !gamma) return set_error(HNH_E_INVALID, "hnh_layer_norm_backward_f64: null pointer");
    const double *ins[] = {G, X, Res, stats, gamma};
    for (const double *o : {(const double *)dX, (const double *)dgamma, (const double *)dbeta})
        for (const double *in : ins)
            if (o == in) return set_error(HNH_E_INVALID, "hnh_layer_norm_backward_f64: an output may not be an input");
    if (dX == dgamma || dX == dbeta) return set_error(HNH_E_INVALID, "hnh_layer_norm_backward_f64: dX and dgamma / dbeta are one buffer");
    const int64_t need = hnh_layer_norm_backward_workspace_bytes(n, r);
    if (!workspace || (int64_t)workspace_bytes < need)
        return set_error(HNH_E_INVALID, "hnh_layer_norm_backward_f64: the workspace needs %lld bytes", (long long)need);
    const bool pairs = r % 2 == 0 && aligned16(dX) && aligned16(G) && aligned16(X) && (!Res || aligned16(Res)) && aligned16(gamma);
    auto k = pairs ? layer_norm_backward_for<true>(r) : layer_norm_backward_for<false>(r);
    int grid;
    int rc = grid_for(k, n, kBlock / 32, &grid);
    if (!rc) rc = launch(k, grid, kBlock, st, "layer_norm_backward_kernel", dX, G, X, Res, stats, gamma, n, r, accumulate ? 1 : 0);
    if (rc) return rc;
    const int64_t chunks = dw_chunks(n), chunk_rows = (n + chunks - 1) / chunks;
    double *partial = (double *)workspace;
    rc = launch(layer_norm_dw_partial_kernel, dim3((unsigned)((r + kBlock - 1) / kBlock), (unsigned)chunks), kBlock, st,
                "layer_norm_dw_partial_kernel", partial, G, X, Res, stats, n, r, chunk_rows);
    if (!rc) rc = grid_for(gate_dw_final_kernel, r, kBlock, &grid, kCtasPerSm);
    if (!rc) rc = launch(gate_dw_final_kernel, grid, kBlock, st, "gate_dw_final_kernel", dgamma, (const double *)partial, chunks, r);
    return rc ? rc : launch(gate_dw_final_kernel, grid, kBlock, st, "gate_dw_final_kernel", dbeta,
                            (const double *)(partial + chunks * r), chunks, r);
}

}  // extern "C"
