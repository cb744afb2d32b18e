// training.cu -- the device side of training (include/hnh/training.hpp): the node-classification loss and the optimizer.
//     loss_i = lse_i - x_i,label  with lse_i = max_i + log sum_k exp(x_ik - max_i)       labelled rows (0 <= label < C)
//     dlogits_ik = (exp(x_ik - lse_i) - [k == label_i]) inv_count,  0 on ignored rows
//     correct_i = [argmax_k x_ik == label_i]   (ties to the lowest k, as torch.argmax)       (cross_entropy_kernel)
//     sums = (sum_i loss_i, sum_i correct_i)   per-row values, then the two-stage fixed-order reduction of row_regs.cuh
//                                              (cross_entropy_partial_kernel, gate_dw_final_kernel)
//     AdamW as torch.optim.AdamW(foreach=False), one tensor, in place                      (adamw_kernel)
//     (total, coef) = (sqrt(sum of the spans' squared norms, in order), min(1, max_norm / (total + 1e-6)))
//                                              torch.nn.utils.clip_grad_norm_'s coefficient (clip_coef_kernel)
// The cross-entropy kernel runs one warp per row.  Up to C = 1536 a lane keeps its share of the row in registers, so
// the row is read once; wider rows are reread in every pass.  Row max (with its index), sum and the label's logit end
// in fixed xor butterflies, so every lane holds the same bits.  The label only ever meets a column index in a
// comparison: no load depends on it.  No floating-point atomics anywhere: repeated calls are bit-identical.
#include <cmath>

#include "row_regs.cuh"

namespace {

using hnh::grid_for;
using hnh::launch;
using hnh::set_error;

constexpr int kCtasPerSm = 16;  // grid cap of the elementwise kernel
constexpr int kCeWidest = 24;   // register rows up to C = 64 * this

// (v, k) becomes the maximum over the warp of the lanes' (v, k), ties to the lowest k: the same on every lane
__device__ __forceinline__ void argmax_allreduce(double &v, int64_t &k) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const double ov = __shfl_xor_sync(0xffffffffu, v, o);
        const int64_t ok = __shfl_xor_sync(0xffffffffu, k, o);
        if (ov > v || (ov == v && ok < k)) {
            v = ov;
            k = ok;
        }
    }
}

__device__ __forceinline__ void argmax_step(double x, int64_t col, double &v, int64_t &k) {
    if (x > v || (x == v && col < k)) {
        v = x;
        k = col;
    }
}

// Row i of logits (leading dimension ld) -> dlogits (same ld) and (loss_i, correct_i) at row_out[2i].  kN as in
// ln_load; kN = 0 rereads the row in scalars.
template <bool kPairs, int kN>
__global__ void __launch_bounds__(kBlock, 1)
cross_entropy_kernel(double *__restrict__ dlogits, double *__restrict__ row_out, const double *__restrict__ logits,
                     const int32_t *__restrict__ labels, int64_t n, int64_t C, int64_t ld, double inv_count) {
    const int lane = threadIdx.x & 31;
    const int64_t warps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t i = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; i < n; i += warps) {
        const double *x = logits + i * ld;
        double *d = dlogits + i * ld;
        const int64_t label = __ldg(labels + i);
        const bool labelled = label >= 0 && label < C;
        double mx = -INFINITY, xl = 0.0, s = 0.0;
        int64_t am = INT64_MAX;
        if constexpr (kN > 0) {
            double v[2 * kN];
            ln_load<kPairs, kN>(v, x, nullptr, C, lane);
#pragma unroll
            for (int j = 0; j < 2 * kN; j++) {
                const int64_t col = ln_col<kPairs>(j, lane);
                if (col < C) argmax_step(v[j], col, mx, am);
                if (col == label) xl = v[j];
            }
            argmax_allreduce(mx, am);
#pragma unroll
            for (int j = 0; j < 2 * kN; j++)
                if (ln_col<kPairs>(j, lane) < C) s += exp(v[j] - mx);
            s = group_allreduce<32>(s, 0xffffffffu);
            const double ls = log(s);
            // d_k = exp(x_k - max - log s) inv - [k == label] inv; 0 on an ignored row
            auto grad = [&](int j) {
                return labelled ? fma(exp(v[j] - mx - ls), inv_count, ln_col<kPairs>(j, lane) == label ? -inv_count : 0.0) : 0.0;
            };
            if (kPairs) {
                double2 *d2 = reinterpret_cast<double2 *>(d);
#pragma unroll
                for (int j = 0; j < kN; j++) {
                    const int64_t k = lane + 32 * j;
                    if (k < C / 2) __stcs(d2 + k, make_double2(grad(2 * j), grad(2 * j + 1)));
                }
            } else {
#pragma unroll
                for (int j = 0; j < 2 * kN; j++) {
                    const int64_t k = lane + 32 * j;
                    if (k < C) __stcs(d + k, grad(j));
                }
            }
        } else {
            for (int64_t k = lane; k < C; k += 32) {
                const double v = x[k];
                argmax_step(v, k, mx, am);
                if (k == label) xl = v;
            }
            argmax_allreduce(mx, am);
            for (int64_t k = lane; k < C; k += 32) s += exp(x[k] - mx);
            s = group_allreduce<32>(s, 0xffffffffu);
            const double ls = log(s);
            for (int64_t k = lane; k < C; k += 32)
                d[k] = labelled ? fma(exp(x[k] - mx - ls), inv_count, k == label ? -inv_count : 0.0) : 0.0;
        }
        xl = group_allreduce<32>(xl, 0xffffffffu);  // one lane holds the label's logit, the others 0
        if (lane == 0) {
            row_out[2 * i] = labelled ? -((xl - mx) - log(s)) : 0.0;
            row_out[2 * i + 1] = labelled && am == label ? 1.0 : 0.0;
        }
    }
}

// partial[2c + j] = sum over the rows of chunk c of row_out[2i + j], j = 0 (loss) and 1 (correct): one warp per chunk,
// lane l takes rows i0 + l + 32 t in order, then the xor butterfly.  The order depends on n only.
__global__ void __launch_bounds__(kBlock)
cross_entropy_partial_kernel(double *__restrict__ partial, const double *__restrict__ row_out, int64_t n, int64_t chunks,
                             int64_t chunk_rows) {
    const int lane = threadIdx.x & 31;
    const int64_t c = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (c >= chunks) return;
    const int64_t i0 = c * chunk_rows, i1 = n < i0 + chunk_rows ? n : i0 + chunk_rows;
    double a = 0.0, b = 0.0;
    for (int64_t i = i0 + lane; i < i1; i += 32) {
        a += row_out[2 * i];
        b += row_out[2 * i + 1];
    }
    a = group_allreduce<32>(a, 0xffffffffu);
    b = group_allreduce<32>(b, 0xffffffffu);
    if (lane == 0) {
        partial[2 * c] = a;
        partial[2 * c + 1] = b;
    }
}

template <bool kPairs>
auto cross_entropy_for(int64_t C) {
    return pick_ln<kCeWidest>(C, cross_entropy_kernel<kPairs, 1>, cross_entropy_kernel<kPairs, 2>, cross_entropy_kernel<kPairs, 4>,
                              cross_entropy_kernel<kPairs, 8>, cross_entropy_kernel<kPairs, 12>, cross_entropy_kernel<kPairs, 16>,
                              cross_entropy_kernel<kPairs, 24>, cross_entropy_kernel<kPairs, 0>);
}

// torch's single-tensor AdamW on one element, with g already multiplied by the clip coefficient:
//     p *= 1 - lr wd;  m = lerp(m, g, 1 - beta1);  v = v beta2 + (1 - beta2) g g;
//     p += -step_size m / (sqrt(v) / sqrt(bc2) + eps),  step_size = lr / bc1
struct AdamWArgs {
    double decay, w1, beta2, w2, neg_step, bc2_sqrt, eps;
};
__device__ __forceinline__ void adamw_one(double &p, double &m, double &v, double g, const AdamWArgs &a) {
    p *= a.decay;
    m = a.w1 < 0.5 ? m + a.w1 * (g - m) : g - (g - m) * (1.0 - a.w1);  // torch's lerp
    v = v * a.beta2 + a.w2 * g * g;
    p = p + a.neg_step * m / (sqrt(v) / a.bc2_sqrt + a.eps);
}

template <bool kPairs>
__global__ void __launch_bounds__(kBlock)
adamw_kernel(double *__restrict__ P, double *__restrict__ M, double *__restrict__ V, const double *__restrict__ G, int64_t n,
             AdamWArgs a, const double *__restrict__ clip) {
    const double coef = clip ? __ldg(clip) : 1.0;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x, t0 = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (kPairs) {
        double2 *p2 = reinterpret_cast<double2 *>(P), *m2 = reinterpret_cast<double2 *>(M), *v2 = reinterpret_cast<double2 *>(V);
        const double2 *g2 = reinterpret_cast<const double2 *>(G);
        for (int64_t i = t0; i < n / 2; i += stride) {
            double2 p = p2[i], m = m2[i], v = v2[i];
            const double2 g = __ldcs(g2 + i);
            adamw_one(p.x, m.x, v.x, clip ? g.x * coef : g.x, a);
            adamw_one(p.y, m.y, v.y, clip ? g.y * coef : g.y, a);
            p2[i] = p;
            m2[i] = m;
            v2[i] = v;
        }
        if (n % 2 && t0 == 0) adamw_one(P[n - 1], M[n - 1], V[n - 1], clip ? G[n - 1] * coef : G[n - 1], a);
    } else {
        for (int64_t i = t0; i < n; i += stride) adamw_one(P[i], M[i], V[i], clip ? G[i] * coef : G[i], a);
    }
}

// out[0] = sqrt(sum of sq in order), out[1] = min(1, max_norm / (out[0] + 1e-6)); one thread
__global__ void clip_coef_kernel(double *__restrict__ out, const double *__restrict__ sq, int64_t count, double max_norm) {
    double t = 0.0;
    for (int64_t i = 0; i < count; i++) t += sq[i];
    const double total = sqrt(t);
    out[0] = total;
    out[1] = fmin(1.0, max_norm / (total + 1e-6));
}

}  // namespace

extern "C" {

int64_t hnh_cross_entropy_workspace_bytes(int64_t n) {
    if (n < 0) return set_error(HNH_E_INVALID, "hnh_cross_entropy_workspace_bytes: negative size");
    return (int64_t)sizeof(double) * 2 * (n + dw_chunks(n));
}

int hnh_cross_entropy_f64(double *dlogits, double *sums, const double *logits, const int32_t *labels, int64_t n, int64_t C,
                          int64_t ld, double inv_count, void *workspace, size_t workspace_bytes, void *stream) {
    if (n < 0) return set_error(HNH_E_INVALID, "hnh_cross_entropy_f64: negative size");
    if (C <= 0) return set_error(HNH_E_INVALID, "hnh_cross_entropy_f64: the class count must be positive");
    if (ld < C) return set_error(HNH_E_INVALID, "hnh_cross_entropy_f64: ld = %lld is below C = %lld", (long long)ld, (long long)C);
    if (!(inv_count >= 0.0) || !std::isfinite(inv_count))
        return set_error(HNH_E_INVALID, "hnh_cross_entropy_f64: inv_count must be finite and >= 0");
    if (!sums) return set_error(HNH_E_INVALID, "hnh_cross_entropy_f64: null pointer");
    cudaStream_t st = (cudaStream_t)stream;
    if (n == 0) return hnh::check_cuda(cudaMemsetAsync(sums, 0, 2 * sizeof(double), st), "sums");
    if (!dlogits || !logits || !labels) return set_error(HNH_E_INVALID, "hnh_cross_entropy_f64: null pointer");
    if ((const void *)dlogits == (const void *)logits || (const void *)sums == (const void *)logits ||
        (const void *)sums == (const void *)labels || (const void *)dlogits == (const void *)labels || sums == dlogits)
        return set_error(HNH_E_INVALID, "hnh_cross_entropy_f64: an output may not be an input or the other output");
    const int64_t need = hnh_cross_entropy_workspace_bytes(n);
    if (!workspace || (int64_t)workspace_bytes < need)
        return set_error(HNH_E_INVALID, "hnh_cross_entropy_f64: the workspace needs %lld bytes", (long long)need);
    const bool pairs = C % 2 == 0 && ld % 2 == 0 && aligned16(dlogits) && aligned16(logits);
    auto k = pairs ? cross_entropy_for<true>(C) : cross_entropy_for<false>(C);
    double *row_out = (double *)workspace, *partial = row_out + 2 * n;
    int grid = 0;
    int rc = grid_for(k, n, kBlock / 32, &grid);
    if (!rc) rc = launch(k, grid, kBlock, st, "cross_entropy_kernel", dlogits, row_out, logits, labels, n, C, ld, inv_count);
    if (rc) return rc;
    const int64_t chunks = dw_chunks(n), chunk_rows = (n + chunks - 1) / chunks;
    rc = launch(cross_entropy_partial_kernel, (unsigned)((chunks * 32 + kBlock - 1) / kBlock), kBlock, st,
                "cross_entropy_partial_kernel", partial, (const double *)row_out, n, chunks, chunk_rows);
    return rc ? rc : launch(gate_dw_final_kernel, 1, kBlock, st, "gate_dw_final_kernel", sums, (const double *)partial, chunks, (int64_t)2);
}

int64_t hnh_pair_sums_workspace_bytes(int64_t n) {
    if (n < 0) return set_error(HNH_E_INVALID, "hnh_pair_sums_workspace_bytes: negative size");
    return (int64_t)sizeof(double) * 2 * dw_chunks(n);
}

int hnh_pair_sums_f64(double *sums, const double *pairs, int64_t n, void *workspace, size_t workspace_bytes, void *stream) {
    if (n < 0) return set_error(HNH_E_INVALID, "hnh_pair_sums_f64: negative size");
    if (!sums) return set_error(HNH_E_INVALID, "hnh_pair_sums_f64: null pointer");
    cudaStream_t st = (cudaStream_t)stream;
    if (n == 0) return hnh::check_cuda(cudaMemsetAsync(sums, 0, 2 * sizeof(double), st), "sums");
    if (!pairs) return set_error(HNH_E_INVALID, "hnh_pair_sums_f64: null pointer");
    const int64_t need = hnh_pair_sums_workspace_bytes(n);
    if (!workspace || (int64_t)workspace_bytes < need)
        return set_error(HNH_E_INVALID, "hnh_pair_sums_f64: the workspace needs %lld bytes", (long long)need);
    double *partial = (double *)workspace;
    const int64_t chunks = dw_chunks(n), chunk_rows = (n + chunks - 1) / chunks;
    int rc = launch(cross_entropy_partial_kernel, (unsigned)((chunks * 32 + kBlock - 1) / kBlock), kBlock, st,
                    "cross_entropy_partial_kernel", partial, pairs, n, chunks, chunk_rows);
    return rc ? rc : launch(gate_dw_final_kernel, 1, kBlock, st, "gate_dw_final_kernel", sums, (const double *)partial, chunks, (int64_t)2);
}

int hnh_adamw_f64(double *param, double *m, double *v, const double *grad, int64_t n, double lr, double beta1, double beta2,
                  double eps, double weight_decay, double bias_correction1, double bias_correction2, const double *clip_coef,
                  void *stream) {
    if (n < 0) return set_error(HNH_E_INVALID, "hnh_adamw_f64: negative size");
    if (!(lr >= 0.0) || !std::isfinite(lr)) return set_error(HNH_E_INVALID, "hnh_adamw_f64: lr must be finite and >= 0");
    if (!(beta1 >= 0.0 && beta1 < 1.0) || !(beta2 >= 0.0 && beta2 < 1.0))
        return set_error(HNH_E_INVALID, "hnh_adamw_f64: the betas must lie in [0, 1)");
    if (!(eps > 0.0) || !std::isfinite(eps)) return set_error(HNH_E_INVALID, "hnh_adamw_f64: eps must be finite and > 0");
    if (!(weight_decay >= 0.0) || !std::isfinite(weight_decay))
        return set_error(HNH_E_INVALID, "hnh_adamw_f64: weight_decay must be finite and >= 0");
    if (!(bias_correction1 > 0.0 && bias_correction1 <= 1.0) || !(bias_correction2 > 0.0 && bias_correction2 <= 1.0))
        return set_error(HNH_E_INVALID, "hnh_adamw_f64: the bias corrections must lie in (0, 1]");
    if (n == 0) return HNH_OK;
    if (!param || !m || !v || !grad) return set_error(HNH_E_INVALID, "hnh_adamw_f64: null pointer");
    const void *ptrs[] = {param, m, v, grad, clip_coef};
    for (int a = 0; a < 5; a++)
        for (int b = a + 1; b < 5; b++)
            if (ptrs[a] && ptrs[a] == ptrs[b]) return set_error(HNH_E_INVALID, "hnh_adamw_f64: param, m, v, grad and clip_coef must be distinct");
    const AdamWArgs a{1.0 - lr * weight_decay, 1.0 - beta1, beta2, 1.0 - beta2, -(lr / bias_correction1), std::sqrt(bias_correction2), eps};
    const bool pairs = aligned16(param) && aligned16(m) && aligned16(v) && aligned16(grad);
    auto k = pairs ? adamw_kernel<true> : adamw_kernel<false>;
    int grid = 0;
    int rc = grid_for(k, pairs ? n / 2 + 1 : n, kBlock, &grid, kCtasPerSm);
    return rc ? rc : launch(k, grid, kBlock, (cudaStream_t)stream, "adamw_kernel", param, m, v, grad, n, a, clip_coef);
}

int hnh_clip_coef_f64(double *total_coef, const double *squared_norms, int64_t count, double max_norm, void *stream) {
    if (count < 0) return set_error(HNH_E_INVALID, "hnh_clip_coef_f64: negative count");
    if (!(max_norm >= 0.0)) return set_error(HNH_E_INVALID, "hnh_clip_coef_f64: max_norm must be >= 0 (+inf: no clipping)");
    if (!total_coef || (count > 0 && !squared_norms)) return set_error(HNH_E_INVALID, "hnh_clip_coef_f64: null pointer");
    return launch(clip_coef_kernel, 1, 1, (cudaStream_t)stream, "clip_coef_kernel", total_coef, squared_norms, count, max_norm);
}

}  // extern "C"
