// row_regs.cuh -- the pieces shared by the one-warp-per-row kernels that keep a row in registers (the LayerNorm kernels of
// graph_transformer.cu, the cross-entropy kernel of training.cu) and by their column or scalar reductions:
//   - the register-row layout (ln_col, ln_load) and its width table (pick_ln);
//   - the two-stage fixed-order reduction: partial sums over fixed row chunks (dw_chunks: depending on n only, never on
//     the device), then the chunks summed in order (gate_dw_final_kernel).  No atomics, so repeated calls are
//     bit-identical everywhere.
#pragma once
#include "row_gather.cuh"

namespace {

constexpr int64_t kMaxChunks = 128;    // partial sums: at most this many row chunks ...
constexpr int64_t kMinChunkRows = 512; // ... of at least this many rows (fewer chunks for small n)

int64_t dw_chunks(int64_t n) { return std::max<int64_t>(1, std::min<int64_t>(kMaxChunks, (n + kMinChunkRows - 1) / kMinChunkRows)); }

// dw[j] = sum over the chunks, in order, of partial[c, j]
__global__ void __launch_bounds__(kBlock)
gate_dw_final_kernel(double *__restrict__ dw, const double *__restrict__ partial, int64_t chunks, int64_t len) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; j < len; j += stride) {
        double s = 0.0;
        for (int64_t c = 0; c < chunks; c++) s += partial[c * len + j];
        dw[j] = s;
    }
}

// Register rows.  kN > 0: a lane keeps 2 kN elements of the row in registers (r <= 64 kN), so the row is read once;
// with kPairs they are the pairs lane + 32 j (j < kN), else the scalars lane + 32 j (j < 2 kN).  kN = 0: any r, every
// pass rereads the row (from L1 / L2).  Slot j of a lane holds column ln_col<kPairs>(j, lane); a lane's columns rise
// with j.
template <bool kPairs>
__device__ __forceinline__ int64_t ln_col(int j, int lane) {
    return kPairs ? 2 * (int64_t)(lane + 32 * (j >> 1)) + (j & 1) : (int64_t)lane + 32 * j;
}

// v = p[row] (+ q[row] when q is not null), zero past the row end
template <bool kPairs, int kN>
__device__ __forceinline__ void ln_load(double (&v)[2 * kN], const double *p, const double *q, int64_t r, int lane) {
    if (kPairs) {
        const double2 *p2 = reinterpret_cast<const double2 *>(p), *q2 = reinterpret_cast<const double2 *>(q);
#pragma unroll
        for (int j = 0; j < kN; j++) {
            const int64_t k = lane + 32 * j;
            double2 a = make_double2(0.0, 0.0);
            if (k < r / 2) {
                a = __ldcs(p2 + k);
                if (q) {
                    const double2 c = __ldcs(q2 + k);
                    a = make_double2(a.x + c.x, a.y + c.y);
                }
            }
            v[2 * j] = a.x;
            v[2 * j + 1] = a.y;
        }
    } else {
#pragma unroll
        for (int j = 0; j < 2 * kN; j++) {
            const int64_t k = lane + 32 * j;
            v[j] = k < r ? (q ? __ldcs(p + k) + __ldcs(q + k) : __ldcs(p + k)) : 0.0;
        }
    }
}

// the register-row instantiation for width r (kN = 0 past the widest)
template <int kWidest, typename K>
K pick_ln(int64_t r, K k1, K k2, K k4, K k8, K k12, K k16, K k24, K k0) {
    const int64_t per = (r + 63) / 64;
    K k = per <= 1 ? k1 : per <= 2 ? k2 : per <= 4 ? k4 : per <= 8 ? k8 : per <= 12 ? k12 : per <= 16 ? k16 : per <= 24 ? k24 : k0;
    return per <= kWidest ? k : k0;
}

}  // namespace
