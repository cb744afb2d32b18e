// kernels.cuh -- sm_90a device code for the HnH local kernels (K1 SDDMM, K2 SpMM,
// K3 fused SDDMM->SpMM).
//
// What these replace (reference, CPU): StandardKernel::sddmm_local
// (sparse_kernels.cpp:13-57, an OpenMP loop over nonzeros) and
// StandardKernel::spmm_local (sparse_kernels.cpp:59-127, mkl_sparse_d_mm).
//
// Design (see DESIGN.md section 3): the path is an r-wide gather-dot, HBM-bound
// (~0.24 flop/B in fp64); no tensor-core path.  One group of G lanes owns one CSR row:
//   * the row-side factor row (X[row], r doubles) lives in registers for the whole row;
//   * a chunk of G nonzeros' (col, value) is read coalesced, one per lane, and broadcast
//     inside the group with shuffles;
//   * each gathered Y row is read with 128-bit loads (the widest global load on sm_90),
//     UN rows in flight per lane (K3 at G = 32: through a per-warp cp.async ring, fused_ring_kernel);
//   * the r-wide dot is reduced with an xor-butterfly of width G;
//   * results of a chunk are written back coalesced (lane k owns nonzero k).
// SpMM / fused accumulate the output row in registers in stored CSR order (bit-compatible
// with the row-major CSR restatement in oracle/hnh_oracle.c) and touch Y[row] once.
#pragma once
#include "row_gather.cuh"

namespace hnh {

// SDDMM epilogue.  Plain: values[j] = d.  With `scale` (the caller's S values, aligned with `values`) the Hadamard
// product of the reference's `SValues.cwiseProduct(getCSRValues())` (15D_dense_shift.hpp:364-368) is applied at the
// only moment the finished dot is in a register: scaled_out[j] = scale[j] * d (the user-visible SDDMM result); with
// scale but no scaled_out (or with scale_values) the scaled value replaces d in `values` itself (what the fused SDDMM -> SpMM of the
// replication-reuse strategy wants: the SpMM pass then reads the CSR values directly, no setCSRValues copy).
__device__ __forceinline__ void sddmm_store(double *__restrict__ values, const double *__restrict__ scale,
                                            double *__restrict__ scaled_out, bool scale_values, int64_t j, double d) {
    if (scale != nullptr) {
        const double sd = ld_stream_f64(scale + j) * d;
        if (scaled_out != nullptr) scaled_out[j] = sd;
        values[j] = (scale_values || scaled_out == nullptr) ? sd : d;
    } else {
        values[j] = d;
    }
}

// ------------------------------------------------------------------ K1: SDDMM ------------
// values[j] += X[row] . Y[col_idx[j]] for every nonzero j of every CSR row.
template <int R, int G, int VW, int UN, bool BETA0>
__global__ void __launch_bounds__(256)
sddmm_row_kernel(const int64_t *__restrict__ rowStart, const int64_t *__restrict__ col_idx,
                 double *__restrict__ values, int64_t rows, const double *__restrict__ X,
                 const double *__restrict__ Y, const double *__restrict__ scale, double *__restrict__ scaled_out,
                 bool scale_values) {
    constexpr int NV = R / (G * VW);
    static_assert(NV * G * VW == R, "R must equal NV*G*VW");
    const int lane = threadIdx.x & 31;
    const int gl = lane & (G - 1);
    const unsigned gmask = group_mask<G>(lane);
    const int64_t ngroups = (int64_t)gridDim.x * (blockDim.x / G);
    for (int64_t row = (int64_t)blockIdx.x * (blockDim.x / G) + threadIdx.x / G; row < rows;
         row += ngroups) {
        double x[NV][VW];
#pragma unroll
        for (int v = 0; v < NV; v++) ld_gather<VW>(x[v], X + row * R + (v * G + gl) * VW);
        const int64_t s = ld_stream_i64(rowStart + row);
        const int64_t e = ld_stream_i64(rowStart + row + 1);
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
                        for (int v = 0; v < NV; v++)
                            ld_gather<VW>(y[u][v], Y + c * R + (v * G + gl) * VW);
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
                        for (int w = 0; w < VW; w++) d = fma(x[v][w], y[u][v][w], d);
                    d = group_allreduce<G>(d, gmask);
                    if (gl == k0 + u) mine = d;
                }
            }
            if (gl < cnt) {
                if (!BETA0) mine += values[j + gl];
                sddmm_store(values, scale, scaled_out, scale_values, j + gl, mine);
            }
        }
    }
}

// ------------------------------------------------------------------ K2: SpMM -------------
// Y[row] += sum_j values[j] * X[col_idx[j]]   (row-major, alpha = beta = 1).
template <int R, int G, int VW, int UN, bool BETA0>
__global__ void __launch_bounds__(256)
spmm_row_kernel(const int64_t *__restrict__ rowStart, const int64_t *__restrict__ col_idx,
                const double *__restrict__ values, int64_t rows, const double *__restrict__ X,
                double *__restrict__ Y) {
    constexpr int NV = R / (G * VW);
    static_assert(NV * G * VW == R, "R must equal NV*G*VW");
    const int lane = threadIdx.x & 31;
    const int gl = lane & (G - 1);
    const unsigned gmask = group_mask<G>(lane);
    const int64_t ngroups = (int64_t)gridDim.x * (blockDim.x / G);
    for (int64_t row = (int64_t)blockIdx.x * (blockDim.x / G) + threadIdx.x / G; row < rows;
         row += ngroups) {
        const int64_t s = ld_stream_i64(rowStart + row);
        const int64_t e = ld_stream_i64(rowStart + row + 1);
        if (!BETA0 && s == e) continue;  // Y[row] += 0
        double acc[NV][VW];
#pragma unroll
        for (int v = 0; v < NV; v++) {
            if (BETA0) {
#pragma unroll
                for (int w = 0; w < VW; w++) acc[v][w] = 0.0;
            } else {
                ld_rw<VW>(acc[v], Y + row * R + (v * G + gl) * VW);
            }
        }
        for (int64_t j = s; j < e; j += G) {
            const int cnt = (e - j < G) ? (int)(e - j) : G;
            int64_t mycol = 0;
            double myval = 0.0;
            if (gl < cnt) {
                mycol = ld_stream_i64(col_idx + j + gl);
                myval = ld_stream_f64(values + j + gl);
            }
            for (int k0 = 0; k0 < cnt; k0 += UN) {
                double xg[UN][NV][VW];
                double vv[UN];
#pragma unroll
                for (int u = 0; u < UN; u++) {
                    const int k = k0 + u;
                    const int src = k < G ? k : G - 1;
                    const int64_t c = __shfl_sync(gmask, mycol, src, G);
                    vv[u] = __shfl_sync(gmask, myval, src, G);
                    if (k < cnt) {
#pragma unroll
                        for (int v = 0; v < NV; v++)
                            ld_gather<VW>(xg[u][v], X + c * R + (v * G + gl) * VW);
                    } else {
                        vv[u] = 0.0;
#pragma unroll
                        for (int v = 0; v < NV; v++)
#pragma unroll
                            for (int w = 0; w < VW; w++) xg[u][v][w] = 0.0;
                    }
                }
#pragma unroll
                for (int u = 0; u < UN; u++)
#pragma unroll
                    for (int v = 0; v < NV; v++)
#pragma unroll
                        for (int w = 0; w < VW; w++)
                            acc[v][w] = fma(vv[u], xg[u][v][w], acc[v][w]);
            }
        }
#pragma unroll
        for (int v = 0; v < NV; v++) st_rw<VW>(Y + row * R + (v * G + gl) * VW, acc[v]);
    }
}

// ------------------------------------------------------------------ K3: fused ------------
// values[j] += X[row].Y[col_j];  Out[row] += sum_j values[j] * Y[col_j]; one gather per nnz.
// BV: values = dot (old values not read).  BO: Out = result (old Out not read); Out may then
// alias X (each row of X is read only by the group that later writes that row of Out).
// SC: values[j] = scale[j] * (X[row].Y[col_j]) -- the reference's Hadamard product with the caller's S values between
// its SDDMM and SpMM passes (distributed_sparse.h:289-312) -- and scaled_out[j] (if given) receives the same number.
template <int R, int G, int VW, int UN, bool BV, bool BO, bool SC = false>
__global__ void __launch_bounds__(256)
fused_row_kernel(const int64_t *__restrict__ rowStart, const int64_t *__restrict__ col_idx,
                 double *__restrict__ values, int64_t rows, const double *X,
                 const double *__restrict__ Y, double *Out, const double *__restrict__ scale = nullptr,
                 double *__restrict__ scaled_out = nullptr) {
    constexpr int NV = R / (G * VW);
    static_assert(NV * G * VW == R, "R must equal NV*G*VW");
    const int lane = threadIdx.x & 31;
    const int gl = lane & (G - 1);
    const unsigned gmask = group_mask<G>(lane);
    const int64_t ngroups = (int64_t)gridDim.x * (blockDim.x / G);
    for (int64_t row = (int64_t)blockIdx.x * (blockDim.x / G) + threadIdx.x / G; row < rows;
         row += ngroups) {
        const int64_t s = ld_stream_i64(rowStart + row);
        const int64_t e = ld_stream_i64(rowStart + row + 1);
        if (!BO && s == e) continue;
        double x[NV][VW], acc[NV][VW];
#pragma unroll
        for (int v = 0; v < NV; v++) {
            ld_rw<VW>(x[v], X + row * R + (v * G + gl) * VW);
            if (BO) {
#pragma unroll
                for (int w = 0; w < VW; w++) acc[v][w] = 0.0;
            } else {
                ld_rw<VW>(acc[v], Out + row * R + (v * G + gl) * VW);
            }
        }
        for (int64_t j = s; j < e; j += G) {
            const int cnt = (e - j < G) ? (int)(e - j) : G;
            int64_t mycol = 0;
            double myval = 0.0, mysc = 1.0;
            if (gl < cnt) {
                mycol = ld_stream_i64(col_idx + j + gl);
                if (!BV) myval = values[j + gl];
                if (SC) mysc = ld_stream_f64(scale + j + gl);
            }
            for (int k0 = 0; k0 < cnt; k0 += UN) {
                double y[UN][NV][VW];
                double vold[UN], vsc[UN];
#pragma unroll
                for (int u = 0; u < UN; u++) {
                    const int k = k0 + u;
                    const int src = k < G ? k : G - 1;
                    const int64_t c = __shfl_sync(gmask, mycol, src, G);
                    vold[u] = __shfl_sync(gmask, myval, src, G);
                    if (SC) vsc[u] = __shfl_sync(gmask, mysc, src, G);
                    if (k < cnt) {
#pragma unroll
                        for (int v = 0; v < NV; v++)
                            ld_gather<VW>(y[u][v], Y + c * R + (v * G + gl) * VW);
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
                        for (int w = 0; w < VW; w++) d = fma(x[v][w], y[u][v][w], d);
                    d = group_allreduce<G>(d, gmask);
                    const double vnew = SC ? (vold[u] + d) * vsc[u] : vold[u] + d;
                    if (gl == k0 + u) myval = vnew;
                    if (k0 + u < cnt) {
#pragma unroll
                        for (int v = 0; v < NV; v++)
#pragma unroll
                            for (int w = 0; w < VW; w++)
                                acc[v][w] = fma(vnew, y[u][v][w], acc[v][w]);
                    }
                }
            }
            if (gl < cnt) {
                values[j + gl] = myval;
                if (SC && scaled_out != nullptr) scaled_out[j + gl] = myval;
            }
        }
#pragma unroll
        for (int v = 0; v < NV; v++) st_rw<VW>(Out + row * R + (v * G + gl) * VW, acc[v]);
    }
}

__device__ __forceinline__ unsigned smem_u32(const void *p) { return (unsigned)__cvta_generic_to_shared(p); }
// 16 bytes global -> shared, bypassing L1 (SASS LDGSTS); completion is tracked per thread in commit groups
__device__ __forceinline__ void cp_async16(void *smem_dst, const void *gmem_src) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_u32(smem_dst)), "l"(gmem_src) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
// wait until at most N of this thread's committed groups are still in flight
template <int N>
__device__ __forceinline__ void cp_async_wait() {
    asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory");
}

// K3 with the gathered rows staged through a per-warp shared-memory ring (the G = 32 widths; see DESIGN.md section 3).
// Same contract, lane shape (one warp per CSR row, VW = 2) and arithmetic as fused_row_kernel: per entry the same FMA
// order over (v, w), the same xor-butterfly, the same accumulator FMAs in stored CSR order, so the results are
// bit-identical.  What differs is where a gathered row waits: each lane copies its own 16-byte slices of the warp's
// next batches of UN rows into a ring of S slots with cp.async (one commit group per batch), and reads back only the
// bytes it wrote itself -- so no barrier or __syncwarp is needed and the LDS.128 reads are bank-conflict-free.  While
// batch k is reduced, batches k+1 .. k+S-1 are in flight.  The copy side walks the warp's own stream of entries
// (its rows, row += grid stride) independently of the compute side, so the ring runs across row ends; it keeps the
// bounds of its next two rows and the next row's first chunk of column indices loaded ahead, so starting a row costs
// no dependent index round trip.
template <int R, int UN, int S, int MINB, bool BV, bool BO, bool SC = false>
__global__ void __launch_bounds__(256, MINB)
fused_ring_kernel(const int64_t *__restrict__ rowStart, const int64_t *__restrict__ col_idx,
                  double *__restrict__ values, int64_t rows, const double *X,
                  const double *__restrict__ Y, double *Out, const double *__restrict__ scale = nullptr,
                  double *__restrict__ scaled_out = nullptr) {
    constexpr int G = 32, VW = 2, NV = R / (G * VW);
    static_assert(NV * G * VW == R, "R must be a multiple of 64");
    static_assert(G % UN == 0 && S >= 2, "a batch never straddles a chunk of G entries; the ring has 2+ slots");
    __shared__ alignas(16) double ring[kBlock / 32][S][UN][R];
    const int lane = threadIdx.x & 31;
    double(*const my)[UN][R] = ring[threadIdx.x >> 5];
    const unsigned gmask = 0xffffffffu;
    const int64_t ngroups = (int64_t)gridDim.x * (blockDim.x / G);
    const int64_t first = (int64_t)blockIdx.x * (blockDim.x / G) + threadIdx.x / G;

    // ---- copy side: p_row's entries [p_j, p_e), chunk of G column indices at p_c0 (lane k holds entry p_c0 + k);
    // the next row's bounds and first chunk (n1_*) and the bounds of the row after it (n2_*) are already loaded
    int64_t p_row = first - ngroups, p_j = 0, p_e = 0, p_c0 = 0, p_col = 0;
    int64_t n1_s = 0, n1_e = 0, n1_col = 0, n2_s = 0, n2_e = 0;
    if (first < rows) {
        n1_s = ld_stream_i64(rowStart + first);
        n1_e = ld_stream_i64(rowStart + first + 1);
        if (lane < n1_e - n1_s) n1_col = ld_stream_i64(col_idx + n1_s + lane);
    }
    if (first + ngroups < rows) {
        n2_s = ld_stream_i64(rowStart + first + ngroups);
        n2_e = ld_stream_i64(rowStart + first + ngroups + 1);
    }
    int p_slot = 0;
    // one commit group per call: the next batch of up to UN entries of the stream, or nothing once it has ended
    auto issue_batch = [&]() {
        while (p_j == p_e && p_row < rows) {  // row done (or empty): step to the next one
            p_row += ngroups;
            if (p_row >= rows) break;
            p_j = p_c0 = n1_s;
            p_e = n1_e;
            p_col = n1_col;
            n1_s = n2_s;
            n1_e = n2_e;
            n1_col = 0;
            if (p_row + ngroups < rows && lane < n1_e - n1_s) n1_col = ld_stream_i64(col_idx + n1_s + lane);
            if (p_row + 2 * ngroups < rows) {
                n2_s = ld_stream_i64(rowStart + p_row + 2 * ngroups);
                n2_e = ld_stream_i64(rowStart + p_row + 2 * ngroups + 1);
            }
        }
        if (p_j < p_e) {
            if (p_j == p_c0 + G) {  // the row's next chunk of G entries
                p_c0 = p_j;
                p_col = lane < p_e - p_j ? ld_stream_i64(col_idx + p_j + lane) : 0;
            }
            const int k0 = (int)(p_j - p_c0);
            const int64_t left = (p_e < p_c0 + G ? p_e : p_c0 + G) - p_j;
            const int n = left < UN ? (int)left : UN;
#pragma unroll
            for (int u = 0; u < UN; u++) {
                const int64_t c = __shfl_sync(gmask, p_col, k0 + u);
                if (u < n) {
#pragma unroll
                    for (int v = 0; v < NV; v++)
                        cp_async16(&my[p_slot][u][(v * G + lane) * VW], Y + c * R + (v * G + lane) * VW);
                }
            }
            p_j += n;
        }
        cp_async_commit();
        p_slot = p_slot + 1 == S ? 0 : p_slot + 1;
    };
#pragma unroll
    for (int b = 0; b < S - 1; b++) issue_batch();

    // ---- compute side: fused_row_kernel's row loop, reading each batch from the ring
    int c_slot = 0;
    int64_t s = 0, e = 0;
    if (first < rows) {
        s = ld_stream_i64(rowStart + first);
        e = ld_stream_i64(rowStart + first + 1);
    }
    for (int64_t row = first; row < rows; row += ngroups) {
        const int64_t rs = s, re = e;
        if (row + ngroups < rows) {  // the next row's bounds, used one row later
            s = ld_stream_i64(rowStart + row + ngroups);
            e = ld_stream_i64(rowStart + row + ngroups + 1);
        }
        if (!BO && rs == re) continue;
        double x[NV][VW], acc[NV][VW];
#pragma unroll
        for (int v = 0; v < NV; v++) {
            ld_rw<VW>(x[v], X + row * R + (v * G + lane) * VW);
            if (BO) {
#pragma unroll
                for (int w = 0; w < VW; w++) acc[v][w] = 0.0;
            } else {
                ld_rw<VW>(acc[v], Out + row * R + (v * G + lane) * VW);
            }
        }
        for (int64_t j = rs; j < re; j += G) {
            const int cnt = (re - j < G) ? (int)(re - j) : G;
            double myval = 0.0, mysc = 1.0;
            if (lane < cnt) {
                if (!BV) myval = values[j + lane];
                if (SC) mysc = ld_stream_f64(scale + j + lane);
            }
            for (int k0 = 0; k0 < cnt; k0 += UN) {
                issue_batch();
                cp_async_wait<S - 1>();  // this lane's slices of batch (row, j, k0) have landed
                const double(*const yb)[R] = my[c_slot];
                c_slot = c_slot + 1 == S ? 0 : c_slot + 1;
#pragma unroll
                for (int u = 0; u < UN; u++) {
                    if (k0 + u < cnt) {
                        double y[NV][VW];
#pragma unroll
                        for (int v = 0; v < NV; v++) {
                            const double2 t = *reinterpret_cast<const double2 *>(&yb[u][(v * G + lane) * VW]);
                            y[v][0] = t.x;
                            y[v][1] = t.y;
                        }
                        // BV: the old value is 0.0; the addition stays, so that a -0.0 dot is stored as +0.0
                        const double vold = BV ? 0.0 : __shfl_sync(gmask, myval, k0 + u);
                        double d = 0.0;
#pragma unroll
                        for (int v = 0; v < NV; v++)
#pragma unroll
                            for (int w = 0; w < VW; w++) d = fma(x[v][w], y[v][w], d);
                        d = group_allreduce<G>(d, gmask);
                        const double vnew = SC ? (vold + d) * __shfl_sync(gmask, mysc, k0 + u) : vold + d;
                        if (lane == k0 + u) myval = vnew;
#pragma unroll
                        for (int v = 0; v < NV; v++)
#pragma unroll
                            for (int w = 0; w < VW; w++) acc[v][w] = fma(vnew, y[v][w], acc[v][w]);
                    }
                }
            }
            if (lane < cnt) {
                values[j + lane] = myval;
                if (SC && scaled_out != nullptr) scaled_out[j + lane] = myval;
            }
        }
#pragma unroll
        for (int v = 0; v < NV; v++) st_rw<VW>(Out + row * R + (v * G + lane) * VW, acc[v]);
    }
    cp_async_wait<0>();
}

// ------------------------------------------------------------------ TMA-staged variants ---
// The row-side factor tile X[row0 .. row0+TR) of the TR = 8 rows a CTA works on is one contiguous
// TR*R*8-byte span: a single elected thread fetches it with ONE bulk asynchronous copy
// (cp.async.bulk.shared::cluster.global, SASS UBLKCP) that signals an mbarrier, and -- because each
// warp moves its row into registers as soon as the tile has landed -- the copy of the NEXT tile is
// issued right away and flies while the current tile's rows are being gathered.  The X stream thus
// costs no LSU instruction and no exposed latency.  The gathered Y rows stay direct 128-bit loads
// into registers (random 8R-byte rows consumed once: staging them would add a shared-memory hop
// and remove no HBM traffic).  Selected with HNH_FLAG_TMA_STAGE; compared with the direct-load
// kernels.  G and VW equal the direct kernels' (32, 2), so both compute in the same order.
__device__ __forceinline__ void mbar_init(uint64_t *bar, unsigned count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void bulk_load(void *smem_dst, const void *gmem_src, unsigned bytes, uint64_t *bar) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                     smem_u32(smem_dst)),
                 "l"(gmem_src), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t *bar, unsigned parity) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "HNH_WAIT:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra HNH_DONE;\n"
        "bra HNH_WAIT;\n"
        "HNH_DONE:\n"
        "}\n" ::"r"(smem_u32(bar)),
        "r"(parity)
        : "memory");
}

// FUSED == false: SDDMM (values (+)= X.Y).  FUSED == true: SDDMM -> SpMM with one gather.
template <int R, int UN, bool FUSED, bool BV, bool BO>
__global__ void __launch_bounds__(256)
tma_row_kernel(const int64_t *__restrict__ rowStart, const int64_t *__restrict__ col_idx, double *__restrict__ values,
               int64_t rows, const double *X, const double *__restrict__ Y, double *Out, const double *__restrict__ scale,
               double *__restrict__ scaled_out, bool scale_values) {
    constexpr int G = 32, VW = 2, TR = 8;
    constexpr int NV = R / (G * VW);
    static_assert(NV * G * VW == R, "R must be a multiple of 64");
    __shared__ alignas(128) double xs[TR][R];
    __shared__ alignas(8) uint64_t bar;
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    const unsigned gmask = 0xffffffffu;
    const int64_t ntiles = (rows + TR - 1) / TR;
    if (threadIdx.x == 0) mbar_init(&bar, 1);
    __syncthreads();
    int64_t tile = blockIdx.x;
    auto issue = [&](int64_t t) {
        const int64_t r0 = t * TR;
        const int64_t nr = rows - r0 < TR ? rows - r0 : TR;
        bulk_load(&xs[0][0], X + r0 * R, (unsigned)(nr * R * sizeof(double)), &bar);
    };
    if (threadIdx.x == 0 && tile < ntiles) issue(tile);
    unsigned parity = 0;
    for (; tile < ntiles; tile += gridDim.x) {
        const int64_t row = tile * TR + w;
        mbar_wait(&bar, parity);
        parity ^= 1;
        double x[NV][VW];
#pragma unroll
        for (int v = 0; v < NV; v++)
#pragma unroll
            for (int q = 0; q < VW; q++) x[v][q] = xs[w][(v * G + lane) * VW + q];
        __syncthreads();  // every warp holds its row in registers: the tile buffer is free again
        if (threadIdx.x == 0 && tile + gridDim.x < ntiles) issue(tile + gridDim.x);  // prefetch
        if (row >= rows) continue;
        const int64_t s = ld_stream_i64(rowStart + row);
        const int64_t e = ld_stream_i64(rowStart + row + 1);
        double acc[NV][VW];
        if (FUSED) {
            if (!BO && s == e) continue;
#pragma unroll
            for (int v = 0; v < NV; v++) {
                if (BO) {
#pragma unroll
                    for (int q = 0; q < VW; q++) acc[v][q] = 0.0;
                } else {
                    ld_rw<VW>(acc[v], Out + row * R + (v * G + lane) * VW);
                }
            }
        }
        for (int64_t j = s; j < e; j += G) {
            const int cnt = (e - j < G) ? (int)(e - j) : G;
            int64_t mycol = 0;
            double myval = 0.0;
            if (lane < cnt) {
                mycol = ld_stream_i64(col_idx + j + lane);
                if (!BV) myval = values[j + lane];
            }
            for (int k0 = 0; k0 < cnt; k0 += UN) {
                double y[UN][NV][VW];
                double vold[UN];
#pragma unroll
                for (int u = 0; u < UN; u++) {
                    const int k = k0 + u;
                    const int src = k < G ? k : G - 1;
                    const int64_t c = __shfl_sync(gmask, mycol, src, G);
                    vold[u] = __shfl_sync(gmask, myval, src, G);
                    if (k < cnt) {
#pragma unroll
                        for (int v = 0; v < NV; v++) ld_gather<VW>(y[u][v], Y + c * R + (v * G + lane) * VW);
                    } else {
#pragma unroll
                        for (int v = 0; v < NV; v++)
#pragma unroll
                            for (int q = 0; q < VW; q++) y[u][v][q] = 0.0;
                    }
                }
#pragma unroll
                for (int u = 0; u < UN; u++) {
                    double d = 0.0;
#pragma unroll
                    for (int v = 0; v < NV; v++)
#pragma unroll
                        for (int q = 0; q < VW; q++) d = fma(x[v][q], y[u][v][q], d);
                    d = group_allreduce<G>(d, gmask);
                    const double vnew = vold[u] + d;
                    if (lane == k0 + u) myval = vnew;
                    if (FUSED && k0 + u < cnt) {
#pragma unroll
                        for (int v = 0; v < NV; v++)
#pragma unroll
                            for (int q = 0; q < VW; q++) acc[v][q] = fma(vnew, y[u][v][q], acc[v][q]);
                    }
                }
            }
            if (lane < cnt) {
                if (FUSED) values[j + lane] = myval;
                else sddmm_store(values, scale, scaled_out, scale_values, j + lane, myval);
            }
        }
        if (FUSED) {
#pragma unroll
            for (int v = 0; v < NV; v++) st_rw<VW>(Out + row * R + (v * G + lane) * VW, acc[v]);
        }
    }
}

// Per-warp variant (HNH_FLAG_TMA_WARP; experimental, never the default): every warp owns two
// row-sized shared-memory slots and two mbarriers and prefetches the X row of its NEXT CSR row with
// its own bulk copy while it gathers for the current one.  No block-wide barrier, so the warps of a
// CTA do not wait for each other's longest row (the cost that makes tma_row_kernel lose at r = 128
// for the fused kernel).
template <int R, int UN, bool FUSED, bool BV, bool BO>
__global__ void __launch_bounds__(256)
tma_warp_kernel(const int64_t *__restrict__ rowStart, const int64_t *__restrict__ col_idx, double *__restrict__ values,
                int64_t rows, const double *X, const double *__restrict__ Y, double *Out, const double *__restrict__ scale,
               double *__restrict__ scaled_out, bool scale_values) {
    constexpr int G = 32, VW = 2, NW = 8;
    constexpr int NV = R / (G * VW);
    static_assert(NV * G * VW == R, "R must be a multiple of 64");
    __shared__ alignas(128) double xs[NW][2][R];
    __shared__ alignas(8) uint64_t bars[NW][2];
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    const unsigned gmask = 0xffffffffu;
    const int64_t stride = (int64_t)gridDim.x * NW;
    int64_t row = (int64_t)blockIdx.x * NW + w;
    if (lane == 0) {
        mbar_init(&bars[w][0], 1);
        mbar_init(&bars[w][1], 1);
    }
    __syncwarp();
    unsigned par0 = 0, par1 = 0;
    int slot = 0;
    if (lane == 0 && row < rows) bulk_load(&xs[w][0][0], X + row * R, (unsigned)(R * sizeof(double)), &bars[w][0]);
    for (; row < rows; row += stride) {
        const int64_t next = row + stride;
        if (lane == 0 && next < rows)
            bulk_load(&xs[w][slot ^ 1][0], X + next * R, (unsigned)(R * sizeof(double)), &bars[w][slot ^ 1]);
        if (slot == 0) { mbar_wait(&bars[w][0], par0); par0 ^= 1; }
        else { mbar_wait(&bars[w][1], par1); par1 ^= 1; }
        double x[NV][VW];
#pragma unroll
        for (int v = 0; v < NV; v++)
#pragma unroll
            for (int q = 0; q < VW; q++) x[v][q] = xs[w][slot][(v * G + lane) * VW + q];
        __syncwarp();  // the slot may be refilled from the next iteration on
        slot ^= 1;
        const int64_t s = ld_stream_i64(rowStart + row);
        const int64_t e = ld_stream_i64(rowStart + row + 1);
        if (FUSED && !BO && s == e) continue;
        double acc[NV][VW];
        if (FUSED) {
#pragma unroll
            for (int v = 0; v < NV; v++) {
                if (BO) {
#pragma unroll
                    for (int q = 0; q < VW; q++) acc[v][q] = 0.0;
                } else {
                    ld_rw<VW>(acc[v], Out + row * R + (v * G + lane) * VW);
                }
            }
        }
        for (int64_t j = s; j < e; j += G) {
            const int cnt = (e - j < G) ? (int)(e - j) : G;
            int64_t mycol = 0;
            double myval = 0.0;
            if (lane < cnt) {
                mycol = ld_stream_i64(col_idx + j + lane);
                if (!BV) myval = values[j + lane];
            }
            for (int k0 = 0; k0 < cnt; k0 += UN) {
                double y[UN][NV][VW];
                double vold[UN];
#pragma unroll
                for (int u = 0; u < UN; u++) {
                    const int k = k0 + u;
                    const int src = k < G ? k : G - 1;
                    const int64_t c = __shfl_sync(gmask, mycol, src, G);
                    vold[u] = __shfl_sync(gmask, myval, src, G);
                    if (k < cnt) {
#pragma unroll
                        for (int v = 0; v < NV; v++) ld_gather<VW>(y[u][v], Y + c * R + (v * G + lane) * VW);
                    } else {
#pragma unroll
                        for (int v = 0; v < NV; v++)
#pragma unroll
                            for (int q = 0; q < VW; q++) y[u][v][q] = 0.0;
                    }
                }
#pragma unroll
                for (int u = 0; u < UN; u++) {
                    double d = 0.0;
#pragma unroll
                    for (int v = 0; v < NV; v++)
#pragma unroll
                        for (int q = 0; q < VW; q++) d = fma(x[v][q], y[u][v][q], d);
                    d = group_allreduce<G>(d, gmask);
                    const double vnew = vold[u] + d;
                    if (lane == k0 + u) myval = vnew;
                    if (FUSED && k0 + u < cnt) {
#pragma unroll
                        for (int v = 0; v < NV; v++)
#pragma unroll
                            for (int q = 0; q < VW; q++) acc[v][q] = fma(vnew, y[u][v][q], acc[v][q]);
                    }
                }
            }
            if (lane < cnt) {
                if (FUSED) values[j + lane] = myval;
                else sddmm_store(values, scale, scaled_out, scale_values, j + lane, myval);
            }
        }
        if (FUSED) {
#pragma unroll
            for (int v = 0; v < NV; v++) st_rw<VW>(Out + row * R + (v * G + lane) * VW, acc[v]);
        }
    }
}

// ------------------------------------------------------------------ small-r kernels ------
// For narrow factors (r <= 32) a row is too short to feed a whole warp, so the G = GK*GN lanes
// that own a CSR row are laid out in two dimensions: GK lanes split the r columns (VW doubles
// each, one vector load), GN lanes split the row's NONZEROS (lane np takes nonzeros
// j0 + u*GN + np).  Consecutive lanes then read consecutive col_idx / values entries
// (coalesced streams, no shuffle broadcast), every lane keeps UN gathers in flight, the r-wide
// dot needs only log2(GK) shuffles, and SpMM's per-lane partial output rows are combined with
// log2(GN) shuffles at the end of the row.  The summation order over a row's nonzeros is a
// fixed tree (deterministic), not the oracle's sequential order.
template <int G, int GK>
__device__ __forceinline__ double reduce_over_k(double d, unsigned mask) {
#pragma unroll
    for (int o = GK / 2; o > 0; o >>= 1) d += __shfl_xor_sync(mask, d, o, G);
    return d;
}
template <int G, int GK>
__device__ __forceinline__ double reduce_over_n(double d, unsigned mask) {
#pragma unroll
    for (int o = GK; o < G; o <<= 1) d += __shfl_xor_sync(mask, d, o, G);
    return d;
}

template <int R, int GK, int GN, int VW, int UN, bool BETA0>
__global__ void __launch_bounds__(256)
sddmm_split_kernel(const int64_t *__restrict__ rowStart, const int64_t *__restrict__ col_idx,
                   double *__restrict__ values, int64_t rows, const double *__restrict__ X,
                   const double *__restrict__ Y, const double *__restrict__ scale, double *__restrict__ scaled_out,
                 bool scale_values) {
    constexpr int G = GK * GN;
    constexpr int NV = R / (GK * VW);
    static_assert(NV * GK * VW == R && G <= 32, "bad split shape");
    const int lane = threadIdx.x & 31;
    const int gl = lane & (G - 1);
    const int kp = gl % GK, np = gl / GK;
    const unsigned gmask = group_mask<G>(lane);
    const int64_t ngroups = (int64_t)gridDim.x * (blockDim.x / G);
    for (int64_t row = (int64_t)blockIdx.x * (blockDim.x / G) + threadIdx.x / G; row < rows;
         row += ngroups) {
        const int64_t s = ld_stream_i64(rowStart + row);
        const int64_t e = ld_stream_i64(rowStart + row + 1);
        if (s == e) continue;
        double x[NV][VW];
#pragma unroll
        for (int v = 0; v < NV; v++) ld_gather<VW>(x[v], X + row * R + (v * GK + kp) * VW);
        for (int64_t j0 = s; j0 < e; j0 += GN * UN) {
            double y[UN][NV][VW];
            double vold[UN];
#pragma unroll
            for (int u = 0; u < UN; u++) {
                const int64_t j = j0 + u * GN + np;
                vold[u] = 0.0;
                if (j < e) {
                    const int64_t c = ld_stream_i64(col_idx + j);
                    if (!BETA0) vold[u] = ld_rw_f64(values + j);
#pragma unroll
                    for (int v = 0; v < NV; v++)
                        ld_gather<VW>(y[u][v], Y + c * R + (v * GK + kp) * VW);
                } else {
#pragma unroll
                    for (int v = 0; v < NV; v++)
#pragma unroll
                        for (int w = 0; w < VW; w++) y[u][v][w] = 0.0;
                }
            }
#pragma unroll
            for (int u = 0; u < UN; u++) {
                const int64_t j = j0 + u * GN + np;
                double d = 0.0;
#pragma unroll
                for (int v = 0; v < NV; v++)
#pragma unroll
                    for (int w = 0; w < VW; w++) d = fma(x[v][w], y[u][v][w], d);
                d = reduce_over_k<G, GK>(d, gmask);
                if (j < e && kp == 0) sddmm_store(values, scale, scaled_out, scale_values, j, vold[u] + d);
            }
        }
    }
}

template <int R, int GK, int GN, int VW, int UN, bool BETA0>
__global__ void __launch_bounds__(256)
spmm_split_kernel(const int64_t *__restrict__ rowStart, const int64_t *__restrict__ col_idx,
                  const double *__restrict__ values, int64_t rows, const double *__restrict__ X,
                  double *__restrict__ Y) {
    constexpr int G = GK * GN;
    constexpr int NV = R / (GK * VW);
    static_assert(NV * GK * VW == R && G <= 32, "bad split shape");
    const int lane = threadIdx.x & 31;
    const int gl = lane & (G - 1);
    const int kp = gl % GK, np = gl / GK;
    const unsigned gmask = group_mask<G>(lane);
    const int64_t ngroups = (int64_t)gridDim.x * (blockDim.x / G);
    for (int64_t row = (int64_t)blockIdx.x * (blockDim.x / G) + threadIdx.x / G; row < rows;
         row += ngroups) {
        const int64_t s = ld_stream_i64(rowStart + row);
        const int64_t e = ld_stream_i64(rowStart + row + 1);
        if (!BETA0 && s == e) continue;
        double acc[NV][VW];
#pragma unroll
        for (int v = 0; v < NV; v++)
#pragma unroll
            for (int w = 0; w < VW; w++) acc[v][w] = 0.0;
        for (int64_t j0 = s; j0 < e; j0 += GN * UN) {
            double xg[UN][NV][VW];
            double vv[UN];
#pragma unroll
            for (int u = 0; u < UN; u++) {
                const int64_t j = j0 + u * GN + np;
                if (j < e) {
                    const int64_t c = ld_stream_i64(col_idx + j);
                    vv[u] = ld_stream_f64(values + j);
#pragma unroll
                    for (int v = 0; v < NV; v++)
                        ld_gather<VW>(xg[u][v], X + c * R + (v * GK + kp) * VW);
                } else {
                    vv[u] = 0.0;
#pragma unroll
                    for (int v = 0; v < NV; v++)
#pragma unroll
                        for (int w = 0; w < VW; w++) xg[u][v][w] = 0.0;
                }
            }
#pragma unroll
            for (int u = 0; u < UN; u++)
#pragma unroll
                for (int v = 0; v < NV; v++)
#pragma unroll
                    for (int w = 0; w < VW; w++) acc[v][w] = fma(vv[u], xg[u][v][w], acc[v][w]);
        }
#pragma unroll
        for (int v = 0; v < NV; v++)
#pragma unroll
            for (int w = 0; w < VW; w++) acc[v][w] = reduce_over_n<G, GK>(acc[v][w], gmask);
        if (np == 0) {
#pragma unroll
            for (int v = 0; v < NV; v++) {
                if (!BETA0) {
                    double old[VW];
                    ld_rw<VW>(old, Y + row * R + (v * GK + kp) * VW);
#pragma unroll
                    for (int w = 0; w < VW; w++) acc[v][w] += old[w];
                }
                st_rw<VW>(Y + row * R + (v * GK + kp) * VW, acc[v]);
            }
        }
    }
}

template <int R, int GK, int GN, int VW, int UN, bool BV, bool BO, bool SC = false>
__global__ void __launch_bounds__(256)
fused_split_kernel(const int64_t *__restrict__ rowStart, const int64_t *__restrict__ col_idx,
                   double *__restrict__ values, int64_t rows, const double *X,
                   const double *__restrict__ Y, double *Out, const double *__restrict__ scale = nullptr,
                   double *__restrict__ scaled_out = nullptr) {
    constexpr int G = GK * GN;
    constexpr int NV = R / (GK * VW);
    static_assert(NV * GK * VW == R && G <= 32, "bad split shape");
    const int lane = threadIdx.x & 31;
    const int gl = lane & (G - 1);
    const int kp = gl % GK, np = gl / GK;
    const unsigned gmask = group_mask<G>(lane);
    const int64_t ngroups = (int64_t)gridDim.x * (blockDim.x / G);
    for (int64_t row = (int64_t)blockIdx.x * (blockDim.x / G) + threadIdx.x / G; row < rows;
         row += ngroups) {
        const int64_t s = ld_stream_i64(rowStart + row);
        const int64_t e = ld_stream_i64(rowStart + row + 1);
        if (!BO && s == e) continue;
        double x[NV][VW], acc[NV][VW];
#pragma unroll
        for (int v = 0; v < NV; v++) {
            ld_rw<VW>(x[v], X + row * R + (v * GK + kp) * VW);
#pragma unroll
            for (int w = 0; w < VW; w++) acc[v][w] = 0.0;
        }
        for (int64_t j0 = s; j0 < e; j0 += GN * UN) {
            double y[UN][NV][VW];
            double vold[UN], vsc[UN];
#pragma unroll
            for (int u = 0; u < UN; u++) {
                const int64_t j = j0 + u * GN + np;
                vold[u] = 0.0;
                vsc[u] = 1.0;
                if (j < e) {
                    const int64_t c = ld_stream_i64(col_idx + j);
                    if (!BV) vold[u] = ld_rw_f64(values + j);
                    if (SC) vsc[u] = ld_stream_f64(scale + j);
#pragma unroll
                    for (int v = 0; v < NV; v++)
                        ld_gather<VW>(y[u][v], Y + c * R + (v * GK + kp) * VW);
                } else {
#pragma unroll
                    for (int v = 0; v < NV; v++)
#pragma unroll
                        for (int w = 0; w < VW; w++) y[u][v][w] = 0.0;
                }
            }
#pragma unroll
            for (int u = 0; u < UN; u++) {
                const int64_t j = j0 + u * GN + np;
                double d = 0.0;
#pragma unroll
                for (int v = 0; v < NV; v++)
#pragma unroll
                    for (int w = 0; w < VW; w++) d = fma(x[v][w], y[u][v][w], d);
                d = reduce_over_k<G, GK>(d, gmask);
                const double vnew = SC ? (vold[u] + d) * vsc[u] : vold[u] + d;
                if (j < e) {
                    if (kp == 0) {
                        values[j] = vnew;
                        if (SC && scaled_out != nullptr) scaled_out[j] = vnew;
                    }
#pragma unroll
                    for (int v = 0; v < NV; v++)
#pragma unroll
                        for (int w = 0; w < VW; w++) acc[v][w] = fma(vnew, y[u][v][w], acc[v][w]);
                }
            }
        }
#pragma unroll
        for (int v = 0; v < NV; v++)
#pragma unroll
            for (int w = 0; w < VW; w++) acc[v][w] = reduce_over_n<G, GK>(acc[v][w], gmask);
        if (np == 0) {
#pragma unroll
            for (int v = 0; v < NV; v++) {
                if (!BO) {
                    double old[VW];
                    ld_rw<VW>(old, Out + row * R + (v * GK + kp) * VW);
#pragma unroll
                    for (int w = 0; w < VW; w++) acc[v][w] += old[w];
                }
                st_rw<VW>(Out + row * R + (v * GK + kp) * VW, acc[v]);
            }
        }
    }
}

// ------------------------------------------------------------------ COO-driven SDDMM -----
// The reference's literal formulation: per nonzero i, rows from row_idx[i]
// (sparse_kernels.cpp:45-47).  G lanes per nonzero, chunks of G nonzeros per group.
template <int R, int G, int VW, int UN>
__global__ void __launch_bounds__(256)
sddmm_coo_kernel(const int64_t *__restrict__ row_idx, const int64_t *__restrict__ col_idx,
                 double *__restrict__ values, int64_t nnz, const double *__restrict__ X,
                 const double *__restrict__ Y) {
    constexpr int NV = R / (G * VW);
    static_assert(NV * G * VW == R, "R must equal NV*G*VW");
    const int lane = threadIdx.x & 31;
    const int gl = lane & (G - 1);
    const unsigned gmask = group_mask<G>(lane);
    const int64_t ngroups = (int64_t)gridDim.x * (blockDim.x / G);
    const int64_t nchunks = (nnz + G - 1) / G;
    for (int64_t ch = (int64_t)blockIdx.x * (blockDim.x / G) + threadIdx.x / G; ch < nchunks;
         ch += ngroups) {
        const int64_t j = ch * G;
        const int cnt = (nnz - j < G) ? (int)(nnz - j) : G;
        int64_t mycol = 0, myrow = 0;
        if (gl < cnt) {
            mycol = ld_stream_i64(col_idx + j + gl);
            myrow = ld_stream_i64(row_idx + j + gl);
        }
        double mine = 0.0;
        for (int k0 = 0; k0 < cnt; k0 += UN) {
            double y[UN][NV][VW], x[UN][NV][VW];
#pragma unroll
            for (int u = 0; u < UN; u++) {
                const int k = k0 + u;
                const int src = k < G ? k : G - 1;
                const int64_t c = __shfl_sync(gmask, mycol, src, G);
                const int64_t rr = __shfl_sync(gmask, myrow, src, G);
                if (k < cnt) {
#pragma unroll
                    for (int v = 0; v < NV; v++) {
                        ld_gather<VW>(y[u][v], Y + c * R + (v * G + gl) * VW);
                        ld_gather<VW>(x[u][v], X + rr * R + (v * G + gl) * VW);
                    }
                } else {
#pragma unroll
                    for (int v = 0; v < NV; v++)
#pragma unroll
                        for (int w = 0; w < VW; w++) y[u][v][w] = x[u][v][w] = 0.0;
                }
            }
#pragma unroll
            for (int u = 0; u < UN; u++) {
                double d = 0.0;
#pragma unroll
                for (int v = 0; v < NV; v++)
#pragma unroll
                    for (int w = 0; w < VW; w++) d = fma(x[u][v][w], y[u][v][w], d);
                d = group_allreduce<G>(d, gmask);
                if (gl == k0 + u) mine = d;
            }
        }
        if (gl < cnt) values[j + gl] += mine;
    }
}

// ------------------------------------------------------------------ any-r kernels --------
// Warp per row, scalar strided loads; correct for every r >= 1 and any alignment.
__global__ void __launch_bounds__(256)
sddmm_generic_kernel(const int64_t *__restrict__ rowStart, const int64_t *__restrict__ col_idx,
                     double *__restrict__ values, int64_t rows, const double *__restrict__ X,
                     const double *__restrict__ Y, int r) {
    const int lane = threadIdx.x & 31;
    const int64_t nwarps = (int64_t)gridDim.x * (blockDim.x >> 5);
    for (int64_t row = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); row < rows;
         row += nwarps) {
        const int64_t s = rowStart[row], e = rowStart[row + 1];
        const double *xr = X + row * (int64_t)r;
        for (int64_t j = s; j < e; j++) {
            const double *yr = Y + col_idx[j] * (int64_t)r;
            double d = 0.0;
            for (int k = lane; k < r; k += 32) d = fma(xr[k], yr[k], d);
            d = group_allreduce<32>(d, 0xffffffffu);
            if (lane == 0) values[j] += d;
        }
    }
}

__global__ void __launch_bounds__(256)
sddmm_coo_generic_kernel(const int64_t *__restrict__ row_idx,
                         const int64_t *__restrict__ col_idx, double *__restrict__ values,
                         int64_t nnz, const double *__restrict__ X,
                         const double *__restrict__ Y, int r) {
    const int lane = threadIdx.x & 31;
    const int64_t nwarps = (int64_t)gridDim.x * (blockDim.x >> 5);
    for (int64_t j = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); j < nnz;
         j += nwarps) {
        const double *xr = X + row_idx[j] * (int64_t)r;
        const double *yr = Y + col_idx[j] * (int64_t)r;
        double d = 0.0;
        for (int k = lane; k < r; k += 32) d = fma(xr[k], yr[k], d);
        d = group_allreduce<32>(d, 0xffffffffu);
        if (lane == 0) values[j] += d;
    }
}

__global__ void __launch_bounds__(256)
spmm_generic_kernel(const int64_t *__restrict__ rowStart, const int64_t *__restrict__ col_idx,
                    const double *__restrict__ values, int64_t rows,
                    const double *__restrict__ X, double *__restrict__ Y, int r) {
    const int lane = threadIdx.x & 31;
    const int64_t nwarps = (int64_t)gridDim.x * (blockDim.x >> 5);
    for (int64_t row = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); row < rows;
         row += nwarps) {
        const int64_t s = rowStart[row], e = rowStart[row + 1];
        if (s == e) continue;
        for (int k = lane; k < r; k += 32) {
            double acc = Y[row * (int64_t)r + k];
            for (int64_t j = s; j < e; j++)
                acc = fma(values[j], X[col_idx[j] * (int64_t)r + k], acc);
            Y[row * (int64_t)r + k] = acc;
        }
    }
}

__global__ void __launch_bounds__(256)
fused_generic_kernel(const int64_t *__restrict__ rowStart, const int64_t *__restrict__ col_idx,
                     double *values, int64_t rows, const double *__restrict__ X,
                     const double *__restrict__ Y, double *__restrict__ Out, int r) {
    const int lane = threadIdx.x & 31;
    const int64_t nwarps = (int64_t)gridDim.x * (blockDim.x >> 5);
    for (int64_t row = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); row < rows;
         row += nwarps) {
        const int64_t s = rowStart[row], e = rowStart[row + 1];
        if (s == e) continue;
        const double *xr = X + row * (int64_t)r;
        for (int64_t j = s; j < e; j++) {
            const double *yr = Y + col_idx[j] * (int64_t)r;
            double d = 0.0;
            for (int k = lane; k < r; k += 32) d = fma(xr[k], yr[k], d);
            d = group_allreduce<32>(d, 0xffffffffu);
            if (lane == 0) values[j] += d;
        }
        __syncwarp();
        for (int k = lane; k < r; k += 32) {
            double acc = Out[row * (int64_t)r + k];
            for (int64_t j = s; j < e; j++)
                acc = fma(values[j], Y[col_idx[j] * (int64_t)r + k], acc);
            Out[row * (int64_t)r + k] = acc;
        }
    }
}

}  // namespace hnh
