// link_ranking.cu -- the kernels of filtered link ranking (include/hnh/link_ranking.hpp): every query's score against
// every local row, compared with the query's true score and counted, without the score matrix ever reaching memory.
//
// hnh_rank_count_f64 is dgemm_nt_kernel's tiling (gat_kernels.cu) with a counting epilogue: C = Z Q^T in 64 x 64 CTA
// tiles (rows x queries), 4 warps of 32 x 32, K in steps of 16 through shared memory, on DMMA.  Each thread compares
// its 32 accumulators in registers with the true score of their query column and counts; the counts are summed over
// the 8 row groups of a warp with shuffles, over the 2 warps sharing a column half through shared-memory atomics, and
// reach gt / ge with one 64-bit integer atomic per CTA tile and query.  Integer sums do not depend on their order, so
// every call is bit-reproducible.
//
// hnh_rank_pairs_f64 scores listed (query, row) pairs with the count kernel's arithmetic: the same instruction, the same
// chain of k steps from a zero accumulator (K padded with zeros to a multiple of 16), and the pair placed at the
// fragment position the count kernel gives it (row % 8 in the A fragment, query % 8 in the B fragment).  A score the
// count kernel compared is therefore recomputed bit for bit, and can be counted back out exactly.
#include "dmma.cuh"
#include "launch.h"

namespace {

using hnh::grid_for;
using hnh::kBlock;
using hnh::launch;
using hnh::set_error;

constexpr int kCtasPerSm = 8;
constexpr int RM = 64, RN = 64, RK = 16, R_LD = RK + 4;  // the row stride 20 keeps both fragment loads conflict-free

__global__ void __launch_bounds__(128)
rank_count_kernel(const double *__restrict__ Z, int64_t ldz, int64_t rows, const double *__restrict__ Q, int64_t ldq, int64_t n_q,
                  int r, const double *__restrict__ s_true, unsigned long long *__restrict__ gt, unsigned long long *__restrict__ ge) {
    __shared__ double Zs[RM][R_LD];
    __shared__ double Qs[RN][R_LD];
    __shared__ unsigned cnt[2][RN];  // [0]: greater, [1]: greater or equal, per query column of the tile
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int g = lane >> 2, t = lane & 3;
    const int wr = (warp >> 1) * 32, wc = (warp & 1) * 32;
    const int64_t col_tiles = (n_q + RN - 1) / RN, row_tiles = (rows + RM - 1) / RM;
    (&cnt[0][0])[threadIdx.x] = 0;
    for (int64_t tile = blockIdx.x; tile < row_tiles * col_tiles; tile += gridDim.x) {
        const int64_t row0 = (tile / col_tiles) * RM, col0 = (tile % col_tiles) * RN;
        double acc[4][4][2];
#pragma unroll
        for (int i = 0; i < 4; i++)
#pragma unroll
            for (int j = 0; j < 4; j++) acc[i][j][0] = acc[i][j][1] = 0.0;
        for (int k0 = 0; k0 < r; k0 += RK) {
            __syncthreads();
#pragma unroll
            for (int e = threadIdx.x; e < RM * RK; e += 128) {
                const int a = e / RK, c = e % RK;
                Zs[a][c] = (row0 + a < rows && k0 + c < r) ? Z[(row0 + a) * ldz + k0 + c] : 0.0;
                Qs[a][c] = (col0 + a < n_q && k0 + c < r) ? Q[(col0 + a) * ldq + k0 + c] : 0.0;
            }
            __syncthreads();
#pragma unroll
            for (int kk = 0; kk < RK; kk += 4) {
                double a[4], b[4];
#pragma unroll
                for (int i = 0; i < 4; i++) a[i] = Zs[wr + i * 8 + g][kk + t];
#pragma unroll
                for (int j = 0; j < 4; j++) b[j] = Qs[wc + j * 8 + g][kk + t];
#pragma unroll
                for (int i = 0; i < 4; i++)
#pragma unroll
                    for (int j = 0; j < 4; j++) dmma_8x8x4(acc[i][j][0], acc[i][j][1], a[i], b[j]);
            }
        }
        // per column (j, e) of this lane: (greater) + (greater or equal) << 16 over its valid rows
        unsigned packed[4][2];
#pragma unroll
        for (int j = 0; j < 4; j++)
#pragma unroll
            for (int e = 0; e < 2; e++) {
                const int64_t c = col0 + wc + j * 8 + 2 * t + e;
                const double s = c < n_q ? s_true[c] : 0.0;
                unsigned v = 0;
#pragma unroll
                for (int i = 0; i < 4; i++) {
                    const bool ok = c < n_q && row0 + wr + i * 8 + g < rows;
                    v += (ok && acc[i][j][e] > s) + ((unsigned)(ok && acc[i][j][e] >= s) << 16);
                }
#pragma unroll
                for (int m = 4; m < 32; m <<= 1) v += __shfl_xor_sync(0xffffffffu, v, m);  // over g
                packed[j][e] = v;
            }
        if (g == 0) {
#pragma unroll
            for (int j = 0; j < 4; j++)
#pragma unroll
                for (int e = 0; e < 2; e++) {
                    const int c = wc + j * 8 + 2 * t + e;
                    atomicAdd(&cnt[0][c], packed[j][e] & 0xffffu);
                    atomicAdd(&cnt[1][c], packed[j][e] >> 16);
                }
        }
        __syncthreads();
        {  // thread x owns counter x: it publishes it and clears it for the next tile
            const int kind = threadIdx.x / RN, c = threadIdx.x % RN;
            const unsigned v = cnt[kind][c];
            if (v != 0) atomicAdd((kind == 0 ? gt : ge) + col0 + c, (unsigned long long)v);
            cnt[kind][c] = 0;
        }
    }
}

// Q[q, :] = Z[anchor_q - row0, :] o D[rel_q, :] (Z's row alone when D is null) where this rank holds the anchor's row,
// 0 elsewhere and for a relation outside [0, R)
__global__ void rank_queries_kernel(double *__restrict__ Q, int64_t ldq, int64_t n_q, const double *__restrict__ Z, int64_t ldz,
                                    int64_t row0, int64_t rows, const int64_t *__restrict__ anchors, const int64_t *__restrict__ rels,
                                    const double *__restrict__ D, int64_t ldd, int R, int r) {
    const int64_t n = n_q * r, stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t x = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; x < n; x += stride) {
        const int64_t q = x / r, k = x - q * r;
        const int64_t a = anchors[q] - row0;
        double v = 0.0;
        if (a >= 0 && a < rows) {
            v = Z[a * ldz + k];
            if (D) {
                const int64_t rho = rels[q];
                v = rho >= 0 && rho < R ? v * D[rho * ldd + k] : 0.0;
            }
        }
        Q[q * ldq + k] = v;
    }
}

// One warp per pair (q, u): the count kernel's k chain at the count kernel's fragment position.  The lane holding the
// element writes the score, and counts it back out of gt / ge against s_true.
__global__ void __launch_bounds__(kBlock)
rank_pairs_kernel(const double *__restrict__ Z, int64_t ldz, int64_t rows, const double *__restrict__ Q, int64_t ldq, int64_t n_q,
                  int r, const int64_t *__restrict__ pair_q, const int64_t *__restrict__ pair_row, int64_t n_pairs,
                  double *__restrict__ scores, const double *__restrict__ s_true, unsigned long long *__restrict__ gt,
                  unsigned long long *__restrict__ ge) {
    const int lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
    const int64_t warps = (int64_t)gridDim.x * (blockDim.x >> 5);
    const int k_end = (r + RK - 1) / RK * RK;
    for (int64_t p = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); p < n_pairs; p += warps) {
        const int64_t q = pair_q[p], u = pair_row[p];
        if (q < 0 || q >= n_q || u < 0 || u >= rows) continue;  // warp-uniform
        const bool a_lane = g == (int)(u & 7), b_lane = g == (int)(q & 7);
        double c0 = 0.0, c1 = 0.0;
        for (int k = t; k < k_end + t; k += 4) {
            const double a = a_lane && k < r ? Z[u * ldz + k] : 0.0;
            const double b = b_lane && k < r ? Q[q * ldq + k] : 0.0;
            dmma_8x8x4(c0, c1, a, b);
        }
        if (a_lane && t == (int)((q & 7) >> 1)) {
            const double s = (q & 1) ? c1 : c0;
            if (scores) scores[p] = s;
            if (gt) {
                const double st = s_true[q];
                if (s > st) atomicAdd(gt + q, ~0ull);  // -1
                if (s >= st) atomicAdd(ge + q, ~0ull);
            }
        }
    }
}

bool shape_ok(int64_t rows, int64_t n_q, int r, int64_t ldz, int64_t ldq) {
    return rows >= 0 && n_q >= 0 && r >= 1 && ldz >= r && ldq >= r && rows < INT64_MAX / ldz && n_q < INT64_MAX / ldq;
}

}  // namespace

extern "C" {

int hnh_rank_count_f64(const double *Z, int64_t ldz, int64_t rows, const double *Q, int64_t ldq, int64_t n_q, int r,
                       const double *s_true, int64_t *gt, int64_t *ge, void *stream) {
    if (!shape_ok(rows, n_q, r, ldz, ldq))
        return set_error(HNH_E_INVALID, "hnh_rank_count_f64: bad shape: %lld rows, %lld queries, r = %d, ldz = %lld, ldq = %lld",
                         (long long)rows, (long long)n_q, r, (long long)ldz, (long long)ldq);
    if (rows == 0 || n_q == 0) return HNH_OK;
    if (!Z || !Q || !s_true || !gt || !ge) return set_error(HNH_E_INVALID, "hnh_rank_count_f64: null pointer");
    if (gt == ge) return set_error(HNH_E_INVALID, "hnh_rank_count_f64: gt and ge must be separate arrays");
    const int64_t tiles = ((rows + RM - 1) / RM) * ((n_q + RN - 1) / RN);
    int grid = 1;
    int rc = grid_for(rank_count_kernel, tiles, 1, &grid, kCtasPerSm);
    return rc ? rc
              : launch(rank_count_kernel, grid, 128, (cudaStream_t)stream, "rank_count_kernel", Z, ldz, rows, Q, ldq, n_q, r, s_true,
                       (unsigned long long *)gt, (unsigned long long *)ge);
}

int hnh_rank_queries_f64(double *Q, int64_t ldq, int64_t n_q, const double *Z, int64_t ldz, int64_t row0, int64_t rows,
                         const int64_t *anchors, const int64_t *rels, const double *D, int64_t ldd, int R, int r, void *stream) {
    if (!shape_ok(rows, n_q, r, ldz, ldq) || (D && (R < 1 || ldd < r)))
        return set_error(HNH_E_INVALID, "hnh_rank_queries_f64: bad shape: %lld rows, %lld queries, r = %d, R = %d, ld %lld / %lld / %lld",
                         (long long)rows, (long long)n_q, r, R, (long long)ldz, (long long)ldq, (long long)ldd);
    if (n_q == 0) return HNH_OK;
    if (!Q || !anchors || (rows > 0 && !Z) || (D && !rels)) return set_error(HNH_E_INVALID, "hnh_rank_queries_f64: null pointer");
    int grid = 1;
    int rc = grid_for(rank_queries_kernel, n_q * r, kBlock * 4, &grid, kCtasPerSm);
    return rc ? rc
              : launch(rank_queries_kernel, grid, kBlock, (cudaStream_t)stream, "rank_queries_kernel", Q, ldq, n_q, Z, ldz, row0, rows,
                       anchors, rels, D, ldd, R, r);
}

int hnh_rank_pairs_f64(const double *Z, int64_t ldz, int64_t rows, const double *Q, int64_t ldq, int64_t n_q, int r,
                       const int64_t *pair_q, const int64_t *pair_row, int64_t n_pairs, double *scores, const double *s_true,
                       int64_t *gt, int64_t *ge, void *stream) {
    if (!shape_ok(rows, n_q, r, ldz, ldq) || n_pairs < 0)
        return set_error(HNH_E_INVALID, "hnh_rank_pairs_f64: bad shape: %lld rows, %lld queries, %lld pairs, r = %d, ldz = %lld, ldq = %lld",
                         (long long)rows, (long long)n_q, (long long)n_pairs, r, (long long)ldz, (long long)ldq);
    if (n_pairs == 0 || rows == 0 || n_q == 0) return HNH_OK;
    if (!Z || !Q || !pair_q || !pair_row) return set_error(HNH_E_INVALID, "hnh_rank_pairs_f64: null pointer");
    if ((gt != nullptr) != (ge != nullptr) || (gt && !s_true))
        return set_error(HNH_E_INVALID, "hnh_rank_pairs_f64: gt and ge go together, with s_true");
    if (gt && gt == ge) return set_error(HNH_E_INVALID, "hnh_rank_pairs_f64: gt and ge must be separate arrays");
    int grid = 1;
    int rc = grid_for(rank_pairs_kernel, n_pairs, kBlock / 32, &grid, kCtasPerSm);
    return rc ? rc
              : launch(rank_pairs_kernel, grid, kBlock, (cudaStream_t)stream, "rank_pairs_kernel", Z, ldz, rows, Q, ldq, n_q, r, pair_q,
                       pair_row, n_pairs, scores, s_true, (unsigned long long *)gt, (unsigned long long *)ge);
}

}  // extern "C"
