// graph_readout.cu -- the readout of graph-level prediction (include/hnh/graph_readout.hpp): pooling the rows of the
// model's output H into one row per graph, and the gradient of that pooling.  A rank's rows are grouped by graph in a
// segment CSR, segment g = graph g: its rows seg_rows[seg_start[g] .. seg_start[g + 1]), in ascending order.
//     pool:   P_g = sum_{u in g} H_u                 (sum)
//             (P_g,k, C_g,k) = (max_u H_u,k, #{u : H_u,k == max})   (max; (-inf, 0) for an empty segment)
//     grad:   dH_u = scale_g dP_g                    (sum, mean; scale null: 1)
//             dH_u,k = [H_u,k == P_g,k] dP_g,k / C_g,k  (max)
//             dH_u = 0 for a row in no graph
// A segment of one graph can hold most of the rows, so the pool does not give a segment to one lane group: every
// segment is cut into chunks of HNH_SEGMENT_CHUNK rows (an empty segment is one empty chunk), and a group of G lanes
// owns one chunk, with the row's columns across its lanes as in link_bce_kernel (128-bit loads, UN rows in flight).
// A segment of one chunk writes its result straight into P; the chunks of a longer one write partial rows into a
// workspace, which segment_pool_merge_kernel then combines: one CTA per (segment, 32-column slab), warp w taking the
// chunks w, w + 8, .. in order, then the 8 warps' results in warp order.  The order of every sum is fixed by the
// segment lengths and two constants, never by the grid, and nothing uses atomics: repeated calls are bit-identical.
// Widths 4..256 (powers of two) with 16-byte aligned operands and even leading dimensions take the 128-bit chunk and
// row kernels; every other width takes one-warp-per-chunk (pool, in column windows of 256) and one-warp-per-row (grad)
// generic kernels.
#include <cmath>

#include "row_gather.cuh"

namespace {

using hnh::grid_for;
using hnh::launch;
using hnh::set_error;

constexpr int64_t kChunk = HNH_SEGMENT_CHUNK;
constexpr int kWindow = 256;               // the widest column window of one generic pool launch
constexpr int kMergeWarps = kBlock / 32;   // the warps of one merge CTA

// chunk k: its segment s and its rows [b, e) of seg_rows; single = the segment has no other chunk
struct Chunk {
    int64_t s, b, e;
    bool single;
};
__device__ __forceinline__ Chunk chunk_of(int64_t k, const int64_t *seg_start, const int64_t *chunk_first, const int32_t *chunk_seg) {
    const int64_t s = chunk_seg[k];
    const int64_t c0 = chunk_first[s], s1 = seg_start[s + 1];
    const int64_t b = seg_start[s] + (k - c0) * kChunk;
    return {s, b, b + kChunk < s1 ? b + kChunk : s1, chunk_first[s + 1] - c0 == 1};
}

// ---- fast chunk kernel ------------------------------------------------------------------------------------------------
template <int R, int G, int VW, int UN, bool kMax>
__global__ void __launch_bounds__(kBlock, 1)
segment_pool_kernel(const int64_t *__restrict__ seg_start, const int64_t *__restrict__ seg_rows, const int64_t *__restrict__ chunk_first,
                    const int32_t *__restrict__ chunk_seg, int64_t chunks, const double *__restrict__ H, int64_t ldh,
                    double *__restrict__ P, int64_t ldp, double *__restrict__ C, int64_t ldc, double *__restrict__ W, int64_t ldw) {
    constexpr int NV = R / (G * VW);
    static_assert(NV * G * VW == R, "R must equal NV*G*VW");
    const int lane = threadIdx.x & 31;
    const int gl = lane & (G - 1);
    const unsigned gmask = group_mask<G>(lane);
    const int64_t ngroups = (int64_t)gridDim.x * (blockDim.x / G);
    for (int64_t k = (int64_t)blockIdx.x * (blockDim.x / G) + threadIdx.x / G; k < chunks; k += ngroups) {
        const Chunk ch = chunk_of(k, seg_start, chunk_first, chunk_seg);
        double a[NV][VW], n[NV][VW];
#pragma unroll
        for (int v = 0; v < NV; v++)
#pragma unroll
            for (int w = 0; w < VW; w++) {
                a[v][w] = kMax ? -INFINITY : 0.0;
                n[v][w] = 0.0;
            }
        for (int64_t j = ch.b; j < ch.e; j += G) {
            const int cnt = (ch.e - j < G) ? (int)(ch.e - j) : G;
            const int64_t myrow = gl < cnt ? ld_stream_i64(seg_rows + j + gl) : 0;
            for (int k0 = 0; k0 < cnt; k0 += UN) {
                double y[UN][NV][VW];
#pragma unroll
                for (int u = 0; u < UN; u++) {
                    const int q = k0 + u;
                    const int64_t row = __shfl_sync(gmask, myrow, q < G ? q : G - 1, G);
                    if (q < cnt) {
#pragma unroll
                        for (int v = 0; v < NV; v++) ld_gather<VW>(y[u][v], H + row * ldh + (v * G + gl) * VW);
                    }
                }
                // in row order: the sums' order, and which of tied +0.0 / -0.0 a maximum keeps, depend on it only
#pragma unroll
                for (int u = 0; u < UN; u++)
                    if (k0 + u < cnt) {
#pragma unroll
                        for (int v = 0; v < NV; v++)
#pragma unroll
                            for (int w = 0; w < VW; w++) {
                                if constexpr (kMax)
                                    max_take(a[v][w], n[v][w], y[u][v][w]);
                                else
                                    a[v][w] += y[u][v][w];
                            }
                    }
            }
        }
        // a segment of one chunk writes P (and C); the chunks of a longer one their workspace rows [W | W + chunks ldw]
        double *po = ch.single ? P + ch.s * ldp : W + k * ldw;
        double *co = kMax ? (ch.single ? C + ch.s * ldc : W + (chunks + k) * ldw) : nullptr;
#pragma unroll
        for (int v = 0; v < NV; v++) {
            const int64_t col = (v * G + gl) * VW;
            st_rw<VW>(po + col, a[v]);
            if constexpr (kMax) st_rw<VW>(co + col, n[v]);
        }
    }
}

// ---- generic chunk kernel: a window of width f <= 32 kS, any leading dimension, any alignment; one warp per chunk ------
template <int kS, bool kMax>
__global__ void __launch_bounds__(kBlock, 1)
segment_pool_generic_kernel(const int64_t *__restrict__ seg_start, const int64_t *__restrict__ seg_rows,
                            const int64_t *__restrict__ chunk_first, const int32_t *__restrict__ chunk_seg, int64_t chunks,
                            const double *__restrict__ H, int64_t ldh, int f, double *__restrict__ P, int64_t ldp,
                            double *__restrict__ C, int64_t ldc, double *__restrict__ W, int64_t ldw) {
    const int lane = threadIdx.x & 31;
    const int64_t warps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t k = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; k < chunks; k += warps) {
        const Chunk ch = chunk_of(k, seg_start, chunk_first, chunk_seg);
        double a[kS], n[kS];
#pragma unroll
        for (int t = 0; t < kS; t++) {
            a[t] = kMax ? -INFINITY : 0.0;
            n[t] = 0.0;
        }
        for (int64_t j = ch.b; j < ch.e; j++) {
            const double *hr = H + seg_rows[j] * ldh;
#pragma unroll
            for (int t = 0; t < kS; t++) {
                const int c = lane + 32 * t;
                if (c < f) {
                    if constexpr (kMax)
                        max_take(a[t], n[t], hr[c]);
                    else
                        a[t] += hr[c];
                }
            }
        }
        double *po = ch.single ? P + ch.s * ldp : W + k * ldw;
        double *co = kMax ? (ch.single ? C + ch.s * ldc : W + (chunks + k) * ldw) : nullptr;
#pragma unroll
        for (int t = 0; t < kS; t++) {
            const int c = lane + 32 * t;
            if (c < f) {
                po[c] = a[t];
                if constexpr (kMax) co[c] = n[t];
            }
        }
    }
}

// ---- second stage: the segments of more than one chunk ------------------------------------------------------------------
// CTA item i = (segment i / slabs, columns 32 (i % slabs) ..): warp w combines chunks c0 + w, c0 + w + kMergeWarps, ..
// in order, lane l column l of the slab; then thread (0, l) combines the warps' results in warp order.
template <bool kMax>
__global__ void __launch_bounds__(kBlock)
segment_pool_merge_kernel(const int64_t *__restrict__ chunk_first, int64_t segments, int64_t chunks, int r,
                          const double *__restrict__ W, int64_t ldw, double *__restrict__ P, int64_t ldp, double *__restrict__ C,
                          int64_t ldc) {
    __shared__ double sa[kMergeWarps][32], sn[kMergeWarps][32];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int64_t slabs = (r + 31) / 32;
    for (int64_t i = blockIdx.x; i < segments * slabs; i += gridDim.x) {
        const int64_t s = i / slabs;
        const int64_t c0 = chunk_first[s], c1 = chunk_first[s + 1];
        if (c1 - c0 < 2) continue;  // the same on every thread of the CTA: no barrier is skipped by some only
        const int col = (int)(i % slabs) * 32 + lane;
        double a = kMax ? -INFINITY : 0.0, n = 0.0;
        if (col < r) {
            for (int64_t k = c0 + warp; k < c1; k += kMergeWarps) {
                const double x = W[k * ldw + col];
                if constexpr (kMax)
                    max_merge(a, n, x, W[(chunks + k) * ldw + col]);
                else
                    a += x;
            }
        }
        sa[warp][lane] = a;
        sn[warp][lane] = n;
        __syncthreads();
        if (warp == 0 && col < r) {
            double t = sa[0][lane], m = sn[0][lane];
            for (int w = 1; w < kMergeWarps; w++) {
                if constexpr (kMax)
                    max_merge(t, m, sa[w][lane], sn[w][lane]);
                else
                    t += sa[w][lane];
            }
            P[s * ldp + col] = t;
            if constexpr (kMax) C[s * ldc + col] = m;
        }
        __syncthreads();
    }
}

// ---- gradient ----------------------------------------------------------------------------------------------------------
// the gradient of one element: w dp (sum, mean), or [x == p] dp / c (max)
template <bool kMax>
__device__ __forceinline__ double pool_grad(double dp, double w, double x, double p, double c) {
    if constexpr (kMax)
        return x == p && c != 0.0 ? dp / c : 0.0;
    else
        return w * dp;
}

template <int R, int G, int VW, bool kMax>
__global__ void __launch_bounds__(kBlock, 1)
segment_pool_grad_kernel(const int32_t *__restrict__ row_graph, int64_t rows, int64_t graphs, const double *__restrict__ dP,
                         int64_t lddp, const double *__restrict__ scale, const double *__restrict__ H, int64_t ldh,
                         const double *__restrict__ P, int64_t ldp, const double *__restrict__ C, int64_t ldc,
                         double *__restrict__ dH, int64_t lddh) {
    constexpr int NV = R / (G * VW);
    static_assert(NV * G * VW == R, "R must equal NV*G*VW");
    const int gl = threadIdx.x & (G - 1);
    const int64_t ngroups = (int64_t)gridDim.x * (blockDim.x / G);
    for (int64_t u = (int64_t)blockIdx.x * (blockDim.x / G) + threadIdx.x / G; u < rows; u += ngroups) {
        const int64_t g = row_graph[u];
        const bool in = g >= 0 && g < graphs;
        const double w = in && scale ? scale[g] : 1.0;
#pragma unroll
        for (int v = 0; v < NV; v++) {
            const int64_t col = (v * G + gl) * VW;
            double o[VW] = {};
            if (in) {
                double dp[VW], x[VW] = {}, p[VW] = {}, c[VW] = {};
                ld_gather<VW>(dp, dP + g * lddp + col);
                if constexpr (kMax) {
                    ld_gather<VW>(x, H + u * ldh + col);
                    ld_gather<VW>(p, P + g * ldp + col);
                    ld_gather<VW>(c, C + g * ldc + col);
                }
#pragma unroll
                for (int q = 0; q < VW; q++) o[q] = pool_grad<kMax>(dp[q], w, x[q], p[q], c[q]);
            }
            st_rw<VW>(dH + u * lddh + col, o);
        }
    }
}

template <bool kMax>
__global__ void __launch_bounds__(kBlock, 1)
segment_pool_grad_generic_kernel(const int32_t *__restrict__ row_graph, int64_t rows, int64_t graphs, const double *__restrict__ dP,
                                 int64_t lddp, const double *__restrict__ scale, const double *__restrict__ H, int64_t ldh,
                                 const double *__restrict__ P, int64_t ldp, const double *__restrict__ C, int64_t ldc, int r,
                                 double *__restrict__ dH, int64_t lddh) {
    const int lane = threadIdx.x & 31;
    const int64_t warps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t u = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; u < rows; u += warps) {
        const int64_t g = row_graph[u];
        const bool in = g >= 0 && g < graphs;
        const double w = in && scale ? scale[g] : 1.0;
        for (int k = lane; k < r; k += 32) {
            double o = 0.0;
            if (in) {
                if constexpr (kMax)
                    o = pool_grad<true>(dP[g * lddp + k], 1.0, H[u * ldh + k], P[g * ldp + k], C[g * ldc + k]);
                else
                    o = pool_grad<false>(dP[g * lddp + k], w, 0.0, 0.0, 0.0);
            }
            dH[u * lddh + k] = o;
        }
    }
}

__global__ void __launch_bounds__(kBlock, 1)
max_count_merge_kernel(double *__restrict__ C, const double *__restrict__ local_max, const double *__restrict__ global_max, int64_t n) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride)
        if (local_max[i] != global_max[i]) C[i] = 0.0;
}

template <typename K>
K pick_generic(int f, K k1, K k2, K k4, K k8) {
    return f <= 32 ? k1 : f <= 64 ? k2 : f <= 128 ? k4 : k8;
}

template <bool kMax>
int pool_launch(const int64_t *seg_start, const int64_t *seg_rows, const int64_t *chunk_first, const int32_t *chunk_seg,
                int64_t segments, int64_t chunks, const double *H, int64_t ldh, int r, double *P, int64_t ldp, double *C, int64_t ldc,
                double *W, cudaStream_t st) {
    int rc = HNH_OK;
    for (int c0 = 0; c0 < r && rc == HNH_OK; c0 += kWindow) {
        const int w = std::min(kWindow, r - c0);
        const double *Hw = H + c0;
        double *Pw = P + c0, *Cw = kMax ? C + c0 : nullptr, *Ww = W ? W + c0 : nullptr;
        int grid = 0;
        if (table_width(w) && aligned16(Hw) && aligned16(Pw) && ldh % 2 == 0 && ldp % 2 == 0 && r % 2 == 0 && (!Ww || aligned16(Ww)) &&
            (!kMax || (aligned16(Cw) && ldc % 2 == 0))) {
#define SP(RR, G, VW, UN)                                                                                                  \
    {                                                                                                                      \
        auto k = segment_pool_kernel<RR, G, VW, UN, kMax>;                                                                 \
        rc = grid_for(k, chunks, kBlock / G, &grid);                                                                       \
        if (!rc)                                                                                                           \
            rc = launch(k, grid, kBlock, st, "segment_pool_kernel", seg_start, seg_rows, chunk_first, chunk_seg, chunks, Hw, ldh, Pw, \
                        ldp, Cw, ldc, Ww, (int64_t)r);                                                                     \
    }
            HNH_DISPATCH_R(w, SP, )
#undef SP
            continue;
        }
        auto k = pick_generic(w, segment_pool_generic_kernel<1, kMax>, segment_pool_generic_kernel<2, kMax>,
                              segment_pool_generic_kernel<4, kMax>, segment_pool_generic_kernel<8, kMax>);
        rc = grid_for(k, chunks, kBlock / 32, &grid);
        if (!rc)
            rc = launch(k, grid, kBlock, st, "segment_pool_generic_kernel", seg_start, seg_rows, chunk_first, chunk_seg, chunks, Hw, ldh,
                        w, Pw, ldp, Cw, ldc, Ww, (int64_t)r);
    }
    if (rc || chunks == segments) return rc;  // every segment one chunk: nothing to merge
    auto k = segment_pool_merge_kernel<kMax>;
    int grid = 0;
    rc = grid_for(k, segments * ((r + 31) / 32), 1, &grid);
    return rc ? rc : launch(k, grid, kBlock, st, "segment_pool_merge_kernel", chunk_first, segments, chunks, r, (const double *)W,
                            (int64_t)r, P, ldp, C, ldc);
}

template <bool kMax>
int grad_launch(const int32_t *row_graph, int64_t rows, int64_t graphs, const double *dP, int64_t lddp, const double *scale,
                const double *H, int64_t ldh, const double *P, int64_t ldp, const double *C, int64_t ldc, int r, double *dH,
                int64_t lddh, cudaStream_t st) {
    int grid = 0, rc = HNH_OK;
    if (table_width(r) && aligned16(dP) && aligned16(dH) && lddp % 2 == 0 && lddh % 2 == 0 &&
        (!kMax || (aligned16(H) && aligned16(P) && aligned16(C) && ldh % 2 == 0 && ldp % 2 == 0 && ldc % 2 == 0))) {
#define SG(RR, G, VW, UN)                                                                                                  \
    {                                                                                                                      \
        auto k = segment_pool_grad_kernel<RR, G, VW, kMax>;                                                                \
        rc = grid_for(k, rows, kBlock / G, &grid);                                                                         \
        if (!rc)                                                                                                           \
            rc = launch(k, grid, kBlock, st, "segment_pool_grad_kernel", row_graph, rows, graphs, dP, lddp, scale, H, ldh, P, ldp, C, \
                        ldc, dH, lddh);                                                                                    \
    }
        HNH_DISPATCH_R(r, SG, )
#undef SG
        return rc;
    }
    auto k = segment_pool_grad_generic_kernel<kMax>;
    rc = grid_for(k, rows, kBlock / 32, &grid);
    return rc ? rc
              : launch(k, grid, kBlock, st, "segment_pool_grad_generic_kernel", row_graph, rows, graphs, dP, lddp, scale, H, ldh, P, ldp,
                       C, ldc, r, dH, lddh);
}

}  // namespace

extern "C" {

int64_t hnh_segment_pool_workspace_bytes(int64_t chunks, int r, int with_counts) {
    if (chunks < 0 || r < 1) return set_error(HNH_E_INVALID, "hnh_segment_pool_workspace_bytes: bad size");
    return chunks * (int64_t)r * (with_counts ? 2 : 1) * (int64_t)sizeof(double);
}

int hnh_segment_pool_f64(const int64_t *seg_start, const int64_t *seg_rows, const int64_t *chunk_first, const int32_t *chunk_seg,
                         int64_t segments, int64_t chunks, const double *H, int64_t ldh, int r, double *P, int64_t ldp, double *C,
                         int64_t ldc, void *workspace, size_t workspace_bytes, void *stream) {
    const char *who = "hnh_segment_pool_f64";
    if (segments < 0 || chunks < segments) return set_error(HNH_E_INVALID, "%s: bad segment or chunk count", who);
    if (r < 1) return set_error(HNH_E_INVALID, "%s: r must be positive (got %d)", who, r);
    if (ldh < r || ldp < r || (C && ldc < r)) return set_error(HNH_E_INVALID, "%s: a leading dimension is below r = %d", who, r);
    if (segments == 0) return HNH_OK;
    // seg_rows may be null when no segment has a row: it is then never read
    if (!seg_start || !chunk_first || !chunk_seg || !H || !P) return set_error(HNH_E_INVALID, "%s: null pointer", who);
    if (P == H || C == H) return set_error(HNH_E_INVALID, "%s: an output may not be the input", who);
    if (C == P) return set_error(HNH_E_INVALID, "%s: P and C must be distinct", who);
    const int64_t need = hnh_segment_pool_workspace_bytes(chunks, r, C != nullptr);
    if (chunks > segments && (!workspace || workspace_bytes < (size_t)need))
        return set_error(HNH_E_INVALID, "%s: the workspace must hold %lld bytes", who, (long long)need);
    cudaStream_t st = (cudaStream_t)stream;
    double *W = (double *)workspace;
    return C ? pool_launch<true>(seg_start, seg_rows, chunk_first, chunk_seg, segments, chunks, H, ldh, r, P, ldp, C, ldc, W, st)
             : pool_launch<false>(seg_start, seg_rows, chunk_first, chunk_seg, segments, chunks, H, ldh, r, P, ldp, nullptr, r, W, st);
}

int hnh_segment_max_count_merge_f64(double *C, const double *local_max, const double *global_max, int64_t n, void *stream) {
    const char *who = "hnh_segment_max_count_merge_f64";
    if (n < 0) return set_error(HNH_E_INVALID, "%s: negative size", who);
    if (n == 0) return HNH_OK;
    if (!C || !local_max || !global_max) return set_error(HNH_E_INVALID, "%s: null pointer", who);
    if (C == local_max || C == global_max) return set_error(HNH_E_INVALID, "%s: C may not be a maximum", who);
    int grid = 0;
    int rc = grid_for(max_count_merge_kernel, n, kBlock * 4, &grid);
    return rc ? rc : launch(max_count_merge_kernel, grid, kBlock, (cudaStream_t)stream, "max_count_merge_kernel", C, local_max, global_max, n);
}

int hnh_segment_pool_grad_f64(const int32_t *row_graph, int64_t rows, int64_t graphs, const double *dP, int64_t lddp,
                              const double *scale, const double *H, int64_t ldh, const double *P, int64_t ldp, const double *C,
                              int64_t ldc, int r, double *dH, int64_t lddh, void *stream) {
    const char *who = "hnh_segment_pool_grad_f64";
    if (rows < 0 || graphs < 0) return set_error(HNH_E_INVALID, "%s: negative size", who);
    if (r < 1) return set_error(HNH_E_INVALID, "%s: r must be positive (got %d)", who, r);
    const bool mx = H || P || C;
    if (mx && (!H || !P || !C)) return set_error(HNH_E_INVALID, "%s: max takes H, P and C together", who);
    if (mx && scale) return set_error(HNH_E_INVALID, "%s: max takes no scale", who);
    if (lddp < r || lddh < r || (mx && (ldh < r || ldp < r || ldc < r)))
        return set_error(HNH_E_INVALID, "%s: a leading dimension is below r = %d", who, r);
    if (rows == 0) return HNH_OK;
    if (!row_graph || !dH || (graphs > 0 && !dP)) return set_error(HNH_E_INVALID, "%s: null pointer", who);
    const void *ins[] = {dP, scale, H, P, C, row_graph};
    for (const void *i : ins)
        if (i && i == dH) return set_error(HNH_E_INVALID, "%s: dH may not be an input", who);
    cudaStream_t st = (cudaStream_t)stream;
    return mx ? grad_launch<true>(row_graph, rows, graphs, dP, lddp, nullptr, H, ldh, P, ldp, C, ldc, r, dH, lddh, st)
              : grad_launch<false>(row_graph, rows, graphs, dP, lddp, scale, nullptr, r, nullptr, r, nullptr, r, r, dH, lddh, st);
}

}  // extern "C"
