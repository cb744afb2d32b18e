/*
 * hnh_b200.h -- C ABI of the H100-native local kernels (libhnh_b200.so).
 *
 * This is the drop-in boundary under the reference's C++ plugin interface
 * `KernelImplementation` (reference sparse_kernels.h:15-79).  Every entry point is
 * `extern "C"`, takes plain pointers and sizes (no torch / Eigen / MKL types), enqueues
 * its work on the CUDA stream passed as `void *stream` (NULL = legacy default stream) and
 * returns 0 on success or a negative HNH_E_* code -- it never prints-and-exits the way the
 * reference does (sparse_kernels.cpp:75-83).  `hnh_last_error_string()` describes the last
 * failure on the calling thread.
 *
 * Unless a name ends in `_host`, all data pointers are DEVICE pointers.
 * Dense operands are row-major, contiguous, leading dimension = r (reference common.h:13,
 * `DenseMatrix`), fp64.  Index arrays are int64 (MKL_INT under -DMKL_ILP64, reference
 * CMakeLists.txt:37).  CSR arrays are the four vectors of the reference's `CSRHandle`
 * (SpmatLocal.hpp:55-62): values, col_idx, rowStart (rows+1 entries), row_idx (expanded).
 *
 * There is no CPU fallback behind this ABI: without a CUDA device every compute entry
 * point fails with HNH_E_CUDA.
 */
#ifndef HNH_B200_H
#define HNH_B200_H

#include <stdint.h>
#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

#define HNH_OK 0
#define HNH_E_INVALID (-1) /* bad argument (null pointer, negative size, r <= 0 ...)     */
#define HNH_E_CUDA (-2)    /* a CUDA runtime call or kernel launch failed                */
#define HNH_E_MODE (-3)    /* block transposition does not match the requested SpMM mode */
#define HNH_E_ALLOC (-4)   /* device or pinned-host allocation failed                    */
#define HNH_E_COMM (-5)    /* NCCL / transport failure                                   */

/* flags (bit set) */
#define HNH_FLAG_DEFAULT 0
#define HNH_FLAG_FORCE_GENERIC 1 /* use the any-r scalar kernel (testing)                  */
#define HNH_FLAG_FORCE_DIRECT 2  /* use the direct-load row kernels instead of TMA-staged */
/* BETA0: overwrite instead of accumulate -- sddmm: values = dot; spmm: Y = CSR*X;
 * fused: values = dot, Out = result (Out may then alias X).  Equivalent to zeroing the
 * output first (setValuesConstant(0) / setZero(), SpmatLocal.hpp:595-605,
 * distributed_sparse.h:275) but without the extra pass over memory. */
#define HNH_FLAG_BETA0 4
/* fused only: overwrite just the values (each block is visited once per FusedMM) or just Out */
#define HNH_FLAG_BETA0_VALUES 16
#define HNH_FLAG_BETA0_OUT 32
/* sddmm / fused, r in {128, 256}: stage the row-side factor tile with bulk asynchronous copies
 * (cp.async.bulk + mbarrier, SASS UBLKCP) instead of direct loads.  Without this flag the library picks
 * per kernel from measurements (TMA for SDDMM and for the r = 256 overwrite-fused kernel; direct loads
 * otherwise); HNH_FLAG_FORCE_DIRECT or env HNH_TMA=0 force the direct-load kernels, HNH_TMA=1 the
 * TMA-staged ones. */
#define HNH_FLAG_TMA_STAGE 64
/* experimental: per-warp TMA slots (no block barrier); never selected automatically */
#define HNH_FLAG_TMA_WARP 128
/* hnh_sddmm_scaled_f64 with scaled_out: the block's values receive scale * dot as well (default: the plain dot) */
#define HNH_FLAG_SCALE_VALUES 256

/* ABI / build identification. */
int hnh_abi_version(void);
const char *hnh_build_info(void);
const char *hnh_last_error_string(void);
/* Number of kernel launches issued through this library by the calling process so far
 * (bench.py reports the delta over its timed region as `gpu_launches`). */
uint64_t hnh_launch_count(void);

/* ---- K1: SDDMM -- replaces StandardKernel::sddmm_local (sparse_kernels.cpp:13-57) ------
 * values[i] += sum_k X[row(i), k] * Y[col_idx[i], k]   for every nonzero i of the block.
 * (X, Y) are already role-resolved: (A, B) for a non-transposed block, (B, A) for a
 * transposed one (sparse_kernels.cpp:29-38).  `rows` = number of CSR rows of the block,
 * rowStart[rows] == nnz.  Accumulates (+=), exactly like the reference; callers zero
 * `values` first (SpmatLocal::setValuesConstant, SpmatLocal.hpp:595-605).
 * nnz == 0 or rows == 0 is a successful no-op (sparse_kernels.cpp:25-27). */
int hnh_sddmm_f64(const int64_t *rowStart, const int64_t *col_idx, double *values,
                  int64_t rows, int64_t nnz, const double *X, const double *Y, int r,
                  int flags, void *stream);
/* The same with the Hadamard epilogue of the reference's `SValues.cwiseProduct(getCSRValues())`
 * (15D_dense_shift.hpp:364-368, SpmatLocal.hpp:571-593) folded in: `scale` is aligned with `values`
 * (scale[i] belongs to nonzero i of this block).  scaled_out != NULL: values[i] = dot (as above) and
 * scaled_out[i] = scale[i] * dot.  scaled_out == NULL: values[i] = scale[i] * dot.  scale == NULL is
 * hnh_sddmm_f64.  HNH_FLAG_SCALE_VALUES: with scaled_out, values[i] = scale[i] * dot too.  With accumulation
 * (no BETA0) the old value is added to the dot BEFORE scaling. */
int hnh_sddmm_scaled_f64(const int64_t *rowStart, const int64_t *col_idx, double *values, int64_t rows,
                         int64_t nnz, const double *X, const double *Y, int r, int flags, const double *scale,
                         double *scaled_out, void *stream);

/* Same operation driven by the expanded COO arrays the reference kernel actually reads
 * (`row_idx[i]`, `col_idx[i]`, sparse_kernels.cpp:45-47); needs no rowStart. */
int hnh_sddmm_coo_f64(const int64_t *row_idx, const int64_t *col_idx, double *values,
                      int64_t nnz, const double *X, const double *Y, int r, int flags,
                      void *stream);

/* ---- K2: SpMM -- replaces StandardKernel::spmm_local (sparse_kernels.cpp:59-127) -------
 * Y[rows x r] += CSR[rows x *] * X   (alpha = beta = 1, row-major, ld = r: the
 * mkl_sparse_d_mm call at sparse_kernels.cpp:95-120).  X is gathered by col_idx.  The
 * kernel never bounds-checks col_idx against a column count (the reference declares too few
 * columns in 15D_sparse_shift.hpp:132). */
int hnh_spmm_f64(const int64_t *rowStart, const int64_t *col_idx, const double *values,
                 int64_t rows, int64_t nnz, const double *X, double *Y, int r, int flags,
                 void *stream);

/* ---- K3: fused SDDMM -> SpMM on one block ------------------------------------------------
 * Replaces the two back-to-back triple_function calls of the fusion-2 loop body
 * (15D_dense_shift.hpp:203-217):  values[i] += X[row(i)] . Y[col(i)];  then
 * Out[row] += sum_{i in row} values[i] * Y[col(i)]   -- with ONE gather of each Y row. */
int hnh_fused_f64(const int64_t *rowStart, const int64_t *col_idx, double *values,
                  int64_t rows, int64_t nnz, const double *X, const double *Y, double *Out,
                  int r, int flags, void *stream);
/* The same with the caller's S values folded in (the Hadamard product the reference applies between its SDDMM and
 * SpMM passes, distributed_sparse.h:289-312): values[i] = scale[i] * dot, Out += sum_i values[i] * Y[col_i], and
 * scaled_out[i] (optional) = values[i] -- the user-visible SDDMM result.  Needs HNH_FLAG_BETA0_VALUES, a table width
 * and aligned operands (HNH_E_INVALID otherwise: use the separate calls). */
int hnh_fused_scaled_f64(const int64_t *rowStart, const int64_t *col_idx, double *values, int64_t rows,
                         int64_t nnz, const double *X, const double *Y, double *Out, int r, int flags,
                         const double *scale, double *scaled_out, void *stream);

/* ---- K4: value plumbing (SpmatLocal.hpp:571-605, 15D_dense_shift.hpp:366) -------------- */
int hnh_fill_f64(double *dst, int64_t n, double value, void *stream);
/* dst[i] = uniform(-1,1) from a counter-based hash of (seed, i) -- DenseMatrix::setRandom
 * (als_conjugate_gradients.cpp:143-146) */
int hnh_random_uniform_f64(double *dst, int64_t n, uint64_t seed, void *stream);
/* dst[i] = a[i] * b[i]  (VectorXd::cwiseProduct of SValues and getCSRValues()) */
int hnh_hadamard_f64(double *dst, const double *a, const double *b, int64_t n, void *stream);
/* row_idx[i] = CSR row of nonzero i (SpmatLocal.hpp:139-147,160-163) */
int hnh_expand_row_idx(const int64_t *rowStart, int64_t rows, int64_t nnz, int64_t *row_idx,
                       void *stream);

/* ---- dense row algebra used between fusedSpMM calls by the ALS-CG caller
 *      (als_conjugate_gradients.cpp:9-29,99-138) ------------------------------------------ */
/* out[i] = sum_k A[i,k] * B[i,k]   (batch_dot_product) */
int hnh_batch_dot_f64(double *out, const double *A, const double *B, int64_t rows, int r,
                      void *stream);
/* D[i,k] = C[i,k] + alpha * s[i] * M[i,k]   (X += scale_matrix_rows(s, M) and friends;
 * s may be NULL meaning all-ones; C may be NULL meaning zero; D may alias C or M) */
int hnh_row_axpy_f64(double *D, const double *C, double alpha, const double *s,
                     const double *M, int64_t rows, int r, void *stream);
/* elementwise vector helpers: out = (a + ca) / (b + cb); b == NULL: out = a + ca */
int hnh_vec_quotient_f64(double *out, const double *a, double ca, const double *b, double cb,
                         int64_t n, void *stream);
/* dst = alpha * x + beta * y elementwise (y may be NULL when beta == 0) */
int hnh_axpby_f64(double *dst, double alpha, const double *x, double beta, const double *y,
                  int64_t n, void *stream);
/* *out (device scalar) = sum x[i]^2 */
int hnh_squared_norm_f64(double *out, const double *x, int64_t n, void *stream);

/* ---- GAT forward pass helpers (reference gat.hpp:84-113; include/hnh/gat.hpp) --------------
 * dst[i] = max(src[i], 0) + alpha * min(src[i], 0)   (gat.hpp:98; dst may alias src) */
int hnh_leaky_relu_f64(double *dst, const double *src, int64_t n, double alpha, void *stream);
/* dst[i, col0 + j] = max(src[i, j], 0) for a rows x cols src and a dst with ld_dst columns
 * (buffers[i+1].middleCols(j * w, w) = A.array().max(0), gat.hpp:104) */
int hnh_relu_cols_f64(double *dst, int64_t ld_dst, int64_t col0, const double *src, int64_t rows,
                      int64_t cols, void *stream);
/* C (m x n) = A (m x k) * B (k x n), all row-major and contiguous (buffers[i] * wMats[j],
 * gat.hpp:90).  This library's own kernel: fp64 tensor-core MMA (mma.sync m8n8k4) over shared-memory tiles. */
int hnh_dgemm_f64(double *C, const double *A, const double *B, int64_t m, int64_t n, int64_t k,
                  void *stream);

/* ---- GAT backward pass helpers (include/hnh/gat.hpp, GAT::backwardPass) ----------------------
 * dst[i] = src[i] > 0 ? 1 : alpha   (derivative of hnh_leaky_relu_f64; alpha at 0; dst may alias src) */
int hnh_leaky_relu_grad_f64(double *dst, const double *src, int64_t n, double alpha, void *stream);
/* dst[i, j] = out[i, col0 + j] > 0 ? grad[i, col0 + j] : 0 for a rows x cols contiguous dst; grad and out
 * have ld columns (the gradient through hnh_relu_cols_f64; 0 at 0) */
int hnh_relu_cols_backward_f64(double *dst, const double *grad, const double *out, int64_t ld, int64_t col0,
                               int64_t rows, int64_t cols, void *stream);
/* C (m x n) = A^T * B with A k x m and B k x n, all row-major and contiguous (the weight gradient X^T dP).
 * fp64 tensor-core MMA; k is split over the CTAs and the partial tiles go to `workspace`, which must hold
 * hnh_dgemm_tn_workspace_bytes(m, n, k) bytes (0: none needed); a second pass adds them in a fixed order, so
 * repeated calls give bit-identical results.  m, n <= 2^20.  The workspace size depends on the shape only;
 * it is negative (HNH_E_INVALID) for a bad shape. */
int64_t hnh_dgemm_tn_workspace_bytes(int64_t m, int64_t n, int64_t k);
int hnh_dgemm_tn_f64(double *C, const double *A, const double *B, int64_t m, int64_t n, int64_t k,
                     void *workspace, size_t workspace_bytes, void *stream);
/* C (m x n) = A * B^T (accumulate == 0) or C += A * B^T (accumulate != 0), with A m x k and B n x k, all
 * row-major and contiguous (the input gradient dP W^T).  fp64 tensor-core MMA, the tiling of hnh_dgemm_f64. */
int hnh_dgemm_nt_f64(double *C, const double *A, const double *B, int64_t m, int64_t n, int64_t k,
                     int accumulate, void *stream);

/* ---- edge softmax: a softmax over the entries of each row (Distributed_Sparse::edgeSoftmax) ----------
 * x is a value vector of n entries; keys[i] in [0, num_rows) is the row of entry i.  A plan groups the
 * entries by row: perm (n) lists them by ascending key, stably; row u's entries are
 * perm[row_start[u] .. row_start[u + 1]); each row is cut into pieces of at most 1024 entries, the pieces of
 * row u are piece_first[u] .. piece_first[u + 1] - 1 and piece_row[q] is the row of piece q.  Reductions
 * run one warp per piece, then one warp per row, in an order fixed by the plan: no floating-point atomics,
 * repeated calls give bit-identical results.  Empty input is a no-op.
 *
 * keys[i] = (int32) (idx[i] + offset): the global row of the entries of one CSR block from its stored row or
 * column index */
#define HNH_EDGE_PIECE 1024 /* the most entries of one piece */
int hnh_edge_keys_from_index(int32_t *keys, const int64_t *idx, int64_t n, int64_t offset, void *stream);
/* out[i] = (double) (idx[i] + offset): the same as doubles, exact below 2^53 (Distributed_Sparse::entryCoordinates) */
int hnh_entry_coords_from_index_f64(double *out, const int64_t *idx, int64_t n, int64_t offset, void *stream);
/* room for piece_row that any plan of n entries over num_rows rows fits in (negative: bad size) */
int64_t hnh_edge_softmax_piece_bound(int64_t n, int64_t num_rows);
/* Builds the plan of `keys` (synchronises): perm (n), row_start and piece_first (num_rows + 1 each),
 * piece_row (piece_capacity); *num_pieces receives the piece count.  n and num_rows below 2^31 - 1;
 * HNH_E_INVALID when a key lies outside [0, num_rows). */
int hnh_edge_softmax_plan(const int32_t *keys, int64_t n, int64_t num_rows, int32_t *perm, int32_t *row_start,
                          int32_t *piece_first, int32_t *piece_row, int64_t piece_capacity, int64_t *num_pieces,
                          void *stream);
/* row_max[u] = max of x over row u, row_sum[u] = sum of exp(x - row_max[u]) over row u, for every row
 * (-inf and 0 for a row without entries).  A -inf entry (a masked edge) adds nothing to row_sum, so the
 * apply step gives it alpha = 0; a row whose entries are all -inf gets (-inf, 0) like an empty row, and
 * the apply step gives its entries NaN, as torch.softmax does.  piece_max / piece_sum: num_pieces doubles
 * of workspace. */
int hnh_edge_softmax_stats_f64(const double *x, const int32_t *perm, const int32_t *row_start,
                               const int32_t *piece_first, const int32_t *piece_row, int64_t num_rows,
                               int64_t num_pieces, double *piece_max, double *piece_sum, double *row_max,
                               double *row_sum, void *stream);
/* row_sum[u] *= exp(local_max[u] - global_max[u]) (0 where local_max[u] = -inf): a sum made relative to
 * this rank's row maximum, made relative to the maximum over all ranks */
int hnh_edge_softmax_rescale_f64(double *row_sum, const double *local_max, const double *global_max,
                                 int64_t num_rows, void *stream);
/* alpha[i] = exp(x[i] - row_max[keys[i]]) / row_sum[keys[i]]   (alpha may alias x) */
int hnh_edge_softmax_apply_f64(double *alpha, const double *x, const int32_t *keys, int64_t n,
                               const double *row_max, const double *row_sum, void *stream);
/* row_dot[u] = sum over row u of alpha[i] * grad[i] (0 for a row without entries); piece_dot: num_pieces
 * doubles of workspace */
int hnh_edge_softmax_dot_f64(const double *alpha, const double *grad, const int32_t *perm, const int32_t *row_start,
                             const int32_t *piece_first, const int32_t *piece_row, int64_t num_rows,
                             int64_t num_pieces, double *piece_dot, double *row_dot, void *stream);
/* dx[i] = alpha[i] * (grad[i] - row_dot[keys[i]])   (dx may alias grad) */
int hnh_edge_softmax_backward_f64(double *dx, const double *alpha, const double *grad, const int32_t *keys,
                                  int64_t n, const double *row_dot, void *stream);
/* row_sum[u] = sum over row u of x[i] (0 for a row without entries), in the order of hnh_edge_softmax_dot_f64;
 * piece_sum: num_pieces doubles of workspace.  With a plan keyed by column, the column sums. */
int hnh_edge_sum_f64(const double *x, const int32_t *perm, const int32_t *row_start, const int32_t *piece_first,
                     const int32_t *piece_row, int64_t num_rows, int64_t num_pieces, double *piece_sum,
                     double *row_sum, void *stream);

/* ---- additive graph attention (GAT::set_attention("additive"); csrc/gat_additive.cu) ------------------
 * s[i] = sum_k P[i, k] a1[k] and t[i] = sum_k P[i, k] a2[k] for a row-major n x d P, in one read of P; the
 * summation order is fixed (repeated calls are bit-identical) */
int hnh_gat_node_scalars_f64(double *s, double *t, const double *P, const double *a1, const double *a2, int64_t n,
                             int64_t d, void *stream);
/* out[k] = LeakyReLU(s[row_key[k]] + t[col_key[k]]) (hnh_leaky_relu_f64's formula), or, derivative != 0, its
 * derivative: 1 where s + t > 0, alpha elsewhere (hnh_leaky_relu_grad_f64's convention).  Elementwise in the order
 * of the keys. */
int hnh_gat_edge_scores_f64(double *out, const double *s, const double *t, const int32_t *row_key,
                            const int32_t *col_key, int64_t n, double alpha, int derivative, void *stream);
/* dP[i, :] += ds[i] * a1 + dt[i] * a2 for a row-major n x d dP (the backward's rank-2 row update) */
int hnh_gat_rank2_update_f64(double *dP, const double *ds, const double *dt, const double *a1, const double *a2,
                             int64_t n, int64_t d, void *stream);

/* ---- GATv2 attention (GAT::set_attention("gatv2"); csrc/gatv2.cu) ----------------------------------------
 * One CSR block (rowStart: rows + 1 offsets from 0, col_idx: nnz column indices).  The "row side" R is the
 * dense operand indexed by the stored row, the "gathered side" Y the one indexed by col_idx; both are row-major
 * r-wide rows with their own leading dimensions (ldr, ldy >= r), so either may be the left or right half of a
 * 2r-wide matrix.  sigma(z) = LeakyReLU(z) = z > 0 ? z : alpha z, sigma'(z) = z > 0 ? 1 : alpha
 * (hnh_leaky_relu_grad_f64's convention); a holds r doubles.  The formulas are symmetric in R and Y.  No
 * floating-point atomics: repeated calls give bit-identical results.  Empty input is a no-op.
 *
 * out[i] = sum_k a[k] sigma(R[row(i), k] + Y[col_idx[i], k]) for every entry i (overwritten, not accumulated) */
int hnh_gatv2_scores_f64(const int64_t *rowStart, const int64_t *col_idx, int64_t rows, int64_t nnz,
                         const double *R, int64_t ldr, const double *Y, int64_t ldy, const double *a, int r,
                         double alpha, double *out, void *stream);
/* dR[row, :] += a o sum_{i in row} g[i] sigma'(R[row] + Y[col_idx[i]]) (dR: leading dimension lddr >= r; it
 * may share rows with R, e.g. R = Q and dR = Q + r for Q = [R | dR] with ldr = lddr = 2r).  With da != NULL,
 * also da[k] += sum_i g[i] sigma(R[row(i), k] + Y[col_idx[i], k]): per-CTA partials go to `workspace`, of at
 * least hnh_gatv2_grad_workspace_bytes(rows, r) bytes, and a second kernel adds them in a fixed order. */
int64_t hnh_gatv2_grad_workspace_bytes(int64_t rows, int r);
int hnh_gatv2_grad_f64(const int64_t *rowStart, const int64_t *col_idx, const double *g, int64_t rows, int64_t nnz,
                       const double *R, int64_t ldr, const double *Y, int64_t ldy, const double *a, int r,
                       double alpha, double *dR, int64_t lddr, double *da, void *workspace, size_t workspace_bytes,
                       void *stream);

/* ---- fused sparse attention (Distributed_Sparse::sparseAttention; csrc/sparse_attention.cu) ---------------
 * One CSR block (rowStart, col_idx as above) with stored row u and gathered row v = col_idx[i].  Every dense
 * operand is a pointer plus its own leading dimension: d-wide rows (ld >= d) or one scalar per row (ld >= 1,
 * e.g. column h of a rows x H matrix is L + h with ld = H), so head windows of an H*d-wide matrix and packed
 * matrices are views.  x_uv = scale <Q_u, K_v>; scale must be finite.  No floating-point atomics: repeated
 * calls give bit-identical results.  No rows or no entries: a no-op.
 *
 * step: continues the online softmax of every stored row over the block's entries (a row whose entries lie in
 * several blocks is carried from call to call):
 *     m' = max(m, max_i x_i),  s' = e^(m - m') s + sum_i e^(x_i - m'),  acc' = e^(m - m') acc + sum_i e^(x_i - m') V_v
 * Start from acc = 0, s = 0 (m = -inf; m is not read while s = 0).  Rows without entries are not touched. */
int hnh_sparse_attention_step_f64(const int64_t *rowStart, const int64_t *col_idx, int64_t rows, int64_t nnz, int d,
                                  const double *Q, int64_t ldq, const double *K, int64_t ldk, const double *V,
                                  int64_t ldv, double scale, double *acc, int64_t ldacc, double *m, int64_t ldm,
                                  double *s, int64_t lds, void *stream);
/* finish: Z = acc / s and L = m + log s per row; Z = 0 and L = -inf where s = 0.  In place allowed: Z may be acc
 * and L may be m (same pointer and leading dimension). */
int hnh_sparse_attention_finish_f64(int64_t rows, int d, const double *acc, int64_t ldacc, const double *m,
                                    int64_t ldm, const double *s, int64_t lds, double *Z, int64_t ldz, double *L,
                                    int64_t ldl, void *stream);
/* Backward, with L the finished log-sum-exp and t_u = <dZ_u, Z_u>; alpha_uv = exp(x_uv - L_u) and
 * dx_uv = alpha_uv (<dZ_u, V_v> - t_u).
 * grad_q (stored rows are query rows u): dQ_u += scale sum_v dx_uv K_v.
 * grad_kv (stored rows are key rows v; L and t gathered by col_idx): dK_v += scale sum_u dx_uv Q_u and
 * dV_v += sum_u alpha_uv dZ_u. */
int hnh_sparse_attention_grad_q_f64(const int64_t *rowStart, const int64_t *col_idx, int64_t rows, int64_t nnz, int d,
                                    const double *Q, int64_t ldq, const double *dZ, int64_t lddz, const double *L,
                                    int64_t ldl, const double *t, int64_t ldt, const double *K, int64_t ldk,
                                    const double *V, int64_t ldv, double scale, double *dQ, int64_t lddq, void *stream);
int hnh_sparse_attention_grad_kv_f64(const int64_t *rowStart, const int64_t *col_idx, int64_t rows, int64_t nnz, int d,
                                     const double *K, int64_t ldk, const double *V, int64_t ldv, const double *Q,
                                     int64_t ldq, const double *dZ, int64_t lddz, const double *L, int64_t ldl,
                                     const double *t, int64_t ldt, double scale, double *dK, int64_t lddk, double *dV,
                                     int64_t lddv, void *stream);
/* Attention dropout: the same three calls with (p, seed, u0, v0) before the stream.  Entry (u, v) has the global
 * query row u and key row v: step and grad_q, u = u0 + stored row, v = v0 + col_idx[i]; grad_kv, u = u0 + col_idx[i],
 * v = v0 + stored row; u and v below 2^32.  Its keep bit is
 *     D_uv = (uint32_t)(mix64(mix64(seed) ^ ((uint64_t)u << 32 | (uint64_t)v)) >> 32) >= T,
 *     T = min(ceil(p 2^32), 2^32 - 1),
 * with mix64 the splitmix64 finaliser: z += 0x9E3779B97F4A7C15; z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9;
 * z = (z ^ (z >> 27)) * 0x94D049BB133111EB; return z ^ (z >> 31).  So p = 0 keeps every entry, the keep probability
 * is exactly 1 - T / 2^32, and the mask is a function of (seed, u, v) alone: not of an entry's position, its block
 * or the call, so the three passes see the same mask, and stored duplicates of one (u, v) share one bit.
 * Distributed_Sparse::sparseAttention passes seed + h for head h.  With w = 1 / (1 - p):
 * step: s' as above (every entry counts, so L stays the log-sum-exp of all scores), and
 *     acc' = e^(m - m') acc + sum_i D_i w e^(x_i - m') V_v   (finish is unchanged: Z = sum_v D_uv w alpha_uv V_v);
 * grad_q, grad_kv: dx_uv = alpha_uv (D_uv w <dZ_u, V_v> - t_u), and dV_v += sum_u D_uv w alpha_uv dZ_u.
 * p < 0, p >= 1, NaN, u0 < 0 or v0 < 0: HNH_E_INVALID before any launch.  At p = 0 the results are bit-identical
 * to the calls without dropout. */
int hnh_sparse_attention_step_dropout_f64(const int64_t *rowStart, const int64_t *col_idx, int64_t rows, int64_t nnz,
                                          int d, const double *Q, int64_t ldq, const double *K, int64_t ldk,
                                          const double *V, int64_t ldv, double scale, double *acc, int64_t ldacc,
                                          double *m, int64_t ldm, double *s, int64_t lds, double p, uint64_t seed,
                                          int64_t u0, int64_t v0, void *stream);
int hnh_sparse_attention_grad_q_dropout_f64(const int64_t *rowStart, const int64_t *col_idx, int64_t rows,
                                            int64_t nnz, int d, const double *Q, int64_t ldq, const double *dZ,
                                            int64_t lddz, const double *L, int64_t ldl, const double *t, int64_t ldt,
                                            const double *K, int64_t ldk, const double *V, int64_t ldv, double scale,
                                            double *dQ, int64_t lddq, double p, uint64_t seed, int64_t u0, int64_t v0,
                                            void *stream);
int hnh_sparse_attention_grad_kv_dropout_f64(const int64_t *rowStart, const int64_t *col_idx, int64_t rows,
                                             int64_t nnz, int d, const double *K, int64_t ldk, const double *V,
                                             int64_t ldv, const double *Q, int64_t ldq, const double *dZ, int64_t lddz,
                                             const double *L, int64_t ldl, const double *t, int64_t ldt, double scale,
                                             double *dK, int64_t lddk, double *dV, int64_t lddv, double p,
                                             uint64_t seed, int64_t u0, int64_t v0, void *stream);
/* Additive score bias: the dropout calls with `bias` (and, for the gradients, `dbias`) before the stream; p = 0
 * means no dropout.  bias is block-local: entry i (the i-th stored entry, in col_idx order) reads bias[i], and
 *     x_i = scale <Q_u, K_v> + bias[i]      (the bias is added after the scale and is not scaled).
 * The step, finish, L, t and the dropout mask are those above on these scores; the gradients keep their formulas
 * with alpha computed from the biased x, and grad_q / grad_kv add dx_i = alpha_i (D_i w <dZ_u, V_v> - t_u) (the
 * bias gradient; D w = 1 without dropout) to dbias[i] when dbias is not null.  The caller zeroes dbias.
 * Masking: bias[i] = -inf masks entry i: alpha_i = 0, it adds nothing to acc or s, and dx_i = 0.  A row whose
 * entries are all masked keeps s = 0, so finish gives it Z = 0, L = -inf, and its gradients are 0 (as for a row
 * without entries; the edge softmax gives NaN there instead).  bias = +inf or NaN is not checked: the row's results
 * are then NaN.  A bias of zeros gives results bit-identical to the calls without bias.
 * The backward's grad_q reads the bias of its (A-order) block and grad_kv that of its transpose (B-order): both
 * must hold the same b(u, v) for every stored (u, v), as the step did.
 * bias null, p < 0, p >= 1, NaN, u0 < 0 or v0 < 0: HNH_E_INVALID before any launch. */
int hnh_sparse_attention_step_bias_f64(const int64_t *rowStart, const int64_t *col_idx, int64_t rows, int64_t nnz, int d,
                                       const double *Q, int64_t ldq, const double *K, int64_t ldk, const double *V,
                                       int64_t ldv, double scale, double *acc, int64_t ldacc, double *m, int64_t ldm,
                                       double *s, int64_t lds, double p, uint64_t seed, int64_t u0, int64_t v0,
                                       const double *bias, void *stream);
int hnh_sparse_attention_grad_q_bias_f64(const int64_t *rowStart, const int64_t *col_idx, int64_t rows, int64_t nnz,
                                         int d, const double *Q, int64_t ldq, const double *dZ, int64_t lddz,
                                         const double *L, int64_t ldl, const double *t, int64_t ldt, const double *K,
                                         int64_t ldk, const double *V, int64_t ldv, double scale, double *dQ,
                                         int64_t lddq, double p, uint64_t seed, int64_t u0, int64_t v0,
                                         const double *bias, double *dbias, void *stream);
int hnh_sparse_attention_grad_kv_bias_f64(const int64_t *rowStart, const int64_t *col_idx, int64_t rows, int64_t nnz,
                                          int d, const double *K, int64_t ldk, const double *V, int64_t ldv,
                                          const double *Q, int64_t ldq, const double *dZ, int64_t lddz, const double *L,
                                          int64_t ldl, const double *t, int64_t ldt, double scale, double *dK,
                                          int64_t lddk, double *dV, int64_t lddv, double p, uint64_t seed, int64_t u0,
                                          int64_t v0, const double *bias, double *dbias, void *stream);
/* Edge features: the bias calls with a nullable bias (null: no bias; p = 0: no dropout) and, before the stream, a
 * d-wide row per entry, E_i at E + i lde (block-local, in col_idx order), added to the key and to the value:
 *     x_i = scale <Q_u, K_v + E_i> + bias[i],     Z_u = sum_i D_i w alpha_i (V_v + E_i)
 * (D w = 1 without dropout).  The gradients use g_i = <dZ_u, V_v + E_i> and dx_i = alpha_i (D_i w g_i - t_u):
 *     dQ_u += scale sum_i dx_i (K_v + E_i),  dK_v += scale sum_i dx_i Q_u,  dV_v += sum_i D_i w alpha_i dZ_u,
 * dbias as above, and grad_q also writes (overwrites, once per entry)
 *     dE_i = scale dx_i Q_u + D_i w alpha_i dZ_u
 * to dE + i ldde when dE is not null (0 for a masked entry; scale dx_i Q_u for a dropped one).  grad_q reads E in
 * the order of its (A-order) block, grad_kv in that of its transpose (B order): both must hold the same e(u, v) for
 * every stored (u, v), as the step did.  Masking and rows without live entries are as for the bias.  E = 0 gives
 * results bit-identical to the calls without E (finite inputs, no signed zeros).  The fast kernels need E (and dE)
 * 16-byte aligned with an even leading dimension, as the other d-wide operands; else the generic kernels run.
 * E null, lde < d, dE with ldde < d, dE == E, dbias without bias, p < 0, p >= 1, NaN, u0 < 0 or v0 < 0:
 * HNH_E_INVALID before any launch. */
int hnh_sparse_attention_step_edge_f64(const int64_t *rowStart, const int64_t *col_idx, int64_t rows, int64_t nnz, int d,
                                       const double *Q, int64_t ldq, const double *K, int64_t ldk, const double *V,
                                       int64_t ldv, double scale, double *acc, int64_t ldacc, double *m, int64_t ldm,
                                       double *s, int64_t lds, double p, uint64_t seed, int64_t u0, int64_t v0,
                                       const double *bias, const double *E, int64_t lde, void *stream);
int hnh_sparse_attention_grad_q_edge_f64(const int64_t *rowStart, const int64_t *col_idx, int64_t rows, int64_t nnz,
                                         int d, const double *Q, int64_t ldq, const double *dZ, int64_t lddz,
                                         const double *L, int64_t ldl, const double *t, int64_t ldt, const double *K,
                                         int64_t ldk, const double *V, int64_t ldv, double scale, double *dQ,
                                         int64_t lddq, double p, uint64_t seed, int64_t u0, int64_t v0,
                                         const double *bias, double *dbias, const double *E, int64_t lde, double *dE,
                                         int64_t ldde, void *stream);
int hnh_sparse_attention_grad_kv_edge_f64(const int64_t *rowStart, const int64_t *col_idx, int64_t rows, int64_t nnz,
                                          int d, const double *K, int64_t ldk, const double *V, int64_t ldv,
                                          const double *Q, int64_t ldq, const double *dZ, int64_t lddz, const double *L,
                                          int64_t ldl, const double *t, int64_t ldt, double scale, double *dK,
                                          int64_t lddk, double *dV, int64_t lddv, double p, uint64_t seed, int64_t u0,
                                          int64_t v0, const double *bias, double *dbias, const double *E, int64_t lde,
                                          void *stream);

/* ---- graph transformer (GraphTransformer, include/hnh/graph_transformer.hpp; csrc/graph_transformer.cu) --------
 * Row-major contiguous n x r matrices; w_beta (nullable: no gate) holds 3r doubles [w1 | w2 | w3].  Rows take
 * 16-byte pair loads when r is even and every matrix and vector is 16-byte aligned, scalars otherwise.  Fixed
 * summation orders: repeated calls give bit-identical results.  Empty input is a no-op.
 *
 * X[i, :] += b for every row i (the projection biases; b holds r doubles) */
int hnh_row_bias_add_f64(double *X, const double *b, int64_t n, int64_t r, void *stream);
/* The gate forward: with beta_i = sigmoid(<w1, M_i> + <w2, R_i> + <w3, M_i - R_i>),
 *     Y_i = beta_i R_i + (1 - beta_i) M_i    (Y = M + R when w_beta is null),
 * then Y = max(Y, 0) when relu != 0.  Y may be neither M nor R. */
int hnh_gt_gate_f64(double *Y, const double *M, const double *R, const double *w_beta, int64_t n, int64_t r, int relu,
                    void *stream);
/* The gate backward, given G = dL/dY (after the ReLU when relu != 0; Y is then the forward's output and dY = G
 * where Y > 0, else 0): with ds_i = <dY_i, R_i - M_i> beta_i (1 - beta_i),
 *     dM_i = (1 - beta_i) dY_i + ds_i (w1 + w3),  dR_i = beta_i dY_i + ds_i (w2 - w3),
 *     dw_beta = sum_i ds_i [M_i, R_i, M_i - R_i]    (3r doubles, overwritten; 0 for n = 0),
 * or, with a null w_beta, dM = dY and dR (nullable) = dY, and dw_beta must be null.  dw_beta is reduced in two
 * stages, over fixed row chunks (depending on n only) and then over the chunks in order, in a workspace of
 * hnh_gt_gate_backward_workspace_bytes(n, r) bytes (needed with the gate only).  Outputs may not alias inputs. */
int64_t hnh_gt_gate_backward_workspace_bytes(int64_t n, int64_t r);
int hnh_gt_gate_backward_f64(double *dM, double *dR, double *dw_beta, const double *G, const double *Y, const double *M,
                             const double *R, const double *w_beta, int64_t n, int64_t r, int relu, void *workspace,
                             size_t workspace_bytes, void *stream);
/* The transformer block (GraphTransformer with ffn_ratio > 0).  Z = max(A + b, 0) row by row (the first feed-forward
 * layer's bias and ReLU; b holds r doubles).  Z may be neither A nor b. */
int hnh_row_bias_relu_f64(double *Z, const double *A, const double *b, int64_t n, int64_t r, void *stream);
/* LayerNorm of every row of x = X + Res (Res nullable: x = X):
 *     Y_i = gamma (x_i - mean_i) rstd_i + beta,  rstd_i = 1 / sqrt(var_i + eps)   (biased variance over the r columns),
 * as torch.nn.functional.layer_norm.  stats (2n doubles) receives (mean_i, rstd_i) at [2i, 2i + 1].  The variance is
 * taken from the centred values.  eps must be finite and > 0; Y and stats may not be inputs.  One warp per row; up to
 * r = 1536 a row is read once and kept in registers. */
int hnh_layer_norm_f64(double *Y, double *stats, const double *X, const double *Res, const double *gamma, const double *beta,
                       int64_t n, int64_t r, double eps, void *stream);
/* Its backward, given G = dL/dY and the forward's X, Res and stats: with g = G gamma and xh = (x - mean) rstd,
 *     dX_i = rstd_i (g_i - mean(g_i) - xh_i mean(g_i xh_i))   (written, or added to dX when accumulate != 0),
 *     dgamma = sum_i G_i xh_i,  dbeta = sum_i G_i            (r doubles each, overwritten; 0 for n = 0).
 * dX is also the gradient of Res.  dgamma and dbeta are reduced as dw_beta is, over fixed row chunks and then the
 * chunks in order, in a workspace of hnh_layer_norm_backward_workspace_bytes(n, r) bytes: no atomics, repeated calls
 * are bit-identical.  Outputs may not alias inputs or each other. */
int64_t hnh_layer_norm_backward_workspace_bytes(int64_t n, int64_t r);
int hnh_layer_norm_backward_f64(double *dX, double *dgamma, double *dbeta, const double *G, const double *X, const double *Res,
                                const double *stats, const double *gamma, int64_t n, int64_t r, int accumulate,
                                void *workspace, size_t workspace_bytes, void *stream);

/* ---- training (include/hnh/training.hpp; csrc/training.cu) ---------------------------------------------------------
 * Cross-entropy of n rows of logits (n x C, leading dimension ld >= C) against int32 labels: a row is labelled when
 * 0 <= labels[i] < C and ignored otherwise.  With lse_i = max_i + log sum_k exp(x_ik - max_i):
 *     dlogits_ik = (exp(x_ik - lse_i) - [k == labels[i]]) * inv_count   (0 on ignored rows; same ld as logits),
 *     sums[0] = sum over labelled rows of lse_i - x_i,labels[i],
 *     sums[1] = the number of labelled rows whose argmax (ties to the lowest index, as torch.argmax) is their label.
 * inv_count is the caller's 1 / (labelled rows), e.g. over all ranks; sums are not scaled by it.  The label is only
 * compared with column indices, never used to address memory.  One warp per row; up to C = 1536 the row is read once.
 * sums are reduced over per-row values in the fixed two-stage order of hnh_layer_norm_backward_f64, in a workspace of
 * hnh_cross_entropy_workspace_bytes(n) bytes: repeated calls are bit-identical.  dlogits may not be logits; n = 0
 * writes sums = 0. */
int64_t hnh_cross_entropy_workspace_bytes(int64_t n);
int hnh_cross_entropy_f64(double *dlogits, double *sums, const double *logits, const int32_t *labels, int64_t n, int64_t C,
                          int64_t ld, double inv_count, void *workspace, size_t workspace_bytes, void *stream);
/* One AdamW step on one tensor of n doubles, in place on param, m and v, as torch.optim.AdamW(foreach=False,
 * amsgrad=False) with g = grad * (*clip_coef) (clip_coef: a nullable DEVICE scalar, so a clip coefficient computed on
 * the device needs no host round trip; null = 1):
 *     param *= 1 - lr weight_decay;  m = lerp(m, g, 1 - beta1);  v = v beta2 + (1 - beta2) g g;
 *     param -= lr / bias_correction1 * m / (sqrt(v) / sqrt(bias_correction2) + eps),
 * with bias_correction_k = 1 - beta_k^t from the caller.  grad is not written.  lr, weight_decay >= 0, betas in [0, 1),
 * eps > 0, bias corrections in (0, 1], all finite; param, m, v, grad distinct. */
int hnh_adamw_f64(double *param, double *m, double *v, const double *grad, int64_t n, double lr, double beta1, double beta2,
                  double eps, double weight_decay, double bias_correction1, double bias_correction2, const double *clip_coef,
                  void *stream);
/* The coefficient of torch.nn.utils.clip_grad_norm_ from per-tensor squared norms (hnh_squared_norm_f64 of each):
 * total_coef[0] = sqrt(sum of squared_norms[0 .. count) in order), total_coef[1] = min(1, max_norm / (total + 1e-6)).
 * max_norm >= 0; +inf gives coef = 1. */
int hnh_clip_coef_f64(double *total_coef, const double *squared_norms, int64_t count, double max_norm, void *stream);
/* sums[j] = sum over i < n of pairs[2i + j], j = 0, 1 (n rows of 2 contiguous doubles), in the fixed two-stage order of
 * hnh_cross_entropy_f64's sums, in a workspace of hnh_pair_sums_workspace_bytes(n) bytes.  n = 0 writes sums = 0. */
int64_t hnh_pair_sums_workspace_bytes(int64_t n);
int hnh_pair_sums_f64(double *sums, const double *pairs, int64_t n, void *workspace, size_t workspace_bytes, void *stream);

/* ---- link prediction (Distributed_Sparse::linkLoss; csrc/link_prediction.cu) --------------------------------------
 * The dot-product edge decoder with binary cross-entropy on one CSR block: X (rows x r, leading dimension ldx) is
 * indexed by the stored row u, Y (ldy) gathered by col_idx v, and target[i] = y_uv is entry i's target.  Per entry:
 *     s = <X_u, Y_v>,  loss = max(s, 0) - s y + log1p(exp(-|s|)),  correct = [(s > 0) == (y > 0.5)],
 *     g = (sigmoid(s) - y) inv_count,
 * and the nullable outputs: dX_u += sum_v g Y_v (lddx), stats[u * lds] += sum_v loss, stats[u * lds + 1] += sum_v
 * correct (lds >= 2), scores[i] = s.  Rows without entries are not touched.  r >= 1, every leading dimension >= r (the
 * stats' >= 2), inv_count finite and >= 0; an output may not be an input or another output.  Widths 4..256 (powers
 * of two) with 16-byte aligned X, Y, dX and even leading dimensions take a row kernel with X_u in registers and
 * 128-bit gathers; others a one-warp-per-row kernel.  No atomics: repeated calls are bit-identical. */
int hnh_link_bce_f64(const int64_t *rowStart, const int64_t *col_idx, const double *target, int64_t rows, int64_t nnz,
                     const double *X, int64_t ldx, const double *Y, int64_t ldy, int r, double inv_count, double *dX,
                     int64_t lddx, double *stats, int64_t lds, double *scores, void *stream);
/* bad[0] (device) += the number of target[0 .. n) that are not in [0, 1] (NaN and infinities count) */
int hnh_link_target_check_f64(double *bad, const double *target, int64_t n, void *stream);

/* ---- relation-aware link prediction (Distributed_Sparse::distmultLoss; csrc/distmult.cu) ----------------------------
 * The DistMult edge decoder with binary cross-entropy on one CSR block.  values[i] is entry i's relation rho, an integer
 * in [0, R) (any other value: the entry contributes nothing, and its score and g are 0); D (R x r, leading dimension
 * ldd) is the relation table and `target` (in [0, 1]) the target of every entry of the call.  X is indexed by the stored
 * row u, Y gathered by col_idx v.  Per entry:
 *     s = sum_k X_u,k D_rho,k Y_v,k,  loss, correct and g = (sigmoid(s) - target) inv_count as hnh_link_bce_f64,
 * hnh_distmult_bce_f64 (the A order) with the nullable outputs dX_u += sum_v g (D_rho o Y_v), stats[u * lds] += sum
 * loss, stats[u * lds + 1] += sum correct (lds >= 2), scores[i] = s and g[i] = g; hnh_distmult_bce_grad_f64 (the B
 * order: X is the B side) only dX_v += sum_u g (D_rho o Y_u).  Rows without entries are not touched.  r, R >= 1, every
 * leading dimension >= r (the stats' >= 2), inv_count finite and >= 0; an output may not be an input or another output.
 * Widths 4..256 (powers of two) with 16-byte aligned X, Y, D, dX and even leading dimensions take a row kernel with X_u
 * in registers and 128-bit gathers, D with an L2 evict-last policy and the block's index and value streams with
 * evict-first; others a one-warp-per-row kernel.  No atomics: repeated calls are bit-identical.
 * hnh_distmult_relation_grad_f64: the relation-table gradient of one block from a plan of its entries keyed by relation
 * (hnh_relation_keys over R + 1 keys, then hnh_edge_softmax_plan): num_pieces pieces, the key of piece q piece_key[q]
 * (the plan's piece_row), and
 *     dD[rho, :] += sum over the entries i of relation rho of g[i] (X[row_idx[i], :] o Y[col_idx[i], :])   (rho < R)
 * with row_idx / col_idx the entries' stored rows and gathered rows.  Each piece's sum goes to row q of `partial`
 * (num_pieces x r, contiguous), then the pieces of each relation are added in plan order: repeated calls are
 * bit-identical. */
int hnh_distmult_bce_f64(const int64_t *rowStart, const int64_t *col_idx, const double *values, int64_t rows, int64_t nnz, int R,
                         const double *X, int64_t ldx, const double *Y, int64_t ldy, const double *D, int64_t ldd, int r,
                         double target, double inv_count, double *dX, int64_t lddx, double *stats, int64_t lds, double *scores,
                         double *g, void *stream);
int hnh_distmult_bce_grad_f64(const int64_t *rowStart, const int64_t *col_idx, const double *values, int64_t rows, int64_t nnz,
                              int R, const double *X, int64_t ldx, const double *Y, int64_t ldy, const double *D, int64_t ldd, int r,
                              double target, double inv_count, double *dX, int64_t lddx, void *stream);
int hnh_distmult_relation_grad_f64(const int32_t *perm, const int32_t *key_start, const int32_t *piece_first, const int32_t *piece_key,
                                   int64_t num_pieces, int R, const int64_t *row_idx, const int64_t *col_idx, const double *g,
                                   const double *X, int64_t ldx, const double *Y, int64_t ldy, int r, double *partial, double *dD,
                                   int64_t ldd, void *stream);

/* ---- filtered link ranking (include/hnh/link_ranking.hpp; csrc/link_ranking.cu) ----------------------------------
 * Z is `rows` x r (leading dimension ldz): the rows that are ranking candidates; Q is n_q x r (ldq): one query vector
 * per row; scores are s(u, q) = sum_k Z_u,k Q_q,k.  r >= 1 and every leading dimension >= r; ids are 0-based.
 * hnh_rank_count_f64: gt[q] += #{u < rows : s(u, q) > s_true[q]} and ge[q] += #{u < rows : s(u, q) >= s_true[q]}, for
 *     every q < n_q, in 64-bit integers (gt and ge separate arrays).  The n_q x rows scores are compared where they are
 *     computed and never stored.  fp64 DMMA (mma.sync m8n8k4) in 64 x 64 tiles with K in steps of 16; integer atomics,
 *     so repeated calls are bit-identical.
 * hnh_rank_queries_f64: Q[q, :] = Z[anchors[q] - row0, :] o D[rels[q], :] for the anchors in [row0, row0 + rows) (Z's
 *     row alone when D is null), and 0 for every other anchor and for a relation outside [0, R) (D: R x r, ldd).
 * hnh_rank_pairs_f64: for the pairs p < n_pairs, s = s(pair_row[p], pair_q[p]) with hnh_rank_count_f64's arithmetic,
 *     bit for bit: the same instruction, k steps and zero padding, at the count kernel's fragment position.  Nullable
 *     outputs: scores[p] = s; with gt, ge and s_true, gt[q] -= (s > s_true[q]) and ge[q] -= (s >= s_true[q]), which
 *     takes a pair the count kernel counted back out exactly.  Pairs with q outside [0, n_q) or a row outside
 *     [0, rows) are skipped. */
int hnh_rank_count_f64(const double *Z, int64_t ldz, int64_t rows, const double *Q, int64_t ldq, int64_t n_q, int r,
                       const double *s_true, int64_t *gt, int64_t *ge, void *stream);
int hnh_rank_queries_f64(double *Q, int64_t ldq, int64_t n_q, const double *Z, int64_t ldz, int64_t row0, int64_t rows,
                         const int64_t *anchors, const int64_t *rels, const double *D, int64_t ldd, int R, int r, void *stream);
int hnh_rank_pairs_f64(const double *Z, int64_t ldz, int64_t rows, const double *Q, int64_t ldq, int64_t n_q, int r,
                       const int64_t *pair_q, const int64_t *pair_row, int64_t n_pairs, double *scores, const double *s_true,
                       int64_t *gt, int64_t *ge, void *stream);

/* ---- max aggregation (Distributed_Sparse::maxAggregate; csrc/graph_sage.cu) ----------------------------------------
 * The SpMM over the (max, .) semiring on one CSR block, and its gradient.  S's values are not read; duplicates count.
 * hnh_max_aggregate_step_f64: for every stored row u, over its entries v (X: gathered, leading dimension ldx),
 *     (Z_u,k, C_u,k) = merge((Z_u,k, C_u,k), (max_v X_v,k, #{v : X_v,k == max}))
 * where merge keeps the larger maximum and adds the counts of equal ones.  Z and C are read and written once per row
 * (they may carry the state of earlier blocks); before the first block they hold (-inf, 0).  Rows without entries are
 * not touched.  hnh_max_aggregate_finish_f64 then sets Z[i] = 0 where C[i] = 0 (n contiguous doubles).
 * hnh_max_aggregate_grad_scale_f64: G[i] = dZ[i] / C[i], and 0 where C[i] = 0 (n contiguous doubles; G may be dZ).
 * hnh_max_aggregate_grad_f64, on a block whose stored rows are X's (the B order): for every stored row v, over its
 * entries u (Z, G gathered),
 *     dX_v,k += sum_u [X_v,k == Z_u,k] G_u,k         (accumulated in stored order, then one read-modify-write of dX)
 * f >= 1, every leading dimension >= f; outputs may not alias inputs.  Column windows of 256 run separately (max is
 * independent per column); a window of width 4..256 (a power of two) with 16-byte aligned operands and even leading
 * dimensions takes a row kernel with 128-bit gathers, others a one-warp-per-row kernel.  No atomics: repeated calls
 * are bit-identical. */
int hnh_max_aggregate_step_f64(const int64_t *rowStart, const int64_t *col_idx, int64_t rows, int64_t nnz, const double *X,
                               int64_t ldx, int f, double *Z, int64_t ldz, double *C, int64_t ldc, void *stream);
int hnh_max_aggregate_finish_f64(double *Z, const double *C, int64_t n, void *stream);
int hnh_max_aggregate_grad_scale_f64(double *G, const double *dZ, const double *C, int64_t n, void *stream);
int hnh_max_aggregate_grad_f64(const int64_t *rowStart, const int64_t *col_idx, int64_t rows, int64_t nnz, const double *X,
                               int64_t ldx, const double *Z, int64_t ldz, const double *G, int64_t ldg, int f, double *dX,
                               int64_t lddx, void *stream);

/* ---- multi-statistic aggregation (Distributed_Sparse::multiAggregate, PNA; csrc/pna.cu) -----------------------------
 * Several statistics of the gathered rows of every CSR row in one pass.  `which` selects them (any non-empty union of
 * the flags); the state A of a row holds the selected f-wide windows side by side in the fixed order
 *     [S1 | S2 | MAX | CMAX | MIN | CMIN]          (HNH_MULTI_MOMENTS: S1, S2; HNH_MULTI_MAX: MAX, CMAX; HNH_MULTI_MIN: MIN, CMIN)
 * so it is 2 f, 4 f or 6 f wide.  S's values are not read; duplicates count.
 * hnh_multi_aggregate_step_f64: for every stored row u, over its entries v (X: gathered, leading dimension ldx),
 *     S1_u += sum_v X_v,   S2_u += sum_v X_v^2,   (MAX_u, CMAX_u) = merge(.., (max_v X_v, #{v : X_v == max})),
 *     (MIN_u, CMIN_u) likewise with the minimum
 * merging as hnh_max_aggregate_step_f64 does.  A is read and written once per row (it may carry earlier blocks); before
 * the first block it holds (0, 0, -inf, 0, +inf, 0).  Rows without entries are not touched.
 * hnh_multi_aggregate_finish_f64 then sets MAX and MIN to 0 where their count is 0 (rows x f per window).
 * hnh_multi_aggregate_grad_prep_f64: D (A's layout) = [dA_S1 | dA_S2 | MAX | dA_MAX / CMAX | MIN | dA_MIN / CMIN], the
 * quotients 0 where the count is 0; dA has A's layout (its count windows are not read).
 * hnh_multi_aggregate_grad_f64, on a block whose stored rows are X's (the B order): for every stored row v, over its
 * entries u (D gathered),
 *     dX_v += sum_u D_S1,u + 2 X_v sum_u D_S2,u + sum_u [X_v == MAX_u] D_CMAX,u + sum_u [X_v == MIN_u] D_CMIN,u
 * (each sum in stored order in registers, then one read-modify-write of dX).
 * f >= 1, the state's width below 2^31, every leading dimension >= its operand's width; outputs may not alias inputs.
 * Column windows of 256 run separately; a window of width 4..256 (a power of two) with 16-byte aligned windows and
 * even leading dimensions takes a row kernel with 128-bit gathers, others a one-warp-per-row kernel.  No atomics:
 * repeated calls are bit-identical.
 * hnh_pna_combine_f64 / _grad_f64: PNA's aggregators and degree scalers (include/hnh/pna.hpp) for rows x f elements.
 * aggs and scalers hold n_aggs (1..6) and n_scalers (1..5) of the codes below, 4 bits each, the first in the lowest
 * bits; deg (stride ldg) holds each row's entry count.  With h_uv = C_u + z_v and A the state of z:
 *     P_u = [X_u | scale_s0(u) [agg_0(u) .. agg_n-1(u)] | scale_s1(u) [..] | ..]          ((n_aggs n_scalers + 1) f wide)
 * and the gradient writes dC (rows x f) and dA (A's layout, count windows 0) from dP.  An aggregator whose statistic
 * `which` does not hold (min without HNH_MULTI_MIN, max without HNH_MULTI_MAX, the others without HNH_MULTI_MOMENTS)
 * is refused. */
#define HNH_MULTI_MOMENTS 1
#define HNH_MULTI_MAX 2
#define HNH_MULTI_MIN 4
#define HNH_MULTI_ALL 7
#define HNH_PNA_MEAN 0
#define HNH_PNA_SUM 1
#define HNH_PNA_MIN 2
#define HNH_PNA_MAX 3
#define HNH_PNA_VAR 4
#define HNH_PNA_STD 5
#define HNH_PNA_IDENTITY 0
#define HNH_PNA_AMPLIFICATION 1
#define HNH_PNA_ATTENUATION 2
#define HNH_PNA_LINEAR 3
#define HNH_PNA_INVERSE_LINEAR 4
int hnh_multi_aggregate_step_f64(const int64_t *rowStart, const int64_t *col_idx, int64_t rows, int64_t nnz, const double *X,
                                 int64_t ldx, int f, int which, double *A, int64_t lda, void *stream);
int hnh_multi_aggregate_finish_f64(double *A, int64_t lda, int64_t rows, int f, int which, void *stream);
int hnh_multi_aggregate_grad_prep_f64(const double *A, int64_t lda, const double *dA, int64_t ldda, int64_t rows, int f, int which,
                                      double *D, int64_t ldd, void *stream);
int hnh_multi_aggregate_grad_f64(const int64_t *rowStart, const int64_t *col_idx, int64_t rows, int64_t nnz, const double *X,
                                 int64_t ldx, const double *D, int64_t ldd, int f, int which, double *dX, int64_t lddx, void *stream);
int hnh_pna_combine_f64(const double *X, int64_t ldx, const double *C, int64_t ldc, const double *A, int64_t lda, int which,
                        const double *deg, int64_t ldg, int64_t rows, int f, unsigned aggs, int n_aggs, unsigned scalers, int n_scalers,
                        double avg_deg_lin, double avg_deg_log, double *P, int64_t ldp, void *stream);
int hnh_pna_combine_grad_f64(const double *dP, int64_t lddp, const double *A, int64_t lda, int which, const double *deg, int64_t ldg,
                             int64_t rows, int f, unsigned aggs, int n_aggs, unsigned scalers, int n_scalers, double avg_deg_lin,
                             double avg_deg_log, double *dC, int64_t lddc, double *dA, int64_t ldda, void *stream);

/* ---- edge-ReLU aggregation (Distributed_Sparse::edgeReluAggregate, GINE; csrc/gine.cu) ------------------------------
 * Entry i of the block (u its stored row, v = col_idx[i]) reads the f-wide edge row E_i at E + i lde.
 * hnh_edge_relu_aggregate_step_f64:      A_u  += sum_i ReLU(X_v + E_i)           (X gathered; A read and written once per
 *                                                                                 row, so it may carry earlier blocks)
 * hnh_edge_relu_aggregate_grad_f64:      dX_v += sum_i [X_v + E_i > 0] dA_u       (stored rows are X's: the B order; dA
 *                                                                                 gathered; one read-modify-write of dX)
 * hnh_edge_relu_aggregate_edge_grad_f64: dE_i  = [X_v + E_i > 0] dA_u             (stored rows are dA's: the A order; X
 *                                                                                 gathered; every row of dE written once)
 * The mask is strict (torch's relu backward).  Rows without entries are not touched.  S's values are not read.  f >= 1,
 * every leading dimension >= f; outputs may not alias inputs.  Column windows of 256 run separately; a window of width
 * 4..256 (a power of two) with 16-byte aligned operands and even leading dimensions takes a row kernel with 128-bit
 * loads, others a one-warp-per-row kernel.  E is streamed with an L2 evict-first policy.  No atomics: repeated calls
 * are bit-identical.
 * hnh_gin_combine_f64:      H = M + (1 + *eps) X over n contiguous elements (eps a device scalar; H may be M).
 * hnh_gin_combine_grad_f64: dX = (1 + *eps) dH over n elements and, unless deps is null, *deps (device) = sum dH X in
 *                           an order fixed by the device and n (repeated calls are bit-identical). */
int hnh_edge_relu_aggregate_step_f64(const int64_t *rowStart, const int64_t *col_idx, int64_t rows, int64_t nnz, const double *X,
                                     int64_t ldx, const double *E, int64_t lde, int f, double *A, int64_t lda, void *stream);
int hnh_edge_relu_aggregate_grad_f64(const int64_t *rowStart, const int64_t *col_idx, int64_t rows, int64_t nnz, const double *X,
                                     int64_t ldx, const double *E, int64_t lde, const double *dA, int64_t ldda, int f, double *dX,
                                     int64_t lddx, void *stream);
int hnh_edge_relu_aggregate_edge_grad_f64(const int64_t *rowStart, const int64_t *col_idx, int64_t rows, int64_t nnz,
                                          const double *dA, int64_t ldda, const double *X, int64_t ldx, const double *E, int64_t lde,
                                          int f, double *dE, int64_t ldde, void *stream);
int hnh_gin_combine_f64(double *H, const double *M, const double *X, const double *eps, int64_t n, void *stream);
int hnh_gin_combine_grad_f64(double *dX, double *deps, const double *dH, const double *X, const double *eps, int64_t n, void *stream);

/* ---- graph readout (include/hnh/graph_readout.hpp; csrc/graph_readout.cu) -------------------------------------------
 * Pools the rows of H (rows x r, leading dimension ldh) into one row per segment.  The segment CSR lists, for segment
 * g < segments, the rows seg_rows[seg_start[g] .. seg_start[g + 1]) of H (any order; the sums run in the listed order).
 * The chunk plan cuts every segment into chunks of HNH_SEGMENT_CHUNK rows, an empty segment into one empty chunk:
 * chunk_first[g] (segments + 1 entries) is the first chunk of segment g, chunk_first[segments] = chunks, and
 * chunk_seg[k] (chunks entries) the segment of chunk k.  Row indices are not bounds-checked; seg_rows may be null when
 * no segment has a row.
 * hnh_segment_pool_f64 overwrites row g of P (leading dimension ldp) for every segment; C null gives the sum
 *     P_g = sum_{u in g} H_u                                           (0 for an empty segment)
 * and C non-null (leading dimension ldc) the maximum with its tie count, as hnh_max_aggregate_step_f64:
 *     (P_g,k, C_g,k) = (max_u H_u,k, #{u : H_u,k == max})              ((-inf, 0) for an empty segment)
 * Every chunk's rows are read once, by its own lane group; the segments of more than one chunk then combine their
 * chunk results from `workspace` (hnh_segment_pool_workspace_bytes(chunks, r, C != 0) bytes; none needed, and null
 * allowed, when chunks == segments) in an order fixed by the segment lengths.  r >= 1, every leading dimension >= r;
 * P and C may not be H or each other.
 * hnh_segment_max_count_merge_f64: C[i] = 0 where local_max[i] != global_max[i] (n contiguous doubles): the counts of a
 * rank whose maximum is not the maximum over all ranks drop out before the counts are summed over the ranks.
 * hnh_segment_pool_grad_f64 overwrites every row u < rows of dH (leading dimension lddh): with g = row_graph[u],
 *     dH_u = scale[g] dP_g                          (H, P, C null; scale nullable: 1) -- sum and mean
 *     dH_u,k = [H_u,k == P_g,k] dP_g,k / C_g,k      (H, P, C all non-null, scale null; 0 where C = 0) -- max
 * and dH_u = 0 where g lies outside [0, graphs).  dH may not be an input.
 * Widths 4..256 (powers of two) with 16-byte aligned operands and even leading dimensions take 128-bit chunk and row
 * kernels; others one-warp-per-chunk and one-warp-per-row kernels.  No atomics: repeated calls are bit-identical. */
#define HNH_SEGMENT_CHUNK 256
int64_t hnh_segment_pool_workspace_bytes(int64_t chunks, int r, int with_counts);
int hnh_segment_pool_f64(const int64_t *seg_start, const int64_t *seg_rows, const int64_t *chunk_first, const int32_t *chunk_seg,
                         int64_t segments, int64_t chunks, const double *H, int64_t ldh, int r, double *P, int64_t ldp, double *C,
                         int64_t ldc, void *workspace, size_t workspace_bytes, void *stream);
int hnh_segment_max_count_merge_f64(double *C, const double *local_max, const double *global_max, int64_t n, void *stream);
int hnh_segment_pool_grad_f64(const int32_t *row_graph, int64_t rows, int64_t graphs, const double *dP, int64_t lddp,
                              const double *scale, const double *H, int64_t ldh, const double *P, int64_t ldp, const double *C,
                              int64_t ldc, int r, double *dH, int64_t lddh, void *stream);

/* ---- relational aggregation (Distributed_Sparse::relationalAggregate; csrc/rgcn.cu) ---------------------------------
 * R-GCN's neighbour aggregation on one CSR block: the stored value of an entry is its relation rho, an integer in
 * [0, R).  An entry whose value is anything else (negative, >= R, fractional, infinite, NaN) contributes nothing and
 * its gathered row is not read.
 * hnh_relational_aggregate_f64: for every stored row u and entry (v, rho) (X: gathered, leading dimension ldx),
 *     A[u, rho f + k] += X[v, k]          (A is R f wide; the caller zeroes it before the first block)
 * The relations present in a row are swept in increasing order, each one's entries summed in registers in stored order
 * and added to the (row, relation) window with one read-modify-write; windows without entries are not touched.
 * hnh_relational_aggregate_grad_f64, on a block whose stored rows are X's (the B order): for every stored row v and
 * entry (u, rho) (dA gathered),
 *     dX[v, k] += dA[u, rho f + k]         (accumulated in stored order, then one read-modify-write of dX)
 * f >= 1, R >= 1, R f < 2^31, every leading dimension >= its operand's width; outputs may not alias inputs.  Column
 * windows of 256 run separately; a window of width 4..256 (a power of two) with 16-byte aligned operands, even leading
 * dimensions and an even f takes a row kernel with 128-bit gathers, others a one-warp-per-row kernel.  No atomics:
 * repeated calls are bit-identical.
 * hnh_window_scale_f64: A[u, rho f + k] = A[u, rho f + k] / C[u, rho], and 0 where C[u, rho] = 0, for u < n (the mean
 * of R-GCN, forward and backward; C holds the per-(row, relation) entry counts).
 * hnh_relation_check_f64: bad[0] (device) += the number of values[0 .. n) that are not integers in [0, R). */
int hnh_relational_aggregate_f64(const int64_t *rowStart, const int64_t *col_idx, const double *values, int64_t rows, int64_t nnz,
                                 const double *X, int64_t ldx, int f, int R, double *A, int64_t lda, void *stream);
int hnh_relational_aggregate_grad_f64(const int64_t *rowStart, const int64_t *col_idx, const double *values, int64_t rows,
                                      int64_t nnz, const double *dA, int64_t ldda, int f, int R, double *dX, int64_t lddx,
                                      void *stream);
int hnh_window_scale_f64(double *A, int64_t lda, const double *C, int64_t ldc, int64_t n, int f, int R, void *stream);
int hnh_relation_check_f64(double *bad, const double *values, int64_t n, int R, void *stream);

/* ---- basis aggregation (Distributed_Sparse::basisAggregate; csrc/rgcn.cu) ---------------------------------------------
 * R-GCN with basis decomposition on one CSR block.  comp is the R x B coefficient matrix (row-major, device), scale
 * (nullable: all ones) holds a weight per (stored row of the A order, relation) with leading dimension lds, and rho is
 * an entry's relation as for hnh_relational_aggregate_f64 (an entry that is no relation contributes nothing and its
 * gathered row is not read).
 * hnh_basis_aggregate_f64: for every stored row u and entry (v, rho) (X gathered),
 *     H[u, b f + k] += scale[u, rho] comp[rho, b] X[v, k]        (H is B f wide; the caller zeroes it first)
 * summed in stored order in registers, up to a fixed number of bases at a time (more bases re-gather the row per chunk);
 * every window of H of a row with entries is read and written once per call, so H may carry earlier blocks' sums.
 * hnh_basis_aggregate_grad_f64, on a block whose stored rows are X's (the B order): for every stored row v and entry
 * (u, rho) (dH and scale gathered),
 *     dX[v, k] += scale[u, rho] sum_b comp[rho, b] dH[u, b f + k]   (in registers, one read-modify-write of dX per row)
 * and with a non-null `products`, for entry j of the block (its CSR position),
 *     products[b ldp + j] = scale[u, rho] <dH[u, b f .. b f + f), X[v, 0 .. f)>      (0 for an entry that is no relation)
 * f, R, B >= 1, B f and R B < 2^31, every leading dimension >= its operand's width (ldp >= nnz); outputs may not alias
 * inputs.  Column windows of 256 run separately; a window of width 4..256 (a power of two) with 16-byte aligned
 * operands, even leading dimensions and an even f takes a row kernel with 128-bit gathers, others a one-warp-per-row
 * kernel.  No atomics: repeated calls are bit-identical.
 * hnh_relation_keys: keys[i] = the relation of values[i], or R for a value that is no relation (the keys of an
 * hnh_edge_softmax_plan over R + 1 rows, which sums the products by relation). */
int hnh_basis_aggregate_f64(const int64_t *rowStart, const int64_t *col_idx, const double *values, int64_t rows, int64_t nnz,
                            const double *X, int64_t ldx, int f, const double *scale, int64_t lds, const double *comp, int R, int B,
                            double *H, int64_t ldh, void *stream);
int hnh_basis_aggregate_grad_f64(const int64_t *rowStart, const int64_t *col_idx, const double *values, int64_t rows, int64_t nnz,
                                 const double *dH, int64_t lddh, const double *scale, int64_t lds, const double *comp, int R, int B,
                                 const double *X, int64_t ldx, int f, double *dX, int64_t lddx, double *products, int64_t ldp,
                                 void *stream);
int hnh_relation_keys(int32_t *keys, const double *values, int64_t n, int R, void *stream);

/* ---- host-side setup helpers (untimed; HOST pointers) --------------------------------------
 * hnh_er_generate_host replaces the CombBLAS Graph500 generator call of
 * SpmatLocal::loadTuples(false, logM, nnz_per_row) (SpmatLocal.hpp:499-516): rows
 * [row_lo,row_hi) of the seeded N x N Erdos-Renyi matrix, sorted (row, col), unique, values 1.
 * Returns the tuple count (>= 0) or a negative HNH_E_* code. */
int64_t hnh_er_generate_host(int logM, int nnz_per_row, uint64_t seed, int64_t row_lo,
                             int64_t row_hi, uint64_t *rows_out, uint64_t *cols_out,
                             double *vals_out, int64_t capacity);
/* hnh_coo_to_csr_host replaces the MKL inspector sequence of the CSRLocal constructor
 * (SpmatLocal.hpp:117-147): COO -> CSR, optional transpose, stable.  rowStart has
 * (transpose ? cols : rows) + 1 entries; row_idx (expanded stored-row index) may be NULL. */
int hnh_coo_to_csr_host(int64_t rows, int64_t cols, int64_t nnz, const uint64_t *r,
                        const uint64_t *c, const double *v, int transpose, int64_t *rowStart,
                        int64_t *col_idx, int64_t *row_idx, double *values);

/* Device versions of the two helpers above (DEVICE pointers; untimed setup; they synchronise `stream`
 * before returning).  Output is bit-identical with the host versions: the generator is a pure function
 * of (seed, row, k), the CSR order is a stable sort by stored row.  nnz_per_row <= 128; one block holds
 * fewer than 2^31 entries. */
int64_t hnh_er_generate_device(int logM, int nnz_per_row, uint64_t seed, int64_t row_lo,
                               int64_t row_hi, uint64_t *rows_out, uint64_t *cols_out,
                               double *vals_out, int64_t capacity, void *stream);
int hnh_coo_to_csr_device(int64_t rows, int64_t cols, int64_t nnz, const uint64_t *r,
                          const uint64_t *c, const double *v, int transpose, int64_t *rowStart,
                          int64_t *col_idx, int64_t *row_idx, double *values, void *stream);

/* Device-resident tuple pipeline of the setup path (SoA tuples r / c / v in HBM; reference: host vectors of
 * spcoord_t, SpmatLocal.hpp:389-462).  All synchronise `stream` before returning; fewer than 2^31 tuples per call.
 *  - bucket_by_owner: owner(i) = table[rb * table_cols + cb] with (rb, cb) = (r/rows_in_block, c/cols_in_block), or
 *    (c/rows_in_block, r/cols_in_block) when `transpose` (NonzeroDistribution::getOwner, SpmatLocal.hpp:45-52); the
 *    table is a HOST array filled from the distribution's blockOwner().  Output: the tuples grouped by owner in
 *    input order (stable), r and c exchanged when `transpose`; starts_host[nbuckets + 1] = segment offsets.
 *  - sort_colmajor: in place, ascending (c, r), ties in input order (the order redistribute_nonzeros leaves,
 *    SpmatLocal.hpp:458).  max_r / max_c bound the keys (number of radix bits).
 *  - mod: r %= mod_r, c %= mod_c (0 = leave).   - block_starts: first position with c >= k * block_width. */
int hnh_tuples_bucket_by_owner_device(const uint64_t *r, const uint64_t *c, const double *v, int64_t n, int transpose,
                                      int64_t rows_in_block, int64_t cols_in_block, const int *owner_table_host,
                                      int64_t table_rows, int64_t table_cols, int nbuckets, uint64_t *r_out,
                                      uint64_t *c_out, double *v_out, int64_t *starts_host, void *stream);
int hnh_tuples_sort_colmajor_device(uint64_t *r, uint64_t *c, double *v, int64_t n, uint64_t max_r, uint64_t max_c,
                                    void *stream);
int hnh_tuples_mod_device(uint64_t *r, uint64_t *c, int64_t n, uint64_t mod_r, uint64_t mod_c, void *stream);
int hnh_tuples_block_starts_device(const uint64_t *c_sorted, int64_t n, uint64_t block_width, int divisions,
                                   int64_t *starts_host, void *stream);

/* ---- host-buffer entry points (pinned or pageable HOST pointers) -------------------------
 * One call = H2D of the dense operands and values, the kernel(s), D2H of the results, all
 * inside the call; the block's CSR structure is taken from a resident handle made once with
 * hnh_block_create_host (the reference also builds its CSR once, SpmatLocal.hpp:78-188).
 * These are what bench.py's `e2e` leg times. */
typedef struct hnh_block hnh_block_t;
int hnh_block_create_host(const int64_t *rowStart, const int64_t *col_idx, int64_t rows,
                          int64_t cols, int64_t nnz, int r_max, hnh_block_t **out);
void hnh_block_destroy(hnh_block_t *blk);
/* op: 0 = sddmm (values_io += X.Y), 1 = spmm (Out += CSR*Y with values_io), 2 = fused.
 * X: rows x r, Y: cols x r, Out: rows x r (op 1, 2), values_io: nnz.
 * run_flags: HNH_RUN_ZERO_VALUES = start from values == 0 on the device instead of copying
 * values_io in (SpmatLocal::setValuesConstant(0), SpmatLocal.hpp:595-605);
 * HNH_RUN_ZERO_OUT = start from Out == 0 on the device instead of copying Out in
 * (`localA.setZero()`, distributed_sparse.h:275,304). */
#define HNH_RUN_ZERO_VALUES 1
#define HNH_RUN_ZERO_OUT 2
int hnh_block_run_host(hnh_block_t *blk, int op, const double *X, const double *Y,
                       double *values_io, double *Out, int r, int run_flags, void *stream);

/* One-shot forms with HOST pointers for a reference-side KernelImplementation that keeps the
 * reference's host data structures (include/hnh/reference_plugin/cuda_kernel.h): operands are
 * mirrored on the device for the call, the result is copied back, the call synchronises.
 * hnh_sddmm_coo_host: values[i] += X[row_idx[i]] . Y[col_idx[i]]  (StandardKernel::sddmm_local,
 * sparse_kernels.cpp:44-55; X has x_rows rows, Y has y_rows rows, both r wide).
 * hnh_spmm_host: Y[rows x r] += CSR * X  (the mkl_sparse_d_mm call, sparse_kernels.cpp:95-120;
 * X has x_rows rows). */
int hnh_sddmm_coo_host(const int64_t *row_idx, const int64_t *col_idx, double *values, int64_t nnz,
                       const double *X, int64_t x_rows, const double *Y, int64_t y_rows, int r);
int hnh_spmm_host(const int64_t *rowStart, const int64_t *col_idx, const double *values,
                  int64_t rows, int64_t nnz, const double *X, int64_t x_rows, double *Y, int r);

#ifdef __cplusplus
}
#endif
#endif /* HNH_B200_H */
