/*
 * hnh_b200_driver.h -- C ABI over the C++ host classes of libhnh_b200.so
 * (SpmatLocal, FlexibleGrid, Distributed_Sparse and its 1.5D / 2.5D subclasses,
 * benchmark_algorithm), for callers that are not C++: bench.py and the tests bind it with
 * ctypes.  C++ callers include the headers under include/hnh/ directly -- they carry the
 * reference's own class and method names (see INTEGRATION.md).
 *
 * All functions return 0 or a negative HNH_E_* code (hnh_b200.h); hnh_last_error_string()
 * describes the failure.  One process = one rank = one GPU.
 */
#ifndef HNH_B200_DRIVER_H
#define HNH_B200_DRIVER_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define HNHD_NCCL_ID_BYTES 128

/* Caller-supplied transport on HOST buffers (the "External" transport of hnh/comm.h).  Each
 * callback returns 0 on success.  `comm` is an integer handle; 0 is the world.  These map
 * one-to-one onto the MPI calls of the reference (MPI_Sendrecv distributed_sparse.h:351-361,
 * MPI_Allgather 15D_dense_shift.hpp:194, MPI_Reduce_scatter :240, MPI_Alltoallv
 * SpmatLocal.hpp:451, MPI_Barrier, MPI_Comm_split FlexibleGrid.hpp:80-88). */
typedef struct hnhd_external_transport {
    void *ctx;
    int (*sendrecv)(void *ctx, int comm, const void *sbuf, size_t sbytes, int dst, void *rbuf,
                    size_t rbytes, int src);
    int (*allgather)(void *ctx, int comm, const void *sbuf, void *rbuf, size_t bytes_each);
    int (*reduce_scatter_f64)(void *ctx, int comm, const double *sbuf, double *rbuf,
                              size_t count_each);
    int (*allreduce_f64)(void *ctx, int comm, double *buf, size_t count);
    int (*alltoallv)(void *ctx, int comm, const void *sbuf, const size_t *sbytes,
                     const size_t *sdispls, void *rbuf, const size_t *rbytes,
                     const size_t *rdispls);
    int (*barrier)(void *ctx, int comm);
    int (*split)(void *ctx, int comm, int color, int key, int *new_comm, int *new_rank,
                 int *new_size);
} hnhd_external_transport_t;

/* ---- world (replaces MPI_Init / MPI_Finalize, bench_erdos_renyi.cpp:20,120) ---------------- */
int hnhd_init_self(void);
int hnhd_nccl_unique_id(char out[HNHD_NCCL_ID_BYTES]);
int hnhd_init_nccl(int rank, int world_size, const char unique_id[HNHD_NCCL_ID_BYTES]);
int hnhd_init_external(int rank, int world_size, const hnhd_external_transport_t *cb);
int hnhd_finalize(void);
int hnhd_world_rank(void);
int hnhd_world_size(void);
int hnhd_barrier(void);
int hnhd_device_synchronize(void);

/* ---- SpmatLocal ----------------------------------------------------------------------------- */
typedef struct hnhd_spmat hnhd_spmat_t;
/* SpmatLocal::loadTuples(false, logM, nnz_per_row, "") (SpmatLocal.hpp:467-533) with the
 * repo's seeded Erdos-Renyi generator; every rank generates its 1-D row slice. */
int hnhd_spmat_load_er(int logM, int nnz_per_row, uint64_t seed, hnhd_spmat_t **out);
/* SpmatLocal::loadTuples(true, -1, -1, filename): MatrixMarket coordinate file (general / symmetric, real /
 * integer / pattern); every rank keeps a share of the entries (SpmatLocal.hpp:479-491 reads with CombBLAS). */
int hnhd_spmat_load_file(const char *filename, hnhd_spmat_t **out);
/* Arbitrary local tuples of a global M x N matrix (any distribution over the ranks). */
int hnhd_spmat_from_tuples(uint64_t M, uint64_t N, const uint64_t *rows, const uint64_t *cols,
                           const double *vals, int64_t n_local, hnhd_spmat_t **out);
int hnhd_spmat_info(const hnhd_spmat_t *S, uint64_t *M, uint64_t *N, uint64_t *dist_nnz,
                    int64_t *local_tuples);
int hnhd_spmat_tuples(const hnhd_spmat_t *S, uint64_t *rows, uint64_t *cols, double *vals,
                      int64_t capacity);
void hnhd_spmat_destroy(hnhd_spmat_t *S);

/* ---- Distributed_Sparse subclasses ---------------------------------------------------------- */
typedef struct hnhd_alg hnhd_alg_t;
/* name: "15d_fusion1" | "15d_fusion2" | "15d_sparse" | "25d_dense_replicate" |
 * "25d_sparse_replicate"  (the selectors of benchmark_dist.cpp:45-82).  The kernel plugged in
 * is the library's StandardKernel (CUDA). */
int hnhd_alg_create(const char *name, hnhd_spmat_t *S, int R, int c, hnhd_alg_t **out);
void hnhd_alg_destroy(hnhd_alg_t *alg);

typedef struct hnhd_alg_dims {
    int64_t M, N, R;
    int p, c;
    int localArows, localAcols, localBrows, localBcols;
    int64_t s_values, st_values; /* like_S_values / like_ST_values lengths */
    int r_split;
    int grid_i, grid_j, grid_k;
    int n_a_submatrices, n_b_submatrices;
} hnhd_alg_dims_t;
int hnhd_alg_dims(hnhd_alg_t *alg, hnhd_alg_dims_t *out);
/* aSubmatrices / bSubmatrices (distributed_sparse.h:57-58): 4 ints each
 * (topRow, leftCol, rowCount, colCount). which: 0 = A, 1 = B. */
int hnhd_alg_submatrices(hnhd_alg_t *alg, int which, int *out4, int capacity);
/* JSON text of json_algorithm_info() / json_perf_statistics() (distributed_sparse.h:131-179,
 * 245-261).  Collective.  Returns the length written (excluding NUL) or a negative code. */
/* Wall-clock seconds of the setup phases of this process so far (tuple generation, redistribution, COO -> CSR), as
 * a JSON object {phase: seconds}; reset != 0 clears the counters afterwards. */
int hnhd_setup_times_json(char *out, size_t capacity, int reset);
int hnhd_alg_info_json(hnhd_alg_t *alg, char *out, size_t capacity);
int hnhd_alg_perf_json(hnhd_alg_t *alg, char *out, size_t capacity);
int hnhd_alg_reset_timers(hnhd_alg_t *alg);

/* Local CSR blocks of S (which = 0) or ST (which = 1), copied to HOST arrays: for tests.
 * block_count -> number of blocks; for each block: rows, cols, nnz, transpose, is_null. */
int hnhd_alg_block_count(hnhd_alg_t *alg, int which);
int hnhd_alg_block_meta(hnhd_alg_t *alg, int which, int block, int64_t *rows, int64_t *cols,
                        int64_t *nnz, int *transpose, int *is_null);
int hnhd_alg_block_arrays(hnhd_alg_t *alg, int which, int block, int64_t *rowStart,
                          int64_t *col_idx, int64_t *row_idx, double *values);

/* ---- resident dense matrices / value vectors (DenseMatrix / VectorXd on the device) -------- */
typedef struct hnhd_dense hnhd_dense_t;
typedef struct hnhd_vec hnhd_vec_t;
int hnhd_dense_create(int64_t rows, int64_t cols, double value, hnhd_dense_t **out);
int hnhd_dense_like(hnhd_alg_t *alg, int which /*0=A,1=B*/, double value, hnhd_dense_t **out);
int hnhd_dense_fill(hnhd_dense_t *m, double value);
int hnhd_dense_dummy_initialize(hnhd_alg_t *alg, hnhd_dense_t *m, int which); /* :322-346 */
int hnhd_dense_from_host(hnhd_dense_t *m, const double *host); /* rows*cols doubles */
int hnhd_dense_to_host(const hnhd_dense_t *m, double *host);
int hnhd_dense_shape(const hnhd_dense_t *m, int64_t *rows, int64_t *cols);
/* Device pointer of the matrix storage.  NOT stable across operations: spmm / fusedSpMM / ring shifts may return
 * their result by swapping the matrix's storage with an internal buffer (instead of the reference's copy-back,
 * common.h:88-92), after which an earlier pointer refers to recycled memory.  Re-query after every operation. */
void *hnhd_dense_data(hnhd_dense_t *m);
void hnhd_dense_destroy(hnhd_dense_t *m);
int hnhd_vec_create(int64_t n, double value, hnhd_vec_t **out);
int hnhd_vec_like(hnhd_alg_t *alg, int which /*0=S,1=ST*/, double value, hnhd_vec_t **out);
int hnhd_vec_fill(hnhd_vec_t *v, double value);
int hnhd_vec_from_host(hnhd_vec_t *v, const double *host);
int hnhd_vec_to_host(const hnhd_vec_t *v, double *host);
int64_t hnhd_vec_size(const hnhd_vec_t *v);
void hnhd_vec_destroy(hnhd_vec_t *v);

/* ---- the public operations (distributed_sparse.h:266-320) ----------------------------------- */
#define HNHD_OP_SDDMM_A 0
#define HNHD_OP_SDDMM_B 1
#define HNHD_OP_SPMM_A 2
#define HNHD_OP_SPMM_B 3
#define HNHD_OP_FUSED_A 4 /* fusedSpMM(A, B, S, result, Amat) */
#define HNHD_OP_FUSED_B 5
#define HNHD_OP_INITIAL_SHIFT 6 /* aux = KernelMode (0 sddmmA,1 spmmA,2 spmmB,3 sddmmB) */
#define HNHD_OP_DE_SHIFT 7
/* Enqueues the operation (stream-ordered; returns before the GPU finishes).  svals / result
 * may be NULL where the operation does not use them (spmm: result unused). */
int hnhd_alg_op(hnhd_alg_t *alg, int op, hnhd_dense_t *A, hnhd_dense_t *B, hnhd_vec_t *svals,
                hnhd_vec_t *result, int aux);

/* fusedSpMM on HOST operands (Distributed_Sparse::fusedSpMM_host, include/hnh/distributed_sparse.h): hostA / hostB
 * are this rank's local shards in (preferably pinned) host memory, hostOut receives the SpMM result; A and B are
 * the device staging matrices.  mode: 0 = Amat, 1 = Bmat.  chunk_rows > 0 sets the row chunk of the upload /
 * kernel / download pipeline the 1.5D dense-shift algorithm runs on one rank, 0 keeps the default, < 0 turns the
 * pipeline off (copy in, fusedSpMM, copy out).  Returns after hostOut is complete. */
int hnhd_alg_fused_host(hnhd_alg_t *alg, hnhd_dense_t *A, hnhd_dense_t *B, hnhd_vec_t *svals, hnhd_vec_t *result,
                        const double *hostA, const double *hostB, double *hostOut, int mode, int64_t chunk_rows);

/* Edge softmax (Distributed_Sparse::edgeSoftmax): vec becomes, in place, the softmax of its entries over each
 * row of S; mode 0 = A order (hnhd_vec_like(.., 0, ..): sddmmA / spmmA values), 1 = B order (ST values).
 * Backward (edgeSoftmaxBackward): grad = dL/d alpha becomes dL/d(scores) = alpha o (grad - t), with t the row
 * sums of alpha o grad.  Collective, stream-ordered.  HNH_E_INVALID on every rank where a rank does not hold
 * full-width rows (R-split layouts at p > 1; 1.5D dense shift with local kernel fusion at c > 1). */
int hnhd_alg_edge_softmax(hnhd_alg_t *alg, hnhd_vec_t *vec, int mode);
int hnhd_alg_edge_softmax_backward(hnhd_alg_t *alg, const hnhd_vec_t *alpha, hnhd_vec_t *grad, int mode);
/* Additive attention (Distributed_Sparse::additiveScores / edgeSums).  out (a value vector of `mode`, as above)
 * becomes LeakyReLU(s[u] + t[v]) for every stored entry (u, v) of S, or with derivative != 0 its derivative (1
 * where s[u] + t[v] > 0, alpha elsewhere); s and t are whole node vectors (at least M and N entries), indexed by
 * global row and column.  No communication.  edge_sums: row_sums[u] / col_sums[v] become the sums of `values`
 * (A order) over row u / column v of S on all ranks (entries past M / N: 0); collective.  HNH_E_INVALID where
 * hnhd_alg_edge_softmax is. */
int hnhd_alg_additive_scores(hnhd_alg_t *alg, const hnhd_vec_t *s, const hnhd_vec_t *t, hnhd_vec_t *out, int mode,
                             double alpha, int derivative);
int hnhd_alg_edge_sums(hnhd_alg_t *alg, const hnhd_vec_t *values, hnhd_vec_t *row_sums, hnhd_vec_t *col_sums);
/* GATv2 attention (Distributed_Sparse::gatv2Scores / gatv2Backward), with A and B this rank's A- and B-shaped
 * operands (u = S-row, v = S-column), r = a's length wide, and sigma = LeakyReLU(., alpha):
 * gatv2_scores: out (a value vector of `mode`, as above) becomes sum_k a_k sigma(A[u, k] + B[v, k]) for every
 * stored (u, v) of S.  gatv2_backward: with grad_A / grad_B = dL/d scores in the A and B orders, dA += the
 * row-side gradient, dB += the column-side one, and da (resized to r) = the gradient of a summed over all ranks.
 * dA and dB may be the same matrix.  Collective; HNH_E_INVALID where hnhd_alg_edge_softmax is, and for
 * mismatched shapes. */
int hnhd_alg_gatv2_scores(hnhd_alg_t *alg, hnhd_dense_t *A, hnhd_dense_t *B, const hnhd_vec_t *a, hnhd_vec_t *out,
                          int mode, double alpha);
int hnhd_alg_gatv2_backward(hnhd_alg_t *alg, hnhd_dense_t *A, hnhd_dense_t *B, const hnhd_vec_t *a,
                            const hnhd_vec_t *grad_A, const hnhd_vec_t *grad_B, hnhd_dense_t *dA, hnhd_dense_t *dB,
                            hnhd_vec_t *da, double alpha);
/* Fused sparse attention (Distributed_Sparse::sparseAttention / sparseAttentionBackward): per head h of width
 * d = r / heads, Z_u,h = sum over the stored (u, v) of S of softmax_v(scale <Q_u,h, K_v,h>) V_v,h, with Q and Z
 * A-shaped, K and V B-shaped, all r wide; L (localArows x heads, from hnhd_dense_create) receives the rows'
 * log-sum-exp (-inf, and Z = 0, for a row without entries).  The backward, given dZ (A-shaped), overwrites dQ, dK
 * and dV.  S's values are not read.  `scale` must be finite.  Collective; HNH_E_INVALID where hnhd_alg_edge_softmax
 * is, and for mismatched shapes. */
int hnhd_alg_sparse_attention(hnhd_alg_t *alg, hnhd_dense_t *Q, hnhd_dense_t *K, hnhd_dense_t *V, hnhd_dense_t *Z,
                              hnhd_dense_t *L, int heads, double scale);
int hnhd_alg_sparse_attention_backward(hnhd_alg_t *alg, hnhd_dense_t *Q, hnhd_dense_t *K, hnhd_dense_t *V,
                                       hnhd_dense_t *Z, hnhd_dense_t *L, hnhd_dense_t *dZ, hnhd_dense_t *dQ,
                                       hnhd_dense_t *dK, hnhd_dense_t *dV, int heads, double scale);
/* The same with attention dropout of probability `dropout` in [0, 1) (Distributed_Sparse::sparseAttention with
 * dropout and seed): the kept entries' alpha is scaled by 1 / (1 - dropout), L stays the log-sum-exp of all scores,
 * and the mask of head h is that of hnh_sparse_attention_step_dropout_f64 at seed + h and the global S-row and
 * S-column.  The backward must get its forward's dropout and seed, and every rank the same values.  dropout = 0
 * equals the calls above.  HNH_E_INVALID as above, and for dropout outside [0, 1) or NaN. */
int hnhd_alg_sparse_attention_dropout(hnhd_alg_t *alg, hnhd_dense_t *Q, hnhd_dense_t *K, hnhd_dense_t *V,
                                      hnhd_dense_t *Z, hnhd_dense_t *L, int heads, double scale, double dropout,
                                      uint64_t seed);
int hnhd_alg_sparse_attention_backward_dropout(hnhd_alg_t *alg, hnhd_dense_t *Q, hnhd_dense_t *K, hnhd_dense_t *V,
                                               hnhd_dense_t *Z, hnhd_dense_t *L, hnhd_dense_t *dZ, hnhd_dense_t *dQ,
                                               hnhd_dense_t *dK, hnhd_dense_t *dV, int heads, double scale,
                                               double dropout, uint64_t seed);
/* With an additive score bias (Distributed_Sparse::sparseAttention / sparseAttentionBackward with bias pointers):
 * bias / bias_A an A-order vector, bias_B a B-order one, of length n or heads * n; dbias_A / dbias_B nullable.
 * A null bias (both null in the backward) is the call without bias. */
int hnhd_alg_sparse_attention_bias(hnhd_alg_t *alg, hnhd_dense_t *Q, hnhd_dense_t *K, hnhd_dense_t *V, hnhd_dense_t *Z,
                                   hnhd_dense_t *L, int heads, double scale, double dropout, uint64_t seed,
                                   const hnhd_vec_t *bias);
int hnhd_alg_sparse_attention_backward_bias(hnhd_alg_t *alg, hnhd_dense_t *Q, hnhd_dense_t *K, hnhd_dense_t *V,
                                            hnhd_dense_t *Z, hnhd_dense_t *L, hnhd_dense_t *dZ, hnhd_dense_t *dQ,
                                            hnhd_dense_t *dK, hnhd_dense_t *dV, int heads, double scale, double dropout,
                                            uint64_t seed, const hnhd_vec_t *bias_A, const hnhd_vec_t *bias_B,
                                            hnhd_vec_t *dbias_A, hnhd_vec_t *dbias_B);
/* With edge features added to the keys and values (Distributed_Sparse::sparseAttention / sparseAttentionBackward with
 * edge pointers): edge / edge_A an A-order matrix, edge_B a B-order one, each n x r (n the order's local entry
 * count); dedge (nullable) is resized to edge_A's shape and overwritten.  Bias pointers as in the _bias calls,
 * nullable.  A null edge (both null in the backward) is the call without edge features. */
int hnhd_alg_sparse_attention_edge(hnhd_alg_t *alg, hnhd_dense_t *Q, hnhd_dense_t *K, hnhd_dense_t *V, hnhd_dense_t *Z,
                                   hnhd_dense_t *L, int heads, double scale, double dropout, uint64_t seed,
                                   const hnhd_vec_t *bias, const hnhd_dense_t *edge);
int hnhd_alg_sparse_attention_backward_edge(hnhd_alg_t *alg, hnhd_dense_t *Q, hnhd_dense_t *K, hnhd_dense_t *V,
                                            hnhd_dense_t *Z, hnhd_dense_t *L, hnhd_dense_t *dZ, hnhd_dense_t *dQ,
                                            hnhd_dense_t *dK, hnhd_dense_t *dV, int heads, double scale, double dropout,
                                            uint64_t seed, const hnhd_vec_t *bias_A, const hnhd_vec_t *bias_B,
                                            hnhd_vec_t *dbias_A, hnhd_vec_t *dbias_B, const hnhd_dense_t *edge_A,
                                            const hnhd_dense_t *edge_B, hnhd_dense_t *dedge);
/* rows / cols (resized) become the global S-row and S-column of every entry of this rank's value vector of `mode`
 * (0 = A order, 1 = B order) (Distributed_Sparse::entryCoordinates). */
int hnhd_alg_entry_coordinates(hnhd_alg_t *alg, int mode, hnhd_vec_t *rows, hnhd_vec_t *cols);

/* CUDA-event timing on the library's compute stream: start, ..., stop -> milliseconds. */
int hnhd_timer_start(void);
int hnhd_timer_stop(double *ms_out);

/* benchmark_algorithm (benchmark_dist.cpp:26-167): constructs the algorithm, runs
 * `trials` timed FusedMM (or SDDMM+SpMM when fused == 0) calls after `warmup` untimed ones,
 * appends the reference-schema JSON record to output_file on rank 0 (NULL = no file) and
 * returns the record in json_out. */
int hnhd_benchmark_algorithm(hnhd_spmat_t *S, const char *algorithm_name, const char *output_file,
                             int fused, int R, int c, const char *app, int trials, int warmup,
                             char *json_out, size_t capacity);

/* Distributed_ALS on `alg` (als_conjugate_gradients.cpp): artificial ground truth, initializeEmbeddings(),
 * residual, `steps` alternating cg_optimizer(Amat, 10) / cg_optimizer(Bmat, 10) rounds, residual again.
 * out2 = {residual before, residual after} (world-reduced, identical on every rank).  Collective. */
int hnhd_als_residuals(hnhd_alg_t *alg, int steps, double *out2);

/* The same alternating rounds on CALLER inputs, for parity tests against the reference's Distributed_ALS: ground
 * truth = SDDMM of the local shards hostAgt / hostBgt over the all-ones pattern (as the constructor builds it,
 * als_conjugate_gradients.cpp:166-186), embeddings = hostA0 / hostB0 (instead of initializeEmbeddings()'s random
 * draw), `steps` rounds of cg_optimizer(Amat, cg_iters); cg_optimizer(Bmat, cg_iters).  out2 = residual before /
 * after; hostA_out / hostB_out (may be NULL) receive the local embeddings.  Collective. */
int hnhd_als_run(hnhd_alg_t *alg, const double *hostAgt, const double *hostBgt, const double *hostA0,
                 const double *hostB0, int steps, int cg_iters, double *out2, double *hostA_out,
                 double *hostB_out);

/* ---- training (include/hnh/training.hpp): cross-entropy, clipping and AdamW on the device -------------------------
 * Labels of this rank's rows of the model's output buffer (alg's localArows of them), one int32 per row: a class in
 * [0, num_classes) or negative for "ignored" (padding rows and unlabelled nodes must be negative).  Collective: a bad
 * label or count on one rank is refused with HNH_E_INVALID on every rank.  The host array is copied. */
typedef struct hnhd_labels hnhd_labels_t;
int hnhd_labels_create(hnhd_alg_t *alg, const int32_t *host_labels, int64_t n, int num_classes, hnhd_labels_t **out);
void hnhd_labels_destroy(hnhd_labels_t *labels);
/* torch.optim.AdamW(lr, (beta1, beta2), eps, weight_decay, amsgrad=False, foreach=False) with one parameter group, and
 * max_grad_norm > 0: torch.nn.utils.clip_grad_norm_(max_grad_norm) before every step (0: no clipping).  HNH_E_INVALID
 * for lr < 0, a beta outside [0, 1), eps <= 0, weight_decay < 0, max_grad_norm < 0, or any of them NaN or infinite
 * (max_grad_norm may be +inf).  The moments are allocated on the first step; an optimizer is tied to the parameter
 * sizes of its first model, and a train step with another is refused.  set_lr changes lr from the next step on. */
typedef struct hnhd_adamw hnhd_adamw_t;
int hnhd_adamw_create(double lr, double beta1, double beta2, double eps, double weight_decay, double max_grad_norm,
                      hnhd_adamw_t **out);
int hnhd_adamw_set_lr(hnhd_adamw_t *opt, double lr);
void hnhd_adamw_destroy(hnhd_adamw_t *opt);

/* ---- link prediction: a dot-product edge decoder with binary cross-entropy (Distributed_Sparse::linkLoss) ---------
 * On the algorithm object of a target matrix T (its stored values are the targets y_uv in [0, 1]; an SDDMM, SpMM or
 * FusedMM on that object overwrites them): s_uv = <H_A[u], H_B[v]> for every stored (u, v), with H_A A-shaped and H_B
 * B-shaped (one matrix may be both), and the mean of F.binary_cross_entropy_with_logits over T's entries on all ranks.
 * out = {loss, correct, count}: the mean loss, the entries with (s > 0) == (y > 0.5), and T's entry count over all
 * ranks (0 loss and gradient when there is none).  dH_A, dH_B (nullable) are overwritten with the gradients of the
 * mean loss (the sum of both when they are one matrix); scores (nullable, of hnhd_vec_like(T, 0) length) = s in the A
 * order.  The targets are not checked here (hnhd_link_targets_create does).  Collective; HNH_E_INVALID on every rank
 * where hnhd_alg_edge_softmax is, and for mismatched shapes or a gradient that is an H. */
int hnhd_alg_link_loss(hnhd_alg_t *T, hnhd_dense_t *H_A, hnhd_dense_t *H_B, hnhd_dense_t *dH_A, hnhd_dense_t *dH_B,
                       hnhd_vec_t *scores, double out[3]);
/* The link targets of a model (hnh::LinkTargets): T's algorithm object, of the model's layout (algorithm, fusion, p,
 * c, M = N, local rows).  Collective; HNH_E_INVALID on every rank for another layout, a T that is not square or a
 * target outside [0, 1] (NaN included) on any rank.  Both algorithm objects must outlive it. */
typedef struct hnhd_link_targets hnhd_link_targets_t;
int hnhd_link_targets_create(hnhd_alg_t *model, hnhd_alg_t *T, hnhd_link_targets_t **out);
void hnhd_link_targets_destroy(hnhd_link_targets_t *t);

/* ---- relation-aware link prediction: a DistMult edge decoder (Distributed_Sparse::distmultLoss) --------------------
 * On the algorithm object of a target matrix T whose stored values are relations in [0, num_relations) (any other value
 * contributes nothing): s_uv = sum_k H_A[u, k] D[rho, k] H_B[v, k] for every stored (u, v) of relation rho, D the
 * num_relations x r relation table (the same on every rank), and the binary cross-entropy of s against `target` in
 * [0, 1], each entry weighted by inv_count.  out = {loss sum, correct} of this call over all ranks.  dH_A, dH_B, dD
 * (nullable) receive the gradients of the weighted loss, overwritten or, with accumulate != 0, added to; scores (nullable,
 * of hnhd_vec_like(T, 0) length) = s in the A order.  Collective; HNH_E_INVALID on every rank where hnhd_alg_link_loss
 * is, for num_relations < 1, a D or dD that is not num_relations x r, a target outside [0, 1], and a gradient that is an
 * input. */
int hnhd_alg_distmult_loss(hnhd_alg_t *T, hnhd_dense_t *H_A, hnhd_dense_t *H_B, hnhd_dense_t *D, int num_relations, double target,
                           double inv_count, hnhd_dense_t *dH_A, hnhd_dense_t *dH_B, hnhd_dense_t *dD, hnhd_vec_t *scores,
                           int accumulate, double out[2]);
/* The DistMult decoder of a model (hnh::DistMultDecoder, include/hnh/distmult.hpp): its relation table "rel"
 * (num_relations x width, zero after creation; PyG's rel_emb with no transpose) and, after a relational train step, its
 * gradient.  model: the model's algorithm object; width: the model's output width. */
typedef struct hnhd_distmult hnhd_distmult_t;
int hnhd_distmult_create(hnhd_alg_t *model, int num_relations, int width, hnhd_distmult_t **out);
void hnhd_distmult_destroy(hnhd_distmult_t *d);
int hnhd_distmult_param_shape(hnhd_distmult_t *d, const char *name, int64_t *rows, int64_t *cols);
int hnhd_distmult_set_param(hnhd_distmult_t *d, const char *name, const double *host);
int hnhd_distmult_get_param(hnhd_distmult_t *d, const char *name, double *host);
int hnhd_distmult_get_param_grad(hnhd_distmult_t *d, const char *name, double *host);
/* The relational link targets of a model (hnh::RelationalLinkTargets): T_pos (target 1) and T_neg (target 0; it may
 * have no entry), each an algorithm object of the model's layout whose stored values are relations in [0,
 * num_relations).  Collective; HNH_E_INVALID on every rank for another layout, a T that is not square, num_relations <
 * 1 or a stored value that is no relation on any rank.  The three algorithm objects must outlive it. */
typedef struct hnhd_relational_link_targets hnhd_relational_link_targets_t;
int hnhd_relational_link_targets_create(hnhd_alg_t *model, hnhd_alg_t *T_pos, hnhd_alg_t *T_neg, int num_relations,
                                        hnhd_relational_link_targets_t **out);
void hnhd_relational_link_targets_destroy(hnhd_relational_link_targets_t *t);

/* ---- max aggregation (Distributed_Sparse::maxAggregate) -------------------------------------------------------------
 * Z, C (A-shaped, f wide) = the per-column maximum of X (B-shaped) over the stored entries of each S-row and the number
 * of entries that attain it; Z = C = 0 on a row without entries.  The backward overwrites dX (or adds to it with
 * accumulate != 0) with sum_u [X_v == Z_u] dZ_u / C_u.  Collective; HNH_E_INVALID on every rank where
 * hnhd_alg_edge_softmax is, for wrong shapes, and for an output that is another operand. */
int hnhd_alg_max_aggregate(hnhd_alg_t *a, hnhd_dense_t *X, hnhd_dense_t *Z, hnhd_dense_t *C);
int hnhd_alg_max_aggregate_backward(hnhd_alg_t *a, hnhd_dense_t *X, hnhd_dense_t *Z, hnhd_dense_t *C, hnhd_dense_t *dZ,
                                    hnhd_dense_t *dX, int accumulate);

/* ---- multi-statistic aggregation (Distributed_Sparse::multiAggregate) ----------------------------------------------
 * which: a non-empty union of HNH_MULTI_MOMENTS (1), HNH_MULTI_MAX (2) and HNH_MULTI_MIN (4).  A (A-shaped, W f wide with
 * W = 2 per selected flag) = the selected windows of [sum_v X_v | sum_v X_v^2 | max_v X_v | #ties | min_v X_v | #ties]
 * over the stored entries (u, v) of each S-row (X B-shaped, f wide), 0 on a row without entries.  The backward overwrites
 * dX (or adds to it with accumulate != 0) with sum_u dA_sum[u] + 2 X_v dA_sq[u] + [X_v == max_u] dA_max[u] / C_max[u] +
 * [X_v == min_u] dA_min[u] / C_min[u], dA in A's layout (its count windows are not read).  Collective; HNH_E_INVALID on
 * every rank where hnhd_alg_edge_softmax is, for an empty or unknown `which`, W f >= 2^31, wrong shapes, and for an
 * output that is another operand. */
int hnhd_alg_multi_aggregate(hnhd_alg_t *a, hnhd_dense_t *X, hnhd_dense_t *A, int which);
int hnhd_alg_multi_aggregate_backward(hnhd_alg_t *a, hnhd_dense_t *X, hnhd_dense_t *A, hnhd_dense_t *dA, hnhd_dense_t *dX, int which,
                                      int accumulate);

/* ---- edge-ReLU aggregation (Distributed_Sparse::edgeReluAggregate, GINE) ----------------------------------------------
 * A (A-shaped, f wide) = sum_i ReLU(X_v + E_A,i) over the stored entries i = (u, v) of each S-row (X B-shaped, f wide;
 * 0 on a row without entries).  E_A / E_B are per-entry rows of the A / B value orders (len(like_S_values) /
 * len(like_ST_values) x f, rows in the order of hnhd_alg_entry_coordinates) holding the same e(u, v) in both.  The
 * backward overwrites dX (or adds to it with accumulate != 0) with sum_i [X_v + E_i > 0] dA_u and, unless dE_A is null,
 * sets dE_A (resized to E_A's shape) to [X_v + E_i > 0] dA_u per entry of the A order.  Collective; HNH_E_INVALID on
 * every rank where hnhd_alg_edge_softmax is, for wrong shapes, only one of E_A / E_B, and an output that is another
 * operand. */
int hnhd_alg_edge_relu_aggregate(hnhd_alg_t *a, hnhd_dense_t *X, hnhd_dense_t *E_A, hnhd_dense_t *A);
int hnhd_alg_edge_relu_aggregate_backward(hnhd_alg_t *a, hnhd_dense_t *X, hnhd_dense_t *E_A, hnhd_dense_t *E_B, hnhd_dense_t *dA,
                                          hnhd_dense_t *dX, hnhd_dense_t *dE_A, int accumulate);

/* ---- relational aggregation (Distributed_Sparse::relationalAggregate) -----------------------------------------------
 * A (A-shaped, num_relations * f wide) = for each S-row u and relation rho, the sum of X_v (B-shaped, f wide) over the
 * stored entries (u, v) whose value is rho (0 where there are none; entries whose value is not an integer in
 * [0, num_relations) count nowhere).  The backward overwrites dX (or adds to it with accumulate != 0) with
 * dX_v = sum over the stored (u, v) of dA[u, rho f .. rho f + f).  Collective; HNH_E_INVALID on every rank where
 * hnhd_alg_edge_softmax is, for num_relations < 1, wrong shapes, and for an output that is another operand. */
int hnhd_alg_relational_aggregate(hnhd_alg_t *a, hnhd_dense_t *X, hnhd_dense_t *A, int num_relations);
int hnhd_alg_relational_aggregate_backward(hnhd_alg_t *a, hnhd_dense_t *dA, hnhd_dense_t *dX, int num_relations, int accumulate);

/* ---- basis aggregation (Distributed_Sparse::basisAggregate) ----------------------------------------------------------
 * hnhd_alg_basis_aggregate: H (A-shaped, B f wide, B = comp's columns) = for each S-row u and basis b, the sum over the
 * stored entries (u, v) of scale[u, rho] comp[rho, b] X_v (X B-shaped, f wide; comp R x B; scale A-shaped and R wide,
 * or null for ones).  hnhd_alg_basis_aggregate_backward: dX (overwritten, or added to with accumulate != 0) =
 * sum over the stored (u, v) of scale[u, rho] sum_b comp[rho, b] dH[u, b f .. b f + f), and dcomp (R x B, overwritten,
 * the same on every rank) = sum over the stored entries of relation rho on all ranks of scale[u, rho]
 * <dH[u, b f .. b f + f), X_v>.  Collective; HNH_E_INVALID on every rank where hnhd_alg_edge_softmax is, for
 * num_relations < 1, B < 1, wrong shapes, and for an output that is another operand. */
int hnhd_alg_basis_aggregate(hnhd_alg_t *a, hnhd_dense_t *X, hnhd_dense_t *H, hnhd_dense_t *comp, int num_relations,
                             hnhd_dense_t *scale);
int hnhd_alg_basis_aggregate_backward(hnhd_alg_t *a, hnhd_dense_t *dH, hnhd_dense_t *X, hnhd_dense_t *dX, hnhd_dense_t *comp,
                                      hnhd_dense_t *dcomp, int num_relations, hnhd_dense_t *scale, int accumulate);

/* ---- graph models: GAT, the graph transformer, GraphSAGE and R-GCN behind one handle ---------------------------------
 * The constructors below return an hnhd_model_t; every hnhd_model_* call takes any of them, the GAT and graph transformer
 * calls below only a model of their kind (another kind is refused with HNH_E_INVALID).  A model keeps a pointer to its `alg`,
 * which must outlive it.  Buffers: 0 is the network input (B-shaped), i + 1 the output of layer i (A-shaped), this
 * rank's rows.  Parameters are zero after construction unless stated otherwise.  Changing a parameter, the input (or a
 * model's own state: GAT's attention, the graph transformer's edge attributes) makes the activations stale; a backward
 * pass on stale activations, and a gradient read before the first backward pass, are refused with HNH_E_INVALID.
 * Gradients of parameters are summed over all ranks (identical on every rank).  Forward, backward and the steps are
 * collective and refuse, on every rank before any launch, a layout the model does not support. */
typedef struct hnhd_model hnhd_model_t;
int hnhd_model_buffer_shape(hnhd_model_t *m, int buffer, int64_t *rows, int64_t *cols);
int hnhd_model_set_input(hnhd_model_t *m, const double *host);         /* buffer 0 */
int hnhd_model_get_buffer(hnhd_model_t *m, int buffer, double *host);  /* synchronises */
/* Forward pass with attention dropout `dropout` in [0, 1) and `seed` (the graph transformer; every rank passes the same
 * values).  The other models have no dropout and refuse dropout != 0.  Stream-ordered. */
int hnhd_model_forward(hnhd_model_t *m, double dropout, uint64_t seed);
/* host_output_grad = dL/d(the last buffer), this rank's rows, in the shape hnhd_model_buffer_shape reports for it */
int hnhd_model_backward(hnhd_model_t *m, const double *host_output_grad);
/* dL/d buffer 0 (this rank's rows) after hnhd_model_backward */
int hnhd_model_get_input_grad(hnhd_model_t *m, double *host);
/* A parameter by layer and name (see the models below): rows x cols doubles, row-major.  get_param synchronises;
 * get_param_grad reads dL/d param after hnhd_model_backward.  GAT has no parameters by name and refuses: its weights and
 * attention vectors are read and written by (layer, head) with the GAT calls below. */
int hnhd_model_param_shape(hnhd_model_t *m, int layer, const char *name, int64_t *rows, int64_t *cols);
int hnhd_model_set_param(hnhd_model_t *m, int layer, const char *name, const double *host);
int hnhd_model_get_param(hnhd_model_t *m, int layer, const char *name, double *host);
int hnhd_model_get_param_grad(hnhd_model_t *m, int layer, const char *name, double *host);
/* One training step: forward(dropout, seed), the mean cross-entropy of the output buffer against the labels over all
 * ranks, the backward pass, clipping and AdamW.  out = {loss, correct, labelled, grad_norm}: the loss, the labelled rows
 * whose argmax is their label and the labelled rows (all ranks), and the gradient norm before clipping.  With no
 * labelled row the loss and the gradient are 0.  Collective; afterwards the activations are stale.  HNH_E_INVALID on
 * every rank before any launch for labels of another row or class count, an optimizer of other parameter sizes,
 * dropout on a model without it, and layouts without a backward pass. */
int hnhd_model_train_step(hnhd_model_t *m, const hnhd_labels_t *labels, hnhd_adamw_t *opt, double dropout, uint64_t seed,
                          double out[4]);
/* One link-prediction training step: forward(dropout, seed), the mean binary cross-entropy of the output buffer's
 * dot-product scores over T's entries, the backward pass, clipping and AdamW.  out = {loss, correct, count, grad_norm}.
 * GAT's last layer keeps its ReLU, so its scores are >= 0; the other models' last layers have none.  Collective;
 * HNH_E_INVALID on every rank before any launch for targets of another model's algorithm object, an optimizer of other
 * parameter sizes, dropout on a model without it, and layouts without a backward pass. */
int hnhd_model_link_train_step(hnhd_model_t *m, const hnhd_link_targets_t *t, hnhd_adamw_t *opt, double dropout,
                               uint64_t seed, double out[4]);
/* A forward pass without dropout and the link loss without gradients: out = {loss, correct, count}; scores (nullable)
 * is resized and receives s in the A order of T (hnhd_alg_entry_coordinates(T, 0, ..) gives the pairs).  Collective. */
int hnhd_model_link_evaluate(hnhd_model_t *m, const hnhd_link_targets_t *t, hnhd_vec_t *scores, double out[3]);
/* One relational link-prediction step (hnh::relationalLinkTrainStep): forward(dropout, seed), the mean binary
 * cross-entropy of the DistMult scores over the pairs of T_pos and T_neg, the backward pass, clipping and AdamW over the
 * model's parameters and then the decoder's.  out = {loss, correct, pair count, grad_norm}.  Collective; HNH_E_INVALID on
 * every rank before any launch for targets or a decoder of another model's algorithm object, a decoder of another
 * relation count or width, an optimizer of other parameter sizes, dropout on a model without it, and layouts without a
 * backward pass. */
int hnhd_model_relational_link_train_step(hnhd_model_t *m, hnhd_distmult_t *d, const hnhd_relational_link_targets_t *t,
                                          hnhd_adamw_t *opt, double dropout, uint64_t seed, double out[4]);
/* A forward pass without dropout and the relational link loss without gradients: out = {loss, correct, pair count};
 * scores_pos / scores_neg (nullable) are resized and receive s in the A order of T_pos / T_neg.  Collective. */
int hnhd_model_relational_link_evaluate(hnhd_model_t *m, hnhd_distmult_t *d, const hnhd_relational_link_targets_t *t,
                                        hnhd_vec_t *scores_pos, hnhd_vec_t *scores_neg, double out[3]);
/* Filtered link ranking (include/hnh/link_ranking.hpp).  A ranking holds the filter F, the known triples (heads[i],
 * rels[i], tails[i]), i < n, of a model's nodes (model: the model's algorithm object).  Collective; HNH_E_INVALID on
 * every rank for a layout without full rows, num_relations < 1, a node outside [0, M), a relation outside
 * [0, num_relations) or triples that differ between ranks.  hnhd_model_link_rank: forward without dropout, then the
 * filtered tail and head ranks of the n_q query triples (host arrays of n_q doubles, the same on every rank) by the
 * DistMult scores of decoder d, or by dot products when d is null (the ranking then has 1 relation); *mrr = the mean
 * of 1 / rank over the 2 n_q ranks.  Collective; HNH_E_INVALID on every rank before any launch for a ranking or
 * decoder of another model's algorithm object, a decoder of another relation count or width, a null decoder with
 * num_relations != 1, and queries that are out of range on any rank or differ between ranks. */
typedef struct hnhd_link_ranking hnhd_link_ranking_t;
int hnhd_link_ranking_create(hnhd_alg_t *model, const int64_t *heads, const int64_t *rels, const int64_t *tails, int64_t n,
                             int num_relations, hnhd_link_ranking_t **out);
void hnhd_link_ranking_destroy(hnhd_link_ranking_t *r);
int hnhd_model_link_rank(hnhd_model_t *m, const hnhd_link_ranking_t *ranking, hnhd_distmult_t *d, const int64_t *heads,
                         const int64_t *rels, const int64_t *tails, int64_t n_q, double *tail_ranks, double *head_ranks, double *mrr);
void hnhd_model_destroy(hnhd_model_t *m);

/* ---- graph-level prediction (include/hnh/graph_readout.hpp) ---------------------------------------------------------
 * A readout of a model: batch (n = the model's localArows entries) gives the graph of each of this rank's output rows,
 * in [0, num_graphs) or negative for none (padding rows must be negative); pool is "sum", "mean" or "max";
 * num_classes = 0 pools without a head (the logits are the pooled rows, so the class count is the output width r),
 * > 0 adds a Linear(r, num_classes) head with the parameters "weight" (r x C) and "bias" (C x 1), zero after
 * construction.  Collective; HNH_E_INVALID on every rank before any launch for a layout where check_full_rows fails,
 * a batch of another length, num_graphs < 1, num_graphs or num_graphs r >= 2^31, an id >= num_graphs or on a padding
 * row on any rank, a graph count differing between ranks, an unknown pool and num_classes < 0.  The model must
 * outlive the readout. */
typedef struct hnhd_readout hnhd_readout_t;
int hnhd_readout_create(hnhd_model_t *m, const int64_t *batch, int64_t n, int64_t num_graphs, const char *pool, int num_classes,
                        hnhd_readout_t **out);
void hnhd_readout_destroy(hnhd_readout_t *r);
/* P (resized to num_graphs x r) = the pool of H (the model's output shape) over all ranks.  Collective. */
int hnhd_readout_pool(hnhd_readout_t *r, hnhd_dense_t *H, hnhd_dense_t *P);
/* dH (resized to H's shape) = dL/dH given dP = dL/dP (num_graphs x r, the same on every rank), for the H of the last
 * pool (max reads that pool's maxima and counts).  No communication. */
int hnhd_readout_pool_backward(hnhd_readout_t *r, hnhd_dense_t *H, hnhd_dense_t *dP, hnhd_dense_t *dH);
/* the head's parameters by name; HNH_E_INVALID without a head or for another name, and for a gradient before a graph
 * train step */
int hnhd_readout_param_shape(hnhd_readout_t *r, const char *name, int64_t *rows, int64_t *cols);
int hnhd_readout_set_param(hnhd_readout_t *r, const char *name, const double *host);
int hnhd_readout_get_param(hnhd_readout_t *r, const char *name, double *host);
int hnhd_readout_get_param_grad(hnhd_readout_t *r, const char *name, double *host);
/* The labels of a readout's num_graphs graphs, in [0, num_classes) or negative for "ignored", the same on every rank.
 * Collective; HNH_E_INVALID on every rank for n != num_graphs, num_classes other than the logits' width, a label >=
 * num_classes, or labels differing between ranks. */
typedef struct hnhd_graph_labels hnhd_graph_labels_t;
int hnhd_graph_labels_create(hnhd_readout_t *r, const int32_t *host_labels, int64_t n, int num_classes, hnhd_graph_labels_t **out);
void hnhd_graph_labels_destroy(hnhd_graph_labels_t *l);
/* One graph-classification step: forward(dropout, seed), pool, head, the mean cross-entropy over the labelled graphs,
 * the backward pass, clipping and AdamW over the model's parameters and then the head's.  out = {loss, correct,
 * labelled graphs, grad_norm}.  Collective; HNH_E_INVALID on every rank before any launch for a readout of another
 * model, labels of another readout, an optimizer of other parameter sizes, dropout on a model without it, and layouts
 * without a backward pass. */
int hnhd_model_graph_train_step(hnhd_model_t *m, hnhd_readout_t *r, const hnhd_graph_labels_t *labels, hnhd_adamw_t *opt,
                                double dropout, uint64_t seed, double out[4]);
/* A forward pass without dropout, the readout and the loss without gradients: out = {loss, correct, labelled graphs};
 * host_logits (nullable) receives the num_graphs x C logits, row-major.  Collective. */
int hnhd_model_graph_evaluate(hnhd_model_t *m, hnhd_readout_t *r, const hnhd_graph_labels_t *labels, double *host_logits,
                              double out[3]);

/* ---- GAT (include/hnh/gat.hpp; reference gat.hpp:26-113) --------------------------------------------------------------
 * layers3: n_layers triples (input_features, features_per_head, num_heads).  Weights are input_width x head_width,
 * row-major, as hnhd_gat_weight_shape reports.  The backward pass is refused on every rank where the layout has none
 * (R-split layouts at p > 1; 1.5D dense shift with local kernel fusion at c > 1). */
int hnhd_gat_create(hnhd_alg_t *alg, int n_layers, const int *layers3, double leaky_relu_alpha, hnhd_model_t **out);
int hnhd_gat_weight_shape(hnhd_model_t *g, int layer, int head, int64_t *rows, int64_t *cols);
int hnhd_gat_set_weight(hnhd_model_t *g, int layer, int head, const double *host);
int hnhd_gat_get_weight(hnhd_model_t *g, int layer, int head, double *host); /* synchronises (e.g. after train steps) */
/* dL/d weight (layer, head) after hnhd_model_backward; hnhd_gat_weight_shape's shape */
int hnhd_gat_get_weight_grad(hnhd_model_t *g, int layer, int head, double *host);
/* attention of every head (GAT::set_attention): "leaky" (the default: LeakyReLU of the scores, the
 * reference's formula), "softmax" (their edge softmax over each row of S) or "additive" (below).  Makes the
 * activations stale.
 * With "softmax" the forward pass raises HNH_E_INVALID on every rank, before any launch, where the layout has
 * no edge softmax (as hnhd_alg_edge_softmax). */
int hnhd_gat_set_attention(hnhd_model_t *g, const char *kind);
/* "gatv2": x_uv = a1 . LeakyReLU(h_u + h_v) (GATv2 with shared weights, Brody, Alon and Yahav 2022), then the edge
 * softmax; a1 is set with hnhd_gat_set_attention_vectors (a2 is not read, its gradient stays zero).  Defined on
 * the layouts where "softmax" is. */
/* additive attention ("additive": x_uv = LeakyReLU(a1 . h_u + a2 . h_v) with h = X W the head's projection,
 * then the edge softmax; Velickovic et al. 2018): the attention vectors of (layer, head), features_per_head
 * doubles each (host pointers; zero after hnhd_gat_create: uniform attention).  Makes the activations stale.
 * "additive" is defined on the layouts where "softmax" is. */
int hnhd_gat_set_attention_vectors(hnhd_model_t *g, int layer, int head, const double *a1, const double *a2);
int hnhd_gat_get_attention_vectors(hnhd_model_t *g, int layer, int head, double *a1, double *a2); /* synchronises */
/* dL/d a1 and dL/d a2 of (layer, head) after hnhd_model_backward (features_per_head doubles each, summed over all
 * ranks; zero unless the attention reads them).  HNH_E_INVALID before the first backward pass. */
int hnhd_gat_get_attention_grads(hnhd_model_t *g, int layer, int head, double *da1, double *da2);

/* ---- graph transformer (include/hnh/graph_transformer.hpp): TransformerConv layers on fused sparse attention ---
 * layers3: n_layers triples (input_features, features_per_head, num_heads); every layer concatenates its heads, so
 * layer i + 1 takes features_per_head * num_heads of layer i.  edge_dim > 0 adds edge features (attributes of S's
 * entries projected by each layer's "edge" weight onto the keys and values), beta != 0 the gated skip connection.
 * HNH_E_INVALID on every rank, before any launch, where the layout has no fused sparse attention (as
 * hnhd_alg_edge_softmax), and for bad layer sizes. */
int hnhd_gt_create(hnhd_alg_t *alg, int n_layers, const int *layers3, int edge_dim, int beta, hnhd_model_t **out);
/* The same with transformer blocks: ffn_ratio = k >= 1 makes every layer a post-norm block, LN2(H1 + FFN(H1)) with
 * H1 = LN1(the layer's output without ReLU) and a ReLU FFN of hidden width k r; LayerNorm epsilon norm_eps.  ffn_ratio
 * = 0 is hnhd_gt_create.  HNH_E_INVALID for ffn_ratio < 0 or a norm_eps that is not finite and > 0. */
int hnhd_gt_create_block(hnhd_alg_t *alg, int n_layers, const int *layers3, int edge_dim, int beta, int ffn_ratio,
                         double norm_eps, hnhd_model_t **out);
/* Parameters by layer and name: "query", "key", "value", "skip" (input_features x r, row-major: the transpose of
 * PyG's lin_*.weight), "query_bias", "key_bias", "value_bias", "skip_bias" (r x 1), "edge" (edge_dim x r; models
 * with edge features only), "beta" (3r x 1, the weight of PyG's lin_beta; gated models only).  Models with blocks
 * (ffn_ratio > 0, hidden width h) add "norm1", "norm1_bias" (r x 1; LN1's weight and bias), "ffn1" ((r + 1) x h:
 * lin1.weight^T with lin1.bias as the last row), "ffn2" ((h + 1) x r), "norm2", "norm2_bias".  The LayerNorm weights
 * start at 1.  Layer l of the forward pass uses the dropout seed seed + the heads of the layers before it; the backward
 * pass regenerates the forward's masks.  The forward refuses a bad dropout and a model with edge features whose
 * attributes were not set. */
/* Edge attributes of this rank's entries in both value orders: attr_A is n_A x edge_dim in the order of
 * hnhd_vec_like(.., 0, ..) (hnhd_alg_entry_coordinates mode 0), attr_B n_B x edge_dim in the B order; n_A and n_B
 * must be this rank's entry counts.  Both hold the same attribute for every stored (u, v).  Makes the activations
 * stale.  HNH_E_INVALID for a model without edge features or wrong counts. */
int hnhd_gt_set_edge_attributes(hnhd_model_t *g, const double *attr_A, int64_t n_A, const double *attr_B, int64_t n_B);

/* ---- GraphSAGE (include/hnh/graph_sage.hpp) ----------------------------------------------------------------------
 * Layers of PyG's SAGEConv(aggr, root_weight = True): layers2 = {input_features, output_features} per layer; aggr is
 * "mean", "sum" or "max".  Every layer but the last ends in a ReLU.  Parameters by layer and name: "neigh"
 * (input_features x r: lin_l.weight.T), "neigh_bias" (r x 1: lin_l.bias), "root" (input_features x r: lin_r.weight.T).
 * HNH_E_INVALID on every rank before any launch where hnhd_alg_edge_softmax is, for unknown aggregations, non-positive
 * sizes and widths that do not chain. */
int hnhd_sage_create(hnhd_alg_t *alg, int n_layers, const int *layers2, const char *aggr, hnhd_model_t **out);

/* ---- GIN and GINE (include/hnh/gin.hpp) ------------------------------------------------------------------------------
 * Layers of PyG's GINConv(nn, eps, train_eps), or GINEConv(nn, eps, train_eps, edge_dim) with edge_dim > 0, where nn =
 * Sequential(Linear(f, h), ReLU(), Linear(h, r)): layers3 = {f, h, r} per layer.  Every layer but the last ends in a
 * ReLU.  Parameters by layer and name: "lin1" (f x h: nn.0.weight.T), "lin1_bias" (h x 1), "lin2" (h x r: nn.2.weight.T),
 * "lin2_bias" (r x 1), with edge features "edge" (edge_dim x f: lin.weight.T) and "edge_bias" (f x 1), and "eps" (1 x 1;
 * trained only with train_eps != 0).  hnhd_gin_set_edge_attributes is hnhd_gt_set_edge_attributes for a GIN handle
 * and refuses any other.  Collective; HNH_E_INVALID on every rank before any launch where hnhd_alg_edge_softmax is,
 * for non-positive sizes, widths that do not chain, a negative edge_dim and a non-finite eps. */
int hnhd_gin_create(hnhd_alg_t *alg, int n_layers, const int *layers3, int edge_dim, double eps, int train_eps, hnhd_model_t **out);
int hnhd_gin_set_edge_attributes(hnhd_model_t *g, const double *attr_A, int64_t n_A, const double *attr_B, int64_t n_B);

/* ---- PNA (include/hnh/pna.hpp) --------------------------------------------------------------------------------------
 * Layers of PyG's PNAConv(towers = 1, pre_layers = 1, post_layers = 1, divide_input = False, edge_dim = None):
 * layers2 = {input_features, output_features} per layer; aggregators is a comma-separated, order-preserving list of
 * mean, sum, min, max, var, std and scalers one of identity, amplification, attenuation, linear, inverse_linear;
 * avg_deg_lin and avg_deg_log are PyG's averages of d and log(d + 1) over the degree histogram (read only when a scaler
 * uses them; NaN is refused always, and marks a histogram the caller refused).  Every layer but the last ends in a ReLU.  Parameters by layer and name: "pre" (2f x f:
 * pre_nns.0.0.weight.T), "pre_bias" (f x 1), "post" ((A S + 1) f x r: post_nns.0.0.weight.T), "post_bias" (r x 1),
 * "lin" (r x r: lin.weight.T), "lin_bias" (r x 1).  Collective; HNH_E_INVALID on every rank before any launch where
 * hnhd_alg_edge_softmax is, for an empty, unknown or repeated aggregator or scaler, a NaN average, an average a scaler
 * uses that is not finite and > 0, non-positive sizes, widths that do not chain, (A S + 1) f >= 2^31, and arguments that differ between
 * ranks. */
int hnhd_pna_create(hnhd_alg_t *alg, int n_layers, const int *layers2, const char *aggregators, const char *scalers,
                    double avg_deg_lin, double avg_deg_log, hnhd_model_t **out);

/* ---- R-GCN (include/hnh/rgcn.hpp) ----------------------------------------------------------------------------------
 * Layers of PyG's RGCNConv(in, out, num_relations, aggr, root_weight = True, bias = True) without basis or block
 * decomposition: layers2 = {input_features, output_features} per layer; aggr is "mean" or "sum".  The relation of each
 * stored entry of S is its stored value, an integer in [0, num_relations); create refuses any other value on any rank.
 * Every layer but the last ends in a ReLU.  Parameters by layer and name: "weight" (num_relations * input_features x r:
 * RGCNConv.weight reshaped, no transpose), "bias" (r x 1), "root" (input_features x r).  HNH_E_INVALID on every rank
 * before any launch where hnhd_alg_edge_softmax is, for unknown aggregations, num_relations < 1, non-positive sizes,
 * widths that do not chain and R f >= 2^31.
 * hnhd_rgcn_create_bases: the same with PyG's num_bases = B >= 1: W_rho = sum_b comp[rho, b] V_b.  Parameters by layer
 * and name: "weight" (B f x r: RGCNConv.weight.reshape(-1, r)), "comp" (R x B), "bias" and "root" as without bases.
 * Refuses num_bases < 1 and B f or R B >= 2^31 besides what hnhd_rgcn_create refuses. */
int hnhd_rgcn_create(hnhd_alg_t *alg, int n_layers, const int *layers2, int num_relations, const char *aggr,
                     hnhd_model_t **out);
int hnhd_rgcn_create_bases(hnhd_alg_t *alg, int n_layers, const int *layers2, int num_relations, int num_bases,
                           const char *aggr, hnhd_model_t **out);

#ifdef __cplusplus
}
#endif
#endif /* HNH_B200_DRIVER_H */
