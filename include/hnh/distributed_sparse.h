// hnh/distributed_sparse.h -- Distributed_Sparse, the abstract base of the 1.5D / 2.5D
// algorithms (reference distributed_sparse.h:32-388): public operation facade (sddmmA/B,
// spmmA/B, fusedSpMM), layout descriptors, perf counters and the dense ring-shift helper.
//
// H100-native differences:
//   * dense matrices and value vectors live in HBM; every operation is enqueued on
//     hnh::Runtime's streams and returns without waiting for the GPU;
//   * the ring shift is a grouped NCCL send/recv on the communication stream
//     (reference: blocking MPI_Sendrecv from MPI_ANY_SOURCE + a world barrier,
//     distributed_sparse.h:351-361, 15D_dense_shift.hpp:353-356).  NCCL has no ANY_SOURCE: the
//     source is the rank whose destination is this rank (explicit `recv_src`);
//   * `DenseRing` overlaps the transfer of step t+1 with the kernel of step t whenever the
//     riding matrix is only READ by the kernel, using three buffers so the caller's matrix is
//     never overwritten and the last, home-bound shift of the reference is not needed;
//   * perf counters are CUDA-event spans on the stream each region runs on; the reference's
//     keys and JSON schema are kept (distributed_sparse.h:131-179,205-261).
#pragma once
#include <cassert>
#include <functional>
#include <map>
#include <memory>
#include <string>
#include <vector>

#include "hnh/FlexibleGrid.hpp"
#include "hnh/SpmatLocal.hpp"
#include "hnh/common.h"
#include "hnh/json.h"
#include "hnh/peer_ring.h"
#include "hnh/sparse_kernels.h"

class DenseSubmatrix {
public:
    int topRow, leftCol, rowCount, colCount;
    DenseSubmatrix(int tR, int lC, int rC, int cC) : topRow(tR), leftCol(lC), rowCount(rC), colCount(cC) {}
};

class Distributed_Sparse;

// The entries of a value order grouped by relation, block by block: for block b with entries, an edge-softmax plan
// (hnh_edge_softmax_plan) of its entries over R + 1 keys, key R holding the entries that are no relation.  Built by
// Distributed_Sparse::relationPlan from the stored values as they are then; distmultLoss's relation-table gradient
// walks it.
struct RelationPlan {
    struct Block {
        hnh::DeviceBuffer<int32_t> perm, key_start, piece_first, piece_key;
        int64_t pieces = 0;
    };
    const Distributed_Sparse *owner = nullptr;
    int num_relations = 0;
    vector<std::unique_ptr<Block>> blocks;  // null for a block without entries
};

class Distributed_Sparse {
public:
    int proc_rank;  // global rank
    int p, c;       // number of ranks, replication factor

    string algorithm_name;
    vector<string> proc_grid_names;

    vector<string> perf_counter_keys;
    map<string, int> call_count;
    map<string, double> total_time;

    int64_t M, N, R;
    int localArows, localAcols, localBrows, localBcols;
    vector<DenseSubmatrix> aSubmatrices;
    vector<DenseSubmatrix> bSubmatrices;

    unique_ptr<SpmatLocal> S;
    unique_ptr<SpmatLocal> ST;
    shared_ptr<FlexibleGrid> grid;

    int superclass_constructor_sentinel;
    KernelImplementation *kernel;  // non-owning, like the reference

    bool r_split;
    shared_ptr<hnh::Comm> A_R_split_world, B_R_split_world;

    bool verbose;
    string debug_msg;
    // overlap ring shifts with kernels where legal (results never change); on by default
    bool overlap;

    explicit Distributed_Sparse(KernelImplementation *k);
    virtual ~Distributed_Sparse() { release_edge_softmax(); }

    virtual void setRValue(int R) = 0;
    void check_initialized();

    json json_algorithm_info();
    void print_algorithm_info();
    void setVerbose(bool value) { verbose = value; }

    // lengths of the value vectors that go with sddmmA/spmmA/fusedSpMM(Amat) (S) and with the
    // B-variants (ST); like_S_values / like_ST_values allocate them on the device
    virtual int64_t num_S_values() { return S->owned_coords_end - S->owned_coords_start; }
    virtual int64_t num_ST_values() { return ST->owned_coords_end - ST->owned_coords_start; }
    virtual VectorXd like_S_values(double value) { return VectorXd::Constant(num_S_values(), value); }
    virtual VectorXd like_ST_values(double value) { return VectorXd::Constant(num_ST_values(), value); }
    DenseMatrix like_A_matrix(double value) { return DenseMatrix::Constant(localArows, localAcols, value); }
    DenseMatrix like_B_matrix(double value) { return DenseMatrix::Constant(localBrows, localBcols, value); }

    // ---- perf counters (keys must be registered in perf_counter_keys) -------------------
    void reset_performance_timers();
    void stop_clock_and_add(my_timer_t &start, string counter_name);  // host wall clock
    void region_begin(const string &counter_name, cudaStream_t s);    // CUDA-event span
    void region_end(const string &counter_name, cudaStream_t s);
    void print_performance_statistics();
    json json_perf_statistics();  // collective; averages over ranks like the reference

    virtual void initial_shift(DenseMatrix *localA, DenseMatrix *localB, KernelMode op) = 0;
    virtual void de_shift(DenseMatrix *localA, DenseMatrix *localB, KernelMode op) = 0;

    // ---- the five convenience operations (reference :274-312) ---------------------------
    void spmmA(DenseMatrix &localA, DenseMatrix &localB, VectorXd &SValues) {
        localA.setZero();
        algorithm(localA, localB, SValues, nullptr, k_spmmA, true);
    }
    void spmmB(DenseMatrix &localA, DenseMatrix &localB, VectorXd &SValues) {
        localB.setZero();
        algorithm(localA, localB, SValues, nullptr, k_spmmB, true);
    }
    void sddmmA(DenseMatrix &localA, DenseMatrix &localB, VectorXd &SValues, VectorXd &sddmm_result) {
        algorithm(localA, localB, SValues, &sddmm_result, k_sddmmA, true);
    }
    void sddmmB(DenseMatrix &localA, DenseMatrix &localB, VectorXd &SValues, VectorXd &sddmm_result) {
        algorithm(localA, localB, SValues, &sddmm_result, k_sddmmB, true);
    }
    // SDDMM then SpMM with "replication reuse": the second pass skips the replication step.
    virtual void fusedSpMM(DenseMatrix &localA, DenseMatrix &localB, VectorXd &Svalues, VectorXd &sddmm_buffer,
                           MatMode mode);

    // fusedSpMM on HOST operands, as the reference's callers hold them (Eigen matrices in host memory):
    // hostA / hostB are this rank's local shards (row-major, like_A_matrix / like_B_matrix shapes), hostOut
    // receives the SpMM result (the shape of the `mode` operand).  localA / localB are the device staging
    // matrices.  Returns when hostOut is complete.  Subclasses may overlap the copies with the kernels.
    virtual void fusedSpMM_host(const double *hostA, const double *hostB, double *hostOut, DenseMatrix &localA,
                                DenseMatrix &localB, VectorXd &Svalues, VectorXd &sddmm_buffer, MatMode mode) {
        localA.copy_from_host(hostA);
        localB.copy_from_host(hostB);
        fusedSpMM(localA, localB, Svalues, sddmm_buffer, mode);
        (mode == Amat ? localA : localB).copy_to_host(hostOut);
    }

    virtual void algorithm(DenseMatrix &localA, DenseMatrix &localB, VectorXd &SValues, VectorXd *sddmm_result_ptr,
                           KernelMode mode, bool initial_replicate) = 0;

    // X[g_row, g_col] = g_row * R + g_col on the local submatrices (reference :322-346)
    void dummyInitialize(DenseMatrix &loc, MatMode mode);

    // Ring-shift a double-buffered matrix: send the active buffer to send_dst, receive the
    // passive one from recv_src, swap.  recv_src < 0: assume a constant-offset ring
    // (src = 2*rank - dst).  Enqueued on stream s (default: the comm stream, chained behind the
    // compute stream and joined back into it).
    void shiftDenseMatrix(BufferPair &buf, hnh::Comm &world, int send_dst, int tag, int recv_src = -1);

    // world-summed squared norms of a local matrix / vector ("fingerprints", scratch.cpp:26-76)
    double fingerprint(const DenseMatrix &m);
    double fingerprint(const VectorXd &v);

    // ---- edge softmax: a softmax over the stored entries of each row of S ----------------------------------
    // edgeSoftmax: values (a value vector of `order`: k_sddmmA for like_S_values, k_sddmmB for like_ST_values)
    // becomes alpha_uv = exp(x_uv - m_u) / s_u, with m_u the maximum and s_u the sum of exp(x_uv - m_u) over the
    // stored entries of row u of S on all ranks -- the normalisation of graph attention between an SDDMM and an
    // SpMM.  edgeSoftmaxBackward: grad (dL/d alpha, the same order) becomes dL/dx = alpha o (grad - t), with
    // t_u = sum over row u of alpha o grad.  Collective, in place, stream-ordered.  Each call builds its row
    // statistics from the vector it is given, which holds every stored entry of S exactly once over all ranks;
    // row statistics are M-long vectors reduced over the world (forward: one max and one sum all-reduce,
    // backward: one sum all-reduce; none at p = 1).  The A and B orders sum in different orders, so a softmax
    // of the same scores in the two orders may differ in the last bits.  The first call per order builds the
    // entries' row keys and a stable grouping by row on the device and keeps them until this object is destroyed
    // (in a table beside the object: the class layout and its virtual table stay those of earlier releases, so
    // programs compiled against earlier headers keep working with this library).
    // Defined where every rank holds full-width rows (check_full_rows); HNH_E_INVALID on every rank elsewhere.
    void edgeSoftmax(VectorXd &values, KernelMode order);
    void edgeSoftmaxBackward(const VectorXd &alpha, VectorXd &grad, KernelMode order);

    // Throws HNH_E_INVALID ("<operation>: not defined for <algorithm> at p = .., c = ..") unless every rank holds
    // full-width rows of the dense operands and the A and B layouts coincide: p = 1 (any algorithm), and 1.5D
    // dense shift with replication reuse (fusion 1) at any c or with local kernel fusion (fusion 2) at c = 1.
    // GAT's backward pass and softmax attention and edgeSoftmax need this.  Decided from global quantities
    // only, so every rank throws together and no collective is left waiting.
    void check_full_rows(const string &operation) const;

    // ---- additive graph attention (GAT::set_attention("additive")) ------------------------------------------
    // additiveScores: out (a value vector of `order`) becomes LeakyReLU(s[u] + t[v]) for every stored entry (u, v)
    // of S -- or, with `derivative`, its derivative: 1 where s[u] + t[v] > 0, alpha elsewhere.  s is indexed by
    // global S-row (at least M entries), t by global S-column (at least N): node vectors every rank holds whole.
    // Elementwise, no communication.  edgeSums: row_sums[u] / col_sums[v] become the sums of `values` (an A-order
    // vector) over the stored entries of row u / column v of S on all ranks, in a fixed order (bit-identical
    // repeats); entries past M / N are set to 0.  Two sum all-reduces at p > 1.  The first call per order builds
    // the entries' column keys, and edgeSums the grouping of the A order by column; they are kept with
    // edgeSoftmax's row grouping.  Defined where check_full_rows passes; HNH_E_INVALID on every rank elsewhere.
    void additiveScores(const VectorXd &s, const VectorXd &t, VectorXd &out, KernelMode order, double alpha, bool derivative);
    void edgeSums(const VectorXd &values, VectorXd &row_sums, VectorXd &col_sums);

    // ---- GATv2 attention (GAT::set_attention("gatv2")) --------------------------------------------------------
    // With sigma = LeakyReLU(., alpha), u = S-row and v = S-column, localA the A-shaped operand (rows u) and
    // localB the B-shaped one (rows v), both r = a.size() wide, as in sddmmA / sddmmB:
    // gatv2Scores: out (a value vector of `order`: k_sddmmA for like_S_values, k_sddmmB for like_ST_values) becomes
    //     x_uv = sum_k a_k sigma(localA[u, k] + localB[v, k]) for every stored (u, v) of S (overwritten).
    // gatv2Backward: with grad_A / grad_B = dL/dx in the A and B orders,
    //     dA[u] += a o sum_v g_uv sigma'(localA[u] + localB[v]),  dB[v] += a o sum_u g_uv sigma'(...),
    //     da = sum_uv g_uv sigma(localA[u] + localB[v]) over all ranks (overwritten; resized to r; the same on
    //     every rank).  sigma'(z) = 1 where z > 0, alpha elsewhere.  dA and dB may be the same matrix.
    // Each gradient comes from the order whose CSR blocks hold that side as stored rows, through a kernel that owns
    // those rows: no scatter, no atomic.  Where the operands travel: p = 1, none; 1.5D dense shift with local kernel
    // fusion (c = 1): the stored-row side stays, the gathered side rides read-only; with replication reuse (any c):
    // the gathered side is replicated over the layer and the stored-row side rides -- for gatv2Backward together
    // with its gradient, as one 2r-wide matrix that ends at home.  Collective; defined where check_full_rows
    // passes, HNH_E_INVALID on every rank elsewhere.
    void gatv2Scores(DenseMatrix &localA, DenseMatrix &localB, const VectorXd &a, VectorXd &out, KernelMode order,
                     double alpha);
    void gatv2Backward(DenseMatrix &localA, DenseMatrix &localB, const VectorXd &a, const VectorXd &grad_A,
                       const VectorXd &grad_B, DenseMatrix &dA, DenseMatrix &dB, VectorXd &da, double alpha);

    // ---- fused sparse attention over the pattern of S --------------------------------------------------------
    // Q (A-shaped: this rank's S-rows) and K, V (B-shaped: its S-columns) are r wide, r = heads * d.  For head h,
    // over the column window [h d, (h + 1) d), and every stored (u, v) of S (duplicates count; S's values are not
    // read):  x_uv = scale <Q_u,h, K_v,h>,  L_u,h = log sum_v exp(x_uv),  Z_u,h = sum_v exp(x_uv - L_u,h) V_v,h.
    // sparseAttention overwrites Z (A-shaped, r wide) and L (localArows x heads); a row without entries gets Z = 0
    // and L = -inf.  sparseAttentionBackward, given dZ and the forward's Z and L, overwrites dQ, dK and dV:
    //     t_u,h = <dZ_u,h, Z_u,h>,  dx_uv = alpha_uv (<dZ_u,h, V_v,h> - t_u,h),
    //     dQ_u,h = scale sum_v dx_uv K_v,h,  dK_v,h = scale sum_u dx_uv Q_u,h,  dV_v,h = sum_u alpha_uv dZ_u,h.
    // One fused pass per head for the forward (an online softmax carried from block to block), two for the
    // backward (A order for dQ, B order for dK and dV); no score vector, no row grouping, and no collective beyond
    // the ring shifts of gather_pass.  `scale` must be finite.  Collective; defined where check_full_rows passes,
    // HNH_E_INVALID on every rank elsewhere.
    void sparseAttention(DenseMatrix &Q, DenseMatrix &K, DenseMatrix &V, DenseMatrix &Z, DenseMatrix &L, int heads,
                         double scale);
    void sparseAttentionBackward(DenseMatrix &Q, DenseMatrix &K, DenseMatrix &V, DenseMatrix &Z, DenseMatrix &L,
                                 DenseMatrix &dZ, DenseMatrix &dQ, DenseMatrix &dK, DenseMatrix &dV, int heads,
                                 double scale);
    // The same with attention dropout of probability `dropout` in [0, 1): with D_uv,h the keep bit of the stored
    // (u, v) in head h and w = 1 / (1 - dropout),
    //     Z_u,h = sum_v D_uv,h w alpha_uv V_v,h,  with L_u,h still the log-sum-exp of all scores, and
    //     dx_uv = alpha_uv (D_uv,h w <dZ_u,h, V_v,h> - t_u,h),  dV_v,h = sum_u D_uv,h w alpha_uv dZ_u,h.
    // D_uv,h is the mask of hnh_sparse_attention_step_dropout_f64 (include/hnh_b200.h) at seed + h and the global
    // S-row u and S-column v, so it is the same on every layout, and stored duplicates of (u, v) share it.  A
    // backward must get the forward's dropout and seed, and every rank the same values.  dropout = 0 runs the
    // kernels without dropout (the overloads above forward here with (0, 0)).  dropout outside [0, 1), NaN, or,
    // with dropout > 0, S wider or taller than 2^32: HNH_E_INVALID on every rank before any launch.
    void sparseAttention(DenseMatrix &Q, DenseMatrix &K, DenseMatrix &V, DenseMatrix &Z, DenseMatrix &L, int heads,
                         double scale, double dropout, uint64_t seed);
    void sparseAttentionBackward(DenseMatrix &Q, DenseMatrix &K, DenseMatrix &V, DenseMatrix &Z, DenseMatrix &L,
                                 DenseMatrix &dZ, DenseMatrix &dQ, DenseMatrix &dK, DenseMatrix &dV, int heads,
                                 double scale, double dropout, uint64_t seed);
    // The same with an additive score bias: x_uv,h = scale <Q_u,h, K_v,h> + b_uv,h (added after the scale, not
    // scaled); L, Z, t and the dropout mask are the above on these scores, and dQ, dK, dV keep their formulas with
    // alpha from the biased x.  The backward also writes dbias_uv,h = dx_uv,h = alpha_uv (D w <dZ_u, V_v> - t_u).
    // A bias is a value vector of the order it is used in (like_S_values for the A order, like_ST_values for the
    // B order) of length n (every head reads it; its gradient is sum_h dx_h) or heads * n (head h reads
    // [h n, (h + 1) n)), n that order's local entry count.  The forward and the backward's dQ pass read `bias` /
    // `bias_A` (A order), the backward's dK, dV pass `bias_B` (B order).  Contract, not checked: bias_A and bias_B
    // hold the same b(u, v), a function of the global S-row and S-column (entryCoordinates gives them), so stored
    // duplicates of (u, v) share one bias; the backward gets the forward's bias; every rank passes matching vectors.
    // b = -inf masks an entry: alpha = 0, nothing added to Z, dbias = 0.  A row masked throughout gets Z = 0,
    // L = -inf and zero gradients, as a row without entries (edgeSoftmax gives NaN there).  +inf or NaN: not
    // checked, the row's results are NaN.  dbias_A / dbias_B (nullable) are resized to their bias's length and
    // overwritten; the heads accumulate into a shared bias's gradient in a fixed order (bit-identical repeats).
    // A null bias (both null in the backward) runs the kernels without bias: the overloads above forward here with
    // null pointers.  HNH_E_INVALID on every rank before any launch for a bias length other than n or heads * n,
    // bias_A and bias_B of different head multiplicity, only one of them, a dbias without its bias, or a dbias that
    // is a bias.
    void sparseAttention(DenseMatrix &Q, DenseMatrix &K, DenseMatrix &V, DenseMatrix &Z, DenseMatrix &L, int heads,
                         double scale, double dropout, uint64_t seed, const VectorXd *bias);
    void sparseAttentionBackward(DenseMatrix &Q, DenseMatrix &K, DenseMatrix &V, DenseMatrix &Z, DenseMatrix &L,
                                 DenseMatrix &dZ, DenseMatrix &dQ, DenseMatrix &dK, DenseMatrix &dV, int heads,
                                 double scale, double dropout, uint64_t seed, const VectorXd *bias_A,
                                 const VectorXd *bias_B, VectorXd *dbias_A, VectorXd *dbias_B);
    // The same with edge features added to the keys and values (TransformerConv with edge_dim): per entry i = (u, v)
    // and head h, x_i,h = scale <Q_u,h, K_v,h + E_i,h> + b_i,h and Z_u,h = sum_i D_i w alpha_i (V_v,h + E_i,h); the
    // backward uses g_i = <dZ_u, V_v + E_i> in dx_i = alpha_i (D_i w g_i - t_u), dQ_u = scale sum_i dx_i (K_v + E_i),
    // dK_v and dV_v keep their formulas, and it writes dE_i = scale dx_i Q_u + D_i w alpha_i dZ_u.  E is a
    // DenseMatrix of n x r, n the local entry count of the order it is used in (num_S_values / num_ST_values, the
    // order of like_S_values / like_ST_values): row i belongs to entry i of that order's value vector and head h
    // reads its columns [h d, (h + 1) d).  It stays on the rank that owns the entry; no ring carries it.  The forward
    // and the dQ pass read `edge` / `edge_A` (A order), the dK, dV pass `edge_B` (B order).  `dedge` (nullable) is
    // resized to edge_A's shape and overwritten in the A order; a masked entry's row is 0.  Contract, not checked:
    // edge_A and edge_B hold the same e(u, v), a function of the global S-row and S-column (entryCoordinates), so
    // stored duplicates of (u, v) share one row; the backward gets the forward's E; every rank passes its part of
    // the same E.  E = 0 gives the bits of the call without E.  A null edge (both null in the backward) is the call
    // without E: the overloads above forward here with null pointers.  HNH_E_INVALID on every rank before any
    // launch for an E that is not n x r, only one of edge_A / edge_B, a dedge without E, or a dedge that is another
    // operand of the call.
    void sparseAttention(DenseMatrix &Q, DenseMatrix &K, DenseMatrix &V, DenseMatrix &Z, DenseMatrix &L, int heads,
                         double scale, double dropout, uint64_t seed, const VectorXd *bias, const DenseMatrix *edge);
    void sparseAttentionBackward(DenseMatrix &Q, DenseMatrix &K, DenseMatrix &V, DenseMatrix &Z, DenseMatrix &L,
                                 DenseMatrix &dZ, DenseMatrix &dQ, DenseMatrix &dK, DenseMatrix &dV, int heads,
                                 double scale, double dropout, uint64_t seed, const VectorXd *bias_A,
                                 const VectorXd *bias_B, VectorXd *dbias_A, VectorXd *dbias_B, const DenseMatrix *edge_A,
                                 const DenseMatrix *edge_B, DenseMatrix *dedge);
    // rows / cols (resized to the order's local entry count) become the global S-row and S-column of every entry
    // of this rank's value vector of `order` (k_sddmmA: like_S_values, k_sddmmB: like_ST_values), as exact
    // doubles.  No communication.  Defined where check_full_rows passes; HNH_E_INVALID on every rank elsewhere.
    void entryCoordinates(KernelMode order, VectorXd &rows, VectorXd &cols);

    // ---- link prediction: a dot-product edge decoder with binary cross-entropy -------------------------------------
    // Called on the object of the target matrix T: its S holds the node pairs to score, its stored values y_uv in [0, 1]
    // the targets (1 positive, 0 negative, soft targets allowed), as built -- an SDDMM, SpMM or FusedMM on this object
    // overwrites its block values.  H_A (localArows x r) and H_B (localBrows x r) are the A- and B-shaped node
    // embeddings; a model whose A and B rows are the same nodes passes its output buffer as both.  For every stored
    // (u, v) of T (duplicates count):
    //     s_uv = <H_A[u], H_B[v]>,  l_uv = max(s, 0) - s y + log1p(exp(-|s|)),  g_uv = (sigmoid(s_uv) - y_uv) inv_count,
    // torch's F.binary_cross_entropy_with_logits per entry.  sums (device, 2 doubles) receives (sum l_uv, the number of
    // entries with (s > 0) == (y > 0.5)) over all ranks, the same on every rank; dH_A (nullable) = sum_v g_uv H_B[v]
    // and dH_B (nullable) = sum_u g_uv H_A[u], overwritten (the sum of both when they are one matrix); scores
    // (nullable, an A-order vector: like_S_values) = s.  H_A and H_B may be one matrix.  One gather_pass in the A
    // order (H_A, dH_A and the rows' loss and count on the stored-row side), a second in the B order only with dH_B;
    // the row statistics are summed in a fixed order, then one world all-reduce of 2 doubles.  No atomics: repeated
    // calls are bit-identical.  Collective; defined where check_full_rows passes.  HNH_E_INVALID on every rank before
    // any launch for H_A / H_B that are not localArows / localBrows rows of one width r >= 1, a gradient of another
    // shape or that is an H, scores of another length, a null sums or an inv_count that is not finite and >= 0.
    void linkLoss(DenseMatrix &H_A, DenseMatrix &H_B, double inv_count, DenseMatrix *dH_A, DenseMatrix *dH_B,
                  VectorXd *scores, double *sums);
    // The number of stored entries of S over all ranks, after checking on the device that every stored value lies in
    // [0, 1] (link targets).  Collective: one world all-reduce of 2 doubles; a value elsewhere (NaN and infinities
    // included) on any rank is refused with HNH_E_INVALID on every rank.  Defined where check_full_rows passes.
    int64_t linkTargetCount();

    // ---- relation-aware link prediction: the DistMult edge decoder with binary cross-entropy ---------------------------
    // Called on the object of a target matrix T whose stored values are relations: the relation rho of a stored (u, v)
    // is its value, an integer in [0, num_relations) as for relationalAggregate (an entry with any other value
    // contributes nothing: no loss, no count, no gradient, score 0).  H_A (localArows x r) and H_B (localBrows x r) are
    // the embeddings as for linkLoss, D (num_relations x r, the same on every rank) the relation table and `target` in
    // [0, 1] the target of every entry of the call.  For every stored (u, v) of T (duplicates count, each under its own
    // relation):
    //     s_uv = sum_k H_A[u, k] D[rho, k] H_B[v, k],   l and g = (sigmoid(s) - target) inv_count as linkLoss,
    // torch's (z[src] * rel_emb[edge_type] * z[dst]).sum(-1) and F.binary_cross_entropy_with_logits.  sums (device, 2
    // doubles) += (sum l, the entries with (s > 0) == (target > 0.5)) over all ranks; dH_A (nullable) = sum_v g D[rho] o
    // H_B[v], dH_B (nullable) = sum_u g D[rho] o H_A[u] (the sum of both when they are one matrix), dD (nullable,
    // num_relations x r, the same on every rank) = sum over the entries of relation rho on all ranks of g H_A[u] o H_B[v];
    // the gradients are overwritten or, with `accumulate`, added to, so calls for the positive and the negative
    // targets sum into one gradient.  scores (nullable, an A-order vector: like_S_values) = s.  Passes: one gather_pass
    // in the A order (scores, dH_A, the rows' loss and count, and every entry's g when dD is wanted), one in the B order
    // only with dH_B, and for dD one more in the A order that walks `plan` (relationPlan(num_relations) of this object;
    // null: built for the call), writes one r-wide partial per piece and sums each relation's pieces in plan order, then
    // one world all-reduce of R r doubles.  The row statistics are summed in a fixed order and all-reduced (2 doubles).
    // No atomics: repeated calls are bit-identical.  Collective; defined where check_full_rows passes.  HNH_E_INVALID on
    // every rank before any launch for linkLoss's refusals, num_relations < 1, a D or dD that is not num_relations x r,
    // a target outside [0, 1], a gradient that is H_A, H_B or D, or a plan of another object or relation count.
    void distmultLoss(DenseMatrix &H_A, DenseMatrix &H_B, const DenseMatrix &D, int num_relations, double target, double inv_count,
                      DenseMatrix *dH_A, DenseMatrix *dH_B, DenseMatrix *dD, VectorXd *scores, double *sums, bool accumulate,
                      const RelationPlan *plan = nullptr);
    // The A order's entries grouped by relation for distmultLoss (the relations as the stored values are now).
    // No communication.  Defined where check_full_rows passes; HNH_E_INVALID for num_relations < 1.
    std::unique_ptr<RelationPlan> relationPlan(int num_relations);

    // ---- max aggregation: the SpMM over the (max, .) semiring (GraphSAGE's max aggregator) ---------------------------
    // X (localBrows x f, the B-shaped operand: rows are S-columns v) is gathered over the stored entries (u, v) of S on
    // all ranks (duplicates count; S's values are not read).  maxAggregate overwrites Z and C (localArows x f each):
    //     Z_u,k = max_v X_v,k,   C_u,k = the number of stored entries of row u with X_v,k == Z_u,k,
    // and Z = C = 0 on a row without entries -- torch's zeros(M, f).scatter_reduce(0, u, X[v], "amax",
    // include_self = False), which is PyG's MaxAggregation.  -0.0 and +0.0 tie; which of the two Z holds is not
    // specified.  NaN is not checked.  maxAggregateBackward, given the forward's Z and C and dZ (A-shaped), writes
    //     dX_v,k = sum_u [X_v,k == Z_u,k] dZ_u,k / C_u,k
    // (ties share the gradient equally), overwriting dX or, with `accumulate`, adding to it.  (torch's autograd of that
    // scatter_reduce also counts the untouched zero of `self` as a tie where the maximum is exactly 0, and gives each
    // entry dZ / (C + 1) there; this op splits dZ over the stored entries only.)  One gather_pass for the
    // forward (A order: [Z | C] on the stored-row side, read-modify-written once per row and ring step, holding
    // (-inf, 0) before it and finished elementwise after it), one for the backward (B order: X and dX on the stored-row
    // side, [Z | dZ / C] gathered).  gather_pass never adds the written operands of a riding side: under replication
    // reuse they ride the output ring from kernel to kernel and come home, and no layout where check_full_rows passes
    // reduce-scatters.  The forward has no floating-point sum and no atomics: repeated calls are bit-identical, and so
    // is the backward (sums in stored order).  Collective; defined where check_full_rows passes.  HNH_E_INVALID on every
    // rank before any launch for an X that is not localBrows rows of width 1 <= f < 2^31, a Z, C or dZ that is not
    // localArows x f, a dX that is not X's shape, or an output that is another operand of the call.
    void maxAggregate(DenseMatrix &X, DenseMatrix &Z, DenseMatrix &C);
    void maxAggregateBackward(DenseMatrix &X, DenseMatrix &Z, DenseMatrix &C, DenseMatrix &dZ, DenseMatrix &dX, bool accumulate);

    // ---- multi-statistic aggregation (PNA): several statistics of each row's neighbours in one gather ----------------
    // `which` is a non-empty union of HNH_MULTI_MOMENTS, HNH_MULTI_MAX and HNH_MULTI_MIN (hnh_b200.h).  multiAggregate
    // overwrites A (localArows x W f, W = 2, 4 or 6) with the selected f-wide windows, in the fixed order
    //     [sum_v X_v | sum_v X_v^2 | max_v X_v | #ties of the max | min_v X_v | #ties of the min]
    // over the stored entries (u, v) of S on all ranks (duplicates count; S's values are not read), every window 0 on a
    // row without entries.  The maxima and minima follow maxAggregate.  multiAggregateBackward, given the forward's A
    // and dA (A's layout; its count windows are not read), writes
    //     dX_v = sum_u dA_sum[u] + 2 X_v dA_sq[u] + [X_v == max_u] dA_max[u] / C_max[u] + [X_v == min_u] dA_min[u] / C_min[u]
    // overwriting dX or, with `accumulate`, adding to it.  One gather_pass each, as maxAggregate: the forward in A order
    // with A riding with the stored rows, the backward in B order with X and dX on the stored-row side.  Sums run in
    // stored order without atomics: repeated calls are bit-identical.  Collective; defined where check_full_rows passes.
    // HNH_E_INVALID on every rank before any launch for an empty or unknown `which`, an X that is not localBrows rows of
    // width f >= 1, a total width W f of 2^31 or more, an A or dA that is not localArows x W f, a dX that is not X's
    // shape, or an output that is another operand of the call.
    void multiAggregate(DenseMatrix &X, DenseMatrix &A, int which);
    void multiAggregateBackward(DenseMatrix &X, DenseMatrix &A, DenseMatrix &dA, DenseMatrix &dX, int which, bool accumulate);

    // ---- edge-ReLU aggregation (GINE): a per-entry vector added to each gathered row before a ReLU ---------------------
    // E_A (num_S_values x f) and E_B (num_ST_values x f) are per-entry rows in the A and B value orders, laid out as
    // sparseAttention's edge features (entry i of block b at row blockStarts[b] + i; they stay on the rank that owns the
    // entry) and holding the same e(u, v) for every stored (u, v), so stored duplicates share one row.  Over the stored
    // entries i = (u, v) of S on all ranks (duplicates count; S's values are not read):
    //     edgeReluAggregate:          A_u  = sum_i ReLU(X_v + E_i)                  (0 on a row without entries)
    //     edgeReluAggregateBackward:  dX_v (+)= sum_i [X_v + E_i > 0] dA_u,   dE_A,i = [X_v + E_i > 0] dA_u
    // with the strict mask of torch's relu backward.  One gather_pass each: the forward in A order with A riding with
    // the stored rows, dX in B order (X and dX stored, dA gathered, E_B read), dE_A in A order (dA stored, X gathered,
    // E_A read; every row written once) and skipped for a null dE_A.  dX is overwritten or, with `accumulate`, added
    // to.  Sums run in stored order without atomics: repeated calls are bit-identical.  Collective; defined where
    // check_full_rows passes.  HNH_E_INVALID on every rank before any launch for an X that is not localBrows rows of
    // width 1 <= f < 2^31, an A or dA that is not localArows x f, a dX that is not X's shape, an E_A or E_B that is not
    // its order's entry count x f, only one of E_A / E_B, or an output that is another operand of the call.
    void edgeReluAggregate(DenseMatrix &X, const DenseMatrix &E_A, DenseMatrix &A);
    void edgeReluAggregateBackward(DenseMatrix &X, const DenseMatrix *E_A, const DenseMatrix *E_B, DenseMatrix &dA, DenseMatrix &dX,
                                   DenseMatrix *dE_A, bool accumulate);

    // ---- relational aggregation (R-GCN): each stored entry's value picks the window its neighbour is summed into ------
    // The relation of a stored entry (u, v) of S is its stored value (SpmatLocal::from_tuples' vals; an SDDMM or
    // FusedMM on this object overwrites it), an integer in [0, num_relations).  An entry with any other value
    // (negative, too large, fractional, infinite, NaN) contributes nothing.  relationalAggregate overwrites A
    // (localArows x R f) with
    //     A[u, rho f + k] = sum of X[v, k] over the stored entries (u, v) of relation rho on all ranks
    // (duplicates count, each under its own relation; 0 where there are none), X being localBrows x f.
    // relationalAggregateBackward, given dA (localArows x R f), writes
    //     dX[v, k] = sum of dA[u, rho f + k] over the stored entries (u, v), rho their relation
    // overwriting dX (localBrows x f) or, with `accumulate`, adding to it.  One gather_pass each: the forward in A
    // order (A rides with the stored rows under replication reuse and accumulates across the ring steps), the backward
    // in B order (dX with the stored rows, dA gathered: at c > 1 the all-gather carries R f columns).  Sums run in
    // stored order without atomics: repeated calls are bit-identical.  Collective; defined where check_full_rows passes.
    // HNH_E_INVALID on every rank before any launch for num_relations < 1, R f >= 2^31, wrong shapes, or an output that
    // is another operand.
    void relationalAggregate(DenseMatrix &X, DenseMatrix &A, int num_relations);
    void relationalAggregateBackward(DenseMatrix &dA, DenseMatrix &dX, int num_relations, bool accumulate);
    // The number of stored entries of S over all ranks, all of whose values are relations in [0, num_relations).
    // Collective: one world all-reduce of 2 doubles; a value elsewhere on any rank is refused with HNH_E_INVALID on
    // every rank.  Defined where check_full_rows passes.
    int64_t relationCheck(int num_relations);

    // ---- basis aggregation (R-GCN with basis decomposition): one window per basis instead of one per relation ---------
    // comp (R x B, every rank the same) mixes the relations into B bases; scale (nullable: all ones) is localArows x R,
    // a weight per (S-row, relation) -- 1 / |N_rho(u)| for R-GCN's mean.  With rho the relation of a stored entry as for
    // relationalAggregate (an entry that is no relation contributes nothing), basisAggregate overwrites H
    // (localArows x B f) with
    //     H[u, b f + k] = sum over the stored entries (u, v) on all ranks of scale[u, rho] comp[rho, b] X[v, k]
    // X being localBrows x f.  basisAggregateBackward, given dH (localArows x B f), writes
    //     dX[v, k] = sum over the stored entries (u, v) of scale[u, rho] sum_b comp[rho, b] dH[u, b f + k]
    // overwriting dX (localBrows x f) or, with `accumulate`, adding to it, and overwrites dcomp (R x B) with
    //     dcomp[rho, b] = sum over the stored entries of relation rho on all ranks of scale[u, rho] <dH[u, b f ..], X[v]>
    // the same on every rank.  One gather_pass each: the forward in A order (H and scale with the stored rows, X
    // gathered), the backward in B order (X and dX with the stored rows, dH and scale gathered) whose kernel also writes
    // every local entry's B products; these are summed by relation with an edge-softmax plan keyed by relation, built
    // per call (relations are S's values, which an SDDMM may overwrite), then one world all-reduce of R B doubles.  No
    // atomics: repeated calls are bit-identical.  Collective; defined where check_full_rows passes.  HNH_E_INVALID on
    // every rank before any launch for num_relations < 1, B < 1, B f or R B >= 2^31, wrong shapes, or an output that is
    // another operand.
    void basisAggregate(DenseMatrix &X, DenseMatrix &H, const DenseMatrix &comp, int num_relations, const DenseMatrix *scale);
    void basisAggregateBackward(DenseMatrix &dH, DenseMatrix &X, DenseMatrix &dX, const DenseMatrix &comp, DenseMatrix &dcomp,
                                int num_relations, const DenseMatrix *scale, bool accumulate);
    // frees what edgeSoftmax keeps for this object (the destructor calls it)
    void release_edge_softmax();

protected:
    hnh::EventTimers timers_;
    cudaStream_t compute() { return hnh::Runtime::get().compute_stream(); }
    cudaStream_t comm() { return hnh::Runtime::get().comm_stream(); }

    // result = SValues o (CSR values of all blocks of m), written straight into `result`
    // (reference: `*sddmm_result_ptr = SValues.cwiseProduct(choice->getCSRValues())`, e.g.
    // 15D_dense_shift.hpp:366, which allocates two temporaries and makes three extra passes)
    void hadamard_values(VectorXd &result, VectorXd &SValues, SpmatLocal &m);

    // copy-engine rings (hnh/peer_ring.h), one per (ring communicator, shard size), built on first use
    std::map<std::pair<hnh::Comm *, size_t>, std::unique_ptr<hnh::PeerRing>> peer_rings_;
    bool peer_ring_broken_ = false;
    hnh::PeerRing *peer_ring(std::shared_ptr<hnh::Comm> world, size_t bytes);
    // the same for a riding CSR block: the ring pushes straight into the next rank's passive CSRHandle
    std::map<std::pair<hnh::Comm *, CSRLocal *>, std::unique_ptr<hnh::PeerRing>> sparse_rings_;
    hnh::PeerRing *sparse_ring(std::shared_ptr<hnh::Comm> world, CSRLocal *blk);
    // One ring step of a CSR block over a copy-engine ring.  Call early() before the kernel that uses
    // the block (ships what the kernel does not write), late() after it (ships the rest, publishes,
    // commits).  `values_written`: the kernel accumulates into the block's values (SDDMM).
    void sparse_push_early(hnh::PeerRing &pr, CSRLocal &blk, bool values_written);
    void sparse_push_late(hnh::PeerRing &pr, CSRLocal &blk, bool values_written, bool early_done, int64_t incoming);

    // Driver of a dense ring over `world` (+1 direction, `steps` = world size):
    //   step t: body(t, riding) on the compute stream, then the riding matrix moves one rank on.
    // riding_is_input == true : the kernel only reads the riding matrix.  Three buffers are
    //     used, the caller's matrix is never written, transfers overlap kernels and the last
    //     (home-bound) shift is skipped.
    // riding_is_input == false: the kernel accumulates into the riding matrix (fusion-1 SpMM):
    //     kernel -> shift strictly alternate, `steps` shifts, the result ends up in `home`.
    template <class Body>
    void ring_dense(DenseMatrix &home, std::shared_ptr<hnh::Comm> world_ptr, bool riding_is_input, const string &shift_key,
                    const string &compute_key, Body body);

    // One pass of a row-owning kernel over the CSR blocks of a value order (gatv2_pass, sparseAttention): each
    // side of S has a list of operands, column windows of A-shaped (A_side) or B-shaped (B_side) matrices.  For
    // every block with entries, kernel(block, blk, rows_are_A, rows, gathered) runs where the block meets them, with
    // rows[i] the view of operand i of the side whose rows the block stores and gathered[i] that of operand i of
    // the other side (null for a written one: a kernel writes the stored-row side only).  Where the operands
    // travel: p = 1, none; 1.5D dense shift with local kernel fusion (c = 1): the stored-row side stays, the
    // gathered side rides read-only; with replication reuse (any c): the gathered side is stationary, all-gathered
    // over the layer when c > 1, and the stored-row side rides -- with its written operands on the output-riding
    // ring, complete when it comes home.  A side that moves travels as its one operand when that is a whole matrix,
    // else packed into one matrix of the operands' windows side by side.
    struct PassOperand {
        DenseMatrix *m;
        int64_t col0, cols;
        bool written;  // the kernel accumulates into it
    };
    struct PassView {
        double *p;  // row 0 of the window
        int64_t ld;
    };
    using PassKernel = std::function<void(int, CSRLocal &, bool, const PassView *, const PassView *)>;
    void gather_pass(KernelMode order, const vector<PassOperand> &A_side, const vector<PassOperand> &B_side,
                     const PassKernel &kernel);

    // One GATv2 pass over the CSR blocks of a value order (gatv2Scores, gatv2Backward): kernel(block, blk, R, ldr,
    // Y, ldy, dR, lddr) runs once per block with entries, with R the stored-row side, Y the gathered side and dR
    // the stored-row side's gradient (dA or dB; null when both are null), each at the rank and ring step where the
    // block meets them.
    using Gatv2Kernel = std::function<void(int, CSRLocal &, const double *, int64_t, const double *, int64_t, double *, int64_t)>;
    void gatv2_pass(KernelMode order, DenseMatrix &localA, DenseMatrix &localB, DenseMatrix *dA, DenseMatrix *dB,
                    const Gatv2Kernel &kernel);
};

// ------------------------------------------------------------------ ring driver ----------
template <class Body>
void Distributed_Sparse::ring_dense(DenseMatrix &home, std::shared_ptr<hnh::Comm> world_ptr, bool riding_is_input,
                                    const string &shift_key, const string &compute_key, Body body) {
    hnh::Runtime &rt = hnh::Runtime::get();
    hnh::Comm &world = *world_ptr;
    const int steps = world.size();
    const int me = world.rank();
    const int dst = pMod(me + 1, steps), src = pMod(me - 1, steps);
    if (steps == 1) {
        region_begin(compute_key, compute());
        body(0, home);
        region_end(compute_key, compute());
        return;
    }
    const size_t bytes = sizeof(double) * (size_t)home.size();
    hnh::PeerRing *pr = (riding_is_input && overlap) ? peer_ring(world_ptr, bytes) : nullptr;
    if (pr) {
        // Copy engines push the shard of step t into the next rank's slot (t+1)%2 while kernel t
        // runs; flags in peer memory order the two processes (no host, no SM involved).
        rt.chain(compute(), comm());  // `home` is up to date for the first push
        for (int t = 0; t < steps; t++) {
            const int k = t & 1;
            const void *cur = t == 0 ? (const void *)home.data() : pr->slot(k);
            if (t >= 1) pr->expect_arrival(k);
            if (t + 1 < steps) {
                region_begin(shift_key, comm());
                if (t >= 1) pr->wait_arrival(k, comm());
                pr->push((t + 1) & 1, cur, bytes, comm());
                region_end(shift_key, comm());
            }
            if (t >= 1) pr->wait_arrival(k, compute());
            region_begin(compute_key, compute());
            if (t == 0) {
                body(t, home);
            } else {
                DenseMatrix shard = DenseMatrix::view((double *)pr->slot(k), home.rows(), home.cols());
                body(t, shard);
            }
            region_end(compute_key, compute());
            if (t >= 1) {
                rt.chain(compute(), comm());  // slot k is free once kernel t and push t are done
                pr->release(k, comm());
            }
        }
        rt.chain(comm(), compute());
        return;
    }
    if (riding_is_input && overlap) {
        DenseMatrix e1(home.rows(), home.cols()), e2(home.rows(), home.cols());
        DenseMatrix *bufs[3] = {&home, &e1, &e2};
        auto at = [&](int t) -> DenseMatrix * { return t == 0 ? bufs[0] : bufs[1 + ((t - 1) & 1)]; };
        // the comm stream must see everything enqueued so far (home is up to date, e1/e2 free)
        rt.chain(compute(), comm());
        for (int t = 0; t < steps; t++) {
            if (t + 1 < steps) {
                // T_t: at(t) -> next rank's at(t+1).  at(t+1) was last read by K_{t-1}, which the
                // comm stream already waited for (chain below, issued after K_{t-1}).
                region_begin(shift_key, comm());
                world.sendrecv(at(t)->data(), bytes, dst, at(t + 1)->data(), bytes, src, comm());
                region_end(shift_key, comm());
            }
            region_begin(compute_key, compute());
            body(t, *at(t));
            region_end(compute_key, compute());
            if (t + 1 < steps) {
                rt.chain(comm(), compute());  // K_{t+1} needs T_t
                rt.chain(compute(), comm());  // T_{t+1} overwrites at(t+2) == at(t): needs K_t
            }
        }
        rt.chain(comm(), compute());
        return;
    }
    // output rides (or overlap disabled): kernel and shift strictly alternate
    hnh::PeerRing *pro = (!riding_is_input && overlap && hnh::PeerRing::all_shifts()) ? peer_ring(world_ptr, bytes) : nullptr;
    if (pro) {
        // copy engines instead of NCCL p2p (which gets few channels per peer at 8 ranks): the
        // accumulating shard hops through the ring slots and is copied home at the end
        for (int t = 0; t < steps; t++) {
            const int k = t & 1;
            if (t >= 1) {
                pro->expect_arrival(k);
                pro->wait_arrival(k, compute());
            }
            region_begin(compute_key, compute());
            if (t == 0) {
                body(t, home);
            } else {
                DenseMatrix shard = DenseMatrix::view((double *)pro->slot(k), home.rows(), home.cols());
                body(t, shard);
            }
            region_end(compute_key, compute());
            rt.chain(compute(), comm());
            region_begin(shift_key, comm());
            pro->push((t + 1) & 1, t == 0 ? (const void *)home.data() : pro->slot(k), bytes, comm());
            if (t >= 1) pro->release(k, comm());
            region_end(shift_key, comm());
        }
        const int kf = steps & 1;
        pro->expect_arrival(kf);
        region_begin(shift_key, comm());
        pro->wait_arrival(kf, comm());
        hnh::cuda_check(cudaMemcpyAsync(home.data(), pro->slot(kf), bytes, cudaMemcpyDeviceToDevice, comm()), "ring copy-back");
        pro->release(kf, comm());
        region_end(shift_key, comm());
        rt.chain(comm(), compute());
        return;
    }
    BufferPair pair(&home);
    for (int t = 0; t < steps; t++) {
        region_begin(compute_key, compute());
        body(t, *pair.getActive());
        region_end(compute_key, compute());
        rt.chain(compute(), comm());
        region_begin(shift_key, comm());
        world.sendrecv(pair.getActive()->data(), bytes, dst, pair.getPassive()->data(), bytes, src, comm());
        region_end(shift_key, comm());
        pair.swapActive();
        rt.chain(comm(), compute());
    }
    pair.sync_active();
}
