// distributed_sparse.cpp -- non-template members of Distributed_Sparse (hnh/distributed_sparse.h).
#include "hnh/distributed_sparse.h"

#include <algorithm>
#include <array>
#include <cmath>
#include <iostream>
#include <mutex>
#include <optional>
#include <tuple>

#include "hnh/15D_dense_shift.hpp"
#include "hnh/25D_cannon_dense.hpp"
#include "hnh_b200.h"

using hnh::Runtime;

Distributed_Sparse::Distributed_Sparse(KernelImplementation *k) {
    auto world = hnh::Comm::world();
    proc_rank = world->rank();
    p = world->size();
    verbose = false;
    overlap = true;
    kernel = k;
    algorithm_name = "";
    M = N = R = -1;
    localArows = localAcols = localBrows = localBcols = -1;
    c = -1;
    r_split = false;
    superclass_constructor_sentinel = 3;
}

void Distributed_Sparse::check_initialized() {
    auto need = [](bool ok, const char *what) {
        if (!ok) throw hnh::Error(HNH_E_INVALID, string("Distributed_Sparse subclass left uninitialised: ") + what);
    };
    need(algorithm_name != "", "algorithm_name");
    need(!proc_grid_names.empty(), "proc_grid_names");
    need(!perf_counter_keys.empty(), "perf_counter_keys");
    need(M != -1 && N != -1 && R != -1, "M/N/R");
    need(localAcols != -1 && localBcols != -1 && localArows != -1 && localBrows != -1, "local dims");
    need(c >= 1, "c");
    need(superclass_constructor_sentinel == 3, "base constructor");
    need(!aSubmatrices.empty() && !bSubmatrices.empty(), "submatrix descriptors");
    need(S && ST && S->initialized && ST->initialized, "S/ST");
    need(S->coordinate_ownership_initialized && ST->coordinate_ownership_initialized, "coordinate ownership");
    need(!S->blockStarts.empty() && !ST->blockStarts.empty(), "blockStarts");
    need(S->csr_initialized && ST->csr_initialized, "CSR blocks");
}

json Distributed_Sparse::json_algorithm_info() {
    json j = json::object();
    j["alg_name"] = algorithm_name;
    j["m"] = (long long)M;
    j["n"] = (long long)N;
    j["nnz"] = (unsigned long long)S->dist_nnz;
    j["r"] = (long long)R;
    j["adjacency_mode"] = grid->adjacency;
    j["p"] = p;
    j["c"] = c;
    json interp = json::array(), vals = json::array();
    for (size_t i = 0; i < proc_grid_names.size(); i++) {
        interp.push_back(proc_grid_names[i]);
        vals.push_back(grid->dim_list[i]);
    }
    j["dim_interpretations"] = interp;
    j["dim_values"] = vals;
    // per-rank nonzero counts (load imbalance report)
    uint64_t mine[2] = {(uint64_t)(S->owned_coords_end - S->owned_coords_start),
                        (uint64_t)(ST->owned_coords_end - ST->owned_coords_start)};
    vector<uint64_t> all((size_t)2 * p);
    hnh::Comm::world()->host_allgather(mine, all.data(), sizeof(mine));
    json nnz = json::array(), nnz_t = json::array();
    for (int i = 0; i < p; i++) {
        nnz.push_back((unsigned long long)all[2 * i]);
        nnz_t.push_back((unsigned long long)all[2 * i + 1]);
    }
    j["nnz_procs"] = nnz;
    j["nnz_tpose_procs"] = nnz_t;
    // not in the reference's record: what actually carries the ring shifts of this object
    j["transport"] = hnh::Comm::world()->transport_name();
    j["peer_rings"] = (int)(peer_rings_.size() + sparse_rings_.size());
    j["ring"] = p == 1 ? "none" : (!peer_rings_.empty() || !sparse_rings_.empty())
                                      ? "peer_ring (copy engines into CUDA-IPC mapped peer slots, stream memory-op flags)"
                                      : "send/recv of the transport";
    return j;
}

void Distributed_Sparse::print_algorithm_info() {
    json j = json_algorithm_info();
    if (proc_rank == 0) cout << j.dump(4) << endl;
}

void Distributed_Sparse::reset_performance_timers() {
    for (auto &key : perf_counter_keys) {
        call_count[key] = 0;
        total_time[key] = 0.0;
    }
    timers_.reset();
}

static void require_key(const vector<string> &keys, const string &name) {
    if (find(keys.begin(), keys.end(), name) == keys.end())
        throw hnh::Error(HNH_E_INVALID, "Error, performance counter " + name + " not registered.");
}

void Distributed_Sparse::stop_clock_and_add(my_timer_t &start, string counter_name) {
    require_key(perf_counter_keys, counter_name);
    call_count[counter_name]++;
    total_time[counter_name] += stop_clock_get_elapsed(start);
}

void Distributed_Sparse::region_begin(const string &name, cudaStream_t s) {
    require_key(perf_counter_keys, name);
    timers_.start(name, s);
}

void Distributed_Sparse::region_end(const string &name, cudaStream_t s) {
    timers_.stop(name, s);
    call_count[name]++;
}

json Distributed_Sparse::json_perf_statistics() {
    json j = json::object();
    vector<double> vals;
    for (auto &key : perf_counter_keys) vals.push_back(total_time[key] + timers_.total_seconds(key));
    hnh::Comm::world()->host_allreduce_sum_f64(vals.data(), vals.size());
    for (size_t i = 0; i < perf_counter_keys.size(); i++) j[perf_counter_keys[i]] = vals[i] / p;
    return j;
}

void Distributed_Sparse::print_performance_statistics() {
    json info = json_algorithm_info();
    json stats = json_perf_statistics();
    if (proc_rank == 0) {
        cout << endl
             << "================================" << endl
             << "==== Performance Statistics ====" << endl
             << "================================" << endl
             << info.dump(4) << endl
             << stats.dump(4) << endl
             << "=================================" << endl;
    }
}

void Distributed_Sparse::fusedSpMM(DenseMatrix &localA, DenseMatrix &localB, VectorXd &Svalues, VectorXd &sddmm_buffer,
                                   MatMode mode) {
    if (mode == Amat) {
        algorithm(localA, localB, Svalues, &sddmm_buffer, k_sddmmA, true);
        localA.setZero();
        algorithm(localA, localB, sddmm_buffer, nullptr, k_spmmA, false);
    } else {
        algorithm(localA, localB, Svalues, &sddmm_buffer, k_sddmmB, true);
        localB.setZero();
        algorithm(localA, localB, sddmm_buffer, nullptr, k_spmmB, false);
    }
}

void Distributed_Sparse::dummyInitialize(DenseMatrix &loc, MatMode mode) {
    vector<DenseSubmatrix> &subs = (mode == Amat) ? aSubmatrices : bSubmatrices;
    vector<double> host((size_t)loc.size());
    size_t at = 0;
    for (const DenseSubmatrix &s : subs)
        for (int i = 0; i < s.rowCount; i++)
            for (int j = 0; j < s.colCount; j++) host[at++] = (double)(s.topRow + i) * (double)R + (double)(s.leftCol + j);
    if ((int64_t)at != loc.size()) throw hnh::Error(HNH_E_INVALID, "dummyInitialize: submatrices do not tile the local matrix");
    loc.copy_from_host(host.data());
}

void Distributed_Sparse::shiftDenseMatrix(BufferPair &buf, hnh::Comm &world, int send_dst, int /*tag*/, int recv_src) {
    Runtime &rt = Runtime::get();
    const int n = world.size();
    if (recv_src < 0) recv_src = pMod(2 * world.rank() - send_dst, n);
    const size_t bytes = sizeof(double) * (size_t)buf.getActive()->size();
    rt.chain(compute(), comm());
    world.sendrecv(buf.getActive()->data(), bytes, send_dst, buf.getPassive()->data(), bytes, recv_src, comm());
    rt.chain(comm(), compute());
    buf.swapActive();
}

double Distributed_Sparse::fingerprint(const DenseMatrix &m) {
    double v = m.squaredNorm();
    hnh::Comm::world()->host_allreduce_sum_f64(&v, 1);
    return v;
}

double Distributed_Sparse::fingerprint(const VectorXd &v) {
    double x = v.squaredNorm();
    hnh::Comm::world()->host_allreduce_sum_f64(&x, 1);
    return x;
}

void Distributed_Sparse::hadamard_values(VectorXd &result, VectorXd &SValues, SpmatLocal &m) {
    const int64_t total = (int64_t)m.blockStarts.back();
    if (SValues.size() != total)
        throw hnh::Error(HNH_E_INVALID, "SValues has " + to_string(SValues.size()) + " entries, the local sparse matrix " +
                                            to_string(total));
    if (result.size() != total) result.resize(total);
    for (size_t b = 0; b + 1 < m.blockStarts.size(); b++) {
        const int64_t off = (int64_t)m.blockStarts[b], n = (int64_t)m.blockStarts[b + 1] - off;
        if (n == 0) continue;
        if (m.csr_blocks[b])
            hnh::abi_check(hnh_hadamard_f64(result.data() + off, SValues.data() + off,
                                            m.csr_blocks[b]->getActive()->values.data(), n, compute()),
                           "hadamard");
        else
            hnh::cuda_check(cudaMemsetAsync(result.data() + off, 0, sizeof(double) * (size_t)n, compute()), "memset");
    }
}

// ---- edge softmax ------------------------------------------------------------------------------------------
void Distributed_Sparse::check_full_rows(const string &operation) const {
    if (p == 1) return;
    const string where = algorithm_name + " at p = " + std::to_string(p) + ", c = " + std::to_string(c);
    if (r_split) throw hnh::Error(HNH_E_INVALID, operation + ": not defined for " + where + ": the layout splits the dense operands along R");
    const Sparse15D_Dense_Shift *dense_shift = dynamic_cast<const Sparse15D_Dense_Shift *>(this);
    if (dense_shift == nullptr) throw hnh::Error(HNH_E_INVALID, operation + ": not defined for " + where);
    if (dense_shift->fusionApproach == 2 && c > 1)
        throw hnh::Error(HNH_E_INVALID, operation + ": not defined for " + where +
                                            " with local kernel fusion (fusion 2): the forward SpMM accumulates onto the "
                                            "gathered projection when c > 1");
}

namespace {

// The row grouping of one value order (edgeSoftmax), built on first use.  Kept in a table keyed by the algorithm
// object rather than in the object, so that the layout of Distributed_Sparse and of its subclasses is unchanged.
// Additive attention adds, also on first use, the entries' global S-columns (`cols`: additiveScores) and, for the A
// order, their grouping by column (`col_perm` .. `col_pieces`: edgeSums).
struct EdgeRows {
    hnh::DeviceBuffer<int32_t> keys, perm, row_start, piece_first, piece_row;
    int64_t n = 0, pieces = 0;
    hnh::DeviceBuffer<int32_t> cols, col_perm, col_start, col_piece_first, col_piece_row;
    bool has_cols = false;
    int64_t col_pieces = -1;  // -1: no column grouping yet
};
std::mutex edge_rows_mutex;
using EdgeRowsTable = std::map<const Distributed_Sparse *, std::array<std::unique_ptr<EdgeRows>, 2>>;
// never destroyed: an object still alive at exit must not free device memory after the runtime has gone
EdgeRowsTable &edge_rows_table() {
    static EdgeRowsTable *t = new EdgeRowsTable;
    return *t;
}

// The SpmatLocal whose CSR blocks, concatenated in blockStarts order, hold the entries of a value vector of `order`
// (the one algorithm() works on for that mode), and the global S-row of local index 0 in block b of it: S keeps
// the S-rows as its local rows, ST as its local columns.  Exact wherever check_full_rows passes.
SpmatLocal *values_matrix(const Distributed_Sparse &d, KernelMode order) {
    bool in_ST = order == k_sddmmB;
    if (const Sparse15D_Dense_Shift *ds = dynamic_cast<const Sparse15D_Dense_Shift *>(&d))
        in_ST = (ds->fusionApproach == 1) == (order == k_sddmmA);  // fusion 1 keeps A-order values in ST's blocks
    else if (dynamic_cast<const Sparse25D_Cannon_Dense *>(&d))
        in_ST = order == k_sddmmA;  // blocks stored transposed: A-order values in ST's block
    return in_ST ? d.ST.get() : d.S.get();
}
int64_t values_row_offset(const Distributed_Sparse &d, const SpmatLocal &m, int block) {
    // p = 1: one block starting at row 0.  1.5D dense shift: S holds block row grid->i (height localArows * c), block b
    // of ST holds S-rows [b * localArows, (b + 1) * localArows)
    if (d.p == 1) return 0;
    return &m == d.ST.get() ? (int64_t)block * d.localArows : (int64_t)d.grid->i * d.localArows * d.c;
}
// The same for S-columns (additive attention), with the A and B roles swapped: block b of S holds S-columns
// [b * localBrows, (b + 1) * localBrows), ST holds block row grid->i (height localBrows * c) of S^T.
int64_t values_col_offset(const Distributed_Sparse &d, const SpmatLocal &m, int block) {
    if (d.p == 1) return 0;
    return &m == d.ST.get() ? (int64_t)d.grid->i * d.localBrows * d.c : (int64_t)block * d.localBrows;
}

// For each block of a value vector of `order` with n entries that has entries: fn(its first entry, its entry count,
// the index array that holds its entries' local S-rows (columns == false) or S-columns (columns == true), and the
// offset that makes them global), from the CSR blocks that hold that order
template <typename F>
void for_entry_index(Distributed_Sparse &d, KernelMode order, int64_t n, bool columns, const string &who, F fn) {
    SpmatLocal &m = *values_matrix(d, order);
    const bool is_ST = &m == d.ST.get();
    if ((int64_t)m.blockStarts.back() != n) throw hnh::Error(HNH_E_INVALID, who + ": the value vector does not cover the local blocks");
    for (size_t b = 0; b + 1 < m.blockStarts.size(); b++) {
        const int64_t off = (int64_t)m.blockStarts[b], nb = (int64_t)m.blockStarts[b + 1] - off;
        if (nb == 0) continue;
        CSRLocal *blk = m.csr_blocks[b];
        if (blk == nullptr || blk->num_coords != nb)
            throw hnh::Error(HNH_E_INVALID, who + ": block " + to_string(b) + " does not match its value range");
        // S stores its rows as rows, ST as columns; a transposed block swaps the two
        const bool stored_row = (is_ST == blk->transpose) != columns;
        const int64_t *idx = stored_row ? blk->row_idx_device() : blk->getActive()->col_idx.data();
        fn(off, nb, idx, columns ? values_col_offset(d, m, (int)b) : values_row_offset(d, m, (int)b));
    }
}

// keys[i] = the global S-row (columns == false) or S-column (columns == true) of entry i of a value vector of `order`
// with n entries
void entry_keys(Distributed_Sparse &d, KernelMode order, int64_t n, int32_t *keys, bool columns, cudaStream_t s) {
    for_entry_index(d, order, n, columns, "edgeSoftmax", [&](int64_t off, int64_t nb, const int64_t *idx, int64_t offset) {
        hnh::abi_check(hnh_edge_keys_from_index(keys + off, idx, nb, offset, s), "edge_keys_from_index");
    });
}

EdgeRows &edge_rows(Distributed_Sparse &d, KernelMode order, int64_t n) {
    if (order != k_sddmmA && order != k_sddmmB)
        throw hnh::Error(HNH_E_INVALID, "edgeSoftmax: the value order must be k_sddmmA or k_sddmmB");
    const int64_t want = order == k_sddmmA ? d.num_S_values() : d.num_ST_values();
    if (n != want)
        throw hnh::Error(HNH_E_INVALID, "edgeSoftmax: the value vector has " + to_string(n) + " entries, this order " + to_string(want));
    std::unique_ptr<EdgeRows> *slot;
    {
        std::lock_guard<std::mutex> lock(edge_rows_mutex);
        slot = &edge_rows_table()[&d][order == k_sddmmA ? 0 : 1];
    }
    if (*slot) return **slot;
    const int64_t M = d.M;
    if (M >= INT32_MAX) throw hnh::Error(HNH_E_INVALID, "edgeSoftmax: S has " + to_string(M) + " rows; at most 2^31 - 2");
    cudaStream_t s = Runtime::get().compute_stream();
    std::unique_ptr<EdgeRows> e(new EdgeRows);
    e->n = n;
    e->keys.resize((size_t)n);
    e->perm.resize((size_t)n);
    e->row_start.resize((size_t)M + 1);
    e->piece_first.resize((size_t)M + 1);
    const int64_t bound = hnh_edge_softmax_piece_bound(n, M);
    if (bound < 0) hnh::abi_check((int)bound, "edge_softmax_piece_bound");
    e->piece_row.resize((size_t)std::max<int64_t>(bound, 1));
    entry_keys(d, order, n, e->keys.data(), false, s);
    int64_t pieces = 0;
    hnh::abi_check(hnh_edge_softmax_plan(e->keys.data(), n, M, e->perm.data(), e->row_start.data(), e->piece_first.data(),
                                         e->piece_row.data(), (int64_t)e->piece_row.size(), &pieces, s),
                   "edge_softmax_plan");
    e->pieces = pieces;
    *slot = std::move(e);
    return **slot;
}

// edge_rows with the entries' S-columns (additive attention)
EdgeRows &edge_cols(Distributed_Sparse &d, KernelMode order, int64_t n) {
    EdgeRows &e = edge_rows(d, order, n);
    if (e.has_cols) return e;
    if (d.N >= INT32_MAX) throw hnh::Error(HNH_E_INVALID, "additive attention: S has " + to_string(d.N) + " columns; at most 2^31 - 2");
    e.cols.resize((size_t)n);
    entry_keys(d, order, n, e.cols.data(), true, Runtime::get().compute_stream());
    e.has_cols = true;
    return e;
}

// edge_cols of the A order with the entries grouped by S-column, as edge_rows groups them by S-row
EdgeRows &edge_col_plan(Distributed_Sparse &d, int64_t n) {
    EdgeRows &e = edge_cols(d, k_sddmmA, n);
    if (e.col_pieces >= 0) return e;
    const int64_t N = d.N;
    e.col_perm.resize((size_t)n);
    e.col_start.resize((size_t)N + 1);
    e.col_piece_first.resize((size_t)N + 1);
    const int64_t bound = hnh_edge_softmax_piece_bound(n, N);
    if (bound < 0) hnh::abi_check((int)bound, "edge_softmax_piece_bound");
    e.col_piece_row.resize((size_t)std::max<int64_t>(bound, 1));
    int64_t pieces = 0;
    hnh::abi_check(hnh_edge_softmax_plan(e.cols.data(), n, N, e.col_perm.data(), e.col_start.data(), e.col_piece_first.data(),
                                         e.col_piece_row.data(), (int64_t)e.col_piece_row.size(), &pieces,
                                         Runtime::get().compute_stream()),
                   "edge_softmax_plan");
    e.col_pieces = pieces;
    return e;
}

}  // namespace

void Distributed_Sparse::entryCoordinates(KernelMode order, VectorXd &rows, VectorXd &cols) {
    check_full_rows("entryCoordinates");
    if (order != k_sddmmA && order != k_sddmmB)
        throw hnh::Error(HNH_E_INVALID, "entryCoordinates: the value order must be k_sddmmA or k_sddmmB");
    const int64_t n = order == k_sddmmA ? num_S_values() : num_ST_values();
    rows.resize(n);
    cols.resize(n);
    for (bool columns : {false, true}) {
        double *out = columns ? cols.data() : rows.data();
        for_entry_index(*this, order, n, columns, "entryCoordinates", [&](int64_t off, int64_t nb, const int64_t *idx, int64_t offset) {
            hnh::abi_check(hnh_entry_coords_from_index_f64(out + off, idx, nb, offset, compute()), "entry_coords_from_index");
        });
    }
}

void Distributed_Sparse::release_edge_softmax() {
    std::lock_guard<std::mutex> lock(edge_rows_mutex);
    edge_rows_table().erase(this);
}

namespace {
// dst op= over the world (sum or max), ordered on the compute stream
void allreduce_rows(double *d, int64_t n, bool max) {
    std::shared_ptr<hnh::Comm> world = hnh::Comm::world();
    if (world->size() == 1) return;
    Runtime &rt = Runtime::get();
    rt.chain(rt.compute_stream(), rt.comm_stream());
    if (max) world->allreduce_max_f64(d, (size_t)n, rt.comm_stream());
    else world->allreduce_sum_f64(d, (size_t)n, rt.comm_stream());
    rt.chain(rt.comm_stream(), rt.compute_stream());
}
}  // namespace

void Distributed_Sparse::edgeSoftmax(VectorXd &values, KernelMode order) {
    check_full_rows("edgeSoftmax");
    EdgeRows &e = edge_rows(*this, order, values.size());
    VectorXd piece_max(e.pieces), piece_sum(e.pieces), row_max(M), row_sum(M);
    hnh::abi_check(hnh_edge_softmax_stats_f64(values.data(), e.perm.data(), e.row_start.data(), e.piece_first.data(),
                                              e.piece_row.data(), M, e.pieces, piece_max.data(), piece_sum.data(),
                                              row_max.data(), row_sum.data(), compute()),
                   "edge_softmax_stats");
    if (p > 1) {
        VectorXd local_max = row_max;
        allreduce_rows(row_max.data(), M, true);
        hnh::abi_check(hnh_edge_softmax_rescale_f64(row_sum.data(), local_max.data(), row_max.data(), M, compute()),
                       "edge_softmax_rescale");
        allreduce_rows(row_sum.data(), M, false);
    }
    hnh::abi_check(hnh_edge_softmax_apply_f64(values.data(), values.data(), e.keys.data(), e.n, row_max.data(), row_sum.data(),
                                              compute()),
                   "edge_softmax_apply");
}

void Distributed_Sparse::edgeSoftmaxBackward(const VectorXd &alpha, VectorXd &grad, KernelMode order) {
    check_full_rows("edgeSoftmaxBackward");
    if (alpha.size() != grad.size())
        throw hnh::Error(HNH_E_INVALID, "edgeSoftmaxBackward: alpha has " + to_string(alpha.size()) + " entries, grad " +
                                            to_string(grad.size()));
    EdgeRows &e = edge_rows(*this, order, grad.size());
    VectorXd piece_dot(e.pieces), row_dot(M);
    hnh::abi_check(hnh_edge_softmax_dot_f64(alpha.data(), grad.data(), e.perm.data(), e.row_start.data(), e.piece_first.data(),
                                            e.piece_row.data(), M, e.pieces, piece_dot.data(), row_dot.data(), compute()),
                   "edge_softmax_dot");
    allreduce_rows(row_dot.data(), M, false);
    hnh::abi_check(hnh_edge_softmax_backward_f64(grad.data(), alpha.data(), grad.data(), e.keys.data(), e.n, row_dot.data(),
                                                 compute()),
                   "edge_softmax_backward");
}

// ---- additive attention --------------------------------------------------------------------------------------
void Distributed_Sparse::additiveScores(const VectorXd &s, const VectorXd &t, VectorXd &out, KernelMode order, double alpha,
                                        bool derivative) {
    check_full_rows("additiveScores");
    if (s.size() < M || t.size() < N)
        throw hnh::Error(HNH_E_INVALID, "additiveScores: s has " + to_string(s.size()) + " entries and t " + to_string(t.size()) +
                                            "; S is " + to_string(M) + " x " + to_string(N));
    EdgeRows &e = edge_cols(*this, order, out.size());
    hnh::abi_check(hnh_gat_edge_scores_f64(out.data(), s.data(), t.data(), e.keys.data(), e.cols.data(), e.n, alpha,
                                           derivative ? 1 : 0, compute()),
                   "gat_edge_scores");
}

void Distributed_Sparse::edgeSums(const VectorXd &values, VectorXd &row_sums, VectorXd &col_sums) {
    check_full_rows("edgeSums");
    if (row_sums.size() < M || col_sums.size() < N)
        throw hnh::Error(HNH_E_INVALID, "edgeSums: room for " + to_string(row_sums.size()) + " row sums and " +
                                            to_string(col_sums.size()) + " column sums; S is " + to_string(M) + " x " +
                                            to_string(N));
    EdgeRows &e = edge_col_plan(*this, values.size());
    VectorXd piece(std::max<int64_t>({e.pieces, e.col_pieces, 1}));
    row_sums.setZero();  // the entries past M / N stay 0
    col_sums.setZero();
    hnh::abi_check(hnh_edge_sum_f64(values.data(), e.perm.data(), e.row_start.data(), e.piece_first.data(), e.piece_row.data(), M,
                                    e.pieces, piece.data(), row_sums.data(), compute()),
                   "edge_sum rows");
    hnh::abi_check(hnh_edge_sum_f64(values.data(), e.col_perm.data(), e.col_start.data(), e.col_piece_first.data(),
                                    e.col_piece_row.data(), N, e.col_pieces, piece.data(), col_sums.data(), compute()),
                   "edge_sum columns");
    allreduce_rows(row_sums.data(), M, false);
    allreduce_rows(col_sums.data(), N, false);
}

// ---- GATv2 attention -----------------------------------------------------------------------------------------
namespace {
// dst[:, dst_col0 .. + cols) = src[:, src_col0 .. + cols) for matrices of the same height, on the compute stream
void copy_cols(DenseMatrix &dst, int64_t dst_col0, const DenseMatrix &src, int64_t src_col0, int64_t cols) {
    if (dst.rows() == 0 || cols == 0) return;
    const size_t d = sizeof(double);
    hnh::cuda_check(cudaMemcpy2DAsync(dst.data() + dst_col0, d * (size_t)dst.cols(), src.data() + src_col0, d * (size_t)src.cols(),
                                      d * (size_t)cols, (size_t)dst.rows(), cudaMemcpyDeviceToDevice, Runtime::get().compute_stream()),
                    "column copy");
}
}  // namespace

void Distributed_Sparse::gather_pass(KernelMode order, const vector<PassOperand> &A_side, const vector<PassOperand> &B_side,
                                     const PassKernel &kernel) {
    SpmatLocal &m = *values_matrix(*this, order);
    const bool is_ST = &m == ST.get();
    // block b with its entries, or null when it has none
    auto block = [&](int b) -> CSRLocal * {
        const int64_t nb = (int64_t)m.blockStarts[(size_t)b + 1] - (int64_t)m.blockStarts[(size_t)b];
        if (nb == 0) return nullptr;
        CSRLocal *blk = m.csr_blocks[(size_t)b];
        if (blk == nullptr || blk->num_coords != nb)
            throw hnh::Error(HNH_E_INVALID, "gather_pass: block " + to_string(b) + " does not match its value range");
        return blk;
    };
    // the operands' views at home
    auto home = [](const vector<PassOperand> &ops, bool gathered) {
        vector<PassView> v;
        for (const PassOperand &o : ops)
            v.push_back(gathered && o.written ? PassView{nullptr, 0} : PassView{o.m->data() + o.col0, o.m->cols()});
        return v;
    };
    auto run = [&](int b, CSRLocal &blk, bool rows_are_A, const vector<PassView> &R, int64_t R_rows, const vector<PassView> &Y,
                   int64_t Y_rows) {
        if (blk.rows > R_rows || blk.cols > Y_rows)
            throw hnh::Error(HNH_E_INVALID, "gather_pass: block " + to_string(b) + " (" + to_string(blk.rows) + " x " +
                                                to_string(blk.cols) + ") does not fit its dense operands (" + to_string(R_rows) +
                                                " and " + to_string(Y_rows) + " rows)");
        kernel(b, blk, rows_are_A, R.data(), Y.data());
    };
    if (p == 1) {
        const vector<PassView> hA = home(A_side, false), hB = home(B_side, false), gA = home(A_side, true), gB = home(B_side, true);
        for (int b = 0; b + 1 < (int)m.blockStarts.size(); b++) {
            CSRLocal *blk = block(b);
            if (blk == nullptr) continue;
            // S stores its rows as rows, ST as columns; a transposed block swaps the two
            const bool rows_are_A = is_ST == blk->transpose;
            run(b, *blk, rows_are_A, rows_are_A ? hA : hB, (rows_are_A ? A_side : B_side).front().m->rows(), rows_are_A ? gB : gA,
                (rows_are_A ? B_side : A_side).front().m->rows());
        }
        return;
    }
    // check_full_rows has passed: 1.5D dense shift, fusion 1 at any c or fusion 2 at c = 1.  Its blocks are stored
    // transposed exactly under fusion 1 (Sparse15D_Dense_Shift's constructor).
    Sparse15D_Dense_Shift &ds = dynamic_cast<Sparse15D_Dense_Shift &>(*this);
    const bool fusion1 = ds.fusionApproach == 1;
    const bool rows_are_A = is_ST == fusion1;
    const vector<PassOperand> &rowOps = rows_are_A ? A_side : B_side, &gathOps = rows_are_A ? B_side : A_side;
    // A side as one matrix that can travel: the operand itself when it is the side's only one (written ones left
    // out with `skip_written`) and a whole matrix, else the windows packed side by side.  offset[i]: operand i's
    // first column in it (-1: left out).
    struct Travelling {
        DenseMatrix packed;
        DenseMatrix *whole = nullptr;
        vector<int64_t> offset;
        Travelling(const vector<PassOperand> &ops, bool skip_written) {
            int64_t width = 0, n = 0;
            const PassOperand *only = nullptr;
            for (const PassOperand &o : ops) {
                const bool in = !(skip_written && o.written);
                offset.push_back(in ? width : -1);
                if (in) {
                    width += o.cols;
                    n++;
                    only = &o;
                }
            }
            if (n == 1 && only->col0 == 0 && only->cols == only->m->cols()) {
                whole = only->m;
                return;
            }
            packed.resize(ops.front().m->rows(), width);
            for (size_t i = 0; i < ops.size(); i++)
                if (offset[i] >= 0) copy_cols(packed, offset[i], *ops[i].m, ops[i].col0, ops[i].cols);
        }
        DenseMatrix &mat() { return whole ? *whole : packed; }
        vector<PassView> views(DenseMatrix &at) const {
            vector<PassView> v;
            for (int64_t off : offset) v.push_back(off < 0 ? PassView{nullptr, 0} : PassView{at.data() + off, at.cols()});
            return v;
        }
    };
    if (!fusion1) {
        // local kernel fusion, c = 1: the stored-row side stays, the gathered side rides read-only
        if (c != 1) throw hnh::Error(HNH_E_INVALID, "gather_pass: local kernel fusion at c > 1");
        const vector<PassView> R = home(rowOps, false);
        Travelling g(gathOps, true);
        ring_dense(g.mat(), grid->col_world, true, "Cyclic Shift Time", "Computation Time", [&](int step, DenseMatrix &shard) {
            const int b = ds.block_at(step);
            if (CSRLocal *blk = block(b)) run(b, *blk, rows_are_A, R, rowOps.front().m->rows(), g.views(shard), shard.rows());
        });
        return;
    }
    // replication reuse: the gathered side is stationary, all-gathered over the layer (row_world); the stored-row side
    // rides the column ring
    vector<PassView> Y = home(gathOps, true);
    int64_t Y_rows = gathOps.front().m->rows();
    std::optional<Travelling> g;
    DenseMatrix replicated;
    if (c > 1) {
        g.emplace(gathOps, true);
        Runtime &rt = Runtime::get();
        replicated.resize(g->mat().rows() * c, g->mat().cols());
        rt.chain(compute(), comm());
        region_begin("Replication Time", comm());
        grid->row_world->allgather(g->mat().data(), replicated.data(), sizeof(double) * (size_t)g->mat().size(), comm());
        region_end("Replication Time", comm());
        rt.chain(comm(), compute());
        Y = g->views(replicated);
        Y_rows = replicated.rows();
    }
    // written operands ride with the rows they belong to, on the output-riding ring (kernel and shift alternate), and
    // are back home after the last shift
    bool written = false;
    for (const PassOperand &o : rowOps) written = written || o.written;
    Travelling r(rowOps, false);
    ring_dense(r.mat(), grid->col_world, !written, "Cyclic Shift Time", "Computation Time", [&](int step, DenseMatrix &shard) {
        const int b = ds.block_at(step);
        if (CSRLocal *blk = block(b)) run(b, *blk, rows_are_A, r.views(shard), shard.rows(), Y, Y_rows);
    });
    if (r.whole == nullptr)
        for (size_t i = 0; i < rowOps.size(); i++)
            if (rowOps[i].written) copy_cols(*rowOps[i].m, rowOps[i].col0, r.packed, r.offset[i], rowOps[i].cols);
}

void Distributed_Sparse::gatv2_pass(KernelMode order, DenseMatrix &localA, DenseMatrix &localB, DenseMatrix *dA, DenseMatrix *dB,
                                    const Gatv2Kernel &kernel) {
    const int64_t r = localA.cols();
    // each side: its operand, then its gradient; the gradients ride with the stored rows as one 2r-wide matrix
    vector<PassOperand> A_side{{&localA, 0, r, false}}, B_side{{&localB, 0, r, false}};
    const bool grads = dA != nullptr || dB != nullptr;
    if (grads) {
        A_side.push_back({dA, 0, r, true});
        B_side.push_back({dB, 0, r, true});
    }
    gather_pass(order, A_side, B_side, [&](int b, CSRLocal &blk, bool, const PassView *R, const PassView *Y) {
        kernel(b, blk, R[0].p, R[0].ld, Y[0].p, Y[0].ld, grads ? R[1].p : nullptr, grads ? R[1].ld : r);
    });
}

namespace {
void check_gatv2_operands(const Distributed_Sparse &d, const char *who, const DenseMatrix &A, const DenseMatrix &B, const VectorXd &a) {
    const int64_t r = a.size();
    if (r < 1 || r > INT32_MAX || A.cols() != r || B.cols() != r)
        throw hnh::Error(HNH_E_INVALID, string(who) + ": the operands are " + to_string(A.cols()) + " and " + to_string(B.cols()) +
                                            " wide, the attention vector has " + to_string(r) + " entries");
    if (A.rows() != d.localArows || B.rows() != d.localBrows)
        throw hnh::Error(HNH_E_INVALID, string(who) + ": the operands have " + to_string(A.rows()) + " and " + to_string(B.rows()) +
                                            " rows; like_A_matrix / like_B_matrix have " + to_string(d.localArows) + " and " +
                                            to_string(d.localBrows));
}
int64_t order_size(Distributed_Sparse &d, const char *who, KernelMode order) {
    if (order != k_sddmmA && order != k_sddmmB)
        throw hnh::Error(HNH_E_INVALID, string(who) + ": the value order must be k_sddmmA or k_sddmmB");
    return order == k_sddmmA ? d.num_S_values() : d.num_ST_values();
}
}  // namespace

void Distributed_Sparse::gatv2Scores(DenseMatrix &localA, DenseMatrix &localB, const VectorXd &a, VectorXd &out, KernelMode order,
                                     double alpha) {
    check_full_rows("gatv2Scores");
    check_gatv2_operands(*this, "gatv2Scores", localA, localB, a);
    const int64_t want = order_size(*this, "gatv2Scores", order);
    if (out.size() != want)
        throw hnh::Error(HNH_E_INVALID, "gatv2Scores: the value vector has " + to_string(out.size()) + " entries, this order " + to_string(want));
    SpmatLocal &m = *values_matrix(*this, order);
    const int r = (int)a.size();
    gatv2_pass(order, localA, localB, nullptr, nullptr,
               [&](int b, CSRLocal &blk, const double *R, int64_t ldr, const double *Y, int64_t ldy, double *, int64_t) {
                   CSRHandle *h = blk.getActive();
                   hnh::abi_check(hnh_gatv2_scores_f64(h->rowStart.data(), h->col_idx.data(), blk.rows, blk.num_coords, R, ldr, Y, ldy,
                                                       a.data(), r, alpha, out.data() + (int64_t)m.blockStarts[(size_t)b], compute()),
                                  "gatv2_scores");
               });
}

void Distributed_Sparse::gatv2Backward(DenseMatrix &localA, DenseMatrix &localB, const VectorXd &a, const VectorXd &grad_A,
                                       const VectorXd &grad_B, DenseMatrix &dA, DenseMatrix &dB, VectorXd &da, double alpha) {
    check_full_rows("gatv2Backward");
    check_gatv2_operands(*this, "gatv2Backward", localA, localB, a);
    check_gatv2_operands(*this, "gatv2Backward (gradients)", dA, dB, a);
    if (grad_A.size() != num_S_values() || grad_B.size() != num_ST_values())
        throw hnh::Error(HNH_E_INVALID, "gatv2Backward: the gradients have " + to_string(grad_A.size()) + " and " +
                                            to_string(grad_B.size()) + " entries, the A and B orders " + to_string(num_S_values()) +
                                            " and " + to_string(num_ST_values()));
    const int r = (int)a.size();
    VectorXd da_local = VectorXd::Constant(r, 0.0);
    // the da partials of the A-order blocks (one kernel at a time uses it)
    int64_t most_rows = 0;
    for (CSRLocal *blk : values_matrix(*this, k_sddmmA)->csr_blocks)
        if (blk) most_rows = std::max(most_rows, blk->rows);
    const int64_t ws_bytes = hnh_gatv2_grad_workspace_bytes(most_rows, r);
    if (ws_bytes < 0) hnh::abi_check((int)ws_bytes, "gatv2_grad_workspace_bytes");
    VectorXd workspace(std::max<int64_t>((ws_bytes + 7) / 8, 1));
    for (KernelMode order : {k_sddmmA, k_sddmmB}) {
        SpmatLocal &m = *values_matrix(*this, order);
        const VectorXd &g = order == k_sddmmA ? grad_A : grad_B;
        // da counts every stored entry once over all ranks: from the A order only
        const bool with_da = order == k_sddmmA;
        gatv2_pass(order, localA, localB, &dA, &dB,
                   [&](int b, CSRLocal &blk, const double *R, int64_t ldr, const double *Y, int64_t ldy, double *dR, int64_t lddr) {
                       const size_t ws = with_da ? (size_t)workspace.size() * sizeof(double) : 0;
                       CSRHandle *h = blk.getActive();
                       hnh::abi_check(hnh_gatv2_grad_f64(h->rowStart.data(), h->col_idx.data(), g.data() + (int64_t)m.blockStarts[(size_t)b],
                                                         blk.rows, blk.num_coords, R, ldr, Y, ldy, a.data(), r, alpha, dR, lddr,
                                                         with_da ? da_local.data() : nullptr, with_da ? workspace.data() : nullptr, ws,
                                                         compute()),
                                      "gatv2_grad");
                   });
    }
    allreduce_rows(da_local.data(), r, false);
    da = std::move(da_local);
}

// ---- fused sparse attention ------------------------------------------------------------------------------------
namespace {
// the shape checks of sparseAttention / sparseAttentionBackward; returns the head width d = r / heads
int64_t check_attention(const Distributed_Sparse &dist, const string &who, std::initializer_list<const DenseMatrix *> A_like,
                        std::initializer_list<const DenseMatrix *> B_like, const DenseMatrix &L, int heads, double scale) {
    const int64_t r = (*A_like.begin())->cols();
    for (const DenseMatrix *m : A_like)
        if (m->rows() != dist.localArows || m->cols() != r)
            throw hnh::Error(HNH_E_INVALID, who + ": an A-shaped operand is " + to_string(m->rows()) + " x " + to_string(m->cols()) +
                                                "; like_A_matrix has " + to_string(dist.localArows) + " rows, Q is " + to_string(r) +
                                                " wide");
    for (const DenseMatrix *m : B_like)
        if (m->rows() != dist.localBrows || m->cols() != r)
            throw hnh::Error(HNH_E_INVALID, who + ": a B-shaped operand is " + to_string(m->rows()) + " x " + to_string(m->cols()) +
                                                "; like_B_matrix has " + to_string(dist.localBrows) + " rows, Q is " + to_string(r) +
                                                " wide");
    if (heads < 1 || r < 1 || r % heads != 0 || r / heads > INT32_MAX)
        throw hnh::Error(HNH_E_INVALID, who + ": " + to_string(heads) + " heads do not divide the width " + to_string(r));
    if (!std::isfinite(scale)) throw hnh::Error(HNH_E_INVALID, who + ": the scale must be finite");
    if (L.rows() != dist.localArows || L.cols() != heads)
        throw hnh::Error(HNH_E_INVALID, who + ": L is " + to_string(L.rows()) + " x " + to_string(L.cols()) + ", not localArows x heads = " +
                                            to_string(dist.localArows) + " x " + to_string(heads));
    return r / heads;
}
void need_rows(bool rows_are_A, bool want, const char *who) {
    if (rows_are_A != want)
        throw hnh::Error(HNH_E_INVALID, string(who) + ": a block of this order does not hold the " + (want ? "query" : "key") +
                                            " side as its stored rows");
}
// the dropout checks: a probability in [0, 1), and global S-rows and S-columns that fit the mask's 32-bit halves
void check_dropout(const Distributed_Sparse &dist, const string &who, double dropout) {
    if (!(dropout >= 0.0 && dropout < 1.0))
        throw hnh::Error(HNH_E_INVALID, who + ": the dropout probability must lie in [0, 1), got " + std::to_string(dropout));
    if (dropout > 0.0 && (dist.M > ((int64_t)1 << 32) || dist.N > ((int64_t)1 << 32)))
        throw hnh::Error(HNH_E_INVALID, who + ": dropout keys S-rows and S-columns by 32 bits; S is " + to_string(dist.M) + " x " +
                                            to_string(dist.N));
}
// The (u0, v0) of block b of `order`'s values matrix: the global S-row and S-column of its local row and column 0,
// as the edge softmax keys its entries (entry_keys)
struct BlockOrigin {
    const Distributed_Sparse &dist;
    const SpmatLocal &m;
    BlockOrigin(const Distributed_Sparse &d, KernelMode order) : dist(d), m(*values_matrix(d, order)) {}
    int64_t u0(int b) const { return values_row_offset(dist, m, b); }
    int64_t v0(int b) const { return values_col_offset(dist, m, b); }
};
// A bias vector of `order` as sparseAttention reads it: block b of head h starts at at(h, b)
struct BiasView {
    const VectorXd *v = nullptr;
    VectorXd *grad = nullptr;
    const SpmatLocal *m = nullptr;
    int64_t head_stride = 0;  // n for a per-head bias, 0 for a shared one
    const double *at(int h, int b) const { return v->data() + h * head_stride + (int64_t)m->blockStarts[(size_t)b]; }
    double *grad_at(int h, int b) const {
        return grad ? grad->data() + h * head_stride + (int64_t)m->blockStarts[(size_t)b] : nullptr;
    }
};
// The head multiplicity of a bias of `order`: 1 (shared), heads (per head) or 0 (either: the order has no local
// entries); HNH_E_INVALID for any other length
int64_t bias_heads(Distributed_Sparse &d, const string &who, const char *name, const VectorXd &b, KernelMode order, int heads) {
    const int64_t n = order == k_sddmmA ? d.num_S_values() : d.num_ST_values();
    if (n == 0 && b.size() == 0) return 0;
    if (b.size() == n) return 1;
    if (b.size() == (int64_t)heads * n) return heads;
    throw hnh::Error(HNH_E_INVALID, who + ": " + name + " has " + to_string(b.size()) + " entries; its order has " + to_string(n) +
                                        " per head and there are " + to_string(heads) + " heads");
}
BiasView bias_view(Distributed_Sparse &d, const VectorXd *b, VectorXd *grad, KernelMode order, int64_t multiplicity) {
    BiasView v;
    if (b == nullptr) return v;
    v.v = b;
    v.grad = grad;
    v.m = values_matrix(d, order);
    v.head_stride = multiplicity > 1 ? (order == k_sddmmA ? d.num_S_values() : d.num_ST_values()) : 0;
    return v;
}
// Edge features of `order` as sparseAttention reads them: block b of head h starts at at(h, b), leading dimension r
// (its gradient likewise); a null E gives null pointers
struct EdgeView {
    const DenseMatrix *E = nullptr;
    DenseMatrix *grad = nullptr;
    const SpmatLocal *m = nullptr;
    int64_t d = 0;
    int64_t offset(int h, int b) const { return (int64_t)m->blockStarts[(size_t)b] * E->cols() + h * d; }
    const double *at(int h, int b) const { return E ? E->data() + offset(h, b) : nullptr; }
    int64_t ld() const { return E ? E->cols() : d; }
    double *grad_at(int h, int b) const { return grad ? grad->data() + offset(h, b) : nullptr; }
};
// The view of edge features of `order`, checked to be n x r (n that order's local entry count); HNH_E_INVALID else
EdgeView edge_view(Distributed_Sparse &dist, const string &who, const char *name, const DenseMatrix *E, DenseMatrix *grad,
                   KernelMode order, int64_t r, int64_t d) {
    EdgeView v;
    if (E == nullptr) return v;
    const int64_t n = order == k_sddmmA ? dist.num_S_values() : dist.num_ST_values();
    if (E->rows() != n || E->cols() != r)
        throw hnh::Error(HNH_E_INVALID, who + ": " + name + " is " + to_string(E->rows()) + " x " + to_string(E->cols()) +
                                            "; its order has " + to_string(n) + " entries and Q is " + to_string(r) + " wide");
    v.E = E;
    v.grad = grad;
    v.m = values_matrix(dist, order);
    v.d = d;
    return v;
}
}  // namespace

void Distributed_Sparse::sparseAttention(DenseMatrix &Q, DenseMatrix &K, DenseMatrix &V, DenseMatrix &Z, DenseMatrix &L, int heads,
                                         double scale) {
    sparseAttention(Q, K, V, Z, L, heads, scale, 0.0, 0);
}

void Distributed_Sparse::sparseAttentionBackward(DenseMatrix &Q, DenseMatrix &K, DenseMatrix &V, DenseMatrix &Z, DenseMatrix &L,
                                                 DenseMatrix &dZ, DenseMatrix &dQ, DenseMatrix &dK, DenseMatrix &dV, int heads,
                                                 double scale) {
    sparseAttentionBackward(Q, K, V, Z, L, dZ, dQ, dK, dV, heads, scale, 0.0, 0);
}

void Distributed_Sparse::sparseAttention(DenseMatrix &Q, DenseMatrix &K, DenseMatrix &V, DenseMatrix &Z, DenseMatrix &L, int heads,
                                         double scale, double dropout, uint64_t seed) {
    sparseAttention(Q, K, V, Z, L, heads, scale, dropout, seed, nullptr);
}

void Distributed_Sparse::sparseAttentionBackward(DenseMatrix &Q, DenseMatrix &K, DenseMatrix &V, DenseMatrix &Z, DenseMatrix &L,
                                                 DenseMatrix &dZ, DenseMatrix &dQ, DenseMatrix &dK, DenseMatrix &dV, int heads,
                                                 double scale, double dropout, uint64_t seed) {
    sparseAttentionBackward(Q, K, V, Z, L, dZ, dQ, dK, dV, heads, scale, dropout, seed, nullptr, nullptr, nullptr, nullptr);
}

void Distributed_Sparse::sparseAttention(DenseMatrix &Q, DenseMatrix &K, DenseMatrix &V, DenseMatrix &Z, DenseMatrix &L, int heads,
                                         double scale, double dropout, uint64_t seed, const VectorXd *bias) {
    sparseAttention(Q, K, V, Z, L, heads, scale, dropout, seed, bias, nullptr);
}

void Distributed_Sparse::sparseAttentionBackward(DenseMatrix &Q, DenseMatrix &K, DenseMatrix &V, DenseMatrix &Z, DenseMatrix &L,
                                                 DenseMatrix &dZ, DenseMatrix &dQ, DenseMatrix &dK, DenseMatrix &dV, int heads,
                                                 double scale, double dropout, uint64_t seed, const VectorXd *bias_A,
                                                 const VectorXd *bias_B, VectorXd *dbias_A, VectorXd *dbias_B) {
    sparseAttentionBackward(Q, K, V, Z, L, dZ, dQ, dK, dV, heads, scale, dropout, seed, bias_A, bias_B, dbias_A, dbias_B, nullptr,
                            nullptr, nullptr);
}

void Distributed_Sparse::sparseAttention(DenseMatrix &Q, DenseMatrix &K, DenseMatrix &V, DenseMatrix &Z, DenseMatrix &L, int heads,
                                         double scale, double dropout, uint64_t seed, const VectorXd *bias, const DenseMatrix *edge) {
    check_full_rows("sparseAttention");
    const int64_t d = check_attention(*this, "sparseAttention", {&Q, &Z}, {&K, &V}, L, heads, scale);
    check_dropout(*this, "sparseAttention", dropout);
    const BiasView bv =
        bias_view(*this, bias, nullptr, k_sddmmA, bias ? bias_heads(*this, "sparseAttention", "the bias", *bias, k_sddmmA, heads) : 0);
    const EdgeView ev = edge_view(*this, "sparseAttention", "the edge features", edge, nullptr, k_sddmmA, Q.cols(), d);
    const BlockOrigin at(*this, k_sddmmA);
    // the online-softmax state of row u, head h: acc in Z's window, m in L[u, h], s in s[u, h]; m is not read while
    // s = 0, and the finish turns (acc, m, s) into (Z, L) in place
    Z.setZero();
    DenseMatrix s(localArows, heads);
    s.setZero();
    for (int h = 0; h < heads; h++) {
        const vector<PassOperand> A_side{{&Q, h * d, d, false}, {&Z, h * d, d, true}, {&L, h, 1, true}, {&s, h, 1, true}};
        const vector<PassOperand> B_side{{&K, h * d, d, false}, {&V, h * d, d, false}};
        gather_pass(k_sddmmA, A_side, B_side, [&](int b, CSRLocal &blk, bool rows_are_A, const PassView *R, const PassView *Y) {
            need_rows(rows_are_A, true, "sparseAttention");
            CSRHandle *hd = blk.getActive();
            if (edge)
                hnh::abi_check(hnh_sparse_attention_step_edge_f64(hd->rowStart.data(), hd->col_idx.data(), blk.rows, blk.num_coords,
                                                                  (int)d, R[0].p, R[0].ld, Y[0].p, Y[0].ld, Y[1].p, Y[1].ld, scale,
                                                                  R[1].p, R[1].ld, R[2].p, R[2].ld, R[3].p, R[3].ld, dropout,
                                                                  seed + (uint64_t)h, at.u0(b), at.v0(b),
                                                                  bias ? bv.at(h, b) : nullptr, ev.at(h, b), ev.ld(), compute()),
                               "sparse_attention_step_edge");
            else if (bias)
                hnh::abi_check(hnh_sparse_attention_step_bias_f64(hd->rowStart.data(), hd->col_idx.data(), blk.rows, blk.num_coords,
                                                                  (int)d, R[0].p, R[0].ld, Y[0].p, Y[0].ld, Y[1].p, Y[1].ld, scale,
                                                                  R[1].p, R[1].ld, R[2].p, R[2].ld, R[3].p, R[3].ld, dropout,
                                                                  seed + (uint64_t)h, at.u0(b), at.v0(b), bv.at(h, b), compute()),
                               "sparse_attention_step_bias");
            else if (dropout == 0.0)
                hnh::abi_check(hnh_sparse_attention_step_f64(hd->rowStart.data(), hd->col_idx.data(), blk.rows, blk.num_coords,
                                                             (int)d, R[0].p, R[0].ld, Y[0].p, Y[0].ld, Y[1].p, Y[1].ld, scale, R[1].p,
                                                             R[1].ld, R[2].p, R[2].ld, R[3].p, R[3].ld, compute()),
                               "sparse_attention_step");
            else
                hnh::abi_check(hnh_sparse_attention_step_dropout_f64(hd->rowStart.data(), hd->col_idx.data(), blk.rows,
                                                                     blk.num_coords, (int)d, R[0].p, R[0].ld, Y[0].p, Y[0].ld,
                                                                     Y[1].p, Y[1].ld, scale, R[1].p, R[1].ld, R[2].p, R[2].ld,
                                                                     R[3].p, R[3].ld, dropout, seed + (uint64_t)h, at.u0(b),
                                                                     at.v0(b), compute()),
                               "sparse_attention_step_dropout");
        });
        hnh::abi_check(hnh_sparse_attention_finish_f64(localArows, (int)d, Z.data() + h * d, Z.cols(), L.data() + h, heads,
                                                       s.data() + h, heads, Z.data() + h * d, Z.cols(), L.data() + h, heads,
                                                       compute()),
                       "sparse_attention_finish");
    }
}

void Distributed_Sparse::sparseAttentionBackward(DenseMatrix &Q, DenseMatrix &K, DenseMatrix &V, DenseMatrix &Z, DenseMatrix &L,
                                                 DenseMatrix &dZ, DenseMatrix &dQ, DenseMatrix &dK, DenseMatrix &dV, int heads,
                                                 double scale, double dropout, uint64_t seed, const VectorXd *bias_A,
                                                 const VectorXd *bias_B, VectorXd *dbias_A, VectorXd *dbias_B,
                                                 const DenseMatrix *edge_A, const DenseMatrix *edge_B, DenseMatrix *dedge) {
    const string who = "sparseAttentionBackward";
    check_full_rows(who);
    const int64_t d = check_attention(*this, who, {&Q, &Z, &dZ, &dQ}, {&K, &V, &dK, &dV}, L, heads, scale);
    check_dropout(*this, who, dropout);
    if ((bias_A == nullptr) != (bias_B == nullptr))
        throw hnh::Error(HNH_E_INVALID, who + ": a bias needs both orders, bias_A and bias_B");
    if ((dbias_A && !bias_A) || (dbias_B && !bias_B)) throw hnh::Error(HNH_E_INVALID, who + ": a bias gradient without its bias");
    for (const VectorXd *g : {(const VectorXd *)dbias_A, (const VectorXd *)dbias_B})
        if (g && (g == bias_A || g == bias_B)) throw hnh::Error(HNH_E_INVALID, who + ": a bias gradient may not be a bias");
    if (dbias_A && dbias_A == dbias_B) throw hnh::Error(HNH_E_INVALID, who + ": dbias_A and dbias_B are one vector");
    const bool with_bias = bias_A != nullptr;
    int64_t mA = 0, mB = 0;
    if (with_bias) {
        mA = bias_heads(*this, who, "bias_A", *bias_A, k_sddmmA, heads);
        mB = bias_heads(*this, who, "bias_B", *bias_B, k_sddmmB, heads);
        if (mA != 0 && mB != 0 && mA != mB)
            throw hnh::Error(HNH_E_INVALID, who + ": bias_A is " + (mA > 1 ? "per head" : "shared") + ", bias_B " +
                                                (mB > 1 ? "per head" : "shared"));
    }
    if ((edge_A == nullptr) != (edge_B == nullptr))
        throw hnh::Error(HNH_E_INVALID, who + ": edge features need both orders, edge_A and edge_B");
    if (dedge && !edge_A) throw hnh::Error(HNH_E_INVALID, who + ": an edge-feature gradient without edge features");
    for (const DenseMatrix *o : {(const DenseMatrix *)&Q, (const DenseMatrix *)&K, (const DenseMatrix *)&V, (const DenseMatrix *)&Z,
                                 (const DenseMatrix *)&L, (const DenseMatrix *)&dZ, (const DenseMatrix *)&dQ, (const DenseMatrix *)&dK,
                                 (const DenseMatrix *)&dV, edge_A, edge_B})
        if (dedge && dedge == o) throw hnh::Error(HNH_E_INVALID, who + ": dedge may not be another operand of the call");
    const bool with_edge = edge_A != nullptr;
    const EdgeView evA = edge_view(*this, who, "edge_A", edge_A, dedge, k_sddmmA, Q.cols(), d),
                   evB = edge_view(*this, who, "edge_B", edge_B, nullptr, k_sddmmB, Q.cols(), d);
    if (dedge) dedge->resize(edge_A->rows(), edge_A->cols());
    const BlockOrigin atA(*this, k_sddmmA), atB(*this, k_sddmmB);
    for (auto [g, b] : {std::make_pair(dbias_A, bias_A), std::make_pair(dbias_B, bias_B)})
        if (g) {
            g->resize(b->size());
            g->setZero();
        }
    const BiasView bvA = bias_view(*this, bias_A, dbias_A, k_sddmmA, mA), bvB = bias_view(*this, bias_B, dbias_B, k_sddmmB, mB);
    // t[u, h] = <dZ_u,h, Z_u,h>: Z and dZ read as localArows * heads rows of d
    DenseMatrix t(localArows, heads);
    hnh::abi_check(hnh_batch_dot_f64(t.data(), dZ.data(), Z.data(), localArows * heads, (int)d, compute()), "batch_dot");
    dQ.setZero();
    dK.setZero();
    dV.setZero();
    for (int h = 0; h < heads; h++) {
        const int64_t w = h * d;
        // query rows own dQ (A order)
        gather_pass(k_sddmmA, {{&Q, w, d, false}, {&dZ, w, d, false}, {&L, h, 1, false}, {&t, h, 1, false}, {&dQ, w, d, true}},
                    {{&K, w, d, false}, {&V, w, d, false}},
                    [&](int b, CSRLocal &blk, bool rows_are_A, const PassView *R, const PassView *Y) {
                        need_rows(rows_are_A, true, "sparseAttentionBackward");
                        CSRHandle *hd = blk.getActive();
                        if (with_edge)
                            hnh::abi_check(hnh_sparse_attention_grad_q_edge_f64(
                                               hd->rowStart.data(), hd->col_idx.data(), blk.rows, blk.num_coords, (int)d, R[0].p,
                                               R[0].ld, R[1].p, R[1].ld, R[2].p, R[2].ld, R[3].p, R[3].ld, Y[0].p, Y[0].ld, Y[1].p,
                                               Y[1].ld, scale, R[4].p, R[4].ld, dropout, seed + (uint64_t)h, atA.u0(b), atA.v0(b),
                                               with_bias ? bvA.at(h, b) : nullptr, bvA.grad_at(h, b), evA.at(h, b), evA.ld(),
                                               evA.grad_at(h, b), evA.ld(), compute()),
                                           "sparse_attention_grad_q_edge");
                        else if (with_bias)
                            hnh::abi_check(hnh_sparse_attention_grad_q_bias_f64(
                                               hd->rowStart.data(), hd->col_idx.data(), blk.rows, blk.num_coords, (int)d, R[0].p,
                                               R[0].ld, R[1].p, R[1].ld, R[2].p, R[2].ld, R[3].p, R[3].ld, Y[0].p, Y[0].ld, Y[1].p,
                                               Y[1].ld, scale, R[4].p, R[4].ld, dropout, seed + (uint64_t)h, atA.u0(b), atA.v0(b),
                                               bvA.at(h, b), bvA.grad_at(h, b), compute()),
                                           "sparse_attention_grad_q_bias");
                        else if (dropout == 0.0)
                            hnh::abi_check(hnh_sparse_attention_grad_q_f64(hd->rowStart.data(), hd->col_idx.data(), blk.rows,
                                                                           blk.num_coords, (int)d, R[0].p, R[0].ld, R[1].p, R[1].ld,
                                                                           R[2].p, R[2].ld, R[3].p, R[3].ld, Y[0].p, Y[0].ld, Y[1].p,
                                                                           Y[1].ld, scale, R[4].p, R[4].ld, compute()),
                                           "sparse_attention_grad_q");
                        else
                            hnh::abi_check(hnh_sparse_attention_grad_q_dropout_f64(
                                               hd->rowStart.data(), hd->col_idx.data(), blk.rows, blk.num_coords, (int)d, R[0].p,
                                               R[0].ld, R[1].p, R[1].ld, R[2].p, R[2].ld, R[3].p, R[3].ld, Y[0].p, Y[0].ld, Y[1].p,
                                               Y[1].ld, scale, R[4].p, R[4].ld, dropout, seed + (uint64_t)h, atA.u0(b), atA.v0(b),
                                               compute()),
                                           "sparse_attention_grad_q_dropout");
                    });
        // key rows own dK and dV (B order)
        gather_pass(k_sddmmB, {{&Q, w, d, false}, {&dZ, w, d, false}, {&L, h, 1, false}, {&t, h, 1, false}},
                    {{&K, w, d, false}, {&V, w, d, false}, {&dK, w, d, true}, {&dV, w, d, true}},
                    [&](int b, CSRLocal &blk, bool rows_are_A, const PassView *R, const PassView *Y) {
                        need_rows(rows_are_A, false, "sparseAttentionBackward");
                        CSRHandle *hd = blk.getActive();
                        if (with_edge)
                            hnh::abi_check(hnh_sparse_attention_grad_kv_edge_f64(
                                               hd->rowStart.data(), hd->col_idx.data(), blk.rows, blk.num_coords, (int)d, R[0].p,
                                               R[0].ld, R[1].p, R[1].ld, Y[0].p, Y[0].ld, Y[1].p, Y[1].ld, Y[2].p, Y[2].ld, Y[3].p,
                                               Y[3].ld, scale, R[2].p, R[2].ld, R[3].p, R[3].ld, dropout, seed + (uint64_t)h,
                                               atB.u0(b), atB.v0(b), with_bias ? bvB.at(h, b) : nullptr, bvB.grad_at(h, b),
                                               evB.at(h, b), evB.ld(), compute()),
                                           "sparse_attention_grad_kv_edge");
                        else if (with_bias)
                            hnh::abi_check(hnh_sparse_attention_grad_kv_bias_f64(
                                               hd->rowStart.data(), hd->col_idx.data(), blk.rows, blk.num_coords, (int)d, R[0].p,
                                               R[0].ld, R[1].p, R[1].ld, Y[0].p, Y[0].ld, Y[1].p, Y[1].ld, Y[2].p, Y[2].ld, Y[3].p,
                                               Y[3].ld, scale, R[2].p, R[2].ld, R[3].p, R[3].ld, dropout, seed + (uint64_t)h,
                                               atB.u0(b), atB.v0(b), bvB.at(h, b), bvB.grad_at(h, b), compute()),
                                           "sparse_attention_grad_kv_bias");
                        else if (dropout == 0.0)
                            hnh::abi_check(hnh_sparse_attention_grad_kv_f64(hd->rowStart.data(), hd->col_idx.data(), blk.rows,
                                                                            blk.num_coords, (int)d, R[0].p, R[0].ld, R[1].p, R[1].ld,
                                                                            Y[0].p, Y[0].ld, Y[1].p, Y[1].ld, Y[2].p, Y[2].ld, Y[3].p,
                                                                            Y[3].ld, scale, R[2].p, R[2].ld, R[3].p, R[3].ld, compute()),
                                           "sparse_attention_grad_kv");
                        else
                            hnh::abi_check(hnh_sparse_attention_grad_kv_dropout_f64(
                                               hd->rowStart.data(), hd->col_idx.data(), blk.rows, blk.num_coords, (int)d, R[0].p,
                                               R[0].ld, R[1].p, R[1].ld, Y[0].p, Y[0].ld, Y[1].p, Y[1].ld, Y[2].p, Y[2].ld, Y[3].p,
                                               Y[3].ld, scale, R[2].p, R[2].ld, R[3].p, R[3].ld, dropout, seed + (uint64_t)h,
                                               atB.u0(b), atB.v0(b), compute()),
                                           "sparse_attention_grad_kv_dropout");
                    });
    }
}

// ---- link prediction -----------------------------------------------------------------------------------------
void Distributed_Sparse::linkLoss(DenseMatrix &H_A, DenseMatrix &H_B, double inv_count, DenseMatrix *dH_A, DenseMatrix *dH_B,
                                  VectorXd *scores, double *sums) {
    const string who = "linkLoss";
    check_full_rows(who);
    const int64_t r = H_A.cols();
    if (H_A.rows() != localArows || H_B.rows() != localBrows || H_B.cols() != r || r < 1 || r > INT32_MAX)
        throw hnh::Error(HNH_E_INVALID, who + ": H_A is " + to_string(H_A.rows()) + " x " + to_string(r) + " and H_B " +
                                            to_string(H_B.rows()) + " x " + to_string(H_B.cols()) + "; like_A_matrix has " +
                                            to_string(localArows) + " rows and like_B_matrix " + to_string(localBrows) +
                                            ", both of one width");
    for (auto [g, h, name] : {std::make_tuple(dH_A, &H_A, "dH_A"), std::make_tuple(dH_B, &H_B, "dH_B")}) {
        if (g && (g == &H_A || g == &H_B)) throw hnh::Error(HNH_E_INVALID, who + ": " + name + " may not be H_A or H_B");
        if (g && (g->rows() != h->rows() || g->cols() != r))
            throw hnh::Error(HNH_E_INVALID, who + ": " + name + " is " + to_string(g->rows()) + " x " + to_string(g->cols()) +
                                                ", its H " + to_string(h->rows()) + " x " + to_string(r));
    }
    if (scores && scores->size() != num_S_values())
        throw hnh::Error(HNH_E_INVALID, who + ": the scores have " + to_string(scores->size()) + " entries, the A order " +
                                            to_string(num_S_values()));
    if (!(inv_count >= 0.0) || !std::isfinite(inv_count)) throw hnh::Error(HNH_E_INVALID, who + ": inv_count must be finite and >= 0");
    if (sums == nullptr) throw hnh::Error(HNH_E_INVALID, who + ": null sums");
    // the rows' (loss sum, correct count), accumulated over the ring steps
    DenseMatrix stats(localArows, 2);
    stats.setZero();
    if (dH_A) dH_A->setZero();
    if (dH_B && dH_B != dH_A) dH_B->setZero();
    // one pass: the stored-row side is [H, its gradient (when wanted), the row statistics (A order only)]
    auto pass = [&](KernelMode order, DenseMatrix &H, DenseMatrix *dH, DenseMatrix &G, DenseMatrix *st) {
        const bool a_rows = order == k_sddmmA;
        vector<PassOperand> rows{{&H, 0, r, false}}, gathered{{&G, 0, r, false}};
        const int i_grad = dH ? (int)rows.size() : -1;
        if (dH) rows.push_back({dH, 0, r, true});
        const int i_stats = st ? (int)rows.size() : -1;
        if (st) rows.push_back({st, 0, 2, true});
        const SpmatLocal &m = *values_matrix(*this, order);
        gather_pass(order, a_rows ? rows : gathered, a_rows ? gathered : rows,
                    [&](int b, CSRLocal &blk, bool rows_are_A, const PassView *R, const PassView *Y) {
                        if (rows_are_A != a_rows)
                            throw hnh::Error(HNH_E_INVALID, who + ": a block of this order does not hold the expected side as its rows");
                        CSRHandle *h = blk.getActive();
                        double *sc = scores && a_rows ? scores->data() + (int64_t)m.blockStarts[(size_t)b] : nullptr;
                        hnh::abi_check(hnh_link_bce_f64(h->rowStart.data(), h->col_idx.data(), h->values.data(), blk.rows,
                                                        blk.num_coords, R[0].p, R[0].ld, Y[0].p, Y[0].ld, (int)r, inv_count,
                                                        i_grad >= 0 ? R[i_grad].p : nullptr, i_grad >= 0 ? R[i_grad].ld : r,
                                                        i_stats >= 0 ? R[i_stats].p : nullptr, i_stats >= 0 ? R[i_stats].ld : 2,
                                                        sc, compute()),
                                       "link_bce");
                    });
    };
    pass(k_sddmmA, H_A, dH_A, H_B, &stats);
    if (dH_B) pass(k_sddmmB, H_B, dH_B, H_A, nullptr);
    const int64_t ws_bytes = hnh_pair_sums_workspace_bytes(localArows);
    if (ws_bytes < 0) hnh::abi_check((int)ws_bytes, "pair_sums_workspace_bytes");
    VectorXd ws(std::max<int64_t>(ws_bytes / 8, 1));
    hnh::abi_check(hnh_pair_sums_f64(sums, stats.data(), localArows, ws.data(), (size_t)ws_bytes, compute()), "pair_sums");
    allreduce_rows(sums, 2, false);
}

int64_t Distributed_Sparse::linkTargetCount() {
    check_full_rows("linkTargetCount");
    const int64_t n = num_S_values();
    SpmatLocal &m = *values_matrix(*this, k_sddmmA);
    VectorXd bad(1);
    bad.setZero();
    for (size_t b = 0; b + 1 < m.blockStarts.size(); b++) {
        const int64_t nb = (int64_t)m.blockStarts[b + 1] - (int64_t)m.blockStarts[b];
        if (nb == 0) continue;
        CSRLocal *blk = m.csr_blocks[b];
        if (blk == nullptr || blk->num_coords != nb)
            throw hnh::Error(HNH_E_INVALID, "linkTargetCount: block " + to_string(b) + " does not match its value range");
        hnh::abi_check(hnh_link_target_check_f64(bad.data(), blk->getActive()->values.data(), nb, compute()), "link_target_check");
    }
    double mine = 0.0;
    hnh::cuda_check(cudaMemcpyAsync(&mine, bad.data(), sizeof mine, cudaMemcpyDeviceToHost, compute()), "target check");
    hnh::cuda_check(cudaStreamSynchronize(compute()), "target check");
    double x[2] = {mine > 0.0 ? 1.0 : 0.0, (double)n};
    hnh::Comm::world()->host_allreduce_sum_f64(x, 2);
    if (mine > 0.0)
        throw hnh::Error(HNH_E_INVALID, "link targets: " + to_string((int64_t)mine) + " stored values of this rank are not in [0, 1]");
    if (x[0] != 0.0) throw hnh::Error(HNH_E_INVALID, "link targets: another rank's stored values are not all in [0, 1]");
    return (int64_t)x[1];
}

// ---- relation-aware link prediction ------------------------------------------------------------------------------
std::unique_ptr<RelationPlan> Distributed_Sparse::relationPlan(int num_relations) {
    const string who = "relationPlan";
    check_full_rows(who);
    if (num_relations < 1) throw hnh::Error(HNH_E_INVALID, who + ": the relation count must be positive, got " + to_string(num_relations));
    std::unique_ptr<RelationPlan> plan(new RelationPlan);
    plan->owner = this;
    plan->num_relations = num_relations;
    SpmatLocal &m = *values_matrix(*this, k_sddmmA);
    const int64_t keys_n = (int64_t)num_relations + 1;
    for (size_t b = 0; b + 1 < m.blockStarts.size(); b++) {
        const int64_t nb = (int64_t)m.blockStarts[b + 1] - (int64_t)m.blockStarts[b];
        plan->blocks.emplace_back();
        if (nb == 0) continue;
        CSRLocal *blk = m.csr_blocks[b];
        if (blk == nullptr || blk->num_coords != nb)
            throw hnh::Error(HNH_E_INVALID, who + ": block " + to_string(b) + " does not match its value range");
        if (nb >= INT32_MAX) throw hnh::Error(HNH_E_INVALID, who + ": " + to_string(nb) + " entries in one block; at most 2^31 - 2");
        std::unique_ptr<RelationPlan::Block> p(new RelationPlan::Block);
        hnh::DeviceBuffer<int32_t> keys((size_t)nb);
        hnh::abi_check(hnh_relation_keys(keys.data(), blk->getActive()->values.data(), nb, num_relations, compute()), "relation_keys");
        p->perm.resize((size_t)nb);
        p->key_start.resize((size_t)keys_n + 1);
        p->piece_first.resize((size_t)keys_n + 1);
        const int64_t bound = hnh_edge_softmax_piece_bound(nb, keys_n);
        if (bound < 0) hnh::abi_check((int)bound, "edge_softmax_piece_bound");
        p->piece_key.resize((size_t)std::max<int64_t>(bound, 1));
        hnh::abi_check(hnh_edge_softmax_plan(keys.data(), nb, keys_n, p->perm.data(), p->key_start.data(), p->piece_first.data(),
                                             p->piece_key.data(), (int64_t)p->piece_key.size(), &p->pieces, compute()),
                       "edge_softmax_plan");
        blk->row_idx_device();  // the dD pass reads every entry's stored row
        plan->blocks.back() = std::move(p);
    }
    return plan;
}

void Distributed_Sparse::distmultLoss(DenseMatrix &H_A, DenseMatrix &H_B, const DenseMatrix &D, int num_relations, double target,
                                      double inv_count, DenseMatrix *dH_A, DenseMatrix *dH_B, DenseMatrix *dD, VectorXd *scores,
                                      double *sums, bool accumulate, const RelationPlan *plan) {
    const string who = "distmultLoss";
    check_full_rows(who);
    const int64_t r = H_A.cols();
    if (H_A.rows() != localArows || H_B.rows() != localBrows || H_B.cols() != r || r < 1 || r > INT32_MAX)
        throw hnh::Error(HNH_E_INVALID, who + ": H_A is " + to_string(H_A.rows()) + " x " + to_string(r) + " and H_B " +
                                            to_string(H_B.rows()) + " x " + to_string(H_B.cols()) + "; like_A_matrix has " +
                                            to_string(localArows) + " rows and like_B_matrix " + to_string(localBrows) +
                                            ", both of one width");
    if (num_relations < 1) throw hnh::Error(HNH_E_INVALID, who + ": the relation count must be positive, got " + to_string(num_relations));
    for (auto [m, name] : {std::make_pair(&D, "D"), std::make_pair((const DenseMatrix *)dD, "dD")})
        if (m && (m->rows() != num_relations || m->cols() != r))
            throw hnh::Error(HNH_E_INVALID, who + ": " + name + " is " + to_string(m->rows()) + " x " + to_string(m->cols()) +
                                                ", not num_relations x r = " + to_string(num_relations) + " x " + to_string(r));
    using Grad = std::tuple<const DenseMatrix *, const DenseMatrix *, const char *>;
    for (auto [g, h, name] : {Grad(dH_A, &H_A, "dH_A"), Grad(dH_B, &H_B, "dH_B"), Grad(dD, &D, "dD")}) {
        if (g && (g == &H_A || g == &H_B || g == &D)) throw hnh::Error(HNH_E_INVALID, who + ": " + name + " may not be H_A, H_B or D");
        if (g && (g->rows() != h->rows() || g->cols() != r))
            throw hnh::Error(HNH_E_INVALID, who + ": " + name + " is " + to_string(g->rows()) + " x " + to_string(g->cols()) +
                                                ", its input " + to_string(h->rows()) + " x " + to_string(r));
    }
    if (dD && (dD == dH_A || dD == dH_B)) throw hnh::Error(HNH_E_INVALID, who + ": dD may not be dH_A or dH_B");
    if (scores && scores->size() != num_S_values())
        throw hnh::Error(HNH_E_INVALID, who + ": the scores have " + to_string(scores->size()) + " entries, the A order " +
                                            to_string(num_S_values()));
    if (!(target >= 0.0 && target <= 1.0)) throw hnh::Error(HNH_E_INVALID, who + ": the target must lie in [0, 1]");
    if (!(inv_count >= 0.0) || !std::isfinite(inv_count)) throw hnh::Error(HNH_E_INVALID, who + ": inv_count must be finite and >= 0");
    if (sums == nullptr) throw hnh::Error(HNH_E_INVALID, who + ": null sums");
    if (plan && (plan->owner != this || plan->num_relations != num_relations))
        throw hnh::Error(HNH_E_INVALID, who + ": the relation plan was made for another object or relation count");
    std::unique_ptr<RelationPlan> own;
    if (dD && !plan) {
        own = relationPlan(num_relations);
        plan = own.get();
    }
    DenseMatrix stats(localArows, 2);
    stats.setZero();
    if (!accumulate) {
        if (dH_A) dH_A->setZero();
        if (dH_B && dH_B != dH_A) dH_B->setZero();
    }
    SpmatLocal &mA = *values_matrix(*this, k_sddmmA);
    VectorXd g(dD ? std::max<int64_t>(num_S_values(), 1) : 0);
    // one pass: the stored-row side is [H, its gradient (when wanted), the row statistics (A order only)]
    auto pass = [&](KernelMode order, DenseMatrix &H, DenseMatrix *dH, DenseMatrix &G, DenseMatrix *st) {
        const bool a_rows = order == k_sddmmA;
        vector<PassOperand> rows{{&H, 0, r, false}}, gathered{{&G, 0, r, false}};
        const int i_grad = dH ? (int)rows.size() : -1;
        if (dH) rows.push_back({dH, 0, r, true});
        const int i_stats = st ? (int)rows.size() : -1;
        if (st) rows.push_back({st, 0, 2, true});
        gather_pass(order, a_rows ? rows : gathered, a_rows ? gathered : rows,
                    [&](int b, CSRLocal &blk, bool rows_are_A, const PassView *R, const PassView *Y) {
                        if (rows_are_A != a_rows)
                            throw hnh::Error(HNH_E_INVALID, who + ": a block of this order does not hold the expected side as its rows");
                        CSRHandle *h = blk.getActive();
                        double *dR = i_grad >= 0 ? R[i_grad].p : nullptr;
                        const int64_t lddr = i_grad >= 0 ? R[i_grad].ld : r;
                        if (!a_rows) {
                            hnh::abi_check(hnh_distmult_bce_grad_f64(h->rowStart.data(), h->col_idx.data(), h->values.data(), blk.rows,
                                                                     blk.num_coords, num_relations, R[0].p, R[0].ld, Y[0].p, Y[0].ld,
                                                                     D.data(), r, (int)r, target, inv_count, dR, lddr, compute()),
                                           "distmult_bce_grad");
                            return;
                        }
                        const int64_t off = (int64_t)mA.blockStarts[(size_t)b];
                        hnh::abi_check(hnh_distmult_bce_f64(h->rowStart.data(), h->col_idx.data(), h->values.data(), blk.rows,
                                                            blk.num_coords, num_relations, R[0].p, R[0].ld, Y[0].p, Y[0].ld, D.data(), r,
                                                            (int)r, target, inv_count, dR, lddr, i_stats >= 0 ? R[i_stats].p : nullptr,
                                                            i_stats >= 0 ? R[i_stats].ld : 2, scores ? scores->data() + off : nullptr,
                                                            dD ? g.data() + off : nullptr, compute()),
                                       "distmult_bce");
                    });
    };
    pass(k_sddmmA, H_A, dH_A, H_B, &stats);
    if (dH_B) pass(k_sddmmB, H_B, dH_B, H_A, nullptr);
    if (dD) {
        // the relation-table gradient of this rank's entries, block by block in a fixed order, then over the world
        DenseMatrix local(num_relations, r);
        local.setZero();
        VectorXd partial;
        gather_pass(k_sddmmA, {{&H_A, 0, r, false}}, {{&H_B, 0, r, false}},
                    [&](int b, CSRLocal &blk, bool rows_are_A, const PassView *R, const PassView *Y) {
                        if (!rows_are_A) throw hnh::Error(HNH_E_INVALID, who + ": an A-order block does not hold H_A's rows");
                        const RelationPlan::Block *p = (size_t)b < plan->blocks.size() ? plan->blocks[(size_t)b].get() : nullptr;
                        if (p == nullptr) throw hnh::Error(HNH_E_INVALID, who + ": the relation plan has no block " + to_string(b));
                        if (partial.size() < p->pieces * r) partial.resize(p->pieces * r);
                        hnh::abi_check(hnh_distmult_relation_grad_f64(p->perm.data(), p->key_start.data(), p->piece_first.data(),
                                                                      p->piece_key.data(), p->pieces, num_relations, blk.row_idx_device(),
                                                                      blk.getActive()->col_idx.data(),
                                                                      g.data() + (int64_t)mA.blockStarts[(size_t)b], R[0].p, R[0].ld,
                                                                      Y[0].p, Y[0].ld, (int)r, partial.data(), local.data(), r,
                                                                      compute()),
                                       "distmult_relation_grad");
                    });
        allreduce_rows(local.data(), local.size(), false);
        hnh::abi_check(hnh_row_axpy_f64(dD->data(), accumulate ? dD->data() : nullptr, 1.0, nullptr, local.data(), num_relations, (int)r,
                                        compute()),
                       "row_axpy");
    }
    const int64_t ws_bytes = hnh_pair_sums_workspace_bytes(localArows);
    if (ws_bytes < 0) hnh::abi_check((int)ws_bytes, "pair_sums_workspace_bytes");
    VectorXd ws(std::max<int64_t>(ws_bytes / 8, 1)), call(2);
    hnh::abi_check(hnh_pair_sums_f64(call.data(), stats.data(), localArows, ws.data(), (size_t)ws_bytes, compute()), "pair_sums");
    allreduce_rows(call.data(), 2, false);
    hnh::abi_check(hnh_row_axpy_f64(sums, sums, 1.0, nullptr, call.data(), 1, 2, compute()), "row_axpy");
}

// ---- max aggregation -------------------------------------------------------------------------------------------------
namespace {
// the shape and aliasing checks of maxAggregate / maxAggregateBackward (every rank decides alike: shapes are local, but
// a layout gives every rank the same widths and the caller passes the same matrices); returns f
int64_t check_max_aggregate(const Distributed_Sparse &d, const string &who, const DenseMatrix &X,
                            std::initializer_list<const DenseMatrix *> A_like, std::initializer_list<const DenseMatrix *> outs,
                            const DenseMatrix *dX) {
    const int64_t f = X.cols();
    if (X.rows() != d.localBrows || f < 1 || f > INT32_MAX)
        throw hnh::Error(HNH_E_INVALID, who + ": X is " + to_string(X.rows()) + " x " + to_string(f) + "; like_B_matrix has " +
                                            to_string(d.localBrows) + " rows and the width must be positive");
    for (const DenseMatrix *m : A_like)
        if (m->rows() != d.localArows || m->cols() != f)
            throw hnh::Error(HNH_E_INVALID, who + ": an A-shaped operand is " + to_string(m->rows()) + " x " + to_string(m->cols()) +
                                                ", not localArows x f = " + to_string(d.localArows) + " x " + to_string(f));
    if (dX && (dX->rows() != X.rows() || dX->cols() != f))
        throw hnh::Error(HNH_E_INVALID, who + ": dX is " + to_string(dX->rows()) + " x " + to_string(dX->cols()) + ", X " +
                                            to_string(X.rows()) + " x " + to_string(f));
    vector<const DenseMatrix *> all{&X};
    all.insert(all.end(), A_like.begin(), A_like.end());
    if (dX) all.push_back(dX);
    for (const DenseMatrix *o : outs) {
        int same = 0;
        for (const DenseMatrix *m : all) same += m == o || (o->size() > 0 && m->data() == o->data());
        if (same != 1) throw hnh::Error(HNH_E_INVALID, who + ": an output may not be another operand of the call");
    }
    return f;
}
}  // namespace

void Distributed_Sparse::maxAggregate(DenseMatrix &X, DenseMatrix &Z, DenseMatrix &C) {
    const string who = "maxAggregate";
    check_full_rows(who);
    const int64_t f = check_max_aggregate(*this, who, X, {&Z, &C}, {&Z, &C}, nullptr);
    Z.setConstant(-INFINITY);
    C.setZero();
    gather_pass(k_sddmmA, {{&Z, 0, f, true}, {&C, 0, f, true}}, {{&X, 0, f, false}},
                [&](int, CSRLocal &blk, bool rows_are_A, const PassView *R, const PassView *Y) {
                    need_rows(rows_are_A, true, "maxAggregate");
                    CSRHandle *h = blk.getActive();
                    hnh::abi_check(hnh_max_aggregate_step_f64(h->rowStart.data(), h->col_idx.data(), blk.rows, blk.num_coords, Y[0].p,
                                                              Y[0].ld, (int)f, R[0].p, R[0].ld, R[1].p, R[1].ld, compute()),
                                   "max_aggregate_step");
                });
    hnh::abi_check(hnh_max_aggregate_finish_f64(Z.data(), C.data(), Z.size(), compute()), "max_aggregate_finish");
}

void Distributed_Sparse::maxAggregateBackward(DenseMatrix &X, DenseMatrix &Z, DenseMatrix &C, DenseMatrix &dZ, DenseMatrix &dX,
                                              bool accumulate) {
    const string who = "maxAggregateBackward";
    check_full_rows(who);
    const int64_t f = check_max_aggregate(*this, who, X, {&Z, &C, &dZ}, {&dX}, &dX);
    // G = dZ / C, 0 where C = 0: the share of dZ_u,k each tied entry gets
    DenseMatrix G(localArows, f);
    hnh::abi_check(hnh_max_aggregate_grad_scale_f64(G.data(), dZ.data(), C.data(), G.size(), compute()), "max_aggregate_grad_scale");
    if (!accumulate) dX.setZero();
    gather_pass(k_sddmmB, {{&Z, 0, f, false}, {&G, 0, f, false}}, {{&X, 0, f, false}, {&dX, 0, f, true}},
                [&](int, CSRLocal &blk, bool rows_are_A, const PassView *R, const PassView *Y) {
                    need_rows(rows_are_A, false, "maxAggregateBackward");
                    CSRHandle *h = blk.getActive();
                    hnh::abi_check(hnh_max_aggregate_grad_f64(h->rowStart.data(), h->col_idx.data(), blk.rows, blk.num_coords, R[0].p,
                                                              R[0].ld, Y[0].p, Y[0].ld, Y[1].p, Y[1].ld, (int)f, R[1].p, R[1].ld,
                                                              compute()),
                                   "max_aggregate_grad");
                });
}

// ---- multi-statistic aggregation -------------------------------------------------------------------------------------
namespace {
// the checks of multiAggregate / multiAggregateBackward (every rank decides alike: a layout gives every rank the same
// widths and the caller passes the same matrices); returns f
int64_t check_multi_aggregate(const Distributed_Sparse &d, const string &who, const DenseMatrix &X, int which,
                              std::initializer_list<const DenseMatrix *> A_like, std::initializer_list<const DenseMatrix *> outs,
                              const DenseMatrix *dX) {
    if (which < 1 || which > HNH_MULTI_ALL)
        throw hnh::Error(HNH_E_INVALID, who + ": which = " + to_string(which) + " selects no statistic or an unknown one");
    const int64_t f = X.cols();
    const int64_t W = 2 * (((which & HNH_MULTI_MOMENTS) != 0) + ((which & HNH_MULTI_MAX) != 0) + ((which & HNH_MULTI_MIN) != 0));
    if (X.rows() != d.localBrows || f < 1 || f > INT32_MAX / W)
        throw hnh::Error(HNH_E_INVALID, who + ": X is " + to_string(X.rows()) + " x " + to_string(f) + "; like_B_matrix has " +
                                            to_string(d.localBrows) + " rows and the width f must be positive with " + to_string(W) +
                                            " f below 2^31");
    for (const DenseMatrix *m : A_like)
        if (m->rows() != d.localArows || m->cols() != W * f)
            throw hnh::Error(HNH_E_INVALID, who + ": an A-shaped operand is " + to_string(m->rows()) + " x " + to_string(m->cols()) +
                                                ", not localArows x " + to_string(W) + " f = " + to_string(d.localArows) + " x " +
                                                to_string(W * f));
    if (dX && (dX->rows() != X.rows() || dX->cols() != f))
        throw hnh::Error(HNH_E_INVALID, who + ": dX is " + to_string(dX->rows()) + " x " + to_string(dX->cols()) + ", X " +
                                            to_string(X.rows()) + " x " + to_string(f));
    vector<const DenseMatrix *> all{&X};
    all.insert(all.end(), A_like.begin(), A_like.end());
    if (dX) all.push_back(dX);
    for (const DenseMatrix *o : outs) {
        int same = 0;
        for (const DenseMatrix *m : all) same += m == o || (o->size() > 0 && m->data() == o->data());
        if (same != 1) throw hnh::Error(HNH_E_INVALID, who + ": an output may not be another operand of the call");
    }
    return f;
}
}  // namespace

void Distributed_Sparse::multiAggregate(DenseMatrix &X, DenseMatrix &A, int which) {
    const string who = "multiAggregate";
    check_full_rows(who);
    const int64_t f = check_multi_aggregate(*this, who, X, which, {&A}, {&A}, nullptr);
    const int64_t w = A.cols();
    // the initial state: sums 0, maxima -inf, minima +inf, counts 0
    A.setZero();
    int64_t col = (which & HNH_MULTI_MOMENTS) ? 2 * f : 0;
    for (int flag : {HNH_MULTI_MAX, HNH_MULTI_MIN})
        if (which & flag) {
            DenseMatrix init = DenseMatrix::Constant(A.rows(), f, flag == HNH_MULTI_MAX ? -INFINITY : INFINITY);
            copy_cols(A, col, init, 0, f);
            col += 2 * f;
        }
    gather_pass(k_sddmmA, {{&A, 0, w, true}}, {{&X, 0, f, false}},
                [&](int, CSRLocal &blk, bool rows_are_A, const PassView *R, const PassView *Y) {
                    need_rows(rows_are_A, true, "multiAggregate");
                    CSRHandle *h = blk.getActive();
                    hnh::abi_check(hnh_multi_aggregate_step_f64(h->rowStart.data(), h->col_idx.data(), blk.rows, blk.num_coords,
                                                                Y[0].p, Y[0].ld, (int)f, which, R[0].p, R[0].ld, compute()),
                                   "multi_aggregate_step");
                });
    hnh::abi_check(hnh_multi_aggregate_finish_f64(A.data(), w, A.rows(), (int)f, which, compute()), "multi_aggregate_finish");
}

void Distributed_Sparse::multiAggregateBackward(DenseMatrix &X, DenseMatrix &A, DenseMatrix &dA, DenseMatrix &dX, int which,
                                                bool accumulate) {
    const string who = "multiAggregateBackward";
    check_full_rows(who);
    const int64_t f = check_multi_aggregate(*this, who, X, which, {&A, &dA}, {&dX}, &dX);
    const int64_t w = A.cols();
    // D = [dS1 | dS2 | max | dA_max / C_max | min | dA_min / C_min]: what every entry of a row gathers
    DenseMatrix D(localArows, w);
    hnh::abi_check(hnh_multi_aggregate_grad_prep_f64(A.data(), w, dA.data(), w, A.rows(), (int)f, which, D.data(), w, compute()),
                   "multi_aggregate_grad_prep");
    if (!accumulate) dX.setZero();
    gather_pass(k_sddmmB, {{&D, 0, w, false}}, {{&X, 0, f, false}, {&dX, 0, f, true}},
                [&](int, CSRLocal &blk, bool rows_are_A, const PassView *R, const PassView *Y) {
                    need_rows(rows_are_A, false, "multiAggregateBackward");
                    CSRHandle *h = blk.getActive();
                    hnh::abi_check(hnh_multi_aggregate_grad_f64(h->rowStart.data(), h->col_idx.data(), blk.rows, blk.num_coords,
                                                                R[0].p, R[0].ld, Y[0].p, Y[0].ld, (int)f, which, R[1].p, R[1].ld,
                                                                compute()),
                                   "multi_aggregate_grad");
                });
}

// ---- edge-ReLU aggregation -------------------------------------------------------------------------------------------
namespace {
// the checks of edgeReluAggregate / edgeReluAggregateBackward (every rank decides alike: a layout gives every rank the
// same widths and the caller passes the same matrices); returns f
int64_t check_edge_relu(const Distributed_Sparse &d, const string &who, const DenseMatrix &X,
                        std::initializer_list<const DenseMatrix *> A_like, std::initializer_list<const DenseMatrix *> outs,
                        std::initializer_list<const DenseMatrix *> others) {
    const int64_t f = X.cols();
    if (X.rows() != d.localBrows || f < 1 || f > INT32_MAX)
        throw hnh::Error(HNH_E_INVALID, who + ": X is " + to_string(X.rows()) + " x " + to_string(f) + "; like_B_matrix has " +
                                            to_string(d.localBrows) + " rows and the width must lie in [1, 2^31)");
    for (const DenseMatrix *m : A_like)
        if (m->rows() != d.localArows || m->cols() != f)
            throw hnh::Error(HNH_E_INVALID, who + ": an A-shaped operand is " + to_string(m->rows()) + " x " + to_string(m->cols()) +
                                                ", not localArows x f = " + to_string(d.localArows) + " x " + to_string(f));
    vector<const DenseMatrix *> all{&X};
    all.insert(all.end(), A_like.begin(), A_like.end());
    all.insert(all.end(), others.begin(), others.end());
    for (const DenseMatrix *o : outs) {
        if (!o) continue;
        int same = 0;
        for (const DenseMatrix *m : all) same += m && (m == o || (o->size() > 0 && m->data() == o->data()));
        if (same != 1) throw hnh::Error(HNH_E_INVALID, who + ": an output may not be another operand of the call");
    }
    return f;
}
}  // namespace

void Distributed_Sparse::edgeReluAggregate(DenseMatrix &X, const DenseMatrix &E_A, DenseMatrix &A) {
    const string who = "edgeReluAggregate";
    check_full_rows(who);
    const int64_t f = check_edge_relu(*this, who, X, {&A}, {&A}, {&E_A});
    const EdgeView ev = edge_view(*this, who, "E_A", &E_A, nullptr, k_sddmmA, f, f);
    A.setZero();
    gather_pass(k_sddmmA, {{&A, 0, f, true}}, {{&X, 0, f, false}},
                [&](int b, CSRLocal &blk, bool rows_are_A, const PassView *R, const PassView *Y) {
                    need_rows(rows_are_A, true, "edgeReluAggregate");
                    CSRHandle *h = blk.getActive();
                    hnh::abi_check(hnh_edge_relu_aggregate_step_f64(h->rowStart.data(), h->col_idx.data(), blk.rows, blk.num_coords,
                                                                    Y[0].p, Y[0].ld, ev.at(0, b), ev.ld(), (int)f, R[0].p, R[0].ld,
                                                                    compute()),
                                   "edge_relu_aggregate_step");
                });
}

void Distributed_Sparse::edgeReluAggregateBackward(DenseMatrix &X, const DenseMatrix *E_A, const DenseMatrix *E_B, DenseMatrix &dA,
                                                   DenseMatrix &dX, DenseMatrix *dE_A, bool accumulate) {
    const string who = "edgeReluAggregateBackward";
    check_full_rows(who);
    if (E_A == nullptr || E_B == nullptr) throw hnh::Error(HNH_E_INVALID, who + ": the edge rows need both orders, E_A and E_B");
    const int64_t f = check_edge_relu(*this, who, X, {&dA}, {&dX, dE_A}, {E_A, E_B, &dX, dE_A});
    if (dX.rows() != X.rows() || dX.cols() != f)
        throw hnh::Error(HNH_E_INVALID, who + ": dX is " + to_string(dX.rows()) + " x " + to_string(dX.cols()) + ", X " +
                                            to_string(X.rows()) + " x " + to_string(f));
    const EdgeView evA = edge_view(*this, who, "E_A", E_A, dE_A, k_sddmmA, f, f),
                   evB = edge_view(*this, who, "E_B", E_B, nullptr, k_sddmmB, f, f);
    if (!accumulate) dX.setZero();
    gather_pass(k_sddmmB, {{&dA, 0, f, false}}, {{&X, 0, f, false}, {&dX, 0, f, true}},
                [&](int b, CSRLocal &blk, bool rows_are_A, const PassView *R, const PassView *Y) {
                    need_rows(rows_are_A, false, "edgeReluAggregateBackward");
                    CSRHandle *h = blk.getActive();
                    hnh::abi_check(hnh_edge_relu_aggregate_grad_f64(h->rowStart.data(), h->col_idx.data(), blk.rows, blk.num_coords,
                                                                    R[0].p, R[0].ld, evB.at(0, b), evB.ld(), Y[0].p, Y[0].ld, (int)f,
                                                                    R[1].p, R[1].ld, compute()),
                                   "edge_relu_aggregate_grad");
                });
    if (!dE_A) return;
    dE_A->resize(E_A->rows(), f);
    gather_pass(k_sddmmA, {{&dA, 0, f, false}}, {{&X, 0, f, false}},
                [&](int b, CSRLocal &blk, bool rows_are_A, const PassView *R, const PassView *Y) {
                    need_rows(rows_are_A, true, "edgeReluAggregateBackward");
                    CSRHandle *h = blk.getActive();
                    hnh::abi_check(hnh_edge_relu_aggregate_edge_grad_f64(h->rowStart.data(), h->col_idx.data(), blk.rows,
                                                                         blk.num_coords, R[0].p, R[0].ld, Y[0].p, Y[0].ld,
                                                                         evA.at(0, b), evA.ld(), (int)f, evA.grad_at(0, b), evA.ld(),
                                                                         compute()),
                                   "edge_relu_aggregate_edge_grad");
                });
}

// ---- relational aggregation --------------------------------------------------------------------------------------------
namespace {
// the shape and aliasing checks of relationalAggregate / relationalAggregateBackward: X-shaped (localBrows x f) and
// A-shaped (localArows x R f), distinct (every rank decides alike: a layout gives every rank the same widths)
void check_relational(const Distributed_Sparse &d, const string &who, const DenseMatrix &X, const DenseMatrix &A, int num_relations) {
    const int64_t f = X.cols();
    if (num_relations < 1) throw hnh::Error(HNH_E_INVALID, who + ": the relation count must be positive, got " + to_string(num_relations));
    if (X.rows() != d.localBrows || f < 1 || f * num_relations > INT32_MAX)
        throw hnh::Error(HNH_E_INVALID, who + ": the B-shaped operand is " + to_string(X.rows()) + " x " + to_string(f) +
                                            "; like_B_matrix has " + to_string(d.localBrows) +
                                            " rows and the width f must be positive with R f below 2^31");
    if (A.rows() != d.localArows || A.cols() != f * num_relations)
        throw hnh::Error(HNH_E_INVALID, who + ": the A-shaped operand is " + to_string(A.rows()) + " x " + to_string(A.cols()) +
                                            ", not localArows x R f = " + to_string(d.localArows) + " x " + to_string(f * num_relations));
    if (&A == &X || (A.size() > 0 && A.data() == X.data()))
        throw hnh::Error(HNH_E_INVALID, who + ": an output may not be another operand of the call");
}
}  // namespace

void Distributed_Sparse::relationalAggregate(DenseMatrix &X, DenseMatrix &A, int num_relations) {
    const string who = "relationalAggregate";
    check_full_rows(who);
    check_relational(*this, who, X, A, num_relations);
    const int64_t f = X.cols(), w = f * num_relations;
    A.setZero();
    gather_pass(k_sddmmA, {{&A, 0, w, true}}, {{&X, 0, f, false}},
                [&](int, CSRLocal &blk, bool rows_are_A, const PassView *R, const PassView *Y) {
                    need_rows(rows_are_A, true, "relationalAggregate");
                    CSRHandle *h = blk.getActive();
                    hnh::abi_check(hnh_relational_aggregate_f64(h->rowStart.data(), h->col_idx.data(), h->values.data(), blk.rows,
                                                                blk.num_coords, Y[0].p, Y[0].ld, (int)f, num_relations, R[0].p,
                                                                R[0].ld, compute()),
                                   "relational_aggregate");
                });
}

void Distributed_Sparse::relationalAggregateBackward(DenseMatrix &dA, DenseMatrix &dX, int num_relations, bool accumulate) {
    const string who = "relationalAggregateBackward";
    check_full_rows(who);
    check_relational(*this, who, dX, dA, num_relations);
    const int64_t f = dX.cols(), w = f * num_relations;
    if (!accumulate) dX.setZero();
    gather_pass(k_sddmmB, {{&dA, 0, w, false}}, {{&dX, 0, f, true}},
                [&](int, CSRLocal &blk, bool rows_are_A, const PassView *R, const PassView *Y) {
                    need_rows(rows_are_A, false, "relationalAggregateBackward");
                    CSRHandle *h = blk.getActive();
                    hnh::abi_check(hnh_relational_aggregate_grad_f64(h->rowStart.data(), h->col_idx.data(), h->values.data(),
                                                                     blk.rows, blk.num_coords, Y[0].p, Y[0].ld, (int)f, num_relations,
                                                                     R[0].p, R[0].ld, compute()),
                                   "relational_aggregate_grad");
                });
}

int64_t Distributed_Sparse::relationCheck(int num_relations) {
    check_full_rows("relationCheck");
    if (num_relations < 1)
        throw hnh::Error(HNH_E_INVALID, "relationCheck: the relation count must be positive, got " + to_string(num_relations));
    const int64_t n = num_S_values();
    SpmatLocal &m = *values_matrix(*this, k_sddmmA);
    VectorXd bad(1);
    bad.setZero();
    for (size_t b = 0; b + 1 < m.blockStarts.size(); b++) {
        const int64_t nb = (int64_t)m.blockStarts[b + 1] - (int64_t)m.blockStarts[b];
        if (nb == 0) continue;
        CSRLocal *blk = m.csr_blocks[b];
        if (blk == nullptr || blk->num_coords != nb)
            throw hnh::Error(HNH_E_INVALID, "relationCheck: block " + to_string(b) + " does not match its value range");
        hnh::abi_check(hnh_relation_check_f64(bad.data(), blk->getActive()->values.data(), nb, num_relations, compute()), "relation_check");
    }
    double mine = 0.0;
    hnh::cuda_check(cudaMemcpyAsync(&mine, bad.data(), sizeof mine, cudaMemcpyDeviceToHost, compute()), "relation check");
    hnh::cuda_check(cudaStreamSynchronize(compute()), "relation check");
    double x[2] = {mine > 0.0 ? 1.0 : 0.0, (double)n};
    hnh::Comm::world()->host_allreduce_sum_f64(x, 2);
    if (mine > 0.0)
        throw hnh::Error(HNH_E_INVALID, "relations: " + to_string((int64_t)mine) + " stored values of this rank are not integers in [0, " +
                                            to_string(num_relations) + ")");
    if (x[0] != 0.0)
        throw hnh::Error(HNH_E_INVALID, "relations: another rank's stored values are not all integers in [0, " + to_string(num_relations) + ")");
    return (int64_t)x[1];
}

// ---- basis aggregation -----------------------------------------------------------------------------------------------
namespace {
// the shape and aliasing checks of basisAggregate / basisAggregateBackward: X-shaped (localBrows x f), A-shaped
// (localArows x B f), comp and dcomp R x B, scale localArows x R; B = comp.cols()
void check_basis(const Distributed_Sparse &d, const string &who, const vector<const DenseMatrix *> &X_like,
                 const vector<const DenseMatrix *> &H_like, const DenseMatrix &comp, const DenseMatrix *dcomp, const DenseMatrix *scale,
                 int num_relations, const vector<const DenseMatrix *> &outs) {
    if (num_relations < 1) throw hnh::Error(HNH_E_INVALID, who + ": the relation count must be positive, got " + to_string(num_relations));
    const int64_t B = comp.cols(), f = X_like.front()->cols();
    if (B < 1) throw hnh::Error(HNH_E_INVALID, who + ": the basis count must be positive, got " + to_string(B));
    if (comp.rows() != num_relations)
        throw hnh::Error(HNH_E_INVALID, who + ": comp is " + to_string(comp.rows()) + " x " + to_string(B) + ", not R x B with R = " +
                                            to_string(num_relations));
    if (f < 1 || B * f > INT32_MAX || (int64_t)num_relations * B > INT32_MAX)
        throw hnh::Error(HNH_E_INVALID, who + ": the width f must be positive with B f and R B below 2^31 (f = " + to_string(f) +
                                            ", B = " + to_string(B) + ")");
    for (const DenseMatrix *m : X_like)
        if (m->rows() != d.localBrows || m->cols() != f)
            throw hnh::Error(HNH_E_INVALID, who + ": a B-shaped operand is " + to_string(m->rows()) + " x " + to_string(m->cols()) +
                                                ", not like_B_matrix's " + to_string(d.localBrows) + " rows of width f = " + to_string(f));
    for (const DenseMatrix *m : H_like)
        if (m->rows() != d.localArows || m->cols() != B * f)
            throw hnh::Error(HNH_E_INVALID, who + ": an A-shaped operand is " + to_string(m->rows()) + " x " + to_string(m->cols()) +
                                                ", not localArows x B f = " + to_string(d.localArows) + " x " + to_string(B * f));
    if (dcomp && (dcomp->rows() != num_relations || dcomp->cols() != B))
        throw hnh::Error(HNH_E_INVALID, who + ": dcomp is " + to_string(dcomp->rows()) + " x " + to_string(dcomp->cols()) +
                                            ", not R x B = " + to_string(num_relations) + " x " + to_string(B));
    if (scale && (scale->rows() != d.localArows || scale->cols() != num_relations))
        throw hnh::Error(HNH_E_INVALID, who + ": scale is " + to_string(scale->rows()) + " x " + to_string(scale->cols()) +
                                            ", not localArows x R = " + to_string(d.localArows) + " x " + to_string(num_relations));
    vector<const DenseMatrix *> all(X_like);
    all.insert(all.end(), H_like.begin(), H_like.end());
    all.push_back(&comp);
    if (dcomp) all.push_back(dcomp);
    if (scale) all.push_back(scale);
    for (const DenseMatrix *o : outs) {
        int same = 0;
        for (const DenseMatrix *m : all) same += m == o || (o->size() > 0 && m->data() == o->data());
        if (same != 1) throw hnh::Error(HNH_E_INVALID, who + ": an output may not be another operand of the call");
    }
}
}  // namespace

void Distributed_Sparse::basisAggregate(DenseMatrix &X, DenseMatrix &H, const DenseMatrix &comp, int num_relations,
                                        const DenseMatrix *scale) {
    const string who = "basisAggregate";
    check_full_rows(who);
    check_basis(*this, who, {&X}, {&H}, comp, nullptr, scale, num_relations, {&H});
    const int64_t f = X.cols(), B = comp.cols();
    H.setZero();
    vector<PassOperand> A_side{{&H, 0, B * f, true}};
    if (scale) A_side.push_back({const_cast<DenseMatrix *>(scale), 0, num_relations, false});
    gather_pass(k_sddmmA, A_side, {{&X, 0, f, false}}, [&](int, CSRLocal &blk, bool rows_are_A, const PassView *R, const PassView *Y) {
        need_rows(rows_are_A, true, "basisAggregate");
        CSRHandle *h = blk.getActive();
        hnh::abi_check(hnh_basis_aggregate_f64(h->rowStart.data(), h->col_idx.data(), h->values.data(), blk.rows, blk.num_coords,
                                               Y[0].p, Y[0].ld, (int)f, scale ? R[1].p : nullptr, scale ? R[1].ld : 0, comp.data(),
                                               num_relations, (int)B, R[0].p, R[0].ld, compute()),
                       "basis_aggregate");
    });
}

void Distributed_Sparse::basisAggregateBackward(DenseMatrix &dH, DenseMatrix &X, DenseMatrix &dX, const DenseMatrix &comp,
                                                DenseMatrix &dcomp, int num_relations, const DenseMatrix *scale, bool accumulate) {
    const string who = "basisAggregateBackward";
    check_full_rows(who);
    check_basis(*this, who, {&X, &dX}, {&dH}, comp, &dcomp, scale, num_relations, {&dX, &dcomp});
    const int64_t f = X.cols(), B = comp.cols(), n = num_ST_values();
    if (n >= INT32_MAX) throw hnh::Error(HNH_E_INVALID, who + ": " + to_string(n) + " local entries; at most 2^31 - 2");
    if (!accumulate) dX.setZero();
    // P[b n + j]: entry j's product for basis b, written block by block at the block's offset in the B-order values
    SpmatLocal &m = *values_matrix(*this, k_sddmmB);
    VectorXd P(std::max<int64_t>(n * B, 1));
    vector<PassOperand> A_side{{&dH, 0, B * f, false}};
    if (scale) A_side.push_back({const_cast<DenseMatrix *>(scale), 0, num_relations, false});
    gather_pass(k_sddmmB, A_side, {{&X, 0, f, false}, {&dX, 0, f, true}},
                [&](int b, CSRLocal &blk, bool rows_are_A, const PassView *R, const PassView *Y) {
                    need_rows(rows_are_A, false, "basisAggregateBackward");
                    CSRHandle *h = blk.getActive();
                    hnh::abi_check(hnh_basis_aggregate_grad_f64(h->rowStart.data(), h->col_idx.data(), h->values.data(), blk.rows,
                                                                blk.num_coords, Y[0].p, Y[0].ld, scale ? Y[1].p : nullptr,
                                                                scale ? Y[1].ld : 0, comp.data(), num_relations, (int)B, R[0].p,
                                                                R[0].ld, (int)f, R[1].p, R[1].ld,
                                                                P.data() + (int64_t)m.blockStarts[(size_t)b], n, compute()),
                                   "basis_aggregate_grad");
                });
    // dcomp: P summed by relation in the fixed order of an edge-softmax plan over R + 1 keys (key R: no relation)
    const int64_t keys_n = (int64_t)num_relations + 1;
    hnh::DeviceBuffer<int32_t> keys((size_t)std::max<int64_t>(n, 1)), perm((size_t)std::max<int64_t>(n, 1)),
        row_start((size_t)keys_n + 1), piece_first((size_t)keys_n + 1);
    for (size_t b = 0; b + 1 < m.blockStarts.size(); b++) {
        const int64_t off = (int64_t)m.blockStarts[b], nb = (int64_t)m.blockStarts[b + 1] - off;
        if (nb == 0) continue;
        CSRLocal *blk = m.csr_blocks[b];
        if (blk == nullptr || blk->num_coords != nb)
            throw hnh::Error(HNH_E_INVALID, who + ": block " + to_string(b) + " does not match its value range");
        hnh::abi_check(hnh_relation_keys(keys.data() + off, blk->getActive()->values.data(), nb, num_relations, compute()), "relation_keys");
    }
    const int64_t bound = hnh_edge_softmax_piece_bound(n, keys_n);
    if (bound < 0) hnh::abi_check((int)bound, "edge_softmax_piece_bound");
    hnh::DeviceBuffer<int32_t> piece_row((size_t)std::max<int64_t>(bound, 1));
    int64_t pieces = 0;
    hnh::abi_check(hnh_edge_softmax_plan(keys.data(), n, keys_n, perm.data(), row_start.data(), piece_first.data(), piece_row.data(),
                                         (int64_t)piece_row.size(), &pieces, compute()),
                   "edge_softmax_plan");
    // sums[b (R + 1) + rho], then dcomp[rho, b] = sums[b (R + 1) + rho] for rho < R
    VectorXd piece(std::max<int64_t>(pieces, 1)), sums(keys_n * B);
    for (int64_t b = 0; b < B; b++)
        hnh::abi_check(hnh_edge_sum_f64(P.data() + b * n, perm.data(), row_start.data(), piece_first.data(), piece_row.data(), keys_n,
                                        pieces, piece.data(), sums.data() + b * keys_n, compute()),
                       "edge_sum");
    const size_t d = sizeof(double);
    for (int64_t b = 0; b < B; b++)
        hnh::cuda_check(cudaMemcpy2DAsync(dcomp.data() + b, d * (size_t)B, sums.data() + b * keys_n, d, d, (size_t)num_relations,
                                          cudaMemcpyDeviceToDevice, compute()),
                        "dcomp copy");
    allreduce_rows(dcomp.data(), dcomp.size(), false);
}

hnh::PeerRing *Distributed_Sparse::peer_ring(std::shared_ptr<hnh::Comm> world, size_t bytes) {
    if (peer_ring_broken_ || !hnh::PeerRing::enabled() || world->size() < 2) return nullptr;
    auto key = std::make_pair(world.get(), bytes);
    auto it = peer_rings_.find(key);
    if (it != peer_rings_.end()) return it->second.get();
    try {
        peer_rings_[key].reset(new hnh::PeerRing(world, bytes));
    } catch (const hnh::Error &e) {
        // peer mapping unavailable (e.g. no NVLink/IPC): the NCCL ring below does the same job
        if (verbose) cout << "PeerRing unavailable, using NCCL send/recv: " << e.what() << endl;
        peer_rings_.erase(key);
        peer_ring_broken_ = true;
        return nullptr;
    }
    return peer_rings_[key].get();
}

hnh::PeerRing *Distributed_Sparse::sparse_ring(std::shared_ptr<hnh::Comm> world, CSRLocal *blk) {
    if (peer_ring_broken_ || !hnh::PeerRing::all_shifts() || world->size() < 2 || blk == nullptr) return nullptr;
    auto key = std::make_pair(world.get(), blk);
    auto it = sparse_rings_.find(key);
    if (it != sparse_rings_.end()) return it->second.get();
    try {
        sparse_rings_[key].reset(new hnh::PeerRing(world, blk->ring_buffers(), blk->active));
    } catch (const hnh::Error &e) {
        if (verbose) cout << "sparse PeerRing unavailable, using NCCL send/recv: " << e.what() << endl;
        sparse_rings_.erase(key);
        peer_ring_broken_ = true;
        return nullptr;
    }
    return sparse_rings_[key].get();
}

// logical buffers of CSRLocal::ring_buffers(): 0 = values, 1 = col_idx, 2 = rowStart
void Distributed_Sparse::sparse_push_early(hnh::PeerRing &pr, CSRLocal &blk, bool values_written) {
    const int k = 1 - blk.active;  // the downstream rank's passive handle (all ranks flip together)
    CSRHandle *h = blk.getActive();
    pr.begin_push(k, comm());
    const size_t nz = (size_t)blk.num_coords;
    if (nz) hnh::cuda_check(cudaMemcpyAsync(pr.dst_ptr(1, k), h->col_idx.data(), sizeof(int64_t) * nz, cudaMemcpyDeviceToDevice, comm()), "push col_idx");
    hnh::cuda_check(cudaMemcpyAsync(pr.dst_ptr(2, k), h->rowStart.data(), sizeof(int64_t) * (size_t)(blk.rows + 1), cudaMemcpyDeviceToDevice, comm()), "push rowStart");
    if (!values_written && nz)
        hnh::cuda_check(cudaMemcpyAsync(pr.dst_ptr(0, k), h->values.data(), sizeof(double) * nz, cudaMemcpyDeviceToDevice, comm()), "push values");
}

void Distributed_Sparse::sparse_push_late(hnh::PeerRing &pr, CSRLocal &blk, bool values_written, bool early_done, int64_t incoming) {
    const int a = blk.active, k = 1 - a;
    if (!early_done) sparse_push_early(pr, blk, false);  // everything in one go, after the kernel
    else if (values_written && blk.num_coords)
        hnh::cuda_check(cudaMemcpyAsync(pr.dst_ptr(0, k), blk.getActive()->values.data(), sizeof(double) * (size_t)blk.num_coords,
                                        cudaMemcpyDeviceToDevice, comm()), "push values");
    pr.end_push(k, comm());
    pr.release(a, comm());  // my handle `a` has been read by the kernel and by the push: upstream may refill it
    blk.shift_commit(incoming);
    pr.expect_arrival(k);
    pr.wait_arrival(k, comm());
}
