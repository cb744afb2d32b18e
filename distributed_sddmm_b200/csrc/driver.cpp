// driver.cpp -- extern "C" driver ABI (include/hnh_b200_driver.h) over the C++ host classes.
#include "hnh_b200_driver.h"

#include <cmath>
#include <cstring>
#include <memory>

#include "hnh/15D_dense_shift.hpp"
#include "hnh/15D_sparse_shift.hpp"
#include "hnh/25D_cannon_dense.hpp"
#include "hnh/25D_cannon_sparse.hpp"
#include "hnh/als_conjugate_gradients.h"
#include "hnh/benchmark_dist.hpp"
#include "hnh/distributed_sparse.h"
#include "hnh/gat.hpp"
#include "hnh/graph_sage.hpp"
#include "hnh/graph_transformer.hpp"
#include "hnh/rgcn.hpp"
#include "hnh/training.hpp"
#include "hnh_b200.h"
#include "launch.h"

Distributed_Sparse *hnh_make_algorithm(const string &name, SpmatLocal *spmat, int R, int c, KernelImplementation *k);

struct hnhd_spmat {
    SpmatLocal m;
};
struct hnhd_alg {
    StandardKernel kernel;
    std::unique_ptr<Distributed_Sparse> alg;
};
struct hnhd_dense {
    DenseMatrix m;
};
struct hnhd_vec {
    VectorXd v;
};
struct hnhd_model {
    std::unique_ptr<GraphModel> m;
};
struct hnhd_labels {
    std::unique_ptr<hnh::NodeLabels> l;
};
struct hnhd_adamw {
    std::unique_ptr<hnh::AdamW> o;
};
struct hnhd_link_targets {
    std::unique_ptr<hnh::LinkTargets> t;
};

namespace {

// run f, translating C++ exceptions into error codes
template <class F>
int guarded(F f) {
    try {
        f();
        return HNH_OK;
    } catch (const hnh::Error &e) {
        return hnh::set_error(e.code, "%s", e.what());
    } catch (const std::bad_alloc &) {
        return hnh::set_error(HNH_E_ALLOC, "out of host memory");
    } catch (const std::exception &e) {
        return hnh::set_error(HNH_E_INVALID, "%s", e.what());
    }
}

int copy_json(const json &j, char *out, size_t capacity) {
    const string s = j.dump();
    if (!out || capacity < s.size() + 1)
        return hnh::set_error(HNH_E_INVALID, "json buffer too small (%zu needed)", s.size() + 1);
    std::memcpy(out, s.c_str(), s.size() + 1);
    return (int)s.size();
}

cudaEvent_t g_t0 = nullptr, g_t1 = nullptr;

// ---- graph model handles: the model behind one, its buffers and its parameters by name
GraphModel &model(hnhd_model_t *m) {
    if (!m) throw hnh::Error(HNH_E_INVALID, "null model");
    return *m->m;
}
// the model behind a handle as a T (`kind` names it), refused for a model of another kind
template <class T>
T &model_as(hnhd_model_t *m, const char *kind) {
    T *t = dynamic_cast<T *>(&model(m));
    if (!t) throw hnh::Error(HNH_E_INVALID, string("this call takes a ") + kind + " model, not a " + m->m->model_name + " one");
    return *t;
}
DenseMatrix &model_buffer(hnhd_model_t *m, int buffer) {
    GraphModel &g = model(m);
    if (buffer < 0 || buffer >= (int)g.buffers.size()) throw hnh::Error(HNH_E_INVALID, g.model_name + ": no such buffer");
    return g.buffers[(size_t)buffer];
}
ParamRef model_param(hnhd_model_t *m, int layer, const char *name) {
    GraphModel &g = model(m);
    if (!name) throw hnh::Error(HNH_E_INVALID, g.model_name + ": null argument");
    return g.param(layer, name);
}
// copy n doubles between host and device on the compute stream and wait for the copy
void sync_copy(double *dst, const double *src, int64_t n, cudaMemcpyKind kind) {
    cudaStream_t s = hnh::Runtime::get().compute_stream();
    if (n > 0) hnh::cuda_check(cudaMemcpyAsync(dst, src, sizeof(double) * (size_t)n, kind, s), "model parameter copy");
    hnh::cuda_check(cudaStreamSynchronize(s), "model parameter copy");
}

}  // namespace

extern "C" {

int hnhd_init_self(void) { return guarded([] { hnh::Comm::init_self(); }); }
int hnhd_nccl_unique_id(char out[HNHD_NCCL_ID_BYTES]) { return guarded([&] { hnh::Comm::nccl_unique_id(out); }); }
int hnhd_init_nccl(int rank, int world_size, const char uid[HNHD_NCCL_ID_BYTES]) {
    return guarded([&] { hnh::Comm::init_nccl(rank, world_size, uid); });
}
int hnhd_init_external(int rank, int world_size, const hnhd_external_transport_t *cb) {
    return guarded([&] { hnh::Comm::init_external(rank, world_size, cb); });
}
int hnhd_finalize(void) {
    return guarded([] {
        if (hnh::Runtime::get().has_device()) hnh::Runtime::get().sync_all();
        hnh::Comm::finalize();
    });
}
int hnhd_world_rank(void) { return hnh::Comm::world_initialised() ? hnh::Comm::world()->rank() : -1; }
int hnhd_world_size(void) { return hnh::Comm::world_initialised() ? hnh::Comm::world()->size() : -1; }
int hnhd_barrier(void) { return guarded([] { hnh::Comm::world()->barrier(); }); }
int hnhd_device_synchronize(void) { return guarded([] { hnh::Runtime::get().sync_all(); }); }

int hnhd_setup_times_json(char *out, size_t capacity, int reset) {
    int n = 0;
    int rc = guarded([&] {
        json j = json::object();
        for (auto &kv : hnh::setup_times()) j[kv.first] = kv.second;
        n = copy_json(j, out, capacity);
        if (reset) hnh::setup_times_reset();
    });
    return rc ? rc : n;
}

// ---- SpmatLocal ---------------------------------------------------------------------------------
int hnhd_spmat_load_er(int logM, int nnz_per_row, uint64_t seed, hnhd_spmat_t **out) {
    return guarded([&] {
        if (!out) throw hnh::Error(HNH_E_INVALID, "null out");
        std::unique_ptr<hnhd_spmat> s(new hnhd_spmat);
        SpmatLocal::er_seed = seed;
        s->m.loadTuples(false, logM, nnz_per_row, "");
        *out = s.release();
    });
}
int hnhd_spmat_load_file(const char *filename, hnhd_spmat_t **out) {
    return guarded([&] {
        if (!filename || !out) throw hnh::Error(HNH_E_INVALID, "null argument");
        std::unique_ptr<hnhd_spmat> s(new hnhd_spmat);
        s->m.loadTuples(true, -1, -1, filename);
        *out = s.release();
    });
}
int hnhd_spmat_from_tuples(uint64_t M, uint64_t N, const uint64_t *rows, const uint64_t *cols, const double *vals,
                           int64_t n_local, hnhd_spmat_t **out) {
    return guarded([&] {
        if (!out || n_local < 0 || (n_local > 0 && (!rows || !cols || !vals))) throw hnh::Error(HNH_E_INVALID, "bad argument");
        std::unique_ptr<hnhd_spmat> s(new hnhd_spmat);
        s->m.setTuples(M, N, rows, cols, vals, n_local);
        *out = s.release();
    });
}
int hnhd_spmat_info(const hnhd_spmat_t *S, uint64_t *M, uint64_t *N, uint64_t *dist_nnz, int64_t *local_tuples) {
    if (!S) return hnh::set_error(HNH_E_INVALID, "null spmat");
    if (M) *M = S->m.M;
    if (N) *N = S->m.N;
    if (dist_nnz) *dist_nnz = S->m.dist_nnz;
    if (local_tuples) *local_tuples = S->m.local_tuple_count();
    return HNH_OK;
}
int hnhd_spmat_tuples(const hnhd_spmat_t *S, uint64_t *rows, uint64_t *cols, double *vals, int64_t capacity) {
    if (!S || S->m.local_tuple_count() > capacity) return hnh::set_error(HNH_E_INVALID, "bad argument / capacity");
    if (S->m.tuples_on_device()) {
        int rc = guarded([&] { const_cast<hnhd_spmat_t *>(S)->m.tuples_to_host(); });
        if (rc) return rc;
    }
    for (size_t i = 0; i < S->m.coords.size(); i++) {
        rows[i] = S->m.coords[i].r;
        cols[i] = S->m.coords[i].c;
        vals[i] = S->m.coords[i].value;
    }
    return HNH_OK;
}
void hnhd_spmat_destroy(hnhd_spmat_t *S) { delete S; }

// ---- algorithms ---------------------------------------------------------------------------------
int hnhd_alg_create(const char *name, hnhd_spmat_t *S, int R, int c, hnhd_alg_t **out) {
    return guarded([&] {
        if (!name || !S || !out) throw hnh::Error(HNH_E_INVALID, "null argument");
        std::unique_ptr<hnhd_alg> a(new hnhd_alg);
        a->alg.reset(hnh_make_algorithm(name, &S->m, R, c, &a->kernel));
        *out = a.release();
    });
}
void hnhd_alg_destroy(hnhd_alg_t *alg) { delete alg; }

int hnhd_alg_dims(hnhd_alg_t *a, hnhd_alg_dims_t *o) {
    return guarded([&] {
        if (!a || !o) throw hnh::Error(HNH_E_INVALID, "null argument");
        Distributed_Sparse &d = *a->alg;
        o->M = d.M; o->N = d.N; o->R = d.R; o->p = d.p; o->c = d.c;
        o->localArows = d.localArows; o->localAcols = d.localAcols;
        o->localBrows = d.localBrows; o->localBcols = d.localBcols;
        o->s_values = d.num_S_values();
        o->st_values = d.num_ST_values();
        o->r_split = d.r_split ? 1 : 0;
        o->grid_i = d.grid->i; o->grid_j = d.grid->j; o->grid_k = d.grid->k;
        o->n_a_submatrices = (int)d.aSubmatrices.size();
        o->n_b_submatrices = (int)d.bSubmatrices.size();
    });
}
int hnhd_alg_submatrices(hnhd_alg_t *a, int which, int *out4, int capacity) {
    if (!a || !out4) return hnh::set_error(HNH_E_INVALID, "null argument");
    const vector<DenseSubmatrix> &v = which == 0 ? a->alg->aSubmatrices : a->alg->bSubmatrices;
    if ((int)v.size() * 4 > capacity) return hnh::set_error(HNH_E_INVALID, "capacity too small");
    for (size_t i = 0; i < v.size(); i++) {
        out4[4 * i] = v[i].topRow; out4[4 * i + 1] = v[i].leftCol;
        out4[4 * i + 2] = v[i].rowCount; out4[4 * i + 3] = v[i].colCount;
    }
    return (int)v.size();
}
int hnhd_alg_info_json(hnhd_alg_t *a, char *out, size_t capacity) {
    int n = 0;
    int rc = guarded([&] { n = copy_json(a->alg->json_algorithm_info(), out, capacity); });
    return rc ? rc : n;
}
int hnhd_alg_perf_json(hnhd_alg_t *a, char *out, size_t capacity) {
    int n = 0;
    int rc = guarded([&] { n = copy_json(a->alg->json_perf_statistics(), out, capacity); });
    return rc ? rc : n;
}
int hnhd_alg_reset_timers(hnhd_alg_t *a) { return guarded([&] { a->alg->reset_performance_timers(); }); }

static SpmatLocal *pick(hnhd_alg_t *a, int which) { return which == 0 ? a->alg->S.get() : a->alg->ST.get(); }
int hnhd_alg_block_count(hnhd_alg_t *a, int which) { return a ? (int)pick(a, which)->csr_blocks.size() : -1; }
int hnhd_alg_block_meta(hnhd_alg_t *a, int which, int block, int64_t *rows, int64_t *cols, int64_t *nnz, int *transpose,
                        int *is_null) {
    if (!a) return hnh::set_error(HNH_E_INVALID, "null argument");
    SpmatLocal *m = pick(a, which);
    if (block < 0 || block >= (int)m->csr_blocks.size()) return hnh::set_error(HNH_E_INVALID, "block out of range");
    CSRLocal *b = m->csr_blocks[block];
    *is_null = b == nullptr;
    *rows = b ? b->rows : 0;
    *cols = b ? b->cols : 0;
    *nnz = b ? b->num_coords : 0;
    *transpose = b ? (int)b->transpose : 0;
    return HNH_OK;
}
int hnhd_alg_block_arrays(hnhd_alg_t *a, int which, int block, int64_t *rowStart, int64_t *col_idx, int64_t *row_idx,
                          double *values) {
    return guarded([&] {
        CSRLocal *b = pick(a, which)->csr_blocks.at((size_t)block);
        if (!b) throw hnh::Error(HNH_E_INVALID, "null block");
        CSRLocal::HostCSR h = b->to_host();
        std::memcpy(rowStart, h.rowStart.data(), sizeof(int64_t) * h.rowStart.size());
        std::memcpy(col_idx, h.col_idx.data(), sizeof(int64_t) * h.col_idx.size());
        std::memcpy(row_idx, h.row_idx.data(), sizeof(int64_t) * h.row_idx.size());
        std::memcpy(values, h.values.data(), sizeof(double) * h.values.size());
    });
}

// ---- dense / vectors ------------------------------------------------------------------------------
int hnhd_dense_create(int64_t rows, int64_t cols, double value, hnhd_dense_t **out) {
    return guarded([&] {
        std::unique_ptr<hnhd_dense> d(new hnhd_dense);
        d->m = DenseMatrix::Constant(rows, cols, value);
        *out = d.release();
    });
}
int hnhd_dense_like(hnhd_alg_t *a, int which, double value, hnhd_dense_t **out) {
    return guarded([&] {
        std::unique_ptr<hnhd_dense> d(new hnhd_dense);
        d->m = which == 0 ? a->alg->like_A_matrix(value) : a->alg->like_B_matrix(value);
        *out = d.release();
    });
}
int hnhd_dense_fill(hnhd_dense_t *m, double value) { return guarded([&] { m->m.setConstant(value); }); }
int hnhd_dense_dummy_initialize(hnhd_alg_t *a, hnhd_dense_t *m, int which) {
    return guarded([&] { a->alg->dummyInitialize(m->m, which == 0 ? Amat : Bmat); });
}
int hnhd_dense_from_host(hnhd_dense_t *m, const double *host) { return guarded([&] { m->m.copy_from_host(host); }); }
int hnhd_dense_to_host(const hnhd_dense_t *m, double *host) {
    return guarded([&] { m->m.copy_to_host(host); });
}
int hnhd_dense_shape(const hnhd_dense_t *m, int64_t *rows, int64_t *cols) {
    *rows = m->m.rows();
    *cols = m->m.cols();
    return HNH_OK;
}
void *hnhd_dense_data(hnhd_dense_t *m) { return m->m.data(); }
void hnhd_dense_destroy(hnhd_dense_t *m) { delete m; }

int hnhd_vec_create(int64_t n, double value, hnhd_vec_t **out) {
    return guarded([&] {
        std::unique_ptr<hnhd_vec> v(new hnhd_vec);
        v->v = VectorXd::Constant(n, value);
        *out = v.release();
    });
}
int hnhd_vec_like(hnhd_alg_t *a, int which, double value, hnhd_vec_t **out) {
    return guarded([&] {
        std::unique_ptr<hnhd_vec> v(new hnhd_vec);
        v->v = which == 0 ? a->alg->like_S_values(value) : a->alg->like_ST_values(value);
        *out = v.release();
    });
}
int hnhd_vec_fill(hnhd_vec_t *v, double value) { return guarded([&] { v->v.setConstant(value); }); }
int hnhd_vec_from_host(hnhd_vec_t *v, const double *host) { return guarded([&] { v->v.copy_from_host(host); }); }
int hnhd_vec_to_host(const hnhd_vec_t *v, double *host) {
    return guarded([&] {
        vector<double> h = v->v.to_host();
        std::memcpy(host, h.data(), sizeof(double) * h.size());
    });
}
int64_t hnhd_vec_size(const hnhd_vec_t *v) { return v ? v->v.size() : -1; }
void hnhd_vec_destroy(hnhd_vec_t *v) { delete v; }

// ---- operations -------------------------------------------------------------------------------------
int hnhd_alg_op(hnhd_alg_t *a, int op, hnhd_dense_t *A, hnhd_dense_t *B, hnhd_vec_t *svals, hnhd_vec_t *result, int aux) {
    return guarded([&] {
        if (!a) throw hnh::Error(HNH_E_INVALID, "null algorithm");
        Distributed_Sparse &d = *a->alg;
        auto needAB = [&] { if (!A || !B) throw hnh::Error(HNH_E_INVALID, "A and B are required"); };
        auto needS = [&] { if (!svals) throw hnh::Error(HNH_E_INVALID, "svals is required"); };
        auto needR = [&] { if (!result) throw hnh::Error(HNH_E_INVALID, "result is required"); };
        switch (op) {
            case HNHD_OP_SDDMM_A: needAB(); needS(); needR(); d.sddmmA(A->m, B->m, svals->v, result->v); break;
            case HNHD_OP_SDDMM_B: needAB(); needS(); needR(); d.sddmmB(A->m, B->m, svals->v, result->v); break;
            case HNHD_OP_SPMM_A: needAB(); needS(); d.spmmA(A->m, B->m, svals->v); break;
            case HNHD_OP_SPMM_B: needAB(); needS(); d.spmmB(A->m, B->m, svals->v); break;
            case HNHD_OP_FUSED_A: needAB(); needS(); needR(); d.fusedSpMM(A->m, B->m, svals->v, result->v, Amat); break;
            case HNHD_OP_FUSED_B: needAB(); needS(); needR(); d.fusedSpMM(A->m, B->m, svals->v, result->v, Bmat); break;
            case HNHD_OP_INITIAL_SHIFT: d.initial_shift(A ? &A->m : nullptr, B ? &B->m : nullptr, (KernelMode)aux); break;
            case HNHD_OP_DE_SHIFT: d.de_shift(A ? &A->m : nullptr, B ? &B->m : nullptr, (KernelMode)aux); break;
            default: throw hnh::Error(HNH_E_INVALID, "unknown op");
        }
    });
}

int hnhd_alg_fused_host(hnhd_alg_t *a, hnhd_dense_t *A, hnhd_dense_t *B, hnhd_vec_t *svals, hnhd_vec_t *result,
                        const double *hostA, const double *hostB, double *hostOut, int mode, int64_t chunk_rows) {
    return guarded([&] {
        if (!a || !A || !B || !svals || !result || !hostA || !hostB || !hostOut || (mode != 0 && mode != 1))
            throw hnh::Error(HNH_E_INVALID, "hnhd_alg_fused_host: bad argument");
        Distributed_Sparse &d = *a->alg;
        Sparse15D_Dense_Shift *ds = dynamic_cast<Sparse15D_Dense_Shift *>(&d);
        const int64_t keep = ds ? ds->host_pipeline_chunk_rows : 0;
        if (ds && chunk_rows != 0) ds->host_pipeline_chunk_rows = chunk_rows;
        try {
            d.fusedSpMM_host(hostA, hostB, hostOut, A->m, B->m, svals->v, result->v, mode == 0 ? Amat : Bmat);
        } catch (...) {
            if (ds) ds->host_pipeline_chunk_rows = keep;
            throw;
        }
        if (ds) ds->host_pipeline_chunk_rows = keep;
    });
}

static KernelMode value_order(int mode) {
    if (mode != 0 && mode != 1) throw hnh::Error(HNH_E_INVALID, "edge softmax: mode must be 0 (A order) or 1 (B order)");
    return mode == 0 ? k_sddmmA : k_sddmmB;
}
int hnhd_alg_edge_softmax(hnhd_alg_t *a, hnhd_vec_t *vec, int mode) {
    return guarded([&] {
        if (!a || !vec) throw hnh::Error(HNH_E_INVALID, "hnhd_alg_edge_softmax: null argument");
        a->alg->edgeSoftmax(vec->v, value_order(mode));
    });
}
int hnhd_alg_edge_softmax_backward(hnhd_alg_t *a, const hnhd_vec_t *alpha, hnhd_vec_t *grad, int mode) {
    return guarded([&] {
        if (!a || !alpha || !grad) throw hnh::Error(HNH_E_INVALID, "hnhd_alg_edge_softmax_backward: null argument");
        a->alg->edgeSoftmaxBackward(alpha->v, grad->v, value_order(mode));
    });
}

int hnhd_alg_additive_scores(hnhd_alg_t *a, const hnhd_vec_t *s, const hnhd_vec_t *t, hnhd_vec_t *out, int mode, double alpha,
                              int derivative) {
    return guarded([&] {
        if (!a || !s || !t || !out) throw hnh::Error(HNH_E_INVALID, "hnhd_alg_additive_scores: null argument");
        a->alg->additiveScores(s->v, t->v, out->v, value_order(mode), alpha, derivative != 0);
    });
}
int hnhd_alg_edge_sums(hnhd_alg_t *a, const hnhd_vec_t *values, hnhd_vec_t *row_sums, hnhd_vec_t *col_sums) {
    return guarded([&] {
        if (!a || !values || !row_sums || !col_sums) throw hnh::Error(HNH_E_INVALID, "hnhd_alg_edge_sums: null argument");
        a->alg->edgeSums(values->v, row_sums->v, col_sums->v);
    });
}

int hnhd_alg_gatv2_scores(hnhd_alg_t *a, hnhd_dense_t *A, hnhd_dense_t *B, const hnhd_vec_t *va, hnhd_vec_t *out, int mode,
                          double alpha) {
    return guarded([&] {
        if (!a || !A || !B || !va || !out) throw hnh::Error(HNH_E_INVALID, "hnhd_alg_gatv2_scores: null argument");
        a->alg->gatv2Scores(A->m, B->m, va->v, out->v, value_order(mode), alpha);
    });
}
int hnhd_alg_gatv2_backward(hnhd_alg_t *a, hnhd_dense_t *A, hnhd_dense_t *B, const hnhd_vec_t *va, const hnhd_vec_t *grad_A,
                            const hnhd_vec_t *grad_B, hnhd_dense_t *dA, hnhd_dense_t *dB, hnhd_vec_t *da, double alpha) {
    return guarded([&] {
        if (!a || !A || !B || !va || !grad_A || !grad_B || !dA || !dB || !da)
            throw hnh::Error(HNH_E_INVALID, "hnhd_alg_gatv2_backward: null argument");
        a->alg->gatv2Backward(A->m, B->m, va->v, grad_A->v, grad_B->v, dA->m, dB->m, da->v, alpha);
    });
}

int hnhd_alg_sparse_attention(hnhd_alg_t *a, hnhd_dense_t *Q, hnhd_dense_t *K, hnhd_dense_t *V, hnhd_dense_t *Z, hnhd_dense_t *L,
                              int heads, double scale) {
    return guarded([&] {
        if (!a || !Q || !K || !V || !Z || !L) throw hnh::Error(HNH_E_INVALID, "hnhd_alg_sparse_attention: null argument");
        if (!std::isfinite(scale)) throw hnh::Error(HNH_E_INVALID, "hnhd_alg_sparse_attention: the scale must be finite");
        a->alg->sparseAttention(Q->m, K->m, V->m, Z->m, L->m, heads, scale);
    });
}
int hnhd_alg_sparse_attention_backward(hnhd_alg_t *a, hnhd_dense_t *Q, hnhd_dense_t *K, hnhd_dense_t *V, hnhd_dense_t *Z,
                                       hnhd_dense_t *L, hnhd_dense_t *dZ, hnhd_dense_t *dQ, hnhd_dense_t *dK, hnhd_dense_t *dV,
                                       int heads, double scale) {
    return guarded([&] {
        if (!a || !Q || !K || !V || !Z || !L || !dZ || !dQ || !dK || !dV)
            throw hnh::Error(HNH_E_INVALID, "hnhd_alg_sparse_attention_backward: null argument");
        if (!std::isfinite(scale)) throw hnh::Error(HNH_E_INVALID, "hnhd_alg_sparse_attention_backward: the scale must be finite");
        a->alg->sparseAttentionBackward(Q->m, K->m, V->m, Z->m, L->m, dZ->m, dQ->m, dK->m, dV->m, heads, scale);
    });
}
int hnhd_alg_sparse_attention_dropout(hnhd_alg_t *a, hnhd_dense_t *Q, hnhd_dense_t *K, hnhd_dense_t *V, hnhd_dense_t *Z,
                                      hnhd_dense_t *L, int heads, double scale, double dropout, uint64_t seed) {
    return guarded([&] {
        if (!a || !Q || !K || !V || !Z || !L) throw hnh::Error(HNH_E_INVALID, "hnhd_alg_sparse_attention_dropout: null argument");
        if (!std::isfinite(scale)) throw hnh::Error(HNH_E_INVALID, "hnhd_alg_sparse_attention_dropout: the scale must be finite");
        a->alg->sparseAttention(Q->m, K->m, V->m, Z->m, L->m, heads, scale, dropout, seed);
    });
}
int hnhd_alg_sparse_attention_backward_dropout(hnhd_alg_t *a, hnhd_dense_t *Q, hnhd_dense_t *K, hnhd_dense_t *V, hnhd_dense_t *Z,
                                               hnhd_dense_t *L, hnhd_dense_t *dZ, hnhd_dense_t *dQ, hnhd_dense_t *dK,
                                               hnhd_dense_t *dV, int heads, double scale, double dropout, uint64_t seed) {
    return guarded([&] {
        if (!a || !Q || !K || !V || !Z || !L || !dZ || !dQ || !dK || !dV)
            throw hnh::Error(HNH_E_INVALID, "hnhd_alg_sparse_attention_backward_dropout: null argument");
        if (!std::isfinite(scale))
            throw hnh::Error(HNH_E_INVALID, "hnhd_alg_sparse_attention_backward_dropout: the scale must be finite");
        a->alg->sparseAttentionBackward(Q->m, K->m, V->m, Z->m, L->m, dZ->m, dQ->m, dK->m, dV->m, heads, scale, dropout, seed);
    });
}
int hnhd_alg_sparse_attention_bias(hnhd_alg_t *a, hnhd_dense_t *Q, hnhd_dense_t *K, hnhd_dense_t *V, hnhd_dense_t *Z,
                                   hnhd_dense_t *L, int heads, double scale, double dropout, uint64_t seed,
                                   const hnhd_vec_t *bias) {
    return guarded([&] {
        if (!a || !Q || !K || !V || !Z || !L) throw hnh::Error(HNH_E_INVALID, "hnhd_alg_sparse_attention_bias: null argument");
        if (!std::isfinite(scale)) throw hnh::Error(HNH_E_INVALID, "hnhd_alg_sparse_attention_bias: the scale must be finite");
        a->alg->sparseAttention(Q->m, K->m, V->m, Z->m, L->m, heads, scale, dropout, seed, bias ? &bias->v : nullptr);
    });
}
int hnhd_alg_sparse_attention_backward_bias(hnhd_alg_t *a, hnhd_dense_t *Q, hnhd_dense_t *K, hnhd_dense_t *V, hnhd_dense_t *Z,
                                            hnhd_dense_t *L, hnhd_dense_t *dZ, hnhd_dense_t *dQ, hnhd_dense_t *dK,
                                            hnhd_dense_t *dV, int heads, double scale, double dropout, uint64_t seed,
                                            const hnhd_vec_t *bias_A, const hnhd_vec_t *bias_B, hnhd_vec_t *dbias_A,
                                            hnhd_vec_t *dbias_B) {
    return guarded([&] {
        if (!a || !Q || !K || !V || !Z || !L || !dZ || !dQ || !dK || !dV)
            throw hnh::Error(HNH_E_INVALID, "hnhd_alg_sparse_attention_backward_bias: null argument");
        if (!std::isfinite(scale))
            throw hnh::Error(HNH_E_INVALID, "hnhd_alg_sparse_attention_backward_bias: the scale must be finite");
        a->alg->sparseAttentionBackward(Q->m, K->m, V->m, Z->m, L->m, dZ->m, dQ->m, dK->m, dV->m, heads, scale, dropout, seed,
                                        bias_A ? &bias_A->v : nullptr, bias_B ? &bias_B->v : nullptr,
                                        dbias_A ? &dbias_A->v : nullptr, dbias_B ? &dbias_B->v : nullptr);
    });
}
int hnhd_alg_sparse_attention_edge(hnhd_alg_t *a, hnhd_dense_t *Q, hnhd_dense_t *K, hnhd_dense_t *V, hnhd_dense_t *Z,
                                   hnhd_dense_t *L, int heads, double scale, double dropout, uint64_t seed,
                                   const hnhd_vec_t *bias, const hnhd_dense_t *edge) {
    return guarded([&] {
        if (!a || !Q || !K || !V || !Z || !L) throw hnh::Error(HNH_E_INVALID, "hnhd_alg_sparse_attention_edge: null argument");
        if (!std::isfinite(scale)) throw hnh::Error(HNH_E_INVALID, "hnhd_alg_sparse_attention_edge: the scale must be finite");
        a->alg->sparseAttention(Q->m, K->m, V->m, Z->m, L->m, heads, scale, dropout, seed, bias ? &bias->v : nullptr,
                                edge ? &edge->m : nullptr);
    });
}
int hnhd_alg_sparse_attention_backward_edge(hnhd_alg_t *a, hnhd_dense_t *Q, hnhd_dense_t *K, hnhd_dense_t *V, hnhd_dense_t *Z,
                                            hnhd_dense_t *L, hnhd_dense_t *dZ, hnhd_dense_t *dQ, hnhd_dense_t *dK,
                                            hnhd_dense_t *dV, int heads, double scale, double dropout, uint64_t seed,
                                            const hnhd_vec_t *bias_A, const hnhd_vec_t *bias_B, hnhd_vec_t *dbias_A,
                                            hnhd_vec_t *dbias_B, const hnhd_dense_t *edge_A, const hnhd_dense_t *edge_B,
                                            hnhd_dense_t *dedge) {
    return guarded([&] {
        if (!a || !Q || !K || !V || !Z || !L || !dZ || !dQ || !dK || !dV)
            throw hnh::Error(HNH_E_INVALID, "hnhd_alg_sparse_attention_backward_edge: null argument");
        if (!std::isfinite(scale))
            throw hnh::Error(HNH_E_INVALID, "hnhd_alg_sparse_attention_backward_edge: the scale must be finite");
        a->alg->sparseAttentionBackward(Q->m, K->m, V->m, Z->m, L->m, dZ->m, dQ->m, dK->m, dV->m, heads, scale, dropout, seed,
                                        bias_A ? &bias_A->v : nullptr, bias_B ? &bias_B->v : nullptr,
                                        dbias_A ? &dbias_A->v : nullptr, dbias_B ? &dbias_B->v : nullptr,
                                        edge_A ? &edge_A->m : nullptr, edge_B ? &edge_B->m : nullptr, dedge ? &dedge->m : nullptr);
    });
}
int hnhd_alg_entry_coordinates(hnhd_alg_t *a, int mode, hnhd_vec_t *rows, hnhd_vec_t *cols) {
    return guarded([&] {
        if (!a || !rows || !cols) throw hnh::Error(HNH_E_INVALID, "hnhd_alg_entry_coordinates: null argument");
        if (rows == cols) throw hnh::Error(HNH_E_INVALID, "hnhd_alg_entry_coordinates: rows and cols are one vector");
        a->alg->entryCoordinates(value_order(mode), rows->v, cols->v);
    });
}

int hnhd_timer_start(void) {
    return guarded([] {
        if (!g_t0) {
            hnh::cuda_check(cudaEventCreate(&g_t0), "cudaEventCreate");
            hnh::cuda_check(cudaEventCreate(&g_t1), "cudaEventCreate");
        }
        hnh::cuda_check(cudaEventRecord(g_t0, hnh::Runtime::get().compute_stream()), "cudaEventRecord");
    });
}
int hnhd_timer_stop(double *ms_out) {
    return guarded([&] {
        if (!g_t0) throw hnh::Error(HNH_E_INVALID, "hnhd_timer_stop without start");
        hnh::cuda_check(cudaEventRecord(g_t1, hnh::Runtime::get().compute_stream()), "cudaEventRecord");
        hnh::cuda_check(cudaEventSynchronize(g_t1), "cudaEventSynchronize");
        float ms = 0.f;
        hnh::cuda_check(cudaEventElapsedTime(&ms, g_t0, g_t1), "cudaEventElapsedTime");
        *ms_out = ms;
    });
}

int hnhd_benchmark_algorithm(hnhd_spmat_t *S, const char *algorithm_name, const char *output_file, int fused, int R, int c,
                             const char *app, int trials, int warmup, char *json_out, size_t capacity) {
    int n = 0;
    int rc = guarded([&] {
        json j = benchmark_algorithm_ex(&S->m, algorithm_name, output_file ? output_file : "", fused != 0, R, c,
                                        app ? app : "vanilla", trials, warmup);
        n = json_out ? copy_json(j, json_out, capacity) : 0;
    });
    return rc ? rc : n;
}

int hnhd_als_residuals(hnhd_alg_t *a, int steps, double *out2) {
    return guarded([&] {
        if (!a || !out2) throw hnh::Error(HNH_E_INVALID, "null argument");
        Distributed_ALS als(a->alg.get(), true);
        als.initializeEmbeddings();
        out2[0] = als.computeResidual();
        for (int i = 0; i < steps; i++) {
            als.cg_optimizer(Amat, 10);
            als.cg_optimizer(Bmat, 10);
        }
        out2[1] = als.computeResidual();
    });
}

int hnhd_als_run(hnhd_alg_t *a, const double *hostAgt, const double *hostBgt, const double *hostA0, const double *hostB0,
                 int steps, int cg_iters, double *out2, double *hostA_out, double *hostB_out) {
    return guarded([&] {
        if (!a || !hostAgt || !hostBgt || !hostA0 || !hostB0 || !out2 || steps < 0 || cg_iters < 0)
            throw hnh::Error(HNH_E_INVALID, "hnhd_als_run: bad argument");
        Distributed_Sparse *d = a->alg.get();
        Distributed_ALS als(d, false);
        DenseMatrix Agt = d->like_A_matrix(0.0), Bgt = d->like_B_matrix(0.0);
        Agt.copy_from_host(hostAgt);
        Bgt.copy_from_host(hostBgt);
        VectorXd ones = d->like_S_values(1.0);
        als.ground_truth = d->like_S_values(0.0);
        d->initial_shift(&Agt, &Bgt, k_sddmmA);
        d->sddmmA(Agt, Bgt, ones, als.ground_truth);
        d->de_shift(&Agt, &Bgt, k_sddmmA);
        VectorXd ones_t = d->like_ST_values(1.0);
        als.ground_truth_transpose = d->like_ST_values(0.0);
        d->initial_shift(&Agt, &Bgt, k_sddmmB);
        d->sddmmB(Agt, Bgt, ones_t, als.ground_truth_transpose);
        d->de_shift(&Agt, &Bgt, k_sddmmB);
        als.A = d->like_A_matrix(0.0);
        als.B = d->like_B_matrix(0.0);
        als.A.copy_from_host(hostA0);
        als.B.copy_from_host(hostB0);
        out2[0] = als.computeResidual();
        for (int i = 0; i < steps; i++) {
            als.cg_optimizer(Amat, cg_iters);
            als.cg_optimizer(Bmat, cg_iters);
        }
        out2[1] = als.computeResidual();
        if (hostA_out) als.A.copy_to_host(hostA_out);
        if (hostB_out) als.B.copy_to_host(hostB_out);
    });
}

// ---- training ------------------------------------------------------------------------------------------
int hnhd_labels_create(hnhd_alg_t *a, const int32_t *host, int64_t n, int num_classes, hnhd_labels_t **out) {
    return guarded([&] {
        if (!a || !out) throw hnh::Error(HNH_E_INVALID, "hnhd_labels_create: null argument");
        std::unique_ptr<hnhd_labels> l(new hnhd_labels);
        l->l.reset(new hnh::NodeLabels(host, n, a->alg->localArows, num_classes));
        *out = l.release();
    });
}
void hnhd_labels_destroy(hnhd_labels_t *l) { delete l; }

int hnhd_adamw_create(double lr, double beta1, double beta2, double eps, double weight_decay, double max_grad_norm,
                      hnhd_adamw_t **out) {
    return guarded([&] {
        if (!out) throw hnh::Error(HNH_E_INVALID, "hnhd_adamw_create: null argument");
        std::unique_ptr<hnhd_adamw> o(new hnhd_adamw);
        o->o.reset(new hnh::AdamW(lr, beta1, beta2, eps, weight_decay, max_grad_norm));
        *out = o.release();
    });
}
int hnhd_adamw_set_lr(hnhd_adamw_t *opt, double lr) {
    return guarded([&] {
        if (!opt) throw hnh::Error(HNH_E_INVALID, "hnhd_adamw_set_lr: null optimizer");
        opt->o->set_lr(lr);
    });
}
void hnhd_adamw_destroy(hnhd_adamw_t *opt) { delete opt; }

// ---- link prediction -----------------------------------------------------------------------------------------
int hnhd_alg_link_loss(hnhd_alg_t *T, hnhd_dense_t *H_A, hnhd_dense_t *H_B, hnhd_dense_t *dH_A, hnhd_dense_t *dH_B,
                       hnhd_vec_t *scores, double out[3]) {
    return guarded([&] {
        if (!T || !H_A || !H_B || !out) throw hnh::Error(HNH_E_INVALID, "hnhd_alg_link_loss: null argument");
        const int64_t count = (int64_t)T->alg->S->dist_nnz;
        VectorXd sums(2);
        T->alg->linkLoss(H_A->m, H_B->m, count > 0 ? 1.0 / (double)count : 0.0, dH_A ? &dH_A->m : nullptr,
                         dH_B ? &dH_B->m : nullptr, scores ? &scores->v : nullptr, sums.data());
        double h[2];
        cudaStream_t s = hnh::Runtime::get().compute_stream();
        hnh::cuda_check(cudaMemcpyAsync(h, sums.data(), sizeof h, cudaMemcpyDeviceToHost, s), "link loss results");
        hnh::cuda_check(cudaStreamSynchronize(s), "link loss results");
        out[0] = count > 0 ? h[0] / (double)count : 0.0;
        out[1] = h[1];
        out[2] = (double)count;
    });
}
int hnhd_link_targets_create(hnhd_alg_t *model, hnhd_alg_t *T, hnhd_link_targets_t **out) {
    return guarded([&] {
        if (!model || !T || !out) throw hnh::Error(HNH_E_INVALID, "hnhd_link_targets_create: null argument");
        std::unique_ptr<hnhd_link_targets> t(new hnhd_link_targets);
        t->t.reset(new hnh::LinkTargets(*model->alg, *T->alg));
        *out = t.release();
    });
}
void hnhd_link_targets_destroy(hnhd_link_targets_t *t) { delete t; }

// ---- max aggregation -------------------------------------------------------------------------------------------------
int hnhd_alg_max_aggregate(hnhd_alg_t *a, hnhd_dense_t *X, hnhd_dense_t *Z, hnhd_dense_t *C) {
    return guarded([&] {
        if (!a || !X || !Z || !C) throw hnh::Error(HNH_E_INVALID, "hnhd_alg_max_aggregate: null argument");
        a->alg->maxAggregate(X->m, Z->m, C->m);
    });
}
int hnhd_alg_max_aggregate_backward(hnhd_alg_t *a, hnhd_dense_t *X, hnhd_dense_t *Z, hnhd_dense_t *C, hnhd_dense_t *dZ,
                                    hnhd_dense_t *dX, int accumulate) {
    return guarded([&] {
        if (!a || !X || !Z || !C || !dZ || !dX) throw hnh::Error(HNH_E_INVALID, "hnhd_alg_max_aggregate_backward: null argument");
        a->alg->maxAggregateBackward(X->m, Z->m, C->m, dZ->m, dX->m, accumulate != 0);
    });
}

// ---- relational aggregation ------------------------------------------------------------------------------------------
int hnhd_alg_relational_aggregate(hnhd_alg_t *a, hnhd_dense_t *X, hnhd_dense_t *A, int num_relations) {
    return guarded([&] {
        if (!a || !X || !A) throw hnh::Error(HNH_E_INVALID, "hnhd_alg_relational_aggregate: null argument");
        a->alg->relationalAggregate(X->m, A->m, num_relations);
    });
}
int hnhd_alg_relational_aggregate_backward(hnhd_alg_t *a, hnhd_dense_t *dA, hnhd_dense_t *dX, int num_relations, int accumulate) {
    return guarded([&] {
        if (!a || !dA || !dX) throw hnh::Error(HNH_E_INVALID, "hnhd_alg_relational_aggregate_backward: null argument");
        a->alg->relationalAggregateBackward(dA->m, dX->m, num_relations, accumulate != 0);
    });
}

int hnhd_alg_basis_aggregate(hnhd_alg_t *a, hnhd_dense_t *X, hnhd_dense_t *H, hnhd_dense_t *comp, int num_relations,
                             hnhd_dense_t *scale) {
    return guarded([&] {
        if (!a || !X || !H || !comp) throw hnh::Error(HNH_E_INVALID, "hnhd_alg_basis_aggregate: null argument");
        a->alg->basisAggregate(X->m, H->m, comp->m, num_relations, scale ? &scale->m : nullptr);
    });
}
int hnhd_alg_basis_aggregate_backward(hnhd_alg_t *a, hnhd_dense_t *dH, hnhd_dense_t *X, hnhd_dense_t *dX, hnhd_dense_t *comp,
                                      hnhd_dense_t *dcomp, int num_relations, hnhd_dense_t *scale, int accumulate) {
    return guarded([&] {
        if (!a || !dH || !X || !dX || !comp || !dcomp) throw hnh::Error(HNH_E_INVALID, "hnhd_alg_basis_aggregate_backward: null argument");
        a->alg->basisAggregateBackward(dH->m, X->m, dX->m, comp->m, dcomp->m, num_relations, scale ? &scale->m : nullptr,
                                       accumulate != 0);
    });
}

// ---- graph models: one handle for GAT, the graph transformer, GraphSAGE and R-GCN -------------------------------------
int hnhd_gat_create(hnhd_alg_t *a, int n_layers, const int *layers3, double alpha, hnhd_model_t **out) {
    return guarded([&] {
        if (!a || !layers3 || !out || n_layers <= 0) throw hnh::Error(HNH_E_INVALID, "hnhd_gat_create: bad argument");
        vector<GATLayer> layers;
        for (int i = 0; i < n_layers; i++) {
            if (layers3[3 * i] <= 0 || layers3[3 * i + 1] <= 0 || layers3[3 * i + 2] <= 0)
                throw hnh::Error(HNH_E_INVALID, "hnhd_gat_create: layer sizes must be positive");
            layers.emplace_back(layers3[3 * i], layers3[3 * i + 1], layers3[3 * i + 2]);
        }
        std::unique_ptr<GAT> g(new GAT(layers, a->alg.get()));
        g->leaky_relu_alpha = alpha;
        *out = new hnhd_model{std::move(g)};
    });
}
int hnhd_gt_create(hnhd_alg_t *a, int n_layers, const int *layers3, int edge_dim, int beta, hnhd_model_t **out) {
    return guarded([&] {
        if (!a || !layers3 || !out || n_layers <= 0) throw hnh::Error(HNH_E_INVALID, "hnhd_gt_create: bad argument");
        vector<GraphTransformerLayer> layers;
        for (int i = 0; i < n_layers; i++) layers.emplace_back(layers3[3 * i], layers3[3 * i + 1], layers3[3 * i + 2]);
        *out = new hnhd_model{std::unique_ptr<GraphModel>(new GraphTransformer(layers, a->alg.get(), edge_dim, beta != 0))};
    });
}
int hnhd_gt_create_block(hnhd_alg_t *a, int n_layers, const int *layers3, int edge_dim, int beta, int ffn_ratio, double norm_eps,
                         hnhd_model_t **out) {
    return guarded([&] {
        if (!a || !layers3 || !out || n_layers <= 0) throw hnh::Error(HNH_E_INVALID, "hnhd_gt_create_block: bad argument");
        vector<GraphTransformerLayer> layers;
        for (int i = 0; i < n_layers; i++) layers.emplace_back(layers3[3 * i], layers3[3 * i + 1], layers3[3 * i + 2]);
        *out = new hnhd_model{
            std::unique_ptr<GraphModel>(new GraphTransformer(layers, a->alg.get(), edge_dim, beta != 0, ffn_ratio, norm_eps))};
    });
}
int hnhd_sage_create(hnhd_alg_t *a, int n_layers, const int *layers2, const char *aggr, hnhd_model_t **out) {
    return guarded([&] {
        if (!a || !layers2 || !aggr || !out || n_layers <= 0) throw hnh::Error(HNH_E_INVALID, "hnhd_sage_create: bad argument");
        vector<GraphSAGELayer> layers;
        for (int i = 0; i < n_layers; i++) layers.emplace_back(layers2[2 * i], layers2[2 * i + 1]);
        *out = new hnhd_model{std::unique_ptr<GraphModel>(new GraphSAGE(layers, a->alg.get(), aggr))};
    });
}
static int rgcn_create(hnhd_alg_t *a, int n_layers, const int *layers2, int num_relations, const char *aggr, int num_bases,
                       hnhd_model_t **out, const char *who) {
    return guarded([&] {
        if (!a || !layers2 || !aggr || !out || n_layers <= 0) throw hnh::Error(HNH_E_INVALID, string(who) + ": bad argument");
        // refused before the device is touched
        vector<std::pair<int, int>> widths;
        for (int i = 0; i < n_layers; i++) widths.emplace_back(layers2[2 * i], layers2[2 * i + 1]);
        RGCN::parse(aggr);
        RGCN::check_layers(widths, num_relations, num_bases);
        vector<RGCNLayer> layers;
        for (auto [f, r] : widths) layers.emplace_back(f, r);
        *out = new hnhd_model{std::unique_ptr<GraphModel>(new RGCN(layers, a->alg.get(), num_relations, aggr, num_bases))};
    });
}
int hnhd_rgcn_create(hnhd_alg_t *a, int n_layers, const int *layers2, int num_relations, const char *aggr, hnhd_model_t **out) {
    return rgcn_create(a, n_layers, layers2, num_relations, aggr, 0, out, "hnhd_rgcn_create");
}
int hnhd_rgcn_create_bases(hnhd_alg_t *a, int n_layers, const int *layers2, int num_relations, int num_bases, const char *aggr,
                           hnhd_model_t **out) {
    if (num_bases < 1) return hnh::set_error(HNH_E_INVALID, "hnhd_rgcn_create_bases: the basis count must be positive (got %d)", num_bases);
    return rgcn_create(a, n_layers, layers2, num_relations, aggr, num_bases, out, "hnhd_rgcn_create_bases");
}

// ---- every model
int hnhd_model_buffer_shape(hnhd_model_t *m, int buffer, int64_t *rows, int64_t *cols) {
    return guarded([&] {
        DenseMatrix &b = model_buffer(m, buffer);
        if (rows) *rows = b.rows();
        if (cols) *cols = b.cols();
    });
}
int hnhd_model_set_input(hnhd_model_t *m, const double *host) {
    return guarded([&] {
        DenseMatrix &b = model_buffer(m, 0);
        if (!host) throw hnh::Error(HNH_E_INVALID, "null host pointer");
        b.copy_from_host(host);
        m->m->activations_current = false;
    });
}
int hnhd_model_get_buffer(hnhd_model_t *m, int buffer, double *host) {
    return guarded([&] {
        DenseMatrix &b = model_buffer(m, buffer);
        if (!host) throw hnh::Error(HNH_E_INVALID, "null host pointer");
        b.copy_to_host(host);
    });
}
int hnhd_model_forward(hnhd_model_t *m, double dropout, uint64_t seed) {
    return guarded([&] { model(m).forward(dropout, seed); });
}
int hnhd_model_backward(hnhd_model_t *m, const double *host_output_grad) {
    return guarded([&] {
        GraphModel &g = model(m);
        if (!host_output_grad) throw hnh::Error(HNH_E_INVALID, "null host pointer");
        const DenseMatrix &out = g.buffers.back();
        DenseMatrix grad = DenseMatrix::from_host(host_output_grad, out.rows(), out.cols());
        g.backwardPass(grad);
    });
}
int hnhd_model_get_input_grad(hnhd_model_t *m, double *host) {
    return guarded([&] {
        GraphModel &g = model(m);
        if (!host) throw hnh::Error(HNH_E_INVALID, "null host pointer");
        if (g.input_grad.size() != g.buffers[0].size()) throw hnh::Error(HNH_E_INVALID, g.model_name + ": no backward pass has run");
        g.input_grad.copy_to_host(host);
    });
}
int hnhd_model_param_shape(hnhd_model_t *m, int layer, const char *name, int64_t *rows, int64_t *cols) {
    return guarded([&] {
        const ParamRef p = model_param(m, layer, name);
        if (rows) *rows = p.rows;
        if (cols) *cols = p.cols;
    });
}
int hnhd_model_set_param(hnhd_model_t *m, int layer, const char *name, const double *host) {
    return guarded([&] {
        const ParamRef p = model_param(m, layer, name);
        if (!host) throw hnh::Error(HNH_E_INVALID, "null host pointer");
        sync_copy(p.value, host, p.rows * p.cols, cudaMemcpyHostToDevice);
        m->m->activations_current = false;
    });
}
int hnhd_model_get_param(hnhd_model_t *m, int layer, const char *name, double *host) {
    return guarded([&] {
        const ParamRef p = model_param(m, layer, name);
        if (!host) throw hnh::Error(HNH_E_INVALID, "null host pointer");
        sync_copy(host, p.value, p.rows * p.cols, cudaMemcpyDeviceToHost);
    });
}
int hnhd_model_get_param_grad(hnhd_model_t *m, int layer, const char *name, double *host) {
    return guarded([&] {
        const ParamRef p = model_param(m, layer, name);
        if (!host) throw hnh::Error(HNH_E_INVALID, "null host pointer");
        if (!p.grad) throw hnh::Error(HNH_E_INVALID, m->m->model_name + ": no backward pass has run");
        sync_copy(host, p.grad, p.rows * p.cols, cudaMemcpyDeviceToHost);
    });
}
static void train_out(const hnh::TrainResult &r, double out[4]) {
    out[0] = r.loss;
    out[1] = (double)r.correct;
    out[2] = (double)r.labelled;
    out[3] = r.grad_norm;
}
int hnhd_model_train_step(hnhd_model_t *m, const hnhd_labels_t *labels, hnhd_adamw_t *opt, double dropout, uint64_t seed,
                          double out[4]) {
    return guarded([&] {
        if (!m || !labels || !opt || !out) throw hnh::Error(HNH_E_INVALID, "hnhd_model_train_step: null argument");
        train_out(hnh::trainStep(*m->m, *labels->l, *opt->o, dropout, seed), out);
    });
}
int hnhd_model_link_train_step(hnhd_model_t *m, const hnhd_link_targets_t *t, hnhd_adamw_t *opt, double dropout, uint64_t seed,
                               double out[4]) {
    return guarded([&] {
        if (!m || !t || !opt || !out) throw hnh::Error(HNH_E_INVALID, "hnhd_model_link_train_step: null argument");
        train_out(hnh::linkTrainStep(*m->m, *t->t, *opt->o, dropout, seed), out);
    });
}
int hnhd_model_link_evaluate(hnhd_model_t *m, const hnhd_link_targets_t *t, hnhd_vec_t *scores, double out[3]) {
    return guarded([&] {
        if (!m || !t || !out) throw hnh::Error(HNH_E_INVALID, "hnhd_model_link_evaluate: null argument");
        const hnh::LinkResult r = hnh::linkEvaluate(*m->m, *t->t, scores ? &scores->v : nullptr);
        out[0] = r.loss;
        out[1] = (double)r.correct;
        out[2] = (double)r.count;
    });
}
void hnhd_model_destroy(hnhd_model_t *m) { delete m; }

// ---- GAT only: weights and attention vectors by (layer, head)
// the layer of a (layer, head) pair, refused for another model, layer or head
static GATLayer &gat_layer(hnhd_model_t *m, int layer, int head) {
    GAT &g = model_as<GAT>(m, "GAT");
    if (layer < 0 || layer >= (int)g.layers.size()) throw hnh::Error(HNH_E_INVALID, "gat: no such layer");
    GATLayer &l = g.layers[(size_t)layer];
    if (head < 0 || head >= l.num_heads) throw hnh::Error(HNH_E_INVALID, "gat: no such head");
    return l;
}
int hnhd_gat_weight_shape(hnhd_model_t *m, int layer, int head, int64_t *rows, int64_t *cols) {
    return guarded([&] {
        DenseMatrix &w = gat_layer(m, layer, head).wMats[(size_t)head];
        if (rows) *rows = w.rows();
        if (cols) *cols = w.cols();
    });
}
int hnhd_gat_set_weight(hnhd_model_t *m, int layer, int head, const double *host) {
    return guarded([&] {
        if (!host) throw hnh::Error(HNH_E_INVALID, "null host pointer");
        gat_layer(m, layer, head).wMats[(size_t)head].copy_from_host(host);
        m->m->activations_current = false;
    });
}
int hnhd_gat_get_weight(hnhd_model_t *m, int layer, int head, double *host) {
    return guarded([&] {
        if (!host) throw hnh::Error(HNH_E_INVALID, "null host pointer");
        gat_layer(m, layer, head).wMats[(size_t)head].copy_to_host(host);
    });
}
int hnhd_gat_get_weight_grad(hnhd_model_t *m, int layer, int head, double *host) {
    return guarded([&] {
        if (!host) throw hnh::Error(HNH_E_INVALID, "null host pointer");
        const GATLayer &l = gat_layer(m, layer, head);
        if (l.wGrads.size() != l.wMats.size()) throw hnh::Error(HNH_E_INVALID, "gat: no backward pass has run");
        l.wGrads[(size_t)head].copy_to_host(host);
    });
}
int hnhd_gat_set_attention(hnhd_model_t *m, const char *kind) {
    return guarded([&] {
        if (!m || !kind) throw hnh::Error(HNH_E_INVALID, "hnhd_gat_set_attention: null argument");
        model_as<GAT>(m, "GAT").set_attention(kind);
    });
}
int hnhd_gat_set_attention_vectors(hnhd_model_t *m, int layer, int head, const double *a1, const double *a2) {
    return guarded([&] {
        if (!a1 || !a2) throw hnh::Error(HNH_E_INVALID, "null host pointer");
        GATLayer &l = gat_layer(m, layer, head);
        const int64_t off = (int64_t)head * l.features_per_head;
        sync_copy(l.a1.data() + off, a1, l.features_per_head, cudaMemcpyHostToDevice);
        sync_copy(l.a2.data() + off, a2, l.features_per_head, cudaMemcpyHostToDevice);
        m->m->activations_current = false;
    });
}
int hnhd_gat_get_attention_vectors(hnhd_model_t *m, int layer, int head, double *a1, double *a2) {
    return guarded([&] {
        if (!a1 || !a2) throw hnh::Error(HNH_E_INVALID, "null host pointer");
        GATLayer &l = gat_layer(m, layer, head);
        const int64_t off = (int64_t)head * l.features_per_head;
        sync_copy(a1, l.a1.data() + off, l.features_per_head, cudaMemcpyDeviceToHost);
        sync_copy(a2, l.a2.data() + off, l.features_per_head, cudaMemcpyDeviceToHost);
    });
}
int hnhd_gat_get_attention_grads(hnhd_model_t *m, int layer, int head, double *da1, double *da2) {
    return guarded([&] {
        if (!da1 || !da2) throw hnh::Error(HNH_E_INVALID, "null host pointer");
        const GATLayer &l = gat_layer(m, layer, head);
        if (l.a1Grads.size() != l.a1.size() || l.a2Grads.size() != l.a2.size())
            throw hnh::Error(HNH_E_INVALID, "gat: no backward pass has run");
        const int64_t off = (int64_t)head * l.features_per_head;
        sync_copy(da1, l.a1Grads.data() + off, l.features_per_head, cudaMemcpyDeviceToHost);
        sync_copy(da2, l.a2Grads.data() + off, l.features_per_head, cudaMemcpyDeviceToHost);
    });
}

// ---- graph transformer only
int hnhd_gt_set_edge_attributes(hnhd_model_t *m, const double *attr_A, int64_t n_A, const double *attr_B, int64_t n_B) {
    return guarded([&] {
        GraphTransformer &g = model_as<GraphTransformer>(m, "graph transformer");
        if ((n_A > 0 && !attr_A) || (n_B > 0 && !attr_B)) throw hnh::Error(HNH_E_INVALID, "null host pointer");
        g.setEdgeAttributes(attr_A, n_A, attr_B, n_B);
    });
}

}  // extern "C"
