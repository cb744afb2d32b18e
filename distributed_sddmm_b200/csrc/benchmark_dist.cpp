// benchmark_dist.cpp -- benchmark_algorithm for the H100-native library (see the header).
#include "hnh/benchmark_dist.hpp"

#include <cstring>
#include <ctime>

#include <unistd.h>

#include <cstdlib>
#include <fstream>
#include <iostream>
#include <memory>

#include "hnh/15D_dense_shift.hpp"
#include "hnh/15D_sparse_shift.hpp"
#include "hnh/25D_cannon_dense.hpp"
#include "hnh/25D_cannon_sparse.hpp"
#include "hnh/als_conjugate_gradients.h"
#include "hnh/gat.hpp"
#include "hnh/graph_transformer.hpp"
#include "hnh_b200.h"

Distributed_Sparse *hnh_make_algorithm(const string &name, SpmatLocal *spmat, int R, int c, KernelImplementation *k) {
    if (name == "15d_fusion1") return new Sparse15D_Dense_Shift(spmat, R, c, 1, k);
    if (name == "15d_fusion2") return new Sparse15D_Dense_Shift(spmat, R, c, 2, k);
    if (name == "15d_sparse") return new Sparse15D_Sparse_Shift(spmat, R, c, k);
    if (name == "25d_dense_replicate") return new Sparse25D_Cannon_Dense(spmat, R, c, k);
    if (name == "25d_sparse_replicate") return new Sparse25D_Cannon_Sparse(spmat, R, c, k);
    throw hnh::Error(HNH_E_INVALID, "unknown algorithm name: " + name);
}

json benchmark_algorithm_ex(SpmatLocal *spmat, string algorithm_name, string output_file, bool fused, int R, int c,
                            string app, int trials, int warmup) {
    auto world = hnh::Comm::world();
    const int rank = world->rank();
    hnh::Runtime &rt = hnh::Runtime::get();
    StandardKernel local_ops;
    std::unique_ptr<Distributed_Sparse> d_ops(hnh_make_algorithm(algorithm_name, spmat, R, c, &local_ops));
    std::unique_ptr<Distributed_ALS> d_als;
    std::unique_ptr<GAT> gnn;
    std::unique_ptr<GraphTransformer> transformer;
    DenseMatrix gat_output_grad;
    const bool gat_app = app == "gat" || app == "gat_train" || app == "gat_softmax" || app == "gat_softmax_train" ||
                         app == "gat_additive" || app == "gat_additive_train" || app == "gat_v2" || app == "gat_v2_train";
    const bool gat_train =
        app == "gat_train" || app == "gat_softmax_train" || app == "gat_additive_train" || app == "gat_v2_train";
    const bool gt_block = app == "graph_transformer_block" || app == "graph_transformer_block_train";
    const bool gt_train = app == "graph_transformer_train" || app == "graph_transformer_block_train";
    const bool gt_app = app == "graph_transformer" || app == "graph_transformer_train" || gt_block;
    if (gt_app) {
        // GAT's three layer shapes as TransformerConv layers (no edge features, no gate; the parameters stay zero,
        // as GAT's weights do); graph_transformer_block*: as transformer blocks with ffn_ratio = 2 (LayerNorm gains
        // 1); *_train: forwardPass() then backwardPass(dL/d output = ones) per call
        vector<GraphTransformerLayer> layers{GraphTransformerLayer(256, 256, 4), GraphTransformerLayer(1024, 256, 4),
                                             GraphTransformerLayer(1024, 256, 6)};
        transformer.reset(new GraphTransformer(layers, d_ops.get(), 0, false, gt_block ? 2 : 0));
        if (gt_train)
            gat_output_grad = DenseMatrix::Constant(transformer->buffers.back().rows(), transformer->buffers.back().cols(), 1.0);
    } else if (gat_app) {
        // the three layers of the reference's GAT benchmark: (input width, width per head, heads)
        vector<GATLayer> layers{GATLayer(256, 256, 4), GATLayer(1024, 256, 4), GATLayer(1024, 256, 6)};
        gnn.reset(new GAT(layers, d_ops.get()));
        // gat_softmax*: softmax attention (the edge softmax of the scores) instead of the reference's
        if (app == "gat_softmax" || app == "gat_softmax_train") {
            d_ops->check_full_rows("GAT softmax attention");
            gnn->set_attention("softmax");
        }
        // gat_additive*: additive attention (the attention vectors stay zero, as the weights do)
        if (app == "gat_additive" || app == "gat_additive_train") {
            d_ops->check_full_rows("GAT additive attention");
            gnn->set_attention("additive");
        }
        // gat_v2*: GATv2 attention (the attention vectors stay zero, as the weights do)
        if (app == "gat_v2" || app == "gat_v2_train") {
            d_ops->check_full_rows("GAT GATv2 attention");
            gnn->set_attention("gatv2");
        }
        // gat_train / gat_softmax_train / gat_additive_train / gat_v2_train: forwardPass() then backwardPass(dL/d output = ones) per call
        if (gat_train) {
            gnn->check_backward_supported();
            gat_output_grad = DenseMatrix::Constant(gnn->buffers.back().rows(), gnn->buffers.back().cols(), 1.0);
        }
    } else if (app == "als") {
        d_als.reset(new Distributed_ALS(d_ops.get(), true));
    } else if (app != "vanilla") {
        throw hnh::Error(HNH_E_INVALID, "app must be \"vanilla\", \"als\", \"gat\", \"gat_train\", \"gat_softmax\", "
                                        "\"gat_softmax_train\", \"gat_additive\", \"gat_additive_train\", \"gat_v2\", "
                                        "\"gat_v2_train\", \"graph_transformer\", \"graph_transformer_train\", "
                                        "\"graph_transformer_block\" or \"graph_transformer_block_train\"");
    }

    DenseMatrix A = d_ops->like_A_matrix(0.001);
    DenseMatrix B = d_ops->like_B_matrix(0.001);
    VectorXd Sv = d_ops->like_S_values(1.0);
    VectorXd sddmm_result = d_ops->like_S_values(0.0);
    if (rank == 0) std::cout << "Starting benchmark " << app << std::endl;

    double application_communication_time = 0.0;
    auto one_call = [&]() {
        if (app == "vanilla") {
            if (fused) {
                d_ops->fusedSpMM(A, B, Sv, sddmm_result, Amat);
            } else {
                d_ops->sddmmA(A, B, Sv, sddmm_result);
                d_ops->spmmA(A, B, Sv);
            }
        } else if (gt_app) {
            transformer->forwardPass(0.0, 0);
            if (gt_train) transformer->backwardPass(gat_output_grad);
        } else if (gat_app) {
            gnn->forwardPass();
            if (gat_train) gnn->backwardPass(gat_output_grad);
        } else {
            d_als->application_communication_time = 0.0;
            d_als->run_cg(1);
            application_communication_time = d_als->application_communication_time;
        }
    };
    for (int w = 0; w < warmup; w++) one_call();
    rt.sync_all();
    world->barrier();
    d_ops->reset_performance_timers();

    cudaEvent_t e0, e1;
    hnh::cuda_check(cudaEventCreate(&e0), "cudaEventCreate");
    hnh::cuda_check(cudaEventCreate(&e1), "cudaEventCreate");
    my_timer_t t = start_clock();
    hnh::cuda_check(cudaEventRecord(e0, rt.compute_stream()), "cudaEventRecord");
    int num_trials = 0;
    do {
        num_trials++;
        one_call();
    } while (num_trials < trials);
    hnh::cuda_check(cudaEventRecord(e1, rt.compute_stream()), "cudaEventRecord");
    rt.sync_all();
    world->barrier();
    const double wall = stop_clock_get_elapsed(t);
    float dev_ms = 0.f;
    hnh::cuda_check(cudaEventElapsedTime(&dev_ms, e0, e1), "cudaEventElapsedTime");
    cudaEventDestroy(e0);
    cudaEventDestroy(e1);
    // device time, max over ranks (all ranks are event-timed on their own GPU)
    vector<double> all((size_t)world->size());
    double mine = dev_ms * 1e-3;
    world->host_allgather(&mine, all.data(), sizeof(double));
    const double elapsed = *std::max_element(all.begin(), all.end());

    const double ops = 2.0 * (double)spmat->dist_nnz * 2.0 * R * num_trials;
    json j = json::object();
    j["elapsed"] = elapsed;
    j["elapsed_wall"] = wall;
    j["overall_throughput"] = ops / elapsed / 1e9;
    j["fused"] = fused;
    j["num_trials"] = num_trials;
    j["warmup"] = warmup;
    j["alg_name"] = algorithm_name;
    j["alg_info"] = d_ops->json_algorithm_info();
    j["application_communication_time"] = application_communication_time;
    j["perf_stats"] = d_ops->json_perf_statistics();
    if (rank == 0 && !output_file.empty()) {
        std::ofstream fout(output_file, std::ios_base::app);
        fout << j.dump(4) << "," << std::endl;
    }
    return j;
}

void benchmark_algorithm(SpmatLocal *spmat, string algorithm_name, string output_file, bool fused, int R, int c,
                         string app) {
    benchmark_algorithm_ex(spmat, algorithm_name, output_file, fused, R, c, app, 5, 0);
}

void hnh_world_init_from_env() {
    const char *ws = getenv("WORLD_SIZE"), *rk = getenv("RANK"), *lr = getenv("LOCAL_RANK");
    const int size = ws ? atoi(ws) : 1, rank = rk ? atoi(rk) : 0;
    if (lr) hnh::cuda_check(cudaSetDevice(atoi(lr)), "cudaSetDevice");
    if (size <= 1) {
        hnh::Comm::init_self();
        return;
    }
    const char *path = getenv("HNH_NCCL_ID_FILE");
    if (!path) throw hnh::Error(HNH_E_COMM, "WORLD_SIZE > 1 needs HNH_NCCL_ID_FILE (shared path for the NCCL unique id)");
    // The file must belong to THIS launch: a leftover from an earlier run (or from a crash before the clean-up
    // below) would hand the readers a dead id and ncclCommInitRank would hang.  Three guards: (1) the record
    // carries a launch nonce (HNH_LAUNCH_ID, else TORCHELASTIC_RUN_ID, else MASTER_ADDR:MASTER_PORT) that the
    // readers verify; (2) rank 0 unlinks the path before writing and again once every rank has joined the
    // communicator; (3) with no nonce in the environment, a record written more than two minutes before the
    // reader started is rejected as stale.
    struct Record {
        char magic[8];
        char nonce[120];
        int64_t written_at;
        char id[HNHD_NCCL_ID_BYTES];
    } rec;
    string nonce;
    if (const char *e = getenv("HNH_LAUNCH_ID")) nonce = e;
    else if (const char *e2 = getenv("TORCHELASTIC_RUN_ID")) nonce = e2;
    else if (getenv("MASTER_PORT")) nonce = string(getenv("MASTER_ADDR") ? getenv("MASTER_ADDR") : "") + ":" + getenv("MASTER_PORT");
    if (nonce.size() >= sizeof rec.nonce) nonce.resize(sizeof rec.nonce - 1);
    const int64_t started = (int64_t)time(nullptr);
    char id[HNHD_NCCL_ID_BYTES];
    if (rank == 0) {
        unlink(path);
        hnh::Comm::nccl_unique_id(id);
        std::memset(&rec, 0, sizeof rec);
        std::memcpy(rec.magic, "HNHNCCL1", 8);
        std::memcpy(rec.nonce, nonce.c_str(), nonce.size());
        rec.written_at = (int64_t)time(nullptr);
        std::memcpy(rec.id, id, sizeof id);
        string tmp = string(path) + ".tmp." + std::to_string((long long)getpid());
        std::ofstream f(tmp, std::ios::binary);
        f.write((const char *)&rec, sizeof rec);
        f.close();
        if (!f || rename(tmp.c_str(), path) != 0) throw hnh::Error(HNH_E_COMM, string("cannot write the NCCL id file ") + path);
    } else {
        for (int tries = 0;; tries++) {
            std::ifstream f(path, std::ios::binary);
            if (f && f.read((char *)&rec, sizeof rec) && std::memcmp(rec.magic, "HNHNCCL1", 8) == 0) {
                rec.nonce[sizeof rec.nonce - 1] = 0;
                const bool mine = nonce.empty() ? rec.written_at >= started - 120 : nonce == rec.nonce;
                if (mine) break;  // otherwise: a stale record, rank 0 will replace it
            }
            if (tries > 6000) throw hnh::Error(HNH_E_COMM, "timed out waiting for this launch's NCCL unique id file");
            usleep(10000);
        }
        std::memcpy(id, rec.id, sizeof id);
    }
    hnh::Comm::init_nccl(rank, size, id);
    hnh::Comm::world()->barrier();  // every rank has read the record
    if (rank == 0) unlink(path);
}

void hnh_compat_allreduce_sum_f64(double *buf, size_t count, hnh::Comm &comm) {
    cudaPointerAttributes attr;
    const bool device_side = hnh::Runtime::get().has_device() && cudaPointerGetAttributes(&attr, buf) == cudaSuccess &&
                             (attr.type == cudaMemoryTypeDevice || attr.type == cudaMemoryTypeManaged);
    if (!device_side) {
        cudaGetLastError();
        comm.host_allreduce_sum_f64(buf, count);
        return;
    }
    cudaStream_t s = hnh::Runtime::get().compute_stream();
    comm.allreduce_sum_f64(buf, count, s);
    hnh::cuda_check(cudaStreamSynchronize(s), "MPI_Allreduce stand-in");
}

void hnh_world_finalize() {
    if (hnh::Runtime::get().has_device()) hnh::Runtime::get().sync_all();
    hnh::Comm::finalize();
}
