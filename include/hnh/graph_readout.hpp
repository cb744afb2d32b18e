// hnh/graph_readout.hpp -- graph-level prediction: a readout that pools the model's output rows into one row per
// graph, an optional linear head, and graph train and evaluate steps for every GraphModel.  torch is the definition:
//     P = torch.zeros(G, r).index_add_(0, batch, H)                                      "sum"  (global_add_pool)
//     P = sum / n_g  (0 for an empty graph)                                              "mean" (global_mean_pool)
//     P = torch.zeros(G, r).scatter_reduce(0, batch, H, "amax", include_self = False)    "max"  (0 for an empty graph)
//     logits = torch.nn.Linear(r, C)(P)  with the head, P itself without (then r must equal C)
//     loss = F.cross_entropy(logits, y, ignore_index = <any negative>, reduction = "mean") over the labelled graphs
// H is the model's output buffer (buffers.back(), localArows x r on every rank) and batch[u] the graph of this rank's
// row u: in [0, G), or negative for a row in no graph (padding rows, global row >= M, must be negative).  n_g counts a
// graph's rows over all ranks.  The gradient of max goes in equal shares to the C_g,k rows of all ranks attaining the
// maximum, with -0.0 and +0.0 tying: the convention of Distributed_Sparse::maxAggregate (torch's autograd differs at a
// maximum of exactly 0, where it also counts the zero it started from).
//
// Placement.  The readout builds, once and on the host, this rank's segments (segment g: the rows of graph g, in
// ascending order) and their chunk plan, and uploads them (hnh_segment_pool_f64).  pool: the segment kernel reads each
// local row once and writes this rank's partial P (G x r), then one world all-reduce of G r doubles; mean divides by
// n_g, whose G counts came from one all-reduce when the readout was built.  max: the kernel writes the local (max,
// count) pairs; an all-reduce max of P, the counts of ranks whose maximum is not the global one set to 0
// (hnh_segment_max_count_merge_f64), an all-reduce sum of the counts, and P = 0 where no row attains it (an empty
// graph).  The head, the cross-entropy over the G rows and their gradients then run identically on every rank on the
// identical all-reduced P: they need no communication, and the head's gradients no all-reduce.  poolBackward writes
// dH_u = w_u dP_g(u) on every local row (hnh_segment_pool_grad_f64) without communication; the model's backwardPass
// all-reduces the model's gradients as always.  Memory: G r doubles for P (and G r for the counts of max), the
// segments (8 bytes per local row in a graph, 16 per graph), 4 bytes per local row, G r more for the local maxima of
// max at p > 1, and, when some graph has more than HNH_SEGMENT_CHUNK local rows, a workspace of r (2r for max) doubles
// per chunk of the plan: the workspace is indexed by chunk, so it holds one row for every graph's chunks (at least G),
// not for the long graphs' chunks alone.
//
// The head's parameters are one vector [W; b], (r + 1) x C: W = Linear.weight.T in the first r rows, b = Linear.bias
// the last; zero after construction, like the models' parameters.  The optimizer steps the model's spans, then the
// head's.
#pragma once
#include <cstdint>
#include <string>
#include <vector>

#include "hnh/comm.h"
#include "hnh/distributed_sparse.h"
#include "hnh/model.hpp"
#include "hnh/training.hpp"
#include "hnh/world_allreduce.hpp"
#include "hnh_b200.h"

namespace hnh {

namespace detail {
// x[0] = a refusal flag, then (part, part^2) for the 16-bit parts of each value, summed over the world in one host
// all-reduce.  True when the ranks' values agree: p sum(v^2) == (sum v)^2 holds only when every v is the same.
inline std::vector<double> agreement_sums(bool refused, const std::vector<uint64_t> &values) {
    std::vector<double> x{refused ? 1.0 : 0.0};
    for (uint64_t v : values)
        for (int shift = 0; shift < 64; shift += 16) {
            const double part = (double)((v >> shift) & 0xffff);
            x.push_back(part);
            x.push_back(part * part);
        }
    Comm::world()->host_allreduce_sum_f64(x.data(), x.size());
    return x;
}
inline bool agree(const std::vector<double> &x) {
    const double p = (double)Comm::world()->size();
    for (size_t i = 1; i + 1 < x.size(); i += 2)
        if (x[i] * x[i] != p * x[i + 1]) return false;
    return true;
}
}  // namespace detail

class GraphReadout {
public:
    enum Pool { kSum, kMean, kMax };

    const GraphModel *net;  // the model the readout was made for
    int64_t rows;           // this rank's output rows (localArows)
    int64_t num_graphs;     // G
    Pool pool_kind = kSum;
    int width;        // r, the model's output width
    int num_classes;  // C, the logits' width (r without a head)
    bool head;
    VectorXd params, grads;      // [W; b] of the head, (r + 1) x C; empty without a head.  grads after a graph step
    DenseMatrix pooled, counts;  // P (G x r) of the last pool, and the tie counts of max

    // Collective.  num_classes = 0: no head, and the logits are P, r wide (GraphLabels of another class count are
    // refused).  Refuses with HNH_E_INVALID on every rank, before any launch: a layout where check_full_rows fails, a
    // batch that is not localArows long, G < 1, G or G r >= 2^31, an id >= G or an id on a padding row on any rank, G
    // differing between ranks, an unknown pool and num_classes < 0.
    GraphReadout(GraphModel &model, const int64_t *batch, int64_t n, int64_t G, const string &pool, int classes)
        : net(&model), rows(model.d_ops->localArows), num_graphs(G), width((int)model.buffers.back().cols()),
          num_classes(classes > 0 ? classes : width), head(classes > 0) {
        const Distributed_Sparse &d = *model.d_ops;
        d.check_full_rows("GraphReadout");
        const int64_t top = d.aSubmatrices.empty() ? 0 : d.aSubmatrices[0].topRow;
        std::string why;
        if (pool == "sum") pool_kind = kSum;
        else if (pool == "mean") pool_kind = kMean;
        else if (pool == "max") pool_kind = kMax;
        else why = "unknown pool \"" + pool + "\" (sum, mean or max)";
        const int64_t limit = int64_t(1) << 31;
        if (!why.empty()) {
            // the pool's refusal stands
        } else if (classes < 0) {
            why = "num_classes must be >= 0 (0: no head)";
        } else if (G < 1 || G >= limit || G * width >= limit) {
            why = std::to_string(G) + " graphs of width " + std::to_string(width) + ": G must be >= 1 and G, G r below 2^31";
        } else if (n != rows) {
            why = "a batch of " + std::to_string(n) + " ids for " + std::to_string(rows) + " output rows";
        } else if (n > 0 && !batch) {
            why = "null batch";
        }
        for (int64_t i = 0; why.empty() && i < n; i++) {
            if (batch[i] >= G) why = "graph id " + std::to_string(batch[i]) + " of row " + std::to_string(i) + " is not below " + std::to_string(G);
            else if (batch[i] >= 0 && top + i >= (int64_t)d.M) why = "padding row " + std::to_string(i) + " has a graph id";
        }
        const std::vector<double> x = detail::agreement_sums(!why.empty(), {(uint64_t)(G >= 0 && G < limit ? G : 0)});
        if (!why.empty()) throw Error(HNH_E_INVALID, "GraphReadout: " + why);
        if (x[0] != 0.0) throw Error(HNH_E_INVALID, "GraphReadout: another rank's batch was refused");
        if (!detail::agree(x)) throw Error(HNH_E_INVALID, "GraphReadout: the graph count differs between ranks");
        build_segments(batch, n);
        if (head) params = VectorXd::Constant(((int64_t)width + 1) * classes, 0.0);
    }

    // The head's parameters by name: "weight" (r x C, Linear.weight.T) and "bias" (C x 1)
    ParamRef param(const string &name) {
        if (!head) throw Error(HNH_E_INVALID, "GraphReadout: no head (num_classes = 0), so no parameter \"" + name + "\"");
        const bool has_grads = grads.size() == params.size();
        if (name == "weight") return {params.data(), has_grads ? grads.data() : nullptr, width, num_classes};
        if (name == "bias") {
            const int64_t off = (int64_t)width * num_classes;
            return {params.data() + off, has_grads ? grads.data() + off : nullptr, num_classes, 1};
        }
        throw Error(HNH_E_INVALID, "GraphReadout: no parameter \"" + name + "\" (weight or bias)");
    }
    std::vector<ParamSpan> parameters() {
        if (!head) return {};
        return {{params.data(), grads.size() == params.size() ? grads.data() : nullptr, params.size()}};
    }

    // P = pool(H) over all ranks into `pooled` (and `counts` for max).  Collective.
    const DenseMatrix &pool(const DenseMatrix &H) {
        if (H.rows() != rows || H.cols() != width)
            throw Error(HNH_E_INVALID, "GraphReadout::pool: H is " + std::to_string(H.rows()) + " x " + std::to_string(H.cols()) +
                                           ", the model's output " + std::to_string(rows) + " x " + std::to_string(width));
        cudaStream_t s = stream();
        const int64_t n = num_graphs * width;
        pooled.resize(num_graphs, width);
        if (pool_kind == kMax) counts.resize(num_graphs, width);
        abi_check(hnh_segment_pool_f64(seg_start_.data(), seg_rows_.data(), chunk_first_.data(), chunk_seg_.data(), num_graphs, chunks_,
                                       H.data(), width, width, pooled.data(), width, pool_kind == kMax ? counts.data() : nullptr,
                                       width, workspace_.data(), workspace_.size(), s),
                  "segment_pool");
        if (pool_kind == kMax) {
            if (Comm::world()->size() > 1) {
                local_max_ = pooled;  // reuses its storage after the first pool
                allreduce_world_max(pooled.data(), n);
                abi_check(hnh_segment_max_count_merge_f64(counts.data(), local_max_.data(), pooled.data(), n, s), "segment_max_count_merge");
                allreduce_world(counts);
            }
            abi_check(hnh_max_aggregate_finish_f64(pooled.data(), counts.data(), n, s), "max_aggregate_finish");
        } else {
            allreduce_world(pooled);
            if (pool_kind == kMean)
                abi_check(hnh_row_axpy_f64(pooled.data(), nullptr, 1.0, inv_size_.data(), pooled.data(), num_graphs, width, s), "row_axpy");
        }
        return pooled;
    }

    // dH = dL/dH given dP = dL/dP (G x r, the same on every rank) for the H of the last pool.  No communication.
    void poolBackward(const DenseMatrix &H, const DenseMatrix &dP, DenseMatrix &dH) {
        if (H.rows() != rows || H.cols() != width || dP.rows() != num_graphs || dP.cols() != width)
            throw Error(HNH_E_INVALID, "GraphReadout::poolBackward: H must be " + std::to_string(rows) + " x " + std::to_string(width) +
                                           " and dP " + std::to_string(num_graphs) + " x " + std::to_string(width));
        const bool mx = pool_kind == kMax;
        if (mx && (pooled.rows() != num_graphs || counts.rows() != num_graphs))
            throw Error(HNH_E_INVALID, "GraphReadout::poolBackward: the max readout needs a pool first");
        dH.resize(rows, width);
        abi_check(hnh_segment_pool_grad_f64(row_graph_.data(), rows, num_graphs, dP.data(), width,
                                            pool_kind == kMean ? inv_size_.data() : nullptr, mx ? H.data() : nullptr, width,
                                            mx ? pooled.data() : nullptr, width, mx ? counts.data() : nullptr, width, width, dH.data(),
                                            width, stream()),
                  "segment_pool_grad");
    }

    // the logits of the last pool: P W + b with the head, P itself without; lastLogits() gives them again
    const DenseMatrix &lastLogits() const { return head ? logits_ : pooled; }
    const DenseMatrix &logits() {
        if (!head) return pooled;
        logits_ = pooled * weight();
        abi_check(hnh_row_bias_add_f64(logits_.data(), params.data() + (int64_t)width * num_classes, num_graphs, num_classes, stream()),
                  "row_bias_add");
        return logits_;
    }
    // given dlogits: the head's gradients into grads, and dP (G x r).  The same on every rank; no communication.
    void headBackward(const DenseMatrix &dlogits, DenseMatrix &dP) {
        if (!head) {
            dP = dlogits;
            return;
        }
        if (grads.size() != params.size()) grads = VectorXd(params.size());
        DenseMatrix::view(grads.data(), width, num_classes).setTransposeTimes(pooled, dlogits);
        DenseMatrix::view(grads.data() + (int64_t)width * num_classes, 1, num_classes)
            .setTransposeTimes(DenseMatrix::Constant(num_graphs, 1, 1.0), dlogits);
        dP.resize(num_graphs, width);
        dP.setTimesTranspose(dlogits, weight(), false);
    }

private:
    int64_t chunks_ = 0;
    DeviceBuffer<int64_t> seg_start_, seg_rows_, chunk_first_;
    DeviceBuffer<int32_t> chunk_seg_, row_graph_;
    DeviceBuffer<char> workspace_;
    VectorXd inv_size_;  // 1 / n_g (0 for an empty graph), for mean
    DenseMatrix logits_;
    DenseMatrix local_max_;  // this rank's maxima before the all-reduce (max at p > 1)

    static cudaStream_t stream() { return Runtime::get().compute_stream(); }
    DenseMatrix weight() { return DenseMatrix::view(params.data(), width, num_classes); }

    // this rank's segments, their chunk plan and the rows' graphs, uploaded; n_g over all ranks for mean (collective)
    void build_segments(const int64_t *batch, int64_t n) {
        const int64_t G = num_graphs;
        std::vector<int64_t> start((size_t)G + 1, 0), first((size_t)G + 1, 0);
        std::vector<int32_t> row_graph((size_t)n);
        for (int64_t i = 0; i < n; i++) {
            row_graph[(size_t)i] = batch[i] >= 0 ? (int32_t)batch[i] : -1;
            if (batch[i] >= 0) start[(size_t)batch[i] + 1]++;
        }
        std::vector<double> sizes((size_t)G);
        for (int64_t g = 0; g < G; g++) sizes[(size_t)g] = (double)start[(size_t)g + 1];
        for (int64_t g = 0; g < G; g++) start[(size_t)g + 1] += start[(size_t)g];
        std::vector<int64_t> seg_rows((size_t)start[(size_t)G]), fill(start.begin(), start.end() - 1);
        for (int64_t i = 0; i < n; i++)
            if (batch[i] >= 0) seg_rows[(size_t)fill[(size_t)batch[i]]++] = i;  // ascending rows within each segment
        std::vector<int32_t> chunk_seg;
        for (int64_t g = 0; g < G; g++) {
            const int64_t len = start[(size_t)g + 1] - start[(size_t)g];
            const int64_t c = len > 0 ? (len + HNH_SEGMENT_CHUNK - 1) / HNH_SEGMENT_CHUNK : 1;
            first[(size_t)g + 1] = first[(size_t)g] + c;
            chunk_seg.insert(chunk_seg.end(), (size_t)c, (int32_t)g);
        }
        chunks_ = first[(size_t)G];
        cudaStream_t s = stream();
        seg_start_.upload(start.data(), start.size(), s);
        seg_rows_.upload(seg_rows.data(), seg_rows.size(), s);
        chunk_first_.upload(first.data(), first.size(), s);
        chunk_seg_.upload(chunk_seg.data(), chunk_seg.size(), s);
        row_graph_.upload(row_graph.data(), row_graph.size(), s);
        if (chunks_ > G) workspace_.resize((size_t)hnh_segment_pool_workspace_bytes(chunks_, width, pool_kind == kMax));
        if (pool_kind == kMean) {
            Comm::world()->host_allreduce_sum_f64(sizes.data(), sizes.size());
            for (double &v : sizes) v = v > 0.0 ? 1.0 / v : 0.0;
            inv_size_ = VectorXd::from_host(sizes.data(), G);
        }
        cuda_check(cudaStreamSynchronize(s), "GraphReadout upload");
    }
};

// The labels of a readout's G graphs, in [0, C) or negative for "ignored", identical on every rank (train, validation
// and test splits are negative labels).  Collective: one host all-reduce of (a refusal flag, a 64-bit hash of the
// labels); labels that are not G long, hold a label >= C, or differ between ranks are refused with HNH_E_INVALID on
// every rank, before any launch.
class GraphLabels {
public:
    const GraphReadout *readout;
    int64_t labelled;  // the graphs with a label
    double inv_count;  // 1 / labelled, 0 when no graph is labelled

    GraphLabels(const GraphReadout &ro, const int32_t *host, int64_t n, int classes) : readout(&ro) {
        std::string why;
        int64_t count = 0;
        uint64_t hash = 1469598103934665603ull;  // FNV-1a over the labels' bytes
        if (n != ro.num_graphs)
            why = std::to_string(n) + " labels for " + std::to_string(ro.num_graphs) + " graphs";
        else if (classes != ro.num_classes)
            why = "labels of " + std::to_string(classes) + " classes for logits " + std::to_string(ro.num_classes) + " wide";
        else if (n > 0 && !host)
            why = "null labels";
        for (int64_t i = 0; why.empty() && i < n; i++) {
            if (host[i] >= classes) why = "label " + std::to_string(host[i]) + " of graph " + std::to_string(i) + " is not below num_classes";
            count += host[i] >= 0;
            for (int b = 0; b < 4; b++) hash = (hash ^ (((uint32_t)host[i] >> (8 * b)) & 0xff)) * 1099511628211ull;
        }
        const std::vector<double> x = detail::agreement_sums(!why.empty(), {why.empty() ? hash : 0});
        if (!why.empty()) throw Error(HNH_E_INVALID, "GraphLabels: " + why);
        if (x[0] != 0.0) throw Error(HNH_E_INVALID, "GraphLabels: another rank's labels were refused");
        if (!detail::agree(x)) throw Error(HNH_E_INVALID, "GraphLabels: the labels differ between ranks");
        labelled = count;
        inv_count = count > 0 ? 1.0 / (double)count : 0.0;
        cudaStream_t s = Runtime::get().compute_stream();
        labels_.upload(host, (size_t)n, s);
        cuda_check(cudaStreamSynchronize(s), "GraphLabels upload");
    }
    const int32_t *data() const { return labels_.data(); }

private:
    DeviceBuffer<int32_t> labels_;
};

namespace detail {
// the model's spans, then the head's
inline std::vector<ParamSpan> graphSpans(GraphModel &net, GraphReadout &ro) {
    std::vector<ParamSpan> s = net.parameters();
    for (const ParamSpan &p : ro.parameters()) s.push_back(p);
    return s;
}
// refusals every rank decides alike, before any launch
inline void check_graph(GraphModel &net, GraphReadout &ro, const GraphLabels &labels, const AdamW *opt, const char *who) {
    if (ro.net != &net) throw Error(HNH_E_INVALID, string(who) + ": the readout was made for another model");
    if (labels.readout != &ro) throw Error(HNH_E_INVALID, string(who) + ": the labels were made for another readout");
    if (opt) opt->check_spans(graphSpans(net, ro));
}
// pool, head and cross-entropy of H against the labels: sums (device, 2 doubles) = (loss sum, correct) -- the same on
// every rank, so no all-reduce; with dH, the gradient of the mean loss through the head and the pool.
inline void graphLoss(GraphReadout &ro, const DenseMatrix &H, const GraphLabels &labels, DenseMatrix *dH, double *sums) {
    ro.pool(H);
    const DenseMatrix &logits = ro.logits();
    DenseMatrix dlogits(logits.rows(), logits.cols());
    const int64_t n = logits.rows(), ws_bytes = hnh_cross_entropy_workspace_bytes(n);
    if (ws_bytes < 0) abi_check((int)ws_bytes, "cross_entropy");
    DeviceBuffer<char> ws((size_t)ws_bytes);
    abi_check(hnh_cross_entropy_f64(dlogits.data(), sums, logits.data(), labels.data(), n, logits.cols(), logits.cols(), labels.inv_count,
                                    ws.data(), (size_t)ws_bytes, Runtime::get().compute_stream()),
              "cross_entropy");
    if (!dH) return;
    DenseMatrix dP;
    ro.headBackward(dlogits, dP);
    ro.poolBackward(H, dP, *dH);
}
}  // namespace detail

// One graph-classification step: forward(dropout, seed) -- models without dropout refuse dropout != 0 --, pool, head,
// cross-entropy over the labelled graphs, their gradients, backwardPass(dH), clip and AdamW over the model's spans and
// then the head's.  TrainResult's `labelled` is the labelled graph count.  Collective.  Refuses, on every rank before
// any launch, a readout made for another model, labels made for another readout, an optimizer of other parameters and
// a layout the model refuses.  Leaves the activations stale.
inline TrainResult graphTrainStep(GraphModel &net, GraphReadout &ro, const GraphLabels &labels, AdamW &opt, double dropout, uint64_t seed) {
    detail::check_graph(net, ro, labels, &opt, "graphTrainStep");
    net.check_trainable();
    net.forward(dropout, seed);
    return detail::finishStep(
        net, labels.labelled, opt, [&](DenseMatrix &dH, double *sums) { detail::graphLoss(ro, net.buffers.back(), labels, &dH, sums); },
        [&](const DenseMatrix &dH) { net.backwardPass(dH); }, [&] { return detail::graphSpans(net, ro); });
}

// A forward pass without dropout, the readout and the loss without gradients: (mean loss, correct, labelled graphs)
// as a LinkResult's (loss, correct, count), the same on every rank, and host_logits (nullable: G x C doubles, row-major) the logits.  Collective.
inline LinkResult graphEvaluate(GraphModel &net, GraphReadout &ro, const GraphLabels &labels, double *host_logits) {
    detail::check_graph(net, ro, labels, nullptr, "graphEvaluate");
    net.forward(0.0, 0);
    VectorXd sums(2);
    detail::graphLoss(ro, net.buffers.back(), labels, nullptr, sums.data());
    double h[2];
    cudaStream_t s = Runtime::get().compute_stream();
    cuda_check(cudaMemcpyAsync(h, sums.data(), sizeof h, cudaMemcpyDeviceToHost, s), "graph results");
    if (host_logits) ro.lastLogits().copy_to_host(host_logits);
    cuda_check(cudaStreamSynchronize(s), "graph results");
    return {labels.labelled > 0 ? h[0] / (double)labels.labelled : 0.0, (int64_t)h[1], labels.labelled};
}

}  // namespace hnh
