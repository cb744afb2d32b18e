// hnh/training.hpp -- training the graph models on the device: a masked cross-entropy loss for node
// classification, gradient-norm clipping and AdamW, and one collective train step.  torch is the definition:
//     loss = F.cross_entropy(logits, labels, ignore_index = <any negative>, reduction = "mean") over the labelled rows of
//            all ranks (0 and a zero gradient when no row is labelled anywhere; torch gives NaN there)
//     torch.nn.utils.clip_grad_norm_(parameters, max_grad_norm)      only with max_grad_norm set; the norm is always taken
//     torch.optim.AdamW(parameters, lr, betas, eps, weight_decay, amsgrad = False, foreach = False), one group, t from 1
// trainStep = forward, cross-entropy of the model's output buffer (its rows and width: the logits as the model computes
// them; GAT's last layer keeps its ReLU), backwardPass, clip, AdamW.  Communication per step beyond the backward's own
// all-reduces: one world all-reduce of 2 doubles (the loss sum and the correct count); the gradients are identical on
// every rank after the backward, so the norm and the update need none.  Host traffic: 4 doubles down per step.
//
// Link prediction (LinkTargets, linkTrainStep, linkEvaluate, at the end) shares the step: its loss is the binary
// cross-entropy of dot-product scores over the entries of a target matrix (Distributed_Sparse::linkLoss).
//
// One step serves every GraphModel (hnh/model.hpp): GAT, GraphTransformer, GraphSAGE and RGCN.  Parameters are device
// spans read afresh at every step (set_weight may replace a matrix's storage), in a fixed order:
//     GraphTransformer, GraphSAGE, RGCN: each layer's params vector with its grads, one span per layer;
//     GAT: every (layer, head) weight with its gradient, then a1 and a2 of every layer with theirs.  Where an attention
//     kind does not read a1 or a2 their gradient is 0, and AdamW's decoupled decay alone moves them.
#pragma once
#include <cmath>
#include <cstring>
#include <string>
#include <vector>

#include "hnh/15D_dense_shift.hpp"
#include "hnh/comm.h"
#include "hnh/model.hpp"
#include "hnh/world_allreduce.hpp"
#include "hnh_b200.h"

namespace hnh {

// The labels of one rank: one per row of the model's output buffer (`rows`, this rank's localArows), in [0,
// num_classes) or negative for "ignored" (padding rows and unlabelled nodes must be negative).  Collective: one world
// all-reduce of (a refusal flag, the labelled count), so a bad label on one rank is refused with HNH_E_INVALID on every
// rank, before any launch.
class NodeLabels {
public:
    int64_t rows;
    int num_classes;
    int64_t labelled;  // over all ranks
    double inv_count;  // 1 / labelled, 0 when no row is labelled anywhere

    NodeLabels(const int32_t *host, int64_t n, int64_t expected_rows, int classes) : rows(n), num_classes(classes) {
        std::string why;
        int64_t count = 0;
        if (n != expected_rows)
            why = std::to_string(n) + " labels for " + std::to_string(expected_rows) + " output rows";
        else if (classes <= 0)
            why = "num_classes must be positive";
        else if (n > 0 && !host)
            why = "null labels";
        for (int64_t i = 0; why.empty() && i < n; i++) {
            if (host[i] >= classes) why = "label " + std::to_string(host[i]) + " of row " + std::to_string(i) + " is not below num_classes";
            count += host[i] >= 0;
        }
        double x[2] = {why.empty() ? 0.0 : 1.0, (double)count};
        Comm::world()->host_allreduce_sum_f64(x, 2);
        if (!why.empty()) throw Error(HNH_E_INVALID, "NodeLabels: " + why);
        if (x[0] != 0.0) throw Error(HNH_E_INVALID, "NodeLabels: another rank's labels were refused");
        labelled = (int64_t)x[1];
        inv_count = labelled > 0 ? 1.0 / (double)labelled : 0.0;
        cudaStream_t s = Runtime::get().compute_stream();
        labels_.upload(host, (size_t)n, s);
        cuda_check(cudaStreamSynchronize(s), "NodeLabels upload");
    }
    const int32_t *data() const { return labels_.data(); }

private:
    DeviceBuffer<int32_t> labels_;
};

// torch.optim.AdamW with one parameter group, and the clipping of clip_grad_norm_ (max_grad_norm > 0; 0 is off).  The
// moments m and v are allocated on the first step, by position in the span list; a later list of another length or
// other sizes is refused.
class AdamW {
public:
    double lr, beta1, beta2, eps, weight_decay, max_grad_norm;
    int64_t t = 0;  // steps taken

    AdamW(double lr_, double b1, double b2, double eps_, double wd, double max_norm)
        : lr(lr_), beta1(b1), beta2(b2), eps(eps_), weight_decay(wd), max_grad_norm(max_norm) {
        check_lr(lr_);
        if (!(b1 >= 0.0 && b1 < 1.0) || !(b2 >= 0.0 && b2 < 1.0)) throw Error(HNH_E_INVALID, "AdamW: the betas must lie in [0, 1)");
        if (!(eps_ > 0.0) || !std::isfinite(eps_)) throw Error(HNH_E_INVALID, "AdamW: eps must be finite and > 0");
        if (!(wd >= 0.0) || !std::isfinite(wd)) throw Error(HNH_E_INVALID, "AdamW: weight_decay must be finite and >= 0");
        if (!(max_norm >= 0.0)) throw Error(HNH_E_INVALID, "AdamW: max_grad_norm must be >= 0 (0: no clipping)");
    }
    void set_lr(double v) {
        check_lr(v);
        lr = v;
    }

    // Throws HNH_E_INVALID unless the spans fit the moments (or there are none yet).  Decided from sizes only: every
    // rank decides alike.
    void check_spans(const std::vector<ParamSpan> &spans) const {
        if (m_.empty()) return;
        bool same = spans.size() == m_.size();
        for (size_t i = 0; same && i < spans.size(); i++) same = spans[i].n == m_[i].size();
        if (!same) throw Error(HNH_E_INVALID, "AdamW: the parameters are not those of the optimizer's first step");
    }

    // One step on the spans with their gradients.  stats (device, 2 doubles) receives (total gradient norm, clip
    // coefficient); the coefficient is applied only with max_grad_norm > 0.  Stream-ordered, no host synchronisation.
    void step(const std::vector<ParamSpan> &spans, double *stats) {
        check_spans(spans);
        for (const ParamSpan &p : spans)
            if (!p.grad && p.n > 0) throw Error(HNH_E_INVALID, "AdamW: a parameter has no gradient");
        cudaStream_t s = Runtime::get().compute_stream();
        if (m_.empty())
            for (const ParamSpan &p : spans) {
                m_.push_back(VectorXd::Constant(p.n, 0.0));
                v_.push_back(VectorXd::Constant(p.n, 0.0));
            }
        VectorXd sq((int64_t)spans.size());
        for (size_t i = 0; i < spans.size(); i++) abi_check(hnh_squared_norm_f64(sq.data() + i, spans[i].grad, spans[i].n, s), "squared_norm");
        const bool clip = max_grad_norm > 0.0;
        abi_check(hnh_clip_coef_f64(stats, sq.data(), sq.size(), clip ? max_grad_norm : INFINITY, s), "clip_coef");
        t++;
        const double bc1 = 1.0 - std::pow(beta1, (double)t), bc2 = 1.0 - std::pow(beta2, (double)t);
        for (size_t i = 0; i < spans.size(); i++)
            abi_check(hnh_adamw_f64(spans[i].param, m_[i].data(), v_[i].data(), spans[i].grad, spans[i].n, lr, beta1, beta2, eps,
                                    weight_decay, bc1, bc2, clip ? stats + 1 : nullptr, s),
                      "adamw");
    }

private:
    std::vector<VectorXd> m_, v_;
    static void check_lr(double v) {
        if (!(v >= 0.0) || !std::isfinite(v)) throw Error(HNH_E_INVALID, "AdamW: lr must be finite and >= 0");
    }
};

struct TrainResult {
    double loss;  // mean over the labelled rows of all ranks
    int64_t correct, labelled;
    double grad_norm;  // before clipping
};

// Cross-entropy of logits against labels into dlogits (resized to the logits' shape): stats[0] = the loss sum and
// stats[1] = the correct count over all ranks (device).  One kernel, then one world all-reduce of the 2 doubles.
inline void crossEntropy(const DenseMatrix &logits, const NodeLabels &labels, DenseMatrix &dlogits, double *stats) {
    if (labels.rows != logits.rows() || labels.num_classes != logits.cols())
        throw Error(HNH_E_INVALID, "crossEntropy: labels for " + std::to_string(labels.rows) + " rows of " +
                                       std::to_string(labels.num_classes) + " classes, logits " + std::to_string(logits.rows()) +
                                       " x " + std::to_string(logits.cols()));
    dlogits.resize(logits.rows(), logits.cols());
    const int64_t n = logits.rows(), ws_bytes = hnh_cross_entropy_workspace_bytes(n);
    if (ws_bytes < 0) abi_check((int)ws_bytes, "cross_entropy");
    DeviceBuffer<char> ws((size_t)ws_bytes);
    abi_check(hnh_cross_entropy_f64(dlogits.data(), stats, logits.data(), labels.data(), n, logits.cols(), logits.cols(),
                                    labels.inv_count, ws.data(), (size_t)ws_bytes, Runtime::get().compute_stream()),
              "cross_entropy");
    allreduce_world(stats, 2);
}

namespace detail {
// refusals every rank decides alike, before any launch
inline void check_train(const DenseMatrix &out, const NodeLabels &labels, const AdamW &opt, const std::vector<ParamSpan> &spans) {
    if (labels.rows != out.rows())
        throw Error(HNH_E_INVALID, "trainStep: labels for " + std::to_string(labels.rows) + " rows, the output has " +
                                       std::to_string(out.rows()));
    if (labels.num_classes != out.cols())
        throw Error(HNH_E_INVALID, "trainStep: labels for " + std::to_string(labels.num_classes) + " classes, the output is " +
                                       std::to_string(out.cols()) + " wide");
    opt.check_spans(spans);
}
// the loss (by the caller's `loss`: the output buffer's gradient and the device sums (loss sum, correct) over all
// ranks), backward (by the caller's `backward`), clip and AdamW on the span list `spans()` returns after the backward
// (a first backward pass allocates the gradients); then the 4 scalars to the host.  count: the denominator of the
// mean loss (labelled rows, link targets or labelled graphs).
template <class Model, class Loss, class Backward, class Spans>
TrainResult finishStep(Model &net, int64_t count, AdamW &opt, Loss loss, Backward backward, Spans spans) {
    VectorXd stats(4);  // loss sum, correct, total norm, clip coefficient
    DenseMatrix dlogits;
    loss(dlogits, stats.data());
    backward(dlogits);
    dlogits = DenseMatrix();
    opt.step(spans(), stats.data() + 2);
    net.activations_current = false;
    double h[4];
    cudaStream_t s = Runtime::get().compute_stream();
    cuda_check(cudaMemcpyAsync(h, stats.data(), sizeof h, cudaMemcpyDeviceToHost, s), "train step results");
    cuda_check(cudaStreamSynchronize(s), "train step results");
    return {count > 0 ? h[0] / (double)count : 0.0, (int64_t)h[1], count, h[2]};
}
}  // namespace detail

// One training step (see the top of this file): forward(dropout, seed) -- models without dropout refuse dropout != 0 --,
// cross-entropy, backward, clip and AdamW.  Collective.  Refuses, on every rank before any launch, labels of another row
// count or class count, an optimizer of other parameters and a layout the model refuses.  Leaves the activations stale.
inline TrainResult trainStep(GraphModel &net, const NodeLabels &labels, AdamW &opt, double dropout, uint64_t seed) {
    detail::check_train(net.buffers.back(), labels, opt, net.parameters());
    net.check_trainable();
    net.forward(dropout, seed);
    return detail::finishStep(
        net, labels.labelled, opt, [&](DenseMatrix &g, double *sums) { crossEntropy(net.buffers.back(), labels, g, sums); },
        [&](const DenseMatrix &g) { net.backwardPass(g); }, [&] { return net.parameters(); });
}

// ---- link prediction ----------------------------------------------------------------------------------------------
namespace detail {
inline int fusion(const Distributed_Sparse &d) {
    const Sparse15D_Dense_Shift *ds = dynamic_cast<const Sparse15D_Dense_Shift *>(&d);
    return ds ? ds->fusionApproach : 0;
}
// why a target matrix T's layout is not the model's ("" when it is): link targets (LinkTargets, and
// RelationalLinkTargets in hnh/distmult.hpp) live in an algorithm object of the model's layout.  Global quantities
// only, so every rank decides alike.
inline string link_layout_mismatch(const Distributed_Sparse &m, const Distributed_Sparse &t) {
    auto dims = [](const Distributed_Sparse &d) {
        return std::to_string(d.p) + ", c = " + std::to_string(d.c) + ", " + std::to_string(d.M) + " x " + std::to_string(d.N) +
               ", local rows " + std::to_string(d.localArows) + " / " + std::to_string(d.localBrows);
    };
    if (t.algorithm_name != m.algorithm_name || fusion(t) != fusion(m) || t.p != m.p || t.c != m.c || t.M != m.M || t.N != m.N ||
        t.localArows != m.localArows || t.localBrows != m.localBrows)
        return "T's layout (" + t.algorithm_name + ", fusion " + std::to_string(fusion(t)) + ", p = " + dims(t) +
               ") is not the model's (" + m.algorithm_name + ", fusion " + std::to_string(fusion(m)) + ", p = " + dims(m) + ")";
    if (t.M != t.N) return "T is " + std::to_string(t.M) + " x " + std::to_string(t.N) + "; link targets are square";
    return "";
}
}  // namespace detail

// The link targets of a model: T, a square sparse matrix over the model's nodes in its own algorithm object of the
// model's layout (algorithm, fusion, p, c, M = N = the model's S dimensions, localArows, localBrows), so the dense row
// partition is the model's.  T's stored values are the targets y_uv in [0, 1] (1 a positive pair, 0 a negative one,
// soft targets allowed; duplicates count), as Distributed_Sparse::linkLoss reads them.  The loss is
//     F.binary_cross_entropy_with_logits(s, y, reduction = "mean") over the stored entries of T on all ranks,
// s_uv = <H_u, H_v> with H the model's output buffer (0 and a zero gradient when T has no entry anywhere), and the
// correct count the entries with (s > 0) == (y > 0.5).  GAT's last layer keeps its ReLU (the reference's formula), so
// its scores are >= 0: the graph transformer is the model for link prediction.  Collective: refuses, with
// HNH_E_INVALID on every rank, a T of another layout, a T that is not square and a target outside [0, 1] on any rank
// (a device check, then one world all-reduce of 2 doubles).  Both algorithm objects must outlive this one.
class LinkTargets {
public:
    const Distributed_Sparse *model;
    Distributed_Sparse *T;
    int64_t count;     // stored entries of T over all ranks
    double inv_count;  // 1 / count, 0 when T has no entry anywhere

    LinkTargets(const Distributed_Sparse &model_ops, Distributed_Sparse &T_ops) : model(&model_ops), T(&T_ops) {
        const string why = detail::link_layout_mismatch(model_ops, T_ops);
        if (!why.empty()) throw Error(HNH_E_INVALID, "LinkTargets: " + why);
        count = T_ops.linkTargetCount();
        inv_count = count > 0 ? 1.0 / (double)count : 0.0;
    }
    // sums (device, 2 doubles) = (loss sum, correct count) over all ranks; dH (nullable, resized to H's shape) = dL/dH
    // of the mean loss; scores (nullable, resized to T's A-order length) = s in the order of T's like_S_values
    void loss(DenseMatrix &H, DenseMatrix *dH, VectorXd *scores, double *sums) const {
        if (dH) dH->resize(H.rows(), H.cols());
        if (scores) scores->resize(T->num_S_values());
        T->linkLoss(H, H, inv_count, dH, dH, scores, sums);
    }
};

struct LinkResult {
    double loss;  // mean over the stored entries of T on all ranks
    int64_t correct, count;
};

namespace detail {
// refusals every rank decides alike, before any launch
inline void check_link(const Distributed_Sparse *ops, const LinkTargets &targets, const AdamW *opt, const std::vector<ParamSpan> &spans,
                       const char *who) {
    if (ops != targets.model) throw Error(HNH_E_INVALID, string(who) + ": the link targets were made for another model's algorithm object");
    if (opt) opt->check_spans(spans);
}
inline LinkResult linkResult(DenseMatrix &H, const LinkTargets &targets, VectorXd *scores) {
    VectorXd sums(2);
    targets.loss(H, nullptr, scores, sums.data());
    double h[2];
    cudaStream_t s = Runtime::get().compute_stream();
    cuda_check(cudaMemcpyAsync(h, sums.data(), sizeof h, cudaMemcpyDeviceToHost, s), "link results");
    cuda_check(cudaStreamSynchronize(s), "link results");
    return {targets.count > 0 ? h[0] / (double)targets.count : 0.0, (int64_t)h[1], targets.count};
}
}  // namespace detail

// One link-prediction training step: forward(dropout, seed), the mean binary cross-entropy of the scores of T's entries
// (LinkTargets) with its gradient dH from Distributed_Sparse::linkLoss, backwardPass(dH), clip and AdamW, as trainStep.
// TrainResult's `labelled` is the entry count of T.  Collective.  Refuses, on every rank before any launch, targets made
// for another model's algorithm object, an optimizer of other parameters and a layout the model refuses.  Leaves the
// activations stale.  GAT's last layer keeps its ReLU, so its scores are >= 0; the other models' last layers have none.
inline TrainResult linkTrainStep(GraphModel &net, const LinkTargets &targets, AdamW &opt, double dropout, uint64_t seed) {
    detail::check_link(net.d_ops, targets, &opt, net.parameters(), "linkTrainStep");
    net.check_trainable();
    net.forward(dropout, seed);
    return detail::finishStep(
        net, targets.count, opt, [&](DenseMatrix &g, double *sums) { targets.loss(net.buffers.back(), &g, nullptr, sums); },
        [&](const DenseMatrix &g) { net.backwardPass(g); }, [&] { return net.parameters(); });
}

// A forward pass without dropout and the link loss without gradients: (mean loss, correct, count) over all ranks, and
// scores (nullable, resized) = s in the order of T's like_S_values (Distributed_Sparse::entryCoordinates(k_sddmmA) of
// T gives their node pairs).  Collective.
inline LinkResult linkEvaluate(GraphModel &net, const LinkTargets &targets, VectorXd *scores) {
    detail::check_link(net.d_ops, targets, nullptr, {}, "linkEvaluate");
    net.forward(0.0, 0);
    return detail::linkResult(net.buffers.back(), targets, scores);
}

}  // namespace hnh
