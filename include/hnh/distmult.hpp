// hnh/distmult.hpp -- relation-aware link prediction (knowledge-graph completion): a DistMult decoder over relation-typed
// target pairs, and relational link train and evaluate steps for every GraphModel.  PyG's examples/rgcn_link_pred.py is
// the definition:
//     s = (z[src] * rel_emb[edge_type] * z[dst]).sum(-1)
//     loss = F.binary_cross_entropy_with_logits(cat([s_pos, s_neg]), cat([ones, zeros]))      (the mean over all pairs)
// z is the model's output buffer H, rel_emb the decoder's relation table D (R x r).  The pairs are the stored entries of
// two target matrices T_pos and T_neg in algorithm objects of the model's layout (as LinkTargets, hnh/training.hpp),
// whose stored values are the pairs' relations; each is scored by Distributed_Sparse::distmultLoss, the positives with
// target 1 and the negatives with target 0, both with inv_count = 1 / (n_pos + n_neg), the second call accumulating
// into the first's gradients.  The step is trainStep's: forward, the loss, backwardPass(dH), clip and AdamW over the
// model's spans and then the decoder's.  Communication per step beyond the model's own: per target matrix one world
// all-reduce of 2 doubles (the loss sums) and, in a train step, one of R r doubles (dD); the gradients are then the
// same on every rank.
#pragma once
#include <cstdint>
#include <memory>
#include <string>
#include <vector>

#include "hnh/distributed_sparse.h"
#include "hnh/model.hpp"
#include "hnh/training.hpp"
#include "hnh_b200.h"

namespace hnh {

// The relation table D of a model's DistMult decoder: R x r, zero after construction, with its gradient after a
// relational train step.  `model` is the model's algorithm object and r the width of its output buffer.
class DistMultDecoder {
public:
    const Distributed_Sparse *model;
    int num_relations, width;
    DenseMatrix rel, grad;  // D (R x r) and dL/dD, the same on every rank

    DistMultDecoder(const Distributed_Sparse &model_ops, int R, int r) : model(&model_ops), num_relations(R), width(r) {
        if (R < 1 || r < 1 || (int64_t)R * r >= (int64_t(1) << 31))
            throw Error(HNH_E_INVALID, "DistMultDecoder: " + std::to_string(R) + " relations of width " + std::to_string(r) +
                                           ": both must be positive and R r below 2^31");
        rel = DenseMatrix::Constant(R, r, 0.0);
    }
    // "rel": the relation table, R x r (the example's rel_emb, no transpose)
    ParamRef param(const string &name) {
        if (name != "rel") throw Error(HNH_E_INVALID, "DistMultDecoder: no parameter \"" + name + "\" (rel)");
        return {rel.data(), grad.size() == rel.size() ? grad.data() : nullptr, num_relations, width};
    }
    std::vector<ParamSpan> parameters() { return {{rel.data(), grad.size() == rel.size() ? grad.data() : nullptr, rel.size()}}; }
};

// The relational link targets of a model: T_pos and T_neg, each in its own algorithm object of the model's layout (see
// LinkTargets), whose stored values are relations in [0, R): the positive pairs (target 1) and the negative ones (target
// 0; T_neg may have no entry).  Duplicates count, each under its own relation.  Fresh negatives every epoch are a new
// T_neg and a new targets object.  Collective: refuses, with HNH_E_INVALID on every rank, a T of another layout, a T
// that is not square, R < 1 and a stored value that is no relation on any rank (Distributed_Sparse::relationCheck: one
// world all-reduce of 2 doubles per matrix).  Builds each matrix's grouping by relation (relationPlan) once, for the
// gradient of D.  The three algorithm objects must outlive this one, and T's stored values must stay as they are.
class RelationalLinkTargets {
public:
    const Distributed_Sparse *model;
    Distributed_Sparse *pos, *neg;
    int num_relations;
    int64_t count_pos, count_neg, count;  // stored entries over all ranks; count = count_pos + count_neg
    double inv_count;                     // 1 / count, 0 when there is no pair anywhere

    RelationalLinkTargets(const Distributed_Sparse &model_ops, Distributed_Sparse &T_pos, Distributed_Sparse &T_neg, int R)
        : model(&model_ops), pos(&T_pos), neg(&T_neg), num_relations(R) {
        for (const Distributed_Sparse *t : {&T_pos, &T_neg}) {
            const string why = detail::link_layout_mismatch(model_ops, *t);
            if (!why.empty()) throw Error(HNH_E_INVALID, string("RelationalLinkTargets: ") + (t == &T_pos ? "T_pos: " : "T_neg: ") + why);
        }
        if (R < 1) throw Error(HNH_E_INVALID, "RelationalLinkTargets: the relation count must be positive, got " + std::to_string(R));
        count_pos = T_pos.relationCheck(R);
        count_neg = T_neg.relationCheck(R);
        count = count_pos + count_neg;
        inv_count = count > 0 ? 1.0 / (double)count : 0.0;
        plan_pos_ = T_pos.relationPlan(R);
        plan_neg_ = T_neg.relationPlan(R);
    }

    // sums (device, 2 doubles) = (loss sum, correct count) over both matrices and all ranks; dH (nullable, resized to H's
    // shape) and dD (nullable, resized to D's) = the gradients of the mean loss; scores_pos / scores_neg (nullable,
    // resized to the A-order length of T_pos / T_neg) = s in the order of each matrix's like_S_values
    void loss(DenseMatrix &H, const DistMultDecoder &dec, DenseMatrix *dH, DenseMatrix *dD, VectorXd *scores_pos, VectorXd *scores_neg,
              double *sums) const {
        if (dH) dH->resize(H.rows(), H.cols());
        if (dD) dD->resize(dec.num_relations, dec.width);
        if (scores_pos) scores_pos->resize(pos->num_S_values());
        if (scores_neg) scores_neg->resize(neg->num_S_values());
        cuda_check(cudaMemsetAsync(sums, 0, 2 * sizeof(double), Runtime::get().compute_stream()), "relational link sums");
        pos->distmultLoss(H, H, dec.rel, num_relations, 1.0, inv_count, dH, dH, dD, scores_pos, sums, false, plan_pos_.get());
        neg->distmultLoss(H, H, dec.rel, num_relations, 0.0, inv_count, dH, dH, dD, scores_neg, sums, true, plan_neg_.get());
    }

private:
    std::unique_ptr<RelationPlan> plan_pos_, plan_neg_;
};

namespace detail {
// the model's spans, then the decoder's
inline std::vector<ParamSpan> relationalSpans(GraphModel &net, DistMultDecoder &dec) {
    std::vector<ParamSpan> s = net.parameters();
    for (const ParamSpan &p : dec.parameters()) s.push_back(p);
    return s;
}
// refusals every rank decides alike, before any launch
inline void check_relational(GraphModel &net, const RelationalLinkTargets &targets, DistMultDecoder &dec, const AdamW *opt,
                             const char *who) {
    if (targets.model != net.d_ops) throw Error(HNH_E_INVALID, string(who) + ": the targets were made for another model's algorithm object");
    if (dec.model != net.d_ops) throw Error(HNH_E_INVALID, string(who) + ": the decoder was made for another model's algorithm object");
    if (dec.num_relations != targets.num_relations)
        throw Error(HNH_E_INVALID, string(who) + ": the decoder has " + std::to_string(dec.num_relations) + " relations, the targets " +
                                       std::to_string(targets.num_relations));
    if (dec.width != net.buffers.back().cols())
        throw Error(HNH_E_INVALID, string(who) + ": the decoder is " + std::to_string(dec.width) + " wide, the model's output " +
                                       std::to_string(net.buffers.back().cols()));
    if (opt) opt->check_spans(relationalSpans(net, dec));
}
}  // namespace detail

// One relational link-prediction step: forward(dropout, seed), the mean binary cross-entropy of the DistMult scores of
// both target matrices (RelationalLinkTargets::loss) with dH and dD, backwardPass(dH), clip and AdamW over the model's
// spans and then the decoder's.  TrainResult's `labelled` is the pair count.  Collective.  Refuses, on every rank before
// any launch, targets or a decoder made for another model's algorithm object, a decoder whose relation count differs
// from the targets' or whose width differs from the model's output, an optimizer of other parameters and a layout the
// model refuses.  Leaves the activations stale.
inline TrainResult relationalLinkTrainStep(GraphModel &net, const RelationalLinkTargets &targets, DistMultDecoder &dec, AdamW &opt,
                                           double dropout, uint64_t seed) {
    detail::check_relational(net, targets, dec, &opt, "relationalLinkTrainStep");
    net.check_trainable();
    net.forward(dropout, seed);
    return detail::finishStep(
        net, targets.count, opt, [&](DenseMatrix &g, double *sums) { targets.loss(net.buffers.back(), dec, &g, &dec.grad, nullptr, nullptr, sums); },
        [&](const DenseMatrix &g) { net.backwardPass(g); }, [&] { return detail::relationalSpans(net, dec); });
}

// A forward pass without dropout and the loss without gradients: (mean loss, correct, pair count) over all ranks, and
// scores_pos / scores_neg (nullable, resized) = s in the A order of T_pos / T_neg (entryCoordinates(k_sddmmA) of each
// gives their node pairs), for a ranking metric.  Collective; refuses as relationalLinkTrainStep.
inline LinkResult relationalLinkEvaluate(GraphModel &net, const RelationalLinkTargets &targets, DistMultDecoder &dec, VectorXd *scores_pos,
                                         VectorXd *scores_neg) {
    detail::check_relational(net, targets, dec, nullptr, "relationalLinkEvaluate");
    net.forward(0.0, 0);
    VectorXd sums(2);
    targets.loss(net.buffers.back(), dec, nullptr, nullptr, scores_pos, scores_neg, sums.data());
    double h[2];
    cudaStream_t s = Runtime::get().compute_stream();
    cuda_check(cudaMemcpyAsync(h, sums.data(), sizeof h, cudaMemcpyDeviceToHost, s), "relational link results");
    cuda_check(cudaStreamSynchronize(s), "relational link results");
    return {targets.count > 0 ? h[0] / (double)targets.count : 0.0, (int64_t)h[1], targets.count};
}

}  // namespace hnh
