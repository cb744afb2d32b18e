// hnh/rgcn.hpp -- R-GCN: layers of PyG's RGCNConv(in, out, num_relations = R, num_bases = B, aggr, root_weight = True,
// bias = True), without decomposition or with basis decomposition, with the mean or sum aggregator, forward and backward,
// with the weight gradients summed over all ranks.
//
// The relation of a stored entry (u, v) of S is its stored value (Distributed_Sparse::relationalAggregate), an integer
// in [0, R); the constructor refuses any other value on any rank.  Layer l has input width f and output width r.  With
// X the layer input and N_rho(u) the stored entries of row u of relation rho on all ranks (duplicates counting):
//     A[u, rho]  = sum_{v in N_rho(u)} X_v                    relationalAggregate (f wide per relation, 0 when empty)
//     Ab[u, rho] = A[u, rho] / |N_rho(u)|   (mean)   or   A[u, rho]   (sum)         hnh_window_scale_f64 for the mean
//     Y = [Ab_0 | ... | Ab_{R-1}] [W_0; ...; W_{R-1}] + X W_root + b                  2 GEMMs (K = R f and f), a bias row
//     X_{l+1} = ReLU(Y) for every layer but the last, which outputs Y (as GraphSAGE)
// The counts |N_rho(u)| come once per model from relationalAggregate of a ones column (R doubles per row).
//
// Backward of layer l, given G = dL/d X_{l+1}:
//     dY = G where X_{l+1} > 0 (G itself for the last layer)
//     [dW_0; ...; dW_{R-1}] = Ab^T dY,  db = 1^T dY,  dW_root = X^T dY              3 TN GEMMs, each straight into the
//                                                                                   gradient vector
//     dAb = dY [W_0; ...]^T,  dA = dAb / |N_rho(u)| (mean),  dX = dY W_root^T + relationalAggregateBackward(dA)
// then one sum all-reduce of the layer's gradients (allreduce_world).  The bias gradient is a product with a ones
// column kept by the model, so Ab is used in place (no [Ab 1] copy of an R f wide matrix).  The forward keeps Ab of
// every layer (R f doubles per row per layer), so the backward runs no forward sparse pass; the backward allocates dA
// (R f doubles per row) for one layer at a time.
//
// Parameters of a layer live in one device vector, in the order of its gradients: [W_0; ...; W_{R-1}; b]
// ((R f + 1) x r), then W_root (f x r).  All are zero after construction.  A PyG RGCNConv state dict maps onto them as
// weight.reshape(R f, r) -> "weight", bias -> "bias", root -> "root", with no transpose.
//
// With B >= 1 bases, W_rho = sum_b comp[rho, b] V_b (PyG's num_bases = B), and the aggregation writes one window per
// basis instead of one per relation (Distributed_Sparse::basisAggregate), so memory and traffic depend on B, not R:
//     H[u, b] = sum_{(u, v) stored} w(u, rho_uv) comp[rho_uv, b] X_v,   w = 1 / |N_rho(u)| (mean) or 1 (sum)
//     Y = [H_0 | ... | H_{B-1}] [V_0; ...; V_{B-1}] + X W_root + b
// The mean's weights 1 / |N_rho(u)| (0 where the count is 0) are computed once per model from the same counts.  The
// forward keeps H (B f doubles per row per layer).  The backward computes dV = H^T dY, db and dW_root as above,
// dH = dY [V_0; ...]^T, and dX = dY W_root^T + basisAggregateBackward(dH), which also gives dcomp already summed over
// all ranks; the all-reduce of the layer's other gradients follows.  The parameter vector is [V_0; ...; V_{B-1}; b]
// ((B f + 1) x r), W_root (f x r), then comp (R x B), so that the all-reduce covers the prefix before comp.  PyG's
// RGCNConv(num_bases = B) maps onto it as weight.reshape(B f, r) -> "weight", comp -> "comp", bias, root.
//
// Defined where Distributed_Sparse::check_full_rows passes (every rank holds full-width rows and the A and B layouts
// coincide); elsewhere the constructor throws HNH_E_INVALID on every rank before any launch.
#pragma once
#include <string>
#include <utility>
#include <vector>

#include "hnh/distributed_sparse.h"
#include "hnh/model.hpp"
#include "hnh/world_allreduce.hpp"
#include "hnh_b200.h"

class RGCNLayer {
public:
    int input_features;
    int output_features;

    VectorXd params;  // the layout above; zero after construction
    VectorXd grads;   // the same layout: dL/d params after RGCN::backwardPass (same on every rank)

    RGCNLayer(int in_width, int out_width) : input_features(in_width), output_features(out_width) {}
    int64_t bias_offset(int R) const { return (int64_t)R * input_features * output_features; }
    int64_t root_offset(int R) const { return ((int64_t)R * input_features + 1) * output_features; }
    int64_t param_count(int R) const { return (((int64_t)R + 1) * input_features + 1) * output_features; }
};

class RGCN : public GraphModel {
public:
    enum Aggregation { kMean, kSum };

    vector<RGCNLayer> layers;
    const int num_relations;
    const Aggregation aggr;
    vector<DenseMatrix> aggregated;  // Ab (localArows x R f), or H with bases (localArows x B f), of every layer
    const int num_bases;  // B >= 1: basis decomposition; 0: none

    // aggr: "mean" or "sum".  Collective: checks every stored value of S (Distributed_Sparse::relationCheck).
    RGCN(vector<RGCNLayer> &l_input, Distributed_Sparse *ops, int relations, const string &aggregation)
        : RGCN(l_input, ops, relations, aggregation, 0) {}

    // The same with `bases` bases (0: without decomposition, as above).
    RGCN(vector<RGCNLayer> &l_input, Distributed_Sparse *ops, int relations, const string &aggregation, int bases)
        : GraphModel(ops, "RGCN"), layers(l_input), num_relations(relations), aggr(parse(aggregation)), num_bases(bases) {
        vector<std::pair<int, int>> widths;
        for (const RGCNLayer &l : layers) widths.emplace_back(l.input_features, l.output_features);
        const vector<LayerWidths> chain = check_layers(widths, num_relations, num_bases);
        d_ops->check_full_rows("RGCN");
        refuse("RGCN", rows_problem());
        d_ops->relationCheck(num_relations);
        allocate_buffers(chain);
        for (RGCNLayer &layer : layers) layer.params = VectorXd::Constant(param_count(layer), 0.0);
        ones = DenseMatrix::Constant(d_ops->localArows, 1, 1.0);
        if (aggr == kMean) {
            // |N_rho(u)| over all ranks: the relational sum of a ones column
            DenseMatrix one_col = DenseMatrix::Constant(d_ops->localBrows, 1, 1.0);
            counts.resize(d_ops->localArows, num_relations);
            d_ops->relationalAggregate(one_col, counts, num_relations);
            if (num_bases > 0) {
                // basisAggregate's scale: 1 / |N_rho(u)|, 0 where the count is 0
                DenseMatrix inv = DenseMatrix::Constant(d_ops->localArows, num_relations, 1.0);
                hnh::abi_check(hnh_max_aggregate_grad_scale_f64(inv.data(), inv.data(), counts.data(), inv.size(), stream()),
                               "max_aggregate_grad_scale");
                counts.take(inv);
            }
        }
    }

    // the checks that need no device, on the (input, output) widths of the layers: a relation count >= 1, a basis count
    // >= 0, positive widths that chain, R f < 2^31, and with bases B f and R B < 2^31.  Returns the widths as
    // allocate_buffers takes them.
    static vector<LayerWidths> check_layers(const vector<std::pair<int, int>> &widths, int num_relations, int num_bases = 0) {
        if (widths.empty()) throw hnh::Error(HNH_E_INVALID, "RGCN: no layers");
        if (num_relations < 1) throw hnh::Error(HNH_E_INVALID, "RGCN: the relation count must be positive");
        if (num_bases < 0) throw hnh::Error(HNH_E_INVALID, "RGCN: the basis count must not be negative");
        if ((int64_t)num_relations * num_bases > INT32_MAX) throw hnh::Error(HNH_E_INVALID, "RGCN: R B must be below 2^31");
        vector<LayerWidths> chain;
        for (const auto &[f, r] : widths) chain.push_back({f, r, f > 0 && r > 0});
        refuse("RGCN", layer_chain_problem(chain, [&](size_t i) -> string {
                   const int64_t f = chain[i].in;
                   if (num_bases == 0 && num_relations * f > INT32_MAX) return "layer " + std::to_string(i) + ": R f must be below 2^31";
                   if (num_bases * f > INT32_MAX) return "layer " + std::to_string(i) + ": B f must be below 2^31";
                   return "";
               }));
        return chain;
    }

    static Aggregation parse(const string &a) {
        if (a == "mean") return kMean;
        if (a == "sum") return kSum;
        throw hnh::Error(HNH_E_INVALID, "RGCN: unknown aggregation \"" + a + "\" (mean or sum)");
    }

    // the aggregation's windows per row: B with bases, else R
    int windows() const { return num_bases > 0 ? num_bases : num_relations; }
    // where comp (R x B) starts in a layer's params and grads, and their length
    int64_t comp_offset(const RGCNLayer &l) const { return l.param_count(windows()); }
    int64_t param_count(const RGCNLayer &l) const { return comp_offset(l) + (int64_t)num_relations * num_bases; }

    // [W_0; ...; W_{R-1}] (R f x r) or [V_0; ...; V_{B-1}] (B f x r), b (1 x r), W_root (f x r) and comp (R x B) of a
    // layer's params or grads, as views
    DenseMatrix weight(VectorXd &v, const RGCNLayer &l) const {
        return DenseMatrix::view(v.data(), (int64_t)windows() * l.input_features, l.output_features);
    }
    DenseMatrix bias(VectorXd &v, const RGCNLayer &l) const {
        return DenseMatrix::view(v.data() + l.bias_offset(windows()), 1, l.output_features);
    }
    DenseMatrix root(VectorXd &v, const RGCNLayer &l) const {
        return DenseMatrix::view(v.data() + l.root_offset(windows()), l.input_features, l.output_features);
    }
    DenseMatrix comp(VectorXd &v, const RGCNLayer &l) const {
        return DenseMatrix::view(v.data() + comp_offset(l), num_relations, num_bases);
    }

    // Each layer's params with its grads, one span per layer
    std::vector<ParamSpan> parameters() override { return layer_spans(layers); }

    // By name (the layout above): "weight" (R f x r, or B f x r with bases), "bias" (r x 1), "root" (f x r), and with
    // bases "comp" (R x B)
    ParamRef param(int layer, const string &name) override {
        if (layer < 0 || layer >= (int)layers.size()) throw hnh::Error(HNH_E_INVALID, "RGCN: no such layer");
        RGCNLayer &l = layers[(size_t)layer];
        const int64_t f = l.input_features, r = l.output_features, K = windows();
        if (name == "weight") return slice(l.params, l.grads, 0, K * f, r);
        if (name == "bias") return slice(l.params, l.grads, l.bias_offset(windows()), r, 1);
        if (name == "root") return slice(l.params, l.grads, l.root_offset(windows()), f, r);
        if (name == "comp" && num_bases > 0) return slice(l.params, l.grads, comp_offset(l), num_relations, num_bases);
        if (num_bases > 0) throw hnh::Error(HNH_E_INVALID, "RGCN: no parameter \"" + name + "\" (weight, comp, bias or root)");
        throw hnh::Error(HNH_E_INVALID, "RGCN: no parameter \"" + name + "\" (weight, bias or root)");
    }

    // Collective.
    void forwardPass() {
        d_ops->check_full_rows("RGCN::forwardPass");
        aggregated.resize(layers.size());
        for (size_t i = 0; i < layers.size(); i++) {
            RGCNLayer &layer = layers[i];
            DenseMatrix &X = buffers[i], &A = aggregated[i];
            const int64_t f = X.cols();
            A.resize(d_ops->localArows, f * windows());
            if (num_bases > 0) {
                d_ops->basisAggregate(X, A, comp(layer.params, layer), num_relations, aggr == kMean ? &counts : nullptr);
            } else {
                d_ops->relationalAggregate(X, A, num_relations);
                if (aggr == kMean) window_scale(A, (int)f);
            }
            DenseMatrix Y = A * weight(layer.params, layer);
            hnh::abi_check(hnh_row_bias_add_f64(Y.data(), bias(layer.params, layer).data(), Y.rows(), Y.cols(), stream()), "row_bias_add");
            Y += X * root(layer.params, layer);
            set_layer_output(i, Y);
        }
        activations_current = true;
    }
    void forward(double dropout, uint64_t) override {
        refuse_dropout(dropout);
        forwardPass();
    }

    // output_grad = dL/d buffers.back() (this rank's rows).  Leaves dL/d params in layers[i].grads (summed over all
    // ranks) and dL/d buffers[0] in input_grad.  Collective.
    void backwardPass(const DenseMatrix &output_grad) override {
        d_ops->check_full_rows("RGCN::backwardPass");
        check_backward("RGCN::backwardPass", "the parameters or the input", output_grad);
        backward_layers(output_grad, [&](int i, const DenseMatrix &G, DenseMatrix &dX) { backwardLayer(i, G, dX); });
    }

private:
    DenseMatrix ones;    // localArows x 1 of 1.0: the bias gradient is its product with dY
    DenseMatrix counts;  // mean: |N_rho(u)| (localArows x R); with bases 1 / |N_rho(u)|, 0 where the count is 0

    // M[u, rho f + k] /= |N_rho(u)| (0 where the count is 0)
    void window_scale(DenseMatrix &M, int f) {
        hnh::abi_check(hnh_window_scale_f64(M.data(), M.cols(), counts.data(), counts.cols(), M.rows(), f, num_relations, stream()),
                       "window_scale");
    }

    // layer i: G = dL/d buffers[i + 1]; writes layers[i].grads and dX = dL/d buffers[i]
    void backwardLayer(int i, const DenseMatrix &G, DenseMatrix &dX) {
        RGCNLayer &layer = layers[(size_t)i];
        DenseMatrix &X = buffers[(size_t)i], &A = aggregated[(size_t)i];
        const int64_t f = X.cols();
        if (layer.grads.size() != layer.params.size()) layer.grads = VectorXd(layer.params.size());
        DenseMatrix dY_relu;
        const DenseMatrix &dY = relu_grad_unless_last(i, G, dY_relu);
        weight(layer.grads, layer).setTransposeTimes(A, dY);
        bias(layer.grads, layer).setTransposeTimes(ones, dY);
        root(layer.grads, layer).setTransposeTimes(X, dY);
        dX.setTimesTranspose(dY, root(layer.params, layer), false);
        if (num_bases > 0) {
            DenseMatrix dH, dcomp = comp(layer.grads, layer);
            dH.setTimesTranspose(dY, weight(layer.params, layer), false);
            d_ops->basisAggregateBackward(dH, X, dX, comp(layer.params, layer), dcomp, num_relations,
                                          aggr == kMean ? &counts : nullptr, true);
            allreduce_world(layer.grads.data(), comp_offset(layer));  // dcomp is summed over the ranks already
            return;
        }
        {
            DenseMatrix dA;
            dA.setTimesTranspose(dY, weight(layer.params, layer), false);
            if (aggr == kMean) window_scale(dA, (int)f);
            d_ops->relationalAggregateBackward(dA, dX, num_relations, true);
        }
        allreduce_world(layer.grads);
    }
};
