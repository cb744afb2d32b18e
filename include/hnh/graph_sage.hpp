// hnh/graph_sage.hpp -- GraphSAGE: layers of PyG's SAGEConv(aggr, root_weight = True, project = False, normalize =
// False) with the mean, sum or max aggregator, forward and backward, with the weight gradients summed over all ranks.
//
// Layer l has input width f and output width r.  With X the layer input (rows of the nodes) and u an S-row:
//     A = aggr(X):  sum   A_u = sum_v X_v                 over the stored entries (u, v) of S on all ranks, duplicates
//                   mean  A_u = sum_v X_v / deg_u         counting; deg_u the stored-entry count of row u
//                   max   A_u,k = max_v X_v,k             (Distributed_Sparse::maxAggregate, which also gives the tie
//                                                          counts C)
//                   A_u = 0 for a row without entries, as in PyG
//     Y = A W_l + b_l + X W_r                              2 GEMMs (hnh_dgemm_f64) and a bias row
//     X_{l+1} = ReLU(Y) for every layer but the last, which outputs Y (as the graph transformer)
// sum and mean are one spmmA at width f with per-entry weights: 1 for sum, 1 / deg_u for mean, in both value orders.
// The degrees come once per model from Distributed_Sparse::edgeSums of a ones vector, and the weights from
// additiveScores(s = 1 / deg, t = 0): LeakyReLU(s_u + 0) = s_u exactly, since s_u > 0.
//
// Backward of layer l, given G = dL/d X_{l+1}:
//     dY = G where X_{l+1} > 0 (G itself for the last layer)
//     [dW_l; db_l] = [A 1]^T dY,  dW_r = X^T dY                       2 TN GEMMs (the bias gradient is the product
//                                                                     with the ones column, in the GEMM's fixed order)
//     dA = dY W_l^T,  dX = dY W_r^T + aggr^T(dA)                       2 NT GEMMs; aggr^T: spmmB with the B-order
//                                                                     weights (sum, mean), maxAggregateBackward adding
//                                                                     into dX (max)
// then one sum all-reduce of the layer's gradients (allreduce_world).  The forward keeps A of every layer (and C for
// max: f, or 2f, doubles per row per layer), so the backward runs no forward sparse pass.
//
// Parameters of a layer live in one device vector, in the order of its gradients: [W_l; b_l] ((f + 1) x r: W_l in the
// first f rows, b_l the last), then W_r (f x r).  All are zero after construction.  Weights are stored input-major: a
// PyG SAGEConv state dict maps onto them as lin_l.weight.T, lin_l.bias and lin_r.weight.T.
//
// Defined where Distributed_Sparse::check_full_rows passes (every rank holds full-width rows and the A and B layouts
// coincide); elsewhere the constructor throws HNH_E_INVALID on every rank before any launch.
#pragma once
#include <string>
#include <vector>

#include "hnh/distributed_sparse.h"
#include "hnh/model.hpp"
#include "hnh/world_allreduce.hpp"
#include "hnh_b200.h"

class GraphSAGELayer {
public:
    int input_features;
    int output_features;

    VectorXd params;  // the layout above; zero after construction
    VectorXd grads;   // the same layout: dL/d params after GraphSAGE::backwardPass (same on every rank)

    GraphSAGELayer(int in_width, int out_width) : input_features(in_width), output_features(out_width) {}
    int64_t root_offset() const { return ((int64_t)input_features + 1) * output_features; }
    int64_t param_count() const { return (2 * (int64_t)input_features + 1) * output_features; }
};

class GraphSAGE : public GraphModel {
public:
    enum Aggregation { kMean, kSum, kMax };

    vector<GraphSAGELayer> layers;
    const Aggregation aggr;
    vector<DenseMatrix> aggregated, counts;  // A (and C for max) of every layer from the last forward pass

    // aggr: "mean", "sum" or "max"
    GraphSAGE(vector<GraphSAGELayer> &l_input, Distributed_Sparse *ops, const string &aggregation)
        : GraphModel(ops, "GraphSAGE"), layers(l_input), aggr(parse(aggregation)) {
        d_ops->check_full_rows("GraphSAGE");
        if (layers.empty()) throw hnh::Error(HNH_E_INVALID, "GraphSAGE: no layers");
        vector<LayerWidths> widths;
        for (const GraphSAGELayer &l : layers)
            widths.push_back({l.input_features, l.output_features, l.input_features > 0 && l.output_features > 0});
        refuse("GraphSAGE", layer_chain_problem(widths));
        refuse("GraphSAGE", rows_problem());
        allocate_buffers(widths);
        for (GraphSAGELayer &layer : layers) layer.params = VectorXd::Constant(layer.param_count(), 0.0);
        if (aggr == kSum) {
            weights_A = d_ops->like_S_values(1.0);
            weights_B = d_ops->like_ST_values(1.0);
        } else if (aggr == kMean) {
            // deg_u over all ranks, then 1 / deg_u per entry in both orders (rows without entries have no entry to weigh)
            VectorXd ones = d_ops->like_S_values(1.0), deg(d_ops->M), col_sums(d_ops->N);
            d_ops->edgeSums(ones, deg, col_sums);
            VectorXd inv(d_ops->M), t = VectorXd::Constant(d_ops->N, 0.0);
            inv.setQuotient(VectorXd::Constant(d_ops->M, 1.0), 0.0, deg, 0.0);
            weights_A = d_ops->like_S_values(0.0);
            weights_B = d_ops->like_ST_values(0.0);
            d_ops->additiveScores(inv, t, weights_A, k_sddmmA, 0.0, false);
            d_ops->additiveScores(inv, t, weights_B, k_sddmmB, 0.0, false);
        }
    }

    static Aggregation parse(const string &a) {
        if (a == "mean") return kMean;
        if (a == "sum") return kSum;
        if (a == "max") return kMax;
        throw hnh::Error(HNH_E_INVALID, "GraphSAGE: unknown aggregation \"" + a + "\" (mean, sum or max)");
    }

    // [W_l; b_l] of a layer ((f + 1) x r, or f x r without the bias row), its bias, and W_r, as views
    static DenseMatrix neigh(VectorXd &v, const GraphSAGELayer &l, bool with_bias) {
        return DenseMatrix::view(v.data(), l.input_features + (with_bias ? 1 : 0), l.output_features);
    }
    static double *neigh_bias(VectorXd &v, const GraphSAGELayer &l) {
        return v.data() + (int64_t)l.input_features * l.output_features;
    }
    static DenseMatrix root(VectorXd &v, const GraphSAGELayer &l) {
        return DenseMatrix::view(v.data() + l.root_offset(), l.input_features, l.output_features);
    }

    // Each layer's params with its grads, one span per layer
    std::vector<ParamSpan> parameters() override { return layer_spans(layers); }

    // By name (the layout above): "neigh" (W_l, f x r), "neigh_bias" (b_l, r x 1), "root" (W_r, f x r)
    ParamRef param(int layer, const string &name) override {
        if (layer < 0 || layer >= (int)layers.size()) throw hnh::Error(HNH_E_INVALID, "GraphSAGE: no such layer");
        GraphSAGELayer &l = layers[(size_t)layer];
        const int64_t f = l.input_features, r = l.output_features;
        if (name == "neigh") return slice(l.params, l.grads, 0, f, r);
        if (name == "neigh_bias") return slice(l.params, l.grads, f * r, r, 1);
        if (name == "root") return slice(l.params, l.grads, l.root_offset(), f, r);
        throw hnh::Error(HNH_E_INVALID, "GraphSAGE: no parameter \"" + name + "\" (neigh, neigh_bias or root)");
    }

    // Collective.
    void forwardPass() {
        d_ops->check_full_rows("GraphSAGE::forwardPass");
        aggregated.resize(layers.size());
        if (aggr == kMax) counts.resize(layers.size());
        for (size_t i = 0; i < layers.size(); i++) {
            GraphSAGELayer &layer = layers[i];
            DenseMatrix &X = buffers[i];
            aggregate(i, X);
            DenseMatrix Y = aggregated[i] * neigh(layer.params, layer, false);
            hnh::abi_check(hnh_row_bias_add_f64(Y.data(), neigh_bias(layer.params, layer), Y.rows(), Y.cols(), stream()), "row_bias_add");
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
        d_ops->check_full_rows("GraphSAGE::backwardPass");
        check_backward("GraphSAGE::backwardPass", "the parameters or the input", output_grad);
        backward_layers(output_grad, [&](int i, const DenseMatrix &G, DenseMatrix &dX) { backwardLayer(i, G, dX); });
    }

private:
    VectorXd weights_A, weights_B;  // sum / mean: the aggregation weight of every entry in the A and B orders

    // aggregated[i] (and counts[i]) = aggr(X)
    void aggregate(size_t i, DenseMatrix &X) {
        const int64_t f = X.cols();
        DenseMatrix &A = aggregated[i];
        A.resize(d_ops->localArows, f);
        if (aggr == kMax) {
            counts[i].resize(d_ops->localArows, f);
            d_ops->maxAggregate(X, A, counts[i]);
        } else {
            d_ops->setRValue((int)f);
            d_ops->spmmA(A, X, weights_A);
        }
    }

    // layer i: G = dL/d buffers[i + 1]; writes layers[i].grads and dX = dL/d buffers[i]
    void backwardLayer(int i, const DenseMatrix &G, DenseMatrix &dX) {
        GraphSAGELayer &layer = layers[(size_t)i];
        DenseMatrix &X = buffers[(size_t)i], &A = aggregated[(size_t)i];
        const int64_t f = X.cols();
        if (layer.grads.size() != layer.params.size()) layer.grads = VectorXd(layer.params.size());
        DenseMatrix dY_relu;
        const DenseMatrix &dY = relu_grad_unless_last(i, G, dY_relu);
        {
            DenseMatrix Aa = with_ones(A);
            neigh(layer.grads, layer, true).setTransposeTimes(Aa, dY);
        }
        root(layer.grads, layer).setTransposeTimes(X, dY);
        DenseMatrix dA;
        dA.setTimesTranspose(dY, neigh(layer.params, layer, false), false);
        dX.setTimesTranspose(dY, root(layer.params, layer), false);
        if (aggr == kMax) {
            d_ops->maxAggregateBackward(X, A, counts[(size_t)i], dA, dX, true);
        } else {
            d_ops->setRValue((int)f);
            DenseMatrix back = d_ops->like_B_matrix(0.0);
            d_ops->spmmB(dA, back, weights_B);
            dX += back;
        }
        allreduce_world(layer.grads);
    }
};
