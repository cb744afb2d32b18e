// hnh/gin.hpp -- GIN and GINE: layers of PyG's GINConv(nn, eps, train_eps) (Xu et al., 2019) or, with edge features
// (edge_dim > 0), GINEConv(nn, eps, train_eps, edge_dim) (Hu et al., 2020), with nn = Sequential(Linear(f, h), ReLU(),
// Linear(h, r)), forward and backward, with the weight gradients summed over all ranks.
//
// Layer l is an (f, h, r) triple.  With X the layer input (rows of the nodes) and the stored entries i = (u, v) of S on
// all ranks (duplicates count; rows without entries aggregate to 0):
//     E_A = attr_A W_e + b_e,  E_B = attr_B W_e + b_e     (edge_dim > 0: GINEConv's lin, on the attributes of both orders)
//     M_u = sum_i X_v                                      GIN: spmmA with weights 1 (GraphSAGE-sum's aggregation)
//     M_u = sum_i ReLU(X_v + E_i)                          GINE: Distributed_Sparse::edgeReluAggregate
//     H = M + (1 + eps) X                                  (hnh_gin_combine_f64: eps is read on the device)
//     Z = ReLU(H W1 + b1),  Y = Z W2 + b2                  2 GEMMs and bias rows
//     X_{l+1} = ReLU(Y) for every layer but the last, which outputs Y (as the other models, so link prediction works)
//
// Backward of layer l, given G = dL/d X_{l+1}:
//     dY = G where X_{l+1} > 0 (G itself for the last layer)
//     [dW2; db2] = [Z 1]^T dY,  dP = dY W2^T where Z > 0,  [dW1; db1] = [H 1]^T dP,  dH = dP W1^T
//                                                          (TN GEMMs with a ones column, as GraphSAGE; H recomputed)
//     dX = (1 + eps) dH + aggr^T(dH),  deps = sum_u <dH_u, X_u>      (hnh_gin_combine_grad_f64, on the device)
//              aggr^T: spmmB with weights 1 (GIN); edgeReluAggregateBackward's dX pass (GINE), whose dE pass gives
//              dE_A and [dW_e; db_e] = [attr_A 1]^T dE_A
// then one sum all-reduce of the layer's gradient vector (allreduce_world).  The forward keeps M (f doubles per row) and
// Z (h doubles per row) of every layer, so the backward runs no forward sparse pass; E_A and E_B are recomputed by GEMMs
// in the backward, so its peak adds E_A + E_B + dE_A, 3 n f doubles for the widest layer (n this rank's entries).
//
// Parameters of a layer live in one device vector, in the order of its gradients: [W1; b1] ((f + 1) x h), [W2; b2]
// ((h + 1) x r), with edge features [W_e; b_e] ((edge_dim + 1) x f), and eps last.  All are zero after construction
// except eps, which starts at the constructor's value.  Weights are stored input-major: a GINConv / GINEConv state dict
// maps onto them as nn.0.weight.T, nn.0.bias, nn.2.weight.T, nn.2.bias, lin.weight.T, lin.bias and eps.  Without
// train_eps, eps is a constant: it is not in parameters(), so no optimizer step (weight decay included) moves it, and
// its gradient reads 0; param(l, "eps") still reads and sets it.
//
// Defined where Distributed_Sparse::check_full_rows passes (every rank holds full-width rows and the A and B layouts
// coincide); elsewhere the constructor throws HNH_E_INVALID on every rank before any launch.
#pragma once
#include <cmath>
#include <string>
#include <vector>

#include "hnh/distributed_sparse.h"
#include "hnh/model.hpp"
#include "hnh/world_allreduce.hpp"
#include "hnh_b200.h"

class GINLayer {
public:
    int input_features;   // f
    int hidden_features;  // h
    int output_features;  // r

    VectorXd params;  // the layout above
    VectorXd grads;   // the same layout: dL/d params after GIN::backwardPass (same on every rank)

    GINLayer(int in_width, int hidden_width, int out_width)
        : input_features(in_width), hidden_features(hidden_width), output_features(out_width) {}

    // the offsets of [W1; b1], [W2; b2], [W_e; b_e] and eps in params / grads
    int64_t lin2_offset() const { return ((int64_t)input_features + 1) * hidden_features; }
    int64_t edge_offset() const { return lin2_offset() + ((int64_t)hidden_features + 1) * output_features; }
    int64_t eps_offset(int edge_dim) const { return edge_offset() + (edge_dim > 0 ? ((int64_t)edge_dim + 1) * input_features : 0); }
    int64_t param_count(int edge_dim) const { return eps_offset(edge_dim) + 1; }
};

class GIN : public GraphModel {
public:
    vector<GINLayer> layers;
    const int edge_dim;
    const bool train_eps;
    DenseMatrix edge_attr_A, edge_attr_B;  // num_S_values x edge_dim and num_ST_values x edge_dim
    bool has_edge_attributes = false;
    vector<DenseMatrix> aggregated, hidden;  // M and Z of every layer from the last forward pass
    // activations_current also covers the edge attributes

    GIN(vector<GINLayer> &l_input, Distributed_Sparse *ops, int edge_features, double eps, bool train)
        : GraphModel(ops, "GIN"), layers(l_input), edge_dim(edge_features), train_eps(train) {
        d_ops->check_full_rows("GIN");
        if (layers.empty()) throw hnh::Error(HNH_E_INVALID, "GIN: no layers");
        if (edge_dim < 0) throw hnh::Error(HNH_E_INVALID, "GIN: edge_dim must not be negative");
        if (!std::isfinite(eps)) throw hnh::Error(HNH_E_INVALID, "GIN: eps must be finite");
        vector<LayerWidths> widths;
        for (const GINLayer &l : layers)
            widths.push_back({l.input_features, l.output_features, l.input_features > 0 && l.hidden_features > 0 && l.output_features > 0});
        refuse("GIN", layer_chain_problem(widths));
        refuse("GIN", rows_problem());
        allocate_buffers(widths);
        for (GINLayer &layer : layers) {
            layer.params = VectorXd::Constant(layer.param_count(edge_dim), 0.0);
            hnh::abi_check(hnh_fill_f64(layer.params.data() + layer.eps_offset(edge_dim), 1, eps, stream()), "fill");
        }
        if (edge_dim == 0) {
            ones_A = d_ops->like_S_values(1.0);
            ones_B = d_ops->like_ST_values(1.0);
        }
    }

    // Edge attributes of S's entries in both value orders (row i belongs to entry i of like_S_values /
    // like_ST_values); every rank passes its part of the same attributes.  Makes the activations stale.
    void setEdgeAttributes(const double *host_A, int64_t n_A, const double *host_B, int64_t n_B) {
        uploadEdgeAttributes("GIN", edge_dim, host_A, n_A, host_B, n_B, edge_attr_A, edge_attr_B);
        has_edge_attributes = true;
    }

    // Each layer's params with its grads, one span per layer; eps (the last entry) only with train_eps
    std::vector<ParamSpan> parameters() override {
        std::vector<ParamSpan> s = layer_spans(layers);
        if (!train_eps)
            for (ParamSpan &p : s) p.n -= 1;
        return s;
    }

    // By name (the layout above): "lin1" (f x h), "lin1_bias" (h x 1), "lin2" (h x r), "lin2_bias" (r x 1), with edge
    // features "edge" (edge_dim x f) and "edge_bias" (f x 1), and "eps" (1 x 1)
    ParamRef param(int layer, const string &name) override {
        if (layer < 0 || layer >= (int)layers.size()) throw hnh::Error(HNH_E_INVALID, "GIN: no such layer");
        GINLayer &l = layers[(size_t)layer];
        const int64_t f = l.input_features, h = l.hidden_features, r = l.output_features;
        auto at = [&](int64_t offset, int64_t rows, int64_t cols) { return slice(l.params, l.grads, offset, rows, cols); };
        if (name == "lin1") return at(0, f, h);
        if (name == "lin1_bias") return at(f * h, h, 1);
        if (name == "lin2") return at(l.lin2_offset(), h, r);
        if (name == "lin2_bias") return at(l.lin2_offset() + h * r, r, 1);
        if (name == "edge" && edge_dim > 0) return at(l.edge_offset(), edge_dim, f);
        if (name == "edge_bias" && edge_dim > 0) return at(l.edge_offset() + (int64_t)edge_dim * f, f, 1);
        if (name == "eps") return at(l.eps_offset(edge_dim), 1, 1);
        throw hnh::Error(HNH_E_INVALID, "GIN: no parameter \"" + name + "\" in this model");
    }

    // Collective.
    void forwardPass() {
        check_supported("GIN::forwardPass");
        aggregated.resize(layers.size());
        hidden.resize(layers.size());
        for (size_t i = 0; i < layers.size(); i++) {
            GINLayer &l = layers[i];
            DenseMatrix &X = buffers[i];
            const int64_t n = X.rows(), h = l.hidden_features, r = l.output_features;
            aggregate(i, X);
            hidden[i].resize(n, h);
            {
                DenseMatrix H = combine(l, aggregated[i], X);
                DenseMatrix P = H * block(l.params, l, 0, false);
                hnh::abi_check(hnh_row_bias_relu_f64(hidden[i].data(), P.data(), bias(l.params, l, 0), n, h, stream()), "row_bias_relu");
            }
            DenseMatrix Y = hidden[i] * block(l.params, l, 1, false);
            hnh::abi_check(hnh_row_bias_add_f64(Y.data(), bias(l.params, l, 1), n, r, stream()), "row_bias_add");
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
        check_supported("GIN::backwardPass");
        check_backward("GIN::backwardPass", "the parameters, the input or the edge attributes", output_grad);
        backward_layers(output_grad, [&](int i, const DenseMatrix &G, DenseMatrix &dX) { backwardLayer(i, G, dX); });
    }

private:
    VectorXd ones_A, ones_B;  // GIN: the aggregation weight 1 of every entry in the A and B orders

    void check_supported(const string &who) const {
        d_ops->check_full_rows(who);
        if (edge_dim > 0 && !has_edge_attributes)
            throw hnh::Error(HNH_E_INVALID, who + ": the model has edge features and no edge attributes were set");
    }

    // MLP layer j (0: [W1; b1], 1: [W2; b2]) or the edge projection (j = 2: [W_e; b_e]) of a layer, with or without its
    // bias row, and that bias row
    DenseMatrix block(VectorXd &v, const GINLayer &l, int j, bool with_bias) const {
        const int64_t offsets[3] = {0, l.lin2_offset(), l.edge_offset()};
        const int64_t in[3] = {l.input_features, l.hidden_features, edge_dim};
        const int64_t out[3] = {l.hidden_features, l.output_features, l.input_features};
        return DenseMatrix::view(v.data() + offsets[j], in[j] + (with_bias ? 1 : 0), out[j]);
    }
    double *bias(VectorXd &v, const GINLayer &l, int j) const { return block(v, l, j, true).data() + block(v, l, j, false).size(); }
    double *eps(GINLayer &l) const { return l.params.data() + l.eps_offset(edge_dim); }

    // attr W_e + b_e
    DenseMatrix project_edges(const DenseMatrix &attr, GINLayer &l) const {
        DenseMatrix E = attr * block(l.params, l, 2, false);
        hnh::abi_check(hnh_row_bias_add_f64(E.data(), bias(l.params, l, 2), E.rows(), E.cols(), stream()), "row_bias_add");
        return E;
    }

    // aggregated[i] = M of layer i
    void aggregate(size_t i, DenseMatrix &X) {
        GINLayer &l = layers[i];
        DenseMatrix &M = aggregated[i];
        M.resize(d_ops->localArows, l.input_features);
        if (edge_dim > 0) {
            DenseMatrix E_A = project_edges(edge_attr_A, l);
            d_ops->edgeReluAggregate(X, E_A, M);
        } else {
            d_ops->setRValue(l.input_features);
            d_ops->spmmA(M, X, ones_A);
        }
    }

    // H = M + (1 + eps) X
    DenseMatrix combine(GINLayer &l, const DenseMatrix &M, const DenseMatrix &X) const {
        DenseMatrix H(X.rows(), X.cols());
        hnh::abi_check(hnh_gin_combine_f64(H.data(), M.data(), X.data(), eps(l), X.size(), stream()), "gin_combine");
        return H;
    }

    // layer i: G = dL/d buffers[i + 1]; writes layers[i].grads and dX = dL/d buffers[i]
    void backwardLayer(int i, const DenseMatrix &G, DenseMatrix &dX) {
        GINLayer &l = layers[(size_t)i];
        DenseMatrix &X = buffers[(size_t)i], &Z = hidden[(size_t)i];
        const int64_t n = X.rows(), f = l.input_features, h = l.hidden_features;
        if (l.grads.size() != l.params.size()) l.grads = VectorXd(l.params.size());
        DenseMatrix dY_relu;
        const DenseMatrix &dY = relu_grad_unless_last(i, G, dY_relu);
        {
            DenseMatrix Za = with_ones(Z);
            block(l.grads, l, 1, true).setTransposeTimes(Za, dY);
        }
        DenseMatrix dP(n, h);
        {
            DenseMatrix dZ;
            dZ.setTimesTranspose(dY, block(l.params, l, 1, false), false);
            dP.setMiddleColsReluGrad(dZ, Z, 0);  // Z > 0 exactly where H W1 + b1 > 0
        }
        {
            DenseMatrix Ha = with_ones(combine(l, aggregated[(size_t)i], X));
            block(l.grads, l, 0, true).setTransposeTimes(Ha, dP);
        }
        DenseMatrix dH;
        dH.setTimesTranspose(dP, block(l.params, l, 0, false), false);
        dP = DenseMatrix();
        dX.resize(n, f);
        double *deps = l.grads.data() + l.eps_offset(edge_dim);
        hnh::abi_check(hnh_gin_combine_grad_f64(dX.data(), train_eps ? deps : nullptr, dH.data(), X.data(), eps(l), X.size(), stream()),
                       "gin_combine_grad");
        if (!train_eps) hnh::cuda_check(cudaMemsetAsync(deps, 0, sizeof(double), stream()), "eps gradient");
        if (edge_dim > 0) {
            DenseMatrix E_A = project_edges(edge_attr_A, l), E_B = project_edges(edge_attr_B, l), dE;
            d_ops->edgeReluAggregateBackward(X, &E_A, &E_B, dH, dX, &dE, true);
            E_A = DenseMatrix();
            E_B = DenseMatrix();
            DenseMatrix dWe = block(l.grads, l, 2, true);
            if (edge_attr_A.rows() > 0)
                dWe.setTransposeTimes(with_ones(edge_attr_A), dE);
            else
                dWe.setZero();
        } else {
            d_ops->setRValue((int)f);
            DenseMatrix back = d_ops->like_B_matrix(0.0);
            d_ops->spmmB(dH, back, ones_B);
            dX += back;
        }
        allreduce_world(l.grads);
    }
};
