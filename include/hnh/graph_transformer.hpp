// hnh/graph_transformer.hpp -- a graph transformer on fused sparse attention: layers of PyG's
// TransformerConv(concat = True, root_weight = True), with edge features (edge_dim > 0) and the gated skip
// (beta = true) as options, forward and backward, with the weight gradients summed over all ranks.  It does for
// Distributed_Sparse::sparseAttention what GAT (hnh/gat.hpp) does for the composed SDDMM / softmax / SpMM path.
//
// Layer l has input width f, H heads of width d and r = H d.  With X the layer input (rows of the nodes):
//     Q = X W_q + b_q,  K = X W_k + b_k,  V = X W_v + b_v,  R = X W_s + b_s       4 GEMMs (hnh_dgemm_f64) + bias rows
//     E_A = attr_A W_e,  E_B = attr_B W_e   (edge_dim > 0; the attributes of S's entries in the A and B value orders)
//     M, L = sparseAttention(Q, K, V, heads = H, scale = 1 / sqrt(d), dropout, seed_l, edge = E_A)   1 fused pass/head
//     Y = M + R,  or with the gate  beta_u = sigmoid(w_beta . [M_u, R_u, M_u - R_u]),  Y = beta R + (1 - beta) M
//     X_{l+1} = ReLU(Y) for every layer but the last, which outputs Y             (hnh_gt_gate_f64: one row pass)
// seed_l = seed + sum_{k < l} H_k, so every (layer, head) draws its own stream seed_l + h of the dropout hash.
//
// Backward of layer l, given G = dL/d X_{l+1}:
//     dY = G (where X_{l+1} > 0 unless last),  ds_u = <dY_u, R_u - M_u> beta_u (1 - beta_u)
//     dM = (1 - beta) dY + ds (w1 + w3),  dR = beta dY + ds (w2 - w3),  dw_beta = sum_u ds_u [M_u, R_u, M_u - R_u]
//                                    (hnh_gt_gate_backward_f64: one row pass and a two-stage fixed-order reduction)
//     dQ, dK, dV, dE_A = sparseAttentionBackward(..., dZ = dM)                     2 fused passes per head
//     [dW_j; db_j] = [X 1]^T dP_j for (j, P) in (q, Q), (k, K), (v, V), (s, R)     4 GEMMs (hnh_dgemm_tn_f64; the bias
//                                    gradient is the product with the ones column, in the GEMM's fixed order)
//     dW_e = attr_A^T dE_A,  dX = dQ W_q^T + dK W_k^T + dV W_v^T + dR W_s^T         1 + 4 GEMMs (hnh_dgemm_nt_f64)
// then one sum all-reduce of all the layer's gradients (allreduce_world).  R, Q, K, V and E are recomputed by the
// GEMMs; the forward keeps M and L of every layer (r + H doubles per row per layer) so that the backward needs no
// second forward sparse pass.
//
// Parameters of a layer live in one device vector, in the order of its gradients: for j in (query, key, value, skip)
// an (f + 1) x r block of W_j (f rows) and b_j (the last row), then W_e (edge_dim x r) and w_beta (3r) when present.
// All are zero after construction.  Weights are stored input-major (f x r): a PyG TransformerConv state dict maps
// onto them by transposing lin_*.weight.
//
// Transformer blocks (ffn_ratio = k >= 1; 0, the default, is the model above): every layer becomes a post-norm
// transformer block with hidden width h = k r.  Y is the gate's output without the ReLU, and no ReLU follows a layer:
//     H1 = LN1(Y),  Z = ReLU(H1 W1 + b1),  F = Z W2 + b2,  X_{l+1} = LN2(H1 + F)
// with LN(x) = gamma (x - mean(x)) / sqrt(var(x) + norm_eps) + beta per row (biased variance over r), as torch's
// norm2(h + lin2(relu(lin1(h)))) with h = norm1(conv(x)).  Backward, before the gate's (which then runs with no ReLU):
//     dU, dgamma2, dbeta2 = LN2 backward of G                  (hnh_layer_norm_backward_f64, on H1 + F)
//     [dW2; db2] = [Z 1]^T dU,  dA = dU W2^T where Z > 0        (TN GEMM; NT GEMM and hnh_relu_cols_backward_f64)
//     [dW1; db1] = [H1 1]^T dA,  dH1 = dU + dA W1^T             (TN GEMM; NT GEMM accumulating into dU)
//     dY, dgamma1, dbeta1 = LN1 backward of dH1
// The forward keeps (mean, rstd) of both norms per row (4 doubles per row per layer) beside M and L; the backward
// recomputes Y, H1, Z and F (rewriting the same statistics) and uses them.  The block's parameters follow w_beta, in
// the order of their gradients: gamma1 (r), beta1 (r), [W1; b1] ((r + 1) x h), [W2; b2] ((h + 1) x r), gamma2 (r),
// beta2 (r); the gammas are 1 after construction (as torch's), the rest 0.  One all-reduce still covers the layer.
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

class GraphTransformerLayer {
public:
    int input_features;
    int features_per_head;
    int num_heads;

    VectorXd params;  // the layout above; zero after construction
    VectorXd grads;   // the same layout: dL/d params after GraphTransformer::backwardPass (same on every rank)

    GraphTransformerLayer(int in_width, int head_width, int heads)
        : input_features(in_width), features_per_head(head_width), num_heads(heads) {}
    int output_features() const { return features_per_head * num_heads; }

    // offset of projection j (0 query, 1 key, 2 value, 3 skip) and of the edge and gate blocks in params / grads
    int64_t projection_offset(int j) const { return (int64_t)j * (input_features + 1) * output_features(); }
    int64_t edge_offset() const { return projection_offset(4); }
    int64_t beta_offset(int edge_dim) const { return edge_offset() + (int64_t)edge_dim * output_features(); }
    int64_t block_offset(int edge_dim, bool beta) const { return beta_offset(edge_dim) + (beta ? 3 * output_features() : 0); }
    int64_t hidden_features(int ffn_ratio) const { return (int64_t)ffn_ratio * output_features(); }
    // offset of block part j (0 gamma1, 1 beta1, 2 [W1; b1], 3 [W2; b2], 4 gamma2, 5 beta2) in params / grads
    int64_t block_part_offset(int edge_dim, bool beta, int ffn_ratio, int j) const {
        const int64_t r = output_features(), h = hidden_features(ffn_ratio);
        const int64_t sizes[6] = {r, r, (r + 1) * h, (h + 1) * r, r, r};
        int64_t off = block_offset(edge_dim, beta);
        for (int k = 0; k < j; k++) off += sizes[k];
        return off;
    }
    int64_t param_count(int edge_dim, bool beta, int ffn_ratio = 0) const {
        return ffn_ratio > 0 ? block_part_offset(edge_dim, beta, ffn_ratio, 6) : block_offset(edge_dim, beta);
    }
};

class GraphTransformer : public GraphModel {
public:
    vector<GraphTransformerLayer> layers;
    const int edge_dim;
    const bool beta;
    const int ffn_ratio;    // > 0: transformer blocks with hidden width ffn_ratio * r
    const double norm_eps;  // their LayerNorms' epsilon
    DenseMatrix edge_attr_A, edge_attr_B;  // num_S_values x edge_dim and num_ST_values x edge_dim
    bool has_edge_attributes = false;
    vector<DenseMatrix> attention, lse;   // M and L of every layer from the last forward pass
    vector<DenseMatrix> norm_stats;       // with blocks: (mean, rstd) per row of LN1 and LN2 of layer i at [2i], [2i + 1]
    // activations_current also covers the edge attributes

    GraphTransformer(vector<GraphTransformerLayer> &l_input, Distributed_Sparse *ops, int edge_features, bool gate,
                     int ffn = 0, double eps = 1e-5)
        : GraphModel(ops, "graph transformer"), layers(l_input), edge_dim(edge_features), beta(gate), ffn_ratio(ffn), norm_eps(eps) {
        d_ops->check_full_rows("GraphTransformer");
        if (layers.empty()) throw hnh::Error(HNH_E_INVALID, "GraphTransformer: no layers");
        if (edge_dim < 0) throw hnh::Error(HNH_E_INVALID, "GraphTransformer: edge_dim must not be negative");
        if (ffn_ratio < 0) throw hnh::Error(HNH_E_INVALID, "GraphTransformer: ffn_ratio must not be negative");
        if (!(norm_eps > 0.0) || !std::isfinite(norm_eps))
            throw hnh::Error(HNH_E_INVALID, "GraphTransformer: norm_eps must be finite and > 0");
        vector<LayerWidths> widths;
        for (const GraphTransformerLayer &l : layers)
            widths.push_back({l.input_features, (int64_t)l.features_per_head * l.num_heads,
                              l.input_features > 0 && l.features_per_head > 0 && l.num_heads > 0});
        refuse("GraphTransformer", layer_chain_problem(widths, [&](size_t i) -> string {
                   const int64_t r = widths[i].out;
                   return r > INT32_MAX || r * std::max(ffn_ratio, 1) > INT32_MAX ? "layer " + std::to_string(i) + " is too wide" : "";
               }));
        refuse("GraphTransformer", rows_problem());
        allocate_buffers(widths);
        for (GraphTransformerLayer &layer : layers) {
            layer.params = VectorXd::Constant(layer.param_count(edge_dim, beta, ffn_ratio), 0.0);
            if (ffn_ratio > 0)
                for (int j : {0, 4}) block_vector(layer.params, layer, j).setConstant(1.0);  // the LayerNorm gains
        }
    }

    // the weights (f x r), bias (r), edge projection (edge_dim x r) and gate vector (3r) of a layer, as views
    static DenseMatrix weight(VectorXd &v, const GraphTransformerLayer &l, int j) {
        return DenseMatrix::view(v.data() + l.projection_offset(j), l.input_features, l.output_features());
    }
    static double *bias(VectorXd &v, const GraphTransformerLayer &l, int j) {
        return v.data() + l.projection_offset(j) + (int64_t)l.input_features * l.output_features();
    }
    DenseMatrix edge_weight(VectorXd &v, const GraphTransformerLayer &l) const {
        return DenseMatrix::view(v.data() + l.edge_offset(), edge_dim, l.output_features());
    }
    // block part j of a layer (see block_part_offset): the vectors (j = 0, 1, 4, 5) as 1 x r, the FFN layers (j = 2, 3)
    // as their (input + 1) x output blocks, and those blocks' weights without the bias row
    DenseMatrix block_vector(VectorXd &v, const GraphTransformerLayer &l, int j) const {
        return DenseMatrix::view(v.data() + l.block_part_offset(edge_dim, beta, ffn_ratio, j), 1, l.output_features());
    }
    DenseMatrix ffn_block(VectorXd &v, const GraphTransformerLayer &l, int j, bool with_bias) const {
        const int64_t r = l.output_features(), h = l.hidden_features(ffn_ratio);
        const int64_t in = j == 2 ? r : h, out = j == 2 ? h : r;
        return DenseMatrix::view(v.data() + l.block_part_offset(edge_dim, beta, ffn_ratio, j), in + (with_bias ? 1 : 0), out);
    }

    // Edge attributes of S's entries in both value orders (row i belongs to entry i of like_S_values /
    // like_ST_values); every rank passes its part of the same attributes.  Makes the activations stale.
    void setEdgeAttributes(const double *host_A, int64_t n_A, const double *host_B, int64_t n_B) {
        uploadEdgeAttributes("GraphTransformer", edge_dim, host_A, n_A, host_B, n_B, edge_attr_A, edge_attr_B);
        has_edge_attributes = true;
    }

    // Each layer's params with its grads, one span per layer
    std::vector<ParamSpan> parameters() override { return layer_spans(layers); }

    // By name (the layout above): "query", "key", "value", "skip" (f x r) and their "_bias" (r x 1), "edge" (edge_dim x
    // r) with edge features, "beta" (3r x 1) with the gate; with blocks "norm1", "norm1_bias" (r x 1), "ffn1" ((r + 1) x
    // h), "ffn2" ((h + 1) x r), "norm2", "norm2_bias"
    ParamRef param(int layer, const string &name) override {
        if (layer < 0 || layer >= (int)layers.size()) throw hnh::Error(HNH_E_INVALID, "graph transformer: no such layer");
        GraphTransformerLayer &l = layers[(size_t)layer];
        const int64_t f = l.input_features, r = l.output_features();
        auto at = [&](int64_t offset, int64_t rows, int64_t cols) { return slice(l.params, l.grads, offset, rows, cols); };
        static const char *const projections[4] = {"query", "key", "value", "skip"};
        for (int j = 0; j < 4; j++) {
            if (name == projections[j]) return at(l.projection_offset(j), f, r);
            if (name == string(projections[j]) + "_bias") return at(l.projection_offset(j) + f * r, r, 1);
        }
        if (name == "edge" && edge_dim > 0) return at(l.edge_offset(), edge_dim, r);
        if (name == "beta" && beta) return at(l.beta_offset(edge_dim), 3 * r, 1);
        if (ffn_ratio > 0) {
            const int64_t h = l.hidden_features(ffn_ratio);
            static const char *const block[6] = {"norm1", "norm1_bias", "ffn1", "ffn2", "norm2", "norm2_bias"};
            const int64_t rows[6] = {r, r, r + 1, h + 1, r, r}, cols[6] = {1, 1, h, r, 1, 1};
            for (int j = 0; j < 6; j++)
                if (name == block[j]) return at(l.block_part_offset(edge_dim, beta, ffn_ratio, j), rows[j], cols[j]);
        }
        throw hnh::Error(HNH_E_INVALID, "graph transformer: no parameter \"" + name + "\" in this model");
    }

    // Collective.  dropout in [0, 1) and seed go to every layer's attention (seed_l as above); the backward pass
    // regenerates the same masks.
    void forwardPass(double dropout, uint64_t seed) {
        check_supported("GraphTransformer::forwardPass", dropout);
        uint64_t seed_l = seed;
        attention.resize(layers.size());
        lse.resize(layers.size());
        if (ffn_ratio > 0) norm_stats.resize(2 * layers.size());
        for (size_t i = 0; i < layers.size(); i++) {
            GraphTransformerLayer &layer = layers[i];
            const DenseMatrix &X = buffers[i];
            const int64_t n = X.rows(), r = layer.output_features();
            attention[i].resize(n, r);
            lse[i].resize(d_ops->localArows, layer.num_heads);
            {
                DenseMatrix Q = project(X, layer, 0), K = project(X, layer, 1), V = project(X, layer, 2), E;
                if (edge_dim > 0) E = edge_attr_A * edge_weight(layer.params, layer);
                d_ops->sparseAttention(Q, K, V, attention[i], lse[i], layer.num_heads, scale(layer), dropout, seed_l, nullptr,
                                       edge_dim > 0 ? &E : nullptr);
            }
            DenseMatrix R = project(X, layer, 3);
            if (ffn_ratio == 0) {
                hnh::abi_check(hnh_gt_gate_f64(buffers[i + 1].data(), attention[i].data(), R.data(),
                                               beta ? layer.params.data() + layer.beta_offset(edge_dim) : nullptr, n, r,
                                               i + 1 < layers.size() ? 1 : 0, stream()),
                               "gt_gate");
            } else {
                DenseMatrix Y = gate(layer, attention[i], R);
                R = DenseMatrix();
                DenseMatrix H1, F;
                blockHidden(i, Y, H1, F);
                Y = DenseMatrix();
                layerNorm(buffers[i + 1], norm_stats[2 * i + 1], F, &H1, layer, 4);
            }
            seed_l += (uint64_t)layer.num_heads;
        }
        dropout_ = dropout;
        seed_ = seed;
        activations_current = true;
    }
    void forward(double dropout, uint64_t seed) override { forwardPass(dropout, seed); }

    // output_grad = dL/d buffers.back() (this rank's rows).  Leaves dL/d params in layers[i].grads (summed over all
    // ranks) and dL/d buffers[0] in input_grad.  Collective.  Uses the forward pass's dropout and seed.
    void backwardPass(const DenseMatrix &output_grad) override {
        check_supported("GraphTransformer::backwardPass", dropout_);
        check_backward("GraphTransformer::backwardPass", "the parameters, the input or the edge attributes", output_grad);
        uint64_t seed_l = seed_;
        vector<uint64_t> seeds;
        for (const GraphTransformerLayer &layer : layers) {
            seeds.push_back(seed_l);
            seed_l += (uint64_t)layer.num_heads;
        }
        backward_layers(output_grad, [&](int i, const DenseMatrix &G, DenseMatrix &dX) { backwardLayer(i, G, dX, seeds[(size_t)i]); });
    }

private:
    double dropout_ = 0.0;
    uint64_t seed_ = 0;

    static double scale(const GraphTransformerLayer &l) { return 1.0 / std::sqrt((double)l.features_per_head); }

    // Everything a pass needs that every rank decides alike, checked before any launch
    void check_supported(const string &who, double dropout) const {
        d_ops->check_full_rows(who);
        if (!(dropout >= 0.0 && dropout < 1.0))
            throw hnh::Error(HNH_E_INVALID, who + ": the dropout probability must lie in [0, 1), got " + std::to_string(dropout));
        if (edge_dim > 0 && !has_edge_attributes)
            throw hnh::Error(HNH_E_INVALID, who + ": the model has edge features and no edge attributes were set");
    }

    // X W_j + b_j
    static DenseMatrix project(const DenseMatrix &X, GraphTransformerLayer &layer, int j) {
        DenseMatrix P = X * weight(layer.params, layer, j);
        hnh::abi_check(hnh_row_bias_add_f64(P.data(), bias(layer.params, layer, j), P.rows(), P.cols(), stream()), "row_bias_add");
        return P;
    }

    // The gate's output without a ReLU: Y = M + R, or beta R + (1 - beta) M
    DenseMatrix gate(GraphTransformerLayer &layer, const DenseMatrix &M, const DenseMatrix &R) const {
        DenseMatrix Y(M.rows(), M.cols());
        hnh::abi_check(hnh_gt_gate_f64(Y.data(), M.data(), R.data(), beta ? layer.params.data() + layer.beta_offset(edge_dim) : nullptr,
                                       M.rows(), M.cols(), 0, stream()),
                       "gt_gate");
        return Y;
    }

    // out = LN(X + Res) with the gain and bias at block part j (0: LN1, 4: LN2); (mean, rstd) per row into stats
    void layerNorm(DenseMatrix &out, DenseMatrix &stats, const DenseMatrix &X, const DenseMatrix *Res, GraphTransformerLayer &layer,
                   int j) const {
        const int64_t n = X.rows(), r = X.cols();
        if (out.rows() != n || out.cols() != r) out.resize(n, r);
        stats.resize(n, 2);
        hnh::abi_check(hnh_layer_norm_f64(out.data(), stats.data(), X.data(), Res ? Res->data() : nullptr,
                                          block_vector(layer.params, layer, j).data(), block_vector(layer.params, layer, j + 1).data(),
                                          n, r, norm_eps, stream()),
                       "layer_norm");
    }

    // The block from the gate's output Y up to LN2's input: H1 = LN1(Y) (its statistics into norm_stats[2i]) and
    // F = ReLU(H1 W1 + b1) W2 + b2.  With Z given, Z = ReLU(H1 W1 + b1) is kept there.
    void blockHidden(size_t i, const DenseMatrix &Y, DenseMatrix &H1, DenseMatrix &F, DenseMatrix *keep_Z = nullptr) {
        GraphTransformerLayer &layer = layers[i];
        layerNorm(H1, norm_stats[2 * i], Y, nullptr, layer, 0);
        const int64_t n = Y.rows(), r = Y.cols(), h = layer.hidden_features(ffn_ratio);
        DenseMatrix Z(n, h);
        {
            DenseMatrix A = H1 * ffn_block(layer.params, layer, 2, false);
            hnh::abi_check(hnh_row_bias_relu_f64(Z.data(), A.data(), layer.params.data() + layer.block_part_offset(edge_dim, beta, ffn_ratio, 2) + r * h,
                                                 n, h, stream()),
                           "row_bias_relu");
        }
        F = Z * ffn_block(layer.params, layer, 3, false);
        hnh::abi_check(hnh_row_bias_add_f64(F.data(), layer.params.data() + layer.block_part_offset(edge_dim, beta, ffn_ratio, 3) + h * r,
                                            n, r, stream()),
                       "row_bias_add");
        if (keep_Z) *keep_Z = std::move(Z);
    }

    // LN backward of G for block part j (0: LN1 on X, 4: LN2 on X + Res) into dX, its gain and bias gradients into grads
    void layerNormBackward(DenseMatrix &dX, const DenseMatrix &G, const DenseMatrix &X, const DenseMatrix *Res,
                           const DenseMatrix &stats, GraphTransformerLayer &layer, int j) const {
        const int64_t n = X.rows(), r = X.cols();
        dX.resize(n, r);
        const int64_t ws_bytes = hnh_layer_norm_backward_workspace_bytes(n, r);
        if (ws_bytes < 0) hnh::abi_check((int)ws_bytes, "layer_norm_backward");
        hnh::DeviceBuffer<char> ws((size_t)ws_bytes);
        hnh::abi_check(hnh_layer_norm_backward_f64(dX.data(), block_vector(layer.grads, layer, j).data(),
                                                   block_vector(layer.grads, layer, j + 1).data(), G.data(), X.data(),
                                                   Res ? Res->data() : nullptr, stats.data(), block_vector(layer.params, layer, j).data(),
                                                   n, r, 0, ws.data(), (size_t)ws_bytes, stream()),
                       "layer_norm_backward");
    }

    // The block's backward of layer i from G = dL/d buffers[i + 1] down to dL/dY, given the gate's output Y; writes
    // the block's part of layers[i].grads
    DenseMatrix blockBackward(size_t i, const DenseMatrix &G, const DenseMatrix &Y) {
        GraphTransformerLayer &layer = layers[i];
        const int64_t n = Y.rows(), h = layer.hidden_features(ffn_ratio);
        DenseMatrix H1, F, Z, dU;
        blockHidden(i, Y, H1, F, &Z);
        layerNormBackward(dU, G, F, &H1, norm_stats[2 * i + 1], layer, 4);
        F = DenseMatrix();
        {
            DenseMatrix Za = with_ones(Z);
            ffn_block(layer.grads, layer, 3, true).setTransposeTimes(Za, dU);
        }
        DenseMatrix dA(n, h);
        {
            DenseMatrix dZ;
            dZ.setTimesTranspose(dU, ffn_block(layer.params, layer, 3, false), false);
            dA.setMiddleColsReluGrad(dZ, Z, 0);  // Z > 0 exactly where H1 W1 + b1 > 0
        }
        Z = DenseMatrix();
        {
            DenseMatrix H1a = with_ones(H1);
            ffn_block(layer.grads, layer, 2, true).setTransposeTimes(H1a, dA);
        }
        H1 = DenseMatrix();
        dU.setTimesTranspose(dA, ffn_block(layer.params, layer, 2, false), true);  // dH1 = dU + dA W1^T
        dA = DenseMatrix();
        DenseMatrix dY;
        layerNormBackward(dY, dU, Y, nullptr, norm_stats[2 * i], layer, 0);
        return dY;
    }

    // layer i: G = dL/d buffers[i + 1]; writes layers[i].grads and dX = dL/d buffers[i]
    void backwardLayer(int i, const DenseMatrix &G, DenseMatrix &dX, uint64_t seed_l) {
        GraphTransformerLayer &layer = layers[(size_t)i];
        const DenseMatrix &X = buffers[(size_t)i], &out = buffers[(size_t)i + 1];
        const int64_t n = X.rows(), f = X.cols(), r = layer.output_features();
        if (layer.grads.size() != layer.params.size()) layer.grads = VectorXd(layer.params.size());
        const bool relu = ffn_ratio == 0 && i + 1 < (int)layers.size();

        DenseMatrix Xa = with_ones(X);
        auto grad_block = [&](int j) { return DenseMatrix::view(layer.grads.data() + layer.projection_offset(j), f + 1, r); };

        // the gate: dM, dR (dR = dM without it) and dw_beta
        DenseMatrix dM(n, r), dR;
        {
            DenseMatrix R = project(X, layer, 3);
            DenseMatrix dY;  // with blocks: dL/d the gate's output
            if (ffn_ratio > 0) dY = blockBackward((size_t)i, G, gate(layer, attention[(size_t)i], R));
            if (beta) dR.resize(n, r);
            const int64_t ws_bytes = beta ? hnh_gt_gate_backward_workspace_bytes(n, r) : 0;
            if (ws_bytes < 0) hnh::abi_check((int)ws_bytes, "gt_gate_backward");
            hnh::DeviceBuffer<char> ws((size_t)ws_bytes);
            hnh::abi_check(hnh_gt_gate_backward_f64(dM.data(), beta ? dR.data() : nullptr,
                                                    beta ? layer.grads.data() + layer.beta_offset(edge_dim) : nullptr,
                                                    ffn_ratio > 0 ? dY.data() : G.data(),
                                                    relu ? out.data() : nullptr, attention[(size_t)i].data(), R.data(),
                                                    beta ? layer.params.data() + layer.beta_offset(edge_dim) : nullptr, n, r,
                                                    relu ? 1 : 0, ws.data(), (size_t)ws_bytes, stream()),
                           "gt_gate_backward");
        }
        {
            const DenseMatrix &dRs = beta ? dR : dM;
            grad_block(3).setTransposeTimes(Xa, dRs);
            dX.setTimesTranspose(dRs, weight(layer.params, layer, 3), false);
        }
        dR = DenseMatrix();

        // attention: Q, K, V and E recomputed
        DenseMatrix Q = project(X, layer, 0), K = project(X, layer, 1), V = project(X, layer, 2);
        DenseMatrix dQ(n, r), dK(n, r), dV(n, r), E_A, E_B, dE;
        if (edge_dim > 0) {
            E_A = edge_attr_A * edge_weight(layer.params, layer);
            E_B = edge_attr_B * edge_weight(layer.params, layer);
        }
        d_ops->sparseAttentionBackward(Q, K, V, attention[(size_t)i], lse[(size_t)i], dM, dQ, dK, dV, layer.num_heads, scale(layer),
                                       dropout_, seed_l, nullptr, nullptr, nullptr, nullptr, edge_dim > 0 ? &E_A : nullptr,
                                       edge_dim > 0 ? &E_B : nullptr, edge_dim > 0 ? &dE : nullptr);
        Q = DenseMatrix();
        K = DenseMatrix();
        V = DenseMatrix();
        E_A = DenseMatrix();
        E_B = DenseMatrix();
        dM = DenseMatrix();
        const DenseMatrix *dP[3] = {&dQ, &dK, &dV};
        for (int j = 0; j < 3; j++) {
            grad_block(j).setTransposeTimes(Xa, *dP[j]);
            dX.setTimesTranspose(*dP[j], weight(layer.params, layer, j), true);
        }
        if (edge_dim > 0) {
            DenseMatrix dWe = edge_weight(layer.grads, layer);
            if (edge_attr_A.rows() > 0)
                dWe.setTransposeTimes(edge_attr_A, dE);
            else
                dWe.setZero();
        }
        allreduce_world(layer.grads);
    }
};
