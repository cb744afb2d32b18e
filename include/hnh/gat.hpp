// hnh/gat.hpp -- multi-head graph attention on top of a Distributed_Sparse object: forward pass and the
// gradients of the weights and of the network input.  The second application that benchmark_algorithm can run
// (app == "gat", and "gat_train" = forward + backward).  Class and member names follow the reference (GATLayer,
// GAT{d_ops, layers, buffers, leaky_relu_alpha, computeSelfAttentionHead, forwardPass}: gat.hpp:26-113; used at
// benchmark_dist.cpp:88-94,133-135) so that its callers compile.  The reference has no backward pass.
//
// One head of one layer:
//     H      = X_in * W                       dense projection          (hnh_dgemm_f64: own fp64 DMMA kernel)
//     e_uv   = <H_u, H_v> for every edge      SDDMM through d_ops       (K1)
//     e_uv   = LeakyReLU(e_uv)                                           (hnh_leaky_relu_f64)
//     Z      = E * H                          SpMM through d_ops        (K2)
//     X_out[:, head window] = ReLU(Z)                                    (hnh_relu_cols_f64)
// All operands stay in HBM between the steps.  The weights are whatever the caller stores in
// layers[i].wMats[j]; the reference leaves them zero and never assigns leaky_relu_alpha (reading it is
// undefined there) -- this implementation defaults alpha to 0.2.
//
// Backward of one head, given G = dL/d X_out (backwardHead; P = H, S = the sparsity pattern, a = LeakyReLU(e)):
//     dZ  = G[:, head window] where X_out[:, head window] > 0, else 0     (hnh_relu_cols_backward_f64)
//     de  = LeakyReLU'(e) o S o (dZ P^T)      SDDMM with SValues = LeakyReLU'(e)
//     dP  = S_de P + S_a^T dZ + S_de^T P      one A-mode and two B-mode SpMMs
//     dW  = X_in^T dP, summed over all ranks  (hnh_dgemm_tn_f64, then an all-reduce over the world)
//     dX_in += dP W^T                         (hnh_dgemm_nt_f64)
// P and e are recomputed (the forward stores nothing extra).  A-mode and B-mode value vectors are in different
// orders, so the B-mode vectors come from B-mode SDDMMs of the same operands, never from a permutation.  Per head:
// 4 SDDMM passes (e and de in both orders), 3 SpMM passes and 3 GEMMs (P, dW, dX).
//
// Softmax attention (set_attention("softmax"); the default "leaky" is the reference's formula above) normalises
// the scores over each node's neighbours: alpha_u. = softmax over the stored entries of row u of LeakyReLU(e_u.)
// (Distributed_Sparse::edgeSoftmax, on the A-order scores), and Z = S_alpha H.  Its backward, with
// a = LeakyReLU(e):
//     dalpha = S o (dZ P^T)                              SDDMM with SValues = 1, both orders
//     de     = LeakyReLU'(e) o alpha o (dalpha - t)      t_u = sum_v alpha_uv dalpha_uv (edgeSoftmaxBackward)
//     dP     = S_de P + S_alpha^T dZ + S_de^T P          the leaky formula with a_B replaced by alpha_B
// alpha is recomputed in both orders.  Per head this adds one O(nnz) softmax to the forward pass, and four O(nnz)
// softmax calls (and, at p > 1, six M-long all-reduces) to the backward pass; the sparse pass count is unchanged.
//
// Additive attention (set_attention("additive"), the attention of Velickovic et al. 2018) scores an edge from two
// node scalars instead of an r-wide dot product.  With a1, a2 the head's slices [j * fph, (j + 1) * fph) of
// layer.a1 / layer.a2 (zero after construction: uniform attention, i.e. mean aggregation):
//     s = P a1, t = P a2                   over this rank's rows, gathered into whole node vectors  (hnh_gat_node_scalars_f64)
//     alpha = edge softmax of x_uv = LeakyReLU(s_u + t_v)                  (Distributed_Sparse::additiveScores, edgeSoftmax)
//     Z = S_alpha P, X_out[:, head window] = ReLU(Z)
// Backward, with x' = LeakyReLU'(s_u + t_v):
//     dalpha = S o (dZ P^T)                                  SDDMM with SValues = 1, A order only
//     de     = x' o edgeSoftmaxBackward(alpha, dalpha)       A order
//     ds_u = sum_v de_uv, dt_v = sum_u de_uv                 world row and column sums (Distributed_Sparse::edgeSums)
//     dP     = S_alpha^T dZ + ds a1^T + dt a2^T              one B-order SpMM (alpha recomputed in the B order from s and
//                                                            t), then a rank-2 row update (hnh_gat_rank2_update_f64)
//     da1 = P^T ds, da2 = P^T dt over this rank's rows, summed over all ranks (layer.a1Grads / a2Grads); dW, dX as above
// Per head: forward 1 SpMM pass, backward 1 SDDMM and 1 SpMM pass, against 1 + 1 and 4 + 3 for the dot-product
// attention.  The forward stores nothing extra: P, s, t and alpha are recomputed.
//
// GATv2 attention (set_attention("gatv2"), Brody, Alon and Yahav 2022; the shared-weights form) applies the
// nonlinearity before the attention vector, so that a node's ranking of its neighbours depends on the node.  With a
// the head's slice of layer.a1 (a2 is not read; its gradient stays zero) and sigma = LeakyReLU(., leaky_relu_alpha):
//     x_uv  = sum_k a_k sigma(P_uk + P_vk)                     (Distributed_Sparse::gatv2Scores, A order)
//     alpha = edge softmax of x, Z = S_alpha P, X_out[:, head window] = ReLU(Z)
// Backward, with z_uv = P_u + P_v:
//     dalpha = S o (dZ P^T), de = edgeSoftmaxBackward(alpha, dalpha)         both orders
//     dP     = S_alpha^T dZ + sum_v de_uv a o sigma'(z_uv) (rows u) + sum_u de_uv a o sigma'(z_uv) (rows v)
//     da     = sum_uv de_uv sigma(z_uv), summed over all ranks (layer.a1Grads)  (Distributed_Sparse::gatv2Backward)
// Per head: forward 1 score pass + 1 SpMM; backward 2 score passes (alpha recomputed in both orders), 2 SDDMMs,
// 2 gradient passes and 1 SpMM -- 7 sparse passes, as for the dot-product attention.  The forward stores nothing extra.
//
// The forward pass is the GAT formula only where every rank holds full-width rows and the A and B layouts coincide:
// p = 1 (any algorithm), 1.5D dense shift with replication reuse (fusion 1) at any c, and with local kernel fusion
// (fusion 2) at c = 1 (Distributed_Sparse::check_full_rows).  Only there are the backward pass and softmax, additive
// and GATv2 attention defined; elsewhere they throw HNH_E_INVALID on every rank.
#pragma once
#include <string>
#include <vector>

#include "hnh/15D_dense_shift.hpp"
#include "hnh/distributed_sparse.h"
#include "hnh/model.hpp"
#include "hnh/world_allreduce.hpp"
#include "hnh_b200.h"

class GATLayer {
public:
    int input_features;
    int features_per_head;
    int num_heads;

    vector<DenseMatrix> wMats;  // one input_width x head_width projection per head
    vector<DenseMatrix> wGrads; // dL/d wMats[j] after GAT::backwardPass (empty before the first one); same on every rank
    // attention vectors (declared by the reference, unused by its forward pass): num_heads * features_per_head
    // doubles each, head j's at [j * features_per_head, (j + 1) * features_per_head).  GAT allocates them as zeros;
    // additive attention reads both, GATv2 attention a1 only.
    VectorXd a1;
    VectorXd a2;
    VectorXd a1Grads;  // dL/d a1, dL/d a2 after GAT::backwardPass (empty before the first one; zero for the attention
    VectorXd a2Grads;  // kinds that do not read them); same on every rank

    GATLayer(int in_width, int head_width, int heads)
        : input_features(in_width), features_per_head(head_width), num_heads(heads) {}
    int output_features() const { return features_per_head * num_heads; }
};

class GAT : public GraphModel {
public:
    vector<GATLayer> layers;
    double leaky_relu_alpha = 0.2;

    GAT(vector<GATLayer> &l_input, Distributed_Sparse *ops) : GraphModel(ops, "gat"), layers(l_input) {
        if (layers.empty()) throw hnh::Error(-1, "GAT: no layers");
        for (size_t i = 1; i < layers.size(); i++)
            if (layers[i].input_features != layers[i - 1].output_features())
                throw hnh::Error(-1, "GAT: layer " + std::to_string(i) + " does not take the width layer " +
                                         std::to_string(i - 1) + " produces");
        // Shapes come from the algorithm object at the R in force, as in the reference (gat.hpp:60-79):
        // the input is B-shaped at R = input width, layer outputs are A-shaped at R = heads * head width,
        // a head's projection maps the previous buffer's local columns onto localAcols at R = head width.
        d_ops->setRValue(layers.front().input_features);
        buffers.push_back(d_ops->like_B_matrix(0.0));
        for (GATLayer &layer : layers) {
            const int64_t in_cols = buffers.back().cols();
            d_ops->setRValue(layer.output_features());
            buffers.push_back(d_ops->like_A_matrix(0.0));
            d_ops->setRValue(layer.features_per_head);
            layer.wMats.clear();
            for (int h = 0; h < layer.num_heads; h++)
                layer.wMats.push_back(DenseMatrix::Constant(in_cols, d_ops->localAcols, 0.0));
            layer.a1 = VectorXd::Constant((int64_t)layer.num_heads * layer.features_per_head, 0.0);
            layer.a2 = VectorXd::Constant((int64_t)layer.num_heads * layer.features_per_head, 0.0);
        }
    }

    // GAT's key function, defined in the library (csrc/benchmark_dist.cpp): the vtable, and the backward pass it names
    // (which calls the CUDA runtime), are emitted there, so a program that only constructs GAT and runs forwardPass
    // links without the CUDA runtime, as the reference's drivers do
    ~GAT() override;

    // head j of layer i: reads buffers[i], writes its column window of buffers[i + 1]
    void computeSelfAttentionHead(int i, int j) {
        GATLayer &layer = layers.at((size_t)i);
        DenseMatrix &input = buffers[(size_t)i], &output = buffers[(size_t)i + 1];
        d_ops->setRValue(layer.features_per_head);

        DenseMatrix projected = input * layer.wMats.at((size_t)j);
        DenseMatrix neighbours = projected;  // the same projection in the role of the other SDDMM operand
        d_ops->de_shift(&neighbours, nullptr, k_spmmA);

        VectorXd scores = d_ops->like_S_values(1.0);
        if (gatv2_) {
            d_ops->gatv2Scores(projected, neighbours, head_vector(layer.a1, layer, j), scores, k_sddmmA, leaky_relu_alpha);
            d_ops->edgeSoftmax(scores, k_sddmmA);
        } else if (additive_) {
            VectorXd s, t;
            node_scalars(layer, j, projected, s, t);
            d_ops->additiveScores(s, t, scores, k_sddmmA, leaky_relu_alpha, false);
            d_ops->edgeSoftmax(scores, k_sddmmA);
        } else {
            VectorXd pattern = d_ops->like_S_values(1.0);
            d_ops->algorithm(projected, neighbours, pattern, &scores, k_sddmmA, true);
            scores.leakyRelu(leaky_relu_alpha);
            if (softmax_) d_ops->edgeSoftmax(scores, k_sddmmA);
        }

        projected.setZero();  // becomes the SpMM accumulator
        // replication reuse: the SDDMM pass has replicated the stationary operand, except with additive and GATv2
        // attention, which have no SDDMM pass
        d_ops->algorithm(projected, neighbours, scores, nullptr, k_spmmA, additive_ || gatv2_);
        output.setMiddleColsRelu((int64_t)j * projected.cols(), projected);
    }

    void forwardPass() {
        if (softmax_) d_ops->check_full_rows("GAT softmax attention");
        if (additive_) d_ops->check_full_rows("GAT additive attention");
        if (gatv2_) d_ops->check_full_rows("GAT GATv2 attention");
        for (size_t i = 0; i < layers.size(); i++)
            for (int j = 0; j < layers[i].num_heads; j++) computeSelfAttentionHead((int)i, j);
        activations_current = true;
    }
    void forward(double dropout, uint64_t) override {
        refuse_dropout(dropout);
        forwardPass();
    }

    // ---- backward pass -------------------------------------------------------------------------------
    // Throws HNH_E_INVALID unless the backward pass is defined on this algorithm object (see the top of this
    // file).  Decided from global quantities only, so every rank throws together and no collective is left waiting.
    void check_backward_supported() const { d_ops->check_full_rows("GAT::backwardPass"); }
    void check_trainable() const override { check_backward_supported(); }

    // Every (layer, head) weight with its gradient, then a1 and a2 of every layer with theirs; grad is null before the
    // first backward pass.
    std::vector<ParamSpan> parameters() override {
        std::vector<ParamSpan> s;
        for (GATLayer &l : layers)
            for (size_t h = 0; h < l.wMats.size(); h++)
                s.push_back({l.wMats[h].data(), l.wGrads.size() == l.wMats.size() ? l.wGrads[h].data() : nullptr, l.wMats[h].size()});
        for (GATLayer &l : layers) {
            s.push_back({l.a1.data(), l.a1Grads.size() == l.a1.size() ? l.a1Grads.data() : nullptr, l.a1.size()});
            s.push_back({l.a2.data(), l.a2Grads.size() == l.a2.size() ? l.a2Grads.data() : nullptr, l.a2.size()});
        }
        return s;
    }

    // "leaky" (the reference's attention, the default), "softmax", "additive" or "gatv2" (see the top of this file).
    // Changing it makes the activations stale.
    const string &attention() const { return attention_; }
    void set_attention(const string &kind) {
        if (kind != "leaky" && kind != "softmax" && kind != "additive" && kind != "gatv2")
            throw hnh::Error(HNH_E_INVALID, "GAT: attention must be \"leaky\", \"softmax\", \"additive\" or \"gatv2\", not \"" +
                                                kind + "\"");
        if (kind != attention_) activations_current = false;
        attention_ = kind;
        softmax_ = kind == "softmax";
        additive_ = kind == "additive";
        gatv2_ = kind == "gatv2";
    }

    // output_grad = dL/d buffers.back() (this rank's rows).  Leaves dL/d wMats in layers[i].wGrads and dL/d a1 / a2
    // in layers[i].a1Grads / a2Grads (summed over all ranks: identical everywhere), and dL/d buffers[0] in
    // input_grad.  Collective.  Reads buffers, wMats, a1, a2 and leaky_relu_alpha and changes none of them; gradient
    // storage is allocated on the first call.
    void backwardPass(const DenseMatrix &output_grad) override {
        check_backward_supported();
        if (!activations_current)
            throw hnh::Error(HNH_E_INVALID, "GAT::backwardPass: no forward pass since the weights or the input changed");
        if (output_grad.rows() != buffers.back().rows() || output_grad.cols() != buffers.back().cols())
            throw hnh::Error(HNH_E_INVALID, "GAT::backwardPass: the output gradient is " + std::to_string(output_grad.rows()) +
                                                " x " + std::to_string(output_grad.cols()) + ", the network output " +
                                                std::to_string(buffers.back().rows()) + " x " +
                                                std::to_string(buffers.back().cols()));
        for (GATLayer &layer : layers)
            if (layer.wGrads.size() != layer.wMats.size()) {
                layer.wGrads.clear();
                for (const DenseMatrix &w : layer.wMats) layer.wGrads.emplace_back(w.rows(), w.cols());
            }
        for (GATLayer &layer : layers)
            // additive attention writes every entry of both, GATv2 attention every entry of a1Grads; a2Grads and the
            // kinds that do not read the vectors leave zeros
            if (layer.a1Grads.size() != layer.a1.size() || !additive_) {
                layer.a1Grads = VectorXd::Constant(layer.a1.size(), 0.0);
                layer.a2Grads = VectorXd::Constant(layer.a2.size(), 0.0);
            }
        // two layer gradients are live at a time: that of the layer's output (upstream) and that of its input
        DenseMatrix upstream;
        for (int i = (int)layers.size() - 1; i >= 0; i--) {
            const DenseMatrix &G = i + 1 == (int)layers.size() ? output_grad : upstream;
            DenseMatrix downstream;
            DenseMatrix &dX = i == 0 ? input_grad : downstream;
            dX.resize(buffers[(size_t)i].rows(), buffers[(size_t)i].cols());
            for (int j = 0; j < layers[(size_t)i].num_heads; j++) backwardHead(i, j, G, dX, j > 0);
            if (i > 0) upstream = std::move(downstream);
        }
    }

    // head j of layer i: G = dL/d buffers[i + 1]; writes layers[i].wGrads[j] and adds (or, accumulate == false,
    // writes) the head's share of dL/d buffers[i] into dX
    void backwardHead(int i, int j, const DenseMatrix &G, DenseMatrix &dX, bool accumulate) {
        if (additive_) return backwardHeadAdditive(i, j, G, dX, accumulate);
        if (gatv2_) return backwardHeadGatv2(i, j, G, dX, accumulate);
        GATLayer &layer = layers.at((size_t)i);
        const DenseMatrix &input = buffers[(size_t)i], &output = buffers[(size_t)i + 1];
        const DenseMatrix &W = layer.wMats.at((size_t)j);
        d_ops->setRValue(layer.features_per_head);
        // In every supported layout initial_shift / de_shift are identities, and the SDDMMs only read their operands,
        // so P serves as both of them.
        DenseMatrix P = input * W;

        // attention scores in both value orders; g = LeakyReLU'(e) (A order, B order), a = LeakyReLU(e) (B order; with
        // softmax attention alpha = edge softmax of LeakyReLU(e), both orders)
        VectorXd ones_A = d_ops->like_S_values(1.0), ones_B = d_ops->like_ST_values(1.0);
        VectorXd g_A = d_ops->like_S_values(0.0), g_B = d_ops->like_ST_values(0.0);
        d_ops->sddmmA(P, P, ones_A, g_A);
        d_ops->sddmmB(P, P, ones_B, g_B);
        VectorXd a_A, a_B = g_B;
        a_B.leakyRelu(leaky_relu_alpha);
        if (softmax_) {
            a_A = g_A;
            a_A.leakyRelu(leaky_relu_alpha);
            d_ops->edgeSoftmax(a_A, k_sddmmA);
            d_ops->edgeSoftmax(a_B, k_sddmmB);
        }
        g_A.leakyReluGrad(leaky_relu_alpha);
        g_B.leakyReluGrad(leaky_relu_alpha);

        // dZ, then de = g o S o (dZ P^T) in both orders: the SDDMM multiplies its dots by SValues = g.  (Not
        // fusedSpMM: the fusion-2 one ignores SValues.)  Softmax attention: dalpha = S o (dZ P^T) in both orders,
        // then de = g o edgeSoftmaxBackward(alpha, dalpha).
        DenseMatrix dZ(P.rows(), P.cols());
        dZ.setMiddleColsReluGrad(G, output, (int64_t)j * layer.features_per_head);
        VectorXd de_A = d_ops->like_S_values(0.0), de_B = d_ops->like_ST_values(0.0);
        if (softmax_) {
            d_ops->sddmmA(dZ, P, ones_A, de_A);
            d_ops->sddmmB(dZ, P, ones_B, de_B);
            d_ops->edgeSoftmaxBackward(a_A, de_A, k_sddmmA);
            d_ops->edgeSoftmaxBackward(a_B, de_B, k_sddmmB);
            scale_in_place(de_A, g_A);
            scale_in_place(de_B, g_B);
        } else {
            d_ops->sddmmA(dZ, P, g_A, de_A);
            d_ops->sddmmB(dZ, P, g_B, de_B);
        }

        // dP = S_de P + S_a^T dZ + S_de^T P (A- and B-shaped rows coincide in every supported layout)
        DenseMatrix dP = d_ops->like_A_matrix(0.0), part = d_ops->like_B_matrix(0.0);
        d_ops->spmmA(dP, P, de_A);
        d_ops->spmmB(dZ, part, a_B);
        dP += part;
        d_ops->spmmB(P, part, de_B);
        dP += part;

        // dW = X^T dP summed over the ranks (each holds its own rows); dX (+)= dP W^T
        DenseMatrix &dW = layer.wGrads.at((size_t)j);
        dW.setTransposeTimes(input, dP);
        allreduce_world(dW);
        dX.setTimesTranspose(dP, W, accumulate);
    }

    // backwardHead with additive attention (see the top of this file)
    void backwardHeadAdditive(int i, int j, const DenseMatrix &G, DenseMatrix &dX, bool accumulate) {
        GATLayer &layer = layers.at((size_t)i);
        const DenseMatrix &input = buffers[(size_t)i], &output = buffers[(size_t)i + 1];
        const DenseMatrix &W = layer.wMats.at((size_t)j);
        d_ops->setRValue(layer.features_per_head);
        cudaStream_t st = hnh::Runtime::get().compute_stream();
        DenseMatrix P = input * W;
        VectorXd s, t;
        node_scalars(layer, j, P, s, t);

        // alpha in both orders, each from s and t
        VectorXd alpha_A = d_ops->like_S_values(0.0), alpha_B = d_ops->like_ST_values(0.0);
        d_ops->additiveScores(s, t, alpha_A, k_sddmmA, leaky_relu_alpha, false);
        d_ops->edgeSoftmax(alpha_A, k_sddmmA);
        d_ops->additiveScores(s, t, alpha_B, k_sddmmB, leaky_relu_alpha, false);
        d_ops->edgeSoftmax(alpha_B, k_sddmmB);

        // de = x' o edgeSoftmaxBackward(alpha, S o (dZ P^T)), A order
        DenseMatrix dZ(P.rows(), P.cols());
        dZ.setMiddleColsReluGrad(G, output, (int64_t)j * layer.features_per_head);
        VectorXd ones_A = d_ops->like_S_values(1.0), de = d_ops->like_S_values(0.0), x_grad = d_ops->like_S_values(0.0);
        d_ops->sddmmA(dZ, P, ones_A, de);
        d_ops->edgeSoftmaxBackward(alpha_A, de, k_sddmmA);
        d_ops->additiveScores(s, t, x_grad, k_sddmmA, leaky_relu_alpha, true);
        scale_in_place(de, x_grad);

        // ds, dt: the row and column sums of de over all ranks, in the node vectors' layout (s and t are done with)
        VectorXd &ds = s, &dt = t;
        d_ops->edgeSums(de, ds, dt);

        // dP = S_alpha^T dZ + ds a1^T + dt a2^T on this rank's rows (A- and B-shaped rows coincide where this runs)
        const int64_t top = d_ops->aSubmatrices.at(0).topRow, off = (int64_t)j * layer.features_per_head;
        DenseMatrix dP = d_ops->like_B_matrix(0.0);
        d_ops->spmmB(dZ, dP, alpha_B);
        hnh::abi_check(hnh_gat_rank2_update_f64(dP.data(), ds.data() + top, dt.data() + top, layer.a1.data() + off,
                                                layer.a2.data() + off, dP.rows(), dP.cols(), st),
                       "gat_rank2_update");

        // [da1 da2] = P^T [ds dt] over this rank's rows, summed over the ranks
        const size_t d = sizeof(double);
        DenseMatrix dst(P.rows(), 2), da(P.cols(), 2);
        hnh::cuda_check(cudaMemcpy2DAsync(dst.data(), 2 * d, ds.data() + top, d, d, (size_t)P.rows(), cudaMemcpyDeviceToDevice, st), "ds column");
        hnh::cuda_check(cudaMemcpy2DAsync(dst.data() + 1, 2 * d, dt.data() + top, d, d, (size_t)P.rows(), cudaMemcpyDeviceToDevice, st), "dt column");
        da.setTransposeTimes(P, dst);
        allreduce_world(da);
        hnh::cuda_check(cudaMemcpy2DAsync(layer.a1Grads.data() + off, d, da.data(), 2 * d, d, (size_t)P.cols(), cudaMemcpyDeviceToDevice, st), "da1");
        hnh::cuda_check(cudaMemcpy2DAsync(layer.a2Grads.data() + off, d, da.data() + 1, 2 * d, d, (size_t)P.cols(), cudaMemcpyDeviceToDevice, st), "da2");

        DenseMatrix &dW = layer.wGrads.at((size_t)j);
        dW.setTransposeTimes(input, dP);
        allreduce_world(dW);
        dX.setTimesTranspose(dP, W, accumulate);
    }

    // backwardHead with GATv2 attention (see the top of this file)
    void backwardHeadGatv2(int i, int j, const DenseMatrix &G, DenseMatrix &dX, bool accumulate) {
        GATLayer &layer = layers.at((size_t)i);
        const DenseMatrix &input = buffers[(size_t)i], &output = buffers[(size_t)i + 1];
        const DenseMatrix &W = layer.wMats.at((size_t)j);
        d_ops->setRValue(layer.features_per_head);
        DenseMatrix P = input * W;
        const VectorXd a = head_vector(layer.a1, layer, j);

        // alpha in both orders, each from its own score pass
        VectorXd alpha_A = d_ops->like_S_values(0.0), alpha_B = d_ops->like_ST_values(0.0);
        d_ops->gatv2Scores(P, P, a, alpha_A, k_sddmmA, leaky_relu_alpha);
        d_ops->edgeSoftmax(alpha_A, k_sddmmA);
        d_ops->gatv2Scores(P, P, a, alpha_B, k_sddmmB, leaky_relu_alpha);
        d_ops->edgeSoftmax(alpha_B, k_sddmmB);

        // de = edgeSoftmaxBackward(alpha, S o (dZ P^T)) in both orders
        DenseMatrix dZ(P.rows(), P.cols());
        dZ.setMiddleColsReluGrad(G, output, (int64_t)j * layer.features_per_head);
        VectorXd ones_A = d_ops->like_S_values(1.0), ones_B = d_ops->like_ST_values(1.0);
        VectorXd de_A = d_ops->like_S_values(0.0), de_B = d_ops->like_ST_values(0.0);
        d_ops->sddmmA(dZ, P, ones_A, de_A);
        d_ops->sddmmB(dZ, P, ones_B, de_B);
        d_ops->edgeSoftmaxBackward(alpha_A, de_A, k_sddmmA);
        d_ops->edgeSoftmaxBackward(alpha_B, de_B, k_sddmmB);

        // dP = S_alpha^T dZ, then the score gradient of both endpoints (P is both of them: shared weights); da
        DenseMatrix dP = d_ops->like_B_matrix(0.0);
        d_ops->spmmB(dZ, dP, alpha_B);
        VectorXd da;
        d_ops->gatv2Backward(P, P, a, de_A, de_B, dP, dP, da, leaky_relu_alpha);
        const int64_t off = (int64_t)j * layer.features_per_head;
        hnh::abi_check(hnh_axpby_f64(layer.a1Grads.data() + off, 1.0, da.data(), 0.0, nullptr, da.size(),
                                     hnh::Runtime::get().compute_stream()),
                       "da");

        DenseMatrix &dW = layer.wGrads.at((size_t)j);
        dW.setTransposeTimes(input, dP);
        allreduce_world(dW);
        dX.setTimesTranspose(dP, W, accumulate);
    }

private:
    string attention_ = "leaky";
    bool softmax_ = false;
    bool additive_ = false;
    bool gatv2_ = false;

    // head j's slice [j * features_per_head, (j + 1) * features_per_head) of an attention vector, as its own vector
    // (copied by a library kernel: the forward pass stays free of direct CUDA runtime calls)
    static VectorXd head_vector(const VectorXd &v, const GATLayer &layer, int j) {
        VectorXd out(layer.features_per_head);
        hnh::abi_check(hnh_axpby_f64(out.data(), 1.0, v.data() + (int64_t)j * layer.features_per_head, 0.0, nullptr,
                                     layer.features_per_head, hnh::Runtime::get().compute_stream()),
                       "attention vector slice");
        return out;
    }

    // Head j's node scalars s = P a1 and t = P a2 as whole node vectors (localArows * p entries, at least M and N;
    // those at or past M are 0): each rank writes its own rows at aSubmatrices[0].topRow into zeros, and a sum
    // all-reduce -- exact, every entry has one contributor -- gives every rank all of them.
    void node_scalars(const GATLayer &layer, int j, const DenseMatrix &P, VectorXd &s, VectorXd &t) {
        const int64_t len = std::max<int64_t>((int64_t)d_ops->localArows * d_ops->p, std::max(d_ops->M, d_ops->N));
        const int64_t top = d_ops->aSubmatrices.at(0).topRow, off = (int64_t)j * layer.features_per_head;
        if (top + P.rows() > len || P.cols() != layer.features_per_head)
            throw hnh::Error(HNH_E_INVALID, "GAT additive attention: the projection does not fit the node vectors");
        s = VectorXd::Constant(len, 0.0);
        t = VectorXd::Constant(len, 0.0);
        hnh::abi_check(hnh_gat_node_scalars_f64(s.data() + top, t.data() + top, P.data(), layer.a1.data() + off,
                                                layer.a2.data() + off, P.rows(), P.cols(), hnh::Runtime::get().compute_stream()),
                       "gat_node_scalars");
        allreduce_world(s);
        allreduce_world(t);
    }

    // v[i] *= s[i]
    static void scale_in_place(VectorXd &v, const VectorXd &s) {
        hnh::abi_check(hnh_hadamard_f64(v.data(), v.data(), s.data(), v.size(), hnh::Runtime::get().compute_stream()), "hadamard");
    }

};
