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
// The forward pass is the GAT formula only where every rank holds full-width rows and the A and B layouts coincide:
// p = 1 (any algorithm), 1.5D dense shift with replication reuse (fusion 1) at any c, and with local kernel fusion
// (fusion 2) at c = 1.  Only there is the backward defined; elsewhere backwardPass throws HNH_E_INVALID on every rank.
#pragma once
#include <string>
#include <vector>

#include "hnh/15D_dense_shift.hpp"
#include "hnh/distributed_sparse.h"
#include "hnh_b200.h"

class GATLayer {
public:
    int input_features;
    int features_per_head;
    int num_heads;

    vector<DenseMatrix> wMats;  // one input_width x head_width projection per head
    vector<DenseMatrix> wGrads; // dL/d wMats[j] after GAT::backwardPass (empty before the first one); same on every rank
    VectorXd a1;                // attention vectors: declared by the reference, unused by its forward pass
    VectorXd a2;

    GATLayer(int in_width, int head_width, int heads)
        : input_features(in_width), features_per_head(head_width), num_heads(heads) {}
    int output_features() const { return features_per_head * num_heads; }
};

class GAT {
public:
    Distributed_Sparse *d_ops;
    vector<GATLayer> layers;
    vector<DenseMatrix> buffers;  // [0] network input (B-shaped), [i + 1] output of layer i (A-shaped)
    double leaky_relu_alpha = 0.2;

    GAT(vector<GATLayer> &l_input, Distributed_Sparse *ops) : d_ops(ops), layers(l_input) {
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
        }
    }

    // head j of layer i: reads buffers[i], writes its column window of buffers[i + 1]
    void computeSelfAttentionHead(int i, int j) {
        GATLayer &layer = layers.at((size_t)i);
        DenseMatrix &input = buffers[(size_t)i], &output = buffers[(size_t)i + 1];
        d_ops->setRValue(layer.features_per_head);

        DenseMatrix projected = input * layer.wMats.at((size_t)j);
        DenseMatrix neighbours = projected;  // the same projection in the role of the other SDDMM operand
        d_ops->de_shift(&neighbours, nullptr, k_spmmA);

        VectorXd pattern = d_ops->like_S_values(1.0);
        VectorXd scores = d_ops->like_S_values(1.0);
        d_ops->algorithm(projected, neighbours, pattern, &scores, k_sddmmA, true);
        scores.leakyRelu(leaky_relu_alpha);

        projected.setZero();  // becomes the SpMM accumulator
        d_ops->algorithm(projected, neighbours, scores, nullptr, k_spmmA, false);
        output.setMiddleColsRelu((int64_t)j * projected.cols(), projected);
    }

    void forwardPass() {
        for (size_t i = 0; i < layers.size(); i++)
            for (int j = 0; j < layers[i].num_heads; j++) computeSelfAttentionHead((int)i, j);
        activations_current = true;
    }

    // ---- backward pass -------------------------------------------------------------------------------
    DenseMatrix input_grad;  // dL/d buffers[0] after backwardPass (B-shaped, like buffers[0])
    // The activations in `buffers` belong to the current wMats and input.  forwardPass sets it; whoever changes
    // wMats or buffers[0] clears it (the driver ABI does), and backwardPass refuses to run on stale activations.
    bool activations_current = false;

    // Throws HNH_E_INVALID unless the backward pass is defined on this algorithm object (see the top of this
    // file).  Decided from global quantities only, so every rank throws together and no collective is left waiting.
    void check_backward_supported() const {
        const string where = d_ops->algorithm_name + " at p = " + std::to_string(d_ops->p) + ", c = " +
                             std::to_string(d_ops->c);
        if (d_ops->p == 1) return;
        if (d_ops->r_split)
            throw hnh::Error(HNH_E_INVALID, "GAT::backwardPass: not defined for " + where +
                                                ": the layout splits the dense operands along R");
        const Sparse15D_Dense_Shift *dense_shift = dynamic_cast<const Sparse15D_Dense_Shift *>(d_ops);
        if (dense_shift == nullptr)
            throw hnh::Error(HNH_E_INVALID, "GAT::backwardPass: not defined for " + where);
        if (dense_shift->fusionApproach == 2 && d_ops->c > 1)
            throw hnh::Error(HNH_E_INVALID, "GAT::backwardPass: not defined for " + where +
                                                " with local kernel fusion (fusion 2): the forward SpMM accumulates "
                                                "onto the gathered projection when c > 1");
    }

    // output_grad = dL/d buffers.back() (this rank's rows).  Leaves dL/d wMats in layers[i].wGrads (summed over all
    // ranks: identical everywhere) and dL/d buffers[0] in input_grad.  Collective.  Reads buffers, wMats and
    // leaky_relu_alpha and changes none of them; gradient storage is allocated on the first call.
    void backwardPass(const DenseMatrix &output_grad) {
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
        GATLayer &layer = layers.at((size_t)i);
        const DenseMatrix &input = buffers[(size_t)i], &output = buffers[(size_t)i + 1];
        const DenseMatrix &W = layer.wMats.at((size_t)j);
        d_ops->setRValue(layer.features_per_head);
        // In every supported layout initial_shift / de_shift are identities, and the SDDMMs only read their operands,
        // so P serves as both of them.
        DenseMatrix P = input * W;

        // attention scores in both value orders; g = LeakyReLU'(e) (A order, B order), a = LeakyReLU(e) (B order)
        VectorXd ones_A = d_ops->like_S_values(1.0), ones_B = d_ops->like_ST_values(1.0);
        VectorXd g_A = d_ops->like_S_values(0.0), g_B = d_ops->like_ST_values(0.0);
        d_ops->sddmmA(P, P, ones_A, g_A);
        d_ops->sddmmB(P, P, ones_B, g_B);
        VectorXd a_B = g_B;
        a_B.leakyRelu(leaky_relu_alpha);
        g_A.leakyReluGrad(leaky_relu_alpha);
        g_B.leakyReluGrad(leaky_relu_alpha);

        // dZ, then de = g o S o (dZ P^T) in both orders: the SDDMM multiplies its dots by SValues = g.  (Not
        // fusedSpMM: the fusion-2 one ignores SValues.)
        DenseMatrix dZ(P.rows(), P.cols());
        dZ.setMiddleColsReluGrad(G, output, (int64_t)j * layer.features_per_head);
        VectorXd de_A = d_ops->like_S_values(0.0), de_B = d_ops->like_ST_values(0.0);
        d_ops->sddmmA(dZ, P, g_A, de_A);
        d_ops->sddmmB(dZ, P, g_B, de_B);

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

private:
    static void allreduce_world(DenseMatrix &m) {
        std::shared_ptr<hnh::Comm> world = hnh::Comm::world();
        if (world->size() == 1) return;
        hnh::Runtime &rt = hnh::Runtime::get();
        rt.chain(rt.compute_stream(), rt.comm_stream());
        world->allreduce_sum_f64(m.data(), (size_t)m.size(), rt.comm_stream());
        rt.chain(rt.comm_stream(), rt.compute_stream());
    }
};
