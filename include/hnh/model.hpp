// hnh/model.hpp -- what GAT, GraphTransformer, GraphSAGE, RGCN, PNA and GIN share, so that one train step
// (hnh/training.hpp) and one driver handle (hnhd_model_t) serve them all: the algorithm object, the activation buffers,
// the input gradient, the staleness flag, and virtual forward, backward, parameter list and parameter lookup; and the
// host helpers several models use.  Host-side dispatch only; the device work of each model is its own.
#pragma once
#include <cstdint>
#include <string>
#include <vector>

#include "hnh/distributed_sparse.h"
#include "hnh/runtime.h"
#include "hnh_b200.h"

// One parameter tensor of a model as the optimizer sees it: n doubles on the device with their gradient
struct ParamSpan {
    double *param;
    const double *grad;  // null before the model's first backward pass
    int64_t n;
};

// One named parameter of one layer: rows x cols doubles, row-major, on the device
struct ParamRef {
    double *value;
    const double *grad;  // null before the model's first backward pass
    int64_t rows, cols;
};

class GraphModel {
public:
    Distributed_Sparse *d_ops;
    vector<DenseMatrix> buffers;  // [0] network input (B-shaped), [i + 1] output of layer i (A-shaped)
    DenseMatrix input_grad;       // dL/d buffers[0] after backwardPass (B-shaped, like buffers[0])
    // The activations in `buffers` belong to the current parameters and input: a forward pass sets it, whoever changes
    // one of them clears it, and backwardPass refuses to run on stale activations.
    bool activations_current = false;
    const string model_name;  // the model's word in error messages

    GraphModel(Distributed_Sparse *ops, const string &name) : d_ops(ops), model_name(name) {}
    virtual ~GraphModel() = default;

    // Collective.  dropout in [0, 1) and seed are the attention dropout of models that have one; the others refuse
    // dropout != 0 with HNH_E_INVALID before any launch.
    virtual void forward(double dropout, uint64_t seed) = 0;
    // output_grad = dL/d buffers.back() (this rank's rows).  Leaves the parameters' gradients (summed over all ranks)
    // and dL/d buffers[0] in input_grad.  Collective.
    virtual void backwardPass(const DenseMatrix &output_grad) = 0;
    // Every parameter with its gradient, in the model's fixed order.  Read afresh for every use: a parameter's storage
    // may be replaced.
    virtual std::vector<ParamSpan> parameters() = 0;
    // Throws HNH_E_INVALID, on every rank alike, where a train step cannot run; called before the step's forward pass.
    virtual void check_trainable() const {}
    // The parameter `name` of `layer`.  Throws HNH_E_INVALID for an unknown layer or name.  The default, GAT's, has no
    // names: its weights and attention vectors are addressed by (layer, head).
    virtual ParamRef param(int, const string &name) {
        throw hnh::Error(HNH_E_INVALID, model_name + ": no parameter \"" + name +
                                            "\" by name: the weights and attention vectors are addressed by (layer, head)");
    }

protected:
    void refuse_dropout(double dropout) const {
        if (dropout != 0.0)
            throw hnh::Error(HNH_E_INVALID, model_name + ": the model has no dropout, got dropout = " + std::to_string(dropout));
    }
    // Edge attributes of S's entries in both value orders, edge_dim wide (row i of host_A / host_B belongs to entry i of
    // like_S_values / like_ST_values; every rank passes its part of the same attributes), uploaded into attr_A / attr_B.
    // Makes the activations stale.  HNH_E_INVALID, `who` first, for a model without edge features (edge_dim = 0) or
    // entry counts that are not this rank's.
    void uploadEdgeAttributes(const string &who, int edge_dim, const double *host_A, int64_t n_A, const double *host_B, int64_t n_B,
                              DenseMatrix &attr_A, DenseMatrix &attr_B) {
        if (edge_dim == 0) throw hnh::Error(HNH_E_INVALID, who + ": the model has no edge features (edge_dim = 0)");
        if (n_A != d_ops->num_S_values() || n_B != d_ops->num_ST_values())
            throw hnh::Error(HNH_E_INVALID, who + ": edge attributes for " + std::to_string(n_A) + " and " + std::to_string(n_B) +
                                                " entries; this rank holds " + std::to_string(d_ops->num_S_values()) + " (A order) and " +
                                                std::to_string(d_ops->num_ST_values()) + " (B order)");
        attr_A = DenseMatrix::from_host(host_A, n_A, edge_dim);
        attr_B = DenseMatrix::from_host(host_B, n_B, edge_dim);
        activations_current = false;
    }
    // [A 1]: the bias gradients are the products with its ones column
    static DenseMatrix with_ones(const DenseMatrix &A) {
        const int64_t n = A.rows(), f = A.cols();
        DenseMatrix Aa = DenseMatrix::Constant(n, f + 1, 1.0);
        const size_t dsz = sizeof(double);
        hnh::cuda_check(cudaMemcpy2DAsync(Aa.data(), (f + 1) * dsz, A.data(), f * dsz, f * dsz, (size_t)n, cudaMemcpyDeviceToDevice,
                                          hnh::Runtime::get().compute_stream()),
                        "[A 1]");
        return Aa;
    }
    // the span of one layer's parameter vector, and a named slice of it
    static ParamSpan span(VectorXd &params, VectorXd &grads) {
        return {params.data(), grads.size() == params.size() ? grads.data() : nullptr, params.size()};
    }
    static ParamRef slice(VectorXd &params, VectorXd &grads, int64_t offset, int64_t rows, int64_t cols) {
        return {params.data() + offset, grads.size() == params.size() ? grads.data() + offset : nullptr, rows, cols};
    }
};
