// hnh/model.hpp -- what GAT, GraphTransformer, GraphSAGE and RGCN share, so that one train step (hnh/training.hpp) and
// one driver handle (hnhd_model_t) serve them all: the algorithm object, the activation buffers, the input gradient,
// the staleness flag, and virtual forward, backward, parameter list and parameter lookup.  Host-side dispatch only; the
// device work of each model is its own.
#pragma once
#include <cstdint>
#include <string>
#include <vector>

#include "hnh/distributed_sparse.h"
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
    // the span of one layer's parameter vector, and a named slice of it
    static ParamSpan span(VectorXd &params, VectorXd &grads) {
        return {params.data(), grads.size() == params.size() ? grads.data() : nullptr, params.size()};
    }
    static ParamRef slice(VectorXd &params, VectorXd &grads, int64_t offset, int64_t rows, int64_t cols) {
        return {params.data() + offset, grads.size() == params.size() ? grads.data() + offset : nullptr, rows, cols};
    }
};
