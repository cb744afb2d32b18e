// hnh/model.hpp -- what GAT, GraphTransformer, GraphSAGE, RGCN, PNA and GIN share, so that one train step
// (hnh/training.hpp) and one driver handle (hnhd_model_t) serve them all: the algorithm object, the activation buffers,
// the input gradient, the staleness flag, and virtual forward, backward, parameter list and parameter lookup; and the
// host helpers several models use.  Host-side dispatch only; the device work of each model is its own.
#pragma once
#include <cstdint>
#include <functional>
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
    // One layer of a stack as layer_chain_problem and allocate_buffers see it: its input and output widths, and whether
    // every size the layer is built from is positive
    struct LayerWidths {
        int64_t in, out;
        bool positive;
    };

    static cudaStream_t stream() { return hnh::Runtime::get().compute_stream(); }

    // HNH_E_INVALID "<who>: <problem>" unless problem is ""
    static void refuse(const string &who, const string &problem) {
        if (!problem.empty()) throw hnh::Error(HNH_E_INVALID, who + ": " + problem);
    }
    // "" or the first fault of a stack of layers, without the model's prefix.  Layer by layer: a size that is not
    // positive, then before_chain(i), then an input width other than the output width of layer i - 1, then
    // after_chain(i); the two are a model's own checks of layer i, "" or the fault.
    static string layer_chain_problem(const vector<LayerWidths> &widths, const std::function<string(size_t)> &before_chain = nullptr,
                                      const std::function<string(size_t)> &after_chain = nullptr) {
        for (size_t i = 0; i < widths.size(); i++) {
            if (!widths[i].positive) return "layer " + std::to_string(i) + ": sizes must be positive";
            if (const string p = before_chain ? before_chain(i) : ""; !p.empty()) return p;
            if (i > 0 && widths[i].in != widths[i - 1].out)
                return "layer " + std::to_string(i) + " does not take the width layer " + std::to_string(i - 1) + " produces";
            if (const string p = after_chain ? after_chain(i) : ""; !p.empty()) return p;
        }
        return "";
    }
    // "" or "the A and B layouts hold different rows": the models combine A-shaped and B-shaped matrices row by row
    string rows_problem() const { return d_ops->localArows != d_ops->localBrows ? "the A and B layouts hold different rows" : ""; }
    // buffers[0] B-shaped at the first layer's input width, then one A-shaped buffer per layer at its output width
    void allocate_buffers(const vector<LayerWidths> &widths) {
        d_ops->setRValue((int)widths.front().in);
        buffers.push_back(d_ops->like_B_matrix(0.0));
        for (const LayerWidths &w : widths) {
            d_ops->setRValue((int)w.out);
            buffers.push_back(d_ops->like_A_matrix(0.0));
        }
    }
    // buffers[i + 1] = ReLU(Y), or Y itself (its storage taken) for the last layer
    void set_layer_output(size_t i, DenseMatrix &Y) {
        if (i + 2 < buffers.size())
            buffers[i + 1].setMiddleColsRelu(0, Y);
        else
            buffers[i + 1].take(Y);
    }

    // What every backwardPass refuses before any launch, `who` first: activations from before a change of
    // `what_changed`, and an output gradient of another shape than the network output
    void check_backward(const string &who, const string &what_changed, const DenseMatrix &output_grad) const {
        if (!activations_current) throw hnh::Error(HNH_E_INVALID, who + ": no forward pass since " + what_changed + " changed");
        const DenseMatrix &out = buffers.back();
        if (output_grad.rows() != out.rows() || output_grad.cols() != out.cols())
            throw hnh::Error(HNH_E_INVALID, who + ": the output gradient is " + std::to_string(output_grad.rows()) + " x " +
                                                std::to_string(output_grad.cols()) + ", the network output " + std::to_string(out.rows()) +
                                                " x " + std::to_string(out.cols()));
    }
    // The layers' backward passes, last to first: layer(i, G, dX) is given G = dL/d buffers[i + 1] (output_grad for the
    // last layer) and writes dX = dL/d buffers[i] (input_grad for layer 0).  Two layer gradients are live at a time:
    // that of the layer's output (upstream) and that of its input.
    template <class F>
    void backward_layers(const DenseMatrix &output_grad, F layer) {
        DenseMatrix upstream;
        for (int i = (int)buffers.size() - 2; i >= 0; i--) {
            const DenseMatrix &G = i + 2 == (int)buffers.size() ? output_grad : upstream;
            DenseMatrix downstream;
            layer(i, G, i == 0 ? input_grad : downstream);
            if (i > 0) upstream = std::move(downstream);
        }
    }
    // dY of layer i from G = dL/d buffers[i + 1]: G where buffers[i + 1] > 0, written into storage, or G itself for the
    // last layer, whose output has no ReLU
    const DenseMatrix &relu_grad_unless_last(int i, const DenseMatrix &G, DenseMatrix &storage) const {
        if (i + 2 == (int)buffers.size()) return G;
        storage.resize(G.rows(), G.cols());
        storage.setMiddleColsReluGrad(G, buffers[(size_t)i + 1], 0);
        return storage;
    }

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
        hnh::cuda_check(cudaMemcpy2DAsync(Aa.data(), (f + 1) * dsz, A.data(), f * dsz, f * dsz, (size_t)n, cudaMemcpyDeviceToDevice, stream()),
                        "[A 1]");
        return Aa;
    }
    // one span per layer: each layer's params with its grads
    template <class Layer>
    static std::vector<ParamSpan> layer_spans(vector<Layer> &layers) {
        std::vector<ParamSpan> s;
        for (Layer &l : layers) s.push_back({l.params.data(), l.grads.size() == l.params.size() ? l.grads.data() : nullptr, l.params.size()});
        return s;
    }
    // a named slice of one layer's parameter vector
    static ParamRef slice(VectorXd &params, VectorXd &grads, int64_t offset, int64_t rows, int64_t cols) {
        return {params.data() + offset, grads.size() == params.size() ? grads.data() + offset : nullptr, rows, cols};
    }
};
