// hnh/pna.hpp -- PNA: layers of PyG's PNAConv(f, r, aggregators, scalers, deg, towers = 1, pre_layers = 1,
// post_layers = 1, divide_input = False, edge_dim = None, train_norm = False), forward and backward, with the weight
// gradients summed over all ranks (Corso et al., 2020).
//
// Layer l has input width f and output width r.  With X the layer input, u an S-row and its messages the stored
// entries (u, v) of S on all ranks (duplicates count; deg_u of them):
//     h_uv = [X_u, X_v] W_pre + b_pre = c_u + z_v,   c = X W_pre[0:f] + b_pre,   z = X W_pre[f:2f]
//     agg_a(u) over v of h_uv: mean, sum, min, max, var = mean(h^2) - mean(h)^2, std = sqrt(clamp(var, 1e-5)) set to 0
//              where it is <= sqrt(1e-5) (PyG's StdAggregation); 0 on a row without entries
//     scale_s(u): identity 1, amplification log(d + 1) / delta_log, attenuation delta_log / log(d + 1), linear
//              d / delta_lin, inverse_linear delta_lin / d, with d = max(deg_u, 1)
//     P_u = [X_u | scale_s0(u) [agg_a0(u) .. agg_aA-1(u)] | scale_s1(u) [..] | ..]        ((A S + 1) f wide)
//     Y = (P W_post + b_post) W_lin + b_lin,   X_{l+1} = ReLU(Y) for every layer but the last, which outputs Y
// Since h_uv = c_u + z_v, every aggregate comes from four statistics of z over a row -- sum z, sum z^2, max z and min z
// (var and std are shift-invariant) -- which one Distributed_Sparse::multiAggregate of z gathers, f wide.  The
// degrees come once per model from multiAggregate of a ones column (the moments' sum window).
//
// Backward of layer l, given G = dL/d X_{l+1}:
//     dY = G where X_{l+1} > 0 (G itself for the last layer)
//     dW_lin = Q^T dY, db_lin = 1^T dY, dQ = dY W_lin^T       (Q = P W_post + b_post)
//     dW_post = P^T dQ, db_post = 1^T dQ, dP = dQ W_post^T
//     dc, dS = the gradients of the aggregates through the scalers and the clamp and mask of std (hnh_pna_combine_grad_f64):
//              dc_u = deg_u dSum + dMean + dMax + dMin on rows with entries
//     dz = multiAggregateBackward(z, dS) (ties of min and max share their gradient equally, as maxAggregate)
//     dW_pre = [X^T dc; X^T dz], db_pre = 1^T dc, dX = dP[:, 0:f] + dc W_pre[0:f]^T + dz W_pre[f:2f]^T
// then one sum all-reduce of the layer's gradients (allreduce_world).  The forward keeps z, the statistics, P and Q of
// every layer, so the backward runs no forward sparse pass.
//
// Parameters of a layer live in one device vector, in the order of its gradients: W_pre (2f x f), b_pre (f), W_post
// ((A S + 1) f x r), b_post (r), W_lin (r x r), b_lin (r).  All are zero after construction.  Weights are stored
// input-major: a PNAConv state dict maps onto them as pre_nns.0.0.weight.T, pre_nns.0.0.bias, post_nns.0.0.weight.T,
// post_nns.0.0.bias, lin.weight.T and lin.bias.
//
// Defined where Distributed_Sparse::check_full_rows passes (every rank holds full-width rows and the A and B layouts
// coincide); elsewhere the constructor throws HNH_E_INVALID on every rank before any launch.
#pragma once
#include <cmath>
#include <cstring>
#include <string>
#include <vector>

#include "hnh/comm.h"
#include "hnh/distributed_sparse.h"
#include "hnh/graph_readout.hpp"
#include "hnh/model.hpp"
#include "hnh/world_allreduce.hpp"
#include "hnh_b200.h"

class PNALayer {
public:
    int input_features;
    int output_features;

    VectorXd params;  // the layout above; zero after construction
    VectorXd grads;   // the same layout: dL/d params after PNA::backwardPass (same on every rank)

    PNALayer(int in_width, int out_width) : input_features(in_width), output_features(out_width) {}
};

class PNA : public GraphModel {
public:
    vector<PNALayer> layers;
    vector<int> aggregators, scalers;  // HNH_PNA_* codes, in the user's order
    const double avg_deg_lin, avg_deg_log;
    // what the backward needs, per layer, from the last forward pass: z, the statistics of z, P and Q = P W_post + b_post
    vector<DenseMatrix> zs, stats, Ps, Qs;

    // aggregators: a comma-separated list of mean, sum, min, max, var, std; scalers: of identity, amplification,
    // attenuation, linear, inverse_linear.  avg_deg_lin / avg_deg_log: PyG's averages of d and log(d + 1) over the
    // training degree histogram, finite and > 0 where a scaler reads them, and never NaN (the Python front end passes NaN
    // for a histogram it refuses, so that every rank refuses together).  Collective: every rank checks its arguments
    // and one host all-reduce makes every rank refuse when any rank's are bad or differ from the others'.
    PNA(vector<PNALayer> &l_input, Distributed_Sparse *ops, const string &aggregator_list, const string &scaler_list, double delta_lin,
        double delta_log)
        : GraphModel(ops, "PNA"), layers(l_input), avg_deg_lin(delta_lin), avg_deg_log(delta_log) {
        d_ops->check_full_rows("PNA");
        vector<LayerWidths> widths;
        for (const PNALayer &l : layers)
            widths.push_back({l.input_features, l.output_features, l.input_features > 0 && l.output_features > 0});
        string problem;
        try {
            aggregators = parse_codes(aggregator_list, kAggregators, 6);
            scalers = parse_codes(scaler_list, kScalers, 5);
            problem = check_arguments(widths);
        } catch (const hnh::Error &e) {
            problem = e.what();
        }
        // every rank refuses alike: its own problem, another rank's, or arguments that differ between ranks (the sums
        // of the values and of their squares agree only where every rank holds the same values)
        const bool ok = problem.empty();
        const std::vector<double> x = hnh::detail::agreement_sums(
            !ok, {ok ? packed(aggregators) : 0u, ok ? packed(scalers) : 0u, ok && uses_lin() ? bits(avg_deg_lin) : 0,
                  ok && uses_log() ? bits(avg_deg_log) : 0});
        if (!ok) throw hnh::Error(HNH_E_INVALID, "PNA: " + problem);
        if (x[0] != 0.0) throw hnh::Error(HNH_E_INVALID, "PNA: another rank's arguments are bad");
        if (!hnh::detail::agree(x))
            throw hnh::Error(HNH_E_INVALID, "PNA: the aggregators, scalers or degree averages differ between ranks");
        allocate_buffers(widths);
        for (PNALayer &layer : layers) layer.params = VectorXd::Constant(param_count(layer), 0.0);
        // deg_u over all ranks: the sum window of a ones column
        DenseMatrix ones = DenseMatrix::Constant(d_ops->localBrows, 1, 1.0);
        degree.resize(d_ops->localArows, 2);
        d_ops->multiAggregate(ones, degree, HNH_MULTI_MOMENTS);
        row_ones = DenseMatrix::Constant(d_ops->localArows, 1, 1.0);
    }

    static constexpr const char *kAggregators[6] = {"mean", "sum", "min", "max", "var", "std"};
    static constexpr const char *kScalers[5] = {"identity", "amplification", "attenuation", "linear", "inverse_linear"};

    // the codes of a comma-separated list; an empty list, an unknown name or a repeated one throws HNH_E_INVALID
    static vector<int> parse_codes(const string &list, const char *const *names, int count) {
        vector<int> out;
        size_t start = 0;
        while (start <= list.size()) {
            const size_t end = std::min(list.find(',', start), list.size());
            const string name = list.substr(start, end - start);
            int code = -1;
            for (int i = 0; i < count; i++)
                if (name == names[i]) code = i;
            string known;
            for (int i = 0; i < count; i++) known += (i ? ", " : "") + string(names[i]);
            if (code < 0) throw hnh::Error(HNH_E_INVALID, "unknown name \"" + name + "\" in \"" + list + "\" (" + known + ")");
            for (int c : out)
                if (c == code) throw hnh::Error(HNH_E_INVALID, "\"" + name + "\" appears twice in \"" + list + "\"");
            out.push_back(code);
            start = end + 1;
        }
        return out;
    }

    int64_t post_rows(const PNALayer &l) const { return ((int64_t)aggregators.size() * scalers.size() + 1) * l.input_features; }
    int64_t param_count(const PNALayer &l) const {
        const int64_t f = l.input_features, r = l.output_features;
        return (2 * f + 1) * f + (post_rows(l) + 1) * r + (r + 1) * r;
    }
    // the offsets of the six parameters in a layer's vector
    int64_t off_pre_bias(const PNALayer &l) const { return 2 * (int64_t)l.input_features * l.input_features; }
    int64_t off_post(const PNALayer &l) const { return off_pre_bias(l) + l.input_features; }
    int64_t off_post_bias(const PNALayer &l) const { return off_post(l) + post_rows(l) * l.output_features; }
    int64_t off_lin(const PNALayer &l) const { return off_post_bias(l) + l.output_features; }
    int64_t off_lin_bias(const PNALayer &l) const { return off_lin(l) + (int64_t)l.output_features * l.output_features; }

    // Each layer's params with its grads, one span per layer
    std::vector<ParamSpan> parameters() override { return layer_spans(layers); }

    // By name (the layout above): "pre" (2f x f), "pre_bias" (f x 1), "post" ((A S + 1) f x r), "post_bias" (r x 1),
    // "lin" (r x r), "lin_bias" (r x 1)
    ParamRef param(int layer, const string &name) override {
        if (layer < 0 || layer >= (int)layers.size()) throw hnh::Error(HNH_E_INVALID, "PNA: no such layer");
        PNALayer &l = layers[(size_t)layer];
        const int64_t f = l.input_features, r = l.output_features;
        if (name == "pre") return slice(l.params, l.grads, 0, 2 * f, f);
        if (name == "pre_bias") return slice(l.params, l.grads, off_pre_bias(l), f, 1);
        if (name == "post") return slice(l.params, l.grads, off_post(l), post_rows(l), r);
        if (name == "post_bias") return slice(l.params, l.grads, off_post_bias(l), r, 1);
        if (name == "lin") return slice(l.params, l.grads, off_lin(l), r, r);
        if (name == "lin_bias") return slice(l.params, l.grads, off_lin_bias(l), r, 1);
        throw hnh::Error(HNH_E_INVALID, "PNA: no parameter \"" + name + "\" (pre, pre_bias, post, post_bias, lin or lin_bias)");
    }

    // Collective.
    void forwardPass() {
        d_ops->check_full_rows("PNA::forwardPass");
        zs.resize(layers.size());
        stats.resize(layers.size());
        Ps.resize(layers.size());
        Qs.resize(layers.size());
        const int which = statistics();
        for (size_t i = 0; i < layers.size(); i++) {
            PNALayer &l = layers[i];
            DenseMatrix &X = buffers[i];
            const int64_t n = X.rows(), f = l.input_features;
            DenseMatrix c = X * view(l.params, 0, f, f);
            hnh::abi_check(hnh_row_bias_add_f64(c.data(), l.params.data() + off_pre_bias(l), n, f, stream()), "row_bias_add");
            zs[i] = X * view(l.params, f * f, f, f);
            stats[i].resize(d_ops->localArows, state_width(f));
            d_ops->multiAggregate(zs[i], stats[i], which);
            Ps[i].resize(n, post_rows(l));
            hnh::abi_check(hnh_pna_combine_f64(X.data(), f, c.data(), f, stats[i].data(), stats[i].cols(), which, degree.data(), 2, n, (int)f,
                                               packed(aggregators), (int)aggregators.size(), packed(scalers), (int)scalers.size(),
                                               avg_deg_lin, avg_deg_log, Ps[i].data(), Ps[i].cols(), stream()),
                           "pna_combine");
            Qs[i] = Ps[i] * view(l.params, off_post(l), post_rows(l), l.output_features);
            hnh::abi_check(hnh_row_bias_add_f64(Qs[i].data(), l.params.data() + off_post_bias(l), n, l.output_features, stream()),
                           "row_bias_add");
            DenseMatrix Y = Qs[i] * view(l.params, off_lin(l), l.output_features, l.output_features);
            hnh::abi_check(hnh_row_bias_add_f64(Y.data(), l.params.data() + off_lin_bias(l), n, l.output_features, stream()),
                           "row_bias_add");
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
        d_ops->check_full_rows("PNA::backwardPass");
        check_backward("PNA::backwardPass", "the parameters or the input", output_grad);
        backward_layers(output_grad, [&](int i, const DenseMatrix &G, DenseMatrix &dX) { backwardLayer(i, G, dX); });
    }

private:
    DenseMatrix degree;    // localArows x 2: deg_u over all ranks in column 0 (the moments of a ones column)
    DenseMatrix row_ones;  // localArows x 1 ones: the bias gradients are products with it

    static DenseMatrix view(VectorXd &v, int64_t offset, int64_t rows, int64_t cols) {
        return DenseMatrix::view(v.data() + offset, rows, cols);
    }
    static uint64_t bits(double v) {
        uint64_t b;
        std::memcpy(&b, &v, sizeof b);
        return b;
    }
    static unsigned packed(const vector<int> &codes) {
        unsigned p = 0;
        for (size_t i = 0; i < codes.size(); i++) p |= (unsigned)codes[i] << (4 * i);
        return p;
    }
    bool has_scaler(int code) const {
        for (int s : scalers)
            if (s == code) return true;
        return false;
    }
    bool uses_lin() const { return has_scaler(HNH_PNA_LINEAR) || has_scaler(HNH_PNA_INVERSE_LINEAR); }
    bool uses_log() const { return has_scaler(HNH_PNA_AMPLIFICATION) || has_scaler(HNH_PNA_ATTENUATION); }
    // the statistics of z the aggregators need
    int statistics() const {
        int which = 0;
        for (int a : aggregators)
            which |= a == HNH_PNA_MIN ? HNH_MULTI_MIN : a == HNH_PNA_MAX ? HNH_MULTI_MAX : HNH_MULTI_MOMENTS;
        return which;
    }
    int64_t state_width(int64_t f) const {
        const int w = statistics();
        return 2 * f * (((w & HNH_MULTI_MOMENTS) != 0) + ((w & HNH_MULTI_MAX) != 0) + ((w & HNH_MULTI_MIN) != 0));
    }

    // "" or what is wrong with this rank's arguments; widths are the layers'
    string check_arguments(const vector<LayerWidths> &widths) const {
        if (layers.empty()) return "no layers";
        const string chain = layer_chain_problem(widths, nullptr, [&](size_t i) -> string {
            if (post_rows(layers[i]) >= INT32_MAX || state_width(layers[i].input_features) >= INT32_MAX)
                return "layer " + std::to_string(i) + ": (A S + 1) f must be below 2^31";
            return "";
        });
        if (!chain.empty()) return chain;
        if (const string rows = rows_problem(); !rows.empty()) return rows;
        if (std::isnan(avg_deg_lin) || std::isnan(avg_deg_log)) return "a degree average is NaN: the degree histogram was refused";
        if (uses_lin() && !(std::isfinite(avg_deg_lin) && avg_deg_lin > 0.0))
            return "the average degree delta_lin = " + std::to_string(avg_deg_lin) + " must be finite and > 0";
        if (uses_log() && !(std::isfinite(avg_deg_log) && avg_deg_log > 0.0))
            return "the average log-degree delta_log = " + std::to_string(avg_deg_log) + " must be finite and > 0";
        return "";
    }

    // layer i: G = dL/d buffers[i + 1]; writes layers[i].grads and dX = dL/d buffers[i]
    void backwardLayer(int i, const DenseMatrix &G, DenseMatrix &dX) {
        PNALayer &l = layers[(size_t)i];
        DenseMatrix &X = buffers[(size_t)i];
        const int64_t n = G.rows(), f = l.input_features, r = l.output_features, pw = post_rows(l);
        const int which = statistics();
        if (l.grads.size() != l.params.size()) l.grads = VectorXd(l.params.size());
        DenseMatrix dY_relu;
        const DenseMatrix &dY = relu_grad_unless_last(i, G, dY_relu);
        view(l.grads, off_lin(l), r, r).setTransposeTimes(Qs[(size_t)i], dY);
        view(l.grads, off_lin_bias(l), 1, r).setTransposeTimes(row_ones, dY);
        DenseMatrix dQ;
        dQ.setTimesTranspose(dY, view(l.params, off_lin(l), r, r), false);
        view(l.grads, off_post(l), pw, r).setTransposeTimes(Ps[(size_t)i], dQ);
        view(l.grads, off_post_bias(l), 1, r).setTransposeTimes(row_ones, dQ);
        DenseMatrix dP;
        dP.setTimesTranspose(dQ, view(l.params, off_post(l), pw, r), false);
        DenseMatrix &S = stats[(size_t)i];
        DenseMatrix dc(n, f), dS(S.rows(), S.cols());
        hnh::abi_check(hnh_pna_combine_grad_f64(dP.data(), pw, S.data(), S.cols(), which, degree.data(), 2, n, (int)f, packed(aggregators),
                                                (int)aggregators.size(), packed(scalers), (int)scalers.size(), avg_deg_lin, avg_deg_log,
                                                dc.data(), f, dS.data(), dS.cols(), stream()),
                       "pna_combine_grad");
        DenseMatrix dz(n, f);
        d_ops->multiAggregateBackward(zs[(size_t)i], S, dS, dz, which, false);
        view(l.grads, 0, f, f).setTransposeTimes(X, dc);
        view(l.grads, f * f, f, f).setTransposeTimes(X, dz);
        view(l.grads, off_pre_bias(l), 1, f).setTransposeTimes(row_ones, dc);
        // dX = dP[:, 0:f] + dc W_pre[0:f]^T + dz W_pre[f:2f]^T
        dX.resize(n, f);
        const size_t d = sizeof(double);
        hnh::cuda_check(cudaMemcpy2DAsync(dX.data(), f * d, dP.data(), pw * d, f * d, (size_t)n, cudaMemcpyDeviceToDevice, stream()),
                        "dP[:, 0:f]");
        dX.setTimesTranspose(dc, view(l.params, 0, f, f), true);
        dX.setTimesTranspose(dz, view(l.params, f * f, f, f), true);
        allreduce_world(l.grads);
    }
};
