// hnh/world_allreduce.hpp -- the sum all-reduce over the world that the models (GAT, GraphTransformer) apply to their
// weight gradients: in place, stream-ordered on the communication stream between the compute stream's work before
// and after it; nothing at p = 1.  Every rank must call it with the same length.
#pragma once
#include <memory>

#include "hnh/common.h"
#include "hnh/comm.h"
#include "hnh/runtime.h"

inline void allreduce_world(double *p, int64_t n) {
    std::shared_ptr<hnh::Comm> world = hnh::Comm::world();
    if (world->size() == 1) return;
    hnh::Runtime &rt = hnh::Runtime::get();
    rt.chain(rt.compute_stream(), rt.comm_stream());
    world->allreduce_sum_f64(p, (size_t)n, rt.comm_stream());
    rt.chain(rt.comm_stream(), rt.compute_stream());
}
// the element-wise maximum over the world, as allreduce_world (the max readout of hnh/graph_readout.hpp)
inline void allreduce_world_max(double *p, int64_t n) {
    std::shared_ptr<hnh::Comm> world = hnh::Comm::world();
    if (world->size() == 1) return;
    hnh::Runtime &rt = hnh::Runtime::get();
    rt.chain(rt.compute_stream(), rt.comm_stream());
    world->allreduce_max_f64(p, (size_t)n, rt.comm_stream());
    rt.chain(rt.comm_stream(), rt.compute_stream());
}
inline void allreduce_world(DenseMatrix &m) { allreduce_world(m.data(), m.size()); }
inline void allreduce_world(VectorXd &v) { allreduce_world(v.data(), v.size()); }
