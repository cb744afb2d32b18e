// dmma.cuh -- the fp64 tensor-core instruction (mma.sync m8n8k4, DMMA) of the GEMMs in gat_kernels.cu and the ranking
// kernels in link_ranking.cu.  Fragment layout (PTX ISA), with g = lane / 4 and t = lane % 4: a = A[g][t], b = B[t][g],
// and the accumulators c0 = C[g][2t], c1 = C[g][2t + 1].  Hopper's wgmma has no fp64 kind, so this is the fp64 tensor
// path on sm_90a.
#pragma once

namespace {

__device__ __forceinline__ void dmma_8x8x4(double &c0, double &c1, double a, double b) {
    asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};"
                 : "+d"(c0), "+d"(c1)
                 : "d"(a), "d"(b));
}

}  // namespace
