// mix64.cuh -- the splitmix64 finaliser, the one hash of the device code: the seeded Erdos-Renyi draws of
// device_setup.cu and the attention-dropout mask of sparse_attention.cu (include/hnh_b200.h states both recipes).
// host_setup.cpp, plain C++, keeps its own copy.
#pragma once
#include <cstdint>

namespace {

__host__ __device__ inline uint64_t mix64(uint64_t z) {
    z += 0x9E3779B97F4A7C15ull;
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    return z ^ (z >> 31);
}

}  // namespace
