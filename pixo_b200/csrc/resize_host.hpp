// resize_host.hpp — host half of the resizers: pixo's Lanczos3 contribution tables (resize_host.cpp).
#pragma once

#include <stddef.h>
#include <stdint.h>

#include <vector>

namespace pixo {

// f32::sin as pixo's wasm build computes it: the libm port of musl's sinf (see resize_host.cpp)
float resize_sinf(float x);

// precompute_contributions (src/resize.rs:416-456) for one axis: destination index d reads source indices
// start[d] .. start[d] + count[d] - 1 with the normalised weights w[offset[d] ..]
struct ResizeAxis {
    std::vector<uint32_t> start, count;
    std::vector<uint64_t> offset;
    std::vector<float> w;
};
// ranges only (offset and the total number of weights) when weights is false
void resize_axis(uint32_t src_size, uint32_t dst_size, bool weights, ResizeAxis &a);

}  // namespace pixo
