// Pieces of the feature-map distillation loss (feature_loss.cu) that the decoded-feature loss (decoder_loss.cu)
// shares.
#pragma once

#include "common.cuh"

namespace sgb {

// valid[0] += number of pixels of the (C, N) planar target whose column has a non-zero element (the cosine loss's
// Nv).  `valid` must hold 0 (or a count to add to) in stream order before the call.  T = float or __half.
template <typename T>
int count_valid_pixels(int C, long long N, const T* target, double* valid, cudaStream_t s);

}  // namespace sgb
