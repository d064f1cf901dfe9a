// Launchers of semantic.cu shared with other translation units.
#pragma once
#include <cuda_runtime.h>

namespace sgb {

// out[p][k] = sum_c features[p][c] * text[k][c] (+ kbias[k] when kbias is not NULL) for k < K, row pitch Kpad,
// columns K..Kpad-1 zero.  features (P, C), text (K, C) row-major fp32.  With kbias NULL this is sgb_feature_logits.
int launch_feature_logits(int P, int C, int K, int Kpad, const float* features, const float* text, const float* kbias,
                          float* out, cudaStream_t s);

}  // namespace sgb
