// What the fp32 (sparse_conv.cu) and half-precision (sparse_conv_half.cu) products of the sparse 3D convolution share:
// the host copy of a kernel map's offsets, their argument checks, and the chunking and chunk-order reduction of the
// weight gradient.
#pragma once

#include "common.cuh"

namespace sgb {

constexpr long long kChunk = 2048;     // pairs per weight-gradient partial

struct ConvOffsets {
    long long at[SGB_SPARSE_MAX_K + 1];
};

// Which (offset, first pair, end) chunk c is.  K <= SGB_SPARSE_MAX_K; one short loop per CTA.
__device__ __forceinline__ int chunk_of(const ConvOffsets& off, int K, long long c, long long& p0, long long& p1) {
    for (int d = 0; d < K; d++) {
        const long long n = off.at[d + 1] - off.at[d];
        const long long nc = (n + kChunk - 1) / kChunk;
        if (c < nc) {
            p0 = off.at[d] + c * kChunk;
            p1 = min(p0 + kChunk, off.at[d + 1]);
            return d;
        }
        c -= nc;
    }
    return -1;
}

long long total_chunks(const ConvOffsets& off, int K);

// Validates K, the channel counts and the offsets, and copies the offsets.
int check_offsets(const char* fn, int32_t K, const int64_t* offsets_host, int32_t C_in, int32_t C_out,
                  ConvOffsets& off);

// check_offsets, the row counts, and the pairs (which may be null only when there are none).
int check_conv_args(const char* fn, int32_t K, const int64_t* offsets_host, const int32_t* pairs, int64_t n_in,
                    int32_t C_in, int64_t n_out, int32_t C_out, ConvOffsets& off);

// dW[d] (C_in x C_out, fp32) = sum of offset d's chunk partials (CC = C_in * C_out floats each, chunks in the order of
// chunk_of) in chunk order; 0 for an offset without pairs.
int launch_wgrad_reduce(const ConvOffsets& off, int K, long long CC, const float* partial, float* dW,
                        cudaStream_t s);

}  // namespace sgb
