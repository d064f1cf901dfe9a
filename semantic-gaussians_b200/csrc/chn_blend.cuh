// C-channel blend, "weights once" pipeline (C > 4).
//
// Measured on the K3 scene (1 M Gaussians, 1080p): a tile walks ~280 list entries before all its
// pixels saturate, but only ~115 of them touch any pixel of the tile (the reference bins by the
// 3-sigma square of the major axis, rasterizer_impl.cu:91 / forward.cu:229-235), and the scalar
// alpha / transmittance chain costs about as many issue slots as a 64-channel accumulation.  A
// kernel that fused chain and accumulation per channel chunk would spend most of its instructions
// re-deriving the same weights in every chunk, forward and backward.  Here the chain runs ONCE per
// view:
//
//   alpha_pass        one CTA per tile, thread = pixel: the reference's chain verbatim
//                     (forward.cu:326-363) -> final_T, n_contrib, and for every Gaussian that
//                     touches the tile a 1 KB row of weights w[pixel] = alpha * T (0 where the
//                     pixel skips it) appended to a per-tile linked list of 16-entry chunks.
//   blend_forward     persistent CTAs claim (tile, up to 128 channels) items: a producer warp
//                     streams the tile's 16-entry pool chunks (weight rows and the item's feature
//                     slices, by bulk copy, or staged with cp.async when the feature rows are not
//                     16-byte aligned slices) through one ring, every compute warp owns a 32-pixel
//                     strip and all the item's channels, every lane an 8 px x 16 ch register tile
//                     (setmaxnreg moves the producer group's registers to the compute groups); the
//                     output leaves through shared memory as TMA tensor stores.
//   chain_backward    CTA = tile, warp = 32-pixel strip: s = <feature, dL/dout> per (pixel,
//                     Gaussian) for all channels over the strip's own entries (register
//                     micro-tiles), then the reference's back-to-front chain (backward.cu:477-550)
//                     in dot-product form -> dL/dmean2D, dL/dconic, dL/dopacity.
//   dfeature          persistent CTAs claim (tile, up to 256 channels) items: dL/dfeature[g][ch] =
//                     sum_px w * dL/dout, a producer warp streams 32-pixel weight and dL slabs by TMA
//                     through one ring, every compute warp owns 32 channels of all the tile's entries
//                     (setmaxnreg moves the producer group's registers to them), one 16-byte
//                     reduction per (Gaussian, tile, 4 channels).
//
// Results are unchanged: the integer outputs come from the verbatim chain; every accumulator still
// adds its Gaussians in depth order.
#pragma once
#include "weight_pool.cuh"

namespace sgb {

// ------------------------------------------------------------------------------------ stage launchers
// Each takes the PoolView of its view (weight_pool_settle / weight_rows_for_backward) and looks up nothing.  A batched
// backward runs all dL/dfeature kernels first, records the feature-gradient event, then the chain kernels.
int chn_forward(sgb_ctx* ctx, const ViewState& w, const PoolView& pv, float* out_color, cudaStream_t s);
// dL_dcolors[g][c] += sum_px w * dL_dpix[c][px]; fp32 for a backward, fp32 or fp16 for a lift's feature map
int chn_dfeature(sgb_ctx* ctx, const ViewState& w, const PoolView& pv, const float* dL_dpix, float* dL_dcolors,
                 cudaStream_t s);
int chn_dfeature(sgb_ctx* ctx, const ViewState& w, const PoolView& pv, const __half* dL_dpix, float* dL_dcolors,
                 cudaStream_t s);
int chn_chain(sgb_ctx* ctx, const ViewState& w, const PoolView& pv, const float* dL_dpix, float* dL_dmean2D,
              float* dL_dconic, float* dL_dopacity, cudaStream_t s);

// ------------------------------------------------------------------------------------ GEMM-shaped kernels
// With the weights materialised per tile, the three C-wide contractions are small dense GEMMs over the
// tile's touching Gaussians (G ~ 115 on K3), done in fp32 on the CUDA cores (north_star: no tensor cores;
// the 1e-4 fp32 bar rules out TF32 anyway):
//     forward   out[256 px][128 ch] = W^T[256 px][G]  . F[G][128 ch]     K = G      lane tile 8 px x 16 ch
//     s-pass    S[32 px][32]        = dL[32 px][C]    . F^T[C][32]       K = C      lane tile 8 px x 4 entries
//               (per warp: its strip and a 32-entry segment of the strip's entries)
//     dfeature  dF[G][256 ch]       = W[G][256 px]    . dL[256 px][256]  K = 256 px lane tile <= 8 entries x 16 ch
// Register tiles give every shared-memory load several FMAs and need no cross-lane reductions (a
// shuffle-reduce formulation spends its issue slots on SHFL/FSEL/FADD instead).

// Lane -> operand-group mapping of the register-tiled GEMM loops: a warp-wide LDS.128 costs 2 shared-memory
// wavefronts when every aligned group of 4 lanes reads at most 2 distinct 16-byte chunks and each half-warp at most 8
// (conflict-free) chunks, and 4 wavefronts otherwise.  With the natural split (one operand indexed by lane & 7, the
// other by lane >> 3) the lane & 7 operand pays 4 per load, and the shared-memory pipe rather than the FMA pipe limits
// the contraction kernels.  Giving each operand exactly one of the two low lane bits makes every operand load a
// 2-wavefront load.
__device__ __forceinline__ int lane_group8(int lane) { return (lane & 1) | (((lane >> 2) & 3) << 1); }  // bits 0, 2, 3
__device__ __forceinline__ int lane_group4(int lane) { return ((lane >> 1) & 1) | ((lane >> 4) << 1); } // bits 1, 4

}  // namespace sgb
