// Persistent warp-specialised kernels (chn_forward.cu, chn_dfeature.cu): the mbarrier ring between the producer warp
// and the compute warps, register rebalancing, the work claim and the launch.
#pragma once
#include "common.cuh"
#include "tma.cuh"

namespace sgb {

// Ring of S stages from one producer warp to the consumer warps of a CTA: per stage a header and a full / empty
// mbarrier pair.  Each side counts its steps from 0; step k uses stage k % S for the (k / S)-th time.  The producer's
// acquire(k) waits until every consumer warp released the stage's previous use; the warp then writes hdr[stage],
// issues the copies and arms full[stage]: lane 0 arrives with the transaction bytes and, if init got lanes_arrive,
// every lane arrives once more for what it staged itself (cp.async or plain stores).  A consumer warp's wait(k)
// returns when full[stage] completes, and release(stage) is its one arrival on empty[stage].  finish(k) is the
// producer's last step: a header with `end` set, on which every consumer warp leaves.  There is no CTA-wide barrier
// after the set-up, so a step sequence the two sides do not share leaves a wait unsatisfied: mbar_wait traps.
template <int S, typename Hdr>
struct MbarRing {
    Hdr hdr[S];  // Hdr has an `int end`
    uint64_t full[S], empty[S];
    // one thread, before the CTA's first barrier
    __device__ __forceinline__ void init(bool lanes_arrive, uint32_t consumer_warps) {
        for (int i = 0; i < S; i++) {
            mbar_init(&full[i], lanes_arrive ? 33 : 1);
            mbar_init(&empty[i], consumer_warps);
        }
        mbar_fence_init();
    }
    __device__ __forceinline__ int acquire(uint32_t step) {
        const int st = (int)(step % S);
        if (step >= S) mbar_wait(&empty[st], ((step / S) - 1) & 1u);
        return st;
    }
    __device__ __forceinline__ int wait(uint32_t step) {
        const int st = (int)(step % S);
        mbar_wait(&full[st], (step / S) & 1u);
        return st;
    }
    __device__ __forceinline__ void release(int st, int lane) {
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty[st]);
    }
    __device__ __forceinline__ void finish(uint32_t step, bool lanes_arrive, int lane) {
        const int st = acquire(step);
        if (lane == 0) hdr[st].end = 1;
        __syncwarp();
        if (lanes_arrive) mbar_arrive(&full[st]);
        if (lane == 0) mbar_arrive(&full[st]);
    }
};

// Register rebalancing: the producer warp group gives registers back, the compute warp groups take them.
template <uint32_t Regs>
__device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(Regs)); }
template <uint32_t Regs>
__device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(Regs)); }

// Next work item of the calling (converged) warp: lane 0 claims it, every lane receives it.
__device__ __forceinline__ int claim_item(int* counter, int lane) {
    int k = 0;
    if (lane == 0) k = atomicAdd(counter, 1);
    return __shfl_sync(0xffffffffu, k, 0);
}

// One producer warp group at producer_regs and compute_warps warps at compute_regs fit the register file.
constexpr bool warp_group_regs_fit(uint32_t producer_regs, int compute_warps, uint32_t compute_regs) {
    return 128 * producer_regs + 32 * compute_warps * compute_regs <= 65536;
}

// A tile's C channels as the fewest work items no wider than `widest`, all of width CW, a multiple of 16.
struct ItemSplit { int nitems, CW; };
inline ItemSplit split_channels(int C, int widest) {
    const int nitems = (C + widest - 1) / widest;
    return {nitems, ((C + nitems - 1) / nitems + 15) / 16 * 16};
}

// For one launch of the persistent kernel K on `items` work items: ensures the work counter in ctx->work and zeroes it
// on s, and sets *grid to as many CTAs as are co-resident on the device, at most `items`.  The occupancy (with `smem`
// bytes of dynamic shared memory opted in) is found once per device.
template <auto K>
int persistent_grid(sgb_ctx* ctx, int threads, size_t smem, int items, cudaStream_t s, int* grid) {
    static DeviceOnce attr_set;
    static int grid_of_device[64];
    if (int rc = ctx->work.ensure(sizeof(int))) return rc;
    int dev = 0;
    SGB_CUDA(cudaGetDevice(&dev));
    int& g = grid_of_device[dev < 64 ? dev : 63];
    if (attr_set.first_use_on_device()) {
        SGB_CUDA(cudaFuncSetAttribute(K, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        int per_sm = 0, sms = 0;
        SGB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, K, threads, smem));
        SGB_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
        g = per_sm * sms > 0 ? per_sm * sms : 1;
    }
    SGB_CUDA(cudaMemsetAsync(ctx->work.p, 0, sizeof(int), s));
    *grid = g < items ? g : items;
    return SGB_OK;
}

}  // namespace sgb
