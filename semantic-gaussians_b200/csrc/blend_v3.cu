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
//   blend_forward     CTA = (tile, 64-channel chunk): the tile's weight rows and feature slices
//                     stream through a TMA-fed shared-memory ring (plain loads from L2 when the
//                     feature rows are not 16-byte aligned slices) and every lane accumulates an
//                     8 px x 8 ch register micro-tile (outer product, paired FMAs).
//   chain_backward    CTA = tile, warp = 32-pixel strip: s = <feature, dL/dout> per (pixel,
//                     Gaussian) for all channels over the strip's own entries (register
//                     micro-tiles), then the reference's back-to-front chain (backward.cu:477-550)
//                     in dot-product form -> dL/dmean2D, dL/dconic, dL/dopacity.
//   dfeature          persistent CTAs claim (tile, 64-channel chunk) items: dL/dfeature[g][ch] = sum_px
//                     w * dL/dout, a producer warp streams dL tiles and weight slabs by TMA, every
//                     compute warp owns 8 channels of all the tile's entries, one 16-byte reduction
//                     per (Gaussian, tile, 4 channels).
//
// Results are unchanged: the integer outputs come from the verbatim chain; every accumulator still
// adds its Gaussians in depth order.
#include <cstddef>
#include <cstring>
#include "common.cuh"
#include "blend_pool.cuh"

namespace sgb {

namespace {

constexpr int kThreads = SGB_TILE_PIX;

// Lane -> operand-group mapping of the register-tiled GEMM loops: a warp-wide LDS.128 costs 2 shared-memory
// wavefronts when every aligned group of 4 lanes reads at most 2 distinct 16-byte chunks and each half-warp at most 8
// (conflict-free) chunks, and 4 wavefronts otherwise.  With the natural split (one operand indexed by lane & 7, the
// other by lane >> 3) the lane & 7 operand pays 4 per load, and the shared-memory pipe rather than the FMA pipe limits
// the contraction kernels.  Giving each operand exactly one of the two low lane bits makes every operand load a
// 2-wavefront load.
__device__ __forceinline__ int lane_group8(int lane) { return (lane & 1) | (((lane >> 2) & 3) << 1); }  // bits 0, 2, 3
__device__ __forceinline__ int lane_group4(int lane) { return ((lane >> 1) & 1) | ((lane >> 4) << 1); } // bits 1, 4

// ------------------------------------------------------------------------------------ alpha pass
constexpr int kAB = 32;  // list entries per staging round

struct __align__(16) AlphaSmem {
    float4 recA[kAB];
    float4 recB[kAB];
    uint32_t ids[kAB];
    float wbuf[kAB][SGB_TILE_PIX];
    uint32_t wmask[8];
    uint32_t slot_chunk[kAB];
    uint32_t cur_chunk;
    uint32_t s_last;
};

__global__ void __launch_bounds__(kThreads) alpha_pass_kernel(
    const uint2* __restrict__ ranges, const uint32_t* __restrict__ point_list, int W, int H,
    const SplatRec* __restrict__ rec, float* __restrict__ final_T, uint32_t* __restrict__ n_contrib,
    uint32_t* __restrict__ tile_last, PoolView pool) {
    extern __shared__ __align__(128) unsigned char smem_raw[];
    AlphaSmem& sm = *reinterpret_cast<AlphaSmem*>(smem_raw);

    const int tiles_x = (W + SGB_TILE - 1) / SGB_TILE;
    const int tile = blockIdx.x;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const uint32_t tx = tid & (SGB_TILE - 1), ty = tid >> 4;
    const uint2 pix = {(uint32_t)(tile % tiles_x) * SGB_TILE + tx, (uint32_t)(tile / tiles_x) * SGB_TILE + ty};
    const uint32_t pix_id = W * pix.y + pix.x;
    const float2 pixf = {(float)pix.x, (float)pix.y};
    const bool inside = pix.x < (uint32_t)W && pix.y < (uint32_t)H;
    bool done = !inside;

    const uint2 range = ranges[tile];
    const int total = (int)(range.y - range.x);
    const int nbatches = (total + kAB - 1) / kAB;
    const uint32_t dbase = range.x / kChunkEntries + (uint32_t)tile;
    if (tid == 0) { sm.cur_chunk = kNone; sm.s_last = 0; }

    float T = 1.0f;
    uint32_t last_contributor = 0;
    uint32_t n_tile = 0;  // entries appended so far (uniform)
    uint32_t n_blend = 0; // Gaussians blended into this pixel

    // Staging of the (id, splat record) batches is software-pipelined in warp 0's registers: the ids run two
    // batches ahead, the records (a dependent gather through the id) one batch ahead, so neither round trip
    // sits between two batches of the chain (it used to: two dependent L2/DRAM latencies per 32 entries).
    auto load_id = [&](int bb) -> uint32_t {
        const int i = bb * kAB + tid;
        return (tid < kAB && bb < nbatches && i < total) ? __ldg(point_list + range.x + i) : 0u;
    };
    uint32_t id_cur = load_id(0), id_nxt = load_id(1);
    float4 rA = make_float4(0.f, 0.f, 0.f, 0.f), rB = rA;
    if (tid < kAB && tid < total) {
        const float4* rp = reinterpret_cast<const float4*>(rec + id_cur);
        rA = __ldg(rp);
        rB = __ldg(rp + 1);
    }
    for (int b = 0; b < nbatches; b++) {
        const int num_done = __syncthreads_count(done);  // forward.cu:310-312
        if (num_done == kThreads) break;
        const int base = b * kAB;
        const int cnt = min(kAB, total - base);
        if (tid < cnt) {
            sm.ids[tid] = id_cur;
            sm.recA[tid] = rA;
            sm.recB[tid] = rB;
        }
        __syncthreads();
        if (tid < kAB) {  // records of batch b+1 (its ids are already here), ids of batch b+2
            id_cur = id_nxt;
            if (base + kAB + tid < total) {
                const float4* rp = reinterpret_cast<const float4*>(rec + id_cur);
                rA = __ldg(rp);
                rB = __ldg(rp + 1);
            }
            id_nxt = load_id(b + 2);
        }
        uint32_t my_mask = 0;
        for (int j = 0; j < cnt; j++) {
            float w = 0.f;
            if (!done) {
                // forward.cu:333-362 verbatim
                const float4 a = sm.recA[j];
                const float2 xy = {a.x, a.y};
                const float2 d = {xy.x - pixf.x, xy.y - pixf.y};
                const float4 con_o = sm.recB[j];
                const float power = -0.5f * (con_o.x * d.x * d.x + con_o.z * d.y * d.y) - con_o.y * d.x * d.y;
                if (!(power > 0.0f)) {
                    const float alpha = min(0.99f, con_o.w * exp(power));
                    if (!(alpha < 1.0f / 255.0f)) {
                        const float test_T = T * (1 - alpha);
                        if (test_T < 0.0001f) {
                            done = true;
                        } else {
                            w = alpha * T;
                            T = test_T;
                            last_contributor = (uint32_t)(base + j + 1);
                        }
                    }
                }
            }
            sm.wbuf[j][tid] = w;
            n_blend += (w != 0.f);
            if (__ballot_sync(0xffffffffu, w != 0.f)) my_mask |= 1u << j;
        }
        if (lane == 0) sm.wmask[warp] = my_mask;
        __syncthreads();
        uint32_t tm = 0;
#pragma unroll
        for (int q = 0; q < 8; q++) tm |= sm.wmask[q];
        const int n_act = __popc(tm);
        if (n_act) {
            if (tid == 0) {
                uint32_t e = n_tile, cur = sm.cur_chunk;
                for (int k = 0; k < n_act; k++, e++) {
                    if ((e & (kChunkEntries - 1)) == 0) {
                        uint32_t nw = atomicAdd(&pool.hdr->counter, 1u);
                        if (nw >= pool.capacity) {
                            pool.hdr->overflow = 1;
                            nw = pool.capacity - 1;
                        }
                        pool.dir[dbase + e / kChunkEntries] = nw;
                        cur = nw;
                    }
                    sm.slot_chunk[k] = cur;
                }
                sm.cur_chunk = cur;
            }
            __syncthreads();
            int k = 0;
            for (uint32_t m = tm; m; m &= m - 1, k++) {
                const int j = __ffs(m) - 1;
                const uint32_t e = n_tile + k;
                WChunk& ck = pool.chunks[sm.slot_chunk[k]];
                const int s = e & (kChunkEntries - 1);
                ck.w[s][tid] = sm.wbuf[j][tid];
                if (tid == 0) {
                    uint32_t strips = 0;
#pragma unroll
                    for (int q = 0; q < 8; q++) strips |= ((sm.wmask[q] >> j) & 1u) << q;
                    ck.meta[s] = make_uint2(sm.ids[j], strips);
                }
            }
            n_tile += n_act;
        }
    }
    if (inside) {
        final_T[pix_id] = T;
        n_contrib[pix_id] = last_contributor;
        atomicMax(&sm.s_last, last_contributor);
    }
    n_blend = __reduce_add_sync(0xffffffffu, n_blend);
    if (lane == 0 && n_blend) atomicAdd(&pool.hdr->blended, (unsigned long long)n_blend);
    __syncthreads();
    if (tid == 0) {
        tile_last[tile] = sm.s_last;
        pool.count[tile] = n_tile;
        pool.dirbase[tile] = dbase;
    }
}

// ------------------------------------------------------------------------------------ forward
// Non-finite features.  The GEMM-shaped kernels multiply every (pixel, entry) pair of a tile, zero weights
// included, and 0 * inf = NaN: one non-finite feature row would poison every pixel of every tile its Gaussian is
// binned to, where the reference only touches the pixels that actually blend it (forward.cu:340-356 `continue`s
// before the accumulation).  A pair is blended exactly when its weight alpha * T is non-zero (alpha >= 1/255 and
// T >= 1e-4 on that path), so the exact semantics are "accumulate only where w != 0".  Guarding every FMA would
// double the inner loop; instead the epilogue tests the accumulators (acc * 0 summed: NaN iff any accumulator is
// non-finite, 32 paired FMAs per lane) and only a warp that sees a non-finite value recomputes its 32 px x CH
// slice with the guarded loop below, straight from the weight rows and feature rows in global memory.
template <int MCH>
__device__ __forceinline__ bool acc_nonfinite(const float2 (&acc)[8][MCH / 2]) {
    float2 z = make_float2(0.f, 0.f);
#pragma unroll
    for (int i = 0; i < 8; i++)
#pragma unroll
        for (int k = 0; k < MCH / 2; k++) z = ffma2(acc[i][k], make_float2(0.f, 0.f), z);
    const float t = z.x + z.y;
    return __any_sync(0xffffffffu, t != t);
}

// RING = true: lane cg owns channels {4cg..4cg+3} U {32+4cg..} of the slice (blend_forward_tma_kernel);
// false: channels cg*MCH .. cg*MCH+MCH-1 (blend_forward_v3_kernel).  Self-contained (own accumulators, own
// stores) so that the fast path's accumulators never have their address taken.
template <int MCH, bool RING>
__device__ __noinline__ void forward_redo_guarded(const PoolView& pool, uint32_t n, uint32_t dbase,
                                                  const float* __restrict__ features, int C, int ch0, int nch,
                                                  int warp, int woff, int cg, const float* __restrict__ bg_color,
                                                  const float* __restrict__ final_T, int W, int H, uint32_t row,
                                                  uint32_t col0, float* __restrict__ out_color) {
    float acc[8][MCH];
#pragma unroll
    for (int i = 0; i < 8; i++)
#pragma unroll
        for (int k = 0; k < MCH; k++) acc[i][k] = 0.f;
    for (uint32_t e = 0; e < n; e++) {
        const WChunk* ck = pool.chunks + chunk_of(pool, dbase, (int)(e / kChunkEntries));
        const int s = (int)(e & (kChunkEntries - 1));
        const uint2 meta = ck->meta[s];
        if (!((meta.y >> warp) & 1u)) continue;
        const float* fr = features + (size_t)meta.x * C + ch0;
        float f[MCH];
#pragma unroll
        for (int k = 0; k < MCH; k++) {
            const int chl = RING ? ((k >> 2) * 32 + cg * 4 + (k & 3)) : (cg * MCH + k);
            f[k] = chl < nch ? __ldg(fr + chl) : 0.f;
        }
#pragma unroll
        for (int i = 0; i < 8; i++) {
            const float w = ck->w[s][woff + i];
            if (w != 0.f) {
#pragma unroll
                for (int k = 0; k < MCH; k++) acc[i][k] = fmaf(f[k], w, acc[i][k]);
            }
        }
    }
    if (row >= (uint32_t)H) return;
    const size_t plane = (size_t)H * W;
#pragma unroll
    for (int k = 0; k < MCH; k++) {
        const int chl = RING ? ((k >> 2) * 32 + cg * 4 + (k & 3)) : (cg * MCH + k);
        if (chl >= nch) continue;
        const float bgc = bg_color[ch0 + chl];
        float* dst = out_color + (size_t)(ch0 + chl) * plane + (size_t)W * row + col0;
#pragma unroll
        for (int i = 0; i < 8; i++)
            if (col0 + i < (uint32_t)W) dst[i] = acc[i][k] + final_T[(size_t)W * row + col0 + i] * bgc;
    }
}

template <int CH>
__global__ void __launch_bounds__(kThreads, 2) blend_forward_v3_kernel(
    int W, int H, int C, const float* __restrict__ features, const float* __restrict__ bg_color,
    const float* __restrict__ final_T, PoolView pool, float* __restrict__ out_color) {
    constexpr int MCH = CH / 8;
    const int tiles_x = (W + SGB_TILE - 1) / SGB_TILE;
    const int nchunksC = (C + CH - 1) / CH;
    const int tile = blockIdx.x / nchunksC;           // chunk index fastest: the CTAs of one tile are
    const int ch0 = (blockIdx.x % nchunksC) * CH;     // co-scheduled and share its weight rows in L2
    const int nch = min(CH, C - ch0);
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int pg = lane >> 3, cg = lane & 7;
    const uint2 pix_min = {(uint32_t)(tile % tiles_x) * SGB_TILE, (uint32_t)(tile / tiles_x) * SGB_TILE};

    float2 acc[8][MCH / 2];
#pragma unroll
    for (int i = 0; i < 8; i++)
#pragma unroll
        for (int k = 0; k < MCH / 2; k++) acc[i][k] = make_float2(0.f, 0.f);

    const uint32_t n = pool.count[tile];
    const uint32_t dbase = pool.dirbase[tile];
    const int woff = warp * 32 + pg * 8;
    const int foff = ch0 + cg * MCH;
    for (uint32_t e = 0; e < n;) {
        const WChunk* ck = pool.chunks + chunk_of(pool, dbase, (int)(e / kChunkEntries));
        const int m = (int)min((uint32_t)kChunkEntries, n - e);
        for (int s = 0; s < m; s++) {
            const uint2 meta = ck->meta[s];
            if (!((meta.y >> warp) & 1u)) continue;
            const float4* wp = reinterpret_cast<const float4*>(&ck->w[s][woff]);
            const float4 w0 = wp[0], w1 = wp[1];
            const float* fr = features + (size_t)meta.x * C + foff;
            float2 f[MCH / 2];
#pragma unroll
            for (int k = 0; k < MCH / 2; k++) {
                f[k].x = (cg * MCH + 2 * k < nch) ? __ldg(fr + 2 * k) : 0.f;
                f[k].y = (cg * MCH + 2 * k + 1 < nch) ? __ldg(fr + 2 * k + 1) : 0.f;
            }
            const float wv[8] = {w0.x, w0.y, w0.z, w0.w, w1.x, w1.y, w1.z, w1.w};
#pragma unroll
            for (int i = 0; i < 8; i++) {
                const float2 w2 = make_float2(wv[i], wv[i]);
#pragma unroll
                for (int k = 0; k < MCH / 2; k++) acc[i][k] = ffma2(f[k], w2, acc[i][k]);
            }
        }
        e += m;
    }
    // out = acc + T * bg (forward.cu:372-373)
    const uint32_t row = pix_min.y + 2 * warp + (pg >> 1);
    const uint32_t col0 = pix_min.x + (pg & 1) * 8;
    if (acc_nonfinite<MCH>(acc)) {
        forward_redo_guarded<MCH, false>(pool, n, dbase, features, C, ch0, nch, warp, woff, cg, bg_color, final_T, W, H,
                                         row, col0, out_color);
        return;
    }
    if (row < (uint32_t)H) {
        const size_t plane = (size_t)H * W;
        const bool vec = ((W & 3) == 0) && (col0 + 8 <= (uint32_t)W);
        float Tv[8];
#pragma unroll
        for (int i = 0; i < 8; i++) Tv[i] = (col0 + i < (uint32_t)W) ? final_T[(size_t)W * row + col0 + i] : 0.f;
#pragma unroll
        for (int k = 0; k < MCH; k++) {
            const int chl = cg * MCH + k;
            if (chl >= nch) continue;
            const float bgc = bg_color[ch0 + chl];
            float* dst = out_color + (size_t)(ch0 + chl) * plane + (size_t)W * row + col0;
            float o[8];
#pragma unroll
            for (int i = 0; i < 8; i++) o[i] = ((k & 1) ? acc[i][k / 2].y : acc[i][k / 2].x) + Tv[i] * bgc;
            if (vec) {
                reinterpret_cast<float4*>(dst)[0] = make_float4(o[0], o[1], o[2], o[3]);
                reinterpret_cast<float4*>(dst)[1] = make_float4(o[4], o[5], o[6], o[7]);
            } else {
#pragma unroll
                for (int i = 0; i < 8; i++)
                    if (col0 + i < (uint32_t)W) dst[i] = o[i];
            }
        }
    }
}

// ------------------------------------------------------------------------------------ async-copy helpers
// 3-D tensor tile global -> shared through the TMA engine (SASS: UTMALDG): box corner (x, y, z) in elements, out-of-range
// elements arrive as zeros; completion is signalled on `bar` as the box's bytes.  dst 128-byte aligned.
__device__ __forceinline__ void tma_tile3d_g2s(void* dst_smem, const CUtensorMap* map, int x, int y, int z, uint64_t* bar) {
    asm volatile(
        "cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4}], [%5];" ::"r"(
            smem_u32(dst_smem)),
        "l"(reinterpret_cast<uint64_t>(map)), "r"(x), "r"(y), "r"(z), "r"(smem_u32(bar))
        : "memory");
}
// Orders this thread's earlier generic-proxy shared-memory accesses before later async-proxy (TMA) writes.
__device__ __forceinline__ void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// ------------------------------------------------------------------------------------ GEMM-shaped kernels
// With the weights materialised per tile, the three C-wide contractions are small dense GEMMs over the
// tile's touching Gaussians (G ~ 115 on K3), done in fp32 on the CUDA cores (north_star: no tensor cores;
// the 1e-4 fp32 bar rules out TF32 anyway):
//     forward   out[256 px][64 ch]  = W^T[256 px][G]  . F[G][64 ch]      K = G      lane tile 8 px x 8 ch
//     s-pass    S[32 px][32]        = dL[32 px][C]    . F^T[C][32]       K = C      lane tile 8 px x 4 entries
//               (per warp: its strip and a 32-entry segment of the strip's entries)
//     dfeature  dF[G][64 ch]        = W[G][256 px]    . dL[256 px][64]   K = 256 px lane tile <= 8 entries x 4 ch
// Register tiles give every shared-memory load several FMAs and need no cross-lane reductions (a
// shuffle-reduce formulation spends its issue slots on SHFL/FSEL/FADD instead).
// Forward GEMM with a TMA-fed ring.  With plain loads of the weight rows every warp waits an L2/DRAM round
// trip per entry.  Here one ring stage = one 16-entry chunk: per staged
// Gaussian two 1-D bulk copies (cp.async.bulk: the 1 KB weight row and the 256 B feature slice), NS stages
// guarded by full/empty mbarriers.  Warp 0 is producer AND consumer, so nothing it does for production may
// block its math: the chunk indices come from the tile's directory (copied to shared memory up front, no
// pointer chasing), the (id, mask) records of the NEXT batch are fetched into registers one whole batch of
// math before they are needed, and the stage it refills is the one everybody left TWO batches ago, so the
// empty-barrier wait is already satisfied (refilling the stage of the previous batch would couple warp 0 to
// the slowest warp on every batch).
template <int CH, int NS>
__global__ void __launch_bounds__(kThreads, 2) blend_forward_tma_kernel(
    int W, int H, int C, const float* __restrict__ features, const float* __restrict__ bg_color,
    const float* __restrict__ final_T, PoolView pool, float* __restrict__ out_color) {
    constexpr int MCH = CH / 8;
    constexpr int ES = kChunkEntries;  // entries per stage
    constexpr int LA = NS - 2;         // batches in flight ahead of the one being consumed
    constexpr int kDirCap = 192;       // directory entries cached in shared memory (3072 active Gaussians / tile)
    struct Stage {
        float w[ES][SGB_TILE_PIX];
        float f[ES][CH];
    };
    extern __shared__ __align__(128) unsigned char smem_raw[];
    Stage* stg = reinterpret_cast<Stage*>(smem_raw);
    __shared__ uint64_t full_bar[NS], empty_bar[NS];
    __shared__ uint32_t Cdir[kDirCap];
    __shared__ __align__(16) float Tsm[SGB_TILE_PIX];  // final_T of the tile (the epilogue used to stall on these loads)
    __shared__ float bgS[CH];

    const int tiles_x = (W + SGB_TILE - 1) / SGB_TILE;
    const int nchunksC = (C + CH - 1) / CH;
    const int tile = blockIdx.x / nchunksC;
    const int ch0 = (blockIdx.x % nchunksC) * CH;
    const int nch = min(CH, C - ch0);
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int pg = lane_group4(lane), cg = lane_group8(lane);
    const uint2 pix_min = {(uint32_t)(tile % tiles_x) * SGB_TILE, (uint32_t)(tile / tiles_x) * SGB_TILE};

    const uint32_t n = pool.count[tile];
    const int nb = (int)((n + ES - 1) / ES);
    const uint32_t dbase = pool.dirbase[tile];
    if (tid == 0) {
        for (int i = 0; i < NS; i++) {
            mbar_init(&full_bar[i], 1);
            mbar_init(&empty_bar[i], kThreads / 32);
        }
        mbar_fence_init();
    }
    for (int k = tid; k < min(nb, kDirCap); k += kThreads) Cdir[k] = chunk_of(pool, dbase, k);
    {
        const uint32_t x = pix_min.x + (tid & (SGB_TILE - 1)), y = pix_min.y + (tid >> 4);
        Tsm[tid] = (x < (uint32_t)W && y < (uint32_t)H) ? final_T[(size_t)W * y + x] : 0.f;
        if (tid < nch) bgS[tid] = bg_color[ch0 + tid];
    }
    if (nch < CH)  // zero the never-written tail of every feature row once
        for (int e = tid; e < NS * ES * CH; e += kThreads) {
            const int k = e % CH;
            if (k >= nch) stg[e / (ES * CH)].f[(e / CH) % ES][k] = 0.f;
        }
    __syncthreads();

    // ---- producer (warp 0, lanes 0..15 = entry slots of a chunk)
    auto chunk_ptr = [&](int bi) {
        return pool.chunks + (bi < kDirCap ? Cdir[bi] : chunk_of(pool, dbase, bi));
    };
    auto load_meta = [&](int bi) {  // (Gaussian id, strip mask) of this lane's entry of batch bi
        uint2 m = make_uint2(0u, 0u);
        if (bi < nb && lane < min(ES, (int)n - bi * ES)) m = __ldg(&chunk_ptr(bi)->meta[lane]);
        return m;
    };
    auto issue = [&](int bi, uint2 meta) {  // warp 0, converged; bi < nb
        const int st = bi % NS;
        const int cnt = min(ES, (int)n - bi * ES);
        if (bi >= NS) mbar_wait(&empty_bar[st], (uint32_t)(((bi / NS) - 1) & 1));  // batch bi-NS released by all warps
        if (lane < cnt) {
            const WChunk* ck = chunk_ptr(bi);
            bulk_g2s(&stg[st].w[lane][0], &ck->w[lane][0], SGB_TILE_PIX * 4u, &full_bar[st]);
            bulk_g2s(&stg[st].f[lane][0], features + (size_t)meta.x * C + ch0, (uint32_t)nch * 4u, &full_bar[st]);
        }
        __syncwarp();
        if (lane == 0) mbar_arrive_expect_tx(&full_bar[st], (uint32_t)cnt * (SGB_TILE_PIX * 4u + (uint32_t)nch * 4u));
    };
    uint2 meta_next = make_uint2(0u, 0u);  // record of batch `pb`, the next one to issue
    int pb = 0;
    if (warp == 0) {
        uint2 m[LA];
#pragma unroll
        for (int i = 0; i < LA; i++) m[i] = load_meta(i);  // independent loads, one round trip
#pragma unroll
        for (int i = 0; i < LA; i++)
            if (i < nb) issue(i, m[i]);
        pb = min(LA, nb);
        meta_next = load_meta(pb);
    }

    float2 acc[8][MCH / 2];
#pragma unroll
    for (int i = 0; i < 8; i++)
#pragma unroll
        for (int k = 0; k < MCH / 2; k++) acc[i][k] = make_float2(0.f, 0.f);

    const int woff = warp * 32 + pg * 8;
    // Lane cg accumulates channels {4cg..4cg+3} and {32+4cg..32+4cg+3} of the slice: each of its two LDS.128 then
    // reads 8 x 16 B that are contiguous across the 8 channel lanes (one 128-byte wavefront); the natural
    // assignment 8cg..8cg+7 spread them over 256 B = two wavefronts per load.
    auto entry = [&](const Stage& sg, int e) {
        const float4 w0 = *reinterpret_cast<const float4*>(&sg.w[e][woff]);
        const float4 w1 = *reinterpret_cast<const float4*>(&sg.w[e][woff + 4]);
        float2 f[MCH / 2];
#pragma unroll
        for (int q = 0; q < MCH / 4; q++) {
            const float4 t = *reinterpret_cast<const float4*>(&sg.f[e][q * 32 + cg * 4]);
            f[2 * q] = make_float2(t.x, t.y);
            f[2 * q + 1] = make_float2(t.z, t.w);
        }
        const float wv[8] = {w0.x, w0.y, w0.z, w0.w, w1.x, w1.y, w1.z, w1.w};
#pragma unroll
        for (int i = 0; i < 8; i++) {
            const float2 w2 = make_float2(wv[i], wv[i]);
#pragma unroll
            for (int k = 0; k < MCH / 2; k++) acc[i][k] = ffma2(f[k], w2, acc[i][k]);
        }
    };
    for (int b = 0; b < nb; b++) {
        const int st = b % NS;
        const int cnt = min(ES, (int)n - b * ES);
        if (warp == 0 && pb < nb) {  // refill the stage of batch b-2 with batch b+LA
            issue(pb, meta_next);
            pb++;
            meta_next = load_meta(pb);  // lands while this batch is being consumed
        }
        mbar_wait(&full_bar[st], (uint32_t)((b / NS) & 1));
        // dense on purpose: skipping strips whose 32 weights are all zero breaks the unrolled load/FMA
        // software pipeline
        if (cnt == ES) {
#pragma unroll
            for (int e = 0; e < ES; e++) entry(stg[st], e);
        } else {
            for (int e = 0; e < cnt; e++) entry(stg[st], e);
        }
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty_bar[st]);
    }
    const uint32_t row = pix_min.y + 2 * warp + (pg >> 1);
    const uint32_t col0 = pix_min.x + (pg & 1) * 8;
    if (acc_nonfinite<MCH>(acc)) {
        forward_redo_guarded<MCH, true>(pool, n, dbase, features, C, ch0, nch, warp, woff, cg, bg_color, final_T, W, H,
                                        row, col0, out_color);
        return;
    }
    if (row < (uint32_t)H) {
        const size_t plane = (size_t)H * W;
        const bool vec = ((W & 3) == 0) && (col0 + 8 <= (uint32_t)W);
        const float4 t0 = *reinterpret_cast<const float4*>(&Tsm[(2 * warp + (pg >> 1)) * SGB_TILE + (pg & 1) * 8]);
        const float4 t1 = *reinterpret_cast<const float4*>(&Tsm[(2 * warp + (pg >> 1)) * SGB_TILE + (pg & 1) * 8 + 4]);
        const float Tv[8] = {t0.x, t0.y, t0.z, t0.w, t1.x, t1.y, t1.z, t1.w};
#pragma unroll
        for (int k = 0; k < MCH; k++) {
            const int chl = (k >> 2) * 32 + cg * 4 + (k & 3);  // see `entry`: lane cg owns channels cg*4.. and 32+cg*4..
            if (chl >= nch) continue;
            const float bgc = bgS[chl];
            float* dst = out_color + (size_t)(ch0 + chl) * plane + (size_t)W * row + col0;
            float o[8];
#pragma unroll
            for (int i = 0; i < 8; i++) o[i] = ((k & 1) ? acc[i][k / 2].y : acc[i][k / 2].x) + Tv[i] * bgc;
            if (vec) {
                reinterpret_cast<float4*>(dst)[0] = make_float4(o[0], o[1], o[2], o[3]);
                reinterpret_cast<float4*>(dst)[1] = make_float4(o[4], o[5], o[6], o[7]);
            } else {
#pragma unroll
                for (int i = 0; i < 8; i++)
                    if (col0 + i < (uint32_t)W) dst[i] = o[i];
            }
        }
    }
}

// dF[entry][ch] = sum over the tile's 256 pixels of w[entry][px] * dL/dout[px][ch]   (K = pixels).
// Persistent: the grid fills the GPU once and every CTA claims work items (tile, 64-channel chunk; the chunk varies
// fastest, so the CTAs of one tile meet its weight rows in L2) from a counter until none are left; an empty tile
// costs one claim.  Warp 8 is the producer and warps 0-7 only compute:
//   * the dL tile of an item, [16 rows][64 ch][16 px] = 64 KB, is ONE 3-D TMA box into one of two buffers.  The
//     producer issues the next item's box while the current item is being contracted (at its 5th weight slab, when
//     every warp has provably released the buffer).  Layouts TMA cannot take (a row pitch or base that is not a
//     multiple of 16 bytes: W % 4 != 0 in fp32, W % 8 != 0 in fp16) are staged by the producer warp into the same
//     (swizzled) layout on the same mbarrier, with 4-byte cp.async (fp32) or plain loads (fp16);
//   * the weight rows of a pass (up to 128 entries) stream as 32-pixel slabs, one 3-D TMA box [16 rows][32 px] per
//     16-entry pool chunk, through a ring of kDfStages stages.
// Every hand-off is a full/empty mbarrier pair; there is no CTA-wide barrier after the set-up.  Warp w owns channels
// 8w..8w+7 of the chunk and ALL entries of the pass, so every warp computes on every item however few entries the
// tile has.  Lane (eg = lane >> 1, cgp = lane & 1) accumulates entries {eg + 16j, j < R} x channels 8w + 4cgp + {0..3}
// in scalar registers, R = ceil(entries / 16) <= 8: per 4-pixel K step 16R FMAs for R + 4 LDS.128.  The TMA swizzles
// keep every operand load at 2 shared-memory wavefronts or less (see lane_group8):
//   * weights, SWIZZLE_128B: quad q of the 128-byte row e sits at q ^ (e & 7); each 4-lane group reads 2 rows and each
//     half-warp 8 consecutive rows -> 8 distinct bank groups;
//   * dL, SWIZZLE_64B over a [row][ch][16 px] box: quad p of channel c sits at p ^ ((c >> 1) & 3), so channels c and
//     c + 4 (the two cgp halves of a load) land in different banks.
constexpr int kDfCH = 64;                   // channels per work item
constexpr int kDfStages = 4;                // weight-slab ring depth
constexpr int kDfThreads = kThreads + 32;   // 8 compute warps + 1 producer warp
constexpr int kDfPass = 128;                // entries per pass (8 pool chunks)
constexpr int kDfSlabs = SGB_TILE_PIX / 32;  // 32-pixel K slabs per pass

struct DfHdr {  // one weight-ring stage's description, written by the producer before the stage is armed
    int end;            // no more work
    int cnt;            // entries of the pass
    int slab;           // pixels 32 slab .. 32 slab + 31
    int first, last;    // first slab of the item (wait for its dL tile) / last slab of the item (release the tile)
    int dbuf;           // dL buffer of the item and the parity of its fill
    uint32_t dpar;
    int ch0, nch;
    uint32_t gid[kDfPass];  // Gaussian ids of the pass (written for the last slab of a pass)
};
// T: element type of dL/dout as it sits in global memory (float, or __half for an fp16 feature map that is lifted
// onto the Gaussians); the dL tile keeps it in shared memory and is widened to fp32 in the compute warps' loads.
template <typename T>
struct DfSmem {  // at a 1024-byte aligned offset of the dynamic shared memory (TMA swizzle atoms)
    T dl[2][SGB_TILE_PIX * kDfCH];
    float w[kDfStages][kDfPass * 32];
    DfHdr hdr[kDfStages];
    uint64_t wfull[kDfStages], wempty[kDfStages], dfull[2], dempty[2];
};
template <typename T>
constexpr size_t kDfSmemBytes = sizeof(DfSmem<T>) + 1024;
template <typename T>
constexpr uint32_t kDfTileBytes = SGB_TILE_PIX * kDfCH * sizeof(T);
static_assert(kDfSmemBytes<float> <= 227 * 1024, "dL/dfeature shared memory exceeds the sm_90 opt-in limit");

// Pixels 4 (Q & 3) .. 4 (Q & 3) + 3 of tile row Q >> 2, channel cl + k, of an item's dL tile; dl points at channel cl
// (a multiple of 4) and swz = df_swz<T>(cl).  The tile is the TMA box under its swizzle, 16 px per channel row:
//   fp32, 64 B rows, SWIZZLE_64B: 4-px quad p of channel c sits at p ^ ((c >> 1) & 3);
//   fp16, 32 B rows, SWIZZLE_32B: 8-px half h of channel c sits at h ^ ((c >> 2) & 1).
// Either way channels c and c + 4, the two halves of a warp's load, land in different banks.
template <typename T>
__device__ __forceinline__ int df_swz(int cl) { return sizeof(T) == 4 ? (cl >> 1) & 3 : (cl >> 2) & 1; }
__device__ __forceinline__ float4 df_dl4(const float* dl, int Q, int k, int swz) {
    return *reinterpret_cast<const float4*>(dl + (Q >> 2) * (kDfCH * 16) + k * 16 + (((Q & 3) ^ swz ^ (k >> 1)) << 2));
}
__device__ __forceinline__ float4 df_dl4(const __half* dl, int Q, int k, int swz) {
    const uint2 r = *reinterpret_cast<const uint2*>(dl + (Q >> 2) * (kDfCH * 16) + k * 16 +
                                                    ((((Q & 3) >> 1) ^ swz) << 3) + ((Q & 1) << 2));
    const float2 a = __half22float2(*reinterpret_cast<const __half2*>(&r.x));
    const float2 b = __half22float2(*reinterpret_cast<const __half2*>(&r.y));
    return make_float4(a.x, a.y, b.x, b.y);
}

__device__ __forceinline__ void cp_async4(void* dst_smem, const void* src, int src_bytes) {
    asm volatile("cp.async.ca.shared.global [%0], [%1], 4, %2;" ::"r"(smem_u32(dst_smem)), "l"(src), "r"(src_bytes)
                 : "memory");
}
// Arrives on `bar` once every cp.async this thread issued so far has landed (the arrival is part of the init count).
__device__ __forceinline__ void cp_async_mbar_arrive_noinc(uint64_t* bar) {
    asm volatile("cp.async.mbarrier.arrive.noinc.shared::cta.b64 [%0];" ::"r"(smem_u32(bar)) : "memory");
}

// One 32-pixel slab of a pass: acc[j][k] += sum over the slab of w[eg + 16j][px] * dL[px][cl + k].
// dl points at channel cl of the item's dL buffer, ws at the stage's weight rows; swz = df_swz<T>(cl).
template <int R, typename T>
__device__ __forceinline__ void df_slab(float (&acc)[8][4], const float* __restrict__ ws, const T* __restrict__ dl,
                                        int slab, int eg, int swz) {
#pragma unroll
    for (int q = 0; q < 8; q++) {
        const int Q = slab * 8 + q;  // pixel quad of the tile: row Q >> 2, quad Q & 3 of the row
        float4 d[4];
#pragma unroll
        for (int k = 0; k < 4; k++) d[k] = df_dl4(dl, Q, k, swz);
#pragma unroll
        for (int j = 0; j < R; j++) {
            const float4 wv = *reinterpret_cast<const float4*>(ws + (eg + 16 * j) * 32 + ((q ^ (eg & 7)) << 2));
#pragma unroll
            for (int k = 0; k < 4; k++) {
                acc[j][k] = fmaf(wv.x, d[k].x, acc[j][k]);
                acc[j][k] = fmaf(wv.y, d[k].y, acc[j][k]);
                acc[j][k] = fmaf(wv.z, d[k].z, acc[j][k]);
                acc[j][k] = fmaf(wv.w, d[k].w, acc[j][k]);
            }
        }
    }
}

template <typename T>
__global__ void __launch_bounds__(kDfThreads, 1) dfeature_persistent_kernel(
    int W, int H, int C, const T* __restrict__ dL_dpixels, PoolView pool, float* __restrict__ dL_dcolors,
    int* __restrict__ work_counter, const __grid_constant__ CUtensorMap dl_map,
    const __grid_constant__ CUtensorMap w_map, const int use_tma) {
    extern __shared__ __align__(128) unsigned char smem_raw[];
    DfSmem<T>& sm = *reinterpret_cast<DfSmem<T>*>(smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u));
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    constexpr int kComputeWarps = kThreads / 32;
    if (tid == 0) {
        for (int i = 0; i < kDfStages; i++) {
            mbar_init(&sm.wfull[i], 1);
            mbar_init(&sm.wempty[i], kComputeWarps);
        }
        for (int i = 0; i < 2; i++) {
            mbar_init(&sm.dfull[i], use_tma ? 1 : 32);
            mbar_init(&sm.dempty[i], kComputeWarps);
        }
        mbar_fence_init();
    }
    __syncthreads();

    if (warp < kComputeWarps) {
        const int eg = lane >> 1, cgp = lane & 1;
        const int cl = warp * 8 + cgp * 4;  // channel (within the chunk) of k = 0
        const bool red16 = ((C & 3) == 0) && ((reinterpret_cast<uintptr_t>(dL_dcolors) & 15) == 0);
        float acc[8][4];
        for (uint32_t step = 0;; step++) {
            const int st = (int)(step % kDfStages);
            mbar_wait(&sm.wfull[st], (step / kDfStages) & 1u);
            const DfHdr& h = sm.hdr[st];
            if (h.end) break;
            const int slab = h.slab, cnt = h.cnt, dbuf = h.dbuf, nch = h.nch, last = h.last;
            const int R = (cnt + 15) >> 4;
            if (h.first) mbar_wait(&sm.dfull[dbuf], h.dpar);
            if (slab == 0) {
#pragma unroll
                for (int j = 0; j < 8; j++)
#pragma unroll
                    for (int k = 0; k < 4; k++) acc[j][k] = 0.f;
            }
            if (warp * 8 < nch) {
                const float* ws = sm.w[st];
                const T* dl = sm.dl[dbuf] + cl * 16;
                const int swz = df_swz<T>(cl);
                switch (R) {
                    case 1: df_slab<1, T>(acc, ws, dl, slab, eg, swz); break;
                    case 2: df_slab<2, T>(acc, ws, dl, slab, eg, swz); break;
                    case 3: df_slab<3, T>(acc, ws, dl, slab, eg, swz); break;
                    case 4: df_slab<4, T>(acc, ws, dl, slab, eg, swz); break;
                    case 5: df_slab<5, T>(acc, ws, dl, slab, eg, swz); break;
                    case 6: df_slab<6, T>(acc, ws, dl, slab, eg, swz); break;
                    case 7: df_slab<7, T>(acc, ws, dl, slab, eg, swz); break;
                    default: df_slab<8, T>(acc, ws, dl, slab, eg, swz); break;
                }
                if (slab == kDfSlabs - 1 && cl < nch) {
                    const int ch0 = h.ch0;
#pragma unroll
                    for (int j = 0; j < 8; j++) {
                        const int e = eg + 16 * j;
                        if (j >= R || e >= cnt) continue;
                        float* dst = dL_dcolors + (size_t)h.gid[e] * C + ch0 + cl;
                        if (red16 && cl + 4 <= nch) {
                            red_add_v4_f32(dst, make_float4(acc[j][0], acc[j][1], acc[j][2], acc[j][3]));
                        } else {
#pragma unroll
                            for (int k = 0; k < 4; k++)
                                if (cl + k < nch) red_add_f32(dst + k, acc[j][k]);
                        }
                    }
                }
            }
            __syncwarp();
            if (lane == 0) {
                mbar_arrive(&sm.wempty[st]);
                if (last) mbar_arrive(&sm.dempty[dbuf]);
            }
        }
        return;
    }

    // ---- producer warp
    const int tiles_x = (W + SGB_TILE - 1) / SGB_TILE;
    const int tiles = tiles_x * ((H + SGB_TILE - 1) / SGB_TILE);
    const int nchunksC = (C + kDfCH - 1) / kDfCH;
    const int total = tiles * nchunksC;
    const size_t plane = (size_t)H * W;
    uint32_t step = 0;   // ring stages armed so far
    uint32_t items = 0;  // non-empty items whose dL tile was issued
    struct Item { int tile, ch0; uint32_t n; int dbuf; uint32_t dpar; };
    auto acquire = [&]() -> int {  // next ring stage, once the compute warps released its previous use
        const int st = (int)(step % kDfStages);
        if (step >= kDfStages) mbar_wait(&sm.wempty[st], ((step / kDfStages) - 1) & 1u);
        return st;
    };
    // Claims items until a non-empty one and issues its dL tile; tile < 0 when the work is exhausted.
    auto claim = [&]() -> Item {
        Item it{-1, 0, 0u, 0, 0u};
        for (;;) {
            int k = 0;
            if (lane == 0) k = atomicAdd(work_counter, 1);
            k = __shfl_sync(0xffffffffu, k, 0);
            if (k >= total) return it;
            it.tile = k / nchunksC;
            it.ch0 = (k % nchunksC) * kDfCH;
            it.n = pool.count[it.tile];
            if (it.n != 0) break;
        }
        it.dbuf = (int)(items & 1);
        it.dpar = (items >> 1) & 1u;
        if (items >= 2) mbar_wait(&sm.dempty[it.dbuf], ((items >> 1) - 1) & 1u);  // item `items - 2` released it
        items++;
        const int x0 = (it.tile % tiles_x) * SGB_TILE, y0 = (it.tile / tiles_x) * SGB_TILE;
        T* dst = sm.dl[it.dbuf];
        if (use_tma) {
            if (lane == 0) {
                mbar_arrive_expect_tx(&sm.dfull[it.dbuf], kDfTileBytes<T>);
                tma_tile3d_g2s(dst, &dl_map, x0, it.ch0, y0, &sm.dfull[it.dbuf]);
            }
        } else if constexpr (sizeof(T) == 2) {
            // cp.async has no 2-byte size: plain loads into the TMA layout, then one release-arrive per lane
#pragma unroll 8
            for (int idx = lane; idx < SGB_TILE_PIX * kDfCH; idx += 32) {
                const int x = idx & (SGB_TILE - 1), r = (idx >> 4) & (SGB_TILE - 1), c = idx >> 8;
                const int gx = x0 + x, gy = y0 + r;
                const bool ok = it.ch0 + c < C && gx < W && gy < H;
                dst[r * (kDfCH * 16) + c * 16 + ((((x >> 3) ^ ((c >> 2) & 1)) << 3) | (x & 7))] =
                    ok ? dL_dpixels[(size_t)(it.ch0 + c) * plane + (size_t)W * gy + gx] : T(0.f);
            }
            mbar_arrive(&sm.dfull[it.dbuf]);
        } else {
            for (int idx = lane; idx < SGB_TILE_PIX * kDfCH; idx += 32) {
                const int x = idx & (SGB_TILE - 1), r = (idx >> 4) & (SGB_TILE - 1), c = idx >> 8;
                const int gx = x0 + x, gy = y0 + r;
                const bool ok = it.ch0 + c < C && gx < W && gy < H;
                const float* src = ok ? dL_dpixels + (size_t)(it.ch0 + c) * plane + (size_t)W * gy + gx : dL_dpixels;
                cp_async4(dst + r * (kDfCH * 16) + c * 16 + ((((x >> 2) ^ ((c >> 1) & 3)) << 2) | (x & 3)), src,
                          ok ? 4 : 0);
            }
            cp_async_mbar_arrive_noinc(&sm.dfull[it.dbuf]);
        }
        return it;
    };

    Item cur = claim();
    while (cur.tile >= 0) {
        Item nxt{-1, 0, 0u, 0, 0u};
        bool claimed = false;
        const uint32_t dbase = pool.dirbase[cur.tile];
        const int nch = min(kDfCH, C - cur.ch0);
        int slab_of_item = 0;
        for (uint32_t base = 0; base < cur.n; base += kDfPass) {
            const int cnt = (int)min((uint32_t)kDfPass, cur.n - base);
            const int nck = (cnt + kChunkEntries - 1) / kChunkEntries;
            const uint32_t cid = lane < nck ? chunk_of(pool, dbase, (int)(base / kChunkEntries) + lane) : 0u;
            uint32_t gid[kDfPass / 32];
#pragma unroll
            for (int i = 0; i < kDfPass / 32; i++) {
                const int e = lane + 32 * i;
                const uint32_t c = __shfl_sync(0xffffffffu, cid, e / kChunkEntries);
                gid[i] = e < cnt ? pool.chunks[c].meta[e & (kChunkEntries - 1)].x : 0u;
            }
            for (int s = 0; s < kDfSlabs; s++, slab_of_item++) {
                if (!claimed && slab_of_item == kDfStages) {
                    // the stage acquired below was released by every warp after the item's first slab, so every
                    // warp is past the previous item and its dL buffer is free: prefetch the next item's tile now
                    nxt = claim();
                    claimed = true;
                }
                const int st = acquire();
                DfHdr& h = sm.hdr[st];
                if (lane == 0) {
                    h.end = 0;
                    h.cnt = cnt;
                    h.slab = s;
                    h.first = base == 0 && s == 0;
                    h.last = base + kDfPass >= cur.n && s == kDfSlabs - 1;
                    h.dbuf = cur.dbuf;
                    h.dpar = cur.dpar;
                    h.ch0 = cur.ch0;
                    h.nch = nch;
                }
                if (s == kDfSlabs - 1) {
#pragma unroll
                    for (int i = 0; i < kDfPass / 32; i++) h.gid[lane + 32 * i] = gid[i];
                }
                if (lane < nck)
                    tma_tile3d_g2s(&sm.w[st][lane * kChunkEntries * 32], &w_map, 32 * s, 0, (int)cid, &sm.wfull[st]);
                __syncwarp();
                if (lane == 0) mbar_arrive_expect_tx(&sm.wfull[st], (uint32_t)nck * (kChunkEntries * 32 * 4));
                step++;
            }
        }
        if (!claimed) nxt = claim();
        cur = nxt;
    }
    const int st = acquire();
    if (lane == 0) {
        sm.hdr[st].end = 1;
        mbar_arrive(&sm.wfull[st]);
    }
}

// weight_sum[g] += sum over the tile's pixels of w[entry][px], for every entry of every tile of a view's pool: the
// denominator of a lift (sgb_lift_batch).  CTA = tile, warp = one 16-entry chunk at a time; every row is read once,
// by all 32 lanes (two coalesced float4 per lane), and reduced across the warp.
__global__ void __launch_bounds__(kThreads) pool_weight_sum_kernel(PoolView pool, float* __restrict__ weight_sum) {
    const int tile = blockIdx.x, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const uint32_t n = pool.count[tile];
    const uint32_t dbase = pool.dirbase[tile];
    const int nck = (int)((n + kChunkEntries - 1) / kChunkEntries);
    for (int k = warp; k < nck; k += kThreads / 32) {
        const WChunk* ck = pool.chunks + chunk_of(pool, dbase, k);
        const int m = (int)min((uint32_t)kChunkEntries, n - (uint32_t)k * kChunkEntries);
#pragma unroll 4
        for (int s = 0; s < m; s++) {
            const float4 a = __ldg(reinterpret_cast<const float4*>(&ck->w[s][4 * lane]));
            const float4 b = __ldg(reinterpret_cast<const float4*>(&ck->w[s][128 + 4 * lane]));
            float t = ((a.x + a.y) + (a.z + a.w)) + ((b.x + b.y) + (b.z + b.w));
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
            if (lane == 0) red_add_f32(weight_sum + __ldg(&ck->meta[s].x), t);
        }
    }
}

// ------------------------------------------------------------------------------------ warp-autonomous chain backward
// A warp's 32-pixel strip is touched by only part of the tile's entries, so every warp owns its strip end to end and
// nothing is CTA-synchronous after the prologue:
//   * the warp walks the tile list from the back and COMPACTS it on the fly to the entries whose strip-mask bit is
//     set (ballot + popc ranks), 32 entries per segment: no zero-strip work, padding <= 31 slots per strip;
//   * s-pass per segment: S[32 px][32 entries] over all channels, lane tile 8 px x 4 entries (16 paired FMAs per 3
//     LDS.128); the warp stages its own operands — the dL/dout slab [16 ch][32 px] by TMA (plain loads for rows that
//     are not 16-byte aligned), the feature slab by 4 x LDG.128 per lane (lane = entry) one slab ahead in registers,
//     stored transposed [ch][entry];
//   * S is parked in the warp's dL slab region (XOR-swizzled 16-byte chunks: conflict-free both ways) and lane = pixel
//     runs the reference's back-to-front chain (backward.cu:477-550, dot-product form) over the 32 entries.
// Shared memory 9.3 KB per warp, 128 registers, 2 CTAs/SM (a third CTA would leave less L1 for the gathered feature
// rows); the warps of a tile share their feature rows through L1/L2 only.
constexpr int kChainRG = 5;  // entries whose six gradient terms are summed over the strip per flush (30 of 32 lanes busy)
struct __align__(16) ChainWarpSmem {
    float DS[2][16][32];   // dL/dout slabs [buf][ch][px of the strip]; S[32 entries][32 px] aliases it after the s-pass
    union {
        float FT[2][16][36];           // s-pass: feature slabs [buf][ch][entry]
        float RB[kChainRG * 6][32];    // chain phase: partial gradient terms, one row per (entry of the group, term)
    };
    float4 RecA[32], RecB[32];
    const float* Wrow[32];
    uint32_t Gid[32];
};
constexpr int kMetaCap = 512;  // tile-list entries whose (id, mask) records are cached in shared memory

// dL slab sl [16 ch][32 px of strip `warp`] by plain loads, for image rows that are not 16-byte aligned (no tensor
// map): lane -> (channel row (lane >> 3) + 4 i of the slab, 4-pixel piece pc = lane & 7: tile row pc >> 2 of the strip,
// columns (pc & 3) * 4 ..).  Out of line so that its addressing holds no registers in the kernel, which runs at its
// 128-register limit.
__device__ __noinline__ void dl_slab_plain(float (*DS)[32], const float* __restrict__ dL_dpixels, int W, int H, int C,
                                           uint2 pix_min, int warp, int lane, int sl) {
    constexpr int CK = 16;
    const size_t plane = (size_t)H * W;
    const int pc = lane & 7;
    const uint32_t y = pix_min.y + 2 * warp + (pc >> 2), x = pix_min.x + (pc & 3) * 4;
    const float* srcs = dL_dpixels + (size_t)(sl * CK + (lane >> 3)) * plane + (size_t)W * y + x;
#pragma unroll
    for (int i = 0; i < CK / 4; i++) {
        const int chl = (lane >> 3) + 4 * i;
        const bool chin = sl * CK + chl < C;
        const float* src = srcs + (size_t)(4 * i) * plane;
#pragma unroll
        for (int u = 0; u < 4; u++)
            DS[chl][pc * 4 + u] = (chin && y < (uint32_t)H && x + u < (uint32_t)W) ? __ldg(src + u) : 0.f;
    }
}

template <bool VEC>
__global__ void __launch_bounds__(kThreads, 2) chain_backward_warp_kernel(
    int W, int H, int C, const float* __restrict__ bg_color, const SplatRec* __restrict__ rec,
    const float* __restrict__ features, const float* __restrict__ final_Ts, const float* __restrict__ dL_dpixels,
    PoolView pool, float* __restrict__ dL_dmean2D, float* __restrict__ dL_dconic2D, float* __restrict__ dL_dopacity,
    const __grid_constant__ CUtensorMap dl_map, const int use_tma) {
    constexpr int CK = 16;
    extern __shared__ __align__(128) unsigned char smem_raw[];
    __shared__ uint2 MetaS[kMetaCap];
    __shared__ uint64_t dbar[kThreads / 32][2];  // per warp, per dL slab buffer: TMA completion
    __shared__ uint32_t Cdir[kMetaCap / kChunkEntries];

    const int tiles_x = (W + SGB_TILE - 1) / SGB_TILE;
    const int tile = blockIdx.x;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int pg = lane_group4(lane), eg = lane_group8(lane);
    ChainWarpSmem& ws = reinterpret_cast<ChainWarpSmem*>(smem_raw)[warp];
    const uint2 pix_min = {(uint32_t)(tile % tiles_x) * SGB_TILE, (uint32_t)(tile / tiles_x) * SGB_TILE};
    const uint32_t tx = tid & (SGB_TILE - 1), ty = tid >> 4;
    const uint2 pix = {pix_min.x + tx, pix_min.y + ty};
    const uint32_t pix_id = W * pix.y + pix.x;
    const float2 pixf = {(float)pix.x, (float)pix.y};
    const bool inside = pix.x < (uint32_t)W && pix.y < (uint32_t)H;
    const uint32_t n = pool.count[tile];
    if (n == 0) return;
    const uint32_t dbase = pool.dirbase[tile];
    const size_t plane = (size_t)H * W;
    const int woff = warp * 32 + lane;

    // ---- CTA prologue: directory + (id, mask) records of the tile list -> shared memory; background flag
    const uint32_t ncache = min(n, (uint32_t)kMetaCap);
    for (uint32_t k = tid; k * kChunkEntries < ncache; k += kThreads) Cdir[k] = chunk_of(pool, dbase, (int)k);
    if (lane == 0) {
        mbar_init(&dbar[warp][0], 1);
        mbar_init(&dbar[warp][1], 1);
        mbar_fence_init();
    }
    int bg_nonzero = 0;
    for (int ch = tid; ch < C; ch += kThreads) bg_nonzero |= (bg_color[ch] != 0.f);
    bg_nonzero = __syncthreads_or(bg_nonzero);   // also orders the Cdir stores and the barrier inits
    for (uint32_t e = tid; e < ncache; e += kThreads)
        MetaS[e] = __ldg(&pool.chunks[Cdir[e / kChunkEntries]].meta[e & (kChunkEntries - 1)]);
    __syncthreads();
    auto chunk_ptr = [&](uint32_t e) -> const WChunk* {
        return pool.chunks + (e < ncache ? Cdir[e / kChunkEntries] : chunk_of(pool, dbase, (int)(e / kChunkEntries)));
    };
    auto meta_of = [&](uint32_t e) -> uint2 {
        return e < ncache ? MetaS[e] : __ldg(&chunk_ptr(e)->meta[e & (kChunkEntries - 1)]);
    };

    // background term of the own pixel over all channels (backward.cu:527-529); zero background: term vanishes
    float bgdot = 0.f;
    if (inside && bg_nonzero)
        for (int ch = 0; ch < C; ch++) bgdot += bg_color[ch] * __ldg(dL_dpixels + (size_t)ch * plane + pix_id);

    const float T_final = inside ? final_Ts[pix_id] : 0.f;
    float T = T_final;
    float last_alpha = 0.f, s_last = 0.f, A = 0.f;
    const float ddelx_dx = 0.5f * W, ddely_dy = 0.5f * H;
    const int nslab = (C + CK - 1) / CK;
    float (*S)[32] = reinterpret_cast<float (*)[32]>(&ws.DS[0][0][0]);

    // dL slab [CK ch][32 px of this strip].  TMA path (image rows 16-byte aligned; the map is encoded per launch by
    // the host): ONE instruction of one lane fetches the whole [16 ch][2 rows][16 px] box — rows below the image, columns right of it and channels >= C arrive
    // as zeros — and none of it passes through the LSU data pipe (the four LDGSTS per lane it replaces were 64 of the
    // ~210 L1 wavefronts per slab, and the L1 data pipe bounds this kernel).
    uint32_t dphase = 0;  // bit b: parity the next wait on buffer b expects
    auto dissue = [&](int sl, int buf) {
        if (use_tma) {
            if (lane == 0) {
                fence_proxy_async_smem();  // S of the previous segment was written to this memory by generic stores
                mbar_arrive_expect_tx(&dbar[warp][buf], CK * 32 * sizeof(float));
                tma_tile3d_g2s(&ws.DS[buf][0][0], &dl_map, (int)pix_min.x, (int)pix_min.y + 2 * warp, sl * CK,
                               &dbar[warp][buf]);
            }
            return;
        }
        dl_slab_plain(ws.DS[buf], dL_dpixels, W, H, C, pix_min, warp, lane, sl);  // ordered by the slab loop's barrier
    };

    uint32_t cursor = n;  // tile-list entries [0, cursor) are still to be visited (back to front)
    while (cursor > 0) {
        // ---- gather the next <= 32 entries of THIS strip, walking the tile list backwards.  Slot 0 = furthest back.
        int cnt = 0;
        while (cnt < 32 && cursor > 0) {
            const bool valid = (uint32_t)lane < cursor;
            const uint32_t e = valid ? cursor - 1 - (uint32_t)lane : 0u;
            const uint2 mt = valid ? meta_of(e) : make_uint2(0u, 0u);
            const bool bit = valid && ((mt.y >> warp) & 1u);
            const uint32_t bal = __ballot_sync(0xffffffffu, bit);
            const int room = 32 - cnt;
            const int nset = __popc(bal);
            const int rank = __popc(bal & ((1u << lane) - 1u));
            if (bit && rank < room) {
                const int slot = cnt + rank;
                const WChunk* ck = chunk_ptr(e);
                ws.Wrow[slot] = &ck->w[e & (kChunkEntries - 1)][0];
                ws.Gid[slot] = mt.x;
                const float4* rp = reinterpret_cast<const float4*>(rec + mt.x);
                ws.RecA[slot] = __ldg(rp);
                ws.RecB[slot] = __ldg(rp + 1);
            }
            if (nset <= room) {
                cursor -= min(32u, cursor);
                cnt += nset;
            } else {  // segment full: resume right after the last entry taken
                const int last_lane = __ffs(__ballot_sync(0xffffffffu, bit && rank == room - 1)) - 1;
                cursor -= (uint32_t)(last_lane + 1);
                cnt = 32;
            }
        }
        __syncwarp();
        if (cnt == 0) break;

        // ---- s-pass: S[px][entry] = sum_ch dL[px][ch] * F[entry][ch]
        float2 acc[8][2];  // [px][entry pair]
#pragma unroll
        for (int i = 0; i < 8; i++) acc[i][0] = acc[i][1] = make_float2(0.f, 0.f);
        // Feature slab [32 entries][16 ch] -> FT[ch][entry].  Fast path (16-byte aligned rows, full slab): lane
        // (r8 = lane >> 2, c4 = lane & 3) loads channels 4c4..4c4+3 of entries r8 + 8q, so one LDG.128 covers 8 rows x
        // 64 contiguous bytes (8 L1 tag lookups, where lane = entry would touch a separate line per lane).  FT rows of channels 8..15 hold their 8-entry
        // blocks swapped pairwise (block b at b ^ 1) — with the 36-float pitch that makes the transposing stores of
        // this mapping conflict-free; the s-pass reads entry group eg of channel k at chunk eg ^ ((k >> 3) << 1).
        float4 fpre[CK / 4];
        const int f_r8 = lane >> 2, f_c4 = lane & 3;
        const float* frow = features + (size_t)ws.Gid[min(lane, cnt - 1)] * C;          // general path: lane = entry
        uint32_t f_gid[CK / 4];                                                            // fast path: 4 rows per lane
#pragma unroll
        for (int q = 0; q < CK / 4; q++) f_gid[q] = ws.Gid[min(f_r8 + 8 * q, cnt - 1)];    // rows >= cnt: duplicates
        auto slab_fast = [&](int sl) { return VEC && (sl + 1) * CK <= C; };
        auto fload = [&](int sl) {
            if (slab_fast(sl)) {
                const int choff = sl * CK + f_c4 * 4;
#pragma unroll
                for (int q = 0; q < CK / 4; q++)
                    fpre[q] = __ldg(reinterpret_cast<const float4*>(features + (size_t)f_gid[q] * C + choff));
                return;
            }
#pragma unroll
            for (int q = 0; q < CK / 4; q++) {
                const int chb = sl * CK + q * 4;
                fpre[q] = make_float4(0.f, 0.f, 0.f, 0.f);
                if (lane < cnt) {
                    if (VEC && chb + 4 <= C) fpre[q] = __ldg(reinterpret_cast<const float4*>(frow + chb));
                    else {
                        if (chb < C) fpre[q].x = __ldg(frow + chb);
                        if (chb + 1 < C) fpre[q].y = __ldg(frow + chb + 1);
                        if (chb + 2 < C) fpre[q].z = __ldg(frow + chb + 2);
                        if (chb + 3 < C) fpre[q].w = __ldg(frow + chb + 3);
                    }
                }
            }
        };
        const int f_swap = (f_c4 >> 1) * 8;  // channels 8..15: 8-entry blocks swapped pairwise
        auto fstore = [&](int buf, int sl) {
            if (slab_fast(sl)) {
#pragma unroll
                for (int q = 0; q < CK / 4; q++) {
                    float* col = &ws.FT[buf][f_c4 * 4][8 * q + f_r8 + ((q & 1) ? -f_swap : f_swap)];
                    col[0 * 36] = fpre[q].x;
                    col[1 * 36] = fpre[q].y;
                    col[2 * 36] = fpre[q].z;
                    col[3 * 36] = fpre[q].w;
                }
                return;
            }
#pragma unroll
            for (int q = 0; q < CK / 4; q++) {  // lane = entry, channels 4q..4q+3
                const int pos = lane ^ ((q >> 1) << 3);
                ws.FT[buf][q * 4 + 0][pos] = fpre[q].x;
                ws.FT[buf][q * 4 + 1][pos] = fpre[q].y;
                ws.FT[buf][q * 4 + 2][pos] = fpre[q].z;
                ws.FT[buf][q * 4 + 3][pos] = fpre[q].w;
            }
        };
        // One warp barrier per slab: at the top of iteration sl every lane has finished the math of slab sl-1, so the
        // other buffers (dL by TMA or plain loads, features from the registers loaded one slab earlier) can be refilled BEFORE
        // the math of slab sl and their latency hides behind it.
        fload(0);
        dissue(0, 0);
        fstore(0, 0);
        if (nslab > 1) fload(1);
        for (int sl = 0; sl < nslab; sl++) {
            const int buf = sl & 1;
            if (use_tma) {
                mbar_wait(&dbar[warp][buf], (dphase >> buf) & 1u);
                dphase ^= 1u << buf;
            }
            __syncwarp();  // DS[buf] landed, FT[buf] stored by every lane; DS/FT[buf ^ 1] are free
            if (sl + 1 < nslab) {
                dissue(sl + 1, buf ^ 1);
                fstore(buf ^ 1, sl + 1);
                if (sl + 2 < nslab) fload(sl + 2);
            }
#pragma unroll 8
            for (int k = 0; k < CK; k++) {
                const float4 d0 = *reinterpret_cast<const float4*>(&ws.DS[buf][k][pg * 8]);
                const float4 d1 = *reinterpret_cast<const float4*>(&ws.DS[buf][k][pg * 8 + 4]);
                const float4 f0 = *reinterpret_cast<const float4*>(&ws.FT[buf][k][(eg ^ ((k >> 3) << 1)) * 4]);
                const float2 fa = make_float2(f0.x, f0.y), fb = make_float2(f0.z, f0.w);
                const float d[8] = {d0.x, d0.y, d0.z, d0.w, d1.x, d1.y, d1.z, d1.w};
#pragma unroll
                for (int i = 0; i < 8; i++) {
                    const float2 d2 = make_float2(d[i], d[i]);
                    acc[i][0] = ffma2(fa, d2, acc[i][0]);
                    acc[i][1] = ffma2(fb, d2, acc[i][1]);
                }
            }
        }
        __syncwarp();  // every lane is done with DS / FT
        // ---- park S[entry][px] in the (now free) dL slab region; 16-byte chunk c of row r sits at chunk c ^ (r >> 2)
#pragma unroll
        for (int j = 0; j < 4; j++) {
            const int r = eg * 4 + j;
            float v[8];
#pragma unroll
            for (int i = 0; i < 8; i++) v[i] = (j & 1) ? acc[i][j >> 1].y : acc[i][j >> 1].x;
            *reinterpret_cast<float4*>(&S[r][((2 * pg) ^ eg) * 4]) = make_float4(v[0], v[1], v[2], v[3]);
            *reinterpret_cast<float4*>(&S[r][((2 * pg + 1) ^ eg) * 4]) = make_float4(v[4], v[5], v[6], v[7]);
        }
        __syncwarp();

        // ---- back-to-front chain over the segment (backward.cu:477-550 in dot-product form); slot 0 is the
        // furthest-back entry.  Entries go in groups of kChainRG, fully unrolled (every shared-memory address of the
        // group is a constant plus a lane term, where a runtime-indexed loop spends instructions on address
        // arithmetic); the own-pixel weights of the next group are in flight during the current
        // one.  The six per-Gaussian sums over the strip's 32 pixels go through shared memory instead of a shuffle
        // butterfly: every lane parks its terms as rows of RB, then lane r adds up row r with 8 x LDS.128 and issues
        // that row's one red.global.  16-byte chunk c of row r sits at c ^ (r & 7): conflict-free both ways.
        // The transmittance in front of an entry is recovered as T_behind + w (w = alpha T_front is what the forward
        // stored): one add instead of the reference's T / (1 - alpha), same value to an ulp and no error build-up.
        constexpr int RG = kChainRG;
        float wc[RG], wn[RG];
#pragma unroll
        for (int u = 0; u < RG; u++) wc[u] = u < cnt ? __ldg(ws.Wrow[u] + woff) : 0.f;
        for (int base = 0; base < cnt; base += RG) {
#pragma unroll
            for (int u = 0; u < RG; u++) wn[u] = base + RG + u < cnt ? __ldg(ws.Wrow[base + RG + u] + woff) : 0.f;
#pragma unroll
            for (int u = 0; u < RG; u++) {
                const int li = base + u;
                if (li < cnt) {  // warp-uniform
                    // Branch-free per lane (selects instead of `if (w != 0)`): the five entries of a group then sit in
                    // one basic block and the scheduler overlaps their LDS -> exp -> product latencies.
                    const float w = wc[u];
                    const bool on = w != 0.f;
                    const float sdot = S[li][(((lane >> 2) ^ (li >> 2)) << 2) | (lane & 3)];
                    const float4 a = ws.RecA[li], con_o = ws.RecB[li];
                    const float2 d = {a.x - pixf.x, a.y - pixf.y};
                    const float power = -0.5f * (con_o.x * d.x * d.x + con_o.z * d.y * d.y) - con_o.y * d.x * d.y;
                    const float G = __expf(power);
                    const float alpha = fminf(0.99f, con_o.w * G);
                    T += w;
                    const float A_new = last_alpha * s_last + (1.f - last_alpha) * A;
                    A = on ? A_new : A;
                    s_last = on ? sdot : s_last;
                    last_alpha = on ? alpha : last_alpha;
                    float dL_dalpha = (sdot - A) * T;
                    if (bg_nonzero) dL_dalpha -= T_final / (1.f - alpha) * bgdot;
                    const float dL_dG = con_o.w * dL_dalpha;
                    const float gdx = G * d.x, gdy = G * d.y;
                    const float dG_ddelx = -gdx * con_o.x - gdy * con_o.y;
                    const float dG_ddely = -gdy * con_o.z - gdx * con_o.y;
                    float gv[6];
                    gv[0] = dL_dG * dG_ddelx * ddelx_dx;
                    gv[1] = dL_dG * dG_ddely * ddely_dy;
                    gv[2] = -0.5f * gdx * d.x * dL_dG;
                    gv[3] = -0.5f * gdx * d.y * dL_dG;
                    gv[4] = -0.5f * gdy * d.y * dL_dG;
                    gv[5] = G * dL_dalpha;
#pragma unroll
                    for (int v = 0; v < 6; v++) {
                        const int r = u * 6 + v;  // compile-time
                        ws.RB[r][(((lane >> 2) ^ (r & 7)) << 2) | (lane & 3)] = on ? gv[v] : 0.f;
                    }
                }
            }
            __syncwarp();
            const int nvalid = min(RG, cnt - base);
            if (lane < nvalid * 6) {
                const float4* row = reinterpret_cast<const float4*>(&ws.RB[lane][0]);
                float4 t = row[lane & 7];  // chunk 0 of row `lane`
#pragma unroll
                for (int q = 1; q < 8; q++) {
                    const float4 uu = row[q ^ (lane & 7)];
                    t.x += uu.x; t.y += uu.y; t.z += uu.z; t.w += uu.w;
                }
                const float tot = (t.x + t.y) + (t.z + t.w);
                const int slot = lane / 6, comp = lane - slot * 6;
                const size_t id = ws.Gid[base + slot];
                float* dst = comp < 2 ? dL_dmean2D + id * 3 + comp
                           : comp < 5 ? dL_dconic2D + id * 4 + (comp == 4 ? 3 : comp - 2)
                                      : dL_dopacity + id;
                red_add_f32(dst, tot);
            }
            __syncwarp();
#pragma unroll
            for (int u = 0; u < RG; u++) wc[u] = wn[u];
        }
        __syncwarp();  // the next segment's gather / dL slab overwrite Gid, Wrow, Rec and S
    }
}

// ------------------------------------------------------------------------------------ host side
size_t pool_bytes(int tiles, uint32_t chunks, int64_t R, PoolView* v, void* base) {
    size_t off = 0;
    char* p = (char*)base;
    auto take = [&](size_t n) { size_t o = off; off += align_up(n); return p ? p + o : nullptr; };
    void* hdr = take(sizeof(PoolHdr));
    void* dbase = take(4 * (size_t)tiles);
    void* cnt = take(4 * (size_t)tiles);
    void* dir = take(4 * ((size_t)(R / kChunkEntries) + (size_t)tiles + 1));
    void* ch = take(sizeof(WChunk) * (size_t)chunks);
    if (v) {
        v->hdr = (PoolHdr*)hdr; v->dirbase = (uint32_t*)dbase; v->count = (uint32_t*)cnt; v->dir = (uint32_t*)dir;
        v->chunks = (WChunk*)ch; v->capacity = chunks;
    }
    return off;
}

}  // namespace

// ---- weight-pool slots ---------------------------------------------------------------------------------------
// A view's slot is the one keyed by its binning-state pointer.  The pool header of slot i is read back through
// pinned header i: the views of one batch have distinct slots, so one sync reads all their headers.
constexpr int kMaxAlphaPasses = 4;  // per view and call: the first guess and up to three grown pools

static inline int num_tiles(const sgb_view_inputs& in) {
    return ((in.W + SGB_TILE - 1) / SGB_TILE) * ((in.H + SGB_TILE - 1) / SGB_TILE);
}

static PoolSlot* slot_of(sgb_ctx* ctx, const ViewState& w) {
    for (PoolSlot& sl : ctx->pools)
        if (sl.key_bin == (const void*)w.b.point_list) return &sl;
    return nullptr;
}

// pinned readback layout: [0, 8 * SGB_MAX_BATCH) the R values of a geometry batch; then one PoolHdr (16 B) per slot
static inline PoolHdr* pinned_hdr(sgb_ctx* ctx, const PoolSlot* sl) {
    return reinterpret_cast<PoolHdr*>(reinterpret_cast<char*>(ctx->pinned) + 8 * SGB_MAX_BATCH) + (sl - ctx->pools);
}

static PoolView slot_view(const ViewState& w, const PoolSlot& sl) {
    PoolView pv;
    pool_bytes(num_tiles(w.in), sl.chunks, w.R, &pv, sl.mem.p);
    return pv;
}

static uint64_t pool_first_guess(sgb_ctx* ctx, int tiles, int64_t R) {
    // ~8 chunks (128 touching Gaussians) per tile, bounded by the instance count, at least the high-water mark
    uint64_t guess = (uint64_t)tiles * 8;
    const uint64_t by_R = (uint64_t)(R / kChunkEntries) + (uint64_t)tiles;
    if (guess > by_R) guess = by_R;
    if (guess < ctx->pool_chunks_hint) guess = ctx->pool_chunks_hint;
    if (guess < 16) guess = 16;
    return guess;
}

// Slot of a view that is about to be (re)built: the one already keyed by its binning state (a new forward through
// the same pointer replaces it), else an empty one, else the least recently used.  It is carved for the first guess,
// or keeps a larger existing carve that its memory still holds.
int weight_pool_build(sgb_ctx* ctx, const ViewState& w, cudaStream_t s) {
    PoolSlot* sl = slot_of(ctx, w);
    if (!sl)
        for (PoolSlot& c : ctx->pools)
            if (!c.valid && !c.key_bin) { sl = &c; break; }
    if (!sl) {
        sl = &ctx->pools[0];
        for (PoolSlot& c : ctx->pools)
            if (c.stamp < sl->stamp) sl = &c;
    }
    sl->valid = false;
    sl->key_bin = (const void*)w.b.point_list;
    sl->stamp = ++ctx->pool_clock;
    const int tiles = num_tiles(w.in);
    uint64_t want = pool_first_guess(ctx, tiles, w.R);
    if (sl->chunks > want && sl->mem.cap >= pool_bytes(tiles, sl->chunks, w.R, nullptr, nullptr)) want = sl->chunks;
    const uint32_t chunks = (uint32_t)want;
    int rc = sl->mem.ensure(pool_bytes(tiles, chunks, w.R, nullptr, nullptr));
    if (rc) return rc;
    sl->chunks = chunks;
    const PoolView pv = slot_view(w, *sl);
    const size_t smem = sizeof(AlphaSmem);
    static DeviceOnce attr_set;
    if (attr_set.first_use_on_device())
        SGB_CUDA(cudaFuncSetAttribute(alpha_pass_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    SGB_CUDA(cudaMemsetAsync(pv.hdr, 0, sizeof(PoolHdr), s));
    {
        StageTimer t(ctx, ST_ALPHA, s);
        alpha_pass_kernel<<<tiles, kThreads, smem, s>>>(w.im.ranges, w.b.point_list, w.in.W, w.in.H, w.g.rec,
                                                        w.im.final_T, w.im.n_contrib, w.im.tile_last, pv);
        SGB_LAUNCH_CHECK("alpha_pass_kernel", w.in.debug, s);
        ctx->launches += 1;
    }
    SGB_CUDA(cudaMemcpyAsync(pinned_hdr(ctx, sl), pv.hdr, sizeof(PoolHdr), cudaMemcpyDeviceToHost, s));
    return SGB_OK;
}

// A pool that overflowed is re-carved for the demand its header reports (the counter keeps counting past capacity)
// and built again; the rebuilt views are checked after one more sync.
int weight_pool_settle(sgb_ctx* ctx, int V, const ViewState* vw, PoolView* pv, cudaStream_t s, const bool* only) {
    bool pending[SGB_MAX_BATCH];
    for (int v = 0; v < V; v++) pending[v] = !only || only[v];
    for (int pass = 1;; pass++) {
        SGB_CUDA(cudaStreamSynchronize(s));
        bool again = false;
        for (int v = 0; v < V; v++) {
            if (!pending[v]) continue;
            const ViewState& w = vw[v];
            PoolSlot* sl = slot_of(ctx, w);
            if (!sl) { set_error("weight-pool slot of the view vanished"); return SGB_E_INVALID; }
            const PoolHdr h = *pinned_hdr(ctx, sl);
            if (h.overflow) {
                const uint64_t need = (uint64_t)h.counter + h.counter / 8 + 64;
                if (need > ctx->pool_chunks_hint) ctx->pool_chunks_hint = need;
                sl->chunks = 0;  // re-carve with the new hint
                if (pass == kMaxAlphaPasses) { set_error("weight pool kept overflowing"); return SGB_E_NOMEM; }
                int rc = weight_pool_build(ctx, w, s);
                if (rc) return rc;
                again = true;
                continue;
            }
            ctx->stat_blended_pairs = (int64_t)h.blended;
            ctx->stat_pool_chunks = h.counter;
            if (h.counter > ctx->pool_chunks_hint) ctx->pool_chunks_hint = (uint64_t)h.counter + h.counter / 16 + 16;
            sl->valid = true;
            sl->key_R = w.R;
            sl->key_W = w.in.W;
            sl->key_H = w.in.H;
            sl->key_P = w.in.P;
            pv[v] = slot_view(w, *sl);
            pending[v] = false;
        }
        if (!again) return SGB_OK;
    }
}

// A rebuild is needed only when the forward ran through another ctx or its slot was recycled.  Every hit is stamped
// before the first miss takes a slot, so the least recently used slot a miss may evict is never one of this batch.
int weight_rows_for_backward(sgb_ctx* ctx, int V, const ViewState* vw, PoolView* pv, cudaStream_t s) {
    bool miss[SGB_MAX_BATCH] = {};
    bool any = false;
    for (int v = 0; v < V; v++) {
        const ViewState& w = vw[v];
        if (w.R <= 0) continue;
        PoolSlot* sl = slot_of(ctx, w);
        if (sl && sl->valid && sl->key_R == w.R && sl->key_W == w.in.W && sl->key_H == w.in.H && sl->key_P == w.in.P) {
            sl->stamp = ++ctx->pool_clock;
            pv[v] = slot_view(w, *sl);
        } else {
            miss[v] = any = true;
        }
    }
    if (!any) return SGB_OK;
    for (int v = 0; v < V; v++) {
        if (!miss[v]) continue;
        int rc = weight_pool_build(ctx, vw[v], s);
        if (rc) return rc;
    }
    return weight_pool_settle(ctx, V, vw, pv, s, miss);
}

// A lift keeps nothing for a backward: its slots are emptied (not left valid under a scratch address that a later
// binning state could reuse) and are the first a later build takes, ahead of any training forward's slot.
void weight_pool_release(sgb_ctx* ctx, int V, const ViewState* vw) {
    for (int v = 0; v < V; v++)
        if (PoolSlot* sl = slot_of(ctx, vw[v])) {
            sl->valid = false;
            sl->key_bin = nullptr;
        }
}

// Forward GEMM of one view.  The host waited for the alpha passes only, so the caller keeps enqueueing the rest of
// its step while the GEMM runs.
int blend_forward_v3(sgb_ctx* ctx, const ViewState& w, const PoolView& pv, float* out_color, cudaStream_t s) {
    const sgb_view_inputs& in = w.in;
    const int tiles = num_tiles(in);
    const int chunks = (in.C + 63) / 64;
    const bool vec = (in.C % 4 == 0) && ((reinterpret_cast<uintptr_t>(w.colors) & 15) == 0);
    StageTimer t(ctx, ST_BLEND_FWD, s);
    ctx->launches += 1;
    if (vec) {
        constexpr int NS = 5;
        const size_t smem_f = (size_t)NS * kChunkEntries * (SGB_TILE_PIX + 64) * sizeof(float);
        static DeviceOnce fattr;
        if (fattr.first_use_on_device()) {
            SGB_CUDA(cudaFuncSetAttribute(blend_forward_tma_kernel<64, NS>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                          (int)smem_f));
        }
        blend_forward_tma_kernel<64, NS><<<tiles * chunks, kThreads, smem_f, s>>>(in.W, in.H, in.C, w.colors,
                                                                                  in.background, w.im.final_T, pv,
                                                                                  out_color);
    } else {
        // feature rows that are not 16-byte aligned slices (C % 4 != 0) cannot be bulk-copied: plain loads
        blend_forward_v3_kernel<64><<<tiles * chunks, kThreads, 0, s>>>(in.W, in.H, in.C, w.colors, in.background,
                                                                         w.im.final_T, pv, out_color);
    }
    SGB_LAUNCH_CHECK("blend_forward kernel", in.debug, s);
    return SGB_OK;
}

// dL/dout (C, H, W), fp32 or fp16, for dfeature_persistent_kernel<T>, described with its dimensions in the order
// (x, channel, y) so that one [16 px][64 ch][16 rows] box lands as [row][ch][16 px] under the swizzle df_dl4 reads
// (64-byte rows of fp32, 32-byte rows of fp16).  Returns false (the kernel then stages the tile itself) when the layout
// does not meet the TMA rules (base and row pitch multiples of 16 bytes: W % 4 == 0 in fp32, W % 8 == 0 in fp16) or
// the driver entry point is not available.
template <typename T>
static bool encode_dfeature_dl_map(CUtensorMap* map, const T* dL_dpix, int W, int H, int C) {
    const TensorMapEncodeFn encode = tensor_map_encoder();
    memset(map, 0, sizeof(*map));
    if (!encode || ((size_t)W * sizeof(T)) % 16 != 0 || (reinterpret_cast<uintptr_t>(dL_dpix) & 15) != 0) return false;
    const cuuint64_t dims[3] = {(cuuint64_t)W, (cuuint64_t)C, (cuuint64_t)H};
    const cuuint64_t strides[2] = {(cuuint64_t)W * H * sizeof(T), (cuuint64_t)W * sizeof(T)};
    const cuuint32_t box[3] = {SGB_TILE, kDfCH, SGB_TILE};
    const cuuint32_t estr[3] = {1, 1, 1};
    const bool f32 = sizeof(T) == 4;
    return encode(map, f32 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 3,
                  const_cast<T*>(dL_dpix), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                  f32 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_32B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

// The weight rows of a pool as (pixel, row of the chunk, chunk): a [32 px][16 rows] box is one 32-pixel slab of a
// 16-entry chunk, stored under the 128-byte swizzle.
static bool encode_dfeature_w_map(CUtensorMap* map, const PoolView& pv) {
    const TensorMapEncodeFn encode = tensor_map_encoder();
    memset(map, 0, sizeof(*map));
    if (!encode) return false;
    const cuuint64_t dims[3] = {(cuuint64_t)SGB_TILE_PIX, (cuuint64_t)kChunkEntries, (cuuint64_t)pv.capacity};
    const cuuint64_t strides[2] = {(cuuint64_t)SGB_TILE_PIX * sizeof(float), (cuuint64_t)sizeof(WChunk)};
    const cuuint32_t box[3] = {32, kChunkEntries, 1};
    const cuuint32_t estr[3] = {1, 1, 1};
    return encode(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, reinterpret_cast<char*>(pv.chunks) + offsetof(WChunk, w),
                  dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                  CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

template <typename T>
int blend_backward_v3_dfeature(sgb_ctx* ctx, const ViewState& w, const PoolView& pv, const T* dL_dpix,
                               float* dL_dcolors, cudaStream_t s) {
    const sgb_view_inputs& in = w.in;
    const int items = num_tiles(in) * ((in.C + kDfCH - 1) / kDfCH);
    if (items == 0) return SGB_OK;
    CUtensorMap dl_map, w_map;
    const int use_tma = encode_dfeature_dl_map(&dl_map, dL_dpix, in.W, in.H, in.C) ? 1 : 0;
    if (!encode_dfeature_w_map(&w_map, pv)) {
        set_error("dL/dfeature: cuTensorMapEncodeTiled is unavailable or rejected the weight pool");
        return SGB_E_CUDA;
    }
    int rc = ctx->work.ensure(sizeof(int));
    if (rc) return rc;
    // persistent grid: as many CTAs as are co-resident on the device
    static DeviceOnce attr_set;
    static int grid_of_device[64];
    int dev = 0;
    SGB_CUDA(cudaGetDevice(&dev));
    int& grid = grid_of_device[dev < 64 ? dev : 63];
    if (attr_set.first_use_on_device()) {
        SGB_CUDA(cudaFuncSetAttribute(dfeature_persistent_kernel<T>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                      (int)kDfSmemBytes<T>));
        int per_sm = 0, sms = 0;
        SGB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, dfeature_persistent_kernel<T>, kDfThreads,
                                                               kDfSmemBytes<T>));
        SGB_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
        grid = per_sm * sms > 0 ? per_sm * sms : 1;
    }
    int* counter = static_cast<int*>(ctx->work.p);
    StageTimer t(ctx, ST_DFEATURE, s);
    SGB_CUDA(cudaMemsetAsync(counter, 0, sizeof(int), s));
    ctx->launches += 1;
    dfeature_persistent_kernel<T><<<grid < items ? grid : items, kDfThreads, kDfSmemBytes<T>, s>>>(
        in.W, in.H, in.C, dL_dpix, pv, dL_dcolors, counter, dl_map, w_map, use_tma);
    SGB_LAUNCH_CHECK("dfeature_persistent_kernel", in.debug, s);
    return SGB_OK;
}

template int blend_backward_v3_dfeature<float>(sgb_ctx*, const ViewState&, const PoolView&, const float*, float*,
                                               cudaStream_t);
template int blend_backward_v3_dfeature<__half>(sgb_ctx*, const ViewState&, const PoolView&, const __half*, float*,
                                                cudaStream_t);

int pool_weight_sums(sgb_ctx* ctx, const ViewState& w, const PoolView& pv, float* weight_sum, cudaStream_t s) {
    StageTimer t(ctx, ST_WEIGHT_SUM, s);
    ctx->launches += 1;
    pool_weight_sum_kernel<<<num_tiles(w.in), kThreads, 0, s>>>(pv, weight_sum);
    SGB_LAUNCH_CHECK("pool_weight_sum_kernel", w.in.debug, s);
    return SGB_OK;
}

// Tensor map of dL/dout (C, H, W) fp32 with a [16 ch][2 rows][16 px] box for the chain kernel's slab loads.  Returns
// false (the kernel then loads the slabs with plain loads) when the layout does not meet the TMA rules (base and row
// pitch multiples of 16 bytes) or the driver entry point is not available.
static bool encode_dl_map(CUtensorMap* map, const float* dL_dpix, int W, int H, int C) {
    const TensorMapEncodeFn encode = tensor_map_encoder();
    memset(map, 0, sizeof(*map));
    if (!encode || (W & 3) != 0 || (reinterpret_cast<uintptr_t>(dL_dpix) & 15) != 0) return false;
    const cuuint64_t dims[3] = {(cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)C};
    const cuuint64_t strides[2] = {(cuuint64_t)W * sizeof(float), (cuuint64_t)W * H * sizeof(float)};
    const cuuint32_t box[3] = {SGB_TILE, 2, 16};
    const cuuint32_t estr[3] = {1, 1, 1};
    return encode(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, const_cast<float*>(dL_dpix), dims, strides, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

int blend_backward_v3_chain(sgb_ctx* ctx, const ViewState& w, const PoolView& pv, const float* dL_dpix,
                            float* dL_dmean2D, float* dL_dconic, float* dL_dopacity, cudaStream_t s) {
    const sgb_view_inputs& in = w.in;
    const int tiles = num_tiles(in);
    const bool vec = (in.C % 4 == 0) && ((reinterpret_cast<uintptr_t>(w.colors) & 15) == 0);
    const size_t smem = sizeof(ChainWarpSmem) * (kThreads / 32);
    static DeviceOnce attr_set;
    if (attr_set.first_use_on_device()) {
        SGB_CUDA(cudaFuncSetAttribute(chain_backward_warp_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        SGB_CUDA(cudaFuncSetAttribute(chain_backward_warp_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    }
    StageTimer t(ctx, ST_BLEND_BWD, s);
    ctx->launches += 1;
    CUtensorMap dl_map;
    const int use_tma = encode_dl_map(&dl_map, dL_dpix, in.W, in.H, in.C) ? 1 : 0;
    auto kern = vec ? chain_backward_warp_kernel<true> : chain_backward_warp_kernel<false>;
    kern<<<tiles, kThreads, smem, s>>>(in.W, in.H, in.C, in.background, w.g.rec, w.colors, w.im.final_T, dL_dpix, pv,
                                       dL_dmean2D, dL_dconic, dL_dopacity, dl_map, use_tma);
    SGB_LAUNCH_CHECK("chain backward kernel", in.debug, s);
    return SGB_OK;
}

}  // namespace sgb
