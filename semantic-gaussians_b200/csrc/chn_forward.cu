// Forward contraction of the C-channel blend (chn_blend.cuh): out[px][ch] = sum over the tile's weight rows.
#include "chn_blend.cuh"
#include "tma.cuh"

namespace sgb {

namespace {

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
// false: channels cg*MCH .. cg*MCH+MCH-1 (blend_forward_ldg_kernel).  Self-contained (own accumulators, own
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
__global__ void __launch_bounds__(kTileThreads, 2) blend_forward_ldg_kernel(
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
__global__ void __launch_bounds__(kTileThreads, 2) blend_forward_tma_kernel(
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
            mbar_init(&empty_bar[i], kTileThreads / 32);
        }
        mbar_fence_init();
    }
    for (int k = tid; k < min(nb, kDirCap); k += kTileThreads) Cdir[k] = chunk_of(pool, dbase, k);
    {
        const uint32_t x = pix_min.x + (tid & (SGB_TILE - 1)), y = pix_min.y + (tid >> 4);
        Tsm[tid] = (x < (uint32_t)W && y < (uint32_t)H) ? final_T[(size_t)W * y + x] : 0.f;
        if (tid < nch) bgS[tid] = bg_color[ch0 + tid];
    }
    if (nch < CH)  // zero the never-written tail of every feature row once
        for (int e = tid; e < NS * ES * CH; e += kTileThreads) {
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

}  // namespace

// Forward GEMM of one view.  The host waited for the alpha passes only, so the caller keeps enqueueing the rest of
// its step while the GEMM runs.
int chn_forward(sgb_ctx* ctx, const ViewState& w, const PoolView& pv, float* out_color, cudaStream_t s) {
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
        blend_forward_tma_kernel<64, NS><<<tiles * chunks, kTileThreads, smem_f, s>>>(in.W, in.H, in.C, w.colors,
                                                                                  in.background, w.im.final_T, pv,
                                                                                  out_color);
    } else {
        // feature rows that are not 16-byte aligned slices (C % 4 != 0) cannot be bulk-copied: plain loads
        blend_forward_ldg_kernel<64><<<tiles * chunks, kTileThreads, 0, s>>>(in.W, in.H, in.C, w.colors, in.background,
                                                                          w.im.final_T, pv, out_color);
    }
    SGB_LAUNCH_CHECK("blend_forward kernel", in.debug, s);
    return SGB_OK;
}

}  // namespace sgb
