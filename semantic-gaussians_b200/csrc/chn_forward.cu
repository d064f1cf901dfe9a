// Forward contraction of the C-channel blend (chn_blend.cuh): out[px][ch] = sum over the tile's weight rows.
#include <cstring>
#include "chn_blend.cuh"
#include "persistent.cuh"

namespace sgb {

namespace {

// out[px][ch] = sum over the tile's entries e of w[e][px] * f[gid(e)][ch]   (K = entries), then + T[px] * bg[ch].
// Persistent: the grid fills the GPU once and every CTA claims work items (tile, up to 128 channels; a wider C splits
// into items of equal width, a multiple of 16, with the channel part varying fastest so that the items of a tile run
// at the same time and share its weight rows in L2) from a counter until none are left.  Three warp groups:
//   * WG0 is the producer.  It gives up registers (setmaxnreg) and one warp streams the tile's pool chunks through a
//     ring of kFwStages stages, one 16-entry chunk per stage: the chunk's weight rows w[16][256] (one 16 KB bulk
//     copy: they are contiguous in WChunk) and the 16 feature slices of the item's channels (one bulk copy per entry,
//     lanes 0-15).  Feature rows that are not 16-byte slices (C % 4 != 0 or a misaligned table) are staged by the
//     producer warp into the same layout on the same mbarrier with 4-byte cp.async (zero-filled past the item).  An
//     empty tile still takes one stage, with no copies: its output is T * bg.
//   * WG1 and WG2 compute (8 warps) and take the registers WG0 gave up.  Warp w owns strip w of the tile (tile rows
//     2w and 2w + 1, 32 px) and every channel of the item.  Lane (pg = lane_group4, cg = lane_group8) accumulates
//     8 px x 16 channels {32q + 4cg .. 32q + 4cg + 3, q < 4} in 128 scalar registers: per entry 2 LDS.128 of weights
//     and 4 of features (the 8 cg lanes read 128 contiguous bytes), each one wavefront, for 128 FMAs.  Channel groups
//     q past the item are not computed and a lane's channels at or past the item's width read as zero, so a stale
//     ring slot never reaches an accumulator.
// The compute warps release a stage before the item's epilogue, so the producer fills the next item's stages while
// they store this one.  The epilogue writes the warp's 32 px x item slice into its own shared-memory box and one lane
// hands the box to the TMA engine as a tensor store, so the 64 KB per item and warp group drain to global memory
// while the warps compute the next item.  With plain stores the 8 compute warps of a CTA reach their epilogue
// together and stall on the store queue: about 0.57 of 3.24 ms at K3 (H100 80GB HBM3, 700 W).  The output boxes
// (128 KB) leave room for a ring of 4 stages.  Plain stores remain for rows that are not 16-byte multiples
// (W % 4 != 0) or an unaligned output.
// Each accumulator starts at 0 and adds the tile's entries 0 .. n-1 in order with fmaf.
constexpr int kFwCH = 128;                   // widest work item (channels)
constexpr int kFwStages = 4;                 // ring depth (one 16-entry pool chunk per stage)
constexpr int kFwComputeWarps = SGB_TILE_PIX / 32;     // 2 warp groups, one 32-pixel strip per warp
constexpr int kFwThreads = 128 + 32 * kFwComputeWarps;  // producer warp group + 2 compute warp groups
constexpr uint32_t kFwProducerRegs = 56, kFwComputeRegs = 224;
static_assert(warp_group_regs_fit(kFwProducerRegs, kFwComputeWarps, kFwComputeRegs),
              "forward: the warp groups' register limits exceed the register file");

struct FwHdr {  // one ring stage's description, written by the producer before the stage is armed
    int end;             // no more work
    int cnt;             // entries of the chunk (0: empty tile)
    int first, last;     // first / last chunk of the item
    int tile, ch0, nch;  // the item
    uint32_t n, dbase;   // the tile's entry count and directory base (for the guarded recompute)
};
struct FwStage {
    float w[kChunkEntries][SGB_TILE_PIX];
    float f[kChunkEntries][kFwCH];
};
struct FwSmem {
    FwStage stg[kFwStages];
    float out[kFwComputeWarps][kFwCH][2][SGB_TILE];  // each compute warp's output box [channel][tile row][16 px]
    MbarRing<kFwStages, FwHdr> ring;
};
constexpr size_t kFwSmemBytes = sizeof(FwSmem);
static_assert(kFwSmemBytes <= 227 * 1024, "forward shared memory exceeds the sm_90 opt-in limit");

// Channel (within the item) of accumulator column k of lane group cg.
__device__ __forceinline__ int fw_channel(int k, int cg) { return (k >> 2) * 32 + cg * 4 + (k & 3); }

// Non-finite features.  The contraction multiplies every (pixel, entry) pair of a tile, zero weights included, and
// 0 * inf = NaN: one non-finite feature row would poison every pixel of every tile its Gaussian is binned to, where
// the reference only touches the pixels that actually blend it (forward.cu:340-356 `continue`s before the
// accumulation).  A pair is blended exactly when its weight alpha * T is non-zero (alpha >= 1/255 and T >= 1e-4 on
// that path), so the exact semantics are "accumulate only where w != 0".  Guarding every FMA would double the inner
// loop; instead the epilogue tests the accumulators (acc * 0 summed: NaN iff any accumulator is non-finite) and only
// a warp that sees a non-finite value recomputes its 32 px x item slice with the guarded loop below before it stores.
__device__ __forceinline__ bool acc_nonfinite(const float (&acc)[8][16]) {
    float z0 = 0.f, z1 = 0.f;
#pragma unroll
    for (int i = 0; i < 8; i++)
#pragma unroll
        for (int k = 0; k < 16; k += 2) {
            z0 = fmaf(acc[i][k], 0.f, z0);
            z1 = fmaf(acc[i][k + 1], 0.f, z1);
        }
    const float t = z0 + z1;
    return __any_sync(0xffffffffu, t != t);
}

// The guarded recompute of one warp's strip into the same register tile: straight from the pool and the feature
// table, entries in order, only where w != 0.  Reusing the fast path's accumulators (every index a constant) keeps
// the kernel free of a call and of a stack frame.
__device__ __forceinline__ void forward_redo_guarded(float (&acc)[8][16], const PoolView& pool, uint32_t n,
                                                     uint32_t dbase, const float* __restrict__ features, int C,
                                                     int ch0, int nch, int strip, int woff, int cg) {
#pragma unroll
    for (int i = 0; i < 8; i++)
#pragma unroll
        for (int k = 0; k < 16; k++) acc[i][k] = 0.f;
#pragma unroll 1
    for (uint32_t e = 0; e < n; e++) {
        const WChunk* ck = pool.chunks + chunk_of(pool, dbase, (int)(e / kChunkEntries));
        const int s = (int)(e & (kChunkEntries - 1));
        const uint2 meta = ck->meta[s];
        if (!((meta.y >> strip) & 1u)) continue;
        const float* fr = features + (size_t)meta.x * C + ch0;
        float f[16];
#pragma unroll
        for (int k = 0; k < 16; k++) {
            const int chl = fw_channel(k, cg);
            f[k] = chl < nch ? __ldg(fr + chl) : 0.f;
        }
#pragma unroll
        for (int i = 0; i < 8; i++) {
            const float w = ck->w[s][woff + i];
            if (w != 0.f) {
#pragma unroll
                for (int k = 0; k < 16; k++) acc[i][k] = fmaf(f[k], w, acc[i][k]);
            }
        }
    }
}

// One entry of a stage: acc[i][4q + j] += f[32q + 4cg + j] * w[woff + i], q < NQ.  MASK: the last group q = NQ - 1 of
// this lane reads as zero unless last_ok (its channels are past the item).
template <int NQ, bool MASK>
__device__ __forceinline__ void fw_entry(float (&acc)[8][16], const float* __restrict__ wr,
                                         const float* __restrict__ fr, bool last_ok) {
    const float4 w0 = *reinterpret_cast<const float4*>(wr);
    const float4 w1 = *reinterpret_cast<const float4*>(wr + 4);
    float4 f[NQ];
#pragma unroll
    for (int q = 0; q < NQ; q++) f[q] = *reinterpret_cast<const float4*>(fr + q * 32);
    if (MASK && !last_ok) f[NQ - 1] = make_float4(0.f, 0.f, 0.f, 0.f);
    const float wv[8] = {w0.x, w0.y, w0.z, w0.w, w1.x, w1.y, w1.z, w1.w};
#pragma unroll
    for (int i = 0; i < 8; i++) {
#pragma unroll
        for (int q = 0; q < NQ; q++) {
            acc[i][4 * q + 0] = fmaf(f[q].x, wv[i], acc[i][4 * q + 0]);
            acc[i][4 * q + 1] = fmaf(f[q].y, wv[i], acc[i][4 * q + 1]);
            acc[i][4 * q + 2] = fmaf(f[q].z, wv[i], acc[i][4 * q + 2]);
            acc[i][4 * q + 3] = fmaf(f[q].w, wv[i], acc[i][4 * q + 3]);
        }
    }
}

// The cnt entries of one stage; ws / fs point at this lane's pixels of weight row 0 and its channels of feature row 0.
// Dense on purpose: skipping strips whose 32 weights are all zero breaks the unrolled load / FMA pipeline.
template <int NQ, bool MASK>
__device__ __forceinline__ void fw_chunk(float (&acc)[8][16], const float* __restrict__ ws,
                                         const float* __restrict__ fs, int cnt, bool last_ok) {
    if (cnt == kChunkEntries) {
#pragma unroll
        for (int e = 0; e < kChunkEntries; e++)
            fw_entry<NQ, MASK>(acc, ws + e * SGB_TILE_PIX, fs + e * kFwCH, last_ok);
    } else {
#pragma unroll 1
        for (int e = 0; e < cnt; e++) fw_entry<NQ, MASK>(acc, ws + e * SGB_TILE_PIX, fs + e * kFwCH, last_ok);
    }
}

// CW: channels per work item (a multiple of 16, at most kFwCH).  use_bulk: the feature slices are 16-byte aligned
// (C % 4 == 0 and an aligned table) and go through bulk copies; otherwise the producer warp stages them.
__global__ void __launch_bounds__(kFwThreads, 1) blend_forward_persistent_kernel(
    int W, int H, int C, int CW, const float* __restrict__ features, const float* __restrict__ bg_color,
    const float* __restrict__ final_T, PoolView pool, float* __restrict__ out_color, int* __restrict__ work_counter,
    const int use_bulk, const __grid_constant__ CUtensorMap out_map, const int use_tma_store) {
    extern __shared__ __align__(128) unsigned char smem_raw[];
    FwSmem& sm = *reinterpret_cast<FwSmem*>(smem_raw);
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int tiles_x = (W + SGB_TILE - 1) / SGB_TILE;
    if (tid == 0) sm.ring.init(!use_bulk, kFwComputeWarps);
    __syncthreads();

    if (warp >= 4) {
        setmaxnreg_inc<kFwComputeRegs>();
        const int strip = warp - 4;
        const int pg = lane_group4(lane), cg = lane_group8(lane);
        const int woff = strip * 32 + pg * 8;  // this lane's 8 pixels (tile-local)
        const size_t plane = (size_t)H * W;
        float acc[8][16];
        float Tl = 0.f, bgl[4] = {0.f, 0.f, 0.f, 0.f};  // final_T of strip pixel `lane`, bg of item channel lane + 32q
        for (uint32_t step = 0;; step++) {
            const int st = sm.ring.wait(step);
            const FwHdr& h = sm.ring.hdr[st];
            if (h.end) break;
            const int cnt = h.cnt, last = h.last, tile = h.tile, ch0 = h.ch0, nch = h.nch;
            const uint32_t n = h.n, dbase = h.dbase;
            const uint32_t x0 = (uint32_t)(tile % tiles_x) * SGB_TILE, y0 = (uint32_t)(tile / tiles_x) * SGB_TILE;
            if (h.first) {
#pragma unroll
                for (int i = 0; i < 8; i++)
#pragma unroll
                    for (int k = 0; k < 16; k++) acc[i][k] = 0.f;
                // the epilogue's operands, loaded now so that they have landed by the item's end
                const uint32_t x = x0 + (lane & 15), y = y0 + 2 * strip + (lane >> 4);
                Tl = (x < (uint32_t)W && y < (uint32_t)H) ? __ldg(final_T + (size_t)W * y + x) : 0.f;
#pragma unroll
                for (int q = 0; q < 4; q++) bgl[q] = lane + 32 * q < nch ? __ldg(bg_color + ch0 + lane + 32 * q) : 0.f;
            }
            if (cnt > 0) {
                const float* ws = &sm.stg[st].w[0][woff];
                const float* fs = &sm.stg[st].f[0][cg * 4];
                const int nq = (nch + 31) >> 5;
                const bool last_ok = (nq - 1) * 32 + cg * 4 < nch;
                if (nq == 4 && (nch & 31) == 0) {
                    fw_chunk<4, false>(acc, ws, fs, cnt, true);
                } else {
                    switch (nq) {
                        case 1: fw_chunk<1, true>(acc, ws, fs, cnt, last_ok); break;
                        case 2: fw_chunk<2, true>(acc, ws, fs, cnt, last_ok); break;
                        case 3: fw_chunk<3, true>(acc, ws, fs, cnt, last_ok); break;
                        default: fw_chunk<4, true>(acc, ws, fs, cnt, last_ok); break;
                    }
                }
            }
            sm.ring.release(st, lane);
            if (!last) continue;

            // ---- epilogue: out = acc + T * bg (forward.cu:372-373)
            const uint32_t row = y0 + 2 * strip + (pg >> 1);
            const uint32_t col0 = x0 + (pg & 1) * 8;
            float Tv[8], bgv[16];
#pragma unroll
            for (int i = 0; i < 8; i++) Tv[i] = __shfl_sync(0xffffffffu, Tl, pg * 8 + i);
#pragma unroll
            for (int k = 0; k < 16; k++) bgv[k] = __shfl_sync(0xffffffffu, bgl[k >> 2], cg * 4 + (k & 3));
            if (acc_nonfinite(acc)) forward_redo_guarded(acc, pool, n, dbase, features, C, ch0, nch, strip, woff, cg);
            if (use_tma_store) {
                // into the warp's box, then one tensor store that the TMA engine drains while the warp computes the
                // next item; channels past the item and pixels past the image lie outside the tensor or the box
                float(&box)[kFwCH][2][SGB_TILE] = sm.out[strip];
                if (lane == 0) bulk_wait_read_all();  // the previous item's store has read the box
                __syncwarp();
#pragma unroll
                for (int k = 0; k < 16; k++) {
                    float o[8];
#pragma unroll
                    for (int i = 0; i < 8; i++) o[i] = acc[i][k] + Tv[i] * bgv[k];
                    float4* dst = reinterpret_cast<float4*>(&box[fw_channel(k, cg)][pg >> 1][(pg & 1) * 8]);
                    dst[0] = make_float4(o[0], o[1], o[2], o[3]);
                    dst[1] = make_float4(o[4], o[5], o[6], o[7]);
                }
                fence_proxy_async_smem();
                __syncwarp();
                if (lane == 0) tma_store3d_s2g(&out_map, (int)x0, (int)y0 + 2 * strip, ch0, &box[0][0][0]);
            } else if (row < (uint32_t)H) {
                const bool vec = ((W & 3) == 0) && (col0 + 8 <= (uint32_t)W);
#pragma unroll
                for (int k = 0; k < 16; k++) {
                    const int chl = fw_channel(k, cg);
                    if (chl >= nch) continue;
                    float* dst = out_color + (size_t)(ch0 + chl) * plane + (size_t)W * row + col0;
                    float o[8];
#pragma unroll
                    for (int i = 0; i < 8; i++) o[i] = acc[i][k] + Tv[i] * bgv[k];
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
        if (use_tma_store && lane == 0) bulk_wait_all();
        return;
    }

    // ---- producer warp group: warp 0 streams, warps 1-3 only hand their registers back
    setmaxnreg_dec<kFwProducerRegs>();
    if (warp != 0) return;
    const int tiles = tiles_x * ((H + SGB_TILE - 1) / SGB_TILE);
    const int nitems = (C + CW - 1) / CW;
    const int total = tiles * nitems;
    uint32_t step = 0;  // ring stages armed so far
    for (;;) {
        const int k = claim_item(work_counter, lane);
        if (k >= total) break;
        const int tile = k / nitems, ch0 = (k % nitems) * CW;
        const int nch = min(CW, C - ch0);
        const int nch4 = (nch + 3) & ~3;  // staged feature columns (zero past nch)
        const uint32_t n = pool.count[tile];
        const uint32_t dbase = pool.dirbase[tile];
        const int nck = (int)((n + kChunkEntries - 1) / kChunkEntries);
        // chunk ids of chunks 32b .. 32b + 31 of the tile, one per lane; the Gaussian ids of chunk j + 1 are fetched
        // while chunk j waits for its stage
        uint32_t cid = 0u;
        auto chunk_id = [&](int j) {
            if ((j & 31) == 0) cid = lane < nck - j ? chunk_of(pool, dbase, j + lane) : 0u;
            return __shfl_sync(0xffffffffu, cid, j & 31);
        };
        auto gid_of = [&](uint32_t c, int j) {  // lanes 0-15: Gaussian id of entry `lane` of chunk j
            const int cntj = min(kChunkEntries, (int)n - j * kChunkEntries);
            return lane < cntj ? __ldg(&pool.chunks[c].meta[lane].x) : 0u;
        };
        uint32_t c_cur = 0u, g_cur = 0u;
        if (nck > 0) {
            c_cur = chunk_id(0);
            g_cur = gid_of(c_cur, 0);
        }
        for (int j = 0; j < max(nck, 1); j++) {
            const int cnt = nck > 0 ? min(kChunkEntries, (int)n - j * kChunkEntries) : 0;
            uint32_t c_next = 0u, g_next = 0u;
            if (j + 1 < nck) {
                c_next = chunk_id(j + 1);
                g_next = gid_of(c_next, j + 1);
            }
            const int st = sm.ring.acquire(step);
            FwHdr& h = sm.ring.hdr[st];
            if (lane == 0) {
                h.end = 0;
                h.cnt = cnt;
                h.first = j == 0;
                h.last = j + 1 >= nck;
                h.tile = tile;
                h.ch0 = ch0;
                h.nch = nch;
                h.n = n;
                h.dbase = dbase;
            }
            FwStage& sg = sm.stg[st];
            if (cnt > 0 && lane == 0)
                bulk_g2s(&sg.w[0][0], &pool.chunks[c_cur].w[0][0], (uint32_t)cnt * (SGB_TILE_PIX * 4u), &sm.ring.full[st]);
            if (use_bulk) {
                if (lane < cnt)
                    bulk_g2s(&sg.f[lane][0], features + (size_t)g_cur * C + ch0, (uint32_t)nch * 4u, &sm.ring.full[st]);
            } else {
#pragma unroll 1
                for (int e = 0; e < cnt; e++) {
                    const float* src = features + (size_t)__shfl_sync(0xffffffffu, g_cur, e) * C + ch0;
                    for (int c = lane; c < nch4; c += 32) cp_async4(&sg.f[e][c], c < nch ? src + c : src, c < nch ? 4 : 0);
                }
                cp_async_mbar_arrive_noinc(&sm.ring.full[st]);
            }
            __syncwarp();
            if (lane == 0)
                mbar_arrive_expect_tx(&sm.ring.full[st], (uint32_t)cnt * (SGB_TILE_PIX * 4u + (use_bulk ? (uint32_t)nch * 4u : 0u)));
            step++;
            c_cur = c_next;
            g_cur = g_next;
        }
    }
    sm.ring.finish(step, !use_bulk, lane);
}

}  // namespace

// The output (C, H, W) as (x, y, channel): one [16 px][2 rows][CW channels] box is a compute warp's strip of an item.
// False (the kernel then stores with plain stores) when a row is not a multiple of 16 bytes (W % 4 != 0), the base is
// not 16-byte aligned or the driver entry point is not available.
static bool encode_forward_out_map(CUtensorMap* map, float* out, int W, int H, int C, int CW) {
    memset(map, 0, sizeof(*map));
    if ((W & 3) != 0 || (reinterpret_cast<uintptr_t>(out) & 15) != 0) return false;
    const cuuint64_t dims[3] = {(cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)C};
    const cuuint64_t strides[2] = {(cuuint64_t)W * sizeof(float), (cuuint64_t)W * H * sizeof(float)};
    const cuuint32_t box[3] = {SGB_TILE, 2, (cuuint32_t)CW};
    return encode_tiled_map(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, out, dims, strides, box,
                            CU_TENSOR_MAP_SWIZZLE_NONE);
}

// Forward GEMM of one view.  The host waited for the alpha passes only, so the caller keeps enqueueing the rest of
// its step while the GEMM runs.
int chn_forward(sgb_ctx* ctx, const ViewState& w, const PoolView& pv, float* out_color, cudaStream_t s) {
    const sgb_view_inputs& in = w.in;
    const ItemSplit sp = split_channels(in.C, kFwCH);  // one item at C <= 128, two at C = 256, four at C = 512
    const int CW = sp.CW;
    const int items = num_tiles(in) * sp.nitems;
    if (items == 0) return SGB_OK;
    const int use_bulk = (in.C % 4 == 0) && ((reinterpret_cast<uintptr_t>(w.colors) & 15) == 0);
    CUtensorMap out_map;
    const int use_tma_store = encode_forward_out_map(&out_map, out_color, in.W, in.H, in.C, CW) ? 1 : 0;
    StageTimer t(ctx, ST_BLEND_FWD, s);
    int grid = 0;
    const int rc = persistent_grid<blend_forward_persistent_kernel>(ctx, kFwThreads, kFwSmemBytes, items, s, &grid);
    if (rc) return rc;
    ctx->launches += 1;
    blend_forward_persistent_kernel<<<grid, kFwThreads, kFwSmemBytes, s>>>(
        in.W, in.H, in.C, CW, w.colors, in.background, w.im.final_T, pv, out_color, static_cast<int*>(ctx->work.p),
        use_bulk, out_map, use_tma_store);
    SGB_LAUNCH_CHECK("blend_forward_persistent_kernel", in.debug, s);
    return SGB_OK;
}

}  // namespace sgb
