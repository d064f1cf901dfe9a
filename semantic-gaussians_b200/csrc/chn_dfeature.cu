// dL/dfeature contraction of the C-channel blend (chn_blend.cuh); also the numerator of a lift (sgb_lift_batch).
#include <cstddef>
#include <cstring>
#include "chn_blend.cuh"
#include "tma.cuh"

namespace sgb {

namespace {

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
constexpr int kDfThreads = kTileThreads + 32;   // 8 compute warps + 1 producer warp
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
    constexpr int kComputeWarps = kTileThreads / 32;
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

}  // namespace

// dL/dout (C, H, W), fp32 or fp16, for dfeature_persistent_kernel<T>, described with its dimensions in the order
// (x, channel, y) so that one [16 px][64 ch][16 rows] box lands as [row][ch][16 px] under the swizzle df_dl4 reads
// (64-byte rows of fp32, 32-byte rows of fp16).  Returns false (the kernel then stages the tile itself) when the layout
// does not meet the TMA rules (base and row pitch multiples of 16 bytes: W % 4 == 0 in fp32, W % 8 == 0 in fp16) or
// the driver entry point is not available.
template <typename T>
static bool encode_dfeature_dl_map(CUtensorMap* map, const T* dL_dpix, int W, int H, int C) {
    memset(map, 0, sizeof(*map));
    if (((size_t)W * sizeof(T)) % 16 != 0 || (reinterpret_cast<uintptr_t>(dL_dpix) & 15) != 0) return false;
    const cuuint64_t dims[3] = {(cuuint64_t)W, (cuuint64_t)C, (cuuint64_t)H};
    const cuuint64_t strides[2] = {(cuuint64_t)W * H * sizeof(T), (cuuint64_t)W * sizeof(T)};
    const cuuint32_t box[3] = {SGB_TILE, kDfCH, SGB_TILE};
    const bool f32 = sizeof(T) == 4;
    return encode_tiled_map(map, f32 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 3, dL_dpix,
                            dims, strides, box, f32 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_32B);
}

// The weight rows of a pool as (pixel, row of the chunk, chunk): a [32 px][16 rows] box is one 32-pixel slab of a
// 16-entry chunk, stored under the 128-byte swizzle.
static bool encode_dfeature_w_map(CUtensorMap* map, const PoolView& pv) {
    memset(map, 0, sizeof(*map));
    const cuuint64_t dims[3] = {(cuuint64_t)SGB_TILE_PIX, (cuuint64_t)kChunkEntries, (cuuint64_t)pv.capacity};
    const cuuint64_t strides[2] = {(cuuint64_t)SGB_TILE_PIX * sizeof(float), (cuuint64_t)sizeof(WChunk)};
    const cuuint32_t box[3] = {32, kChunkEntries, 1};
    return encode_tiled_map(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3,
                            reinterpret_cast<char*>(pv.chunks) + offsetof(WChunk, w), dims, strides, box,
                            CU_TENSOR_MAP_SWIZZLE_128B);
}

template <typename T>
static int launch_dfeature(sgb_ctx* ctx, const ViewState& w, const PoolView& pv, const T* dL_dpix, float* dL_dcolors,
                           cudaStream_t s) {
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

// fp16 before fp32 on purpose.  The order of these two definitions is the order in which the kernels are instantiated,
// and with fp32 first nvcc 12.9 emits the fp32 kernel's accumulator-reset selects in an order that changes from one
// compile of the same source to the next (equivalent code, but ptxas then schedules ~10 % of the kernel differently).
// In this order 40 of 40 compiles gave the same PTX.
int chn_dfeature(sgb_ctx* ctx, const ViewState& w, const PoolView& pv, const __half* dL_dpix, float* dL_dcolors,
                 cudaStream_t s) {
    return launch_dfeature(ctx, w, pv, dL_dpix, dL_dcolors, s);
}
int chn_dfeature(sgb_ctx* ctx, const ViewState& w, const PoolView& pv, const float* dL_dpix, float* dL_dcolors,
                 cudaStream_t s) {
    return launch_dfeature(ctx, w, pv, dL_dpix, dL_dcolors, s);
}

}  // namespace sgb
