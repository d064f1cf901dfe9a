// dL/dfeature contraction of the C-channel blend (chn_blend.cuh); also the numerator of a lift (sgb_lift_batch).
#include <cstddef>
#include <cstring>
#include "chn_blend.cuh"
#include "persistent.cuh"

namespace sgb {

namespace {

// dF[entry][ch] = sum over the tile's 256 pixels of w[entry][px] * dL/dout[px][ch]   (K = pixels).
// Persistent: the grid fills the GPU once and every CTA claims work items (tile, up to 256 channels; at C = 256 an item
// is a tile, so each weight row is staged once; a wider C splits into items of equal width, a multiple of 16, with the
// channel part varying fastest) from a counter until none are left; an empty tile costs one claim.  Three warp groups:
//   * WG0 is the producer.  It gives up registers (setmaxnreg) and one warp streams both operands of a pass (up to
//     128 entries) through a ring of kDfStages stages, one 32-pixel K slab per stage:
//       - the weight slab [128 entries][32 px], one 3-D TMA box [16 rows][32 px] per 16-entry pool chunk;
//       - the dL slab [2 tile rows][item channels][16 px], ONE 3-D TMA box.  A tile with more than 128 entries
//         re-streams its dL slabs once per pass.  Layouts TMA cannot take (a row pitch or base that is not a multiple
//         of 16 bytes: W % 4 != 0 in fp32, W % 8 != 0 in fp16) are staged by the producer warp into the same
//         (swizzled) layout on the same mbarrier, with 4-byte cp.async (fp32) or plain loads (fp16).
//   * WG1 and WG2 compute (8 warps) and take the registers WG0 gave up.  Warp w owns channels 32w..32w+31 of the item
//     and ALL entries of the pass.  Lane (eg = lane >> 1, h = lane & 1) accumulates entries {eg + 16j, j < R} x
//     channels 32w + 4h + 8g + {0..3}, g < 4, in 128 scalar registers, R = ceil(entries / 16) <= 8: per 4-pixel K step
//     64R FMAs for R + 16 LDS.128 (512 per 24 at R = 8).  (16 warps of 16 channels, 64 accumulators each, would leave
//     a compute thread at most 120 registers, and ptxas spills the slab loop at that limit.)
// Each accumulator adds the pixels of the tile in order 0..255, and each (Gaussian, tile, 4 channels) is one 16-byte
// reduction.  The TMA swizzles keep every operand load at 2 shared-memory wavefronts or less, 1 for dL (see
// lane_group8):
//   * weights, SWIZZLE_128B: quad q of the 128-byte row e sits at q ^ (e & 7); each 4-lane group reads 2 rows and each
//     half-warp 8 consecutive rows -> 8 distinct bank groups;
//   * dL, SWIZZLE_64B over a [row][ch][16 px] box: quad p of channel c sits at p ^ ((c >> 1) & 3), so channels c and
//     c + 4 (the two h halves of a load) land in different banks.
constexpr int kDfCH = 256;                  // widest work item (channels)
constexpr int kDfStages = 4;                // ring depth
constexpr int kDfPass = 128;                // entries per pass (8 pool chunks)
constexpr int kDfSlabPix = 32;              // pixels (2 tile rows) per K slab
constexpr int kDfSlabs = SGB_TILE_PIX / kDfSlabPix;
constexpr int kDfComputeWarps = kDfCH / 32;                // 2 warp groups, 32 channels per warp
constexpr int kDfThreads = 128 + 32 * kDfComputeWarps;  // producer warp group + 2 compute warp groups
constexpr uint32_t kDfProducerRegs = 56, kDfComputeRegs = 224;
static_assert(warp_group_regs_fit(kDfProducerRegs, kDfComputeWarps, kDfComputeRegs),
              "dL/dfeature: the warp groups' register limits exceed the register file");

struct DfHdr {  // one ring stage's description, written by the producer before the stage is armed
    int end;            // no more work
    int cnt;            // entries of the pass
    int slab;           // pixels 32 slab .. 32 slab + 31
    int ch0, nch;       // channels of the item
    uint32_t gid[kDfPass];  // Gaussian ids of the pass (written for the last slab of a pass)
};
// T: element type of dL/dout as it sits in global memory (float, or __half for an fp16 feature map that is lifted
// onto the Gaussians); the dL slab keeps it in shared memory and is widened to fp32 in the compute warps' loads.
template <typename T>
struct DfSmem {  // at a 1024-byte aligned offset of the dynamic shared memory (TMA swizzle atoms)
    float w[kDfStages][kDfPass * kDfSlabPix];
    T dl[kDfStages][kDfSlabPix * kDfCH];
    MbarRing<kDfStages, DfHdr> ring;
};
template <typename T>
constexpr size_t kDfSmemBytes = sizeof(DfSmem<T>) + 1024;
static_assert(kDfSmemBytes<float> <= 227 * 1024, "dL/dfeature shared memory exceeds the sm_90 opt-in limit");

// Pixels 4 (q & 3) .. 4 (q & 3) + 3 of slab row q >> 2, channel cl + k, of a stage's dL slab; dl points at channel cl
// (a multiple of 4) of row 0, rs is the row pitch in elements (16 x the item's channels) and swz = df_swz<T>(cl).  The
// slab is the TMA box under its swizzle, 16 px per channel row:
//   fp32, 64 B rows, SWIZZLE_64B: 4-px quad p of channel c sits at p ^ ((c >> 1) & 3);
//   fp16, 32 B rows, SWIZZLE_32B: 8-px half h of channel c sits at h ^ ((c >> 2) & 1).
// Either way channels c and c + 4, the two halves of a warp's load, land in different banks, and channel c + 8 has the
// swizzle of channel c.
template <typename T>
__device__ __forceinline__ int df_swz(int cl) { return sizeof(T) == 4 ? (cl >> 1) & 3 : (cl >> 2) & 1; }
__device__ __forceinline__ float4 df_dl4(const float* dl, int q, int k, int swz, int rs) {
    return *reinterpret_cast<const float4*>(dl + (q >> 2) * rs + k * 16 + (((q & 3) ^ swz ^ (k >> 1)) << 2));
}
__device__ __forceinline__ float4 df_dl4(const __half* dl, int q, int k, int swz, int rs) {
    const uint2 r = *reinterpret_cast<const uint2*>(dl + (q >> 2) * rs + k * 16 + ((((q & 3) >> 1) ^ swz) << 3) +
                                                    ((q & 1) << 2));
    const float2 a = __half22float2(*reinterpret_cast<const __half2*>(&r.x));
    const float2 b = __half22float2(*reinterpret_cast<const __half2*>(&r.y));
    return make_float4(a.x, a.y, b.x, b.y);
}

// One 32-pixel slab of a pass: acc[j][4g + k] += sum over the slab of w[eg + 16j][px] * dL[px][cl + 8g + k], g < 4.
// dl points at channel cl of the stage's dL slab, ws at its weight rows; swz = df_swz<T>(cl), rs the dL row pitch.
template <int R, typename T>
__device__ __forceinline__ void df_slab(float (&acc)[8][16], const float* __restrict__ ws, const T* __restrict__ dl,
                                        int rs, int eg, int swz) {
#pragma unroll 1
    for (int q = 0; q < kDfSlabPix / 4; q++) {
        float4 d[16];
#pragma unroll
        for (int k = 0; k < 16; k++) d[k] = df_dl4(dl + (k >> 2) * (8 * 16), q, k & 3, swz, rs);
#pragma unroll
        for (int j = 0; j < R; j++) {
            const float4 wv = *reinterpret_cast<const float4*>(ws + (eg + 16 * j) * 32 + ((q ^ (eg & 7)) << 2));
#pragma unroll
            for (int k = 0; k < 16; k++) {
                acc[j][k] = fmaf(wv.x, d[k].x, acc[j][k]);
                acc[j][k] = fmaf(wv.y, d[k].y, acc[j][k]);
                acc[j][k] = fmaf(wv.z, d[k].z, acc[j][k]);
                acc[j][k] = fmaf(wv.w, d[k].w, acc[j][k]);
            }
        }
    }
}

// CW: channels per work item (a multiple of 16, at most kDfCH); the TMA dL box is [16 px][CW][2 rows].
template <typename T>
__global__ void __launch_bounds__(kDfThreads, 1) dfeature_persistent_kernel(
    int W, int H, int C, int CW, const T* __restrict__ dL_dpixels, PoolView pool, float* __restrict__ dL_dcolors,
    int* __restrict__ work_counter, const __grid_constant__ CUtensorMap dl_map,
    const __grid_constant__ CUtensorMap w_map, const int use_tma) {
    extern __shared__ __align__(128) unsigned char smem_raw[];
    DfSmem<T>& sm = *reinterpret_cast<DfSmem<T>*>(smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u));
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if (tid == 0) sm.ring.init(!use_tma, kDfComputeWarps);
    __syncthreads();

    if (warp >= 4) {
        setmaxnreg_inc<kDfComputeRegs>();
        const int cw = warp - 4;
        const int eg = lane >> 1;
        const int cl = cw * 32 + (lane & 1) * 4;  // channel (within the item) of k = 0; k = 4g..4g+3 are cl + 8g + {0..3}
        const int rs = CW * 16;
        const int swz = df_swz<T>(cl);
        const bool red16 = ((C & 3) == 0) && ((reinterpret_cast<uintptr_t>(dL_dcolors) & 15) == 0);
        float acc[8][16];
        for (uint32_t step = 0;; step++) {
            const int st = sm.ring.wait(step);
            const DfHdr& h = sm.ring.hdr[st];
            if (h.end) break;
            const int slab = h.slab, cnt = h.cnt, nch = h.nch;
            const int R = (cnt + 15) >> 4;
            if (slab == 0) {
#pragma unroll
                for (int j = 0; j < 8; j++)
#pragma unroll
                    for (int k = 0; k < 16; k++) acc[j][k] = 0.f;
            }
            if (cw * 32 < nch) {
                const float* ws = sm.w[st];
                const T* dl = sm.dl[st] + cl * 16;
                switch (R) {
                    case 1: df_slab<1, T>(acc, ws, dl, rs, eg, swz); break;
                    case 2: df_slab<2, T>(acc, ws, dl, rs, eg, swz); break;
                    case 3: df_slab<3, T>(acc, ws, dl, rs, eg, swz); break;
                    case 4: df_slab<4, T>(acc, ws, dl, rs, eg, swz); break;
                    case 5: df_slab<5, T>(acc, ws, dl, rs, eg, swz); break;
                    case 6: df_slab<6, T>(acc, ws, dl, rs, eg, swz); break;
                    case 7: df_slab<7, T>(acc, ws, dl, rs, eg, swz); break;
                    default: df_slab<8, T>(acc, ws, dl, rs, eg, swz); break;
                }
                if (slab == kDfSlabs - 1) {
                    const int ch0 = h.ch0;
#pragma unroll
                    for (int j = 0; j < 8; j++) {
                        const int e = eg + 16 * j;
                        if (j >= R || e >= cnt) continue;
                        float* dst = dL_dcolors + (size_t)h.gid[e] * C + ch0 + cl;
#pragma unroll
                        for (int g = 0; g < 4; g++) {
                            const int c = cl + 8 * g;
                            if (red16 && c + 4 <= nch) {
                                red_add_v4_f32(dst + 8 * g, make_float4(acc[j][4 * g], acc[j][4 * g + 1],
                                                                        acc[j][4 * g + 2], acc[j][4 * g + 3]));
                            } else {
#pragma unroll
                                for (int k = 0; k < 4; k++)
                                    if (c + k < nch) red_add_f32(dst + 8 * g + k, acc[j][4 * g + k]);
                            }
                        }
                    }
                }
            }
            sm.ring.release(st, lane);
        }
        return;
    }

    // ---- producer warp group: warp 0 streams, warps 1-3 only hand their registers back
    setmaxnreg_dec<kDfProducerRegs>();
    if (warp != 0) return;
    const int tiles_x = (W + SGB_TILE - 1) / SGB_TILE;
    const int tiles = tiles_x * ((H + SGB_TILE - 1) / SGB_TILE);
    const int nitems = (C + CW - 1) / CW;
    const int total = tiles * nitems;
    const size_t plane = (size_t)H * W;
    const uint32_t dl_bytes = use_tma ? (uint32_t)(kDfSlabPix * CW * sizeof(T)) : 0u;
    uint32_t step = 0;  // ring stages armed so far
    for (;;) {
        const int k = claim_item(work_counter, lane);
        if (k >= total) break;
        const int tile = k / nitems, ch0 = (k % nitems) * CW;
        const uint32_t n = pool.count[tile];
        if (n == 0) continue;
        const uint32_t dbase = pool.dirbase[tile];
        const int nch = min(CW, C - ch0);
        const int x0 = (tile % tiles_x) * SGB_TILE, y0 = (tile / tiles_x) * SGB_TILE;
        for (uint32_t base = 0; base < n; base += kDfPass) {
            const int cnt = (int)min((uint32_t)kDfPass, n - base);
            const int nck = (cnt + kChunkEntries - 1) / kChunkEntries;
            const uint32_t cid = lane < nck ? chunk_of(pool, dbase, (int)(base / kChunkEntries) + lane) : 0u;
            uint32_t gid[kDfPass / 32];
#pragma unroll
            for (int i = 0; i < kDfPass / 32; i++) {
                const int e = lane + 32 * i;
                const uint32_t c = __shfl_sync(0xffffffffu, cid, e / kChunkEntries);
                gid[i] = e < cnt ? pool.chunks[c].meta[e & (kChunkEntries - 1)].x : 0u;
            }
            for (int s = 0; s < kDfSlabs; s++) {
                const int st = sm.ring.acquire(step);
                DfHdr& h = sm.ring.hdr[st];
                if (lane == 0) {
                    h.end = 0;
                    h.cnt = cnt;
                    h.slab = s;
                    h.ch0 = ch0;
                    h.nch = nch;
                }
                if (s == kDfSlabs - 1) {
#pragma unroll
                    for (int i = 0; i < kDfPass / 32; i++) h.gid[lane + 32 * i] = gid[i];
                }
                if (lane < nck)
                    tma_tile3d_g2s(&sm.w[st][lane * kChunkEntries * 32], &w_map, 32 * s, 0, (int)cid, &sm.ring.full[st]);
                const int ys = y0 + 2 * s;  // first tile row of the slab
                T* dst = sm.dl[st];
                if (use_tma) {
                    if (lane == 0) tma_tile3d_g2s(dst, &dl_map, x0, ch0, ys, &sm.ring.full[st]);
                } else if constexpr (sizeof(T) == 2) {
                    // cp.async has no 2-byte size: plain loads into the TMA layout, then one release-arrive per lane
#pragma unroll 1
                    for (int idx = lane; idx < 2 * 16 * CW; idx += 32) {
                        const int x = idx & 15, r = (idx >> 4) >= CW, c = (idx >> 4) - r * CW;
                        const int gx = x0 + x, gy = ys + r;
                        const bool ok = c < nch && gx < W && gy < H;
                        dst[r * CW * 16 + c * 16 + ((((x >> 3) ^ ((c >> 2) & 1)) << 3) | (x & 7))] =
                            ok ? dL_dpixels[(size_t)(ch0 + c) * plane + (size_t)W * gy + gx] : T(0.f);
                    }
                    mbar_arrive(&sm.ring.full[st]);
                } else {
#pragma unroll 1
                    for (int idx = lane; idx < 2 * 16 * CW; idx += 32) {
                        const int x = idx & 15, r = (idx >> 4) >= CW, c = (idx >> 4) - r * CW;
                        const int gx = x0 + x, gy = ys + r;
                        const bool ok = c < nch && gx < W && gy < H;
                        const float* src = ok ? dL_dpixels + (size_t)(ch0 + c) * plane + (size_t)W * gy + gx : dL_dpixels;
                        cp_async4(dst + r * CW * 16 + c * 16 + ((((x >> 2) ^ ((c >> 1) & 3)) << 2) | (x & 3)), src,
                                  ok ? 4 : 0);
                    }
                    cp_async_mbar_arrive_noinc(&sm.ring.full[st]);
                }
                __syncwarp();
                if (lane == 0)
                    mbar_arrive_expect_tx(&sm.ring.full[st], (uint32_t)nck * (kChunkEntries * 32 * 4) + dl_bytes);
                step++;
            }
        }
    }
    sm.ring.finish(step, !use_tma, lane);
}

}  // namespace

// dL/dout (C, H, W), fp32 or fp16, for dfeature_persistent_kernel<T>, described with its dimensions in the order
// (x, channel, y) so that one [16 px][CW ch][2 rows] box lands as [row][ch][16 px] under the swizzle df_dl4 reads
// (64-byte rows of fp32, 32-byte rows of fp16).  Returns false (the kernel then stages the slabs itself) when the
// layout does not meet the TMA rules (base and row pitch multiples of 16 bytes: W % 4 == 0 in fp32, W % 8 == 0 in fp16)
// or the driver entry point is not available.
template <typename T>
static bool encode_dfeature_dl_map(CUtensorMap* map, const T* dL_dpix, int W, int H, int C, int CW) {
    memset(map, 0, sizeof(*map));
    if (((size_t)W * sizeof(T)) % 16 != 0 || (reinterpret_cast<uintptr_t>(dL_dpix) & 15) != 0) return false;
    const cuuint64_t dims[3] = {(cuuint64_t)W, (cuuint64_t)C, (cuuint64_t)H};
    const cuuint64_t strides[2] = {(cuuint64_t)W * H * sizeof(T), (cuuint64_t)W * sizeof(T)};
    const cuuint32_t box[3] = {SGB_TILE, (cuuint32_t)CW, kDfSlabPix / SGB_TILE};
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
    const cuuint32_t box[3] = {kDfSlabPix, kChunkEntries, 1};
    return encode_tiled_map(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3,
                            reinterpret_cast<char*>(pv.chunks) + offsetof(WChunk, w), dims, strides, box,
                            CU_TENSOR_MAP_SWIZZLE_128B);
}

template <typename T>
static int launch_dfeature(sgb_ctx* ctx, const ViewState& w, const PoolView& pv, const T* dL_dpix, float* dL_dcolors,
                           cudaStream_t s) {
    const sgb_view_inputs& in = w.in;
    const ItemSplit sp = split_channels(in.C, kDfCH);  // one item at C <= 256, two at C = 512
    const int CW = sp.CW;
    const int items = num_tiles(in) * sp.nitems;
    if (items == 0) return SGB_OK;
    CUtensorMap dl_map, w_map;
    const int use_tma = encode_dfeature_dl_map(&dl_map, dL_dpix, in.W, in.H, in.C, CW) ? 1 : 0;
    if (!encode_dfeature_w_map(&w_map, pv)) {
        set_error("dL/dfeature: cuTensorMapEncodeTiled is unavailable or rejected the weight pool");
        return SGB_E_CUDA;
    }
    StageTimer t(ctx, ST_DFEATURE, s);
    int grid = 0;
    const int rc = persistent_grid<dfeature_persistent_kernel<T>>(ctx, kDfThreads, kDfSmemBytes<T>, items, s, &grid);
    if (rc) return rc;
    ctx->launches += 1;
    dfeature_persistent_kernel<T><<<grid, kDfThreads, kDfSmemBytes<T>, s>>>(
        in.W, in.H, in.C, CW, dL_dpix, pv, dL_dcolors, static_cast<int*>(ctx->work.p), dl_map, w_map, use_tma);
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
