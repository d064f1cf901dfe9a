// Chain backward of the C-channel blend (chn_blend.cuh): dL/dmean2D, dL/dconic, dL/dopacity.
#include <cstring>
#include "chn_blend.cuh"
#include "tma.cuh"

namespace sgb {

namespace {

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
__global__ void __launch_bounds__(kTileThreads, 2) chain_backward_warp_kernel(
    int W, int H, int C, const float* __restrict__ bg_color, const SplatRec* __restrict__ rec,
    const float* __restrict__ features, const float* __restrict__ final_Ts, const float* __restrict__ dL_dpixels,
    PoolView pool, float* __restrict__ dL_dmean2D, float* __restrict__ dL_dconic2D, float* __restrict__ dL_dopacity,
    const __grid_constant__ CUtensorMap dl_map, const int use_tma) {
    constexpr int CK = 16;
    extern __shared__ __align__(128) unsigned char smem_raw[];
    __shared__ uint2 MetaS[kMetaCap];
    __shared__ uint64_t dbar[kTileThreads / 32][2];  // per warp, per dL slab buffer: TMA completion
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
    for (uint32_t k = tid; k * kChunkEntries < ncache; k += kTileThreads) Cdir[k] = chunk_of(pool, dbase, (int)k);
    if (lane == 0) {
        mbar_init(&dbar[warp][0], 1);
        mbar_init(&dbar[warp][1], 1);
        mbar_fence_init();
    }
    int bg_nonzero = 0;
    for (int ch = tid; ch < C; ch += kTileThreads) bg_nonzero |= (bg_color[ch] != 0.f);
    bg_nonzero = __syncthreads_or(bg_nonzero);   // also orders the Cdir stores and the barrier inits
    for (uint32_t e = tid; e < ncache; e += kTileThreads)
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

}  // namespace

// Tensor map of dL/dout (C, H, W) fp32 with a [16 ch][2 rows][16 px] box for the chain kernel's slab loads.  Returns
// false (the kernel then loads the slabs with plain loads) when the layout does not meet the TMA rules (base and row
// pitch multiples of 16 bytes) or the driver entry point is not available.
static bool encode_dl_map(CUtensorMap* map, const float* dL_dpix, int W, int H, int C) {
    memset(map, 0, sizeof(*map));
    if ((W & 3) != 0 || (reinterpret_cast<uintptr_t>(dL_dpix) & 15) != 0) return false;
    const cuuint64_t dims[3] = {(cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)C};
    const cuuint64_t strides[2] = {(cuuint64_t)W * sizeof(float), (cuuint64_t)W * H * sizeof(float)};
    const cuuint32_t box[3] = {SGB_TILE, 2, 16};
    return encode_tiled_map(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, dL_dpix, dims, strides, box,
                            CU_TENSOR_MAP_SWIZZLE_NONE);
}

int chn_chain(sgb_ctx* ctx, const ViewState& w, const PoolView& pv, const float* dL_dpix, float* dL_dmean2D,
              float* dL_dconic, float* dL_dopacity, cudaStream_t s) {
    const sgb_view_inputs& in = w.in;
    const int tiles = num_tiles(in);
    const bool vec = (in.C % 4 == 0) && ((reinterpret_cast<uintptr_t>(w.colors) & 15) == 0);
    const size_t smem = sizeof(ChainWarpSmem) * (kTileThreads / 32);
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
    kern<<<tiles, kTileThreads, smem, s>>>(in.W, in.H, in.C, in.background, w.g.rec, w.colors, w.im.final_T, dL_dpix,
                                           pv, dL_dmean2D, dL_dconic, dL_dopacity, dl_map, use_tma);
    SGB_LAUNCH_CHECK("chain backward kernel", in.debug, s);
    return SGB_OK;
}

}  // namespace sgb
