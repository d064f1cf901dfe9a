// Per-tile back-to-front blend backward for the RGB / RGB-D path (C <= 4).  Contract: reference
// backward.cu:394-552.  (Wider rasters: chn_blend.cuh.)
//
// Decomposition: one CTA per tile, thread = pixel, like the forward.  The
// reference keeps accum_rec[C], last_color[C], dL_dpixel[C] per thread (backward.cu:444-451) and
// issues 9 + C global atomics per (pixel, Gaussian) pair (:519, :540-549).  Here
//   * dL/dalpha is linear in dL_dpixel, so each channel chunk contributes an independent partial
//     through two scalars per pixel: s = <feature_chunk, dL_dpixel_chunk> and the running
//     A = <accum_rec_chunk, dL_dpixel_chunk>, with A' = last_alpha * s_last + (1 - last_alpha) * A
//     (the dot-product form of :511-516); the geometry gradients are linear in dL/dalpha, so the
//     chunk partials simply add up in the per-Gaussian accumulators;
//   * the transmittance chain T <- T / (1 - alpha) walks back from final_T exactly like :498;
//   * per-pair atomics become: warp shuffle reductions -> warp-private shared-memory partials ->
//     one block-level sum per staged Gaussian -> one red.global.add per (Gaussian, tile, channel).
// With EXP_ALPHA the expected depth E and accumulated opacity A of blend_fwd.cu are two more channels with features
// z_i and 1 over background 0: their upstream gradients join s and A (bgdot is unchanged), and
// dL/dz_i = sum_p alpha_i T_i dL/dE_p is reduced like a seventh geometry partial into dL_ddepth [P], which the
// geometry backward carries into dL/dmeans3D.
#include <cstdlib>
#include "common.cuh"

namespace sgb {

namespace {

constexpr int kThreads = SGB_TILE_PIX;
constexpr int kWarps = kThreads / 32;
constexpr int kBatchB = 32;  // Gaussians per stage (one bit each in the per-warp activity mask)
constexpr int CH = 4;        // channels per CTA: all of them (C <= 4)

struct __align__(16) BwdSmem {
    float4 recA[2][kBatchB];
    float4 recB[2][kBatchB];
    uint32_t ids[2][kBatchB];
    float feat[2][kBatchB][CH];
    float dF[kWarps][kBatchB][CH];  // warp-private partial dL/dfeature of the current batch
    float geo[kWarps][kBatchB][8];  // warp-private partial geometry gradients (6 used)
    uint32_t active[kWarps];        // bit j: warp wrote slot j of its dF/geo slice this batch
};

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o >= 1; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

template <bool EXP_ALPHA>
__global__ void __launch_bounds__(kThreads) blend_backward_kernel(
    const uint2* __restrict__ ranges, const uint32_t* __restrict__ point_list, int W, int H, int C,
    const float* __restrict__ bg_color, const SplatRec* __restrict__ rec, const float* __restrict__ colors,
    const float* __restrict__ final_Ts, const uint32_t* __restrict__ n_contrib,
    const uint32_t* __restrict__ tile_last, const float* __restrict__ dL_dpixels, float* __restrict__ dL_dmean2D,
    float* __restrict__ dL_dconic2D, float* __restrict__ dL_dopacity, float* __restrict__ dL_dcolors,
    const float* __restrict__ dL_dexp_depth, const float* __restrict__ dL_dalpha, float* __restrict__ dL_ddepth) {
    constexpr int kGeo = EXP_ALPHA ? 7 : 6;  // geometry partials per Gaussian: means2D xy, conic 3, opacity[, z]
    extern __shared__ __align__(128) unsigned char smem_raw[];
    BwdSmem& sm = *reinterpret_cast<BwdSmem*>(smem_raw);

    const int tiles_x = (W + SGB_TILE - 1) / SGB_TILE;
    const int tile = blockIdx.x;
    const int ch0 = blockIdx.y * CH;
    const int nch = min(CH, C - ch0);
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const uint32_t tx = tid & (SGB_TILE - 1), ty = tid >> 4;
    const uint2 pix = {(uint32_t)(tile % tiles_x) * SGB_TILE + tx, (uint32_t)(tile / tiles_x) * SGB_TILE + ty};
    const uint32_t pix_id = W * pix.y + pix.x;
    const float2 pixf = {(float)pix.x, (float)pix.y};
    const bool inside = pix.x < (uint32_t)W && pix.y < (uint32_t)H;
    const uint2 range = ranges[tile];
    // Entries at list position >= n_contrib never contribute (backward.cu:481-483); the tile only
    // needs its first tile_last entries.
    const int total = (int)min(tile_last[tile], range.y - range.x);
    const int nbatches = (total + kBatchB - 1) / kBatchB;
    if (nbatches == 0) return;

    // Unused tail of the last (partial) chunk must read as zero: it is multiplied into sums.
    if (nch < CH)
        for (int e = tid; e < 2 * kBatchB * CH; e += kThreads) {
            const int k = e % CH;
            if (k >= nch) (&sm.feat[0][0][0])[e] = 0.f;
        }
    __syncthreads();

    // Batch b covers list positions [hi - cnt, hi) with hi = total - b*kBatchB; slot j <-> position hi-1-j.
    auto issue = [&](int b) {
        const int st = b & 1;
        const int hi = total - b * kBatchB;
        const int cnt = min(kBatchB, hi);
        if (tid < cnt) {
            const uint32_t id = point_list[range.x + hi - 1 - tid];
            sm.ids[st][tid] = id;
            const float4* rp = reinterpret_cast<const float4*>(rec + id);
            sm.recA[st][tid] = __ldg(rp);
            sm.recB[st][tid] = __ldg(rp + 1);
        }
        for (int e = tid; e < cnt * nch; e += kThreads) {
            const int j = e / nch, k = e - j * nch;
            const uint32_t id = point_list[range.x + hi - 1 - j];
            sm.feat[st][j][k] = __ldg(colors + (size_t)id * C + ch0 + k);
        }
    };

    // Per-pixel state.
    float dL[CH];
    float bgdot = 0.f;
    const size_t plane = (size_t)H * W;
#pragma unroll
    for (int k = 0; k < CH; k++) {
        dL[k] = (inside && k < nch) ? __ldg(dL_dpixels + (size_t)(ch0 + k) * plane + pix_id) : 0.f;
        if (k < nch) bgdot += bg_color[ch0 + k] * dL[k];  // backward.cu:527-529, chunk partial
    }
    // dL/dE and dL/dA of this pixel (an absent plane has zero gradient)
    const float dLE = (EXP_ALPHA && inside && dL_dexp_depth) ? __ldg(dL_dexp_depth + pix_id) : 0.f;
    const float dLA = (EXP_ALPHA && inside && dL_dalpha) ? __ldg(dL_dalpha + pix_id) : 0.f;
    const float T_final = inside ? final_Ts[pix_id] : 0.f;
    float T = T_final;
    const int last_contributor = inside ? (int)n_contrib[pix_id] : 0;
    float last_alpha = 0.f, s_last = 0.f, A = 0.f;
    const float ddelx_dx = 0.5f * W, ddely_dy = 0.5f * H;  // backward.cu:455-456

    issue(0);
    for (int b = 0; b < nbatches; b++) {
        const int st = b & 1;
        const int hi = total - b * kBatchB;
        const int cnt = min(kBatchB, hi);
        __syncthreads();  // batch b-1 fully consumed and flushed: stage (b+1)&1 and dF/geo are free
        if (b + 1 < nbatches) issue(b + 1);
        __syncthreads();  // batch b staged by every thread
        uint32_t my_active = 0;

        for (int j = 0; j < cnt; j++) {
            const int pos = hi - 1 - j;  // 0-based list position of this Gaussian
            const float4 a = sm.recA[st][j];
            const float4 con_o = sm.recB[st][j];
            const float2 d = {a.x - pixf.x, a.y - pixf.y};
            const float power = -0.5f * (con_o.x * d.x * d.x + con_o.z * d.y * d.y) - con_o.y * d.x * d.y;
            const float G = exp(power);
            const float alpha = min(0.99f, con_o.w * G);
            const bool contributes = (pos < last_contributor) && !(power > 0.0f) && !(alpha < 1.0f / 255.0f);
            if (!__any_sync(0xffffffffu, contributes)) continue;

            float w = 0.f, g0 = 0.f, g1 = 0.f, g2 = 0.f, g3 = 0.f, g4 = 0.f, g5 = 0.f, g6 = 0.f;
            if (contributes) {
                T = T / (1.f - alpha);  // backward.cu:498
                w = alpha * T;          // dchannel_dcolor, :499
                float s = 0.f;
#pragma unroll
                for (int k = 0; k < CH; k++) s += sm.feat[st][j][k] * dL[k];
                if (EXP_ALPHA) {
                    s += a.z * dLE;
                    s += 1.0f * dLA;
                    g6 = w * dLE;
                }
                A = last_alpha * s_last + (1.f - last_alpha) * A;  // :511 in dot-product form
                s_last = s;
                float dL_dalpha = (s - A) * T;                           // :515, :521
                last_alpha = alpha;                                      // :523
                dL_dalpha += (-T_final / (1.f - alpha)) * bgdot;         // :530
                const float dL_dG = con_o.w * dL_dalpha;                 // :533-537
                const float gdx = G * d.x, gdy = G * d.y;
                const float dG_ddelx = -gdx * con_o.x - gdy * con_o.y;
                const float dG_ddely = -gdy * con_o.z - gdx * con_o.y;
                g0 = dL_dG * dG_ddelx * ddelx_dx;  // :540-549
                g1 = dL_dG * dG_ddely * ddely_dy;
                g2 = -0.5f * gdx * d.x * dL_dG;
                g3 = -0.5f * gdx * d.y * dL_dG;
                g4 = -0.5f * gdy * d.y * dL_dG;
                g5 = G * dL_dalpha;
            }
            g0 = warp_sum(g0); g1 = warp_sum(g1); g2 = warp_sum(g2);
            g3 = warp_sum(g3); g4 = warp_sum(g4); g5 = warp_sum(g5);
            if (lane == 0) {
                float* gp = sm.geo[warp][j];
                *reinterpret_cast<float4*>(gp) = make_float4(g0, g1, g2, g3);
                *reinterpret_cast<float2*>(gp + 4) = make_float2(g4, g5);
            }
            if (EXP_ALPHA) {
                g6 = warp_sum(g6);
                if (lane == 0) sm.geo[warp][j][6] = g6;
            }
#pragma unroll
            for (int k = 0; k < CH; k++) {
                const float t = warp_sum(w * dL[k]);  // :519
                if (lane == 0) sm.dF[warp][j][k] = t;
            }
            my_active |= 1u << j;
        }
        if (lane == 0) sm.active[warp] = my_active;
        __syncthreads();

        // Flush: one sum over the warps and one global reduction per (Gaussian, channel).
        for (int e = tid; e < cnt * CH; e += kThreads) {
            const int j = e / CH, k = e - j * CH;
            if (k >= nch) continue;
            float t = 0.f;
            bool any = false;
#pragma unroll
            for (int wv = 0; wv < kWarps; wv++)
                if (sm.active[wv] >> j & 1u) { t += sm.dF[wv][j][k]; any = true; }
            if (any) red_add_f32(dL_dcolors + (size_t)sm.ids[st][j] * C + ch0 + k, t);
        }
        for (int e = tid; e < cnt * kGeo; e += kThreads) {
            const int j = e / kGeo, q = e - j * kGeo;
            float t = 0.f;
            bool any = false;
#pragma unroll
            for (int wv = 0; wv < kWarps; wv++)
                if (sm.active[wv] >> j & 1u) { t += sm.geo[wv][j][q]; any = true; }
            if (any) {
                const size_t id = sm.ids[st][j];
                float* dst = q < 2 ? dL_dmean2D + id * 3 + q                        // float3 .x .y
                           : q < 5 ? dL_dconic2D + id * 4 + (q == 4 ? 3 : q - 2)    // float4 .x .y .w
                           : q == 5 ? dL_dopacity + id
                                    : dL_ddepth + id;
                red_add_f32(dst, t);
            }
        }
    }
}

}  // namespace

int launch_blend_backward(const sgb_view_inputs& in, GeomView g, BinView b, ImgView im, const float* colors,
                          const float* dL_dpix, float* dL_dmean2D, float* dL_dconic, float* dL_dopacity,
                          float* dL_dcolors, const float* dL_dexp_depth, const float* dL_dalpha, float* dL_ddepth,
                          cudaStream_t s) {
    if (in.C > 4) {  // wider rasters: chn_blend.cuh
        set_error("launch_blend_backward handles C <= 4 only");
        return SGB_E_INVALID;
    }
    const int tiles = ((in.W + SGB_TILE - 1) / SGB_TILE) * ((in.H + SGB_TILE - 1) / SGB_TILE);
    const int chunks = (in.C + CH - 1) / CH;
    const size_t smem = sizeof(BwdSmem);
    const bool exp_alpha = dL_ddepth != nullptr;
    auto kern = exp_alpha ? blend_backward_kernel<true> : blend_backward_kernel<false>;
    static DeviceOnce attr_set[2];
    if (attr_set[exp_alpha].first_use_on_device()) {
        SGB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    }
    kern<<<dim3(tiles, chunks), kThreads, smem, s>>>(
        im.ranges, b.point_list, in.W, in.H, in.C, in.background, g.rec, colors, im.final_T, im.n_contrib,
        im.tile_last, dL_dpix, dL_dmean2D, dL_dconic, dL_dopacity, dL_dcolors, dL_dexp_depth, dL_dalpha, dL_ddepth);
    SGB_LAUNCH_CHECK("blend_backward_kernel", in.debug, s);
    return SGB_OK;
}

}  // namespace sgb
