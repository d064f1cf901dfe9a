// Per-tile front-to-back alpha compositing (forward) for the RGB / RGB-D path (C <= 4).
// Contract: reference forward.cu:262-375 and rgbd/cuda_rasterizer/forward.cu:261-393 (median depth).
//
// One CTA per 16x16 tile, thread = pixel, Gaussians staged in shared memory per batch like the
// reference.  The per-pixel alpha / transmittance chain and the accumulation `C[ch] += f*alpha*T`
// are the reference's statement sequence verbatim, so pixels, depth, final_T and n_contrib are
// bit-identical.  Wider rasters go through the weights-once pipeline (chn_blend.cuh).
//
// With EXP_ALPHA the walk also accumulates, with the colour channels' own statement, the expected depth
// E = sum_i z_i alpha_i T_i and the accumulated opacity A = sum_i alpha_i T_i (no background term): E and A are
// bit for bit what the same walk gives for a feature [z, 1] over background 0.
#include <cstdlib>
#include "common.cuh"

namespace sgb {

namespace {

constexpr int kThreads = SGB_TILE_PIX;  // 256, one per pixel
constexpr int kBatch = 64;              // Gaussians per pipeline stage
constexpr int CH = 4;                   // channels per CTA: all of them (C <= 4)

struct __align__(16) FwdStage {
    float4 recA[kBatch];     // mx, my, depth, pad
    float4 recB[kBatch];     // conic.x, conic.y, conic.z, opacity
    float feat[kBatch][CH];  // feature slice [ch0, ch0+CH) of each staged Gaussian
};

template <bool DEPTH, bool EXP_ALPHA>
__global__ void __launch_bounds__(kThreads) blend_forward_kernel(
    const uint2* __restrict__ ranges, const uint32_t* __restrict__ point_list, int W, int H, int C,
    const SplatRec* __restrict__ rec, const float* __restrict__ features, const float* __restrict__ bg_color,
    float* __restrict__ final_T, uint32_t* __restrict__ n_contrib, uint32_t* __restrict__ tile_last,
    float* __restrict__ out_color, float* __restrict__ out_depth, float* __restrict__ out_exp_depth,
    float* __restrict__ out_alpha) {
    extern __shared__ __align__(128) unsigned char smem_raw[];
    FwdStage* stage = reinterpret_cast<FwdStage*>(smem_raw);
    __shared__ uint32_t s_last;

    const int tiles_x = (W + SGB_TILE - 1) / SGB_TILE;
    const int tile = blockIdx.x;
    const int ch0 = blockIdx.y * CH;
    const int nch = min(CH, C - ch0);
    const int tid = threadIdx.x;
    const uint32_t tx = tid & (SGB_TILE - 1), ty = tid >> 4;
    const uint2 pix_min = {(uint32_t)(tile % tiles_x) * SGB_TILE, (uint32_t)(tile / tiles_x) * SGB_TILE};
    const uint2 pix = {pix_min.x + tx, pix_min.y + ty};
    const uint32_t pix_id = W * pix.y + pix.x;
    const float2 pixf = {(float)pix.x, (float)pix.y};
    const bool inside = pix.x < (uint32_t)W && pix.y < (uint32_t)H;
    bool done = !inside;

    const uint2 range = ranges[tile];
    const int total = (int)(range.y - range.x);
    const int nbatches = (total + kBatch - 1) / kBatch;

    if (tid == 0) s_last = 0;
    __syncthreads();

    auto issue = [&](int b) {
        FwdStage& st = stage[b & 1];
        const int base = b * kBatch;
        const int cnt = min(kBatch, total - base);
        if (tid < cnt) {
            const uint32_t id = point_list[range.x + base + tid];
            const float4* rp = reinterpret_cast<const float4*>(rec + id);
            st.recA[tid] = __ldg(rp);
            st.recB[tid] = __ldg(rp + 1);
        }
        for (int e = tid; e < cnt * nch; e += kThreads) {
            const int j = e / nch, k = e - j * nch;
            const uint32_t id = point_list[range.x + base + j];
            st.feat[j][k] = __ldg(features + (size_t)id * C + ch0 + k);
        }
    };

    float T = 1.0f;
    uint32_t contributor = 0;
    uint32_t last_contributor = 0;
    float D = 15.0f;  // rgbd forward.cu:308: default median depth
    float acc[CH];
#pragma unroll
    for (int k = 0; k < CH; k++) acc[k] = 0.f;
    float acc_z = 0.f, acc_w = 0.f;  // E and A

    if (nbatches > 0) issue(0);

    for (int b = 0; b < nbatches; b++) {
        // Block-wide early out (forward.cu:310-312).  Also the WAR fence of the stage that the
        // prefetch below overwrites: every thread has finished reading batch b-1.
        const int num_done = __syncthreads_count(done);
        if (num_done == kThreads) break;
        if (b + 1 < nbatches) issue(b + 1);
        __syncthreads();  // batch b staged by every thread

        const FwdStage& st = stage[b & 1];
        const int cnt = min(kBatch, total - b * kBatch);
        for (int j = 0; !done && j < cnt; j++) {
            contributor++;
            // forward.cu:333-352, verbatim arithmetic
            const float4 a = st.recA[j];
            const float2 xy = {a.x, a.y};
            const float2 d = {xy.x - pixf.x, xy.y - pixf.y};
            const float4 con_o = st.recB[j];
            const float power = -0.5f * (con_o.x * d.x * d.x + con_o.z * d.y * d.y) - con_o.y * d.x * d.y;
            if (power > 0.0f) continue;
            const float alpha = min(0.99f, con_o.w * exp(power));
            if (alpha < 1.0f / 255.0f) continue;
            const float test_T = T * (1 - alpha);
            if (test_T < 0.0001f) {
                done = true;
                continue;
            }
#pragma unroll
            for (int k = 0; k < CH; k++)
                if (k < nch) acc[k] += st.feat[j][k] * alpha * T;  // forward.cu:355-356
            if (DEPTH) {
                if (T > 0.5f && test_T < 0.5) D = a.z;  // rgbd forward.cu:368-372: median depth
            }
            if (EXP_ALPHA) {
                acc_z += a.z * alpha * T;
                acc_w += 1.0f * alpha * T;
            }
            T = test_T;
            last_contributor = contributor;
        }
    }

    if (blockIdx.y == 0) {
        if (inside) {
            final_T[pix_id] = T;
            n_contrib[pix_id] = last_contributor;
            if (DEPTH) out_depth[pix_id] = D;
            if (EXP_ALPHA) {
                out_exp_depth[pix_id] = acc_z;
                out_alpha[pix_id] = acc_w;
            }
            atomicMax(&s_last, last_contributor);
        }
        __syncthreads();
        if (tid == 0) tile_last[tile] = s_last;
    }
    if (inside) {
        const size_t plane = (size_t)H * W;
#pragma unroll
        for (int k = 0; k < CH; k++)
            if (k < nch) out_color[(size_t)(ch0 + k) * plane + pix_id] = acc[k] + T * bg_color[ch0 + k];
    }
}

template <bool DEPTH, bool EXP_ALPHA>
int launch_one(const sgb_view_inputs& in, GeomView g, BinView b, ImgView im, const float* colors,
               float* out_color, float* out_depth, float* out_exp_depth, float* out_alpha, cudaStream_t s) {
    const int tiles = ((in.W + SGB_TILE - 1) / SGB_TILE) * ((in.H + SGB_TILE - 1) / SGB_TILE);
    const int chunks = (in.C + CH - 1) / CH;
    const size_t smem = 2 * sizeof(FwdStage);
    auto kern = blend_forward_kernel<DEPTH, EXP_ALPHA>;
    static DeviceOnce attr_set;
    if (attr_set.first_use_on_device()) {
        SGB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    }
    kern<<<dim3(tiles, chunks), kThreads, smem, s>>>(im.ranges, b.point_list, in.W, in.H, in.C, g.rec, colors,
                                                    in.background, im.final_T, im.n_contrib, im.tile_last,
                                                    out_color, out_depth, out_exp_depth, out_alpha);
    SGB_LAUNCH_CHECK("blend_forward_kernel", in.debug, s);
    return SGB_OK;
}

}  // namespace

int launch_blend_forward(const sgb_view_inputs& in, GeomView g, BinView b, ImgView im, const float* colors,
                         float* out_color, float* out_depth, float* out_exp_depth, float* out_alpha, cudaStream_t s) {
    // RGB / RGB-D path (C <= 4): the reference's accumulation order, bit for bit.  Wider rasters go
    // through the weights-once pipeline (chn_blend.cuh).
    if (in.C > 4) {
        set_error("launch_blend_forward handles C <= 4 only");
        return SGB_E_INVALID;
    }
    if (out_exp_depth) {  // E and A come together (api.cu)
        if (out_depth) return launch_one<true, true>(in, g, b, im, colors, out_color, out_depth, out_exp_depth, out_alpha, s);
        return launch_one<false, true>(in, g, b, im, colors, out_color, nullptr, out_exp_depth, out_alpha, s);
    }
    if (out_depth) return launch_one<true, false>(in, g, b, im, colors, out_color, out_depth, nullptr, nullptr, s);
    return launch_one<false, false>(in, g, b, im, colors, out_color, nullptr, nullptr, nullptr, s);
}

}  // namespace sgb
