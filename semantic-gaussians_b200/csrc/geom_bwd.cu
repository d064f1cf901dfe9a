// Per-Gaussian backward of the geometry stage: one thread per visible Gaussian, one pass over its inputs.  All the
// algebra lives in geom_grad.cuh (matrix-calculus form, shared with the CPU test); this file only moves data.
// Reference semantics matched (1e-4 on every output, tests/test_*_gpu.py): backward.cu:141-271 (screen covariance),
// :341-391 (projected centre, SH colour), :275-336 (scale / rotation).  The reference runs two kernels that both re-read
// the per-Gaussian inputs and accumulate dL/dmean through global memory; here the three contributions to dL/dmean are
// summed in registers and stored once.  With camera gradients the same kernel also sums every Gaussian's camera terms
// per view (fp64 per-CTA partials in ctx scratch, then one fixed-order pass): no float atomics, so identical backward
// passes give bitwise-identical camera gradients.
#include "common.cuh"
#include "geom_grad.cuh"

namespace sgb {

namespace {

// The camera-gradient entries the forward reads: view rows 0-2 (t = W p + t0), proj rows 0, 1, 3 (the projected
// centre's x, y, w) and campos, one reduction slot each; the other 8 entries are written 0.
constexpr int kCamSlots = 27;
__host__ __device__ constexpr int cam_slot_entry(int k) {  // index into view (16) | proj (16) | campos (3)
    return k < 12 ? 4 * (k / 3) + k % 3 : k < 24 ? 16 + 4 * ((k - 12) / 3) + ((k - 12) % 3 == 2 ? 3 : (k - 12) % 3)
                                                 : 32 + (k - 24);
}

// CAM = false: the per-Gaussian gradients only.  CAM = true: the same per-Gaussian outputs (the same statements), and
// each CTA also sums its Gaussians' camera terms (geom_grad.cuh camera_grad) in fp64 - over the warp by shuffles in a
// fixed order, then over the warps in order - and writes one partial per reduction slot to cam_partial[k][blockIdx.x].
// AA: anti-aliasing (geom_grad.cuh).  dL_dopacity holds dL/d(o h), the blend backwards' sum; it is overwritten with
// dL/do = h dL/d(o h), and dL/dr = o dL/d(o h) / (2 h) joins the covariance gradient.  h and its branch are the
// forward's, read from the record (SplatRec::pad).
template <bool CAM, bool AA>
__global__ void __launch_bounds__(256) geom_backward_kernel(
    int P, int D, int M, const float* __restrict__ means, const int* __restrict__ radii,
    const float* __restrict__ shs, const uint8_t* __restrict__ clamped, const float* __restrict__ scales,
    const float* __restrict__ rotations, const float scale_modifier, const float* __restrict__ cov3Ds,
    const float* __restrict__ view_matrix, const float* __restrict__ proj, const float focal_x, const float focal_y,
    const float tan_fovx, const float tan_fovy, const float* __restrict__ campos, const float* __restrict__ dL_dmean2D,
    const float* __restrict__ dL_dconics, float* __restrict__ dL_dmeans, const float* __restrict__ dL_dcolor,
    float* __restrict__ dL_dcov, float* __restrict__ dL_dsh, float* __restrict__ dL_dscale,
    float* __restrict__ dL_drot, const float* __restrict__ dL_ddepth, double* __restrict__ cam_partial,
    const SplatRec* __restrict__ rec, const float* __restrict__ opacities, float* __restrict__ dL_dopacity) {
    __shared__ float cam[35];  // view (16) | proj (16) | campos (3): read by every thread, staged once per CTA
    if (threadIdx.x < 16) {
        cam[threadIdx.x] = view_matrix[threadIdx.x];
        cam[16 + threadIdx.x] = proj[threadIdx.x];
    } else if (threadIdx.x < 19) {
        cam[16 + threadIdx.x] = campos ? campos[threadIdx.x - 16] : 0.f;
    }
    __syncthreads();
    const size_t g = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    float gcam[CAM ? 35 : 1];  // CAM: this Gaussian's camera terms, view (16) | proj (16) | campos (3)
    auto one_gaussian = [&]() {
        const float p[3] = {means[3 * g], means[3 * g + 1], means[3 * g + 2]};
        float cov6[6];
#pragma unroll
        for (int i = 0; i < 6; i++) cov6[i] = cov3Ds[6 * g + i];
        const float g_conic[3] = {dL_dconics[4 * g], dL_dconics[4 * g + 1], dL_dconics[4 * g + 3]};
        const float g_ndc[2] = {dL_dmean2D[3 * g], dL_dmean2D[3 * g + 1]};

        float g_r = 0.f;
        if constexpr (AA) {
            const float hs = rec[g].pad, h = fabsf(hs);
            const float g_op = dL_dopacity[g];
            dL_dopacity[g] = h * g_op;
            if (hs > 0.f) g_r = opacities[g] * g_op / (2.f * h);
        }

        float g_mean[3], g_cov[6];
        geomgrad::ProjectTerms terms;
        geomgrad::project_grad(p, cov6, cam, cam + 16, focal_x, focal_y, tan_fovx, tan_fovy, g_conic, g_ndc, g_mean,
                               g_cov, CAM ? &terms : nullptr, AA ? &g_r : nullptr);
#pragma unroll
        for (int i = 0; i < 6; i++) dL_dcov[6 * g + i] = g_cov[i];

        float g_campos[3];
        if (shs) {  // colours from SH: the colour gradient flows to the coefficients and, through the view direction, to p
            float g_rgb[3];
#pragma unroll
            for (int c = 0; c < 3; c++) g_rgb[c] = clamped[3 * g + c] ? 0.f : dL_dcolor[3 * g + c];
            geomgrad::colour_grad(D, p, cam + 32, shs + g * (size_t)M * 3, g_rgb, dL_dsh + g * (size_t)M * 3, g_mean,
                                  CAM ? g_campos : nullptr);
        }
        float gz = 0.f;
        if (dL_ddepth) {  // view-space z = V[2] x + V[6] y + V[10] z + V[14] (transformPoint4x3), as blended into E
            gz = dL_ddepth[g];
            g_mean[0] += gz * cam[2];
            g_mean[1] += gz * cam[6];
            g_mean[2] += gz * cam[10];
        }
#pragma unroll
        for (int i = 0; i < 3; i++) dL_dmeans[3 * g + i] = g_mean[i];
        if constexpr (CAM) geomgrad::camera_grad(p, terms, gz, shs ? g_campos : nullptr, gcam, gcam + 16, gcam + 32);

        if (scales) {  // covariance built from scale / rotation in the forward: continue through the factorisation
            const float q[4] = {rotations[4 * g], rotations[4 * g + 1], rotations[4 * g + 2], rotations[4 * g + 3]};
            const float s[3] = {scale_modifier * scales[3 * g], scale_modifier * scales[3 * g + 1],
                                scale_modifier * scales[3 * g + 2]};
            float g_s[3], g_q[4];
            geomgrad::factor_grad(g_cov, q, s, g_s, g_q);
#pragma unroll
            for (int i = 0; i < 3; i++) dL_dscale[3 * g + i] = g_s[i];
            // scalar stores: dL_drot may be any 4-byte-aligned view, as the other per-Gaussian buffers
#pragma unroll
            for (int i = 0; i < 4; i++) dL_drot[4 * g + i] = g_q[i];
        }
    };
    if constexpr (!CAM) {
        if (g >= (size_t)P || !(radii[g] > 0)) return;  // culled Gaussians keep the caller's zeros (backward.cu:163,350)
        one_gaussian();
    } else {
        // every thread takes part in the reduction; a culled Gaussian contributes zeros
#pragma unroll
        for (int i = 0; i < 35; i++) gcam[i] = 0.f;
        if (g < (size_t)P && radii[g] > 0) one_gaussian();
        __shared__ double warp_sum[256 / 32][kCamSlots];
        const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
        for (int k = 0; k < kCamSlots; k++) {
            double x = gcam[cam_slot_entry(k)];
#pragma unroll
            for (int off = 16; off > 0; off >>= 1) x += __shfl_down_sync(0xffffffffu, x, off);
            if (lane == 0) warp_sum[warp][k] = x;
        }
        __syncthreads();
        if (threadIdx.x < kCamSlots) {
            double x = warp_sum[0][threadIdx.x];
#pragma unroll
            for (int w = 1; w < 256 / 32; w++) x += warp_sum[w][threadIdx.x];
            cam_partial[(size_t)threadIdx.x * gridDim.x + blockIdx.x] = x;
        }
    }
}

// One warp per reduction slot: the slot's per-CTA partials summed in a fixed order (four strided fp64 chains per lane,
// then a shuffle tree), written once in fp32.  Warp kCamSlots writes the 8 entries the forward never reads as 0.
__global__ void __launch_bounds__(1024) camera_grad_finalize_kernel(int nblocks, const double* __restrict__ partial,
                                                                    float* __restrict__ dview, float* __restrict__ dproj,
                                                                    float* __restrict__ dcampos) {
    const int lane = threadIdx.x & 31, k = threadIdx.x >> 5;
    auto out = [&](int e) -> float* { return e < 16 ? dview + e : e < 32 ? dproj + (e - 16) : dcampos + (e - 32); };
    if (k == kCamSlots) {
        if (lane < 8) *out(lane < 4 ? 4 * lane + 3 : 16 + 4 * (lane - 4) + 2) = 0.f;
        return;
    }
    if (k > kCamSlots) return;
    const double* src = partial + (size_t)k * nblocks;
    double a0 = 0.0, a1 = 0.0, a2 = 0.0, a3 = 0.0;
    int b = lane;
    for (; b + 96 < nblocks; b += 128) {
        a0 += src[b];
        a1 += src[b + 32];
        a2 += src[b + 64];
        a3 += src[b + 96];
    }
    for (; b < nblocks; b += 32) a0 += src[b];
    double x = (a0 + a1) + (a2 + a3);
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) x += __shfl_down_sync(0xffffffffu, x, off);
    if (lane == 0) *out(cam_slot_entry(k)) = (float)x;
}

}  // namespace

int launch_geom_backward(const sgb_view_inputs& in, GeomView g, const int32_t* radii, const float* cov3D,
                         const float* dL_dcolor_rgb, const sgb_view_grads& gr, const float* dL_ddepth,
                         const sgb_camera_grads* cam_grads, double* cam_partial, cudaStream_t s) {
    const float focal_y = in.H / (2.0f * in.tan_fovy);
    const float focal_x = in.W / (2.0f * in.tan_fovx);
    const int blocks = (in.P + 255) / 256;
    auto kernel = cam_grads ? (in.antialiasing ? geom_backward_kernel<true, true> : geom_backward_kernel<true, false>)
                            : (in.antialiasing ? geom_backward_kernel<false, true> : geom_backward_kernel<false, false>);
    kernel<<<blocks, 256, 0, s>>>(
        in.P, in.D, in.M, in.means3D, radii, in.shs, g.clamped, in.scales,
        in.rotations, in.scale_modifier, cov3D, in.viewmatrix, in.projmatrix, focal_x, focal_y,
        in.tan_fovx, in.tan_fovy, in.campos, gr.dL_dmeans2D, gr.dL_dconic, gr.dL_dmeans3D, dL_dcolor_rgb,
        gr.dL_dcov3D, gr.dL_dsh, gr.dL_dscales, gr.dL_drotations, dL_ddepth, cam_partial, g.rec, in.opacities,
        gr.dL_dopacity);
    SGB_LAUNCH_CHECK("geom_backward_kernel", in.debug, s);
    if (!cam_grads) return SGB_OK;
    camera_grad_finalize_kernel<<<1, 1024, 0, s>>>(blocks, cam_partial, cam_grads->dL_dviewmatrix,
                                                   cam_grads->dL_dprojmatrix, cam_grads->dL_dcampos);
    SGB_LAUNCH_CHECK("camera_grad_finalize_kernel", in.debug, s);
    return SGB_OK;
}

size_t camera_grad_partial_bytes(int32_t P) { return sizeof(double) * kCamSlots * (size_t)((P + 255) / 256); }

}  // namespace sgb
