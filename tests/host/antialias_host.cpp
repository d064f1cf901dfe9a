// TEST INFRASTRUCTURE: compiles the product's anti-aliasing terms (semantic-gaussians_b200/csrc/geom_grad.cuh:
// aa_scale as preprocess_kernel<true> calls it, and project_grad with aa_g_r as geom_backward_kernel<*, true> calls it)
// for the host so that tests/test_antialias_cpu.py and tests/test_antialias_ref_cpu.py can compare them with the
// float64 restatements without a GPU.
#include <cmath>
#include <cstddef>
#include <cstdint>
#include "geom_grad.cuh"

// Signed h of n screen covariances C0 = (a0, b, c0), with det C formed from C0 + 0.3 I in the preprocess's order.
extern "C" void host_aa_scale(int n, const float* a0, const float* b, const float* c0, float* out_h) {
    for (int i = 0; i < n; i++) {
        const float a = a0[i] + 0.3f, c = c0[i] + 0.3f;
        out_h[i] = sgb::geomgrad::aa_scale(a0[i], b[i], c0[i], a * c - b[i] * b[i]);
    }
}

// g_r dr/d(a0, b, c0) of n covariances, 3 per row.
extern "C" void host_aa_cov_grad(int n, const float* a0, const float* b, const float* c0, const float* g_r,
                                 float* out) {
    for (int i = 0; i < n; i++) {
        const float a = a0[i] + 0.3f, c = c0[i] + 0.3f;
        sgb::geomgrad::aa_cov_grad(a0[i], b[i], c0[i], a * c - b[i] * b[i], g_r[i], out + 3 * i);
    }
}

// project_grad of n Gaussians with the anti-aliasing term (aa_g_r[i]) and the given conic / centre gradients:
// out_mean (n, 3), out_cov (n, 6).
extern "C" void host_project_grad_aa(int n, const float* means3D, const float* cov3Ds, const float* view,
                                     const float* proj, float fx, float fy, float tan_x, float tan_y,
                                     const float* g_conic, const float* g_ndc, const float* aa_g_r, float* out_mean,
                                     float* out_cov) {
    for (size_t g = 0; g < (size_t)n; g++)
        sgb::geomgrad::project_grad(means3D + 3 * g, cov3Ds + 6 * g, view, proj, fx, fy, tan_x, tan_y, g_conic + 3 * g,
                                    g_ndc + 2 * g, out_mean + 3 * g, out_cov + 6 * g, nullptr, aa_g_r + g);
}

// geom_backward_kernel<false, true> for the host: the argument list of host_geom_backward (geom_grad_host.cpp) plus
// the raw opacities, the signed h of the forward (aa_h, as preprocess_kernel<true> stores it) and dL_dopacity, which
// holds dL/d(o h) on entry and dL/do = |h| dL/d(o h) on return.
extern "C" void host_geom_backward_aa(int P, int D, int M, const float* means3D, const int* radii, const float* shs,
                                      const uint8_t* clamped, const float* scales, const float* rotations,
                                      float scale_modifier, const float* cov3Ds, const float* view, const float* proj,
                                      float focal_x, float focal_y, float tan_fovx, float tan_fovy,
                                      const float* campos, const float* dL_dmean2D, const float* dL_dconics,
                                      float* dL_dmeans, const float* dL_dcolor, float* dL_dcov, float* dL_dsh,
                                      float* dL_dscale, float* dL_drot, const float* opacities, const float* aa_h,
                                      float* dL_dopacity) {
    using namespace sgb::geomgrad;
    for (size_t g = 0; g < (size_t)P; g++) {
        if (!(radii[g] > 0)) continue;
        const float* p = means3D + 3 * g;
        const float g_conic[3] = {dL_dconics[4 * g], dL_dconics[4 * g + 1], dL_dconics[4 * g + 3]};
        const float g_ndc[2] = {dL_dmean2D[3 * g], dL_dmean2D[3 * g + 1]};
        const float hs = aa_h[g], h = std::fabs(hs);
        const float g_op = dL_dopacity[g];
        dL_dopacity[g] = h * g_op;
        const float g_r = hs > 0.f ? opacities[g] * g_op / (2.f * h) : 0.f;
        float g_mean[3], g_cov[6];
        project_grad(p, cov3Ds + 6 * g, view, proj, focal_x, focal_y, tan_fovx, tan_fovy, g_conic, g_ndc, g_mean, g_cov,
                     nullptr, &g_r);
        for (int i = 0; i < 6; i++) dL_dcov[6 * g + i] = g_cov[i];
        if (shs) {
            float g_rgb[3];
            for (int c = 0; c < 3; c++) g_rgb[c] = clamped[3 * g + c] ? 0.f : dL_dcolor[3 * g + c];
            colour_grad(D, p, campos, shs + g * (size_t)M * 3, g_rgb, dL_dsh + g * (size_t)M * 3, g_mean);
        }
        for (int i = 0; i < 3; i++) dL_dmeans[3 * g + i] = g_mean[i];
        if (scales) {
            const float s[3] = {scale_modifier * scales[3 * g], scale_modifier * scales[3 * g + 1],
                                scale_modifier * scales[3 * g + 2]};
            float g_s[3], g_q[4];
            factor_grad(g_cov, rotations + 4 * g, s, g_s, g_q);
            for (int i = 0; i < 3; i++) dL_dscale[3 * g + i] = g_s[i];
            for (int i = 0; i < 4; i++) dL_drot[4 * g + i] = g_q[i];
        }
    }
}
