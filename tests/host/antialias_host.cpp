// TEST INFRASTRUCTURE: compiles the product's anti-aliasing terms (semantic-gaussians_b200/csrc/geom_grad.cuh:
// aa_scale as preprocess_kernel<true> calls it, and project_grad with aa_g_r as geom_backward_kernel<*, true> calls it)
// for the host so that tests/test_antialias_cpu.py can compare them with a float64 restatement without a GPU.
#include <cmath>
#include <cstddef>
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
