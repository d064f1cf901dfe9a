// TEST INFRASTRUCTURE: compiles the product's per-Gaussian camera terms (semantic-gaussians_b200/csrc/geom_grad.cuh:
// project_grad's ProjectTerms, colour_grad's campos_grad and camera_grad, as geom_backward_kernel<true> calls them)
// for the host so that tests/test_camera_grad_cpu.py can compare them with a float64 restatement without a GPU.
// Writes one row of 35 per Gaussian (view 16 | proj 16 | campos 3); culled Gaussians get zeros.
#include <cmath>
#include <cstddef>
#include <cstdint>
#include "geom_grad.cuh"

extern "C" void host_camera_grad(int P, int D, int M, const float* means3D, const int* radii, const float* shs,
                                 const uint8_t* clamped, const float* cov3Ds, const float* view, const float* proj,
                                 float focal_x, float focal_y, float tan_fovx, float tan_fovy, const float* campos,
                                 const float* dL_dmean2D, const float* dL_dconics, const float* dL_dcolor,
                                 const float* dL_ddepth, float* sh_scratch, float* out_cam) {
    using namespace sgb::geomgrad;
    for (size_t g = 0; g < (size_t)P; g++) {
        float* row = out_cam + 35 * g;
        for (int i = 0; i < 35; i++) row[i] = 0.f;
        if (!(radii[g] > 0)) continue;
        const float* p = means3D + 3 * g;
        const float g_conic[3] = {dL_dconics[4 * g], dL_dconics[4 * g + 1], dL_dconics[4 * g + 3]};
        const float g_ndc[2] = {dL_dmean2D[3 * g], dL_dmean2D[3 * g + 1]};
        float g_mean[3], g_cov[6], g_campos[3];
        ProjectTerms terms;
        project_grad(p, cov3Ds + 6 * g, view, proj, focal_x, focal_y, tan_fovx, tan_fovy, g_conic, g_ndc, g_mean, g_cov,
                     &terms);
        if (shs) {
            float g_rgb[3];
            for (int c = 0; c < 3; c++) g_rgb[c] = clamped[3 * g + c] ? 0.f : dL_dcolor[3 * g + c];
            colour_grad(D, p, campos, shs + g * (size_t)M * 3, g_rgb, sh_scratch, g_mean, g_campos);
        }
        camera_grad(p, terms, dL_ddepth ? dL_ddepth[g] : 0.f, shs ? g_campos : nullptr, row, row + 16, row + 32);
    }
}
