// Per-Gaussian forward geometry: near cull, projection, 3D->2D covariance (EWA), conic, radius,
// tile rectangle, optional SH->RGB.  Behavioural contract: reference forward.cu:155-256 with its
// helpers (:20-151) and auxiliary.h:41-164.
//
// The integer outputs of this stage (radii, tile rects, tiles_touched) and the depth bits that
// drive the sort must equal the reference's bit for bit, and the floats that feed the alpha
// thresholds downstream (means2D, conic) too, or n_contrib flips at decision boundaries.  fp32
// rounding therefore has to match the reference *as nvcc compiles it* (mul/add contraction
// included).  The arithmetic below is written with the same expression trees the reference's
// GLM templates expand to (column-major 3x3 products with their zero terms kept), which nvcc
// contracts identically; tests/test_parity_gpu.py checks bit equality against the compiled
// reference on >= 10^6 Gaussians.
#include "common.cuh"
#include "geom_grad.cuh"
#include "linalg.cuh"

namespace sgb {

namespace {

// forward.cu:118-151.  Quaternion used as given (normalisation commented out there, :127).
__device__ void computeCov3D(const float3 scale, float mod, const float4 rot, float* cov3D) {
    M3 S = cols(1.0f, 0.f, 0.f, 0.f, 1.0f, 0.f, 0.f, 0.f, 1.0f);
    S.m[0][0] = mod * scale.x;
    S.m[1][1] = mod * scale.y;
    S.m[2][2] = mod * scale.z;
    float r = rot.x, x = rot.y, y = rot.z, z = rot.w;
    // r * y + x * z and r * x + y * z: the operand order the reference's GLM code reaches in PTX.  The sum is the
    // same either way, but ptxas fuses one of the two products into an FFMA, and on sm_90 it picks by operand order.
    M3 R = cols(1.f - 2.f * (y * y + z * z), 2.f * (x * y - r * z), 2.f * (r * y + x * z),
                2.f * (x * y + r * z), 1.f - 2.f * (x * x + z * z), 2.f * (y * z - r * x),
                2.f * (x * z - r * y), 2.f * (r * x + y * z), 1.f - 2.f * (x * x + y * y));
    M3 M = S * R;
    M3 Sigma = transpose(M) * M;
    cov3D[0] = Sigma.m[0][0];
    cov3D[1] = Sigma.m[0][1];
    cov3D[2] = Sigma.m[0][2];
    cov3D[3] = Sigma.m[1][1];
    cov3D[4] = Sigma.m[1][2];
    cov3D[5] = Sigma.m[2][2];
}

// forward.cu:74-113.  cov0: NULL, or receives the covariance before the 0.3 px² dilation (anti-aliasing).
__device__ float3 computeCov2D(const float3& mean, float focal_x, float focal_y, float tan_fovx,
                               float tan_fovy, const float* cov3D, const float* viewmatrix, float3* cov0 = nullptr) {
    float3 t = transformPoint4x3(mean, viewmatrix);
    const float limx = 1.3f * tan_fovx;
    const float limy = 1.3f * tan_fovy;
    const float txtz = t.x / t.z;
    const float tytz = t.y / t.z;
    t.x = min(limx, max(-limx, txtz)) * t.z;
    t.y = min(limy, max(-limy, tytz)) * t.z;
    M3 J = cols(focal_x / t.z, 0.0f, -(focal_x * t.x) / (t.z * t.z), 0.0f, focal_y / t.z,
                -(focal_y * t.y) / (t.z * t.z), 0, 0, 0);
    M3 W = cols(viewmatrix[0], viewmatrix[4], viewmatrix[8], viewmatrix[1], viewmatrix[5], viewmatrix[9],
                viewmatrix[2], viewmatrix[6], viewmatrix[10]);
    M3 T = W * J;
    M3 Vrk = cols(cov3D[0], cov3D[1], cov3D[2], cov3D[1], cov3D[3], cov3D[4], cov3D[2], cov3D[4], cov3D[5]);
    M3 cov = transpose(T) * transpose(Vrk) * T;
    if (cov0) *cov0 = {float(cov.m[0][0]), float(cov.m[0][1]), float(cov.m[1][1])};
    cov.m[0][0] += 0.3f;
    cov.m[1][1] += 0.3f;
    return {float(cov.m[0][0]), float(cov.m[0][1]), float(cov.m[1][1])};
}

// forward.cu:20-71
__device__ V3 computeColorFromSH(int idx, int deg, int max_coeffs, const float* means, const float* campos,
                                 const float* shs, uint8_t* clamped) {
    V3 pos = {means[3 * idx], means[3 * idx + 1], means[3 * idx + 2]};
    V3 cam = {campos[0], campos[1], campos[2]};
    V3 dir = pos - cam;
    float len = sqrtf(dir.x * dir.x + dir.y * dir.y + dir.z * dir.z);
    dir = {dir.x / len, dir.y / len, dir.z / len};
    const V3* sh = reinterpret_cast<const V3*>(shs) + (size_t)idx * max_coeffs;
    V3 result = SH_C0 * sh[0];
    if (deg > 0) {
        float x = dir.x, y = dir.y, z = dir.z;
        result = result - SH_C1 * y * sh[1] + SH_C1 * z * sh[2] - SH_C1 * x * sh[3];
        if (deg > 1) {
            float xx = x * x, yy = y * y, zz = z * z;
            float xy = x * y, yz = y * z, xz = x * z;
            result = result + SH_C2[0] * xy * sh[4] + SH_C2[1] * yz * sh[5] +
                     SH_C2[2] * (2.0f * zz - xx - yy) * sh[6] + SH_C2[3] * xz * sh[7] + SH_C2[4] * (xx - yy) * sh[8];
            if (deg > 2) {
                result = result + SH_C3[0] * y * (3.0f * xx - yy) * sh[9] + SH_C3[1] * xy * z * sh[10] +
                         SH_C3[2] * y * (4.0f * zz - xx - yy) * sh[11] +
                         SH_C3[3] * z * (2.0f * zz - 3.0f * xx - 3.0f * yy) * sh[12] +
                         SH_C3[4] * x * (4.0f * zz - xx - yy) * sh[13] + SH_C3[5] * z * (xx - yy) * sh[14] +
                         SH_C3[6] * x * (xx - 3.0f * yy) * sh[15];
            }
        }
    }
    result = result + 0.5f;
    clamped[3 * idx + 0] = (result.x < 0);
    clamped[3 * idx + 1] = (result.y < 0);
    clamped[3 * idx + 2] = (result.z < 0);
    return {fmaxf(result.x, 0.0f), fmaxf(result.y, 0.0f), fmaxf(result.z, 0.0f)};
}

// AA: anti-aliasing (geom_grad.cuh aa_scale).  The record's opacity is o h and its fourth float keeps the signed h for
// the geometry backward; everything else is what AA = false writes.
template <bool AA>
__global__ void __launch_bounds__(256) preprocess_kernel(
    int P, int D, int M, const float* __restrict__ orig_points, const float3* __restrict__ scales,
    const float scale_modifier, const float* __restrict__ rotations, const float* __restrict__ opacities,
    const float* __restrict__ shs, uint8_t* __restrict__ clamped, const float* __restrict__ cov3D_precomp,
    const float* __restrict__ colors_precomp, const float* __restrict__ viewmatrix,
    const float* __restrict__ projmatrix, const float* __restrict__ cam_pos, const int W, int H,
    const float tan_fovx, float tan_fovy, const float focal_x, float focal_y, int* __restrict__ radii,
    SplatRec* __restrict__ rec, float* __restrict__ cov3Ds, float* __restrict__ rgb, const dim3 grid,
    uint32_t* __restrict__ tiles_touched, uint32_t* __restrict__ depth_keys, bool prefiltered) {
    int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= P) return;

    radii[idx] = 0;
    tiles_touched[idx] = 0;
    depth_keys[idx] = 0xFFFFFFFFu;  // culled Gaussians order last; they emit no instance

    // in_frustum, auxiliary.h:139-164: near plane only.
    float3 p_orig = {orig_points[3 * idx], orig_points[3 * idx + 1], orig_points[3 * idx + 2]};
    float3 p_view = transformPoint4x3(p_orig, viewmatrix);
    if (p_view.z <= 0.2f) {
        if (prefiltered) {
            printf("Point is filtered although prefiltered is set. This shouldn't happen!");
            __trap();
        }
        return;
    }

    float4 p_hom = transformPoint4x4(p_orig, projmatrix);
    float p_w = 1.0f / (p_hom.w + 0.0000001f);
    float3 p_proj = {p_hom.x * p_w, p_hom.y * p_w, p_hom.z * p_w};

    const float* cov3D;
    if (cov3D_precomp != nullptr) {
        cov3D = cov3D_precomp + (size_t)idx * 6;
    } else {
        // scalar loads: the caller's rotations may be any 4-byte-aligned view (e.g. into a flat parameter buffer)
        const float* q = rotations + (size_t)idx * 4;
        computeCov3D(scales[idx], scale_modifier, make_float4(q[0], q[1], q[2], q[3]), cov3Ds + (size_t)idx * 6);
        cov3D = cov3Ds + (size_t)idx * 6;
    }

    float3 cov0;
    float3 cov = computeCov2D(p_orig, focal_x, focal_y, tan_fovx, tan_fovy, cov3D, viewmatrix, AA ? &cov0 : nullptr);

    float det = (cov.x * cov.z - cov.y * cov.y);
    if (det == 0.0f) return;
    float det_inv = 1.f / det;
    float3 conic = {cov.z * det_inv, -cov.y * det_inv, cov.x * det_inv};

    float mid = 0.5f * (cov.x + cov.z);
    float lambda1 = mid + sqrt(max(0.1f, mid * mid - det));
    float lambda2 = mid - sqrt(max(0.1f, mid * mid - det));
    float my_radius = ceil(3.f * sqrt(max(lambda1, lambda2)));
    float2 point_image = {ndc2Pix(p_proj.x, W), ndc2Pix(p_proj.y, H)};
    uint2 rect_min, rect_max;
    get_rect(point_image, my_radius, rect_min, rect_max, grid);
    if ((rect_max.x - rect_min.x) * (rect_max.y - rect_min.y) == 0) return;

    if (colors_precomp == nullptr) {
        V3 result = computeColorFromSH(idx, D, M, orig_points, cam_pos, shs, clamped);
        rgb[idx * 3 + 0] = result.x;
        rgb[idx * 3 + 1] = result.y;
        rgb[idx * 3 + 2] = result.z;
    }

    radii[idx] = my_radius;
    SplatRec r;
    r.mx = point_image.x;
    r.my = point_image.y;
    r.depth = p_view.z;
    r.pad = 0.f;
    r.cx = conic.x;
    r.cy = conic.y;
    r.cz = conic.z;
    r.op = opacities[idx];
    if constexpr (AA) {
        r.pad = geomgrad::aa_scale(cov0.x, cov0.y, cov0.z, det);
        r.op *= fabsf(r.pad);
    }
    float4* rp = reinterpret_cast<float4*>(rec + idx);
    rp[0] = make_float4(r.mx, r.my, r.depth, r.pad);
    rp[1] = make_float4(r.cx, r.cy, r.cz, r.op);
    tiles_touched[idx] = (rect_max.y - rect_min.y) * (rect_max.x - rect_min.x);
    depth_keys[idx] = __float_as_uint(p_view.z);
}

// rasterizer_impl.cu:54-66
__global__ void mark_visible_kernel(int P, const float* __restrict__ orig_points,
                                    const float* __restrict__ viewmatrix, uint8_t* __restrict__ present) {
    int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= P) return;
    float3 p = {orig_points[3 * idx], orig_points[3 * idx + 1], orig_points[3 * idx + 2]};
    float3 p_view = transformPoint4x3(p, viewmatrix);
    present[idx] = !(p_view.z <= 0.2f);
}

}  // namespace

int launch_preprocess(const sgb_view_inputs& in, GeomView g, int32_t* radii, uint32_t* depth_keys,
                      cudaStream_t s) {
    const float focal_y = in.H / (2.0f * in.tan_fovy);  // rasterizer_impl.cu:223-224
    const float focal_x = in.W / (2.0f * in.tan_fovx);
    dim3 tile_grid((in.W + SGB_TILE - 1) / SGB_TILE, (in.H + SGB_TILE - 1) / SGB_TILE, 1);
    auto kernel = in.antialiasing ? preprocess_kernel<true> : preprocess_kernel<false>;
    kernel<<<(in.P + 255) / 256, 256, 0, s>>>(
        in.P, in.D, in.M, in.means3D, (const float3*)in.scales, in.scale_modifier, in.rotations,
        in.opacities, in.shs, g.clamped, in.cov3D_precomp, in.colors_precomp, in.viewmatrix, in.projmatrix,
        in.campos, in.W, in.H, in.tan_fovx, in.tan_fovy, focal_x, focal_y, radii, g.rec, g.cov3D, g.rgb, tile_grid,
        g.tiles_touched, depth_keys, in.prefiltered != 0);
    SGB_LAUNCH_CHECK("preprocess_kernel", in.debug, s);
    return SGB_OK;
}

int launch_mark_visible(int P, const float* means3D, const float* view, uint8_t* present, cudaStream_t s) {
    mark_visible_kernel<<<(P + 255) / 256, 256, 0, s>>>(P, means3D, view, present);
    SGB_LAUNCH_CHECK("mark_visible_kernel", 0, s);
    return SGB_OK;
}

}  // namespace sgb
