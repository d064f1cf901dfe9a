// Per-Gaussian gradient algebra of the geometry stage, written as matrix calculus on small dense arrays.
//
// What it differentiates (reference forward.cu:74-118, 154-256): the screen-space conic K = (A S A^T + 0.3 I)^-1 of a
// Gaussian with world covariance S = R diag(s)^2 R^T, where A = J(t) W is the 2x3 perspective Jacobian at the
// (frustum-clamped) view-space centre t times the camera rotation W; the projected centre; the SH colour.  The
// reference differentiates these with two kernels of hand-expanded scalar expressions (backward.cu:141-271, :275-391).
// Here every step is one line of linear algebra:
//
//     K = C^-1                    =>  dL/dC = -C^-1 (dL/dK) C^-1 = -adj(C) (dL/dK) adj(C) / det(C)^2
//     C = A S A^T + 0.3 I         =>  dL/dS = A^T (dL/dC) A,      dL/dA = 2 (dL/dC) A S
//     A_0j = fx/tz (W_0j - u W_2j),  A_1j = fy/tz (W_1j - v W_2j),  u = tx/tz, v = ty/tz (clamped)
//     S = L L^T, L = R diag(s)    =>  dL/dL = 2 (dL/dS) L,  dL/ds_k = <dL/dL_:k, R_:k>,  dL/dR = dL/dL diag(s)
//     c = sum_k Y_k(d) sh_k       =>  dL/dsh_k = Y_k dL/dc,  dL/dd = sum_k grad Y_k <sh_k, dL/dc>,  d = v/|v|
//
// Conventions kept from the reference because they are visible in its outputs: dL/dK_xy arrives already halved
// (backward.cu:545) and the symmetric 3x3 gradient leaves as six numbers with the off-diagonal ones doubled
// (backward.cu:205-210); det^2 is regularised by 1e-7 (:186); the clamp masks only the direct tx, ty terms (:252-253);
// the scale gradient is taken w.r.t. the already-modified scale (:316-318); the quaternion is not re-normalised.
//
// The functions are __host__ __device__ so that tests/test_geom_grad_cpu.py can compile them with g++ and compare them
// with the oracle on the CPU box; the product calls them from geom_backward_kernel only.
#pragma once

#if defined(__CUDACC__)
#define SGB_HD __host__ __device__ __forceinline__
#else
#define SGB_HD inline
#endif

namespace sgb {
namespace geomgrad {

// What project_grad knows on the way that the camera gradient needs (camera_grad below): dL/dt of the view-space
// centre, dL/dA of A = J W, the Jacobian's scale and clamped evaluation point, and dL/d(homogeneous projected centre).
struct ProjectTerms {
    float gt[3];
    float gA[2][3];
    float ax, ay, u, v;
    float g_hom[4];
};

// ---------------------------------------------------------------- anti-aliasing: opacity-compensated 0.3 px² dilation
// The screen-space filter of Mip-Splatting as 3DGS ships it: with C0 = (a0, b; b, c0) the screen covariance before
// the dilation and C = C0 + s I (s = 0.3, the conic's matrix), the blend reads the opacity o h with
//     r = det C0 / det C,   h = sqrt(max(eps, r)),   eps = 2.5e-5
// so a Gaussian keeps the integral o 2 pi sqrt(det C0) of its undilated footprint at every image size.  The floor keeps
// degenerate and flat Gaussians finite (det C0 can round negative) and has zero gradient.
constexpr float kAADilation = 0.3f;
constexpr float kAAFloor = 2.5e-5f;

// h of one Gaussian from C0 and the det C the conic inversion uses, signed: negative on the floor branch (r <= eps),
// where the backward adds no covariance term.  The geometry state keeps it for the backward.
SGB_HD float aa_scale(float a0, float b, float c0, float det) {
    const float r = (a0 * c0 - b * b) / det;
    return r > kAAFloor ? sqrtf(r) : -sqrtf(kAAFloor);
}

// dL/d(a0, b, c0) = g_r dr/d(a0, b, c0) with D = det C:
//     dr/da0 = s (c0^2 + s c0 + b^2) / D^2,  dr/dc0 = s (a0^2 + s a0 + b^2) / D^2,  dr/db = -2 s b (a0 + c0 + s) / D^2
// b is the off-diagonal VALUE (one variable, appearing twice in C), so out[1] is the full dL/db.
SGB_HD void aa_cov_grad(float a0, float b, float c0, float D, float g_r, float out[3]) {
    const float s = kAADilation;
    const float k = g_r * s / (D * D);
    out[0] = k * (c0 * c0 + s * c0 + b * b);
    out[1] = -2.f * k * b * (a0 + c0 + s);
    out[2] = k * (a0 * a0 + s * a0 + b * b);
}

// ---------------------------------------------------------------- conic / centre -> world mean and covariance
// view, proj: column-major 4x4 as the reference passes them (element (row i, col j) at [4 j + i]).
// g_conic = (dL/dK_xx, dL/dK_xy [halved], dL/dK_yy), g_ndc = dL/d(projected centre in NDC units).
// out_mean[3] = dL/dp (both paths summed), out_cov[6] = dL/d(S_xx, S_xy, S_xz, S_yy, S_yz, S_zz).
// terms: NULL, or filled for camera_grad.  Filling it only copies values already computed (no value computed for
// out_mean / out_cov gains a use that could change how it is rounded).
// aa_g_r: NULL without anti-aliasing, else dL/dr of the opacity factor above (0 on its floor branch); its covariance
// term joins dL/dC before anything is formed from it, so it reaches the mean, covariance and camera gradients.
SGB_HD void project_grad(const float p[3], const float cov6[6], const float* view, const float* proj, float fx, float fy,
                         float tan_x, float tan_y, const float g_conic[3], const float g_ndc[2], float out_mean[3],
                         float out_cov[6], ProjectTerms* terms = nullptr, const float* aa_g_r = nullptr) {
    // view-space centre, frustum clamp of the Jacobian's evaluation point
    float t[3];
#pragma unroll
    for (int i = 0; i < 3; i++) t[i] = view[i] * p[0] + view[4 + i] * p[1] + view[8 + i] * p[2] + view[12 + i];
    const float lim_u = 1.3f * tan_x, lim_v = 1.3f * tan_y;
    const float u_raw = t[0] / t[2], v_raw = t[1] / t[2];
    const float u = fminf(lim_u, fmaxf(-lim_u, u_raw)), v = fminf(lim_v, fmaxf(-lim_v, v_raw));
    const float pass_u = (u_raw < -lim_u || u_raw > lim_u) ? 0.f : 1.f;
    const float pass_v = (v_raw < -lim_v || v_raw > lim_v) ? 0.f : 1.f;
    const float iz = 1.f / t[2];
    const float ax = fx * iz, ay = fy * iz;

    // A = J W (2x3), B = A S (2x3), C = B A^T + 0.3 I
    float A[2][3], B[2][3];
#pragma unroll
    for (int j = 0; j < 3; j++) {
        A[0][j] = ax * (view[4 * j + 0] - u * view[4 * j + 2]);
        A[1][j] = ay * (view[4 * j + 1] - v * view[4 * j + 2]);
    }
    const float S[3][3] = {{cov6[0], cov6[1], cov6[2]}, {cov6[1], cov6[3], cov6[4]}, {cov6[2], cov6[4], cov6[5]}};
#pragma unroll
    for (int r = 0; r < 2; r++)
#pragma unroll
        for (int j = 0; j < 3; j++) B[r][j] = A[r][0] * S[0][j] + A[r][1] * S[1][j] + A[r][2] * S[2][j];
    const float ca = B[0][0] * A[0][0] + B[0][1] * A[0][1] + B[0][2] * A[0][2] + 0.3f;
    const float cb = B[0][0] * A[1][0] + B[0][1] * A[1][1] + B[0][2] * A[1][2];
    const float cc = B[1][0] * A[1][0] + B[1][1] * A[1][1] + B[1][2] * A[1][2] + 0.3f;

    // dL/dC = -adj(C) G adj(C) / (det^2 + 1e-7), G = [[gx, gy], [gy, gz]]
    const float det = ca * cc - cb * cb;
    const float scale = 1.f / (det * det + 0.0000001f);
    float m00 = 0.f, m01 = 0.f, m11 = 0.f;
    if (scale != 0.f) {
        const float gx = g_conic[0], gy = g_conic[1], gz = g_conic[2];
        // rows of adj(C) G:  [cc gx - cb gy, cc gy - cb gz],  [ca gy - cb gx, ca gz - cb gy]
        const float h00 = cc * gx - cb * gy, h01 = cc * gy - cb * gz;
        const float h10 = ca * gy - cb * gx, h11 = ca * gz - cb * gy;
        m00 = -scale * (h00 * cc - h01 * cb);
        m01 = -scale * (h01 * ca - h00 * cb);
        m11 = -scale * (h11 * ca - h10 * cb);
    }
    if (aa_g_r && *aa_g_r != 0.f) {
        // M is dL/dC as a symmetric matrix (dL/dA = 2 M B): the off-diagonal entry takes half of dL/db
        const float a0 = B[0][0] * A[0][0] + B[0][1] * A[0][1] + B[0][2] * A[0][2];
        const float c0 = B[1][0] * A[1][0] + B[1][1] * A[1][1] + B[1][2] * A[1][2];
        float g[3];
        aa_cov_grad(a0, cb, c0, det, *aa_g_r, g);
        m00 += g[0];
        m01 += 0.5f * g[1];
        m11 += g[2];
    }

    // dL/dS = A^T M A (symmetric; off-diagonal outputs doubled), dL/dA = 2 M B
    float N[2][3], gA[2][3];
#pragma unroll
    for (int j = 0; j < 3; j++) {
        N[0][j] = m00 * A[0][j] + m01 * A[1][j];
        N[1][j] = m01 * A[0][j] + m11 * A[1][j];
        gA[0][j] = 2.f * (m00 * B[0][j] + m01 * B[1][j]);
        gA[1][j] = 2.f * (m01 * B[0][j] + m11 * B[1][j]);
    }
    out_cov[0] = A[0][0] * N[0][0] + A[1][0] * N[1][0];
    out_cov[3] = A[0][1] * N[0][1] + A[1][1] * N[1][1];
    out_cov[5] = A[0][2] * N[0][2] + A[1][2] * N[1][2];
    out_cov[1] = 2.f * (A[0][0] * N[0][1] + A[1][0] * N[1][1]);
    out_cov[2] = 2.f * (A[0][0] * N[0][2] + A[1][0] * N[1][2]);
    out_cov[4] = 2.f * (A[0][1] * N[0][2] + A[1][1] * N[1][2]);

    // dL/dJ (the four entries that depend on t) and dL/dt
    float j00 = 0.f, j02 = 0.f, j11 = 0.f, j12 = 0.f;
#pragma unroll
    for (int j = 0; j < 3; j++) {
        j00 += gA[0][j] * view[4 * j + 0];
        j02 += gA[0][j] * view[4 * j + 2];
        j11 += gA[1][j] * view[4 * j + 1];
        j12 += gA[1][j] * view[4 * j + 2];
    }
    const float iz2 = iz * iz;
    const float gt[3] = {-pass_u * fx * iz2 * j02, -pass_v * fy * iz2 * j12,
                         iz2 * (2.f * (fx * u * j02 + fy * v * j12) - fx * j00 - fy * j11)};

    // projected centre: ndc_k = hom_k / (hom_w + 1e-7)
    float hom[4];
#pragma unroll
    for (int k = 0; k < 4; k++) hom[k] = proj[k] * p[0] + proj[4 + k] * p[1] + proj[8 + k] * p[2] + proj[12 + k];
    const float iw = 1.f / (hom[3] + 0.0000001f);
    const float along = (g_ndc[0] * hom[0] + g_ndc[1] * hom[1]) * iw;
#pragma unroll
    for (int j = 0; j < 3; j++) {
        const float via_cov = view[4 * j + 0] * gt[0] + view[4 * j + 1] * gt[1] + view[4 * j + 2] * gt[2];
        const float via_ndc = iw * (g_ndc[0] * proj[4 * j + 0] + g_ndc[1] * proj[4 * j + 1] - proj[4 * j + 3] * along);
        out_mean[j] = via_cov + via_ndc;
    }
    if (terms) {
#pragma unroll
        for (int i = 0; i < 3; i++) {
            terms->gt[i] = gt[i];
            terms->gA[0][i] = gA[0][i];
            terms->gA[1][i] = gA[1][i];
        }
        terms->ax = ax;
        terms->ay = ay;
        terms->u = u;
        terms->v = v;
        // ndc_k = hom_k iw, iw = 1 / (hom_w + 1e-7)
        terms->g_hom[0] = g_ndc[0] * iw;
        terms->g_hom[1] = g_ndc[1] * iw;
        terms->g_hom[2] = 0.f;
        terms->g_hom[3] = -along * iw;
    }
}

// ---------------------------------------------------------------- one Gaussian's camera gradient
// ADDS this Gaussian's contribution to dL/dview[16], dL/dproj[16] (element order of view / proj above) and, with
// g_campos (the SH colour's view-direction term, colour_grad's campos_grad) non-NULL, dL/dcampos[3].  t = W p + t0:
//     via t:        dL/dW_ij += gt_i p_j,  dL/dt0_i += gt_i
//     via A = J W:  A_0j = ax (W_0j - u W_2j), A_1j = ay (W_1j - v W_2j) with the clamped u, v held as the forward holds
//                   them (their dependence on t is gt's)
//     via z = t_2:  dL/dW_2j += gz p_j, dL/dt0_2 += gz   (expected depth; gz = 0 without it)
//     via hom = Proj (p, 1):  dL/dProj_kj += dL/dhom_k p_j
// Entries the forward never reads (view row 3, proj row 2) receive nothing.  Focal lengths and tan(fov) are constants.
SGB_HD void camera_grad(const float p[3], const ProjectTerms& k, float gz, const float* g_campos, float dview[16],
                        float dproj[16], float dcampos[3]) {
    const float ph[4] = {p[0], p[1], p[2], 1.f};
#pragma unroll
    for (int j = 0; j < 4; j++) {
#pragma unroll
        for (int i = 0; i < 3; i++) dview[4 * j + i] += k.gt[i] * ph[j];
        dview[4 * j + 2] += gz * ph[j];
        dproj[4 * j + 0] += k.g_hom[0] * ph[j];
        dproj[4 * j + 1] += k.g_hom[1] * ph[j];
        dproj[4 * j + 3] += k.g_hom[3] * ph[j];
    }
#pragma unroll
    for (int j = 0; j < 3; j++) {
        dview[4 * j + 0] += k.ax * k.gA[0][j];
        dview[4 * j + 1] += k.ay * k.gA[1][j];
        dview[4 * j + 2] -= k.ax * k.u * k.gA[0][j] + k.ay * k.v * k.gA[1][j];
    }
    if (g_campos) {
#pragma unroll
        for (int i = 0; i < 3; i++) dcampos[i] += g_campos[i];
    }
}

// ---------------------------------------------------------------- world covariance -> scale, rotation
// g_cov6: as out_cov above.  q = (r, x, y, z).  s = scale_modifier * scale.
SGB_HD void factor_grad(const float g_cov6[6], const float q[4], const float s[3], float out_scale[3], float out_q[4]) {
    const float r = q[0], x = q[1], y = q[2], z = q[3];
    const float R[3][3] = {{1.f - 2.f * (y * y + z * z), 2.f * (x * y - r * z), 2.f * (x * z + r * y)},
                           {2.f * (x * y + r * z), 1.f - 2.f * (x * x + z * z), 2.f * (y * z - r * x)},
                           {2.f * (x * z - r * y), 2.f * (y * z + r * x), 1.f - 2.f * (x * x + y * y)}};
    const float G[3][3] = {{g_cov6[0], 0.5f * g_cov6[1], 0.5f * g_cov6[2]},
                           {0.5f * g_cov6[1], g_cov6[3], 0.5f * g_cov6[4]},
                           {0.5f * g_cov6[2], 0.5f * g_cov6[4], g_cov6[5]}};
    float D[3][3];  // dL/dR = 2 G R diag(s)^2 ... built column by column: H = 2 G L, D_:k = s_k H_:k
#pragma unroll
    for (int k = 0; k < 3; k++) {
        float dot = 0.f;
#pragma unroll
        for (int i = 0; i < 3; i++) {
            const float h = 2.f * s[k] * (G[i][0] * R[0][k] + G[i][1] * R[1][k] + G[i][2] * R[2][k]);
            dot += h * R[i][k];
            D[i][k] = h * s[k];
        }
        out_scale[k] = dot;
    }
    // R(q) is quadratic in q: antisymmetric part of D pairs with r, symmetric part with (x, y, z)
    const float a0 = D[2][1] - D[1][2], a1 = D[0][2] - D[2][0], a2 = D[1][0] - D[0][1];
    const float s01 = D[0][1] + D[1][0], s02 = D[0][2] + D[2][0], s12 = D[1][2] + D[2][1];
    out_q[0] = 2.f * (x * a0 + y * a1 + z * a2);
    out_q[1] = 2.f * (r * a0 + y * s01 + z * s02) - 4.f * x * (D[1][1] + D[2][2]);
    out_q[2] = 2.f * (r * a1 + x * s01 + z * s12) - 4.f * y * (D[0][0] + D[2][2]);
    out_q[3] = 2.f * (r * a2 + x * s02 + y * s12) - 4.f * z * (D[0][0] + D[1][1]);
}

// ---------------------------------------------------------------- SH colour -> coefficients, view direction
// Real SH basis up to degree 3 in the reference's ordering and sign convention (sh_utils.py:56-115, auxiliary.h:22-39)
// and its Cartesian gradient.  n = number of coefficients of the active degree ((deg + 1)^2).
SGB_HD void sh_basis(int deg, float x, float y, float z, float Y[16], float dY[16][3]) {
    const float k0 = 0.28209479177387814f, k1 = 0.4886025119029199f;
    const float k2a = 1.0925484305920792f, k2b = 0.31539156525252005f, k2c = 0.5462742152960396f;
    const float k3a = 0.5900435899266435f, k3b = 2.890611442640554f, k3c = 0.4570457994644658f;
    const float k3d = 0.3731763325901154f, k3e = 1.445305721320277f;
    Y[0] = k0; dY[0][0] = dY[0][1] = dY[0][2] = 0.f;
    if (deg < 1) return;
    Y[1] = -k1 * y; dY[1][0] = 0.f;  dY[1][1] = -k1; dY[1][2] = 0.f;
    Y[2] = k1 * z;  dY[2][0] = 0.f;  dY[2][1] = 0.f; dY[2][2] = k1;
    Y[3] = -k1 * x; dY[3][0] = -k1;  dY[3][1] = 0.f; dY[3][2] = 0.f;
    if (deg < 2) return;
    const float xx = x * x, yy = y * y, zz = z * z, xy = x * y, yz = y * z, xz = x * z;
    Y[4] = k2a * xy;                  dY[4][0] = k2a * y;        dY[4][1] = k2a * x;        dY[4][2] = 0.f;
    Y[5] = -k2a * yz;                 dY[5][0] = 0.f;            dY[5][1] = -k2a * z;       dY[5][2] = -k2a * y;
    Y[6] = k2b * (2.f * zz - xx - yy); dY[6][0] = -2.f * k2b * x; dY[6][1] = -2.f * k2b * y; dY[6][2] = 4.f * k2b * z;
    Y[7] = -k2a * xz;                 dY[7][0] = -k2a * z;       dY[7][1] = 0.f;            dY[7][2] = -k2a * x;
    Y[8] = k2c * (xx - yy);           dY[8][0] = 2.f * k2c * x;  dY[8][1] = -2.f * k2c * y; dY[8][2] = 0.f;
    if (deg < 3) return;
    Y[9] = -k3a * y * (3.f * xx - yy);
    dY[9][0] = -6.f * k3a * xy; dY[9][1] = -3.f * k3a * (xx - yy); dY[9][2] = 0.f;
    Y[10] = k3b * xy * z;
    dY[10][0] = k3b * yz; dY[10][1] = k3b * xz; dY[10][2] = k3b * xy;
    Y[11] = -k3c * y * (4.f * zz - xx - yy);
    dY[11][0] = 2.f * k3c * xy; dY[11][1] = -k3c * (4.f * zz - xx - 3.f * yy); dY[11][2] = -8.f * k3c * yz;
    Y[12] = k3d * z * (2.f * zz - 3.f * xx - 3.f * yy);
    dY[12][0] = -6.f * k3d * xz; dY[12][1] = -6.f * k3d * yz; dY[12][2] = 3.f * k3d * (2.f * zz - xx - yy);
    Y[13] = -k3c * x * (4.f * zz - xx - yy);
    dY[13][0] = -k3c * (4.f * zz - 3.f * xx - yy); dY[13][1] = 2.f * k3c * xy; dY[13][2] = -8.f * k3c * xz;
    Y[14] = k3e * z * (xx - yy);
    dY[14][0] = 2.f * k3e * xz; dY[14][1] = -2.f * k3e * yz; dY[14][2] = k3e * (xx - yy);
    Y[15] = -k3a * x * (xx - 3.f * yy);
    dY[15][0] = -3.f * k3a * (xx - yy); dY[15][1] = 6.f * k3a * xy; dY[15][2] = 0.f;
}

// sh: the Gaussian's [max_coeffs][3] coefficients; g_rgb: dL/d(colour), already zeroed where the forward clamped.
// Writes out_sh[(deg+1)^2][3]; ADDS the view-direction path to mean_grad[3].  campos_grad: NULL, or receives the same
// path for the camera centre, v = p - campos: -(what mean_grad gains), written as d <d, g> / |v| - g / |v| so that the
// product added to mean_grad keeps its single use (and so its rounding).
SGB_HD void colour_grad(int deg, const float p[3], const float* campos, const float* sh, const float g_rgb[3],
                        float* out_sh, float mean_grad[3], float* campos_grad = nullptr) {
    const float v[3] = {p[0] - campos[0], p[1] - campos[1], p[2] - campos[2]};
    const float len2 = v[0] * v[0] + v[1] * v[1] + v[2] * v[2];
    const float ilen = 1.f / sqrtf(len2);
    const float d[3] = {v[0] * ilen, v[1] * ilen, v[2] * ilen};
    float Y[16], dY[16][3];
    sh_basis(deg, d[0], d[1], d[2], Y, dY);
    const int n = (deg + 1) * (deg + 1);
    float gd[3] = {0.f, 0.f, 0.f};
#pragma unroll
    for (int k = 0; k < 16; k++) {
        if (k < n) {
            out_sh[3 * k + 0] = Y[k] * g_rgb[0];
            out_sh[3 * k + 1] = Y[k] * g_rgb[1];
            out_sh[3 * k + 2] = Y[k] * g_rgb[2];
            const float w = sh[3 * k] * g_rgb[0] + sh[3 * k + 1] * g_rgb[1] + sh[3 * k + 2] * g_rgb[2];
            gd[0] += dY[k][0] * w;
            gd[1] += dY[k][1] * w;
            gd[2] += dY[k][2] * w;
        }
    }
    // d = v / |v|:  dL/dv = (g - d <d, g>) / |v|
    const float radial = d[0] * gd[0] + d[1] * gd[1] + d[2] * gd[2];
#pragma unroll
    for (int i = 0; i < 3; i++) mean_grad[i] += (gd[i] - d[i] * radial) * ilen;
    if (campos_grad) {
        const float radial_ilen = radial * ilen;
#pragma unroll
        for (int i = 0; i < 3; i++) campos_grad[i] = d[i] * radial_ilen - gd[i] * ilen;
    }
}

}  // namespace geomgrad
}  // namespace sgb
