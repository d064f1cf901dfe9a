// Photometric training loss of train.py:141-149:  L = (1 - lambda) * L1(x, y) + lambda * (1 - SSIM(x, y)),
// with SSIM as utils/loss_utils.py:38-72 computes it (11x11 Gaussian window, sigma 1.5, zero padding).
//
// The reference runs five depthwise 11x11 convolutions and ~15 full-size temporaries, then autograd replays all
// of it.  Here the loss is two kernels over fp32 planes (one plane = one channel of one image):
//
//   ssim_fwd_kernel  one 32x32 output tile of one plane per CTA.  x and y are staged with a 5-pixel halo (zeros
//                    outside the plane == conv2d's padding), the five moments x, y, x^2, y^2, xy are filtered
//                    as two separable 11-tap passes, and each pixel gives S, |x - y| (summed into two doubles) and
//                    the three maps a, b, c the gradient needs (written only when a gradient is wanted).
//   ssim_bwd_kernel  the same tiling over (a, b, c):  d(sum S)/dx = w*a + 2x (w*b) + y (w*c)  (the window is
//                    symmetric, so the adjoint of the correlation is the correlation itself), combined with the
//                    L1 term and the upstream weights read from device memory.
//
// Storing a, b, c (12 B per plane-pixel each way) rather than recomputing them in backward from x and y keeps
// the backward halo at 5 pixels and its arithmetic at three moments instead of five plus the per-pixel S
// algebra over a 42x42 (rather than 32x32) region.  Loads are scalar: a warp reads 32 consecutive floats of one
// row, which coalesces for any W and any crop offset, and the halo rows are not 16-byte aligned anyway.
#include <cstdint>

#include "common.cuh"

namespace sgb {
namespace {

constexpr int kLossTile = 32;                         // output tile: 32 x 32 pixels of one plane
constexpr int kLossHalo = 5;                          // window radius
constexpr int kLossIn = kLossTile + 2 * kLossHalo;    // 42: staged rows / columns
constexpr int kLossThreads = 256;                     // 8 warps; thread = one column x 4 consecutive rows
constexpr int kLossRows = kLossTile / (kLossThreads / kLossTile);  // 4

// gaussian(11, 1.5) of utils/loss_utils.py:26-28: fp32 exp values divided by their fp32 sum.
__constant__ float kSsimTaps[11] = {0x1.0d956cp-10f, 0x1.f1fe02p-8f, 0x1.26eb18p-5f, 0x1.bff0fep-4f,
                                    0x1.b43c3ep-3f,  0x1.106560p-2f, 0x1.b43c3ep-3f, 0x1.bff0fep-4f,
                                    0x1.26eb18p-5f,  0x1.f1fe02p-8f, 0x1.0d956cp-10f};
constexpr float kC1 = 0.01f * 0.01f;
constexpr float kC2 = 0.03f * 0.03f;

struct PlaneView {  // plane p, row r, column c  ->  base[p * ps + r * rs + c]
    const float* base;
    long long ps, rs;
    __device__ __forceinline__ float at(int p, int r, int c) const {
        return __ldg(base + (long long)p * ps + (long long)r * rs + c);
    }
};

// Stage NM planes of the tile's 42x42 window into s[m][42][42], zeros outside the h x w plane.
template <int NM>
__device__ __forceinline__ void stage_tile(float (*s)[kLossIn][kLossIn], const PlaneView* src, int p, int h, int w,
                                           int r0, int c0) {
    for (int i = threadIdx.x; i < kLossIn * kLossIn; i += kLossThreads) {
        const int r = i / kLossIn, c = i - r * kLossIn;
        const int gr = r0 + r - kLossHalo, gc = c0 + c - kLossHalo;
        const bool in = gr >= 0 && gr < h && gc >= 0 && gc < w;
#pragma unroll
        for (int m = 0; m < NM; m++) s[m][r][c] = in ? src[m].at(p, gr, gc) : 0.f;
    }
}

// Vertical 11-tap pass over hm[m][42][32] for this thread's column and 4 rows: out[j][m].
template <int NM>
__device__ __forceinline__ void vertical_pass(const float (*hm)[kLossIn][kLossTile], int col, int row0,
                                              float (&out)[kLossRows][NM]) {
#pragma unroll
    for (int j = 0; j < kLossRows; j++)
#pragma unroll
        for (int m = 0; m < NM; m++) out[j][m] = 0.f;
#pragma unroll
    for (int k = 0; k < kLossRows + 2 * kLossHalo; k++) {
        float v[NM];
#pragma unroll
        for (int m = 0; m < NM; m++) v[m] = hm[m][row0 + k][col];
#pragma unroll
        for (int j = 0; j < kLossRows; j++) {
            const int t = k - j;
            if (t >= 0 && t <= 2 * kLossHalo) {
#pragma unroll
                for (int m = 0; m < NM; m++) out[j][m] = fmaf(kSsimTaps[t], v[m], out[j][m]);
            }
        }
    }
}

__global__ void __launch_bounds__(kLossThreads) ssim_fwd_kernel(int planes, int h, int w, PlaneView X, PlaneView Y,
                                                                 double* __restrict__ sums, float* __restrict__ abc) {
    __shared__ float sxy[2][kLossIn][kLossIn];
    __shared__ float hm[5][kLossIn][kLossTile];
    __shared__ double wsum[kLossThreads / 32][2];
    const int c0 = blockIdx.x * kLossTile, r0 = blockIdx.y * kLossTile;
    const int col = threadIdx.x & 31, row0 = (threadIdx.x >> 5) * kLossRows;
    const long long hw = (long long)h * w;
    float l1 = 0.f, ssum = 0.f;
    for (int p = blockIdx.z; p < planes; p += gridDim.z) {
        const PlaneView src[2] = {X, Y};
        stage_tile<2>(sxy, src, p, h, w, r0, c0);
        __syncthreads();
        // horizontal pass: warp = one of the 42 staged rows, lane = output column
        for (int i = threadIdx.x; i < kLossIn * kLossTile; i += kLossThreads) {
            const int r = i >> 5, c = i & 31;
            float mx = 0.f, my = 0.f, mxx = 0.f, myy = 0.f, mxy = 0.f;
#pragma unroll
            for (int t = 0; t <= 2 * kLossHalo; t++) {
                const float a = sxy[0][r][c + t], b = sxy[1][r][c + t], g = kSsimTaps[t];
                const float ga = g * a, gb = g * b;
                mx += ga;
                my += gb;
                mxx = fmaf(ga, a, mxx);
                myy = fmaf(gb, b, myy);
                mxy = fmaf(ga, b, mxy);
            }
            hm[0][r][c] = mx; hm[1][r][c] = my; hm[2][r][c] = mxx; hm[3][r][c] = myy; hm[4][r][c] = mxy;
        }
        __syncthreads();
        float mom[kLossRows][5];
        vertical_pass<5>(hm, col, row0, mom);
        const int gc = c0 + col;
#pragma unroll
        for (int j = 0; j < kLossRows; j++) {
            const int gr = r0 + row0 + j;
            if (gr >= h || gc >= w) continue;
            const float x = sxy[0][row0 + j + kLossHalo][col + kLossHalo];
            const float y = sxy[1][row0 + j + kLossHalo][col + kLossHalo];
            const float mux = mom[j][0], muy = mom[j][1];
            const float vx = mom[j][2] - mux * mux, vy = mom[j][3] - muy * muy, cxy = mom[j][4] - mux * muy;
            const float A1 = 2.f * mux * muy + kC1, A2 = 2.f * cxy + kC2;
            const float B1 = mux * mux + muy * muy + kC1, B2 = vx + vy + kC2;
            const float r = 1.f / (B1 * B2);
            const float S = A1 * A2 * r;
            l1 += fabsf(x - y);
            ssum += S;
            if (abc) {
                // a = 2 muy A2/(B1 B2) - muy c + 2 mux S (1/B2 - 1/B1),  b = -S/B2,  c = 2 A1/(B1 B2)
                const float c = 2.f * A1 * r;
                const float a = muy * (2.f * A2 * r - c) + 2.f * mux * S * r * (B1 - B2);
                const float b = -S * B1 * r;
                const long long o = (long long)p * hw + (long long)gr * w + gc;
                abc[o] = a;
                abc[(long long)planes * hw + o] = b;
                abc[2 * (long long)planes * hw + o] = c;
            }
        }
        __syncthreads();  // sxy / hm are restaged for the next plane
    }
    double d0 = (double)l1, d1 = (double)ssum;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        d0 += __shfl_xor_sync(0xffffffffu, d0, o);
        d1 += __shfl_xor_sync(0xffffffffu, d1, o);
    }
    if ((threadIdx.x & 31) == 0) { wsum[threadIdx.x >> 5][0] = d0; wsum[threadIdx.x >> 5][1] = d1; }
    __syncthreads();
    if (threadIdx.x == 0) {
        double t0 = 0.0, t1 = 0.0;
        for (int i = 0; i < kLossThreads / 32; i++) { t0 += wsum[i][0]; t1 += wsum[i][1]; }
        atomicAdd(sums, t0);
        atomicAdd(sums + 1, t1);
    }
}

__global__ void __launch_bounds__(kLossThreads) ssim_bwd_kernel(int planes, int h, int w, PlaneView X, PlaneView Y,
                                                                 const float* __restrict__ abc,
                                                                 const float* __restrict__ coef, float* __restrict__ dx,
                                                                 long long dx_ps, long long dx_rs) {
    __shared__ float sm[3][kLossIn][kLossIn];
    __shared__ float hm[3][kLossIn][kLossTile];
    const int c0 = blockIdx.x * kLossTile, r0 = blockIdx.y * kLossTile;
    const int col = threadIdx.x & 31, row0 = (threadIdx.x >> 5) * kLossRows;
    const long long hw = (long long)h * w;
    const float k_l1 = __ldg(coef), k_ssim = __ldg(coef + 1);
    for (int p = blockIdx.z; p < planes; p += gridDim.z) {
        const PlaneView src[3] = {{abc, hw, w}, {abc + (long long)planes * hw, hw, w},
                                  {abc + 2 * (long long)planes * hw, hw, w}};
        stage_tile<3>(sm, src, p, h, w, r0, c0);
        __syncthreads();
        for (int i = threadIdx.x; i < kLossIn * kLossTile; i += kLossThreads) {
            const int r = i >> 5, c = i & 31;
            float ma = 0.f, mb = 0.f, mc = 0.f;
#pragma unroll
            for (int t = 0; t <= 2 * kLossHalo; t++) {
                const float g = kSsimTaps[t];
                ma = fmaf(g, sm[0][r][c + t], ma);
                mb = fmaf(g, sm[1][r][c + t], mb);
                mc = fmaf(g, sm[2][r][c + t], mc);
            }
            hm[0][r][c] = ma; hm[1][r][c] = mb; hm[2][r][c] = mc;
        }
        __syncthreads();
        float f[kLossRows][3];
        vertical_pass<3>(hm, col, row0, f);
        const int gc = c0 + col;
#pragma unroll
        for (int j = 0; j < kLossRows; j++) {
            const int gr = r0 + row0 + j;
            if (gr >= h || gc >= w) continue;
            const float x = X.at(p, gr, gc), y = Y.at(p, gr, gc);
            const float d = x - y;
            const float sgn = (float)((d > 0.f) - (d < 0.f));  // sign(0) = 0, as abs()'s backward
            const float dS = f[j][0] + 2.f * x * f[j][1] + y * f[j][2];
            dx[(long long)p * dx_ps + (long long)gr * dx_rs + gc] = fmaf(k_l1, sgn, k_ssim * dS);
        }
        __syncthreads();
    }
}

// Grid: 32x32 tiles in x/y, planes in z (looped beyond the 65535 limit of gridDim.z).
dim3 loss_grid(int planes, int h, int w) {
    return dim3((unsigned)((w + kLossTile - 1) / kLossTile), (unsigned)((h + kLossTile - 1) / kLossTile),
                (unsigned)(planes < 65535 ? planes : 65535));
}

// A plane of h rows, w pixels, unit pixel stride: rows must not overlap, and neither may planes (when there
// are several).  Returns an error message or nullptr.
const char* check_layout(int planes, int h, int w, long long ps, long long rs) {
    if (rs < (h > 1 ? (long long)w : 0) || rs < 0) return "row stride smaller than the row";
    if (planes > 1 && ps < (long long)(h - 1) * rs + w) return "plane stride smaller than the plane";
    return nullptr;
}

int check_sizes(const char* fn, int planes, int h, int w) {
    if (planes <= 0 || h <= 0 || w <= 0) {
        set_error("%s: need planes > 0, h > 0, w > 0 (got %d, %d, %d)", fn, planes, h, w);
        return SGB_E_INVALID;
    }
    if ((h + kLossTile - 1) / kLossTile > 65535) {
        set_error("%s: h = %d exceeds %d rows", fn, h, 65535 * kLossTile);
        return SGB_E_INVALID;
    }
    return SGB_OK;
}

int check_strides(const char* fn, const char* what, int planes, int h, int w, long long ps, long long rs) {
    if (const char* why = check_layout(planes, h, w, ps, rs)) {
        set_error("%s: %s: %s (plane stride %lld, row stride %lld, %d x %d)", fn, what, why, ps, rs, h, w);
        return SGB_E_INVALID;
    }
    return SGB_OK;
}

}  // namespace
}  // namespace sgb

using namespace sgb;

extern "C" {

int sgb_photometric_forward(int32_t planes, int32_t h, int32_t w, const float* x, int64_t x_plane_stride,
                            int64_t x_row_stride, const float* y, int64_t y_plane_stride, int64_t y_row_stride,
                            double* sums, float* partials, void* stream) {
    static const char* fn = "sgb_photometric_forward";
    int rc = check_sizes(fn, planes, h, w);
    if (rc) return rc;
    if (!x || !y || !sums) { set_error("%s: null x, y or sums", fn); return SGB_E_INVALID; }
    if ((rc = check_strides(fn, "x", planes, h, w, x_plane_stride, x_row_stride))) return rc;
    if ((rc = check_strides(fn, "y", planes, h, w, y_plane_stride, y_row_stride))) return rc;
    cudaStream_t s = (cudaStream_t)stream;
    SGB_CUDA(cudaMemsetAsync(sums, 0, 2 * sizeof(double), s));
    ssim_fwd_kernel<<<loss_grid(planes, h, w), kLossThreads, 0, s>>>(
        planes, h, w, PlaneView{x, x_plane_stride, x_row_stride}, PlaneView{y, y_plane_stride, y_row_stride}, sums,
        partials);
    SGB_LAUNCH_CHECK("ssim_fwd_kernel", 0, s);
    return SGB_OK;
}

int sgb_photometric_backward(int32_t planes, int32_t h, int32_t w, const float* x, int64_t x_plane_stride,
                             int64_t x_row_stride, const float* y, int64_t y_plane_stride, int64_t y_row_stride,
                             const float* partials, const float* coef, float* dL_dx, int64_t dx_plane_stride,
                             int64_t dx_row_stride, void* stream) {
    static const char* fn = "sgb_photometric_backward";
    int rc = check_sizes(fn, planes, h, w);
    if (rc) return rc;
    if (!x || !y || !partials || !coef || !dL_dx) {
        set_error("%s: null x, y, partials, coef or dL_dx", fn);
        return SGB_E_INVALID;
    }
    if ((rc = check_strides(fn, "x", planes, h, w, x_plane_stride, x_row_stride))) return rc;
    if ((rc = check_strides(fn, "y", planes, h, w, y_plane_stride, y_row_stride))) return rc;
    if ((rc = check_strides(fn, "dL_dx", planes, h, w, dx_plane_stride, dx_row_stride))) return rc;
    cudaStream_t s = (cudaStream_t)stream;
    ssim_bwd_kernel<<<loss_grid(planes, h, w), kLossThreads, 0, s>>>(
        planes, h, w, PlaneView{x, x_plane_stride, x_row_stride}, PlaneView{y, y_plane_stride, y_row_stride},
        partials, coef, dL_dx, dx_plane_stride, dx_row_stride);
    SGB_LAUNCH_CHECK("ssim_bwd_kernel", 0, s);
    return SGB_OK;
}

}  // extern "C"
