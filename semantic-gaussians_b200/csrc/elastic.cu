// Elastic distortion of a point cloud: the per-point half of dataset/augmentation.py ElasticDistortion, that is
//
//   interp = RegularGridInterpolator(ax, noise, bounds_error=0, fill_value=0)      (scipy, method "linear")
//   out    = coords + interp(coords) * magnitude
//
// for a small (nx, ny, nz, 3) fp32 noise grid on ascending fp64 axes.  The noise itself (np.random.randn and the
// scipy.ndimage box filters) stays on the host, so a seeded run draws what the reference draws.  The lookup is
// restated as scipy 1.18 evaluates it (_rgi.py _evaluate_linear over _rgi_cython.find_indices), in fp64 with every
// product and sum rounded alone:
//   - per axis the cell i with g[i] <= x < g[i+1] (the last cell when x == g[n-1]),
//     t = (x - g[i]) / (g[i+1] - g[i]);
//   - the 8 corners in itertools.product order (axis 0 slowest; the lower corner pairs with 1 - t, the upper with t),
//     weight ((1 * w0) * w1) * w2, value = ((0 + v_0 w_0) + v_1 w_1) + ... + v_7 w_7;
//   - a point below g[0] or above g[n-1] on any axis gets 0; a point with a NaN coordinate gets NaN.
// Thread = one point.  The grid is a few thousand entries and stays in L1 / L2.
#include "common.cuh"

namespace sgb {
namespace {

constexpr int kElThreads = 256;

// find_interval_ascending of scipy's _rgi_cython for a value inside [g[0], g[n-1]]: the largest i <= n - 2 with
// g[i] <= x.  For a strictly ascending axis that is the unique cell the binary search there lands in.
__device__ __forceinline__ int el_cell(const double* __restrict__ g, int n, double x) {
    int lo = 0, hi = n - 2;
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (g[mid] <= x) lo = mid;
        else hi = mid - 1;
    }
    return lo;
}

template <typename Coord>
__global__ void __launch_bounds__(kElThreads) elastic_displace_kernel(long long P, const Coord* xyz,
                                                                      const float* __restrict__ grid, int nx, int ny,
                                                                      int nz, const double* __restrict__ axes,
                                                                      double magnitude, double* out) {
    const long long p = (long long)blockIdx.x * kElThreads + threadIdx.x;
    if (p >= P) return;
    const double x[3] = {(double)xyz[3 * p], (double)xyz[3 * p + 1], (double)xyz[3 * p + 2]};
    const int n[3] = {nx, ny, nz};
    const double* g[3] = {axes, axes + nx, axes + nx + ny};
    bool nan = false, outside = false;
    int cell[3];
    double t[3];
#pragma unroll
    for (int a = 0; a < 3; a++) {
        nan |= isnan(x[a]);
        outside |= x[a] < g[a][0] || x[a] > g[a][n[a] - 1];
        cell[a] = 0;
        t[a] = 0.0;
    }
    double v[3] = {0.0, 0.0, 0.0};
    if (!nan && !outside) {
#pragma unroll
        for (int a = 0; a < 3; a++) {
            cell[a] = el_cell(g[a], n[a], x[a]);
            t[a] = __ddiv_rn(__dsub_rn(x[a], g[a][cell[a]]), __dsub_rn(g[a][cell[a] + 1], g[a][cell[a]]));
        }
        const double u[3] = {__dsub_rn(1.0, t[0]), __dsub_rn(1.0, t[1]), __dsub_rn(1.0, t[2])};
#pragma unroll
        for (int c = 0; c < 8; c++) {
            const int b0 = (c >> 2) & 1, b1 = (c >> 1) & 1, b2 = c & 1;
            double w = __dmul_rn(1.0, b0 ? t[0] : u[0]);
            w = __dmul_rn(w, b1 ? t[1] : u[1]);
            w = __dmul_rn(w, b2 ? t[2] : u[2]);
            const float* e = grid + 3 * (((long long)(cell[0] + b0) * ny + (cell[1] + b1)) * nz + (cell[2] + b2));
#pragma unroll
            for (int k = 0; k < 3; k++) v[k] = __dadd_rn(v[k], __dmul_rn((double)__ldg(e + k), w));
        }
    }
#pragma unroll
    for (int k = 0; k < 3; k++) {
        const double r = nan ? __longlong_as_double(0x7ff8000000000000ll) : v[k];
        out[3 * p + k] = __dadd_rn(x[k], __dmul_rn(r, magnitude));
    }
}

}  // namespace
}  // namespace sgb

using namespace sgb;

extern "C" {

int sgb_elastic_displace(int64_t P, const void* xyz, int32_t xyz_is_f64, const float* grid, int32_t nx, int32_t ny,
                         int32_t nz, const double* axes, double magnitude, double* out, void* stream) {
    static const char* fn = "sgb_elastic_displace";
    if (P <= 0 || P > INT32_MAX) {
        set_error("%s: P = %lld outside [1, %d]", fn, (long long)P, INT32_MAX);
        return SGB_E_INVALID;
    }
    if (xyz_is_f64 != 0 && xyz_is_f64 != 1) { set_error("%s: xyz_is_f64 = %d (0 or 1)", fn, xyz_is_f64); return SGB_E_INVALID; }
    if (nx < 2 || ny < 2 || nz < 2) {
        set_error("%s: grid %d x %d x %d needs at least 2 nodes per axis", fn, nx, ny, nz);
        return SGB_E_INVALID;
    }
    if ((long long)nx * ny * nz * 3 > INT32_MAX) {
        set_error("%s: grid %d x %d x %d x 3 exceeds %d entries", fn, nx, ny, nz, INT32_MAX);
        return SGB_E_INVALID;
    }
    if (!xyz || !grid || !axes || !out) { set_error("%s: null xyz / grid / axes / out", fn); return SGB_E_INVALID; }
    if (!xyz_is_f64 && (const void*)out == xyz) {
        set_error("%s: out may alias xyz only when xyz is float64", fn);
        return SGB_E_INVALID;
    }
    cudaStream_t s = (cudaStream_t)stream;
    const unsigned blocks = (unsigned)((P + kElThreads - 1) / kElThreads);
    if (xyz_is_f64)
        elastic_displace_kernel<double><<<blocks, kElThreads, 0, s>>>(P, (const double*)xyz, grid, nx, ny, nz, axes,
                                                                      magnitude, out);
    else
        elastic_displace_kernel<float><<<blocks, kElThreads, 0, s>>>(P, (const float*)xyz, grid, nx, ny, nz, axes,
                                                                     magnitude, out);
    SGB_LAUNCH_CHECK("elastic_displace_kernel", 0, s);
    return SGB_OK;
}

}  // extern "C"
