// 2D-feature -> 3D-Gaussian fusion.  Contract: PointCloudToImageMapper.compute_mapping
// (reference dataset/fusion_utils.py:30-78) and the per-view gather / accumulate / final divide of
// fusion.py:127-148.  The reference does this per view on the CPU in numpy — GPU->CPU copies of
// xyz, the view matrix and the rendered depth, a fancy-index gather of a (C,h,w) map for ALL P
// points, then a P x C host->device copy.  Here one view is: projection + visibility test on the
// device (float64 like numpy), a counting sort of the visible Gaussians by pixel, and one fused
// gather-accumulate kernel that reads the PLANAR (C,h,w) map directly: a warp takes 32 pixel-sorted
// Gaussians, so for every channel its 32 two-byte reads fall into a few neighbouring sectors of that
// channel plane, stages [32 Gaussians][128 channels] in shared memory and adds each row to the fp32
// sums as contiguous 128-byte pieces.  (Round 1 transposed the whole map to pixel-major first: 630 MB
// of traffic per view that the algorithm does not need — the map is now read at most once, and only
// where visible Gaussians land.)
//
// Numerics: projection in float64 with numpy's promotion rules (float32 inputs widened), pixel =
// round-half-to-even; the per-Gaussian sums add the views in call order in fp32 exactly like
// `_features_semantic[mask] += features_mapping[mask]`, so they are bit-identical to the reference.
#include <cub/cub.cuh>
#include <cuda_fp16.h>
#include "common.cuh"

namespace sgb {

namespace {

constexpr double kSurfaceInit = 999999.0;  // fusion_utils.py:58

struct Proj {
    double z;
    long long u, v;  // pi[0], pi[1]
    bool inside;
};

__device__ __forceinline__ long long round_to_ll(double r) {
    // np.round(...).astype(int): non-finite / out-of-range doubles become INT64_MIN on x86-64
    if (!(fabs(r) < 9.2e18)) return (long long)0x8000000000000000ull;
    return __double2ll_rn(r);  // round-half-to-even like np.round
}

__device__ __forceinline__ Proj project(const sgb_fusion_view& v, const float* __restrict__ w2c_t, int i) {
    // p = W2C @ [x,y,z,1] with W2C = world_to_camera.T (fusion_utils.py:42-45): p[k] = sum_j w2c_t[j][k]*c[j]
    const double x = (double)v.xyz[3 * (size_t)i], y = (double)v.xyz[3 * (size_t)i + 1],
                 z = (double)v.xyz[3 * (size_t)i + 2];
    double p[3];
#pragma unroll
    for (int k = 0; k < 3; k++)
        p[k] = (double)w2c_t[0 * 4 + k] * x + (double)w2c_t[1 * 4 + k] * y + (double)w2c_t[2 * 4 + k] * z +
               (double)w2c_t[3 * 4 + k];
    Proj r;
    r.z = p[2];
    const double pu = (p[0] * v.fx) / p[2] + v.cx;  // fusion_utils.py:46-47
    const double pv = (p[1] * v.fy) / p[2] + v.cy;
    r.u = round_to_ll(rint(pu));
    r.v = round_to_ll(rint(pv));
    r.inside = (r.u >= v.cut_bound) && (r.v >= v.cut_bound) && (r.u < v.w - v.cut_bound) &&
               (r.v < v.h - v.cut_bound);  // fusion_utils.py:50-55
    return r;
}

__global__ void surface_init_kernel(int n, double* zbuf) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) zbuf[i] = kSurfaceInit;
}

// fusion_utils.py:57-61: z-buffer of the points themselves (min over p.z > 0.2 inside the image)
__global__ void surface_zbuf_kernel(sgb_fusion_view v, double* zbuf) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= v.P) return;
    Proj p = project(v, v.world_to_camera, i);
    if (p.z > 0.2 && p.inside) {
        // positive doubles order like their bit patterns
        atomicMin(reinterpret_cast<unsigned long long*>(zbuf + p.v * v.w + p.u),
                  (unsigned long long)__double_as_longlong(p.z));
    }
}

// Visibility of Gaussian i in this view -> linear pixel index v*w+u, or -1.
__device__ __forceinline__ int visible_pixel(const sgb_fusion_view& v, const double* zbuf, int i, Proj& p) {
    p = project(v, v.world_to_camera, i);
    bool vis = p.inside;
    if (vis) {
        if (v.depth_mode == SGB_DEPTH_NONE) {
            vis = p.z > 0;  // fusion_utils.py:70-72
        } else {
            double dcur, thr;
            const size_t o = (size_t)p.v * v.w + p.u;
            if (v.depth_mode == SGB_DEPTH_F32) {
                const float df = static_cast<const float*>(v.depth)[o];
                dcur = (double)df;
                thr = (double)((float)v.vis_thres * df);  // python float * float32 array -> float32
            } else {
                dcur = v.depth_mode == SGB_DEPTH_F64 ? static_cast<const double*>(v.depth)[o] : zbuf[o];
                thr = v.vis_thres * dcur;
            }
            vis = fabs(dcur - p.z) <= thr;  // fusion_utils.py:63-69
        }
    }
    return vis ? (int)(p.v * v.w + p.u) : -1;
}

__global__ void fusion_map_kernel(sgb_fusion_view v, const double* zbuf, long long* __restrict__ mapping) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= v.P) return;
    Proj p;
    const int pix = visible_pixel(v, zbuf, i, p);
    mapping[3 * (size_t)i + 0] = pix >= 0 ? p.v : 0;  // fusion_utils.py:73-75
    mapping[3 * (size_t)i + 1] = pix >= 0 ? p.u : 0;
    mapping[3 * (size_t)i + 2] = pix >= 0 ? 1 : 0;
}

// Visibility of every Gaussian in this view; count += 1 for the visible ones (fusion.py:143); per-pixel histogram of
// the visible Gaussians (input of the counting sort).
__global__ void fusion_pix_kernel(sgb_fusion_view v, const double* zbuf, int* __restrict__ pix_of,
                                  float* __restrict__ count, int* __restrict__ n_visible,
                                  uint32_t* __restrict__ hist) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    int pix = -1;
    if (i < v.P) {
        Proj p;
        pix = visible_pixel(v, zbuf, i, p);
        pix_of[i] = pix;
        if (pix >= 0) {
            count[i] += 1.0f;  // gaussians._times[mask] += 1, fusion.py:143
            atomicAdd(hist + pix, 1u);
        }
    }
    if (n_visible) {
        unsigned m = __ballot_sync(0xffffffffu, pix >= 0);
        if ((threadIdx.x & 31) == 0 && m) atomicAdd(n_visible, __popc(m));
    }
}

// Counting sort, scatter step: `cursor` holds the exclusive scan of the histogram and is advanced atomically.  The
// order inside a pixel is arbitrary — every Gaussian owns its own accumulator row.
__global__ void fusion_scatter_kernel(int P, const int* __restrict__ pix_of, uint32_t* __restrict__ cursor,
                                      uint32_t* __restrict__ sorted_ids, uint32_t* __restrict__ sorted_pix) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= P) return;
    const int pix = pix_of[i];
    if (pix < 0) return;
    const uint32_t pos = atomicAdd(cursor + pix, 1u);
    sorted_ids[pos] = (uint32_t)i;
    sorted_pix[pos] = (uint32_t)pix;
}

__device__ __forceinline__ float to_f32(__half h) { return __half2float(h); }
__device__ __forceinline__ float to_f32(float f) { return f; }

// feat_sum[g, :] += map[:, pix(g)] for the visible Gaussians, in pixel order.  Work item of a warp = (32 consecutive
// entries of the pixel-sorted list, one pass of CHP channels); items are handed out grid-stride with the pass index
// fastest, so a view with few visible Gaussians still spreads over many warps (a first version walked all passes of a
// batch in one warp: serial latency per view however few Gaussians were visible).  Per item: load phase
// (lane = Gaussian, one element per channel plane, 16 loads in flight) into a private shared-memory tile [32][CHP]
// (odd word pitch: the per-lane row writes and the per-row reads are both conflict-free), then the accumulate phase
// adds 16 rows at a time to the fp32 sums, lanes along the channels (128-byte pieces, 32 loads in flight).
template <typename T, int CHP>
__global__ void __launch_bounds__(256) fusion_gather_sorted_kernel(const int* __restrict__ n_visible, int C, int npix,
                                                                   const uint32_t* __restrict__ sorted_ids,
                                                                   const uint32_t* __restrict__ sorted_pix,
                                                                   const T* __restrict__ fm,
                                                                   float* __restrict__ feat_sum) {
    constexpr int PITCH = CHP + (sizeof(T) == 2 ? 2 : 1);  // elements; 65 32-bit words either way
    constexpr int KP = CHP / 32;
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    T* tile = reinterpret_cast<T*>(smem_raw) + (size_t)warp * 32 * PITCH;
    const int nvis = *n_visible;
    const int npass = (C + CHP - 1) / CHP;
    const long long items = (long long)((nvis + 31) / 32) * npass;
    const int warps_total = (gridDim.x * blockDim.x) >> 5;
    for (long long it = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; it < items; it += warps_total) {
        const int b = (int)(it / npass), c0 = (int)(it % npass) * CHP;
        const int nc = min(CHP, C - c0);
        const int j = b * 32 + lane;
        const bool valid = j < nvis;
        const uint32_t gid = valid ? sorted_ids[j] : 0u;
        uint32_t pix = valid ? sorted_pix[j] : 0u;
        const uint32_t pix0 = __shfl_sync(0xffffffffu, pix, 0);  // executed by every lane (lane 0 is always valid)
        pix = valid ? pix : pix0;                                // idle lanes re-read lane 0's pixel (in range, cached)
        const int nrows = min(32, nvis - b * 32);
        const T* src = fm + (size_t)c0 * npix + pix;
        // load phase
#pragma unroll 16
        for (int c = 0; c < CHP; c++)
            if (c < nc) tile[lane * PITCH + c] = src[(size_t)c * npix];
        __syncwarp();
        // accumulate phase
        constexpr int RGRP = KP > 2 ? 8 : 16;   // rows per group: 32 loads in flight per lane
        for (int g0 = 0; g0 < nrows; g0 += RGRP) {
            float v[RGRP][KP];
            float* dst[RGRP];
#pragma unroll
            for (int u = 0; u < RGRP; u++) {
                const uint32_t gg = __shfl_sync(0xffffffffu, gid, (g0 + u) & 31);
                dst[u] = feat_sum + (size_t)gg * C + c0;
#pragma unroll
                for (int k = 0; k < KP; k++) {
                    const int c = lane + 32 * k;
                    v[u][k] = (g0 + u < nrows && c < nc) ? dst[u][c] : 0.f;
                }
            }
#pragma unroll
            for (int u = 0; u < RGRP; u++)
#pragma unroll
                for (int k = 0; k < KP; k++) {
                    const int c = lane + 32 * k;
                    if (g0 + u < nrows && c < nc) dst[u][c] = v[u][k] + to_f32(tile[(g0 + u) * PITCH + c]);
                }
        }
        __syncwarp();
    }
}

// fusion.py:146-147
__global__ void fusion_normalize_kernel(int P, int C, float* __restrict__ feat_sum, float* __restrict__ count) {
    const size_t n = (size_t)P * C;
    for (size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += (size_t)gridDim.x * blockDim.x) {
        const size_t g = e / C;
        float t = count[g];
        if (t == 0.f) t = 1e-5f;
        feat_sum[e] = feat_sum[e] / t;
    }
}
__global__ void fusion_fix_count_kernel(int P, float* __restrict__ count) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < P && count[i] == 0.f) count[i] = 1e-5f;
}

int prepare_zbuf(sgb_ctx* ctx, const sgb_fusion_view& v, size_t extra, double** zbuf, char** extra_ptr,
                 cudaStream_t s) {
    const size_t npix = (size_t)v.w * v.h;
    const size_t zb = (v.depth_mode == SGB_DEPTH_SURFACE) ? align_up(npix * sizeof(double)) : 0;
    int rc = ctx->misc.ensure(zb + extra + 256);
    if (rc) return rc;
    *zbuf = zb ? (double*)ctx->misc.p : nullptr;
    *extra_ptr = (char*)ctx->misc.p + zb;
    if (zb) {
        surface_init_kernel<<<(unsigned)((npix + 255) / 256), 256, 0, s>>>((int)npix, *zbuf);
        surface_zbuf_kernel<<<(v.P + 255) / 256, 256, 0, s>>>(v, *zbuf);
        SGB_LAUNCH_CHECK("surface_zbuf_kernel", 0, s);
    }
    return SGB_OK;
}

int check_view(const sgb_fusion_view* v) {
    if (!v || v->P < 0 || (v->P > 0 && !v->xyz) || !v->world_to_camera || v->w <= 0 || v->h <= 0) {
        set_error("fusion view: null pointer or non-positive size");
        return SGB_E_INVALID;
    }
    if ((v->depth_mode == SGB_DEPTH_F32 || v->depth_mode == SGB_DEPTH_F64) && !v->depth) {
        set_error("fusion view: depth_mode needs a depth map");
        return SGB_E_INVALID;
    }
    if (v->depth_mode < 0 || v->depth_mode > 3) {
        set_error("fusion view: unknown depth_mode %d", v->depth_mode);
        return SGB_E_INVALID;
    }
    return SGB_OK;
}

}  // namespace
}  // namespace sgb

using namespace sgb;

extern "C" int sgb_fusion_map(sgb_ctx* ctx, const sgb_fusion_view* v, int64_t* mapping, void* stream) {
    cudaStream_t s = (cudaStream_t)stream;
    int rc = check_view(v);
    if (rc) return rc;
    if (v->P == 0) return SGB_OK;
    if (!ctx || !mapping) { set_error("sgb_fusion_map: null ctx/mapping"); return SGB_E_INVALID; }
    double* zbuf; char* extra;
    rc = prepare_zbuf(ctx, *v, 0, &zbuf, &extra, s);
    if (rc) return rc;
    fusion_map_kernel<<<(v->P + 255) / 256, 256, 0, s>>>(*v, zbuf, (long long*)mapping);
    SGB_LAUNCH_CHECK("fusion_map_kernel", 0, s);
    return SGB_OK;
}

extern "C" int sgb_fusion_accumulate(sgb_ctx* ctx, const sgb_fusion_view* v, const void* features, int32_t C,
                                     int32_t feat_dtype, float* feat_sum, float* count, int32_t* n_visible_dev,
                                     void* stream) {
    cudaStream_t s = (cudaStream_t)stream;
    int rc = check_view(v);
    if (rc) return rc;
    if (!ctx || !features || !feat_sum || !count || C <= 0 || (feat_dtype != SGB_FEAT_F16 && feat_dtype != SGB_FEAT_F32)) {
        set_error("sgb_fusion_accumulate: bad arguments");
        return SGB_E_INVALID;
    }
    if (n_visible_dev) SGB_CUDA(cudaMemsetAsync(n_visible_dev, 0, sizeof(int32_t), s));
    if (v->P == 0) return SGB_OK;
    const size_t npix = (size_t)v->w * v->h;
    // scratch: pix_of [P] | sorted ids [P] | sorted pix [P] | histogram / cursor [npix] | n_visible | cub temp
    size_t scan_tmp = 0;
    cub::DeviceScan::ExclusiveSum(nullptr, scan_tmp, (uint32_t*)nullptr, (uint32_t*)nullptr, (int)npix, s);
    const size_t parr = align_up(sizeof(int) * (size_t)v->P), harr = align_up(sizeof(uint32_t) * npix);
    double* zbuf; char* extra;
    rc = prepare_zbuf(ctx, *v, 3 * parr + 2 * harr + 256 + align_up(scan_tmp), &zbuf, &extra, s);
    if (rc) return rc;
    int* pix_of = (int*)extra;
    uint32_t* sorted_ids = (uint32_t*)(extra + parr);
    uint32_t* sorted_pix = (uint32_t*)(extra + 2 * parr);
    uint32_t* hist = (uint32_t*)(extra + 3 * parr);
    uint32_t* cursor = (uint32_t*)(extra + 3 * parr + harr);
    int* nvis_own = (int*)(extra + 3 * parr + 2 * harr);
    void* cub_tmp = extra + 3 * parr + 2 * harr + 256;
    int* nvis = n_visible_dev ? n_visible_dev : nvis_own;
    if (!n_visible_dev) SGB_CUDA(cudaMemsetAsync(nvis_own, 0, sizeof(int), s));
    {
        StageTimer t(ctx, ST_FUSION_PROJECT, s);
        SGB_CUDA(cudaMemsetAsync(hist, 0, sizeof(uint32_t) * npix, s));
        fusion_pix_kernel<<<(v->P + 255) / 256, 256, 0, s>>>(*v, zbuf, pix_of, count, nvis, hist);
        SGB_LAUNCH_CHECK("fusion_pix_kernel", 0, s);
    }
    {
        StageTimer t(ctx, ST_FUSION_SORT, s);
        SGB_CUDA(cub::DeviceScan::ExclusiveSum(cub_tmp, scan_tmp, hist, cursor, (int)npix, s));
        fusion_scatter_kernel<<<(v->P + 255) / 256, 256, 0, s>>>(v->P, pix_of, cursor, sorted_ids, sorted_pix);
        SGB_LAUNCH_CHECK("fusion_scatter_kernel", 0, s);
        ctx->lib_launches += 1;
    }
    {
        StageTimer t(ctx, ST_FUSION_GATHER, s);
        const int gblocks = kNumSMs * 3;  // 3 CTAs/SM by shared memory (66 KB each); items are handed out grid-stride
        if (feat_dtype == SGB_FEAT_F16) {
            constexpr int CHP = 128;  // channels per pass
            const size_t smem = 8 * 32 * (CHP + 2) * sizeof(__half);
            static DeviceOnce once;
            if (once.first_use_on_device())
                SGB_CUDA(cudaFuncSetAttribute(fusion_gather_sorted_kernel<__half, CHP>,
                                              cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
            fusion_gather_sorted_kernel<__half, CHP><<<gblocks, 256, smem, s>>>(nvis, C, (int)npix, sorted_ids, sorted_pix,
                                                                               (const __half*)features, feat_sum);
        } else {
            constexpr int CHP = 64;
            const size_t smem = 8 * 32 * (CHP + 1) * sizeof(float);
            static DeviceOnce once;
            if (once.first_use_on_device())
                SGB_CUDA(cudaFuncSetAttribute(fusion_gather_sorted_kernel<float, CHP>,
                                              cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
            fusion_gather_sorted_kernel<float, CHP><<<gblocks, 256, smem, s>>>(nvis, C, (int)npix, sorted_ids, sorted_pix,
                                                                              (const float*)features, feat_sum);
        }
        SGB_LAUNCH_CHECK("fusion_gather_sorted_kernel", 0, s);
    }
    ctx->launches += 3;
    return SGB_OK;
}

extern "C" int sgb_fusion_normalize(int32_t P, int32_t C, float* feat_sum, float* count, void* stream) {
    cudaStream_t s = (cudaStream_t)stream;
    if (P < 0 || C <= 0 || !feat_sum || !count) { set_error("sgb_fusion_normalize: bad arguments"); return SGB_E_INVALID; }
    if (P == 0) return SGB_OK;
    fusion_normalize_kernel<<<kNumSMs * 8, 256, 0, s>>>(P, C, feat_sum, count);
    fusion_fix_count_kernel<<<(P + 255) / 256, 256, 0, s>>>(P, count);
    SGB_LAUNCH_CHECK("fusion_normalize_kernel", 0, s);
    return SGB_OK;
}
