// sgb200 internal header: state layouts, error handling, small device helpers.
#pragma once
#include <cstdint>
#include <cstdio>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include "../../include/sgb200.h"

#define SGB_TILE_PIX (SGB_TILE * SGB_TILE)

namespace sgb {

// ------------------------------------------------------------------ errors
void set_error(const char* fmt, ...);
int cuda_fail(cudaError_t e, const char* what);
#define SGB_CUDA(call)                                            \
    do {                                                          \
        cudaError_t e__ = (call);                                 \
        if (e__ != cudaSuccess) return sgb::cuda_fail(e__, #call); \
    } while (0)
#define SGB_LAUNCH_CHECK(what, dbg, stream)                                   \
    do {                                                                      \
        cudaError_t e__ = cudaGetLastError();                                 \
        if (e__ == cudaSuccess && (dbg)) e__ = cudaStreamSynchronize(stream); \
        if (e__ != cudaSuccess) return sgb::cuda_fail(e__, what);             \
    } while (0)

// ------------------------------------------------------------------ opaque state layouts
// One 32-byte record per Gaussian: everything the blend needs, one DRAM sector per gather
// (the reference gathers means2D 8 B + conic_opacity 16 B [+ depth 4 B] from three arrays,
// forward.cu:318-321).
struct __align__(16) SplatRec {
    float mx, my;          // pixel-space mean            (GeometryState::means2D)
    float depth;           // view-space z                (GeometryState::depths)
    float pad;
    float cx, cy, cz, op;  // conic (a,b,c) and opacity   (GeometryState::conic_opacity)
};
static_assert(sizeof(SplatRec) == 32, "SplatRec must be 32 bytes");

static inline size_t align_up(size_t x, size_t a = 256) { return (x + a - 1) / a * a; }

struct GeomView {  // carved out of geometry_state (caller-owned, P-sized)
    SplatRec* rec;
    float* cov3D;            // [P,6]
    float* rgb;              // [P,3]   SH path only
    uint8_t* clamped;        // [P,3]
    uint32_t* tiles_touched; // [P]
    uint32_t* perm;          // [P] Gaussian ids in (depth bits, id) order
    uint32_t* offsets;       // [P] inclusive scan of tiles_touched in that order (GeometryState::point_offsets)
    size_t bytes;
    static GeomView carve(void* base, int64_t P) {
        GeomView g;
        char* p = (char*)base;
        size_t off = 0;
        g.rec = (SplatRec*)(p + off); off += align_up(sizeof(SplatRec) * P);
        g.cov3D = (float*)(p + off); off += align_up(sizeof(float) * 6 * P);
        g.rgb = (float*)(p + off); off += align_up(sizeof(float) * 3 * P);
        g.clamped = (uint8_t*)(p + off); off += align_up(3 * (size_t)P);
        g.tiles_touched = (uint32_t*)(p + off); off += align_up(sizeof(uint32_t) * P);
        g.perm = (uint32_t*)(p + off); off += align_up(sizeof(uint32_t) * P);
        g.offsets = (uint32_t*)(p + off); off += align_up(sizeof(uint32_t) * P);
        g.bytes = off;
        return g;
    }
};

struct BinView {  // carved out of binning_state (R-sized)
    uint32_t* point_list;  // [R] Gaussian ids, sorted by (tile, depth bits, id)
    size_t bytes;
    static BinView carve(void* base, int64_t R) {
        BinView b;
        b.point_list = (uint32_t*)base;
        b.bytes = align_up(sizeof(uint32_t) * (size_t)(R > 0 ? R : 1));
        return b;
    }
};

struct ImgView {  // carved out of image_state
    float* final_T;        // [H*W]   ImageState::accum_alpha
    uint32_t* n_contrib;   // [H*W]
    uint2* ranges;         // [tiles]
    uint32_t* tile_last;   // [tiles] max n_contrib inside the tile (backward start point)
    size_t bytes;
    static ImgView carve(void* base, int W, int H) {
        ImgView v;
        char* p = (char*)base;
        size_t N = (size_t)W * H;
        size_t tiles = (size_t)((W + SGB_TILE - 1) / SGB_TILE) * ((H + SGB_TILE - 1) / SGB_TILE);
        size_t off = 0;
        v.final_T = (float*)(p + off); off += align_up(4 * N);
        v.n_contrib = (uint32_t*)(p + off); off += align_up(4 * N);
        v.ranges = (uint2*)(p + off); off += align_up(8 * tiles);
        v.tile_last = (uint32_t*)(p + off); off += align_up(4 * tiles);
        v.bytes = off;
        return v;
    }
};

// `in` with the camera of `cam`: the views of a batched call share every other input.
static inline sgb_view_inputs with_camera(const sgb_view_inputs& in, const sgb_camera& cam) {
    sgb_view_inputs o = in;
    o.viewmatrix = cam.viewmatrix;
    o.projmatrix = cam.projmatrix;
    o.campos = cam.campos;
    o.tan_fovx = cam.tan_fovx;
    o.tan_fovy = cam.tan_fovy;
    return o;
}

struct ViewState {  // one view of a render or backward call: its inputs, instance count and carved states
    sgb_view_inputs in;
    int64_t R;
    GeomView g;
    BinView b;
    ImgView im;
    const float* colors;
    static ViewState carve(const sgb_view_inputs& shared, const sgb_camera& cam, int64_t num_rendered,
                           const void* geometry_state, const void* binning_state, const void* image_state) {
        ViewState w;
        w.in = with_camera(shared, cam);
        w.R = w.in.P > 0 ? num_rendered : 0;
        w.g = GeomView::carve(const_cast<void*>(geometry_state), w.in.P > 0 ? w.in.P : 1);
        w.b = BinView::carve(const_cast<void*>(binning_state), w.R);
        w.im = ImgView::carve(const_cast<void*>(image_state), w.in.W, w.in.H);
        w.colors = w.in.colors_precomp ? w.in.colors_precomp : w.g.rgb;  // rasterizer_impl.cu:324
        return w;
    }
};

// ------------------------------------------------------------------ scratch context
struct Scratch {
    void* p = nullptr;
    size_t cap = 0;
    int ensure(size_t n);  // grows (cudaFree + cudaMalloc); returns SGB_OK / SGB_E_NOMEM
};

// ------------------------------------------------------------------ stage tracing
// Built-in stage tracing (the reference has none; its only timing hook is train.py's per-iteration
// event pair).  When enabled, every stage is bracketed by a CUDA event pair recorded on the
// caller's stream; sgb_profile_read() sums the pairs recorded since the last read.
enum Stage {
    ST_PREPROCESS = 0, ST_DEPTH_SORT, ST_SCAN, ST_EMIT, ST_TILE_SORT, ST_RANGES, ST_BLEND_FWD,
    ST_BLEND_BWD, ST_GEOM_BWD, ST_FUSION_PROJECT, ST_FUSION_SORT, ST_FUSION_GATHER, ST_ALPHA, ST_DFEATURE,
    ST_WEIGHT_SUM, ST_COUNT
};
constexpr int kProfRing = 320;
struct Profiler {
    bool on = false;
    cudaEvent_t ev[ST_COUNT][kProfRing][2];
    int n[ST_COUNT];
    bool created = false;
};

constexpr int kNumSMs = 132;  // H100 SXM: sizes the grids of the grid-stride kernels

struct WeightPools;  // weight_pool.cuh
struct Readback;
}  // namespace sgb

struct sgb_ctx {
    int device = 0;
    sgb::Profiler prof;
    uint64_t launches = 0;       // kernels of this library launched through this ctx
    uint64_t lib_launches = 0;   // CUB device-wide calls (each several kernels)
    sgb::Scratch geom;     // depth-sort keys, iota values, CUB temp, 64-bit instance total (shared by a batch's views)
    sgb::Scratch bin;      // unsorted / sorted tile keys, unsorted values, CUB temp
    sgb::Scratch misc;     // fusion: pixel-sorted visible list, z-buffer
    sgb::Scratch work;     // work-item counter of the persistent kernels (chn_forward.cu, chn_dfeature.cu)
    sgb::Scratch depth_grad;  // [P] dL/d(view-space z) of the view being differentiated (expected-depth backward)
    sgb::Scratch cam_partial; // per-CTA fp64 camera-gradient partials of the view being differentiated
    sgb::Scratch lift_state;  // sgb_lift_batch: geometry state, radii and image state of every view of the call
    sgb::Scratch lift_bin;    // sgb_lift_batch: binning states of the views
    // What the ctx carries from one call to the next: the weight rows of the C-channel blend, one pool per view of a
    // batch.  Owned; its layout is the weight-pool module's (weight_pool.cuh).
    sgb::WeightPools* pools = nullptr;
    sgb::Readback* pinned = nullptr;  // host-pinned readback buffer (weight_pool.cuh)
    cudaEvent_t feature_grad_event = nullptr;  // caller-owned; recorded when dL_dcolors is final (sgb200.h)
};

namespace sgb {

struct StageTimer {  // RAII event pair around one stage
    sgb_ctx* c; int st; cudaStream_t s; int slot;
    StageTimer(sgb_ctx* ctx, int stage, cudaStream_t stream) : c(ctx), st(stage), s(stream), slot(-1) {
        if (c && c->prof.on && c->prof.n[st] < kProfRing) {
            slot = c->prof.n[st]++;
            cudaEventRecord(c->prof.ev[st][slot][0], s);
        }
    }
    ~StageTimer() {
        if (slot >= 0) cudaEventRecord(c->prof.ev[st][slot][1], s);
    }
};

// cudaFuncSetAttribute is per device: a process-wide "done" flag would leave the second device of a
// single-process multi-GPU caller without its opt-in shared-memory size.  Returns true the first time it is
// called with this flag array on the current device.
struct DeviceOnce {
    bool done[64] = {};
    bool first_use_on_device() {
        int dev = 0;
        cudaGetDevice(&dev);
        if (dev < 0 || dev >= 64) return true;
        if (done[dev]) return false;
        done[dev] = true;
        return true;
    }
};

// ------------------------------------------------------------------ stage launchers
int launch_preprocess(const sgb_view_inputs& in, GeomView g, int32_t* radii, uint32_t* depth_keys,
                      cudaStream_t s);
int launch_mark_visible(int P, const float* means3D, const float* view, uint8_t* present, cudaStream_t s);
// Depth order + scan of V views of the same Gaussians (cams[v] replaces the camera fields of `in`) into each view's
// geometry state: everything is enqueued back to back, ONE stream sync reads all R.
int run_depth_order_and_scan(sgb_ctx* ctx, const sgb_view_inputs& in, int V, const sgb_camera* cams,
                             void* const* geometry_states, int32_t* const* radii, int64_t* R_host, cudaStream_t s);
int reserve_binning(sgb_ctx* ctx, const sgb_view_inputs& in, int64_t R, cudaStream_t s);
int run_binning(sgb_ctx* ctx, const sgb_view_inputs& in, int64_t R, GeomView g, BinView b, ImgView im,
                const int32_t* radii, cudaStream_t s);
// C <= 4 blend.  out_exp_depth / out_alpha (given together or not at all): expected depth and accumulated opacity.
// dL_ddepth non-null selects the backward with those two extra channels (either upstream plane may be null = zero);
// it accumulates dL/dz per Gaussian into dL_ddepth, which the caller zeroes and passes on to launch_geom_backward.
int launch_blend_forward(const sgb_view_inputs& in, GeomView g, BinView b, ImgView im, const float* colors,
                         float* out_color, float* out_depth, float* out_exp_depth, float* out_alpha, cudaStream_t s);
int launch_blend_backward(const sgb_view_inputs& in, GeomView g, BinView b, ImgView im, const float* colors,
                          const float* dL_dpix, float* dL_dmean2D, float* dL_dconic, float* dL_dopacity,
                          float* dL_dcolors, const float* dL_dexp_depth, const float* dL_dalpha, float* dL_ddepth,
                          cudaStream_t s);
// C > 4 blend: weight_pool.cuh (the alpha pass and the pools it fills) and chn_blend.cuh (the contraction stages).
// cam_grads non-NULL: also this view's camera gradient (sgb200.h sgb_camera_grads), through cam_partial, a device
// buffer of camera_grad_partial_bytes(in.P) that the call's two kernels use in stream order.
int launch_geom_backward(const sgb_view_inputs& in, GeomView g, const int32_t* radii, const float* cov3D,
                         const float* dL_dcolor_rgb, const sgb_view_grads& gr, const float* dL_ddepth,
                         const sgb_camera_grads* cam_grads, double* cam_partial, cudaStream_t s);
size_t camera_grad_partial_bytes(int32_t P);

// ------------------------------------------------------------------ device helpers
#ifdef __CUDACC__
// d.xy = a.xy * b.xy + c.xy as two round-to-nearest FMAs (sm_90 has no packed fp32 FMA).
__device__ __forceinline__ float2 ffma2(float2 a, float2 b, float2 c) {
    return make_float2(fmaf(a.x, b.x, c.x), fmaf(a.y, b.y, c.y));
}
// auxiliary.h:46-56 (getRect).  max_radius is an int parameter: the float radius is converted at
// the call.  Used by preprocess and re-derived by the instance emitter exactly like
// duplicateWithKeys does (rasterizer_impl.cu:91).
__device__ __forceinline__ void get_rect(const float2 p, int max_radius, uint2& rect_min, uint2& rect_max,
                                         dim3 grid) {
    rect_min = {min(grid.x, max((int)0, (int)((p.x - max_radius) / SGB_TILE))),
                min(grid.y, max((int)0, (int)((p.y - max_radius) / SGB_TILE)))};
    rect_max = {min(grid.x, max((int)0, (int)((p.x + max_radius + SGB_TILE - 1) / SGB_TILE))),
                min(grid.y, max((int)0, (int)((p.y + max_radius + SGB_TILE - 1) / SGB_TILE)))};
}
__device__ __forceinline__ float4 ldg_nc_f4(const float* p) {
    return __ldg(reinterpret_cast<const float4*>(p));
}
__device__ __forceinline__ void red_add_f32(float* addr, float v) {
    asm volatile("red.global.add.f32 [%0], %1;" ::"l"(addr), "f"(v) : "memory");
}
__device__ __forceinline__ void red_add_v4_f32(float* addr, float4 v) {
    asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(addr), "f"(v.x), "f"(v.y), "f"(v.z),
                 "f"(v.w)
                 : "memory");
}
#endif

}  // namespace sgb
