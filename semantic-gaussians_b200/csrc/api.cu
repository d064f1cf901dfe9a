// C-ABI entry points (include/sgb200.h): argument validation, state carving, stage sequencing.
#include <cstdarg>
#include <cstdlib>
#include <cstring>
#include "common.cuh"
#include "chn_blend.cuh"

namespace sgb {

static thread_local char g_err[512] = "";

void set_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof g_err, fmt, ap);
    va_end(ap);
}
int cuda_fail(cudaError_t e, const char* what) {
    set_error("CUDA error in %s: %s", what, cudaGetErrorString(e));
    cudaGetLastError();
    return SGB_E_CUDA;
}

namespace {

// Same argument rules as GaussianRasterizer.forward (channel_rasterization/__init__.py:258-264)
// and Rasterizer::forward (rasterizer_impl.cu:243-246).
int check_inputs(const sgb_view_inputs& in) {
    if (in.P < 0 || in.W <= 0 || in.H <= 0 || in.C <= 0) {
        set_error("invalid sizes P=%d W=%d H=%d C=%d", in.P, in.W, in.H, in.C);
        return SGB_E_INVALID;
    }
    if ((in.shs == nullptr) == (in.colors_precomp == nullptr)) {
        set_error("Please provide excatly one of either SHs or precomputed colors!");
        return SGB_E_INVALID;
    }
    const bool sr = in.scales != nullptr && in.rotations != nullptr;
    const bool any_sr = in.scales != nullptr || in.rotations != nullptr;
    if ((!sr && in.cov3D_precomp == nullptr) || (any_sr && in.cov3D_precomp != nullptr)) {
        set_error("Please provide exactly one of either scale/rotation pair or precomputed 3D covariance!");
        return SGB_E_INVALID;
    }
    if (in.C != 3 && in.colors_precomp == nullptr) {
        set_error("For non-RGB, provide precomputed Gaussian colors!");
        return SGB_E_INVALID;
    }
    if (in.shs && (in.M <= 0 || in.M > SGB_MAX_SH_COEFFS || in.D < 0 || (in.D + 1) * (in.D + 1) > in.M)) {
        set_error("SH degree %d needs %d coefficients, got M=%d", in.D, (in.D + 1) * (in.D + 1), in.M);
        return SGB_E_INVALID;
    }
    if (!in.background || !in.means3D || !in.opacities || !in.viewmatrix || !in.projmatrix || !in.campos) {
        set_error("null required input pointer");
        return SGB_E_INVALID;
    }
    if (in.antialiasing != 0 && in.antialiasing != 1) {
        set_error("antialiasing must be 0 or 1, got %d", in.antialiasing);
        return SGB_E_INVALID;
    }
    return SGB_OK;
}

__global__ void extract_rec_kernel(int P, const SplatRec* __restrict__ rec, int what, float* __restrict__ dst) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= P) return;
    const SplatRec r = rec[i];
    if (what == 0) dst[i] = r.depth;
    else if (what == 1) { dst[2 * i] = r.mx; dst[2 * i + 1] = r.my; }
    else { dst[4 * i] = r.cx; dst[4 * i + 1] = r.cy; dst[4 * i + 2] = r.cz; dst[4 * i + 3] = r.op; }
}

}  // namespace
}  // namespace sgb

using namespace sgb;

extern "C" {

const char* sgb_last_error(void) { return g_err; }
const char* sgb_version(void) { return "sgb200 0.2.0 (sm_90a)"; }
#ifndef SGB_BUILD_ID
#define SGB_BUILD_ID "unknown"
#endif
const char* sgb_build_id(void) { return "sgb200 0.2.0 src:" SGB_BUILD_ID; }

int sgb_ctx_create(sgb_ctx** out, int device) {
    if (!out) { set_error("null out"); return SGB_E_INVALID; }
    // the caller's current device is left as it was (a host framework tracks it; changing it behind its back makes
    // later launches land on streams of a non-current device)
    int prev = -1;
    SGB_CUDA(cudaGetDevice(&prev));
    SGB_CUDA(cudaSetDevice(device));
    sgb_ctx* c = new sgb_ctx();
    c->device = device;
    c->pools = new WeightPools();
    cudaError_t e = cudaMallocHost(&c->pinned, sizeof(Readback));
    if (prev >= 0 && prev != device) cudaSetDevice(prev);
    if (e != cudaSuccess) { sgb_ctx_destroy(c); return cuda_fail(e, "cudaMallocHost"); }
    *out = c;
    return SGB_OK;
}

void sgb_ctx_destroy(sgb_ctx* c) {
    if (!c) return;
    if (c->prof.created)
        for (int st = 0; st < ST_COUNT; st++)
            for (int i = 0; i < kProfRing; i++) {
                cudaEventDestroy(c->prof.ev[st][i][0]);
                cudaEventDestroy(c->prof.ev[st][i][1]);
            }
    if (c->geom.p) cudaFree(c->geom.p);
    if (c->bin.p) cudaFree(c->bin.p);
    if (c->misc.p) cudaFree(c->misc.p);
    if (c->work.p) cudaFree(c->work.p);
    if (c->depth_grad.p) cudaFree(c->depth_grad.p);
    if (c->cam_partial.p) cudaFree(c->cam_partial.p);
    if (c->lift_state.p) cudaFree(c->lift_state.p);
    if (c->lift_bin.p) cudaFree(c->lift_bin.p);
    delete c->pools;
    if (c->pinned) cudaFreeHost(c->pinned);
    delete c;
}

int sgb_profile_enable(sgb_ctx* c, int on) {
    if (!c) { set_error("null ctx"); return SGB_E_INVALID; }
    if (on && !c->prof.created) {
        for (int st = 0; st < ST_COUNT; st++)
            for (int i = 0; i < kProfRing; i++) {
                SGB_CUDA(cudaEventCreate(&c->prof.ev[st][i][0]));
                SGB_CUDA(cudaEventCreate(&c->prof.ev[st][i][1]));
            }
        c->prof.created = true;
    }
    for (int st = 0; st < ST_COUNT; st++) c->prof.n[st] = 0;
    c->prof.on = on != 0;
    return SGB_OK;
}

int sgb_profile_read(sgb_ctx* c, float* ms_sum, int32_t* count) {
    if (!c || !ms_sum || !count) { set_error("null argument"); return SGB_E_INVALID; }
    for (int st = 0; st < ST_COUNT; st++) {
        float acc = 0.f;
        for (int i = 0; i < c->prof.n[st]; i++) {
            SGB_CUDA(cudaEventSynchronize(c->prof.ev[st][i][1]));
            float ms = 0.f;
            SGB_CUDA(cudaEventElapsedTime(&ms, c->prof.ev[st][i][0], c->prof.ev[st][i][1]));
            acc += ms;
        }
        ms_sum[st] = acc;
        count[st] = c->prof.n[st];
        c->prof.n[st] = 0;
    }
    return SGB_OK;
}

int sgb_profile_num_stages(void) { return ST_COUNT; }
const char* sgb_profile_stage_name(int st) {
    static const char* names[ST_COUNT] = {"preprocess", "depth_sort", "scan", "emit", "tile_sort", "ranges",
                                          "blend_fwd", "blend_bwd", "geom_bwd", "fusion_project",
                                          "fusion_sort", "fusion_gather", "alpha_pass", "dfeature", "weight_sum"};
    return (st >= 0 && st < ST_COUNT) ? names[st] : "";
}
uint64_t sgb_ctx_launch_count(const sgb_ctx* c, int library_calls) {
    return c ? (library_calls ? c->lib_launches : c->launches) : 0;
}

size_t sgb_ctx_scratch_bytes(const sgb_ctx* c) {
    if (!c) return 0;
    return c->geom.cap + c->bin.cap + c->misc.cap + c->work.cap + c->depth_grad.cap + c->cam_partial.cap +
           c->lift_state.cap + c->lift_bin.cap + c->pools->bytes();
}

size_t sgb_geometry_bytes(int32_t P) { return GeomView::carve(nullptr, P > 0 ? P : 1).bytes; }
size_t sgb_binning_bytes(int64_t R) { return BinView::carve(nullptr, R).bytes; }
size_t sgb_image_bytes(int32_t W, int32_t H) { return ImgView::carve(nullptr, W, H).bytes; }

// ---- forward / backward, single view and batched (the single-view entry points are the V = 1 case) -----------
static int check_batch(const sgb_view_inputs* in, int32_t V, const sgb_camera* cams) {
    if (!in) { set_error("null sgb_view_inputs"); return SGB_E_INVALID; }
    if (V < 1 || V > SGB_MAX_BATCH) { set_error("batch of %d views: need 1 <= V <= %d", V, SGB_MAX_BATCH); return SGB_E_INVALID; }
    if (!cams) { set_error("null camera array"); return SGB_E_INVALID; }
    for (int v = 0; v < V; v++) {
        int rc = check_inputs(with_camera(*in, cams[v]));
        if (rc) return rc;
    }
    return SGB_OK;
}

// The camera of a single-view call, for its V = 1 batch.
static sgb_camera camera_of(const sgb_view_inputs& in) {
    return {in.viewmatrix, in.projmatrix, in.campos, in.tan_fovx, in.tan_fovy};
}

static int forward_geometry_impl(sgb_ctx* ctx, const sgb_view_inputs& in, int V, const sgb_camera* cams,
                                 void* const* geometry_states, int32_t* const* radii, int64_t* num_rendered_host,
                                 cudaStream_t s) {
    for (int v = 0; v < V; v++) num_rendered_host[v] = 0;
    if (in.P == 0) return SGB_OK;  // rasterize_points.cu:84: nothing to do for an empty scene
    int rc = run_depth_order_and_scan(ctx, in, V, cams, geometry_states, radii, num_rendered_host, s);
    if (rc) return rc;
    for (int v = 0; v < V; v++)
        if (num_rendered_host[v] > 0x7fffffffLL) {
            set_error("num_rendered %lld exceeds int32", (long long)num_rendered_host[v]);
            return SGB_E_OVERFLOW;
        }
    return SGB_OK;
}

// The RGB inputs with the feature table in place of the colours: the view the feature stages see.  Geometry, binning
// and image state are the RGB render's (neither depends on the colours), so the feature blend reads the same lists.
static sgb_view_inputs feature_inputs(const sgb_view_inputs& rgb, const float* features, int32_t c,
                                      const float* bg_features) {
    sgb_view_inputs f = rgb;
    f.C = c;
    f.shs = nullptr;
    f.M = 0;
    f.colors_precomp = features;
    f.background = bg_features;
    return f;
}

static int check_feature_table(const char* what, const sgb_view_inputs& in, const float* features, int32_t c,
                               const float* bg_features) {
    if (in.C != 3) { set_error("%s: the colour image has C = 3, got C = %d", what, in.C); return SGB_E_INVALID; }
    if (c < 1) { set_error("%s: need a feature table with c >= 1 channels, got c = %d", what, c); return SGB_E_INVALID; }
    if (!features || !bg_features) { set_error("%s: null feature table or feature background", what); return SGB_E_INVALID; }
    return SGB_OK;
}

// The argument rules of a render call, checked before anything is enqueued.  A joint call (`joint`: the image of `in`
// is the RGB image, and a feature table is rendered from the same lists) also needs an RGB `in`, the feature table,
// its background and outputs, and the median depth.
static int check_render(const char* what, bool joint, sgb_ctx* ctx, const sgb_view_inputs* in, int32_t V,
                        const sgb_camera* cams, const int64_t* num_rendered, void* const* geometry_states,
                        void* const* binning_states, void* const* image_states, const int32_t* const* radii,
                        float* const* out_colors, float* const* out_depths, float* const* out_exp_depths,
                        float* const* out_alphas, const float* features, int32_t c, const float* bg_features,
                        float* const* out_features) {
    int rc = check_batch(in, V, cams);
    if (rc) return rc;
    if (joint) {
        rc = check_feature_table(what, *in, features, c, bg_features);
        if (rc) return rc;
    }
    if (!ctx || !num_rendered || !geometry_states || !binning_states || !image_states || !radii || !out_colors ||
        (joint && (!out_depths || !out_features))) {
        set_error("%s: null argument", what);
        return SGB_E_INVALID;
    }
    if (in->C > 4 && out_depths) {
        set_error("out_depth is only produced by the 3-channel RGB-D path (C <= 4)");
        return SGB_E_INVALID;
    }
    if (in->C > 4 && (out_exp_depths || out_alphas)) {
        set_error("expected depth and alpha are only produced by the C <= 4 path");
        return SGB_E_INVALID;
    }
    if ((out_exp_depths == nullptr) != (out_alphas == nullptr)) {
        set_error("out_exp_depths and out_alphas are given together or not at all");
        return SGB_E_INVALID;
    }
    for (int v = 0; v < V; v++)
        if (!image_states[v] || !out_colors[v] || (in->P > 0 && (!geometry_states[v] || !radii[v])) ||
            (num_rendered[v] > 0 && !binning_states[v]) || (out_exp_depths && (!out_exp_depths[v] || !out_alphas[v])) ||
            (joint && (!out_features[v] || !out_depths[v]))) {
            set_error("%s: null state/output of view %d", what, v);
            return SGB_E_INVALID;
        }
    return SGB_OK;
}

// The argument rules of a backward call, checked before anything is enqueued; `joint` as in check_render, with the
// feature image's upstream gradients and the feature gradient buffer.
static int check_backward(const char* what, bool joint, sgb_ctx* ctx, const sgb_view_inputs* in, int32_t V,
                          const sgb_camera* cams, const int64_t* num_rendered, const int32_t* const* radii,
                          const void* const* geometry_states, const void* const* binning_states,
                          const void* const* image_states, const float* const* dL_dpix,
                          const float* const* dL_dexp_depth, const float* const* dL_dalpha,
                          const sgb_view_grads* grads, const float* features, int32_t c, const float* bg_features,
                          const float* const* dL_dfeature_pix, float* dL_dfeatures) {
    int rc = check_batch(in, V, cams);
    if (rc) return rc;
    if (joint) {
        rc = check_feature_table(what, *in, features, c, bg_features);
        if (rc) return rc;
    }
    if (in->C > 4 && (dL_dexp_depth || dL_dalpha)) {
        set_error("expected depth and alpha are only produced by the C <= 4 path");
        return SGB_E_INVALID;
    }
    if (!ctx || !num_rendered || !radii || !geometry_states || !binning_states || !image_states || !dL_dpix || !grads ||
        (joint && (!dL_dfeature_pix || !dL_dfeatures))) {
        set_error("%s: null argument", what);
        return SGB_E_INVALID;
    }
    for (int v = 0; v < V; v++) {
        if ((dL_dexp_depth && !dL_dexp_depth[v]) || (dL_dalpha && !dL_dalpha[v])) {
            set_error("%s: null dL_dexp_depth / dL_dalpha of view %d", what, v);
            return SGB_E_INVALID;
        }
        if (in->P == 0) continue;
        const sgb_view_grads& gr = grads[v];
        if (!geometry_states[v] || !radii[v] || !image_states[v] || !dL_dpix[v] || (joint && !dL_dfeature_pix[v]) ||
            !gr.dL_dmeans2D || !gr.dL_dconic || !gr.dL_dopacity || !gr.dL_dcolors || !gr.dL_dmeans3D ||
            !gr.dL_dcov3D || (in->shs && !gr.dL_dsh) || (in->scales && (!gr.dL_dscales || !gr.dL_drotations))) {
            set_error("%s: null state or gradient buffer of view %d", what, v);
            return SGB_E_INVALID;
        }
    }
    // with SH colours the geometry kernel of view v reads dL_dcolors as view v's RGB gradient, after view v's blend
    // has added into it: a buffer shared with an earlier view would carry that view's gradient too
    if (in->shs)
        for (int v = 1; v < V; v++)
            for (int u = 0; u < v; u++)
                if (grads[v].dL_dcolors == grads[u].dL_dcolors) {
                    set_error("%s: views %d and %d share one dL_dcolors buffer; with shs every view needs its own "
                              "dL_dcolors", what, u, v);
                    return SGB_E_INVALID;
                }
    return SGB_OK;
}

// The camera-gradient outputs of a _cam backward call (NULL: none): every pointer set, no pointer used twice.
static int check_camera_grads(const char* what, int32_t V, const sgb_camera_grads* cg) {
    if (!cg) return SGB_OK;
    const float* seen[3 * SGB_MAX_BATCH];
    int n = 0;
    for (int v = 0; v < V; v++)
        for (const float* q : {cg[v].dL_dviewmatrix, cg[v].dL_dprojmatrix, cg[v].dL_dcampos}) {
            if (!q) {
                set_error("%s: null camera-gradient output of view %d", what, v);
                return SGB_E_INVALID;
            }
            for (int i = 0; i < n; i++)
                if (seen[i] == q) {
                    set_error("%s: one camera-gradient buffer is given twice (view %d)", what, v);
                    return SGB_E_INVALID;
                }
            seen[n++] = q;
        }
    return SGB_OK;
}

// Per view: binning once, then the images on its lists.  The POOLED image is the feature image `fin` when given, else
// the image of `in`.  When its C > 4, its alpha pass builds the weight pool (for a joint call the same walk is the RGB
// blend of `in`, median depth and expected depth / alpha included), and after the one pool check of the batch the
// forward contraction renders it.  Otherwise the small-C blend renders the image of `in` and then `fin`.  Every walk
// writes final_T / n_contrib / tile_last with the RGB blend's statement sequence, so the image state is the same
// whichever renders it.
static int forward_render_impl(sgb_ctx* ctx, const sgb_view_inputs& in, const sgb_view_inputs* fin, int V,
                               const sgb_camera* cams, const int64_t* num_rendered, void* const* geometry_states,
                               void* const* binning_states, void* const* image_states, const int32_t* const* radii,
                               float* const* out_colors, float* const* out_depths, float* const* out_exp_depths,
                               float* const* out_alphas, float* const* out_features, cudaStream_t s) {
    int64_t maxR = 0;
    for (int v = 0; v < V; v++) maxR = num_rendered[v] > maxR ? num_rendered[v] : maxR;
    int rc = reserve_binning(ctx, in, in.P > 0 ? maxR : 0, s);
    if (rc) return rc;
    const sgb_view_inputs& pooled = fin ? *fin : in;
    float* const* out_pooled = fin ? out_features : out_colors;
    const bool wide = pooled.C > 4;
    ViewState vp[SGB_MAX_BATCH];
    for (int v = 0; v < V; v++) {
        const ViewState w = ViewState::carve(in, cams[v], num_rendered[v], geometry_states[v], binning_states[v],
                                             image_states[v]);
        vp[v] = ViewState::carve(pooled, cams[v], num_rendered[v], geometry_states[v], binning_states[v],
                                 image_states[v]);
        rc = run_binning(ctx, w.in, w.R, w.g, w.b, w.im, radii[v], s);
        if (rc) return rc;
        float* const out_depth = out_depths ? out_depths[v] : nullptr;
        float* const out_exp_depth = out_exp_depths ? out_exp_depths[v] : nullptr;
        float* const out_alpha = out_alphas ? out_alphas[v] : nullptr;
        if (wide) {
            const AlphaRgb rgb{w.colors, w.in.background, out_colors[v], out_depth, out_exp_depth, out_alpha};
            rc = weight_pool_build(ctx, vp[v], s, fin ? &rgb : nullptr);
            if (rc) return rc;
            continue;
        }
        StageTimer t(ctx, ST_BLEND_FWD, s);
        ctx->launches += fin ? 2 : 1;
        rc = launch_blend_forward(w.in, w.g, w.b, w.im, w.colors, out_colors[v], out_depth, out_exp_depth, out_alpha,
                                  s);
        if (!rc && fin)
            rc = launch_blend_forward(vp[v].in, vp[v].g, vp[v].b, vp[v].im, vp[v].colors, out_features[v], nullptr,
                                      nullptr, nullptr, s);
        if (rc) return rc;
    }
    if (!wide) return SGB_OK;
    // the host waits for the alpha passes only; the forward GEMMs are enqueued once all weight pools are checked
    PoolView pv[SGB_MAX_BATCH];
    rc = weight_pool_settle(ctx, V, vp, pv, s);
    if (rc) return rc;
    for (int v = 0; v < V; v++) {
        rc = chn_forward(ctx, vp[v], pv[v], out_pooled[v], s);
        if (rc) return rc;
    }
    return SGB_OK;
}

// The backward of forward_render_impl.  The pooled image's gradient target is dL_dfeatures for a joint call, else
// grads[v].dL_dcolors.  When its C > 4, dL/dfeature of every view runs first: it needs only the weight rows and
// dL/dout, it is the one large gradient and it accumulates across the views of a batch, so a data-parallel caller can
// start exchanging it (the feature-gradient event) while the chain / geometry kernels of the whole batch run
// (sgb200.h).  Then per view: the pooled image's chain (or small-C blend) backward, for a joint call the RGB blend
// backward, and ONE geometry backward with the RGB colour gradient.  The blend that carries the dL_dexp_depth /
// dL_dalpha terms is the one of `in`.  All blend backwards add into the same dL_dmeans2D / dL_dconic / dL_dopacity.
// cam_grads (NULL or [V]): the geometry backward of view v also writes view v's camera gradient.
static int backward_impl(sgb_ctx* ctx, const sgb_view_inputs& in, const sgb_view_inputs* fin, int V,
                         const sgb_camera* cams, const int64_t* num_rendered, const int32_t* const* radii,
                         const void* const* geometry_states, const void* const* binning_states,
                         const void* const* image_states, const float* const* dL_dpix,
                         const float* const* dL_dexp_depth, const float* const* dL_dalpha, const sgb_view_grads* grads,
                         const float* const* dL_dfeature_pix, float* dL_dfeatures, const sgb_camera_grads* cam_grads,
                         cudaStream_t s) {
    if (in.P == 0) {
        if (ctx->feature_grad_event) SGB_CUDA(cudaEventRecord(ctx->feature_grad_event, s));
        for (int v = 0; cam_grads && v < V; v++) {  // no Gaussian: a zero camera gradient
            SGB_CUDA(cudaMemsetAsync(cam_grads[v].dL_dviewmatrix, 0, 16 * sizeof(float), s));
            SGB_CUDA(cudaMemsetAsync(cam_grads[v].dL_dprojmatrix, 0, 16 * sizeof(float), s));
            SGB_CUDA(cudaMemsetAsync(cam_grads[v].dL_dcampos, 0, 3 * sizeof(float), s));
        }
        return SGB_OK;
    }
    const sgb_view_inputs& pooled = fin ? *fin : in;
    const float* const* dL_dpooled_pix = fin ? dL_dfeature_pix : dL_dpix;
    auto pooled_target = [&](int v) { return fin ? dL_dfeatures : grads[v].dL_dcolors; };
    ViewState vw[SGB_MAX_BATCH], vp[SGB_MAX_BATCH];
    for (int v = 0; v < V; v++) {
        vw[v] = ViewState::carve(in, cams[v], num_rendered[v], geometry_states[v], binning_states[v], image_states[v]);
        vp[v] = ViewState::carve(pooled, cams[v], num_rendered[v], geometry_states[v], binning_states[v],
                                 image_states[v]);
    }
    const bool wide = pooled.C > 4;
    int rc;
    // expected depth / alpha: one [P] dL/dz buffer, zeroed before each view's blend and read by its geometry kernel
    float* dL_ddepth = nullptr;
    if (dL_dexp_depth || dL_dalpha) {
        rc = ctx->depth_grad.ensure(sizeof(float) * (size_t)in.P);
        if (rc) return rc;
        dL_ddepth = (float*)ctx->depth_grad.p;
    }
    if (cam_grads) {
        rc = ctx->cam_partial.ensure(camera_grad_partial_bytes(in.P));
        if (rc) return rc;
    }
    // the small-C blend backward of image w of view v; the one of `in` carries the depth terms
    auto blend_backward = [&](const ViewState& w, int v, const float* dL_dout, float* dL_dcolor, bool depth) -> int {
        if (depth && dL_ddepth) SGB_CUDA(cudaMemsetAsync(dL_ddepth, 0, sizeof(float) * (size_t)in.P, s));
        const sgb_view_grads& gr = grads[v];
        StageTimer t(ctx, ST_BLEND_BWD, s);
        ctx->launches += 1;
        return launch_blend_backward(w.in, w.g, w.b, w.im, w.colors, dL_dout, gr.dL_dmeans2D, gr.dL_dconic,
                                     gr.dL_dopacity, dL_dcolor, depth && dL_dexp_depth ? dL_dexp_depth[v] : nullptr,
                                     depth && dL_dalpha ? dL_dalpha[v] : nullptr, depth ? dL_ddepth : nullptr, s);
    };
    PoolView pv[SGB_MAX_BATCH];
    if (wide) {
        rc = weight_rows_for_backward(ctx, V, vp, pv, s);
        if (rc) return rc;
        for (int v = 0; v < V; v++) {
            if (vp[v].R <= 0) continue;
            rc = chn_dfeature(ctx, vp[v], pv[v], dL_dpooled_pix[v], pooled_target(v), s);
            if (rc) return rc;
        }
        if (ctx->feature_grad_event) SGB_CUDA(cudaEventRecord(ctx->feature_grad_event, s));
    }
    for (int v = 0; v < V; v++) {
        const sgb_view_grads& gr = grads[v];
        if (vp[v].R > 0 && wide) {
            rc = chn_chain(ctx, vp[v], pv[v], dL_dpooled_pix[v], gr.dL_dmeans2D, gr.dL_dconic, gr.dL_dopacity, s);
            if (rc) return rc;
        } else if (vp[v].R > 0) {
            rc = blend_backward(vp[v], v, dL_dpooled_pix[v], pooled_target(v), !fin);
            if (rc) return rc;
        }
        if (!wide && v == V - 1 && ctx->feature_grad_event) SGB_CUDA(cudaEventRecord(ctx->feature_grad_event, s));
        if (fin && vw[v].R > 0) {
            rc = blend_backward(vw[v], v, dL_dpix[v], gr.dL_dcolors, true);
            if (rc) return rc;
        }
        const float* cov3D = in.cov3D_precomp ? in.cov3D_precomp : vw[v].g.cov3D;  // rasterizer_impl.cu:417
        StageTimer t(ctx, ST_GEOM_BWD, s);
        ctx->launches += cam_grads ? 2 : 1;
        // a view without instances has no blend and so no depth gradient
        rc = launch_geom_backward(vw[v].in, vw[v].g, radii[v], cov3D, gr.dL_dcolors, gr, vw[v].R > 0 ? dL_ddepth : nullptr,
                                  cam_grads ? &cam_grads[v] : nullptr, (double*)ctx->cam_partial.p, s);
        if (rc) return rc;
    }
    return SGB_OK;
}

int sgb_forward_geometry(sgb_ctx* ctx, const sgb_view_inputs* in, void* geometry_state, int32_t* radii,
                         int64_t* num_rendered_host, void* stream) {
    if (!in) { set_error("null sgb_view_inputs"); return SGB_E_INVALID; }
    const sgb_camera cam = camera_of(*in);
    return sgb_forward_geometry_batch(ctx, in, 1, &cam, &geometry_state, &radii, num_rendered_host, stream);
}

int sgb_forward_geometry_batch(sgb_ctx* ctx, const sgb_view_inputs* in, int32_t V, const sgb_camera* cams,
                               void* const* geometry_states, int32_t* const* radii, int64_t* num_rendered_host,
                               void* stream) {
    int rc = check_batch(in, V, cams);
    if (rc) return rc;
    if (!ctx || !num_rendered_host || !geometry_states || !radii) {
        set_error("sgb_forward_geometry_batch: null ctx/state/radii/num_rendered");
        return SGB_E_INVALID;
    }
    if (in->P > 0)
        for (int v = 0; v < V; v++)
            if (!geometry_states[v] || !radii[v]) { set_error("sgb_forward_geometry_batch: null state of view %d", v); return SGB_E_INVALID; }
    return forward_geometry_impl(ctx, *in, V, cams, geometry_states, radii, num_rendered_host, (cudaStream_t)stream);
}

int sgb_forward_render(sgb_ctx* ctx, const sgb_view_inputs* in, int64_t num_rendered, void* geometry_state,
                       void* binning_state, void* image_state, const int32_t* radii, float* out_color,
                       float* out_depth, void* stream) {
    if (!in) { set_error("null sgb_view_inputs"); return SGB_E_INVALID; }
    const sgb_camera cam = camera_of(*in);
    return sgb_forward_render_batch(ctx, in, 1, &cam, &num_rendered, &geometry_state, &binning_state, &image_state,
                                    &radii, &out_color, out_depth ? &out_depth : nullptr, stream);
}

int sgb_forward_render_batch(sgb_ctx* ctx, const sgb_view_inputs* in, int32_t V, const sgb_camera* cams,
                             const int64_t* num_rendered, void* const* geometry_states, void* const* binning_states,
                             void* const* image_states, const int32_t* const* radii, float* const* out_colors,
                             float* const* out_depths, void* stream) {
    return sgb_forward_render_batch_ext(ctx, in, V, cams, num_rendered, geometry_states, binning_states, image_states,
                                        radii, out_colors, out_depths, nullptr, nullptr, stream);
}

int sgb_forward_render_batch_ext(sgb_ctx* ctx, const sgb_view_inputs* in, int32_t V, const sgb_camera* cams,
                                 const int64_t* num_rendered, void* const* geometry_states,
                                 void* const* binning_states, void* const* image_states, const int32_t* const* radii,
                                 float* const* out_colors, float* const* out_depths, float* const* out_exp_depths,
                                 float* const* out_alphas, void* stream) {
    int rc = check_render("sgb_forward_render_batch", false, ctx, in, V, cams, num_rendered, geometry_states,
                          binning_states, image_states, radii, out_colors, out_depths, out_exp_depths, out_alphas,
                          nullptr, 0, nullptr, nullptr);
    if (rc) return rc;
    return forward_render_impl(ctx, *in, nullptr, V, cams, num_rendered, geometry_states, binning_states, image_states,
                               radii, out_colors, out_depths, out_exp_depths, out_alphas, nullptr,
                               (cudaStream_t)stream);
}

int sgb_backward(sgb_ctx* ctx, const sgb_view_inputs* in, int64_t num_rendered, const int32_t* radii,
                 const void* geometry_state, const void* binning_state, const void* image_state,
                 const float* dL_dpix, const sgb_view_grads* gr, void* stream) {
    if (!in) { set_error("null sgb_view_inputs"); return SGB_E_INVALID; }
    const sgb_camera cam = camera_of(*in);
    // a null image state or dL/dout is passed as a null array: the batch call checks the arrays for every P, their
    // entries only for P > 0
    return sgb_backward_batch(ctx, in, 1, &cam, &num_rendered, &radii, &geometry_state, &binning_state,
                              image_state ? &image_state : nullptr, dL_dpix ? &dL_dpix : nullptr, gr, stream);
}

int sgb_backward_batch(sgb_ctx* ctx, const sgb_view_inputs* in, int32_t V, const sgb_camera* cams,
                       const int64_t* num_rendered, const int32_t* const* radii, const void* const* geometry_states,
                       const void* const* binning_states, const void* const* image_states,
                       const float* const* dL_dpix, const sgb_view_grads* grads, void* stream) {
    return sgb_backward_batch_ext(ctx, in, V, cams, num_rendered, radii, geometry_states, binning_states, image_states,
                                  dL_dpix, nullptr, nullptr, grads, stream);
}

int sgb_backward_batch_ext(sgb_ctx* ctx, const sgb_view_inputs* in, int32_t V, const sgb_camera* cams,
                           const int64_t* num_rendered, const int32_t* const* radii,
                           const void* const* geometry_states, const void* const* binning_states,
                           const void* const* image_states, const float* const* dL_dpix,
                           const float* const* dL_dexp_depth, const float* const* dL_dalpha,
                           const sgb_view_grads* grads, void* stream) {
    return sgb_backward_batch_cam(ctx, in, V, cams, num_rendered, radii, geometry_states, binning_states, image_states,
                                  dL_dpix, dL_dexp_depth, dL_dalpha, grads, nullptr, stream);
}

int sgb_backward_batch_cam(sgb_ctx* ctx, const sgb_view_inputs* in, int32_t V, const sgb_camera* cams,
                           const int64_t* num_rendered, const int32_t* const* radii,
                           const void* const* geometry_states, const void* const* binning_states,
                           const void* const* image_states, const float* const* dL_dpix,
                           const float* const* dL_dexp_depth, const float* const* dL_dalpha,
                           const sgb_view_grads* grads, const sgb_camera_grads* cam_grads, void* stream) {
    int rc = check_backward("sgb_backward_batch", false, ctx, in, V, cams, num_rendered, radii, geometry_states,
                            binning_states, image_states, dL_dpix, dL_dexp_depth, dL_dalpha, grads, nullptr, 0,
                            nullptr, nullptr, nullptr);
    if (!rc) rc = check_camera_grads("sgb_backward_batch", V, cam_grads);
    if (rc) return rc;
    return backward_impl(ctx, *in, nullptr, V, cams, num_rendered, radii, geometry_states, binning_states, image_states,
                         dL_dpix, dL_dexp_depth, dL_dalpha, grads, nullptr, nullptr, cam_grads, (cudaStream_t)stream);
}

// ---- colour and a feature table through one geometry pass and one binning per view ---------------------------
int sgb_forward_render_joint_batch(sgb_ctx* ctx, const sgb_view_inputs* in, int32_t V, const sgb_camera* cams,
                                   const int64_t* num_rendered, void* const* geometry_states,
                                   void* const* binning_states, void* const* image_states,
                                   const int32_t* const* radii, float* const* out_colors, float* const* out_depths,
                                   float* const* out_exp_depths, float* const* out_alphas, const float* features,
                                   int32_t c, const float* bg_features, float* const* out_features, void* stream) {
    int rc = check_render("sgb_forward_render_joint_batch", true, ctx, in, V, cams, num_rendered, geometry_states,
                          binning_states, image_states, radii, out_colors, out_depths, out_exp_depths, out_alphas,
                          features, c, bg_features, out_features);
    if (rc) return rc;
    const sgb_view_inputs fin = feature_inputs(*in, features, c, bg_features);
    return forward_render_impl(ctx, *in, &fin, V, cams, num_rendered, geometry_states, binning_states, image_states,
                               radii, out_colors, out_depths, out_exp_depths, out_alphas, out_features,
                               (cudaStream_t)stream);
}

int sgb_backward_joint_batch(sgb_ctx* ctx, const sgb_view_inputs* in, int32_t V, const sgb_camera* cams,
                             const int64_t* num_rendered, const int32_t* const* radii,
                             const void* const* geometry_states, const void* const* binning_states,
                             const void* const* image_states, const float* const* dL_dpix,
                             const float* const* dL_dexp_depth, const float* const* dL_dalpha,
                             const sgb_view_grads* grads, const float* features, int32_t c, const float* bg_features,
                             const float* const* dL_dfeature_pix, float* dL_dfeatures, void* stream) {
    return sgb_backward_joint_batch_cam(ctx, in, V, cams, num_rendered, radii, geometry_states, binning_states,
                                        image_states, dL_dpix, dL_dexp_depth, dL_dalpha, grads, features, c,
                                        bg_features, dL_dfeature_pix, dL_dfeatures, nullptr, stream);
}

int sgb_backward_joint_batch_cam(sgb_ctx* ctx, const sgb_view_inputs* in, int32_t V, const sgb_camera* cams,
                                 const int64_t* num_rendered, const int32_t* const* radii,
                                 const void* const* geometry_states, const void* const* binning_states,
                                 const void* const* image_states, const float* const* dL_dpix,
                                 const float* const* dL_dexp_depth, const float* const* dL_dalpha,
                                 const sgb_view_grads* grads, const float* features, int32_t c,
                                 const float* bg_features, const float* const* dL_dfeature_pix, float* dL_dfeatures,
                                 const sgb_camera_grads* cam_grads, void* stream) {
    int rc = check_backward("sgb_backward_joint_batch", true, ctx, in, V, cams, num_rendered, radii, geometry_states,
                            binning_states, image_states, dL_dpix, dL_dexp_depth, dL_dalpha, grads, features, c,
                            bg_features, dL_dfeature_pix, dL_dfeatures);
    if (!rc) rc = check_camera_grads("sgb_backward_joint_batch", V, cam_grads);
    if (rc) return rc;
    const sgb_view_inputs fin = feature_inputs(*in, features, c, bg_features);
    return backward_impl(ctx, *in, &fin, V, cams, num_rendered, radii, geometry_states, binning_states, image_states,
                         dL_dpix, dL_dexp_depth, dL_dalpha, grads, dL_dfeature_pix, dL_dfeatures, cam_grads,
                         (cudaStream_t)stream);
}

// ---- lifting feature maps onto the Gaussians by their blend weights ------------------------------------------
// Per view: geometry, binning and the alpha pass (the weight pool) into ctx scratch, then the dL/dfeature contraction
// with the map as dL/dout and the per-Gaussian weight-row sums.  No colour blend, no chain or geometry backward.
static int lift_impl(sgb_ctx* ctx, const sgb_view_inputs& in, int V, const sgb_camera* cams, const void* const* maps,
                     int32_t map_dtype, float* feat_sum, float* weight_sum, cudaStream_t s) {
    const int P = in.P;
    const size_t geom_b = sgb_geometry_bytes(P), radii_b = align_up(sizeof(int32_t) * (size_t)P),
                 img_b = sgb_image_bytes(in.W, in.H), per_view = geom_b + radii_b + img_b;
    int rc = ctx->lift_state.ensure((size_t)V * per_view);
    if (rc) return rc;
    void* geom[SGB_MAX_BATCH];
    void* img[SGB_MAX_BATCH];
    int32_t* radii[SGB_MAX_BATCH];
    for (int v = 0; v < V; v++) {
        char* base = (char*)ctx->lift_state.p + (size_t)v * per_view;
        geom[v] = base;
        radii[v] = (int32_t*)(base + geom_b);
        img[v] = base + geom_b + radii_b;
    }
    int64_t R[SGB_MAX_BATCH];
    rc = forward_geometry_impl(ctx, in, V, cams, geom, radii, R, s);  // the first sync: the V instance counts
    if (rc) return rc;
    int64_t maxR = 0;
    size_t bin_total = 0;
    for (int v = 0; v < V; v++) {
        maxR = R[v] > maxR ? R[v] : maxR;
        bin_total += sgb_binning_bytes(R[v]);
    }
    if (maxR == 0) return SGB_OK;
    rc = reserve_binning(ctx, in, maxR, s);
    if (rc) return rc;
    rc = ctx->lift_bin.ensure(bin_total);
    if (rc) return rc;
    ViewState vw[SGB_MAX_BATCH];
    int nv = 0;  // views with instances, compacted to the front of vw
    size_t bin_off = 0;
    for (int v = 0; v < V; v++) {
        if (R[v] == 0) continue;
        ViewState& w = vw[nv];
        w = ViewState::carve(in, cams[v], R[v], geom[v], (char*)ctx->lift_bin.p + bin_off, img[v]);
        bin_off += sgb_binning_bytes(R[v]);
        rc = run_binning(ctx, w.in, w.R, w.g, w.b, w.im, radii[v], s);
        if (!rc) rc = weight_pool_build(ctx, w, s);
        if (rc) {
            weight_pool_release(ctx, nv + 1, vw);
            return rc;
        }
        nv++;
    }
    PoolView pv[SGB_MAX_BATCH];
    rc = weight_pool_settle(ctx, nv, vw, pv, s);  // the second sync: the weight-pool checks
    for (int k = 0, v = 0; !rc && v < V; v++) {
        if (R[v] == 0) continue;
        if (map_dtype == SGB_FEAT_F16)
            rc = chn_dfeature(ctx, vw[k], pv[k], static_cast<const __half*>(maps[v]), feat_sum, s);
        else
            rc = chn_dfeature(ctx, vw[k], pv[k], static_cast<const float*>(maps[v]), feat_sum, s);
        if (!rc) rc = pool_weight_sums(ctx, vw[k], pv[k], weight_sum, s);
        k++;
    }
    weight_pool_release(ctx, nv, vw);
    return rc;
}

int sgb_lift_batch(sgb_ctx* ctx, const sgb_view_inputs* in, int32_t V, const sgb_camera* cams,
                   const void* const* maps, int32_t map_dtype, float* feat_sum, float* weight_sum, void* stream) {
    if (!ctx || !in || !cams || !maps || !feat_sum || !weight_sum) {
        set_error("sgb_lift_batch: null argument");
        return SGB_E_INVALID;
    }
    if (V < 1 || V > SGB_MAX_BATCH) { set_error("batch of %d views: need 1 <= V <= %d", V, SGB_MAX_BATCH); return SGB_E_INVALID; }
    if (map_dtype != SGB_FEAT_F16 && map_dtype != SGB_FEAT_F32) {
        set_error("sgb_lift_batch: unknown map dtype %d", map_dtype);
        return SGB_E_INVALID;
    }
    if (in->shs || in->colors_precomp || in->background) {
        set_error("sgb_lift_batch: shs, colors_precomp and background must be NULL (the maps are the features)");
        return SGB_E_INVALID;
    }
    for (int v = 0; v < V; v++)
        if (!maps[v]) { set_error("sgb_lift_batch: null map of view %d", v); return SGB_E_INVALID; }
    // the forward's argument rules with placeholders for the absent colours and background; preprocess only tests
    // colors_precomp against NULL (to skip the SH colours) and nothing here reads either
    sgb_view_inputs g = *in;
    g.colors_precomp = in->means3D;
    g.background = in->means3D;
    int rc = check_batch(&g, V, cams);
    if (rc) return rc;
    if (in->P == 0) return SGB_OK;
    return lift_impl(ctx, g, V, cams, maps, map_dtype, feat_sum, weight_sum, (cudaStream_t)stream);
}

int64_t sgb_ctx_view_stat(const sgb_ctx* ctx, int which) {
    if (!ctx) return -1;
    return which == 0 ? ctx->pools->stat_blended_pairs : which == 1 ? ctx->pools->stat_pool_chunks : -1;
}

int sgb_ctx_set_feature_grad_event(sgb_ctx* ctx, void* cuda_event) {
    if (!ctx) { set_error("sgb_ctx_set_feature_grad_event: null ctx"); return SGB_E_INVALID; }
    ctx->feature_grad_event = (cudaEvent_t)cuda_event;
    return SGB_OK;
}

int sgb_mark_visible(int32_t P, const float* means3D, const float* viewmatrix, const float* projmatrix,
                     uint8_t* present, void* stream) {
    (void)projmatrix;  // the reference computes p_proj but only tests view-space z (auxiliary.h:149-154)
    if (P < 0 || (P > 0 && (!means3D || !viewmatrix || !present))) {
        set_error("sgb_mark_visible: bad arguments");
        return SGB_E_INVALID;
    }
    if (P == 0) return SGB_OK;
    return launch_mark_visible(P, means3D, viewmatrix, present, (cudaStream_t)stream);
}

int64_t sgb_state_field(const char* name, int32_t P, int64_t R, int32_t W, int32_t H, const void* geometry_state,
                        const void* binning_state, const void* image_state, void* dst, void* stream) {
    cudaStream_t s = (cudaStream_t)stream;
    if (!name || !dst) { set_error("sgb_state_field: null"); return SGB_E_INVALID; }
    const size_t N = (size_t)W * H;
    const size_t tiles = (size_t)((W + SGB_TILE - 1) / SGB_TILE) * ((H + SGB_TILE - 1) / SGB_TILE);
    const void* src = nullptr;
    size_t n = 0;
    if (geometry_state && P > 0) {
        GeomView g = GeomView::carve(const_cast<void*>(geometry_state), P);
        int what = !strcmp(name, "depths") ? 0 : !strcmp(name, "means2D") ? 1 : !strcmp(name, "conic_opacity") ? 2 : -1;
        if (what >= 0) {
            extract_rec_kernel<<<(P + 255) / 256, 256, 0, s>>>(P, g.rec, what, (float*)dst);
            SGB_LAUNCH_CHECK("extract_rec_kernel", 0, s);
            return (int64_t)P * (what == 0 ? 4 : what == 1 ? 8 : 16);
        }
        if (!strcmp(name, "cov3D")) { src = g.cov3D; n = (size_t)P * 24; }
        else if (!strcmp(name, "rgb")) { src = g.rgb; n = (size_t)P * 12; }
        else if (!strcmp(name, "clamped")) { src = g.clamped; n = (size_t)P * 3; }
        else if (!strcmp(name, "tiles_touched")) { src = g.tiles_touched; n = (size_t)P * 4; }
    }
    if (!src && image_state) {
        ImgView im = ImgView::carve(const_cast<void*>(image_state), W, H);
        if (!strcmp(name, "final_T")) { src = im.final_T; n = N * 4; }
        else if (!strcmp(name, "n_contrib")) { src = im.n_contrib; n = N * 4; }
        else if (!strcmp(name, "ranges")) { src = im.ranges; n = tiles * 8; }
        else if (!strcmp(name, "tile_last")) { src = im.tile_last; n = tiles * 4; }
    }
    if (!src && !strcmp(name, "point_list")) {
        if (R == 0) return 0;
        if (!binning_state) { set_error("no binning state"); return SGB_E_INVALID; }
        src = BinView::carve(const_cast<void*>(binning_state), R).point_list;
        n = (size_t)R * 4;
    }
    if (!src) { set_error("unknown or unavailable state field '%s'", name); return SGB_E_INVALID; }
    SGB_CUDA(cudaMemcpyAsync(dst, src, n, cudaMemcpyDeviceToDevice, s));
    return (int64_t)n;
}

}  // extern "C"
