/*
 * sgb200 — H100 (sm_90a) Gaussian-splatting rasterizer + 2D->3D fusion kernels: C ABI.
 *
 * This is the drop-in boundary for the reference's native rasterizer library.  Each entry
 * point names the reference interface it replaces (paths relative to
 * /root/reference/submodules/channel-rasterization unless prefixed):
 *
 *   sgb_forward_geometry + sgb_forward_render
 *        == CudaRasterizer::Rasterizer::forward           cuda_rasterizer/rasterizer.h:30-53,
 *           rgbd variant (out_depth)                      rgbd/cuda_rasterizer/rasterizer.h:31-53
 *   sgb_backward
 *        == CudaRasterizer::Rasterizer::backward          cuda_rasterizer/rasterizer.h:55-84
 *   sgb_mark_visible
 *        == CudaRasterizer::Rasterizer::markVisible       cuda_rasterizer/rasterizer.h:23-28
 *   sgb_fusion_map / sgb_fusion_accumulate / sgb_fusion_normalize
 *        == PointCloudToImageMapper.compute_mapping       dataset/fusion_utils.py:30-78
 *           + the per-view gather/accumulate and final divide   fusion.py:127-148
 *
 * Conventions
 *   - extern "C", plain pointers and sizes, no C++/torch types.  Every array argument is a
 *     DEVICE pointer unless its name ends in _host.  An absent optional input is NULL
 *     (the reference encodes it the same way: rasterizer_impl.cu:243,324,394,417).  The
 *     per-Gaussian float arrays, their gradients and dL/dout need 4-byte alignment only: a view into a larger
 *     buffer at any float offset is accepted.
 *   - Every call takes the CUDA stream to launch on (cudaStream_t passed as void*); the
 *     reference launches on the legacy default stream.  Calls are asynchronous except
 *     sgb_forward_geometry, which returns num_rendered and therefore synchronises the stream
 *     once — the reference does the same with a blocking cudaMemcpy (rasterizer_impl.cu:283).
 *   - Return value: SGB_OK (0) or a negative error code; sgb_last_error() gives the message of
 *     the last failure on the calling thread.  (Reference: C++ exceptions,
 *     rasterizer_impl.cu:245, auxiliary.h:166-173.)
 *   - Ownership: the caller owns every buffer.  Forward fills three opaque state buffers
 *     (geometry / binning / image) that backward consumes — same contract as the reference's
 *     geomBuffer/binningBuffer/imgBuffer (rasterize_points.cu:28-36,73-80), but sized up
 *     front through sgb_*_bytes() instead of std::function resize callbacks.  Scratch that does
 *     not outlive a call (sort double-buffers, CUB temp storage) lives in the sgb_ctx.
 *   - Render and backward read only the states, radii and num_rendered they are given, which must
 *     come from one geometry call for the same inputs (as in the reference).  Calls may interleave
 *     on a ctx, and a render may run on another ctx than its geometry call.  The one thing a ctx
 *     carries from call to call is the weight-pool cache of the C > 4 blend: keyed by binning
 *     state, checked on use and rebuilt on a miss.
 *   - A ctx is bound to one device and must not be used by two streams concurrently.
 */
#ifndef SGB200_H_INCLUDED
#define SGB200_H_INCLUDED

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define SGB_OK 0
#define SGB_E_INVALID (-1)   /* bad argument combination (reference: "provide exactly one of ...") */
#define SGB_E_CUDA (-2)      /* CUDA runtime / launch error */
#define SGB_E_NOMEM (-3)     /* scratch allocation failed */
#define SGB_E_OVERFLOW (-4)  /* num_rendered does not fit in int32 */

#define SGB_TILE 16          /* BLOCK_X = BLOCK_Y = 16, cuda_rasterizer/config.h:16-17 */
#define SGB_MAX_SH_COEFFS 16

typedef struct sgb_ctx sgb_ctx;

/* Inputs of one view.  Field-for-field the argument list of Rasterizer::forward. */
typedef struct sgb_view_inputs {
    int32_t P;                   /* number of Gaussians */
    int32_t D;                   /* active SH degree (0..3) */
    int32_t M;                   /* SH coefficients per colour channel in `shs` (0 if shs NULL) */
    int32_t W, H;                /* image size in pixels */
    int32_t C;                   /* channels: 3 for RGB; run-time C for the feature raster */
    const float* background;     /* [C] */
    const float* means3D;        /* [P,3] */
    const float* shs;            /* [P,M,3] or NULL (requires C == 3) */
    const float* colors_precomp; /* [P,C] or NULL */
    const float* opacities;      /* [P] */
    const float* scales;         /* [P,3] or NULL */
    float scale_modifier;
    const float* rotations;      /* [P,4] (w,x,y,z), used as given, or NULL */
    const float* cov3D_precomp;  /* [P,6] or NULL */
    const float* viewmatrix;     /* [16]  W2C transposed (scene/camera.py:87) */
    const float* projmatrix;     /* [16]  (P*W2C) transposed (scene/camera.py:91-93) */
    const float* campos;         /* [3] */
    float tan_fovx, tan_fovy;
    int32_t prefiltered;         /* trap if a Gaussian fails the near cull (auxiliary.h:156-160) */
    int32_t debug;               /* synchronise + check after every stage (auxiliary.h:166-173) */
    /* Anti-aliasing (3DGS's PipelineParams.antialiasing, Mip-Splatting's screen-space filter): 0 = off, 1 = on; any
     * other value returns SGB_E_INVALID before anything is enqueued.  With C0 the screen covariance before the fixed
     * 0.3 px^2 dilation and C = C0 + 0.3 I, every blend reads the opacity o h, h = sqrt(max(2.5e-5, det C0 / det C)):
     * a Gaussian keeps the integral of its undilated footprint at every image size.  Conics, radii, tiles, binning
     * and depth order are unchanged; the geometry backward carries dL/do = h dL/d(o h) and the covariance term of h
     * (to means3D, cov3D, scales / rotations and the camera).  Honoured by every call that takes sgb_view_inputs,
     * sgb_lift_batch included; the backward must be given the forward's value.  This field grew the struct by 4 bytes
     * (no padding change before it); a zero-initialised struct keeps the behaviour without it. */
    int32_t antialiasing;
} sgb_view_inputs;

/* Gradients of one view (all caller-zero-filled, as rasterize_points.cu:157-165 does). */
typedef struct sgb_view_grads {
    float* dL_dmeans2D;   /* [P,3]   .xy in the reference's units (backward.cu:455-456,540-541) */
    float* dL_dconic;     /* [P,4]   (x, y, _, w) as backward.cu:544-546 */
    float* dL_dopacity;   /* [P] */
    float* dL_dcolors;    /* [P,C]   any C (the reference ships C==3 only); see sgb_backward_batch for sharing */
    float* dL_dmeans3D;   /* [P,3] */
    float* dL_dcov3D;     /* [P,6] */
    float* dL_dsh;        /* [P,M,3] or NULL when shs is NULL */
    float* dL_dscales;    /* [P,3]  or NULL when scales is NULL */
    float* dL_drotations; /* [P,4]  or NULL when rotations is NULL */
} sgb_view_grads;

const char* sgb_last_error(void);
const char* sgb_version(void);

int sgb_ctx_create(sgb_ctx** out, int device);
void sgb_ctx_destroy(sgb_ctx* ctx);
/* Bytes of device scratch the ctx currently holds (diagnostics). */
size_t sgb_ctx_scratch_bytes(const sgb_ctx* ctx);

/* Stage tracing: when enabled, every stage of the calls made through this ctx is bracketed by a
 * CUDA event pair on the caller's stream.  sgb_profile_read synchronises those events and returns,
 * per stage, the summed milliseconds and the number of intervals since the previous read
 * (arrays of sgb_profile_num_stages() entries).  At most 128 intervals per stage are kept. */
int sgb_profile_enable(sgb_ctx* ctx, int on);
int sgb_profile_read(sgb_ctx* ctx, float* ms_sum, int32_t* count);
int sgb_profile_num_stages(void);
const char* sgb_profile_stage_name(int stage);
/* Kernels of this library launched through ctx so far (library_calls = 0), or the number of
 * CUB device-wide calls (library_calls = 1; each is several kernels). */
uint64_t sgb_ctx_launch_count(const sgb_ctx* ctx, int library_calls);
/* Statistics of the most recent C > 4 view rendered through ctx (no synchronisation: the values were read
 * back with the weight-pool header).  which = 0: blended (pixel, Gaussian) pairs, i.e. n-bar * W * H, the
 * quantity the blend's algorithmic flops scale with; 1: 16-entry weight-row chunks in use.  -1 if unknown. */
int64_t sgb_ctx_view_stat(const sgb_ctx* ctx, int which);
/* Optional cudaEvent_t that sgb_backward records on its stream as soon as dL_dcolors (the (P, C)
 * feature gradient — the only large per-Gaussian gradient) is final, i.e. BEFORE the chain and
 * geometry gradient kernels.  A data-parallel caller lets its communication stream wait on this
 * event so that the all-reduce of the feature gradient overlaps the rest of the backward pass
 * (the reference is single-GPU and has no counterpart).  NULL (default) disables it. */
int sgb_ctx_set_feature_grad_event(sgb_ctx* ctx, void* cuda_event);

/* Sizes of the three caller-owned state buffers (multiples of 256 B). */
size_t sgb_geometry_bytes(int32_t P);
size_t sgb_binning_bytes(int64_t num_rendered);
size_t sgb_image_bytes(int32_t W, int32_t H);

/*
 * Stage 1 of forward: per-Gaussian projection / covariance / conic / radius / tile rect / SH
 * colour (forward.cu:155-256), depth ordering and the scan over tiles_touched
 * (rasterizer_impl.cu:279).  Writes `radii` [P] int32 and *num_rendered_host (instances R).
 */
int sgb_forward_geometry(sgb_ctx* ctx, const sgb_view_inputs* in, void* geometry_state,
                         int32_t* radii, int64_t* num_rendered_host, void* stream);

/*
 * Stage 2 of forward: instance emission, tile sort, tile ranges (rasterizer_impl.cu:291-321) and
 * the per-tile front-to-back blend (forward.cu:262-375; rgbd/forward.cu:261-393 when out_depth
 * is non-NULL).  out_color [C,H,W]; out_depth [1,H,W] or NULL.  Every pixel is written, so the
 * outputs need no zero-fill.
 */
int sgb_forward_render(sgb_ctx* ctx, const sgb_view_inputs* in, int64_t num_rendered,
                       void* geometry_state, void* binning_state, void* image_state,
                       const int32_t* radii, float* out_color, float* out_depth, void* stream);

/* backward.cu:394-552 (blend), :141-271 (cov2D), :341-391 (projection / SH / scale+rot). */
int sgb_backward(sgb_ctx* ctx, const sgb_view_inputs* in, int64_t num_rendered,
                 const int32_t* radii, const void* geometry_state, const void* binning_state,
                 const void* image_state, const float* dL_dpix /* [C,H,W] */,
                 const sgb_view_grads* grads, void* stream);

/* ---- batched views (BASELINE config K4): V views of the SAME Gaussians in one call.
 *
 * The reference renders one view per call in a Python loop (eval_segmentation.py:146-157, fusion.py:58-64,106-144);
 * a view-sharded training / evaluation step renders a batch of views per GPU (K4: 32 views over 8 GPUs = 4 each).
 * `in` carries everything the views share (sizes, Gaussian arrays, background, flags); its camera fields are
 * ignored and replaced by cams[v].  Per view the results are IDENTICAL to V single-view calls; what the batch
 * removes is per-view overhead:
 *   - sgb_forward_geometry_batch enqueues the V projection / depth-order / scan sequences back to back and
 *     synchronises the stream ONCE for all V instance counts (the single-view call synchronises per view);
 *   - sgb_forward_render_batch enqueues binning, alpha pass and blend of all V views and synchronises ONCE for
 *     the V weight-pool checks; every view keeps its own weight-pool slot inside the ctx (V <= SGB_MAX_BATCH),
 *     so sgb_backward_batch reuses the rows of all V forwards;
 *   - sgb_backward_batch accumulates: with colors_precomp, grads[v].dL_dcolors may be THE SAME (P, C) buffer for
 *     every view — the per-Gaussian feature gradient is summed over the local views in place (one zero-fill, no
 *     V x (P, C) temporaries, no V-way add), which is what a data-parallel step exchanges.  With shs it may not:
 *     view v's geometry kernel reads dL_dcolors as view v's RGB gradient, so every view needs its own buffer, and
 *     a call whose views share one returns SGB_E_INVALID before anything is enqueued.  All V dL/dfeature kernels run
 *     first, then the feature-gradient event (sgb_ctx_set_feature_grad_event) is recorded, then the V chain /
 *     geometry kernels: the exchange of the big gradient overlaps the rest of the whole batch.  The small
 *     per-Gaussian gradients (means2D, conic, opacity, means3D, cov3D, scales, rotations, sh) are per view
 *     (distinct buffers per grads[v]; viewspace gradients feed per-view densification statistics).
 */
#define SGB_MAX_BATCH 8

typedef struct sgb_camera {
    const float* viewmatrix;     /* [16] device */
    const float* projmatrix;     /* [16] device */
    const float* campos;         /* [3]  device */
    float tan_fovx, tan_fovy;
} sgb_camera;

int sgb_forward_geometry_batch(sgb_ctx* ctx, const sgb_view_inputs* in, int32_t V, const sgb_camera* cams,
                               void* const* geometry_states, int32_t* const* radii,
                               int64_t* num_rendered_host /* [V] */, void* stream);
int sgb_forward_render_batch(sgb_ctx* ctx, const sgb_view_inputs* in, int32_t V, const sgb_camera* cams,
                             const int64_t* num_rendered /* [V] host */, void* const* geometry_states,
                             void* const* binning_states, void* const* image_states,
                             const int32_t* const* radii, float* const* out_colors,
                             float* const* out_depths /* NULL or [V] (C <= 4 only) */, void* stream);
int sgb_backward_batch(sgb_ctx* ctx, const sgb_view_inputs* in, int32_t V, const sgb_camera* cams,
                       const int64_t* num_rendered, const int32_t* const* radii,
                       const void* const* geometry_states, const void* const* binning_states,
                       const void* const* image_states, const float* const* dL_dpix,
                       const sgb_view_grads* grads /* [V] */, void* stream);

/* ---- differentiable expected depth and accumulated opacity (C <= 4 only).
 *
 * Per pixel, over the Gaussians the blend composites, in blend order, with w_i = alpha_i T_i as the forward
 * computes it and z_i the view-space depth of the Gaussian's centre (the "depths" state field, the value the median
 * depth uses):
 *     expected depth  E = sum_i w_i z_i        accumulated opacity  A = sum_i w_i
 * with no background term.  Both are accumulated with the colour channels' own statement, so they are bit for bit
 * the blend of a feature [z, 1] over background 0.  A caller's normalised depth is E / max(A, eps).
 *
 * sgb_forward_render_batch_ext is sgb_forward_render_batch plus out_exp_depths and out_alphas ([V] arrays of [1,H,W]
 * planes), given together or both NULL.  sgb_backward_batch_ext is sgb_backward_batch plus the upstream gradients
 * dL_dexp_depth and dL_dalpha ([V] arrays of [1,H,W] planes, each NULL when absent): E and A are two more channels
 * with features z_i and 1 over background 0, so their gradients reach means2D, conic and opacity through the colour
 * channels' paths, and dL/dz_i = sum_p w_ip dL/dE_p reaches dL_dmeans3D through the view transform.  The per-view
 * dL/dz lives in ctx scratch.  The non-_ext calls are these with NULL arrays.  C > 4 with any of the new arrays
 * returns SGB_E_INVALID before anything is enqueued. */
int sgb_forward_render_batch_ext(sgb_ctx* ctx, const sgb_view_inputs* in, int32_t V, const sgb_camera* cams,
                                 const int64_t* num_rendered /* [V] host */, void* const* geometry_states,
                                 void* const* binning_states, void* const* image_states,
                                 const int32_t* const* radii, float* const* out_colors,
                                 float* const* out_depths /* NULL or [V] */,
                                 float* const* out_exp_depths /* NULL or [V] */,
                                 float* const* out_alphas /* NULL or [V] */, void* stream);
int sgb_backward_batch_ext(sgb_ctx* ctx, const sgb_view_inputs* in, int32_t V, const sgb_camera* cams,
                           const int64_t* num_rendered, const int32_t* const* radii,
                           const void* const* geometry_states, const void* const* binning_states,
                           const void* const* image_states, const float* const* dL_dpix,
                           const float* const* dL_dexp_depth /* NULL or [V] */,
                           const float* const* dL_dalpha /* NULL or [V] */,
                           const sgb_view_grads* grads /* [V] */, void* stream);

/* ---- colour and a feature field in one pass: what a joint RGB + feature training step renders.
 *
 * sgb_forward_render_joint_batch is sgb_forward_render_batch_ext of the RGB render in `in` (C = 3, shs or
 * colors_precomp, RGB background; out_depths required, out_exp_depths / out_alphas as there, given together or not
 * at all) that ALSO writes out_features[v] (c, H, W): the render of the second colour table `features` (P, c) over
 * `bg_features` (c), bit for bit what sgb_forward_render_batch gives with colors_precomp = features.  Both images come
 * from one geometry state per view (one sgb_forward_geometry_batch call with the RGB inputs) and ONE binning per view.
 * For c > 4 one walk of the view's tile lists is both the RGB blend and the alpha pass that builds the feature image's
 * weight pool; the forward contraction follows the one weight-pool check of the batch.  For c <= 4 the small-C blend
 * runs once per image on the same lists.  Any c >= 1.
 *
 * sgb_backward_joint_batch is the backward of both images: per view dL/dfeature (c > 4, every view first, then the
 * feature-gradient event), the feature image's chain / blend backward, the RGB blend backward (with the
 * dL_dexp_depth / dL_dalpha terms when given) and ONE geometry backward with the RGB colour gradient.  The two
 * blend backwards add into the same grads[v].dL_dmeans2D / dL_dconic / dL_dopacity, so those hold the sum of both
 * images' gradients.  dL_dfeatures (P, c) is accumulated over the views (caller zero-fills); grads[v].dL_dcolors is
 * the RGB colour gradient with sgb_backward_batch's sharing rule (with shs every view needs its own).
 *
 * Both calls return SGB_E_INVALID before enqueuing anything for: in->C != 3, c < 1, a null feature table, feature
 * background, output (median depth included) or upstream array or entry, shared dL_dcolors under shs,
 * out_exp_depths without out_alphas or the reverse, and every argument rule of the RGB entry points.  Neither
 * synchronises beyond what
 * sgb_forward_render_batch does (one sync for the weight-pool checks when c > 4; the backward syncs only when it must
 * rebuild a pool its forward no longer holds). */
int sgb_forward_render_joint_batch(sgb_ctx* ctx, const sgb_view_inputs* in, int32_t V, const sgb_camera* cams,
                                   const int64_t* num_rendered /* [V] host */, void* const* geometry_states,
                                   void* const* binning_states, void* const* image_states,
                                   const int32_t* const* radii, float* const* out_colors,
                                   float* const* out_depths /* [V] */,
                                   float* const* out_exp_depths /* NULL or [V] */,
                                   float* const* out_alphas /* NULL or [V] */, const float* features /* (P, c) */,
                                   int32_t c, const float* bg_features /* (c) */,
                                   float* const* out_features /* [V] (c, H, W) */, void* stream);
int sgb_backward_joint_batch(sgb_ctx* ctx, const sgb_view_inputs* in, int32_t V, const sgb_camera* cams,
                             const int64_t* num_rendered, const int32_t* const* radii,
                             const void* const* geometry_states, const void* const* binning_states,
                             const void* const* image_states, const float* const* dL_dpix /* [V] (3, H, W) */,
                             const float* const* dL_dexp_depth /* NULL or [V] */,
                             const float* const* dL_dalpha /* NULL or [V] */,
                             const sgb_view_grads* grads /* [V] */, const float* features /* (P, c) */, int32_t c,
                             const float* bg_features /* (c) */,
                             const float* const* dL_dfeature_pix /* [V] (c, H, W) */,
                             float* dL_dfeatures /* (P, c) */, void* stream);

/* ---- camera gradients: what camera pose refinement needs from the backward.
 *
 * sgb_backward_batch_cam is sgb_backward_batch_ext, and sgb_backward_joint_batch_cam sgb_backward_joint_batch, that
 * also write, for every view v with cam_grads non-NULL, the gradient of the loss with respect to that view's camera:
 * cam_grads[v].dL_dviewmatrix [16], dL_dprojmatrix [16] and dL_dcampos [3], device fp32, in the element order of
 * sgb_camera's viewmatrix / projmatrix / campos.  The geometry backward of the view forms every visible Gaussian's
 * contribution (through the view-space centre and the perspective Jacobian, the projected centre, the expected
 * depth when dL_dexp_depth / dL_dalpha are given, and the SH view direction when shs is given) and sums them:
 *   - fp64 partials per CTA in ctx scratch, then one fixed-order pass that writes fp32 once: no float atomics, so
 *     identical calls give bitwise-identical camera gradients;
 *   - the outputs are overwritten, not accumulated; entries the forward never reads (viewmatrix 3, 7, 11, 15 and
 *     projmatrix 2, 6, 10, 14) are exactly 0, and so is dL_dcampos without shs; a view with P = 0 or no instance
 *     gets zeros;
 *   - focal lengths and tan(fov) are constants (no intrinsics gradient);
 *   - a joint call's one geometry backward per view carries both images' losses, and so does its camera gradient;
 *   - every per-Gaussian gradient is bitwise what the same call with cam_grads = NULL writes.
 * Besides the argument rules of the call it extends, a null pointer in any entry, or one pointer used for two
 * outputs, returns SGB_E_INVALID before anything is enqueued.  The camera-gradient reduction is timed inside the
 * geom_bwd profiler stage. */
typedef struct sgb_camera_grads {
    float* dL_dviewmatrix;  /* [16] device, element order of sgb_camera.viewmatrix */
    float* dL_dprojmatrix;  /* [16] device */
    float* dL_dcampos;      /* [3]  device */
} sgb_camera_grads;

int sgb_backward_batch_cam(sgb_ctx* ctx, const sgb_view_inputs* in, int32_t V, const sgb_camera* cams,
                           const int64_t* num_rendered, const int32_t* const* radii,
                           const void* const* geometry_states, const void* const* binning_states,
                           const void* const* image_states, const float* const* dL_dpix,
                           const float* const* dL_dexp_depth /* NULL or [V] */,
                           const float* const* dL_dalpha /* NULL or [V] */,
                           const sgb_view_grads* grads /* [V] */,
                           const sgb_camera_grads* cam_grads /* NULL or [V], host array */, void* stream);
int sgb_backward_joint_batch_cam(sgb_ctx* ctx, const sgb_view_inputs* in, int32_t V, const sgb_camera* cams,
                                 const int64_t* num_rendered, const int32_t* const* radii,
                                 const void* const* geometry_states, const void* const* binning_states,
                                 const void* const* image_states, const float* const* dL_dpix /* [V] (3, H, W) */,
                                 const float* const* dL_dexp_depth /* NULL or [V] */,
                                 const float* const* dL_dalpha /* NULL or [V] */,
                                 const sgb_view_grads* grads /* [V] */, const float* features /* (P, c) */,
                                 int32_t c, const float* bg_features /* (c) */,
                                 const float* const* dL_dfeature_pix /* [V] (c, H, W) */,
                                 float* dL_dfeatures /* (P, c) */,
                                 const sgb_camera_grads* cam_grads /* NULL or [V], host array */, void* stream);

/* Identity of the build: "<version> src:<sha256 prefix of csrc/ + include/>" (set by build.py; bench.py prints
 * it so that a stale prebuilt library cannot be mistaken for the sources next to it). */
const char* sgb_build_id(void);

/* rasterizer_impl.cu:54-66,141-153: present[i] = (view-space z > 0.2). present is uint8 [P]. */
int sgb_mark_visible(int32_t P, const float* means3D, const float* viewmatrix,
                     const float* projmatrix, uint8_t* present, void* stream);

/* Named read-only views into the opaque state, for tests and diagnostics.  Copies the field
 * into dst (device) and returns the byte count, or a negative error.  Fields: "depths",
 * "means2D", "conic_opacity", "cov3D", "rgb", "clamped", "tiles_touched", "point_list",
 * "ranges", "n_contrib", "final_T". */
int64_t sgb_state_field(const char* name, int32_t P, int64_t num_rendered, int32_t W, int32_t H,
                        const void* geometry_state, const void* binning_state,
                        const void* image_state, void* dst, void* stream);

/* ------------------------------------------------------------------ fusion (2D -> 3D) ---- */

#define SGB_DEPTH_NONE 0     /* fusion.depth == None   : keep points with z > 0          */
#define SGB_DEPTH_F32 1      /* depth map float32 [h,w] ("render", fusion.py:106-120)     */
#define SGB_DEPTH_F64 2      /* depth map float64 [h,w] ("image": png / depth_scale)      */
#define SGB_DEPTH_SURFACE 3  /* z-buffer of the points themselves (fusion_utils.py:57-61) */

#define SGB_FEAT_F16 0
#define SGB_FEAT_F32 1
#define SGB_FEAT_BF16 2   /* the half-precision sparse convolution, and the output of the split voxel feature loss;
                             no feature loss accepts it as a target */

typedef struct sgb_fusion_view {
    int32_t P;
    const float* xyz;            /* [P,3] */
    const float* world_to_camera;/* [16] = view.world_view_transform (W2C transposed), f32 */
    double fx, fy, cx, cy;       /* intrinsics AFTER the img_dim rescale of fusion_utils.py:23-28 */
    int32_t w, h;                /* image_dim = [w, h] */
    int32_t cut_bound;
    double vis_thres;
    int32_t depth_mode;
    const void* depth;           /* [h,w] f32 or f64 per depth_mode, or NULL */
} sgb_fusion_view;

/* compute_mapping: mapping int64 [P,3] = (v, u, mask) exactly as fusion_utils.py:73-78. */
int sgb_fusion_map(sgb_ctx* ctx, const sgb_fusion_view* v, int64_t* mapping, void* stream);

/*
 * One fused view of fusion.py:127-144 without the host round trip: project, test, gather the
 * C-channel pixel feature from `features` ([C,h,w], f16 or f32) and add it into feat_sum [P,C]
 * f32; count [P] f32 += 1 for every visible Gaussian.  n_visible_dev (int32, device, may be
 * NULL) receives the number of visible Gaussians of this view.
 */
int sgb_fusion_accumulate(sgb_ctx* ctx, const sgb_fusion_view* v, const void* features,
                          int32_t C, int32_t feat_dtype, float* feat_sum, float* count,
                          int32_t* n_visible_dev, void* stream);

/* fusion.py:146-147: count[count==0] = 1e-5; feat_sum /= count (in place). */
int sgb_fusion_normalize(int32_t P, int32_t C, float* feat_sum, float* count, void* stream);

/* ---- lifting feature maps onto the Gaussians by their blend weights (the adjoint of rendering).
 *
 * For V views of the same Gaussians (V <= SGB_MAX_BATCH), with w_i^v(p) = alpha_i T_i as the forward blend computes it
 * (0 where the walk skips Gaussian i at pixel p or has stopped) and no background term:
 *     feat_sum[i][c] += sum_v sum_p w_i^v(p) map_v[c][p]          weight_sum[i] += sum_v sum_p w_i^v(p)
 * feat_sum is what sgb_backward's dL_dcolors would receive with dL/dout = map_v.  sgb_fusion_normalize(P, C,
 * feat_sum, weight_sum) then gives each Gaussian the weighted mean of the pixels it shows in, a convex combination of
 * map values (0 for a Gaussian that no pixel shows).  Occlusion comes from the transmittance: no depth test.
 *
 * in: P, W, H, C (the map channels, any C >= 1), means3D, opacities, scales + rotations or cov3D_precomp,
 * scale_modifier, prefiltered, debug; shs, colors_precomp and background must be NULL; the camera fields are ignored
 * (cams[v] is view v).  maps[v]: (C, H, W) contiguous, SGB_FEAT_F16 or SGB_FEAT_F32, any 2-byte / 4-byte alignment
 * (fp16 maps are read as fp16 and widened on chip; sums are fp32).  feat_sum (P, C) and weight_sum (P) fp32 are
 * accumulated into: the caller zero-fills them once and may lift any number of calls into them.
 * Per view: geometry, binning and the alpha pass (weight pool) of the C > 4 blend, then the dL/dfeature contraction
 * with the map as dL/dout and a pass over the weight rows; never the colour blend, the chain or the geometry backward.
 * The per-view states live in ctx scratch and nothing outlives the call; the weight-pool slots it took are left empty,
 * and a later sgb_backward_batch rebuilds the rows of any forward whose slot it took.  The host synchronises twice, as
 * sgb_forward_geometry_batch + sgb_forward_render_batch do: once for the V instance counts, once for the V weight-pool
 * checks (plus one per rebuilt pool when a pool overflows).  Bad arguments return SGB_E_INVALID before anything is
 * enqueued: V outside 1..SGB_MAX_BATCH, C < 1, an unknown map_dtype, a null array or map, shs / colors_precomp /
 * background given, or the forward's scale/rotation-versus-cov3D_precomp rule. */
int sgb_lift_batch(sgb_ctx* ctx, const sgb_view_inputs* in, int32_t V, const sgb_camera* cams,
                   const void* const* maps /* [V] (C,H,W) */, int32_t map_dtype /* SGB_FEAT_F16 | SGB_FEAT_F32 */,
                   float* feat_sum /* (P,C) */, float* weight_sum /* (P) */, void* stream);

/* ---- semantic head: what every render_chn caller runs on the rendered feature image.
 *
 * sgb_semantic_head: render (C, N) planar fp32 with N = H*W, text (K, C) row-major:
 *     sim[k][p]  = sum_c text[k][c] * render[c][p] / (||render[:, p]||_2 + 1e-8)   eval_segmentation.py:155-156
 *     label[p]   = argmax_{k >= first_class} sim[k][p] - first_class                eval_segmentation.py:157
 * in ONE pass over the image.  sim (K, N) and label (N, int64) are optional (NULL to skip; a label-only
 * call never writes the K planes).  ctx is needed only for K > 32 with a label map (scratch), else may be NULL.
 *
 * sgb_feature_logits: out[p][k] = sum_c features[p][c] * text[k][c]  (einsum "cq,dq->dc",
 * eval_segmentation.py:132, view_viser.py:185) with row pitch Kpad >= K, columns K..Kpad-1 zeroed — blending is
 * linear, so rendering these Kpad channels gives the un-normalised similarities (and hence the label map)
 * without ever materialising the (C, H, W) feature image.
 *
 * sgb_label_argmax: label[p] = argmax_{first_class <= k < K} planes[k][p] - first_class
 * (rendering[1:].argmax(dim=0), eval_segmentation.py:144). */
/* Distillation loss of a rendered feature image against per-pixel class embeddings and its gradient, one pass:
 *     loss = -(1 / (C Nv)) sum_p <render[:, p], class_emb[label(p)]>,   dL_drender[c][p] = -class_emb[label(p)][c] / (C Nv)
 * render / dL_drender (C, N) planar fp32, class_emb (K, C), labels (N) int32 or int64.  A label outside [0, K)
 * (e.g. -1 / 255 "unannotated") marks an IGNORED pixel: zero gradient, no loss term, not counted in the normaliser
 * Nv = number of valid pixels (Nv = N when every label is in range).
 * loss: TWO doubles on the device (zeroed by the call): [0] the loss, [1] Nv. */
int sgb_distill_loss(int32_t C, int32_t K, int64_t N, const float* render, const float* class_emb, const void* labels,
                     int32_t labels_are_int64, float* dL_drender, double* loss, void* stream);
/* Distillation loss of a rendered feature image against a 2D model's feature map (distill.py:111-124) and its
 * gradient.  render / dL_drender (C, N) planar fp32, target (C, N) planar, SGB_FEAT_F16 or SGB_FEAT_F32; pixel p is
 * the row x_p = render[:, p], y_p = target[:, p] (converted to fp32):
 *     SGB_FEATLOSS_COSINE  loss = (1 / Nv) sum_{p valid} (1 - cos_p),  cos_p = x_p.y_p / (max(|x_p|, 1e-8) max(|y_p|, 1e-8))
 *                          (torch.nn.CosineSimilarity), dL_drender its torch autograd gradient on valid pixels and
 *                          0 elsewhere.  Valid: y_p has a non-zero element; Nv = the number of valid pixels.
 *                          Nv = 0 gives loss 0 and an all-zero gradient.
 *     SGB_FEATLOSS_L1      loss = (1 / (N C)) sum |x - y|,     dL_drender = sign(x - y) / (N C), sign(0) = 0
 *     SGB_FEATLOSS_L2      loss = (1 / (N C)) sum (x - y)^2,   dL_drender = 2 (x - y) / (N C)
 * loss: TWO doubles on the device (zeroed by the call): [0] the loss, [1] the pixels the mean runs over (Nv for
 * cosine, N for l1 / l2), so a caller can skip an empty step without a host sync.  1 <= C <= 1024.  Each input is
 * read once and dL_drender written once.  Asynchronous on `stream`, no host copy, no ctx; N == 0 only zeroes loss. */
#define SGB_FEATLOSS_COSINE 0
#define SGB_FEATLOSS_L1 1
#define SGB_FEATLOSS_L2 2
int sgb_feature_map_loss(int32_t C, int64_t N, const float* render, const void* target,
                         int32_t target_dtype /* SGB_FEAT_F16 | SGB_FEAT_F32 */, int32_t loss_type,
                         float* dL_drender, double* loss /* [2] device: loss, Nv; zeroed by the call */,
                         void* stream);
/* The same loss on a compact rendered field through a per-pixel linear decoder (a 1x1 conv / nn.Linear(c, C)), with
 * every gradient, without materialising the decoded (C, N) image.  render / dL_drender (c, N) planar fp32, weight /
 * dL_dweight (C, c) row-major fp32 (nn.Linear(c, C).weight), bias / dL_dbias (C) fp32 or both NULL, target (C, N)
 * planar, SGB_FEAT_F16 or SGB_FEAT_F32.  Per pixel x_p = weight render[:, p] + bias, and the loss on x against the
 * target is exactly that of sgb_feature_map_loss (same loss_type values, the same loss[2] output).  With g_p = dLoss/dx_p:
 *     dL_drender[:, p] = weight^T g_p      dL_dweight = sum_p g_p render[:, p]^T      dL_dbias = sum_p g_p
 * dL_dweight and dL_dbias are overwritten, not added to.  workspace: caller-allocated device scratch of
 * sgb_decoded_feature_loss_workspace_bytes(C, c, N) bytes, 16-byte aligned (it depends on C and c only).  Every output
 * is bitwise identical from call to call (no float atomics).  1 <= C <= 1024, 1 <= c <= 128; a bad argument returns
 * SGB_E_INVALID before anything is enqueued.  Asynchronous on `stream`, no host copy, no ctx; N == 0 only zeroes loss,
 * dL_dweight and dL_dbias.  The workspace-size call returns 0 for C, c or N outside those limits. */
size_t sgb_decoded_feature_loss_workspace_bytes(int32_t C, int32_t c, int64_t N);
int sgb_decoded_feature_loss(int32_t C, int32_t c, int64_t N, const float* render, const float* weight,
                             const float* bias /* NULL */, const void* target,
                             int32_t target_dtype /* SGB_FEAT_F16 | SGB_FEAT_F32 */, int32_t loss_type,
                             float* dL_drender, float* dL_dweight, float* dL_dbias /* NULL iff bias NULL */,
                             void* workspace, double* loss /* [2] device: loss, pixels averaged over */, void* stream);
/* The same three losses on the masked rows of a 3D network's (M, F) row-major fp32 output (MinkUNet's .F), as
 * distill.py:111-124 takes them: x_k = output[i_k, head*C : head*C + C] for the k-th row i_k with mask[i_k] != 0, and
 * target (K, C) row-major (one row per masked output row, in row order; SGB_FEAT_F16 or SGB_FEAT_F32, converted to
 * fp32).  cosine averages over the Nv target rows with a non-zero element, l1 / l2 over K * C.  grad (M, F) fp32 is
 * overwritten: d loss / d output on the head's columns of masked rows, 0 everywhere else.  loss (device, 2 doubles)
 * receives the loss and the count averaged over (Nv for cosine, K for l1 / l2); both are 0 when nothing is averaged
 * over, and both are NaN when the mask selects other than K rows.  workspace: device scratch of
 * sgb_voxel_feature_loss_workspace_bytes(M) bytes, 16-byte aligned.  Every output is bitwise identical from call to
 * call (no float atomics).  0 <= M <= 2^31 - 1, 0 <= K <= M, 1 <= C <= 1024, head >= 0, head*C + C <= F; a bad
 * argument returns SGB_E_INVALID before anything is enqueued.  Asynchronous on `stream`, no host copy, no ctx.  The
 * workspace-size call returns 0 for M outside those limits. */
size_t sgb_voxel_feature_loss_workspace_bytes(int64_t M);
int sgb_voxel_feature_loss(int64_t M, int32_t F, const float* output, const uint8_t* mask /* (M) bool */, int64_t K,
                           int32_t C, int32_t head, const void* target,
                           int32_t target_dtype /* SGB_FEAT_F16 | SGB_FEAT_F32 */, int32_t loss_type, float* grad,
                           void* workspace, double* loss /* [2] device: loss, count */, void* stream);
/* The same loss split into a forward and a gradient pass, for an output in its own dtype (output_dtype
 * SGB_FEAT_F32, SGB_FEAT_F16 or SGB_FEAT_BF16, e.g. MinkUNet's .F under autocast); targets stay SGB_FEAT_F16 /
 * SGB_FEAT_F32.  Half values widen to fp32 exactly, and both passes run sgb_voxel_feature_loss's per-row sums in its
 * order on those fp32 values.
 *   _forward writes loss[2] exactly as sgb_voxel_feature_loss does on output widened to fp32 (the NaN and 0 / 0 cases
 *     included) and no gradient.  It leaves the mask's row flags and ranks and the cosine count in the workspace
 *     (sgb_voxel_feature_loss_workspace_bytes(M) bytes, 16-byte aligned).
 *   _backward reads that workspace, which must hold a _forward pass on the same M, mask and target, and overwrites grad
 *     (M, F) in output_dtype with grad = round(float(*dloss) * g): g the fp32 gradient sgb_voxel_feature_loss writes
 *     for that element (0 outside the masked rows and the head's columns), *dloss the upstream gradient of the loss
 *     (device, one double, e.g. a GradScaler scale).  The scale multiplies the finished g, so for a power-of-two scale
 *     grad is exactly g scaled and rounded once to the output type; for fp32 output and *dloss = 1 it is g bitwise.
 *     Cosine rows recompute x.y, |x|^2 and |y|^2 from output and target; nothing per row is stored between the passes.
 * Argument rules are sgb_voxel_feature_loss's; an unknown output_dtype, a null dloss and an output or grad not aligned
 * to its element size also return SGB_E_INVALID before anything is enqueued.  No float atomics, no host copy, no
 * synchronisation; M == 0 only zeroes loss (_forward) or does nothing (_backward). */
int sgb_voxel_feature_loss_forward(int64_t M, int32_t F, const void* output,
                                   int32_t output_dtype /* SGB_FEAT_F32 | SGB_FEAT_F16 | SGB_FEAT_BF16 */,
                                   const uint8_t* mask /* (M) bool */, int64_t K, int32_t C, int32_t head,
                                   const void* target, int32_t target_dtype /* SGB_FEAT_F16 | SGB_FEAT_F32 */,
                                   int32_t loss_type, void* workspace, double* loss /* [2] device: loss, count */,
                                   void* stream);
int sgb_voxel_feature_loss_backward(int64_t M, int32_t F, const void* output, int32_t output_dtype, int64_t K,
                                    int32_t C, int32_t head, const void* target, int32_t target_dtype,
                                    int32_t loss_type, const void* workspace, const double* dloss /* device, 1 */,
                                    void* grad /* (M, F) in output_dtype */, void* stream);
int sgb_semantic_head(sgb_ctx* ctx, int32_t C, int32_t K, int64_t N, const float* render, const float* text,
                      int32_t first_class, float* sim, int64_t* label, void* stream);
int sgb_feature_logits(int32_t P, int32_t C, int32_t K, int32_t Kpad, const float* features, const float* text,
                       float* out, void* stream);
int sgb_label_argmax(int32_t K, int32_t first_class, int64_t N, const float* planes, int64_t* label, void* stream);
/* The semantic head of a compact field through its linear decoder, without the decoded (C, N) image.  render (c, N)
 * planar fp32, weight (C, c) row-major fp32 (nn.Linear(c, C).weight), bias (C) fp32 or NULL, text (K, C) row-major
 * fp32.  With x_p = weight render[:, p] + bias:
 *     sim[k][p] = sum_C text[k][C] x_p[C] / (||x_p||_2 + 1e-8)                 (sgb_semantic_head on x)
 *     label[p]  = argmax_{first_class <= k < K} sum_C text[k][C] x_p[C] - first_class
 * computed as A render[:, p] + beta with A = text weight, beta = text bias (float64 sums, rounded to fp32 once), and
 * ||x_p||^2 as the float64 quadratic form r^T (W^T W) r + 2 (W^T b) . r + ||b||^2 (a negative rounding counts as 0).
 * The label is the arg-max of the un-normalised numerators (first maximum wins) in both modes, so a label-only call
 * gives the labels of a sim + label call bitwise; it never forms ||x_p|| and never writes K planes.  sim (K, N) and
 * label (N) int64 are optional (NULL to skip).  workspace: caller-allocated device scratch of
 * sgb_decoded_semantic_head_workspace_bytes(C, c, K) bytes, 16-byte aligned (it depends on the widths only).
 * 1 <= C <= 1024, 1 <= c <= 128, 1 <= K <= 1024, 0 <= first_class < K; a bad argument returns SGB_E_INVALID before
 * anything is enqueued.  Every output is bitwise identical from call to call (no float atomics).  Asynchronous on
 * `stream`, no host copy, no ctx; N == 0 or no output does nothing.  The workspace-size call returns 0 for widths
 * outside those limits.
 *
 * sgb_decoded_feature_logits: out[j][k] = text[k] . (weight features[j] + bias) for k < K, row pitch Kpad >= K,
 * columns K..Kpad-1 zero (sgb_feature_logits on the decoded features, which are never formed: it runs
 * feature_logits_kernel on A with beta added to each finished dot product; with bias NULL it is sgb_feature_logits
 * on A).  features (P, c) row-major fp32; the workspace is the head's (same size call).  Same limits and rules. */
size_t sgb_decoded_semantic_head_workspace_bytes(int32_t C, int32_t c, int32_t K);
int sgb_decoded_semantic_head(int32_t C, int32_t c, int32_t K, int64_t N, const float* render, const float* weight,
                              const float* bias /* NULL */, const float* text, int32_t first_class,
                              float* sim /* (K, N) or NULL */, int64_t* label /* (N) or NULL */, void* workspace,
                              void* stream);
int sgb_decoded_feature_logits(int32_t P, int32_t C, int32_t c, int32_t K, int32_t Kpad, const float* features,
                               const float* weight, const float* bias /* NULL */, const float* text,
                               float* out /* (P, Kpad) */, void* workspace, void* stream);

/* ---- segmentation confusion matrix: the counting of utils/metric.py::confusion_matrix, on the device.
 *
 * sgb_confusion_accumulate adds N (prediction, ground truth) pairs into counts, a full (nb, nb) row-major uint64
 * histogram with nb = num_classes + 1 (rows: prediction, columns: ground truth; the caller drops column 0 as the
 * reference does).  For every p:
 *     pr  = pred[p] + pred_offset                 (the reference's `label += 1` is pred_offset = 1)
 *     g   = gt[p]
 *     bin = pr * nb + g                           (exact, 64-bit)
 *     pr < 0 or g < 0 or bin >= nb * nb  ->  *invalid += 1
 *     otherwise                          ->  counts[bin] += 1
 * The reference raises on a view with such a pair (negative bincount input, failed reshape).  The exceptions are a
 * negative g whose flat bin stays >= 0 and labels near 2^63 whose int64 sum wraps into range: numpy silently counts
 * those in the wrong cell, and they are invalid here (pr and bin are exact).
 * The upper test is on the flat index, as np.bincount + reshape do: a g > num_classes whose bin still fits counts
 * in the next row.  counts and invalid accumulate across calls; the call never zeroes them.
 * pred: SGB_LABEL_I32 or SGB_LABEL_I64; gt: SGB_LABEL_U8, SGB_LABEL_I32 or SGB_LABEL_I64.  pred / gt may have any
 * alignment (views into larger tensors).  1 <= num_classes <= 225: (num_classes + 1)^2 uint32 bins must fit one
 * CTA's shared memory.  Enqueued on `stream`, no host synchronisation, no ctx.  N == 0 launches nothing. */
#define SGB_LABEL_U8 0
#define SGB_LABEL_I32 1
#define SGB_LABEL_I64 2
int sgb_confusion_accumulate(int64_t N, const void* pred, int32_t pred_dtype, const void* gt, int32_t gt_dtype,
                             int32_t pred_offset, int32_t num_classes, uint64_t* counts, uint32_t* invalid,
                             void* stream);

/* ---- voxelization: Voxelizer.voxelize + sparse_quantize of dataset/fusion_utils.py, bit for bit, on the device.
 *
 * For every point p of xyz (P,3) fp32 and the row-major 3x4 fp64 transform T (host memory, 12 doubles):
 *     v[a]  = floor(((x T[4a] + y T[4a+1]) + z T[4a+2]) + T[4a+3])     fp64, every product and sum rounded alone
 *     u[a]  = v[a] - min_p v[a]                                         origin-aligned voxel coordinate
 *     key   = FNV-1a 64 of (u[0], u[1], u[2]): h = 14695981039346656037; per axis h *= 1099511628211, h ^= u[a]
 * and then np.unique(key, return_index=True, return_inverse=True):
 *     first_index[0..M)  the first point of each distinct key, in ascending key order (return_index)
 *     inverse[p]         the rank of p's key among the M distinct keys (return_inverse)
 *     coords[0..M)       (M,3) int32 u of the point first_index[r]
 * Two voxels whose keys collide are one voxel here, as in the reference (the first point's coordinates win).
 *
 * counts (device, 3 int64) receives [0] M, [1] the number of points with a non-finite v (the reference's result is
 * undefined then) and [2] SGB_E_OVERFLOW when an axis spans 2^31 voxels or more (coords are int32), else SGB_OK.
 * The outputs are only meaningful when counts[1] == 0 and counts[2] == SGB_OK; they never index out of range
 * otherwise.  The status words live on the device because the call never synchronises.
 *
 * workspace: device scratch of sgb_voxelize_workspace_bytes(P) bytes, 16-byte aligned.  1 <= P <= 2^31 - 1; a bad
 * argument returns SGB_E_INVALID before anything is enqueued.  Asynchronous on `stream`, no host copy, no ctx; the
 * same inputs give bitwise identical outputs.  The workspace-size call returns 0 for P outside those limits. */
size_t sgb_voxelize_workspace_bytes(int64_t P);
int sgb_voxelize(int64_t P, const float* xyz, const double* transform /* [12] host */, void* workspace,
                 int64_t* first_index /* (P) */, int64_t* inverse /* (P) */, int32_t* coords /* (P,3) */,
                 int64_t* counts /* [3] */, void* stream);
/* The same for a float64 cloud (e.g. after sgb_elastic_displace); the fp32 call's results are those of this one on the
 * fp32 cloud promoted to fp64. */
int sgb_voxelize_f64(int64_t P, const double* xyz, const double* transform /* [12] host */, void* workspace,
                     int64_t* first_index /* (P) */, int64_t* inverse /* (P) */, int32_t* coords /* (P,3) */,
                     int64_t* counts /* [3] */, void* stream);

/* ---- elastic distortion: the per-point half of dataset/augmentation.py ElasticDistortion.elastic_distortion,
 *     out = xyz + RegularGridInterpolator(axes, grid, bounds_error=0, fill_value=0)(xyz) * magnitude
 * bitwise as scipy 1.18 evaluates it (trilinear, fp64, every product and sum rounded alone, corners in
 * itertools.product order, 0 outside the grid, NaN for a point with a NaN coordinate).  xyz (P,3) device, fp32 or fp64
 * (xyz_is_f64); grid (nx,ny,nz,3) fp32 device (the smoothed noise); axes device fp64, nx then ny then nz strictly
 * ascending nodes; out (P,3) fp64 device, which may be xyz itself when xyz is fp64.  1 <= P <= 2^31 - 1, every
 * n >= 2; a bad argument returns SGB_E_INVALID before anything is enqueued.  Asynchronous on `stream`, no host copy. */
int sgb_elastic_displace(int64_t P, const void* xyz, int32_t xyz_is_f64, const float* grid, int32_t nx, int32_t ny,
                         int32_t nz, const double* axes, double magnitude, double* out, void* stream);

/* ---- 3-nearest-neighbour mean squared distance: `distCUDA2` of the reference's
 * simple-knn extension (submodules/simple-knn/simple_knn.cu:185-220, spatial.cu), used by
 * GaussianModel.create_from_pcd (model/gaussian_model.py:150-186).  points (P,3) fp32 device, mean_dist2 (P) fp32
 * device: (d1+d2+d3)/3 of the three smallest squared distances to OTHER points (exact, bit-identical to the
 * reference).  Fewer than 4 points leave FLT_MAX terms, as in the reference. */
int sgb_knn_mean_dist2(sgb_ctx* ctx, int32_t P, const float* points, float* mean_dist2, void* stream);

/* ---- nearest reference point of every query point: label / feature transfer from Gaussians onto scan vertices.
 *
 * For every query q of query_xyz (M,3) fp32 device and every row j of ref_xyz (P,3) fp32 device:
 *     d2(q, j) = (dx*dx + dy*dy) + dz*dz,   dx = q.x - r_j.x, dy = q.y - r_j.y, dz = q.z - r_j.z
 * in fp32, every product and sum rounded alone (no FMA contraction).  Then
 *     index[q] = the j minimising d2(q, j) over the rows with d2(q, j) <= max_dist2; on ties the smallest j
 *     dist2[q] = d2(q, index[q])
 * and a query with no such row gets index -1 and dist2 +inf.  max_dist2 = +inf sets no limit; a negative one matches
 * nothing.  A reference row with a non-finite coordinate is never returned; a query with a non-finite coordinate gets
 * -1.  P == 0 gives -1 everywhere; M == 0 launches nothing.  The result is exact (not approximate), so it does not
 * depend on the order the library visits candidates in.
 *
 * index (M) int64 device, dist2 (M) fp32 device.  Bad arguments return SGB_E_INVALID before anything is enqueued: a
 * null ctx, P or M outside [0, 2^31 - 1], a NaN max_dist2, a null ref_xyz with P > 0, or a null query_xyz / index /
 * dist2 with M > 0.  Uses the ctx's scratch (grown on demand, about 32 (P + M) bytes).  Asynchronous on `stream`, no
 * host synchronisation; the same inputs give bitwise identical outputs. */
int sgb_nearest(sgb_ctx* ctx, int64_t P, const float* ref_xyz, int64_t M, const float* query_xyz, float max_dist2,
                int64_t* index, float* dist2, void* stream);

/* ---- photometric training loss: the RGB loss of the reference's training step (train.py:141-149)
 *     loss = (1 - lambda) * L1(x, y) + lambda * (1 - SSIM(x, y))
 * with SSIM as utils/loss_utils.py:38-72 computes it: an 11x11 Gaussian window (sigma 1.5, fp32 taps divided by
 * their fp32 sum) over zero padding, C1 = 0.01^2, C2 = 0.03^2, averaged over every pixel.
 *
 * x (the rendered image) and y (the target) are `planes` fp32 planes of h x w (one plane = one channel of one
 * image: C planes for (C,H,W), N*C for (N,C,H,W)), each given as a base pointer plus a plane stride and a row
 * stride in elements; the pixel stride is 1.  A border crop (train.py's cut_edge) is thus a pointer offset with
 * the full image's strides.  The plane stride is ignored when planes == 1.
 *
 * sgb_photometric_forward: sums (2 doubles, device, zeroed by the call) receive [0] sum |x - y| and [1] sum of
 * the per-pixel SSIM map over all planes.  partials (device, (3, planes, h, w) fp32, contiguous) receives the
 * three per-pixel maps backward needs; NULL when no gradient is wanted.
 *
 * sgb_photometric_backward: dL_dx[p][r][c] (written through its own strides, only inside the h x w planes) =
 *     coef[0] * sign(x - y) + coef[1] * d(sum SSIM map)/dx
 * with coef (2 floats, DEVICE) = {g (1 - lambda) / n, -g lambda / n} for the loss above (n = planes * h * w,
 * g = the upstream gradient), or {0, g / n} for mean SSIM alone.  sign(0) = 0.
 *
 * Both calls are asynchronous on `stream` and never copy to the host. */
int sgb_photometric_forward(int32_t planes, int32_t h, int32_t w, const float* x, int64_t x_plane_stride,
                            int64_t x_row_stride, const float* y, int64_t y_plane_stride, int64_t y_row_stride,
                            double* sums, float* partials, void* stream);
int sgb_photometric_backward(int32_t planes, int32_t h, int32_t w, const float* x, int64_t x_plane_stride,
                             int64_t x_row_stride, const float* y, int64_t y_plane_stride, int64_t y_row_stride,
                             const float* partials, const float* coef, float* dL_dx, int64_t dx_plane_stride,
                             int64_t dx_row_stride, void* stream);

/* ---- optimizer step: torch.optim.Adam (no amsgrad, no weight_decay, maximize=False) over up to
 * SGB_ADAM_MAX_TENSORS parameter tables in ONE kernel launch, with an optional per-row visibility mask.
 *
 * A tensor is `rows` rows of `row_len` contiguous fp32 values (for a Gaussian table: one row per Gaussian).  Per
 * element of a row that is stepped, in fp32:
 *     m = m + (g - m) * (1 - beta1)          v = beta2 * v + (1 - beta2) * g * g
 *     p = p - step_size * (m / (sqrtf(v) / bias_correction2_sqrt + eps))
 * with IEEE sqrtf and division.  step_size = lr / (1 - beta1^t) and bias_correction2_sqrt = sqrt(1 - beta2^t) are
 * the caller's, computed in double from its step count t.
 *
 * visible: NULL steps every row.  Otherwise row r is stepped where visible[r] != 0; of a row with visible[r] == 0
 * only that byte is read: no element of param / grad / exp_avg / exp_avg_sq is loaded or stored (so they stay
 * bitwise as they were, and a NaN in such a row's gradient is never seen).  This is 3DGS's `sparse_adam` rule, with
 * the bias corrections kept.
 *
 * The descriptors are host memory and travel as kernel parameters: nothing is copied to the device.  Rows are
 * accessed 16 bytes wide where row_len % 4 == 0 and the four base pointers are 16-byte aligned (a tensor without a
 * mask is one flat run, so there rows * row_len % 4 == 0 is enough); any other layout takes a scalar path with the
 * same result.  No ctx, no scratch, no host synchronisation; asynchronous on `stream`; the same inputs give bitwise
 * identical outputs.  Tensors with rows == 0 are skipped and a call with no work launches nothing.
 *
 * SGB_E_INVALID, before anything is enqueued: n outside [0, SGB_ADAM_MAX_TENSORS]; tensors NULL with n > 0; and per
 * tensor rows < 0, row_len < 1, a NULL param / grad / exp_avg / exp_avg_sq with rows > 0, beta1 or beta2 outside
 * [0, 1), eps < 0, a non-finite step_size, bias_correction2_sqrt outside (0, 1]. */
#define SGB_ADAM_MAX_TENSORS 8
typedef struct sgb_adam_tensor {
    float* param;                /* (rows, row_len) */
    const float* grad;           /* (rows, row_len) */
    float* exp_avg;              /* (rows, row_len) first moment m */
    float* exp_avg_sq;           /* (rows, row_len) second moment v */
    const uint8_t* visible;      /* [rows], 0 = skip the row; NULL = every row */
    int64_t rows;
    int32_t row_len;
    double beta1, beta2, eps;    /* double as torch holds them: the kernel uses fp32(1 - beta), not 1 - fp32(beta) */
    float step_size;             /* lr / (1 - beta1^t) */
    float bias_correction2_sqrt; /* sqrt(1 - beta2^t) */
} sgb_adam_tensor;
int sgb_adam_step(const sgb_adam_tensor* tensors_host, int32_t n, void* stream);

/* ---- sparse 3D convolution: the coordinate maps, kernel maps and products of MinkowskiEngine's
 * MinkowskiConvolution / MinkowskiConvolutionTranspose as MinkUNet uses them (sparse.py, mink_unet.py).
 *
 * Coordinates are (N,4) int32 rows (b, x, y, z), 16-byte aligned, 1 <= N <= 2^31 - 1.  A coordinate map at tensor
 * stride t holds rows whose x, y, z are multiples of t.  Its hash table (sgb_coord_map_bytes(N) bytes of device
 * memory) is keyed on all four values: two different rows never share an entry.
 *
 * sgb_coord_map_build: builds the table of `coords`.  status (device, 2 int64, zeroed by the call) receives [0] the
 * number of rows equal to an earlier-inserted row and [1] the number of rows with a negative x, y or z.  The map is
 * only valid when both are 0.
 *
 * sgb_coord_stride: the map at stride 2t from the map at stride t (`stride` = t): rows (b, floor(x / 2t) * 2t, ...),
 * unique, in the order in which their first child row appears in `coords`.  out_coords has room for N rows;
 * out_count (device, 1 int64) receives the row count.  workspace: sgb_coord_stride_workspace_bytes(N) bytes.
 *
 * sgb_kernel_map_count / sgb_kernel_map_fill: the (input row, output row) pairs of kernel size k in {2, 3, 5} over an
 * input map at stride t (`stride`).  Offset index d = jx + k jy + k^2 jz, offset per axis lb + j t with
 * lb = -((k - 1) / 2) t (C division): {-t, 0, t} for k = 3, {0, t} for k = 2.  Output row o pairs with input row i
 * at d when coord(i) = coord(o) + offset and the b values are equal.  count writes offsets (device, k^3 + 1 int64):
 * offset d's pairs are pairs[offsets[d] .. offsets[d+1]).  The caller reads offsets[k^3] to size `pairs` (int32
 * (in, out) pairs, 8 bytes each) and then calls fill with the same arguments and the workspace
 * (sgb_kernel_map_workspace_bytes(N_out, k) bytes) the count call left.  Within an offset the pairs ascend in the
 * output row.  A transposed layer uses the pairs of the matching stride-2 layer with the roles swapped.
 *
 * Products (kernel (K, C_in, C_out) fp32 row-major, 1 <= K <= SGB_SPARSE_MAX_K, C_in, C_out >= 1; offsets_host is
 * the host copy of the kernel map's offsets, pairs may be NULL when offsets_host[K] == 0).  transposed = 0:
 *     forward   out[o] = sum_d x[i] W_d                 over offset d's pairs (i, o)
 *     input     dx[i]  = sum_d dy[o] W_d^T
 *     weight    dW_d   = sum over d's pairs of x[i]^T dy[o]
 * transposed = 1 swaps the roles of i and o (x and dx then live on the pairs' output-row side).  n_in / C_in describe
 * x and dx, n_out / C_out describe out and dy.  out, dx and dkernel are overwritten.  The weight gradient needs
 * sgb_sparse_conv_backward_weight_workspace_bytes(...) bytes of 16-byte aligned workspace.  No float atomics: the
 * same inputs give bitwise identical outputs.
 *
 * Every call validates its arguments (SGB_E_INVALID) before anything is enqueued, is asynchronous on `stream` and
 * never synchronises; the workspace-size calls return 0 for arguments the calls would reject. */
#define SGB_SPARSE_MAX_K 125
size_t sgb_coord_map_bytes(int64_t N);
int sgb_coord_map_build(int64_t N, const int32_t* coords, void* table, int64_t* status /* [2] */, void* stream);
size_t sgb_coord_stride_workspace_bytes(int64_t N);
int sgb_coord_stride(int64_t N, const int32_t* coords, int32_t stride, void* workspace, int32_t* out_coords,
                     int64_t* out_count /* [1] */, void* stream);
size_t sgb_kernel_map_workspace_bytes(int64_t N_out, int32_t k);
int sgb_kernel_map_count(int64_t N_in, const int32_t* in_coords, const void* in_table, int64_t N_out,
                         const int32_t* out_coords, int32_t k, int32_t stride, void* workspace,
                         int64_t* offsets /* [k^3 + 1] */, void* stream);
int sgb_kernel_map_fill(int64_t N_in, const int32_t* in_coords, const void* in_table, int64_t N_out,
                        const int32_t* out_coords, int32_t k, int32_t stride, const void* workspace,
                        int32_t* pairs /* (offsets[k^3], 2) */, void* stream);
int sgb_sparse_conv_forward(int32_t K, const int64_t* offsets_host, const int32_t* pairs, int32_t transposed,
                            int64_t n_in, int32_t C_in, const float* x, const float* kernel, int64_t n_out,
                            int32_t C_out, float* out, void* stream);
int sgb_sparse_conv_backward_input(int32_t K, const int64_t* offsets_host, const int32_t* pairs, int32_t transposed,
                                   int64_t n_in, int32_t C_in, float* dx, const float* kernel, int64_t n_out,
                                   int32_t C_out, const float* dy, void* stream);
size_t sgb_sparse_conv_backward_weight_workspace_bytes(int32_t K, const int64_t* offsets_host, int32_t C_in,
                                                       int32_t C_out);
int sgb_sparse_conv_backward_weight(int32_t K, const int64_t* offsets_host, const int32_t* pairs, int32_t transposed,
                                    int64_t n_in, int32_t C_in, const float* x, int64_t n_out, int32_t C_out,
                                    const float* dy, void* workspace, float* dkernel, void* stream);

/* Half-precision products (sparse_conv_half.cu): the same three products over the same kernel maps (offsets_host,
 * pairs) the fp32 products take, with the same argument rules, on tensor cores.  dtype is SGB_FEAT_F16 or
 * SGB_FEAT_BF16; x, dy, out, dx and the kernel ((K, C_in, C_out) row-major) are in that type.
 *   forward / input: the products of every offset are accumulated in fp32, in offset order, in the workspace
 *     (sgb_sparse_conv_half_{forward,backward_input}_workspace_bytes(...) bytes, 16-byte aligned: one fp32 copy of
 *     out / dx), and each element is rounded to the half type once, at the end.
 *   weight: dkernel is fp32 (the kernel parameter it updates is fp32), accumulated in fp32 in the fp32 product's
 *     chunk partials and summed in chunk order; workspace sgb_sparse_conv_half_backward_weight_workspace_bytes(...).
 * Half x half products are exact in fp32: only the fp32 accumulation (and, for out / dx, the one final rounding)
 * rounds.  Any C_in, C_out >= 1; rows whose width is a multiple of 8 elements take the fast path.  No float atomics:
 * the same inputs give bitwise identical outputs.  Validation, asynchrony and the workspace-size rule are those of
 * the fp32 products. */
size_t sgb_sparse_conv_half_forward_workspace_bytes(int32_t dtype, int32_t K, const int64_t* offsets_host,
                                                    int64_t n_in, int32_t C_in, int64_t n_out, int32_t C_out);
int sgb_sparse_conv_half_forward(int32_t dtype, int32_t K, const int64_t* offsets_host, const int32_t* pairs,
                                 int32_t transposed, int64_t n_in, int32_t C_in, const void* x, const void* kernel,
                                 int64_t n_out, int32_t C_out, void* workspace, void* out, void* stream);
size_t sgb_sparse_conv_half_backward_input_workspace_bytes(int32_t dtype, int32_t K, const int64_t* offsets_host,
                                                           int64_t n_in, int32_t C_in, int64_t n_out, int32_t C_out);
int sgb_sparse_conv_half_backward_input(int32_t dtype, int32_t K, const int64_t* offsets_host, const int32_t* pairs,
                                        int32_t transposed, int64_t n_in, int32_t C_in, void* dx, const void* kernel,
                                        int64_t n_out, int32_t C_out, const void* dy, void* workspace, void* stream);
size_t sgb_sparse_conv_half_backward_weight_workspace_bytes(int32_t dtype, int32_t K, const int64_t* offsets_host,
                                                            int32_t C_in, int32_t C_out);
int sgb_sparse_conv_half_backward_weight(int32_t dtype, int32_t K, const int64_t* offsets_host, const int32_t* pairs,
                                         int32_t transposed, int64_t n_in, int32_t C_in, const void* x, int64_t n_out,
                                         int32_t C_out, const void* dy, void* workspace, float* dkernel,
                                         void* stream);

#ifdef __cplusplus
}
#endif
#endif /* SGB200_H_INCLUDED */
