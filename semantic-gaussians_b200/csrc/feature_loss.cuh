// The feature distillation loss of the reference's distill.py:111-124, defined once for its three fused forms: the
// feature-map loss and the voxel-row loss (feature_loss.cu) and the decoded-feature loss (decoder_loss.cu).
#pragma once

#include <cuda_bf16.h>
#include <cuda_fp16.h>

#include "common.cuh"

namespace sgb {

constexpr int kFeatMaxC = 1024;  // widest feature map accepted (OpenSeg 768, LSeg 512)

// Half values widen to fp32 exactly; from_f32 rounds to nearest even, as torch's .to(dtype) does.
__device__ __forceinline__ float to_f32(float v) { return v; }
__device__ __forceinline__ float to_f32(__half v) { return __half2float(v); }
__device__ __forceinline__ float to_f32(__nv_bfloat16 v) { return __bfloat162float(v); }
template <typename T> __device__ __forceinline__ T from_f32(float v);
template <> __device__ __forceinline__ float from_f32<float>(float v) { return v; }
template <> __device__ __forceinline__ __half from_f32<__half>(float v) { return __float2half_rn(v); }
template <> __device__ __forceinline__ __nv_bfloat16 from_f32<__nv_bfloat16>(float v) { return __float2bfloat16_rn(v); }
// One value of T as fp32, through the read-only cache.
template <typename T> __device__ __forceinline__ float load_f32(const T* p) { return to_f32(__ldg(p)); }

// Four consecutive values as fp32; p is 16- (fp32) or 8-byte (fp16) aligned.
struct Quad { float v[4]; };
__device__ __forceinline__ Quad load4(const float* p) {
    const float4 q = __ldg(reinterpret_cast<const float4*>(p));
    return {{q.x, q.y, q.z, q.w}};
}
__device__ __forceinline__ Quad load4(const __half* p) {
    const uint2 r = __ldg(reinterpret_cast<const uint2*>(p));
    const float2 a = __half22float2(*reinterpret_cast<const __half2*>(&r.x));
    const float2 b = __half22float2(*reinterpret_cast<const __half2*>(&r.y));
    return {{a.x, a.y, b.x, b.y}};
}

// Cosine rule of one row x against its target y, from dot = x.y, xx = |x|^2, yy = |y|^2 (torch.nn.CosineSimilarity
// with eps = 1e-8: each norm clamped separately).  valid: y has a non-zero element (and the row exists); inv_nv =
// 1 / Nv, or 0 when Nv = 0.  The row's gradient is u y + v x; the return value is its loss term 1 - cos, which the
// caller adds to its sum for valid rows only.
__device__ __forceinline__ double cosine_rule(float dot, float xx, float yy, bool valid, float inv_nv, float& u,
                                              float& v) {
    const float nx = sqrtf(xx), a = fmaxf(nx, 1e-8f), b = fmaxf(sqrtf(yy), 1e-8f);
    const float cosv = dot / (a * b);
    // d cos / dx = y / (a b) - cos x / (a |x|): the norm's own derivative x / |x| is unclamped (torch clamps the norms
    // under no_grad), and is zero for x = 0
    u = valid ? -inv_nv / (a * b) : 0.f;
    v = valid && nx > 0.f ? inv_nv * cosv / (a * nx) : 0.f;
    return 1.0 - (double)cosv;
}

// l1 / l2 rule of one element, d = x - y, gs = 1 / M (l1) or 2 / M (l2) over the M elements averaged: g = the
// gradient, sign(d) gs (sign(0) = 0, as abs()'s backward) or gs d; returns the loss term |d| or d^2.
template <int LOSS>
__device__ __forceinline__ float elementwise_rule(float d, float gs, float& g) {
    g = LOSS == SGB_FEATLOSS_L2 ? gs * d : gs * (float)((d > 0.f) - (d < 0.f));
    return LOSS == SGB_FEATLOSS_L2 ? d * d : fabsf(d);
}

// SGB_OK, or SGB_E_INVALID with the error set under `fn` when C is outside [1, kFeatMaxC], target_dtype is not
// SGB_FEAT_F16 / _F32 or loss_type not SGB_FEATLOSS_COSINE / _L1 / _L2.
int check_feature_loss_args(const char* fn, int C, int target_dtype, int loss_type);

// valid[0] += number of pixels of the (C, N) planar target whose column has a non-zero element (the cosine loss's
// Nv).  `valid` must hold 0 (or a count to add to) in stream order before the call.  T = float or __half.
template <typename T>
int count_valid_pixels(int C, long long N, const T* target, double* valid, cudaStream_t s);

}  // namespace sgb
