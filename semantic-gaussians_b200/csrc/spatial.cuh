// Spatial sorting helpers shared by the exact neighbour searches (knn.cu, nearest.cu): axis-aligned boxes, the
// order-preserving float <-> uint mapping their atomic bounds use, and the 30-bit Morton code of a point inside
// those bounds.
#pragma once
#include <cstdint>
#include <cstring>

namespace sgb {

struct Aabb {
    float lo[3], hi[3];
};

// order-preserving float <-> uint mapping for atomicMin / atomicMax
__device__ __forceinline__ uint32_t f2key(float f) {
    const uint32_t b = __float_as_uint(f);
    return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}
__host__ __device__ __forceinline__ float key2f(uint32_t k) {
    const uint32_t b = (k & 0x80000000u) ? (k & 0x7FFFFFFFu) : ~k;
#ifdef __CUDA_ARCH__
    return __uint_as_float(b);
#else
    float f;
    memcpy(&f, &b, 4);
    return f;
#endif
}

__device__ __forceinline__ uint32_t spread10(uint32_t v) {  // abcdefghij -> a00b00c00d00e00f00g00h00i00j
    v &= 0x3FFu;
    v = (v ^ (v << 16)) & 0xFF0000FFu;
    v = (v ^ (v << 8)) & 0x0300F00Fu;
    v = (v ^ (v << 4)) & 0x030C30C3u;
    v = (v ^ (v << 2)) & 0x09249249u;
    return v;
}

// Morton code of p on a 1024^3 grid over the bounds mm = (min keys [3], max keys [3]); outside points clamp.
__device__ __forceinline__ uint32_t morton30(const float* p, const uint32_t* __restrict__ mm) {
    uint32_t q[3];
#pragma unroll
    for (int a = 0; a < 3; a++) {
        const float lo = key2f(mm[a]), hi = key2f(mm[3 + a]);
        const float ext = hi - lo;
        const float t = ext > 0.f ? (p[a] - lo) / ext : 0.f;
        q[a] = (uint32_t)fminf(fmaxf(t * 1023.f, 0.f), 1023.f);
    }
    return spread10(q[0]) | (spread10(q[1]) << 1) | (spread10(q[2]) << 2);
}

}  // namespace sgb
