// Mean squared distance to the 3 nearest neighbours of every point: the contract of
// the reference's `distCUDA2` (submodules/simple-knn/simple_knn.cu:185-220, called from
// model/gaussian_model.py:150-186 create_from_pcd to initialise the Gaussian scales).
//
// The result is exact: out[i] = (d1 + d2 + d3) / 3 with d1 <= d2 <= d3 the three smallest values of
// |p_j - p_i|^2, j != i (other points at the same position count, distance 0), evaluated in fp32 with the
// expression of simple_knn.cu:140-141, so it is bit-identical to the reference whatever the visiting order.
//
// Organisation (not the reference's): points are sorted along a 30-bit Morton curve and physically
// reordered; consecutive runs of 256 sorted points form boxes with an AABB.  One CTA owns one box: its 256
// points sit in registers (one per thread), candidate boxes are staged through shared memory as whole
// tiles (coalesced 16-byte loads, broadcast reads) and are pruned for the WHOLE CTA by the box-to-box
// distance against the largest current third-neighbour distance of the CTA, then per thread by the
// point-to-box distance.  The reference scans every candidate box per thread with dependent gathers
// points[indices[i]].
#include <cfloat>
#include <cub/cub.cuh>
#include "common.cuh"
#include "spatial.cuh"

namespace sgb {

namespace {

constexpr int kBox = 256;

__global__ void knn_bounds_init_kernel(uint32_t* mm) {
    if (threadIdx.x < 3) mm[threadIdx.x] = 0xFFFFFFFFu;       // min keys
    else if (threadIdx.x < 6) mm[threadIdx.x] = 0u;           // max keys
}

__global__ void knn_bounds_kernel(int P, const float* __restrict__ pts, uint32_t* mm) {
    float lo[3] = {FLT_MAX, FLT_MAX, FLT_MAX}, hi[3] = {-FLT_MAX, -FLT_MAX, -FLT_MAX};
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < P; i += gridDim.x * blockDim.x) {
#pragma unroll
        for (int a = 0; a < 3; a++) {
            const float v = pts[3 * (size_t)i + a];
            lo[a] = fminf(lo[a], v);
            hi[a] = fmaxf(hi[a], v);
        }
    }
#pragma unroll
    for (int a = 0; a < 3; a++) {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            lo[a] = fminf(lo[a], __shfl_xor_sync(0xffffffffu, lo[a], o));
            hi[a] = fmaxf(hi[a], __shfl_xor_sync(0xffffffffu, hi[a], o));
        }
    }
    if ((threadIdx.x & 31) == 0) {
#pragma unroll
        for (int a = 0; a < 3; a++) {
            atomicMin(&mm[a], f2key(lo[a]));
            atomicMax(&mm[3 + a], f2key(hi[a]));
        }
    }
}

__global__ void knn_morton_kernel(int P, const float* __restrict__ pts, const uint32_t* __restrict__ mm,
                                  uint32_t* __restrict__ codes, uint32_t* __restrict__ ids) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= P) return;
    codes[i] = morton30(pts + 3 * (size_t)i, mm);
    ids[i] = (uint32_t)i;
}

// sorted, padded copy: ps[i] = (x, y, z, original index); slots >= P hold +inf coordinates
__global__ void knn_gather_kernel(int P, int Ppad, const float* __restrict__ pts, const uint32_t* __restrict__ order,
                                  float4* __restrict__ ps) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= Ppad) return;
    if (i < P) {
        const uint32_t o = order[i];
        ps[i] = make_float4(pts[3 * (size_t)o], pts[3 * (size_t)o + 1], pts[3 * (size_t)o + 2], __uint_as_float(o));
    } else {
        ps[i] = make_float4(INFINITY, INFINITY, INFINITY, __uint_as_float(0xFFFFFFFFu));
    }
}

__global__ void __launch_bounds__(kBox) knn_boxes_kernel(int P, const float4* __restrict__ ps, Aabb* __restrict__ boxes) {
    __shared__ float red[6][kBox / 32];
    const int i = blockIdx.x * kBox + threadIdx.x;
    float v[6] = {FLT_MAX, FLT_MAX, FLT_MAX, -FLT_MAX, -FLT_MAX, -FLT_MAX};
    if (i < P) {
        const float4 p = ps[i];
        v[0] = v[3] = p.x; v[1] = v[4] = p.y; v[2] = v[5] = p.z;
    }
#pragma unroll
    for (int a = 0; a < 6; a++) {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            const float w = __shfl_xor_sync(0xffffffffu, v[a], o);
            v[a] = a < 3 ? fminf(v[a], w) : fmaxf(v[a], w);
        }
        if ((threadIdx.x & 31) == 0) red[a][threadIdx.x >> 5] = v[a];
    }
    __syncthreads();
    if (threadIdx.x < 6) {
        const int a = threadIdx.x;
        float r = red[a][0];
        for (int w = 1; w < kBox / 32; w++) r = a < 3 ? fminf(r, red[a][w]) : fmaxf(r, red[a][w]);
        if (a < 3) boxes[blockIdx.x].lo[a] = r;
        else boxes[blockIdx.x].hi[a - 3] = r;
    }
}

__device__ __forceinline__ void keep3(float (&best)[3], float dist) {  // simple_knn.cu:142-150
#pragma unroll
    for (int j = 0; j < 3; j++) {
        if (best[j] > dist) {
            const float t = best[j];
            best[j] = dist;
            dist = t;
        }
    }
}

__device__ __forceinline__ float box_box_dist2(const Aabb& a, const Aabb& b) {  // lower bound for any pair
    float s = 0.f;
#pragma unroll
    for (int k = 0; k < 3; k++) {
        const float g = fmaxf(0.f, fmaxf(a.lo[k] - b.hi[k], b.lo[k] - a.hi[k]));
        s += g * g;
    }
    return s;
}

__device__ __forceinline__ float point_box_dist2(const Aabb& b, float x, float y, float z) {  // simple_knn.cu:124-134
    const float p[3] = {x, y, z};
    float s = 0.f;
#pragma unroll
    for (int k = 0; k < 3; k++) {
        float d = 0.f;
        if (p[k] < b.lo[k] || p[k] > b.hi[k]) d = fminf(fabsf(p[k] - b.lo[k]), fabsf(p[k] - b.hi[k]));
        s += d * d;
    }
    return s;
}

__global__ void __launch_bounds__(kBox) knn_kernel(int P, const float4* __restrict__ ps, const Aabb* __restrict__ boxes,
                                                   int nboxes, float* __restrict__ out) {
    __shared__ float4 tile[kBox];
    __shared__ float lbs[kBox];
    __shared__ float wmax[kBox / 32];
    __shared__ Aabb cbox;
    const int b = blockIdx.x, t = threadIdx.x;
    const int self = b * kBox + t;
    const bool valid = self < P;
    const float4 me = ps[self];  // padded array: always readable
    const Aabb mybox = boxes[b];
    float best[3] = {FLT_MAX, FLT_MAX, FLT_MAX};

    auto scan_tile = [&](int skip) {  // all 256 slots; padding slots are at +inf and never selected
#pragma unroll 8
        for (int j = 0; j < kBox; j++) {
            const float4 q = tile[j];
            const float dx = q.x - me.x, dy = q.y - me.y, dz = q.z - me.z;
            const float dist = dx * dx + dy * dy + dz * dz;  // simple_knn.cu:140-141
            if (j != skip) keep3(best, dist);
        }
    };
    auto block_max_best = [&]() {  // largest third-neighbour distance among the CTA's real points
        float v = valid ? best[2] : 0.f;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
        __syncthreads();  // previous readers of wmax / tile are done
        if ((t & 31) == 0) wmax[t >> 5] = v;
        __syncthreads();
        float r = wmax[0];
#pragma unroll
        for (int w = 1; w < kBox / 32; w++) r = fmaxf(r, wmax[w]);
        return r;
    };

    tile[t] = me;
    __syncthreads();
    scan_tile(t);
    float reject = block_max_best();

    for (int c0 = 0; c0 < nboxes; c0 += kBox) {
        __syncthreads();  // lbs of the previous group consumed
        lbs[t] = c0 + t < nboxes ? box_box_dist2(mybox, boxes[c0 + t]) : FLT_MAX;
        __syncthreads();
        const int lim = min(kBox, nboxes - c0);
        for (int j = 0; j < lim; j++) {
            const int c = c0 + j;
            // uniform: shared value against a CTA-wide bound.  The own box was done above (with the self
            // test); it must be skipped explicitly — with < 4 points `reject` is still FLT_MAX.
            if (c == b || lbs[j] > reject) continue;
            __syncthreads();  // tile / cbox free
            tile[t] = ps[(size_t)c * kBox + t];
            if (t == 0) cbox = boxes[c];
            __syncthreads();
            if (valid && !(point_box_dist2(cbox, me.x, me.y, me.z) > best[2])) scan_tile(-1);
            reject = block_max_best();
        }
    }
    if (valid) out[__float_as_uint(me.w)] = (best[0] + best[1] + best[2]) / 3.0f;  // simple_knn.cu:183
}

}  // namespace

}  // namespace sgb

using namespace sgb;

extern "C" int sgb_knn_mean_dist2(sgb_ctx* ctx, int32_t P, const float* points, float* mean_dist2, void* stream) {
    cudaStream_t s = (cudaStream_t)stream;
    if (!ctx || P < 0) { set_error("sgb_knn_mean_dist2: null ctx or negative P"); return SGB_E_INVALID; }
    if (P == 0) return SGB_OK;
    if (!points || !mean_dist2) { set_error("sgb_knn_mean_dist2: null argument"); return SGB_E_INVALID; }
    const int nboxes = (P + kBox - 1) / kBox;
    const int Ppad = nboxes * kBox;
    size_t sort_tmp = 0;
    cub::DeviceRadixSort::SortPairs(nullptr, sort_tmp, (uint32_t*)nullptr, (uint32_t*)nullptr, (uint32_t*)nullptr,
                                    (uint32_t*)nullptr, P, 0, 30, s);
    const size_t arr = align_up(sizeof(uint32_t) * (size_t)P);
    const size_t need = 256 + 4 * arr + align_up(sizeof(float4) * (size_t)Ppad) + align_up(sizeof(Aabb) * (size_t)nboxes) +
                        align_up(sort_tmp);
    int rc = ctx->misc.ensure(need);
    if (rc) return rc;
    char* base = (char*)ctx->misc.p;
    uint32_t* mm = (uint32_t*)base;
    uint32_t* codes = (uint32_t*)(base + 256);
    uint32_t* codes_s = (uint32_t*)(base + 256 + arr);
    uint32_t* ids = (uint32_t*)(base + 256 + 2 * arr);
    uint32_t* ids_s = (uint32_t*)(base + 256 + 3 * arr);
    float4* ps = (float4*)(base + 256 + 4 * arr);
    Aabb* boxes = (Aabb*)((char*)ps + align_up(sizeof(float4) * (size_t)Ppad));
    void* cub_tmp = (char*)boxes + align_up(sizeof(Aabb) * (size_t)nboxes);

    knn_bounds_init_kernel<<<1, 32, 0, s>>>(mm);
    knn_bounds_kernel<<<min((P + 255) / 256, kNumSMs * 8), 256, 0, s>>>(P, points, mm);
    knn_morton_kernel<<<(P + 255) / 256, 256, 0, s>>>(P, points, mm, codes, ids);
    SGB_LAUNCH_CHECK("knn_morton_kernel", 0, s);
    SGB_CUDA(cub::DeviceRadixSort::SortPairs(cub_tmp, sort_tmp, codes, codes_s, ids, ids_s, P, 0, 30, s));
    knn_gather_kernel<<<(Ppad + 255) / 256, 256, 0, s>>>(P, Ppad, points, ids_s, ps);
    knn_boxes_kernel<<<nboxes, kBox, 0, s>>>(P, ps, boxes);
    knn_kernel<<<nboxes, kBox, 0, s>>>(P, ps, boxes, nboxes, mean_dist2);
    SGB_LAUNCH_CHECK("knn_kernel", 0, s);
    ctx->launches += 6;
    ctx->lib_launches += 1;
    return SGB_OK;
}
