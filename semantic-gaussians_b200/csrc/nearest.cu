// Exact nearest neighbour of every query point in a reference cloud (sgb_nearest): the label / feature transfer
// from Gaussians onto scan vertices that a per-point 3D evaluation needs.
//
// The result is exact, not approximate: index[q] minimises the fp32 key (d2, j) with
//     d2 = (dx*dx + dy*dy) + dz*dz,  dx = q.x - r_j.x, ...   every product and sum rounded alone
// over the finite reference rows with d2 <= max_dist2, so it does not depend on the order candidates are visited in.
//
// Organisation (the scheme of knn.cu): both sets are sorted along one 30-bit Morton curve over the bounds of the
// finite reference rows.  Consecutive runs of 256 sorted reference points form boxes with an AABB; each CTA owns 256 sorted
// queries (one per thread) and their AABB.  A CTA first scans the reference box its queries' Morton codes fall in,
// which gives every thread a near match, then walks all boxes: a box is skipped for the whole CTA when its distance to
// the query box exceeds the largest current best d2 of the CTA, and per thread when its distance to the thread's
// query exceeds that thread's best.  Both bounds are computed with the d2 expression on the per-axis gaps; fp32
// rounding is monotone, so a bound never exceeds the computed d2 of any point it covers, and the pruning is exact.
#include <cfloat>
#include <cub/cub.cuh>
#include "common.cuh"
#include "spatial.cuh"

namespace sgb {

namespace {

constexpr int kBox = 256;                       // reference points per box = queries per CTA
constexpr uint32_t kNone = 0xFFFFFFFFu;         // no match / padding slot
constexpr uint32_t kNonFinite = 1u << 30;       // sort key of a non-finite row: after every Morton code
constexpr int kSortBits = 31;

__device__ __forceinline__ bool finite3(float x, float y, float z) {
    return isfinite(x) && isfinite(y) && isfinite(z);
}

// the contract's d2, with no FMA contraction
__device__ __forceinline__ float d2_of(float dx, float dy, float dz) {
    return __fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz));
}

// per-axis gap of two intervals; never larger than the rounded difference of any two points they hold
__device__ __forceinline__ float gap(float alo, float ahi, float blo, float bhi) {
    return fmaxf(0.f, fmaxf(__fsub_rn(alo, bhi), __fsub_rn(blo, ahi)));
}

__device__ __forceinline__ float box_box_d2(const Aabb& a, const Aabb& b) {
    return d2_of(gap(a.lo[0], a.hi[0], b.lo[0], b.hi[0]), gap(a.lo[1], a.hi[1], b.lo[1], b.hi[1]),
                 gap(a.lo[2], a.hi[2], b.lo[2], b.hi[2]));
}

__device__ __forceinline__ float point_box_d2(const Aabb& b, float x, float y, float z) {
    return d2_of(gap(x, x, b.lo[0], b.hi[0]), gap(y, y, b.lo[1], b.hi[1]), gap(z, z, b.lo[2], b.hi[2]));
}

// min / max keys of the finite rows of an (n,3) set into mm (initialised by the caller)
__global__ void nearest_bounds_kernel(int64_t n, const float* __restrict__ pts, uint32_t* mm) {
    float lo[3] = {FLT_MAX, FLT_MAX, FLT_MAX}, hi[3] = {-FLT_MAX, -FLT_MAX, -FLT_MAX};
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const float x = pts[3 * i], y = pts[3 * i + 1], z = pts[3 * i + 2];
        if (!finite3(x, y, z)) continue;
        lo[0] = fminf(lo[0], x); lo[1] = fminf(lo[1], y); lo[2] = fminf(lo[2], z);
        hi[0] = fmaxf(hi[0], x); hi[1] = fmaxf(hi[1], y); hi[2] = fmaxf(hi[2], z);
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

__global__ void nearest_morton_kernel(int64_t n, const float* __restrict__ pts, const uint32_t* __restrict__ mm,
                                      uint32_t* __restrict__ codes, uint32_t* __restrict__ ids) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float* p = pts + 3 * i;
    codes[i] = finite3(p[0], p[1], p[2]) ? morton30(p, mm) : kNonFinite;
    ids[i] = (uint32_t)i;
}

// sorted, padded copy: s[i] = (x, y, z, original index).  Non-finite rows and the padding slots >= n hold NaN
// coordinates, so their d2 is NaN and never compares as a match; padding slots carry index kNone.
__global__ void nearest_gather_kernel(int64_t n, int64_t npad, const float* __restrict__ pts,
                                      const uint32_t* __restrict__ order, float4* __restrict__ s) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= npad) return;
    float4 v = make_float4(NAN, NAN, NAN, __uint_as_float(kNone));
    if (i < n) {
        const uint32_t o = order[i];
        const float x = pts[3 * (size_t)o], y = pts[3 * (size_t)o + 1], z = pts[3 * (size_t)o + 2];
        v.w = __uint_as_float(o);
        if (finite3(x, y, z)) v.x = x, v.y = y, v.z = z;
    }
    s[i] = v;
}

// AABB of each run of kBox sorted slots over their finite points (fminf / fmaxf skip the NaN slots).  A run with no
// finite point gets lo = +inf > hi = -inf.
__global__ void __launch_bounds__(kBox) nearest_boxes_kernel(const float4* __restrict__ s, Aabb* __restrict__ boxes) {
    __shared__ float red[6][kBox / 32];
    const float4 p = s[(size_t)blockIdx.x * kBox + threadIdx.x];
    float v[6] = {p.x, p.y, p.z, p.x, p.y, p.z};
#pragma unroll
    for (int a = 0; a < 6; a++) {
        if (isnan(v[a])) v[a] = a < 3 ? INFINITY : -INFINITY;
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

__global__ void __launch_bounds__(kBox) nearest_kernel(const float4* __restrict__ rs, const Aabb* __restrict__ rboxes,
                                                       int nboxes, const uint32_t* __restrict__ rcodes, int64_t P,
                                                       const float4* __restrict__ qs, const Aabb* __restrict__ qboxes,
                                                       const uint32_t* __restrict__ qcodes, int64_t M, float max_dist2,
                                                       int64_t* __restrict__ index, float* __restrict__ dist2) {
    __shared__ float4 tile[kBox];
    __shared__ float lbs[kBox];
    __shared__ float wmax[kBox / 32];
    __shared__ Aabb cbox;
    __shared__ int seed_box;
    const int b = blockIdx.x, t = threadIdx.x;
    const float4 me = qs[(size_t)b * kBox + t];    // padded array: always readable
    const bool valid = finite3(me.x, me.y, me.z);
    const Aabb qbox = qboxes[b];
    // (best, bestj) is the smallest (d2, j) so far; starting from (max_dist2, kNone) admits exactly d2 <= max_dist2
    float best = max_dist2;
    uint32_t bestj = kNone;

    auto visit = [&](int c) {  // scan box c for the threads it can improve
        __syncthreads();       // tile / cbox free
        tile[t] = rs[(size_t)c * kBox + t];
        if (t == 0) cbox = rboxes[c];
        __syncthreads();
        if (!valid || point_box_d2(cbox, me.x, me.y, me.z) > best) return;
#pragma unroll 8
        for (int j = 0; j < kBox; j++) {
            const float4 r = tile[j];
            const float d = d2_of(__fsub_rn(me.x, r.x), __fsub_rn(me.y, r.y), __fsub_rn(me.z, r.z));
            const uint32_t id = __float_as_uint(r.w);
            if (d < best || (d == best && id < bestj)) {
                best = d;
                bestj = id;
            }
        }
    };
    auto block_max_best = [&]() {  // largest best d2 among the CTA's finite queries; -inf when there is none
        float v = valid ? best : -INFINITY;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
        __syncthreads();  // previous readers of wmax are done
        if ((t & 31) == 0) wmax[t >> 5] = v;
        __syncthreads();
        float r = wmax[0];
#pragma unroll
        for (int w = 1; w < kBox / 32; w++) r = fmaxf(r, wmax[w]);
        return r;
    };

    if (qbox.lo[0] <= qbox.hi[0]) {  // uniform: the CTA holds a finite query
        if (t == 0) {
            // the reference box of the first finite reference code >= the code of the CTA's middle query
            const uint32_t key = qcodes[min((int64_t)b * kBox + kBox / 2, M - 1)];
            int64_t lo = 0, hi = P;
            while (lo < hi) {
                const int64_t mid = (lo + hi) / 2;
                if (rcodes[mid] < key) lo = mid + 1;
                else hi = mid;
            }
            if (lo > 0 && (lo == P || rcodes[lo] == kNonFinite)) lo--;
            seed_box = (int)(lo / kBox);
        }
        __syncthreads();
        const int seed = seed_box;
        visit(seed);
        float reject = block_max_best();
        for (int c0 = 0; c0 < nboxes; c0 += kBox) {
            __syncthreads();  // lbs of the previous group consumed
            if (c0 + t < nboxes) {
                const Aabb rb = rboxes[c0 + t];
                // an empty box gets NaN, which no comparison below admits
                lbs[t] = rb.lo[0] <= rb.hi[0] ? box_box_d2(qbox, rb) : NAN;
            }
            __syncthreads();
            const int lim = min(kBox, nboxes - c0);
            for (int j = 0; j < lim; j++) {
                const int c = c0 + j;
                if (c == seed || !(lbs[j] <= reject)) continue;  // uniform: shared value against a CTA-wide bound
                visit(c);
                reject = block_max_best();
            }
        }
    }
    const uint32_t q = __float_as_uint(me.w);
    if (q != kNone) {
        index[q] = bestj == kNone ? -1 : (int64_t)bestj;
        dist2[q] = bestj == kNone ? INFINITY : best;
    }
}

__global__ void nearest_none_kernel(int64_t M, int64_t* __restrict__ index, float* __restrict__ dist2) {
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < M; i += (int64_t)gridDim.x * blockDim.x) {
        index[i] = -1;
        dist2[i] = INFINITY;
    }
}

}  // namespace

}  // namespace sgb

using namespace sgb;

extern "C" int sgb_nearest(sgb_ctx* ctx, int64_t P, const float* ref_xyz, int64_t M, const float* query_xyz,
                           float max_dist2, int64_t* index, float* dist2, void* stream) {
    cudaStream_t s = (cudaStream_t)stream;
    const int64_t kMax = 0x7FFFFFFF;
    if (!ctx) { set_error("sgb_nearest: null ctx"); return SGB_E_INVALID; }
    if (P < 0 || P > kMax || M < 0 || M > kMax) {
        set_error("sgb_nearest: P = %lld and M = %lld must lie in [0, 2^31 - 1]", (long long)P, (long long)M);
        return SGB_E_INVALID;
    }
    if (max_dist2 != max_dist2) { set_error("sgb_nearest: max_dist2 is NaN"); return SGB_E_INVALID; }
    if ((P > 0 && !ref_xyz) || (M > 0 && (!query_xyz || !index || !dist2))) {
        set_error("sgb_nearest: null argument");
        return SGB_E_INVALID;
    }
    if (M == 0) return SGB_OK;
    if (P == 0) {
        nearest_none_kernel<<<(int)std::min<int64_t>((M + 255) / 256, kNumSMs * 8), 256, 0, s>>>(M, index, dist2);
        SGB_LAUNCH_CHECK("nearest_none_kernel", 0, s);
        ctx->launches += 1;
        ctx->lib_launches += 1;
        return SGB_OK;
    }
    const int64_t nboxes = (P + kBox - 1) / kBox, Ppad = nboxes * kBox;
    const int64_t nq = (M + kBox - 1) / kBox, Mpad = nq * kBox;
    size_t sort_p = 0, sort_m = 0;
    cub::DeviceRadixSort::SortPairs(nullptr, sort_p, (uint32_t*)nullptr, (uint32_t*)nullptr, (uint32_t*)nullptr,
                                    (uint32_t*)nullptr, (int)P, 0, kSortBits, s);
    cub::DeviceRadixSort::SortPairs(nullptr, sort_m, (uint32_t*)nullptr, (uint32_t*)nullptr, (uint32_t*)nullptr,
                                    (uint32_t*)nullptr, (int)M, 0, kSortBits, s);
    const size_t arr_p = align_up(sizeof(uint32_t) * (size_t)P), arr_m = align_up(sizeof(uint32_t) * (size_t)M);
    const size_t need = 256 + 4 * arr_p + 4 * arr_m + align_up(sizeof(float4) * (size_t)Ppad) +
                        align_up(sizeof(float4) * (size_t)Mpad) + align_up(sizeof(Aabb) * (size_t)nboxes) +
                        align_up(sizeof(Aabb) * (size_t)nq) + align_up(std::max(sort_p, sort_m));
    int rc = ctx->misc.ensure(need);
    if (rc) return rc;
    char* p = (char*)ctx->misc.p;
    auto carve = [&](size_t bytes) { char* r = p; p += bytes; return r; };
    uint32_t* mm = (uint32_t*)carve(256);
    uint32_t* rcode = (uint32_t*)carve(arr_p);
    uint32_t* rcode_s = (uint32_t*)carve(arr_p);
    uint32_t* rid = (uint32_t*)carve(arr_p);
    uint32_t* rid_s = (uint32_t*)carve(arr_p);
    uint32_t* qcode = (uint32_t*)carve(arr_m);
    uint32_t* qcode_s = (uint32_t*)carve(arr_m);
    uint32_t* qid = (uint32_t*)carve(arr_m);
    uint32_t* qid_s = (uint32_t*)carve(arr_m);
    float4* rs = (float4*)carve(align_up(sizeof(float4) * (size_t)Ppad));
    float4* qs = (float4*)carve(align_up(sizeof(float4) * (size_t)Mpad));
    Aabb* rboxes = (Aabb*)carve(align_up(sizeof(Aabb) * (size_t)nboxes));
    Aabb* qboxes = (Aabb*)carve(align_up(sizeof(Aabb) * (size_t)nq));
    void* cub_tmp = carve(0);

    // One Morton frame, the bounds of the finite reference rows, for both sets: a query's code then locates its seed
    // box, and queries outside the cloud clamp onto its faces instead of stretching the frame.
    SGB_CUDA(cudaMemsetAsync(mm, 0xFF, 3 * sizeof(uint32_t), s));      // min keys
    SGB_CUDA(cudaMemsetAsync(mm + 3, 0, 3 * sizeof(uint32_t), s));     // max keys
    nearest_bounds_kernel<<<(int)std::min<int64_t>((P + 255) / 256, kNumSMs * 8), 256, 0, s>>>(P, ref_xyz, mm);
    nearest_morton_kernel<<<(int)((P + 255) / 256), 256, 0, s>>>(P, ref_xyz, mm, rcode, rid);
    nearest_morton_kernel<<<(int)((M + 255) / 256), 256, 0, s>>>(M, query_xyz, mm, qcode, qid);
    SGB_LAUNCH_CHECK("nearest_morton_kernel", 0, s);
    SGB_CUDA(cub::DeviceRadixSort::SortPairs(cub_tmp, sort_p, rcode, rcode_s, rid, rid_s, (int)P, 0, kSortBits, s));
    SGB_CUDA(cub::DeviceRadixSort::SortPairs(cub_tmp, sort_m, qcode, qcode_s, qid, qid_s, (int)M, 0, kSortBits, s));
    nearest_gather_kernel<<<(int)((Ppad + 255) / 256), 256, 0, s>>>(P, Ppad, ref_xyz, rid_s, rs);
    nearest_gather_kernel<<<(int)((Mpad + 255) / 256), 256, 0, s>>>(M, Mpad, query_xyz, qid_s, qs);
    nearest_boxes_kernel<<<(int)nboxes, kBox, 0, s>>>(rs, rboxes);
    nearest_boxes_kernel<<<(int)nq, kBox, 0, s>>>(qs, qboxes);
    nearest_kernel<<<(int)nq, kBox, 0, s>>>(rs, rboxes, (int)nboxes, rcode_s, P, qs, qboxes, qcode_s, M, max_dist2,
                                            index, dist2);
    SGB_LAUNCH_CHECK("nearest_kernel", 0, s);
    ctx->launches += 8;
    ctx->lib_launches += 2;
    return SGB_OK;
}
