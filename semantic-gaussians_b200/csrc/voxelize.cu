// Voxelization of a point cloud on the device: the Voxelizer.voxelize + sparse_quantize of dataset/fusion_utils.py
//
//   coords_aug = floor(homo_coords @ T.T)                  (fp64)
//   coords_aug = floor(coords_aug - coords_aug.min(0))
//   key        = fnv_hash_vec(coords_aug)                  (FNV-1a 64 over the three uint64 coordinates)
//   _, inds, inds_reconstruct = np.unique(key, return_index=True, return_inverse=True)
//
// reproduced bit for bit.  The transform is evaluated as ((x T0 + y T1) + z T2) + T3 with separately rounded
// products and sums (no FMA contraction), which is what numpy computes for these 3x4 products.  The floors are
// integers, so their per-axis minimum is an exact int64 atomicMin.  A stable radix sort of (key, p) with p ascending
// on input makes the first element of every run of equal keys numpy's return_index (np.unique's stable mergesort),
// and the runs come out in ascending key order as np.unique's do; a scan over the run heads gives return_inverse.
//
// Passes: init -> bounds (floor, min / max, non-finite count) -> keys -> cub::DeviceRadixSort -> heads ->
// cub::DeviceScan -> scatter.  Nothing is copied to the host: M and the status words are written to `counts`.
#include <climits>
#include <cub/cub.cuh>
#include "common.cuh"

namespace sgb {

namespace {

constexpr int kVoxThreads = 256;
constexpr uint64_t kFnvOffset = 14695981039346656037ull;
constexpr uint64_t kFnvPrime = 1099511628211ull;
// Floors at or beyond 2^62 in magnitude are kept out of the int64 bounds (their difference could wrap) and flag the
// call as overflowing: no extent below 2^31 can contain them together with anything else representable.
constexpr double kVoxHuge = 4611686018427387904.0;   // 2^62

struct VoxTransform { double t[12]; };   // row-major 3x4

struct VoxHeader {       // first 256 bytes of the workspace
    long long lo[3];     // per-axis minimum floor over the finite points
    long long hi[3];     // per-axis maximum
    unsigned long long nonfinite;
    unsigned long long huge;
};

struct VoxWorkspace {
    VoxHeader* hdr;
    uint64_t* keys_in;      // [P]; after the sort: int32 heads [P] | int32 run ends [P]
    uint64_t* keys_out;     // [P]
    uint32_t* vals_in;      // [P]
    uint32_t* vals_out;     // [P]
    void* tmp;              // cub temporary storage
    size_t tmp_bytes;
    size_t bytes;
};

// Voxel floors of point p; false when any axis is not finite.  Coord = float or double: either is promoted to double
// exactly before the transform.
template <typename Coord>
__device__ __forceinline__ bool vox_floor(const Coord* __restrict__ xyz, long long p, const VoxTransform& T,
                                          double (&v)[3]) {
    const double x = xyz[3 * p], y = xyz[3 * p + 1], z = xyz[3 * p + 2];
    bool finite = true;
#pragma unroll
    for (int a = 0; a < 3; a++) {
        const double* r = T.t + 4 * a;
        const double s = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(x, r[0]), __dmul_rn(y, r[1])), __dmul_rn(z, r[2])),
                                   r[3]);
        v[a] = floor(s);
        finite &= isfinite(v[a]);
    }
    return finite;
}

__global__ void vox_init_kernel(VoxHeader* hdr, int64_t* counts) {
    if (threadIdx.x < 3) {
        hdr->lo[threadIdx.x] = LLONG_MAX;
        hdr->hi[threadIdx.x] = LLONG_MIN;
        counts[threadIdx.x] = 0;
    }
    if (threadIdx.x == 0) hdr->nonfinite = hdr->huge = 0;
}

template <typename Coord>
__global__ void __launch_bounds__(kVoxThreads) vox_bounds_kernel(long long P, const Coord* __restrict__ xyz,
                                                                 VoxTransform T, VoxHeader* hdr) {
    long long lo[3] = {LLONG_MAX, LLONG_MAX, LLONG_MAX}, hi[3] = {LLONG_MIN, LLONG_MIN, LLONG_MIN};
    unsigned nonfinite = 0, huge = 0;
    for (long long p = (long long)blockIdx.x * kVoxThreads + threadIdx.x; p < P; p += (long long)gridDim.x * kVoxThreads) {
        double v[3];
        if (!vox_floor(xyz, p, T, v)) { nonfinite++; continue; }
#pragma unroll
        for (int a = 0; a < 3; a++) {
            if (fabs(v[a]) >= kVoxHuge) { huge++; continue; }
            const long long q = (long long)v[a];
            lo[a] = min(lo[a], q);
            hi[a] = max(hi[a], q);
        }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
#pragma unroll
        for (int a = 0; a < 3; a++) {
            lo[a] = min(lo[a], __shfl_xor_sync(0xffffffffu, lo[a], o));
            hi[a] = max(hi[a], __shfl_xor_sync(0xffffffffu, hi[a], o));
        }
    }
    nonfinite = __reduce_add_sync(0xffffffffu, nonfinite);
    huge = __reduce_add_sync(0xffffffffu, huge);
    if ((threadIdx.x & 31) == 0) {
#pragma unroll
        for (int a = 0; a < 3; a++) {
            if (lo[a] != LLONG_MAX) atomicMin(&hdr->lo[a], lo[a]);
            if (hi[a] != LLONG_MIN) atomicMax(&hdr->hi[a], hi[a]);
        }
        if (nonfinite) atomicAdd(&hdr->nonfinite, (unsigned long long)nonfinite);
        if (huge) atomicAdd(&hdr->huge, (unsigned long long)huge);
    }
}

// Origin-aligned voxel coordinate of one axis.  Only meaningful for a call that reports no non-finite point and no
// overflow; otherwise any value (never a fault) may come out.
__device__ __forceinline__ uint64_t vox_rel(double v, long long lo) {
    const long long q = isfinite(v) && fabs(v) < kVoxHuge ? (long long)v : 0;
    return (uint64_t)q - (uint64_t)lo;
}

template <typename Coord>
__global__ void __launch_bounds__(kVoxThreads) vox_key_kernel(long long P, const Coord* __restrict__ xyz,
                                                              VoxTransform T, const VoxHeader* __restrict__ hdr,
                                                              uint64_t* __restrict__ keys, uint32_t* __restrict__ vals,
                                                              int64_t* __restrict__ counts) {
    const long long lo[3] = {hdr->lo[0], hdr->lo[1], hdr->lo[2]};
    const long long p = (long long)blockIdx.x * kVoxThreads + threadIdx.x;
    if (p == 0) {
        counts[1] = (int64_t)hdr->nonfinite;
        bool overflow = hdr->huge != 0;
        for (int a = 0; a < 3; a++)   // empty axis (every point non-finite): lo > hi, no overflow from it
            overflow |= hdr->lo[a] <= hdr->hi[a] && (uint64_t)hdr->hi[a] - (uint64_t)hdr->lo[a] >= (1ull << 31);
        counts[2] = overflow ? SGB_E_OVERFLOW : SGB_OK;
    }
    if (p >= P) return;
    double v[3];
    vox_floor(xyz, p, T, v);
    // fnv_hash_vec: h = offset basis; per axis h *= prime, h ^= u
    uint64_t h = kFnvOffset;
#pragma unroll
    for (int a = 0; a < 3; a++) {
        h *= kFnvPrime;
        h ^= vox_rel(v[a], lo[a]);
    }
    keys[p] = h;
    vals[p] = (uint32_t)p;
}

__global__ void __launch_bounds__(kVoxThreads) vox_head_kernel(long long P, const uint64_t* __restrict__ keys,
                                                               int* __restrict__ heads) {
    const long long i = (long long)blockIdx.x * kVoxThreads + threadIdx.x;
    if (i < P) heads[i] = i == 0 || keys[i] != keys[i - 1];
}

// runs[i] = number of run heads in sorted positions [0, i]: the run of position i is runs[i] - 1.
template <typename Coord>
__global__ void __launch_bounds__(kVoxThreads) vox_scatter_kernel(long long P, const Coord* __restrict__ xyz,
                                                                  VoxTransform T, const VoxHeader* __restrict__ hdr,
                                                                  const uint32_t* __restrict__ order,
                                                                  const int* __restrict__ heads,
                                                                  const int* __restrict__ runs,
                                                                  int64_t* __restrict__ first_index,
                                                                  int64_t* __restrict__ inverse,
                                                                  int32_t* __restrict__ coords,
                                                                  int64_t* __restrict__ counts) {
    const long long i = (long long)blockIdx.x * kVoxThreads + threadIdx.x;
    if (i >= P) return;
    const uint32_t p = order[i];
    const int r = runs[i] - 1;
    inverse[p] = r;
    if (heads[i]) {
        first_index[r] = p;
        double v[3];
        vox_floor(xyz, p, T, v);
#pragma unroll
        for (int a = 0; a < 3; a++) coords[3 * (long long)r + a] = (int32_t)(uint32_t)vox_rel(v[a], hdr->lo[a]);
    }
    if (i == P - 1) counts[0] = runs[i];
}

int carve_workspace(long long P, void* base, VoxWorkspace& w) {
    size_t sort_tmp = 0, scan_tmp = 0;
    SGB_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, sort_tmp, (uint64_t*)nullptr, (uint64_t*)nullptr,
                                             (uint32_t*)nullptr, (uint32_t*)nullptr, (int)P, 0, 64));
    SGB_CUDA(cub::DeviceScan::InclusiveSum(nullptr, scan_tmp, (int*)nullptr, (int*)nullptr, (int)P));
    char* p = (char*)base;
    size_t off = 0;
    w.hdr = (VoxHeader*)(p + off); off += align_up(sizeof(VoxHeader));
    w.keys_in = (uint64_t*)(p + off); off += align_up(sizeof(uint64_t) * (size_t)P);
    w.keys_out = (uint64_t*)(p + off); off += align_up(sizeof(uint64_t) * (size_t)P);
    w.vals_in = (uint32_t*)(p + off); off += align_up(sizeof(uint32_t) * (size_t)P);
    w.vals_out = (uint32_t*)(p + off); off += align_up(sizeof(uint32_t) * (size_t)P);
    w.tmp = p + off;
    w.tmp_bytes = sort_tmp > scan_tmp ? sort_tmp : scan_tmp;
    off += align_up(w.tmp_bytes);
    w.bytes = off;
    return SGB_OK;
}

bool vox_p_ok(int64_t P) { return P >= 1 && P <= INT32_MAX; }

template <typename Coord>
int voxelize(const char* fn, int64_t P, const Coord* xyz, const double* transform, void* workspace,
             int64_t* first_index, int64_t* inverse, int32_t* coords, int64_t* counts, void* stream) {
    if (P <= 0) { set_error("%s: P = %lld (need at least one point)", fn, (long long)P); return SGB_E_INVALID; }
    if (P > INT32_MAX) { set_error("%s: P = %lld exceeds %d points", fn, (long long)P, INT32_MAX); return SGB_E_INVALID; }
    if (!xyz) { set_error("%s: null xyz", fn); return SGB_E_INVALID; }
    if (!transform) { set_error("%s: null transform", fn); return SGB_E_INVALID; }
    if (!workspace) { set_error("%s: null workspace", fn); return SGB_E_INVALID; }
    if (reinterpret_cast<uintptr_t>(workspace) % 16) {
        set_error("%s: workspace is not 16-byte aligned", fn);
        return SGB_E_INVALID;
    }
    if (!first_index || !inverse || !coords) { set_error("%s: null first_index / inverse / coords", fn); return SGB_E_INVALID; }
    if (!counts) { set_error("%s: null counts", fn); return SGB_E_INVALID; }

    VoxTransform T;
    for (int i = 0; i < 12; i++) T.t[i] = transform[i];
    cudaStream_t s = (cudaStream_t)stream;
    VoxWorkspace w;
    int rc = carve_workspace((long long)P, workspace, w);
    if (rc) return rc;
    const long long n = (long long)P;
    const unsigned blocks = (unsigned)((n + kVoxThreads - 1) / kVoxThreads);
    int dev = 0, sms = 0;
    SGB_CUDA(cudaGetDevice(&dev));
    SGB_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    const unsigned bound_blocks = (unsigned)min((long long)blocks, 8ll * sms);   // one wave; grid-stride inside

    vox_init_kernel<<<1, 32, 0, s>>>(w.hdr, counts);
    SGB_LAUNCH_CHECK("vox_init_kernel", 0, s);
    vox_bounds_kernel<<<bound_blocks, kVoxThreads, 0, s>>>(n, xyz, T, w.hdr);
    SGB_LAUNCH_CHECK("vox_bounds_kernel", 0, s);
    vox_key_kernel<<<blocks, kVoxThreads, 0, s>>>(n, xyz, T, w.hdr, w.keys_in, w.vals_in, counts);
    SGB_LAUNCH_CHECK("vox_key_kernel", 0, s);
    size_t tmp_bytes = w.tmp_bytes;
    SGB_CUDA(cub::DeviceRadixSort::SortPairs(w.tmp, tmp_bytes, w.keys_in, w.keys_out, w.vals_in, w.vals_out, (int)n,
                                             0, 64, s));
    // keys_in is free after the sort: heads in its first half, their inclusive scan in the second
    int* heads = reinterpret_cast<int*>(w.keys_in);
    int* runs = heads + n;
    vox_head_kernel<<<blocks, kVoxThreads, 0, s>>>(n, w.keys_out, heads);
    SGB_LAUNCH_CHECK("vox_head_kernel", 0, s);
    tmp_bytes = w.tmp_bytes;
    SGB_CUDA(cub::DeviceScan::InclusiveSum(w.tmp, tmp_bytes, heads, runs, (int)n, s));
    vox_scatter_kernel<<<blocks, kVoxThreads, 0, s>>>(n, xyz, T, w.hdr, w.vals_out, heads, runs, first_index, inverse,
                                                      coords, counts);
    SGB_LAUNCH_CHECK("vox_scatter_kernel", 0, s);
    return SGB_OK;
}

}  // namespace

}  // namespace sgb

using namespace sgb;

extern "C" {

size_t sgb_voxelize_workspace_bytes(int64_t P) {
    if (!vox_p_ok(P)) return 0;
    VoxWorkspace w;
    return carve_workspace((long long)P, nullptr, w) == SGB_OK ? w.bytes : 0;
}

int sgb_voxelize(int64_t P, const float* xyz, const double* transform, void* workspace, int64_t* first_index,
                 int64_t* inverse, int32_t* coords, int64_t* counts, void* stream) {
    return voxelize<float>("sgb_voxelize", P, xyz, transform, workspace, first_index, inverse, coords, counts, stream);
}

int sgb_voxelize_f64(int64_t P, const double* xyz, const double* transform, void* workspace, int64_t* first_index,
                     int64_t* inverse, int32_t* coords, int64_t* counts, void* stream) {
    return voxelize<double>("sgb_voxelize_f64", P, xyz, transform, workspace, first_index, inverse, coords, counts,
                            stream);
}

}  // extern "C"
