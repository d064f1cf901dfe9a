// Coordinate maps and kernel maps of the sparse 3D convolution (sparse.py): what MinkowskiEngine's coordinate manager
// computes for MinkUNet, on the device.
//
// A coordinate map is N int32 rows (b, x, y, z) plus an open-addressing hash table of int32 row ids (capacity: the
// smallest power of two >= 2N, at least 64; linear probing; -1 = empty).  The table is keyed on all four values and
// compares rows exactly, so two different rows never merge (unlike sgb_voxelize's FNV key, whose collisions merge voxels
// on purpose).  Which row wins a slot race does not matter: a lookup returns the one row holding that coordinate.
//
// Strided map: parent(c) = (b, floor(x / 2t) * 2t, ...), unique.  Each parent is represented by its smallest child row
// (atomicMin in the slot), and the output rows are the parents in ascending order of that row: a scan over the
// "I am the representative" flags numbers them.  So the order is the order of first appearance in the input.
//
// Kernel map: for offset index d = jx + k*jy + k*k*jz (x fastest) the offset is lb + j*t per axis, lb = -((k-1)/2)*t,
// and output row o pairs with input row i when coord(i) = coord(o) + offset.  A count pass over (output block, offset)
// and an exclusive scan place every block's pairs; the fill pass recomputes the lookups and writes (in, out) int2
// pairs, grouped by offset and ascending in the output row within an offset.  The workspace carries the scan from the
// count call to the fill call; the caller reads the per-offset offsets back once in between to size the pair buffer.
#include <cub/cub.cuh>
#include "common.cuh"

namespace sgb {

namespace {

constexpr int kCoordThreads = 256;
constexpr int32_t kEmpty = -1;

uint64_t table_capacity(long long n) {
    uint64_t c = 64;
    while (c < 2 * (uint64_t)n) c <<= 1;
    return c;
}

__device__ __forceinline__ uint64_t mix64(uint64_t z) {   // splitmix64 finaliser
    z = (z ^ (z >> 30)) * 0xbf58476d1ce4e5b9ull;
    z = (z ^ (z >> 27)) * 0x94d049bb133111ebull;
    return z ^ (z >> 31);
}

__device__ __forceinline__ uint64_t coord_hash(int4 c) {
    const uint64_t lo = ((uint64_t)(uint32_t)c.x << 32) | (uint32_t)c.y;
    const uint64_t hi = ((uint64_t)(uint32_t)c.z << 32) | (uint32_t)c.w;
    return mix64(lo ^ mix64(hi + 0x9e3779b97f4a7c15ull));
}

__device__ __forceinline__ bool same(int4 a, int4 b) { return a.x == b.x && a.y == b.y && a.z == b.z && a.w == b.w; }

// Row holding coordinate q, or -1.
__device__ __forceinline__ int32_t coord_find(const int32_t* __restrict__ table, uint64_t mask,
                                              const int4* __restrict__ coords, int4 q) {
    for (uint64_t s = coord_hash(q) & mask;; s = (s + 1) & mask) {
        const int32_t r = __ldg(table + s);
        if (r == kEmpty) return -1;
        if (same(__ldg(coords + r), q)) return r;
    }
}

__global__ void __launch_bounds__(kCoordThreads) coord_insert_kernel(long long n, const int4* __restrict__ coords,
                                                                     int32_t* __restrict__ table, uint64_t mask,
                                                                     unsigned long long* __restrict__ status) {
    const long long i = (long long)blockIdx.x * kCoordThreads + threadIdx.x;
    if (i >= n) return;
    const int4 c = coords[i];
    if (c.y < 0 || c.z < 0 || c.w < 0) atomicAdd(&status[1], 1ull);
    for (uint64_t s = coord_hash(c) & mask;; s = (s + 1) & mask) {
        const int32_t old = atomicCAS(table + s, kEmpty, (int32_t)i);
        if (old == kEmpty) return;
        if (same(coords[old], c)) { atomicAdd(&status[0], 1ull); return; }
    }
}

__device__ __forceinline__ int4 parent_of(int4 c, int t2) {
    return make_int4(c.x, c.y / t2 * t2, c.z / t2 * t2, c.w / t2 * t2);   // c >= 0: division is floor
}

__global__ void __launch_bounds__(kCoordThreads) stride_insert_kernel(long long n, const int4* __restrict__ coords,
                                                                      int t2, int32_t* __restrict__ table,
                                                                      uint64_t mask) {
    const long long i = (long long)blockIdx.x * kCoordThreads + threadIdx.x;
    if (i >= n) return;
    const int4 p = parent_of(coords[i], t2);
    for (uint64_t s = coord_hash(p) & mask;; s = (s + 1) & mask) {
        const int32_t old = atomicCAS(table + s, kEmpty, (int32_t)i);
        if (old == kEmpty) return;
        // every row ever held by this slot has parent p, so the comparison stays valid under the atomicMin
        if (same(parent_of(coords[old], t2), p)) { atomicMin(table + s, (int32_t)i); return; }
    }
}

__global__ void __launch_bounds__(kCoordThreads) stride_head_kernel(long long n, const int4* __restrict__ coords,
                                                                    int t2, const int32_t* __restrict__ table,
                                                                    uint64_t mask, int* __restrict__ heads) {
    const long long i = (long long)blockIdx.x * kCoordThreads + threadIdx.x;
    if (i >= n) return;
    const int4 p = parent_of(coords[i], t2);
    for (uint64_t s = coord_hash(p) & mask;; s = (s + 1) & mask) {
        const int32_t r = table[s];
        if (same(parent_of(coords[r], t2), p)) { heads[i] = r == (int32_t)i; return; }
    }
}

__global__ void __launch_bounds__(kCoordThreads) stride_scatter_kernel(long long n, const int4* __restrict__ coords,
                                                                       int t2, const int* __restrict__ heads,
                                                                       const int* __restrict__ rank,
                                                                       int4* __restrict__ out, int64_t* out_count) {
    const long long i = (long long)blockIdx.x * kCoordThreads + threadIdx.x;
    if (i >= n) return;
    if (heads[i]) out[rank[i]] = parent_of(coords[i], t2);
    if (i == n - 1) *out_count = (int64_t)rank[i] + heads[i];
}

struct KmapQuery {
    int k, t, lb;
};

// Input row paired with output row o at offset d, or -1.
__device__ __forceinline__ int32_t kmap_lookup(long long o, int d, KmapQuery q, const int4* __restrict__ out_coords,
                                               const int4* __restrict__ in_coords, const int32_t* __restrict__ table,
                                               uint64_t mask) {
    const int4 c = __ldg(out_coords + o);
    const long long x = (long long)c.y + q.lb + (long long)(d % q.k) * q.t;
    const long long y = (long long)c.z + q.lb + (long long)(d / q.k % q.k) * q.t;
    const long long z = (long long)c.w + q.lb + (long long)(d / (q.k * q.k)) * q.t;
    if (x < 0 || y < 0 || z < 0 || x > INT32_MAX || y > INT32_MAX || z > INT32_MAX) return -1;   // never in a map
    return coord_find(table, mask, in_coords, make_int4(c.x, (int)x, (int)y, (int)z));
}

__global__ void __launch_bounds__(kCoordThreads) kmap_count_kernel(long long n_out, KmapQuery q,
                                                                   const int4* __restrict__ out_coords,
                                                                   const int4* __restrict__ in_coords,
                                                                   const int32_t* __restrict__ table, uint64_t mask,
                                                                   long long* __restrict__ counts) {
    const long long o = (long long)blockIdx.x * kCoordThreads + threadIdx.x;
    const int d = blockIdx.y;
    const bool hit = o < n_out && kmap_lookup(o, d, q, out_coords, in_coords, table, mask) >= 0;
    const int n = __syncthreads_count(hit);
    if (threadIdx.x == 0) counts[(long long)d * gridDim.x + blockIdx.x] = n;
}

__global__ void kmap_offsets_kernel(int K, long long nblk, const long long* __restrict__ counts,
                                    const long long* __restrict__ starts, int64_t* __restrict__ offsets) {
    const int d = blockIdx.x * blockDim.x + threadIdx.x;
    if (d < K) offsets[d] = starts[(long long)d * nblk];
    if (d == K) offsets[K] = starts[K * nblk - 1] + counts[K * nblk - 1];
}

__global__ void __launch_bounds__(kCoordThreads) kmap_fill_kernel(long long n_out, KmapQuery q,
                                                                  const int4* __restrict__ out_coords,
                                                                  const int4* __restrict__ in_coords,
                                                                  const int32_t* __restrict__ table, uint64_t mask,
                                                                  const long long* __restrict__ starts,
                                                                  int2* __restrict__ pairs) {
    __shared__ int warp_base[kCoordThreads / 32];
    const long long o = (long long)blockIdx.x * kCoordThreads + threadIdx.x;
    const int d = blockIdx.y;
    const int32_t in = o < n_out ? kmap_lookup(o, d, q, out_coords, in_coords, table, mask) : -1;
    const unsigned ballot = __ballot_sync(0xffffffffu, in >= 0);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (lane == 0) warp_base[warp] = __popc(ballot);
    __syncthreads();
    if (threadIdx.x == 0) {
        int run = 0;
        for (int w = 0; w < kCoordThreads / 32; w++) { const int c = warp_base[w]; warp_base[w] = run; run += c; }
    }
    __syncthreads();
    if (in >= 0) {
        const long long at = starts[(long long)d * gridDim.x + blockIdx.x] + warp_base[warp] +
                             __popc(ballot & ((1u << lane) - 1));
        pairs[at] = make_int2(in, (int32_t)o);
    }
}

struct StrideWorkspace {
    int32_t* table;
    int* heads;    // [N]
    int* rank;     // [N]
    void* tmp;
    size_t tmp_bytes;
    uint64_t cap;
    size_t bytes;
};

int carve_stride(long long n, void* base, StrideWorkspace& w) {
    SGB_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, w.tmp_bytes, (int*)nullptr, (int*)nullptr, (int)n));
    char* p = (char*)base;
    size_t off = 0;
    w.cap = table_capacity(n);
    w.table = (int32_t*)(p + off); off += align_up(sizeof(int32_t) * w.cap);
    w.heads = (int*)(p + off); off += align_up(sizeof(int) * (size_t)n);
    w.rank = (int*)(p + off); off += align_up(sizeof(int) * (size_t)n);
    w.tmp = p + off; off += align_up(w.tmp_bytes);
    w.bytes = off;
    return SGB_OK;
}

struct KmapWorkspace {
    long long* counts;   // [K * nblk] pairs of each (offset, output block)
    long long* starts;   // [K * nblk] their exclusive scan: where the block's pairs begin
    void* tmp;
    size_t tmp_bytes;
    long long nblk;
    size_t bytes;
};

int carve_kmap(long long n_out, int K, void* base, KmapWorkspace& w) {
    w.nblk = (n_out + kCoordThreads - 1) / kCoordThreads;
    const long long m = w.nblk * K;
    SGB_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, w.tmp_bytes, (long long*)nullptr, (long long*)nullptr, (int)m));
    char* p = (char*)base;
    size_t off = 0;
    w.counts = (long long*)(p + off); off += align_up(sizeof(long long) * (size_t)m);
    w.starts = (long long*)(p + off); off += align_up(sizeof(long long) * (size_t)m);
    w.tmp = p + off; off += align_up(w.tmp_bytes);
    w.bytes = off;
    return SGB_OK;
}

bool rows_ok(int64_t n) { return n >= 1 && n <= INT32_MAX; }

bool aligned16(const void* p) { return reinterpret_cast<uintptr_t>(p) % 16 == 0; }

int check_rows(const char* fn, const char* what, int64_t n, const void* coords) {
    if (!rows_ok(n)) { set_error("%s: %s = %lld (need 1 <= N <= 2^31 - 1)", fn, what, (long long)n); return SGB_E_INVALID; }
    if (!coords) { set_error("%s: null coordinates for %s", fn, what); return SGB_E_INVALID; }
    if (!aligned16(coords)) { set_error("%s: coordinates for %s are not 16-byte aligned", fn, what); return SGB_E_INVALID; }
    return SGB_OK;
}

// Kernel sizes and strides of the supported layers: k in {2, 3, 5}, 1 <= t <= 2^24 (far below any overflow of
// coordinate + offset in int64).
int check_kmap_args(const char* fn, int64_t n_in, const int32_t* in_coords, const void* in_table, int64_t n_out,
                    const int32_t* out_coords, int32_t k, int32_t stride, const void* workspace) {
    if (int rc = check_rows(fn, "N_in", n_in, in_coords)) return rc;
    if (int rc = check_rows(fn, "N_out", n_out, out_coords)) return rc;
    if (!in_table) { set_error("%s: null input table", fn); return SGB_E_INVALID; }
    if (k != 2 && k != 3 && k != 5) { set_error("%s: kernel size %d (supported: 2, 3, 5)", fn, k); return SGB_E_INVALID; }
    if (stride < 1 || stride > (1 << 24)) { set_error("%s: tensor stride %d out of range", fn, stride); return SGB_E_INVALID; }
    if (!workspace || !aligned16(workspace)) { set_error("%s: null or unaligned workspace", fn); return SGB_E_INVALID; }
    return SGB_OK;
}

unsigned blocks_for(long long n) { return (unsigned)((n + kCoordThreads - 1) / kCoordThreads); }

}  // namespace

}  // namespace sgb

using namespace sgb;

extern "C" {

size_t sgb_coord_map_bytes(int64_t N) {
    if (!rows_ok(N)) return 0;
    return align_up(sizeof(int32_t) * table_capacity(N));
}

int sgb_coord_map_build(int64_t N, const int32_t* coords, void* table, int64_t* status, void* stream) {
    const char* fn = "sgb_coord_map_build";
    if (int rc = check_rows(fn, "N", N, coords)) return rc;
    if (!table) { set_error("%s: null table", fn); return SGB_E_INVALID; }
    if (!status) { set_error("%s: null status", fn); return SGB_E_INVALID; }
    cudaStream_t s = (cudaStream_t)stream;
    const uint64_t cap = table_capacity(N);
    SGB_CUDA(cudaMemsetAsync(table, 0xff, sizeof(int32_t) * cap, s));
    SGB_CUDA(cudaMemsetAsync(status, 0, 2 * sizeof(int64_t), s));
    coord_insert_kernel<<<blocks_for(N), kCoordThreads, 0, s>>>(N, (const int4*)coords, (int32_t*)table, cap - 1,
                                                               (unsigned long long*)status);
    SGB_LAUNCH_CHECK("coord_insert_kernel", 0, s);
    return SGB_OK;
}

size_t sgb_coord_stride_workspace_bytes(int64_t N) {
    if (!rows_ok(N)) return 0;
    StrideWorkspace w;
    return carve_stride(N, nullptr, w) == SGB_OK ? w.bytes : 0;
}

int sgb_coord_stride(int64_t N, const int32_t* coords, int32_t stride, void* workspace, int32_t* out_coords,
                     int64_t* out_count, void* stream) {
    const char* fn = "sgb_coord_stride";
    if (int rc = check_rows(fn, "N", N, coords)) return rc;
    if (stride < 1 || stride > (1 << 24)) { set_error("%s: tensor stride %d out of range", fn, stride); return SGB_E_INVALID; }
    if (!workspace || !aligned16(workspace)) { set_error("%s: null or unaligned workspace", fn); return SGB_E_INVALID; }
    if (!out_coords || !aligned16(out_coords)) { set_error("%s: null or unaligned out_coords", fn); return SGB_E_INVALID; }
    if (!out_count) { set_error("%s: null out_count", fn); return SGB_E_INVALID; }
    cudaStream_t s = (cudaStream_t)stream;
    StrideWorkspace w;
    if (int rc = carve_stride(N, workspace, w)) return rc;
    const int t2 = 2 * stride;
    const unsigned blocks = blocks_for(N);
    const int4* c = (const int4*)coords;
    SGB_CUDA(cudaMemsetAsync(w.table, 0xff, sizeof(int32_t) * w.cap, s));
    stride_insert_kernel<<<blocks, kCoordThreads, 0, s>>>(N, c, t2, w.table, w.cap - 1);
    SGB_LAUNCH_CHECK("stride_insert_kernel", 0, s);
    stride_head_kernel<<<blocks, kCoordThreads, 0, s>>>(N, c, t2, w.table, w.cap - 1, w.heads);
    SGB_LAUNCH_CHECK("stride_head_kernel", 0, s);
    size_t tmp = w.tmp_bytes;
    SGB_CUDA(cub::DeviceScan::ExclusiveSum(w.tmp, tmp, w.heads, w.rank, (int)N, s));
    stride_scatter_kernel<<<blocks, kCoordThreads, 0, s>>>(N, c, t2, w.heads, w.rank, (int4*)out_coords, out_count);
    SGB_LAUNCH_CHECK("stride_scatter_kernel", 0, s);
    return SGB_OK;
}

size_t sgb_kernel_map_workspace_bytes(int64_t N_out, int32_t k) {
    if (!rows_ok(N_out) || k < 1 || k > 5) return 0;
    KmapWorkspace w;
    return carve_kmap(N_out, k * k * k, nullptr, w) == SGB_OK ? w.bytes : 0;
}

int sgb_kernel_map_count(int64_t N_in, const int32_t* in_coords, const void* in_table, int64_t N_out,
                         const int32_t* out_coords, int32_t k, int32_t stride, void* workspace, int64_t* offsets,
                         void* stream) {
    const char* fn = "sgb_kernel_map_count";
    if (int rc = check_kmap_args(fn, N_in, in_coords, in_table, N_out, out_coords, k, stride, workspace)) return rc;
    if (!offsets) { set_error("%s: null offsets", fn); return SGB_E_INVALID; }
    cudaStream_t s = (cudaStream_t)stream;
    const int K = k * k * k;
    KmapWorkspace w;
    if (int rc = carve_kmap(N_out, K, workspace, w)) return rc;
    const KmapQuery q{k, stride, -((k - 1) / 2) * stride};
    const dim3 grid((unsigned)w.nblk, (unsigned)K);
    kmap_count_kernel<<<grid, kCoordThreads, 0, s>>>(N_out, q, (const int4*)out_coords, (const int4*)in_coords,
                                                    (const int32_t*)in_table, table_capacity(N_in) - 1, w.counts);
    SGB_LAUNCH_CHECK("kmap_count_kernel", 0, s);
    size_t tmp = w.tmp_bytes;
    SGB_CUDA(cub::DeviceScan::ExclusiveSum(w.tmp, tmp, w.counts, w.starts, (int)(w.nblk * K), s));
    kmap_offsets_kernel<<<1, 128, 0, s>>>(K, w.nblk, w.counts, w.starts, offsets);
    SGB_LAUNCH_CHECK("kmap_offsets_kernel", 0, s);
    return SGB_OK;
}

int sgb_kernel_map_fill(int64_t N_in, const int32_t* in_coords, const void* in_table, int64_t N_out,
                        const int32_t* out_coords, int32_t k, int32_t stride, const void* workspace, int32_t* pairs,
                        void* stream) {
    const char* fn = "sgb_kernel_map_fill";
    if (int rc = check_kmap_args(fn, N_in, in_coords, in_table, N_out, out_coords, k, stride, workspace)) return rc;
    if (!pairs || reinterpret_cast<uintptr_t>(pairs) % 8) { set_error("%s: null or unaligned pairs", fn); return SGB_E_INVALID; }
    cudaStream_t s = (cudaStream_t)stream;
    const int K = k * k * k;
    KmapWorkspace w;
    if (int rc = carve_kmap(N_out, K, const_cast<void*>(workspace), w)) return rc;
    const KmapQuery q{k, stride, -((k - 1) / 2) * stride};
    const dim3 grid((unsigned)w.nblk, (unsigned)K);
    kmap_fill_kernel<<<grid, kCoordThreads, 0, s>>>(N_out, q, (const int4*)out_coords, (const int4*)in_coords,
                                                   (const int32_t*)in_table, table_capacity(N_in) - 1, w.starts,
                                                   (int2*)pairs);
    SGB_LAUNCH_CHECK("kmap_fill_kernel", 0, s);
    return SGB_OK;
}

}  // extern "C"
