// Binning: depth order of the Gaussians, offsets scan, (tile, Gaussian) instance emission, tile
// sort and per-tile ranges.  Contract: the sorted Gaussian-id list and the tile ranges equal the
// reference's point_list / ranges bit for bit (rasterizer_impl.cu:70-138, :277-321).
//
// The reference sorts R instances by a 64-bit key [tile | depth bits] with one stable radix sort
// (~6 passes over 12 B/instance, R ~ 25-30 x P).  The same total order — tile, then depth bits,
// then ascending Gaussian id for ties (stability) — is produced here by
//   1. a stable sort of the P Gaussians by depth bits (32-bit keys, P items; input order is the
//      id order, so ties keep ascending id),
//   2. emitting instances in that order with a 32-bit tile key,
//   3. a stable radix sort of the R instances by the tile bits only (ceil(log2(#tiles)) bits,
//      2 passes for 8160 tiles) carrying the 32-bit Gaussian id.
// A stable sort by tile of a depth-ordered sequence is depth-ordered inside every tile, so the
// result is identical while the R-sized traffic drops from ~6x(12+12) B to 2x(8+8) B per instance.
#include <cub/cub.cuh>
#include "common.cuh"
#include "weight_pool.cuh"

namespace sgb {

namespace {

__global__ void iota_kernel(int P, uint32_t* v) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < P) v[i] = i;
}

// tiles_touched in depth order (input of the offsets scan)
// Also sums the counts in 64 bits: the 32-bit scan below wraps silently once the instance count reaches 2^32,
// and a wrapped (small) R would pass the int32 check in sgb_forward_geometry and let the emitter write past
// the binning buffer.
__global__ void gather_counts_kernel(int P, const uint32_t* __restrict__ perm,
                                     const uint32_t* __restrict__ tiles_touched, uint32_t* __restrict__ out,
                                     unsigned long long* __restrict__ total64) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    uint32_t n = 0;
    if (i < P) {
        n = tiles_touched[perm[i]];
        out[i] = n;
    }
    unsigned long long t = n;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
    if ((threadIdx.x & 31) == 0 && t) atomicAdd(total64, t);
}

// One warp handles 32 consecutive slots of the depth order; for each visible Gaussian its lanes
// write the tile keys / ids of its rectangle cooperatively (coalesced), instead of one thread
// walking the whole rectangle (duplicateWithKeys, rasterizer_impl.cu:70-111).
template <typename KeyT>
__global__ void __launch_bounds__(256) emit_instances_kernel(int P, const uint32_t* __restrict__ perm,
                                                             const uint32_t* __restrict__ offsets,
                                                             const SplatRec* __restrict__ rec,
                                                             const int* __restrict__ radii, dim3 grid,
                                                             KeyT* __restrict__ keys,
                                                             uint32_t* __restrict__ vals) {
    int slot = blockIdx.x * blockDim.x + threadIdx.x;
    int lane = threadIdx.x & 31;
    uint32_t gid = 0, off = 0, n = 0, x0 = 0, y0 = 0, w = 0;
    if (slot < P) {
        gid = perm[slot];
        int r = radii[gid];
        if (r > 0) {
            off = (slot == 0) ? 0 : offsets[slot - 1];
            float4 a = __ldg(reinterpret_cast<const float4*>(rec + gid));
            uint2 rmin, rmax;
            get_rect(make_float2(a.x, a.y), r, rmin, rmax, grid);
            x0 = rmin.x; y0 = rmin.y;
            w = rmax.x - rmin.x;
            n = w * (rmax.y - rmin.y);
        }
    }
    unsigned any = __ballot_sync(0xffffffffu, n > 0);
    while (any) {
        int src = __ffs(any) - 1;
        any &= any - 1;
        uint32_t g = __shfl_sync(0xffffffffu, gid, src);
        uint32_t o = __shfl_sync(0xffffffffu, off, src);
        uint32_t nn = __shfl_sync(0xffffffffu, n, src);
        uint32_t xx = __shfl_sync(0xffffffffu, x0, src);
        uint32_t yy = __shfl_sync(0xffffffffu, y0, src);
        uint32_t ww = __shfl_sync(0xffffffffu, w, src);
        for (uint32_t k = lane; k < nn; k += 32) {
            uint32_t ty = k / ww, tx = k - ty * ww;
            keys[o + k] = (KeyT)((yy + ty) * grid.x + (xx + tx));  // key = y*grid.x + x, rasterizer_impl.cu:102
            vals[o + k] = g;
        }
    }
}

// Tile ranges of the sorted instance list: same result as identifyTileRanges
// (rasterizer_impl.cu:116-138 — {start, end} of every tile that owns instances, {0, 0} otherwise),
// computed by one thread per TILE with two binary searches instead of one thread per instance
// re-reading the whole key array (R = 45 M keys on K2/K3).
template <typename KeyT>
__global__ void tile_ranges_kernel(int64_t L, uint32_t tiles, const KeyT* __restrict__ keys,
                                   uint2* __restrict__ ranges) {
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= tiles) return;
    auto lower = [&](uint32_t v) {  // first index with key >= v
        int64_t lo = 0, hi = L;
        while (lo < hi) {
            const int64_t mid = (lo + hi) >> 1;
            if ((uint32_t)keys[mid] < v) lo = mid + 1;
            else hi = mid;
        }
        return lo;
    };
    const int64_t a = lower(t), b = lower(t + 1);
    ranges[t] = (b > a) ? make_uint2((uint32_t)a, (uint32_t)b) : make_uint2(0u, 0u);
}

// rasterizer_impl.cu:35-50
uint32_t higher_msb(uint32_t n) {
    uint32_t msb = sizeof(n) * 4;
    uint32_t step = msb;
    while (step > 1) {
        step /= 2;
        if (n >> msb) msb += step;
        else msb -= step;
    }
    if (n >> msb) msb++;
    return msb;
}

}  // namespace

int Scratch::ensure(size_t n) {
    if (n <= cap) return SGB_OK;
    if (p) cudaFree(p);
    p = nullptr;
    cap = 0;
    size_t want = n + (n >> 3) + 4096;
    cudaError_t e = cudaMalloc(&p, want);
    if (e != cudaSuccess) {
        cudaGetLastError();
        set_error("scratch allocation of %zu bytes failed: %s", want, cudaGetErrorString(e));
        p = nullptr;
        return SGB_E_NOMEM;
    }
    cap = want;
    return SGB_OK;
}

// preprocess -> depth order -> scan -> R for V views (one stream sync for all of them; the reference blocks once
// per view, rasterizer_impl.cu:283).  The depth order and the scan land in each view's geometry state, where the
// render call reads them; the views run in stream order, so one scratch slice serves them all.
int run_depth_order_and_scan(sgb_ctx* ctx, const sgb_view_inputs& in_common, int V, const sgb_camera* cams,
                             void* const* geometry_states, int32_t* const* radii_v, int64_t* R_host, cudaStream_t s) {
    const int P = in_common.P;
    // scratch layout: keys_in | keys_out | vals_in | cub temp | 64-bit total
    size_t sort_tmp = 0, scan_tmp = 0;
    cub::DeviceRadixSort::SortPairs(nullptr, sort_tmp, (uint32_t*)nullptr, (uint32_t*)nullptr, (uint32_t*)nullptr,
                                    (uint32_t*)nullptr, P, 0, 32, s);
    cub::DeviceScan::InclusiveSum(nullptr, scan_tmp, (uint32_t*)nullptr, (uint32_t*)nullptr, P, s);
    const size_t arr = align_up(sizeof(uint32_t) * (size_t)P);
    const size_t tmp = align_up(sort_tmp > scan_tmp ? sort_tmp : scan_tmp);
    int rc = ctx->geom.ensure(3 * arr + tmp + 256);
    if (rc) return rc;
    char* base = (char*)ctx->geom.p;
    uint32_t* keys_in = (uint32_t*)(base);
    uint32_t* keys_out = (uint32_t*)(base + arr);
    uint32_t* vals_in = (uint32_t*)(base + 2 * arr);
    void* cub_tmp = base + 3 * arr;
    unsigned long long* total64 = (unsigned long long*)(base + 3 * arr + tmp);
    unsigned long long* h = ctx->pinned->num_rendered;
    for (int v = 0; v < V; v++) {
        const sgb_view_inputs in = with_camera(in_common, cams[v]);
        GeomView g = GeomView::carve(geometry_states[v], P);
        {
            StageTimer t(ctx, ST_PREPROCESS, s);
            rc = launch_preprocess(in, g, radii_v[v], keys_in, s);
            if (rc) return rc;
            ctx->launches += 1;
        }
        {
            StageTimer t(ctx, ST_DEPTH_SORT, s);
            iota_kernel<<<(P + 255) / 256, 256, 0, s>>>(P, vals_in);
            SGB_LAUNCH_CHECK("iota_kernel", in.debug, s);
            SGB_CUDA(cub::DeviceRadixSort::SortPairs(cub_tmp, sort_tmp, keys_in, keys_out, vals_in, g.perm, P, 0, 32, s));
            ctx->launches += 1;
            ctx->lib_launches += 1;
        }
        {
            StageTimer t(ctx, ST_SCAN, s);
            ctx->lib_launches += 1;
            ctx->launches += 1;
            // keys_in is free after the sort: reuse it for the permuted counts
            SGB_CUDA(cudaMemsetAsync(total64, 0, sizeof(unsigned long long), s));
            gather_counts_kernel<<<(P + 255) / 256, 256, 0, s>>>(P, g.perm, g.tiles_touched, keys_in, total64);
            SGB_LAUNCH_CHECK("gather_counts_kernel", in.debug, s);
            SGB_CUDA(cub::DeviceScan::InclusiveSum(cub_tmp, scan_tmp, keys_in, g.offsets, P, s));
        }
        SGB_CUDA(cudaMemcpyAsync(h + v, total64, sizeof(unsigned long long), cudaMemcpyDeviceToHost, s));
    }
    SGB_CUDA(cudaStreamSynchronize(s));
    // 64-bit sums == last element of the 32-bit scans whenever they fit (the caller rejects anything above int32)
    for (int v = 0; v < V; v++) R_host[v] = (int64_t)h[v];
    return SGB_OK;
}

template <typename KeyT>
static int run_binning_t(sgb_ctx* ctx, const sgb_view_inputs& in, int64_t R, GeomView g, BinView b, ImgView im,
                         const int32_t* radii, dim3 tile_grid, cudaStream_t s) {
    const uint32_t tiles = tile_grid.x * tile_grid.y;
    size_t sort_tmp = 0;
    const int bits = (int)higher_msb(tiles);
    cub::DeviceRadixSort::SortPairs(nullptr, sort_tmp, (KeyT*)nullptr, (KeyT*)nullptr, (uint32_t*)nullptr,
                                    (uint32_t*)nullptr, R, 0, bits, s);
    const size_t karr = align_up(sizeof(KeyT) * (size_t)R), varr = align_up(sizeof(uint32_t) * (size_t)R);
    int rc = ctx->bin.ensure(2 * karr + varr + align_up(sort_tmp));
    if (rc) return rc;
    char* base = (char*)ctx->bin.p;
    KeyT* keys_unsorted = (KeyT*)base;
    KeyT* keys_sorted = (KeyT*)(base + karr);
    uint32_t* vals_unsorted = (uint32_t*)(base + 2 * karr);
    void* cub_tmp = base + 2 * karr + varr;
    {
        StageTimer t(ctx, ST_EMIT, s);
        emit_instances_kernel<KeyT><<<(in.P + 255) / 256, 256, 0, s>>>(in.P, g.perm, g.offsets, g.rec, radii, tile_grid,
                                                                      keys_unsorted, vals_unsorted);
        SGB_LAUNCH_CHECK("emit_instances_kernel", in.debug, s);
        ctx->launches += 1;
    }
    {
        StageTimer t(ctx, ST_TILE_SORT, s);
        SGB_CUDA(cub::DeviceRadixSort::SortPairs(cub_tmp, sort_tmp, keys_unsorted, keys_sorted, vals_unsorted,
                                                 b.point_list, R, 0, bits, s));
        ctx->lib_launches += 1;
    }
    {
        StageTimer t(ctx, ST_RANGES, s);
        tile_ranges_kernel<KeyT><<<(tiles + 127) / 128, 128, 0, s>>>(R, tiles, keys_sorted, im.ranges);
        SGB_LAUNCH_CHECK("tile_ranges_kernel", in.debug, s);
        ctx->launches += 1;
    }
    return SGB_OK;
}

// Grows the tile-sort scratch to what R instances need (a batch reserves for its largest view up front so that
// no cudaFree / cudaMalloc — an implicit device sync — lands between the views).
int reserve_binning(sgb_ctx* ctx, const sgb_view_inputs& in, int64_t R, cudaStream_t s) {
    if (R <= 0) return SGB_OK;
    const size_t tiles = (size_t)((in.W + SGB_TILE - 1) / SGB_TILE) * ((in.H + SGB_TILE - 1) / SGB_TILE);
    const int bits = (int)higher_msb((uint32_t)tiles);
    size_t sort_tmp = 0;
    size_t ksz = 4;
    if (tiles <= 0xFFFFu) {
        ksz = 2;
        cub::DeviceRadixSort::SortPairs(nullptr, sort_tmp, (uint16_t*)nullptr, (uint16_t*)nullptr, (uint32_t*)nullptr,
                                        (uint32_t*)nullptr, R, 0, bits, s);
    } else {
        cub::DeviceRadixSort::SortPairs(nullptr, sort_tmp, (uint32_t*)nullptr, (uint32_t*)nullptr, (uint32_t*)nullptr,
                                        (uint32_t*)nullptr, R, 0, bits, s);
    }
    return ctx->bin.ensure(2 * align_up(ksz * (size_t)R) + align_up(sizeof(uint32_t) * (size_t)R) + align_up(sort_tmp));
}

int run_binning(sgb_ctx* ctx, const sgb_view_inputs& in, int64_t R, GeomView g, BinView b, ImgView im,
                const int32_t* radii, cudaStream_t s) {
    dim3 tile_grid((in.W + SGB_TILE - 1) / SGB_TILE, (in.H + SGB_TILE - 1) / SGB_TILE, 1);
    const size_t tiles = (size_t)tile_grid.x * tile_grid.y;
    if (R == 0) {
        SGB_CUDA(cudaMemsetAsync(im.ranges, 0, tiles * sizeof(uint2), s));  // rasterizer_impl.cu:313
        return SGB_OK;
    }
    // 16-bit tile keys halve the key traffic of the R-sized sort whenever the tile count allows it
    if (tiles <= 0xFFFFu) return run_binning_t<uint16_t>(ctx, in, R, g, b, im, radii, tile_grid, s);
    return run_binning_t<uint32_t>(ctx, in, R, g, b, im, radii, tile_grid, s);
}

}  // namespace sgb
