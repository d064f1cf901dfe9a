// Weight pool of the C-channel blend: per tile the alpha * T rows of every Gaussian that touches it, in 16-entry
// chunks found through a per-tile directory.  One pool holds the rows of ONE view; it is built by the view's alpha
// pass and read by the contraction stages (chn_blend.cuh).  The pools are the only thing a ctx carries from one call
// to the next.
#pragma once
#include "common.cuh"

namespace sgb {

constexpr int kTileThreads = SGB_TILE_PIX;  // the alpha pass and every consumer of a pool: CTA thread = tile pixel
constexpr int kChunkEntries = 16;
constexpr uint32_t kNone = 0xFFFFFFFFu;

static inline int num_tiles(const sgb_view_inputs& in) {
    return ((in.W + SGB_TILE - 1) / SGB_TILE) * ((in.H + SGB_TILE - 1) / SGB_TILE);
}

struct __align__(16) WChunk {
    uint32_t pad[4];
    uint2 meta[kChunkEntries];             // x: Gaussian id, y: bit w = strip (warp) w has a non-zero weight
    float w[kChunkEntries][SGB_TILE_PIX];  // alpha * T per pixel (tile-local index ty*16+tx)
};
static_assert(sizeof(WChunk) % 16 == 0, "WChunk must keep 16-byte alignment in an array");

struct PoolHdr {
    uint32_t counter;   // chunks handed out (keeps counting past capacity: the true demand)
    uint32_t overflow;  // set when counter ran past capacity (results invalid, caller retries)
    unsigned long long blended;  // (pixel, Gaussian) pairs that were blended: n-bar * W * H (reported by bench.py)
};

// A tile's chunks are found through a DIRECTORY (no linked list, no pointer chasing): chunk k of tile t is
// dir[dirbase[t] + k] with dirbase[t] = ranges[t].x / 16 + t.  The tile ranges are disjoint intervals of the
// sorted instance list, a tile with `len` instances needs at most ceil(len / 16) chunks, and
// floor(x/16) + ceil(len/16) <= floor((x+len)/16) + 1, so the regions cannot overlap and R/16 + tiles + 1
// directory slots always suffice — no scan, no capacity guess.
struct PoolView {
    PoolHdr* hdr;
    uint32_t* dirbase;  // [tiles] first directory slot of the tile
    uint32_t* count;    // [tiles] entries
    uint32_t* dir;      // [R/16 + tiles + 1] chunk indices
    WChunk* chunks;
    uint32_t capacity;
};

__device__ __forceinline__ uint32_t chunk_of(const PoolView& pool, uint32_t dbase, int k) {
    return min(__ldg(pool.dir + dbase + k), pool.capacity - 1);
}

// ------------------------------------------------------------------ what a ctx keeps
// A slot is identified by the view's binning-state pointer: a new forward through the same pointer necessarily
// overwrites that slot, so a slot can never describe a different view's instance list.
struct PoolSlot {
    Scratch mem;
    bool valid = false;
    const void* key_bin = nullptr;
    int64_t key_R = 0;
    int key_W = 0, key_H = 0, key_P = 0;
    uint32_t chunks = 0;   // capacity the slot was carved with
    uint64_t stamp = 0;    // LRU clock
};

struct WeightPools {
    // As many slots as views per batch, so that the backward of each view of a batch (or of a forward-forward-...-
    // backward-backward sequence) finds the rows its forward built: the backward resolves the rows of all V views
    // before its first kernel, and V <= slots guarantees that rebuilding one view cannot evict another view of the
    // same batch.
    PoolSlot slots[SGB_MAX_BATCH];
    uint64_t clock = 0;
    uint64_t chunks_hint = 0;        // high-water mark of the pool demand (chunks)
    int64_t stat_blended_pairs = 0;  // last alpha pass: blended (pixel, Gaussian) pairs
    int64_t stat_pool_chunks = 0;    // last alpha pass: 16-entry weight-row chunks in use
    ~WeightPools() {
        for (PoolSlot& sl : slots)
            if (sl.mem.p) cudaFree(sl.mem.p);
    }
    size_t bytes() const {
        size_t n = 0;
        for (const PoolSlot& sl : slots) n += sl.mem.cap;
        return n;
    }
};

// The ctx's host-pinned buffer: what a call reads back under one stream sync.  The views of one batch have distinct
// slots, so one sync reads all their pool headers.
struct Readback {
    unsigned long long num_rendered[SGB_MAX_BATCH];  // instance count of every view of a geometry batch (binning.cu)
    PoolHdr pool_hdr[SGB_MAX_BATCH];                 // pool header of every slot
};

// The RGB image a view's alpha pass may produce on the same walk (the joint colour + feature render): the blend of
// `colors` (P, 3) over `bg` (3) into out_color (3, H, W) and the median depth into out_depth (1, H, W), bit for bit
// what launch_blend_forward writes; out_exp_depth / out_alpha (both or neither) the expected depth and alpha.
struct AlphaRgb {
    const float* colors;
    const float* bg;
    float* out_color;
    float* out_depth;
    float* out_exp_depth;
    float* out_alpha;
};

// ------------------------------------------------------------------ host entry points
//   weight_pool_build         enqueue the alpha pass of one view into its slot (no sync), so that a batch enqueues
//                             the alpha passes of all its views before the one sync that checks their pools (with
//                             `rgb`, the same walk is also the view's RGB blend; a rebuild after an overflow runs
//                             without it, since the walk and so the RGB outputs do not depend on the pool)
//   weight_pool_settle        one stream sync, then the pool check of views [0, V) (of those with only[v], when
//                             given); a view whose pool overflowed is grown and built again; fills pv[v]
//   weight_rows_for_backward  pv[v] of every view with R > 0: the slot its forward filled, else rebuilt (all misses
//                             under one sync)
//   weight_pool_release       empties the slots of views [0, V): a lift keeps nothing for a backward
// The blend kernels take the PoolView and look up nothing.
int weight_pool_build(sgb_ctx* ctx, const ViewState& w, cudaStream_t s, const AlphaRgb* rgb = nullptr);
int weight_pool_settle(sgb_ctx* ctx, int V, const ViewState* vw, PoolView* pv, cudaStream_t s,
                       const bool* only = nullptr);
int weight_rows_for_backward(sgb_ctx* ctx, int V, const ViewState* vw, PoolView* pv, cudaStream_t s);
void weight_pool_release(sgb_ctx* ctx, int V, const ViewState* vw);
// weight_sum[g] += sum_px w over every entry of the view's pool (the denominator of a lift)
int pool_weight_sums(sgb_ctx* ctx, const ViewState& w, const PoolView& pv, float* weight_sum, cudaStream_t s);

}  // namespace sgb
