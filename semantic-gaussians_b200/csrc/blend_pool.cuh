// Weight pool of the C-channel blend (blend_v3.cu): per tile the alpha * T rows of every Gaussian that touches it,
// in 16-entry chunks found through a per-tile directory.
#pragma once
#include "common.cuh"

namespace sgb {

constexpr int kChunkEntries = 16;
constexpr uint32_t kNone = 0xFFFFFFFFu;

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

}  // namespace sgb
