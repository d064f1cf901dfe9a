// Weight pool of the C-channel blend (weight_pool.cuh): the alpha pass that builds a view's pool, the slots a ctx
// keeps, the build / check / regrow protocol, and the per-Gaussian sums of a pool's rows.
#include "weight_pool.cuh"

namespace sgb {

namespace {

// ------------------------------------------------------------------------------------ alpha pass
constexpr int kAB = 32;  // list entries per staging round

struct __align__(16) AlphaSmem {
    float4 recA[kAB];
    float4 recB[kAB];
    uint32_t ids[kAB];
    float wbuf[kAB][SGB_TILE_PIX];
    uint32_t wmask[8];
    uint32_t slot_chunk[kAB];
    uint32_t cur_chunk;
    uint32_t s_last;
};
struct __align__(16) AlphaSmemRgb : AlphaSmem {  // the RGB walk's staging: AlphaSmem's layout, then the colours
    float rgb[kAB][3];
};

// The alpha pass of a view: one walk of its tile lists that writes final_T / n_contrib / tile_last and appends the
// alpha * T row of every blended Gaussian to the weight pool.  With RGB the same walk is also the view's RGB blend
// (the joint colour + feature render): blend_fwd.cu's per-pixel colour accumulation C[k] += f * alpha * T, median
// depth and (EXP_ALPHA) expected depth / alpha in blend_forward_kernel's order, so the RGB outputs are bit for bit
// that kernel's.  The RGB parts are `if constexpr`: a plain `if` changes the integer instruction selection of the
// <false, false> pass.
template <bool RGB, bool EXP_ALPHA>
__global__ void __launch_bounds__(kTileThreads) alpha_pass_kernel(
    const uint2* __restrict__ ranges, const uint32_t* __restrict__ point_list, int W, int H,
    const SplatRec* __restrict__ rec, float* __restrict__ final_T, uint32_t* __restrict__ n_contrib,
    uint32_t* __restrict__ tile_last, PoolView pool, AlphaRgb rgb) {
    extern __shared__ __align__(128) unsigned char smem_raw[];
    AlphaSmem& sm = *reinterpret_cast<AlphaSmem*>(smem_raw);
    float (*s_rgb)[3] = reinterpret_cast<AlphaSmemRgb*>(smem_raw)->rgb;

    const int tiles_x = (W + SGB_TILE - 1) / SGB_TILE;
    const int tile = blockIdx.x;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const uint32_t tx = tid & (SGB_TILE - 1), ty = tid >> 4;
    const uint2 pix = {(uint32_t)(tile % tiles_x) * SGB_TILE + tx, (uint32_t)(tile / tiles_x) * SGB_TILE + ty};
    const uint32_t pix_id = W * pix.y + pix.x;
    const float2 pixf = {(float)pix.x, (float)pix.y};
    const bool inside = pix.x < (uint32_t)W && pix.y < (uint32_t)H;
    bool done = !inside;

    const uint2 range = ranges[tile];
    const int total = (int)(range.y - range.x);
    const int nbatches = (total + kAB - 1) / kAB;
    const uint32_t dbase = range.x / kChunkEntries + (uint32_t)tile;
    if (tid == 0) { sm.cur_chunk = kNone; sm.s_last = 0; }

    float T = 1.0f;
    uint32_t last_contributor = 0;
    uint32_t n_tile = 0;  // entries appended so far (uniform)
    uint32_t n_blend = 0; // Gaussians blended into this pixel

    // Staging of the (id, splat record) batches is software-pipelined in warp 0's registers: the ids run two
    // batches ahead, the records (a dependent gather through the id) one batch ahead, so neither round trip
    // sits between two batches of the chain (it used to: two dependent L2/DRAM latencies per 32 entries).
    auto load_id = [&](int bb) -> uint32_t {
        const int i = bb * kAB + tid;
        return (tid < kAB && bb < nbatches && i < total) ? __ldg(point_list + range.x + i) : 0u;
    };
    uint32_t id_cur = load_id(0), id_nxt = load_id(1);
    float4 rA = make_float4(0.f, 0.f, 0.f, 0.f), rB = rA;
    float c0 = 0.f, c1 = 0.f, c2 = 0.f;  // RGB: the colour of the record in rA / rB
    if (tid < kAB && tid < total) {
        const float4* rp = reinterpret_cast<const float4*>(rec + id_cur);
        rA = __ldg(rp);
        rB = __ldg(rp + 1);
        if constexpr (RGB) {
            c0 = __ldg(rgb.colors + (size_t)id_cur * 3);
            c1 = __ldg(rgb.colors + (size_t)id_cur * 3 + 1);
            c2 = __ldg(rgb.colors + (size_t)id_cur * 3 + 2);
        }
    }
    float acc0 = 0.f, acc1 = 0.f, acc2 = 0.f;  // RGB
    float D = 15.0f;                           // RGB: rgbd forward.cu:308, default median depth
    float acc_z = 0.f, acc_w = 0.f;            // EXP_ALPHA: E and A
    for (int b = 0; b < nbatches; b++) {
        const int num_done = __syncthreads_count(done);  // forward.cu:310-312
        if (num_done == kTileThreads) break;
        const int base = b * kAB;
        const int cnt = min(kAB, total - base);
        if (tid < cnt) {
            sm.ids[tid] = id_cur;
            sm.recA[tid] = rA;
            sm.recB[tid] = rB;
            if constexpr (RGB) {
                s_rgb[tid][0] = c0;
                s_rgb[tid][1] = c1;
                s_rgb[tid][2] = c2;
            }
        }
        __syncthreads();
        if (tid < kAB) {  // records of batch b+1 (its ids are already here), ids of batch b+2
            id_cur = id_nxt;
            if (base + kAB + tid < total) {
                const float4* rp = reinterpret_cast<const float4*>(rec + id_cur);
                rA = __ldg(rp);
                rB = __ldg(rp + 1);
                if constexpr (RGB) {
                    c0 = __ldg(rgb.colors + (size_t)id_cur * 3);
                    c1 = __ldg(rgb.colors + (size_t)id_cur * 3 + 1);
                    c2 = __ldg(rgb.colors + (size_t)id_cur * 3 + 2);
                }
            }
            id_nxt = load_id(b + 2);
        }
        uint32_t my_mask = 0;
        for (int j = 0; j < cnt; j++) {
            float w = 0.f;
            if (!done) {
                // forward.cu:333-362 verbatim
                const float4 a = sm.recA[j];
                const float2 xy = {a.x, a.y};
                const float2 d = {xy.x - pixf.x, xy.y - pixf.y};
                const float4 con_o = sm.recB[j];
                const float power = -0.5f * (con_o.x * d.x * d.x + con_o.z * d.y * d.y) - con_o.y * d.x * d.y;
                if (!(power > 0.0f)) {
                    const float alpha = min(0.99f, con_o.w * exp(power));
                    if (!(alpha < 1.0f / 255.0f)) {
                        const float test_T = T * (1 - alpha);
                        if (test_T < 0.0001f) {
                            done = true;
                        } else {
                            if constexpr (RGB) {
                                // blend_fwd.cu: forward.cu:355-356, median and expected depth, in its order
                                acc0 += s_rgb[j][0] * alpha * T;
                                acc1 += s_rgb[j][1] * alpha * T;
                                acc2 += s_rgb[j][2] * alpha * T;
                                if (T > 0.5f && test_T < 0.5) D = a.z;
                                if constexpr (EXP_ALPHA) {
                                    acc_z += a.z * alpha * T;
                                    // blend_fwd.cu's `acc_w += 1.0f * alpha * T` compiles to one FFMA; here the
                                    // product alpha * T is also the weight, and would be reused rounded
                                    acc_w = __fmaf_rn(alpha, T, acc_w);
                                }
                            }
                            w = alpha * T;
                            T = test_T;
                            last_contributor = (uint32_t)(base + j + 1);
                        }
                    }
                }
            }
            sm.wbuf[j][tid] = w;
            n_blend += (w != 0.f);
            if (__ballot_sync(0xffffffffu, w != 0.f)) my_mask |= 1u << j;
        }
        if (lane == 0) sm.wmask[warp] = my_mask;
        __syncthreads();
        uint32_t tm = 0;
#pragma unroll
        for (int q = 0; q < 8; q++) tm |= sm.wmask[q];
        const int n_act = __popc(tm);
        if (n_act) {
            if (tid == 0) {
                uint32_t e = n_tile, cur = sm.cur_chunk;
                for (int k = 0; k < n_act; k++, e++) {
                    if ((e & (kChunkEntries - 1)) == 0) {
                        uint32_t nw = atomicAdd(&pool.hdr->counter, 1u);
                        if (nw >= pool.capacity) {
                            pool.hdr->overflow = 1;
                            nw = pool.capacity - 1;
                        }
                        pool.dir[dbase + e / kChunkEntries] = nw;
                        cur = nw;
                    }
                    sm.slot_chunk[k] = cur;
                }
                sm.cur_chunk = cur;
            }
            __syncthreads();
            int k = 0;
            for (uint32_t m = tm; m; m &= m - 1, k++) {
                const int j = __ffs(m) - 1;
                const uint32_t e = n_tile + k;
                WChunk& ck = pool.chunks[sm.slot_chunk[k]];
                const int s = e & (kChunkEntries - 1);
                ck.w[s][tid] = sm.wbuf[j][tid];
                if (tid == 0) {
                    uint32_t strips = 0;
#pragma unroll
                    for (int q = 0; q < 8; q++) strips |= ((sm.wmask[q] >> j) & 1u) << q;
                    ck.meta[s] = make_uint2(sm.ids[j], strips);
                }
            }
            n_tile += n_act;
        }
    }
    if (inside) {
        final_T[pix_id] = T;
        n_contrib[pix_id] = last_contributor;
        atomicMax(&sm.s_last, last_contributor);
        if constexpr (RGB) {
            const size_t plane = (size_t)H * W;
            rgb.out_color[pix_id] = acc0 + T * rgb.bg[0];
            rgb.out_color[plane + pix_id] = acc1 + T * rgb.bg[1];
            rgb.out_color[2 * plane + pix_id] = acc2 + T * rgb.bg[2];
            rgb.out_depth[pix_id] = D;
            if constexpr (EXP_ALPHA) {
                rgb.out_exp_depth[pix_id] = acc_z;
                rgb.out_alpha[pix_id] = acc_w;
            }
        }
    }
    n_blend = __reduce_add_sync(0xffffffffu, n_blend);
    if (lane == 0 && n_blend) atomicAdd(&pool.hdr->blended, (unsigned long long)n_blend);
    __syncthreads();
    if (tid == 0) {
        tile_last[tile] = sm.s_last;
        pool.count[tile] = n_tile;
        pool.dirbase[tile] = dbase;
    }
}


// weight_sum[g] += sum over the tile's pixels of w[entry][px], for every entry of every tile of a view's pool: the
// denominator of a lift (sgb_lift_batch).  CTA = tile, warp = one 16-entry chunk at a time; every row is read once,
// by all 32 lanes (two coalesced float4 per lane), and reduced across the warp.
__global__ void __launch_bounds__(kTileThreads) pool_weight_sum_kernel(PoolView pool, float* __restrict__ weight_sum) {
    const int tile = blockIdx.x, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const uint32_t n = pool.count[tile];
    const uint32_t dbase = pool.dirbase[tile];
    const int nck = (int)((n + kChunkEntries - 1) / kChunkEntries);
    for (int k = warp; k < nck; k += kTileThreads / 32) {
        const WChunk* ck = pool.chunks + chunk_of(pool, dbase, k);
        const int m = (int)min((uint32_t)kChunkEntries, n - (uint32_t)k * kChunkEntries);
#pragma unroll 4
        for (int s = 0; s < m; s++) {
            const float4 a = __ldg(reinterpret_cast<const float4*>(&ck->w[s][4 * lane]));
            const float4 b = __ldg(reinterpret_cast<const float4*>(&ck->w[s][128 + 4 * lane]));
            float t = ((a.x + a.y) + (a.z + a.w)) + ((b.x + b.y) + (b.z + b.w));
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
            if (lane == 0) red_add_f32(weight_sum + __ldg(&ck->meta[s].x), t);
        }
    }
}

// ------------------------------------------------------------------------------------ host side
size_t pool_bytes(int tiles, uint32_t chunks, int64_t R, PoolView* v, void* base) {
    size_t off = 0;
    char* p = (char*)base;
    auto take = [&](size_t n) { size_t o = off; off += align_up(n); return p ? p + o : nullptr; };
    void* hdr = take(sizeof(PoolHdr));
    void* dbase = take(4 * (size_t)tiles);
    void* cnt = take(4 * (size_t)tiles);
    void* dir = take(4 * ((size_t)(R / kChunkEntries) + (size_t)tiles + 1));
    void* ch = take(sizeof(WChunk) * (size_t)chunks);
    if (v) {
        v->hdr = (PoolHdr*)hdr; v->dirbase = (uint32_t*)dbase; v->count = (uint32_t*)cnt; v->dir = (uint32_t*)dir;
        v->chunks = (WChunk*)ch; v->capacity = chunks;
    }
    return off;
}

}  // namespace

// ---- weight-pool slots ---------------------------------------------------------------------------------------
// A view's slot is the one keyed by its binning-state pointer.
constexpr int kMaxAlphaPasses = 4;  // per view and call: the first guess and up to three grown pools

static PoolSlot* slot_of(sgb_ctx* ctx, const ViewState& w) {
    for (PoolSlot& sl : ctx->pools->slots)
        if (sl.key_bin == (const void*)w.b.point_list) return &sl;
    return nullptr;
}

// The pool header of slot i is read back through pinned header i.
static inline PoolHdr* pinned_hdr(sgb_ctx* ctx, const PoolSlot* sl) {
    return &ctx->pinned->pool_hdr[sl - ctx->pools->slots];
}

static PoolView slot_view(const ViewState& w, const PoolSlot& sl) {
    PoolView pv;
    pool_bytes(num_tiles(w.in), sl.chunks, w.R, &pv, sl.mem.p);
    return pv;
}

static uint64_t pool_first_guess(sgb_ctx* ctx, int tiles, int64_t R) {
    // ~8 chunks (128 touching Gaussians) per tile, bounded by the instance count, at least the high-water mark
    uint64_t guess = (uint64_t)tiles * 8;
    const uint64_t by_R = (uint64_t)(R / kChunkEntries) + (uint64_t)tiles;
    if (guess > by_R) guess = by_R;
    if (guess < ctx->pools->chunks_hint) guess = ctx->pools->chunks_hint;
    if (guess < 16) guess = 16;
    return guess;
}

// Slot of a view that is about to be (re)built: the one already keyed by its binning state (a new forward through
// the same pointer replaces it), else an empty one, else the least recently used.  It is carved for the first guess,
// or keeps a larger existing carve that its memory still holds.
int weight_pool_build(sgb_ctx* ctx, const ViewState& w, cudaStream_t s, const AlphaRgb* rgb) {
    PoolSlot* sl = slot_of(ctx, w);
    if (!sl)
        for (PoolSlot& c : ctx->pools->slots)
            if (!c.valid && !c.key_bin) { sl = &c; break; }
    if (!sl) {
        sl = &ctx->pools->slots[0];
        for (PoolSlot& c : ctx->pools->slots)
            if (c.stamp < sl->stamp) sl = &c;
    }
    sl->valid = false;
    sl->key_bin = (const void*)w.b.point_list;
    sl->stamp = ++ctx->pools->clock;
    const int tiles = num_tiles(w.in);
    uint64_t want = pool_first_guess(ctx, tiles, w.R);
    if (sl->chunks > want && sl->mem.cap >= pool_bytes(tiles, sl->chunks, w.R, nullptr, nullptr)) want = sl->chunks;
    const uint32_t chunks = (uint32_t)want;
    int rc = sl->mem.ensure(pool_bytes(tiles, chunks, w.R, nullptr, nullptr));
    if (rc) return rc;
    sl->chunks = chunks;
    const PoolView pv = slot_view(w, *sl);
    static DeviceOnce attr_set;
    if (attr_set.first_use_on_device()) {
        SGB_CUDA(cudaFuncSetAttribute(alpha_pass_kernel<false, false>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                      (int)sizeof(AlphaSmem)));
        SGB_CUDA(cudaFuncSetAttribute(alpha_pass_kernel<true, false>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                      (int)sizeof(AlphaSmemRgb)));
        SGB_CUDA(cudaFuncSetAttribute(alpha_pass_kernel<true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                      (int)sizeof(AlphaSmemRgb)));
    }
    SGB_CUDA(cudaMemsetAsync(pv.hdr, 0, sizeof(PoolHdr), s));
    {
        StageTimer t(ctx, ST_ALPHA, s);
        auto kern = !rgb ? alpha_pass_kernel<false, false>
                    : rgb->out_exp_depth ? alpha_pass_kernel<true, true> : alpha_pass_kernel<true, false>;
        kern<<<tiles, kTileThreads, rgb ? sizeof(AlphaSmemRgb) : sizeof(AlphaSmem), s>>>(
            w.im.ranges, w.b.point_list, w.in.W, w.in.H, w.g.rec, w.im.final_T, w.im.n_contrib, w.im.tile_last, pv,
            rgb ? *rgb : AlphaRgb{});
        SGB_LAUNCH_CHECK("alpha_pass_kernel", w.in.debug, s);
        ctx->launches += 1;
    }
    SGB_CUDA(cudaMemcpyAsync(pinned_hdr(ctx, sl), pv.hdr, sizeof(PoolHdr), cudaMemcpyDeviceToHost, s));
    return SGB_OK;
}

// A pool that overflowed is re-carved for the demand its header reports (the counter keeps counting past capacity)
// and built again; the rebuilt views are checked after one more sync.
int weight_pool_settle(sgb_ctx* ctx, int V, const ViewState* vw, PoolView* pv, cudaStream_t s, const bool* only) {
    bool pending[SGB_MAX_BATCH];
    for (int v = 0; v < V; v++) pending[v] = !only || only[v];
    for (int pass = 1;; pass++) {
        SGB_CUDA(cudaStreamSynchronize(s));
        bool again = false;
        for (int v = 0; v < V; v++) {
            if (!pending[v]) continue;
            const ViewState& w = vw[v];
            PoolSlot* sl = slot_of(ctx, w);
            if (!sl) { set_error("weight-pool slot of the view vanished"); return SGB_E_INVALID; }
            const PoolHdr h = *pinned_hdr(ctx, sl);
            if (h.overflow) {
                const uint64_t need = (uint64_t)h.counter + h.counter / 8 + 64;
                if (need > ctx->pools->chunks_hint) ctx->pools->chunks_hint = need;
                sl->chunks = 0;  // re-carve with the new hint
                if (pass == kMaxAlphaPasses) { set_error("weight pool kept overflowing"); return SGB_E_NOMEM; }
                int rc = weight_pool_build(ctx, w, s);
                if (rc) return rc;
                again = true;
                continue;
            }
            ctx->pools->stat_blended_pairs = (int64_t)h.blended;
            ctx->pools->stat_pool_chunks = h.counter;
            if (h.counter > ctx->pools->chunks_hint) ctx->pools->chunks_hint = (uint64_t)h.counter + h.counter / 16 + 16;
            sl->valid = true;
            sl->key_R = w.R;
            sl->key_W = w.in.W;
            sl->key_H = w.in.H;
            sl->key_P = w.in.P;
            pv[v] = slot_view(w, *sl);
            pending[v] = false;
        }
        if (!again) return SGB_OK;
    }
}

// A rebuild is needed only when the forward ran through another ctx or its slot was recycled.  Every hit is stamped
// before the first miss takes a slot, so the least recently used slot a miss may evict is never one of this batch.
int weight_rows_for_backward(sgb_ctx* ctx, int V, const ViewState* vw, PoolView* pv, cudaStream_t s) {
    bool miss[SGB_MAX_BATCH] = {};
    bool any = false;
    for (int v = 0; v < V; v++) {
        const ViewState& w = vw[v];
        if (w.R <= 0) continue;
        PoolSlot* sl = slot_of(ctx, w);
        if (sl && sl->valid && sl->key_R == w.R && sl->key_W == w.in.W && sl->key_H == w.in.H && sl->key_P == w.in.P) {
            sl->stamp = ++ctx->pools->clock;
            pv[v] = slot_view(w, *sl);
        } else {
            miss[v] = any = true;
        }
    }
    if (!any) return SGB_OK;
    for (int v = 0; v < V; v++) {
        if (!miss[v]) continue;
        int rc = weight_pool_build(ctx, vw[v], s);
        if (rc) return rc;
    }
    return weight_pool_settle(ctx, V, vw, pv, s, miss);
}

// A lift keeps nothing for a backward: its slots are emptied (not left valid under a scratch address that a later
// binning state could reuse) and are the first a later build takes, ahead of any training forward's slot.
void weight_pool_release(sgb_ctx* ctx, int V, const ViewState* vw) {
    for (int v = 0; v < V; v++)
        if (PoolSlot* sl = slot_of(ctx, vw[v])) {
            sl->valid = false;
            sl->key_bin = nullptr;
        }
}

int pool_weight_sums(sgb_ctx* ctx, const ViewState& w, const PoolView& pv, float* weight_sum, cudaStream_t s) {
    StageTimer t(ctx, ST_WEIGHT_SUM, s);
    ctx->launches += 1;
    pool_weight_sum_kernel<<<num_tiles(w.in), kTileThreads, 0, s>>>(pv, weight_sum);
    SGB_LAUNCH_CHECK("pool_weight_sum_kernel", w.in.debug, s);
    return SGB_OK;
}

}  // namespace sgb
