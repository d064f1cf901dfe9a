// OPT-IN tensor-core versions of the three C-channel contractions (SGB_BLEND_MMA=1) — an experiment, not the
// default path.
//
// With the per-tile weights materialised once (blend_v3.cu) the forward is a dense contraction
// out[256 px][C] = W^T[256 px][n] . F[n][C], and the backward has two more of the same shape (dL/dfeature and the
// s-pass of the chain).  The default kernels run them on the CUDA cores in fp32.  This file runs them on the Hopper
// tensor cores (wgmma.mma_async, operands in shared memory, fp32 accumulators in registers) with fp32 accuracy
// recovered by the error-compensated 3 x TF32 split
//     x = hi + lo,  hi = tf32(x) (round to nearest),  lo = tf32(x - hi)       (|lo| <= 2^-12 |x|)
//     w * f  ~=  hi_w * hi_f + hi_w * lo_f + lo_w * hi_f                      (lo_w * lo_f <= 2^-24 |w f| dropped)
// three kind::tf32 MMAs per K block accumulating in fp32.
//
// Kernel layout: CTA = (tile, 128-channel slice), 256 threads = 2 warpgroups.  Per batch of 16 list entries every
// thread moves 6 x 16 B of raw fp32 operands global -> registers (two batches ahead) -> hi / lo copies in shared
// memory, laid out as the canonical K-major no-swizzle operand (16-byte chunk = 4 consecutive entries k of one row,
// 8 rows = one 128-byte core matrix; LBO = distance of the two K halves, SBO = distance of 8-row groups).  After a
// CTA barrier each warpgroup issues the wgmma of its own 128-pixel half (2 x m64n128k8 per K block and product) and
// commits them as one group; a stage buffer is refilled only after wgmma.wait_group has retired the group that read
// it in both warpgroups.  The epilogue reads the accumulators from registers, adds T * bg and stores the planar image.
// Reference semantics: forward.cu:355-356, 372-373 (accumulation order differs: fp32 tree inside the tensor core).
#include <cstdlib>
#include "common.cuh"
#include "blend_pool.cuh"

namespace sgb {

namespace {

constexpr int kMmaThreads = 256;
constexpr int kNch = 128;              // channels per CTA (MMA N)
constexpr int kBatch = 16;             // list entries per pipeline stage = 2 K blocks of 8
// Operand blocks (one K block of 8 entries x 128 rows).  Operands written by TRANSPOSING scalar stores use a padded
// geometry — leading offset (second K half) 144 B, row-group stride 288 B instead of 128 / 256 — which the matrix
// descriptor expresses directly (LBO / SBO are free parameters) and which makes the 32 scalar stores of a warp hit 32
// distinct banks.  Operands stored with 16-byte pieces in their natural order keep the dense 128 / 256 geometry.
constexpr uint32_t kLboPad = 144, kSboPad = 288;
constexpr uint32_t kABlk = 16 * kSboPad;   // bytes of one (K block, pixel half) operand block: 16 row groups
constexpr uint32_t kBBlk = (kNch / 8) * kSboPad;
constexpr uint32_t kStageA = 2 * 2 * kABlk;   // [kb][mh]
constexpr uint32_t kStageB = 2 * kBBlk;       // [kb]
constexpr uint32_t kStageBytes = 2 * kStageA + 2 * kStageB;   // hi + lo of both operands = 48 KB
constexpr int kStages = 2;

__device__ __forceinline__ uint64_t wgmma_desc(uint32_t saddr, uint32_t lead_bytes, uint32_t stride_bytes) {
    uint64_t d = 0;
    d |= (uint64_t)((saddr >> 4) & 0x3FFF);
    d |= (uint64_t)((lead_bytes >> 4) & 0x3FFF) << 16;
    d |= (uint64_t)((stride_bytes >> 4) & 0x3FFF) << 32;
    return d;  // base offset 0, no swizzle
}
// D[64 rows][128 cols] += A[64][8] . B[128][8]^T, both operands K-major in shared memory, fp32 accumulators in the
// warpgroup's registers: row (warp % 4) * 16 + lane / 4 + 8 i, column 8 n + 2 (lane % 4) + j  <->  d[4 n + 2 i + j].
__device__ __forceinline__ void wgmma_tf32_m64n128(float (&d)[64], uint64_t da, uint64_t db) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "l"(da), "l"(db));
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait_acc(float (&d)[N]) {  // keeps the accumulators live across the wait
    wgmma_wait<0>();
#pragma unroll
    for (int i = 0; i < N; i++) asm volatile("" : "+f"(d[i])::"memory");
}
__device__ __forceinline__ float tf32_rna(float x) {  // round to nearest TF32 (low 13 mantissa bits zero)
    uint32_t u;
    asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(u) : "f"(x));
    return __uint_as_float(u);
}
__device__ __forceinline__ float4 tf32_hi(float4 x) {
    return make_float4(tf32_rna(x.x), tf32_rna(x.y), tf32_rna(x.z), tf32_rna(x.w));
}
__device__ __forceinline__ float4 sub4(float4 a, float4 b) { return make_float4(a.x - b.x, a.y - b.y, a.z - b.z, a.w - b.w); }
// three products of the 3 x TF32 split, small terms first
__device__ __forceinline__ void mma3(float (&d)[64], uint32_t a_hi, uint32_t a_lo, uint32_t a_lbo, uint32_t a_sbo,
                                     uint32_t b_hi, uint32_t b_lo, uint32_t b_lbo, uint32_t b_sbo) {
    const uint64_t dah = wgmma_desc(a_hi, a_lbo, a_sbo), dal = wgmma_desc(a_lo, a_lbo, a_sbo);
    const uint64_t dbh = wgmma_desc(b_hi, b_lbo, b_sbo), dbl = wgmma_desc(b_lo, b_lbo, b_sbo);
    wgmma_tf32_m64n128(d, dal, dbh);
    wgmma_tf32_m64n128(d, dah, dbl);
    wgmma_tf32_m64n128(d, dah, dbh);
}

__global__ void __launch_bounds__(kMmaThreads, 1) blend_forward_mma_kernel(
    int W, int H, int C, const float* __restrict__ features, const float* __restrict__ bg_color,
    const float* __restrict__ final_T, PoolView pool, float* __restrict__ out_color) {
    extern __shared__ __align__(128) unsigned char smem_raw[];
    __shared__ uint32_t Cdir[192];
    __shared__ float bgS[kNch];

    const int tiles_x = (W + SGB_TILE - 1) / SGB_TILE;
    const int nslices = (C + kNch - 1) / kNch;
    const int tile = blockIdx.x / nslices;
    const int ch0 = (blockIdx.x % nslices) * kNch;
    const int nch = min(kNch, C - ch0);
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, wg = warp >> 2;
    const uint2 pix_min = {(uint32_t)(tile % tiles_x) * SGB_TILE, (uint32_t)(tile / tiles_x) * SGB_TILE};
    const size_t plane = (size_t)H * W;
    const uint32_t n = pool.count[tile];
    const uint32_t dbase = pool.dirbase[tile];
    if (tid < nch) bgS[tid] = bg_color[ch0 + tid];

    if (n == 0) {  // nothing blended: out = T * bg (forward.cu:372-373)
        __syncthreads();
        const uint32_t px = pix_min.x + (tid & 15), py = pix_min.y + (tid >> 4);
        if (px < (uint32_t)W && py < (uint32_t)H) {
            const float Tfin = final_T[(size_t)W * py + px];
            for (int c = 0; c < nch; c++) out_color[(size_t)(ch0 + c) * plane + (size_t)W * py + px] = Tfin * bgS[c];
        }
        return;
    }
    const int nb = (int)((n + kBatch - 1) / kBatch);
    for (int k = tid; k < min(nb, 192); k += kMmaThreads) Cdir[k] = chunk_of(pool, dbase, k);
    __syncthreads();

    auto chunk_ptr = [&](int bi) { return pool.chunks + (bi < 192 ? Cdir[bi] : chunk_of(pool, dbase, bi)); };

    // ---- staging roles.  lane -> (qq = lane >> 3: one of 4 adjacent 16-byte pieces, e8 = lane & 7: entry of the K
    // block): 8 lanes fill one 128-byte core matrix, a warp 512 contiguous bytes; per row 64 contiguous global bytes.
    const int qq = lane >> 3, e8 = lane & 7;
    // raw operands of the next TWO batches live in two explicit register sets (global latency >> one batch of MMAs)
    float4 wregA[4], fregA[2], wregB[4], fregB[2];
    auto load_batch = [&](int b, float4 (&wreg)[4], float4 (&freg)[2]) {
        const WChunk* ck = chunk_ptr(b);
        const int left = (int)n - b * kBatch;  // entries of this batch that exist
#pragma unroll
        for (int it = 0; it < 4; it++) {
            const int c = it * 8 + warp, kb = c >> 4, qblk = c & 15;
            const int e = kb * 8 + e8;
            wreg[it] = make_float4(0.f, 0.f, 0.f, 0.f);
            if (e < left) wreg[it] = __ldg(reinterpret_cast<const float4*>(&ck->w[e][(qblk * 4 + qq) * 4]));
        }
#pragma unroll
        for (int it = 0; it < 2; it++) {
            const int e = it * 8 + e8;           // kb = it
            const int chl = (warp * 4 + qq) * 4; // channel of this 16-byte piece inside the slice
            freg[it] = make_float4(0.f, 0.f, 0.f, 0.f);
            if (e < left && chl < nch) {
                const uint32_t gid = __ldg(&ck->meta[e].x);
                freg[it] = __ldg(reinterpret_cast<const float4*>(features + (size_t)gid * C + ch0 + chl));
            }
        }
    };
    // K-major no-swizzle operand block: element (row r of the 128-row block, entry k of the 8-entry K block) at
    //     (r / 8) * SBO + (k / 4) * LBO + (r % 8) * 16 + (k % 4) * 4          (LBO = 144 B, SBO = 288 B, see above).
    // A thread holds 4 consecutive rows of ONE entry (a 16-byte piece of a weight / feature row), i.e. 4 scalar stores.
    auto put4 = [&](unsigned char* blk, int r0, float4 v) {
        const uint32_t col = (uint32_t)(e8 >> 2) * kLboPad + (uint32_t)(e8 & 3) * 4u;
        const float x[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
        for (int j = 0; j < 4; j++) {
            const int r = r0 + j;
            *reinterpret_cast<float*>(blk + (uint32_t)(r >> 3) * kSboPad + (uint32_t)(r & 7) * 16u + col) = x[j];
        }
    };
    auto store_batch = [&](int st, float4 (&wreg)[4], float4 (&freg)[2]) {
        unsigned char* base = smem_raw + (size_t)st * kStageBytes;
        unsigned char* a_hi = base;
        unsigned char* a_lo = base + kStageA;
        unsigned char* b_hi = base + 2 * kStageA;
        unsigned char* b_lo = base + 2 * kStageA + kStageB;
#pragma unroll
        for (int it = 0; it < 4; it++) {
            const int c = it * 8 + warp, kb = c >> 4, qblk = c & 15;
            const int q = qblk * 4 + qq, mh = q >> 5, ql = q & 31;
            const uint32_t blk = (uint32_t)(kb * 2 + mh) * kABlk;
            const float4 hi = tf32_hi(wreg[it]);
            put4(a_hi + blk, ql * 4, hi);
            put4(a_lo + blk, ql * 4, tf32_hi(sub4(wreg[it], hi)));
        }
#pragma unroll
        for (int it = 0; it < 2; it++) {
            const int q = warp * 4 + qq;
            const float4 hi = tf32_hi(freg[it]);
            put4(b_hi + (uint32_t)it * kBBlk, q * 4, hi);
            put4(b_lo + (uint32_t)it * kBBlk, q * 4, tf32_hi(sub4(freg[it], hi)));
        }
    };

    float acc[2][64];  // this warpgroup's pixel half as two 64-row blocks
#pragma unroll
    for (int m = 0; m < 2; m++)
#pragma unroll
        for (int i = 0; i < 64; i++) acc[m][i] = 0.f;

    auto step = [&](int b, float4 (&wreg)[4], float4 (&freg)[2]) {
        const int st = b % kStages;
        if (b >= kStages) {  // the MMAs of batch b - 2 (the last reader of this stage buffer) retired in both warpgroups
            wgmma_wait<kStages - 1>();
            __syncthreads();
        }
        store_batch(st, wreg, freg);
        if (b + 2 < nb) load_batch(b + 2, wreg, freg);  // lands while the tensor core works on this batch and the next
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");  // generic stores -> visible to the tensor core
        __syncthreads();
        const uint32_t sbase = smem_u32(smem_raw) + (uint32_t)st * kStageBytes;
        const int nkb = ((int)n - b * kBatch > 8) ? 2 : 1;  // a batch whose second K block is empty skips it
        wgmma_fence();
        for (int kb = 0; kb < nkb; kb++) {
            const uint32_t bh = sbase + 2 * kStageA + kb * kBBlk, bl = bh + kStageB;
#pragma unroll
            for (int m = 0; m < 2; m++) {
                const uint32_t ah = sbase + (uint32_t)(kb * 2 + wg) * kABlk + (uint32_t)m * 8u * kSboPad, al = ah + kStageA;
                mma3(acc[m], ah, al, kLboPad, kSboPad, bh, bl, kLboPad, kSboPad);
            }
        }
        wgmma_commit();
    };
    load_batch(0, wregA, fregA);
    if (nb > 1) load_batch(1, wregB, fregB);
    for (int b = 0; b < nb; b += 2) {
        step(b, wregA, fregA);
        if (b + 1 < nb) step(b + 1, wregB, fregB);
    }
    wgmma_wait_acc(acc[0]);
    wgmma_wait_acc(acc[1]);

    // ---- epilogue: out = acc + T * bg.  Non-finite features: 0 * inf = NaN inside the dense product, where the
    // reference only touches the pixels that blend the Gaussian (see blend_v3.cu).  A value that came out non-finite
    // is recomputed with the guarded scalar loop straight from global memory (rare path).
#pragma unroll
    for (int m = 0; m < 2; m++) {
#pragma unroll
        for (int i = 0; i < 2; i++) {
            const int p_tile = wg * 128 + m * 64 + (warp & 3) * 16 + (lane >> 2) + 8 * i;
            const uint32_t px = pix_min.x + (p_tile & 15), py = pix_min.y + (p_tile >> 4);
            if (px >= (uint32_t)W || py >= (uint32_t)H) continue;
            const size_t pix = (size_t)W * py + px;
            const float Tfin = final_T[pix];
#pragma unroll
            for (int n8 = 0; n8 < 16; n8++) {
#pragma unroll
                for (int j = 0; j < 2; j++) {
                    const int c = n8 * 8 + (lane & 3) * 2 + j;
                    if (c >= nch) continue;
                    float v = acc[m][n8 * 4 + i * 2 + j];
                    if (!(fabsf(v) <= 3.0e38f)) {
                        v = 0.f;
                        for (uint32_t e = 0; e < n; e++) {
                            const WChunk* ck = pool.chunks + chunk_of(pool, dbase, (int)(e / kChunkEntries));
                            const int s = (int)(e & (kChunkEntries - 1));
                            const float w = ck->w[s][p_tile];
                            if (w == 0.f) continue;
                            v = fmaf(__ldg(features + (size_t)ck->meta[s].x * C + ch0 + c), w, v);
                        }
                    }
                    out_color[(size_t)(ch0 + c) * plane + pix] = v + Tfin * bgS[c];
                }
            }
        }
    }
}

// ------------------------------------------------------------------------------------ dL/dfeature on the tensor core
// dF[entry][ch] = sum over the tile's 256 pixels of w[entry][px] * dL/dout[px][ch]     (backward.cu:519 summed per tile)
// as  D[M = 128 entries][N = 128 channels] += A[M][K = 8 pixels] . B[N][K]^T,  32 K blocks per tile; warpgroup g owns
// entries 64 g .. 64 g + 63.  Both operands are K-major as they lie in memory (a weight row is contiguous in pixels, a
// dL/dout channel plane row too), so staging is a straight 16-byte copy plus the hi / lo split.  CTA = (tile,
// 128-channel slice); one pipeline stage = one tile row (16 pixels = 2 K blocks): 128 x 64 B of weights and 128 x 64 B
// of dL/dout; 3 stages, operands loaded two stages ahead into registers.  Epilogue: each thread adds its entries'
// channel pairs to dL_dcolors with 8-byte vector reductions.  Lists longer than 128 entries take further passes.
constexpr int kDfStages = 3;
constexpr uint32_t kDfBlk = 16 * 256;                 // one K block of a 128-row operand
constexpr uint32_t kDfStageBytes = 4 * 2 * kDfBlk;    // {A hi, A lo, B hi, B lo} x 2 K blocks = 32 KB

__device__ __forceinline__ void red_add_v2(float* addr, float a, float b) {
    asm volatile("red.global.add.v2.f32 [%0], {%1, %2};" ::"l"(addr), "f"(a), "f"(b) : "memory");
}

__global__ void __launch_bounds__(kMmaThreads, 2) dfeature_mma_kernel(int W, int H, int C,
                                                                      const float* __restrict__ dL_dpixels,
                                                                      PoolView pool, float* __restrict__ dL_dcolors) {
    extern __shared__ __align__(1024) unsigned char smem_raw[];
    __shared__ const float* Wrow[128];
    __shared__ uint32_t Gid[128];

    const int tiles_x = (W + SGB_TILE - 1) / SGB_TILE;
    const int nslices = (C + kNch - 1) / kNch;
    const int tile = blockIdx.x / nslices;
    const int ch0 = (blockIdx.x % nslices) * kNch;
    const int nch = min(kNch, C - ch0);
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, wg = warp >> 2;
    const uint32_t n = pool.count[tile];
    if (n == 0) return;
    const uint32_t dbase = __ldg(pool.dirbase + tile);
    const uint2 pix_min = {(uint32_t)(tile % tiles_x) * SGB_TILE, (uint32_t)(tile / tiles_x) * SGB_TILE};
    const size_t plane = (size_t)H * W;
    const bool rows16 = (W & 3) == 0 && (reinterpret_cast<uintptr_t>(dL_dpixels) & 15) == 0;

    // staging role: quarter-warp = 8 consecutive rows of one 16-byte piece (conflict-free 128-byte stores), the four
    // quarter-warps = the four pieces of a 64-byte row segment (8 rows x 64 contiguous global bytes per instruction)
    const int r8 = lane & 7, quad = lane >> 3;
    const uint32_t soff = (uint32_t)(quad >> 1) * kDfBlk + (uint32_t)(quad & 1) * 128u + (uint32_t)r8 * 16u;
    int gstage = 0;  // stages issued so far over all passes (stage buffer = gstage % kDfStages)
    float acc[64];

    for (uint32_t base = 0; base < n; base += 128) {
        const int cnt = (int)min(128u, n - base);
        __syncthreads();  // previous pass finished with Wrow / Gid
        if (tid < 128) {
            if (tid < cnt) {
                const WChunk* ck = pool.chunks + chunk_of(pool, dbase, (int)((base + tid) / kChunkEntries));
                const int sidx = (base + tid) & (kChunkEntries - 1);
                Wrow[tid] = &ck->w[sidx][0];
                Gid[tid] = ck->meta[sidx].x;
            } else {
                Wrow[tid] = nullptr;
            }
        }
        __syncthreads();
#pragma unroll
        for (int i = 0; i < 64; i++) acc[i] = 0.f;
        float4 aA[2], bA[2], aB[2], bB[2];
        auto load_stage = [&](int ty, float4 (&a)[2], float4 (&b)[2]) {  // tile row ty: pixels 16 ty .. 16 ty + 15
#pragma unroll
            for (int i = 0; i < 2; i++) {
                const int row = (i * 8 + warp) * 8 + r8;   // entry (A) / channel (B) row of this thread
                const float* wr = Wrow[row];
                a[i] = wr ? __ldg(reinterpret_cast<const float4*>(wr + ty * 16 + quad * 4)) : make_float4(0.f, 0.f, 0.f, 0.f);
                const uint32_t y = pix_min.y + ty, x = pix_min.x + quad * 4;
                b[i] = make_float4(0.f, 0.f, 0.f, 0.f);
                if (row < nch && y < (uint32_t)H) {
                    const float* src = dL_dpixels + (size_t)(ch0 + row) * plane + (size_t)W * y + x;
                    if (rows16 && x + 4 <= (uint32_t)W) b[i] = __ldg(reinterpret_cast<const float4*>(src));
                    else {
                        if (x < (uint32_t)W) b[i].x = __ldg(src);
                        if (x + 1 < (uint32_t)W) b[i].y = __ldg(src + 1);
                        if (x + 2 < (uint32_t)W) b[i].z = __ldg(src + 2);
                        if (x + 3 < (uint32_t)W) b[i].w = __ldg(src + 3);
                    }
                }
            }
        };
        auto step = [&](int ty, float4 (&a)[2], float4 (&b)[2]) {
            const int st = gstage % kDfStages;
            if (gstage >= kDfStages) {  // the group that last read this buffer retired in both warpgroups
                wgmma_wait<kDfStages - 1>();
                __syncthreads();
            }
            unsigned char* sb = smem_raw + (size_t)st * kDfStageBytes;
#pragma unroll
            for (int i = 0; i < 2; i++) {
                const uint32_t off = soff + (uint32_t)(i * 8 + warp) * 256u;
                const float4 ah = tf32_hi(a[i]), bh = tf32_hi(b[i]);
                *reinterpret_cast<float4*>(sb + off) = ah;
                *reinterpret_cast<float4*>(sb + 2 * kDfBlk + off) = tf32_hi(sub4(a[i], ah));
                *reinterpret_cast<float4*>(sb + 4 * kDfBlk + off) = bh;
                *reinterpret_cast<float4*>(sb + 6 * kDfBlk + off) = tf32_hi(sub4(b[i], bh));
            }
            if (ty + 2 < SGB_TILE) load_stage(ty + 2, a, b);
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
            __syncthreads();
            const uint32_t s0 = smem_u32(smem_raw) + (uint32_t)st * kDfStageBytes;
            wgmma_fence();
#pragma unroll
            for (int kb = 0; kb < 2; kb++) {
                const uint32_t ah = s0 + kb * kDfBlk + (uint32_t)wg * 8u * 256u;   // rows 64 wg .. 64 wg + 63
                mma3(acc, ah, ah + 2 * kDfBlk, 128, 256, s0 + (4 + kb) * kDfBlk, s0 + (6 + kb) * kDfBlk, 128, 256);
            }
            wgmma_commit();
            gstage++;
        };
        load_stage(0, aA, bA);
        load_stage(1, aB, bB);
#pragma unroll 1
        for (int ty = 0; ty < SGB_TILE; ty += 2) {
            step(ty, aA, bA);
            step(ty + 1, aB, bB);
        }
        wgmma_wait_acc(acc);

        // ---- epilogue: entry 64 wg + 16 (warp % 4) + lane / 4 + 8 i, channel pairs 8 n8 + 2 (lane % 4)
#pragma unroll
        for (int i = 0; i < 2; i++) {
            const int e = wg * 64 + (warp & 3) * 16 + (lane >> 2) + 8 * i;
            if (e >= cnt) continue;
            float* dst = dL_dcolors + (size_t)Gid[e] * C + ch0;
#pragma unroll
            for (int n8 = 0; n8 < 16; n8++) {
                const int c = n8 * 8 + (lane & 3) * 2;
                if (c < nch)   // C % 4 == 0 on this path: a channel pair is in range as a whole
                    red_add_v2(dst + c, acc[n8 * 4 + i * 2], acc[n8 * 4 + i * 2 + 1]);
            }
        }
    }
}

// ------------------------------------------------------------------------------------ chain backward on the tensor core
// s-pass  S[px][entry] = sum_ch dL/dout[px][ch] * F[entry][ch]  as  D[M = 128 px][N = 128 entries] per pixel half
// (warpgroup g owns half g), K = channels (8 per K block), then the reference's back-to-front chain
// (backward.cu:477-550 in dot-product form, the code of chain_backward_warp_kernel) with thread = pixel.  CTA = tile;
// the list is walked in passes of 128 entries from the back.  A = dL/dout is MN-major in memory (pixels contiguous):
// the staging threads transpose it into the K-major operand with scalar stores; B = features is K-major as it lies
// (channels of a row contiguous).  Stage = 16 channels; 2 stages of 48 KB.  When the s-pass of a pass has retired,
// the accumulators are parked in shared memory as S[entry][pixel] (over the idle stage memory) for the chain phase.
constexpr uint32_t kChBBlk = 16 * 256;   // features: dense geometry (LBO 128, SBO 256)
constexpr uint32_t kChStageA = 2 * 2 * kABlk, kChStageB = 2 * kChBBlk;
constexpr uint32_t kChStageBytes = 2 * kChStageA + 2 * kChStageB;   // 48 KB
constexpr int kSRow = 260;                                          // S row stride (floats): conflict-free parking
constexpr uint32_t kSBytes = 128u * kSRow * 4u;
constexpr uint32_t kRbBytes = 8u * 576u * 4u;                       // per-warp reduction rows
constexpr uint32_t kChSmem = (2 * kChStageBytes > kSBytes + kRbBytes) ? 2 * kChStageBytes : kSBytes + kRbBytes;

__global__ void __launch_bounds__(kMmaThreads, 1) chain_backward_mma_kernel(
    int W, int H, int C, const float* __restrict__ bg_color, const SplatRec* __restrict__ rec,
    const float* __restrict__ features, const float* __restrict__ final_Ts, const float* __restrict__ dL_dpixels,
    PoolView pool, float* __restrict__ dL_dmean2D, float* __restrict__ dL_dconic2D, float* __restrict__ dL_dopacity) {
    extern __shared__ __align__(128) unsigned char smem_raw[];
    __shared__ const float* Wrow[128];
    __shared__ uint32_t Gid[128], Mask[128];
    __shared__ float4 RecA[128], RecB[128];
    __shared__ int BufCol[8][4];

    const int tiles_x = (W + SGB_TILE - 1) / SGB_TILE;
    const int tile = blockIdx.x;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, wg = warp >> 2;
    const uint32_t n = pool.count[tile];
    if (n == 0) return;
    const uint32_t dbase = pool.dirbase[tile];
    const uint2 pix_min = {(uint32_t)(tile % tiles_x) * SGB_TILE, (uint32_t)(tile / tiles_x) * SGB_TILE};
    const size_t plane = (size_t)H * W;
    const bool rows16 = ((W & 3) == 0) && ((reinterpret_cast<uintptr_t>(dL_dpixels) & 15) == 0);

    // own pixel (chain phase): tile pixel = tid; warp = strip of 32 pixels, as in the pool masks
    const int p_tile = tid;
    const uint2 pix = {pix_min.x + (uint32_t)(p_tile & 15), pix_min.y + (uint32_t)(p_tile >> 4)};
    const uint32_t pix_id = W * pix.y + pix.x;
    const float2 pixf = {(float)pix.x, (float)pix.y};
    const bool inside = pix.x < (uint32_t)W && pix.y < (uint32_t)H;

    int bg_nonzero = 0;
    for (int ch = tid; ch < C; ch += kMmaThreads) bg_nonzero |= (bg_color[ch] != 0.f);
    bg_nonzero = __syncthreads_or(bg_nonzero);

    float bgdot = 0.f;  // backward.cu:527-529; vanishes for an all-zero background
    if (inside && bg_nonzero)
        for (int ch = 0; ch < C; ch++) bgdot += bg_color[ch] * __ldg(dL_dpixels + (size_t)ch * plane + pix_id);
    const float T_final = inside ? final_Ts[pix_id] : 0.f;
    float T = T_final;
    float last_alpha = 0.f, s_last = 0.f, A = 0.f;
    const float ddelx_dx = 0.5f * W, ddely_dy = 0.5f * H;

    const int nst = (C + 15) / 16;          // stages (16 channels) per pass
    const int k8 = lane & 7, qq = lane >> 3;  // dL staging: channel k8 of the K block, 16-byte piece qq of a tile row
    int gstage = 0;
    // chain-phase views of the (idle) stage memory: S[128 entries][kSRow] and 18 reduction rows per warp
    float* Sf = reinterpret_cast<float*>(smem_raw);
    float* RB = reinterpret_cast<float*>(smem_raw + kSBytes) + warp * 576;
    float acc[2][64];

    const int npass = (int)((n + 127) / 128);
    for (int ps = npass - 1; ps >= 0; ps--) {
        const uint32_t base = (uint32_t)ps * 128u;
        const int cnt = (int)min(128u, n - base);
        __syncthreads();  // previous pass: chain phase done with S / RB / entry records
        if (tid < 128) {
            if (tid < cnt) {
                const WChunk* ck = pool.chunks + chunk_of(pool, dbase, (int)((base + tid) / kChunkEntries));
                const int sidx = (base + tid) & (kChunkEntries - 1);
                const uint2 mt = ck->meta[sidx];
                Wrow[tid] = &ck->w[sidx][0];
                Gid[tid] = mt.x;
                Mask[tid] = mt.y;
                const float4* rp = reinterpret_cast<const float4*>(rec + mt.x);
                RecA[tid] = __ldg(rp);
                RecB[tid] = __ldg(rp + 1);
            } else {
                Mask[tid] = 0u;
            }
        }
        __syncthreads();
#pragma unroll
        for (int m = 0; m < 2; m++)
#pragma unroll
            for (int i = 0; i < 64; i++) acc[m][i] = 0.f;
        // ---- s-pass on the tensor core
        float4 dA[4], fA[2], dB[4], fB[2];
        auto load_stage = [&](int sl, float4 (&d)[4], float4 (&f)[2]) {
#pragma unroll
            for (int it = 0; it < 4; it++) {   // dL/dout: channel (kb, k8), tile row ty, columns qq*4..
                const int c = it * 8 + warp, kb = c >> 4, ty = c & 15;
                const int ch = sl * 16 + kb * 8 + k8;
                const uint32_t y = pix_min.y + ty, x = pix_min.x + qq * 4;
                d[it] = make_float4(0.f, 0.f, 0.f, 0.f);
                if (ch < C && y < (uint32_t)H) {
                    const float* src = dL_dpixels + (size_t)ch * plane + (size_t)W * y + x;
                    if (rows16 && x + 4 <= (uint32_t)W) d[it] = __ldg(reinterpret_cast<const float4*>(src));
                    else {
                        if (x < (uint32_t)W) d[it].x = __ldg(src);
                        if (x + 1 < (uint32_t)W) d[it].y = __ldg(src + 1);
                        if (x + 2 < (uint32_t)W) d[it].z = __ldg(src + 2);
                        if (x + 3 < (uint32_t)W) d[it].w = __ldg(src + 3);
                    }
                }
            }
#pragma unroll
            for (int i = 0; i < 2; i++) {      // features: entry row (i*8+warp)*8 + k8, channels sl*16 + qq*4 ..
                const int row = (i * 8 + warp) * 8 + k8;
                const int chb = sl * 16 + qq * 4;
                f[i] = make_float4(0.f, 0.f, 0.f, 0.f);
                if (row < cnt && chb < C) f[i] = __ldg(reinterpret_cast<const float4*>(features + (size_t)Gid[row] * C + chb));
            }
        };
        auto step = [&](int sl, float4 (&d)[4], float4 (&f)[2]) {
            const int st = gstage & 1;
            if (sl >= 2) {  // the group that last read this buffer retired in both warpgroups
                wgmma_wait<1>();
                __syncthreads();
            }
            unsigned char* sb = smem_raw + (size_t)st * kChStageBytes;
            unsigned char* a_hi = sb;
            unsigned char* a_lo = sb + kChStageA;
            unsigned char* b_hi = sb + 2 * kChStageA;
            unsigned char* b_lo = sb + 2 * kChStageA + kChStageB;
#pragma unroll
            for (int it = 0; it < 4; it++) {
                const int c = it * 8 + warp, kb = c >> 4, ty = c & 15;
                const int p0 = ty * 16 + qq * 4, mh = p0 >> 7, r0 = p0 & 127;
                const uint32_t blk = (uint32_t)(kb * 2 + mh) * kABlk;
                const uint32_t col = (uint32_t)(k8 >> 2) * kLboPad + (uint32_t)(k8 & 3) * 4u;
                const float4 hi = tf32_hi(d[it]);
                const float4 lo = tf32_hi(sub4(d[it], hi));
                const float xh[4] = {hi.x, hi.y, hi.z, hi.w}, xl[4] = {lo.x, lo.y, lo.z, lo.w};
#pragma unroll
                for (int j = 0; j < 4; j++) {
                    const int r = r0 + j;
                    const uint32_t off = blk + (uint32_t)(r >> 3) * kSboPad + (uint32_t)(r & 7) * 16u + col;
                    *reinterpret_cast<float*>(a_hi + off) = xh[j];
                    *reinterpret_cast<float*>(a_lo + off) = xl[j];
                }
            }
#pragma unroll
            for (int i = 0; i < 2; i++) {
                const uint32_t off = (uint32_t)(qq >> 1) * kChBBlk + (uint32_t)(i * 8 + warp) * 256u + (uint32_t)(qq & 1) * 128u +
                                     (uint32_t)k8 * 16u;
                const float4 hi = tf32_hi(f[i]);
                *reinterpret_cast<float4*>(b_hi + off) = hi;
                *reinterpret_cast<float4*>(b_lo + off) = tf32_hi(sub4(f[i], hi));
            }
            if (sl + 2 < nst) load_stage(sl + 2, d, f);
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
            __syncthreads();
            const uint32_t s0 = smem_u32(smem_raw) + (uint32_t)st * kChStageBytes;
            const int nkb = (C - sl * 16 > 8) ? 2 : 1;
            wgmma_fence();
            for (int kb = 0; kb < nkb; kb++) {
                const uint32_t bh = s0 + 2 * kChStageA + kb * kChBBlk, bl = bh + kChStageB;
#pragma unroll
                for (int m = 0; m < 2; m++) {
                    const uint32_t ah = s0 + (uint32_t)(kb * 2 + wg) * kABlk + (uint32_t)m * 8u * kSboPad;
                    mma3(acc[m], ah, ah + kChStageA, kLboPad, kSboPad, bh, bl, 128, 256);
                }
            }
            wgmma_commit();
            gstage++;
        };
        load_stage(0, dA, fA);
        if (nst > 1) load_stage(1, dB, fB);
#pragma unroll 1
        for (int sl = 0; sl < nst; sl += 2) {
            step(sl, dA, fA);
            if (sl + 1 < nst) step(sl + 1, dB, fB);
        }
        wgmma_wait_acc(acc[0]);
        wgmma_wait_acc(acc[1]);
        __syncthreads();  // every warpgroup's MMAs have read the stage memory: it becomes S
#pragma unroll
        for (int m = 0; m < 2; m++)
#pragma unroll
            for (int i = 0; i < 2; i++) {
                const int p = wg * 128 + m * 64 + (warp & 3) * 16 + (lane >> 2) + 8 * i;
#pragma unroll
                for (int n8 = 0; n8 < 16; n8++)
#pragma unroll
                    for (int j = 0; j < 2; j++) Sf[(n8 * 8 + (lane & 3) * 2 + j) * kSRow + p] = acc[m][n8 * 4 + i * 2 + j];
            }
        __syncthreads();

        // ---- chain phase: 32-entry column chunks from the back, the chain of chain_backward_warp_kernel
        for (int cc = (cnt - 1) >> 5; cc >= 0; cc--) {
            const int jhi = min(31, cnt - 1 - cc * 32);
            constexpr int RG = 3;
            int nbuf = 0;
            for (int j = jhi; j >= 0; j--) {
                const int col = cc * 32 + j;
                const bool mine = (Mask[col] >> warp) & 1u;   // uniform per warp (warp = strip)
                float gv[6];
#pragma unroll
                for (int v = 0; v < 6; v++) gv[v] = 0.f;
                if (mine) {
                    const float w = __ldg(Wrow[col] + p_tile);
                    if (w != 0.f) {
                        const float sdot = Sf[col * kSRow + p_tile];
                        const float4 a = RecA[col], con_o = RecB[col];
                        const float2 d = {a.x - pixf.x, a.y - pixf.y};
                        const float power = -0.5f * (con_o.x * d.x * d.x + con_o.z * d.y * d.y) - con_o.y * d.x * d.y;
                        const float G = exp(power);
                        const float alpha = min(0.99f, con_o.w * G);
                        T = T / (1.f - alpha);
                        A = last_alpha * s_last + (1.f - last_alpha) * A;
                        s_last = sdot;
                        float dL_dalpha = (sdot - A) * T;
                        last_alpha = alpha;
                        dL_dalpha += (-T_final / (1.f - alpha)) * bgdot;
                        const float dL_dG = con_o.w * dL_dalpha;
                        const float gdx = G * d.x, gdy = G * d.y;
                        const float dG_ddelx = -gdx * con_o.x - gdy * con_o.y;
                        const float dG_ddely = -gdy * con_o.z - gdx * con_o.y;
                        gv[0] = dL_dG * dG_ddelx * ddelx_dx;
                        gv[1] = dL_dG * dG_ddely * ddely_dy;
                        gv[2] = -0.5f * gdx * d.x * dL_dG;
                        gv[3] = -0.5f * gdx * d.y * dL_dG;
                        gv[4] = -0.5f * gdy * d.y * dL_dG;
                        gv[5] = G * dL_dalpha;
                    }
#pragma unroll
                    for (int v = 0; v < 6; v++) {
                        const int rr = nbuf * 6 + v;
                        RB[rr * 32 + ((((lane >> 2) ^ (rr & 7)) << 2) | (lane & 3))] = gv[v];
                    }
                    if (lane == 0) BufCol[warp][nbuf] = col;   // which list entry each buffered slot belongs to
                    nbuf++;
                }
                // flush when the buffer is full or the chunk ends
                if (nbuf == RG || (j == 0 && nbuf > 0)) {
                    __syncwarp();
                    if (lane < nbuf * 6) {
                        const float4* row = reinterpret_cast<const float4*>(RB + lane * 32);
                        float4 t = row[lane & 7];
#pragma unroll
                        for (int q = 1; q < 8; q++) {
                            const float4 u = row[q ^ (lane & 7)];
                            t.x += u.x; t.y += u.y; t.z += u.z; t.w += u.w;
                        }
                        const float tot = (t.x + t.y) + (t.z + t.w);
                        const int slot = lane / 6, comp = lane - slot * 6;
                        const size_t id = Gid[BufCol[warp][slot]];
                        float* dst = comp < 2 ? dL_dmean2D + id * 3 + comp
                                   : comp < 5 ? dL_dconic2D + id * 4 + (comp == 4 ? 3 : comp - 2)
                                              : dL_dopacity + id;
                        red_add_f32(dst, tot);
                    }
                    __syncwarp();
                    nbuf = 0;
                }
            }
        }
    }
}

}  // namespace

bool blend_mma_enabled() {
    static const bool on = [] { const char* e = getenv("SGB_BLEND_MMA"); return e && e[0] == '1'; }();
    return on;
}

int launch_forward_mma(sgb_ctx* ctx, const sgb_view_inputs& in, ImgView im, const float* colors, float* out_color,
                       const PoolView& pv, cudaStream_t s) {
    const int tiles = ((in.W + SGB_TILE - 1) / SGB_TILE) * ((in.H + SGB_TILE - 1) / SGB_TILE);
    const int slices = (in.C + kNch - 1) / kNch;
    const size_t smem = (size_t)kStages * kStageBytes + 128;
    static DeviceOnce attr;
    if (attr.first_use_on_device())
        SGB_CUDA(cudaFuncSetAttribute(blend_forward_mma_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    StageTimer t(ctx, ST_BLEND_FWD, s);
    ctx->launches += 1;
    blend_forward_mma_kernel<<<tiles * slices, kMmaThreads, smem, s>>>(in.W, in.H, in.C, colors, in.background, im.final_T,
                                                                       pv, out_color);
    SGB_LAUNCH_CHECK("blend_forward_mma_kernel", in.debug, s);
    return SGB_OK;
}

int launch_dfeature_mma(sgb_ctx* ctx, const sgb_view_inputs& in, const float* dL_dpix, float* dL_dcolors,
                        const PoolView& pv, cudaStream_t s) {
    const int tiles = ((in.W + SGB_TILE - 1) / SGB_TILE) * ((in.H + SGB_TILE - 1) / SGB_TILE);
    const int slices = (in.C + kNch - 1) / kNch;
    const size_t smem = (size_t)kDfStages * kDfStageBytes + 1024;
    static DeviceOnce attr;
    if (attr.first_use_on_device())
        SGB_CUDA(cudaFuncSetAttribute(dfeature_mma_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    StageTimer t(ctx, ST_DFEATURE, s);
    ctx->launches += 1;
    dfeature_mma_kernel<<<tiles * slices, kMmaThreads, smem, s>>>(in.W, in.H, in.C, dL_dpix, pv, dL_dcolors);
    SGB_LAUNCH_CHECK("dfeature_mma_kernel", in.debug, s);
    return SGB_OK;
}

int launch_chain_mma(sgb_ctx* ctx, const sgb_view_inputs& in, GeomView g, ImgView im, const float* colors,
                     const float* dL_dpix, float* dL_dmean2D, float* dL_dconic, float* dL_dopacity, const PoolView& pv,
                     cudaStream_t s) {
    const int tiles = ((in.W + SGB_TILE - 1) / SGB_TILE) * ((in.H + SGB_TILE - 1) / SGB_TILE);
    const size_t smem = (size_t)kChSmem + 128;
    static DeviceOnce attr;
    if (attr.first_use_on_device())
        SGB_CUDA(cudaFuncSetAttribute(chain_backward_mma_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    StageTimer t(ctx, ST_BLEND_BWD, s);
    ctx->launches += 1;
    chain_backward_mma_kernel<<<tiles, kMmaThreads, smem, s>>>(in.W, in.H, in.C, in.background, g.rec, colors, im.final_T,
                                                               dL_dpix, pv, dL_dmean2D, dL_dconic, dL_dopacity);
    SGB_LAUNCH_CHECK("chain_backward_mma_kernel", in.debug, s);
    return SGB_OK;
}

}  // namespace sgb
