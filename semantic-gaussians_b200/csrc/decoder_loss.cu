// Distillation loss of a compact rendered feature image through a per-pixel linear decoder, and its gradients.
// The field renders c channels, R (c, N) planar; a 1x1 decoder lifts each pixel to the C channels of the 2D model's
// feature map Y (C, N) planar, fp16 or fp32:
//
//   x_p = W r_p + b          W (C, c) row-major (nn.Linear(c, C).weight), b (C) or absent
//
// and the loss on x against Y is that of feature_loss.cuh (cosine with its valid-pixel mask, l1, l2).  With
// g_p = dLoss / dx_p the call returns dL/dR[:, p] = W^T g_p, dL/dW = sum_p g_p r_p^T and dL/db = sum_p g_p, without
// writing x or g anywhere but shared memory.
//
// Work split: persistent CTAs (at most one per SM), each with a static, contiguous range of 128-pixel blocks.  Per
// block the CTA stages R_blk (c x 128) in shared memory once and walks C in chunks of 64 decoded channels; per chunk
// it stages the chunk's rows of W (row-major and transposed, packed beforehand into the workspace with zero padding
// to CP = 16 / 32 / 64 / 128 columns and a multiple of 64 rows) and runs, as FP32 FFMA register tiles over shared
// operands:
//   decode     X = W_ch R_blk + b_ch     (64 x 128, 4 rows x 8 pixels per thread, K = CP)
//   gradient   G = dLoss/dX from X and the target tile (read from global memory into registers), written to smem
//   dL/dR     += W_ch^T G               (CP x 128, CP/16 channels x 8 pixels per thread, kept in registers)
//   dL/dW_ch   = G R_blk^T              (64 x CP, 4 rows x CP/16 channels per thread, K = 128 pixels)
// cosine needs x.y, |x|^2 and |y|^2 over all C before any g_p exists, so it decodes twice: a first pass over the
// chunks accumulates the three sums (and reads the target), a second recomputes X and forms G.  The target is read
// once when the block's C x 128 target tile fits the shared memory left over (then the second pass reads it from
// there), twice otherwise; l1 / l2 are one pass.  The normaliser 1/Nv of cosine is global: feature_loss.cu's count
// kernel writes Nv into loss[1] first and the main kernel reads it in stream order.
//
// Determinism: every CTA keeps its dL/dW and dL/db partials (workspace slab of 64-padded C x CP floats, shared
// array of C floats) and its loss terms, each summed in a fixed order by a fixed thread; a second kernel adds the
// CTA partials in CTA order.  No float atomics: every output is bitwise identical from call to call.
//
// Precision: FFMA in fp32 throughout.  Plain TF32 operands (10-bit mantissa) miss the 1e-5 tolerances against a
// float64 reference; a 3xTF32 tensor-core split would meet them.  The kernel does 6 N C c flops (8 N C c for cosine)
// on N (C b_target + 8 c) bytes: at C = 512, c = 64 with an fp16 target that is 128 (cosine 170) flops per byte,
// far above the H100's ~20, so it is bound by FFMA issue and shared-memory operand traffic, not by HBM.
//
// H100 80GB HBM3 at 700 W, fp16 target (tools/time_decoder_loss.py): C = 512, c = 64, 968 x 1296: cosine main kernel
// 14.4 ms (22.8 TFLOP/s), l1 / l2 10.9-11.2 ms; C = 768, c = 128, 1080 x 1920: cosine 59.5 ms (27.4 TFLOP/s), l1 / l2
// 42.6-42.9 ms (28.5-28.7 TFLOP/s), against 67 TFLOP/s data-sheet FP32.
#include <algorithm>
#include <cuda_fp16.h>

#include "common.cuh"
#include "feature_loss.cuh"

namespace sgb {
namespace {

constexpr int kDlThreads = 256;
constexpr int kDlPB = 128;            // pixels per block
constexpr int kDlCC = 64;             // decoded channels per chunk
constexpr int kDlPitch = kDlPB + 4;   // shared row pitch of the R and G tiles: float4 rows 1..15 apart hit other banks
constexpr int kDlMaxc = 128;          // widest compact field accepted
constexpr int kDlMaxCtas = kNumSMs;
constexpr int kDlMaxSmem = 226 * 1024;  // dynamic: the 227 KB per-CTA opt-in limit less the static wsum[]

inline int padded_c(int c) { return c <= 16 ? 16 : c <= 32 ? 32 : c <= 64 ? 64 : 128; }
__host__ __device__ inline int padded_C(int C) { return (C + kDlCC - 1) / kDlCC * kDlCC; }

// Workspace: packed W (row-major and chunk-transposed), packed b, then per-CTA dL/dW and dL/db partials and loss
// terms.  Byte offsets, each 256-aligned.
struct DlWorkspace {
    size_t wp, wt, bp, dw, db, loss, total;
};
DlWorkspace workspace_layout(int C, int c) {
    const size_t Cp = padded_C(C), cp = padded_c(c);
    auto up = [](size_t b) { return (b + 255) & ~(size_t)255; };
    DlWorkspace w;
    w.wp = 0;
    w.wt = w.wp + up(Cp * cp * sizeof(float));
    w.bp = w.wt + up(Cp * cp * sizeof(float));
    w.dw = w.bp + up(Cp * sizeof(float));
    w.db = w.dw + up((size_t)kDlMaxCtas * Cp * cp * sizeof(float));
    w.loss = w.db + up((size_t)kDlMaxCtas * Cp * sizeof(float));
    w.total = w.loss + up((size_t)kDlMaxCtas * sizeof(double));
    return w;
}

// W (C, c) and b into the layouts the main kernel stages, zero outside (C, c): Wp [Cp][cp] row-major, Wt
// [Cp / 64][cp][64] (each chunk's 64 rows as contiguous columns), bp [Cp].
__global__ void __launch_bounds__(256) decoder_pack_kernel(int C, int c, int cp, const float* __restrict__ W,
                                                           const float* __restrict__ b, float* __restrict__ Wp,
                                                           float* __restrict__ Wt, float* __restrict__ bp) {
    const int total = padded_C(C) * cp;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
        const int r = i / cp, k = i % cp;
        const float v = r < C && k < c ? W[(size_t)r * c + k] : 0.f;
        Wp[i] = v;
        Wt[(size_t)(r / kDlCC) * cp * kDlCC + k * kDlCC + r % kDlCC] = v;
        if (k == 0) bp[r] = b && r < C ? b[r] : 0.f;
    }
}

// Four consecutive pixels of one target plane, `rem` of them inside the image.  VEC: p is 16- (fp32) or 8-byte
// (fp16) aligned and rem is a multiple of 4.
template <typename T>
__device__ __forceinline__ Quad load_target4(const T* p, long long rem, bool vec) {
    Quad q;
    if (vec && rem >= 4) {
        q = load4(p);
    } else {
#pragma unroll
        for (int j = 0; j < 4; j++) q.v[j] = j < rem ? to_f32(p[j]) : 0.f;
    }
    return q;
}

struct DlArgs {
    int C, c;
    long long N;
    int nblk, ycache, vec;
    const float* R;
    const float* Wp;
    const float* Wt;
    const float* bp;
    const void* Y;
    float* dR;
    float* dw_part;
    float* db_part;
    double* loss_part;
    const double* loss;
};

// Thread (tx, ty) = (tid % 16, tid / 16).  Its 8 pixel columns of a block are px(q) = 4 tx + q % 4 + 64 (q / 4), its
// 4 decoded rows of a chunk 4 ty + i, its dL/dR channels CP/16 ty + j, its dL/dW columns tx + 16 j.
template <typename T, int CP, int LOSS>
__global__ void __launch_bounds__(kDlThreads, 1) decoder_loss_kernel(const DlArgs a) {
    constexpr int TC = CP / 16;
    const int C = a.C, c = a.c, Cp = padded_C(C), nch = Cp / kDlCC;
    const long long N = a.N;
    const T* __restrict__ Y = static_cast<const T*>(a.Y);
    extern __shared__ __align__(16) float dl_smem[];
    float* Rs = dl_smem;                  // [CP][kDlPitch]  the block's compact features (zero past c and N)
    float* Gs = Rs + CP * kDlPitch;       // [kDlCC][kDlPitch] g of the chunk; cosine: first the per-pixel sums
    float* Ws = Gs + kDlCC * kDlPitch;    // [kDlCC][CP]     the chunk's rows of W
    float* Wts = Ws + kDlCC * CP;         // [CP][kDlCC]     the same, transposed
    float* bs = Wts + CP * kDlCC;         // [kDlCC]
    float* cu = bs + kDlCC;               // [kDlPB] cosine: g_p = cu[p] y_p + cv[p] x_p
    float* cv = cu + kDlPB;               // [kDlPB]
    float* dbs = cv + kDlPB;              // [Cp] this CTA's dL/db
    T* Yc = reinterpret_cast<T*>(dbs + Cp);  // [Cp][kDlPB] cosine with ycache: the block's target

    const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
    const int b_begin = (int)((long long)blockIdx.x * a.nblk / gridDim.x);
    const int b_end = (int)((long long)(blockIdx.x + 1) * a.nblk / gridDim.x);
    float* dwp = a.dw_part + (size_t)blockIdx.x * Cp * CP;
    for (int i = tid; i < Cp; i += kDlThreads) dbs[i] = 0.f;
    float inv_nv = 0.f;
    if (LOSS == SGB_FEATLOSS_COSINE) {
        const double nv = a.loss[1];
        inv_nv = nv > 0.0 ? (float)(1.0 / nv) : 0.f;
    }
    const float gs = (float)((LOSS == SGB_FEATLOSS_L2 ? 2.0 : 1.0) / ((double)N * C));
    double lsum = 0.0;

    auto px = [&](int q) { return 4 * tx + (q & 3) + 64 * (q >> 2); };
    auto stage_chunk = [&](int ch, bool rows) {
        const float4* wt = reinterpret_cast<const float4*>(a.Wt + (size_t)ch * CP * kDlCC);
        for (int e = tid; e < CP * kDlCC / 4; e += kDlThreads) reinterpret_cast<float4*>(Wts)[e] = __ldg(wt + e);
        if (rows) {
            const float4* wp = reinterpret_cast<const float4*>(a.Wp + (size_t)ch * kDlCC * CP);
            for (int e = tid; e < CP * kDlCC / 4; e += kDlThreads) reinterpret_cast<float4*>(Ws)[e] = __ldg(wp + e);
        }
        if (tid < kDlCC) bs[tid] = __ldg(a.bp + ch * kDlCC + tid);
    };
    // X = W_ch R_blk + b_ch on this thread's 4 rows x 8 pixels
    auto decode = [&](float (&x)[4][8]) {
#pragma unroll
        for (int i = 0; i < 4; i++) {
            const float b = bs[4 * ty + i];
#pragma unroll
            for (int q = 0; q < 8; q++) x[i][q] = b;
        }
#pragma unroll 4
        for (int k = 0; k < CP; k++) {
            const float4 w = *reinterpret_cast<const float4*>(Wts + k * kDlCC + 4 * ty);
            const float4 r0 = *reinterpret_cast<const float4*>(Rs + k * kDlPitch + 4 * tx);
            const float4 r1 = *reinterpret_cast<const float4*>(Rs + k * kDlPitch + 64 + 4 * tx);
            const float wv[4] = {w.x, w.y, w.z, w.w};
            const float rv[8] = {r0.x, r0.y, r0.z, r0.w, r1.x, r1.y, r1.z, r1.w};
#pragma unroll
            for (int i = 0; i < 4; i++)
#pragma unroll
                for (int q = 0; q < 8; q++) x[i][q] = fmaf(wv[i], rv[q], x[i][q]);
        }
    };
    // the target tile matching decode(); rows past C are zero
    auto load_target = [&](int ch, long long p0, bool from_cache, float (&y)[4][8]) {
#pragma unroll
        for (int i = 0; i < 4; i++) {
            const int r = ch * kDlCC + 4 * ty + i;
#pragma unroll
            for (int h = 0; h < 2; h++) {
                const int pc = 4 * tx + 64 * h;
                Quad q;
                if (from_cache) {
#pragma unroll
                    for (int j = 0; j < 4; j++) q.v[j] = to_f32(Yc[(size_t)r * kDlPB + pc + j]);
                } else if (r < C) {
                    q = load_target4(Y + (size_t)r * N + p0 + pc, N - p0 - pc, a.vec);
                } else {
                    q = {{0.f, 0.f, 0.f, 0.f}};
                }
#pragma unroll
                for (int j = 0; j < 4; j++) y[i][4 * h + j] = q.v[j];
            }
        }
    };

    for (int blk = b_begin; blk < b_end; blk++) {
        const long long p0 = (long long)blk * kDlPB;
        __syncthreads();  // the previous block's readers of Rs, Gs and cu / cv are done
        for (int e = tid; e < CP * kDlPB; e += kDlThreads) {
            const int k = e / kDlPB, p = e % kDlPB;
            Rs[k * kDlPitch + p] = k < c && p0 + p < N ? __ldg(a.R + (size_t)k * N + p0 + p) : 0.f;
        }
        float u[8], v[8];
        if constexpr (LOSS == SGB_FEATLOSS_COSINE) {
            float dot[8], xx[8], yy[8];
            unsigned nz = 0;
#pragma unroll
            for (int q = 0; q < 8; q++) dot[q] = xx[q] = yy[q] = 0.f;
            for (int ch = 0; ch < nch; ch++) {
                __syncthreads();
                stage_chunk(ch, false);
                __syncthreads();
                float x[4][8], y[4][8];
                decode(x);
                load_target(ch, p0, false, y);
#pragma unroll
                for (int i = 0; i < 4; i++)
#pragma unroll
                    for (int q = 0; q < 8; q++) {
                        if (a.ycache) Yc[(size_t)(ch * kDlCC + 4 * ty + i) * kDlPB + px(q)] = T(y[i][q]);
                        dot[q] = fmaf(x[i][q], y[i][q], dot[q]);
                        xx[q] = fmaf(x[i][q], x[i][q], xx[q]);
                        yy[q] = fmaf(y[i][q], y[i][q], yy[q]);
                        nz |= (unsigned)(y[i][q] != 0.f) << q;
                    }
            }
            // per-pixel sums over the 16 row groups, added in a fixed order
            float* red = Gs;  // [4][16][kDlPB]
#pragma unroll
            for (int q = 0; q < 8; q++) {
                red[(0 * 16 + ty) * kDlPB + px(q)] = dot[q];
                red[(1 * 16 + ty) * kDlPB + px(q)] = xx[q];
                red[(2 * 16 + ty) * kDlPB + px(q)] = yy[q];
                red[(3 * 16 + ty) * kDlPB + px(q)] = (float)((nz >> q) & 1u);
            }
            __syncthreads();
            if (tid < kDlPB) {
                float d = 0.f, a2 = 0.f, b2 = 0.f, any = 0.f;
                for (int k = 0; k < 16; k++) {
                    d += red[(0 * 16 + k) * kDlPB + tid];
                    a2 += red[(1 * 16 + k) * kDlPB + tid];
                    b2 += red[(2 * 16 + k) * kDlPB + tid];
                    any += red[(3 * 16 + k) * kDlPB + tid];
                }
                const bool valid = any > 0.f && p0 + tid < N;
                const double t = cosine_rule(d, a2, b2, valid, inv_nv, cu[tid], cv[tid]);
                if (valid) lsum += t;
            }
            __syncthreads();
#pragma unroll
            for (int q = 0; q < 8; q++) {
                u[q] = cu[px(q)];
                v[q] = cv[px(q)];
            }
        }

        float acc[TC][8];
#pragma unroll
        for (int j = 0; j < TC; j++)
#pragma unroll
            for (int q = 0; q < 8; q++) acc[j][q] = 0.f;
        for (int ch = 0; ch < nch; ch++) {
            __syncthreads();  // the previous chunk's readers of Ws, Wts, bs and Gs are done
            stage_chunk(ch, true);
            __syncthreads();
            {
                float x[4][8], y[4][8];
                decode(x);
                load_target(ch, p0, LOSS == SGB_FEATLOSS_COSINE && a.ycache, y);
                float lpart = 0.f;
#pragma unroll
                for (int i = 0; i < 4; i++) {
                    float g[8], rs = 0.f;
#pragma unroll
                    for (int q = 0; q < 8; q++) {
                        if constexpr (LOSS == SGB_FEATLOSS_COSINE) {
                            g[q] = fmaf(u[q], y[i][q], v[q] * x[i][q]);
                        } else {
                            float ge;
                            const float t = elementwise_rule<LOSS>(x[i][q] - y[i][q], gs, ge);
                            const bool in = p0 + px(q) < N;
                            g[q] = in ? ge : 0.f;
                            lpart += in ? t : 0.f;
                        }
                        rs += g[q];
                    }
                    float* grow = Gs + (4 * ty + i) * kDlPitch + 4 * tx;
                    *reinterpret_cast<float4*>(grow) = make_float4(g[0], g[1], g[2], g[3]);
                    *reinterpret_cast<float4*>(grow + 64) = make_float4(g[4], g[5], g[6], g[7]);
                    // dL/db: this row's 128 pixels, over the 16 tx lanes in a fixed tree
#pragma unroll
                    for (int o = 8; o > 0; o >>= 1) rs += __shfl_xor_sync(0xffffffffu, rs, o);
                    if (tx == 0) dbs[ch * kDlCC + 4 * ty + i] += rs;
                }
                if (LOSS != SGB_FEATLOSS_COSINE) lsum += (double)lpart;
            }
            __syncthreads();
            // dL/dR += W_ch^T G
#pragma unroll 2
            for (int r = 0; r < kDlCC; r++) {
                float w[TC];
                if constexpr (TC >= 4) {
#pragma unroll
                    for (int j = 0; j < TC; j += 4) {
                        const float4 f = *reinterpret_cast<const float4*>(Ws + r * CP + TC * ty + j);
                        w[j] = f.x, w[j + 1] = f.y, w[j + 2] = f.z, w[j + 3] = f.w;
                    }
                } else {
#pragma unroll
                    for (int j = 0; j < TC; j++) w[j] = Ws[r * CP + TC * ty + j];
                }
                const float4 g0 = *reinterpret_cast<const float4*>(Gs + r * kDlPitch + 4 * tx);
                const float4 g1 = *reinterpret_cast<const float4*>(Gs + r * kDlPitch + 64 + 4 * tx);
                const float gv[8] = {g0.x, g0.y, g0.z, g0.w, g1.x, g1.y, g1.z, g1.w};
#pragma unroll
                for (int j = 0; j < TC; j++)
#pragma unroll
                    for (int q = 0; q < 8; q++) acc[j][q] = fmaf(w[j], gv[q], acc[j][q]);
            }
            // dL/dW_ch = G R_blk^T, added to this CTA's slab (the same thread owns an element in every block)
            float dw[4][TC];
#pragma unroll
            for (int i = 0; i < 4; i++)
#pragma unroll
                for (int j = 0; j < TC; j++) dw[i][j] = 0.f;
#pragma unroll 2
            for (int p = 0; p < kDlPB; p += 4) {
                float4 gr[4];
#pragma unroll
                for (int i = 0; i < 4; i++) gr[i] = *reinterpret_cast<const float4*>(Gs + (4 * ty + i) * kDlPitch + p);
#pragma unroll
                for (int j = 0; j < TC; j++) {
                    const float4 rr = *reinterpret_cast<const float4*>(Rs + (tx + 16 * j) * kDlPitch + p);
#pragma unroll
                    for (int i = 0; i < 4; i++) {
                        float s = dw[i][j];
                        s = fmaf(gr[i].x, rr.x, s);
                        s = fmaf(gr[i].y, rr.y, s);
                        s = fmaf(gr[i].z, rr.z, s);
                        dw[i][j] = fmaf(gr[i].w, rr.w, s);
                    }
                }
            }
#pragma unroll
            for (int i = 0; i < 4; i++)
#pragma unroll
                for (int j = 0; j < TC; j++) {
                    float* o = dwp + (size_t)(ch * kDlCC + 4 * ty + i) * CP + tx + 16 * j;
                    *o = blk == b_begin ? dw[i][j] : *o + dw[i][j];
                }
        }
        // dL/dR of the block
#pragma unroll
        for (int j = 0; j < TC; j++) {
            const int k = TC * ty + j;
            if (k >= c) continue;
#pragma unroll
            for (int h = 0; h < 2; h++) {
                const long long p = p0 + 4 * tx + 64 * h;
                float* o = a.dR + (size_t)k * N + p;
                if (a.vec && p + 4 <= N) {
                    *reinterpret_cast<float4*>(o) = make_float4(acc[j][4 * h], acc[j][4 * h + 1], acc[j][4 * h + 2],
                                                                acc[j][4 * h + 3]);
                } else {
#pragma unroll
                    for (int q = 0; q < 4; q++)
                        if (p + q < N) o[q] = acc[j][4 * h + q];
                }
            }
        }
    }

    __syncthreads();
    for (int i = tid; i < Cp; i += kDlThreads) a.db_part[(size_t)blockIdx.x * Cp + i] = dbs[i];
    __shared__ double wsum[kDlThreads / 32];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) lsum += __shfl_xor_sync(0xffffffffu, lsum, o);
    if ((tid & 31) == 0) wsum[tid >> 5] = lsum;
    __syncthreads();
    if (tid == 0) {
        double t = 0.0;
        for (int w = 0; w < kDlThreads / 32; w++) t += wsum[w];
        a.loss_part[blockIdx.x] = t;
    }
}

// dL/dW, dL/db and the loss from the CTA partials, each summed in CTA order.
__global__ void __launch_bounds__(256) decoder_reduce_kernel(int C, int c, int cp, int ncta, long long N, int loss_type,
                                                             const float* __restrict__ dw_part,
                                                             const float* __restrict__ db_part,
                                                             const double* __restrict__ loss_part,
                                                             float* __restrict__ dW, float* __restrict__ db,
                                                             double* __restrict__ loss) {
    const int Cp = padded_C(C);
    const long long nw = (long long)C * c, total = nw + (db ? C : 0);
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        float s = 0.f;
        if (i < nw) {
            const float* p = dw_part + (size_t)(i / c) * cp + i % c;
            for (int t = 0; t < ncta; t++) s += p[(size_t)t * Cp * cp];
            dW[i] = s;
        } else {
            const float* p = db_part + (i - nw);
            for (int t = 0; t < ncta; t++) s += p[(size_t)t * Cp];
            db[i - nw] = s;
        }
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) {
        double t = 0.0;
        for (int k = 0; k < ncta; k++) t += loss_part[k];
        if (loss_type == SGB_FEATLOSS_COSINE) {
            const double nv = loss[1];
            loss[0] = nv > 0.0 ? t / nv : 0.0;
        } else {
            loss[0] = t / ((double)N * C);
            loss[1] = (double)N;  // every pixel takes part in the mean
        }
    }
}

size_t main_smem_bytes(int CP, int Cp) {
    return sizeof(float) * ((size_t)CP * kDlPitch + kDlCC * kDlPitch + 2 * kDlCC * CP + kDlCC + 2 * kDlPB + Cp);
}

template <typename T, int CP, int LOSS>
int launch_main(DlArgs& a, int ncta, cudaStream_t s) {
    const int Cp = padded_C(a.C);
    const size_t base = main_smem_bytes(CP, Cp), yc = (size_t)Cp * kDlPB * sizeof(T);
    a.ycache = LOSS == SGB_FEATLOSS_COSINE && base + yc <= (size_t)kDlMaxSmem;
    const size_t smem = base + (a.ycache ? yc : 0);
    static DeviceOnce attr_set;
    if (attr_set.first_use_on_device())
        SGB_CUDA(cudaFuncSetAttribute(decoder_loss_kernel<T, CP, LOSS>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                      kDlMaxSmem));
    decoder_loss_kernel<T, CP, LOSS><<<ncta, kDlThreads, smem, s>>>(a);
    SGB_LAUNCH_CHECK("decoder_loss_kernel", 0, s);
    return SGB_OK;
}

template <typename T, int CP>
int launch_loss(int loss_type, DlArgs& a, int ncta, cudaStream_t s) {
    if (loss_type == SGB_FEATLOSS_COSINE) return launch_main<T, CP, SGB_FEATLOSS_COSINE>(a, ncta, s);
    if (loss_type == SGB_FEATLOSS_L1) return launch_main<T, CP, SGB_FEATLOSS_L1>(a, ncta, s);
    return launch_main<T, CP, SGB_FEATLOSS_L2>(a, ncta, s);
}

template <typename T>
int launch_width(int loss_type, DlArgs& a, int ncta, cudaStream_t s) {
    switch (padded_c(a.c)) {
        case 16: return launch_loss<T, 16>(loss_type, a, ncta, s);
        case 32: return launch_loss<T, 32>(loss_type, a, ncta, s);
        case 64: return launch_loss<T, 64>(loss_type, a, ncta, s);
        default: return launch_loss<T, 128>(loss_type, a, ncta, s);
    }
}

}  // namespace
}  // namespace sgb

using namespace sgb;

extern "C" {

size_t sgb_decoded_feature_loss_workspace_bytes(int32_t C, int32_t c, int64_t N) {
    if (C < 1 || C > kFeatMaxC || c < 1 || c > kDlMaxc || N < 0) return 0;
    return workspace_layout(C, c).total;
}

int sgb_decoded_feature_loss(int32_t C, int32_t c, int64_t N, const float* render, const float* weight,
                             const float* bias, const void* target, int32_t target_dtype, int32_t loss_type,
                             float* dL_drender, float* dL_dweight, float* dL_dbias, void* workspace, double* loss,
                             void* stream) {
    static const char* fn = "sgb_decoded_feature_loss";
    if (check_feature_loss_args(fn, C, target_dtype, loss_type) != SGB_OK) return SGB_E_INVALID;
    if (c <= 0 || c > kDlMaxc) { set_error("%s: c = %d outside [1, %d]", fn, c, kDlMaxc); return SGB_E_INVALID; }
    if (N < 0) { set_error("%s: N = %lld is negative", fn, (long long)N); return SGB_E_INVALID; }
    if (!loss) { set_error("%s: null loss", fn); return SGB_E_INVALID; }
    if (!dL_dweight) { set_error("%s: null dL_dweight", fn); return SGB_E_INVALID; }
    if (dL_dbias && !bias) { set_error("%s: dL_dbias given without bias", fn); return SGB_E_INVALID; }
    if (bias && !dL_dbias) { set_error("%s: bias given without dL_dbias", fn); return SGB_E_INVALID; }
    if (N > 0 && !render) { set_error("%s: null render", fn); return SGB_E_INVALID; }
    if (N > 0 && !weight) { set_error("%s: null weight", fn); return SGB_E_INVALID; }
    if (N > 0 && !target) { set_error("%s: null target", fn); return SGB_E_INVALID; }
    if (N > 0 && !dL_drender) { set_error("%s: null dL_drender", fn); return SGB_E_INVALID; }
    if (N > 0 && !workspace) { set_error("%s: null workspace", fn); return SGB_E_INVALID; }
    if (N > 0 && (reinterpret_cast<uintptr_t>(workspace) & 15) != 0) {
        set_error("%s: workspace is not 16-byte aligned", fn);
        return SGB_E_INVALID;
    }
    cudaStream_t s = (cudaStream_t)stream;
    SGB_CUDA(cudaMemsetAsync(loss, 0, 2 * sizeof(double), s));
    if (N == 0) {
        SGB_CUDA(cudaMemsetAsync(dL_dweight, 0, (size_t)C * c * sizeof(float), s));
        if (dL_dbias) SGB_CUDA(cudaMemsetAsync(dL_dbias, 0, (size_t)C * sizeof(float), s));
        return SGB_OK;
    }

    const DlWorkspace L = workspace_layout(C, c);
    unsigned char* ws = static_cast<unsigned char*>(workspace);
    const int cp = padded_c(c);
    float* Wp = reinterpret_cast<float*>(ws + L.wp);
    float* Wt = reinterpret_cast<float*>(ws + L.wt);
    float* bp = reinterpret_cast<float*>(ws + L.bp);
    const int pack_blocks = (padded_C(C) * cp + 255) / 256;
    decoder_pack_kernel<<<pack_blocks, 256, 0, s>>>(C, c, cp, weight, bias, Wp, Wt, bp);
    SGB_LAUNCH_CHECK("decoder_pack_kernel", 0, s);
    if (loss_type == SGB_FEATLOSS_COSINE) {
        const int rc = target_dtype == SGB_FEAT_F16
                           ? count_valid_pixels<__half>(C, (long long)N, (const __half*)target, loss + 1, s)
                           : count_valid_pixels<float>(C, (long long)N, (const float*)target, loss + 1, s);
        if (rc != SGB_OK) return rc;
    }

    const size_t tsize = target_dtype == SGB_FEAT_F16 ? 2 : 4;
    DlArgs a;
    a.C = C;
    a.c = c;
    a.N = (long long)N;
    a.nblk = (int)((N + kDlPB - 1) / kDlPB);
    a.ycache = 0;
    a.vec = N % 4 == 0 && (reinterpret_cast<uintptr_t>(target) & (4 * tsize - 1)) == 0 &&
            (reinterpret_cast<uintptr_t>(dL_drender) & 15) == 0;
    a.R = render;
    a.Wp = Wp;
    a.Wt = Wt;
    a.bp = bp;
    a.Y = target;
    a.dR = dL_drender;
    a.dw_part = reinterpret_cast<float*>(ws + L.dw);
    a.db_part = reinterpret_cast<float*>(ws + L.db);
    a.loss_part = reinterpret_cast<double*>(ws + L.loss);
    a.loss = loss;
    const int ncta = std::min(kDlMaxCtas, a.nblk);
    const int rc = target_dtype == SGB_FEAT_F16 ? launch_width<__half>(loss_type, a, ncta, s)
                                                : launch_width<float>(loss_type, a, ncta, s);
    if (rc != SGB_OK) return rc;
    const long long nout = (long long)C * c + (dL_dbias ? C : 0);
    const unsigned rblocks = (unsigned)std::min<long long>((nout + 255) / 256, (long long)kNumSMs * 4);
    decoder_reduce_kernel<<<rblocks, 256, 0, s>>>(C, c, cp, ncta, (long long)N, loss_type, a.dw_part, a.db_part,
                                                  a.loss_part, dL_dweight, dL_dbias, loss);
    SGB_LAUNCH_CHECK("decoder_reduce_kernel", 0, s);
    return SGB_OK;
}

}  // extern "C"
