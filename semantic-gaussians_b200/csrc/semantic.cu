// Open-vocabulary semantic head that every render_chn caller of the reference runs right after the
// rasterizer:
//
//   rendering = rendering / (rendering.norm(dim=0, keepdim=True) + 1e-8)      eval_segmentation.py:155,255,396
//   sim       = torch.einsum("cq,qhw->chw", text_features, rendering)         eval_segmentation.py:156,256,397
//   label     = sim[1:].argmax(dim=0)                                         eval_segmentation.py:157,257,398
//
// and its per-Gaussian twin  sim = einsum("cq,dq->dc", text_features, features)  (eval_segmentation.py:132,232;
// view_viser.py:185,217).  In torch that is four passes over the (C,H,W) image (norm, divide, einsum,
// arg-max: ~4x 2.1 GB at K3 sizes); here the image is read ONCE: every thread owns four pixels, walks
// the channel planes with 16-byte loads and keeps K running dot products plus the squared norm in
// registers; the class embeddings sit transposed in shared memory and are read as broadcasts.
#include "common.cuh"
#include "semantic.cuh"
#include "tma.cuh"

namespace sgb {

namespace {

constexpr int kHeadThreads = 256;
constexpr int kHeadPix = 4;       // pixels per thread
constexpr int kHeadSlab = 128;    // channels of the class embeddings staged per shared-memory slab
constexpr int kMaxKC = 32;        // classes per pass (one register accumulator per class and pixel)

// NK4 = (classes per pass) / 4.  VEC: the N-float planes are 16-byte aligned (N % 4 == 0): pixel
// group = 4 consecutive pixels, one LDG.128 per channel; otherwise the thread's 4 pixels are strided
// by the block width and loaded as scalars (still coalesced across the warp).
template <int NK4, bool VEC>
__global__ void __launch_bounds__(kHeadThreads) semantic_head_kernel(
    int C, int K, long long N, const float* __restrict__ render, const float* __restrict__ text, int first_class,
    float* __restrict__ sim, long long* __restrict__ label, float* __restrict__ best_val, int k0, int multi) {
    constexpr int KC = NK4 * 4;
    __shared__ __align__(16) float Ts[kHeadSlab][KC];  // [channel][class], zero padded
    const int tid = threadIdx.x;
    // k0: first class of this pass; multi: 0 = the only pass, 1 = first of several, 2 = a later pass
    const int kc = min(KC, K - k0);
    const long long blk = (long long)blockIdx.x * (kHeadThreads * kHeadPix);
    long long px[kHeadPix];
#pragma unroll
    for (int i = 0; i < kHeadPix; i++) px[i] = VEC ? blk + (long long)tid * kHeadPix + i : blk + (long long)i * kHeadThreads + tid;
    // VEC: N % 4 == 0, so a group of four pixels is inside the image as soon as its first pixel is
    const bool any = px[0] < N;

    float2 acc[kHeadPix / 2][KC];  // [pixel pair][class]
#pragma unroll
    for (int p = 0; p < kHeadPix / 2; p++)
#pragma unroll
        for (int k = 0; k < KC; k++) acc[p][k] = make_float2(0.f, 0.f);
    float2 nrm[kHeadPix / 2] = {make_float2(0.f, 0.f), make_float2(0.f, 0.f)};

    for (int c0 = 0; c0 < C; c0 += kHeadSlab) {
        const int cs = min(kHeadSlab, C - c0);
        __syncthreads();
        for (int e = tid; e < kHeadSlab * KC; e += kHeadThreads) {
            const int c = e / KC, k = e - c * KC;
            Ts[c][k] = (c < cs && k < kc) ? __ldg(text + (size_t)(k0 + k) * C + c0 + c) : 0.f;
        }
        __syncthreads();
        if (!any) continue;
        const float* src = render + (size_t)c0 * N;
#pragma unroll 4
        for (int c = 0; c < cs; c++) {
            float x[kHeadPix];
            if (VEC) {
                const float4 v = __ldg(reinterpret_cast<const float4*>(src + (size_t)c * N + px[0]));
                x[0] = v.x; x[1] = v.y; x[2] = v.z; x[3] = v.w;
            } else {
#pragma unroll
                for (int i = 0; i < kHeadPix; i++) x[i] = px[i] < N ? __ldg(src + (size_t)c * N + px[i]) : 0.f;
            }
            const float2 x01 = make_float2(x[0], x[1]), x23 = make_float2(x[2], x[3]);
            nrm[0] = ffma2(x01, x01, nrm[0]);
            nrm[1] = ffma2(x23, x23, nrm[1]);
#pragma unroll
            for (int q = 0; q < NK4; q++) {
                const float4 t = *reinterpret_cast<const float4*>(&Ts[c][q * 4]);
                const float tt[4] = {t.x, t.y, t.z, t.w};
#pragma unroll
                for (int j = 0; j < 4; j++) {
                    const float2 t2 = make_float2(tt[j], tt[j]);
                    acc[0][q * 4 + j] = ffma2(x01, t2, acc[0][q * 4 + j]);
                    acc[1][q * 4 + j] = ffma2(x23, t2, acc[1][q * 4 + j]);
                }
            }
        }
    }
    if (!any) return;

    // sim = dot / (||x|| + 1e-8)
    float inv[kHeadPix];
    inv[0] = 1.f / (sqrtf(nrm[0].x) + 1e-8f);
    inv[1] = 1.f / (sqrtf(nrm[0].y) + 1e-8f);
    inv[2] = 1.f / (sqrtf(nrm[1].x) + 1e-8f);
    inv[3] = 1.f / (sqrtf(nrm[1].y) + 1e-8f);
    float bv[kHeadPix];
    int bk[kHeadPix];
#pragma unroll
    for (int i = 0; i < kHeadPix; i++) { bv[i] = 0.f; bk[i] = -1; }
#pragma unroll
    for (int k = 0; k < KC; k++) {
        if (k >= kc) break;
        float s[kHeadPix] = {acc[0][k].x * inv[0], acc[0][k].y * inv[1], acc[1][k].x * inv[2], acc[1][k].y * inv[3]};
        if (sim) {
            float* dst = sim + (size_t)(k0 + k) * N;
            if (VEC) *reinterpret_cast<float4*>(dst + px[0]) = make_float4(s[0], s[1], s[2], s[3]);
            else {
#pragma unroll
                for (int i = 0; i < kHeadPix; i++) if (px[i] < N) dst[px[i]] = s[i];
            }
        }
        if (k0 + k >= first_class) {
#pragma unroll
            for (int i = 0; i < kHeadPix; i++)
                if (bk[i] < 0 || s[i] > bv[i]) { bv[i] = s[i]; bk[i] = k0 + k; }  // first maximum wins, like torch.argmax
        }
    }
    if (label) {
#pragma unroll
        for (int i = 0; i < kHeadPix; i++) {
            if (px[i] >= N || bk[i] < 0) continue;
            if (multi == 0) {
                label[px[i]] = (long long)(bk[i] - first_class);
            } else {
                // more than 32 classes: the passes are separate launches, one after another on the
                // stream, and keep the running maximum in best_val (strictly greater: first maximum wins)
                if (multi == 1 || bv[i] > best_val[px[i]]) {
                    best_val[px[i]] = bv[i];
                    label[px[i]] = (long long)(bk[i] - first_class);
                }
            }
        }
    }
}

// Same head, fed by TMA.  The register-file version above keeps only ~4 x 16 B of loads in flight per
// thread at 8 warps/SM (146 registers); here the channel planes of a
// 1024-pixel block stream through a ring of kHNS stages x kHCS channels x 4 KB filled by 1-D bulk copies
// (cp.async.bulk + mbarrier complete_tx), ~96 KB in flight per SM, and the math never waits on a global
// load.  Full stages run a branch-free fully unrolled 8-channel body (the per-channel tail test and the
// per-stage barrier bookkeeping cost a large share of the instructions with 4-channel stages).  512 threads x 2
// pixels: half the accumulators per thread of the 4-pixel layout, so 16 warps per SM fit the register file.
// Requires the VEC conditions (N % 4 == 0, 16-byte aligned planes) and the transposed class embeddings of
// one pass to fit next to the ring.
constexpr int kHCS = 8;   // channels per stage
constexpr int kHNS = 4;   // stages
constexpr int kTmaThreads = 512;
constexpr int kHeadBlockPix = kTmaThreads * 2;  // 1024
constexpr size_t kHeadRingBytes = (size_t)kHNS * kHCS * kHeadBlockPix * sizeof(float);

template <int NK4>
__global__ void __launch_bounds__(kTmaThreads, 1) semantic_head_tma_kernel(
    int C, int K, long long N, const float* __restrict__ render, const float* __restrict__ text, int first_class,
    float* __restrict__ sim, long long* __restrict__ label, float* __restrict__ best_val, int k0, int multi) {
    constexpr int KC = NK4 * 4;
    extern __shared__ __align__(128) unsigned char smem_raw[];
    float(*X)[kHCS][kHeadBlockPix] = reinterpret_cast<float(*)[kHCS][kHeadBlockPix]>(smem_raw);
    float* Ts = reinterpret_cast<float*>(smem_raw + kHeadRingBytes);  // [C][KC], zero padded
    __shared__ uint64_t full_bar[kHNS], empty_bar[kHNS];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int kc = min(KC, K - k0);
    const long long blk = (long long)blockIdx.x * kHeadBlockPix;
    const uint32_t npx = (uint32_t)min((long long)kHeadBlockPix, N - blk);  // multiple of 4
    const long long px0 = blk + (long long)tid * 2;
    const bool any = px0 < N;  // N is even: both pixels of the pair are inside

    if (tid == 0) {
        for (int i = 0; i < kHNS; i++) {
            mbar_init(&full_bar[i], 1);
            mbar_init(&empty_bar[i], kTmaThreads / 32);
        }
        mbar_fence_init();
    }
    for (int e = tid; e < C * KC; e += kTmaThreads) {
        const int c = e / KC, k = e - c * KC;
        Ts[e] = k < kc ? __ldg(text + (size_t)(k0 + k) * C + c) : 0.f;
    }
    __syncthreads();

    const int nb = (C + kHCS - 1) / kHCS;
    int pb = 0;  // next stage-batch to issue (warp 0)
    auto produce = [&]() {  // warp 0, converged
        const int st = pb % kHNS;
        const int cnt = min(kHCS, C - pb * kHCS);
        if (pb >= kHNS) mbar_wait(&empty_bar[st], (uint32_t)(((pb / kHNS) - 1) & 1));  // all warps released it
        if (lane < cnt)
            bulk_g2s(&X[st][lane][0], render + (size_t)(pb * kHCS + lane) * N + blk, npx * 4u, &full_bar[st]);
        __syncwarp();
        if (lane == 0) mbar_arrive_expect_tx(&full_bar[st], (uint32_t)cnt * npx * 4u);
        pb++;
    };
    if (warp == 0)
        for (int i = 0; i < kHNS - 1 && pb < nb; i++) produce();

    float2 acc[KC];
#pragma unroll
    for (int k = 0; k < KC; k++) acc[k] = make_float2(0.f, 0.f);
    float2 nrm = make_float2(0.f, 0.f);

    for (int b = 0; b < nb; b++) {
        const int st = b % kHNS;
        const int cnt = min(kHCS, C - b * kHCS);
        if (warp == 0 && pb < nb) produce();  // refill the stage everybody left one batch ago
        mbar_wait(&full_bar[st], (uint32_t)((b / kHNS) & 1));
        if (any) {
            const float* trow0 = Ts + (size_t)(b * kHCS) * KC;
            auto channel = [&](int c) {
                const float2 x = *reinterpret_cast<const float2*>(&X[st][c][tid * 2]);
                nrm = ffma2(x, x, nrm);
                const float* trow = trow0 + c * KC;
#pragma unroll
                for (int q = 0; q < NK4; q++) {
                    const float4 t = *reinterpret_cast<const float4*>(trow + q * 4);
                    acc[q * 4 + 0] = ffma2(x, make_float2(t.x, t.x), acc[q * 4 + 0]);
                    acc[q * 4 + 1] = ffma2(x, make_float2(t.y, t.y), acc[q * 4 + 1]);
                    acc[q * 4 + 2] = ffma2(x, make_float2(t.z, t.z), acc[q * 4 + 2]);
                    acc[q * 4 + 3] = ffma2(x, make_float2(t.w, t.w), acc[q * 4 + 3]);
                }
            };
            if (cnt == kHCS) {
#pragma unroll
                for (int c = 0; c < kHCS; c++) channel(c);
            } else {
                for (int c = 0; c < cnt; c++) channel(c);
            }
        }
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty_bar[st]);
    }
    if (!any) return;

    const float inv0 = 1.f / (sqrtf(nrm.x) + 1e-8f), inv1 = 1.f / (sqrtf(nrm.y) + 1e-8f);
    float bv0 = 0.f, bv1 = 0.f;
    int bk0 = -1, bk1 = -1;
#pragma unroll
    for (int k = 0; k < KC; k++) {
        if (k >= kc) break;
        const float s0 = acc[k].x * inv0, s1 = acc[k].y * inv1;
        if (sim) *reinterpret_cast<float2*>(sim + (size_t)(k0 + k) * N + px0) = make_float2(s0, s1);
        if (k0 + k >= first_class) {  // first maximum wins, like torch.argmax
            if (bk0 < 0 || s0 > bv0) { bv0 = s0; bk0 = k0 + k; }
            if (bk1 < 0 || s1 > bv1) { bv1 = s1; bk1 = k0 + k; }
        }
    }
    if (label && bk0 >= 0) {
        long long l0 = (long long)(bk0 - first_class), l1 = (long long)(bk1 - first_class);
        if (multi != 0) {
            if (multi == 1 || bv0 > best_val[px0]) best_val[px0] = bv0;
            else l0 = label[px0];
            if (multi == 1 || bv1 > best_val[px0 + 1]) best_val[px0 + 1] = bv1;
            else l1 = label[px0 + 1];
        }
        *reinterpret_cast<longlong2*>(label + px0) = make_longlong2(l0, l1);  // px0 even: 16-byte aligned
    }
}

// Per-Gaussian similarities  out[p][k] = sum_c features[p][c] * text[k][c]  (einsum "cq,dq->dc"),
// written with a row pitch of Kpad floats, columns K..Kpad-1 zero.  Thread = two Gaussian rows, walked with
// 16-byte loads (a row's 128-byte lines stay in L1 between iterations, so DRAM sees every line once); the
// class embeddings sit transposed [C][KC] in shared memory and are read as broadcast LDS.128, 2 x KC register
// accumulators, no cross-lane reduction.  (The first version — warp per row, butterfly reduction of every
// class — spends most of its issue slots on SHFL/FADD.)
template <int NK4>
__global__ void __launch_bounds__(256) feature_logits_kernel(int P, int C, int K, int Kpad, int k0,
                                                             const float* __restrict__ features,
                                                             const float* __restrict__ text,
                                                             const float* __restrict__ kbias, float* __restrict__ out) {
    constexpr int KC = NK4 * 4;
    extern __shared__ __align__(16) float Ts[];  // [Cp][KC], Cp = C rounded up to 4, zero padded
    const int Cp = (C + 3) & ~3;
    const int kc = min(KC, K - k0);              // real classes in this pass (may be <= 0 for a pure padding pass)
    for (int e = threadIdx.x; e < Cp * KC; e += blockDim.x) {
        const int c = e / KC, k = e - c * KC;
        Ts[e] = (c < C && k < kc) ? __ldg(text + (size_t)(k0 + k) * C + c) : 0.f;
    }
    __syncthreads();
    const bool vec = (C & 3) == 0 && ((reinterpret_cast<uintptr_t>(features) & 15) == 0);
    const int cols = min(KC, Kpad - k0);         // columns this pass writes (classes + zero padding)
    const bool vout = (Kpad & 3) == 0 && (k0 & 3) == 0 && ((reinterpret_cast<uintptr_t>(out) & 15) == 0);
    for (long long p0 = 2ll * (blockIdx.x * blockDim.x + threadIdx.x); p0 < P; p0 += 2ll * gridDim.x * blockDim.x) {
        const bool two = p0 + 1 < P;
        const float* r0 = features + (size_t)p0 * C;
        const float* r1 = two ? r0 + C : r0;
        float a0[KC], a1[KC];
#pragma unroll
        for (int k = 0; k < KC; k++) { a0[k] = 0.f; a1[k] = 0.f; }
#pragma unroll 2
        for (int c = 0; c < Cp; c += 4) {
            float f0[4], f1[4];
            if (vec) {
                const float4 v0 = __ldg(reinterpret_cast<const float4*>(r0 + c));
                const float4 v1 = __ldg(reinterpret_cast<const float4*>(r1 + c));
                f0[0] = v0.x; f0[1] = v0.y; f0[2] = v0.z; f0[3] = v0.w;
                f1[0] = v1.x; f1[1] = v1.y; f1[2] = v1.z; f1[3] = v1.w;
            } else {
#pragma unroll
                for (int j = 0; j < 4; j++) {
                    f0[j] = c + j < C ? __ldg(r0 + c + j) : 0.f;
                    f1[j] = c + j < C ? __ldg(r1 + c + j) : 0.f;
                }
            }
#pragma unroll
            for (int j = 0; j < 4; j++) {
                const float* trow = Ts + (size_t)(c + j) * KC;
#pragma unroll
                for (int q = 0; q < NK4; q++) {
                    const float4 t = *reinterpret_cast<const float4*>(trow + 4 * q);
                    a0[4 * q + 0] = fmaf(f0[j], t.x, a0[4 * q + 0]);
                    a0[4 * q + 1] = fmaf(f0[j], t.y, a0[4 * q + 1]);
                    a0[4 * q + 2] = fmaf(f0[j], t.z, a0[4 * q + 2]);
                    a0[4 * q + 3] = fmaf(f0[j], t.w, a0[4 * q + 3]);
                    a1[4 * q + 0] = fmaf(f1[j], t.x, a1[4 * q + 0]);
                    a1[4 * q + 1] = fmaf(f1[j], t.y, a1[4 * q + 1]);
                    a1[4 * q + 2] = fmaf(f1[j], t.z, a1[4 * q + 2]);
                    a1[4 * q + 3] = fmaf(f1[j], t.w, a1[4 * q + 3]);
                }
            }
        }
        // padding columns (k >= kc) accumulated zeros: the embedding table is zero there
        if (kbias) {  // per-class constant added to the finished dot product (decoded logits: beta = text . bias)
#pragma unroll
            for (int k = 0; k < KC; k++)
                if (k < kc) {
                    const float bk = __ldg(kbias + k0 + k);
                    a0[k] += bk;
                    a1[k] += bk;
                }
        }
        float* o0 = out + (size_t)p0 * Kpad + k0;
        float* o1 = o0 + Kpad;
        if (vout) {
#pragma unroll
            for (int q = 0; q < NK4; q++) {
                if (4 * q >= cols) break;
                *reinterpret_cast<float4*>(o0 + 4 * q) = make_float4(a0[4 * q], a0[4 * q + 1], a0[4 * q + 2], a0[4 * q + 3]);
                if (two)
                    *reinterpret_cast<float4*>(o1 + 4 * q) = make_float4(a1[4 * q], a1[4 * q + 1], a1[4 * q + 2], a1[4 * q + 3]);
            }
        } else {
#pragma unroll
            for (int k = 0; k < KC; k++) {
                if (k >= cols) break;
                o0[k] = a0[k];
                if (two) o1[k] = a1[k];
            }
        }
    }
}

// label[p] = argmax_{k in [first_class, K)} planes[k][p] - first_class   (rendering[1:].argmax(dim=0),
// eval_segmentation.py:144,244,375,418)
__global__ void label_argmax_kernel(int K, int first_class, long long N, const float* __restrict__ planes,
                                    long long* __restrict__ label) {
    const long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= N) return;
    float bv = __ldg(planes + (size_t)first_class * N + p);
    int bk = first_class;
    for (int k = first_class + 1; k < K; k++) {
        const float v = __ldg(planes + (size_t)k * N + p);
        if (v > bv) { bv = v; bk = k; }
    }
    label[p] = (long long)(bk - first_class);
}

// Training counterpart of the head: open-vocabulary distillation loss of a rendered feature image against
// per-pixel class embeddings,  L = -(1 / (C N)) sum_p <render[:, p], E[label(p)]>,  and its gradient
// dL/drender[c][p] = -E[label(p)][c] / (C N), in ONE pass (render read once, gradient written once; the torch
// formulation — index_select of the (C,K) table + dot — moves 1.5x the bytes in three kernels).  Thread = 4
// consecutive pixels, the pre-scaled table sits transposed [C][K+1] in shared memory (odd pitch: lanes with
// different labels hit different banks, equal labels broadcast).
// Pixels whose label lies outside [0, K) are IGNORED (ScanNet-style -1 / 255 "unannotated"): zero gradient, no loss
// term, and they do not count in the normaliser.  The number of valid pixels is counted first (loss[1]).
template <typename LabelT>
__global__ void __launch_bounds__(256) count_valid_labels_kernel(int K, long long N, const LabelT* __restrict__ labels,
                                                                 double* __restrict__ valid) {
    long long n = 0;
    for (long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x; p < N; p += (long long)gridDim.x * blockDim.x) {
        const long long l = (long long)labels[p];
        n += (l >= 0 && l < K);
    }
    int ni = (int)n;
    ni = __reduce_add_sync(0xffffffffu, ni);
    if ((threadIdx.x & 31) == 0 && ni) atomicAdd(valid, (double)ni);
}

template <bool VEC, typename LabelT>
__global__ void __launch_bounds__(256) distill_loss_kernel(int C, int K, long long N, const float* __restrict__ render,
                                                           const float* __restrict__ emb, const LabelT* __restrict__ labels,
                                                           float* __restrict__ dL, double* __restrict__ loss) {
    extern __shared__ float Es[];  // [C][Kp]; column K is all zero: the "ignored" class
    const int Kp = (K + 1) | 1;
    const double nvalid = loss[1];
    const float scale = (float)(-1.0 / ((double)C * (nvalid > 0.0 ? nvalid : 1.0)));
    for (int e = threadIdx.x; e < C * K; e += blockDim.x) {
        const int k = e / C, c = e - k * C;  // coalesced read of emb (K,C)
        Es[c * Kp + k] = __ldg(emb + e) * scale;
    }
    for (int c = threadIdx.x; c < C; c += blockDim.x) Es[c * Kp + K] = 0.f;
    __syncthreads();
    const long long p0 = VEC ? ((long long)blockIdx.x * 256 + threadIdx.x) * 4 : (long long)blockIdx.x * 1024 + threadIdx.x;
    long long px[4];
    int lab[4];
#pragma unroll
    for (int i = 0; i < 4; i++) {
        px[i] = VEC ? p0 + i : p0 + (long long)i * 256;
        const long long l = px[i] < N ? (long long)labels[px[i]] : -1;
        lab[i] = (l >= 0 && l < K) ? (int)l : K;  // out-of-range labels read the zero column: ignored
    }
    float acc = 0.f;
    if (px[0] < N) {
#pragma unroll 4
        for (int c = 0; c < C; c++) {
            const float* row = Es + c * Kp;
            const float e0 = row[lab[0]], e1 = row[lab[1]], e2 = row[lab[2]], e3 = row[lab[3]];
            const size_t off = (size_t)c * N;
            if (VEC) {
                const float4 x = __ldg(reinterpret_cast<const float4*>(render + off + px[0]));
                acc = fmaf(x.x, e0, fmaf(x.y, e1, fmaf(x.z, e2, fmaf(x.w, e3, acc))));
                *reinterpret_cast<float4*>(dL + off + px[0]) = make_float4(e0, e1, e2, e3);
            } else {
                const float ev[4] = {e0, e1, e2, e3};
#pragma unroll
                for (int i = 0; i < 4; i++)
                    if (px[i] < N) {
                        acc = fmaf(__ldg(render + off + px[i]), ev[i], acc);
                        dL[off + px[i]] = ev[i];
                    }
            }
        }
    }
    double d = (double)acc;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) d += __shfl_xor_sync(0xffffffffu, d, o);
    __shared__ double wsum[8];
    if ((threadIdx.x & 31) == 0) wsum[threadIdx.x >> 5] = d;
    __syncthreads();
    if (threadIdx.x == 0) {
        double t = 0.0;
        for (int w = 0; w < 8; w++) t += wsum[w];
        atomicAdd(loss, t);
    }
}

template <int NK4>
void launch_head_t(int C, int K, long long N, const float* render, const float* text, int first_class, float* sim,
                   long long* label, float* best_val, int k0, int multi, cudaStream_t s) {
    const bool vec = (N % 4 == 0) && ((reinterpret_cast<uintptr_t>(render) & 15) == 0) &&
                     (!sim || (reinterpret_cast<uintptr_t>(sim) & 15) == 0);
    const unsigned blocks = (unsigned)((N + kHeadBlockPix - 1) / kHeadBlockPix);  // 1024 pixels per CTA either way
    const size_t smem_tma = kHeadRingBytes + sizeof(float) * (size_t)C * NK4 * 4;
    if (vec && smem_tma <= 224 * 1024 && (!label || (reinterpret_cast<uintptr_t>(label) & 15) == 0)) {
        static DeviceOnce attr_set;
        if (attr_set.first_use_on_device()) {
            cudaFuncSetAttribute(semantic_head_tma_kernel<NK4>, cudaFuncAttributeMaxDynamicSharedMemorySize, 224 * 1024);
        }
        semantic_head_tma_kernel<NK4><<<blocks, kTmaThreads, smem_tma, s>>>(C, K, N, render, text, first_class, sim,
                                                                            label, best_val, k0, multi);
        return;
    }
    if (vec)
        semantic_head_kernel<NK4, true><<<blocks, kHeadThreads, 0, s>>>(C, K, N, render, text, first_class, sim, label,
                                                                       best_val, k0, multi);
    else
        semantic_head_kernel<NK4, false><<<blocks, kHeadThreads, 0, s>>>(C, K, N, render, text, first_class, sim, label,
                                                                        best_val, k0, multi);
}

}  // namespace

static int launch_semantic_head(sgb_ctx* ctx, int C, int K, long long N, const float* render, const float* text,
                         int first_class, float* sim, long long* label, cudaStream_t s) {
    const int passes = (K + kMaxKC - 1) / kMaxKC;
    float* best_val = nullptr;
    if (passes > 1 && label) {
        if (!ctx) { set_error("sgb_semantic_head: more than %d classes with a label map needs a ctx (scratch)", kMaxKC); return SGB_E_INVALID; }
        int rc = ctx->misc.ensure(sizeof(float) * (size_t)N);
        if (rc) return rc;
        best_val = (float*)ctx->misc.p;
    }
    for (int pass = 0; pass < passes; pass++) {
        const int k0 = pass * kMaxKC;
        const int kc = min(kMaxKC, K - k0);
        // a pass entirely below first_class still writes its sim planes but takes no part in the arg-max;
        // the first pass that does initialises best_val
        const int multi = passes == 1 ? 0 : (pass == first_class / kMaxKC ? 1 : 2);
        long long* lab = (k0 + kc <= first_class) ? nullptr : label;
        if (!sim && !lab) continue;
        const int nk4 = (kc + 3) / 4;
        if (nk4 <= 2) launch_head_t<2>(C, K, N, render, text, first_class, sim, lab, best_val, k0, multi, s);
        else if (nk4 <= 4) launch_head_t<4>(C, K, N, render, text, first_class, sim, lab, best_val, k0, multi, s);
        else if (nk4 <= 6) launch_head_t<6>(C, K, N, render, text, first_class, sim, lab, best_val, k0, multi, s);
        else launch_head_t<8>(C, K, N, render, text, first_class, sim, lab, best_val, k0, multi, s);
        SGB_LAUNCH_CHECK("semantic_head_kernel", 0, s);
        if (ctx) ctx->launches += 1;
    }
    return SGB_OK;
}

template <int NK4>
static int launch_logits_t(int P, int C, int K, int Kpad, int k0, const float* features, const float* text,
                           const float* kbias, float* out, cudaStream_t s) {
    const int Cp = (C + 3) & ~3;
    const size_t smem = sizeof(float) * (size_t)NK4 * 4 * Cp;
    if (smem > 200 * 1024) {
        set_error("sgb_feature_logits: C = %d too large (class embeddings must fit shared memory)", C);
        return SGB_E_INVALID;
    }
    static DeviceOnce attr_set;
    if (attr_set.first_use_on_device()) {
        SGB_CUDA(cudaFuncSetAttribute(feature_logits_kernel<NK4>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    }
    const int blocks = min((P + 511) / 512, kNumSMs * 8);
    feature_logits_kernel<NK4><<<blocks, 256, smem, s>>>(P, C, K, Kpad, k0, features, text, kbias, out);
    SGB_LAUNCH_CHECK("feature_logits_kernel", 0, s);
    return SGB_OK;
}

int launch_feature_logits(int P, int C, int K, int Kpad, const float* features, const float* text, const float* kbias,
                          float* out, cudaStream_t s) {
    for (int k0 = 0; k0 < Kpad; k0 += 32) {
        const int span = min(32, Kpad - k0);  // columns this pass writes (classes + zero padding)
        int rc;
        if (span <= 8) rc = launch_logits_t<2>(P, C, K, Kpad, k0, features, text, kbias, out, s);
        else if (span <= 16) rc = launch_logits_t<4>(P, C, K, Kpad, k0, features, text, kbias, out, s);
        else if (span <= 24) rc = launch_logits_t<6>(P, C, K, Kpad, k0, features, text, kbias, out, s);
        else rc = launch_logits_t<8>(P, C, K, Kpad, k0, features, text, kbias, out, s);
        if (rc) return rc;
    }
    return SGB_OK;
}

static int launch_label_argmax(int K, int first_class, long long N, const float* planes, long long* label, cudaStream_t s) {
    label_argmax_kernel<<<(unsigned)((N + 255) / 256), 256, 0, s>>>(K, first_class, N, planes, label);
    SGB_LAUNCH_CHECK("label_argmax_kernel", 0, s);
    return SGB_OK;
}

}  // namespace sgb

using namespace sgb;

extern "C" {

int sgb_distill_loss(int32_t C, int32_t K, int64_t N, const float* render, const float* class_emb, const void* labels,
                     int32_t labels_are_int64, float* dL_drender, double* loss, void* stream) {
    cudaStream_t s = (cudaStream_t)stream;
    if (C <= 0 || K <= 0 || N < 0) { set_error("sgb_distill_loss: need C > 0, K > 0, N >= 0"); return SGB_E_INVALID; }
    if (!loss) { set_error("sgb_distill_loss: null loss"); return SGB_E_INVALID; }
    SGB_CUDA(cudaMemsetAsync(loss, 0, 2 * sizeof(double), s));
    if (N == 0) return SGB_OK;
    if (!render || !class_emb || !labels || !dL_drender) { set_error("sgb_distill_loss: null argument"); return SGB_E_INVALID; }
    const size_t smem = sizeof(float) * (size_t)C * ((K + 1) | 1);
    if (smem > 200 * 1024) { set_error("sgb_distill_loss: C x K = %d x %d does not fit shared memory", C, K); return SGB_E_INVALID; }
    if (labels_are_int64)
        count_valid_labels_kernel<long long><<<kNumSMs * 4, 256, 0, s>>>(K, (long long)N, (const long long*)labels, loss + 1);
    else
        count_valid_labels_kernel<int><<<kNumSMs * 4, 256, 0, s>>>(K, (long long)N, (const int*)labels, loss + 1);
    const bool vec = (N % 4 == 0) && ((reinterpret_cast<uintptr_t>(render) & 15) == 0) &&
                     ((reinterpret_cast<uintptr_t>(dL_drender) & 15) == 0);
    const unsigned blocks = (unsigned)((N + 1023) / 1024);
#define SGB_DISTILL(VECF, T)                                                                                          \
    do {                                                                                                              \
        static DeviceOnce once;                                                                                       \
        if (once.first_use_on_device())                                                                               \
            SGB_CUDA(cudaFuncSetAttribute(distill_loss_kernel<VECF, T>, cudaFuncAttributeMaxDynamicSharedMemorySize,  \
                                          200 * 1024));                                                               \
        distill_loss_kernel<VECF, T><<<blocks, 256, smem, s>>>(C, K, (long long)N, render, class_emb, (const T*)labels, \
                                                               dL_drender, loss);                                     \
    } while (0)
    if (vec && labels_are_int64) SGB_DISTILL(true, long long);
    else if (vec) SGB_DISTILL(true, int);
    else if (labels_are_int64) SGB_DISTILL(false, long long);
    else SGB_DISTILL(false, int);
#undef SGB_DISTILL
    SGB_LAUNCH_CHECK("distill_loss_kernel", 0, s);
    return SGB_OK;
}

int sgb_semantic_head(sgb_ctx* ctx, int32_t C, int32_t K, int64_t N, const float* render, const float* text,
                      int32_t first_class, float* sim, int64_t* label, void* stream) {
    if (C <= 0 || K <= 0 || N < 0 || first_class < 0 || first_class >= K) {
        set_error("sgb_semantic_head: need C > 0, K > 0, N >= 0 and 0 <= first_class < K");
        return SGB_E_INVALID;
    }
    if (N == 0 || (!sim && !label)) return SGB_OK;
    if (!render || !text) { set_error("sgb_semantic_head: null input"); return SGB_E_INVALID; }
    return launch_semantic_head(ctx, C, K, (long long)N, render, text, first_class, sim, (long long*)label,
                                (cudaStream_t)stream);
}

int sgb_feature_logits(int32_t P, int32_t C, int32_t K, int32_t Kpad, const float* features, const float* text,
                       float* out, void* stream) {
    if (P < 0 || C <= 0 || K <= 0 || Kpad < K) {
        set_error("sgb_feature_logits: need P >= 0, C > 0, K > 0, Kpad >= K");
        return SGB_E_INVALID;
    }
    if (P == 0) return SGB_OK;
    if (!features || !text || !out) { set_error("sgb_feature_logits: null argument"); return SGB_E_INVALID; }
    return launch_feature_logits(P, C, K, Kpad, features, text, nullptr, out, (cudaStream_t)stream);
}

int sgb_label_argmax(int32_t K, int32_t first_class, int64_t N, const float* planes, int64_t* label, void* stream) {
    if (K <= 0 || first_class < 0 || first_class >= K || N < 0) {
        set_error("sgb_label_argmax: need K > 0, 0 <= first_class < K, N >= 0");
        return SGB_E_INVALID;
    }
    if (N == 0) return SGB_OK;
    if (!planes || !label) { set_error("sgb_label_argmax: null argument"); return SGB_E_INVALID; }
    return launch_label_argmax(K, first_class, (long long)N, planes, (long long*)label, (cudaStream_t)stream);
}

}  // extern "C"
