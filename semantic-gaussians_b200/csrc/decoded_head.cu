// Open-vocabulary semantic head of a compact feature field seen through its linear decoder.  The field renders c
// channels, R (c, N) planar; the decoder lifts pixel p to x_p = W r_p + b (W (C, c) row-major, b (C) or absent) in
// the C channels of the text embeddings T (K, C).  Because the decoder is linear, nothing of size C x N is needed:
//
//   T x_p     = A r_p + beta                        A = T W (K x c),  beta = T b (K)
//   |x_p|^2   = r_p^T G r_p + 2 u . r_p + |b|^2     G = W^T W (c x c),  u = W^T b
//
// so   sim[k][p] = (A r_p + beta)_k / (|x_p| + 1e-8)   and   label[p] = argmax_{k >= first_class} (A r_p + beta)_k.
// The positive divisor does not move the arg-max, so the label is taken from the numerators in both modes and a
// label-only call never forms |x_p|: one read of R and K c FFMA per pixel.
//
// Prologue (decoded_head_prologue_kernel): A, beta, G, u and |b|^2, each entry a float64 dot product over C in index
// order.  A and beta are rounded to fp32 (the numerators are fp32 FFMA); G, u and |b|^2 stay float64.  The quadratic
// form is evaluated per pixel in float64 from the fp32 r_p: in fp32 it cancels when |x_p| << | |W| |r_p| + |b| |
// (a relative error growing like eps kappa^2), in float64 the same cancellation stays far below fp32 resolution.
//
// Main kernel (decoded_head_kernel): one CTA per 128-pixel block stages R_blk (c x 128) in shared memory once.
//   norm      (sim only) Y = G R_blk + 2u as float64 register tiles (8 rows x 4 pixels per thread), q_p = r_p . y_p
//             summed over the 8 row groups in a fixed order; den_p = sqrt(max(q_p, 0)) + 1e-8.
//   classes   per chunk of 64 classes, the chunk of A (transposed, packed by the prologue) and beta in shared memory,
//             numerators as fp32 register tiles (4 classes x 8 pixels per thread), sim written straight from the
//             tile, running arg-max per thread; the 16 class groups are merged in a fixed order at the end.
// Every sum has a fixed order and there are no atomics: every output is bitwise reproducible.
//
// sgb_decoded_feature_logits is the per-Gaussian twin: the prologue's A and beta fed to feature_logits_kernel
// (semantic.cu) as the class table and a per-class constant.
#include <algorithm>

#include "common.cuh"
#include "feature_loss.cuh"
#include "semantic.cuh"

namespace sgb {
namespace {

constexpr int kDhThreads = 256;
constexpr int kDhPB = 128;            // pixels per block
constexpr int kDhKC = 64;             // classes per chunk
constexpr int kDhPitch = kDhPB + 4;   // shared row pitch of the R tile
constexpr int kDhMaxc = 128;          // widest compact field accepted
constexpr int kDhMaxK = 1024;         // most classes accepted
constexpr int kDhMaxSmem = 227 * 1024;

inline int padded_c(int c) { return c <= 16 ? 16 : c <= 32 ? 32 : c <= 64 ? 64 : 128; }
__host__ __device__ inline int padded_K(int K) { return (K + kDhKC - 1) / kDhKC * kDhKC; }

// Workspace: A row-major (K, c) for the logits, A chunk-transposed [Kp / 64][cp][64] for the head, beta [Kp], G [cp][cp]
// and 2u [cp] in float64, |b|^2.  Byte offsets, each 256-aligned; zero outside (K, c).
struct DhWorkspace {
    size_t ar, at, beta, g, u2, bb, total;
};
DhWorkspace workspace_layout(int c, int K) {
    const size_t cp = padded_c(c), Kp = padded_K(K);
    auto up = [](size_t b) { return (b + 255) & ~(size_t)255; };
    DhWorkspace w;
    w.ar = 0;
    w.at = w.ar + up((size_t)K * c * sizeof(float));
    w.beta = w.at + up(Kp * cp * sizeof(float));
    w.g = w.beta + up(Kp * sizeof(float));
    w.u2 = w.g + up(cp * cp * sizeof(double));
    w.bb = w.u2 + up(cp * sizeof(double));
    w.total = w.bb + up(sizeof(double));
    return w;
}

struct DhTables {
    float* Ar;
    float* At;
    float* beta;
    double* G;
    double* u2;
    double* bb;
};

DhTables tables(void* workspace, int c, int K) {
    const DhWorkspace L = workspace_layout(c, K);
    unsigned char* ws = static_cast<unsigned char*>(workspace);
    return {reinterpret_cast<float*>(ws + L.ar), reinterpret_cast<float*>(ws + L.at),
            reinterpret_cast<float*>(ws + L.beta), reinterpret_cast<double*>(ws + L.g),
            reinterpret_cast<double*>(ws + L.u2), reinterpret_cast<double*>(ws + L.bb)};
}

// One thread per table entry, each a float64 dot product over the C decoded channels in index order.  norm == 0
// skips G, u and |b|^2 (the logits need A and beta only).
__global__ void __launch_bounds__(256) decoded_head_prologue_kernel(int C, int c, int K, int cp, int norm,
                                                                    const float* __restrict__ T,
                                                                    const float* __restrict__ W,
                                                                    const float* __restrict__ b, DhTables t) {
    const long long Kp = padded_K(K);
    const long long nA = Kp * cp, nB = Kp, nG = norm ? (long long)cp * cp : 0, nU = norm ? cp : 0, nBB = norm ? 1 : 0;
    const long long total = nA + nB + nG + nU + nBB;
    for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < total;
         e += (long long)gridDim.x * blockDim.x) {
        if (e < nA) {
            const int k = (int)(e / cp), j = (int)(e % cp);
            float v = 0.f;
            if (k < K && j < c) {
                double s = 0.0;
                for (int i = 0; i < C; i++) s = fma((double)__ldg(T + (size_t)k * C + i), (double)__ldg(W + (size_t)i * c + j), s);
                v = (float)s;
                t.Ar[(size_t)k * c + j] = v;
            }
            t.At[(size_t)(k / kDhKC) * cp * kDhKC + (size_t)j * kDhKC + k % kDhKC] = v;
            continue;
        }
        long long f = e - nA;
        if (f < nB) {
            const int k = (int)f;
            double s = 0.0;
            if (k < K && b)
                for (int i = 0; i < C; i++) s = fma((double)__ldg(T + (size_t)k * C + i), (double)__ldg(b + i), s);
            t.beta[k] = (float)s;
            continue;
        }
        f -= nB;
        if (f < nG) {
            const int r = (int)(f / cp), j = (int)(f % cp);
            double s = 0.0;
            if (r < c && j < c)
                for (int i = 0; i < C; i++)
                    s = fma((double)__ldg(W + (size_t)i * c + r), (double)__ldg(W + (size_t)i * c + j), s);
            t.G[f] = s;
            continue;
        }
        f -= nG;
        if (f < nU) {
            const int j = (int)f;
            double s = 0.0;
            if (j < c && b)
                for (int i = 0; i < C; i++) s = fma((double)__ldg(W + (size_t)i * c + j), (double)__ldg(b + i), s);
            t.u2[j] = 2.0 * s;
            continue;
        }
        double s = 0.0;
        if (b)
            for (int i = 0; i < C; i++) s = fma((double)__ldg(b + i), (double)__ldg(b + i), s);
        *t.bb = s;
    }
}

struct DhArgs {
    int K, c, first_class, vec;
    long long N;
    const float* R;
    DhTables t;
    float* sim;
    long long* label;
};

template <int CP, bool NORM>
size_t head_smem_bytes() {
    const size_t region = NORM ? std::max<size_t>((size_t)CP * CP * sizeof(double), (size_t)CP * kDhKC * sizeof(float))
                               : (size_t)CP * kDhKC * sizeof(float);
    return region + (NORM ? CP * sizeof(double) : 0)      // u2s
           + 16 * kDhPB * 2 * sizeof(float)               // red: q partials / arg-max merge
           + (size_t)CP * kDhPitch * sizeof(float)        // Rs
           + kDhKC * sizeof(float) + kDhPB * sizeof(float);  // bs, den
}

// NORM: sim is written (and |x_p| formed); otherwise a label-only call.
template <int CP, bool NORM>
__global__ void __launch_bounds__(kDhThreads, 1) decoded_head_kernel(const DhArgs a) {
    constexpr int RT = CP / 8 < 8 ? CP / 8 : 8;   // norm: rows per thread in a row chunk of 8 RT rows
    constexpr int NRC = CP / (8 * RT);            // norm: row chunks
    constexpr size_t kRegion = NORM ? (CP * CP * sizeof(double) > CP * kDhKC * sizeof(float) ? CP * CP * sizeof(double)
                                                                                             : CP * kDhKC * sizeof(float))
                                    : CP * kDhKC * sizeof(float);
    extern __shared__ __align__(16) unsigned char dh_smem[];
    double* Gs = reinterpret_cast<double*>(dh_smem);                 // [CP][CP]       (norm phase)
    float* Ats = reinterpret_cast<float*>(dh_smem);                  // [CP][kDhKC]    (class phase, same bytes)
    double* u2s = reinterpret_cast<double*>(dh_smem + kRegion);      // [CP]
    unsigned char* red = dh_smem + kRegion + (NORM ? CP * sizeof(double) : 0);  // 16 KB
    float* Rs = reinterpret_cast<float*>(red + 16 * kDhPB * 2 * sizeof(float));  // [CP][kDhPitch]
    float* bs = Rs + CP * kDhPitch;                                  // [kDhKC]
    float* den = bs + kDhKC;                                         // [kDhPB]

    const int tid = threadIdx.x;
    const long long N = a.N;
    const int K = a.K, c = a.c;
    const long long p0 = (long long)blockIdx.x * kDhPB;
    for (int e = tid; e < CP * kDhPB; e += kDhThreads) {
        const int k = e / kDhPB, p = e % kDhPB;
        Rs[k * kDhPitch + p] = k < c && p0 + p < N ? __ldg(a.R + (size_t)k * N + p0 + p) : 0.f;
    }

    if constexpr (NORM) {
        for (int e = tid; e < CP * CP / 2; e += kDhThreads)
            reinterpret_cast<double2*>(Gs)[e] = __ldg(reinterpret_cast<const double2*>(a.t.G) + e);
        for (int e = tid; e < CP; e += kDhThreads) u2s[e] = __ldg(a.t.u2 + e);
        __syncthreads();
        // q_p = sum_i r_i (sum_j G_ij r_j + 2 u_i): thread (tx, ty) = (tid % 32, tid / 32), pixels 4 tx .. 4 tx + 3
        const int tx = tid & 31, ty = tid >> 5;
        double q[4] = {0.0, 0.0, 0.0, 0.0};
#pragma unroll 1
        for (int rc = 0; rc < NRC; rc++) {
            const int row0 = rc * 8 * RT + ty * RT;
            double y[RT][4];
#pragma unroll
            for (int i = 0; i < RT; i++)
#pragma unroll
                for (int j = 0; j < 4; j++) y[i][j] = u2s[row0 + i];
#pragma unroll 4
            for (int k = 0; k < CP; k++) {
                const float4 r = *reinterpret_cast<const float4*>(Rs + k * kDhPitch + 4 * tx);
                const double rv[4] = {(double)r.x, (double)r.y, (double)r.z, (double)r.w};
                double g[RT];
#pragma unroll
                for (int i = 0; i < RT; i += 2) {
                    const double2 g2 = *reinterpret_cast<const double2*>(Gs + k * CP + row0 + i);  // G symmetric
                    g[i] = g2.x;
                    g[i + 1] = g2.y;
                }
#pragma unroll
                for (int i = 0; i < RT; i++)
#pragma unroll
                    for (int j = 0; j < 4; j++) y[i][j] = fma(g[i], rv[j], y[i][j]);
            }
#pragma unroll
            for (int i = 0; i < RT; i++) {
                const float4 r = *reinterpret_cast<const float4*>(Rs + (row0 + i) * kDhPitch + 4 * tx);
                q[0] = fma((double)r.x, y[i][0], q[0]);
                q[1] = fma((double)r.y, y[i][1], q[1]);
                q[2] = fma((double)r.z, y[i][2], q[2]);
                q[3] = fma((double)r.w, y[i][3], q[3]);
            }
        }
        double* qred = reinterpret_cast<double*>(red);  // [8][kDhPB]
#pragma unroll
        for (int j = 0; j < 4; j++) qred[ty * kDhPB + 4 * tx + j] = q[j];
        __syncthreads();
        if (tid < kDhPB) {
            double s = *a.t.bb;
            for (int t = 0; t < 8; t++) s += qred[t * kDhPB + tid];
            den[tid] = (float)(sqrt(s > 0.0 ? s : 0.0) + 1e-8);  // a negative rounding of the square counts as 0
        }
    }

    // numerators: thread (tx, ty) = (tid % 16, tid / 16), pixels px(q) = 4 tx + q % 4 + 64 (q / 4), classes 4 ty + i
    const int tx = tid & 15, ty = tid >> 4;
    auto px = [&](int q) { return 4 * tx + (q & 3) + 64 * (q >> 2); };
    float bv[8];
    int bk[8];
#pragma unroll
    for (int q = 0; q < 8; q++) { bv[q] = 0.f; bk[q] = -1; }
    const int nch = (K + kDhKC - 1) / kDhKC;
    for (int ch = 0; ch < nch; ch++) {
        __syncthreads();  // the norm phase's readers of Gs / the previous chunk's readers of Ats and bs are done
        const float4* src = reinterpret_cast<const float4*>(a.t.At + (size_t)ch * CP * kDhKC);
        for (int e = tid; e < CP * kDhKC / 4; e += kDhThreads) reinterpret_cast<float4*>(Ats)[e] = __ldg(src + e);
        if (tid < kDhKC) bs[tid] = __ldg(a.t.beta + ch * kDhKC + tid);
        __syncthreads();
        float acc[4][8];
#pragma unroll
        for (int i = 0; i < 4; i++)
#pragma unroll
            for (int q = 0; q < 8; q++) acc[i][q] = 0.f;
#pragma unroll 4
        for (int k = 0; k < CP; k++) {
            const float4 w = *reinterpret_cast<const float4*>(Ats + k * kDhKC + 4 * ty);
            const float4 r0 = *reinterpret_cast<const float4*>(Rs + k * kDhPitch + 4 * tx);
            const float4 r1 = *reinterpret_cast<const float4*>(Rs + k * kDhPitch + 64 + 4 * tx);
            const float wv[4] = {w.x, w.y, w.z, w.w};
            const float rv[8] = {r0.x, r0.y, r0.z, r0.w, r1.x, r1.y, r1.z, r1.w};
#pragma unroll
            for (int i = 0; i < 4; i++)
#pragma unroll
                for (int q = 0; q < 8; q++) acc[i][q] = fmaf(wv[i], rv[q], acc[i][q]);
        }
#pragma unroll
        for (int i = 0; i < 4; i++) {
            const int k = ch * kDhKC + 4 * ty + i;
            if (k >= K) break;
            const float beta = bs[4 * ty + i];
            float num[8];
#pragma unroll
            for (int q = 0; q < 8; q++) num[q] = acc[i][q] + beta;
            if constexpr (NORM) {
#pragma unroll
                for (int h = 0; h < 2; h++) {
                    const long long p = p0 + 4 * tx + 64 * h;
                    float s[4];
#pragma unroll
                    for (int j = 0; j < 4; j++) s[j] = num[4 * h + j] / den[4 * tx + 64 * h + j];
                    float* o = a.sim + (size_t)k * N + p;
                    if (a.vec && p + 4 <= N) {
                        *reinterpret_cast<float4*>(o) = make_float4(s[0], s[1], s[2], s[3]);
                    } else {
#pragma unroll
                        for (int j = 0; j < 4; j++)
                            if (p + j < N) o[j] = s[j];
                    }
                }
            }
            if (k >= a.first_class) {
#pragma unroll
                for (int q = 0; q < 8; q++)
                    if (bk[q] < 0 || num[q] > bv[q]) { bv[q] = num[q]; bk[q] = k; }  // first maximum wins
            }
        }
    }
    if (!a.label) return;
    // merge the 16 class groups of each pixel in group order; equal values keep the smaller class (torch.argmax)
    __syncthreads();
    float* mv = reinterpret_cast<float*>(red);       // [16][kDhPB]
    int* mk = reinterpret_cast<int*>(mv + 16 * kDhPB);  // [16][kDhPB]
#pragma unroll
    for (int q = 0; q < 8; q++) {
        mv[ty * kDhPB + px(q)] = bv[q];
        mk[ty * kDhPB + px(q)] = bk[q];
    }
    __syncthreads();
    if (tid < kDhPB && p0 + tid < N) {
        float v = 0.f;
        int kb = -1;
        for (int t = 0; t < 16; t++) {
            const int k = mk[t * kDhPB + tid];
            const float x = mv[t * kDhPB + tid];
            if (k >= 0 && (kb < 0 || x > v || (x == v && k < kb))) { v = x; kb = k; }
        }
        a.label[p0 + tid] = (long long)(kb - a.first_class);
    }
}

template <int CP, bool NORM>
int launch_head(const DhArgs& a, cudaStream_t s) {
    const size_t smem = head_smem_bytes<CP, NORM>();
    static DeviceOnce attr_set;
    if (attr_set.first_use_on_device())
        SGB_CUDA(cudaFuncSetAttribute(decoded_head_kernel<CP, NORM>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                      kDhMaxSmem));
    const unsigned blocks = (unsigned)((a.N + kDhPB - 1) / kDhPB);
    decoded_head_kernel<CP, NORM><<<blocks, kDhThreads, smem, s>>>(a);
    SGB_LAUNCH_CHECK("decoded_head_kernel", 0, s);
    return SGB_OK;
}

template <bool NORM>
int launch_head_width(const DhArgs& a, cudaStream_t s) {
    switch (padded_c(a.c)) {
        case 16: return launch_head<16, NORM>(a, s);
        case 32: return launch_head<32, NORM>(a, s);
        case 64: return launch_head<64, NORM>(a, s);
        default: return launch_head<128, NORM>(a, s);
    }
}

int launch_prologue(int C, int c, int K, int norm, const float* text, const float* weight, const float* bias,
                    const DhTables& t, cudaStream_t s) {
    const int cp = padded_c(c);
    const long long Kp = padded_K(K);
    const long long total = Kp * cp + Kp + (norm ? (long long)cp * cp + cp + 1 : 0);
    const int blocks = (int)std::min<long long>((total + 255) / 256, (long long)kNumSMs * 8);
    decoded_head_prologue_kernel<<<blocks, 256, 0, s>>>(C, c, K, cp, norm, text, weight, bias, t);
    SGB_LAUNCH_CHECK("decoded_head_prologue_kernel", 0, s);
    return SGB_OK;
}

int check_widths(const char* fn, int C, int c, int K) {
    if (C < 1 || C > kFeatMaxC) { set_error("%s: C = %d outside [1, %d]", fn, C, kFeatMaxC); return SGB_E_INVALID; }
    if (c < 1 || c > kDhMaxc) { set_error("%s: c = %d outside [1, %d]", fn, c, kDhMaxc); return SGB_E_INVALID; }
    if (K < 1 || K > kDhMaxK) { set_error("%s: K = %d outside [1, %d]", fn, K, kDhMaxK); return SGB_E_INVALID; }
    return SGB_OK;
}

int check_workspace(const char* fn, const void* workspace) {
    if (!workspace) { set_error("%s: null workspace", fn); return SGB_E_INVALID; }
    if ((reinterpret_cast<uintptr_t>(workspace) & 15) != 0) {
        set_error("%s: workspace is not 16-byte aligned", fn);
        return SGB_E_INVALID;
    }
    return SGB_OK;
}

}  // namespace
}  // namespace sgb

using namespace sgb;

extern "C" {

size_t sgb_decoded_semantic_head_workspace_bytes(int32_t C, int32_t c, int32_t K) {
    if (C < 1 || C > kFeatMaxC || c < 1 || c > kDhMaxc || K < 1 || K > kDhMaxK) return 0;
    return workspace_layout(c, K).total;
}

int sgb_decoded_semantic_head(int32_t C, int32_t c, int32_t K, int64_t N, const float* render, const float* weight,
                              const float* bias, const float* text, int32_t first_class, float* sim, int64_t* label,
                              void* workspace, void* stream) {
    static const char* fn = "sgb_decoded_semantic_head";
    if (check_widths(fn, C, c, K) != SGB_OK) return SGB_E_INVALID;
    if (N < 0) { set_error("%s: N = %lld is negative", fn, (long long)N); return SGB_E_INVALID; }
    if (first_class < 0 || first_class >= K) {
        set_error("%s: first_class = %d outside [0, K = %d)", fn, first_class, K);
        return SGB_E_INVALID;
    }
    if (N == 0 || (!sim && !label)) return SGB_OK;
    if (!render) { set_error("%s: null render", fn); return SGB_E_INVALID; }
    if (!weight) { set_error("%s: null weight", fn); return SGB_E_INVALID; }
    if (!text) { set_error("%s: null text", fn); return SGB_E_INVALID; }
    if (check_workspace(fn, workspace) != SGB_OK) return SGB_E_INVALID;
    if (label && (reinterpret_cast<uintptr_t>(label) & 7) != 0) {
        set_error("%s: label is not 8-byte aligned", fn);
        return SGB_E_INVALID;
    }
    cudaStream_t s = (cudaStream_t)stream;
    const DhTables t = tables(workspace, c, K);
    int rc = launch_prologue(C, c, K, sim != nullptr, text, weight, bias, t, s);
    if (rc != SGB_OK) return rc;
    DhArgs a;
    a.K = K;
    a.c = c;
    a.first_class = first_class;
    a.N = (long long)N;
    a.vec = N % 4 == 0 && (reinterpret_cast<uintptr_t>(sim) & 15) == 0;
    a.R = render;
    a.t = t;
    a.sim = sim;
    a.label = (long long*)label;
    return sim ? launch_head_width<true>(a, s) : launch_head_width<false>(a, s);
}

int sgb_decoded_feature_logits(int32_t P, int32_t C, int32_t c, int32_t K, int32_t Kpad, const float* features,
                               const float* weight, const float* bias, const float* text, float* out, void* workspace,
                               void* stream) {
    static const char* fn = "sgb_decoded_feature_logits";
    if (check_widths(fn, C, c, K) != SGB_OK) return SGB_E_INVALID;
    if (P < 0) { set_error("%s: P = %d is negative", fn, P); return SGB_E_INVALID; }
    if (Kpad < K) { set_error("%s: Kpad = %d is less than K = %d", fn, Kpad, K); return SGB_E_INVALID; }
    if (P == 0) return SGB_OK;
    if (!features) { set_error("%s: null features", fn); return SGB_E_INVALID; }
    if (!weight) { set_error("%s: null weight", fn); return SGB_E_INVALID; }
    if (!text) { set_error("%s: null text", fn); return SGB_E_INVALID; }
    if (!out) { set_error("%s: null out", fn); return SGB_E_INVALID; }
    if (check_workspace(fn, workspace) != SGB_OK) return SGB_E_INVALID;
    cudaStream_t s = (cudaStream_t)stream;
    const DhTables t = tables(workspace, c, K);
    int rc = launch_prologue(C, c, K, 0, text, weight, bias, t, s);
    if (rc != SGB_OK) return rc;
    // without a bias beta is zero: leave it out, so the call is sgb_feature_logits on A bitwise
    return launch_feature_logits(P, c, K, Kpad, features, t.Ar, bias ? t.beta : nullptr, out, s);
}

}  // extern "C"
