// Feature-map distillation loss of a rendered (C, H, W) feature image against a 2D model's feature map of the same
// shape (fp16 or fp32), and its gradient, in the three forms of the reference's distill.py:111-124:
//
//   cosine   (1 / Nv) sum_{p valid} (1 - cos_p),  cos_p = x_p.y_p / (max(|x_p|, 1e-8) max(|y_p|, 1e-8))
//            (torch.nn.CosineSimilarity(eps=1e-8): each norm clamped separately; valid = y_p has a non-zero element)
//   l1       (1 / (N C)) sum |x - y|          (torch.nn.L1Loss)
//   l2       (1 / (N C)) sum (x - y)^2        (torch.nn.MSELoss)
//
// Each input is read once and the gradient written once.  l1 / l2 are elementwise over the N*C values (16-byte
// loads where the layout allows).  cosine needs three reductions over C per pixel (x.y, |x|^2, |y|^2) before any
// gradient element of that pixel can be written, and both images are planar with plane stride N: a CTA owns a
// block of PB pixels and stages their full C-long columns of render and target in shared memory (a TMA tensor copy
// of a (channels x PB) box, or plain loads when the layout does not meet the TMA rules), reduces per pixel and
// writes the gradient from the staged copy.  The normaliser 1/Nv is global, so a small pre-pass counts the valid
// pixels into loss[1] (a pixel's column is read only up to its first non-zero channel: about one plane on real
// feature maps) and the main kernel reads it from device memory in stream order.
//
// H100 80GB HBM3 at 700 W, 256 x 1080 x 1920, fp16 target (tools/time_feature_loss.py): count 0.08 ms + cosine
// kernel 1.94 ms; l1 / l2 kernel 1.85 ms (2.9 TB/s over the 5.3 GB that must move).
#include <algorithm>
#include <cstring>
#include <cuda_fp16.h>
#include <cub/cub.cuh>

#include "common.cuh"
#include "feature_loss.cuh"
#include "tma.cuh"

namespace sgb {
namespace {

constexpr int kFlThreads = 256;
constexpr int kFlMaxBox = 256;             // TMA box limit per dimension
constexpr size_t kFlStageTarget = 48 * 1024;  // staged bytes per CTA aimed at: four CTAs per SM

// loss[1] = number of pixels whose target column has a non-zero element (features_gt.norm(dim=-1) > 0).  Thread =
// one pixel.  Channel 0 decides almost every pixel of a real feature map; the rest of a column is read in groups of
// kCountGroup independent loads, so an all-zero column costs C / kCountGroup dependent memory round trips, not C.
constexpr int kCountGroup = 16;
template <typename T>
__global__ void __launch_bounds__(256) count_valid_pixels_kernel(int C, long long N, const T* __restrict__ y,
                                                                 double* __restrict__ valid) {
    __shared__ int wn[8];
    const long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    int nz = 0;
    if (p < N) {
        nz = to_f32(y[p]) != 0.f;
        for (int c0 = 1; !nz && c0 < C; c0 += kCountGroup) {
            float v[kCountGroup];
#pragma unroll
            for (int j = 0; j < kCountGroup; j++) v[j] = c0 + j < C ? to_f32(y[(size_t)(c0 + j) * N + p]) : 0.f;
#pragma unroll
            for (int j = 0; j < kCountGroup; j++) nz |= v[j] != 0.f;
        }
    }
    const int n = __reduce_add_sync(0xffffffffu, nz);
    if ((threadIdx.x & 31) == 0) wn[threadIdx.x >> 5] = n;
    __syncthreads();
    if (threadIdx.x == 0) {
        int t = 0;
        for (int w = 0; w < 8; w++) t += wn[w];
        if (t) atomicAdd(valid, (double)t);
    }
}

// Cosine loss: CTA = PB = 2^pb_log2 consecutive pixels.  Shared memory holds Xs [Cs][PB] fp32 and, 128-byte aligned
// after it, Ys [Cs][PB] of the target type, Cs = nbox * box_c >= C (rows past C arrive as zeros and are not read).
// Thread t reduces pixel t % PB over channels t / PB, t / PB + G, ... (G = 256 / PB); the G partial sums of a pixel
// are added in a fixed order, so the gradient is bit-reproducible.
template <typename T>
__global__ void __launch_bounds__(kFlThreads) feature_cosine_kernel(int C, long long N, int pb_log2, int box_c, int nbox,
                                                                    const float* __restrict__ render,
                                                                    const T* __restrict__ target, float* __restrict__ dL,
                                                                    double* __restrict__ loss,
                                                                    const __grid_constant__ CUtensorMap xmap,
                                                                    const __grid_constant__ CUtensorMap ymap, int use_tma) {
    extern __shared__ __align__(128) unsigned char fl_smem[];
    __shared__ uint64_t bar;
    __shared__ float red[3][kFlThreads];
    __shared__ int nzs[kFlThreads];
    __shared__ float coef[2][kFlThreads];
    __shared__ double wsum[kFlThreads / 32];
    const int PB = 1 << pb_log2, G = kFlThreads >> pb_log2;
    const int Cs = nbox * box_c;
    const size_t ys_off = ((size_t)Cs * PB * sizeof(float) + 127) & ~(size_t)127;
    float* Xs = reinterpret_cast<float*>(fl_smem);
    T* Ys = reinterpret_cast<T*>(fl_smem + ys_off);
    const int tid = threadIdx.x;
    const long long p0 = (long long)blockIdx.x * PB;

    if (use_tma) {
        if (tid == 0) {
            mbar_init(&bar, 1);
            mbar_fence_init();
        }
        __syncthreads();
        if (tid == 0) {
            mbar_arrive_expect_tx(&bar, (uint32_t)((size_t)Cs * PB * (sizeof(float) + sizeof(T))));
            for (int k = 0; k < nbox; k++) {
                tma_tile2d_g2s(Xs + (size_t)k * box_c * PB, &xmap, (int)p0, k * box_c, &bar);
                tma_tile2d_g2s(Ys + (size_t)k * box_c * PB, &ymap, (int)p0, k * box_c, &bar);
            }
        }
        mbar_wait(&bar, 0);
    } else {
        const int npx = (int)min((long long)PB, N - p0);
#pragma unroll 4
        for (int e = tid; e < C * PB; e += kFlThreads) {
            const int c = e >> pb_log2, p = e & (PB - 1);
            const size_t o = (size_t)c * N + p0 + p;
            Xs[e] = p < npx ? __ldg(render + o) : 0.f;
            Ys[e] = p < npx ? target[o] : T(0.f);
        }
        __syncthreads();
    }

    const int tp = tid & (PB - 1), g = tid >> pb_log2;
    float dot = 0.f, xx = 0.f, yy = 0.f;
    int nz = 0;
    for (int c = g; c < C; c += G) {
        const float x = Xs[c * PB + tp], y = to_f32(Ys[c * PB + tp]);
        dot = fmaf(x, y, dot);
        xx = fmaf(x, x, xx);
        yy = fmaf(y, y, yy);
        nz |= y != 0.f;
    }
    red[0][tid] = dot;
    red[1][tid] = xx;
    red[2][tid] = yy;
    nzs[tid] = nz;
    __syncthreads();

    double term = 0.0;
    if (tid < PB) {
        float d = 0.f, a2 = 0.f, b2 = 0.f;
        int any = 0;
        for (int k = 0; k < G; k++) {
            d += red[0][k * PB + tid];
            a2 += red[1][k * PB + tid];
            b2 += red[2][k * PB + tid];
            any |= nzs[k * PB + tid];
        }
        const double nv = loss[1];
        const float inv_nv = nv > 0.0 ? (float)(1.0 / nv) : 0.f;
        const bool valid = any && p0 + tid < N;
        const double t = cosine_rule(d, a2, b2, valid, inv_nv, coef[0][tid], coef[1][tid]);
        term = valid ? t : 0.0;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) term += __shfl_xor_sync(0xffffffffu, term, o);
    if ((tid & 31) == 0) wsum[tid >> 5] = term;
    __syncthreads();
    if (tid == 0) {
        double t = 0.0;
        for (int w = 0; w < kFlThreads / 32; w++) t += wsum[w];
        const double nv = loss[1];
        if (nv > 0.0 && t != 0.0) atomicAdd(loss, t / nv);
    }

    if (p0 + tp >= N) return;
    const float u = coef[0][tp], v = coef[1][tp];
    float* out = dL + p0 + tp;
    for (int c = g; c < C; c += G) out[(size_t)c * N] = fmaf(u, to_f32(Ys[c * PB + tp]), v * Xs[c * PB + tp]);
}

// l1 / l2 over the M = N*C values.  VEC: render, target and dL start 16-/8-byte aligned, so the first M - M % 4
// values go as 4-wide loads.
template <typename T, int LOSS, bool VEC>
__global__ void __launch_bounds__(256) feature_elementwise_kernel(long long M, long long N, const float* __restrict__ x,
                                                                  const T* __restrict__ y, float* __restrict__ dL,
                                                                  double* __restrict__ loss) {
    const double inv_m = 1.0 / (double)M;
    const float gs = (float)((LOSS == SGB_FEATLOSS_L2 ? 2.0 : 1.0) * inv_m);
    const long long t0 = (long long)blockIdx.x * blockDim.x + threadIdx.x, stride = (long long)gridDim.x * blockDim.x;
    double acc = 0.0;
    long long tail = 0;
    if (VEC) {
        const long long M4 = M >> 2;
        for (long long i = t0; i < M4; i += stride) {
            const Quad a = load4(x + 4 * i), b = load4(y + 4 * i);
            float g[4], s = 0.f;
#pragma unroll
            for (int j = 0; j < 4; j++) s += elementwise_rule<LOSS>(a.v[j] - b.v[j], gs, g[j]);
            *reinterpret_cast<float4*>(dL + 4 * i) = make_float4(g[0], g[1], g[2], g[3]);
            acc += (double)s;
        }
        tail = M4 << 2;
    }
    for (long long i = tail + t0; i < M; i += stride) {
        float g;
        acc += (double)elementwise_rule<LOSS>(__ldg(x + i) - to_f32(y[i]), gs, g);
        dL[i] = g;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    __shared__ double wsum[8];
    if ((threadIdx.x & 31) == 0) wsum[threadIdx.x >> 5] = acc;
    __syncthreads();
    if (threadIdx.x == 0) {
        double t = 0.0;
        for (int w = 0; w < 8; w++) t += wsum[w];
        atomicAdd(loss, t * inv_m);
        if (blockIdx.x == 0) loss[1] = (double)N;  // every pixel takes part in the mean
    }
}

// Target of the cosine kernel as a (pixel, channel) tensor with a (PB, box_c) box.  False when the layout does not
// meet the TMA rules (plane pitch and base multiples of 16 bytes, coordinates in int32) or the driver entry point is
// missing; the kernel then stages with plain loads.
bool encode_plane_map(CUtensorMap* map, const void* base, CUtensorMapDataType type, size_t es, int C, long long N,
                      int PB, int box_c) {
    memset(map, 0, sizeof(*map));
    if (((size_t)N * es) % 16 != 0 || (reinterpret_cast<uintptr_t>(base) & 15) != 0 || N > 0x7fffffffll) return false;
    const cuuint64_t dims[2] = {(cuuint64_t)N, (cuuint64_t)C};
    const cuuint64_t strides[1] = {(cuuint64_t)N * es};
    const cuuint32_t box[2] = {(cuuint32_t)PB, (cuuint32_t)box_c};
    return encode_tiled_map(map, type, 2, base, dims, strides, box, CU_TENSOR_MAP_SWIZZLE_NONE);
}

template <typename T>
int launch_cosine(int C, long long N, const float* render, const T* target, float* dL, double* loss, cudaStream_t s) {
    const int rc = count_valid_pixels<T>(C, N, target, loss + 1, s);
    if (rc != SGB_OK) return rc;
    // channels in nbox TMA boxes of box_c rows; a box after the first starts 128-byte aligned in shared memory
    const int nbox = (C + kFlMaxBox - 1) / kFlMaxBox;
    const int box_c = nbox == 1 ? C : ((C + nbox - 1) / nbox + 15) & ~15;
    const size_t row = sizeof(float) + sizeof(T);
    // the widest pixel block (a power of two, 16-byte box rows, at least one 32-byte sector of target per row) whose
    // staged columns fit the per-CTA target
    const int pb_min = sizeof(T) == 2 ? 16 : 8;
    int pb_log2 = 8;
    while ((1 << pb_log2) > pb_min && (size_t)nbox * box_c * (1 << pb_log2) * row > kFlStageTarget) pb_log2--;
    const int PB = 1 << pb_log2;
    const size_t xs = ((size_t)nbox * box_c * PB * sizeof(float) + 127) & ~(size_t)127;
    const size_t smem = xs + (size_t)nbox * box_c * PB * sizeof(T);
    constexpr size_t kMaxSmem = 96 * 1024 + 128;  // C = 1024, fp16: 16 px x 1024 x 6 B
    static DeviceOnce attr_set;
    if (attr_set.first_use_on_device())
        SGB_CUDA(cudaFuncSetAttribute(feature_cosine_kernel<T>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kMaxSmem));
    CUtensorMap xmap, ymap;
    const CUtensorMapDataType ytype = sizeof(T) == 2 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32;
    const int use_tma = encode_plane_map(&xmap, render, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, sizeof(float), C, N, PB, box_c) &&
                        encode_plane_map(&ymap, target, ytype, sizeof(T), C, N, PB, box_c);
    const unsigned blocks = (unsigned)((N + PB - 1) / PB);
    feature_cosine_kernel<T><<<blocks, kFlThreads, smem, s>>>(C, N, pb_log2, box_c, nbox, render, target, dL, loss, xmap,
                                                             ymap, use_tma);
    SGB_LAUNCH_CHECK("feature_cosine_kernel", 0, s);
    return SGB_OK;
}

template <typename T, int LOSS>
int launch_elementwise(int C, long long N, const float* render, const T* target, float* dL, double* loss, cudaStream_t s) {
    const long long M = N * C;
    const bool vec = (reinterpret_cast<uintptr_t>(render) & 15) == 0 && (reinterpret_cast<uintptr_t>(dL) & 15) == 0 &&
                     (reinterpret_cast<uintptr_t>(target) & (4 * sizeof(T) - 1)) == 0;
    const long long work = vec ? M / 4 : M;
    const unsigned blocks = (unsigned)std::max(1ll, std::min((work + 255) / 256, (long long)kNumSMs * 8));
    if (vec) feature_elementwise_kernel<T, LOSS, true><<<blocks, 256, 0, s>>>(M, N, render, target, dL, loss);
    else feature_elementwise_kernel<T, LOSS, false><<<blocks, 256, 0, s>>>(M, N, render, target, dL, loss);
    SGB_LAUNCH_CHECK("feature_elementwise_kernel", 0, s);
    return SGB_OK;
}

template <typename T>
int launch_feature_loss(int loss_type, int C, long long N, const float* render, const T* target, float* dL,
                        double* loss, cudaStream_t s) {
    if (loss_type == SGB_FEATLOSS_COSINE) return launch_cosine<T>(C, N, render, target, dL, loss, s);
    if (loss_type == SGB_FEATLOSS_L1) return launch_elementwise<T, SGB_FEATLOSS_L1>(C, N, render, target, dL, loss, s);
    return launch_elementwise<T, SGB_FEATLOSS_L2>(C, N, render, target, dL, loss, s);
}

// ---- Masked-row loss of a (M, F) row-major network output (MinkUNet's .F) against one (K, C) target row per masked
// output row, on the column block [h0, h0 + C) (distill.py:111-124 after `output = model_3d(sinput).F[mask]`).
// Passes: flags -> cub::DeviceScan (rank of each masked row among the masked rows) -> [cosine: count of non-zero target
// rows] -> one warp per output row, which reads its slice and target row once and writes its whole gradient row
// once -> one CTA that adds the per-CTA partial sums in a fixed order.  The only atomic is the integer row count,
// so every output is bitwise reproducible.
constexpr int kVlRows = 8;                   // warps (= output rows) per CTA
constexpr int kVlThreads = 32 * kVlRows;
constexpr int kVlPerLane = kFeatMaxC / 32;

struct VlWorkspace {
    unsigned long long* nv;   // number of target rows with a non-zero element (cosine)
    int* flags;               // [M] mask[i] != 0
    int* rank;                // [M] exclusive scan of flags
    double* partial;          // [ceil(M / kVlRows)] per-CTA loss sums
    void* tmp;
    size_t tmp_bytes;
    size_t bytes;
};

int carve_vl_workspace(long long M, void* base, VlWorkspace& w) {
    size_t scan_tmp = 0;
    SGB_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, scan_tmp, (int*)nullptr, (int*)nullptr, (int)M));
    char* p = (char*)base;
    size_t off = 0;
    w.nv = (unsigned long long*)(p + off); off += align_up(sizeof(unsigned long long));
    w.flags = (int*)(p + off); off += align_up(sizeof(int) * (size_t)M);
    w.rank = (int*)(p + off); off += align_up(sizeof(int) * (size_t)M);
    w.partial = (double*)(p + off); off += align_up(sizeof(double) * (size_t)((M + kVlRows - 1) / kVlRows));
    w.tmp = p + off;
    w.tmp_bytes = scan_tmp;
    off += align_up(scan_tmp);
    w.bytes = off;
    return SGB_OK;
}

__global__ void __launch_bounds__(256) vl_flags_kernel(long long M, const uint8_t* __restrict__ mask,
                                                       int* __restrict__ flags, unsigned long long* nv) {
    const long long i = (long long)blockIdx.x * 256 + threadIdx.x;
    if (i == 0) *nv = 0;
    if (i < M) flags[i] = mask[i] != 0;
}

// nv += number of target rows with a non-zero element (features_gt.norm(dim=-1) > 0).  Warp = one row.
template <typename T>
__global__ void __launch_bounds__(kVlThreads) vl_count_kernel(long long K, int C, const T* __restrict__ y,
                                                              unsigned long long* nv) {
    __shared__ int wn[kVlRows];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const long long k = (long long)blockIdx.x * kVlRows + warp;
    int nz = 0;
    if (k < K)
        for (int c = lane; c < C && !nz; c += 32) nz = to_f32(y[k * C + c]) != 0.f;
    nz = __any_sync(0xffffffffu, nz);
    if (lane == 0) wn[warp] = nz;
    __syncthreads();
    if (threadIdx.x == 0) {
        int t = 0;
        for (int j = 0; j < kVlRows; j++) t += wn[j];
        if (t) atomicAdd(nv, (unsigned long long)t);
    }
}

// What one vl_loss_kernel launch writes.  kVlFused: the per-CTA loss partials and the fp32 gradient
// (sgb_voxel_feature_loss).  kVlForward: the partials only.  kVlBackward: only the gradient, each element
// from_f32(*dloss * g) with g the fp32 value kVlFused writes; the scale multiplies the finished g, so a power-of-two
// scale gives exactly the rounded, scaled kVlFused gradient.
enum VlPass { kVlFused, kVlForward, kVlBackward };

// TX: the output's element type (float, __half or __nv_bfloat16), which is also the gradient's.  Half values widen
// to fp32 exactly, so every pass sees the fp32 values of x and runs the same per-lane sums and butterflies.
template <typename TX, typename T, int LOSS, int PASS>
__global__ void __launch_bounds__(kVlThreads) vl_loss_kernel(long long M, int F, const TX* __restrict__ x,
                                                             long long K, int C, int h0, const T* __restrict__ y,
                                                             const int* __restrict__ flags,
                                                             const int* __restrict__ rank,
                                                             const unsigned long long* __restrict__ nv_count,
                                                             const double* __restrict__ dloss,
                                                             TX* __restrict__ grad, double* __restrict__ partial) {
    __shared__ double wsum[kVlRows];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const long long i = (long long)blockIdx.x * kVlRows + warp;
    double term = 0.0;
    if (i < M) {
        const TX* xr = x + i * F;
        TX* gr = grad + i * F;
        const float scale = PASS == kVlBackward ? (float)*dloss : 1.f;
        // element c of the head's gradient slice
        auto store = [&](int c, float g) {
            if (PASS == kVlFused) gr[h0 + c] = g;
            if (PASS == kVlBackward) gr[h0 + c] = from_f32<TX>(scale * g);
        };
        if (PASS != kVlForward) {
            for (int c = lane; c < h0; c += 32) gr[c] = from_f32<TX>(0.f);
            for (int c = h0 + C + lane; c < F; c += 32) gr[c] = from_f32<TX>(0.f);
        }
        const long long r = flags[i] ? (long long)rank[i] : -1;
        if (r < 0 || r >= K) {
            if (PASS != kVlForward)
                for (int c = lane; c < C; c += 32) gr[h0 + c] = from_f32<TX>(0.f);
        } else {
            const T* yr = y + r * C;
            float xv[kVlPerLane], yv[kVlPerLane];
#pragma unroll
            for (int j = 0; j < kVlPerLane; j++) {
                const int c = lane + 32 * j;
                xv[j] = c < C ? load_f32(xr + h0 + c) : 0.f;
                yv[j] = c < C ? to_f32(yr[c]) : 0.f;
            }
            if (LOSS == SGB_FEATLOSS_COSINE) {
                float dot = 0.f, xx = 0.f, yy = 0.f;
                int nz = 0;
#pragma unroll
                for (int j = 0; j < kVlPerLane; j++) {
                    dot = fmaf(xv[j], yv[j], dot);
                    xx = fmaf(xv[j], xv[j], xx);
                    yy = fmaf(yv[j], yv[j], yy);
                    nz |= yv[j] != 0.f;
                }
                // xor butterflies: every lane ends with the same, fixed-order sums
#pragma unroll
                for (int o = 16; o > 0; o >>= 1) {
                    dot += __shfl_xor_sync(0xffffffffu, dot, o);
                    xx += __shfl_xor_sync(0xffffffffu, xx, o);
                    yy += __shfl_xor_sync(0xffffffffu, yy, o);
                }
                const bool valid = __any_sync(0xffffffffu, nz);
                const double nv = (double)*nv_count;
                const float inv_nv = nv > 0.0 ? (float)(1.0 / nv) : 0.f;
                float u, v;
                const double t = cosine_rule(dot, xx, yy, valid, inv_nv, u, v);
#pragma unroll
                for (int j = 0; j < kVlPerLane; j++) {
                    const int c = lane + 32 * j;
                    if (c < C) store(c, fmaf(u, yv[j], v * xv[j]));
                }
                term = valid && lane == 0 ? t : 0.0;
            } else {
                const float gs = (float)((LOSS == SGB_FEATLOSS_L2 ? 2.0 : 1.0) / ((double)K * (double)C));
                double acc = 0.0;
#pragma unroll
                for (int j = 0; j < kVlPerLane; j++) {
                    const int c = lane + 32 * j;
                    if (c < C) {
                        float g;
                        const float t = elementwise_rule<LOSS>(xv[j] - yv[j], gs, g);
                        store(c, g);
                        acc += (double)t;
                    }
                }
#pragma unroll
                for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
                term = lane == 0 ? acc : 0.0;
            }
        }
    }
    if (PASS == kVlBackward) return;
    if (lane == 0) wsum[warp] = term;
    __syncthreads();
    if (threadIdx.x == 0) {
        double t = 0.0;
        for (int j = 0; j < kVlRows; j++) t += wsum[j];
        partial[blockIdx.x] = t;
    }
}

// loss[0] = sum of the partials / the count, loss[1] = the count (non-zero target rows for cosine, K for l1 / l2;
// the l1 / l2 mean is over K * C).  A mask whose row count is not K makes both NaN.
__global__ void __launch_bounds__(256) vl_finish_kernel(long long nb, const double* __restrict__ partial, long long M,
                                                        const int* __restrict__ flags, const int* __restrict__ rank,
                                                        long long K, int C, int loss_type,
                                                        const unsigned long long* __restrict__ nv, double* loss) {
    __shared__ double s[256];
    double t = 0.0;
    for (long long j = threadIdx.x; j < nb; j += 256) t += partial[j];
    s[threadIdx.x] = t;
    __syncthreads();
    for (int o = 128; o > 0; o >>= 1) {
        if (threadIdx.x < o) s[threadIdx.x] += s[threadIdx.x + o];
        __syncthreads();
    }
    if (threadIdx.x != 0) return;
    const long long masked = (long long)rank[M - 1] + flags[M - 1];
    if (masked != K) {
        loss[0] = loss[1] = __longlong_as_double(0x7ff8000000000000ll);
        return;
    }
    if (loss_type == SGB_FEATLOSS_COSINE) {
        const double n = (double)*nv;
        loss[0] = n > 0.0 ? s[0] / n : 0.0;
        loss[1] = n;
    } else {
        loss[0] = K > 0 ? s[0] * (1.0 / ((double)K * (double)C)) : 0.0;
        loss[1] = (double)K;
    }
}

// One call's operands, untyped until the dispatch below picks TX and T.  grad is null for kVlForward, dloss is
// non-null for kVlBackward only, and loss and mask are not read by kVlBackward.
struct VlCall {
    long long M;
    int F;
    const void* x;
    const uint8_t* mask;
    long long K;
    int C, h0;
    const void* y;
    const double* dloss;
    void* grad;
    VlWorkspace w;
    double* loss;
    cudaStream_t s;
};

// kVlFused and kVlForward: flags, rank and (cosine) Nv into the workspace, the rows, then loss[0..1].  kVlBackward:
// the rows alone, on the flags, rank and Nv a kVlForward pass on the same mask and target left in the workspace.
template <int PASS, typename TX, typename T, int LOSS>
int launch_voxel_loss(const VlCall& a) {
    const VlWorkspace& w = a.w;
    const T* y = (const T*)a.y;
    cudaStream_t s = a.s;
    if (PASS != kVlBackward) {
        vl_flags_kernel<<<(unsigned)((a.M + 255) / 256), 256, 0, s>>>(a.M, a.mask, w.flags, w.nv);
        SGB_LAUNCH_CHECK("vl_flags_kernel", 0, s);
        size_t tmp_bytes = w.tmp_bytes;
        SGB_CUDA(cub::DeviceScan::ExclusiveSum(w.tmp, tmp_bytes, w.flags, w.rank, (int)a.M, s));
        if (LOSS == SGB_FEATLOSS_COSINE && a.K > 0) {
            vl_count_kernel<T><<<(unsigned)((a.K + kVlRows - 1) / kVlRows), kVlThreads, 0, s>>>(a.K, a.C, y, w.nv);
            SGB_LAUNCH_CHECK("vl_count_kernel", 0, s);
        }
    }
    const long long nb = (a.M + kVlRows - 1) / kVlRows;
    vl_loss_kernel<TX, T, LOSS, PASS><<<(unsigned)nb, kVlThreads, 0, s>>>(
        a.M, a.F, (const TX*)a.x, a.K, a.C, a.h0, y, w.flags, w.rank, w.nv, a.dloss, (TX*)a.grad, w.partial);
    SGB_LAUNCH_CHECK("vl_loss_kernel", 0, s);
    if (PASS != kVlBackward) {
        vl_finish_kernel<<<1, 256, 0, s>>>(nb, w.partial, a.M, w.flags, w.rank, a.K, a.C, LOSS, w.nv, a.loss);
        SGB_LAUNCH_CHECK("vl_finish_kernel", 0, s);
    }
    return SGB_OK;
}

template <int PASS, typename TX, typename T>
int launch_voxel_loss(int loss_type, const VlCall& a) {
    if (loss_type == SGB_FEATLOSS_COSINE) return launch_voxel_loss<PASS, TX, T, SGB_FEATLOSS_COSINE>(a);
    if (loss_type == SGB_FEATLOSS_L1) return launch_voxel_loss<PASS, TX, T, SGB_FEATLOSS_L1>(a);
    return launch_voxel_loss<PASS, TX, T, SGB_FEATLOSS_L2>(a);
}

template <int PASS, typename TX>
int launch_voxel_loss(int target_dtype, int loss_type, const VlCall& a) {
    if (target_dtype == SGB_FEAT_F16) return launch_voxel_loss<PASS, TX, __half>(loss_type, a);
    return launch_voxel_loss<PASS, TX, float>(loss_type, a);
}

template <int PASS>
int launch_voxel_loss(int output_dtype, int target_dtype, int loss_type, const VlCall& a) {
    if (output_dtype == SGB_FEAT_F16) return launch_voxel_loss<PASS, __half>(target_dtype, loss_type, a);
    if (output_dtype == SGB_FEAT_BF16) return launch_voxel_loss<PASS, __nv_bfloat16>(target_dtype, loss_type, a);
    return launch_voxel_loss<PASS, float>(target_dtype, loss_type, a);
}

bool vl_m_ok(int64_t M) { return M >= 0 && M <= INT32_MAX; }

// The argument rules every voxel-row entry point shares: M, C, target_dtype, loss_type, head and K.
int check_voxel_loss_args(const char* fn, int64_t M, int32_t F, int64_t K, int32_t C, int32_t head,
                          int32_t target_dtype, int32_t loss_type) {
    if (!vl_m_ok(M)) { set_error("%s: M = %lld outside [0, %d]", fn, (long long)M, INT32_MAX); return SGB_E_INVALID; }
    if (check_feature_loss_args(fn, C, target_dtype, loss_type) != SGB_OK) return SGB_E_INVALID;
    if (head < 0 || (int64_t)head * C + C > F) {
        set_error("%s: head %d of width %d does not fit in F = %d columns", fn, head, C, F);
        return SGB_E_INVALID;
    }
    if (K < 0 || K > M) { set_error("%s: K = %lld target rows outside [0, M = %lld]", fn, (long long)K, (long long)M); return SGB_E_INVALID; }
    return SGB_OK;
}

// The output dtype's element size, or 0 (error set) for an unknown code.
size_t vl_output_size(const char* fn, int32_t output_dtype) {
    if (output_dtype == SGB_FEAT_F32) return 4;
    if (output_dtype == SGB_FEAT_F16 || output_dtype == SGB_FEAT_BF16) return 2;
    set_error("%s: unknown output_dtype %d (SGB_FEAT_F32, SGB_FEAT_F16 or SGB_FEAT_BF16)", fn, output_dtype);
    return 0;
}

int check_vl_alignment(const char* fn, const char* name, const void* p, size_t es) {
    if (reinterpret_cast<uintptr_t>(p) % es) {
        set_error("%s: %s is not %d-byte aligned for its dtype", fn, name, (int)es);
        return SGB_E_INVALID;
    }
    return SGB_OK;
}

}  // namespace

template <typename T>
int count_valid_pixels(int C, long long N, const T* target, double* valid, cudaStream_t s) {
    count_valid_pixels_kernel<T><<<(unsigned)((N + 255) / 256), 256, 0, s>>>(C, N, target, valid);
    SGB_LAUNCH_CHECK("count_valid_pixels_kernel", 0, s);
    return SGB_OK;
}
template int count_valid_pixels<float>(int, long long, const float*, double*, cudaStream_t);
template int count_valid_pixels<__half>(int, long long, const __half*, double*, cudaStream_t);

int check_feature_loss_args(const char* fn, int C, int target_dtype, int loss_type) {
    if (C <= 0 || C > kFeatMaxC) { set_error("%s: C = %d outside [1, %d]", fn, C, kFeatMaxC); return SGB_E_INVALID; }
    if (target_dtype != SGB_FEAT_F16 && target_dtype != SGB_FEAT_F32) {
        set_error("%s: unknown target_dtype %d (SGB_FEAT_F16 or SGB_FEAT_F32)", fn, target_dtype);
        return SGB_E_INVALID;
    }
    if (loss_type != SGB_FEATLOSS_COSINE && loss_type != SGB_FEATLOSS_L1 && loss_type != SGB_FEATLOSS_L2) {
        set_error("%s: unknown loss_type %d (SGB_FEATLOSS_COSINE, _L1 or _L2)", fn, loss_type);
        return SGB_E_INVALID;
    }
    return SGB_OK;
}

}  // namespace sgb

using namespace sgb;

extern "C" {

int sgb_feature_map_loss(int32_t C, int64_t N, const float* render, const void* target, int32_t target_dtype,
                         int32_t loss_type, float* dL_drender, double* loss, void* stream) {
    static const char* fn = "sgb_feature_map_loss";
    if (check_feature_loss_args(fn, C, target_dtype, loss_type) != SGB_OK) return SGB_E_INVALID;
    if (N < 0) { set_error("%s: N = %lld is negative", fn, (long long)N); return SGB_E_INVALID; }
    if (!loss) { set_error("%s: null loss", fn); return SGB_E_INVALID; }
    if (N > 0 && !render) { set_error("%s: null render", fn); return SGB_E_INVALID; }
    if (N > 0 && !target) { set_error("%s: null target", fn); return SGB_E_INVALID; }
    if (N > 0 && !dL_drender) { set_error("%s: null dL_drender", fn); return SGB_E_INVALID; }
    cudaStream_t s = (cudaStream_t)stream;
    SGB_CUDA(cudaMemsetAsync(loss, 0, 2 * sizeof(double), s));
    if (N == 0) return SGB_OK;
    if (target_dtype == SGB_FEAT_F16)
        return launch_feature_loss<__half>(loss_type, C, (long long)N, render, (const __half*)target, dL_drender, loss, s);
    return launch_feature_loss<float>(loss_type, C, (long long)N, render, (const float*)target, dL_drender, loss, s);
}

size_t sgb_voxel_feature_loss_workspace_bytes(int64_t M) {
    if (!vl_m_ok(M)) return 0;
    VlWorkspace w;
    return carve_vl_workspace((long long)M, nullptr, w) == SGB_OK ? w.bytes : 0;
}

int sgb_voxel_feature_loss(int64_t M, int32_t F, const float* output, const uint8_t* mask, int64_t K, int32_t C,
                           int32_t head, const void* target, int32_t target_dtype, int32_t loss_type, float* grad,
                           void* workspace, double* loss, void* stream) {
    static const char* fn = "sgb_voxel_feature_loss";
    if (check_voxel_loss_args(fn, M, F, K, C, head, target_dtype, loss_type) != SGB_OK) return SGB_E_INVALID;
    if (!loss) { set_error("%s: null loss", fn); return SGB_E_INVALID; }
    if (M > 0 && (!output || !mask || !grad)) { set_error("%s: null output / mask / grad", fn); return SGB_E_INVALID; }
    if (K > 0 && !target) { set_error("%s: null target", fn); return SGB_E_INVALID; }
    if (M > 0 && !workspace) { set_error("%s: null workspace", fn); return SGB_E_INVALID; }
    if (reinterpret_cast<uintptr_t>(workspace) % 16) { set_error("%s: workspace is not 16-byte aligned", fn); return SGB_E_INVALID; }
    cudaStream_t s = (cudaStream_t)stream;
    if (M == 0) {
        SGB_CUDA(cudaMemsetAsync(loss, 0, 2 * sizeof(double), s));
        return SGB_OK;
    }
    VlCall a{(long long)M, F, output, mask, (long long)K, C, head * C, target, nullptr, grad, {}, loss, s};
    const int rc = carve_vl_workspace((long long)M, workspace, a.w);
    if (rc) return rc;
    return launch_voxel_loss<kVlFused, float>(target_dtype, loss_type, a);
}

int sgb_voxel_feature_loss_forward(int64_t M, int32_t F, const void* output, int32_t output_dtype,
                                   const uint8_t* mask, int64_t K, int32_t C, int32_t head, const void* target,
                                   int32_t target_dtype, int32_t loss_type, void* workspace, double* loss,
                                   void* stream) {
    static const char* fn = "sgb_voxel_feature_loss_forward";
    if (check_voxel_loss_args(fn, M, F, K, C, head, target_dtype, loss_type) != SGB_OK) return SGB_E_INVALID;
    const size_t es = vl_output_size(fn, output_dtype);
    if (!es) return SGB_E_INVALID;
    if (!loss) { set_error("%s: null loss", fn); return SGB_E_INVALID; }
    if (M > 0 && (!output || !mask)) { set_error("%s: null output / mask", fn); return SGB_E_INVALID; }
    if (K > 0 && !target) { set_error("%s: null target", fn); return SGB_E_INVALID; }
    if (M > 0 && !workspace) { set_error("%s: null workspace", fn); return SGB_E_INVALID; }
    if (reinterpret_cast<uintptr_t>(workspace) % 16) { set_error("%s: workspace is not 16-byte aligned", fn); return SGB_E_INVALID; }
    if (check_vl_alignment(fn, "output", output, es) != SGB_OK) return SGB_E_INVALID;
    cudaStream_t s = (cudaStream_t)stream;
    if (M == 0) {
        SGB_CUDA(cudaMemsetAsync(loss, 0, 2 * sizeof(double), s));
        return SGB_OK;
    }
    VlCall a{(long long)M, F, output, mask, (long long)K, C, head * C, target, nullptr, nullptr, {}, loss, s};
    const int rc = carve_vl_workspace((long long)M, workspace, a.w);
    if (rc) return rc;
    return launch_voxel_loss<kVlForward>(output_dtype, target_dtype, loss_type, a);
}

int sgb_voxel_feature_loss_backward(int64_t M, int32_t F, const void* output, int32_t output_dtype, int64_t K,
                                    int32_t C, int32_t head, const void* target, int32_t target_dtype,
                                    int32_t loss_type, const void* workspace, const double* dloss, void* grad,
                                    void* stream) {
    static const char* fn = "sgb_voxel_feature_loss_backward";
    if (check_voxel_loss_args(fn, M, F, K, C, head, target_dtype, loss_type) != SGB_OK) return SGB_E_INVALID;
    const size_t es = vl_output_size(fn, output_dtype);
    if (!es) return SGB_E_INVALID;
    if (!dloss) { set_error("%s: null dloss", fn); return SGB_E_INVALID; }
    if (M > 0 && (!output || !grad)) { set_error("%s: null output / grad", fn); return SGB_E_INVALID; }
    if (K > 0 && !target) { set_error("%s: null target", fn); return SGB_E_INVALID; }
    if (M > 0 && !workspace) { set_error("%s: null workspace", fn); return SGB_E_INVALID; }
    if (reinterpret_cast<uintptr_t>(workspace) % 16) { set_error("%s: workspace is not 16-byte aligned", fn); return SGB_E_INVALID; }
    if (check_vl_alignment(fn, "output", output, es) != SGB_OK) return SGB_E_INVALID;
    if (check_vl_alignment(fn, "grad", grad, es) != SGB_OK) return SGB_E_INVALID;
    if (M == 0) return SGB_OK;
    VlCall a{(long long)M, F, output, nullptr, (long long)K, C, head * C, target, dloss, grad, {}, nullptr,
             (cudaStream_t)stream};
    // the carve is a pure function of M: it finds what the forward pass left where that pass put it
    const int rc = carve_vl_workspace((long long)M, const_cast<void*>(workspace), a.w);
    if (rc) return rc;
    return launch_voxel_loss<kVlBackward>(output_dtype, target_dtype, loss_type, a);
}

}  // extern "C"
