// Products of the sparse 3D convolution on fp16 / bf16 features, on tensor cores, over the same kernel maps and with
// the same structure as the fp32 products of sparse_conv.cu:
//
//   forward        out[o]  = sum_d x[i_d(o)] W_d           x, W, out in the half type
//   input grad     dx[i]   = sum_d dy[o_d(i)] W_d^T        dy, W, dx in the half type
//   weight grad    dW_d    = sum_pairs x[src]^T dy[dst]    x, dy in the half type, dW in fp32
//
// Forward and input gradient: one gather-GEMM-scatter launch per non-empty offset, in offset order, each adding its
// product into a zeroed fp32 scratch (an offset's pairs are one-to-one: no atomics).  One pass then rounds the scratch
// to the half type, so every output element is rounded once, not once per offset.
//
// Weight gradient: kChunk-pair chunks write fp32 partials (accumulated per kInnerH-pair block, then over the blocks),
// and the reduction of sparse_conv.cu adds each offset's partials in chunk order.  dW stays fp32: the kernel parameter
// it updates is fp32.
//
// Products: mma.sync m16n8k16 with fp32 accumulation.  Half x half products are exact in fp32, so only the fp32
// accumulation rounds.  Tiles: 64 x 64 per CTA of 4 warps (32 x 32 each), 32-deep shared operands fed by ldmatrix and
// double-buffered.  Rows whose width in elements is a multiple of 8 (16 bytes) are gathered with 16-byte cp.async;
// other widths (and unaligned bases) take a staging path that loads each element on its own.
#include <algorithm>

#include <cuda_bf16.h>

#include "sparse_conv.cuh"

namespace sgb {

namespace {

constexpr int kHM = 64, kHN = 64, kHK = 32, kHThreads = 128;
constexpr int kPad = 8;          // elements of padding per shared row: 16-byte aligned, conflict-free ldmatrix rows
constexpr int kInnerH = 128;     // pairs per inner accumulation block of the weight gradient

__device__ __forceinline__ uint32_t smem_addr(const void* p) {
    return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

// 16 bytes global -> shared; zero-filled when !valid (src is then not read).
__device__ __forceinline__ void cp_async16(void* dst, const void* src, bool valid) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(smem_addr(dst)), "l"(src),
                 "r"(valid ? 16 : 0)
                 : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
__device__ __forceinline__ void cp_async_wait_one() { asm volatile("cp.async.wait_group 1;" ::: "memory"); }

__device__ __forceinline__ void ldmatrix_x4(uint32_t r[4], const void* p) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];"
                 : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3])
                 : "r"(smem_addr(p)));
}
__device__ __forceinline__ void ldmatrix_x4_trans(uint32_t r[4], const void* p) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0, %1, %2, %3}, [%4];"
                 : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3])
                 : "r"(smem_addr(p)));
}

// c += a b on one m16n8k16 tile, fp32 accumulation.
__device__ __forceinline__ void mma(float c[4], const uint32_t a[4], const uint32_t b[2], __half) {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, "
                 "{%0, %1, %2, %3};"
                 : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
}
__device__ __forceinline__ void mma(float c[4], const uint32_t a[4], const uint32_t b[2], __nv_bfloat16) {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, "
                 "{%0, %1, %2, %3};"
                 : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
}

__device__ __forceinline__ void round_to(float v, __half& o) { o = __float2half_rn(v); }
__device__ __forceinline__ void round_to(float v, __nv_bfloat16& o) { o = __float2bfloat16_rn(v); }

// B fragments of n8 tiles j and j + 1 at depth ks.  kNK: shared B is [n][k] (ldmatrix); otherwise [k][n]
// (ldmatrix.trans).
template <bool kNK, int kRow>
__device__ __forceinline__ void load_b(uint32_t b[4][2], const __half* Bs, int j, int n, int ks, int lane) {
    uint32_t r[4];
    if (kNK)
        ldmatrix_x4(r, Bs + (n + (lane % 8) + (lane / 16) * 8) * kRow + ks + ((lane / 8) % 2) * 8);
    else
        ldmatrix_x4_trans(r, Bs + (ks + (lane % 8) + ((lane / 8) % 2) * 8) * kRow + n + (lane / 16) * 8);
    b[j][0] = r[0], b[j][1] = r[1], b[j + 1][0] = r[2], b[j + 1][1] = r[3];
}

// Y[dst(p)] += X[src(p)] B (Y fp32) for the n pairs at `pairs`, where B(k, n) = kTrans ? W[n * Kd + k] : W[k * Nd + n].
// Kd: columns of X (reduction depth), Nd: columns of Y.  kVec: Kd and Nd are multiples of 8 and X, W 16-byte aligned.
template <typename T, bool kTrans, bool kVec>
__global__ void __launch_bounds__(kHThreads) sparse_gather_mma_kernel(const int2* __restrict__ pairs, long long n,
                                                                      int src_side, const T* __restrict__ X, int Kd,
                                                                      const T* __restrict__ W, int Nd,
                                                                      float* __restrict__ Y) {
    constexpr int kARow = kHK + kPad, kBRow = (kTrans ? kHK : kHN) + kPad, kBRows = kTrans ? kHN : kHK;
    __shared__ __align__(16) T As[2][kHM * kARow];      // [pair][k]
    __shared__ __align__(16) T Bs[2][kBRows * kBRow];   // [n][k] when kTrans, else [k][n]
    __shared__ int src[kHM], dst[kHM];
    const int tid = threadIdx.x, warp = tid / 32, lane = tid % 32;
    const long long m0 = (long long)blockIdx.x * kHM;
    const int n0 = blockIdx.y * kHN;
    if (tid < kHM) {
        const long long p = m0 + tid;
        const int2 pr = p < n ? pairs[p] : make_int2(-1, -1);
        src[tid] = src_side ? pr.y : pr.x;
        dst[tid] = src_side ? pr.x : pr.y;
    }
    __syncthreads();

    auto load = [&](int st, int k0) {
        T* as = As[st];
        T* bs = Bs[st];
        if constexpr (kVec) {
#pragma unroll
            for (int u = 0; u < 2; u++) {
                const int c = tid + u * kHThreads;
                const int r = c / 4, kc = (c % 4) * 8, s = src[r], k = k0 + kc;
                const bool ok = s >= 0 && k < Kd;
                cp_async16(as + r * kARow + kc, ok ? X + (long long)s * Kd + k : X, ok);
                if constexpr (kTrans) {           // 64 rows n x 4 runs of k
                    const int nn = n0 + r;
                    const bool okb = nn < Nd && k < Kd;
                    cp_async16(bs + r * kBRow + kc, okb ? W + (long long)nn * Kd + k : W, okb);
                } else {                          // 32 rows k x 8 runs of n
                    const int rk = c / 8, nc = (c % 8) * 8, kk = k0 + rk, nn = n0 + nc;
                    const bool okb = kk < Kd && nn < Nd;
                    cp_async16(bs + rk * kBRow + nc, okb ? W + (long long)kk * Nd + nn : W, okb);
                }
            }
        } else {
            for (int e = tid; e < kHM * kHK; e += kHThreads) {
                const int r = e / kHK, kk = e % kHK, s = src[r], k = k0 + kk;
                as[r * kARow + kk] = s >= 0 && k < Kd ? X[(long long)s * Kd + k] : T(0.f);
                if constexpr (kTrans) {
                    const int nn = n0 + r;
                    bs[r * kBRow + kk] = nn < Nd && k < Kd ? W[(long long)nn * Kd + k] : T(0.f);
                } else {
                    const int rk = e / kHN, c = e % kHN, kb = k0 + rk, nn = n0 + c;
                    bs[rk * kBRow + c] = kb < Kd && nn < Nd ? W[(long long)kb * Nd + nn] : T(0.f);
                }
            }
        }
    };

    const int wm = (warp / 2) * 32, wn = (warp % 2) * 32;
    float acc[2][4][4] = {};
    const int nk = (Kd + kHK - 1) / kHK;
    load(0, 0);
    cp_async_commit();
    for (int kt = 0; kt < nk; kt++) {
        if (kt + 1 < nk) load((kt + 1) & 1, (kt + 1) * kHK);
        cp_async_commit();
        cp_async_wait_one();
        __syncthreads();
        const __half* as = reinterpret_cast<const __half*>(As[kt & 1]);
        const __half* bs = reinterpret_cast<const __half*>(Bs[kt & 1]);
#pragma unroll
        for (int ks = 0; ks < kHK; ks += 16) {
            uint32_t a[2][4], b[4][2];
#pragma unroll
            for (int i = 0; i < 2; i++)
                ldmatrix_x4(a[i], as + (wm + i * 16 + (lane % 16)) * kARow + ks + (lane / 16) * 8);
            load_b<kTrans, kBRow>(b, bs, 0, wn, ks, lane);
            load_b<kTrans, kBRow>(b, bs, 2, wn + 16, ks, lane);
#pragma unroll
            for (int i = 0; i < 2; i++)
#pragma unroll
                for (int j = 0; j < 4; j++) mma(acc[i][j], a[i], b[j], T());
        }
        __syncthreads();
    }

#pragma unroll
    for (int i = 0; i < 2; i++)
#pragma unroll
        for (int h = 0; h < 2; h++) {
            const int d = dst[wm + i * 16 + h * 8 + lane / 4];
            if (d < 0) continue;
            float* y = Y + (long long)d * Nd;
#pragma unroll
            for (int j = 0; j < 4; j++) {
                const int c = n0 + wn + j * 8 + (lane % 4) * 2;
                if (kVec) {
                    if (c < Nd) {
                        float2 v = *reinterpret_cast<float2*>(y + c);
                        v.x += acc[i][j][2 * h];
                        v.y += acc[i][j][2 * h + 1];
                        *reinterpret_cast<float2*>(y + c) = v;
                    }
                } else {
                    if (c < Nd) y[c] += acc[i][j][2 * h];
                    if (c + 1 < Nd) y[c + 1] += acc[i][j][2 * h + 1];
                }
            }
        }
}

// out[e] = Y[e] rounded to the half type.
template <typename T>
__global__ void round_rows_kernel(const float* __restrict__ Y, long long n, T* __restrict__ out) {
    for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += (long long)gridDim.x * blockDim.x)
        round_to(Y[e], out[e]);
}

// partial[c] (Ci x Co, fp32) = sum over chunk c's pairs of X[xs]^T DY[ys], one 64 x 64 tile per CTA (grid.y, grid.z).
// kVec: Ci and Co are multiples of 8 and X, DY 16-byte aligned.
template <typename T, bool kVec>
__global__ void __launch_bounds__(kHThreads) sparse_wgrad_mma_kernel(ConvOffsets off, int K,
                                                                     const int2* __restrict__ pairs, int x_side,
                                                                     const T* __restrict__ X, int Ci,
                                                                     const T* __restrict__ DY, int Co,
                                                                     float* __restrict__ partial) {
    constexpr int kRow = kHM + kPad;
    static_assert(kHM == kHN, "one shared row width for both operands");
    __shared__ __align__(16) T As[2][kHK * kRow];   // [pair][input channel]
    __shared__ __align__(16) T Bs[2][kHK * kRow];   // [pair][output channel]
    long long p0, p1;
    if (chunk_of(off, K, blockIdx.x, p0, p1) < 0) return;
    const int tid = threadIdx.x, warp = tid / 32, lane = tid % 32;
    const int m0 = blockIdx.y * kHM, n0 = blockIdx.z * kHN;

    auto load = [&](int st, long long q0) {
        T* as = As[st];
        T* bs = Bs[st];
        if constexpr (kVec) {
#pragma unroll
            for (int u = 0; u < 2; u++) {
                const int c = tid + u * kHThreads, r = c / 8, cc = (c % 8) * 8;
                const long long p = q0 + r;
                int xr = -1, yr = -1;
                if (p < p1) {
                    const int2 pr = __ldg(pairs + p);
                    xr = x_side ? pr.y : pr.x;
                    yr = x_side ? pr.x : pr.y;
                }
                const int ci = m0 + cc, co = n0 + cc;
                const bool oka = xr >= 0 && ci < Ci, okb = yr >= 0 && co < Co;
                cp_async16(as + r * kRow + cc, oka ? X + (long long)xr * Ci + ci : X, oka);
                cp_async16(bs + r * kRow + cc, okb ? DY + (long long)yr * Co + co : DY, okb);
            }
        } else {
            for (int e = tid; e < kHK * kHM; e += kHThreads) {
                const int r = e / kHM, cc = e % kHM;
                const long long p = q0 + r;
                int xr = -1, yr = -1;
                if (p < p1) {
                    const int2 pr = __ldg(pairs + p);
                    xr = x_side ? pr.y : pr.x;
                    yr = x_side ? pr.x : pr.y;
                }
                const int ci = m0 + cc, co = n0 + cc;
                as[r * kRow + cc] = xr >= 0 && ci < Ci ? X[(long long)xr * Ci + ci] : T(0.f);
                bs[r * kRow + cc] = yr >= 0 && co < Co ? DY[(long long)yr * Co + co] : T(0.f);
            }
        }
    };

    const int wm = (warp / 2) * 32, wn = (warp % 2) * 32;
    float acc[2][4][4] = {}, blk[2][4][4] = {};
    load(0, p0);
    cp_async_commit();
    for (long long q0 = p0; q0 < p1; q0 += kHK) {
        const int st = (int)((q0 - p0) / kHK) & 1;
        if (q0 + kHK < p1) load(st ^ 1, q0 + kHK);
        cp_async_commit();
        cp_async_wait_one();
        __syncthreads();
        const __half* as = reinterpret_cast<const __half*>(As[st]);
        const __half* bs = reinterpret_cast<const __half*>(Bs[st]);
#pragma unroll
        for (int ks = 0; ks < kHK; ks += 16) {
            uint32_t a[2][4], b[4][2];
#pragma unroll
            for (int i = 0; i < 2; i++)   // A(ci, pair) from [pair][ci]
                ldmatrix_x4_trans(a[i], as + (ks + (lane % 8) + (lane / 16) * 8) * kRow + wm + i * 16 +
                                            ((lane / 8) % 2) * 8);
            load_b<false, kRow>(b, bs, 0, wn, ks, lane);
            load_b<false, kRow>(b, bs, 2, wn + 16, ks, lane);
#pragma unroll
            for (int i = 0; i < 2; i++)
#pragma unroll
                for (int j = 0; j < 4; j++) mma(blk[i][j], a[i], b[j], T());
        }
        __syncthreads();
        if ((q0 - p0 + kHK) % kInnerH == 0 || q0 + kHK >= p1) {
#pragma unroll
            for (int i = 0; i < 2; i++)
#pragma unroll
                for (int j = 0; j < 4; j++)
#pragma unroll
                    for (int e = 0; e < 4; e++) { acc[i][j][e] += blk[i][j][e]; blk[i][j][e] = 0.f; }
        }
    }
    float* out = partial + (long long)blockIdx.x * Ci * Co;
#pragma unroll
    for (int i = 0; i < 2; i++)
#pragma unroll
        for (int h = 0; h < 2; h++) {
            const int ci = m0 + wm + i * 16 + h * 8 + lane / 4;
            if (ci >= Ci) continue;
#pragma unroll
            for (int j = 0; j < 4; j++) {
                const int co = n0 + wn + j * 8 + (lane % 4) * 2;
                if (co < Co) out[(long long)ci * Co + co] = acc[i][j][2 * h];
                if (co + 1 < Co) out[(long long)ci * Co + co + 1] = acc[i][j][2 * h + 1];
            }
        }
}

bool aligned16(const void* p) { return reinterpret_cast<uintptr_t>(p) % 16 == 0; }

int check_dtype(const char* fn, int32_t dtype) {
    if (dtype != SGB_FEAT_F16 && dtype != SGB_FEAT_BF16) {
        set_error("%s: dtype %d (need SGB_FEAT_F16 or SGB_FEAT_BF16)", fn, dtype);
        return SGB_E_INVALID;
    }
    return SGB_OK;
}

// Bytes of the fp32 scratch of a forward / input-gradient call writing `rows` x `cols`; 0 when the arguments would be
// rejected.
size_t scratch_bytes(const char* fn, int32_t dtype, int32_t K, const int64_t* offsets_host, int64_t n_in, int32_t C_in,
                     int64_t n_out, int32_t C_out, int64_t rows, int32_t cols) {
    ConvOffsets off;
    if (check_dtype(fn, dtype) || check_offsets(fn, K, offsets_host, C_in, C_out, off)) return 0;
    if (n_in < 0 || n_out < 0 || n_in > INT32_MAX || n_out > INT32_MAX) return 0;
    return align_up(sizeof(float) * (size_t)(rows > 0 ? rows : 1) * cols);
}

int check_workspace(const char* fn, const void* workspace) {
    if (!workspace || !aligned16(workspace)) {
        set_error("%s: null or unaligned workspace", fn);
        return SGB_E_INVALID;
    }
    return SGB_OK;
}

// out (rows x Nd, half type) = the sum over offsets of the gathered products, accumulated offset by offset in the
// fp32 scratch Y and rounded once.
template <typename T, bool kTrans>
int run_gather_mma(const char* fn, const ConvOffsets& off, int K, const int32_t* pairs, int src_side, const T* X,
                   int Kd, const T* W, int Nd, float* Y, T* out, long long rows, cudaStream_t s) {
    const size_t total = (size_t)rows * Nd;
    SGB_CUDA(cudaMemsetAsync(Y, 0, sizeof(float) * total, s));
    const bool vec = Kd % 8 == 0 && Nd % 8 == 0 && aligned16(X) && aligned16(W);
    const long long wstride = (long long)Kd * Nd;
    for (int d = 0; d < K; d++) {
        const long long n = off.at[d + 1] - off.at[d];
        if (n == 0) continue;
        const dim3 grid((unsigned)((n + kHM - 1) / kHM), (unsigned)((Nd + kHN - 1) / kHN));
        const int2* p = reinterpret_cast<const int2*>(pairs) + off.at[d];
        if (vec)
            sparse_gather_mma_kernel<T, kTrans, true><<<grid, kHThreads, 0, s>>>(p, n, src_side, X, Kd,
                                                                                 W + d * wstride, Nd, Y);
        else
            sparse_gather_mma_kernel<T, kTrans, false><<<grid, kHThreads, 0, s>>>(p, n, src_side, X, Kd,
                                                                                  W + d * wstride, Nd, Y);
        SGB_LAUNCH_CHECK(fn, 0, s);
    }
    const long long blocks = std::min<long long>(((long long)total + 255) / 256, 16LL * kNumSMs);
    round_rows_kernel<T><<<(unsigned)blocks, 256, 0, s>>>(Y, (long long)total, out);
    SGB_LAUNCH_CHECK("round_rows_kernel", 0, s);
    return SGB_OK;
}

template <typename T>
int run_wgrad_mma(const ConvOffsets& off, int K, const int32_t* pairs, int x_side, const T* x, int C_in, const T* dy,
                  int C_out, float* partial, float* dkernel, cudaStream_t s) {
    const long long chunks = total_chunks(off, K);
    if (chunks > 0) {
        const dim3 grid((unsigned)chunks, (unsigned)((C_in + kHM - 1) / kHM), (unsigned)((C_out + kHN - 1) / kHN));
        const int2* p = reinterpret_cast<const int2*>(pairs);
        if (C_in % 8 == 0 && C_out % 8 == 0 && aligned16(x) && aligned16(dy))
            sparse_wgrad_mma_kernel<T, true><<<grid, kHThreads, 0, s>>>(off, K, p, x_side, x, C_in, dy, C_out,
                                                                        partial);
        else
            sparse_wgrad_mma_kernel<T, false><<<grid, kHThreads, 0, s>>>(off, K, p, x_side, x, C_in, dy, C_out,
                                                                         partial);
        SGB_LAUNCH_CHECK("sparse_wgrad_mma_kernel", 0, s);
    }
    return launch_wgrad_reduce(off, K, (long long)C_in * C_out, partial, dkernel, s);
}

}  // namespace

}  // namespace sgb

using namespace sgb;

extern "C" {

size_t sgb_sparse_conv_half_forward_workspace_bytes(int32_t dtype, int32_t K, const int64_t* offsets_host,
                                                    int64_t n_in, int32_t C_in, int64_t n_out, int32_t C_out) {
    return scratch_bytes("sgb_sparse_conv_half_forward_workspace_bytes", dtype, K, offsets_host, n_in, C_in, n_out,
                         C_out, n_out, C_out);
}

int sgb_sparse_conv_half_forward(int32_t dtype, int32_t K, const int64_t* offsets_host, const int32_t* pairs,
                                 int32_t transposed, int64_t n_in, int32_t C_in, const void* x, const void* kernel,
                                 int64_t n_out, int32_t C_out, void* workspace, void* out, void* stream) {
    const char* fn = "sgb_sparse_conv_half_forward";
    ConvOffsets off;
    if (int rc = check_dtype(fn, dtype)) return rc;
    if (int rc = check_conv_args(fn, K, offsets_host, pairs, n_in, C_in, n_out, C_out, off)) return rc;
    if (!x || !kernel || !out) { set_error("%s: null x / kernel / out", fn); return SGB_E_INVALID; }
    if (int rc = check_workspace(fn, workspace)) return rc;
    if (n_out == 0) return SGB_OK;
    const int side = transposed ? 1 : 0;
    cudaStream_t s = (cudaStream_t)stream;
    float* Y = (float*)workspace;
    if (dtype == SGB_FEAT_F16)
        return run_gather_mma<__half, false>(fn, off, K, pairs, side, (const __half*)x, C_in, (const __half*)kernel,
                                             C_out, Y, (__half*)out, n_out, s);
    return run_gather_mma<__nv_bfloat16, false>(fn, off, K, pairs, side, (const __nv_bfloat16*)x, C_in,
                                                (const __nv_bfloat16*)kernel, C_out, Y, (__nv_bfloat16*)out, n_out, s);
}

size_t sgb_sparse_conv_half_backward_input_workspace_bytes(int32_t dtype, int32_t K, const int64_t* offsets_host,
                                                           int64_t n_in, int32_t C_in, int64_t n_out, int32_t C_out) {
    return scratch_bytes("sgb_sparse_conv_half_backward_input_workspace_bytes", dtype, K, offsets_host, n_in, C_in,
                         n_out, C_out, n_in, C_in);
}

int sgb_sparse_conv_half_backward_input(int32_t dtype, int32_t K, const int64_t* offsets_host, const int32_t* pairs,
                                        int32_t transposed, int64_t n_in, int32_t C_in, void* dx, const void* kernel,
                                        int64_t n_out, int32_t C_out, const void* dy, void* workspace, void* stream) {
    const char* fn = "sgb_sparse_conv_half_backward_input";
    ConvOffsets off;
    if (int rc = check_dtype(fn, dtype)) return rc;
    if (int rc = check_conv_args(fn, K, offsets_host, pairs, n_in, C_in, n_out, C_out, off)) return rc;
    if (!dx || !kernel || !dy) { set_error("%s: null dx / kernel / dy", fn); return SGB_E_INVALID; }
    if (int rc = check_workspace(fn, workspace)) return rc;
    if (n_in == 0) return SGB_OK;
    const int side = transposed ? 0 : 1;
    cudaStream_t s = (cudaStream_t)stream;
    float* Y = (float*)workspace;
    if (dtype == SGB_FEAT_F16)
        return run_gather_mma<__half, true>(fn, off, K, pairs, side, (const __half*)dy, C_out, (const __half*)kernel,
                                            C_in, Y, (__half*)dx, n_in, s);
    return run_gather_mma<__nv_bfloat16, true>(fn, off, K, pairs, side, (const __nv_bfloat16*)dy, C_out,
                                               (const __nv_bfloat16*)kernel, C_in, Y, (__nv_bfloat16*)dx, n_in, s);
}

size_t sgb_sparse_conv_half_backward_weight_workspace_bytes(int32_t dtype, int32_t K, const int64_t* offsets_host,
                                                            int32_t C_in, int32_t C_out) {
    if (check_dtype("sgb_sparse_conv_half_backward_weight_workspace_bytes", dtype)) return 0;
    return sgb_sparse_conv_backward_weight_workspace_bytes(K, offsets_host, C_in, C_out);
}

int sgb_sparse_conv_half_backward_weight(int32_t dtype, int32_t K, const int64_t* offsets_host, const int32_t* pairs,
                                         int32_t transposed, int64_t n_in, int32_t C_in, const void* x, int64_t n_out,
                                         int32_t C_out, const void* dy, void* workspace, float* dkernel,
                                         void* stream) {
    const char* fn = "sgb_sparse_conv_half_backward_weight";
    ConvOffsets off;
    if (int rc = check_dtype(fn, dtype)) return rc;
    if (int rc = check_conv_args(fn, K, offsets_host, pairs, n_in, C_in, n_out, C_out, off)) return rc;
    if (!x || !dy || !dkernel) { set_error("%s: null x / dy / dkernel", fn); return SGB_E_INVALID; }
    if (int rc = check_workspace(fn, workspace)) return rc;
    const int side = transposed ? 1 : 0;
    cudaStream_t s = (cudaStream_t)stream;
    float* partial = (float*)workspace;
    if (dtype == SGB_FEAT_F16)
        return run_wgrad_mma<__half>(off, K, pairs, side, (const __half*)x, C_in, (const __half*)dy, C_out, partial,
                                     dkernel, s);
    return run_wgrad_mma<__nv_bfloat16>(off, K, pairs, side, (const __nv_bfloat16*)x, C_in, (const __nv_bfloat16*)dy,
                                        C_out, partial, dkernel, s);
}

}  // extern "C"
