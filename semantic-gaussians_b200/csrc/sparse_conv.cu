// Products of the sparse 3D convolution over a kernel map (sparse_coords.cu): fp32 in, fp32 out, FP32 accumulation.
//
// Pairs are int2 (in row, out row), grouped by offset; offsets[d] .. offsets[d+1] are offset d's pairs and, within one
// offset, every row appears at most once on either side.  The kernel is (K, C_in, C_out), row-major.
//
//   forward        out[o]  = sum_d x[i_d(o)] W_d           (transposed layer: out[i] = sum_d x[o_d(i)] W_d)
//   input grad     dx[i]   = sum_d dy[o_d(i)] W_d^T        (transposed layer: dx[o] = sum_d dy[i_d(o)] W_d^T)
//   weight grad    dW_d    = sum_pairs x[src]^T dy[dst]
//
// Forward and input gradient: one gather-GEMM-scatter launch per non-empty offset, in offset order, each adding its
// product into the zeroed output.  Because an offset's pairs are one-to-one, no two threads of a launch touch the same
// output row, and the stream orders the launches: no atomics, the same sums in the same order on every call.  Work is
// proportional to the pair count; an offset without pairs launches nothing.
//
// Weight gradient: the pairs of each offset are cut into chunks of kChunk; one CTA per (chunk, 64 x 64 tile of dW_d)
// writes its partial sum to the workspace (accumulated per 128-pair block, then summed over the blocks, to keep the
// rounding error of long reductions small), and a second pass adds each offset's chunk partials in chunk order.
//
// Tiles: 64 rows x 64 columns per CTA of 256 threads, each thread a 4 x 4 FFMA register tile over 16-deep shared
// operands.
#include "sparse_conv.cuh"

namespace sgb {

namespace {

constexpr int kBM = 64, kBN = 64, kBK = 16, kConvThreads = 256;
constexpr int kInner = 128;            // pairs per inner accumulation block of the weight gradient

// Y[dst(p)] += X[src(p)] B for the n pairs at `pairs`, where B(k, n) = trans ? W[n * Kd + k] : W[k * Nd + n].
// Kd: columns of X (reduction depth), Nd: columns of Y.
template <bool kTrans>
__global__ void __launch_bounds__(kConvThreads) sparse_gather_gemm_kernel(const int2* __restrict__ pairs, long long n,
                                                                          int src_side, const float* __restrict__ X,
                                                                          int Kd, const float* __restrict__ W, int Nd,
                                                                          float* __restrict__ Y) {
    __shared__ __align__(16) float As[kBK][kBM];
    __shared__ __align__(16) float Bs[kBK][kBN];
    __shared__ int src[kBM], dst[kBM];
    const int tid = threadIdx.x, tx = tid % 16, ty = tid / 16;
    const long long m0 = (long long)blockIdx.x * kBM;
    const int n0 = blockIdx.y * kBN;
    if (tid < kBM) {
        const long long p = m0 + tid;
        int2 pr = p < n ? pairs[p] : make_int2(-1, -1);
        src[tid] = src_side ? pr.y : pr.x;
        dst[tid] = src_side ? pr.x : pr.y;
    }
    __syncthreads();
    float acc[4][4] = {};
    const int a_row = tid / 4, a_k = (tid % 4) * 4;
    const int b_k = tid / 16, b_n = (tid % 16) * 4;
    const int a_src = src[a_row];
    for (int k0 = 0; k0 < Kd; k0 += kBK) {
#pragma unroll
        for (int u = 0; u < 4; u++) {
            const int k = k0 + a_k + u;
            As[a_k + u][a_row] = a_src >= 0 && k < Kd ? __ldg(X + (long long)a_src * Kd + k) : 0.f;
            const int kb = k0 + b_k, nb = n0 + b_n + u;
            Bs[b_k][b_n + u] = kb < Kd && nb < Nd ? __ldg(W + (kTrans ? (long long)nb * Kd + kb : (long long)kb * Nd + nb))
                                                  : 0.f;
        }
        __syncthreads();
#pragma unroll
        for (int kk = 0; kk < kBK; kk++) {
            const float4 a = *reinterpret_cast<const float4*>(&As[kk][ty * 4]);
            const float4 b = *reinterpret_cast<const float4*>(&Bs[kk][tx * 4]);
            const float av[4] = {a.x, a.y, a.z, a.w}, bv[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
            for (int i = 0; i < 4; i++)
#pragma unroll
                for (int j = 0; j < 4; j++) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
        }
        __syncthreads();
    }
#pragma unroll
    for (int i = 0; i < 4; i++) {
        const int d = dst[ty * 4 + i];
        if (d < 0) continue;
        float* y = Y + (long long)d * Nd;
#pragma unroll
        for (int j = 0; j < 4; j++) {
            const int c = n0 + tx * 4 + j;
            if (c < Nd) y[c] += acc[i][j];
        }
    }
}

// partial[c] (Ci x Co) = sum over chunk c's pairs of X[xs]^T DY[ys], one 64 x 64 tile per CTA (grid.y, grid.z).
__global__ void __launch_bounds__(kConvThreads) sparse_wgrad_partial_kernel(ConvOffsets off, int K,
                                                                            const int2* __restrict__ pairs,
                                                                            int x_side, const float* __restrict__ X,
                                                                            int Ci, const float* __restrict__ DY, int Co,
                                                                            float* __restrict__ partial) {
    __shared__ __align__(16) float As[kBK][kBM];   // [pair][input channel]
    __shared__ __align__(16) float Bs[kBK][kBN];   // [pair][output channel]
    long long p0, p1;
    if (chunk_of(off, K, blockIdx.x, p0, p1) < 0) return;
    const int tid = threadIdx.x, tx = tid % 16, ty = tid / 16;
    const int m0 = blockIdx.y * kBM, n0 = blockIdx.z * kBN;
    const int l_k = tid / 16, l_c = (tid % 16) * 4;
    float acc[4][4] = {}, blk[4][4] = {};
    for (long long q0 = p0; q0 < p1; q0 += kBK) {
        const long long p = q0 + l_k;
        int xr = -1, yr = -1;
        if (p < p1) {
            const int2 pr = __ldg(pairs + p);
            xr = x_side ? pr.y : pr.x;
            yr = x_side ? pr.x : pr.y;
        }
#pragma unroll
        for (int u = 0; u < 4; u++) {
            const int ci = m0 + l_c + u, co = n0 + l_c + u;
            As[l_k][l_c + u] = xr >= 0 && ci < Ci ? __ldg(X + (long long)xr * Ci + ci) : 0.f;
            Bs[l_k][l_c + u] = yr >= 0 && co < Co ? __ldg(DY + (long long)yr * Co + co) : 0.f;
        }
        __syncthreads();
#pragma unroll
        for (int kk = 0; kk < kBK; kk++) {
            const float4 a = *reinterpret_cast<const float4*>(&As[kk][ty * 4]);
            const float4 b = *reinterpret_cast<const float4*>(&Bs[kk][tx * 4]);
            const float av[4] = {a.x, a.y, a.z, a.w}, bv[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
            for (int i = 0; i < 4; i++)
#pragma unroll
                for (int j = 0; j < 4; j++) blk[i][j] = fmaf(av[i], bv[j], blk[i][j]);
        }
        __syncthreads();
        if ((q0 - p0 + kBK) % kInner == 0 || q0 + kBK >= p1) {
#pragma unroll
            for (int i = 0; i < 4; i++)
#pragma unroll
                for (int j = 0; j < 4; j++) { acc[i][j] += blk[i][j]; blk[i][j] = 0.f; }
        }
    }
    float* out = partial + (long long)blockIdx.x * Ci * Co;
#pragma unroll
    for (int i = 0; i < 4; i++) {
        const int ci = m0 + ty * 4 + i;
        if (ci >= Ci) continue;
#pragma unroll
        for (int j = 0; j < 4; j++) {
            const int co = n0 + tx * 4 + j;
            if (co < Co) out[(long long)ci * Co + co] = acc[i][j];
        }
    }
}

// dW[d][e] = sum of offset d's chunk partials in chunk order (0 for an offset without pairs).
__global__ void sparse_wgrad_reduce_kernel(ConvOffsets off, int K, long long CC, const float* __restrict__ partial,
                                           float* __restrict__ dW) {
    const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const int d = blockIdx.y;
    if (e >= CC) return;
    long long c0 = 0;
    for (int j = 0; j < d; j++) c0 += (off.at[j + 1] - off.at[j] + kChunk - 1) / kChunk;
    const long long nc = (off.at[d + 1] - off.at[d] + kChunk - 1) / kChunk;
    float s = 0.f;
    for (long long c = 0; c < nc; c++) s += partial[(c0 + c) * CC + e];
    dW[(long long)d * CC + e] = s;
}

// Y (rows x Nd, zeroed here) = sum over offsets of the gathered products, offset by offset.
int run_gather_gemm(const char* fn, const ConvOffsets& off, int K, const int32_t* pairs, int src_side, bool trans,
                    const float* X, int Kd, const float* W, int Nd, float* Y, long long rows, cudaStream_t s) {
    SGB_CUDA(cudaMemsetAsync(Y, 0, sizeof(float) * (size_t)rows * Nd, s));
    const long long wstride = (long long)Kd * Nd;
    for (int d = 0; d < K; d++) {
        const long long n = off.at[d + 1] - off.at[d];
        if (n == 0) continue;
        const dim3 grid((unsigned)((n + kBM - 1) / kBM), (unsigned)((Nd + kBN - 1) / kBN));
        const int2* p = reinterpret_cast<const int2*>(pairs) + off.at[d];
        if (trans)
            sparse_gather_gemm_kernel<true><<<grid, kConvThreads, 0, s>>>(p, n, src_side, X, Kd, W + d * wstride, Nd, Y);
        else
            sparse_gather_gemm_kernel<false><<<grid, kConvThreads, 0, s>>>(p, n, src_side, X, Kd, W + d * wstride, Nd, Y);
        SGB_LAUNCH_CHECK(fn, 0, s);
    }
    return SGB_OK;
}

}  // namespace

long long total_chunks(const ConvOffsets& off, int K) {
    long long n = 0;
    for (int d = 0; d < K; d++) n += (off.at[d + 1] - off.at[d] + kChunk - 1) / kChunk;
    return n;
}

int check_offsets(const char* fn, int32_t K, const int64_t* offsets_host, int32_t C_in, int32_t C_out,
                  ConvOffsets& off) {
    if (K < 1 || K > SGB_SPARSE_MAX_K) { set_error("%s: K = %d (need 1 <= K <= %d)", fn, K, SGB_SPARSE_MAX_K); return SGB_E_INVALID; }
    if (C_in <= 0 || C_out <= 0) { set_error("%s: C_in = %d, C_out = %d (need > 0)", fn, C_in, C_out); return SGB_E_INVALID; }
    if (!offsets_host) { set_error("%s: null offsets", fn); return SGB_E_INVALID; }
    if (offsets_host[0] != 0) { set_error("%s: offsets[0] = %lld (need 0)", fn, (long long)offsets_host[0]); return SGB_E_INVALID; }
    for (int d = 0; d <= K; d++) {
        if (d > 0 && offsets_host[d] < offsets_host[d - 1]) { set_error("%s: offsets decrease at %d", fn, d); return SGB_E_INVALID; }
        off.at[d] = offsets_host[d];
    }
    return SGB_OK;
}

int check_conv_args(const char* fn, int32_t K, const int64_t* offsets_host, const int32_t* pairs, int64_t n_in,
                    int32_t C_in, int64_t n_out, int32_t C_out, ConvOffsets& off) {
    if (int rc = check_offsets(fn, K, offsets_host, C_in, C_out, off)) return rc;
    if (n_in < 0 || n_out < 0 || n_in > INT32_MAX || n_out > INT32_MAX) {
        set_error("%s: row counts %lld, %lld out of range", fn, (long long)n_in, (long long)n_out);
        return SGB_E_INVALID;
    }
    if (off.at[K] > 0 && (!pairs || reinterpret_cast<uintptr_t>(pairs) % 8)) {
        set_error("%s: null or unaligned pairs", fn);
        return SGB_E_INVALID;
    }
    return SGB_OK;
}

int launch_wgrad_reduce(const ConvOffsets& off, int K, long long CC, const float* partial, float* dW,
                        cudaStream_t s) {
    const dim3 grid((unsigned)((CC + 255) / 256), (unsigned)K);
    sparse_wgrad_reduce_kernel<<<grid, 256, 0, s>>>(off, K, CC, partial, dW);
    SGB_LAUNCH_CHECK("sparse_wgrad_reduce_kernel", 0, s);
    return SGB_OK;
}

}  // namespace sgb

using namespace sgb;

extern "C" {

int sgb_sparse_conv_forward(int32_t K, const int64_t* offsets_host, const int32_t* pairs, int32_t transposed,
                            int64_t n_in, int32_t C_in, const float* x, const float* kernel, int64_t n_out,
                            int32_t C_out, float* out, void* stream) {
    const char* fn = "sgb_sparse_conv_forward";
    ConvOffsets off;
    if (int rc = check_conv_args(fn, K, offsets_host, pairs, n_in, C_in, n_out, C_out, off)) return rc;
    if (!x || !kernel || !out) { set_error("%s: null x / kernel / out", fn); return SGB_E_INVALID; }
    if (n_out == 0) return SGB_OK;
    return run_gather_gemm(fn, off, K, pairs, transposed ? 1 : 0, false, x, C_in, kernel, C_out, out, n_out,
                           (cudaStream_t)stream);
}

int sgb_sparse_conv_backward_input(int32_t K, const int64_t* offsets_host, const int32_t* pairs, int32_t transposed,
                                   int64_t n_in, int32_t C_in, float* dx, const float* kernel, int64_t n_out,
                                   int32_t C_out, const float* dy, void* stream) {
    const char* fn = "sgb_sparse_conv_backward_input";
    ConvOffsets off;
    if (int rc = check_conv_args(fn, K, offsets_host, pairs, n_in, C_in, n_out, C_out, off)) return rc;
    if (!dx || !kernel || !dy) { set_error("%s: null dx / kernel / dy", fn); return SGB_E_INVALID; }
    if (n_in == 0) return SGB_OK;
    return run_gather_gemm(fn, off, K, pairs, transposed ? 0 : 1, true, dy, C_out, kernel, C_in, dx, n_in,
                           (cudaStream_t)stream);
}

size_t sgb_sparse_conv_backward_weight_workspace_bytes(int32_t K, const int64_t* offsets_host, int32_t C_in,
                                                       int32_t C_out) {
    ConvOffsets off;
    if (check_offsets("sgb_sparse_conv_backward_weight_workspace_bytes", K, offsets_host, C_in, C_out, off)) return 0;
    const long long n = total_chunks(off, K);
    return align_up(sizeof(float) * (size_t)(n > 0 ? n : 1) * C_in * C_out);
}

int sgb_sparse_conv_backward_weight(int32_t K, const int64_t* offsets_host, const int32_t* pairs, int32_t transposed,
                                    int64_t n_in, int32_t C_in, const float* x, int64_t n_out, int32_t C_out,
                                    const float* dy, void* workspace, float* dkernel, void* stream) {
    const char* fn = "sgb_sparse_conv_backward_weight";
    ConvOffsets off;
    if (int rc = check_conv_args(fn, K, offsets_host, pairs, n_in, C_in, n_out, C_out, off)) return rc;
    if (!x || !dy || !dkernel) { set_error("%s: null x / dy / dkernel", fn); return SGB_E_INVALID; }
    if (!workspace || reinterpret_cast<uintptr_t>(workspace) % 16) {
        set_error("%s: null or unaligned workspace", fn);
        return SGB_E_INVALID;
    }
    cudaStream_t s = (cudaStream_t)stream;
    const long long chunks = total_chunks(off, K);
    float* partial = (float*)workspace;
    if (chunks > 0) {
        const dim3 grid((unsigned)chunks, (unsigned)((C_in + kBM - 1) / kBM), (unsigned)((C_out + kBN - 1) / kBN));
        sparse_wgrad_partial_kernel<<<grid, kConvThreads, 0, s>>>(off, K, reinterpret_cast<const int2*>(pairs),
                                                                  transposed ? 1 : 0, x, C_in, dy, C_out, partial);
        SGB_LAUNCH_CHECK("sparse_wgrad_partial_kernel", 0, s);
    }
    return launch_wgrad_reduce(off, K, (long long)C_in * C_out, partial, dkernel, s);
}

}  // extern "C"
