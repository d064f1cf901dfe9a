// Adam step of up to SGB_ADAM_MAX_TENSORS parameter tables in one launch, with a per-row visibility mask
// (sgb_adam_step, include/sgb200.h).  torch.optim.Adam without amsgrad / weight_decay, in torch's order of operations:
//
//   m = m + (g - m) (1 - beta1)      v = beta2 v + (1 - beta2) g g      p = p - step_size (m / (sqrt(v) / bc2 + eps))
//
// The step is pure streaming: 28 bytes per fp32 element (p, g, m, v read, p, m, v written) and nothing to reuse, so
// the kernel's only job is to touch each visible element once with wide, coalesced accesses and to touch nothing of
// an invisible row beyond its mask byte.
//
// Work item = (tensor, block of consecutive rows), one CTA each; the host sizes the row blocks from the shapes so
// that an item covers about kAdamItemElems elements, and passes descriptors and the item layout as kernel
// parameters.  Inside an item the rows are one flat run of elements and consecutive threads take consecutive
// 16-byte (or, on the scalar path, 4-byte) pieces of it: a wide row is read along its length by whole warps, a
// narrow table (row_len 1, 3, 4, 45, 48) packs many rows into a warp.  A piece finds its row by one integer
// division and reads that row's mask byte; pieces of an invisible row issue no other access.  A tensor without a
// mask has no row structure to respect and is laid out as rows of one piece.
//
// H100 80GB HBM3 at 700 W (tools/time_adam.py), the six geometry tables + a (P, C) feature table: 1 M x 256 dense
// 2.98 ms (2.96 TB/s over 28 B/element), 24 % of the rows visible 0.97 ms; 3 M x 512 dense 16.2 ms (2.95 TB/s), 26 %
// visible 5.04 ms.  62 registers, no spills.
#include <algorithm>
#include <cmath>

#include "common.cuh"

namespace sgb {
namespace {

constexpr int kAdamThreads = 256;
constexpr uint32_t kAdamItemElems = 4096;  // elements per work item aimed at: 16 KB of each of p, g, m, v

struct AdamCoef {
    float w1, beta2, w2, eps, step_size, bc2;  // w = 1 - beta, rounded to fp32 from the caller's double
};

struct AdamTable {  // one tensor of the call as the kernel sees it
    float* param;
    const float* grad;
    float* exp_avg;
    float* exp_avg_sq;
    const uint8_t* visible;
    int64_t rows;
    uint32_t row_len;
    uint32_t rows_per_item;
    uint32_t first_item;  // its work items are [first_item, first_item of the next table)
    uint32_t wide;        // 16-byte access
    AdamCoef c;
};

struct AdamLaunch {
    AdamTable t[SGB_ADAM_MAX_TENSORS];
    int32_t n;
};

__device__ __forceinline__ void adam_update(float& p, float g, float& m, float& v, const AdamCoef& c) {
    m = m + (g - m) * c.w1;
    v = c.beta2 * v + c.w2 * g * g;
    p = p - c.step_size * (m / (sqrtf(v) / c.bc2 + c.eps));
}
__device__ __forceinline__ void adam_update(float4& p, float4 g, float4& m, float4& v, const AdamCoef& c) {
    adam_update(p.x, g.x, m.x, v.x, c);
    adam_update(p.y, g.y, m.y, v.y, c);
    adam_update(p.z, g.z, m.z, v.z, c);
    adam_update(p.w, g.w, m.w, v.w, c);
}

// The rows [row0, row0 + nrows) of one tensor as pieces of type T (float4 or float).  U pieces per thread are
// loaded before the first is updated, so that a thread has 4 U loads in flight.
template <typename T, int U>
__device__ __forceinline__ void adam_rows(float* __restrict__ param, const float* __restrict__ grad,
                                          float* __restrict__ exp_avg, float* __restrict__ exp_avg_sq,
                                          const uint8_t* __restrict__ visible, uint32_t row_len, uint32_t nrows,
                                          const AdamCoef c) {
    constexpr uint32_t W = sizeof(T) / sizeof(float);
    T* p = reinterpret_cast<T*>(param);
    const T* g = reinterpret_cast<const T*>(grad);
    T* m = reinterpret_cast<T*>(exp_avg);
    T* v = reinterpret_cast<T*>(exp_avg_sq);
    const uint32_t pieces = nrows * row_len / W;
    for (uint32_t base = threadIdx.x; base < pieces; base += kAdamThreads * U) {
        T pv[U], gv[U], mv[U], vv[U];
        bool on[U];
#pragma unroll
        for (int u = 0; u < U; u++) {
            const uint32_t i = base + u * kAdamThreads;
            on[u] = i < pieces && (!visible || visible[i * W / row_len] != 0);
            if (on[u]) {
                gv[u] = __ldg(g + i);
                pv[u] = p[i];
                mv[u] = m[i];
                vv[u] = v[i];
            }
        }
#pragma unroll
        for (int u = 0; u < U; u++) {
            if (!on[u]) continue;
            const uint32_t i = base + u * kAdamThreads;
            adam_update(pv[u], gv[u], mv[u], vv[u], c);
            p[i] = pv[u];
            m[i] = mv[u];
            v[i] = vv[u];
        }
    }
}

__global__ void __launch_bounds__(kAdamThreads, 4) sgb_adam_step_kernel(const __grid_constant__ AdamLaunch L) {
    int ti = 0;
    while (ti + 1 < L.n && blockIdx.x >= L.t[ti + 1].first_item) ti++;
    const AdamTable& t = L.t[ti];
    const int64_t row0 = (int64_t)(blockIdx.x - t.first_item) * t.rows_per_item;
    const uint32_t nrows = (uint32_t)min((int64_t)t.rows_per_item, t.rows - row0);
    const size_t off = (size_t)row0 * t.row_len;
    const uint8_t* vis = t.visible ? t.visible + row0 : nullptr;
    if (t.wide)
        adam_rows<float4, 2>(t.param + off, t.grad + off, t.exp_avg + off, t.exp_avg_sq + off, vis, t.row_len, nrows, t.c);
    else
        adam_rows<float, 4>(t.param + off, t.grad + off, t.exp_avg + off, t.exp_avg_sq + off, vis, t.row_len, nrows, t.c);
}

bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

}  // namespace
}  // namespace sgb

using namespace sgb;

extern "C" {

int sgb_adam_step(const sgb_adam_tensor* tensors_host, int32_t n, void* stream) {
    static const char* fn = "sgb_adam_step";
    if (n < 0 || n > SGB_ADAM_MAX_TENSORS) {
        set_error("%s: n = %d outside [0, %d]", fn, n, SGB_ADAM_MAX_TENSORS);
        return SGB_E_INVALID;
    }
    if (n > 0 && !tensors_host) { set_error("%s: null tensors", fn); return SGB_E_INVALID; }
    AdamLaunch L = {};
    uint64_t items = 0;
    for (int i = 0; i < n; i++) {
        const sgb_adam_tensor& t = tensors_host[i];
        if (t.rows < 0) { set_error("%s: tensor %d: rows = %lld is negative", fn, i, (long long)t.rows); return SGB_E_INVALID; }
        if (t.row_len < 1) { set_error("%s: tensor %d: row_len = %d < 1", fn, i, t.row_len); return SGB_E_INVALID; }
        if (t.rows > 0 && !t.param) { set_error("%s: tensor %d: null param", fn, i); return SGB_E_INVALID; }
        if (t.rows > 0 && !t.grad) { set_error("%s: tensor %d: null grad", fn, i); return SGB_E_INVALID; }
        if (t.rows > 0 && !t.exp_avg) { set_error("%s: tensor %d: null exp_avg", fn, i); return SGB_E_INVALID; }
        if (t.rows > 0 && !t.exp_avg_sq) { set_error("%s: tensor %d: null exp_avg_sq", fn, i); return SGB_E_INVALID; }
        if (!(t.beta1 >= 0.0 && t.beta1 < 1.0)) { set_error("%s: tensor %d: beta1 = %g outside [0, 1)", fn, i, t.beta1); return SGB_E_INVALID; }
        if (!(t.beta2 >= 0.0 && t.beta2 < 1.0)) { set_error("%s: tensor %d: beta2 = %g outside [0, 1)", fn, i, t.beta2); return SGB_E_INVALID; }
        if (!(t.eps >= 0.0)) { set_error("%s: tensor %d: eps = %g is negative", fn, i, t.eps); return SGB_E_INVALID; }
        if (!std::isfinite(t.step_size)) { set_error("%s: tensor %d: step_size is not finite", fn, i); return SGB_E_INVALID; }
        if (!(t.bias_correction2_sqrt > 0.f && t.bias_correction2_sqrt <= 1.f)) {
            set_error("%s: tensor %d: bias_correction2_sqrt = %g outside (0, 1]", fn, i, t.bias_correction2_sqrt);
            return SGB_E_INVALID;
        }
        if (t.rows == 0) continue;
        AdamTable& d = L.t[L.n];
        d.param = t.param;
        d.grad = t.grad;
        d.exp_avg = t.exp_avg;
        d.exp_avg_sq = t.exp_avg_sq;
        d.visible = t.visible;
        d.rows = t.rows;
        d.row_len = (uint32_t)t.row_len;
        d.c = {(float)(1.0 - t.beta1), (float)t.beta2, (float)(1.0 - t.beta2), (float)t.eps, t.step_size,
               t.bias_correction2_sqrt};
        const bool al = aligned16(t.param) && aligned16(t.grad) && aligned16(t.exp_avg) && aligned16(t.exp_avg_sq);
        if (!t.visible) {  // one flat run of elements: rows of one piece
            const uint64_t total = (uint64_t)t.rows * (uint64_t)t.row_len;
            d.row_len = al && total % 4 == 0 ? 4 : 1;
            d.rows = (int64_t)(total / d.row_len);
        }
        d.wide = al && d.row_len % 4 == 0;
        d.rows_per_item = std::max(1u, kAdamItemElems / d.row_len);
        d.first_item = (uint32_t)items;
        items += ((uint64_t)d.rows + d.rows_per_item - 1) / d.rows_per_item;
        if (items > 0x7fffffffull) {
            set_error("%s: %llu work items exceed one grid", fn, (unsigned long long)items);
            return SGB_E_INVALID;
        }
        L.n++;
    }
    if (L.n == 0) return SGB_OK;
    cudaStream_t s = (cudaStream_t)stream;
    sgb_adam_step_kernel<<<(unsigned)items, kAdamThreads, 0, s>>>(L);
    SGB_LAUNCH_CHECK("sgb_adam_step_kernel", 0, s);
    return SGB_OK;
}

}  // extern "C"
