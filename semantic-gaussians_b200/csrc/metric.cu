// Segmentation confusion matrix on the device: the counting of utils/metric.py::confusion_matrix
//
//   confusion = np.bincount(pred * (num_classes + 1) + gt, minlength=(num_classes + 1) ** 2).reshape(nb, nb)
//
// added into a caller-owned (nb, nb) uint64 histogram, nb = num_classes + 1, with no host round trip per view.
// Every CTA keeps a private uint32 histogram of all nb^2 bins in shared memory, walks its share of the pixels with a
// grid-stride loop and flushes its non-zero bins with one 64-bit atomic each.  Label maps are spatially coherent
// (a wall is one (pred, gt) pair for thousands of pixels), so the lanes of a warp that hit the same bin are merged
// first (__match_any_sync) and their leader adds the popcount: one shared atomic per distinct bin and warp instead
// of 32 to the same address.  Integer counts make the result exact whatever the order of the atomics.
#include "common.cuh"

namespace sgb {

namespace {

constexpr int kConfThreads = 256;
constexpr int kConfVec = 4;                   // labels per lane and step on the vector path
constexpr size_t kConfMaxSmem = 200 * 1024;   // private histogram: nb^2 uint32 bins in one CTA's shared memory
constexpr int kBinNone = -2;                  // lane without a pixel this step
constexpr int kBinInvalid = -1;               // pair the reference rejects

constexpr int max_classes_for(size_t smem) {
    int nb = 1;
    while (sizeof(unsigned) * (size_t)(nb + 1) * (nb + 1) <= smem) nb++;
    return nb - 1;
}
constexpr int kConfMaxClasses = max_classes_for(kConfMaxSmem);   // 225
static_assert(kConfMaxClasses >= 200, "the private histogram must hold ScanNet200");

// Flat bin of one (pred, gt) pair as numpy computes it, or kBinInvalid where the reference raises: a negative
// label (bincount of a negative value) or pred * nb + gt >= nb^2 (reshape of a longer histogram).  The test is
// on the flat index, so a gt > num_classes that still lands inside counts in the next row, as in numpy.  pr is
// the int64 label plus an int32 offset; where that sum wraps, the exact value lies outside [0, nb) as well.
__device__ __forceinline__ int conf_bin(long long pred, long long gt, int off, int nb) {
    const long long pr = (long long)((unsigned long long)pred + (unsigned long long)(long long)off);
    if (pr < 0 || gt < 0 || pr >= nb) return kBinInvalid;
    const long long room = (long long)nb * nb - pr * nb;   // gt must stay below it
    return gt < room ? (int)(pr * nb + gt) : kBinInvalid;
}

// All 32 lanes call this with the same trip count.
__device__ __forceinline__ void conf_count(unsigned* hist, int bin, int lane, unsigned& n_invalid) {
    const unsigned peers = __match_any_sync(0xffffffffu, bin);
    if (bin >= 0 && lane == __ffs(peers) - 1) atomicAdd(&hist[bin], (unsigned)__popc(peers));
    n_invalid += bin == kBinInvalid;
}

// Four consecutive labels with one 16-byte load (uint8: one 4-byte load; int64: two 16-byte loads).
__device__ __forceinline__ void load4(const int* p, long long (&v)[4]) {
    const int4 a = __ldg(reinterpret_cast<const int4*>(p));
    v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w;
}
__device__ __forceinline__ void load4(const long long* p, long long (&v)[4]) {
    const longlong2 a = __ldg(reinterpret_cast<const longlong2*>(p));
    const longlong2 b = __ldg(reinterpret_cast<const longlong2*>(p) + 1);
    v[0] = a.x; v[1] = a.y; v[2] = b.x; v[3] = b.y;
}
__device__ __forceinline__ void load4(const uint8_t* p, long long (&v)[4]) {
    const uchar4 a = __ldg(reinterpret_cast<const uchar4*>(p));
    v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w;
}

// VEC: both label arrays are aligned to 4 labels; lane = 4 consecutive pixels per step, the N % 4 tail is
// counted by the first warp of the grid.  Otherwise lane = one pixel per step.
template <typename PT, typename GT, bool VEC>
__global__ void __launch_bounds__(kConfThreads) confusion_kernel(long long N, const PT* __restrict__ pred,
                                                                 const GT* __restrict__ gt, int off, int nb,
                                                                 unsigned long long* __restrict__ counts,
                                                                 unsigned* __restrict__ invalid) {
    extern __shared__ unsigned hist[];  // [nb * nb]
    const int nbins = nb * nb;
    for (int i = threadIdx.x; i < nbins; i += kConfThreads) hist[i] = 0u;
    __syncthreads();

    const int lane = threadIdx.x & 31;
    const long long warp = ((long long)blockIdx.x * kConfThreads + threadIdx.x) >> 5;
    const long long nwarps = ((long long)gridDim.x * kConfThreads) >> 5;
    unsigned n_invalid = 0;
    if (VEC) {
        const long long groups = N / kConfVec;
        for (long long base = warp * 32; base < groups; base += nwarps * 32) {
            const long long q = base + lane;
            long long pv[kConfVec], gv[kConfVec];
            if (q < groups) {
                load4(pred + q * kConfVec, pv);
                load4(gt + q * kConfVec, gv);
            }
#pragma unroll
            for (int j = 0; j < kConfVec; j++)
                conf_count(hist, q < groups ? conf_bin(pv[j], gv[j], off, nb) : kBinNone, lane, n_invalid);
        }
        if (warp == 0) {
            const long long p = groups * kConfVec + lane;
            conf_count(hist, p < N ? conf_bin((long long)pred[p], (long long)gt[p], off, nb) : kBinNone, lane,
                       n_invalid);
        }
    } else {
        for (long long base = warp * 32; base < N; base += nwarps * 32) {
            const long long p = base + lane;
            conf_count(hist, p < N ? conf_bin((long long)pred[p], (long long)gt[p], off, nb) : kBinNone, lane,
                       n_invalid);
        }
    }

    const unsigned warp_invalid = __reduce_add_sync(0xffffffffu, n_invalid);
    if (lane == 0 && warp_invalid) atomicAdd(invalid, warp_invalid);
    __syncthreads();
    for (int i = threadIdx.x; i < nbins; i += kConfThreads) {
        const unsigned h = hist[i];
        if (h) atomicAdd(counts + i, (unsigned long long)h);
    }
}

template <typename PT, typename GT>
int launch_confusion_t(long long N, const void* pred_v, const void* gt_v, int off, int nb, uint64_t* counts,
                       uint32_t* invalid, cudaStream_t s) {
    const PT* pred = static_cast<const PT*>(pred_v);
    const GT* gt = static_cast<const GT*>(gt_v);
    // load4 alignment: 16 bytes for int32 / int64 labels, 4 bytes for uint8
    const bool vec = reinterpret_cast<uintptr_t>(pred) % min(kConfVec * sizeof(PT), (size_t)16) == 0 &&
                     reinterpret_cast<uintptr_t>(gt) % min(kConfVec * sizeof(GT), (size_t)16) == 0;
    auto kern = vec ? confusion_kernel<PT, GT, true> : confusion_kernel<PT, GT, false>;
    const size_t smem = sizeof(unsigned) * (size_t)nb * nb;
    static DeviceOnce attr_set;
    if (attr_set.first_use_on_device()) {
        SGB_CUDA(cudaFuncSetAttribute(confusion_kernel<PT, GT, true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                      (int)kConfMaxSmem));
        SGB_CUDA(cudaFuncSetAttribute(confusion_kernel<PT, GT, false>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                      (int)kConfMaxSmem));
    }
    int dev = 0, sms = 0, per_sm = 0;
    SGB_CUDA(cudaGetDevice(&dev));
    SGB_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    SGB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, kConfThreads, smem));
    // Every CTA zeroes and flushes all nb^2 bins, so it gets at least that many pixels (and 8 per thread); the grid
    // never exceeds one wave.  At least one CTA per 2^31 pixels keeps the private uint32 bins exact.
    const long long per_cta = max((long long)kConfThreads * 8, (long long)nb * nb);
    long long blocks = min((long long)max(per_sm, 1) * sms, (N + per_cta - 1) / per_cta);
    blocks = max(blocks, (N >> 31) + 1);
    kern<<<(unsigned)blocks, kConfThreads, smem, s>>>(N, pred, gt, off, nb, (unsigned long long*)counts, invalid);
    SGB_LAUNCH_CHECK("confusion_kernel", 0, s);
    return SGB_OK;
}

template <typename PT>
int launch_confusion_gt(long long N, const void* pred, const void* gt, int32_t gt_dtype, int off, int nb,
                        uint64_t* counts, uint32_t* invalid, cudaStream_t s) {
    switch (gt_dtype) {
        case SGB_LABEL_U8: return launch_confusion_t<PT, uint8_t>(N, pred, gt, off, nb, counts, invalid, s);
        case SGB_LABEL_I32: return launch_confusion_t<PT, int>(N, pred, gt, off, nb, counts, invalid, s);
        default: return launch_confusion_t<PT, long long>(N, pred, gt, off, nb, counts, invalid, s);
    }
}

}  // namespace

}  // namespace sgb

using namespace sgb;

extern "C" {

int sgb_confusion_accumulate(int64_t N, const void* pred, int32_t pred_dtype, const void* gt, int32_t gt_dtype,
                             int32_t pred_offset, int32_t num_classes, uint64_t* counts, uint32_t* invalid,
                             void* stream) {
    if (N < 0) { set_error("sgb_confusion_accumulate: N = %lld < 0", (long long)N); return SGB_E_INVALID; }
    if (pred_dtype != SGB_LABEL_I32 && pred_dtype != SGB_LABEL_I64) {
        set_error("sgb_confusion_accumulate: pred dtype code %d (need SGB_LABEL_I32 or SGB_LABEL_I64)", pred_dtype);
        return SGB_E_INVALID;
    }
    if (gt_dtype != SGB_LABEL_U8 && gt_dtype != SGB_LABEL_I32 && gt_dtype != SGB_LABEL_I64) {
        set_error("sgb_confusion_accumulate: gt dtype code %d (need SGB_LABEL_U8, _I32 or _I64)", gt_dtype);
        return SGB_E_INVALID;
    }
    if (num_classes < 1 || num_classes > kConfMaxClasses) {
        set_error("sgb_confusion_accumulate: num_classes = %d (need 1 <= num_classes <= %d: (num_classes + 1)^2 "
                  "uint32 bins must fit one CTA's shared memory)", num_classes, kConfMaxClasses);
        return SGB_E_INVALID;
    }
    if (!counts || !invalid) { set_error("sgb_confusion_accumulate: null counts / invalid"); return SGB_E_INVALID; }
    if (N > 0 && (!pred || !gt)) { set_error("sgb_confusion_accumulate: null pred / gt"); return SGB_E_INVALID; }
    if (N == 0) return SGB_OK;
    const int nb = num_classes + 1;
    cudaStream_t s = (cudaStream_t)stream;
    if (pred_dtype == SGB_LABEL_I32)
        return launch_confusion_gt<int>((long long)N, pred, gt, gt_dtype, pred_offset, nb, counts, invalid, s);
    return launch_confusion_gt<long long>((long long)N, pred, gt, gt_dtype, pred_offset, nb, counts, invalid, s);
}

}  // extern "C"
