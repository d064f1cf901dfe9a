// TMA plumbing: mbarrier and bulk / tensor copy wrappers for the kernels, tensor-map encoding for their launchers.
#pragma once
#include <cstdint>
#include <cuda.h>  // CUtensorMap (types only: the encoder is fetched through cudaGetDriverEntryPoint)
#include <cuda_runtime.h>

namespace sgb {

using TensorMapEncodeFn = CUresult (*)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                       const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                       CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
// cuTensorMapEncodeTiled through the runtime's driver entry point (no libcuda link); nullptr when unavailable.
inline TensorMapEncodeFn tensor_map_encoder() {
    static const TensorMapEncodeFn encode = [] {
        void* fn = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &q) != cudaSuccess ||
            q != cudaDriverEntryPointSuccess)
            fn = nullptr;
        return (TensorMapEncodeFn)fn;
    }();
    return encode;
}

// Tiled tensor map of `rank` dimensions, innermost first: dims[rank] and box[rank] in elements, strides[rank - 1] in
// bytes (the innermost dimension is dense).  Unit element strides, no interleave, 128-byte L2 promotion, out-of-range
// elements read as zeros.  False when the driver entry point is missing or rejects the layout.
inline bool encode_tiled_map(CUtensorMap* map, CUtensorMapDataType type, int rank, const void* base,
                             const cuuint64_t* dims, const cuuint64_t* strides, const cuuint32_t* box,
                             CUtensorMapSwizzle swizzle) {
    const TensorMapEncodeFn encode = tensor_map_encoder();
    const cuuint32_t estr[5] = {1, 1, 1, 1, 1};  // a tensor map has at most 5 dimensions
    return encode &&
           encode(map, type, (cuuint32_t)rank, const_cast<void*>(base), dims, strides, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

#ifdef __CUDACC__
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
    return (uint32_t)__cvta_generic_to_shared(p);
}
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_fence_init() {
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
                 : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
// Waits for the phase with the given parity.  try_wait sleeps in hardware between polls; a bounded
// spin turns a protocol bug into a trap (launch failure) instead of a hung GPU.
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    uint32_t done = 0;
    for (uint32_t spins = 0; !done; spins++) {
        asm volatile(
            "{\n\t.reg .pred p;\n\t"
            "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
            "selp.u32 %0, 1, 0, p;\n\t}"
            : "=r"(done)
            : "r"(smem_u32(bar)), "r"(parity)
            : "memory");
        if (spins > (1u << 24)) __trap();
    }
}
// 1-D bulk copy global -> shared through the TMA engine (SASS: UBLKCP); dst/src 16-B aligned,
// bytes a multiple of 16; completion is signalled on `bar` as transaction bytes.
__device__ __forceinline__ void bulk_g2s(void* dst_smem, const void* src_gmem, uint32_t bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                     smem_u32(dst_smem)),
                 "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}
// 2-D tensor tile global -> shared (SASS: UTMALDG): box corner (x, y) in elements, out-of-range elements arrive as
// zeros; completion is signalled on `bar` as the box's bytes.
__device__ __forceinline__ void tma_tile2d_g2s(void* dst_smem, const CUtensorMap* map, int x, int y, uint64_t* bar) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];" ::"r"(
            smem_u32(dst_smem)),
        "l"(reinterpret_cast<uint64_t>(map)), "r"(x), "r"(y), "r"(smem_u32(bar))
        : "memory");
}
// 3-D tensor tile global -> shared through the TMA engine (SASS: UTMALDG): box corner (x, y, z) in elements, out-of-range
// elements arrive as zeros; completion is signalled on `bar` as the box's bytes.  dst 128-byte aligned.
__device__ __forceinline__ void tma_tile3d_g2s(void* dst_smem, const CUtensorMap* map, int x, int y, int z, uint64_t* bar) {
    asm volatile(
        "cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4}], [%5];" ::"r"(
            smem_u32(dst_smem)),
        "l"(reinterpret_cast<uint64_t>(map)), "r"(x), "r"(y), "r"(z), "r"(smem_u32(bar))
        : "memory");
}
// 3-D tensor tile shared -> global through the TMA engine (SASS: UTMASTG), committed to this thread's bulk group: box
// corner (x, y, z) in elements, elements outside the tensor are not written.  src 16-byte aligned; the generic-proxy
// writes that filled it must be ordered before by fence_proxy_async_smem.
__device__ __forceinline__ void tma_store3d_s2g(const CUtensorMap* map, int x, int y, int z, const void* src_smem) {
    asm volatile("cp.async.bulk.tensor.3d.global.shared::cta.bulk_group [%0, {%1, %2, %3}], [%4];" ::"l"(
                     reinterpret_cast<uint64_t>(map)),
                 "r"(x), "r"(y), "r"(z), "r"(smem_u32(src_smem))
                 : "memory");
    asm volatile("cp.async.bulk.commit_group;" ::: "memory");
}
// Waits until this thread's committed bulk stores have read their shared-memory sources (the buffer may be rewritten).
__device__ __forceinline__ void bulk_wait_read_all() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
// Waits until this thread's committed bulk stores have completed.
__device__ __forceinline__ void bulk_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }
// 4-byte cp.async global -> shared; src_bytes 0 writes a zero instead of reading src.
__device__ __forceinline__ void cp_async4(void* dst_smem, const void* src, int src_bytes) {
    asm volatile("cp.async.ca.shared.global [%0], [%1], 4, %2;" ::"r"(smem_u32(dst_smem)), "l"(src), "r"(src_bytes)
                 : "memory");
}
// Arrives on `bar` once every cp.async this thread issued so far has landed (the arrival is part of the init count).
__device__ __forceinline__ void cp_async_mbar_arrive_noinc(uint64_t* bar) {
    asm volatile("cp.async.mbarrier.arrive.noinc.shared::cta.b64 [%0];" ::"r"(smem_u32(bar)) : "memory");
}
// Orders this thread's earlier generic-proxy shared-memory accesses before later async-proxy (TMA) writes.
__device__ __forceinline__ void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
#endif

}  // namespace sgb
