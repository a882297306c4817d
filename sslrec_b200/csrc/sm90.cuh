// Hopper (sm_90a) primitives shared by the InfoNCE contraction kernels (nce_gemm.cu, nce_gemm_tc.cu, nce_gemm_f16x3.cu):
// mbarriers, bulk and tensor-map copies, wgmma synchronisation, named barriers, and on the host the tensor-map encoder
// and the once-per-device launch configuration.  Kept out of common.cuh, which is also compiled for the host alone.
#pragma once
#include <cuda.h>

#include "common.cuh"

namespace ssl {

// ---- device side ----
__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t *bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t *bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t *bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t parity) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "LAB_WAIT:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra DONE;\n"
        "bra LAB_WAIT;\n"
        "DONE:\n"
        "}\n" ::"r"(smem_u32(bar)), "r"(parity) : "memory");
}
// 1-D bulk copy global -> shared, completing on ``bar``
__device__ __forceinline__ void bulk_g2s(void *dst, const void *src, uint32_t bytes, uint64_t *bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst)),
                 "l"(src), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}
// box (c0, c1) of a 2-D tensor map -> shared, completing on ``bar``
__device__ __forceinline__ void tma_load_2d(void *dst, const CUtensorMap *map, int c0, int c1, uint64_t *bar) {
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
                 ::"r"(smem_u32(dst)), "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1) : "memory");
}
__device__ __forceinline__ float ex2(float x) {
    float y;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}

__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_wait0() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }
// named barriers over the two consumer warpgroups (256 threads); id 0 is __syncthreads'
__device__ __forceinline__ void named_sync(int id) { asm volatile("bar.sync %0, 256;" ::"r"(id) : "memory"); }
__device__ __forceinline__ void named_arrive(int id) { asm volatile("bar.arrive %0, 256;" ::"r"(id) : "memory"); }
// keeps registers an asynchronous wgmma reads or writes live (and in place) up to this point
template <int N>
__device__ __forceinline__ void reg_fence(float (&r)[N]) {
#pragma unroll
    for (int i = 0; i < N; ++i) asm volatile("" : "+f"(r[i])::"memory");
}
template <int N>
__device__ __forceinline__ void reg_fence(uint32_t (&r)[N]) {
#pragma unroll
    for (int i = 0; i < N; ++i) asm volatile("" : "+r"(r[i])::"memory");
}

// ---- host side ----
// cuTensorMapEncodeTiled through the driver entry point (no link-time libcuda dependency); nullptr when the driver lacks it
typedef CUresult (*EncodeTiledFn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *, const cuuint64_t *,
                                  const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

inline EncodeTiledFn encode_tiled_fn() {
    static EncodeTiledFn fn = nullptr;
    if (fn == nullptr) {
        void *p = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess)
            fn = reinterpret_cast<EncodeTiledFn>(p);
    }
    return fn;
}

// A 2-D tensor map over [rows, cols] elements of ``type``, rows ``pitch_bytes`` apart, read in boxes of box_cols x box_rows
// with ``swizzle``; out-of-range rows / columns read as 0
inline int make_map_2d(CUtensorMap *map, CUtensorMapDataType type, const void *base, int64_t rows, int64_t cols, int64_t pitch_bytes,
                       int box_cols, int box_rows, CUtensorMapSwizzle swizzle) {
    EncodeTiledFn fn = encode_tiled_fn();
    if (fn == nullptr) {
        set_error("cuTensorMapEncodeTiled is not available from this driver");
        return SSL_E_CUDA;
    }
    cuuint64_t gdim[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
    cuuint64_t gstride[1] = {(cuuint64_t)pitch_bytes};
    cuuint32_t box[2] = {(cuuint32_t)box_cols, (cuuint32_t)box_rows};
    cuuint32_t estr[2] = {1u, 1u};
    CUresult r = fn(map, type, 2, const_cast<void *>(base), gdim, gstride, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle,
                    CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) {
        set_error("cuTensorMapEncodeTiled failed with CUresult %d", (int)r);
        return SSL_E_CUDA;
    }
    return SSL_OK;
}

// Before a launch of ``Kernel`` with ``smem`` bytes of dynamic shared memory: sets its limit on the current device the first
// time, and returns that device's SM count in *n_sm.  cudaFuncSetAttribute is per device and per kernel, so the statics are
// keyed on the kernel itself (a non-type template parameter): instantiations that share a function type, such as one kernel
// at two dims, each get their own.
template <auto Kernel>
int configure_once(size_t smem, int *n_sm) {
    static bool configured[64] = {};
    static int sm_count[64] = {};
    int dev = 0;
    SSL_CUDA(cudaGetDevice(&dev));
    if (dev >= 0 && dev < 64 && configured[dev]) {
        *n_sm = sm_count[dev];
        return SSL_OK;
    }
    SSL_CUDA(cudaFuncSetAttribute(Kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    SSL_CUDA(cudaDeviceGetAttribute(n_sm, cudaDevAttrMultiProcessorCount, dev));
    if (dev >= 0 && dev < 64) {
        sm_count[dev] = *n_sm;
        configured[dev] = true;
    }
    return SSL_OK;
}

// the grid of a persistent kernel: one CTA per SM, each looping over units blockIdx.x, + gridDim.x, ...
inline int64_t persistent_grid(int64_t units, int n_sm) { return units < n_sm ? units : n_sm; }

}  // namespace ssl
