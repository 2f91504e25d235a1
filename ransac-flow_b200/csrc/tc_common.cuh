// mbarrier / TMA / wgmma building blocks of the tensor-core translation unit (sm_90a): PTX wrappers, shared-memory matrix
// descriptors and the cached tensor-map encoder.
#pragma once
#include <cuda.h>
#include <cuda_fp16.h>

#include "common.cuh"
#include "wgmma.cuh"

namespace rf {

constexpr int TC_BK = 32;                 // fp32 elements per 128-byte swizzle row
constexpr int TC_BK_F16 = 64;             // fp16 elements per 128-byte swizzle row
constexpr int TC_A_BYTES = 128 * 128;     // 128 rows x 128 B


// ------------------------------------------------------------------ PTX wrappers
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(ok) : "r"(smem_u32(bar)), "r"(parity) : "memory");
    return ok != 0;
}
// bounded wait: a lost arrival becomes a CUDA error (trap) instead of a hung GPU
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    for (uint32_t spin = 0; !mbar_try_wait(bar, parity); ++spin)
        if (spin > (1u << 26)) __trap();
}
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

__device__ __forceinline__ void tma_load_2d(void* smem_dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1) {
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
                 ::"r"(smem_u32(smem_dst)), "l"((uint64_t)map), "r"(smem_u32(bar)), "r"(c0), "r"(c1) : "memory");
}
__device__ __forceinline__ void tma_load_3d(void* smem_dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1, int c2) {
    asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
                 ::"r"(smem_u32(smem_dst)), "l"((uint64_t)map), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2) : "memory");
}
__device__ __forceinline__ void tma_load_4d(void* smem_dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1, int c2, int c3) {
    asm volatile("cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
                 ::"r"(smem_u32(smem_dst)), "l"((uint64_t)map), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3) : "memory");
}
// shared -> global tensor stores (the map's bounds clip the box), committed as one bulk group per call of bulk_commit
__device__ __forceinline__ void tma_store_3d(const CUtensorMap* map, const void* smem_src, int c0, int c1, int c2) {
    asm volatile("cp.async.bulk.tensor.3d.global.shared::cta.bulk_group [%0, {%2, %3, %4}], [%1];"
                 ::"l"((uint64_t)map), "r"(smem_u32(smem_src)), "r"(c0), "r"(c1), "r"(c2) : "memory");
}
__device__ __forceinline__ void tma_store_4d(const CUtensorMap* map, const void* smem_src, int c0, int c1, int c2, int c3) {
    asm volatile("cp.async.bulk.tensor.4d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5}], [%1];"
                 ::"l"((uint64_t)map), "r"(smem_u32(smem_src)), "r"(c0), "r"(c1), "r"(c2), "r"(c3) : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
// every committed store has finished reading shared memory (the source may be overwritten)
__device__ __forceinline__ void bulk_wait_read() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
// every committed store is complete
__device__ __forceinline__ void bulk_wait() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* map) {
    asm volatile("prefetch.tensormap [%0];" ::"l"((uint64_t)map) : "memory");
}

// wgmma shared-memory matrix descriptor: K-major tile, 128-byte swizzle, 8-row atoms 1024 B apart.  Advancing K by 32 bytes
// inside the atom is +2 on the start-address field.
__device__ __forceinline__ uint64_t wg_desc(uint32_t saddr) {
    uint64_t d = 0;
    d |= (uint64_t)((saddr & 0x3FFFFu) >> 4);          // start address, bits [0,14)
    d |= (uint64_t)1 << 16;                            // leading byte offset (unused for swizzled K-major), bits [16,30)
    d |= (uint64_t)(1024 >> 4) << 32;                  // stride byte offset between 8-row groups, bits [32,46)
    d |= (uint64_t)1 << 62;                            // layout type SWIZZLE_128B, bits [62,64)
    return d;
}
__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wg_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from touching accumulator registers across the asynchronous wgmma window
template <int N>
__device__ __forceinline__ void wg_fence_regs(float (&d)[N]) {
#pragma unroll
    for (int i = 0; i < N; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// cached cuTensorMapEncodeTiled (gemm_tc.cu): fp32 (esize 4) or fp16 (esize 2) tensor (d0 innermost, d1, d2[, d3]), dense strides
// except the outermost one of the 4-D form (`plane_bytes`), box of (b0, b1, b2[, b3]) ELEMENTS LOADED, traversal stride `es` on
// d1 / d2, 128-byte swizzle, zero fill out of bounds
int get_map(CUtensorMap* out, const void* ptr, unsigned long long d0, unsigned long long d1, unsigned long long d2,
            unsigned b0, unsigned b1, unsigned b2, unsigned es_ = 1, unsigned esize = 4);
int get_map4(CUtensorMap* out, const void* ptr, unsigned long long d0, unsigned long long d1, unsigned long long d2, unsigned long long d3,
             unsigned long long plane_bytes, unsigned b0, unsigned b1, unsigned b2, unsigned b3, unsigned es_, unsigned esize);
int pick_tw(int Ho, int Wo);

}  // namespace rf
