// cfb_tma.cuh -- sm_90a bulk-tensor copy (TMA) + mbarrier primitives used by the level-1 kernels, and the host-side
// tensor-map encoder.  Hand-written PTX (no CUTLASS/CuTe dependency): cp.async.bulk.tensor.2d (SASS: UTMALDG / UTMASTG),
// mbarrier.* (SYNCS), one elected lane per warp issues, every lane of the warp waits.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace cfb {

// ---- device ------------------------------------------------------------------------------------------------------
__device__ __forceinline__ unsigned smem_u32(const void *p) { return (unsigned)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(unsigned bar, unsigned count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" :: "r"(bar), "r"(count) : "memory");
}
// makes the initialised barriers visible to the async (TMA) proxy
__device__ __forceinline__ void mbar_fence_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_expect_tx(unsigned bar, unsigned bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" :: "r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(unsigned bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" :: "r"(bar) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(unsigned bar, unsigned parity) {
    unsigned ok;
    asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                 : "=r"(ok) : "r"(bar), "r"(parity) : "memory");
    return ok != 0;
}
__device__ __forceinline__ void mbar_wait(unsigned bar, unsigned parity) {
    while (!mbar_try_wait(bar, parity)) { }
}
// global (tensor map, element coordinates x, y) -> shared; completion is signalled on `bar` (complete_tx::bytes)
__device__ __forceinline__ void tma_load_2d(unsigned dst, const void *tmap, int x, int y, unsigned bar) {
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];"
                 :: "r"(dst), "l"(tmap), "r"(x), "r"(y), "r"(bar) : "memory");
}
__device__ __forceinline__ void tma_load_3d(unsigned dst, const void *tmap, int x, int y, int z, unsigned bar) {
    asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4}], [%5];"
                 :: "r"(dst), "l"(tmap), "r"(x), "r"(y), "r"(z), "r"(bar) : "memory");
}
// shared -> global (tensor map); completion tracked by bulk async-groups
__device__ __forceinline__ void tma_store_2d(const void *tmap, int x, int y, unsigned src) {
    asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.tile.bulk_group [%0, {%1, %2}], [%3];"
                 :: "l"(tmap), "r"(x), "r"(y), "r"(src) : "memory");
}
__device__ __forceinline__ void tma_store_3d(const void *tmap, int x, int y, int z, unsigned src) {
    asm volatile("cp.async.bulk.tensor.3d.global.shared::cta.tile.bulk_group [%0, {%1, %2, %3}], [%4];"
                 :: "l"(tmap), "r"(x), "r"(y), "r"(z), "r"(src) : "memory");
}
__device__ __forceinline__ void tma_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
// wait until at most N of this thread's bulk groups still READ their shared-memory source
template <int N> __device__ __forceinline__ void tma_wait_read() { asm volatile("cp.async.bulk.wait_group.read %0;" :: "n"(N) : "memory"); }
template <int N> __device__ __forceinline__ void tma_wait_all() { asm volatile("cp.async.bulk.wait_group %0;" :: "n"(N) : "memory"); }
// generic-proxy writes to shared memory (st.shared) -> visible to the async proxy (TMA store)
__device__ __forceinline__ void fence_async_shared() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void prefetch_tmap(const void *tmap) { asm volatile("prefetch.tensormap [%0];" :: "l"(tmap) : "memory"); }

__device__ __forceinline__ uint4 lds128(unsigned addr) {
    uint4 v;
    asm volatile("ld.shared.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(addr));
    return v;
}
__device__ __forceinline__ uint2 lds64(unsigned addr) {
    uint2 v;
    asm volatile("ld.shared.v2.u32 {%0, %1}, [%2];" : "=r"(v.x), "=r"(v.y) : "r"(addr));
    return v;
}
__device__ __forceinline__ unsigned lds32(unsigned addr) {
    unsigned v;
    asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(addr));
    return v;
}
__device__ __forceinline__ unsigned lds_u16(unsigned addr) {
    unsigned v;
    asm volatile("ld.shared.u16 %0, [%1];" : "=r"(v) : "r"(addr));
    return v;
}
__device__ __forceinline__ void sts64(unsigned addr, unsigned a, unsigned b) {
    asm volatile("st.shared.v2.u32 [%0], {%1, %2};" :: "r"(addr), "r"(a), "r"(b) : "memory");
}
__device__ __forceinline__ void sts32(unsigned addr, unsigned a) {
    asm volatile("st.shared.u32 [%0], %1;" :: "r"(addr), "r"(a) : "memory");
}
__device__ __forceinline__ void sts128(unsigned addr, uint4 v) {
    asm volatile("st.shared.v4.u32 [%0], {%1, %2, %3, %4};" :: "r"(addr), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}

// ---- host ----------------------------------------------------------------------------------------------------------
// 2-D (or 3-D) tiled tensor map over 32-bit (or, elem_bytes = 8, 64-bit: boxes up to 2 KB wide) elements.  row_bytes /
// pitch / box_bytes in BYTES (multiples of elem_bytes / 16 / 16).
// The driver entry point is resolved through the runtime (cudart is linked statically; libcuda is never linked).
cudaError_t tmap_encode_2d(CUtensorMap *out, const void *base, uint64_t row_bytes, uint64_t rows, uint64_t pitch_bytes,
                           uint32_t box_bytes, uint32_t box_rows, int elem_bytes = 4);
cudaError_t tmap_encode_3d(CUtensorMap *out, const void *base, uint64_t row_bytes, uint64_t rows, uint64_t pitch_bytes,
                           uint64_t planes, uint64_t plane_bytes, uint32_t box_bytes, uint32_t box_rows, uint32_t box_planes);

}  // namespace cfb
