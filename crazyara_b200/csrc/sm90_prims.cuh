// sm_90a primitives: mbarrier, TMA (cp.async.bulk.tensor), bulk copies, clusters, wgmma descriptors and fences
// (the wgmma instructions: wgmma.cuh).
// Hand-written inline PTX; no CUTLASS/CuTe dependency.  Only meaningful when compiled for sm_90a.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <cuda_fp16.h>
#include <stdint.h>

namespace ara {

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
    return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

// ---------------------------------------------------------------- programmatic dependent launch (PDL)
// wait: block until the prerequisite grid has completed and its memory is visible (no-op without the launch attribute)
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
// launch_dependents: allow the next kernel in the stream to start its prologue while this grid is still running
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

// ---------------------------------------------------------------- mbarrier
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_mbar_init() {
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n\t.reg .pred P1;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 P1, [%1], %2, %3;\n\t"
        "selp.b32 %0, 1, 0, P1;\n\t}"
        : "=r"(ok)
        : "r"(smem_u32(bar)), "r"(parity), "r"(0x989680u)  // suspend-time hint: sleep in hardware instead of
        : "memory");                                        // re-polling (polls cost issue slots and smem wavefronts)
    return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    while (!mbar_try_wait(bar, parity)) {
    }
}

// for waiters that run far ahead of their consumer (weight producers): back off between polls so that the polling
// does not take issue slots from the warps doing the work
__device__ __forceinline__ void mbar_wait_relaxed(uint64_t* bar, uint32_t parity) {
    while (!mbar_try_wait(bar, parity)) __nanosleep(200);
}

// ---------------------------------------------------------------- thread-block clusters / distributed shared memory
__device__ __forceinline__ void cluster_sync_all() {  // every thread of every CTA of the cluster
    asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}
// shared-memory address of `local` in the CTA with rank `cta` of this cluster
__device__ __forceinline__ uint32_t cluster_map(const void* local, uint32_t cta) {
    uint32_t r;
    asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(smem_u32(local)), "r"(cta));
    return r;
}
__device__ __forceinline__ uint32_t cluster_ctarank() {
    uint32_t r;
    asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
    return r;
}
__device__ __forceinline__ void st_cluster_v4(uint32_t raddr, uint32_t a, uint32_t b, uint32_t c, uint32_t d) {
    asm volatile("st.shared::cluster.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(raddr), "r"(a), "r"(b), "r"(c), "r"(d) : "memory");
}
// store into another CTA's shared memory that completes 4 bytes on the receiver's mbarrier (raddr and rbar: cluster_map
// addresses in the same CTA).  The receiver's wait on the barrier phase sees the value; no fence is issued.
__device__ __forceinline__ void st_async_cluster_b32(uint32_t raddr, uint32_t v, uint32_t rbar) {
    asm volatile("st.async.shared::cluster.mbarrier::complete_tx::bytes.b32 [%0], %1, [%2];" ::"r"(raddr), "r"(v), "r"(rbar)
                 : "memory");
}
// bulk copy of this CTA's shared memory into another CTA's (dst and bar: cluster_map addresses); completes `bytes` on
// the receiver's mbarrier.  Sizes and addresses are multiples of 16.
__device__ __forceinline__ void bulk_copy_to_cta(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
    asm volatile("cp.async.bulk.shared::cluster.shared::cta.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst),
                 "r"(smem_u32(src)), "r"(bytes), "r"(bar)
                 : "memory");
}
// arrive on an mbarrier of another CTA of the cluster; release at cluster scope: the arriving thread's earlier
// remote stores are visible to whoever acquires the barrier phase
__device__ __forceinline__ void mbar_arrive_cluster(uint32_t rbar) {
    asm volatile("mbarrier.arrive.release.cluster.shared::cluster.b64 _, [%0];" ::"r"(rbar) : "memory");
}
// arrive on an mbarrier of another CTA that tells it a buffer is free: this CTA's reads of the buffer are complete and
// it publishes no data, so the arrival releases at CTA scope only.  The cluster-scope release above costs a
// MEMBAR.ALL.GPU per arrival; data goes with st_async_cluster_b32 or a bulk copy instead.
__device__ __forceinline__ void mbar_arrive_cluster_free(uint32_t rbar) {
    asm volatile("mbarrier.arrive.shared::cluster.b64 _, [%0];" ::"r"(rbar) : "memory");
}
__device__ __forceinline__ void mbar_wait_cluster(uint64_t* bar, uint32_t parity) {
    uint32_t ok = 0;
    while (!ok) {
        asm volatile(
            "{\n\t.reg .pred P1;\n\t"
            "mbarrier.try_wait.parity.acquire.cluster.shared::cta.b64 P1, [%1], %2;\n\t"
            "selp.b32 %0, 1, 0, P1;\n\t}"
            : "=r"(ok)
            : "r"(smem_u32(bar)), "r"(parity)
            : "memory");
    }
}

// ---------------------------------------------------------------- TMA
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* m) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
__device__ __forceinline__ void tma_load_2d(void* smem_dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
        ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
        : "memory");
}
__device__ __forceinline__ void tma_load_4d(void* smem_dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1,
                                            int c2, int c3) {
    asm volatile(
        "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], "
        "[%2];" ::"r"(smem_u32(smem_dst)),
        "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
        : "memory");
}

// ---------------------------------------------------------------- bulk copies, wgmma descriptors and fences
// 1-D bulk copy global -> shared (no tensor map): bytes and both addresses are multiples of 16
__device__ __forceinline__ void bulk_load_1d(void* smem_dst, const void* gsrc, uint32_t bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                     smem_u32(smem_dst)),
                 "l"(gsrc), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}

// generic-proxy shared-memory writes of this thread become visible to the async proxy (wgmma / bulk copies)
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// K-major, SWIZZLE_128B shared-memory matrix descriptor of wgmma (sm_90).
// Canonical layout ((8,n),(T,2)):((8T,SBO),(1,T)), T = 8 halfs: rows are 128 B apart, 8-row groups SBO apart.
// The tile base is 1 KB aligned; a K step of 16 halfs advances the start address by 32 B.
__device__ __forceinline__ uint64_t wgmma_desc_k_sw128(uint32_t saddr, uint32_t sbo_bytes) {
    uint64_t d = 0;
    d |= static_cast<uint64_t>((saddr & 0x3FFFF) >> 4);             // start address  [0,14)
    d |= static_cast<uint64_t>(1) << 16;                            // LBO (ignored for swizzled K-major) [16,30)
    d |= static_cast<uint64_t>((sbo_bytes >> 4) & 0x3FFF) << 32;    // SBO            [32,46)
    d |= static_cast<uint64_t>(1) << 62;                            // layout type: SWIZZLE_128B
    return d;
}

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// pins the accumulator registers in place around a wait: ordinary code must not touch them while a wgmma owns them
template <int R>
__device__ __forceinline__ void wgmma_fence_regs(float (&d)[R]) {
#pragma unroll
    for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

}  // namespace ara
