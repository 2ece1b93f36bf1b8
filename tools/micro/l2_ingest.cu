// Microbenchmark: how fast can ONE SM pull an L2-resident weight stream into shared memory?
//   modes: 0 = 1-D bulk copies issued by one thread; 1 = by two threads (two rings); 2 = cluster multicast (every CTA
//   of the cluster issues 1/csz of each slot to all members); 3 = ld.global.v4 + st.shared by all threads.
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -Icrazyara_b200/csrc -Iinclude tools/micro/l2_ingest.cu -o build/l2_ingest
#include <cuda.h>
#include <cstdio>
#include <cstdlib>
#include <vector>
#include "sm90_prims.cuh"
using namespace ara;

__device__ __forceinline__ void bulk_load_1d_mc(void* smem_dst, const void* gsrc, uint32_t bytes, uint64_t* bar, uint16_t mask) {
    asm volatile(
        "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster [%0], [%1], %2, [%3], %4;"
        ::"r"(smem_u32(smem_dst)), "l"(gsrc), "r"(bytes), "r"(smem_u32(bar)), "h"(mask)
        : "memory");
}
__device__ __forceinline__ uint32_t cluster_ctarank() {
    uint32_t r;
    asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
    return r;
}

// slot bytes = `slot`; `ring` slots; total `n_slots` per CTA
__global__ void __launch_bounds__(288, 1) ingest_kernel(const uint8_t* flat, size_t flat_bytes, int mode, int slot, int ring,
                                                        int n_slots, int csz, unsigned long long* cycles, int nprod) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint64_t* full = reinterpret_cast<uint64_t*>(smem + ring * slot);
    uint64_t* empty = full + 32;
    const uint32_t rank = csz > 1 ? cluster_ctarank() : 0;
    if (threadIdx.x == 0) {
        for (int i = 0; i < ring; ++i) mbar_init(&full[i], 1), mbar_init(&empty[i], csz);
        fence_mbar_init();
    }
    __syncthreads();
    if (csz > 1) cluster_sync_all();
    const long long t0 = clock64();
    const size_t base = (static_cast<size_t>(blockIdx.x / csz) * 7919 * 4096) % (flat_bytes / 2);
    if (mode == 3) {
        // all threads: 16-byte loads, coalesced, straight to shared memory
        const int per = slot / 16;
        for (int i = 0; i < n_slots; ++i) {
            const uint4* src = reinterpret_cast<const uint4*>(flat + (base + static_cast<size_t>(i) * slot) % (flat_bytes - slot));
            uint4* dst = reinterpret_cast<uint4*>(smem + (i % ring) * slot);
            for (int j = threadIdx.x; j < per; j += blockDim.x) dst[j] = __ldcg(src + j);
        }
    } else if (threadIdx.x == 0 || (mode == 1 && threadIdx.x >= 64 && (threadIdx.x & 31) == 0 && (threadIdx.x >> 5) - 1 < nprod)) {
        const int lanes = mode == 1 ? nprod : 1, me = threadIdx.x == 0 ? 0 : (threadIdx.x >> 5) - 1;
        for (int i = me; i < n_slots; i += lanes) {
            const int s = i % ring;
            mbar_wait(&empty[s], ((i / ring) & 1) ^ 1);
            mbar_arrive_expect_tx(&full[s], slot);
            const uint8_t* src = flat + (base + static_cast<size_t>(i) * slot) % (flat_bytes - slot);
            if (mode == 2) {
                const int piece = slot / csz;
                bulk_load_1d_mc(smem + s * slot + rank * piece, src + rank * piece, piece, &full[s], static_cast<uint16_t>((1u << csz) - 1));
            } else {
                bulk_load_1d(smem + s * slot, src, slot, &full[s]);
            }
        }
    } else if (threadIdx.x == 32) {  // consumer: frees the slot (in every CTA of the cluster) as soon as it is full
        for (int i = 0; i < n_slots; ++i) {
            const int s = i % ring;
            mbar_wait(&full[s], (i / ring) & 1);
            if (csz > 1) {
                for (int c = 0; c < csz; ++c) mbar_arrive_cluster(cluster_map(&empty[s], c));
            } else {
                mbar_arrive(&empty[s]);
            }
        }
    }
    __syncthreads();
    if (csz > 1) cluster_sync_all();
    const long long t1 = clock64();
    if (mode == 3 && smem[threadIdx.x * 16] == 77) cycles[512 + threadIdx.x] = 1;  // keeps the stores alive
    if (threadIdx.x == 0) cycles[blockIdx.x] = static_cast<unsigned long long>(t1 - t0);
}

int main() {
    const size_t flat_bytes = 16u << 20;  // L2-resident
    uint8_t* flat;
    cudaMalloc(&flat, flat_bytes);
    cudaMemset(flat, 1, flat_bytes);
    unsigned long long* d_cycles;
    cudaMalloc(&d_cycles, 1024 * sizeof(unsigned long long));
    cudaFuncSetAttribute(ingest_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
    cudaFuncSetAttribute(ingest_kernel, cudaFuncAttributeNonPortableClusterSizeAllowed, 1);
    struct Cfg { int mode, slot, ring, csz, grid, nprod; };
    std::vector<Cfg> cfgs;
    for (int slot : {8192, 16384, 32768, 65536}) cfgs.push_back({0, slot, 196608 / slot > 8 ? 8 : 196608 / slot, 1, 64, 1});
    for (int np : {2, 3, 4, 6}) {
        cfgs.push_back({1, 8192, 12, 1, 64, np});
        cfgs.push_back({1, 16384, 12, 1, 64, np});
        cfgs.push_back({1, 16384, 12, 1, 132, np});
    }
    cfgs.push_back({1, 32768, 6, 1, 64, 2});
    cfgs.push_back({1, 32768, 6, 1, 64, 3});
    for (const Cfg& c : cfgs) {
        const int n_slots = (8 << 20) / c.slot;  // 8 MB per CTA
        cudaLaunchConfig_t lc = {};
        lc.gridDim = dim3(c.grid);
        lc.blockDim = dim3(288);
        lc.dynamicSmemBytes = c.ring * c.slot + 2048;
        cudaLaunchAttribute at[1];
        at[0].id = cudaLaunchAttributeClusterDimension;
        at[0].val.clusterDim.x = c.csz;
        at[0].val.clusterDim.y = 1;
        at[0].val.clusterDim.z = 1;
        lc.attrs = at;
        lc.numAttrs = 1;
        double best = 0;
        for (int rep = 0; rep < 3; ++rep) {
            cudaError_t e = cudaLaunchKernelEx(&lc, ingest_kernel, (const uint8_t*)flat, flat_bytes, c.mode, c.slot, c.ring, n_slots, c.csz, d_cycles, c.nprod);
            if (e != cudaSuccess || (e = cudaDeviceSynchronize()) != cudaSuccess) {
                printf("mode %d slot %d ring %d csz %d grid %d: %s\n", c.mode, c.slot, c.ring, c.csz, c.grid, cudaGetErrorString(e));
                return 1;
            }
            std::vector<unsigned long long> h(c.grid);
            cudaMemcpy(h.data(), d_cycles, c.grid * sizeof(unsigned long long), cudaMemcpyDeviceToHost);
            unsigned long long mx = 0;
            for (auto v : h) mx = v > mx ? v : mx;
            const double bpc = static_cast<double>(n_slots) * c.slot / static_cast<double>(mx);
            best = bpc > best ? bpc : best;
        }
        printf("mode %d slot %6d ring %2d nprod %d csz %d grid %3d: %6.1f B/clk per SM (slowest CTA), %7.0f B/clk chip\n", c.mode, c.slot, c.ring,
               c.nprod, c.csz, c.grid, best, best * c.grid);
    }
    return 0;
}
