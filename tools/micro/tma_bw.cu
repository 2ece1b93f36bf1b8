// Microbenchmark: per-SM L2->shared bandwidth of TMA tensor loads vs 1-D bulk copies (weights resident in L2).
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -Icrazyara_b200/csrc -Iinclude tools/micro/tma_bw.cu -o build/tma_bw -lcuda
#include <cuda.h>
#include <cuda_fp16.h>
#include <cstdio>
#include <cstdlib>
#include <vector>
#include "sm90_prims.cuh"
using namespace ara;

typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

constexpr int kSlot = 16384;

// mode 0: 2 boxes {64 K, 64 rows} per slot from W1 [rows][256]; mode 1: 1 box {64 K, 128 rows} from W2 [256][C2];
// mode 2: one 1-D bulk copy of 16 KB; mode 3: 16 x 1-D bulk copies of 1 KB
__global__ void __launch_bounds__(64, 1) tma_bw_kernel(const __grid_constant__ CUtensorMap tm1, const __grid_constant__ CUtensorMap tm2,
                                                       const uint8_t* flat, int mode, int ring, int n_slots_total, int rows_total,
                                                       unsigned long long* cycles) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint64_t* full = reinterpret_cast<uint64_t*>(smem + ring * kSlot);
    uint64_t* empty = full + 16;
    if (threadIdx.x == 0) {
        for (int i = 0; i < ring; ++i) mbar_init(&full[i], 1), mbar_init(&empty[i], 1);
        fence_mbar_init();
    }
    __syncthreads();
    const long long t0 = clock64();
    if (threadIdx.x == 0) {  // producer
        for (int i = 0; i < n_slots_total; ++i) {
            const int s = i % ring;
            mbar_wait(&empty[s], ((i / ring) & 1) ^ 1);
            mbar_arrive_expect_tx(&full[s], kSlot);
            uint8_t* dst = smem + s * kSlot;
            const int chunk = i >> 1, h = i & 1;
            if (mode == 0) {
                const int row = (chunk * 64) % rows_total;
                tma_load_2d(dst, &tm1, &full[s], (2 * h) * 64, row);
                tma_load_2d(dst + 8192, &tm1, &full[s], (2 * h + 1) * 64, row);
            } else if (mode == 1) {
                const int k = (chunk * 64) % rows_total;
                tma_load_2d(dst, &tm2, &full[s], k, h * 128);
            } else if (mode == 2) {
                bulk_load_1d(dst, flat + (static_cast<size_t>(i) * kSlot) % (static_cast<size_t>(rows_total) * 512), kSlot, &full[s]);
            } else {
                for (int q = 0; q < 16; ++q)
                    bulk_load_1d(dst + q * 1024, flat + (static_cast<size_t>(i) * kSlot + q * 1024) % (static_cast<size_t>(rows_total) * 512), 1024, &full[s]);
            }
        }
    } else if (threadIdx.x == 32) {  // consumer: frees the slot as soon as it is full
        for (int i = 0; i < n_slots_total; ++i) {
            const int s = i % ring;
            mbar_wait(&full[s], (i / ring) & 1);
            mbar_arrive(&empty[s]);
        }
    }
    __syncthreads();
    if (threadIdx.x == 0 && blockIdx.x == 0) *cycles = static_cast<unsigned long long>(clock64() - t0);
}

int main() {
    const int rows = 6656;  // stacked operating channels of RISEv2 (sum of 64-padded c_op)
    void* fn = nullptr;
    cudaDriverEntryPointQueryResult q;
    cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &q);
    PFN_encodeTiled enc = reinterpret_cast<PFN_encodeTiled>(fn);
    __half *w1, *w2;
    cudaMalloc(&w1, static_cast<size_t>(rows) * 256 * 2);
    cudaMalloc(&w2, static_cast<size_t>(rows) * 256 * 2);
    cudaMemset(w1, 0, static_cast<size_t>(rows) * 256 * 2);
    cudaMemset(w2, 0, static_cast<size_t>(rows) * 256 * 2);
    CUtensorMap tm1, tm2;
    {
        cuuint64_t dims[2] = {256, (cuuint64_t)rows};
        cuuint64_t strides[1] = {512};
        cuuint32_t box[2] = {64, 64};
        cuuint32_t es[2] = {1, 1};
        enc(&tm1, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, w1, dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
            CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    }
    {
        cuuint64_t dims[2] = {(cuuint64_t)rows, 256};
        cuuint64_t strides[1] = {(cuuint64_t)rows * 2};
        cuuint32_t box[2] = {64, 128};
        cuuint32_t es[2] = {1, 1};
        enc(&tm2, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, w2, dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
            CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    }
    unsigned long long* d_cyc;
    cudaMalloc(&d_cyc, 8);
    cudaFuncSetAttribute(tma_bw_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
    const int n_slots = 2 * 104 * 2;  // about two trunk passes of W1 half chunks
    const char* names[4] = {"tensor 2x{64x64} (W1 rows)", "tensor {64x128} (W2 cols)", "bulk 1-D 16 KB", "bulk 1-D 16 x 1 KB"};
    for (int grid : {1, 32, 132})
        for (int mode = 0; mode < 4; ++mode)
            for (int ring : {2, 3, 6, 10}) {
                unsigned long long cyc = 0;
                for (int rep = 0; rep < 3; ++rep) {
                    tma_bw_kernel<<<grid, 64, ring * kSlot + 2048>>>(tm1, tm2, reinterpret_cast<const uint8_t*>(w1), mode, ring, n_slots,
                                                                      rows, d_cyc);
                    cudaDeviceSynchronize();
                }
                cudaMemcpy(&cyc, d_cyc, 8, cudaMemcpyDeviceToHost);
                cudaError_t e = cudaGetLastError();
                printf("grid %3d  %-28s ring %2d: %8.1f kcycles  %6.1f B/clk per SM%s\n", grid, names[mode], ring, cyc / 1e3,
                       static_cast<double>(n_slots) * kSlot / cyc, e == cudaSuccess ? "" : cudaGetErrorString(e));
            }
    return 0;
}
