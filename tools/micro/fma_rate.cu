// Microbenchmark: issue rate of FFMA, the fp16 x fp16 + fp32 FMA of the depthwise stage (two halves widened to fp32, then
// FFMA; sm_90 has no mixed-precision FMA) and HFMA2 on one SM (16 warps, 8 independent chains).
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 tools/micro/fma_rate.cu -o build/fma_rate
#include <cuda_fp16.h>
#include <cstdio>
template <int MODE>
__global__ void k(float* out, unsigned a0, unsigned b0, int iters, unsigned long long* cyc) {
    float acc[8];
    unsigned h[8];
    for (int i = 0; i < 8; ++i) acc[i] = threadIdx.x * 0.001f + i, h[i] = a0 + i;
    unsigned a = a0 + threadIdx.x, b = b0;
    __syncthreads();
    const long long t0 = clock64();
    for (int it = 0; it < iters; ++it) {
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            if (MODE == 0) {
                acc[i] = fmaf(acc[i], __uint_as_float(a), __uint_as_float(b));
            } else if (MODE == 1) {
                const unsigned x = a + i;  // (per chain, so that the widening is not hoisted out of the loop)
                acc[i] = fmaf(__low2float(*reinterpret_cast<const __half2*>(&x)),
                              __low2float(*reinterpret_cast<const __half2*>(&b)), acc[i]);
            } else {
                asm volatile("fma.rn.f16x2 %0, %1, %2, %0;" : "+r"(h[i]) : "r"(a), "r"(b));
            }
        }
    }
    const long long t1 = clock64();
    float s = 0;
    for (int i = 0; i < 8; ++i) s += acc[i] + __uint_as_float(h[i]);
    out[blockIdx.x * blockDim.x + threadIdx.x] = s;
    if (threadIdx.x == 0) *cyc = t1 - t0;
}
int main() {
    float* out; unsigned long long* cyc;
    cudaMalloc(&out, 1 << 20); cudaMalloc(&cyc, 8);
    const int iters = 4096;
    const char* names[3] = {"FFMA", "widened fp16 FMA", "HFMA2 (fma.rn.f16x2)"};
    for (int warps : {1, 4, 16}) {
        for (int mode = 0; mode < 3; ++mode) {
            unsigned long long c = 0;
            for (int rep = 0; rep < 2; ++rep) {
                if (mode == 0) k<0><<<1, warps * 32>>>(out, 0x3c003c00u, 0x3c003c00u, iters, cyc);
                if (mode == 1) k<1><<<1, warps * 32>>>(out, 0x3c003c00u, 0x3c003c00u, iters, cyc);
                if (mode == 2) k<2><<<1, warps * 32>>>(out, 0x3c003c00u, 0x3c003c00u, iters, cyc);
                cudaDeviceSynchronize();
            }
            cudaMemcpy(&c, cyc, 8, cudaMemcpyDeviceToHost);
            const double instr = double(iters) * 8 * warps;
            printf("%2d warps  %-24s %8.0f cycles  %.2f warp-instr/clk/SM  (%.2f cycles per instr per warp)\n", warps, names[mode],
                   double(c), instr / c, double(c) / (iters * 8));
        }
    }
    return 0;
}
