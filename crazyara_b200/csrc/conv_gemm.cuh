// Convolution-as-GEMM on the Hopper tensor cores (wgmma, register accumulators, TMA operand feeds).
//
// Computes, for a batch of 8x8 boards stored NHWC in fp16,
//     out[m, n] = epi( sum_{tap, c} act[board(m), sq(m)+tap, c] * w[n, tap*cw + c] + bias[n] )
// i.e. the 1x1 convolutions (ksize 1) and the 3x3 convolutions (ksize 3, pad 1) of the RISE stack
// (reference semantics: DeepCrazyhouse/src/domain/neural_net/architectures/pytorch/builder_util.py:154-178
//  _Stem, :437-475 _BottlekneckResidualBlock, :206-243 _PolicyHead), BatchNorm folded into w/bias.
//
// Tiling: one CTA = 128 output rows (two boards) x BN output channels.  The A operand tile for tap (dy,dx)
// is ONE 4-D TMA box {64 ch, 8 files, 8 ranks, 2 boards} fetched at coordinates (c0, dx, dy, 2*m_tile):
// the halo of the 3x3 taps falls outside the tensor and is zero-filled by the TMA unit, so the 3x3
// convolutions are implicit GEMMs with no im2col buffer.  Both operands land K-major with the 128-byte
// swizzle; two consumer warpgroups (one board = 64 rows each) run wgmma M=64 N=BN on the staged tiles and apply the
// epilogue straight from their accumulator registers, one producer warp keeps the TMA ring full.
//
// Precision float32 (the reference's `Precision float32`, uci/optionsuci.cpp:144, nn/tensorrtapi.cpp:334-360) runs on
// the SAME kernel: an fp32 value x is carried as the fp16 pair hi = fp16(x), lo = fp16(x - hi), activations are stored
// with their channels tripled [hi | hi | lo] and weights per tap as [hi | lo | hi], so that ONE GEMM over 3*Cin
// "channels" accumulates  a_hi*w_hi + a_hi*w_lo + a_lo*w_hi  in the fp32 accumulator (the dropped a_lo*w_lo term
// is 2^-22 relative); the epilogue adds an fp32 residual and writes fp32 and / or the split form for the next layer.
#pragma once
#include "wgmma.cuh"

namespace ara {

struct ConvGemmArgs {
    int M;         // valid output rows (= boards * 64)
    int N;         // valid output channels
    int c_chunks;  // ceil(Cin / 64): K blocks per tap
    int cw;        // weight column pitch per tap (= c_chunks * 64)
    int ksize;     // 1 or 3
    int relu;
    const float* bias;       // [ldo] (zero padded) or nullptr
    const __half* residual;  // [M, ldr] added after activation, or nullptr
    int ldr;
    __half* out_h;  // [M, ldo] fp16 output (or nullptr)
    float* out_f;   // [M, ldo] fp32 output (or nullptr)
    int ldo;        // multiple of 32
    // device-side batch size (or nullptr): number of boards that really hold input; M tiles beyond it leave at once, so
    // a launch sized for the largest batch costs only what the rows in use cost
    const int* boards_dev;
    // ---- Precision float32 (net.cu): fp32 activations between the layers, fp16 hi + lo operand splitting
    const float* residual_f;  // [M, ldr] fp32 residual (instead of `residual`), or nullptr
    __half* out_split;        // [M, 3 * split_cs] fp16: the result as hi | hi | lo (x = hi + lo to ~2^-22), or nullptr
    int split_cs;             // channel pitch of one part (multiple of 64)
};

constexpr int kGemmConsumers = 2;                        // warpgroups, one board (64 rows) each
constexpr int kGemmThreads = kGemmConsumers * 128 + 32;  // + warp 8: TMA producer
constexpr int kBlockM = 128;
constexpr int kBlockK = 64;

template <int BN>
struct ConvGemmCfg {
    static constexpr int kABytes = kBlockM * kBlockK * 2;
    static constexpr int kBBytes = BN * kBlockK * 2;
    static constexpr int kStageBytes = kABytes + kBBytes;
    static constexpr int kStages = (BN <= 64) ? 8 : (BN <= 128 ? 6 : 4);
    static constexpr int kSmemBytes = kStages * kStageBytes + 1024 /*align slack*/ + 256 /*barriers*/;
};

template <int BN>
__global__ void __launch_bounds__(kGemmThreads, 1)
conv_gemm_kernel(const __grid_constant__ CUtensorMap tm_a, const __grid_constant__ CUtensorMap tm_b,
                 const ConvGemmArgs args) {
#if defined(__CUDA_ARCH__) && (__CUDA_ARCH__ >= 900)
    using Cfg = ConvGemmCfg<BN>;
    extern __shared__ uint8_t smem_raw[];
    // 1 KB alignment by offset arithmetic on the shared array itself: a pointer -> integer -> pointer round trip would
    // make every access below a GENERIC load/store (LD.E / ST.E) instead of LDS / STS
    uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + Cfg::kStages * Cfg::kStageBytes);
    uint64_t* empty_bar = full_bar + Cfg::kStages;

    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;
    const int m_tile = blockIdx.x;
    const int n_tile = blockIdx.y;
    if (args.boards_dev != nullptr && m_tile * (kBlockM / 64) >= *args.boards_dev) return;  // written >= 2 launches upstream
    const int taps = args.ksize * args.ksize;
    const int num_kb = taps * args.c_chunks;

    if (threadIdx.x == 0) {
        tma_prefetch_desc(&tm_a);
        tma_prefetch_desc(&tm_b);
        for (int i = 0; i < Cfg::kStages; ++i) {
            mbar_init(&full_bar[i], 1);
            mbar_init(&empty_bar[i], kGemmConsumers * 4);  // lane 0 of every consumer warp
        }
        fence_mbar_init();
    }
    __syncthreads();
    // PDL: everything above overlapped the tail of the previous kernel; its outputs are only touched below
    pdl_wait();
    pdl_launch_dependents();

    if (warp == kGemmConsumers * 4) {
        if (lane == 0) {
            const int half_k = args.ksize >> 1;
            for (int kb = 0; kb < num_kb; ++kb) {
                const int s = kb % Cfg::kStages;
                const uint32_t ph = (kb / Cfg::kStages) & 1;
                mbar_wait(&empty_bar[s], ph ^ 1);
                mbar_arrive_expect_tx(&full_bar[s], Cfg::kStageBytes);
                const int tap = kb / args.c_chunks;
                const int cc = kb - tap * args.c_chunks;
                const int dy = tap / args.ksize - half_k;
                const int dx = tap % args.ksize - half_k;
                uint8_t* sa = smem + s * Cfg::kStageBytes;
                uint8_t* sb = sa + Cfg::kABytes;
                tma_load_4d(sa, &tm_a, &full_bar[s], cc * kBlockK, dx, dy, m_tile * 2);
                tma_load_2d(sb, &tm_b, &full_bar[s], tap * args.cw + cc * kBlockK, n_tile * BN);
            }
        }
        return;
    }
    // ---- consumer warpgroup wg: rows 64 wg .. 64 wg + 63 of the tile (board 2 m_tile + wg)
    const int wg = warp >> 2;
    float acc[BN / 2];
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) acc[i] = 0.0f;
    for (int kb = 0; kb < num_kb; ++kb) {
        const int s = kb % Cfg::kStages;
        mbar_wait(&full_bar[s], (kb / Cfg::kStages) & 1);
        const uint32_t sa = smem_u32(smem + s * Cfg::kStageBytes) + wg * (64 * 128);
        const uint32_t sb = smem_u32(smem + s * Cfg::kStageBytes) + Cfg::kABytes;
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < kBlockK / 16; ++k)
            wgmma_f16<BN>(acc, wgmma_desc_k_sw128(sa + k * 32, 1024), wgmma_desc_k_sw128(sb + k * 32, 1024),
                          (kb > 0 || k > 0) ? 1u : 0u);
        wgmma_commit();
        // the stage before this one is free once its wgmma group has retired (one group stays in flight)
        wgmma_wait<1>();
        wgmma_fence_regs(acc);
        if (kb > 0 && lane == 0) mbar_arrive(&empty_bar[(kb - 1) % Cfg::kStages]);
    }
    wgmma_wait<0>();
    wgmma_fence_regs(acc);

    // ---- epilogue from the accumulator fragments: rows r0, r0 + 8; columns 8 j + 2 (lane % 4) (+ 1)
    const int r0 = m_tile * kBlockM + wg * 64 + (warp & 3) * 16 + (lane >> 2);
#pragma unroll
    for (int j = 0; j < BN / 8; ++j) {
        const int g0 = n_tile * BN + 8 * j;
        if (g0 >= args.ldo) break;  // uniform
        const int n = g0 + 2 * (lane & 3);
        float2 b = make_float2(0.0f, 0.0f);
        if (args.bias != nullptr) b = __ldg(reinterpret_cast<const float2*>(args.bias + n));
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int m = r0 + 8 * h;
            float f0 = acc[4 * j + 2 * h] + b.x, f1 = acc[4 * j + 2 * h + 1] + b.y;
            if (args.relu) f0 = fmaxf(f0, 0.0f), f1 = fmaxf(f1, 0.0f);
            if (m >= args.M) continue;
            if (args.residual != nullptr) {
                const float2 x = __half22float2(*reinterpret_cast<const __half2*>(args.residual + static_cast<size_t>(m) * args.ldr + n));
                f0 += x.x, f1 += x.y;
            }
            if (args.residual_f != nullptr) {
                const float2 x = __ldg(reinterpret_cast<const float2*>(args.residual_f + static_cast<size_t>(m) * args.ldr + n));
                f0 += x.x, f1 += x.y;
            }
            if (args.out_split != nullptr && g0 < args.split_cs) {
                __half* base = args.out_split + static_cast<size_t>(m) * (3 * args.split_cs) + n;
                const __half2 hi = __floats2half2_rn(f0, f1);
                const float2 hf = __half22float2(hi);
                *reinterpret_cast<__half2*>(base) = hi;
                *reinterpret_cast<__half2*>(base + args.split_cs) = hi;
                *reinterpret_cast<__half2*>(base + 2 * args.split_cs) = __floats2half2_rn(f0 - hf.x, f1 - hf.y);
            }
            if (args.out_h != nullptr)
                *reinterpret_cast<__half2*>(args.out_h + static_cast<size_t>(m) * args.ldo + n) = __floats2half2_rn(f0, f1);
            if (args.out_f != nullptr)
                *reinterpret_cast<float2*>(args.out_f + static_cast<size_t>(m) * args.ldo + n) = make_float2(f0, f1);
        }
    }
#endif
}

}  // namespace ara
