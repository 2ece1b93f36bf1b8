// Fully-connected policy head (the reference trainer's select_policy_from_plane = False, builder_util.py:206-243
// _PolicyHead body2 / body3): logits[b, l] = W_fc[l] . relu(conv2(x))[b] + b_fc[l] onto the classic label list, then the
// softmax the engine's backend appends (tensorrtapi.cpp:378-380).
//
// policy_fc_kernel: the GEMM on wgmma with the operands swapped, so that the ~2k labels are the M side and the at most
// 128 boards of a search batch the N side.  A = W_fc [lp][K] fp16, 64-label tiles; B = the policy convolution's output,
// one board per row [rows_cap][K] fp16 (a board's 64 x ldp NHWC values are one contiguous row: Net permutes the columns
// of W_fc from the trainer's NCHW flatten c * 64 + sq to sq * ldp + c at upload, so no transpose runs).  Both operands
// come in by TMA through an mbarrier ring (one producer warp); one consumer warpgroup accumulates in fp32 registers.
// K is split across CTAs (grid.y) so that a forward of any batch size fills the SMs; every split writes its fp32
// partial sums, and policy_fc_softmax_kernel (net_kernels.cuh) adds them in split order (no atomics): a board's logits are the same bits
// in every row of every batch, as the policy-map head's are.  The split count follows from L and K only.
//
// Precision float32: the same kernel on the split operands of conv_gemm.cuh, activations [hi | hi | lo] and weights
// [hi | lo | hi] per square (K = 64 * 3 * cs).
#pragma once
#include "wgmma.cuh"

namespace ara {

constexpr int kFcThreads = 128 + 32;  // one consumer warpgroup + a TMA producer warp
constexpr int kFcStages = 4;
constexpr int kFcTargetCtas = 264;    // label tiles x splits: two waves of CTAs on the 132 SMs of an H100 SXM

template <int BN>
struct PolicyFcCfg {
    static constexpr int kABytes = 64 * 64 * 2;
    static constexpr int kBBytes = BN * 64 * 2;
    static constexpr int kStageBytes = kABytes + kBBytes;
    static constexpr int kSmemBytes = kFcStages * kStageBytes + 1024 /*align slack*/ + 128 /*barriers*/;
};

struct PolicyFcArgs {
    int kb_per_split;  // 64-wide K blocks per split (the last split may have fewer)
    int num_kb;        // K / 64
    int lp;            // padded label count (multiple of 64): row pitch of the partial sums
    int rows_cap;      // boards per split slab of `part`
    float* part;       // [splits][rows_cap][lp] fp32 partial sums
    const int* boards_dev;  // device-side count of the boards in use, or nullptr
};

template <int BN>
__global__ void __launch_bounds__(kFcThreads)
policy_fc_kernel(const __grid_constant__ CUtensorMap tm_w, const __grid_constant__ CUtensorMap tm_x, const PolicyFcArgs args) {
#if defined(__CUDA_ARCH__) && (__CUDA_ARCH__ >= 900)
    using Cfg = PolicyFcCfg<BN>;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + kFcStages * Cfg::kStageBytes);
    uint64_t* empty_bar = full_bar + kFcStages;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int m_tile = blockIdx.x, split = blockIdx.y, n_tile = blockIdx.z;
    if (args.boards_dev != nullptr && n_tile * BN >= *args.boards_dev) return;  // written >= 2 launches upstream
    const int kb0 = split * args.kb_per_split;
    const int nkb = min(args.kb_per_split, args.num_kb - kb0);
    if (threadIdx.x == 0) {
        tma_prefetch_desc(&tm_w);
        tma_prefetch_desc(&tm_x);
        for (int i = 0; i < kFcStages; ++i) {
            mbar_init(&full_bar[i], 1);
            mbar_init(&empty_bar[i], 4);  // lane 0 of every consumer warp
        }
        fence_mbar_init();
    }
    __syncthreads();
    pdl_wait();
    pdl_launch_dependents();
    if (warp == 4) {
        if (lane == 0) {
            for (int kb = 0; kb < nkb; ++kb) {
                const int s = kb % kFcStages;
                mbar_wait(&empty_bar[s], ((kb / kFcStages) & 1) ^ 1);
                mbar_arrive_expect_tx(&full_bar[s], Cfg::kStageBytes);
                uint8_t* sa = smem + s * Cfg::kStageBytes;
                tma_load_2d(sa, &tm_w, &full_bar[s], (kb0 + kb) * 64, m_tile * 64);
                tma_load_2d(sa + Cfg::kABytes, &tm_x, &full_bar[s], (kb0 + kb) * 64, n_tile * BN);
            }
        }
        return;
    }
    float acc[BN / 2];
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) acc[i] = 0.0f;
    for (int kb = 0; kb < nkb; ++kb) {
        const int s = kb % kFcStages;
        mbar_wait(&full_bar[s], (kb / kFcStages) & 1);
        const uint32_t sa = smem_u32(smem + s * Cfg::kStageBytes);
        const uint32_t sb = sa + Cfg::kABytes;
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < 4; ++k)
            wgmma_f16<BN>(acc, wgmma_desc_k_sw128(sa + k * 32, 1024), wgmma_desc_k_sw128(sb + k * 32, 1024), (kb > 0 || k > 0) ? 1u : 0u);
        wgmma_commit();
        wgmma_wait<1>();
        wgmma_fence_regs(acc);
        if (kb > 0 && lane == 0) mbar_arrive(&empty_bar[(kb - 1) % kFcStages]);
    }
    wgmma_wait<0>();
    wgmma_fence_regs(acc);
    // acc[4 j + 2 h + e] = D[label 16 warp + lane / 4 + 8 h][board 8 j + 2 (lane % 4) + e]
    const int l0 = m_tile * 64 + warp * 16 + (lane >> 2);
    float* part = args.part + static_cast<size_t>(split) * args.rows_cap * args.lp;
#pragma unroll
    for (int j = 0; j < BN / 8; ++j)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
            const int b = n_tile * BN + 8 * j + 2 * (lane & 3) + e;
            if (b >= args.rows_cap) continue;
            part[static_cast<size_t>(b) * args.lp + l0] = acc[4 * j + e];
            part[static_cast<size_t>(b) * args.lp + l0 + 8] = acc[4 * j + 2 + e];
        }
#endif
}

}  // namespace ara
