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
// Resident A (the 3x3 layers whose A tiles all fit, conv_resident_a): fetching the shifted tile per (tap, chunk) reads
// each activation nine times from L2, once more for every N tile.  Instead the producer loads the CTA's c_chunks tiles
// once, at tap (0, 0), and only B tiles go through the ring; the consumers build each tap's shifted A operand in
// registers with ldmatrix (the halo from a zero row in shared memory) and issue the register-A wgmma, in the same k
// order as the streaming loop, so the two give the same bits.
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
    int n_end;      // columns n_end.. of the output are left alone (= ldo unless a layer writes a channel slice of a row)
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

constexpr int kConvMaxSmem = 232448;  // dynamic shared memory of one block on sm_90

template <int BN>
struct ConvGemmCfg {
    static constexpr int kABytes = kBlockM * kBlockK * 2;
    static constexpr int kBBytes = BN * kBlockK * 2;
    static constexpr int kStageBytes = kABytes + kBBytes;
    static constexpr int kStages = (BN <= 64) ? 8 : (BN <= 128 ? 6 : 4);
    static constexpr int kSmemBytes = kStages * kStageBytes + 1024 /*align slack*/ + 256 /*barriers*/;
    // resident A (3x3 layers): the c_chunks A tiles of the CTA, then a ring of B tiles only, the barriers and one
    // 128-byte zero row (the halo)
    static constexpr int kResidentFixedBytes = kStages * kBBytes + 1024 /*align slack*/ + 256 /*barriers*/ + 128 /*zero row*/;
    static constexpr int kResidentMaxChunks = (kConvMaxSmem - kResidentFixedBytes) / kABytes;
    static constexpr int resident_smem_bytes(int c_chunks) { return c_chunks * kABytes + kResidentFixedBytes; }
    static_assert((2 * kStages + kResidentMaxChunks) * 8 <= 256, "conv_gemm barriers exceed their 256 bytes");
};

// Resident A: the m16k16 fragments of k block kb (tap, chunk cc) for one warp, built with ldmatrix.x4 from the CTA's
// unshifted chunk tile (the TMA image of tap (0, 0): row 64 board + 8 y + x, 16-byte piece j at j ^ x).  ldmatrix.x4
// lane l addresses output square (y, x) = (2 (warp & 3) + ((l >> 3) & 1), l & 7), channels 8 (l >> 4) of the k16 step;
// a lane whose shifted square (y + dy, x + dx) is off the board addresses the zero row instead, which is the zero fill
// the streaming path gets from TMA.  The zero row's pieces are taken at j ^ ((x + dx) & 7) so that the eight lanes of
// a matrix hit eight different bank groups either way.  In tap 0 the chunk tile itself may still be in flight.
template <int BN>
__device__ __forceinline__ void conv_resident_frags(uint32_t (&fa)[4][4], int kb, int c_chunks, uint32_t a_board,
                                                    uint32_t zero_row, int y, int x, int c_hi, uint64_t* a_bar) {
    const int tap = kb / c_chunks;
    const int cc = kb - tap * c_chunks;
    const int sy = y + tap / 3 - 1, sx = x + tap % 3 - 1;
    if (tap == 0) mbar_wait(&a_bar[cc], 0);
    const bool on_board = static_cast<unsigned>(sy) < 8u && static_cast<unsigned>(sx) < 8u;
    const uint32_t row = on_board ? a_board + cc * ConvGemmCfg<BN>::kABytes + (sy * 8 + sx) * 128 : zero_row;
    const int sw = sx & 7;
#pragma unroll
    for (int k = 0; k < kBlockK / 16; ++k)
        asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];"
                     : "=r"(fa[k][0]), "=r"(fa[k][1]), "=r"(fa[k][2]), "=r"(fa[k][3])
                     : "r"(row + (((2 * k + c_hi) ^ sw) << 4))
                     : "memory");
}

// Resident A, k block kb of a consumer warpgroup: the register-A wgmmas of its fragments fa (loaded one block earlier)
// against the staged B tile, then the fragments of block kb + 1 into nx while this block's group runs, then the wait
// that retires block kb - 1 and releases its B stage.  Three fragment sets rotate: when nx is written, the groups of
// blocks kb - 1 and kb may be in flight and read the other two; block kb - 2, the last reader of nx, retired at the
// previous block's wgmma_wait<1>.
template <int BN>
__device__ __forceinline__ void conv_resident_kblock(float (&acc)[BN / 2], const uint32_t (&fa)[4][4], uint32_t (&nx)[4][4],
                                                     int kb, int num_kb, int c_chunks, uint32_t a_board, uint32_t zero_row,
                                                     uint32_t ring, int y, int x, int c_hi, uint64_t* full_bar,
                                                     uint64_t* empty_bar, uint64_t* a_bar, int lane) {
    using Cfg = ConvGemmCfg<BN>;
    const int s = kb % Cfg::kStages;
    mbar_wait(&full_bar[s], (kb / Cfg::kStages) & 1);
    const uint32_t sb = ring + s * Cfg::kBBytes;
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < kBlockK / 16; ++k)
        wgmma_f16_rs<BN>(acc, fa[k], wgmma_desc_k_sw128(sb + k * 32, 1024), (kb > 0 || k > 0) ? 1u : 0u);
    wgmma_commit();
    if (kb + 1 < num_kb) conv_resident_frags<BN>(nx, kb + 1, c_chunks, a_board, zero_row, y, x, c_hi, a_bar);
    wgmma_wait<1>();
    wgmma_fence_regs(acc);
    if (kb > 0 && lane == 0) mbar_arrive(&empty_bar[(kb - 1) % Cfg::kStages]);
}

// kResidentA (3x3 layers whose chunks fit, conv_resident_a): the producer loads each of the CTA's c_chunks A tiles
// once, then streams only B tiles through the ring; the k order (tap, chunk, k16) and the epilogue are the streaming
// path's, so both give the same bits.
template <int BN, bool kResidentA>
__global__ void __launch_bounds__(kGemmThreads, 1)
conv_gemm_kernel(const __grid_constant__ CUtensorMap tm_a, const __grid_constant__ CUtensorMap tm_b,
                 const ConvGemmArgs args) {
#if defined(__CUDA_ARCH__) && (__CUDA_ARCH__ >= 900)
    using Cfg = ConvGemmCfg<BN>;
    extern __shared__ uint8_t smem_raw[];
    // 1 KB alignment by offset arithmetic on the shared array itself: a pointer -> integer -> pointer round trip would
    // make every access below a GENERIC load/store (LD.E / ST.E) instead of LDS / STS
    uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
    // streaming: stage s holds an A and a B tile; resident A: the A tiles first, then stages of one B tile
    constexpr int kStageBytes = kResidentA ? Cfg::kBBytes : Cfg::kStageBytes;
    uint8_t* ring = smem + (kResidentA ? args.c_chunks * Cfg::kABytes : 0);
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(ring + Cfg::kStages * kStageBytes);
    uint64_t* empty_bar = full_bar + Cfg::kStages;
    uint64_t* a_bar = empty_bar + Cfg::kStages;  // resident A: one per chunk tile
    uint8_t* zero_row = reinterpret_cast<uint8_t*>(full_bar) + 256;

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
        if (kResidentA)
            for (int i = 0; i < args.c_chunks; ++i) mbar_init(&a_bar[i], 1);
        fence_mbar_init();
    }
    if (kResidentA && threadIdx.x < 8) reinterpret_cast<uint4*>(zero_row)[threadIdx.x] = make_uint4(0u, 0u, 0u, 0u);
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
                const int tap = kb / args.c_chunks;
                const int cc = kb - tap * args.c_chunks;
                const int dy = tap / args.ksize - half_k;
                const int dx = tap % args.ksize - half_k;
                uint8_t* st = ring + s * kStageBytes;
                if (kResidentA) {
                    // chunk kb's A tile goes out beside tap 0's B tiles, so tap 0 starts on chunk 0 at once.  With
                    // more chunks than stages, a late chunk's load waits behind the empty wait of block kb - 1, which
                    // needs block kb - 1 - kStages released.  The consumers first wait for chunk kb when they load block
                    // kb's fragments, by then with every block up to kb - 3 released: no cycle for kStages >= 2.
                    if (kb < args.c_chunks) {
                        mbar_arrive_expect_tx(&a_bar[kb], Cfg::kABytes);
                        tma_load_4d(smem + kb * Cfg::kABytes, &tm_a, &a_bar[kb], kb * kBlockK, 0, 0, m_tile * 2);
                    }
                    mbar_wait(&empty_bar[s], ph ^ 1);
                    mbar_arrive_expect_tx(&full_bar[s], Cfg::kBBytes);
                    tma_load_2d(st, &tm_b, &full_bar[s], tap * args.cw + cc * kBlockK, n_tile * BN);
                } else {
                    mbar_wait(&empty_bar[s], ph ^ 1);
                    mbar_arrive_expect_tx(&full_bar[s], Cfg::kStageBytes);
                    tma_load_4d(st, &tm_a, &full_bar[s], cc * kBlockK, dx, dy, m_tile * 2);
                    tma_load_2d(st + Cfg::kABytes, &tm_b, &full_bar[s], tap * args.cw + cc * kBlockK, n_tile * BN);
                }
            }
        }
        return;
    }
    // ---- consumer warpgroup wg: rows 64 wg .. 64 wg + 63 of the tile (board 2 m_tile + wg)
    const int wg = warp >> 2;
    float acc[BN / 2];
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) acc[i] = 0.0f;
    if (kResidentA) {
        const uint32_t a_board = smem_u32(smem) + wg * (64 * 128);
        const int y = 2 * (warp & 3) + ((lane >> 3) & 1), x = lane & 7, c_hi = lane >> 4;
        const uint32_t z = smem_u32(zero_row), r = smem_u32(ring);
        // three fragment sets in rotation (register arrays need compile-time indices): num_kb = 9 c_chunks is a
        // multiple of 3
        uint32_t f0[4][4], f1[4][4], f2[4][4];
        conv_resident_frags<BN>(f0, 0, args.c_chunks, a_board, z, y, x, c_hi, a_bar);
        for (int kb = 0; kb < num_kb; kb += 3) {
            conv_resident_kblock<BN>(acc, f0, f1, kb, num_kb, args.c_chunks, a_board, z, r, y, x, c_hi, full_bar, empty_bar, a_bar, lane);
            conv_resident_kblock<BN>(acc, f1, f2, kb + 1, num_kb, args.c_chunks, a_board, z, r, y, x, c_hi, full_bar, empty_bar, a_bar,
                                     lane);
            conv_resident_kblock<BN>(acc, f2, f0, kb + 2, num_kb, args.c_chunks, a_board, z, r, y, x, c_hi, full_bar, empty_bar, a_bar,
                                     lane);
        }
    } else {
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
    }
    wgmma_wait<0>();
    wgmma_fence_regs(acc);

    // ---- epilogue from the accumulator fragments: rows r0, r0 + 8; columns 8 j + 2 (lane % 4) (+ 1)
    const int r0 = m_tile * kBlockM + wg * 64 + (warp & 3) * 16 + (lane >> 2);
#pragma unroll
    for (int j = 0; j < BN / 8; ++j) {
        const int g0 = n_tile * BN + 8 * j;
        if (g0 >= args.n_end) break;  // uniform
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
