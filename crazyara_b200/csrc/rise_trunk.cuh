// The whole RISE residual tower as ONE persistent kernel (builder_util.py:437-475 _BottlekneckResidualBlock, repeated
// for every block of rise_mobile_v2 / v3; the squeeze-excitation of a block acts on its input, in place).
// One consumer warpgroup owns one board (64 rows) from the stem output to the tower output; its activation tile X stays
// in shared memory, 128B-swizzled K-major (wgmma's A operand).  Per 64-channel chunk of a block:
//     MMA1  D1[64x64] = X . W1^T (wgmma m64n64) -> relu(D1 + b1) -> H1 -> depthwise kxk, + bd, relu -> H2
//     MMA2  D2[64x256] += H2 . W2^T (wgmma m64n256, accumulator in registers for the whole block)
// then X <- (D2 + b2) + X.  Pre-tiled weight images (rise_trunk_host.cu) stream through one bulk-copy ring per CTA.
// Every board runs the same instructions whatever NB is: its outputs do not depend on the batch.
#pragma once
#include "rise_trunk_args.h"
#include "wgmma.cuh"

namespace ara {

// ring of weight units: unit 2 c = W1 image of chunk c (tile + vectors), unit 2 c + 1 = its W2 image
constexpr int kRtSlot = kTrunkW1Image;
template <int NB>
struct RtCfg {
    static constexpr int kRing = NB == 1 ? 4 : 3;
    // + the producer: a warp, or with two boards a warpgroup (setmaxnreg hands registers over per warpgroup)
    static constexpr int kThreads = NB * 128 + (NB == 1 ? 32 : 128);
    static constexpr int kOffBoard = kRing * kRtSlot;
    // per board: X [4 K panels][64 rows][128 B] | H2 [64 rows][128 B] | H1 [8 groups][64 squares][16 B] | SE scratch
    static constexpr int kBoardBytes = 32768 + 8192 + 8192 + 2048;
    static constexpr int kOffBar = kOffBoard + NB * kBoardBytes;
    static constexpr int kSmemBytes = kOffBar + 256 + 1024 /*align slack*/;
    static_assert(kSmemBytes <= 232448, "trunk kernel shared memory exceeds the sm_90 limit of 227 KB per block");
};

// -DARA_TRUNK_PROF: per-role cycle counters of CTA 0 (args.prof[role * 16 + slot]; role 1: rise_trunk_kernel, role 0:
// rise_trunk_pair_kernel); see tools/prof_trunk.py
#if defined(ARA_TRUNK_PROF)
#define RT_PROF_DECL() long long pt_ = clock64(); unsigned long long pacc_[16] = {}
#define RT_PROF(idx)                                               \
    do {                                                           \
        const long long now_ = clock64();                          \
        pacc_[idx] += static_cast<unsigned long long>(now_ - pt_); \
        pt_ = now_;                                                \
    } while (0)
#define RT_PROF_FLUSH(role)                                                          \
    do {                                                                             \
        if (args.prof != nullptr && blockIdx.x == 0 && lane == 0)                    \
            for (int i_ = 0; i_ < 16; ++i_) args.prof[(role) * 16 + i_] = pacc_[i_]; \
    } while (0)
#else
#define RT_PROF_DECL() do { } while (0)
#define RT_PROF(idx) do { } while (0)
#define RT_PROF_FLUSH(role) do { } while (0)
#endif

__device__ __forceinline__ float rt_hard_sigmoid(float x) { return fminf(fmaxf(x * (1.0f / 6.0f) + 0.5f, 0.0f), 1.0f); }
// the squeeze-excitation gate of a block; kernels built without MX only have the torch one
template <bool MX>
__device__ __forceinline__ float rt_gate(float x, int gate) {
    if (!MX || gate == kTrunkGateHard6) return rt_hard_sigmoid(x);
    if (gate == kTrunkGateHard5) return fminf(fmaxf(x * 0.2f + 0.5f, 0.0f), 1.0f);
    return 1.0f / (1.0f + expf(-x));
}
// b[i] + a when the block has that bias (MXNet ca_se fully-connected layers), else a
template <bool MX>
__device__ __forceinline__ float rt_add_bias(const float* b, int i, float a) { return MX && b != nullptr ? __ldg(b + i) + a : a; }
__device__ __forceinline__ float2 rt_unpack(uint32_t v) { return __half22float2(*reinterpret_cast<const __half2*>(&v)); }
__device__ __forceinline__ uint32_t rt_pack(float a, float b) {
    const __half2 h = __floats2half2_rn(a, b);
    return *reinterpret_cast<const uint32_t*>(&h);
}

// depthwise k x k, + bd, relu for the whole column x (8 squares) of the channel pair 8 g + 2 p, 8 g + 2 p + 1, into the
// H2 tile.  sH1: [8 groups][64 squares][8 channels] fp16; aux: b1[64] f32 | bd[64] f32 | wd[k*k][64] f16.
// Each H1 value and each weight is loaded and widened once; the 16 accumulators stay in registers.  Every output
// keeps one FMA order: bd, then dxi outer (columns outside the board skipped), dyi inner (rows outside the board as
// zero operands), each a fp32 fmaf of the widened fp16 operands (their product is exact in fp32, so this gives the bits
// of a mixed-precision fp16 x fp16 + fp32 FMA).  The three tower shapes share that order, so their outputs are the same
// bits; tests/test_trunk_depthwise_bits_gpu.py pins it.
template <int K>
__device__ __forceinline__ void rt_depthwise_column(const uint8_t* sH1, const uint8_t* aux, uint8_t* sH2, int g, int p, int x) {
    constexpr int R = K / 2;
    const float2 b0 = *reinterpret_cast<const float2*>(reinterpret_cast<const float*>(aux + 256) + g * 8 + 2 * p);
    const uint8_t* wd = aux + 512 + g * 16 + p * 4;
    const uint8_t* col = sH1 + g * 1024 + p * 4;  // square s of the pair: col + 16 s
    float acc[8][2];
#pragma unroll
    for (int y = 0; y < 8; ++y) acc[y][0] = b0.x, acc[y][1] = b0.y;
#pragma unroll
    for (int dxi = 0; dxi < K; ++dxi) {
        const int xx = x + dxi - R;
        if (xx < 0 || xx > 7) continue;
        float2 in[8], w[K];
#pragma unroll
        for (int yy = 0; yy < 8; ++yy) in[yy] = rt_unpack(*reinterpret_cast<const uint32_t*>(col + ((yy * 8 + xx) << 4)));
#pragma unroll
        for (int dyi = 0; dyi < K; ++dyi) w[dyi] = rt_unpack(*reinterpret_cast<const uint32_t*>(wd + (dyi * K + dxi) * 128));
#pragma unroll
        for (int y = 0; y < 8; ++y)
#pragma unroll
            for (int dyi = 0; dyi < K; ++dyi) {
                const int yy = y + dyi - R;
                const float2 v = yy >= 0 && yy <= 7 ? in[yy] : make_float2(0.0f, 0.0f);
                acc[y][0] = fmaf(v.x, w[dyi].x, acc[y][0]);
                acc[y][1] = fmaf(v.y, w[dyi].y, acc[y][1]);
            }
    }
    // H2 row s = 8 y + x (s & 7 = x): channel group g sits in 16-byte chunk g ^ x
#pragma unroll
    for (int y = 0; y < 8; ++y)
        *reinterpret_cast<uint32_t*>(sH2 + (y * 8 + x) * 128 + ((g ^ x) << 4) + p * 4) =
            rt_pack(fmaxf(acc[y][0], 0.0f), fmaxf(acc[y][1], 0.0f));
}


__device__ __forceinline__ void rt_wg_sync(int wg) { asm volatile("bar.sync %0, 128;" ::"r"(1 + wg) : "memory"); }
// byte offset of the fp16 element (row, channel) in the swizzled X tile
__device__ __forceinline__ uint32_t rt_x_off(int row, int ch) {
    return static_cast<uint32_t>((ch >> 6) * 8192 + row * 128 + ((((ch & 63) >> 3) ^ (row & 7)) << 4) + (ch & 7) * 2);
}

// The stages below are shared by every shape of the tower kernel; t is the thread's index in its warpgroup.

// stem output of `board` -> the X tile (16-byte pieces into the swizzled layout); a board without input: zeros.
// The caller synchronises the warpgroup.
__device__ __forceinline__ void rt_load_x(uint8_t* sX, const __half* x_in, int board, bool board_ok, int t) {
    const uint4* src = reinterpret_cast<const uint4*>(x_in + static_cast<size_t>(board) * 64 * 256);
#pragma unroll 4
    for (int i = 0; i < 16; ++i) {
        const int p = t + i * 128, r = p >> 5, c16 = p & 31;
        const uint4 v = board_ok ? __ldg(src + p) : make_uint4(0u, 0u, 0u, 0u);
        *reinterpret_cast<uint4*>(sX + (c16 >> 3) * 8192 + r * 128 + (((c16 & 7) ^ (r & 7)) << 4)) = v;
    }
    fence_proxy_async();
}

// squeeze-excitation on the block input, in place: thread t owns channels 2t, 2t+1
template <bool MX>
__device__ __forceinline__ void rt_squeeze_excite(const TrunkBlock& B, uint8_t* sX, float* sPool, float* sHid, int t, int wg) {
    float s0 = 0.0f, s1 = 0.0f;
#pragma unroll 8
    for (int r = 0; r < 64; ++r) {
        const float2 f = __half22float2(*reinterpret_cast<const __half2*>(sX + rt_x_off(r, 2 * t)));
        s0 += f.x, s1 += f.y;
    }
    sPool[2 * t] = s0 * (1.0f / 64.0f);
    sPool[2 * t + 1] = s1 * (1.0f / 64.0f);
    rt_wg_sync(wg);
    float sc0, sc1;
    if (B.se_type == 1) {  // fc1 256 -> 128 (relu), fc2 128 -> 256 (hard sigmoid)
        float a = 0.0f;
#pragma unroll 16
        for (int k = 0; k < 256; ++k) a = fmaf(__half2float(B.se_w1t[k * 128 + t]), sPool[k], a);
        sHid[t] = fmaxf(rt_add_bias<MX>(B.se_b1, t, a), 0.0f);
        rt_wg_sync(wg);
        float a0 = 0.0f, a1 = 0.0f;
        const __half2* w2 = reinterpret_cast<const __half2*>(B.se_w2t) + t;
#pragma unroll 16
        for (int j = 0; j < 128; ++j) {
            const float2 wf = __half22float2(__ldg(w2 + j * 128));
            a0 = fmaf(wf.x, sHid[j], a0);
            a1 = fmaf(wf.y, sHid[j], a1);
        }
        sc0 = rt_gate<MX>(rt_add_bias<MX>(B.se_b, 2 * t, a0), B.gate);
        sc1 = rt_gate<MX>(rt_add_bias<MX>(B.se_b, 2 * t + 1, a1), B.gate);
    } else {  // 256 -> 256 + bias (hard sigmoid)
        float a0 = 0.0f, a1 = 0.0f;
        const __half2* w1 = reinterpret_cast<const __half2*>(B.se_w1t) + t;
#pragma unroll 16
        for (int k = 0; k < 256; ++k) {
            const float2 wf = __half22float2(__ldg(w1 + k * 128));
            a0 = fmaf(wf.x, sPool[k], a0);
            a1 = fmaf(wf.y, sPool[k], a1);
        }
        sc0 = rt_gate<MX>(__ldg(B.se_b + 2 * t) + a0, B.gate), sc1 = rt_gate<MX>(__ldg(B.se_b + 2 * t + 1) + a1, B.gate);
    }
#pragma unroll 8
    for (int r = 0; r < 64; ++r) {
        __half2* x = reinterpret_cast<__half2*>(sX + rt_x_off(r, 2 * t));
        const float2 f = __half22float2(*x);
        *x = __floats2half2_rn(f.x * sc0, f.y * sc1);
    }
    fence_proxy_async();
    rt_wg_sync(wg);
}

// epilogue 1: relu(D1 + b1) -> H1 for the N / 4 8-channel groups g0 .. g0 + N / 4 - 1.  acc1: the N accumulator
// registers of a wgmma m64n(2 N) over those channels.  aux: the vectors of the chunk's W1 image
template <int N>
__device__ __forceinline__ void rt_epilogue1(const float (&acc1)[N], const uint8_t* aux, uint8_t* sH1, int fr, int fc, int g0 = 0) {
#pragma unroll
    for (int jj = 0; jj < N / 4; ++jj) {
        const int g = g0 + jj;
        const float2 b1 = *reinterpret_cast<const float2*>(reinterpret_cast<const float*>(aux) + 8 * g + fc);
#pragma unroll
        for (int h = 0; h < 2; ++h)
            *reinterpret_cast<__half2*>(sH1 + g * 1024 + (fr + 8 * h) * 16 + fc * 2) =
                __floats2half2_rn(fmaxf(acc1[4 * jj + 2 * h] + b1.x, 0.0f), fmaxf(acc1[4 * jj + 2 * h + 1] + b1.y, 0.0f));
    }
}

// depthwise k x k of H1 -> H2 (A operand of MMA2) in the 128B-swizzled K-major layout, for the NG 8-channel groups
// g0 .. g0 + NG - 1, by the 128 threads of a warpgroup.  Warp w takes groups g0 + w, g0 + w + 4, ...: lane = 4 x + p,
// so that each row of a group is one conflict-free 128-byte load of the warp, and each H2 row one conflict-free store.
template <int NG = 8>
__device__ __forceinline__ void rt_depthwise_stage(const uint8_t* sH1, const uint8_t* aux, uint8_t* sH2, int ksize, int t, int g0 = 0) {
    const int x = (t >> 2) & 7, p = t & 3;
#pragma unroll
    for (int i = 0; i < NG / 4; ++i) {
        const int g = g0 + (t >> 5) + 4 * i;
        if (ksize == 3)
            rt_depthwise_column<3>(sH1, aux, sH2, g, p, x);
        else
            rt_depthwise_column<5>(sH1, aux, sH2, g, p, x);
    }
}

// MX: the kernel also runs the blocks of MXNet RISE symbols (TrunkBlock::flags, gate, se_b1)
template <int NB, bool MX>
// A consumer needs ~230 registers (accumulators: 160).  Two boards = 12 warps, 3 per 16 K-register SM sub-partition:
// 168 each at launch, then the producer warpgroup drops to 40 and the consumers grow to 232 (2 x 232 + 40 = 504).
__global__ void __launch_bounds__(RtCfg<NB>::kThreads, 1) rise_trunk_kernel(const __grid_constant__ TrunkArgs args) {
#if defined(__CUDA_ARCH__) && (__CUDA_ARCH__ >= 900)
    using Cfg = RtCfg<NB>;
    constexpr int R = Cfg::kRing;
    extern __shared__ uint8_t smem_raw[];
    // 1 KB alignment by offset arithmetic on the shared array itself: a pointer -> integer -> pointer round trip would
    // make every access below a GENERIC load/store (LD.E / ST.E) instead of LDS / STS
    uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
    uint64_t* full = reinterpret_cast<uint64_t*>(smem + Cfg::kOffBar);
    uint64_t* empty = full + R;

    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;
    const int n_blocks = args.n_blocks;
    // device-side batch size: a CTA whose boards hold no input leaves before it touches anything
    if (args.boards_dev != nullptr && static_cast<int>(blockIdx.x) * NB >= *args.boards_dev) return;

    if (threadIdx.x == 0) {
        for (int i = 0; i < R; ++i) {
            mbar_init(&full[i], 1);
            mbar_init(&empty[i], NB);  // one arrival per warpgroup
        }
        fence_mbar_init();
    }
    __syncthreads();
    pdl_wait();
    pdl_launch_dependents();

    if (warp >= NB * 4) {
        if (NB > 1) asm volatile("setmaxnreg.dec.sync.aligned.u32 40;" ::: "memory");
        // ---------------------------------------------------------------- producer: the weight stream
        if (warp == NB * 4 && lane == 0) {
            const TrunkBlock& L = args.blk[n_blocks - 1];
            const int n_units = 2 * (L.chunk0 + L.n_chunks);
            for (int u = 0; u < n_units; ++u) {
                const int s = u % R;
                mbar_wait_relaxed(&empty[s], ((u / R) & 1) ^ 1);
                const size_t c = static_cast<size_t>(u >> 1);
                const uint32_t bytes = (u & 1) ? kTrunkW2Image : kTrunkW1Image;
                const uint8_t* src = (u & 1) ? args.w2_img + c * kTrunkW2Image : args.w1_img + c * kTrunkW1Image;
                mbar_arrive_expect_tx(&full[s], bytes);
                bulk_load_1d(smem + s * kRtSlot, src, bytes, &full[s]);
            }
        }
        return;
    }

    // -------------------------------------------------------------------- consumer warpgroup wg: one board
    if (NB > 1) asm volatile("setmaxnreg.inc.sync.aligned.u32 232;" ::: "memory");
    const int wg = warp >> 2;
    const int t = threadIdx.x & 127;
    const int w = t >> 5;
    const int board = static_cast<int>(blockIdx.x) * NB + wg;
    const bool board_ok = board * 64 < args.M;
    uint8_t* sX = smem + Cfg::kOffBoard + wg * Cfg::kBoardBytes;
    uint8_t* sH2 = sX + 32768;
    uint8_t* sH1 = sH2 + 8192;
    float* sPool = reinterpret_cast<float*>(sH1 + 8192);  // [256]
    float* sHid = sPool + 256;                             // [256]
    const uint32_t aX = smem_u32(sX), aH2 = smem_u32(sH2);
    // accumulator fragment of this thread: rows fr, fr + 8; columns 8 j + fc, 8 j + fc + 1
    const int fr = w * 16 + (lane >> 2), fc = 2 * (lane & 3);
    RT_PROF_DECL();

    rt_load_x(sX, args.x_in, board, board_ok, t);
    rt_wg_sync(wg);
    RT_PROF(0);  // X load

    float acc2[128];
    int u = 0;  // position in the weight stream
    for (int b = 0; b < n_blocks; ++b) {
        const TrunkBlock& B = args.blk[b];
        const int nch = B.n_chunks;
        // shortcut from the block input before the squeeze-excitation: MMA2 accumulates onto it
        const bool pre = MX && (B.flags & kTrunkShortcutPreSe);
        if (pre)
#pragma unroll
            for (int jj = 0; jj < 32; ++jj)
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const float2 xr = __half22float2(*reinterpret_cast<const __half2*>(sX + rt_x_off(fr + 8 * h, 8 * jj + fc)));
                    acc2[4 * jj + 2 * h] = xr.x, acc2[4 * jj + 2 * h + 1] = xr.y;
                }
        if (B.se_type != 0) rt_squeeze_excite<MX>(B, sX, sPool, sHid, t, wg);
        RT_PROF(1);  // squeeze-excitation

        for (int j = 0; j < nch; ++j) {
            // ---- MMA1: D1 = X . W1^T (4 K panels of 64)
            const int s1 = u % R;
            mbar_wait(&full[s1], (u / R) & 1);
            RT_PROF(2);  // wait for the W1 image
            const uint8_t* w1 = smem + s1 * kRtSlot;
            const uint32_t aW1 = smem_u32(w1);
            float acc1[32];
            wgmma_fence();
#pragma unroll
            for (int p = 0; p < 4; ++p)
#pragma unroll
                for (int k = 0; k < 4; ++k)
                    wgmma_f16<64>(acc1, wgmma_desc_k_sw128(aX + p * 8192 + k * 32, 1024),
                                  wgmma_desc_k_sw128(aW1 + p * 8192 + k * 32, 1024), (p > 0 || k > 0) ? 1u : 0u);
            wgmma_commit();
            wgmma_wait<0>();
            wgmma_fence_regs(acc1);
            RT_PROF(3);  // MMA1
            // ---- epilogue 1: relu(D1 + b1) -> H1
            const uint8_t* aux = w1 + kTrunkW1Tile;
            rt_epilogue1(acc1, aux, sH1, fr, fc);
            rt_wg_sync(wg);  // H1 complete (and MMA2 of the previous chunk, waited by every thread, is done with H2)
            RT_PROF(4);  // epilogue 1
            // ---- depthwise k x k -> H2 (A operand of MMA2) in the 128B-swizzled K-major layout
            rt_depthwise_stage(sH1, aux, sH2, B.ksize, t);
            fence_proxy_async();
            rt_wg_sync(wg);
            if (t == 0) mbar_arrive(&empty[s1]);  // the W1 image (tile and vectors) is no longer read
            ++u;
            RT_PROF(5);  // depthwise
            // ---- MMA2: D2 += H2 . W2^T
            const int s2 = u % R;
            mbar_wait(&full[s2], (u / R) & 1);
            RT_PROF(6);  // wait for the W2 image
            const uint32_t aW2 = smem_u32(smem + s2 * kRtSlot);
            wgmma_fence();
#pragma unroll
            for (int k = 0; k < 4; ++k)
                wgmma_f16<256>(acc2, wgmma_desc_k_sw128(aH2 + k * 32, 1024), wgmma_desc_k_sw128(aW2 + k * 32, 1024),
                               (pre || j > 0 || k > 0) ? 1u : 0u);
            wgmma_commit();
            wgmma_wait<0>();
            wgmma_fence_regs(acc2);
            if (t == 0) mbar_arrive(&empty[s2]);
            ++u;
            RT_PROF(7);  // MMA2
        }
        // ---- block epilogue: X <- (D2 + b2) + X, or D2 + b2 with the shortcut in D2 (the last block: to global memory)
        const bool last = b == n_blocks - 1;
#pragma unroll
        for (int jj = 0; jj < 32; ++jj) {
            const int c = 8 * jj + fc;
            const float2 b2 = __ldg(reinterpret_cast<const float2*>(B.b2 + c));
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int r = fr + 8 * h;
                __half2* x = reinterpret_cast<__half2*>(sX + rt_x_off(r, c));
                const float2 xr = pre ? make_float2(0.0f, 0.0f) : __half22float2(*x);
                const __half2 y = pre ? __floats2half2_rn(acc2[4 * jj + 2 * h] + b2.x, acc2[4 * jj + 2 * h + 1] + b2.y)
                                      : __floats2half2_rn((acc2[4 * jj + 2 * h] + b2.x) + xr.x, (acc2[4 * jj + 2 * h + 1] + b2.y) + xr.y);
                if (!last)
                    *x = y;
                else if (board_ok)
                    *reinterpret_cast<__half2*>(args.out + (static_cast<size_t>(board) * 64 + r) * 256 + c) = y;
            }
        }
        fence_proxy_async();
        rt_wg_sync(wg);
        RT_PROF(8);  // block epilogue
    }
    if (t == 0 && wg == 0) RT_PROF_FLUSH(1);
#endif
}


// ------------------------------------------------------------------------------------------------------------------
// Small batches: ONE BOARD PER CLUSTER OF TWO CTAs, which puts a 64-board batch on 128 SMs and halves each CTA's
// depthwise work and weight stream.  Chunk gc (counted over the whole tower) belongs to CTA gc & 1: the owner streams its
// W1 image, runs MMA1, epilogue 1 and the depthwise stage, and bulk-copies the 8 KB H2 tile into the partner's buffer of
// the same index.  Both CTAs run MMA2 for every chunk, in chunk order, each for its own 128 trunk channels (rows
// 128 r .. 128 r + 127 of the W2 image).
// Each CTA has two consumer warpgroups split by output channel, so that two warps share every SM sub-partition in the
// CUDA-core stages.  Warpgroup w runs MMA1 (wgmma m64n32), epilogue 1 and the depthwise stage for operating channels
// 32 w .. 32 w + 31 of a chunk (H1 / H2 channel groups 4 w .. 4 w + 3), and MMA2 (m64n64) and the block epilogue for trunk
// channels 128 r + 64 w .. 128 r + 64 w + 63, which are K panel 2 r + w of X: the new panel goes to the partner as one
// 8 KB bulk copy.  The squeeze-excitation is split across the pair: each CTA computes the outputs of its own channels
// from weights streamed through its W2 ring and stores them into both CTAs over DSMEM, so both scale their X copies
// with the same bits.  Every sum has the operands and the order of the one-CTA kernel: the outputs are the same bits.
struct RtPairCfg {
    static constexpr int kW1Ring = 2, kW2Ring = 4, kH2Bufs = 4;  // H2 buffer gc & 3 is filled by CTA gc & 1
    static constexpr int kW2Half = kTrunkW2Image / 2;
    static constexpr int kSeUnits = kTrunkSeImage / kW2Half;  // W2 ring units of a block's SE image, all resident at once
    static constexpr int kThreads = 256 + 64;  // two consumer warpgroups + the W1 and W2 producer warps
    static constexpr int kOffW1 = 0;
    static constexpr int kOffW2 = kOffW1 + kW1Ring * kTrunkW1Image;
    static constexpr int kOffX = kOffW2 + kW2Ring * kW2Half;  // [4 K panels][64 rows][128 B]
    static constexpr int kOffH2 = kOffX + 32768;              // [4 buffers][64 rows][128 B]
    static constexpr int kOffH1 = kOffH2 + kH2Bufs * 8192;    // [8 groups][64 squares][16 B]
    static constexpr int kOffSe = kOffH1 + 8192;              // pool[256] | hid[128] | scale[256] f32
    static constexpr int kOffBar = kOffSe + 2560;
    static constexpr int kSmemBytes = kOffBar + 256 + 1024 /*align slack*/;
    static_assert(kSeUnits <= kW2Ring, "a block's SE image must fit the W2 ring");
    static_assert(kSmemBytes <= 232448, "pair trunk kernel shared memory exceeds the sm_90 limit of 227 KB per block");
};

// both consumer warpgroups of a pair CTA (named barrier 3; 1 and 2 are the warpgroups' own)
__device__ __forceinline__ void rt_pair_sync() { asm volatile("bar.sync 3, 256;" ::: "memory"); }

// squeeze-excitation of the pair on the block input, in place; tid: 0 .. 255 over both consumer warpgroups.  Each CTA
// pools all 256 channels of its own X copy (thread tid: channel tid), then computes the outputs of its rank r from its
// SE image (unit i in ring slot (u2 + i) % kW2Ring), each one sequential sum: ca_se hidden 64 r .. 64 r + 63 (threads
// 0..63), exchanged through hid_bar, then the scales of channels 128 r .. 128 r + 127 (threads 0..127); eca_se those
// scales directly.  Every output is stored into both CTAs; the partner's stores are st.async that complete bytes on
// hid_bar / scale_bar, which thread 0 arms for 64 / 128 values.  hid_bar advances on ca_se blocks only, scale_bar on
// every SE block, so each has its own phase parity.  On return no thread reads the SE image any more.
template <bool MX>
__device__ __forceinline__ void rt_pair_squeeze_excite(const TrunkBlock& B, uint8_t* sX, const uint8_t* ring, int u2, float* sPool,
                                                       float* sHid, float* sScale, uint64_t* hid_bar, uint64_t* scale_bar,
                                                       uint32_t hid_parity, uint32_t scale_parity, uint32_t rank, int tid) {
    const uint32_t peer = rank ^ 1u;
    const auto unit = [&](int i) {
        return reinterpret_cast<const __half*>(ring + ((u2 + i) % RtPairCfg::kW2Ring) * RtPairCfg::kW2Half);
    };
    // thread 0 waited for the previous phase of both barriers in the previous SE.  The partner's stores of this phase may
    // land before the arm; those of the next phase cannot: the partner makes them only after it has received this CTA's
    // X panels of this block, which this CTA sends after this SE.
    if (tid == 0) {
        if (B.se_type == 1) mbar_arrive_expect_tx(hid_bar, 64 * 4);
        mbar_arrive_expect_tx(scale_bar, 128 * 4);
    }
    float s = 0.0f;
#pragma unroll 8
    for (int r = 0; r < 64; ++r) s += __half2float(*reinterpret_cast<const __half*>(sX + rt_x_off(r, tid)));
    sPool[tid] = s * (1.0f / 64.0f);
    rt_pair_sync();
    float sc = 0.0f;
    if (B.se_type == 1) {  // fc1 256 -> 128 (relu), fc2 128 -> 256 (hard sigmoid)
        if (tid < 64) {
            float a = 0.0f;
#pragma unroll 1
            for (int q = 0; q < 2; ++q) {  // [256 k][64]: 128 k per unit
                const __half* wq = unit(q) + tid;
#pragma unroll 16
                for (int k = 0; k < 128; ++k) a = fmaf(__half2float(wq[k * 64]), sPool[128 * q + k], a);
            }
            const int o = 64 * static_cast<int>(rank) + tid;
            const float h = fmaxf(rt_add_bias<MX>(B.se_b1, o, a), 0.0f);
            sHid[o] = h;
            st_async_cluster_b32(cluster_map(sHid + o, peer), __float_as_uint(h), cluster_map(hid_bar, peer));
        }
        if (tid < 128) {
            rt_wg_sync(0);                       // the own hidden values
            mbar_wait_cluster(hid_bar, hid_parity);  // the partner's
            float a = 0.0f;
#pragma unroll 1
            for (int q = 0; q < 2; ++q) {  // [128 j][128]: 64 j per unit
                const __half* wq = unit(2 + q) + tid;
#pragma unroll 16
                for (int j = 0; j < 64; ++j) a = fmaf(__half2float(wq[j * 128]), sHid[64 * q + j], a);
            }
            sc = rt_gate<MX>(rt_add_bias<MX>(B.se_b, 128 * static_cast<int>(rank) + tid, a), B.gate);
        }
    } else if (tid < 128) {  // 256 -> 256 + bias (hard sigmoid): [256 k][128], 64 k per unit
        float a = 0.0f;
#pragma unroll 1
        for (int q = 0; q < 4; ++q) {
            const __half* wq = unit(q) + tid;
#pragma unroll 16
            for (int k = 0; k < 64; ++k) a = fmaf(__half2float(wq[k * 128]), sPool[64 * q + k], a);
        }
        sc = rt_gate<MX>(__ldg(B.se_b + 128 * rank + tid) + a, B.gate);
    }
    if (tid < 128) {
        const int c = 128 * static_cast<int>(rank) + tid;
        sScale[c] = sc;
        st_async_cluster_b32(cluster_map(sScale + c, peer), __float_as_uint(sc), cluster_map(scale_bar, peer));
    }
    mbar_wait_cluster(scale_bar, scale_parity);  // the partner's scales
    rt_pair_sync();                        // the own scales
    // X *= scale: thread tid scales channels 2 (tid & 127), 2 (tid & 127) + 1 in rows 32 (tid >> 7) .. + 31
    const int cp = 2 * (tid & 127), r0 = 32 * (tid >> 7);
    const float sc0 = sScale[cp], sc1 = sScale[cp + 1];
#pragma unroll 8
    for (int r = r0; r < r0 + 32; ++r) {
        __half2* x = reinterpret_cast<__half2*>(sX + rt_x_off(r, cp));
        const float2 f = __half22float2(*x);
        *x = __floats2half2_rn(f.x * sc0, f.y * sc1);
    }
    fence_proxy_async();
    rt_pair_sync();
}

// launched with clusters of 2 CTAs along x: CTAs 2 i and 2 i + 1 run board i.  MX: as in rise_trunk_kernel
template <bool MX>
__global__ void __launch_bounds__(RtPairCfg::kThreads, 1) rise_trunk_pair_kernel(const __grid_constant__ TrunkArgs args) {
#if defined(__CUDA_ARCH__) && (__CUDA_ARCH__ >= 900)
    using Cfg = RtPairCfg;
    constexpr int R2 = Cfg::kW2Ring;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
    uint64_t* bars = reinterpret_cast<uint64_t*>(smem + Cfg::kOffBar);
    uint64_t* w1_full = bars;                        // [2]
    uint64_t* w1_empty = w1_full + Cfg::kW1Ring;     // [2]
    uint64_t* w2_full = w1_empty + Cfg::kW1Ring;     // [4]
    uint64_t* w2_empty = w2_full + R2;               // [4] one arrival per consumer warpgroup
    uint64_t* h2_full = w2_empty + R2;               // [4] (partner's buffers) local arm + the partner's bulk copy
    uint64_t* h2_free = h2_full + Cfg::kH2Bufs;      // [4] (own buffers) MMA2 done with it, both warpgroups of both CTAs
    uint64_t* x_full = h2_free + Cfg::kH2Bufs;       // local arm + the partner's two bulk copies of its X panels
    uint64_t* x_free = x_full + 1;                   // the partner no longer reads its X tile of this block
    uint64_t* se_hid = x_free + 1;                   // local arm + the partner's 64 ca_se hidden values (st.async)
    uint64_t* se_scale = se_hid + 1;                 // local arm + the partner's 128 SE scales (st.async)

    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;
    const uint32_t rank = cluster_ctarank(), peer = rank ^ 1u;
    const int board = static_cast<int>(blockIdx.x) >> 1;
    const int n_blocks = args.n_blocks;
    const int n_chunks = args.blk[n_blocks - 1].chunk0 + args.blk[n_blocks - 1].n_chunks;
    // device-side batch size: both CTAs of a cluster share the board, so they leave together
    if (args.boards_dev != nullptr && board >= *args.boards_dev) return;

    if (threadIdx.x == 0) {
        for (int i = 0; i < Cfg::kW1Ring; ++i) mbar_init(&w1_full[i], 1), mbar_init(&w1_empty[i], 1);
        for (int i = 0; i < R2; ++i) mbar_init(&w2_full[i], 1), mbar_init(&w2_empty[i], 2);
        for (int i = 0; i < Cfg::kH2Bufs; ++i) mbar_init(&h2_full[i], 1), mbar_init(&h2_free[i], 4);
        mbar_init(x_full, 1);
        mbar_init(x_free, 1);
        mbar_init(se_hid, 1);
        mbar_init(se_scale, 1);
        fence_mbar_init();
    }
    pdl_wait();
    pdl_launch_dependents();

    const int wg = warp >> 2;
    const int t = threadIdx.x & 127;
    const int w = t >> 5;
    const bool board_ok = board * 64 < args.M;
    uint8_t* sX = smem + Cfg::kOffX;
    uint8_t* sH1 = smem + Cfg::kOffH1;
    float* sPool = reinterpret_cast<float*>(smem + Cfg::kOffSe);
    float* sHid = sPool + 256;
    float* sScale = sHid + 128;
    RT_PROF_DECL();
    if (warp < 4) rt_load_x(sX, args.x_in, board, board_ok, t);
    // the partner's barriers exist before anything arrives on them, and both CTAs have read their input before either
    // writes the output (which may alias it)
    cluster_sync_all();

    if (warp >= 8) {
        // ---------------------------------------------------------------- producers: W1 images of the own chunks; SE
        // images and W2 halves of every block, in the order the consumers read them
        if (lane == 0) {
            if (warp == 8) {
                for (int gc = static_cast<int>(rank), u = 0; gc < n_chunks; gc += 2, ++u) {
                    const int s = u % Cfg::kW1Ring;
                    mbar_wait_relaxed(&w1_empty[s], ((u / Cfg::kW1Ring) & 1) ^ 1);
                    mbar_arrive_expect_tx(&w1_full[s], kTrunkW1Image);
                    bulk_load_1d(smem + Cfg::kOffW1 + s * kTrunkW1Image, args.w1_img + static_cast<size_t>(gc) * kTrunkW1Image,
                                 kTrunkW1Image, &w1_full[s]);
                }
            } else {
                int u = 0;
                for (int b = 0; b < n_blocks; ++b) {
                    const TrunkBlock& B = args.blk[b];
                    const int n_se = B.se_type != 0 ? Cfg::kSeUnits : 0;
                    for (int i = 0; i < n_se + B.n_chunks; ++i, ++u) {
                        const int s = u % R2;
                        mbar_wait_relaxed(&w2_empty[s], ((u / R2) & 1) ^ 1);
                        const uint8_t* src = i < n_se ? B.se_img + rank * kTrunkSeImage + i * Cfg::kW2Half
                                                      : args.w2_img + static_cast<size_t>(B.chunk0 + i - n_se) * kTrunkW2Image + rank * Cfg::kW2Half;
                        mbar_arrive_expect_tx(&w2_full[s], Cfg::kW2Half);
                        bulk_load_1d(smem + Cfg::kOffW2 + s * Cfg::kW2Half, src, Cfg::kW2Half, &w2_full[s]);
                    }
                }
            }
        }
        __syncwarp();
    } else {
        // -------------------------------------------------------------------- consumer warpgroup wg: a quarter of one board
        const uint32_t aX = smem_u32(sX);
        const int fr = w * 16 + (lane >> 2), fc = 2 * (lane & 3);
        RT_PROF(0);  // X load (and the cluster barrier)
        float acc2[32];
        int u2 = 0;    // position in the W2 ring's stream
        int n_se = 0;  // squeeze-excitations so far (phase of se_scale)
        int n_ca = 0;  // ca_se squeeze-excitations so far (phase of se_hid: eca_se blocks do not arrive on it)
        for (int b = 0; b < n_blocks; ++b) {
            const TrunkBlock& B = args.blk[b];
            const int nch = B.n_chunks;
            const int panel = 2 * static_cast<int>(rank) + wg;
            // shortcut from the block input before the squeeze-excitation: MMA2 accumulates onto it
            const bool pre = MX && (B.flags & kTrunkShortcutPreSe);
            if (pre)
#pragma unroll
                for (int jj = 0; jj < 8; ++jj)
#pragma unroll
                    for (int h = 0; h < 2; ++h) {
                        const float2 xr =
                            __half22float2(*reinterpret_cast<const __half2*>(sX + rt_x_off(fr + 8 * h, 64 * panel + 8 * jj + fc)));
                        acc2[4 * jj + 2 * h] = xr.x, acc2[4 * jj + 2 * h + 1] = xr.y;
                    }
            if (B.se_type != 0) {
                for (int i = 0; i < Cfg::kSeUnits; ++i) mbar_wait(&w2_full[(u2 + i) % R2], ((u2 + i) / R2) & 1);
                RT_PROF(1);  // wait for the SE image
                rt_pair_squeeze_excite<MX>(B, sX, smem + Cfg::kOffW2, u2, sPool, sHid, sScale, se_hid, se_scale, n_ca & 1, n_se & 1, rank,
                                       threadIdx.x);
                if (t == 0)
                    for (int i = 0; i < Cfg::kSeUnits; ++i) mbar_arrive(&w2_empty[(u2 + i) % R2]);
                u2 += Cfg::kSeUnits;
                ++n_se;
                n_ca += B.se_type == 1;
            }
            RT_PROF(2);  // squeeze-excitation
            int own = B.chunk0 + ((B.chunk0 & 1) != static_cast<int>(rank));  // the next own chunk without its H2
            for (int j = 0; j < nch; ++j) {
                const int gc = B.chunk0 + j;
                // the own chunk of {gc, gc + 1} first, so that the two CTAs run their depthwise stages side by side
                for (; own < B.chunk0 + nch && own <= gc + 1; own += 2) {
                    // ---- MMA1, epilogue 1, depthwise -> H2 buffer (this warpgroup's 32 channels), its copy to the partner
                    const int u1 = own >> 1, s1 = u1 % Cfg::kW1Ring;
                    uint8_t* oH2 = smem + Cfg::kOffH2 + (own & 3) * 8192;
                    mbar_wait(&w1_full[s1], (u1 / Cfg::kW1Ring) & 1);
                    RT_PROF(3);  // wait for the W1 image
                    const uint8_t* w1 = smem + Cfg::kOffW1 + s1 * kTrunkW1Image;
                    const uint32_t aW1 = smem_u32(w1) + wg * 4096;  // rows 32 wg .. of every K panel
                    float acc1[16];
                    wgmma_fence();
#pragma unroll
                    for (int p = 0; p < 4; ++p)
#pragma unroll
                        for (int k = 0; k < 4; ++k)
                            wgmma_f16<32>(acc1, wgmma_desc_k_sw128(aX + p * 8192 + k * 32, 1024),
                                          wgmma_desc_k_sw128(aW1 + p * 8192 + k * 32, 1024), (p > 0 || k > 0) ? 1u : 0u);
                    wgmma_commit();
                    wgmma_wait<0>();
                    wgmma_fence_regs(acc1);
                    RT_PROF(4);  // MMA1
                    const uint8_t* aux = w1 + kTrunkW1Tile;
                    rt_epilogue1(acc1, aux, sH1, fr, fc, 4 * wg);
                    rt_wg_sync(wg);  // the warpgroup's H1 groups are complete
                    RT_PROF(5);  // epilogue 1
                    // both CTAs' MMA2 of chunk own - 4 are done with the buffer
                    mbar_wait_cluster(&h2_free[own & 3], ((own >> 2) & 1) ^ 1);
                    RT_PROF(6);  // wait for the H2 buffer
                    rt_depthwise_stage<4>(sH1, aux, oH2, B.ksize, t, 4 * wg);
                    fence_proxy_async();
                    rt_pair_sync();  // H2 complete; no warpgroup reads the W1 image any more
                    if (threadIdx.x == 0) {
                        mbar_arrive(&w1_empty[s1]);
                        bulk_copy_to_cta(cluster_map(oH2, peer), oH2, 8192, cluster_map(&h2_full[own & 3], peer));
                    }
                    RT_PROF(7);  // depthwise
                }
                const int buf = gc & 3;
                uint8_t* sH2 = smem + Cfg::kOffH2 + buf * 8192;
                if ((gc & 1) != static_cast<int>(rank)) {
                    // ---- the partner's H2 of this chunk
                    if (threadIdx.x == 0) mbar_arrive_expect_tx(&h2_full[buf], 8192);
                    mbar_wait(&h2_full[buf], (gc >> 2) & 1);
                    RT_PROF(8);  // wait for the partner's H2
                }
                // ---- MMA2: D2[:, 64 p .. 64 p + 63] += H2 . W2[64 p .. 64 p + 63]^T, p = 2 r + wg
                const int s2 = u2 % R2;
                mbar_wait(&w2_full[s2], (u2 / R2) & 1);
                RT_PROF(9);  // wait for the W2 half
                const uint32_t aW2 = smem_u32(smem + Cfg::kOffW2 + s2 * Cfg::kW2Half) + wg * 8192, aH2 = smem_u32(sH2);
                wgmma_fence();
#pragma unroll
                for (int k = 0; k < 4; ++k)
                    wgmma_f16<64>(acc2, wgmma_desc_k_sw128(aH2 + k * 32, 1024), wgmma_desc_k_sw128(aW2 + k * 32, 1024),
                                  (pre || j > 0 || k > 0) ? 1u : 0u);
                wgmma_commit();
                wgmma_wait<0>();
                wgmma_fence_regs(acc2);
                if (t == 0) {
                    mbar_arrive(&w2_empty[s2]);
                    if ((gc & 1) == static_cast<int>(rank))
                        mbar_arrive(&h2_free[buf]);
                    else  // the partner overwrites this buffer with its next H2 (a bulk copy) after this arrival
                        mbar_arrive_cluster_free(cluster_map(&h2_free[buf], peer));
                }
                ++u2;
                RT_PROF(10);  // MMA2
            }
            // ---- block epilogue: X <- (D2 + b2) + X for K panel 2 r + wg, copied into the partner's X tile (the last
            // block: to global memory)
            const bool last = b == n_blocks - 1;
            rt_pair_sync();  // neither warpgroup reads this block's X any more
            if (!last) {
                if (threadIdx.x == 0) {
                    mbar_arrive_expect_tx(x_full, 2 * 8192);
                    // the partner bulk-copies its panels 2 peer + {0, 1} into this CTA's X tile after this arrival.  It
                    // publishes no data: this CTA's MMA1 reads of X completed at wgmma.wait_group and its SE reads were
                    // consumed before the pair barrier above, and its block epilogue touches only its own panels.
                    mbar_arrive_cluster_free(cluster_map(x_free, peer));
                }
                mbar_wait_cluster(x_free, b & 1);
            }
            RT_PROF(11);  // wait for the partner to release its X tile
#pragma unroll
            for (int jj = 0; jj < 8; ++jj) {
                const int c = 64 * panel + 8 * jj + fc;
                const float2 b2 = __ldg(reinterpret_cast<const float2*>(B.b2 + c));
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const int r = fr + 8 * h;
                    __half2* x = reinterpret_cast<__half2*>(sX + rt_x_off(r, c));
                    const float2 xr = pre ? make_float2(0.0f, 0.0f) : __half22float2(*x);
                    const __half2 y = pre ? __floats2half2_rn(acc2[4 * jj + 2 * h] + b2.x, acc2[4 * jj + 2 * h + 1] + b2.y)
                                          : __floats2half2_rn((acc2[4 * jj + 2 * h] + b2.x) + xr.x, (acc2[4 * jj + 2 * h + 1] + b2.y) + xr.y);
                    if (!last)
                        *x = y;
                    else if (board_ok)
                        *reinterpret_cast<__half2*>(args.out + (static_cast<size_t>(board) * 64 + r) * 256 + c) = y;
                }
            }
            if (!last) {
                fence_proxy_async();
                rt_wg_sync(wg);
                // nothing waits for this copy to finish reading the panel: the panel is written again (the next SE's
                // scaling, the next block epilogue) only after the partner has waited x_full for the copy and then
                // arrived on se_scale or x_free.  Keep that order when changing either step.
                if (t == 0) {
                    uint8_t* pX = sX + panel * 8192;
                    bulk_copy_to_cta(cluster_map(pX, peer), pX, 8192, cluster_map(x_full, peer));
                }
                RT_PROF(12);  // block epilogue and the copy
                mbar_wait(x_full, b & 1);  // the partner's two panels
                rt_pair_sync();            // the other warpgroup's panel
                RT_PROF(13);  // wait for the partner's channels of X
            }
        }
        if (t == 0 && wg == 0 && rank == 0) RT_PROF_FLUSH(0);
    }
    // no CTA leaves while its partner may still copy into or arrive on its shared memory
    cluster_sync_all();
#endif
}

}  // namespace ara
