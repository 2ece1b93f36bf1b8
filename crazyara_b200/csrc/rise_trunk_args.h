// Argument block of the persistent trunk kernel (rise_trunk.cuh): every bottleneck block of the RISE tower.
#pragma once
#include <cuda_fp16.h>
#include <stdint.h>

namespace ara {

constexpr int kTrunkMaxBlocks = 24;
// One 64-channel chunk of a block travels as two pre-tiled images (exact shared-memory byte images, 128B-swizzled
// K-major, so that each is ONE 1-D bulk copy):
//   W1 image: [64 rows x 256 K] fp16 as 4 K-panels of 8 KB, then b1[64] f32 | bd[64] f32 | wd[k*k][64] f16
//   W2 image: [256 rows x 64 K] fp16
constexpr int kTrunkW1Tile = 32768;
constexpr int kTrunkAuxBytes = 3712;   // 64 f32 + 64 f32 + 25 * 64 f16
constexpr int kTrunkW1Image = 36864;   // tile + aux, padded to 1 KB
constexpr int kTrunkW2Image = 32768;
// Squeeze-excitation image of a block for one CTA of rise_trunk_pair_kernel (rank r), fp16:
//   ca_se:  fc1 columns 64 r .. 64 r + 63 as [256 k][64]  |  fc2 columns 128 r .. 128 r + 127 as [128 j][128]
//   eca_se: columns 128 r .. 128 r + 127 as [256 k][128]
constexpr int kTrunkSeImage = 65536;

// the residual adds the block input as it was before the squeeze-excitation scaled it (MXNet RISE symbols)
constexpr int kTrunkShortcutPreSe = 1;
// squeeze-excitation gates: clamp(x / 6 + 0.5) (torch Hardsigmoid), clamp(0.2 x + 0.5) (MXNet hard_sigmoid), sigmoid
constexpr int kTrunkGateHard6 = 0, kTrunkGateHard5 = 1, kTrunkGateSigmoid = 2;

struct TrunkBlock {
    int n_chunks;     // ceil(Cop / 64)
    int ksize;        // depthwise kernel: 3 or 5
    int se_type;      // 0 none, 1 ca_se, 2 eca_se (applied to the block input, in place)
    int chunk0;       // index of the block's first chunk in the image arrays
    const float* b2;       // [256]
    const __half* se_w1t;  // ca_se: [256][128]; eca_se: [256][256] (transposed, fp16 copy owned by the trunk)
    const __half* se_w2t;  // ca_se: [128][256]
    const float* se_b;     // eca_se: [256]; ca_se: fc2 bias [256] or null
    const uint8_t* se_img;  // [2 ranks][kTrunkSeImage] (rise_trunk_pair_kernel)
    // read only by the kernels built for the MXNet semantics (RiseTrunk::mx):
    int flags;             // kTrunkShortcutPreSe
    int gate;              // squeeze-excitation gate, kTrunkGate*
    const float* se_b1;    // ca_se: fc1 bias [128] or null
};

struct TrunkArgs {
    int M;         // valid rows (= boards * 64)
    int n_blocks;
    const uint8_t* w1_img;  // [chunks][kTrunkW1Image]
    const uint8_t* w2_img;  // [chunks][kTrunkW2Image]
    const __half* x_in;     // [M, 256] stem output
    __half* out;            // [M, 256]
    const int* boards_dev;     // device-side count of the boards in use (or nullptr): CTAs beyond it leave at once
    unsigned long long* prof;  // profiling builds (-DARA_TRUNK_PROF): [2][16] cycle counters of CTA 0, else unused
    TrunkBlock blk[kTrunkMaxBlocks];
};

}  // namespace ara
