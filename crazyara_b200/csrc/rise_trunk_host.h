// Host handle of the persistent trunk kernel (rise_trunk.cuh): stacks the weights of every bottleneck block into the
// two matrices the kernel streams through its weight ring and builds the per-chunk vector records.
#pragma once
#include <cuda.h>

#include <vector>

#include "abi_common.h"
#include "rise_trunk_args.h"

namespace ara {

struct TrunkBlockHost {
    int c_op = 0, ksize = 3, se_type = 0;
    std::vector<float> w1;  // [c_op][256]   conv1x1 256 -> c_op (BN folded)
    std::vector<float> b1;  // [c_op]
    std::vector<float> wd;  // [c_op][k*k]   depthwise (BN folded)
    std::vector<float> bd;  // [c_op]
    std::vector<float> w2;  // [256][c_op]   conv1x1 c_op -> 256 (BN folded)
    std::vector<float> b2;  // [256]
    std::vector<float> se_w1t;  // transposed squeeze-excitation, see TrunkBlock: ca_se [256][128], eca_se [256][256]
    std::vector<float> se_w2t;  // ca_se: [128][256]
    std::vector<float> se_b;    // eca_se: [256]; ca_se: fc2 bias [256] or empty
    std::vector<float> se_b1;   // ca_se: fc1 bias [128] or empty
    int flags = 0, gate = kTrunkGateHard6;  // see TrunkBlock
};

struct RiseTrunk {
    TrunkArgs args;
    int sm_count = 0;
    int pair_clusters = 0;  // CTA pairs of rise_trunk_pair_kernel resident at once
    bool mx = false;        // some block needs the kernels built for the MXNet semantics
    unsigned long long* d_prof = nullptr;  // [2][16] cycle counters, written only by -DARA_TRUNK_PROF builds
    DeviceBuffers mem;  // everything the pointers in args and d_prof point to
};

// x_in: [boards, 8, 8, 256] fp16 (stem output); out: [boards*64, 256] fp16 (may alias x_in: every CTA reads its
// own rows before it writes them)
int rise_trunk_init(RiseTrunk* T, const std::vector<TrunkBlockHost>& blocks, const __half* x_in, __half* out);
// x_in (optional): another stem-output buffer than the one given to rise_trunk_init (a second input / output set)
int rise_trunk_launch(const RiseTrunk* T, int boards, cudaStream_t stream, const int* boards_dev = nullptr, const __half* x_in = nullptr);
// the CTAs of that launch
int rise_trunk_ctas(const RiseTrunk* T, int boards);

}  // namespace ara
