// Host-side handle for one wgmma convolution layer (tensor maps + epilogue arguments).
#pragma once
#include "abi_common.h"
#include "conv_gemm.cuh"

namespace ara {

struct ConvLayer {
    CUtensorMap tm_a;
    CUtensorMap tm_b;
    ConvGemmArgs args;
    int bn;
    int n_out;
};

// Heuristic N-tile: biggest tile that still yields >= 120 CTAs, else 64.
int conv_layer_choose_bn(int boards, int n_out);

// act:  [boards_cap, 8, 8, cin] fp16 (boards_cap even), w: [w_rows, taps*ceil64(cin)] fp16 (w_rows % bn == 0),
// bias: [ldo] fp32 zero padded (or null), out: [boards*64, ldo].
int conv_layer_init(ConvLayer* L, const __half* act, int boards_cap, int cin, const __half* w, int w_rows, int n_out,
                    int ksize, const float* bias, int relu, const __half* residual, int ldr, __half* out_h,
                    float* out_f, int ldo, int bn);

// activations [boards_cap, 8, 8, cin] fp16 as the 4-D map the A operand is fetched through (conv_layer_init builds the
// same one): lets a layer be re-pointed at another input buffer
int make_act_tensor_map(CUtensorMap* m, const __half* act, int boards_cap, int cin);

// Precision float32: fp32 residual [M, ldr] instead of the fp16 one, and / or the hi | hi | lo split output
// [M, 3 * split_cs] (see conv_gemm.cuh); call after conv_layer_init.
void conv_layer_set_precise(ConvLayer* L, const float* residual_f, int ldr, __half* out_split, int split_cs);

// boards_dev (optional): device-side count of the boards in use, <= boards (see ConvGemmArgs::boards_dev)
int conv_layer_launch(const ConvLayer* L, int boards, cudaStream_t stream, const int* boards_dev = nullptr);

}  // namespace ara
