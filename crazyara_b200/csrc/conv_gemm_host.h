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
// Which main loop a layer runs: true for the 3x3 layers whose c_chunks A tiles fit in shared memory beside the B ring
// of N tile bn (each CTA loads its activations once and feeds every tap from them); false for the streaming loop, which
// fetches the shifted A tile of every (tap, chunk) by TMA and runs any layer.
bool conv_resident_a(int ksize, int c_chunks, int bn);

// act:  [boards_cap, 8, 8, cin] fp16 (boards_cap even), w: [w_rows, taps*ceil64(cin)] fp16 (w_rows % bn == 0),
// bias: [ldo] fp32 zero padded (or null), out: [boards*64, ldo].  act_pitch (0: cin): the activation rows are act_pitch
// channels apart, so a layer can read channels 0..cin-1 of a wider row (act 16-byte aligned, act_pitch % 8 == 0).
// args.n_end (set to ldo here) may be lowered afterwards so that the layer writes only columns 0..n_end-1 of its rows.
int conv_layer_init(ConvLayer* L, const __half* act, int boards_cap, int cin, const __half* w, int w_rows, int n_out,
                    int ksize, const float* bias, int relu, const __half* residual, int ldr, __half* out_h,
                    float* out_f, int ldo, int bn, int act_pitch = 0);

// activations [boards_cap, 8, 8, cin] fp16 as the 4-D map the A operand is fetched through (conv_layer_init builds the
// same one): lets a layer be re-pointed at another input buffer
int make_act_tensor_map(CUtensorMap* m, const __half* act, int boards_cap, int cin, int pitch = 0);
// a K-major fp16 matrix [rows][k_total] as the 2-D map with box {64 k, box_rows} and the 128-byte swizzle the wgmma
// operand descriptors read (the layers' weights; the fully-connected policy head's operands)
int make_weight_tensor_map(CUtensorMap* m, const __half* w, int k_total, int rows, int box_rows);

// Precision float32: fp32 residual [M, ldr] instead of the fp16 one, and / or the hi | hi | lo split output
// [M, 3 * split_cs] (see conv_gemm.cuh); call after conv_layer_init.
void conv_layer_set_precise(ConvLayer* L, const float* residual_f, int ldr, __half* out_split, int split_cs);

// boards_dev (optional): device-side count of the boards in use, <= boards (see ConvGemmArgs::boards_dev)
int conv_layer_launch(const ConvLayer* L, int boards, cudaStream_t stream, const int* boards_dev = nullptr);
// the CTAs of that launch
int conv_layer_ctas(const ConvLayer* L, int boards);

// Where one conv_gemm layer reads and writes.  act: the activations, rows act_pitch channels apart (0: act_cin); float16
// reads channels 0 .. act_cin (0: the layer's cin), float32 the split [.., 3 * ceil64(cin)].  The epilogue adds the fp16
// or fp32 residual (rows ldr apart) and writes columns 0 .. n_end (0: ldo) of the fp16, fp32 and / or split outputs
// (rows ldo apart, split parts split_cs wide).
struct ConvIo {
    const __half* act = nullptr;
    int act_cin = 0, act_pitch = 0;
    const __half* res_h = nullptr;
    const float* res_f = nullptr;
    int ldr = 0;
    __half* out_h = nullptr;
    float* out_f = nullptr;
    __half* out_s = nullptr;
    int ldo = 0, n_end = 0, split_cs = 0;
};

// One layer of a network in `precision` (0 float16, 1 float32 = split operands): the weight image w [w_rows][taps *
// parts * ceil64(cin)] (parts 1, or 3 for [hi | lo | hi], Net::upload_conv_w), bias [w_rows] or null, the activations and
// outputs of io, N tile bn.  Net::build_conv and ara_debug_conv both build their layers here.
int conv_layer_build(ConvLayer* L, const __half* w, int w_rows, const float* bias, int n_out, int cin, int ksize, int relu,
                     int precision, int boards_cap, int bn, const ConvIo& io);

}  // namespace ara
