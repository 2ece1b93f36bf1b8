// Host side of the wgmma convolution GEMM: TMA tensor-map construction and launch.
#include "conv_gemm_host.h"

#include <cstring>

namespace ara {

typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static PFN_encodeTiled get_encode_fn() {
    static PFN_encodeTiled fn = nullptr;
    if (fn == nullptr) {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) != cudaSuccess ||
            q != cudaDriverEntryPointSuccess)
            return nullptr;
        fn = reinterpret_cast<PFN_encodeTiled>(p);
    }
    return fn;
}

// activations [boards_cap, 8, 8, cin] fp16 as a 4-D map with box {64 ch, 8, 8, 2 boards}, 128-B swizzle, zero OOB fill
int make_act_tensor_map(CUtensorMap* m, const __half* act, int boards_cap, int cin) {
    PFN_encodeTiled enc = get_encode_fn();
    if (enc == nullptr) return set_error("cuTensorMapEncodeTiled entry point not available");
    if (cin % 8 != 0 || boards_cap < 2 || (boards_cap & 1)) return set_error("make_act_tensor_map: bad shape (%d, %d)", boards_cap, cin);
    cuuint64_t dims[4] = {(cuuint64_t)cin, 8, 8, (cuuint64_t)boards_cap};
    cuuint64_t strides[3] = {(cuuint64_t)cin * 2, (cuuint64_t)cin * 16, (cuuint64_t)cin * 128};
    cuuint32_t box[4] = {64, 8, 8, 2};
    cuuint32_t estr[4] = {1, 1, 1, 1};
    CUresult r = enc(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4, const_cast<__half*>(act), dims, strides, box, estr,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) return set_error("cuTensorMapEncodeTiled(act) failed: %d", (int)r);
    return 0;
}
// weights [rows, k_total] fp16 K-major as a 2-D map with box {64 k, box_rows}
int make_weight_tensor_map(CUtensorMap* m, const __half* w, int k_total, int rows, int box_rows) {
    PFN_encodeTiled enc = get_encode_fn();
    if (enc == nullptr) return set_error("cuTensorMapEncodeTiled entry point not available");
    cuuint64_t dims[2] = {(cuuint64_t)k_total, (cuuint64_t)rows};
    cuuint64_t strides[1] = {(cuuint64_t)k_total * 2};
    cuuint32_t box[2] = {64, (cuuint32_t)box_rows};
    cuuint32_t estr[2] = {1, 1};
    CUresult r = enc(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, const_cast<__half*>(w), dims, strides, box, estr,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) return set_error("cuTensorMapEncodeTiled(weights) failed: %d", (int)r);
    return 0;
}

int conv_layer_choose_bn(int boards, int n_out) {
    const int m_tiles = (boards + 1) / 2;
    const int cands[3] = {256, 128, 64};
    for (int i = 0; i < 3; ++i) {
        const int bn = cands[i];
        if (bn > 64 && n_out < bn) continue;
        const int tiles = m_tiles * ((n_out + bn - 1) / bn);
        if (tiles >= 120) return bn;
    }
    return 64;
}

template <int BN>
static cudaError_t allow_smem() {
    return cudaFuncSetAttribute(conv_gemm_kernel<BN>, cudaFuncAttributeMaxDynamicSharedMemorySize, ConvGemmCfg<BN>::kSmemBytes);
}

int conv_layer_init(ConvLayer* L, const __half* act, int boards_cap, int cin, const __half* w, int w_rows,
                    int n_out, int ksize, const float* bias, int relu, const __half* residual, int ldr,
                    __half* out_h, float* out_f, int ldo, int bn) {
    if (cin % 8 != 0) return set_error("conv_layer_init: cin=%d must be a multiple of 8", cin);
    if (ldo % 32 != 0) return set_error("conv_layer_init: ldo=%d must be a multiple of 32", ldo);
    if (boards_cap < 2 || (boards_cap & 1)) return set_error("conv_layer_init: boards_cap=%d must be even >= 2", boards_cap);
    if (ksize != 1 && ksize != 3) return set_error("conv_layer_init: ksize=%d unsupported", ksize);
    if (bn != 64 && bn != 128 && bn != 256) return set_error("conv_layer_init: bn=%d unsupported", bn);
    if (w_rows % bn != 0) return set_error("conv_layer_init: weight rows %d not a multiple of bn %d", w_rows, bn);
    memset(L, 0, sizeof(*L));
    const int c_chunks = (cin + 63) / 64;
    const int cw = c_chunks * 64;
    const int taps = ksize * ksize;
    if (make_act_tensor_map(&L->tm_a, act, boards_cap, cin) || make_weight_tensor_map(&L->tm_b, w, taps * cw, w_rows, bn)) return -1;
    ARA_CUDA_OK(bn == 64 ? allow_smem<64>() : bn == 128 ? allow_smem<128>() : allow_smem<256>());
    L->bn = bn;
    L->n_out = n_out;
    L->args.M = 0;
    L->args.N = n_out;
    L->args.c_chunks = c_chunks;
    L->args.cw = cw;
    L->args.ksize = ksize;
    L->args.relu = relu;
    L->args.bias = bias;
    L->args.residual = residual;
    L->args.ldr = ldr;
    L->args.out_h = out_h;
    L->args.out_f = out_f;
    L->args.ldo = ldo;
    return 0;
}

void conv_layer_set_precise(ConvLayer* L, const float* residual_f, int ldr, __half* out_split, int split_cs) {
    L->args.residual_f = residual_f;
    if (residual_f != nullptr) L->args.ldr = ldr;
    L->args.out_split = out_split;
    L->args.split_cs = split_cs;
}

template <int BN>
static int launch_bn(const ConvLayer* L, const ConvGemmArgs& a, dim3 grid, cudaStream_t stream) {
    ARA_CUDA_OK(launch_pdl(conv_gemm_kernel<BN>, grid, dim3(kGemmThreads), ConvGemmCfg<BN>::kSmemBytes, stream, L->tm_a, L->tm_b, a));
    return 0;
}

int conv_layer_launch(const ConvLayer* L, int boards, cudaStream_t stream, const int* boards_dev) {
    ConvGemmArgs a = L->args;
    a.M = boards * 64;
    a.boards_dev = boards_dev;
    dim3 grid((boards + 1) / 2, (L->n_out + L->bn - 1) / L->bn, 1);
    switch (L->bn) {
        case 64: return launch_bn<64>(L, a, grid, stream);
        case 128: return launch_bn<128>(L, a, grid, stream);
        case 256: return launch_bn<256>(L, a, grid, stream);
    }
    return set_error("conv_layer_launch: bad bn %d", L->bn);
}

}  // namespace ara

// Debug / unit-test entry: run one convolution layer on caller-provided device buffers.
extern "C" int ara_debug_conv(const void* act_half, int boards_cap, int boards, int cin, const void* w_half, int w_rows,
                              int n_out, int ksize, const float* bias, int relu, const void* residual, int ldr,
                              void* out_half, float* out_f32, int ldo, int bn, void* stream) {
    ara::ConvLayer L;
    if (bn == 0) bn = ara::conv_layer_choose_bn(boards, n_out);
    int rc = ara::conv_layer_init(&L, (const __half*)act_half, boards_cap, cin, (const __half*)w_half, w_rows, n_out,
                                  ksize, bias, relu, (const __half*)residual, ldr, (__half*)out_half, out_f32, ldo, bn);
    if (rc != 0) return rc;
    rc = ara::conv_layer_launch(&L, boards, (cudaStream_t)stream);
    if (rc != 0) return rc;
    cudaError_t e = cudaStreamSynchronize((cudaStream_t)stream);
    if (e != cudaSuccess) return ara::set_error("ara_debug_conv: %s", cudaGetErrorString(e));
    return 0;
}

extern "C" int ara_debug_choose_bn(int boards, int n_out) { return ara::conv_layer_choose_bn(boards, n_out); }
