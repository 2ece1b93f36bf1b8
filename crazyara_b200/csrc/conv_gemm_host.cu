// Host side of the wgmma convolution GEMM: TMA tensor-map construction and launch.
#include "conv_gemm_host.h"

#include <cstring>

#include "ara_b200.h"

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

// activations [boards_cap, 8, 8, cin] fp16 (rows `pitch` >= cin channels apart) as a 4-D map with box {64 ch, 8, 8, 2 boards},
// 128-B swizzle, zero OOB fill: channels cin.. of a box read as zero
int make_act_tensor_map(CUtensorMap* m, const __half* act, int boards_cap, int cin, int pitch) {
    PFN_encodeTiled enc = get_encode_fn();
    if (enc == nullptr) return set_error("cuTensorMapEncodeTiled entry point not available");
    if (pitch == 0) pitch = cin;
    if (cin % 8 != 0 || pitch % 8 != 0 || pitch < cin || boards_cap < 2 || (boards_cap & 1) || (reinterpret_cast<uintptr_t>(act) & 15))
        return set_error("make_act_tensor_map: bad shape (%d, %d, pitch %d)", boards_cap, cin, pitch);
    cuuint64_t dims[4] = {(cuuint64_t)cin, 8, 8, (cuuint64_t)boards_cap};
    cuuint64_t strides[3] = {(cuuint64_t)pitch * 2, (cuuint64_t)pitch * 16, (cuuint64_t)pitch * 128};
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

// N tiles up to 128: at 256 the accumulators (128 registers) leave no room beside them for the fragment sets of the
// resident loop under the 168-register ceiling of a 288-thread block, and groups of half a k block ran slower than streaming
bool conv_resident_a(int ksize, int c_chunks, int bn) {
    if (ksize != 3) return false;
    if (bn == 64) return c_chunks <= ConvGemmCfg<64>::kResidentMaxChunks;
    if (bn == 128) return c_chunks <= ConvGemmCfg<128>::kResidentMaxChunks;
    return false;
}

template <int BN>
static cudaError_t allow_smem() {
    using Cfg = ConvGemmCfg<BN>;
    cudaError_t e = cudaFuncSetAttribute(conv_gemm_kernel<BN, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::kSmemBytes);
    if constexpr (BN <= 128)
        if (e == cudaSuccess)
            e = cudaFuncSetAttribute(conv_gemm_kernel<BN, true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                     Cfg::resident_smem_bytes(Cfg::kResidentMaxChunks));
    return e;
}

int conv_layer_init(ConvLayer* L, const __half* act, int boards_cap, int cin, const __half* w, int w_rows,
                    int n_out, int ksize, const float* bias, int relu, const __half* residual, int ldr,
                    __half* out_h, float* out_f, int ldo, int bn, int act_pitch) {
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
    if (make_act_tensor_map(&L->tm_a, act, boards_cap, cin, act_pitch) || make_weight_tensor_map(&L->tm_b, w, taps * cw, w_rows, bn)) return -1;
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
    L->args.n_end = ldo;
    return 0;
}

void conv_layer_set_precise(ConvLayer* L, const float* residual_f, int ldr, __half* out_split, int split_cs) {
    L->args.residual_f = residual_f;
    if (residual_f != nullptr) L->args.ldr = ldr;
    L->args.out_split = out_split;
    L->args.split_cs = split_cs;
}

int conv_layer_build(ConvLayer* L, const __half* w, int w_rows, const float* bias, int n_out, int cin, int ksize, int relu,
                     int precision, int boards_cap, int bn, const ConvIo& io) {
    const int act_cin = precision == 0 ? (io.act_cin ? io.act_cin : cin) : 3 * ((cin + 63) / 64 * 64);
    if (conv_layer_init(L, io.act, boards_cap, act_cin, w, w_rows, n_out, ksize, bias, relu, io.res_h, io.ldr, io.out_h, io.out_f,
                        io.ldo, bn, io.act_pitch))
        return -1;
    if (precision == 1) conv_layer_set_precise(L, io.res_f, io.ldr, io.out_s, io.split_cs);
    if (io.n_end) L->args.n_end = io.n_end;
    return 0;
}

template <int BN>
static int launch_bn(const ConvLayer* L, const ConvGemmArgs& a, dim3 grid, cudaStream_t stream) {
    using Cfg = ConvGemmCfg<BN>;
    if constexpr (BN <= 128)
        if (conv_resident_a(a.ksize, a.c_chunks, BN)) {
            ARA_CUDA_OK(launch_pdl(conv_gemm_kernel<BN, true>, grid, dim3(kGemmThreads), Cfg::resident_smem_bytes(a.c_chunks),
                                   stream, L->tm_a, L->tm_b, a));
            return 0;
        }
    ARA_CUDA_OK(launch_pdl(conv_gemm_kernel<BN, false>, grid, dim3(kGemmThreads), Cfg::kSmemBytes, stream, L->tm_a, L->tm_b, a));
    return 0;
}

static dim3 conv_layer_grid(const ConvLayer* L, int boards) { return dim3((boards + 1) / 2, (L->n_out + L->bn - 1) / L->bn, 1); }

int conv_layer_ctas(const ConvLayer* L, int boards) {
    const dim3 g = conv_layer_grid(L, boards);
    return static_cast<int>(g.x * g.y);
}

int conv_layer_launch(const ConvLayer* L, int boards, cudaStream_t stream, const int* boards_dev) {
    ConvGemmArgs a = L->args;
    a.M = boards * 64;
    a.boards_dev = boards_dev;
    const dim3 grid = conv_layer_grid(L, boards);
    switch (L->bn) {
        case 64: return launch_bn<64>(L, a, grid, stream);
        case 128: return launch_bn<128>(L, a, grid, stream);
        case 256: return launch_bn<256>(L, a, grid, stream);
    }
    return set_error("conv_layer_launch: bad bn %d", L->bn);
}

}  // namespace ara

// Debug / unit-test entry: one convolution layer on caller-provided device buffers, built and launched as a network's.
extern "C" int ara_debug_conv(const ara_debug_conv_t* a, void* stream) {
    if (a == nullptr) return ara::set_error("ara_debug_conv: null arguments");
    // the argument block is read on the host: a device pointer in its place (e.g. a buffer handed over where the struct
    // belongs) is refused here instead of being dereferenced
    cudaPointerAttributes pa;
    if (cudaPointerGetAttributes(&pa, a) != cudaSuccess) {
        cudaGetLastError();
        return ara::set_error("ara_debug_conv: the argument pointer is not a host address");
    }
    if (pa.type == cudaMemoryTypeDevice) return ara::set_error("ara_debug_conv: the arguments are in device memory, not on the host");
    if (a->precision != ARA_PRECISION_FLOAT16 && a->precision != ARA_PRECISION_FLOAT32)
        return ara::set_error("ara_debug_conv: precision %d (0 = float16, 1 = float32)", a->precision);
    if (a->boards < 1 || a->boards > a->boards_cap) return ara::set_error("ara_debug_conv: %d boards of %d", a->boards, a->boards_cap);
    ara::ConvIo io;
    io.act = (const __half*)a->act;
    io.act_cin = a->act_cin;
    io.act_pitch = a->act_pitch;
    io.res_h = (const __half*)a->res_h;
    io.res_f = a->res_f;
    io.ldr = a->ldr;
    io.out_h = (__half*)a->out_h;
    io.out_f = a->out_f;
    io.out_s = (__half*)a->out_s;
    io.ldo = a->ldo;
    io.n_end = a->n_end;
    io.split_cs = a->split_cs;
    const int bn = a->bn ? a->bn : ara::conv_layer_choose_bn(a->boards, a->n_out);
    ara::ConvLayer L;
    int rc = ara::conv_layer_build(&L, (const __half*)a->w, a->w_rows, a->bias, a->n_out, a->cin, a->ksize, a->relu, a->precision,
                                   a->boards_cap, bn, io);
    if (rc != 0) return rc;
    rc = ara::conv_layer_launch(&L, a->boards, (cudaStream_t)stream, a->boards_dev);
    if (rc != 0) return rc;
    cudaError_t e = cudaStreamSynchronize((cudaStream_t)stream);
    if (e != cudaSuccess) return ara::set_error("ara_debug_conv: %s", cudaGetErrorString(e));
    return 0;
}

extern "C" int ara_debug_choose_bn(int boards, int n_out) { return ara::conv_layer_choose_bn(boards, n_out); }
