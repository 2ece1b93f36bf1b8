#include "rise_trunk_host.h"

#include <cstdlib>
#include <cstring>

#include "rise_trunk.cuh"

namespace ara {

namespace {

// byte offset of element (row, k) inside a K-major tile with 128-byte rows and the 128B swizzle (16-byte chunks XORed
// with the row index modulo 8): the layout TMA's SWIZZLE_128B produces and the wgmma shared-memory descriptor reads
inline size_t sw128_offset(int row, int k) { return static_cast<size_t>(row) * 128 + ((((k >> 3) ^ (row & 7)) << 4)) + (k & 7) * 2; }

template <typename T>
int upload(DeviceBuffers& mem, const std::vector<T>& h, const T** dst) {
    T* d = nullptr;
    if (mem.dalloc(&d, h.size())) return -1;
    ARA_CUDA_OK(cudaMemcpy(d, h.data(), h.size() * sizeof(T), cudaMemcpyHostToDevice));
    *dst = d;
    return 0;
}

}  // namespace

int rise_trunk_init(RiseTrunk* T, const std::vector<TrunkBlockHost>& blocks, const __half* x_in, __half* out) {
    const int nb = static_cast<int>(blocks.size());
    if (nb < 1 || nb > kTrunkMaxBlocks) return set_error("rise_trunk_init: %d blocks unsupported (max %d)", nb, kTrunkMaxBlocks);
    memset(&T->args, 0, sizeof(T->args));
    int chunks = 0;
    for (int i = 0; i < nb; ++i) {
        const TrunkBlockHost& h = blocks[i];
        if (h.ksize != 3 && h.ksize != 5) return set_error("rise_trunk_init: depthwise kernel %d unsupported", h.ksize);
        if (h.c_op < 1) return set_error("rise_trunk_init: block %d has no operating channels", i);
        TrunkBlock& B = T->args.blk[i];
        B.n_chunks = (h.c_op + 63) / 64;
        B.ksize = h.ksize;
        B.se_type = h.se_type;
        B.chunk0 = chunks;
        B.flags = h.flags;
        B.gate = h.gate;
        if (h.gate < kTrunkGateHard6 || h.gate > kTrunkGateSigmoid) return set_error("rise_trunk_init: block %d has gate %d", i, h.gate);
        T->mx = T->mx || h.flags != 0 || h.gate != kTrunkGateHard6 || !h.se_b1.empty();
        if (upload(T->mem, h.b2, &B.b2)) return -1;
        if (h.se_type != 0) {  // fp16 copies of the squeeze-excitation matrices (the kernel is bound by their traffic)
            const size_t n1 = h.se_type == 1 ? 256 * 128 : 256 * 256, n2 = h.se_type == 1 ? 128 * 256 : 0;
            if (!h.se_b.empty() && upload(T->mem, h.se_b, &B.se_b)) return -1;
            if (!h.se_b1.empty() && upload(T->mem, h.se_b1, &B.se_b1)) return -1;
            std::vector<__half> hh(n1 + n2);
            for (size_t k = 0; k < n1; ++k) hh[k] = __float2half_rn(h.se_w1t[k]);
            for (size_t k = 0; k < n2; ++k) hh[n1 + k] = __float2half_rn(h.se_w2t[k]);
            if (upload(T->mem, hh, &B.se_w1t)) return -1;
            B.se_w2t = n2 ? B.se_w1t + n1 : nullptr;
            // the pair kernel's images: each CTA gets the columns of the outputs it computes
            std::vector<__half> img(2 * kTrunkSeImage / sizeof(__half));
            for (int r = 0; r < 2; ++r) {
                __half* o = img.data() + r * kTrunkSeImage / sizeof(__half);
                if (h.se_type == 1) {
                    for (int k = 0; k < 256; ++k)
                        for (int i = 0; i < 64; ++i) o[k * 64 + i] = hh[k * 128 + 64 * r + i];
                    for (int j = 0; j < 128; ++j)
                        for (int i = 0; i < 128; ++i) o[256 * 64 + j * 128 + i] = hh[n1 + j * 256 + 128 * r + i];
                } else {
                    for (int k = 0; k < 256; ++k)
                        for (int i = 0; i < 128; ++i) o[k * 128 + i] = hh[k * 256 + 128 * r + i];
                }
            }
            const __half* d_img = nullptr;
            if (upload(T->mem, img, &d_img)) return -1;
            B.se_img = reinterpret_cast<const uint8_t*>(d_img);
        }
        chunks += B.n_chunks;
    }
    T->args.n_blocks = nb;
    T->args.x_in = x_in;
    T->args.out = out;
    // pre-tiled images: every chunk's weights laid out exactly as the bytes the kernel wants in shared memory
    std::vector<uint8_t> w1(static_cast<size_t>(chunks) * kTrunkW1Image, 0);
    std::vector<uint8_t> w2(static_cast<size_t>(chunks) * kTrunkW2Image, 0);
    for (int i = 0; i < nb; ++i) {
        const TrunkBlockHost& h = blocks[i];
        const TrunkBlock& B = T->args.blk[i];
        const int kk = h.ksize * h.ksize;
        for (int j = 0; j < B.n_chunks; ++j) {
            uint8_t* img1 = w1.data() + static_cast<size_t>(B.chunk0 + j) * kTrunkW1Image;
            uint8_t* img2 = w2.data() + static_cast<size_t>(B.chunk0 + j) * kTrunkW2Image;
            float* aux_f = reinterpret_cast<float*>(img1 + kTrunkW1Tile);
            __half* aux_w = reinterpret_cast<__half*>(img1 + kTrunkW1Tile + 512);
            for (int cc = 0; cc < 64; ++cc) {
                const int c = j * 64 + cc;
                if (c >= h.c_op) break;
                // W1 tile: row = operating channel, K = the 256 trunk channels in 4 panels of 64
                for (int k = 0; k < 256; ++k)
                    *reinterpret_cast<__half*>(img1 + (k >> 6) * 8192 + sw128_offset(cc, k & 63)) =
                        __float2half_rn(h.w1[static_cast<size_t>(c) * 256 + k]);
                // W2 tile: row = trunk channel, K = the 64 operating channels of this chunk
                for (int n = 0; n < 256; ++n)
                    *reinterpret_cast<__half*>(img2 + sw128_offset(n, cc)) = __float2half_rn(h.w2[static_cast<size_t>(n) * h.c_op + c]);
                aux_f[cc] = h.b1[c];
                aux_f[64 + cc] = h.bd[c];
                for (int q = 0; q < kk; ++q) aux_w[q * 64 + cc] = __float2half_rn(h.wd[static_cast<size_t>(c) * kk + q]);
            }
        }
    }
    if (upload(T->mem, w1, &T->args.w1_img) || upload(T->mem, w2, &T->args.w2_img)) return -1;
    if (T->mem.dalloc(&T->d_prof, 32)) return -1;
    T->args.prof = T->d_prof;
    const auto k1 = T->mx ? rise_trunk_kernel<1, true> : rise_trunk_kernel<1, false>;
    const auto k2 = T->mx ? rise_trunk_kernel<2, true> : rise_trunk_kernel<2, false>;
    const auto kp = T->mx ? rise_trunk_pair_kernel<true> : rise_trunk_pair_kernel<false>;
    ARA_CUDA_OK(cudaFuncSetAttribute(k1, cudaFuncAttributeMaxDynamicSharedMemorySize, RtCfg<1>::kSmemBytes));
    ARA_CUDA_OK(cudaFuncSetAttribute(k2, cudaFuncAttributeMaxDynamicSharedMemorySize, RtCfg<2>::kSmemBytes));
    ARA_CUDA_OK(cudaFuncSetAttribute(kp, cudaFuncAttributeMaxDynamicSharedMemorySize, RtPairCfg::kSmemBytes));
    {
        int dev = 0;
        cudaDeviceProp prop;
        ARA_CUDA_OK(cudaGetDevice(&dev));
        ARA_CUDA_OK(cudaGetDeviceProperties(&prop, dev));
        T->sm_count = prop.multiProcessorCount;
        // how many CTA pairs can be resident at once (a cluster lives inside one GPC, so this can be below sm_count / 2)
        cudaLaunchConfig_t cfg = {};
        cfg.gridDim = dim3(2 * (T->sm_count / 2));
        cfg.blockDim = dim3(RtPairCfg::kThreads);
        cfg.dynamicSmemBytes = RtPairCfg::kSmemBytes;
        cudaLaunchAttribute attr[1];
        attr[0].id = cudaLaunchAttributeClusterDimension;
        attr[0].val.clusterDim.x = 2;
        attr[0].val.clusterDim.y = 1;
        attr[0].val.clusterDim.z = 1;
        cfg.attrs = attr;
        cfg.numAttrs = 1;
        ARA_CUDA_OK(cudaOccupancyMaxActiveClusters(&T->pair_clusters, kp, &cfg));
    }
    return 0;
}

// one board per CTA pair while every pair is resident at once, else one board per CTA while that fits one wave, else
// two boards per CTA sharing a weight stream.  ARA_TRUNK_ROWS (trunk rows per CTA) forces a shape: 32 = the pair
// (half of a board's channels per CTA), 64 = one board per CTA, any other value = two boards per CTA.
static int trunk_rows(const RiseTrunk* T, int boards) {
    const char* force = getenv("ARA_TRUNK_ROWS");
    return force ? atoi(force) : boards <= T->pair_clusters ? 32 : boards <= T->sm_count ? 64 : 128;
}

int rise_trunk_ctas(const RiseTrunk* T, int boards) {
    const int rows = trunk_rows(T, boards);
    return rows == 32 ? 2 * boards : rows == 64 ? boards : (boards + 1) / 2;
}

int rise_trunk_launch(const RiseTrunk* T, int boards, cudaStream_t stream, const int* boards_dev, const __half* x_in) {
    TrunkArgs a = T->args;
    if (x_in != nullptr) a.x_in = x_in;
    a.M = boards * 64;
    a.boards_dev = boards_dev;
    const int rows = trunk_rows(T, boards);
    if (rows == 32)
        ARA_CUDA_OK(launch_pdl_cluster(T->mx ? rise_trunk_pair_kernel<true> : rise_trunk_pair_kernel<false>, dim3(2 * boards),
                                       dim3(RtPairCfg::kThreads), RtPairCfg::kSmemBytes, stream, 2u, a));
    else if (rows == 64)
        ARA_CUDA_OK(launch_pdl(T->mx ? rise_trunk_kernel<1, true> : rise_trunk_kernel<1, false>, dim3(boards), dim3(RtCfg<1>::kThreads),
                               RtCfg<1>::kSmemBytes, stream, a));
    else
        ARA_CUDA_OK(launch_pdl(T->mx ? rise_trunk_kernel<2, true> : rise_trunk_kernel<2, false>, dim3((boards + 1) / 2),
                               dim3(RtCfg<2>::kThreads), RtCfg<2>::kSmemBytes, stream, a));
    return 0;
}

namespace {

// the squeeze-excitation arguments of ara_debug_trunk_se; all null: no block has one
struct DebugSe {
    const int *se_type = nullptr, *gate = nullptr, *flags = nullptr, *se_bias = nullptr;
    const float *se_w1t = nullptr, *se_w2t = nullptr, *se_b = nullptr, *se_b1 = nullptr;
};

int debug_trunk_run(const __half* x_h, int n, int n_blocks, const int* c_op, const int* ksize, const float* w1, const float* b1,
                    const float* wd, const float* bd, const float* w2, const float* b2, const DebugSe& se, __half* out_h, int* mx) {
    if (n < 1 || n_blocks < 1 || n_blocks > kTrunkMaxBlocks) return set_error("ara_debug_trunk: %d boards, %d blocks", n, n_blocks);
    const size_t x_count = static_cast<size_t>(n) * 64 * 256;
    std::vector<TrunkBlockHost> blocks(n_blocks);
    const float *se_w1t = se.se_w1t, *se_w2t = se.se_w2t, *se_b = se.se_b, *se_b1 = se.se_b1;
    for (int i = 0; i < n_blocks; ++i) {
        TrunkBlockHost& h = blocks[i];
        const int c = c_op[i], kk = ksize[i] * ksize[i];
        if (c < 1) return set_error("ara_debug_trunk: block %d has no operating channels", i);
        h.c_op = c;
        h.ksize = ksize[i];
        h.w1.assign(w1, w1 + static_cast<size_t>(c) * 256);
        h.b1.assign(b1, b1 + c);
        h.wd.assign(wd, wd + static_cast<size_t>(c) * kk);
        h.bd.assign(bd, bd + c);
        h.w2.assign(w2, w2 + static_cast<size_t>(256) * c);
        h.b2.assign(b2 + 256 * i, b2 + 256 * (i + 1));
        w1 += static_cast<size_t>(c) * 256, b1 += c, wd += static_cast<size_t>(c) * kk, bd += c, w2 += static_cast<size_t>(256) * c;
        if (se.se_type == nullptr) continue;
        // only what a weight blob can describe (net.cu): the kernels take a ca_se block's two biases together or not at all
        const int type = se.se_type[i], bias = se.se_bias[i];
        if (type < 0 || type > 2) return set_error("ara_debug_trunk_se: block %d has squeeze-excitation type %d", i, type);
        if (se.gate[i] < kTrunkGateHard6 || se.gate[i] > kTrunkGateSigmoid) return set_error("ara_debug_trunk_se: block %d has gate %d", i, se.gate[i]);
        if ((se.flags[i] & ~kTrunkShortcutPreSe) != 0) return set_error("ara_debug_trunk_se: block %d has flags %d", i, se.flags[i]);
        const bool bias_ok = type == 0 ? bias == 0 : type == 2 ? bias == 1 : bias == 0 || bias == 3;
        if (!bias_ok)
            return set_error("ara_debug_trunk_se: block %d (squeeze-excitation type %d) has biases %d: eca_se takes se_b, ca_se "
                             "both se_b and se_b1 or neither, a block without squeeze-excitation none", i, type, bias);
        h.se_type = type;
        h.gate = se.gate[i];
        h.flags = se.flags[i];
        if (type == 0) continue;
        if (se_w1t == nullptr || (type == 1 && se_w2t == nullptr) || ((bias & 1) && se_b == nullptr) || ((bias & 2) && se_b1 == nullptr))
            return set_error("ara_debug_trunk_se: block %d: a squeeze-excitation array is null", i);
        const size_t n1 = type == 1 ? 256 * 128 : 256 * 256, n2 = type == 1 ? 128 * 256 : 0;
        h.se_w1t.assign(se_w1t, se_w1t + n1);
        h.se_w2t.assign(se_w2t, se_w2t + n2);
        se_w1t += n1, se_w2t += n2;
        if (bias & 1) h.se_b.assign(se_b, se_b + 256), se_b += 256;
        if (bias & 2) h.se_b1.assign(se_b1, se_b1 + 128), se_b1 += 128;
    }
    DeviceBuffers mem;
    __half *d_x = nullptr, *d_out = nullptr;
    if (mem.dalloc(&d_x, x_count) || mem.dalloc(&d_out, x_count)) return -1;
    ARA_CUDA_OK(cudaMemcpy(d_x, x_h, x_count * sizeof(__half), cudaMemcpyHostToDevice));
    RiseTrunk T;
    if (rise_trunk_init(&T, blocks, d_x, d_out)) return -1;
    if (mx != nullptr) *mx = T.mx ? 1 : 0;
    if (rise_trunk_launch(&T, n, nullptr)) return -1;
    ARA_CUDA_OK(cudaStreamSynchronize(nullptr));
    ARA_CUDA_OK(cudaMemcpy(out_h, d_out, x_count * sizeof(__half), cudaMemcpyDeviceToHost));
    return 0;
}

}  // namespace

}  // namespace ara

// Debug / unit-test entry: the tower kernel alone, on the shape ARA_TRUNK_ROWS selects (else the one the batch
// selects).  Host buffers: x_half and out_half [n][64 squares][256] fp16; the folded weights of the blocks (no
// squeeze-excitation) one block after the other in the layouts of TrunkBlockHost; b2 [n_blocks][256].
extern "C" int ara_debug_trunk(const void* x_half, int n, int n_blocks, const int* c_op, const int* ksize, const float* w1,
                               const float* b1, const float* wd, const float* bd, const float* w2, const float* b2, void* out_half) {
    return ara::debug_trunk_run(static_cast<const __half*>(x_half), n, n_blocks, c_op, ksize, w1, b1, wd, bd, w2, b2, {},
                                static_cast<__half*>(out_half), nullptr);
}

// ara_debug_trunk with the squeeze-excitation and MXNet block fields of TrunkBlockHost: per block se_type, gate, flags
// and se_bias (bit 0: se_b given, bit 1: se_b1 given); se_w1t, se_w2t, se_b and se_b1 concatenated over the blocks
// that have them.  *mx_out (if not null): 1 when rise_trunk_init chose the kernels built for the MXNet semantics.
extern "C" int ara_debug_trunk_se(const void* x_half, int n, int n_blocks, const int* c_op, const int* ksize, const int* se_type,
                                  const int* gate, const int* flags, const int* se_bias, const float* w1, const float* b1,
                                  const float* wd, const float* bd, const float* w2, const float* b2, const float* se_w1t,
                                  const float* se_w2t, const float* se_b, const float* se_b1, void* out_half, int* mx_out) {
    if (se_type == nullptr || gate == nullptr || flags == nullptr || se_bias == nullptr)
        return ara::set_error("ara_debug_trunk_se: null per-block argument");
    ara::DebugSe se;
    se.se_type = se_type, se.gate = gate, se.flags = flags, se.se_bias = se_bias;
    se.se_w1t = se_w1t, se.se_w2t = se_w2t, se.se_b = se_b, se.se_b1 = se_b1;
    return ara::debug_trunk_run(static_cast<const __half*>(x_half), n, n_blocks, c_op, ksize, w1, b1, wd, bd, w2, b2, se,
                                static_cast<__half*>(out_half), mx_out);
}
