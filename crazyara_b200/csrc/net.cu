// RISE network: blob loader, weight re-layout for the wgmma GEMMs, forward launch sequence, C-ABI.
#include "net.h"

#include <cstdio>
#include <cstring>
#include <memory>

#include "ara_b200.h"
#include "net_kernels.cuh"

namespace ara {

namespace {

struct BlobReader {
    FILE* f = nullptr;
    ~BlobReader() {
        if (f) fclose(f);
    }
    bool read(void* dst, size_t bytes) { return fread(dst, 1, bytes, f) == bytes; }
    bool tensor(std::vector<float>& out, size_t expect) {
        long long count = 0;
        if (!read(&count, 8)) return false;
        if (static_cast<size_t>(count) != expect) {
            set_error("weight blob: tensor has %lld values, expected %zu", count, expect);
            return false;
        }
        out.resize(expect);
        return read(out.data(), expect * 4);
    }
};

inline int round_up(int v, int m) { return (v + m - 1) / m * m; }

}  // namespace

int Net::upload_f32(const float* src, size_t count, size_t padded, float** dst) {
    if (mem_.dalloc(dst, padded) != 0) return -1;
    ARA_CUDA_OK(cudaMemcpy(*dst, src, count * 4, cudaMemcpyHostToDevice));
    return 0;
}

// w: [n_out, cin, k, k] fp32 -> fp16 [rows, taps * cw], column = tap * cw + c, rows padded to 256.
int Net::upload_conv_w(const float* w, int n_out, int cin, int ksize, __half** dst, int* rows) {
    const int taps = ksize * ksize;
    const int cw = round_up(cin, 64);
    const int r = round_up(n_out, 256);
    std::vector<__half> h(static_cast<size_t>(r) * taps * cw, __float2half(0.0f));
    for (int n = 0; n < n_out; ++n)
        for (int c = 0; c < cin; ++c)
            for (int t = 0; t < taps; ++t)
                h[(static_cast<size_t>(n) * taps + t) * cw + c] = __float2half_rn(w[(static_cast<size_t>(n) * cin + c) * taps + t]);
    if (mem_.dalloc(dst, h.size()) != 0) return -1;
    ARA_CUDA_OK(cudaMemcpy(*dst, h.data(), h.size() * sizeof(__half), cudaMemcpyHostToDevice));
    *rows = r;
    return 0;
}

// Precision float32: w [n_out, cin, k, k] fp32 -> fp16 [rows, taps * 3 * cw]; per tap the columns are
// hi(w) [cw] | lo(w) [cw] | hi(w) [cw], matching activations stored as hi | hi | lo (conv_gemm.cuh).
int Net::upload_conv_w_split(const float* w, int n_out, int cin, int ksize, __half** dst, int* rows) {
    const int taps = ksize * ksize;
    const int cw = round_up(cin, 64);
    const int r = round_up(n_out, 256);
    std::vector<__half> h(static_cast<size_t>(r) * taps * 3 * cw, __float2half(0.0f));
    for (int n = 0; n < n_out; ++n)
        for (int c = 0; c < cin; ++c)
            for (int t = 0; t < taps; ++t) {
                const float v = w[(static_cast<size_t>(n) * cin + c) * taps + t];
                const __half hi = __float2half_rn(v);
                const __half lo = __float2half_rn(v - __half2float(hi));
                __half* col = &h[(static_cast<size_t>(n) * taps + t) * 3 * cw];
                col[c] = hi;
                col[cw + c] = lo;
                col[2 * cw + c] = hi;
            }
    if (mem_.dalloc(dst, h.size()) != 0) return -1;
    ARA_CUDA_OK(cudaMemcpy(*dst, h.data(), h.size() * sizeof(__half), cudaMemcpyHostToDevice));
    *rows = r;
    return 0;
}

Net::~Net() {
    cudaSetDevice(device);
    for (auto& family : graphs_)
        for (auto& g : family) cudaGraphExecDestroy(g.second);
    if (stream) cudaStreamDestroy(stream);
    if (head_stream) cudaStreamDestroy(head_stream);
    if (ev_fork) cudaEventDestroy(ev_fork);
    if (ev_join) cudaEventDestroy(ev_join);
}

int Net::read_blob(const char* blob_path, HostWeights* hw) {
    BlobReader rd;
    rd.f = fopen(blob_path, "rb");
    if (!rd.f) return set_error("ara_net_create: cannot open weight blob '%s'", blob_path);
    // ARAB2001: the networks of the reference's PyTorch definition.  ARAB2002 (the MXNet symbols) adds the header flags
    // stem_act and policy_bias, and per block flags and the squeeze-excitation gate.
    char magic[8];
    if (!rd.read(magic, 8) || (memcmp(magic, "ARAB2001", 8) != 0 && memcmp(magic, "ARAB2002", 8) != 0))
        return set_error("ara_net_create: '%s' is not an ARAB2001 / ARAB2002 weight blob", blob_path);
    const bool v2 = magic[7] == '2';
    int h[10] = {0, 0, 0, 0, 0, 0, 0, 0, 1, 0};
    if (!rd.read(h, (v2 ? 10 : 8) * sizeof(int))) return set_error("ara_net_create: truncated header");
    hdr.in_channels = h[0];
    hdr.policy_channels = h[1];
    hdr.n_blocks = h[2];
    hdr.channels = h[3];
    hdr.value_channels = h[4];
    hdr.value_fc = h[5];
    hdr.wdl_mode = h[6];
    hdr.input_version = h[7];
    hdr.stem_act = h[8];
    hdr.policy_bias = h[9];
    if ((hdr.stem_act != 0 && hdr.stem_act != 1) || (hdr.policy_bias != 0 && hdr.policy_bias != 1))
        return set_error("ara_net_create: header flags stem_act %d policy_bias %d", hdr.stem_act, hdr.policy_bias);
    if (hdr.channels != 256 || hdr.value_channels != 8 || hdr.value_fc != 256)
        return set_error("ara_net_create: unsupported trunk geometry (channels %d, value %d/%d)", hdr.channels,
                         hdr.value_channels, hdr.value_fc);
    if (hdr.n_blocks < 1 || hdr.n_blocks > 64 || hdr.in_channels < 1 || hdr.in_channels > 256 ||
        hdr.policy_channels < 1 || hdr.policy_channels > 256)
        return set_error("ara_net_create: implausible header");
    blocks.resize(hdr.n_blocks);
    max_cop_ = 0;
    for (auto& b : blocks) {
        int t[5] = {0, 0, 0, 0, kTrunkGateHard6};
        if (!rd.read(t, (v2 ? 5 : 3) * sizeof(int))) return set_error("ara_net_create: truncated block table");
        b.c_op = t[0];
        b.kernel = t[1];
        b.se_type = t[2];
        b.flags = t[3];
        b.gate = t[4];
        if (b.c_op % 32 != 0 || b.c_op < 32 || (b.kernel != 3 && b.kernel != 5) || b.se_type < 0 || b.se_type > 2)
            return set_error("ara_net_create: unsupported block (c_op %d kernel %d se %d)", b.c_op, b.kernel, b.se_type);
        if ((b.flags & ~(kBlobShortcutPreSe | kBlobSeBias)) != 0 || b.gate < kTrunkGateHard6 || b.gate > kTrunkGateSigmoid ||
            ((b.flags & kBlobSeBias) && b.se_type != 1))
            return set_error("ara_net_create: unsupported block flags %d gate %d (se %d)", b.flags, b.gate, b.se_type);
        if (b.c_op > max_cop_) max_cop_ = b.c_op;
    }
    const size_t C = hdr.channels;
    if (!rd.tensor(hw->stem_w, C * hdr.in_channels * 9) || !rd.tensor(hw->stem_b, C)) return -1;
    hw->blocks.resize(hdr.n_blocks);
    for (int i = 0; i < hdr.n_blocks; ++i) {
        const BlockDesc& bd = blocks[i];
        HostBlock& hb = hw->blocks[i];
        const size_t cop = bd.c_op, kk = static_cast<size_t>(bd.kernel) * bd.kernel;
        const bool se_bias = (bd.flags & kBlobSeBias) != 0;
        if (bd.se_type == 1 && (!rd.tensor(hb.se_a, 128 * 256) || (se_bias && !rd.tensor(hb.se_b1, 128)) ||
                                !rd.tensor(hb.se_b, 256 * 128) || (se_bias && !rd.tensor(hb.se_b2, 256))))
            return -1;
        if (bd.se_type == 2 && (!rd.tensor(hb.se_a, 256 * 256) || !rd.tensor(hb.se_b, 256))) return -1;
        if (!rd.tensor(hb.w1, cop * C) || !rd.tensor(hb.b1, cop) || !rd.tensor(hb.wd, cop * kk) || !rd.tensor(hb.bd, cop) ||
            !rd.tensor(hb.w2, C * cop) || !rd.tensor(hb.b2, C))
            return -1;
    }
    if (!rd.tensor(hw->vh_wv, 8 * 256) || !rd.tensor(hw->vh_bv, 8)) return -1;
    if (!hdr.wdl_mode) {
        if (!rd.tensor(hw->vh_a, 256 * 512) || !rd.tensor(hw->vh_ab, 256) || !rd.tensor(hw->vh_b, 256) || !rd.tensor(hw->vh_bb, 1))
            return -1;
    } else {
        if (!rd.tensor(hw->vh_a, 3 * 512) || !rd.tensor(hw->vh_ab, 3) || !rd.tensor(hw->vh_b, 512) || !rd.tensor(hw->vh_bb, 1))
            return -1;
    }
    if (!rd.tensor(hw->pol_w1, C * C * 9) || !rd.tensor(hw->pol_b1, C) ||
        !rd.tensor(hw->pol_w2, static_cast<size_t>(hdr.policy_channels) * C * 9) ||
        (hdr.policy_bias && !rd.tensor(hw->pol_b2, hdr.policy_channels)))
        return -1;
    char tail;
    if (fread(&tail, 1, 1, rd.f) != 0) return set_error("ara_net_create: trailing bytes in weight blob");
    return 0;
}

// squeeze-excitation matrices, transposed for coalesced reads: ca_se fc1 [128][256] -> [256][128], fc2 [256][128] ->
// [128][256]; eca_se centre tap [out][in] -> [in][out] + bias
static void se_transposed(const BlockDesc& bd, const HostBlock& hb, std::vector<float>* a, std::vector<float>* b) {
    if (bd.se_type == 1) {
        a->assign(256 * 128, 0.f);
        for (int j = 0; j < 128; ++j)
            for (int k = 0; k < 256; ++k) (*a)[k * 128 + j] = hb.se_a[j * 256 + k];
        b->assign(128 * 256, 0.f);
        for (int c = 0; c < 256; ++c)
            for (int j = 0; j < 128; ++j) (*b)[j * 256 + c] = hb.se_b[c * 128 + j];
    } else if (bd.se_type == 2) {
        a->assign(256 * 256, 0.f);
        for (int c = 0; c < 256; ++c)
            for (int k = 0; k < 256; ++k) (*a)[k * 256 + c] = hb.se_a[c * 256 + k];
        *b = hb.se_b;
    }
}

// the bias of the last policy convolution (ARAB2002 policy_bias), zero padded to the weight rows; else none
int Net::upload_policy_bias(const HostWeights& hw, int rows) {
    if (!hdr.policy_bias) return 0;
    return upload_f32(hw.pol_b2.data(), hw.pol_b2.size(), rows, &pol_b2);
}

int Net::upload_value_head(const HostWeights& hw) {
    if (upload_f32(hw.vh_wv.data(), hw.vh_wv.size(), hw.vh_wv.size(), &vh_wv)) return -1;
    if (upload_f32(hw.vh_bv.data(), 8, 8, &vh_bv)) return -1;
    if (!hdr.wdl_mode) {
        std::vector<float> t2(512 * 256, 0.f);  // fc1 [256][512] -> [512][256]
        for (int o = 0; o < 256; ++o)
            for (int i = 0; i < 512; ++i) t2[i * 256 + o] = hw.vh_a[o * 512 + i];
        if (upload_f32(t2.data(), t2.size(), t2.size(), &vh_w1t)) return -1;
        if (upload_f32(hw.vh_ab.data(), 256, 256, &vh_b1)) return -1;
        if (upload_f32(hw.vh_b.data(), 256, 256, &vh_w2)) return -1;
        if (upload_f32(hw.vh_bb.data(), 1, 1, &vh_b2)) return -1;
    } else {
        if (upload_f32(hw.vh_a.data(), hw.vh_a.size(), hw.vh_a.size(), &vh_wdl_w)) return -1;
        if (upload_f32(hw.vh_ab.data(), 3, 4, &vh_wdl_b)) return -1;
        if (upload_f32(hw.vh_b.data(), 512, 512, &vh_plys_w)) return -1;
        if (upload_f32(hw.vh_bb.data(), 1, 1, &vh_plys_b)) return -1;
    }
    return 0;
}

// Precision float16: stem (wgmma implicit GEMM) -> persistent tower kernel -> heads
int Net::build_half(const HostWeights& hw) {
    const int C = hdr.channels;
    const size_t rows = static_cast<size_t>(batch_cap) * 64;
    if (hdr.n_blocks > kTrunkMaxBlocks) return set_error("ara_net_create: %d blocks (max %d)", hdr.n_blocks, kTrunkMaxBlocks);
    if (mem_.dalloc(&d_in_h, rows * cin_pad)) return -1;
    if (mem_.dalloc(&d_x[0], rows * C) || mem_.dalloc(&d_x[1], rows * C) || mem_.dalloc(&d_p1, rows * C)) return -1;
    int wrows = 0;
    if (upload_conv_w(hw.stem_w.data(), C, hdr.in_channels, 3, &stem_w, &wrows)) return -1;
    if (upload_f32(hw.stem_b.data(), C, 256, &stem_b)) return -1;
    if (conv_layer_init(&stem_conv, d_in_h, batch_cap, cin_pad, stem_w, wrows, C, 3, stem_b, hdr.stem_act, nullptr, 0, d_x[0], nullptr, C,
                        conv_layer_choose_bn(batch, C)))
        return -1;
    std::vector<TrunkBlockHost> tb(hdr.n_blocks);
    for (int i = 0; i < hdr.n_blocks; ++i) {
        const BlockDesc& bd = blocks[i];
        const HostBlock& hb = hw.blocks[i];
        tb[i].c_op = bd.c_op;
        tb[i].ksize = bd.kernel;
        tb[i].se_type = bd.se_type;
        tb[i].w1 = hb.w1;
        tb[i].b1 = hb.b1;
        tb[i].wd = hb.wd;
        tb[i].bd = hb.bd;
        tb[i].w2 = hb.w2;
        tb[i].b2 = hb.b2;
        se_transposed(bd, hb, &tb[i].se_w1t, bd.se_type == 1 ? &tb[i].se_w2t : &tb[i].se_b);
        tb[i].flags = bd.flags & kBlobShortcutPreSe ? kTrunkShortcutPreSe : 0;
        tb[i].gate = bd.gate;
        if (bd.se_type == 1) tb[i].se_b1 = hb.se_b1, tb[i].se_b = hb.se_b2;
    }
    __half* xfinal = d_x[1];
    if (rise_trunk_init(&trunk_, tb, d_x[0], xfinal)) return -1;
    if (upload_conv_w(hw.pol_w1.data(), C, C, 3, &pol_w1, &wrows)) return -1;
    if (upload_f32(hw.pol_b1.data(), C, 256, &pol_b1)) return -1;
    if (conv_layer_init(&pol_conv1, xfinal, batch_cap, C, pol_w1, wrows, C, 3, pol_b1, 1, nullptr, 0, d_p1, nullptr, C,
                        conv_layer_choose_bn(batch, C)))
        return -1;
    if (upload_conv_w(hw.pol_w2.data(), hdr.policy_channels, C, 3, &pol_w2, &wrows)) return -1;
    if (upload_policy_bias(hw, wrows)) return -1;
    if (conv_layer_init(&pol_conv2, d_p1, batch_cap, C, pol_w2, wrows, hdr.policy_channels, 3, pol_b2, 0, nullptr, 0, nullptr,
                        d_logits, ldp, conv_layer_choose_bn(batch, hdr.policy_channels)))
        return -1;
    return 0;
}

// Precision float32: every layer a launch; GEMMs on wgmma with fp16 hi + lo operand splitting (3x the K extent),
// fp32 activations in HBM between the layers, CUDA-core stages in fp32
int Net::build_precise(const HostWeights& hw) {
    const int C = hdr.channels;
    const size_t rows = static_cast<size_t>(batch_cap) * 64;
    const int max_cp = round_up(max_cop_, 64);
    if (mem_.dalloc(&d_in_h, rows * 3 * cin_pad)) return -1;
    for (int k = 0; k < 2; ++k)
        if (mem_.dalloc(&d_xf[k], rows * C) || mem_.dalloc(&d_xs[k], rows * 3 * C)) return -1;
    if (mem_.dalloc(&d_h1f, rows * max_cop_) || mem_.dalloc(&d_h2s, rows * 3 * max_cp) || mem_.dalloc(&d_p1, rows * 3 * C)) return -1;
    int wrows = 0;
    if (upload_conv_w_split(hw.stem_w.data(), C, hdr.in_channels, 3, &stem_w, &wrows)) return -1;
    if (upload_f32(hw.stem_b.data(), C, 256, &stem_b)) return -1;
    if (conv_layer_init(&stem_conv, d_in_h, batch_cap, 3 * cin_pad, stem_w, wrows, C, 3, stem_b, hdr.stem_act, nullptr, 0, nullptr, d_xf[0], C,
                        conv_layer_choose_bn(batch, C)))
        return -1;
    conv_layer_set_precise(&stem_conv, nullptr, 0, d_xs[0], C);
    pb_.resize(hdr.n_blocks);
    std::vector<float> ta, tbv, t2;
    for (int i = 0; i < hdr.n_blocks; ++i) {
        const BlockDesc& bd = blocks[i];
        const HostBlock& hb = hw.blocks[i];
        PreciseBlock& w = pb_[i];
        const int cp = round_up(bd.c_op, 64);
        const int in = i & 1, out = (i + 1) & 1;
        if (bd.se_type != 0) {
            se_transposed(bd, hb, &ta, &tbv);
            if (upload_f32(ta.data(), ta.size(), ta.size(), &w.se_w1t)) return -1;
            if (upload_f32(tbv.data(), tbv.size(), tbv.size(), bd.se_type == 1 ? &w.se_w2t : &w.se_b)) return -1;
            if (!hb.se_b1.empty() && (upload_f32(hb.se_b1.data(), 128, 128, &w.se_b1) || upload_f32(hb.se_b2.data(), 256, 256, &w.se_b)))
                return -1;
        }
        // conv1 1x1 256 -> c_op, ReLU: split X -> fp32 H1
        if (upload_conv_w_split(hb.w1.data(), bd.c_op, C, 1, &w.w1, &wrows)) return -1;
        if (upload_f32(hb.b1.data(), bd.c_op, round_up(bd.c_op, 256), &w.b1)) return -1;
        if (conv_layer_init(&w.conv1, d_xs[in], batch_cap, 3 * C, w.w1, wrows, bd.c_op, 1, w.b1, 1, nullptr, 0, nullptr, d_h1f,
                            bd.c_op, conv_layer_choose_bn(batch, bd.c_op)))
            return -1;
        // depthwise k x k: blob [c_op][k][k] -> device [k*k][c_op]
        const int kk = bd.kernel * bd.kernel;
        t2.assign(static_cast<size_t>(kk) * bd.c_op, 0.f);
        for (int c = 0; c < bd.c_op; ++c)
            for (int q = 0; q < kk; ++q) t2[static_cast<size_t>(q) * bd.c_op + c] = hb.wd[static_cast<size_t>(c) * kk + q];
        if (upload_f32(t2.data(), t2.size(), t2.size(), &w.wd)) return -1;
        if (upload_f32(hb.bd.data(), bd.c_op, cp, &w.bd)) return -1;
        // conv2 1x1 c_op -> 256 + fp32 residual: split H2 [.., 3*cp] -> fp32 X' and split X'
        if (upload_conv_w_split(hb.w2.data(), C, bd.c_op, 1, &w.w2, &wrows)) return -1;
        if (upload_f32(hb.b2.data(), C, 256, &w.b2)) return -1;
        if (conv_layer_init(&w.conv2, d_h2s, batch_cap, 3 * cp, w.w2, wrows, C, 1, w.b2, 0, nullptr, 0, nullptr, d_xf[out], C,
                            conv_layer_choose_bn(batch, C)))
            return -1;
        conv_layer_set_precise(&w.conv2, d_xf[in], C, d_xs[out], C);
    }
    const int fin = hdr.n_blocks & 1;
    if (upload_conv_w_split(hw.pol_w1.data(), C, C, 3, &pol_w1, &wrows)) return -1;
    if (upload_f32(hw.pol_b1.data(), C, 256, &pol_b1)) return -1;
    if (conv_layer_init(&pol_conv1, d_xs[fin], batch_cap, 3 * C, pol_w1, wrows, C, 3, pol_b1, 1, nullptr, 0, nullptr, nullptr, C,
                        conv_layer_choose_bn(batch, C)))
        return -1;
    conv_layer_set_precise(&pol_conv1, nullptr, 0, d_p1, C);
    if (upload_conv_w_split(hw.pol_w2.data(), hdr.policy_channels, C, 3, &pol_w2, &wrows)) return -1;
    if (upload_policy_bias(hw, wrows)) return -1;
    if (conv_layer_init(&pol_conv2, d_p1, batch_cap, 3 * C, pol_w2, wrows, hdr.policy_channels, 3, pol_b2, 0, nullptr, 0, nullptr,
                        d_logits, ldp, conv_layer_choose_bn(batch, hdr.policy_channels)))
        return -1;
    ARA_CUDA_OK(cudaFuncSetAttribute(value_head_kernel<float>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                     value_head_smem<float>()));
    ARA_CUDA_OK(cudaFuncSetAttribute(nchw_f32_to_nhwc_split_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                     hdr.in_channels * 65 * 4));
    return 0;
}

int Net::init(const char* blob_path, int dev, int batch_size, int prec) {
    device = dev;
    batch = batch_size;
    precision = prec;
    if (batch < 1) return set_error("ara_net_create: batch %d < 1", batch);
    if (precision != 0 && precision != 1)
        return set_error("ara_net_create: precision %d (0 = float16, 1 = float32)", precision);
    batch_cap = round_up(batch < 2 ? 2 : batch, 2);
    ARA_CUDA_OK(cudaSetDevice(device));
    {
        cudaDeviceProp prop;
        ARA_CUDA_OK(cudaGetDeviceProperties(&prop, device));
        if (prop.major != 9 || prop.minor != 0)
            return set_error("ara_net_create: device %d is sm_%d%d; this library only runs on sm_90a (H100)", device,
                             prop.major, prop.minor);
    }
    ARA_CUDA_OK(cudaStreamCreateWithFlags(&stream, cudaStreamNonBlocking));
    ARA_CUDA_OK(cudaStreamCreateWithFlags(&head_stream, cudaStreamNonBlocking));
    ARA_CUDA_OK(cudaEventCreateWithFlags(&ev_fork, cudaEventDisableTiming));
    ARA_CUDA_OK(cudaEventCreateWithFlags(&ev_join, cudaEventDisableTiming));

    HostWeights hw;
    if (read_blob(blob_path, &hw)) return -1;
    cin_pad = round_up(hdr.in_channels, 64);
    ldp = round_up(hdr.policy_channels, 32);
    const size_t rows = static_cast<size_t>(batch_cap) * 64;
    if (mem_.dalloc(&d_in_f32, static_cast<size_t>(batch) * hdr.in_channels * 64)) return -1;
    if (mem_.dalloc(&d_logits, rows * ldp)) return -1;
    if (mem_.dalloc(&d_prob, static_cast<size_t>(batch) * n_labels())) return -1;
    if (mem_.dalloc(&d_value, batch)) return -1;
    if (mem_.dalloc(&d_aux, static_cast<size_t>(batch) * 4)) return -1;
    if (upload_value_head(hw)) return -1;
    if (precision == 0 ? build_half(hw) : build_precise(hw)) return -1;
    io_in_h[0] = d_in_h, io_prob[0] = d_prob, io_value[0] = d_value, io_aux[0] = d_aux;
    ARA_CUDA_OK(cudaFuncSetAttribute(value_head_kernel<__half>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                     value_head_smem<__half>()));
    ARA_CUDA_OK(cudaFuncSetAttribute(policy_softmax_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                     n_labels() * 4));
    ARA_CUDA_OK(cudaFuncSetAttribute(nchw_f32_to_nhwc_f16_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                     hdr.in_channels * 65 * 4));
    ARA_CUDA_OK(cudaDeviceSynchronize());
    return 0;
}

int Net::enable_second_io() {
    if (io_in_h[1] != nullptr) return 0;
    ARA_CUDA_OK(cudaSetDevice(device));
    const size_t rows = static_cast<size_t>(batch_cap) * 64;
    const int cin = precision == 0 ? cin_pad : 3 * cin_pad;
    if (mem_.dalloc(&io_in_h[1], rows * cin)) return -1;
    if (mem_.dalloc(&io_prob[1], static_cast<size_t>(batch) * n_labels())) return -1;
    if (mem_.dalloc(&io_value[1], batch) || mem_.dalloc(&io_aux[1], static_cast<size_t>(batch) * 4)) return -1;
    stem_conv2 = stem_conv;  // same weights and epilogue; the activation map differs ...
    if (make_act_tensor_map(&stem_conv2.tm_a, io_in_h[1], batch_cap, cin)) return -1;
    if (precision == 0) {  // ... and the output buffer: the two sets' stems may then run while the other set's tower reads its own
        if (mem_.dalloc(&d_x0_alt, rows * static_cast<size_t>(hdr.channels))) return -1;
        stem_conv2.args.out_h = d_x0_alt;
    }
    return 0;
}

int Net::enqueue_precise(int n, cudaStream_t s, bool from_f32, const int* cnt, int io) {
    if (from_f32) {
        ARA_CUDA_OK(launch_pdl(nchw_f32_to_nhwc_split_kernel, dim3(n), dim3(256), hdr.in_channels * 65 * 4, s, d_in_f32, io_in_h[io],
                               hdr.in_channels, cin_pad));
        ++launches;
    }
    if (conv_layer_launch(io ? &stem_conv2 : &stem_conv, n, s, cnt)) return -1;
    ++launches;
    for (int i = 0; i < hdr.n_blocks; ++i) {
        const BlockDesc& bd = blocks[i];
        PreciseBlock& w = pb_[i];
        const int in = i & 1;
        if (bd.se_type != 0) {
            ARA_CUDA_OK(launch_pdl(se_f32_kernel, dim3(n), dim3(256), 0, s, d_xf[in], d_xs[in], w.se_w1t, w.se_w2t, w.se_b, w.se_b1,
                                   bd.se_type, bd.gate, (bd.flags & kBlobShortcutPreSe) ? 1 : 0));
            ++launches;
        }
        if (conv_layer_launch(&w.conv1, n, s)) return -1;
        const long long total = static_cast<long long>(n) * 64 * bd.c_op;
        const int grid = static_cast<int>((total + 255) / 256);
        const int cp = round_up(bd.c_op, 64);
        if (bd.kernel == 3)
            ARA_CUDA_OK(launch_pdl(dwconv_f32_kernel<3>, dim3(grid), dim3(256), 0, s, d_h1f, w.wd, w.bd, d_h2s, n, bd.c_op, cp));
        else
            ARA_CUDA_OK(launch_pdl(dwconv_f32_kernel<5>, dim3(grid), dim3(256), 0, s, d_h1f, w.wd, w.bd, d_h2s, n, bd.c_op, cp));
        if (conv_layer_launch(&w.conv2, n, s)) return -1;
        launches += 3;
    }
    const float* xfinal = d_xf[hdr.n_blocks & 1];
    ValueHeadW vw{vh_wv, vh_bv, vh_w1t, vh_b1, vh_w2, vh_b2, vh_wdl_w, vh_wdl_b, vh_plys_w, vh_plys_b, hdr.wdl_mode};
    ARA_CUDA_OK(launch_pdl(value_head_kernel<float>, dim3(n), dim3(256), value_head_smem<float>(), s, xfinal, vw, io_value[io], io_aux[io], cnt));
    if (conv_layer_launch(&pol_conv1, n, s, cnt)) return -1;
    if (conv_layer_launch(&pol_conv2, n, s, cnt)) return -1;
    ARA_CUDA_OK(launch_pdl(policy_softmax_kernel, dim3(n), dim3(256), n_labels() * 4, s, d_logits, io_prob[io], hdr.policy_channels, ldp, cnt));
    launches += 4;
    ARA_CUDA_OK(cudaGetLastError());
    return 0;
}

int Net::stem_device(int n, cudaStream_t s, const int* cnt, int io) {
    if (!stem_splittable() || io < 0 || io > 1) return set_error("stem_device: needs Precision float16 and two input / output sets");
    if (conv_layer_launch(io ? &stem_conv2 : &stem_conv, n, s, cnt)) return -1;
    return 0;  // (the caller counts the launch: it may sit in a captured graph)
}

int Net::enqueue(int n, cudaStream_t s, bool from_f32, const int* cnt, int io, bool stem_done) {
    if (precision == 1) return enqueue_precise(n, s, from_f32, cnt, io);
    if (from_f32) {
        ARA_CUDA_OK(launch_pdl(nchw_f32_to_nhwc_f16_kernel, dim3(n), dim3(256), hdr.in_channels * 65 * 4, s, d_in_f32, io_in_h[io], hdr.in_channels, cin_pad));
        ++launches;
    }
    if (!stem_done) {
        if (conv_layer_launch(io ? &stem_conv2 : &stem_conv, n, s, cnt)) return -1;
        ++launches;
    }
    {   // two input / output sets = a search with Threads = 2: the tower is the first kernel of this stream's chain and
        // must not sit on its SMs waiting for the tree stream's event (see PdlSuspend); the small kernels behind it keep
        // their programmatic launches (the tower triggers them at its last block)
        PdlSuspend no_pdl(io_in_h[1] != nullptr);
        if (rise_trunk_launch(&trunk_, n, s, cnt, (io == 1 && d_x0_alt != nullptr) ? d_x0_alt : nullptr)) return -1;
    }
    ++launches;
    __half* xfinal = d_x[1];
    ValueHeadW vw{vh_wv, vh_bv, vh_w1t, vh_b1, vh_w2, vh_b2, vh_wdl_w, vh_wdl_b, vh_plys_w, vh_plys_b, hdr.wdl_mode};
    // value head on the side stream (a second branch of the captured graph), policy head on s
    ARA_CUDA_OK(cudaEventRecord(ev_fork, s));
    ARA_CUDA_OK(cudaStreamWaitEvent(head_stream, ev_fork, 0));
    value_head_kernel<__half><<<dim3(n), dim3(256), value_head_smem<__half>(), head_stream>>>(xfinal, vw, io_value[io], io_aux[io], cnt);
    ARA_CUDA_OK(cudaEventRecord(ev_join, head_stream));
    if (conv_layer_launch(&pol_conv1, n, s, cnt)) return -1;
    if (conv_layer_launch(&pol_conv2, n, s, cnt)) return -1;
    ARA_CUDA_OK(launch_pdl(policy_softmax_kernel, dim3(n), dim3(256), n_labels() * 4, s, d_logits, io_prob[io], hdr.policy_channels, ldp, cnt));
    ARA_CUDA_OK(cudaStreamWaitEvent(s, ev_join, 0));
    launches += 4;
    ARA_CUDA_OK(cudaGetLastError());
    return 0;
}

int Net::forward_device(int n, cudaStream_t s, const int* cnt, int io, bool stem_done) {
    if (stem_done && !stem_splittable()) return set_error("forward: stem_done needs Precision float16 and two input / output sets");
    if (n < 1 || n > batch) return set_error("forward: n=%d outside [1,%d]", n, batch);
    if (io != 0 && (io != 1 || io_in_h[1] == nullptr)) return set_error("forward: input/output set %d not enabled", io);
    // two input / output sets = a search with Threads = 2: this forward runs on the network stream beside the other
    // thread's tree kernels (see PdlSuspend)
    PdlSuspend no_pdl(io_in_h[1] != nullptr && (precision != 0 || !stem_done));  // (not split: everything plain, as before)
    {   // inside somebody else's capture (the search's iteration graph) the kernels go in directly
        cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
        ARA_CUDA_OK(cudaStreamIsCapturing(s, &cs));
        if (cs == cudaStreamCaptureStatusActive) return enqueue(n, s, false, cnt, io, stem_done);
    }
    const int gk = stem_done ? 4 + io : (io == 1 ? 3 : (cnt != nullptr ? 2 : 0));
    const int*& baked = baked_[gk];
    if ((gk >= 3 || cnt != nullptr) && cnt != baked) {  // graphs captured with another counter are of no use
        for (auto& g : graphs_[gk]) cudaGraphExecDestroy(g.second);
        graphs_[gk].clear();
        baked = cnt;
    }
    return launch_graph(gk, n, s, false, cnt, io, stem_done);
}

int Net::forward_from_f32_device(int n, cudaStream_t s) {
    if (n < 1 || n > batch) return set_error("forward: n=%d outside [1,%d]", n, batch);
    return launch_graph(1, n, s, true, nullptr, 0, false);
}

// The forward as one launch of graph family `family`'s graph for n boards.  The first forward of a size runs eagerly as a
// warm-up and is then captured; the launches of the capture are not counted.
int Net::launch_graph(int family, int n, cudaStream_t s, bool from_f32, const int* cnt, int io, bool stem_done) {
    auto& graphs = graphs_[family];
    auto it = graphs.find(n);
    if (it == graphs.end()) {
        if (enqueue(n, s, from_f32, cnt, io, stem_done)) return -1;
        ARA_CUDA_OK(cudaStreamSynchronize(s));
        const long long before = launches;
        cudaGraphExec_t ge;
        const int rc = capture_graph(s, &ge, [&] { return enqueue(n, s, from_f32, cnt, io, stem_done); });
        launches = before;
        if (rc) return -1;
        it = graphs.emplace(n, ge).first;
    }
    ARA_CUDA_OK(cudaGraphLaunch(it->second, s));
    launches += kernels_per_forward(from_f32) - (stem_done ? 1 : 0);
    return 0;
}

int Net::trunk_cycles(unsigned long long* out32) {
    if (precision != 0 || trunk_.d_prof == nullptr) return set_error("trunk kernel not in use");
    ARA_CUDA_OK(cudaSetDevice(device));
    ARA_CUDA_OK(cudaStreamSynchronize(stream));
    ARA_CUDA_OK(cudaMemcpy(out32, trunk_.d_prof, 32 * sizeof(unsigned long long), cudaMemcpyDeviceToHost));
    return 0;
}

int Net::kernels_per_forward(bool from_f32) const {
    int k = from_f32 ? 1 : 0;
    k += 1;  // stem
    if (precision == 0)
        k += 1;  // the tower kernel
    else
        for (const auto& b : blocks) k += 3 + (b.se_type != 0 ? 1 : 0);
    k += 4;  // value head, policy conv x2, softmax
    return k;
}

int Net::predict(const float* planes_host, int n, float* value_host, float* prob_host, float* aux_host) {
    ARA_CUDA_OK(cudaSetDevice(device));
    if (n < 1 || n > batch) return set_error("ara_net_predict: n=%d outside [1,%d]", n, batch);
    if (planes_host == nullptr || value_host == nullptr) return set_error("ara_net_predict: null planes/value buffer");
    ARA_CUDA_OK(cudaMemcpyAsync(d_in_f32, planes_host, static_cast<size_t>(n) * hdr.in_channels * 64 * 4,
                                cudaMemcpyHostToDevice, stream));
    if (forward_from_f32_device(n, stream)) return -1;
    ARA_CUDA_OK(cudaMemcpyAsync(value_host, d_value, static_cast<size_t>(n) * 4, cudaMemcpyDeviceToHost, stream));
    if (prob_host != nullptr)
        ARA_CUDA_OK(cudaMemcpyAsync(prob_host, d_prob, static_cast<size_t>(n) * n_labels() * 4, cudaMemcpyDeviceToHost,
                                    stream));
    if (aux_host != nullptr && hdr.wdl_mode)
        ARA_CUDA_OK(cudaMemcpyAsync(aux_host, d_aux, static_cast<size_t>(n) * 4 * 4, cudaMemcpyDeviceToHost, stream));
    ARA_CUDA_OK(cudaStreamSynchronize(stream));
    return 0;
}

int Net::predict_priors(const float* planes_host, int n, const int* policy_idx, const int* counts, int stride, float* value_host,
                        float* priors_host, float* aux_host) {
    ARA_CUDA_OK(cudaSetDevice(device));
    if (n < 1 || n > batch) return set_error("ara_net_predict_priors: n=%d outside [1,%d]", n, batch);
    if (!planes_host || !value_host || !policy_idx || !counts || !priors_host || stride < 1 || stride > 512)
        return set_error("ara_net_predict_priors: bad arguments");
    if (stride > gather_stride) {
        if (mem_.dalloc(&d_gather_idx, static_cast<size_t>(batch) * stride) || mem_.dalloc(&d_gather_out, static_cast<size_t>(batch) * stride)) return -1;
        if (d_gather_cnt == nullptr && mem_.dalloc(&d_gather_cnt, batch)) return -1;
        gather_stride = stride;
    }
    ARA_CUDA_OK(cudaMemcpyAsync(d_in_f32, planes_host, static_cast<size_t>(n) * hdr.in_channels * 64 * 4, cudaMemcpyHostToDevice, stream));
    ARA_CUDA_OK(cudaMemcpyAsync(d_gather_idx, policy_idx, static_cast<size_t>(n) * stride * 4, cudaMemcpyHostToDevice, stream));
    ARA_CUDA_OK(cudaMemcpyAsync(d_gather_cnt, counts, static_cast<size_t>(n) * 4, cudaMemcpyHostToDevice, stream));
    if (forward_from_f32_device(n, stream)) return -1;
    gather_priors_kernel<<<n, 128, 0, stream>>>(d_prob, n_labels(), d_gather_idx, d_gather_cnt, stride, d_gather_out);
    ++launches;
    ARA_CUDA_OK(cudaMemcpyAsync(value_host, d_value, static_cast<size_t>(n) * 4, cudaMemcpyDeviceToHost, stream));
    ARA_CUDA_OK(cudaMemcpyAsync(priors_host, d_gather_out, static_cast<size_t>(n) * stride * 4, cudaMemcpyDeviceToHost, stream));
    if (aux_host != nullptr && hdr.wdl_mode)
        ARA_CUDA_OK(cudaMemcpyAsync(aux_host, d_aux, static_cast<size_t>(n) * 4 * 4, cudaMemcpyDeviceToHost, stream));
    ARA_CUDA_OK(cudaStreamSynchronize(stream));
    return 0;
}

}  // namespace ara

// ------------------------------------------------------------------------------------------- C-ABI
using ara::Net;

extern "C" ara_net_t ara_net_create(const char* weights_path, int device, int batch_size, int precision) {
    std::unique_ptr<Net> net(new Net());
    if (net->init(weights_path, device, batch_size, precision) != 0) return nullptr;
    return reinterpret_cast<ara_net_t>(net.release());
}

extern "C" void ara_net_destroy(ara_net_t h) { delete reinterpret_cast<Net*>(h); }

extern "C" int ara_net_shape(ara_net_t h, int* in_channels, int* n_labels, int* n_aux, int* is_policy_map,
                             int* input_version, int* batch_size) {
    if (h == nullptr) return ara::set_error("ara_net_shape: null handle");
    Net* net = reinterpret_cast<Net*>(h);
    if (in_channels) *in_channels = net->hdr.in_channels;
    if (n_labels) *n_labels = net->n_labels();
    if (n_aux) *n_aux = net->n_aux();
    if (is_policy_map) *is_policy_map = 1;  // the policy head is a convolution onto P x 8 x 8 planes (builder_util.py:206-243,
                                            // select_policy_from_plane): every blob this loader accepts is a policy map
    if (input_version) *input_version = net->hdr.input_version;
    if (batch_size) *batch_size = net->batch;
    return 0;
}

extern "C" int ara_net_predict(ara_net_t h, const float* planes, int n, float* value, float* prob, float* aux) {
    if (h == nullptr) return ara::set_error("ara_net_predict: null handle");
    return reinterpret_cast<Net*>(h)->predict(planes, n, value, prob, aux);
}

extern "C" int ara_net_predict_priors(ara_net_t h, const float* planes, int n, const int* policy_idx, const int* counts, int stride,
                                      float* value, float* priors_out, float* aux) {
    if (h == nullptr) return ara::set_error("ara_net_predict_priors: null handle");
    return reinterpret_cast<Net*>(h)->predict_priors(planes, n, policy_idx, counts, stride, value, priors_out, aux);
}

extern "C" void* ara_host_alloc(unsigned long long bytes) {
    void* p = nullptr;
    if (cudaMallocHost(&p, bytes) != cudaSuccess) {
        ara::set_error("ara_host_alloc: cudaMallocHost(%llu) failed", bytes);
        return nullptr;
    }
    return p;
}
extern "C" void ara_host_free(void* p) {
    if (p != nullptr) cudaFreeHost(p);
}

extern "C" int ara_net_forward_device(ara_net_t h, const float* planes_dev, int n, float** value_dev, float** prob_dev) {
    if (h == nullptr) return ara::set_error("ara_net_forward_device: null handle");
    Net* net = reinterpret_cast<Net*>(h);
    if (cudaSetDevice(net->device) != cudaSuccess) return ara::set_error("cudaSetDevice failed");
    if (planes_dev != nullptr) {
        cudaError_t e = cudaMemcpyAsync(net->d_in_f32, planes_dev, static_cast<size_t>(n) * net->hdr.in_channels * 64 * 4,
                                        cudaMemcpyDeviceToDevice, net->stream);
        if (e != cudaSuccess) return ara::set_error("ara_net_forward_device: %s", cudaGetErrorString(e));
        if (net->forward_from_f32_device(n, net->stream)) return -1;
    } else {
        if (net->forward_device(n, net->stream)) return -1;
    }
    cudaError_t e = cudaStreamSynchronize(net->stream);
    if (e != cudaSuccess) return ara::set_error("ara_net_forward_device: %s", cudaGetErrorString(e));
    if (value_dev) *value_dev = net->d_value;
    if (prob_dev) *prob_dev = net->d_prob;
    return 0;
}

extern "C" long long ara_net_launch_count(ara_net_t h) { return h ? reinterpret_cast<Net*>(h)->launches : 0; }

extern "C" int ara_net_debug_trunk_cycles(ara_net_t h, unsigned long long* out32) {
    if (h == nullptr || out32 == nullptr) return ara::set_error("ara_net_debug_trunk_cycles: null argument");
    return reinterpret_cast<Net*>(h)->trunk_cycles(out32);
}
