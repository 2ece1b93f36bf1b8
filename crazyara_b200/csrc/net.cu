// RISE network: blob loader, weight re-layout for the wgmma GEMMs, forward launch sequence, C-ABI.
#include "net.h"

#include <cstdio>
#include <cstring>
#include <memory>

#include "ara_b200.h"
#include "net_kernels.cuh"
#include "ntb_attention.cuh"

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

// w: [n_out, cin, k, k] fp32 -> fp16 [round_up(n_out, 256), taps * parts * cw] with cw = ceil64(cin); per tap the
// columns are w [cw] (parts 1), or for Precision float32 hi(w) [cw] | lo(w) [cw] | hi(w) [cw] (parts 3), matching
// activations stored as hi | hi | lo (conv_gemm.cuh).
int Net::upload_conv_w(const float* w, int n_out, int cin, int ksize, int parts, __half** dst) {
    const int taps = ksize * ksize;
    const int cw = round_up(cin, 64);
    std::vector<__half> h(static_cast<size_t>(round_up(n_out, 256)) * taps * parts * cw, __float2half(0.0f));
    for (int n = 0; n < n_out; ++n)
        for (int c = 0; c < cin; ++c)
            for (int t = 0; t < taps; ++t) {
                const float v = w[(static_cast<size_t>(n) * cin + c) * taps + t];
                const __half hi = __float2half_rn(v);
                __half* col = &h[(static_cast<size_t>(n) * taps + t) * parts * cw];
                col[c] = hi;
                if (parts == 3) {
                    col[cw + c] = __float2half_rn(v - __half2float(hi));
                    col[2 * cw + c] = hi;
                }
            }
    if (mem_.dalloc(dst, h.size()) != 0) return -1;
    ARA_CUDA_OK(cudaMemcpy(*dst, h.data(), h.size() * sizeof(__half), cudaMemcpyHostToDevice));
    return 0;
}

// One conv_gemm layer: uploads its weights w [n_out][cin][k][k] (split in float32), then its bias [n_out] (none if
// empty), both zero padded to round_up(n_out, 256) rows, and points L at them and at io.
int Net::build_conv(ConvLayer* L, const std::vector<float>& w, const std::vector<float>& bias, int n_out, int cin, int ksize,
                    int relu, const ConvIo& io) {
    const int rows = round_up(n_out, 256);
    __half* dw = nullptr;
    float* db = nullptr;
    if (upload_conv_w(w.data(), n_out, cin, ksize, precision == 0 ? 1 : 3, &dw)) return -1;
    if (!bias.empty() && upload_f32(bias.data(), bias.size(), rows, &db)) return -1;
    return conv_layer_build(L, dw, rows, db, n_out, cin, ksize, relu, precision, batch_cap, conv_layer_choose_bn(batch, n_out), io);
}

template <typename... KArgs, typename... Args>
int Net::launch(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t s, Args... args) {
    ARA_CUDA_OK(launch_pdl(kernel, grid, block, smem, s, args...));
    ++launches;
    return 0;
}

int Net::launch_conv(const ConvLayer& L, int n, cudaStream_t s, const int* cnt) {
    if (conv_layer_launch(&L, n, s, cnt)) return -1;
    ++launches;
    return 0;
}

int Net::launch_tower(size_t segment, int n, cudaStream_t s, const int* cnt, const __half* x_in) {
    if (rise_trunk_launch(trunks_[segment].get(), n, s, cnt, x_in)) return -1;
    ++launches;
    return 0;
}

Net::~Net() {
    cudaSetDevice(device);
    for (auto& family : graphs_)
        for (auto& g : family) cudaGraphExecDestroy(g.second.exec);
    if (stream) cudaStreamDestroy(stream);
    if (head_stream) cudaStreamDestroy(head_stream);
    if (ev_fork) cudaEventDestroy(ev_fork);
    if (ev_join) cudaEventDestroy(ev_join);
}

// zero-pads a tensor [a][b][c] to [a2][b2][c]
static void pad3(std::vector<float>* v, int a, int b, int c, int a2, int b2) {
    std::vector<float> o(static_cast<size_t>(a2) * b2 * c, 0.f);
    for (int i = 0; i < a; ++i)
        for (int j = 0; j < b; ++j)
            memcpy(&o[(static_cast<size_t>(i) * b2 + j) * c], &(*v)[(static_cast<size_t>(i) * b + j) * c], c * sizeof(float));
    v->swap(o);
}

int Net::read_blob(const char* blob_path, HostWeights* hw) {
    BlobReader rd;
    rd.f = fopen(blob_path, "rb");
    if (!rd.f) return set_error("ara_net_create: cannot open weight blob '%s'", blob_path);
    // ARAB2001: the networks of the reference's PyTorch definition.  ARAB2002 (the MXNet symbols) adds the header flags
    // stem_act and policy_bias, and per block flags and the squeeze-excitation gate.  ARAB2003 (AlphaVile) has the header
    // of ARAB2002 with trunks of 64..256 channels and a type word per block: 0 an ARAB2001 bottleneck block, 1 an NTB.
    // ARAB2004 is one of the three with a fully-connected policy head (the trainer's select_policy_from_plane = False): the
    // base format (1, 2 or 3) and the label count L, the base blob from its header on, then the head's tensors.
    char magic[8];
    if (!rd.read(magic, 8) || memcmp(magic, "ARAB200", 7) != 0 || magic[7] < '1' || magic[7] > '4')
        return set_error("ara_net_create: '%s' is not an ARAB2001 / ARAB2002 / ARAB2003 / ARAB2004 weight blob", blob_path);
    int base = magic[7] - '0';
    hdr.n_classic = 0;
    if (base == 4) {
        int w[2];
        if (!rd.read(w, sizeof(w))) return set_error("ara_net_create: truncated header");
        base = w[0];
        hdr.n_classic = w[1];
        if (base < 1 || base > 3) return set_error("ara_net_create: ARAB2004 wraps base format %d (1, 2 or 3)", base);
        if (hdr.n_classic != 1968 && hdr.n_classic != 2272 && hdr.n_classic != 2316)
            return set_error("ara_net_create: %d policy labels (the classic label lists have 1968, 2272 or 2316)", hdr.n_classic);
    }
    const bool v2 = base == 2, v3 = base == 3;
    int h[10] = {0, 0, 0, 0, 0, 0, 0, 0, 1, 0};
    if (!rd.read(h, (v2 || v3 ? 10 : 8) * sizeof(int))) return set_error("ara_net_create: truncated header");
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
    if (hdr.n_classic && hdr.policy_bias)
        return set_error("ara_net_create: ARAB2004 carries the policy convolution's bias with its head, not in the base header");
    // the value head's kind: 0 standard, 1 WDL + plies (value P(win) - P(loss)), 2 the same feeding the value MLP, 3 / 4
    // the MXNet symbols' head: a hidden layer of value_fc units (any base format) in front of the outputs of 1 / 2
    const int kind = hdr.wdl_mode;
    const bool mx_head = kind == kValueHeadMxWdl || kind == kValueHeadMxWdlMlp;
    if (kind < kValueHeadStandard || kind > kValueHeadMxWdlMlp) return set_error("ara_net_create: value head of unknown kind %d", kind);
    if (mx_head && (hdr.value_fc < 1 || hdr.value_fc > 256))
        return set_error("ara_net_create: value head: hidden layer of %d units (1 .. 256)", hdr.value_fc);
    if (v3 ? (hdr.channels % 32 != 0 || hdr.channels < 64 || hdr.channels > 256 || hdr.value_channels != 8 || hdr.value_fc < 1 ||
              hdr.value_fc > 256)
           : (hdr.channels != 256 || hdr.value_channels != 8 || (hdr.value_fc != 256 && !mx_head)))
        return set_error("ara_net_create: unsupported trunk geometry (channels %d, value %d/%d)", hdr.channels,
                         hdr.value_channels, hdr.value_fc);
    if (hdr.n_blocks < 1 || hdr.n_blocks > 64) return set_error("ara_net_create: %d blocks (1 .. 64)", hdr.n_blocks);
    if (hdr.in_channels < 1 || hdr.in_channels > 256 || hdr.policy_channels < 1 || hdr.policy_channels > 256)
        return set_error("ara_net_create: in_channels %d, policy_channels %d (1 .. 256 each)", hdr.in_channels, hdr.policy_channels);
    const int C = hdr.channels;
    blocks.resize(hdr.n_blocks);
    max_cop_ = 0;
    for (int i = 0; i < hdr.n_blocks; ++i) {
        BlockDesc& b = blocks[i];
        int type = 0;
        if (v3 && !rd.read(&type, sizeof(int))) return set_error("ara_net_create: truncated block table");
        b = BlockDesc{0, 3, 0, 0, kTrunkGateHard6, type == 1, 0, 0, 0};
        if (type == 1) {
            int w[3];
            if (!rd.read(w, sizeof(w))) return set_error("ara_net_create: truncated block table");
            b.ntb_m = w[0], b.ntb_ca = w[1], b.ntb_h = w[2];
            if (i == 0) return set_error("ara_net_create: block 0 is an NTB (the tower has to start with a bottleneck block)");
            if (b.ntb_m < 32 || b.ntb_m % 32 != 0 || (b.ntb_ca != 32 && b.ntb_ca != 64) || b.ntb_m + b.ntb_ca != C ||
                b.ntb_h < 64 || b.ntb_h > 1024 || b.ntb_h % 64 != 0)
                return set_error("ara_net_create: block %d: unsupported NTB widths M %d Ca %d H %d (trunk %d channels)", i, b.ntb_m,
                                 b.ntb_ca, b.ntb_h, C);
            if (b.ntb_m > max_m_) max_m_ = b.ntb_m;
            if (b.ntb_ca > max_ca_) max_ca_ = b.ntb_ca;
            if (b.ntb_h > max_h_) max_h_ = b.ntb_h;
            continue;
        }
        if (type != 0) return set_error("ara_net_create: block %d has type %d", i, type);
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
        if (b.se_type != 0 && C != 256)
            return set_error("ara_net_create: block %d: squeeze-excitation on a %d-channel trunk (only 256)", i, C);
        if (b.c_op > max_cop_) max_cop_ = b.c_op;
    }
    if (!rd.tensor(hw->stem_w, static_cast<size_t>(C) * hdr.in_channels * 9) || !rd.tensor(hw->stem_b, C)) return -1;
    hw->blocks.resize(hdr.n_blocks);
    for (int i = 0; i < hdr.n_blocks; ++i) {
        const BlockDesc& bd = blocks[i];
        HostBlock& hb = hw->blocks[i];
        if (bd.ntb) {
            const size_t M = bd.ntb_m, Ca = bd.ntb_ca, H = bd.ntb_h;
            if (!rd.tensor(hb.pe_w, M * C) || !rd.tensor(hb.pe_b, M) || !rd.tensor(hb.qkv_w, 3 * M * M) || !rd.tensor(hb.qkv_b, 3 * M) ||
                !rd.tensor(hb.proj_w, M * M) || !rd.tensor(hb.proj_b, M) || !rd.tensor(hb.prj_w, Ca * M) || !rd.tensor(hb.prj_b, Ca) ||
                !rd.tensor(hb.gc_w, Ca * 32 * 9) || !rd.tensor(hb.gc_b, Ca) || !rd.tensor(hb.mh_w, Ca * Ca) ||
                !rd.tensor(hb.mlp1_w, H * C) || !rd.tensor(hb.mlp1_b, H) || !rd.tensor(hb.mlp2_w, C * H) || !rd.tensor(hb.mlp2_b, C))
                return -1;
            continue;
        }
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
    const int fc = hdr.value_fc;
    if (!rd.tensor(hw->vh_wv, 8 * static_cast<size_t>(C)) || !rd.tensor(hw->vh_bv, 8)) return -1;
    if (!hdr.wdl_mode) {
        if (!rd.tensor(hw->vh_a, static_cast<size_t>(fc) * 512) || !rd.tensor(hw->vh_ab, fc) || !rd.tensor(hw->vh_b, fc) ||
            !rd.tensor(hw->vh_bb, 1))
            return -1;
    } else {
        const size_t hid = mx_head ? fc : 512;  // the features the WDL and plies outputs take
        if (mx_head && (!rd.tensor(hw->vh_hid_w, static_cast<size_t>(fc) * 512) || !rd.tensor(hw->vh_hid_b, fc))) return -1;
        if (!rd.tensor(hw->vh_a, 3 * hid) || !rd.tensor(hw->vh_ab, 3) || !rd.tensor(hw->vh_b, hid) || !rd.tensor(hw->vh_bb, 1))
            return -1;
        if (kind == kValueHeadWdlMlp || kind == kValueHeadMxWdlMlp) {
            long long count = 0;
            if (!rd.read(&count, 8)) return set_error("ara_net_create: truncated value head");
            if (count != 4 * kValueMlp)
                return set_error("ara_net_create: value head: MLP of width %g (the trainers' MLP has %d)", count / 4.0, kValueMlp);
            std::vector<float> w0(4 * kValueMlp), b0, w1, b1;
            if (!rd.read(w0.data(), w0.size() * 4) || !rd.tensor(b0, kValueMlp) || !rd.tensor(w1, kValueMlp) || !rd.tensor(b1, 1))
                return -1;
            hw->vh_mlp = w0;
            hw->vh_mlp.insert(hw->vh_mlp.end(), b0.begin(), b0.end());
            hw->vh_mlp.insert(hw->vh_mlp.end(), w1.begin(), w1.end());
            hw->vh_mlp.insert(hw->vh_mlp.end(), b1.begin(), b1.end());
        }
    }
    if (!rd.tensor(hw->pol_w1, static_cast<size_t>(C) * C * 9) || !rd.tensor(hw->pol_b1, C) ||
        !rd.tensor(hw->pol_w2, static_cast<size_t>(hdr.policy_channels) * C * 9) ||
        (hdr.policy_bias && !rd.tensor(hw->pol_b2, hdr.policy_channels)))
        return -1;
    if (hdr.n_classic && (!rd.tensor(hw->pol_b2, hdr.policy_channels) ||
                          !rd.tensor(hw->fc_w, static_cast<size_t>(hdr.n_classic) * hdr.policy_channels * 64) ||
                          !rd.tensor(hw->fc_b, hdr.n_classic)))
        return -1;
    char tail;
    if (fread(&tail, 1, 1, rd.f) != 0) return set_error("ara_net_create: trailing bytes in weight blob");
    if (C != 256 || fc != 256) {
        // a narrower trunk runs as a 256-channel one: zero weights and biases keep channels C..255 at zero through every
        // ReLU and residual, so everything downstream sees the 256-wide weights of the other networks
        pad3(&hw->stem_w, C, hdr.in_channels * 9, 1, 256, hdr.in_channels * 9);
        pad3(&hw->stem_b, C, 1, 1, 256, 1);
        for (int i = 0; i < hdr.n_blocks; ++i) {
            const BlockDesc& bd = blocks[i];
            HostBlock& hb = hw->blocks[i];
            if (bd.ntb) {
                pad3(&hb.pe_w, bd.ntb_m, C, 1, bd.ntb_m, 256);
                pad3(&hb.mlp1_w, bd.ntb_h, C, 1, bd.ntb_h, 256);
                pad3(&hb.mlp2_w, C, bd.ntb_h, 1, 256, bd.ntb_h);
                pad3(&hb.mlp2_b, C, 1, 1, 256, 1);
            } else {
                pad3(&hb.w1, bd.c_op, C, 1, bd.c_op, 256);
                pad3(&hb.w2, C, bd.c_op, 1, 256, bd.c_op);
                pad3(&hb.b2, C, 1, 1, 256, 1);
            }
        }
        pad3(&hw->vh_wv, 8, C, 1, 8, 256);
        if (!hdr.wdl_mode) {
            pad3(&hw->vh_a, fc, 512, 1, 256, 512);
            pad3(&hw->vh_ab, fc, 1, 1, 256, 1);
            pad3(&hw->vh_b, fc, 1, 1, 256, 1);
        } else if (mx_head) {  // zero hidden units: relu(0) = 0, and zero weights behind them
            pad3(&hw->vh_hid_w, fc, 512, 1, 256, 512);
            pad3(&hw->vh_hid_b, fc, 1, 1, 256, 1);
            pad3(&hw->vh_a, 3, fc, 1, 3, 256);
            pad3(&hw->vh_b, fc, 1, 1, 256, 1);
        }
        pad3(&hw->pol_w1, C, C, 9, 256, 256);
        pad3(&hw->pol_b1, C, 1, 1, 256, 1);
        pad3(&hw->pol_w2, hdr.policy_channels, C, 9, hdr.policy_channels, 256);
        hdr.channels = 256;
        hdr.value_fc = 256;
    }
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

int Net::upload_value_head(const HostWeights& hw) {
    if (upload_f32(hw.vh_wv.data(), hw.vh_wv.size(), hw.vh_wv.size(), &vh_wv)) return -1;
    if (upload_f32(hw.vh_bv.data(), 8, 8, &vh_bv)) return -1;
    // fc1 [256][512] -> [512][256]: the standard head's first layer, or the MXNet WDL heads' hidden layer value_fc0
    auto upload_w1t = [&](const std::vector<float>& w, const std::vector<float>& b) {
        std::vector<float> t2(512 * 256, 0.f);
        for (int o = 0; o < 256; ++o)
            for (int i = 0; i < 512; ++i) t2[i * 256 + o] = w[o * 512 + i];
        return upload_f32(t2.data(), t2.size(), t2.size(), &vh_w1t) || upload_f32(b.data(), 256, 256, &vh_b1);
    };
    if (!hdr.wdl_mode) {
        if (upload_w1t(hw.vh_a, hw.vh_ab)) return -1;
        if (upload_f32(hw.vh_b.data(), 256, 256, &vh_w2)) return -1;
        if (upload_f32(hw.vh_bb.data(), 1, 1, &vh_b2)) return -1;
    } else {
        if (!hw.vh_hid_w.empty() && upload_w1t(hw.vh_hid_w, hw.vh_hid_b)) return -1;
        if (upload_f32(hw.vh_a.data(), hw.vh_a.size(), hw.vh_a.size(), &vh_wdl_w)) return -1;
        if (upload_f32(hw.vh_ab.data(), 3, 4, &vh_wdl_b)) return -1;
        if (upload_f32(hw.vh_b.data(), hw.vh_b.size(), hw.vh_b.size(), &vh_plys_w)) return -1;
        if (upload_f32(hw.vh_bb.data(), 1, 1, &vh_plys_b)) return -1;
        if (!hw.vh_mlp.empty() && upload_f32(hw.vh_mlp.data(), hw.vh_mlp.size(), hw.vh_mlp.size(), &vh_mlp)) return -1;
    }
    return 0;
}

// the NTB weights both precisions upload beyond the blob's: q | k | v with the attention scale 32^-0.5 folded into the q
// rows (so that the attention kernels apply none), and the group convolution as a dense 3x3 with block-diagonal weights
// [Ca][Ca][9] (groups of 32 channels)
static void ntb_device_weights(const BlockDesc& bd, const HostBlock& hb, std::vector<float>* qkv_w, std::vector<float>* qkv_b,
                               std::vector<float>* gc) {
    const int M = bd.ntb_m, Ca = bd.ntb_ca;
    const float scale = static_cast<float>(1.0 / sqrt(static_cast<double>(kNtbHeadDim)));
    *qkv_w = hb.qkv_w;
    *qkv_b = hb.qkv_b;
    for (size_t k = 0; k < static_cast<size_t>(M) * M; ++k) (*qkv_w)[k] *= scale;
    for (int k = 0; k < M; ++k) (*qkv_b)[k] *= scale;
    gc->assign(static_cast<size_t>(Ca) * Ca * 9, 0.f);
    for (int o = 0; o < Ca; ++o)
        for (int c = 0; c < 32; ++c)
            for (int t = 0; t < 9; ++t) (*gc)[(static_cast<size_t>(o) * Ca + (o / 32) * 32 + c) * 9 + t] = hb.gc_w[(static_cast<size_t>(o) * 32 + c) * 9 + t];
}

// Precision float16 NTB: GEMMs on d_x[1] -> d_nt (y1 | z2 | 0) -> d_x[1], see enqueue_ntb_half
int Net::build_ntb_half(const BlockDesc& bd, const HostBlock& hb, NtbLayers* L) {
    const int M = bd.ntb_m, Ca = bd.ntb_ca, H = bd.ntb_h;
    std::vector<float> qkv_w, qkv_b, gc;
    ntb_device_weights(bd, hb, &qkv_w, &qkv_b, &gc);
    __half *x = d_x[1], *z = d_nt + M;
    // y1 and z2 share the rows of d_nt: the layers reading y1 map its M channels only (cin, not rounded to 64), and the
    // layers writing y1 or z2 end at their own columns (n_end)
    if (build_conv(&L->pe, hb.pe_w, hb.pe_b, M, 256, 1, 0, {.act = x, .out_h = d_nt, .ldo = 256, .n_end = M}) ||
        build_conv(&L->qkv, qkv_w, qkv_b, 3 * M, M, 1, 0, {.act = d_nt, .act_pitch = 256, .out_h = d_qkv, .ldo = 3 * M}) ||
        build_conv(&L->proj, hb.proj_w, hb.proj_b, M, M, 1, 0,
                   {.act = d_att, .res_h = d_nt, .ldr = 256, .out_h = d_nt, .ldo = 256, .n_end = M}) ||
        build_conv(&L->prj, hb.prj_w, hb.prj_b, Ca, M, 1, 0, {.act = d_nt, .act_pitch = 256, .out_h = z, .ldo = 256, .n_end = Ca}) ||
        build_conv(&L->gc, gc, hb.gc_b, Ca, Ca, 3, 1, {.act = z, .act_pitch = 256, .out_h = d_g, .ldo = Ca}) ||
        build_conv(&L->mh, hb.mh_w, {}, Ca, Ca, 1, 0, {.act = d_g, .res_h = z, .ldr = 256, .out_h = z, .ldo = 256, .n_end = Ca}) ||
        build_conv(&L->mlp1, hb.mlp1_w, hb.mlp1_b, H, 256, 1, 1, {.act = d_nt, .out_h = d_hid, .ldo = H}) ||
        build_conv(&L->mlp2, hb.mlp2_w, hb.mlp2_b, 256, H, 1, 0, {.act = d_hid, .res_h = d_nt, .ldr = 256, .out_h = x, .ldo = 256}))
        return -1;
    return 0;
}

// Precision float16: stem (wgmma implicit GEMM) -> persistent tower kernel per run of bottleneck blocks, NTB layers
// between them -> heads
int Net::build_half(const HostWeights& hw) {
    const int C = hdr.channels;
    const size_t rows = static_cast<size_t>(batch_cap) * 64;
    if (mem_.dalloc(&d_in_h, rows * cin_pad)) return -1;
    if (mem_.dalloc(&d_x[0], rows * C) || mem_.dalloc(&d_x[1], rows * C) || mem_.dalloc(&d_p1, rows * C)) return -1;
    if (max_m_ > 0 && (mem_.dalloc(&d_nt, rows * 256) || mem_.dalloc(&d_qkv, rows * 3 * max_m_) || mem_.dalloc(&d_att, rows * max_m_) ||
                       mem_.dalloc(&d_g, rows * max_ca_) || mem_.dalloc(&d_hid, rows * max_h_)))
        return -1;
    if (build_conv(&stem_conv, hw.stem_w, hw.stem_b, C, hdr.in_channels, 3, hdr.stem_act,
                   {.act = d_in_h, .act_cin = cin_pad, .out_h = d_x[0], .ldo = C}))
        return -1;
    // the first segment reads the stem output d_x[0]; every later step reads and writes d_x[1] (the tower kernel may run in
    // place, and an NTB's first GEMM reads d_x[1] before its last one writes it)
    std::vector<TrunkBlockHost> tb;
    auto flush = [&]() {
        if (tb.empty()) return 0;
        stages_.push_back({false, static_cast<int>(trunks_.size()), -1});
        trunks_.emplace_back(new RiseTrunk());
        if (rise_trunk_init(trunks_.back().get(), tb, trunks_.size() == 1 ? d_x[0] : d_x[1], d_x[1])) return -1;
        tb.clear();
        return 0;
    };
    for (int i = 0; i < hdr.n_blocks; ++i) {
        const BlockDesc& bd = blocks[i];
        const HostBlock& hb = hw.blocks[i];
        if (bd.ntb) {
            if (flush()) return -1;
            stages_.push_back({true, static_cast<int>(ntbs_.size()), i});
            ntbs_.emplace_back();
            if (build_ntb_half(bd, hb, &ntbs_.back())) return -1;
            continue;
        }
        // a run of more blocks than one tower kernel's argument block holds continues in the next segment: the trunk
        // passes between segments as fp16 in d_x[1], as the kernel keeps it between its own blocks
        if (tb.size() == static_cast<size_t>(kTrunkMaxBlocks) && flush()) return -1;
        tb.emplace_back();
        TrunkBlockHost& t = tb.back();
        t.c_op = bd.c_op;
        t.ksize = bd.kernel;
        t.se_type = bd.se_type;
        t.w1 = hb.w1;
        t.b1 = hb.b1;
        t.wd = hb.wd;
        t.bd = hb.bd;
        t.w2 = hb.w2;
        t.b2 = hb.b2;
        se_transposed(bd, hb, &t.se_w1t, bd.se_type == 1 ? &t.se_w2t : &t.se_b);
        t.flags = bd.flags & kBlobShortcutPreSe ? kTrunkShortcutPreSe : 0;
        t.gate = bd.gate;
        if (bd.se_type == 1) t.se_b1 = hb.se_b1, t.se_b = hb.se_b2;
    }
    if (flush()) return -1;
    if (build_conv(&pol_conv1, hw.pol_w1, hw.pol_b1, C, C, 3, 1, {.act = d_x[1], .out_h = d_p1, .ldo = C})) return -1;
    if (!is_policy_map()) {  // relu(conv2) in fp16 for the fully-connected layer
        if (mem_.dalloc(&d_pol_x, rows * ldp)) return -1;
        return build_conv(&pol_conv2, hw.pol_w2, hw.pol_b2, hdr.policy_channels, C, 3, 1, {.act = d_p1, .out_h = d_pol_x, .ldo = ldp}) ||
               build_policy_fc(hw);
    }
    if (build_conv(&pol_conv2, hw.pol_w2, hw.pol_b2, hdr.policy_channels, C, 3, 0, {.act = d_p1, .out_f = d_logits, .ldo = ldp}))
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
    if (build_conv(&stem_conv, hw.stem_w, hw.stem_b, C, hdr.in_channels, 3, hdr.stem_act,
                   {.act = d_in_h, .out_f = d_xf[0], .out_s = d_xs[0], .ldo = C, .split_cs = C}))
        return -1;
    if (max_m_ > 0) {
        const size_t ms = round_up(max_m_, 64);
        if (mem_.dalloc(&d_yf, rows * max_m_) || mem_.dalloc(&d_qkvf, rows * 3 * max_m_) || mem_.dalloc(&d_zf, rows * max_ca_) ||
            mem_.dalloc(&d_x2f, rows * 256) || mem_.dalloc(&d_ys, rows * 3 * ms) || mem_.dalloc(&d_atts, rows * 3 * ms) ||
            mem_.dalloc(&d_zs, rows * 3 * 64) || mem_.dalloc(&d_gs, rows * 3 * 64) || mem_.dalloc(&d_x2s, rows * 768) ||
            mem_.dalloc(&d_hs, rows * 3 * max_h_))
            return -1;
    }
    pb_.resize(hdr.n_blocks);
    std::vector<float> ta, tbv, t2;
    for (int i = 0; i < hdr.n_blocks; ++i) {
        const BlockDesc& bd = blocks[i];
        const HostBlock& hb = hw.blocks[i];
        PreciseBlock& w = pb_[i];
        const int cp = round_up(bd.c_op, 64);
        const int in = i & 1, out = (i + 1) & 1;
        if (bd.ntb) {
            ntbs_.emplace_back();
            if (build_ntb_precise(bd, hb, in, out, &ntbs_.back())) return -1;
            continue;
        }
        if (bd.se_type != 0) {
            se_transposed(bd, hb, &ta, &tbv);
            if (upload_f32(ta.data(), ta.size(), ta.size(), &w.se_w1t)) return -1;
            if (upload_f32(tbv.data(), tbv.size(), tbv.size(), bd.se_type == 1 ? &w.se_w2t : &w.se_b)) return -1;
            if (!hb.se_b1.empty() && (upload_f32(hb.se_b1.data(), 128, 128, &w.se_b1) || upload_f32(hb.se_b2.data(), 256, 256, &w.se_b)))
                return -1;
        }
        // conv1 1x1 256 -> c_op, ReLU: split X -> fp32 H1
        if (build_conv(&w.conv1, hb.w1, hb.b1, bd.c_op, C, 1, 1, {.act = d_xs[in], .out_f = d_h1f, .ldo = bd.c_op})) return -1;
        // depthwise k x k: blob [c_op][k][k] -> device [k*k][c_op]
        const int kk = bd.kernel * bd.kernel;
        t2.assign(static_cast<size_t>(kk) * bd.c_op, 0.f);
        for (int c = 0; c < bd.c_op; ++c)
            for (int q = 0; q < kk; ++q) t2[static_cast<size_t>(q) * bd.c_op + c] = hb.wd[static_cast<size_t>(c) * kk + q];
        if (upload_f32(t2.data(), t2.size(), t2.size(), &w.wd)) return -1;
        if (upload_f32(hb.bd.data(), bd.c_op, cp, &w.bd)) return -1;
        // conv2 1x1 c_op -> 256 + fp32 residual: split H2 [.., 3*cp] -> fp32 X' and split X'
        if (build_conv(&w.conv2, hb.w2, hb.b2, C, bd.c_op, 1, 0,
                       {.act = d_h2s, .res_f = d_xf[in], .ldr = C, .out_f = d_xf[out], .out_s = d_xs[out], .ldo = C, .split_cs = C}))
            return -1;
    }
    if (build_conv(&pol_conv1, hw.pol_w1, hw.pol_b1, C, C, 3, 1, {.act = d_xs[hdr.n_blocks & 1], .out_s = d_p1, .ldo = C, .split_cs = C}))
        return -1;
    if (!is_policy_map()) {  // relu(conv2) split for the fully-connected layer
        const int cs = round_up(hdr.policy_channels, 64);
        if (mem_.dalloc(&d_pol_x, rows * 3 * cs) ||
            build_conv(&pol_conv2, hw.pol_w2, hw.pol_b2, hdr.policy_channels, C, 3, 1, {.act = d_p1, .out_s = d_pol_x, .ldo = cs, .split_cs = cs}) ||
            build_policy_fc(hw))
            return -1;
    } else if (build_conv(&pol_conv2, hw.pol_w2, hw.pol_b2, hdr.policy_channels, C, 3, 0, {.act = d_p1, .out_f = d_logits, .ldo = ldp})) {
        return -1;
    }
    ARA_CUDA_OK(cudaFuncSetAttribute(value_head_kernel<float>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                     value_head_smem<float>()));
    ARA_CUDA_OK(cudaFuncSetAttribute(nchw_f32_to_nhwc_split_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                     hdr.in_channels * 65 * 4));
    return 0;
}

// Precision float32 NTB: reads the split d_xs[in], writes d_xf[out] and its split d_xs[out], see enqueue_ntb_precise
int Net::build_ntb_precise(const BlockDesc& bd, const HostBlock& hb, int in, int out, NtbLayers* L) {
    const int M = bd.ntb_m, Ca = bd.ntb_ca, H = bd.ntb_h, ms = round_up(M, 64);
    std::vector<float> qkv_w, qkv_b, gc;
    ntb_device_weights(bd, hb, &qkv_w, &qkv_b, &gc);
    if (build_conv(&L->pe, hb.pe_w, hb.pe_b, M, 256, 1, 0, {.act = d_xs[in], .out_f = d_yf, .out_s = d_ys, .ldo = M, .split_cs = ms}) ||
        build_conv(&L->qkv, qkv_w, qkv_b, 3 * M, M, 1, 0, {.act = d_ys, .out_f = d_qkvf, .ldo = 3 * M}) ||
        build_conv(&L->proj, hb.proj_w, hb.proj_b, M, M, 1, 0,
                   {.act = d_atts, .res_f = d_yf, .ldr = M, .out_f = d_x2f, .out_s = d_ys, .ldo = 256, .n_end = M, .split_cs = ms}) ||
        build_conv(&L->prj, hb.prj_w, hb.prj_b, Ca, M, 1, 0, {.act = d_ys, .out_f = d_zf, .out_s = d_zs, .ldo = Ca, .split_cs = 64}) ||
        build_conv(&L->gc, gc, hb.gc_b, Ca, Ca, 3, 1, {.act = d_zs, .out_s = d_gs, .ldo = Ca, .split_cs = 64}) ||
        build_conv(&L->mh, hb.mh_w, {}, Ca, Ca, 1, 0,
                   {.act = d_gs, .res_f = d_zf, .ldr = Ca, .out_f = d_x2f + M, .ldo = 256, .n_end = Ca}) ||
        build_conv(&L->mlp1, hb.mlp1_w, hb.mlp1_b, H, 256, 1, 1, {.act = d_x2s, .out_s = d_hs, .ldo = H, .split_cs = H}) ||
        build_conv(&L->mlp2, hb.mlp2_w, hb.mlp2_b, 256, H, 1, 0,
                   {.act = d_hs, .res_f = d_x2f, .ldr = 256, .out_f = d_xf[out], .out_s = d_xs[out], .ldo = 256, .split_cs = 256}))
        return -1;
    return 0;
}

int policy_fc_square_cols(int P, int precision) { return precision == 0 ? round_up(P, 32) : 3 * round_up(P, 64); }

std::vector<__half> policy_fc_weight_image(const float* w_fc, int L, int P, int precision) {
    const int parts = precision == 0 ? 1 : 3;
    const int cs = policy_fc_square_cols(P, precision) / parts;
    const int K = 64 * parts * cs;
    std::vector<__half> h(static_cast<size_t>(round_up(L, 64)) * K, __float2half(0.0f));
    for (int l = 0; l < L; ++l)
        for (int c = 0; c < P; ++c)
            for (int sq = 0; sq < 64; ++sq) {
                const float v = w_fc[(static_cast<size_t>(l) * P + c) * 64 + sq];
                const __half hi = __float2half_rn(v);
                __half* col = &h[static_cast<size_t>(l) * K + static_cast<size_t>(sq) * parts * cs];
                col[c] = hi;
                if (parts == 3) {
                    col[cs + c] = __float2half_rn(v - __half2float(hi));
                    col[2 * cs + c] = hi;
                }
            }
    return h;
}

void policy_fc_split(int L, int K, int* kb_per_split, int* splits) {
    const int m_tiles = round_up(L, 64) / 64, num_kb = K / 64;
    const int want = (kFcTargetCtas + m_tiles - 1) / m_tiles;
    *kb_per_split = (num_kb + want - 1) / want;
    *splits = (num_kb + *kb_per_split - 1) / *kb_per_split;
}

int policy_fc_choose_bn(int batch) { return batch <= 32 ? 32 : batch <= 64 ? 64 : 128; }

int policy_fc_build(PolicyFcLayer* F, const __half* w, const float* bias, const __half* x, float* part, int L, int P,
                    int precision, int rows_cap, int bn) {
    const int lp = round_up(L, 64);
    const int K = 64 * policy_fc_square_cols(P, precision);
    int kb_per = 0;
    policy_fc_split(L, K, &kb_per, &F->splits);
    F->args = PolicyFcArgs{kb_per, K / 64, lp, rows_cap, part, nullptr};
    F->bias = bias;
    F->L = L;
    F->bn = bn;
    if (make_weight_tensor_map(&F->tm_w, w, K, lp, 64) || make_weight_tensor_map(&F->tm_x, x, K, rows_cap, bn)) return -1;
    switch (bn) {
        case 32: ARA_CUDA_OK(cudaFuncSetAttribute(policy_fc_kernel<32>, cudaFuncAttributeMaxDynamicSharedMemorySize, PolicyFcCfg<32>::kSmemBytes)); break;
        case 64: ARA_CUDA_OK(cudaFuncSetAttribute(policy_fc_kernel<64>, cudaFuncAttributeMaxDynamicSharedMemorySize, PolicyFcCfg<64>::kSmemBytes)); break;
        case 128: ARA_CUDA_OK(cudaFuncSetAttribute(policy_fc_kernel<128>, cudaFuncAttributeMaxDynamicSharedMemorySize, PolicyFcCfg<128>::kSmemBytes)); break;
        default: return set_error("policy_fc_build: N tile %d (32, 64 or 128)", bn);
    }
    ARA_CUDA_OK(cudaFuncSetAttribute(policy_fc_softmax_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, L * 4));
    return 0;
}

int policy_fc_launch(const PolicyFcLayer& F, int n, float* prob, cudaStream_t s, const int* boards_dev) {
    PolicyFcArgs a = F.args;
    a.boards_dev = boards_dev;
    const dim3 grid(a.lp / 64, F.splits, (n + F.bn - 1) / F.bn);
    ARA_CUDA_OK(F.bn == 32 ? launch_pdl(policy_fc_kernel<32>, grid, dim3(kFcThreads), PolicyFcCfg<32>::kSmemBytes, s, F.tm_w, F.tm_x, a)
                : F.bn == 64 ? launch_pdl(policy_fc_kernel<64>, grid, dim3(kFcThreads), PolicyFcCfg<64>::kSmemBytes, s, F.tm_w, F.tm_x, a)
                             : launch_pdl(policy_fc_kernel<128>, grid, dim3(kFcThreads), PolicyFcCfg<128>::kSmemBytes, s, F.tm_w, F.tm_x, a));
    ARA_CUDA_OK(launch_pdl(policy_fc_softmax_kernel, dim3(n), dim3(256), F.L * 4, s, static_cast<const float*>(a.part), F.bias, prob,
                           F.L, a.lp, F.splits, a.rows_cap, boards_dev));
    return 0;
}

// The fully-connected policy head on d_pol_x: float16 rows [batch_cap][64 ldp], float32 the split rows
int Net::build_policy_fc(const HostWeights& hw) {
    const int L = hdr.n_classic, P = hdr.policy_channels, lp = round_up(L, 64);
    const std::vector<__half> h = policy_fc_weight_image(hw.fc_w.data(), L, P, precision);
    if (mem_.dalloc(&fc_w, h.size())) return -1;
    ARA_CUDA_OK(cudaMemcpy(fc_w, h.data(), h.size() * sizeof(__half), cudaMemcpyHostToDevice));
    if (upload_f32(hw.fc_b.data(), L, lp, &fc_b)) return -1;
    int kb_per = 0, splits = 0;
    policy_fc_split(L, 64 * policy_fc_square_cols(P, precision), &kb_per, &splits);
    if (mem_.dalloc(&d_fc_part, static_cast<size_t>(splits) * batch_cap * lp)) return -1;
    return policy_fc_build(&fc_, fc_w, fc_b, d_pol_x, d_fc_part, L, P, precision, batch_cap, policy_fc_choose_bn(batch));
}

// The policy head after the first convolution: the second convolution, then the softmax over its P * 64 logits, or the
// fully-connected layer and the softmax over its L logits
int Net::launch_policy_head(int n, cudaStream_t s, const int* cnt, int io) {
    if (launch_conv(pol_conv2, n, s, cnt)) return -1;
    if (is_policy_map())
        return launch(policy_softmax_kernel, dim3(n), dim3(256), n_labels() * 4, s, d_logits, io_prob[io], hdr.policy_channels, ldp, cnt);
    if (policy_fc_launch(fc_, n, io_prob[io], s, cnt)) return -1;
    launches += 2;
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
    HostWeights hw;  // (host work only: a malformed blob is reported before any device is touched)
    if (read_blob(blob_path, &hw)) return -1;
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
    if (is_policy_map())  // (the fully-connected head's softmax: policy_fc_build)
        ARA_CUDA_OK(cudaFuncSetAttribute(policy_softmax_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, n_labels() * 4));
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
    if (from_f32 && launch(nchw_f32_to_nhwc_split_kernel, dim3(n), dim3(256), hdr.in_channels * 65 * 4, s, d_in_f32, io_in_h[io],
                           hdr.in_channels, cin_pad))
        return -1;
    if (launch_conv(io ? stem_conv2 : stem_conv, n, s, cnt)) return -1;
    for (int i = 0, k = 0; i < hdr.n_blocks; ++i) {
        const BlockDesc& bd = blocks[i];
        PreciseBlock& w = pb_[i];
        const int in = i & 1;
        if (bd.ntb) {
            if (enqueue_ntb_precise(bd, ntbs_[k++], n, s, cnt)) return -1;
            continue;
        }
        if (bd.se_type != 0 && launch(se_f32_kernel, dim3(n), dim3(256), 0, s, d_xf[in], d_xs[in], w.se_w1t, w.se_w2t, w.se_b, w.se_b1,
                                      bd.se_type, bd.gate, (bd.flags & kBlobShortcutPreSe) ? 1 : 0))
            return -1;
        if (launch_conv(w.conv1, n, s)) return -1;
        const long long total = static_cast<long long>(n) * 64 * bd.c_op;
        const int grid = static_cast<int>((total + 255) / 256);
        const int cp = round_up(bd.c_op, 64);
        if (launch(bd.kernel == 3 ? dwconv_f32_kernel<3> : dwconv_f32_kernel<5>, dim3(grid), dim3(256), 0, s, d_h1f, w.wd, w.bd, d_h2s, n,
                   bd.c_op, cp))
            return -1;
        if (launch_conv(w.conv2, n, s)) return -1;
    }
    const float* xfinal = d_xf[hdr.n_blocks & 1];
    ValueHeadW vw{vh_wv, vh_bv, vh_w1t, vh_b1, vh_w2, vh_b2, vh_wdl_w, vh_wdl_b, vh_plys_w, vh_plys_b, vh_mlp, hdr.wdl_mode};
    if (launch(value_head_kernel<float>, dim3(n), dim3(256), value_head_smem<float>(), s, xfinal, vw, io_value[io], io_aux[io], cnt) ||
        launch_conv(pol_conv1, n, s, cnt) || launch_policy_head(n, s, cnt, io))
        return -1;
    ARA_CUDA_OK(cudaGetLastError());
    return 0;
}

// The attention of an NTB of width M over n boards: grid (boards, heads).  float16: qkv [n * 64][3M] fp16 -> out
// [n * 64][M] fp16; float32: qkv fp32 -> out the split [n * 64][3 * ceil64(M)] (hi | hi | lo).
static cudaError_t ntb_attention_launch(int precision, const void* qkv, __half* out, int M, int n, cudaStream_t s, const int* cnt) {
    if (precision == 0)
        return launch_pdl(ntb_attention_kernel, dim3(n, M / kNtbHeadDim), dim3(128), 0, s, static_cast<const __half*>(qkv), out, M, cnt);
    return launch_pdl(ntb_attention_f32_kernel, dim3(n, M / kNtbHeadDim), dim3(64), 0, s, static_cast<const float*>(qkv), out, M,
                      round_up(M, 64), cnt);
}

int Net::launch_attention(const void* qkv, __half* out, int M, int n, cudaStream_t s, const int* cnt) {
    ARA_CUDA_OK(ntb_attention_launch(precision, qkv, out, M, n, s, cnt));
    ++launches;
    return 0;
}

// y = patch_embed(x); q|k|v; attention; y1 = y + proj(attention); z = projection(y1); z2 = z + conv1x1(relu(group
// conv(z))); x' = x2 + mlp2(relu(mlp1(x2))) with x2 = y1 | z2 -- 9 launches, next_vit_official_modules.py:321-335
int Net::enqueue_ntb_half(const BlockDesc& bd, const NtbLayers& L, int n, cudaStream_t s, const int* cnt) {
    if (launch_conv(L.pe, n, s, cnt) || launch_conv(L.qkv, n, s, cnt) ||
        launch_attention(d_qkv, d_att, bd.ntb_m, n, s, cnt) ||
        launch_conv(L.proj, n, s, cnt) || launch_conv(L.prj, n, s, cnt) || launch_conv(L.gc, n, s, cnt) || launch_conv(L.mh, n, s, cnt) ||
        launch_conv(L.mlp1, n, s, cnt) || launch_conv(L.mlp2, n, s, cnt))
        return -1;
    return 0;
}

// the same in split form: fp32 activations, the split operand of every GEMM in its own buffer, one fp32 -> split
// conversion of x2 -- 10 launches
int Net::enqueue_ntb_precise(const BlockDesc& bd, const NtbLayers& L, int n, cudaStream_t s, const int* cnt) {
    if (launch_conv(L.pe, n, s, cnt) || launch_conv(L.qkv, n, s, cnt) ||
        launch_attention(d_qkvf, d_atts, bd.ntb_m, n, s, cnt) ||
        launch_conv(L.proj, n, s, cnt) || launch_conv(L.prj, n, s, cnt) || launch_conv(L.gc, n, s, cnt) || launch_conv(L.mh, n, s, cnt) ||
        launch(f32_to_split256_kernel, dim3(n * 64), dim3(256), 0, s, d_x2f, d_x2s, cnt) || launch_conv(L.mlp1, n, s, cnt) ||
        launch_conv(L.mlp2, n, s, cnt))
        return -1;
    return 0;
}

bool Net::stem_beside_tower(int n) const {
    return precision == 0 && d_x0_alt != nullptr &&
           rise_trunk_ctas(trunks_[0].get(), n) + conv_layer_ctas(&stem_conv2, n) <= trunks_[0]->sm_count;
}

int Net::stem_device(int n, cudaStream_t s, const int* cnt, int io) {
    if (!stem_beside_tower(n) || io < 0 || io > 1) return set_error("stem_device: needs Precision float16, two input / output sets and room beside the tower");
    return launch_conv(io ? stem_conv2 : stem_conv, n, s, cnt);
}

int Net::enqueue(int n, cudaStream_t s, bool from_f32, const int* cnt, int io, bool stem_done) {
    if (precision == 1) return enqueue_precise(n, s, from_f32, cnt, io);
    if (from_f32 && launch(nchw_f32_to_nhwc_f16_kernel, dim3(n), dim3(256), hdr.in_channels * 65 * 4, s, d_in_f32, io_in_h[io],
                           hdr.in_channels, cin_pad))
        return -1;
    if (!stem_done && launch_conv(io ? stem_conv2 : stem_conv, n, s, cnt)) return -1;
    {   // two input / output sets = a search with Threads = 2: the tower is the first kernel of this stream's chain and
        // must not sit on its SMs waiting for the tree stream's event (see PdlSuspend); the small kernels behind it keep
        // their programmatic launches (the tower triggers them at its last block)
        PdlSuspend no_pdl(io_in_h[1] != nullptr);
        if (launch_tower(0, n, s, cnt, (io == 1 && d_x0_alt != nullptr) ? d_x0_alt : nullptr)) return -1;
    }
    for (size_t k = 1; k < stages_.size(); ++k) {
        const Stage& st = stages_[k];
        if (st.ntb ? enqueue_ntb_half(blocks[st.block], ntbs_[st.index], n, s, cnt) : launch_tower(st.index, n, s, cnt)) return -1;
    }
    __half* xfinal = d_x[1];
    ValueHeadW vw{vh_wv, vh_bv, vh_w1t, vh_b1, vh_w2, vh_b2, vh_wdl_w, vh_wdl_b, vh_plys_w, vh_plys_b, vh_mlp, hdr.wdl_mode};
    // value head on the side stream (a second branch of the captured graph), policy head on s
    ARA_CUDA_OK(cudaEventRecord(ev_fork, s));
    ARA_CUDA_OK(cudaStreamWaitEvent(head_stream, ev_fork, 0));
    value_head_kernel<__half><<<dim3(n), dim3(256), value_head_smem<__half>(), head_stream>>>(xfinal, vw, io_value[io], io_aux[io], cnt);
    ++launches;
    ARA_CUDA_OK(cudaEventRecord(ev_join, head_stream));
    if (launch_conv(pol_conv1, n, s, cnt) || launch_policy_head(n, s, cnt, io)) return -1;
    ARA_CUDA_OK(cudaStreamWaitEvent(s, ev_join, 0));
    ARA_CUDA_OK(cudaGetLastError());
    return 0;
}

int Net::forward_device(int n, cudaStream_t s, const int* cnt, int io, bool stem_done) {
    if (stem_done && !stem_beside_tower(n)) return set_error("forward: stem_done needs Precision float16, two input / output sets and room beside the tower");
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
        for (auto& g : graphs_[gk]) cudaGraphExecDestroy(g.second.exec);
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
// warm-up and is then captured; the launches the capture enqueued are counted at each replay instead.
int Net::launch_graph(int family, int n, cudaStream_t s, bool from_f32, const int* cnt, int io, bool stem_done) {
    auto& graphs = graphs_[family];
    auto it = graphs.find(n);
    if (it == graphs.end()) {
        if (enqueue(n, s, from_f32, cnt, io, stem_done)) return -1;
        ARA_CUDA_OK(cudaStreamSynchronize(s));
        const long long before = launches;
        cudaGraphExec_t ge;
        const int rc = capture_graph(s, &ge, [&] { return enqueue(n, s, from_f32, cnt, io, stem_done); });
        const long long captured = launches - before;
        launches = before;
        if (rc) return -1;
        it = graphs.emplace(n, Captured{ge, captured}).first;
    }
    ARA_CUDA_OK(cudaGraphLaunch(it->second.exec, s));
    launches += it->second.launches;
    return 0;
}

int Net::trunk_cycles(unsigned long long* out32) {
    if (precision != 0 || trunks_.empty()) return set_error("trunk kernel not in use");
    ARA_CUDA_OK(cudaSetDevice(device));
    ARA_CUDA_OK(cudaStreamSynchronize(stream));
    ARA_CUDA_OK(cudaMemcpy(out32, trunks_[0]->d_prof, 32 * sizeof(unsigned long long), cudaMemcpyDeviceToHost));
    return 0;
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
    // 1: the policy head is a convolution onto P x 8 x 8 planes; 0: a fully-connected layer onto the classic label list
    // (builder_util.py:206-243, select_policy_from_plane)
    if (is_policy_map) *is_policy_map = net->is_policy_map() ? 1 : 0;
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

namespace {
// the device-side board count of the debug entries: count >= 0 in a fresh device int, -1 none
int debug_count(ara::DeviceBuffers* mem, int count, int** dev) {
    *dev = nullptr;
    if (count < 0) return 0;
    if (mem->dalloc(dev, 1)) return -1;
    ARA_CUDA_OK(cudaMemcpy(*dev, &count, sizeof(int), cudaMemcpyHostToDevice));
    return 0;
}
}  // namespace

extern "C" int ara_debug_ntb_attention(const void* qkv, int n, int M, int precision, int count, void* out) {
    if (M < 32 || M % 32 != 0 || M > 224) return ara::set_error("ara_debug_ntb_attention: M %d (32 .. 224 in steps of 32)", M);
    if (n < 1) return ara::set_error("ara_debug_ntb_attention: %d boards", n);
    if (precision != ARA_PRECISION_FLOAT16 && precision != ARA_PRECISION_FLOAT32)
        return ara::set_error("ara_debug_ntb_attention: precision %d (0 = float16, 1 = float32)", precision);
    if (count < -1 || count > n) return ara::set_error("ara_debug_ntb_attention: board count %d of %d boards", count, n);
    if (qkv == nullptr || out == nullptr) return ara::set_error("ara_debug_ntb_attention: null buffer");
    const size_t rows = static_cast<size_t>(n) * 64;
    const size_t in_bytes = rows * 3 * M * (precision == 0 ? 2 : 4);
    const size_t out_bytes = rows * (precision == 0 ? M : 3 * ara::round_up(M, 64)) * 2;
    ara::DeviceBuffers mem;
    uint8_t *d_in = nullptr, *d_out = nullptr;
    int* d_cnt = nullptr;
    if (mem.dalloc(&d_in, in_bytes) || mem.dalloc(&d_out, out_bytes) || debug_count(&mem, count, &d_cnt)) return -1;
    ARA_CUDA_OK(cudaMemcpy(d_in, qkv, in_bytes, cudaMemcpyHostToDevice));
    ARA_CUDA_OK(cudaMemcpy(d_out, out, out_bytes, cudaMemcpyHostToDevice));
    ARA_CUDA_OK(ara::ntb_attention_launch(precision, d_in, reinterpret_cast<__half*>(d_out), M, n, nullptr, d_cnt));
    ARA_CUDA_OK(cudaMemcpy(out, d_out, out_bytes, cudaMemcpyDeviceToHost));
    return 0;
}

extern "C" int ara_debug_policy_fc(int precision, int P, int L, int boards, int batch, int bn, int count, const float* w_fc,
                                   const float* b_fc, const void* x, float* part, float* prob, int* splits_out, int* kb_per_split_out) {
    if (precision != ARA_PRECISION_FLOAT16 && precision != ARA_PRECISION_FLOAT32)
        return ara::set_error("ara_debug_policy_fc: precision %d (0 = float16, 1 = float32)", precision);
    if (P < 1 || P > 256) return ara::set_error("ara_debug_policy_fc: %d policy planes (1 .. 256)", P);
    if (L != 1968 && L != 2272 && L != 2316) return ara::set_error("ara_debug_policy_fc: %d labels (1968, 2272 or 2316)", L);
    if (batch < 1 || boards < 1 || boards > batch) return ara::set_error("ara_debug_policy_fc: %d boards of a batch of %d", boards, batch);
    if (bn != 0 && bn != 32 && bn != 64 && bn != 128) return ara::set_error("ara_debug_policy_fc: N tile %d (0, 32, 64 or 128)", bn);
    if (count < -1 || count > boards) return ara::set_error("ara_debug_policy_fc: board count %d of %d boards", count, boards);
    const int K = 64 * ara::policy_fc_square_cols(P, precision);
    int kb_per = 0, splits = 0;
    ara::policy_fc_split(L, K, &kb_per, &splits);
    if (splits_out) *splits_out = splits;
    if (kb_per_split_out) *kb_per_split_out = kb_per;
    if (x == nullptr && part == nullptr && prob == nullptr) return 0;
    if (w_fc == nullptr || b_fc == nullptr || x == nullptr || part == nullptr || prob == nullptr)
        return ara::set_error("ara_debug_policy_fc: null buffer");
    const int rows_cap = ara::round_up(batch < 2 ? 2 : batch, 2), lp = ara::round_up(L, 64);  // Net::batch_cap
    const size_t part_bytes = static_cast<size_t>(splits) * rows_cap * lp * 4, prob_bytes = static_cast<size_t>(boards) * L * 4;
    const std::vector<__half> img = ara::policy_fc_weight_image(w_fc, L, P, precision);
    ara::DeviceBuffers mem;
    __half *d_w = nullptr, *d_x = nullptr;
    float *d_b = nullptr, *d_part = nullptr, *d_prob = nullptr;
    int* d_cnt = nullptr;
    if (mem.dalloc(&d_w, img.size()) || mem.dalloc(&d_x, static_cast<size_t>(rows_cap) * K) || mem.dalloc(&d_b, lp) ||
        mem.dalloc(&d_part, part_bytes / 4) || mem.dalloc(&d_prob, prob_bytes / 4) || debug_count(&mem, count, &d_cnt))
        return -1;
    ARA_CUDA_OK(cudaMemcpy(d_w, img.data(), img.size() * sizeof(__half), cudaMemcpyHostToDevice));
    ARA_CUDA_OK(cudaMemcpy(d_x, x, static_cast<size_t>(rows_cap) * K * sizeof(__half), cudaMemcpyHostToDevice));
    ARA_CUDA_OK(cudaMemcpy(d_b, b_fc, static_cast<size_t>(L) * 4, cudaMemcpyHostToDevice));
    ARA_CUDA_OK(cudaMemcpy(d_part, part, part_bytes, cudaMemcpyHostToDevice));
    ARA_CUDA_OK(cudaMemcpy(d_prob, prob, prob_bytes, cudaMemcpyHostToDevice));
    ara::PolicyFcLayer F;
    if (ara::policy_fc_build(&F, d_w, d_b, d_x, d_part, L, P, precision, rows_cap, bn ? bn : ara::policy_fc_choose_bn(batch)) ||
        ara::policy_fc_launch(F, boards, d_prob, nullptr, d_cnt))
        return -1;
    ARA_CUDA_OK(cudaMemcpy(part, d_part, part_bytes, cudaMemcpyDeviceToHost));
    ARA_CUDA_OK(cudaMemcpy(prob, d_prob, prob_bytes, cudaMemcpyDeviceToHost));
    return 0;
}
