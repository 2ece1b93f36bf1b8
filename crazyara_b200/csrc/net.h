// RISE network instance on one GPU stream: weights resident in HBM, activation buffers, launch sequence.
// Mirrors the role of the reference's NeuralNetAPI/TensorrtAPI (engine/src/nn/neuralnetapi.h:148-311,
// engine/src/nn/tensorrtapi.cpp:160-237) but the "engine" is our own kernel sequence.
#pragma once
#include <map>
#include <memory>
#include <string>
#include <vector>

#include "conv_gemm_host.h"
#include "policy_fc.cuh"
#include "rise_trunk_host.h"

namespace ara {

struct BlockDesc {
    int c_op;
    int kernel;   // 3 or 5
    int se_type;  // 0 none, 1 ca_se, 2 eca_se
    int flags;    // ARAB2002: kBlobShortcutPreSe | kBlobSeBias
    int gate;     // ARAB2002: squeeze-excitation gate (kTrunkGate*)
    bool ntb;     // ARAB2003: a NextViT transformer block (AlphaVile) with the widths below instead of a bottleneck block
    int ntb_m, ntb_ca, ntb_h;  // MHSA width M, MHCA width Ca (M + Ca = trunk channels), MLP hidden width H
};
// ARAB2002 block flags: the shortcut adds the block input before the squeeze-excitation; the ca_se fully-connected layers
// have biases
constexpr int kBlobShortcutPreSe = 1, kBlobSeBias = 2;
// the base header's WDL word: the value head's kind (net_kernels.cuh value_head_kernel, weights.py VALUE_HEADS)
constexpr int kValueHeadStandard = 0, kValueHeadWdl = 1, kValueHeadWdlMlp = 2, kValueHeadMxWdl = 3, kValueHeadMxWdlMlp = 4;
constexpr int kValueMlp = 8;  // the hidden width of the trainers' value MLP on (WDL, plies)

// The fully-connected policy layer as a network builds and launches it: policy_fc_kernel<bn> over `splits` K ranges,
// then policy_fc_softmax_kernel.  Net::build_policy_fc and ara_debug_policy_fc both build through policy_fc_build.
struct PolicyFcLayer {
    CUtensorMap tm_w, tm_x;
    PolicyFcArgs args;
    const float* bias;  // [lp] zero padded
    int L, bn, splits;
};
// the columns of one square in a board's row of the layer's input: float16 ceil32(P) (the policy convolution's row
// pitch), float32 3 * ceil64(P) (its split output hi | hi | lo); K = 64 times this
int policy_fc_square_cols(int P, int precision);
// W_fc [L][P * 64] (the trainer's NCHW flatten c * 64 + sq) -> the fp16 image [ceil64(L)][K] with the columns in the
// order of the input rows: float16 sq * ceil32(P) + c, float32 per square hi | lo | hi parts ceil64(P) wide against the
// activations' hi | hi | lo.  Padding rows and columns are zero.
std::vector<__half> policy_fc_weight_image(const float* w_fc, int L, int P, int precision);
// 64-wide K blocks per split and the split count: from L and K only, never from the batch, so that a board's partial
// sums are the same in any batch
void policy_fc_split(int L, int K, int* kb_per_split, int* splits);
// the N tile (boards per CTA) for a layer built for `batch` boards
int policy_fc_choose_bn(int batch);
// w: the image of policy_fc_weight_image, bias [ceil64(L)], x: the input rows [rows_cap][K], part: [splits][rows_cap]
// [ceil64(L)] fp32 partial sums
int policy_fc_build(PolicyFcLayer* F, const __half* w, const float* bias, const __half* x, float* part, int L, int P,
                    int precision, int rows_cap, int bn);
// the two launches of the layer for n boards: prob [n][L]; boards_dev as in PolicyFcArgs
int policy_fc_launch(const PolicyFcLayer& F, int n, float* prob, cudaStream_t s, const int* boards_dev);

struct NetHeader {
    int in_channels;
    int policy_channels;
    int n_blocks;
    int channels;        // 256 (ARAB2003: 64..256, zero padded to 256 at load)
    int value_channels;  // 8
    int value_fc;        // 256 (ARAB2003: <= 256, zero padded to 256 at load)
    int wdl_mode;        // the value head's kind (kValueHead*): WDL + plies-to-end auxiliary outputs from 1 on
    int input_version;   // e.g. 10 = v1.0, 30 = v3.0
    int stem_act;        // 1: ReLU behind the stem convolution (ARAB2001: always)
    int policy_bias;     // 1: the last policy convolution has a bias (ARAB2001: never)
    int n_classic;       // ARAB2004: the fully-connected policy head's label count L (0: a policy-map head)
};

// One NTB as GEMM launches (conv_gemm.cuh) around the attention kernel (ntb_attention.cuh), both precisions
struct NtbLayers {
    ConvLayer pe, qkv, proj, prj, gc, mh, mlp1, mlp2;
};

// Precision float32: one bottleneck block as separate launches on fp32 activations (net.cu, conv_gemm.cuh)
struct PreciseBlock {
    float *se_w1t = nullptr, *se_w2t = nullptr, *se_b = nullptr, *se_b1 = nullptr;
    float *wd = nullptr, *bd = nullptr;
    ConvLayer conv1, conv2;
};

// the tensors of a weight blob, host side, in blob order (weights.py)
struct HostBlock {
    std::vector<float> se_a, se_b;  // ca_se: fc1 [128][256], fc2 [256][128]; eca_se: centre tap [256][256], bias [256]
    std::vector<float> se_b1, se_b2;  // ca_se with kBlobSeBias: fc1 bias [128], fc2 bias [256]
    std::vector<float> w1, b1, wd, bd, w2, b2;
    // NTB (BatchNorms folded, weights [out][in]): patch_embed, q | k | v, proj, projection, group conv [Ca][32][3][3],
    // MHCA conv1x1 (no bias), MLP conv1 / conv2
    std::vector<float> pe_w, pe_b, qkv_w, qkv_b, proj_w, proj_b, prj_w, prj_b, gc_w, gc_b, mh_w, mlp1_w, mlp1_b, mlp2_w, mlp2_b;
};
struct HostWeights {
    std::vector<float> stem_w, stem_b;
    std::vector<HostBlock> blocks;
    std::vector<float> vh_wv, vh_bv, vh_a, vh_ab, vh_b, vh_bb;  // standard: fc1 / b1 / fc2 / b2; WDL: wdl w / b, plys w / b
    std::vector<float> vh_hid_w, vh_hid_b;  // MXNet WDL heads: value_fc0 [value_fc][512], [value_fc]
    std::vector<float> vh_mlp;              // value MLP: w0 [8][4] | b0 [8] | w1 [8] | b1 [1]
    std::vector<float> pol_w1, pol_b1, pol_w2, pol_b2;  // pol_b2: [policy_channels] when hdr.policy_bias or hdr.n_classic
    std::vector<float> fc_w, fc_b;                      // ARAB2004: [L][policy_channels * 64] (NCHW flatten), [L]
};

class Net {
   public:
    Net() = default;
    ~Net();
    // precision: 0 = float16 operands / fp32 accumulate (the reference's default `Precision float16`,
    // uci/optionsuci.cpp:144), 1 = float32 (fp16 hi + lo operand splitting, fp32 activations between the layers)
    int init(const char* blob_path, int device, int batch, int precision);
    // host-buffer API (reference NeuralNetAPI::predict semantics, synchronous)
    int predict(const float* planes_host, int n, float* value_host, float* prob_host, float* aux_host);
    // the same forward, but only the policy entries named by policy_idx come back (ara_net_predict_priors)
    int predict_priors(const float* planes_host, int n, const int* policy_idx, const int* counts, int stride, float* value_host,
                       float* priors_host, float* aux_host);
    // device-resident API: input already in in_h (NHWC fp16), outputs stay in d_value / d_prob
    // boards_dev (optional): device-side count (<= n) of the input rows that really hold positions -- the launch is
    // sized for n, thread blocks of the rows beyond the count leave at once; the pointer is baked into the CUDA graph
    // io: which input / output buffer set (0, or 1 after enable_second_io()): a search with Threads = 2 keeps two
    // batches in flight -- one set is being written / read by the tree kernels while the other is at the network
    // stem_done: the stem convolution of this batch has already run (stem_device, on the caller's own stream)
    int forward_device(int n, cudaStream_t stream, const int* boards_dev = nullptr, int io = 0, bool stem_done = false);
    // The stem convolution alone, into the stem-output buffer of input / output set `io` (stem_beside_tower(n)): a
    // search with two logical threads runs it on its tree stream right behind the plane encoding, which takes it off the
    // network stream's critical path.
    int stem_device(int n, cudaStream_t stream, const int* boards_dev, int io);
    // Precision float16 with two sets enabled, and the stem of n boards fits on the SMs beside the tower of n boards.
    // Where the tower fills the SMs (64 boards on 132 SMs) a stem on the tree stream would wait for the other set's
    // tower and hold up this set's forward: then the forward starts at the stem.
    bool stem_beside_tower(int n) const;
    __half* d_x0_alt = nullptr;  // stem output of set 1 (set 0: d_x[0])
    int enable_second_io();
    int forward_from_f32_device(int n, cudaStream_t stream);  // converts d_in_f32 -> in_h first

    NetHeader hdr{};
    std::vector<BlockDesc> blocks;
    int device = 0;
    int precision = 0;
    int batch = 0;      // max boards per call
    int batch_cap = 0;  // even, >= 2
    int cin_pad = 0;
    int ldp = 0;  // padded policy channels (multiple of 32)
    int n_labels() const { return hdr.n_classic ? hdr.n_classic : hdr.policy_channels * 64; }
    // the policy is P x 64 planes (the convolution's output); false: the classic label list of a fully-connected head
    bool is_policy_map() const { return hdr.n_classic == 0; }
    int n_aux() const { return hdr.wdl_mode ? 4 : 0; }
    int trunk_cycles(unsigned long long* out32);  // -DARA_TRUNK_PROF builds: per-role cycle counters of CTA 0 (first segment)
    cudaStream_t stream = nullptr;
    // the value head runs beside the policy head: forked side stream, joined before the forward ends
    cudaStream_t head_stream = nullptr;
    cudaEvent_t ev_fork = nullptr, ev_join = nullptr;

    // device buffers
    float* d_in_f32 = nullptr;   // [batch, C, 64]
    __half* d_in_h = nullptr;    // [batch_cap, 64, cin_pad] (float32: [batch_cap, 64, 3 * cin_pad] split)
    __half* d_x[2] = {nullptr, nullptr};  // float16: stem output / tower output [batch_cap*64, 256]
    __half* d_p1 = nullptr;      // [batch_cap*64, 256] (float32: [.., 768] split)
    float* d_logits = nullptr;   // [batch_cap*64, ldp]
    float* d_prob = nullptr;     // [batch, L]
    float* d_value = nullptr;    // [batch]
    float* d_aux = nullptr;      // [batch, 4]
    // second input / output set (enable_second_io): [1] of each pair, [0] aliases the members above
    __half* io_in_h[2] = {nullptr, nullptr};
    float* io_prob[2] = {nullptr, nullptr};
    float* io_value[2] = {nullptr, nullptr};
    float* io_aux[2] = {nullptr, nullptr};
    // float32 only: trunk ping-pong in fp32 + split copies, bottleneck intermediates
    float* d_xf[2] = {nullptr, nullptr};  // [batch_cap*64, 256]
    __half* d_xs[2] = {nullptr, nullptr};  // [batch_cap*64, 768]
    float* d_h1f = nullptr;                // [batch_cap*64, max_cop]
    __half* d_h2s = nullptr;               // [batch_cap*64, 3 * ceil64(max_cop)]
    int* d_gather_idx = nullptr;   // predict_priors: [batch, gather_stride] policy indices, [batch] counts, [batch, stride] priors
    int* d_gather_cnt = nullptr;
    float* d_gather_out = nullptr;
    int gather_stride = 0;
    long long launches = 0;      // kernels launched so far (bench bookkeeping)

   private:
    int enqueue(int n, cudaStream_t s, bool from_f32, const int* boards_dev = nullptr, int io = 0, bool stem_done = false);
    int read_blob(const char* blob_path, HostWeights* hw);
    int build_half(const HostWeights& hw);
    int build_precise(const HostWeights& hw);
    int build_conv(ConvLayer* L, const std::vector<float>& w, const std::vector<float>& bias, int n_out, int cin, int ksize,
                   int relu, const ConvIo& io);
    int upload_value_head(const HostWeights& hw);
    // the kernel launches of a forward, each counted in `launches`
    template <typename... KArgs, typename... Args>
    int launch(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t s, Args... args);
    int launch_conv(const ConvLayer& L, int n, cudaStream_t s, const int* boards_dev = nullptr);
    int launch_tower(size_t segment, int n, cudaStream_t s, const int* boards_dev, const __half* x_in = nullptr);
    int enqueue_precise(int n, cudaStream_t s, bool from_f32, const int* boards_dev, int io);
    int launch_graph(int family, int n, cudaStream_t s, bool from_f32, const int* boards_dev, int io, bool stem_done);
    int build_ntb_half(const BlockDesc& bd, const HostBlock& hb, NtbLayers* L);
    int build_ntb_precise(const BlockDesc& bd, const HostBlock& hb, int in, int out, NtbLayers* L);
    int enqueue_ntb_half(const BlockDesc& bd, const NtbLayers& L, int n, cudaStream_t s, const int* boards_dev);
    int enqueue_ntb_precise(const BlockDesc& bd, const NtbLayers& L, int n, cudaStream_t s, const int* boards_dev);
    int launch_attention(const void* qkv, __half* out, int M, int n, cudaStream_t s, const int* boards_dev);
    DeviceBuffers mem_;
    int max_cop_ = 0;
    ConvLayer stem_conv;
    ConvLayer stem_conv2;  // the stem reading the second input set
    std::vector<PreciseBlock> pb_;
    // float16: the tower as segments, one tower kernel per run of at most kTrunkMaxBlocks bottleneck blocks
    std::vector<std::unique_ptr<RiseTrunk>> trunks_;
    std::vector<NtbLayers> ntbs_;  // one per NTB, in block order (both precisions)
    // float16: what runs between the stem and the heads, in block order, as build_half laid it out: tower segment
    // trunks_[index] or NTB ntbs_[index] (of block `block`).  Stage 0 is a tower segment (the blob reader refuses an NTB
    // at block 0).
    struct Stage {
        bool ntb;
        int index, block;
    };
    std::vector<Stage> stages_;
    int max_m_ = 0, max_ca_ = 0, max_h_ = 0;  // the widest NTB
    // NTB activations.  float16: d_nt [rows, 256] = y1 | z2 | 0, d_qkv [rows, 3M], d_att [rows, M], d_g [rows, Ca],
    // d_hid [rows, H].  float32: fp32 y / q|k|v / z / x2 and split y, attention, z, group conv, x2, hidden.
    __half *d_nt = nullptr, *d_qkv = nullptr, *d_att = nullptr, *d_g = nullptr, *d_hid = nullptr;
    float *d_yf = nullptr, *d_qkvf = nullptr, *d_zf = nullptr, *d_x2f = nullptr;
    __half *d_ys = nullptr, *d_atts = nullptr, *d_zs = nullptr, *d_gs = nullptr, *d_x2s = nullptr, *d_hs = nullptr;
    float *vh_wv = nullptr, *vh_bv = nullptr, *vh_w1t = nullptr, *vh_b1 = nullptr, *vh_w2 = nullptr, *vh_b2 = nullptr;
    float *vh_wdl_w = nullptr, *vh_wdl_b = nullptr, *vh_plys_w = nullptr, *vh_plys_b = nullptr, *vh_mlp = nullptr;
    ConvLayer pol_conv1, pol_conv2;
    // fully-connected policy head (policy_fc.cuh): relu(conv2) as fp16 (float32: split) rows, one board per row, weights
    // [lp][K] with their tensor maps, bias, split-K partial sums.  Like d_logits, shared by both input / output sets: their
    // forwards follow each other on the network stream.
    __half* d_pol_x = nullptr;
    __half* fc_w = nullptr;
    float* fc_b = nullptr;
    float* d_fc_part = nullptr;
    PolicyFcLayer fc_{};
    int build_policy_fc(const HostWeights& hw);
    int launch_policy_head(int n, cudaStream_t s, const int* boards_dev, int io);
    struct Captured {
        cudaGraphExec_t exec;
        long long launches;  // the kernel launches the capture enqueued
    };
    std::map<int, Captured> graphs_[6];  // plain, from fp32 input, with a device-side count (io 0), the same for io 1
    const int* baked_[6] = {};           // the counter pointer each graph family was captured with
    int upload_conv_w(const float* w, int n_out, int cin, int ksize, int parts, __half** dst);
    int upload_f32(const float* src, size_t count, size_t padded, float** dst);
};

}  // namespace ara
