// RISE network instance on one GPU stream: weights resident in HBM, activation buffers, launch sequence.
// Mirrors the role of the reference's NeuralNetAPI/TensorrtAPI (engine/src/nn/neuralnetapi.h:148-311,
// engine/src/nn/tensorrtapi.cpp:160-237) but the "engine" is our own kernel sequence.
#pragma once
#include <map>
#include <string>
#include <vector>

#include "conv_gemm_host.h"
#include "rise_trunk_host.h"

namespace ara {

struct BlockDesc {
    int c_op;
    int kernel;   // 3 or 5
    int se_type;  // 0 none, 1 ca_se, 2 eca_se
    int flags;    // ARAB2002: kBlobShortcutPreSe | kBlobSeBias
    int gate;     // ARAB2002: squeeze-excitation gate (kTrunkGate*)
};
// ARAB2002 block flags: the shortcut adds the block input before the squeeze-excitation; the ca_se fully-connected layers
// have biases
constexpr int kBlobShortcutPreSe = 1, kBlobSeBias = 2;

struct NetHeader {
    int in_channels;
    int policy_channels;
    int n_blocks;
    int channels;        // 256
    int value_channels;  // 8
    int value_fc;        // 256
    int wdl_mode;        // 1: value head with WDL + plys-to-end auxiliary outputs
    int input_version;   // e.g. 10 = v1.0, 30 = v3.0
    int stem_act;        // 1: ReLU behind the stem convolution (ARAB2001: always)
    int policy_bias;     // 1: the last policy convolution has a bias (ARAB2001: never)
};

// Precision float32: one bottleneck block as separate launches on fp32 activations (net.cu, conv_gemm.cuh)
struct PreciseBlock {
    float *se_w1t = nullptr, *se_w2t = nullptr, *se_b = nullptr, *se_b1 = nullptr;
    __half *w1 = nullptr, *w2 = nullptr;  // operand-split weights [rows][3 * cw] per tap: hi | lo | hi
    float *b1 = nullptr, *wd = nullptr, *bd = nullptr, *b2 = nullptr;
    ConvLayer conv1, conv2;
};

// the tensors of a weight blob, host side, in blob order (weights.py)
struct HostBlock {
    std::vector<float> se_a, se_b;  // ca_se: fc1 [128][256], fc2 [256][128]; eca_se: centre tap [256][256], bias [256]
    std::vector<float> se_b1, se_b2;  // ca_se with kBlobSeBias: fc1 bias [128], fc2 bias [256]
    std::vector<float> w1, b1, wd, bd, w2, b2;
};
struct HostWeights {
    std::vector<float> stem_w, stem_b;
    std::vector<HostBlock> blocks;
    std::vector<float> vh_wv, vh_bv, vh_a, vh_ab, vh_b, vh_bb;  // standard: fc1 / b1 / fc2 / b2; WDL: wdl w / b, plys w / b
    std::vector<float> pol_w1, pol_b1, pol_w2, pol_b2;  // pol_b2: [policy_channels] when hdr.policy_bias
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
    // The stem convolution alone, into the stem-output buffer of input / output set `io` (Precision float16 with two
    // sets enabled): a search with two logical threads runs it on its tree stream right behind the plane encoding, which
    // takes it off the network stream's critical path.
    int stem_device(int n, cudaStream_t stream, const int* boards_dev, int io);
    bool stem_splittable() const { return precision == 0 && d_x0_alt != nullptr; }
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
    int n_labels() const { return hdr.policy_channels * 64; }
    int n_aux() const { return hdr.wdl_mode ? 4 : 0; }
    int kernels_per_forward(bool from_f32) const;
    int trunk_cycles(unsigned long long* out32);  // -DARA_TRUNK_PROF builds: per-role cycle counters of CTA 0
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
    int upload_value_head(const HostWeights& hw);
    int upload_policy_bias(const HostWeights& hw, int rows);
    int enqueue_precise(int n, cudaStream_t s, bool from_f32, const int* boards_dev, int io);
    int launch_graph(int family, int n, cudaStream_t s, bool from_f32, const int* boards_dev, int io, bool stem_done);
    DeviceBuffers mem_;
    int max_cop_ = 0;
    __half* stem_w = nullptr;
    float* stem_b = nullptr;
    ConvLayer stem_conv;
    ConvLayer stem_conv2;  // the stem reading the second input set
    std::vector<PreciseBlock> pb_;
    RiseTrunk trunk_;
    float *vh_wv = nullptr, *vh_bv = nullptr, *vh_w1t = nullptr, *vh_b1 = nullptr, *vh_w2 = nullptr, *vh_b2 = nullptr;
    float *vh_wdl_w = nullptr, *vh_wdl_b = nullptr, *vh_plys_w = nullptr, *vh_plys_b = nullptr;
    __half *pol_w1 = nullptr, *pol_w2 = nullptr;
    float *pol_b1 = nullptr, *pol_b2 = nullptr;
    ConvLayer pol_conv1, pol_conv2;
    std::map<int, cudaGraphExec_t> graphs_[6];  // plain, from fp32 input, with a device-side count (io 0), the same for io 1
    const int* baked_[6] = {};                  // the counter pointer each graph family was captured with
    int upload_conv_w(const float* w, int n_out, int cin, int ksize, __half** dst, int* rows);
    int upload_conv_w_split(const float* w, int n_out, int cin, int ksize, __half** dst, int* rows);
    int upload_f32(const float* src, size_t count, size_t padded, float** dst);
};

}  // namespace ara
