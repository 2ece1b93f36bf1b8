// CUDA-core kernels of the RISE forward pass that surround the wgmma GEMMs: layout conversion, value head, policy
// softmax; for Precision float32 also depthwise convolution and squeeze-excitation (in Precision float16 those live
// inside the persistent tower kernel, rise_trunk.cuh).  Activations are NHWC ([board*64+sq, C]).
// Reference semantics: DeepCrazyhouse/src/domain/neural_net/architectures/pytorch/builder_util.py
//   _ChannelAttentionModule :83-114, _EfficientChannelAttentionModule :49-80, _ValueHead :246-326,
//   _BottlekneckResidualBlock :437-475 (depthwise conv + BN + ReLU), softmax appended by the backend
//   (engine/src/nn/tensorrtapi.cpp:378-380).
#pragma once
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "sm90_prims.cuh"

namespace ara {

// ---------------------------------------------------------------------------------------------
// [n, C, 64] fp32 (reference NCHW planes) -> [n, 64, cpad] fp16 (zero padded channels).  One CTA per board.
__global__ void nchw_f32_to_nhwc_f16_kernel(const float* __restrict__ in, __half* __restrict__ out, int C, int cpad) {
    extern __shared__ float s_planes[];  // [C][65]
    pdl_wait();
    pdl_launch_dependents();
    const int b = blockIdx.x;
    const float* src = in + static_cast<size_t>(b) * C * 64;
    for (int i = threadIdx.x; i < C * 64; i += blockDim.x) {
        const int c = i >> 6, sq = i & 63;
        s_planes[c * 65 + sq] = src[i];
    }
    __syncthreads();
    __half* dst = out + static_cast<size_t>(b) * 64 * cpad;
    for (int i = threadIdx.x; i < 64 * cpad; i += blockDim.x) {
        const int sq = i / cpad, c = i - sq * cpad;
        dst[i] = __float2half_rn(c < C ? s_planes[c * 65 + sq] : 0.0f);
    }
}

// =============================================================================================
// Precision float32 (the reference's `Precision float32`): fp32 activations between the layers; every tensor that feeds
// a wgmma GEMM is ALSO stored split as fp16 [hi | hi | lo] with the channel pitch cs (conv_gemm.cuh).  The CUDA-core
// stages below read / write fp32.
__device__ __forceinline__ void store_split(__half* row3, int cs, int c, float v) {
    const __half hi = __float2half_rn(v);
    row3[c] = hi;
    row3[cs + c] = hi;
    row3[2 * cs + c] = __float2half_rn(v - __half2float(hi));
}

// [n, C, 64] fp32 planes -> [n, 64, 3 * cpad] fp16 split (zero padded channels).  One CTA per board.
__global__ void nchw_f32_to_nhwc_split_kernel(const float* __restrict__ in, __half* __restrict__ out, int C, int cpad) {
    extern __shared__ float s_planes[];  // [C][65]
    pdl_wait();
    pdl_launch_dependents();
    const int b = blockIdx.x;
    const float* src = in + static_cast<size_t>(b) * C * 64;
    for (int i = threadIdx.x; i < C * 64; i += blockDim.x) {
        const int c = i >> 6, sq = i & 63;
        s_planes[c * 65 + sq] = src[i];
    }
    __syncthreads();
    __half* dst = out + static_cast<size_t>(b) * 64 * 3 * cpad;
    for (int i = threadIdx.x; i < 64 * cpad; i += blockDim.x) {
        const int sq = i / cpad, c = i - sq * cpad;
        store_split(dst + static_cast<size_t>(sq) * 3 * cpad, cpad, c, c < C ? s_planes[c * 65 + sq] : 0.0f);
    }
}

// Depthwise KxK convolution (pad K/2) + bias + ReLU (builder_util.py:437-475, BN folded).  in: [boards*64, C] fp32,
// w: [K*K][C] fp32, bias: [C] fp32, out: split [boards*64, 3*cs] (channels C..cs-1 stay zero).  One thread = one
// channel of one square, channel fastest.
template <int K>
__global__ void dwconv_f32_kernel(const float* __restrict__ in, const float* __restrict__ w, const float* __restrict__ bias,
                                  __half* __restrict__ out, int boards, int C, int cs) {
    pdl_wait();
    pdl_launch_dependents();
    const long long total = static_cast<long long>(boards) * 64 * C;
    const long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (idx >= total) return;
    const int c = static_cast<int>(idx % C);
    const long long row = idx / C;
    const int sq = static_cast<int>(row & 63);
    const long long b = row >> 6;
    const int y = sq >> 3, x = sq & 7;
    float acc = __ldg(bias + c);
    constexpr int R = K / 2;
#pragma unroll
    for (int dy = -R; dy <= R; ++dy) {
        const int yy = y + dy;
        if (yy < 0 || yy > 7) continue;
#pragma unroll
        for (int dx = -R; dx <= R; ++dx) {
            const int xx = x + dx;
            if (xx < 0 || xx > 7) continue;
            acc = fmaf(__ldg(in + ((b << 6) + yy * 8 + xx) * C + c), __ldg(w + ((dy + R) * K + (dx + R)) * C + c), acc);
        }
    }
    store_split(out + row * 3 * cs, cs, c, fmaxf(acc, 0.0f));
}

// Squeeze-excitation on the 256-channel trunk (builder_util.py:49-114), fp32 in place + the split copy.  One CTA (256
// threads) per board.
//   mode 1 ("ca_se"):  s = gate(W2 * relu(W1 * mean + b1) + b)      W1t: [256][128], W2t: [128][256] (transposed)
//   mode 2 ("eca_se"): s = gate(Wc * mean + b)                      W1t: [256][256] centre tap transposed, b: [256]
// b1, b (ca_se): the MXNet symbols' fully-connected biases, or null.  gate: kTrunkGate* (rise_trunk_args.h).
// keep_x: the block's shortcut is its input before the squeeze-excitation (MXNet symbols), so only the split copy, which
// the block's first convolution reads, is scaled and x stays as it is.
__device__ __forceinline__ float hard_sigmoid(float x) { return fminf(fmaxf(x * (1.0f / 6.0f) + 0.5f, 0.0f), 1.0f); }
__device__ __forceinline__ float se_gate(float x, int gate) {
    if (gate == 0) return hard_sigmoid(x);
    if (gate == 1) return fminf(fmaxf(x * 0.2f + 0.5f, 0.0f), 1.0f);
    return 1.0f / (1.0f + expf(-x));
}

__global__ void __launch_bounds__(256) se_f32_kernel(float* __restrict__ x, __half* __restrict__ xs,
                                                       const float* __restrict__ w1t, const float* __restrict__ w2t,
                                                       const float* __restrict__ bias, const float* __restrict__ b1, int mode,
                                                       int gate, int keep_x) {
    __shared__ float s_pool[256];
    __shared__ float s_hid[128];
    pdl_wait();
    pdl_launch_dependents();
    const int b = blockIdx.x;
    const int c = threadIdx.x;
    float* xb = x + static_cast<size_t>(b) * 64 * 256;
    __half* sb = xs + static_cast<size_t>(b) * 64 * 768;
    float sum = 0.0f;
#pragma unroll 8
    for (int sq = 0; sq < 64; ++sq) sum += xb[sq * 256 + c];
    s_pool[c] = sum * (1.0f / 64.0f);
    __syncthreads();
    float scale;
    if (mode == 1) {
        if (c < 128) {
            float h = b1 != nullptr ? __ldg(b1 + c) : 0.0f;
            for (int k = 0; k < 256; ++k) h = fmaf(__ldg(w1t + k * 128 + c), s_pool[k], h);
            s_hid[c] = fmaxf(h, 0.0f);
        }
        __syncthreads();
        float o = bias != nullptr ? __ldg(bias + c) : 0.0f;
        for (int j = 0; j < 128; ++j) o = fmaf(__ldg(w2t + j * 256 + c), s_hid[j], o);
        scale = se_gate(o, gate);
    } else {
        float o = __ldg(bias + c);
        for (int k = 0; k < 256; ++k) o = fmaf(__ldg(w1t + k * 256 + c), s_pool[k], o);
        scale = se_gate(o, gate);
    }
#pragma unroll 8
    for (int sq = 0; sq < 64; ++sq) {
        const float v = xb[sq * 256 + c] * scale;
        if (!keep_x) xb[sq * 256 + c] = v;
        store_split(sb + sq * 768, 256, c, v);
    }
}

// ---------------------------------------------------------------------------------------------
// Value head.  One CTA (256 threads) per board.  The kinds (wdl_mode, net.h kValueHead*):
//   f[j*64+sq] = relu(sum_c x[sq][c] * wv[j][c] + bv[j])            (conv1x1 256->8 + BN folded, NCHW flatten)
//   0 standard:  value = tanh(w2 . relu(W1 f + b1) + b2)             W1t: [512][256] (transposed)
//   1 wdl+plys:  wdl = Ww f + bw (3), plys = sigmoid(wp . f + bp); value = -softmax(wdl)[0] + softmax(wdl)[2];
//                aux = [wdl0, wdl1, wdl2, plys] (the logits, as the PyTorch network outputs them)
//   2 as 1, value = tanh(m1 . relu(M0 [wdl logits, plys] + c0) + c1)  (use_mlp_wdl_ply: M0 [8][4], m1 [8]); aux as 1
//   3 MXNet:     g = relu(W1 f + b1) (value_fc0, zero-padded to 256 units, W1t as the standard head's), then 1 on g
//                (Ww [3][256], wp [256]); aux = [softmax(wdl), plys] (the probabilities SoftmaxOutput outputs)
//   4 as 3, value = the MLP of 2 on [softmax(wdl), plys]; aux as 3
// Every kind's arithmetic after the convolution is fp32 and per board.
struct ValueHeadW {
    const float* wv;   // [8][256]
    const float* bv;   // [8]
    const float* w1t;  // [512][256]
    const float* b1;   // [256]
    const float* w2;   // [256]
    const float* b2;   // [1]
    const float* wdl_w;   // [3][512] (kinds 3 / 4: [3][256])
    const float* wdl_b;   // [3]
    const float* plys_w;  // [512] (kinds 3 / 4: [256])
    const float* plys_b;  // [1]
    const float* mlp;     // kinds 2 / 4: M0 [8][4] | c0 [8] | m1 [8] | c1 [1]
    int wdl_mode;
};

__device__ __forceinline__ float act_to_float(__half v) { return __half2float(v); }
__device__ __forceinline__ float act_to_float(float v) { return v; }

// relu(W1 f + b1) of thread t's unit: 512 L2-resident weight loads per thread, four independent chains, 16 loads in flight
__device__ __forceinline__ float value_hidden_unit(const float* __restrict__ w1t, const float* __restrict__ b1, const float* f,
                                                   int t) {
    float h0 = __ldg(b1 + t), h1 = 0.0f, h2 = 0.0f, h3 = 0.0f;
    const float* wp = w1t + t;
#pragma unroll 4
    for (int i = 0; i < 512; i += 4) {
        h0 = fmaf(__ldg(wp + (i + 0) * 256), f[i + 0], h0);
        h1 = fmaf(__ldg(wp + (i + 1) * 256), f[i + 1], h1);
        h2 = fmaf(__ldg(wp + (i + 2) * 256), f[i + 2], h2);
        h3 = fmaf(__ldg(wp + (i + 3) * 256), f[i + 3], h3);
    }
    const float h = (h0 + h1) + (h2 + h3);
    return fmaxf(h, 0.0f);
}

// Kinds 2, 3 and 4 from the four outputs s_red (WDL logits, plies logit): *value and aux[0 .. 4).  Not inlined, so that
// kind 1's code in the kernel, and with it its floating-point contractions, stays as it was.
__device__ __noinline__ void value_wdl_finish(const float* s_red, int mode, const float* __restrict__ mlp, float* value,
                                              float* aux) {
    const float l0 = s_red[0], l1 = s_red[1], l2 = s_red[2];
    const float m = fmaxf(l0, fmaxf(l1, l2));
    const float e0 = expf(l0 - m), e1 = expf(l1 - m), e2 = expf(l2 - m);
    const float inv = 1.0f / (e0 + e1 + e2);
    const float plys = 1.0f / (1.0f + expf(-s_red[3]));
    // what the network outputs as its WDL: PyTorch the logits, MXNet the SoftmaxOutput's probabilities
    const bool mx = mode >= 3;
    const float o0 = mx ? e0 * inv : l0, o1 = mx ? e1 * inv : l1, o2 = mx ? e2 * inv : l2;
    if (mode == 3) {
        *value = -e0 * inv + e2 * inv;
    } else {  // the value MLP on (WDL, plies): 4 -> 8, ReLU, 8 -> 1, tanh
        float v = __ldg(mlp + 48);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            float h = __ldg(mlp + 32 + j);
            h = fmaf(__ldg(mlp + j * 4 + 0), o0, h);
            h = fmaf(__ldg(mlp + j * 4 + 1), o1, h);
            h = fmaf(__ldg(mlp + j * 4 + 2), o2, h);
            h = fmaf(__ldg(mlp + j * 4 + 3), plys, h);
            v = fmaf(__ldg(mlp + 40 + j), fmaxf(h, 0.0f), v);
        }
        *value = tanhf(v);
    }
    if (aux != nullptr) {
        aux[0] = o0;
        aux[1] = o1;
        aux[2] = o2;
        aux[3] = plys;
    }
}

template <typename T>  // T = __half (Precision float16) or float (Precision float32)
__global__ void __launch_bounds__(256) value_head_kernel(const T* __restrict__ x, ValueHeadW w,
                                                           float* __restrict__ value, float* __restrict__ aux,
                                                           const int* __restrict__ boards_dev) {
    if (boards_dev != nullptr && static_cast<int>(blockIdx.x) >= *boards_dev) return;  // row without input
    constexpr int kPitch = 256 + 16 / static_cast<int>(sizeof(T));  // padded rows
    extern __shared__ __align__(16) uint8_t s_x_raw[];
    T* s_x = reinterpret_cast<T*>(s_x_raw);
    __shared__ float s_wv[8 * 256];  // (kinds 3 / 4: then the hidden units g)
    __shared__ float s_f[512];
    __shared__ float s_red[8];
    pdl_wait();
    pdl_launch_dependents();
    const int b = blockIdx.x;
    const int t = threadIdx.x;
    const T* xb = x + static_cast<size_t>(b) * 64 * 256;
    constexpr int kVec = 16 / static_cast<int>(sizeof(T));  // elements per 16-byte vector
    constexpr int kVecRow = 256 / kVec;
    for (int i = t; i < 64 * kVecRow; i += 256) {
        const int sq = i / kVecRow, v = i - sq * kVecRow;
        *reinterpret_cast<uint4*>(&s_x[sq * kPitch + v * kVec]) = __ldg(reinterpret_cast<const uint4*>(xb + sq * 256 + v * kVec));
    }
    for (int i = t; i < 8 * 256; i += 256) s_wv[i] = __ldg(w.wv + i);
    __syncthreads();
    for (int o = t; o < 512; o += 256) {
        const int j = o >> 6, sq = o & 63;
        float acc = __ldg(w.bv + j);
        const T* xr = &s_x[sq * kPitch];
        const float* wr = &s_wv[j * 256];
#pragma unroll 8
        for (int c = 0; c < 256; ++c) acc = fmaf(act_to_float(xr[c]), wr[c], acc);
        s_f[o] = fmaxf(acc, 0.0f);
    }
    __syncthreads();
    const int warp = t >> 5, lane = t & 31;
    const int mode = w.wdl_mode;
    if (!mode) {
        float h = value_hidden_unit(w.w1t, w.b1, s_f, t) * __ldg(w.w2 + t);
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) h += __shfl_xor_sync(0xffffffffu, h, off);
        if (lane == 0) s_red[warp] = h;
        __syncthreads();
        if (t == 0) {
            float s = __ldg(w.b2);
            for (int i = 0; i < 8; ++i) s += s_red[i];
            value[b] = tanhf(s);
        }
    } else {
        const bool mx = mode >= 3;
        const float* feat = s_f;
        int nf = 512;
        if (mx) {  // s_wv is free: every thread is past the convolution
            s_wv[t] = value_hidden_unit(w.w1t, w.b1, s_f, t);
            __syncthreads();
            feat = s_wv;
            nf = 256;
        }
        // warps 0..3 each reduce one dot product over the features
        if (warp < 4) {
            const float* wr = (warp < 3) ? (w.wdl_w + warp * nf) : w.plys_w;
            float s = 0.0f;
            for (int i = lane; i < nf; i += 32) s = fmaf(__ldg(wr + i), feat[i], s);
#pragma unroll
            for (int off = 16; off > 0; off >>= 1) s += __shfl_xor_sync(0xffffffffu, s, off);
            if (lane == 0) s_red[warp] = s + ((warp < 3) ? __ldg(w.wdl_b + warp) : __ldg(w.plys_b));
        }
        __syncthreads();
        if (t == 0) {
            if (mode == 1) {
                const float l0 = s_red[0], l1 = s_red[1], l2 = s_red[2];
                const float m = fmaxf(l0, fmaxf(l1, l2));
                const float e0 = expf(l0 - m), e1 = expf(l1 - m), e2 = expf(l2 - m);
                const float inv = 1.0f / (e0 + e1 + e2);
                value[b] = -e0 * inv + e2 * inv;
                if (aux != nullptr) {
                    aux[b * 4 + 0] = l0;
                    aux[b * 4 + 1] = l1;
                    aux[b * 4 + 2] = l2;
                    aux[b * 4 + 3] = 1.0f / (1.0f + expf(-s_red[3]));
                }
            } else {
                value_wdl_finish(s_red, mode, w.mlp, value + b, aux != nullptr ? aux + b * 4 : nullptr);
            }
        }
    }
}

template <typename T>
constexpr int value_head_smem() { return 64 * (256 + 16 / static_cast<int>(sizeof(T))) * static_cast<int>(sizeof(T)); }

// ---------------------------------------------------------------------------------------------
// The softmax of the policy heads over one board's L logits staged in shared memory (s_l, overwritten), mx their maximum
// as this thread saw it; writes prob[0 .. L).  One CTA of 256 threads.
__device__ __forceinline__ void block_softmax_256(float* s_l, int L, float mx, float* __restrict__ prob, float* s_red, float* s_bcast) {
    const int t = threadIdx.x;
    const int warp = t >> 5, lane = t & 31;
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, off));
    if (lane == 0) s_red[warp] = mx;
    __syncthreads();
    if (t == 0) {
        float m = s_red[0];
        for (int i = 1; i < 8; ++i) m = fmaxf(m, s_red[i]);
        *s_bcast = m;
    }
    __syncthreads();
    mx = *s_bcast;
    float sum = 0.0f;
    for (int i = t; i < L; i += 256) {
        const float e = expf(s_l[i] - mx);
        s_l[i] = e;
        sum += e;
    }
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, off);
    __syncthreads();
    if (lane == 0) s_red[warp] = sum;
    __syncthreads();
    if (t == 0) {
        float s = 0.0f;
        for (int i = 0; i < 8; ++i) s += s_red[i];
        *s_bcast = 1.0f / s;
    }
    __syncthreads();
    const float inv = *s_bcast;
    for (int i = t; i < L; i += 256) prob[i] = s_l[i] * inv;
}

// Policy softmax over all P*64 logits of a board (illegal moves included, as the reference backend does).
// logits: [boards*64, ldp] fp32 (NHWC, channel = policy plane), prob: [boards, P*64] fp32 with index ch*64+sq
// (the reference's NCHW flatten, builder_util.py:229).  One CTA (256 threads) per board.
__global__ void __launch_bounds__(256) policy_softmax_kernel(const float* __restrict__ logits, float* __restrict__ prob,
                                                               int P, int ldp, const int* __restrict__ boards_dev) {
    extern __shared__ float s_l[];  // [P*64] in output order
    __shared__ float s_red[8];
    __shared__ float s_bcast;
    if (boards_dev != nullptr && static_cast<int>(blockIdx.x) >= *boards_dev) return;  // row without input
    pdl_wait();
    pdl_launch_dependents();
    const int b = blockIdx.x;
    const int t = threadIdx.x;
    const int L = P * 64;
    const float* lb = logits + static_cast<size_t>(b) * 64 * ldp;
    float mx = -INFINITY;
    for (int i = t; i < 64 * P; i += 256) {
        const int sq = i / P, ch = i - sq * P;
        const float v = __ldg(lb + sq * ldp + ch);
        s_l[ch * 64 + sq] = v;
        mx = fmaxf(mx, v);
    }
    block_softmax_256(s_l, L, mx, prob + static_cast<size_t>(b) * L, s_red, &s_bcast);
}

// logits[b, l] = b_fc[l] + part[0][b][l] + part[1][b][l] + ... (split order), then the softmax over the L labels into
// prob [boards, L].  One CTA (256 threads) per board.
__global__ void __launch_bounds__(256) policy_fc_softmax_kernel(const float* __restrict__ part, const float* __restrict__ bias,
                                                                  float* __restrict__ prob, int L, int lp, int splits, int rows_cap,
                                                                  const int* __restrict__ boards_dev) {
    extern __shared__ float s_l[];  // [L]
    __shared__ float s_red[8];
    __shared__ float s_bcast;
    if (boards_dev != nullptr && static_cast<int>(blockIdx.x) >= *boards_dev) return;  // row without input
    pdl_wait();
    pdl_launch_dependents();
    const int b = blockIdx.x;
    float mx = -INFINITY;
    for (int i = threadIdx.x; i < L; i += 256) {
        float v = __ldg(bias + i);
        for (int s = 0; s < splits; ++s) v += part[(static_cast<size_t>(s) * rows_cap + b) * lp + i];
        s_l[i] = v;
        mx = fmaxf(mx, v);
    }
    block_softmax_256(s_l, L, mx, prob + static_cast<size_t>(b) * L, s_red, &s_bcast);
}

// Node::set_probabilities_for_moves (node.cpp:961-979) for a whole batch: out[b][i] = prob[b][idx[b][i]], i < counts[b].
// One CTA per position.
__global__ void gather_priors_kernel(const float* __restrict__ prob, int n_labels, const int* __restrict__ idx,
                                     const int* __restrict__ counts, int stride, float* __restrict__ out) {
    const int b = blockIdx.x;
    const int k = min(counts[b], stride);
    for (int i = threadIdx.x; i < k; i += blockDim.x) {
        const int j = idx[static_cast<size_t>(b) * stride + i];
        out[static_cast<size_t>(b) * stride + i] = (j >= 0 && j < n_labels) ? __ldg(prob + static_cast<size_t>(b) * n_labels + j) : 0.0f;
    }
}

}  // namespace ara
