// Batched rules / plane kernels over arrays of 128-byte boards: one warp per board.
//   encode_planes_*  : a1 of the hot path (board -> input planes), pure HBM-bound streaming kernel
//   legal_moves      : device move generator exposed for parity tests and batched expansion
//   do_move          : apply one move per board
// C-ABI wrappers take HOST buffers (copies inside) or DEVICE buffers (the *_device variants used by bench.py).
#include <vector>

#include "abi_common.h"
#include "ara_b200.h"
#include "chess_host.h"
#include "planes_dev.cuh"

namespace ara {

constexpr int kWarpsPerBlock = 4;

__global__ void __launch_bounds__(32 * kWarpsPerBlock)
encode_planes_f32_kernel(const Board* boards, int n, int mode, int version, int normalize, float* out, int channels) {
    __shared__ Board sb[kWarpsPerBlock];
    const int w = threadIdx.x >> 5;
    const int i = blockIdx.x * kWarpsPerBlock + w;
    if (i >= n) return;
    if (ARA_LANE < 8) reinterpret_cast<uint4*>(&sb[w])[ARA_LANE] = reinterpret_cast<const uint4*>(&boards[i])[ARA_LANE];
    __syncwarp();
    encode_planes_nchw_f32(sb[w], mode, version, normalize != 0, out + static_cast<size_t>(i) * channels * 64);
}

__global__ void __launch_bounds__(32 * kWarpsPerBlock)
encode_planes_f16_kernel(const Board* boards, int n, int mode, int version, __half* out, int cpad) {
    __shared__ Board sb[kWarpsPerBlock];
    const int w = threadIdx.x >> 5;
    const int i = blockIdx.x * kWarpsPerBlock + w;
    if (i >= n) return;
    if (ARA_LANE < 8) reinterpret_cast<uint4*>(&sb[w])[ARA_LANE] = reinterpret_cast<const uint4*>(&boards[i])[ARA_LANE];
    __syncwarp();
    encode_planes_nhwc_f16(sb[w], mode, version, out + static_cast<size_t>(i) * 64 * cpad, cpad);
}

__global__ void __launch_bounds__(32 * kWarpsPerBlock)
legal_moves_kernel(const Board* boards, int n, Move* moves_out, int* counts, int* terminal, int* policy_idx) {
    __shared__ Board sb[kWarpsPerBlock];
    __shared__ Move scratch[kWarpsPerBlock][kMaxMoves];
    __shared__ MoveGenScratch mg[kWarpsPerBlock];
    const int w = threadIdx.x >> 5;
    const int i = blockIdx.x * kWarpsPerBlock + w;
    if (i >= n) return;
    if (ARA_LANE < 8) reinterpret_cast<uint4*>(&sb[w])[ARA_LANE] = reinterpret_cast<const uint4*>(&boards[i])[ARA_LANE];
    __syncwarp();
    Move* out = moves_out + static_cast<size_t>(i) * kMaxMoves;
    const int cnt = gen_legal(sb[w], mg[w], scratch[w], out);
    const bool checked = mg[w].checked != 0;
    if (policy_idx != nullptr)
        for (int k = ARA_LANE; k < cnt; k += 32)
            policy_idx[static_cast<size_t>(i) * kMaxMoves + k] = policy_map_index(out[k], sb[w].stm, sb[w].chess960);
    if (ARA_LANE == 0) {
        counts[i] = cnt;
        if (terminal != nullptr) terminal[i] = terminal_type(sb[w], cnt, checked);
    }
}

static int check_device() {
    int dev = 0;
    ARA_CUDA_OK(cudaGetDevice(&dev));
    cudaDeviceProp prop;
    ARA_CUDA_OK(cudaGetDeviceProperties(&prop, dev));
    if (prop.major != 9 || prop.minor != 0) return set_error("this library only runs on sm_90a (H100); device %d is sm_%d%d", dev, prop.major, prop.minor);
    return 0;
}

}  // namespace ara

using namespace ara;

// ---- host-side board helpers (control plane: FEN, UCI strings, game history) -----------------------------------
extern "C" int ara_board_from_fen(const char* fen, int variant, int is960, ara_board_t* out) {
    if (fen == nullptr || out == nullptr) return set_error("ara_board_from_fen: null argument");
    if (variant < 0 || variant > V_THREECHECK) return set_error("ara_board_from_fen: unsupported variant %d", variant);
    Board b;
    if (!board_from_fen(&b, fen, variant, is960)) return set_error("ara_board_from_fen: cannot parse '%s'", fen);
    memcpy(out, &b, sizeof(b));
    return 0;
}
extern "C" int ara_board_to_fen(const ara_board_t* board, char* buf, int buf_len) {
    Board b;
    memcpy(&b, board, sizeof(b));
    const std::string s = board_to_fen(b);
    if (static_cast<int>(s.size()) + 1 > buf_len) return set_error("ara_board_to_fen: buffer too small");
    memcpy(buf, s.c_str(), s.size() + 1);
    return 0;
}
extern "C" int ara_move_to_uci(unsigned short move, int is960, char* buf8) {
    const std::string s = move_to_uci(move, is960 != 0);
    memcpy(buf8, s.c_str(), s.size() + 1);
    return 0;
}

// ---- GPU kernels through host buffers ----------------------------------------------------------------------------
extern "C" int ara_encode_planes(const ara_board_t* boards, int n, int mode, int version, int normalize, float* planes_out) {
    if (check_device()) return -1;
    const int c = planes_channels(mode, version);
    if (c < 0) return set_error("ara_encode_planes: unsupported mode %d / version %d", mode, version);
    if (n <= 0) return 0;
    DeviceBuffers mem;
    Board* d_b = nullptr;
    float* d_o = nullptr;
    if (mem.dalloc(&d_b, n) || mem.dalloc(&d_o, static_cast<size_t>(n) * c * 64)) return -1;
    ARA_CUDA_OK(cudaMemcpy(d_b, boards, sizeof(Board) * n, cudaMemcpyHostToDevice));
    encode_planes_f32_kernel<<<(n + kWarpsPerBlock - 1) / kWarpsPerBlock, 32 * kWarpsPerBlock>>>(d_b, n, mode, version, normalize, d_o, c);
    ARA_CUDA_OK(cudaMemcpy(planes_out, d_o, sizeof(float) * n * c * 64, cudaMemcpyDeviceToHost));
    return 0;
}

extern "C" int ara_encode_planes_device(const void* boards_dev, int n, int mode, int version, int normalize, float* planes_dev,
                                        void* planes_half_nhwc_dev, int cpad, void* stream) {
    const int c = planes_channels(mode, version);
    if (c < 0) return set_error("ara_encode_planes_device: unsupported mode %d / version %d", mode, version);
    const int grid = (n + kWarpsPerBlock - 1) / kWarpsPerBlock;
    if (planes_dev != nullptr)
        encode_planes_f32_kernel<<<grid, 32 * kWarpsPerBlock, 0, (cudaStream_t)stream>>>((const Board*)boards_dev, n, mode, version, normalize, planes_dev, c);
    if (planes_half_nhwc_dev != nullptr) {
        if (cpad < c || (cpad != 64 && cpad != 128)) return set_error("ara_encode_planes_device: cpad %d must be 64 or 128", cpad);
        encode_planes_f16_kernel<<<grid, 32 * kWarpsPerBlock, 0, (cudaStream_t)stream>>>((const Board*)boards_dev, n, mode, version, (__half*)planes_half_nhwc_dev, cpad);
    }
    ARA_CUDA_OK(cudaGetLastError());
    return 0;
}

extern "C" int ara_legal_moves(const ara_board_t* boards, int n, unsigned short* moves_out, int* counts, int* terminal,
                               int* policy_idx) {
    if (check_device()) return -1;
    if (n <= 0) return 0;
    DeviceBuffers mem;
    Board* d_b = nullptr;
    Move* d_m = nullptr;
    int *d_c = nullptr, *d_t = nullptr, *d_p = nullptr;
    if (mem.dalloc(&d_b, n) || mem.dalloc(&d_m, static_cast<size_t>(n) * kMaxMoves) || mem.dalloc(&d_c, n) || mem.dalloc(&d_t, n) ||
        mem.dalloc(&d_p, static_cast<size_t>(n) * kMaxMoves))
        return -1;
    ARA_CUDA_OK(cudaMemcpy(d_b, boards, sizeof(Board) * n, cudaMemcpyHostToDevice));
    legal_moves_kernel<<<(n + kWarpsPerBlock - 1) / kWarpsPerBlock, 32 * kWarpsPerBlock>>>(d_b, n, d_m, d_c, d_t, d_p);
    ARA_CUDA_OK(cudaMemcpy(moves_out, d_m, sizeof(Move) * n * kMaxMoves, cudaMemcpyDeviceToHost));
    ARA_CUDA_OK(cudaMemcpy(counts, d_c, sizeof(int) * n, cudaMemcpyDeviceToHost));
    if (terminal) ARA_CUDA_OK(cudaMemcpy(terminal, d_t, sizeof(int) * n, cudaMemcpyDeviceToHost));
    if (policy_idx) ARA_CUDA_OK(cudaMemcpy(policy_idx, d_p, sizeof(int) * n * kMaxMoves, cudaMemcpyDeviceToHost));
    return 0;
}
