// Test scaffolding: stand-in for the NETWORK entry points of the C-ABI (and the two GPU kernels RawNetAgent calls around
// them), pre-loaded in front of libara_b200.so next to stub_search.c so that the UCI front-end's Use_Raw_Network path can
// be exercised on a box without a GPU.  The legal moves and their policy indices are the host rules' own; the "network"
// gives every legal move the prior policy_index / 10000, so the raw move is the legal move with the largest policy index,
// and the value 0.5.  Never part of the product.
#include <cstdio>
#include <cstdlib>
#include <cstring>

#include "ara_b200.h"
#include "chess_host.h"
#include "planes_dev.cuh"

using namespace ara;

namespace {
void log_line(const char* line) {  // ARA_STUB_LOG=<file>: one line per call of interest, as stub_search.c writes them
    const char* path = getenv("ARA_STUB_LOG");
    if (!path) return;
    FILE* f = fopen(path, "a");
    if (!f) return;
    fprintf(f, "%s\n", line);
    fclose(f);
}
}  // namespace

extern "C" {

ara_net_t ara_net_create(const char*, int, int, int) { return reinterpret_cast<ara_net_t>(0x2); }
void ara_net_destroy(ara_net_t) {}
int ara_net_shape(ara_net_t, int* in_channels, int* n_labels, int* n_aux, int* is_policy_map, int* input_version, int* batch_size) {
    *in_channels = 80, *n_labels = 5184, *n_aux = 0, *is_policy_map = 1, *input_version = 1, *batch_size = 1;
    return 0;
}
int ara_encode_planes(const ara_board_t*, int n, int mode, int version, int, float* planes_out) {
    const int c = planes_channels(mode, version);
    if (c < 0) return -1;
    memset(planes_out, 0, sizeof(float) * static_cast<size_t>(n) * c * 64);
    return 0;
}
int ara_legal_moves(const ara_board_t* boards, int n, unsigned short* moves_out, int* counts, int* terminal, int* policy_idx) {
    for (int i = 0; i < n; ++i) {
        Board b;
        memcpy(&b, &boards[i], sizeof(b));
        const std::vector<Move> mv = legal_moves_host(b);
        counts[i] = static_cast<int>(mv.size());
        for (size_t k = 0; k < mv.size(); ++k) {
            moves_out[static_cast<size_t>(i) * kMaxMoves + k] = mv[k];
            if (policy_idx) policy_idx[static_cast<size_t>(i) * kMaxMoves + k] = policy_map_index(mv[k], b.stm, b.chess960);
        }
        if (terminal) terminal[i] = 4;
    }
    return 0;
}
int ara_net_predict_priors(ara_net_t, const float*, int n, const int* policy_idx, const int* counts, int stride, float* value,
                           float* priors_out, float*) {
    for (int i = 0; i < n; ++i) {
        value[i] = 0.5f;
        for (int k = 0; k < counts[i]; ++k)
            priors_out[static_cast<size_t>(i) * stride + k] = policy_idx[static_cast<size_t>(i) * stride + k] / 10000.0f;
        char line[64];
        snprintf(line, sizeof(line), "predict_priors n=%d count=%d", n, counts[i]);
        log_line(line);
    }
    return 0;
}
}
