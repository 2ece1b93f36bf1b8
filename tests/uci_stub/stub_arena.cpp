// Test scaffolding: stand-in for the SEARCH and NETWORK entry points of the C-ABI that `ara_uci arena` calls, pre-loaded in
// front of libara_b200.so so that the arena's host logic (game pairs, colours, idle trees, move sampling, tree reuse,
// PGN, result) can be checked against crazyara_b200.match.Match on a box without a GPU.  The "search" of a tree is a
// deterministic function of its root: the legal moves of the host rules (chess_dev.cuh compiled as host code), each with
// the weight 1 + hash(board, move) % 1000, normalised, and the heaviest (first) move as the best one.
// tests/test_arena_uci_host_logic.py holds its Python twin.  Never part of the product.
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <mutex>
#include <string>
#include <vector>

#include "ara_b200.h"
#include "chess_host.h"

using namespace ara;

namespace {
std::mutex gMutex;
int gHandles = 0;

void log_line(const std::string& line) {  // ARA_STUB_LOG=<file>: one line per call of interest
    const char* path = getenv("ARA_STUB_LOG");
    if (!path) return;
    std::lock_guard<std::mutex> lock(gMutex);
    FILE* f = fopen(path, "a");
    if (!f) return;
    fprintf(f, "%s\n", line.c_str());
    fclose(f);
}

unsigned long long mix(unsigned long long x) {
    x ^= x >> 33;
    x *= 0xff51afd7ed558ccdULL;
    x ^= x >> 33;
    return x;
}

struct Handle {
    int id = 0;
    std::vector<ara_board_t> roots;
    std::vector<int> active;
    std::vector<ara_search_result_t> results;
};
}  // namespace

struct ara_search_s : Handle {};

extern "C" {

ara_net_t ara_net_create(const char*, int, int, int) { return reinterpret_cast<ara_net_t>(0x2); }
void ara_net_destroy(ara_net_t) {}
int ara_net_shape(ara_net_t, int* in_channels, int* n_labels, int* n_aux, int* is_policy_map, int* input_version, int* batch_size) {
    *in_channels = 39, *n_labels = 4992, *n_aux = 0, *is_policy_map = 1, *input_version = 1, *batch_size = 1;
    return 0;
}

ara_search_t ara_search_create(ara_net_t, const ara_search_settings_t* s, int, int n_trees, int max_nodes) {
    ara_search_s* h = new ara_search_s;
    {
        std::lock_guard<std::mutex> lock(gMutex);
        h->id = gHandles++;
    }
    h->roots.resize(n_trees);
    h->active.assign(n_trees, 1);
    h->results.resize(n_trees);
    for (auto& r : h->results) memset(&r, 0, sizeof(r));
    log_line("create handle=" + std::to_string(h->id) + " trees=" + std::to_string(n_trees) + " max_nodes=" + std::to_string(max_nodes) +
             " seed=" + std::to_string(s->seed) + " batch_size=" + std::to_string(s->batch_size));
    return h;
}
void ara_search_destroy(ara_search_t s) { delete s; }
int ara_search_set_position(ara_search_t s, int tree, const ara_board_t* root, const unsigned long long*, const short*, int) {
    s->roots[tree] = *root;
    return 0;
}
int ara_search_set_active(ara_search_t s, int tree, int active) {
    for (int t = 0; t < static_cast<int>(s->active.size()); ++t)
        if (tree < 0 || t == tree) s->active[t] = active != 0;
    return 0;
}
int ara_search_go(ara_search_t s) {
    std::string trees;
    for (size_t t = 0; t < s->active.size(); ++t) {
        if (!s->active[t]) continue;
        trees += (trees.empty() ? "" : ",") + std::to_string(t);
        Board b;
        memcpy(&b, &s->roots[t], sizeof(b));
        unsigned long long key = 1469598103934665603ULL;  // FNV-1a over the board's 16 words
        for (int i = 0; i < 16; ++i) key = (key ^ s->roots[t].w[i]) * 1099511628211ULL;
        const std::vector<Move> moves = legal_moves_host(b);
        ara_search_result_t& r = s->results[t];
        memset(&r, 0, sizeof(r));
        r.n_moves = static_cast<int>(moves.size());
        r.best_idx = moves.empty() ? -1 : 0;
        unsigned long long sum = 0;
        std::vector<unsigned long long> w(moves.size());
        for (size_t k = 0; k < moves.size(); ++k) {
            w[k] = 1 + mix(key ^ (moves[k] * 0x9E3779B97F4A7C15ULL)) % 1000;
            sum += w[k];
            r.moves[k] = moves[k];
            if (w[k] > w[r.best_idx]) r.best_idx = static_cast<int>(k);
        }
        for (size_t k = 0; k < moves.size(); ++k) r.policy[k] = static_cast<double>(w[k]) / static_cast<double>(sum);
    }
    if (trees.empty()) return -1;  // the arena never searches a handle whose trees are all idle
    log_line("go handle=" + std::to_string(s->id) + " trees=" + trees);
    return 0;
}
int ara_search_result(ara_search_t s, int tree, ara_search_result_t* out) {
    *out = s->results[tree];
    return 0;
}
int ara_search_apply_move(ara_search_t s, int tree, unsigned short move) {
    log_line("apply_move handle=" + std::to_string(s->id) + " tree=" + std::to_string(tree) + " move=" + std::to_string(move));
    return 0;
}
}
