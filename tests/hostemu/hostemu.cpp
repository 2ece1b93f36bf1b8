// Host emulation of the DEVICE rules / plane / search code (1-lane warp) for CPU-only unit tests.
// Test scaffolding: compiled by tests/ with g++, never part of the product library.
#include <cstring>
#include <string>
#include <vector>

#include "chess_host.h"
#include "planes_dev.cuh"

using namespace ara;

struct HeState {
    Board b;
    std::vector<uint64_t> keys;
    std::vector<int16_t> reps;
};

extern "C" {

HeState* he_new(const char* fen, int variant, int is960) {
    HeState* s = new HeState();
    if (!board_from_fen(&s->b, fen, variant, is960)) {
        delete s;
        return nullptr;
    }
    return s;
}
void he_free(HeState* s) { delete s; }
HeState* he_clone(const HeState* s) { return new HeState(*s); }
int he_legal_moves(const HeState* s, uint16_t* out) {
    std::vector<Move> mv = legal_moves_host(s->b);
    for (size_t i = 0; i < mv.size(); ++i) out[i] = mv[i];
    return static_cast<int>(mv.size());
}
void he_move_uci(const HeState* s, uint16_t m, char* buf) { strcpy(buf, move_to_uci(m, s->b.chess960 != 0).c_str()); }
uint16_t he_uci_move(const HeState* s, const char* uci) { return uci_to_move(s->b, uci); }
void he_do_move(HeState* s, uint16_t m) {
    s->keys.push_back(s->b.key);
    s->reps.push_back(s->b.repetition);
    do_move(s->b, m);
    s->b.repetition = static_cast<int16_t>(
        repetition_from_history(s->b, s->keys.data(), s->reps.data(), static_cast<int>(s->keys.size())));
}
void he_fen(const HeState* s, char* buf) { strcpy(buf, board_to_fen(s->b).c_str()); }
unsigned long long he_key(const HeState* s) { return s->b.key; }
unsigned long long he_key_scratch(const HeState* s) { return compute_key(s->b); }
int he_in_check(const HeState* s) { return in_check(s->b) ? 1 : 0; }
int he_repetition(const HeState* s) { return s->b.repetition; }
int he_terminal(const HeState* s) {
    Move scratch[kMaxMoves], out[kMaxMoves];
    MoveGenScratch mg;
    const int n = gen_legal(s->b, mg, scratch, out);
    return terminal_type(s->b, n, mg.checked != 0);
}
int he_policy_index(const HeState* s, uint16_t m) { return policy_map_index(m, s->b.stm, s->b.chess960); }
int he_planes(const HeState* s, int mode, int version, int normalize, float* out) {
    const int c = planes_channels(mode, version);
    if (c < 0) return -1;
    encode_planes_nchw_f32(s->b, mode, version, normalize != 0, out);
    return c;
}
int he_sizeof_board() { return static_cast<int>(sizeof(Board)); }
const void* he_board(const HeState* s) { return &s->b; }
}

// ---------------------------------------------------------------------------------------------------------------
// 1-lane emulation of the GPU search (search_dev.cuh) with host arrays standing in for the HBM pools.
#include <cmath>

#include "search_dev.cuh"

struct HostWriterFactory {
    float* base;
    int channels;
    struct Target {
        float* out;
        void encode(const Board& b, int mode, int version) const { encode_planes_nchw_f32(b, mode, version, true, out); }
    };
    Target make(int slot) const { return Target{base + static_cast<size_t>(slot) * channels * 64}; }
};

// one mini-batch in flight (a logical search thread): its arrays, its view of the tree, its planes
struct HeBatch {
    BatchState bs;
    TreeDev t;
    std::vector<int32_t> new_node, traj_node, traj_len, traj_start, exp_parent;
    std::vector<uint16_t> traj_ci;
    std::vector<uint32_t> traj_edge;
    std::vector<float> planes;
};

struct HeSearch {
    SearchParams sp;
    TreeDev& t = batch[0].t;  // root creation, results, tree reuse go through the first view
    TreeState st;
    std::vector<NodeHdr> hdr;
    std::vector<Board> board;
    std::vector<float> P, Q;
    std::vector<uint32_t> N;
    std::vector<int32_t> child;
    std::vector<Move> move;
    std::vector<uint8_t> vl, etype;
    std::vector<uint32_t> cbase;
    std::vector<Board> prep_board;
    std::vector<int16_t> prep_ci;
    std::vector<uint8_t> prep_term;
    std::vector<uint64_t> hist_keys;
    std::vector<int16_t> hist_reps;
    std::vector<float> lut;
    std::vector<double> sqrt_lut;
    HeBatch batch[2];
    WarpScratch ws;
    int channels, n_labels;
    Board root;
    SearchResult result;
};

extern "C" {

HeSearch* he_search_new(const SearchParams* sp, int max_nodes, int max_edges) {
    HeSearch* s = new HeSearch();
    s->sp = *sp;
    const int B = sp->batch_size;
    s->hdr.resize(max_nodes);
    s->board.resize(max_nodes);
    s->P.resize(max_edges);
    s->Q.resize(max_edges);
    s->N.resize(max_edges);
    s->child.resize(max_edges);
    s->cbase.resize(max_edges);
    s->move.resize(max_edges);
    s->vl.resize(max_edges);
    s->etype.resize(max_edges);
    s->channels = planes_channels(sp->mode, sp->input_version);
    s->n_labels = policy_labels(sp->mode);
    const int lut_len = 1 << 16;
    s->lut.resize(lut_len);
    for (int i = 0; i < lut_len; ++i) s->lut[i] = logf((static_cast<float>(i) + sp->cpuct_base + 1) / sp->cpuct_base) + sp->cpuct_init;
    s->sqrt_lut.resize(lut_len);
    for (int i = 0; i < lut_len; ++i) s->sqrt_lut[i] = sqrt(static_cast<double>(i));
    memset(&s->st, 0, sizeof(s->st));
    s->st.rng = minstd_seed(sp->seed, 0);
    crand_seed(s->st.crand_r, &s->st.crand_f, static_cast<unsigned>(sp->seed));
    s->prep_board.resize(static_cast<size_t>(max_nodes) * kPrepSlots);
    s->prep_ci.assign(static_cast<size_t>(max_nodes) * kPrepSlots, -1);
    s->prep_term.resize(static_cast<size_t>(max_nodes) * kPrepSlots);
    for (HeBatch& bt : s->batch) {
        memset(&bt.bs, 0, sizeof(bt.bs));
        bt.new_node.resize(B);
        bt.traj_node.resize(2 * B * kMaxDepth);
        bt.traj_ci.resize(2 * B * kMaxDepth);
        bt.traj_len.resize(2 * B);
        bt.traj_start.assign(2 * B, 0);
        bt.traj_edge.resize(2 * B * kMaxDepth);
        bt.exp_parent.resize(3 * B);
        bt.planes.assign(static_cast<size_t>(B) * s->channels * 64, 0.0f);
        TreeDev& t = bt.t;
        t.hdr = s->hdr.data();
        t.board = s->board.data();
        t.P = s->P.data();
        t.Q = s->Q.data();
        t.N = s->N.data();
        t.child = s->child.data();
        t.cbase = s->cbase.data();
        t.move = s->move.data();
        t.vl = s->vl.data();
        t.etype = s->etype.data();
        t.st = &s->st;
        t.bs = &bt.bs;
        t.new_node = bt.new_node.data();
        t.traj_node = bt.traj_node.data();
        t.traj_ci = bt.traj_ci.data();
        t.traj_len = bt.traj_len.data();
        t.traj_start = bt.traj_start.data();
        t.traj_edge = bt.traj_edge.data();
        t.exp_parent = bt.exp_parent.data();
        t.prep_board = s->prep_board.data();
        t.prep_ci = s->prep_ci.data();
        t.prep_term = s->prep_term.data();
        t.hist_keys = nullptr;
        t.hist_reps = nullptr;
        t.hist_len = 0;
        t.cput_lut = s->lut.data();
        t.sqrt_lut = s->sqrt_lut.data();
        t.cput_lut_len = lut_len;
        t.max_nodes = max_nodes;
        t.max_edges = max_edges;
        t.slot_base = 0;
    }
    return s;
}
void he_search_free(HeSearch* s) { delete s; }
int he_search_channels(const HeSearch* s) { return s->channels; }
int he_search_n_labels(const HeSearch* s) { return s->n_labels; }
const float* he_search_planes_t(const HeSearch* s, int th) { return s->batch[th].planes.data(); }
const float* he_search_planes(const HeSearch* s) { return he_search_planes_t(s, 0); }

int he_search_set_root(HeSearch* s, const HeState* root) {
    s->root = root->b;
    s->hist_keys = root->keys;
    s->hist_reps = root->reps;
    for (HeBatch& bt : s->batch) {
        bt.t.hist_keys = s->hist_keys.data();
        bt.t.hist_reps = s->hist_reps.data();
        bt.t.hist_len = static_cast<int>(s->hist_keys.size());
        memset(&bt.bs, 0, sizeof(bt.bs));
    }
    HeBatch& b0 = s->batch[0];
    if (reuse_root(s->t, s->sp, &s->root)) return s->st.done ? 0 : 2;  // 2: the kept subtree is searched on
    create_root(s->t, s->sp, s->ws, &s->root);
    HostWriterFactory wf{b0.planes.data(), s->channels};
    for (int b = 0; b < b0.bs.n_new; ++b) {
        const auto target = wf.make(b);
        expand_pending(s->t, s->sp, s->ws, b0.new_node[b], &target);
    }
    return b0.bs.n_new;
}
void he_search_apply_move(HeSearch* s, unsigned short move) { advance_root(s->t, move); }
void he_search_root_results(HeSearch* s, const float* values, const float* probs) {
    backup_results(s->t, s->sp, values);  // (independent of the scatter step: the device runs them side by side)
    for (int b = 0; b < s->batch[0].bs.n_new; ++b) scatter_pending(s->t, s->sp, s->ws, b, values, probs, s->n_labels);
    finalize_root(s->t, s->sp, s->ws);
    for (int item = 0; item < 4 * s->sp.batch_size; ++item) prepare_item(s->t, s->sp, s->ws, item);
}
// logical search thread `th` (0 or 1): SearchThread::create_mini_batch / the rest of thread_iteration
int he_search_create_mini_batch_t(HeSearch* s, int th) {
    HeBatch& bt = s->batch[th];
    if (s->sp.epsilon_greedy_counter != 0 || s->sp.epsilon_checks_counter != 0)
        create_mini_batch<true>(bt.t, s->sp, s->ws);
    else
        create_mini_batch<false>(bt.t, s->sp, s->ws);
    HostWriterFactory wf{bt.planes.data(), s->channels};
    for (int b = 0; b < bt.bs.n_new; ++b) {
        const auto target = wf.make(b);
        expand_pending(bt.t, s->sp, s->ws, bt.new_node[b], &target);
    }
    return bt.bs.n_new;
}
void he_search_apply_results_t(HeSearch* s, int th, const float* values, const float* probs) {
    HeBatch& bt = s->batch[th];
    backup_results(bt.t, s->sp, values);
    for (int b = 0; b < bt.bs.n_new; ++b) scatter_pending(bt.t, s->sp, s->ws, b, values, probs, s->n_labels);
    for (int item = 0; item < 4 * s->sp.batch_size; ++item) prepare_item(bt.t, s->sp, s->ws, item);
}
int he_search_create_mini_batch(HeSearch* s) { return he_search_create_mini_batch_t(s, 0); }
void he_search_apply_results(HeSearch* s, const float* values, const float* probs) { he_search_apply_results_t(s, 0, values, probs); }
void he_search_batch_keys_t(const HeSearch* s, int th, unsigned long long* out) {
    for (int i = 0; i < s->batch[th].bs.n_new; ++i) out[i] = s->hdr[s->batch[th].new_node[i]].key;
}
void he_search_batch_keys(const HeSearch* s, unsigned long long* out) { he_search_batch_keys_t(s, 0, out); }
int he_search_done(const HeSearch* s) { return s->st.done || s->st.error; }
int he_search_thread_done(const HeSearch* s, int th) { return s->st.done || s->st.error || s->batch[th].bs.done; }
int he_search_error(const HeSearch* s) { return s->st.error; }
const SearchResult* he_search_result(HeSearch* s) {
    collect_result(s->t, s->sp, &s->result);
    return &s->result;
}
void he_fake_eval(unsigned long long key, int n_labels, float* value, float* prob) {
    *value = fake_value(key);
    for (int i = 0; i < n_labels; ++i) prob[i] = fake_prob(key, i);
}
int he_sizeof_result() { return static_cast<int>(sizeof(SearchResult)); }
// root statistics of the ThreadManager heuristics: {node_count, first, second, max_q_is_max_visits, valid}, {q1, q2, eval}
void he_search_time_stats(HeSearch* s, unsigned* iout, float* fout) {
    RootTimeStats r;
    collect_time_stats(s->t, &r);
    iout[0] = r.node_count, iout[1] = r.first_visits, iout[2] = r.second_visits;
    iout[3] = static_cast<unsigned>(r.max_q_is_max_visits), iout[4] = static_cast<unsigned>(r.valid);
    fout[0] = r.q_first, fout[1] = r.q_second, fout[2] = r.value_eval;
}

// first_and_second_max as collect_time_stats applies it: a root with k open, childless edges of the given visit counts
// and Q values; iout = {first, second, max_q_is_max_visits}, fout = {q_first, q_second, value_eval}.
void he_time_stats_of(int k, const unsigned* n, const float* q, unsigned* iout, float* fout) {
    std::vector<uint32_t> N(n, n + k);
    std::vector<float> Q(q, q + k);
    std::vector<int32_t> child(k, -1);
    NodeHdr root{};
    root.no_visit_idx = static_cast<uint16_t>(k);
    root.n_moves = static_cast<uint16_t>(k);
    root.edge_base = 0;
    root.flags = NF_HAS_D | NF_SORTED | NF_HAS_NN;
    root.node_type = NT_UNSOLVED;
    for (int i = 0; i < k; ++i) root.visit_sum += N[i];
    root.real_visits = root.visit_sum;
    TreeState st{};
    st.n_nodes = 1;
    st.root = 0;
    TreeDev t{};
    t.hdr = &root;
    t.N = N.data();
    t.Q = Q.data();
    t.child = child.data();
    t.st = &st;
    RootTimeStats r;
    collect_time_stats(t, &r);
    iout[0] = r.first_visits, iout[1] = r.second_visits, iout[2] = static_cast<unsigned>(r.max_q_is_max_visits);
    fout[0] = r.q_first, fout[1] = r.q_second, fout[2] = r.value_eval;
}

// Select-step unit hook: k open children with the given statistics; out = {sure, fast_ci, exact_ci}.
void he_pick_both(int k, const float* p, const float* q, const unsigned* n, float cput, unsigned visit_sum, int* out) {
    std::vector<float> P(p, p + k), Q(q, q + k);
    std::vector<uint32_t> N(n, n + k), cb(k, 0);
    std::vector<int32_t> child(k, -1);
    std::vector<uint8_t> vl(k, 0);
    TreeDev t{};
    t.P = P.data();
    t.Q = Q.data();
    t.N = N.data();
    t.cbase = cb.data();
    t.child = child.data();
    t.vl = vl.data();
    NodeHdr h{};
    h.no_visit_idx = static_cast<uint16_t>(k);
    h.edge_base = 0;
    h.cput = cput;
    h.visit_sum = visit_sum;
    h.sqrt_vs = sqrt(static_cast<double>(visit_sum));
    const EdgeRegs pre = load_edge(t, 0);
    bool sure = false;
    const SelectPick f = pick_fast(t, h, pre, &sure);
    const SelectPick e = pick_exact(t, h, pre);
    out[0] = sure ? 1 : 0;
    out[1] = f.ci;
    out[2] = e.ci;
}
}

// ---------------------------------------------------------------- glibc powf / logf restatement vs the live libm
#include <math.h>

#include "glibc_flt32.cuh"
extern "C" {
float he_powf(float x, float y) { return ara::glibc::powf_(x, y); }
float he_logf(float x) { return ara::glibc::logf_(x); }
// bit patterns [lo, hi) step `stride` as x; counts disagreements with libm, first one into *bad
unsigned long long he_powf_sweep(unsigned lo, unsigned hi, unsigned stride, float y, unsigned* bad) {
    unsigned long long n = 0;
    for (unsigned long long u = lo; u < hi; u += stride) {
        const float x = ara::glibc::u2f(static_cast<uint32_t>(u));
        const uint32_t a = ara::glibc::f2u(ara::glibc::powf_(x, y)), b = ara::glibc::f2u(powf(x, y));
        if (a != b && !((a & 0x7fffffffu) > 0x7f800000u && (b & 0x7fffffffu) > 0x7f800000u)) {
            if (n == 0 && bad) *bad = static_cast<uint32_t>(u);
            ++n;
        }
    }
    return n;
}
unsigned long long he_logf_sweep(unsigned lo, unsigned hi, unsigned stride, unsigned* bad) {
    unsigned long long n = 0;
    for (unsigned long long u = lo; u < hi; u += stride) {
        const float x = ara::glibc::u2f(static_cast<uint32_t>(u));
        const uint32_t a = ara::glibc::f2u(ara::glibc::logf_(x)), b = ara::glibc::f2u(logf(x));
        if (a != b) {
            if (n == 0 && bad) *bad = static_cast<uint32_t>(u);
            ++n;
        }
    }
    return n;
}
// the live libm on arrays (numpy's own float32 pow / log are not glibc's)
void he_libm_powf_array(const float* x, const float* y, int n, float* out) {
    for (int i = 0; i < n; ++i) out[i] = powf(x[i], y[i]);
}
void he_libm_logf_array(const float* x, int n, float* out) {
    for (int i = 0; i < n; ++i) out[i] = logf(x[i]);
}
}
