// GPU MCTS: flat SoA node / edge pools in HBM and the warp-level search primitives that walk them.
//
// One warp owns one tree.  Playouts of a tree are SEQUENTIAL inside the warp (each playout sees the virtual visits
// of the previous one, exactly as the reference's single search thread does) -- lanes parallelise the child argmax,
// move legality, plane encoding, the repetition scan and the prior sort; independent trees run on independent warps.
//
// Reference semantics restated here (engine/src of QueensGambit/CrazyAra):
//   select   node.cpp:1150-1167 select_child_node, :1056-1063 get_current_u_values, :1243-1246 get_current_cput
//   virtual  node.cpp:507-529 apply_virtual_loss_to_child, node.h:199-246 revert_virtual_loss_and_update,
//            node.cpp:661-679 revert_virtual_loss, node.h:819-843 backup_value
//   expand   node.cpp:82-106 Node ctor, :880-904 check_for_terminal, :571-580 increment_no_visit_idx,
//            searchthread.cpp:164-271 get_new_child_to_evaluate, :347-380 create_mini_batch
//   scatter  searchthread.cpp:290-324, node.cpp:961-979 set_probabilities_for_moves, util/blazeutil.h:78-88,
//            node.cpp:464-470 sort_moves_by_probabilities, :634-644 prepare_node_for_visits
//   solver   node.cpp:108-173, :265-297, :365-453, :1006-1010
//   results  node.cpp:1070-1148, evalinfo.cpp:112-121, :195-249
// Everything is __host__ __device__ over the lane abstraction so the whole search also runs as a 1-lane emulation on
// the CPU for unit tests (tests/hostemu); that build is scaffolding, not a fallback.
#pragma once
#include <math.h>

#include "ara_b200.h"
#include "chess_dev.cuh"
#include "glibc_flt32.cuh"
#include "planes_dev.cuh"
#include "time_manager.h"

namespace ara {

constexpr int kMaxDepth = 256;
constexpr int kPrepSlots = 2;  // prepared children per node (TreeDev::prep_board)
constexpr int kNoCheckmate = 65535;
constexpr float kQInit = -1.0f;
enum : int { VS_VIRTUAL_LOSS = 0, VS_VIRTUAL_VISIT = 1, VS_VIRTUAL_OFFSET = 2, VS_VIRTUAL_MIX = 3 };
enum : int { NT_WIN = 0, NT_DRAW = 1, NT_LOSS = 2, NT_UNSOLVED = 3 };
enum : int { NF_TERMINAL = 1, NF_HAS_NN = 2, NF_HAS_D = 4, NF_SORTED = 8, NF_INSPECTED = 16 };

// The structs that cross the C-ABI are the public header's: the kernels read and fill them as the caller sees them.
// OSettings (oracle/mcts.h) restates the settings with the same field names for the oracle.
using SearchParams = ara_search_settings_t;
using SearchResult = ara_search_result_t;
using NodeView = ara_node_view_t;
static_assert(sizeof(SearchResult::moves) / sizeof(Move) == kMaxMoves && sizeof(NodeView::moves) / sizeof(Move) == kMaxMoves,
              "the header's move arrays hold kMaxMoves entries");
static_assert(sizeof(SearchResult::pv) / sizeof(Move) == kMaxDepth, "the header's principal variation holds kMaxDepth moves");

struct alignas(16) NodeHdr {  // 64 B: one line per visited node on the select path
    double value_sum;
    uint64_t key;
    uint32_t real_visits;
    uint32_t visit_sum;
    uint32_t free_visits;
    uint32_t edge_base;
    int32_t parent;
    uint16_t n_moves;
    uint16_t no_visit_idx;
    uint16_t checkmate_idx;
    uint16_t end_in_ply;
    uint16_t n_unsolved;
    uint16_t parent_ci;
    int16_t repetition;
    uint8_t node_type;
    uint8_t flags;
    float cput;      // get_current_cput(visit_sum) and
    double sqrt_vs;  // sqrt(double(visit_sum)): refreshed by whoever changes visit_sum, which keeps both off the select path
};
static_assert(sizeof(NodeHdr) == 64, "NodeHdr must be 64 bytes");
static_assert(kMaxDepth * sizeof(uint64_t) >= kMaxMoves * sizeof(float), "fill_nn_results borrows path_key as float[kMaxMoves]");

// One mini-batch in flight (the members of a SearchThread of the reference that describe its current batch).  A search
// with Threads = 2 has two per tree: two logical search threads take turns on the tree (search.cu), each with its own
// new leaves, trajectories and rows of the network batch.
struct BatchState {
    int n_new;   // new leaves waiting for network results (newNodes)
    int n_coll;  // collision trajectories to revert (collisionTrajectories)
    int n_exp;   // expansions of the mini-batch (entries of exp_parent)
    int done;    // this thread's run_search_thread loop has ended (searchthread.cpp:418-426); it never starts again
};

struct TreeState {
    int n_nodes;
    int n_edges;
    // Dirichlet generator (minstd_rand0 state): seeded once when the search handle is created -- from the settings' seed
    // and the tree's index -- and ADVANCED by every root noise draw, like the reference's one process-wide
    // std::default_random_engine (util/randomgen.h:35): successive searches, and different trees, see different noise
    uint32_t rng;
    // SearchLimits of the current go (searchlimits.h): by default the settings' values; ara_search_set_limits overrides
    // them per tree (self-play jitters the node budget of every search, rl/selfplay.cpp:146-152)
    uint32_t limit_simulations;
    uint32_t limit_nodes;
    // the settings' Q-value weight (posterior) and Dirichlet epsilon (root noise) of the current go, unless
    // ara_search_set_tree_settings overrides them per tree (self-play's quick searches, rl/selfplay.cpp:214-241)
    float q_value_weight;
    float dirichlet_epsilon;
    int root;        // node id of the current root (0 for a new tree, the re-rooted child when the tree is reused)
    int next_root;   // candidate root after ara_search_apply_move (MCTSAgent::ownNextRoot / opponentsNextRoot), -1 none
    int next_valid;  // apply_move has been called since the last search: only next_root may be reused
    int live_threads;  // logical search threads whose loop has not ended yet
    int done;      // nothing (more) to search: terminal root, or every thread's loop condition has failed
    int error;     // 1 node pool, 2 edge pool, 3 depth overflow
    unsigned iterations;
    unsigned evals;
    unsigned pre_nodes;  // EvalInfo::nodesPreSearch: node count of the root when the search began (0 for a new tree)
    unsigned long long sum_select_k;
    unsigned long long sum_depth;
    // SM-clock cycles spent per phase of create_mini_batch (lane 0): 0 descent, 1 board copy + do_move, 2 repetition +
    // move generation, 3 node/edge allocation + init, 4 plane encoding, 5 terminal backups, 6 trajectory bookkeeping
    unsigned long long prof[8];
    // rand() of the epsilon-greedy / epsilon-check exploration: glibc's TYPE_3 generator (crand_next), seeded when the
    // handle is created (srand(seed ^ tree index)) and advanced across searches like the C library's process-wide state
    int32_t crand_r[31];
    int32_t crand_f;  // front index; the rear index is (front + 28) % 31
};

#if defined(__CUDA_ARCH__)
#define ARA_CLOCK() clock64()
#else
#define ARA_CLOCK() 0LL
#endif
#define ARA_PROF(st, idx, t0)                                                      \
    do {                                                                           \
        const long long now_ = ARA_CLOCK();                                        \
        if (ARA_LANE == 0) (st).prof[idx] += static_cast<unsigned long long>(now_ - (t0)); \
        (t0) = now_;                                                               \
    } while (0)

// -DARA_PROF_FINE: split the descent into edge wait (slot 4), PUCT arithmetic + reductions (slot 7) and child-header
// wait (slot 5).  The clock is read through an asm that consumes `dep`, so it cannot be scheduled before dep arrives.
#if defined(ARA_PROF_FINE) && defined(__CUDA_ARCH__)
#define ARA_FINE(stp, idx, t0, dep)                                                         \
    do {                                                                                    \
        long long now_;                                                                     \
        asm volatile("mov.u64 %0, %%clock64;" : "=l"(now_) : "r"(static_cast<int>(dep)) : "memory"); \
        if (ARA_LANE == 0) (stp)->prof[idx] += static_cast<unsigned long long>(now_ - (t0)); \
        (t0) = now_;                                                                        \
    } while (0)
#define ARA_FINE_T0(t0) long long t0 = clock64()
#else
#define ARA_FINE(stp, idx, t0, dep) do { } while (0)
#define ARA_FINE_T0(t0) do { } while (0)
#endif

struct TreeDev {
    NodeHdr* hdr;
    Board* board;
    float* P;
    float* Q;
    uint32_t* N;
    int32_t* child;
    uint32_t* cbase;  // edge_base of the child behind every edge: lets one round trip fetch a child's header AND edges
    Move* move;
    uint8_t* vl;
    uint8_t* etype;
    TreeState* st;
    BatchState* bs;  // the mini-batch this view of the tree works on (everything from exp_parent to traj_len and slot_base
                     // below belongs to it; the pools above are the tree's)
    // "prepared child": at every node exactly one child can be expanded next (index no_visit_idx-1, opened in prior
    // order); its position, repetition state and terminal verdict depend on the node alone (the tree has no
    // transpositions), so they are computed ahead of time by parallel warps (prepare_child) and the sequential
    // select only copies them
    Board* prep_board;      // [max_nodes][kPrepSlots]
    int16_t* prep_ci;       // [max_nodes][kPrepSlots] child index the slot holds, -1 = none
    uint8_t* prep_term;     // [max_nodes][kPrepSlots] its terminal type
    int32_t* exp_parent;    // [3B] nodes that had a child expanded in the last mini-batch
    int32_t* new_node;      // [B]
    int32_t* traj_node;     // [2B][kMaxDepth]   rows 0..B-1 new leaves, B..2B-1 collisions
    uint16_t* traj_ci;      // [2B][kMaxDepth]
    uint32_t* traj_edge;    // [2B][kMaxDepth]   absolute edge index (edge_base + ci) of every step
    int32_t* traj_len;      // [2B]   plies below the root of the trajectory's leaf
    int32_t* traj_start;    // [2B]   first ply that belongs to the trajectory (0 unless the exploration started it deeper)
    const uint64_t* hist_keys;  // positions before the root, oldest first
    const int16_t* hist_reps;
    int hist_len;
    const float* cput_lut;  // cput for visit_sum < cput_lut_len, computed on the host with the host libm
    int cput_lut_len;
    const double* sqrt_lut;  // sqrt(double(visit_sum)) for visit_sum < cput_lut_len
    int max_nodes;
    int max_edges;
    int slot_base;  // first row of this tree in the network batch
};

struct WarpScratch {  // per-warp shared memory (stack on the host)
    Board parent;
    Board child;
    Move scratch[kMaxMoves];
    Move legal[kMaxMoves];
    uint64_t path_key[kMaxDepth];
    int16_t path_rep[kMaxDepth];
    int32_t traj_node[kMaxDepth];
    uint16_t traj_ci[kMaxDepth];
    uint32_t traj_edge[kMaxDepth];
    float sort_p[kMaxMoves];
    MoveGenScratch mg;
    TreeState st_local;  // the tree's counters live in shared memory while the select kernel runs
    int bcast[4];
};

// The kernels that run while the other logical thread's forward occupies the SMs (Threads = 2) hold only what they use
// in shared memory, so that a CTA fits beside a tower CTA (search.cu checks the sizes).  The functions they call are
// templates over the layout; the select kernels and the host emulation pass a whole WarpScratch.
struct ExpandScratch {  // expand_pending
    Board child;
    Move scratch[kMaxMoves];
    Move legal[kMaxMoves];
    MoveGenScratch mg;
    PlaneExchange planes;
    int bcast[4];
};
struct ScatterScratch {  // fill_nn_results
    Move scratch[kMaxMoves];
    Move legal[kMaxMoves];
    float sort_p[kMaxMoves];
    uint64_t path_key[kMaxDepth];  // the priors in policy-index order when a temperature applies (as in WarpScratch)
};
struct PrepareScratch {  // prepare_child
    Board child;
    Move scratch[kMaxMoves];
    Move legal[kMaxMoves];
    uint64_t path_key[kMaxDepth];
    int16_t path_rep[kMaxDepth];
    MoveGenScratch mg;
};
union UpdateScratch {  // one warp scatters a leaf, then prepares a child
    ScatterScratch scatter;
    PrepareScratch prepare;
};

// ------------------------------------------------------------------ small helpers
ARA_HD int virtual_style_of(const SearchParams& sp, uint32_t visits) {  // node.h:87-95
    if (sp.virtual_style == VS_VIRTUAL_MIX) return visits > sp.virtual_mix_threshold ? VS_VIRTUAL_LOSS : VS_VIRTUAL_VISIT;
    return sp.virtual_style;
}
ARA_HD float node_value(const NodeHdr& h) { return static_cast<float>(h.value_sum / h.real_visits); }
ARA_HD void node_set_value(NodeHdr& h, float v) {  // node.cpp:716-720
    ++h.real_visits;
    h.value_sum = static_cast<double>(v * static_cast<float>(h.real_visits));
}
ARA_HD float current_cput(const TreeDev& t, const SearchParams& sp, uint32_t visit_sum) {
    if (static_cast<int>(visit_sum) < t.cput_lut_len) return t.cput_lut[visit_sum];
    return logf((static_cast<float>(visit_sum) + sp.cpuct_base + 1) / sp.cpuct_base) + sp.cpuct_init;
}
ARA_HD double sqrt_visits(const TreeDev& t, uint32_t visit_sum) {
    if (static_cast<int>(visit_sum) < t.cput_lut_len) return t.sqrt_lut[visit_sum];
    return sqrt(static_cast<double>(visit_sum));
}
template <typename T>
ARA_HD T bcast0(T v) {
    return ARA_SHFL(v, 0);
}

// copy one 128-byte board between memories, cooperatively
ARA_HD void copy_board(Board* dst, const Board* src) {
#if defined(__CUDA_ARCH__)
    if (ARA_LANE < 8) reinterpret_cast<uint4*>(dst)[ARA_LANE] = reinterpret_cast<const uint4*>(src)[ARA_LANE];
#else
    *dst = *src;
#endif
    ARA_WARP_SYNC();
}

// ------------------------------------------------------------------ select + virtual visit (one fused warp step)
// Node::select_child_node (node.cpp:1150-1167, first maximum wins) followed by apply_virtual_loss_to_child
// (node.cpp:507-529).  Written for a single in-order warp, where every load->use pair costs a full memory latency and
// every dependent arithmetic chain is exposed.  Per tree level the chain is
//     edge arrays (one round trip; the header refresh values sqrt(visit_sum+1) and cput(visit_sum+1) are computed
//     while it is in flight) -> FP64 PUCT term -> two warp reductions -> child header (one round trip; the virtual
//     visit and the header update are stored while it is in flight).
//   * the caller hands in the 64-byte header in registers (it came back from the previous level's step);
//   * sqrt(visit_sum) and cput(visit_sum) are cached in the header by whoever changes visit_sum;
//   * the argmax is redux.max over an order-preserving integer image of Q+U, then redux.min over the indices of the
//     lanes that hold the maximum (first maximum wins, as in the reference);
//   * the lane that owns the winning edge applies the virtual visit from its registers, lane 0 updates the header.
ARA_HD void prefetch_line(const void* p) {
#if defined(__CUDA_ARCH__)
    asm volatile("prefetch.global.L1 [%0];" ::"l"(p));
#else
    (void)p;
#endif
}

ARA_HD void load_hdr(NodeHdr* dst, const NodeHdr* src) {
#if defined(__CUDA_ARCH__)
    const uint4* s4 = reinterpret_cast<const uint4*>(src);
    uint4* d4 = reinterpret_cast<uint4*>(dst);
    const uint4 a = s4[0], b = s4[1], c = s4[2], d = s4[3];
    d4[0] = a;
    d4[1] = b;
    d4[2] = c;
    d4[3] = d;
#else
    *dst = *src;
#endif
}

// the per-edge statistics one lane holds for one candidate child
struct EdgeRegs {
    int c;         // child node id (-1: not expanded yet)
    float p, q;
    uint32_t n;
    uint32_t cb;   // edge_base of the child (valid once the child has been expanded)
    uint8_t vl;
};
ARA_HD EdgeRegs load_edge(const TreeDev& t, uint32_t idx) {
    EdgeRegs x;
    x.c = t.child[idx];
    x.p = t.P[idx];
    x.q = t.Q[idx];
    x.n = t.N[idx];
    x.cb = t.cbase[idx];
    x.vl = t.vl[idx];
    return x;
}
// order-preserving integer image of a float (x + 0 folds -0 into +0, so equal floats have equal images)
ARA_HD uint32_t float_image(float v) {
#if defined(__CUDA_ARCH__)
    const uint32_t fb = __float_as_uint(v + 0.0f);
#else
    union { float f; uint32_t u; } cv;
    cv.f = v + 0.0f;
    const uint32_t fb = cv.u;
#endif
    return (fb & 0x80000000u) ? ~fb : (fb | 0x80000000u);
}

struct SelectStep {
    int ci;        // selected child index
    int child;     // its node id (-1: not expanded yet)
    NodeHdr ch;    // header of `child` (valid when child >= 0)
    EdgeRegs pre;  // and this lane's edge of it (edge index ARA_LANE)
};

struct SelectPick {
    int ci;         // winning child index (same in every lane)
    bool owner;     // this lane holds the winning edge in `x`
    EdgeRegs x;
    // set by pick_child: what the pick adds to sum_select_k, and the node's header refresh after the visit
    int counted_k;
    uint32_t vs_new;  // visit_sum + 1, its cput and sqrt
    float cput_new;
    double sqrt_new;
};

// Exact arithmetic of the reference (get_current_u_values, node.cpp:1056-1063): the blaze expression
//     cput * subvector(P) * (sqrt(N) / (n + 1.0))
// is (float scalar * float vector) * double vector; blaze restructures (v*s)*w to (v*w)*s (DVecScalarMultExpr's
// restructuring operators), so element i is  float( (double(P_i) * (sqrt(N) / (double(n_i) + 1.0))) * double(cput) ).
// First maximum of Q + U over the open children.
ARA_HD SelectPick pick_exact(const TreeDev& t, const NodeHdr& h, const EdgeRegs& pre) {
    const int k = h.no_visit_idx;
    const uint32_t e = h.edge_base;
    const float cput = h.cput;
    const double sq = h.sqrt_vs;
    SelectPick r;
    r.x = pre;
    int best_i = 0x7fffffff;
    float best_v = 0.0f;
    for (int i = ARA_LANE; i < k; i += ARA_WARP_N) {
        const EdgeRegs x = i == ARA_LANE ? pre : load_edge(t, e + i);
        const float u = static_cast<float>((static_cast<double>(x.p) * (sq / (static_cast<double>(x.n) + 1.0))) * static_cast<double>(cput));
        const float v = x.q + u;
        if (best_i == 0x7fffffff || v > best_v) best_v = v, best_i = i, r.x = x;
    }
    const uint32_t img = best_i == 0x7fffffff ? 0u : float_image(best_v);
    const uint32_t top = ARA_REDUCE_MAX(img);
    r.ci = static_cast<int>(ARA_REDUCE_MIN(img == top ? static_cast<uint32_t>(best_i) : 0x7fffffffu));
    r.owner = best_i == r.ci;
    return r;
}

// Same decision from fp32 arithmetic with a rigorous error margin.  With U the real value of cput*P*sqrt(N)/(n+1):
// the reference's u is U(1+d), |d| <= 2^-24 (the double operations contribute < 2^-50); the fp32 value uf below
// carries at most five roundings (float(sqrt), float(n), +1, *, /), so |uf - u| < 6e-7 uf.  Adding the two roundings
// of q + u and of the bounds themselves, the exact Q+U of a candidate lies within E = 6e-7 uf + 2.6e-7 |vf| + 1e-30
// of vf.  If the fp32 winner's lower bound exceeds every other candidate's upper bound it is the reference's strict
// maximum; otherwise (near-ties, exact ties) `sure` is false and the caller falls back to pick_exact.
ARA_HD SelectPick pick_fast(const TreeDev& t, const NodeHdr& h, const EdgeRegs& pre, bool* sure) {
    const int k = h.no_visit_idx;
    const uint32_t e = h.edge_base;
    const float cput = h.cput;
    const float sqf = static_cast<float>(h.sqrt_vs);
    const float ninf = -3.0e38f;
    SelectPick r;
    r.x = pre;
    int best_i = 0x7fffffff;
    float best_v = 0.0f, best_hi = ninf, best_lo = 0.0f, oth_hi = ninf;
    if (ARA_LANE < k) {  // the usual case: at most one candidate per lane, already in registers
        const float uf = (cput * pre.p) * sqf / (static_cast<float>(pre.n) + 1.0f);
        const float err = uf * 6e-7f + fabsf(pre.q + uf) * 2.6e-7f + 1e-30f;
        best_v = pre.q + uf, best_hi = best_v + err, best_lo = best_v - err, best_i = ARA_LANE;
    }
#if defined(__CUDA_ARCH__)
#pragma unroll 1
#endif
    for (int i = ARA_LANE + ARA_WARP_N; i < k; i += ARA_WARP_N) {  // more open children than lanes
        const EdgeRegs x = load_edge(t, e + i);
        const float uf = (cput * x.p) * sqf / (static_cast<float>(x.n) + 1.0f);
        const float vf = x.q + uf;
        const float err = uf * 6e-7f + fabsf(vf) * 2.6e-7f + 1e-30f;
        const float hi = vf + err;
        if (vf > best_v) {
            if (best_hi > oth_hi) oth_hi = best_hi;
            best_v = vf, best_hi = hi, best_lo = vf - err, best_i = i, r.x = x;
        } else if (hi > oth_hi) {
            oth_hi = hi;
        }
    }
    const uint32_t img = best_i == 0x7fffffff ? 0u : float_image(best_v);
    const uint32_t top = ARA_REDUCE_MAX(img);
    r.ci = static_cast<int>(ARA_REDUCE_MIN(img == top ? static_cast<uint32_t>(best_i) : 0x7fffffffu));
    r.owner = best_i == r.ci;
    // the winner's lower bound, broadcast from its lane, against every other candidate's upper bound (one vote)
    const float lo_w = ARA_SHFL(best_lo, r.ci & (ARA_WARP_N - 1));
    const float others = r.owner ? oth_hi : (best_hi > oth_hi ? best_hi : oth_hi);
    *sure = ARA_ALL(others < lo_w);
    return r;
}

// The child select_child_node picks at a node with header `h` (`pre`: this lane's edge).  forced >= 0: the child index
// was chosen by the exploration prologue (eps_prologue) -- no selection, the visit only.
ARA_HD SelectPick pick_child(const TreeDev& t, const SearchParams& sp, const NodeHdr& h, const EdgeRegs& pre, int forced) {
    const int k = h.no_visit_idx;
    const bool single = forced >= 0 || k == 1 || h.checkmate_idx != kNoCheckmate;
    // header refresh values, off the dependent chain
    const uint32_t vs_new = h.visit_sum + 1;
    const float cput_new = current_cput(t, sp, vs_new);
    const double sqrt_new = sqrt_visits(t, vs_new);
    SelectPick pk;
    if (single) {  // only one open child, or a forced win
        pk.ci = forced >= 0 ? forced : (k == 1 ? 0 : h.checkmate_idx);
        pk.owner = ARA_LANE == (pk.ci & (ARA_WARP_N - 1));
        pk.x = pre;
        if (pk.owner && pk.ci != ARA_LANE) pk.x = load_edge(t, h.edge_base + pk.ci);
    } else {
        bool sure = false;
        pk = pick_fast(t, h, pre, &sure);
        if (!sure) pk = pick_exact(t, h, pre);
    }
    // (sum_select_k counts what select_child_node reads: nothing for a forced child, nor for its two shortcuts)
    pk.counted_k = single ? 0 : k;
    pk.vs_new = vs_new;
    pk.cput_new = cput_new;
    pk.sqrt_new = sqrt_new;
    return pk;
}

// The virtual visit of the picked child of node `nid`: apply_virtual_loss_to_child on the owner lane (registers in,
// stores out), and the header refresh on lane 0.
ARA_HD void apply_visit(const TreeDev& t, const SearchParams& sp, int nid, const NodeHdr& h, const SelectPick& pk) {
    if (pk.owner) {
        const uint32_t ee = h.edge_base + static_cast<uint32_t>(pk.ci);
        if (virtual_style_of(sp, pk.x.n) == VS_VIRTUAL_LOSS)
            t.Q[ee] = static_cast<float>((static_cast<double>(pk.x.q) * pk.x.n - 1) / static_cast<double>(pk.x.n + 1));
        t.N[ee] = pk.x.n + 1;
        t.vl[ee] = static_cast<uint8_t>(pk.x.vl + 1);
    }
    if (ARA_LANE == 0) {
        NodeHdr* hp = &t.hdr[nid];
        hp->visit_sum = pk.vs_new;
        hp->cput = pk.cput_new;
        hp->sqrt_vs = pk.sqrt_new;
        if (!(h.flags & NF_HAS_D)) hp->flags = h.flags | NF_HAS_D | NF_SORTED;  // prepare_node_for_visits (lazy flag)
    }
}

ARA_HD SelectStep select_and_visit(const TreeDev& t, const SearchParams& sp, int nid, const NodeHdr& h,
                                   const EdgeRegs& pre, int forced = -1) {
    ARA_FINE_T0(tf);
    // (prefetching every open child's header and edge lines here was measured: 2 % slower, the issue slots cost more
    // than the earlier start of the round trip saves)
    ARA_FINE(t.st, 4, tf, pre.c ^ static_cast<int>(pre.n));
    const SelectPick pk = pick_child(t, sp, h, pre, forced);
    SelectStep r;
    r.ci = pk.ci;
    const int owner_lane = pk.ci & (ARA_WARP_N - 1);
    (void)owner_lane;  // the 1-lane host build has no shuffles
    r.child = ARA_SHFL(pk.x.c, owner_lane);
    const uint32_t cb = ARA_SHFL(pk.x.cb, owner_lane);
    ARA_FINE(t.st, 7, tf, r.child);
    if (r.child >= 0) {  // next level: header and this lane's edge, one round trip, in flight during the stores below
        load_hdr(&r.ch, &t.hdr[r.child]);
        r.pre = load_edge(t, cb + ARA_LANE);
    }
#if defined(ARA_PROF_FINE)
    ARA_FINE(t.st, 5, tf, r.child >= 0 ? (r.ch.flags ^ r.pre.c) : 0);
#endif
    apply_visit(t, sp, nid, h, pk);
    // (last: placed ahead of the look-ahead loads, its shared-memory round trip delayed them -- measured 1.6 % slower)
    if (ARA_LANE == 0) t.st->sum_select_k += static_cast<unsigned long long>(pk.counted_k);
    return r;
}

// ------------------------------------------------------------------ MCTS solver (lane 0 only; TWO_PLAYER, no tablebases)
ARA_HD void disable_action(const TreeDev& t, uint32_t e) {
    t.P[e] = 0.0f;
    t.Q[e] = static_cast<float>(-2147483647);
}
ARA_HD bool at_least_one_drawn_child(const TreeDev& t, const NodeHdr& h) {
    bool drawn = false;
    for (int i = 0; i < h.no_visit_idx; ++i) {
        const int c = t.child[h.edge_base + i];
        if (c < 0) return false;
        const NodeHdr& ch = t.hdr[c];
        if (!(ch.flags & NF_HAS_D) || (ch.node_type != NT_DRAW && ch.node_type != NT_WIN)) return false;
        if (ch.node_type == NT_DRAW) drawn = true;
    }
    return drawn;
}
ARA_HD bool only_won_children(const TreeDev& t, const NodeHdr& h) {
    for (int i = 0; i < h.no_visit_idx; ++i) {
        const int c = t.child[h.edge_base + i];
        if (c < 0 || t.hdr[c].node_type != NT_WIN) return false;
    }
    return true;
}
ARA_HD void define_end_ply(const TreeDev& t, NodeHdr& h, const NodeHdr& ch) {  // node.cpp:265-289
    if (h.node_type == NT_LOSS) {
        for (int i = 0; i < h.no_visit_idx; ++i) {
            const int c = t.child[h.edge_base + i];
            if (c >= 0 && t.hdr[c].end_in_ply + 1 > h.end_in_ply) h.end_in_ply = static_cast<uint16_t>(t.hdr[c].end_in_ply + 1);
        }
        return;
    }
    if (h.node_type == NT_DRAW) {
        for (int i = 0; i < h.no_visit_idx; ++i) {
            const int c = t.child[h.edge_base + i];
            if (c >= 0 && t.hdr[c].node_type == NT_DRAW && t.hdr[c].end_in_ply + 1 < h.end_in_ply)
                h.end_in_ply = static_cast<uint16_t>(t.hdr[c].end_in_ply + 1);
        }
        return;
    }
    h.end_in_ply = static_cast<uint16_t>(ch.end_in_ply + 1);
}
ARA_HD void update_solved_terminal(const TreeDev& t, NodeHdr& h, const NodeHdr& ch, int ci, int target) {
    define_end_ply(t, h, ch);
    node_set_value(h, static_cast<float>(target));
    t.Q[h.edge_base + ci] = static_cast<float>(target);
}
ARA_HD bool solve_for_terminal(const TreeDev& t, int nid, int ci) {  // node.cpp:365-453
    NodeHdr& h = t.hdr[nid];
    const int c = t.child[h.edge_base + ci];
    const NodeHdr& ch = t.hdr[c];
    if (!(ch.flags & NF_HAS_D)) return false;
    if (ch.node_type == NT_UNSOLVED) return false;
    if (h.node_type != NT_UNSOLVED) return false;
    const uint32_t e = h.edge_base + ci;
    if (t.etype[e] == NT_UNSOLVED) {
        --h.n_unsolved;
        t.etype[e] = ch.node_type;
        if (ch.node_type == NT_WIN) disable_action(t, e);
    }
    if (ch.node_type == NT_LOSS) {
        h.node_type = NT_WIN;
        update_solved_terminal(t, h, ch, ci, 1);
        h.checkmate_idx = static_cast<uint16_t>(ci);
        return true;
    }
    if (h.n_unsolved == 0 && ch.node_type == NT_WIN && only_won_children(t, h)) {
        h.node_type = NT_LOSS;
        update_solved_terminal(t, h, ch, ci, -1);
        return true;
    }
    if (h.n_unsolved == 0 && ch.node_type != NT_LOSS && at_least_one_drawn_child(t, h)) {
        h.node_type = NT_DRAW;
        update_solved_terminal(t, h, ch, ci, 0);
        return true;
    }
    return false;
}

// ------------------------------------------------------------------ backup (lane 0 only)
ARA_HD void revert_virtual_loss_and_update(const TreeDev& t, const SearchParams& sp, int nid, int ci, float value,
                                           bool free_backup, bool solve) {  // node.h:199-246
    NodeHdr& h = t.hdr[nid];
    const uint32_t e = h.edge_base + ci;
    h.value_sum += value;
    ++h.real_visits;
    if (t.N[e] == 1) {
        t.Q[e] = value;
    } else {
        const int style = virtual_style_of(sp, t.N[e]);
        if (style == VS_VIRTUAL_LOSS) {
            t.Q[e] = static_cast<float>((static_cast<double>(t.Q[e]) * t.N[e] + 1 + value) / t.N[e]);
        } else if (style == VS_VIRTUAL_VISIT) {
            const uint32_t real = t.N[e] - t.vl[e];
            t.Q[e] = static_cast<float>((static_cast<double>(t.Q[e]) * real + value) / (real + 1));
        }
    }
    --t.vl[e];
    if (free_backup) ++h.free_visits;
    if (solve) solve_for_terminal(t, nid, ci);
}
ARA_HD void backup_value(const TreeDev& t, const SearchParams& sp, float value, const int32_t* tn, const uint16_t* tc,
                         int len, bool free_backup, bool solve) {  // node.h:819-843 (transposition branches are dead)
    for (int i = len - 1; i >= 0; --i) {
        value = -value;
        revert_virtual_loss_and_update(t, sp, tn[i], tc[i], value, free_backup, solve);
    }
}
ARA_HD void revert_virtual_loss(const TreeDev& t, const SearchParams& sp, int nid, int ci) {  // node.cpp:661-679
    NodeHdr& h = t.hdr[nid];
    const uint32_t e = h.edge_base + ci;
    if (virtual_style_of(sp, t.N[e]) == VS_VIRTUAL_LOSS)
        t.Q[e] = static_cast<float>((static_cast<double>(t.Q[e]) * t.N[e] + 1) / (t.N[e] - 1));
    --t.N[e];
    const uint32_t vs = h.visit_sum - 1;
    h.visit_sum = vs;
    h.cput = current_cput(t, sp, vs);
    h.sqrt_vs = sqrt_visits(t, vs);
    --t.vl[e];
}

// ------------------------------------------------------------------ repetition over (pre-root history + tree path)
// ws.path_key/rep[0..depth) hold root..current; ws.child is the new position (depth plies below the root).
template <class WS>
ARA_HD int repetition_on_path(const TreeDev& t, const WS& ws, int depth) {
    const Board& b = ws.child;
    const int total = t.hist_len + depth;  // number of earlier positions
    int end = repetition_end(b);
    if (end > total) end = total;
    for (int base = 4; base <= end; base += 2 * ARA_WARP_N) {
        const int i = base + 2 * ARA_LANE;
        bool hit = false;
        int rep = 0;
        if (i <= end) {
            const int idx = total - i;
            const uint64_t k = idx < t.hist_len ? t.hist_keys[idx] : ws.path_key[idx - t.hist_len];
            if (k == b.key) {
                hit = true;
                rep = idx < t.hist_len ? t.hist_reps[idx] : ws.path_rep[idx - t.hist_len];
            }
        }
        const uint32_t m = ARA_BALLOT(hit);
        if (m) {
#if defined(__CUDA_ARCH__)
            const int src = __ffs(m) - 1;
#else
            const int src = 0;
            (void)src;
#endif
            const int ri = ARA_SHFL(rep, src);
            const int ii = ARA_SHFL(i, src);
            return ri ? -ii : ii;
        }
    }
    return 0;
}

// ------------------------------------------------------------------ expansion
// Expansion is split in two so that only what the reference's SEQUENTIAL semantics need stays in the per-tree loop:
//   expand_node_seq   (inside create_mini_batch, one warp per tree): repetition info, terminal verdict, node id,
//                     header, board, child link.  The verdict needs "is there any legal move", answered without the
//                     full list whenever some piece that is not on a line with the king has a pseudo-legal move.
//   expand_pending    (one warp per NEW leaf, all leaves of all trees in parallel): full legal move list, edge
//                     allocation + initialisation, policy indices, input planes.

// Does the side to move have a legal move?  Warp-collective; *checked_out = side to move is in check.
template <class WS>
ARA_HD bool any_legal_move(const Board& b, WS& ws, bool* checked_out) {
    const int us = b.stm, them = us ^ 1;
    const uint64_t own = b.by_color[us], opp = b.by_color[them], occ = own | opp;
    const int ksq = king_square(b, us);
    const bool checked = ksq >= 0 && attackers_of(b, ksq, occ, them, opp) != 0;
    *checked_out = checked;
    if (variant_end(b)) return false;
    if (!checked) {
        if (b.variant == V_CRAZYHOUSE) {
            const uint64_t empty = ~occ;
            bool nonpawn = false;
            for (int pt = PT_KNIGHT; pt <= PT_QUEEN; ++pt) nonpawn = nonpawn || b.hand[us][pt] != 0;
            if ((nonpawn && empty) || (b.hand[us][PT_PAWN] && (empty & ~(kRank1 | kRank8)))) return true;
        }
        // a piece that is not aligned with its king cannot be pinned: any pseudo-legal move of it is legal
        // (en passant excluded: it can uncover a rank attack through two removed pawns)
        const uint64_t king_lines = ksq >= 0 ? (rook_attacks_bb(bit(ksq), 0) | bishop_attacks_bb(bit(ksq), 0) | bit(ksq)) : 0;
        const uint64_t ep_bit = b.ep != 0xFF ? bit(b.ep) : 0;
        bool found = false;
        for (int sq = ARA_LANE; sq < 64; sq += ARA_WARP_N) {
            if (!(own & bit(sq)) || (king_lines & bit(sq))) continue;
            const int pt = piece_type_on(b, sq);
            uint64_t tg = piece_targets(b, sq, pt, us, own, opp, occ);
            if (pt == PT_PAWN) tg &= ~ep_bit;
            if (tg) found = true;
        }
        if (ARA_BALLOT(found)) return true;
    }
    return gen_legal(b, ws.mg, ws.scratch, ws.legal) > 0;
}

// Creates the node for ws.child (already moved), child `ci` of `parent` (or the root if parent < 0).
// Returns the new node id (uniform), or -1 on pool exhaustion.  *is_terminal receives the terminal verdict.
// Repetition state and terminal verdict of ws.child (already moved), `depth` plies below the root with the keys of the
// path in ws.path_key / path_rep.  Warp-collective; writes b.repetition.
template <class WS>
ARA_HD int leaf_verdict(const TreeDev& t, WS& ws, int depth) {
    Board& b = ws.child;
    const int rep = repetition_on_path(t, ws, depth);
    if (ARA_LANE == 0) b.repetition = static_cast<int16_t>(rep);
    ARA_WARP_SYNC();
    bool checked = false;
    const bool any = any_legal_move(b, ws, &checked);
    return terminal_type(b, any ? 1 : 0, checked);
}

// tt_known >= 0: ws.child comes from the node's prepared-child slot (repetition already set, verdict known).
// The ordered half of expand_node_seq: node id, header, child link, board (verdict `tt` already known).
ARA_HD int expand_node_alloc(const TreeDev& t, const SearchParams& sp, WarpScratch& ws, int parent, int ci, int tt,
                             uint32_t parent_edge_base) {
    Board& b = ws.child;
    int nid = -1;
    if (ARA_LANE == 0) {
        TreeState& st = *t.st;
        if (st.n_nodes >= t.max_nodes) {
            st.error = 1;
        } else {
            nid = st.n_nodes++;
            NodeHdr h;
            h.value_sum = 0.0;
            h.key = b.key;
            h.real_visits = 0;
            h.visit_sum = 0;
            h.free_visits = 0;
            h.edge_base = 0;
            h.parent = parent;
            h.n_moves = 0;  // filled by expand_pending
            h.no_visit_idx = 1;
            h.checkmate_idx = kNoCheckmate;
            h.end_in_ply = 0;
            h.n_unsolved = 0;
            h.parent_ci = static_cast<uint16_t>(ci < 0 ? 0 : ci);
            h.repetition = b.repetition;
            h.node_type = NT_UNSOLVED;
            h.flags = 0;
            h.cput = current_cput(t, sp, 0);
            h.sqrt_vs = 0.0;
            if (tt != TERM_NONE) {  // check_for_terminal node.cpp:880-904 + mark_as_terminal
                h.flags = NF_TERMINAL | NF_HAS_D | NF_SORTED;
                h.no_visit_idx = 0;
                if (tt == TERM_WIN) {
                    node_set_value(h, 1.0f);
                    h.node_type = NT_WIN;
                } else if (tt == TERM_DRAW) {
                    node_set_value(h, 0.0f);
                    h.node_type = NT_DRAW;
                } else {
                    node_set_value(h, -1.0f);
                    h.node_type = NT_LOSS;
                }
            }
            t.hdr[nid] = h;
            for (int s = 0; s < kPrepSlots; ++s) t.prep_ci[nid * kPrepSlots + s] = -1;
            if (parent >= 0) t.child[parent_edge_base + ci] = nid;
        }
    }
    nid = bcast0(nid);
    if (nid < 0) return -1;
    copy_board(&t.board[nid], &b);
    return nid;
}
ARA_HD int expand_node_seq(const TreeDev& t, const SearchParams& sp, WarpScratch& ws, int parent, int ci, int depth,
                           int* is_terminal, int tt_known = -1, uint32_t parent_edge_base = 0) {
    long long tp = ARA_CLOCK();
    const int tt = tt_known >= 0 ? tt_known : leaf_verdict(t, ws, depth);
    ARA_PROF(*t.st, 2, tp);
    *is_terminal = tt != TERM_NONE;
    const int nid = expand_node_alloc(t, sp, ws, parent, ci, tt, parent_edge_base);
    ARA_PROF(*t.st, 3, tp);
    return nid;
}

// Fills the prepared-child slot of node X (see TreeDev::prep_board).  Warp-collective, one warp per node, any number
// of nodes of any trees concurrently; runs after the backup of a mini-batch, when nothing else touches the tree.
// Children are expanded in index order, so the slots hold the next kPrepSlots unexpanded children (slot = index mod
// kPrepSlots): a node that is expanded twice within one mini-batch still finds its second child prepared.
template <class WS>
ARA_HD void prepare_child(const TreeDev& t, WS& ws, int X) {
    const NodeHdr& hx = t.hdr[X];
    if (!(hx.flags & NF_HAS_NN) || (hx.flags & NF_TERMINAL)) return;
    const int first = static_cast<int>(hx.no_visit_idx) - 1;
    int depth = -1;
    for (int idx = first; idx < first + kPrepSlots; ++idx) {
        if (idx < 0 || idx >= hx.n_moves) continue;
        const int slot = X * kPrepSlots + (idx % kPrepSlots);
        if (t.child[hx.edge_base + idx] >= 0 || t.prep_ci[slot] == idx) continue;  // expanded / prepared already
        if (depth < 0) {
            // keys of the path root..X, in that order (the repetition scan of a leaf below X needs them)
            depth = 0;
            if (ARA_LANE == 0) {
                for (int n = X; n >= 0; n = t.hdr[n].parent) ++depth;
                if (depth <= kMaxDepth) {
                    int i = depth;
                    for (int n = X; n >= 0; n = t.hdr[n].parent) {
                        --i;
                        ws.path_key[i] = t.hdr[n].key;
                        ws.path_rep[i] = t.hdr[n].repetition;
                    }
                }
            }
            depth = bcast0(depth);
            if (depth > kMaxDepth) return;  // the select loop reports the overflow
        }
        copy_board(&ws.child, &t.board[X]);
        if (ARA_LANE == 0) do_move(ws.child, t.move[hx.edge_base + idx]);
        ARA_WARP_SYNC();
        const int tt = leaf_verdict(t, ws, depth);
        copy_board(&t.prep_board[slot], &ws.child);
        if (ARA_LANE == 0) {
            t.prep_term[slot] = static_cast<uint8_t>(tt);
            t.prep_ci[slot] = static_cast<int16_t>(idx);
        }
        ARA_WARP_SYNC();
    }
}
// item < B: the new leaves of the last mini-batch (their first child); item >= B: the nodes expanded in it
template <class WS>
ARA_HD void prepare_item(const TreeDev& t, const SearchParams& sp, WS& ws, int item) {
    const TreeState& st = *t.st;
    const BatchState& bs = *t.bs;
    if (st.error) return;
    const int B = sp.batch_size;
    if (item < B) {
        if (item < bs.n_new) prepare_child(t, ws, t.new_node[item]);
    } else if (item - B < bs.n_exp) {
        prepare_child(t, ws, t.exp_parent[item - B]);
    }
}

// Second half of the expansion of node `nid` (non-terminal, freshly created by expand_node_seq).  Warp-collective;
// different nodes are processed by different warps concurrently, the edge pool is claimed with one atomic.
template <class WS, class PlaneTarget>
ARA_HD void expand_pending(const TreeDev& t, const SearchParams& sp, WS& ws, int nid, const PlaneTarget* target) {
    copy_board(&ws.child, &t.board[nid]);
    const Board& b = ws.child;
    const int n_moves = gen_legal(b, ws.mg, ws.scratch, ws.legal);
    if (ARA_LANE == 0) {
        TreeState& st = *t.st;
#if defined(__CUDA_ARCH__)
        const int e0 = atomicAdd(&st.n_edges, n_moves);
#else
        const int e0 = st.n_edges;
        st.n_edges += n_moves;
#endif
        NodeHdr& h = t.hdr[nid];
        if (e0 + n_moves > t.max_edges) {
            st.error = 2;
            h.edge_base = 0;
            h.n_moves = 0;
            ws.bcast[0] = -1;
        } else {
            h.edge_base = static_cast<uint32_t>(e0);
            h.n_moves = static_cast<uint16_t>(n_moves);
            h.n_unsolved = static_cast<uint16_t>(n_moves);
            if (h.parent >= 0) t.cbase[t.hdr[h.parent].edge_base + h.parent_ci] = static_cast<uint32_t>(e0);
            ws.bcast[0] = e0;
        }
    }
    ARA_WARP_SYNC();
    const int e0 = ws.bcast[0];
    if (e0 >= 0) {
        const uint32_t e = static_cast<uint32_t>(e0);
        for (int i = ARA_LANE; i < n_moves; i += ARA_WARP_N) {
            const Move m = ws.legal[i];
            t.move[e + i] = m;
            // the policy-vector index is parked in P until the network results arrive (set_probabilities_for_moves)
            const int pidx = policy_map_index(m, b.stm, b.chess960);
#if defined(__CUDA_ARCH__)
            t.P[e + i] = __int_as_float(pidx);
#else
            union { int i; float f; } u;
            u.i = pidx;
            t.P[e + i] = u.f;
#endif
            t.Q[e + i] = kQInit;
            t.N[e + i] = 0;
            t.child[e + i] = -1;
            t.cbase[e + i] = 0;
            t.vl[e + i] = 0;
            t.etype[e + i] = NT_UNSOLVED;
        }
        if (target != nullptr) target->encode(b, sp.mode, sp.input_version);
    }
    ARA_WARP_SYNC();
}

// ------------------------------------------------------------------ scatter of network results into a new node
// prob: this node's row of the soft-maxed policy; value: its value output.  Warp-collective.
template <class WS>
ARA_HD void fill_nn_results(const TreeDev& t, const SearchParams& sp, WS& ws, int nid, float value,
                            const float* prob) {
    NodeHdr& h = t.hdr[nid];
    const int n = h.n_moves;
    const uint32_t e = h.edge_base;
    // set_probabilities_for_moves
    for (int i = ARA_LANE; i < n; i += ARA_WARP_N) {
#if defined(__CUDA_ARCH__)
        const int pidx = __float_as_int(t.P[e + i]);
#else
        union { int i; float f; } u;
        u.f = t.P[e + i];
        const int pidx = u.i;
#endif
        ws.sort_p[i] = prob[pidx];
        ws.scratch[i] = t.move[e + i];
        ws.legal[i] = static_cast<Move>(pidx);  // tie-break key (policy indices are < 65536)
    }
    ARA_WARP_SYNC();
    // apply_temperature (blazeutil.h:78-88): no renormalisation at T == 1.  The power is glibc's powf restated
    // (glibc_flt32.cuh); the normalising sum is SEQUENTIAL, in ascending policy-index order: the reference sums in
    // the order of Stockfish's move generator (through blaze's reduction), which neither this generator nor the
    // oracle's reproduces, so both sides agree on the generator-independent order instead.
    if (sp.node_policy_temperature != 1.0f) {
        const float inv_t = 1.0f / sp.node_policy_temperature;
        float* by_index = reinterpret_cast<float*>(ws.path_key);  // kMaxMoves floats; the descent's path is not live here
        for (int i = ARA_LANE; i < n; i += ARA_WARP_N) {
            const float p = glibc::powf_(ws.sort_p[i], inv_t);
            const Move pi = ws.legal[i];
            int rank = 0;
            for (int j = 0; j < n; ++j) rank += (ws.legal[j] < pi || (ws.legal[j] == pi && j < i)) ? 1 : 0;
            ws.sort_p[i] = p;
            by_index[rank] = p;
        }
        ARA_WARP_SYNC();
        float sum = 0.0f;
        if (ARA_LANE == 0)
            for (int r = 0; r < n; ++r) sum += by_index[r];
        sum = ARA_SHFL(sum, 0);
        for (int i = ARA_LANE; i < n; i += ARA_WARP_N) ws.sort_p[i] = ws.sort_p[i] / sum;
        ARA_WARP_SYNC();
    }
    // sort_moves_by_probabilities: descending prior; the reference's std::sort leaves ties unspecified, we order
    // them by ascending policy-vector index (independent of move-generation order).  Rank counting, O(n^2 / 32).
    for (int i = ARA_LANE; i < n; i += ARA_WARP_N) {
        const float p = ws.sort_p[i];
        const Move pi = ws.legal[i];
        int rank = 0;
        for (int j = 0; j < n; ++j) {
            const float q = ws.sort_p[j];
            rank += (q > p || (q == p && ws.legal[j] < pi)) ? 1 : 0;
        }
        t.P[e + rank] = p;
        t.move[e + rank] = ws.scratch[i];
    }
    if (ARA_LANE == 0) {
        node_set_value(h, value);  // node_assign_value
        h.flags |= NF_HAS_NN;
    }
    ARA_WARP_SYNC();
}

// ------------------------------------------------------------------ Dirichlet noise (libstdc++ gamma_distribution<float>
// over minstd_rand0, util/blazeutil.h:113-124) with an explicit seed.  Lane 0 only.
struct MinStd {
    uint32_t x;
};
ARA_HD uint32_t minstd_next(MinStd& g) {
    g.x = static_cast<uint32_t>((static_cast<uint64_t>(g.x) * 16807ULL) % 2147483647ULL);
    return g.x;
}
ARA_HD float canonical_f(MinStd& g) {
    const float sum = static_cast<float>(minstd_next(g) - 1u);
    float r = sum / 2147483648.0f;
    if (r >= 1.0f) r = 0.99999994f;  // nextafterf(1, 0)
    return r;
}
// std::default_random_engine(seed): minstd_rand0 state = seed mod (2^31 - 1), 0 -> 1; tree `index` of a handle is seeded
// with seed ^ index * golden ratio, so that tree 0 uses the settings' seed itself
ARA_HD uint32_t minstd_seed(unsigned long long seed, int index) {
    const unsigned long long s = seed ^ (static_cast<unsigned long long>(index) * 0x9E3779B97F4A7C15ULL);
    const uint32_t x = static_cast<uint32_t>(s % 2147483647ULL);
    return x == 0 ? 1u : x;
}
ARA_HD float gamma_f(MinStd& g, float alpha) {
    const float malpha = alpha < 1.0f ? alpha + 1.0f : alpha;
    const float a1 = malpha - 1.0f / 3.0f;
    const float a2 = 1.0f / sqrtf(9.0f * a1);
    bool saved_ok = false;
    float saved = 0.0f, u, v, n;
    do {
        do {
            if (saved_ok) {
                saved_ok = false;
                n = saved;
            } else {
                float x, y, r2;
                do {
                    x = static_cast<float>(2.0f * canonical_f(g) - 1.0);
                    y = static_cast<float>(2.0f * canonical_f(g) - 1.0);
                    r2 = x * x + y * y;
                } while (r2 > 1.0 || r2 == 0.0);
                const float mult = sqrtf(-2 * glibc::logf_(r2) / r2);
                saved = x * mult;
                saved_ok = true;
                n = y * mult;
            }
            v = 1.0f + a2 * n;
        } while (v <= 0.0);
        v = v * v * v;
        u = canonical_f(g);
    } while (u > 1.0f - 0.0331 * n * n * n * n && (glibc::logf_(u) > (0.5 * n * n + a1 * (1.0 - v + glibc::logf_(v)))));
    if (alpha == malpha) return a1 * v * 1.0f;
    do u = canonical_f(g);
    while (u == 0.0);
    return glibc::powf_(u, 1.0f / alpha) * a1 * v * 1.0f;
}
// MCTSAgent::evaluate_board_state :311-316: noise on the (sorted) root priors, then open all children.  Lane 0.
ARA_HD void apply_dirichlet_to_root(const TreeDev& t, const SearchParams& sp, WarpScratch& ws) {
    NodeHdr& h = t.hdr[t.st->root];
    const int n = h.n_moves;
    MinStd g;
    g.x = t.st->rng;  // (never 0: minstd_seed)
    float sum = 0.0f;
    for (int i = 0; i < n; ++i) {
        ws.sort_p[i] = gamma_f(g, sp.dirichlet_alpha);
        sum += ws.sort_p[i];
    }
    const float eps = t.st->dirichlet_epsilon;
    for (int i = 0; i < n; ++i) {
        const float noise = ws.sort_p[i] / sum;
        t.P[h.edge_base + i] = (1 - eps) * t.P[h.edge_base + i] + eps * noise;
    }
    t.st->rng = g.x;
    h.no_visit_idx = static_cast<uint16_t>(n);  // fully_expand_node (edges are pre-initialised)
    h.flags |= NF_SORTED | NF_HAS_D;
}

// ------------------------------------------------------------------ epsilon-greedy / epsilon-check exploration
// (searchthread.cpp:124-185, :451-473, :497-501; Centi_Epsilon_Greedy 5 and Centi_Epsilon_Checks 1 in the reference's
// default UCI option set, optionsuci.cpp:89-90).  Lane 0 only, global memory: 6 % of the playouts take this path.
// glibc rand(): r[f] += r[f - 3 mod 31]; output >> 1 (stdlib/random_r.c, TYPE_3); seeding: crand_seed.
ARA_HD void crand_seed(int32_t* r, int32_t* f, unsigned seed) {
    if (seed == 0) seed = 1;
    r[0] = static_cast<int32_t>(seed);
    int32_t word = static_cast<int32_t>(seed);
    for (int i = 1; i < 31; ++i) {
        const long long hi = word / 127773, lo = word % 127773;
        long long w = 16807 * lo - 2836 * hi;
        if (w < 0) w += 2147483647;
        word = static_cast<int32_t>(w);
        r[i] = word;
    }
    int fi = 3, bi = 0;
    for (int i = 0; i < 310; ++i) {
        r[fi] = static_cast<int32_t>(static_cast<uint32_t>(r[fi]) + static_cast<uint32_t>(r[bi]));
        fi = (fi + 1) % 31;
        bi = (bi + 1) % 31;
    }
    *f = fi;
}
ARA_HD int crand_next(TreeState& st) {
    const int fi = st.crand_f, bi = (fi + 28) % 31;
    const uint32_t v = static_cast<uint32_t>(st.crand_r[fi]) + static_cast<uint32_t>(st.crand_r[bi]);
    st.crand_r[fi] = static_cast<int32_t>(v);
    st.crand_f = (fi + 1) % 31;
    return static_cast<int>(v >> 1);
}
// get_random_depth (searchthread.cpp:497-501): ceil(-log2(1 - r / 100.0) - 1) for r = rand() % 100 + 1, tabulated with
// the host libm; r = 100 gives size_t(+inf), which GCC on x86-64 turns into 0 (checked against the compiled reference)
ARA_HD int eps_random_depth(int r) {
    return r <= 50 ? 0 : r <= 75 ? 1 : r <= 87 ? 2 : r <= 93 ? 3 : r <= 96 ? 4 : r <= 98 ? 5 : r == 99 ? 6 : 0;
}
// get_best_action_index(node, fast = true) (node.cpp:1123-1143)
ARA_HD int eps_best_action_fast(const TreeDev& t, const NodeHdr& h) {
    if (h.checkmate_idx != kNoCheckmate) return h.checkmate_idx;
    if (h.node_type == NT_LOSS) {
        int longest = 0, idx = 0;
        for (int i = 0; i < h.n_moves; ++i) {
            const int c = t.child[h.edge_base + i];
            const int e = c >= 0 ? t.hdr[c].end_in_ply : 0;
            if (e > longest) longest = e, idx = i;
        }
        return idx;
    }
    int b = 0;
    for (int i = 1; i < h.no_visit_idx; ++i)
        if (t.N[h.edge_base + i] > t.N[h.edge_base + b]) b = i;
    return b;
}
ARA_HD void eps_increment_no_visit_idx(NodeHdr& h) {  // Node::increment_no_visit_idx (node.cpp:571-580)
    if (h.no_visit_idx < h.n_moves) ++h.no_visit_idx;
}
// random_playout (searchthread.cpp:124-142): the forced child index, or -1 for the ordinary selection
ARA_HD int eps_random_playout(const TreeDev& t, TreeState& st, int cur) {
    NodeHdr& h = t.hdr[cur];
    if (h.n_moves == h.no_visit_idx) {  // is_fully_expanded
        const int idx = static_cast<int>(static_cast<unsigned long long>(crand_next(st)) % static_cast<unsigned long long>(h.n_moves));
        const int c = t.child[h.edge_base + idx];
        if (c < 0 || !(t.hdr[c].flags & NF_HAS_D) || t.hdr[c].node_type == NT_UNSOLVED) return idx;
        return -1;
    }
    const int idx = h.no_visit_idx < h.n_moves - 1 ? h.no_visit_idx : h.n_moves - 1;
    eps_increment_no_visit_idx(h);
    return idx;
}
// select_enhanced_move (searchthread.cpp:451-473): the first unopened move that gives check, opened with everything
// before it; a node is inspected once.  `scratch`: a board to play the moves on.
ARA_HD int eps_select_enhanced_move(const TreeDev& t, int cur, Board& scratch) {
    NodeHdr& h = t.hdr[cur];
    if (!(h.flags & NF_HAS_D) || (h.flags & NF_INSPECTED) || (h.flags & NF_TERMINAL)) return -1;
    for (int c = h.no_visit_idx; c < h.n_moves; ++c) {
        scratch = t.board[cur];
        do_move(scratch, t.move[h.edge_base + c]);
        if (in_check(scratch)) {  // State::gives_check
            for (int i = h.no_visit_idx; i < c + 1; ++i) eps_increment_no_visit_idx(h);
            return c;
        }
    }
    h.flags |= NF_INSPECTED;
    return -1;
}
// The exploration prologue of get_new_child_to_evaluate (searchthread.cpp:171-185): may move the start of the playout
// down the most visited line (get_starting_node, :144-162: the trajectory -- and therefore the backup -- begins THERE)
// and force its first child.  Lane 0 computes, all lanes get (cur, depth, forced); the keys of the skipped levels go to
// ws.path_key / path_rep like the descent's.
ARA_HD void eps_prologue(const TreeDev& t, const SearchParams& sp, WarpScratch& ws, int* cur_io, int* depth_io, int* forced_io) {
    int cur = *cur_io, depth = 0, forced = -1;
    if (ARA_LANE == 0) {
        TreeState& st = *t.st;
        const int egc = sp.epsilon_greedy_counter, ecc = sp.epsilon_checks_counter;
        const bool playout_root = (t.hdr[st.root].flags & NF_HAS_D) != 0;
        int branch = 0;  // 1 random playout, 2 enhanced move
        if (egc && playout_root && crand_next(st) % egc == 0) branch = 1;
        else if (ecc && playout_root && crand_next(st) % ecc == 0) branch = 2;
        if (branch) {
            const int d = eps_random_depth(crand_next(st) % 100 + 1);  // get_starting_node
            for (int k = 0; k < d && depth < kMaxDepth - 1; ++k) {
                const NodeHdr& h = t.hdr[cur];
                const int ci = eps_best_action_fast(t, h);
                const int next = t.child[h.edge_base + ci];
                if (next < 0) break;
                const NodeHdr& nh = t.hdr[next];
                if (!(nh.flags & NF_HAS_D) || nh.visit_sum < static_cast<uint32_t>(egc) || nh.node_type != NT_UNSOLVED) break;
                ws.path_key[depth] = h.key;
                ws.path_rep[depth] = h.repetition;
                cur = next;
                ++depth;
            }
            if (branch == 2) forced = eps_select_enhanced_move(t, cur, ws.child);
            if (forced < 0) forced = eps_random_playout(t, st, cur);
        }
        ws.bcast[0] = cur, ws.bcast[1] = depth, ws.bcast[2] = forced;
    }
    ARA_WARP_SYNC();
    *cur_io = ws.bcast[0];
    *depth_io = ws.bcast[1];
    *forced_io = ws.bcast[2];
    ARA_WARP_SYNC();
}

// ------------------------------------------------------------------ the steps of create_mini_batch shared by both select
// kernels: create_mini_batch_impl below (one warp per tree) and wave_mini_batch (search_wave.cuh, a wavefront of warps)
ARA_HD void clear_batch(BatchState& bs) { bs.n_new = bs.n_coll = bs.n_exp = 0; }

// A search begins on the tree's root: the settings' SearchLimits, Q-value weight and Dirichlet epsilon (root_kernel
// applies the tree's own), every logical thread live, the counters at zero.  pre_nodes: EvalInfo::nodesPreSearch.  Lane 0.
ARA_HD void begin_search(TreeState& st, BatchState& bs, const SearchParams& sp, unsigned pre_nodes) {
    clear_batch(bs);
    bs.done = 0;
    st.live_threads = sp.threads == 2 ? 2 : 1;
    st.limit_simulations = sp.simulations;
    st.limit_nodes = sp.nodes;
    st.q_value_weight = sp.q_value_weight;
    st.dirichlet_epsilon = sp.dirichlet_epsilon;
    st.done = 0;
    st.iterations = 0;
    st.evals = 0;
    st.pre_nodes = pre_nodes;
    st.sum_select_k = 0;
    st.sum_depth = 0;
    for (int i = 0; i < 8; ++i) st.prof[i] = 0;
}

// The tree's own Q-value weight and Dirichlet epsilon (ara_search_set_tree_settings) over the settings' values that
// begin_search put in place; a negative value keeps the settings' value.  After reuse_root / create_root.  Lane 0.
ARA_HD void apply_tree_settings(TreeState& st, float q_value_weight, float dirichlet_epsilon) {
    if (q_value_weight >= 0) st.q_value_weight = q_value_weight;
    if (dirichlet_epsilon >= 0) st.dirichlet_epsilon = dirichlet_epsilon;
}

// the most edges one node can have: the legal-move bound the edge pools are sized by (chess, else drop variants)
ARA_HD int pool_edge_bound(const SearchParams& sp) { return sp.mode == 1 ? 128 : 320; }

// run_search_thread loop condition (searchthread.cpp:326-340, :418-426), checked before every mini-batch.  True: this
// thread makes no mini-batch now and its counters are cleared.  A thread whose condition fails leaves its loop for good,
// like a returning run_search_thread; the search is over when the last thread has left.  Stores on lane 0.
ARA_HD bool thread_loop_ends(const TreeDev& t, const SearchParams& sp) {
    TreeState& st = *t.st;
    BatchState& bs = *t.bs;
    if (st.done || st.error || bs.done) {
        if (ARA_LANE == 0) clear_batch(bs);
        return true;
    }
    const NodeHdr& r = t.hdr[st.root];
    const uint32_t node_count = r.visit_sum - r.free_visits;
    const bool limits_ok = (st.limit_nodes == 0 || node_count < st.limit_nodes) &&
                           (st.limit_simulations == 0 || r.visit_sum < st.limit_simulations);
    // Room for another mini-batch: at most 3B + 8 new nodes, each with at most the per-node edge bound.  (A pool sized
    // for a visit budget can never trip this before the budget does, and there the edge test follows from the node
    // test.  It ends time-limited searches whose pools are full: at their size or cap, or, for pools mapped as the tree
    // grows, where growth stopped short of the device's free memory.)
    const int grow = 3 * sp.batch_size + 8;
    const bool pool_ok = st.n_nodes + grow <= t.max_nodes && st.n_edges <= t.max_edges - grow * pool_edge_bound(sp);
    if (!(limits_ok && r.node_type == NT_UNSOLVED) || r.n_moves <= 1 || !pool_ok) {
        if (ARA_LANE == 0) {
            bs.done = 1;
            clear_batch(bs);
            if (--st.live_threads <= 0) st.done = 1;
        }
        return true;
    }
    return false;
}

// A step of the descent from node `cur` (header `h`) to its child `ci`, at ply `depth` below the root: the trajectory
// entry, and the node's key for the repetition scan.  Indexed by the ply below the root even when the trajectory starts
// deeper (EPS): the backup kernel gives every ply its own lane, which is what keeps two trajectories' updates of one node
// in order.  Lane 0.
ARA_HD void record_step(WarpScratch& ws, int depth, int cur, int ci, const NodeHdr& h) {
    ws.traj_node[depth] = cur;
    ws.traj_ci[depth] = static_cast<uint16_t>(ci);
    ws.traj_edge[depth] = h.edge_base + static_cast<uint32_t>(ci);
    ws.path_key[depth] = h.key;
    ws.path_rep[depth] = h.repetition;
}

// The position of a new leaf, child `ci` of node `cur` (header `h`), into ws.child.  It was usually prepared by a
// parallel warp after the previous mini-batch (prepare_child), and then its verdict is returned as well; otherwise
// (second expansion of a node within one mini-batch) the move is made here and -1 returned: leaf_verdict is still to
// run.  *slot_out / *prepared_out: the prepared-child slot, for commit_parent.  Warp-collective.
ARA_HD int leaf_board(const TreeDev& t, WarpScratch& ws, int cur, int ci, const NodeHdr& h, int* slot_out,
                      bool* prepared_out) {
    // (slot index, verdict and board are fetched together, speculatively: one round trip)
    const int slot = cur * kPrepSlots + (ci % kPrepSlots);
    const int slot_ci = t.prep_ci[slot];
    const int slot_tt = t.prep_term[slot];
#if defined(__CUDA_ARCH__)
    uint4 slot_b = make_uint4(0u, 0u, 0u, 0u);
    if (ARA_LANE < 8) slot_b = reinterpret_cast<const uint4*>(&t.prep_board[slot])[ARA_LANE];
#endif
    const bool prepared = slot_ci == ci;
    *slot_out = slot;
    *prepared_out = prepared;
    if (prepared) {
#if defined(__CUDA_ARCH__)
        if (ARA_LANE < 8) reinterpret_cast<uint4*>(&ws.child)[ARA_LANE] = slot_b;
        ARA_WARP_SYNC();
#else
        ws.child = t.prep_board[slot];
#endif
        return slot_tt;
    }
    copy_board(&ws.child, &t.board[cur]);
    if (ARA_LANE == 0) do_move(ws.child, t.move[h.edge_base + ci]);
    ARA_WARP_SYNC();
    return -1;
}

// The parent's share of the expansion of one of its children: increment_no_visit_idx opens the next-best sibling (its
// edge slots are pre-initialised), the prepared slot the child came from is used up, and the parent is listed in
// exp_parent for prepare_item.  Lane 0; n_exp counts the mini-batch's exp_parent entries.
ARA_HD void commit_parent(const TreeDev& t, int cur, const NodeHdr& h, int slot, bool prepared, int& n_exp, int B) {
    if (h.no_visit_idx < h.n_moves) t.hdr[cur].no_visit_idx = static_cast<uint16_t>(h.no_visit_idx + 1);
    if (prepared) t.prep_ci[slot] = -1;
    if (n_exp < 3 * B) t.exp_parent[n_exp++] = cur;
}

// The end of a playout of `type` (0 new leaf, 1 collision, 2 terminal) that reached `leaf`, `depth` plies below the
// root, with its trajectory in ws.traj_* from ply `start` on.  A terminal is backed up at once, for free, sequentially
// leaf -> root because the MCTS solver propagates bottom-up; the others become trajectory `row` of the mini-batch, which
// backup_results backs up or reverts.  Warp-collective.
ARA_HD void store_trajectory(const TreeDev& t, const SearchParams& sp, WarpScratch& ws, int type, int row, int start,
                             int depth, int leaf) {
    if (type == 2) {
        if (ARA_LANE == 0) {
            t.st->sum_depth += static_cast<unsigned long long>(depth);
            backup_value(t, sp, node_value(t.hdr[leaf]), ws.traj_node + start, ws.traj_ci + start, depth - start, true,
                         sp.mcts_solver != 0);
        }
        return;
    }
    for (int i = start + ARA_LANE; i < depth; i += ARA_WARP_N) {
        t.traj_node[row * kMaxDepth + i] = ws.traj_node[i];
        t.traj_ci[row * kMaxDepth + i] = ws.traj_ci[i];
        t.traj_edge[row * kMaxDepth + i] = ws.traj_edge[i];
    }
    if (ARA_LANE == 0) {
        t.st->sum_depth += static_cast<unsigned long long>(depth);
        t.traj_len[row] = depth;
        if (type == 0) t.new_node[row] = leaf;
    }
}

// What the mini-batch hands to the steps after the select, and the search's counters.  Lane 0.
ARA_HD void end_mini_batch(TreeState& st, BatchState& bs, int n_new, int n_coll, int n_exp) {
    bs.n_new = n_new;
    bs.n_coll = n_coll;
    bs.n_exp = n_exp;
    st.iterations++;
    st.evals += static_cast<unsigned>(n_new);
}

// ------------------------------------------------------------------ one mini-batch: SearchThread::create_mini_batch
// Sequential per tree (one warp).  New leaves are only created here (expand_node_seq); their move lists, edges and
// input planes are produced afterwards by expand_pending, one warp per leaf.
// EPS: epsilon-greedy / epsilon-check exploration compiled in (its own instantiation: the ordinary descent stays as lean
// as it is).  With it a playout may start below the root: `depth` counts plies below the root (path keys, repetition),
// `skipped` the plies above the trajectory (which is what is stored and backed up).
template <bool EPS>
ARA_HD void create_mini_batch_impl(const TreeDev& t, const SearchParams& sp, WarpScratch& ws) {
    if (thread_loop_ends(t, sp)) return;
    TreeState& st = *t.st;
    const int B = sp.batch_size;
    int n_new = 0, n_coll = 0, n_term = 0;
    int n_exp = 0;  // lane 0's count of exp_parent entries
    while (n_new < B && n_coll != B && n_term < 2 * B) {
        int cur = st.root, depth = 0, type = -1, leaf = -1;  // type: 0 new, 1 collision, 2 terminal
        int forced = -1, skipped = 0;  // EPS: first child forced by the prologue; plies skipped above the trajectory
        long long tq = ARA_CLOCK();
        if (EPS) {
            eps_prologue(t, sp, ws, &cur, &depth, &forced);
            skipped = depth;
        }
        NodeHdr h;
        load_hdr(&h, &t.hdr[cur]);
        EdgeRegs pre = load_edge(t, h.edge_base + ARA_LANE);
        for (;;) {
            if (depth >= kMaxDepth) {
                if (ARA_LANE == 0) st.error = 3;
                type = -2;
                break;
            }
            const SelectStep step = EPS ? select_and_visit(t, sp, cur, h, pre, forced) : select_and_visit(t, sp, cur, h, pre);
            forced = -1;
            const int ci = step.ci;
            const int next = step.child;
            if (ARA_LANE == 0) record_step(ws, depth, cur, ci, h);
            ARA_WARP_SYNC();
            depth++;
            if (next < 0) {
                ARA_PROF(st, 0, tq);
                int slot = 0;
                bool prepared = false;
                const int tt_known = leaf_board(t, ws, cur, ci, h, &slot, &prepared);
                if (ARA_LANE == 0) commit_parent(t, cur, h, slot, prepared, n_exp, B);
                ARA_WARP_SYNC();
                ARA_PROF(st, 1, tq);
                int is_term = 0;
                leaf = expand_node_seq(t, sp, ws, cur, ci, depth, &is_term, tt_known, h.edge_base);
                if (leaf < 0) {
                    type = -2;
                    break;
                }
                type = is_term ? 2 : 0;
                tq = ARA_CLOCK();
                break;
            }
            if (step.ch.flags & NF_TERMINAL) {
                type = 2;
                leaf = next;
                break;
            }
            if (!(step.ch.flags & NF_HAS_NN)) {
                type = 1;
                leaf = next;
                break;
            }
            cur = next;
            h = step.ch;
            pre = step.pre;
        }
        if (type == -2) break;
        if (type != 0) ARA_PROF(st, 0, tq);
        const int row = type == 1 ? B + n_coll : n_new;
        store_trajectory(t, sp, ws, type, row, skipped, depth, leaf);
        if (EPS && type != 2 && ARA_LANE == 0) t.traj_start[row] = skipped;  // (stays 0 without the exploration)
        ARA_WARP_SYNC();
        ARA_PROF(st, type == 2 ? 5 : 6, tq);
        if (type == 2) ++n_term;
        else if (type == 1) ++n_coll;
        else ++n_new;
    }
    if (ARA_LANE == 0) end_mini_batch(st, *t.bs, n_new, n_coll, n_exp);
    ARA_WARP_SYNC();
}

template <bool EPS>
ARA_HD void create_mini_batch(const TreeDev& t_in, const SearchParams& sp, WarpScratch& ws) {
    // every `st.x += ...` of the sequential loop would otherwise be a global-memory round trip on the critical path
    TreeDev t = t_in;
    if (ARA_LANE == 0) ws.st_local = *t_in.st;
    ARA_WARP_SYNC();
    t.st = &ws.st_local;
    create_mini_batch_impl<EPS>(t, sp, ws);
    ARA_WARP_SYNC();
    if (ARA_LANE == 0) *t_in.st = ws.st_local;
    ARA_WARP_SYNC();
}

// set_nn_results_to_child_nodes (searchthread.cpp:301-310) for new leaf `b` of the tree: one warp per leaf.
template <class WS>
ARA_HD void scatter_pending(const TreeDev& t, const SearchParams& sp, WS& ws, int b, const float* values,
                            const float* probs, int n_labels) {
    const int slot = t.slot_base + b;
    fill_nn_results(t, sp, ws, t.new_node[b], values[slot], probs + static_cast<size_t>(slot) * n_labels);
}

// backup_value_outputs + backup_collisions (searchthread.cpp:312-324): one warp per tree.
// `values`: the network's value output; the new leaf b of this tree sits in row slot_base + b (a fresh leaf has
// real_visits 1 and value_sum double(v), so its node value is the network value itself).  Reads nothing the scatter
// step writes and writes nothing the scatter / prepare steps read, so it may run beside them.
ARA_HD void backup_results(const TreeDev& t, const SearchParams& sp, const float* values) {
    const int B = sp.batch_size;
    const int n_new = t.bs->n_new, n_coll = t.bs->n_coll;
    // backup_value (node.h:819-843) without solver: the levels of one trajectory are distinct nodes/edges, so lane d
    // updates depth d of every trajectory, in trajectory order (value sign alternates with the distance to the leaf).
    // Backups that share a node or an edge share its depth and therefore its lane, which preserves the reference's
    // update order node by node and edge by edge.  The node sums and the edge statistics a lane is working on stay in
    // registers while consecutive trajectories pass through the same node / edge (always true at the root); indices
    // are loaded two trajectories ahead and the statistics one trajectory ahead, so that the per-trajectory chain is
    // the FP64 arithmetic alone instead of four dependent L2 round trips.
    int max_len = 0;
    for (int b = ARA_LANE; b < n_new; b += ARA_WARP_N) max_len = t.traj_len[b] > max_len ? t.traj_len[b] : max_len;
    max_len = ARA_REDUCE_MAX(max_len);
    for (int d0 = 0; d0 < max_len; d0 += ARA_WARP_N) {
        const int d = d0 + ARA_LANE;
        int c_nid = -1;
        double c_vsum = 0.0;
        uint32_t c_rv = 0;
        uint32_t c_e = 0xffffffffu, c_n = 0;
        float c_q = 0.0f;
        uint8_t c_vl = 0;
        // software pipeline: the indices of trajectory b+2 are requested while b is processed (unconditionally: the
        // trajectory arrays are dense, entries beyond a trajectory's length are simply not used), and the node sums
        // and edge statistics of trajectory b+1 are LOADED (p_*) while b's FP64 chain runs.  A pre-loaded value is
        // current when it is used: this lane is the only writer of its depth's nodes and edges, it writes them only
        // when its register copy moves on to another node / edge, and that store is issued before the pre-load of the
        // same iteration; if b+1 stays on b's node / edge the register copy is used and the pre-load is ignored.
        const int dd = d < kMaxDepth ? d : kMaxDepth - 1;
        const float* leaf_values = values + t.slot_base;
        int len_n = n_new > 0 ? t.traj_len[0] : 0, len_nn = n_new > 1 ? t.traj_len[1] : 0;
        int start_n = n_new > 0 ? t.traj_start[0] : 0, start_nn = n_new > 1 ? t.traj_start[1] : 0;
        float leaf_n = n_new > 0 ? leaf_values[0] : 0.0f, leaf_nn = n_new > 1 ? leaf_values[1] : 0.0f;
        int nid_n = n_new > 0 ? t.traj_node[dd] : -1, nid_nn = n_new > 1 ? t.traj_node[kMaxDepth + dd] : -1;
        uint32_t e_n = n_new > 0 ? t.traj_edge[dd] : 0, e_nn = n_new > 1 ? t.traj_edge[kMaxDepth + dd] : 0;
#if defined(__CUDA_ARCH__)
        // further ahead: the lines of trajectories b+3 / b+4 are pulled into L1 (prefetch hints, no registers tied up), so
        // that the pre-loads above find them there.  This lane is the only writer of those lines; a load after its own
        // store returns the stored value whatever the hint fetched.
        int nid_3 = n_new > 2 ? t.traj_node[2 * kMaxDepth + dd] : -1, nid_4 = n_new > 3 ? t.traj_node[3 * kMaxDepth + dd] : -1;
        uint32_t e_3 = n_new > 2 ? t.traj_edge[2 * kMaxDepth + dd] : 0, e_4 = n_new > 3 ? t.traj_edge[3 * kMaxDepth + dd] : 0;
#endif
        double p_vsum = 0.0;
        uint32_t p_rv = 0, p_n = 0;
        float p_q = 0.0f;
        uint8_t p_vl = 0;
        if (n_new > 0 && d < len_n && d >= start_n) {  // pre-load of trajectory 0
            p_vsum = t.hdr[nid_n].value_sum, p_rv = t.hdr[nid_n].real_visits;
            p_q = t.Q[e_n], p_n = t.N[e_n], p_vl = t.vl[e_n];
        }
        for (int b = 0; b < n_new; ++b) {
            const int len = len_n, start = start_n, nid = nid_n;
            const uint32_t e = e_n;
            const float leaf_v = leaf_n;
            const double l_vsum = p_vsum;
            const uint32_t l_rv = p_rv, l_n = p_n;
            const float l_q = p_q;
            const uint8_t l_vl = p_vl;
            len_n = len_nn, start_n = start_nn, leaf_n = leaf_nn, nid_n = nid_nn, e_n = e_nn;
#if defined(__CUDA_ARCH__)
            if (b + 2 < n_new) {
                len_nn = t.traj_len[b + 2];
                start_nn = t.traj_start[b + 2];
                leaf_nn = leaf_values[b + 2];
                nid_nn = nid_3, e_nn = e_3;
            }
            nid_3 = nid_4, e_3 = e_4;
            if (b + 4 < n_new) {
                nid_4 = t.traj_node[(b + 4) * kMaxDepth + dd];
                e_4 = t.traj_edge[(b + 4) * kMaxDepth + dd];
            }
            if (b + 3 < n_new && nid_3 >= 0 && d < kMaxDepth) {  // (nid_3 / e_3: trajectory b+3, indices requested two iterations ago)
                asm volatile("prefetch.global.L1 [%0];" ::"l"(&t.hdr[nid_3].value_sum));
                asm volatile("prefetch.global.L1 [%0];" ::"l"(&t.Q[e_3]));
                asm volatile("prefetch.global.L1 [%0];" ::"l"(&t.N[e_3]));
                asm volatile("prefetch.global.L1 [%0];" ::"l"(&t.vl[e_3]));
            }
#else
            if (b + 2 < n_new) {
                len_nn = t.traj_len[b + 2];
                start_nn = t.traj_start[b + 2];
                leaf_nn = leaf_values[b + 2];
                nid_nn = t.traj_node[(b + 2) * kMaxDepth + dd];
                e_nn = t.traj_edge[(b + 2) * kMaxDepth + dd];
            }
#endif
            const bool active = d < len && d >= start;
            if (active) {  // move the register copies on to this trajectory's node / edge (stores first)
                if (nid != c_nid) {
                    if (c_nid >= 0) t.hdr[c_nid].value_sum = c_vsum, t.hdr[c_nid].real_visits = c_rv;
                    c_nid = nid;
                    c_vsum = l_vsum;
                    c_rv = l_rv;
                }
                if (e != c_e) {
                    if (c_e != 0xffffffffu) t.Q[c_e] = c_q, t.vl[c_e] = c_vl;
                    c_e = e;
                    c_q = l_q;
                    c_n = l_n;
                    c_vl = l_vl;
                }
            }
            if (b + 1 < n_new && d < len_n && d >= start_n) {  // pre-load of trajectory b+1, in flight during the arithmetic below
                p_vsum = t.hdr[nid_n].value_sum, p_rv = t.hdr[nid_n].real_visits;
                p_q = t.Q[e_n], p_n = t.N[e_n], p_vl = t.vl[e_n];
            }
            if (!active) continue;
            const float v = ((len - d) & 1) ? -leaf_v : leaf_v;
            // revert_virtual_loss_and_update (node.h:199-246) on the register copies
            c_vsum += v;
            ++c_rv;
            if (c_n == 1) {
                c_q = v;
            } else {
                const int style = virtual_style_of(sp, c_n);
                if (style == VS_VIRTUAL_LOSS) {
                    c_q = static_cast<float>((static_cast<double>(c_q) * c_n + 1 + v) / c_n);
                } else if (style == VS_VIRTUAL_VISIT) {
                    const uint32_t real = c_n - c_vl;
                    c_q = static_cast<float>((static_cast<double>(c_q) * real + v) / (real + 1));
                }
            }
            --c_vl;
        }
        if (c_nid >= 0) t.hdr[c_nid].value_sum = c_vsum, t.hdr[c_nid].real_visits = c_rv;
        if (c_e != 0xffffffffu) t.Q[c_e] = c_q, t.vl[c_e] = c_vl;
    }
    ARA_WARP_SYNC();
    for (int c = 0; c < n_coll; ++c) {
        const int row = B + c;
        const int len = t.traj_len[row];
        for (int i = t.traj_start[row] + ARA_LANE; i < len; i += ARA_WARP_N)
            revert_virtual_loss(t, sp, t.traj_node[row * kMaxDepth + i], t.traj_ci[row * kMaxDepth + i]);
    }
    ARA_WARP_SYNC();
    // (n_new / n_coll stay as the select step left them: the scatter and prepare steps, which may run concurrently,
    // read n_new; the next select step overwrites both)
}

// Root creation: MCTSAgent::create_new_root_node (mctsagent.cpp:180-196), first half (before the network call).
ARA_HD void create_root(const TreeDev& t, const SearchParams& sp, WarpScratch& ws, const Board* root_board) {
    copy_board(&ws.child, root_board);
    if (ARA_LANE == 0) {
        TreeState& st = *t.st;
        st.root = 0;
        st.next_root = -1;
        st.next_valid = 0;
        st.n_nodes = 0;
        st.n_edges = 0;
        st.error = 0;
        begin_search(st, *t.bs, sp, 0);
    }
    ARA_WARP_SYNC();
    int is_term = 0;
    // repetition info is recomputed from the game history (depth 0 = history only)
    const int nid = expand_node_seq(t, sp, ws, -1, -1, 0, &is_term);
    if (ARA_LANE == 0 && nid == 0) {
        TreeState& st = *t.st;
        if (is_term) {
            st.done = 1;
        } else {
            t.bs->n_new = 1;  // the root is the single "new node" of the first network call
            t.new_node[0] = 0;
            t.traj_len[0] = 0;
            st.evals = 1;
        }
    }
    ARA_WARP_SYNC();
}
// MCTSAgent::apply_move_to_tree + pick_next_node (mctsagent.cpp:230-247): the child behind `move` becomes the candidate
// root of the next search; a second call (the opponent's reply) descends once more.  Lane 0.
ARA_HD void advance_root(const TreeDev& t, Move move) {
    TreeState& st = *t.st;
    const int base = st.next_valid ? st.next_root : (st.n_nodes > 0 ? st.root : -1);
    st.next_root = -1;
    st.next_valid = 1;
    if (base < 0) return;
    const NodeHdr& h = t.hdr[base];
    if (!(h.flags & NF_HAS_D) || !(h.flags & NF_HAS_NN)) return;  // is_playout_node
    for (int i = 0; i < h.n_moves; ++i)
        if (t.move[h.edge_base + i] == move) {
            st.next_root = t.child[h.edge_base + i];
            break;
        }
}

// MCTSAgent::init_root_node / get_root_node_from_tree (mctsagent.cpp:113-160): if the candidate root is the searched
// position, is a playout node with visits of its own and the pools have room for another search, the subtree is kept
// (make_to_root) and the search continues on its statistics.  Returns 1 if the tree is reused.  Warp-uniform.
// room in the pools for another search on top of n_nodes / n_edges entries in use
ARA_HD bool pools_have_room(const SearchParams& sp, int max_nodes, int max_edges, int n_nodes, long long n_edges) {
    // a time-limited search has no visit budget: it keeps the tree only while half of the pool is still free
    const unsigned limit = sp.simulations ? sp.simulations : sp.nodes;
    const unsigned budget = limit ? limit : static_cast<unsigned>(max_nodes / 2);
    return n_nodes + static_cast<long long>(budget) + 4 * sp.batch_size + 64 <= max_nodes &&
           n_edges + (static_cast<long long>(budget) + 4 * sp.batch_size + 64) * pool_edge_bound(sp) <= max_edges;
}
// the candidate root of the next search (ara_search_apply_move) if it is the searched position and a playout node with
// visits of its own, else -1
ARA_HD int kept_subtree_root(const TreeDev& t, const Board* root_board) {
    const TreeState& st = *t.st;
    const int cand = (st.next_valid && st.n_nodes > 0 && !st.error) ? st.next_root : -1;
    if (cand < 0) return -1;
    const NodeHdr& h = t.hdr[cand];
    const bool ok = h.key == root_board->key && (h.flags & NF_HAS_D) && (h.flags & NF_HAS_NN) && h.visit_sum - h.free_visits > 0;
    return ok ? cand : -1;
}
// (room: whether the pools have room for another search on top of the subtree -- decided by the host for pools mapped
// as the tree grows, which measure it against their reservation)
ARA_HD int reuse_root(const TreeDev& t, const SearchParams& sp, const Board* root_board, bool room) {
    TreeState& st = *t.st;
    const int cand = kept_subtree_root(t, root_board);
    const int ok = cand >= 0 && room ? 1 : 0;
    ARA_WARP_SYNC();
    if (ARA_LANE == 0) {
        st.next_root = -1;
        st.next_valid = 0;
        if (ok) {
            NodeHdr& h = t.hdr[cand];
            st.root = cand;
            h.parent = -1;  // make_to_root: the path walks of prepare_child stop here
            begin_search(st, *t.bs, sp, h.visit_sum - h.free_visits);
            if ((h.flags & NF_TERMINAL) || h.n_moves == 0) st.done = 1;
        }
    }
    ARA_WARP_SYNC();
    return ok;
}

ARA_HD int reuse_root(const TreeDev& t, const SearchParams& sp, const Board* root_board) {
    return reuse_root(t, sp, root_board, pools_have_room(sp, t.max_nodes, t.max_edges, t.st->n_nodes, t.st->n_edges));
}

// The root phase of a tree left out of a go (ara_search_set_active), in place of reuse_root / create_root: the tree, its
// Dirichlet generator and a candidate root kept by advance_root stay as they are.  `done` makes every later kernel of
// the go pass the tree by; the mini-batch counters are cleared because the root phase's scatter / backup / prepare steps
// and pack_kernel read them, and left over from the tree's last mini-batch they would apply that batch again.  Lane 0.
ARA_HD void idle_root(const TreeDev& t) {
    t.st->done = 1;
    clear_batch(*t.bs);
}

// second half: after expand_pending + network + scatter_pending + backup_results (root trajectory is empty)
ARA_HD void finalize_root(const TreeDev& t, const SearchParams& sp, WarpScratch& ws) {
    if (ARA_LANE == 0 && !t.st->done && !t.st->error) {
        NodeHdr& h = t.hdr[t.st->root];
        h.flags |= NF_HAS_D | NF_SORTED;  // prepare_node_for_visits
        if (t.st->dirichlet_epsilon > 0.009f && h.n_moves > 1) apply_dirichlet_to_root(t, sp, ws);
    }
    ARA_WARP_SYNC();
}

// ------------------------------------------------------------------ root statistics for the ThreadManager heuristics
// RootTimeStats (time_manager.h) of the tree's root.  Lane 0.
ARA_HD void collect_time_stats(const TreeDev& t, RootTimeStats* r) {
    const TreeState& st = *t.st;
    const NodeHdr& h = t.hdr[st.root];
    r->node_count = h.visit_sum - h.free_visits;
    r->first_visits = r->second_visits = 0;
    r->q_first = r->q_second = 0.0f;
    r->max_q_is_max_visits = 0;
    r->value_eval = h.real_visits ? node_value(h) : 0.0f;
    r->valid = 0;
    const int k = h.no_visit_idx;
    if (st.n_nodes <= 0 || k <= 0 || !(h.flags & NF_HAS_D)) return;
    r->valid = 1;
    const uint32_t e = h.edge_base;
    // first_and_second_max (util/blazeutil.h:149-177): strict '>' scans, so the first maximum wins
    uint32_t first = t.N[e], second = 0;
    int a1 = 0, a2 = 0, best_q = 0;
    for (int i = 1; i < k; ++i) {
        const uint32_t n = t.N[e + i];
        if (n > first) {
            second = first, a2 = a1;
            first = n, a1 = i;
        } else if (n > second) {
            second = n, a2 = i;
        }
        if (t.Q[e + i] > t.Q[e + best_q]) best_q = i;
    }
    r->max_q_is_max_visits = best_q == a1;
    r->q_first = t.Q[e + a1];
    r->q_second = t.Q[e + a2];
    const int c1 = t.child[e + a1], c2 = t.child[e + a2];
    if (c1 >= 0 && (t.hdr[c1].flags & NF_HAS_D)) first -= t.hdr[c1].free_visits;
    if (c2 >= 0 && (t.hdr[c2].flags & NF_HAS_D)) second -= t.hdr[c2].free_visits;
    r->first_visits = first;
    r->second_visits = second;
    if ((h.flags & NF_SORTED) && h.visit_sum != 1) {
        if (h.node_type == NT_WIN) r->value_eval = 1.0f;
        else if (h.node_type == NT_DRAW) r->value_eval = 0.0f;
        else if (h.node_type == NT_LOSS) r->value_eval = -1.0f;
        else r->value_eval = t.Q[e + a1];
    }
}

// ------------------------------------------------------------------ results: the view of one node, update_eval_info
ARA_HD void collect_node_view(const TreeDev& t, int nid, NodeView* v) {  // lane-strided; nid < 0 = the current root
    const TreeState& st = *t.st;
    const int id = nid < 0 ? st.root : nid;
    const bool ok = id >= 0 && id < st.n_nodes;
    if (ARA_LANE == 0) {
        v->node_id = ok ? id : -1;
        v->n_moves = 0;
    }
    ARA_WARP_SYNC();
    if (!ok) return;
    const NodeHdr& h = t.hdr[id];
    if (ARA_LANE == 0) {
        v->parent = h.parent;
        v->parent_child_idx = h.parent_ci;
        v->n_moves = h.n_moves;
        v->no_visit_idx = (h.flags & NF_HAS_D) ? h.no_visit_idx : 0;
        v->node_type = h.node_type;
        v->flags = h.flags;
        v->checkmate_idx = h.checkmate_idx;
        v->end_in_ply = h.end_in_ply;
        v->n_unsolved = h.n_unsolved;
        v->repetition = h.repetition;
        v->pad_ = 0;
        v->visit_sum = h.visit_sum;
        v->real_visits = h.real_visits;
        v->free_visits = h.free_visits;
        v->value = h.real_visits ? node_value(h) : 0.0f;
        v->value_sum = h.value_sum;
        v->key = h.key;
    }
    const bool has_edges = (h.flags & NF_HAS_NN) != 0;  // edges exist once the node has been expanded and evaluated
    for (int i = ARA_LANE; i < h.n_moves; i += ARA_WARP_N) {
        const uint32_t e = h.edge_base + static_cast<uint32_t>(i);
        v->moves[i] = t.move[e];
        v->child[i] = has_edges ? t.child[e] : -1;
        v->visits[i] = has_edges ? t.N[e] : 0;
        v->q[i] = has_edges ? t.Q[e] : kQInit;
        v->prior[i] = has_edges ? t.P[e] : 0.0f;
        v->vl[i] = has_edges ? t.vl[e] : 0;
        v->child_type[i] = has_edges ? t.etype[e] : NT_UNSOLVED;
    }
}

ARA_HD int mcts_policy(const TreeDev& t, const SearchParams& sp, const NodeHdr& h, double* out) {  // node.cpp:1070-1109
    const int k = h.no_visit_idx;
    const uint32_t e = h.edge_base;
    for (int i = 0; i < h.n_moves; ++i) out[i] = 0.0;
    if (h.node_type == NT_WIN) {
        for (int i = 0; i < k; ++i) {
            const int c = t.child[e + i];
            if (c >= 0 && (t.hdr[c].flags & NF_HAS_D) && t.hdr[c].node_type == NT_LOSS) out[i] = 1.0;
        }
    } else if (h.node_type == NT_LOSS) {
        int longest = 0, end = 0;
        for (int i = 0; i < k; ++i) {
            const int c = t.child[e + i];
            if (c >= 0 && (t.hdr[c].flags & NF_HAS_D) && t.hdr[c].end_in_ply > end) end = t.hdr[c].end_in_ply, longest = i;
        }
        out[longest] = 1.0;
    } else {
        for (int i = 0; i < k; ++i) out[i] = static_cast<double>(t.N[e + i]);
        if (h.n_unsolved != h.n_moves && h.node_type != NT_LOSS)
            for (int i = 0; i < k; ++i) {
                const int c = t.child[e + i];
                if (c >= 0 && (t.hdr[c].flags & NF_HAS_D) && t.hdr[c].node_type == NT_WIN) out[i] = 0;
            }
        const float q_value_weight = t.st->q_value_weight;
        if (q_value_weight > 0) {
            int best_q = 0;
            for (int i = 1; i < k; ++i)
                if (t.Q[e + i] > t.Q[e + best_q]) best_q = i;
            double first = out[0], second = 2.2250738585072014e-308;
            int first_arg = 0, second_arg = 0;
            for (int i = 1; i < k; ++i) {
                if (out[i] > first) {
                    second = first;
                    second_arg = first_arg;
                    first = out[i];
                    first_arg = i;
                } else if (out[i] > second) {
                    second = out[i];
                    second_arg = i;
                }
            }
            const int best = first_arg;
            if (sp.q_veto_delta != 0 && best_q != best && t.Q[e + best_q] > t.Q[e + best] + sp.q_veto_delta && t.N[e + best_q] > 1) {
                if (out[best] > out[best_q]) {
                    const double save = out[best_q];
                    out[best_q] = out[best];
                    out[best] = save;
                }
            } else if (best != second_arg && t.Q[e + second_arg] > t.Q[e + best]) {
                const float q_diff = t.Q[e + second_arg] - t.Q[e + best];
                out[second_arg] += q_diff * q_value_weight * out[best];
            }
        }
    }
    double sum = 0;
    for (int i = 0; i < k; ++i) sum += out[i];
    for (int i = 0; i < k; ++i) out[i] /= sum;
    int b = 0;
    for (int i = 1; i < k; ++i)
        if (out[i] > out[b]) b = i;
    return b;
}
ARA_HD int best_action_index(const TreeDev& t, const SearchParams& sp, const NodeHdr& h, bool fast, double* tmp) {
    if (h.checkmate_idx != kNoCheckmate) return h.checkmate_idx;
    if (h.node_type == NT_LOSS) {
        int longest = 0, idx = 0;
        for (int i = 0; i < h.n_moves; ++i) {
            const int c = t.child[h.edge_base + i];
            if (c >= 0 && t.hdr[c].end_in_ply > longest) longest = t.hdr[c].end_in_ply, idx = i;
        }
        return idx;
    }
    if (fast) {
        int b = 0;
        for (int i = 1; i < h.no_visit_idx; ++i)
            if (t.N[h.edge_base + i] > t.N[h.edge_base + b]) b = i;
        return b;
    }
    return mcts_policy(t, sp, h, tmp);
}
ARA_HD float value_display(const NodeHdr& h) {
    if (h.node_type == NT_WIN) return 1.0f;
    if (h.node_type == NT_LOSS) return -1.0f;
    if (h.node_type == NT_DRAW) return 0.0f;
    return node_value(h);
}
ARA_HD void collect_result(const TreeDev& t, const SearchParams& sp, SearchResult* r) {  // lane 0
    const TreeState& st = *t.st;
    const NodeHdr& h = t.hdr[t.st->root];
    r->error = st.error;
    r->tree_nodes = st.n_nodes;
    r->nodes_pre_search = st.pre_nodes;
    r->iterations = st.iterations;
    r->evals = st.evals;
    r->sum_select_k = st.sum_select_k;
    r->sum_depth = st.sum_depth;
    r->n_moves = h.n_moves;
    const bool has_d = (h.flags & NF_HAS_D) != 0;
    r->no_visit_idx = has_d ? h.no_visit_idx : 0;
    r->node_type = has_d ? h.node_type : NT_UNSOLVED;
    r->visit_sum = has_d ? h.visit_sum : 0;
    r->free_visits = has_d ? h.free_visits : 0;
    r->root_value = h.real_visits ? node_value(h) : 0.0f;
    r->best_idx = -1;
    r->best_move_q = 0.0f;
    r->pv_len = 0;
    if (h.n_moves == 0 || (h.flags & NF_TERMINAL)) return;
    const uint32_t e = h.edge_base;
    for (int i = 0; i < h.n_moves; ++i) {
        r->moves[i] = t.move[e + i];
        r->visits[i] = i < h.no_visit_idx ? t.N[e + i] : 0;
        r->q[i] = i < h.no_visit_idx ? t.Q[e + i] : -1.0f;
        r->prior[i] = t.P[e + i];
        r->policy[i] = 0.0;
    }
    if (!(h.flags & NF_HAS_NN)) return;
    // get_best_action_index(root, fast = false) and the posterior (evalinfo.cpp:199-206)
    int bi = 0;
    if (h.n_moves == 1) {
        r->policy[0] = 1.0;
    } else {
        bi = mcts_policy(t, sp, h, r->policy);
    }
    if (h.checkmate_idx != kNoCheckmate) bi = h.checkmate_idx;
    else if (h.node_type == NT_LOSS) bi = best_action_index(t, sp, h, true, nullptr);
    r->best_idx = bi;
    // set_eval_for_single_pv (evalinfo.cpp:123-178) + get_principal_variation (node.cpp:1111-1121)
    int n = 0;
    r->pv[n++] = t.move[e + bi];
    int c = t.child[e + bi];
    if (c < 0) {
        r->best_move_q = kQInit;
    } else {
        const NodeHdr& ch = t.hdr[c];
        r->best_move_q = (ch.flags & NF_HAS_D) ? -value_display(ch) : -node_value(ch);
        while (c >= 0 && (t.hdr[c].flags & NF_HAS_D) && !(t.hdr[c].flags & NF_TERMINAL) && n < kMaxDepth) {
            const NodeHdr& cur = t.hdr[c];
            const int ci = best_action_index(t, sp, cur, true, nullptr);
            r->pv[n++] = t.move[cur.edge_base + ci];
            c = t.child[cur.edge_base + ci];
        }
    }
    r->pv_len = n;
}

// ------------------------------------------------------------------ hash-derived fake network (test backend)
// Same definition as oracle/fake.c: every output is (9-bit integer) * 2^k, exact in fp32.
ARA_HD uint64_t zmix64(uint64_t z) {
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ULL;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBULL;
    return z ^ (z >> 31);
}
ARA_HD float fake_value(uint64_t key) {
    const uint64_t h0 = zmix64(key ^ 0x9E3779B97F4A7C15ULL);
    return static_cast<float>(static_cast<int>((h0 >> 11) & 0xFFFF) - 32768) * (1.0f / 65536.0f);
}
ARA_HD float fake_prob(uint64_t key, int i) {
    const uint64_t h = zmix64(key + static_cast<uint64_t>(i + 1) * 0xD6E8FEB86659FD93ULL);
    const uint32_t lo = static_cast<uint32_t>(h) | 0x80u;
#if defined(__CUDA_ARCH__)
    const int tz = __ffs(static_cast<int>(lo)) - 1;
#else
    const int tz = __builtin_ctz(lo);
#endif
    const int m = static_cast<int>((h >> 40) & 0xFF);
    return static_cast<float>(256 + m) * (1.0f / 65536.0f) * static_cast<float>(1 << tz);
}

}  // namespace ara
