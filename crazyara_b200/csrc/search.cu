// GPU MCTS engine: kernels around search_dev.cuh, the host-side driver (MCTSAgent::evaluate_board_state /
// SearchThread::thread_iteration of the reference) and the C-ABI.
//
// Per search iteration these are enqueued, with no host round trip in between:
//   select   create_mini_batch: one warp per tree (select_kernel), or a wavefront of 12 warps per tree when there are few
//            trees (select_wave_kernel, search_wave.cuh) -- sequential semantics either way
//   (pack)   many trees: the new leaves' rows of the network batch; expand: move lists, edges, planes written straight into
//            the network's NHWC input, one warp per new leaf
//   network  wgmma conv stack (CUDA graph), or the hash-derived fake backend for search-parity tests
//   update   scatter priors / values into the new nodes, prepare their next children, backups, collision reverts
// Threads = 1: all on one stream.  Threads = 2: the two logical threads' tree kernels on one stream in the fixed schedule
// of oracle/mcts.h, their forwards on a second stream (enqueue_slot).  The host only looks at the per-tree `done` flag
// once per chunk of iterations.
// This translation unit is compiled with -fmad=false: the PUCT / Q arithmetic must round exactly like the
// reference's (and the oracle's) scalar C++ code.
#include <atomic>
#include <chrono>
#include <cmath>
#include <cstring>
#include <memory>
#include <vector>

#include "abi_common.h"
#include "ara_b200.h"
#include "net.h"
#include "search_dev.cuh"
#include "search_wave.cuh"
#include "time_manager.h"

namespace ara {

struct DevWriterFactory {
    __half* base;
    int cpad;
    int split;  // Precision float32: rows of 3 * cpad halves, every channel as hi | hi | lo (conv_gemm.cuh)
    struct Target {
        __half* out;
        int cpad;
        int split;
        ARA_HD void encode(const Board& b, int mode, int version) const {
#if defined(__CUDA_ARCH__)
            if (split)
                encode_planes_nhwc_split(b, mode, version, out, cpad);
            else
                encode_planes_nhwc_f16(b, mode, version, out, cpad);
#endif
        }
    };
    ARA_HD Target make(int slot) const {
        return Target{base + static_cast<size_t>(slot) * 64 * cpad * (split ? 3 : 1), cpad, split};
    }
};
struct NullWriterFactory {  // fake backend: no planes needed
    struct Target {
        ARA_HD void encode(const Board&, int, int) const {}
    };
    ARA_HD Target make(int) const { return Target{}; }
};

// limits: per tree {simulations, nodes} of this go (ara_search_set_limits), or the settings' for every tree
__global__ void __launch_bounds__(32) root_kernel(const TreeDev* trees, SearchParams sp, const Board* roots, const uint2* limits) {
    __shared__ WarpScratch ws;
    const TreeDev t = trees[blockIdx.x];
    // the subtree kept by ara_search_apply_move is searched on if it is this position, else a new tree starts
    if (!reuse_root(t, sp, &roots[blockIdx.x])) create_root(t, sp, ws, &roots[blockIdx.x]);
    __syncwarp();
    if (threadIdx.x == 0) {
        t.st->limit_simulations = limits[blockIdx.x].x;
        t.st->limit_nodes = limits[blockIdx.x].y;
    }
}

// MCTSAgent::apply_move_to_tree for one tree
__global__ void __launch_bounds__(32) advance_kernel(const TreeDev* trees, int tree, Move move) {
    const TreeDev t = trees[tree];
    if (threadIdx.x == 0) advance_root(t, move);
}

// ------------------------------------------------------------------ node-pool compaction (tree reuse over long games)
// A kept subtree lives wherever its nodes were allocated: after a few searches the pools are full of the dead siblings
// of the moves that were played, and reuse_root would have to start a new tree.  Instead the subtree behind the new
// root is copied to the front of a second set of pools (node ids and edge ranges keep their relative order, so the new
// root becomes node 0), the pool pointers are swapped and the search goes on with every statistic it had.
struct CompactInfo {
    int need;    // the kept subtree is the searched position but the pools have no room left for another search
    int cand;    // its root
    int n_nodes, n_edges;
};
__global__ void __launch_bounds__(32) compact_decide_kernel(const TreeDev* trees, SearchParams sp, const Board* roots, CompactInfo* info) {
    if (threadIdx.x != 0) return;
    const TreeDev t = trees[blockIdx.x];
    const int cand = kept_subtree_root(t, &roots[blockIdx.x]);
    CompactInfo c;
    c.cand = cand;
    c.n_nodes = t.st->n_nodes;
    c.n_edges = t.st->n_edges;
    c.need = cand >= 0 && !pools_have_room(sp, t.max_nodes, t.max_edges, c.n_nodes, c.n_edges);
    info[blockIdx.x] = c;
}
// keep_n[i] = 1 if node i lies in the subtree of `cand`, keep_e[i] = its number of edges then
__global__ void compact_mark_kernel(TreeDev t, int cand, int n_nodes, int* keep_n, int* keep_e) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_nodes) return;
    int j = i;
    while (j > cand) j = t.hdr[j].parent;  // (a child is always allocated after its parent)
    const bool keep = j == cand;
    keep_n[i] = keep ? 1 : 0;
    keep_e[i] = keep ? t.hdr[i].n_moves : 0;
}
// exclusive prefix sum of a[0..n) in place, one thread block; total[0] = the sum
__global__ void __launch_bounds__(1024) compact_scan_kernel(int* a, int n, int* total) {
    __shared__ int part[1024];
    const int per = (n + 1023) / 1024;
    const int lo = threadIdx.x * per, hi = min(n, lo + per);
    int s = 0;
    for (int i = lo; i < hi; ++i) s += a[i];
    part[threadIdx.x] = s;
    __syncthreads();
    for (int off = 1; off < 1024; off <<= 1) {
        const int v = threadIdx.x >= off ? part[threadIdx.x - off] : 0;
        __syncthreads();
        part[threadIdx.x] += v;
        __syncthreads();
    }
    int run = part[threadIdx.x] - s;
    for (int i = lo; i < hi; ++i) {
        const int v = a[i];
        a[i] = run;
        run += v;
    }
    if (threadIdx.x == 1023) *total = part[1023];
}
// one warp per node of the old pools: a kept node and its edges go to their new places in `d`
__global__ void compact_gather_kernel(TreeDev s, TreeDev d, int cand, int n_nodes, const int* new_id, const int* new_eb) {
    const int i = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (i >= n_nodes) return;
    {   // (the marks were overwritten by their prefix sums: walk up again)
        int a = i;
        while (a > cand) a = s.hdr[a].parent;
        if (a != cand) return;
    }
    const int j = new_id[i];
    const NodeHdr h = s.hdr[i];
    if (lane < 4) reinterpret_cast<uint4*>(&d.hdr[j])[lane] = reinterpret_cast<const uint4*>(&s.hdr[i])[lane];
    else if (lane < 12) reinterpret_cast<uint4*>(&d.board[j])[lane - 4] = reinterpret_cast<const uint4*>(&s.board[i])[lane - 4];
    else if (lane < 12 + 8 * kPrepSlots && lane < 32) {
        const int q = lane - 12;
        reinterpret_cast<uint4*>(&d.prep_board[j * kPrepSlots])[q] = reinterpret_cast<const uint4*>(&s.prep_board[i * kPrepSlots])[q];
    }
    if (lane < kPrepSlots) {
        d.prep_ci[j * kPrepSlots + lane] = s.prep_ci[i * kPrepSlots + lane];
        d.prep_term[j * kPrepSlots + lane] = s.prep_term[i * kPrepSlots + lane];
    }
    __syncwarp();
    const uint32_t eb = static_cast<uint32_t>(new_eb[i]);
    if (lane == 0) {
        d.hdr[j].parent = i == cand ? -1 : new_id[h.parent];
        d.hdr[j].edge_base = eb;
    }
    for (int k = lane; k < h.n_moves; k += 32) {
        const uint32_t e = h.edge_base + k, f = eb + k;
        const int c = s.child[e];
        d.P[f] = s.P[e];
        d.Q[f] = s.Q[e];
        d.N[f] = s.N[e];
        d.move[f] = s.move[e];
        d.vl[f] = s.vl[e];
        d.etype[f] = s.etype[e];
        d.child[f] = c >= 0 ? new_id[c] : c;
        d.cbase[f] = c >= 0 ? static_cast<uint32_t>(new_eb[c]) : s.cbase[e];
    }
}
__global__ void compact_finish_kernel(TreeState* st, int n_nodes, int n_edges) {
    st->n_nodes = n_nodes;
    st->n_edges = n_edges;
    st->next_root = 0;  // the subtree's root is its first node
}

// one warp per tree: the sequential part of SearchThread::create_mini_batch
// EPS: with the epsilon-greedy / epsilon-check exploration (its own kernel: the ordinary select stays as lean as it is)
// count != nullptr (single-tree searches): the number of new leaves for the network kernels, what pack_kernel computes
// for many trees
template <bool EPS>
__global__ void __launch_bounds__(32) select_kernel(const TreeDev* trees, SearchParams sp, int* count) {
    __shared__ WarpScratch ws;
    const TreeDev t = trees[blockIdx.x];
    create_mini_batch<EPS>(t, sp, ws);
    if (count != nullptr && threadIdx.x == 0) *count = t.st->error ? 0 : t.bs->n_new;
}

// The same mini-batch by kWaveWarps warps per tree (search_wave.cuh): consecutive playouts of one tree overlap, the result
// is the sequential one.  Used when there are too few trees to fill the SMs with one warp each.
__global__ void __launch_bounds__(32 * kWaveWarps) select_wave_kernel(const TreeDev* trees, SearchParams sp, int* count) {
    extern __shared__ __align__(16) unsigned char wave_smem[];
    WaveShared& S = *reinterpret_cast<WaveShared*>(wave_smem);
    WaveWarp& W = reinterpret_cast<WaveWarp*>(wave_smem + kWaveSharedBytes)[threadIdx.x >> 5];
    const TreeDev t = trees[blockIdx.x];
    wave_mini_batch(t, sp, S, W);
    if (count != nullptr && threadIdx.x == 0) *count = t.st->error ? 0 : t.bs->n_new;  // (thread 0 wrote both at the end)
}

// Multi-tree searches: the new leaves of all trees are packed into consecutive rows of the network batch (tree i gets
// the rows after those of trees 0..i-1) and their total goes to `count`, which the network kernels read to skip the
// unused rows: a search of many small mini-batches (self-play: Batch_Size 8, often 2-3 new leaves per tree) then
// costs what its leaves cost, not what the widest possible batch costs.  One warp.
__global__ void __launch_bounds__(32) pack_kernel(TreeDev* trees, int n_trees, int* count) {
    int base = 0;
    for (int i0 = 0; i0 < n_trees; i0 += 32) {
        const int i = i0 + static_cast<int>(threadIdx.x);
        const int n = i < n_trees ? (trees[i].st->error ? 0 : trees[i].bs->n_new) : 0;
        int incl = n;
#pragma unroll
        for (int off = 1; off < 32; off <<= 1) {
            const int v = __shfl_up_sync(0xffffffffu, incl, off);
            if (static_cast<int>(threadIdx.x) >= off) incl += v;
        }
        if (i < n_trees) trees[i].slot_base = base + incl - n;
        base += __shfl_sync(0xffffffffu, incl, 31);
    }
    if (threadIdx.x == 0) *count = base;
}

// one warp per (tree, new leaf): move lists, edges, policy indices, input planes of all new leaves in parallel
__global__ void __launch_bounds__(32) expand_kernel(const TreeDev* trees, SearchParams sp, int batch, __half* in_h, int cpad,
                                                    int split) {
    __shared__ WarpScratch ws;
    const int tree = blockIdx.x / batch, b = blockIdx.x - tree * batch;
    const TreeDev t = trees[tree];
    if (b >= t.bs->n_new || t.st->error) return;
    const int nid = t.new_node[b];
    if (in_h != nullptr) {
        const DevWriterFactory wf{in_h, cpad, split};
        const auto target = wf.make(t.slot_base + b);
        expand_pending(t, sp, ws, nid, &target);
    } else {
        expand_pending(t, sp, ws, nid, static_cast<const NullWriterFactory::Target*>(nullptr));
    }
}

// one warp per (tree, new leaf): priors of the legal moves out of the soft-maxed policy, temperature, sort, value
__global__ void __launch_bounds__(32) scatter_kernel(const TreeDev* trees, SearchParams sp, int batch, const float* values,
                                                     const float* probs, int n_labels) {
    __shared__ WarpScratch ws;
    const int tree = blockIdx.x / batch, b = blockIdx.x - tree * batch;
    const TreeDev t = trees[tree];
    if (b >= t.bs->n_new || t.st->error) return;
    scatter_pending(t, sp, ws, b, values, probs, n_labels);
}

// one warp per tree: value backups along the stored trajectories, collision reverts
__global__ void __launch_bounds__(32) backup_kernel(const TreeDev* trees, SearchParams sp, int finalize, const float* values) {
    __shared__ WarpScratch ws;
    const TreeDev t = trees[blockIdx.x];
    backup_results(t, sp, values);
    if (finalize) finalize_root(t, sp, ws);
}

// one warp per (tree, item): prepared-child slots of the new leaves and of the nodes expanded in the last mini-batch
__global__ void __launch_bounds__(32) prepare_kernel(const TreeDev* trees, SearchParams sp, int items) {
    __shared__ WarpScratch ws;
    const int tree = blockIdx.x / items, item = blockIdx.x - tree * items;
    const TreeDev t = trees[tree];
    prepare_item(t, sp, ws, item);
}

// scatter and prepare in one warp (the iterations' path): warp `item` < B scatters leaf `item` and goes straight on to
// prepare that leaf's first child; the other warps prepare the next children of the nodes expanded in the mini-batch,
// which depend on neither.  Saves a dependent launch per iteration and takes the parents' work off the critical path.
__device__ __forceinline__ void scatter_prepare_item(const TreeDev t, const SearchParams& sp, WarpScratch& ws, int item, int batch,
                                                     const float* values, const float* probs, int n_labels) {
    if (t.st->error) return;
    if (item < batch) {
        if (item >= t.bs->n_new) return;
        scatter_pending(t, sp, ws, item, values, probs, n_labels);
        __syncwarp();
    }
    prepare_item(t, sp, ws, item);
}

__global__ void __launch_bounds__(32) scatter_prepare_kernel(const TreeDev* trees, SearchParams sp, int batch, int items,
                                                             const float* values, const float* probs, int n_labels) {
    __shared__ WarpScratch ws;
    const int tree = blockIdx.x / items, item = blockIdx.x - tree * items;
    scatter_prepare_item(trees[tree], sp, ws, item, batch, values, probs, n_labels);
}

// The whole update step of an iteration in ONE launch: the first n_trees warps run the value backups (one per tree, the
// long pole: scheduled first), the others scatter + prepare.  Backups read nothing the scatter / prepare steps write and
// write nothing they read (backup_results), so they need no order between them -- and no second stream with its fork /
// join events either.
__global__ void __launch_bounds__(32) update_kernel(const TreeDev* trees, SearchParams sp, int n_trees, int batch, int items,
                                                    const float* values, const float* probs, int n_labels) {
    __shared__ WarpScratch ws;
    if (static_cast<int>(blockIdx.x) < n_trees) {
        backup_results(trees[blockIdx.x], sp, values);
        return;
    }
    const int blk = static_cast<int>(blockIdx.x) - n_trees;
    const int tree = blk / items, item = blk - tree * items;
    scatter_prepare_item(trees[tree], sp, ws, item, batch, values, probs, n_labels);
}

__global__ void __launch_bounds__(32) result_kernel(const TreeDev* trees, SearchParams sp, SearchResult* out) {
    const TreeDev t = trees[blockIdx.x];
    if (threadIdx.x == 0) collect_result(t, sp, &out[blockIdx.x]);
}

__global__ void __launch_bounds__(32) node_view_kernel(const TreeDev* trees, int tree, int node_id, NodeView* out) {
    collect_node_view(trees[tree], node_id, out);
}

__global__ void __launch_bounds__(32) time_stats_kernel(const TreeDev* trees, RootTimeStats* out) {
    const TreeDev t = trees[blockIdx.x];
    if (threadIdx.x == 0) collect_time_stats(t, &out[blockIdx.x]);
}

// Fake backend: value/prob rows of the pending new nodes from their Zobrist keys (oracle/fake.c definition).
__global__ void fake_eval_kernel(const TreeDev* trees, int n_trees, int batch, float* values, float* probs, int n_labels) {
    const int tree = blockIdx.x / batch, b = blockIdx.x - tree * batch;
    if (tree >= n_trees) return;
    const TreeDev t = trees[tree];
    if (b >= t.bs->n_new) return;
    const int slot = t.slot_base + b;  // row of this leaf in the (possibly packed) batch
    const uint64_t key = t.hdr[t.new_node[b]].key;
    if (threadIdx.x == 0) values[slot] = fake_value(key);
    for (int i = threadIdx.x; i < n_labels; i += blockDim.x) probs[static_cast<size_t>(slot) * n_labels + i] = fake_prob(key, i);
}

// ---------------------------------------------------------------------------------------------------------------
class Search {
   public:
    ~Search();
    int init(Net* net, const SearchParams& sp, int device, int n_trees, int max_nodes);
    int set_position(int tree, const Board& root, const uint64_t* hist_keys, const int16_t* hist_reps, int hist_len);
    int go();
    int apply_move(int tree, unsigned short move);
    void request_stop() { stop_requested_.store(true, std::memory_order_relaxed); }
    int fetch_results();
    int begin();
    int step(int n_batches);
    int poll_running();
    int node_view(int tree, int node_id, NodeView* out);
    NodeView* d_node_view_ = nullptr;
    int debug_cycles(int tree, unsigned long long* out8) {
        TreeState st;
        ARA_CUDA_OK(cudaMemcpy(&st, d_states_[tree], sizeof(st), cudaMemcpyDeviceToHost));
        for (int i = 0; i < 8; ++i) out8[i] = st.prof[i];
        return 0;
    }
    SearchParams sp{};
    int n_trees = 0;
    std::vector<SearchResult> results;
    long long launches = 0;
    double last_go_ms = 0.0;
    double movetime_ms = 0.0;  // > 0: stop issuing iterations once this much wall time has passed (UCI `go movetime`)
    // ThreadManager heuristics (time_manager.h): parameters, and what happened in the last go
    bool use_tc = false;
    ara_time_control_t tc{};
    ara_time_report_t tr{};
    // one iteration as a CUDA graph
    bool iter_warm_ = false;
    cudaGraphExec_t iter_graph_ = nullptr;
    cudaStream_t side_stream_ = nullptr;  // second branch of an iteration (value backups)
    cudaEvent_t ev_fork_ = nullptr, ev_join_ = nullptr;
    int enqueue_iteration(bool with_events);
    // ---- Threads = 2 (sp.threads): two logical search threads per tree, each with its own batch state ("slot": views
    // of the trees with their own new-leaf / trajectory arrays, their own rows of the network's second input / output
    // set).  The tree kernels of both threads run on stream_ in the fixed order
    //     S0 S1 | U0 S0 U1 S1 | U0 S0 ...     (S = select + pack + expand, U = scatter + prepare || backup)
    // and each thread's network forward on net_stream_, between its S and its next U: while one thread's batch is at
    // the network the other thread selects.  (oracle/mcts.h describes the schedule; tests compare all three.)
    int threads_ = 1;
    bool eps_ = false;  // epsilon-greedy / epsilon-check exploration on: the select_kernel<true> instantiation
    bool wave_ = false;  // few trees: select_wave_kernel (several warps per tree) instead of one warp per tree
    void launch_select(const TreeDev* trees, int* count = nullptr) {
        if (eps_) select_kernel<true><<<n_trees, 32, 0, stream_>>>(trees, sp, count);
        else if (wave_) select_wave_kernel<<<n_trees, 32 * kWaveWarps, kWaveSmemBytes, stream_>>>(trees, sp, count);
        else select_kernel<false><<<n_trees, 32, 0, stream_>>>(trees, sp, count);
    }
    bool primed_ = false;                  // S0 S1 of the current go have been enqueued
    TreeDev* d_trees_slot_[2] = {nullptr, nullptr};
    std::vector<TreeDev> h_trees1_;        // slot 1 views (h_trees_ = slot 0); their batch arrays are slot 1's own
    // node-pool compaction: the second set of pools per tree (allocated at the first compaction), scan scratch
    std::vector<TreeDev> shadow_;
    std::vector<char> advanced_;           // ara_search_apply_move since the last go
    CompactInfo* d_cinfo_ = nullptr;
    int* d_keep_n_ = nullptr;
    int* d_keep_e_ = nullptr;
    int* d_ctotal_ = nullptr;
    long long compactions = 0;
    int compact_pools();
    int* d_count_slot_[2] = {nullptr, nullptr};
    float *d_values_slot_[2] = {nullptr, nullptr}, *d_probs_slot_[2] = {nullptr, nullptr};  // fake backend, per slot
    cudaStream_t net_stream_ = nullptr;
    cudaEvent_t ev_sel_[2] = {nullptr, nullptr}, ev_net_[2] = {nullptr, nullptr};
    cudaGraphExec_t slot_graph_[2][2] = {{nullptr, nullptr}, {nullptr, nullptr}};  // [slot][with update]
    bool slot_warm_ = false;
    int enqueue_slot(int slot, bool with_update);
    int enqueue_slot_tree_ops(int slot, bool with_update);
    int iterate2(int cycles);
    std::vector<uint2> h_limits_;  // per tree {simulations, nodes} of the next go
    uint2* d_limits_ = nullptr;
    int set_limits(int tree, unsigned simulations, unsigned nodes);
    int* d_count_ = nullptr;  // multi-tree searches: rows of the network batch in use (written by pack_kernel)
    RootTimeStats* d_tstats_ = nullptr;
    RootTimeStats* h_tstats_ = nullptr;  // pinned
    int read_time_stats(RootStatsHost* out);
    // per-phase device times of the last go (CUDA events on the search stream), filled when profile is on
    bool profile = false;
    double select_ms = 0.0, net_ms = 0.0, apply_ms = 0.0;
    long long net_forwards = 0;

   private:
    // The arrays of TreeDev, listed once: f(member, length) for each.  A tree's node, edge and prepared-child pools
    // (the compaction swaps them for its second set) ...
    template <typename F>
    void for_each_pool(F&& f) const {
        const size_t nodes = max_nodes_, edges = max_edges_, slots = nodes * kPrepSlots;
        f(&TreeDev::hdr, nodes), f(&TreeDev::board, nodes);
        f(&TreeDev::P, edges), f(&TreeDev::Q, edges), f(&TreeDev::N, edges), f(&TreeDev::child, edges), f(&TreeDev::cbase, edges);
        f(&TreeDev::move, edges), f(&TreeDev::vl, edges), f(&TreeDev::etype, edges);
        f(&TreeDev::prep_board, slots), f(&TreeDev::prep_ci, slots), f(&TreeDev::prep_term, slots);
    }
    // ... and the batch arrays of one view of a tree (Threads = 2: each logical thread's view has its own)
    template <typename F>
    void for_each_batch_array(F&& f) const {
        const size_t B = sp.batch_size, traj = 2 * B * kMaxDepth;
        f(&TreeDev::bs, 1), f(&TreeDev::exp_parent, 3 * B), f(&TreeDev::new_node, B);
        f(&TreeDev::traj_node, traj), f(&TreeDev::traj_ci, traj), f(&TreeDev::traj_edge, traj);
        f(&TreeDev::traj_len, 2 * B), f(&TreeDev::traj_start, 2 * B);
    }
    int alloc_pools(TreeDev& t) {
        int rc = 0;
        for_each_pool([&](auto m, size_t n) { rc = rc ? rc : mem_.dalloc(&(t.*m), n); });
        return rc;
    }
    int alloc_batch_arrays(TreeDev& t) {
        int rc = 0;
        for_each_batch_array([&](auto m, size_t n) { rc = rc ? rc : mem_.dalloc(&(t.*m), n); });
        return rc;
    }
    int iterate(int count);
    Net* net_ = nullptr;
    bool searched_ = false;  // a go has run: the device holds trees that apply_move may keep
    // UCI `stop` (SearchThread::stop): set from another host thread while go() runs; go() leaves its loop at the next poll
    std::atomic<bool> stop_requested_{false};
    int device_ = 0;
    cudaStream_t stream_ = nullptr;
    bool own_stream_ = false;
    int max_nodes_ = 0, max_edges_ = 0, n_labels_ = 0, hist_cap_ = 512;
    DeviceBuffers mem_;
    std::vector<TreeDev> h_trees_;
    TreeDev* d_trees_ = nullptr;
    Board* d_roots_ = nullptr;
    std::vector<Board> h_roots_;
    std::vector<TreeState*> d_states_;
    std::vector<uint64_t*> d_hist_keys_;
    std::vector<int16_t*> d_hist_reps_;
    float* d_lut_ = nullptr;
    double* d_sqrt_lut_ = nullptr;
    float *d_values_ = nullptr, *d_probs_ = nullptr;  // fake backend buffers
    SearchResult* d_results_ = nullptr;
    int* h_done_ = nullptr;  // pinned
    cudaEvent_t ev0_ = nullptr, ev1_ = nullptr;
    std::vector<cudaEvent_t> prof_events_;
    size_t prof_used_ = 0;
    cudaEvent_t prof_event();
    int prof_collect();
};

cudaEvent_t Search::prof_event() {
    if (prof_used_ == prof_events_.size()) {
        cudaEvent_t e;
        cudaEventCreate(&e);
        prof_events_.push_back(e);
    }
    cudaEvent_t e = prof_events_[prof_used_++];
    cudaEventRecord(e, stream_);
    return e;
}
int Search::prof_collect() {  // events come in groups of four: before select, before net, after net, after apply
    select_ms = net_ms = apply_ms = 0.0;
    if (threads_ == 2) {  // groups of four per turn: tree ops begin / end on stream_, forward begin / end on net_stream_;
                          // select_ms = the tree stream's time (backups + scatter + select + expand), apply_ms stays 0
        for (size_t i = 0; i + 3 < prof_used_; i += 4) {
            float a = 0, b = 0;
            ARA_CUDA_OK(cudaEventElapsedTime(&a, prof_events_[i], prof_events_[i + 1]));
            ARA_CUDA_OK(cudaEventElapsedTime(&b, prof_events_[i + 2], prof_events_[i + 3]));
            select_ms += a;
            net_ms += b;
        }
        return 0;
    }
    for (size_t i = 0; i + 3 < prof_used_; i += 4) {
        float a = 0, b = 0, c = 0;
        ARA_CUDA_OK(cudaEventElapsedTime(&a, prof_events_[i], prof_events_[i + 1]));
        ARA_CUDA_OK(cudaEventElapsedTime(&b, prof_events_[i + 1], prof_events_[i + 2]));
        ARA_CUDA_OK(cudaEventElapsedTime(&c, prof_events_[i + 2], prof_events_[i + 3]));
        select_ms += a;
        net_ms += b;
        apply_ms += c;
    }
    return 0;
}

Search::~Search() {
    cudaSetDevice(device_);
    if (stream_) cudaStreamSynchronize(stream_);
    if (h_done_) cudaFreeHost(h_done_);
    if (h_tstats_) cudaFreeHost(h_tstats_);
    if (iter_graph_) cudaGraphExecDestroy(iter_graph_);
    for (auto& a : slot_graph_)
        for (auto g : a)
            if (g) cudaGraphExecDestroy(g);
    if (net_stream_) cudaStreamDestroy(net_stream_);
    for (cudaEvent_t e : ev_sel_)
        if (e) cudaEventDestroy(e);
    for (cudaEvent_t e : ev_net_)
        if (e) cudaEventDestroy(e);
    if (side_stream_) cudaStreamDestroy(side_stream_);
    if (ev_fork_) cudaEventDestroy(ev_fork_);
    if (ev_join_) cudaEventDestroy(ev_join_);
    if (ev0_) cudaEventDestroy(ev0_);
    if (ev1_) cudaEventDestroy(ev1_);
    for (cudaEvent_t e : prof_events_) cudaEventDestroy(e);
    if (own_stream_ && stream_) cudaStreamDestroy(stream_);
}

int Search::init(Net* net, const SearchParams& params, int device, int trees, int max_nodes) {
    sp = params;
    net_ = net;
    device_ = net ? net->device : device;
    n_trees = trees;
    if (sp.batch_size < 1 || sp.batch_size > 1024) return set_error("ara_search_create: batch_size %d out of range", sp.batch_size);
    if (n_trees < 1) return set_error("ara_search_create: n_trees %d < 1", n_trees);
    if (planes_channels(sp.mode, sp.input_version) < 0)
        return set_error("ara_search_create: unsupported mode %d / input version %d", sp.mode, sp.input_version);
    if (sp.threads == 0) sp.threads = 1;
    if (sp.threads != 1 && sp.threads != 2) return set_error("ara_search_create: Threads %d (1 or 2)", sp.threads);
    // the virtual visits in flight on an edge are counted in a uint8 like the reference's (nodedata.h:93)
    if (sp.threads * sp.batch_size > 255 && sp.threads > 1)
        return set_error("ara_search_create: Threads %d x Batch_Size %d exceeds the 255 virtual visits an edge can carry", sp.threads, sp.batch_size);
    threads_ = sp.threads;
    if (sp.epsilon_greedy_counter < 0 || sp.epsilon_greedy_counter > 255 || sp.epsilon_checks_counter < 0 || sp.epsilon_checks_counter > 255)
        return set_error("ara_search_create: epsilon counters must be in [0, 255] (round(100 / Centi_Epsilon_*), uint8 in the reference)");
    eps_ = sp.epsilon_greedy_counter != 0 || sp.epsilon_checks_counter != 0;
    ARA_CUDA_OK(cudaSetDevice(device_));
    {
        cudaDeviceProp prop;
        ARA_CUDA_OK(cudaGetDeviceProperties(&prop, device_));
        if (prop.major != 9 || prop.minor != 0) return set_error("ara_search_create: device %d is not sm_90a (H100)", device_);
    }
    // few trees cannot fill the SMs with one warp each: their playouts overlap inside a CTA instead (search_wave.cuh)
    wave_ = !eps_ && ((n_trees <= 16 && sp.batch_size >= 8) || (n_trees <= 32 && sp.batch_size >= 16));
    if (const char* e = getenv("ARA_WAVE")) wave_ = !eps_ && atoi(e) != 0;
    if (wave_)
        ARA_CUDA_OK(cudaFuncSetAttribute(select_wave_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(kWaveSmemBytes)));
    n_labels_ = (sp.mode == MODE_CRAZYHOUSE ? 81 : (sp.mode == MODE_CHESS ? 76 : 84)) * 64;
    if (net_ != nullptr) {
        if (net_->batch < n_trees * sp.batch_size)
            return set_error("ara_search_create: network batch %d < trees %d x Batch_Size %d", net_->batch, n_trees, sp.batch_size);
        if (net_->n_labels() != n_labels_ || net_->hdr.in_channels != planes_channels(sp.mode, sp.input_version))
            return set_error("ara_search_create: network shape (C=%d, L=%d) does not match mode/version (C=%d, L=%d)",
                             net_->hdr.in_channels, net_->n_labels(), planes_channels(sp.mode, sp.input_version), n_labels_);
        stream_ = net_->stream;
    } else {
        ARA_CUDA_OK(cudaStreamCreateWithFlags(&stream_, cudaStreamNonBlocking));
        own_stream_ = true;
        if (mem_.dalloc(&d_values_, static_cast<size_t>(n_trees) * sp.batch_size)) return -1;
        if (mem_.dalloc(&d_probs_, static_cast<size_t>(n_trees) * sp.batch_size * n_labels_)) return -1;
    }
    if (max_nodes <= 0) {
        const unsigned budget = sp.simulations ? sp.simulations : (sp.nodes ? sp.nodes * 2 : 0);
        if (budget == 0) return set_error("ara_search_create: max_nodes must be given when neither Simulations nor Nodes is set");
        max_nodes = static_cast<int>(budget) + 4 * sp.batch_size * sp.threads + 64;
    }
    max_nodes_ = max_nodes;
    // edge pool: average legal moves per node is ~35 (chess) but drop-heavy crazyhouse positions reach 200-300
    {
        // sized for the worst case per node; computed in 64 bits: 2^24 nodes x 320 edges does not fit an int
        const long long want = static_cast<long long>(max_nodes) * (sp.mode == MODE_CHESS ? 128 : 320) + 1024;
        if (want > 2147483647LL)
            return set_error("ara_search_create: a pool of %d nodes needs %lld edge slots (more than 2^31 - 1); lower max_nodes", max_nodes, want);
        max_edges_ = static_cast<int>(want);
    }
    const int B = sp.batch_size;
    // cput look-up table with the HOST libm: bit-identical to the reference's scalar code (node.cpp:1243-1246)
    {
        int len = max_nodes_ + 8;
        if (len > (1 << 22)) len = 1 << 22;
        std::vector<float> lut(len);
        for (int i = 0; i < len; ++i) lut[i] = logf((static_cast<float>(i) + sp.cpuct_base + 1) / sp.cpuct_base) + sp.cpuct_init;
        if (mem_.dalloc(&d_lut_, lut.size())) return -1;
        ARA_CUDA_OK(cudaMemcpy(d_lut_, lut.data(), lut.size() * 4, cudaMemcpyHostToDevice));
        // sqrt(double(visit_sum)): IEEE-exact on both sides, tabulated only to keep the instruction chain short
        std::vector<double> sq(len);
        for (int i = 0; i < len; ++i) sq[i] = sqrt(static_cast<double>(i));
        if (mem_.dalloc(&d_sqrt_lut_, sq.size())) return -1;
        ARA_CUDA_OK(cudaMemcpy(d_sqrt_lut_, sq.data(), sq.size() * 8, cudaMemcpyHostToDevice));
        h_trees_.resize(n_trees);
        for (auto& t : h_trees_) t.cput_lut_len = len;
    }
    d_states_.resize(n_trees);
    d_hist_keys_.resize(n_trees);
    d_hist_reps_.resize(n_trees);
    for (int i = 0; i < n_trees; ++i) {
        TreeDev& t = h_trees_[i];
        if (alloc_pools(t) || alloc_batch_arrays(t) || mem_.dalloc(&t.st, 1)) return -1;
        if (mem_.dalloc(&d_hist_keys_[i], hist_cap_) || mem_.dalloc(&d_hist_reps_[i], hist_cap_)) return -1;
        t.hist_keys = d_hist_keys_[i];
        t.hist_reps = d_hist_reps_[i];
        t.hist_len = 0;
        t.cput_lut = d_lut_;
        t.sqrt_lut = d_sqrt_lut_;
        t.max_nodes = max_nodes_;
        t.max_edges = max_edges_;
        t.slot_base = i * B;
        d_states_[i] = t.st;
    }
    if (mem_.dalloc(&d_trees_, n_trees) || mem_.dalloc(&d_roots_, n_trees) || mem_.dalloc(&d_results_, n_trees) || mem_.dalloc(&d_limits_, n_trees) ||
        mem_.dalloc(&d_tstats_, 1) || mem_.dalloc(&d_count_, 1) || mem_.dalloc(&d_node_view_, 1))
        return -1;
    h_limits_.assign(n_trees, make_uint2(sp.simulations, sp.nodes));
    for (int i = 0; i < n_trees; ++i) {  // the trees' Dirichlet generators (TreeState::rng)
        const uint32_t x = minstd_seed(sp.seed, i);
        ARA_CUDA_OK(cudaMemcpy(&d_states_[i]->rng, &x, sizeof(x), cudaMemcpyHostToDevice));
        TreeState tmp;  // rand() of the exploration branches: srand(seed ^ tree index * golden ratio)
        crand_seed(tmp.crand_r, &tmp.crand_f, static_cast<unsigned>(sp.seed ^ (static_cast<unsigned long long>(i) * 0x9E3779B97F4A7C15ULL)));
        ARA_CUDA_OK(cudaMemcpy(d_states_[i]->crand_r, tmp.crand_r, sizeof(tmp.crand_r), cudaMemcpyHostToDevice));
        ARA_CUDA_OK(cudaMemcpy(&d_states_[i]->crand_f, &tmp.crand_f, sizeof(tmp.crand_f), cudaMemcpyHostToDevice));
    }
    d_trees_slot_[0] = d_trees_;
    if (threads_ == 2) {
        h_trees1_.resize(n_trees);
        for (auto& t : h_trees1_)
            if (alloc_batch_arrays(t)) return -1;
        if (mem_.dalloc(&d_trees_slot_[1], n_trees)) return -1;
        if (net_ != nullptr) {
            if (net_->enable_second_io()) return -1;
        } else {
            d_values_slot_[0] = d_values_, d_probs_slot_[0] = d_probs_;
            if (mem_.dalloc(&d_values_slot_[1], static_cast<size_t>(n_trees) * sp.batch_size)) return -1;
            if (mem_.dalloc(&d_probs_slot_[1], static_cast<size_t>(n_trees) * sp.batch_size * n_labels_)) return -1;
        }
        // the network stream has the same (default) priority as the tree stream: neither yields to the other
        ARA_CUDA_OK(cudaStreamCreateWithFlags(&net_stream_, cudaStreamNonBlocking));
        for (int k = 0; k < 2; ++k) {
            ARA_CUDA_OK(cudaEventCreateWithFlags(&ev_sel_[k], cudaEventDisableTiming));
            ARA_CUDA_OK(cudaEventCreateWithFlags(&ev_net_[k], cudaEventDisableTiming));
        }
        if (mem_.dalloc(&d_count_slot_[1], 1)) return -1;
    }
    h_roots_.resize(n_trees);
    results.resize(n_trees);
    ARA_CUDA_OK(cudaMallocHost(&h_done_, sizeof(int) * n_trees));
    ARA_CUDA_OK(cudaMallocHost(&h_tstats_, sizeof(RootTimeStats)));
    d_count_slot_[0] = d_count_;
    ARA_CUDA_OK(cudaStreamCreateWithFlags(&side_stream_, cudaStreamNonBlocking));
    ARA_CUDA_OK(cudaEventCreateWithFlags(&ev_fork_, cudaEventDisableTiming));
    ARA_CUDA_OK(cudaEventCreateWithFlags(&ev_join_, cudaEventDisableTiming));
    ARA_CUDA_OK(cudaEventCreate(&ev0_));
    ARA_CUDA_OK(cudaEventCreate(&ev1_));
    return 0;
}

int Search::set_position(int tree, const Board& root, const uint64_t* hist_keys, const int16_t* hist_reps, int hist_len) {
    if (tree < 0 || tree >= n_trees) return set_error("ara_search_set_position: tree %d out of range", tree);
    ARA_CUDA_OK(cudaSetDevice(device_));
    h_roots_[tree] = root;
    // keep the most recent hist_cap_ plies (rule50 bounds the look-back to 100 plies in chess; crazyhouse looks back
    // over the whole game, truncated here to hist_cap_ plies)
    int skip = hist_len > hist_cap_ ? hist_len - hist_cap_ : 0;
    const int len = hist_len - skip;
    if (len > 0) {
        ARA_CUDA_OK(cudaMemcpyAsync(d_hist_keys_[tree], hist_keys + skip, sizeof(uint64_t) * len, cudaMemcpyHostToDevice, stream_));
        ARA_CUDA_OK(cudaMemcpyAsync(d_hist_reps_[tree], hist_reps + skip, sizeof(int16_t) * len, cudaMemcpyHostToDevice, stream_));
    }
    h_trees_[tree].hist_len = len;
    ARA_CUDA_OK(cudaStreamSynchronize(stream_));
    return 0;
}

// One search iteration on the stream: select -> (pack) -> expand -> network -> scatter -> backup -> prepare.
int Search::enqueue_iteration(bool with_events) {
    __half* in_h = net_ ? net_->d_in_h : nullptr;
    const int cpad = net_ ? net_->cin_pad : 0;
    const int B = sp.batch_size;
    const float* values = net_ ? net_->d_value : d_values_;
    const float* probs = net_ ? net_->d_prob : d_probs_;
    if (with_events) prof_event();
    launch_select(d_trees_);
    if (n_trees > 1) pack_kernel<<<1, 32, 0, stream_>>>(d_trees_, n_trees, d_count_);
    expand_kernel<<<n_trees * B, 32, 0, stream_>>>(d_trees_, sp, B, in_h, cpad, net_ ? net_->precision : 0);
    if (with_events) prof_event();
    if (net_) {
        if (net_->forward_device(n_trees * B, stream_, n_trees > 1 ? d_count_ : nullptr)) return -1;
    } else {
        fake_eval_kernel<<<n_trees * B, 128, 0, stream_>>>(d_trees_, n_trees, B, d_values_, d_probs_, n_labels_);
    }
    if (with_events) prof_event();
    // the value backups (one warp per tree, a latency chain) run beside scatter -> prepare: neither reads what the
    // other writes (backup_results); a second branch of the iteration graph
    if (n_trees > 1) {
        update_kernel<<<n_trees + n_trees * 4 * B, 32, 0, stream_>>>(d_trees_, sp, n_trees, B, 4 * B, values, probs, n_labels_);
    } else {
        // (one tree, one thread: measured 2 % faster with the backup warp as a kernel of its own on a second branch of the
        // iteration graph than inside the scatter / prepare grid)
        ARA_CUDA_OK(cudaEventRecord(ev_fork_, stream_));
        ARA_CUDA_OK(cudaStreamWaitEvent(side_stream_, ev_fork_, 0));
        backup_kernel<<<n_trees, 32, 0, side_stream_>>>(d_trees_, sp, 0, values);
        ARA_CUDA_OK(cudaEventRecord(ev_join_, side_stream_));
        scatter_prepare_kernel<<<n_trees * 4 * B, 32, 0, stream_>>>(d_trees_, sp, B, 4 * B, values, probs, n_labels_);
        ARA_CUDA_OK(cudaStreamWaitEvent(stream_, ev_join_, 0));
    }
    if (with_events) prof_event();
    return 0;
}

// `count` iterations.  Outside profiling runs an iteration is ONE graph launch: the kernels of an iteration never
// change (same pointers, same grids), so the sequence is captured once per handle -- the network's own graph becomes a
// child node -- and the dependent-launch gaps between the seven search kernels shrink to graph-edge latency.
// Threads = 2: the tree kernels of one turn of logical thread `slot` -- U (the backups and the scatter / prepare step of
// its previous batch) then S (its next select, pack, expand) -- on stream_.
int Search::enqueue_slot_tree_ops(int slot, bool with_update) {
    const int B = sp.batch_size;
    TreeDev* trees = d_trees_slot_[slot];
    const float* values = net_ ? net_->io_value[slot] : d_values_slot_[slot];
    const float* probs = net_ ? net_->io_prob[slot] : d_probs_slot_[slot];
    if (with_update) {
        update_kernel<<<n_trees + n_trees * 4 * B, 32, 0, stream_>>>(trees, sp, n_trees, B, 4 * B, values, probs, n_labels_);
    }
    if (n_trees == 1) {  // (one tree: its rows start at 0, the select kernel itself leaves the count)
        launch_select(trees, d_count_slot_[slot]);
    } else {
        launch_select(trees);
        pack_kernel<<<1, 32, 0, stream_>>>(trees, n_trees, d_count_slot_[slot]);
    }
    expand_kernel<<<n_trees * B, 32, 0, stream_>>>(trees, sp, B, net_ ? net_->io_in_h[slot] : nullptr, net_ ? net_->cin_pad : 0,
                                                    net_ ? net_->precision : 0);
    // the stem convolution of the new batch right here, on the tree stream (which has the slack): the network stream's
    // chain starts at the tower
    if (net_ && net_->stem_splittable() && net_->stem_device(n_trees * B, stream_, d_count_slot_[slot], slot)) return -1;
    return 0;
}

// one turn of logical thread `slot`: wait for its batch at the network, U + S on the tree stream, then hand the new batch
// to the network stream
int Search::enqueue_slot(int slot, bool with_update) {
    const int B = sp.batch_size;
    if (with_update) ARA_CUDA_OK(cudaStreamWaitEvent(stream_, ev_net_[slot], 0));
    cudaGraphExec_t& ge = slot_graph_[slot][with_update ? 1 : 0];
    if (profile) prof_event();
    if (!profile && ge != nullptr) {
        ARA_CUDA_OK(cudaGraphLaunch(ge, stream_));
    } else if (!profile && slot_warm_) {
        if (capture_graph(stream_, &ge, [&] { return enqueue_slot_tree_ops(slot, with_update); })) return -1;
        ARA_CUDA_OK(cudaGraphLaunch(ge, stream_));
    } else {
        if (enqueue_slot_tree_ops(slot, with_update)) return -1;
    }
    if (profile) prof_event();
    launches += (n_trees == 1 ? 2 : 3) + (with_update ? 1 : 0);
    if (net_ && net_->stem_splittable()) ++net_->launches;  // (the stem ran with the tree kernels, possibly from their graph)
    ARA_CUDA_OK(cudaEventRecord(ev_sel_[slot], stream_));
    ARA_CUDA_OK(cudaStreamWaitEvent(net_stream_, ev_sel_[slot], 0));
    if (profile) {
        cudaEvent_t e = prof_event();  // (recorded on stream_; re-record it on the network stream)
        ARA_CUDA_OK(cudaEventRecord(e, net_stream_));
    }
    if (net_) {
        if (net_->forward_device(n_trees * B, net_stream_, d_count_slot_[slot], slot, net_->stem_splittable())) return -1;
    } else {
        fake_eval_kernel<<<n_trees * B, 128, 0, net_stream_>>>(d_trees_slot_[slot], n_trees, B, d_values_slot_[slot],
                                                               d_probs_slot_[slot], n_labels_);
        ++launches;
    }
    if (profile) {
        cudaEvent_t e = prof_event();
        ARA_CUDA_OK(cudaEventRecord(e, net_stream_));
    }
    ARA_CUDA_OK(cudaEventRecord(ev_net_[slot], net_stream_));
    ++net_forwards;
    return 0;
}

// `cycles` turns of both logical threads (two mini-batches each cycle)
int Search::iterate2(int cycles) {
    if (!primed_) {  // S0 S1: nothing to back up yet (the root's batch was applied by the root phase)
        if (enqueue_slot(0, false) || enqueue_slot(1, false)) return -1;
        primed_ = true;
        slot_warm_ = true;
        --cycles;
    }
    for (int c = 0; c < cycles; ++c)
        if (enqueue_slot(0, true) || enqueue_slot(1, true)) return -1;
    ARA_CUDA_OK(cudaGetLastError());
    return 0;
}

int Search::iterate(int count) {
    if (threads_ == 2) return iterate2((count + 1) / 2);
    const int search_kernels = 4 + (net_ ? 0 : 1);  // (one tree: select, expand, scatter+prepare, backup; many: + pack, one update launch)
    for (int it = 0; it < count; ++it) {
        if (!profile && iter_graph_ != nullptr) {
            ARA_CUDA_OK(cudaGraphLaunch(iter_graph_, stream_));
            if (net_) net_->launches += net_->kernels_per_forward(false);
        } else if (!profile && iter_warm_) {
            // second iteration of the handle's life (the first one ran eagerly and warmed the network's graph up)
            const long long net_before = net_ ? net_->launches : 0;
            const int rc = capture_graph(stream_, &iter_graph_, [&] { return enqueue_iteration(false); });
            if (net_) net_->launches = net_before;
            if (rc) return -1;
            --it;  // nothing ran yet: launch the graph in the next pass
            continue;
        } else {
            if (enqueue_iteration(profile)) return -1;
            iter_warm_ = true;
        }
        ++net_forwards;
        launches += search_kernels;
    }
    ARA_CUDA_OK(cudaGetLastError());
    return 0;
}

// Before a go that may continue on a kept subtree: where the pools have no room for another search, the subtree moves to
// the front of the tree's second set of pools (see compact_decide_kernel).  h_trees_ is updated; the caller uploads it.
int Search::compact_pools() {
    bool any = false;
    for (char a : advanced_) any = any || a != 0;
    if (!any) return 0;
    advanced_.assign(n_trees, 0);
    if (d_cinfo_ == nullptr) {
        if (mem_.dalloc(&d_cinfo_, n_trees) || mem_.dalloc(&d_keep_n_, static_cast<size_t>(max_nodes_) + 1) ||
            mem_.dalloc(&d_keep_e_, static_cast<size_t>(max_nodes_) + 1) || mem_.dalloc(&d_ctotal_, 2))
            return -1;
        shadow_.resize(n_trees);
        for (auto& t : shadow_) t.hdr = nullptr;
    }
    compact_decide_kernel<<<n_trees, 32, 0, stream_>>>(d_trees_, sp, d_roots_, d_cinfo_);
    std::vector<CompactInfo> info(n_trees);
    ARA_CUDA_OK(cudaMemcpyAsync(info.data(), d_cinfo_, sizeof(CompactInfo) * n_trees, cudaMemcpyDeviceToHost, stream_));
    ARA_CUDA_OK(cudaStreamSynchronize(stream_));
    ++launches;
    for (int i = 0; i < n_trees; ++i) {
        const CompactInfo& c = info[i];
        if (!c.need || c.n_nodes <= 0) continue;
        TreeDev& t = h_trees_[i];
        compact_mark_kernel<<<(c.n_nodes + 255) / 256, 256, 0, stream_>>>(t, c.cand, c.n_nodes, d_keep_n_, d_keep_e_);
        compact_scan_kernel<<<1, 1024, 0, stream_>>>(d_keep_n_, c.n_nodes, d_ctotal_);
        compact_scan_kernel<<<1, 1024, 0, stream_>>>(d_keep_e_, c.n_nodes, d_ctotal_ + 1);
        int total[2] = {0, 0};
        ARA_CUDA_OK(cudaMemcpyAsync(total, d_ctotal_, sizeof(total), cudaMemcpyDeviceToHost, stream_));
        ARA_CUDA_OK(cudaStreamSynchronize(stream_));
        launches += 3;
        if (!pools_have_room(sp, max_nodes_, max_edges_, total[0], total[1])) continue;  // even the subtree alone is too big: new tree
        TreeDev& d = shadow_[i];
        if (d.hdr == nullptr) {
            d = t;
            if (alloc_pools(d)) return -1;
        }
        compact_gather_kernel<<<(c.n_nodes + 7) / 8, 256, 0, stream_>>>(t, d, c.cand, c.n_nodes, d_keep_n_, d_keep_e_);
        compact_finish_kernel<<<1, 1, 0, stream_>>>(t.st, total[0], total[1]);
        launches += 2;
        // swap the pools: the tree now lives in what was the second set
        for_each_pool([&](auto m, size_t) { std::swap(t.*m, d.*m); });
        ++compactions;
    }
    ARA_CUDA_OK(cudaGetLastError());
    ARA_CUDA_OK(cudaMemcpyAsync(d_trees_, h_trees_.data(), sizeof(TreeDev) * n_trees, cudaMemcpyHostToDevice, stream_));
    return 0;
}

// MCTSAgent::evaluate_board_state up to the first mini-batch: roots created (or taken over), evaluated, noised
int Search::begin() {
    ARA_CUDA_OK(cudaSetDevice(device_));
    prof_used_ = 0;
    net_forwards = 0;
    searched_ = true;
    stop_requested_.store(false, std::memory_order_relaxed);
    ARA_CUDA_OK(cudaEventRecord(ev0_, stream_));
    ARA_CUDA_OK(cudaMemcpyAsync(d_trees_, h_trees_.data(), sizeof(TreeDev) * n_trees, cudaMemcpyHostToDevice, stream_));
    ARA_CUDA_OK(cudaMemcpyAsync(d_roots_, h_roots_.data(), sizeof(Board) * n_trees, cudaMemcpyHostToDevice, stream_));
    if (compact_pools()) return -1;
    if (threads_ == 2) {  // the second thread's views of the trees: same pools, its own batch arrays
        for (int i = 0; i < n_trees; ++i) {
            TreeDev v = h_trees_[i];
            for_each_batch_array([&](auto m, size_t) { v.*m = h_trees1_[i].*m; });
            h_trees1_[i] = v;
            ARA_CUDA_OK(cudaMemsetAsync(v.bs, 0, sizeof(BatchState), stream_));
        }
        ARA_CUDA_OK(cudaMemcpyAsync(d_trees_slot_[1], h_trees1_.data(), sizeof(TreeDev) * n_trees, cudaMemcpyHostToDevice, stream_));
        primed_ = false;
    }
    __half* in_h = net_ ? net_->d_in_h : nullptr;
    const int cpad = net_ ? net_->cin_pad : 0;
    const int B = sp.batch_size;
    // root: create, expand, evaluate (set_root_node_predictions), scatter, prepare_node_for_visits (+ Dirichlet)
    ARA_CUDA_OK(cudaMemcpyAsync(d_limits_, h_limits_.data(), sizeof(uint2) * n_trees, cudaMemcpyHostToDevice, stream_));
    root_kernel<<<n_trees, 32, 0, stream_>>>(d_trees_, sp, d_roots_, d_limits_);
    if (n_trees > 1) {
        pack_kernel<<<1, 32, 0, stream_>>>(d_trees_, n_trees, d_count_);
        ++launches;
    }
    expand_kernel<<<n_trees * B, 32, 0, stream_>>>(d_trees_, sp, B, in_h, cpad, net_ ? net_->precision : 0);
    if (net_) {
        // a single-tree search only needs row 0; the new roots of a multi-tree search are packed into the first rows
        if (net_->forward_device(n_trees == 1 ? 1 : n_trees * B, stream_, n_trees > 1 ? d_count_ : nullptr)) return -1;
    } else {
        fake_eval_kernel<<<n_trees * B, 128, 0, stream_>>>(d_trees_, n_trees, B, d_values_, d_probs_, n_labels_);
        ++launches;
    }
    scatter_kernel<<<n_trees * B, 32, 0, stream_>>>(d_trees_, sp, B, net_ ? net_->d_value : d_values_,
                                                     net_ ? net_->d_prob : d_probs_, n_labels_);
    backup_kernel<<<n_trees, 32, 0, stream_>>>(d_trees_, sp, 1, net_ ? net_->d_value : d_values_);
    prepare_kernel<<<n_trees * 4 * B, 32, 0, stream_>>>(d_trees_, sp, 4 * B);
    launches += 5;
    ARA_CUDA_OK(cudaGetLastError());
    return 0;
}

// how many trees are still searching (reads the `done` flags; synchronises the search stream)
int Search::poll_running() {
    for (int i = 0; i < n_trees; ++i)
        ARA_CUDA_OK(cudaMemcpyAsync(&h_done_[i], &d_states_[i]->done, sizeof(int), cudaMemcpyDeviceToHost, stream_));
    ARA_CUDA_OK(cudaStreamSynchronize(stream_));
    int running = 0;
    for (int i = 0; i < n_trees; ++i) running += h_done_[i] == 0;
    if (running) {
        for (int i = 0; i < n_trees; ++i) {
            TreeState st;
            ARA_CUDA_OK(cudaMemcpy(&st, d_states_[i], sizeof(st), cudaMemcpyDeviceToHost));
            if (st.error)
                return set_error("ara_search: device search error %d (1 node pool, 2 edge pool, 3 depth > %d)", st.error, kMaxDepth);
        }
    }
    return running;
}

// SearchThread::thread_iteration n times (Threads = 2: n turns of each thread); returns the trees still running
int Search::step(int n_batches) {
    ARA_CUDA_OK(cudaSetDevice(device_));
    if (!searched_) return set_error("ara_search_step: ara_search_begin has not been called");
    if (n_batches < 1) return set_error("ara_search_step: n_batches %d < 1", n_batches);
    if (iterate(threads_ == 2 ? 2 * n_batches : n_batches)) return -1;
    const int running = poll_running();
    if (running < 0 || fetch_results()) return -1;  // ara_search_result between steps shows the tree as it is now
    return running;
}

int Search::node_view(int tree, int node_id, NodeView* out) {
    if (tree < 0 || tree >= n_trees) return set_error("ara_search_node: tree %d out of range", tree);
    if (!searched_) return set_error("ara_search_node: no search has been started on this handle");
    ARA_CUDA_OK(cudaSetDevice(device_));
    node_view_kernel<<<1, 32, 0, stream_>>>(d_trees_, tree, node_id, d_node_view_);
    ++launches;
    ARA_CUDA_OK(cudaMemcpyAsync(out, d_node_view_, sizeof(NodeView), cudaMemcpyDeviceToHost, stream_));
    ARA_CUDA_OK(cudaStreamSynchronize(stream_));
    if (out->node_id < 0) return set_error("ara_search_node: tree %d has no node %d", tree, node_id);
    return 0;
}

int Search::go() {
    if (begin()) return -1;
    const int B = sp.batch_size;
    // main loop: enqueue the iterations the visit budget certainly needs, then poll `done` in small chunks
    unsigned budget = sp.simulations ? sp.simulations : sp.nodes;
    int first = budget ? static_cast<int>(budget / (static_cast<unsigned>(B) * 1u)) : 8;
    if (first < 1) first = 1;
    // movetime (ThreadManager's stop after curMovetime, manager/threadmanager.cpp): iterations go out in small chunks
    // and the wall clock is read between them
    const auto t_start = std::chrono::steady_clock::now();
    auto elapsed_ms = [&]() { return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t_start).count(); };
    const bool managed = use_tc && n_trees == 1 && tc.movetime_ms > 0.0;
    const double move_ms = managed ? tc.movetime_ms : movetime_ms;
    const bool timed = move_ms > 0.0;
    if (timed && first > 4) first = 4;
    bool all_done = false;
    int chunk = first;
    int guard = 0;
    bool polled_root = false;
    // ThreadManager::stop_search_based_on_limits: the move time is spent in update intervals; after each one the early
    // stopping rule is consulted, and when a period of move time is over the search may be prolonged by another one
    double period_end = move_ms;
    double next_check = managed ? tc.update_interval_ms : 0.0;
    int checked = 0;
    float last_eval = tc.last_value_eval;
    tr = ara_time_report_t{};
    while (!all_done) {
        if (polled_root && stop_requested_.load(std::memory_order_relaxed)) break;
        if (timed && polled_root) {
            const double now = elapsed_ms();
            if (managed && now >= next_check && now < period_end) {
                RootStatsHost rs;
                if (read_time_stats(&rs)) return -1;
                const double remaining = period_end - next_check;  // remainingMoveTimeMS after this interval
                next_check += tc.update_interval_ms;
                tr.value_eval = rs.value_eval;
                if (checked == 0) {
                    const int rule = tm_early_stopping(tc, remaining, rs);
                    if (rule != 0 && !tm_continue_search(tc, remaining, rs, &checked, &last_eval)) {
                        tr.early_stopped = rule;
                        tr.saved_ms = remaining;
                        break;
                    }
                }
            }
            if (now >= period_end) {
                // `while (continue_search())` of the reference: what is left of the period by then is the division
                // remainder of move time by update interval, below the interval, so the literal rule cannot extend
                // the search here -- evaluated all the same, with the same arguments
                bool more = false;
                if (managed) {
                    RootStatsHost rs;
                    if (read_time_stats(&rs)) return -1;
                    tr.value_eval = rs.value_eval;
                    const double left = move_ms - std::floor(move_ms / tc.update_interval_ms) * tc.update_interval_ms;
                    more = tm_continue_search(tc, left, rs, &checked, &last_eval);
                }
                if (!more) break;
                period_end += move_ms;  // "Increase search time"
                next_check = now + tc.update_interval_ms;
            }
        }
        if (polled_root && iterate(chunk)) return -1;
        const int running = poll_running();
        if (running < 0) return -1;
        all_done = running == 0;
        if (polled_root) chunk = timed ? 4 : 2;
        polled_root = true;
        if (++guard > (1 << 22)) return set_error("ara_search_go: search did not terminate");
    }
    tr.prolonged = checked;
    tr.elapsed_ms = elapsed_ms();
    ARA_CUDA_OK(cudaEventRecord(ev1_, stream_));
    ARA_CUDA_OK(cudaEventSynchronize(ev1_));
    float ms = 0.0f;
    ARA_CUDA_OK(cudaEventElapsedTime(&ms, ev0_, ev1_));
    last_go_ms = ms;
    if (profile && prof_collect()) return -1;
    return 0;
}

int Search::set_limits(int tree, unsigned simulations, unsigned nodes) {
    if (tree < -1 || tree >= n_trees) return set_error("ara_search_set_limits: tree %d out of range", tree);
    if (simulations == 0 && nodes == 0) return set_error("ara_search_set_limits: neither Simulations nor Nodes given");
    for (int i = 0; i < n_trees; ++i)
        if (tree < 0 || tree == i) h_limits_[i] = make_uint2(simulations, nodes);
    return 0;
}

int Search::read_time_stats(RootStatsHost* out) {
    time_stats_kernel<<<1, 32, 0, stream_>>>(d_trees_, d_tstats_);
    ++launches;
    ARA_CUDA_OK(cudaMemcpyAsync(h_tstats_, d_tstats_, sizeof(RootTimeStats), cudaMemcpyDeviceToHost, stream_));
    ARA_CUDA_OK(cudaStreamSynchronize(stream_));
    static_assert(sizeof(RootStatsHost) == sizeof(RootTimeStats), "root statistics layout");
    memcpy(out, h_tstats_, sizeof(*out));
    return 0;
}

int Search::apply_move(int tree, unsigned short move) {
    if (tree < 0 || tree >= n_trees) return set_error("ara_search_apply_move: tree %d out of range", tree);
    ARA_CUDA_OK(cudaSetDevice(device_));
    if (!searched_) return 0;  // nothing to keep before the first search
    // d_trees_ still holds the descriptors of the last go (pool pointers never change)
    advance_kernel<<<1, 32, 0, stream_>>>(d_trees_, tree, static_cast<Move>(move));
    if (advanced_.empty()) advanced_.assign(n_trees, 0);
    advanced_[tree] = 1;
    ++launches;
    ARA_CUDA_OK(cudaGetLastError());
    return 0;
}

int Search::fetch_results() {
    ARA_CUDA_OK(cudaSetDevice(device_));
    result_kernel<<<n_trees, 32, 0, stream_>>>(d_trees_, sp, d_results_);
    ++launches;
    ARA_CUDA_OK(cudaMemcpyAsync(results.data(), d_results_, sizeof(SearchResult) * n_trees, cudaMemcpyDeviceToHost, stream_));
    ARA_CUDA_OK(cudaStreamSynchronize(stream_));
    for (const auto& r : results)
        if (r.error) return set_error("search error %d on device (1 node pool, 2 edge pool, 3 depth overflow)", r.error);
    return 0;
}

}  // namespace ara

// --------------------------------------------------------------------------------------------------------- C-ABI
using ara::Search;
static_assert(sizeof(ara_search_settings_t) == sizeof(ara::SearchParams), "settings layout");
static_assert(sizeof(ara_search_result_t) == sizeof(ara::SearchResult), "result layout");
static_assert(sizeof(ara_board_t) == sizeof(ara::Board), "board layout");

extern "C" void ara_search_default_settings(ara_search_settings_t* s, int mode) {
    // uci/optionsuci.cpp:66-220 (non-RL build)
    memset(s, 0, sizeof(*s));
    s->batch_size = mode == ara::MODE_CHESS ? 64 : 16;
    s->dirichlet_epsilon = 0.0f;
    s->dirichlet_alpha = 0.2f;
    s->node_policy_temperature = 1.7f;
    s->q_value_weight = 1.0f;
    s->q_veto_delta = 0.4f;
    s->cpuct_init = 2.5f;
    s->cpuct_base = 19652.0f;
    s->mcts_solver = 1;
    s->virtual_style = ara::VS_VIRTUAL_MIX;
    s->virtual_mix_threshold = 1000;
    s->seed = 42;
    s->threads = 1;  // the deterministic parity setting; the reference's UCI default is 2 (uci/optionsuci.cpp:182)
    s->mode = mode;
    s->input_version = mode == ara::MODE_CHESS ? 3 : 1;
}

extern "C" ara_search_t ara_search_create(ara_net_t net, const ara_search_settings_t* settings, int device, int n_trees,
                                          int max_nodes) {
    if (settings == nullptr) {
        ara::set_error("ara_search_create: null settings");
        return nullptr;
    }
    ara::SearchParams sp;
    memcpy(&sp, settings, sizeof(sp));
    std::unique_ptr<Search> s(new Search());
    if (s->init(reinterpret_cast<ara::Net*>(net), sp, device, n_trees, max_nodes) != 0) return nullptr;
    return reinterpret_cast<ara_search_t>(s.release());
}
extern "C" void ara_search_destroy(ara_search_t h) { delete reinterpret_cast<Search*>(h); }

extern "C" int ara_search_set_position(ara_search_t h, int tree, const ara_board_t* root, const unsigned long long* hist_keys,
                                       const short* hist_reps, int hist_len) {
    if (h == nullptr || root == nullptr) return ara::set_error("ara_search_set_position: null argument");
    ara::Board b;
    memcpy(&b, root, sizeof(b));
    return reinterpret_cast<Search*>(h)->set_position(tree, b, reinterpret_cast<const uint64_t*>(hist_keys), hist_reps, hist_len);
}
extern "C" int ara_search_go(ara_search_t h) {
    if (h == nullptr) return ara::set_error("ara_search_go: null handle");
    Search* s = reinterpret_cast<Search*>(h);
    if (s->go()) return -1;
    return s->fetch_results();
}
static_assert(sizeof(ara_node_view_t) == sizeof(ara::NodeView), "node view layout");
extern "C" int ara_search_begin(ara_search_t h) {
    if (h == nullptr) return ara::set_error("ara_search_begin: null handle");
    return reinterpret_cast<Search*>(h)->begin();
}
extern "C" int ara_search_step(ara_search_t h, int n_batches) {
    if (h == nullptr) return ara::set_error("ara_search_step: null handle");
    return reinterpret_cast<Search*>(h)->step(n_batches);
}
extern "C" int ara_search_node(ara_search_t h, int tree, int node_id, ara_node_view_t* out) {
    if (h == nullptr || out == nullptr) return ara::set_error("ara_search_node: null argument");
    return reinterpret_cast<Search*>(h)->node_view(tree, node_id, reinterpret_cast<ara::NodeView*>(out));
}

extern "C" int ara_search_result(ara_search_t h, int tree, ara_search_result_t* out) {
    if (h == nullptr || out == nullptr) return ara::set_error("ara_search_result: null argument");
    Search* s = reinterpret_cast<Search*>(h);
    if (tree < 0 || tree >= s->n_trees) return ara::set_error("ara_search_result: tree %d out of range", tree);
    memcpy(out, &s->results[tree], sizeof(*out));
    return 0;
}
extern "C" int ara_search_apply_move(ara_search_t h, int tree, unsigned short move) {
    if (h == nullptr) return ara::set_error("ara_search_apply_move: null handle");
    return reinterpret_cast<Search*>(h)->apply_move(tree, move);
}
extern "C" int ara_search_set_limits(ara_search_t h, int tree, unsigned simulations, unsigned nodes) {
    if (h == nullptr) return ara::set_error("ara_search_set_limits: null handle");
    return reinterpret_cast<Search*>(h)->set_limits(tree, simulations, nodes);
}

extern "C" int ara_search_stop(ara_search_t h) {
    if (h == nullptr) return ara::set_error("ara_search_stop: null handle");
    reinterpret_cast<Search*>(h)->request_stop();
    return 0;
}
extern "C" int ara_search_set_movetime(ara_search_t h, double ms) {
    if (h == nullptr) return ara::set_error("ara_search_set_movetime: null handle");
    reinterpret_cast<Search*>(h)->movetime_ms = ms > 0.0 ? ms : 0.0;
    return 0;
}
extern "C" int ara_search_set_time_control(ara_search_t h, const ara_time_control_t* tc) {
    if (h == nullptr) return ara::set_error("ara_search_set_time_control: null handle");
    Search* s = reinterpret_cast<Search*>(h);
    if (tc == nullptr) {
        s->use_tc = false;
        return 0;
    }
    if (!(tc->movetime_ms > 0.0) || !(tc->update_interval_ms > 0.0))
        return ara::set_error("ara_search_set_time_control: movetime %.1f ms / update interval %.1f ms must be positive",
                              tc->movetime_ms, tc->update_interval_ms);
    if (s->n_trees != 1) return ara::set_error("ara_search_set_time_control: the time manager drives single-tree searches");
    s->tc = *tc;
    s->use_tc = true;
    return 0;
}
extern "C" int ara_search_time_report(ara_search_t h, ara_time_report_t* out) {
    if (h == nullptr || out == nullptr) return ara::set_error("ara_search_time_report: null argument");
    *out = reinterpret_cast<Search*>(h)->tr;
    return 0;
}
extern "C" int ara_time_for_move(long movetime_ms, int time_me_ms, int inc_me_ms, int movestogo, int move_overhead_ms,
                                 int move_number) {
    return ara::tm_time_for_move(movetime_ms, time_me_ms, inc_me_ms, movestogo, move_overhead_ms, move_number);
}
extern "C" int ara_time_early_stopping(const ara_time_control_t* tc, double remaining_ms, unsigned node_count,
                                       int max_q_is_max_visits, unsigned first_visits, unsigned second_visits, float q_first,
                                       float q_second) {
    if (tc == nullptr) return ara::set_error("ara_time_early_stopping: null argument");
    const ara::RootStatsHost r{node_count, first_visits, second_visits, q_first, q_second, max_q_is_max_visits, 0.0f, 1};
    return ara::tm_early_stopping(*tc, remaining_ms, r);
}
extern "C" int ara_time_continue_search(const ara_time_control_t* tc, double remaining_ms, float value_eval, int* checked,
                                        float* last_value_eval) {
    if (tc == nullptr || checked == nullptr || last_value_eval == nullptr)
        return ara::set_error("ara_time_continue_search: null argument");
    ara::RootStatsHost r{};
    r.value_eval = value_eval;
    r.valid = 1;
    return ara::tm_continue_search(*tc, remaining_ms, r, checked, last_value_eval) ? 1 : 0;
}
extern "C" int ara_search_set_profile(ara_search_t h, int on) {
    if (h == nullptr) return ara::set_error("ara_search_set_profile: null handle");
    reinterpret_cast<Search*>(h)->profile = on != 0;
    return 0;
}
extern "C" int ara_search_profile(ara_search_t h, double* select_ms, double* net_ms, double* apply_ms, long long* net_forwards) {
    if (h == nullptr) return ara::set_error("ara_search_profile: null handle");
    Search* s = reinterpret_cast<Search*>(h);
    if (select_ms) *select_ms = s->select_ms;
    if (net_ms) *net_ms = s->net_ms;
    if (apply_ms) *apply_ms = s->apply_ms;
    if (net_forwards) *net_forwards = s->net_forwards;
    return 0;
}
extern "C" int ara_search_debug_cycles(ara_search_t h, int tree, unsigned long long* out8) {
    if (h == nullptr || out8 == nullptr) return ara::set_error("ara_search_debug_cycles: null argument");
    return reinterpret_cast<Search*>(h)->debug_cycles(tree, out8);
}
extern "C" double ara_search_last_go_ms(ara_search_t h) { return h ? reinterpret_cast<Search*>(h)->last_go_ms : 0.0; }
extern "C" long long ara_search_launch_count(ara_search_t h) { return h ? reinterpret_cast<Search*>(h)->launches : 0; }
extern "C" long long ara_search_compaction_count(ara_search_t h) { return h ? reinterpret_cast<Search*>(h)->compactions : 0; }

// ---- debug / unit-test entry: the device build of the glibc powf / logf restatement (glibc_flt32.cuh) on host buffers
__global__ void glibc_flt32_kernel(const float* x, const float* y, int n, float* pow_out, float* log_out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    if (pow_out) pow_out[i] = ara::glibc::powf_(x[i], y[i]);
    if (log_out) log_out[i] = ara::glibc::logf_(x[i]);
}
extern "C" int ara_debug_powf_logf(const float* x, const float* y, int n, float* pow_out, float* log_out) {
    if (n <= 0 || !x || !y) return ara::set_error("ara_debug_powf_logf: bad arguments");
    ara::DeviceBuffers mem;
    float *dx = nullptr, *dy = nullptr, *dp = nullptr, *dl = nullptr;
    const size_t bytes = sizeof(float) * static_cast<size_t>(n);
    if (mem.dalloc(&dx, n) || mem.dalloc(&dy, n) || mem.dalloc(&dp, n) || mem.dalloc(&dl, n)) return -1;
    ARA_CUDA_OK(cudaMemcpy(dx, x, bytes, cudaMemcpyHostToDevice));
    ARA_CUDA_OK(cudaMemcpy(dy, y, bytes, cudaMemcpyHostToDevice));
    glibc_flt32_kernel<<<(n + 255) / 256, 256>>>(dx, dy, n, pow_out ? dp : nullptr, log_out ? dl : nullptr);
    ARA_CUDA_OK(cudaGetLastError());
    if (pow_out) ARA_CUDA_OK(cudaMemcpy(pow_out, dp, bytes, cudaMemcpyDeviceToHost));
    if (log_out) ARA_CUDA_OK(cudaMemcpy(log_out, dl, bytes, cudaMemcpyDeviceToHost));
    return 0;
}
