// create_mini_batch as a WAVEFRONT over several warps of one CTA (device only).
//
// The reference's search thread runs its playouts one after the other (searchthread.cpp:347-380); a playout is a chain
// of dependent memory round trips, so one warp per tree leaves the SM idle most of the time.  Here kWaveWarps warps of
// one CTA run consecutive playouts of the SAME tree concurrently, and the result is still the sequential one:
//
//   * playout k takes its step at ply L only after every older playout in flight has taken (or will never take) its
//     own step at ply L -- so at every node it sees exactly the virtual visits of the playouts before it;
//   * what a playout changes apart from its virtual visits happens at its COMMIT, and commits are in playout order:
//       - new leaf: node id, header, child link, the parent's no_visit_idx, the trajectory row.  The parent is
//         published as blocked (`blk`) before the step is released, younger playouts wait in front of that node;
//       - collision: the trajectory row only;
//       - terminal: the free backup rewrites Q/N along the path.  Younger playouts in flight have read values the
//         sequential order would have shown them AFTER that backup: they take their virtual visits back (youngest
//         first, restoring what they overwrote) and start again once the backup is done;
//   * a playout starts only if the loop condition of create_mini_batch holds for it whatever the older playouts in
//     flight turn out to be (new / collision / terminal), so nothing ever has to be cut off at the end of a batch.
//
// Shared-memory flags carry the hand-offs (`__threadfence_block()` orders the global stores around them).  Every spin
// is bounded: a protocol error ends the batch with TreeState::error = 4 instead of hanging the GPU.
#pragma once
#include "search_dev.cuh"

#if defined(__CUDACC__)
namespace ara {

#if !defined(ARA_WAVE_WARPS)
#define ARA_WAVE_WARPS 12
#endif
constexpr int kWaveWarps = ARA_WAVE_WARPS;
constexpr int kWaveNone = 0x7fffffff;
constexpr int kWaveLevelBits = 10;
constexpr int kWaveLevelOver = (1 << kWaveLevelBits) - 1;  // the playout's descent is over: it passes every deeper ply
constexpr int kWaveSpinLimit = 1 << 24;
static_assert(kMaxDepth < kWaveLevelOver, "ply counter of the wavefront state word");

struct WaveShared {
    TreeState st;                     // the tree's counters while the kernel runs (written back at the end)
    volatile int state[kWaveWarps];   // playout << 10 | plies passed, of the warp's playout in flight; -1: none
    volatile int blk[kWaveWarps];     // node whose expansion that playout will commit; -1: none
    volatile int ack[kWaveWarps];     // last abort (playout index of the terminal) this warp has answered
    volatile int started;             // youngest playout that has published its state (playouts start in order)
    volatile int committed;           // youngest committed playout
    volatile int abort_at;            // playout that is committing a terminal, kWaveNone otherwise
    volatile int over;                // 1: mini-batch complete (or failed), 2: the thread left its loop before the batch
    volatile int n_new, n_coll, n_term;
    int n_exp;
};
struct WaveUndo {  // what a playout overwrote, per step
    float q[kMaxDepth];
    uint8_t flags[kMaxDepth];
};
struct alignas(16) WaveWarp {
    WarpScratch ws;
    WaveUndo undo;
};
constexpr size_t kWaveSharedBytes = (sizeof(WaveShared) + 15) / 16 * 16;
constexpr size_t kWaveSmemBytes = kWaveSharedBytes + kWaveWarps * sizeof(WaveWarp);

// -DARA_PROF_FINE: warp-cycles per phase, summed over the warps into TreeState::prof (tools/prof_select.py):
// 0 start gate, 1 ply hand-off waits, 2 steps (loads, argmax, stores), 3 leaf preparation, 4 commit wait, 5 commit,
// 6 answering a terminal's abort, 7 number of playouts taken back
#if defined(ARA_PROF_FINE)
#define WAVE_PROF(S, idx, t0)                                                                          \
    do {                                                                                               \
        const long long now_ = clock64();                                                              \
        if (ARA_LANE == 0) atomicAdd(&(S).st.prof[idx], static_cast<unsigned long long>(now_ - (t0))); \
        (t0) = now_;                                                                                   \
    } while (0)
#define WAVE_COUNT(S, idx) do { if (ARA_LANE == 0) atomicAdd(&(S).st.prof[idx], 1ull); } while (0)
#else
#define WAVE_PROF(S, idx, t0) do { } while (0)
#define WAVE_COUNT(S, idx) do { } while (0)
#endif

__device__ __forceinline__ void wave_fail(WaveShared& S, int code) {
    if (ARA_LANE == 0) {
        if (!S.st.error) S.st.error = code;
        S.over = 1;
    }
    __syncwarp();
}
__device__ __forceinline__ void wave_backoff() { __nanosleep(40); }

// every older playout in flight has passed ply `level` and none of them holds `node` for an expansion
__device__ __forceinline__ bool wave_can_step(const WaveShared& S, int w, int k, int level, int node) {
    bool ok = true;
    if (ARA_LANE < kWaveWarps && ARA_LANE != w) {
        const int s = S.state[ARA_LANE];
        if (s >= 0 && (s >> kWaveLevelBits) < k)
            ok = (s & kWaveLevelOver) > level && S.blk[ARA_LANE] != node;
    }
    return __all_sync(0xffffffffu, ok);
}

// 0: go, 1: a terminal is being committed (take the visits back), 2: the batch is over
__device__ __forceinline__ int wave_acquire(WaveShared& S, int w, int k, int level, int node) {
    for (int spin = 0;; ++spin) {
        const int ab = S.abort_at, ov = S.over;
        if (__any_sync(0xffffffffu, ov != 0)) return 2;
        if (__any_sync(0xffffffffu, ab != kWaveNone)) return 1;
        if (wave_can_step(S, w, k, level, node)) break;
        if (spin > kWaveSpinLimit) {
            wave_fail(S, 4);
            return 2;
        }
        wave_backoff();
    }
    __threadfence_block();
    return 0;
}

// A terminal (playout S.abort_at) is being committed.  k >= 0: this warp's playout in flight with `steps` virtual
// visits applied -- taken back here, after every younger playout has taken back its own.  Returns when the backup is done.
__device__ void wave_answer_abort(WaveShared& S, const TreeDev& t, const SearchParams& sp, WaveWarp& W, int w, int k,
                                  int steps) {
    const int epoch = __shfl_sync(0xffffffffu, S.abort_at, 0);
    if (epoch == kWaveNone) return;
    if (k >= 0) {
        for (int spin = 0;; ++spin) {
            bool ok = true;
            if (ARA_LANE < kWaveWarps && ARA_LANE != w) {
                const int s = S.state[ARA_LANE];
                if (s >= 0 && (s >> kWaveLevelBits) > k) ok = S.ack[ARA_LANE] == epoch;
            }
            if (__all_sync(0xffffffffu, ok)) break;
            if (spin > kWaveSpinLimit || S.over) {
                wave_fail(S, 4);
                return;
            }
            wave_backoff();
        }
        __threadfence_block();
        if (ARA_LANE == 0) {
            for (int i = steps - 1; i >= 0; --i) {
                const uint32_t e = W.ws.traj_edge[i];
                const uint32_t n = t.N[e] - 1;
                t.N[e] = n;
                t.vl[e] = static_cast<uint8_t>(t.vl[e] - 1);
                if (virtual_style_of(sp, n) == VS_VIRTUAL_LOSS) t.Q[e] = W.undo.q[i];
                NodeHdr* hp = &t.hdr[W.ws.traj_node[i]];
                const uint32_t vs = hp->visit_sum - 1;
                hp->visit_sum = vs;
                hp->cput = current_cput(t, sp, vs);
                hp->sqrt_vs = sqrt_visits(t, vs);
                hp->flags = W.undo.flags[i];
            }
            __threadfence_block();
            S.blk[w] = -1;
            S.state[w] = -1;
        }
    }
    if (ARA_LANE == 0) {
        __threadfence_block();
        S.ack[w] = epoch;
    }
    __syncwarp();
    for (int spin = 0;; ++spin) {
        const int ab = S.abort_at, ov = S.over;
        if (__all_sync(0xffffffffu, ab != epoch) || __any_sync(0xffffffffu, ov != 0)) break;
        if (spin > kWaveSpinLimit) {
            wave_fail(S, 4);
            return;
        }
        wave_backoff();
    }
    __threadfence_block();
}

// One mini-batch of tree `t_in` by the kWaveWarps warps of this CTA (blockDim.x == 32 * kWaveWarps).
__device__ void wave_mini_batch(const TreeDev& t_in, const SearchParams& sp, WaveShared& S, WaveWarp& W) {
    const int w = static_cast<int>(threadIdx.x) >> 5;
    WarpScratch& ws = W.ws;
    TreeDev t = t_in;
    t.st = &S.st;
    if (w == 0) {
        if (ARA_LANE == 0) {
            S.st = *t_in.st;
            for (int i = 0; i < kWaveWarps; ++i) S.state[i] = -1, S.blk[i] = -1, S.ack[i] = -1;
            S.started = -1, S.committed = -1, S.abort_at = kWaveNone, S.over = 0;
            S.n_new = 0, S.n_coll = 0, S.n_term = 0, S.n_exp = 0;
            if (thread_loop_ends(t, sp)) S.over = 2;
        }
    }
    __syncthreads();
    const int B = sp.batch_size;
    const int root = S.st.root;

    for (int k = w; !__any_sync(0xffffffffu, S.over != 0); k += kWaveWarps) {
    restart:
        long long tw = clock64();
        (void)tw;
        // ---------------------------------------------------------------- start gate
        for (int spin = 0;; ++spin) {
            if (__any_sync(0xffffffffu, S.over != 0)) goto out;
            if (__any_sync(0xffffffffu, S.abort_at != kWaveNone)) {
                WAVE_PROF(S, 0, tw);
                wave_answer_abort(S, t, sp, W, w, -1, 0);
                WAVE_PROF(S, 6, tw);
                continue;
            }
            bool go = false;
            if (ARA_LANE == 0 && S.started == k - 1) {
                const int c = S.committed;
                const int nn = S.n_new, nc = S.n_coll, nt = S.n_term;
                __threadfence_block();
                const int infl = k - 1 - c;
                go = S.committed == c && nn + infl < B && nc + infl < B && nt + infl < 2 * B;
            }
            if (__any_sync(0xffffffffu, go)) break;
            if (spin > kWaveSpinLimit) {
                wave_fail(S, 4);
                goto out;
            }
            wave_backoff();
        }
        if (ARA_LANE == 0) {
            S.blk[w] = -1;
            S.state[w] = k << kWaveLevelBits;
            __threadfence_block();
            S.started = k;
        }
        __syncwarp();
        WAVE_PROF(S, 0, tw);
        {
            // ------------------------------------------------------------ descent
            int cur = root, depth = 0, type = -1, leaf = -1, ci = 0;
            unsigned long long sel_k = 0;
            NodeHdr h;
            EdgeRegs pre;
            int rc = wave_acquire(S, w, k, 0, cur);
            WAVE_PROF(S, 1, tw);
            if (rc == 0) {
                load_hdr(&h, &t.hdr[cur]);
                pre = load_edge(t, h.edge_base + ARA_LANE);
            }
            while (rc == 0) {
                if (depth >= kMaxDepth) {
                    wave_fail(S, 3);
                    rc = 2;
                    break;
                }
                // select_and_visit without the look-ahead loads (h and pre were read after wave_acquire); the edge's old
                // Q goes to the undo record
                const SelectPick pk = pick_child(t, sp, h, pre, -1);
                ci = pk.ci;
                const int owner_lane = ci & (ARA_WARP_N - 1);
                const int next = __shfl_sync(0xffffffffu, pk.x.c, owner_lane);
                const uint32_t cb = __shfl_sync(0xffffffffu, pk.x.cb, owner_lane);
                const float old_q = __shfl_sync(0xffffffffu, pk.x.q, owner_lane);
                apply_visit(t, sp, cur, h, pk);
                sel_k += static_cast<unsigned long long>(pk.counted_k);
                if (ARA_LANE == 0) {
                    record_step(ws, depth, cur, ci, h);
                    W.undo.q[depth] = old_q;
                    W.undo.flags[depth] = h.flags;
                    if (next < 0) S.blk[w] = cur;
                }
                depth++;
                __threadfence_block();  // the step's stores (all lanes) before the hand-off
                __syncwarp();
                if (ARA_LANE == 0) S.state[w] = (k << kWaveLevelBits) | depth;
                if (next < 0) {
                    type = 0;
                    break;
                }
                // the child: if nobody older can still touch it the loads below are final, otherwise wait and reload
                const bool fresh = wave_can_step(S, w, k, depth, next) && __all_sync(0xffffffffu, S.abort_at == kWaveNone);
                __threadfence_block();
                NodeHdr ch;
                load_hdr(&ch, &t.hdr[next]);
                EdgeRegs cpre = load_edge(t, cb + ARA_LANE);
                if (ch.flags & NF_TERMINAL) {  // (these two flags of an existing node do not change inside this kernel)
                    type = 2, leaf = next;
                    break;
                }
                if (!(ch.flags & NF_HAS_NN)) {
                    type = 1, leaf = next;
                    break;
                }
                if (!fresh) {
                    WAVE_PROF(S, 2, tw);
                    rc = wave_acquire(S, w, k, depth, next);
                    WAVE_PROF(S, 1, tw);
                    if (rc) break;
                    load_hdr(&ch, &t.hdr[next]);
                    cpre = load_edge(t, cb + ARA_LANE);
                }
                cur = next;
                h = ch;
                pre = cpre;
            }
            int tt = TERM_NONE, slot = 0;
            bool prepared = false;
            WAVE_PROF(S, 2, tw);
            if (rc == 0) {
                __syncwarp();
                if (ARA_LANE == 0) S.state[w] = (k << kWaveLevelBits) | kWaveLevelOver;
                if (type == 0) {
                    // the unordered half of the expansion: position, repetition state and verdict of the new leaf
                    // (the parent is blocked for younger playouts, its prepared slots are stable)
                    tt = leaf_board(t, ws, cur, ci, h, &slot, &prepared);
                    if (tt < 0) tt = leaf_verdict(t, ws, depth);
                }
                WAVE_PROF(S, 3, tw);
                // ---------------------------------------------------------- wait for the commit turn
                for (int spin = 0;; ++spin) {
                    const int ab = S.abort_at, ov = S.over, c = S.committed;
                    if (__any_sync(0xffffffffu, ov != 0)) {
                        rc = 2;
                        break;
                    }
                    if (__any_sync(0xffffffffu, ab != kWaveNone)) {
                        rc = 1;
                        break;
                    }
                    if (__all_sync(0xffffffffu, c == k - 1)) break;
                    if (spin > kWaveSpinLimit) {
                        wave_fail(S, 4);
                        rc = 2;
                        break;
                    }
                    wave_backoff();
                }
            }
            WAVE_PROF(S, 4, tw);
            if (rc == 2) goto out;
            if (rc == 1) {
                wave_answer_abort(S, t, sp, W, w, k, depth);
                WAVE_PROF(S, 6, tw);
                WAVE_COUNT(S, 7);
                goto restart;
            }
            __threadfence_block();
            // -------------------------------------------------------------- commit (playout order)
            if (type == 0) {
                if (ARA_LANE == 0) commit_parent(t, cur, h, slot, prepared, S.n_exp, B);
                __syncwarp();
                leaf = expand_node_alloc(t, sp, ws, cur, ci, tt, h.edge_base);
                if (leaf < 0) {
                    wave_fail(S, 1);
                    goto out;
                }
                if (tt != TERM_NONE) type = 2;
            }
            if (type == 2) {
                // younger playouts in flight give their virtual visits back before the backup rewrites the path
                if (ARA_LANE == 0) {
                    __threadfence_block();
                    S.abort_at = k;
                }
                __syncwarp();
                for (int spin = 0;; ++spin) {
                    bool ok = true;
                    if (ARA_LANE < kWaveWarps && ARA_LANE != w) ok = S.ack[ARA_LANE] == k;
                    if (__all_sync(0xffffffffu, ok)) break;
                    if (spin > kWaveSpinLimit || S.over) {
                        wave_fail(S, 4);
                        goto out;
                    }
                    wave_backoff();
                }
                __threadfence_block();
                if (ARA_LANE == 0) S.started = k;
            }
            store_trajectory(t, sp, ws, type, type == 1 ? B + S.n_coll : S.n_new, 0, depth, leaf);
            __syncwarp();
            if (ARA_LANE == 0) {
                S.st.sum_select_k += sel_k;
                int nn = S.n_new, nc = S.n_coll, nt = S.n_term;
                if (type == 2) S.n_term = ++nt;
                else if (type == 1) S.n_coll = ++nc;
                else S.n_new = ++nn;
                if (!(nn < B && nc != B && nt < 2 * B)) S.over = 1;
                __threadfence_block();
                S.blk[w] = -1;
                S.state[w] = -1;
                S.committed = k;
                __threadfence_block();
                if (type == 2) S.abort_at = kWaveNone;
            }
            __syncwarp();
            WAVE_PROF(S, 5, tw);
        }
    }
out:
    __syncthreads();
    if (threadIdx.x == 0) {
        if (S.over != 2) end_mini_batch(S.st, *t.bs, S.n_new, S.n_coll, S.n_exp);
        *t_in.st = S.st;
    }
}

}  // namespace ara
#endif
