/* ara_b200.h -- C-ABI of the H100-native (sm_90a) leaf-evaluation + MCTS engine.
 *
 * Every entry point is what the reference's C++ seam for this hot path would bind (file:line refer to
 * QueensGambit/CrazyAra, engine/src/...).  Plain pointers and sizes only; all functions return 0 on success
 * and -1 on failure with a message retrievable through ara_last_error() (thread local).  There is no CPU
 * fallback: creation fails on anything that is not an sm_90 device.
 */
#ifndef ARA_B200_H
#define ARA_B200_H

#ifdef __cplusplus
extern "C" {
#endif

typedef struct ara_net_s* ara_net_t;

/* Last error message of the calling thread ("" if none). */
const char* ara_last_error(void);

/* ---- Neural network seam: replaces NeuralNetAPI (nn/neuralnetapi.h:148-311) / TensorrtAPI (nn/tensorrtapi.cpp).
 *
 * ara_net_create  <-> TensorrtAPI::TensorrtAPI + NeuralNetAPI::initialize (nn/tensorrtapi.cpp:43-63,
 *                     nn/neuralnetapi.cpp:93-99): loads an ARAB2001 weight blob (crazyara_b200/weights.py), binds
 *                     device buffers and one CUDA stream on `device`, fixed maximum batch size.  `precision` is the
 *                     reference's UCI option `Precision` (uci/optionsuci.cpp:144, nn/tensorrtapi.cpp:334-360):
 *                     ARA_PRECISION_FLOAT16 (its default) = fp16 tensor-core operands, fp32 accumulation, fp16
 *                     activations; ARA_PRECISION_FLOAT32 = fp32-accurate: the same wgmma GEMMs with every operand
 *                     carried as an fp16 hi + lo pair (3x the K extent), fp32 activations between the layers --
 *                     value / probabilities within 1e-4 of an fp32 evaluation (tests/test_net_gpu.py).
 * ara_net_shape   <-> get_nb_input_values_total / get_nb_policy_values / get_nb_auxiliary_outputs /
 *                     is_policy_map / get_version / get_batch_size (nn/neuralnetapi.h:116-293).
 * ara_net_predict <-> NeuralNetAPI::predict(float* inputPlanes, float* valueOutput, float* probOutputs,
 *                     float* auxiliaryOutputs) (nn/neuralnetapi.h:237, nn/tensorrtapi.cpp:195-237):
 *                     planes [n, C, 8, 8] fp32 host -> value [n], prob [n, L] (softmax over ALL L labels, policy-map
 *                     order channel*64+square; with is_policy_map = 0, a fully-connected policy head's, the order of
 *                     the classic label list, crazyara_b200/labels.py), aux [n, A].  Synchronous.  n <= batch_size rows are evaluated
 *                     (the reference always runs the full batch; n < B just skips the unused rows).
 */
#define ARA_PRECISION_FLOAT16 0
#define ARA_PRECISION_FLOAT32 1
ara_net_t ara_net_create(const char* weights_path, int device, int batch_size, int precision);
void ara_net_destroy(ara_net_t net);
int ara_net_shape(ara_net_t net, int* in_channels, int* n_labels, int* n_aux, int* is_policy_map, int* input_version,
                  int* batch_size);
int ara_net_predict(ara_net_t net, const float* planes, int n, float* value, float* prob, float* aux);

/* Device-resident variant (inputs already in HBM; outputs stay in HBM): planes_dev [n, C, 8, 8] fp32 device
 * pointer, or NULL to evaluate the net's own NHWC fp16 input buffer filled by ara_encode_planes_device. */
int ara_net_forward_device(ara_net_t net, const float* planes_dev, int n, float** value_dev, float** prob_dev);

/* fill_nn_results for a host that keeps its own tree (searchthread.cpp:290-299 -> Node::set_probabilities_for_moves,
 * node.cpp:961-979): like ara_net_predict, but instead of the whole soft-maxed policy (L floats per position: 1.3 MB
 * at 64 x 5184) only the entries of each position's legal moves come back.  policy_idx [n][stride]: index into the
 * policy vector per legal move (ara_legal_moves gives them), counts [n] how many; priors_out [n][stride]. */
int ara_net_predict_priors(ara_net_t net, const float* planes, int n, const int* policy_idx, const int* counts, int stride,
                           float* value, float* priors_out, float* aux);
/* Pinned host memory for the caller-owned predict buffers, as NeuralNetAPIUser allocates them under TensorRT
 * (cudaMallocHost, nn/neuralnetapiuser.cpp:52-59): copies from / to it overlap and run at full PCIe / C2C speed. */
void* ara_host_alloc(unsigned long long bytes);
void ara_host_free(void* p);

/* Number of CUDA kernels this net has launched so far (bench bookkeeping). */
long long ara_net_launch_count(ara_net_t net);
/* profiling builds (-DARA_TRUNK_PROF) only: SM-clock cycles of CTA 0 of the last trunk-kernel launch, [0..15] MMA
 * issuer, [16..31] compute warp; all zero in the product build */
int ara_net_debug_trunk_cycles(ara_net_t net, unsigned long long* out32);

/* ---- Position seam: replaces State / BoardState for the supported variants (engine/src/state.h:287-509,
 * environments/chess_related/boardstate.{h,cpp}).  A position is one opaque 128-byte line (bitboards, pockets,
 * castling rooks, counters, Zobrist key, last 8 moves); it is what the device kernels read.
 * Variants: 0 chess (incl. chess960), 1 crazyhouse, 2 King of the Hill, 3 Three-check.
 * Moves are 16-bit: from | to<<6 | flag<<12 (flag 0 normal, 1-4 promotion N/B/R/Q, 5 en passant,
 * 6 castling king-from -> rook-from, 8+pt drop with from == to).
 */
typedef struct ara_board_s {
    unsigned long long w[16];
} ara_board_t;

/* State::set(fen, isChess960, variant) / State::fen() / StateConstants::action_to_uci -- host control plane */
int ara_board_from_fen(const char* fen, int variant, int is960, ara_board_t* out);
int ara_board_to_fen(const ara_board_t* board, char* buf, int buf_len);
int ara_move_to_uci(unsigned short move, int is960, char* buf8);

/* State::get_state_planes(normalize, float* planes, version) (state.h:354; board_to_planes,
 * inputrepresentation.cpp:628-680) for n positions at once: one warp per position on the GPU.
 * mode: 0 MODE_CRAZYHOUSE, 1 MODE_CHESS, 2 MODE_LICHESS (the reference's compile-time product mode);
 * version: 1, 2, 3.  planes_out: [n, C, 8, 8] fp32, C = 34/51/64, 39/52, 63/80.  Host buffers. */
int ara_encode_planes(const ara_board_t* boards, int n, int mode, int version, int normalize, float* planes_out);
/* device-resident variant: boards_dev [n] in HBM -> planes_dev [n,C,8,8] fp32 and/or planes_half_nhwc_dev
 * [n, 64, cpad] fp16 (the stem convolution's input layout, cpad 64 or 128 >= C, channels >= C zero); asynchronous on
 * `stream`.  The fp16 output is always normalised, as the network reads it: with planes_half_nhwc_dev set, normalize = 0
 * is refused.  n = 0 launches nothing and returns 0; n < 0 is refused. */
int ara_encode_planes_device(const void* boards_dev, int n, int mode, int version, int normalize, float* planes_dev,
                             void* planes_half_nhwc_dev, int cpad, void* stream);

/* State::legal_actions() + State::is_terminal() + StateConstants::action_to_index<normal, mirrored?> for n positions
 * (boardstate.cpp:61-69, :143-226, boardstate.h:73-97): moves_out [n][512], counts [n], terminal [n] (TerminalType:
 * 0 loss, 1 draw, 2 win, 4 none; repetition taken from the board's stored repetition info), policy_idx [n][512]
 * (index into the policy-map vector).  terminal / policy_idx may be NULL.  Host buffers, GPU kernel. */
int ara_legal_moves(const ara_board_t* boards, int n, unsigned short* moves_out, int* counts, int* terminal, int* policy_idx);

/* Game state with history (BoardState: position + the StateInfo chain that repetition detection walks).  Host control
 * plane for UCI "position ... moves ..." and the self-play loop; hands roots to ara_search_set_position. */
typedef struct ara_state_s* ara_state_t;
ara_state_t ara_state_create(const char* fen_or_null, int variant, int is960); /* State::set / State::init */
ara_state_t ara_state_clone(ara_state_t s);                                    /* State::clone */
void ara_state_destroy(ara_state_t s);
int ara_state_do_move(ara_state_t s, unsigned short move);                     /* State::do_action */
int ara_state_do_uci(ara_state_t s, const char* uci);                          /* uci_to_action + do_action */
int ara_state_board(ara_state_t s, ara_board_t* out);
int ara_state_history(ara_state_t s, const unsigned long long** keys, const short** reps, int* len);
int ara_state_fen(ara_state_t s, char* buf, int buf_len);                      /* State::fen */
int ara_state_legal_moves(ara_state_t s, unsigned short* moves_out);           /* returns the count */
int ara_state_side_to_move(ara_state_t s);
int ara_state_is_terminal(ara_state_t s);                                      /* TerminalType */
int ara_state_in_check(ara_state_t s);                                         /* 1 if the side to move is in check */
/* State::action_to_san -> pgn_move (environments/chess_related/board.cpp:277-359): SAN as the reference's PGN files
   spell it (promotion without '=', "O-O", drops "N@f3"); leads_to_win turns a trailing '+' into '#'.  buf16: >= 16 B */
int ara_state_move_to_san(ara_state_t s, unsigned short move, int leads_to_win, char* buf16);

/* ---- Search seam: replaces MCTSAgent::evaluate_board_state + SearchThread::thread_iteration + Node
 * (agents/mctsagent.cpp:292-337, searchthread.cpp:403-426, node.{h,cpp}) with a device-resident tree.
 * ara_search_settings_t carries SearchSettings + SearchLimits (agents/config/searchsettings.h:51-98,
 * searchlimits.h:37-61) with the reference's UCI defaults (uci/optionsuci.cpp:66-220).
 */
typedef struct ara_search_s* ara_search_t;
typedef struct ara_search_settings_s {
    int batch_size;                 /* Batch_Size */
    float dirichlet_epsilon;        /* Centi_Dirichlet_Epsilon / 100 */
    float dirichlet_alpha;          /* Centi_Dirichlet_Alpha / 100 */
    float node_policy_temperature;  /* Centi_Node_Temperature / 100 */
    float q_value_weight;           /* Centi_Q_Value_Weight / 100 */
    float q_veto_delta;             /* Centi_Q_Veto_Delta / 100 */
    float cpuct_init;               /* Centi_CPuct_Init / 100 */
    float cpuct_base;               /* CPuct_Base */
    int mcts_solver;                /* MCTS_Solver */
    int virtual_style;              /* 0 virtual_loss, 1 virtual_visit, 3 virtual_mix */
    unsigned virtual_mix_threshold; /* Virtual_Mix_Threshold */
    unsigned simulations;           /* SearchLimits::simulations (0 = no limit) */
    unsigned nodes;                 /* SearchLimits::nodes (0 = no limit) */
    unsigned long long seed;        /* seed of the Dirichlet generators: tree i of a handle starts from seed ^ i * 0x9E37..., and
                                       every root noise draw advances it (the reference seeds one process-wide
                                       std::default_random_engine from std::random_device, util/randomgen.h:35) */
    int mode;                       /* 0 MODE_CRAZYHOUSE, 1 MODE_CHESS, 2 MODE_LICHESS */
    int input_version;              /* input representation version 1, 2, 3 */
    int threads;                    /* Threads: 1 (deterministic parity mode) or 2 (the reference's default,
                                       uci/optionsuci.cpp:182): two logical search threads take turns on the tree in a
                                       fixed schedule, so that one thread's network batch is evaluated while the other
                                       thread selects its next one */
    int epsilon_greedy_counter;     /* round(100 / Centi_Epsilon_Greedy), 0 = off (uci/crazyara.cpp:748-749) */
    int epsilon_checks_counter;     /* round(100 / Centi_Epsilon_Checks), 0 = off */
    int reserved;
} ara_search_settings_t;

/* What update_eval_info (evalinfo.cpp:195-249) exposes: per root move visits / Q / prior / MCTS posterior, best
 * move, root value, node counters (nodes = visit_sum - free_visits, evalinfo.cpp:73-85), principal variation. */
typedef struct ara_search_result_s {
    int n_moves;
    int no_visit_idx;
    int best_idx;
    int node_type; /* 0 win, 1 draw, 2 loss, 3 unsolved */
    int pv_len;
    float root_value;
    float best_move_q;
    unsigned visit_sum;
    unsigned free_visits;
    unsigned iterations;
    unsigned evals;
    int tree_nodes;
    int error;
    unsigned nodes_pre_search; /* EvalInfo::nodesPreSearch: nodes of the kept subtree when the search began, 0 for a new tree */
    unsigned long long sum_select_k; /* sum over selections of the number of open children read (HBM accounting) */
    unsigned long long sum_depth;
    unsigned short moves[512];
    unsigned int visits[512];
    float q[512];
    float prior[512];
    double policy[512];
    unsigned short pv[256];
} ara_search_result_t;

void ara_search_default_settings(ara_search_settings_t* s, int mode);
/* net: handle whose batch size is >= n_trees * batch_size, or NULL to run the hash-derived fake backend (search-parity
 * tests).  n_trees independent positions are searched concurrently, one warp per tree, sharing each network batch.
 * Each tree's node, edge and prepared-child pools are reserved as device address ranges:
 *   - with Simulations or Nodes set, max_nodes <= 0 sizes them from that budget, max_nodes > 0 gives their size; they are
 *     mapped whole at creation;
 *   - without either, one tree's pools are reserved for max_nodes > 0 (a cap: the search ends when the tree reaches it)
 *     or, for max_nodes <= 0, for what the device's memory could hold (at most 2^31 - 1 edges), and mapped as the tree
 *     grows, ahead of every chunk of mini-batches.  Growth stops at the reservation or where it would leave the device
 *     less than a fixed margin of free memory; the search then ends as a full pool ends it, with its result.  Several
 *     trees without a budget need max_nodes (their pools are mapped whole). */
ara_search_t ara_search_create(ara_net_t net, const ara_search_settings_t* settings, int device, int n_trees, int max_nodes);
void ara_search_destroy(ara_search_t s);
/* root position of tree `tree` plus the (key, repetition) history of the game before it, oldest first */
int ara_search_set_position(ara_search_t s, int tree, const ara_board_t* root, const unsigned long long* hist_keys,
                            const short* hist_reps, int hist_len);
/* SearchLimits of the following go calls (searchlimits.h:37-61): simulations / nodes of tree `tree` (-1 = every tree)
 * instead of the settings' values.  Pools mapped whole at creation hold what the handle was created for, so the limits
 * must stay within that budget (ara_search_create max_nodes); pools that grow with the tree hold what their cap or the
 * device's memory allows.  Self-play jitters the node budget of every search
 * (SelfPlay::adjust_node_count, rl/selfplay.cpp:146-152). */
int ara_search_set_limits(ara_search_t s, int tree, unsigned simulations, unsigned nodes);
/* The Q-value weight of the posterior (Centi_Q_Value_Weight / 100, 0..999.99) and the Dirichlet epsilon of the root
 * noise (Centi_Dirichlet_Epsilon / 100, 0..1) of the following go calls for tree `tree` (-1 = every tree) instead of
 * the settings' values; a negative value means the settings' value again.  Like the limits, the values last until they
 * are changed.  Self-play's quick searches use it: a game that draws a quick search gets a smaller node budget, its
 * own Q-value weight and epsilon for that one search while the handle's other trees search as usual
 * (SelfPlay::generate_game, rl/selfplay.cpp:214-241). */
int ara_search_set_tree_settings(ara_search_t s, int tree, float q_value_weight, float dirichlet_epsilon);
/* tree -1 = every tree.  An inactive tree is left out of the following ara_search_begin / step / go calls until it is
 * made active again; new handles start with every tree active.  The set is read when a search begins.  An idle tree is
 * not touched: its statistics, its Dirichlet generator and a subtree kept by ara_search_apply_move stay as they are
 * (a second apply_move still descends from that subtree), it adds no row to the network batch, and ara_search_result
 * gives its last search's result (n_moves 0 if it has never searched).  With every tree idle no network forward runs
 * and step / go report 0 trees running.  A match between two networks uses this: each player's handle searches only
 * the games in which that player is to move (crazyara_b200/match.py). */
int ara_search_set_active(ara_search_t s, int tree, int active);
/* runs all trees to their limits (synchronous) and fetches the results */
int ara_search_go(ara_search_t s);
int ara_search_result(ara_search_t s, int tree, ara_search_result_t* out);
/* ---- stepping and inspection: SearchThread::thread_iteration (searchthread.cpp:403-416) and the Node getters
 * (node.h:97-124, :345-460; Node::print_node_statistics node.cpp:1248-1301) for a host that drives the search itself.
 *   ara_search_begin: MCTSAgent::evaluate_board_state up to the first mini-batch (agents/mctsagent.cpp:292-322): roots
 *                     created or taken over from the kept subtrees, evaluated, Dirichlet noise applied.
 *   ara_search_step:  n_batches more mini-batches per tree (thread_iteration n times; with Threads = 2, n_batches turns
 *                     of each thread); synchronous; returns the number of trees whose search loop has NOT ended yet
 *                     (0 = every tree is done; further calls are no-ops), or -1 on error.
 *   ara_search_go == ara_search_begin + ara_search_step until 0 (+ the time management).  ara_search_result may be
 *   called between steps.
 *   ara_search_node:  a read-only view of one node (node_id from ara_node_view_t.child[]; -1 = the current root). */
typedef struct ara_node_view_s {
    int node_id;          /* -1: no such node */
    int parent;           /* node id of the parent, -1 for the root of the tree */
    int parent_child_idx;
    int n_moves;          /* Node::get_number_child_nodes */
    int no_visit_idx;     /* Node::get_no_visit_idx: children opened so far; 0 until the node is a playout node */
    int node_type;        /* 0 win, 1 draw, 2 loss, 3 unsolved (nodedata.h NodeType) */
    int flags;            /* 1 terminal, 2 has NN results, 4 playout node (NodeData exists), 8 sorted */
    int checkmate_idx;    /* 65535 = none */
    int end_in_ply;
    int n_unsolved;
    int repetition;
    int pad_;
    unsigned visit_sum;   /* Node::get_visits */
    unsigned real_visits; /* Node::get_real_visits */
    unsigned free_visits;
    float value;          /* Node::get_value = valueSum / realVisits */
    double value_sum;
    unsigned long long key;      /* Node::hash_key */
    unsigned short moves[512];   /* Node::get_action(i), 16-bit move codes, sorted by prior once the node is visited */
    int child[512];              /* node id of child i or -1 (Node::get_child_node) */
    unsigned visits[512];        /* childNumberVisits */
    float q[512];                /* qValues */
    float prior[512];            /* policyProbSmall */
    unsigned char vl[512];       /* virtualLossCounter */
    unsigned char child_type[512];
} ara_node_view_t;
int ara_search_begin(ara_search_t s);
int ara_search_step(ara_search_t s, int n_batches);
int ara_search_node(ara_search_t s, int tree, int node_id, ara_node_view_t* out);
/* per-phase device times of the last go (CUDA events on the search stream); enable before ara_search_go */
/* MCTSAgent::apply_move_to_tree (agents/mctsagent.cpp:230-247): tells the tree which move was played.  The next go
 * on the position after that move (after both moves, when called twice) continues on the subtree behind it
 * (init_root_node / get_root_node_from_tree, :113-160) instead of starting a new tree -- provided the subtree's root is
 * that position, has been visited, and the node pool (ara_search_create max_nodes) has room for another search.  When
 * the dead siblings of the played moves have eaten that room, the kept subtree is first copied to the front of a second
 * set of pools (compaction; mapped at the first need), so a long game keeps its statistics as long as the subtree
 * itself plus one search fits.  Pools that grow with the tree compact every kept subtree at the start of the next go
 * and give the old set's memory back: such a handle holds the kept subtree plus what one search adds.
 * `move` is the engine's 16-bit move code (ara_search_result_t.moves). */
int ara_search_apply_move(ara_search_t s, int tree, unsigned short move);
/* ThreadManager's time stop (manager/threadmanager.cpp, SearchLimits::movetime): ms > 0 makes the following go calls
 * stop issuing mini-batches once that much wall time has passed (besides the Simulations / Nodes limits); 0 = off */
int ara_search_set_movetime(ara_search_t s, double ms);
/* UCI `stop` (SearchThread::stop, searchthread.cpp): may be called from another host thread while ara_search_go runs on
 * this handle; the go call returns after the mini-batches already enqueued (the result is valid as usual).  The only
 * entry point that may be used concurrently with another call on the same handle. */
int ara_search_stop(ara_search_t s);
/* ThreadManager's in-game heuristics (manager/threadmanager.cpp:68-178), evaluated every update interval on the root's
 * statistics: early stopping once the move is decided, one or two prolongations when the evaluation dropped.  The
 * parameters are what MCTSAgent::run_mcts_search hands to the ThreadManager (agents/mctsagent.cpp:350-352). */
typedef struct {
    double movetime_ms;        /* TimeManager::get_time_for_move; > 0 */
    double update_interval_ms; /* ThreadManagerParams::updateIntervalMS (250) */
    double overall_nps;        /* MCTSAgent::overallNPS, running mean over the game's searches; 0 = heuristics off */
    double safe_remaining_ms;  /* SearchLimits::get_safe_remaining_time(side to move) */
    double move_overhead_ms;   /* SearchLimits::moveOverhead */
    float last_value_eval;     /* MCTSAgent::lastValueEval: best-move Q of the previous search, -1 after ucinewgame */
    int in_game;               /* is_game_sceneario: wtime / btime / movestogo given */
    int can_prolong;           /* can_prolong_search(move number, TimeManager thresh move) */
} ara_time_control_t;
typedef struct {
    int early_stopped; /* 0 no, 1 "max nodes" rule, 2 "second move cannot catch up" rule */
    int prolonged;     /* number of times the search time was extended (checkedContinueSearch) */
    double saved_ms;   /* remaining move time when the search stopped early */
    double elapsed_ms; /* wall time of the go loop */
    float value_eval;  /* Node::updated_value_eval of the root at the last check */
} ara_time_report_t;
/* tc != NULL: the following go calls run under these limits (tc->movetime_ms replaces ara_search_set_movetime);
 * NULL switches the manager off again.  Single-tree searches only. */
int ara_search_set_time_control(ara_search_t s, const ara_time_control_t* tc);
int ara_search_time_report(ara_search_t s, ara_time_report_t* out);
/* TimeManager::get_time_for_move (manager/timemanager.cpp:51-98; constants.h:94-98; random factor off): the move time
 * in ms from `go movetime` / the mover's clock and increment / movestogo, less the move overhead.  Pure function. */
int ara_time_for_move(long movetime_ms, int time_me_ms, int inc_me_ms, int movestogo, int move_overhead_ms, int move_number);
/* the two decisions as pure functions (no device): root statistics in, verdict out -- for tests and host-side reuse */
int ara_time_early_stopping(const ara_time_control_t* tc, double remaining_ms, unsigned node_count, int max_q_is_max_visits,
                            unsigned first_visits, unsigned second_visits, float q_first, float q_second);
int ara_time_continue_search(const ara_time_control_t* tc, double remaining_ms, float value_eval, int* checked,
                             float* last_value_eval);
int ara_search_set_profile(ara_search_t s, int on);
int ara_search_profile(ara_search_t s, double* select_ms, double* net_ms, double* apply_ms, long long* net_forwards);
/* SM-clock cycles per phase of the select kernel in the last go (0 descent, 1 do_move, 2 movegen, 3 node init,
 * 4 plane encode, 5 terminal backup, 6 bookkeeping) -- profiling aid */
int ara_search_debug_cycles(ara_search_t s, int tree, unsigned long long* out8);
double ara_search_last_go_ms(ara_search_t s);       /* device time of the last go (CUDA events) */
long long ara_search_launch_count(ara_search_t s); /* search kernels launched so far */
/* How often a kept subtree (ara_search_apply_move) was moved to the front of the node / edge pools because they had no
 * room left for another search on top of the dead siblings (instead of giving the tree up). */
long long ara_search_compaction_count(ara_search_t s);
/* The pools of one tree (ara_search_pool). */
typedef struct {
    long long nodes;        /* nodes in use */
    long long edges;        /* edges in use */
    long long mapped_nodes; /* node capacity mapped: the device's pool test ends a search that reaches it */
    long long mapped_edges; /* edge capacity mapped */
    long long cap_nodes;    /* the reservation: max_nodes, the budget's pool, or what the device's memory could hold */
    long long cap_edges;
    long long mapped_bytes; /* device memory mapped for the tree's pools, both sets */
    long long spare_bytes;  /* of which the compaction's second set (0 after a growing tree's compaction) */
    long long grows;        /* times pools of the handle were mapped further since its creation */
    int growing;            /* 1: mapped as the tree grows; 0: mapped whole at creation */
} ara_search_pool_t;
int ara_search_pool(ara_search_t s, int tree, ara_search_pool_t* out);

/* ---- debug / unit-test entries
 * ara_debug_conv: one wgmma convolution layer on caller-provided device buffers, built and launched as the network builds
 * and launches each of its convolutions (Net::build_conv, Net::launch_conv); synchronous on `stream`.
 *   act        fp16 activations [boards_cap][64][act_pitch]; float16 reads channels 0 .. act_cin (0: cin), float32 the
 *              split [hi | hi | lo] of 3 * ceil64(cin) channels (act_cin ignored); act_pitch 0: as many as it reads
 *   w          fp16 weight image [w_rows][ksize^2 * parts * ceil64(cin)], per tap w (parts 1) or, float32, hi | lo | hi
 *   bias       fp32 [w_rows] zero padded, or NULL
 *   res_h      fp16 residual (float16) / res_f fp32 residual (float32), rows ldr apart, added after the ReLU, or NULL
 *   out_h, out_f, out_s   fp16, fp32 (rows ldo apart) and, float32 only, split outputs [rows][3 * split_cs], or NULL;
 *              columns 0 .. n_end (0: ldo) are written, rows 0 .. 64 * boards
 *   boards_dev device-side count of the boards in use (<= boards): M tiles beyond it leave at once; or NULL
 *   bn         the N tile, 64, 128 or 256; 0: the one ara_debug_choose_bn(boards, n_out) gives */
typedef struct ara_debug_conv_s {
    const void* act;
    const void* w;
    const float* bias;
    const void* res_h;
    const float* res_f;
    void* out_h;
    float* out_f;
    void* out_s;
    const int* boards_dev;
    int precision;
    int boards_cap;
    int boards;
    int cin;
    int n_out;
    int ksize;
    int relu;
    int w_rows;
    int act_cin;
    int act_pitch;
    int ldr;
    int ldo;
    int n_end;
    int split_cs;
    int bn;
} ara_debug_conv_t;
int ara_debug_conv(const ara_debug_conv_t* args, void* stream);
int ara_debug_choose_bn(int boards, int n_out);
/* ara_debug_ntb_attention: the attention of one NTB of width M (M / 32 heads) on host buffers, launched as the network
 * launches it (Net::enqueue_ntb_half / enqueue_ntb_precise); synchronous.
 *   qkv   [n * 64][3M] q | k | v: fp16 for precision 0, fp32 for precision 1
 *   count >= 0: a device-side board count of that value (<= n), as a search passes; -1: none
 *   out   in: the initial contents, out: the result; fp16 [n * 64][M], or for precision 1 the split [n * 64][3 * ceil64(M)]
 *         (hi | hi | lo)
 * M outside 32 .. 224 or not a multiple of 32, n < 1 and other precisions are refused before any device call. */
int ara_debug_ntb_attention(const void* qkv, int n, int M, int precision, int count, void* out);
/* ara_debug_policy_fc: the fully-connected policy layer (policy_fc_kernel, then policy_fc_softmax_kernel) on host
 * buffers, built and launched as the network builds and launches it (Net::build_policy_fc, launch_policy_head);
 * synchronous.
 *   P, L      policy planes (1 .. 256) and labels (1968, 2272 or 2316)
 *   boards    boards launched, 1 .. batch; batch: the batch the layer is built for, which fixes the N tile and rows_cap
 *             (batch rounded up to even, at least 2); bn 32, 64 or 128 forces the N tile, 0 takes the network's
 *   count     >= 0: a device-side board count of that value (<= boards); -1: none
 *   w_fc      [L][P * 64] (the trainer's NCHW flatten), b_fc [L]
 *   x         the policy convolution's output as the layer reads it: fp16 [rows_cap][64 * ceil32(P)], or for precision 1
 *             the split [rows_cap][64 * 3 * ceil64(P)] (per square hi | hi | lo)
 *   part      in: initial contents, out: the fp32 partial sums [splits][rows_cap][ceil64(L)]
 *   prob      in: initial contents, out: the probabilities [boards][L]
 *   splits, kb_per_split   out (or NULL): the split count and the 64-wide K blocks per split of the layer
 * With x, part and prob all NULL only splits and kb_per_split are reported, and no device is touched. */
int ara_debug_policy_fc(int precision, int P, int L, int boards, int batch, int bn, int count, const float* w_fc,
                        const float* b_fc, const void* x, float* part, float* prob, int* splits, int* kb_per_split);
/* the residual tower kernel alone on host buffers, on the shape ARA_TRUNK_ROWS selects: x_half, out_half [n][64][256]
 * fp16; per block (no squeeze-excitation), one after the other: w1 [c_op][256], b1 [c_op], wd [c_op][k*k], bd [c_op],
 * w2 [256][c_op], b2 [256] (BN folded) */
int ara_debug_trunk(const void* x_half, int n, int n_blocks, const int* c_op, const int* ksize, const float* w1,
                    const float* b1, const float* wd, const float* bd, const float* w2, const float* b2, void* out_half);
/* ara_debug_trunk with squeeze-excitation and the MXNet block semantics.  Per block: se_type (0 none, 1 ca_se, 2 eca_se),
 * gate (0 hard sigmoid x / 6 + 0.5, 1 hard sigmoid 0.2 x + 0.5, 2 logistic), flags (1: the shortcut is the block input
 * before the squeeze-excitation) and se_bias (bit 0: se_b given, bit 1: se_b1 given).  Concatenated over the blocks
 * that have them: se_w1t (ca_se [256][128], eca_se [256][256], transposed), se_w2t (ca_se [128][256]), se_b [256] (eca_se
 * bias, ca_se fc2 bias), se_b1 [128] (ca_se fc1 bias).  eca_se takes se_b; ca_se both biases or neither; a gate out of
 * range or other flags are refused.  A block with a flag, a gate other than 0 or se_b1 selects the kernels built for
 * the MXNet semantics, and *mx_out (if not NULL) reports that choice (1) or the PyTorch one (0). */
int ara_debug_trunk_se(const void* x_half, int n, int n_blocks, const int* c_op, const int* ksize, const int* se_type,
                       const int* gate, const int* flags, const int* se_bias, const float* w1, const float* b1, const float* wd,
                       const float* bd, const float* w2, const float* b2, const float* se_w1t, const float* se_w2t,
                       const float* se_b, const float* se_b1, void* out_half, int* mx_out);
/* the device build of the glibc powf / logf restatement the search uses for apply_temperature (util/blazeutil.h:78-88)
 * and the Dirichlet gamma sampler (:113-124): pow_out[i] = powf(x[i], y[i]), log_out[i] = logf(x[i]); host buffers,
 * either output may be NULL.  tests/test_glibc_flt32.py compares it with the host libm bit for bit. */
int ara_debug_powf_logf(const float* x, const float* y, int n, float* pow_out, float* log_out);

#ifdef __cplusplus
}
#endif
#endif /* ARA_B200_H */
