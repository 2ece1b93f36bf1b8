// C++ host classes over the C-ABI (include/ara_b200.h), keeping the reference's engine surface:
//   NeuralNetAPI   engine/src/nn/neuralnetapi.h:148-311      (predict on caller-owned host buffers, shape getters)
//   BoardState     engine/src/environments/chess_related/boardstate.h (State interface, engine/src/state.h:287-509)
//   SearchSettings / SearchLimits   engine/src/agents/config/searchsettings.h, searchlimits.h
//   EvalInfo       engine/src/evalinfo.h
//   MCTSAgent      engine/src/agents/mctsagent.h: evaluate_board_state() -> device-resident search
//   RawNetAgent    engine/src/agents/rawnetagent.h: evaluate_board_state() -> the network's policy alone
//   SearchThread   engine/src/searchthread.h: thread_iteration() = one mini-batch of the device search (ara_search_step)
//   Node           engine/src/node.h: read-only view of a node of the device-resident tree (ara_search_node)
// Errors are rethrown as std::runtime_error / std::invalid_argument like the reference's backends do.
#pragma once
#include <cmath>
#include <cstring>
#include <memory>
#include <stdexcept>
#include <string>
#include <vector>

#include "ara_b200.h"

namespace crazyara {

using Action = unsigned short;

class NeuralNetAPI {
   public:
    // precision: the UCI option `Precision` (uci/optionsuci.cpp:144): "float16" (default) or "float32"
    NeuralNetAPI(const std::string& ctx, int deviceID, unsigned int batchSize, const std::string& modelFile,
                 const std::string& precision = "float16")
        : deviceID_(deviceID), batchSize_(batchSize) {
        if (ctx != "gpu") throw std::invalid_argument("crazyara_b200 has no CPU context");
        if (precision != "float16" && precision != "float32") throw std::invalid_argument("Precision must be float16 or float32");
        net_ = ara_net_create(modelFile.c_str(), deviceID, static_cast<int>(batchSize),
                              precision == "float32" ? ARA_PRECISION_FLOAT32 : ARA_PRECISION_FLOAT16);
        if (net_ == nullptr) throw std::invalid_argument(ara_last_error());
        int b = 0;
        ara_net_shape(net_, &nbInputChannels_, &nbPolicyValues_, &nbAux_, &isPolicyMap_, &version_, &b);
    }
    ~NeuralNetAPI() { ara_net_destroy(net_); }
    NeuralNetAPI(const NeuralNetAPI&) = delete;
    NeuralNetAPI& operator=(const NeuralNetAPI&) = delete;
    void predict(float* inputPlanes, float* valueOutput, float* probOutputs, float* auxiliaryOutputs) {
        if (ara_net_predict(net_, inputPlanes, static_cast<int>(batchSize_), valueOutput, probOutputs, auxiliaryOutputs) != 0)
            throw std::runtime_error(ara_last_error());
    }
    unsigned int get_batch_size() const { return batchSize_; }
    unsigned int get_nb_input_values_total() const { return nbInputChannels_ * 64; }
    unsigned int get_nb_policy_values() const { return nbPolicyValues_; }
    unsigned int get_nb_auxiliary_outputs() const { return nbAux_; }
    bool is_policy_map() const { return isPolicyMap_ != 0; }
    int get_version() const { return version_; }
    ara_net_t handle() const { return net_; }

   private:
    ara_net_t net_ = nullptr;
    int deviceID_;
    unsigned int batchSize_;
    int nbInputChannels_ = 0, nbPolicyValues_ = 0, nbAux_ = 0, isPolicyMap_ = 1, version_ = 0;
};

enum TerminalType { TERMINAL_LOSS = 0, TERMINAL_DRAW = 1, TERMINAL_WIN = 2, TERMINAL_CUSTOM = 3, TERMINAL_NONE = 4 };

class BoardState {
   public:
    BoardState() = default;
    ~BoardState() { ara_state_destroy(st_); }
    BoardState(const BoardState& o) : st_(ara_state_clone(o.st_)), variant_(o.variant_), is960_(o.is960_) {}
    BoardState& operator=(const BoardState& o) {
        if (this != &o) {
            ara_state_destroy(st_);
            st_ = ara_state_clone(o.st_);
            variant_ = o.variant_;
            is960_ = o.is960_;
        }
        return *this;
    }
    void set(const std::string& fenStr, bool isChess960, int variant) {
        ara_state_destroy(st_);
        st_ = ara_state_create(fenStr.empty() ? nullptr : fenStr.c_str(), variant, isChess960 ? 1 : 0);
        if (st_ == nullptr) throw std::invalid_argument(ara_last_error());
        variant_ = variant;
        is960_ = isChess960;
    }
    void init(int variant, bool isChess960) { set("", isChess960, variant); }
    BoardState* clone() const { return new BoardState(*this); }
    std::vector<Action> legal_actions() const {
        Action buf[512];
        const int n = ara_state_legal_moves(st_, buf);
        return std::vector<Action>(buf, buf + (n > 0 ? n : 0));
    }
    void do_action(Action a) {
        if (ara_state_do_move(st_, a) != 0) throw std::runtime_error(ara_last_error());
    }
    Action uci_to_action(const std::string& uci) const {
        for (Action a : legal_actions())
            if (action_to_uci(a) == uci) return a;
        return 0;
    }
    std::string action_to_uci(Action a) const {
        char b[8];
        ara_move_to_uci(a, is960_ ? 1 : 0, b);
        return b;
    }
    std::string fen() const {
        char b[256];
        ara_state_fen(st_, b, sizeof(b));
        return b;
    }
    int side_to_move() const { return ara_state_side_to_move(st_); }
    // full-move counter of the position (last FEN field), the TimeManager's moveNumber
    int move_number() const {
        const std::string f = fen();
        const size_t p = f.find_last_of(' ');
        return p == std::string::npos ? 1 : std::max(1, atoi(f.c_str() + p + 1));
    }
    bool is_chess960() const { return is960_; }
    TerminalType is_terminal() const { return static_cast<TerminalType>(ara_state_is_terminal(st_)); }
    // State::get_state_planes(normalize, inputPlanes, version): GPU plane-encode kernel through host buffers
    void get_state_planes(bool normalize, float* inputPlanes, int mode, int version) const {
        ara_board_t b;
        ara_state_board(st_, &b);
        if (ara_encode_planes(&b, 1, mode, version, normalize ? 1 : 0, inputPlanes) != 0) throw std::runtime_error(ara_last_error());
    }
    ara_state_t handle() const { return st_; }
    int variant() const { return variant_; }

   private:
    ara_state_t st_ = nullptr;
    int variant_ = 0;
    bool is960_ = false;
};

struct SearchSettings : ara_search_settings_t {
    explicit SearchSettings(int mode = 0) { ara_search_default_settings(this, mode); }
};

struct EvalInfo {  // engine/src/evalinfo.h
    std::vector<Action> legalMoves;
    std::vector<unsigned int> childNumberVisits;
    std::vector<float> qValues;
    std::vector<float> priors;
    std::vector<double> policyProbSmall;
    std::vector<Action> pv;
    Action bestMove = 0;
    float bestMoveQ = 0.0f;
    float rootValue = 0.0f;
    int centipawns = 0;
    size_t nodes = 0, nodesPreSearch = 0, depth = 0, selDepth = 0;
    double elapsedMs = 0.0;
    size_t calculate_nps() const {  // evalinfo.cpp:73-85
        const double ms = elapsedMs <= 0 ? 1.0 : elapsedMs;
        return static_cast<size_t>((nodes - nodesPreSearch) / (ms / 1000.0) + 0.5);
    }
};

inline int value_to_centipawn(float value, float param) {  // evalinfo.cpp:102-110
    if (std::fabs(value) >= 1) return (value > 0 ? 1 : -1) * 9999;
    const int sgn = (value > 0) - (value < 0);
    return static_cast<int>(-(sgn * std::log(1.0f - std::fabs(value)) / std::log(param)) * 100.0f);
}

// Node (engine/src/node.h:97-124): the getters the reference's UCI / agent code reads (node.h:345-460), over one
// ara_search_node snapshot.  Read-only: the tree lives on the device and is changed by the search kernels only.
class Node {
   public:
    Node(ara_search_t search, int tree, int nodeId) : search_(search), tree_(tree), view_(new ara_node_view_t) {
        if (ara_search_node(search, tree, nodeId, view_.get()) != 0) throw std::runtime_error(ara_last_error());
    }
    size_t get_number_child_nodes() const { return static_cast<size_t>(view_->n_moves); }
    unsigned get_no_visit_idx() const { return static_cast<unsigned>(view_->no_visit_idx); }
    unsigned get_visits() const { return view_->visit_sum; }
    unsigned get_real_visits() const { return view_->real_visits; }
    unsigned get_free_visits() const { return view_->free_visits; }
    unsigned get_node_count() const { return view_->visit_sum - view_->free_visits; }  // node.cpp:1303-1306
    float get_value() const { return view_->value; }
    double get_value_sum() const { return view_->value_sum; }
    unsigned long long hash_key() const { return view_->key; }
    int get_node_type() const { return view_->node_type; }  // 0 win, 1 draw, 2 loss, 3 unsolved
    bool is_terminal() const { return (view_->flags & 1) != 0; }
    bool has_nn_results() const { return (view_->flags & 2) != 0; }
    bool is_playout_node() const { return (view_->flags & 4) != 0; }
    bool is_root_node() const { return view_->parent < 0; }
    int get_checkmate_idx() const { return view_->checkmate_idx; }
    int get_end_in_ply() const { return view_->end_in_ply; }
    Action get_action(size_t childIdx) const { return view_->moves[childIdx]; }
    std::vector<Action> get_legal_actions() const { return std::vector<Action>(view_->moves, view_->moves + view_->n_moves); }
    std::vector<unsigned> get_child_number_visits() const { return std::vector<unsigned>(view_->visits, view_->visits + view_->no_visit_idx); }
    std::vector<float> get_q_values() const { return std::vector<float>(view_->q, view_->q + view_->no_visit_idx); }
    std::vector<float> get_policy_prob_small() const { return std::vector<float>(view_->prior, view_->prior + view_->n_moves); }
    float get_q_value(size_t childIdx) const { return view_->q[childIdx]; }
    unsigned get_virtual_loss_counter(size_t childIdx) const { return view_->vl[childIdx]; }
    // Node::get_child_node: a fresh view of the child, or nullptr while it has not been expanded
    std::unique_ptr<Node> get_child_node(size_t childIdx) const {
        if (childIdx >= get_number_child_nodes() || view_->child[childIdx] < 0) return nullptr;
        return std::unique_ptr<Node>(new Node(search_, tree_, view_->child[childIdx]));
    }
    int id() const { return view_->node_id; }
    const ara_node_view_t& view() const { return *view_; }

   private:
    ara_search_t search_;
    int tree_;
    std::unique_ptr<ara_node_view_t> view_;
};

// SearchThread (engine/src/searchthread.h): set_root_state + thread_iteration() drive the device search one mini-batch
// at a time (searchthread.cpp:403-416: create_mini_batch, predict, set_nn_results_to_child_nodes, the backups -- all on
// the device), get_root_node() reads the tree.  One tree per SearchThread.
class SearchThread {
   public:
    SearchThread(NeuralNetAPI* net, const ara_search_settings_t& settings, int deviceID = 0, int maxNodes = 0) : settings_(settings) {
        search_ = ara_search_create(net ? net->handle() : nullptr, &settings_, deviceID, 1, maxNodes);
        if (search_ == nullptr) throw std::invalid_argument(ara_last_error());
    }
    ~SearchThread() { ara_search_destroy(search_); }
    SearchThread(const SearchThread&) = delete;
    // set_root_state + set_root_node + the root's evaluation (MCTSAgent::evaluate_board_state up to the first iteration)
    void set_root_state(const BoardState& state) {
        ara_board_t root;
        const unsigned long long* keys = nullptr;
        const short* reps = nullptr;
        int n = 0;
        ara_state_board(state.handle(), &root);
        ara_state_history(state.handle(), &keys, &reps, &n);
        if (ara_search_set_position(search_, 0, &root, keys, reps, n) != 0 || ara_search_begin(search_) != 0)
            throw std::runtime_error(ara_last_error());
        running_ = true;
    }
    // one mini-batch; false once the loop condition of run_search_thread (searchthread.cpp:418-426) has failed
    bool thread_iteration() {
        const int rc = ara_search_step(search_, 1);
        if (rc < 0) throw std::runtime_error(ara_last_error());
        running_ = rc > 0;
        return running_;
    }
    bool is_running() const { return running_; }
    Node get_root_node() const { return Node(search_, 0, -1); }
    ara_search_t handle() const { return search_; }

   private:
    ara_search_settings_t settings_;
    ara_search_t search_ = nullptr;
    bool running_ = false;
};

class MCTSAgent {
   public:
    MCTSAgent(NeuralNetAPI* net, const SearchSettings& settings, int deviceID = 0, int maxNodes = 0) : settings_(settings) {
        search_ = ara_search_create(net ? net->handle() : nullptr, &settings_, deviceID, 1, maxNodes);
        if (search_ == nullptr) throw std::invalid_argument(ara_last_error());
    }
    ~MCTSAgent() { ara_search_destroy(search_); }
    MCTSAgent(const MCTSAgent&) = delete;
    // the tree's pools: nodes in use, capacity mapped, cap, device bytes (ara_search_pool)
    ara_search_pool_t pool() const {
        ara_search_pool_t p{};
        if (ara_search_pool(search_, 0, &p) != 0) throw std::runtime_error(ara_last_error());
        return p;
    }
    void evaluate_board_state(const BoardState& state, EvalInfo& evalInfo) {
        ara_board_t root;
        const unsigned long long* keys = nullptr;
        const short* reps = nullptr;
        int n = 0;
        ara_state_board(state.handle(), &root);
        ara_state_history(state.handle(), &keys, &reps, &n);
        if (ara_search_set_position(search_, 0, &root, keys, reps, n) != 0 || ara_search_go(search_) != 0)
            throw std::runtime_error(ara_last_error());
        if (ara_search_result(search_, 0, &result_) != 0) throw std::runtime_error(ara_last_error());
        const ara_search_result_t& r = result_;
        evalInfo.legalMoves.assign(r.moves, r.moves + r.n_moves);
        evalInfo.childNumberVisits.assign(r.visits, r.visits + r.n_moves);
        evalInfo.qValues.assign(r.q, r.q + r.n_moves);
        evalInfo.priors.assign(r.prior, r.prior + r.n_moves);
        evalInfo.policyProbSmall.assign(r.policy, r.policy + r.n_moves);
        evalInfo.pv.assign(r.pv, r.pv + r.pv_len);
        evalInfo.bestMove = r.best_idx >= 0 ? r.moves[r.best_idx] : 0;
        evalInfo.bestMoveQ = r.best_move_q;
        evalInfo.rootValue = r.root_value;
        evalInfo.centipawns = value_to_centipawn(r.best_move_q, settings_.mode == 1 ? 1.4f : 1.2f);
        evalInfo.nodes = r.visit_sum - r.free_visits;
        evalInfo.nodesPreSearch = r.nodes_pre_search;
        evalInfo.depth = static_cast<size_t>(r.pv_len);
        evalInfo.elapsedMs = ara_search_last_go_ms(search_);
        lastValueEval_ = evalInfo.bestMoveQ;                                       // mctsagent.cpp:331
        if (useNPSTimemanager && evalInfo.elapsedMs > 0) {                         // update_nps_measurement, :222-228
            ++nbNPSentries_;
            overallNPS_ += 1.0f / nbNPSentries_ * (static_cast<float>(evalInfo.calculate_nps()) - overallNPS_);
        }
    }
    // MCTSAgent::clear_game_history (mctsagent.cpp:249-258): the per-game measurements start over
    void clear_game_history() {
        lastValueEval_ = -1.0f;
        nbNPSentries_ = 0;
        overallNPS_ = 0.0f;
    }
    // run_mcts_search (mctsagent.cpp:350-352): the next searches run under the ThreadManager's heuristics with this
    // move time; inGame = is_game_sceneario(limits), canProlong = can_prolong_search(move number, thresh move)
    void set_time_control(double movetimeMs, bool inGame, bool canProlong, double safeRemainingMs, double moveOverheadMs) {
        ara_time_control_t tc{};
        tc.movetime_ms = movetimeMs;
        tc.update_interval_ms = 250;
        tc.overall_nps = overallNPS_;
        tc.safe_remaining_ms = safeRemainingMs;
        tc.move_overhead_ms = moveOverheadMs;
        tc.last_value_eval = lastValueEval_;
        tc.in_game = inGame ? 1 : 0;
        tc.can_prolong = canProlong ? 1 : 0;
        if (ara_search_set_time_control(search_, &tc) != 0) throw std::runtime_error(ara_last_error());
    }
    void clear_time_control() { ara_search_set_time_control(search_, nullptr); }
    ara_time_report_t time_report() const {
        ara_time_report_t r{};
        ara_search_time_report(search_, &r);
        return r;
    }
    bool useNPSTimemanager = true;  // UCI option Use_NPS_Time_Manager
    const ara_search_result_t& last_result() const { return result_; }
    // MCTSAgent::get_root_node: read-only view of the root of the last search
    Node get_root_node() const { return Node(search_, 0, -1); }
    // MCTSAgent::apply_move_to_tree: the subtree behind `move` is kept for the next search
    void apply_move_to_tree(Action move) {
        if (ara_search_apply_move(search_, 0, move) != 0) throw std::runtime_error(ara_last_error());
    }
    // MCTSAgent::stop (UCI `stop`): callable from another thread while evaluate_board_state runs
    void stop() { ara_search_stop(search_); }
    // SearchLimits::movetime: the following searches also stop after `ms` of wall time (0 = off)
    void set_movetime(double ms) {
        if (ara_search_set_movetime(search_, ms) != 0) throw std::runtime_error(ara_last_error());
    }
    // MCTSAgent::update_q_value_weight / update_dirichlet_epsilon: the following searches use this value instead of the
    // settings' (a negative value restores the settings' value)
    void update_q_value_weight(float value) {
        qValueWeight_ = value;
        set_tree_settings();
    }
    void update_dirichlet_epsilon(float value) {
        dirichletEpsilon_ = value;
        set_tree_settings();
    }

   private:
    void set_tree_settings() {
        if (ara_search_set_tree_settings(search_, -1, qValueWeight_, dirichletEpsilon_) != 0) throw std::invalid_argument(ara_last_error());
    }
    SearchSettings settings_;
    ara_search_t search_ = nullptr;
    ara_search_result_t result_{};
    float lastValueEval_ = -1.0f, overallNPS_ = 0.0f;
    float qValueWeight_ = -1.0f, dirichletEpsilon_ = -1.0f;
    size_t nbNPSentries_ = 0;
};

// RawNetAgent (agents/rawnetagent.cpp:45-83): the move the network's policy prefers, without a search.  mode / inputVersion
// are the input representation the searches of the same network use (SearchSettings::mode / input_version).
class RawNetAgent {
   public:
    RawNetAgent(NeuralNetAPI* net, int mode, int inputVersion) : net_(net), mode_(mode), inputVersion_(inputVersion) {
        if (net == nullptr) throw std::invalid_argument("RawNetAgent needs a network");
    }
    void evaluate_board_state(const BoardState& state, EvalInfo& evalInfo) {
        evalInfo = EvalInfo();
        evalInfo.legalMoves = state.legal_actions();
        if (evalInfo.legalMoves.empty()) throw std::runtime_error("no legal move in " + state.fen());
        const float param = mode_ == 1 ? 1.4f : 1.2f;
        if (evalInfo.legalMoves.size() == 1) {  // a single legal move is played without a forward (depth and nodes 0)
            evalInfo.policyProbSmall.assign(1, 1.0);
            evalInfo.bestMove = evalInfo.legalMoves[0];
            evalInfo.pv = {evalInfo.bestMove};
            evalInfo.centipawns = value_to_centipawn(0.0f, param);
            return;
        }
        // ara_legal_moves gives policy-map indices: the classic labels of a fully-connected policy head are not mapped yet
        if (!net_->is_policy_map())
            throw std::runtime_error("RawNetAgent: the network has a fully-connected policy head (classic labels); only "
                                     "policy-map networks are supported");
        ara_board_t board;
        ara_state_board(state.handle(), &board);
        Action moves[512];
        int policyIdx[512], count = 0;
        if (ara_legal_moves(&board, 1, moves, &count, nullptr, policyIdx) != 0) throw std::runtime_error(ara_last_error());
        std::vector<float> planes(net_->get_nb_input_values_total()), priors(count);
        state.get_state_planes(true, planes.data(), mode_, inputVersion_);
        float value = 0.0f;
        if (ara_net_predict_priors(net_->handle(), planes.data(), 1, policyIdx, &count, count, &value, priors.data(), nullptr) != 0)
            throw std::runtime_error(ara_last_error());
        evalInfo.legalMoves.assign(moves, moves + count);
        evalInfo.policyProbSmall.assign(priors.begin(), priors.end());
        evalInfo.priors = priors;
        size_t best = 0;  // argmax: the first of equal priors
        for (size_t i = 1; i < priors.size(); ++i)
            if (priors[i] > priors[best]) best = i;
        evalInfo.bestMove = moves[best];
        evalInfo.pv = {evalInfo.bestMove};
        evalInfo.rootValue = value;
        evalInfo.centipawns = value_to_centipawn(value, param);
        evalInfo.depth = evalInfo.selDepth = evalInfo.nodes = 1;
    }

   private:
    NeuralNetAPI* net_;
    int mode_, inputVersion_;
};

}  // namespace crazyara
