// SelfPlay (rl/selfplay.cpp:192-261, :367-385) for the UCI `selfplay` command: crazyara_b200.selfplay.Arena.step restated
// over the C-ABI.  `games` games run at once, each one tree of a single search handle, so their leaves share every
// network batch; after each search every game samples its move on the host.  The draws come from NumpyRandom in the
// order Arena makes them, so for the same seed and settings both drivers play the same games and write the same
// data_<device>.zarr and games_<device>.pgn.
#pragma once
#include <algorithm>
#include <chrono>
#include <fstream>
#include <iomanip>
#include <iostream>
#include <limits>
#include <memory>

#include "selfplay_io.h"

namespace crazyara {

struct RLSettings {                   // uci/optionsuci.cpp:198-218 and the play settings (:102-154)
    double nodeRandomFactor = 0.1;    // Centi_Node_Random_Factor / 100
    double quickDirichletEpsilon = 0; // Centi_Quick_Dirichlet_Epsilon / 100
    double quickProbability = 0;      // Centi_Quick_Probability / 100
    double quickQValueWeight = 0.7;   // Centi_Quick_Q_Value_Weight / 100
    int quickNodes = 100;             // Quick_Nodes
    double rawProbTemperature = 0.25; // Centi_Raw_Prob_Temperature / 100
    int maxInitPly = 30;              // MaxInitPly
    double meanInitPly = 15;          // MeanInitPly
    std::string epdFilePath;          // EPD_File_Path ("" or "<empty>": the variant's start position)
    double resignProbability = 0.9;   // Centi_Resign_Probability / 100
    double resignThreshold = -0.9;    // Centi_Resign_Threshold / 100
    double policyClipThresh = 0;      // Milli_Policy_Clip_Thresh / 1000
    long numberChunks = 640, chunkSize = 128;  // Selfplay_Number_Chunks, Selfplay_Chunk_Size
    double temperature = 0.8;         // Centi_Temperature / 100
    int temperatureMoves = 15;        // Temperature_Moves
    double temperatureDecay = 0.92;   // Centi_Temperature_Decay / 100
    double quantileClipping = 0;      // Centi_Quantile_Clipping / 100
    bool reuseTree = false;           // Reuse_Tree
    int games = 64;                   // Selfplay_Games: concurrent games of the handle (not in the reference)
    uint64_t seed = 0;                // Selfplay_Seed (not in the reference)
    int maxPlies = 512;
};

// apply_quantile_clipping / get_quantile (agents/agent.cpp:118-127, blazeutil.h:187-212), in float32 as Arena does
inline std::vector<double> quantile_clip(const std::vector<double>& p, double quantile) {
    std::vector<float> v(p.begin(), p.end());
    std::sort(v.begin(), v.end());
    if (v[0] >= quantile) return p;
    float acc = 0.0f;
    for (size_t i = 1; i < v.size(); ++i) {
        acc = acc + v[i];
        if (acc >= quantile) {
            const double thresh = static_cast<double>(v[i - 1]) + static_cast<double>(std::numeric_limits<float>::epsilon());
            std::vector<double> q(p.size());
            for (size_t k = 0; k < p.size(); ++k) q[k] = p[k] < thresh ? 0.0 : p[k];
            const double s = pairwise_sum(q);
            for (double& x : q) x /= s;
            return q;
        }
    }
    return p;
}

// sharpen_distribution (blazeutil.h:94-105): entries below thresh -> 0, renormalised; untouched if even the maximum is below
inline std::vector<double> sharpen_distribution(const std::vector<double>& p, double thresh) {
    if (thresh <= 0 || p.empty() || *std::max_element(p.begin(), p.end()) < thresh) return p;
    std::vector<double> q(p.size());
    for (size_t k = 0; k < p.size(); ++k) q[k] = p[k] < thresh ? 0.0 : p[k];
    const double s = pairwise_sum(q);
    for (double& x : q) x /= s;
    return q;
}

inline std::vector<double> normalised_power(const std::vector<double>& p, double exponent) {  // apply_temperature
    std::vector<double> q(p.size());
    for (size_t k = 0; k < p.size(); ++k) q[k] = std::pow(p[k], exponent);
    const double s = pairwise_sum(q);
    for (double& x : q) x /= s;
    return q;
}

// load_random_fen (selfplay.cpp:58-79): a uniformly drawn line of the EPD file without its trailing ';'; "" (the
// variant's start position) without a file ("" or "<empty>")
inline std::string load_random_fen(const std::string& path, NumpyRandom& rng) {
    if (path.empty() || path == "<empty>") return "";
    std::ifstream in(path);
    if (!in) throw std::runtime_error(path + ": cannot open");
    std::vector<std::string> lines;
    for (std::string l; std::getline(in, l);) lines.push_back(l);
    if (lines.empty()) throw std::runtime_error(path + ": no positions");
    std::string line = lines[rng.integers(static_cast<int64_t>(lines.size()))];
    if (!line.empty() && line.back() == ';') line.pop_back();
    return line;
}

inline std::string chess960_fen(NumpyRandom& rng) {  // chess960fen (chess960position.h:36-80) on the driver's generator
    char p[8] = {0};
    p[2 * rng.integers(4)] = 'B';
    p[2 * rng.integers(4) + 1] = 'B';
    for (char c : std::string("QNN"))
        while (true) {
            const long loc = rng.integers(8);
            if (!p[loc]) {
                p[loc] = c;
                break;
            }
        }
    for (char c : std::string("RKR")) *std::find(p, p + 8, 0) = c;
    std::string first(p, 8), lower = first;
    for (char& c : lower) c = static_cast<char>(std::tolower(c));
    return lower + "/pppppppp/8/8/8/8/PPPPPPPP/" + first + " w KQkq - 0 1";
}

// the FEN of a new game: a random EPD line, else a random chess960 set-up (chess only), else "" (the start position)
inline std::string start_fen(NumpyRandom& rng, int variant, bool is960, const std::string& epdFilePath) {
    std::string fen = load_random_fen(epdFilePath, rng);
    if (fen.empty() && is960 && variant == 0) fen = chess960_fen(rng);
    return fen;
}

// Agent::set_best_move (agents/agent.cpp:38-53) with get_current_temperature (playsettings.cpp:31-34): the index of the
// move to play at game ply `ply`, sampled from the search's policy while the temperature lasts, else the best move
inline size_t set_best_move(const std::vector<double>& pol, int bestIdx, int ply, NumpyRandom& rng, const RLSettings& rl) {
    if (ply < rl.temperatureMoves && rl.temperature > 0.01 && pairwise_sum(pol) > 0) {
        const double temp = rl.temperature * std::pow(rl.temperatureDecay, ply);
        std::vector<double> p = normalised_power(pol, 1.0 / temp);
        if (rl.quantileClipping != 0) p = quantile_clip(p, rl.quantileClipping);
        return rng.choice(p);
    }
    return static_cast<size_t>(bestIdx);
}

// WHITE_WIN / BLACK_WIN / DRAWN of a game that ended with `term`, `stmAtEnd` (0 white) to move: that side lost (mate,
// variant loss) or won (variant win); everything else is a draw
inline Result game_result(TerminalType term, int stmAtEnd) {
    return term == TERMINAL_LOSS ? (stmAtEnd == 0 ? BLACK_WIN : WHITE_WIN)
                                 : (term == TERMINAL_WIN ? (stmAtEnd == 0 ? WHITE_WIN : BLACK_WIN) : DRAWN);
}

class SelfPlay {
   public:
    // net: batch size >= rl.games * settings.batch_size; files go to the working directory, named after `device`
    SelfPlay(NeuralNetAPI* net, const SearchSettings& settings, const RLSettings& rl, int variant, bool is960, int deviceID)
        : net_(net), settings_(settings), rl_(rl), variant_(variant), is960_(is960), rng_(rl.seed), n_(rl.games) {
        if (rl.meanInitPly > 0 && rl.maxInitPly <= 0) throw std::invalid_argument("MaxInitPly must be positive when MeanInitPly is");
        if (rl.quickProbability >= 0.01 && rl.quickNodes <= 0) throw std::invalid_argument("Quick_Nodes must be positive when Centi_Quick_Probability is");
        if (n_ <= 0) throw std::invalid_argument("Selfplay_Games must be positive");
        // the trees' Dirichlet generators: one seed per arena seed, as Arena derives it for its (single) group of games
        settings_.seed = settings.seed + 1000003ULL * rl.seed;
        int maxNodes = 0;
        const double budget = settings.simulations ? settings.simulations : 2.0 * settings.nodes;
        if (rl.reuseTree) maxNodes = static_cast<int>(8 * (settings.simulations ? settings.simulations : settings.nodes) + 4 * settings.batch_size + 64);
        else if (rl.nodeRandomFactor > 0) maxNodes = static_cast<int>(budget * (1 + rl.nodeRandomFactor)) + 8 * settings.batch_size + 64;
        search_.reset(ara_search_create(net->handle(), &settings_, deviceID, n_, maxNodes));
        if (!search_) throw std::invalid_argument(ara_last_error());
        channels_ = static_cast<int>(net->get_nb_input_values_total() / 64);
        const std::string dev = "gpu_" + std::to_string(deviceID);
        static const int kLabels[3] = {2272, 1968, 2316};
        exporter_.reset(new TrainDataExporter("data_" + dev + ".zarr", settings.mode, channels_, kLabels[settings.mode], rl.numberChunks,
                                              rl.chunkSize));
        pgnPath_ = "games_" + dev + ".pgn";
        gameIdxPath_ = "gameIdx_" + dev + ".txt";
        std::ofstream(pgnPath_, std::ios::trunc);
        std::ofstream(gameIdxPath_, std::ios::trunc);
        const std::string date = GamePGN::now();
        states_.resize(n_);
        initPlies_.assign(n_, 0);
        plies_.assign(n_, 0);
        quick_.assign(n_, false);
        records_.resize(n_);
        for (int t = 0; t < n_; ++t) new_state(t);
        for (int t = 0; t < n_; ++t) allowResign_.push_back(draw_resign());
        for (int t = 0; t < n_; ++t) {
            pgns_.emplace_back(variant_, is960_, "CrazyAra-B200", "CrazyAra-B200", date);
            pgns_[t].fen = states_[t].fen();
        }
        gameStart_.assign(n_, std::chrono::steady_clock::now());
        play_openings();
    }
    SelfPlay(const SelfPlay&) = delete;

    // SelfPlay::go: numberOfGames > 0 plays until that many games have ended (games that end in the same move are kept);
    // 0 until the data file holds Selfplay_Number_Chunks x Selfplay_Chunk_Size samples.  gameIdx_<device>.txt counts the
    // games behind the data: those that ended while the file still had room (SelfPlay::export_number_generated_games),
    // not the games of the last move that ended after it was filled (they are in the PGN only).
    void go(long numberOfGames) {
        while (true) {
            step();
            if (numberOfGames > 0 && finished_ >= numberOfGames) break;
            if (exporter_->is_file_full()) break;
        }
        write_game_idx(gameIdxPath_, gameIdx_);
    }
    long finished() const { return finished_; }

   private:
    void new_state(int t) {  // generate_game (selfplay.cpp:196-202): the opening's ply count, then the start position
        initPlies_[t] = 0;
        if (rl_.meanInitPly > 0) {
            long ply = static_cast<long>(rng_.exponential(rl_.meanInitPly) + 0.5);
            if (ply > rl_.maxInitPly) ply = rng_.integers(int64_t{1} << 31) % rl_.maxInitPly;
            initPlies_[t] = static_cast<int>(ply);
        }
        states_[t].set(start_fen(rng_, variant_, is960_, rl_.epdFilePath), is960_, variant_);
    }
    bool draw_resign() { return rl_.resignProbability >= 0.01 && rng_.random() < rl_.resignProbability; }

    // init_starting_state_from_raw_policy (selfplay.cpp:423-452) for the games that just started: ply by ply, one
    // network forward (per network batch) over all of them
    void play_openings() {
        std::vector<int> todo;
        for (int t = 0; t < n_; ++t)
            if (initPlies_[t] > 0) todo.push_back(t);
        while (!todo.empty()) {
            const int n = static_cast<int>(todo.size());
            std::vector<ara_board_t> boards(n);
            for (int i = 0; i < n; ++i) ara_state_board(states_[todo[i]].handle(), &boards[i]);
            std::vector<unsigned short> moves(static_cast<size_t>(n) * 512);
            std::vector<int> counts(n), pidx(static_cast<size_t>(n) * 512);
            if (ara_legal_moves(boards.data(), n, moves.data(), counts.data(), nullptr, pidx.data()) != 0) throw std::runtime_error(ara_last_error());
            std::vector<float> planes(static_cast<size_t>(n) * channels_ * 64);
            if (ara_encode_planes(boards.data(), n, settings_.mode, settings_.input_version, 1, planes.data()) != 0)
                throw std::runtime_error(ara_last_error());
            const int B = static_cast<int>(net_->get_batch_size());
            std::vector<float> priors(static_cast<size_t>(n) * 512);
            for (int lo = 0; lo < n; lo += B) {  // RawNetAgent.predict: one forward per network batch
                const int hi = std::min(lo + B, n);
                int stride = 1;
                for (int i = lo; i < hi; ++i) stride = std::max(stride, counts[i]);
                std::vector<int> idx(static_cast<size_t>(hi - lo) * stride, 0);
                for (int i = lo; i < hi; ++i) std::copy(&pidx[i * 512], &pidx[i * 512] + counts[i], &idx[(i - lo) * stride]);
                std::vector<float> value(hi - lo), pri(static_cast<size_t>(hi - lo) * stride);
                if (ara_net_predict_priors(net_->handle(), &planes[static_cast<size_t>(lo) * channels_ * 64], hi - lo, idx.data(), &counts[lo],
                                           stride, value.data(), pri.data(), nullptr) != 0)
                    throw std::runtime_error(ara_last_error());
                for (int i = lo; i < hi; ++i) std::copy(&pri[(i - lo) * stride], &pri[(i - lo) * stride] + counts[i], &priors[i * 512]);
            }
            std::vector<int> next;
            for (int i = 0; i < n; ++i) {
                const int t = todo[i];
                if (counts[i] == 0) {
                    initPlies_[t] = 0;
                    continue;
                }
                std::vector<double> p(&priors[i * 512], &priors[i * 512] + counts[i]);
                if (rng_.random() < rl_.rawProbTemperature) {  // apply_raw_policy_temp (selfplay.cpp:474-487)
                    const double u = rng_.random();
                    p = normalised_power(p, 1.0 / (u < 0.05 ? 10.0 : (u < 0.25 ? 5.0 : 2.0)));
                }
                const double s = pairwise_sum(p);
                for (double& x : p) x /= s;
                const Action move = moves[i * 512 + rng_.choice(p)];
                BoardState after(states_[t]);
                after.do_action(move);
                if (after.is_terminal() != TERMINAL_NONE) {
                    initPlies_[t] = 0;
                    continue;
                }
                pgns_[t].play_move(states_[t], move);
                ++plies_[t];
                if (--initPlies_[t] > 0) next.push_back(t);
            }
            todo.swap(next);
        }
    }

    // the draws before a search (selfplay.cpp:212-220): adjust_node_count's integer, is_quick_search, the node jitter
    std::pair<long, bool> search_budget() {
        long nodes = settings_.nodes;
        const bool quickOn = rl_.quickProbability >= 0.01;
        long span = rl_.nodeRandomFactor > 0 ? static_cast<long>(nodes * rl_.nodeRandomFactor) : 0;
        const long randInt = span || quickOn ? rng_.integers(int64_t{1} << 31) : 0;
        const bool quick = quickOn && rng_.random() < rl_.quickProbability;
        if (quick) {
            nodes = rl_.quickNodes;
            span = rl_.nodeRandomFactor > 0 ? static_cast<long>(nodes * rl_.nodeRandomFactor) : 0;
        }
        if (span) nodes += randInt % span - span / 2;
        return {span || quick ? nodes : -1, quick};
    }

    void game_over(int t, TerminalType term, int stmAtEnd) {
        const Result result = game_result(term, stmAtEnd);
        if (!exporter_->is_file_full()) ++gameIdx_;
        const long samples = exporter_->export_game_samples(records_[t], result);
        records_[t] = TrainDataExporter::Game();
        new_state(t);
        plies_[t] = 0;
        allowResign_[t] = draw_resign();
        pgns_[t].result = result_string(result);
        pgns_[t].write(pgnPath_);
        pgns_[t].new_game();
        pgns_[t].fen = states_[t].fen();
        // speed_statistic_report (selfplay.cpp:339-351): running means over the finished games
        const auto now = std::chrono::steady_clock::now();
        const float minutes = std::chrono::duration_cast<std::chrono::milliseconds>(now - gameStart_[t]).count() / 60000.f;
        gameStart_[t] = now;
        gamesPerMin_ = (finished_ * gamesPerMin_ + (1 / minutes)) / (finished_ + 1);
        samplesPerMin_ = (finished_ * samplesPerMin_ + (samples / minutes)) / (finished_ + 1);
        std::cout << "    games    |  games/min  | samples/min \n-------------+-------------+-------------\n"
                  << std::setprecision(5) << std::setw(13) << finished_ << '|' << std::setw(13) << gamesPerMin_ << '|'
                  << std::setw(13) << samplesPerMin_ << "\n" << std::endl;
        ++finished_;
    }

    void step() {  // Arena.step: one move in every running game
        for (int t = 0; t < n_; ++t) {
            ara_board_t b;
            const unsigned long long* keys = nullptr;
            const short* reps = nullptr;
            int hl = 0;
            ara_state_board(states_[t].handle(), &b);
            ara_state_history(states_[t].handle(), &keys, &reps, &hl);
            if (ara_search_set_position(search_.get(), t, &b, keys, reps, hl) != 0) throw std::runtime_error(ara_last_error());
            const auto budget = search_budget();
            if (budget.first >= 0 || quick_[t])  // (after a quick search the settings' budget comes back)
                check(ara_search_set_limits(search_.get(), t, settings_.simulations,
                                            budget.first >= 0 ? static_cast<unsigned>(budget.first) : settings_.nodes));
            if (budget.second)
                check(ara_search_set_tree_settings(search_.get(), t, static_cast<float>(rl_.quickQValueWeight), static_cast<float>(rl_.quickDirichletEpsilon)));
            else if (quick_[t])  // reset_search_params (selfplay.cpp:183-190)
                check(ara_search_set_tree_settings(search_.get(), t, -1.0f, -1.0f));
            quick_[t] = budget.second;
        }
        check(ara_search_go(search_.get()));
        std::vector<ara_board_t> boards(n_);
        for (int t = 0; t < n_; ++t) ara_state_board(states_[t].handle(), &boards[t]);
        std::vector<float> planes(static_cast<size_t>(n_) * channels_ * 64);  // un-normalised, one call for every game
        check(ara_encode_planes(boards.data(), n_, settings_.mode, settings_.input_version, 0, planes.data()));
        for (int t = 0; t < n_; ++t) {
            BoardState& st = states_[t];
            check(ara_search_result(search_.get(), t, &result_));
            const ara_search_result_t& r = result_;
            if (r.n_moves == 0) {
                game_over(t, st.is_terminal(), st.side_to_move());
                continue;
            }
            const std::vector<double> policy(r.policy, r.policy + r.n_moves);
            const size_t idx = set_best_move(policy, r.best_idx, plies_[t], rng_, rl_);
            if (!quick_[t]) {  // a quick search exports nothing (selfplay.cpp:228); the policy is sharpened after the pick
                const std::vector<double> sharp = sharpen_distribution(policy, rl_.policyClipThresh);
                exporter_->save_sample(records_[t], &planes[static_cast<size_t>(t) * channels_ * 64], r.moves, sharp.data(), r.n_moves,
                                       r.best_move_q, st.side_to_move(), is960_);
            }
            if (rl_.reuseTree) check(ara_search_apply_move(search_.get(), t, r.moves[idx]));
            pgns_[t].play_move(st, r.moves[idx]);
            ++plies_[t];
            TerminalType term = st.is_terminal();
            if (term == TERMINAL_NONE && allowResign_[t] && static_cast<double>(r.best_move_q) < rl_.resignThreshold)
                term = TERMINAL_WIN;  // check_for_resignation (selfplay.cpp:170-182): the side now to move has won
            if (term != TERMINAL_NONE || plies_[t] >= rl_.maxPlies) game_over(t, term, st.side_to_move());
        }
        play_openings();
    }

    static void check(int rc) {
        if (rc != 0) throw std::runtime_error(ara_last_error());
    }

    NeuralNetAPI* net_;
    SearchSettings settings_;
    RLSettings rl_;
    int variant_;
    bool is960_;
    NumpyRandom rng_;
    int n_, channels_ = 0;
    std::unique_ptr<ara_search_s, decltype(&ara_search_destroy)> search_{nullptr, ara_search_destroy};
    ara_search_result_t result_{};
    std::unique_ptr<TrainDataExporter> exporter_;
    std::string pgnPath_, gameIdxPath_;
    std::vector<BoardState> states_;
    std::vector<int> initPlies_, plies_;
    std::vector<bool> quick_, allowResign_;
    std::vector<TrainDataExporter::Game> records_;
    std::vector<GamePGN> pgns_;
    std::vector<std::chrono::steady_clock::time_point> gameStart_;
    long finished_ = 0, gameIdx_ = 0;
    float gamesPerMin_ = 0, samplesPerMin_ = 0;
};

}  // namespace crazyara
