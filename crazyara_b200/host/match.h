// Arena matches for the UCI `arena` command (SelfPlay::go_arena / generate_arena_game, rl/selfplay.cpp:263-307,
// :387-420): crazyara_b200.match.Match restated over the C-ABI.  Games come in colour-swapped pairs from one start
// position; `slots` games run in lock-step, each player owning one search handle with one tree per slot, and in each
// step a handle searches only the trees of the games in which its player is to move (the others are idle).  The draws
// come from NumpyRandom in the order Match makes them, so for the same seed and settings both drivers play the same
// games and write the same arena_games_gpu_<device>.pgn.  No resignation, no node jitter, no quick searches and no
// raw-network openings, as in the reference's arena games; a game is adjudicated a draw after RLSettings::maxPlies.
#pragma once
#include <exception>
#include <iostream>
#include <memory>
#include <thread>

#include "selfplay.h"

namespace crazyara {

// MCTSAgent::get_name (agents/mctsagent.cpp:266-269): engine name - model name (the file name without its extension,
// as os.path.splitext splits it); `fake` without a model
inline std::string player_name(const std::string& modelPath) {
    if (modelPath.empty()) return "fake";
    std::string base = modelPath.substr(modelPath.find_last_of('/') == std::string::npos ? 0 : modelPath.find_last_of('/') + 1);
    const size_t dot = base.find_last_of('.');
    if (dot != std::string::npos && base.find_first_not_of('.') < dot) base.resize(dot);
    return "CrazyAra-B200-" + base;
}

class Match {
   public:
    enum { PRODUCER = 0, CONTENDER = 1 };
    // producer / contender: networks whose batch holds min(rl.games, nGames) x settings.batch_size rows, or the same
    // network twice (both handles then search one after the other); the games are appended to `pgnPath`, and with
    // `verbose` every finished game is also printed to stdout
    Match(NeuralNetAPI* producer, NeuralNetAPI* contender, const std::string& producerName, const std::string& contenderName,
          const SearchSettings& settings, const RLSettings& rl, long nGames, int variant, bool is960, int deviceID,
          const std::string& pgnPath, bool verbose)
        : rl_(rl), nGames_(nGames), variant_(variant), is960_(is960), rng_(rl.seed), pgnPath_(pgnPath), verbose_(verbose),
          sharedNet_(producer == contender) {
        if (nGames <= 0) throw std::invalid_argument("the arena needs at least one game");
        if (rl.games <= 0) throw std::invalid_argument("Selfplay_Games must be positive");
        nSlots_ = static_cast<int>(std::min<long>(rl.games, nGames));
        names_[PRODUCER] = producerName;
        names_[CONTENDER] = contenderName;
        result_.playerA = contenderName;
        result_.playerB = producerName;
        int maxNodes = 0;  // with tree reuse: room for the kept subtrees of several moves before a tree starts over
        if (rl.reuseTree) maxNodes = static_cast<int>(8 * (settings.simulations ? settings.simulations : settings.nodes) + 4 * settings.batch_size + 64);
        NeuralNetAPI* nets[2] = {producer, contender};
        for (int i = 0; i < 2; ++i) {
            // distinct root-noise generators for the two players
            settings_[i] = settings;
            settings_[i].seed = settings.seed + 1000003ULL * rl.seed + 7919ULL * i;
            search_[i].reset(ara_search_create(nets[i]->handle(), &settings_[i], deviceID, nSlots_, maxNodes));
            if (!search_[i]) throw std::invalid_argument(ara_last_error());
        }
        date_ = GamePGN::now();
        slots_.resize(nSlots_);
        for (int s = 0; s < nSlots_; ++s) start(s);
    }
    Match(const Match&) = delete;

    // plays until every game is finished
    const TournamentResult& run() {
        while (step()) {
        }
        return result_;
    }

   private:
    struct Game {
        bool running = false;
        int white = CONTENDER, plies = 0;
        BoardState state;
        std::unique_ptr<GamePGN> pgn;
    };

    void start(int s) {  // Match._start: the next game of the queue in slot s, or nothing (the slot is idle from now on)
        Game& g = slots_[s];
        if (nextGame_ >= nGames_) {
            g.running = false;
            return;
        }
        const long k = nextGame_++;
        if (k % 2 == 0) pairFen_ = start_fen(rng_, variant_, is960_, rl_.epdFilePath);
        g.running = true;
        g.white = k % 2 == 0 ? CONTENDER : PRODUCER;
        g.plies = 0;
        g.state.set(pairFen_, is960_, variant_);
        g.pgn.reset(new GamePGN(variant_, is960_, names_[g.white], names_[1 - g.white], date_));
        g.pgn->fen = g.state.fen();
        if (rl_.reuseTree)  // clear_game_history of both players: move code 0 is never legal, so nothing of the slot's last game is kept
            for (auto& h : search_) check(ara_search_apply_move(h.get(), s, 0));
    }

    int mover(const Game& g) const { return g.state.side_to_move() == 0 ? g.white : 1 - g.white; }

    void finish(int s, TerminalType term) {
        Game& g = slots_[s];
        const Result res = game_result(term, g.state.side_to_move());
        if (res == DRAWN) ++result_.draws;
        else if ((res == WHITE_WIN) == (g.white == CONTENDER)) ++result_.wins;
        else ++result_.losses;
        g.pgn->result = result_string(res);
        g.pgn->write(pgnPath_);
        if (verbose_) std::cout << "\n" << g.pgn->str() << std::endl;  // write_game_to_pgn(..., verbose)
        start(s);
    }

    // Match.step: one move in every running game; false once every game is finished (and nothing was searched)
    bool step() {
        std::vector<int> running;
        for (int s = 0; s < nSlots_; ++s)
            if (slots_[s].running) running.push_back(s);
        if (running.empty()) return false;
        std::vector<int> searching;
        for (int p = 0; p < 2; ++p) {
            int n = 0;
            for (int s = 0; s < nSlots_; ++s) {
                const bool on = slots_[s].running && mover(slots_[s]) == p;
                check(ara_search_set_active(search_[p].get(), s, on ? 1 : 0));
                if (!on) continue;
                ara_board_t b;
                const unsigned long long* keys = nullptr;
                const short* reps = nullptr;
                int hl = 0;
                ara_state_board(slots_[s].state.handle(), &b);
                ara_state_history(slots_[s].state.handle(), &keys, &reps, &hl);
                check(ara_search_set_position(search_[p].get(), s, &b, keys, reps, hl));
                ++n;
            }
            if (n) searching.push_back(p);
        }
        if (searching.size() == 1 || sharedNet_) {
            for (int p : searching) check(ara_search_go(search_[p].get()));
        } else {  // two networks: one player's tree kernels run while the other's forward does
            std::exception_ptr errors[2];
            std::thread other([&]() {
                try {
                    check(ara_search_go(search_[searching[1]].get()));
                } catch (...) {
                    errors[1] = std::current_exception();
                }
            });
            try {
                check(ara_search_go(search_[searching[0]].get()));
            } catch (...) {
                errors[0] = std::current_exception();
            }
            other.join();
            for (const auto& e : errors)
                if (e) std::rethrow_exception(e);
        }
        for (int s : running) {
            Game& g = slots_[s];
            const int p = mover(g);
            check(ara_search_result(search_[p].get(), s, &res_));
            if (res_.n_moves == 0) {
                finish(s, g.state.is_terminal());
                continue;
            }
            const std::vector<double> policy(res_.policy, res_.policy + res_.n_moves);
            const Action move = res_.moves[set_best_move(policy, res_.best_idx, g.plies, rng_, rl_)];
            if (rl_.reuseTree) {
                check(ara_search_apply_move(search_[p].get(), s, move));
                if (g.plies != 0) check(ara_search_apply_move(search_[1 - p].get(), s, move));  // State::steps_from_null() != 0
            }
            const TerminalType term = g.pgn->play_move(g.state, move);
            ++g.plies;
            if (term != TERMINAL_NONE || g.plies >= rl_.maxPlies) finish(s, term);
        }
        return true;
    }

    static void check(int rc) {
        if (rc != 0) throw std::runtime_error(ara_last_error());
    }

    RLSettings rl_;
    long nGames_;
    int variant_;
    bool is960_;
    NumpyRandom rng_;
    std::string pgnPath_;
    bool verbose_, sharedNet_;
    int nSlots_ = 0;
    std::string names_[2], date_, pairFen_;
    SearchSettings settings_[2];
    std::unique_ptr<ara_search_s, decltype(&ara_search_destroy)> search_[2] = {{nullptr, ara_search_destroy}, {nullptr, ara_search_destroy}};
    ara_search_result_t res_{};
    std::vector<Game> slots_;
    TournamentResult result_;
    long nextGame_ = 0;
};

}  // namespace crazyara
