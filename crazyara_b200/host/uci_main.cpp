// Minimal UCI front-end over the C++ host classes (engine/src/uci/crazyara.cpp:76-143 command loop, option names of
// uci/optionsuci.cpp:66-220).  Supported: uci, isready, setoption, ucinewgame, position [startpos|fen] [moves ...],
// go [nodes N | movetime T | wtime W btime B [winc I] [binc I] [movestogo M]] (or the Simulations / Nodes options),
// go infinite + stop, benchmark <movetime>, inference [warmup N] [iterations N], root, quit.  The move time follows TimeManager::get_time_for_move (manager/timemanager.cpp:51-100) without its
// random factor; the search then also stops after that much wall time (ara_search_set_movetime), and in clock games
// the ThreadManager's early stopping / prolongation rules run on top (ara_search_set_time_control).
#include <algorithm>
#include <atomic>
#include <cmath>
#include <chrono>
#include <thread>
#include <iomanip>
#include <iostream>
#include <map>
#include <memory>
#include <sstream>
#include <vector>

#include "ara_host.h"
#include "benchmark_positions.h"

using namespace crazyara;

namespace {

struct Options {
    std::map<std::string, std::string> kv = {{"UCI_Variant", "crazyhouse"}, {"Model_Path", ""},        {"Batch_Size", "16"},
                                             {"Simulations", "800"},        {"Nodes", "0"},            {"Centi_CPuct_Init", "250"},
                                             {"CPuct_Base", "19652"},       {"Centi_Node_Temperature", "170"},
                                             {"Centi_Dirichlet_Epsilon", "0"}, {"Centi_Dirichlet_Alpha", "20"},
                                             {"Centi_Q_Value_Weight", "100"},  {"Centi_Q_Veto_Delta", "40"},
                                             {"MCTS_Solver", "true"},       {"Virtual_Style", "virtual_mix"},
                                             {"Virtual_Mix_Threshold", "1000"}, {"First_Device_ID", "0"},
                                             {"UCI_Chess960", "false"},     {"Input_Version", "0"},    {"Dirichlet_Seed", "42"},
                                             {"Move_Overhead", "20"},       {"Timed_Search_Nodes", "1000000"},
                                             {"Reuse_Tree", "true"},           {"Use_NPS_Time_Manager", "true"},
                                             {"Precision", "float16"},
                                             // the reference's defaults (optionsuci.cpp:89-90, :182); Threads 1 and both epsilons 0
                                             // give the deterministic single-threaded search
                                             {"Threads", "2"},              {"Centi_Epsilon_Greedy", "5"},
                                             {"Centi_Epsilon_Checks", "1"}};
    int i(const std::string& k) const { return std::stoi(kv.at(k)); }
    bool b(const std::string& k) const { return kv.at(k) == "true"; }
};

int variant_id(const std::string& v) {
    if (v == "crazyhouse") return 1;
    if (v == "kingofthehill") return 2;
    if (v == "3check" || v == "threecheck") return 3;
    return 0;
}
int mode_of_variant(int variant) { return variant == 0 ? 1 : (variant == 1 ? 0 : 2); }

// TimeManager::get_time_for_move with the reference's constants (constants.h:94-98): expected game length 38,
// proportional system from move 35 with 14 moves to go, increment factor 0.7, safety buffer 30 x overhead
struct GoLimits {
    long movetime = 0, time[2] = {0, 0}, inc[2] = {0, 0}, movestogo = 0;
    bool infinite = false;  // `go infinite`: search until `stop` (or until the node pool is full)
    bool any() const { return movetime || time[0] || time[1] || infinite; }
};
long time_for_move(const GoLimits& g, int me, int move_number, long overhead) {
    return ara_time_for_move(g.movetime, static_cast<int>(g.time[me]), static_cast<int>(g.inc[me]), static_cast<int>(g.movestogo),
                             static_cast<int>(overhead), move_number);
}

}  // namespace

int main() {
    Options opt;
    std::unique_ptr<NeuralNetAPI> net;
    std::unique_ptr<MCTSAgent> agent;
    BoardState state;
    EvalInfo info;
    bool ready = false;
    bool timed = false;  // the current agent was built for time-limited searches
    // game of the last searched position (base + moves): a `position` that extends it walks the kept tree
    // (MCTSAgent::apply_move_to_tree, mctsagent.cpp:230) instead of discarding it
    std::string searchedBase, gameBase;
    std::vector<std::string> searchedMoves, gameMoves;
    bool searched = false;
    auto variant = [&]() { return variant_id(opt.kv["UCI_Variant"]); };
    auto new_game = [&]() { state.init(variant(), opt.b("UCI_Chess960")); };
    auto prepare = [&]() {  // CrazyAra::is_ready (crazyara.cpp:597): build net + agent from the options
        const int mode = mode_of_variant(variant());
        SearchSettings s(mode);
        s.batch_size = opt.i("Batch_Size");
        s.simulations = static_cast<unsigned>(opt.i("Simulations"));
        s.nodes = static_cast<unsigned>(opt.i("Nodes"));
        s.cpuct_init = opt.i("Centi_CPuct_Init") / 100.0f;
        s.cpuct_base = static_cast<float>(opt.i("CPuct_Base"));
        s.node_policy_temperature = opt.i("Centi_Node_Temperature") / 100.0f;
        s.dirichlet_epsilon = opt.i("Centi_Dirichlet_Epsilon") / 100.0f;
        s.dirichlet_alpha = opt.i("Centi_Dirichlet_Alpha") / 100.0f;
        s.q_value_weight = opt.i("Centi_Q_Value_Weight") / 100.0f;
        s.q_veto_delta = opt.i("Centi_Q_Veto_Delta") / 100.0f;
        s.mcts_solver = opt.b("MCTS_Solver") ? 1 : 0;
        const std::string vs = opt.kv["Virtual_Style"];
        s.virtual_style = vs == "virtual_loss" ? 0 : (vs == "virtual_visit" ? 1 : 3);
        s.virtual_mix_threshold = static_cast<unsigned>(opt.i("Virtual_Mix_Threshold"));
        s.seed = static_cast<unsigned long long>(opt.i("Dirichlet_Seed"));
        s.threads = opt.i("Threads") >= 2 && 2 * s.batch_size <= 255 ? 2 : 1;  // (two logical threads at most; see ara_b200.h)
        // round(100 / centi), 0 = off (uci/crazyara.cpp:748-749)
        s.epsilon_greedy_counter = opt.i("Centi_Epsilon_Greedy") > 0 ? static_cast<int>(std::lround(100.0 / opt.i("Centi_Epsilon_Greedy"))) : 0;
        s.epsilon_checks_counter = opt.i("Centi_Epsilon_Checks") > 0 ? static_cast<int>(std::lround(100.0 / opt.i("Centi_Epsilon_Checks"))) : 0;
        if (opt.i("Input_Version") > 0) s.input_version = opt.i("Input_Version");
        agent.reset();
        net.reset();
        if (!opt.kv["Model_Path"].empty())
            net.reset(new NeuralNetAPI("gpu", opt.i("First_Device_ID"), static_cast<unsigned>(s.batch_size), opt.kv["Model_Path"],
                                       opt.kv["Precision"]));
        // a time-limited search has no visit budget to size the node pool from
        // a kept subtree lives in the same pools as the next search: room for a few searches, then the library compacts
        // the subtree to the front of its second set of pools (ara_search_apply_move)
        const long budget = s.simulations ? s.simulations : s.nodes;
        const int pool = timed ? opt.i("Timed_Search_Nodes")
                               : (opt.b("Reuse_Tree") ? static_cast<int>(std::min(8 * budget + 4L * s.batch_size + 64, 1L << 24)) : 0);
        if (timed) s.simulations = 0, s.nodes = 0;
        searched = false;
        agent.reset(new MCTSAgent(net.get(), s, opt.i("First_Device_ID"), pool));
        ready = true;
    };
    new_game();
    // every `go` runs on a worker thread so that `stop` / `isready` are read while it searches (the reference's search
    // threads + CrazyAra::stop_search, crazyara.cpp).  `stop` and `quit` end the running search; any other command first
    // waits for a limited search (nodes / time) to finish by itself -- scripted sessions keep their results -- and ends
    // an infinite one.
    std::thread worker;
    std::atomic<bool> searching{false};
    bool infiniteSearch = false;
    auto print_result = [&]() {
        if (info.nodesPreSearch) std::cout << "info string reused " << info.nodesPreSearch << " nodes" << std::endl;
        std::cout << "info depth " << info.depth << " nodes " << info.nodes << " nps " << info.calculate_nps() << " score cp "
                  << info.centipawns << " time " << static_cast<long>(info.elapsedMs) << " pv";
        for (Action a : info.pv) std::cout << " " << state.action_to_uci(a);
        std::cout << "\nbestmove " << (info.bestMove ? state.action_to_uci(info.bestMove) : std::string("(none)")) << std::endl;
    };
    auto stop_and_join = [&](bool stop) {
        if (!worker.joinable()) return;
        while (stop && searching.load()) {  // a stop that arrives before the search loop has started would be reset by it
            agent->stop();
            std::this_thread::sleep_for(std::chrono::milliseconds(2));
        }
        worker.join();
    };
    std::string line;
    while (std::getline(std::cin, line)) {
        std::istringstream ss(line);
        std::string cmd;
        ss >> cmd;
        if (worker.joinable()) {  // a search is (or was) running
            if (cmd == "isready" && searching.load()) {
                std::cout << "readyok" << std::endl;
                continue;
            }
            stop_and_join(cmd == "stop" || cmd == "quit" || infiniteSearch);
            if (cmd == "stop") continue;
        } else if (cmd == "stop") {
            continue;
        }
        try {
            if (cmd == "uci") {
                std::cout << "id name CrazyAra-B200\nid author crazyara_b200 (hot path of QueensGambit/CrazyAra on sm_90a)\n";
                for (const auto& kv : opt.kv) std::cout << "option name " << kv.first << " type string default " << kv.second << "\n";
                std::cout << "uciok" << std::endl;
            } else if (cmd == "isready") {
                if (!ready) prepare();
                std::cout << "readyok" << std::endl;
            } else if (cmd == "setoption") {
                std::string tok, name, value;
                ss >> tok;  // "name"
                while (ss >> tok && tok != "value") name += (name.empty() ? "" : " ") + tok;
                while (ss >> tok) value += (value.empty() ? "" : " ") + tok;
                if (opt.kv.count(name) == 0) {
                    std::cout << "info string unknown option " << name << std::endl;
                } else {
                    opt.kv[name] = value;
                    ready = false;
                    if (name == "UCI_Variant" || name == "UCI_Chess960") new_game();
                }
            } else if (cmd == "ucinewgame") {
                new_game();
                searched = false;
                if (agent) agent->clear_game_history();
            } else if (cmd == "position") {
                std::string tok, fen;
                ss >> tok;
                if (tok == "startpos") {
                    new_game();
                    ss >> tok;  // optional "moves"
                } else if (tok == "fen") {
                    while (ss >> tok && tok != "moves") fen += (fen.empty() ? "" : " ") + tok;
                    state.set(fen, opt.b("UCI_Chess960"), variant());
                }
                gameBase = fen.empty() ? "startpos" : fen;
                gameMoves.clear();
                while (ss >> tok) gameMoves.push_back(tok);
                const bool extends = searched && ready && agent && opt.b("Reuse_Tree") && gameBase == searchedBase &&
                                     gameMoves.size() > searchedMoves.size() &&
                                     std::equal(searchedMoves.begin(), searchedMoves.end(), gameMoves.begin());
                for (size_t i = 0; i < gameMoves.size(); ++i) {
                    const Action a = state.uci_to_action(gameMoves[i]);
                    if (a == 0) {
                        std::cout << "info string illegal move " << gameMoves[i] << std::endl;
                        gameMoves.resize(i);
                        break;
                    }
                    if (extends && i >= searchedMoves.size()) agent->apply_move_to_tree(a);
                    state.do_action(a);
                }
            } else if (cmd == "go") {
                std::string tok;
                GoLimits lim;
                while (ss >> tok) {
                    if (tok == "nodes") {
                        ss >> tok;
                        if (opt.kv["Nodes"] != tok) ready = false;
                        opt.kv["Nodes"] = tok;
                    } else if (tok == "movetime") {
                        ss >> lim.movetime;
                    } else if (tok == "wtime") {
                        ss >> lim.time[0];
                    } else if (tok == "btime") {
                        ss >> lim.time[1];
                    } else if (tok == "winc") {
                        ss >> lim.inc[0];
                    } else if (tok == "binc") {
                        ss >> lim.inc[1];
                    } else if (tok == "movestogo") {
                        ss >> lim.movestogo;
                    } else if (tok == "infinite") {
                        lim.infinite = true;
                    }
                }
                if (lim.any() != timed) {
                    timed = lim.any();
                    ready = false;
                }
                if (!ready) prepare();
                const bool inGame = lim.time[0] != 0 || lim.time[1] != 0 || lim.movestogo != 0;  // is_game_sceneario
                agent->clear_time_control();
                const bool report = timed && inGame && !lim.infinite;
                if (lim.infinite) {
                    agent->set_movetime(0.0);
                } else if (timed) {
                    const int me = state.side_to_move();
                    const long overhead = opt.i("Move_Overhead");
                    const long ms = time_for_move(lim, me, state.move_number(), overhead);
                    agent->set_movetime(static_cast<double>(ms));
                    // the ThreadManager's early stopping / prolongation applies to clock games only
                    if (inGame)
                        agent->set_time_control(static_cast<double>(ms), true, state.move_number() < 35,
                                                static_cast<double>(std::max(lim.time[me] - overhead * 30, 1L)),
                                                static_cast<double>(overhead));
                    std::cout << "info string movetime " << ms << std::endl;
                } else {
                    agent->set_movetime(0.0);
                }
                agent->useNPSTimemanager = opt.b("Use_NPS_Time_Manager");
                searched = true;
                searchedBase = gameBase;
                searchedMoves = gameMoves;
                infiniteSearch = lim.infinite;
                searching.store(true);
                worker = std::thread([&, report]() {
                    try {
                        agent->evaluate_board_state(state, info);
                        if (report) {
                            const ara_time_report_t tr = agent->time_report();
                            if (tr.early_stopped)
                                std::cout << "info string Early stopping" << (tr.early_stopped == 1 ? " (max nodes)" : "")
                                          << ", saved time: " << static_cast<long>(tr.saved_ms) << std::endl;
                            if (tr.prolonged) std::cout << "info string Increase search time" << std::endl;
                        }
                        print_result();
                    } catch (const std::exception& e) {
                        std::cout << "info string error: " << e.what() << std::endl;
                    }
                    searching.store(false);
                });
            } else if (cmd == "benchmark") {  // CrazyAra::benchmark (crazyara.cpp:287-330): `benchmark <movetime ms>`
                long moveTime = 3000;
                ss >> moveTime;
                if (variant() != 1) {
                    std::cout << "info string the benchmark positions are crazyhouse positions (set UCI_Variant)" << std::endl;
                    continue;
                }
                if (!timed) {
                    timed = true;
                    ready = false;
                }
                if (!ready) prepare();
                agent->clear_time_control();
                agent->set_movetime(static_cast<double>(moveTime));
                searched = false;  // every position is searched on a tree of its own
                int passed = 0;
                long totalNPS = 0, totalDepth = 0;
                std::vector<long> nps;
                const size_t n = sizeof(kBenchmarkPositions) / sizeof(kBenchmarkPositions[0]);
                for (const TestPosition& tp : kBenchmarkPositions) {
                    BoardState bs;
                    bs.set(tp.fen, false, 1);
                    EvalInfo ei;
                    agent->evaluate_board_state(bs, ei);
                    const std::string uciMove = ei.bestMove ? bs.action_to_uci(ei.bestMove) : std::string("(none)");
                    if (uciMove != tp.blunderMove) {
                        std::cout << "passed      -- " << uciMove << " != " << tp.blunderMove << std::endl;
                        ++passed;
                    } else {
                        std::cout << "failed      -- " << uciMove << " == " << tp.blunderMove << std::endl;
                    }
                    std::cout << "alternative -- " << uciMove << (uciMove == tp.alternativeMove ? " == " : " != ") << tp.alternativeMove
                              << std::endl;
                    const long cur = static_cast<long>(ei.calculate_nps());
                    totalNPS += cur;
                    totalDepth += static_cast<long>(ei.depth);
                    nps.push_back(cur);
                }
                std::sort(nps.begin(), nps.end());
                std::cout << "\nSummary\n----------------------\nPassed:\t\t" << passed << "/" << n << "\nNPS (avg):\t" << totalNPS / static_cast<long>(n)
                          << "\nNPS (median):\t" << nps[nps.size() / 2] << "\nPV-Depth:\t" << totalDepth / static_cast<long>(n) << std::endl;
            } else if (cmd == "inference") {  // CrazyAra::inference (crazyara.cpp:156-181): `inference [warmup N] [iterations N]`
                size_t warmupIterations = 100, iterations = 3000;
                std::string tok;
                while (ss >> tok) {
                    if (tok == "warmup") ss >> warmupIterations;
                    if (tok == "iterations") ss >> iterations;
                }
                if (!ready) prepare();
                if (!net) {
                    std::cout << "info string inference needs a network (setoption name Model_Path)" << std::endl;
                    continue;
                }
                const unsigned B = net->get_batch_size();
                std::cout << "info string running " << warmupIterations << " warmup iteration...\ninfo string running " << iterations
                          << " iterations...\ninfo string batch-size: " << B << std::endl;
                // NeuralNetAPIUser::run_inference (neuralnetapiuser.cpp:104-110): predict() on the caller's host buffers
                std::vector<float> planes(static_cast<size_t>(B) * net->get_nb_input_values_total(), 0.0f), value(B),
                    prob(static_cast<size_t>(B) * net->get_nb_policy_values()),
                    aux(static_cast<size_t>(B) * std::max(1u, net->get_nb_auxiliary_outputs()));
                for (size_t i = 0; i < warmupIterations; ++i) net->predict(planes.data(), value.data(), prob.data(), aux.data());
                const auto t0 = std::chrono::steady_clock::now();
                for (size_t i = 0; i < iterations; ++i) net->predict(planes.data(), value.data(), prob.data(), aux.data());
                const double elapsedMS = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
                std::cout << "info string Inference results\ninfo string -----------------\ninfo string Elapsed time: " << elapsedMS / 1000.0
                          << " s\ninfo string Evaluations per second: " << (iterations / elapsedMS) * 1000.0 * B << " nps" << std::endl;
            } else if (cmd == "root") {  // Node::print_node_statistics (node.cpp:1248-1301): the parity dump format
                std::cout << "  #  | Move  |    Visits    |  Policy   |  Q-values  |  CP   \n";
                std::cout << std::fixed << std::setprecision(7);
                for (size_t i = 0; i < info.legalMoves.size(); ++i)
                    std::cout << " " << std::setw(3) << std::setfill('0') << i << std::setfill(' ') << " | " << std::setw(5)
                              << state.action_to_uci(info.legalMoves[i]) << " | " << std::setw(12) << info.childNumberVisits[i] << " | "
                              << std::setw(9) << info.priors[i] << " | " << std::setw(10) << info.qValues[i] << " | " << std::setw(5)
                              << value_to_centipawn(info.qValues[i], 1.2f) << "\n";
                std::cout << "value:\t" << info.rootValue << "\nVisits:\t" << info.nodes << std::endl;
            } else if (cmd == "quit") {
                break;
            }
        } catch (const std::exception& e) {
            std::cout << "info string error: " << e.what() << std::endl;
        }
    }
    stop_and_join(true);
    return 0;
}
