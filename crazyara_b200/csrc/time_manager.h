// Host-side stop / prolong decisions of the reference's ThreadManager (manager/threadmanager.cpp:114-178) as pure
// functions of the root statistics, so that they can be unit-tested without a clock.  The search loop (search.cu)
// evaluates them every update interval on statistics read back from the device tree.
#pragma once
#include <algorithm>

#include "../../include/ara_b200.h"

namespace ara {

// What ThreadManager::early_stopping / continue_search (manager/threadmanager.cpp:114-178) read off the root while the
// search runs; collect_time_stats (search_dev.cuh) fills it on the device.
struct RootTimeStats {
    unsigned node_count;      // Node::get_node_count(): visits - free visits of the root
    unsigned first_visits;    // first_and_second_max over the open children, each less its child's free visits
    unsigned second_visits;
    float q_first, q_second;  // Node::get_q_value of those two
    int max_q_is_max_visits;  // max_q_child() == max_visits_child()
    float value_eval;         // Node::updated_value_eval (node.cpp:784-810)
    int valid;                // the root has at least one open child
};

// TimeManager::get_time_for_move (manager/timemanager.cpp:51-98) for a search without node / depth limits, with the
// engine's constants (constants.h:94-98: expected game length 38, proportional system from move 35 with 14 moves to
// go, increment factor 0.7) and the random factor off.  The arithmetic is the reference's: integer division of the
// safe remaining time, the float increment term added to it, the sum truncated.
inline int tm_time_for_move(long movetime, int time_me, int inc_me, int movestogo, int move_overhead, int move_number) {
    const int safe = std::max(time_me - move_overhead * 30, 1);  // SearchLimits::get_safe_remaining_time
    auto constant_movetime = [&](int moves_to_go) { return static_cast<int>(safe / moves_to_go + 0.7f * inc_me); };
    int cur;
    if (movetime != 0)
        cur = static_cast<int>(movetime);
    else if (movestogo != 0)
        cur = constant_movetime(movestogo);
    else if (time_me != 0)
        cur = move_number < 35 ? constant_movetime(38 - move_number) : constant_movetime(14);
    else
        cur = 1000;
    cur -= move_overhead;
    if (cur <= 0) cur = move_overhead * 2;
    return time_me != 0 ? std::min(safe, cur) : cur;
}

// ThreadManager::early_stopping: 1 "max nodes" rule, 2 "second move cannot catch up" rule, 0 keep searching
inline int tm_early_stopping(const ara_time_control_t& tc, double remaining_ms, const RootTimeStats& r) {
    if (!tc.in_game || tc.overall_nps == 0.0 || !r.valid) return 0;
    if (r.node_count > tc.overall_nps * (tc.movetime_ms / 1000.0f) * 2 && r.max_q_is_max_visits) return 1;
    // (the reference divides the NPS by 1000 in float before multiplying by the remaining milliseconds)
    if (r.second_visits + static_cast<float>(remaining_ms) * (static_cast<float>(tc.overall_nps) / 1000) < r.first_visits * 2.0f &&
        r.q_first > r.q_second)
        return 2;
    return 0;
}

// ThreadManager::continue_search: prolong by another move time if the evaluation dropped since the last move.
// `checked` is checkedContinueSearch, `last_eval` tData->lastValueEval; both are updated like the reference does.
inline bool tm_continue_search(const ara_time_control_t& tc, double remaining_ms, const RootTimeStats& r, int* checked,
                               float* last_eval) {
    if (!tc.in_game || !tc.can_prolong || tc.overall_nps == 0.0 || *checked > 1) return false;
    if (tc.movetime_ms * 2 > tc.safe_remaining_ms) return false;  // make sure not to flag when continuing
    if (r.value_eval < *last_eval) {
        if (remaining_ms < tc.update_interval_ms + tc.move_overhead_ms) return false;
        *last_eval = r.value_eval;
        ++*checked;
        return true;
    }
    return false;
}

}  // namespace ara
