// Test infrastructure: a C entry point over the UNMODIFIED reference TournamentResult (engine/src/rl/tournamentresult.{h,cpp}).
// Built by `make -C oracle -f ref_tournament.mk` into oracle/_ref/libref_tournament.so; used only by tests/ to pin
// crazyara_b200/match.py::TournamentResult.
#include <cstring>
#include <sstream>
#include <string>

#include "rl/tournamentresult.h"

// operator<< of the result into `out` (cap bytes), its CSV line (write_tournament_result_to_csv appends it to csv_path
// when that is not NULL); returns score()
extern "C" float ref_tournament_result(const char* player_a, const char* player_b, unsigned long long wins,
                                       unsigned long long draws, unsigned long long losses, char* out, int cap,
                                       const char* csv_path) {
    TournamentResult r;
    r.playerA = player_a;
    r.playerB = player_b;
    r.numberWins = wins;
    r.numberDraws = draws;
    r.numberLosses = losses;
    std::ostringstream os;
    os << r;
    const std::string s = os.str();
    if (static_cast<int>(s.size()) + 1 <= cap) memcpy(out, s.c_str(), s.size() + 1);
    else if (cap > 0) out[0] = 0;
    if (csv_path != nullptr) write_tournament_result_to_csv(r, csv_path);
    return r.score();
}
