// Test driver of TournamentResult in crazyara_b200/host/selfplay_io.h (built by tests/test_arena_uci_host_logic.py):
//   tournament_driver <csv>   reads "A<TAB>B<TAB>W<TAB>D<TAB>L" lines from stdin; per line prints the text, the score's
//                             float32 bits and the verdict, one per line, and appends the CSV line to <csv>
#include <cstring>
#include <iostream>

#include "selfplay_io.h"

using namespace crazyara;

int main(int argc, char** argv) {
    if (argc != 2) {
        std::cerr << "usage: tournament_driver <csv>\n";
        return 2;
    }
    for (std::string line; std::getline(std::cin, line);) {
        std::istringstream in(line);
        TournamentResult r;
        std::getline(in, r.playerA, '\t');
        std::getline(in, r.playerB, '\t');
        in >> r.wins >> r.draws >> r.losses;
        if (!in) return 1;
        const float score = r.score();
        uint32_t bits;
        std::memcpy(&bits, &score, sizeof(bits));
        std::cout << r.str() << "\n" << bits << "\n" << r.verdict() << "\n";
        r.write_csv(argv[1]);
    }
    return 0;
}
