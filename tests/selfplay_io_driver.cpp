// Test driver of crazyara_b200/host/selfplay_io.h (built by tests/test_selfplay_io.py):
//   selfplay_io_driver write <records> <out_dir>   the records' games through TrainDataExporter and GamePGN
//   selfplay_io_driver rng <seed> <n>              n rounds of NumpyRandom draws, pairwise sums and exponentials, one line per value
#include <iomanip>
#include <iostream>

#include "selfplay_io.h"

using namespace crazyara;

static int write(const char* records, const std::string& out) {
    std::ifstream in(records);
    int mode, channels, labels, games;
    long chunks, chunkSize;
    in >> mode >> channels >> labels >> chunks >> chunkSize >> games;
    TrainDataExporter exporter(out + "/data.zarr", mode, channels, labels, chunks, chunkSize);
    for (int g = 0; g < games; ++g) {
        int variant, is960, result, samples, plies;
        in >> variant >> is960 >> result >> samples >> plies;
        std::string fen, date;
        std::getline(in >> std::ws, fen);
        std::getline(in, date);
        BoardState st;
        st.set(fen, is960 != 0, variant);
        GamePGN pgn(variant, is960 != 0, "CrazyAra-B200", "CrazyAra-B200", date);
        pgn.fen = st.fen();
        for (int i = 0; i < plies; ++i) {
            unsigned m;
            in >> m;
            pgn.play_move(st, static_cast<Action>(m));
        }
        TrainDataExporter::Game rec;
        for (int s = 0; s < samples; ++s) {
            int stm, n;
            float q;
            in >> stm >> q >> n;
            std::vector<float> planes(static_cast<size_t>(channels) * 64);
            for (float& x : planes) in >> x;
            std::vector<Action> moves(n);
            std::vector<double> policy(n);
            for (Action& m : moves) in >> m;
            for (double& p : policy) in >> p;
            exporter.save_sample(rec, planes.data(), moves.data(), policy.data(), n, q, stm, is960 != 0);
        }
        exporter.export_game_samples(rec, static_cast<Result>(result));
        pgn.result = result_string(static_cast<Result>(result));
        pgn.write(out + "/games.pgn");
    }
    write_game_idx(out + "/gameIdx.txt", games);
    return in ? 0 : 1;
}

static int rng(uint64_t seed, int n) {
    NumpyRandom r(seed);
    std::cout << std::setprecision(17);
    std::vector<double> p = {0.05, 0.2, 0.0, 0.3, 0.45};
    for (int i = 0; i < n; ++i) {
        std::cout << r.integers(4) << "\n" << r.random() << "\n" << r.integers(int64_t{1} << 31) << "\n" << r.integers(8) << "\n"
                  << r.choice(p) << "\n" << r.integers(37) << "\n";
        std::vector<double> v(1 + (i * 37) % 300);
        for (double& x : v) x = r.random();
        std::cout << pairwise_sum(v) << "\n";
        for (int k = 0; k < 1 + i % 40; ++k) std::cout << r.exponential(15.0) << "\n";
    }
    return 0;
}

int main(int argc, char** argv) {
    const std::string cmd = argc > 1 ? argv[1] : "";
    if (cmd == "write" && argc == 4) return write(argv[2], argv[3]);
    if (cmd == "rng" && argc == 4) return rng(std::stoull(argv[2]), std::stoi(argv[3]));
    std::cerr << "usage: selfplay_io_driver write <records> <out_dir> | rng <seed> <n>\n";
    return 2;
}
