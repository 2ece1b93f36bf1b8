// Self-play output and randomness for the C++ host, byte for byte what the Python arena writes and draws:
//   NumpyRandom      numpy.random.default_rng(seed) (SeedSequence -> PCG64) for the calls crazyara_b200.selfplay.Arena makes
//   pairwise_sum     numpy's float64 sum (add.reduce's pairwise summation), which Arena normalises distributions with
//   TrainDataExporter  crazyara_b200.export.TrainDataExporter (rl/traindataexporter.cpp): the uncompressed zarr v2 store
//   GamePGN          crazyara_b200.pgn.GamePGN (rl/gamepgn.cpp): the PGN stream of the self-play games
//   write_game_idx   SelfPlay::export_number_generated_games (rl/selfplay.cpp:353-359): gameIdx_<device>.txt
//   TournamentResult crazyara_b200.match.TournamentResult (rl/tournamentresult.{h,cpp}): an arena's score, its text and
//                    CSV line, and the verdict
// Header-only; no CUDA in this file (the classic-label index is the __host__ __device__ one of chess_dev.cuh).
#pragma once
#include <sys/stat.h>

#include <algorithm>
#include <cerrno>
#include <cmath>
#include <ctime>
#include <cstdint>
#include <cstdio>
#include <fstream>
#include <iomanip>
#include <sstream>
#include <stdexcept>
#include <string>
#include <vector>

#include "ara_host.h"
#include "chess_dev.cuh"
#include "ziggurat_exp.h"

namespace crazyara {

// ---------------------------------------------------------------------------------------------------- NumpyRandom
// numpy.random.Generator(PCG64(SeedSequence(seed))) for integers(n) / integers(0, n), random(), choice(len(p), p=p) and
// exponential(scale): the same 64-bit stream and the same draws per call.  exponential() is NumPy's ziggurat
// (random_standard_exponential) on the tables of ziggurat_exp.h.
class NumpyRandom {
   public:
    explicit NumpyRandom(uint64_t seed) {
        // SeedSequence(seed): the entropy's 32-bit words mixed into a pool of 4, then generate_state(4, uint64)
        std::vector<uint32_t> entropy;
        do {
            entropy.push_back(static_cast<uint32_t>(seed));
            seed >>= 32;
        } while (seed);
        uint32_t pool[4], hashConst = 0x43b0d7e5;
        auto hashmix = [&hashConst](uint32_t v) {
            v ^= hashConst;
            hashConst *= 0x931e8875;
            v *= hashConst;
            return v ^ (v >> 16);
        };
        auto mix = [](uint32_t x, uint32_t y) {
            uint32_t r = 0xca01f9dd * x - 0x4973f715 * y;
            return r ^ (r >> 16);
        };
        for (int i = 0; i < 4; ++i) pool[i] = hashmix(i < static_cast<int>(entropy.size()) ? entropy[i] : 0);
        for (int s = 0; s < 4; ++s)
            for (int d = 0; d < 4; ++d)
                if (s != d) pool[d] = mix(pool[d], hashmix(pool[s]));
        for (size_t s = 4; s < entropy.size(); ++s)
            for (int d = 0; d < 4; ++d) pool[d] = mix(pool[d], hashmix(entropy[s]));
        uint32_t words[8], hb = 0x8b51f9dd;
        for (int i = 0; i < 8; ++i) {
            uint32_t v = pool[i % 4] ^ hb;
            hb *= 0x58f38ded;
            v *= hb;
            words[i] = v ^ (v >> 16);
        }
        uint64_t val[4];
        for (int i = 0; i < 4; ++i) val[i] = words[2 * i] | static_cast<uint64_t>(words[2 * i + 1]) << 32;
        // pcg64_set_seed: state = (val[0] << 64 | val[1]), increment from (val[2] << 64 | val[3])
        inc_ = (static_cast<u128>(val[2]) << 64 | val[3]) << 1 | 1;
        state_ = 0;
        step();
        state_ += static_cast<u128>(val[0]) << 64 | val[1];
        step();
    }
    uint64_t next64() {  // pcg_setseq_128_xsl_rr_64
        step();
        const uint64_t v = static_cast<uint64_t>(state_ >> 64) ^ static_cast<uint64_t>(state_);
        const unsigned rot = static_cast<unsigned>(state_ >> 122);
        return (v >> rot) | (v << ((64 - rot) & 63));
    }
    uint32_t next32() {  // the upper half of a 64-bit output is kept for the next call
        if (hasUint32_) {
            hasUint32_ = false;
            return uinteger_;
        }
        const uint64_t n = next64();
        hasUint32_ = true;
        uinteger_ = static_cast<uint32_t>(n >> 32);
        return static_cast<uint32_t>(n);
    }
    double random() { return (next64() >> 11) * (1.0 / 9007199254740992.0); }
    // integers(0, n): Lemire's bounded draw on 32-bit outputs for ranges below 2^32 (numpy's scalar int64 path)
    int64_t integers(int64_t n) {
        if (n <= 0 || n > (int64_t{1} << 32)) throw std::invalid_argument("integers: range out of support");
        const uint64_t rng = static_cast<uint64_t>(n) - 1;
        if (rng == 0) return 0;
        if (rng == 0xFFFFFFFFu) return next32();
        const uint32_t excl = static_cast<uint32_t>(rng + 1);
        uint64_t m = static_cast<uint64_t>(next32()) * excl;
        uint32_t left = static_cast<uint32_t>(m);
        if (left < excl) {
            const uint32_t threshold = static_cast<uint32_t>(0xFFFFFFFFu - rng) % excl;
            while (left < threshold) {
                m = static_cast<uint64_t>(next32()) * excl;
                left = static_cast<uint32_t>(m);
            }
        }
        return static_cast<int64_t>(m >> 32);
    }
    double exponential(double scale) { return scale * standard_exponential(); }
    double standard_exponential() {
        while (true) {
            uint64_t ri = next64() >> 3;
            const int idx = static_cast<int>(ri & 0xFF);
            ri >>= 8;
            const double x = static_cast<double>(ri) * zig::kExpW[idx];
            if (ri < zig::kExpK[idx]) return x;  // the common path: one 64-bit output
            if (idx == 0) return zig::kExpR - std::log1p(-random());
            if ((zig::kExpF[idx - 1] - zig::kExpF[idx]) * random() + zig::kExpF[idx] < std::exp(-x)) return x;
        }
    }
    // choice(len(p), p=p): cdf = cumsum(p) / cdf[-1], the first index whose cdf exceeds one random()
    size_t choice(const std::vector<double>& p) {
        std::vector<double> cdf(p.size());
        double acc = 0.0;
        for (size_t i = 0; i < p.size(); ++i) cdf[i] = acc += p[i];
        for (double& c : cdf) c /= cdf.back();
        const double u = random();
        size_t i = 0;
        while (i < cdf.size() && !(cdf[i] > u)) ++i;
        return i < cdf.size() ? i : cdf.size() - 1;
    }

   private:
    using u128 = unsigned __int128;
    void step() { state_ = state_ * ((static_cast<u128>(0x2360ED051FC65DA4ULL) << 64) | 0x4385DF649FCCF645ULL) + inc_; }
    u128 state_ = 0, inc_ = 0;
    bool hasUint32_ = false;
    uint32_t uinteger_ = 0;
};

// numpy's pairwise summation of contiguous float64 (blocks of 8 partial sums up to 128 values, halves above)
inline double pairwise_sum(const double* a, size_t n) {
    if (n < 8) {
        double r = 0.0;
        for (size_t i = 0; i < n; ++i) r += a[i];
        return r;
    }
    if (n <= 128) {
        double r[8];
        for (int k = 0; k < 8; ++k) r[k] = a[k];
        size_t i = 8;
        for (; i < n - n % 8; i += 8)
            for (int k = 0; k < 8; ++k) r[k] += a[i + k];
        double res = ((r[0] + r[1]) + (r[2] + r[3])) + ((r[4] + r[5]) + (r[6] + r[7]));
        for (; i < n; ++i) res += a[i];
        return res;
    }
    size_t n2 = n / 2;
    n2 -= n2 % 8;
    return pairwise_sum(a, n2) + pairwise_sum(a + n2, n - n2);
}
inline double pairwise_sum(const std::vector<double>& v) { return pairwise_sum(v.data(), v.size()); }

// ---------------------------------------------------------------------------------------------------- zarr store
enum Result { WHITE_WIN = 0, BLACK_WIN = 1, DRAWN = 2 };

inline void make_dir(const std::string& path) {
    if (mkdir(path.c_str(), 0777) != 0 && errno != EEXIST) throw std::runtime_error("cannot create " + path);
}

// one uncompressed zarr v2 array, chunked along the first axis only
class ZArray {
   public:
    ZArray() = default;
    ZArray(const std::string& root, const std::string& name, std::vector<long> shape, long chunk, const char* dtype, size_t itemsize)
        : dir_(root + "/" + name), shape_(shape), chunk_(chunk), itemsize_(itemsize) {
        make_dir(dir_);
        std::ostringstream m;  // json.dump's layout
        m << "{\"zarr_format\": 2, \"shape\": " << list(shape) << ", \"chunks\": ";
        shape[0] = chunk;
        m << list(shape) << ", \"dtype\": \"" << dtype
          << "\", \"compressor\": null, \"fill_value\": 0, \"order\": \"C\", \"filters\": null}";
        std::ofstream(dir_ + "/.zarray", std::ios::binary) << m.str();
        row_ = itemsize;
        for (size_t i = 1; i < shape_.size(); ++i) row_ *= static_cast<size_t>(shape_[i]);
    }
    // rows [start, start + n) along the first axis; each touched chunk file is written whole
    void write(long start, const void* data, long n) {
        const char* src = static_cast<const char*>(data);
        long pos = 0;
        while (pos < n) {
            const long r = start + pos, ci = r / chunk_, off = r % chunk_, k = std::min(chunk_ - off, n - pos);
            const std::string path = chunk_path(ci);
            std::vector<char> buf(static_cast<size_t>(chunk_) * row_, 0);
            std::ifstream in(path, std::ios::binary);
            if (in) in.read(buf.data(), static_cast<std::streamsize>(buf.size()));
            std::copy(src + pos * row_, src + (pos + k) * row_, buf.begin() + off * row_);
            std::ofstream(path, std::ios::binary).write(buf.data(), static_cast<std::streamsize>(buf.size()));
            pos += k;
        }
    }

   private:
    static std::string list(const std::vector<long>& v) {
        std::string s = "[";
        for (size_t i = 0; i < v.size(); ++i) s += (i ? ", " : "") + std::to_string(v[i]);
        return s + "]";
    }
    std::string chunk_path(long ci) const {
        std::string p = dir_ + "/" + std::to_string(ci);
        for (size_t i = 1; i < shape_.size(); ++i) p += ".0";
        return p;
    }
    std::string dir_;
    std::vector<long> shape_;
    long chunk_ = 1;
    size_t itemsize_ = 1, row_ = 1;
};

// TrainDataExporter: x int16 [N, C, 8, 8], y_value int16, y_policy float32 [N, labels] on the classic label indices,
// y_best_move_q float32, plys_to_end int16, phase_vector int16, start_indices int32; N = number_chunks * chunk_size
class TrainDataExporter {
   public:
    struct Game {
        std::vector<int16_t> x, value, phase;
        std::vector<float> policy, q;
        size_t size() const { return q.size(); }
    };
    // mode: 0 crazyhouse, 1 chess, 2 lichess (the label list); n_labels its length
    TrainDataExporter(const std::string& path, int mode, int channels, int n_labels, long numberChunks = 200, long chunkSize = 128)
        : mode_(mode), channels_(channels), nLabels_(n_labels), numberSamples_(numberChunks * chunkSize) {
        make_dir(path);
        std::ofstream(path + "/.zgroup", std::ios::binary) << "{\"zarr_format\": 2}";
        const long N = numberSamples_, cs = chunkSize;
        x_ = ZArray(path, "x", {N, channels, 8, 8}, cs, "<i2", 2);
        value_ = ZArray(path, "y_value", {N}, cs, "<i2", 2);
        policy_ = ZArray(path, "y_policy", {N, n_labels}, cs, "<f4", 4);
        q_ = ZArray(path, "y_best_move_q", {N}, cs, "<f4", 4);
        plys_ = ZArray(path, "plys_to_end", {N}, cs, "<i2", 2);
        phase_ = ZArray(path, "phase_vector", {N}, cs, "<i2", 2);
        start_ = ZArray(path, "start_indices", {N}, cs, "<i4", 4);
        const int32_t zero = 0;
        start_.write(0, &zero, 1);
    }
    bool is_file_full() const { return startIdx_ >= numberSamples_; }
    long samples() const { return startIdx_; }
    // planes: un-normalised [C, 8, 8]; moves / policy: the searched position's legal moves and their posterior;
    // side_to_move 0 white, 1 black (its moves are looked up mirrored)
    void save_sample(Game& g, const float* planes, const Action* moves, const double* policy, int n, float bestMoveQ,
                     int sideToMove, bool is960, int phase = 0) const {
        for (int i = 0; i < channels_ * 64; ++i) g.x.push_back(static_cast<int16_t>(planes[i]));
        const size_t row = g.policy.size();
        g.policy.resize(row + nLabels_, 0.0f);
        for (int i = 0; i < n; ++i) {
            const int li = ara::classic_label_index(moves[i], sideToMove, is960 ? 1 : 0, mode_);
            if (li < 0 || li >= nLabels_) throw std::runtime_error("move without a classic label");
            g.policy[row + li] = static_cast<float>(policy[i]);
        }
        g.q.push_back(bestMoveQ);
        g.value.push_back(static_cast<int16_t>(sideToMove == 0 ? 1 : -1));
        g.phase.push_back(static_cast<int16_t>(phase));
    }
    long export_game_samples(const Game& g, Result result) {
        long n = static_cast<long>(g.size());
        if (n == 0 || is_file_full()) return 0;
        n = std::min(n, numberSamples_ - startIdx_);
        std::vector<int16_t> value(g.value.begin(), g.value.begin() + n), plys(n);
        for (long i = 0; i < n; ++i) {
            if (result == BLACK_WIN) value[i] = static_cast<int16_t>(-value[i]);
            if (result == DRAWN) value[i] = 0;
            plys[i] = static_cast<int16_t>(static_cast<long>(g.size()) - i);
        }
        const long s = startIdx_;
        x_.write(s, g.x.data(), n);
        value_.write(s, value.data(), n);
        q_.write(s, g.q.data(), n);
        policy_.write(s, g.policy.data(), n);
        plys_.write(s, plys.data(), n);
        phase_.write(s, g.phase.data(), n);
        startIdx_ += n;
        ++gameIdx_;
        const int32_t si = static_cast<int32_t>(startIdx_);
        start_.write(gameIdx_, &si, 1);
        return n;
    }

   private:
    int mode_, channels_, nLabels_;
    long numberSamples_, startIdx_ = 0, gameIdx_ = 0;
    ZArray x_, value_, policy_, q_, plys_, phase_, start_;
};

// ---------------------------------------------------------------------------------------------------- PGN
inline std::string result_string(Result r) { return r == WHITE_WIN ? "1-0" : (r == BLACK_WIN ? "0-1" : "1/2-1/2"); }

class GamePGN {
   public:
    // variant: the C-ABI's variant id; date as strftime("%Y.%m.%d %X")
    GamePGN(int variant, bool is960, const std::string& white, const std::string& black, const std::string& date)
        : date(date), white(white), black(black) {
        static const char* names[] = {"chess", "crazyhouse", "kingofthehill", "3check"};
        const std::string v = names[variant];
        this->variant = (!is960 && v == "chess") ? "standard" : v + (is960 ? "960" : "");
    }
    static std::string now() {
        char buf[80];
        const time_t t = time(nullptr);
        struct tm tm;
        localtime_r(&t, &tm);
        strftime(buf, sizeof(buf), "%Y.%m.%d %X", &tm);
        return buf;
    }
    void new_game() {
        moves.clear();
        result = "?";
    }
    // play_move_and_update (selfplay.cpp:38-55): the move's SAN, the move made, '#' on a move that ends the game with a win
    TerminalType play_move(BoardState& state, Action a) {
        char buf[16];
        if (ara_state_move_to_san(state.handle(), a, 0, buf) != 0) throw std::runtime_error(ara_last_error());
        std::string san = buf;
        state.do_action(a);
        const TerminalType term = state.is_terminal();
        if (term == TERMINAL_LOSS || term == TERMINAL_WIN) {
            if (!san.empty() && san.back() == '+') san.pop_back();
            san += "#";
        }
        moves.push_back(san);
        return term;
    }
    std::string str() const {
        std::ostringstream o;
        o << "[Variant \"" << variant << "\"]\n[Event \"" << event << "\"]\n[Date \"" << date << "\"]\n[Site \"" << site
          << "\"]\n[Round \"" << round << "\"]\n[FEN \"" << fen << "\"]\n[White \"" << white << "\"]\n[Black \"" << black
          << "\"]\n[Result \"" << result << "\"]\n[PlyCount \"" << moves.size() << "\"]\n[TimeControl \"" << timeControl << "\"]\n\n";
        for (size_t ply = 0; ply < moves.size(); ++ply) {
            if (ply % 2 == 0) o << ply / 2 + 1 << ". ";
            o << moves[ply] << " ";
            if ((ply + 1) % 8 == 0) o << "\n";
        }
        o << result << "\n\n";
        return o.str();
    }
    // write_game_to_pgn (selfplay.cpp:315-324): the game appended, then an empty line
    void write(const std::string& path) const { std::ofstream(path, std::ios::app | std::ios::binary) << str() << "\n"; }

    std::string variant, event = "SelfPlay", date, site = "Darmstadt, GER", round = "?", white, black, timeControl = "?";
    std::string fen = "?", result = "?";
    std::vector<std::string> moves;
};

inline void write_game_idx(const std::string& path, long games) { std::ofstream(path, std::ios::binary | std::ios::trunc) << games; }

// ---------------------------------------------------------------------------------------------------- arena result
// The result of a match from the view of player A (the contender).
struct TournamentResult {
    std::string playerA, playerB;
    long wins = 0, draws = 0, losses = 0;

    long games() const { return wins + draws + losses; }
    float score() const {  // (W + 0.5 D) / games in float32, as score() computes it
        return (static_cast<float>(wins) + static_cast<float>(draws) * 0.5f) / static_cast<float>(games());
    }
    // what the arena prints after its summary: the contender replaces the producer if it scored above 0.5
    const char* verdict() const { return score() > 0.5f ? "replace" : "keep"; }
    std::string str() const {  // operator<<: "<A>-<B>: W - D - L [score]", the score at precision 2
        std::ostringstream o;
        o << playerA << "-" << playerB << ": " << wins << " - " << draws << " - " << losses << " [" << std::setprecision(2) << score() << "]";
        return o.str();
    }
    std::string csv_line() const {
        return playerA + "," + playerB + "," + std::to_string(wins) + "," + std::to_string(draws) + "," + std::to_string(losses) + "\n";
    }
    // write_tournament_result_to_csv: appends "A,B,W,D,L"
    void write_csv(const std::string& path) const { std::ofstream(path, std::ios::app | std::ios::binary) << csv_line(); }
};

}  // namespace crazyara
