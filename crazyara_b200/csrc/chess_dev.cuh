// Device-side chess rules for the GPU search: bitboard position (128 B, one cache line), legal move generation,
// do_move with incremental Zobrist key, terminal rules, policy-map indexing.
//
// Stands in for the reference's Stockfish-fork seam (engine/src/environments/chess_related/board.{h,cpp},
// boardstate.{h,cpp}: legal_actions, do_action, hash_key, is_terminal, number_repetitions) for the variants the
// configs name: chess / chess960, crazyhouse, King of the Hill, Three-check.
// Written independently of oracle/chess.c (mailbox) -- bitboards with Kogge-Stone fills, no lookup tables -- and
// compared against it move-set by move-set.  All functions are __host__ __device__ so that the same source is
// unit-tested on the CPU (tests/hostemu) before it runs inside the search kernels; the warp-cooperative pieces use
// the lane abstraction of warp_ctx.cuh (1 lane on the host).
#pragma once
#include <stdint.h>

#include "warp_ctx.cuh"

namespace ara {

enum : int { V_CHESS = 0, V_CRAZYHOUSE = 1, V_KOTH = 2, V_THREECHECK = 3 };
enum : int { PT_PAWN = 0, PT_KNIGHT = 1, PT_BISHOP = 2, PT_ROOK = 3, PT_QUEEN = 4, PT_KING = 5 };
// TerminalType of the reference (engine/src/state.h)
enum : int { TERM_LOSS = 0, TERM_DRAW = 1, TERM_WIN = 2, TERM_CUSTOM = 3, TERM_NONE = 4 };

// Move: bits 0-5 from, 6-11 to, 12-15 flag.  Castling is king-from -> rook-from (as the reference's engine encodes it).
typedef uint16_t Move;
enum : int { MF_NORMAL = 0, MF_PROMO_N = 1, MF_PROMO_B = 2, MF_PROMO_R = 3, MF_PROMO_Q = 4, MF_EP = 5, MF_CASTLE = 6, MF_DROP = 8 };
ARA_HD Move make_move(int from, int to, int flag) { return static_cast<Move>(from | (to << 6) | (flag << 12)); }
ARA_HD int mv_from(Move m) { return m & 63; }
ARA_HD int mv_to(Move m) { return (m >> 6) & 63; }
ARA_HD int mv_flag(Move m) { return m >> 12; }
ARA_HD bool mv_is_drop(Move m) { return (m >> 12) >= MF_DROP; }
ARA_HD int mv_drop_pt(Move m) { return (m >> 12) - MF_DROP; }
constexpr int kMaxMoves = 512;

struct alignas(16) Board {
    uint64_t by_type[6];
    uint64_t by_color[2];
    uint64_t promoted;
    uint64_t key;
    uint16_t last_moves[8];  // most recent first (Board::lastMoves, board.cpp:216-225)
    uint8_t hand[2][5];
    uint8_t castle_rook[4];  // W-OO, W-OOO, B-OO, B-OOO rook origin, 0xFF = no right
    uint8_t ep;              // 0xFF = none
    uint8_t stm;
    uint8_t rule50;
    uint8_t checks;  // checks given: white in bits 0-1, black in bits 2-3
    uint16_t game_ply;
    int16_t repetition;  // Stockfish StateInfo::repetition semantics
    uint16_t plies_from_null;
    uint8_t variant;
    uint8_t chess960;
    uint8_t n_last;
    uint8_t pad_;
};
static_assert(sizeof(Board) == 128, "Board must be one 128-byte line");

constexpr uint64_t kFileA = 0x0101010101010101ULL;
constexpr uint64_t kFileH = 0x8080808080808080ULL;
constexpr uint64_t kRank1 = 0xFFULL;
constexpr uint64_t kRank8 = 0xFF00000000000000ULL;
constexpr uint64_t kCenter = (1ULL << 27) | (1ULL << 28) | (1ULL << 35) | (1ULL << 36);

ARA_HD int popc64(uint64_t x) {
#ifdef __CUDA_ARCH__
    return __popcll(x);
#else
    return __builtin_popcountll(x);
#endif
}
ARA_HD int lsb64(uint64_t x) {
#ifdef __CUDA_ARCH__
    return __ffsll(static_cast<long long>(x)) - 1;
#else
    return __builtin_ctzll(x);
#endif
}
ARA_HD uint64_t bit(int s) { return 1ULL << s; }

// ------------------------------------------------------------------ Zobrist (same definition as oracle/chess.c)
ARA_HD uint64_t zobrist(int idx) {
    uint64_t z = static_cast<uint64_t>(idx) * 0x9E3779B97F4A7C15ULL + 0xD1B54A32D192ED03ULL;
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ULL;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBULL;
    return z ^ (z >> 31);
}
// piece code of the oracle: white 1..6, black 9..14
ARA_HD uint64_t z_piece(int color, int pt, int sq) { return zobrist(((color << 3) | (pt + 1)) * 64 + sq); }
ARA_HD uint64_t z_stm() { return zobrist(1024); }
ARA_HD uint64_t z_castle(int r) { return zobrist(1025 + r); }
ARA_HD uint64_t z_ep(int file) { return zobrist(1029 + file); }
ARA_HD uint64_t z_hand(int color, int pt, int cnt) { return cnt > 0 ? zobrist(1040 + (color * 8 + pt + 1) * 32 + (cnt & 31)) : 0; }
ARA_HD uint64_t z_checks(int color, int n) { return n > 0 ? zobrist(1600 + color * 4 + (n & 3)) : 0; }

ARA_HD int checks_given(const Board& b, int color) { return (b.checks >> (2 * color)) & 3; }

ARA_HD uint64_t compute_key(const Board& b) {
    uint64_t k = 0;
    for (int c = 0; c < 2; ++c)
        for (int pt = 0; pt < 6; ++pt) {
            uint64_t bb = b.by_type[pt] & b.by_color[c];
            while (bb) {
                const int s = lsb64(bb);
                bb &= bb - 1;
                k ^= z_piece(c, pt, s);
            }
        }
    if (b.stm) k ^= z_stm();
    for (int r = 0; r < 4; ++r)
        if (b.castle_rook[r] != 0xFF) k ^= z_castle(r);
    if (b.ep != 0xFF) k ^= z_ep(b.ep & 7);
    if (b.variant == V_CRAZYHOUSE)
        for (int c = 0; c < 2; ++c)
            for (int pt = 0; pt < 5; ++pt) k ^= z_hand(c, pt, b.hand[c][pt]);
    if (b.variant == V_THREECHECK)
        for (int c = 0; c < 2; ++c) k ^= z_checks(c, checks_given(b, c));
    return k;
}

// ------------------------------------------------------------------ attack sets (no tables)
ARA_HD uint64_t knight_attacks_bb(uint64_t n) {
    const uint64_t l1 = (n >> 1) & ~kFileH, l2 = (n >> 2) & ~(kFileH | (kFileH >> 1));
    const uint64_t r1 = (n << 1) & ~kFileA, r2 = (n << 2) & ~(kFileA | (kFileA << 1));
    const uint64_t h1 = l1 | r1, h2 = l2 | r2;
    return (h1 << 16) | (h1 >> 16) | (h2 << 8) | (h2 >> 8);
}
ARA_HD uint64_t king_attacks_bb(uint64_t k) {
    uint64_t a = ((k << 1) & ~kFileA) | ((k >> 1) & ~kFileH);
    k |= a;
    return a | (k << 8) | (k >> 8);
}
// squares attacked by pawns of `color`
ARA_HD uint64_t pawn_attacks_bb(uint64_t p, int color) {
    return color == 0 ? (((p << 9) & ~kFileA) | ((p << 7) & ~kFileH)) : (((p >> 7) & ~kFileA) | ((p >> 9) & ~kFileH));
}
ARA_HD uint64_t fill_n(uint64_t g, uint64_t p) { g |= p & (g << 8); p &= p << 8; g |= p & (g << 16); p &= p << 16; g |= p & (g << 32); return g; }
ARA_HD uint64_t fill_s(uint64_t g, uint64_t p) { g |= p & (g >> 8); p &= p >> 8; g |= p & (g >> 16); p &= p >> 16; g |= p & (g >> 32); return g; }
ARA_HD uint64_t fill_e(uint64_t g, uint64_t p) { p &= ~kFileA; g |= p & (g << 1); p &= p << 1; g |= p & (g << 2); p &= p << 2; g |= p & (g << 4); return g; }
ARA_HD uint64_t fill_w(uint64_t g, uint64_t p) { p &= ~kFileH; g |= p & (g >> 1); p &= p >> 1; g |= p & (g >> 2); p &= p >> 2; g |= p & (g >> 4); return g; }
ARA_HD uint64_t fill_ne(uint64_t g, uint64_t p) { p &= ~kFileA; g |= p & (g << 9); p &= p << 9; g |= p & (g << 18); p &= p << 18; g |= p & (g << 36); return g; }
ARA_HD uint64_t fill_nw(uint64_t g, uint64_t p) { p &= ~kFileH; g |= p & (g << 7); p &= p << 7; g |= p & (g << 14); p &= p << 14; g |= p & (g << 28); return g; }
ARA_HD uint64_t fill_se(uint64_t g, uint64_t p) { p &= ~kFileA; g |= p & (g >> 7); p &= p >> 7; g |= p & (g >> 14); p &= p >> 14; g |= p & (g >> 28); return g; }
ARA_HD uint64_t fill_sw(uint64_t g, uint64_t p) { p &= ~kFileH; g |= p & (g >> 9); p &= p >> 9; g |= p & (g >> 18); p &= p >> 18; g |= p & (g >> 36); return g; }
// attacks of rook-like / bishop-like sliders standing on the set `s`, with occupancy `occ`
ARA_HD uint64_t rook_attacks_bb(uint64_t s, uint64_t occ) {
    const uint64_t e = ~occ;
    return (fill_n(s, e) << 8) | (fill_s(s, e) >> 8) | ((fill_e(s, e) << 1) & ~kFileA) | ((fill_w(s, e) >> 1) & ~kFileH);
}
ARA_HD uint64_t bishop_attacks_bb(uint64_t s, uint64_t occ) {
    const uint64_t e = ~occ;
    return ((fill_ne(s, e) << 9) & ~kFileA) | ((fill_nw(s, e) << 7) & ~kFileH) | ((fill_se(s, e) >> 7) & ~kFileA) |
           ((fill_sw(s, e) >> 9) & ~kFileH);
}

ARA_HD uint64_t occupied(const Board& b) { return b.by_color[0] | b.by_color[1]; }
ARA_HD uint64_t pieces(const Board& b, int color, int pt) { return b.by_type[pt] & b.by_color[color]; }
ARA_HD int king_square(const Board& b, int color) {
    const uint64_t k = pieces(b, color, PT_KING);
    return k ? lsb64(k) : -1;
}

// pieces of colour `by` (restricted to the set `by_set`, i.e. after removing a captured piece) that attack `sq`
ARA_HD uint64_t attackers_of(const Board& b, int sq, uint64_t occ, int by, uint64_t by_set) {
    const uint64_t s = bit(sq);
    uint64_t a = pawn_attacks_bb(s, by ^ 1) & b.by_type[PT_PAWN];
    a |= knight_attacks_bb(s) & b.by_type[PT_KNIGHT];
    a |= king_attacks_bb(s) & b.by_type[PT_KING];
    a |= rook_attacks_bb(s, occ) & (b.by_type[PT_ROOK] | b.by_type[PT_QUEEN]);
    a |= bishop_attacks_bb(s, occ) & (b.by_type[PT_BISHOP] | b.by_type[PT_QUEEN]);
    return a & by_set;
}
ARA_HD uint64_t checkers_bb(const Board& b) {
    const int k = king_square(b, b.stm);
    return k < 0 ? 0 : attackers_of(b, k, occupied(b), b.stm ^ 1, b.by_color[b.stm ^ 1]);
}
ARA_HD bool in_check(const Board& b) { return checkers_bb(b) != 0; }

ARA_HD int piece_type_on(const Board& b, int sq) {
    const uint64_t s = bit(sq);
    for (int pt = 0; pt < 6; ++pt)
        if (b.by_type[pt] & s) return pt;
    return -1;
}

ARA_HD void castle_targets(int us, bool king_side, int* kto, int* rto) {
    const int r = us ? 56 : 0;
    *kto = r + (king_side ? 6 : 2);
    *rto = r + (king_side ? 5 : 3);
}
ARA_HD uint64_t between_incl(int a, int c) {  // squares from a to c on one rank, inclusive
    const int lo = a < c ? a : c, hi = a < c ? c : a;
    return (hi == 63 ? ~0ULL : (bit(hi + 1) - 1)) & ~(bit(lo) - 1);
}

// ------------------------------------------------------------------ legality of one pseudo-legal move
ARA_HD bool leaves_king_safe(const Board& b, Move m) {
    const int us = b.stm, them = us ^ 1;
    const int from = mv_from(m), to = mv_to(m), flag = mv_flag(m);
    uint64_t occ = occupied(b);
    uint64_t enemy = b.by_color[them];
    int ksq = king_square(b, us);
    if (ksq < 0) return true;
    if (flag >= MF_DROP) {
        occ |= bit(to);
    } else if (flag == MF_CASTLE) {
        int kto, rto;
        castle_targets(us, (to & 7) > (from & 7), &kto, &rto);
        occ &= ~(bit(from) | bit(to));
        occ |= bit(kto) | bit(rto);
        ksq = kto;
    } else {
        occ &= ~bit(from);
        if (flag == MF_EP) {
            const int cap = (from & 56) | (to & 7);
            occ &= ~bit(cap);
            enemy &= ~bit(cap);
        }
        enemy &= ~bit(to);
        occ |= bit(to);
        if (ksq == from) ksq = to;
    }
    return attackers_of(b, ksq, occ, them, enemy) == 0;
}

ARA_HD bool variant_end(const Board& b) {
    if (b.variant == V_KOTH) return (b.by_type[PT_KING] & kCenter) != 0;
    if (b.variant == V_THREECHECK) return checks_given(b, 0) >= 3 || checks_given(b, 1) >= 3;
    return false;
}

// ------------------------------------------------------------------ legal move generation (warp-cooperative)
// Work is split by SQUARE: virtual lane l owns squares l and l+32.  Phases (separated by warp syncs; on the host the
// 32 virtual lanes are simply looped, so the very same partitioning is unit-tested on the CPU):
//   A  per own piece: pseudo-legal target set + move count; per empty square: number of droppable piece types
//   B  exclusive prefix sums -> write offsets
//   C  emission of the pseudo-legal list
//   D  legality: only moves that CAN expose the king (king moves, en passant, castling, pieces on a line with the king,
//      everything when in check) go through the full "apply and look at the king" test; survivors are compacted in order.
struct MoveGenScratch {
    uint64_t tgt[64];
    uint16_t cnt[64];
    uint16_t dcnt[64];
    uint16_t off[64];
    uint16_t doff[64];
    int n_pseudo;
    int castle_mask;  // bit 0: O-O possible, bit 1: O-O-O possible
    int checked;
};

#if defined(__CUDA_ARCH__)
#define ARA_FOR_VLANES(l) for (int l = ARA_LANE, once_ = 1; once_; once_ = 0)
#else
#define ARA_FOR_VLANES(l) for (int l = 0; l < 32; ++l)
#endif

ARA_HD uint64_t piece_targets(const Board& b, int sq, int pt, int us, uint64_t own, uint64_t opp, uint64_t occ) {
    const uint64_t s = bit(sq);
    switch (pt) {
        case PT_PAWN: {
            const uint64_t empty = ~occ;
            uint64_t t;
            if (us == 0) {
                const uint64_t one = (s << 8) & empty;
                t = one | (((one & (0xFFULL << 16)) << 8) & empty);
            } else {
                const uint64_t one = (s >> 8) & empty;
                t = one | (((one & (0xFFULL << 40)) >> 8) & empty);
            }
            uint64_t caps = opp;
            if (b.ep != 0xFF) caps |= bit(b.ep);
            return t | (pawn_attacks_bb(s, us) & caps);
        }
        case PT_KNIGHT: return knight_attacks_bb(s) & ~own;
        case PT_BISHOP: return bishop_attacks_bb(s, occ) & ~own;
        case PT_ROOK: return rook_attacks_bb(s, occ) & ~own;
        case PT_QUEEN: return (rook_attacks_bb(s, occ) | bishop_attacks_bb(s, occ)) & ~own;
        default: return king_attacks_bb(s) & ~own;
    }
}

// castling rights that are currently executable (Position::castling_impeded + the "not through check" rule);
// the 960 "attacker hidden behind the castling rook" case is left to the final legality test
ARA_HD int castle_mask_of(const Board& b, int ksq, uint64_t occ, uint64_t opp) {
    const int us = b.stm, them = us ^ 1;
    int mask = 0;
    for (int side = 0; side < 2; ++side) {
        const int rs = b.castle_rook[us * 2 + side];
        if (rs == 0xFF) continue;
        int kto, rto;
        castle_targets(us, side == 0, &kto, &rto);
        const uint64_t path = (between_incl(ksq, kto) | between_incl(rs, rto)) & ~(bit(ksq) | bit(rs));
        if (path & occ) continue;
        uint64_t kpath = between_incl(ksq, kto) & ~bit(ksq);
        bool ok = true;
        while (kpath && ok) {
            const int s = lsb64(kpath);
            kpath &= kpath - 1;
            if (attackers_of(b, s, occ, them, opp)) ok = false;
        }
        if (ok) mask |= 1 << side;
    }
    return mask;
}

// Returns the number of legal moves written to `out` (uniform across lanes); mg.checked tells whether the side to move
// is in check.  `scratch` receives the pseudo-legal list.
ARA_HD int gen_legal(const Board& b, MoveGenScratch& mg, Move* scratch, Move* out) {
    const int us = b.stm, them = us ^ 1;
    const uint64_t own = b.by_color[us], opp = b.by_color[them], occ = own | opp;
    const int ksq = king_square(b, us);
    const bool checked = ksq >= 0 && attackers_of(b, ksq, occ, them, opp) != 0;
    if (ARA_LANE == 0) {
        mg.checked = checked ? 1 : 0;
        mg.castle_mask = 0;
    }
    ARA_WARP_SYNC();
    if (variant_end(b)) return 0;
    const bool house = b.variant == V_CRAZYHOUSE;
    int hand_types = 0, hand_nonpawn = 0;
    if (house)
        for (int pt = 0; pt < 5; ++pt)
            if (b.hand[us][pt]) {
                ++hand_types;
                if (pt != PT_PAWN) ++hand_nonpawn;
            }
    const uint64_t promo_from = us ? (0xFFULL << 8) : (0xFFULL << 48);
    // ---- phase A
    ARA_FOR_VLANES(l) {
        for (int sq = l; sq < 64; sq += 32) {
            uint64_t t = 0;
            int c = 0, d = 0;
            if (own & bit(sq)) {
                const int pt = piece_type_on(b, sq);
                t = piece_targets(b, sq, pt, us, own, opp, occ);
                c = popc64(t);
                if (pt == PT_PAWN && (bit(sq) & promo_from)) c *= 4;
                if (pt == PT_KING && !checked && (b.castle_rook[us * 2] != 0xFF || b.castle_rook[us * 2 + 1] != 0xFF)) {
                    const int cm = castle_mask_of(b, sq, occ, opp);
                    mg.castle_mask = cm;
                    c += (cm & 1) + ((cm >> 1) & 1);
                } else if (pt == PT_KING) {
                    mg.castle_mask = 0;
                }
            } else if (house && !(occ & bit(sq))) {
                d = ((sq >> 3) == 0 || (sq >> 3) == 7) ? hand_nonpawn : hand_types;
            }
            mg.tgt[sq] = t;
            mg.cnt[sq] = static_cast<uint16_t>(c);
            mg.dcnt[sq] = static_cast<uint16_t>(d);
        }
    }
    ARA_WARP_SYNC();
    // ---- phase B (lane 0: 128 additions)
    if (ARA_LANE == 0) {
        int acc = 0;
        for (int sq = 0; sq < 64; ++sq) {
            mg.off[sq] = static_cast<uint16_t>(acc);
            acc += mg.cnt[sq];
        }
        for (int sq = 0; sq < 64; ++sq) {
            mg.doff[sq] = static_cast<uint16_t>(acc);
            acc += mg.dcnt[sq];
        }
        mg.n_pseudo = acc;
    }
    ARA_WARP_SYNC();
    // ---- phase C
    ARA_FOR_VLANES(l) {
        for (int sq = l; sq < 64; sq += 32) {
            uint64_t t = mg.tgt[sq];
            if (t || mg.cnt[sq]) {
                int o = mg.off[sq];
                const int pt = piece_type_on(b, sq);
                const bool promo = pt == PT_PAWN && (bit(sq) & promo_from);
                for (; t; t &= t - 1) {
                    const int to = lsb64(t);
                    if (promo) {
                        for (int f = MF_PROMO_Q; f >= MF_PROMO_N; --f) scratch[o++] = make_move(sq, to, f);
                    } else {
                        const bool ep = pt == PT_PAWN && b.ep != 0xFF && to == b.ep && ((to ^ sq) & 7) != 0;
                        scratch[o++] = make_move(sq, to, ep ? MF_EP : MF_NORMAL);
                    }
                }
                if (pt == PT_KING) {
                    const int cm = mg.castle_mask;
                    if (cm & 1) scratch[o++] = make_move(sq, b.castle_rook[us * 2], MF_CASTLE);
                    if (cm & 2) scratch[o++] = make_move(sq, b.castle_rook[us * 2 + 1], MF_CASTLE);
                }
            }
            if (mg.dcnt[sq]) {
                int o = mg.doff[sq];
                const bool edge = (sq >> 3) == 0 || (sq >> 3) == 7;
                for (int pt = 0; pt < 5; ++pt)
                    if (b.hand[us][pt] && !(pt == PT_PAWN && edge)) scratch[o++] = make_move(sq, sq, MF_DROP + pt);
            }
        }
    }
    ARA_WARP_SYNC();
    // ---- phase D
    const int n = mg.n_pseudo;
    const uint64_t king_lines = ksq >= 0 ? (rook_attacks_bb(bit(ksq), 0) | bishop_attacks_bb(bit(ksq), 0)) : 0;
    int k = 0;
    for (int base = 0; base < n; base += ARA_WARP_N) {
        const int i = base + ARA_LANE;
        bool ok = false;
        if (i < n) {
            const Move m = scratch[i];
            const int flag = mv_flag(m), from = mv_from(m);
            const bool risky = checked || flag == MF_EP || flag == MF_CASTLE ||
                               (flag < MF_DROP && (from == ksq || (bit(from) & king_lines)));
            ok = !risky || leaves_king_safe(b, m);
        }
        const uint32_t mask = ARA_BALLOT(ok);
        if (ok) out[k + ARA_POPC_BELOW(mask)] = scratch[i];
        k += ARA_POPC(mask);
    }
    ARA_WARP_SYNC();
    return k;
}

// ------------------------------------------------------------------ do_move (Position::do_move + Board::do_move)
// `rep_hist`: callback-free repetition: the caller supplies the keys / repetition values of earlier positions through
// compute_repetition() after the key is known; do_move itself leaves b.repetition = 0.
ARA_HD void do_move(Board& b, Move m) {
    const int us = b.stm, them = us ^ 1;
    const int from = mv_from(m), to = mv_to(m), flag = mv_flag(m);
    // last-move list, most recent first
    for (int i = (b.n_last < 8 ? b.n_last : 7); i > 0; --i) b.last_moves[i] = b.last_moves[i - 1];
    b.last_moves[0] = m;
    if (b.n_last < 8) b.n_last++;

    uint64_t key = b.key;
    if (b.ep != 0xFF) key ^= z_ep(b.ep & 7);
    int rule50 = b.rule50 + 1;
    int new_ep = 0xFF;
    uint8_t old_castle[4] = {b.castle_rook[0], b.castle_rook[1], b.castle_rook[2], b.castle_rook[3]};

    if (flag >= MF_DROP) {
        const int pt = flag - MF_DROP;
        b.by_type[pt] |= bit(to);
        b.by_color[us] |= bit(to);
        key ^= z_piece(us, pt, to);
        key ^= z_hand(us, pt, b.hand[us][pt]);
        b.hand[us][pt]--;
        key ^= z_hand(us, pt, b.hand[us][pt]);
        if (pt == PT_PAWN) rule50 = 0;
    } else if (flag == MF_CASTLE) {
        int kto, rto;
        castle_targets(us, (to & 7) > (from & 7), &kto, &rto);
        b.by_type[PT_KING] ^= bit(from);
        b.by_type[PT_ROOK] ^= bit(to);
        b.by_color[us] &= ~(bit(from) | bit(to));
        b.by_type[PT_KING] |= bit(kto);
        b.by_type[PT_ROOK] |= bit(rto);
        b.by_color[us] |= bit(kto) | bit(rto);
        b.promoted &= ~(bit(from) | bit(to) | bit(kto) | bit(rto));
        key ^= z_piece(us, PT_KING, from) ^ z_piece(us, PT_KING, kto) ^ z_piece(us, PT_ROOK, to) ^ z_piece(us, PT_ROOK, rto);
        b.castle_rook[us * 2] = b.castle_rook[us * 2 + 1] = 0xFF;
    } else {
        const int pt = piece_type_on(b, from);
        const int capsq = flag == MF_EP ? ((from & 56) | (to & 7)) : to;
        if (b.by_color[them] & bit(capsq)) {
            const int cpt = piece_type_on(b, capsq);
            b.by_type[cpt] &= ~bit(capsq);
            b.by_color[them] &= ~bit(capsq);
            key ^= z_piece(them, cpt, capsq);
            if (b.variant == V_CRAZYHOUSE) {
                const int hpt = (b.promoted & bit(capsq)) ? PT_PAWN : cpt;
                key ^= z_hand(us, hpt, b.hand[us][hpt]);
                b.hand[us][hpt]++;
                key ^= z_hand(us, hpt, b.hand[us][hpt]);
            }
            b.promoted &= ~bit(capsq);
            rule50 = 0;
            for (int r = 0; r < 2; ++r)
                if (b.castle_rook[them * 2 + r] == capsq) b.castle_rook[them * 2 + r] = 0xFF;
        }
        const bool was_promoted = (b.promoted & bit(from)) != 0;
        b.by_type[pt] &= ~bit(from);
        b.by_color[us] &= ~bit(from);
        b.promoted &= ~bit(from);
        key ^= z_piece(us, pt, from);
        int npt = pt;
        if (pt == PT_PAWN) {
            rule50 = 0;
            if (flag >= MF_PROMO_N && flag <= MF_PROMO_Q) {
                npt = flag;  // MF_PROMO_N..Q == PT_KNIGHT..PT_QUEEN
            } else if ((to ^ from) == 16) {
                // en-passant square only if an enemy pawn attacks it
                const int eps = (from + to) >> 1;
                if (pawn_attacks_bb(bit(eps), us) & pieces(b, them, PT_PAWN)) new_ep = eps;
            }
        }
        b.by_type[npt] |= bit(to);
        b.by_color[us] |= bit(to);
        key ^= z_piece(us, npt, to);
        if (npt != pt) {
            if (b.variant == V_CRAZYHOUSE) b.promoted |= bit(to);
        } else if (was_promoted) {
            b.promoted |= bit(to);
        }
        if (pt == PT_KING) b.castle_rook[us * 2] = b.castle_rook[us * 2 + 1] = 0xFF;
        for (int r = 0; r < 2; ++r)
            if (b.castle_rook[us * 2 + r] == from) b.castle_rook[us * 2 + r] = 0xFF;
    }
    for (int r = 0; r < 4; ++r)
        if (old_castle[r] != 0xFF && b.castle_rook[r] == 0xFF) key ^= z_castle(r);
    b.ep = static_cast<uint8_t>(new_ep);
    if (new_ep != 0xFF) key ^= z_ep(new_ep & 7);
    b.stm = static_cast<uint8_t>(them);
    key ^= z_stm();
    b.rule50 = static_cast<uint8_t>(rule50 > 255 ? 255 : rule50);
    b.game_ply++;
    b.plies_from_null++;
    if (b.variant == V_THREECHECK) {
        b.key = key;
        if (in_check(b)) {
            const int g = checks_given(b, us);
            key ^= z_checks(us, g);
            b.checks = static_cast<uint8_t>(b.checks + (1 << (2 * us)));
            key ^= z_checks(us, g + 1);
        }
    }
    b.key = key;
    b.repetition = 0;
}

// Repetition info of a position reached `1` ply after hist[len-1]: hist arrays hold (key, repetition) of all earlier
// positions, most recent last (Position::do_move tail; crazyhouse looks back over the whole game).
ARA_HD int repetition_end(const Board& b) {
    return b.variant == V_CRAZYHOUSE ? b.plies_from_null : (b.rule50 < b.plies_from_null ? b.rule50 : b.plies_from_null);
}

// Sequential form of the repetition scan (host classes / tests).  keys/reps: earlier positions, oldest first, the
// last entry being the position one ply before `b`.  The search kernels use a lane-parallel version of the same
// rule over (pre-root history + tree path).
ARA_HD int repetition_from_history(const Board& b, const uint64_t* keys, const int16_t* reps, int len) {
    int end = repetition_end(b);
    if (end > len) end = len;
    for (int i = 4; i <= end; i += 2)
        if (keys[len - i] == b.key) return reps[len - i] ? -i : i;
    return 0;
}

ARA_HD bool insufficient_material(const Board& b) {  // board.cpp:170-213
    if (b.variant != V_CHESS) return false;
    const int all = popc64(occupied(b));
    if (all > 4) return false;
    const int bishops = popc64(b.by_type[PT_BISHOP]), knights = popc64(b.by_type[PT_KNIGHT]);
    return all == 2 || (all == 3 && bishops == 1) || (all == 3 && knights == 1) ||
           (all == 4 && (popc64(pieces(b, 0, PT_KNIGHT)) == 2 || popc64(pieces(b, 1, PT_KNIGHT)) == 2));
}

// BoardState::is_terminal (boardstate.cpp:143-226) for the supported variants
ARA_HD int terminal_type(const Board& b, int n_legal, bool checked) {
    if (b.variant == V_KOTH) {
        if (pieces(b, b.stm, PT_KING) & kCenter) return TERM_WIN;
        if (pieces(b, b.stm ^ 1, PT_KING) & kCenter) return TERM_LOSS;
    }
    if (b.variant == V_THREECHECK) {
        if (checks_given(b, b.stm) >= 3) return TERM_WIN;
        if (checks_given(b, b.stm ^ 1) >= 3) return TERM_LOSS;
    }
    if (n_legal == 0) return checked ? TERM_LOSS : TERM_DRAW;
    if (b.repetition < 0) return TERM_DRAW;
    if (b.variant != V_CRAZYHOUSE && b.rule50 > 99) return TERM_DRAW;
    if (insufficient_material(b)) return TERM_DRAW;
    return TERM_NONE;
}

// ------------------------------------------------------------------ policy-map index of a move
// = FLAT_PLANE_IDX[label(mirrored UCI string)] (policymaprepresentation.h; plane_policy_representation.py:167-213),
// computed arithmetically.  Black's moves are rank-mirrored (node.cpp:970-977); non-960 castling is the king's
// two-square move, 960 castling king-from -> rook-square (sfutil.cpp:199-285).
ARA_HD int policy_map_index(Move m, int stm, int chess960) {
    int from = mv_from(m), to = mv_to(m);
    const int flag = mv_flag(m);
    if (flag == MF_CASTLE && !chess960) to = (from & 56) | ((to & 7) > (from & 7) ? 6 : 2);
    if (stm) {
        from ^= 56;
        to ^= 56;
    }
    if (flag >= MF_DROP) return (76 + (flag - MF_DROP)) * 64 + to;
    const int dy = (to >> 3) - (from >> 3), dx = (to & 7) - (from & 7);
    if (flag >= MF_PROMO_N && flag <= MF_PROMO_Q) return (64 + (flag - 1) * 3 + (dx + 1)) * 64 + from;
    const int ax = dx < 0 ? -dx : dx, ay = dy < 0 ? -dy : dy;
    if ((ax == 1 && ay == 2) || (ax == 2 && ay == 1)) {
        int c;
        if (dy == 2) c = dx == 1 ? 0 : 7;
        else if (dy == 1) c = dx == 2 ? 1 : 6;
        else if (dy == -1) c = dx == 2 ? 2 : 5;
        else c = dx == 1 ? 3 : 4;
        return (56 + c) * 64 + from;
    }
    const int len = (ax > ay ? ax : ay) - 1;
    int dir;
    if (dx == 0) dir = dy > 0 ? 0 : 4;
    else if (dy == 0) dir = dx > 0 ? 2 : 6;
    else if (dx > 0) dir = dy > 0 ? 1 : 3;
    else dir = dy > 0 ? 7 : 5;
    return (dir * 7 + len) * 64 + from;
}

// ------------------------------------------------------------------ classic-label index of a move
// Index of the (rank-mirrored for black) UCI string in the classic label list of `mode` (0 crazyhouse 2272 labels,
// 1 chess 1968, 2 lichess 2316; generate_uci_labels / generate_dropping_moves, outputrepresentation.cpp:108-163), what
// a fully-connected policy head and the training data's y_policy are indexed by.  The list is computed arithmetically
// in its generation order:
//   1. per origin square, file-major (a1, a2, ..., h8): the rank destinations, the file destinations, both diagonals,
//      the eight knight jumps -- 1792 labels;
//   2. per origin file: the promotions to q, r, b, n (and k in mode 2), each as 2->1 and 7->8 straight, then to the
//      left file, then to the right file;
//   3. the drops P, N, B, R, Q per square, file-major, pawns not on the first and last rank (modes 0 and 2).
// Castling is spelt as the policy map spells it: e1g1 / e1c1 outside chess960, king to rook square in chess960.
ARA_HD int classic_moves_from(int f, int r) {  // labels of part 1 with origin file f, rank r
    const int d1 = (f < r ? 7 - r + f : 7 - f + r), d2 = (f + r < 7 ? f + r : 14 - f - r);
    int kn = 0;
    const int kdx[8] = {-2, -1, -2, 1, 2, -1, 2, 1}, kdy[8] = {-1, -2, 1, -2, -1, 2, 1, 2};
    for (int k = 0; k < 8; ++k) kn += (f + kdx[k] >= 0 && f + kdx[k] < 8 && r + kdy[k] >= 0 && r + kdy[k] < 8);
    return 14 + d1 + d2 + kn;
}
ARA_HD int classic_label_index(Move m, int stm, int chess960, int mode) {
    int from = mv_from(m), to = mv_to(m);
    const int flag = mv_flag(m);
    if (flag == MF_CASTLE && !chess960) to = (from & 56) | ((to & 7) > (from & 7) ? 6 : 2);
    if (stm) {
        from ^= 56;
        to ^= 56;
    }
    constexpr int kQueenKnight = 1792;
    const int n_promo = mode == 2 ? 5 : 4;
    const int tf = to & 7, tr = to >> 3;
    if (flag >= MF_DROP) {  // 5 labels per square, 4 on the first and last rank (no pawn)
        if (mode == 1) return -1;
        const int pt = flag - MF_DROP, sq = tf * 8 + tr;
        const int before = 5 * sq - 2 * tf - (tr > 0 ? 1 : 0);  // pawnless squares (rank 1 and 8) of earlier files and this one
        return kQueenKnight + n_promo * 44 + before + (tr == 0 || tr == 7 ? pt - 1 : pt);
    }
    const int ff = from & 7, fr = from >> 3;
    if (flag >= MF_PROMO_N && flag <= MF_PROMO_Q) {
        int start = kQueenKnight;
        for (int f = 0; f < ff; ++f) start += n_promo * (2 + 2 * (f > 0) + 2 * (f < 7));
        const int per = 2 + 2 * (ff > 0) + 2 * (ff < 7);
        const int side = tf == ff ? 1 : (tf == ff - 1 ? 3 : (ff > 0 ? 5 : 3));
        return start + (MF_PROMO_Q - flag) * per + side;
    }
    int idx = 0;
    for (int s = 0; s < ff * 8 + fr; ++s) idx += classic_moves_from(s >> 3, s & 7);
    const int dx = tf - ff, dy = tr - fr;
    if (dy == 0) return idx + (tf < ff ? tf : tf - 1);
    idx += 7;
    if (dx == 0) return idx + (tr < fr ? tr : tr - 1);
    idx += 7;
    const int lo1 = -(ff < fr ? ff : fr), n1 = (ff < fr ? 7 - fr + ff : 7 - ff + fr);
    if (dx == dy) return idx + dx - lo1 - (dx > 0 ? 1 : 0);
    idx += n1;
    const int lo2 = -(ff < 7 - fr ? ff : 7 - fr), n2 = (ff + fr < 7 ? ff + fr : 14 - ff - fr);
    if (dx == -dy) return idx + dx - lo2 - (dx > 0 ? 1 : 0);
    idx += n2;
    const int kdx[8] = {-2, -1, -2, 1, 2, -1, 2, 1}, kdy[8] = {-1, -2, 1, -2, -1, 2, 1, 2};
    for (int k = 0; k < 8; ++k) {
        const int x = ff + kdx[k], y = fr + kdy[k];
        if (x < 0 || x >= 8 || y < 0 || y >= 8) continue;
        if (x == tf && y == tr) return idx;
        ++idx;
    }
    return -1;
}

}  // namespace ara
