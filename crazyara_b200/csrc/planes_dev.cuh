// Board -> network input planes on the device (and, for tests, on the host through the same source).
//
// Semantics: engine/src/environments/chess_related/inputrepresentation.cpp (board_to_planes :628-680 and the
// per-version bodies :426-624) with the constants of boardstate.h:207-245.  The reference's compile-time MODE_*
// is the run-time `mode`.
//
// Every plane of every layout is either a bitboard plane (value v on the squares of a 64-bit mask) or a constant
// plane, so the encoder walks the layout once and hands each channel to a sink as (mask in OUTPUT coordinates, v):
//   * NCHW fp32 sink (the reference's [C,8,8] float tensor, State::get_state_planes): lanes write 2 squares each,
//     coalesced 256 B per plane;
//   * NHWC fp16 sink (the wgmma stem convolution's A operand): lane l keeps the descriptors of channels l, l+32,
//     l+64 and then writes row after row, 64 contiguous bytes per warp store.
// The reference fills plane after plane with a bit-serial loop (set_bits_from_bitmap :33-46).
#pragma once
#include "chess_dev.cuh"
#if defined(__CUDACC__)
#include <cuda_fp16.h>
#endif

namespace ara {

enum : int { MODE_CRAZYHOUSE = 0, MODE_CHESS = 1, MODE_LICHESS = 2 };

ARA_HD int planes_channels(int mode, int version) {
    if (version <= 1) return mode == MODE_CRAZYHOUSE ? 34 : (mode == MODE_CHESS ? 39 : 63);
    if (mode == MODE_CRAZYHOUSE) return version == 2 ? 51 : 64;
    if (mode == MODE_CHESS) return version == 3 ? 52 : -1;
    return version == 3 ? 80 : 63;
}

// length of the policy-map vector: 64 squares x the mode's move planes
ARA_HD int policy_labels(int mode) { return (mode == MODE_CRAZYHOUSE ? 81 : (mode == MODE_CHESS ? 76 : 84)) * 64; }

ARA_HD uint64_t bswap64_portable(uint64_t x) {  // flip_vertical (sfutil.cpp:178)
    x = ((x & 0x00FF00FF00FF00FFULL) << 8) | ((x >> 8) & 0x00FF00FF00FF00FFULL);
    x = ((x & 0x0000FFFF0000FFFFULL) << 16) | ((x >> 16) & 0x0000FFFF0000FFFFULL);
    return (x << 32) | (x >> 32);
}

struct PlaneCtx {
    const Board* b;
    int mode, flip, me, you;
    bool normalize;
    uint64_t own, opp, checkers;
    int cnt[2][6];
    bool opp_bishops;
};

ARA_HD PlaneCtx make_plane_ctx(const Board& b, int mode, bool normalize) {
    PlaneCtx p;
    p.b = &b;
    p.mode = mode;
    p.flip = b.stm != 0;  // racing kings (never flipped) is not a supported variant
    p.me = b.stm;
    p.you = b.stm ^ 1;
    p.normalize = normalize;
    p.own = b.by_color[p.me];
    p.opp = b.by_color[p.you];
    p.checkers = checkers_bb(b);
    for (int pt = 0; pt < 6; ++pt) {
        p.cnt[0][pt] = popc64(b.by_type[pt] & p.own);
        p.cnt[1][pt] = popc64(b.by_type[pt] & p.opp);
    }
    const uint64_t wb = pieces(b, 0, PT_BISHOP), bb = pieces(b, 1, PT_BISHOP);
    p.opp_bishops = false;
    if (popc64(wb) == 1 && popc64(bb) == 1) {
        const int ws = lsb64(wb), bs = lsb64(bb);
        p.opp_bishops = (((ws >> 3) + (ws & 7)) & 1) != (((bs >> 3) + (bs & 7)) & 1);
    }
    return p;
}

// Calls sink(mask, value) once per channel, in channel order.  mask is already in output coordinates.
template <class Sink>
ARA_HD void for_each_plane(const PlaneCtx& p, int version, Sink& sink) {
    const Board& b = *p.b;
    const float max_prisoners = p.mode == MODE_CRAZYHOUSE ? 32.0f : 16.0f;
    const float max_no_progress = p.mode == MODE_CRAZYHOUSE ? 40.0f : 50.0f;
    auto bb_plane = [&](uint64_t bb) { sink(p.flip ? bswap64_portable(bb) : bb, 1.0f); };
    auto const_plane = [&](float v) { sink(v != 0.0f ? ~0ULL : 0ULL, v); };
    auto square_plane = [&](int sq, bool on) { sink(on ? bit(p.flip ? (sq ^ 56) : sq) : 0ULL, 1.0f); };

    auto pieces_planes = [&]() {
        for (int k = 0; k < 2; ++k) {
            const int col = k == 0 ? p.me : p.you;
            for (int pt = 0; pt < 6; ++pt) bb_plane(b.by_type[pt] & b.by_color[col]);
        }
    };
    auto repetition_planes = [&]() {  // Board::number_repetitions never returns 2 (board.cpp:132-141)
        const_plane(b.repetition != 0 ? 1.0f : 0.0f);
        const_plane(0.0f);
    };
    auto pockets_planes = [&]() {
        for (int k = 0; k < 2; ++k) {
            const int col = k == 0 ? p.me : p.you;
            for (int pt = 0; pt < 5; ++pt) {
                const int cnt = b.variant == V_CRAZYHOUSE ? b.hand[col][pt] : 0;
                const_plane(cnt > 0 ? (p.normalize ? cnt / max_prisoners : static_cast<float>(cnt)) : 0.0f);
            }
        }
    };
    auto promoted_planes = [&]() {
        bb_plane(b.promoted & p.own);
        bb_plane(b.promoted & p.opp);
    };
    auto ep_plane = [&]() { square_plane(b.ep & 63, b.ep != 0xFF); };
    auto color_plane = [&]() { const_plane(p.me == 0 ? 1.0f : 0.0f); };
    auto move_count_plane = [&]() {
        const float v = static_cast<float>((b.game_ply / 2) + 1);
        const_plane(p.normalize ? v / 500.0f : v);
    };
    auto castling_planes = [&]() {  // me-OO, me-OOO, you-OO, you-OOO (:174-213)
        for (int k = 0; k < 2; ++k) {
            const int col = k == 0 ? p.me : p.you;
            for (int side = 0; side < 2; ++side) const_plane(b.castle_rook[col * 2 + side] != 0xFF ? 1.0f : 0.0f);
        }
    };
    auto no_progress_plane = [&]() {
        const float v = static_cast<float>(b.rule50);
        const_plane(p.normalize ? v / max_no_progress : v);
    };
    auto remaining_checks_planes = [&]() {  // :221-242
        for (int k = 0; k < 2; ++k) {
            const int col = k == 0 ? p.me : p.you;
            const int g = b.variant == V_THREECHECK ? checks_given(b, col) : 0;
            const_plane(g != 0 ? 1.0f : 0.0f);
            const_plane(g >= 2 ? 1.0f : 0.0f);
        }
    };
    auto variant_960_planes = [&]() {  // :246-260, CHANNEL_MAPPING_VARIANTS boardstate.h:269-279
        const int vc = b.variant + 1;
        for (int k = 0; k < 9; ++k) const_plane((k == 0 ? b.chess960 != 0 : k == vc) ? 1.0f : 0.0f);
    };
    auto last_moves_planes = [&]() {  // :262-282
        for (int i = 0; i < 8; ++i) {
            const bool have = i < b.n_last;
            const Move m = have ? b.last_moves[i] : 0;
            square_plane(mv_from(m), have && !mv_is_drop(m));
            square_plane(mv_to(m), have);
        }
    };
    auto is960_plane = [&]() { const_plane(b.chess960 ? 1.0f : 0.0f); };
    auto masks_planes = [&]() {
        bb_plane(p.own);
        bb_plane(p.opp);
    };
    auto checkerboard_plane = [&]() { sink(0x55AA55AA55AA55AAULL, 1.0f); };  // written unflipped, [0,0] = 0 (:301-313)
    auto rel_count = [&](float rel) { const_plane(rel != 0 ? (p.normalize ? rel / 8.0f : rel) : 0.0f); };
    auto material_diff_planes = [&](int npt) {
        for (int pt = 0; pt < npt; ++pt) rel_count(static_cast<float>(p.cnt[0][pt] - p.cnt[1][pt]));
    };
    auto material_count_planes = [&](int npt) {
        for (int pt = 0; pt < npt; ++pt) rel_count(static_cast<float>(p.cnt[0][pt]));
    };
    auto opp_bishops_plane = [&]() { const_plane(p.opp_bishops ? 1.0f : 0.0f); };
    auto checkers_plane = [&]() { bb_plane(p.checkers); };
    auto chess_v3 = [&]() {  // :536-566
        pieces_planes(); repetition_planes(); ep_plane(); castling_planes(); no_progress_plane(); last_moves_planes();
        is960_plane(); masks_planes(); checkerboard_plane(); material_diff_planes(5); opp_bishops_plane();
        checkers_plane(); material_count_planes(5);
    };

    if (version <= 1 || (p.mode == MODE_LICHESS && version == 2)) {  // default_board_to_planes :426-501
        pieces_planes();
        repetition_planes();
        if (p.mode != MODE_CHESS) { pockets_planes(); promoted_planes(); }
        ep_plane(); color_plane(); move_count_plane(); castling_planes(); no_progress_plane();
        if (p.mode == MODE_LICHESS) { remaining_checks_planes(); variant_960_planes(); }
        if (p.mode == MODE_CHESS) is960_plane();
        if (p.mode != MODE_CRAZYHOUSE) last_moves_planes();
    } else if (p.mode == MODE_CHESS) {
        chess_v3();
    } else if (p.mode == MODE_CRAZYHOUSE) {
        if (version == 3) {  // :569-577
            chess_v3(); pockets_planes(); promoted_planes();
        } else {  // v2 :579-595
            pieces_planes(); repetition_planes(); pockets_planes(); promoted_planes(); ep_plane(); color_plane();
            move_count_plane(); castling_planes(); no_progress_plane(); is960_plane(); last_moves_planes();
        }
    } else {  // lichess v3 :599-624
        pieces_planes(); repetition_planes(); pockets_planes(); promoted_planes(); ep_plane();
        const_plane(0.0f); const_plane(0.0f);  // colour info and move count are skipped
        castling_planes(); no_progress_plane(); remaining_checks_planes(); variant_960_planes(); last_moves_planes();
        masks_planes(); checkerboard_plane(); material_diff_planes(6); opp_bishops_plane(); checkers_plane();
        material_count_planes(6);
    }
}

// ---- sinks ------------------------------------------------------------------------------------------------------
struct NchwF32Sink {  // [C, 8, 8] fp32
    float* out;
    int c = 0;
#if defined(__CUDA_ARCH__)
    // Two planes per store instruction: lanes 0..15 write the pending plane, lanes 16..31 the current one, four squares
    // (16 bytes) each -- 512 contiguous bytes per warp instruction instead of 128, a quarter of the store instructions.
    uint64_t pm = 0;
    float pv = 0.0f;
    __device__ __forceinline__ void emit(uint64_t mask, float v, int plane, int quarter) {
        const unsigned bits = static_cast<unsigned>(mask >> (4 * quarter)) & 15u;
        const float4 o = make_float4((bits & 1u) ? v : 0.0f, (bits & 2u) ? v : 0.0f, (bits & 4u) ? v : 0.0f, (bits & 8u) ? v : 0.0f);
        __stcs(reinterpret_cast<float4*>(out + plane * 64) + quarter, o);  // (streamed: nothing reads the planes back soon)
    }
    __device__ __forceinline__ void operator()(uint64_t mask, float v) {
        if (c & 1) {
            const int lane = threadIdx.x & 31;
            if (lane < 16) emit(pm, pv, c - 1, lane);
            else emit(mask, v, c, lane - 16);
        } else {
            pm = mask, pv = v;
        }
        ++c;
    }
    __device__ __forceinline__ void flush() {  // an odd number of planes: the last one is still pending
        const int lane = threadIdx.x & 31;
        if ((c & 1) && lane < 16) emit(pm, pv, c - 1, lane);
    }
#else
    ARA_HD void operator()(uint64_t mask, float v) {
        for (int sq = ARA_LANE; sq < 64; sq += ARA_WARP_N) out[c * 64 + sq] = ((mask >> sq) & 1) ? v : 0.0f;
        ++c;
    }
    ARA_HD void flush() {}
#endif
};

struct LaneCaptureSink {  // keeps the descriptors of channels lane, lane+32, lane+64
    int lane;
    int c = 0;
    uint64_t m0 = 0, m1 = 0, m2 = 0;
    float v0 = 0.0f, v1 = 0.0f, v2 = 0.0f;
    ARA_HD void operator()(uint64_t mask, float v) {
        if (c == lane) { m0 = mask; v0 = v; }
        if (c == lane + 32) { m1 = mask; v1 = v; }
        if (c == lane + 64) { m2 = mask; v2 = v; }
        ++c;
    }
};

// the reference layout; warp-collective (1 lane on the host)
ARA_HD void encode_planes_nchw_f32(const Board& b, int mode, int version, bool normalize, float* out) {
    const PlaneCtx p = make_plane_ctx(b, mode, normalize);
    NchwF32Sink sink{out};
    for_each_plane(p, version, sink);
    sink.flush();
}

// where the lanes of one warp trade the channel descriptors of a board (encode_planes_nhwc_f16): shared memory of the
// calling kernel
struct PlaneExchange {
    uint64_t mask[96];
    uint16_t val[96];
};

#if defined(__CUDACC__)
// [64, cpad] fp16 rows (cpad = 64 or 128); channels >= C are written as zero.  Device only, warp-collective; `x` is the
// warp's own exchange in shared memory.
__device__ __forceinline__ void encode_planes_nhwc_f16(const Board& b, int mode, int version, __half* out, int cpad, PlaneExchange& x) {
    uint64_t* s_mask = x.mask;
    uint16_t* s_val = x.val;
    const PlaneCtx p = make_plane_ctx(b, mode, true);
    LaneCaptureSink sink;
    sink.lane = threadIdx.x & 31;
    for_each_plane(p, version, sink);
    const int lane = sink.lane;
    // every lane has computed the descriptors (square mask, value) of three channels; a row of the output is written in
    // 16-byte pieces of eight channels, so the descriptors change hands through shared memory once per board ...
    s_mask[lane] = sink.m0, s_mask[lane + 32] = sink.m1, s_mask[lane + 64] = sink.m2;
    s_val[lane] = __half_as_ushort(__float2half_rn(sink.v0));
    s_val[lane + 32] = __half_as_ushort(__float2half_rn(sink.v1));
    s_val[lane + 64] = __half_as_ushort(__float2half_rn(sink.v2));
    __syncwarp();
    const int chunks = cpad >> 3;                                // pieces per row: 8 (cpad 64) or 16 (cpad 128)
    const int j = lane % chunks, s0 = lane / chunks, step = 32 / chunks;
    uint64_t m[8];
    uint32_t v[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        const int ch = 8 * j + i;
        m[i] = ch < 96 ? s_mask[ch] : 0ull;
        v[i] = ch < 96 ? s_val[ch] : 0u;
    }
    // ... and every store instruction of the warp writes 512 contiguous bytes (4 or 2 whole rows)
    for (int sq = s0; sq < 64; sq += step) {
        uint32_t h[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) h[i] = ((m[i] >> sq) & 1ull) ? v[i] : 0u;
        const uint4 o = make_uint4(h[0] | (h[1] << 16), h[2] | (h[3] << 16), h[4] | (h[5] << 16), h[6] | (h[7] << 16));
        *reinterpret_cast<uint4*>(out + sq * cpad + 8 * j) = o;
    }
    __syncwarp();
}
// Precision float32: the same rows with every channel as the fp16 pair hi | hi | lo (conv_gemm.cuh), [64, 3 * cpad]
__device__ __forceinline__ void encode_planes_nhwc_split(const Board& b, int mode, int version, __half* out, int cpad) {
    const PlaneCtx p = make_plane_ctx(b, mode, true);
    LaneCaptureSink sink;
    sink.lane = threadIdx.x & 31;
    for_each_plane(p, version, sink);
    const int lane = sink.lane;
    const __half z = __float2half_rn(0.0f);
    const __half h0 = __float2half_rn(sink.v0), h1 = __float2half_rn(sink.v1), h2 = __float2half_rn(sink.v2);
    const __half l0 = __float2half_rn(sink.v0 - __half2float(h0)), l1 = __float2half_rn(sink.v1 - __half2float(h1)),
                 l2 = __float2half_rn(sink.v2 - __half2float(h2));
#pragma unroll 2
    for (int sq = 0; sq < 64; ++sq) {
        __half* row = out + sq * 3 * cpad;
        const bool b0 = (sink.m0 >> sq) & 1, b1 = (sink.m1 >> sq) & 1, b2 = (sink.m2 >> sq) & 1;
        row[lane] = row[cpad + lane] = b0 ? h0 : z;
        row[2 * cpad + lane] = b0 ? l0 : z;
        row[lane + 32] = row[cpad + lane + 32] = b1 ? h1 : z;
        row[2 * cpad + lane + 32] = b1 ? l1 : z;
        if (cpad > 64) {
            row[lane + 64] = row[cpad + lane + 64] = b2 ? h2 : z;
            row[2 * cpad + lane + 64] = b2 ? l2 : z;
            row[lane + 96] = row[cpad + lane + 96] = row[2 * cpad + lane + 96] = z;
        }
    }
}
#endif

}  // namespace ara
