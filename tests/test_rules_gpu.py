"""Device move generator, terminal rules, policy-map indices and the plane-encode kernel on the GPU, through the
C-ABI with host buffers, against the CPU oracle: bit-exact on seeded random playouts and on the reference's
PlaneStatistics literals (engine/tests/tests.cpp)."""
import ctypes
import random

import numpy as np
import pytest

from oracle.chess import Position, lib as olib, planes as oplanes

VARIANTS = [("chess", 0), ("crazyhouse", 1), ("kingofthehill", 2), ("3check", 3)]


def _collect_positions(name, vid, rnd, games, max_plies):
    from crazyara_b200.engine import BoardState
    out = []
    for _ in range(games):
        pos = Position(variant=name)
        st = BoardState().set("", False, vid)
        for _ in range(max_plies):
            moves = pos.legal_uci()
            out.append((pos.clone(), st.clone()))
            if pos.terminal(len(moves)) != 4 or not moves:
                break
            u = rnd.choice(sorted(moves))
            pos.push_uci(u)
            st.do_uci(u)
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("name,vid", VARIANTS)
def test_gpu_movegen_terminal_policy_planes_match_oracle(name, vid):
    from crazyara_b200.engine import encode_planes, legal_moves_gpu, move_to_uci
    L = olib()
    L.opolicy_move_index.argtypes = [ctypes.c_void_p, ctypes.c_uint32, ctypes.c_int, ctypes.c_int]
    rnd = random.Random(99 + vid)
    positions = _collect_positions(name, vid, rnd, games=10, max_plies=160)
    boards = [st.board() for _, st in positions]
    moves, term, pidx = legal_moves_gpu(boards)
    policy_mode = 0 if vid == 1 else (1 if vid == 0 else 2)
    for (pos, st), mv, tt, pi in zip(positions, moves, term, pidx):
        assert st.fen() == pos.fen()
        o = {pos.uci(m): L.opolicy_move_index(pos._buf, m, policy_mode, 1) for m in pos.legal_moves()}
        g = {move_to_uci(m, False): p for m, p in zip(mv, pi)}
        assert o == g, pos.fen()
        assert tt == pos.terminal(len(o)), pos.fen()
    mode_versions = {0: [(1, 1), (1, 3)], 1: [(0, 1), (0, 2), (0, 3)], 2: [(2, 1), (2, 3)], 3: [(2, 1), (2, 3)]}[vid]
    for mode, version in mode_versions:
        for norm in (False, True):
            got = encode_planes(boards, mode, version, norm)
            for i, (pos, _) in enumerate(positions):
                assert np.array_equal(got[i], oplanes(pos, mode, version, norm)), (pos.fen(), mode, version, norm)


# Every input layout per variant: (mode, version) with mode 0 crazyhouse, 1 chess, 2 lichess
LAYOUTS = {0: [(1, 1), (1, 3)], 1: [(0, 1), (0, 2), (0, 3)], 2: [(2, 1), (2, 2), (2, 3)], 3: [(2, 1), (2, 2), (2, 3)]}

# Positions whose planes fp16 cannot hold exactly (rule50 / 40 or / 50, full-move numbers / 500), full pockets, promoted
# pieces of both colours, en passant, checks given in Three-check, partial chess960 castling rights, both sides to move:
# (variant id, FEN or None for the start position, chess960, moves played from it; every prefix is encoded)
CRAFTED = [
    (0, "8/8/4k3/8/8/3K4/8/R7 w - - 97 431", False, []),
    (0, "8/8/4k3/8/8/3K4/8/R7 b - - 99 612", False, []),
    (0, "bqnb1rkr/pp3ppp/3ppn2/2p5/5P2/P2P4/NPP1P1PP/BQ1BNRKR w Hf - 2 9", True, ["f4f5"]),
    (0, "nrbbqnkr/pppppppp/8/8/8/8/PPPPPPPP/NR4KR w B - 0 1", True, ["g1b1"]),
    (0, "bnnrkbrq/pppppppp/8/8/8/8/PPPPPPPP/BN1RK1RQ w Dg - 0 1", True, ["e1d1"]),
    (0, None, False, ["e2e4", "a7a6", "e4e5", "d7d5"]),
    (1, "r3k2r/1Q~6/8/8/8/8/6q~1/R3K2R[NNbbPPpp] b KQkq - 38 401", False, ["e8g8"]),
    (1, "rnbqkbnr/pppppppp/8/8/8/8/PPPPPPPP/RNBQKBNR[QQRRBBNNPPPPPPPPqqrrbbnnpppppppp] w KQkq - 39 250", False, ["Q@e3"]),
    (1, "4R2b~/1N3rkb/1p2P1pp/p2P4/2P1P3/8/PP4Q~1/3R3K[QRBBNNNPPPPpp] w - - 37 253", False, ["g2g3"]),
    (1, None, False, ["e2e4", "a7a6", "e4e5", "d7d5"]),
    (2, None, False, ["e2e4", "e7e5", "e1e2", "e8e7", "e2e3"]),
    (2, "8/8/3k4/8/8/3K4/8/8 b - - 93 421", False, ["d6c5"]),
    (3, None, False, ["e2e4", "e7e5", "f1c4", "f8c5", "c4f7", "e8f7", "d1h5", "g7g6", "h5e5", "c5f2"]),
]


def _crafted_positions(vid):
    from crazyara_b200.engine import BoardState
    name = [v[0] for v in VARIANTS if v[1] == vid][0]
    out = []
    for v, fen, is960, moves in CRAFTED:
        if v != vid:
            continue
        pos, st = Position(fen, name, is960), BoardState().set(fen or "", is960, vid)
        out.append((pos.clone(), st.clone()))
        for u in moves:
            pos.push_uci(u)
            st.do_uci(u)
            out.append((pos.clone(), st.clone()))
    return out


def _encode_device(boards, mode, version, normalize, f32, f16, cpad, n=None):
    """ara_encode_planes_device on torch device buffers (n boards, default all); returns the call's return code"""
    import torch
    from crazyara_b200 import lib
    from crazyara_b200.engine import AraBoard
    L = lib()
    L.ara_encode_planes_device.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int,
                                           ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p]
    n = len(boards) if n is None else n
    host = np.frombuffer((AraBoard * max(len(boards), 1))(*boards), np.uint8).reshape(-1, 128)
    d_b = torch.from_numpy(host.copy()).cuda()
    rc = L.ara_encode_planes_device(d_b.data_ptr(), n, mode, version, normalize, None if f32 is None else f32.data_ptr(),
                                    None if f16 is None else f16.data_ptr(), cpad, torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    return rc


@pytest.mark.gpu
@pytest.mark.parametrize("name,vid", VARIANTS)
def test_gpu_device_encoder_fp16_nhwc_matches_oracle(name, vid):
    """The stem's input as the device search writes it (encode_planes_nhwc_f16, expand_kernel's float16 sink) through
    ara_encode_planes_device: [64, cpad] half rows, bit for bit the oracle's normalised planes rounded to nearest even
    (numpy's float16 conversion, as __float2half_rn), channels C..cpad zero, at cpad 64 and 128 for every layout that
    fits; the fp32 output of the same call equals ara_encode_planes."""
    import torch
    from crazyara_b200.engine import encode_planes
    positions = _crafted_positions(vid) + _collect_positions(name, vid, random.Random(7 + vid), games=3, max_plies=160)
    boards = [st.board() for _, st in positions]
    for pos, st in positions:
        assert st.fen() == pos.fen()
    n = len(boards)
    for mode, version in LAYOUTS[vid]:
        want = np.stack([oplanes(pos, mode, version, True) for pos, _ in positions])
        c = want.shape[1]
        want_f32 = encode_planes(boards, mode, version, True)
        assert np.array_equal(want_f32, want)
        rows = want.astype(np.float16).reshape(n, c, 64).transpose(0, 2, 1)
        for cpad in [p for p in (64, 128) if p >= c]:
            want_h = np.zeros((n, 64, cpad), np.float16)
            want_h[:, :, :c] = rows
            f32 = torch.full((n, c, 8, 8), float("nan"), dtype=torch.float32, device="cuda")
            f16 = torch.full((n, 64, cpad), float("nan"), dtype=torch.float16, device="cuda")
            assert _encode_device(boards, mode, version, 1, f32, f16, cpad) == 0
            got_h = f16.cpu().numpy().view(np.uint16)
            bad = np.nonzero((got_h != want_h.view(np.uint16)).any(axis=(1, 2)))[0]
            assert bad.size == 0, (mode, version, cpad, positions[bad[0]][0].fen())
            assert np.array_equal(f32.cpu().numpy(), want_f32), (mode, version, cpad)
        # the fp32 output alone, not normalised
        f32 = torch.full((n, c, 8, 8), float("nan"), dtype=torch.float32, device="cuda")
        assert _encode_device(boards, mode, version, 0, f32, None, 0) == 0
        assert np.array_equal(f32.cpu().numpy(), encode_planes(boards, mode, version, False)), (mode, version)


@pytest.mark.gpu
def test_gpu_device_encoder_argument_rules():
    """The fp16 output is the network's input and always normalised: normalize = 0 with it is refused (and nothing is
    written); no boards is a successful no-op, a negative count an error."""
    import torch
    from crazyara_b200 import lib
    from crazyara_b200.engine import BoardState
    boards = [BoardState().set("", False, 1).do_uci("e2e4").board()]
    f32 = torch.full((1, 34, 8, 8), float("nan"), dtype=torch.float32, device="cuda")
    f16 = torch.full((1, 64, 64), float("nan"), dtype=torch.float16, device="cuda")
    assert _encode_device(boards, 0, 1, 0, f32, f16, 64) != 0
    assert "normalize = 0" in lib().ara_last_error().decode()
    assert _encode_device(boards, 0, 1, 1, f32, f16, 64, n=-1) != 0
    assert "negative" in lib().ara_last_error().decode()
    assert _encode_device(boards, 0, 1, 1, f32, f16, 64, n=0) == 0
    assert _encode_device(boards, 0, 1, 0, f32, None, 0, n=0) == 0
    assert torch.isnan(f32).all() and torch.isnan(f16).all()
    # a well-formed call still succeeds after the refusals
    assert _encode_device(boards, 0, 1, 1, f32, f16, 64) == 0
    assert not torch.isnan(f32).any() and not torch.isnan(f16).any()


@pytest.mark.gpu
def test_gpu_planes_reference_goldens():
    """engine/tests/tests.cpp:1493-1527 (crazyhouse V1) and :341-365 (chess v3) through the CUDA encoder."""
    from crazyara_b200.engine import BoardState
    st = BoardState().set("5r2/ppp2pkp/3p4/2bP4/2Pnp1N1/3P2pP/PP2n1P1/R2Q1R1K[PBRQnbb] w - - 0 28", False, 1)
    st.do_uci("Q@f6", "g7g8", "R@h8")
    assert st.fen() == "5rkR/ppp2p1p/3p1Q2/2bP4/2Pnp1N1/3P2pP/PP2n1P1/R2Q1R1K[BPbbn] b - - 3 29"
    p = st.get_state_planes(False, 0, 1).reshape(-1).astype(np.float64)
    assert p.sum() == 2395 and p.max() == 29 and (np.arange(p.size) * p).sum() == 4170903 and int(p.argmax()) == 1792
    st = BoardState().set("", False, 0)
    p = st.get_state_planes(False, 1, 3).reshape(-1).astype(np.float64)
    assert p.sum() == 1312 and p.max() == 8 and (np.arange(p.size) * p).sum() == 3430384 and int(p.argmax()) == 3008
    p = st.get_state_planes(True, 1, 3).reshape(-1).astype(np.float64)
    assert p.sum() == 472 and (np.arange(p.size) * p).sum() == 819860
    st = BoardState().set("b1qnrnkr/p2ppppp/1p6/2p1b3/2P5/4N1P1/PP1PPP1P/BBQNRK1R b he - 1 4", True, 0)
    p = st.get_state_planes(False, 1, 3).reshape(-1).astype(np.float64)
    assert p.sum() == 1312 and (np.arange(p.size) * p).sum() == 3512322
