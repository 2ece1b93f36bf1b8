"""classic_label_index (crazyara_b200/csrc/chess_dev.cuh), the move -> classic-label index of the training data's y_policy,
in the host emulation: every legal move of seeded random playouts in the three label modes, both colours, chess960
castling, promotions, en passant and drops, against the oracle (oracle/policy.c opolicy_move_index(..., 0)) and
crazyara_b200.labels.classic_index."""
import ctypes
import os
import random
import subprocess

import pytest

from crazyara_b200.labels import classic_index
from oracle.chess import Position, lib as oracle_lib
from tests.hostemu import HeState

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HOSTEMU = os.path.join(ROOT, "tests", "hostemu")

# (label mode, variant id, chess960, start FEN or None)
CASES = [(0, 1, False, None), (1, 0, False, None), (1, 0, True, None), (2, 2, False, None), (2, 3, False, None),
         (2, 1, False, None),
         # both colours' promotions (straight, both captures) and en passant at once
         (1, 0, False, "1n2k1n1/P1P3P1/8/3pP3/8/8/p1p3p1/1N2K1N1 w - d6 0 1"),
         (2, 0, False, "1n2k1n1/P1P3P1/8/8/3Pp3/8/p1p3p1/1N2K1N1 b - d3 0 1"),
         (0, 1, False, "1n2k1n1/P1P3P1/8/3pP3/8/8/p1p3p1/1N2K1N1[QRBNPqrbnp] w - d6 0 1"),
         # chess960 castling: king and rooks on non-standard files, both sides
         (1, 0, True, "1r2k1r1/pppppppp/8/8/8/8/PPPPPPPP/1R2K1R1 w GBgb - 0 1"),
         (1, 0, True, "1r2k1r1/pppppppp/8/8/8/8/PPPPPPPP/1R2K1R1 b GBgb - 0 1"),
         (1, 0, False, "r3k2r/pppppppp/8/8/8/8/PPPPPPPP/R3K2R b KQkq - 0 1")]
VARIANT_NAMES = {0: "chess", 1: "crazyhouse", 2: "kingofthehill", 3: "3check"}


@pytest.fixture(scope="module")
def ci_lib(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("classic_index") / "libclassic_index.so")
    subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wall", "-I" + os.path.join(ROOT, "crazyara_b200", "csrc"),
                    "-I" + os.path.join(ROOT, "include"), "-x", "c++", os.path.join(HOSTEMU, "classic_index.cpp"), "-o", so],
                   check=True)
    L = ctypes.CDLL(so)
    L.he_classic_index.argtypes = [ctypes.c_void_p, ctypes.c_uint16, ctypes.c_int]
    return L


def _check_position(L, OL, st, pos, mode, seen):
    board = ctypes.create_string_buffer(st.board_bytes(), 128)
    black = st.fen().split()[1] == "b"
    n = 0
    for m in st.legal_moves():
        uci = st.uci(m)
        got = L.he_classic_index(board, m, mode)
        want = classic_index(mode, uci, black)
        assert got == want, (st.fen(), uci, mode, got, want)
        assert OL.opolicy_move_index(pos._buf, pos.move_from_uci(uci), mode, 0) == want, (st.fen(), uci)
        flag = m >> 12
        seen.add(("drop" if flag >= 8 else {1: "promo", 2: "promo", 3: "promo", 4: "promo", 5: "ep", 6: "castle"}.get(flag, "normal"),
                  black))
        n += 1
    return n


@pytest.mark.parametrize("mode,variant,is960,fen", CASES)
def test_classic_index_matches_oracle_and_labels(ci_lib, mode, variant, is960, fen):
    OL = oracle_lib()
    OL.opolicy_move_index.argtypes = [ctypes.c_void_p, ctypes.c_uint32, ctypes.c_int, ctypes.c_int]
    rng = random.Random(1000 * mode + 10 * variant + int(is960))
    seen, total = set(), 0
    for game in range(6 if fen is None else 2):
        st = HeState(fen or Position(None, VARIANT_NAMES[variant], is960).fen(), variant, is960)
        if is960 and fen is None and game > 0:  # random chess960 set-ups as self-play draws them
            from crazyara_b200.selfplay import chess960_fen
            import numpy as np
            st = HeState(chess960_fen(np.random.default_rng(game)), variant, True)
        pos = Position(st.fen(), VARIANT_NAMES[variant], is960)
        for _ in range(160):
            total += _check_position(ci_lib, OL, st, pos, mode, seen)
            moves = st.legal_moves()
            if not moves or st.terminal() != 4:
                break
            m = rng.choice(moves)
            pos.push_uci(st.uci(m))
            st.do_move(m)
    assert total > 0
    if fen is not None:
        kinds = {k for k, _ in seen}
        assert "promo" in kinds or "castle" in kinds
    if variant == 1 and fen is None:
        assert ("drop", False) in seen and ("drop", True) in seen

