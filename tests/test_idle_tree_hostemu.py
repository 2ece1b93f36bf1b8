"""Idle trees (ara_search_set_active): the root phase of a go that leaves a tree out (search_dev.cuh idle_root, what
root_kernel runs for it) in the 1-lane host emulation.  A match needs it between the two moves of a game that a player
sees: its own move is applied to its tree, the tree sits out the opponent's search, then the opponent's reply is applied
-- and the next search must continue on the kept subtree exactly as if the idle go had never happened
(MCTSAgent::apply_move_to_tree(move, false) of the passive player, rl/selfplay.cpp:297-299)."""
import ctypes
import os
import subprocess

import pytest

from oracle import search as osr
from oracle.chess import Position
from crazyara_b200.engine import result_to_dict
from tests.hostemu import HeSearch, HeState
from tests.test_search_hostemu import assert_same_search
from tests.test_tree_reuse_hostemu import CASES


ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HOSTEMU = os.path.join(ROOT, "tests", "hostemu")


@pytest.fixture(scope="module")
def idle_lib(tmp_path_factory):
    """tests/hostemu/idle_root.cpp, built like the host emulation itself (tests/hostemu/__init__.py), into a temporary
    directory"""
    so = str(tmp_path_factory.mktemp("idle_root") / "libidle_root.so")
    subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wall", "-ffp-contract=off", "-I" + os.path.join(ROOT, "crazyara_b200", "csrc"),
                    "-I" + os.path.join(ROOT, "include"), "-x", "c++",
                    os.path.join(HOSTEMU, "idle_root.cpp"), "-o", so], check=True)
    L = ctypes.CDLL(so)
    L.he_search_idle_root.argtypes = [ctypes.c_void_p]
    return L


def _idle_root(L, H):
    L.he_search_idle_root(H.h)


def _result(H, he):
    return result_to_dict(H.L.he_search_result(H.h).contents, he.uci)


@pytest.mark.parametrize("threads", [1, 2])
@pytest.mark.parametrize("variant,vid,mode,batch,sims,extra", CASES)
def test_idle_go_between_the_two_moves_keeps_the_subtree(idle_lib, variant, vid, mode, batch, sims, extra, threads):
    if threads == 2 and 2 * batch >= 256:
        pytest.skip("Threads x Batch_Size")
    st = osr.default_settings(mode, batch_size=batch, simulations=sims, node_policy_temperature=1.0, threads=threads, **extra)
    pos = Position(None, variant, False)
    he = HeState(pos.fen(), vid, False)
    S, H = osr.Search(st), HeSearch(st, max_nodes=1 << 16)
    for ply in range(3):
        ro = S.run(pos, osr.fake_net(S.n_labels), with_keys=True, threads=threads)
        rh = H.run(he, osr.fake_net(H.n_labels), with_keys=True, threads=threads)
        assert S.reused == H.reused == (ply > 0)
        assert_same_search(ro, rh)
        if ply > 0:
            assert rh["nodes_pre_search"] == S.nodes_pre_search > 0
        assert rh["pv_len"] >= 2
        m1, m2 = rh["pv"][0], rh["pv"][1]          # the played move and a reply that has visits in the kept subtree
        S.apply_move(pos.move_from_uci(m1))
        H.apply_move(he.move_from_uci(m1))
        _idle_root(idle_lib, H)                    # the tree sits out the opponent's search ...
        ri = _result(H, he)                        # ... and shows its last result
        assert_same_search(rh, ri)
        assert ri["pv"] == rh["pv"] and ri["nodes_pre_search"] == rh["nodes_pre_search"]
        pos.push_uci(m1)
        he.do_move(he.move_from_uci(m1))
        S.apply_move(pos.move_from_uci(m2))        # the opponent's reply descends from the pending candidate
        H.apply_move(he.move_from_uci(m2))
        pos.push_uci(m2)
        he.do_move(he.move_from_uci(m2))
    ro = S.run(pos, osr.fake_net(S.n_labels), with_keys=True, threads=threads)
    rh = H.run(he, osr.fake_net(H.n_labels), with_keys=True, threads=threads)
    assert S.reused and H.reused and rh["nodes_pre_search"] == S.nodes_pre_search > 0
    assert_same_search(ro, rh)


def test_a_tree_that_never_searched_shows_no_moves(idle_lib):
    st = osr.default_settings("crazyhouse", batch_size=8, simulations=100)
    H = HeSearch(st)
    he = HeState(Position(None, "crazyhouse", False).fen(), 1, False)
    _idle_root(idle_lib, H)
    r = _result(H, he)
    assert r["moves"] == [] and r["visit_sum"] == 0 and r["tree_nodes"] == 0 and r["error"] == 0 and r["best_idx"] == -1
