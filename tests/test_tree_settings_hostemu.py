"""Per-tree Q-value weight and Dirichlet epsilon (ara_search_set_tree_settings) in the 1-lane host emulation: the trees of
one handle share its settings, and each may override the two values for its own searches (self-play's quick searches).
Every tree must then search exactly like a single-tree oracle search (oracle/mcts.c) run with that tree's values; a
tree without an override (negative values) exactly like one with the handle's settings."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

from oracle import search as osr
from oracle.chess import Position
from tests.hostemu import HeSearch, HeState
from tests.test_search_hostemu import assert_same_search

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HOSTEMU = os.path.join(ROOT, "tests", "hostemu")

# (Q-value weight, Dirichlet epsilon) per tree of one handle; negative = the handle's value
TREES = [(-1.0, -1.0), (0.0, 0.25), (0.7, 0.0), (2.0, 0.1), (-1.0, 0.0), (0.0, -1.0)]
# the handle's settings: (mode, variant, moves played, Batch_Size, simulations, extra settings)
HANDLES = [("crazyhouse", "crazyhouse", [], 8, 300, dict(q_value_weight=1.0, dirichlet_epsilon=0.25, dirichlet_alpha=0.3, seed=7)),
           ("chess", "chess", ["e2e4", "c7c5"], 16, 400, dict(q_value_weight=0.0, dirichlet_epsilon=0.0, dirichlet_alpha=0.3, seed=3))]


@pytest.fixture(scope="module")
def ts_lib(tmp_path_factory):
    """tests/hostemu/tree_settings.cpp, built like the host emulation itself (tests/hostemu/__init__.py)"""
    so = str(tmp_path_factory.mktemp("tree_settings") / "libtree_settings.so")
    subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wall", "-ffp-contract=off", "-I" + os.path.join(ROOT, "crazyara_b200", "csrc"),
                    "-I" + os.path.join(ROOT, "include"), "-x", "c++", os.path.join(HOSTEMU, "tree_settings.cpp"), "-o", so], check=True)
    L = ctypes.CDLL(so)
    L.he_search_set_root_with_settings.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_float, ctypes.c_float]
    return L


class _TreeLib:
    """The host emulation's entry points, with the root phase of a tree that carries its own settings"""

    def __init__(self, he_lib, ts_lib, q_value_weight, dirichlet_epsilon):
        self._he, self._ts, self._q, self._eps = he_lib, ts_lib, q_value_weight, dirichlet_epsilon

    def __getattr__(self, name):
        return getattr(self._he, name)

    def he_search_set_root(self, h, root):
        return self._ts.he_search_set_root_with_settings(h, root, self._q, self._eps)


def _tree_search(ts_lib, st, q_value_weight, dirichlet_epsilon):
    H = HeSearch(st, max_nodes=1 << 15)
    # (both libraries are built from hostemu.cpp, so they agree on the layout of the HeSearch they share)
    H.L = _TreeLib(H.L, ts_lib, q_value_weight, dirichlet_epsilon)
    return H


@pytest.mark.parametrize("threads", [1, 2])
@pytest.mark.parametrize("handle", HANDLES, ids=[h[0] for h in HANDLES])
def test_every_tree_searches_like_a_single_tree_with_its_values(ts_lib, handle, threads):
    mode, variant, moves, batch, sims, extra = handle
    vid = {"chess": 0, "crazyhouse": 1}[variant]
    st = osr.default_settings(mode, batch_size=batch, simulations=sims, node_policy_temperature=1.0, threads=threads, **extra)
    pos = Position(None, variant, False)
    he = HeState(pos.fen(), vid, False)
    for m in moves:
        pos.push_uci(m)
        he.do_move(he.move_from_uci(m))
    results = []
    for q, eps in TREES:
        # the single-tree oracle search with this tree's values in place of the handle's
        ost = osr.default_settings(mode, batch_size=batch, simulations=sims, node_policy_temperature=1.0, threads=threads,
                                   **dict(extra, q_value_weight=q if q >= 0 else extra["q_value_weight"],
                                          dirichlet_epsilon=eps if eps >= 0 else extra["dirichlet_epsilon"]))
        S = osr.Search(ost)
        ro = S.run(pos, osr.fake_net(S.n_labels), with_keys=True, threads=threads)
        rh = _tree_search(ts_lib, st, q, eps).run(he, osr.fake_net(S.n_labels), with_keys=True, threads=threads)
        assert_same_search(ro, rh)
        results.append(rh)
    # the trees' values matter: noise on / off changes the priors, the Q-value weight the posterior
    assert any(not np.array_equal(r["prior"], results[0]["prior"]) for r in results[1:])
    assert any(not np.array_equal(r["policy"], results[0]["policy"]) for r in results[1:])
