"""Idle trees (ara_search_set_active) on the device search, and matches between two networks (crazyara_b200/match.py)
on the GPU: idle trees leave the active ones bit-identical and are themselves untouched (statistics, root noise
generator, pending kept subtree); a match of a player against itself is symmetric; a match with tree reuse equals a
host replay of the reference's generate_arena_game; the command line runs end to end."""
import os
import subprocess
import sys

import numpy as np
import pytest

from tests.test_search_hostemu import assert_same_search

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LINES = [[], ["e2e4"], ["e2e4", "e7e5"], ["d2d4", "g8f6", "c2c4"], ["g1f3", "d7d5"], ["e2e4", "c7c5", "g1f3"],
         ["b1c3"], ["d2d4", "d7d5", "c1f4", "g8f6"]]


def _blob(tmp_path, seed):
    from crazyara_b200.weights import export_blob
    from oracle import net as onet
    arch = onet.arch_risev2(34, 81)
    return export_blob(onet.make_state_dict(arch, seed), arch, str(tmp_path / f"risev2_{seed}.arab"), input_version=10)


def _net(tmp_path, seed, batch):
    from crazyara_b200.nn import NeuralNetAPI
    return NeuralNetAPI("gpu", 0, batch, _blob(tmp_path, seed))


def _state(t):
    from crazyara_b200.engine import BoardState
    return BoardState().set("", False, 1).do_uci(*LINES[t % len(LINES)])


def _settings(**kw):
    from crazyara_b200.engine import default_settings
    base = dict(batch_size=8, simulations=200, node_policy_temperature=1.0)
    base.update(kw)
    return default_settings("crazyhouse", **base)


def _same(a, b):
    assert_same_search(a, b)
    assert a["pv"] == b["pv"] and a["nodes_pre_search"] == b["nodes_pre_search"]


@pytest.mark.gpu
@pytest.mark.parametrize("backend", ["fake", "risev2"])
@pytest.mark.parametrize("threads", [1, 2])
@pytest.mark.parametrize("n_trees", [8, 40])     # 8 trees: select_wave_kernel; 40: select_kernel
def test_idle_trees_leave_the_active_trees_alone(tmp_path, backend, threads, n_trees):
    from crazyara_b200.engine import MCTSAgent
    st = _settings(threads=threads, dirichlet_epsilon=0.25, dirichlet_alpha=0.3, seed=7)
    net = _net(tmp_path, 0, n_trees * 8) if backend == "risev2" else None
    full, half = MCTSAgent(net, st, 0, n_trees), MCTSAgent(net, st, 0, n_trees)
    for t in range(n_trees):
        full.set_position(_state(t), t)
        half.set_position(_state(t), t)
        half.set_active(t, t % 2 == 0)
    full.evaluate_board_state()
    half.evaluate_board_state()
    for t in range(0, n_trees, 2):
        a, b = full.result(t), half.result(t)
        _same(a, b)
        assert a["evals"] > 0 and a["best_move"] == b["best_move"]
    for t in range(1, n_trees, 2):
        assert half.result(t)["moves"] == []          # never searched
    full.close()
    half.close()
    if net is not None:
        net.close()


@pytest.mark.gpu
@pytest.mark.parametrize("backend", ["fake", "risev2"])
def test_an_idle_tree_is_untouched(tmp_path, backend):
    """Its node view and result do not change in an idle go, and its next search equals that of a handle that never had
    the idle go: the Dirichlet generator did not advance.  With every tree idle nothing runs on the network."""
    from crazyara_b200.engine import MCTSAgent
    st = _settings(dirichlet_epsilon=0.25, dirichlet_alpha=0.3, seed=11)
    net = _net(tmp_path, 0, 4 * 8) if backend == "risev2" else None
    a, b = MCTSAgent(net, st, 0, 4), MCTSAgent(net, st, 0, 4)
    for h in (a, b):
        for t in range(4):
            h.set_position(_state(t), t)
        h.evaluate_board_state()
    before_node, before_res = a.node(-1, 1), a.result(1)
    a.set_active(1, False)
    for t in (0, 2, 3):
        a.set_position(_state(t + 4), t)
    a.evaluate_board_state()
    after_node, after_res = a.node(-1, 1), a.result(1)
    _same(before_res, after_res)
    for k in ("visits", "real_visits", "free_visits", "value", "key", "moves", "child"):
        assert before_node[k] == after_node[k], k
    for k in ("child_visits", "q", "prior", "virtual_loss"):
        assert np.array_equal(before_node[k], after_node[k]), k
    # every tree idle: no forward, no tree running
    a.set_active(-1, False)
    launches = net.launch_count() if net is not None else None
    a.begin()
    assert a.thread_iteration(1) == 0
    a.evaluate_board_state()
    if net is not None:
        assert net.launch_count() == launches
    _same(after_res, a.result(1))
    # tree 1's next search (a new position: a new root with root noise) in both handles
    a.set_active(-1, True)
    for h in (a, b):
        h.set_position(_state(5), 1)
        h.evaluate_board_state()
    _same(a.result(1), b.result(1))
    a.close()
    b.close()
    if net is not None:
        net.close()


@pytest.mark.gpu
@pytest.mark.parametrize("threads", [1, 2])
def test_pending_reuse_survives_an_idle_go(threads):
    """apply_move(m1), an idle go, apply_move(m2), a go: the same as without the idle go, on the kept subtree."""
    from crazyara_b200.engine import MCTSAgent
    st = _settings(threads=threads, simulations=400, dirichlet_epsilon=0.25, dirichlet_alpha=0.3)
    a, b = MCTSAgent(None, st, 0, 2, 1 << 14), MCTSAgent(None, st, 0, 2, 1 << 14)
    sa, sb = _state(0), _state(0)
    for h, s in ((a, sa), (b, sb)):
        h.set_position(s, 0)
        h.set_position(_state(3), 1)
        h.evaluate_board_state()
    r = a.result(0)
    m1, m2 = r["pv"][0], r["pv"][1]
    for h, s in ((a, sa), (b, sb)):
        h.apply_move_to_tree(m1, 0)
    a.set_active(0, False)
    a.set_position(_state(4), 1)
    a.evaluate_board_state()                           # tree 0 sits this one out
    a.set_active(0, True)
    for h, s in ((a, sa), (b, sb)):
        s.do_uci(m1)
        h.apply_move_to_tree(m2, 0)
        s.do_uci(m2)
        h.set_position(s, 0)
        h.set_active(1, False)
        h.evaluate_board_state()
    ra, rb = a.result(0), b.result(0)
    _same(ra, rb)
    assert ra["nodes_pre_search"] > 0
    a.close()
    b.close()


def _deterministic():
    from crazyara_b200.selfplay import rl_settings
    return rl_settings("crazyhouse", nodes=120, simulations=480, dirichlet_epsilon=0.0)


@pytest.mark.gpu
@pytest.mark.parametrize("backend", ["fake", "risev2"])
def test_a_player_against_itself_scores_one_half(tmp_path, backend):
    from crazyara_b200.match import Match
    n = 6
    net = _net(tmp_path, 0, n * 8) if backend == "risev2" else None
    st = _deterministic()
    m = Match((net, st, "p"), (net, st, "p"), n, variant=1, temperature_moves=0, max_plies=60, seed=2)
    m.run()
    m.close()
    games = sorted(m.finished, key=lambda g: g["game"])
    assert len(games) == n
    for k in range(n // 2):
        assert games[2 * k]["moves"] == games[2 * k + 1]["moves"] and games[2 * k]["result"] == games[2 * k + 1]["result"]
        assert all(np.array_equal(x, y) for x, y in zip(games[2 * k]["visits"], games[2 * k + 1]["visits"]))
    r = m.result
    assert r.wins == r.losses and r.score() == np.float32(0.5) and r.verdict() == "keep"
    if net is not None:
        net.close()


@pytest.mark.gpu
def test_match_equals_a_replay_of_the_reference_game_loop(tmp_path):
    """Two different networks, tree reuse, 4 games: every move and every root's visit counts equal a host replay of
    generate_arena_game (rl/selfplay.cpp:263-307) with one single-tree agent per player, driven one move at a time."""
    from crazyara_b200.engine import BoardState, MCTSAgent
    from crazyara_b200.match import CONTENDER, Match
    n, max_nodes, max_plies = 4, 6000, 40
    nets = [_net(tmp_path, s, n * 8) for s in (0, 1)]
    st = _deterministic()
    m = Match((nets[0], st, "p"), (nets[1], st, "c"), n, variant=1, temperature_moves=0, max_plies=max_plies,
              reuse_tree=True, max_nodes=max_nodes)
    m.run()
    m.close()
    games = sorted(m.finished, key=lambda g: g["game"])
    assert len(games) == n and sum(p > 0 for g in games for p in g["nodes_pre_search"]) > 10
    for g in games:
        players = [MCTSAgent(nets[i], st, 0, 1, max_nodes) for i in (0, 1)]   # fresh trees: clear_game_history
        white = players[g["white"]]
        black = players[1 - g["white"]]
        state = BoardState().set(g["fen"], False, 1)
        moves, visits, pre = [], [], []
        for ply in range(g["plies"]):
            active, passive = (white, black) if state.side_to_move() == 0 else (black, white)
            r = active.evaluate_board_state(state)
            move = r["best_move"]
            action = state.uci_to_action(move)
            active.apply_move_to_tree(action)
            if ply != 0:
                passive.apply_move_to_tree(action)
            state.do_action(action)
            moves.append(move)
            visits.append(r["visits"])
            pre.append(r["nodes_pre_search"])
        assert moves == g["moves"] and pre == g["nodes_pre_search"], g["game"]
        assert all(np.array_equal(x, y) for x, y in zip(visits, g["visits"]))
        for p in players:
            p.close()
    assert {g["white"] for g in games} == {CONTENDER, 1 - CONTENDER}
    for net in nets:
        net.close()


@pytest.mark.gpu
def test_command_line_end_to_end(tmp_path):
    prod, cont = _blob(tmp_path, 0), _blob(tmp_path, 1)
    out = tmp_path / "out"
    n = 3
    cmd = [sys.executable, "-m", "crazyara_b200.match", prod, cont, "--games", str(n), "--devices", "0", "--nodes", "48",
           "--max-plies", "30", "--seed", "5", "--out", str(out)]
    p = subprocess.run(cmd, cwd=ROOT, capture_output=True, text=True, timeout=600)
    assert p.returncode == 0, p.stderr[-3000:]
    lines = p.stdout.strip().splitlines()
    assert lines[-3] == "Arena summary" and lines[-1] in ("replace", "keep")
    assert lines[-2].startswith("Score of Contender vs Producer: CrazyAra-B200-risev2_1-CrazyAra-B200-risev2_0: ")
    w, d, l = (int(x) for x in lines[-2].split(": ")[2].split(" [")[0].split(" - "))
    assert w + d + l == n
    rows = (out / "arena_results.csv").read_text().splitlines()
    assert rows == [f"CrazyAra-B200-risev2_1,CrazyAra-B200-risev2_0,{w},{d},{l}"]
    pgn = (out / "arena_games_gpu_0.pgn").read_text()
    assert pgn.count("[Event ") == n
    assert pgn.count('[White "CrazyAra-B200-risev2_1"]') == 2 and pgn.count('[Black "CrazyAra-B200-risev2_1"]') == 1
