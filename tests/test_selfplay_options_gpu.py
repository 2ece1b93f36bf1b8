"""Per-tree search settings (ara_search_set_tree_settings), quick searches and raw-network openings of the self-play arena,
and RawNetAgent, on the GPU with the synthetic RISEv2 network."""
import os
import subprocess

import numpy as np
import pytest

from tests.test_search_hostemu import assert_same_search

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LINES = [[], ["e2e4"], ["d2d4", "g8f6", "c2c4"], ["g1f3", "d7d5"]]
# (Q-value weight, Dirichlet epsilon) per tree; negative = the handle's value
TREES = [(-1.0, -1.0), (0.0, 0.25), (0.7, 0.0), (2.0, 0.1)]
GOLDEN = 0x9E3779B97F4A7C15


def _blob(tmp_path):
    from crazyara_b200.weights import export_blob
    from oracle import net as onet
    arch = onet.arch_risev2(34, 81)
    return export_blob(onet.make_state_dict(arch, 0), arch, str(tmp_path / "risev2.arab"), input_version=10)


def _state(t):
    from crazyara_b200.engine import BoardState
    return BoardState().set("", False, 1).do_uci(*LINES[t % len(LINES)])


@pytest.mark.gpu
@pytest.mark.parametrize("threads", [1, 2])
@pytest.mark.parametrize("wave", [0, 1])         # select_kernel (one warp per tree) / select_wave_kernel
@pytest.mark.parametrize("batch", [8, 64])
def test_per_tree_settings_equal_single_tree_searches(tmp_path, monkeypatch, batch, wave, threads):
    """Each tree of a handle with per-tree values searches exactly like a one-tree handle whose settings carry those
    values (and whose Dirichlet generator starts where the tree's does: seed ^ tree * golden ratio)."""
    from crazyara_b200.engine import MCTSAgent, default_settings
    from crazyara_b200.nn import NeuralNetAPI
    monkeypatch.setenv("ARA_WAVE", str(wave))
    base = dict(batch_size=batch, simulations=300, node_policy_temperature=1.0, dirichlet_epsilon=0.25, dirichlet_alpha=0.3,
                seed=7, threads=threads, q_value_weight=1.0)
    net = NeuralNetAPI("gpu", 0, len(TREES) * batch, _blob(tmp_path))
    mixed = MCTSAgent(net, default_settings("crazyhouse", **base), 0, len(TREES))
    for t, (q, eps) in enumerate(TREES):
        mixed.set_position(_state(t), t)
        if q >= 0 or eps >= 0:
            mixed.set_tree_settings(q, eps, t)
    mixed.evaluate_board_state()
    results = mixed.results()
    for t, (q, eps) in enumerate(TREES):
        own = dict(base, seed=(7 ^ (t * GOLDEN)) & (2**64 - 1), q_value_weight=q if q >= 0 else base["q_value_weight"],
                   dirichlet_epsilon=eps if eps >= 0 else base["dirichlet_epsilon"])
        single = MCTSAgent(net, default_settings("crazyhouse", **own), 0, 1)
        r = single.evaluate_board_state(_state(t))
        assert_same_search(r, results[t])
        assert r["pv"] == results[t]["pv"] and r["evals"] > 0
        single.close()
    # the values last until they are changed: back to the handle's settings, tree 1 searches like tree 0's settings say
    mixed.set_tree_settings(-1.0, -1.0)
    mixed.evaluate_board_state()
    plain = MCTSAgent(net, default_settings("crazyhouse", **dict(base, seed=(7 ^ GOLDEN) & (2**64 - 1))), 0, 1)
    plain.evaluate_board_state(_state(1))   # (its generator's first draw: tree 1 of `mixed` has drawn once already)
    again = plain.evaluate_board_state(_state(1))
    assert_same_search(again, mixed.result(1))
    plain.close()
    mixed.close()
    net.close()


@pytest.mark.gpu
def test_tree_settings_are_range_checked():
    from crazyara_b200 import AraError
    from crazyara_b200.engine import MCTSAgent, default_settings
    a = MCTSAgent(None, default_settings("crazyhouse", batch_size=8, simulations=50), 0, 2)
    for args in ((0.5, 0.1, 2), (0.5, 0.1, -2), (0.5, 1.5, 0), (float("nan"), 0.1, 0), (1e4, 0.1, 0), (0.5, float("inf"), 1)):
        with pytest.raises(AraError):
            a.set_tree_settings(*args)
    a.set_tree_settings(0.5, 1.0, -1)
    a.close()


@pytest.mark.gpu
def test_arena_with_quick_searches_and_raw_openings(tmp_path):
    from crazyara_b200.export import TrainDataExporter, read_dataset
    from crazyara_b200.nn import NeuralNetAPI
    from crazyara_b200.selfplay import Arena, rl_settings
    n_games, B = 8, 8
    net = NeuralNetAPI("gpu", 0, n_games * B, _blob(tmp_path))
    ex = TrainDataExporter(str(tmp_path / "d.zarr"), "crazyhouse", channels=34, number_chunks=40, chunk_size=16)
    pgn = str(tmp_path / "games.pgn")
    st = rl_settings("crazyhouse", batch_size=B, nodes=60, simulations=240)
    arena = Arena(net, st, variant=1, n_games=n_games, max_plies=40, seed=3, exporter=ex, pgn_path=pgn, quick_probability=0.5,
                  quick_nodes=20, mean_init_ply=4, max_init_ply=8, raw_prob_temperature=0.25)
    opening = list(arena.plies)
    assert sum(opening) > 0 and all(p <= 8 for p in opening)
    res = arena.run(min_games=n_games, max_steps=120)
    arena.close()
    assert res["games"] >= n_games and res["nodes"] > 0
    starts = read_dataset(str(tmp_path / "d.zarr"), "start_indices")
    n = starts[ex.game_idx]
    # quick searches export nothing: fewer samples than searched moves of the finished games, but some
    searched = sum(p for p, _, _ in arena.finished)
    assert ex.game_idx == res["games"] and 0 < n < searched
    pol = read_dataset(str(tmp_path / "d.zarr"), "y_policy")[:n]
    assert np.allclose(pol.sum(axis=1), 1.0, atol=1e-5)
    text = open(pgn).read()
    blocks = text.strip().split("\n\n\n")
    assert len(blocks) == res["games"]
    for block, (plies, _, _) in zip(blocks, arena.finished):
        header, body = block.split("\n\n", 1)
        assert f'[PlyCount "{plies}"]' in header
        tokens = [t for t in body.split() if not t.endswith(".")]
        assert len(tokens) == plies + 1 and tokens[-1] in ("1-0", "0-1", "1/2-1/2")
    net.close()


def _raw_reference(net, state):
    """argmax of the legal moves' entries of the whole soft-maxed policy (NeuralNetAPI.predict)"""
    from crazyara_b200.engine import encode_planes, legal_moves_gpu
    moves, _, pidx = legal_moves_gpu([state.board()])
    x = np.zeros((net.get_batch_size(), 34, 8, 8), np.float32)
    x[0] = encode_planes([state.board()], 0, 1)[0]
    v = np.zeros(net.get_batch_size(), np.float32)
    p = np.zeros((net.get_batch_size(), net.get_nb_policy_values()), np.float32)
    net.predict(x, v, p, None, n=1)
    pri = p[0, pidx[0]]
    return state.action_to_uci(moves[0][int(np.argmax(pri))]), pri


@pytest.mark.gpu
def test_raw_net_agent_and_uci(tmp_path):
    from crazyara_b200.engine import RawNetAgent
    from crazyara_b200.nn import NeuralNetAPI
    blob = _blob(tmp_path)
    net = NeuralNetAPI("gpu", 0, 8, blob)
    agent = RawNetAgent(net, 0, 1)
    want = {}
    for t in range(len(LINES)):
        st = _state(t)
        r = agent.evaluate_board_state(st)
        move, pri = _raw_reference(net, st)
        assert r["best_move"] == move and r["depth"] == r["seldepth"] == r["nodes"] == 1
        np.testing.assert_allclose(r["policy"], pri, rtol=1e-6, atol=1e-7)
        want[t] = move
    # several states in one forward give what one state at a time gives
    many = agent.predict([_state(t) for t in range(len(LINES))])
    for t, (codes, priors, _) in enumerate(many):
        assert _state(t).action_to_uci(codes[int(np.argmax(priors))]) == want[t]
    net.close()
    exe = os.path.join(ROOT, "crazyara_b200", "ara_uci")
    if not os.path.exists(exe):
        subprocess.run(["make", "-C", ROOT, "crazyara_b200/ara_uci"], check=True)
    cmds = ["uci", f"setoption name Model_Path value {blob}", "setoption name Batch_Size value 8",
            "setoption name Use_Raw_Network value true", "isready"]
    for t in range(len(LINES)):
        cmds += ["position startpos" + (" moves " + " ".join(LINES[t]) if LINES[t] else ""), "go nodes 800"]
    out = subprocess.run([exe], input="\n".join(cmds + ["quit"]) + "\n", capture_output=True, text=True, timeout=300).stdout
    best = [line.split()[1] for line in out.splitlines() if line.startswith("bestmove")]
    assert best == [want[t] for t in range(len(LINES))], out
