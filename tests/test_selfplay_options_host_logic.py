"""Quick searches and raw-network openings of the self-play arena (SelfPlay::generate_game, rl/selfplay.cpp:154-241,
:423-487) and Use_Raw_Network of the UCI front-end, on a box without a GPU: the arena runs with the search stand-in of
tests/test_arena_host_logic.py and a scripted priors source in place of RawNetAgent; the UCI binary runs with the
search and network entry points replaced (tests/uci_stub)."""
import os
import subprocess

import numpy as np
import pytest

import crazyara_b200.selfplay as sp
from crazyara_b200.engine import BoardState
from crazyara_b200.export import TrainDataExporter, read_dataset
from tests.test_arena_host_logic import FakeAgent


class QuickAgent(FakeAgent):
    """FakeAgent that also takes per-tree settings; every call is logged with the number of the go it precedes"""

    def __init__(self, *a, **kw):
        super().__init__(*a, **kw)
        self.go, self.log = 0, []

    def set_search_limits(self, simulations, nodes, tree=-1):
        super().set_search_limits(simulations, nodes, tree)
        self.log.append((self.go, tree, "limits", nodes))

    def set_tree_settings(self, q_value_weight=-1.0, dirichlet_epsilon=-1.0, tree=-1):
        self.log.append((self.go, tree, "settings", (q_value_weight, dirichlet_epsilon)))

    def evaluate_board_state(self, state=None):
        super().evaluate_board_state(state)
        self.log += [(self.go, t, "moves", len(r["moves"])) for t, r in enumerate(self.res)]
        self.go += 1


def _arena(monkeypatch, tmp_path, **kw):
    FakeAgent.created = []
    monkeypatch.setattr(sp, "MCTSAgent", QuickAgent)
    monkeypatch.setattr(sp, "encode_planes", lambda boards, mode, version, normalize=False: np.ones((len(boards), 34, 8, 8), np.float32))
    ex = TrainDataExporter(str(tmp_path / "d.zarr"), "crazyhouse", channels=34, number_chunks=40, chunk_size=16)
    saved = []
    save = ex.save_sample
    ex.save_sample = lambda *a: (saved.append(1), save(*a))
    arena = sp.Arena(None, sp.rl_settings("crazyhouse"), variant=1, n_games=kw.pop("n_games", 4), temperature_moves=0,
                     max_plies=kw.pop("max_plies", 30), seed=kw.pop("seed", 4), exporter=ex, **kw)
    return arena, ex, saved


def _searches(agent):
    """per (go, tree): limits, settings, number of legal moves"""
    out = {}
    for go, tree, kind, v in agent.log:
        out.setdefault((go, tree), {})[kind] = v
    return out


def test_every_search_quick(monkeypatch, tmp_path):
    arena, ex, saved = _arena(monkeypatch, tmp_path, quick_probability=1.0)
    res = arena.run(min_games=4, max_steps=200)
    assert res["games"] >= 4
    searches = _searches(FakeAgent.created[0])
    assert len(searches) == res["moves"]
    for (go, tree), s in searches.items():
        # Quick_Nodes 100 with the node jitter of adjust_node_count on top: 100 +- 5 %
        assert 95 <= s["limits"] <= 104 and s["settings"] == (0.7, 0.0), (go, tree, s)
    assert len({s["limits"] for s in searches.values()}) > 3
    assert saved == [] and read_dataset(str(tmp_path / "d.zarr"), "start_indices")[ex.game_idx] == 0


def test_quick_probability_zero_is_the_plain_arena(monkeypatch, tmp_path):
    runs = []
    for kw in ({}, dict(quick_probability=0.0), dict(quick_probability=0.005, quick_nodes=10)):   # below 0.01: off
        arena, ex, saved = _arena(monkeypatch, tmp_path / str(len(runs)), **kw)
        res = arena.run(min_games=4, max_steps=100)
        log = FakeAgent.created[0].log
        assert not [c for c in log if c[2] == "settings"]
        runs.append((res["moves"], arena.finished, [s.fen() for s in arena.states], [c for c in log if c[2] == "limits"], len(saved)))
    assert runs[0] == runs[1] == runs[2]
    assert all(760 <= c[3] <= 840 for c in runs[0][3])


def test_quick_searches_mixed_go_to_the_drawn_trees_and_are_undone(monkeypatch, tmp_path):
    arena, ex, saved = _arena(monkeypatch, tmp_path, quick_probability=0.5, quick_nodes=200, quick_q_value_weight=0.5,
                              quick_dirichlet_epsilon=0.1, n_games=6)
    res = arena.run(max_steps=40)
    searches = _searches(FakeAgent.created[0])
    quick_before, n_quick, n_restored, n_samples = {}, 0, 0, 0
    for (go, tree) in sorted(searches):
        s = searches[go, tree]
        quick = s.get("settings") == (0.5, 0.1)
        if quick:
            n_quick += 1
            assert 190 <= s["limits"] <= 209
        else:
            assert 760 <= s["limits"] <= 840
            if quick_before.get(tree):   # reset_search_params: the handle's values come back
                assert s["settings"] == (-1.0, -1.0)
                n_restored += 1
            else:
                assert "settings" not in s
            n_samples += s["moves"] > 0
        quick_before[tree] = quick
    assert 0.35 < n_quick / len(searches) < 0.65 and n_restored > 0 and res["moves"] == len(searches)
    assert len(saved) == n_samples


def test_init_ply_count_and_clipping():
    mean, cap = 4, 12
    rng, again = np.random.default_rng(1), np.random.default_rng(1)
    plies = []
    for _ in range(2000):
        p = sp.init_ply_count(rng, mean, cap)
        want = int(again.exponential(mean) + 0.5)
        if want > cap:
            want = int(again.integers(0, 1 << 31)) % cap
        assert p == want
        plies.append(p)
    assert max(plies) <= cap and sum(p == cap for p in plies) > 0
    # unclipped, the rounded exponential keeps the mean
    assert abs(np.mean([sp.init_ply_count(rng, mean, 1000) for _ in range(4000)]) - mean) < 0.3
    assert sp.init_ply_count(rng, 50, 3) in (0, 1, 2, 3)
    state = rng.bit_generator.state
    assert sp.init_ply_count(rng, 0, 30) == 0 and rng.bit_generator.state == state   # off: no draw


class _Draws:
    def __init__(self, values):
        self.values = list(values)

    def random(self):
        return self.values.pop(0)


def test_raw_policy_temperature_thresholds():
    p = np.array([0.7, 0.2, 0.1])

    def flat(t):
        q = p ** (1 / t)
        return q / q.sum()
    assert np.allclose(sp.apply_raw_policy_temp(p, 0.25, _Draws([0.1, 0.04])), flat(10))
    assert np.allclose(sp.apply_raw_policy_temp(p, 0.25, _Draws([0.1, 0.05])), flat(5))
    assert np.allclose(sp.apply_raw_policy_temp(p, 0.25, _Draws([0.1, 0.24])), flat(5))
    assert np.allclose(sp.apply_raw_policy_temp(p, 0.25, _Draws([0.1, 0.25])), flat(2))
    assert np.allclose(sp.apply_raw_policy_temp(p, 0.25, _Draws([0.25])), p)          # not drawn: unchanged
    assert np.allclose(sp.apply_raw_policy_temp(p, 0.0, _Draws([0.0])), p)


class ScriptedRaw:
    """RawNetAgent's predict with scripted priors: all the mass on the legal move `pick(state, moves)` chooses"""
    created = []

    def __init__(self, net, mode, input_version):
        self.calls = []
        ScriptedRaw.created.append(self)

    pick = staticmethod(lambda st, moves: 0)

    def predict(self, states):
        self.calls.append(len(states))
        out = []
        for st in states:
            moves = st.legal_actions()
            p = np.full(len(moves), 1e-9, np.float32)
            p[ScriptedRaw.pick(st, moves)] = 1.0
            out.append((moves, p, 0.0))
        return out


def _opening_arena(monkeypatch, tmp_path, pick, epd=None, **kw):
    FakeAgent.created, ScriptedRaw.created = [], []
    monkeypatch.setattr(sp, "MCTSAgent", QuickAgent)
    monkeypatch.setattr(sp, "RawNetAgent", ScriptedRaw)
    monkeypatch.setattr(ScriptedRaw, "pick", staticmethod(pick))
    return sp.Arena(None, sp.rl_settings("chess"), variant=0, n_games=kw.pop("n_games", 5), temperature_moves=0, max_plies=60,
                    seed=kw.pop("seed", 8), pgn_path=str(tmp_path / "games.pgn"), epd_path=epd, **kw)


def test_raw_openings_play_the_drawn_plies_in_lock_step(monkeypatch, tmp_path):
    mean, cap = 6, 10
    arena = _opening_arena(monkeypatch, tmp_path, lambda st, moves: len(moves) - 1, mean_init_ply=mean, max_init_ply=cap)
    # the ply counts the games drew, replayed from the arena's seed (a chess game without an EPD file draws no FEN)
    rng = np.random.default_rng(8)
    want = [sp.init_ply_count(rng, mean, cap) for _ in range(5)]
    assert arena.plies == want and max(want) > 0
    raw = ScriptedRaw.created[0]
    # one forward per ply over the games that still have plies to play
    assert raw.calls == [sum(w > k for w in want) for k in range(max(want))]
    for t, st in enumerate(arena.states):
        replay = BoardState().set("", False, 0)
        sans = []
        for _ in range(want[t]):
            moves = replay.legal_actions()
            sans.append(replay.action_to_san(moves[-1]))
            replay.do_action(moves[-1])
        assert st.fen() == replay.fen()
        assert arena.pgns[t].game_moves == sans and arena.pgns[t].fen == BoardState().set("", False, 0).fen()
    arena.run(min_games=2, max_steps=80)
    blocks = open(tmp_path / "games.pgn").read().strip().split("\n\n\n")
    assert len(blocks) == len(arena.finished) >= 2
    for block, (plies, _, _) in zip(blocks, arena.finished):
        assert f'[PlyCount "{plies}"]' in block   # the opening's plies are moves of the game


def test_raw_opening_stops_before_a_move_that_ends_the_game(monkeypatch, tmp_path):
    # 1. f3 e5 2. g4: black to move can mate (Qh4#); the scripted policy wants that move first, then any other
    fen = "rnbqkbnr/pppp1ppp/8/4p3/6P1/5P2/PPPPP2P/RNBQKBNR b KQkq - 0 2"
    epd = tmp_path / "mate.epd"
    epd.write_text(fen + ";\n")

    def pick(st, moves):
        ucis = [st.action_to_uci(m) for m in moves]
        return ucis.index("d8h4") if "d8h4" in ucis else 0
    arena = _opening_arena(monkeypatch, tmp_path, pick, epd=str(epd), n_games=2, mean_init_ply=50, max_init_ply=40)
    for t in range(2):
        assert arena.plies[t] == 0 and arena.states[t].fen() == fen and arena.pgns[t].game_moves == []
        assert arena.pgns[t].fen == fen and arena.init_plies[t] == 0
    assert ScriptedRaw.created[0].calls == [2]


def test_raw_openings_need_a_ply_cap(monkeypatch, tmp_path):
    with pytest.raises(ValueError):
        _opening_arena(monkeypatch, tmp_path, lambda st, moves: 0, mean_init_ply=4)


def test_launcher_flags_reach_the_arena(monkeypatch):
    seen = {}
    monkeypatch.setattr(sp, "_worker", lambda job, args: seen.update(vars(args)))
    monkeypatch.setattr(sp, "plan_workers", lambda total, devices, out: [dict(rank=0)])

    class _Proc:
        exitcode = 0

        def __init__(self, target, args):
            self.target, self.args = target, args

        def start(self):
            self.target(*self.args)

        def join(self):
            pass

    class _Ctx:
        Process = _Proc
    import multiprocessing as mp
    monkeypatch.setattr(mp, "get_context", lambda name: _Ctx)
    assert sp.main(["m.arab", "--quick-probability", "0.5", "--quick-nodes", "60", "--mean-init-ply", "4", "--max-init-ply", "12",
                    "--raw-prob-temperature", "0.25"]) == 0
    assert seen["quick_probability"] == 0.5 and seen["quick_nodes"] == 60 and seen["quick_q_value_weight"] == 0.7
    assert seen["mean_init_ply"] == 4 and seen["max_init_ply"] == 12 and seen["raw_prob_temperature"] == 0.25


# ---------------------------------------------------------------------------------------------------------- UCI
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXE = os.path.join(ROOT, "crazyara_b200", "ara_uci")
STUB_DIR = os.path.join(ROOT, "tests", "uci_stub")


@pytest.fixture(scope="module")
def uci_env(tmp_path_factory):
    if not os.path.exists(EXE):
        subprocess.run(["make", "-C", ROOT, "crazyara_b200/ara_uci"], check=True)
    d = tmp_path_factory.mktemp("uci_stub")
    search, net = str(d / "libstub_search.so"), str(d / "libstub_net.so")
    subprocess.run(["gcc", "-O1", "-shared", "-fPIC", "-Wall", "-I" + os.path.join(ROOT, "include"),
                    os.path.join(STUB_DIR, "stub_search.c"), "-o", search], check=True)
    subprocess.run(["g++", "-O1", "-std=c++17", "-shared", "-fPIC", "-Wall", "-I" + os.path.join(ROOT, "include"),
                    "-I" + os.path.join(ROOT, "crazyara_b200", "csrc"), "-x", "c++", os.path.join(STUB_DIR, "stub_net.cpp"),
                    "-o", net], check=True)
    e = dict(os.environ)
    e["LD_PRELOAD"] = search + ":" + net
    return e


def _session(env, tmp_path, commands):
    log = tmp_path / "calls.log"
    if log.exists():
        log.unlink()
    e = dict(env, ARA_STUB_LOG=str(log))
    out = subprocess.run([EXE], input="\n".join(commands + ["quit"]) + "\n", capture_output=True, text=True, timeout=60, env=e).stdout
    return out.splitlines(), (log.read_text().splitlines() if log.exists() else [])


def _raw_move(fen):
    """the stand-in network's choice: the legal move with the largest policy index (host emulation of the rules)"""
    from tests.hostemu import HeState
    he = HeState(fen, 0, False)
    moves = he.legal_moves()
    return he.uci(max(moves, key=he.policy_index))


def test_uci_use_raw_network_answers_go_with_the_raw_move(uci_env, tmp_path):
    head = ["setoption name UCI_Variant value chess", "setoption name Model_Path value net.arab",
            "setoption name Use_Raw_Network value true", "isready"]
    lines, calls = _session(uci_env, tmp_path, head + ["position startpos moves e2e4", "go nodes 800",
                                                       "position startpos moves e2e4 e7e5", "go movetime 50"])
    e4 = "rnbqkbnr/pppppppp/8/8/4P3/8/PPPP1PPP/RNBQKBNR b KQkq - 0 1"
    e4e5 = "rnbqkbnr/pppp1ppp/8/4p3/4P3/8/PPPP1PPP/RNBQKBNR w KQkq - 0 2"
    assert [l for l in lines if l.startswith("bestmove")] == ["bestmove " + _raw_move(e4), "bestmove " + _raw_move(e4e5)]
    info = [l for l in lines if l.startswith("info depth")]
    assert len(info) == 2 and all(l.startswith("info depth 1 nodes 1 ") for l in info)
    # value 0.5 -> -log(0.5) / log(1.4) * 100 (value_to_centipawn, MODE_CHESS)
    assert all(" score cp 206 " in l for l in info)
    # one forward per go; no search ran and no move was announced to a tree
    from tests.hostemu import HeState
    assert calls == [f"predict_priors n=1 count={len(HeState(f, 0).legal_moves())}" for f in (e4, e4e5)]
    # a single legal move is answered without a forward
    lines, calls = _session(uci_env, tmp_path, head + ["position fen k7/8/8/8/8/8/6q1/7K w - - 0 1", "go"])
    assert [l for l in lines if l.startswith("bestmove")] == ["bestmove h1g2"] and calls == []
    assert [l for l in lines if l.startswith("info depth")][0].startswith("info depth 0 nodes 0 ")


def test_uci_use_raw_network_needs_a_network_and_is_off_by_default(uci_env, tmp_path):
    lines, calls = _session(uci_env, tmp_path, ["setoption name UCI_Variant value chess", "setoption name Use_Raw_Network value true",
                                                "isready", "position startpos", "go nodes 100"])
    assert any("Use_Raw_Network needs a network" in l for l in lines) and not any(l.startswith("bestmove") for l in lines)
    lines, calls = _session(uci_env, tmp_path, ["setoption name UCI_Variant value chess", "setoption name Model_Path value net.arab",
                                                "isready", "position startpos", "go movetime 60"])
    assert [c for c in calls if c.startswith("go ")] == ["go movetime=40"] and not [c for c in calls if c.startswith("predict")]
    assert [l for l in lines if l.startswith("bestmove")] == ["bestmove e2e4"]
