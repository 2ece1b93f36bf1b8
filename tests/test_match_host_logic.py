"""The match's HOST logic (crazyara_b200/match.py: game pairs, start positions, which trees each player's handle
searches, tree-reuse calls, W / D / L, PGN, the launcher's sharding) with the device search replaced by a stand-in
agent that records its calls, and TournamentResult against the reference's (the real search under the same match is
tests/test_match_gpu.py)."""
import argparse
import json
import os
import struct

import numpy as np
import pytest

import crazyara_b200.match as mt
import crazyara_b200.selfplay as sp
from crazyara_b200.engine import BoardState
from crazyara_b200.export import BLACK_WIN, WHITE_WIN

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "tournament.json")

# Fool's mate both ways: whichever colour the contender has, the producer walks into mate
SCRIPT = {(mt.CONTENDER, 0): ["e2e4", "d2d3", "d1h5"], (mt.PRODUCER, 1): ["f7f6", "g7g5"],
          (mt.PRODUCER, 0): ["f2f3", "g2g4"], (mt.CONTENDER, 1): ["e7e5", "d8h4"]}


class StandInAgent:
    """MCTSAgent's surface as the match uses it.  Its 'search' of tree t: the legal moves, uniform policy, and as best
    move the player's scripted move for the ply if there is one, else a seeded random move."""
    log = []  # (agent index, "apply", tree, move) in call order, over both agents

    def __init__(self, net, settings, device=0, n_trees=1, max_nodes=0):
        self.idx, self.net, self.n_trees = len(StandInAgent.created), net, n_trees
        self.seed, self.max_nodes = int(settings.seed), max_nodes
        self.active, self.states, self.res = [True] * n_trees, [None] * n_trees, [None] * n_trees
        self.gos = []  # the active trees at every go
        self.rng = np.random.default_rng(self.idx)
        StandInAgent.created.append(self)

    def set_active(self, tree, active=True):
        for t in range(self.n_trees) if tree < 0 else [tree]:
            self.active[t] = bool(active)

    def set_position(self, state, tree=0):
        self.states[tree] = state

    def evaluate_board_state(self, state=None):
        act = [t for t in range(self.n_trees) if self.active[t]]
        assert act, "go with every tree idle"
        self.gos.append(act)
        for t in act:
            st = self.states[t]
            moves = [st.action_to_uci(a) for a in st.legal_actions()]
            script = SCRIPT.get((self.net, st.side_to_move()), []) if isinstance(self.net, int) else []
            k = self._ply(st) // 2
            best = moves.index(script[k]) if k < len(script) and script[k] in moves else int(self.rng.integers(len(moves)))
            self.res[t] = dict(moves=moves, policy=np.full(len(moves), 1.0 / len(moves)), best_idx=best,
                               visits=np.zeros(len(moves), np.uint32), nodes=10, nodes_pre_search=0)

    @staticmethod
    def _ply(st):
        return int(st.fen().split()[-1]) * 2 - 2 + st.side_to_move()

    def result(self, tree=0):
        return self.res[tree]

    def apply_move_to_tree(self, move, tree=0):
        StandInAgent.log.append((self.idx, "apply", tree, int(move)))

    def close(self):
        pass


def _match(monkeypatch, producer_net=mt.PRODUCER, contender_net=mt.CONTENDER, **kw):
    StandInAgent.created, StandInAgent.log = [], []
    monkeypatch.setattr(mt, "MCTSAgent", StandInAgent)
    kw.setdefault("variant", 0)
    kw.setdefault("temperature_moves", 0)
    return mt.Match((producer_net, None, "prod"), (contender_net, None, "cont"), **kw)


# ------------------------------------------------------------------------------------------------------ TournamentResult
def _check_against(cases, tmp_path):
    for c in cases:
        r = mt.TournamentResult(c["a"], c["b"], c["w"], c["d"], c["l"])
        assert str(r) == c["text"], c
        assert struct.unpack("<I", struct.pack("<f", r.score()))[0] == c["score_bits"], c
        assert r.verdict() == ("replace" if struct.unpack("<f", struct.pack("<I", c["score_bits"]))[0] > 0.5 else "keep")
        path = tmp_path / "r.csv"
        if path.exists():
            path.unlink()
        r.write_csv(str(path))
        assert path.read_text() == c["csv"]


def test_tournament_result_equals_the_reference_golden(tmp_path):
    """str / score / verdict / CSV line against what the UNMODIFIED reference TournamentResult produced
    (tests/golden/tournament.json, written by tests/golden/gen_tournament_golden.py)."""
    cases = json.load(open(GOLDEN))["cases"]
    assert len(cases) > 400
    texts = {c["text"].rsplit("[", 1)[1] for c in cases}
    assert {"0.12]", "0.38]", "0.62]", "0.88]", "0.5]", "1]", "0]"} <= texts   # ties at two digits, all-draw / win / loss
    _check_against(cases, tmp_path)


def test_tournament_result_equals_the_compiled_reference_live(tmp_path):
    so = os.path.join(ROOT, "oracle", "_ref", "libref_tournament.so")
    if not os.path.exists(so):
        pytest.skip("oracle/_ref not built on this box (no reference sources)")
    from tests.golden.gen_tournament_golden import reference, render
    L = reference()
    rng = np.random.default_rng(3)
    cases = []
    for n in list(range(1, 40)) + [100, 101, 1000, 99999]:
        for _ in range(6):
            w = int(rng.integers(n + 1))
            d = int(rng.integers(n + 1 - w))
            text, bits, line = render(L, "x", "y-z", w, d, n - w - d)
            cases.append(dict(a="x", b="y-z", w=w, d=d, l=n - w - d, text=text, score_bits=bits, csv=line))
    _check_against(cases, tmp_path)


# ------------------------------------------------------------------------------------------------------ the match
def _play(m):
    """runs the match step by step; checks that in every step each handle searched exactly its player's games"""
    steps = 0
    while True:
        movers = {s: m._mover(g) for s, g in enumerate(m.slot) if g is not None}
        before = [len(a.gos) for a in m.agents]
        more = m.step()
        for p, a in enumerate(m.agents):
            new = a.gos[before[p]:]
            want = sorted(s for s, q in movers.items() if q == p)
            assert new == ([want] if want else []), (steps, p)
            # the idle trees of this handle are exactly the slots where the other player moves or no game runs
            assert not more or [t for t in range(a.n_trees) if not a.active[t]] == sorted(set(range(a.n_trees)) - set(want))
        if not more:
            assert not movers and [len(a.gos) for a in m.agents] == before   # nothing searched once all games are done
            return steps
        steps += 1


def test_pairs_share_their_start_with_colours_swapped_and_results_count_for_the_contender(monkeypatch, tmp_path):
    pgn = str(tmp_path / "m.pgn")
    m = _match(monkeypatch, n_games=6, slots=4, pgn_path=pgn)
    _play(m)
    games = sorted(m.finished, key=lambda g: g["game"])
    assert [g["game"] for g in games] == list(range(6))
    assert [g["white"] for g in games] == [mt.CONTENDER, mt.PRODUCER] * 3
    for k in range(3):
        assert games[2 * k]["fen"] == games[2 * k + 1]["fen"] == BoardState().set("", False, 0).fen()
    # the producer is mated in every game: as White (Black wins) and as Black (White wins)
    assert [g["result"] for g in games] == [WHITE_WIN, BLACK_WIN] * 3
    assert [g["plies"] for g in games] == [5, 4] * 3
    r = m.result
    assert (r.wins, r.draws, r.losses) == (6, 0, 0) and r.player_a == "cont" and r.player_b == "prod"
    assert r.verdict() == "replace"
    text = open(pgn).read()
    assert text.count("[Event ") == 6
    assert text.count('[White "cont"]') == 3 and text.count('[White "prod"]') == 3 and text.count('[Black "prod"]') == 3
    assert text.count('[Result "1-0"]') == 3 and text.count('[Result "0-1"]') == 3 and "Qh5#" in text and "Qh4#" in text


def test_losses_draws_and_an_odd_number_of_games(monkeypatch):
    # roles swapped: now the contender walks into mate whatever its colour
    m = _match(monkeypatch, producer_net=mt.CONTENDER, contender_net=mt.PRODUCER, n_games=5, slots=2)
    _play(m)
    assert len(m.finished) == 5 and sorted(g["game"] for g in m.finished) == list(range(5))
    assert (m.result.wins, m.result.draws, m.result.losses) == (0, 0, 5) and m.result.verdict() == "keep"
    assert sum(g["white"] == mt.CONTENDER for g in m.finished) == 3        # games 0, 2, 4: the last pair is incomplete
    m = _match(monkeypatch, n_games=3, max_plies=2)                      # adjudicated draws
    _play(m)
    assert (m.result.wins, m.result.draws, m.result.losses) == (0, 3, 0) and str(m.result) == "cont-prod: 0 - 3 - 0 [0.5]"
    assert m.result.verdict() == "keep"


def test_idle_slots_and_the_end_of_the_match(monkeypatch):
    """More slots than games left: a slot without a game is idle in both handles; the match ends when all are done."""
    m = _match(monkeypatch, n_games=3, slots=3, max_plies=3)
    assert _play(m) == 3 and len(m.finished) == 3
    m = _match(monkeypatch, n_games=4, slots=3, max_plies=3)
    assert _play(m) == 6 and len(m.finished) == 4       # game 3 starts in the first slot free after 3 plies
    assert sorted((g["game"], g["slot"]) for g in m.finished) == [(0, 0), (1, 1), (2, 2), (3, 0)]


def test_tree_reuse_calls_in_the_reference_order(monkeypatch):
    """generate_arena_game (rl/selfplay.cpp:293-299): the mover applies its move, then the other player -- except at a
    game's first ply; a new game in a slot first clears both players' trees (clear_game_history)."""
    m = _match(monkeypatch, n_games=4, slots=2, max_plies=9, reuse_tree=True)
    assert all(a.max_nodes > 0 for a in m.agents)
    _play(m)
    want = {0: [], 1: []}
    for g in sorted(m.finished, key=lambda g: g["game"]):
        seq = want[g["slot"]]
        seq += [(0, 0), (1, 0)]
        st = BoardState().set(g["fen"], False, 0)
        for ply, u in enumerate(g["moves"]):
            a = st.uci_to_action(u)
            mover = g["white"] if ply % 2 == 0 else 1 - g["white"]
            seq.append((mover, a))
            if ply > 0:
                seq.append((1 - mover, a))
            st.do_uci(u)
    got = {0: [], 1: []}
    for idx, _, tree, move in StandInAgent.log:
        got[tree].append((idx, move))
    assert got == want
    m = _match(monkeypatch, n_games=2, max_plies=4)
    _play(m)
    assert StandInAgent.log == []                           # reuse_tree off (rl_config.py:56): no calls at all


def test_start_positions_from_an_epd_file_and_chess960(monkeypatch, tmp_path):
    fens = ["rnbqkbnr/pppppppp/8/8/4P3/8/PPPP1PPP/RNBQKBNR b KQkq - 0 1", "r1bqkbnr/pppppppp/2n5/8/4P3/8/PPPP1PPP/RNBQKBNR w KQkq - 1 2",
            "rnbqkbnr/pp1ppppp/8/2p5/4P3/8/PPPP1PPP/RNBQKBNR w KQkq - 0 2"]
    epd = tmp_path / "openings.epd"
    epd.write_text(fens[0] + ";\n" + fens[1] + "\n" + fens[2] + ";\n")
    assert sp.load_random_fen(None, None) == sp.load_random_fen("", None) == sp.load_random_fen("<empty>", None) == ""
    rng = np.random.default_rng(0)
    drawn = [sp.load_random_fen(str(epd), rng) for _ in range(300)]
    assert set(drawn) == set(fens) and min(drawn.count(f) for f in fens) > 70           # uniform, ';' dropped
    m = _match(monkeypatch, n_games=10, slots=10, max_plies=3, epd_path=str(epd))
    _play(m)
    games = sorted(m.finished, key=lambda g: g["game"])
    for k in range(5):
        assert games[2 * k]["fen"] == games[2 * k + 1]["fen"] and games[2 * k]["fen"] in fens
    assert len({g["fen"] for g in games}) > 1
    m = _match(monkeypatch, n_games=12, slots=4, max_plies=2, is960=True)
    _play(m)
    games = sorted(m.finished, key=lambda g: g["game"])
    for k in range(6):
        assert games[2 * k]["fen"] == games[2 * k + 1]["fen"]
    assert len({g["fen"] for g in games}) >= 4                               # a new set-up per pair


def test_self_play_arena_epd_start_positions(monkeypatch, tmp_path):
    from tests.test_arena_host_logic import FakeAgent
    epd = tmp_path / "o.epd"
    fen = "rnbqkbnr/pppppppp/8/8/3P4/8/PPP1PPPP/RNBQKBNR b KQkq - 0 1"
    epd.write_text(fen + ";\n")
    FakeAgent.created = []
    monkeypatch.setattr(sp, "MCTSAgent", FakeAgent)
    arena = sp.Arena(None, sp.rl_settings("chess"), variant=0, n_games=2, temperature_moves=0, max_plies=4, seed=1,
                     resign_probability=0.0, epd_path=str(epd))
    assert [s.fen() for s in arena.states] == [fen, fen]
    arena.run(max_steps=4)                          # both games adjudicated at 4 plies and started again
    assert len(arena.finished) == 2 and [s.fen() for s in arena.states] == [fen, fen]


def test_players_seeds_names_and_default_settings(monkeypatch):
    m = _match(monkeypatch, n_games=2, seed=3)
    a, b = StandInAgent.created
    assert a.seed != b.seed and a.n_trees == b.n_trees == 2
    m2 = _match(monkeypatch, n_games=2, seed=4)
    assert StandInAgent.created[0].seed != a.seed
    assert not m.shared_net
    net = object()
    assert _match(monkeypatch, producer_net=net, contender_net=net, n_games=2).shared_net   # one network: searched in turn
    del m, m2
    assert mt.player_name("/x/y/model-0042.arab") == "CrazyAra-B200-model-0042" and mt.player_name(None) == "fake"


def test_worker_shards_pairs_and_writes_pgn(monkeypatch, tmp_path):
    """python -m crazyara_b200.match: the launcher's plan and one worker's whole run, device pieces replaced."""
    import crazyara_b200.nn as nn_mod
    plan = mt.plan_workers(7, [0, 1], str(tmp_path))
    assert [(j["n_games"], j["seed_offset"]) for j in plan] == [(4, 0), (3, 2)]        # pairs stay on one GPU
    assert [j["n_games"] for j in mt.plan_workers(100, [0, 1, 2], ".")] == [34, 34, 32]
    assert [j["n_games"] for j in mt.plan_workers(1, [0, 1], ".")] == [1]

    class FakeNet:
        def __init__(self, ctx, device, batch, path):
            self.batch, self.path = batch, path

        def close(self):
            pass

    StandInAgent.created, StandInAgent.log = [], []
    monkeypatch.setattr(mt, "MCTSAgent", StandInAgent)
    monkeypatch.setattr(nn_mod, "NeuralNetAPI", FakeNet)
    args = argparse.Namespace(producer="nets/old.arab", contender="nets/new.arab", mode="crazyhouse", variant=1, chess960=False,
                              input_version=1, batch_size=8, nodes=800, max_plies=6, seed=1, epd=None, temperature=0.6,
                              reuse_tree=False)

    class Queue(list):
        put = list.append
    q = Queue()
    mt._worker(plan[1], args, q)
    assert len(q) == 1 and sum(q[0]) == 3
    assert [a.net.batch for a in StandInAgent.created] == [3 * 8, 3 * 8] and StandInAgent.created[1].net.path == "nets/new.arab"
    text = open(plan[1]["pgn"]).read()
    assert text.count("[Event ") == 3 and '[White "CrazyAra-B200-new"]' in text and '[Black "CrazyAra-B200-old"]' in text
