"""Node and edge pools that grow with the tree: a single tree without a visit budget reserves its pools and maps them as
the search needs them (ara_search_create, ara_search_pool).  Every handle here is capped at a few hundred thousand
nodes (explicit max_nodes) so that no test maps more than a few GB of a shared GPU; the one handle without a cap only
reads its reservation."""
import os
import time

import numpy as np
import pytest

from oracle import search as osr
from oracle.chess import Position
from tests.test_search_hostemu import assert_same_search

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GRAN = 2 << 20  # the H100's mapping granularity for device memory (cuMemGetAllocationGranularity, minimum)
NODE_BYTES, EDGE_BYTES = 64 + 128 + 2 * (128 + 2 + 1), 4 * 5 + 2 + 1 + 1  # TreeDev's arrays per node / per edge


def _settings(mode, **kw):
    from crazyara_b200.engine import SearchSettings
    st = osr.default_settings(mode, **kw)
    s = SearchSettings()
    for f, _ in s._fields_:
        setattr(s, f, getattr(st, f))
    return st, s


def _growing(net, s, cap):
    """a handle whose pools grow with the tree: the settings' budget moved to ara_search_set_limits"""
    from crazyara_b200.engine import MCTSAgent
    sims, nodes = int(s.simulations), int(s.nodes)
    s.simulations, s.nodes = 0, 0
    agent = MCTSAgent(net, s, 0, 1, cap)
    s.simulations, s.nodes = sims, nodes
    if sims or nodes:
        agent.set_search_limits(sims, nodes)
    return agent


def _stepped(agent, state):
    """the search one mini-batch at a time (ara_search_begin / ara_search_step(1)): the pools are grown between steps"""
    agent.begin(state)
    steps = 0
    while agent.thread_iteration(1) > 0:
        steps += 1
        assert steps < 100000
    return agent.result(0)


def _net(tmp_path, batch):
    from crazyara_b200.nn import NeuralNetAPI
    from crazyara_b200.weights import export_blob
    from oracle import net as onet
    arch = onet.arch_risev2(34, 81)
    blob = export_blob(onet.make_state_dict(arch, 0), arch, str(tmp_path / "risev2.arab"), input_version=10)
    return NeuralNetAPI("gpu", 0, batch, blob, precision="float16")


# (network, Threads, epsilon exploration): the wavefront select (B >= 8, no epsilon) and select_kernel<true>
GROW_CASES = [("fake", 1, False), ("fake", 2, False), ("fake", 2, True), ("risev2", 1, False), ("risev2", 2, False)]


@pytest.mark.gpu
@pytest.mark.parametrize("backend,threads,eps", GROW_CASES)
def test_growth_mid_search_keeps_the_bits(tmp_path, backend, threads, eps):
    from crazyara_b200.engine import BoardState, MCTSAgent
    B, sims = 16, 24000
    extra = dict(epsilon_greedy_counter=20, epsilon_checks_counter=100) if eps else {}
    _, s = _settings("crazyhouse", batch_size=B, simulations=sims, node_policy_temperature=1.7, threads=threads, **extra)
    net = _net(tmp_path, B) if backend != "fake" else None
    state = BoardState().set("", False, 1).do_uci("e2e4")
    fixed = MCTSAgent(net, s, 0, 1, 2 * sims)  # (room past the budget: a pool sized for it can fill first with epsilon on)
    rf = _stepped(fixed, state)
    pf = fixed.pool()
    fixed.close()
    grow = _growing(net, s, 1 << 20)
    p0 = grow.pool()
    assert p0["growing"] == 1 and p0["mapped_nodes"] < sims // 2 and p0["cap_nodes"] == 1 << 20
    rg = _stepped(grow, state)
    p1 = grow.pool()
    grow.close()
    if net is not None:
        net.close()
    assert pf["growing"] == 0 and rf["error"] == 0 and rg["error"] == 0
    assert p1["grows"] - p0["grows"] >= 2 and p1["nodes"] > p0["mapped_nodes"]
    assert p1["mapped_nodes"] >= p1["nodes"] and p1["mapped_edges"] >= p1["edges"]
    assert_same_search(rf, rg)
    assert rf["tree_nodes"] == rg["tree_nodes"] and rf["iterations"] == rg["iterations"] and rf["evals"] == rg["evals"]


@pytest.mark.gpu
@pytest.mark.parametrize("threads", [1, 2])
def test_growing_pools_equal_the_oracle(threads):
    from crazyara_b200.engine import BoardState
    st, s = _settings("crazyhouse", batch_size=16, simulations=1500, node_policy_temperature=1.0, threads=threads)
    pos = Position(None, "crazyhouse", False)
    pos.push_uci("e2e4")
    S = osr.Search(st)
    ro = S.run(pos, osr.fake_net(S.n_labels), with_keys=True, threads=threads)
    agent = _growing(None, s, 200000)
    rg = _stepped(agent, BoardState().set("", False, 1).do_uci("e2e4"))
    agent.close()
    assert_same_search(ro, rg)


def _timed_rate(s, cap, vid, ms=200.0):
    """nodes per ms of a short timed search of the fake backend (the settings the timed tests use; the faster of two, the
    first may load the kernels)"""
    from crazyara_b200.engine import BoardState
    rate = 0.0
    for _ in range(2):
        agent = _growing(None, s, cap)
        agent.set_movetime(ms)
        r = agent.evaluate_board_state(BoardState().set("", False, vid))
        agent.close()
        rate = max(rate, r["tree_nodes"] / ms)
    return rate


@pytest.mark.gpu
def test_timed_search_runs_its_time_beyond_the_initial_mapping():
    from crazyara_b200.engine import BoardState
    _, s = _settings("chess", batch_size=16, simulations=0, node_policy_temperature=1.0)
    cap = 300000
    movetime = min(2000.0, 0.5 * cap / _timed_rate(s, cap, 0))  # half the cap at the measured rate
    agent = _growing(None, s, cap)
    p0 = agent.pool()
    agent.set_movetime(movetime)
    r = agent.evaluate_board_state(BoardState().set("", False, 0))
    p1 = agent.pool()
    rep = agent.time_report()
    agent.close()
    assert r["error"] == 0 and rep["elapsed_ms"] >= movetime
    assert p1["mapped_nodes"] > p0["mapped_nodes"] and p1["grows"] > p0["grows"]
    assert p0["mapped_nodes"] < p1["nodes"] < cap


@pytest.mark.gpu
def test_the_cap_still_ends_a_search_cleanly():
    from crazyara_b200.engine import BoardState
    _, s = _settings("crazyhouse", batch_size=16, simulations=0, node_policy_temperature=1.0, threads=2)
    cap = 20000
    agent = _growing(None, s, cap)
    agent.set_movetime(20000.0)
    r = agent.evaluate_board_state(BoardState().set("", False, 1))
    p = agent.pool()
    rep = agent.time_report()
    agent.close()
    assert r["error"] == 0 and rep["elapsed_ms"] < 15000.0
    assert cap - 2 * (3 * 16 + 8) <= p["nodes"] <= cap and p["mapped_nodes"] <= cap and r["tree_nodes"] == p["nodes"]


def _set_bound(p, chunk_batches, B, edge_bound):
    """the most a growing tree's live set maps for what it holds: every array doubled past the entries in use plus one
    chunk of mini-batches (one growth step), rounded up to whole granules"""
    n = p["nodes"] + chunk_batches * (3 * B + 8)
    e = p["edges"] + chunk_batches * (3 * B + 8) * edge_bound
    return 2 * (n * NODE_BYTES + e * EDGE_BYTES) + 13 * GRAN


@pytest.mark.gpu
def test_memory_stays_bounded_over_a_timed_game_with_tree_reuse():
    from crazyara_b200.engine import BoardState
    B = 16
    _, s = _settings("crazyhouse", batch_size=B, simulations=0, node_policy_temperature=1.0, threads=2)
    cap = 300000
    movetime = min(400.0, 0.25 * cap / _timed_rate(s, cap, 1))
    agent = _growing(None, s, cap)
    agent.set_movetime(movetime)
    bs = BoardState().set("", False, 1)
    for ply in range(8):
        r = agent.evaluate_board_state(bs)
        p = agent.pool()
        assert r["error"] == 0 and p["nodes"] == r["tree_nodes"]
        assert (r["nodes_pre_search"] > 0) == (ply > 0)
        # the old set's memory went back at the compaction; the live set holds the subtree plus this search's growth
        # (Threads 2: a chunk of 4 iterations is 4 mini-batches; the root phase is one more)
        assert p["spare_bytes"] == 0 and p["mapped_bytes"] <= _set_bound(p, 5, B, 320), (ply, p)
        assert agent.compaction_count() == ply
        agent.apply_move_to_tree(r["best_move"])
        bs.do_uci(r["best_move"])
    agent.close()


@pytest.mark.gpu
def test_growing_pools_with_tree_reuse_equal_the_oracle():
    from crazyara_b200.engine import BoardState
    st, s = _settings("crazyhouse", batch_size=8, simulations=300, node_policy_temperature=1.0)
    pos = Position(None, "crazyhouse", False)
    bs = BoardState().set("", False, 1)
    S = osr.Search(st)
    agent = _growing(None, s, 1 << 18)
    for ply in range(6):
        ro = S.run(pos, osr.fake_net(S.n_labels), with_keys=True)
        rg = agent.evaluate_board_state(bs)
        assert rg["tree_nodes"] <= ro["tree_nodes"]   # (compaction drops the dead siblings: the one statistic it changes)
        ro["tree_nodes"] = rg["tree_nodes"]
        assert_same_search(ro, rg)
        assert S.reused == (ply > 0) and rg["nodes_pre_search"] == S.nodes_pre_search
        order = np.argsort(-ro["visits"].astype(np.int64), kind="stable")
        uci = ro["moves"][int(order[1 if (ply % 3 == 2 and len(order) > 1 and ro["visits"][order[1]] > 0) else 0])]
        assert S.apply_move(pos.move_from_uci(uci))
        agent.apply_move_to_tree(uci)
        pos.push_uci(uci)
        bs.do_uci(uci)
    assert agent.compaction_count() == 5
    agent.close()


@pytest.mark.gpu
def test_pool_refusals_and_reservations():
    from crazyara_b200.engine import AraError, MCTSAgent
    _, s = _settings("crazyhouse", batch_size=8, simulations=0)
    with pytest.raises(AraError, match="max_nodes"):
        MCTSAgent(None, s, 0, 3)
    several = MCTSAgent(None, s, 0, 3, 5000)          # several trees with a cap: pools mapped whole, as before
    p = several.pool(2)
    several.close()
    assert p["growing"] == 0 and p["mapped_nodes"] == p["cap_nodes"] == 5000
    device = MCTSAgent(None, s, 0, 1, 0)               # as large as the device's memory allows: reserved, not mapped
    p = device.pool()
    device.close()
    assert p["growing"] == 1 and p["cap_nodes"] > 1000000 and p["cap_edges"] == 2**31 - 1
    assert p["mapped_bytes"] < 64 * GRAN
    _, sb = _settings("crazyhouse", batch_size=8, simulations=800)
    budget = MCTSAgent(None, sb, 0, 1)
    p = budget.pool()
    budget.close()
    assert p["growing"] == 0 and p["grows"] == 0
    assert p["mapped_nodes"] == p["cap_nodes"] == 800 + 4 * 8 + 64 and p["mapped_edges"] == p["cap_edges"] == p["cap_nodes"] * 320 + 1024
    assert p["mapped_bytes"] >= p["cap_nodes"] * NODE_BYTES + p["cap_edges"] * EDGE_BYTES


@pytest.mark.gpu
def test_uci_go_infinite_with_default_options_runs_past_the_old_cap():
    """ara_uci's defaults (Threads 2, epsilon exploration, Batch_Size 16, the fake backend): `go infinite` searches until
    `stop`.  A session capped by Timed_Search_Nodes (derived from a short measured run) ends by itself; the default
    session is still searching after twice that time and, stopped, has searched more nodes than the cap."""
    from tests.test_uci_host_logic import Engine
    exe = os.path.join(ROOT, "crazyara_b200", "ara_uci")
    if not os.path.exists(exe):
        import subprocess
        subprocess.run(["make", "-C", ROOT, "crazyara_b200/ara_uci"], check=True)

    def session(extra):
        e = Engine(dict(os.environ))
        e.send("uci")
        e.read_until("uciok", timeout=60)
        for line in extra:
            e.send(line)
        e.send("position startpos moves e2e4")
        return e

    def nodes(e):
        return int([l for l in e.lines if l.startswith("info depth")][-1].split(" nodes ")[1].split()[0])

    e = session([])
    e.send("go movetime 500")
    e.read_until("bestmove", timeout=120)
    cap = 2 * nodes(e)                                   # about a second of search
    e.close()
    capped = session([f"setoption name Timed_Search_Nodes value {cap}"])
    capped.send("go movetime 100")                        # (creates the handle ahead of the timed part)
    capped.read_until("bestmove", timeout=120)
    capped.lines.clear()
    t0 = time.time()
    capped.send("go infinite")
    capped.read_until("bestmove", timeout=120)
    t_capped = time.time() - t0
    capped.send("quit")
    capped.close()
    e = session([])
    e.send("go movetime 100")
    e.read_until("bestmove", timeout=120)
    e.lines.clear()
    e.send("go infinite")
    time.sleep(2 * t_capped)
    e.send("isready")
    assert e.read_until("readyok", timeout=60) and not any(l.startswith("bestmove") for l in e.lines)
    e.send("stop")
    e.read_until("bestmove", timeout=30)
    assert nodes(e) > cap
    e.send("quit")
    e.close()


@pytest.mark.gpu
@pytest.mark.parametrize("variant,vid,mode", [("crazyhouse", 1, "crazyhouse"), ("chess", 0, "chess")])
def test_device_sized_pools_reuse_and_compact_the_kept_tree(variant, vid, mode):
    """max_nodes 0 (ara_uci's default): the reservation's edges are capped at 2^31 - 1, yet a kept subtree has room
    against it -- two timed moves, the second searches on the first's subtree, compacted into the second set"""
    from crazyara_b200.engine import BoardState, MCTSAgent
    _, s = _settings(mode, batch_size=16, simulations=0, node_policy_temperature=1.0, threads=2)
    agent = MCTSAgent(None, s, 0, 1, 0)
    agent.set_movetime(150.0)
    bs = BoardState().set("", False, vid)
    r0 = agent.evaluate_board_state(bs)
    reply = r0["pv"][1]
    for m in (r0["best_move"], reply):
        agent.apply_move_to_tree(m)
        bs.do_uci(m)
    r1 = agent.evaluate_board_state(bs)
    p = agent.pool()
    compactions = agent.compaction_count()
    agent.close()
    assert r0["error"] == 0 and r1["error"] == 0
    assert p["growing"] == 1 and p["cap_edges"] == 2**31 - 1
    assert r1["nodes_pre_search"] > 0 and compactions == 1 and p["spare_bytes"] == 0


@pytest.mark.gpu
def test_uci_default_session_reuses_the_tree():
    """ara_uci with default options (Timed_Search_Nodes 0, Reuse_Tree on): a timed game that extends the searched one
    searches on the kept tree"""
    from tests.test_uci_host_logic import Engine
    e = Engine(dict(os.environ))
    e.send("uci")
    e.read_until("uciok", timeout=60)
    e.send("position startpos")
    e.send("go movetime 300")
    best = e.read_until("bestmove", timeout=120).split()[1]
    pv = [l for l in e.lines if l.startswith("info depth")][-1].split(" pv ")[1].split()
    assert pv[0] == best and len(pv) >= 2
    e.send(f"position startpos moves {best} {pv[1]}")
    e.send("go movetime 300")
    e.read_until("bestmove", timeout=120)
    reused = [l for l in e.lines if l.startswith("info string reused")]
    e.send("quit")
    e.close()
    assert len(reused) == 1 and int(reused[0].split()[3]) > 0
