"""GPU search (one warp per tree, device-resident SoA tree) against the CPU search oracle.

 (a) hash-derived fake backend on both sides -> visit counts, Q, priors, posterior, root value, counters BIT-EXACT
 (b) real wgmma network: the oracle search is driven by the SAME GPU network through its host API, so both sides
     consume identical policy/value floats -> bit-exact at node temperature 1 and at the UCI default 1.7 (glibc's
     powf restated on the device, crazyara_b200/csrc/glibc_flt32.cuh).
"""
import numpy as np
import pytest

from oracle import search as osr
from oracle.chess import Position
from tests.test_search_hostemu import CASES, assert_same_search, case_settings


def _gpu_search(variant_id, fen, is960, premoves, settings, net=None, n_trees=1):
    from crazyara_b200.engine import BoardState, MCTSAgent, SearchSettings
    st = BoardState().set(fen or "", is960, variant_id)
    st.do_uci(*premoves)
    s = SearchSettings()
    for f, _ in s._fields_:
        setattr(s, f, getattr(settings, f))
    agent = MCTSAgent(net, s, 0, n_trees)
    for t in range(n_trees):
        agent.set_position(st, t)
    agent.evaluate_board_state()
    res = agent.results()
    agent.close()
    return res


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=[f"{c[0]}-b{c[6]}-s{c[7]}-{i}" for i, c in enumerate(CASES)])
def test_gpu_search_equals_oracle_fake_backend(case):
    variant, vid, mode, fen, is960, premoves, batch, sims, extra = case
    st = case_settings(mode, batch, sims, extra)
    pos = Position(fen, variant, is960)
    pos.push_uci(*premoves)
    S = osr.Search(st)
    ro = S.run(pos, osr.fake_net(S.n_labels), with_keys=True)
    rg = _gpu_search(vid, fen, is960, premoves, st)[0]
    assert_same_search(ro, rg)


CASES_2T = [c for c in CASES if 2 * c[6] < 256]  # Threads x Batch_Size < 256 (uint8 virtual-visit counter, as in the reference)


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES_2T, ids=[f"{c[0]}-b{c[6]}-s{c[7]}-{i}" for i, c in enumerate(CASES_2T)])
def test_gpu_two_thread_search_equals_oracle_fake_backend(case):
    """Threads = 2 on the device: two logical search threads per tree, their tree kernels on one stream in the fixed
    schedule of oracle/mcts.h, their network batches on a second stream (one thread selects while the other's batch is
    evaluated).  Deterministic, so visit counts / Q / priors / posterior are the oracle's bits in this mode too."""
    variant, vid, mode, fen, is960, premoves, batch, sims, extra = case
    st = case_settings(mode, batch, sims, dict(extra, threads=2))
    pos = Position(fen, variant, is960)
    pos.push_uci(*premoves)
    S = osr.Search(st)
    ro = S.run(pos, osr.fake_net(S.n_labels), with_keys=True, threads=2)
    rg = _gpu_search(vid, fen, is960, premoves, st)[0]
    assert_same_search(ro, rg)


@pytest.mark.gpu
@pytest.mark.parametrize("threads", [1, 2])
@pytest.mark.parametrize("case", CASES_2T[::2], ids=[f"{c[0]}-b{c[6]}-s{c[7]}-{i}" for i, c in enumerate(CASES_2T[::2])])
def test_gpu_epsilon_exploration_equals_oracle(case, threads):
    """Centi_Epsilon_Greedy 5 / Centi_Epsilon_Checks 1 (the reference's UCI defaults) on the device: select_kernel<true>
    with glibc's rand() restated; the oracle it is compared with equals the compiled reference (tests/test_ref_mcts.py)."""
    variant, vid, mode, fen, is960, premoves, batch, sims, extra = case
    st = case_settings(mode, batch, sims, dict(extra, threads=threads, epsilon_greedy_counter=20, epsilon_checks_counter=100))
    pos = Position(fen, variant, is960)
    pos.push_uci(*premoves)
    S = osr.Search(st)
    ro = S.run(pos, osr.fake_net(S.n_labels), with_keys=True, threads=threads)
    rg = _gpu_search(vid, fen, is960, premoves, st)[0]
    assert_same_search(ro, rg)


@pytest.mark.gpu
def test_gpu_two_thread_multi_tree_search_matches_single_tree():
    st = osr.default_settings("crazyhouse", batch_size=8, simulations=300, node_policy_temperature=1.7, threads=2)
    pos = Position(variant="crazyhouse")
    S = osr.Search(st)
    ro = S.run(pos, osr.fake_net(S.n_labels), with_keys=True, threads=2)
    for r in _gpu_search(1, None, False, [], st, n_trees=5):
        assert_same_search(ro, r)


@pytest.mark.gpu
@pytest.mark.parametrize("seed", range(32))
def test_gpu_search_equals_oracle_random_cases(seed):
    """The randomised cases of tests/test_search_fuzz_hostemu.py on the real device search."""
    from tests.test_search_fuzz_hostemu import _random_case
    pos, _, st, (vid, played) = _random_case(seed)
    S = osr.Search(st)
    ro = S.run(pos, osr.fake_net(S.n_labels), with_keys=True)
    rg = _gpu_search(vid, None, False, played, st)[0]
    assert_same_search(ro, rg)


@pytest.mark.gpu
def test_gpu_multi_tree_search_matches_single_tree():
    st = osr.default_settings("crazyhouse", batch_size=8, simulations=300, node_policy_temperature=1.0)
    pos = Position(variant="crazyhouse")
    S = osr.Search(st)
    ro = S.run(pos, osr.fake_net(S.n_labels), with_keys=True)
    for r in _gpu_search(1, None, False, [], st, n_trees=5):
        assert_same_search(ro, r)


def _make_net(tmp_path, arch, batch, version, precision="float16"):
    from crazyara_b200.nn import NeuralNetAPI
    from crazyara_b200.weights import export_blob
    from oracle import net as onet
    sd = onet.make_state_dict(arch, 0)
    blob = export_blob(sd, arch, str(tmp_path / f"{arch['name']}.arab"), input_version=version)
    return NeuralNetAPI("gpu", 0, batch, blob, precision=precision)


def _net_fn(net):
    def fn(planes):
        n = planes.shape[0]
        B = net.get_batch_size()
        x = np.zeros((B,) + planes.shape[1:], np.float32)
        x[:n] = planes
        v = np.zeros(B, np.float32)
        p = np.zeros((B, net.get_nb_policy_values()), np.float32)
        net.predict(x, v, p, None, n=n)
        return v[:n].copy(), p[:n].copy()
    return fn


REAL_CASES = [("crazyhouse", 1, "crazyhouse", "risev2", 34, 81, 1, [], 8, 800),           # BASELINE cfg 2
              ("crazyhouse", 1, "crazyhouse", "risev2", 34, 81, 1, [], 64, 3200),         # the headline workload (bench.py)
              ("crazyhouse", 1, "crazyhouse", "risev2", 34, 81, 1, ["e2e4", "e7e5"], 64, 1600),
              ("chess", 0, "chess", "risev33", 52, 76, 3, [], 64, 1600),                  # BASELINE cfg 3
              ("kingofthehill", 2, "lichess", "risev2", 63, 84, 1, ["e2e4", "e7e5"], 128, 800),   # BASELINE cfg 5
              ("3check", 3, "lichess", "risev2", 63, 84, 1, ["e2e4", "e7e5"], 128, 800)]


@pytest.mark.gpu
@pytest.mark.parametrize("variant,vid,mode,arch_name,cin,pch,version,premoves,batch,sims", REAL_CASES)
def test_gpu_search_real_net_equals_oracle_driven_by_same_net(tmp_path, variant, vid, mode, arch_name, cin, pch, version,
                                                              premoves, batch, sims):
    from oracle import net as onet
    arch = onet.arch_risev2(cin, pch) if arch_name == "risev2" else onet.arch_risev33(cin, pch, True)
    net = _make_net(tmp_path, arch, batch, version * 10)
    st = osr.default_settings(mode, batch_size=batch, simulations=sims, node_policy_temperature=1.0, input_version=version)
    pos = Position(variant=variant)
    pos.push_uci(*premoves)
    S = osr.Search(st)
    ro = S.run(pos, _net_fn(net))
    rg = _gpu_search(vid, None, False, premoves, st, net=net)[0]
    assert_same_search(ro, rg)
    # default node temperature 1.7: glibc powf restated on the device, sequential normalising sum -> still bit-exact
    st2 = osr.default_settings(mode, batch_size=batch, simulations=sims, input_version=version)
    st2.node_policy_temperature = 1.7
    ro2 = osr.Search(st2).run(pos, _net_fn(net))
    rg2 = _gpu_search(vid, None, False, premoves, st2, net=net)[0]
    assert_same_search(ro2, rg2)
    # Threads = 2 with the real network (second input / output set of the net, forwards on the network stream)
    if 2 * batch < 256:
        st3 = osr.default_settings(mode, batch_size=batch, simulations=sims, input_version=version, threads=2)
        st3.node_policy_temperature = 1.7
        ro3 = osr.Search(st3).run(pos, _net_fn(net), threads=2)
        rg3 = _gpu_search(vid, None, False, premoves, st3, net=net)[0]
        assert_same_search(ro3, rg3)
    net.close()


@pytest.mark.gpu
@pytest.mark.parametrize("variant,vid,mode,arch_name,cin,pch,version,batch,sims",
                         [("crazyhouse", 1, "crazyhouse", "risev2", 34, 81, 1, 8, 400),
                          ("chess", 0, "chess", "risev33", 52, 76, 3, 16, 600)])
def test_gpu_search_float32_net_against_oracle_search_with_the_fp32_oracle_network(tmp_path, variant, vid, mode, arch_name,
                                                                                    cin, pch, version, batch, sims):
    """End to end against the reference chain: the ORACLE search driven by the ORACLE's fp32 torch network (oracle/net.py,
    pinned to the reference's module) vs the GPU search with the Precision float32 GPU network.  Network outputs agree
    to ~1e-6, not to the bit, so a visit can land on a neighbouring move where two PUCT scores are that close; the
    contract is north_star's: root value, root priors, Q and the posterior within 1e-4, the same best move, and visit
    counts that differ by a handful at most."""
    from oracle import net as onet
    arch = onet.arch_risev2(cin, pch) if arch_name == "risev2" else onet.arch_risev33(cin, pch, True)
    sd = onet.make_state_dict(arch, 0)
    net = _make_net(tmp_path, arch, batch, version * 10, precision="float32")
    st = osr.default_settings(mode, batch_size=batch, simulations=sims, input_version=version)

    def oracle_net(planes):
        r = onet.forward(sd, arch, planes)
        return r["value"], r["prob"]
    pos = Position(variant=variant)
    ro = osr.Search(st).run(pos, oracle_net)
    rg = _gpu_search(vid, None, False, [], st, net=net)[0]
    net.close()
    assert rg["error"] == 0 and ro["moves"][ro["best_idx"]] == rg["moves"][rg["best_idx"]]
    og = {m: i for i, m in enumerate(rg["moves"])}
    perm = [og[m] for m in ro["moves"]]     # near-equal priors may swap two neighbours in the sorted order
    np.testing.assert_allclose(rg["prior"][perm], ro["prior"], atol=1e-4, rtol=0)
    assert abs(ro["root_value"] - rg["root_value"]) < 1e-4
    assert ro["visit_sum"] == rg["visit_sum"]
    dv = np.abs(ro["visits"].astype(np.int64) - rg["visits"][perm].astype(np.int64))
    assert dv.sum() <= max(4, ro["visit_sum"] // 100), dv
    same = dv == 0                          # Q / posterior of the moves whose visit counts agree
    np.testing.assert_allclose(rg["q"][perm][same], ro["q"][same], atol=1e-4, rtol=0)
    if dv.sum() == 0:
        np.testing.assert_allclose(rg["policy"][perm], ro["policy"], atol=1e-4, rtol=0)


@pytest.mark.gpu
@pytest.mark.parametrize("alpha,seed,temp", [(0.3, 7, 1.0), (0.2, 42, 1.7), (0.3, 2024, 1.7), (1.5, 3, 1.0), (1.0, 9, 1.7)])
def test_gpu_search_dirichlet_equals_oracle(alpha, seed, temp):
    """Root noise: libstdc++ gamma_distribution<float> over minstd_rand0 with glibc logf / powf restated on the device:
    the noised priors, hence every visit count, are the oracle's bits."""
    st = osr.default_settings("crazyhouse", batch_size=8, simulations=400, node_policy_temperature=temp,
                              dirichlet_epsilon=0.25, dirichlet_alpha=alpha, seed=seed)
    pos = Position(variant="crazyhouse")
    S = osr.Search(st)
    ro = S.run(pos, osr.fake_net(S.n_labels), with_keys=True)
    rg = _gpu_search(1, None, False, [], st)[0]
    assert_same_search(ro, rg)


REUSE_CASES = [("crazyhouse", 1, "crazyhouse", 8, 300, {}), ("chess", 0, "chess", 16, 400, {}),
               ("crazyhouse", 1, "crazyhouse", 8, 0, dict(nodes=250, dirichlet_epsilon=0.25, dirichlet_alpha=0.3)),
               ("3check", 3, "lichess", 4, 200, {})]


@pytest.mark.gpu
@pytest.mark.parametrize("variant,vid,mode,batch,sims,extra", REUSE_CASES)
def test_gpu_tree_reuse_equals_oracle(variant, vid, mode, batch, sims, extra):
    """MCTSAgent::apply_move_to_tree / init_root_node (agents/mctsagent.cpp:113-160, 230-247) on the device: a game of
    searched and played moves, every search continuing on the kept subtree, bit-exact with the oracle."""
    from crazyara_b200.engine import BoardState, MCTSAgent, SearchSettings
    st = osr.default_settings(mode, batch_size=batch, simulations=sims, node_policy_temperature=1.0, **extra)
    s = SearchSettings()
    for f, _ in s._fields_:
        setattr(s, f, getattr(st, f))
    pos = Position(None, variant, False)
    bs = BoardState().set("", False, vid)
    S = osr.Search(st)
    agent = MCTSAgent(None, s, 0, 1, 1 << 15)
    for ply in range(6):
        ro = S.run(pos, osr.fake_net(S.n_labels), with_keys=True)
        rg = agent.evaluate_board_state(bs)
        assert_same_search(ro, rg)
        assert S.reused == (ply > 0) and rg["nodes_pre_search"] == S.nodes_pre_search
        order = np.argsort(-ro["visits"].astype(np.int64), kind="stable")
        pick = int(order[1 if (ply % 3 == 2 and len(order) > 1 and ro["visits"][order[1]] > 0) else 0])
        uci = ro["moves"][pick]
        assert S.apply_move(pos.move_from_uci(uci))
        agent.apply_move_to_tree(uci)
        pos.push_uci(uci)
        bs.do_uci(uci)
    # a position that is not the kept one starts a new tree
    other = BoardState().set("", False, vid)
    assert agent.evaluate_board_state(other)["nodes_pre_search"] == 0
    agent.close()


@pytest.mark.gpu
@pytest.mark.parametrize("threads", [1, 2])
def test_gpu_tree_reuse_survives_full_pools_by_compaction(threads):
    """A long game on node pools that hold barely three searches: the kept subtree is copied to the front of the second
    set of pools whenever the dead siblings have eaten the room (search.cu, compact_pools), so EVERY search continues on
    the kept statistics like the oracle's (whose pool is unbounded) -- bit-exact, node ids aside."""
    from crazyara_b200.engine import BoardState, MCTSAgent, SearchSettings
    st = osr.default_settings("crazyhouse", batch_size=16, simulations=400, node_policy_temperature=1.0, threads=threads)
    s = SearchSettings()
    for f, _ in s._fields_:
        setattr(s, f, getattr(st, f))
    pos = Position(None, "crazyhouse", False)
    bs = BoardState().set("", False, 1)
    S = osr.Search(st)
    agent = MCTSAgent(None, s, 0, 1, 1400)
    for ply in range(24):
        ro = S.run(pos, osr.fake_net(S.n_labels), with_keys=True, threads=threads)
        rg = agent.evaluate_board_state(bs)
        if agent.compaction_count() > 0:   # (the pool usage is the one statistic a compaction changes: dead nodes are gone)
            assert rg["tree_nodes"] <= ro["tree_nodes"]
            ro["tree_nodes"] = rg["tree_nodes"]
        assert_same_search(ro, rg)
        assert S.reused == (ply > 0) and rg["nodes_pre_search"] == S.nodes_pre_search
        order = np.argsort(-ro["visits"].astype(np.int64), kind="stable")
        uci = ro["moves"][int(order[0])]
        assert S.apply_move(pos.move_from_uci(uci))
        agent.apply_move_to_tree(uci)
        pos.push_uci(uci)
        bs.do_uci(uci)
    assert agent.compaction_count() >= 5
    agent.close()


@pytest.mark.gpu
def test_gpu_time_manager_early_stop_and_veto():
    """ThreadManager on the device search: with a (deliberately tiny) NPS estimate the early-stopping rules fire at the
    first update interval at which the most visited move also looks best; a dropped evaluation vetoes the stop once
    (continue_search) and the search then runs its whole move time."""
    from crazyara_b200.engine import BoardState, MCTSAgent, TimeControl, default_settings
    # (1.d4 d5 with the hash-derived fake network: the rules hold at > 99 % of the iterations of a host-emulated
    # search, so one of the first update intervals triggers; at the start position they hold at < 10 %)
    s = default_settings("chess", batch_size=16, simulations=0, nodes=0, node_policy_temperature=1.0)
    agent = MCTSAgent(None, s, 0, 1, 150000)
    st = BoardState().set("", False, 0).do_uci("d2d4", "d7d5")
    base = dict(movetime_ms=400.0, update_interval_ms=20.0, overall_nps=1.0, safe_remaining_ms=60000.0, move_overhead_ms=20.0,
                in_game=1, can_prolong=1)
    agent.set_movetime(400.0)
    agent.set_time_control(TimeControl(last_value_eval=-1.0, **base))   # evaluation cannot have dropped below -1
    r = agent.evaluate_board_state(st)
    rep = agent.time_report()
    assert rep["early_stopped"] in (1, 2) and rep["prolonged"] == 0
    assert rep["elapsed_ms"] < 300.0 and rep["saved_ms"] > 0 and r["nodes"] > 100
    agent.set_time_control(TimeControl(last_value_eval=0.999, **base))  # every evaluation is a drop: veto, search on
    r2 = agent.evaluate_board_state(st)
    rep2 = agent.time_report()
    assert rep2["early_stopped"] == 0 and rep2["prolonged"] == 1
    assert 380.0 <= rep2["elapsed_ms"] < 700.0 and r2["nodes"] > r["nodes"]
    agent.set_time_control(None)                                        # manager off: plain move time
    agent.evaluate_board_state(st)
    assert agent.time_report()["early_stopped"] == 0 and agent.time_report()["prolonged"] == 0
    agent.close()


@pytest.mark.gpu
def test_gpu_packed_multi_tree_batches_equal_single_tree_searches(tmp_path):
    """Several trees share each network batch; their new leaves are packed into consecutive rows and the network skips
    the unused rows (device-side count).  Every tree must come out exactly as when it is searched alone."""
    from crazyara_b200.engine import BoardState, MCTSAgent, SearchSettings
    from oracle import net as onet
    B, sims = 8, 240
    lines = [[], ["e2e4"], ["e2e4", "e7e5"], ["d2d4", "g8f6", "c2c4"], ["g1f3", "d7d5"]]
    net = _make_net(tmp_path, onet.arch_risev2(34, 81), len(lines) * B, 10)
    st = osr.default_settings("crazyhouse", batch_size=B, simulations=sims, node_policy_temperature=1.0,
                              dirichlet_epsilon=0.25, dirichlet_alpha=0.3, seed=3)
    s = SearchSettings()
    for f, _ in s._fields_:
        setattr(s, f, getattr(st, f))
    multi = MCTSAgent(net, s, 0, len(lines))
    for t, moves in enumerate(lines):
        multi.set_position(BoardState().set("", False, 1).do_uci(*moves), t)
    multi.evaluate_board_state()
    together = multi.results()
    multi.close()
    for t, moves in enumerate(lines):
        # tree t of a handle seeds its Dirichlet generator with seed ^ t * golden ratio (TreeState::rng): searched
        # alone, the position gets that seed as tree 0 of its own handle
        s.seed = (st.seed ^ (t * 0x9E3779B97F4A7C15)) & 0xFFFFFFFFFFFFFFFF
        alone = MCTSAgent(net, s, 0, 1)
        r = alone.evaluate_board_state(BoardState().set("", False, 1).do_uci(*moves))
        alone.close()
        assert_same_search(r, together[t])
        assert together[t]["evals"] > 0
    net.close()


# Positions in which many playouts of a mini-batch end in terminal nodes: in the wavefront select kernel
# (search_wave.cuh) every terminal commit makes the younger playouts in flight take their virtual visits back and
# start again -- wide mini-batches, so that many playouts are in flight when that happens.
TERMINAL_HEAVY = [
    ("chess", 0, "chess", "6k1/5ppp/8/8/8/8/8/R3K2R w KQ - 0 1", 32, 1200, dict(mcts_solver=0)),
    ("chess", 0, "chess", "6k1/5ppp/8/8/8/8/8/R3K2R w KQ - 0 1", 64, 1600, dict()),
    ("chess", 0, "chess", "7k/5Q2/6K1/8/8/8/8/8 w - - 0 1", 64, 2000, dict(mcts_solver=0)),
    ("chess", 0, "chess", "7k/5Q2/6K1/8/8/8/8/8 w - - 0 1", 16, 600, dict(mcts_solver=0, virtual_style=0)),
    ("crazyhouse", 1, "crazyhouse", "4R2b/1N3rkb/1p2P1pp/p2P4/2P1P3/8/PP4Q1/3R3K[QRBBNNNPPPPpp] w - - 2 53", 32, 1500,
     dict(mcts_solver=0)),
    ("crazyhouse", 1, "crazyhouse", "4R2b/1N3rkb/1p2P1pp/p2P4/2P1P3/8/PP4Q1/3R3K[QRBBNNNPPPPpp] w - - 2 53", 64, 1500,
     dict(node_policy_temperature=1.7, virtual_mix_threshold=50)),
]


@pytest.mark.gpu
@pytest.mark.parametrize("threads", [1, 2])
@pytest.mark.parametrize("case", TERMINAL_HEAVY, ids=[f"{c[0]}-b{c[4]}-s{c[5]}-{i}" for i, c in enumerate(TERMINAL_HEAVY)])
def test_gpu_wavefront_select_with_many_terminal_playouts(case, threads, monkeypatch):
    variant, vid, mode, fen, batch, sims, extra = case
    st = case_settings(mode, batch, sims, dict(extra, threads=threads))
    pos = Position(fen, variant, False)
    S = osr.Search(st)
    ro = S.run(pos, osr.fake_net(S.n_labels), with_keys=True, threads=threads)
    monkeypatch.delenv("ARA_WAVE", raising=False)
    rg = _gpu_search(vid, fen, False, [], st)[0]          # the wavefront kernel (one tree, Batch_Size >= 8)
    assert_same_search(ro, rg)
    monkeypatch.setenv("ARA_WAVE", "0")
    rs = _gpu_search(vid, fen, False, [], st)[0]          # one warp per tree
    assert_same_search(ro, rs)


def _random_gpu_case(seed):
    """random position (legal random play, every variant) and settings; wide mini-batches so that the wavefront select
    (Batch_Size >= 8 for one tree) has playouts in flight, one or two logical threads"""
    rng = np.random.default_rng(1000 + seed)
    variant, vid, mode = [("crazyhouse", 1, "crazyhouse"), ("chess", 0, "chess"), ("kingofthehill", 2, "lichess"),
                          ("3check", 3, "lichess")][seed % 4]
    pos = Position(None, variant, False)
    played = []
    for _ in range(int(rng.integers(0, 60))):
        moves = pos.legal_uci()
        if not moves or pos.terminal(len(moves)) != 4:
            break
        u = moves[int(rng.integers(0, len(moves)))]
        nxt = pos.clone().push_uci(u)
        nm = nxt.legal_uci()
        if not nm or nxt.terminal(len(nm)) != 4:
            continue
        pos.push_uci(u)
        played.append(u)
    batch = int(rng.choice([8, 16, 32, 64, 100]))
    threads = int(rng.choice([1, 2])) if 2 * batch < 256 else 1
    extra = dict(threads=threads)
    if rng.random() < 0.4:
        extra["virtual_style"] = int(rng.choice([0, 1, 3]))
    if rng.random() < 0.4:
        extra["virtual_mix_threshold"] = int(rng.choice([3, 20, 1000]))
    if rng.random() < 0.3:
        extra["mcts_solver"] = 0
    temp = float(rng.choice([1.0, 1.7, 1.7, 0.8]))
    if rng.random() < 0.3:
        extra.update(dirichlet_epsilon=0.25, dirichlet_alpha=float(rng.choice([0.2, 0.3, 1.0])), seed=int(rng.integers(1, 2**31 - 2)))
    sims = int(rng.choice([300, 800, 1500]))
    st = osr.default_settings(mode, batch_size=batch, simulations=sims, node_policy_temperature=temp, **extra)
    return pos, vid, played, st, threads


@pytest.mark.gpu
@pytest.mark.parametrize("seed", range(32))
def test_gpu_random_positions_and_settings_equal_oracle(seed):
    pos, vid, played, st, threads = _random_gpu_case(seed)
    S = osr.Search(st)
    ro = S.run(pos, osr.fake_net(S.n_labels), with_keys=True, threads=threads)
    rg = _gpu_search(vid, None, False, played, st)[0]
    assert_same_search(ro, rg)
