"""`ara_uci arena N` against crazyara_b200.match.Match on the GPU with seeded synthetic RISEv2 networks: for the same
options and seed both drivers must write the same arena_games_gpu_0.pgn (the Date header aside, which is the wall clock),
the same arena_results.csv line and the same summary.  Also: one network against itself, the session's search after an
arena, and the refusal of a fully-connected policy head."""
import json
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXE = os.path.join(ROOT, "crazyara_b200", "ara_uci")

BASE = {"UCI_Variant": "crazyhouse", "UCI_Chess960": "false", "Batch_Size": 8, "Nodes": 64, "Simulations": 0, "Centi_CPuct_Init": 250,
        "CPuct_Base": 19652, "Centi_Node_Temperature": 170, "Centi_Dirichlet_Epsilon": 0, "Centi_Dirichlet_Alpha": 20,
        "Centi_Q_Value_Weight": 100, "Centi_Q_Veto_Delta": 40, "Dirichlet_Seed": 42, "Threads": 1, "Centi_Epsilon_Greedy": 0,
        "Centi_Epsilon_Checks": 0, "Input_Version": 0, "Reuse_Tree": "false", "Selfplay_Games": 4, "Selfplay_Seed": 5,
        "Centi_Temperature": 0, "Temperature_Moves": 15, "Centi_Temperature_Decay": 92, "Centi_Quantile_Clipping": 0,
        "EPD_File_Path": "<empty>"}


def _rl_config_arena():
    """the RL loop's arena settings: its UCI options (tests/golden/rl_config.json) with the arena's temperature, and a
    smaller node budget so that the test stays short"""
    g = json.load(open(os.path.join(ROOT, "tests", "golden", "rl_config.json")))
    keep = ["Batch_Size", "Centi_Dirichlet_Alpha", "Centi_Dirichlet_Epsilon", "Centi_Epsilon_Checks", "Centi_Epsilon_Greedy",
            "Centi_Node_Temperature", "Centi_Q_Value_Weight", "Temperature_Moves"]
    o = {k: g[k] for k in keep}
    o.update(Centi_Temperature=60, Reuse_Tree="true", Threads=2, Nodes=64, Simulations=128)
    return o


CONFIGS = {
    "argmax": (dict(), 4),
    "rl_config_reuse_threads2": (_rl_config_arena(), 4),
    "epd_odd_n_fewer_slots": (dict(EPD_File_Path="EPD", Centi_Temperature=80, Selfplay_Games=2), 5),
    "chess960": (dict(UCI_Variant="chess", UCI_Chess960="true", Input_Version=1, Centi_Temperature=60), 4),
}
EPD = ["rnbqkbnr/pppppppp/8/8/4P3/8/PPPP1PPP/RNBQKBNR[] b KQkq - 0 1",
       "r1bqkbnr/pppppppp/2n5/8/4P3/8/PPPP1PPP/RNBQKBNR[] w KQkq - 1 2",
       "rnbqkbnr/pp1ppppp/8/2p5/4P3/8/PPPP1PPP/RNBQKBNR[] w KQkq - 0 2"]


def _blob(path, seed, in_channels=34, policy_channels=81):
    from crazyara_b200.weights import export_blob
    from oracle import net as onet
    arch = onet.arch_risev2(in_channels, policy_channels)
    os.makedirs(os.path.dirname(path), exist_ok=True)
    return export_blob(onet.make_state_dict(arch, seed), arch, path, input_version=10)


def _session(cmds, cwd, timeout=1200):
    if not os.path.exists(EXE):
        subprocess.run(["make", "-C", ROOT, "crazyara_b200/ara_uci"], check=True)
    os.makedirs(cwd, exist_ok=True)
    return subprocess.run([EXE], input="\n".join(cmds + ["quit"]) + "\n", capture_output=True, text=True, timeout=timeout,
                          cwd=cwd).stdout


def _set(producer, contender, opts):
    return ([f"setoption name Model_Path value {producer}", f"setoption name Model_Path_Contender value {contender}"] +
            [f"setoption name {k} value {v}" for k, v in opts.items()])


def _run_uci(producer, contender, opts, n, cwd):
    out = _session(_set(producer, contender, opts) + [f"arena {n}"], cwd)
    assert "error" not in out and out.rstrip().splitlines()[-1] in ("keep", "replace"), out[-3000:]
    return out.rstrip().splitlines()[-3:]


def _settings(opts):
    """the SearchSettings `arena` builds from the options (CrazyAra::prepare_search_config_structs in ara_uci)"""
    from crazyara_b200.engine import default_settings
    mode = {"crazyhouse": "crazyhouse", "chess": "chess"}[opts["UCI_Variant"]]
    B = int(opts["Batch_Size"])
    st = default_settings(mode, batch_size=B, simulations=int(opts["Simulations"]), nodes=int(opts["Nodes"]),
                          cpuct_init=opts["Centi_CPuct_Init"] / 100, cpuct_base=float(opts["CPuct_Base"]),
                          node_policy_temperature=opts["Centi_Node_Temperature"] / 100,
                          dirichlet_epsilon=opts["Centi_Dirichlet_Epsilon"] / 100, dirichlet_alpha=opts["Centi_Dirichlet_Alpha"] / 100,
                          q_value_weight=opts["Centi_Q_Value_Weight"] / 100, q_veto_delta=opts["Centi_Q_Veto_Delta"] / 100,
                          mcts_solver=1, virtual_style=3, virtual_mix_threshold=1000, seed=int(opts["Dirichlet_Seed"]),
                          threads=2 if int(opts["Threads"]) >= 2 and 2 * B <= 255 else 1,
                          epsilon_greedy_counter=round(100 / opts["Centi_Epsilon_Greedy"]) if opts["Centi_Epsilon_Greedy"] else 0,
                          epsilon_checks_counter=round(100 / opts["Centi_Epsilon_Checks"]) if opts["Centi_Epsilon_Checks"] else 0)
    if int(opts["Input_Version"]) > 0:
        st.input_version = int(opts["Input_Version"])
    return st


def _run_match(producer, contender, opts, n, cwd):
    """Match with what `arena` builds from the same options; returns the summary lines `arena` prints"""
    from crazyara_b200 import match as mt
    from crazyara_b200.nn import NeuralNetAPI
    variant = {"crazyhouse": 1, "chess": 0}[opts["UCI_Variant"]]
    slots = min(int(opts["Selfplay_Games"]), n)
    B = int(opts["Batch_Size"])
    os.makedirs(cwd, exist_ok=True)
    nets = [NeuralNetAPI("gpu", 0, slots * B, producer)]
    nets.append(nets[0] if contender == producer else NeuralNetAPI("gpu", 0, slots * B, contender))
    st = _settings(opts)
    m = mt.Match((nets[0], st, mt.player_name(producer)), (nets[1], st, mt.player_name(contender)), n, variant=variant,
                 is960=opts["UCI_Chess960"] == "true", slots=slots, epd_path=opts["EPD_File_Path"],
                 temperature=opts["Centi_Temperature"] / 100, temperature_moves=int(opts["Temperature_Moves"]),
                 temperature_decay=opts["Centi_Temperature_Decay"] / 100, quantile_clipping=opts["Centi_Quantile_Clipping"] / 100,
                 seed=int(opts["Selfplay_Seed"]), reuse_tree=opts["Reuse_Tree"] == "true",
                 pgn_path=os.path.join(cwd, "arena_games_gpu_0.pgn"))
    m.run()
    m.close()
    for net in set(nets):
        net.close()
    r = m.result
    r.write_csv(os.path.join(cwd, "arena_results.csv"))
    return ["Arena summary", f"Score of Contender vs Producer: {r}", r.verdict()]


def _pgn(path):
    return re.sub(r'\[Date "[^"]*"\]', '[Date "?"]', open(path).read())


def _compare(cpp, py):
    assert _pgn(os.path.join(cpp, "arena_games_gpu_0.pgn")) == _pgn(os.path.join(py, "arena_games_gpu_0.pgn"))
    assert open(os.path.join(cpp, "arena_results.csv")).read() == open(os.path.join(py, "arena_results.csv")).read()


@pytest.mark.gpu
@pytest.mark.parametrize("config", list(CONFIGS))
def test_arena_matches_match_byte_for_byte(tmp_path, config):
    extra, n = CONFIGS[config]
    opts = dict(BASE, **extra)
    if opts["EPD_File_Path"] == "EPD":
        (tmp_path / "openings.epd").write_text(EPD[0] + ";\n" + EPD[1] + "\n" + EPD[2] + ";\n")
        opts["EPD_File_Path"] = str(tmp_path / "openings.epd")
    shape = (39, 76) if opts["UCI_Variant"] == "chess" else (34, 81)
    producer = _blob(str(tmp_path / "nets" / "producer.arab"), 0, *shape)
    contender = _blob(str(tmp_path / "nets" / "contender.arab"), 1, *shape)
    cpp, py = str(tmp_path / "cpp"), str(tmp_path / "py")
    summary = _run_uci(producer, contender, opts, n, cpp)
    assert summary == _run_match(producer, contender, opts, n, py)
    _compare(cpp, py)
    text = open(os.path.join(cpp, "arena_games_gpu_0.pgn")).read()
    assert text.count("[Event ") == n and text.count('[White "CrazyAra-B200-contender"]') == (n + 1) // 2
    if config == "chess960":
        assert '[Variant "chess960"]' in text


@pytest.mark.gpu
def test_one_network_against_itself_mirrors_every_pair(tmp_path):
    """argmax moves of one network: the two games of a pair are the same game with the colours swapped, so W = L; one
    network object (equal paths) and two networks (the blob under a second path) write the same files"""
    blob = _blob(str(tmp_path / "a" / "risev2.arab"), 0)
    copy = str(tmp_path / "b" / "risev2.arab")
    os.makedirs(os.path.dirname(copy))
    shutil.copy(blob, copy)
    opts = dict(BASE, Selfplay_Games=2)
    shared, two = str(tmp_path / "shared"), str(tmp_path / "two")
    s1 = _run_uci(blob, blob, opts, 4, shared)
    s2 = _run_uci(blob, copy, opts, 4, two)
    assert s1 == s2
    _compare(shared, two)
    w, d, l = (int(x) for x in open(os.path.join(shared, "arena_results.csv")).read().strip().split(",")[2:])
    assert w == l and w + d + l == 4 and s1[-1] == "keep"
    games = [g.split("\n\n")[1] for g in _pgn(os.path.join(shared, "arena_games_gpu_0.pgn")).split("[Variant")[1:]]
    assert games[0] == games[1] and games[2] == games[3]


@pytest.mark.gpu
def test_go_after_arena_searches_as_before(tmp_path):
    producer = _blob(str(tmp_path / "nets" / "producer.arab"), 0)
    contender = _blob(str(tmp_path / "nets" / "contender.arab"), 1)
    go = ["position startpos moves e2e4", "go nodes 200"]
    out = _session(_set(producer, contender, dict(BASE, Selfplay_Games=2)) + ["isready"] + go + ["arena 2"] + go, str(tmp_path))
    assert "error" not in out
    lines = out.splitlines()
    best = [l for l in lines if l.startswith("bestmove")]
    nodes = [re.search(r" nodes (\d+) ", l).group(1) for l in lines if l.startswith("info depth")]
    assert len(best) == 2 and best[0] == best[1] and len(nodes) == 2 and nodes[0] == nodes[1]
    k = lines.index("Arena summary")
    assert lines[k + 2] in ("keep", "replace") and best[1] == lines[-1]


@pytest.mark.gpu
@pytest.mark.parametrize("fc_player", ["producer", "contender"])
def test_arena_refuses_a_fully_connected_policy_head(tmp_path, fc_player):
    from crazyara_b200 import synthetic
    from crazyara_b200.weights import export_blob
    arch = synthetic.classic(synthetic.risev2(34, 81), 2272)
    os.makedirs(str(tmp_path / "nets"))
    fc = export_blob(synthetic.random_state_dict(arch, 0), arch, str(tmp_path / "nets" / "fc.arab"), input_version=10)
    other = _blob(str(tmp_path / "nets" / "risev2.arab"), 0)
    pair = (fc, other) if fc_player == "producer" else (other, fc)
    cwd = str(tmp_path / "run")
    out = _session(_set(pair[0], pair[1], dict(BASE, Selfplay_Games=2)) + ["arena 2"], cwd)
    lines = out.splitlines()
    assert len(lines) == 1 and lines[0].startswith("info string") and "fully-connected policy head" in lines[0], out
    assert os.listdir(cwd) == []
