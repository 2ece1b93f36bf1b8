"""`ara_uci arena N` and `activeuci` on the CPU.

  * TournamentResult of the C++ host (host/selfplay_io.h) against the reference's, recorded in tests/golden/tournament.json;
  * the Model_Path_Contender option, `activeuci`, and the refusals of `arena`;
  * the arena's host logic against crazyara_b200.match.Match: the search entry points of the C-ABI are replaced by a
    stand-in (tests/uci_stub/stub_arena.cpp, LD_PRELOADed) whose result for a tree is a function of its root alone, and
    Match runs with its Python twin as agent.  Both must write the same PGN (Date header aside), CSV line and summary, and
    make the same tree calls;
  * where the reference's sources are present, its own RL-loop client (rl/binaryio.py) reads `activeuci` and the
    arena's verdict from the binary."""
import json
import os
import re
import struct
import subprocess
import sys

import numpy as np
import pytest

import crazyara_b200.match as mt
from crazyara_b200.engine import default_settings

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXE = os.path.join(ROOT, "crazyara_b200", "ara_uci")
GOLDEN = os.path.join(ROOT, "tests", "golden", "tournament.json")
REFERENCE = "/root/reference"
M64 = (1 << 64) - 1


def _exe():
    if not os.path.exists(EXE):
        subprocess.run(["make", "-C", ROOT, "crazyara_b200/ara_uci"], check=True)
    return EXE


def _session(cmds, cwd=None, env=None, timeout=120):
    return subprocess.run([_exe()], input="\n".join(cmds + ["quit"]) + "\n", capture_output=True, text=True, timeout=timeout,
                          cwd=cwd, env=env).stdout


# ------------------------------------------------------------------------------------------------------ TournamentResult
@pytest.fixture(scope="module")
def tournament_driver(tmp_path_factory):
    import crazyara_b200
    crazyara_b200.lib()
    exe = str(tmp_path_factory.mktemp("tournament") / "tournament_driver")
    lib_dir = os.path.join(ROOT, "crazyara_b200")
    subprocess.run(["g++", "-O2", "-std=c++17", "-Wall", "-I" + os.path.join(ROOT, "include"), "-I" + os.path.join(lib_dir, "host"),
                    "-I" + os.path.join(lib_dir, "csrc"), os.path.join(ROOT, "tests", "tournament_driver.cpp"), "-o", exe,
                    "-L" + lib_dir, "-lara_b200", "-Wl,-rpath," + lib_dir, "-L/usr/local/cuda/lib64",
                    "-Wl,-rpath,/usr/local/cuda/lib64"], check=True)
    return exe


def test_tournament_result_in_cpp_equals_the_reference_golden(tournament_driver, tmp_path):
    cases = json.load(open(GOLDEN))["cases"]
    csv = tmp_path / "r.csv"
    stdin = "".join(f"{c['a']}\t{c['b']}\t{c['w']}\t{c['d']}\t{c['l']}\n" for c in cases)
    out = subprocess.run([tournament_driver, str(csv)], input=stdin, capture_output=True, text=True, check=True).stdout.splitlines()
    assert len(out) == 3 * len(cases)
    for k, c in enumerate(cases):
        text, bits, verdict = out[3 * k:3 * k + 3]
        assert text == c["text"] and int(bits) == c["score_bits"], c
        assert verdict == ("replace" if struct.unpack("<f", struct.pack("<I", c["score_bits"]))[0] > 0.5 else "keep"), c
    assert csv.read_text() == "".join(c["csv"] for c in cases)


# ------------------------------------------------------------------------------------------------------ options
def _uci_table(out):
    names = []
    for line in out.splitlines():
        if line.startswith("option name "):
            t = line.split()
            names.append((" ".join(t[2:t.index("type")]), t[t.index("type") + 1]))
    return names


def test_uci_lists_model_path_contender_as_a_string_option():
    out = _session(["uci"])
    assert "option name Model_Path_Contender type string default " in out.splitlines()
    assert ("Model_Path_Contender", "string") in _uci_table(out)


def test_activeuci_prints_every_option_with_its_value_then_readyok():
    names = [n for n, _ in _uci_table(_session(["uci"]))]
    out = _session(["setoption name Batch_Size value 8", "setoption name Model_Path_Contender value nets/new model.arab",
                    "setoption name Centi_Temperature value 60", "activeuci"]).splitlines()
    assert out[-1] == "readyok" and len(out) == len(names) + 1
    got = {}
    for line in out[:-1]:
        m = re.fullmatch(r"option name (\S+) value ?(.*)", line)
        assert m, line
        got[m.group(1)] = m.group(2)
    assert sorted(got) == sorted(names)
    assert got["Batch_Size"] == "8" and got["Model_Path_Contender"] == "nets/new model.arab" and got["Centi_Temperature"] == "60"
    assert got["Model_Path"] == "" and got["UCI_Variant"] == "crazyhouse"


def _reference_binaryio():
    rl = os.path.join(REFERENCE, "engine", "src", "rl")
    if not os.path.exists(os.path.join(rl, "binaryio.py")):
        pytest.skip("the reference's sources are not on this machine")
    for p in (REFERENCE, rl):
        if p not in sys.path:
            sys.path.insert(0, p)
    import binaryio
    return binaryio.BinaryIO


def test_the_reference_binaryio_reads_activeuci():
    BinaryIO = _reference_binaryio()
    io = BinaryIO(_exe())
    try:
        io._set_uci_param("Model_Path_Contender", "new.arab")
        io._set_uci_param("Selfplay_Games", 12)
        opts = io.get_uci_options()
    finally:
        io.stop_process()
    assert opts["Model_Path_Contender"] == "new.arab" and opts["Selfplay_Games"] == 12.0 and opts["Model_Path"] == ""
    assert len(opts) == len(_uci_table(_session(["uci"])))


@pytest.mark.parametrize("cmds,message", [
    (["arena 2"], "arena needs the producer's network (setoption name Model_Path)"),
    (["setoption name Model_Path value p.arab", "arena 2"], "arena needs the contender's network (setoption name Model_Path_Contender)"),
    (["setoption name Model_Path value p.arab", "setoption name Model_Path_Contender value c.arab", "arena"],
     "arena takes a number of games of at least 1"),
    (["setoption name Model_Path value p.arab", "setoption name Model_Path_Contender value c.arab", "arena two"],
     "arena takes a number of games of at least 1"),
    (["setoption name Model_Path value p.arab", "setoption name Model_Path_Contender value c.arab", "arena 4x"],
     "arena takes a number of games of at least 1"),
    (["setoption name Model_Path value p.arab", "setoption name Model_Path_Contender value c.arab", "arena 0"],
     "arena takes a number of games of at least 1"),
    (["setoption name Model_Path value p.arab", "setoption name Model_Path_Contender value c.arab", "arena -3"],
     "arena takes a number of games of at least 1"),
], ids=["no_producer", "no_contender", "no_n", "n_not_a_number", "n_trailing", "n_zero", "n_negative"])
def test_arena_refusals_play_nothing(tmp_path, cmds, message):
    out = _session(cmds, cwd=str(tmp_path)).splitlines()
    assert out == ["info string " + message]
    assert os.listdir(tmp_path) == []


# ------------------------------------------------------------------------------------------------------ host logic
@pytest.fixture(scope="module")
def stub_env(tmp_path_factory):
    _exe()
    so = str(tmp_path_factory.mktemp("uci_stub") / "libstub_arena.so")
    subprocess.run(["g++", "-O1", "-std=c++17", "-shared", "-fPIC", "-Wall", "-I" + os.path.join(ROOT, "include"),
                    "-I" + os.path.join(ROOT, "crazyara_b200", "csrc"), "-x", "c++",
                    os.path.join(ROOT, "tests", "uci_stub", "stub_arena.cpp"), "-o", so], check=True)
    return dict(os.environ, LD_PRELOAD=so)


def _mix(x):
    x ^= x >> 33
    x = (x * 0xff51afd7ed558ccd) & M64
    return x ^ (x >> 33)


class TwinAgent:
    """The Python twin of stub_arena.cpp, with MCTSAgent's surface as Match uses it; its calls go to one log, in the
    stand-in's words."""
    created, log = [], []

    def __init__(self, net, settings, device=0, n_trees=1, max_nodes=0):
        self.idx = len(TwinAgent.created)
        TwinAgent.created.append(self)
        self.active, self.states, self.res = [True] * n_trees, [None] * n_trees, [dict(moves=[])] * n_trees
        TwinAgent.log.append(f"create handle={self.idx} trees={n_trees} max_nodes={max_nodes} seed={int(settings.seed)} "
                             f"batch_size={int(settings.batch_size)}")

    def set_active(self, tree, active=True):
        for t in range(len(self.active)) if tree < 0 else [tree]:
            self.active[t] = bool(active)

    def set_position(self, state, tree=0):
        self.states[tree] = state

    def evaluate_board_state(self, state=None):
        act = [t for t in range(len(self.active)) if self.active[t]]
        assert act
        for t in act:
            st = self.states[t]
            key = 1469598103934665603
            for w in st.board().w:
                key = ((key ^ int(w)) * 1099511628211) & M64
            legal = st.legal_actions()
            w = [1 + _mix(key ^ ((m * 0x9E3779B97F4A7C15) & M64)) % 1000 for m in legal]
            self.res[t] = dict(moves=[st.action_to_uci(m) for m in legal], policy=np.array(w, np.float64) / float(sum(w)),
                               best_idx=int(np.argmax(w)) if w else -1, visits=np.zeros(len(w), np.uint32), nodes=0,
                               nodes_pre_search=0)
        TwinAgent.log.append(f"go handle={self.idx} trees=" + ",".join(map(str, act)))

    def result(self, tree=0):
        return self.res[tree]

    def apply_move_to_tree(self, move, tree=0):
        TwinAgent.log.append(f"apply_move handle={self.idx} tree={tree} move={int(move)}")

    def close(self):
        pass


BASE = {"UCI_Variant": "chess", "UCI_Chess960": "false", "Batch_Size": 8, "Nodes": 64, "Simulations": 0, "Dirichlet_Seed": 42,
        "Selfplay_Games": 4, "Selfplay_Seed": 3, "Reuse_Tree": "false", "Centi_Temperature": 0, "Temperature_Moves": 15,
        "Centi_Temperature_Decay": 92, "Centi_Quantile_Clipping": 0, "EPD_File_Path": "<empty>"}
EPD = ["rnbqkbnr/pppppppp/8/8/4P3/8/PPPP1PPP/RNBQKBNR b KQkq - 0 1", "r1bqkbnr/pppppppp/2n5/8/4P3/8/PPPP1PPP/RNBQKBNR w KQkq - 1 2",
       "rnbqkbnr/pp1ppppp/8/2p5/4P3/8/PPPP1PPP/RNBQKBNR w KQkq - 0 2"]
CASES = {
    "argmax": (dict(), 4),
    "temperature_quantiles_refill_reuse": (dict(UCI_Variant="crazyhouse", Centi_Temperature=60, Centi_Quantile_Clipping=25,
                                                Selfplay_Games=2, Reuse_Tree="true", Simulations=100), 6),
    "epd_odd_n_fewer_slots": (dict(EPD_File_Path="EPD", Centi_Temperature=80, Selfplay_Games=3), 5),
    "chess960": (dict(UCI_Chess960="true", Centi_Temperature=60, Selfplay_Seed=11), 4),
}


def _pgn(path):
    return re.sub(r'\[Date "[^"]*"\]', '[Date "?"]', open(path).read())


def _run_cpp(env, opts, n, cwd, producer="producer.arab", contender="contender.arab"):
    log = os.path.join(cwd, "calls.log")
    cmds = [f"setoption name Model_Path value {producer}", f"setoption name Model_Path_Contender value {contender}"]
    cmds += [f"setoption name {k} value {v}" for k, v in opts.items()] + [f"arena {n}"]
    out = _session(cmds, cwd=cwd, env=dict(env, ARA_STUB_LOG=log))
    calls = open(log).read().splitlines()
    os.unlink(log)
    return out, calls


def _run_python(opts, n, cwd, producer="producer.arab", contender="contender.arab"):
    """Match with what `arena` builds from the same options; the summary as `arena` prints it"""
    TwinAgent.created, TwinAgent.log = [], []
    orig = mt.MCTSAgent
    mt.MCTSAgent = TwinAgent
    try:
        variant = {"chess": 0, "crazyhouse": 1}[opts["UCI_Variant"]]
        st = default_settings(mt.MODE_OF_VARIANT[variant], batch_size=int(opts["Batch_Size"]), simulations=int(opts["Simulations"]),
                              nodes=int(opts["Nodes"]), seed=int(opts["Dirichlet_Seed"]))
        nets = ["p", "c"] if producer != contender else ["p", "p"]
        m = mt.Match((nets[0], st, mt.player_name(producer)), (nets[1], st, mt.player_name(contender)), n, variant=variant,
                     is960=opts["UCI_Chess960"] == "true", slots=int(opts["Selfplay_Games"]), epd_path=opts["EPD_File_Path"],
                     temperature=opts["Centi_Temperature"] / 100, temperature_moves=int(opts["Temperature_Moves"]),
                     temperature_decay=opts["Centi_Temperature_Decay"] / 100,
                     quantile_clipping=opts["Centi_Quantile_Clipping"] / 100, seed=int(opts["Selfplay_Seed"]),
                     reuse_tree=opts["Reuse_Tree"] == "true", pgn_path=os.path.join(cwd, "arena_games_gpu_0.pgn"))
        m.run()
    finally:
        mt.MCTSAgent = orig
    r = m.result
    r.write_csv(os.path.join(cwd, "arena_results.csv"))
    return ["Arena summary", f"Score of Contender vs Producer: {r}", r.verdict()], r, m


def _by_handle(calls, kind):
    return {h: [c for c in calls if c.startswith(kind) and f" handle={h} " in c + " "] for h in (0, 1)}


@pytest.mark.parametrize("case", list(CASES))
def test_arena_host_logic_equals_match(stub_env, tmp_path, case):
    extra, n = CASES[case]
    opts = dict(BASE, **extra)
    if opts["EPD_File_Path"] == "EPD":
        epd = tmp_path / "openings.epd"
        epd.write_text(EPD[0] + ";\n" + EPD[1] + "\n" + EPD[2] + ";\n")
        opts["EPD_File_Path"] = str(epd)
    cpp, py = tmp_path / "cpp", tmp_path / "py"
    cpp.mkdir()
    py.mkdir()
    out, calls = _run_cpp(stub_env, opts, n, str(cpp))
    summary, result, match = _run_python(opts, n, str(py))
    lines = out.splitlines()
    assert lines[-3:] == summary, out[-2000:]
    assert "readyok" not in lines and result.games() == n == len(match.finished)
    assert _pgn(cpp / "arena_games_gpu_0.pgn") == _pgn(py / "arena_games_gpu_0.pgn")
    assert (cpp / "arena_results.csv").read_text() == (py / "arena_results.csv").read_text()
    assert sorted(os.listdir(cpp)) == ["arena_games_gpu_0.pgn", "arena_results.csv"]
    # every finished game's PGN is printed too, as the reference's verbose writer does
    games = ["[Variant" + g for g in open(cpp / "arena_games_gpu_0.pgn").read().split("[Variant")[1:]]
    assert "\n".join(lines[:-3]) + "\n" == "".join("\n" + g for g in games) and len(games) == n
    # the same tree calls: handles with their seeds and pool sizes, the trees each go searched, the reuse calls in order
    assert [c for c in calls if c.startswith("create")] == [c for c in TwinAgent.log if c.startswith("create")]
    assert _by_handle(calls, "go ") == _by_handle(TwinAgent.log, "go ")
    applied = [c for c in calls if c.startswith("apply_move")]
    assert applied == [c for c in TwinAgent.log if c.startswith("apply_move")]
    assert bool(applied) == (opts["Reuse_Tree"] == "true")
    if case == "epd_odd_n_fewer_slots":
        fens = re.findall(r'\[FEN "([^"]*)"\]', open(cpp / "arena_games_gpu_0.pgn").read())
        assert set(fens) <= set(EPD)
    if case == "chess960":
        assert '[Variant "chess960"]' in open(cpp / "arena_games_gpu_0.pgn").read()


def test_arena_host_logic_one_network_for_equal_paths(stub_env, tmp_path):
    """Equal paths: one network, both handles on it; the games are those of two networks of the same name."""
    opts = dict(BASE, Centi_Temperature=60)
    cpp, py = tmp_path / "cpp", tmp_path / "py"
    cpp.mkdir()
    py.mkdir()
    out, _ = _run_cpp(stub_env, opts, 4, str(cpp), producer="same.arab", contender="same.arab")
    summary, _, _ = _run_python(opts, 4, str(py), producer="same.arab", contender="same.arab")
    assert out.splitlines()[-3:] == summary
    assert _pgn(cpp / "arena_games_gpu_0.pgn") == _pgn(py / "arena_games_gpu_0.pgn")
    assert "CrazyAra-B200-same-CrazyAra-B200-same: " in summary[1]


def test_the_reference_binaryio_reads_the_verdict(stub_env, tmp_path, monkeypatch):
    BinaryIO = _reference_binaryio()
    opts = dict(BASE, Centi_Temperature=60)
    monkeypatch.chdir(tmp_path)
    monkeypatch.setenv("LD_PRELOAD", stub_env["LD_PRELOAD"])
    io = BinaryIO(_exe())
    try:
        io._set_uci_param("Model_Path", "producer.arab")
        io._set_uci_param("Model_Path_Contender", "contender.arab")
        for k, v in opts.items():
            io._set_uci_param(k, v)
        replace = io.compare_new_weights(6)
    finally:
        io.stop_process()
    monkeypatch.delenv("LD_PRELOAD")
    (tmp_path / "py").mkdir()
    summary, result, _ = _run_python(opts, 6, str(tmp_path / "py"))
    assert replace == (summary[-1] == "replace")
