"""`ara_uci selfplay N` against the Python arena (crazyara_b200.selfplay.Arena) on the GPU with synthetic RISEv2 networks:
for the same options and seed both drivers must write byte-identical data_gpu_0.zarr and games_gpu_0.pgn (the PGN's Date
header aside, which is the wall clock), and gameIdx_gpu_0.txt must hold the number of games behind the data."""
import filecmp
import os
import re
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXE = os.path.join(ROOT, "crazyara_b200", "ara_uci")

# every random feature off: argmax moves, no node jitter, no resignation, no openings, no quick searches, no root noise
OFF = {"Centi_Node_Random_Factor": 0, "Centi_Resign_Probability": 0, "Centi_Temperature": 0, "Temperature_Moves": 0,
       "MeanInitPly": 0, "Centi_Quick_Probability": 0, "Centi_Dirichlet_Epsilon": 0, "Milli_Policy_Clip_Thresh": 0}
# the reference's defaults (node jitter, resignation, temperature sampling) with quick searches and the RL root noise
DEFAULTS_QUICK = {"Centi_Quick_Probability": 30, "Quick_Nodes": 16, "MeanInitPly": 0, "Centi_Dirichlet_Epsilon": 25,
                  "Milli_Policy_Clip_Thresh": 10}
# the defaults of ara_uci: the reference's (openings of MeanInitPly 15 plies from the raw network included), Reuse_Tree on
DEFAULTS = {"Centi_Quick_Probability": 30, "Quick_Nodes": 16, "Centi_Dirichlet_Epsilon": 25, "Reuse_Tree": "true"}
BASE = {"Batch_Size": 8, "Nodes": 64, "Simulations": 0, "Reuse_Tree": "false", "Selfplay_Games": 8, "Selfplay_Seed": 5,
        "Selfplay_Number_Chunks": 40, "Selfplay_Chunk_Size": 128}


def _blob(tmp_path, in_channels=34, policy_channels=81, name="risev2.arab"):
    from crazyara_b200.weights import export_blob
    from oracle import net as onet
    arch = onet.arch_risev2(in_channels, policy_channels)
    return export_blob(onet.make_state_dict(arch, 0), arch, str(tmp_path / name), input_version=10)


def _options(extra):
    o = {"UCI_Variant": "crazyhouse", "UCI_Chess960": "false", "Centi_CPuct_Init": 250, "CPuct_Base": 19652,
         "Centi_Node_Temperature": 170, "Centi_Dirichlet_Epsilon": 0, "Centi_Dirichlet_Alpha": 20, "Centi_Q_Value_Weight": 100,
         "Centi_Q_Veto_Delta": 40, "Dirichlet_Seed": 42, "Threads": 2, "Centi_Epsilon_Greedy": 5, "Centi_Epsilon_Checks": 1,
         "Input_Version": 0,
         "Centi_Node_Random_Factor": 10, "Centi_Quick_Dirichlet_Epsilon": 0, "Centi_Quick_Probability": 0,
         "Centi_Quick_Q_Value_Weight": 70, "Quick_Nodes": 100, "Centi_Raw_Prob_Temperature": 25, "MaxInitPly": 30,
         "MeanInitPly": 15, "Centi_Resign_Probability": 90, "Centi_Resign_Threshold": -90, "Milli_Policy_Clip_Thresh": 0,
         "Centi_Temperature": 80, "Temperature_Moves": 15, "Centi_Temperature_Decay": 92, "Centi_Quantile_Clipping": 0}
    o.update(BASE)
    o.update(extra)
    return o


def _run_uci(blob, opts, games, cwd):
    if not os.path.exists(EXE):
        subprocess.run(["make", "-C", ROOT, "crazyara_b200/ara_uci"], check=True)
    cmds = [f"setoption name Model_Path value {blob}"] + [f"setoption name {k} value {v}" for k, v in opts.items()]
    os.makedirs(cwd, exist_ok=True)
    out = subprocess.run([EXE], input="\n".join(cmds + [f"selfplay {games}", "quit"]) + "\n", capture_output=True, text=True,
                         timeout=1200, cwd=cwd).stdout
    assert "error" not in out and out.rstrip().endswith("readyok"), out[-3000:]
    assert "games/min" in out
    return out


def _run_arena(blob, opts, games, cwd):
    """Arena with what `selfplay` builds from the same options (the settings of CrazyAra::is_ready in ara_uci)"""
    from crazyara_b200.engine import MODES, default_settings
    from crazyara_b200.export import TrainDataExporter
    from crazyara_b200.nn import NeuralNetAPI
    from crazyara_b200.selfplay import Arena
    variant = {"crazyhouse": 1, "chess": 0, "kingofthehill": 2}[opts["UCI_Variant"]]
    mode = {1: "crazyhouse", 0: "chess", 2: "lichess"}[variant]
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
    n = int(opts["Selfplay_Games"])
    os.makedirs(cwd, exist_ok=True)
    net = NeuralNetAPI("gpu", 0, n * B, blob)
    exporter = TrainDataExporter(os.path.join(cwd, "data_gpu_0.zarr"), MODES[mode], net.get_nb_input_values_total() // 64,
                                 number_chunks=int(opts["Selfplay_Number_Chunks"]), chunk_size=int(opts["Selfplay_Chunk_Size"]))
    arena = Arena(net, st, variant=variant, n_games=n, is960=opts["UCI_Chess960"] == "true", seed=int(opts["Selfplay_Seed"]),
                  exporter=exporter, pgn_path=os.path.join(cwd, "games_gpu_0.pgn"), reuse_tree=opts["Reuse_Tree"] == "true",
                  temperature=opts["Centi_Temperature"] / 100, temperature_moves=int(opts["Temperature_Moves"]),
                  temperature_decay=opts["Centi_Temperature_Decay"] / 100, quantile_clipping=opts["Centi_Quantile_Clipping"] / 100,
                  policy_clip_thresh=opts["Milli_Policy_Clip_Thresh"] / 1000, node_random_factor=opts["Centi_Node_Random_Factor"] / 100,
                  resign_probability=opts["Centi_Resign_Probability"] / 100, resign_threshold=opts["Centi_Resign_Threshold"] / 100,
                  quick_probability=opts["Centi_Quick_Probability"] / 100, quick_nodes=int(opts["Quick_Nodes"]),
                  quick_q_value_weight=opts["Centi_Quick_Q_Value_Weight"] / 100,
                  quick_dirichlet_epsilon=opts["Centi_Quick_Dirichlet_Epsilon"] / 100, mean_init_ply=opts["MeanInitPly"],
                  max_init_ply=int(opts["MaxInitPly"]), raw_prob_temperature=opts["Centi_Raw_Prob_Temperature"] / 100)
    res = arena.run(min_games=games)
    arena.close()
    net.close()
    return res


def _tree(d):
    return sorted(os.path.relpath(os.path.join(r, f), d) for r, _, fs in os.walk(d) for f in fs)


def _pgn(path):
    return re.sub(r'\[Date "[^"]*"\]', '[Date "?"]', open(path).read())


def _games(path):
    return open(path).read().count("[Result ")


def _exported_games(cpp):
    """games whose samples are in the store: the last game index start_indices has written"""
    from crazyara_b200.export import read_dataset
    start = read_dataset(os.path.join(cpp, "data_gpu_0.zarr"), "start_indices")
    return int(max(i for i in range(len(start)) if i == 0 or start[i] > 0)), start


def _compare(cpp, py):
    """every file of the store and the PGN byte for byte; gameIdx: the games behind the data"""
    zc, zp = os.path.join(cpp, "data_gpu_0.zarr"), os.path.join(py, "data_gpu_0.zarr")
    assert _tree(zc) == _tree(zp)
    for f in _tree(zc):
        assert filecmp.cmp(os.path.join(zc, f), os.path.join(zp, f), shallow=False), f
    assert _pgn(os.path.join(cpp, "games_gpu_0.pgn")) == _pgn(os.path.join(py, "games_gpu_0.pgn"))
    assert open(os.path.join(cpp, "gameIdx_gpu_0.txt")).read() == str(_exported_games(cpp)[0])


@pytest.mark.gpu
@pytest.mark.parametrize("extra", [OFF, DEFAULTS_QUICK, DEFAULTS], ids=["random_off", "defaults_quick", "defaults_openings_reuse"])
def test_selfplay_matches_the_arena_byte_for_byte(tmp_path, extra):
    blob = _blob(tmp_path)
    opts = _options(extra)
    out = _run_uci(blob, opts, 8, str(tmp_path / "cpp"))
    res = _run_arena(blob, opts, 8, str(tmp_path / "py"))
    assert res["games"] >= 8
    _compare(str(tmp_path / "cpp"), str(tmp_path / "py"))
    cpp = str(tmp_path / "cpp")
    n_games = _games(os.path.join(cpp, "games_gpu_0.pgn"))
    assert out.count("games/min") == n_games == res["games"]
    if extra is DEFAULTS:  # openings are game moves: PlyCount counts them, the samples do not
        _, start = _exported_games(cpp)
        counts = [int(c) for c in re.findall(r'\[PlyCount "(\d+)"\]', open(os.path.join(cpp, "games_gpu_0.pgn")).read())]
        samples = [int(start[i + 1] - start[i]) for i in range(n_games)]
        assert all(c >= s for c, s in zip(counts, samples)) and sum(counts) > sum(samples)


@pytest.mark.gpu
def test_selfplay_0_stops_when_the_data_file_is_full(tmp_path):
    from crazyara_b200.export import read_dataset
    blob = _blob(tmp_path)
    opts = _options(dict(OFF, Selfplay_Number_Chunks=1, Selfplay_Chunk_Size=48))
    _run_uci(blob, opts, 0, str(tmp_path / "cpp"))
    _run_arena(blob, opts, 0, str(tmp_path / "py"))
    _compare(str(tmp_path / "cpp"), str(tmp_path / "py"))
    exported, start = _exported_games(str(tmp_path / "cpp"))
    # the last exported game filled the file; the one before it had not (games of the same move after it are PGN only)
    assert start[exported] == 48 and start[exported - 1] < 48
    assert _games(os.path.join(str(tmp_path / "cpp"), "games_gpu_0.pgn")) >= exported


@pytest.mark.gpu
@pytest.mark.parametrize("variant", ["chess960", "kingofthehill"])
def test_selfplay_chess960_and_king_of_the_hill(tmp_path, variant):
    if variant == "chess960":
        blob = _blob(tmp_path, 39, 76)
        extra = {"UCI_Variant": "chess", "UCI_Chess960": "true", "Input_Version": 1}
    else:
        blob = _blob(tmp_path, 63, 84)
        extra = {"UCI_Variant": "kingofthehill", "Input_Version": 1}
    opts = _options(dict(DEFAULTS_QUICK, **extra))
    _run_uci(blob, opts, 8, str(tmp_path / "cpp"))
    _run_arena(blob, opts, 8, str(tmp_path / "py"))
    _compare(str(tmp_path / "cpp"), str(tmp_path / "py"))
    text = open(os.path.join(str(tmp_path / "cpp"), "games_gpu_0.pgn")).read()
    assert ('[Variant "chess960"]' if variant == "chess960" else '[Variant "kingofthehill"]') in text


@pytest.mark.gpu
def test_selfplay_refuses_a_fully_connected_policy_head(tmp_path):
    from crazyara_b200 import synthetic
    from crazyara_b200.weights import export_blob
    arch = synthetic.classic(synthetic.risev2(34, 81), 2272)
    blob = export_blob(synthetic.random_state_dict(arch, 0), arch, str(tmp_path / "fc.arab"), input_version=10)
    cmds = [f"setoption name Model_Path value {blob}", "setoption name Batch_Size value 8", "setoption name Selfplay_Games value 2",
            "selfplay 1", "quit"]
    out = subprocess.run([EXE], input="\n".join(cmds) + "\n", capture_output=True, text=True, timeout=300, cwd=str(tmp_path)).stdout
    assert "fully-connected policy head" in out and "readyok" not in out
