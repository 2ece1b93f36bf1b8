"""Games per hour and moves per second of `ara_uci arena N` against crazyara_b200.match.Match on the same workload, one
GPU, run alternating: a contender and a producer synthetic RISEv2 network (seeds 1 and 0), N crazyhouse games all
running at once (Selfplay_Games N), the RL loop's search settings (Batch_Size 8, Nodes 800, Simulations 3200, Dirichlet
epsilon 0.25 alpha 0.3, node temperature 1, Q-value weight 0; one logical search thread per tree, no epsilon
exploration) and the arena's temperature 0.6 for the first 15 plies.  Both drivers play the same games for the same seed,
so they take the same number of steps (one move in every running game); the time per step is each driver's wall time
over that count.  ara_uci's wall time is its whole process, Match's starts with the loading of its networks.  The card's
name, power limit and SM clock are read in the same run and printed with every line.

    python tools/bench_arena_uci.py [--rounds 1] [--games 64] [--nodes 800]
"""
import argparse
import json
import os
import re
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    if q.returncode != 0 or not q.stdout.strip():
        raise RuntimeError("nvidia-smi found no GPU: " + q.stderr.strip())
    return q.stdout.strip().splitlines()[0]


def options(games, nodes):
    return {"UCI_Variant": "crazyhouse", "Batch_Size": 8, "Nodes": nodes, "Simulations": 4 * nodes, "Centi_Dirichlet_Epsilon": 25,
            "Centi_Dirichlet_Alpha": 30, "Centi_Node_Temperature": 100, "Centi_Q_Value_Weight": 0, "Threads": 1,
            "Centi_Epsilon_Greedy": 0, "Centi_Epsilon_Checks": 0, "Reuse_Tree": "false", "Selfplay_Games": games,
            "Selfplay_Seed": 0, "Dirichlet_Seed": 42, "Centi_Temperature": 60, "Temperature_Moves": 15}


def run_uci(producer, contender, opts, games, out):
    cmds = [f"setoption name Model_Path value {producer}", f"setoption name Model_Path_Contender value {contender}"]
    cmds += [f"setoption name {k} value {v}" for k, v in opts.items()] + [f"arena {games}", "quit"]
    t0 = time.perf_counter()
    r = subprocess.run([os.path.join(ROOT, "crazyara_b200", "ara_uci")], input="\n".join(cmds) + "\n", capture_output=True,
                       text=True, cwd=out)
    wall = time.perf_counter() - t0
    if r.stdout.rstrip().splitlines()[-1:] not in (["keep"], ["replace"]):
        raise RuntimeError(r.stdout[-2000:] + r.stderr[-2000:])
    text = open(os.path.join(out, "arena_games_gpu_0.pgn")).read()
    moves = sum(int(c) for c in re.findall(r'\[PlyCount "(\d+)"\]', text))
    return dict(games=text.count("[Result "), moves=moves, wall_s=wall, verdict=r.stdout.rstrip().splitlines()[-1])


def run_python(producer, contender, opts, games, out):
    from crazyara_b200.match import Match, player_name
    from crazyara_b200.nn import NeuralNetAPI
    from crazyara_b200.selfplay import rl_settings
    B, nodes = int(opts["Batch_Size"]), int(opts["Nodes"])
    st = rl_settings("crazyhouse", batch_size=B, nodes=nodes, simulations=4 * nodes, seed=int(opts["Dirichlet_Seed"]))
    t0 = time.perf_counter()
    nets = [NeuralNetAPI("gpu", 0, games * B, p) for p in (producer, contender)]
    m = Match((nets[0], st, player_name(producer)), (nets[1], st, player_name(contender)), games, variant=1, slots=games,
              temperature=opts["Centi_Temperature"] / 100, temperature_moves=int(opts["Temperature_Moves"]), seed=int(opts["Selfplay_Seed"]),
              pgn_path=os.path.join(out, "arena_games_gpu_0.pgn"))
    res = m.run()
    m.close()
    for n in nets:
        n.close()
    wall = time.perf_counter() - t0
    return dict(games=res["games"], moves=res["moves"], wall_s=wall, steps=res["steps"], verdict=res["result"].verdict())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=1)
    ap.add_argument("--games", type=int, default=64)
    ap.add_argument("--nodes", type=int, default=800)
    args = ap.parse_args()
    from crazyara_b200 import synthetic
    from crazyara_b200.weights import export_blob
    gpu = card()
    opts = options(args.games, args.nodes)
    with tempfile.TemporaryDirectory() as d:
        arch = synthetic.risev2(34, 81)
        producer = export_blob(synthetic.random_state_dict(arch, 0), arch, os.path.join(d, "producer.arab"), input_version=10)
        contender = export_blob(synthetic.random_state_dict(arch, 1), arch, os.path.join(d, "contender.arab"), input_version=10)
        for r in range(args.rounds):
            runs = {}
            for name, fn in (("python_match", run_python), ("uci_arena", run_uci)):
                out = tempfile.mkdtemp(dir=d)
                runs[name] = fn(producer, contender, opts, args.games, out)
            steps = runs["python_match"]["steps"]  # the same games, so the same steps in both drivers
            for name, x in runs.items():
                print(json.dumps(dict(driver=name, round=r, games=x["games"], moves=x["moves"], steps=steps, wall_s=round(x["wall_s"], 2),
                                      games_per_hour=round(x["games"] / x["wall_s"] * 3600.0, 1),
                                      moves_per_s=round(x["moves"] / x["wall_s"], 1), ms_per_step=round(1000.0 * x["wall_s"] / steps, 1),
                                      verdict=x["verdict"], gpu=gpu, gpu_after=card())), flush=True)
            if runs["python_match"]["moves"] != runs["uci_arena"]["moves"]:
                print(json.dumps(dict(warning="the drivers played different games")), flush=True)


if __name__ == "__main__":
    main()
