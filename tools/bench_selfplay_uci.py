"""Games per hour of `ara_uci selfplay` against `python -m crazyara_b200.selfplay` on the same workload, run alternating:
64 concurrent crazyhouse games, a synthetic RISEv2 network, Batch_Size 8, Nodes 800 (Simulations 3200, the RL
configuration's search settings, one logical search thread per tree and no epsilon exploration in both), each driver
until 64 games have ended.  The drivers differ in their process layout: the launcher splits the games into two handles
searched from two host threads, `ara_uci` runs them as the trees of one handle.  Both write their zarr and PGN files to a
temporary directory; the wall time includes each driver's start-up.  Prints the card and its power limit with one JSON line per run and a summary line.

    python tools/bench_selfplay_uci.py [--rounds 2] [--games 64]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

# the launcher's settings (selfplay.rl_settings on ara_search_default_settings, the Arena defaults): one logical search
# thread, no epsilon exploration, the RL search and play settings, no openings or quick searches
RL = {"Batch_Size": 8, "Nodes": 800, "Simulations": 3200, "Centi_Dirichlet_Epsilon": 25, "Centi_Dirichlet_Alpha": 30,
      "Centi_Node_Temperature": 100, "Centi_Q_Value_Weight": 0, "Threads": 1, "Centi_Epsilon_Greedy": 0,
      "Centi_Epsilon_Checks": 0, "Reuse_Tree": "false", "MeanInitPly": 0, "Centi_Quick_Probability": 0,
      "Milli_Policy_Clip_Thresh": 10, "Selfplay_Number_Chunks": 200, "Selfplay_Seed": 0, "Dirichlet_Seed": 42}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def run_uci(blob, games, out):
    cmds = [f"setoption name Model_Path value {blob}", f"setoption name Selfplay_Games value {games}"]
    cmds += [f"setoption name {k} value {v}" for k, v in RL.items()] + [f"selfplay {games}", "quit"]
    t0 = time.perf_counter()
    r = subprocess.run([os.path.join(ROOT, "crazyara_b200", "ara_uci")], input="\n".join(cmds) + "\n", capture_output=True,
                       text=True, cwd=out)
    wall = time.perf_counter() - t0
    if not r.stdout.rstrip().endswith("readyok"):
        raise RuntimeError(r.stdout[-2000:] + r.stderr[-2000:])
    return open(os.path.join(out, "games_gpu_0.pgn")).read().count("[Result "), wall


def run_python(blob, games, out):
    t0 = time.perf_counter()
    subprocess.run([sys.executable, "-m", "crazyara_b200.selfplay", blob, "--games", str(games), "--games-per-worker", str(games),
                    "--batch-size", "8", "--nodes", "800", "--out", out], check=True, cwd=ROOT, capture_output=True)
    wall = time.perf_counter() - t0
    return open(os.path.join(out, "games_gpu_0.pgn")).read().count("[Result "), wall


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--games", type=int, default=64)
    args = ap.parse_args()
    from crazyara_b200 import synthetic
    from crazyara_b200.weights import export_blob
    gpu = card()
    rates = {"uci": [], "python": []}
    with tempfile.TemporaryDirectory() as d:
        arch = synthetic.risev2(34, 81)
        blob = export_blob(synthetic.random_state_dict(arch, 0), arch, os.path.join(d, "risev2.arab"), input_version=10)
        for r in range(args.rounds):
            for name, fn in (("uci", run_uci), ("python", run_python)):
                out = tempfile.mkdtemp(dir=d)
                n, wall = fn(blob, args.games, out)
                rates[name].append(n / wall * 3600.0)
                print(json.dumps(dict(driver=name, round=r, games=n, wall_s=round(wall, 2), games_per_hour=round(n / wall * 3600.0, 1),
                                      gpu=gpu)), flush=True)
    print(json.dumps(dict(gpu=gpu, uci_games_per_hour=[round(x, 1) for x in rates["uci"]],
                          python_games_per_hour=[round(x, 1) for x in rates["python"]])))


if __name__ == "__main__":
    main()
