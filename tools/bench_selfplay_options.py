"""Games per hour of the self-play arena (crazyara_b200.selfplay.Arena) with and without its two options that trade search
for throughput, in the same run on one GPU: quick searches (quick_probability 0 vs 0.5) and openings from the raw
network (off vs mean_init_ply 15).  The card's name and power limit are printed with the numbers.
    python tools/bench_selfplay_options.py [--games 64] [--batch-size 8] [--nodes 800] [--window 60] [--rounds 3]
Each setting has an arena of its own; the arenas take turns, `--window` seconds each, `--rounds` times, so that a
drift of the clocks or of the other work on the machine falls on every setting alike.  A window counts the games that
finished in it, whenever they started."""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from crazyara_b200 import synthetic  # noqa: E402
from crazyara_b200.nn import NeuralNetAPI  # noqa: E402
from crazyara_b200.selfplay import Arena, rl_settings  # noqa: E402
from crazyara_b200.weights import export_blob  # noqa: E402

SETTINGS = {"plain": {}, "quick 0.5": dict(quick_probability=0.5),
            "raw openings 15": dict(mean_init_ply=15, max_init_ply=30, raw_prob_temperature=0.25)}


def card():
    return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                          capture_output=True, text=True, check=True).stdout.strip()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--games", type=int, default=64)
    ap.add_argument("--batch-size", type=int, default=8)
    ap.add_argument("--nodes", type=int, default=800)
    ap.add_argument("--max-plies", type=int, default=512)
    ap.add_argument("--window", type=float, default=60.0, help="seconds per setting and round")
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    n, B = args.games, args.batch_size
    st = rl_settings("crazyhouse", batch_size=B, nodes=args.nodes, simulations=4 * args.nodes)
    arch = synthetic.risev2(34, 81)
    blob = export_blob(synthetic.random_state_dict(arch, 0), arch, os.path.join(tempfile.mkdtemp(), "w.arab"), input_version=10)
    net = NeuralNetAPI("gpu", 0, n * B, blob)
    arenas = {k: Arena(net, st, variant=1, n_games=n, max_plies=args.max_plies, seed=1, **kw) for k, kw in SETTINGS.items()}
    for a in arenas.values():
        a.run(max_steps=2)  # warm-up: graph captures
    games = {k: 0 for k in arenas}
    wall = {k: 0.0 for k in arenas}
    for _ in range(args.rounds):
        for k, a in arenas.items():
            g0, t0 = len(a.finished), time.perf_counter()
            a.run(max_seconds=args.window)
            wall[k] += time.perf_counter() - t0
            games[k] += len(a.finished) - g0
    info = card()
    for k in arenas:
        print(json.dumps(dict(setting=k, games=games[k], seconds=round(wall[k], 1), games_per_hour=round(games[k] / wall[k] * 3600.0, 1),
                              n_games=n, batch_size=B, nodes=args.nodes, card=info)), flush=True)
    for a in arenas.values():
        a.close()
    net.close()


if __name__ == "__main__":
    main()
