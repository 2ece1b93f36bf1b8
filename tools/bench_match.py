"""Games per hour and moves per second of a match (crazyara_b200.match.Match: two networks, each handle searching only
the games its player is to move in) against a self-play arena (crazyara_b200.selfplay.Arena) with the same search
settings and the same number of concurrent games, on one GPU.  The card's name and power limit are printed with the
numbers.
    python tools/bench_match.py [--games 64] [--batch-size 8] [--nodes 800] [--max-plies 160] [--seconds 600]
The match plays all its games; the arena is timed for as long as the match took.  Neither resigns or jitters the node
budget, both sample with temperature 0.6 for the first 15 plies."""
import argparse
import os
import subprocess
import sys
import tempfile
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from crazyara_b200 import synthetic  # noqa: E402
from crazyara_b200.match import Match  # noqa: E402
from crazyara_b200.nn import NeuralNetAPI  # noqa: E402
from crazyara_b200.selfplay import Arena, rl_settings  # noqa: E402
from crazyara_b200.weights import export_blob  # noqa: E402


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                         capture_output=True, text=True, check=True).stdout.strip()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--games", type=int, default=64)
    ap.add_argument("--batch-size", type=int, default=8)
    ap.add_argument("--nodes", type=int, default=800)
    ap.add_argument("--max-plies", type=int, default=160)
    ap.add_argument("--seconds", type=float, default=600.0, help="cap on the match's wall time")
    args = ap.parse_args()
    n, B = args.games, args.batch_size
    st = rl_settings("crazyhouse", batch_size=B, nodes=args.nodes, simulations=4 * args.nodes)
    arch = synthetic.risev2(34, 81)
    d = tempfile.mkdtemp()
    blobs = [export_blob(synthetic.random_state_dict(arch, s), arch, os.path.join(d, f"w{s}.arab"), input_version=10)
             for s in (0, 1)]
    nets = [NeuralNetAPI("gpu", 0, n * B, b) for b in blobs]

    match = Match((nets[0], st, "producer"), (nets[1], st, "contender"), n, variant=1, max_plies=args.max_plies, seed=1)
    t0 = time.perf_counter()
    while time.perf_counter() - t0 < args.seconds and match.step():
        pass
    m_wall = time.perf_counter() - t0
    m_games, m_moves, m_steps = len(match.finished), match.moves, match.steps
    match.close()

    arena = Arena(nets[0], st, variant=1, n_games=n, temperature=0.6, max_plies=args.max_plies, seed=1,
                  node_random_factor=0.0, resign_probability=0.0)
    arena.run(max_steps=2)  # warm-up: graph captures
    g0, t0, steps = len(arena.finished), time.perf_counter(), 0
    while time.perf_counter() - t0 < m_wall:
        arena.step()
        steps += 1
    a_wall = time.perf_counter() - t0
    a_games, a_moves = len(arena.finished) - g0, steps * n
    arena.close()
    for net in nets:
        net.close()

    print(f"GPU: {card()}")
    print(f"crazyhouse RISEv2 (synthetic weights), Batch_Size {B}, Nodes {args.nodes}, {n} concurrent games, "
          f"max {args.max_plies} plies")
    print(f"match: {m_games} games, {m_steps} steps in {m_wall:.1f} s: {m_games / m_wall * 3600:.0f} games/h, "
          f"{m_moves / m_wall:.0f} moves/s, {m_wall / max(m_steps, 1) * 1e3:.1f} ms/step")
    print(f"self-play arena: {a_games} games, {steps} steps in {a_wall:.1f} s: {a_games / a_wall * 3600:.0f} games/h, "
          f"{a_moves / a_wall:.0f} moves/s, {a_wall / max(steps, 1) * 1e3:.1f} ms/step")


if __name__ == "__main__":
    main()
