"""Matches between two networks (or two search settings): the reference's arena, the gate of its reinforcement-learning
loop that decides whether a newly trained network replaces the one producing the games (rl/rl_loop.py:153-157 ->
UCI `arena N`, uci/crazyara.cpp:366-385).  `selfplay.Arena` already names self-play here, hence `match`.

Counterpart of SelfPlay::go_arena / generate_arena_game (rl/selfplay.cpp:263-307, :387-420):
  * games come in colour-swapped pairs: game 2k starts from a new start position with the contender as White, game
    2k+1 from the same position with the producer as White (a random EPD line, load_random_fen; a random chess960
    set-up; or the variant's start position);
  * every move is the side to move's Agent::set_best_move (agents/agent.cpp:38-53) at the game's ply, with the arena's
    temperature (Centi_Temperature 60, DeepCrazyhouse/configs/rl_config.py:68-73); no resignation, no node jitter;
  * with tree reuse the mover keeps the subtree of its move, and the other player descends along the same move, except
    at a game's first ply (selfplay.cpp:297-299);
  * the contender's wins / draws / losses make a TournamentResult (rl/tournamentresult.{h,cpp}); its score above 0.5
    means `replace`, else `keep`.
The reference plays one game at a time.  Here `slots` games run in lock-step on one GPU: each player owns one search
handle with one tree per game slot, and in each step a handle searches only the trees of the games in which its player
is to move -- the others are idle (ara_search_set_active) and cost its network batch nothing.  The two handles search
from two host threads, so one player's tree kernels run while the other player's network forward does (one after the
other when both players use the same network object).
Unlike the reference, a game is adjudicated a draw after `max_plies` plies, as in self-play.
"""
import copy
import os
import time

import numpy as np

from .engine import BoardState, MCTSAgent, TERMINAL_NONE
from .export import BLACK_WIN, DRAWN, WHITE_WIN
from .pgn import GamePGN, result_string
from .selfplay import game_result, rl_settings, search_concurrently, set_best_move, start_fen

PRODUCER, CONTENDER = 0, 1
MODE_OF_VARIANT = {0: "chess", 1: "crazyhouse"}  # KOTH and three-check are played by a MODE_LICHESS build


class TournamentResult:
    """rl/tournamentresult.{h,cpp}: the result of a match from the view of player A (the contender)."""

    def __init__(self, player_a="", player_b="", wins=0, draws=0, losses=0):
        self.player_a, self.player_b = player_a, player_b
        self.wins, self.draws, self.losses = int(wins), int(draws), int(losses)

    def games(self):
        return self.wins + self.draws + self.losses

    def score(self):
        """(W + 0.5 D) / games in float32, the way score() computes it"""
        f = np.float32
        with np.errstate(invalid="ignore", divide="ignore"):
            return f(f(self.wins) + f(self.draws) * f(0.5)) / f(self.games())

    def verdict(self):
        """what the reference prints after the summary: the contender replaces the producer if it scored above 0.5"""
        return "replace" if self.score() > np.float32(0.5) else "keep"

    def __str__(self):
        """operator<<: "<A>-<B>: W - D - L [score]", the score as C++ prints a float at precision 2"""
        return f"{self.player_a}-{self.player_b}: {self.wins} - {self.draws} - {self.losses} [{'%.2g' % float(self.score())}]"

    def write_csv(self, path):
        """write_tournament_result_to_csv: appends "A,B,W,D,L" """
        with open(path, "a") as f:
            f.write(f"{self.player_a},{self.player_b},{self.wins},{self.draws},{self.losses}\n")


def player_name(model_path):
    """MCTSAgent::get_name (agents/mctsagent.cpp:266-269): engine name - version - model name; `fake` without a model"""
    if not model_path:
        return "fake"
    return "CrazyAra-B200-" + os.path.splitext(os.path.basename(str(model_path)))[0]


class Match:
    """`n_games` games of `contender` against `producer`; each player is (net, SearchSettings or None, name), the net
    None for the hash-derived fake backend.  Default settings: selfplay.rl_settings of the variant's mode."""

    def __init__(self, producer, contender, n_games, variant=1, device=0, is960=False, slots=0, epd_path=None,
                 temperature=0.6, temperature_moves=15, temperature_decay=0.92, quantile_clipping=0.0, max_plies=512,
                 seed=0, max_nodes=0, reuse_tree=False, pgn_path=None):
        self.n_games, self.variant, self.is960, self.epd_path = int(n_games), int(variant), is960, epd_path
        self.temperature, self.temperature_moves = temperature, temperature_moves
        self.temperature_decay, self.quantile_clipping, self.max_plies = temperature_decay, quantile_clipping, max_plies
        self.reuse_tree, self.pgn_path = reuse_tree, pgn_path
        self.rng = np.random.default_rng(seed)
        self.n_slots = min(int(slots) if slots else self.n_games, self.n_games)
        self.names = [producer[2], contender[2]]
        # both players on one network object (a match of two search settings): the handles share its stream and its
        # buffers, so they search one after the other
        self.shared_net = producer[0] is not None and producer[0] is contender[0]
        self.agents = []
        for i, (net, settings, _) in enumerate((producer, contender)):
            st = copy.copy(settings if settings is not None else rl_settings(MODE_OF_VARIANT.get(self.variant, "lichess")))
            # distinct root-noise generators for the two players, and for every worker process (via `seed`)
            st.seed = int(st.seed) + 1000003 * int(seed) + 7919 * i
            mn = max_nodes
            if reuse_tree and mn == 0:  # room for the kept subtrees of several moves before a tree starts over
                mn = 8 * int(st.simulations or st.nodes) + 4 * int(st.batch_size) + 64
            self.agents.append(MCTSAgent(net, st, device, self.n_slots, mn))
        self.result = TournamentResult(self.names[CONTENDER], self.names[PRODUCER])
        self.pair_fen = {}
        self.next_game = 0
        # per finished game: its number, slot, White (PRODUCER / CONTENDER), start FEN, plies, result, and per move the
        # move played, the root's visit counts and EvalInfo::nodesPreSearch
        self.finished = []
        self.steps = self.moves = self.nodes = 0
        self.slot = [None] * self.n_slots
        for s in range(self.n_slots):
            self._start(s)

    def _start(self, s):
        """the next game of the queue in slot `s`, or nothing (the slot is idle from now on)"""
        g = self.next_game
        if g >= self.n_games:
            self.slot[s] = None
            return
        self.next_game += 1
        if g % 2 == 0:
            self.pair_fen[g // 2] = start_fen(self.rng, self.variant, self.is960, self.epd_path)
        fen = self.pair_fen.pop(g // 2) if g % 2 == 1 else self.pair_fen[g // 2]
        state = BoardState().set(fen, self.is960, self.variant)
        white = CONTENDER if g % 2 == 0 else PRODUCER
        pgn = None
        if self.pgn_path is not None:
            pgn = GamePGN(self.variant, self.is960, self.names[white], self.names[1 - white])
            pgn.fen = state.fen()
        self.slot[s] = dict(game=g, white=white, state=state, fen=state.fen(), plies=0, pgn=pgn, moves=[], visits=[], pre=[])
        if self.reuse_tree:
            # MCTSAgent::clear_game_history of both players: move code 0 is never legal, so nothing of the slot's last
            # game is kept for the next search
            for a in self.agents:
                a.apply_move_to_tree(0, s)

    def _mover(self, game):
        return game["white"] if game["state"].side_to_move() == 0 else 1 - game["white"]

    def _finish(self, s, term):
        game = self.slot[s]
        res = game_result(term, game["state"].side_to_move())
        if res == DRAWN:
            self.result.draws += 1
        elif (res == WHITE_WIN) == (game["white"] == CONTENDER):
            self.result.wins += 1
        else:
            self.result.losses += 1
        if game["pgn"] is not None:
            game["pgn"].result = result_string(res)
            game["pgn"].write(self.pgn_path)
        self.finished.append(dict(game=game["game"], slot=s, white=game["white"], fen=game["fen"], plies=game["plies"],
                                  result=res, moves=game["moves"], visits=game["visits"], nodes_pre_search=game["pre"]))
        self._start(s)

    def step(self):
        """One move in every running game; False once every game is finished (and nothing was searched)."""
        running = [s for s in range(self.n_slots) if self.slot[s] is not None]
        if not running:
            return False
        searching = []
        for p, agent in enumerate(self.agents):
            n = 0
            for s in range(self.n_slots):
                on = self.slot[s] is not None and self._mover(self.slot[s]) == p
                agent.set_active(s, on)
                if on:
                    agent.set_position(self.slot[s]["state"], s)
                    n += 1
            if n:
                searching.append(agent)
        if len(searching) == 1 or self.shared_net:
            for a in searching:
                a.evaluate_board_state()
        else:
            search_concurrently(searching)
        for s in running:
            game = self.slot[s]
            st, p = game["state"], self._mover(game)
            res = self.agents[p].result(s)
            self.nodes += int(res["nodes"]) - int(res["nodes_pre_search"])
            if len(res["moves"]) == 0:
                self._finish(s, st.is_terminal())
                continue
            idx = set_best_move(res, game["plies"], self.rng, self.temperature, self.temperature_moves,
                                self.temperature_decay, self.quantile_clipping)
            uci = res["moves"][idx]
            game["moves"].append(uci)
            game["visits"].append(res["visits"])
            game["pre"].append(int(res["nodes_pre_search"]))
            action = st.uci_to_action(uci)
            if self.reuse_tree:
                self.agents[p].apply_move_to_tree(action, s)
                if game["plies"] != 0:  # State::steps_from_null() != 0 (selfplay.cpp:297-299)
                    self.agents[1 - p].apply_move_to_tree(action, s)
            if game["pgn"] is not None:
                term = game["pgn"].play_move(st, action)
            else:
                st.do_action(action)
                term = st.is_terminal()
            game["plies"] += 1
            self.moves += 1
            if term != TERMINAL_NONE or game["plies"] >= self.max_plies:
                self._finish(s, term)
        self.steps += 1
        return True

    def run(self, max_seconds=1e30):
        """Plays until every game is finished (or `max_seconds` have passed); returns the match's counters."""
        t0 = time.perf_counter()
        while time.perf_counter() - t0 < max_seconds and self.step():
            pass
        wall = time.perf_counter() - t0
        games = len(self.finished)
        return dict(games=games, steps=self.steps, moves=self.moves, nodes=self.nodes, wall_s=wall,
                    games_per_hour=games / wall * 3600.0 if wall > 0 else 0.0,
                    moves_per_s=self.moves / wall if wall > 0 else 0.0, result=self.result)

    def close(self):
        for a in self.agents:
            a.close()


# ---------------------------------------------------------------------------------------------------------------------
# Launcher: one process per GPU, as selfplay.main runs.  Game pairs are sharded, so both games of a pair run on one GPU.

def plan_workers(total_games, devices, out_dir):
    """Every worker's GPU, its games (a contiguous range of whole pairs, crazyara_b200.multi.shard_range) and its PGN."""
    from .multi import shard_range
    plan = []
    n_pairs = (int(total_games) + 1) // 2
    for rank, dev in enumerate(devices):
        lo, hi = shard_range(n_pairs, rank, len(devices))
        n = min(2 * hi, int(total_games)) - 2 * lo
        if n > 0:
            plan.append(dict(rank=rank, device=int(dev), n_games=n, seed_offset=lo,
                             pgn=os.path.join(out_dir, f"arena_games_gpu_{dev}.pgn")))
    return plan


def _worker(job, args, queue):
    from .nn import NeuralNetAPI
    st = rl_settings(args.mode, batch_size=args.batch_size, nodes=args.nodes, simulations=4 * args.nodes,
                     input_version=args.input_version)
    nets = [NeuralNetAPI("gpu", job["device"], job["n_games"] * args.batch_size, m) for m in (args.producer, args.contender)]
    match = Match((nets[0], st, player_name(args.producer)), (nets[1], st, player_name(args.contender)), job["n_games"],
                  variant=args.variant, device=job["device"], is960=args.chess960, epd_path=args.epd,
                  temperature=args.temperature, max_plies=args.max_plies, seed=args.seed + job["seed_offset"],
                  reuse_tree=args.reuse_tree, pgn_path=job["pgn"])
    res = match.run()
    match.close()
    for n in nets:
        n.close()
    r = res["result"]
    print(f"[gpu_{job['device']}] {res['games']} games, {res['moves_per_s']:.0f} moves/s, {res['games_per_hour']:.0f} games/h: {r}",
          flush=True)
    queue.put((r.wins, r.draws, r.losses))


def main(argv=None):
    import argparse
    import multiprocessing as mp
    ap = argparse.ArgumentParser(description="match of a contender network against a producer network (the RL loop's "
                                             "arena): colour-swapped game pairs, one process per GPU")
    ap.add_argument("producer", help="weight blob (.arab) of the network producing the games")
    ap.add_argument("contender", help="weight blob (.arab) of the newly trained network")
    ap.add_argument("--games", type=int, default=100)
    ap.add_argument("--devices", default="0", help="comma-separated GPU ids")
    ap.add_argument("--mode", default="crazyhouse", choices=["crazyhouse", "chess", "lichess"])
    ap.add_argument("--variant", type=int, default=1, help="0 chess, 1 crazyhouse, 2 king of the hill, 3 three-check")
    ap.add_argument("--chess960", action="store_true")
    ap.add_argument("--input-version", type=int, default=1)
    ap.add_argument("--batch-size", type=int, default=8)
    ap.add_argument("--nodes", type=int, default=800)
    ap.add_argument("--max-plies", type=int, default=512)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--epd", default=None, help="start positions: one FEN per line, a random line per game pair")
    ap.add_argument("--temperature", type=float, default=0.6)
    ap.add_argument("--reuse-tree", action="store_true")
    ap.add_argument("--out", default=".", help="directory of arena_results.csv and arena_games_gpu_<id>.pgn")
    args = ap.parse_args(argv)
    os.makedirs(args.out, exist_ok=True)
    plan = plan_workers(args.games, [int(d) for d in args.devices.split(",")], args.out)
    ctx = mp.get_context("spawn")
    queue = ctx.Queue()
    procs = [ctx.Process(target=_worker, args=(job, args, queue)) for job in plan]
    for p in procs:
        p.start()
    total = TournamentResult(player_name(args.contender), player_name(args.producer))
    failed = 0
    for p in procs:
        p.join()
        failed = max(failed, p.exitcode or 0)
    if failed:
        return failed
    for _ in procs:
        w, d, l = queue.get()
        total.wins, total.draws, total.losses = total.wins + w, total.draws + d, total.losses + l
    print("Arena summary")
    print(f"Score of Contender vs Producer: {total}")
    print(total.verdict(), flush=True)
    total.write_csv(os.path.join(args.out, "arena_results.csv"))
    return 0


if __name__ == "__main__":
    raise SystemExit(main())
