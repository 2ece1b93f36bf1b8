"""Self-play arena: many concurrent games per GPU, each game one device-resident search tree.

Counterpart of the reference's SelfPlay::go / generate_game loop (engine/src/rl/selfplay.cpp:192-261, :367-385) and its
"one process per GPU" deployment (engine/src/rl/README.md:84-97).  The reference plays ONE game at a time per process;
here `n_games` games advance in lock-step on one GPU: every move, all trees are searched together (one warp per tree,
their leaves share each network batch), then every game samples / plays its move on the host.  Games never interact,
so multi-GPU scaling is N independent processes -- no collective.

Per game, SelfPlay::generate_game (selfplay.cpp:192-261) with the RL defaults of DeepCrazyhouse/configs/rl_config.py:34-65:
  * the node budget of every search is jittered by +-Centi_Node_Random_Factor/2 % (adjust_node_count, :146-152);
  * the move is Agent::set_best_move's (agents/agent.cpp:38-53): argmax of the MCTS posterior, or during the first
    `temperature_moves` plies a sample from posterior^(1/T) with T = temperature * decay^ply
    (get_current_temperature, agents/config/playsettings.cpp:31-34), optionally quantile-clipped;
  * the exported policy is sharpened afterwards (sharpen_distribution with Milli_Policy_Clip_Thresh, :230-232), the
    exported q is EvalInfo::bestMoveQ[0] (traindataexporter.cpp:50-53);
  * a game may be resigned (Centi_Resign_Probability of the games, Centi_Resign_Threshold, :163-190).
Every game may have its own variant (a MODE_LICHESS build plays whatever UCI_Variant is set, selfplay.cpp:367-385):
`variant` may be a list, one entry per game (cycled).  Games may start from random lines of an EPD file (`epd_path`,
load_random_fen, selfplay.cpp:58-79).
Two options buy more games per hour (both off by default, as in rl_config):
  * quick searches (Centi_Quick_Probability, selfplay.cpp:154-159, :183-190, :214-241): each move, with probability
    `quick_probability`, a game runs a cheap search instead -- `quick_nodes`, `quick_q_value_weight`,
    `quick_dirichlet_epsilon` for that tree only (ara_search_set_tree_settings) -- and exports no sample for it;
  * opening plies from the raw network (MeanInitPly, init_starting_state_from_raw_policy, selfplay.cpp:196-202,
    :423-487): before its first search a game plays Exp(1 / `mean_init_ply`) plies (clipped by `max_init_ply`), each
    sampled from the policy of RawNetAgent, sometimes flattened (`raw_prob_temperature`).  All games that start in the
    same step share one network forward per ply.
Optional outputs: training samples (`exporter=`, crazyara_b200.export) and the games as PGN (`pgn_path=`).
"""
import os
import threading
import time

import numpy as np

from .engine import (BoardState, MCTSAgent, RawNetAgent, TERMINAL_DRAW, TERMINAL_LOSS, TERMINAL_NONE, TERMINAL_WIN,
                     default_settings, encode_planes)
from .export import BLACK_WIN, DRAWN, WHITE_WIN
from .pgn import GamePGN, result_string


def rl_settings(mode, **kw):
    """UCIConfig of the reference's RL loop (rl_config.py:34-65)."""
    base = dict(batch_size=8, nodes=800, simulations=3200, dirichlet_alpha=0.3, dirichlet_epsilon=0.25,
                node_policy_temperature=1.0, q_value_weight=0.0, mcts_solver=1)
    base.update(kw)
    return default_settings(mode, **base)


def chess960_fen(rng):
    """chess960fen() of the reference (environments/chess_related/chess960position.h:36-80): bishops on opposite
    colours, then queen and knights on random free files, then rook - king - rook on the free files left to right.
    The reference draws from the unseeded C `rand()`; here the draws come from the arena's seeded generator."""
    p = [None] * 8
    p[2 * int(rng.integers(4))] = "B"
    p[2 * int(rng.integers(4)) + 1] = "B"
    for c in "QNN":
        while True:
            loc = int(rng.integers(8))
            if p[loc] is None:
                p[loc] = c
                break
    for c in "RKR":
        p[p.index(None)] = c
    first = "".join(p)
    return f"{first.lower()}/pppppppp/8/8/8/8/PPPPPPPP/{first} w KQkq - 0 1"


def sharpen_distribution(p, thresh):
    """blazeutil.h:94-105: entries below thresh -> 0, renormalise; untouched if even the maximum is below thresh"""
    p = np.asarray(p, np.float64)
    if thresh <= 0 or len(p) == 0 or p.max() < thresh:
        return p
    q = np.where(p < thresh, 0.0, p)
    return q / q.sum()


def quantile_clip(p, quantile):
    """apply_quantile_clipping / get_quantile (agents/agent.cpp:118-127, blazeutil.h:187-212)"""
    v = np.sort(np.asarray(p, np.float32))
    if v[0] >= quantile:
        return p
    acc, thresh = np.float32(0), None
    for i in range(1, len(v)):
        acc = np.float32(acc + v[i])
        if acc >= quantile:
            thresh = float(v[i - 1]) + float(np.finfo(np.float32).eps)
            break
    if thresh is None:
        return p
    q = np.where(p < thresh, 0.0, p)
    return q / q.sum()


def set_best_move(res, ply, rng, temperature, temperature_moves, temperature_decay=0.92, quantile_clipping=0.0):
    """Agent::set_best_move (agents/agent.cpp:38-53): index of the move to play from a search result at game ply `ply`"""
    pol = res["policy"]
    if ply < temperature_moves and temperature > 0.01 and pol.sum() > 0:
        temp = temperature * temperature_decay ** ply        # get_current_temperature (playsettings.cpp:31-34)
        p = np.power(pol, 1.0 / temp)                         # apply_temperature (blazeutil.h:78-88)
        p = p / p.sum()
        if quantile_clipping != 0:                            # apply_quantile_clipping (agent.cpp:118-127)
            p = quantile_clip(p, quantile_clipping)
        return int(rng.choice(len(p), p=p))
    return int(res["best_idx"])


def init_ply_count(rng, mean_init_ply, max_init_ply):
    """Plies of a game's raw-network opening (generate_game, selfplay.cpp:196-197): size_t(Exp(1 / MeanInitPly) + 0.5),
    and beyond MaxInitPly a draw modulo MaxInitPly instead (clip_ply, :466-472).  0 when MeanInitPly is 0 (no draws)."""
    if mean_init_ply <= 0:
        return 0
    ply = int(rng.exponential(mean_init_ply) + 0.5)
    if ply > max_init_ply:
        ply = int(rng.integers(0, 1 << 31)) % max_init_ply
    return ply


def apply_raw_policy_temp(p, raw_prob_temperature, rng):
    """apply_raw_policy_temp (selfplay.cpp:474-487): with probability `raw_prob_temperature` the raw policy is flattened by
    apply_temperature (blazeutil.h:78-88) with T = 2, or T = 5 / 10 when a second draw falls below 0.25 / 0.05."""
    p = np.asarray(p, np.float64)
    if rng.random() < raw_prob_temperature:
        u = rng.random()
        temp = 10.0 if u < 0.05 else (5.0 if u < 0.25 else 2.0)
        p = np.power(p, 1.0 / temp)
        p = p / p.sum()
    return p


def leads_to_terminal(state, move):
    """State::leads_to_terminal: the position after `move` (16-bit code) ends the game"""
    after = state.clone()
    after.do_action(move)
    return after.is_terminal() != TERMINAL_NONE


def load_random_fen(path, rng):
    """load_random_fen (rl/selfplay.cpp:58-79): a line of the EPD file `path` drawn uniformly, without a trailing ';'.
    No path (None, "" or the reference's "<empty>") gives "", the variant's start position."""
    if not path or path == "<empty>":
        return ""
    with open(path) as f:
        lines = f.read().splitlines()
    if not lines:
        raise ValueError(f"{path}: no positions")
    line = lines[int(rng.integers(len(lines)))]
    return line[:-1] if line.endswith(";") else line


def start_fen(rng, variant, is960, epd_path=None):
    """FEN of a new game: a random EPD line, else a random chess960 set-up (chess only), else "" (the start position)."""
    fen = load_random_fen(epd_path, rng)
    if not fen and is960 and variant == 0:
        fen = chess960_fen(rng)
    return fen


def game_result(term, stm_at_end):
    """WHITE_WIN / BLACK_WIN / DRAWN of a game that ended with TerminalType `term`, `stm_at_end` (0 white) to move: that
    side lost (mate, variant loss) or won (variant win); everything else is a draw"""
    if term == TERMINAL_LOSS:
        return BLACK_WIN if stm_at_end == 0 else WHITE_WIN
    if term == TERMINAL_WIN:
        return WHITE_WIN if stm_at_end == 0 else BLACK_WIN
    return DRAWN


def search_concurrently(agents):
    """evaluate_board_state of every agent, each from its own host thread: the C call releases the GIL, so one agent's
    tree kernels run while another agent's network forward does"""
    errors = []

    def go(a):
        try:
            a.evaluate_board_state()
        except Exception as e:  # noqa: BLE001 -- re-raised below on the calling thread
            errors.append(e)
    threads = [threading.Thread(target=go, args=(a,)) for a in agents]
    for th in threads:
        th.start()
    for th in threads:
        th.join()
    if errors:
        raise errors[0]


class Arena:
    def __init__(self, net, settings, variant, n_games, device=0, is960=False, temperature=0.8, temperature_moves=15,
                 max_plies=512, seed=0, max_nodes=0, exporter=None, reuse_tree=False, pgn_path=None,
                 temperature_decay=0.92, quantile_clipping=0.0, policy_clip_thresh=0.01, node_random_factor=0.1,
                 resign_probability=0.9, resign_threshold=-0.9, epd_path=None, quick_probability=0.0, quick_nodes=100,
                 quick_q_value_weight=0.7, quick_dirichlet_epsilon=0.0, mean_init_ply=0, max_init_ply=0,
                 raw_prob_temperature=0.0):
        if mean_init_ply > 0 and max_init_ply <= 0:
            raise ValueError("max_init_ply must be positive when mean_init_ply is")
        if quick_probability >= 0.01 and quick_nodes <= 0:
            raise ValueError("quick_nodes must be positive when quick_probability is")
        # one variant for all games, or one per game (cycled): KOTH + Three-check mixed = variant=[2, 3]
        self.variants = [int(v) for v in variant] if isinstance(variant, (list, tuple)) else [int(variant)]
        self.variant, self.is960 = self.variants[0], is960
        self.n_games = n_games
        self.temperature, self.temperature_moves, self.max_plies = temperature, temperature_moves, max_plies
        self.temperature_decay, self.quantile_clipping = temperature_decay, quantile_clipping
        self.policy_clip_thresh, self.node_random_factor = policy_clip_thresh, node_random_factor
        self.resign_probability, self.resign_threshold = resign_probability, resign_threshold
        self.rng = np.random.default_rng(seed)
        self.epd_path = epd_path
        self.quick_probability, self.quick_nodes = quick_probability, quick_nodes
        self.quick_q_value_weight, self.quick_dirichlet_epsilon = quick_q_value_weight, quick_dirichlet_epsilon
        self.mean_init_ply, self.max_init_ply, self.raw_prob_temperature = mean_init_ply, max_init_ply, raw_prob_temperature
        # every process / group of games draws its own root noise: the trees' Dirichlet generators start from
        # settings.seed ^ tree index (TreeState::rng), so the groups get distinct seeds derived from the arena's
        import copy
        base_seed = int(settings.seed) + 1000003 * int(seed)
        if reuse_tree and max_nodes == 0:  # room for the kept subtrees of several moves before a tree starts over
            max_nodes = 8 * int(settings.simulations or settings.nodes) + 4 * int(settings.batch_size) + 64
        # `net` may be a list of networks: the games are then split into that many groups, each with its own agent
        # (own stream, own network buffers) searched from its own host thread, so that one group's tree kernels run
        # while another group's network forward does.  Trees never interact, so nothing else changes.
        nets = list(net) if isinstance(net, (list, tuple)) else [net]
        if n_games % len(nets) != 0:
            raise ValueError("n_games must be a multiple of the number of networks (game groups)")
        self.per_group = n_games // len(nets)
        if node_random_factor > 0 and max_nodes == 0 and not reuse_tree:  # room for the jittered node budget
            max_nodes = int((settings.simulations or 2 * settings.nodes) * (1 + node_random_factor)) + 8 * int(settings.batch_size) + 64
        self.agents = []
        for g, n in enumerate(nets):
            st_g = copy.copy(settings)
            st_g.seed = base_seed + 7919 * g
            self.agents.append(MCTSAgent(n, st_g, device, self.per_group, max_nodes))
        self.agent = self.agents[0]
        # the opening plies' priors come from the first group's network (every group runs the same weights)
        self.raw_agent = RawNetAgent(nets[0], settings.mode, settings.input_version) if mean_init_ply > 0 else None
        self.quick = [False] * n_games  # the tree's last search was a quick one: its limits and settings are overridden
        self.init_plies = [0] * n_games  # raw-network plies still to play before the game's first search
        self.game_variant = [self.variants[t % len(self.variants)] for t in range(n_games)]
        self.states = [self._new_state(t) for t in range(n_games)]
        self.allow_resign = [self._draw_resign() for _ in range(n_games)]
        self.plies = [0] * n_games
        self.finished = []  # (plies, terminal type, side to move at the end)
        self.resigned = 0
        self.nodes = 0
        self.reused_nodes = 0  # visits inherited from kept subtrees (EvalInfo::nodesPreSearch summed)
        self.search_ms = 0.0
        # training-sample export (crazyara_b200.export.TrainDataExporter): one sample per searched position
        self.exporter = exporter
        # Reuse_Tree (off in the reference's RL configuration, rl_config.py:56): keep the subtree of the played move
        self.reuse_tree = reuse_tree
        self.settings = settings
        self.records = [exporter.new_game() for _ in range(n_games)] if exporter is not None else None
        # games.pgn of the reference's self-play (selfplay.cpp:315-324): one GamePGN per running game
        self.pgn_path = pgn_path
        self.pgns = None
        if pgn_path is not None:
            self.pgns = [GamePGN(self.game_variant[t], is960, "CrazyAra-B200", "CrazyAra-B200") for t in range(n_games)]
            for g, st in zip(self.pgns, self.states):
                g.fen = st.fen()
        self._play_openings(range(n_games))

    def _new_state(self, t):
        # generate_game (selfplay.cpp:196-202): the opening's ply count, then the start position -- BoardState::init
        # (boardstate.cpp:260-270): chess960 games start from a random chess960 position
        self.init_plies[t] = init_ply_count(self.rng, self.mean_init_ply, self.max_init_ply)
        v = self.game_variant[t]
        return BoardState().set(start_fen(self.rng, v, self.is960, self.epd_path), self.is960, v)

    def _play_openings(self, games):
        """init_starting_state_from_raw_policy (selfplay.cpp:423-452) for the games that just started: ply by ply, one
        network forward over all of them, each game samples its move from its legal moves' priors (apply_raw_policy_temp
        first) and stops early before a move that would end the game.  The moves are game moves: they are in the PGN
        after its start FEN and count as plies of the game."""
        todo = [t for t in games if self.init_plies[t] > 0]
        while todo:
            evals = self.raw_agent.predict([self.states[t] for t in todo])
            nxt = []
            for t, (moves, priors, _) in zip(todo, evals):
                st = self.states[t]
                if len(moves) == 0:  # (a start position without a legal move: the first search ends the game)
                    self.init_plies[t] = 0
                    continue
                p = apply_raw_policy_temp(priors, self.raw_prob_temperature, self.rng)
                move = moves[int(self.rng.choice(len(p), p=p / p.sum()))]
                if leads_to_terminal(st, move):
                    self.init_plies[t] = 0
                    continue
                if self.pgns is not None:
                    self.pgns[t].play_move(st, move)
                else:
                    st.do_action(move)
                self.plies[t] += 1
                self.init_plies[t] -= 1
                if self.init_plies[t] > 0:
                    nxt.append(t)
            todo = nxt

    def _draw_resign(self):
        # SelfPlay::is_resignation_allowed (selfplay.cpp:163-168): decided once per game
        return self.resign_probability >= 0.01 and self.rng.random() < self.resign_probability

    def _search_budget(self):
        """The draws of generate_game before a search (selfplay.cpp:212-220): the random integer of adjust_node_count,
        is_quick_search, then the node jitter on the budget of that search (adjust_node_count, :146-152: nodes +=
        rand % maxRandomNodes - maxRandomNodes / 2).  Returns (node budget or None for the settings' own, quick?)."""
        nodes = int(self.settings.nodes)
        quick_on = self.quick_probability >= 0.01
        span = int(nodes * self.node_random_factor) if self.node_random_factor > 0 else 0
        rand_int = int(self.rng.integers(0, 1 << 31)) if span or quick_on else 0
        quick = quick_on and self.rng.random() < self.quick_probability
        if quick:
            nodes = int(self.quick_nodes)
            span = int(nodes * self.node_random_factor) if self.node_random_factor > 0 else 0
        if span:
            nodes += rand_int % span - span // 2
        return (nodes if span or quick else None), quick

    def _pick(self, res, ply):
        return set_best_move(res, ply, self.rng, self.temperature, self.temperature_moves, self.temperature_decay,
                             self.quantile_clipping)

    def _game_over(self, t, term, stm_at_end):
        self.finished.append((self.plies[t], term, stm_at_end))
        result = game_result(term, stm_at_end)
        if self.exporter is not None:
            self.exporter.export_game_samples(self.records[t], result)
            self.records[t] = self.exporter.new_game()
        self.states[t], self.plies[t] = self._new_state(t), 0
        self.allow_resign[t] = self._draw_resign()
        if self.pgns is not None:
            self.pgns[t].result = result_string(result)
            self.pgns[t].write(self.pgn_path)
            self.pgns[t].new_game()
            self.pgns[t].fen = self.states[t].fen()

    def step(self):
        """One move in every running game."""
        G = self.per_group
        for t, st in enumerate(self.states):
            agent, lt = self.agents[t // G], t % G
            agent.set_position(st, lt)
            nodes, quick = self._search_budget()
            if nodes is not None or self.quick[t]:  # (after a quick search the settings' budget comes back)
                agent.set_search_limits(self.settings.simulations, self.settings.nodes if nodes is None else nodes, lt)
            if quick:
                agent.set_tree_settings(self.quick_q_value_weight, self.quick_dirichlet_epsilon, lt)
            elif self.quick[t]:  # reset_search_params (selfplay.cpp:183-190)
                agent.set_tree_settings(-1.0, -1.0, lt)
            self.quick[t] = quick
        t_search = time.perf_counter()
        if len(self.agents) == 1:
            self.agent.evaluate_board_state()
            self.search_ms += self.agent.last_go_ms()
        else:
            search_concurrently(self.agents)
            self.search_ms += (time.perf_counter() - t_search) * 1e3
        planes = None
        if self.exporter is not None:  # un-normalised planes of every searched position, one GPU call
            planes = encode_planes([st.board() for st in self.states], self.settings.mode, self.settings.input_version,
                                   normalize=False)
        for t, st in enumerate(self.states):
            agent, lt = self.agents[t // G], t % G
            res = agent.result(lt)
            self.nodes += int(res["nodes"]) - int(res["nodes_pre_search"])
            self.reused_nodes += int(res["nodes_pre_search"])
            if len(res["moves"]) == 0:
                self._game_over(t, st.is_terminal(), st.side_to_move())
                continue
            idx = self._pick(res, self.plies[t])
            if self.exporter is not None and not self.quick[t]:  # a quick search exports nothing (selfplay.cpp:228)
                # sharpen_distribution (blazeutil.h:94-105) after the move has been chosen (selfplay.cpp:230-232); the
                # stored q is EvalInfo::bestMoveQ[0], not the Q of the sampled move (traindataexporter.cpp:50-53)
                self.exporter.save_sample(self.records[t], planes[t], res["moves"],
                                          sharpen_distribution(res["policy"], self.policy_clip_thresh), res["best_move_q"],
                                          st.side_to_move())
            if self.reuse_tree:
                agent.apply_move_to_tree(res["moves"][idx], lt)
            if self.pgns is not None:
                self.pgns[t].play_move(st, res["moves"][idx])
            else:
                st.do_uci(res["moves"][idx])
            self.plies[t] += 1
            term = st.is_terminal()
            if term == TERMINAL_NONE and self.allow_resign[t] and res["best_move_q"] < self.resign_threshold:
                # check_for_resignation (selfplay.cpp:170-182): the mover gives up, the side now to move has won
                self.resigned += 1
                term = TERMINAL_WIN
            if term != TERMINAL_NONE or self.plies[t] >= self.max_plies:
                self._game_over(t, term, st.side_to_move())
        self._play_openings(range(self.n_games))  # (the games started in this step: the others have no plies left)

    def run(self, min_games=0, max_steps=1 << 30, max_seconds=1e30):
        t0 = time.perf_counter()
        steps = 0
        while steps < max_steps and (time.perf_counter() - t0) < max_seconds:
            self.step()
            steps += 1
            if min_games and len(self.finished) >= min_games:
                break
            if self.exporter is not None and self.exporter.is_file_full():
                break  # SelfPlay::go (selfplay.cpp:367-385): generate games until the data file is full
        wall = time.perf_counter() - t0
        moves = steps * self.n_games
        return dict(games=len(self.finished), steps=steps, moves=moves, wall_s=wall,
                    games_per_hour=len(self.finished) / wall * 3600.0 if wall > 0 else 0.0,
                    moves_per_s=moves / wall if wall > 0 else 0.0, nodes=self.nodes, reused_nodes=self.reused_nodes,
                    nps=self.nodes / (self.search_ms / 1000.0) if self.search_ms > 0 else 0.0,
                    avg_plies=float(np.mean([g[0] for g in self.finished])) if self.finished else 0.0,
                    resigned=self.resigned)

    def close(self):
        for a in self.agents:
            a.close()


# ---------------------------------------------------------------------------------------------------------------------
# Launcher: one process per GPU, like the reference's `python rl_loop.py --device-id N` per device
# (engine/src/rl/README.md:84-97): games never interact, so the processes share nothing and need no collective.

def plan_workers(total_games, devices, out_dir):
    """What every worker process does: its GPU, its share of the concurrent games (crazyara_b200.multi.shard_range) and
    its output files, named like the reference's (selfplay.cpp:116-127: data_<device>.zarr, games_<device>.pgn with
    device = gpu_<id>)."""
    from .multi import shard_range
    plan = []
    for rank, dev in enumerate(devices):
        lo, hi = shard_range(total_games, rank, len(devices))
        if hi > lo:
            name = f"gpu_{dev}"
            plan.append(dict(rank=rank, device=int(dev), n_games=hi - lo, seed_offset=lo,
                             zarr=os.path.join(out_dir, f"data_{name}.zarr"), pgn=os.path.join(out_dir, f"games_{name}.pgn")))
    return plan


# Arena options of the launcher with the reference's defaults (optionsuci.cpp:200-217), except MeanInitPly / MaxInitPly /
# Centi_Raw_Prob_Temperature, which default to 0 here: openings from the raw network are off unless asked for
_OPTION_DEFAULTS = dict(quick_probability=0.0, quick_nodes=100, quick_q_value_weight=0.7, quick_dirichlet_epsilon=0.0,
                        mean_init_ply=0, max_init_ply=0, raw_prob_temperature=0.0)


def _worker(job, args):
    from .export import TrainDataExporter
    from .nn import NeuralNetAPI
    st = rl_settings(args.mode, batch_size=args.batch_size, nodes=args.nodes, simulations=4 * args.nodes,
                     input_version=args.input_version)
    groups = 2 if job["n_games"] % 2 == 0 and job["n_games"] >= 4 else 1
    nets = [NeuralNetAPI("gpu", job["device"], job["n_games"] // groups * args.batch_size, args.model) for _ in range(groups)]
    channels = nets[0].get_nb_input_values_total() // 64
    exporter = TrainDataExporter(job["zarr"], args.mode, channels, number_chunks=args.chunks) if args.export else None
    variants = [int(v) for v in str(args.variant).split(",")]
    # quick searches and raw-network openings (off unless their flags are given)
    options = {k: getattr(args, k) for k in _OPTION_DEFAULTS if getattr(args, k, None) is not None}
    arena = Arena(nets if groups > 1 else nets[0], st, variant=variants if len(variants) > 1 else variants[0], n_games=job["n_games"], device=job["device"],
                  is960=args.chess960, max_plies=args.max_plies, seed=args.seed + job["seed_offset"], exporter=exporter,
                  pgn_path=job["pgn"] if args.pgn else None, **options)
    res = arena.run(min_games=args.games_per_worker, max_seconds=args.seconds)
    arena.close()
    for n in nets:
        n.close()
    print(f"[{os.path.basename(job['zarr'])}] {res['games']} games, {res['moves_per_s']:.0f} moves/s, "
          f"{res['games_per_hour']:.0f} games/h, search {res['nps']:.0f} nps", flush=True)


def main(argv=None):
    import argparse
    import multiprocessing as mp
    ap = argparse.ArgumentParser(description="self-play on several GPUs: one process per GPU, independent games")
    ap.add_argument("model", help="weight blob (.arab, see crazyara_b200.weights)")
    ap.add_argument("--devices", default="0", help="comma-separated GPU ids")
    ap.add_argument("--games", type=int, default=64, help="concurrent games over all GPUs")
    ap.add_argument("--games-per-worker", type=int, default=0, help="stop a worker after this many finished games (0 = no limit)")
    ap.add_argument("--seconds", type=float, default=1e30, help="stop after this much wall time")
    ap.add_argument("--mode", default="crazyhouse", choices=["crazyhouse", "chess", "lichess"])
    ap.add_argument("--variant", default="1", help="0 chess, 1 crazyhouse, 2 king of the hill, 3 three-check; a comma-separated "
                    "list plays the variants side by side, one per game in turn (needs --mode lichess)")
    ap.add_argument("--chess960", action="store_true")
    ap.add_argument("--input-version", type=int, default=1)
    ap.add_argument("--batch-size", type=int, default=8)
    ap.add_argument("--nodes", type=int, default=800)
    ap.add_argument("--max-plies", type=int, default=512)
    ap.add_argument("--chunks", type=int, default=200, help="zarr chunks of 128 samples per data file")
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--out", default=".", help="directory of data_gpu_<id>.zarr / games_gpu_<id>.pgn")
    ap.add_argument("--no-export", dest="export", action="store_false")
    ap.add_argument("--no-pgn", dest="pgn", action="store_false")
    ap.add_argument("--quick-probability", type=float, default=_OPTION_DEFAULTS["quick_probability"],
                    help="Centi_Quick_Probability / 100: share of the moves searched with the quick settings (no sample exported)")
    ap.add_argument("--quick-nodes", type=int, default=_OPTION_DEFAULTS["quick_nodes"], help="Quick_Nodes")
    ap.add_argument("--quick-q-value-weight", type=float, default=_OPTION_DEFAULTS["quick_q_value_weight"],
                    help="Centi_Quick_Q_Value_Weight / 100")
    ap.add_argument("--quick-dirichlet-epsilon", type=float, default=_OPTION_DEFAULTS["quick_dirichlet_epsilon"],
                    help="Centi_Quick_Dirichlet_Epsilon / 100")
    ap.add_argument("--mean-init-ply", type=float, default=_OPTION_DEFAULTS["mean_init_ply"],
                    help="MeanInitPly: mean number of opening plies sampled from the raw network (0 = off)")
    ap.add_argument("--max-init-ply", type=int, default=_OPTION_DEFAULTS["max_init_ply"], help="MaxInitPly")
    ap.add_argument("--raw-prob-temperature", type=float, default=_OPTION_DEFAULTS["raw_prob_temperature"],
                    help="Centi_Raw_Prob_Temperature / 100: share of the opening plies sampled from a flattened policy")
    args = ap.parse_args(argv)
    os.makedirs(args.out, exist_ok=True)
    plan = plan_workers(args.games, [int(d) for d in args.devices.split(",")], args.out)
    ctx = mp.get_context("spawn")
    procs = [ctx.Process(target=_worker, args=(job, args)) for job in plan]
    for p in procs:
        p.start()
    for p in procs:
        p.join()
    return max((p.exitcode or 0) for p in procs) if procs else 0


if __name__ == "__main__":
    raise SystemExit(main())

