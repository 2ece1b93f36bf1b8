"""Host-side mirror of the reference's engine surface over the C-ABI (include/ara_b200.h):

  BoardState  <-> engine/src/environments/chess_related/boardstate.h  (State interface, engine/src/state.h:287-509)
  SearchSettings / default_settings <-> agents/config/searchsettings.h + uci/optionsuci.cpp defaults
  MCTSAgent   <-> agents/mctsagent.{h,cpp}: evaluate_board_state() runs the device-resident search
  RawNetAgent <-> agents/rawnetagent.{h,cpp}: the network's policy alone, no search
  EvalInfo (dict) <-> evalinfo.{h,cpp}

Same names and argument meaning as the reference so that tests read like the reference's own.  No CPU fallback.
"""
import ctypes

import numpy as np

from ._lib import AraError, check, lib

VARIANTS = {"chess": 0, "standard": 0, "fischerandom": 0, "chess960": 0, "crazyhouse": 1, "kingofthehill": 2, "koth": 2,
            "3check": 3, "threecheck": 3}
MODES = {"crazyhouse": 0, "chess": 1, "lichess": 2}
TERMINAL_LOSS, TERMINAL_DRAW, TERMINAL_WIN, TERMINAL_CUSTOM, TERMINAL_NONE = 0, 1, 2, 3, 4


class AraBoard(ctypes.Structure):
    _fields_ = [("w", ctypes.c_ulonglong * 16)]


class SearchSettings(ctypes.Structure):
    _fields_ = [("batch_size", ctypes.c_int), ("dirichlet_epsilon", ctypes.c_float), ("dirichlet_alpha", ctypes.c_float),
                ("node_policy_temperature", ctypes.c_float), ("q_value_weight", ctypes.c_float),
                ("q_veto_delta", ctypes.c_float), ("cpuct_init", ctypes.c_float), ("cpuct_base", ctypes.c_float),
                ("mcts_solver", ctypes.c_int), ("virtual_style", ctypes.c_int), ("virtual_mix_threshold", ctypes.c_uint),
                ("simulations", ctypes.c_uint), ("nodes", ctypes.c_uint), ("seed", ctypes.c_ulonglong),
                ("mode", ctypes.c_int), ("input_version", ctypes.c_int), ("threads", ctypes.c_int),
                ("epsilon_greedy_counter", ctypes.c_int), ("epsilon_checks_counter", ctypes.c_int), ("reserved", ctypes.c_int)]


class TimeControl(ctypes.Structure):
    """ara_time_control_t: what MCTSAgent::run_mcts_search hands to the ThreadManager (agents/mctsagent.cpp:350-352)."""
    _fields_ = [("movetime_ms", ctypes.c_double), ("update_interval_ms", ctypes.c_double), ("overall_nps", ctypes.c_double),
                ("safe_remaining_ms", ctypes.c_double), ("move_overhead_ms", ctypes.c_double),
                ("last_value_eval", ctypes.c_float), ("in_game", ctypes.c_int), ("can_prolong", ctypes.c_int)]


class TimeReport(ctypes.Structure):
    _fields_ = [("early_stopped", ctypes.c_int), ("prolonged", ctypes.c_int), ("saved_ms", ctypes.c_double),
                ("elapsed_ms", ctypes.c_double), ("value_eval", ctypes.c_float)]


class SearchPool(ctypes.Structure):
    _fields_ = [("nodes", ctypes.c_longlong), ("edges", ctypes.c_longlong), ("mapped_nodes", ctypes.c_longlong),
                ("mapped_edges", ctypes.c_longlong), ("cap_nodes", ctypes.c_longlong), ("cap_edges", ctypes.c_longlong),
                ("mapped_bytes", ctypes.c_longlong), ("spare_bytes", ctypes.c_longlong), ("grows", ctypes.c_longlong), ("growing", ctypes.c_int)]


def early_stopping(tc, remaining_ms, node_count, max_q_is_max_visits, first_visits, second_visits, q_first, q_second):
    """ThreadManager::early_stopping as a pure function: 0 keep searching, 1 'max nodes' rule, 2 'cannot catch up' rule."""
    return _L().ara_time_early_stopping(ctypes.byref(tc), float(remaining_ms), int(node_count), int(max_q_is_max_visits),
                                        int(first_visits), int(second_visits), float(q_first), float(q_second))


def continue_search(tc, remaining_ms, value_eval, checked, last_value_eval):
    """ThreadManager::continue_search as a pure function; returns (prolong?, checked', last_value_eval')."""
    c, l = ctypes.c_int(checked), ctypes.c_float(last_value_eval)
    r = _L().ara_time_continue_search(ctypes.byref(tc), float(remaining_ms), float(value_eval), ctypes.byref(c), ctypes.byref(l))
    return bool(r), c.value, l.value


class SearchResult(ctypes.Structure):
    _fields_ = [("n_moves", ctypes.c_int), ("no_visit_idx", ctypes.c_int), ("best_idx", ctypes.c_int),
                ("node_type", ctypes.c_int), ("pv_len", ctypes.c_int), ("root_value", ctypes.c_float),
                ("best_move_q", ctypes.c_float), ("visit_sum", ctypes.c_uint), ("free_visits", ctypes.c_uint),
                ("iterations", ctypes.c_uint), ("evals", ctypes.c_uint), ("tree_nodes", ctypes.c_int),
                ("error", ctypes.c_int), ("nodes_pre_search", ctypes.c_uint), ("sum_select_k", ctypes.c_ulonglong), ("sum_depth", ctypes.c_ulonglong),
                ("moves", ctypes.c_uint16 * 512), ("visits", ctypes.c_uint32 * 512), ("q", ctypes.c_float * 512),
                ("prior", ctypes.c_float * 512), ("policy", ctypes.c_double * 512), ("pv", ctypes.c_uint16 * 256)]


class NodeView(ctypes.Structure):
    """ara_node_view_t: one node of the device-resident tree (Node's getters, node.h:345-460)."""
    _fields_ = [("node_id", ctypes.c_int), ("parent", ctypes.c_int), ("parent_child_idx", ctypes.c_int), ("n_moves", ctypes.c_int),
                ("no_visit_idx", ctypes.c_int), ("node_type", ctypes.c_int), ("flags", ctypes.c_int), ("checkmate_idx", ctypes.c_int),
                ("end_in_ply", ctypes.c_int), ("n_unsolved", ctypes.c_int), ("repetition", ctypes.c_int), ("pad_", ctypes.c_int),
                ("visit_sum", ctypes.c_uint), ("real_visits", ctypes.c_uint), ("free_visits", ctypes.c_uint), ("value", ctypes.c_float),
                ("value_sum", ctypes.c_double), ("key", ctypes.c_ulonglong), ("moves", ctypes.c_uint16 * 512),
                ("child", ctypes.c_int32 * 512), ("visits", ctypes.c_uint32 * 512), ("q", ctypes.c_float * 512),
                ("prior", ctypes.c_float * 512), ("vl", ctypes.c_uint8 * 512), ("child_type", ctypes.c_uint8 * 512)]


_SIGS = False


def _L():
    global _SIGS
    L = lib()
    if not _SIGS:
        vp, ci, cs = ctypes.c_void_p, ctypes.c_int, ctypes.c_char_p
        L.ara_state_create.restype = vp
        L.ara_state_create.argtypes = [cs, ci, ci]
        L.ara_state_clone.restype = vp
        L.ara_state_clone.argtypes = [vp]
        L.ara_state_destroy.argtypes = [vp]
        L.ara_state_do_move.argtypes = [vp, ctypes.c_ushort]
        L.ara_state_do_uci.argtypes = [vp, cs]
        L.ara_state_board.argtypes = [vp, vp]
        L.ara_state_history.argtypes = [vp, ctypes.POINTER(vp), ctypes.POINTER(vp), ctypes.POINTER(ci)]
        L.ara_state_fen.argtypes = [vp, cs, ci]
        L.ara_state_legal_moves.argtypes = [vp, vp]
        L.ara_state_side_to_move.argtypes = [vp]
        L.ara_state_is_terminal.argtypes = [vp]
        L.ara_state_in_check.argtypes = [vp]
        L.ara_state_move_to_san.argtypes = [vp, ctypes.c_ushort, ci, ctypes.c_char_p]
        L.ara_move_to_uci.argtypes = [ctypes.c_ushort, ci, cs]
        L.ara_board_from_fen.argtypes = [cs, ci, ci, vp]
        L.ara_encode_planes.argtypes = [vp, ci, ci, ci, ci, vp]
        L.ara_legal_moves.argtypes = [vp, ci, vp, vp, vp, vp]
        L.ara_search_default_settings.argtypes = [vp, ci]
        L.ara_search_create.restype = vp
        L.ara_search_create.argtypes = [vp, vp, ci, ci, ci]
        L.ara_search_destroy.argtypes = [vp]
        L.ara_search_set_position.argtypes = [vp, ci, vp, vp, vp, ci]
        L.ara_search_go.argtypes = [vp]
        L.ara_search_begin.argtypes = [vp]
        L.ara_search_step.argtypes = [vp, ci]
        L.ara_search_node.argtypes = [vp, ci, ci, vp]
        L.ara_search_result.argtypes = [vp, ci, vp]
        L.ara_search_set_profile.argtypes = [vp, ci]
        L.ara_search_apply_move.argtypes = [vp, ci, ctypes.c_ushort]
        L.ara_search_set_time_control.argtypes = [vp, vp]
        L.ara_search_stop.argtypes = [vp]
        L.ara_search_time_report.argtypes = [vp, vp]
        L.ara_time_early_stopping.argtypes = [vp, ctypes.c_double, ctypes.c_uint, ci, ctypes.c_uint, ctypes.c_uint,
                                              ctypes.c_float, ctypes.c_float]
        L.ara_time_continue_search.argtypes = [vp, ctypes.c_double, ctypes.c_float, vp, vp]
        L.ara_search_set_movetime.argtypes = [vp, ctypes.c_double]
        L.ara_search_set_limits.argtypes = [vp, ci, ctypes.c_uint, ctypes.c_uint]
        L.ara_search_set_tree_settings.argtypes = [vp, ci, ctypes.c_float, ctypes.c_float]
        L.ara_search_set_active.argtypes = [vp, ci, ci]
        L.ara_search_profile.argtypes = [vp] + [vp] * 4
        L.ara_search_last_go_ms.restype = ctypes.c_double
        L.ara_search_last_go_ms.argtypes = [vp]
        L.ara_search_launch_count.restype = ctypes.c_longlong
        L.ara_search_launch_count.argtypes = [vp]
        L.ara_search_compaction_count.restype = ctypes.c_longlong
        L.ara_search_compaction_count.argtypes = [vp]
        L.ara_search_pool.argtypes = [vp, ci, vp]
        _SIGS = True
    return L


def default_settings(mode, **kw):
    s = SearchSettings()
    _L().ara_search_default_settings(ctypes.byref(s), MODES[mode] if isinstance(mode, str) else mode)
    for k, v in kw.items():
        if not hasattr(s, k):
            raise AttributeError(k)
        setattr(s, k, v)
    return s


def move_to_uci(move, is960=False):
    b = ctypes.create_string_buffer(8)
    _L().ara_move_to_uci(int(move), int(is960), b)
    return b.value.decode()


class BoardState:
    """State interface of the reference (engine/src/state.h:287-509) for chess / chess960 / crazyhouse / KOTH / 3check."""

    def __init__(self, _h=None):
        self._h = _h
        self.variant = 0
        self.is960 = False

    # State::set(fenStr, isChess960, variant) / State::init(variant, isChess960)
    def set(self, fenStr, isChess960=False, variant=0):
        self.close()
        v = VARIANTS[variant] if isinstance(variant, str) else int(variant)
        h = _L().ara_state_create(fenStr.encode() if fenStr else None, v, int(isChess960))
        if not h:
            raise AraError(lib().ara_last_error().decode())
        self._h, self.variant, self.is960 = h, v, bool(isChess960)
        return self

    def init(self, variant=0, isChess960=False):
        return self.set("", isChess960, variant)

    def clone(self):
        c = BoardState(_L().ara_state_clone(self._h))
        c.variant, c.is960 = self.variant, self.is960
        return c

    def close(self):
        if self._h:
            _L().ara_state_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def fen(self):
        b = ctypes.create_string_buffer(256)
        check(_L().ara_state_fen(self._h, b, 256))
        return b.value.decode()

    def legal_actions(self):
        arr = (ctypes.c_uint16 * 512)()
        n = _L().ara_state_legal_moves(self._h, arr)
        return list(arr[:n])

    def action_to_uci(self, action):
        return move_to_uci(action, self.is960)

    def uci_to_action(self, uci):
        for a in self.legal_actions():
            if move_to_uci(a, self.is960) == uci:
                return a
        raise AraError(f"illegal move {uci} in {self.fen()}")

    def do_action(self, action):
        check(_L().ara_state_do_move(self._h, int(action)))

    def in_check(self):
        return bool(_L().ara_state_in_check(self._h))

    def action_to_san(self, action, leads_to_win=False):
        """State::action_to_san -> pgn_move (board.cpp:277-359); `action` may be the 16-bit code or a UCI string."""
        if isinstance(action, str):
            action = self.uci_to_action(action)
        b = ctypes.create_string_buffer(16)
        check(_L().ara_state_move_to_san(self._h, int(action), int(leads_to_win), b))
        return b.value.decode()

    def do_uci(self, *moves):
        for u in moves:
            check(_L().ara_state_do_uci(self._h, u.encode()))
        return self

    def side_to_move(self):
        return _L().ara_state_side_to_move(self._h)

    def is_terminal(self):
        return _L().ara_state_is_terminal(self._h)

    def board(self):
        b = AraBoard()
        check(_L().ara_state_board(self._h, ctypes.byref(b)))
        return b

    def history(self):
        k, r, n = ctypes.c_void_p(), ctypes.c_void_p(), ctypes.c_int()
        check(_L().ara_state_history(self._h, ctypes.byref(k), ctypes.byref(r), ctypes.byref(n)))
        return k, r, n.value

    def get_state_planes(self, normalize, mode, version):
        """State::get_state_planes(normalize, inputPlanes, version): GPU plane encoder through host buffers."""
        return encode_planes([self.board()], mode, version, normalize)[0]


def planes_channels(mode, version):
    """Input channels of the network for a (mode, input version) pair, as planes_channels of csrc/planes_dev.cuh."""
    c = {(0, 1): 34, (0, 2): 51, (0, 3): 64, (1, 1): 39, (1, 3): 52, (2, 1): 63, (2, 2): 63, (2, 3): 80}.get((mode, version))
    if c is None:
        raise AraError(f"no input representation for mode {mode}, version {version}")
    return c


def encode_planes(boards, mode, version, normalize=True):
    m = MODES[mode] if isinstance(mode, str) else mode
    n = len(boards)
    arr = (AraBoard * n)(*boards)
    out = np.full((n, planes_channels(m, version), 8, 8), np.nan, np.float32)
    check(_L().ara_encode_planes(arr, n, m, version, int(bool(normalize)), out.ctypes.data))
    return out


def legal_moves_gpu(boards):
    """Device move generator for a list of boards: (moves per board, terminal types, policy indices per board)."""
    n = len(boards)
    arr = (AraBoard * n)(*boards)
    moves = np.zeros((n, 512), np.uint16)
    counts = np.zeros(n, np.int32)
    term = np.zeros(n, np.int32)
    pidx = np.zeros((n, 512), np.int32)
    check(_L().ara_legal_moves(arr, n, moves.ctypes.data, counts.ctypes.data, term.ctypes.data, pidx.ctypes.data))
    return ([moves[i, :counts[i]].tolist() for i in range(n)], term.tolist(),
            [pidx[i, :counts[i]].tolist() for i in range(n)])


def value_to_centipawn(value, mode):
    """value_to_centipawn (evalinfo.cpp:102-110) with VALUE_TO_CENTI_PARAM 1.4 (MODE_CHESS) or 1.2 (constants.h:90-92)"""
    value = np.float32(value)
    if abs(value) >= 1:
        return int(np.sign(value)) * 9999
    param = np.float32(1.4 if (MODES[mode] if isinstance(mode, str) else mode) == 1 else 1.2)
    return int(-(np.sign(value) * np.log(np.float32(1) - abs(value)) / np.log(param)) * np.float32(100))


class RawNetAgent:
    """RawNetAgent of the reference (agents/rawnetagent.cpp:45-83): the move the network's policy prefers, without a
    search.  `net` is a crazyara_b200.nn.NeuralNetAPI; `mode` / `input_version` are the input representation the
    searches of the same network use (SearchSettings.mode / input_version)."""

    def __init__(self, net, mode, input_version):
        if net is None:
            raise AraError("RawNetAgent needs a network")
        if not net.is_policy_map():  # legal_moves_gpu gives policy-map indices; classic labels are not mapped yet
            raise AraError("RawNetAgent: the network has a fully-connected policy head (classic labels); only policy-map "
                           "networks are supported")
        self.net, self.mode, self.input_version = net, mode, input_version

    def predict(self, states):
        """For every state: its legal moves (16-bit codes), their priors (entries of the soft-maxed policy) and the value.
        One forward per network batch over all the states (ara_net_predict_priors)."""
        boards = [s.board() for s in states]
        moves, _, pidx = legal_moves_gpu(boards)
        planes = encode_planes(boards, self.mode, self.input_version)
        out = []
        B = self.net.get_batch_size()
        for lo in range(0, len(states), B):
            hi = min(lo + B, len(states))
            counts = np.array([len(m) for m in moves[lo:hi]], np.int32)
            idx = np.zeros((hi - lo, max(1, int(counts.max()))), np.int32)
            for i, p in enumerate(pidx[lo:hi]):
                idx[i, :len(p)] = p
            value = np.zeros(hi - lo, np.float32)
            priors = np.zeros(idx.shape, np.float32)
            self.net.predict_priors(np.ascontiguousarray(planes[lo:hi]), idx, counts, value, priors, n=hi - lo)
            out += [(moves[i], priors[i - lo, :counts[i - lo]].copy(), float(value[i - lo])) for i in range(lo, hi)]
        return out

    def evaluate_board_state(self, state):
        """EvalInfo dict of RawNetAgent::evaluate_board_state: a single legal move is returned without a forward, else the
        argmax of the legal moves' priors with the score of the network's value (depth, seldepth and nodes 1)."""
        legal = state.legal_actions()
        if not legal:
            raise AraError(f"no legal move in {state.fen()}")
        if len(legal) == 1:
            m = state.action_to_uci(legal[0])
            return dict(moves=[m], policy=np.ones(1), best_idx=0, best_move=m, pv=[m], centipawns=value_to_centipawn(0.0, self.mode),
                        depth=0, seldepth=0, nodes=0)
        (codes, priors, value), = self.predict([state])
        best = int(np.argmax(priors))
        moves = [state.action_to_uci(a) for a in codes]
        return dict(moves=moves, policy=priors, best_idx=best, best_move=moves[best], pv=[moves[best]], value=value,
                    centipawns=value_to_centipawn(value, self.mode), depth=1, seldepth=1, nodes=1)


def result_to_dict(r, uci_fn):
    """EvalInfo dict of a SearchResult; uci_fn spells a 16-bit move code."""
    k = r.n_moves
    d = dict(moves=[uci_fn(m) for m in r.moves[:k]], visits=np.array(r.visits[:k], np.uint32),
             q=np.array(r.q[:k], np.float32), prior=np.array(r.prior[:k], np.float32),
             policy=np.array(r.policy[:k], np.float64), root_value=r.root_value, visit_sum=r.visit_sum,
             free_visits=r.free_visits, nodes=r.visit_sum - r.free_visits, best_idx=r.best_idx,
             best_move_q=r.best_move_q, node_type=r.node_type, pv_len=r.pv_len, iterations=r.iterations, evals=r.evals,
             tree_nodes=r.tree_nodes, sum_select_k=r.sum_select_k, sum_depth=r.sum_depth, nodes_pre_search=r.nodes_pre_search, error=r.error,
             pv=[uci_fn(m) for m in r.pv[:r.pv_len]])
    if k > 0 and r.best_idx >= 0:
        d["best_move"] = d["moves"][r.best_idx]
    return d


class MCTSAgent:
    """MCTSAgent of the reference (agents/mctsagent.h): evaluate_board_state() searches the given state(s).

    net: crazyara_b200.nn.NeuralNetAPI whose batch size is >= n_trees * settings.batch_size, or None for the
    hash-derived fake backend (search-parity tests)."""

    def __init__(self, net, settings, device=0, n_trees=1, max_nodes=0):
        self.net = net
        self.settings = settings
        self.n_trees = n_trees
        h = _L().ara_search_create(net._h if net is not None else None, ctypes.byref(settings), device, n_trees, max_nodes)
        if not h:
            raise AraError(lib().ara_last_error().decode())
        self._h = h
        self._states = [None] * n_trees

    def set_position(self, state, tree=0):
        k, r, n = state.history()
        b = state.board()
        check(_L().ara_search_set_position(self._h, tree, ctypes.byref(b), k, r, n))
        self._states[tree] = state

    def evaluate_board_state(self, state=None):
        """Runs the search; returns the EvalInfo dict of tree 0 (use results() for all trees)."""
        if state is not None:
            self.set_position(state, 0)
        check(_L().ara_search_go(self._h))
        return self.result(0)

    # ---- SearchThread / Node surface (searchthread.h, node.h): drive the search one mini-batch at a time, read the tree
    def begin(self, state=None):
        """MCTSAgent::evaluate_board_state up to the first mini-batch (roots created or taken over, evaluated, noised)."""
        if state is not None:
            self.set_position(state, 0)
        check(_L().ara_search_begin(self._h))

    def thread_iteration(self, n_batches=1):
        """SearchThread::thread_iteration n times; returns the number of trees whose search loop has not ended."""
        rc = _L().ara_search_step(self._h, int(n_batches))
        if rc < 0:
            raise AraError(lib().ara_last_error().decode())
        return rc

    def node(self, node_id=-1, tree=0):
        """Read-only view of one node (Node's getters): dict with the children's moves / visits / Q / priors / node ids."""
        v = NodeView()
        check(_L().ara_search_node(self._h, tree, int(node_id), ctypes.byref(v)))
        st = self._states[tree]
        k = v.n_moves
        return dict(node_id=v.node_id, parent=v.parent, n_moves=k, no_visit_idx=v.no_visit_idx, node_type=v.node_type,
                    is_terminal=bool(v.flags & 1), has_nn_results=bool(v.flags & 2), is_playout_node=bool(v.flags & 4),
                    visits=v.visit_sum, real_visits=v.real_visits, free_visits=v.free_visits, value=v.value, key=v.key,
                    moves=[move_to_uci(m, st.is960 if st is not None else False) for m in v.moves[:k]],
                    child=list(v.child[:k]), child_visits=np.array(v.visits[:k], np.uint32), q=np.array(v.q[:k], np.float32),
                    prior=np.array(v.prior[:k], np.float32), virtual_loss=np.array(v.vl[:k], np.uint8))

    def result(self, tree=0):
        r = SearchResult()
        check(_L().ara_search_result(self._h, tree, ctypes.byref(r)))
        st = self._states[tree]
        is960 = st.is960 if st is not None else False
        d = result_to_dict(r, lambda m: move_to_uci(m, is960))
        ms = _L().ara_search_last_go_ms(self._h)
        d["elapsed_ms"] = ms
        # EvalInfo::calculate_nps (evalinfo.cpp:73-85): (nodes - nodesPreSearch) / elapsed
        d["nps"] = (d["nodes"] - d["nodes_pre_search"]) / (ms / 1000.0) if ms > 0 else 0.0
        return d

    def results(self):
        return [self.result(t) for t in range(self.n_trees)]

    def apply_move_to_tree(self, move, tree=0):
        """MCTSAgent::apply_move_to_tree: tell the tree which move was played (UCI string of the position last searched,
        or the 16-bit move code); the next search on the resulting position continues on the kept subtree."""
        if isinstance(move, str):
            move = self._states[tree].uci_to_action(move)
        check(_L().ara_search_apply_move(self._h, tree, int(move)))

    def set_time_control(self, tc):
        """ThreadManager heuristics for the following searches (TimeControl), None = off."""
        check(_L().ara_search_set_time_control(self._h, ctypes.byref(tc) if tc is not None else None))

    def time_report(self):
        r = TimeReport()
        check(_L().ara_search_time_report(self._h, ctypes.byref(r)))
        return dict(early_stopped=r.early_stopped, prolonged=r.prolonged, saved_ms=r.saved_ms, elapsed_ms=r.elapsed_ms,
                    value_eval=r.value_eval)

    def stop(self):
        """UCI `stop`: may be called from another thread while evaluate_board_state runs on this agent."""
        check(_L().ara_search_stop(self._h))

    def set_movetime(self, ms):
        """SearchLimits::movetime: following searches also stop after `ms` of wall time (0 = off)."""
        check(_L().ara_search_set_movetime(self._h, float(ms)))

    def set_search_limits(self, simulations, nodes, tree=-1):
        """SearchLimits::simulations / nodes of the following searches of `tree` (-1 = all trees) instead of the settings'."""
        check(_L().ara_search_set_limits(self._h, int(tree), int(simulations), int(nodes)))

    def set_tree_settings(self, q_value_weight=-1.0, dirichlet_epsilon=-1.0, tree=-1):
        """Q-value weight and Dirichlet epsilon of the following searches of `tree` (-1 = all trees) instead of the
        settings'; a negative value restores the settings' value (ara_search_set_tree_settings)."""
        check(_L().ara_search_set_tree_settings(self._h, int(tree), float(q_value_weight), float(dirichlet_epsilon)))

    def set_active(self, tree, active=True):
        """Leave `tree` (-1 = all trees) out of the following searches, or take it back in (ara_search_set_active).  An
        idle tree keeps its statistics, its root noise generator, its last result and a subtree kept by
        apply_move_to_tree, and costs the network batch nothing."""
        check(_L().ara_search_set_active(self._h, int(tree), int(bool(active))))

    def set_profile(self, on=True):
        check(_L().ara_search_set_profile(self._h, int(on)))

    def profile(self):
        """Device time of the last go split into select / network / apply (ms) and the number of network forwards."""
        a, b, c, n = ctypes.c_double(), ctypes.c_double(), ctypes.c_double(), ctypes.c_longlong()
        check(_L().ara_search_profile(self._h, ctypes.byref(a), ctypes.byref(b), ctypes.byref(c), ctypes.byref(n)))
        return dict(select_ms=a.value, net_ms=b.value, apply_ms=c.value, net_forwards=n.value)

    def last_go_ms(self):
        return _L().ara_search_last_go_ms(self._h)

    def launch_count(self):
        return _L().ara_search_launch_count(self._h)

    def compaction_count(self):
        """kept subtrees moved to the front of the node pools so far (ara_search_compaction_count)"""
        return _L().ara_search_compaction_count(self._h)

    def pool(self, tree=0):
        """The tree's pools (ara_search_pool): nodes / edges in use, the capacity mapped, the reservation (cap), the device
        bytes mapped for both sets, how often the handle's pools grew, and whether they grow with the tree."""
        r = SearchPool()
        check(_L().ara_search_pool(self._h, int(tree), ctypes.byref(r)))
        return {n: getattr(r, n) for n, _ in SearchPool._fields_}

    def close(self):
        if getattr(self, "_h", None):
            _L().ara_search_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
