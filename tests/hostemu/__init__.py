"""Builds and loads the 1-lane host emulation of the device rules/search code (test scaffolding only)."""
import ctypes
import os
import subprocess

from crazyara_b200.engine import SearchResult, result_to_dict

_HERE = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.dirname(os.path.dirname(_HERE))
_LIB = None


def lib():
    global _LIB
    if _LIB is None:
        so = os.path.join(_HERE, "libhostemu.so")
        srcs = [os.path.join(_HERE, "hostemu.cpp")] + [os.path.join(_ROOT, "crazyara_b200", "csrc", f) for f in
                                                       os.listdir(os.path.join(_ROOT, "crazyara_b200", "csrc"))
                                                       if f.endswith((".cuh", ".h"))]
        if not os.path.exists(so) or any(os.path.getmtime(s) > os.path.getmtime(so) for s in srcs):
            subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wall", "-ffp-contract=off",
                            "-I" + os.path.join(_ROOT, "crazyara_b200", "csrc"), "-I" + os.path.join(_ROOT, "include"),
                            "-x", "c++", os.path.join(_HERE, "hostemu.cpp"), "-o", so], check=True)
        L = ctypes.CDLL(so)
        L.he_new.restype = ctypes.c_void_p
        L.he_new.argtypes = [ctypes.c_char_p, ctypes.c_int, ctypes.c_int]
        L.he_clone.restype = ctypes.c_void_p
        for n in ("he_free", "he_clone", "he_in_check", "he_repetition", "he_terminal"):
            getattr(L, n).argtypes = [ctypes.c_void_p]
        L.he_legal_moves.argtypes = [ctypes.c_void_p, ctypes.c_void_p]
        L.he_move_uci.argtypes = [ctypes.c_void_p, ctypes.c_uint16, ctypes.c_char_p]
        L.he_uci_move.restype = ctypes.c_uint16
        L.he_uci_move.argtypes = [ctypes.c_void_p, ctypes.c_char_p]
        L.he_do_move.argtypes = [ctypes.c_void_p, ctypes.c_uint16]
        L.he_fen.argtypes = [ctypes.c_void_p, ctypes.c_char_p]
        L.he_key.restype = ctypes.c_ulonglong
        L.he_key.argtypes = [ctypes.c_void_p]
        L.he_key_scratch.restype = ctypes.c_ulonglong
        L.he_key_scratch.argtypes = [ctypes.c_void_p]
        L.he_policy_index.argtypes = [ctypes.c_void_p, ctypes.c_uint16]
        L.he_planes.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_void_p]
        L.he_board.restype = ctypes.c_void_p
        L.he_board.argtypes = [ctypes.c_void_p]
        _LIB = L
    return _LIB


class HeState:
    def __init__(self, fen, variant, is960=False, _h=None):
        self.L = lib()
        self.h = _h if _h is not None else self.L.he_new(fen.encode(), variant, int(is960))
        if not self.h:
            raise ValueError("bad fen")

    def __del__(self):
        if getattr(self, "h", None):
            self.L.he_free(self.h)
            self.h = None

    def clone(self):
        return HeState(None, 0, _h=self.L.he_clone(self.h))

    def legal_moves(self):
        arr = (ctypes.c_uint16 * 512)()
        n = self.L.he_legal_moves(self.h, arr)
        return list(arr[:n])

    def uci(self, m):
        b = ctypes.create_string_buffer(8)
        self.L.he_move_uci(self.h, m, b)
        return b.value.decode()

    def move_from_uci(self, s):
        m = self.L.he_uci_move(self.h, s.encode())
        if m == 0:
            raise ValueError("illegal " + s)
        return m

    def do_move(self, m):
        self.L.he_do_move(self.h, m)

    def fen(self):
        b = ctypes.create_string_buffer(256)
        self.L.he_fen(self.h, b)
        return b.value.decode()

    def key(self):
        return self.L.he_key(self.h)

    def key_scratch(self):
        return self.L.he_key_scratch(self.h)

    def terminal(self):
        return self.L.he_terminal(self.h)

    def repetition(self):
        return self.L.he_repetition(self.h)

    def policy_index(self, m):
        return self.L.he_policy_index(self.h, m)

    def planes(self, mode, version, normalize):
        import numpy as np
        out = np.full((80, 8, 8), np.nan, np.float32)
        c = self.L.he_planes(self.h, mode, version, int(normalize), out.ctypes.data)
        return out[:c]

    def board_bytes(self):
        return ctypes.string_at(self.L.he_board(self.h), 128)


class HeSearch:
    """Host emulation of the GPU search, driven like oracle.search.Search."""

    def __init__(self, settings, max_nodes=1 << 16, max_edges=1 << 21):
        import numpy as np
        self.np = np
        self.L = L = lib()
        L.he_search_new.restype = ctypes.c_void_p
        L.he_search_new.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int]
        for n in ("he_search_free", "he_search_channels", "he_search_n_labels", "he_search_create_mini_batch",
                  "he_search_done", "he_search_error"):
            getattr(L, n).argtypes = [ctypes.c_void_p]
        L.he_search_planes.restype = ctypes.c_void_p
        L.he_search_planes.argtypes = [ctypes.c_void_p]
        L.he_search_set_root.argtypes = [ctypes.c_void_p, ctypes.c_void_p]
        L.he_search_root_results.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]
        L.he_search_apply_results.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]
        L.he_search_batch_keys.argtypes = [ctypes.c_void_p, ctypes.c_void_p]
        L.he_search_create_mini_batch_t.argtypes = [ctypes.c_void_p, ctypes.c_int]
        L.he_search_thread_done.argtypes = [ctypes.c_void_p, ctypes.c_int]
        L.he_search_apply_results_t.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p]
        L.he_search_planes_t.restype = ctypes.c_void_p
        L.he_search_planes_t.argtypes = [ctypes.c_void_p, ctypes.c_int]
        L.he_search_batch_keys_t.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p]
        L.he_search_result.restype = ctypes.POINTER(SearchResult)
        L.he_search_result.argtypes = [ctypes.c_void_p]
        L.he_fake_eval.argtypes = [ctypes.c_ulonglong, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p]
        L.he_search_apply_move.argtypes = [ctypes.c_void_p, ctypes.c_uint16]
        L.he_search_time_stats.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]
        assert L.he_sizeof_result() == ctypes.sizeof(SearchResult)
        self.settings = settings
        self.h = L.he_search_new(ctypes.byref(settings), max_nodes, max_edges)
        self.channels = L.he_search_channels(self.h)
        self.n_labels = L.he_search_n_labels(self.h)
        self.batch = settings.batch_size

    def __del__(self):
        if getattr(self, "h", None):
            self.L.he_search_free(self.h)
            self.h = None

    def _planes(self, n):
        ptr = self.L.he_search_planes(self.h)
        arr = self.np.ctypeslib.as_array(ctypes.cast(ptr, ctypes.POINTER(ctypes.c_float)),
                                         shape=(self.batch, self.channels, 8, 8))
        return arr[:n].copy()

    def _keys(self, n):
        k = self.np.zeros(max(n, 1), self.np.uint64)
        self.L.he_search_batch_keys(self.h, k.ctypes.data)
        return k[:n]

    def apply_move(self, move):
        """MCTSAgent::apply_move_to_tree (16-bit move code of the device rules)."""
        self.L.he_search_apply_move(self.h, int(move))

    def time_stats(self):
        """collect_time_stats of the current tree (what the ThreadManager rules read)."""
        i, f = (ctypes.c_uint * 5)(), (ctypes.c_float * 3)()
        self.L.he_search_time_stats(self.h, i, f)
        return dict(node_count=i[0], first_visits=i[1], second_visits=i[2], max_q_is_max_visits=int(i[3]), valid=int(i[4]),
                    q_first=f[0], q_second=f[1], value_eval=f[2])

    def _eval_thread(self, t, n, net_fn, with_keys):
        np = self.np
        ptr = self.L.he_search_planes_t(self.h, t)
        planes = np.ctypeslib.as_array(ctypes.cast(ptr, ctypes.POINTER(ctypes.c_float)),
                                       shape=(self.batch, self.channels, 8, 8))[:n].copy()
        if not with_keys:
            v, p = net_fn(planes)
        else:
            k = np.zeros(max(n, 1), np.uint64)
            self.L.he_search_batch_keys_t(self.h, t, k.ctypes.data)
            v, p = net_fn(planes, k[:n])
        return np.ascontiguousarray(v, np.float32), np.ascontiguousarray(p, np.float32)

    def _run_two_threads(self, net_fn, with_keys):
        """Threads = 2: the schedule of oracle/mcts.h as the device runs it -- the loop condition lives inside
        create_mini_batch (`done`), a thread whose select finds it set produces an empty batch; one more turn of both
        threads drains the batch still in flight."""
        L, h, np = self.L, self.h, self.np
        pending = [None, None]

        def sel(t):
            n = L.he_search_create_mini_batch_t(h, t)
            pending[t] = None if L.he_search_thread_done(h, t) else n

        def bk(t):
            if pending[t] is None:
                return
            n = pending[t]
            v, p = self._eval_thread(t, n, net_fn, with_keys) if n > 0 else (np.zeros(1, np.float32), np.zeros(1, np.float32))
            L.he_search_apply_results_t(h, t, v.ctypes.data, p.ctypes.data)
            pending[t] = None
        sel(0)
        sel(1)
        while pending[0] is not None or pending[1] is not None:
            for t in (0, 1):
                bk(t)
                sel(t)

    def run(self, he_state, net_fn, with_keys=False, threads=1):
        L, h, np = self.L, self.h, self.np
        n = L.he_search_set_root(h, he_state.h)
        self.reused = n == 2
        if n:
            if n == 2:  # kept subtree: no root evaluation, only the noise / opening step
                v, p = np.zeros(1, np.float32), np.zeros(1, np.float32)
            else:
                v, p = net_fn(self._planes(1), self._keys(1)) if with_keys else net_fn(self._planes(1))
                v, p = np.ascontiguousarray(v, np.float32), np.ascontiguousarray(p, np.float32)
            L.he_search_root_results(h, v.ctypes.data, p.ctypes.data)
            if threads == 2:
                self._run_two_threads(net_fn, with_keys)
            while threads != 2:
                n = L.he_search_create_mini_batch(h)
                if L.he_search_done(h):
                    break
                if n > 0:
                    v, p = net_fn(self._planes(n), self._keys(n)) if with_keys else net_fn(self._planes(n))
                    v, p = np.ascontiguousarray(v, np.float32), np.ascontiguousarray(p, np.float32)
                else:
                    v, p = np.zeros(1, np.float32), np.zeros(1, np.float32)
                L.he_search_apply_results(h, v.ctypes.data, p.ctypes.data)
        return result_to_dict(L.he_search_result(h).contents, he_state.uci)
