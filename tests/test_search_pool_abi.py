"""ara_search_pool_t as engine.py restates it for ctypes: every field at the offset and with the size the C compiler
gives it in include/ara_b200.h."""
import ctypes
import os
import subprocess

from tests.test_abi import ROOT, _header_struct_fields


def test_search_pool_struct_has_the_header_layout(tmp_path):
    from crazyara_b200.engine import SearchPool
    names = _header_struct_fields("ara_search_pool_t")
    assert [n for n, _ in SearchPool._fields_] == names
    lines = ['#include <stddef.h>', '#include <stdio.h>', '#include "ara_b200.h"', 'int main(void) {',
             '    printf(". 0 %zu\\n", sizeof(ara_search_pool_t));']
    lines += [f'    printf("{n} %zu %zu\\n", offsetof(ara_search_pool_t, {n}), sizeof(((ara_search_pool_t*)0)->{n}));'
              for n in names]
    (tmp_path / "layout.c").write_text("\n".join(lines + ["    return 0;", "}", ""]))
    exe = str(tmp_path / "layout")
    subprocess.run(["gcc", "-std=c99", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), str(tmp_path / "layout.c"),
                    "-o", exe], check=True)
    in_c = {}
    for line in subprocess.run([exe], check=True, capture_output=True, text=True).stdout.splitlines():
        n, offset, size = line.split()
        in_c[n] = (int(offset), int(size))
    assert ctypes.sizeof(SearchPool) == in_c["."][1]
    for n in names:
        f = getattr(SearchPool, n)
        assert (f.offset, f.size) == in_c[n], n
