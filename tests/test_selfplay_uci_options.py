"""The self-play options of `ara_uci`: the reference's names, defaults and ranges (tests/golden/selfplay_uci_options.json,
recorded from its option table with USE_RL defined), this engine's own two, and the range check of `setoption`.  `uci`
and `setoption` need no GPU."""
import json
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXE = os.path.join(ROOT, "crazyara_b200", "ara_uci")
GOLD = os.path.join(ROOT, "tests", "golden", "selfplay_uci_options.json")


def _session(cmds):
    if not os.path.exists(EXE):
        subprocess.run(["make", "-C", ROOT, "crazyara_b200/ara_uci"], check=True)
    return subprocess.run([EXE], input="\n".join(cmds + ["quit"]) + "\n", capture_output=True, text=True, timeout=60).stdout


def _options(out):
    opts = {}
    for line in out.splitlines():
        if line.startswith("option name "):
            t = line.split()
            i = t.index("type")
            name, kind = " ".join(t[2:i]), t[i + 1]
            d = t.index("default")
            if kind == "spin":
                opts[name] = [int(t[d + 1]), int(t[t.index("min") + 1]), int(t[t.index("max") + 1])]
            else:
                opts[name] = [" ".join(t[d + 1:]), None, None]
    return opts


def test_uci_lists_the_reference_self_play_options():
    want = json.load(open(GOLD))["options"]
    got = _options(_session(["uci"]))
    for name, spec in want.items():
        assert got.get(name) == spec, name
    # this engine's own: concurrent games per handle and the seed of the move sampling
    assert got["Selfplay_Games"] == [64, 1, 4096] and got["Selfplay_Seed"] == [0, 0, 2147483647]


@pytest.mark.parametrize("name,value,ok", [("Centi_Temperature", "99999", True), ("Centi_Temperature", "100000", False),
                                           ("Centi_Resign_Threshold", "-100", True), ("Centi_Resign_Threshold", "-101", False),
                                           ("Selfplay_Games", "0", False), ("Selfplay_Chunk_Size", "12x", False),
                                           ("EPD_File_Path", "openings.epd", True)])
def test_setoption_keeps_the_ranges(name, value, ok):
    out = _session([f"setoption name {name} value {value}", "uci"])
    got = _options(out)[name][0]
    if ok:
        assert str(got) == value and "info string" not in out
    else:
        assert "takes an integer in" in out and got == json.load(open(GOLD))["options"].get(name, [64])[0]


def test_selfplay_without_a_network_says_so():
    assert "selfplay needs a network" in _session(["selfplay 1"])
