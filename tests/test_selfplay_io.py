"""The C++ self-play writers and generator (crazyara_b200/host/selfplay_io.h) on the CPU: recorded games written through
TrainDataExporter and GamePGN must give files byte-identical to the Python writers' (crazyara_b200.export,
crazyara_b200.pgn) for the same records, and NumpyRandom must draw what numpy.random.default_rng draws for the calls the
self-play arena makes."""
import filecmp
import os
import subprocess

import numpy as np
import pytest

from crazyara_b200.engine import TERMINAL_NONE, BoardState, move_to_uci
from crazyara_b200.export import TrainDataExporter
from crazyara_b200.labels import uci_labels
from crazyara_b200.pgn import GamePGN, result_string

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def driver(tmp_path_factory):
    import crazyara_b200
    crazyara_b200.lib()  # (the driver links the library for the game state and SAN)
    exe = str(tmp_path_factory.mktemp("selfplay_io") / "selfplay_io_driver")
    lib_dir = os.path.join(ROOT, "crazyara_b200")
    subprocess.run(["g++", "-O2", "-std=c++17", "-Wall", "-I" + os.path.join(ROOT, "include"), "-I" + os.path.join(lib_dir, "host"),
                    "-I" + os.path.join(lib_dir, "csrc"), os.path.join(ROOT, "tests", "selfplay_io_driver.cpp"), "-o", exe,
                    "-L" + lib_dir, "-lara_b200", "-Wl,-rpath," + lib_dir, "-L/usr/local/cuda/lib64",
                    "-Wl,-rpath,/usr/local/cuda/lib64"], check=True)
    return exe


# (variant, chess960, label mode, planes channels)
GAMES = [(1, False, 0, 34), (0, True, 1, 39), (2, False, 2, 63), (0, False, 1, 39)]


def _record_games(variant, is960, n_games, seed):
    """random legal games with made-up search outputs: (fen, moves, samples, result) per game"""
    rng = np.random.default_rng(seed)
    games = []
    for g in range(n_games):
        fen = ""
        if is960:
            from crazyara_b200.selfplay import chess960_fen
            fen = chess960_fen(rng)
        st = BoardState().set(fen, is960, variant)
        start, moves, samples = st.fen(), [], []
        for _ in range(int(rng.integers(1, 90))):
            legal = st.legal_actions()
            if not legal or st.is_terminal() != TERMINAL_NONE:
                break
            pol = rng.random(len(legal))
            pol = pol / pol.sum()
            if rng.random() < 0.2:  # sharpened policies hold zeros
                pol[rng.integers(len(legal))] = 0.0
            samples.append((st.side_to_move(), float(np.float32(rng.uniform(-1, 1))), legal, pol))
            m = legal[int(rng.integers(len(legal)))]
            moves.append(m)
            st.do_action(m)
        games.append((start, moves, samples, int(rng.integers(3))))
    return games


def _write_python(games, variant, is960, mode, channels, out, chunks, chunk_size, planes):
    exporter = TrainDataExporter(os.path.join(out, "data.zarr"), mode, channels, number_chunks=chunks, chunk_size=chunk_size)
    for g, (fen, moves, samples, result) in enumerate(games):
        pgn = GamePGN(variant, is960, "CrazyAra-B200", "CrazyAra-B200", date="2026.10.18 12:00:00")
        st = BoardState().set(fen, is960, variant)
        pgn.fen = st.fen()
        for m in moves:
            pgn.play_move(st, m)
        rec = exporter.new_game()
        for s, (stm, q, legal, pol) in enumerate(samples):
            exporter.save_sample(rec, planes[g][s], [move_to_uci(m, is960) for m in legal], pol, q, stm)
        exporter.export_game_samples(rec, result)
        pgn.result = result_string(result)
        pgn.write(os.path.join(out, "games.pgn"))


@pytest.mark.parametrize("variant,is960,mode,channels", GAMES)
@pytest.mark.parametrize("chunks,chunk_size", [(200, 128), (3, 16)], ids=["roomy", "fills_up"])
def test_writers_are_byte_identical_to_the_python_writers(driver, tmp_path, variant, is960, mode, channels, chunks, chunk_size):
    games = _record_games(variant, is960, 5, seed=variant * 10 + int(is960))
    rng = np.random.default_rng(1)
    planes = [[rng.integers(0, 30, (channels, 8, 8)).astype(np.float32) for _ in s] for _, _, s, _ in games]
    lines = [f"{mode} {channels} {len(uci_labels(mode))} {chunks} {chunk_size}", str(len(games))]
    for g, (fen, moves, samples, result) in enumerate(games):
        lines += [f"{variant} {int(is960)} {result} {len(samples)} {len(moves)}", fen or BoardState().set("", is960, variant).fen(),
                  "2026.10.18 12:00:00", " ".join(map(str, moves))]
        for s, (stm, q, legal, pol) in enumerate(samples):
            lines += [f"{stm} {q!r} {len(legal)}", " ".join(str(int(x)) for x in planes[g][s].ravel()), " ".join(map(str, legal)),
                      " ".join(repr(float(p)) for p in pol)]
    rec = tmp_path / "records.txt"
    rec.write_text("\n".join(lines) + "\n")
    cpp, py = tmp_path / "cpp", tmp_path / "py"
    cpp.mkdir()
    py.mkdir()
    subprocess.run([driver, "write", str(rec), str(cpp)], check=True)
    _write_python(games, variant, is960, mode, channels, str(py), chunks, chunk_size, planes)
    tree = lambda d: sorted(os.path.relpath(os.path.join(r, f), d) for r, _, fs in os.walk(d) for f in fs)  # noqa: E731
    assert tree(cpp / "data.zarr") == tree(py / "data.zarr")
    for f in tree(cpp / "data.zarr"):
        assert filecmp.cmp(cpp / "data.zarr" / f, py / "data.zarr" / f, shallow=False), f
    assert (cpp / "games.pgn").read_bytes() == (py / "games.pgn").read_bytes()
    assert (cpp / "gameIdx.txt").read_text() == str(len(games))


@pytest.mark.parametrize("seed", [0, 5, 123456789, 2 ** 40 + 7])
def test_generator_draws_what_numpy_draws(driver, seed):
    n = 3000
    out = subprocess.run([driver, "rng", str(seed), str(n)], check=True, capture_output=True, text=True).stdout.split()
    r = np.random.default_rng(seed)
    p = np.array([0.05, 0.2, 0.0, 0.3, 0.45])
    want = []
    for i in range(n):
        want += [r.integers(4), r.random(), r.integers(0, 1 << 31), r.integers(8), r.choice(5, p=p), r.integers(37)]
        want.append(r.random(1 + (i * 37) % 300).sum())
        want += [r.exponential(15.0) for _ in range(1 + i % 40)]
    assert len(out) == len(want)
    for k, (a, b) in enumerate(zip(out, want)):
        assert float(a) == float(b), (k, a, b)
