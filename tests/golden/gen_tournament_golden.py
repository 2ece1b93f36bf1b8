"""Generates tests/golden/tournament.json from the UNMODIFIED reference TournamentResult (oracle/_ref/libref_tournament.so,
`make -C oracle -f ref_tournament.mk`): operator<<, score() and the CSV line of write_tournament_result_to_csv.  Run in the build
container:
    python tests/golden/gen_tournament_golden.py"""
import ctypes
import json
import os
import struct
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))

# W / D / L: every score of 0 to 12 games (ties at two significant digits: 0.125 -> 0.12, 0.375 -> 0.38, 0.625 -> 0.62,
# 0.875 -> 0.88 round half to even on the binary value), all-draw / all-win / all-loss, the RL loop's 100 games and a few
# large counts
CASES = sorted({(w, d, n - w - d) for n in range(1, 13) for w in range(n + 1) for d in range(n + 1 - w)} |
               {(100, 0, 0), (0, 100, 0), (0, 0, 100), (50, 1, 49), (49, 3, 48), (51, 0, 49), (50, 0, 50), (33, 34, 33),
                (1, 0, 199), (12345, 678, 9012)})
NAMES = [("CrazyAra-B200-contender", "CrazyAra-B200-producer"), ("fake", "fake"), ("A", "B")]


def reference():
    L = ctypes.CDLL(os.path.join(ROOT, "oracle", "_ref", "libref_tournament.so"))
    L.ref_tournament_result.restype = ctypes.c_float
    L.ref_tournament_result.argtypes = [ctypes.c_char_p, ctypes.c_char_p, ctypes.c_ulonglong, ctypes.c_ulonglong,
                                        ctypes.c_ulonglong, ctypes.c_char_p, ctypes.c_int, ctypes.c_char_p]
    return L


def render(L, a, b, w, d, l):
    """(text, score as float32 bits, csv line) of the reference"""
    out = ctypes.create_string_buffer(512)
    with tempfile.TemporaryDirectory() as tmp:
        csv = os.path.join(tmp, "r.csv")
        score = L.ref_tournament_result(a.encode(), b.encode(), w, d, l, out, 512, csv.encode())
        line = open(csv).read()
    return out.value.decode(), struct.unpack("<I", struct.pack("<f", score))[0], line


def main():
    L = reference()
    rows = []
    for i, (w, d, l) in enumerate(CASES):
        a, b = NAMES[i % len(NAMES)]
        text, bits, line = render(L, a, b, w, d, l)
        rows.append(dict(a=a, b=b, w=w, d=d, l=l, text=text, score_bits=bits, csv=line))
    json.dump({"cases": rows}, open(os.path.join(HERE, "tournament.json"), "w"), separators=(",", ":"))
    print(len(rows), "tournament results")


if __name__ == "__main__":
    main()
