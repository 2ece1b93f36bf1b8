"""Generates tests/golden/ref_mcts.npz from the reference's own search (oracle/_ref/libref_mcts.so, `make -C oracle ref`)
on every case of tests/test_ref_mcts.py:  python tests/golden/gen_ref_mcts_golden.py"""
import itertools
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

from oracle import refmcts  # noqa: E402
from oracle import search as osr  # noqa: E402
from tests import test_ref_mcts as T  # noqa: E402


def main():
    assert refmcts.available(), "oracle/_ref/libref_mcts.so not built"
    out = {}

    def record(pos, fen, vid, is960, premoves, st, threads=1):  # stands in for the test's comparison
        S = osr.Search(st)
        out[T.case_key(pos, fen, premoves, st, threads)] = refmcts.run(pos, fen, vid, is960, premoves, st, net_fn=osr.hash_net(S.n_labels),
                                                        channels=S.channels, n_labels=S.n_labels)
        S.close()

    T.assert_oracle_equals_reference = record
    for name in dir(T):  # every parametrised case of every comparison test
        fn = getattr(T, name)
        marks = [m for m in getattr(fn, "pytestmark", []) if m.name == "parametrize"] if name.startswith("test_") else []
        for combo in (itertools.product(*[list(m.args[1]) for m in marks]) if marks else []):
            fn(**{m.args[0]: v for m, v in zip(marks, combo)})
    keys = sorted(out)
    cat = lambda f, t: np.concatenate([np.asarray(out[k][f], t) for k in keys])  # noqa: E731
    np.savez_compressed(os.path.join(HERE, "ref_mcts.npz"), keys=np.array(keys),
                        n_moves=np.array([len(out[k]["moves"]) for k in keys], np.int32),
                        moves=np.array(sum((out[k]["moves"] for k in keys), []), dtype="U8"), visits=cat("visits", np.uint32),
                        q_bits=cat("q", np.float32).view(np.uint32), prior_bits=cat("prior", np.float32).view(np.uint32),
                        policy=cat("policy", np.float64),
                        scalars=np.array([[out[k][x] for x in T.SCALARS] for k in keys], np.float64))


if __name__ == "__main__":
    main()
