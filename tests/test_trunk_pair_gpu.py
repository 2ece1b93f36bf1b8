"""The tower kernel's three shapes give the same bits: one board per CTA pair (the default while every pair fits on
the GPU at once), one board per CTA and two boards per CTA.  Each shape accumulates every sum with the same operands in
the same order, so a position's value and policy do not depend on which shape evaluated it."""
import numpy as np
import pytest

from oracle import net as onet
from tests.golden.gen_net_golden import golden_input

SHAPES = ({"ARA_TRUNK_ROWS": "32"}, {"ARA_TRUNK_ROWS": "64"}, {"ARA_TRUNK_ROWS": "128"})


@pytest.mark.gpu
@pytest.mark.parametrize("name,cin,pch", [("risev2", 34, 81), ("risev33", 52, 76)])
def test_pair_tower_is_bit_identical_to_the_other_shapes(tmp_path, monkeypatch, name, cin, pch):
    from crazyara_b200.nn import NeuralNetAPI
    from crazyara_b200.weights import export_blob
    arch = onet.arch_risev2(cin, pch) if name == "risev2" else onet.arch_risev33(cin, pch, True)
    blob = export_blob(onet.make_state_dict(arch, 0), arch, str(tmp_path / f"{name}.arab"),
                       input_version=10 if name == "risev2" else 30)
    for n in (1, 5, 64, 66):
        x = golden_input(arch, n=n, seed=13)
        outs = []
        for env in SHAPES:
            monkeypatch.setenv("ARA_TRUNK_ROWS", env["ARA_TRUNK_ROWS"])
            net = NeuralNetAPI("gpu", 0, n, blob)
            v, p = np.zeros(n, np.float32), np.zeros((n, pch * 64), np.float32)
            for _ in range(3):  # (repeated: a race in the weight ring or the pair's exchanges would not show every time)
                net.predict(x, v, p, None, n=n)
                outs.append((v.copy(), p.copy()))
            net.close()
        assert np.isfinite(outs[0][0]).all() and np.isfinite(outs[0][1]).all()
        for i, (v, p) in enumerate(outs[1:], 1):
            assert np.array_equal(v, outs[0][0]) and np.array_equal(p, outs[0][1]), \
                f"n={n}: {SHAPES[i // 3]} run {i % 3} differs from the pair"
