"""A tower that mixes the squeeze-excitation flavours block by block (ca_se, eca_se, none; 3x3 and 5x5 depthwise) gives
the same bits in every shape of the tower kernel.  The pair kernel exchanges ca_se hidden values and SE scales between
its two CTAs through barriers that advance on different sets of blocks, which towers with one SE flavour do not
exercise: here an odd number of eca_se blocks comes before the first ca_se block, and the flavours keep alternating."""
import numpy as np
import pytest

from oracle import net as onet
from tests.golden.gen_net_golden import golden_input

SE = ["eca_se", "ca_se", None, "eca_se", "eca_se", "ca_se", "ca_se", "eca_se", "ca_se", None, "eca_se", "ca_se", "ca_se"]
KERNELS = [3, 5, 3, 3, 5, 3, 3, 3, 5, 3, 3, 3, 3]
C_OPS = [128, 160, 192, 256, 224, 320, 384, 96, 448, 512, 256, 576, 640]


def mixed_arch(cin=34, pch=81):
    arch = onet.arch_risev2(cin, pch)
    arch.update(name="mixed_se", se_types=list(SE), kernels=list(KERNELS), c_ops=list(C_OPS))
    return arch


@pytest.mark.gpu
def test_pair_tower_with_mixed_se_flavours_is_bit_identical_to_the_other_shapes(tmp_path, monkeypatch):
    from crazyara_b200.nn import NeuralNetAPI
    from crazyara_b200.weights import export_blob
    arch = mixed_arch()
    blob = export_blob(onet.make_state_dict(arch, 3), arch, str(tmp_path / "mixed.arab"), input_version=10)
    for n in (1, 64):
        x = golden_input(arch, n=n, seed=17)
        outs = {}
        for rows in ("32", "64", "128"):
            monkeypatch.setenv("ARA_TRUNK_ROWS", rows)
            net = NeuralNetAPI("gpu", 0, n, blob)
            v, p = np.zeros(n, np.float32), np.zeros((n, 81 * 64), np.float32)
            runs = []
            for _ in range(3):  # (repeated: a race between the pair's CTAs would not show every time)
                net.predict(x, v, p, None, n=n)
                runs.append((v.copy(), p.copy()))
            net.close()
            outs[rows] = runs
        ref_v, ref_p = outs["64"][0]
        assert np.isfinite(ref_v).all() and np.isfinite(ref_p).all()
        for rows, runs in outs.items():
            for i, (v, p) in enumerate(runs):
                assert np.array_equal(v, ref_v) and np.array_equal(p, ref_p), \
                    f"n={n}: ARA_TRUNK_ROWS={rows} run {i} differs from one board per CTA"

