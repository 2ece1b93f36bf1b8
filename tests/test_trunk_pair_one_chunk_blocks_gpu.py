"""A tower with runs of one-chunk blocks (c_op 64) gives the same bits in every shape of the tower kernel.  The pair
kernel gives chunk gc to CTA gc & 1, so in a one-chunk block one CTA of the pair owns no chunk and only runs the MMA2
of its partner's; two such blocks in a row swap the roles.  Blocks with odd and even chunk counts in between move the
first chunk of the next block between the CTAs, and both SE flavours and both depthwise sizes occur.  The RISE towers
have none of these blocks."""
import numpy as np
import pytest

from oracle import net as onet
from tests.golden.gen_net_golden import golden_input

# chunks per block: 1, 1, 3, 1, 2, 1, 1, 1, 5, 2 (first chunks 0, 1, 2, 5, 6, 8, 9, 10, 11, 16)
SE = ["ca_se", "eca_se", None, "ca_se", "eca_se", None, "ca_se", "eca_se", "ca_se", None]
KERNELS = [3, 5, 3, 5, 3, 3, 5, 3, 3, 5]
C_OPS = [64, 64, 192, 64, 128, 64, 64, 64, 320, 128]


def one_chunk_arch(cin=34, pch=81):
    arch = onet.arch_risev2(cin, pch)
    arch.update(name="one_chunk_blocks", se_types=list(SE), kernels=list(KERNELS), c_ops=list(C_OPS))
    return arch


def test_one_chunk_tower_has_the_blocks_it_is_meant_to_cover():
    chunks = [-(-c // 64) for c in C_OPS]
    assert len(SE) == len(KERNELS) == len(C_OPS)
    assert any(a == b == 1 for a, b in zip(chunks, chunks[1:]))  # consecutive one-chunk blocks
    assert {n % 2 for n in chunks if n > 1} == {0, 1}
    assert {"ca_se", "eca_se"} <= set(SE) and set(KERNELS) == {3, 5}


@pytest.mark.gpu
def test_pair_tower_with_one_chunk_blocks_is_bit_identical_to_the_other_shapes(tmp_path, monkeypatch):
    from crazyara_b200.nn import NeuralNetAPI
    from crazyara_b200.weights import export_blob
    arch = one_chunk_arch()
    blob = export_blob(onet.make_state_dict(arch, 5), arch, str(tmp_path / "one_chunk.arab"), input_version=10)
    for n in (1, 64):
        x = golden_input(arch, n=n, seed=23)
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
