"""The resident-A main loop of the 3x3 convolution GEMM (conv_resident_a) at its chunk limits, bit for bit.

The network's layers reach the resident loop with at most 4 chunk tiles (12 in float32, which streams).  These rows
have more chunk tiles than the B ring has stages, so the producer issues the late chunks' loads behind recycled
stages: 9 and 10 chunks at N tile 64 (8 stages, 10 tiles fit), 8 at N tile 128 (6 stages, 8 fit), and a float32 layer
whose split activations are 9 chunks.  One chunk more than fits runs the streaming loop; those rows pin the boundary
from the other side.  The operands and the model are those of test_conv_gemm_gpu.py (exact sums on a power-of-two
grid), so every output must equal the model's bit for bit.
"""
import numpy as np
import pytest

from tests.test_conv_gemm_gpu import Launcher, R, exact_kinds, exact_operands, expected_buffers, gemm

BOARDS = (2, 7, 64)

# row, N tile
CASES = [
    (R("chunks9[bn64]", 0, 576, 64, 3, 1, ldo=64), 64),
    (R("chunks10[bn64]", 0, 640, 64, 3, 1, ldo=64), 64),
    (R("chunks11-streaming[bn64]", 0, 704, 64, 3, 1, ldo=64), 64),
    (R("chunks8[bn128]", 0, 512, 128, 3, 1, ldo=128), 128),
    (R("chunks9-streaming[bn128]", 0, 576, 128, 3, 1, ldo=128), 128),
    (R("chunks9[bn64]", 1, 192, 64, 3, 1, outs="f", ldo=64), 64),
]


@pytest.mark.gpu
@pytest.mark.parametrize("row,bn", CASES, ids=[r.name for r, _ in CASES])
def test_chunk_limits_bit_for_bit(row, bn):
    for B in BOARDS:
        for kind in exact_kinds(row):
            ops = exact_operands(row, B, kind)
            acc = gemm(row, ops, B, "cuda")
            L = Launcher(row, B, ops)
            for cnt in (None, B // 2 + 1):
                got = L.run(bn, cnt)
                want = expected_buffers(row, B, ops, acc, bn, cnt)
                for k in want:
                    diff = got[k] != want[k]
                    assert not diff.any(), (f"{row.name} {kind} B={B} bn={bn} count={cnt} out_{k}: {int(np.sum(diff))} of "
                                            f"{diff.size} differ, first at {np.argwhere(diff)[0].tolist()}")
