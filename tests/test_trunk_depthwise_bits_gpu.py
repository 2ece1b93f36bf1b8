"""The tower kernel's CUDA-core arithmetic, bit for bit, against a NumPy model.

The tower's 1x1 convolutions here are 0/1 selection matrices: each operating channel picks one trunk channel, and each
trunk channel picks one operating channel.  Every wgmma sum then has one nonzero term, so it is exact in any order, and
what is left is the arithmetic on the CUDA cores:
  H1 = fp16(relu(X[sel1] + b1))
  H2 = fp16(relu(acc)), acc = bd, then for dxi (columns outside the board skipped), for dyi (rows outside the board as
       zeros): acc = fmaf(H1, wd, acc)
  X  = fp16((H2[sel2] + b2) + X)
An fp16 x fp16 product is exact in fp32, so each fmaf equals a float32 add of the exact product: the model below does
those adds in the kernel's order and predicts every output bit.  The shape tests compare the three tower shapes with
each other; this one pins all three to the model."""
import ctypes

import numpy as np
import pytest
import torch
import torch.nn.functional as F

# (c_op, depthwise k): 3x3 and 5x5, one-chunk blocks, a padded chunk (224 = 3.5 chunks), odd and even chunk counts
BLOCKS = [(224, 3), (64, 5), (128, 3), (64, 3), (192, 5), (320, 3), (224, 5)]
SHAPES = ("32", "64", "128")


def selection_tower(seed=3):
    """Folded weights of a tower of BLOCKS (TrunkBlockHost layouts) with 0/1 selection matrices as 1x1 convolutions."""
    rng = np.random.default_rng(seed)
    blocks = []
    for c, k in BLOCKS:
        sel1 = rng.integers(0, 256, c)
        sel2 = np.concatenate([rng.permutation(c), rng.integers(0, c, max(0, 256 - c))])[:256]  # every op channel used
        w1 = np.zeros((c, 256), np.float32)
        w1[np.arange(c), sel1] = 1.0
        w2 = np.zeros((256, c), np.float32)
        w2[np.arange(256), sel2] = 1.0
        nonzero = lambda a: np.where(a == 0, np.float32(0.125), a).astype(np.float32)  # noqa: E731
        blocks.append(dict(
            c_op=c, k=k, w1=w1, w2=w2,
            b1=nonzero(rng.normal(0.0, 0.3, c).astype(np.float32)),
            wd=nonzero(rng.normal(0.0, 0.4, (c, k * k)).astype(np.float16).astype(np.float32)),
            bd=nonzero(rng.normal(0.0, 0.2, c).astype(np.float32)),
            b2=nonzero(rng.normal(0.0, 0.2, 256).astype(np.float32))))
    return blocks


def tower_input(n, seed=5):
    x = np.random.default_rng(seed).normal(0.0, 1.0, (n, 64, 256)).astype(np.float16)
    return np.where(x == 0, np.float16(0.5), x)


def model(x, blocks):
    """The kernel's arithmetic in NumPy float32 / float16: x [n, 64, 256] fp16 -> the tower output, same bits."""
    f32 = np.float32
    x = x.copy()
    n = x.shape[0]
    for b in blocks:
        c, k, r = b["c_op"], b["k"], b["k"] // 2
        sel1, sel2 = b["w1"].argmax(1), b["w2"].argmax(1)
        h1 = np.maximum(x[:, :, sel1].astype(f32) + b["b1"], f32(0)).astype(np.float16)
        hp = np.zeros((n, 8 + 2 * r, 8, c), f32)  # rows padded with zero operands
        hp[:, r:r + 8] = h1.reshape(n, 8, 8, c)
        wd = b["wd"].reshape(c, k, k)  # [c][dyi][dxi]
        acc = np.broadcast_to(b["bd"], (n, 8, 8, c)).copy()
        for xc in range(8):
            for dxi in range(k):
                xx = xc + dxi - r
                if xx < 0 or xx > 7:
                    continue
                for dyi in range(k):
                    acc[:, :, xc] += hp[:, dyi:dyi + 8, xx] * wd[:, dyi, dxi]
        h2 = np.maximum(acc, f32(0)).astype(np.float16).reshape(n, 64, c)
        x = ((h2[:, :, sel2].astype(f32) + b["b2"]) + x.astype(f32)).astype(np.float16)
    return x


def reference(x, blocks):
    """The block of oracle/net.py (1x1 conv, relu, depthwise conv, relu, 1x1 conv, + input) in torch fp32, BN folded."""
    out = torch.from_numpy(x.astype(np.float32)).reshape(-1, 8, 8, 256).permute(0, 3, 1, 2)
    for b in blocks:
        c, k = b["c_op"], b["k"]
        h = F.relu(F.conv2d(out, torch.from_numpy(b["w1"])[:, :, None, None], torch.from_numpy(b["b1"])))
        h = F.relu(F.conv2d(h, torch.from_numpy(b["wd"]).reshape(c, 1, k, k), torch.from_numpy(b["bd"]), padding=k // 2, groups=c))
        out = out + F.conv2d(h, torch.from_numpy(b["w2"])[:, :, None, None], torch.from_numpy(b["b2"]))
    return out.permute(0, 2, 3, 1).reshape(-1, 64, 256).numpy()


def test_selection_towers_and_model_against_the_fp32_block():
    blocks = selection_tower()
    for b, (c, k) in zip(blocks, BLOCKS):
        assert b["w1"].shape == (c, 256) and (b["w1"].sum(1) == 1).all() and set(np.unique(b["w1"])) == {0.0, 1.0}
        assert b["w2"].shape == (256, c) and (b["w2"].sum(1) == 1).all() and set(np.unique(b["w2"])) == {0.0, 1.0}
        assert b["wd"].shape == (c, k * k) and (b["wd"].astype(np.float16).astype(np.float32) == b["wd"]).all()
        if c <= 256:
            assert (b["w2"].sum(0) >= 1).all()  # every depthwise output reaches the tower output
        for v in (b["b1"], b["wd"], b["bd"], b["b2"]):
            assert (v != 0).all()
    x = tower_input(5)
    assert (x != 0).all()
    got, ref = model(x, blocks).astype(np.float32), reference(x, blocks)
    assert np.isfinite(got).all() and np.abs(ref).max() > 1.0
    # the fp16 roundings of H1, H2 and X, a few units in the last place each, over seven blocks; |X| grows to ~100
    np.testing.assert_allclose(got, ref, rtol=5e-3, atol=5e-2)


def _run_trunk(x, blocks):
    from crazyara_b200 import check, lib
    f = lib().ara_debug_trunk
    f.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int] + [ctypes.c_void_p] * 9
    f.restype = ctypes.c_int
    cat = lambda key: np.ascontiguousarray(np.concatenate([b[key].ravel() for b in blocks]).astype(np.float32))  # noqa: E731
    arrs = [np.array([b["c_op"] for b in blocks], np.int32), np.array([b["k"] for b in blocks], np.int32)]
    arrs += [cat(key) for key in ("w1", "b1", "wd", "bd", "w2", "b2")]
    x = np.ascontiguousarray(x)
    out = np.full_like(x, np.float16(np.nan))
    check(f(x.ctypes.data, x.shape[0], len(blocks), *[a.ctypes.data for a in arrs], out.ctypes.data))
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("rows", SHAPES)
def test_tower_matches_the_model_bit_for_bit(monkeypatch, rows):
    monkeypatch.setenv("ARA_TRUNK_ROWS", rows)
    blocks = selection_tower()
    for n in (1, 5, 64, 66):
        x = tower_input(n, seed=n)
        want = model(x, blocks)
        got = _run_trunk(x, blocks)
        diff = got.view(np.uint16) != want.view(np.uint16)
        assert not diff.any(), (f"ARA_TRUNK_ROWS={rows} n={n}: {int(diff.sum())} of {diff.size} outputs differ, "
                                f"first at {np.argwhere(diff)[0].tolist()}")
