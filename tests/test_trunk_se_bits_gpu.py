"""The tower kernel's squeeze-excitation and MXNet block semantics, bit for bit, against a NumPy model, in all six kernel
builds (three shapes, each with and without the MXNet semantics).

This extends tests/test_trunk_depthwise_bits_gpu.py: the 1x1 convolutions are 0/1 selection matrices, so every wgmma
sum has one nonzero term, and the model predicts the CUDA-core arithmetic around it.  Here the blocks also carry a
squeeze-excitation (SE), and the MXNet blocks their own features.  The model restates them in the kernel's order:
  pool  p = (((x0 + x1) + x2) ... + x63) * (1/64) in fp32, rows 0..63 of the block input
  ca_se h = relu([se_b1 +] fmaf(w1[255], p[255], ... fmaf(w1[0], p[0], 0))), w1 rounded to fp16
        g = [se_b +] the same over the 128 hidden values with fp16 w2
  eca_se g = se_b + the same over the 256 pooled values
  gate  Hard6 sat(fmaf(g, f32(1/6), 0.5)), Hard5 sat(fmaf(g, f32(0.2), 0.5)) (one FFMA.SAT each), logistic
  scale x = fp16(f32(x) * gate)
  block shortcut after the SE: x = fp16((H2[sel2] + b2) + x_se); before it (MXNet): fp16((x_in + H2[sel2]) + b2), where
        the wgmma adds H2[sel2] onto the accumulator preloaded with x_in
The pooled values are arbitrary fp32 numbers, so an fmaf is not a float32 multiply-add; fmaf() below rounds once.  The
logistic gate runs on MUFU.EX2, which the model cannot restate; its bit-for-bit blocks use only inputs whose result
does not depend on the approximation (0 -> 0.5, >= 17 -> 1, <= -30 -> a scale whose product with any fp16 rounds to
+-0), and test_logistic_gate_within_one_ulp covers general inputs.
"""
import ctypes
import functools

import numpy as np
import pytest

from tests.test_trunk_depthwise_bits_gpu import SHAPES

f16, f32, f64 = np.float16, np.float32, np.float64
HARD6, HARD5, SIGMOID = 0, 1, 2
NONE, CA, ECA = 0, 1, 2
PRE = 1  # kTrunkShortcutPreSe
LOGISTIC_POINTS = (0.0, 20.0, -40.0)  # gate inputs of the logistic blocks of the bit-for-bit towers
SIGMA_G = {HARD6: 1.5, HARD5: 1.25}  # gate input spread: most inside the linear region (|g| < 3, |g| < 2.5)
LINEAR = {HARD6: 3.0, HARD5: 2.5}

# (se, gate, se biases: 0 none, 3 se_b and se_b1 (ca_se), 1 se_b (eca_se), pre-SE shortcut, SE-only, c_op, k)
# SE-only: W2 = 0, b2 = 0, shortcut after the SE, so the block outputs the SE-scaled input.
S = dict
TOWERS = {
    # PyTorch RISE semantics: the MX=false kernels.  SE first and last, a 1-chunk block with SE (c_op 64 and 32), three
    # eca_se blocks before the first ca_se, consecutive SE blocks, SE blocks at chunk0 = 0, 1, 2, 3 (mod 4).
    "torch": [S(se=CA, c=224, k=3), S(se=ECA, c=64, k=5), S(se=NONE, c=128, k=3), S(se=ECA, c=192, k=3),
              S(se=ECA, c=256, k=5, only=1), S(se=CA, c=64, k=3), S(se=NONE, c=96, k=5), S(se=CA, c=320, k=5, only=1),
              S(se=ECA, c=32, k=3), S(se=NONE, c=224, k=5), S(se=CA, c=128, k=3), S(se=ECA, c=160, k=5),
              S(se=CA, c=64, k=5, only=1), S(se=NONE, c=256, k=3), S(se=ECA, c=128, k=3)],
    # MXNet gates and biases, shortcut after the SE, signed activations
    "mx": [S(se=ECA, gate=HARD5, c=128, k=3), S(se=CA, gate=HARD6, bias=3, c=64, k=5), S(se=CA, gate=HARD5, c=192, k=3),
           S(se=NONE, c=224, k=5), S(se=ECA, gate=SIGMOID, c=96, k=3), S(se=CA, gate=SIGMOID, bias=3, c=32, k=3),
           S(se=ECA, gate=HARD6, c=256, k=3, only=1), S(se=CA, gate=HARD5, bias=3, c=64, k=5, only=1),
           S(se=NONE, c=320, k=3), S(se=ECA, gate=HARD5, c=160, k=5), S(se=CA, gate=SIGMOID, c=128, k=3),
           S(se=ECA, gate=SIGMOID, c=64, k=3, only=1), S(se=CA, gate=HARD5, bias=3, c=96, k=5),
           S(se=CA, gate=HARD6, c=224, k=5)],
    # MXNet shortcut before the SE (and on blocks without SE).  Nonnegative activations and H2 >= 0.25 in these blocks
    # keep every wgmma sum x_in + H2 exact in fp32 (see _pre_sum_exact); a pre-SE block never follows an SE-only one.
    "mx_pre": [S(se=CA, gate=HARD6, bias=3, pre=1, c=128, k=3), S(se=ECA, gate=HARD5, pre=1, c=64, k=5),
               S(se=NONE, pre=1, c=192, k=3), S(se=CA, gate=SIGMOID, bias=3, pre=1, c=96, k=5),
               S(se=ECA, gate=HARD6, c=224, k=3), S(se=CA, gate=HARD5, pre=1, c=32, k=3),
               S(se=ECA, gate=SIGMOID, pre=1, c=128, k=5), S(se=ECA, gate=HARD5, c=256, k=3, only=1),
               S(se=NONE, c=160, k=3), S(se=CA, gate=HARD6, c=64, k=3), S(se=CA, gate=HARD5, bias=3, pre=1, c=64, k=5),
               S(se=NONE, gate=HARD6, c=288, k=5), S(se=ECA, gate=HARD6, pre=1, c=224, k=5)],
}
NS = (1, 5, 64, 66)


# ---------------------------------------------------------------------------------------------------------------- fmaf
def fmaf(a, b, c):
    """Correctly rounded float32 fma, elementwise.  An fp32 x fp32 product is exact in float64 (48 bits); TwoSum gives
    the sum's float64 rounding s and its error e exactly; rounding s to fp32 is then right unless s is an fp32 midpoint
    (a double rounding), where the sign of e decides."""
    a, b, c = (np.asarray(v, f32).astype(f64) for v in (a, b, c))
    p = a * b
    s = p + c
    bb = s - p
    e = (p - (s - bb)) + (c - bb)
    r = s.astype(f32)
    other = np.where(s > r, np.nextafter(r, f32(np.inf)), np.nextafter(r, f32(-np.inf)))
    mid = (s != r) & (s == (r.astype(f64) + other.astype(f64)) * 0.5) & (e != 0)
    up = (e > 0) == (other > r)  # the exact value lies on the side of the other candidate
    return np.where(mid & up, other, r).astype(f32)


# ------------------------------------------------------------------------------------------------------------- weights
def _nonzero(a):
    return np.where(a == 0, f32(0.125), a).astype(f32)


def _block_spec(s):
    d = dict(se=NONE, gate=HARD6, bias=0, pre=0, only=0)
    d.update(s)
    d["bias"] = d["bias"] if d["se"] != ECA else 1
    return d


def build_tower(name, seed=11):
    """Folded weights of a tower (TrunkBlockHost layouts) with selection matrices as 1x1 convolutions.  The SE weights
    are fp32 values the host rounds to fp16; their scale is set from the pooled activations a calibration input
    reaches at the block, so that the gate inputs spread as SIGMA_G asks."""
    rng = np.random.default_rng(seed)
    positive = name == "mx_pre"
    x = tower_input(name, 8, seed=99)
    blocks, chunk0 = [], 0
    for spec in TOWERS[name]:
        b = _block_spec(spec)
        c, k = b["c"], b["k"]
        b.update(c_op=c, chunk0=chunk0)
        chunk0 += (c + 63) // 64
        b["sel1"] = rng.integers(0, 256, c)
        b["sel2"] = np.concatenate([rng.permutation(c), rng.integers(0, c, max(0, 256 - c))])[:256]
        b["b1"] = _nonzero(rng.normal(0.0, 0.3, c).astype(f32))
        if b["pre"]:  # acc >= bd >= 0.25: H2 is at least 0.25
            b["wd"] = rng.uniform(0.0, 0.5 / k ** 2, (c, k * k)).astype(f16).astype(f32)
            b["bd"] = rng.uniform(0.25, 0.5, c).astype(f32)
        else:
            b["wd"] = _nonzero(rng.normal(0.0, 0.8 / k ** 2, (c, k * k)).astype(f16).astype(f32))
            b["bd"] = _nonzero(rng.normal(0.0, 0.2, c).astype(f32))
        b["b2"] = rng.uniform(0.25, 0.5, 256).astype(f32) if positive else _nonzero(rng.normal(0.0, 0.2, 256).astype(f32))
        if b["only"]:
            b["sel2"] = np.full(256, -1)
            b["b2"] = np.zeros(256, f32)
        if b["se"] != NONE:
            _se_weights(b, rng, se_pool(x))
        blocks.append(b)
        x = model(x, [b], mx=tower_mx(blocks))
    return blocks


def _se_weights(b, rng, pool):
    logistic = b["gate"] == SIGMOID
    ms = lambda v: float(np.mean(np.sum(v.astype(f64) ** 2, axis=1)))  # noqa: E731  mean over boards of sum of squares
    sg = SIGMA_G.get(b["gate"], 1.0)
    if b["se"] == ECA:
        b["se_b"] = rng.normal(0.0, 0.5, 256).astype(f32)
        b["se_w1t"] = (rng.normal(0.0, 1.0, (256, 256)) * np.sqrt(sg ** 2 - 0.25) / np.sqrt(ms(pool))).astype(f32)
        b["se_w2t"] = None
        if logistic:
            b["se_w1t"][:] = 0.0
            b["se_b"] = rng.choice(np.array(LOGISTIC_POINTS, f32), 256)
        return
    b["se_w1t"] = (rng.normal(0.0, 1.0, (256, 128)) / np.sqrt(ms(pool))).astype(f32)
    b["se_b1"] = rng.normal(0.0, 0.3, 128).astype(f32) if b["bias"] else None
    a = pool.astype(f64) @ b["se_w1t"].astype(f16).astype(f64) + (0.0 if b["se_b1"] is None else b["se_b1"])
    hid = np.maximum(a, 0.0)
    sb = 0.5 if b["bias"] else 0.0
    b["se_w2t"] = (rng.normal(0.0, 1.0, (128, 256)) * np.sqrt(sg ** 2 - sb ** 2) / np.sqrt(ms(hid))).astype(f32)
    b["se_b"] = rng.normal(0.0, 0.5, 256).astype(f32) if b["bias"] else None
    if logistic:
        b["se_w2t"][:] = 0.0
        if b["bias"]:
            b["se_b"] = rng.choice(np.array(LOGISTIC_POINTS, f32), 256)


def tower_mx(blocks):
    """rise_trunk_init's choice: the MXNet kernels when some block has the flag, a gate other than Hard6 or se_b1."""
    return any(b["pre"] or b["gate"] != HARD6 or b.get("se_b1") is not None for b in blocks)


def tower_input(name, n, seed=5):
    x = np.random.default_rng(seed).normal(0.0, 1.0, (n, 64, 256))
    if name == "mx_pre":
        x = np.abs(x) + 0.25
    x = x.astype(f16)
    return np.where(x == 0, f16(0.5), x)


# --------------------------------------------------------------------------------------------------------------- model
def se_pool(x, mut=()):
    rows = range(63, -1, -1) if "pool_order" in mut else range(64)
    s = np.zeros((x.shape[0], 256), f32)
    for r in rows:
        s = s + x[:, r].astype(f32)
    return s * f32(1.0 / 64.0)


def _dot(w, v):
    """a = fmaf(w[i], v[:, i], a) for i = 0, 1, ...: w [K][N] fp32, v [n][K] -> [n][N]"""
    a = np.zeros((v.shape[0], w.shape[1]), f32)
    for i in range(w.shape[0]):
        a = fmaf(w[i][None, :], v[:, i:i + 1], a)
    return a


def _logistic(g, diag):
    if diag is not None:
        diag.setdefault("logistic", []).append(g.ravel().copy())
    # exact results at the points the bit-for-bit towers use; float64 elsewhere (the oracle comparison)
    return (1.0 / (1.0 + np.exp(-g.astype(f64)))).astype(f32)


def se_gate(g, gate, mut=(), diag=None):
    if "gate_swap" in mut and gate in (HARD6, HARD5):
        gate = HARD5 if gate == HARD6 else HARD6
    if gate == SIGMOID:
        return _logistic(g, diag)
    if diag is not None:
        diag.setdefault(gate, []).append(g.ravel().copy())
    slope = f32(1.0 / 6.0) if gate == HARD6 else f32(0.2)
    y = (g * slope + f32(0.5)).astype(f32) if "gate_mul_add" in mut else fmaf(g, slope, f32(0.5))
    return np.clip(y, f32(0), f32(1))


def se_scales(x, b, mx, mut=(), diag=None):
    """The gate of every channel: x [n][64][256] fp16 -> [n][256] fp32"""
    r16 = (lambda w: w.astype(f32)) if "se_fp32" in mut else (lambda w: w.astype(f16).astype(f32))  # noqa: E731
    pool = se_pool(x, mut)
    gate = b["gate"] if mx else HARD6
    if b["se"] == CA:
        a = _dot(r16(b["se_w1t"]), pool)
        if mx and b.get("se_b1") is not None and "drop_b1" not in mut:
            a = b["se_b1"] + a
        hid = np.maximum(a, f32(0))
        g = _dot(r16(b["se_w2t"]), hid)
        if mx and b.get("se_b") is not None:
            g = b["se_b"] + g
    else:
        g = b["se_b"] + _dot(r16(b["se_w1t"]), pool)
    if diag is not None:
        diag.setdefault("g", []).append(g)
    s = se_gate(g, gate, mut, diag)
    if "swap_halves" in mut:
        s = np.concatenate([s[:, 128:], s[:, :128]], axis=1)
    return s


def _depthwise(h1, wd, bd, k):
    """acc = bd, then dxi outer (columns outside the board skipped), dyi inner (rows outside as zeros), each an add of
    the exact fp16 x fp16 product: h1 [n][64][c] -> [n][8][8][c] fp32, in h1's dtype precision when float64"""
    n, c = h1.shape[0], h1.shape[2]
    r = k // 2
    hp = np.zeros((n, 8 + 2 * r, 8, c), h1.dtype)
    hp[:, r:r + 8] = h1.reshape(n, 8, 8, c)
    w = wd.reshape(c, k, k).astype(h1.dtype)
    acc = np.broadcast_to(bd.astype(h1.dtype), (n, 8, 8, c)).copy()
    for xc in range(8):
        for dxi in range(k):
            xx = xc + dxi - r
            if 0 <= xx <= 7:
                for dyi in range(k):
                    acc[:, :, xc] += hp[:, dyi:dyi + 8, xx] * w[:, dyi, dxi]
    return acc


def _select2(h2, sel2):
    d2 = h2[:, :, np.maximum(sel2, 0)].astype(f32)
    d2[:, :, sel2 < 0] = 0.0
    return d2


def _pre_sum_exact(x_in, d2):
    return (x_in.astype(f32) + d2).astype(f64) == x_in.astype(f64) + d2.astype(f64)


def model(x, blocks, mx, mut=(), diag=None):
    """The kernel's arithmetic in NumPy float32 / float16: x [n, 64, 256] fp16 -> the tower output, same bits.  mut:
    deliberate mistakes (test_each_mutation_changes_the_output); diag: collects gate inputs and checks of the
    preconditions."""
    x = x.copy()
    for b in blocks:
        x_in = x
        if b["se"] != NONE:
            s = se_scales(x, b, mx, mut, diag)
            x = (x.astype(f32) * s[:, None, :]).astype(f16)
        h1 = np.maximum(x[:, :, b["sel1"]].astype(f32) + b["b1"], f32(0)).astype(f16)
        acc = _depthwise(h1.astype(f32), b["wd"], b["bd"], b["k"])
        h2 = np.maximum(acc, f32(0)).astype(f16).reshape(x.shape[0], 64, b["c_op"])
        d2 = _select2(h2, b["sel2"])
        if mx and b["pre"]:
            x_sc = x if "pre_after" in mut else x_in
            if diag is not None:
                diag["pre_inexact"] = diag.get("pre_inexact", 0) + int((~_pre_sum_exact(x_sc, d2)).sum())
            x = ((x_sc.astype(f32) + d2) + b["b2"]).astype(f16)
        else:
            x = ((d2 + b["b2"]) + x.astype(f32)).astype(f16)
    return x


@functools.lru_cache(maxsize=None)
def tower(name):
    return build_tower(name)


@functools.lru_cache(maxsize=None)
def expected(name, n):
    """(input, model output, diagnostics) of a tower on the GPU tests' input of n boards"""
    x = tower_input(name, n, seed=n)
    diag = {}
    out = model(x, tower(name), tower_mx(tower(name)), diag=diag)
    return x, out, diag


# ------------------------------------------------------------------------------------------------------- CPU checks
def test_fmaf_matches_glibc():
    libm = ctypes.CDLL("libm.so.6")
    libm.fmaf.argtypes = [ctypes.c_float] * 3
    libm.fmaf.restype = ctypes.c_float
    rng = np.random.default_rng(1)
    a = rng.normal(0.0, 1.0, 4000).astype(f16).astype(f32)
    b = (rng.normal(0.0, 1.0, 4000) * np.exp2(rng.integers(-12, 12, 4000))).astype(f32)
    c = (rng.normal(0.0, 1.0, 4000) * np.exp2(rng.integers(-12, 12, 4000))).astype(f32)
    # products a b = +-half an ulp of c, less i^2 2^-46 of it: c +- a b lies just inside an fp32 midpoint, closer than
    # half a float64 ulp, so that its float64 rounding is the midpoint itself.  c has an odd last bit, so that rounding
    # the midpoint to even moves away from the right result.
    i = np.arange(1, 301)
    e = rng.integers(-10, 10, i.size).astype(f64)
    sign = rng.choice([-1.0, 1.0], i.size)
    c_mid = (sign * (1.0 + (2 * rng.integers(0, 2 ** 21, i.size) + 1) * 2.0 ** -23) * np.exp2(e)).astype(f32)
    a_mid = (1.0 + i * 2.0 ** -23).astype(f32)
    b_mid = (rng.choice([-1.0, 1.0], i.size) * 2.0 ** -24 * (1.0 - i * 2.0 ** -23) * np.exp2(e)).astype(f32)
    a, b, c = np.concatenate([a, a_mid]), np.concatenate([b, b_mid]), np.concatenate([c, c_mid])
    want = np.array([libm.fmaf(*map(float, t)) for t in zip(a, b, c)], f32)
    got = fmaf(a, b, c)
    assert (got.view(np.uint32) == want.view(np.uint32)).all()
    # the midpoint cases are double roundings: rounding the float64 sum once more would get some of them wrong
    naive = (a.astype(f64) * b.astype(f64) + c.astype(f64)).astype(f32)
    assert (naive != want).sum() >= 100


def test_towers_cover_the_block_kinds():
    seen = set()
    for name in TOWERS:
        blocks = tower(name)
        assert len(blocks) <= 24
        assert tower_mx(blocks) == (name != "torch")
        se = [b for b in blocks if b["se"] != NONE]
        assert blocks[0]["se"] != NONE and blocks[-1]["se"] != NONE
        assert any(b["c_op"] <= 64 for b in se) and any(b["only"] for b in se)
        # the pair kernel's W2 ring offset of the SE image, u2 = chunk0 (mod 4), takes every value
        assert {b["chunk0"] % 4 for b in se} == {0, 1, 2, 3}, name
        assert any(a["se"] != NONE and c["se"] != NONE for a, c in zip(blocks, blocks[1:]))
        # a ca_se block after an odd number of eca_se blocks: the pair's two SE barriers are in different phases
        assert any(b["se"] == CA and sum(a["se"] == ECA for a in blocks[:i]) % 2 == 1 for i, b in enumerate(blocks))
        for a, c in zip(blocks, blocks[1:]):
            assert not (a["only"] and c["pre"])
        for b in blocks:
            if b["se"] == CA:
                assert (b.get("se_b") is None) == (b.get("se_b1") is None)
            seen.add((b["se"], b["gate"] if b["se"] else None, b["bias"] if b["se"] == CA else None, b["pre"], b["k"],
                      name != "torch"))
    for se, gates in ((CA, (HARD6, HARD5, SIGMOID)), (ECA, (HARD6, HARD5, SIGMOID))):
        for g in gates:
            assert any(s[0] == se and s[1] == g and s[5] for s in seen), (se, g)
            assert any(s[0] == se and s[1] == g and s[3] for s in seen), (se, g)  # shortcut before the SE
        assert any(s[0] == se and not s[3] and s[5] for s in seen)
    assert any(s[0] == CA and s[2] == 3 for s in seen) and any(s[0] == CA and s[2] == 0 and s[5] for s in seen)
    assert {s[4] for s in seen if s[0]} == {3, 5} and any(s[0] == NONE and s[5] for s in seen)


@pytest.mark.parametrize("name", list(TOWERS))
def test_preconditions(name):
    """Every wgmma sum the MX shortcut makes is exact in fp32, the logistic gates see only their exact points, the
    activations stay finite, and the Hard6 / Hard5 gate inputs are mostly inside the linear region, with some
    saturated at each end."""
    gates = {}
    for n in NS:
        _, out, diag = expected(name, n)
        assert np.isfinite(out.astype(f32)).all() and np.abs(out.astype(f32)).max() < 2048.0
        assert diag.get("pre_inexact", 0) == 0
        if name == "mx_pre":
            assert (out >= 0).all()
        for g in diag.get("logistic", []):
            assert np.isin(g, np.array(LOGISTIC_POINTS, f32)).all()
        for gate in (HARD6, HARD5):
            gates.setdefault(gate, []).extend(diag.get(gate, []))
    for gate, gs in gates.items():
        if not gs:
            continue
        g = np.concatenate(gs)
        lin = LINEAR[gate]
        inside, low, high = np.mean(np.abs(g) < lin), np.mean(g <= -lin), np.mean(g >= lin)
        assert inside >= 0.75 and low >= 0.01 and high >= 0.01, (name, gate, inside, low, high)


MUTATIONS = {"gate_mul_add": ("torch", "mx"), "pool_order": ("torch", "mx"), "pre_after": ("mx_pre",),
             "swap_halves": ("torch", "mx"), "se_fp32": ("torch",), "gate_swap": ("mx",), "drop_b1": ("mx",)}


@pytest.mark.parametrize("mut", list(MUTATIONS))
def test_each_mutation_changes_the_output(mut):
    """On the GPU tests' own towers and inputs, each plausible mistake in the SE stage changes some output bit: the
    bit-for-bit comparison would catch it."""
    for name in MUTATIONS[mut]:
        for n in NS:
            x, want, _ = expected(name, n)
            got = model(x, tower(name), tower_mx(tower(name)), mut=(mut,))
            if (got.view(np.uint16) != want.view(np.uint16)).any():
                return
    pytest.fail(f"the model with {mut} gives the same bits")


# ---------------------------------------------------------------------------------------------- against the oracles
def _r16(w):
    return w.astype(f16).astype(f32)


def _selection_weights(b):
    w1 = np.eye(256, dtype=f32)[b["sel1"]]  # [c_op][256]
    w2 = np.zeros((256, b["c_op"]), f32)
    w2[np.arange(256)[b["sel2"] >= 0], b["sel2"][b["sel2"] >= 0]] = 1.0
    return w1, w2


def _stem_identity():
    w = np.zeros((256, 256, 3, 3), f32)
    w[np.arange(256), np.arange(256), 1, 1] = 1.0
    return w


def oracle_torch_block(x, b):
    """One block of oracle/net.py (PyTorch RISE): a one-block network whose stem passes x >= 0 through, BN folded into
    identity statistics and the block's biases.  The oracle takes the SE matrices as the host rounds them to fp16."""
    from oracle import net as onet
    c, k, se = b["c_op"], b["k"], {NONE: None, CA: "ca_se", ECA: "eca_se"}[b["se"]]
    arch = dict(name="block", in_channels=256, policy_channels=2, channels=256, kernels=[k], se_types=[se], c_ops=[c],
                wdl=False, value_channels=8, value_fc=256)
    sd = onet.make_state_dict(arch, 0)

    def bn(prefix, bias):
        sd.update({prefix + ".weight": np.ones_like(bias), prefix + ".bias": bias, prefix + ".running_mean": np.zeros_like(bias),
                   prefix + ".running_var": np.full_like(bias, 1.0 - onet.BN_EPS)})
    w1, w2 = _selection_weights(b)
    sd["body_spatial.0.body.0.weight"] = _stem_identity()
    bn("body_spatial.0.body.1", np.zeros(256, f32))
    p = "body_spatial.1"
    sd[p + ".body.0.weight"] = w1[:, :, None, None]
    bn(p + ".body.1", b["b1"])
    sd[p + ".body.3.weight"] = b["wd"].reshape(c, 1, k, k)
    bn(p + ".body.4", b["bd"])
    sd[p + ".body.6.weight"] = w2[:, :, None, None]
    bn(p + ".body.7", b["b2"])
    if b["se"] == CA:
        sd[p + ".se.fc.0.weight"] = _r16(b["se_w1t"]).T.copy()
        sd[p + ".se.fc.2.weight"] = _r16(b["se_w2t"]).T.copy()
    elif b["se"] == ECA:
        w = np.zeros((256, 256, 5), f32)
        w[:, :, 2] = _r16(b["se_w1t"]).T  # a length-1 sequence: only the centre tap meets data
        sd[p + ".se.body.0.weight"], sd[p + ".se.body.0.bias"] = w, b["se_b"]
    n = x.shape[0]
    out = onet.forward(sd, arch, x.astype(f32).reshape(n, 8, 8, 256).transpose(0, 3, 1, 2))["trunk"]
    return out.transpose(0, 2, 3, 1).reshape(n, 64, 256)


def oracle_mx_block(x, b):
    """One block of oracle/net_mx.py (MXNet RISE symbols: shortcut before the SE, ca_se with biases, the block's gate)"""
    from oracle import net_mx as omx
    c, k = b["c_op"], b["k"]
    assert b["se"] != ECA  # the MXNet eca_se is a 5-tap convolution over the channel axis, not a dense matrix
    arch = dict(name="block", in_channels=256, policy_channels=2, channels=256, kernels=[k],
                se_types=["ca_se" if b["se"] == CA else None], c_ops=[c], wdl=False, value_channels=8, value_fc=256,
                semantics="mxnet", bn_names="v2", stem_act=False, policy_bias=False,
                se_gates=[{HARD6: None, HARD5: "hard_sigmoid", SIGMOID: "sigmoid"}[b["gate"]]],
                se_hidden=[128 if b["se"] == CA else None])
    p = omx.make_mx_params(arch, 0)

    def bn(name, bias):
        p.update({name + "_beta": bias, name + "_moving_mean": np.zeros_like(bias),
                  name + "_moving_var": np.full_like(bias, 1.0 - omx.BN_EPS)})
    w1, w2 = _selection_weights(b)
    p["stem_conv0_weight"] = _stem_identity()
    bn("stem_bn0", np.zeros(256, f32))
    q = "bc_res_block0"
    if b["se"] == CA:
        p[q + "_se_fc0_weight"] = _r16(b["se_w1t"]).T.copy()
        p[q + "_se_fc0_bias"] = b["se_b1"] if b.get("se_b1") is not None else np.zeros(128, f32)
        p[q + "_se_fc1_weight"] = _r16(b["se_w2t"]).T.copy()
        p[q + "_se_fc1_bias"] = b["se_b"] if b.get("se_b") is not None else np.zeros(256, f32)
    p[q + "_conv1_weight"] = w1[:, :, None, None]
    bn(q + "_bn1", b["b1"])
    p[q + "_conv2_weight"] = b["wd"].reshape(c, 1, k, k)
    bn(q + "_bn2", b["bd"])
    p[q + "_conv3_weight"] = w2[:, :, None, None]
    bn(q + "_bn3", b["b2"])
    n = x.shape[0]
    out = omx.forward_mx(p, arch, x.astype(f32).reshape(n, 8, 8, 256).transpose(0, 3, 1, 2))["trunk"]
    return out.transpose(0, 2, 3, 1).reshape(n, 64, 256)


def model_error_bound(x, b, mx):
    """A bound on |model - exact block| + |oracle - exact block|, elementwise, from the model's own intermediates.
    u = 2^-11 is fp16's unit roundoff; each fp32 sum of m terms is within gamma(m) = m 2^-24 / (1 - m 2^-24) of the
    sum of its absolute terms (both sides, any order); r = 2^-20 covers the oracle's fp32 batch-norm affines
    (1 / sqrt(var + eps) is 1 within a few 2^-24) and single fp32 adds.  Error terms propagate through the sums with the
    absolute weights and through relu and clamps with slope 1; the gates have slopes 1/6, 0.2 and 1/4, and their own
    evaluation (one FMA, or the logistic in float64 against torch's fp32) adds at most 2^-21; a hard gate clamped over
    the whole interval g +- G contributes no error.
      pool        P = 2 gamma(65) mean|x|
      ca_se       A = P |w1| + 2 gamma(257) (|b1| + |p| |w1|);  G = A |w2| + 2 gamma(129) (|b| + h |w2|)
      eca_se      G = P |w1| + 2 gamma(257) (|b| + |p| |w1|)
      scale       X = |x| (slope G + 2^-21) + (u + r) |x_se|, slope the gate's largest on [g - G, g + G]
      H1          E1 = X[sel1] + (u + r) |h1| + r |b1|
      depthwise   E2 = sum |wd| E1 + 2 gamma(k^2 + 1) (|bd| + sum |wd| |h1|) + r |acc| + u |h2|
      output      E2[sel2] + X (shortcut after the SE) + (u + r) |out| + r (|H2[sel2]| + |b2| + |shortcut|)"""
    u, r = 2.0 ** -11, 2.0 ** -20
    gam = lambda m: m * 2.0 ** -24 / (1 - m * 2.0 ** -24)  # noqa: E731
    xa = np.abs(x.astype(f64))
    xs, X = x, np.zeros_like(xa)
    if b["se"] != NONE:
        pool = np.abs(se_pool(x).astype(f64))
        P = 2 * gam(65) * xa.mean(axis=1)
        w1 = np.abs(_r16(b["se_w1t"]).astype(f64))
        if b["se"] == CA:
            b1 = 0.0 if b.get("se_b1") is None else np.abs(b["se_b1"].astype(f64))
            hid = _hidden(x, b, mx)
            A = P @ w1 + 2 * gam(257) * (b1 + pool @ w1)
            w2 = np.abs(_r16(b["se_w2t"]).astype(f64))
            bb = 0.0 if b.get("se_b") is None else np.abs(b["se_b"].astype(f64))
            G = A @ w2 + 2 * gam(129) * (bb + hid @ w2)
        else:
            G = P @ w1 + 2 * gam(257) * (np.abs(b["se_b"].astype(f64)) + pool @ w1)
        gate, diag = b["gate"] if mx else HARD6, {}
        s = se_scales(x, b, mx, diag=diag)
        g = diag["g"][0].astype(f64)
        if gate == SIGMOID:  # the largest slope of the logistic on [g - G, g + G]
            t = np.clip(0.0, g - G, g + G)
            slope = np.exp(-np.abs(t)) / (1.0 + np.exp(-np.abs(t))) ** 2
        else:  # 0 where the whole interval is clamped
            lin = LINEAR[gate]
            slope = np.where((g - G >= lin) | (g + G <= -lin), 0.0, 1 / 6 if gate == HARD6 else 0.2)
        xs = (x.astype(f32) * s[:, None, :]).astype(f16)
        X = xa * (slope * G + 2.0 ** -21)[:, None, :] + (u + r) * np.abs(xs.astype(f64))
    h1 = np.maximum(xs[:, :, b["sel1"]].astype(f32) + b["b1"], f32(0)).astype(f16)
    E1 = X[:, :, b["sel1"]] + (u + r) * np.abs(h1.astype(f64)) + r * np.abs(b["b1"].astype(f64))
    k, n = b["k"], x.shape[0]
    wd = np.abs(b["wd"].astype(f64))
    acc = _depthwise(h1.astype(f32), b["wd"], b["bd"], k).reshape(n, 64, -1)
    h2 = np.maximum(acc, f32(0)).astype(f16)
    E2 = (_depthwise(E1, wd, np.zeros(b["c_op"]), k) + 2 * gam(k * k + 1) * _depthwise(np.abs(h1.astype(f64)), wd,
          np.abs(b["bd"].astype(f64)), k)).reshape(n, 64, -1) + r * np.abs(acc.astype(f64)) + u * np.abs(h2.astype(f64))
    E3 = np.where(b["sel2"] >= 0, E2[:, :, np.maximum(b["sel2"], 0)], 0.0)
    d2 = np.abs(_select2(h2, b["sel2"]).astype(f64))
    out = np.abs(model(x, [b], mx).astype(f64))
    pre = mx and b["pre"]
    shortcut = xa if pre else np.abs(xs.astype(f64))
    return E3 + (0.0 if pre else X) + (u + r) * out + r * (d2 + np.abs(b["b2"].astype(f64)) + shortcut)


def _hidden(x, b, mx):
    a = _dot(_r16(b["se_w1t"]), se_pool(x))
    if mx and b.get("se_b1") is not None:
        a = b["se_b1"] + a
    return np.maximum(a, f32(0)).astype(f64)


def oracle_cases():
    cases = [(f"torch[{i}]", b, False, oracle_torch_block) for i, b in enumerate(tower("torch"))]
    cases += [(f"mx_pre[{i}]", b, True, oracle_mx_block) for i, b in enumerate(tower("mx_pre"))
              if b["pre"] and b["se"] != ECA]
    # the logistic gate at general inputs, where the bit-for-bit towers do not take it
    cases.append(("mx_pre[0] logistic", dict(tower("mx_pre")[0], gate=SIGMOID), True, oracle_mx_block))
    return cases


@pytest.mark.parametrize("case", range(len(TOWERS["torch"]) + 6))
def test_model_against_the_oracle_blocks(case):
    """Each block of the model against the same block of oracle/net.py (PyTorch RISE: ca_se, eca_se, shortcut after
    the SE) or oracle/net_mx.py (MXNet RISE: shortcut before the SE, ca_se biases, the three gates), one block at a
    time on a nonnegative input (the stem of oracle/net.py ends in a ReLU), within model_error_bound."""
    name, b, mx, oracle = oracle_cases()[case]
    # the PyTorch blocks' SE weights are scaled for the pooled values of a signed input (~N(0, 1/64)): a small input
    # keeps their gates off the clamps
    x = (tower_input("mx_pre", 3, seed=40 + case) * f16(1.0 if mx else 0.15)).astype(f16)
    got = model(x, [b], mx).astype(f64)
    want = oracle(x, b).astype(f64)
    bound = model_error_bound(x, b, mx)
    err = np.abs(got - want)
    assert (err <= bound).all(), f"{name}: {int((err > bound).sum())} outputs outside the bound, by {np.max(err - bound)}"
    assert np.median(bound / np.maximum(np.abs(want), 1e-3)) < 4e-3  # the bound is a few fp16 roundings, not vacuous


# ------------------------------------------------------------------------------------------------------------- GPU runs
def _run_trunk_se(x, blocks):
    """The tower kernel on x through ara_debug_trunk_se -> (output, 1 if the MXNet kernels ran)"""
    from crazyara_b200 import check, lib
    f = lib().ara_debug_trunk_se
    f.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int] + [ctypes.c_void_p] * 18
    f.restype = ctypes.c_int
    ints = lambda v: np.array(v, np.int32)  # noqa: E731

    def cat(key, arrays=None):
        parts = [a.ravel() for a in (arrays if arrays is not None else [b[key] for b in blocks]) if a is not None]
        return np.ascontiguousarray(np.concatenate(parts).astype(f32)) if parts else np.zeros(1, f32)

    w1, w2 = zip(*[_selection_weights(b) for b in blocks])
    arrs = [ints([b["c_op"] for b in blocks]), ints([b["k"] for b in blocks]), ints([b["se"] for b in blocks]),
            ints([b["gate"] for b in blocks]), ints([PRE * b["pre"] for b in blocks]),
            ints([(1 if b.get("se_b") is not None else 0) | (2 if b.get("se_b1") is not None else 0) for b in blocks]),
            cat("w1", w1), cat("b1"), cat("wd"), cat("bd"), cat("w2", w2), cat("b2"),
            cat("se_w1t", [b.get("se_w1t") for b in blocks]), cat("se_w2t", [b.get("se_w2t") for b in blocks]),
            cat("se_b", [b.get("se_b") for b in blocks]), cat("se_b1", [b.get("se_b1") for b in blocks])]
    x = np.ascontiguousarray(x)
    out = np.full_like(x, f16(np.nan))
    mx = ctypes.c_int(-1)
    check(f(x.ctypes.data, x.shape[0], len(blocks), *[a.ctypes.data for a in arrs], out.ctypes.data, ctypes.byref(mx)))
    return out, mx.value


def test_entry_refuses_what_a_weight_blob_cannot_describe():
    """A gate out of range, other flags, se_b1 outside ca_se, and a ca_se block with one of its two biases (the kernels
    take both or neither; without the MXNet semantics a lone se_b would be ignored) are refused before anything runs."""
    from crazyara_b200 import AraError
    base = tower("mx")[1]  # ca_se with both biases
    cases = [(dict(gate=3), "gate 3"), (dict(gate=-1), "gate -1"), (dict(pre=2), "flags 2"),
             (dict(se_b1=None), "biases 1"), (dict(se_b=None), "biases 2"), (dict(se=ECA, se_w2t=None), "biases 3"),
             (dict(se=NONE), "biases 3"), (dict(se=3), "type 3")]
    for change, msg in cases:
        b = dict(base, **change)
        with pytest.raises(AraError, match=msg):
            _run_trunk_se(tower_input("mx", 1), [b])


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(TOWERS))
@pytest.mark.parametrize("rows", SHAPES)
def test_tower_with_se_matches_the_model_bit_for_bit(monkeypatch, rows, name):
    monkeypatch.setenv("ARA_TRUNK_ROWS", rows)
    blocks = tower(name)
    for n in NS:
        x, want, _ = expected(name, n)
        got, mx = _run_trunk_se(x, blocks)
        assert mx == int(name != "torch")  # the MX=true kernels for the MXNet towers, the MX=false ones otherwise
        diff = got.view(np.uint16) != want.view(np.uint16)
        assert not diff.any(), (f"ARA_TRUNK_ROWS={rows} {name} n={n}: {int(diff.sum())} of {diff.size} outputs differ, "
                                f"first at {np.argwhere(diff)[0].tolist()}")


def logistic_block(seed=7):
    """An SE-only eca_se block with the logistic gate, its inputs spread over the whole curve (|g| up to ~10)"""
    rng = np.random.default_rng(seed)
    b = _block_spec(S(se=ECA, gate=SIGMOID, c=64, k=3, only=1))
    b.update(c_op=64, chunk0=0, sel1=rng.integers(0, 256, 64), sel2=np.full(256, -1), b1=np.zeros(64, f32),
             wd=np.zeros((64, 9), f32), bd=np.zeros(64, f32), b2=np.zeros(256, f32),
             se_w1t=rng.normal(0.0, 1.0, (256, 256)).astype(f32) * f32(3.0), se_w2t=None,
             se_b=rng.normal(0.0, 1.5, 256).astype(f32))
    return b


def _ordered(h):
    """fp16 bits -> integers in the order of the values (+0 and -0 both 0): neighbours differ by one"""
    v = h.view(np.uint16).astype(np.int32)
    return np.where(v & 0x8000, -(v & 0x7FFF), v)


@pytest.mark.gpu
@pytest.mark.parametrize("rows", SHAPES)
def test_logistic_gate_within_one_ulp(monkeypatch, rows):
    """The logistic gate at general inputs: the SE-only block outputs fp16(x * s) with s = 1 / (1 + expf(-g)).  expf is
    within 2 ulp of exp (CUDA C Programming Guide, mathematical functions, full range), 1 + expf rounds once and the
    division is IEEE, so s is within ~4 fp32 ulp of the float64 logistic of the model's exact gate input g (2^-22
    relative), and so is the fp32 product x * s.  Rounding two numbers that close to fp16 (2^-11 relative steps) gives
    the same or adjacent values: within one fp16 ulp of fp16(x * logistic(g)) evaluated in float64."""
    monkeypatch.setenv("ARA_TRUNK_ROWS", rows)
    b = logistic_block()
    x = tower_input("mx", 5, seed=3)
    diag = {}
    se_scales(x, b, True, diag=diag)
    g = diag["g"][0].astype(f64)
    assert np.abs(g).max() > 8.0 and np.mean(np.abs(g) < 4.0) > 0.5  # both tails and the curved middle
    want = (x.astype(f64) * (1.0 / (1.0 + np.exp(-g)))[:, None, :]).astype(f16)
    got, mx = _run_trunk_se(x, [b])
    assert mx == 1
    d = np.abs(_ordered(got) - _ordered(want))
    assert d.max() <= 1, f"ARA_TRUNK_ROWS={rows}: {int((d > 1).sum())} outputs more than one ulp away"
    assert (d == 0).mean() > 0.9
