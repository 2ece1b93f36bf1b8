"""The NextViT attention kernels (ntb_attention_kernel, ntb_attention_f32_kernel, ntb_attention.cuh) one launch at a time,
through ara_debug_ntb_attention, at every MHSA width the blob reader accepts (M = 32 .. 224, one to seven heads).

Two kinds of operands:
  exact    (float16 kernel) Q on a 2^-1 grid, K on a 2^-2 grid, V small integers, so that every score Q K^T is exact in
           fp32 and every row's spread keeps P = exp(s - max) >= 2^-6, a normal fp16 number.  The fp32 row sum of the
           fp16 P, P V and 1 / sum are then exact whatever order the tensor cores add in, and the output bits are fixed
           once the rounding of __expf to fp16 is: every exact exp(s - max) lies farther from an fp16 rounding midpoint
           than the documented error of __expf (2 + floor(1.173 |x|) ulp, CUDA C++ Programming Guide, intrinsic
           functions; this covers ex2.approx and the rounded multiply by log2 e).  Query rows that miss that margin are
           drawn again (test_exact_operands_sum_exactly checks every precondition).
  float64  random fp16 (float16 kernel) or fp32 (float32 kernel) q | k | v in five families, against the float64
           attention of the operands the kernel is given, within attention_bound, derived from the kernels' arithmetic.
test_each_mutation_changes_the_output shows that plausible mistakes in the float16 kernel change the exact rows' bits,
and test_bound_catches_precision_bugs that the float32 bound would catch an fp16 P or a dropped lo part.
"""
import ctypes
import zlib

import numpy as np
import pytest
import torch

f16, f32, f64 = np.float16, np.float32, np.float64
MS = tuple(range(32, 225, 32))
BOARDS = (1, 2, 5, 64, 140)  # 140: more boards than an H100 SXM has SMs (132)
SENT = 0x7E5A                # NaN pattern in the output rows and columns the kernel must leave alone
FAMILIES = ("realistic", "sharp", "onehot", "equal", "large")
U = 2.0 ** -24


def ceil64(v):
    return (v + 63) // 64 * 64


def _rng(*key):
    return np.random.default_rng(zlib.crc32(repr(key).encode()))


def heads(a, M):
    """[n * 64][M] -> [n][64][H][32]"""
    return a.reshape(-1, 64, M // 32, 32)


def split_qkv(qkv, M):
    """[n * 64][3M] -> q, k, v as [n][64][H][32] float64"""
    a = qkv.astype(f64).reshape(-1, 64, 3 * M)
    return heads(a[:, :, :M], M), heads(a[:, :, M:2 * M], M), heads(a[:, :, 2 * M:], M)


def scores(q, k):
    return np.einsum("nrhd,njhd->nhrj", q, k)


# ---------------------------------------------------------------------------------------------------- exact operands
def expf_intrinsic_ulps(x):
    """__expf's documented maximum error in ulp at x"""
    return 2.0 + np.floor(1.173 * np.abs(x))


def fp16_midpoint_distance(e):
    """distance of each e (> 0) to the nearest midpoint between two fp16 neighbours"""
    h = e.astype(f16)
    up = np.nextafter(h, f16(np.inf)).astype(f64)
    down = np.nextafter(h, f16(0)).astype(f64)
    h = h.astype(f64)
    return np.minimum(np.abs(e - (h + up) / 2), np.abs(e - (h + down) / 2))


def exp_margin_ok(x):
    """x = s - max (exact, <= 0) -> per element: exp(x) >= 2^-6 and farther from an fp16 midpoint than twice __expf's
    error bound (its ulp taken in the binade of the exact value, doubled for a result in the next one)"""
    e = np.exp(x)
    ulp = 2.0 ** (np.floor(np.log2(e)) - 23)
    return (e >= 2.0 ** -6) & (fp16_midpoint_distance(e) > 2 * expf_intrinsic_ulps(x) * ulp)


def _draw_q(rng, shape):
    return np.where(rng.random(shape + (32,)) < 6 / 32, rng.choice([-0.5, 0.5], shape + (32,)), 0.0)


def exact_operands(n, M):
    """q | k | v [n * 64][3M] fp16 and the number of query rows drawn again for the __expf margin"""
    rng = _rng("exact", n, M)
    H = M // 32
    k = rng.integers(-3, 4, (n, 64, H, 32)) * 0.25
    v = rng.integers(-2, 3, (n, 64, H, 32)).astype(f64)
    q = _draw_q(rng, (n, 64, H))
    redrawn = 0
    for _ in range(100):
        s = scores(q, k)
        bad = ~exp_margin_ok(s - s.max(-1, keepdims=True)).all(-1)  # [n, H, r]
        if not bad.any():
            break
        redrawn += int(bad.sum())
        bad = bad.transpose(0, 2, 1)
        q[bad] = _draw_q(rng, (int(bad.sum()),))
    else:
        raise AssertionError("no exact query rows")
    qkv = np.concatenate([a.reshape(n, 64, M) for a in (q, k, v)], axis=2).reshape(n * 64, 3 * M)
    return qkv.astype(f16), redrawn


MUTATIONS = ["key_swap_in_chunk", "key_chunk_swizzle", "vt_transposed_chunk", "unrounded_sum", "max_rows_r_r8",
             "neighbour_head", "k_v_offsets_swapped"]


def half_model(qkv, M, mut=()):
    """the float16 kernel's output [n * 64][M] fp16 for exact operands, in its order of operations where that decides
    bits: P = fp16(exp(s - max)), sum = the fp32 sum of the fp16 P, O = P V, out = fp16(O * (1 / sum))"""
    q, k, v = split_qkv(qkv, M)
    if "neighbour_head" in mut:
        q, k, v = (np.roll(a, -1, axis=2) for a in (q, k, v))
    if "k_v_offsets_swapped" in mut:
        k, v = v, k
    ks = k.copy()
    if "key_swap_in_chunk" in mut:
        ks = ks[:, np.arange(64) ^ 1]
    if "key_chunk_swizzle" in mut:
        ks[:, 1::8] = ks[:, 1::8][..., np.r_[8:16, 0:8, 16:32]]
    if "vt_transposed_chunk" in mut:
        v = v.copy()
        v[:, :8, :, :8] = v[:, :8, :, :8].transpose(0, 3, 2, 1)
    s = scores(q, ks)
    mx = s.max(-1, keepdims=True)
    if "max_rows_r_r8" in mut:
        g = mx.reshape(mx.shape[0], mx.shape[1], 4, 2, 8, 1)
        mx = np.maximum(g[:, :, :, :1], g[:, :, :, 1:]).repeat(2, axis=3).reshape(mx.shape)
    e = np.exp(s - mx)
    p = e.astype(f16).astype(f64)
    total = (e.astype(f32).astype(f64) if "unrounded_sum" in mut else p).sum(-1)
    o = np.einsum("nhrj,njhd->nrhd", p, v)
    inv = (f32(1) / total.astype(f32)).transpose(0, 2, 1)[..., None]
    return (o.astype(f32) * inv).astype(f16).reshape(-1, M)


# ------------------------------------------------------------------------------------------------- float64 operands
def float64_operands(n, M, family, prec):
    """q | k | v [n * 64][3M] as the kernel reads them: fp16 (prec 0) or fp32 (prec 1)"""
    rng = _rng("float64", n, M, family, prec)
    H = M // 32
    sh = (n, 64, H, 32)
    q, k, v = rng.standard_normal(sh) * 0.6, rng.standard_normal(sh) * 0.6, rng.standard_normal(sh) * 0.4
    if family == "sharp":  # score spread +-30: fp16 P subnormal or zero
        q *= 12
    elif family == "onehot":  # one key per head 144 above the rest: exp underflows to 0 in fp32 and fp16
        q *= 0.1
        q[..., 0] = 12.0
        k[..., 0] = 0.0
        hot = rng.integers(0, 64, (n, H))
        k[np.arange(n)[:, None], hot, np.arange(H)[None, :], 0] = 12.0
    elif family == "equal":
        q[:] = 0.0
    elif family == "large":  # scores near 960 with a spread of a few units: the max subtraction
        q[..., 0] = 32.0
        k[..., 0] = 30.0
    qkv = np.concatenate([a.reshape(n, 64, M) for a in (q, k, v)], axis=2).reshape(n * 64, 3 * M)
    return qkv.astype(f16 if prec == 0 else f32)


def attention_bound(qkv, M, prec, device="cpu"):
    """(float64 attention [n * 64][M], bound before the output rounding, bound on the output) of the operands as given.

    Scores: fp32 accumulation of the 32 products, float16 in two wgmma k-steps (u_acc = 2^-23 per step, as
    tests/test_conv_gemm_gpu.py assumes: E_s = 2 * 2^-23 sum |q k|), float32 in 32 fmaf in order (E_s = 2^-24 sum_d |S_d|,
    S_d the partial sums, 1% added for the second order).  The max is one of
    the computed scores, the subtraction rounds (2^-24 |x|), so the exponent is off by dx = E_s + max E_s + 2^-24 |x|.
    exp: __expf 2 + 1.173 |x| ulp (float16), expf 2 ulp (float32); float16 rounds P to fp16 (2^-11, and 2^-25 absolute
    below the normal range, with 2^-126 for the flush to zero).  P_j = e_j (1 + t_j) + a_j then moves the normalised
    result by at most sum_j (e_j t_j + a_j) |v_j - o| / (sum_j e_j (1 - t_j) - 64 a), since sum_j e_j (v_j - o) = 0.  The
    fp32 sums: P V (float16 four wgmma k-steps, 4 * 2^-23 sum |P v|; float32 64 fmaf, 64 * 2^-24) and sum P (float16 18
    adds in a lane quad, float32 64 adds, n * 2^-24 sum P); IEEE 1 / sum and the product, 2^-24 each.  Output: fp16 half
    an ulp (2^-11 |o| + 2^-25); the split hi + lo 2^-22 |o| + 2^-24."""
    q, k, v = (torch.from_numpy(a).to(device) for a in split_qkv(qkv, M))
    s = torch.einsum("nrhd,njhd->nhrj", q, k)
    A = torch.einsum("nrhd,njhd->nhrj", q.abs(), k.abs())
    m = s.amax(-1, keepdim=True)
    x = s - m
    e = torch.exp(x)
    D = e.sum(-1)
    vv = v.permute(0, 2, 1, 3)  # [n, H, j, d]
    o = torch.einsum("nhrj,nhjd->nhrd", e, vv) / D[..., None]
    if prec == 0:
        Es = 2 * 2.0 ** -23 * A
    else:  # fmaf in order d = 0 .. 31: each rounds its partial sum S_d by at most 2^-24 |S_d|
        Es, S = torch.zeros_like(s), torch.zeros_like(s)
        for d in range(32):
            S += q[:, :, :, d].permute(0, 2, 1)[..., None] * k[:, :, :, d].permute(0, 2, 1)[:, :, None, :]
            Es += S.abs()
        Es = 1.01 * U * Es
    dx = Es + Es.amax(-1, keepdim=True) + U * x.abs()
    ulps = 2.0 + 1.173 * (x.abs() + dx) if prec == 0 else torch.full_like(x, 2.0)
    t = torch.exp(dx) * (1 + ulps * 2.0 ** -23) * (1 + (2.0 ** -11 if prec == 0 else 0.0)) - 1
    a = 2.0 ** -25 + 2.0 ** -125 if prec == 0 else 2.0 ** -140
    diff = (vv[:, :, None, :, :] - o[:, :, :, None, :]).abs()  # [n, H, r, j, d]
    b1 = torch.einsum("nhrj,nhrjd->nhrd", e * t + a, diff)
    d_low = (e * (1 - t)).sum(-1) - 64 * a
    b1 = b1 / d_low[..., None]
    p_hi = e * (1 + t) + a
    EN = (4 * 2.0 ** -23 if prec == 0 else 64 * U) * torch.einsum("nhrj,nhjd->nhrd", p_hi, vv.abs())
    ED = (18 if prec == 0 else 64) * U * p_hi.sum(-1)
    om = o.abs() + b1
    pre = b1 + (EN + om * ED[..., None]) / (d_low - ED)[..., None]
    pre = pre + 2.1 * U * (om + pre)
    out = pre + (2.0 ** -11 * (o.abs() + pre) + 2.0 ** -25 if prec == 0 else 2.0 ** -22 * (o.abs() + pre) + 2.0 ** -24)
    flat = lambda z: z.permute(0, 2, 1, 3).reshape(-1, M)  # noqa: E731
    return flat(o), flat(pre), flat(out)


# --------------------------------------------------------------------------------------------------------- CPU half
@pytest.mark.parametrize("M", MS)
def test_exact_operands_sum_exactly(M):
    """The exact cases' precondition at every batch the GPU test runs: scores exact in fp32 (multiples of 2^-3 far below
    2^21), P >= 2^-6 and the __expf margin, P on the 2^-16 grid, and the P V sums and row sums below 2^24 grid units"""
    for n in BOARDS:
        qkv, _ = exact_operands(n, M)
        q, k, v = split_qkv(qkv, M)
        s = scores(q, k)
        assert (s * 8 == np.round(s * 8)).all() and np.abs(s).max() * 8 < 2 ** 21
        x = s - s.max(-1, keepdims=True)
        assert exp_margin_ok(x).all()
        p = np.exp(x).astype(f16).astype(f64)
        assert (p >= 2.0 ** -6).all() and (p * 2 ** 16 == np.round(p * 2 ** 16)).all()
        assert (np.abs(v) <= 2).all()
        budget = np.einsum("nhrj,njhd->nrhd", p, np.abs(v)).max() * 2 ** 16
        assert budget < 2 ** 24 and p.sum(-1).max() * 2 ** 16 < 2 ** 24
        out = half_model(qkv, M).astype(f64)
        assert np.isfinite(out).all() and (out != np.round(out)).mean() > 0.5  # the division and rounding are exercised


def test_exact_redraws_are_counted():
    """The margin is met by redrawing query rows; report how often (a row of 64 scores rarely misses it)"""
    total = sum(exact_operands(n, M)[1] for M in MS for n in BOARDS)
    rows = sum(n * 64 * (M // 32) for M in MS for n in BOARDS)
    print(f"exact attention cases: {total} of {rows} query rows redrawn for the __expf margin")
    assert total < rows // 4


@pytest.mark.parametrize("mut", MUTATIONS)
def test_each_mutation_changes_the_output(mut):
    """On the GPU test's own operands, each plausible mistake changes at least one bit of the exact output"""
    for M in MS:
        if mut == "neighbour_head" and M == 32:
            continue
        qkv, _ = exact_operands(2, M)
        want = half_model(qkv, M)
        got = half_model(qkv, M, (mut,))
        assert (got.view(np.uint16) != want.view(np.uint16)).any(), f"M={M}: {mut} keeps every bit"


@pytest.mark.parametrize("M", [32, 96, 224])
def test_bound_catches_precision_bugs(M):
    """On the network's spread of scores, the float32 bound is at least 10x below the error of P rounded to fp16 (the
    float16 kernel's arithmetic) and of the lo part dropped, at some output: the GPU test would catch either.  (Sharp
    and large scores carry fp32 score errors that exp amplifies beyond fp16's rounding.)"""
    family = "realistic"
    qkv = float64_operands(2, M, family, 1)
    ref, _, bound = attention_bound(qkv, M, 1)
    q, k, v = split_qkv(qkv, M)
    s = scores(q, k)
    p = np.exp(s - s.max(-1, keepdims=True)).astype(f16).astype(f64)
    fp16_p = torch.from_numpy((np.einsum("nhrj,njhd->nrhd", p, v) /
                               p.sum(-1).transpose(0, 2, 1)[..., None]).reshape(-1, M))
    hi_only = torch.from_numpy(ref.numpy().astype(f16).astype(f64))
    for what, bad in (("fp16 P", fp16_p), ("lo dropped", hi_only)):
        ratio = ((bad - ref).abs() / bound).max().item()
        assert ratio >= 10.0, f"{family}: {what} exceeds the bound by only {ratio:.2f}x"


def _refused(*args):
    from crazyara_b200 import lib
    f = lib().ara_debug_ntb_attention
    f.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_void_p]
    f.restype = ctypes.c_int
    buf = np.zeros(8, f32)
    rc = f(buf.ctypes.data, *args, buf.ctypes.data)
    lib().ara_last_error.restype = ctypes.c_char_p
    return rc != 0 and b"ara_debug_ntb_attention" in lib().ara_last_error()


@pytest.mark.parametrize("n,M,prec,count", [(1, 0, 0, -1), (1, 16, 0, -1), (1, 48, 0, -1), (1, 256, 1, -1), (0, 64, 0, -1),
                                            (1, 64, 2, -1), (1, 64, -1, -1), (2, 64, 0, 3), (2, 64, 0, -2)])
def test_refusals_need_no_device(n, M, prec, count):
    """widths the blob reader refuses, empty batches, unknown precisions and counts beyond the batch are refused by
    name before any device call"""
    assert _refused(n, M, prec, count)


# ---------------------------------------------------------------------------------------------------------- GPU runs
def run(qkv, n, M, prec, count=-1):
    """launch -> the output buffer [n * 64][M] (split: [n * 64][3 * ceil64(M)]) as uint16, initialised to SENT"""
    from crazyara_b200 import check, lib
    width = M if prec == 0 else 3 * ceil64(M)
    out = np.full((n * 64, width), SENT, np.uint16)
    f = lib().ara_debug_ntb_attention
    f.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_void_p]
    f.restype = ctypes.c_int
    qkv = np.ascontiguousarray(qkv)
    check(f(qkv.ctypes.data, n, M, prec, count, out.ctypes.data))
    return out


def _first_diff(got, want):
    d = got != want
    return f"{int(d.sum())} of {d.size} differ, first at {np.argwhere(d)[0].tolist()}"


@pytest.mark.gpu
@pytest.mark.parametrize("M", MS)
def test_exact_bit_for_bit(M):
    """float16 kernel, every batch of BOARDS: the output equals the model's bits; with a device-side count of n // 2 the
    rows of the boards from it keep the sentinel and the others have the bits of the full launch"""
    for n in BOARDS:
        qkv, _ = exact_operands(n, M)
        want = half_model(qkv, M).view(np.uint16)
        got = run(qkv, n, M, 0)
        assert (got == want).all(), f"M={M} n={n}: {_first_diff(got, want)}"
        if n >= 2:
            k = n // 2
            part = run(qkv, n, M, 0, k)
            assert (part[:k * 64] == want[:k * 64]).all() and (part[k * 64:] == SENT).all(), f"M={M} n={n} count={k}"


@pytest.mark.gpu
@pytest.mark.parametrize("prec", [0, 1])
def test_board_gives_the_same_bits_at_any_index(prec):
    """one board's q | k | v at indices 0, 1, 70 and 139 of a 140-board launch and alone: the same output bits"""
    for M in (96, 224):
        qkv = float64_operands(140, M, "realistic", prec).reshape(140, 64, 3 * M)
        for i in (1, 70, 139):
            qkv[i] = qkv[0]
        got = run(qkv.reshape(-1, 3 * M), 140, M, prec).reshape(140, 64, -1)
        alone = run(qkv[0], 1, M, prec)
        for i in (0, 1, 70, 139):
            assert (got[i] == alone).all(), f"prec {prec} M={M}: board at index {i}"


def check_within_bound(n, M, family, prec):
    """-> the largest |error| / bound over the outputs"""
    qkv = float64_operands(n, M, family, prec)
    ref, pre, bound = attention_bound(qkv, M, prec, "cuda")
    got = run(qkv, n, M, prec)
    if prec == 0:
        val = got.view(f16).astype(f64)
    else:
        cs = ceil64(M)
        s = got.reshape(n * 64, 3, cs)
        assert (s[:, :, M:] == SENT).all(), f"M={M}: padding columns written"
        assert (s[:, 0] == s[:, 1]).all(), f"M={M}: the two hi copies differ"
        hi, lo = s[:, 0, :M].view(f16), s[:, 2, :M].view(f16)
        h = hi.astype(f64)
        half_ulp = np.maximum(np.nextafter(hi, f16(np.inf)).astype(f64) - h, h - np.nextafter(hi, f16(-np.inf)).astype(f64)) / 2
        assert (np.abs(lo.astype(f64)) <= half_ulp).all(), f"M={M}: lo is not the remainder of hi"
        r = ref.cpu().numpy()
        sure = fp16_midpoint_distance(np.abs(r)) > pre.cpu().numpy()
        assert (hi.view(np.uint16)[sure] == r.astype(f16).view(np.uint16)[sure]).all(), f"M={M}: hi != fp16(reference)"
        val = hi.astype(f64) + lo.astype(f64)
    err = (torch.from_numpy(val).cuda() - ref).abs()
    assert torch.isfinite(err).all(), f"{family} M={M} n={n}: non-finite output"
    ratio = torch.where(err == 0, 0.0, err / bound).max().item()
    assert ratio <= 1.0, f"{family} prec {prec} M={M} n={n}: error {ratio:.3g}x the bound at {int((err > bound).sum())} outputs"
    if family == "onehot":  # exactly one-hot after rounding: the output is V[argmax] (split: hi = fp16(v), lo the rest)
        q, k, v = split_qkv(qkv, M)
        hot = scores(q, k).argmax(-1)  # [n, H, r]
        vh = v[np.arange(n)[:, None, None], hot, np.arange(M // 32)[None, :, None]]  # [n, H, r, d]
        want = vh.transpose(0, 2, 1, 3).reshape(-1, M).astype(f32)
        want_hi = want.astype(f16)
        if prec == 0:
            assert (got.view(f16) == want_hi).all(), f"M={M}: not V[argmax]"
        else:
            want_lo = (want - want_hi.astype(f32)).astype(f16)
            assert (hi == want_hi).all() and (lo.view(np.uint16) == want_lo.view(np.uint16)).all(), f"M={M}: not V[argmax]"
    return ratio


@pytest.mark.gpu
@pytest.mark.parametrize("prec", [0, 1])
@pytest.mark.parametrize("family", FAMILIES)
def test_float64_within_bound(family, prec):
    worst = 0.0
    for M in MS:
        for n in (BOARDS if family == "realistic" else (5,)):
            worst = max(worst, check_within_bound(n, M, family, prec))
    print(f"attention {family} precision {prec}: largest error / bound {worst:.3g}")
