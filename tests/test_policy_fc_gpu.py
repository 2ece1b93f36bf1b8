"""The fully-connected policy layer (policy_fc_kernel<BN>, policy_fc.cuh, and policy_fc_softmax_kernel, net_kernels.cuh)
one launch at a time, through ara_debug_policy_fc, which builds the layer with the network's own builder
(policy_fc_build, policy_fc_weight_image).

Exact operands on a power-of-two grid make every product and every partial sum of a split exact in fp32 whatever
order the tensor cores add in (test_exact_operands_sum_exactly): every partial sum then equals the float64 sum over its
split's K range, bit for bit, and the logits b_fc + part[0] + part[1] + ... follow in fp32 in split order.  Float32
runs twice, with fp16-exact weights (w_lo = 0) and with fp16-exact activations (a_lo = 0).  The probabilities are
checked against the float64 softmax of those logits within softmax_bound.  test_each_mutation_changes_the_output shows
that plausible mistakes change the exact bits, test_split_order_decides_the_bits that the split-order case pins the
reduction order.
"""
import ctypes
import functools
import zlib

import numpy as np
import pytest
import torch

f16, f32, f64 = np.float16, np.float32, np.float64
# (P, L): the network tables' heads, AlphaVile tiny, and the smallest and largest P and L the blob reader accepts
SHAPES = [(81, 2272), (76, 1968), (2, 2316), (16, 1968), (81, 2316), (1, 1968), (1, 2316), (256, 1968), (256, 2316)]
BATCHES = (1, 31, 32, 33, 64, 65, 66, 127, 128)  # a full and a partial board tile at every N tile
BNS = (32, 64, 128)
KINDS = {0: ("fp16",), 1: ("w_exact", "a_exact")}
SENT = 0x7FC5A5A5  # NaN pattern in the partial sums and probabilities the kernels must leave alone
U = 2.0 ** -24


def ceil_to(v, m):
    return (v + m - 1) // m * m


def _rng(*key):
    return np.random.default_rng(zlib.crc32(repr(key).encode()))


def rows_cap(batch):
    return ceil_to(max(batch, 2), 2)


def square_cols(P, prec):
    return ceil_to(P, 32) if prec == 0 else 3 * ceil_to(P, 64)


def split_formula(L, K):
    """(kb_per_split, splits): about kFcTargetCtas = 264 CTAs of label tiles x splits, from L and K only"""
    m_tiles, num_kb = ceil_to(L, 64) // 64, K // 64
    want = -(-264 // m_tiles)
    kb = -(-num_kb // want)
    return kb, -(-num_kb // kb)


def choose_bn(batch):
    return 32 if batch <= 32 else 64 if batch <= 64 else 128


def weight_image(W, L, P, prec, mut=()):
    """W [L][P * 64] fp32 (NCHW) -> fp16 [ceil64(L)][K]: per square the channels (float16), or hi | lo | hi (float32)"""
    W3 = W.reshape(L, 64, P).transpose(0, 2, 1) if "nchw_not_permuted" in mut else W.reshape(L, P, 64)
    hi = W3.astype(f16)
    lo = (W3 - hi.astype(f32)).astype(f16)
    sc = square_cols(P, prec)
    img = np.zeros((ceil_to(L, 64), 64, sc), f16)
    if prec == 0:
        img[:L, :, :P] = hi.transpose(0, 2, 1)
    else:
        cs = sc // 3
        for i, part in enumerate((hi, hi, lo) if "parts_misaligned" in mut else (hi, lo, hi)):
            img[:L, :, i * cs:i * cs + P] = part.transpose(0, 2, 1)
    return img.reshape(ceil_to(L, 64), 64 * sc)


def k_ranges(K, kb, splits, mut=()):
    num_kb = K // 64
    r = [(s * kb * 64, min((s + 1) * kb, num_kb) * 64) for s in range(splits)]
    if "last_split_full" in mut:
        r[-1] = ((num_kb - kb) * 64, num_kb * 64)
    return r


# --------------------------------------------------------------------------------------------------------- operands
def exact_operands(P, L, prec, kind, batch):
    """W, b, x on a grid: float16 x, W in {0, +-1, +-2(, +-3)} 2^-3; float32 sparse x_hi = +-2^-3 (about 384 nonzero per
    board, so that sums of the 2^-19 products stay below 2^24 units) with the lo parts +-{1, 2, 3} 2^-16"""
    W, b = exact_weights(P, L, prec, kind)
    rng = _rng("exact", P, L, prec, kind, batch)
    cap = rows_cap(batch)
    sc = square_cols(P, prec)
    x = np.zeros((cap, 64, sc), f64)
    if prec == 0:
        x[:, :, :P] = rng.integers(-2, 3, (cap, 64, P)) * 2.0 ** -3
        unit = 2.0 ** -6
    else:
        cs = sc // 3
        dens = min(1.0, 384 / (64 * P))
        xh = np.where(rng.random((cap, 64, P)) < dens, rng.choice([-1.0, 1.0], (cap, 64, P)), 0.0) * 2.0 ** -3
        x[:, :, :P] = xh
        x[:, :, cs:cs + P] = xh
        if kind == "w_exact":
            x[:, :, 2 * cs:2 * cs + P] = np.where(xh != 0, rng.integers(-3, 4, (cap, 64, P)), 0) * 2.0 ** -16
        unit = 2.0 ** -19
    return W.copy(), b.copy(), x.reshape(cap, -1).astype(f16), unit


@functools.lru_cache(maxsize=4)
def exact_weights(P, L, prec, kind):
    rng = _rng("exact weights", P, L, prec, kind)
    w_hi = rng.integers(-3, 4, (L, P * 64)) * 2.0 ** -3
    if kind == "a_exact":
        w_hi = np.where(w_hi == 0, 2.0 ** -3, w_hi)
        W = w_hi + rng.integers(-3, 4, w_hi.shape) * 2.0 ** -16
    else:
        W = w_hi
    b = rng.integers(-8, 9, L) * 2.0 ** -3
    return W.astype(f32), b.astype(f32)


@functools.lru_cache(maxsize=4)
def cached_image(P, L, prec, kind):
    return weight_image(exact_weights(P, L, prec, kind)[0], L, P, prec)


def split_order_operands(batch):
    """P 81, L 2272, float16: for labels 5 and 700 of every board, split 0 sums to 2^24 + 2, split 1 to 1, split 2 to
    -2^24, each exactly; their fp32 sum in split order is 4, in reverse or pairwise order 3"""
    P, L = 81, 2272
    ldp = ceil_to(P, 32)
    K = 64 * ldp
    kb, splits = split_formula(L, K)
    W = np.zeros((L, P * 64), f32)
    x = np.zeros((rows_cap(batch), K), f16)

    def put(k, wv, xv):
        sq, c = divmod(k, ldp)
        assert c < P
        W[[5, 700], c * 64 + sq] = wv
        x[:, k] = xv
    put(0, 2.0 ** 12, 2.0 ** 12)
    put(1, 1.0, 2.0)
    put(kb * 64, 1.0, 1.0)
    put(2 * kb * 64, -2.0 ** 12, 2.0 ** 12)
    return P, L, W, np.zeros(L, f32), x


def partials(img, x, ranges, device="cpu"):
    """[splits][rows][lp] float64 sums over each split's K range"""
    X = torch.from_numpy(x.astype(f64)).to(device)
    I = torch.from_numpy(img.astype(f64)).to(device)
    return torch.stack([X[:, a:b] @ I[:, a:b].T for a, b in ranges]).cpu().numpy()


def written_rows(n, bn, cap, count=None):
    tiles = -(-n // bn)
    rows = np.zeros(cap, bool)
    for t in range(tiles):
        if count is not None and t * bn >= count:
            continue
        rows[t * bn:min(t * bn + bn, cap)] = True
    return rows


def expected_partials(part, n, bn, count=None, mut=()):
    """the partial-sum buffer after the launch: fp32 sums in the written rows, the sentinel elsewhere"""
    splits, cap, lp = part.shape
    want = np.full(part.shape, SENT, np.uint32).view(f32)
    rows = written_rows(n, bn, cap, count)
    val = part.astype(f32)
    if "label_l0_plus_8_dropped" in mut:  # acc of label l0 + 8 lands on l0; l0 + 8 stays unwritten
        v = val.reshape(splits, cap, lp // 16, 2, 8)
        val = np.concatenate([v[:, :, :, 1:], np.full_like(v[:, :, :, :1], np.nan)], axis=3).reshape(part.shape)
    if "board_e_fixed" in mut:  # both boards of a pair written to the even one (the odd one's value last)
        v = val.reshape(splits, cap // 2, 2, lp)
        val = np.stack([v[:, :, 1], np.full_like(v[:, :, 1], np.nan)], axis=2).reshape(part.shape)
    want[:, rows] = val[:, rows]
    return want


def logits_in_split_order(b, part, L, order="split"):
    """fp32 b + part[0] + part[1] + ... [rows][L]"""
    terms = [b.astype(f32)] + [p[:, :L].astype(f32) for p in part]
    if order == "reverse":
        terms = terms[:1] + terms[1:][::-1]
    if order == "pairwise":
        while len(terms) > 1:
            terms = [terms[i] + terms[i + 1] if i + 1 < len(terms) else terms[i] for i in range(0, len(terms), 2)]
        return np.broadcast_to(terms[0], part.shape[1:2] + (L,)).astype(f32)
    acc = np.broadcast_to(terms[0], part.shape[1:2] + (L,)).astype(f32)
    for t in terms[1:]:
        acc = acc + t
    return acc


def softmax_bound(logits):
    """(float64 softmax, bound) per row of fp32 logits.  block_softmax_256: the max is exact, l - max rounds (2^-24 |x|),
    expf 2 ulp, the sum of the e adds at most 10 terms per thread, 5 shuffle levels and 8 warps (23 adds, 23 * 2^-24
    sum e), 1 / sum and e * inv round once each (2^-24); subnormal e and p are off by at most 2^-146 absolute."""
    l = logits.astype(f64)
    x = l - l.max(-1, keepdims=True)
    e = np.exp(x)
    p = e / e.sum(-1, keepdims=True)
    de = 2 * 2.0 ** -23 + U * np.abs(x) * 1.01
    ds = (e * de).sum(-1, keepdims=True) / e.sum(-1, keepdims=True) + 23 * U
    bound = p * ((1 + de) * (1 + U) ** 2 / (1 - ds) - 1) + 2.0 ** -146 * 4
    return p, bound


# ---------------------------------------------------------------------------------------------------------- the entry
_ARGS = [ctypes.c_int] * 7 + [ctypes.c_void_p] * 7


def entry():
    from crazyara_b200 import lib
    f = lib().ara_debug_policy_fc
    f.argtypes = _ARGS
    f.restype = ctypes.c_int
    return f


def reported_split(P, L, prec, batch):
    kb, sp = ctypes.c_int(-1), ctypes.c_int(-1)
    from crazyara_b200 import check
    check(entry()(prec, P, L, batch, batch, 0, -1, None, None, None, None, None, ctypes.addressof(sp), ctypes.addressof(kb)))
    return kb.value, sp.value


def run(P, L, prec, W, b, x, n, batch, bn=0, count=-1):
    """-> (partial sums [splits][rows_cap][lp], probabilities [n][L]) from buffers initialised to SENT"""
    from crazyara_b200 import check
    K = 64 * square_cols(P, prec)
    kb, splits = split_formula(L, K)
    part = np.full((splits, rows_cap(batch), ceil_to(L, 64)), SENT, np.uint32).view(f32)
    prob = np.full((n, L), SENT, np.uint32).view(f32)
    W, b, x = (np.ascontiguousarray(a) for a in (W, b, x))
    sp, kbr = ctypes.c_int(-1), ctypes.c_int(-1)
    check(entry()(prec, P, L, n, batch, bn, count, W.ctypes.data, b.ctypes.data, x.ctypes.data, part.ctypes.data,
                  prob.ctypes.data, ctypes.addressof(sp), ctypes.addressof(kbr)))
    assert (sp.value, kbr.value) == (splits, kb)
    return part, prob


# --------------------------------------------------------------------------------------------------------- CPU half
def test_split_formula_depends_on_l_and_k_only():
    """The entry reports the host model's split count and K blocks per split at every batch (no device needed)"""
    assert split_formula(1968, 64 * 96) == (11, 9)  # L 1968, P 76: 9 splits, the last with 8 of 11 K blocks
    for P, L in SHAPES:
        for prec in (0, 1):
            want = split_formula(L, 64 * square_cols(P, prec))
            for batch in BATCHES:
                assert reported_split(P, L, prec, batch) == want, (P, L, prec, batch)


@pytest.mark.parametrize("P,L", SHAPES)
def test_exact_operands_sum_exactly(P, L):
    """For every exact case: the operands lie on their grid and each output's sum of |products| is below 2^24 grid
    units, so every partial sum of any split, in any order, is exact in fp32"""
    for prec in (0, 1):
        for kind in KINDS[prec]:
            W, b, x, unit = exact_operands(P, L, prec, kind, 66)
            img = weight_image(W, L, P, prec)
            if kind != "a_exact":
                assert (img.astype(f32)[:, :] * 8 == np.round(img.astype(f32) * 8)).all()
            t = partials(np.abs(img), np.abs(x), [(0, img.shape[1])])[0]
            assert t.max() / unit < 2 ** 24, (P, L, prec, kind, t.max() / unit)
            if prec == 1:  # both product terms exercised: hi x hi and one lo part
                cs = square_cols(P, 1) // 3
                xs = x.reshape(x.shape[0], 64, 3, cs)
                im = img.reshape(img.shape[0], 64, 3, cs)
                assert (xs[:, :, 2] != 0).any() if kind == "w_exact" else (im[:, :, 1] != 0).any()
    P2, L2, W, b, x = split_order_operands(3)
    part = partials(weight_image(W, L2, P2, 0), x, k_ranges(x.shape[1], *split_formula(L2, x.shape[1])))
    assert part[0, 0, 5] == 2 ** 24 + 2 and part[1, 0, 5] == 1 and part[2, 0, 5] == -2 ** 24


MUTATIONS = ["label_l0_plus_8_dropped", "board_e_fixed", "last_split_full", "parts_misaligned", "nchw_not_permuted"]


@pytest.mark.parametrize("mut", MUTATIONS)
def test_each_mutation_changes_the_output(mut):
    """On the GPU test's kind of operands (P 76, L 1968: 9 splits, the last one shorter), each plausible mistake changes
    at least one bit of the expected partial sums"""
    P, L, B = 76, 1968, 3
    for prec in (0, 1):
        for kind in KINDS[prec]:
            W, b, x, _ = exact_operands(P, L, prec, kind, B)
            K = x.shape[1]
            kb, splits = split_formula(L, K)
            want = expected_partials(partials(weight_image(W, L, P, prec), x, k_ranges(K, kb, splits)), B, 32)
            got = expected_partials(partials(weight_image(W, L, P, prec, (mut,)), x, k_ranges(K, kb, splits, (mut,))), B, 32,
                                    mut=(mut,))
            if (got.view(np.uint32) != want.view(np.uint32)).any():
                return
    pytest.fail(f"no exact case sees {mut}")


def test_split_order_decides_the_bits():
    P, L, W, b, x = split_order_operands(3)
    K = x.shape[1]
    part = partials(weight_image(W, L, P, 0), x, k_ranges(K, *split_formula(L, K)))
    seq, rev, pair = (logits_in_split_order(b, part, L, o) for o in ("split", "reverse", "pairwise"))
    assert seq[0, 5] == 4 and rev[0, 5] == 3 and pair[0, 5] == 3


def test_softmax_bound_catches_an_fp16_exponential():
    """the bound is at least 10x below the error of e rounded to fp16 before the normalisation"""
    rng = _rng("softmax")
    l = (rng.standard_normal((4, 1968)) * 2).astype(f32)
    p, bound = softmax_bound(l)
    e = np.exp(l.astype(f64) - l.max(-1, keepdims=True)).astype(f16).astype(f64)
    bad = e / e.sum(-1, keepdims=True)
    assert (np.abs(bad - p) / bound).max() >= 10


@pytest.mark.parametrize("args", [
    (2, 76, 1968, 1, 1, 0, -1), (0, 0, 1968, 1, 1, 0, -1), (0, 257, 1968, 1, 1, 0, -1), (0, 76, 2000, 1, 1, 0, -1),
    (0, 76, 1968, 0, 1, 0, -1), (0, 76, 1968, 2, 1, 0, -1), (0, 76, 1968, 1, 1, 16, -1), (0, 76, 1968, 1, 1, 256, -1),
    (0, 76, 1968, 2, 2, 0, 3), (0, 76, 1968, 2, 2, 0, -2)])
def test_refusals_need_no_device(args):
    """precision, P, L, boards beyond the batch, N tiles and counts outside their range are refused by name"""
    from crazyara_b200 import lib
    buf = np.zeros(8, f32)
    assert entry()(*args, *([buf.ctypes.data] * 5), None, None) != 0
    lib().ara_last_error.restype = ctypes.c_char_p
    assert b"ara_debug_policy_fc" in lib().ara_last_error()


# ---------------------------------------------------------------------------------------------------------- GPU runs
def check_exact(P, L, prec, W, b, x, n, batch, bn=0, count=None, what="", img=None):
    K = x.shape[1]
    kb, splits = split_formula(L, K)
    img = weight_image(W, L, P, prec) if img is None else img
    part = partials(img, x, k_ranges(K, kb, splits), "cuda")
    got_part, got_prob = run(P, L, prec, W, b, x, n, batch, bn, -1 if count is None else count)
    want = expected_partials(part, n, bn or choose_bn(batch), count)
    d = got_part.view(np.uint32) != want.view(np.uint32)
    assert not d.any(), f"{what} partial sums: {int(d.sum())} of {d.size} differ, first at {np.argwhere(d)[0].tolist()}"
    live = n if count is None else count
    assert (got_prob[live:].view(np.uint32) == SENT).all(), f"{what}: probabilities written beyond the board count"
    logits = logits_in_split_order(b, part, L)[:live]
    p, bound = softmax_bound(logits)
    err = np.abs(got_prob[:live].astype(f64) - p)
    ratio = np.where(err == 0, 0.0, err / bound).max() if live else 0.0
    assert ratio <= 1.0, f"{what} probabilities: error {ratio:.3g}x the bound"
    assert (np.abs(got_prob[:live].astype(f64).sum(-1) - 1) <= bound.sum(-1) + L * 2.0 ** -53).all(), what
    return ratio


@pytest.mark.gpu
@pytest.mark.parametrize("P,L", SHAPES)
def test_exact_bit_for_bit(P, L):
    """Every batch of BATCHES at the network's N tile, batch 66 at every N tile, and device-side counts ending inside a
    tile and on a tile boundary: partial sums bit for bit (skipped tiles untouched), probabilities within the bound
    (rows beyond the count untouched)"""
    worst = 0.0
    for prec in (0, 1):
        for kind in KINDS[prec]:
            img = cached_image(P, L, prec, kind)
            for batch in BATCHES if prec == 0 else (1, 32, 65, 128):
                W, b, x, _ = exact_operands(P, L, prec, kind, batch)
                worst = max(worst, check_exact(P, L, prec, W, b, x, batch, batch, what=f"{kind} B={batch}", img=img))
            W, b, x, _ = exact_operands(P, L, prec, kind, 66)
            for bn in BNS:
                check_exact(P, L, prec, W, b, x, 66, 66, bn, what=f"{kind} B=66 bn={bn}", img=img)
            for count in (40, 64):
                check_exact(P, L, prec, W, b, x, 66, 66, 32, count, what=f"{kind} B=66 bn=32 count={count}", img=img)
    print(f"policy fc P={P} L={L}: largest probability error / bound {worst:.3g}")


@pytest.mark.gpu
def test_split_order_bit_for_bit():
    P, L, W, b, x = split_order_operands(5)
    part, prob = run(P, L, 0, W, b, x, 5, 5)
    check_exact(P, L, 0, W, b, x, 5, 5, what="split order")
    p, _ = softmax_bound(logits_in_split_order(b, partials(weight_image(W, L, P, 0), x, k_ranges(x.shape[1], *split_formula(
        L, x.shape[1]))), L))
    assert p[0, 5] > p[0, 0] * 50 and prob[0, 5] > prob[0, 0] * 50  # logit 4, not 3


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["onehot", "equal", "apart80"])
def test_probabilities_within_bound(case):
    """one-hot, all-equal, and logits 80 and 160 apart (exp underflows to 0): the float64 softmax within the bound"""
    P, L = 76, 1968
    rng = _rng("prob", case)
    for prec in (0, 1):
        W, b, x, _ = exact_operands(P, L, prec, KINDS[prec][0], 7)
        if case == "onehot":
            x[:] = 0
            b = np.zeros(L, f32)
            b[123] = 100.0
        elif case == "equal":
            x[:] = 0
            b = np.full(L, 0.75, f32)
        else:
            b = rng.choice([0.0, -80.0, -160.0], L).astype(f32)
        check_exact(P, L, prec, W, b, x, 7, 7, what=f"{case} prec {prec}")


@pytest.mark.gpu
@pytest.mark.parametrize("prec", [0, 1])
def test_float64_within_bound(prec):
    """random fp16 (float32: fp32 split into hi + lo) operands against float64: K blocks of 64 in 16-wide wgmma steps,
    u_acc = 2^-23 per step (tests/test_conv_gemm_gpu.py), the split partial sums added in fp32 in split order"""
    worst = 0.0
    for P, L in [(76, 1968), (81, 2272), (256, 2316)]:
        rng = _rng("float64", P, L, prec)
        B = 65
        cap = rows_cap(B)
        W = (rng.standard_normal((L, P * 64)) * 0.05).astype(f32)
        sc = square_cols(P, prec)
        xv = np.maximum(rng.standard_normal((cap, 64, P)), 0).astype(f32)
        x = np.zeros((cap, 64, sc), f16)
        if prec == 0:
            x[:, :, :P] = xv
        else:
            cs = sc // 3
            hi = xv.astype(f16)
            x[:, :, :P] = hi
            x[:, :, cs:cs + P] = hi
            x[:, :, 2 * cs:2 * cs + P] = (xv - hi.astype(f32)).astype(f16)
        x = x.reshape(cap, -1)
        b = (rng.standard_normal(L) * 0.1).astype(f32)
        K = x.shape[1]
        kb, splits = split_formula(L, K)
        img = weight_image(W, L, P, prec)
        got_part, got_prob = run(P, L, prec, W, b, x, B, B)
        X = torch.from_numpy(x.astype(f64)).cuda()
        I = torch.from_numpy(img.astype(f64)).cuda()
        for s, (k0, k1) in enumerate(k_ranges(K, kb, splits)):
            P_ = torch.zeros(cap, I.shape[0], dtype=torch.float64, device="cuda")
            E = torch.zeros_like(P_)
            for k in range(k0, k1, 16):
                g = X[:, k:k + 16] @ I[:, k:k + 16].T
                E += 2.0 ** -23 * (P_.abs() + X[:, k:k + 16].abs() @ I[:, k:k + 16].abs().T)
                P_ += g
            err = (torch.from_numpy(got_part[s].astype(f64)).cuda() - P_).abs()
            ratio = torch.where(err == 0, 0.0, err / E).max().item()
            assert ratio <= 1.0, f"P={P} L={L} prec {prec} split {s}: error {ratio:.3g}x the bound"
            worst = max(worst, ratio)
    print(f"policy fc float64 precision {prec}: largest partial-sum error / bound {worst:.3g}")
