"""The wgmma convolution GEMM (conv_gemm_kernel<BN>, conv_gemm.cuh) one launch at a time, through ara_debug_conv, at
every layer the network builds (Net::build_conv): ROWS has one row per call site and width.

Two kinds of operands:
  exact    small integers on a power-of-two grid, drawn per (board, square, channel) and per weight, bias and residual
           value.  Every product and every partial sum, in any order, is a multiple of the grid unit below 2^24 units
           (test_exact_operands_sum_exactly), so the fp32 accumulator holds the exact sum whatever order the kernel adds
           in, and the fp16, fp32 and split outputs have the model's bits: hi = fp16_rn(v), lo = fp16_rn(v - hi), the ReLU
           before the residual.  Float32 rows run twice, once with fp16-exact weights (w_lo = 0) and once with fp16-exact
           activations (a_lo = 0): the dropped a_lo * w_lo term is then zero and the three kept terms are exercised.
           Every output buffer is compared whole: what the kernel must not write (columns from n_end, split columns from
           split_cs, the phantom board of an odd batch, boards beyond the device-side count) holds a NaN pattern that has
           to survive.  NaN also fills the activation channels from cin up to the pitch (read as zero by TMA) and the
           phantom board's input.
  float64  random fp16 operands (float32 rows: fp32 activations and weights split into hi + lo) against a float64
           convolution of the operands as the kernel sees them, within error_bound.
test_each_mutation_changes_the_output shows that plausible mistakes in the kernel change the exact rows' bits, and
test_bound_catches_precision_bugs that the float64 bound would catch an fp16 accumulator or a dropped a_hi * w_lo term.
"""
import ctypes
import math
import zlib
from collections import namedtuple

import numpy as np
import pytest
import torch

f16, f32, f64 = np.float16, np.float32, np.float64
BOARDS = (1, 2, 3, 7, 64, 133)  # 133: one board more than an H100 SXM has SMs (132)
FORCED_BN_BOARDS = (3, 64)      # the batches that also run at every N tile
FLOAT64_BOARDS = (3, 64)
BNS = (64, 128, 256)
SENT_H, SENT_F = 0x7E5A, 0x7FC5A5A5  # NaN patterns in the output buffers the kernel must leave alone
U_ACC = 2.0 ** -23


class DebugConv(ctypes.Structure):
    """ara_debug_conv_t (include/ara_b200.h)"""
    _fields_ = [("act", ctypes.c_void_p), ("w", ctypes.c_void_p), ("bias", ctypes.c_void_p), ("res_h", ctypes.c_void_p),
                ("res_f", ctypes.c_void_p), ("out_h", ctypes.c_void_p), ("out_f", ctypes.c_void_p), ("out_s", ctypes.c_void_p),
                ("boards_dev", ctypes.c_void_p)] + [(n, ctypes.c_int) for n in (
                    "precision", "boards_cap", "boards", "cin", "n_out", "ksize", "relu", "w_rows", "act_cin", "act_pitch", "ldr",
                    "ldo", "n_end", "split_cs", "bn")]


def ceil_to(v, m):
    return (v + m - 1) // m * m


# ------------------------------------------------------------------------------------------------------------ the rows
# prec 0 float16, 1 float32 (split operands); res: None, "h" (fp16) or "f" (fp32); inplace: the residual is the fp16 output
# buffer itself (res_h == out_h); outs: which of out_h, out_f, out_s the layer writes; act_off / out_off: the activation /
# output pointer is this many channels into a wider row (an NTB's y1 | z2 rows); cnt: the call site passes the device-side
# board count
Row = namedtuple("Row", "name prec cin n_out ksize relu bias res inplace outs act_cin act_pitch act_off ldr ldo out_off n_end "
                        "split_cs cnt")


def R(name, prec, cin, n_out, ksize, relu, bias=True, res=None, inplace=False, outs="h", act_cin=0, act_pitch=0, act_off=0,
      ldr=0, ldo=0, out_off=0, n_end=0, split_cs=0, cnt=True):
    return Row(f"{'f32' if prec else 'f16'}/{name}", prec, cin, n_out, ksize, int(relu), bias, res, inplace, outs, act_cin,
               act_pitch, act_off, ldr, ldo, out_off, n_end, split_cs, cnt)


def site_rows(prec, in_ch, stem_relu, pol, pol_bias, c_ops, ntbs):
    """The build_conv call sites of one network (net.cu) in precision prec: the trunk is 256 channels on the device"""
    rows = []
    if prec == 0:
        # build_half: stem, reading the input planes padded to a multiple of 64 (cin_pad)
        rows.append(R(f"stem[{in_ch},relu{stem_relu}]", 0, in_ch, 256, 3, stem_relu, act_cin=ceil_to(in_ch, 64), ldo=256))
        # build_half: policy conv1 (3x3 + ReLU into d_p1) and conv2 (3x3 into the fp32 logits, ldp = ceil32)
        rows.append(R("pol1", 0, 256, 256, 3, 1, ldo=256))
        rows.append(R(f"pol2[{pol},bias{int(pol_bias)}]", 0, 256, pol, 3, 0, bias=pol_bias, outs="f", ldo=ceil_to(pol, 32)))
        for M, Ca, H in ntbs:  # build_ntb_half: d_nt rows are y1 (M) | z2 (Ca) | 0, 256 wide
            rows += [
                R(f"pe[{M}]", 0, 256, M, 1, 0, ldo=256, n_end=M),                                  # x -> y1 of d_nt
                R(f"qkv[{M}]", 0, M, 3 * M, 1, 0, act_pitch=256, ldo=3 * M),                      # y1 -> d_qkv
                R(f"proj[{M}]", 0, M, M, 1, 0, res="h", inplace=True, ldr=256, ldo=256, n_end=M),  # d_att (+ y1) -> y1
                R(f"prj[{M},{Ca}]", 0, M, Ca, 1, 0, act_pitch=256, ldo=256, out_off=M, n_end=Ca),  # y1 -> z
                R(f"gc[{M},{Ca}]", 0, Ca, Ca, 3, 1, act_pitch=256, act_off=M, ldo=Ca),            # z -> d_g
                R(f"mh[{M},{Ca}]", 0, Ca, Ca, 1, 0, bias=False, res="h", inplace=True, ldr=256, ldo=256, out_off=M,
                  n_end=Ca),                                                                       # d_g (+ z) -> z
                R(f"mlp1[{H}]", 0, 256, H, 1, 1, ldo=H),                                          # d_nt -> d_hid
                R(f"mlp2[{H}]", 0, H, 256, 1, 0, res="h", ldr=256, ldo=256),                      # d_hid (+ d_nt) -> x
            ]
        return rows
    # build_precise: stem into fp32 + split trunk
    rows.append(R(f"stem[{in_ch},relu{stem_relu}]", 1, in_ch, 256, 3, stem_relu, outs="fs", ldo=256, split_cs=256))
    for c in c_ops:
        rows.append(R(f"conv1[{c}]", 1, 256, c, 1, 1, outs="f", ldo=c, cnt=False))  # split X -> fp32 H1
        rows.append(R(f"conv2[{c}]", 1, c, 256, 1, 0, res="f", ldr=256, outs="fs", ldo=256, split_cs=256, cnt=False))
    rows.append(R("pol1", 1, 256, 256, 3, 1, outs="s", ldo=256, split_cs=256))  # split X -> split d_p1
    rows.append(R(f"pol2[{pol},bias{int(pol_bias)}]", 1, 256, pol, 3, 0, bias=pol_bias, outs="f", ldo=ceil_to(pol, 32)))
    for M, Ca, H in ntbs:  # build_ntb_precise
        ms = ceil_to(M, 64)
        rows += [
            R(f"pe[{M}]", 1, 256, M, 1, 0, outs="fs", ldo=M, split_cs=ms),                        # -> d_yf, d_ys
            R(f"qkv[{M}]", 1, M, 3 * M, 1, 0, outs="f", ldo=3 * M),                              # d_ys -> d_qkvf
            R(f"proj[{M}]", 1, M, M, 1, 0, res="f", ldr=M, outs="fs", ldo=256, n_end=M, split_cs=ms),  # -> d_x2f, d_ys
            R(f"prj[{M},{Ca}]", 1, M, Ca, 1, 0, outs="fs", ldo=Ca, split_cs=64),                  # d_ys -> d_zf, d_zs
            R(f"gc[{Ca}]", 1, Ca, Ca, 3, 1, outs="s", ldo=Ca, split_cs=64),                       # d_zs -> d_gs
            R(f"mh[{M},{Ca}]", 1, Ca, Ca, 1, 0, bias=False, res="f", ldr=Ca, outs="f", ldo=256, out_off=M,
              n_end=Ca),                                                                           # d_gs (+ d_zf) -> d_x2f + M
            R(f"mlp1[{H}]", 1, 256, H, 1, 1, outs="s", ldo=H, split_cs=H),                        # d_x2s -> d_hs
            R(f"mlp2[{H}]", 1, H, 256, 1, 0, res="f", ldr=256, outs="fs", ldo=256, split_cs=256),  # d_hs (+ d_x2f) -> x
        ]
    return rows


# The networks of the suite: (input planes, stem ReLU, policy planes, last policy conv with bias, c_op of the float32
# bottleneck blocks, NTB widths (M, Ca, H)).  RISEv2 / v3.3 (oracle/net.py: 34 / 52 planes, 81 / 76 policy planes, c_op
# 128 .. 896 / 224 .. 672), AlphaVile tiny / normal (oracle/net_alphavile.py: NTB 160 | 32, 384 and 160 | 64, 448; c_op 384 /
# 256 and 448 / 320) and the extremes of tests/test_net_geometry_gpu.py (narrow64: NTB 32 | 32, 64, c_op 32; full256_ntb:
# 224 | 32, 1024; mid160: 96 | 64, 320, c_op 1024; heads_max / heads_min: 256 / 1 planes).  The trunk is padded to 256
# channels on the device, so the trunk widths 64 / 160 / 192 / 224 / 256 reach the GEMMs only through M, Ca, H and c_op;
# value_fc belongs to the value head, which is not a GEMM.
NETWORKS = [
    (34, 1, 81, False, (128, 896), ()),                    # RISEv2
    (52, 0, 76, True, (224, 672), ()),                     # RISEv3.3 (MXNet export: no stem ReLU, policy bias)
    (52, 1, 76, True, (384, 256), ((160, 32, 384),)),      # AlphaVile tiny
    (52, 1, 76, True, (448, 320), ((160, 64, 448),)),      # AlphaVile normal
    (34, 1, 81, False, (32,), ((32, 32, 64),)),            # narrow64
    (52, 1, 76, True, (512,), ((224, 32, 1024),)),         # full256_ntb
    (52, 1, 76, True, (1024,), ((96, 64, 320),)),          # mid160
    (256, 1, 256, False, (), ()),                          # heads_max
    (1, 1, 1, False, (32,), ()),                           # heads_min
]


def _rows():
    rows = {}
    for prec in (0, 1):
        for net in NETWORKS:
            for r in site_rows(prec, *net):
                rows.setdefault(r.name, r)  # a layer of the same shape in two networks is one row
    # not a call site: the epilogue writes all three outputs when it is given all three
    rows["f32/all-outputs"] = R("all-outputs", 1, 96, 160, 3, 1, res="f", ldr=160, outs="hfs", ldo=160, split_cs=192)
    return list(rows.values())


ROWS = _rows()
IDS = [r.name for r in ROWS]
ROW = {r.name: r for r in ROWS}


# ------------------------------------------------------------------------------------------------------------- layout
def parts(row):
    return 3 if row.prec else 1


def cw(row):
    return ceil_to(row.cin, 64)


def view_cin(row):
    """channels of an activation row the kernel maps (conv_layer_build's act_cin)"""
    return 3 * cw(row) if row.prec else (row.act_cin or row.cin)


def pitch(row):
    return row.act_pitch or view_cin(row)


def w_rows(row):
    return ceil_to(row.n_out, 256)  # Net::build_conv


def weight_image(w, row):
    """Net::upload_conv_w: w [n_out][cin][k][k] fp32 -> fp16 [ceil256(n_out)][k*k][parts * ceil64(cin)], per tap w [cw]
    (float16) or hi(w) [cw] | lo(w) [cw] | hi(w) [cw] (float32), zero padded"""
    taps, c = row.ksize ** 2, cw(row)
    img = np.zeros((w_rows(row), taps, parts(row) * c), f16)
    wt = w.reshape(row.n_out, row.cin, taps).transpose(0, 2, 1).astype(f32)
    hi = wt.astype(f16)
    img[:row.n_out, :, :row.cin] = hi
    if row.prec:
        img[:row.n_out, :, c:c + row.cin] = (wt - hi.astype(f32)).astype(f16)
        img[:row.n_out, :, 2 * c:2 * c + row.cin] = hi
    return img


def boards_cap(B):
    return max(2, B + (B & 1))


def n_written(row, bn, ignore_n_end=False):
    """columns the kernel writes: every N tile up to n_end (0: ldo)"""
    tiles = -(-row.n_out // bn) * bn
    end = row.ldo - row.out_off if ignore_n_end else (row.n_end or row.ldo)
    return min(end, tiles)


# ----------------------------------------------------------------------------------------------------------- operands
Ops = namedtuple("Ops", "act img bias res kind unit amax")


def _rng(*key):
    return np.random.default_rng(zlib.crc32(repr(key).encode()))


def exact_kinds(row):
    return ("w_exact", "a_exact") if row.prec else ("fp16",)


def grid_range(row):
    """largest |integer| of the activations and weights: the exactness bound (kin R^2 / 2 products of the largest unit)
    stays near 2^22 units; float32 rows' hi products are 2^12 units (their lo parts are 2^-12 of the hi unit)"""
    kin = row.cin * row.ksize ** 2
    if row.prec:
        return int(min(127, max(1, math.isqrt(2 ** 11 // kin))))
    return int(min(127, max(3, math.isqrt(2 ** 23 // kin))))


def _act_buffer(row, B, view):
    """view [boards][64][view_cin] -> the fp16 activation buffer [boards_cap][64][pitch] (+ act_off in front): NaN outside
    the mapped channels and in the phantom board"""
    cap, P = boards_cap(B), pitch(row)
    buf = np.full(row.act_off + cap * 64 * P, f16(np.nan), f16)
    rows = buf[row.act_off:].reshape(cap, 64, P)
    rows[:B, :, :view.shape[2]] = view[:B]
    return buf


def exact_operands(row, B, kind):
    """Integers on a power-of-two grid -> Ops.  Float16: a = i 2^-4, w = i 2^-5, grid unit u = 2^-9.  Float32: a_hi = i,
    a_lo = +-2^-12 where a_hi != 0 (w_exact), w_hi = i 2^-2, w_lo = +-2^-14 where w_hi != 0 (a_exact), u = 2^-14 (lo parts
    stay fp16 normals).  Bias and residual are multiples of u; the fp16 residual has 10 significant bits.  The weights and
    the bias are the same at every batch; amax holds the largest |activation| per channel of the view the draws allow."""
    Rg = grid_range(row)
    c, cap = cw(row), boards_cap(B)
    rw, ra = _rng("exact weights", row.name, kind), _rng("exact", row.name, B, kind)
    ints = lambda rng, r, shape: rng.integers(-r, r + 1, shape)  # noqa: E731
    iw = ints(rw, Rg, (row.n_out, row.cin, row.ksize, row.ksize))
    if not row.prec:
        unit = 2.0 ** -9
        w = (iw * 2.0 ** -5).astype(f32)
        bias = (ints(rw, 2 ** 16, row.n_out) * unit).astype(f32)
        view = (ints(ra, Rg, (cap, 64, view_cin(row))) * 2.0 ** -4).astype(f16)
        amax = np.full(view_cin(row), Rg * 2.0 ** -4)
    else:
        unit = 2.0 ** -14
        w = (iw * 2.0 ** -2 + (ints(rw, 1, iw.shape) * (iw != 0) * 2.0 ** -14 if kind == "a_exact" else 0.0)).astype(f32)
        bias = (ints(rw, 2 ** 20, row.n_out) * unit).astype(f32)
        hi = ints(ra, Rg, (cap, 64, c)).astype(f64)
        lo = ints(ra, 1, hi.shape) * (hi != 0) * 2.0 ** -12 if kind == "w_exact" else np.zeros_like(hi)
        view = np.concatenate([hi, hi, lo], axis=2).astype(f16)
        amax = np.concatenate([np.full(2 * c, float(Rg)), np.full(c, 2.0 ** -12 if kind == "w_exact" else 0.0)])
    res = None
    if row.res == "h":
        res = (ints(ra, 1023, (cap * 64, row.ldr)) * np.exp2(ra.integers(0, 9, (cap * 64, row.ldr))) * unit).astype(f16)
    elif row.res == "f":
        res = (ints(ra, 2 ** 20, (cap * 64, row.ldr)) * unit).astype(f32)
    return Ops(_act_buffer(row, B, view), weight_image(w, row), bias if row.bias else None, res, kind, unit, amax)


def residual_max(row, ops):
    """the largest |residual| the draws of exact_operands allow"""
    return {None: 0.0, "h": 1023 * 2.0 ** 8, "f": 2.0 ** 20}[row.res] * ops.unit


def float64_operands(row, B):
    rng = _rng("float64", row.name, B)
    taps, c, cap = row.ksize ** 2, cw(row), boards_cap(B)
    kin = row.cin * taps
    w = (rng.normal(0.0, 1.0, (row.n_out, row.cin, row.ksize, row.ksize)) / np.sqrt(kin)).astype(f32)
    if row.prec:
        a = rng.normal(0.0, 1.0, (cap, 64, c)).astype(f32)
        hi = a.astype(f16)
        view = np.concatenate([hi, hi, (a - hi.astype(f32)).astype(f16)], axis=2)
    else:
        view = rng.normal(0.0, 1.0, (cap, 64, view_cin(row))).astype(f16)
    bias = rng.normal(0.0, 0.1, row.n_out).astype(f32)
    res = None
    if row.res:
        res = rng.normal(0.0, 0.5, (cap * 64, row.ldr)).astype(f16 if row.res == "h" else f32)
    return Ops(_act_buffer(row, B, view), weight_image(w, row), bias if row.bias else None, res, "float64", None, None)


# -------------------------------------------------------------------------------------------------------------- model
def kernel_view(row, ops, B, mut=()):
    """the A operand as the TMA map reads it: [boards_cap][64][ceil64(view_cin)] float64, channels from view_cin zero"""
    cap, vc = boards_cap(B), view_cin(row)
    P = vc if "pitch_as_cin" in mut else pitch(row)
    flat = ops.act[row.act_off:row.act_off + cap * 64 * P].astype(f64)
    v = np.zeros((cap, 64, ceil_to(vc, 64)))
    v[:, :, :vc] = flat.reshape(cap, 64, P)[:, :, :vc]
    return v


def _shifted(x, ksize, mut):
    """x [boards][8][8][K] -> per tap (dy, dx) of the kernel's order the board shifted by it, outside the board zero"""
    r = ksize // 2
    if "halo_clamp" in mut:
        xp = torch.nn.functional.pad(x.permute(0, 3, 1, 2), (r, r, r, r), mode="replicate").permute(0, 2, 3, 1)
    else:
        xp = torch.nn.functional.pad(x, (0, 0, r, r, r, r))
    for t in range(ksize * ksize):
        dy, dx = t // ksize, t % ksize
        if "dxdy" in mut:
            dy, dx = dx, dy
        yield t, xp[:, dy:dy + 8, dx:dx + 8, :].reshape(-1, x.shape[3])


def gemm(row, ops, B, device, mut=()):
    """sum over taps and channels of view x image in float64 (exact for the exact operands): [boards_cap * 64][ldo]"""
    x = torch.from_numpy(kernel_view(row, ops, B, mut)).to(device).reshape(boards_cap(B), 8, 8, -1)
    img = torch.from_numpy(ops.img.astype(f64)).to(device)
    acc = torch.zeros(x.shape[0] * 64, img.shape[0], dtype=torch.float64, device=device)
    for t, a in _shifted(x, row.ksize, mut):
        acc += a @ img[:, t, :].T
    return acc[:, :row.ldo].cpu().numpy()


def _padded(v, n):
    out = np.zeros(n, f32)
    if v is not None:
        out[:min(n, len(v))] = v[:n]
    return out


def residual_as_read(row, ops, init, m, nw):
    """the residual the epilogue adds at rows 0 .. m, columns 0 .. nw: res[r * ldr + n] of its buffer (the fp16 output
    buffer before the launch when it is read in place), zero past the buffer's end"""
    if ops.res is None:
        return np.zeros((m, nw), f32)
    flat = init["h"].view(f16)[row.out_off:] if row.inplace else ops.res.ravel()
    idx = np.arange(m)[:, None] * row.ldr + np.arange(nw)[None, :]
    return np.where(idx < flat.size, flat[np.minimum(idx, flat.size - 1)], 0).astype(f32)


def epilogue(row, acc, bias, r, bn, mut=()):
    """acc [m][nw] exact sums -> v [m][nw] fp32: bias, ReLU, residual r in the kernel's order"""
    nw = acc.shape[1]
    b = _padded(bias, w_rows(row) + 256)
    b = b[bn:bn + nw] if "bias_tile" in mut else b[:nw]
    v = acc.astype(f32) + b
    if row.relu and "res_before_relu" in mut:
        return np.maximum(v + r, f32(0))
    if row.relu:
        v = np.maximum(v, f32(0))
    return (v + r).astype(f32)


def initial_buffers(row, B, ops):
    """the output buffers before the launch, by name: NaN patterns, and the residual where it is read in place.  One row
    more than the batch has: a write past the last row lands in it."""
    rows = boards_cap(B) * 64 + 1
    bufs = {}
    if "h" in row.outs:
        bufs["h"] = np.full(rows * row.ldo, SENT_H, np.uint16)
        if row.inplace:
            b = bufs["h"].reshape(rows, row.ldo)
            b[:rows - 1, row.out_off:row.out_off + (row.n_end or row.ldo)] = ops.res[:, :(row.n_end or row.ldo)].view(np.uint16)
    if "f" in row.outs:
        bufs["f"] = np.full(rows * row.ldo, SENT_F, np.uint32)
    if "s" in row.outs:
        bufs["s"] = np.full(rows * 3 * row.split_cs, SENT_H, np.uint16)
    return bufs


def written_boards(B, cnt, mut=()):
    if cnt is None:
        return B + 1 if ("phantom" in mut and B & 1) else B
    tiles = -(-cnt // 2) + (1 if "boards_dev" in mut else 0)
    return min(B, 2 * tiles)


def expected_buffers(row, B, ops, acc, bn, cnt=None, mut=()):
    """the output buffers after the launch: v = epilogue(acc) in the rows and columns the kernel writes"""
    bufs = initial_buffers(row, B, ops)
    nb, nw = written_boards(B, cnt, mut), n_written(row, bn, "n_end" in mut)
    m = nb * 64
    v = epilogue(row, acc[:m, :nw], ops.bias, residual_as_read(row, ops, bufs, m, nw), bn, mut)
    if "h" in bufs:
        bufs["h"].reshape(-1, row.ldo)[:m, row.out_off:row.out_off + nw] = v.astype(f16).view(np.uint16)
    if "f" in bufs:
        bufs["f"].reshape(-1, row.ldo)[:m, row.out_off:row.out_off + nw] = v.view(np.uint32)
    if "s" in bufs:
        ns = min(nw, row.split_cs)
        hi = v[:, :ns].astype(f16)
        lo = np.zeros_like(hi) if "split_lo" in mut else (v[:, :ns] - hi.astype(f32)).astype(f16)
        s = bufs["s"].reshape(-1, 3, row.split_cs)
        s[:m, 0, :ns] = hi.view(np.uint16)
        s[:m, 1, :ns] = hi.view(np.uint16)
        s[:m, 2, :ns] = lo.view(np.uint16)
    return bufs


# --------------------------------------------------------------------------------------------- exactness precondition
def exactness_bound(row, ops):
    """per output column, in grid units: the largest |activation| of each channel times |weight|, summed over taps and
    channels, plus the largest |bias| and |residual|.  Every product, every partial sum in any order, and the value after
    the bias and the residual are at most this."""
    w = np.abs(ops.img.astype(f64))  # [w_rows][taps][K]
    amax = np.zeros(w.shape[2])
    amax[:len(ops.amax)] = ops.amax
    s = (w * amax).sum(axis=(1, 2))
    s += 0.0 if ops.bias is None else np.abs(ops.bias.astype(f64)).max()
    s += residual_max(row, ops)
    return s / ops.unit


def test_every_call_site_has_rows():
    sites = {"stem", "pol1", "pol2", "pe", "qkv", "proj", "prj", "gc", "mh", "mlp1", "mlp2"}
    names = {(r.prec, r.name.split("/")[1].split("[")[0]) for r in ROWS}
    assert {(0, s) for s in sites} <= names and {(1, s) for s in sites | {"conv1", "conv2"}} <= names
    assert len(sites) + len(sites | {"conv1", "conv2"}) == 24  # the build_conv calls of net.cu
    shapes = {(r.cin, r.n_out, r.ksize) for r in ROWS}
    assert {(1, 256, 3), (256, 256, 3), (256, 1, 3), (256, 76, 3), (256, 81, 3), (224, 672, 1), (256, 1024, 1),
            (1024, 256, 1), (32, 32, 3), (256, 32, 1)} <= shapes
    assert any(r.act_pitch > view_cin(r) and view_cin(r) % 64 for r in ROWS)  # TMA zero-fills a partial chunk
    assert any(r.inplace for r in ROWS) and any(r.n_end and r.n_end < r.ldo for r in ROWS)


@pytest.mark.parametrize("kind", ["fp16", "w_exact", "a_exact"])
def test_exact_operands_sum_exactly(kind):
    """The exact rows' precondition at every batch the GPU test runs: each output's sum of |products| plus |bias| and
    |residual| is below 2^24 grid units (K = 9 * 256 and the 3 * 1024-wide split rows included), so fp32 holds every
    partial sum; fp16 outputs stay below 2^15; and the outputs have more bits than fp16 keeps, so hi and lo both matter."""
    for row in ROWS:
        if kind not in exact_kinds(row):
            continue
        ops = exact_operands(row, 3, kind)  # the weights and bias of every batch, activations within amax
        s = exactness_bound(row, ops)
        assert s.max() < 2 ** 24, (row.name, s.max())
        if "h" in row.outs or "s" in row.outs:
            assert s.max() * ops.unit < 2 ** 15, row.name
        view = kernel_view(row, ops, 3)[:3, :, :len(ops.amax)]
        assert (np.abs(view) <= ops.amax).all() and (ops.res is None or np.abs(ops.res).max() <= residual_max(row, ops))
        acc = gemm(row, ops, 3, "cpu")[:3 * 64, :row.n_out]
        v = epilogue(row, acc, ops.bias, residual_as_read(row, ops, initial_buffers(row, 3, ops), 3 * 64, row.n_out), 64)
        assert (v.astype(f16).astype(f32) != v).mean() > 0.2, row.name  # the rounding to fp16 is exercised


MUTATIONS = ["dxdy", "halo_clamp", "res_before_relu", "bias_tile", "n_end", "pitch_as_cin", "split_lo", "boards_dev", "phantom"]


@pytest.mark.parametrize("mut", MUTATIONS)
def test_each_mutation_changes_the_output(mut):
    """On the GPU test's own operands, each plausible mistake changes at least one bit of the exact rows' buffers"""
    from crazyara_b200 import lib
    for row in ROWS:
        for kind in exact_kinds(row):
            B = 7
            ops = exact_operands(row, B, kind)
            bn = lib().ara_debug_choose_bn(B, row.n_out)
            acc = gemm(row, ops, B, "cpu")
            cnt = 3 if mut == "boards_dev" and row.cnt else None
            want = expected_buffers(row, B, ops, acc, bn, cnt)
            bad_acc = gemm(row, ops, B, "cpu", (mut,)) if mut in ("dxdy", "halo_clamp", "pitch_as_cin") else acc
            got = expected_buffers(row, B, ops, bad_acc, bn, cnt, (mut,))
            if any((got[k] != want[k]).any() for k in want):
                return
    pytest.fail(f"no exact row sees {mut}")


# ------------------------------------------------------------------------------------------------------ float64 bound
def error_bound(row, ops, B, device):
    """(float64 reference, per-output bound) for the float64 operands, [boards_cap * 64][w_rows] each.

    The reference is the convolution of the operands the kernel is given, in float64: activations (a_hi + a_lo) times
    weights (w_hi + w_lo), plus the bias, ReLU, plus the residual.  Float32 rows keep only three of the four products:
    the bound adds the dropped sum |a_lo w_lo|.  The kernel accumulates in fp32 on wgmma, 16 products (one k-step) at a
    time; the rounding of that accumulation is not documented.  Assumption: each k-step j adds its products to the
    accumulator with an error of at most u_acc (|P_(j-1)| + S_j), u_acc = 2^-23 (one fp32 ulp: covers truncation),
    P_(j-1) the exact sum before the step and S_j the step's sum of |products|; the steps go tap by tap, 16 channels of
    the operand image at a time.  Then
      accumulation   E = u_acc sum_j (|P_(j-1)| + S_j)  (+ sum |a_lo w_lo| in float32)
      epilogue       + 2^-24 (|acc + bias| + |out|) + E: the two fp32 adds, ReLU with slope 1
      output         fp16: + half an fp16 ulp of |out|; split hi + lo: + 2^-22 |out| + 2^-24; fp32: nothing"""
    cap = boards_cap(B)
    x = torch.from_numpy(kernel_view(row, ops, B)).to(device).reshape(cap, 8, 8, -1)
    img = torch.from_numpy(ops.img.astype(f64)).to(device)
    c = cw(row)
    P = torch.zeros(cap * 64, img.shape[0], dtype=torch.float64, device=device)
    E = torch.zeros_like(P)
    full = torch.zeros_like(P)
    steps16 = []
    for t, a in _shifted(x, row.ksize, ()):
        w = img[:, t, :]
        for k in range(0, a.shape[1], 16):
            g = a[:, k:k + 16] @ w[:, k:k + 16].T
            S = a[:, k:k + 16].abs() @ w[:, k:k + 16].abs().T
            E += U_ACC * (P.abs() + S)
            P += g
            steps16.append((t, k, g))
        if row.prec:  # the dropped a_lo w_lo and the full product
            a_lo, w_lo = a[:, 2 * c:], w[:, c:2 * c]
            full += a_lo @ w_lo.T
            E += a_lo.abs() @ w_lo.abs().T
    full += P
    b = torch.from_numpy(_padded(ops.bias, img.shape[0]).astype(f64)).to(device)
    r = torch.zeros_like(P)
    if ops.res is not None:
        k = min(row.ldr, r.shape[1])
        r[:, :k] = torch.from_numpy(ops.res.astype(f64)[:, :k]).to(device)
    pre = full + b
    out = (pre.clamp(min=0) if row.relu else pre) + r
    E = E + 2.0 ** -24 * (pre.abs() + E) + 2.0 ** -24 * (out.abs() + E)
    return out, E, steps16, b, r


def _ratio(err, bound):
    """the largest err / bound, 0 / 0 counted as 0 (columns of zero weights, bias and residual)"""
    return torch.where(err == 0, 0.0, err / bound).max().item()


def output_bound(E, out, which):
    if which == "h":
        return E + 2.0 ** -11 * (out.abs() + E) + 2.0 ** -25
    if which == "s":
        return E + 2.0 ** -22 * (out.abs() + E) + 2.0 ** -24
    return E


def _fp16_accumulation(row, steps16, b, r, rows):
    acc = torch.zeros(rows, b.shape[0], dtype=torch.float64, device=b.device)
    for _, _, g in steps16:
        acc = (acc + g).half().double()
    pre = acc + b
    return (pre.clamp(min=0) if row.relu else pre) + r


def _drop_hi_lo(row, steps16, b, r, rows):
    c = cw(row)
    acc = torch.zeros(rows, b.shape[0], dtype=torch.float64, device=b.device)
    for _, k, g in steps16:
        if not c <= k < 2 * c:
            acc += g
    pre = acc + b
    return (pre.clamp(min=0) if row.relu else pre) + r


@pytest.mark.parametrize("name", IDS)
def test_bound_catches_precision_bugs(name):
    """The float64 bound is at least 10x below the error of the same arithmetic with an fp16 accumulator (and, for
    float32 rows, with the a_hi w_lo products dropped) at some output of every row: the GPU test would catch either."""
    row = ROW[name]
    B = 3
    ops = float64_operands(row, B)
    out, E, steps16, b, r = error_bound(row, ops, B, "cpu")
    m, nw = B * 64, n_written(row, 64)
    outs = row.outs.replace("f", "") or "f"
    bound = output_bound(E, out, "h" if "h" in outs else outs[0])[:m, :nw]
    ref = out[:m, :nw]
    bugs = [("fp16 accumulator", _fp16_accumulation)] + ([("a_hi w_lo dropped", _drop_hi_lo)] if row.prec else [])
    for what, model in bugs:
        got = model(row, steps16, b, r, out.shape[0])[:m, :nw]
        ratio = _ratio((got - ref).abs(), bound)
        assert ratio >= 10.0, f"{name}: {what} exceeds the bound by only {ratio:.2f}x"


# ---------------------------------------------------------------------------------------------------------- GPU runs
def _dev(a):
    return None if a is None else torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _ptr(t):
    return None if t is None else t.data_ptr()


class Launcher:
    """One row's operands on the device; run() launches the layer through ara_debug_conv on fresh output buffers"""

    def __init__(self, row, B, ops):
        self.row, self.B, self.ops = row, B, ops
        self.act, self.img = _dev(ops.act), _dev(ops.img)
        self.bias = _dev(_padded(ops.bias, w_rows(row))) if ops.bias is not None else None
        # a guard row after the residual too: reading it past the columns the layer writes stays inside the buffer
        self.res = None
        if ops.res is not None and not row.inplace:
            self.res = _dev(np.concatenate([ops.res.ravel(), np.zeros(row.ldo, ops.res.dtype)]))

    def run(self, bn, cnt=None):
        from crazyara_b200 import check, lib
        row = self.row
        init = initial_buffers(row, self.B, self.ops)
        bufs = {k: _dev(v) for k, v in init.items()}
        cnt_d = _dev(np.array([cnt if cnt is not None else self.B], np.int32)) if (row.cnt or cnt is not None) else None
        out = {k: None for k in "hfs"}
        for k, t in bufs.items():
            out[k] = t.data_ptr() + (t.element_size() * row.out_off if k != "s" else 0)
        a = DebugConv(act=self.act.data_ptr() + 2 * row.act_off, w=self.img.data_ptr(), bias=_ptr(self.bias),
                      res_h=out["h"] if row.inplace else (_ptr(self.res) if row.res == "h" else None),
                      res_f=_ptr(self.res) if row.res == "f" else None, out_h=out["h"], out_f=out["f"], out_s=out["s"],
                      boards_dev=_ptr(cnt_d), precision=row.prec, boards_cap=boards_cap(self.B), boards=self.B,
                      cin=row.cin, n_out=row.n_out, ksize=row.ksize, relu=row.relu, w_rows=w_rows(row), act_cin=row.act_cin,
                      act_pitch=row.act_pitch, ldr=row.ldr, ldo=row.ldo, n_end=row.n_end, split_cs=row.split_cs, bn=bn)
        f = lib().ara_debug_conv
        f.argtypes = [ctypes.POINTER(DebugConv), ctypes.c_void_p]
        f.restype = ctypes.c_int
        check(f(ctypes.byref(a), None))
        return {k: v.cpu().numpy() for k, v in bufs.items()}


def _bns(row, B):
    from crazyara_b200 import lib
    chosen = lib().ara_debug_choose_bn(B, row.n_out)
    return [chosen] + [bn for bn in BNS if bn != chosen]


@pytest.mark.gpu
@pytest.mark.parametrize("name", IDS)
def test_exact_row_bit_for_bit(name):
    """Every batch of BOARDS at the N tile conv_layer_choose_bn picks (and those of FORCED_BN_BOARDS at each N tile), and
    with a device-side count of half the batch: each output buffer equals the model's, bit for bit, sentinels included"""
    row = ROW[name]
    for B in BOARDS:
        for kind in exact_kinds(row):
            ops = exact_operands(row, B, kind)
            acc = gemm(row, ops, B, "cuda")
            L = Launcher(row, B, ops)
            runs = [(bn, None) for bn in _bns(row, B)[:None if B in FORCED_BN_BOARDS else 1]]
            if row.cnt and B >= 3:
                runs.append((runs[0][0], B // 2))
            for bn, cnt in runs:
                got = L.run(bn, cnt)
                want = expected_buffers(row, B, ops, acc, bn, cnt)
                for k in want:
                    diff = got[k] != want[k]
                    assert not diff.any(), (f"{name} {kind} B={B} bn={bn} count={cnt} out_{k}: {int(diff.sum())} of "
                                            f"{diff.size} differ, first at {np.argwhere(diff)[0].tolist()}")


def check_within_bound(row, B, bn=0):
    """launch with float64 operands -> the largest ratio of |error| to the bound over every output the layer writes"""
    from crazyara_b200 import lib
    ops = float64_operands(row, B)
    out, E, *_ = error_bound(row, ops, B, "cuda")
    bn = bn or lib().ara_debug_choose_bn(B, row.n_out)
    got = Launcher(row, B, ops).run(bn)
    m, nw = B * 64, n_written(row, bn)
    worst = 0.0
    for k, buf in got.items():
        if k == "s":
            s = buf.view(f16).reshape(-1, 3, row.split_cs)[:m].astype(f64)
            ns = min(nw, row.split_cs)
            val, ref, bnd = s[:, 0, :ns] + s[:, 2, :ns], out[:m, :ns], output_bound(E, out, "s")[:m, :ns]
        else:
            v = buf.view(f16 if k == "h" else f32).reshape(-1, row.ldo)[:m, row.out_off:row.out_off + nw].astype(f64)
            val, ref, bnd = v, out[:m, :nw], output_bound(E, out, k)[:m, :nw]
        err = (torch.from_numpy(val).cuda() - ref).abs()
        assert torch.isfinite(err).all(), f"{row.name} B={B} out_{k}: non-finite output"
        ratio = _ratio(err, bnd)
        assert ratio <= 1.0, f"{row.name} B={B} out_{k}: error {ratio:.3g}x the bound at {int((err > bnd).sum())} outputs"
        worst = max(worst, ratio)
    return worst


@pytest.mark.gpu
@pytest.mark.parametrize("name", IDS)
def test_float64_row_within_bound(name):
    worst = max(check_within_bound(ROW[name], B) for B in FLOAT64_BOARDS)
    print(f"{name}: largest error / bound {worst:.3g}")


# assorted fp16 shapes and N tiles outside the case table, against float64 within the derived bound
CASES = [
    # boards, cin, n_out, ksize, relu, res, bn
    (2, 256, 256, 1, True, False, 64),
    (2, 64, 256, 3, True, False, 64),
    (8, 256, 128, 1, True, False, 128),
    (8, 256, 896, 1, True, False, 128),
    (8, 896, 256, 1, False, True, 64),
    (64, 256, 256, 3, True, False, 128),
    (64, 256, 256, 3, True, False, 256),
    (64, 224, 256, 1, False, True, 0),
    (64, 256, 224, 1, True, False, 0),
    (1, 64, 256, 3, True, False, 0),
    (5, 256, 352, 1, True, False, 0),
]


@pytest.mark.gpu
@pytest.mark.parametrize("boards,cin,n_out,ksize,relu,res,bn", CASES)
def test_conv_gemm_cases_within_float64_bound(boards, cin, n_out, ksize, relu, res, bn):
    ldo = ceil_to(n_out, 32)
    row = R(f"case[{cin},{n_out},{ksize}]", 0, cin, n_out, ksize, relu, res="h" if res else None, ldr=ldo, ldo=ldo)
    check_within_bound(row, boards, bn)


@pytest.mark.gpu
def test_conv_gemm_policy_logits_fp32_within_float64_bound():
    check_within_bound(R("policy", 0, 256, 81, 3, 0, outs="f", ldo=96), 64)
