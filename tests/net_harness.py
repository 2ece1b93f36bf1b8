"""The networks the GPU network tests build, and the bounds a forward is held to against the fp32 oracles -- TEST
INFRASTRUCTURE ONLY.

KINDS names every network: its arch, its seeded weights, the exporter and input version of its blob and the oracle
forward it is compared with.  Nets opens one kind's blob and caches its networks and oracle outputs; predict runs a
network on host buffers; check_float16 / check_float32 apply the bounds of the two settings of the reference's UCI
option `Precision` (engine/src/uci/optionsuci.cpp:144):

  float16 (the reference's default): fp16 tensor-core operands and activations, fp32 accumulation.  fp16 errors are
          absolute, so the bounds hold at the scale of the seeded test networks (trunk std ~0.4, policy-logit std ~1).
  float32: the same wgmma GEMMs with fp16 hi + lo operand splitting and fp32 activations between the layers: every
          output within 1e-4 (north_star's float tolerance), in practice ~1e-6."""
from collections import namedtuple

import numpy as np

from crazyara_b200 import synthetic
from crazyara_b200.weights import export_blob, export_mx_blob
from oracle import net as onet
from oracle import net_alphavile as oav
from oracle import net_mx
from tests import classic_head, classic_mx_head
from tests.golden.gen_net_golden import golden_input

# float16
VALUE_ATOL, LOGIT_ATOL, PROB_RTOL, PROB_ATOL, AUX_ATOL = 4e-3, 2.5e-2, 3e-2, 1e-7, 6e-3
# float32: value, probabilities and aux within F32_ATOL, probabilities also relatively, centred logits
F32_ATOL, F32_PROB_RTOL, F32_PROB_ATOL, F32_LOGIT_ATOL = 1e-4, 2e-3, 1e-8, 1e-3
# both: every probability row sums to 1
PROB_SUM_ATOL = 1e-4

TOWER_MAX_BLOCKS = 24  # kTrunkMaxBlocks: the bottleneck blocks one tower kernel launch runs (rise_trunk_args.h)

Kind = namedtuple("Kind", "arch weights export version forward")


def _oracle(arch):
    return oav if "ntb" in arch else onet


def _torch(arch, version, seed):
    """ARAB2001 / ARAB2003: oracle/net.py or, with NTBs, oracle/net_alphavile.py"""
    return Kind(arch, lambda a: _oracle(a).make_state_dict(a, seed), export_blob, version,
                lambda sd, a, x: _oracle(a).forward(sd, a, x))


def _mx(arch, version):
    """ARAB2002: the reference's MXNet symbols, oracle/net_mx.py"""
    return Kind(arch, lambda a: net_mx.make_mx_params(a, 7), export_mx_blob, version, net_mx.forward_mx)


def _fc(base, n_labels, version):
    """ARAB2004: base with the fully-connected policy head onto n_labels classic labels, tests/classic_head.py"""
    return Kind(lambda: synthetic.classic(base(), n_labels),
                lambda a: {**_oracle(a).make_state_dict(a, 0), **synthetic.classic_head(a, n_labels, 0)}, export_blob,
                version, lambda sd, a, x: classic_head.forward(_oracle(a).forward, sd, a, x))


def _fc_mx(base, n_labels, version):
    """ARAB2004 around ARAB2002: the MXNet base with the head of tests/classic_mx_head.py"""
    return Kind(lambda: classic_mx_head.classic_arch(base(), n_labels),
                lambda a: classic_mx_head.make_params(base(), n_labels, 7)[1], export_mx_blob, version,
                classic_mx_head.forward)


# every SE flavour of the MXNet symbols side by side: ca_se with a sigmoid (RISEv2: ratio 2, hidden 128) or a hard
# sigmoid gate (rise_mobile_v3: ratio 16, hidden 16, zero-padded to 128), eca_se, plain blocks, one-chunk blocks
# (c_op <= 64), 3x3 and 5x5 depthwise kernels
MIXED_SE = ["ca_se", "eca_se", None, "ca_se", "eca_se", "ca_se", None, "eca_se", "ca_se", "ca_se"]
MIXED_GATE = ["sigmoid", "hard_sigmoid", None, "hard_sigmoid", "hard_sigmoid", "sigmoid", None, "hard_sigmoid", "hard_sigmoid",
              "sigmoid"]
MIXED_HIDDEN = [128, None, None, 16, None, 128, None, None, 16, 128]
MIXED_K = [3, 5, 3, 5, 3, 3, 5, 3, 3, 5]
MIXED_COP = [64, 128, 32, 224, 256, 96, 320, 64, 448, 160]


def mixed_arch():
    a = net_mx.arch_mx_risev33(52, 76)
    a.update(name="mx_mixed", se_types=list(MIXED_SE), se_gates=list(MIXED_GATE), se_hidden=list(MIXED_HIDDEN),
             kernels=list(MIXED_K), c_ops=list(MIXED_COP))
    return a


def alphavile(C, M, Ca, H, layout, in_channels=52, policy_channels=76, wdl=True, value_fc=None):
    """an ARAB2003 arch; layout: per block (c_op, kernel) for a bottleneck block or "ntb" for an NTB of widths M, Ca, H"""
    ntb = [b == "ntb" for b in layout]
    return dict(name=f"alphavile_{C}_{len(layout)}b", in_channels=in_channels, policy_channels=policy_channels, channels=C,
                kernels=[3 if t else b[1] for b, t in zip(layout, ntb)], se_types=[None] * len(layout),
                c_ops=[0 if t else b[0] for b, t in zip(layout, ntb)], ntb=ntb, mhsa=M, mhca=Ca, mlp=H, wdl=wdl,
                value_channels=8, value_fc=C if value_fc is None else value_fc)


def rise(n_blocks, c_ops=None, in_channels=34, policy_channels=81):
    """an ARAB2001 arch: RISEv2 (oracle.net.arch_risev2) with its 13-block pattern of widths and ca_se blocks repeated"""
    a = onet.arch_risev2(in_channels, policy_channels)
    a.update(name=f"rise_{n_blocks}b", kernels=[3] * n_blocks, c_ops=c_ops or [a["c_ops"][i % 13] for i in range(n_blocks)],
             se_types=[a["se_types"][i % 13] for i in range(n_blocks)])
    return a


KINDS = {
    "risev2": _torch(lambda: onet.arch_risev2(34, 81), 10, 0),
    "risev2_63_84": _torch(lambda: onet.arch_risev2(63, 84), 10, 0),
    "risev33": _torch(lambda: onet.arch_risev33(52, 76, True), 30, 0),
    "risev33_64_81": _torch(lambda: onet.arch_risev33(64, 81, True), 30, 0),
    "mx_risev2": _mx(lambda: net_mx.arch_mx_risev2(34, 81), 10),
    "mx_risev33": _mx(lambda: net_mx.arch_mx_risev33(52, 76), 30),
    "mx_mixed": _mx(mixed_arch, 30),
    "av_tiny": _torch(lambda: oav.arch_alphavile("tiny", 34, 81, False), 10, 7),
    "av_normal": _torch(lambda: oav.arch_alphavile("normal", 52, 76, True), 30, 7),
    # every label count, P from 2 to 81
    "fc_risev2_81_2272": _fc(lambda: onet.arch_risev2(34, 81), 2272, 10),
    "fc_risev2_2_2316": _fc(lambda: onet.arch_risev2(34, 2), 2316, 10),
    "fc_risev2_16_1968": _fc(lambda: onet.arch_risev2(34, 16), 1968, 10),
    "fc_risev33_76_1968": _fc(lambda: onet.arch_risev33(52, 76, True), 1968, 30),
    "fc_av_tiny_2316": _fc(lambda: oav.arch_alphavile("tiny", 34, 81, False), 2316, 10),
    # RISEv2 with sigmoid ca_se, a stem ReLU and no policy bias; RISEv3.3 with eca_se, clamp(0.2 x + 0.5) gates, no stem
    # activation and a policy convolution bias (folded into the head with policy_bn1)
    "fc_mx_risev2_2272": _fc_mx(lambda: net_mx.arch_mx_risev2(34, 81), 2272, 10),
    "fc_mx_risev33_1968": _fc_mx(lambda: net_mx.arch_mx_risev33(52, 76), 1968, 30),
    # geometries across the range the weight-blob reader (Net::read_blob) accepts, with what each exercises:
    # a 21-block tower segment, then one NTB; the non-WDL value head on a 192-channel trunk
    "av_small": _torch(lambda: oav.arch_alphavile("small", 34, 81, False), 30, 7),
    # a 24-block segment (as many as one tower launch holds), NTB, 11 blocks, NTB: 37 blocks
    "av_large": _torch(lambda: oav.arch_alphavile("large", 52, 76, True), 30, 7),
    # one attention head; the smallest MLP; a half-chunk block; a tower segment after the last NTB; value_fc 1
    "narrow64": _torch(lambda: alphavile(64, 32, 32, 64, [(32, 3), (128, 5), "ntb", (32, 5)], wdl=False, value_fc=1), 30, 7),
    # 7 heads, a q | k | v pitch of 672; the largest MLP; a 256-wide trunk (no zero padding); NTB after NTB
    "full256_ntb": _torch(lambda: alphavile(256, 224, 32, 1024, [(512, 3), (384, 5), "ntb", "ntb"]), 30, 7),
    # a one-block first segment (NTB at block 1); 3 heads; a 160-channel trunk; a 16-chunk block (c_op 1024)
    "mid160": _torch(lambda: alphavile(160, 96, 64, 320, [(320, 3), "ntb", (1024, 5), (224, 3)]), 30, 7),
    # the largest input conversion and softmax (256 input planes, 256 policy planes = 16,384 labels)
    "heads_max": _torch(lambda: rise(2, in_channels=256, policy_channels=256), 30, 7),
    # one block of c_op 32, one input plane, one policy plane (64 labels)
    "heads_min": _torch(lambda: rise(1, c_ops=[32], in_channels=1, policy_channels=1), 30, 7),
    # one block more than a tower launch holds: segments of 24 + 1 blocks
    "rise25": _torch(lambda: rise(25), 30, 7),
    # three tower segments (24 + 24 + 1)
    "rise49": _torch(lambda: rise(49), 30, 7),
    # a run of 25 bottleneck blocks before an NTB (segments 24 + 1), then 2 blocks
    "av_long_run": _torch(lambda: alphavile(192, 160, 32, 384, [(384, 3 + 2 * (i % 3 == 1)) for i in range(25)] +
                                            ["ntb", (384, 3), (256, 5)]), 30, 7),
}
GEOMETRIES = ["av_small", "av_large", "narrow64", "full256_ntb", "mid160", "heads_max", "heads_min", "rise25", "rise49",
              "av_long_run"]


def inputs(arch, n, seed):
    """golden_input's boards: 15 % of the squares set, the last three planes scalar (with fewer planes: each plane's set
    squares scaled by a random factor instead)"""
    if arch["in_channels"] >= 3:
        return golden_input(arch, n=n, seed=seed)
    rng = np.random.default_rng(seed)
    x = (rng.random((n, arch["in_channels"], 8, 8)) < 0.15).astype(np.float32)
    return x * (0.5 + rng.random((n, arch["in_channels"], 1, 1))).astype(np.float32)


def n_labels(arch):
    """the policy's width: P * 64 with a policy map, L with a fully-connected head"""
    return arch.get("n_labels") or arch["policy_channels"] * 64


class Nets:
    """One kind's blob, its oracle outputs (cached by n and seed) and its networks (cached by batch and precision),
    closed together."""

    def __init__(self, kind, tmp):
        k = KINDS[kind]
        self.arch = k.arch()
        self.weights, self.forward = k.weights(self.arch), k.forward
        self.blob = k.export(self.weights, self.arch, str(tmp / f"{kind}.arab"), input_version=k.version)
        self.nets, self.opened, self.refs = {}, [], {}

    def net(self, batch, precision="float16"):
        if (batch, precision) not in self.nets:
            self.nets[batch, precision] = self.fresh(batch, precision)
        return self.nets[batch, precision]

    def fresh(self, batch, precision="float16"):
        from crazyara_b200.nn import NeuralNetAPI
        self.opened.append(NeuralNetAPI("gpu", 0, batch, self.blob, precision=precision))
        return self.opened[-1]

    def ref(self, n, seed):
        """-> (input planes, the oracle's outputs)"""
        if (n, seed) not in self.refs:
            x = inputs(self.arch, n, seed)
            self.refs[n, seed] = x, self.forward(self.weights, self.arch, x)
        return self.refs[n, seed]

    def close(self):
        for net in self.opened:
            net.close()


def module_nets(tmp_path_factory):
    """the body of a module fixture: yields kind -> that kind's Nets, opened on first use and closed with the module"""
    opened = {}

    def get(kind):
        if kind not in opened:
            opened[kind] = Nets(kind, tmp_path_factory.mktemp(kind))
        return opened[kind]
    yield get
    for nets in opened.values():
        nets.close()


Out = namedtuple("Out", "value prob aux")


def predict(net, arch, x):
    """-> Out(value [n], prob [n, labels], aux [n, 4] or None without WDL) of the first n = len(x) rows of net's batch.
    Every output starts as NaN, so a row the forward leaves unwritten fails the checks."""
    n, batch = x.shape[0], net.get_batch_size()
    xin = np.zeros((batch,) + x.shape[1:], np.float32)
    xin[:n] = x
    v = np.full(batch, np.nan, np.float32)
    p = np.full((batch, n_labels(arch)), np.nan, np.float32)
    aux = np.full((batch, 4), np.nan, np.float32) if arch["wdl"] else None
    net.predict(xin, v, p, aux, n=n)
    return Out(v[:n].copy(), p[:n].copy(), None if aux is None else aux[:n].copy())


def take(out, sl):
    """-> the rows sl of every output"""
    return Out(*(None if t is None else t[sl] for t in out))


def same_bits(a, b):
    return all((x is None and y is None) or np.array_equal(x, y) for x, y in zip(a, b))


def _centred(logits):
    lg = np.asarray(logits, np.float64)
    return lg - lg.mean(1, keepdims=True)


def _check_rows(out, ref, logit_atol):
    """finite outputs, probability rows that sum to 1, and centred log-probabilities near the oracle's centred logits"""
    assert all(np.isfinite(t).all() for t in out if t is not None), "finite"
    np.testing.assert_allclose(out.prob.sum(1, dtype=np.float64), 1.0, rtol=0, atol=PROB_SUM_ATOL,
                               err_msg="probability row sums")
    err = np.abs(_centred(np.log(out.prob.astype(np.float64))) - _centred(ref["policy_logits"])).max()
    assert err < logit_atol, f"centred logits {err}"


def check_float16(out, ref):
    """Precision float16 against the fp32 oracle's outputs ref"""
    np.testing.assert_allclose(out.value, ref["value"], rtol=0, atol=VALUE_ATOL, err_msg="value")
    np.testing.assert_allclose(out.prob, ref["prob"], rtol=PROB_RTOL, atol=PROB_ATOL, err_msg="probabilities")
    if out.aux is not None:
        np.testing.assert_allclose(out.aux, ref["aux"], rtol=0, atol=AUX_ATOL, err_msg="aux")
    _check_rows(out, ref, LOGIT_ATOL)


def check_float32(out, ref):
    """Precision float32 against the fp32 oracle's outputs ref"""
    np.testing.assert_allclose(out.value, ref["value"], rtol=0, atol=F32_ATOL, err_msg="value")
    np.testing.assert_allclose(out.prob, ref["prob"], rtol=0, atol=F32_ATOL, err_msg="probabilities")
    np.testing.assert_allclose(out.prob, ref["prob"], rtol=F32_PROB_RTOL, atol=F32_PROB_ATOL, err_msg="probabilities")
    if out.aux is not None:
        np.testing.assert_allclose(out.aux, ref["aux"], rtol=0, atol=F32_ATOL, err_msg="aux")
    _check_rows(out, ref, F32_LOGIT_ATOL)


def check_replay_bits(net, arch, x, out):
    """a second forward (a graph replay) gives the bits of out: no stale state"""
    assert same_bits(predict(net, arch, x), out)


def check_tower_shapes(nets, x, monkeypatch, rows=("32", "64", "128"), repeats=1):
    """The tower kernel's shapes, forced by ARA_TRUNK_ROWS (32: a CTA pair per board, 64: one board per CTA, 128: two
    boards per CTA), give the same bits on a new network of batch len(x) each, in every one of `repeats` forwards (a
    race in the weight ring would not show every time).  -> those outputs"""
    outs = []
    for r in rows:
        monkeypatch.setenv("ARA_TRUNK_ROWS", r)
        net = nets.fresh(len(x))
        outs += [(r, predict(net, nets.arch, x)) for _ in range(repeats)]
        net.close()
    monkeypatch.delenv("ARA_TRUNK_ROWS")
    for r, out in outs:
        assert same_bits(out, outs[0][1]), f"ARA_TRUNK_ROWS={r} differs from {outs[0][0]}"
    return outs[0][1]


def check_rows_independent(nets, batch, at, seed, small=3, precision="float16"):
    """A board gives the same bits at each row `at` of a full batch as in a network of batch `small`, where it follows
    another board (alone with small = 1): the search packs a leaf at any row of a batch of any size."""
    x = inputs(nets.arch, batch, seed)
    together = predict(nets.net(batch, precision), nets.arch, x)
    for row in at:
        xin = x[[row]] if small == 1 else x[[(row + 5) % batch, row]]
        out = predict(nets.net(small, precision), nets.arch, xin)
        assert same_bits(take(out, slice(-1, None)), take(together, slice(row, row + 1))), (precision, row)


def tower_segments(arch):
    """float16 tower launches: one per run of at most TOWER_MAX_BLOCKS consecutive bottleneck blocks"""
    runs, run = [], 0
    for t in arch.get("ntb") or [False] * len(arch["kernels"]):
        if t:
            runs.append(run)
            run = 0
        else:
            run += 1
    runs.append(run)
    return sum(-(-r // TOWER_MAX_BLOCKS) for r in runs)


def expected_launches(arch, precision):
    """input conversion, stem, value head, two policy convolutions and the softmax (a fully-connected head adds its
    layer), plus the tower: float16 one launch per tower segment and 9 per NTB, float32 3 per bottleneck block (+1 with
    squeeze-excitation) and 10 per NTB"""
    ntb = arch.get("ntb") or [False] * len(arch["kernels"])
    if precision == "float16":
        tower = tower_segments(arch) + 9 * sum(ntb)
    else:
        tower = sum(10 if t else 3 + (se is not None) for t, se in zip(ntb, arch["se_types"]))
    return 6 + ("n_labels" in arch) + tower


def check_launch_count(nets, precision, n, seed):
    """The first forward of a size runs eagerly (every launch counted) before it is captured; a graph replay then adds
    the launches its capture enqueued.  Both must agree with the layer plan."""
    net, x = nets.fresh(n, precision), inputs(nets.arch, n, seed)
    predict(net, nets.arch, x)
    first = net.launch_count()
    predict(net, nets.arch, x)
    per_forward = net.launch_count() - first
    net.close()
    assert first == 2 * per_forward
    assert per_forward == expected_launches(nets.arch, precision)
