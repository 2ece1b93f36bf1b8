"""Network geometries across the range the weight-blob reader (Net::read_blob) accepts, run through the C-ABI
(ara_net_create / ara_net_predict) against the fp32 oracles (oracle/net.py, oracle/net_alphavile.py), and the reader's
refusals one step outside that range.

Every row of GEOMETRIES is a network built from the oracle's arch helpers with edits, seeded by the oracle's
make_state_dict and written by crazyara_b200.weights.export_blob.  Per row: Precision float16 and float32 against the
oracle with the bounds of tests/test_net_gpu.py (DESIGN.md section 6), identical bits from the three tower kernel shapes
and from every row of a batch, and the launch count of the layer plan.  The float16 bounds hold at the scale of the RISE
test networks (trunk std ~0.4, logit std ~1; fp16 errors are absolute), so each row first checks that its seeded network
is at that scale.

The CPU half (blob round trip, scale, refusals) needs the built library but no device: read_blob runs before
ara_net_create touches a GPU."""
from collections import namedtuple

import numpy as np
import pytest

from oracle import net as onet
from oracle import net_alphavile as oav
from tests.golden.gen_net_golden import golden_input

VALUE_ATOL, LOGIT_ATOL, PROB_RTOL, AUX_ATOL = 4e-3, 2.5e-2, 3e-2, 6e-3  # float16, as tests/test_net_gpu.py
F32_ATOL, F32_LOGIT_ATOL, F32_PROB_RTOL = 1e-4, 1e-3, 2e-3                # float32, as tests/test_net_gpu.py
TOWER_MAX_BLOCKS = 24  # kTrunkMaxBlocks: the bottleneck blocks one tower kernel launch runs (rise_trunk_args.h)

Row = namedtuple("Row", "name arch exercises")


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


GEOMETRIES = [
    Row("av_small", oav.arch_alphavile("small", 34, 81, False),
        "a 21-block tower segment, then one NTB; the non-WDL value head on a 192-channel trunk"),
    Row("av_large", oav.arch_alphavile("large", 52, 76, True),
        "a 24-block segment (as many as one tower launch holds), NTB, 11 blocks, NTB: 37 blocks"),
    Row("narrow64", alphavile(64, 32, 32, 64, [(32, 3), (128, 5), "ntb", (32, 5)], wdl=False, value_fc=1),
        "one attention head; the smallest MLP; a half-chunk block; a tower segment after the last NTB; value_fc 1"),
    Row("full256_ntb", alphavile(256, 224, 32, 1024, [(512, 3), (384, 5), "ntb", "ntb"]),
        "7 heads, a q | k | v pitch of 672; the largest MLP; a 256-wide trunk (no zero padding); NTB after NTB"),
    Row("mid160", alphavile(160, 96, 64, 320, [(320, 3), "ntb", (1024, 5), (224, 3)]),
        "a one-block first segment (NTB at block 1); 3 heads; a 160-channel trunk; a 16-chunk block (c_op 1024)"),
    Row("heads_max", rise(2, in_channels=256, policy_channels=256),
        "the largest input conversion and softmax (256 input planes, 256 policy planes = 16,384 labels)"),
    Row("heads_min", rise(1, c_ops=[32], in_channels=1, policy_channels=1),
        "one block of c_op 32, one input plane, one policy plane (64 labels)"),
    Row("rise25", rise(25), "one block more than a tower launch holds: segments of 24 + 1 blocks"),
    Row("rise49", rise(49), "three tower segments (24 + 24 + 1)"),
    Row("av_long_run", alphavile(192, 160, 32, 384, [(384, 3 + 2 * (i % 3 == 1)) for i in range(25)] + ["ntb", (384, 3), (256, 5)]),
        "a run of 25 bottleneck blocks before an NTB (segments 24 + 1), then 2 blocks"),
]
IDS = [r.name for r in GEOMETRIES]


def planes(arch, n, seed):
    """golden_input's boards: 15 % of the squares set, the last three planes scalar (with fewer planes: each plane's set
    squares scaled by a random factor instead)"""
    if arch["in_channels"] >= 3:
        return golden_input(arch, n=n, seed=seed)
    rng = np.random.default_rng(seed)
    x = (rng.random((n, arch["in_channels"], 8, 8)) < 0.15).astype(np.float32)
    return x * (0.5 + rng.random((n, arch["in_channels"], 1, 1))).astype(np.float32)


def is_alphavile(arch):
    return "ntb" in arch


def state_dict(row):
    """the oracle's seeded parameters: their residual branches are damped enough that 49 blocks stay at the test scale
    (test_row_network_is_at_the_test_scale)"""
    return (oav if is_alphavile(row.arch) else onet).make_state_dict(row.arch, 7)


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
    """input conversion, stem, value head, two policy convolutions and the softmax, plus the tower: float16 one launch per
    tower segment and 9 per NTB, float32 3 per bottleneck block (+1 with squeeze-excitation) and 10 per NTB"""
    ntb = arch.get("ntb") or [False] * len(arch["kernels"])
    if precision == "float16":
        tower = tower_segments(arch) + 9 * sum(ntb)
    else:
        tower = sum(10 if t else 3 + (se is not None) for t, se in zip(ntb, arch["se_types"]))
    return 6 + tower


class RowNets:
    """one row's blob, oracle outputs and networks (cached by batch and precision), closed with the row"""

    def __init__(self, row, tmp):
        from crazyara_b200.weights import export_blob
        self.row, self.arch = row, row.arch
        self.sd = state_dict(row)
        self.blob = export_blob(self.sd, self.arch, str(tmp / f"{row.name}.arab"), input_version=30)
        self.nets, self.fresh_nets, self.refs = {}, [], {}

    def net(self, batch, precision="float16"):
        if (batch, precision) not in self.nets:
            self.nets[batch, precision] = self.fresh(batch, precision)
        return self.nets[batch, precision]

    def fresh(self, batch, precision="float16"):
        from crazyara_b200.nn import NeuralNetAPI
        self.fresh_nets.append(NeuralNetAPI("gpu", 0, batch, self.blob, precision=precision))
        return self.fresh_nets[-1]

    def ref(self, n, seed):
        if (n, seed) not in self.refs:
            x = planes(self.arch, n, seed)
            self.refs[n, seed] = x, (oav if is_alphavile(self.arch) else onet).forward(self.sd, self.arch, x)
        return self.refs[n, seed]

    def predict(self, net, x):
        """-> value [n], prob [n, labels], aux [n, 4] (None without WDL) of the first x.shape[0] rows of net's batch"""
        n, batch = x.shape[0], net.get_batch_size()
        xin = np.zeros((batch, self.arch["in_channels"], 8, 8), np.float32)
        xin[:n] = x
        v = np.full(batch, np.nan, np.float32)
        p = np.full((batch, self.arch["policy_channels"] * 64), np.nan, np.float32)
        aux = np.full((batch, 4), np.nan, np.float32) if self.arch["wdl"] else None
        net.predict(xin, v, p, aux, n=n)
        return v[:n].copy(), p[:n].copy(), None if aux is None else aux[:n].copy()

    def close(self):
        for net in self.fresh_nets:
            net.close()


@pytest.fixture(scope="module", params=GEOMETRIES, ids=IDS)
def geo(request, tmp_path_factory):
    nets = RowNets(request.param, tmp_path_factory.mktemp(request.param.name))
    yield nets
    nets.close()


def batch_sizes():
    """1 board; 7, an odd count in the CTA-pair shape (an H100 holds dozens of CTA pairs at once); one board more than
    the device has SMs, where the default shape is two boards per CTA and the last CTA holds one board"""
    import torch
    return {"one": 1, "odd_pair": 7, "past_sms": torch.cuda.get_device_properties(0).multi_processor_count + 1}


def centred_log(p):
    lp = np.log(p.astype(np.float64))
    return lp - lp.mean(1, keepdims=True)


# ------------------------------------------------------------------------------------------------ CPU half
def test_row_blob_round_trips_through_the_python_reader(geo, tmp_path):
    """export_blob -> weights.read_blob gives back the row's geometry, and write_blob rewrites it byte for byte"""
    from crazyara_b200.weights import read_blob, write_blob
    arch, (got, tensors, version) = geo.arch, read_blob(geo.blob)
    ntb = arch.get("ntb") or [False] * len(arch["kernels"])
    assert version == 30
    for k in ("in_channels", "policy_channels", "wdl"):
        assert got[k] == arch[k], k
    assert got["channels"] == arch.get("channels", 256)
    assert got["value_fc"] == (arch["value_fc"] if is_alphavile(arch) else 256)
    assert (got.get("ntb") or [False] * len(ntb)) == ntb
    plain = [i for i, t in enumerate(ntb) if not t]
    assert [got["c_ops"][i] for i in plain] == [arch["c_ops"][i] for i in plain]
    assert [got["kernels"][i] for i in plain] == [arch["kernels"][i] for i in plain]
    assert [got["se_types"][i] for i in plain] == [arch["se_types"][i] for i in plain]
    if any(ntb):
        assert (got["mhsa"], got["mhca"], got["mlp"]) == (arch["mhsa"], arch["mhca"], arch["mlp"])
    again = write_blob(str(tmp_path / "again.arab"), got, tensors, version)
    assert open(again, "rb").read() == open(geo.blob, "rb").read()


def test_row_network_is_at_the_test_scale(geo):
    """the float16 bounds were set at a trunk std of ~0.4 and a policy-logit std of ~1"""
    _, ref = geo.ref(16, 31)
    trunk_std, logit_std = float(ref["trunk"].std()), float(ref["policy_logits"].std(1).mean())
    assert 0.2 < trunk_std < 0.8, trunk_std
    assert 0.5 < logit_std < 2.0, logit_std
    assert np.isfinite(ref["value"]).all() and np.abs(ref["value"]).max() < 1


def test_geometries_are_inside_the_readers_range():
    for r in GEOMETRIES:
        a, ntb = r.arch, r.arch.get("ntb") or []
        C = a.get("channels", 256)
        assert 64 <= C <= 256 and C % 32 == 0 and 1 <= len(a["kernels"]) <= 64, r.name
        assert 1 <= a["in_channels"] <= 256 and 1 <= a["policy_channels"] <= 256 and 1 <= a["value_fc"] <= 256, r.name
        assert all(c % 32 == 0 and c >= 32 for c, t in zip(a["c_ops"], ntb or [False] * len(a["c_ops"])) if not t), r.name
        if any(ntb):
            assert not ntb[0] and a["mhsa"] % 32 == 0 and a["mhca"] in (32, 64) and a["mhsa"] + a["mhca"] == C, r.name
            assert 64 <= a["mlp"] <= 1024 and a["mlp"] % 64 == 0, r.name


def _refused(tmp_path, arch):
    """the blob of arch with seeded weights -> the AraError message of ara_net_create"""
    from crazyara_b200 import AraError
    from crazyara_b200.nn import NeuralNetAPI
    from crazyara_b200.weights import export_blob
    sd = (oav if is_alphavile(arch) else onet).make_state_dict(arch, 3)
    blob = export_blob(sd, arch, str(tmp_path / "refused.arab"), input_version=30)
    with pytest.raises(AraError) as e:
        NeuralNetAPI("gpu", 0, 1, blob)
    return str(e.value)


_AV = dict(C=224, M=160, Ca=64, H=448, layout=[(448, 3), "ntb", (448, 5)])


def _av(**k):
    return alphavile(**dict(_AV, **k))


REFUSALS = [
    ("channels_48", alphavile(48, 32, 32, 64, [(64, 3), (64, 5)]), "unsupported trunk geometry (channels 48"),
    ("channels_288", alphavile(288, 32, 32, 64, [(64, 3)]), "unsupported trunk geometry (channels 288"),
    ("channels_200", alphavile(200, 32, 32, 64, [(64, 3)]), "unsupported trunk geometry (channels 200"),
    ("ntb_at_block_0", _av(layout=["ntb", (448, 3)]), "block 0 is an NTB"),
    ("mhca_96", _av(C=256, M=160, Ca=96), "unsupported NTB widths M 160 Ca 96 H 448 (trunk 256"),
    ("m_plus_ca_not_c", _av(M=160, Ca=32), "unsupported NTB widths M 160 Ca 32 H 448 (trunk 224"),
    ("mlp_32", _av(H=32), "unsupported NTB widths M 160 Ca 64 H 32 "),
    ("mlp_1088", _av(H=1088), "unsupported NTB widths M 160 Ca 64 H 1088 "),
    ("c_op_16", _av(layout=[(448, 3), "ntb", (16, 3)]), "unsupported block (c_op 16 "),
    ("se_on_224", dict(_av(), se_types=[None, None, "ca_se"]), "block 2: squeeze-excitation on a 224-channel trunk"),
    ("blocks_65", rise(65, c_ops=[32] * 65), "65 blocks (1 .. 64)"),
    ("in_channels_257", rise(1, c_ops=[32], in_channels=257), "in_channels 257, policy_channels 81"),
    ("policy_channels_257", rise(1, c_ops=[32], policy_channels=257), "in_channels 34, policy_channels 257"),
    ("value_fc_257", _av(wdl=False, value_fc=257), "unsupported trunk geometry (channels 224, value 8/257)"),
]


@pytest.mark.parametrize("arch,message", [c[1:] for c in REFUSALS], ids=[c[0] for c in REFUSALS])
def test_reader_refuses_one_step_outside_its_range(tmp_path, arch, message):
    assert message in _refused(tmp_path, arch)


# ------------------------------------------------------------------------------------------------ GPU half
@pytest.mark.gpu
@pytest.mark.parametrize("size", ["one", "odd_pair", "past_sms"])
def test_float16_matches_oracle(geo, size):
    n = batch_sizes()[size]
    x, ref = geo.ref(n, 41)
    v, p, aux = geo.predict(geo.net(n), x)
    assert np.isfinite(v).all() and np.isfinite(p).all()
    np.testing.assert_allclose(p.sum(1), 1.0, atol=1e-4)
    np.testing.assert_allclose(v, ref["value"], atol=VALUE_ATOL, rtol=0)
    assert np.abs(centred_log(p) - centred_log(ref["prob"])).max() < LOGIT_ATOL
    np.testing.assert_allclose(p, ref["prob"], rtol=PROB_RTOL, atol=1e-7)
    if aux is not None:
        np.testing.assert_allclose(aux, ref["aux"], atol=AUX_ATOL, rtol=0)


@pytest.mark.gpu
@pytest.mark.parametrize("size", ["one", "odd_pair"])
def test_float32_within_1e4_of_oracle(geo, size):
    n = batch_sizes()[size]
    x, ref = geo.ref(n, 42)
    v, p, aux = geo.predict(geo.net(n, "float32"), x)
    np.testing.assert_allclose(v, ref["value"], atol=F32_ATOL, rtol=0)
    np.testing.assert_allclose(p, ref["prob"], atol=F32_ATOL, rtol=0)
    np.testing.assert_allclose(p, ref["prob"], rtol=F32_PROB_RTOL, atol=1e-8)
    assert np.abs(centred_log(p) - centred_log(ref["prob"])).max() < F32_LOGIT_ATOL
    if aux is not None:
        np.testing.assert_allclose(aux, ref["aux"], atol=F32_ATOL, rtol=0)


def _same_bits(a, b):
    return all((x is None and y is None) or np.array_equal(x, y) for x, y in zip(a, b))


@pytest.mark.gpu
def test_tower_shapes_are_bit_identical(geo, monkeypatch):
    """ARA_TRUNK_ROWS 32 (the CTA pair), 64 (one board per CTA) and 128 (two boards per CTA) give the same bits"""
    x, _ = geo.ref(5, 43)
    outs = {}
    for rows in ("32", "64", "128"):
        monkeypatch.setenv("ARA_TRUNK_ROWS", rows)
        outs[rows] = geo.predict(geo.fresh(5), x)
    for rows, out in outs.items():
        assert _same_bits(out, outs["64"]), f"ARA_TRUNK_ROWS={rows} differs"


@pytest.mark.gpu
def test_board_output_does_not_depend_on_its_row(geo):
    """a board alone gives the same bits as at the first, a middle and the last row of a batch past the SM count"""
    n = batch_sizes()["past_sms"]
    xs, _ = geo.ref(n, 41)
    together = geo.predict(geo.net(n), xs)
    for row in (0, n // 2, n - 1):
        alone = geo.predict(geo.net(1), xs[row:row + 1])
        assert _same_bits(alone, [None if t is None else t[row:row + 1] for t in together]), f"row {row}"


@pytest.mark.gpu
@pytest.mark.parametrize("precision", ["float16", "float32"])
def test_launch_count_matches_the_layer_plan(geo, precision):
    """the first forward of a size runs eagerly and is then captured (its launches counted once each way); a replay
    counts the launches of the capture"""
    net = geo.fresh(3, precision)
    x, _ = geo.ref(3, 44)
    geo.predict(net, x)
    first = net.launch_count()
    geo.predict(net, x)
    per_forward = net.launch_count() - first
    assert first == 2 * per_forward
    assert per_forward == expected_launches(geo.arch, precision)
