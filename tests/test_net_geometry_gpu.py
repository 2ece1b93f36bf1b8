"""Network geometries across the range the weight-blob reader (Net::read_blob) accepts, run through the C-ABI
(ara_net_create / ara_net_predict) against the fp32 oracles (oracle/net.py, oracle/net_alphavile.py), and the reader's
refusals one step outside that range.

Every row of GEOMETRIES (network kinds of tests/net_harness.py) is a network built from the oracle's arch helpers with
edits, seeded by the oracle's make_state_dict and written by crazyara_b200.weights.export_blob.  Per row: Precision
float16 and float32 against the oracle with the bounds of tests/net_harness.py (DESIGN.md section 6), identical bits
from a graph replay, from the three tower kernel shapes and from every row of a batch, and the launch count of the
layer plan.  The float16 bounds hold at the scale of the RISE
test networks (trunk std ~0.4, logit std ~1; fp16 errors are absolute), so each row first checks that its seeded network
is at that scale.

The CPU half (blob round trip, scale, refusals) needs the built library but no device: read_blob runs before
ara_net_create touches a GPU."""
import numpy as np
import pytest

from oracle import net as onet
from oracle import net_alphavile as oav
from tests import net_harness as nh
from tests.net_harness import alphavile, rise


@pytest.fixture(scope="module", params=nh.GEOMETRIES)
def geo(request, tmp_path_factory):
    nets = nh.Nets(request.param, tmp_path_factory.mktemp(request.param))
    yield nets
    nets.close()


def batch_sizes():
    """1 board; 7, an odd count in the CTA-pair shape (an H100 holds dozens of CTA pairs at once); one board more than
    the device has SMs, where the default shape is two boards per CTA and the last CTA holds one board"""
    import torch
    return {"one": 1, "odd_pair": 7, "past_sms": torch.cuda.get_device_properties(0).multi_processor_count + 1}


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
    assert got["value_fc"] == (arch["value_fc"] if "ntb" in arch else 256)
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
    for name in nh.GEOMETRIES:
        a = nh.KINDS[name].arch()
        ntb = a.get("ntb") or []
        C = a.get("channels", 256)
        assert 64 <= C <= 256 and C % 32 == 0 and 1 <= len(a["kernels"]) <= 64, name
        assert 1 <= a["in_channels"] <= 256 and 1 <= a["policy_channels"] <= 256 and 1 <= a["value_fc"] <= 256, name
        assert all(c % 32 == 0 and c >= 32 for c, t in zip(a["c_ops"], ntb or [False] * len(a["c_ops"])) if not t), name
        if any(ntb):
            assert not ntb[0] and a["mhsa"] % 32 == 0 and a["mhca"] in (32, 64) and a["mhsa"] + a["mhca"] == C, name
            assert 64 <= a["mlp"] <= 1024 and a["mlp"] % 64 == 0, name


def _refused(tmp_path, arch):
    """the blob of arch with seeded weights -> the AraError message of ara_net_create"""
    from crazyara_b200 import AraError
    from crazyara_b200.nn import NeuralNetAPI
    from crazyara_b200.weights import export_blob
    sd = (oav if "ntb" in arch else onet).make_state_dict(arch, 3)
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
    out = nh.predict(geo.net(n), geo.arch, x)
    nh.check_float16(out, ref)
    nh.check_replay_bits(geo.net(n), geo.arch, x, out)


@pytest.mark.gpu
@pytest.mark.parametrize("size", ["one", "odd_pair"])
def test_float32_within_1e4_of_oracle(geo, size):
    n = batch_sizes()[size]
    x, ref = geo.ref(n, 42)
    out = nh.predict(geo.net(n, "float32"), geo.arch, x)
    nh.check_float32(out, ref)
    nh.check_replay_bits(geo.net(n, "float32"), geo.arch, x, out)


@pytest.mark.gpu
def test_tower_shapes_are_bit_identical(geo, monkeypatch):
    nh.check_tower_shapes(geo, geo.ref(5, 43)[0], monkeypatch)


@pytest.mark.gpu
def test_board_output_does_not_depend_on_its_row(geo):
    """a board alone gives the same bits as at the first, a middle and the last row of a batch past the SM count"""
    n = batch_sizes()["past_sms"]
    nh.check_rows_independent(geo, n, (0, n // 2, n - 1), seed=41, small=1)


@pytest.mark.gpu
@pytest.mark.parametrize("precision", ["float16", "float32"])
def test_launch_count_matches_the_layer_plan(geo, precision):
    nh.check_launch_count(geo, precision, n=3, seed=44)
