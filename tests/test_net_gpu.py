"""GPU networks against their fp32 oracles through the C-ABI with host buffers, in both settings of the reference's UCI
option `Precision`, within the bounds of tests/net_harness.py.  One table holds every network family's comparisons:
the torch RISE networks (ARAB2001, oracle/net.py), the reference's MXNet symbols (ARAB2002, oracle/net_mx.py),
AlphaVile (ARAB2003, oracle/net_alphavile.py) and the fully-connected policy head on top of each (ARAB2004,
tests/classic_head.py, tests/classic_mx_head.py)."""
import numpy as np
import pytest

from tests import net_harness as nh

P16, P32 = "float16", "float32"
# (kind, batch, n): batches from 1 to 128, 66 a partial last board tile of the fully-connected head
RISE = [("risev2", 8, 8), ("risev2", 64, 64), ("risev2", 1, 1), ("risev33", 64, 64), ("risev33", 8, 5),
        ("risev2_63_84", 16, 16)]
FC = [("fc_risev2_81_2272", 1, 1), ("fc_risev2_81_2272", 8, 5), ("fc_risev2_81_2272", 64, 64),
      ("fc_risev2_81_2272", 66, 66), ("fc_risev2_81_2272", 128, 128), ("fc_risev33_76_1968", 8, 8),
      ("fc_risev2_2_2316", 8, 8), ("fc_risev2_16_1968", 64, 64), ("fc_av_tiny_2316", 8, 8)]
FC_MX = [("fc_mx_risev2_2272", 1, 1), ("fc_mx_risev2_2272", 8, 5), ("fc_mx_risev2_2272", 66, 66),
         ("fc_mx_risev2_2272", 128, 128), ("fc_mx_risev33_1968", 1, 1), ("fc_mx_risev33_1968", 16, 16),
         ("fc_mx_risev33_1968", 128, 128)]
# (kind, batch, n, precision, input seed), grouped by kind
CASES = sorted([(k, b, n, P16, 5) for k, b, n in RISE] +
               [(k, b, n, P32, 5) for k, b, n in RISE + [("risev2_63_84", 128, 128), ("risev33_64_81", 16, 16)]] +
               [(k, n, n, p, seed) for k in ("mx_risev2", "mx_risev33", "mx_mixed", "av_tiny", "av_normal")
                for p, seed, sizes in ((P16, 21, (1, 5, 64, 66, 128)), (P32, 22, (1, 16))) for n in sizes] +
               [(k, b, n, p, 5) for k, b, n in FC for p in (P16, P32)] +
               [(k, b, n, p, 31) for k, b, n in FC_MX for p in (P16, P32)], key=lambda c: c[0])


@pytest.fixture(scope="module")
def nets(tmp_path_factory):
    yield from nh.module_nets(tmp_path_factory)


@pytest.mark.gpu
@pytest.mark.parametrize("kind,batch,n,precision,seed", CASES)
def test_net_predict_matches_oracle(nets, kind, batch, n, precision, seed):
    kn = nets(kind)
    net, arch = kn.net(batch, precision), kn.arch
    assert net.is_policy_map() == ("n_labels" not in arch) and net.get_nb_policy_values() == nh.n_labels(arch)
    assert net.get_nb_input_values_total() == arch["in_channels"] * 64
    x, ref = kn.ref(n, seed)
    out = nh.predict(net, arch, x)
    (nh.check_float16 if precision == P16 else nh.check_float32)(out, ref)
    nh.check_replay_bits(net, arch, x, out)


@pytest.mark.gpu
@pytest.mark.parametrize("precision", [P16, P32])
@pytest.mark.parametrize("kind", ["risev33", "mx_risev2"])
def test_launch_bookkeeping_matches_the_launches(nets, kind, precision):
    """input conversion, stem, the tower kernel (float16) or per block the squeeze-excitation if any, conv1, depthwise
    and conv2 (float32), value head, two policy convolutions, softmax"""
    nh.check_launch_count(nets(kind), precision, n=4, seed=25)


@pytest.mark.gpu
def test_net_create_fails_loudly_on_bad_blob(tmp_path):
    from crazyara_b200 import AraError
    from crazyara_b200.nn import NeuralNetAPI
    p = tmp_path / "bad.arab"
    p.write_bytes(b"not a blob")
    with pytest.raises(AraError):
        NeuralNetAPI("gpu", 0, 8, str(p))
    with pytest.raises(AraError):
        NeuralNetAPI("gpu", 0, 8, str(tmp_path / "missing.arab"))


@pytest.mark.gpu
def test_net_output_of_a_position_does_not_depend_on_its_batch(nets):
    """The search relies on this: a leaf's value / policy are the same bits whichever mini-batch evaluates it."""
    nh.check_rows_independent(nets("risev2"), 64, (0, 37, 63), seed=9)


@pytest.mark.gpu
def test_float32_net_output_of_a_position_does_not_depend_on_its_batch(nets):
    """The same in Precision float32, where the 1x1 convolutions of the tower are GEMM launches whose tile width follows
    the batch (conv_layer_choose_bn): packed multi-tree float32 searches put a leaf at any row of a batch of any size."""
    nh.check_rows_independent(nets("risev2"), 64, (0, 37, 63), seed=9, precision=P32)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["risev2", "risev33"], ids=["risev2-34-81", "risev33-52-76"])
def test_float16_and_float32_networks_agree(nets, monkeypatch, kind):
    """The tower kernel in each shape (Precision float16) against the layer-by-layer Precision float32 network: same
    weights, fp16 tolerance."""
    kn = nets(kind)
    x = nh.inputs(kn.arch, 6, 3)
    f16 = nh.check_tower_shapes(kn, x, monkeypatch)
    f32 = nh.predict(kn.net(6, P32), kn.arch, x)
    np.testing.assert_allclose(f16.value, f32.value, atol=nh.VALUE_ATOL)
    np.testing.assert_allclose(f16.prob, f32.prob, rtol=nh.PROB_RTOL, atol=1e-6)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["risev2", "risev33"], ids=["risev2-34-81", "risev33-52-76"])
def test_tower_variants_are_bit_identical(nets, monkeypatch, kind):
    """The tower kernel's shapes must give the same bits: a search with many trees evaluates the same positions in
    bigger batches.  At 140 boards (more than the SMs) the default is two boards per CTA."""
    kn = nets(kind)
    for n, rows in ((5, ("32", "64", "128")), (64, ("32", "64", "128")), (140, ("64", "128"))):
        nh.check_tower_shapes(kn, nh.inputs(kn.arch, n, 11), monkeypatch, rows, repeats=3)
