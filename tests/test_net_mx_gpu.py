"""Networks of the reference's MXNet symbols (ARAB2002 blobs, crazyara_b200.weights.export_mx_blob) on the GPU against the
fp32 oracle of those symbols (oracle/net_mx.py): the squeeze-excitation scales only the input of the block's first
convolution, its shortcut adds the unscaled input; ca_se with biases and sigmoid or clamp(0.2 x + 0.5) gates; eca_se as a
1-D convolution over the channels; the v3 stem without activation and the v3 policy convolution with a bias."""
import numpy as np
import pytest

from oracle import net_mx
from oracle import search as osr
from oracle.chess import Position
from tests.golden.gen_net_golden import golden_input
from tests.test_search_gpu import _gpu_search, _net_fn
from tests.test_search_hostemu import assert_same_search

VALUE_ATOL, LOGIT_ATOL, PROB_RTOL = 4e-3, 2.5e-2, 3e-2  # the float16 bounds of tests/test_net_gpu.py
F32_ATOL = 1e-4

# every SE flavour of the symbols side by side: ca_se with a sigmoid (RISEv2: ratio 2, hidden 128) or a hard sigmoid
# gate (rise_mobile_v3: ratio 16, hidden 16, zero-padded to 128), eca_se, plain blocks, one-chunk blocks (c_op <= 64),
# 3x3 and 5x5 depthwise kernels
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


ARCHS = {"mx_risev2": lambda: net_mx.arch_mx_risev2(34, 81), "mx_risev33": lambda: net_mx.arch_mx_risev33(52, 76),
         "mx_mixed": mixed_arch}
VERSION = {"mx_risev2": 10, "mx_risev33": 30, "mx_mixed": 30}


@pytest.fixture
def mx_net(tmp_path):
    """-> make(name, batch, precision) = (NeuralNetAPI on an ARAB2002 blob, arch, params); closes them afterwards"""
    from crazyara_b200.nn import NeuralNetAPI
    from crazyara_b200.weights import export_mx_blob
    nets = []

    def make(name, batch, precision="float16"):
        arch = ARCHS[name]()
        params = net_mx.make_mx_params(arch, 7)
        blob = export_mx_blob(params, arch, str(tmp_path / f"{name}.arab"), input_version=VERSION[name])
        nets.append(NeuralNetAPI("gpu", 0, batch, blob, precision=precision))
        return nets[-1], arch, params
    yield make
    for n in nets:
        n.close()


def _predict(net, arch, x, batch):
    n, pch = x.shape[0], arch["policy_channels"]
    xin = np.zeros((batch, arch["in_channels"], 8, 8), np.float32)
    xin[:n] = x
    v, p = np.full(batch, np.nan, np.float32), np.full((batch, pch * 64), np.nan, np.float32)
    net.predict(xin, v, p, None, n=n)
    return v[:n].copy(), p[:n].copy()


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(ARCHS))
@pytest.mark.parametrize("n", [1, 5, 64, 66, 128])
def test_mx_net_float16_matches_oracle(mx_net, name, n):
    net, arch, params = mx_net(name, n)
    x = golden_input(arch, n=n, seed=21)
    v, p = _predict(net, arch, x, n)
    ref = net_mx.forward_mx(params, arch, x)
    assert np.isfinite(v).all() and np.isfinite(p).all()
    np.testing.assert_allclose(v, ref["value"], atol=VALUE_ATOL)
    lg = np.log(p) - np.log(p).mean(1, keepdims=True)
    lr = ref["policy_logits"] - ref["policy_logits"].mean(1, keepdims=True)
    assert np.abs(lg - lr).max() < LOGIT_ATOL
    np.testing.assert_allclose(p, ref["prob"], rtol=PROB_RTOL, atol=1e-7)


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(ARCHS))
@pytest.mark.parametrize("n", [1, 16])
def test_mx_net_float32_within_1e4_of_oracle(mx_net, name, n):
    net, arch, params = mx_net(name, n, "float32")
    x = golden_input(arch, n=n, seed=22)
    v, p = _predict(net, arch, x, n)
    ref = net_mx.forward_mx(params, arch, x)
    np.testing.assert_allclose(v, ref["value"], atol=F32_ATOL, rtol=0)
    np.testing.assert_allclose(p, ref["prob"], atol=F32_ATOL, rtol=0)


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(ARCHS))
def test_mx_tower_shapes_are_bit_identical(mx_net, monkeypatch, name):
    """ARA_TRUNK_ROWS 32 (the CTA pair), 64 (one board per CTA) and 128 (two boards per CTA) give the same bits, as for
    the PyTorch semantics (tests/test_trunk_pair_gpu.py)."""
    for n in (1, 5, 64):
        arch = ARCHS[name]()
        x = golden_input(arch, n=n, seed=23)
        outs = {}
        for rows in ("32", "64", "128"):
            monkeypatch.setenv("ARA_TRUNK_ROWS", rows)
            net, arch, _ = mx_net(name, n)
            outs[rows] = [_predict(net, arch, x, n) for _ in range(2)]
        ref_v, ref_p = outs["64"][0]
        for rows, runs in outs.items():
            for v, p in runs:
                assert np.array_equal(v, ref_v) and np.array_equal(p, ref_p), f"n={n}: ARA_TRUNK_ROWS={rows} differs"


@pytest.mark.gpu
def test_mx_net_search_equals_oracle_search_driven_by_the_same_net(mx_net):
    net, arch, _ = mx_net("mx_risev2", 8)
    st = osr.default_settings("crazyhouse", batch_size=8, simulations=800, node_policy_temperature=1.0, input_version=1)
    pos = Position(variant="crazyhouse")
    ro = osr.Search(st).run(pos, _net_fn(net))
    rg = _gpu_search(1, None, False, [], st, net=net)[0]
    assert_same_search(ro, rg)
