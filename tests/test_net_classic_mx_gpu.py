"""Networks of the reference's MXNet symbols with a fully-connected policy head (ARAB2004 around ARAB2002, the symbols'
select_policy_from_plane=False) on the GPU against the fp32 oracle of those symbols with the head
(tests/classic_mx_head.py on oracle/net_mx.py): the MXNet trunk semantics of tests/test_net_mx_gpu.py in front of the
classic head of tests/test_net_classic_gpu.py, in both precisions and within the same bounds."""
import numpy as np
import pytest

from oracle import net_mx
from tests import classic_mx_head
from tests.golden.gen_net_golden import golden_input

VALUE_ATOL, LOGIT_ATOL, PROB_RTOL = 4e-3, 2.5e-2, 3e-2  # the float16 bounds of tests/test_net_gpu.py
F32_ATOL = 1e-4

# name: (base arch, L, input version): RISEv2 with sigmoid ca_se, a stem ReLU and no policy bias; RISEv3.3 with eca_se,
# clamp(0.2 x + 0.5) gates, no stem activation and a policy convolution bias (folded into the head with policy_bn1)
ARCHS = {"mx_risev2_2272": (lambda: net_mx.arch_mx_risev2(34, 81), 2272, 10),
         "mx_risev33_1968": (lambda: net_mx.arch_mx_risev33(52, 76), 1968, 30)}


@pytest.fixture
def mx_classic_net(tmp_path):
    """-> make(name, batch, precision) = (NeuralNetAPI on an ARAB2004 blob of export_mx_blob, arch, params)"""
    from crazyara_b200.nn import NeuralNetAPI
    from crazyara_b200.weights import export_mx_blob
    nets = []

    def make(name, batch, precision="float16"):
        base, n_labels, version = ARCHS[name]
        arch, params = classic_mx_head.make_params(base(), n_labels, 7)
        blob = export_mx_blob(params, arch, str(tmp_path / f"{name}.arab"), input_version=version)
        assert open(blob, "rb").read(16)[8:] == np.array([2, n_labels], "<i4").tobytes()  # around ARAB2002
        nets.append(NeuralNetAPI("gpu", 0, batch, blob, precision=precision))
        return nets[-1], arch, params
    yield make
    for n in nets:
        n.close()


def _predict(net, arch, x, batch):
    n = x.shape[0]
    xin = np.zeros((batch, arch["in_channels"], 8, 8), np.float32)
    xin[:n] = x
    v, p = np.full(batch, np.nan, np.float32), np.full((batch, arch["n_labels"]), np.nan, np.float32)
    net.predict(xin, v, p, None, n=n)
    return v[:n].copy(), p[:n].copy()


# (name, batch, n): batches from 1 to 128, 66 a partial last board tile of the head
CASES = [("mx_risev2_2272", 1, 1), ("mx_risev2_2272", 8, 5), ("mx_risev2_2272", 66, 66), ("mx_risev2_2272", 128, 128),
         ("mx_risev33_1968", 1, 1), ("mx_risev33_1968", 16, 16), ("mx_risev33_1968", 128, 128)]


@pytest.mark.gpu
@pytest.mark.parametrize("precision", ["float16", "float32"])
@pytest.mark.parametrize("name,batch,n", CASES)
def test_mx_classic_forward_matches_oracle(mx_classic_net, name, batch, n, precision):
    net, arch, params = mx_classic_net(name, batch, precision)
    assert not net.is_policy_map() and net.get_nb_policy_values() == arch["n_labels"]
    x = golden_input(arch, n=n, seed=31)
    v, p = _predict(net, arch, x, batch)
    ref = classic_mx_head.forward(params, arch, x)
    assert np.isfinite(v).all() and np.isfinite(p).all()
    lg = np.log(p) - np.log(p).mean(1, keepdims=True)
    lr = ref["policy_logits"] - ref["policy_logits"].mean(1, keepdims=True)
    if precision == "float16":
        np.testing.assert_allclose(p.sum(1), 1.0, atol=1e-4)
        np.testing.assert_allclose(v, ref["value"], atol=VALUE_ATOL)
        assert np.abs(lg - lr).max() < LOGIT_ATOL
        np.testing.assert_allclose(p, ref["prob"], rtol=PROB_RTOL, atol=1e-7)
    else:
        np.testing.assert_allclose(v, ref["value"], atol=F32_ATOL, rtol=0)
        np.testing.assert_allclose(p, ref["prob"], atol=F32_ATOL, rtol=0)
        np.testing.assert_allclose(p, ref["prob"], rtol=2e-3, atol=1e-8)  # and small probabilities relatively
        assert np.abs(lg - lr).max() < 1e-3
    # the replayed graph gives the same bits
    v2, p2 = _predict(net, arch, x, batch)
    assert np.array_equal(v2, v) and np.array_equal(p2, p)


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(ARCHS))
def test_mx_classic_onnx_import_runs_as_the_parameter_blob(mx_classic_net, tmp_path, name):
    """the blob import_onnx writes for the same network's MXNet export gives the oracle's policy too"""
    from crazyara_b200.nn import NeuralNetAPI
    from crazyara_b200.onnx_import import import_onnx
    from tests.onnx_classic_writer import add_mx_head
    from tests.onnx_mx_writer import write_mx_onnx
    _, arch, params = mx_classic_net(name, 8)
    blob = str(tmp_path / "onnx.arab")
    import_onnx(add_mx_head(write_mx_onnx(params, arch, str(tmp_path / "m.onnx")), params), blob)
    net = NeuralNetAPI("gpu", 0, 8, blob)
    try:
        x = golden_input(arch, n=8, seed=32)
        v, p = _predict(net, arch, x, 8)
    finally:
        net.close()
    ref = classic_mx_head.forward(params, arch, x)
    np.testing.assert_allclose(v, ref["value"], atol=VALUE_ATOL)
    np.testing.assert_allclose(p, ref["prob"], rtol=PROB_RTOL, atol=1e-7)
