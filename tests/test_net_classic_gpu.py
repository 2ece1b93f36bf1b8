"""Networks with a fully-connected policy head (ARAB2004, the trainer's select_policy_from_plane=False) on the GPU
against the fp32 oracle (tests/classic_head.py on oracle/net.py and oracle/net_alphavile.py): the wgmma split-K layer
of policy_fc.cuh and its softmax, in both precisions, within the bounds tests/test_net_gpu.py holds the policy-map head
to."""
import numpy as np
import pytest

from crazyara_b200 import synthetic
from oracle import net as onet
from oracle import net_alphavile as oav
from tests import classic_head
from tests.golden.gen_net_golden import golden_input

VALUE_ATOL, LOGIT_ATOL, PROB_RTOL = 4e-3, 2.5e-2, 3e-2  # the float16 bounds of tests/test_net_gpu.py
F32_ATOL = 1e-4


def _arch(name, pch, n_labels):
    base = {"risev2": lambda: onet.arch_risev2(34, pch), "risev33": lambda: onet.arch_risev33(52, pch, True),
            "alphavile": lambda: oav.arch_alphavile("tiny", 34, pch, False)}[name]()
    return synthetic.classic(base, n_labels)


@pytest.fixture
def classic_net(tmp_path):
    """-> make(name, P, L, batch, precision) = (NeuralNetAPI on an ARAB2004 blob, arch, state dict, oracle forward)"""
    from crazyara_b200.nn import NeuralNetAPI
    from crazyara_b200.weights import export_blob
    nets = []

    def make(name, pch, n_labels, batch, precision="float16"):
        arch = _arch(name, pch, n_labels)
        om = oav if name == "alphavile" else onet
        sd = om.make_state_dict(arch, 0)
        sd.update(synthetic.classic_head(arch, n_labels, 0))
        blob = export_blob(sd, arch, str(tmp_path / f"{arch['name']}.arab"), input_version=30 if name == "risev33" else 10)
        nets.append(NeuralNetAPI("gpu", 0, batch, blob, precision=precision))
        return nets[-1], arch, sd, om.forward
    yield make
    for n in nets:
        n.close()


def _predict(net, arch, x, batch):
    n = x.shape[0]
    xin = np.zeros((batch, arch["in_channels"], 8, 8), np.float32)
    xin[:n] = x
    value = np.full(batch, np.nan, np.float32)
    prob = np.full((batch, arch["n_labels"]), np.nan, np.float32)
    aux = np.full((batch, 4), np.nan, np.float32)
    net.predict(xin, value, prob, aux if arch["wdl"] else None, n=n)
    return value[:n], prob[:n], aux[:n]


# (family, P, L, batch, n): every label count, P from 2 to 81, batches from 1 to 128 (66: a partial last board tile)
CASES = [("risev2", 81, 2272, 1, 1), ("risev2", 81, 2272, 8, 5), ("risev2", 81, 2272, 64, 64), ("risev2", 81, 2272, 66, 66),
         ("risev2", 81, 2272, 128, 128), ("risev33", 76, 1968, 8, 8), ("risev2", 2, 2316, 8, 8), ("risev2", 16, 1968, 64, 64),
         ("alphavile", 81, 2316, 8, 8)]


@pytest.mark.gpu
@pytest.mark.parametrize("precision", ["float16", "float32"])
@pytest.mark.parametrize("name,pch,n_labels,batch,n", CASES)
def test_classic_head_forward_matches_oracle(classic_net, name, pch, n_labels, batch, n, precision):
    net, arch, sd, forward = classic_net(name, pch, n_labels, batch, precision)
    assert not net.is_policy_map() and net.get_nb_policy_values() == n_labels
    x = golden_input(arch, n=n, seed=5)
    value, prob, aux = _predict(net, arch, x, batch)
    ref = classic_head.forward(forward, sd, arch, x)
    assert np.isfinite(value).all() and np.isfinite(prob).all()
    logit_gpu = np.log(prob) - np.log(prob).mean(1, keepdims=True)
    logit_ref = ref["policy_logits"] - ref["policy_logits"].mean(1, keepdims=True)
    if precision == "float16":
        np.testing.assert_allclose(prob.sum(1), 1.0, atol=1e-4)
        np.testing.assert_allclose(value, ref["value"], atol=VALUE_ATOL)
        assert np.abs(logit_gpu - logit_ref).max() < LOGIT_ATOL
        np.testing.assert_allclose(prob, ref["prob"], rtol=PROB_RTOL, atol=1e-7)
    else:
        np.testing.assert_allclose(value, ref["value"], atol=F32_ATOL, rtol=0)
        np.testing.assert_allclose(prob, ref["prob"], atol=F32_ATOL, rtol=0)
        np.testing.assert_allclose(prob, ref["prob"], rtol=2e-3, atol=1e-8)
        assert np.abs(logit_gpu - logit_ref).max() < 1e-3
        if arch["wdl"]:
            np.testing.assert_allclose(aux, ref["aux"], atol=F32_ATOL)
    # the replayed graph gives the same bits
    value2, prob2, _ = _predict(net, arch, x, batch)
    assert np.array_equal(value2, value) and np.array_equal(prob2, prob)


@pytest.mark.gpu
@pytest.mark.parametrize("precision", ["float16", "float32"])
def test_classic_priors_are_the_gathered_probabilities(classic_net, precision):
    """predict_priors (ara_net_predict_priors) gathers classic label indices from the same forward predict runs"""
    net, arch, _, _ = classic_net("risev2", 81, 2272, 8, precision)
    x = golden_input(arch, n=6, seed=13)
    _, prob, _ = _predict(net, arch, x, 8)
    rng = np.random.default_rng(1)
    stride = 40
    idx = rng.integers(0, 2272, (8, stride)).astype(np.int32)
    counts = np.array([40, 1, 17, 0, 33, 40, 0, 0], np.int32)
    xin = np.zeros((8, 34, 8, 8), np.float32)
    xin[:6] = x
    v, pri = np.zeros(8, np.float32), np.zeros((8, stride), np.float32)
    net.predict_priors(xin, idx, counts, v, pri, n=6)
    for b in range(6):
        assert np.array_equal(pri[b, :counts[b]], prob[b, idx[b, :counts[b]]])


@pytest.mark.gpu
@pytest.mark.parametrize("precision", ["float16", "float32"])
def test_classic_output_of_a_position_does_not_depend_on_its_batch(classic_net, precision):
    """A board's value / policy bits at a row of a batch of 3 equal its bits at its row of a batch of 128 (the head's
    board tile is 32 boards wide in one, 128 in the other; the split-K partial sums add up in the same order)"""
    net128, arch, _, _ = classic_net("risev2", 81, 2272, 128, precision)
    x = golden_input(arch, n=128, seed=9)
    v128, p128, _ = _predict(net128, arch, x, 128)
    net3, _, _, _ = classic_net("risev2", 81, 2272, 3, precision)
    for src in (0, 37, 100, 127):
        xin = np.stack([x[(src + 5) % 128], x[src]])
        v, p, _ = _predict(net3, arch, xin, 3)
        assert v[1] == v128[src] and np.array_equal(p[1], p128[src]), (precision, src)


@pytest.mark.gpu
@pytest.mark.parametrize("precision", ["float16", "float32"])
def test_classic_launch_bookkeeping_matches_the_launches(classic_net, precision):
    """as tests/test_net_gpu.py counts them, with the fully-connected layer and its softmax in place of the softmax"""
    net, arch, _, _ = classic_net("risev33", 76, 1968, 4, precision)
    x = golden_input(arch, n=4, seed=25)
    _predict(net, arch, x, 4)
    first = net.launch_count()
    _predict(net, arch, x, 4)
    per_forward = net.launch_count() - first
    assert first == 2 * per_forward
    tower = 1 if precision == "float16" else sum(3 + (se is not None) for se in arch["se_types"])
    assert per_forward == 1 + 1 + tower + 5


@pytest.mark.gpu
def test_search_refuses_a_classic_net_by_name(classic_net):
    """the device search parks policy-map indices; a fully-connected head's network is refused with that reason"""
    from crazyara_b200 import AraError
    from crazyara_b200.engine import MCTSAgent, default_settings
    net, _, _, _ = classic_net("risev2", 81, 2272, 8)
    with pytest.raises(AraError, match="fully-connected policy head"):
        MCTSAgent(net, default_settings("crazyhouse", batch_size=8, simulations=64), 0, 1)


@pytest.mark.gpu
def test_raw_net_agent_refuses_a_classic_net_by_name(classic_net):
    """RawNetAgent gathers the legal moves' policy-map indices: it must not read a classic head's probabilities with them"""
    from crazyara_b200 import AraError
    from crazyara_b200.engine import RawNetAgent
    net, _, _, _ = classic_net("risev2", 81, 2272, 8)
    with pytest.raises(AraError, match="fully-connected policy head"):
        RawNetAgent(net, "crazyhouse", 10)


@pytest.mark.gpu
def test_uci_refuses_a_classic_net_for_search_and_raw_network(tmp_path):
    """ara_uci with an ARAB2004 blob names the reason instead of answering, with and without Use_Raw_Network (`go` sets the
    search up first, so its refusal is the one reported)"""
    import os
    import subprocess
    from crazyara_b200.weights import export_blob
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    exe = os.path.join(root, "crazyara_b200", "ara_uci")
    arch = synthetic.classic(synthetic.risev2(34, 81), 2272)
    blob = export_blob(synthetic.random_state_dict(arch, 0), arch, str(tmp_path / "fc.arab"), input_version=10)
    head = ["uci", "setoption name UCI_Variant value crazyhouse", "setoption name Batch_Size value 8",
            f"setoption name Model_Path value {blob}"]
    out = subprocess.run([exe], input="\n".join(head + ["isready", "quit"]) + "\n", capture_output=True, text=True,
                         timeout=120).stdout
    assert "fully-connected policy head" in out
    script = head + ["setoption name Use_Raw_Network value true", "isready", "position startpos", "go", "quit"]
    out = subprocess.run([exe], input="\n".join(script) + "\n", capture_output=True, text=True, timeout=120).stdout
    errors = [l for l in out.splitlines() if l.startswith("info string error:")]
    assert errors and all("fully-connected policy head" in l for l in errors), out
    assert "bestmove" not in out
