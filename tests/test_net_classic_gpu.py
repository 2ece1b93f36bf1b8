"""Networks with a fully-connected policy head (ARAB2004, the trainer's select_policy_from_plane=False) on the GPU: the
wgmma split-K layer of policy_fc.cuh and its softmax, in both precisions.  Their comparison with the fp32 oracle
(tests/classic_head.py on oracle/net.py and oracle/net_alphavile.py) is in the table of tests/test_net_gpu.py."""
import numpy as np
import pytest

from crazyara_b200 import synthetic
from tests import net_harness as nh
from tests.golden.gen_net_golden import golden_input

KIND = "fc_risev2_81_2272"


@pytest.fixture(scope="module")
def nets(tmp_path_factory):
    yield from nh.module_nets(tmp_path_factory)


@pytest.mark.gpu
@pytest.mark.parametrize("precision", ["float16", "float32"])
def test_classic_priors_are_the_gathered_probabilities(nets, precision):
    """predict_priors (ara_net_predict_priors) gathers classic label indices from the same forward predict runs"""
    net, arch = nets(KIND).net(8, precision), nets(KIND).arch
    x = golden_input(arch, n=6, seed=13)
    prob = nh.predict(net, arch, x).prob
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
def test_classic_output_of_a_position_does_not_depend_on_its_batch(nets, precision):
    """A board's value / policy bits at a row of a batch of 3 equal its bits at its row of a batch of 128 (the head's
    board tile is 32 boards wide in one, 128 in the other; the split-K partial sums add up in the same order)"""
    nh.check_rows_independent(nets(KIND), 128, (0, 37, 100, 127), seed=9, precision=precision)


@pytest.mark.gpu
@pytest.mark.parametrize("precision", ["float16", "float32"])
def test_classic_launch_bookkeeping_matches_the_launches(nets, precision):
    """as tests/test_net_gpu.py counts them, with the fully-connected layer and its softmax in place of the softmax"""
    nh.check_launch_count(nets("fc_risev33_76_1968"), precision, n=4, seed=25)


@pytest.mark.gpu
def test_search_refuses_a_classic_net_by_name(nets):
    """the device search parks policy-map indices; a fully-connected head's network is refused with that reason"""
    from crazyara_b200 import AraError
    from crazyara_b200.engine import MCTSAgent, default_settings
    with pytest.raises(AraError, match="fully-connected policy head"):
        MCTSAgent(nets(KIND).net(8), default_settings("crazyhouse", batch_size=8, simulations=64), 0, 1)


@pytest.mark.gpu
def test_raw_net_agent_refuses_a_classic_net_by_name(nets):
    """RawNetAgent gathers the legal moves' policy-map indices: it must not read a classic head's probabilities with them"""
    from crazyara_b200 import AraError
    from crazyara_b200.engine import RawNetAgent
    with pytest.raises(AraError, match="fully-connected policy head"):
        RawNetAgent(nets(KIND).net(8), "crazyhouse", 10)


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
