"""Networks of the reference's MXNet symbols (ARAB2002 blobs, crazyara_b200.weights.export_mx_blob) on the GPU: the
squeeze-excitation scales only the input of the block's first convolution, its shortcut adds the unscaled input; ca_se
with biases and sigmoid or clamp(0.2 x + 0.5) gates; eca_se as a 1-D convolution over the channels; the v3 stem without
activation and the v3 policy convolution with a bias.  Their comparison with the fp32 oracle of those symbols
(oracle/net_mx.py) is in the table of tests/test_net_gpu.py."""
import pytest

from oracle import search as osr
from oracle.chess import Position
from tests import net_harness as nh
from tests.test_search_gpu import _gpu_search, _net_fn
from tests.test_search_hostemu import assert_same_search


@pytest.fixture(scope="module")
def nets(tmp_path_factory):
    yield from nh.module_nets(tmp_path_factory)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["mx_mixed", "mx_risev2", "mx_risev33"])
def test_mx_tower_shapes_are_bit_identical(nets, monkeypatch, kind):
    """as for the PyTorch semantics (tests/test_trunk_pair_gpu.py)"""
    for n in (1, 5, 64):
        nh.check_tower_shapes(nets(kind), nh.inputs(nets(kind).arch, n, 23), monkeypatch, repeats=2)


@pytest.mark.gpu
def test_mx_net_search_equals_oracle_search_driven_by_the_same_net(nets):
    net = nets("mx_risev2").fresh(8)
    st = osr.default_settings("crazyhouse", batch_size=8, simulations=800, node_policy_temperature=1.0, input_version=1)
    pos = Position(variant="crazyhouse")
    ro = osr.Search(st).run(pos, _net_fn(net))
    rg = _gpu_search(1, None, False, [], st, net=net)[0]
    assert_same_search(ro, rg)
