"""AlphaVile networks (ARAB2003 blobs: a 192 / 224 channel trunk padded to 256 at load, NextViT transformer blocks run as
GEMM launches around the attention kernel between tower segments) on the GPU.  Their comparison with the fp32 oracle
(oracle/net_alphavile.py) is in the table of tests/test_net_gpu.py."""
import pytest

from oracle import search as osr
from oracle.chess import Position
from tests import net_harness as nh
from tests.test_search_gpu import _gpu_search, _net_fn
from tests.test_search_hostemu import assert_same_search

KINDS = pytest.mark.parametrize("kind", ["av_normal", "av_tiny"], ids=["normal", "tiny"])


@pytest.fixture(scope="module")
def nets(tmp_path_factory):
    yield from nh.module_nets(tmp_path_factory)


@pytest.mark.gpu
@KINDS
def test_alphavile_tower_shapes_are_bit_identical(nets, monkeypatch, kind):
    """every tower segment"""
    for n in (1, 5, 64):
        nh.check_tower_shapes(nets(kind), nh.inputs(nets(kind).arch, n, 23), monkeypatch, repeats=2)


@pytest.mark.gpu
@KINDS
def test_alphavile_board_outputs_do_not_depend_on_its_row(nets, kind):
    """A board gives the same bits alone and at any row of a batch of 64 (the packed multi-tree batches rely on it)."""
    nh.check_rows_independent(nets(kind), 64, (0, 17, 63), seed=24, small=1)


@pytest.mark.gpu
def test_alphavile_two_thread_search_equals_oracle_search_driven_by_the_same_net(nets):
    net = nets("av_tiny").fresh(8)
    st = osr.default_settings("crazyhouse", batch_size=8, simulations=800, node_policy_temperature=1.0, input_version=1,
                              threads=2)
    pos = Position(variant="crazyhouse")
    ro = osr.Search(st).run(pos, _net_fn(net), threads=2)
    rg = _gpu_search(1, None, False, [], st, net=net)[0]
    assert_same_search(ro, rg)


@pytest.mark.gpu
def test_alphavile_packed_two_tree_search_equals_single_tree_searches(nets):
    """Two trees share each network batch (device-side row count): each comes out as when it is searched alone."""
    from crazyara_b200.engine import BoardState, MCTSAgent, SearchSettings
    B, lines = 8, [[], ["e2e4", "e7e5"]]
    net = nets("av_tiny").fresh(len(lines) * B)
    st = osr.default_settings("crazyhouse", batch_size=B, simulations=400, node_policy_temperature=1.0)
    s = SearchSettings()
    for f, _ in s._fields_:
        setattr(s, f, getattr(st, f))
    multi = MCTSAgent(net, s, 0, len(lines))
    for t, moves in enumerate(lines):
        multi.set_position(BoardState().set("", False, 1).do_uci(*moves), t)
    multi.evaluate_board_state()
    together = multi.results()
    multi.close()
    for t, moves in enumerate(lines):
        s.seed = (st.seed ^ (t * 0x9E3779B97F4A7C15)) & 0xFFFFFFFFFFFFFFFF
        alone = MCTSAgent(net, s, 0, 1)
        r = alone.evaluate_board_state(BoardState().set("", False, 1).do_uci(*moves))
        alone.close()
        assert_same_search(r, together[t])
        assert together[t]["evals"] > 0


@pytest.mark.gpu
@pytest.mark.parametrize("precision", ["float16", "float32"])
def test_alphavile_launch_bookkeeping_matches_the_launches(nets, precision):
    """per NTB 9 launches in float16 (10 in float32), one tower launch per segment"""
    nh.check_launch_count(nets("av_normal"), precision, n=4, seed=25)


@pytest.mark.gpu
def test_alphavile_packed_two_tree_search_equals_oracle_searches_driven_by_the_same_net(nets):
    """Two trees, Threads 2, Batch_Size 8, 800 simulations, sharing each network batch through the device-side row count:
    each tree equals the oracle search of its position driven by the same network."""
    from crazyara_b200.engine import BoardState, MCTSAgent, SearchSettings
    B, lines = 8, [[], ["e2e4", "e7e5"]]
    net = nets("av_tiny").fresh(len(lines) * B)
    st = osr.default_settings("crazyhouse", batch_size=B, simulations=800, node_policy_temperature=1.0, input_version=1,
                              threads=2)
    s = SearchSettings()
    for f, _ in s._fields_:
        setattr(s, f, getattr(st, f))
    multi = MCTSAgent(net, s, 0, len(lines))
    for t, moves in enumerate(lines):
        multi.set_position(BoardState().set("", False, 1).do_uci(*moves), t)
    multi.evaluate_board_state()
    together = multi.results()
    multi.close()
    for t, moves in enumerate(lines):
        pos = Position(variant="crazyhouse")
        pos.push_uci(*moves)
        ro = osr.Search(st).run(pos, _net_fn(net), threads=2)
        assert_same_search(ro, together[t])
        assert together[t]["evals"] > 0
