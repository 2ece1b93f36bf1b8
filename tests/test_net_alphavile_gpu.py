"""AlphaVile networks (ARAB2003 blobs: a 192 / 224 channel trunk padded to 256 at load, NextViT transformer blocks run as
GEMM launches around the attention kernel between tower segments) on the GPU against the fp32 oracle
(oracle/net_alphavile.py)."""
import numpy as np
import pytest

from oracle import net_alphavile as oav
from oracle import search as osr
from oracle.chess import Position
from tests.golden.gen_net_golden import golden_input
from tests.test_search_gpu import _gpu_search, _net_fn
from tests.test_search_hostemu import assert_same_search

VALUE_ATOL, LOGIT_ATOL, PROB_RTOL = 4e-3, 2.5e-2, 3e-2  # the float16 bounds of tests/test_net_gpu.py
F32_ATOL = 1e-4
ARCHS = {"tiny": lambda: oav.arch_alphavile("tiny", 34, 81, False), "normal": lambda: oav.arch_alphavile("normal", 52, 76, True)}


@pytest.fixture
def av_net(tmp_path):
    """-> make(name, batch, precision) = (NeuralNetAPI on an ARAB2003 blob, arch, state dict); closes them afterwards"""
    from crazyara_b200.nn import NeuralNetAPI
    from crazyara_b200.weights import export_blob
    nets = []

    def make(name, batch, precision="float16"):
        arch = ARCHS[name]()
        sd = oav.make_state_dict(arch, 7)
        blob = export_blob(sd, arch, str(tmp_path / f"{name}.arab"), input_version=10 if name == "tiny" else 30)
        nets.append(NeuralNetAPI("gpu", 0, batch, blob, precision=precision))
        return nets[-1], arch, sd
    yield make
    for n in nets:
        n.close()


def _predict(net, arch, x, batch, aux=None):
    """aux (optional): [n, 4] buffer for the WDL / plys outputs"""
    n, pch = x.shape[0], arch["policy_channels"]
    xin = np.zeros((batch, arch["in_channels"], 8, 8), np.float32)
    xin[:n] = x
    v, p = np.full(batch, np.nan, np.float32), np.full((batch, pch * 64), np.nan, np.float32)
    a = None if aux is None else np.full((batch, 4), np.nan, np.float32)
    net.predict(xin, v, p, a, n=n)
    if aux is not None:
        aux[:] = a[:n]
    return v[:n].copy(), p[:n].copy()


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(ARCHS))
@pytest.mark.parametrize("n", [1, 5, 64, 66, 128])
def test_alphavile_float16_matches_oracle(av_net, name, n):
    net, arch, sd = av_net(name, n)
    x = golden_input(arch, n=n, seed=21)
    v, p = _predict(net, arch, x, n)
    ref = oav.forward(sd, arch, x)
    assert np.isfinite(v).all() and np.isfinite(p).all()
    np.testing.assert_allclose(v, ref["value"], atol=VALUE_ATOL)
    lg = np.log(p) - np.log(p).mean(1, keepdims=True)
    lr = ref["policy_logits"] - ref["policy_logits"].mean(1, keepdims=True)
    assert np.abs(lg - lr).max() < LOGIT_ATOL
    np.testing.assert_allclose(p, ref["prob"], rtol=PROB_RTOL, atol=1e-7)


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(ARCHS))
@pytest.mark.parametrize("n", [1, 16])
def test_alphavile_float32_within_1e4_of_oracle(av_net, name, n):
    net, arch, sd = av_net(name, n, "float32")
    x = golden_input(arch, n=n, seed=22)
    aux = np.full((n, 4), np.nan, np.float32)
    v, p = _predict(net, arch, x, n, aux if arch["wdl"] else None)
    ref = oav.forward(sd, arch, x)
    np.testing.assert_allclose(v, ref["value"], atol=F32_ATOL, rtol=0)
    np.testing.assert_allclose(p, ref["prob"], atol=F32_ATOL, rtol=0)
    np.testing.assert_allclose(p, ref["prob"], rtol=2e-3, atol=1e-8)  # and small probabilities relatively
    lg = np.log(p) - np.log(p).mean(1, keepdims=True)
    lr = ref["policy_logits"] - ref["policy_logits"].mean(1, keepdims=True)
    assert np.abs(lg - lr).max() < 1e-3
    if arch["wdl"]:
        np.testing.assert_allclose(aux, ref["aux"], atol=F32_ATOL, rtol=0)


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(ARCHS))
def test_alphavile_tower_shapes_are_bit_identical(av_net, monkeypatch, name):
    """ARA_TRUNK_ROWS 32 (the CTA pair), 64 (one board per CTA) and 128 (two boards per CTA) give the same bits for every
    tower segment."""
    for n in (1, 5, 64):
        arch = ARCHS[name]()
        x = golden_input(arch, n=n, seed=23)
        outs = {}
        for rows in ("32", "64", "128"):
            monkeypatch.setenv("ARA_TRUNK_ROWS", rows)
            net, arch, _ = av_net(name, n)
            outs[rows] = [_predict(net, arch, x, n) for _ in range(2)]
        ref_v, ref_p = outs["64"][0]
        for rows, runs in outs.items():
            for v, p in runs:
                assert np.array_equal(v, ref_v) and np.array_equal(p, ref_p), f"n={n}: ARA_TRUNK_ROWS={rows} differs"


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(ARCHS))
def test_alphavile_board_outputs_do_not_depend_on_its_row(av_net, name):
    """A board gives the same bits alone and at any row of a batch of 64 (the packed multi-tree batches rely on it)."""
    net1, arch, _ = av_net(name, 1)
    net64, _, _ = av_net(name, 64)
    xs = golden_input(arch, n=64, seed=24)
    for row in (0, 17, 63):
        v1, p1 = _predict(net1, arch, xs[row:row + 1], 1)
        v, p = _predict(net64, arch, xs, 64)
        assert np.array_equal(v[row:row + 1], v1) and np.array_equal(p[row:row + 1], p1), f"row {row}"


@pytest.mark.gpu
def test_alphavile_two_thread_search_equals_oracle_search_driven_by_the_same_net(av_net):
    net, arch, _ = av_net("tiny", 8)
    st = osr.default_settings("crazyhouse", batch_size=8, simulations=800, node_policy_temperature=1.0, input_version=1,
                              threads=2)
    pos = Position(variant="crazyhouse")
    ro = osr.Search(st).run(pos, _net_fn(net), threads=2)
    rg = _gpu_search(1, None, False, [], st, net=net)[0]
    assert_same_search(ro, rg)


@pytest.mark.gpu
def test_alphavile_packed_two_tree_search_equals_single_tree_searches(av_net):
    """Two trees share each network batch (device-side row count): each comes out as when it is searched alone."""
    from crazyara_b200.engine import BoardState, MCTSAgent, SearchSettings
    B, lines = 8, [[], ["e2e4", "e7e5"]]
    net, arch, _ = av_net("tiny", len(lines) * B)
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
def test_alphavile_launch_bookkeeping_matches_the_launches(av_net, precision):
    """The first forward of a size runs eagerly (every launch counted) before it is captured; a graph replay then adds
    the launches its capture enqueued.  Both must agree with the layer plan: per NTB 9 launches in float16 (10 in
    float32), one tower launch per segment."""
    net, arch, _ = av_net("normal", 4, precision)
    x = golden_input(arch, n=4, seed=25)
    _predict(net, arch, x, 4)
    first = net.launch_count()
    _predict(net, arch, x, 4)
    per_forward = net.launch_count() - first
    assert first == 2 * per_forward
    segments = 1 + sum(1 for i, t in enumerate(arch["ntb"][:-1]) if t and not arch["ntb"][i + 1])
    n_ntb, n_plain = sum(arch["ntb"]), len(arch["ntb"]) - sum(arch["ntb"])
    expect = 1 + 1 + 4 + (segments + 9 * n_ntb if precision == "float16" else 3 * n_plain + 10 * n_ntb)
    assert per_forward == expect


@pytest.mark.gpu
def test_alphavile_packed_two_tree_search_equals_oracle_searches_driven_by_the_same_net(av_net):
    """Two trees, Threads 2, Batch_Size 8, 800 simulations, sharing each network batch through the device-side row count:
    each tree equals the oracle search of its position driven by the same network."""
    from crazyara_b200.engine import BoardState, MCTSAgent, SearchSettings
    B, lines = 8, [[], ["e2e4", "e7e5"]]
    net, arch, _ = av_net("tiny", len(lines) * B)
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
