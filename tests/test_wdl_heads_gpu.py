"""Value heads with WDL and plies-to-end outputs that feed the value, on the device: the PyTorch trainer's value MLP
(use_mlp_wdl_ply, blob kind 2) and the MXNet symbols' head behind value_fc0 (kinds 3 and 4), against the oracles of
tests/wdl_heads.py in both precisions, bit-stable across rows and graph replays, with the launch count of the standard
head, and driving a search bit for bit like the oracle's search driven by the same network."""
import os
import subprocess

import numpy as np
import pytest

from crazyara_b200.weights import export_blob, export_mx_blob
from oracle import net_alphavile as oav
from oracle import net as onet
from oracle import net_mx
from oracle import search as osr
from oracle.chess import Position
from tests import classic_mx_head, net_harness, wdl_heads
from tests.net_harness import Kind
from tests.test_search_gpu import _gpu_search, _net_fn
from tests.test_search_hostemu import assert_same_search
from tests.test_wdl_heads import MALFORMED, malformed_blob

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MX_BASE = lambda: net_mx.arch_mx_risev33(52, 76)


def _torch(arch, version):
    return Kind(arch, lambda a: wdl_heads.mlp_state_dict(a, 7), export_blob, version, wdl_heads.forward_torch)


def _mx(arch, version):
    return Kind(arch, lambda a: wdl_heads.mx_params(a, 7), export_mx_blob, version, wdl_heads.forward_mx)


def _fc_mx(arch, n_labels, version):
    """ARAB2004 around ARAB2002: the head with the fully-connected policy head of tests/classic_mx_head.py"""
    return Kind(lambda: classic_mx_head.classic_arch(arch(), n_labels),
                lambda a: {**wdl_heads.mx_params(a, 7), **classic_mx_head.head_params(a, n_labels, 7)}, export_mx_blob,
                version, lambda p, a, x: wdl_heads.forward_mx(p, a, x, base=classic_mx_head.forward))


KINDS = {
    "risev33_mlp": _torch(lambda: dict(onet.arch_risev33(52, 76, True), value_head="wdl_mlp"), 30),
    "av_tiny_mlp": _torch(lambda: dict(oav.arch_alphavile("tiny", 34, 81, True), value_head="wdl_mlp"), 10),
    "mx_wdl": _mx(lambda: wdl_heads.mx_arch(MX_BASE(), "mx_wdl"), 30),
    "mx_wdl_mlp": _mx(lambda: wdl_heads.mx_arch(MX_BASE(), "mx_wdl_mlp"), 30),
    # a hidden layer narrower than 256 units (zero-padded on the device)
    "mx_wdl_mlp_96": _mx(lambda: wdl_heads.mx_arch(MX_BASE(), "mx_wdl_mlp", 96), 30),
    "fc_mx_wdl_mlp_1968": _fc_mx(lambda: wdl_heads.mx_arch(MX_BASE(), "mx_wdl_mlp"), 1968, 30),
}
F16_BATCHES, F32_BATCHES = (1, 5, 64, 66, 128), (1, 16)


class Nets(net_harness.Nets):
    """net_harness.Nets of one of this file's kinds"""

    def __init__(self, kind, tmp):
        k = KINDS[kind]
        self.arch = k.arch()
        self.weights, self.forward = k.weights(self.arch), k.forward
        self.blob = k.export(self.weights, self.arch, str(tmp / f"{kind}.arab"), input_version=k.version)
        self.nets, self.opened, self.refs = {}, [], {}


@pytest.fixture(scope="module")
def nets(tmp_path_factory):
    opened = {}

    def get(kind):
        if kind not in opened:
            opened[kind] = Nets(kind, tmp_path_factory.mktemp(kind))
        return opened[kind]
    yield get
    for n in opened.values():
        n.close()


@pytest.mark.gpu
@pytest.mark.parametrize("precision", ["float16", "float32"])
@pytest.mark.parametrize("kind", sorted(KINDS))
def test_forward_matches_the_oracle(nets, kind, precision):
    """value, policy and aux (PyTorch: WDL logits and plies; MXNet: WDL probabilities and plies) against the oracle at
    every batch size, and a second forward (a graph replay) with the same bits"""
    n = nets(kind)
    check = net_harness.check_float16 if precision == "float16" else net_harness.check_float32
    for b in F16_BATCHES if precision == "float16" else F32_BATCHES:
        x, ref = n.ref(b, 11)
        out = net_harness.predict(n.net(b, precision), n.arch, x)
        assert out.aux is not None
        check(out, ref)
        net_harness.check_replay_bits(n.net(b, precision), n.arch, x, out)


@pytest.mark.gpu
@pytest.mark.parametrize("precision", ["float16", "float32"])
@pytest.mark.parametrize("kind", ["risev33_mlp", "mx_wdl", "mx_wdl_mlp_96"])
def test_a_board_has_the_same_bits_at_any_row(nets, kind, precision):
    b = 64 if precision == "float16" else 16
    net_harness.check_rows_independent(nets(kind), b, (0, 5, b - 1), 12, precision=precision)


@pytest.mark.gpu
@pytest.mark.parametrize("precision", ["float16", "float32"])
@pytest.mark.parametrize("kind", sorted(KINDS))
def test_launch_count_is_the_standard_heads(nets, kind, precision):
    net_harness.check_launch_count(nets(kind), precision, 5, 13)


@pytest.mark.gpu
@pytest.mark.parametrize("case", sorted(MALFORMED))
def test_net_refuses_a_malformed_head(tmp_path, case):
    from crazyara_b200.nn import NeuralNetAPI
    path, reason = malformed_blob(tmp_path, case)
    with pytest.raises(Exception, match=reason):
        NeuralNetAPI("gpu", 0, 4, path)


@pytest.mark.gpu
@pytest.mark.parametrize("threads", [1, 2])
@pytest.mark.parametrize("precision", ["float16", "float32"])
@pytest.mark.parametrize("kind", ["risev33_mlp", "mx_wdl_mlp"])
def test_search_equals_the_oracle_driven_by_the_same_net(nets, kind, precision, threads):
    """chess v3: the oracle's search through ara_net_predict and the device search with the same network, bit for bit"""
    batch, sims = 16, 600
    net = nets(kind).fresh(batch, precision)
    st = osr.default_settings("chess", batch_size=batch, simulations=sims, node_policy_temperature=1.7, input_version=3,
                              threads=threads)
    pos = Position(None, "chess", False)
    pos.push_uci("e2e4", "c7c5")
    ro = osr.Search(st).run(pos, _net_fn(net), threads=threads)
    rg = _gpu_search(0, None, False, ["e2e4", "c7c5"], st, net=net)[0]
    assert_same_search(ro, rg)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["risev33_mlp", "mx_wdl"])
def test_uci_loads_the_blob_and_answers_go_nodes(nets, kind):
    script = ["uci", "setoption name UCI_Variant value chess", "setoption name Batch_Size value 16",
              f"setoption name Model_Path value {nets(kind).blob}", "isready", "position startpos moves e2e4",
              "go nodes 400", "quit"]
    out = subprocess.run([os.path.join(ROOT, "crazyara_b200", "ara_uci")], input="\n".join(script) + "\n",
                         capture_output=True, text=True, timeout=300)
    best = [line for line in out.stdout.splitlines() if line.startswith("bestmove")]
    assert len(best) == 1 and len(best[0].split()[1]) in (4, 5), out.stdout + out.stderr
