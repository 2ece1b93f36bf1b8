"""The weight import pinned byte for byte: every blob export_blob, export_mx_blob, import_checkpoint and import_onnx write
for the test networks, and the architecture each importer returns, against tests/golden/import_golden.json (written by
tests/golden/gen_import_golden.py); weights.read_blob as the inverse of write_blob; a RISE ONNX file read by its edges
whatever its node order and with the squeeze-excitation as torch.onnx.export writes it; and the graphs the import refuses."""
import json

import pytest

from crazyara_b200 import synthetic
from crazyara_b200.onnx_import import import_onnx, read_graph
from crazyara_b200.weights import export_blob, read_blob, write_blob
from oracle import net_alphavile as oav
from tests.golden import gen_import_golden as gen
from tests.onnx_alphavile_writer import write_alphavile_onnx
from tests.onnx_writer import _ld, _node, _tensor, _vi, write_rise_onnx


@pytest.fixture(scope="module")
def cases(tmp_path_factory):
    return gen.make_cases(str(tmp_path_factory.mktemp("import")))


def test_import_matches_the_golden(cases):
    with open(gen.PATH) as f:
        golden = json.load(f)
    got = gen.record(*cases)
    for part in ("onnx", "blobs", "archs"):
        assert sorted(got[part]) == sorted(golden[part]), part
        assert [k for k in golden[part] if got[part][k] != golden[part][k]] == [], part


def test_write_blob_inverts_read_blob(cases, tmp_path):
    for name, (path, _) in cases[0].items():
        again = write_blob(str(tmp_path / "again.arab"), *read_blob(path))
        assert open(again, "rb").read() == open(path, "rb").read(), name


@pytest.mark.parametrize("shuffle, torch_se", [(5, False), (None, True), (7, True)])
@pytest.mark.parametrize("name", sorted(gen.RISE))
def test_rise_onnx_is_read_by_its_edges(tmp_path, name, shuffle, torch_se):
    make, version = gen.RISE[name]
    arch = make()
    sd = synthetic.random_state_dict(arch, 3)
    ref = export_blob(sd, arch, str(tmp_path / "ref.arab"), input_version=version)
    path = write_rise_onnx(sd, arch, str(tmp_path / "m.onnx"), shuffle=shuffle, torch_se=torch_se)
    ops = [nd[0] for nd in read_graph(path)[0]]
    plain = [nd[0] for nd in read_graph(write_rise_onnx(sd, arch, str(tmp_path / "plain.onnx")))[0]]
    assert (ops != plain) if shuffle is not None else (ops.count("Conv") == plain.count("Conv"))
    assert ops.count("Expand") == (sum(1 for s in arch["se_types"] if s) if torch_se else 0)
    got = import_onnx(path, str(tmp_path / "onnx.arab"))
    assert got == import_onnx(str(tmp_path / "plain.onnx"), str(tmp_path / "plain.arab"))
    assert got["kernels"] == list(arch["kernels"]) and got["se_types"] == list(arch["se_types"])
    assert open(ref, "rb").read() == open(tmp_path / "onnx.arab", "rb").read()


# ------------------------------------------------------------------------------------------------- refusals
def _rewrite(path, edit):
    """the ONNX file at path with its (nodes, initialisers) changed by edit, written back (integer attributes only)"""
    nodes, inits = read_graph(path)
    nodes = edit(nodes, inits)
    graph = (b"".join(_ld(1, _node(op, ins, outs, sorted(attrs.items()))) for op, ins, outs, attrs in nodes) +
             b"".join(_ld(5, _tensor(k, a)) for k, a in inits.items()))
    with open(path, "wb") as f:
        f.write(_vi(1, 8) + _ld(7, graph))
    return path


def _rise_onnx(tmp_path, name):
    arch = gen.RISE[name][0]()
    return write_rise_onnx(synthetic.random_state_dict(arch, 3), arch, str(tmp_path / "m.onnx"))


def _alphavile_onnx(tmp_path, size, **change):
    arch = dict(gen.alphavile_arch(size), **change)
    return write_alphavile_onnx(oav.make_state_dict(arch, 4), arch, str(tmp_path / "m.onnx"))


def test_a_narrow_trunk_without_an_ntb_is_refused(tmp_path):
    arch = gen.alphavile_arch("tiny")
    path = _alphavile_onnx(tmp_path, "tiny", ntb=[False] * len(arch["kernels"]),
                           c_ops=[c or 2 * arch["channels"] for c in arch["c_ops"]])
    with pytest.raises(ValueError, match="192 trunk channels"):
        import_onnx(path, str(tmp_path / "x.arab"))


def test_ntbs_of_two_widths_are_refused(tmp_path):
    def narrower_second_mlp(nodes, inits):
        cat = [nd for nd in nodes if nd[0] == "Concat"][1]
        m1 = next(nd for nd in nodes if nd[0] == "Conv" and nd[1][0] == cat[2][0])
        relu = next(nd for nd in nodes if nd[0] == "Relu" and nd[1][0] == m1[2][0])
        m2 = next(nd for nd in nodes if nd[0] == "Conv" and nd[1][0] == relu[2][0])
        h = inits[m1[1][1]].shape[0] - 64
        inits[m1[1][1]], inits[m1[1][2]], inits[m2[1][1]] = inits[m1[1][1]][:h], inits[m1[1][2]][:h], inits[m2[1][1]][:, :h]
        return nodes
    path = _rewrite(_alphavile_onnx(tmp_path, "normal"), narrower_second_mlp)
    with pytest.raises(ValueError, match="different widths"):
        import_onnx(path, str(tmp_path / "x.arab"))


@pytest.mark.parametrize("net", ["risev2", "alphavile_tiny"])
def test_a_value_head_without_its_first_gemm_is_refused(tmp_path, net):
    path = _rise_onnx(tmp_path, net) if net in gen.RISE else _alphavile_onnx(tmp_path, "tiny")
    value_fc0 = lambda nd, inits: nd[0] == "Gemm" and inits[nd[1][1]].shape[1] == 8 * 64
    path = _rewrite(path, lambda nodes, inits: [nd for nd in nodes if not value_fc0(nd, inits)])
    with pytest.raises(ValueError, match="value head"):
        import_onnx(path, str(tmp_path / "x.arab"))


@pytest.mark.parametrize("name", sorted(gen.RISE))
def test_a_shortcut_from_before_the_squeeze_excitation_is_refused(tmp_path, name):
    """Every SE block's Add takes the block input instead of the Mul output: the MXNet semantics, which ARAB2001 cannot
    hold, in a file whose Conv / Gemm nodes are all in the right order."""
    def shortcut_before_se(nodes, inits):
        pre = {nd[2][0]: nd[1][0] for nd in nodes if nd[0] == "Mul"}
        return [(op, [pre.get(t, t) for t in ins] if op == "Add" else ins, outs, attrs) for op, ins, outs, attrs in nodes]
    path = _rewrite(_rise_onnx(tmp_path, name), shortcut_before_se)
    with pytest.raises(ValueError, match="squeeze-excitation"):
        import_onnx(path, str(tmp_path / "x.arab"))
