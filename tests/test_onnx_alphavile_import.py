"""ONNX import of AlphaVile networks (crazyara_b200/onnx_import.py) against the checkpoint import: the same network written
as an ONNX file by tests/onnx_alphavile_writer.py must give the same ARAB2003 blob, byte for byte.  (Parity unpinned: see
the writer's header.)"""
import pytest

from crazyara_b200.onnx_import import import_onnx
from crazyara_b200.weights import export_blob
from oracle import net_alphavile as oav
from tests.onnx_alphavile_writer import write_alphavile_onnx


@pytest.mark.parametrize("size", oav.SIZES)
def test_onnx_import_equals_checkpoint_import(tmp_path, size):
    arch = oav.arch_alphavile(size, 34, 81, False) if size in ("tiny", "small") else oav.arch_alphavile(size, 52, 76, True)
    sd = oav.make_state_dict(arch, 4)
    version = 10 if size in ("tiny", "small") else 30
    ref = export_blob(sd, arch, str(tmp_path / "ref.arab"), input_version=version)
    got = import_onnx(write_alphavile_onnx(sd, arch, str(tmp_path / "m.onnx")), str(tmp_path / "onnx.arab"))
    assert got["ntb"] == arch["ntb"] and got["channels"] == arch["channels"] and got["wdl"] == arch["wdl"]
    assert open(ref, "rb").read() == open(tmp_path / "onnx.arab", "rb").read()


def test_onnx_import_rejects_a_wrong_attention_scale(tmp_path):
    arch = oav.arch_alphavile("tiny", 34, 81, False)
    path = write_alphavile_onnx(oav.make_state_dict(arch, 4), arch, str(tmp_path / "m.onnx"), scale=0.125)
    with pytest.raises(ValueError, match="attention scale"):
        import_onnx(path, str(tmp_path / "x.arab"))


@pytest.mark.parametrize("name", ["risev2", "risev33"])
def test_rise_graph_with_a_shape_concat_still_imports_as_rise(tmp_path, name):
    """The shape-only Concat a dynamic-batch RISE export carries in front of a view() is not an NTB: the import stays
    byte-identical to the state-dict import."""
    from crazyara_b200 import synthetic
    from tests.onnx_writer import add_shape_concat, write_rise_onnx
    arch = synthetic.risev2(34, 81) if name == "risev2" else synthetic.risev33(52, 76)
    sd = synthetic.random_state_dict(arch, 3)
    ref = export_blob(sd, arch, str(tmp_path / "ref.arab"), input_version=10 if name == "risev2" else 30)
    path = add_shape_concat(write_rise_onnx(sd, arch, str(tmp_path / "m.onnx")))
    got = import_onnx(path, str(tmp_path / "onnx.arab"))
    assert got["kernels"] == list(arch["kernels"]) and "ntb" not in got
    assert open(ref, "rb").read() == open(tmp_path / "onnx.arab", "rb").read()
