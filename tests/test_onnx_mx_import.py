"""ONNX import of networks exported from the reference's MXNet symbols (crazyara_b200/onnx_import.py) against the
parameter conversion (crazyara_b200/weights.py, export_mx_blob): the same network written by tests/onnx_mx_writer.py
must give the same ARAB2002 blob, byte for byte.  PARITY UNPINNED: neither tree holds an MXNet export to read."""
import numpy as np
import pytest

from crazyara_b200.onnx_import import import_onnx
from crazyara_b200.weights import export_mx_blob
from oracle import net_mx
from tests.onnx_mx_writer import write_mx_onnx
from tests.test_net_mx_gpu import mixed_arch

ARCHS = {"mx_risev2": lambda: net_mx.arch_mx_risev2(34, 81), "mx_risev33": lambda: net_mx.arch_mx_risev33(52, 76),
         "mx_mixed": mixed_arch}


@pytest.mark.parametrize("name", sorted(ARCHS))
def test_onnx_mx_import_equals_param_conversion(tmp_path, name):
    arch = ARCHS[name]()
    params = net_mx.make_mx_params(arch, 4)
    # (an ONNX attribute holds the BatchNorm epsilon as a float32)
    ref = export_mx_blob(params, arch, str(tmp_path / "ref.arab"), input_version=30, eps=float(np.float32(1e-3)))
    onnx_path = write_mx_onnx(params, arch, str(tmp_path / "model.onnx"), seed=len(name))
    got = import_onnx(onnx_path, str(tmp_path / "onnx.arab"), input_version=30)
    for key in ("kernels", "c_ops", "se_types", "stem_act", "policy_bias", "in_channels", "policy_channels"):
        assert got[key] == arch[key], key
    assert [g for g, s in zip(got["se_gates"], got["se_types"]) if s] == [g for g, s in zip(arch["se_gates"], arch["se_types"]) if s]
    assert open(ref, "rb").read() == open(tmp_path / "onnx.arab", "rb").read()


def test_onnx_mx_import_honours_the_batchnorm_epsilon(tmp_path):
    arch = net_mx.arch_mx_risev2(34, 81)
    params = net_mx.make_mx_params(arch, 4)
    import_onnx(write_mx_onnx(params, arch, str(tmp_path / "a.onnx"), eps=2e-5), str(tmp_path / "a.arab"))
    ref = export_mx_blob(params, arch, str(tmp_path / "ref.arab"), input_version=10, eps=float(np.float32(2e-5)))
    assert open(ref, "rb").read() == open(tmp_path / "a.arab", "rb").read()
