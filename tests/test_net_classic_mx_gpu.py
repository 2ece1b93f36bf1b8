"""Networks of the reference's MXNet symbols with a fully-connected policy head (ARAB2004 around ARAB2002, the symbols'
select_policy_from_plane=False) on the GPU from the ONNX import: the blob import_onnx writes runs as the one
export_mx_blob writes.  The comparison of the latter with the fp32 oracle (tests/classic_mx_head.py on
oracle/net_mx.py) is in the table of tests/test_net_gpu.py."""
import numpy as np
import pytest

from tests import net_harness as nh


@pytest.fixture(scope="module")
def nets(tmp_path_factory):
    yield from nh.module_nets(tmp_path_factory)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["fc_mx_risev2_2272", "fc_mx_risev33_1968"], ids=["mx_risev2_2272", "mx_risev33_1968"])
def test_mx_classic_onnx_import_runs_as_the_parameter_blob(nets, tmp_path, kind):
    """the blob import_onnx writes for the same network's MXNet export gives the oracle's outputs too"""
    from crazyara_b200.nn import NeuralNetAPI
    from crazyara_b200.onnx_import import import_onnx
    from tests.onnx_classic_writer import add_mx_head
    from tests.onnx_mx_writer import write_mx_onnx
    kn = nets(kind)
    assert open(kn.blob, "rb").read(16)[8:] == np.array([2, kn.arch["n_labels"]], "<i4").tobytes()  # around ARAB2002
    blob = str(tmp_path / "onnx.arab")
    import_onnx(add_mx_head(write_mx_onnx(kn.weights, kn.arch, str(tmp_path / "m.onnx")), kn.weights), blob)
    net = NeuralNetAPI("gpu", 0, 8, blob)
    try:
        x, ref = kn.ref(8, 32)
        out = nh.predict(net, kn.arch, x)
    finally:
        net.close()
    nh.check_float16(out, ref)
