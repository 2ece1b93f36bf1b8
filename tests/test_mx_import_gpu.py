"""Networks imported from MXNet model files (crazyara_b200/mx_import.py, the symbol fixtures under tests/golden/) on the
GPU: the imported blob predicts bit for bit what the blob export_mx_blob writes for the same parameters does, in both
precisions, and drives a crazyhouse search as the oracle's search driven by the same network."""
import numpy as np
import pytest

from crazyara_b200.mx_import import import_mxnet
from crazyara_b200.weights import export_mx_blob
from oracle import search as osr
from oracle.chess import Position
from tests import net_harness as nh
from tests.mx_params_writer import write_params
from tests.test_mx_import import CASES, dump, network, symbol
from tests.test_search_gpu import _gpu_search, _net_fn
from tests.test_search_hostemu import assert_same_search


def _blobs(tmp_path, record):
    """-> (arch, the imported blob, export_mx_blob's blob)"""
    arch, params = network(record, 7)
    got = import_mxnet(dump(symbol(record), tmp_path / "m-symbol.json"), write_params(params, str(tmp_path / "m.params")),
                       str(tmp_path / "imported.arab"))
    ref = export_mx_blob(params, arch, str(tmp_path / "ref.arab"), input_version=CASES[record][2])
    return got, str(tmp_path / "imported.arab"), ref


@pytest.mark.gpu
@pytest.mark.parametrize("precision", ["float16", "float32"])
@pytest.mark.parametrize("record", sorted(CASES))
def test_imported_blob_predicts_as_the_parameter_blob(tmp_path, record, precision):
    from crazyara_b200.nn import NeuralNetAPI
    arch, imported, ref = _blobs(tmp_path, record)
    x = nh.inputs(arch, 8, 11)
    outs = []
    for blob in (imported, ref):
        net = NeuralNetAPI("gpu", 0, 8, blob, precision=precision)
        try:
            outs.append(nh.predict(net, arch, x))
        finally:
            net.close()
    assert np.isfinite(outs[0].value).all() and np.isfinite(outs[0].prob).all()
    assert nh.same_bits(*outs)


@pytest.mark.gpu
def test_imported_risev2_drives_a_crazyhouse_search(tmp_path):
    from crazyara_b200.nn import NeuralNetAPI
    _, imported, _ = _blobs(tmp_path, "mx_net_risev2_34")
    net = NeuralNetAPI("gpu", 0, 8, imported)
    try:
        st = osr.default_settings("crazyhouse", batch_size=8, simulations=200, node_policy_temperature=1.0, input_version=1)
        ro = osr.Search(st).run(Position(variant="crazyhouse"), _net_fn(net))
        rg = _gpu_search(1, None, False, [], st, net=net)[0]
    finally:
        net.close()
    assert_same_search(ro, rg)
