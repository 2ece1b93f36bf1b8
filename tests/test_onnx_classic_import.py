"""Fully-connected policy heads (the trainer's select_policy_from_plane=False) through the ONNX import and the MXNet
parameter conversion: the blob an ONNX export imports to is byte for byte the one the checkpoint or MXNet-parameter path
writes for the same network (ARAB2004 around ARAB2001 / 2002 / 2003); the MXNet head's oracle (tests/classic_mx_head.py)
and the head as the blob stores it are pinned to the reference's own symbols (tests/golden/classic_mx_net_*.json); and a
head the blob cannot hold is refused by name, never dropped."""
import json
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from crazyara_b200.onnx_import import import_onnx
from crazyara_b200.weights import export_blob, export_mx_blob, read_blob
from tests import classic_mx_head
from tests.golden import gen_classic_mx_net_golden as gen_mx
from tests.golden import gen_classic_net_golden as gen_torch
from tests.golden.gen_net_golden import golden_input
from tests.onnx_alphavile_writer import write_alphavile_onnx
from tests.onnx_classic_writer import add_mx_head, add_torch_head
from tests.onnx_mx_writer import write_mx_onnx
from tests.onnx_writer import write_rise_onnx

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
TORCH = {c[0]: c for c in gen_torch.CASES}
MX = {c[0]: c for c in gen_mx.CASES}


def _torch_case(name):
    _, family, cin, pch, wdl, n_labels = TORCH[name]
    arch, sd, _ = gen_torch.case_network(family, cin, pch, wdl, n_labels)
    return arch, sd, (write_alphavile_onnx if family == "alphavile" else write_rise_onnx)


def _bytes(path):
    return open(path, "rb").read()


@pytest.mark.parametrize("shuffle", [None, 11])
@pytest.mark.parametrize("layout", sorted(gen_mx.TORCH_LAYOUTS))
@pytest.mark.parametrize("name", sorted(TORCH))
def test_torch_export_imports_as_the_checkpoint_does(tmp_path, name, layout, shuffle):
    arch, sd, write = _torch_case(name)
    flatten, linear, trans_b = gen_mx.TORCH_LAYOUTS[layout]
    ref = export_blob(sd, arch, str(tmp_path / "ref.arab"), input_version=30 if arch["in_channels"] == 52 else 10)
    onnx = add_torch_head(write(sd, arch, str(tmp_path / "m.onnx")), sd, flatten, linear, trans_b, softmax=shuffle is None,
                          shuffle=shuffle)
    got = import_onnx(onnx, str(tmp_path / "onnx.arab"))
    assert got["n_labels"] == arch["n_labels"] and got["policy_channels"] == arch["policy_channels"]
    assert _bytes(ref) == _bytes(tmp_path / "onnx.arab")
    assert _bytes(ref)[:16] == b"ARAB2004" + np.array([3 if name.startswith("alphavile") else 1, arch["n_labels"]], "<i4").tobytes()


@pytest.mark.parametrize("name", sorted(MX))
def test_mx_export_imports_as_the_parameter_conversion_does(tmp_path, name):
    _, symbol, cin, pch, n_labels, version = MX[name]
    arch, params = gen_mx.case_network(symbol, cin, pch, n_labels)
    # (an ONNX attribute holds the BatchNorm epsilon as a float32)
    ref = export_mx_blob(params, arch, str(tmp_path / "ref.arab"), input_version=version, eps=float(np.float32(1e-3)))
    onnx = add_mx_head(write_mx_onnx(params, arch, str(tmp_path / "m.onnx"), seed=len(name)), params, seed=len(name))
    got = import_onnx(onnx, str(tmp_path / "onnx.arab"), input_version=version)
    for key in ("kernels", "c_ops", "se_types", "stem_act", "in_channels", "policy_channels", "n_labels"):
        assert got[key] == arch[key], key
    assert got["policy_bias"] is False
    assert _bytes(ref) == _bytes(tmp_path / "onnx.arab")
    assert _bytes(ref)[:16] == b"ARAB2004" + np.array([2, n_labels], "<i4").tobytes()


def test_classic_onnx_imports_match_the_hash_record(tmp_path):
    with open(gen_mx.IMPORT_PATH) as f:
        assert gen_mx.import_hashes(str(tmp_path)) == json.load(f)


# ---------------------------------------------------------------------------------------------- the MXNet head's oracle
def _record(name):
    with open(os.path.join(GOLDEN, f"classic_mx_net_{name}.json")) as f:
        return json.load(f)


def _assert_matches(g, value, logits):
    """within the tolerances tests/test_oracle_net_mx.py holds the policy-map oracle to"""
    idx = np.asarray(g["prob_idx"])
    prob = torch.softmax(torch.as_tensor(logits), dim=1).numpy()
    np.testing.assert_allclose(value, g["value"], atol=2e-6)
    np.testing.assert_allclose(prob[:, idx], g["prob"], rtol=1e-4, atol=1e-9)
    logp = np.log(prob)
    np.testing.assert_allclose((logp - logp.mean(1, keepdims=True))[:, idx], g["centred_log_prob"], atol=2e-5)
    assert prob.argmax(1).tolist() == g["argmax"]


@pytest.mark.parametrize("name", sorted(MX))
def test_mx_classic_oracle_matches_the_reference_symbol(name):
    _, symbol, cin, pch, n_labels, _ = MX[name]
    arch, params = gen_mx.case_network(symbol, cin, pch, n_labels)
    g = _record(name)
    assert g["n_labels"] == n_labels and g["param_names"] == sorted(params)
    out = classic_mx_head.forward(params, arch, golden_input(arch))
    assert out["policy_logits"].shape == (4, n_labels)
    _assert_matches(g, out["value"], out["policy_logits"])


@pytest.mark.parametrize("source", ["export_mx_blob", "import_onnx"])
@pytest.mark.parametrize("name", sorted(MX))
def test_mx_classic_blob_computes_the_reference_policy(tmp_path, name, source):
    """the head as the blob holds it (policy_bn1 and the convolution's bias folded, W_fc in the symbol's flatten order) on
    the oracle's trunk, read back with weights.read_blob"""
    _, symbol, cin, pch, n_labels, version = MX[name]
    arch, params = gen_mx.case_network(symbol, cin, pch, n_labels)
    blob = str(tmp_path / "c.arab")
    if source == "export_mx_blob":
        export_mx_blob(params, arch, blob, input_version=version)
    else:
        import_onnx(add_mx_head(write_mx_onnx(params, arch, str(tmp_path / "m.onnx")), params), blob)
    a, tensors, _ = read_blob(blob)
    assert a["n_labels"] == n_labels and a["semantics"] == "mxnet" and not a["policy_bias"]
    x = golden_input(arch)
    out = classic_mx_head.forward(params, arch, x)
    w1, b1, w2, b2, w_fc, b_fc = (torch.as_tensor(t) for t in tensors[-6:])
    C = out["trunk"].shape[1]
    with torch.no_grad():
        h = F.relu(F.conv2d(torch.as_tensor(out["trunk"]), w1.reshape(C, C, 3, 3), b1, padding=1))
        h = F.relu(F.conv2d(h, w2.reshape(pch, C, 3, 3), b2, padding=1)).reshape(x.shape[0], -1)
        logits = F.linear(h, w_fc.reshape(n_labels, pch * 64), b_fc).numpy()
    _assert_matches(_record(name), out["value"], logits)


# ---------------------------------------------------------------------------------------------- refusals
def _head_file(tmp_path, **kw):
    arch, sd, write = _torch_case("risev2_2272")
    return add_torch_head(write(sd, arch, str(tmp_path / "m.onnx")), sd, **kw)


def test_refuses_a_label_count_outside_the_classic_lists(tmp_path):
    _, sd, _ = _torch_case("risev2_2272")
    onnx = _head_file(tmp_path, w_fc=sd["policy_head.body3.0.weight"][:2000])
    with pytest.raises(ValueError, match="onto 2000 labels"):
        import_onnx(onnx, str(tmp_path / "o.arab"))


def test_refuses_a_fully_connected_layer_of_another_width(tmp_path):
    _, sd, _ = _torch_case("risev2_2272")
    onnx = _head_file(tmp_path, w_fc=sd["policy_head.body3.0.weight"][:, :80 * 64], flatten="Reshape")
    with pytest.raises(ValueError, match="takes 5120 features, not the 81 x 64"):
        import_onnx(onnx, str(tmp_path / "o.arab"))


def test_refuses_a_fully_connected_layer_not_behind_the_relu(tmp_path):
    onnx = _head_file(tmp_path, relu=False)
    with pytest.raises(ValueError, match="does not take its flattened ReLU"):
        import_onnx(onnx, str(tmp_path / "o.arab"))


def test_refuses_a_policy_map_convolution_with_a_bias(tmp_path):
    """a policy map (Flatten, Softmax) behind a convolution with a bias: ARAB2001 has no place for it, so the file is
    refused rather than the bias dropped"""
    onnx = _head_file(tmp_path, relu=False, fc=False)
    with pytest.raises(ValueError, match="has a bias but no fully-connected layer"):
        import_onnx(onnx, str(tmp_path / "o.arab"))


def test_refuses_an_mx_head_without_its_batchnorm(tmp_path):
    _, symbol, cin, pch, n_labels, _ = MX["risev2_2272"]
    arch, params = gen_mx.case_network(symbol, cin, pch, n_labels)
    onnx = add_mx_head(write_mx_onnx(params, arch, str(tmp_path / "m.onnx")), params, bn=False)
    with pytest.raises(ValueError, match="no BatchNormalization"):
        import_onnx(onnx, str(tmp_path / "o.arab"))


def test_refuses_an_mx_batchnorm_without_its_fully_connected_layer(tmp_path):
    _, symbol, cin, pch, n_labels, _ = MX["risev2_2272"]
    arch, params = gen_mx.case_network(symbol, cin, pch, n_labels)
    onnx = add_mx_head(write_mx_onnx(params, arch, str(tmp_path / "m.onnx")), params, fc=False)
    with pytest.raises(ValueError, match="BatchNormalization behind the last policy convolution but no fully-connected"):
        import_onnx(onnx, str(tmp_path / "o.arab"))


def test_refuses_an_mx_head_onto_another_label_count(tmp_path):
    _, symbol, cin, pch, n_labels, _ = MX["risev33_1968"]
    arch, params = gen_mx.case_network(symbol, cin, pch, n_labels)
    params = dict(params, policy_out_weight=params["policy_out_weight"][:1000], policy_out_bias=params["policy_out_bias"][:1000])
    onnx = add_mx_head(write_mx_onnx(params, arch, str(tmp_path / "m.onnx")), params)
    with pytest.raises(ValueError, match="onto 1000 labels"):
        import_onnx(onnx, str(tmp_path / "o.arab"))


@pytest.mark.parametrize("name", sorted(TORCH))
def test_policy_map_file_imports_as_before(tmp_path, name):
    """the same networks without the head: the policy-map blob of the checkpoint path, not an ARAB2004 one"""
    arch, sd, write = _torch_case(name)
    arch = {k: v for k, v in arch.items() if k != "n_labels"}
    sd = {k: v for k, v in sd.items() if not k.startswith(("policy_head.body2", "policy_head.body3"))}
    ref = export_blob(sd, arch, str(tmp_path / "ref.arab"), input_version=30 if arch["in_channels"] == 52 else 10)
    got = import_onnx(write(sd, arch, str(tmp_path / "m.onnx")), str(tmp_path / "onnx.arab"))
    assert "n_labels" not in got
    assert _bytes(ref) == _bytes(tmp_path / "onnx.arab")
