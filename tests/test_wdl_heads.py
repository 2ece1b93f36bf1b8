"""Value heads with WDL and plies-to-end outputs that feed the value (tests/wdl_heads.py): the PyTorch trainer's value MLP
(use_mlp_wdl_ply) and the MXNet symbols' head behind value_fc0, with value = win - loss or the MLP.

The oracles against the reference's own network code (tests/golden/wdl_head_golden.json), every import path against the
blob hashes recorded there, the blob reader against the writer, and the refusals of malformed heads."""
import gzip
import hashlib
import json
import os
import struct

import numpy as np
import pytest
import torch

from crazyara_b200 import weights
from crazyara_b200.mx_import import import_mxnet
from crazyara_b200.onnx_import import import_onnx
from crazyara_b200.weights import arch_from_state_dict, export_blob, export_mx_blob, import_checkpoint, read_blob, write_blob
from oracle import net_mx
from tests import classic_mx_head, wdl_heads
from tests.golden.gen_net_golden import golden_input
from tests.golden.gen_wdl_head_golden import VERSION, mx_archs, torch_archs
from tests.mx_params_writer import write_params
from tests.onnx_alphavile_writer import write_alphavile_onnx
from tests.onnx_mx_writer import write_mx_onnx
from tests.onnx_wdl_writer import add_mx_wdl, add_torch_mlp
from tests.onnx_writer import write_rise_onnx
from tests.test_mx_import import parameter_names, reordered, renamed_attrs

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = json.load(open(os.path.join(ROOT, "tests", "golden", "wdl_head_golden.json")))
TORCH, MX = torch_archs(), mx_archs()


def _sha(path):
    return hashlib.sha256(open(path, "rb").read()).hexdigest()


def symbol(head):
    with gzip.open(os.path.join(ROOT, "tests", "golden", f"mx_wdl_net_risev33_52_{head}-symbol.json.gz"), "rt") as f:
        return json.load(f)


def _check_record(out, g, value_atol, aux_atol):
    idx = g["prob_idx"]
    np.testing.assert_allclose(out["value"], g["value"], atol=value_atol)
    np.testing.assert_allclose(out["aux"], g["aux"], atol=aux_atol)
    np.testing.assert_allclose(out["prob"][:, idx], g["prob"], rtol=1e-4, atol=1e-9)
    assert out["prob"].argmax(1).tolist() == g["argmax"]


# ---------------------------------------------------------------------------------------------- oracles
@pytest.mark.parametrize("key", sorted(TORCH))
def test_torch_oracle_matches_the_reference_module(key):
    arch = TORCH[key]
    sd = wdl_heads.mlp_state_dict(arch, 0)
    assert sorted(sd) == GOLDEN[key]["param_names"]
    _check_record(wdl_heads.forward_torch(sd, arch, golden_input(arch)), GOLDEN[key], 2e-6, 2e-6)


@pytest.mark.parametrize("head", sorted(MX))
def test_mx_oracle_matches_the_reference_symbol(head):
    arch = MX[head]
    params = wdl_heads.mx_params(arch, 0)
    assert sorted(params) == GOLDEN[head]["param_names"] == parameter_names(symbol(head))
    out = wdl_heads.forward_mx(params, arch, golden_input(arch))
    assert np.allclose(out["aux"][:, :3].sum(1), 1.0), "MXNet's WDL output is the softmax"
    _check_record(out, GOLDEN[head], 1e-5, 1e-5)


# ---------------------------------------------------------------------------------------------- import paths
@pytest.mark.parametrize("key", sorted(TORCH))
def test_checkpoint_import_writes_the_mlp_head(tmp_path, key):
    """use_mlp_wdl_ply is read off body_final's shape: the blob carries the MLP (kind 2), not a plain WDL head, and an
    AlphaVile header keeps the trunk width as value_fc instead of the MLP's 8 units"""
    arch = TORCH[key]
    sd = wdl_heads.mlp_state_dict(arch, 0)
    torch.save({"model_state_dict": {k: torch.from_numpy(v) for k, v in sd.items()}}, tmp_path / "ck.tar")
    got = import_checkpoint(str(tmp_path / "ck.tar"), str(tmp_path / "net.arab"), VERSION[key])
    assert got["value_head"] == "wdl_mlp" and got["wdl"]
    assert got["value_fc"] == arch["value_fc"]
    assert _sha(tmp_path / "net.arab") == GOLDEN[key]["blob_sha256"]
    kind, = struct.unpack_from("<i", open(tmp_path / "net.arab", "rb").read(), 8 + 24)
    assert kind == 2
    back, tensors, _ = read_blob(str(tmp_path / "net.arab"))
    assert back["value_head"] == "wdl_mlp"
    np.testing.assert_array_equal(tensors[-7], sd["value_head.body_final.0.weight"].reshape(-1))


def test_state_dict_without_the_mlp_stays_a_wdl_head():
    arch = TORCH["risev33_mlp"]
    sd = wdl_heads.mlp_state_dict(arch, 0)
    plain = {k: v for k, v in sd.items() if not k.startswith("value_head.body_final")}
    assert "value_head" not in arch_from_state_dict(plain)
    sd["value_head.body_final.0.weight"] = np.zeros((256, 512), np.float32)  # the reference's unused fc0 layer
    assert "value_head" not in arch_from_state_dict(sd)


@pytest.mark.parametrize("variant", ["", "reordered", "attr"])
@pytest.mark.parametrize("dtype", ["float32", "float16"])
@pytest.mark.parametrize("head", sorted(MX))
def test_mx_model_files_import_writes_the_parameter_blob(tmp_path, head, dtype, variant):
    arch = MX[head]
    params = wdl_heads.mx_params(arch, 0)
    doc = symbol(head)
    doc = reordered(doc, 7) if variant == "reordered" else renamed_attrs(doc, variant) if variant else doc
    with open(tmp_path / "m-symbol.json", "w") as f:
        json.dump(doc, f)
    got = import_mxnet(str(tmp_path / "m-symbol.json"), write_params(params, str(tmp_path / "m.params"), dtype=dtype),
                       str(tmp_path / "m.arab"), VERSION[head])
    assert got["value_head"] == head and got["wdl"] and got["value_fc"] == 256
    held = {k: v.astype(dtype).astype(np.float32) for k, v in params.items()}
    ref = export_mx_blob(held, arch, str(tmp_path / "ref.arab"), input_version=VERSION[head])
    assert open(tmp_path / "m.arab", "rb").read() == open(ref, "rb").read()
    if dtype == "float32":
        assert _sha(tmp_path / "m.arab") == GOLDEN[head]["blob_sha256"]


@pytest.mark.parametrize("shuffle", [None, 0, 1, 2, 3])
@pytest.mark.parametrize("key", sorted(TORCH))
def test_torch_onnx_import_writes_the_checkpoint_blob(tmp_path, key, shuffle):
    """the torch export of the value MLP (tests/onnx_wdl_writer.add_torch_mlp), in the writer's node order and shuffled"""
    arch = TORCH[key]
    sd = wdl_heads.mlp_state_dict(arch, 0)
    path = str(tmp_path / "m.onnx")
    (write_alphavile_onnx(sd, arch, path) if "ntb" in arch else write_rise_onnx(sd, arch, path))
    got = import_onnx(add_torch_mlp(path, sd, shuffle), str(tmp_path / "m.arab"), VERSION[key])
    assert got["value_head"] == "wdl_mlp" and got["wdl"] and got["value_fc"] == arch["value_fc"]
    assert _sha(tmp_path / "m.arab") == GOLDEN[key]["blob_sha256"]


def _mx_onnx(tmp_path, head, shuffle):
    arch = MX[head]
    params = wdl_heads.mx_params(arch, 0)
    plain = dict(params, value_fc1_weight=np.zeros((1, 256), np.float32), value_fc1_bias=np.zeros(1, np.float32))
    path = write_mx_onnx(plain, dict(arch, value_head=None, wdl=False), str(tmp_path / "m.onnx"))
    return add_mx_wdl(path, params, head, shuffle)


@pytest.mark.parametrize("shuffle", range(8))
@pytest.mark.parametrize("head", sorted(MX))
def test_mx_onnx_import_writes_the_parameter_blob(tmp_path, head, shuffle):
    """the MXNet export of the WDL head (tests/onnx_wdl_writer.add_mx_wdl) in shuffled node orders: every Gemm behind
    value_fc0's Relu is read, whichever comes first.  An ONNX BatchNormalization holds its epsilon as a float32, so the
    blob is the parameter conversion's with that epsilon, and the model-file import's of the symbol stating it."""
    got = import_onnx(_mx_onnx(tmp_path, head, shuffle), str(tmp_path / "onnx.arab"))
    assert got["value_head"] == head and got["wdl"] and got["value_fc"] == 256
    assert _sha(tmp_path / "onnx.arab") == GOLDEN[head]["onnx_blob_sha256"]
    doc = symbol(head)
    for nd in doc["nodes"]:
        if nd["op"] == "BatchNorm":
            nd.setdefault("attrs", {})["eps"] = str(float(np.float32(1e-3)))
    with open(tmp_path / "m-symbol.json", "w") as f:
        json.dump(doc, f)
    import_mxnet(str(tmp_path / "m-symbol.json"), write_params(wdl_heads.mx_params(MX[head], 0), str(tmp_path / "m.params")),
                 str(tmp_path / "mx.arab"), VERSION[head])
    assert open(tmp_path / "mx.arab", "rb").read() == open(tmp_path / "onnx.arab", "rb").read()


def test_mx_onnx_import_refuses_a_head_it_cannot_hold(tmp_path):
    """a layer of three units alone behind value_fc0 is neither value_fc1 nor the WDL and plies layers"""
    arch = MX["mx_wdl"]
    params = wdl_heads.mx_params(arch, 0)
    params.update(value_fc1_weight=params["wdl_out_weight"], value_fc1_bias=params["wdl_out_bias"])
    onnx = write_mx_onnx(params, dict(arch, value_head=None, wdl=False), str(tmp_path / "m.onnx"))
    with pytest.raises(ValueError, match=r"fully-connected layers of \[3\] units behind value_fc0"):
        import_onnx(onnx, str(tmp_path / "m.arab"))


# ---------------------------------------------------------------------------------------------- the blob
def _blobs(tmp_path):
    for key, arch in TORCH.items():
        yield key, export_blob(wdl_heads.mlp_state_dict(arch, 0), arch, str(tmp_path / f"{key}.arab"), VERSION[key])
    for head, arch in MX.items():
        yield head, export_mx_blob(wdl_heads.mx_params(arch, 0), arch, str(tmp_path / f"{head}.arab"), VERSION[head])
    # the MXNet head behind 96 hidden units, and with a fully-connected policy head (ARAB2004 around ARAB2002)
    base = net_mx.arch_mx_risev33(52, 76)
    arch = wdl_heads.mx_arch(base, "mx_wdl_mlp", 96)
    yield "mx_96", export_mx_blob(wdl_heads.mx_params(arch, 1), arch, str(tmp_path / "mx_96.arab"), 30)
    arch = classic_mx_head.classic_arch(wdl_heads.mx_arch(base, "mx_wdl"), 1968)
    params = {**wdl_heads.mx_params(arch, 2), **classic_mx_head.head_params(arch, 1968, 2)}
    yield "mx_fc", export_mx_blob(params, arch, str(tmp_path / "mx_fc.arab"), 30)


def test_read_blob_inverts_write_blob(tmp_path):
    for key, path in _blobs(tmp_path):
        arch, tensors, version = read_blob(path)
        assert arch["value_head"] in ("wdl_mlp", "mx_wdl", "mx_wdl_mlp") and arch["wdl"], key
        again = write_blob(str(tmp_path / "again.arab"), arch, tensors, version)
        assert open(again, "rb").read() == open(path, "rb").read(), key


def test_existing_kinds_keep_their_header_word(tmp_path):
    from oracle import net as onet
    for wdl in (False, True):
        arch = onet.arch_risev33(52, 76, wdl)
        path = export_blob(onet.make_state_dict(arch, 0), arch, str(tmp_path / "n.arab"), 30)
        assert struct.unpack_from("<i", open(path, "rb").read(), 32)[0] == int(wdl)
        assert "value_head" not in read_blob(path)[0]


HEADER_FC, HEADER_KIND = 28, 32  # byte offsets of the base header's value_fc and WDL words (ARAB2001 / 2002)


def _mlp_width(width):
    def edit(buf, arch, tensors):
        n = -3 - arch.get("policy_bias", False) - 4  # the MLP in front of the policy map's tensors
        tensors[n:n + 4] = [np.ones(4 * width, np.float32), np.ones(width, np.float32), np.ones(width, np.float32),
                            np.ones(1, np.float32)]
    return edit


def _word(offset, value):
    def edit(buf, arch, tensors):
        struct.pack_into("<i", buf, offset, value)
    return edit


MALFORMED = {"mlp_width_6": ("mx_wdl_mlp", _mlp_width(6), "MLP of width 6"),
             "mlp_width_16": ("risev33_mlp", _mlp_width(16), "MLP of width 16"),
             "hidden_0": ("mx_wdl", _word(HEADER_FC, 0), "hidden layer of 0 units"),
             "hidden_300": ("mx_wdl_mlp", _word(HEADER_FC, 300), "hidden layer of 300 units"),
             "kind_5": ("mx_wdl", _word(HEADER_KIND, 5), "unknown kind 5"),
             "kind_-1": ("risev33_mlp", _word(HEADER_KIND, -1), "unknown kind -1")}


def malformed_blob(tmp_path, case):
    """-> (the path of a blob with the malformed head `case`, the reason both readers give): its tensors rewritten past
    write_blob's own check, or a header word patched"""
    key, edit, reason = MALFORMED[case]
    path = dict(_blobs(tmp_path))[key]
    arch, tensors, version = read_blob(path)
    if case.startswith("mlp"):
        edit(None, arch, tensors)
        check, weights.check_value_head = weights.check_value_head, lambda *a: None
        try:
            path = write_blob(str(tmp_path / "bad.arab"), arch, tensors, version)
        finally:
            weights.check_value_head = check
    else:
        buf = bytearray(open(path, "rb").read())
        edit(buf, arch, tensors)
        path = str(tmp_path / "bad.arab")
        open(path, "wb").write(bytes(buf))
    return path, reason


@pytest.mark.parametrize("case", sorted(MALFORMED))
def test_read_blob_refuses_a_malformed_head(tmp_path, case):
    path, reason = malformed_blob(tmp_path, case)
    with pytest.raises(ValueError, match=reason):
        read_blob(path)


@pytest.mark.parametrize("case", ["hidden_300", "mlp_width_6"])
def test_write_blob_refuses_a_malformed_head(tmp_path, case, monkeypatch):
    path, reason = malformed_blob(tmp_path, case)
    with monkeypatch.context() as m:
        m.setattr(weights, "check_value_head", lambda *a: None)
        arch, tensors, version = read_blob(path)
    with pytest.raises(ValueError, match=reason):
        write_blob(str(tmp_path / "again.arab"), arch, tensors, version)
