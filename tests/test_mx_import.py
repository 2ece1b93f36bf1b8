"""MXNet model files (`-symbol.json` + `.params`) through crazyara_b200/mx_import.py.  The symbols are the reference's own
RISEv2 / RISEv3.3 symbol code serialised by tests/golden/gen_mx_symbol_golden.py (committed gzip-compressed, written out
as plain `-symbol.json` files for the import); the parameter files are written by tests/mx_params_writer.py.  The import must give the blob export_mx_blob writes for the same parameters and the one
import_onnx writes for the same network's MXNet export, byte for byte, and that blob must compute what the stand-in
evaluation of the reference symbol computed (tests/golden/mx_net_*.json, classic_mx_net_*.json).  PARITY UNPINNED: no
file written by MXNet itself is at hand."""
import gzip
import json
import os
import subprocess
import sys

import numpy as np
import pytest

from crazyara_b200.mx_import import import_mxnet, model_files, read_params
from crazyara_b200.onnx_import import import_onnx
from crazyara_b200.weights import export_mx_blob, read_blob, write_blob
from oracle import net_mx
from tests import classic_mx_head
from tests.golden.gen_net_golden import golden_input
from tests.mx_params_writer import array_record, params_bytes, write_params
from tests.onnx_classic_writer import add_mx_head
from tests.onnx_mx_writer import write_mx_onnx
from tests.test_onnx_classic_import import _assert_matches, _record
from tests.test_oracle_net_mx import _blob_forward

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
# symbol record -> (base arch, n_labels of the fully-connected head or None, input version)
CASES = {"mx_net_risev2_34": (lambda: net_mx.arch_mx_risev2(34, 81), None, 10),
         "mx_net_risev33_52": (lambda: net_mx.arch_mx_risev33(52, 76), None, 30),
         "classic_mx_net_risev2_2272": (lambda: net_mx.arch_mx_risev2(34, 81), 2272, 10),
         "classic_mx_net_risev33_1968": (lambda: net_mx.arch_mx_risev33(52, 76), 1968, 30)}


def network(record, seed):
    """-> (arch, parameters under the symbol's names) of a record"""
    base, n_labels, _ = CASES[record]
    if n_labels:
        return classic_mx_head.make_params(base(), n_labels, seed)
    return base(), net_mx.make_mx_params(base(), seed)


def symbol(record):
    with gzip.open(os.path.join(GOLDEN, f"{record}-symbol.json.gz"), "rt") as f:
        return json.load(f)


def dump(doc, path):
    with open(path, "w") as f:
        json.dump(doc, f)
    return str(path)


def parameter_names(doc):
    """the symbol's arguments and aux states without the data input and the output labels"""
    names = [doc["nodes"][i]["name"] for i in doc["arg_nodes"]]
    return sorted(n for n in names if n != "data" and not n.endswith("_label"))


def imported(tmp_path, record, seed=3, doc=None, style="prefixed", dtype="float32", params=None):
    """-> (arch import_mxnet returned, the blob's bytes, the parameters as the file holds them)"""
    arch, ps = network(record, seed)
    ps = ps if params is None else params
    sym = dump(symbol(record) if doc is None else doc, tmp_path / "m-symbol.json")
    got = import_mxnet(sym, write_params(ps, str(tmp_path / "m.params"), style, dtype), str(tmp_path / "m.arab"))
    return got, open(tmp_path / "m.arab", "rb").read(), {k: v.astype(dtype).astype(np.float32) for k, v in ps.items()}


def _bytes(path):
    return open(path, "rb").read()


# ---------------------------------------------------------------------------------------------- one conversion
@pytest.mark.parametrize("dtype", ["float32", "float16"])
@pytest.mark.parametrize("style", ["prefixed", "bare"])
@pytest.mark.parametrize("record", sorted(CASES))
def test_import_writes_the_parameter_conversion_blob(tmp_path, record, style, dtype):
    arch, params = network(record, 3)
    assert parameter_names(symbol(record)) == sorted(params)
    got, blob, held = imported(tmp_path, record, style=style, dtype=dtype)
    for key in ("kernels", "c_ops", "se_types", "stem_act", "policy_bias", "in_channels", "policy_channels", "wdl"):
        assert got[key] == arch[key], key
    assert [g for g, s in zip(got["se_gates"], got["se_types"]) if s] == [g for g, s in zip(arch["se_gates"], arch["se_types"]) if s]
    assert got.get("n_labels") == arch.get("n_labels")
    ref = export_mx_blob(held, arch, str(tmp_path / "ref.arab"), input_version=CASES[record][2])
    assert blob == _bytes(ref)


@pytest.mark.parametrize("record", sorted(CASES))
def test_import_writes_the_onnx_import_blob(tmp_path, record):
    """the same network as its MXNet ONNX export (tests/onnx_mx_writer.py): an ONNX attribute holds the BatchNorm epsilon
    as a float32, so the symbol states that epsilon too"""
    arch, params = network(record, 4)
    onnx = write_mx_onnx(params, arch, str(tmp_path / "m.onnx"))
    if arch.get("n_labels"):
        onnx = add_mx_head(onnx, params)
    import_onnx(onnx, str(tmp_path / "onnx.arab"))
    doc = symbol(record)
    for nd in doc["nodes"]:
        if nd["op"] == "BatchNorm":
            nd.setdefault("attrs", {})["eps"] = str(float(np.float32(1e-3)))
    _, blob, _ = imported(tmp_path, record, seed=4, doc=doc)
    assert blob == _bytes(tmp_path / "onnx.arab")


def reordered(doc, seed):
    """the same graph with its node list permuted and every node reference remapped"""
    perm = np.random.default_rng(seed).permutation(len(doc["nodes"]))
    new = {int(old): i for i, old in enumerate(perm)}
    remap = lambda e: [new[e[0]]] + e[1:]
    nodes = [dict(doc["nodes"][old], inputs=[remap(e) for e in doc["nodes"][old]["inputs"]]) for old in perm]
    return dict(doc, nodes=nodes, arg_nodes=sorted(new[i] for i in doc["arg_nodes"]), heads=[remap(e) for e in doc["heads"]])


def renamed_attrs(doc, key):
    return dict(doc, nodes=[{(key if k == "attrs" else k): v for k, v in nd.items()} for nd in doc["nodes"]])


@pytest.mark.parametrize("variant", ["reordered", "attr", "param"])
@pytest.mark.parametrize("record", sorted(CASES))
def test_node_order_and_attribute_key_do_not_matter(tmp_path, record, variant):
    doc = symbol(record)
    doc = reordered(doc, len(record)) if variant == "reordered" else renamed_attrs(doc, variant)
    _, blob, _ = imported(tmp_path, record, doc=doc)
    (tmp_path / "x").mkdir()
    assert blob == imported(tmp_path / "x", record)[1]


def test_batchnorm_attributes_are_honoured(tmp_path):
    """eps and fix_gamma=False on one BatchNorm change the blob exactly as export_mx_blob's arguments do"""
    arch, params = network("mx_net_risev2_34", 3)
    doc = symbol("mx_net_risev2_34")
    stem = next(nd for nd in doc["nodes"] if nd["name"] == "stem_bn0")
    stem["attrs"] = {"eps": "2e-05", "fix_gamma": "False"}
    _, blob, _ = imported(tmp_path, "mx_net_risev2_34", doc=doc)
    ones = {k: np.ones_like(v) if k.endswith("_gamma") and k != "stem_bn0_gamma" else v for k, v in params.items()}
    ref = export_mx_blob(ones, arch, str(tmp_path / "ref.arab"), eps={"stem_bn0": 2e-5}, fix_gamma=False)
    assert blob == _bytes(ref)


# ---------------------------------------------------------------------------------------------- the reference's outputs
@pytest.mark.parametrize("record", sorted(CASES))
def test_imported_blob_computes_the_reference_symbol(tmp_path, record):
    """the blob, read back by weights.read_blob, on the golden input against the stand-in's evaluation of the reference
    symbol on the same seed-0 parameters, within tests/test_oracle_net_mx.py's and tests/test_onnx_classic_import.py's
    tolerances"""
    arch, _ = network(record, 0)
    got, _, _ = imported(tmp_path, record, seed=0)
    x = golden_input(arch)
    if not got.get("n_labels"):
        with open(os.path.join(GOLDEN, f"{record}.json")) as f:
            g = json.load(f)
        value, logits = _blob_forward(str(tmp_path / "m.arab"), x)
        prob = np.exp(logits - logits.max(1, keepdims=True))
        prob /= prob.sum(1, keepdims=True)
        idx = np.array(g["prob_idx"])
        np.testing.assert_allclose(value, g["value"], atol=1e-5)
        np.testing.assert_allclose(prob[:, idx], g["prob"], atol=1e-5, rtol=1e-4)
        lp = np.log(prob)
        np.testing.assert_allclose((lp - lp.mean(1, keepdims=True))[:, idx], g["centred_log_prob"], atol=1e-4)
        assert prob.argmax(1).tolist() == g["argmax"]
        return
    # the fully-connected head: the base blob with the folded last convolution as a policy map, then ReLU, W_fc, b_fc
    a, tensors, version = read_blob(str(tmp_path / "m.arab"))
    base = {k: v for k, v in a.items() if k != "n_labels"}
    write_blob(str(tmp_path / "base.arab"), dict(base, policy_bias=True), tensors[:-2], version)
    value, conv = _blob_forward(str(tmp_path / "base.arab"), x)
    logits = np.maximum(conv, 0) @ tensors[-2].reshape(a["n_labels"], -1).T + tensors[-1]
    _assert_matches(_record(record[len("classic_mx_net_"):]), value, logits)


# ---------------------------------------------------------------------------------------------- model directories
def test_model_directory_picks_the_float_files_and_the_command_line_imports_it(tmp_path):
    arch, params = network("mx_net_risev33_52", 3)
    d = tmp_path / "model"
    d.mkdir()
    dump(symbol("mx_net_risev33_52"), d / "model-symbol.json")
    write_params(params, str(d / "model-0000.params"))
    (d / "model-int8-symbol.json").write_text("{}")
    (d / "model-int8-0000.params").write_bytes(b"\0")
    assert model_files(str(d)) == (str(d / "model-symbol.json"), str(d / "model-0000.params"))
    out = subprocess.run([sys.executable, "-m", "crazyara_b200.mx_import", str(d), str(tmp_path / "m.arab")], cwd=ROOT,
                         capture_output=True, text=True, check=True).stdout
    assert out.strip() == f"{tmp_path / 'm.arab'}: 15 blocks, 52 -> 76x64, wdl=False"
    ref = export_mx_blob(params, arch, str(tmp_path / "ref.arab"), input_version=30)
    assert _bytes(tmp_path / "m.arab") == _bytes(ref)


@pytest.mark.parametrize("files, message", [
    (["m-symbol.json"], "doesn't contain a file ending with .params"),
    (["m-0000.params", "m-int8-symbol.json"], "doesn't contain a file ending with .json"),
    (["a-symbol.json", "b-symbol.json", "m.params"], "more than one file ending with .json"),
    (["m-symbol.json", "m-0000.params", "m-0001.params"], "more than one file ending with .params")])
def test_model_directory_refuses_a_missing_or_ambiguous_file(tmp_path, files, message):
    for f in files:
        (tmp_path / f).write_bytes(b"")
    with pytest.raises(ValueError, match=message):
        model_files(str(tmp_path))


# ---------------------------------------------------------------------------------------------- .params refusals
def _params_file(tmp_path, data):
    (tmp_path / "bad.params").write_bytes(data)
    return str(tmp_path / "bad.params")


def test_params_reader_reads_both_styles_and_dtypes(tmp_path):
    a = {"x_weight": np.arange(6, dtype=np.float32).reshape(2, 3) / 7, "x_moving_var": np.ones(2, np.float32)}
    for style in ("prefixed", "bare"):
        for dtype in ("float32", "float16"):
            got = read_params(_params_file(tmp_path, params_bytes(a, style, dtype)))
            assert sorted(got) == sorted(a)
            for k in a:
                assert got[k].dtype == np.float32 and np.array_equal(got[k], a[k].astype(dtype).astype(np.float32))


@pytest.mark.parametrize("case, message", [
    ("list magic", "not MXNet's NDArray list magic"), ("array magic", "not the V2 NDArray magic"),
    ("sparse", "sparse storage"), ("float64", "dtype float64"), ("duplicate", "'x_weight' appears twice"),
    ("truncated", "truncated")])
def test_params_reader_refuses(tmp_path, case, message):
    a = {"x_weight": np.ones((2, 3), np.float32), "y_bias": np.zeros(2, np.float32)}
    recs = [array_record(v) for v in a.values()]
    data = {"list magic": lambda: b"\x13" + params_bytes(a)[1:],
            "array magic": lambda: params_bytes(a, records=[array_record(a["x_weight"], magic=0xF993FACA), recs[1]]),
            "sparse": lambda: params_bytes(a, records=[recs[0], array_record(a["y_bias"], stype=1)]),
            "float64": lambda: params_bytes(a, records=[recs[0], array_record(a["y_bias"], "float64")]),
            "duplicate": lambda: params_bytes({"x_weight": a["x_weight"], "arg:x_weight": a["x_weight"]}, style="bare"),
            "truncated": lambda: params_bytes(a)[:-1]}[case]()
    with pytest.raises(ValueError, match=message):
        read_params(_params_file(tmp_path, data))


# ---------------------------------------------------------------------------------------------- symbol refusals
def _add(doc, op, name, inputs, attrs=None):
    doc["nodes"].append({"op": op, "name": name, "inputs": inputs, **({"attrs": attrs} if attrs else {})})
    return [len(doc["nodes"]) - 1, 0, 0]


def _node(doc, name):
    return next(nd for nd in doc["nodes"] if nd["name"] == name)


def _cm_se(doc):  # ca_se with max pooling
    _node(doc, "bc_res_block12_se_avg_pool0")["attrs"]["pool_type"] = "max"


def _cbam(doc):  # channel attention over average and max pooling
    avg = _node(doc, "bc_res_block12_se_avg_pool0")
    mx = _add(doc, "Pooling", "cbam_max_pool0", avg["inputs"], dict(avg["attrs"], pool_type="max"))
    cat = _add(doc, "Concat", "cbam_concat_0", [[doc["nodes"].index(avg), 0, 0], mx], {"dim": "1"})
    _node(doc, "bc_res_block12_se_flatten0")["inputs"] = [cat]


def _sa_se(doc):  # the eca_se's convolution as a 7x7 one over the channel mean: spatial attention
    conv = _node(doc, "convolution0")
    pool = doc["nodes"][doc["nodes"][conv["inputs"][0][0]]["inputs"][0][0]]
    conv["inputs"][0] = _add(doc, "mean", "sa_mean", pool["inputs"][:1], {"axis": "1", "keepdims": "True"})
    conv["attrs"].update(kernel="(7, 7)", pad="(3, 3)")


def _variant_input(doc):  # the variant planes split off the input and concatenated to the trunk
    split = _add(doc, "SliceChannel", "variants_split", [[0, 0, 0]], {"axis": "1", "num_outputs": "34"})
    _add(doc, "Concat", "bc_res_block0_concat", [_node(doc, "bc_res_block0_conv1")["inputs"][0], split])


def _wdl(doc):  # value_fc0's activation also feeds a 3-way FullyConnected (wdl_out)
    act = next(i for i, nd in enumerate(doc["nodes"]) if nd["name"] == "value_act1")
    w = _add(doc, "null", "wdl_out_weight", [])
    b = _add(doc, "null", "wdl_out_bias", [])
    _add(doc, "FullyConnected", "wdl_out", [[act, 0, 0], w, b], {"num_hidden": "3"})


@pytest.mark.parametrize("record, edit, message", [
    ("mx_net_risev2_34", _cm_se, "block 12: cm_se"), ("mx_net_risev2_34", _cbam, "block 12: cbam"),
    ("mx_net_risev33_52", _sa_se, "block 5: sa_se"), ("mx_net_risev2_34", _variant_input, "use_extra_variant_input"),
    ("mx_net_risev33_52", _wdl, "WDL and plies-to-end")], ids=["cm_se", "cbam", "sa_se", "variant_input", "wdl"])
def test_refuses_what_no_blob_format_holds(tmp_path, record, edit, message):
    doc = symbol(record)
    edit(doc)
    params = dict(network(record, 3)[1], wdl_out_weight=np.ones((3, 256), np.float32), wdl_out_bias=np.zeros(3, np.float32))
    with pytest.raises(ValueError, match=message):
        imported(tmp_path, record, doc=doc, params=params)


@pytest.mark.parametrize("cut, message", [(lambda w: w[:1000], "onto 1000 labels"),
                                          (lambda w: w[:, :80 * 64], "takes 5120 features, not the 81 x 64")])
def test_refuses_a_fully_connected_head_of_another_width(tmp_path, cut, message):
    _, params = network("classic_mx_net_risev2_2272", 3)
    params = dict(params, policy_out_weight=cut(params["policy_out_weight"]))
    with pytest.raises(ValueError, match=message):
        imported(tmp_path, "classic_mx_net_risev2_2272", params=params)
