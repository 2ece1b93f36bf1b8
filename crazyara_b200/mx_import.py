"""Weight import from the reference's MXNet model files (SURVEY §8 f3): a `-symbol.json` and a `.params` file, as its MXNet
back-end loads them from a model directory (engine/src/nn/mxnetapi.cpp, fill_model_paths) -> the ARAB2002 blob
weights.export_mx_blob writes (ARAB2004 around it with a fully-connected policy head).  Neither MXNet nor any other
package is needed.

The `.params` file (MXNet 1.x NDArray::Save of a named list, src/ndarray/ndarray.cc), all little-endian:
  uint64 list magic 0x112, uint64 reserved;
  uint64 array count, then per array: uint32 magic 0xF993FAC9 (V2), int32 storage type (0 dense), uint32 ndim and ndim
    int64 dims, int32 dev_type and int32 dev_id (the context), int32 type_flag (0 float32, 2 float16), the raw data;
  uint64 name count, then per name a uint64 length and its bytes.
Names carry `arg:` / `aux:` prefixes (save_checkpoint, export) or none (save_parameters); the prefixes are stripped.  Another
magic, sparse storage, another dtype, a name that appears twice and a file that ends early are refused.
LAYOUT UNPINNED: it is taken from MXNet's source, not checked against a file MXNet wrote; neither tree holds one, so the
reader is tested against tests/mx_params_writer.py, which writes the layout above.

The symbol file (NNVM graph JSON): `nodes` with `op`, `name`, `inputs` ([node, output, version]) and the attributes as
strings under `attrs` (`attr` or `param` in older files); parameters are `null` nodes.  The node order is not trusted:
the walk follows the edges from the data input through the stem, block by block, to the heads, the way
onnx_import._import_mxnet_graph reads an MXNet ONNX export, and shares its edge walks (onnx_import._Graph).  What it
reads -- per block the 1x1 expansion, the 3x3 / 5x5 depthwise kernel, ca_se or eca_se on the block input with the
shortcut taken before it; the value head; a policy map or policy_bn1, activation, Flatten and FullyConnected onto a
classic label list; every BatchNorm's eps and fix_gamma -- becomes the MXNet-named parameters and arch that
export_mx_blob converts.  The value head is the standard one or, with use_wdl and use_plys_to_end, the WDL and plies
outputs behind value_fc0 with value = win - loss or the value MLP (use_mlp_wdl_ply).  Refused by name, as no blob format
holds them: sa_se / sm_se / cm_se / cbam blocks, use_extra_variant_input, a value head with only one of the WDL and
plies-to-end outputs, and a fully-connected policy layer of another width.
"""
import ast
import json
import os
import struct

import numpy as np

from .onnx_import import _Graph
from .weights import CLASSIC_LABELS, MX_BN_EPS, export_mx_blob, input_version_of

LIST_MAGIC, NDARRAY_V2_MAGIC = 0x112, 0xF993FAC9
DTYPES = {0: np.dtype("<f4"), 2: np.dtype("<f2")}  # MXNet type flags read here
_DTYPE_NAMES = {1: "float64", 3: "uint8", 4: "int32", 5: "int8", 6: "int64", 7: "bool", 12: "bfloat16"}
# ops a tensor passes through unchanged for the walk (the SE gate's reshape, the heads' Flatten, the tower's Dropout)
_SKIP = ("Reshape", "reshape", "Flatten", "flatten", "Dropout")
_ADD = ("broadcast_add", "elemwise_add", "_Plus", "_plus")
_MUL = ("broadcast_mul", "elemwise_mul", "_Mul", "_mul")


# ---------------------------------------------------------------------------------------------- .params
def read_params(path):
    """-> {name without arg: / aux: prefix: float32 ndarray}"""
    buf = open(path, "rb").read()
    off = 0

    def take(fmt):
        nonlocal off
        size = struct.calcsize(fmt)
        if off + size > len(buf):
            raise ValueError(f"{path}: truncated at byte {off} (the file has {len(buf)})")
        v = struct.unpack_from(fmt, buf, off)
        off += size
        return v

    magic, _ = take("<QQ")
    if magic != LIST_MAGIC:
        raise ValueError(f"{path}: list magic {magic:#x}, not MXNet's NDArray list magic {LIST_MAGIC:#x}")
    arrays = []
    for i in range(take("<Q")[0]):
        magic, stype = take("<Ii")
        if magic != NDARRAY_V2_MAGIC:
            raise ValueError(f"{path}: array {i} has magic {magic:#x}, not the V2 NDArray magic {NDARRAY_V2_MAGIC:#x}")
        if stype != 0:
            raise ValueError(f"{path}: array {i} has sparse storage (storage type {stype}); only dense arrays are read")
        ndim, = take("<I")
        if ndim == 0:
            raise ValueError(f"{path}: array {i} has no shape")
        shape = take(f"<{ndim}q")
        _, _, flag = take("<iii")  # dev_type, dev_id, type_flag
        if flag not in DTYPES:
            raise ValueError(f"{path}: array {i} has dtype {_DTYPE_NAMES.get(flag, flag)}; only float32 and float16 are read")
        n = int(np.prod(shape))
        data = take(f"{n * DTYPES[flag].itemsize}s")[0]
        arrays.append(np.frombuffer(data, DTYPES[flag]).astype(np.float32).reshape(shape))
    names = []
    for _ in range(take("<Q")[0]):
        length, = take("<Q")
        names.append(take(f"{length}s")[0].decode())
    if off != len(buf):
        raise ValueError(f"{path}: {len(buf) - off} bytes after the names")
    if len(names) != len(arrays):
        raise ValueError(f"{path}: {len(arrays)} arrays but {len(names)} names")
    out = {}
    for name, a in zip(names, arrays):
        key = name[4:] if name.startswith(("arg:", "aux:")) else name
        if key in out:
            raise ValueError(f"{path}: the name '{key}' appears twice")
        out[key] = a
    return out


# ---------------------------------------------------------------------------------------------- -symbol.json
def _value(s):
    """an attribute string -> a Python value: tuples and numbers as literals, booleans in either case, else the string"""
    if s.lower() in ("true", "false"):
        return s.lower() == "true"
    try:
        return ast.literal_eval(s)
    except (ValueError, SyntaxError):
        return s


def read_symbol(path):
    """-> (nodes [(op, inputs, outputs, {attr: value}, name)] of the operators, the variable names).  A tensor is named by its
    variable's name, or `#<node>:<output>` for an operator's output."""
    doc = json.load(open(path))
    raw = doc["nodes"]
    tensor = lambda e: raw[e[0]]["name"] if raw[e[0]]["op"] == "null" else f"#{e[0]}:{e[1]}"
    n_out = [1] * len(raw)
    for e in [e for n in raw for e in n["inputs"]] + doc["heads"]:
        n_out[e[0]] = max(n_out[e[0]], e[1] + 1)
    nodes = []
    for i, n in enumerate(raw):
        if n["op"] == "null":
            continue
        attrs = n.get("attrs", n.get("attr", n.get("param"))) or {}
        nodes.append((n["op"], [tensor(e) for e in n["inputs"]], [f"#{i}:{k}" for k in range(n_out[i])],
                      {k: _value(str(v)) for k, v in attrs.items()}, n["name"]))
    return nodes, [raw[i]["name"] for i in doc["arg_nodes"]]


def _import_symbol(g, variables, arrays, blob_path, input_version, channels):
    """the operator graph of a RISE symbol (rise_mobile_v2.py / rise_mobile_v3.py) -> ARAB2002 blob (ARAB2004 around it)"""
    params, eps = {}, {}
    attr = lambda nd, k, d=None: nd[3].get(k, d)

    def array(name):
        if name not in arrays:
            g.fail(f"'{name}' is not in the parameter file")
        return arrays[name]

    def take(nd, name):  # a Convolution's / FullyConnected's weight and bias under the MXNet layer name
        params[name + "_weight"] = array(nd[1][1])
        if not attr(nd, "no_bias", False):
            params[name + "_bias"] = array(nd[1][2])

    def take_bn(nd, name):  # fix_gamma (MXNet's default): the gamma is 1 whatever the file holds
        for key, i in (("gamma", 1), ("beta", 2), ("moving_mean", 3), ("moving_var", 4)):
            params[f"{name}_{key}"] = array(nd[1][i])
        if attr(nd, "fix_gamma", True):
            params[name + "_gamma"] = np.ones_like(params[name + "_gamma"])
        eps[name] = float(attr(nd, "eps", MX_BN_EPS))

    def relu(t, where):  # the Activation in front of tensor t, which must be a ReLU
        act = g.back(t, "Activation")
        if attr(act, "act_type") != "relu":
            g.fail(f"{where}: activation {attr(act, 'act_type')} (the blob formats hold ReLU)")
        return act

    def relu_out(nd):  # the output of the ReLU behind node nd
        act = g.first(nd[2][0], "Activation")
        if act is None or attr(act, "act_type") != "relu":
            g.fail(f"no ReLU behind {nd[4]}")
        return act[2][0]

    def conv_bn(t, name):  # t = output of Convolution -> BatchNorm: the Convolution node
        bn = g.back(t, "BatchNorm")
        conv = g.back(bn[1][0], "Convolution")
        take(conv, name)
        take_bn(bn, name.replace("conv", "bn"))
        return conv

    # the stem on the data input
    data = [v for v in variables if v not in arrays and any(nd[1][0] == v for nd in g.cons[v])]
    if len(data) != 1:
        g.fail(f"expected one data input, found {data}")
    feeds = g.cons[data[0]]
    if any(nd[0] in ("SliceChannel", "split", "Concat") for nd in feeds):
        g.fail("the input planes feed the blocks (use_extra_variant_input): no blob format holds it")
    stem = [nd for nd in feeds if nd[0] == "Convolution"]
    if len(feeds) != 1 or len(stem) != 1:
        g.fail(f"the data input feeds {sorted(nd[0] for nd in feeds)}, not only the stem convolution")
    stem = stem[0]
    if attr(stem, "num_filter") != channels or tuple(attr(stem, "kernel", ())) != (3, 3):
        g.fail(f"no 3x3 stem convolution with {channels} channels on the data input")
    take(stem, "stem_conv0")
    bn = g.first(stem[2][0], "BatchNorm")
    if bn is None:
        g.fail("no BatchNorm behind the stem")
    take_bn(bn, "stem_bn0")
    act = g.first(bn[2][0], "Activation")
    x, stem_act = (act[2][0], True) if act is not None else (bn[2][0], False)
    if stem_act and attr(act, "act_type") != "relu":
        g.fail(f"stem: activation {attr(act, 'act_type')} (the blob formats hold ReLU)")

    # the blocks: x + bn3(conv3(relu(bn2(dw(relu(bn1(conv1(se(x))))))))), the shortcut before the squeeze-excitation
    kernels, se_types, se_gates, c_ops = [], [], [], []
    while True:
        add = next((nd for op in _ADD for nd in g.cons[x] if nd[0] == op), None)
        if add is None:
            break
        i, p = len(kernels), f"bc_res_block{len(kernels)}"
        conv3 = conv_bn(add[1][1] if add[1][0] == x else add[1][0], p + "_conv3")
        conv2 = conv_bn(relu(conv3[1][0], f"block {i}")[1][0], p + "_conv2")
        t = relu(conv2[1][0], f"block {i}")[1][0]
        if g.prod.get(g.back(t, "BatchNorm")[1][0], ("",))[0] != "Convolution":
            g.fail(f"block {i}: no 1x1 expansion convolution in front of the depthwise convolution")
        conv1 = conv_bn(t, p + "_conv1")
        w1, wd = params[p + "_conv1_weight"], params[p + "_conv2_weight"]
        if (w1.shape[1:] != (channels, 1, 1) or wd.shape[0] != w1.shape[0] or wd.shape[2] not in (3, 5) or
                attr(conv2, "num_group") != w1.shape[0]):
            g.fail(f"block {i} is not a RISE bottleneck block")
        se, gate = None, None
        if conv1[1][0] != x:
            se, gate = _se(g, g.back(conv1[1][0], *_MUL), x, i, take, p, sum(s == "eca_se" for s in se_types))
        kernels.append(int(wd.shape[2])), se_types.append(se), se_gates.append(gate), c_ops.append(int(w1.shape[0]))
        x = add[2][0]
    if not kernels:
        g.fail("no bottleneck block found")

    # the heads: value_conv0 (1x1) and policy_conv0 (3x3) on the tower's output
    heads = g.fwd(x, "Convolution")
    vconv = [nd for nd in heads if tuple(attr(nd, "kernel", ())) == (1, 1)]
    pconv = [nd for nd in heads if tuple(attr(nd, "kernel", ())) == (3, 3)]
    if len(vconv) != 1 or len(pconv) != 1:
        g.fail("value head (1x1 convolution) and policy head (3x3 convolution) not found behind the tower")
    vbn = g.one(vconv[0][2][0], "BatchNorm")
    take(vconv[0], "value_conv0"), take_bn(vbn, "value_bn0")
    fc0 = g.one(relu_out(vbn), "FullyConnected")
    take(fc0, "value_fc0")
    value_head = _value_outputs(g, g.fwd(relu_out(fc0), "FullyConnected"), take, relu_out)
    vc, fc = int(params["value_conv0_weight"].shape[0]), int(params["value_fc0_weight"].shape[0])
    if vc != 8 or (fc != 256 if value_head is None else not 1 <= fc <= 256):
        g.fail(f"value head: {vc} channels and {fc} hidden units (the blob formats hold 8 and 256, or with WDL and "
               f"plies-to-end outputs 1 .. 256 hidden units)")
    pbn = g.one(pconv[0][2][0], "BatchNorm")
    take(pconv[0], "policy_conv0"), take_bn(pbn, "policy_bn0")
    pc1 = g.one(relu_out(pbn), "Convolution")
    take(pc1, "policy_conv1")
    P = int(params["policy_conv1_weight"].shape[0])
    arch = dict(name=f"rise_{len(kernels)}b", semantics="mxnet", in_channels=int(params["stem_conv0_weight"].shape[1]),
                policy_channels=P, channels=channels, kernels=kernels, se_types=se_types, se_gates=se_gates, c_ops=c_ops,
                wdl=value_head is not None, value_channels=vc, value_fc=fc, stem_act=stem_act,
                policy_bias="policy_conv1_bias" in params)
    if value_head is not None:
        arch["value_head"] = value_head
    # select_policy_from_plane=False (builder_util_symbol.py policy_head): policy_bn1, the activation, Flatten, policy_out
    bn1 = g.first(pc1[2][0], "BatchNorm")
    if bn1 is None and g.downstream(pc1[2][0], ("FullyConnected",)) is not None:
        g.fail("policy head: no BatchNorm (policy_bn1) between the last policy convolution and its activation")
    if bn1 is not None:
        out = g.fwd(relu_out(bn1), "FullyConnected")
        if len(out) != 1:
            g.fail("policy head: a BatchNorm behind the last policy convolution but no fully-connected layer on its "
                   "flattened activation")
        take_bn(bn1, "policy_bn1"), take(out[0], "policy_out")
        L, width = params["policy_out_weight"].shape
        if L not in CLASSIC_LABELS:
            g.fail(f"policy head: a fully-connected layer onto {L} labels (the classic label lists have {CLASSIC_LABELS})")
        if width != P * 64:
            g.fail(f"policy head: the fully-connected layer takes {width} features, not the {P} x 64 of the flattened "
                   f"convolution")
        arch.update(policy_bias=False, n_labels=int(L))  # (the convolution's bias is folded with policy_bn1)
    export_mx_blob(params, arch, blob_path, input_version_of(arch, input_version), eps=eps, fix_gamma=False)
    return arch


def _value_outputs(g, fcs, take, relu_out):
    """the value head's layers behind value_fc0 and its activation (builder_util_symbol.py value_head), the FullyConnected
    nodes fcs there -> None for value_fc1 and tanh; with use_wdl and use_plys_to_end, the WDL layer (3 units) into its
    SoftmaxOutput and value_plys_to_end_fc (1 unit) into a sigmoid, then "mx_wdl" for value = win - loss or "mx_wdl_mlp"
    for the MLP (use_mlp_wdl_ply) value_wdl_ply_fc (8 units), activation, value_fc1, tanh on Concat(probabilities, plies)"""
    attr = lambda nd, k, d=None: nd[3].get(k, d)
    if len(fcs) == 1 and attr(fcs[0], "num_hidden") == 1:
        take(fcs[0], "value_fc1")
        return None
    widths = sorted(attr(nd, "num_hidden") for nd in fcs)
    if widths != [1, 3]:
        g.fail(f"value head: fully-connected layers of {widths} units behind value_fc0 (value_fc1, or the WDL and "
               f"plies-to-end layers)")
    wdl, plys = sorted(fcs, key=lambda nd: -attr(nd, "num_hidden"))
    sm = g.first(wdl[2][0], "SoftmaxOutput")
    sig = g.first(plys[2][0], "Activation")
    if sm is None or sig is None or attr(sig, "act_type") != "sigmoid":
        g.fail("value head: WDL and plies-to-end layers behind value_fc0 without a SoftmaxOutput behind the first or a "
               "sigmoid behind the second")
    take(wdl, "wdl_out"), take(plys, "value_plys_to_end_fc")
    m0 = g.downstream(sm[2][0], ("FullyConnected",))
    if m0 is None:  # value = broadcast_add(-loss, win) of the split probabilities
        if g.downstream(sm[2][0], ("SliceChannel", "split")) is None:
            g.fail("value head: neither win - loss nor a value MLP behind the WDL output")
        return "mx_wdl"
    cat = g.back(m0[1][0], "Concat")
    plys_out = lambda t: t == sig[2][0] or (g.prod.get(t, ("",))[0] == "LinearRegressionOutput" and g.prod[t][1][0] == sig[2][0])
    if len(cat[1]) != 2 or cat[1][0] != sm[2][0] or not plys_out(cat[1][1]):
        g.fail("value head: the value MLP does not take Concat(WDL probabilities, plies)")
    m1 = g.one(relu_out(m0), "FullyConnected")
    tanh = g.first(m1[2][0], "Activation")
    if attr(m1, "num_hidden") != 1 or tanh is None or attr(tanh, "act_type") != "tanh":
        g.fail("value head: the value MLP does not end in one unit and tanh")
    take(m0, "value_wdl_ply_fc"), take(m1, "value_fc1")
    return "mx_wdl_mlp"


def _se(g, mul, x, i, take, p, n_eca):
    """block i's squeeze-excitation, the multiplication mul of the block input x with its gate -> (se type, gate);
    ca_se (pooling, FullyConnected, activation, FullyConnected) or eca_se (global pooling, a 1-D Convolution over the
    channels).  The spatial and max-pooling flavours are refused."""
    ins = [t for t in mul[1] if t != x]
    if len(ins) != 1:
        inner = next((g.prod[t] for t in mul[1] if t in g.prod and g.prod[t][0] in _MUL), None)
        g.fail(f"block {i}: {'cbam' if inner is not None else 'a squeeze-excitation not on the block input'}: no blob "
               f"format holds it")
    gate = g.back(ins[0], "Activation", "hard_sigmoid")
    if gate[0] == "hard_sigmoid":
        alpha, beta = gate[3].get("alpha", 0.2), gate[3].get("beta", 0.5)
        if abs(alpha - 0.2) > 1e-6 or abs(beta - 0.5) > 1e-6:
            g.fail(f"block {i}: hard_sigmoid alpha {alpha} beta {beta}")
        kind = "hard_sigmoid"
    elif gate[3].get("act_type") == "sigmoid":
        kind = "sigmoid"
    else:
        g.fail(f"block {i}: squeeze-excitation gate {gate[3].get('act_type')}")
    src = g.back(gate[1][0], "FullyConnected", "Convolution")
    if src[0] == "Convolution":
        k = tuple(src[3].get("kernel", ()))
        if len(k) != 1:  # spatial attention: a 7x7 convolution over the channel mean (sa_se) or max (sm_se)
            red = g.back(src[1][0], "mean", "max", "Concat")
            g.fail(f"block {i}: {dict(mean='sa_se', max='sm_se').get(red[0], 'cbam')}: no blob format holds it")
        pool = g.back(src[1][0], "Pooling")
        if pool[1][0] != x or pool[3].get("pool_type") != "avg":
            g.fail(f"block {i}: the 1-D squeeze-excitation convolution does not take the average of the block input")
        take(src, f"convolution{n_eca}")
        return "eca_se", kind
    act = g.back(src[1][0], "Activation")
    fc0 = g.back(act[1][0], "FullyConnected")
    pool = g.back(fc0[1][0], "Pooling", "Concat")
    if pool[0] == "Concat":
        g.fail(f"block {i}: cbam (average and max pooling): no blob format holds it")
    if pool[3].get("pool_type") == "max":
        g.fail(f"block {i}: cm_se (max pooling): no blob format holds it")
    if pool[1][0] != x or pool[3].get("pool_type") != "avg" or act[3].get("act_type") != "relu":
        g.fail(f"block {i}: not a ca_se on the block input")
    take(fc0, p + "_se_fc0"), take(src, p + "_se_fc1")
    return "ca_se", kind


# ---------------------------------------------------------------------------------------------- entry points
def import_mxnet(symbol_path, params_path, blob_path, input_version=None, channels=256):
    """an MXNet model (`-symbol.json` and `.params`) -> blob at blob_path; returns the arch, as onnx_import.import_onnx"""
    nodes, variables = read_symbol(symbol_path)
    return _import_symbol(_Graph(symbol_path, nodes, {}, _SKIP), variables, read_params(params_path), blob_path,
                          input_version, channels)


def model_files(model_dir):
    """the symbol and parameter files of a model directory as the reference's MXNet back-end picks them (mxnetapi.cpp
    fill_model_paths, float32): the one file ending with .json and the one ending with .params, names containing int8
    skipped"""
    files = sorted(f for f in os.listdir(model_dir) if "int8" not in f)
    picked = []
    for suffix in (".json", ".params"):
        found = [f for f in files if f.endswith(suffix)]
        if not found:
            raise ValueError(f"The given directory at {model_dir} doesn't contain a file ending with {suffix}")
        if len(found) > 1:
            raise ValueError(f"The given directory at {model_dir} contains more than one file ending with {suffix}: "
                             f"{', '.join(found)}")
        picked.append(os.path.join(model_dir, found[0]))
    return tuple(picked)


if __name__ == "__main__":
    import sys
    args = sys.argv[1:]
    files = model_files(args[0]) if args and os.path.isdir(args[0]) else tuple(args[:2])
    rest = args[1:] if args and os.path.isdir(args[0]) else args[2:]
    if len(files) != 2 or not rest or len(rest) > 2:
        raise SystemExit("usage: python -m crazyara_b200.mx_import <model_dir | model-symbol.json model.params> <out.arab> "
                         "[input_version]")
    a = import_mxnet(*files, rest[0], int(rest[1]) if len(rest) > 1 else None)
    policy = f"{a['n_labels']} labels" if a.get("n_labels") else f"{a['policy_channels']}x64"
    print(f"{rest[0]}: {len(a['kernels'])} blocks, {a['in_channels']} -> {policy}, wdl={a['wdl']}")
