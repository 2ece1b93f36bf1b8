"""Weight import from the reference's ONNX artefacts (SURVEY §8 f3): `<prefix>-v<version>[-bsize-<n>].onnx` as written by
`export_to_onnx` (DeepCrazyhouse/src/training/trainer_agent_pytorch.py:588-650: torch.onnx.export in eval mode, then
onnx-simplifier -- BatchNorm folded into the convolutions) -> ARAB2001 blob for ara_net_create.

No `onnx` package is needed (the image has none): the file is read with a minimal protobuf wire-format reader, only the
fields this import uses (graph.node: op_type, inputs, attributes `group` / `transB`; graph.initializer: dims, data type,
raw / float / int64 data).  The graph is not executed; the network structure is the RISE family's and is recovered from
the ORDER of its Conv / Gemm / MatMul nodes (a torch export lists them in execution order):

    stem conv3x3 | per block: [SE: Gemm, Gemm  or  eca Conv1d] conv1x1, depthwise kxk (group = channels), conv1x1 |
    value head: conv1x1, Gemm(s) | policy head: conv3x3, conv3x3

PARITY UNPINNED: /root/reference holds no .onnx file and the `onnx` / `onnxsim` packages are absent, so this reader is
checked against files written by tests/onnx_writer.py (same node kinds and tensor layouts as the torch exporter emits for
these modules), not against an artefact of the reference itself.

A graph exported from the reference's MXNet symbols (`convert_to_onnx.py`) computes another network from the same
layers (crazyara_b200/weights.py, export_mx_blob).  It is recognised by its unfolded `BatchNormalization` nodes and read by
graph edges, not node order: from the stem, each block is the `Add` fed by the block input, traced back through
BatchNormalization / Relu / Conv to its first convolution, whose input is the block input itself or a `Mul` of it with a
squeeze-excitation gate (`Sigmoid`, or `HardSigmoid` with its alpha; behind it a 1-D `Conv` over the channels for eca_se,
or two `Gemm` with biases for ca_se).  The layers go, under the names the symbol code gives them, through export_mx_blob
into an ARAB2002 blob.  PARITY UNPINNED as well: no MXNet export is in either tree; the reader is checked against files
written by tests/onnx_mx_writer.py.
"""
import struct
from collections import defaultdict

import numpy as np

from .weights import SE_CODE, export_mx_blob, write_blob


# ---------------------------------------------------------------------------------------------- protobuf wire format
def _varint(buf, i):
    r, s = 0, 0
    while True:
        b = buf[i]
        i += 1
        r |= (b & 0x7F) << s
        if not b & 0x80:
            return r, i
        s += 7


def _fields(buf):
    """yields (field number, wire type, value) of one message; length-delimited values as memoryview slices"""
    i, n = 0, len(buf)
    while i < n:
        key, i = _varint(buf, i)
        f, w = key >> 3, key & 7
        if w == 0:
            v, i = _varint(buf, i)
        elif w == 1:
            v, i = bytes(buf[i:i + 8]), i + 8
        elif w == 2:
            ln, i = _varint(buf, i)
            v, i = buf[i:i + ln], i + ln
        elif w == 5:
            v, i = bytes(buf[i:i + 4]), i + 4
        else:
            raise ValueError(f"unsupported protobuf wire type {w}")
        yield f, w, v


def _packed_varints(v):
    out, i = [], 0
    while i < len(v):
        x, i = _varint(v, i)
        out.append(x)
    return out


def _tensor(buf):
    """TensorProto -> (name, ndarray float32)"""
    dims, dtype, name, raw, floats, int64s = [], 1, "", None, [], []
    for f, w, v in _fields(buf):
        if f == 1:
            dims += _packed_varints(v) if w == 2 else [v]
        elif f == 2:
            dtype = v
        elif f == 8:
            name = bytes(v).decode()
        elif f == 9:
            raw = bytes(v)
        elif f == 4:
            floats += list(struct.unpack(f"<{len(v) // 4}f", bytes(v))) if w == 2 else [struct.unpack("<f", v)[0]]
        elif f == 7:
            int64s += _packed_varints(v) if w == 2 else [v]
    if dtype == 1:
        a = np.frombuffer(raw, dtype="<f4") if raw is not None else np.asarray(floats, np.float32)
    elif dtype == 10:
        a = np.frombuffer(raw, dtype="<f2").astype(np.float32)
    elif dtype == 11:
        a = np.frombuffer(raw, dtype="<f8").astype(np.float32)
    elif dtype == 7:
        a = (np.frombuffer(raw, dtype="<i8") if raw is not None else np.asarray(int64s, np.int64)).astype(np.float32)
    else:
        return name, None
    return name, np.array(a, dtype=np.float32).reshape(dims if dims else ())


def read_graph(path):
    """-> (nodes [(op_type, inputs, outputs, {attr: int})], initializers {name: ndarray})"""
    model = memoryview(open(path, "rb").read())
    graph = next((v for f, w, v in _fields(model) if f == 7 and w == 2), None)
    if graph is None:
        raise ValueError(f"{path}: no graph in the ONNX model")
    nodes, inits = [], {}
    for f, w, v in _fields(graph):
        if f == 1:
            op, ins, outs, attrs = "", [], [], {}
            for g, gw, gv in _fields(v):
                if g == 1:
                    ins.append(bytes(gv).decode())
                elif g == 2:
                    outs.append(bytes(gv).decode())
                elif g == 4:
                    op = bytes(gv).decode()
                elif g == 5:
                    an, ai, at = "", None, None
                    for h, hw, hv in _fields(gv):
                        if h == 1:
                            an = bytes(hv).decode()
                        elif h == 2 and hw == 5:
                            ai = struct.unpack("<f", hv)[0]  # a float attribute (epsilon, alpha)
                        elif h == 3:
                            ai = hv
                        elif h == 5 and hw == 2:
                            at = hv  # a tensor attribute (Constant nodes)
                    if ai is not None:
                        attrs[an] = ai
                    if at is not None:
                        attrs[an] = _tensor(at)[1]
            nodes.append((op, ins, outs, attrs))
        elif f == 5:
            name, a = _tensor(v)
            if a is not None:
                inits[name] = a
    for op, ins, outs, attrs in nodes:  # weights kept as Constant nodes instead of initializers
        if op == "Constant" and outs and isinstance(attrs.get("value"), np.ndarray):
            inits[outs[0]] = attrs["value"]
    return nodes, inits


# ---------------------------------------------------------------------------------------------- graph -> blob
def import_onnx(onnx_path, blob_path, input_version=None, channels=256):
    nodes, inits = read_graph(onnx_path)
    if any(nd[0] == "BatchNormalization" for nd in nodes):
        return _import_mxnet_graph(onnx_path, nodes, inits, blob_path, input_version, channels)
    order = []  # convolutions and fully-connected layers in execution order
    for op, ins, outs, attrs in nodes:
        if op == "Conv" and len(ins) >= 2 and ins[1] in inits:
            w = inits[ins[1]]
            b = inits[ins[2]] if len(ins) > 2 and ins[2] in inits else np.zeros(w.shape[0], np.float32)
            order.append(("conv", w, b, int(attrs.get("group", 1))))
        elif op in ("Gemm", "MatMul") and len(ins) >= 2 and ins[1] in inits:
            w = inits[ins[1]]
            if op == "MatMul" or not attrs.get("transB", 0):
                w = w.T  # -> [out, in], the layout of torch.nn.Linear.weight
            b = inits[ins[2]] if len(ins) > 2 and ins[2] in inits else np.zeros(w.shape[0], np.float32)
            order.append(("fc", np.ascontiguousarray(w), b, 1))
    if not order or order[0][0] != "conv" or order[0][1].ndim != 4 or order[0][1].shape[2] != 3:
        raise ValueError(f"{onnx_path}: does not start with a 3x3 stem convolution")
    tensors = []
    put = lambda a: tensors.append(np.ascontiguousarray(a, dtype=np.float32).reshape(-1))
    stem_w, stem_b = order[0][1], order[0][2]
    C = stem_w.shape[0]
    if C != channels:
        raise ValueError(f"{onnx_path}: {C} trunk channels, this engine builds {channels}")
    put(stem_w), put(stem_b)
    i, kernels, se_types, c_ops = 1, [], [], []
    while True:
        # squeeze-excitation layers in front of the block (they act on its input)
        se, j = None, i
        fcs = []
        while j < len(order) and (order[j][0] == "fc" or (order[j][0] == "conv" and order[j][1].ndim == 3)):
            fcs.append(order[j])
            j += 1
        # a block = conv1x1 (C -> Cop), depthwise kxk, conv1x1 (Cop -> C)
        if not (j + 2 < len(order) and order[j][0] == "conv" and order[j][1].ndim == 4 and order[j][1].shape[2] == 1 and
                order[j + 1][0] == "conv" and order[j + 1][3] == order[j + 1][1].shape[0] and order[j + 1][3] > 1):
            break
        if fcs:
            if len(fcs) == 2 and fcs[0][0] == "fc":
                se = "ca_se"
                put(fcs[0][1]), put(fcs[1][1])  # (the reference's SE FCs have no bias, builder_util.py:100-116)
            elif len(fcs) == 1 and fcs[0][1].ndim == 3:
                se = "eca_se"
                wc = fcs[0][1]
                put(wc[:, :, wc.shape[2] // 2]), put(fcs[0][2])
            else:
                raise ValueError(f"{onnx_path}: unrecognised squeeze-excitation pattern in front of block {len(kernels)}")
        w1, b1, _ = order[j][1:]
        wd, bd, _ = order[j + 1][1:]
        w2, b2, _ = order[j + 2][1:]
        cop, k = w1.shape[0], wd.shape[2]
        if w1.shape[1] != C or wd.shape[0] != cop or w2.shape[:2] != (C, cop) or k not in (3, 5):
            raise ValueError(f"{onnx_path}: block {len(kernels)} is not a RISE bottleneck block")
        put(w1), put(b1), put(wd), put(bd), put(w2), put(b2)
        kernels.append(int(k)), se_types.append(se), c_ops.append(int(cop))
        i = j + 3
    if not kernels:
        raise ValueError(f"{onnx_path}: no bottleneck block found")
    # value head: conv1x1 (C -> 8) + FC layers; policy head: conv3x3 (C -> C), conv3x3 (C -> P)
    rest = order[i:]
    vconv = [r for r in rest if r[0] == "conv" and r[1].ndim == 4 and r[1].shape[2] == 1]
    heads = [r for r in rest if r[0] == "conv" and r[1].ndim == 4 and r[1].shape[2] == 3]
    fcs = [r for r in rest if r[0] == "fc"]
    if len(vconv) != 1 or vconv[0][1].shape[1] != C:
        raise ValueError(f"{onnx_path}: value head (one 1x1 convolution) not found behind the tower")
    if len(heads) != 2 or heads[0][1].shape[:2] != (C, C) or heads[1][1].shape[1] != C:
        raise ValueError(f"{onnx_path}: policy head (two 3x3 convolutions) not found behind the tower")
    put(vconv[0][1]), put(vconv[0][2])
    # value head variants (builder_util.py:246-330): FC 512 -> 256 -> 1 (tanh), or the WDL head FC -> 3 with the plies FC -> 1
    wdl = len(fcs) == 2 and fcs[0][1].shape[0] == 3
    if wdl:
        put(fcs[0][1]), put(fcs[0][2]), put(fcs[1][1]), put(fcs[1][2])
    elif len(fcs) == 2:
        put(fcs[0][1]), put(fcs[0][2]), put(fcs[1][1]), put(fcs[1][2])
    else:
        raise ValueError(f"{onnx_path}: {len(fcs)} fully-connected layers in the value head (expected 2)")
    put(heads[0][1]), put(heads[0][2])
    put(heads[1][1])
    arch = dict(name=f"rise_{len(kernels)}b", in_channels=int(stem_w.shape[1]), policy_channels=int(heads[1][1].shape[0]),
                channels=int(C), kernels=kernels, se_types=se_types, c_ops=c_ops, wdl=bool(wdl), value_channels=int(vconv[0][1].shape[0]),
                value_fc=256)
    write_blob(blob_path, arch, tensors, _input_version(arch, input_version))
    return arch


def _input_version(arch, input_version):
    if input_version is not None:
        return input_version
    return {34: 10, 63: 10, 39: 10, 51: 20, 52: 30, 64: 30, 80: 30}.get(arch["in_channels"], 10)


def _import_mxnet_graph(onnx_path, nodes, inits, blob_path, input_version, channels):
    """a graph with unfolded BatchNormalization nodes (an MXNet export), read by its edges -> ARAB2002 blob"""
    prod, cons = {}, defaultdict(list)
    for nd in nodes:
        for o in nd[2]:
            prod[o] = nd
        for i in nd[1]:
            cons[i].append(nd)

    def fail(what):
        raise ValueError(f"{onnx_path}: {what}")

    def back(t, *ops):  # the producer of t, skipping shape-only nodes, which must be one of ops
        nd = prod.get(t)
        while nd is not None and nd[0] in ("Reshape", "Flatten", "Squeeze", "Unsqueeze", "Identity"):
            nd = prod.get(nd[1][0])
        if nd is None or nd[0] not in ops:
            fail(f"expected {'/'.join(ops)} in front of '{t}', found {nd[0] if nd else 'a graph input'}")
        return nd

    def fwd(t, op):  # the consumer of t with type op, or None
        return next((nd for nd in cons[t] if nd[0] == op), None)

    params, eps = {}, {}

    def take_bn(nd, name):
        for key, i in (("gamma", 1), ("beta", 2), ("moving_mean", 3), ("moving_var", 4)):
            params[f"{name}_{key}"] = inits[nd[1][i]]
        eps[name] = float(nd[3].get("epsilon", 1e-5))  # (ONNX's default)

    def take(nd, name):  # Conv / Gemm weights and bias under the MXNet layer name
        w = inits[nd[1][1]]
        if nd[0] == "Gemm" and not nd[3].get("transB", 0):
            w = w.T
        params[name + "_weight"] = np.ascontiguousarray(w)
        if len(nd[1]) > 2 and nd[1][2] in inits:
            params[name + "_bias"] = inits[nd[1][2]]

    def conv_bn(t, name):  # t = output of Conv -> BatchNormalization: the Conv node
        bn = back(t, "BatchNormalization")
        conv = back(bn[1][0], "Conv")
        take(conv, name)
        take_bn(bn, name.replace("conv", "bn"))
        return conv

    stem = next((nd for nd in nodes if nd[0] == "Conv" and nd[1][0] not in prod and nd[1][0] not in inits), None)
    if stem is None or inits[stem[1][1]].shape[0] != channels or inits[stem[1][1]].shape[2] != 3:
        fail(f"no 3x3 stem convolution with {channels} channels on the graph input")
    take(stem, "stem_conv0")
    bn = fwd(stem[2][0], "BatchNormalization")
    if bn is None:
        fail("no BatchNormalization behind the stem")
    take_bn(bn, "stem_bn0")
    relu = fwd(bn[2][0], "Relu")
    x, stem_act = (relu[2][0], True) if relu is not None and fwd(relu[2][0], "Add") is not None else (bn[2][0], False)
    kernels, se_types, se_gates, c_ops, n_eca = [], [], [], [], 0
    while True:
        add = next((nd for nd in cons[x] if nd[0] == "Add" and len(nd[1]) == 2), None)
        if add is None:
            break
        i, p = len(kernels), f"bc_res_block{len(kernels)}"
        other = add[1][1] if add[1][0] == x else add[1][0]
        conv3 = conv_bn(other, p + "_conv3")
        conv2 = conv_bn(back(conv3[1][0], "Relu")[1][0], p + "_conv2")
        conv1 = conv_bn(back(conv2[1][0], "Relu")[1][0], p + "_conv1")
        w1, wd = params[p + "_conv1_weight"], params[p + "_conv2_weight"]
        if w1.shape[1] != channels or wd.shape[0] != w1.shape[0] or wd.shape[2] not in (3, 5):
            fail(f"block {i} is not a RISE bottleneck block")
        se, gate = None, None
        if conv1[1][0] != x:
            mul = back(conv1[1][0], "Mul")
            if x not in mul[1]:
                fail(f"block {i}: the squeeze-excitation does not act on the block input")
            g = back(mul[1][1] if mul[1][0] == x else mul[1][0], "Sigmoid", "HardSigmoid")
            if g[0] == "Sigmoid":
                gate = "sigmoid"
            elif abs(g[3].get("alpha", 0.2) - 0.2) < 1e-6 and abs(g[3].get("beta", 0.5) - 0.5) < 1e-6:
                gate = "hard_sigmoid"
            else:
                fail(f"block {i}: HardSigmoid alpha {g[3].get('alpha')} beta {g[3].get('beta')}")
            fc = back(g[1][0], "Gemm", "MatMul", "Conv")
            if fc[0] == "Conv":
                se = "eca_se"
                take(fc, f"convolution{n_eca}")
                n_eca += 1
            else:
                se = "ca_se"
                take(fc, p + "_se_fc1")
                take(back(back(fc[1][0], "Relu")[1][0], "Gemm", "MatMul"), p + "_se_fc0")
        kernels.append(int(wd.shape[2])), se_types.append(se), se_gates.append(gate), c_ops.append(int(w1.shape[0]))
        x = add[2][0]
    if not kernels:
        fail("no bottleneck block found")
    heads = [nd for nd in cons[x] if nd[0] == "Conv"]
    vconv = [nd for nd in heads if inits[nd[1][1]].shape[2] == 1]
    pconv = [nd for nd in heads if inits[nd[1][1]].shape[2] == 3]
    if len(vconv) != 1 or len(pconv) != 1:
        fail("value head (1x1 convolution) and policy head (3x3 convolution) not found behind the tower")
    take(vconv[0], "value_conv0")
    take_bn(fwd(vconv[0][2][0], "BatchNormalization"), "value_bn0")
    g0 = _downstream(cons, vconv[0][2][0], ("Gemm", "MatMul"))
    g1 = g0 and _downstream(cons, g0[2][0], ("Gemm", "MatMul"))
    if g1 is None:
        fail("value head: two fully-connected layers not found")
    take(g0, "value_fc0"), take(g1, "value_fc1")
    take(pconv[0], "policy_conv0")
    take_bn(fwd(pconv[0][2][0], "BatchNormalization"), "policy_bn0")
    take(_downstream(cons, pconv[0][2][0], ("Conv",)), "policy_conv1")
    arch = dict(name=f"rise_{len(kernels)}b", semantics="mxnet", in_channels=int(inits[stem[1][1]].shape[1]),
                policy_channels=int(params["policy_conv1_weight"].shape[0]), channels=channels, kernels=kernels,
                se_types=se_types, se_gates=se_gates, c_ops=c_ops, wdl=False, value_channels=int(params["value_conv0_weight"].shape[0]),
                value_fc=256, stem_act=stem_act, policy_bias="policy_conv1_bias" in params)
    export_mx_blob(params, arch, blob_path, _input_version(arch, input_version), eps=eps, fix_gamma=False)
    return arch


def _downstream(cons, t, ops):
    """the first node of one of ops reached from tensor t along single-consumer element-wise edges"""
    seen = set()
    frontier = [t]
    while frontier:
        nxt = []
        for u in frontier:
            for nd in cons[u]:
                if nd[0] in ops:
                    return nd
                if id(nd) not in seen:
                    seen.add(id(nd))
                    nxt += nd[2]
        frontier = nxt
    return None


if __name__ == "__main__":
    import sys
    if len(sys.argv) < 3:
        raise SystemExit("usage: python -m crazyara_b200.onnx_import <model.onnx> <out.arab> [input_version]")
    a = import_onnx(sys.argv[1], sys.argv[2], int(sys.argv[3]) if len(sys.argv) > 3 else None)
    print(f"{sys.argv[2]}: {len(a['kernels'])} blocks, {a['in_channels']} -> {a['policy_channels']}x64, wdl={a['wdl']}")
