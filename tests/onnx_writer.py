"""A minimal ONNX (protobuf) writer for tests/test_onnx_import.py: a RISE network as torch.onnx.export + onnx-simplifier
leave it (BatchNorm folded into the convolutions, Linear layers as Gemm with transB = 1, weights as initializers with raw
float32 data), from a reference-style state_dict.  Only what the importer reads has to be exact; the element-wise nodes
in between (Relu, Add, Mul, GlobalAveragePool, ...) are written too so that the node list looks like a real export."""
import struct

import numpy as np

from crazyara_b200.weights import _fold, _np


def _varint(x):
    out = bytearray()
    while True:
        b = x & 0x7F
        x >>= 7
        out.append(b | (0x80 if x else 0))
        if not x:
            return bytes(out)


def _ld(field, payload):
    return _varint(field << 3 | 2) + _varint(len(payload)) + payload


def _vi(field, x):
    return _varint(field << 3 | 0) + _varint(x)


def _tensor(name, a):
    a = np.ascontiguousarray(a, dtype=np.float32)
    msg = b"".join(_vi(1, d) for d in a.shape) + _vi(2, 1) + _ld(8, name.encode()) + _ld(9, a.tobytes())
    return msg


def _node(op, ins, outs, attrs=()):
    msg = b"".join(_ld(1, i.encode()) for i in ins) + b"".join(_ld(2, o.encode()) for o in outs) + _ld(4, op.encode())
    for name, val in attrs:  # integer attributes only
        msg += _ld(5, _ld(1, name.encode()) + _vi(3, val) + _vi(20, 2))
    return msg


def write_rise_onnx(sd, arch, path, shuffle=None, torch_se=False):
    """shuffle: a seed to write the nodes in a random order, as tests/onnx_mx_writer.py does; torch_se: the
    squeeze-excitation as torch.onnx.export writes the reference's modules (builder_util.py:86-116), the pooled vector
    reshaped rather than flattened and the gate broadcast by view() and expand_as(x): GlobalAveragePool -> Reshape, gate ->
    Reshape -> Expand -> Mul"""
    nodes, inits, n = [], [], [0]

    def const(a):
        n[0] += 1
        name = f"onnx::w_{n[0]}"
        inits.append(_tensor(name, a))
        return name

    def conv(x, w, b, group=1):
        n[0] += 1
        y = f"t_{n[0]}"
        ins = [x, const(w)] + ([const(b)] if b is not None else [])
        nodes.append(_node("Conv", ins, [y], [("group", group)]))
        return y

    def unary(op, x):
        n[0] += 1
        y = f"t_{n[0]}"
        nodes.append(_node(op, [x], [y]))
        return y

    def gemm(x, w, b):
        n[0] += 1
        y = f"t_{n[0]}"
        ins = [x, const(w)] + ([const(b)] if b is not None else [])
        nodes.append(_node("Gemm", ins, [y], [("transB", 1)]))
        return y

    f32 = lambda a: np.asarray(a, np.float32)
    w, b = _fold(sd, "body_spatial.0.body.0.weight", "body_spatial.0.body.1")
    x = unary("Relu", conv("data", f32(w), f32(b)))
    for i, (k, se, cop) in enumerate(zip(arch["kernels"], arch["se_types"], arch["c_ops"])):
        p = f"body_spatial.{i + 1}"
        xin = x
        if se in ("ca_se", "se"):
            g = unary("Reshape" if torch_se else "Flatten", unary("GlobalAveragePool", x))
            g = unary("Relu", gemm(g, f32(_np(sd[p + ".se.fc.0.weight"])), None))
            g = unary("HardSigmoid", gemm(g, f32(_np(sd[p + ".se.fc.2.weight"])), None))
        elif se == "eca_se":
            g = unary("GlobalAveragePool", x)
            g = unary("HardSigmoid", conv(unary("Reshape", g), f32(_np(sd[p + ".se.body.0.weight"])), f32(_np(sd[p + ".se.body.0.bias"]))))
        if se:
            if torch_se:
                ins = [unary("Reshape", g), unary("Shape", x)]
                n[0] += 1
                nodes.append(_node("Expand", ins, [f"t_{n[0]}"]))
                g = f"t_{n[0]}"
            n[0] += 1
            nodes.append(_node("Mul", [x, g], [f"t_{n[0]}"]))
            xin = f"t_{n[0]}"
        w, b = _fold(sd, p + ".body.0.weight", p + ".body.1")
        y = unary("Relu", conv(xin, f32(w), f32(b)))
        w, b = _fold(sd, p + ".body.3.weight", p + ".body.4")
        y = unary("Relu", conv(y, f32(w), f32(b), group=cop))
        w, b = _fold(sd, p + ".body.6.weight", p + ".body.7")
        y = conv(y, f32(w), f32(b))
        n[0] += 1
        nodes.append(_node("Add", [xin, y], [f"t_{n[0]}"]))
        x = f"t_{n[0]}"
    w, b = _fold(sd, "value_head.body.0.weight", "value_head.body.1")
    v = unary("Flatten", unary("Relu", conv(x, f32(w), f32(b))))
    if arch["wdl"]:
        gemm(v, f32(_np(sd["value_head.body_wdl.0.weight"])), f32(_np(sd["value_head.body_wdl.0.bias"])))
        gemm(v, f32(_np(sd["value_head.body_plys.0.weight"])), f32(_np(sd["value_head.body_plys.0.bias"])))
    else:
        v = unary("Relu", gemm(v, f32(_np(sd["value_head.body_final.0.weight"])), f32(_np(sd["value_head.body_final.0.bias"]))))
        unary("Tanh", gemm(v, f32(_np(sd["value_head.body_final.2.weight"])), f32(_np(sd["value_head.body_final.2.bias"]))))
    w, b = _fold(sd, "policy_head.body.0.weight", "policy_head.body.1")
    y = unary("Relu", conv(x, f32(w), f32(b)))
    unary("Flatten", conv(y, f32(_np(sd["policy_head.body.3.weight"])), None))
    if shuffle is not None:
        nodes = [nodes[j] for j in np.random.default_rng(shuffle).permutation(len(nodes))]
    graph = b"".join(_ld(1, nd) for nd in nodes) + _ld(2, b"torch_jit") + b"".join(_ld(5, t) for t in inits)
    model = _vi(1, 8) + _ld(2, b"pytorch") + _ld(7, graph)
    with open(path, "wb") as f:
        f.write(model)
    return path


def add_shape_concat(path):
    """rewrites the file with the shape arithmetic of a dynamic-batch export in front of a view(): Shape -> Gather ->
    Unsqueeze -> Concat (with a constant) -> Reshape of the stem's output, the Concat taking no activation"""
    from crazyara_b200.onnx_import import _fields
    model = memoryview(open(path, "rb").read())
    out = b""
    for f, w, v in _fields(model):
        if f == 7:
            first = next(bytes(nv) for nf, nw, nv in _fields(v) if nf == 1)
            x = next(bytes(gv).decode() for g, gw, gv in _fields(memoryview(first)) if g == 2)  # the stem's output
            extra = [_node("Shape", [x], ["s_shape"]), _node("Gather", ["s_shape", "s_idx"], ["s_b"]),
                     _node("Unsqueeze", ["s_b"], ["s_bu"]), _node("Concat", ["s_bu", "s_tail"], ["s_new"], [("axis", 0)]),
                     _node("Reshape", [x, "s_new"], ["s_view"])]
            consts = [_tensor("s_idx", np.zeros(1, np.float32)), _tensor("s_tail", np.array([256, 1], np.float32))]
            v = bytes(v) + b"".join(_ld(1, nd) for nd in extra) + b"".join(_ld(5, t) for t in consts)
        out += _vi(f, v) if w == 0 else _ld(f, bytes(v))
    open(path, "wb").write(out)
    return path
