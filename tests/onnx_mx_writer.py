"""Writes a RISE network of the reference's MXNet symbols as an ONNX graph the way an MXNet export leaves it, for
tests/test_onnx_mx_import.py: unfolded BatchNormalization nodes (epsilon attribute, gamma written as ones where the symbol
fixes it), FullyConnected as Gemm with transB = 1 and bias, the squeeze-excitation as Mul of the block input with its gate
(Sigmoid, or HardSigmoid with alpha 0.2 / beta 0.5; eca_se a 1-D Conv between Reshape nodes) and the shortcut as Add of the
block's last BatchNormalization and the block input.  The node list is shuffled: the importer must follow the edges."""
import struct

import numpy as np

from crazyara_b200.weights import mx_bn_prefix, mx_eca_names
from tests.onnx_writer import _ld, _node, _tensor, _varint, _vi


def _fnode(op, ins, outs, fattrs):
    msg = _node(op, ins, outs)
    for name, val in fattrs:  # float attributes: AttributeProto.f (field 2), type FLOAT (1)
        msg += _ld(5, _ld(1, name.encode()) + _varint(2 << 3 | 5) + struct.pack("<f", val) + _vi(20, 1))
    return msg


def write_mx_onnx(params, arch, path, eps=1e-3, seed=0):
    nodes, inits, n = [], [], [0]

    def new():
        n[0] += 1
        return f"t_{n[0]}"

    def init(name, a):
        inits.append(_tensor(name, a))
        return name

    def conv(x, name, group=1):
        y = new()
        ins = [x, init(name + "_weight", params[name + "_weight"])]
        if name + "_bias" in params:
            ins.append(init(name + "_bias", params[name + "_bias"]))
        nodes.append(_node("Conv", ins, [y], [("group", group)]))
        return y

    def bn(x, name):
        name = mx_bn_prefix(params, name)
        y = new()
        c = params[name + "_beta"].size
        ins = [x, init(name + "_gamma", np.ones(c, np.float32)), init(name + "_beta", params[name + "_beta"]),
               init(name + "_moving_mean", params[name + "_moving_mean"]), init(name + "_moving_var", params[name + "_moving_var"])]
        nodes.append(_fnode("BatchNormalization", ins, [y], [("epsilon", eps)]))
        return y

    def op(kind, *xs, fattrs=()):
        y = new()
        nodes.append(_fnode(kind, list(xs), [y], fattrs))
        return y

    def gemm(x, name):
        y = new()
        nodes.append(_node("Gemm", [x, init(name + "_weight", params[name + "_weight"]), init(name + "_bias", params[name + "_bias"])],
                           [y], [("transB", 1)]))
        return y

    def gate(x, g):
        return op("Sigmoid", x) if g == "sigmoid" else op("HardSigmoid", x, fattrs=[("alpha", 0.2), ("beta", 0.5)])

    x = bn(conv("data", "stem_conv0"), "stem_bn0")
    if arch["stem_act"]:
        x = op("Relu", x)
    eca = iter(mx_eca_names(params))
    for i, (k, se, cop) in enumerate(zip(arch["kernels"], arch["se_types"], arch["c_ops"])):
        p = f"bc_res_block{i}"
        xin = x
        if se == "ca_se":
            g = op("Flatten", op("GlobalAveragePool", x))
            g = gate(gemm(op("Relu", gemm(g, p + "_se_fc0")), p + "_se_fc1"), arch["se_gates"][i])
            xin = op("Mul", x, op("Reshape", g))
        elif se == "eca_se":
            g = op("Reshape", op("GlobalAveragePool", x))
            xin = op("Mul", x, op("Reshape", gate(conv(g, next(eca)), arch["se_gates"][i])))
        y = op("Relu", bn(conv(xin, p + "_conv1"), p + "_bn1"))
        y = op("Relu", bn(conv(y, p + "_conv2", group=cop), p + "_bn2"))
        y = bn(conv(y, p + "_conv3"), p + "_bn3")
        x = op("Add", y, x)
    v = op("Flatten", op("Relu", bn(conv(x, "value_conv0"), "value_bn0")))
    op("Tanh", gemm(op("Relu", gemm(v, "value_fc0")), "value_fc1"))
    y = op("Relu", bn(conv(x, "policy_conv0"), "policy_bn0"))
    op("Softmax", op("Flatten", conv(y, "policy_conv1")))
    order = np.random.default_rng(seed).permutation(len(nodes))
    graph = b"".join(_ld(1, nodes[j]) for j in order) + _ld(2, b"mxnet_converted_model") + b"".join(_ld(5, t) for t in inits)
    with open(path, "wb") as f:
        f.write(_vi(1, 8) + _ld(2, b"mxnet2onnx") + _ld(7, graph))
    return path
