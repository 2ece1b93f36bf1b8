"""Fully-connected policy heads (the trainer's select_policy_from_plane=False) for the ONNX files the test writers make
(tests/onnx_writer.py, tests/onnx_alphavile_writer.py, tests/onnx_mx_writer.py), for tests/test_onnx_classic_import.py.
Those writers end the policy head in `Flatten` of the last policy convolution (a policy map); the functions here rewrite
such a file with the head in its place, and leave everything else in the file as the writer made it.

- add_torch_head: as torch.onnx.export + onnx-simplifier leave builder_util.py _PolicyHead (:206-243) -- body2's BatchNorm
  folded into the last convolution, which gains a bias, then Relu, the flatten of `.view(-1, nb_flatten)` (`Flatten`, or
  `Reshape` with an int64 shape initialiser) and body3's Linear (`Gemm` with transB 1 or 0, or `MatMul` + `Add`), and
  optionally the `Softmax` of the backend.
- add_mx_head: as an MXNet export leaves builder_util_symbol.py policy_head (:189-223) -- `BatchNormalization`
  policy_bn1 (epsilon attribute, gamma written as ones), `Relu` policy_act1, `Flatten` policy_flatten0, `Gemm` policy_out
  (transB 1, with bias) and the `Softmax` of SoftmaxOutput.

PARITY UNPINNED, as for the writers: no exporter runs here, so the layouts are the ones those exporters document."""
import numpy as np

from crazyara_b200.onnx_import import _fields
from crazyara_b200.weights import _fold, _np
from tests.onnx_mx_writer import _fnode
from tests.onnx_writer import _ld, _node, _tensor, _vi


def _decode(nd):
    ins, outs, op = [], [], ""
    for f, w, v in _fields(memoryview(nd)):
        if f == 1:
            ins.append(bytes(v).decode())
        elif f == 2:
            outs.append(bytes(v).decode())
        elif f == 4:
            op = bytes(v).decode()
    return op, ins, outs


def _rewrite(path, edit, shuffle):
    """edit(nodes [(bytes, op, ins, outs)], inits {name: bytes}) -> (nodes, inits), applied to the graph of the file"""
    model = memoryview(open(path, "rb").read())
    out = b""
    for f, w, v in _fields(model):
        if f == 7:
            nodes, name, inits = [], b"", {}
            for gf, gw, gv in _fields(v):
                if gf == 1:
                    nodes.append((bytes(gv), *_decode(bytes(gv))))
                elif gf == 2:
                    name = bytes(gv)
                elif gf == 5:
                    inits[next(bytes(tv).decode() for tf, tw, tv in _fields(gv) if tf == 8)] = bytes(gv)
            nodes, inits = edit(nodes, inits)
            if shuffle is not None:
                nodes = [nodes[j] for j in np.random.default_rng(shuffle).permutation(len(nodes))]
            v = b"".join(_ld(1, nd[0]) for nd in nodes) + _ld(2, name) + b"".join(_ld(5, t) for t in inits.values())
        out += _vi(f, v) if w == 0 else _ld(f, bytes(v))
    open(path, "wb").write(out)
    return path


def _policy_flatten(nodes):
    """-> (index of the Flatten behind the last policy convolution, index of that Conv node)"""
    prod = {o: i for i, nd in enumerate(nodes) for o in nd[3]}
    for i, (_, op, ins, _) in enumerate(nodes):
        if op == "Flatten" and ins[0] in prod and nodes[prod[ins[0]]][1] == "Conv":
            return i, prod[ins[0]]
    raise AssertionError("no policy-map Flatten in the graph")


def _int64(name, a):
    a = np.ascontiguousarray(a, dtype="<i8")
    return b"".join(_vi(1, d) for d in a.shape) + _vi(2, 7) + _ld(8, name.encode()) + _ld(9, a.tobytes())


def add_torch_head(path, sd, flatten="Flatten", linear="Gemm", trans_b=1, softmax=True, shuffle=None, w_fc=None,
                   relu=True, fc=True):
    """sd: the state_dict the writer was given, with policy_head.body2 / body3 (crazyara_b200.synthetic.classic_head).
    For the refusal tests: w_fc stands in for the Linear's weight, relu=False leaves the Relu out, and fc=False ends the
    head in the flatten, a policy map behind the biased convolution."""
    f32 = lambda a: np.asarray(a, np.float32)
    w2, b2 = _fold(sd, "policy_head.body.3.weight", "policy_head.body2.0")
    w = f32(_np(sd["policy_head.body3.0.weight"]) if w_fc is None else w_fc)
    b = f32(_np(sd["policy_head.body3.0.bias"]))[:w.shape[0]]

    def edit(nodes, inits):
        fi, ci = _policy_flatten(nodes)
        _, _, (x, w_old), (y,) = nodes[ci]
        del inits[w_old]
        inits["policy_w2"], inits["policy_b2"] = _tensor("policy_w2", f32(w2)), _tensor("policy_b2", f32(b2))
        conv = _node("Conv", [x, "policy_w2", "policy_b2"], [y], [("group", 1)])
        nodes[ci] = (conv, *_decode(conv))
        new = []

        def add(op, ins, out, attrs=()):
            new.append(_node(op, ins, [out], attrs))
            return out

        t = add("Relu", [y], "policy_relu") if relu else y
        if flatten == "Reshape":
            inits["policy_shape"] = _int64("policy_shape", [-1, w.shape[1]])
            t = add("Reshape", [t, "policy_shape"], "policy_flat")
        else:
            t = add("Flatten", [t], "policy_flat", [("axis", 1)])
        if fc and linear == "MatMul":
            inits["policy_fc_w"], inits["policy_fc_b"] = _tensor("policy_fc_w", w.T), _tensor("policy_fc_b", b)
            t = add("Add", [add("MatMul", [t, "policy_fc_w"], "policy_mm"), "policy_fc_b"], "policy_fc")
        elif fc:
            inits["policy_fc_w"] = _tensor("policy_fc_w", w if trans_b else w.T)
            inits["policy_fc_b"] = _tensor("policy_fc_b", b)
            t = add("Gemm", [t, "policy_fc_w", "policy_fc_b"], "policy_fc", [("transB", trans_b)])
        if softmax:
            add("Softmax", [t], "policy_prob", [("axis", 1)])
        return nodes[:fi] + nodes[fi + 1:] + [(nd, *_decode(nd)) for nd in new], inits

    return _rewrite(path, edit, shuffle)


def add_mx_head(path, params, eps=1e-3, seed=0, bn=True, fc=True):
    """params: the ones the writer was given, with policy_bn1 and policy_out (tests/classic_mx_head.py); the nodes are
    shuffled again with seed.  For the refusal tests: bn=False leaves policy_bn1 out, fc=False the FullyConnected."""
    def edit(nodes, inits):
        fi, ci = _policy_flatten(nodes)
        y = nodes[ci][3][0]
        sm = next(i for i, nd in enumerate(nodes) if nd[1] == "Softmax" and nd[2] == [nodes[fi][3][0]])
        new = []
        if bn:
            names = [f"policy_bn1_{k}" for k in ("gamma", "beta", "moving_mean", "moving_var")]
            for n in names:
                inits[n] = _tensor(n, np.ones_like(params["policy_bn1_beta"]) if n.endswith("gamma") else params[n])
            new.append(_fnode("BatchNormalization", [y] + names, ["policy_bn1"], [("epsilon", eps)]))
        new += [_node("Relu", ["policy_bn1" if bn else y], ["policy_act1"]), _node("Flatten", ["policy_act1"], ["policy_flatten0"])]
        if fc:
            for k in ("weight", "bias"):
                inits["policy_out_" + k] = _tensor("policy_out_" + k, params["policy_out_" + k])
            new.append(_node("Gemm", ["policy_flatten0", "policy_out_weight", "policy_out_bias"], ["policy_out"], [("transB", 1)]))
        new.append(_node("Softmax", ["policy_out" if fc else "policy_flatten0"], ["policy"]))
        return [nd for i, nd in enumerate(nodes) if i not in (fi, sm)] + [(nd, *_decode(nd)) for nd in new], inits

    return _rewrite(path, edit, seed)
