"""A NumPy stand-in for `mxnet.sym`, enough to build and evaluate (inference) the reference's RISE symbols
(rise_mobile_v2.py, rise_mobile_v3.py, builder_util_symbol.py) -- TEST INFRASTRUCTURE ONLY, never imported by the product.

MXNet itself is not installed, so the operator semantics below are taken from MXNet's operator documentation (1.x
symbol API), not from executed MXNet:
  Convolution   NC(H)W cross-correlation, kernel / stride (1) / pad (0) / num_group (1) / no_bias (False); 1-D and 2-D
  BatchNorm     inference with the moving statistics: (x - moving_mean) / sqrt(moving_var + eps) * gamma + beta on axis
                1, eps 1e-3, fix_gamma True (gamma taken as 1)
  Activation    relu, sigmoid, tanh, softrelu, softsign;  hard_sigmoid: max(0, min(1, alpha x + beta)), alpha 0.2, beta 0.5
  Pooling       avg / max over `kernel` windows (stride 1, no padding, "valid"), or the whole plane with global_pool
  Flatten       (N, -1);  FullyConnected: flatten=True, x . W^T + b, no_bias False
  reshape       shape codes 0 (copy the input's dimension) and -1 (inferred)
  broadcast_add / broadcast_mul, Concat (dim 1), split (axis 1, squeeze_axis False), Dropout (identity at inference)
  LinearRegressionOutput (identity), SoftmaxOutput (softmax over axis 1 of the 2-D input), Group
Names: an operator without a name gets `<op name in lower case><n>`, counted per operator from 0 for each NameScope
(MXNet's NameManager); parameters are `<name>_weight`, `_bias`, `_gamma`, `_beta` and the aux states `_moving_mean`,
`_moving_var`; the output operators add the label argument `<name>_label`.
"""
import sys
import types

import numpy as np


class NameScope:
    """a fresh auto-naming counter, as one process that builds one symbol has"""
    counter = {}

    def __enter__(self):
        self.saved, NameScope.counter = NameScope.counter, {}
        return self

    def __exit__(self, *a):
        NameScope.counter = self.saved


def _auto(hint, name):
    if name is not None:
        return name
    n = NameScope.counter.get(hint, 0)
    NameScope.counter[hint] = n + 1
    return f"{hint}{n}"


class Symbol:
    def __init__(self, op, inputs, attrs, name, params=(), aux=(), index=None):
        self.op, self.inputs, self.attrs, self.name = op, list(inputs), attrs, name
        self.params, self.aux, self.index = list(params), list(aux), index

    def __neg__(self):
        return Symbol("_neg", [self], {}, _auto("negative", None))

    def __mul__(self, other):
        return broadcast_mul(self, other)

    # graph walks
    def _nodes(self, seen=None, out=None):
        seen = set() if seen is None else seen
        out = [] if out is None else out
        if id(self) in seen:
            return out
        seen.add(id(self))
        for s in self.inputs:
            s._nodes(seen, out)
        out.append(self)
        return out

    def list_arguments(self):
        args = []
        for nd in self._nodes():
            if nd.op == "Variable":
                args.append(nd.name)
            args += nd.params
        return list(dict.fromkeys(args))

    def list_auxiliary_states(self):
        return [a for nd in self._nodes() for a in nd.aux]

    def eval(self, feed):
        """feed: {argument / aux name: ndarray} -> list of the outputs (float64)"""
        r = _ev(self, feed, {})
        return r if isinstance(r, list) else [r]


def _ev(s, feed, cache):
    if id(s) in cache:
        return cache[id(s)]
    a = s.attrs
    x = [_ev(i, feed, cache) for i in s.inputs]
    x1 = [v[0] if isinstance(v, list) and s.op not in ("Group",) else v for v in x]
    if s.op == "Variable":
        r = np.asarray(feed[s.name], np.float64)
    elif s.op == "Group":
        r = [o for v in x for o in (v if isinstance(v, list) else [v])]
    elif s.op == "_split_out":
        r = x[0][s.index]
    else:
        r = _OPS[s.op](s, x1, feed)
    cache[id(s)] = r
    return r


def _conv(s, x, feed):
    a = s.attrs
    d = x[0]
    w = np.asarray(feed[s.name + "_weight"], np.float64)
    k = tuple(a["kernel"])
    nd = len(k)
    pad = tuple(a.get("pad", (0,) * nd))
    stride = tuple(a.get("stride", (1,) * nd))
    g = a.get("num_group", 1)
    d = np.pad(d, [(0, 0), (0, 0)] + [(p, p) for p in pad])
    N, C = d.shape[:2]
    F_ = w.shape[0]
    out_sp = [(d.shape[2 + i] - k[i]) // stride[i] + 1 for i in range(nd)]
    out = np.zeros([N, F_] + out_sp)
    cg, fg = C // g, F_ // g
    for gi in range(g):
        xs = d[:, gi * cg:(gi + 1) * cg]
        ws = w[gi * fg:(gi + 1) * fg]
        for off in np.ndindex(*k):
            sl = tuple(slice(off[i], off[i] + stride[i] * out_sp[i], stride[i]) for i in range(nd))
            patch = xs[(slice(None), slice(None)) + sl]  # [N, cg, *out]
            out[:, gi * fg:(gi + 1) * fg] += np.einsum("nc...,fc->nf...", patch, ws[(slice(None), slice(None)) + off])
    if not a.get("no_bias", False):
        out += np.asarray(feed[s.name + "_bias"], np.float64).reshape([1, -1] + [1] * nd)
    return out


def _bn(s, x, feed):
    a = s.attrs
    d = x[0]
    sh = [1, -1] + [1] * (d.ndim - 2)
    f = lambda n: np.asarray(feed[s.name + n], np.float64).reshape(sh)
    g = 1.0 if a.get("fix_gamma", True) else f("_gamma")
    return (d - f("_moving_mean")) / np.sqrt(f("_moving_var") + a.get("eps", 1e-3)) * g + f("_beta")


def _act(s, x, feed):
    t, d = s.attrs["act_type"], x[0]
    return {"relu": lambda: np.maximum(d, 0), "sigmoid": lambda: 1 / (1 + np.exp(-d)), "tanh": lambda: np.tanh(d),
            "softrelu": lambda: np.log1p(np.exp(d)), "softsign": lambda: d / (1 + np.abs(d))}[t]()


def _pool(s, x, feed):
    a, d = s.attrs, x[0]
    red = np.mean if a.get("pool_type", "max") == "avg" else np.max
    if a.get("global_pool", False):
        return red(d, axis=tuple(range(2, d.ndim)), keepdims=True)
    k = tuple(a["kernel"])
    out_sp = [d.shape[2 + i] - k[i] + 1 for i in range(len(k))]
    out = np.zeros(list(d.shape[:2]) + out_sp)
    for o in np.ndindex(*out_sp):
        sl = tuple(slice(o[i], o[i] + k[i]) for i in range(len(k)))
        out[(slice(None), slice(None)) + o] = red(d[(slice(None), slice(None)) + sl], axis=tuple(range(2, d.ndim)))
    return out


def _reshape(s, x, feed):
    d, shape = x[0], list(s.attrs["shape"])
    shape = [d.shape[i] if v == 0 else v for i, v in enumerate(shape)]
    return d.reshape(shape)


def _fc(s, x, feed):
    d = x[0].reshape(x[0].shape[0], -1)
    out = d @ np.asarray(feed[s.name + "_weight"], np.float64).T
    if not s.attrs.get("no_bias", False):
        out = out + np.asarray(feed[s.name + "_bias"], np.float64)
    return out


def _softmax_out(s, x, feed):
    d = x[0].reshape(x[0].shape[0], -1)
    e = np.exp(d - d.max(axis=1, keepdims=True))
    return e / e.sum(axis=1, keepdims=True)


_OPS = {
    "Convolution": _conv, "BatchNorm": _bn, "Activation": _act, "Pooling": _pool, "Flatten": lambda s, x, f: x[0].reshape(x[0].shape[0], -1),
    "FullyConnected": _fc, "reshape": _reshape, "hard_sigmoid": lambda s, x, f: np.clip(s.attrs.get("alpha", 0.2) * x[0] + s.attrs.get("beta", 0.5), 0, 1),
    "broadcast_add": lambda s, x, f: x[0] + x[1], "broadcast_mul": lambda s, x, f: x[0] * x[1],
    "Concat": lambda s, x, f: np.concatenate(x, axis=s.attrs.get("dim", 1)), "Dropout": lambda s, x, f: x[0],
    "LinearRegressionOutput": lambda s, x, f: x[0], "SoftmaxOutput": _softmax_out, "_neg": lambda s, x, f: -x[0],
    "LeakyReLU": lambda s, x, f: np.where(x[0] > 0, x[0], s.attrs.get("slope", 0.25) * x[0]),
}


# ---------------------------------------------------------------------------------------------- the symbol API
def Variable(name, **kw):
    return Symbol("Variable", [], kw, name)


def Convolution(data, name=None, **kw):
    name = _auto("convolution", name)
    return Symbol("Convolution", [data], kw, name, [name + "_weight"] + ([] if kw.get("no_bias", False) else [name + "_bias"]))


def BatchNorm(data, name=None, **kw):
    name = _auto("batchnorm", name)
    return Symbol("BatchNorm", [data], kw, name, [name + "_gamma", name + "_beta"], [name + "_moving_mean", name + "_moving_var"])


def FullyConnected(data, name=None, **kw):
    name = _auto("fullyconnected", name)
    return Symbol("FullyConnected", [data], kw, name, [name + "_weight"] + ([] if kw.get("no_bias", False) else [name + "_bias"]))


def _simple(op, hint):
    def f(data=None, *args, name=None, **kw):
        ins = [data] + [a for a in args if isinstance(a, Symbol)]
        return Symbol(op, ins, kw, _auto(hint, name))
    return f


def _output(op, hint):
    def f(data, name=None, **kw):
        name = _auto(hint, name)
        return Symbol(op, [data], kw, name, [name + "_label"])  # (the label is not read at inference)
    return f


Activation = _simple("Activation", "activation")
hard_sigmoid = _simple("hard_sigmoid", "hard_sigmoid")
Pooling = _simple("Pooling", "pooling")
Flatten = flatten = _simple("Flatten", "flatten")
reshape = _simple("reshape", "reshape")
Dropout = _simple("Dropout", "dropout")
LeakyReLU = _simple("LeakyReLU", "leakyrelu")
LinearRegressionOutput = _output("LinearRegressionOutput", "linearregressionoutput")
SoftmaxOutput = _output("SoftmaxOutput", "softmaxoutput")


def broadcast_add(lhs, rhs, name=None):
    return Symbol("broadcast_add", [lhs, rhs], {}, _auto("broadcast_add", name))


def broadcast_mul(lhs, rhs, name=None):
    return Symbol("broadcast_mul", [lhs, rhs], {}, _auto("broadcast_mul", name))


def Concat(*data, name=None, **kw):
    return Symbol("Concat", list(data), kw, _auto("concat", name))


concat = Concat


def split(data, num_outputs, axis=1, name=None, **kw):
    name = _auto("split", name)
    whole = Symbol("_split", [data], dict(kw, axis=axis, num_outputs=num_outputs), name)
    return [Symbol("_split_out", [whole], {}, f"{name}_output{i}", index=i) for i in range(num_outputs)]


_OPS["_split"] = lambda s, x, f: np.split(x[0], s.attrs["num_outputs"], axis=s.attrs["axis"])


def Group(symbols):
    return Symbol("Group", list(symbols), {}, "group")


def install():
    """registers the stand-in as `mxnet` (mx.sym and mx.symbol)"""
    mx = types.ModuleType("mxnet")
    sym = types.ModuleType("mxnet.symbol")
    for k, v in globals().items():
        if not k.startswith("__") and k not in ("install", "np", "sys", "types"):
            setattr(sym, k, v)
    mx.sym = mx.symbol = sym
    sys.modules["mxnet"] = mx
    sys.modules["mxnet.symbol"] = sym
    return mx
