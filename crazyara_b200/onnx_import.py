"""Weight import from the reference's ONNX artefacts (SURVEY §8 f3) -> a blob for ara_net_create: the files
`export_to_onnx` writes (DeepCrazyhouse/src/training/trainer_agent_pytorch.py:588-650: torch.onnx.export in eval mode,
then onnx-simplifier, which folds BatchNorm into the convolutions) and the exports of the MXNet symbols
(`convert_to_onnx.py`).  No `onnx` package is needed: a minimal protobuf wire-format reader takes only the fields used here
(graph.node: op_type, inputs, outputs, attributes; graph.initializer: dims, data type, raw / float / int64 data).

The graph is not executed and its node order is not trusted: `_Graph` follows its edges from the stem convolution on the
graph input, block by block, to the heads, looking through shape-only nodes.
- BatchNorm folded (RISE; AlphaVile after merge_bn() has folded norm1 / norm2 into q / k / v and mlp.conv1) -> the blob
  weights.export_blob writes for the same checkpoint, ARAB2001 or ARAB2003.  A block input that feeds a `Mul` with a gate
  has squeeze-excitation, and the `Mul` output is the block's input and shortcut (builder_util.py:473-475).  A block input
  that feeds an `Add` starts a bottleneck block (conv1x1, depthwise, conv1x1, traced back from the Add); any other block
  is a NextViT transformer block (NTB), whose q and k are told apart by the attention-score `MatMul` they feed and v by
  the one behind the `Softmax`.  The policy head's 3x3 convolution ends the tower.
- Unfolded `BatchNormalization` nodes (an MXNet export, SE off the shortcut) -> export_mx_blob's ARAB2002 blob.  Each block
  is the `Add` fed by the block input, traced back through BatchNormalization / Relu / Conv to its first convolution,
  whose input is the block input or its `Mul` with the gate (`Sigmoid`, or `HardSigmoid` with alpha 0.2).
Both trace the gate back to `Gemm, Relu, Gemm` (ca_se) or to a 1-D `Conv` over the channels (eca_se).
A fully-connected policy head (the trainer's select_policy_from_plane=False) is the last policy convolution's output
(an MXNet export: through its BatchNormalization policy_bn1) followed by Relu, a flatten and Gemm (or MatMul + Add) onto
a classic label list; it is written as ARAB2004 around the base format.  Such a layer that does not take the flattened
ReLU, has another label count or another width is refused, as are a bias or a Relu behind a folded policy-map
convolution and a policy_bn1 with no such layer behind it: no blob format holds them, and dropping them would change
the network.
The value head is the standard one, the WDL and plies-to-end layers (a torch export's WDL `Gemm` may feed the value MLP
of use_mlp_wdl_ply: Concat(WDL logits, Sigmoid(plies)) -> Gemm -> Relu -> Gemm -> Tanh), or, in an MXNet export, every
Gemm behind value_fc0's Relu: value_fc1, or the WDL layer into its Softmax and the plies layer into its Sigmoid, then
win - loss (Split) or the value MLP on Concat(probabilities, plies) (crazyara_b200/weights.py VALUE_HEADS).

PARITY UNPINNED: the reference tree holds no .onnx file and no `onnx` / `onnxsim` package is installed, so the readers are
checked against files written by tests/onnx_writer.py, tests/onnx_mx_writer.py and tests/onnx_alphavile_writer.py
(tests/onnx_classic_writer.py adds the fully-connected policy head to them, tests/onnx_wdl_writer.py the value heads
above).
"""
import struct
from collections import defaultdict

import numpy as np

from .weights import CLASSIC_LABELS, export_mx_blob, input_version_of, write_blob

_SHAPE_OPS = ("Reshape", "Flatten", "Squeeze", "Unsqueeze", "Identity")
# a torch export also has the NTB's token transposes and the Expand of the SE gate (x * y.view(b, c, 1, 1).expand_as(x))
_TORCH_SHAPE_OPS = _SHAPE_OPS + ("Transpose", "Expand")


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


# ---------------------------------------------------------------------------------------------- graph walks
class _Graph:
    """One file's nodes, initialisers, producers and consumers, and walks along its edges through the node types `skip`"""

    def __init__(self, path, nodes, inits, skip):
        self.path, self.nodes, self.inits, self.skip = path, nodes, inits, skip
        self.prod, self.cons = {}, defaultdict(list)
        for nd in nodes:
            for o in nd[2]:
                self.prod[o] = nd
            for i in nd[1]:
                self.cons[i].append(nd)

    def fail(self, what):
        raise ValueError(f"{self.path}: {what}")

    def back(self, t, *ops):  # the producer of t, skipping shape-only nodes, which must be one of ops
        nd = self.prod.get(t)
        while nd is not None and nd[0] in self.skip:
            nd = self.prod.get(nd[1][0])
        if nd is None or nd[0] not in ops:
            self.fail(f"expected {'/'.join(ops)} in front of '{t}', found {nd[0] if nd else 'a graph input'}")
        return nd

    def fwd(self, t, op, weighted=None):  # the consumers of t of type op, whose second input is an initialiser if weighted
        out, frontier = [], [t]
        while frontier:
            u = frontier.pop()
            for nd in self.cons[u]:
                if nd[0] in self.skip:
                    frontier.append(nd[2][0])
                elif nd[0] == op and (weighted is None or (len(nd[1]) > 1 and nd[1][1] in self.inits) == weighted):
                    out.append(nd)
        return out

    def first(self, t, op):  # the first direct consumer of t of type op, or None
        return next((nd for nd in self.cons[t] if nd[0] == op), None)

    def one(self, t, op, weighted=None):
        c = self.fwd(t, op, weighted)
        if len(c) != 1:
            self.fail(f"expected one {op} behind '{t}', found {len(c)}")
        return c[0]

    def downstream(self, t, ops):  # the first node of one of ops reached from tensor t, breadth first
        seen, frontier = set(), [t]
        while frontier:
            nxt = []
            for u in frontier:
                for nd in self.cons[u]:
                    if nd[0] in ops:
                        return nd
                    if id(nd) not in seen:
                        seen.add(id(nd))
                        nxt += nd[2]
            frontier = nxt
        return None

    def weight(self, nd):  # a Conv's weight; a Gemm's or MatMul's as [out, in], the layout of torch.nn.Linear.weight
        w = self.inits[nd[1][1]]
        return np.ascontiguousarray(w.T if nd[0] == "MatMul" or (nd[0] == "Gemm" and not nd[3].get("transB", 0)) else w)

    def bias(self, nd):  # a Conv's or Gemm's bias, zeros when it has none
        has = len(nd[1]) > 2 and nd[1][2] in self.inits
        return self.inits[nd[1][2]] if has else np.zeros(self.weight(nd).shape[0], np.float32)

    def linear(self, mm):  # MatMul(x, W[in, out]) + Add(bias) -> ([out, in], bias, output tensor)
        add = self.one(mm[2][0], "Add")
        b = next((self.inits[i] for i in add[1] if i in self.inits), None)
        if b is None:
            self.fail(f"no bias behind MatMul '{mm[2][0]}'")
        return self.weight(mm), b, add[2][0]

    def policy_fc(self, t, P):
        """The fully-connected policy head behind tensor t, the last policy convolution's output (an MXNet export: its
        BatchNorm's): Relu, a flatten (Flatten, or the Reshape of torch's view()), then Gemm or MatMul + Add onto the
        classic labels -> (W_fc [L][P * 64], b_fc [L]); None when no fully-connected layer follows t (a policy map)"""
        fc = self.downstream(t, ("Gemm", "MatMul"))
        if fc is None:
            return None
        relu = self.prod.get(fc[1][0])
        while relu is not None and relu[0] in self.skip:
            relu = self.prod.get(relu[1][0])
        if relu is None or relu[0] != "Relu" or relu[1][0] != t or len(fc[1]) < 2 or fc[1][1] not in self.inits:
            self.fail(f"policy head: the {fc[0]} behind the last policy convolution does not take its flattened ReLU")
        w, b = (self.weight(fc), self.bias(fc)) if fc[0] == "Gemm" else self.linear(fc)[:2]
        if w.shape[0] not in CLASSIC_LABELS:
            self.fail(f"policy head: a fully-connected layer onto {w.shape[0]} labels (the classic label lists have "
                      f"{CLASSIC_LABELS})")
        if w.shape[1] != P * 64:
            self.fail(f"policy head: the fully-connected layer takes {w.shape[1]} features, not the {P} x 64 of the flattened "
                      f"convolution")
        return w, b

    def stem(self):  # the convolution on the graph input
        return next((nd for nd in self.nodes if nd[0] == "Conv" and nd[1][0] not in self.prod and nd[1][0] not in self.inits), None)

    def se(self, mul, x, i):  # block i's Mul(x, gate) -> (gate, [Gemm, Gemm] for ca_se or [Conv] for eca_se)
        if x not in mul[1]:
            self.fail(f"block {i}: the squeeze-excitation does not act on the block input")
        gate = self.back(mul[1][1] if mul[1][0] == x else mul[1][0], "Sigmoid", "HardSigmoid")
        fc = self.back(gate[1][0], "Gemm", "MatMul", "Conv")
        if fc[0] == "Conv":
            return gate, [fc]
        return gate, [self.back(self.back(fc[1][0], "Relu")[1][0], "Gemm", "MatMul"), fc]


# ---------------------------------------------------------------------------------------------- graph -> blob
def import_onnx(onnx_path, blob_path, input_version=None, channels=256):
    nodes, inits = read_graph(onnx_path)
    if any(nd[0] == "BatchNormalization" for nd in nodes):
        return _import_mxnet_graph(_Graph(onnx_path, nodes, inits, _SHAPE_OPS), blob_path, input_version, channels)
    return _import_folded_graph(_Graph(onnx_path, nodes, inits, _TORCH_SHAPE_OPS), blob_path, input_version, channels)


def _import_mxnet_graph(g, blob_path, input_version, channels):
    """a graph with unfolded BatchNormalization nodes (an MXNet export) -> ARAB2002 blob (ARAB2004 around it with a
    fully-connected policy head)"""
    params, eps = {}, {}

    def take_bn(nd, name):
        for key, i in (("gamma", 1), ("beta", 2), ("moving_mean", 3), ("moving_var", 4)):
            params[f"{name}_{key}"] = g.inits[nd[1][i]]
        eps[name] = float(nd[3].get("epsilon", 1e-5))  # (ONNX's default)

    def take(nd, name):  # Conv / Gemm weights and bias under the MXNet layer name
        params[name + "_weight"] = g.weight(nd)
        if len(nd[1]) > 2 and nd[1][2] in g.inits:
            params[name + "_bias"] = g.inits[nd[1][2]]

    def conv_bn(t, name):  # t = output of Conv -> BatchNormalization: the Conv node
        bn = g.back(t, "BatchNormalization")
        conv = g.back(bn[1][0], "Conv")
        take(conv, name)
        take_bn(bn, name.replace("conv", "bn"))
        return conv

    stem = g.stem()
    if stem is None or g.weight(stem).shape[0] != channels or g.weight(stem).shape[2] != 3:
        g.fail(f"no 3x3 stem convolution with {channels} channels on the graph input")
    take(stem, "stem_conv0")
    bn = g.first(stem[2][0], "BatchNormalization")
    if bn is None:
        g.fail("no BatchNormalization behind the stem")
    take_bn(bn, "stem_bn0")
    relu = g.first(bn[2][0], "Relu")
    x, stem_act = (relu[2][0], True) if relu is not None and g.first(relu[2][0], "Add") is not None else (bn[2][0], False)
    kernels, se_types, se_gates, c_ops, n_eca = [], [], [], [], 0
    while True:
        add = g.first(x, "Add")
        if add is None:
            break
        i, p = len(kernels), f"bc_res_block{len(kernels)}"
        conv3 = conv_bn(add[1][1] if add[1][0] == x else add[1][0], p + "_conv3")
        conv2 = conv_bn(g.back(conv3[1][0], "Relu")[1][0], p + "_conv2")
        conv1 = conv_bn(g.back(conv2[1][0], "Relu")[1][0], p + "_conv1")
        w1, wd = params[p + "_conv1_weight"], params[p + "_conv2_weight"]
        if w1.shape[1] != channels or wd.shape[0] != w1.shape[0] or wd.shape[2] not in (3, 5):
            g.fail(f"block {i} is not a RISE bottleneck block")
        se, gate = None, None
        if conv1[1][0] != x:
            gn, fcs = g.se(g.back(conv1[1][0], "Mul"), x, i)
            gate, alpha, beta = ("sigmoid" if gn[0] == "Sigmoid" else "hard_sigmoid"), gn[3].get("alpha", 0.2), gn[3].get("beta", 0.5)
            if gate == "hard_sigmoid" and not (abs(alpha - 0.2) < 1e-6 and abs(beta - 0.5) < 1e-6):
                g.fail(f"block {i}: HardSigmoid alpha {alpha} beta {beta}")
            se = "eca_se" if len(fcs) == 1 else "ca_se"
            if se == "eca_se":
                take(fcs[0], f"convolution{n_eca}")
                n_eca += 1
            else:
                take(fcs[0], p + "_se_fc0"), take(fcs[1], p + "_se_fc1")
        kernels.append(int(wd.shape[2])), se_types.append(se), se_gates.append(gate), c_ops.append(int(w1.shape[0]))
        x = add[2][0]
    if not kernels:
        g.fail("no bottleneck block found")
    heads = [nd for nd in g.cons[x] if nd[0] == "Conv"]
    vconv = [nd for nd in heads if g.weight(nd).shape[2] == 1]
    pconv = [nd for nd in heads if g.weight(nd).shape[2] == 3]
    if len(vconv) != 1 or len(pconv) != 1:
        g.fail("value head (1x1 convolution) and policy head (3x3 convolution) not found behind the tower")
    take(vconv[0], "value_conv0")
    take_bn(g.first(vconv[0][2][0], "BatchNormalization"), "value_bn0")
    g0 = g.downstream(vconv[0][2][0], ("Gemm", "MatMul"))
    act = g0 and g.first(g0[2][0], "Relu")
    behind = (g.fwd(act[2][0], "Gemm", True) or g.fwd(act[2][0], "MatMul", True)) if act is not None else []
    if not behind:
        g.fail("value head: two fully-connected layers not found")
    take(g0, "value_fc0")
    value_head = _mx_value_outputs(g, behind, take)
    fc = int(params["value_fc0_weight"].shape[0])
    if value_head is not None and not 1 <= fc <= 256:
        g.fail(f"value head: {fc} hidden units in front of the WDL and plies-to-end outputs (1 .. 256)")
    take(pconv[0], "policy_conv0")
    take_bn(g.first(pconv[0][2][0], "BatchNormalization"), "policy_bn0")
    pc1 = g.downstream(pconv[0][2][0], ("Conv",))
    take(pc1, "policy_conv1")
    P = int(params["policy_conv1_weight"].shape[0])
    # select_policy_from_plane=False (builder_util_symbol.py policy_head): policy_bn1, the activation, Flatten, policy_out
    bn1 = g.first(pc1[2][0], "BatchNormalization")
    head = g.policy_fc(bn1[2][0] if bn1 is not None else pc1[2][0], P)
    if head is not None and bn1 is None:
        g.fail("policy head: no BatchNormalization (policy_bn1) between the last policy convolution and its ReLU")
    if head is None and bn1 is not None:
        g.fail("policy head: a BatchNormalization behind the last policy convolution but no fully-connected layer")
    arch = dict(name=f"rise_{len(kernels)}b", semantics="mxnet", in_channels=int(g.weight(stem).shape[1]),
                policy_channels=P, channels=channels, kernels=kernels,
                se_types=se_types, se_gates=se_gates, c_ops=c_ops, wdl=value_head is not None,
                value_channels=int(params["value_conv0_weight"].shape[0]), value_fc=256, stem_act=stem_act,
                policy_bias="policy_conv1_bias" in params)
    if value_head is not None:
        arch.update(value_head=value_head, value_fc=fc)
    if head is not None:  # the convolution's bias is folded with policy_bn1 into the head (ARAB2004)
        take_bn(bn1, "policy_bn1")
        params["policy_out_weight"], params["policy_out_bias"] = head
        arch.update(policy_bias=False, n_labels=int(head[0].shape[0]))
    export_mx_blob(params, arch, blob_path, input_version_of(arch, input_version), eps=eps, fix_gamma=False)
    return arch


def _mx_value_outputs(g, fcs, take):
    """the value head of an MXNet export behind value_fc0's Relu, whose Gemm nodes are fcs (builder_util_symbol.py
    value_head) -> None for value_fc1 and Tanh; with use_wdl and use_plys_to_end, the WDL layer (3 units) into the
    Softmax of its SoftmaxOutput and value_plys_to_end_fc (1 unit) into a Sigmoid, then "mx_wdl" for value = win - loss
    (Split, Neg, Add) or "mx_wdl_mlp" for the MLP value_wdl_ply_fc (8 units), Relu, value_fc1, Tanh on
    Concat(probabilities, plies).  All the Gemm nodes behind the Relu are read, so the node order does not matter."""
    widths = sorted(int(g.weight(nd).shape[0]) for nd in fcs)
    if widths == [1]:
        take(fcs[0], "value_fc1")
        return None
    if widths != [1, 3]:
        g.fail(f"value head: fully-connected layers of {widths} units behind value_fc0 (value_fc1, or the WDL and "
               f"plies-to-end layers)")
    wdl, plys = sorted(fcs, key=lambda nd: -int(g.weight(nd).shape[0]))
    sm, sig = g.first(wdl[2][0], "Softmax"), g.first(plys[2][0], "Sigmoid")
    if sm is None or sig is None:
        g.fail("value head: WDL and plies-to-end layers behind value_fc0 without a Softmax behind the first or a Sigmoid "
               "behind the second")
    take(wdl, "wdl_out"), take(plys, "value_plys_to_end_fc")
    m0 = g.downstream(sm[2][0], ("Gemm", "MatMul"))
    if m0 is None:  # value = broadcast_add(-loss, win) of the split probabilities
        if g.downstream(sm[2][0], ("Split",)) is None:
            g.fail("value head: neither win - loss nor a value MLP behind the WDL output")
        return "mx_wdl"
    cat = g.back(m0[1][0], "Concat")
    if len(cat[1]) != 2 or cat[1][0] != sm[2][0] or cat[1][1] != sig[2][0]:
        g.fail("value head: the value MLP does not take Concat(WDL probabilities, plies)")
    m1 = g.one(g.one(m0[2][0], "Relu")[2][0], "Gemm", True)
    if g.weight(m1).shape[0] != 1 or g.first(m1[2][0], "Tanh") is None:
        g.fail("value head: the value MLP does not end in one unit and Tanh")
    take(m0, "value_wdl_ply_fc"), take(m1, "value_fc1")
    return "mx_wdl_mlp"


def _torch_value_mlp(g, wdl, plys):
    """use_mlp_wdl_ply in a torch export (builder_util.py _ValueHead :315-320): behind the WDL Gemm and the plies Gemm's
    Sigmoid, Concat(wdl, plies) -> Gemm (8) -> Relu -> Gemm (1) -> Tanh -> its two layers as [W0, b0, W1, b1]; None for
    the WDL head without it"""
    m0 = g.downstream(wdl[2][0], ("Gemm", "MatMul"))
    if m0 is None:
        return None
    sig = g.first(plys[2][0], "Sigmoid")
    cat = g.back(m0[1][0], "Concat")
    if sig is None or len(cat[1]) != 2 or cat[1][0] != wdl[2][0] or cat[1][1] != sig[2][0]:
        g.fail("value head: a fully-connected layer behind the WDL output that does not take Concat(WDL logits, "
               "sigmoid(plies)), the value MLP's input")
    if m0[0] != "Gemm":
        g.fail("value head: the value MLP's first layer is not a Gemm")
    m1 = g.one(g.one(m0[2][0], "Relu")[2][0], "Gemm", True)
    if g.weight(m1).shape[0] != 1 or g.first(m1[2][0], "Tanh") is None:
        g.fail("value head: the value MLP does not end in one unit and Tanh")
    return [g.weight(m0), g.bias(m0), g.weight(m1), g.bias(m1)]


def _import_folded_graph(g, blob_path, input_version, channels):
    """a BatchNorm-folded export: a RISE network (256-channel trunk) -> ARAB2001 blob, an AlphaVile one -> ARAB2003 (ARAB2004
    around either with a fully-connected policy head)"""
    W, bias = g.weight, g.bias
    mat = lambda a: a.reshape(a.shape[0], -1)
    stem = g.stem()
    if stem is None or W(stem).shape[2] != 3:
        g.fail("no 3x3 stem convolution on the graph input")
    C = int(W(stem).shape[0])
    tensors = [W(stem), bias(stem)]
    x = g.one(stem[2][0], "Relu")[2][0]
    kernels, se_types, c_ops, ntb, widths = [], [], [], [], set()
    while not any(W(nd).shape[2] == 3 for nd in g.fwd(x, "Conv", True)):  # the policy head's 3x3 convolution ends the tower
        i, se = len(kernels), None
        mul = g.first(x, "Mul")
        if mul is not None:  # squeeze-excitation (its gate unchecked: ARAB2001 knows only torch's hard sigmoid)
            _, fcs = g.se(mul, x, i)
            se, w = ("ca_se" if len(fcs) == 2 else "eca_se"), W(fcs[0])
            if se == "eca_se" and w.ndim != 3:
                g.fail(f"block {i}: the eca_se convolution is not 1-D")
            # (the reference's SE FCs have no bias, builder_util.py:100-116; of the eca_se Conv the centre tap and bias)
            tensors += [w, W(fcs[1])] if se == "ca_se" else [w[:, :, w.shape[2] // 2], bias(fcs[0])]
            x = mul[2][0]  # the block's input and its shortcut
        add = g.first(x, "Add")
        if add is not None:  # bottleneck block: x + conv1x1(relu(depthwise(relu(conv1x1(x)))))
            c3 = g.back(add[1][1] if add[1][0] == x else add[1][0], "Conv")
            c2 = g.back(g.back(c3[1][0], "Relu")[1][0], "Conv")
            c1 = g.back(g.back(c2[1][0], "Relu")[1][0], "Conv")
            w1, wd, w3 = W(c1), W(c2), W(c3)
            if (c1[1][0] != x or w1.shape[1] != C or wd.shape[0] != w1.shape[0] or wd.shape[2] not in (3, 5) or
                    w3.shape[:2] != (C, w1.shape[0])):
                g.fail(f"block {i} is not a RISE bottleneck block")
            tensors += [w1, bias(c1), wd, bias(c2), w3, bias(c3)]
            kernels.append(int(wd.shape[2])), se_types.append(se), c_ops.append(int(w1.shape[0])), ntb.append(False)
            x = add[2][0]
            continue
        if se is not None:
            g.fail(f"block {i}: no Add takes the squeeze-excitation's output as the shortcut")
        pe = g.one(x, "Conv", True)
        y = pe[2][0]
        lin = {t: (w, b) for w, b, t in map(g.linear, g.fwd(y, "MatMul", True))}
        if len(lin) != 3:
            g.fail(f"block {i}: {len(lin)} q / k / v projections behind the patch embedding (expected 3)")
        users = {}  # the attention MatMul each projection feeds: q and k the scores Q K^T, v the product P V
        for t in lin:
            u = g.one(t, "MatMul", False)
            users.setdefault(id(u), (u, []))[1].append(t)
        qk = next((nd for nd, ts in users.values() if len(ts) == 2), None)
        if qk is None:
            g.fail(f"block {i}: attention scores Q K^T not found")
        q, k = (g.back(a, "Add")[2][0] for a in qk[1])
        sc = g.fwd(qk[2][0], "Mul") or g.fwd(qk[2][0], "Div")
        s = next((float(g.inits[a].reshape(-1)[0]) for a in sc[0][1] if a in g.inits), None) if len(sc) == 1 else None
        if s is None or abs((s if sc[0][0] == "Mul" else 1.0 / s) - 32 ** -0.5) > 1e-6:
            g.fail(f"block {i}: attention scale {s} (expected 32^-0.5)")
        sm = g.one(sc[0][2][0], "Softmax")
        pv = g.one(sm[2][0], "MatMul", False)
        v = g.back(pv[1][1], "Add")[2][0]
        if len({q, k, v}) != 3:
            g.fail(f"block {i}: q / k / v not told apart")
        wp, bp, o = g.linear(g.one(pv[2][0], "MatMul", True))
        y1_add = g.one(o, "Add")
        if y not in y1_add[1]:
            g.fail(f"block {i}: the attention output is not added to the patch embedding")
        y1 = y1_add[2][0]
        prj = g.one(y1, "Conv", True)
        z = prj[2][0]
        gc = next((nd for nd in g.fwd(z, "Conv", True) if W(nd).shape[2] == 3), None)  # (one group when Ca = 32)
        if gc is None:
            g.fail(f"block {i}: no group convolution behind the projection")
        mh = g.one(g.one(gc[2][0], "Relu")[2][0], "Conv", True)
        if np.any(bias(mh) != 0):
            g.fail(f"block {i}: the MHCA conv1x1 has a bias")
        z2 = g.one(mh[2][0], "Add")
        cat = g.one(y1, "Concat")
        if cat[1] != [y1, z2[2][0]] or z not in z2[1]:
            g.fail(f"block {i}: the NTB does not concatenate y1 | z2")
        m1 = g.one(cat[2][0], "Conv", True)
        m2 = g.one(g.one(m1[2][0], "Relu")[2][0], "Conv", True)
        out = g.one(m2[2][0], "Add")
        if cat[2][0] not in out[1]:
            g.fail(f"block {i}: the MLP output is not added to the concatenation")
        M, Ca, H = int(W(pe).shape[0]), int(W(prj).shape[0]), int(W(m1).shape[0])
        if W(gc).shape[1] != 32 or W(gc).shape[0] != Ca or gc[3].get("group", 1) != Ca // 32:
            g.fail(f"block {i}: group convolution {W(gc).shape} (expected heads of 32 channels)")
        tensors += [mat(W(pe)), bias(pe), np.concatenate([lin[q][0], lin[k][0], lin[v][0]]),
                    np.concatenate([lin[q][1], lin[k][1], lin[v][1]]), wp, bp, mat(W(prj)), bias(prj), W(gc), bias(gc),
                    mat(W(mh)), mat(W(m1)), bias(m1), mat(W(m2)), bias(m2)]
        widths.add((M, Ca, H))
        kernels.append(3), se_types.append(None), c_ops.append(0), ntb.append(True)
        x = out[2][0]
    if not kernels:
        g.fail("no block found")
    if len(widths) > 1:
        g.fail(f"NTB blocks of different widths {sorted(widths)}")
    if not widths and C != channels:
        g.fail(f"{C} trunk channels, this engine builds {channels}")
    heads = g.fwd(x, "Conv", True)
    vconv = [nd for nd in heads if W(nd).shape[2] == 1]
    pconv = [nd for nd in heads if W(nd).shape[2] == 3]
    if len(vconv) != 1 or len(pconv) != 1:
        g.fail("value head (1x1 convolution) and policy head (3x3 convolution) not found behind the tower")
    tensors += [W(vconv[0]), bias(vconv[0])]
    v = g.one(vconv[0][2][0], "Relu")[2][0]
    fc = g.fwd(v, "Gemm", True) or g.fwd(v, "MatMul", True)
    wdl = len(fc) == 2
    if wdl:
        fc = sorted(fc, key=lambda nd: -W(nd).shape[0])  # WDL (3 outputs), then plies (1)
        mlp = _torch_value_mlp(g, *fc)
    elif len(fc) == 1:
        fc = [fc[0], g.downstream(fc[0][2][0], ("Gemm", "MatMul"))]
        if fc[1] is None:
            g.fail("value head: two fully-connected layers not found")
    else:
        g.fail(f"value head: {len(fc)} fully-connected layers behind the convolution")
    for nd in fc:
        tensors += [W(nd), bias(nd)]
    if wdl and mlp is not None:
        tensors += mlp
    p2 = g.downstream(pconv[0][2][0], ("Conv",))
    if p2 is None:
        g.fail("policy head: second convolution not found")
    tensors += [W(pconv[0]), bias(pconv[0]), W(p2)]
    arch = dict(name=f"rise_{len(kernels)}b", in_channels=int(W(stem).shape[1]), policy_channels=int(W(p2).shape[0]),
                channels=C, kernels=kernels, se_types=se_types, c_ops=c_ops, wdl=wdl, value_channels=int(W(vconv[0]).shape[0]),
                value_fc=256)
    if wdl and mlp is not None:
        arch["value_head"] = "wdl_mlp"
    if widths:
        (M, Ca, H), = widths
        arch.update(name=f"alphavile_{len(kernels)}b", ntb=ntb, mhsa=M, mhca=Ca, mlp=H,
                    value_fc=C if wdl else int(W(fc[0]).shape[0]))
    # select_policy_from_plane=False: the exporter has folded the head's BatchNorm (body2) into p2, ReLU, view(), Linear
    head = g.policy_fc(p2[2][0], arch["policy_channels"])
    if head is not None:
        tensors += [bias(p2), *head]
        arch["n_labels"] = int(head[0].shape[0])
    elif np.any(bias(p2) != 0):
        g.fail("policy head: the last policy convolution has a bias but no fully-connected layer behind it (a policy map's "
               "convolution has none)")
    elif g.first(p2[2][0], "Relu") is not None:
        g.fail("policy head: a Relu behind the last policy convolution but no fully-connected layer")
    write_blob(blob_path, arch, tensors, input_version_of(arch, input_version))
    return arch


if __name__ == "__main__":
    import sys
    if len(sys.argv) < 3:
        raise SystemExit("usage: python -m crazyara_b200.onnx_import <model.onnx> <out.arab> [input_version]")
    a = import_onnx(sys.argv[1], sys.argv[2], int(sys.argv[3]) if len(sys.argv) > 3 else None)
    policy = f"{a['n_labels']} labels" if a.get("n_labels") else f"{a['policy_channels']}x64"
    print(f"{sys.argv[2]}: {len(a['kernels'])} blocks, {a['in_channels']} -> {policy}, wdl={a['wdl']}")
