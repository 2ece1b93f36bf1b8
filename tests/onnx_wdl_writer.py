"""Value heads with WDL and plies-to-end outputs that feed the value (tests/wdl_heads.py) for the ONNX files the test
writers make (tests/onnx_writer.py, tests/onnx_alphavile_writer.py, tests/onnx_mx_writer.py), for
tests/test_wdl_heads.py.  The functions here rewrite such a file with the head in place of the one the writer wrote, and
leave everything else in the file as the writer made it.

- add_torch_mlp: as torch.onnx.export leaves builder_util.py _ValueHead (:303-325) with use_mlp_wdl_ply, on a file the
  writer made for the WDL arch (the WDL Gemm and the plies Gemm on the flattened value features): Sigmoid behind the
  plies Gemm, Concat(WDL logits, plies) -> Gemm body_final.0 -> Relu -> Gemm body_final.2 -> Tanh, and the auxiliary
  Concat(WDL logits, plies) of process_value_policy_head.
- add_mx_wdl: as an MXNet export leaves builder_util_symbol.py value_head (:149-186) with use_wdl and use_plys_to_end,
  on a file the writer made with a standard head: behind value_fc0's Relu, Gemm wdl_out -> Softmax (SoftmaxOutput) and
  Gemm value_plys_to_end_fc -> Sigmoid; then Split -> Neg(loss) + win, or Concat(probabilities, plies) -> Gemm
  value_wdl_ply_fc -> Relu -> Gemm value_fc1 -> Tanh; and the auxiliary Concat of the symbol's Group.

Both shuffle the nodes with the seed given.  PARITY UNPINNED, as for the writers: no exporter runs here, so the layouts
are the ones those exporters document."""
import numpy as np

from crazyara_b200.onnx_import import _fields
from tests.onnx_classic_writer import _decode, _rewrite
from tests.onnx_writer import _node, _tensor


def _rows(tensor):
    """the first dimension of a serialised TensorProto"""
    return next(v for f, w, v in _fields(memoryview(tensor)) if f == 1)


def _gemm(x, w, b, out):
    return _node("Gemm", [x, w, b], [out], [("transB", 1)])


def add_torch_mlp(path, sd, shuffle=0):
    """sd: the state_dict the writer was given, with body_final as the value MLP (tests/wdl_heads.mlp_state_dict)"""
    f32 = lambda a: np.asarray(a, np.float32)

    def edit(nodes, inits):
        cons = {}
        for nd in nodes:
            for i in nd[2]:
                cons.setdefault(i, []).append(nd)
        # the flattened value features feed exactly the WDL Gemm (3 outputs) and the plies Gemm (1)
        pair = next(g for g in cons.values() if len(g) == 2 and all(nd[1] == "Gemm" for nd in g))
        wdl, plys = sorted(pair, key=lambda nd: -_rows(inits[nd[2][1]]))
        new = [_node("Sigmoid", [plys[3][0]], ["value_plys"]),
               _node("Concat", [wdl[3][0], "value_plys"], ["value_cat"], [("axis", 1)]),
               _gemm("value_cat", "value_mlp0_w", "value_mlp0_b", "value_mlp0"),
               _node("Relu", ["value_mlp0"], ["value_mlp_act"]),
               _gemm("value_mlp_act", "value_mlp1_w", "value_mlp1_b", "value_mlp1"),
               _node("Tanh", ["value_mlp1"], ["value_out"]),
               _node("Concat", [wdl[3][0], "value_plys"], ["auxiliary_out"], [("axis", 1)])]
        for n, key in (("value_mlp0", "value_head.body_final.0"), ("value_mlp1", "value_head.body_final.2")):
            inits[n + "_w"] = _tensor(n + "_w", f32(sd[key + ".weight"]))
            inits[n + "_b"] = _tensor(n + "_b", f32(sd[key + ".bias"]))
        return nodes + [(nd, *_decode(nd)) for nd in new], inits

    return _rewrite(path, edit, shuffle)


def add_mx_wdl(path, params, value_head, shuffle=0):
    """params: the head's parameters (tests/wdl_heads.mx_params); value_head "mx_wdl" or "mx_wdl_mlp".  The file's value
    head is value_fc0 -> Relu -> Gemm value_fc1 -> Tanh."""
    def edit(nodes, inits):
        fc1 = next(i for i, nd in enumerate(nodes) if nd[1] == "Gemm" and nd[2][1] == "value_fc1_weight")
        r = nodes[fc1][2][0]  # value_fc0's Relu
        tanh = next(i for i, nd in enumerate(nodes) if nd[1] == "Tanh" and nd[2] == [nodes[fc1][3][0]])
        for k in ("weight", "bias"):
            del inits["value_fc1_" + k]
        layers = ["wdl_out", "value_plys_to_end_fc"] + (["value_wdl_ply_fc", "value_fc1"] if value_head == "mx_wdl_mlp" else [])
        for n in layers:
            for k in ("weight", "bias"):
                inits[f"{n}_{k}"] = _tensor(f"{n}_{k}", np.asarray(params[f"{n}_{k}"], np.float32))
        new = [_gemm(r, "wdl_out_weight", "wdl_out_bias", "wdl_fc"), _node("Softmax", ["wdl_fc"], ["wdl"]),
               _gemm(r, "value_plys_to_end_fc_weight", "value_plys_to_end_fc_bias", "plys_fc"),
               _node("Sigmoid", ["plys_fc"], ["plys_to_end"]),
               _node("Concat", ["wdl", "plys_to_end"], ["auxiliary_output"], [("axis", 1)])]
        if value_head == "mx_wdl_mlp":
            new += [_node("Concat", ["wdl", "plys_to_end"], ["value_concat_0"], [("axis", 1)]),
                    _gemm("value_concat_0", "value_wdl_ply_fc_weight", "value_wdl_ply_fc_bias", "value_wdl_ply_fc"),
                    _node("Relu", ["value_wdl_ply_fc"], ["value_wdl_ply_act"]),
                    _gemm("value_wdl_ply_act", "value_fc1_weight", "value_fc1_bias", "value_fc1"),
                    _node("Tanh", ["value_fc1"], ["value_out"])]
        else:
            new += [_node("Split", ["wdl"], ["loss", "draw", "win"], [("axis", 1)]), _node("Neg", ["loss"], ["neg_loss"]),
                    _node("Add", ["neg_loss", "win"], ["value_out"])]
        return [nd for i, nd in enumerate(nodes) if i not in (fc1, tanh)] + [(nd, *_decode(nd)) for nd in new], inits

    return _rewrite(path, edit, shuffle)
