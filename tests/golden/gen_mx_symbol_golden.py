"""Generates tests/golden/<record>-symbol.json.gz: the reference's OWN MXNet symbol code (get_rise_v2_symbol in
rise_mobile_v2.py, get_rise_v33_symbol in rise_mobile_v3.py) built over the NumPy stand-in for mxnet.sym
(tests/golden/mx_standin.py) and written in MXNet's symbol-JSON layout by tojson, gzip-compressed, with the policy-map
head and with the fully-connected one (select_policy_from_plane=False), in the shapes of the records mx_net_risev2_34,
mx_net_risev33_52, classic_mx_net_risev2_2272 and classic_mx_net_risev33_1968.  Run where the reference tree is present
(the GPU machines do not have it):
    python tests/golden/gen_mx_symbol_golden.py
"""
import gzip
import json
import os
import sys
from itertools import accumulate

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from tests.golden import mx_standin  # noqa: E402
from tests.golden.gen_mx_net_golden import load_reference_symbols  # noqa: E402

# record -> (symbol, channels_policy_head, select_policy_from_plane, n_labels)
SYMBOLS = {"mx_net_risev2_34": ("risev2", 81, True, 2272), "mx_net_risev33_52": ("risev33", 76, True, 2272),
           "classic_mx_net_risev2_2272": ("risev2", 81, False, 2272),
           "classic_mx_net_risev33_1968": ("risev33", 76, False, 1968)}
# stand-in operator -> the operator name MXNet writes
_JSON_OPS = {"Variable": "null", "reshape": "Reshape", "_split": "SliceChannel", "_neg": "negative"}


def symbol_path(record):
    return os.path.join(ROOT, "tests", "golden", f"{record}-symbol.json.gz")


def tojson(sym):
    """a stand-in Symbol in MXNet's symbol-JSON layout (Symbol.tojson, NNVM graph JSON): the nodes in topological order,
    each operator's parameters and aux states as "null" nodes in front of it in its input order (data, weight, bias;
    data, gamma, beta, moving_mean, moving_var; data, label), inputs as [node, output, 0], the attributes as strings
    under "attrs", arg_nodes the indices of the "null" nodes and heads the outputs of the Group"""
    nodes, ids = [], {}

    def var(name):
        if name not in ids:
            ids[name] = len(nodes)
            nodes.append({"op": "null", "name": name, "inputs": []})
        return [ids[name], 0, 0]

    def ref(s):
        if s.op == "_split_out":
            return [ref(s.inputs[0])[0], s.index, 0]
        if id(s) not in ids:
            ins = [ref(i) for i in s.inputs]
            if s.op == "Variable":
                return var(s.name)
            ins += [var(n) for n in s.params + s.aux]
            ids[id(s)] = len(nodes)
            nd = {"op": _JSON_OPS.get(s.op, s.op), "name": s.name, "inputs": ins}
            if s.attrs:
                nd["attrs"] = {k: str(v) for k, v in s.attrs.items()}
            nodes.append(nd)
        return [ids[id(s)], 0, 0]

    heads = [ref(s) for s in (sym.inputs if sym.op == "Group" else [sym])]
    rows = accumulate(int(n.get("attrs", {}).get("num_outputs", 1)) for n in nodes)
    return json.dumps({"nodes": nodes, "arg_nodes": [i for i, n in enumerate(nodes) if n["op"] == "null"],
                       "node_row_ptr": [0, *rows], "heads": heads, "attrs": {"mxnet_version": ["int", 10600]}})


def main():
    get_v2, get_v33 = load_reference_symbols()
    for record, (symbol, pch, from_plane, labels) in SYMBOLS.items():
        class Args:
            channels_policy_head = pch
            n_labels = labels
            val_loss_factor = 0.01
            policy_loss_factor = 0.99
            select_policy_from_plane = from_plane

        with mx_standin.NameScope():
            sym = (get_v2 if symbol == "risev2" else get_v33)(Args())
        with open(symbol_path(record), "wb") as f:
            f.write(gzip.compress(tojson(sym).encode(), mtime=0))
        print("wrote", symbol_path(record))


if __name__ == "__main__":
    main()
