"""Generates tests/golden/classic_mx_net_<name>.json by evaluating the reference's OWN MXNet symbol code with a
fully-connected policy head (get_rise_v2_symbol / get_rise_v33_symbol with select_policy_from_plane=False and n_labels =
NB_LABELS, so that builder_util_symbol.py policy_head adds policy_bn1, policy_act1, Flatten and FullyConnected
policy_out) on the seeded parameters of tests/classic_mx_head.py, through the NumPy stand-in for mxnet.sym in
tests/golden/mx_standin.py, as tests/golden/gen_mx_net_golden.py does for the policy-map symbols.  Needs the reference
tree; the GPU machines do not have it, so the records are committed:
    python tests/golden/gen_classic_mx_net_golden.py
It also writes tests/golden/classic_onnx_import_golden.json, the SHA-256 of every ARAB2004 blob the ONNX import and
export_mx_blob write for the test networks with this head (that part needs no reference).
"""
import hashlib
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import net_mx  # noqa: E402
from tests import classic_mx_head  # noqa: E402
from tests.golden import gen_classic_net_golden as gen_torch  # noqa: E402
from tests.golden import mx_standin  # noqa: E402
from tests.golden.gen_mx_net_golden import load_reference_symbols  # noqa: E402
from tests.golden.gen_net_golden import golden_input  # noqa: E402

# (record name, symbol, in_channels, policy_channels, NB_LABELS, input_version)
CASES = (("risev2_2272", "risev2", 34, 81, 2272, 10), ("risev33_1968", "risev33", 52, 76, 1968, 30))
IMPORT_PATH = os.path.join(ROOT, "tests", "golden", "classic_onnx_import_golden.json")
# the ONNX layouts of the torch exports: (flatten, linear, transB)
TORCH_LAYOUTS = {"flatten_gemm": ("Flatten", "Gemm", 1), "reshape_gemm_tb0": ("Reshape", "Gemm", 0),
                 "reshape_matmul": ("Reshape", "MatMul", 1)}


def case_network(symbol, cin, pch, n_labels):
    """-> (classic arch, parameters) of a record"""
    base = net_mx.arch_mx_risev2(cin, pch) if symbol == "risev2" else net_mx.arch_mx_risev33(cin, pch)
    return classic_mx_head.make_params(base, n_labels, 0)


def reference_symbol_forward(arch, params, x):
    """-> (sorted parameter names of the symbol, value [N], policy probabilities [N, L])"""
    get_v2, get_v33 = load_reference_symbols()

    class Args:
        channels_policy_head = arch["policy_channels"]
        n_labels = arch["n_labels"]
        val_loss_factor = 0.01
        policy_loss_factor = 0.99
        select_policy_from_plane = False

    with mx_standin.NameScope():
        sym = (get_v2 if arch["bn_names"] == "v2" else get_v33)(Args())
    names = [a for a in sym.list_arguments() if a != "data" and not a.endswith("_label")] + sym.list_auxiliary_states()
    assert sorted(names) == sorted(params), sorted(set(names) ^ set(params))
    value, prob = sym.eval(dict(params, data=x))[:2]
    return sorted(names), value.reshape(-1), prob


def import_cases(tmp):
    """-> {case: blob path}: import_onnx on the torch writers' files with the head (RISEv2, RISEv3.3 with WDL and
    AlphaVile-tiny of tests/golden/gen_classic_net_golden.py, in each ONNX layout) and on the MXNet writer's, and
    export_mx_blob of the MXNet cases, everything written under tmp"""
    from crazyara_b200.onnx_import import import_onnx
    from crazyara_b200.weights import export_mx_blob
    from tests.onnx_alphavile_writer import write_alphavile_onnx
    from tests.onnx_classic_writer import add_mx_head, add_torch_head
    from tests.onnx_mx_writer import write_mx_onnx
    from tests.onnx_writer import write_rise_onnx
    f = lambda name: os.path.join(tmp, name)
    out = {}
    for name, family, cin, pch, wdl, n_labels in gen_torch.CASES:
        arch, sd, _ = gen_torch.case_network(family, cin, pch, wdl, n_labels)
        write = write_alphavile_onnx if family == "alphavile" else write_rise_onnx
        for layout, (flatten, linear, trans_b) in TORCH_LAYOUTS.items():
            onnx = add_torch_head(write(sd, arch, f(f"{name}-{layout}.onnx")), sd, flatten, linear, trans_b)
            out[f"import_onnx/{name}_{layout}"] = blob = f(f"{name}-{layout}.arab")
            import_onnx(onnx, blob)
    for name, symbol, cin, pch, n_labels, version in CASES:
        arch, params = case_network(symbol, cin, pch, n_labels)
        out["export_mx_blob/mx_" + name] = export_mx_blob(params, arch, f(f"mx_{name}.arab"), input_version=version)
        onnx = add_mx_head(write_mx_onnx(params, arch, f(f"mx_{name}.onnx")), params)
        out["import_onnx/mx_" + name] = blob = f(f"mx_{name}-onnx.arab")
        import_onnx(onnx, blob)
    return out


def import_hashes(tmp):
    return {k: hashlib.sha256(open(p, "rb").read()).hexdigest() for k, p in sorted(import_cases(tmp).items())}


def main():
    for name, symbol, cin, pch, n_labels, _ in CASES:
        arch, params = case_network(symbol, cin, pch, n_labels)
        x = golden_input(arch)
        names, value, prob = reference_symbol_forward(arch, params, x)
        assert prob.shape == (x.shape[0], n_labels)
        idx = np.arange(0, n_labels, 7)  # every 7th label: a flatten or row order off by one moves every one of them
        logp = np.log(prob)
        rec = dict(name=name, symbol=symbol, in_channels=cin, policy_channels=pch, n_labels=n_labels, seed=0, input_seed=123,
                   param_names=names, value=value.tolist(), prob_idx=idx.tolist(), prob=prob[:, idx].tolist(),
                   centred_log_prob=(logp - logp.mean(1, keepdims=True))[:, idx].tolist(), argmax=prob.argmax(1).tolist())
        path = os.path.join(ROOT, "tests", "golden", f"classic_mx_net_{name}.json")
        with open(path, "w") as f:
            json.dump(rec, f)
        print("wrote", path, "value", value)
    import tempfile
    with tempfile.TemporaryDirectory() as d, open(IMPORT_PATH, "w") as f:
        json.dump(import_hashes(d), f, indent=1, sort_keys=True)
    print("wrote", IMPORT_PATH)


if __name__ == "__main__":
    main()
