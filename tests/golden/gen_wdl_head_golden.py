"""Generates tests/golden/wdl_head_golden.json and the symbols tests/golden/mx_wdl_net_risev33_52_<head>-symbol.json.gz
for the value heads of tests/wdl_heads.py, from the reference's OWN network code:
  - get_rise_v33_model and get_alpha_vile_model("tiny") (pytorch/rise_mobile_v3.py, pytorch/alpha_vile.py) with
    use_wdl = use_plys_to_end = use_mlp_wdl_ply = True, on the seeded state dicts of tests/wdl_heads.mlp_state_dict;
  - rise_mobile_v3_symbol (rise_mobile_v3.py) with RISEv3.3's kernels and eca_se blocks (as get_rise_v33_symbol builds
    them), use_wdl = use_plys_to_end = True, without and with use_mlp_wdl_ply, over the NumPy stand-in for mxnet.sym
    (tests/golden/mx_standin.py, whose SoftmaxOutput returns the softmax, MXNet's forward), on the seeded parameters of
    tests/wdl_heads.mx_params.
Each record holds the value, the auxiliary outputs (WDL logits and plies for PyTorch, the symbol's WDL probabilities and
plies for MXNet), a sample of the policy, the parameter names, and the SHA-256 of the blob the exporters write for the
network (weights.export_blob / export_mx_blob), which every import path must reproduce (for MXNet ONNX exports, whose
BatchNormalization epsilon is a float32, the blob folded with that epsilon).  Run where the reference tree is
present (the GPU machines do not have it):
    python tests/golden/gen_wdl_head_golden.py
"""
import gzip
import hashlib
import json
import os
import sys
import tempfile

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import net as onet  # noqa: E402
from oracle import net_alphavile as oav  # noqa: E402
from oracle import net_mx  # noqa: E402
from crazyara_b200.weights import export_blob, export_mx_blob  # noqa: E402
from tests import wdl_heads  # noqa: E402
from tests.golden import mx_standin  # noqa: E402
from tests.golden.gen_mx_net_golden import load_reference_symbols  # noqa: E402
from tests.golden.gen_mx_symbol_golden import tojson  # noqa: E402
from tests.golden.gen_net_golden import golden_input, load_reference_models  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden", "wdl_head_golden.json")
VERSION = {"risev33_mlp": 30, "av_tiny_mlp": 10, "mx_wdl": 30, "mx_wdl_mlp": 30}  # the blobs' input versions


def torch_archs():
    return {"risev33_mlp": dict(onet.arch_risev33(52, 76, True), value_head="wdl_mlp"),
            "av_tiny_mlp": dict(oav.arch_alphavile("tiny", 34, 81, True), value_head="wdl_mlp")}


def mx_archs():
    base = net_mx.arch_mx_risev33(52, 76)
    return {h: wdl_heads.mx_arch(base, h) for h in ("mx_wdl", "mx_wdl_mlp")}


def symbol_path(head):
    return os.path.join(ROOT, "tests", "golden", f"mx_wdl_net_risev33_52_{head}-symbol.json.gz")


def torch_reference(key, arch, sd_np, x):
    load_reference_models()
    from DeepCrazyhouse.src.domain.neural_net.architectures.pytorch.alpha_vile import get_alpha_vile_model
    from DeepCrazyhouse.src.domain.neural_net.architectures.pytorch.rise_mobile_v3 import get_rise_v33_model

    class Args:
        input_shape = (arch["in_channels"], 8, 8)
        channels_policy_head = arch["policy_channels"]
        select_policy_from_plane = True
        n_labels = 2272
        use_wdl = use_plys_to_end = use_mlp_wdl_ply = True

    model = get_alpha_vile_model(Args(), model_size="tiny") if "ntb" in arch else get_rise_v33_model(Args())
    sd = model.state_dict()
    keys = {k for k in sd if not k.endswith("num_batches_tracked")}
    assert keys == set(sd_np), (sorted(keys - set(sd_np)), sorted(set(sd_np) - keys))
    for k, v in sd_np.items():
        assert tuple(sd[k].shape) == tuple(v.shape), (k, sd[k].shape, v.shape)
        sd[k] = torch.from_numpy(v)
    model.load_state_dict(sd)
    model.eval()
    with torch.no_grad():
        out = model(torch.from_numpy(x))
    return sorted(keys), out[0].numpy()[:, 0], torch.softmax(out[1], dim=1).numpy(), out[2].numpy()


def mx_symbol(arch):
    load_reference_symbols()
    from DeepCrazyhouse.src.domain.neural_net.architectures.rise_mobile_v3 import rise_mobile_v3_symbol
    with mx_standin.NameScope():
        return rise_mobile_v3_symbol(channels=256, channels_operating_init=224, channel_expansion=32, act_type="relu",
                                     channels_value_head=8, value_fc_size=arch["value_fc"],
                                     channels_policy_head=arch["policy_channels"], grad_scale_value=0.01,
                                     grad_scale_policy=0.99, dropout_rate=0, select_policy_from_plane=True,
                                     kernels=arch["kernels"], se_types=arch["se_types"], use_avg_features=False,
                                     n_labels=2272, use_wdl=True, use_plys_to_end=True,
                                     use_mlp_wdl_ply=arch["value_head"] == "mx_wdl_mlp")


def mx_reference(arch, params, x):
    sym = mx_symbol(arch)
    names = [a for a in sym.list_arguments() if a != "data" and not a.endswith("_label")] + sym.list_auxiliary_states()
    value, prob, aux = sym.eval(dict(params, data=x))[:3]
    return sym, sorted(names), value.reshape(-1), prob, aux


def blob_sha256(export, weights, arch, version):
    with tempfile.TemporaryDirectory() as d:
        path = export(weights, arch, os.path.join(d, "net.arab"), input_version=version)
        return hashlib.sha256(open(path, "rb").read()).hexdigest()


def record(names, value, prob, aux, sha):
    idx = np.arange(0, prob.shape[1], 97)
    return dict(param_names=names, value=value.tolist(), aux=aux.tolist(), prob_idx=idx.tolist(),
                prob=prob[:, idx].tolist(), argmax=prob.argmax(1).tolist(), blob_sha256=sha)


def main():
    out = {}
    for key, arch in torch_archs().items():
        sd = wdl_heads.mlp_state_dict(arch, 0)
        x = golden_input(arch)
        out[key] = record(*torch_reference(key, arch, sd, x), blob_sha256(export_blob, sd, arch, VERSION[key]))
        print(key, "value", out[key]["value"])
    for head, arch in mx_archs().items():
        params = wdl_heads.mx_params(arch, 0)
        sym, names, value, prob, aux = mx_reference(arch, params, golden_input(arch))
        out[head] = record(names, value, prob, aux, blob_sha256(export_mx_blob, params, arch, VERSION[head]))
        # an ONNX BatchNormalization holds its epsilon as a float32: the MXNet export's blob folds with that epsilon
        f32_eps = lambda *a, **k: export_mx_blob(*a, **k, eps=float(np.float32(1e-3)))
        out[head]["onnx_blob_sha256"] = blob_sha256(f32_eps, params, arch, VERSION[head])
        with open(symbol_path(head), "wb") as f:
            f.write(gzip.compress(tojson(sym).encode(), mtime=0))
        print(head, "value", out[head]["value"], "wrote", symbol_path(head))
    with open(GOLDEN, "w") as f:
        json.dump(out, f)
    print("wrote", GOLDEN)


if __name__ == "__main__":
    main()
