"""Generates tests/golden/mx_net_<arch>.json by evaluating the reference's OWN MXNet symbol code
(get_rise_v2_symbol in rise_mobile_v2.py, get_rise_v33_symbol in rise_mobile_v3.py, over builder_util_symbol.py) on the
seeded parameters of oracle/net_mx.py, through the NumPy stand-in for mxnet.sym in tests/golden/mx_standin.py.  Run where
the reference tree is present (the GPU machines do not have it):
    python tests/golden/gen_mx_net_golden.py
"""
import json
import os
import sys
import types

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import net_mx  # noqa: E402
from tests.golden import mx_standin  # noqa: E402
from tests.golden.gen_net_golden import golden_input  # noqa: E402

REFERENCE = "/root/reference"
ARCHS = {"risev2_34": lambda: net_mx.arch_mx_risev2(34, 81), "risev33_52": lambda: net_mx.arch_mx_risev33(52, 76)}


def load_reference_symbols():
    """the reference's symbol builders over the stand-in; rise_mobile_v2.py's variant constants come from a module that
    needs python-chess, so that module is replaced by the two constants it reads (only used with
    use_extra_variant_input, which RISEv2 leaves off)"""
    mx_standin.install()
    consts = types.ModuleType("DeepCrazyhouse.src.domain.variants.constants")
    consts.NB_CHANNELS_TOTAL, consts.NB_CHANNELS_VARIANTS = 34, 9
    sys.modules.setdefault("DeepCrazyhouse.src.domain.variants.constants", consts)
    if REFERENCE not in sys.path:
        sys.path.insert(0, REFERENCE)
    from DeepCrazyhouse.src.domain.neural_net.architectures.rise_mobile_v2 import get_rise_v2_symbol
    from DeepCrazyhouse.src.domain.neural_net.architectures.rise_mobile_v3 import get_rise_v33_symbol
    return get_rise_v2_symbol, get_rise_v33_symbol


def reference_symbol_forward(arch, params, x):
    """-> (sorted parameter names of the symbol, value [N], policy probabilities [N, P*64])"""
    get_v2, get_v33 = load_reference_symbols()

    class Args:
        channels_policy_head = arch["policy_channels"]
        n_labels = 2272
        val_loss_factor = 0.01
        policy_loss_factor = 0.99
        select_policy_from_plane = True

    with mx_standin.NameScope():
        sym = (get_v2 if arch["bn_names"] == "v2" else get_v33)(Args())
    names = [a for a in sym.list_arguments() if a != "data" and not a.endswith("_label")] + sym.list_auxiliary_states()
    feed = dict(params, data=x)
    value, prob = sym.eval(feed)[:2]
    return sorted(names), value.reshape(-1), prob


def main():
    for key, mk in ARCHS.items():
        arch = mk()
        params = net_mx.make_mx_params(arch, seed=0)
        x = golden_input(arch)
        names, value, prob = reference_symbol_forward(arch, params, x)
        idx = np.arange(0, prob.shape[1], 97)
        logp = np.log(prob)
        rec = dict(arch=arch["name"], in_channels=arch["in_channels"], policy_channels=arch["policy_channels"], seed=0,
                   input_seed=123, param_names=names, value=value.tolist(), prob_idx=idx.tolist(),
                   prob=prob[:, idx].tolist(), centred_log_prob=(logp - logp.mean(1, keepdims=True))[:, idx].tolist(),
                   argmax=prob.argmax(1).tolist())
        path = os.path.join(ROOT, "tests", "golden", f"mx_net_{key}.json")
        with open(path, "w") as f:
            json.dump(rec, f)
        print("wrote", path, "value", value)


if __name__ == "__main__":
    main()
