"""Generates tests/golden/classic_net_<name>.json by running the REAL reference network definitions with a
fully-connected policy head (select_policy_from_plane=False, n_labels = NB_LABELS: rise_mobile_v3.py get_rise_v2_model /
get_rise_v33_model, alpha_vile.py get_alpha_vile_model, whose _PolicyHead, builder_util.py:206-243, then has body2 =
BatchNorm + ReLU and body3 = Linear) on the seeded state dicts of oracle/net.py and oracle/net_alphavile.py with the
head of crazyara_b200.synthetic.classic_head.  Needs the reference tree (and einops for AlphaVile); the GPU box has
neither, so the records are committed:
    python tests/golden/gen_classic_net_golden.py
It also writes tests/golden/classic_import_golden.json, the SHA-256 of the ARAB2004 blob the state-dict import writes for
each of these networks (that part needs no reference).
"""
import hashlib
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from crazyara_b200 import synthetic  # noqa: E402
from oracle import net as onet  # noqa: E402
from oracle import net_alphavile as oav  # noqa: E402
from tests.golden.gen_net_golden import golden_input, load_reference_models  # noqa: E402

# (record name, family, in_channels, policy_channels, wdl, NB_LABELS)
CASES = (("risev2_2272", "risev2", 34, 81, False, 2272), ("risev33_1968", "risev33", 52, 76, True, 1968),
         ("alphavile_tiny_2316", "alphavile", 34, 81, False, 2316))


def case_network(family, cin, pch, wdl, n_labels):
    """-> (arch, state dict, oracle forward) of a record"""
    if family == "alphavile":
        arch, om = oav.arch_alphavile("tiny", cin, pch, wdl), oav
    else:
        arch, om = (onet.arch_risev2(cin, pch) if family == "risev2" else onet.arch_risev33(cin, pch, wdl)), onet
    arch = synthetic.classic(arch, n_labels)
    sd = om.make_state_dict(arch, 0)
    sd.update(synthetic.classic_head(arch, n_labels, 0))
    return arch, sd, om.forward


IMPORT_PATH = os.path.join(ROOT, "tests", "golden", "classic_import_golden.json")


def import_hashes(tmp):
    """{record name: SHA-256 of weights.import_checkpoint's blob of the record's state dict}"""
    from crazyara_b200.weights import import_checkpoint
    out = {}
    for name, family, cin, pch, wdl, n_labels in CASES:
        _, sd, _ = case_network(family, cin, pch, wdl, n_labels)
        ck, blob = os.path.join(tmp, name + ".pt"), os.path.join(tmp, name + ".arab")
        torch.save({"model_state_dict": {k: torch.from_numpy(v) for k, v in sd.items()}}, ck)
        import_checkpoint(ck, blob)
        out[name] = hashlib.sha256(open(blob, "rb").read()).hexdigest()
    return out


def reference_forward(family, arch, sd_np, x):
    get_v2, get_v33 = load_reference_models()

    class Args:
        pass

    a = Args()
    a.input_shape = (arch["in_channels"], 8, 8)
    a.channels_policy_head = arch["policy_channels"]
    a.select_policy_from_plane = False
    a.n_labels = arch["n_labels"]
    a.use_wdl = a.use_plys_to_end = arch["wdl"]
    a.use_mlp_wdl_ply = False
    if family == "alphavile":
        from DeepCrazyhouse.src.domain.neural_net.architectures.pytorch.alpha_vile import get_alpha_vile_model
        model = get_alpha_vile_model(a, model_size="tiny")
    else:
        model = (get_v2 if family == "risev2" else get_v33)(a)
    sd = model.state_dict()
    missing = [k for k in sd if k not in sd_np and not k.endswith("num_batches_tracked")
               and not (arch["wdl"] and k.startswith("value_head.body_final"))]
    assert not missing, missing
    extra = [k for k in sd_np if k not in sd]
    assert not extra, extra
    for k, v in sd_np.items():
        assert tuple(sd[k].shape) == tuple(v.shape), (k, sd[k].shape, v.shape)
        sd[k] = torch.from_numpy(v)
    model.load_state_dict(sd)
    model.eval()
    with torch.no_grad():
        out = model(torch.from_numpy(x))
    return out[0].numpy()[:, 0], out[1].numpy(), out[2].numpy() if arch["wdl"] else None


def main():
    for name, family, cin, pch, wdl, n_labels in CASES:
        arch, sd, _ = case_network(family, cin, pch, wdl, n_labels)
        x = golden_input(arch)
        value, logits, aux = reference_forward(family, arch, sd, x)
        assert logits.shape == (x.shape[0], n_labels)
        prob = torch.softmax(torch.from_numpy(logits), dim=1).numpy()
        idx = np.arange(0, n_labels, 7)  # every 7th label: a flatten or row order off by one moves every one of them
        rec = dict(name=name, family=family, in_channels=cin, policy_channels=pch, wdl=wdl, n_labels=n_labels, seed=0,
                   input_seed=123, value=value.tolist(), aux=None if aux is None else aux.tolist(), logit_idx=idx.tolist(),
                   logits=logits[:, idx].tolist(), prob=prob[:, idx].tolist(), logits_sum=logits.sum(1).tolist(),
                   logits_abs_sum=np.abs(logits).sum(1).tolist(), argmax=logits.argmax(1).tolist())
        path = os.path.join(ROOT, "tests", "golden", f"classic_net_{name}.json")
        with open(path, "w") as f:
            json.dump(rec, f)
        print("wrote", path, "value", value)
    import tempfile
    with tempfile.TemporaryDirectory() as d, open(IMPORT_PATH, "w") as f:
        json.dump(import_hashes(d), f, indent=1, sort_keys=True)
    print("wrote", IMPORT_PATH)


if __name__ == "__main__":
    main()
