"""Pins oracle/net_mx.py (the torch-fp32 restatement of the MXNet RISE symbols) and the ARAB2002 conversion:
 - always: against tests/golden/mx_net_*.json (outputs of the reference's symbol code evaluated by
   tests/golden/mx_standin.py, written by gen_mx_net_golden.py), parameter names included;
 - where the reference tree is present: live against the symbol code;
 - crazyara_b200.weights.export_mx_blob: a NumPy reading of the blob it writes, with the flags it carries, computes the
   oracle's network."""
import json
import os
import struct

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from crazyara_b200.weights import eca_band, export_mx_blob
from oracle import net_mx
from tests.golden.gen_mx_net_golden import ARCHS, REFERENCE, reference_symbol_forward
from tests.golden.gen_net_golden import golden_input

GOLD = os.path.join(os.path.dirname(__file__), "golden")


@pytest.mark.parametrize("name", sorted(ARCHS))
def test_mx_oracle_matches_symbol_golden(name):
    arch = ARCHS[name]()
    with open(os.path.join(GOLD, f"mx_net_{name}.json")) as f:
        g = json.load(f)
    params = net_mx.make_mx_params(arch, g["seed"])
    assert sorted(params) == g["param_names"]
    out = net_mx.forward_mx(params, arch, golden_input(arch, seed=g["input_seed"]))
    idx = np.array(g["prob_idx"])
    np.testing.assert_allclose(out["value"], g["value"], atol=1e-5)
    np.testing.assert_allclose(out["prob"][:, idx], g["prob"], atol=1e-5, rtol=1e-4)
    lp = np.log(out["prob"])
    np.testing.assert_allclose((lp - lp.mean(1, keepdims=True))[:, idx], g["centred_log_prob"], atol=1e-4)
    assert out["prob"].argmax(1).tolist() == g["argmax"]


@pytest.mark.skipif(not os.path.isdir(os.path.join(REFERENCE, "DeepCrazyhouse")), reason="needs the reference tree")
@pytest.mark.parametrize("name", sorted(ARCHS))
def test_mx_oracle_matches_reference_symbols_live(name):
    arch = ARCHS[name]()
    params = net_mx.make_mx_params(arch, 5)
    x = golden_input(arch, n=3, seed=77)
    names, value, prob = reference_symbol_forward(arch, params, x)
    assert names == sorted(params)
    out = net_mx.forward_mx(params, arch, x)
    np.testing.assert_allclose(out["value"], value, atol=1e-5)
    np.testing.assert_allclose(out["prob"], prob, atol=1e-5, rtol=1e-4)


def test_eca_band_is_the_channel_convolution():
    rng = np.random.default_rng(1)
    w, y = rng.standard_normal(5), rng.standard_normal((2, 256))
    conv = F.conv1d(torch.tensor(y)[:, None, :], torch.tensor(w).reshape(1, 1, 5), padding=2)[:, 0].numpy()
    np.testing.assert_allclose(y @ eca_band(w).T, conv, atol=1e-12)


def _blob_forward(path, x):
    """the network an ARAB2002 blob describes (net.cu's reading of it), in torch fp32"""
    b = open(path, "rb").read()
    assert b[:8] == b"ARAB2002"
    h = struct.unpack_from("<10i", b, 8)
    cin, P, nb, stem_act, policy_bias = h[0], h[1], h[2], h[8], h[9]
    o = 48
    blocks = [struct.unpack_from("<5i", b, o + 20 * i) for i in range(nb)]
    o += 20 * nb

    def t(*shape):
        nonlocal o
        n, = struct.unpack_from("<q", b, o)
        a = np.frombuffer(b, "<f4", n, o + 8).copy()
        o += 8 + 4 * n
        return torch.tensor(a).reshape(shape) if shape else torch.tensor(a)

    gates = {0: F.hardsigmoid, 1: lambda y: torch.clamp(0.2 * y + 0.5, 0, 1), 2: torch.sigmoid}
    x = torch.tensor(x)
    out = F.conv2d(x, t(256, cin, 3, 3), t(), padding=1)
    out = F.relu(out) if stem_act else out
    for cop, k, se, flags, gate in blocks:
        d = out
        if se == 1:
            w1, b1 = t(128, 256), t() if flags & 2 else torch.zeros(128)
            w2, b2 = t(256, 128), t() if flags & 2 else torch.zeros(256)
            d = d * gates[gate](F.linear(F.relu(F.linear(d.mean((2, 3)), w1, b1)), w2, b2))[:, :, None, None]
        elif se == 2:
            w, bb = t(256, 256), t()
            d = d * gates[gate](F.linear(d.mean((2, 3)), w, bb))[:, :, None, None]
        hh = F.relu(F.conv2d(d, t(cop, 256, 1, 1), t()))
        hh = F.relu(F.conv2d(hh, t(cop, 1, k, k), t(), padding=k // 2, groups=cop))
        hh = F.conv2d(hh, t(256, cop, 1, 1), t())
        out = hh + (out if flags & 1 else d)
    v = F.relu(F.conv2d(out, t(8, 256, 1, 1), t())).reshape(x.shape[0], -1)
    w1, b1, w2, b2 = t(256, 512), t(), t(1, 256), t()
    v = torch.tanh(F.linear(F.relu(F.linear(v, w1, b1)), w2, b2))[:, 0]
    ph = F.relu(F.conv2d(out, t(256, 256, 3, 3), t(), padding=1))
    w = t(P, 256, 3, 3)
    logits = F.conv2d(ph, w, t() if policy_bias else None, padding=1).reshape(x.shape[0], -1)
    assert o == len(b)
    return v.numpy(), logits.numpy()


@pytest.mark.parametrize("name", sorted(ARCHS))
def test_export_mx_blob_computes_the_oracle_network(tmp_path, name):
    arch = ARCHS[name]()
    params = net_mx.make_mx_params(arch, 2)
    blob = export_mx_blob(params, arch, str(tmp_path / "mx.arab"))
    x = golden_input(arch, n=3, seed=8)
    v, logits = _blob_forward(blob, x)
    ref = net_mx.forward_mx(params, arch, x)
    np.testing.assert_allclose(v, ref["value"], atol=1e-5)
    np.testing.assert_allclose(logits, ref["policy_logits"], atol=2e-4)


def test_export_mx_blob_ignores_fixed_gammas_and_honours_eps(tmp_path):
    arch = net_mx.arch_mx_risev2(34, 81)
    params = net_mx.make_mx_params(arch, 2)
    a = open(export_mx_blob(params, arch, str(tmp_path / "a.arab")), "rb").read()
    params2 = dict(params, stem_bn0_gamma=params["stem_bn0_gamma"] * 3)
    assert open(export_mx_blob(params2, arch, str(tmp_path / "b.arab")), "rb").read() == a
    assert open(export_mx_blob(params2, arch, str(tmp_path / "c.arab"), fix_gamma=False), "rb").read() != a
    assert open(export_mx_blob(params, arch, str(tmp_path / "d.arab"), eps={"stem_bn0": 1e-5}), "rb").read() != a
