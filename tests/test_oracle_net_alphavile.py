"""AlphaVile on the CPU: the oracle (oracle/net_alphavile.py) against the real reference module's outputs
(tests/golden/net_alphavile_*.json, written by tests/golden/gen_alphavile_golden.py), architecture recognition, and the
ARAB2003 blob read back by weights.read_blob and run with the trunk padded to 256 channels the way Net::read_blob does."""
import json
import os
import struct

import numpy as np
import pytest
import torch

from crazyara_b200 import synthetic
from crazyara_b200.weights import arch_from_state_dict, export_blob, import_checkpoint, read_blob
from oracle import net_alphavile as oav
from tests.golden.gen_net_golden import golden_input

GOLD = os.path.join(os.path.dirname(__file__), "golden")
CASES = {"tiny_34": ("tiny", 34, 81, False), "normal_52": ("normal", 52, 76, True)}


def case_arch(name):
    size, cin, pch, wdl = CASES[name]
    return oav.arch_alphavile(size, cin, pch, wdl)


@pytest.mark.parametrize("name", sorted(CASES))
def test_oracle_matches_reference_golden(name):
    arch = case_arch(name)
    with open(os.path.join(GOLD, f"net_alphavile_{name}.json")) as f:
        g = json.load(f)
    out = oav.forward(oav.make_state_dict(arch, g["seed"]), arch, golden_input(arch, seed=g["input_seed"]))
    idx = np.array(g["logit_idx"])
    np.testing.assert_allclose(out["value"], g["value"], atol=2e-6)
    np.testing.assert_allclose(out["policy_logits"][:, idx], g["logits"], atol=2e-5)
    np.testing.assert_allclose(out["prob"][:, idx], g["prob"], rtol=1e-4, atol=1e-9)
    np.testing.assert_allclose(out["policy_logits"].sum(1), g["logits_sum"], rtol=1e-4, atol=1e-2)
    assert out["policy_logits"].argmax(1).tolist() == g["argmax"]
    if g["aux"] is not None:
        np.testing.assert_allclose(out["aux"], g["aux"], atol=2e-6)


@pytest.mark.parametrize("name", sorted(CASES))
def test_seeded_attention_is_neither_uniform_nor_one_hot(name):
    arch = case_arch(name)
    stats = []
    oav.forward(oav.make_state_dict(arch, 0), arch, golden_input(arch), stats)
    assert len(stats) == sum(arch["ntb"])
    for a in stats:
        top = float(a.max(-1).values.mean())
        assert 2.0 / 64 < top < 0.9, top


@pytest.mark.parametrize("size", oav.SIZES)
def test_architecture_is_read_off_the_state_dict(size):
    arch = oav.arch_alphavile(size, 52, 76, size != "tiny")
    got = arch_from_state_dict(oav.make_state_dict(arch, 1))
    for k in ("in_channels", "policy_channels", "channels", "ntb", "mhsa", "mhca", "mlp", "wdl", "value_fc"):
        assert got[k] == arch[k], k
    plain = lambda a: [(k, c) for k, c, t in zip(a["kernels"], a["c_ops"], a["ntb"]) if not t]
    assert plain(got) == plain(arch)


@pytest.mark.parametrize("size", oav.SIZES)
def test_synthetic_table_matches_the_reference(size):
    a, b = synthetic.alpha_vile(size, 34, 81, False), oav.arch_alphavile(size, 34, 81, False)
    assert {k: a[k] for k in b} == b
    sd = synthetic.random_state_dict(a, 0)
    assert set(sd) == set(oav.make_state_dict(b, 0))


def test_checkpoint_import_equals_direct_export(tmp_path):
    arch = case_arch("normal_52")
    sd = oav.make_state_dict(arch, 2)
    ck = tmp_path / "model.tar"
    torch.save({"model_state_dict": {"module." + k: torch.from_numpy(v) for k, v in sd.items()}}, ck)
    a = import_checkpoint(str(ck), str(tmp_path / "a.arab"))
    export_blob(sd, arch, str(tmp_path / "b.arab"), input_version=30)
    assert a["ntb"] == arch["ntb"]
    assert (tmp_path / "a.arab").read_bytes() == (tmp_path / "b.arab").read_bytes()
    assert (tmp_path / "a.arab").read_bytes()[:8] == b"ARAB2003"


# ------------------------------------------------------------------------------------------- ARAB2003 read back
def pad(a, shape):
    o = np.zeros(shape)
    o[tuple(slice(0, s) for s in a.shape)] = a
    return o


def blob_forward(path, x):
    """the network an ARAB2003 blob describes, padded to 256 channels, in float64 NumPy / torch"""
    import torch.nn.functional as F
    arch, ts, _ = read_blob(path)
    C, cin, P, fc = arch["channels"], arch["in_channels"], arch["policy_channels"], arch["value_fc"]
    it = iter(ts)
    nxt = lambda *shape: next(it).astype(np.float64).reshape(shape)
    T = lambda a: torch.from_numpy(np.ascontiguousarray(a))
    conv = lambda x, w, b=None, pd=0, groups=1: F.conv2d(x, T(w), None if b is None else T(b), padding=pd, groups=groups)
    x = torch.as_tensor(x, dtype=torch.float64)
    out = F.relu(conv(x, pad(nxt(C, cin, 3, 3), (256, cin, 3, 3)), pad(nxt(C), (256,)), 1))
    for is_ntb, cop, k in zip(arch["ntb"], arch["c_ops"], arch["kernels"]):
        if not is_ntb:
            h = F.relu(conv(out, pad(nxt(cop, C, 1, 1), (cop, 256, 1, 1)), nxt(cop)))
            h = F.relu(conv(h, nxt(cop, 1, k, k), nxt(cop), k // 2, cop))
            out = out + conv(h, pad(nxt(C, cop, 1, 1), (256, cop, 1, 1)), pad(nxt(C), (256,)))
            continue
        M, Ca, H = arch["mhsa"], arch["mhca"], arch["mlp"]
        y = conv(out, pad(nxt(M, C, 1, 1), (M, 256, 1, 1)), nxt(M))
        qkv = F.conv2d(y, T(nxt(3 * M, M, 1, 1)), T(nxt(3 * M))).flatten(2).transpose(1, 2)  # [B, 64, 3M]
        q, k, v = (qkv[..., i * M:(i + 1) * M].reshape(-1, 64, M // 32, 32).transpose(1, 2) for i in range(3))
        att = torch.softmax(q @ k.transpose(-1, -2) / np.sqrt(32.0), -1) @ v
        att = att.transpose(1, 2).reshape(-1, 64, M).transpose(1, 2).reshape(-1, M, 8, 8)
        y1 = y + conv(att, nxt(M, M, 1, 1), nxt(M))
        z = conv(y1, nxt(Ca, M, 1, 1), nxt(Ca))
        g = F.relu(conv(z, nxt(Ca, 32, 3, 3), nxt(Ca), 1, Ca // 32))
        z2 = z + conv(g, nxt(Ca, Ca, 1, 1))
        x2 = torch.cat([y1, z2, torch.zeros_like(out[:, C:])], 1)
        u = F.relu(conv(x2, pad(nxt(H, C, 1, 1), (H, 256, 1, 1)), nxt(H)))
        out = x2 + conv(u, pad(nxt(C, H, 1, 1), (256, H, 1, 1)), pad(nxt(C), (256,)))
    assert torch.count_nonzero(out[:, C:]) == 0
    vh = F.relu(conv(out, pad(nxt(8, C, 1, 1), (8, 256, 1, 1)), nxt(8))).reshape(x.shape[0], -1)
    if arch["wdl"]:
        wdl = vh @ T(nxt(3, 512)).T + T(nxt(3))
        nxt(1, 512), nxt(1)
        sm = torch.softmax(wdl, 1)
        value = sm[:, 2] - sm[:, 0]
    else:
        h = F.relu(vh @ T(pad(nxt(fc, 512), (256, 512))).T + T(pad(nxt(fc), (256,))))
        value = torch.tanh(h @ T(pad(nxt(1, fc), (1, 256))).T + T(nxt(1)))[:, 0]
    ph = F.relu(conv(out, pad(nxt(C, C, 3, 3), (256, 256, 3, 3)), pad(nxt(C), (256,)), 1))
    logits = conv(ph, pad(nxt(P, C, 3, 3), (P, 256, 3, 3)), None, 1).reshape(x.shape[0], -1)
    assert next(it, None) is None
    return value.numpy(), logits.numpy()


@pytest.mark.parametrize("name", sorted(CASES))
def test_blob_read_back_matches_oracle(tmp_path, name):
    arch = case_arch(name)
    sd = oav.make_state_dict(arch, 3)
    blob = export_blob(sd, arch, str(tmp_path / "w.arab"), input_version=10)
    x = golden_input(arch, n=3, seed=5)
    value, logits = blob_forward(blob, x)
    ref = oav.forward(sd, arch, x)
    np.testing.assert_allclose(value, ref["value"], atol=1e-5)
    np.testing.assert_allclose(logits, ref["policy_logits"], atol=1e-5 * max(1.0, np.abs(ref["policy_logits"]).max()))


# ------------------------------------------------------------------------------------------- malformed blobs
def _rewrite(path, out, header=None, block=None):
    buf = bytearray(open(path, "rb").read())
    if header is not None:
        i, v = header
        struct.pack_into("<i", buf, 8 + 4 * i, v)
    if block is not None:
        b, field, v = block
        struct.pack_into("<i", buf, 48 + 16 * b + 4 * field, v)
    open(out, "wb").write(bytes(buf))
    return str(out)


@pytest.mark.parametrize("edit, message", [
    (dict(header=(3, 200)), "unsupported trunk geometry"),         # channels not a multiple of 32
    (dict(header=(3, 288)), "unsupported trunk geometry"),         # wider than 256
    (dict(header=(5, 300)), "unsupported trunk geometry"),         # value_fc > 256
    (dict(block=(0, 0, 1)), "block 0 is an NTB"),
    (dict(block=(14, 2, 48)), "unsupported NTB widths"),           # Ca not in {32, 64}
    (dict(block=(14, 1, 96)), "unsupported NTB widths"),           # M + Ca != C
    (dict(block=(14, 3, 400)), "unsupported NTB widths"),          # H % 64 != 0
    (dict(block=(3, 3, 1)), "squeeze-excitation on a 192-channel trunk"),
    (dict(block=(3, 0, 7)), "has type 7"),
])
def test_malformed_arab2003_blobs_fail_loudly(tmp_path, edit, message):
    from crazyara_b200._lib import AraError
    from crazyara_b200.nn import NeuralNetAPI
    arch = oav.arch_alphavile("tiny", 34, 81, False)
    good = export_blob(synthetic.random_state_dict(arch, 0), arch, str(tmp_path / "good.arab"), input_version=10)
    bad = _rewrite(good, tmp_path / "bad.arab", **edit)
    with pytest.raises(AraError, match=message):
        NeuralNetAPI("gpu", 0, 1, bad)


def test_truncated_arab2003_blob_fails_loudly(tmp_path):
    from crazyara_b200._lib import AraError
    from crazyara_b200.nn import NeuralNetAPI
    arch = oav.arch_alphavile("tiny", 34, 81, False)
    good = export_blob(synthetic.random_state_dict(arch, 0), arch, str(tmp_path / "good.arab"), input_version=10)
    buf = open(good, "rb").read()
    (tmp_path / "cut.arab").write_bytes(buf[:len(buf) // 2])
    with pytest.raises(AraError):
        NeuralNetAPI("gpu", 0, 1, str(tmp_path / "cut.arab"))
