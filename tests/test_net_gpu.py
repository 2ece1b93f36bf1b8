"""GPU network vs the fp32 oracle (oracle/net.py, pinned to the reference's torch module), through the C-ABI with host
buffers, in both settings of the reference's UCI option `Precision` (engine/src/uci/optionsuci.cpp:144):

  float16 (the reference's default): fp16 tensor-core operands and activations, fp32 accumulation -> value within
          4e-3, probabilities within 3 % of the fp32 oracle;
  float32: the same wgmma GEMMs with fp16 hi + lo operand splitting and fp32 activations between the layers ->
          value and every probability within 1e-4 (north_star's float tolerance), in practice ~1e-6."""
import os

import numpy as np
import pytest

from oracle import net as onet
from tests.golden.gen_net_golden import golden_input

VALUE_ATOL = 4e-3
LOGIT_ATOL = 2.5e-2
PROB_RTOL = 3e-2


F32_ATOL = 1e-4  # north_star: "floats within 1e-4"


def _make_net(tmp_path, arch, batch, version, precision="float16"):
    from crazyara_b200.nn import NeuralNetAPI
    from crazyara_b200.weights import export_blob
    sd = onet.make_state_dict(arch, 0)
    blob = export_blob(sd, arch, str(tmp_path / f"{arch['name']}.arab"), input_version=version)
    return NeuralNetAPI("gpu", 0, batch, blob, precision=precision), sd


CASES = [("risev2", 34, 81, 8, 8), ("risev2", 34, 81, 64, 64), ("risev2", 34, 81, 1, 1), ("risev33", 52, 76, 64, 64),
         ("risev33", 52, 76, 8, 5), ("risev2", 63, 84, 16, 16)]


@pytest.mark.gpu
@pytest.mark.parametrize("name,cin,pch,batch,n", CASES)
def test_net_predict_matches_oracle(tmp_path, name, cin, pch, batch, n):
    arch = onet.arch_risev2(cin, pch) if name == "risev2" else onet.arch_risev33(cin, pch, True)
    net, sd = _make_net(tmp_path, arch, batch, 10 if name == "risev2" else 30)
    assert net.get_nb_policy_values() == pch * 64 and net.get_nb_input_values_total() == cin * 64
    x = golden_input(arch, n=n, seed=5)
    value = np.full(batch, np.nan, np.float32)
    prob = np.full((batch, pch * 64), np.nan, np.float32)
    aux = np.full((batch, 4), np.nan, np.float32)
    xin = np.zeros((batch, cin, 8, 8), np.float32)
    xin[:n] = x
    net.predict(xin, value, prob, aux if arch["wdl"] else None, n=n)
    ref = onet.forward(sd, arch, x)
    assert np.isfinite(value[:n]).all() and np.isfinite(prob[:n]).all()
    np.testing.assert_allclose(prob[:n].sum(1), 1.0, atol=1e-4)
    np.testing.assert_allclose(value[:n], ref["value"], atol=VALUE_ATOL)
    logit_gpu = np.log(prob[:n]) - np.log(prob[:n]).mean(1, keepdims=True)
    logit_ref = ref["policy_logits"] - ref["policy_logits"].mean(1, keepdims=True)
    assert np.abs(logit_gpu - logit_ref).max() < LOGIT_ATOL
    np.testing.assert_allclose(prob[:n], ref["prob"], rtol=PROB_RTOL, atol=1e-7)
    if arch["wdl"]:
        np.testing.assert_allclose(aux[:n], ref["aux"], atol=6e-3)
    # second call must give bit-identical results (graph replay, no stale state)
    value2, prob2 = value.copy(), prob.copy()
    net.predict(xin, value2, prob2, None, n=n)
    assert np.array_equal(value2[:n], value[:n]) and np.array_equal(prob2[:n], prob[:n])
    net.close()


F32_CASES = CASES + [("risev2", 63, 84, 128, 128), ("risev33", 64, 81, 16, 16)]


@pytest.mark.gpu
@pytest.mark.parametrize("name,cin,pch,batch,n", F32_CASES)
def test_net_predict_float32_within_1e4_of_oracle(tmp_path, name, cin, pch, batch, n):
    """Precision float32: value, probabilities (and WDL / plys auxiliary outputs) within 1e-4 of the fp32 oracle."""
    arch = onet.arch_risev2(cin, pch) if name == "risev2" else onet.arch_risev33(cin, pch, True)
    net, sd = _make_net(tmp_path, arch, batch, 10 if name == "risev2" else 30, precision="float32")
    x = golden_input(arch, n=n, seed=5)
    value = np.full(batch, np.nan, np.float32)
    prob = np.full((batch, pch * 64), np.nan, np.float32)
    aux = np.full((batch, 4), np.nan, np.float32)
    xin = np.zeros((batch, cin, 8, 8), np.float32)
    xin[:n] = x
    net.predict(xin, value, prob, aux if arch["wdl"] else None, n=n)
    ref = onet.forward(sd, arch, x)
    np.testing.assert_allclose(value[:n], ref["value"], atol=F32_ATOL, rtol=0)
    np.testing.assert_allclose(prob[:n], ref["prob"], atol=F32_ATOL, rtol=0)
    np.testing.assert_allclose(prob[:n], ref["prob"], rtol=2e-3, atol=1e-8)   # and small probabilities relatively
    logit_gpu = np.log(prob[:n]) - np.log(prob[:n]).mean(1, keepdims=True)
    logit_ref = ref["policy_logits"] - ref["policy_logits"].mean(1, keepdims=True)
    assert np.abs(logit_gpu - logit_ref).max() < 1e-3
    if arch["wdl"]:
        np.testing.assert_allclose(aux[:n], ref["aux"], atol=F32_ATOL)
    value2, prob2 = value.copy(), prob.copy()
    net.predict(xin, value2, prob2, None, n=n)
    assert np.array_equal(value2[:n], value[:n]) and np.array_equal(prob2[:n], prob[:n])
    net.close()


@pytest.mark.gpu
def test_net_create_fails_loudly_on_bad_blob(tmp_path):
    from crazyara_b200 import AraError
    from crazyara_b200.nn import NeuralNetAPI
    p = tmp_path / "bad.arab"
    p.write_bytes(b"not a blob")
    with pytest.raises(AraError):
        NeuralNetAPI("gpu", 0, 8, str(p))
    with pytest.raises(AraError):
        NeuralNetAPI("gpu", 0, 8, str(tmp_path / "missing.arab"))


@pytest.mark.gpu
def test_net_output_of_a_position_does_not_depend_on_its_batch(tmp_path):
    """The search relies on this: a leaf's value / policy are the same bits whichever mini-batch evaluates it."""
    arch = onet.arch_risev2(34, 81)
    x = golden_input(arch, n=64, seed=9)
    net64, _ = _make_net(tmp_path, arch, 64, 10)
    v64, p64 = np.zeros(64, np.float32), np.zeros((64, 81 * 64), np.float32)
    net64.predict(x, v64, p64, None, n=64)
    net64.close()
    net3, _ = _make_net(tmp_path, arch, 3, 10)
    for src in (0, 37, 63):
        xin = np.zeros((3, 34, 8, 8), np.float32)
        xin[1] = x[src]
        xin[0] = x[(src + 5) % 64]
        v, p = np.zeros(3, np.float32), np.zeros((3, 81 * 64), np.float32)
        net3.predict(xin, v, p, None, n=2)
        assert v[1] == v64[src] and np.array_equal(p[1], p64[src])
    net3.close()


@pytest.mark.gpu
@pytest.mark.parametrize("name,cin,pch", [("risev2", 34, 81), ("risev33", 52, 76)])
def test_float16_and_float32_networks_agree(tmp_path, monkeypatch, name, cin, pch):
    """Persistent tower kernel (Precision float16: one board per CTA, then two boards per CTA) against the layer-by-layer
    Precision float32 network: same weights, fp16 tolerance."""
    arch = onet.arch_risev2(cin, pch) if name == "risev2" else onet.arch_risev33(cin, pch, True)
    x = golden_input(arch, n=6, seed=3)
    outs = []
    for env, precision in (({}, "float32"), ({}, "float16"), ({"ARA_TRUNK_ROWS": "128"}, "float16")):
        monkeypatch.delenv("ARA_TRUNK_ROWS", raising=False)
        for k, v in env.items():
            monkeypatch.setenv(k, v)
        net, _ = _make_net(tmp_path, arch, 6, 10 if name == "risev2" else 30, precision=precision)
        v, p = np.zeros(6, np.float32), np.zeros((6, pch * 64), np.float32)
        net.predict(x, v, p, None, n=6)
        net.close()
        outs.append((v, p))
    for v, p in outs[1:]:
        np.testing.assert_allclose(v, outs[0][0], atol=VALUE_ATOL)
        np.testing.assert_allclose(p, outs[0][1], rtol=PROB_RTOL, atol=1e-6)


@pytest.mark.gpu
@pytest.mark.parametrize("name,cin,pch", [("risev2", 34, 81), ("risev33", 52, 76)])
def test_tower_variants_are_bit_identical(tmp_path, monkeypatch, name, cin, pch):
    """The tower kernel's two shapes (one / two boards per CTA) must give the same bits: a search with many trees evaluates
    the same positions in bigger batches.  At 140 boards the default is two boards per CTA."""
    arch = onet.arch_risev2(cin, pch) if name == "risev2" else onet.arch_risev33(cin, pch, True)
    for n, variants in ((5, [{"ARA_TRUNK_ROWS": "128"}, {"ARA_TRUNK_ROWS": "64"}]),
                        (64, [{"ARA_TRUNK_ROWS": "128"}, {"ARA_TRUNK_ROWS": "64"}]),
                        (140, [{}, {"ARA_TRUNK_ROWS": "64"}])):
        x = golden_input(arch, n=n, seed=11)
        outs = []
        for env in variants:
            monkeypatch.delenv("ARA_TRUNK_ROWS", raising=False)
            for k, v in env.items():
                monkeypatch.setenv(k, v)
            net, _ = _make_net(tmp_path, arch, n, 10 if name == "risev2" else 30)
            v, p = np.zeros(n, np.float32), np.zeros((n, pch * 64), np.float32)
            for _ in range(3):  # (repeated: a race in the weight ring would not show every time)
                net.predict(x, v, p, None, n=n)
                outs.append((v.copy(), p.copy()))
            net.close()
        for v, p in outs[1:]:
            assert np.array_equal(v, outs[0][0]) and np.array_equal(p, outs[0][1])
