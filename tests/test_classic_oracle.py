"""The fully-connected policy head's oracle (tests/classic_head.py) and its import pinned to the reference: the real
network definitions with select_policy_from_plane=False (tests/golden/gen_classic_net_golden.py) for RISEv2 (34 planes,
2272 labels), RISEv3.3 with WDL (52 planes, 1968 labels) and AlphaVile-tiny (2316 labels), within the tolerances
tests/test_oracle_net.py holds the policy-map oracle to; and the bytes of the blobs the state-dict import writes."""
import json
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from tests import classic_head
from tests.golden import gen_classic_net_golden as gen
from tests.golden.gen_net_golden import golden_input

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _record(name):
    with open(os.path.join(GOLDEN, f"classic_net_{name}.json")) as f:
        return json.load(f)


def _assert_matches(g, value, logits, aux):
    idx = np.asarray(g["logit_idx"])
    np.testing.assert_allclose(value, g["value"], atol=2e-6)
    np.testing.assert_allclose(logits[:, idx], g["logits"], atol=2e-5)
    prob = torch.softmax(torch.as_tensor(logits), dim=1).numpy()
    np.testing.assert_allclose(prob[:, idx], g["prob"], rtol=1e-4, atol=1e-9)
    np.testing.assert_allclose(logits.sum(1), g["logits_sum"], rtol=1e-4, atol=1e-2)
    np.testing.assert_allclose(np.abs(logits).sum(1), g["logits_abs_sum"], rtol=1e-4)
    assert logits.argmax(1).tolist() == g["argmax"]
    if g["aux"] is not None:
        np.testing.assert_allclose(aux, g["aux"], atol=2e-6)


CASES = {c[0]: c for c in gen.CASES}


@pytest.mark.parametrize("name", sorted(CASES))
def test_classic_oracle_matches_the_reference(name):
    _, family, cin, pch, wdl, n_labels = CASES[name]
    arch, sd, forward = gen.case_network(family, cin, pch, wdl, n_labels)
    g = _record(name)
    assert g["n_labels"] == n_labels
    out = classic_head.forward(forward, sd, arch, golden_input(arch))
    assert out["policy_logits"].shape == (4, n_labels)
    _assert_matches(g, out["value"], out["policy_logits"], out["aux"])


@pytest.mark.parametrize("name", sorted(CASES))
def test_imported_classic_head_computes_the_reference_logits(tmp_path, name):
    """the head as the blob holds it (both BatchNorms folded, W_fc in the trainer's flatten order) on the oracle's trunk"""
    from crazyara_b200.weights import export_blob, read_blob
    _, family, cin, pch, wdl, n_labels = CASES[name]
    arch, sd, forward = gen.case_network(family, cin, pch, wdl, n_labels)
    x = golden_input(arch)
    out = forward(sd, arch, x)
    a, tensors, _ = read_blob(export_blob(sd, arch, str(tmp_path / "c.arab")))
    assert a["n_labels"] == n_labels
    w1, b1, w2, b2, w_fc, b_fc = (torch.as_tensor(t) for t in tensors[-6:])
    C = out["trunk"].shape[1]
    with torch.no_grad():
        h = F.relu(F.conv2d(torch.as_tensor(out["trunk"]), w1.reshape(C, C, 3, 3), b1, padding=1))
        h = F.relu(F.conv2d(h, w2.reshape(pch, C, 3, 3), b2, padding=1)).reshape(x.shape[0], -1)
        logits = F.linear(h, w_fc.reshape(n_labels, pch * 64), b_fc).numpy()
    _assert_matches(_record(name), out["value"], logits, out["aux"])


def test_classic_import_matches_the_hash_record(tmp_path):
    with open(gen.IMPORT_PATH) as f:
        assert gen.import_hashes(str(tmp_path)) == json.load(f)
