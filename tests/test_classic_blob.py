"""ARAB2004 weight blobs: networks with a fully-connected policy head (the trainer's select_policy_from_plane=False)
written from a state_dict, read back byte for byte, and refused where the engine could not run them."""
import struct

import numpy as np
import pytest

from crazyara_b200 import synthetic
from crazyara_b200.weights import arch_from_state_dict, export_blob, read_blob, write_blob


def _blob(tmp_path, arch, n_labels, seed=0):
    arch = synthetic.classic(arch, n_labels)
    sd = synthetic.random_state_dict(arch, seed)
    found = arch_from_state_dict(sd)
    assert found["n_labels"] == n_labels
    return export_blob(sd, found, str(tmp_path / f"{arch['name']}.arab")), sd, arch


@pytest.mark.parametrize("base,arch,n_labels", [(1, synthetic.risev2(34, 81), 2272), (1, synthetic.risev33(52, 76), 1968),
                                               (3, synthetic.alpha_vile("tiny", 52, 16), 2316)])
def test_classic_blob_wraps_its_base_format_and_round_trips(tmp_path, base, arch, n_labels):
    path, sd, arch = _blob(tmp_path, arch, n_labels)
    raw = open(path, "rb").read()
    assert raw[:8] == b"ARAB2004" and struct.unpack_from("<2i", raw, 8) == (base, n_labels)
    a, tensors, version = read_blob(path)
    assert a["n_labels"] == n_labels
    P = arch["policy_channels"]
    # the last policy convolution with the head's BatchNorm folded in, then W_fc and b_fc as the trainer holds them
    w2, b2, w_fc, b_fc = tensors[-4:]
    bn = "policy_head.body2.0"
    s = sd[bn + ".weight"].astype(np.float64) / np.sqrt(sd[bn + ".running_var"].astype(np.float64) + 1e-5)
    np.testing.assert_allclose(w2.reshape(P, -1), sd["policy_head.body.3.weight"].reshape(P, -1) * s[:, None], rtol=1e-6, atol=1e-7)
    np.testing.assert_allclose(b2, sd[bn + ".bias"] - sd[bn + ".running_mean"] * s, rtol=1e-6, atol=1e-7)
    assert np.array_equal(w_fc, sd["policy_head.body3.0.weight"].reshape(-1))
    assert np.array_equal(b_fc, sd["policy_head.body3.0.bias"])
    write_blob(str(tmp_path / "again.arab"), a, tensors, version)
    assert open(tmp_path / "again.arab", "rb").read() == raw


def test_policy_map_blobs_keep_their_format(tmp_path):
    arch = synthetic.risev2(34, 81)
    path = export_blob(synthetic.random_state_dict(arch, 0), arch, str(tmp_path / "map.arab"))
    assert open(path, "rb").read()[:8] == b"ARAB2001" and "n_labels" not in read_blob(path)[0]


@pytest.mark.parametrize("patch", [(12, 2000), (12, 4992), (8, 4), (8, 0)])
def test_classic_blob_reader_refuses_unknown_label_counts_and_bases(tmp_path, patch):
    path, _, _ = _blob(tmp_path, synthetic.risev2(34, 2), 2272)
    raw = bytearray(open(path, "rb").read())
    struct.pack_into("<i", raw, *patch)
    bad = tmp_path / "bad.arab"
    bad.write_bytes(bytes(raw))
    with pytest.raises(ValueError):
        read_blob(str(bad))


def test_classic_head_needs_the_bias_in_its_own_tensors(tmp_path):
    arch = dict(synthetic.classic(synthetic.risev2(34, 2), 2272), semantics="mxnet", policy_bias=True, se_gates=[None] * 13)
    with pytest.raises(ValueError):
        write_blob(str(tmp_path / "x.arab"), arch, [], 10)


def test_classic_blob_reader_refuses_a_base_header_with_policy_bias(tmp_path):
    """ARAB2004 around ARAB2003 (AlphaVile: the header has stem_act and policy_bias) with policy_bias set"""
    path, _, _ = _blob(tmp_path, synthetic.alpha_vile("tiny", 34, 2), 2316)
    raw = bytearray(open(path, "rb").read())
    assert struct.unpack_from("<3i", raw, 8) == (3, 2316, 34) and struct.unpack_from("<i", raw, 16 + 36)[0] == 0
    struct.pack_into("<i", raw, 16 + 36, 1)
    bad = tmp_path / "bad.arab"
    bad.write_bytes(bytes(raw))
    with pytest.raises(ValueError, match="policy convolution's bias"):
        read_blob(str(bad))
