"""Weight import: reference state_dict (PyTorch parameter names of RiseV3) -> ARAB2001 blob for ara_net_create, and
MXNet-named parameters of the reference's symbol networks (rise_mobile_v2.py, rise_mobile_v3.py) -> ARAB2002 blob.

BatchNorm (eval mode, eps 1e-5) is folded into the preceding convolution here, in float64, so the CUDA side only
sees conv weight + bias.  The blob is architecture-described by its header, so any RISEv2 / RISEv3.x checkpoint of
the reference trainer (trainer_agent_pytorch.py:506-516 saves {'model_state_dict': ...}) converts without code
changes.  Tensor order must match crazyara_b200/csrc/net.cu (Net::read_blob).

The MXNet symbols compute a different network from the same layers (export_mx_blob): a block's shortcut is its input
before the squeeze-excitation, ca_se has fully-connected biases and a sigmoid (RISEv2) or clamp(0.2 x + 0.5) gate
(v3), eca_se is a 5-tap convolution over the channel axis with one bias, the v3 stem has no activation and the v3
policy convolution a bias, and BatchNorm has MXNet's defaults (eps 1e-3, gamma fixed to 1).  ARAB2002 carries what
cannot be folded into weights: per block the shortcut flag and the gate, in the header the stem activation and the
policy bias.
"""
import struct

import numpy as np

BN_EPS = 1e-5
SE_CODE = {None: 0, "ca_se": 1, "se": 1, "eca_se": 2}
MX_BN_EPS = 1e-3  # mx.sym.BatchNorm's default
# squeeze-excitation gates: torch Hardsigmoid clamp(x / 6 + 0.5), MXNet hard_sigmoid clamp(0.2 x + 0.5), sigmoid
GATE_CODE = {None: 0, "torch_hard_sigmoid": 0, "hard_sigmoid": 1, "sigmoid": 2}
SHORTCUT_PRE_SE, SE_BIAS = 1, 2  # ARAB2002 block flags


def _np(t):
    if hasattr(t, "detach"):
        t = t.detach().cpu().numpy()
    return np.asarray(t, dtype=np.float64)


def _fold(sd, conv_key, bn_prefix):
    w = _np(sd[conv_key])
    g, b = _np(sd[bn_prefix + ".weight"]), _np(sd[bn_prefix + ".bias"])
    m, v = _np(sd[bn_prefix + ".running_mean"]), _np(sd[bn_prefix + ".running_var"])
    s = g / np.sqrt(v + BN_EPS)
    return w * s.reshape(-1, *([1] * (w.ndim - 1))), b - m * s


def export_blob(sd, arch, path, input_version=10):
    """arch: dict(in_channels, policy_channels, kernels[], se_types[], c_ops[], wdl) as in oracle-free product use;
    see crazyara_b200.nn.ARCH_RISEV2 / ARCH_RISEV33 helpers."""
    tensors = []

    def put(a):
        tensors.append(np.ascontiguousarray(a, dtype=np.float32).reshape(-1))

    w, b = _fold(sd, "body_spatial.0.body.0.weight", "body_spatial.0.body.1")
    put(w), put(b)
    for i, (k, se, cop) in enumerate(zip(arch["kernels"], arch["se_types"], arch["c_ops"])):
        p = f"body_spatial.{i + 1}"
        code = SE_CODE[se]
        if code == 1:
            put(_np(sd[p + ".se.fc.0.weight"])), put(_np(sd[p + ".se.fc.2.weight"]))
        elif code == 2:
            wc = _np(sd[p + ".se.body.0.weight"])
            put(wc[:, :, wc.shape[2] // 2]), put(_np(sd[p + ".se.body.0.bias"]))
        w, b = _fold(sd, p + ".body.0.weight", p + ".body.1")
        assert w.shape[0] == cop
        put(w), put(b)
        w, b = _fold(sd, p + ".body.3.weight", p + ".body.4")
        assert w.shape == (cop, 1, k, k)
        put(w), put(b)
        w, b = _fold(sd, p + ".body.6.weight", p + ".body.7")
        put(w), put(b)
    w, b = _fold(sd, "value_head.body.0.weight", "value_head.body.1")
    put(w), put(b)
    if arch["wdl"]:
        put(_np(sd["value_head.body_wdl.0.weight"])), put(_np(sd["value_head.body_wdl.0.bias"]))
        put(_np(sd["value_head.body_plys.0.weight"])), put(_np(sd["value_head.body_plys.0.bias"]))
    else:
        put(_np(sd["value_head.body_final.0.weight"])), put(_np(sd["value_head.body_final.0.bias"]))
        put(_np(sd["value_head.body_final.2.weight"])), put(_np(sd["value_head.body_final.2.bias"]))
    w, b = _fold(sd, "policy_head.body.0.weight", "policy_head.body.1")
    put(w), put(b)
    put(_np(sd["policy_head.body.3.weight"]))
    return write_blob(path, arch, tensors, input_version)


def write_blob(path, arch, tensors, input_version):
    """Header, block table and the float32 tensors (flattened, in net.cu's order).  ARAB2001 for the PyTorch semantics;
    ARAB2002 when arch["semantics"] == "mxnet" (every block's shortcut from its input before the SE, ca_se with biases)."""
    mx = arch.get("semantics") == "mxnet"
    with open(path, "wb") as f:
        f.write(b"ARAB2002" if mx else b"ARAB2001")
        f.write(struct.pack("<8i", arch["in_channels"], arch["policy_channels"], len(arch["kernels"]), 256, 8, 256,
                            1 if arch["wdl"] else 0, input_version))
        if mx:
            f.write(struct.pack("<2i", int(arch["stem_act"]), int(arch["policy_bias"])))
        for i, (k, se, cop) in enumerate(zip(arch["kernels"], arch["se_types"], arch["c_ops"])):
            if mx:
                flags = SHORTCUT_PRE_SE | (SE_BIAS if SE_CODE[se] == 1 else 0)
                f.write(struct.pack("<5i", cop, k, SE_CODE[se], flags, GATE_CODE[arch["se_gates"][i]]))
            else:
                f.write(struct.pack("<3i", cop, k, SE_CODE[se]))
        for t in tensors:
            t = np.ascontiguousarray(t, dtype=np.float32).reshape(-1)
            f.write(struct.pack("<q", t.size))
            f.write(t.tobytes())
    return path


# ---------------------------------------------------------------------------------------------- MXNet symbols
def mx_bn_prefix(params, prefix):
    """the BatchNorm behind layer `prefix`: `<prefix>` (rise_mobile_v2.py, get_stem, the heads) or `<prefix>_bn1`
    (rise_mobile_v3.py's get_norm_layer appends '_bn1' to the name it is given)"""
    return prefix if prefix + "_moving_mean" in params else prefix + "_bn1"


def mx_eca_names(params):
    """weight names of the eca_se convolutions in block order: the symbol leaves them unnamed, so MXNet names them
    convolution<n> in creation order (builder_util_symbol.py:321)"""
    idx = sorted(int(k[len("convolution"):-len("_weight")]) for k in params
                 if k.startswith("convolution") and k.endswith("_weight") and k[len("convolution"):-len("_weight")].isdigit())
    return [f"convolution{i}" for i in idx]


def _mx_fold(params, conv, bn, eps, fix_gamma):
    w = _np(params[conv + "_weight"])
    e = eps.get(bn, MX_BN_EPS) if isinstance(eps, dict) else eps
    g = np.ones(w.shape[0]) if fix_gamma else _np(params[bn + "_gamma"])
    s = g / np.sqrt(_np(params[bn + "_moving_var"]) + e)
    b = _np(params[bn + "_beta"]) - _np(params[bn + "_moving_mean"]) * s
    if conv + "_bias" in params:  # (the symbols' convolutions in front of a BatchNorm have none)
        b = b + _np(params[conv + "_bias"]) * s
    return w * s.reshape(-1, *([1] * (w.ndim - 1))), b


def eca_band(w, channels=256):
    """a one-filter 1-D convolution over the channel axis (weight [1, 1, k], zero padding k // 2) as the [out][in]
    matrix the eca_se kernels take"""
    taps = np.asarray(w, np.float64).reshape(-1)
    r = taps.size // 2
    m = np.zeros((channels, channels))
    for c in range(channels):
        for t in range(taps.size):
            if 0 <= c + t - r < channels:
                m[c, c + t - r] = taps[t]
    return m


def export_mx_blob(params, arch, path, input_version=10, eps=MX_BN_EPS, fix_gamma=True):
    """MXNet-named parameters (arg and aux params as the reference's symbol code names them) -> ARAB2002 blob.
    arch: as oracle.net_mx.arch_mx_risev2 / arch_mx_risev33 (semantics "mxnet", se_gates, stem_act, policy_bias).
    eps: BatchNorm epsilon, one value or {BatchNorm name: eps} (missing names: MXNet's default 1e-3).  fix_gamma: the
    BatchNorm gammas are fixed to 1 (mx.sym.BatchNorm's default), whatever values the parameters hold.  ca_se hidden
    widths below 128 are zero-padded to 128; the eca_se convolution becomes its banded 256 x 256 matrix."""
    assert arch.get("semantics") == "mxnet"
    tensors = []
    put = tensors.append
    fold = lambda conv, bn: _mx_fold(params, conv, mx_bn_prefix(params, bn), eps, fix_gamma)
    w, b = fold("stem_conv0", "stem_bn0")
    put(w), put(b)
    eca = iter(mx_eca_names(params))
    for i, (k, se, cop) in enumerate(zip(arch["kernels"], arch["se_types"], arch["c_ops"])):
        p = f"bc_res_block{i}"
        if SE_CODE[se] == 1:
            w1, w2 = _np(params[p + "_se_fc0_weight"]), _np(params[p + "_se_fc1_weight"])
            hid = w1.shape[0]
            if hid > 128:
                raise ValueError(f"block {i}: ca_se hidden width {hid} > 128")
            pad = lambda a, ax: np.pad(a, [(0, 128 - hid) if d == ax else (0, 0) for d in range(a.ndim)])
            put(pad(w1, 0)), put(pad(_np(params[p + "_se_fc0_bias"]), 0))
            put(pad(w2, 1)), put(_np(params[p + "_se_fc1_bias"]))
        elif SE_CODE[se] == 2:
            name = next(eca)
            put(eca_band(params[name + "_weight"])), put(np.full(256, _np(params[name + "_bias"]).reshape(-1)[0]))
        w, b = fold(p + "_conv1", p + "_bn1")
        assert w.shape[0] == cop, (i, w.shape, cop)
        put(w), put(b)
        w, b = fold(p + "_conv2", p + "_bn2")
        assert w.shape == (cop, 1, k, k), (i, w.shape)
        put(w), put(b)
        w, b = fold(p + "_conv3", p + "_bn3")
        put(w), put(b)
    w, b = fold("value_conv0", "value_bn0")
    put(w), put(b)
    for n in ("value_fc0", "value_fc1"):
        put(_np(params[n + "_weight"])), put(_np(params[n + "_bias"]))
    w, b = fold("policy_conv0", "policy_bn0")
    put(w), put(b)
    put(_np(params["policy_conv1_weight"]))
    if arch["policy_bias"]:
        put(_np(params["policy_conv1_bias"]))
    return write_blob(path, arch, tensors, input_version)


def arch_from_state_dict(sd):
    """Reads the architecture off a RiseV3 state_dict (rise_mobile_v3.py:81-183): block count, operating channels,
    depthwise kernel sizes, SE flavour per block, WDL head, input / policy channels."""
    keys = set(sd.keys())
    n_blocks = 0
    while f"body_spatial.{n_blocks + 1}.body.0.weight" in keys:
        n_blocks += 1
    if n_blocks == 0:
        raise ValueError("not a RiseV3 state_dict (no body_spatial.1.body.0.weight)")
    kernels, se_types, c_ops = [], [], []
    for i in range(1, n_blocks + 1):
        p = f"body_spatial.{i}"
        dw = sd[p + ".body.3.weight"]
        c_ops.append(int(dw.shape[0]))
        kernels.append(int(dw.shape[-1]))
        if p + ".se.fc.0.weight" in keys:
            se_types.append("ca_se")
        elif p + ".se.body.0.weight" in keys:
            se_types.append("eca_se")
        else:
            se_types.append(None)
    stem = sd["body_spatial.0.body.0.weight"]
    return dict(name=f"rise_{n_blocks}b", in_channels=int(stem.shape[1]), policy_channels=int(sd["policy_head.body.3.weight"].shape[0]),
                channels=int(stem.shape[0]), kernels=kernels, se_types=se_types, c_ops=c_ops,
                wdl="value_head.body_wdl.0.weight" in keys, value_channels=int(sd["value_head.body.0.weight"].shape[0]),
                value_fc=256)


def import_checkpoint(checkpoint_path, blob_path, input_version=None):
    """Reference trainer checkpoint (`torch.save({'model_state_dict': ...})`, trainer_agent_pytorch.py:506-516; a bare
    state_dict is accepted too) -> ARAB2001 blob.  input_version defaults from the input channel count
    (34/63 -> 1.0, 51 -> 2.0, 52/64/80 -> 3.0)."""
    import torch
    ck = torch.load(checkpoint_path, map_location="cpu", weights_only=False)
    sd = ck.get("model_state_dict", ck) if isinstance(ck, dict) else ck
    sd = {k[7:] if k.startswith("module.") else k: v for k, v in sd.items()}  # DataParallel prefix
    arch = arch_from_state_dict(sd)
    if input_version is None:
        input_version = {34: 10, 63: 10, 39: 10, 51: 20, 52: 30, 64: 30, 80: 30}.get(arch["in_channels"], 10)
    export_blob(sd, arch, blob_path, input_version=input_version)
    return arch


if __name__ == "__main__":
    import sys
    if len(sys.argv) < 3:
        raise SystemExit("usage: python -m crazyara_b200.weights <checkpoint.tar|state_dict.pt> <out.arab> [input_version]")
    a = import_checkpoint(sys.argv[1], sys.argv[2], int(sys.argv[3]) if len(sys.argv) > 3 else None)
    print(f"{sys.argv[2]}: {len(a['kernels'])} blocks, {a['in_channels']} -> {a['policy_channels']}x64, wdl={a['wdl']}")
