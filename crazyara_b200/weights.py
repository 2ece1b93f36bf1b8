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

AlphaVile (alpha_vile.py: RiseV3 with a 192 / 224 channel trunk and NextViT transformer blocks, NTB) is written as
ARAB2003: the header of ARAB2002 with any trunk width from 64 to 256, and a type word in front of every block record
(0: a bottleneck block as in ARAB2001, 1: an NTB with its widths M, Ca, H).  The NTB's pre-norms norm1 and norm2 are
folded into q / k / v and mlp.conv1 the way the reference's merge_pre_bn does before its ONNX export.

A network with a fully-connected policy head (the trainer's select_policy_from_plane=False: policy_head.body2 BatchNorm
+ ReLU and policy_head.body3 Linear onto the classic labels; in the MXNet symbols policy_bn1, the activation and
FullyConnected policy_out) is written as ARAB2004 around one of the three (write_blob).

The base header's WDL word is the value head's kind (VALUE_HEADS, arch["value_head"]): 0 the standard head, 1 WDL and
plies-to-end outputs with value = P(win) - P(loss), 2 the same outputs feeding the trainer's value MLP (use_mlp_wdl_ply:
the WDL logits and the plies, 4 -> 8 -> 1, tanh), 3 and 4 the MXNet symbols' head with use_wdl and use_plys_to_end
(builder_util_symbol.py value_head): a hidden layer value_fc0 of value_fc units in front of the WDL and plies outputs,
then win - loss, or the MLP on the WDL probabilities.
"""
import struct

import numpy as np

BN_EPS = 1e-5
SE_CODE = {None: 0, "ca_se": 1, "se": 1, "eca_se": 2}
MX_BN_EPS = 1e-3  # mx.sym.BatchNorm's default
# squeeze-excitation gates: torch Hardsigmoid clamp(x / 6 + 0.5), MXNet hard_sigmoid clamp(0.2 x + 0.5), sigmoid
GATE_CODE = {None: 0, "torch_hard_sigmoid": 0, "hard_sigmoid": 1, "sigmoid": 2}
SHORTCUT_PRE_SE, SE_BIAS = 1, 2  # ARAB2002 block flags
# the base header's WDL word: the value head's kind, by arch["value_head"] (absent: 0 or 1 by arch["wdl"])
VALUE_HEADS = {"wdl_mlp": 2, "mx_wdl": 3, "mx_wdl_mlp": 4}
VALUE_MLP = 8  # the hidden width of the trainers' value MLP (builder_util.py _ValueHead, builder_util_symbol.py value_head)


def value_kind(arch):
    """the value head's kind as the blob header holds it"""
    return VALUE_HEADS[arch["value_head"]] if arch.get("value_head") else int(bool(arch["wdl"]))


def check_value_head(kind, fc, n_policy, sizes):
    """Checks a value head of kind `kind` with header word value_fc = fc against the element counts `sizes` of a blob's
    tensors in order; the value head's tensors sit in front of the policy head's n_policy.  Raises ValueError naming what
    is malformed: an unknown kind, a hidden layer outside 1 .. 256 units, an MLP whose width is not 8, other sizes."""
    if kind not in (0, 1, *VALUE_HEADS.values()):
        raise ValueError(f"value head of unknown kind {kind}")
    if kind < 2:
        return
    if kind in (3, 4) and not 1 <= fc <= 256:
        raise ValueError(f"value head: hidden layer of {fc} units (1 .. 256)")
    hidden = 512 if kind == 2 else fc
    head = ([fc * 512, fc] if kind in (3, 4) else []) + [3 * hidden, 3, hidden, 1]
    if kind in (2, 4):
        head += [4 * VALUE_MLP, VALUE_MLP, VALUE_MLP, 1]
    got = list(sizes[max(len(sizes) - n_policy - len(head), 0):len(sizes) - n_policy])
    if kind in (2, 4) and len(got) == len(head) and got[-4] != 4 * VALUE_MLP:
        raise ValueError(f"value head: MLP of width {got[-4] / 4:g} (the trainers' MLP has {VALUE_MLP})")
    if got != head:
        raise ValueError(f"value head of kind {kind}: tensor sizes {got}, expected {head}")


def _np(t):
    if hasattr(t, "detach"):
        t = t.detach().cpu().numpy()
    return np.asarray(t, dtype=np.float64)


def _bn_affine(gamma, beta, mean, var, eps):  # an eval-mode BatchNorm as (scale, shift): bn(x) = scale x + shift
    s = gamma / np.sqrt(var + eps)
    return s, beta - mean * s


def _pre_bn(sd, prefix):  # the state_dict's BatchNorm `prefix` as (scale, shift)
    return _bn_affine(*(_np(sd[prefix + k]) for k in (".weight", ".bias", ".running_mean", ".running_var")), BN_EPS)


def _fold(sd, conv_key, bn_prefix):
    w, (s, b) = _np(sd[conv_key]), _pre_bn(sd, bn_prefix)
    return w * s.reshape(-1, *([1] * (w.ndim - 1))), b


def input_version_of(arch, input_version=None):
    """input_version, or by default the one the input channel count implies (34/39/63 -> 1.0, 51 -> 2.0, 52/64/80 -> 3.0)"""
    if input_version is not None:
        return input_version
    return {34: 10, 63: 10, 39: 10, 51: 20, 52: 30, 64: 30, 80: 30}.get(arch["in_channels"], 10)


def export_blob(sd, arch, path, input_version=10):
    """arch: dict(in_channels, policy_channels, kernels[], se_types[], c_ops[], wdl) as in oracle-free product use;
    see crazyara_b200.nn.ARCH_RISEV2 / ARCH_RISEV33 helpers."""
    tensors = []
    put = tensors.append  # (write_blob writes each as float32)
    w, b = _fold(sd, "body_spatial.0.body.0.weight", "body_spatial.0.body.1")
    put(w), put(b)
    ntb = arch.get("ntb") or [False] * len(arch["kernels"])
    for i, (k, se, cop) in enumerate(zip(arch["kernels"], arch["se_types"], arch["c_ops"])):
        p = f"body_spatial.{i + 1}"
        if ntb[i]:
            for t in ntb_tensors(sd, p):
                put(t)
            continue
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
        if arch.get("value_head") == "wdl_mlp":  # use_mlp_wdl_ply: body_final is the MLP on cat(wdl logits, plies)
            for n in ("value_head.body_final.0", "value_head.body_final.2"):
                put(_np(sd[n + ".weight"])), put(_np(sd[n + ".bias"]))
    else:
        put(_np(sd["value_head.body_final.0.weight"])), put(_np(sd["value_head.body_final.0.bias"]))
        put(_np(sd["value_head.body_final.2.weight"])), put(_np(sd["value_head.body_final.2.bias"]))
    w, b = _fold(sd, "policy_head.body.0.weight", "policy_head.body.1")
    put(w), put(b)
    if arch.get("n_labels"):  # select_policy_from_plane=False: BatchNorm + ReLU behind the last convolution, then the Linear
        w, b = _fold(sd, "policy_head.body.3.weight", "policy_head.body2.0")
        put(w), put(b)
        put(_np(sd["policy_head.body3.0.weight"])), put(_np(sd["policy_head.body3.0.bias"]))
    else:
        put(_np(sd["policy_head.body.3.weight"]))
    return write_blob(path, arch, tensors, input_version)


def ntb_tensors(sd, p):
    """The blob tensors of the NTB `p` (next_vit_official_modules.py:265-335), BatchNorms folded: patch_embed [M][C] + [M],
    q / k / v stacked [3M][M] + [3M] (norm1 folded in), proj [M][M] + [M], projection [Ca][M] + [Ca], the group conv
    [Ca][32][3][3] + [Ca] (mhca.norm folded in), mhca.projection [Ca][Ca], mlp.conv1 [H][C] + [H] (norm2 folded in),
    mlp.conv2 [C][H] + [C].  The attention scale 32^-0.5 is not folded: the blob holds the network as trained."""
    mat = lambda a: a.reshape(a.shape[0], -1)
    w, b = _fold(sd, p + ".patch_embed.conv.weight", p + ".patch_embed.norm")
    out = [mat(w), b]
    s1, c1 = _pre_bn(sd, p + ".norm1")
    qkv_w, qkv_b = [], []
    for n in ("q", "k", "v"):
        wn, bn = _np(sd[f"{p}.e_mhsa.{n}.weight"]), _np(sd[f"{p}.e_mhsa.{n}.bias"])
        qkv_w.append(wn * s1[None, :]), qkv_b.append(wn @ c1 + bn)
    out += [np.concatenate(qkv_w), np.concatenate(qkv_b)]
    out += [_np(sd[p + ".e_mhsa.proj.weight"]), _np(sd[p + ".e_mhsa.proj.bias"])]
    w, b = _fold(sd, p + ".projection.conv.weight", p + ".projection.norm")
    out += [mat(w), b]
    out += list(_fold(sd, p + ".mhca.group_conv3x3.weight", p + ".mhca.norm"))
    out.append(mat(_np(sd[p + ".mhca.projection.weight"])))
    s2, c2 = _pre_bn(sd, p + ".norm2")
    w1 = mat(_np(sd[p + ".mlp.conv1.weight"]))
    out += [w1 * s2[None, :], w1 @ c2 + _np(sd[p + ".mlp.conv1.bias"])]
    out += [mat(_np(sd[p + ".mlp.conv2.weight"])), _np(sd[p + ".mlp.conv2.bias"])]
    return out


CLASSIC_LABELS = (1968, 2272, 2316)  # NB_LABELS of chess, crazyhouse and the lichess variants (crazyara_b200.labels)


def write_blob(path, arch, tensors, input_version):
    """Header, block table and the float32 tensors (flattened, in net.cu's order).  ARAB2001 for the PyTorch semantics;
    ARAB2002 when arch["semantics"] == "mxnet" (every block's shortcut from its input before the SE, ca_se with biases);
    ARAB2003 for a trunk narrower than 256 channels or with NTB blocks (arch["ntb"], widths mhsa / mhca / mlp).

    A network with a fully-connected policy head (arch["n_labels"] = L, the trainer's select_policy_from_plane=False) is
    ARAB2004: the magic, the base format's number (1, 2 or 3) and L, then the base blob from its header on.  Its last
    policy convolution has the BatchNorm of the head folded in, so the tensors end with that convolution's weight and
    bias [P], W_fc [L][P * 64] (the trainer's NCHW flatten) and b_fc [L]; the base header's policy_bias stays 0."""
    mx = arch.get("semantics") == "mxnet"
    ntb = arch.get("ntb") or [False] * len(arch["kernels"])
    C = arch.get("channels", 256)
    v3 = any(ntb) or C != 256
    if mx and v3:
        raise ValueError("ARAB2003 has no blocks with the MXNet semantics")
    n_labels = arch.get("n_labels")
    if n_labels and arch.get("policy_bias"):
        raise ValueError("ARAB2004 carries the policy convolution's bias with its head (policy_bias must be False)")
    kind = value_kind(arch)
    fc = arch.get("value_fc", 256) if v3 or kind in (3, 4) else 256
    check_value_head(kind, fc, 6 if n_labels else 3 + bool(arch.get("policy_bias")), [np.size(t) for t in tensors])
    with open(path, "wb") as f:
        if n_labels:
            f.write(b"ARAB2004" + struct.pack("<2i", 3 if v3 else 2 if mx else 1, n_labels))
        else:
            f.write(b"ARAB2003" if v3 else b"ARAB2002" if mx else b"ARAB2001")
        f.write(struct.pack("<8i", arch["in_channels"], arch["policy_channels"], len(arch["kernels"]), C, 8,
                            fc, kind, input_version))
        if mx or v3:
            f.write(struct.pack("<2i", int(arch.get("stem_act", True)), int(arch.get("policy_bias", False))))
        for i, (k, se, cop) in enumerate(zip(arch["kernels"], arch["se_types"], arch["c_ops"])):
            if v3:
                f.write(struct.pack("<4i", 1, arch["mhsa"], arch["mhca"], arch["mlp"]) if ntb[i] else
                        struct.pack("<4i", 0, cop, k, SE_CODE[se]))
            elif mx:
                flags = SHORTCUT_PRE_SE | (SE_BIAS if SE_CODE[se] == 1 else 0)
                f.write(struct.pack("<5i", cop, k, SE_CODE[se], flags, GATE_CODE[arch["se_gates"][i]]))
            else:
                f.write(struct.pack("<3i", cop, k, SE_CODE[se]))
        for t in tensors:
            t = np.ascontiguousarray(t, dtype=np.float32).reshape(-1)
            f.write(struct.pack("<q", t.size))
            f.write(t.tobytes())
    return path


def read_blob(path):
    """The inverse of write_blob: an ARAB2001 / 2002 / 2003 / 2004 blob -> (arch, tensors [flat float32], input_version).  arch
    holds what the header and block table say, under write_blob's keys; write_blob(path2, *read_blob(path)) rewrites the
    file byte for byte.  A blob write_blob cannot have written (ARAB2002 block flags other than the ones it sets, an unknown
    block type, a tensor past the end of the file, a malformed value head: check_value_head) is refused."""
    buf = open(path, "rb").read()
    magic = buf[:8]
    if magic not in (b"ARAB2001", b"ARAB2002", b"ARAB2003", b"ARAB2004"):
        raise ValueError(f"{path}: not an ARAB2001 / 2002 / 2003 / 2004 blob")
    off, n_labels = 8, 0
    if magic == b"ARAB2004":
        base, n_labels = struct.unpack_from("<2i", buf, 8)
        if base not in (1, 2, 3):
            raise ValueError(f"{path}: ARAB2004 wraps base format {base}")
        if n_labels not in CLASSIC_LABELS:
            raise ValueError(f"{path}: {n_labels} policy labels (the classic label lists have {CLASSIC_LABELS})")
        magic, off = b"ARAB200%d" % base, 16
    mx, v3 = magic == b"ARAB2002", magic == b"ARAB2003"
    cin, pch, n, C, vc, fc, kind, version = struct.unpack_from("<8i", buf, off)
    arch = dict(in_channels=cin, policy_channels=pch, channels=C, value_channels=vc, value_fc=fc, wdl=bool(kind),
                kernels=[], se_types=[], c_ops=[])
    if kind >= 2:
        arch["value_head"] = {v: k for k, v in VALUE_HEADS.items()}.get(kind, kind)
    if n_labels:
        arch["n_labels"] = n_labels
    off += 32
    if mx or v3:
        stem_act, policy_bias = struct.unpack_from("<2i", buf, off)
        arch.update(stem_act=bool(stem_act), policy_bias=bool(policy_bias))
        off += 8
        if n_labels and policy_bias:
            raise ValueError(f"{path}: ARAB2004 carries the policy convolution's bias with its head, not in the base header")
    if mx:
        arch.update(semantics="mxnet", se_gates=[])
    if v3:
        arch.update(ntb=[], mhsa=0, mhca=0, mlp=0)
    width = 4 if v3 else 5 if mx else 3
    for i in range(n):
        rec = struct.unpack_from(f"<{width}i", buf, off)
        off += 4 * width
        if v3:
            if rec[0] not in (0, 1):
                raise ValueError(f"{path}: block {i} has type {rec[0]}")
            arch["ntb"].append(rec[0] == 1)
            if rec[0] == 1:
                arch.update(mhsa=rec[1], mhca=rec[2], mlp=rec[3])
            rec = (0, 3, 0) if rec[0] == 1 else rec[1:]
        cop, k, se = rec[:3]
        if mx:
            if rec[3] != SHORTCUT_PRE_SE | (SE_BIAS if se == 1 else 0):
                raise ValueError(f"{path}: block {i} has flags {rec[3]}")
            arch["se_gates"].append({0: None, 1: "hard_sigmoid", 2: "sigmoid"}[rec[4]])
        arch["c_ops"].append(cop), arch["kernels"].append(k), arch["se_types"].append({0: None, 1: "ca_se", 2: "eca_se"}[se])
    tensors = []
    while off < len(buf):
        size, = struct.unpack_from("<q", buf, off)
        tensors.append(np.frombuffer(buf, "<f4", size, off + 8).copy())
        off += 8 + 4 * size
    try:
        check_value_head(kind, fc, 6 if n_labels else 3 + arch.get("policy_bias", False), [t.size for t in tensors])
    except ValueError as e:
        raise ValueError(f"{path}: {e}") from None
    return arch, tensors, version


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
    s, b = _bn_affine(g, _np(params[bn + "_beta"]), _np(params[bn + "_moving_mean"]), _np(params[bn + "_moving_var"]), e)
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


# the FullyConnected layers of the symbols' value heads in blob order (builder_util_symbol.py value_head; the WDL layer
# is named main_config["wdl_output"])
MX_VALUE_LAYERS = {None: ("value_fc0", "value_fc1"),
                   "mx_wdl": ("value_fc0", "wdl_out", "value_plys_to_end_fc"),
                   "mx_wdl_mlp": ("value_fc0", "wdl_out", "value_plys_to_end_fc", "value_wdl_ply_fc", "value_fc1")}


def export_mx_blob(params, arch, path, input_version=10, eps=MX_BN_EPS, fix_gamma=True):
    """MXNet-named parameters (arg and aux params as the reference's symbol code names them) -> ARAB2002 blob.
    arch: as oracle.net_mx.arch_mx_risev2 / arch_mx_risev33 (semantics "mxnet", se_gates, stem_act, policy_bias).
    eps: BatchNorm epsilon, one value or {BatchNorm name: eps} (missing names: MXNet's default 1e-3).  fix_gamma: the
    BatchNorm gammas are fixed to 1 (mx.sym.BatchNorm's default), whatever values the parameters hold.  ca_se hidden
    widths below 128 are zero-padded to 128; the eca_se convolution becomes its banded 256 x 256 matrix.
    arch["n_labels"] set (select_policy_from_plane=False, builder_util_symbol.py policy_head): policy_conv1 is folded with
    policy_bn1, its bias included, and FullyConnected policy_out follows; the blob is ARAB2004 around ARAB2002, and
    arch["policy_bias"] has to be False (the bias goes with the head).  arch["value_head"] "mx_wdl" / "mx_wdl_mlp"
    (use_wdl and use_plys_to_end, without or with use_mlp_wdl_ply): the layers MX_VALUE_LAYERS names, value_fc0 of
    arch["value_fc"] units."""
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
    for n in MX_VALUE_LAYERS[arch.get("value_head")]:
        put(_np(params[n + "_weight"])), put(_np(params[n + "_bias"]))
    w, b = fold("policy_conv0", "policy_bn0")
    put(w), put(b)
    if arch.get("n_labels"):  # select_policy_from_plane=False: policy_bn1 and the activation, Flatten, policy_out
        w, b = fold("policy_conv1", "policy_bn1")  # (with the convolution's bias, which the v3 symbol has)
        put(w), put(b)
        put(_np(params["policy_out_weight"])), put(_np(params["policy_out_bias"]))
    else:
        put(_np(params["policy_conv1_weight"]))
        if arch["policy_bias"]:
            put(_np(params["policy_conv1_bias"]))
    return write_blob(path, arch, tensors, input_version)


def arch_from_state_dict(sd):
    """Reads the architecture off a RiseV3 state_dict (rise_mobile_v3.py:81-183): block count, operating channels,
    depthwise kernel sizes, SE flavour per block, WDL head, input / policy channels; for AlphaVile (alpha_vile.py) also
    the trunk width, the NTB positions and widths and the value head's hidden width.  A WDL head whose body_final takes
    4 inputs is the value MLP of use_mlp_wdl_ply (arch["value_head"] = "wdl_mlp")."""
    keys = set(sd.keys())
    is_ntb = lambda i: f"body_spatial.{i}.patch_embed.conv.weight" in keys
    n_blocks = 0
    while f"body_spatial.{n_blocks + 1}.body.0.weight" in keys or is_ntb(n_blocks + 1):
        n_blocks += 1
    if n_blocks == 0:
        raise ValueError("not a RiseV3 state_dict (no body_spatial.1.body.0.weight)")
    kernels, se_types, c_ops, ntb, widths = [], [], [], [], set()
    for i in range(1, n_blocks + 1):
        p = f"body_spatial.{i}"
        ntb.append(is_ntb(i))
        if ntb[-1]:
            widths.add((int(sd[p + ".patch_embed.conv.weight"].shape[0]), int(sd[p + ".projection.conv.weight"].shape[0]),
                        int(sd[p + ".mlp.conv1.weight"].shape[0])))
            kernels.append(3), se_types.append(None), c_ops.append(0)
            continue
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
    C = int(stem.shape[0])
    arch = dict(name=f"rise_{n_blocks}b", in_channels=int(stem.shape[1]), policy_channels=int(sd["policy_head.body.3.weight"].shape[0]),
                channels=C, kernels=kernels, se_types=se_types, c_ops=c_ops,
                wdl="value_head.body_wdl.0.weight" in keys, value_channels=int(sd["value_head.body.0.weight"].shape[0]),
                value_fc=256)
    if "policy_head.body3.0.weight" in keys:  # select_policy_from_plane=False (builder_util.py _PolicyHead body2 / body3)
        arch["n_labels"] = int(sd["policy_head.body3.0.weight"].shape[0])
    fc = sd.get("value_head.body_final.0.weight")
    if arch["wdl"] and fc is not None and tuple(fc.shape)[1:] == (4,):
        # use_mlp_wdl_ply: body_final is the MLP on cat(WDL logits, plies) (builder_util.py:292-296), not a layer of fc0 units
        arch["value_head"] = "wdl_mlp"
        fc = None
    if any(ntb) or C != 256:
        if len(widths) > 1:
            raise ValueError(f"NTB blocks of different widths {sorted(widths)}")
        (M, Ca, H), = widths or {(0, 0, 0)}
        arch.update(name=f"alphavile_{n_blocks}b", ntb=ntb, mhsa=M, mhca=Ca, mlp=H,
                    value_fc=C if fc is None else int(fc.shape[0]))
    return arch


def import_checkpoint(checkpoint_path, blob_path, input_version=None):
    """Reference trainer checkpoint (`torch.save({'model_state_dict': ...})`, trainer_agent_pytorch.py:506-516; a bare
    state_dict is accepted too) -> ARAB2001 blob (ARAB2003 for AlphaVile).  input_version defaults from the input channel count
    (34/63 -> 1.0, 51 -> 2.0, 52/64/80 -> 3.0)."""
    import torch
    ck = torch.load(checkpoint_path, map_location="cpu", weights_only=False)
    sd = ck.get("model_state_dict", ck) if isinstance(ck, dict) else ck
    sd = {k[7:] if k.startswith("module.") else k: v for k, v in sd.items()}  # DataParallel prefix
    arch = arch_from_state_dict(sd)
    export_blob(sd, arch, blob_path, input_version=input_version_of(arch, input_version))
    return arch


if __name__ == "__main__":
    import sys
    if len(sys.argv) < 3:
        raise SystemExit("usage: python -m crazyara_b200.weights <checkpoint.tar|state_dict.pt> <out.arab> [input_version]")
    a = import_checkpoint(sys.argv[1], sys.argv[2], int(sys.argv[3]) if len(sys.argv) > 3 else None)
    print(f"{sys.argv[2]}: {len(a['kernels'])} blocks, {a['in_channels']} -> {a['policy_channels']}x64, wdl={a['wdl']}")
