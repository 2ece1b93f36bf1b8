"""CPU restatement (torch fp32 functional ops) of the reference's RISE networks as its MXNet symbols define them -- TEST
INFRASTRUCTURE ONLY.

Follows QueensGambit/CrazyAra DeepCrazyhouse/src/domain/neural_net/architectures/
  rise_mobile_v2.py:31-71 (bottleneck_residual_block), :150-242 (rise_mobile_v2_symbol, get_rise_v2_symbol)
  rise_mobile_v3.py:35-64 (bottleneck_residual_block_v2), :95-213 (rise_mobile_v3_symbol, get_rise_v33_symbol)
  builder_util_symbol.py:72-88 (get_stem), :100-159 (value_head), :189-223 (policy_head), :251-286
    (channel_attention_module), :303-329 (efficient_channel_attention_module)
and appends the softmax the engine's backend adds.  Against oracle/net.py (the PyTorch definition):
  - a block's shortcut is its input BEFORE the squeeze-excitation (broadcast_add(bn3, data));
  - ca_se: FullyConnected layers with biases, hidden width channels // ratio (v2: ratio 2, sigmoid; v3: ratio 16,
    hard_sigmoid = clamp(0.2 x + 0.5));
  - eca_se: one-filter 1-D convolution over the channel axis (kernel 5 for 256 channels) with one bias;
  - the v3 stem has no activation, the v3 policy convolution has a bias;
  - BatchNorm: eps 1e-3 and fix_gamma=True (gamma taken as 1), MXNet's defaults.

Parameters use the names the symbol code gives them (auto-named eca_se convolutions: convolution<n>).  Parity pin:
tests/test_oracle_net_mx.py against tests/golden/mx_net_*.json, which tests/golden/gen_mx_net_golden.py writes by
evaluating the reference's own symbol code over a NumPy stand-in for mxnet.sym.
"""
import numpy as np
import torch
import torch.nn.functional as F

from oracle import net as onet

BN_EPS = 1e-3


def arch_mx_risev2(in_channels=34, policy_channels=81):
    """get_rise_v2_symbol (rise_mobile_v2.py:227-242): 13 blocks, k = 3, c_op = 128 + 64 i, ca_se (ratio 2, sigmoid) on
    the last five"""
    a = onet.arch_risev2(in_channels, policy_channels)
    a.update(name="mx_risev2", semantics="mxnet", bn_names="v2", stem_act=True, policy_bias=False,
             se_gates=["sigmoid" if s else None for s in a["se_types"]], se_hidden=[128 if s else None for s in a["se_types"]])
    return a


def arch_mx_risev33(in_channels=52, policy_channels=76):
    """get_rise_v33_symbol (rise_mobile_v3.py:189-213): the kernels and eca_se blocks of RISEv3.3, hard_sigmoid gates,
    the plain value head (use_wdl is not passed)"""
    a = onet.arch_risev33(in_channels, policy_channels, wdl=False)
    a.update(name="mx_risev33", semantics="mxnet", bn_names="v3", stem_act=False, policy_bias=True,
             se_gates=["hard_sigmoid" if s else None for s in a["se_types"]], se_hidden=[None] * len(a["se_types"]))
    return a


def _bn_name(arch, prefix, in_block):
    return prefix + "_bn1" if in_block and arch["bn_names"] == "v3" else prefix


def make_mx_params(arch, seed=0):
    """Seeded random parameters under the symbol code's names (arg params and the BatchNorm aux states).  The
    BatchNorm gammas are random too: with fix_gamma the network must ignore them."""
    rng = np.random.default_rng(seed)
    p = {}

    def conv(name, cout, cin, k, groups=1, scale=1.0):
        fan_in = (cin // groups) * k * k
        p[name + "_weight"] = (rng.standard_normal((cout, cin // groups, k, k)) * scale * np.sqrt(2.0 / fan_in)).astype(np.float32)

    def bn(name, c):
        p[name + "_gamma"] = rng.uniform(0.5, 1.5, c).astype(np.float32)
        p[name + "_beta"] = (rng.standard_normal(c) * 0.1).astype(np.float32)
        p[name + "_moving_mean"] = (rng.standard_normal(c) * 0.1).astype(np.float32)
        p[name + "_moving_var"] = rng.uniform(0.5, 1.5, c).astype(np.float32)

    def fc(name, cout, cin, scale=1.0):
        p[name + "_weight"] = (rng.standard_normal((cout, cin)) * scale / np.sqrt(cin)).astype(np.float32)
        p[name + "_bias"] = (rng.standard_normal(cout) * 0.3).astype(np.float32)

    C = arch["channels"]
    conv("stem_conv0", C, arch["in_channels"], 3)
    bn("stem_bn0", C)
    n_eca = 0
    for i, (k, se, cop) in enumerate(zip(arch["kernels"], arch["se_types"], arch["c_ops"])):
        b = f"bc_res_block{i}"
        if se == "ca_se":
            fc(b + "_se_fc0", arch["se_hidden"][i], C, scale=2.0)
            fc(b + "_se_fc1", C, arch["se_hidden"][i], scale=2.0)
        elif se == "eca_se":
            p[f"convolution{n_eca}_weight"] = (rng.standard_normal((1, 1, 5)) * 1.5).astype(np.float32)
            p[f"convolution{n_eca}_bias"] = (rng.standard_normal(1) * 0.5).astype(np.float32)
            n_eca += 1
        conv(b + "_conv1", cop, C, 1)
        bn(_bn_name(arch, b + "_bn1", True), cop)
        conv(b + "_conv2", cop, cop, k, groups=cop)
        bn(_bn_name(arch, b + "_bn2", True), cop)
        conv(b + "_conv3", C, cop, 1, scale=0.1)  # residual branch scaled down: the tower stays O(1)
        bn(_bn_name(arch, b + "_bn3", True), C)
    conv("value_conv0", arch["value_channels"], C, 1)
    bn("value_bn0", arch["value_channels"])
    fc("value_fc0", arch["value_fc"], arch["value_channels"] * 64, scale=0.5)
    fc("value_fc1", 1, arch["value_fc"], scale=0.5)
    conv("policy_conv0", C, C, 3)
    bn("policy_bn0", C)
    conv("policy_conv1", arch["policy_channels"], C, 3)
    if arch["policy_bias"]:
        p["policy_conv1_bias"] = (rng.standard_normal(arch["policy_channels"]) * 0.3).astype(np.float32)
    return p


def _gate(x, gate):
    if gate == "sigmoid":
        return torch.sigmoid(x)
    if gate == "hard_sigmoid":  # mx.sym.hard_sigmoid, alpha 0.2, beta 0.5
        return torch.clamp(0.2 * x + 0.5, 0.0, 1.0)
    return F.hardsigmoid(x)


def forward_mx(params, arch, x, eps=BN_EPS):
    """x: [B, C, 8, 8] fp32 -> dict(value [B], policy_logits [B, P*64], prob [B, P*64], aux None, trunk)."""
    p = {k: torch.as_tensor(v, dtype=torch.float32) for k, v in params.items()}
    x = torch.as_tensor(x, dtype=torch.float32)

    def bn(t, name):  # fix_gamma: gamma = 1
        return F.batch_norm(t, p[name + "_moving_mean"], p[name + "_moving_var"], None, p[name + "_beta"], training=False, eps=eps)

    def conv(t, name, pad=0, groups=1):
        return F.conv2d(t, p[name + "_weight"], p.get(name + "_bias"), padding=pad, groups=groups)

    n_eca = 0
    with torch.no_grad():
        out = bn(conv(x, "stem_conv0", 1), "stem_bn0")
        if arch["stem_act"]:
            out = F.relu(out)
        for i, (k, se) in enumerate(zip(arch["kernels"], arch["se_types"])):
            b = f"bc_res_block{i}"
            data = out
            if se == "ca_se":
                y = data.mean(dim=(2, 3))
                y = F.relu(F.linear(y, p[b + "_se_fc0_weight"], p[b + "_se_fc0_bias"]))
                y = _gate(F.linear(y, p[b + "_se_fc1_weight"], p[b + "_se_fc1_bias"]), arch["se_gates"][i])
                data = data * y[:, :, None, None]
            elif se == "eca_se":
                c = f"convolution{n_eca}"
                n_eca += 1
                y = data.mean(dim=(2, 3))[:, None, :]  # reshape (-1, 1, channels)
                y = F.conv1d(y, p[c + "_weight"], p[c + "_bias"], padding=p[c + "_weight"].shape[-1] // 2)
                data = data * _gate(y, arch["se_gates"][i])[:, 0, :, None, None]
            h = F.relu(bn(conv(data, b + "_conv1"), _bn_name(arch, b + "_bn1", True)))
            h = F.relu(bn(conv(h, b + "_conv2", k // 2, h.shape[1]), _bn_name(arch, b + "_bn2", True)))
            h = bn(conv(h, b + "_conv3"), _bn_name(arch, b + "_bn3", True))
            out = h + out  # broadcast_add(bn3, data): the input before the squeeze-excitation
        v = F.relu(bn(conv(out, "value_conv0"), "value_bn0")).reshape(x.shape[0], -1)
        v = F.relu(F.linear(v, p["value_fc0_weight"], p["value_fc0_bias"]))
        value = torch.tanh(F.linear(v, p["value_fc1_weight"], p["value_fc1_bias"]))[:, 0]
        ph = F.relu(bn(conv(out, "policy_conv0", 1), "policy_bn0"))
        logits = conv(ph, "policy_conv1", 1).reshape(x.shape[0], -1)
        prob = torch.softmax(logits, dim=1)
    return dict(value=value.numpy(), policy_logits=logits.numpy(), prob=prob.numpy(), aux=None, trunk=out.numpy())
