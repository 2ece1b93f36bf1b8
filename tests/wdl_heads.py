"""The value heads with WDL and plies-to-end outputs that feed a value (the trainers' use_mlp_wdl_ply, and the MXNet
symbols' head with use_wdl and use_plys_to_end) on top of the fp32 oracle networks -- TEST INFRASTRUCTURE ONLY.

PyTorch, builder_util.py _ValueHead (:286-325) with use_mlp_wdl_ply: body_final = Linear(4, 8), activation, Linear(8, 1),
tanh on cat(WDL logits, sigmoid plies); the outputs aux = (WDL logits, plies) are the oracle's own (oracle/net.py,
oracle/net_alphavile.py), so only the value is computed here.

MXNet, builder_util_symbol.py value_head (:149-186): value_fc0 and the activation on the flattened value features, then
FullyConnected wdl_out into SoftmaxOutput (whose forward is the softmax) and value_plys_to_end_fc into a sigmoid; the value
is win - loss of the probabilities, or with use_mlp_wdl_ply value_wdl_ply_fc (8), activation, value_fc1, tanh on
Concat(probabilities, plies).  aux = (probabilities, plies), as the symbol outputs them.  The trunk and the policy come
from oracle/net_mx.py, which pins them to the reference's symbols.
"""
import numpy as np
import torch
import torch.nn.functional as F

from oracle import net as onet
from oracle import net_alphavile as oav
from oracle import net_mx

MLP = 8


def _oracle(arch):
    return oav if "ntb" in arch else onet


def _linear(g, out, cin, f32=np.float32):
    return ((g.standard_normal((out, cin)) * 1.5 / np.sqrt(cin)).astype(f32), (g.standard_normal(out) * 0.3).astype(f32))


def mlp_state_dict(arch, seed=0):
    """the state_dict of arch (a WDL arch of oracle/net.py or oracle/net_alphavile.py, value_head "wdl_mlp") with body_final
    as the value MLP, from a generator of its own so that the other parameters stay as the oracle makes them"""
    sd = _oracle(arch).make_state_dict(arch, seed)
    g = np.random.default_rng([seed, 4, 8])
    for name, (out, cin) in (("value_head.body_final.0", (MLP, 4)), ("value_head.body_final.2", (1, MLP))):
        sd[name + ".weight"], sd[name + ".bias"] = _linear(g, out, cin)
    return sd


def _mlp(t, w0, b0, w1, b1):
    return torch.tanh(F.linear(F.relu(F.linear(t, w0, b0)), w1, b1))[:, 0]


def forward_torch(sd_np, arch, x):
    """-> the oracle's outputs with the MLP's value"""
    out = _oracle(arch).forward(sd_np, arch, x)
    sd = {k: torch.as_tensor(v, dtype=torch.float32) for k, v in sd_np.items()}
    with torch.no_grad():
        v = _mlp(torch.as_tensor(out["aux"]), sd["value_head.body_final.0.weight"], sd["value_head.body_final.0.bias"],
                 sd["value_head.body_final.2.weight"], sd["value_head.body_final.2.bias"])
    out["value"] = v.numpy()
    return out


def mx_arch(base, value_head, value_fc=256):
    """an arch of oracle/net_mx.py with the WDL head value_head ("mx_wdl" or "mx_wdl_mlp") behind value_fc hidden units"""
    return dict(base, name=f"{base['name']}_{value_head}_{value_fc}", wdl=True, value_head=value_head, value_fc=value_fc)


def mx_params(arch, seed=0):
    """oracle/net_mx.make_mx_params of arch, with the value head's layers behind value_fc0 (value_fc1 the MLP's last
    layer, or none) from a generator of their own"""
    p = net_mx.make_mx_params(arch, seed)
    del p["value_fc1_weight"], p["value_fc1_bias"]
    g = np.random.default_rng([seed, 4, 8, 2])
    fc = arch["value_fc"]
    layers = [("wdl_out", 3, fc), ("value_plys_to_end_fc", 1, fc)]
    if arch["value_head"] == "mx_wdl_mlp":
        layers += [("value_wdl_ply_fc", MLP, 4), ("value_fc1", 1, MLP)]
    for name, out, cin in layers:
        p[name + "_weight"], p[name + "_bias"] = _linear(g, out, cin)
    return p


def forward_mx(params, arch, x, eps=net_mx.BN_EPS, base=net_mx.forward_mx):
    """-> the trunk and policy of base (oracle/net_mx.forward_mx, or tests/classic_mx_head.forward with a fully-connected
    policy head) with this head's value and aux"""
    fc = arch["value_fc"]
    plain = dict(params, value_fc1_weight=np.zeros((1, fc), np.float32), value_fc1_bias=np.zeros(1, np.float32))
    out = base(plain, arch, x, eps)
    p = {k: torch.as_tensor(v, dtype=torch.float32) for k, v in params.items()}
    lin = lambda t, n: F.linear(t, p[n + "_weight"], p[n + "_bias"])
    with torch.no_grad():
        t = torch.as_tensor(out["trunk"])
        v = F.conv2d(t, p["value_conv0_weight"])
        v = F.batch_norm(v, p["value_bn0_moving_mean"], p["value_bn0_moving_var"], None, p["value_bn0_beta"], training=False,
                         eps=eps)
        h = F.relu(lin(F.relu(v).reshape(t.shape[0], -1), "value_fc0"))
        prob = torch.softmax(lin(h, "wdl_out"), dim=1)
        plys = torch.sigmoid(lin(h, "value_plys_to_end_fc"))
        aux = torch.cat((prob, plys), dim=1)
        if arch["value_head"] == "mx_wdl_mlp":
            value = _mlp(aux, p["value_wdl_ply_fc_weight"], p["value_wdl_ply_fc_bias"], p["value_fc1_weight"],
                         p["value_fc1_bias"])
        else:
            value = -prob[:, 0] + prob[:, 2]
    out.update(value=value.numpy(), aux=aux.numpy())
    return out
