"""The fully-connected policy head of the reference's MXNet symbols (select_policy_from_plane=False) on top of the fp32
oracle of those symbols (oracle/net_mx.py) -- TEST INFRASTRUCTURE ONLY.

Follows builder_util_symbol.py policy_head (:189-223): policy_conv0 + policy_bn0 + activation, policy_conv1 (a bias in
the v3 symbol, none in v2), then BatchNorm policy_bn1 with MXNet's defaults (eps 1e-3, gamma fixed to 1), the activation
policy_act1, Flatten (NCHW order) and FullyConnected policy_out onto the classic labels; then the SoftmaxOutput.  The
trunk and the value head come from oracle/net_mx.py, which pins them to the reference's symbols.
"""
import numpy as np
import torch
import torch.nn.functional as F

from crazyara_b200 import synthetic
from oracle import net_mx


def classic_arch(base, n_labels):
    """an arch of oracle/net_mx.py with the head onto n_labels classic labels; its header's policy_bias is 0 (ARAB2004
    carries the convolution's bias with the head)"""
    return synthetic.classic(dict(base, policy_bias=False), n_labels)


def head_params(arch, n_labels, seed=0):
    """Seeded parameters of policy_bn1 and policy_out under the symbol's names, from a generator of their own so that the
    rest of the parameters stay as oracle/net_mx.make_mx_params makes them.  The gamma is random too: fix_gamma ignores
    it.  The logits come out with a spread of a few units, as a trained head's do."""
    g = np.random.default_rng([seed, n_labels, 2])
    P, f32 = arch["policy_channels"], np.float32
    k = P * 64
    return {"policy_bn1_gamma": g.uniform(0.5, 1.5, P).astype(f32),
            "policy_bn1_beta": (g.standard_normal(P) * 0.1).astype(f32),
            "policy_bn1_moving_mean": (g.standard_normal(P) * 0.1).astype(f32),
            "policy_bn1_moving_var": g.uniform(0.5, 1.5, P).astype(f32),
            "policy_out_weight": (g.standard_normal((n_labels, k)) * 2.0 / np.sqrt(k)).astype(f32),
            "policy_out_bias": (g.standard_normal(n_labels) * 0.1).astype(f32)}


def make_params(base, n_labels, seed=0):
    """-> (classic arch, parameters): oracle/net_mx.make_mx_params of the base arch (policy_conv1's bias where the
    symbol has one) and the head's"""
    params = net_mx.make_mx_params(base, seed)
    params.update(head_params(base, n_labels, seed))
    return classic_arch(base, n_labels), params


def forward(params, arch, x, eps=net_mx.BN_EPS):
    """-> oracle/net_mx.forward_mx's outputs with policy_logits / prob [B, L]"""
    out = net_mx.forward_mx(params, arch, x, eps)
    p = {k: torch.as_tensor(v, dtype=torch.float32) for k, v in params.items()}
    bn = lambda t, n: F.batch_norm(t, p[n + "_moving_mean"], p[n + "_moving_var"], None, p[n + "_beta"], training=False, eps=eps)
    with torch.no_grad():
        t = torch.as_tensor(out["trunk"])
        ph = F.relu(bn(F.conv2d(t, p["policy_conv0_weight"], padding=1), "policy_bn0"))
        ph = F.conv2d(ph, p["policy_conv1_weight"], p.get("policy_conv1_bias"), padding=1)
        ph = F.relu(bn(ph, "policy_bn1")).reshape(t.shape[0], -1)
        logits = F.linear(ph, p["policy_out_weight"], p["policy_out_bias"])
        out.update(policy_logits=logits.numpy(), prob=torch.softmax(logits, dim=1).numpy())
    return out
