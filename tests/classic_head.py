"""The fully-connected policy head (the reference trainer's select_policy_from_plane=False) on top of the fp32 oracle
networks -- TEST INFRASTRUCTURE ONLY.

Follows builder_util.py _PolicyHead (:206-243): body = conv3x3 + BN + ReLU + conv3x3 (no bias), body2 = BN + ReLU,
flatten in NCHW order, body3 = Linear onto the classic labels; then the softmax the engine's backend appends
(tensorrtapi.cpp:378-380).  The trunk comes from the oracle networks (oracle/net.py, oracle/net_alphavile.py), which
already pin the trunk, the value head and the first policy convolution to the reference.
"""
import torch
import torch.nn.functional as F

BN_EPS = 1e-5


def _bn(x, sd, p):
    return F.batch_norm(x, sd[p + ".running_mean"], sd[p + ".running_var"], sd[p + ".weight"], sd[p + ".bias"],
                        training=False, eps=BN_EPS)


def forward(oracle_forward, sd_np, arch, x):
    """oracle_forward: oracle.net.forward or oracle.net_alphavile.forward; sd_np: its state_dict with the head's
    parameters (crazyara_b200.synthetic.classic_head) -> the oracle's outputs with policy_logits / prob [B, L]."""
    out = oracle_forward(sd_np, arch, x)
    sd = {k: torch.as_tensor(v, dtype=torch.float32) for k, v in sd_np.items()}
    with torch.no_grad():
        t = torch.as_tensor(out["trunk"])
        ph = F.relu(_bn(F.conv2d(t, sd["policy_head.body.0.weight"], padding=1), sd, "policy_head.body.1"))
        ph = F.conv2d(ph, sd["policy_head.body.3.weight"], padding=1)
        ph = F.relu(_bn(ph, sd, "policy_head.body2.0")).reshape(t.shape[0], -1)
        logits = F.linear(ph, sd["policy_head.body3.0.weight"], sd["policy_head.body3.0.bias"])
        out.update(policy_logits=logits.numpy(), prob=torch.softmax(logits, dim=1).numpy())
    return out
