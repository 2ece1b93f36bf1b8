"""Random-weight networks of the reference's architectures, for benchmarks and profiling without trained weights.

Counterpart of the reference's DeepCrazyhouse/src/domain/neural_net/generate_random_nn.py (a script that writes randomly initialised networks
of the right shapes so that the engine can be benchmarked without a trained model).  The architecture tables follow
DeepCrazyhouse/src/domain/neural_net/architectures/pytorch/rise_mobile_v3.py (:217-241 get_rise_v2_model: 13 blocks,
operating channels 128 + 64 i, channel attention on the last five; :186-214 get_rise_v33_model: 15 blocks, mixed 3x3 /
5x5 depthwise, efficient channel attention, WDL head; :36-78 _get_res_blocks), the parameter names are the reference
trainer's state_dict keys, so the result goes through the same import path as a real checkpoint
(crazyara_b200.weights.export_blob).  alpha_vile follows DeepCrazyhouse/src/domain/neural_net/architectures/pytorch/
alpha_vile.py (get_alpha_vile_model, generate_random_nn.py --model-type alpha_vile).
"""
import numpy as np


def risev2(in_channels=34, policy_channels=81):
    n = 13
    return dict(name="risev2", in_channels=in_channels, policy_channels=policy_channels, channels=256,
                kernels=[3] * n, se_types=[("ca_se" if i >= 8 else None) for i in range(n)],
                c_ops=[128 + 64 * i for i in range(n)], wdl=False, value_channels=8, value_fc=256)


def risev33(in_channels=52, policy_channels=76, wdl=True):
    kernels = [5 if i in (7, 11, 12, 13) else 3 for i in range(15)]
    se = [("eca_se" if i in (5, 8, 12, 13, 14) else None) for i in range(15)]
    c_ops = [(224 + 32 * i) - (32 * (i // 2) if k == 5 else 0) for i, k in enumerate(kernels)]
    return dict(name="risev33", in_channels=in_channels, policy_channels=policy_channels, channels=256, kernels=kernels,
                se_types=se, c_ops=c_ops, wdl=wdl, value_channels=8, value_fc=256)


_AV_K5 = {"tiny": (1, 2, 6, 7, 8, 9, 10), "small": (0, 4, 5, 6, 10, 11, 13, 15, 17, 20),
          "normal": (0, 4, 5, 7, 10, 12, 15, 16, 20, 21, 22, 23, 24, 25),
          "large": (1, 6, 7, 9, 10, 14, 18, 19, 23, 25, 26, 27, 28, 29, 33, 34, 35)}


def alpha_vile(size="normal", in_channels=52, policy_channels=76, wdl=True):
    """get_alpha_vile_model (alpha_vile.py:14-141): trunk 192 (tiny, small) or 224 (normal, large) channels, 15 / 22 / 26 /
    37 blocks, operating width 2 C (5x5 blocks: 0.68 of it, rounded to 32), NextViT transformer blocks (ntb) at the
    positions _get_res_blocks' rule gives, MHSA width 160, MHCA width C - 160, MLP width 2 C, value_fc = C."""
    C = 192 if size in ("tiny", "small") else 224
    depth = {"tiny": 15, "small": 22, "normal": 26, "large": 37}[size]
    step = depth // (2 if size in ("tiny", "small") else 3)
    ntb = [False] * depth
    for i in range(depth % step + 2 * step - 1, depth, step):
        ntb[i] = True
    kernels = [5 if i in _AV_K5[size] else 3 for i in range(depth)]
    k5 = int(2 * C * 0.68 / 32 + 0.5) * 32
    return dict(name=f"alphavile_{size}", in_channels=in_channels, policy_channels=policy_channels, channels=C,
                kernels=kernels, se_types=[None] * depth, c_ops=[k5 if k == 5 else 2 * C for k in kernels], ntb=ntb,
                mhsa=160, mhca=C - 160, mlp=2 * C, wdl=wdl, value_channels=8, value_fc=C)


def random_state_dict(arch, seed=0):
    """Seeded parameters with activations of order one through the whole tower (He-scaled convolutions, a damped
    residual branch) and non-trivial BatchNorm statistics, so that BN folding and the fp16 range are exercised."""
    g = np.random.default_rng(seed)
    sd = {}
    f32 = np.float32

    def normal(shape, std):
        return (g.standard_normal(shape) * std).astype(f32)

    def batchnorm(key, c):
        sd[key + ".weight"] = g.uniform(0.8, 1.2, c).astype(f32)
        sd[key + ".bias"] = normal(c, 0.1)
        sd[key + ".running_mean"] = normal(c, 0.1)
        sd[key + ".running_var"] = g.uniform(0.5, 1.5, c).astype(f32)

    C = arch["channels"]
    sd["body_spatial.0.body.0.weight"] = normal((C, arch["in_channels"], 3, 3), np.sqrt(2.0 / (9 * arch["in_channels"])))
    batchnorm("body_spatial.0.body.1", C)
    ntb = arch.get("ntb") or [False] * len(arch["kernels"])
    for i, (k, se, cop) in enumerate(zip(arch["kernels"], arch["se_types"], arch["c_ops"]), start=1):
        blk = f"body_spatial.{i}"
        if ntb[i - 1]:  # NextViT transformer block (next_vit_official_modules.py:265-335), head width 32
            M, Ca, H = arch["mhsa"], arch["mhca"], arch["mlp"]
            sd[blk + ".patch_embed.conv.weight"] = normal((M, C, 1, 1), 0.3 / np.sqrt(C))
            batchnorm(blk + ".patch_embed.norm", M)
            batchnorm(blk + ".norm1", M)
            for n, std in (("q", 9.0), ("k", 9.0), ("v", 1.0), ("proj", 0.5)):
                sd[f"{blk}.e_mhsa.{n}.weight"], sd[f"{blk}.e_mhsa.{n}.bias"] = normal((M, M), std / np.sqrt(M)), normal(M, 0.1)
            sd[blk + ".projection.conv.weight"] = normal((Ca, M, 1, 1), np.sqrt(2.0 / M))
            batchnorm(blk + ".projection.norm", Ca)
            sd[blk + ".mhca.group_conv3x3.weight"] = normal((Ca, 32, 3, 3), np.sqrt(2.0 / (32 * 9)))
            batchnorm(blk + ".mhca.norm", Ca)
            sd[blk + ".mhca.projection.weight"] = normal((Ca, Ca, 1, 1), 0.5 / np.sqrt(Ca))
            batchnorm(blk + ".norm2", C)
            sd[blk + ".mlp.conv1.weight"], sd[blk + ".mlp.conv1.bias"] = normal((H, C, 1, 1), np.sqrt(2.0 / C)), normal(H, 0.1)
            sd[blk + ".mlp.conv2.weight"], sd[blk + ".mlp.conv2.bias"] = normal((C, H, 1, 1), 0.25 / np.sqrt(H)), normal(C, 0.1)
            continue
        if se == "ca_se":
            sd[blk + ".se.fc.0.weight"] = normal((C // 2, C), 2.0 / np.sqrt(C))
            sd[blk + ".se.fc.2.weight"] = normal((C, C // 2), 2.0 / np.sqrt(C // 2))
        elif se == "eca_se":
            sd[blk + ".se.body.0.weight"] = normal((C, C, 5), 2.0 / np.sqrt(C))
            sd[blk + ".se.body.0.bias"] = normal(C, 0.5)
        sd[blk + ".body.0.weight"] = normal((cop, C, 1, 1), np.sqrt(2.0 / C))
        batchnorm(blk + ".body.1", cop)
        sd[blk + ".body.3.weight"] = normal((cop, 1, k, k), np.sqrt(2.0 / (k * k)))
        batchnorm(blk + ".body.4", cop)
        sd[blk + ".body.6.weight"] = normal((C, cop, 1, 1), 0.5 / np.sqrt(cop))
        batchnorm(blk + ".body.7", C)
    vc = arch["value_channels"]
    sd["value_head.body.0.weight"] = normal((vc, C, 1, 1), np.sqrt(2.0 / C))
    batchnorm("value_head.body.1", vc)
    if arch["wdl"]:
        for name, n_out in (("body_wdl", 3), ("body_plys", 1)):
            sd[f"value_head.{name}.0.weight"] = normal((n_out, vc * 64), 1.0 / np.sqrt(vc * 64))
            sd[f"value_head.{name}.0.bias"] = normal(n_out, 0.1)
    else:
        fc = arch["value_fc"]
        sd["value_head.body_final.0.weight"] = normal((fc, vc * 64), 1.4 / np.sqrt(vc * 64))
        sd["value_head.body_final.0.bias"] = normal(fc, 0.1)
        sd["value_head.body_final.2.weight"] = normal((1, fc), 1.4 / np.sqrt(fc))
        sd["value_head.body_final.2.bias"] = normal(1, 0.1)
    sd["policy_head.body.0.weight"] = normal((C, C, 3, 3), np.sqrt(2.0 / (9 * C)))
    batchnorm("policy_head.body.1", C)
    sd["policy_head.body.3.weight"] = normal((arch["policy_channels"], C, 3, 3), 2.0 * np.sqrt(2.0 / (9 * C)))
    if arch.get("n_labels"):
        sd.update(classic_head(arch, arch["n_labels"], seed))
    return sd


def classic(arch, n_labels):
    """the same network with a fully-connected policy head onto the n_labels classic labels (the trainer's
    select_policy_from_plane=False, builder_util.py _PolicyHead): 1968 chess, 2272 crazyhouse, 2316 lichess variants"""
    return dict(arch, name=f"{arch['name']}_fc{n_labels}", n_labels=n_labels)


def classic_head(arch, n_labels, seed=0):
    """Seeded parameters of the fully-connected policy head under the state_dict names (policy_head.body2.0 BatchNorm2d,
    policy_head.body3.0 Linear), from a generator of their own so that the rest of a state_dict stays as it is.  The
    logits come out with a spread of a few units, as a trained head's do."""
    g = np.random.default_rng([seed, n_labels])
    P, f32 = arch["policy_channels"], np.float32
    k = P * 64
    return {"policy_head.body2.0.weight": g.uniform(0.8, 1.2, P).astype(f32),
            "policy_head.body2.0.bias": (g.standard_normal(P) * 0.1).astype(f32),
            "policy_head.body2.0.running_mean": (g.standard_normal(P) * 0.1).astype(f32),
            "policy_head.body2.0.running_var": g.uniform(0.5, 1.5, P).astype(f32),
            "policy_head.body3.0.weight": (g.standard_normal((n_labels, k)) * 2.0 / np.sqrt(k)).astype(f32),
            "policy_head.body3.0.bias": (g.standard_normal(n_labels) * 0.1).astype(f32)}


def mx_twin(arch):
    """the same tower as the reference's MXNet symbols define it (rise_mobile_v2.py / rise_mobile_v3.py; see
    crazyara_b200.weights.export_mx_blob): v2 (ca_se) with sigmoid gates, a stem ReLU and no policy bias; v3 (eca_se) with
    clamp(0.2 x + 0.5) gates, no stem activation, a policy bias and the plain value head"""
    v2 = "ca_se" in arch["se_types"]
    return dict(arch, name="mx_" + arch["name"], semantics="mxnet", wdl=False, stem_act=v2, policy_bias=not v2,
                se_gates=[(("sigmoid" if v2 else "hard_sigmoid") if s else None) for s in arch["se_types"]])


def random_mx_params(arch, seed=0):
    """Seeded parameters of an mx_twin network under the symbol code's names (BatchNorm as name_gamma / _beta /
    _moving_mean / _moving_var, eca_se convolutions as convolution<n>), scaled like random_state_dict"""
    g = np.random.default_rng(seed)
    p = {}
    normal = lambda shape, std: (g.standard_normal(shape) * std).astype(np.float32)

    def conv_bn(name, bn, cout, cin, k, groups=1, std=None):
        p[name + "_weight"] = normal((cout, cin // groups, k, k), std or np.sqrt(2.0 / (cin // groups * k * k)))
        p[bn + "_gamma"], p[bn + "_beta"] = np.ones(cout, np.float32), normal(cout, 0.1)
        p[bn + "_moving_mean"], p[bn + "_moving_var"] = normal(cout, 0.1), g.uniform(0.5, 1.5, cout).astype(np.float32)

    C, n_eca = arch["channels"], 0
    conv_bn("stem_conv0", "stem_bn0", C, arch["in_channels"], 3)
    for i, (k, se, cop) in enumerate(zip(arch["kernels"], arch["se_types"], arch["c_ops"])):
        b = f"bc_res_block{i}"
        if se == "ca_se":
            p[b + "_se_fc0_weight"], p[b + "_se_fc0_bias"] = normal((C // 2, C), 2.0 / np.sqrt(C)), normal(C // 2, 0.1)
            p[b + "_se_fc1_weight"], p[b + "_se_fc1_bias"] = normal((C, C // 2), 2.0 / np.sqrt(C // 2)), normal(C, 0.1)
        elif se == "eca_se":
            p[f"convolution{n_eca}_weight"], p[f"convolution{n_eca}_bias"] = normal((1, 1, 5), 1.0), normal(1, 0.5)
            n_eca += 1
        conv_bn(b + "_conv1", b + "_bn1", cop, C, 1)
        conv_bn(b + "_conv2", b + "_bn2", cop, cop, k, groups=cop)
        conv_bn(b + "_conv3", b + "_bn3", C, cop, 1, std=0.5 / np.sqrt(cop))
    conv_bn("value_conv0", "value_bn0", arch["value_channels"], C, 1)
    n = arch["value_channels"] * 64
    p["value_fc0_weight"], p["value_fc0_bias"] = normal((arch["value_fc"], n), 1.0 / np.sqrt(n)), normal(arch["value_fc"], 0.1)
    p["value_fc1_weight"], p["value_fc1_bias"] = normal((1, arch["value_fc"]), 1.0 / np.sqrt(arch["value_fc"])), normal(1, 0.1)
    conv_bn("policy_conv0", "policy_bn0", C, C, 3)
    p["policy_conv1_weight"] = normal((arch["policy_channels"], C, 3, 3), np.sqrt(2.0 / (9 * C)))
    if arch["policy_bias"]:
        p["policy_conv1_bias"] = normal(arch["policy_channels"], 0.1)
    return p
