"""Raw network throughput (the reference's UCI `inference` command, engine/src/uci/crazyara.cpp:156-181).

A name with the suffix _fc<L> (risev2_fc2272, risev33_fc1968, alphavile_tiny_fc2316, ...) is the same network with a
fully-connected policy head onto L classic labels (ARAB2004); for those the time of the head's two kernels
(policy_fc_kernel, policy_fc_softmax_kernel) per forward is read from a torch.profiler trace of a separate run.

risev33_wdl_mlp (the trainer's value MLP, use_mlp_wdl_ply), mx_risev33_wdl and mx_risev33_wdl_mlp (the MXNet symbols'
WDL head, win - loss or the MLP) carry the value heads of kinds 2, 3 and 4 (crazyara_b200/weights.py VALUE_HEADS).  For
every network the time of value_head_kernel per forward is read from the same kind of trace."""
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from crazyara_b200.nn import NeuralNetAPI  # noqa: E402
from crazyara_b200.weights import export_blob, export_mx_blob  # noqa: E402
from crazyara_b200 import synthetic  # noqa: E402


def _blob(name, d):
    """the PyTorch-defined networks (ARAB2001), their MXNet-symbol twins (ARAB2002: SE off the shortcut) and AlphaVile
    (ARAB2003: alphavile_tiny, crazyhouse 34 -> 81; alphavile_normal, chess 52 -> 76 with WDL)"""
    path = os.path.join(d, "w.arab")
    g = np.random.default_rng(1)
    linear = lambda out, cin: ((g.standard_normal((out, cin)) / np.sqrt(cin)).astype(np.float32),
                               (g.standard_normal(out) * 0.1).astype(np.float32))
    if name == "risev33_wdl_mlp":
        arch = dict(synthetic.risev33(52, 76, True), value_head="wdl_mlp")
        sd = synthetic.random_state_dict(arch, 0)
        for key, (out, cin) in (("value_head.body_final.0", (8, 4)), ("value_head.body_final.2", (1, 8))):
            sd[key + ".weight"], sd[key + ".bias"] = linear(out, cin)
        return arch, export_blob(sd, arch, path, input_version=30)
    if name in ("mx_risev33_wdl", "mx_risev33_wdl_mlp"):
        arch = dict(synthetic.mx_twin(synthetic.risev33(52, 76)), wdl=True, value_head="mx_" + name[len("mx_risev33_"):],
                    value_fc=256)
        params = synthetic.random_mx_params(arch, 0)
        layers = [("wdl_out", 3, 256), ("value_plys_to_end_fc", 1, 256)]
        layers += [("value_wdl_ply_fc", 8, 4), ("value_fc1", 1, 8)] if arch["value_head"] == "mx_wdl_mlp" else []
        for key, out, cin in layers:
            params[key + "_weight"], params[key + "_bias"] = linear(out, cin)
        return arch, export_mx_blob(params, arch, path, input_version=30)
    if "_fc" in name:
        base, n_labels = name.rsplit("_fc", 1)
        arch, _ = _blob(base, d)
        arch = synthetic.classic(arch, int(n_labels))
        return arch, export_blob(synthetic.random_state_dict(arch, 0), arch, path, input_version=30 if arch["wdl"] else 10)
    if name.startswith("alphavile_"):
        size = name[len("alphavile_"):]
        arch = synthetic.alpha_vile(size, 34, 81, False) if size in ("tiny", "small") else synthetic.alpha_vile(size, 52, 76, True)
        return arch, export_blob(synthetic.random_state_dict(arch, 0), arch, path, input_version=10 if size in ("tiny", "small") else 30)
    if name == "risev2":
        arch = synthetic.risev2(34, 81)
        return arch, export_blob(synthetic.random_state_dict(arch, 0), arch, path, input_version=10)
    if name == "risev33":
        arch = synthetic.risev33(52, 76, True)
        return arch, export_blob(synthetic.random_state_dict(arch, 0), arch, path, input_version=30)
    arch = synthetic.mx_twin(synthetic.risev2(34, 81) if name == "mx_risev2" else synthetic.risev33(52, 76))
    return arch, export_mx_blob(synthetic.random_mx_params(arch, 0), arch, path, input_version=10 if name == "mx_risev2" else 30)


def _head_us(net, xd, batch, iters):
    """device time per forward of the value head's kernel and the fully-connected policy head's, from a torch.profiler
    trace"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(iters):
            net.forward_device(xd.data_ptr(), batch)
        torch.cuda.synchronize()
    times = {}
    for e in prof.events():
        if e.device_type == torch.autograd.DeviceType.CUDA and ("policy_fc" in e.name or "value_head" in e.name):
            key = "value" if "value_head" in e.name else "softmax" if "softmax" in e.name else "gemm"
            times[key] = times.get(key, 0.0) + e.device_time / iters
    return times


def main():
    import torch
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip().splitlines()
    print(f"card: {card[0] if card else 'unknown'}", flush=True)
    iters = int(os.environ.get("ITERS", "200"))
    names = os.environ.get("NETS", "risev2,risev33").split(",")  # also: mx_risev2, mx_risev33, alphavile_<size>, the
    # value heads risev33_wdl_mlp, mx_risev33_wdl, mx_risev33_wdl_mlp
    batches = [int(b) for b in os.environ.get("BATCHES", "1,8,64,128").split(",")]
    for name in names:
        with tempfile.TemporaryDirectory() as d:
            arch, blob = _blob(name, d)
            for batch in batches:
                net = NeuralNetAPI("gpu", 0, batch, blob)
                C = arch["in_channels"]
                x = torch.rand(batch, C, 8, 8).pin_memory()
                v = torch.empty(batch).pin_memory()
                p = torch.empty(batch, arch.get("n_labels") or arch["policy_channels"] * 64).pin_memory()
                xn, vn, pn = x.numpy(), v.numpy(), p.numpy()
                for _ in range(5):
                    net.predict(xn, vn, pn, None)
                t0 = time.perf_counter()
                for _ in range(iters):
                    net.predict(xn, vn, pn, None)
                t_host = (time.perf_counter() - t0) / iters
                xd = x.cuda()
                for _ in range(5):
                    net.forward_device(xd.data_ptr(), batch)
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                for _ in range(iters):
                    net.forward_device(xd.data_ptr(), batch)
                t_dev = (time.perf_counter() - t0) / iters
                t = _head_us(net, xd, batch, min(iters, 50))
                fc = f"  value head {t.get('value', 0.0):6.1f} us"
                if arch.get("n_labels"):
                    fc += f"  fc head: gemm {t.get('gemm', 0.0):6.1f} us + softmax {t.get('softmax', 0.0):6.1f} us"
                print(f"{name} B={batch:4d} host-api {t_host*1e6:8.1f} us ({batch/t_host:10.0f} evals/s)  "
                      f"device {t_dev*1e6:8.1f} us ({batch/t_dev:10.0f} evals/s){fc}", flush=True)
                net.close()


if __name__ == "__main__":
    main()
