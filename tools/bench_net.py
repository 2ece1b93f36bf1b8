"""Raw network throughput (the reference's UCI `inference` command, engine/src/uci/crazyara.cpp:156-181).

A name with the suffix _fc<L> (risev2_fc2272, risev33_fc1968, alphavile_tiny_fc2316, ...) is the same network with a
fully-connected policy head onto L classic labels (ARAB2004); for those the time of the head's two kernels
(policy_fc_kernel, policy_fc_softmax_kernel) per forward is read from a torch.profiler trace of a separate run."""
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


def _fc_head_us(net, xd, batch, iters):
    """device time per forward of the fully-connected head's kernels, from a torch.profiler trace"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(iters):
            net.forward_device(xd.data_ptr(), batch)
        torch.cuda.synchronize()
    times = {}
    for e in prof.events():
        if e.device_type == torch.autograd.DeviceType.CUDA and "policy_fc" in e.name:
            key = "softmax" if "softmax" in e.name else "gemm"
            times[key] = times.get(key, 0.0) + e.device_time / iters
    return times


def main():
    import torch
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip().splitlines()
    print(f"card: {card[0] if card else 'unknown'}", flush=True)
    iters = int(os.environ.get("ITERS", "200"))
    names = os.environ.get("NETS", "risev2,risev33").split(",")  # also: mx_risev2, mx_risev33, alphavile_<size>
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
                fc = ""
                if arch.get("n_labels"):
                    t = _fc_head_us(net, xd, batch, min(iters, 50))
                    fc = f"  fc head: gemm {t.get('gemm', 0.0):6.1f} us + softmax {t.get('softmax', 0.0):6.1f} us"
                print(f"{name} B={batch:4d} host-api {t_host*1e6:8.1f} us ({batch/t_host:10.0f} evals/s)  "
                      f"device {t_dev*1e6:8.1f} us ({batch/t_dev:10.0f} evals/s){fc}", flush=True)
                net.close()


if __name__ == "__main__":
    main()
