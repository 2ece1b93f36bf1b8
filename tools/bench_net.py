"""Raw network throughput (the reference's UCI `inference` command, engine/src/uci/crazyara.cpp:156-181)."""
import os
import sys
import tempfile
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from crazyara_b200.nn import NeuralNetAPI  # noqa: E402
from crazyara_b200.weights import export_blob, export_mx_blob  # noqa: E402
from crazyara_b200 import synthetic  # noqa: E402


def _blob(name, d):
    """the PyTorch-defined networks (ARAB2001) and their MXNet-symbol twins (ARAB2002: SE off the shortcut)"""
    path = os.path.join(d, "w.arab")
    if name == "risev2":
        arch = synthetic.risev2(34, 81)
        return arch, export_blob(synthetic.random_state_dict(arch, 0), arch, path, input_version=10)
    if name == "risev33":
        arch = synthetic.risev33(52, 76, True)
        return arch, export_blob(synthetic.random_state_dict(arch, 0), arch, path, input_version=30)
    arch = synthetic.mx_twin(synthetic.risev2(34, 81) if name == "mx_risev2" else synthetic.risev33(52, 76))
    return arch, export_mx_blob(synthetic.random_mx_params(arch, 0), arch, path, input_version=10 if name == "mx_risev2" else 30)


def main():
    import torch
    iters = int(os.environ.get("ITERS", "200"))
    names = os.environ.get("NETS", "risev2,risev33").split(",")  # also: mx_risev2, mx_risev33
    batches = [int(b) for b in os.environ.get("BATCHES", "1,8,64,128").split(",")]
    for name in names:
        with tempfile.TemporaryDirectory() as d:
            arch, blob = _blob(name, d)
            for batch in batches:
                net = NeuralNetAPI("gpu", 0, batch, blob)
                C = arch["in_channels"]
                x = torch.rand(batch, C, 8, 8).pin_memory()
                v = torch.empty(batch).pin_memory()
                p = torch.empty(batch, arch["policy_channels"] * 64).pin_memory()
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
                print(f"{name} B={batch:4d} host-api {t_host*1e6:8.1f} us ({batch/t_host:10.0f} evals/s)  "
                      f"device {t_dev*1e6:8.1f} us ({batch/t_dev:10.0f} evals/s)", flush=True)
                net.close()


if __name__ == "__main__":
    main()
