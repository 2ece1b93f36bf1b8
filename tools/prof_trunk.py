"""Per-role cycle breakdown of the persistent trunk kernel (CTA 0), from the -DARA_TRUNK_PROF build:
    make tprof && ARA_B200_LIB=build/libara_b200_tprof.so python tools/prof_trunk.py [arch] [batch]"""
import ctypes
import os
import sys
import tempfile

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from crazyara_b200 import lib
from crazyara_b200.nn import NeuralNetAPI
from crazyara_b200.weights import export_blob
from crazyara_b200 import synthetic

arch_name = sys.argv[1] if len(sys.argv) > 1 else "risev2"
B = int(sys.argv[2]) if len(sys.argv) > 2 else 64
arch = synthetic.risev2(34, 81) if arch_name == "risev2" else synthetic.risev33(52, 76)
d = tempfile.mkdtemp()
blob = export_blob(synthetic.random_state_dict(arch, 0), arch, os.path.join(d, "w.arab"), input_version=10 if arch_name == "risev2" else 30)
net = NeuralNetAPI("gpu", 0, B, blob)
x = np.random.default_rng(0).random((B, arch["in_channels"], 8, 8), dtype=np.float32)
val = np.zeros(B, np.float32)
prob = np.zeros((B, arch["policy_channels"] * 64), np.float32)
for _ in range(5):
    net.predict(x, val, prob)
out = (ctypes.c_ulonglong * 32)()
L = lib()
L.ara_net_debug_trunk_cycles.argtypes = [ctypes.c_void_p, ctypes.c_void_p]
if L.ara_net_debug_trunk_cycles(net._h, out) != 0:
    raise SystemExit(L.ara_last_error().decode())
# RT_PROF slots of the consumer warpgroup of board 0 (rise_trunk.cuh): rise_trunk_kernel flushes at offset 16, the pair
# kernel (warpgroup 0 of its CTA of rank 0) at offset 0
if any(out[i] for i in range(16)):
    shape, base = "pair kernel, warpgroup 0 of the CTA of rank 0", 0
    names = ["X load + cluster barrier", "wait SE image", "squeeze-excitation (split)", "wait W1 image",
             "MMA1 (wgmma m64n32)", "epilogue 1 (relu + b1 -> H1)", "wait own H2 buffer free",
             "depthwise -> H2 + copy", "wait partner's H2", "wait W2 half", "MMA2 (wgmma m64n64)",
             "wait partner's X free", "block epilogue + X panel copy", "wait partner's X"]
else:
    shape, base = "one / two boards per CTA", 16
    names = ["X load", "squeeze-excitation", "wait W1 image", "MMA1 (wgmma m64n64)", "epilogue 1 (relu + b1 -> H1)",
             "depthwise -> H2", "wait W2 image", "MMA2 (wgmma m64n256)", "block epilogue (D2 + b2 + X)"]
vals = [out[base + i] for i in range(len(names))]
tot = sum(vals)
print(f"consumer warpgroup of board 0 ({shape}): {tot / 1e3:.1f} kcycles")
for n, v in zip(names, vals):
    print(f"    {n:34s} {v / 1e3:9.1f} kcycles {100.0 * v / max(1, tot):5.1f}%")
