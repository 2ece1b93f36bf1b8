"""Generates tests/golden/import_golden.json: the SHA-256 of every blob the weight import writes for the networks the tests
use (export_blob, export_mx_blob with each BatchNorm option, import_checkpoint, import_onnx on each test writer's file),
the architecture dicts the importers return, and the SHA-256 of each test writer's ONNX file.  tests/test_import_golden.py
recomputes every entry, so a change to the import code that moves a byte of any blob fails there.
    python tests/golden/gen_import_golden.py
"""
import hashlib
import json
import os
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from crazyara_b200 import synthetic  # noqa: E402
from crazyara_b200.onnx_import import import_onnx  # noqa: E402
from crazyara_b200.weights import export_blob, export_mx_blob, import_checkpoint  # noqa: E402
from oracle import net as onet  # noqa: E402
from oracle import net_alphavile as oav  # noqa: E402
from oracle import net_mx  # noqa: E402
from tests.onnx_alphavile_writer import write_alphavile_onnx  # noqa: E402
from tests.onnx_mx_writer import write_mx_onnx  # noqa: E402
from tests.onnx_writer import add_shape_concat, write_rise_onnx  # noqa: E402
from tests.net_harness import mixed_arch  # noqa: E402

PATH = os.path.join(ROOT, "tests", "golden", "import_golden.json")
RISE = {"risev2": (lambda: synthetic.risev2(34, 81), 10), "risev33": (lambda: synthetic.risev33(52, 76), 30)}
MX = {"mx_risev2": lambda: net_mx.arch_mx_risev2(34, 81), "mx_risev33": lambda: net_mx.arch_mx_risev33(52, 76),
      "mx_mixed": mixed_arch}
MX_BN = {"default": {}, "eps_f32": dict(eps=float(np.float32(1e-3))),
         "eps_dict": dict(eps={"stem_bn0": 1e-5, "bc_res_block0_bn1": 2e-5, "bc_res_block0_bn1_bn1": 2e-5}),
         "gamma": dict(fix_gamma=False)}


def alphavile_arch(size):
    return oav.arch_alphavile(size, 34, 81, False) if size in ("tiny", "small") else oav.arch_alphavile(size, 52, 76, True)


def make_cases(tmp):
    """-> ({case: (blob path, returned arch or None)}, {ONNX file: path}), everything written under tmp"""
    import torch
    blobs, onnx = {}, {}
    f = lambda name: os.path.join(tmp, name)
    for name, (make, version) in RISE.items():
        arch = make()
        sd = synthetic.random_state_dict(arch, 3)
        blobs["export_blob/" + name] = (export_blob(sd, arch, f(name + ".arab"), input_version=version), None)
        onnx["rise/" + name] = write_rise_onnx(sd, arch, f(name + ".onnx"))
        blobs["import_onnx/" + name] = (f(name + "-onnx.arab"), import_onnx(onnx["rise/" + name], f(name + "-onnx.arab")))
        concat = add_shape_concat(write_rise_onnx(sd, arch, f(name + "-concat.onnx")))
        blobs["import_onnx/" + name + "_shape_concat"] = (f(name + "-concat.arab"), import_onnx(concat, f(name + "-concat.arab")))
    for size in oav.SIZES:
        arch = alphavile_arch(size)
        sd = oav.make_state_dict(arch, 4)
        version = 10 if size in ("tiny", "small") else 30
        blobs["export_blob/alphavile_" + size] = (export_blob(sd, arch, f(size + ".arab"), input_version=version), None)
        onnx["alphavile/" + size] = write_alphavile_onnx(sd, arch, f(size + ".onnx"))
        blobs["import_onnx/alphavile_" + size] = (f(size + "-onnx.arab"), import_onnx(onnx["alphavile/" + size], f(size + "-onnx.arab")))
    for name, make in MX.items():
        arch = make()
        params = net_mx.make_mx_params(arch, 4)
        for bn, kw in MX_BN.items():
            blobs[f"export_mx_blob/{name}_{bn}"] = (export_mx_blob(params, arch, f(f"{name}-{bn}.arab"), **kw), None)
        onnx["mx/" + name] = write_mx_onnx(params, arch, f(name + ".onnx"))
        blobs["import_onnx/" + name] = (f(name + "-onnx.arab"), import_onnx(onnx["mx/" + name], f(name + "-onnx.arab")))
    arch = net_mx.arch_mx_risev2(34, 81)
    eps = write_mx_onnx(net_mx.make_mx_params(arch, 4), arch, f("mx-eps.onnx"), eps=2e-5)
    blobs["import_onnx/mx_risev2_eps_2e-5"] = (f("mx-eps.arab"), import_onnx(eps, f("mx-eps.arab")))
    for name, arch, make_sd in (("rise", onet.arch_risev33(52, 76, True), onet.make_state_dict),
                                ("alphavile", alphavile_arch("normal"), oav.make_state_dict)):
        sd = make_sd(arch, 2)
        ck = f(name + ".tar")
        torch.save({"model_state_dict": {"module." + k: torch.from_numpy(np.asarray(v)) for k, v in sd.items()}}, ck)
        blobs["import_checkpoint/" + name] = (f(name + "-ck.arab"), import_checkpoint(ck, f(name + "-ck.arab")))
    return blobs, onnx


def sha(path):
    return hashlib.sha256(open(path, "rb").read()).hexdigest()


def record(blobs, onnx):
    """the golden record of make_cases' output, as JSON types"""
    return json.loads(json.dumps(dict(blobs={k: sha(p) for k, (p, _) in sorted(blobs.items())},
                                      archs={k: a for k, (_, a) in sorted(blobs.items()) if a is not None},
                                      onnx={k: sha(p) for k, p in sorted(onnx.items())})))


def main():
    with tempfile.TemporaryDirectory() as tmp:
        rec = record(*make_cases(tmp))
    with open(PATH, "w") as f:
        json.dump(rec, f, indent=1, sort_keys=True)
        f.write("\n")
    print("wrote", PATH, len(rec["blobs"]), "blobs,", len(rec["archs"]), "archs,", len(rec["onnx"]), "ONNX files")


if __name__ == "__main__":
    main()
