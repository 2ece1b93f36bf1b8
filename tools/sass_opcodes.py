"""Per-kernel counts of Hopper SASS opcodes in the built library: HGMMA / WARPGROUP (wgmma), UTMALDG (TMA), UBLKCP
(bulk copies), SYNCS (mbarrier), REDUX and the total.  CPU only:  python tools/sass_opcodes.py"""
import collections
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "crazyara_b200", "libara_b200.so")
OPS = ["HGMMA", "WARPGROUP", "UTMALDG", "UTMASTG", "UBLKCP", "SYNCS", "REDUX", "HMMA", "FFMA", "HFMA2", "DFMA", "LDS", "STS", "LDG", "STG"]


def main():
    txt = subprocess.run(["cuobjdump", "-sass", LIB], capture_output=True, text=True, check=True).stdout
    kernels = collections.OrderedDict()
    cur = None
    for line in txt.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            cur = kernels.setdefault(m.group(1), collections.Counter())
            continue
        if cur is None:
            continue
        m = re.match(r"\s*/\*[0-9a-f]{4,}\*/\s+(?:@!?U?P\d+\s+)?([A-Z0-9_]+)", line)
        if m:
            op = m.group(1)
            cur["total"] += 1
            for o in OPS:
                if op == o or op.startswith(o + ".") or op.startswith(o):
                    cur[o] += 1
                    break
    demangle = subprocess.run(["c++filt"], input="\n".join(kernels), capture_output=True, text=True).stdout.splitlines()
    print(f"# {os.path.relpath(LIB, ROOT)}: SASS opcode counts per kernel (cuobjdump -sass, sm_90a)")
    print("# " + " ".join(f"{o:>8}" for o in ["total"] + OPS) + "  kernel")
    for (name, c), dn in zip(kernels.items(), demangle):
        short = re.sub(r"\(.*", "", dn)
        print("  " + " ".join(f"{c.get(o, 0):>8}" for o in ["total"] + OPS) + "  " + short)


if __name__ == "__main__":
    sys.exit(main())
