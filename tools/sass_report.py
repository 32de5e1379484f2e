"""SASS evidence (no GPU needed): per-kernel opcode histogram of model_optimizer_b200/lib/libb200quant.so from
`cuobjdump -sass`, written to profiles/.  The .so is git-ignored; this text is what the repo carries to show the
instruction mix (LDG.E.128 / STG.E.128, F2FP e4m3 converts, UBLKCP bulk copies, REDUX, RED/ATOMS).

usage: python tools/sass_report.py [out.txt]"""
import collections
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "model_optimizer_b200", "lib", "libb200quant.so")
KEY = ("LDG", "STG", "LDS", "STS", "ATOMS", "ATOMG", "RED", "REDG", "REDUX", "F2FP", "UBLKCP", "SYNCS", "FENCE", "MUFU",
       "HMMA", "UTCMMA", "SHFL", "VIMNMX", "FMNMX", "FFMA", "FMUL", "FADD", "I2F", "F2I", "BAR", "CALL")


def main():
    out = sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "profiles", "r02_sass_excerpt.txt")
    txt = subprocess.run(["cuobjdump", "-sass", LIB], capture_output=True, text=True, check=True).stdout
    demangle = {}
    kernels = collections.OrderedDict()
    cur = None
    for line in txt.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            cur = m.group(1)
            kernels[cur] = collections.Counter()
            continue
        m = re.match(r"\s+/\*[0-9a-f]{4,}\*/\s+(?:@!?U?P\d+\s+)?([A-Z0-9_]+(?:\.[A-Z0-9_.]+)?)", line)
        if m and cur:
            kernels[cur][m.group(1)] += 1
    names = list(kernels)
    dm = subprocess.run(["c++filt", "-p"], input="\n".join(names), capture_output=True, text=True).stdout.splitlines()
    demangle = dict(zip(names, dm)) if len(dm) == len(names) else {n: n for n in names}
    total = collections.Counter()
    lines = [f"# cuobjdump -sass {os.path.relpath(LIB, ROOT)}  ({len(kernels)} sm_90a kernels)",
             "# per kernel: instruction count, then the memory / convert / reduction opcodes that characterise it", ""]
    for k, c in kernels.items():
        n = sum(c.values())
        pick = {op: v for op, v in c.items() if op.split(".")[0] in KEY and (op.split(".")[0] not in ("FFMA", "FMUL", "FADD") )}
        for op, v in c.items():
            total[op] += v
        top = ", ".join(f"{op} x{v}" for op, v in sorted(pick.items(), key=lambda kv: (-kv[1], kv[0]))[:14])
        lines.append(f"{demangle[k][:150]}\n    {n} instr | {top}")
    lines += ["", "# library-wide totals of the opcodes that identify the design"]
    for pat in ("LDG.E.NA.ENL2.256", "LDG.E.ENL2.256", "STG.E.ENL2.256", "LDG.E.NA.128", "UBLKCP", "SYNCS", "FENCE.VIEW.ASYNC",
                "F2FP", "REDUX", "ATOMS", "RED", "HMMA", "UTCMMA", "MUFU.RCP"):
        v = sum(c for op, c in total.items() if op.startswith(pat))
        lines.append(f"{pat:22s} {v}")
    os.makedirs(os.path.dirname(out), exist_ok=True)
    with open(out, "w") as f:
        f.write("\n".join(lines) + "\n")
    print("wrote", out, len(kernels), "kernels")


if __name__ == "__main__":
    main()
