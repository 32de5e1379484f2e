"""SASS evidence (no GPU needed): per-kernel opcode histogram of model_optimizer_b200/lib/libb200quant.so from
`cuobjdump -sass`, with each kernel's registers and spills from `cuobjdump -res-usage`, written to profiles/.  The .so
is git-ignored; this text is what the repo carries to show the instruction mix (LDG.E.128 / STG.E.128, F2FP e4m3
converts, UBLKCP bulk copies, REDUX, RED/ATOMS) and the control flow left in a kernel (FSETP / FSEL / BRA / BSSY).

usage: python tools/sass_report.py [out.txt] [--lib PATH] [--kernel REGEX]"""
import argparse
import collections
import os
import re
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "model_optimizer_b200", "lib", "libb200quant.so")
KEY = ("LDG", "STG", "LDS", "STS", "ATOMS", "ATOMG", "RED", "REDG", "REDUX", "F2FP", "UBLKCP", "SYNCS", "FENCE", "MUFU",
       "HMMA", "UTCMMA", "SHFL", "VIMNMX", "FMNMX", "FFMA", "FMUL", "FADD", "I2F", "F2I", "BAR", "CALL")
CONTROL = ("FSETP", "FSEL", "BRA", "BSSY")      # always listed: the compare / select / branch count of a kernel


def res_usage(lib):
    """mangled kernel name -> (registers, local-memory bytes)"""
    txt = subprocess.run(["cuobjdump", "-res-usage", lib], capture_output=True, text=True, check=True).stdout
    out, cur = {}, None
    for line in txt.splitlines():
        m = re.match(r"\s*Function (\S+):", line)
        if m:
            cur = m.group(1)
            continue
        m = re.search(r"REG:(\d+).*LOCAL:(\d+)", line)
        if m and cur:
            out[cur] = (int(m.group(1)), int(m.group(2)))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out", nargs="?", default=os.path.join(ROOT, "profiles", "r02_sass_excerpt.txt"))
    ap.add_argument("--lib", default=LIB)
    ap.add_argument("--kernel", default=None, help="only kernels whose demangled name matches this regex")
    args = ap.parse_args()
    txt = subprocess.run(["cuobjdump", "-sass", args.lib], capture_output=True, text=True, check=True).stdout
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
    if args.kernel:
        kernels = collections.OrderedDict((k, c) for k, c in kernels.items() if re.search(args.kernel, demangle[k]))
    regs = res_usage(args.lib)
    total = collections.Counter()
    lines = [f"# cuobjdump -sass {os.path.relpath(args.lib, ROOT)}  ({len(kernels)} sm_90a kernels)",
             "# per kernel: instruction count, registers, local memory (spills), then the memory / convert / reduction /",
             "# control-flow opcodes that characterise it", ""]
    for k, c in kernels.items():
        n = sum(c.values())
        base = collections.Counter()
        for op, v in c.items():
            total[op] += v
            base[op.split(".")[0]] += v
        pick = {op: v for op, v in c.items() if op.split(".")[0] in KEY and op.split(".")[0] not in ("FFMA", "FMUL", "FADD")}
        top = ", ".join(f"{op} x{v}" for op, v in sorted(pick.items(), key=lambda kv: (-kv[1], kv[0]))[:14])
        ctl = ", ".join(f"{op} x{base[op]}" for op in CONTROL)
        reg, local = regs.get(k, (None, None))
        lines.append(f"{demangle[k][:150]}\n    {n} instr | {reg} registers, {local} B local | {ctl} | {top}")
    lines += ["", "# totals over the kernels above of the opcodes that identify the design"]
    for pat in ("LDG.E.NA.ENL2.256", "LDG.E.ENL2.256", "STG.E.ENL2.256", "LDG.E.NA.128", "UBLKCP", "SYNCS", "FENCE.VIEW.ASYNC",
                "F2FP", "REDUX", "ATOMS", "RED", "HMMA", "UTCMMA", "MUFU.RCP"):
        v = sum(c for op, c in total.items() if op.startswith(pat))
        lines.append(f"{pat:22s} {v}")
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
        f.write("\n".join(lines) + "\n")
    print("wrote", args.out, len(kernels), "kernels")


if __name__ == "__main__":
    main()
