"""A/B of two builds of the library on bench.py's one-GPU workload (the Llama-3-8B NVFP4 calibration step).

Runs ``bench.py --steps 10 --warmup 3 --llama-ptq 0 --no-cpu-baseline`` alternately against the two library files,
``--rounds`` rounds (the order of the two flips every round), by swapping ``model_optimizer_b200/lib/libb200quant.so``
between subprocesses; the file that was there is restored at the end.  The first round of each build also passes
``--dump-outputs`` (written after the timed steps, into a temporary directory), and the two dumps are compared bit
for bit.  Prints one JSON line: per build the median and range of ``value``, ``breakdown.fake_quant_ms`` and
``roofline.frac`` and the median SM clock bench.py sampled; whether the outputs are bit-identical; and the card's
name, power limit and maximum SM clock, read in the same run.

usage: python tools/fused_ab.py --base BASE.so [--new NEW.so] [--rounds 5]
       (--new defaults to the library in the tree)"""

from __future__ import annotations

import argparse
import hashlib
import json
import os
import shutil
import statistics
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "model_optimizer_b200", "lib", "libb200quant.so")
BENCH = [sys.executable, os.path.join(ROOT, "bench.py"), "--gpus", "1", "--steps", "10", "--warmup", "3",
         "--llama-ptq", "0", "--no-cpu-baseline"]


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader",
                            "-i", os.environ.get("CUDA_VISIBLE_DEVICES", "0").split(",")[0]],
                           capture_output=True, text=True, timeout=30).stdout.strip()
        name, power, clock = (s.strip() for s in q.split(","))
        return {"name": name, "power_limit": power, "sm_clock_max": clock}
    except Exception as e:  # noqa: BLE001
        return {"error": repr(e)[:200]}


def sha256(path):
    with open(path, "rb") as f:
        return hashlib.sha256(f.read()).hexdigest()[:16]


def install(lib):
    tmp = LIB + ".ab.tmp"                    # copy aside, then rename: the subprocess never sees a partial file
    shutil.copyfile(lib, tmp)
    os.replace(tmp, LIB)


def run_bench(extra):
    r = subprocess.run(BENCH + extra, cwd=ROOT, capture_output=True, text=True)
    lines = [ln for ln in r.stdout.splitlines() if ln.startswith("{")]
    if r.returncode != 0 or not lines:
        raise RuntimeError(f"bench.py failed ({r.returncode}):\n{r.stdout[-2000:]}\n{r.stderr[-3000:]}")
    return json.loads(lines[-1])


def spread(xs):
    return {"median": statistics.median(xs), "min": min(xs), "max": max(xs)}


def same_dumps(a, b):
    """(bit-identical, files that differ or exist on one side only) of two --dump-outputs directories"""
    import numpy as np

    fa, fb = set(os.listdir(a)), set(os.listdir(b))
    bad = sorted(fa ^ fb)
    for f in sorted(fa & fb):
        x, y = np.load(os.path.join(a, f)), np.load(os.path.join(b, f))
        if x.shape != y.shape or x.dtype != y.dtype or not np.array_equal(x.view(np.uint8), y.view(np.uint8)):
            bad.append(f)
    return not bad and bool(fa), bad


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--base", required=True, help="library file of the base build")
    ap.add_argument("--new", default=None, help="library file of the new build (default: the one in the tree)")
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    if args.rounds < 5:
        ap.error("--rounds must be at least 5")

    with tempfile.TemporaryDirectory() as tmp:
        saved = os.path.join(tmp, "saved.so")
        shutil.copyfile(LIB, saved)
        libs = {"base": os.path.abspath(args.base), "new": os.path.abspath(args.new) if args.new else saved}
        shas = {k: sha256(v) for k, v in libs.items()}
        runs = {k: [] for k in libs}
        dumps = {k: os.path.join(tmp, "dump_" + k) for k in libs}
        info = card()
        try:
            for r in range(args.rounds):
                for k in (("base", "new") if r % 2 == 0 else ("new", "base")):
                    install(libs[k])
                    runs[k].append(run_bench(["--dump-outputs", dumps[k]] if r == 0 else []))
                    print(f"round {r} {k}: {runs[k][-1]['value']}", file=sys.stderr, flush=True)
        finally:
            install(saved)
        identical, differing = same_dumps(dumps["base"], dumps["new"])

    builds = {}
    for k, rs in runs.items():
        clocks = [x["clocks"]["sm_mhz"] for x in rs if (x.get("clocks") or {}).get("sm_mhz")]
        builds[k] = {"lib_sha256": shas[k],
                     "value": spread([x["value"] for x in rs]),
                     "fake_quant_ms": spread([x["breakdown"]["fake_quant_ms"] for x in rs]),
                     "roofline_frac": spread([x["roofline"]["frac"] for x in rs]),
                     "sm_mhz_median": statistics.median(clocks) if clocks else None,
                     "values": [x["value"] for x in rs]}
    b, n = builds["base"]["value"], builds["new"]["value"]
    print(json.dumps({
        "tool": "fused_ab", "bench": " ".join(BENCH[1:]).replace(ROOT + os.sep, ""), "rounds": args.rounds,
        "card": info, "builds": builds,
        "value_gain": round(n["median"] / b["median"] - 1.0, 4),
        "ranges_overlap": n["min"] <= b["max"] and b["min"] <= n["max"],
        "outputs_bit_identical": identical, "outputs_differing": differing}), flush=True)


if __name__ == "__main__":
    main()
