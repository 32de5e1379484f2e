"""Kernel micro-benchmarks (GPU box): algorithmic GB/s of each hot kernel at the BASELINE tensor
(4096 x 4096 bf16) and at the down_proj activation shape, rotating through buffers larger than L2.

usage: python tools/microbench.py [--sweep] [--out gpurun_out/microbench.jsonl]
"""

from __future__ import annotations

import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from model_optimizer_b200 import _lib, ops  # noqa: E402


def peak_gbs():
    p = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(p):
        return float(json.load(open(p))["hbm_gbs"]), "measured"
    return 6650.0, "fallback"


USE_GRAPH = False


def timeit_graph(fn, bufs, reps=10):
    """GPU-side back-to-back time: capture one launch per buffer into a CUDA graph, replay."""
    n = len(bufs)
    for i in range(n):
        fn(bufs[i])
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    g = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s):
        fn(bufs[0])
        torch.cuda.synchronize()
        with torch.cuda.graph(g, stream=s):
            for i in range(n):
                fn(bufs[i])
    g.replay()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        g.replay()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1e3 / (reps * n)


def ref_reduce_amax_axis(t):  # core_utils.py:178-180 on the reshaped clone (reduce_block_amax :64)
    return torch.maximum(torch.abs(torch.amax(t, dim=1)), torch.abs(torch.amin(t, dim=1)))


def timeit(fn, bufs, iters=200, warmup=20):
    if USE_GRAPH:
        return timeit_graph(fn, bufs)
    n = len(bufs)
    for i in range(warmup):
        fn(bufs[i % n])
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(iters):
        fn(bufs[i % n])
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1e3 / iters  # us per launch


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sweep", action="store_true")
    ap.add_argument("--out", default=os.path.join(ROOT, "gpurun_out", "microbench.jsonl"))
    ap.add_argument("--shapes", default="4096x4096,4096x14336")
    ap.add_argument("--graph", action="store_true", help="time CUDA-graph replays (no CPU launch cost)")
    ap.add_argument("--quick", action="store_true", help="few iterations (for ncu)")
    ap.add_argument("--only", default="", help="'mx': only the MX-format kernels; 'hist': only the histogram variants")
    ap.add_argument("--tma", action="store_true", help="sweep the cp.async.bulk variant of the amax kernel")
    args = ap.parse_args()
    global USE_GRAPH
    USE_GRAPH = args.graph
    if args.quick:
        global timeit
        _t = timeit
        timeit = lambda fn, bufs, iters=6, warmup=2: _t(fn, bufs, iters, warmup)  # noqa: E731
    os.makedirs(os.path.dirname(args.out), exist_ok=True)
    peak, peak_kind = peak_gbs()
    results = []
    dev = torch.device("cuda:0")

    def record(name, shape, us, bytes_per_launch, **kw):
        gbs = bytes_per_launch / us / 1e3
        r = {"kernel": name, "shape": shape, "us": round(us, 3), "GBps": round(gbs, 1),
             "frac_of_peak": round(gbs / peak, 4), "peak": peak, "peak_kind": peak_kind, **kw}
        results.append(r)
        print(json.dumps(r), flush=True)

    for shp in args.shapes.split(","):
        r, c = (int(v) for v in shp.split("x"))
        n = r * c
        nbuf = max(4, int((768 << 20) / (n * 2)))  # >= 768 MiB of distinct inputs (L2 is 50 MB)
        xs = [torch.randn(r, c, device=dev).to(torch.bfloat16) for _ in range(nbuf)]
        ys = [torch.empty_like(xs[0]) for _ in range(min(nbuf, 8))]
        slot = torch.zeros(1, dtype=torch.float32, device=dev)
        ops.amax_per_tensor_(slot, xs[0])
        amax_bf = ops.amax_export(slot, torch.bfloat16)
        rows = torch.zeros(r, dtype=torch.float32, device=dev)
        cols = torch.zeros(c, dtype=torch.float32, device=dev)
        blk = torch.zeros(n // 16, dtype=torch.float32, device=dev)
        ops.amax_rows_(rows, xs[0], c)
        ops.amax_rows_(blk, xs[0], 16)
        packed = torch.empty(n // 2, dtype=torch.uint8, device=dev)

        def sweep(key, values, fn, name, nbytes):
            for v in values:
                _lib.set_tuning(key, v)
                us = timeit(fn, list(range(nbuf)))
                record(name, shp, us, nbytes, **{key: v})
            _lib.set_tuning(key, 0)

        cnt = [0]

        def yb():
            cnt[0] += 1
            return ys[cnt[0] % len(ys)]

        k_amax = lambda i: ops.amax_per_tensor_(slot, xs[i])
        k_rows = lambda i: ops.amax_rows_(rows, xs[i], c)
        k_cols = lambda i: ops.amax_cols_(cols, xs[i])
        k_blk = lambda i: ops.amax_rows_(blk, xs[i], 16)
        k_int8 = lambda i: ops.fake_quant_int(xs[i], slot, 8, False, False, out=yb())
        k_int8r = lambda i: ops.fake_quant_int(xs[i], rows, 8, False, False, outer=c, out=yb())
        k_int4b = lambda i: ops.fake_quant_int(xs[i], blk[: n // 128], 4, False, False, outer=128, out=yb())
        k_fp8 = lambda i: ops.fake_quant_fp8(xs[i], slot, out=yb())
        k_fp4 = lambda i: ops.fake_quant_nvfp4(xs[i], slot, out=yb())
        k_fp4s = lambda i: ops.fake_quant_nvfp4_static(xs[i], blk, slot, True, 448.0, out=yb())
        k_copy = lambda i: yb().copy_(xs[i])

        idx = list(range(nbuf))

        def mx_section():
            q8 = torch.empty(n, dtype=torch.uint8, device=dev)
            q8, s8 = ops.pack_mxfp8(xs[0])
            q4, s4 = ops.pack_mxfp4(xs[0], 32)
            for name in ("E4M3", "E2M1", "E3M2", "INT8", "E5M2", "E3M0"):
                record(f"fake_quant_mx_{name}_b32", shp, timeit(lambda i: ops.fake_quant_mx(xs[i], 32, name, out=yb()), idx), 4 * n)
            record("fake_quant_mx_E4M3_b16", shp, timeit(lambda i: ops.fake_quant_mx(xs[i], 16, "E4M3", out=yb()), idx), 4 * n)
            record("pack_mxfp8", shp, timeit(lambda i: ops.pack_mxfp8(xs[i]), idx), int(n * (2 + 1 + 1 / 32)))
            record("pack_mxfp4", shp, timeit(lambda i: ops.pack_mxfp4(xs[i], 32), idx), int(n * (2 + 0.5 + 1 / 32)))
            record("unpack_mxfp8", shp, timeit(lambda i: ops.unpack_mxfp8(q8, s8, torch.bfloat16), idx), int(n * (2 + 1 + 1 / 32)))
            record("unpack_mxfp4", shp, timeit(lambda i: ops.unpack_mxfp4(q4, s4, 32, torch.bfloat16), idx), int(n * (2 + 0.5 + 1 / 32)))
            qn, sn = ops.pack_nf4(xs[0], 64)
            record("pack_nf4_b64", shp, timeit(lambda i: ops.pack_nf4(xs[i], 64), idx), int(n * (2 + 0.5 + 2 / 64)))
            record("unpack_nf4_b64", shp, timeit(lambda i: ops.unpack_nf4(qn, sn, 64), idx), int(n * (2 + 0.5 + 2 / 64)))
            mxs = torch.full((c,), float("-inf"), dtype=torch.float32, device=dev)
            mns = torch.full((c,), float("inf"), dtype=torch.float32, device=dev)
            sms = torch.zeros(c, dtype=torch.float32, device=dev)
            record("bias_reduce_keep_cols(max+min+sum)", shp,
                   timeit(lambda i: ops.reduce_keep_(xs[i], 1, 1, r, c, mxs, mns, sms), idx), 2 * n)
            record("bias_reduce_keep_[8,H=8,T,C=128]", shp,
                   timeit(lambda i: ops.reduce_keep_(xs[i], 8, 8, n // (8 * 8 * 128), 128, mxs[:1024], mns[:1024], sms[:1024]), idx), 2 * n)

        def hist_section():
            hist = torch.zeros(2048, dtype=torch.float32, device=dev)
            record("histogram_2048", shp, timeit(lambda i: ops.histogram_(hist, xs[i], slot), idx), 2 * n)
            hscratch = ops.hist_scratch(dev)
            record("histogram_2048_patterns", shp, timeit(lambda i: ops.histogram_(hist, xs[i], slot, scratch=hscratch), idx), 2 * n)
            _lib.set_tuning("hist_hot", 2)
            record("histogram_2048_patterns_table", shp, timeit(lambda i: ops.histogram_(hist, xs[i], slot, scratch=hscratch), idx), 2 * n)
            _lib.set_tuning("hist_hot", 0)
            _lib.set_tuning("hist_variant", 1)
            record("histogram_2048_lane_private", shp, timeit(lambda i: ops.histogram_(hist, xs[i], slot), idx), 2 * n)
            _lib.set_tuning("hist_variant", 2)
            for cps in (1, 3, 4):
                _lib.set_tuning("hist_ctas_per_sm", cps)
                record(f"histogram_2048_ctas{cps}", shp, timeit(lambda i: ops.histogram_(hist, xs[i], slot), idx), 2 * n)
            _lib.set_tuning("hist_ctas_per_sm", 0)
            _lib.set_tuning("hist_variant", 0)

        if args.only == "hist":
            hist_section()
            del xs, ys
            continue
        if args.only == "mx":
            mx_section()
            del xs, ys
            continue
        record("torch_copy(ref)", shp, timeit(k_copy, idx), 4 * n)
        record("torch_amax(ref)", shp, timeit(lambda i: torch.amax(xs[i].abs() if False else xs[i]), idx), 2 * n)
        # the reference's calibration collect is pure ATen on every device: restated op for op
        def ref_reduce_amax(t):  # quantization/utils/core_utils.py:172-174
            return torch.maximum(torch.abs(torch.max(t)), torch.abs(torch.min(t)))

        state = {"amax": None}

        def ref_max_collect(i):  # quantization/calib/max.py:53-86 (three host-syncing asserts included)
            local = ref_reduce_amax(xs[i])
            assert not torch.any(torch.isnan(local))
            assert torch.all(local >= 0)
            assert not torch.any(torch.isinf(local))
            state["amax"] = local if state["amax"] is None else torch.max(state["amax"], local)

        record("ref_aten_reduce_amax", shp, timeit(lambda i: ref_reduce_amax(xs[i]), idx), 2 * n)
        if not USE_GRAPH:
            record("ref_aten_MaxCalibrator.collect", shp, timeit(ref_max_collect, idx), 2 * n)
        def ref_fp8_eager(t, amax):  # quantization/tensor_quant.py:46-59 (the reference's non-extension path)
            a = amax.to(torch.float32)
            safe = torch.where(a <= 1.0 / (1 << 24), torch.ones_like(a), a)
            scale = 448.0 / safe
            q = (t.to(torch.float32) * scale).clamp(min=-448.0, max=448.0).to(torch.float8_e4m3fn)
            return (q.to(torch.float32) * (1 / scale)).to(t.dtype)

        def ref_tensor_quant(t, amax):  # quantization/tensor_quant.py:607-645, 8 bit
            a = amax.float()
            scale = 127.0 / a
            return (torch.clamp((t.float() * scale).round_(), -128, 127) / scale).to(t.dtype)

        record("ref_aten_fp8_eager", shp, timeit(lambda i: ref_fp8_eager(xs[i], slot), idx), 4 * n)
        record("ref_aten_tensor_quant_int8", shp, timeit(lambda i: ref_tensor_quant(xs[i], slot), idx), 4 * n)
        record("ref_aten_block_amax16", shp, timeit(lambda i: ref_reduce_amax_axis(xs[i].clone().reshape(-1, 16)), idx), 2 * n)
        record("amax_per_tensor", shp, timeit(k_amax, idx), 2 * n)
        record("amax_rows", shp, timeit(k_rows, idx), 2 * n)
        record("amax_cols", shp, timeit(k_cols, idx), 2 * n)
        record("amax_block16", shp, timeit(k_blk, idx), 2 * n)
        record("fake_quant_int8_tensor", shp, timeit(k_int8, idx), 4 * n)
        record("fake_quant_int8_rows", shp, timeit(k_int8r, idx), 4 * n)
        record("fake_quant_int4_block128", shp, timeit(k_int4b, idx), 4 * n)
        record("fake_quant_fp8_tensor", shp, timeit(k_fp8, idx), 4 * n)
        record("fake_quant_nvfp4_dynamic", shp, timeit(k_fp4, idx), 4 * n)
        record("fake_quant_nvfp4_static", shp, timeit(k_fp4s, idx), 4 * n)
        _lib.set_tuning("nvfp4_tma_store", 1)
        record("fake_quant_nvfp4_dynamic_tma_store", shp, timeit(k_fp4, idx), 4 * n)
        _lib.set_tuning("nvfp4_tma_store", 2)
        xs16 = xs[:16]
        t_amax = ops.TensorTable(xs16, unit="vec32")
        ys16 = [torch.empty_like(xs[0]) for _ in range(16)]
        t_fq = ops.TensorTable(xs16, None, ys16, "block16")
        slots16 = torch.zeros(16, dtype=torch.float32, device=dev)
        amax16 = amax_bf.reshape(1).repeat(16).contiguous()
        record("amax_per_tensor_grouped16", shp, timeit(lambda i: ops.amax_per_tensor_multi_(slots16, t_amax), [0, 1, 2, 3]) / 16, 2 * n)
        record("fake_quant_nvfp4_grouped16", shp, timeit(lambda i: ops.fake_quant_nvfp4_multi(t_fq, amax16), [0, 1, 2, 3]) / 16, 4 * n)
        del ys16
        record("pack_int4_block128", shp, timeit(lambda i: ops.pack_int4_blockwise(xs[i], 128), idx), int(n * (2 + 0.5 + 2 / 128)))
        record("pack_fp8_tensor", shp, timeit(lambda i: ops.pack_fp8(xs[i], amax_bf), idx), 3 * n)
        hist_section()
        try:
            g = slot
            record("pack_nvfp4", shp, timeit(lambda i: ops.pack_nvfp4(xs[i], g), idx), int(n * (2 + 0.5 + 1 / 16)))
            _lib.set_tuning("pack_unroll", 1)
            record("pack_nvfp4_unroll1", shp, timeit(lambda i: ops.pack_nvfp4(xs[i], g), idx), int(n * (2 + 0.5 + 1 / 16)))
            _lib.set_tuning("pack_unroll", 0)
        except Exception as e:  # noqa: BLE001
            print("pack_nvfp4 failed:", e)

        mx_section()
        if args.tma:
            for cps in (1, 2, 3):
                for stages in (2, 4, 8):
                    for kb in (8, 16, 32):
                        if stages * kb * cps > 200:
                            continue
                        _lib.set_tuning("amax_tma", 1)
                        _lib.set_tuning("tma_ctas_per_sm", cps)
                        _lib.set_tuning("tma_stages", stages)
                        _lib.set_tuning("tma_tile_kb", kb)
                        record("amax_per_tensor_tma", shp, timeit(k_amax, idx), 2 * n, ctas_per_sm=cps, stages=stages, tile_kb=kb)
            _lib.set_tuning("amax_tma", 2)
            record("amax_per_tensor_ldg", shp, timeit(k_amax, idx), 2 * n)
        if args.sweep:
            sweep("amax_unroll", [1, 2, 4, 8], k_amax, "amax_per_tensor", 2 * n)
            _lib.set_tuning("vec_bytes", 16)
            sweep("amax_unroll", [2, 4, 8], k_amax, "amax_per_tensor_v16", 2 * n)
            _lib.set_tuning("vec_bytes", 0)
            for cps in (1, 2, 4, 8):
                _lib.set_tuning("amax_ctas_per_sm", cps)
                sweep("amax_unroll", [2, 4, 8], k_amax, f"amax_per_tensor_persist{cps}", 2 * n)
            _lib.set_tuning("amax_ctas_per_sm", 0)
            sweep("ew_unroll", [1, 2, 4], k_fp8, "fake_quant_fp8_tensor", 4 * n)
            sweep("ew_unroll", [1, 2, 4], k_int8, "fake_quant_int8_tensor", 4 * n)
            sweep("nvfp4_unroll", [1, 2, 4], k_fp4, "fake_quant_nvfp4_dynamic", 4 * n)
            _lib.set_tuning("vec_bytes", 16)
            sweep("ew_unroll", [1, 2, 4], k_fp8, "fake_quant_fp8_tensor_v16", 4 * n)
            sweep("nvfp4_unroll", [1, 2, 4], k_fp4, "fake_quant_nvfp4_dynamic_v16", 4 * n)
            _lib.set_tuning("vec_bytes", 0)
        del xs, ys

    with open(args.out, "w") as f:
        for r in results:
            f.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
