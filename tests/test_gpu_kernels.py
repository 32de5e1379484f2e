"""GPU parity: every CUDA kernel, called through the C-ABI (model_optimizer_b200.ops -> ctypes ->
libb200quant.so), against the CPU oracle and the committed reference fixtures.

Bar: bit-exact (integer / byte / index work and fake-quant values); amax exact.
"""

import os

import numpy as np
import pytest
import torch

from oracle import oracle_np as o

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

TD = {"bf16": torch.bfloat16, "f16": torch.float16, "f32": torch.float32}


@pytest.fixture(scope="module")
def ops():
    from model_optimizer_b200 import ops as _ops

    return _ops


def dev(x, d):
    return torch.from_numpy(np.ascontiguousarray(x, dtype=np.float32)).to("cuda").to(TD[d])


def host(t):
    return t.detach().float().cpu().numpy()


def rnd(shape, d, seed, scale=1.0, heavy=False):
    g = np.random.default_rng(seed)
    x = g.standard_normal(shape).astype(np.float32) * np.float32(scale)
    if heavy:
        x = x * (1 + 20 * (g.random(shape) < 1e-3)).astype(np.float32)
    return o.round_to(x, d)


def same(a, b, what=""):
    a = np.ascontiguousarray(a)
    b = np.ascontiguousarray(b)
    assert a.shape == b.shape, (what, a.shape, b.shape)
    if a.dtype.kind == "f":
        a = a.astype(np.float32)
        b = b.astype(np.float32)
        ok = (a.view(np.uint32) == b.view(np.uint32)) | (np.isnan(a) & np.isnan(b))
    else:
        ok = a == b
    nbad = int(np.sum(~ok))
    if nbad:
        i = np.argwhere(~ok)[0]
        raise AssertionError(f"{what}: {nbad}/{a.size} mismatches, first at {tuple(i)}: got {a[tuple(i)]!r} want {b[tuple(i)]!r}")


def cases(golden):
    return [str(c) for c in golden["cases"]]


def zslots(n):
    return torch.zeros(n, dtype=torch.float32, device="cuda")


# ------------------------------------------------------------------------------------------------
def test_library_loads_and_is_hopper(ops):
    from model_optimizer_b200 import _lib

    sm, major, minor = _lib.device_info()     # the library is built for sm_90a only
    assert sm > 0 and (major, minor) == (9, 0), (sm, major, minor)


def test_exact_division_selftest(ops):
    for seed in (1, 2, 3):
        assert ops.selftest_fastdiv(seed, 1 << 24) == 0


# ---- collect -----------------------------------------------------------------------------------
def test_amax_golden(ops, golden):
    for k in cases(golden):
        d = k.split("_")[0]
        x = golden[f"{k}/x"]
        xt = dev(x, d)
        s = zslots(1)
        ops.amax_per_tensor_(s, xt)
        same(host(s)[0], golden[f"{k}/amax_tensor"], f"{k} tensor")
        r = zslots(x.shape[0])
        ops.amax_rows_(r, xt, x.shape[1])
        same(host(r), golden[f"{k}/amax_rows"].ravel(), f"{k} rows")
        c = zslots(x.shape[1])
        ops.amax_cols_(c, xt)
        same(host(c), golden[f"{k}/amax_cols"].ravel(), f"{k} cols")
        for blk in (16, 128):
            b = zslots(x.size // blk)
            ops.amax_rows_(b, xt, blk)
            same(host(b), golden[f"{k}/amax_block{blk}"].ravel(), f"{k} block{blk}")


@pytest.mark.parametrize("d", ["bf16", "f16", "f32"])
def test_amax_running_max_and_shapes(ops, d):
    # running max over batches == MaxCalibrator; ragged sizes, unaligned views
    for n, off in ((1, 0), (7, 0), (4099, 1), (1 << 20, 0), ((1 << 20) + 13, 3), (4096 * 1024, 0)):
        x1 = rnd((n + off,), d, n)[off:]
        x2 = rnd((n + off,), d, n + 1, scale=0.5)[off:]
        s = zslots(1)
        t1 = dev(rnd((n + off,), d, n), d)[off:]
        t2 = dev(rnd((n + off,), d, n + 1, scale=0.5), d)[off:]
        ops.amax_per_tensor_(s, t1)
        ops.amax_per_tensor_(s, t2)
        cal = o.MaxCalibrator(None)
        cal.collect(x1)
        cal.collect(x2)
        same(host(s)[0], cal.compute_amax(), f"n={n} off={off}")


def test_amax_rows_channel_fold_and_odd_rows(ops):
    d = "bf16"
    x = rnd((6, 10, 72), d, 5)  # rows of 72 (not a multiple of 16 elements), fold 6 leading dims
    xt = dev(x, d)
    s = zslots(10)
    ops.amax_rows_(s, xt, 72)  # row r -> channel r % 10
    same(host(s), o.reduce_amax(x, axis=(0, 2)).ravel(), "fold")
    x = rnd((33, 13), d, 6)  # scalar fallback
    s = zslots(33)
    ops.amax_rows_(s, dev(x, d), 13)
    same(host(s), o.reduce_amax(x, axis=1).ravel(), "odd rows")
    x = rnd((1000, 4096), d, 7)
    s = zslots(1000)
    ops.amax_rows_(s, dev(x, d), 4096)
    same(host(s), o.reduce_amax(x, axis=1).ravel(), "long rows")


def test_amax_cols_shapes(ops):
    for d in ("bf16", "f32"):
        for shape in ((1, 8), (1000, 264), (257, 4096), (5, 13)):
            x = rnd(shape, d, shape[0])
            s = zslots(shape[1])
            ops.amax_cols_(s, dev(x, d))
            same(host(s), o.reduce_amax(x, axis=0).ravel(), f"{d} {shape}")


def test_abssum_cols(ops):
    x = rnd((513, 1024), "bf16", 3)
    s = zslots(1024)
    ops.abssum_cols_(s, dev(x, "bf16"))
    ref = np.abs(x.astype(np.float64)).sum(0)
    assert np.allclose(host(s), ref, rtol=1e-5)


def test_amax_nan_propagates(ops):
    x = rnd((4096,), "bf16", 1)
    x[77] = np.nan
    s = zslots(1)
    ops.amax_per_tensor_(s, dev(x, "bf16"))
    assert np.isnan(host(s)[0])


def test_amax_export(ops):
    s = torch.tensor([0.0, 1.0, 3.14159, 65504.0], device="cuda")
    same(host(ops.amax_export(s, torch.bfloat16)), o.round_bf16(host(s)))
    same(host(ops.amax_export(s, torch.float16)), o.round_f16(host(s)))


# ---- integer fake quant ------------------------------------------------------------------------
@pytest.mark.parametrize("bits,narrow", [(8, False), (8, True), (4, False), (3, True), (11, False)])
def test_int_fake_quant_golden(ops, golden, bits, narrow):
    for k in cases(golden):
        d = k.split("_")[0]
        x = golden[f"{k}/x"]
        amax = o.reduce_amax(x)
        got = host(ops.fake_quant_int(dev(x, d), dev(amax, d), bits, False, narrow))
        same(got, o.fake_quant_int(x, amax, bits, False, narrow, 1, d), f"{k} oracle")
        key = f"{k}/int{bits}_n{int(narrow)}_tensor"
        if key in golden and amax > 2.0**-24:
            same(got, golden[key], f"{k} reference fixture")


def test_int_fake_quant_axis_and_blocks(ops, golden):
    for k in cases(golden):
        d = k.split("_")[0]
        x = golden[f"{k}/x"]
        xt = dev(x, d)
        ar = o.reduce_amax(x, axis=1)
        got = host(ops.fake_quant_int(xt, dev(ar, d), 8, False, False, outer=x.shape[1]))
        same(got, o.fake_quant_int(x, ar, 8, False, False, x.shape[1], d), f"{k} rows")
        if "sparse" not in k:
            same(got, golden[f"{k}/int8_rows"], f"{k} rows fixture")
        xb = x.reshape(-1, 128)
        ab = o.reduce_amax(xb, axis=1)
        got = host(ops.fake_quant_int(xt, dev(ab, "f32"), 4, False, False, outer=128))
        same(got, o.fake_quant_int(xb, ab, 4, False, False, 128, d).reshape(x.shape), f"{k} block128")
        # last-axis channels (outer = 1)
        ac = o.reduce_amax(x, axis=0)
        got = host(ops.fake_quant_int(xt, dev(ac, "f32"), 8, False, True, outer=1))
        same(got, o.fake_quant_int(x, ac, 8, False, True, 1, d), f"{k} cols")


def test_int_fake_quant_inplace_unsigned_tiny_unaligned(ops):
    d = "bf16"
    x = rnd((3, 1000), d, 11)
    amax = o.reduce_amax(x)
    xt = dev(x, d)
    ops.fake_quant_int(xt, dev(amax, "f32"), 8, False, True, out=xt)  # fake_tensor_quant_
    same(host(xt), o.fake_quant_int(x, amax, 8, False, True, 1, d), "inplace")
    xa = np.abs(rnd((777,), d, 12))
    same(host(ops.fake_quant_int(dev(xa, d), dev(o.reduce_amax(xa), "f32"), 8, True, True)),
         o.fake_quant_int(xa, o.reduce_amax(xa), 8, True, True, 1, d), "unsigned")
    xt = np.array([[0, 1e-9], [-1e-9, 1e-9]], dtype=np.float32)
    same(host(ops.fake_quant_int(dev(xt, "f32"), dev(np.float32(1e-9), "f32"), 8, False, True)),
         np.zeros_like(xt), "tiny amax")  # test_tensor_quant_cuda.py:115-119
    big = rnd((4097 * 3 + 1,), d, 13)
    v = dev(np.concatenate([[0], big]).astype(np.float32), d)[1:]  # 2-byte offset view
    same(host(ops.fake_quant_int(v, dev(o.reduce_amax(big), "f32"), 8, False, False)),
         o.fake_quant_int(big, o.reduce_amax(big), 8, False, False, 1, d), "unaligned")


# ---- fp8 fake quant ----------------------------------------------------------------------------
def test_fp8_fake_quant(ops, golden):
    for k in cases(golden):
        d = k.split("_")[0]
        x = golden[f"{k}/x"]
        xt = dev(x, d)
        at = o.reduce_amax(x)
        same(host(ops.fake_quant_fp8(xt, dev(at, d))), o.fake_quant_fp8(x, at, 1, d), f"{k} tensor")
        ar = o.reduce_amax(x, axis=1)
        same(host(ops.fake_quant_fp8(xt, dev(ar, d), outer=x.shape[1])),
             o.fake_quant_fp8(x, ar, x.shape[1], d), f"{k} rows")
        got = host(ops.fake_quant_fp8(xt, None))
        same(got, o.fake_quant_fp8(x, None, 1, d), f"{k} noamax")
        same(got, golden[f"{k}/fp8_noamax"], f"{k} noamax fixture")


def test_fp8_saturation_and_specials(ops):
    x = np.array([0, -0.0, 1e-10, 448, 449, 465, 1e6, -1e6, np.inf, -np.inf, 2.0**-9, 2.0**-10, 3 * 2.0**-10],
                 dtype=np.float32)
    x = np.concatenate([x, np.zeros(3, np.float32)])
    amax = np.float32(448.0)
    same(host(ops.fake_quant_fp8(dev(x, "f32"), dev(amax, "f32"))), o.fake_quant_fp8(x, amax, 1, "f32"))


# ---- nvfp4 -------------------------------------------------------------------------------------
def test_nvfp4_dynamic(ops, golden):
    for k in cases(golden):
        d = k.split("_")[0]
        x = golden[f"{k}/x"]
        g = o.reduce_amax(x)
        got = host(ops.fake_quant_nvfp4(dev(x, d), dev(g, d)))
        same(got, o.fake_quant_nvfp4(x, g, d), f"{k} oracle")
        if f"{k}/nvfp4_deq" in golden and "gauss" in k:
            # equal up to the sign of zero (Triton keeps -0.0, the QTensor LUT has +0.0 for code 8)
            same(got + np.float32(0), golden[f"{k}/nvfp4_deq"] + np.float32(0), f"{k} == reference QTensor round trip")


def test_nvfp4_dynamic_boundaries_and_ragged(ops):
    # test_tensor_quant_cuda.py:236-262 boundary vectors
    base = np.array([0.25, 0.75, 1.25, 1.75, 2.5, 3.5, 5, 6], dtype=np.float32)
    for sign in (1.0, -1.0):
        x = (np.concatenate([base, base]) * np.float32(sign)).reshape(1, 16)
        got = host(ops.fake_quant_nvfp4(dev(x, "f32"), dev(np.float32(6.0), "f32")))
        same(got[0, :8] * np.float32(sign), np.array([0, 1, 1, 2, 2, 4, 4, 6], dtype=np.float32), "ties")
    for d in ("bf16", "f16", "f32"):
        for shape in ((5, 40), (3, 17), (2, 3, 24), (7, 16), (129, 4096)):
            x = rnd(shape, d, shape[-1], heavy=True)
            g = o.reduce_amax(x)
            same(host(ops.fake_quant_nvfp4(dev(x, d), dev(g, "f32"))), o.fake_quant_nvfp4(x, g, d), f"{d} {shape}")
    # calibrated amax smaller than the data (clamp to 448), zero amax, zero blocks, -0.0
    x = rnd((8, 64), "bf16", 3)
    x[0] = 0
    x[1, :16] = -0.0
    x[2] *= np.float32(1e-20)
    for g in (np.float32(0.5), np.float32(0.0), np.float32(1e-30), np.float32(3e38)):
        same(host(ops.fake_quant_nvfp4(dev(x, "bf16"), dev(g, "f32"))), o.fake_quant_nvfp4(x, g, "bf16"), f"g={g}")


def test_nvfp4_static(ops, golden):
    for k in cases(golden):
        d = k.split("_")[0]
        x = golden[f"{k}/x"]
        bam = o.reduce_block_amax(x, 16)
        g = o.reduce_amax(x)
        for quant, m in ((True, 448.0), (True, 256.0), (False, 448.0)):
            got = host(ops.fake_quant_nvfp4_static(dev(x, d), dev(bam, "f32"), dev(g, "f32"), quant, m))
            same(got, o.fake_quant_nvfp4_static(x, bam, g, quant, m, d), f"{k} q={quant} m={m}")
    # zero amax zeroes the block (test_tensor_quant_cuda.py:195-203)
    x = np.ones((1, 16), dtype=np.float32)
    got = host(ops.fake_quant_nvfp4_static(dev(x, "f32"), zslots(1), None, False))
    same(got, np.zeros_like(x))


def test_nvfp4_pack_matches_reference_fixture(ops, golden):
    n = 0
    for k in cases(golden):
        if f"{k}/nvfp4_packed" not in golden:
            continue
        n += 1
        d = k.split("_")[0]
        x = golden[f"{k}/x"]
        packed, scales, wsf2 = ops.pack_nvfp4(dev(x, d), dev(o.reduce_amax(x), "f32"))
        same(packed.cpu().numpy(), golden[f"{k}/nvfp4_packed"], f"{k} packed")
        same(scales.view(torch.uint8).cpu().numpy(), golden[f"{k}/nvfp4_scales"], f"{k} scales")
        same(host(wsf2), golden[f"{k}/nvfp4_wsf2"], f"{k} wsf2")
        deq = ops.unpack_nvfp4(packed, scales, wsf2, TD[d])
        same(host(deq), golden[f"{k}/nvfp4_deq"], f"{k} dequant")
        # static branch
        bam = o.reduce_block_amax(x, 16)
        packed, scales, wsf2 = ops.pack_nvfp4(dev(x, d), dev(o.reduce_amax(x), "f32"), dev(bam, "f32"))
        same(packed.cpu().numpy(), golden[f"{k}/nvfp4s_packed"], f"{k} static packed")
        same(scales.view(torch.uint8).cpu().numpy(), golden[f"{k}/nvfp4s_scales"], f"{k} static scales")
        same(host(wsf2), golden[f"{k}/nvfp4s_wsf2"], f"{k} static wsf2")
    assert n >= 6


def test_nvfp4_pack_large_roundtrip_properties(ops):
    # size-independent properties at a BASELINE-sized tensor: unpack(pack(x)) == fake_quant-like
    # round trip, packing is idempotent on its own output
    d = "bf16"
    x = torch.randn(4096, 4096, device="cuda", generator=torch.Generator("cuda").manual_seed(0)).to(torch.bfloat16)
    g = zslots(1)
    ops.amax_per_tensor_(g, x)
    packed, scales, wsf2 = ops.pack_nvfp4(x, g)
    deq = ops.unpack_nvfp4(packed, scales, wsf2, torch.bfloat16)
    g2 = zslots(1)
    ops.amax_per_tensor_(g2, deq)
    p2, s2, w2 = ops.pack_nvfp4(deq, g)  # same global amax: codes must not move
    # ... except "-0" codes (8): they dequantise to +0.0 (reference LUT) and re-encode as 0
    t = packed & 0x77
    canon = t | (packed & (((t + 0x77) & 0x88)))
    assert torch.equal(p2, canon) and torch.equal(s2.view(torch.uint8), scales.view(torch.uint8))
    fq = ops.fake_quant_nvfp4(x, g)
    assert (fq != deq).float().mean().item() < 1e-4


# ---- INT4 / FP8 packs, histogram ------------------------------------------------------------------
def test_int4_blockwise_pack_cuda_semantics(ops, golden):
    for k in cases(golden):
        d = k.split("_")[0]
        x = golden[f"{k}/x"]
        for bs in (128, 16, 32, 64):
            packed, scales = ops.pack_int4_blockwise(dev(x, d), bs)
            rp, rs = o.pack_int4_blockwise_cuda(x, bs, d)
            same(host(scales), rs, f"{k} bs={bs} scales")
            if "sparse" not in k:
                same(packed.cpu().numpy(), rp, f"{k} bs={bs} packed")
            deq = ops.unpack_int4_blockwise(packed, scales, bs)
            same(host(deq), o.unpack_int4_blockwise(packed.cpu().numpy(), host(scales), bs, d), f"{k} bs={bs} unpack")
        if f"{k}/int4cpu_scales" in golden:  # scales do not depend on the rounding branch
            _, scales = ops.pack_int4_blockwise(dev(x, d), 128)
            same(host(scales), golden[f"{k}/int4cpu_scales"], f"{k} scales == reference fixture")
    # reference known-answer vector (test_qtensor_cuda.py:141-150), block 4 -> generic kernel
    x8 = np.arange(8, dtype=np.float32).reshape(1, 8)
    p, s = ops.pack_int4_blockwise(dev(x8, "bf16"), 4)
    got = host(ops.unpack_int4_blockwise(p, s, 4)).reshape(1, 8)
    assert np.allclose(got, [[0.0, 0.8516, 2.1406, 2.9844, 4, 5, 6, 7]], atol=4e-3)
    rp, rs = o.pack_int4_blockwise_cuda(x8, 4, "bf16")
    same(p.cpu().numpy(), rp, "block4 packed")


def test_int4_export_pack_matches_reference_fixture(ops, golden):
    n = 0
    for k in cases(golden):
        if f"{k}/int4exp_packed" not in golden:
            continue
        n += 1
        d = k.split("_")[0]
        x = golden[f"{k}/x"]
        got = ops.pack_int4_export(dev(x, d), dev(golden[f"{k}/int4exp_scale"], "f32"))
        same(got.cpu().numpy(), golden[f"{k}/int4exp_packed"], f"{k} fp32 scale")
        got = ops.pack_int4_export(dev(x, d), dev(golden[f"{k}/int4exp_scale_same"], d))
        same(got.cpu().numpy(), golden[f"{k}/int4exp_packed_same"], f"{k} same-dtype scale")
    assert n >= 5


def test_fp8_pack_matches_reference_fixture(ops, golden):
    n = 0
    for k in cases(golden):
        if f"{k}/fp8pack_tensor" not in golden:
            continue
        n += 1
        d = k.split("_")[0]
        x = golden[f"{k}/x"]
        xt = dev(x, d)
        sc = golden[f"{k}/fp8pack_tensor_scale"]
        q = ops.pack_fp8(xt, dev(sc, d))
        same(q.view(torch.uint8).cpu().numpy(), golden[f"{k}/fp8pack_tensor"], f"{k} per-tensor")
        same(host(ops.unpack_fp8(q, dev(sc, d), TD[d])), o.unpack_fp8(golden[f"{k}/fp8pack_tensor"], sc, 1, d), f"{k} unpack")
        scr = golden[f"{k}/fp8pack_rows_scale"]
        q = ops.pack_fp8(xt, dev(scr, d), outer=x.shape[1])
        same(q.view(torch.uint8).cpu().numpy(), golden[f"{k}/fp8pack_rows"], f"{k} per-row")
        s0 = dev(golden[f"{k}/fp8pack_export_scale"], "f32")
        q = ops.pack_fp8(xt, s0.reshape(()))
        same(q.view(torch.uint8).cpu().numpy(), golden[f"{k}/fp8pack_export"], f"{k} export (0-dim fp32 scale)")
        # the same scale WITH a dim (what unified_export_hf passes): torch promotes the quotient to fp32
        q = ops.pack_fp8(xt, s0.reshape(1))
        want = o.pack_fp8(x, golden[f"{k}/fp8pack_export_scale"], 1, d, "f32", scale_is_0dim=False)
        same(q.view(torch.uint8).cpu().numpy(), want, f"{k} export ((1,) fp32 scale)")
        same(want, golden[f"{k}/fp8pack_export1"], f"{k} oracle vs reference to_quantized_weight")
    assert n >= 6


def test_histogram(ops, golden):
    for k in cases(golden):
        d = k.split("_")[0]
        x = golden[f"{k}/x"]
        for bins in (2048, 100, 5000, 30000):
            vmax = np.abs(x).max()
            h = zslots(bins)
            ops.histogram_(h, dev(x, d), dev(vmax, "f32").reshape(1))
            same(host(h), o.histc(np.abs(x), bins, vmax), f"{k} bins={bins}")
        if f"{k}/hist1" in golden:
            h = zslots(2048)
            ops.histogram_(h, dev(x, d), dev(np.abs(x).max(), "f32").reshape(1))
            diff = np.abs(host(h) - golden[f"{k}/hist1"]).sum()
            assert diff <= 8, diff  # CPU histc (fixture) vs CUDA formula: edge elements only
    # accumulation across batches + odd length / offset view
    x = rnd((100003,), "bf16", 9)
    vmax = np.float32(np.abs(x).max() * 2)
    h = zslots(2048)
    xt = dev(np.concatenate([[0], x]).astype(np.float32), "bf16")[1:]
    ops.histogram_(h, xt, dev(vmax, "f32").reshape(1))
    ops.histogram_(h, xt, dev(vmax, "f32").reshape(1))
    same(host(h), 2 * o.histc(np.abs(x), 2048, vmax), "accumulate")


def test_histogram_equals_torch_histc_on_cuda(ops):
    """HistogramCalibrator.collect on a GPU calls ATen's CUDA histc (calib/histogram.py:118,128): run THAT next to
    the fused kernel, on the reference's own op sequence x.abs().float() -> histc(bins, min=0, max=x.max())."""
    for d in ("bf16", "f16", "f32"):
        for seed, scale, bins in ((1, 1.0, 2048), (2, 37.5, 2048), (3, 1e-3, 4096), (4, 5.0, 100)):
            g = torch.Generator(device="cuda").manual_seed(seed)
            x = (torch.randn(513, 1031, device="cuda", generator=g) * scale).to(TD[d])
            xa = x.abs().float()
            vmax = xa.max()
            ref = torch.histc(xa, bins=bins, min=0, max=float(vmax))
            h = zslots(bins)
            ops.histogram_(h, x, vmax.reshape(1))
            assert torch.equal(h, ref), (d, seed, int((h != ref).sum()))


@pytest.mark.timeout(120)
def test_amax_tma_variant_matches(ops):
    """cp.async.bulk + mbarrier ring variant of the per-tensor collect == the vector-load kernel."""
    from model_optimizer_b200 import _lib

    try:
        for d in ("bf16", "f32"):
            for n, off in ((8, 0), (4099, 1), (1 << 20, 0), ((1 << 22) + 24, 8), (4096 * 4096, 0)):
                x = rnd((n + off,), d, n + 7)
                xt = dev(x, d)[off:]
                for stages, kb in ((4, 16), (2, 32), (8, 8)):
                    _lib.set_tuning("amax_tma", 1)
                    _lib.set_tuning("tma_stages", stages)
                    _lib.set_tuning("tma_tile_kb", kb)
                    s = zslots(1)
                    ops.amax_per_tensor_(s, xt)
                    same(host(s)[0], o.reduce_amax(x[off:]), f"tma {d} n={n} off={off} stages={stages} kb={kb}")
    finally:
        _lib.set_tuning("amax_tma", 2)
        _lib.set_tuning("tma_stages", 0)
        _lib.set_tuning("tma_tile_kb", 0)


_TMA_STORE_SCRIPT = r"""
import sys, torch
sys.path.insert(0, sys.argv[1])
from model_optimizer_b200 import _lib, ops
g = torch.Generator(device="cuda").manual_seed(9)
n = 0
for dt in (torch.bfloat16, torch.float16, torch.float32):
    for shape in ((512, 4096), (64, 1024), (32, 256)):
        x = (torch.randn(shape, device="cuda", generator=g) * 3).to(dt)
        amax = x.abs().max().float().reshape(1)
        _lib.set_tuning("nvfp4_tma_store", 2)       # off
        want = ops.fake_quant_nvfp4(x, amax)
        _lib.set_tuning("nvfp4_tma_store", 1)
        got = ops.fake_quant_nvfp4(x, amax)
        torch.cuda.synchronize()
        assert torch.equal(want.view(torch.uint8), got.view(torch.uint8)), (dt, shape)
        n += 1
print("tma_store_ok", n)
"""


def test_nvfp4_tma_store_variant_matches():
    """The TMA-store variant of the NVFP4 fake quant (results staged in shared memory, one cp.async.bulk
    shared -> global per CTA; opt-in knob) == the STG.E.256 kernel, bit for bit.  Runs in its own process: an
    experimental kernel must not be able to poison this process's CUDA context."""
    import subprocess
    import sys

    r = subprocess.run([sys.executable, "-c", _TMA_STORE_SCRIPT, ROOT], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and "tma_store_ok 9" in r.stdout, r.stdout[-1500:] + r.stderr[-1500:]


# ---- BASELINE-sized tensors: size-independent properties (the oracle would take minutes here) -------
@pytest.mark.parametrize("shape", [(4096, 4096), (4096, 14336)])
def test_full_size_properties(ops, shape):
    g = torch.Generator("cuda").manual_seed(shape[1])
    x = torch.randn(shape, device="cuda", generator=g).to(torch.bfloat16)
    x[17, 33] = 37.5  # a unique maximum
    # collect: exact against torch's own reduction; linear under power-of-two scaling; order independent
    s = zslots(1)
    ops.amax_per_tensor_(s, x)
    assert float(s) == float(x.abs().max()) == 37.5
    s2 = zslots(1)
    ops.amax_per_tensor_(s2, x * 4)
    assert float(s2) == 4 * float(s)
    r = zslots(shape[0])
    ops.amax_rows_(r, x, shape[1])
    assert torch.equal(r, x.abs().amax(dim=1).float())
    c = zslots(shape[1])
    ops.amax_cols_(c, x)
    assert torch.equal(c, x.abs().amax(dim=0).float())
    assert float(r.max()) == float(c.max()) == float(s)  # a maximum of maxima
    b = zslots(x.numel() // 16)
    ops.amax_rows_(b, x, 16)
    assert torch.equal(b, x.abs().reshape(-1, 16).amax(dim=1).float())
    # fake quant: idempotent for static scales (INT8, FP8), bounded by amax, sign preserving
    amax = ops.amax_export(s, torch.bfloat16)
    for fq in (lambda t: ops.fake_quant_int(t, amax, 8, False, False), lambda t: ops.fake_quant_fp8(t, amax)):
        y = fq(x)
        assert torch.equal(fq(y), y), "fake quant is not idempotent"
        assert float(y.abs().max()) <= float(amax), (float(y.abs().max()), float(amax))
        assert bool(((y == 0) | (torch.sign(y) == torch.sign(x))).all()), "sign flipped"
    # NVFP4: every output block has at most 8 distinct magnitudes, all multiples of its block scale;
    # quantising with a larger global amax never increases the number of exactly representable values
    y = ops.fake_quant_nvfp4(x, s)
    yb = y.float().abs().reshape(-1, 16)
    smin = torch.where(yb > 0, yb, torch.full_like(yb, float("inf"))).amin(dim=1, keepdim=True)
    ratio = torch.where(yb > 0, yb / smin, torch.zeros_like(yb))
    assert float(ratio.max()) <= 12.0 * (1 + 2.0**-6), float(ratio.max())  # 6 / 0.5, outputs rounded to bf16
    err = (y.float() - x.float()).abs().reshape(-1, 16).amax(dim=1)
    bmax = x.float().abs().reshape(-1, 16).amax(dim=1)
    worst = float((err / bmax.clamp_min(1e-30)).max())
    assert worst <= 0.26, worst  # <= half the widest E2M1 gap (2 of 6) plus scale rounding
    # pack -> unpack == fake quant up to the sign of zero, at full size
    packed, scales, wsf2 = ops.pack_nvfp4(x, s)
    deq = ops.unpack_nvfp4(packed, scales, wsf2, torch.bfloat16)
    mism = float((deq.float() + 0 != y.float() + 0).float().mean())
    assert mism < 1e-5, mism
    # FP8 pack round trip equals FP8 fake quant when the scale is a power of two (no scale rounding)
    p2 = torch.tensor(64.0 / 448.0, device="cuda", dtype=torch.float32)
    q = ops.pack_fp8(x, p2)
    back = ops.unpack_fp8(q, p2.to(torch.bfloat16), torch.bfloat16)
    worst = float((back.float() - x.float()).abs().max())
    assert worst <= 64.0 / 448.0 * 16 * 1.05 + 0.2, worst  # half an e4m3 step at 262 + bf16 scale rounding


def test_empty_and_single_element_tensors(ops):
    e = torch.empty(0, 16, device="cuda", dtype=torch.bfloat16)
    s = zslots(1)
    ops.amax_per_tensor_(s, e)
    assert float(s) == 0.0
    assert ops.fake_quant_fp8(e, torch.ones((), device="cuda")).shape == e.shape
    assert ops.fake_quant_nvfp4(e, torch.ones((), device="cuda")).shape == e.shape
    one = torch.tensor([-3.0], device="cuda", dtype=torch.bfloat16)
    ops.amax_per_tensor_(s, one)
    assert float(s) == 3.0
    same(host(ops.fake_quant_int(one, s, 8, False, False)), o.fake_quant_int(host(one), np.float32(3.0), 8, False, False, 1, "bf16"))
    same(host(ops.fake_quant_nvfp4(one, s)), o.fake_quant_nvfp4(host(one).reshape(1, 1), np.float32(3.0), "bf16").reshape(1))


def test_nvfp4_pack_block_sizes_32_64(ops):
    import os

    g = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_nvfp4_blocks.npz"))
    keys = sorted({k.rsplit("/x", 1)[0] for k in g.files if k.endswith("/x")})
    for k in keys:
        bs, d = int(k.split("/")[-1]), k.split("/")[1]
        x = g[k + "/x"]
        gam = dev(np.abs(x).max(), "f32").reshape(1)
        packed, scales, wsf2 = ops.pack_nvfp4(dev(x, d), gam, block_size=bs)
        same(packed.cpu().numpy(), g[k + "/packed"], k + " packed")
        same(scales.view(torch.uint8).cpu().numpy(), g[k + "/scale"], k + " scale")
        assert np.float32(wsf2.item()) == g[k + "/sf2"], k
        same(host(ops.unpack_nvfp4(packed, scales, wsf2, TD[d])), g[k + "/deq"], k + " deq")
    # static branch with per-block amax at block 32 + a 4096-wide tensor against the oracle
    x = rnd((64, 4096), "bf16", 5, heavy=True)
    for bs in (32, 128):
        bam = o.reduce_block_amax(x, bs).reshape(-1) * np.float32(0.75)
        gm = np.float32(bam.max())
        p, s, s2 = ops.pack_nvfp4(dev(x, "bf16"), dev(gm, "f32").reshape(1), dev(bam, "f32"), block_size=bs)
        wp, ws, ws2 = o.pack_nvfp4(x, gm, bam.reshape(64, -1), block_size=bs)
        same(p.cpu().numpy(), wp, f"static packed {bs}")
        same(s.view(torch.uint8).cpu().numpy(), ws, f"static scale {bs}")


def test_multi_tensor_launches_equal_single_launches(ops):
    """b200q_amax_per_tensor_multi / b200q_fake_quant_nvfp4_multi: one grid over a table of tensors == the per-tensor
    launches, bit for bit (ragged CTA counts, a tensor smaller than one CTA tile, running max over two calls)."""
    g = torch.Generator(device="cuda").manual_seed(5)
    shapes = [(512, 4096), (8, 16), (300, 1024), (64, 14336), (1, 4096)]
    xs = [(torch.randn(s, device="cuda", generator=g) * (0.5 + i)).to(torch.bfloat16) for i, s in enumerate(shapes)]
    slots = torch.zeros(8, dtype=torch.float32, device="cuda")
    order = [3, 0, 7, 5, 1]
    table = ops.TensorTable(xs, order, None, "vec32")
    ops.amax_per_tensor_multi_(slots, table)
    for x, s in zip(xs, order):
        assert float(slots[s]) == float(x.abs().max())
    assert float(slots[2]) == 0 and float(slots[4]) == 0 and float(slots[6]) == 0
    xs[1].mul_(100.0)
    ops.amax_per_tensor_multi_(slots, table)               # running max, same table (raw pointers)
    assert float(slots[order[1]]) == float(xs[1].abs().max())
    assert float(slots[order[0]]) == float(xs[0].abs().max())
    ys = [torch.empty_like(x) for x in xs]
    amax = torch.zeros(8, dtype=torch.bfloat16, device="cuda")
    for x, s in zip(xs, order):
        amax[s] = x.abs().max()
    ops.fake_quant_nvfp4_multi(ops.TensorTable(xs, order, ys, "block16"), amax)
    for x, y, s in zip(xs, ys, order):
        assert torch.equal(y, ops.fake_quant_nvfp4(x, amax[s:s + 1])), tuple(x.shape)
    with pytest.raises(Exception):
        ops.TensorTable([xs[0][:, 1:]], None, None, "vec32")          # not contiguous / not 32-byte aligned


def test_engine_grouped_launches_equal_per_quantizer_launches():
    from model_optimizer_b200.engine import TINY, ShardedPTQEngine

    res = {}
    for grouped in (False, True):
        eng = ShardedPTQEngine(TINY, 256, "nvfp4", torch.bfloat16, "cuda", grouped=grouped)
        acts = eng.alloc_activations(seed=3)
        outs = eng.alloc_outputs(len(eng.quantizers))      # one output per quantizer: nothing is overwritten
        eng.capture(acts, outs)
        for _ in range(2):
            eng.step_graph()
        torch.cuda.synchronize()
        written = [outs[i][: x.numel()].clone() for i, x in enumerate(acts)]     # the tails of the ring are never written
        res[grouped] = (eng.arena.freeze().clone(), eng.amax_arena.clone(), written, eng.launches_per_step())
    assert torch.equal(res[False][0], res[True][0]) and torch.equal(res[False][1], res[True][1])
    for a, b in zip(res[False][2], res[True][2]):
        assert torch.equal(a, b)
    assert res[True][3] == 3 and res[False][3] == 2 * 28 + 1


def test_histogram_pattern_path_equals_elementwise(ops):
    """16-bit inputs: counting the 2^15 |x| bit patterns and binning each pattern once == the element-wise kernel
    (same exact histc formula), incl. unaligned / ragged tensors, zeros, NaN / inf and values above the range."""
    g = torch.Generator(device="cuda").manual_seed(21)
    for dt in (torch.bfloat16, torch.float16):
        for n, off, outlier in ((4096 * 512, 0, 0.0), (100003, 1, 0.0), (37, 3, 0.0), (8 * 1024 + 8, 0, 0.0),
                                (4096 * 64 + 5, 0, 3.0e4), (4096 * 64, 2, 1.0e-3)):
            x = (torch.randn(n + off, device="cuda", generator=g) * 2).to(dt)[off:]
            if outlier > 1.0:
                x[11] = outlier             # most elements fall far below the top of the range (outside the hot window)
            elif outlier > 0.0:
                x *= outlier                # small magnitudes: bf16 / fp16 subnormal-adjacent patterns under the window
            x[::97] = 0
            if n > 1000:
                x[5], x[6], x[7] = float("nan"), float("inf"), -float("inf")
            for nbins, scale in ((2048, 1.0), (512, 0.5), (5000, 1.0)):
                rng = (x[torch.isfinite(x)].abs().max().float() * scale).reshape(1)
                h0 = torch.zeros(nbins, dtype=torch.float32, device="cuda")
                h1 = torch.zeros_like(h0)
                scratch = ops.hist_scratch("cuda")
                ops.histogram_(h0, x, rng)
                ops.histogram_(h1, x, rng, scratch=scratch)
                ops.histogram_(h1, x, rng, scratch=scratch)          # scratch is left zeroed: a second batch adds up
                assert torch.equal(h1, 2 * h0), (dt, n, off, nbins, float((h1 - 2 * h0).abs().sum()))
                assert int(scratch[:32768].abs().sum()) == 0      # the atomic counters are left zeroed
