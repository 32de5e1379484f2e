"""Every 16-bit input value, and a structured fp32 set, through each quantization kernel at scales on both sides of
every window edge of the exact division, bit for bit against the CPU oracle.

The block quantizers divide with ExactDiv's bare FFMA triple inside per-block windows (``csrc/common.cuh``); the
arguments for why those quotients round as div.rn.f32's would live in comments, and seeded data at ordinary scales
almost never meets the values that would break them (fp32-range bf16 values, subnormals, exact ties at every scale,
quotients that overflow).  Inputs and the scale grid come from ``tests/_value_sweep.py``; ``test_value_sweep_cpu.py``
checks there that they reach both sides of every branch.  Bar: bit-exact, NaN positions equal."""

import numpy as np
import pytest
import torch

from oracle import oracle_np as o
import _value_sweep as vs
from tools import gptq_oracle as orc

pytestmark = pytest.mark.gpu

TD = {"bf16": torch.bfloat16, "f16": torch.float16, "f32": torch.float32}
S = vs.scale_grid()
S_COARSE = vs.coarse(S)


@pytest.fixture(scope="module")
def ops():
    from model_optimizer_b200 import ops as _ops

    return _ops


def dev(x, dt):
    """fp32 values exactly representable in ``dt`` -> a CUDA tensor of ``dt`` holding the same bit patterns."""
    x = np.ascontiguousarray(x, dtype=np.float32)
    if dt == "f32":
        return torch.from_numpy(x.copy()).cuda()
    if dt == "bf16":
        bits = (x.view(np.uint32) >> 16).astype(np.uint16)
    else:
        bits = x.astype(np.float16).view(np.uint16)
    return torch.from_numpy(bits.view(np.int16)).cuda().view(TD[dt])


def dev16(dt, rows):
    """``rows`` copies of all 65536 patterns of a 16-bit type, built on the device from the patterns themselves."""
    p = torch.arange(65536, dtype=torch.int32, device="cuda").to(torch.int16).view(TD[dt])
    return p.unsqueeze(0).repeat(rows, 1)


def host(t):
    return t.detach().float().cpu().numpy()


def same(got, want, what, x=None):
    """Bit equality (NaN == NaN); on failure the first mismatches, with the input row's values when ``x`` is given."""
    got = np.ascontiguousarray(got)
    want = np.ascontiguousarray(want)
    assert got.shape == want.shape, (what, got.shape, want.shape)
    if got.dtype.kind == "f":
        g32, w32 = got.astype(np.float32), want.astype(np.float32)
        ok = (g32.view(np.uint32) == w32.view(np.uint32)) | (np.isnan(g32) & np.isnan(w32))
    else:
        ok = got == want
    nbad = int((~ok).sum())
    if nbad:
        lines = []
        for i in map(tuple, np.argwhere(~ok)[:4]):
            ctx = ""
            if x is not None and np.shape(x) == got.shape:
                ctx = f" input {np.asarray(x)[i]!r}"
            elif x is not None:
                xr = np.asarray(x).reshape(got.shape[0], -1) if got.ndim > 1 else np.asarray(x).reshape(1, -1)
                ctx = f" input row {xr[i[0]] if got.ndim > 1 else xr[0]}"
            lines.append(f"at {i}: got {got[i]!r} want {want[i]!r}{ctx}")
        raise AssertionError(f"{what}: {nbad}/{ok.size} mismatches\n" + "\n".join(lines))


def rows_input(dt, units, ts, mult=32):
    """(device tensor, fp32 host values) of one row per scale: all 16-bit patterns, or the fp32 rows with the
    boundary values of each row's unit."""
    if dt == "f32":
        x = vs.fp32_rows(units, ts, mult)
        return dev(x, dt), x
    xd = dev16(dt, len(units))
    return xd, np.tile(vs.values16(dt), (len(units), 1))


# ------------------------------------------------------------------------------------------------
# INT / FP8 fake quant: the scale is a free input
# ------------------------------------------------------------------------------------------------
INT_CFGS = [(8, False, True), (8, False, False), (4, False, False), (4, True, False), (8, True, True)]


@pytest.mark.parametrize("dt", vs.DTYPES)
@pytest.mark.parametrize("bits,unsigned,narrow", INT_CFGS)
def test_int_fake_quant_per_row(ops, dt, bits, unsigned, narrow):
    bound = (1 << (bits - 1 + int(unsigned))) - 1
    with np.errstate(all="ignore"):
        units = (S / np.float32(bound)).astype(np.float32)
    xd, x = rows_input(dt, units, vs.int_t(bound))
    amax = torch.from_numpy(S.copy()).cuda()
    y = ops.fake_quant_int(xd, amax, bits, unsigned, narrow, outer=x.shape[1])
    want = o.fake_quant_int(x, S, bits, unsigned, narrow, outer=x.shape[1], dtype=dt)
    same(host(y), want, f"int{bits} u={unsigned} n={narrow} {dt} per-row")
    # offset by one element: the scalar kernel (its own apply2 form); the row pattern shifts by one
    flat = torch.zeros(xd.numel() + 1, dtype=xd.dtype, device="cuda")
    flat[1:] = xd.reshape(-1)
    y1 = ops.fake_quant_int(flat[1:], amax, bits, unsigned, narrow, outer=x.shape[1])
    same(host(y1).reshape(x.shape), want, f"int{bits} u={unsigned} n={narrow} {dt} per-row, unaligned")


@pytest.mark.parametrize("dt", vs.DTYPES)
def test_int_fake_quant_per_tensor(ops, dt):
    x = vs.domain(dt)
    xd = dev(x, dt)
    for bits, unsigned, narrow in INT_CFGS[:3]:
        for a in S_COARSE:
            amax = torch.tensor([a], dtype=torch.float32, device="cuda")
            y = ops.fake_quant_int(xd, amax, bits, unsigned, narrow)
            same(host(y), o.fake_quant_int(x, a, bits, unsigned, narrow, dtype=dt), f"int{bits} {dt} amax={a!r}")


@pytest.mark.parametrize("dt", vs.DTYPES)
@pytest.mark.parametrize("eager", [False, True])
def test_fp8_fake_quant(ops, dt, eager):
    with np.errstate(all="ignore"):
        units = (S / np.float32(448.0)).astype(np.float32)
    xd, x = rows_input(dt, units, vs.E4M3_T)
    amax = torch.from_numpy(S.copy()).cuda()
    y = ops.fake_quant_fp8(xd, amax, outer=x.shape[1], eager=eager)
    want = o.fake_quant_fp8(x, S, outer=x.shape[1], dtype=dt, eager=eager)
    same(host(y), want, f"fp8 eager={eager} {dt} per-row")
    flat = torch.zeros(xd.numel() + 1, dtype=xd.dtype, device="cuda")
    flat[1:] = xd.reshape(-1)
    y1 = ops.fake_quant_fp8(flat[1:], amax, outer=x.shape[1], eager=eager)
    same(host(y1).reshape(x.shape), want, f"fp8 eager={eager} {dt} per-row, unaligned")
    xs, xsd = vs.domain(dt), dev(vs.domain(dt), dt)
    for a in S_COARSE:
        y = ops.fake_quant_fp8(xsd, torch.tensor([a], device="cuda"), eager=eager)
        same(host(y), o.fake_quant_fp8(xs, a, dtype=dt, eager=eager), f"fp8 eager={eager} {dt} amax={a!r}")


# ------------------------------------------------------------------------------------------------
# NVFP4 fake quant
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dt", vs.DTYPES)
def test_nvfp4_static_block_scale_is_the_grid(ops, dt):
    """quantize_block_scales=False: block amax 6 * S[r] makes the block scale S[r] itself."""
    xd, x = rows_input(dt, S, vs.E2M1_T)
    with np.errstate(over="ignore"):
        bam = np.repeat((S * np.float32(6.0)).astype(np.float32), x.shape[1] // 16)
    y = ops.fake_quant_nvfp4_static(xd, torch.from_numpy(bam).cuda(), quantize_block_scales=False)
    same(host(y), o.fake_quant_nvfp4_static(x, bam, None, False, dtype=dt), f"nvfp4 static {dt} unquantized scales")


@pytest.mark.parametrize("dt", vs.DTYPES)
@pytest.mark.parametrize("fmn", [448.0, 256.0])
def test_nvfp4_static_quantized_block_scales(ops, dt, fmn):
    """The FP8 block scale is e4m3(6 * S[r] * fmn / g): with these global amaxes the rows reach E4M3 zero (a zeroed
    block), subnormals, normals and the 448 clamp."""
    xd, x = rows_input(dt, S, vs.E2M1_T)
    with np.errstate(over="ignore"):
        bam = np.repeat((S * np.float32(6.0)).astype(np.float32), x.shape[1] // 16)
    for g in (6.0 * fmn, 6.0 * fmn * 2.0 ** -40, 6.0 * fmn * 2.0 ** 40, 1.0):
        gt = torch.tensor([g], dtype=torch.float32, device="cuda")
        y = ops.fake_quant_nvfp4_static(xd, torch.from_numpy(bam).cuda(), gt, True, fmn)
        want = o.fake_quant_nvfp4_static(x, bam, np.float32(g), True, fmn, dtype=dt)
        same(host(y), want, f"nvfp4 static {dt} fmn={fmn} g={g!r}")


@pytest.mark.parametrize("dt", vs.DTYPES)
def test_nvfp4_dynamic_global_amax_sweep(ops, dt):
    for g in S_COARSE:
        x = vs.nvfp4_dynamic_input(dt, g)
        xd = dev(x, dt)
        y = ops.fake_quant_nvfp4(xd, torch.tensor([g], dtype=torch.float32, device="cuda"))
        same(host(y), o.fake_quant_nvfp4(x, g, dtype=dt), f"nvfp4 dynamic {dt} g={g!r}", x)


# ------------------------------------------------------------------------------------------------
# NVFP4 pack
# ------------------------------------------------------------------------------------------------
def _check_pack(ops, x, dt, got, want, what):
    packed, scales, wsf2 = got
    wp, wb, ws = want
    same(host(wsf2).reshape(()), np.float32(ws), what + " wsf2")
    same(scales.view(torch.uint8).cpu().numpy(), wb, what + " scales", x)
    same(packed.cpu().numpy(), wp, what + " codes", x)
    y = ops.unpack_nvfp4(packed, scales, wsf2, TD[dt])
    same(host(y), o.unpack_nvfp4(wp, wb, ws, dtype=dt), what + " unpack")


@pytest.mark.parametrize("dt", vs.DTYPES)
def test_nvfp4_pack_given_wsf2(ops, dt):
    """A caller-given weights_scaling_factor_2 w puts the clamped block's divisor at fl(448 * w): across kBlockMin,
    kMaxDenom and far outside the window."""
    for w in vs.pack_wsf2_grid():
        x = vs.nvfp4_dynamic_input(dt, np.float32(w * np.float32(2688.0)))
        xd = dev(x, dt)
        got = ops.pack_nvfp4(xd, None, wsf2=torch.tensor(w, dtype=torch.float32))
        want = o.pack_nvfp4(x, wsf2=w)
        _check_pack(ops, x, dt, got, (want[0], want[1].reshape(-1, 1), want[2]), f"pack {dt} wsf2={w!r}")


@pytest.mark.parametrize("dt", vs.DTYPES)
def test_nvfp4_pack_dynamic_global_amax_sweep(ops, dt):
    for g in S_COARSE:
        x = vs.nvfp4_dynamic_input(dt, g)
        xd = dev(x, dt)
        got = ops.pack_nvfp4(xd, torch.tensor(g, dtype=torch.float32))
        _check_pack(ops, x, dt, got, o.pack_nvfp4(x, global_amax=g), f"pack {dt} g={g!r}")


@pytest.mark.parametrize("dt", vs.DTYPES)
def test_nvfp4_pack_static_block_amax(ops, dt):
    xd, x = rows_input(dt, S, vs.E2M1_T)
    x16 = x.reshape(-1, 16)
    with np.errstate(over="ignore"):
        bam = np.repeat((S * np.float32(6.0)).astype(np.float32), x.shape[1] // 16)
    for g, fmn in ((2688.0, 448.0), (2.0 ** -30, 448.0), (2.0 ** 40, 256.0)):
        got = ops.pack_nvfp4(xd.reshape(-1, 16), torch.tensor(g, dtype=torch.float32),
                             block_amax=torch.from_numpy(bam), fp8_max_norm=fmn)
        want = o.pack_nvfp4(x16, global_amax=g, block_amax=bam, fp8_max_norm=fmn)
        _check_pack(ops, x16, dt, got, want, f"pack static {dt} g={g!r} fmn={fmn}")


@pytest.mark.parametrize("dt", ["bf16", "f32"])
def test_nvfp4_pack_overflowing_quotient_keeps_its_sign(ops, dt):
    """A block inside the divisor window whose quotient overflows: -1e30 / ~5e-10 is -inf, code 0xF (the reference's
    _cast_fp4 takes the sign from y < 0 and the ordinal 7 from |y| = inf)."""
    x = np.zeros((1, 16), dtype=np.float32)
    x[0, 0], x[0, 1], x[0, 2] = -1e30, 1e30, -1.0
    x = o.round_to(x, dt)
    got = ops.pack_nvfp4(dev(x, dt), torch.tensor(3e-9, dtype=torch.float32))
    want = o.pack_nvfp4(x, global_amax=np.float32(3e-9))
    assert want[0][0, 0] == 0x7F and want[0][0, 1] & 0xF == 0xF
    _check_pack(ops, x, dt, got, want, f"pack {dt} overflow")


# ------------------------------------------------------------------------------------------------
# NF4, INT8 and FP8 pack: per-block / per-row scales
# ------------------------------------------------------------------------------------------------
NF4_S = vs.coarse(S, 3)


@pytest.mark.parametrize("dt", vs.DTYPES)
def test_nf4_pack_given_scales(ops, dt):
    sc = o.round_to(NF4_S, dt)
    sc = sc[np.isfinite(sc)]
    xd, x = rows_input(dt, sc, vs.NF4_T, mult=64)
    scales = np.repeat(sc, x.shape[1] // 64)
    packed, _ = ops.pack_nf4(xd, 64, dev(scales.reshape(-1, 1), dt))
    want, _ = o.pack_nf4(x, 64, dtype=dt, scales=scales)
    same(packed.cpu().numpy(), want, f"nf4 {dt} given scales")


@pytest.mark.parametrize("dt", vs.DTYPES)
@pytest.mark.parametrize("block", [16, 64])
def test_nf4_pack_computed_scales(ops, dt, block):
    x = vs.mx_input(dt, block).reshape(-1)
    x = x[: x.size // block * block]
    packed, sc = ops.pack_nf4(dev(x, dt), block)
    want, wsc = o.pack_nf4(x, block, dtype=dt)
    same(host(sc), wsc, f"nf4 {dt} b{block} scales")
    same(packed.cpu().numpy(), want, f"nf4 {dt} b{block} codes")


@pytest.mark.parametrize("dt", vs.DTYPES)
@pytest.mark.parametrize("kind", ["int8", "fp8"])
@pytest.mark.parametrize("scale_dt", ["same", "f32"])
def test_int8_fp8_pack_per_row(ops, dt, kind, scale_dt):
    sdt = dt if scale_dt == "same" else "f32"
    sc = o.round_to(S, sdt)
    sc = sc[np.isfinite(sc) & (sc > 0)]
    xd, x = rows_input(dt, sc, vs.int_t(127) if kind == "int8" else vs.E4M3_T)
    sct = dev(sc, sdt)
    pack = ops.pack_int8 if kind == "int8" else ops.pack_fp8
    q = pack(xd, sct, outer=x.shape[1])
    ref = o.pack_int8 if kind == "int8" else o.pack_fp8
    want = ref(x, sc, outer=x.shape[1], x_dtype=dt, scale_dtype=sdt)
    if kind == "int8":
        same(q.cpu().numpy(), want, f"int8 pack {dt} scale {sdt}")
    else:
        same(q.view(torch.uint8).cpu().numpy(), want, f"fp8 pack {dt} scale {sdt}", x)


# ------------------------------------------------------------------------------------------------
# MX: the scale comes from the block max; setters steer it over the whole E8M0 range
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dt", vs.DTYPES)
@pytest.mark.parametrize("block", [16, 32])
def test_mx_fake_quant(ops, dt, block):
    x = vs.mx_input(dt, block)
    xd = dev(x, dt)
    for name, fmt in ops.MX_FORMATS.items():
        if name == "E8M0":
            continue
        y = ops.fake_quant_mx(xd, block, name)
        same(host(y), o.fake_quant_mx(x, block, fmt, dtype=dt), f"mx {name} {dt} b{block}")


@pytest.mark.parametrize("dt", vs.DTYPES)
def test_mxfp8_mxfp4_pack(ops, dt):
    x = vs.mx_input(dt, 32)
    xd = dev(x, dt)
    q, s = ops.pack_mxfp8(xd)
    wq, ws = o.pack_mxfp8(x)
    same(s.cpu().numpy(), ws, f"mxfp8 {dt} scales", x)
    same(q.view(torch.uint8).cpu().numpy(), wq, f"mxfp8 {dt} codes", x)
    fin = np.isfinite(x).all(axis=1)            # MXFP4QTensor.quantize: finite blocks (log2 of the block max)
    xf = x[fin]
    q4, s4 = ops.pack_mxfp4(dev(xf, dt), 32)
    wq4, ws4 = o.pack_mxfp4(xf, 32)
    same(s4.cpu().numpy(), ws4, f"mxfp4 {dt} scales", xf)
    same(q4.cpu().numpy(), wq4, f"mxfp4 {dt} codes", xf)


# ------------------------------------------------------------------------------------------------
# GPTQ column kernel: with U = I no error reaches another column, so the update is the plain fake quant (INT, FP8,
# static NVFP4) or the column loop's oracle (dynamic NVFP4)
# ------------------------------------------------------------------------------------------------
def _gptq_weight():
    w = np.concatenate([vs.values16("bf16"), vs.values16("f16"), vs.fp32_structured()])
    w = w[np.isfinite(w)]                       # an inf / NaN error would reach the other columns as inf * 0
    nb = 64
    n = -(-w.size // nb) * nb
    out = np.zeros(n, dtype=np.float32)
    out[:w.size] = w
    return out.reshape(-1, nb)


def test_gptq_identity_update_equals_fake_quant(ops):
    w = _gptq_weight()
    rows, nb = w.shape
    u = torch.eye(nb, dtype=torch.float32, device="cuda")
    ra = S[np.arange(rows) % S.size]                               # one amax per row, cycling through S
    ra_t = torch.from_numpy(ra.copy()).cuda()
    cases = [
        (dict(fmt=ops.GPTQ_INT, amax=ra_t, amax_row_stride=1, num_bits=8, narrow_range=True),
         o.fake_quant_int(w, ra, 8, False, True, outer=nb, dtype="f32"), "int8"),
        (dict(fmt=ops.GPTQ_INT, amax=ra_t, amax_row_stride=1, num_bits=4),
         o.fake_quant_int(w, ra, 4, False, False, outer=nb, dtype="f32"), "int4"),
        (dict(fmt=ops.GPTQ_FP8, amax=ra_t, amax_row_stride=1),
         o.fake_quant_fp8(w, ra, outer=nb, dtype="f32"), "fp8"),
    ]
    with np.errstate(over="ignore"):
        bam = np.repeat((ra * np.float32(6.0)).astype(np.float32), nb // 16)
    for g in (2688.0, 2.0 ** -30):
        cases.append((dict(fmt=ops.GPTQ_NVFP4_STATIC, amax=torch.from_numpy(bam).cuda(), amax_row_stride=nb // 16,
                           amax_col_block=16, global_amax=torch.tensor(g, dtype=torch.float32, device="cuda")),
                      o.fake_quant_nvfp4_static(w, bam, np.float32(g), True, dtype="f32"), f"nvfp4 static g={g}"))
    # dynamic NVFP4 takes each column's block max from the working block, whose earlier columns already hold their
    # quantized values: the plain fake quant only where that leaves the max alone, so the C oracle of the column loop
    eye = np.eye(nb, dtype=np.float32)
    for g in S_COARSE:
        want, _ = orc.gptq_block(w, eye, orc.FMT_NVFP4_DYNAMIC, amax=np.array([g], dtype=np.float32))
        cases.append((dict(fmt=ops.GPTQ_NVFP4_DYNAMIC, amax=torch.tensor([g], dtype=torch.float32, device="cuda")),
                      want, f"nvfp4 dynamic g={g!r}"))
    for kw, want, what in cases:
        wd = torch.from_numpy(w.copy()).cuda()
        ops.gptq_block_update(wd, u, **kw)
        same(host(wd), want, f"gptq {what}")


# ------------------------------------------------------------------------------------------------
# Independent second opinions: torch's own CUDA ops, and the reference's compiled CUDA extensions
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dt", vs.DTYPES)
def test_fp8_pack_equals_torch_cuda_division(ops, dt):
    """FP8QTensor.quantize is ``(x / scale).to(torch.float8_e4m3fn)`` (qtensor/fp8_tensor.py:107): the same torch ops
    on the same CUDA tensors must give the kernel's bytes for every pattern, NaN of either sign included (CUDA
    arithmetic returns a NaN with the sign bit clear, so -NaN packs to 0x7f)."""
    sc = o.round_to(S, dt)
    sc = sc[np.isfinite(sc) & (sc > 0)]
    xd, x = rows_input(dt, sc, vs.E4M3_T)
    for sdt in sorted({dt, "f32"}):
        s = o.round_to(sc, sdt)
        st = dev(s, sdt)
        want = (xd / st.reshape(-1, 1)).to(torch.float8_e4m3fn).view(torch.uint8)
        got = ops.pack_fp8(xd, st, outer=x.shape[1]).view(torch.uint8)
        same(got.cpu().numpy(), want.cpu().numpy(), f"fp8 pack {dt} scale {sdt} vs torch", x)
    ibits = xd[0].view(torch.int32 if dt == "f32" else torch.int16)
    assert bool((torch.isnan(xd[0]) & (ibits < 0)).any()), "the domain holds negative NaNs"


@pytest.mark.parametrize("dt", vs.DTYPES)
def test_mxfp8_pack_equals_torch_cuda_ops(ops, dt):
    """MXFP8QTensor.quantize_with_scale (qtensor/mxfp8_tensor.py:150-180) in torch on the GPU, with the E8M0 bytes the
    kernel computed (compared with the oracle in test_mxfp8_mxfp4_pack): the kernel's codes, -NaN included."""
    x = vs.mx_input(dt, 32)
    xd = dev(x, dt)
    q, s = ops.pack_mxfp8(xd)
    sf = torch.exp2(127 - s.float())
    want = torch.clamp(xd.view(-1, 1, 32) * sf.unsqueeze(-1), min=-448.0, max=448.0).to(torch.float8_e4m3fn)
    same(q.view(torch.uint8).cpu().numpy(), want.view(torch.uint8).reshape(q.shape).cpu().numpy(),
         f"mxfp8 {dt} vs torch", x)
    q2, _ = ops.pack_mxfp8(xd, s)
    same(q2.view(torch.uint8).cpu().numpy(), q.view(torch.uint8).cpu().numpy(), f"mxfp8 {dt} given scales")


def _ref_ext(name):
    """A reference CUDA extension built into oracle/_ref (skip when it was not built)."""
    import importlib.machinery
    import importlib.util
    import os

    path = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle", "_ref", name + ".so")
    if not os.path.exists(path):
        pytest.skip(f"{path} not built (python oracle/build_ref_ext.py where the reference sources exist)")
    loader = importlib.machinery.ExtensionFileLoader(name, path)
    mod = importlib.util.module_from_spec(importlib.util.spec_from_loader(name, loader))
    loader.exec_module(mod)
    return mod


@pytest.mark.parametrize("dt", vs.DTYPES)
def test_int_fake_quant_vs_reference_ext(ops, dt):
    ext = _ref_ext("modelopt_cuda_ext")
    amax = torch.from_numpy(S.copy()).cuda()
    for bits, unsigned, narrow in INT_CFGS:
        bound = (1 << (bits - 1 + int(unsigned))) - 1
        with np.errstate(all="ignore"):
            units = (S / np.float32(bound)).astype(np.float32)
        xd, x = rows_input(dt, units, vs.int_t(bound))
        if unsigned:       # the extension asserts x >= 0 on the device for unsigned quantization: negatives and NaN -> 0
            xd = torch.where(xd >= 0, xd, torch.zeros_like(xd))
            x = np.where(x >= 0, x, np.float32(0)).astype(np.float32)
        ref = ext.fake_tensor_quant_with_axis(xd, amax, 0, bits, unsigned, narrow)
        got = ops.fake_quant_int(xd, amax, bits, unsigned, narrow, outer=x.shape[1])
        same(host(got), host(ref), f"int{bits} u={unsigned} n={narrow} {dt} per-row vs ext", x)
    xs = dev(vs.domain(dt), dt)
    for a in S_COARSE:                                 # signed: the extension's unsigned kernel asserts x >= 0
        at = torch.tensor([a], dtype=torch.float32, device="cuda")
        same(host(ops.fake_quant_int(xs, at, 8, False, True)), host(ext.fake_tensor_quant(xs, at, 8, False, True)),
             f"int8 {dt} amax={a!r} vs ext", vs.domain(dt))


@pytest.mark.parametrize("dt", vs.DTYPES)
def test_fp8_fake_quant_vs_reference_ext(ops, dt):
    ext = _ref_ext("modelopt_cuda_ext_fp8")
    amax = torch.from_numpy(S.copy()).cuda()
    with np.errstate(all="ignore"):
        units = (S / np.float32(448.0)).astype(np.float32)
    xd, x = rows_input(dt, units, vs.E4M3_T)
    same(host(ops.fake_quant_fp8(xd, amax, outer=x.shape[1])), host(ext.fake_e4m3fy_with_axis(xd, amax, 0)),
         f"fp8 {dt} per-row vs ext", x)
    xs = dev(vs.domain(dt), dt)
    for a in S_COARSE:
        at = torch.tensor([a], dtype=torch.float32, device="cuda")
        same(host(ops.fake_quant_fp8(xs, at)), host(ext.fake_e4m3fy(xs, at)), f"fp8 {dt} amax={a!r} vs ext",
             vs.domain(dt))


@pytest.mark.parametrize("dt", vs.DTYPES)
def test_nf4_pack_vs_reference_ext(ops, dt):
    ext = _ref_ext("modelopt_cuda_ext")
    sc = o.round_to(NF4_S, dt)
    sc = sc[np.isfinite(sc)]
    xd, x = rows_input(dt, sc, vs.NF4_T, mult=64)
    scales = dev(np.repeat(sc, x.shape[1] // 64).reshape(-1, 1), dt)
    flat = xd.reshape(-1)
    same(ops.pack_nf4(flat, 64, scales)[0].cpu().numpy(), ext.NF4_quantize(flat, scales, 64).reshape(-1).cpu().numpy(),
         f"nf4 {dt} given scales vs ext")
    for block in (16, 64):
        xm = vs.mx_input(dt, block).reshape(-1)
        xm = dev(xm[: xm.size // block * block], dt)
        got, got_sc = ops.pack_nf4(xm, block)
        tsc = xm.view(-1, block).abs().amax(dim=-1, keepdim=True)        # what NF4QTensor.quantize computes
        same(host(got_sc), host(tsc), f"nf4 {dt} b{block} scales vs torch")
        same(got.cpu().numpy(), ext.NF4_quantize(xm, tsc, block).reshape(-1).cpu().numpy(), f"nf4 {dt} b{block} vs ext")


@pytest.mark.parametrize("dt", vs.DTYPES)
@pytest.mark.parametrize("block", [16, 32])
def test_mx_fake_quant_vs_reference_ext(ops, dt, block):
    """fused_amax_convert with an E8M0 scale, on the blocks the extension computes as its source says.  It is built
    with --use_fast_math as the reference builds it: denormal operands, results and intermediates flush to zero (a block
    whose amax / format max is below 2^-126 gets scale 1 there, one whose ratio is above 2^126 a scale 2^-127 that
    flushes to zero), and its `sign` is uninitialised for zero inputs (tensor_quant_mx.cu:39-43).  So blocks holding a
    denormal input, a non-finite input or an amax ratio outside [2^-126, 2^126] are
    left to the oracle comparison above (the oracle is pinned to host builds of the same source); results are compared
    after flushing denormals, and zeros by value."""
    ext = _ref_ext("modelopt_cuda_ext_mx")
    x = vs.mx_input(dt, block)
    xd = dev(x, dt)
    with np.errstate(invalid="ignore"):
        a = np.abs(x)
        plain = np.isfinite(x).all(axis=1) & ~((a > 0) & (a < np.float32(2.0 ** -126))).any(axis=1)
    amax = np.where(plain, a.max(axis=1), np.float32(0))
    ftz = lambda v: np.where(np.abs(v) < np.float32(2.0 ** -126), np.float32(0), v)  # noqa: E731
    for name, fmt in ops.MX_FORMATS.items():
        if name == "E8M0":
            continue
        ratio = amax / np.float32(o.MX_FORMAT_MAX[fmt])
        keep = plain & ((amax == 0) | ((ratio >= np.float32(2.0 ** -126)) & (ratio <= np.float32(2.0 ** 126))))
        assert keep.mean() > 0.5, (name, dt, block, keep.mean())
        ref = host(ext.fused_amax_convert(xd, block, getattr(ext.Types, name), ext.Types.E8M0, None))
        got = host(ops.fake_quant_mx(xd, block, name))
        same(ftz(got)[keep] + np.float32(0), ftz(ref)[keep] + np.float32(0), f"mx {name} {dt} b{block} vs ext",
             x[keep])
