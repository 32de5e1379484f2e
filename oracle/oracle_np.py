"""CPU ORACLE -- test infrastructure, NOT product code.

A NumPy restatement of the reference's algorithms for the PTQ hot path (calibration collect,
fake-quant forward, weight quant-and-pack).  Only ``tests/``, ``__graft_entry__.smoke()`` and
``bench.py``'s ``cpu_baseline`` / ``--impl reference`` legs may import it; the product path
(``model_optimizer_b200``) never does and has no CPU fallback.

Pinned: ``tests/golden/*.npz`` hold outputs of the REAL reference (imported from
/root/reference through the shim in ``oracle/gen_golden.py``; the MX section through host builds of
the reference's C++ in ``oracle/_ref``) and the reference's own golden vectors;
``tests/test_oracle_golden.py`` / ``test_oracle_algos.py`` / ``test_oracle_mx.py`` assert this file
reproduces them bit-for-bit.  On the GPU box the reference's compiled CUDA extensions and AOT-compiled
Triton kernels (``oracle/_ref``, built by ``build_ref_ext.py`` / ``build_ref_triton.py``) run next to
the product kernels (``tests/test_gpu_vs_reference_ext.py`` / ``_triton.py``).

All paths cited below are relative to the reference tree ``modelopt/torch/``.

Conventions: tensors are float32 NumPy arrays holding values exactly representable in the
tensor's nominal dtype (``"bf16"``, ``"f16"`` or ``"f32"``); ``dtype`` arguments say which
rounding the reference would apply when it stores a result.  All arithmetic is IEEE fp32.
"""

from __future__ import annotations

import numpy as np

F32 = np.float32
E2M1_VALUES = np.array([0, 0.5, 1, 1.5, 2, 3, 4, 6], dtype=F32)
E2M1_BOUNDS = np.array([0.25, 0.75, 1.25, 1.75, 2.5, 3.5, 5.0], dtype=F32)
EPS24 = F32(1.0 / (1 << 24))


# ------------------------------------------------------------------------------------------------
# storage formats
# ------------------------------------------------------------------------------------------------
def round_bf16(x):
    """float32 -> nearest bfloat16 (RNE), returned as float32."""
    shape = np.shape(x)
    x = np.ascontiguousarray(x, dtype=F32).reshape(-1)
    b = x.view(np.uint32).astype(np.uint64)
    r = ((b + 0x7FFF + ((b >> 16) & 1)) >> 16) << 16
    out = (r & 0xFFFFFFFF).astype(np.uint32).view(F32).copy()
    nan = np.isnan(x)
    if nan.any():
        out[nan] = np.nan
    return out.reshape(shape)


def round_f16(x):
    with np.errstate(over="ignore"):
        return np.asarray(x, dtype=F32).astype(np.float16).astype(F32)


def round_to(x, dtype):
    if dtype == "bf16":
        return round_bf16(x)
    if dtype == "f16":
        return round_f16(x)
    if dtype == "f32":
        return np.asarray(x, dtype=F32)
    raise ValueError(dtype)


def bf16_bits(x):
    """uint16 bit patterns of bf16-representable float32 values."""
    return (np.ascontiguousarray(x, dtype=F32).view(np.uint32) >> 16).astype(np.uint16)


def from_bf16_bits(b):
    return (np.asarray(b, dtype=np.uint16).astype(np.uint32) << 16).view(F32)


def e4m3_round(v):
    """float(e4m3_rne_satfinite(v)): cvt.rn.satfinite.e4m3x2.f32 / __nv_fp8_e4m3 semantics
    (kernels/quantization/gemm/tensor_quant_gpu_fp8.cu:41-43).  NaN stays NaN, +-inf -> +-448."""
    v = np.asarray(v, dtype=F32)
    a = np.abs(v)
    with np.errstate(invalid="ignore", over="ignore"):
        # normal range: keep 3 mantissa bits (RNE on the fp32 bit pattern)
        b = a.view(np.uint32).astype(np.uint64)
        r = (b + 0x7FFFF + ((b >> 20) & 1)) & ~np.uint64(0xFFFFF)
        normal = (r & 0xFFFFFFFF).astype(np.uint32).view(F32)
        sub = np.rint(a * F32(512.0)) / F32(512.0)  # subnormal grid 2^-9
        out = np.where(a < F32(2.0**-6), sub, normal).astype(F32)
        out = np.minimum(out, F32(448.0))
        out = np.where(np.isnan(v), F32(np.nan), out)
    return np.copysign(out, v).astype(F32)


def e4m3_bits(v_rounded):
    """Bit pattern (uint8) of values already on the e4m3fn grid (|v| <= 448 or NaN)."""
    v = np.asarray(v_rounded, dtype=F32)
    a = np.abs(v)
    sign = (np.signbit(v)).astype(np.uint8) << 7
    with np.errstate(divide="ignore", invalid="ignore"):
        e = np.floor(np.log2(np.where(a > 0, a, 1.0))).astype(np.int32)
    e = np.clip(e, -6, 8)
    is_sub = a < F32(2.0**-6)
    mant_sub = np.rint(a * 512.0).astype(np.int32)
    mant_norm = np.rint((a / np.exp2(e.astype(np.float64)) - 1.0) * 8.0).astype(np.int32)
    bits = np.where(is_sub, mant_sub, ((e + 7) << 3) | mant_norm).astype(np.uint8)
    bits = np.where(np.isnan(v), np.uint8(0x7F), bits)
    return (bits | sign).astype(np.uint8)


def e4m3_from_bits(b):
    b = np.asarray(b, dtype=np.uint8).astype(np.int32)
    s = np.where(b & 0x80, -1.0, 1.0)
    e = (b >> 3) & 0xF
    m = b & 7
    val = np.where(e == 0, m / 512.0, (1.0 + m / 8.0) * np.exp2((e - 7).astype(np.float64)))
    val = np.where((b & 0x7F) == 0x7F, np.nan, val)
    return (s * val).astype(F32)


def e4m3fn_torch_cast(v):
    """``tensor.to(torch.float8_e4m3fn)`` (c10/util/Float8_e4m3fn.h, third party, pinned by
    tests/gpu/torch/quantization/test_qtensor_cuda.py:110-254): RNE, |v| > 464 -> NaN.  Returns
    (float32 values, uint8 bits)."""
    v = np.asarray(v, dtype=F32)
    r = e4m3_round(v)
    with np.errstate(invalid="ignore"):
        over = ~(np.abs(v) <= F32(464.0))
    r = np.where(over, F32(np.nan), r)
    bits = e4m3_bits(np.where(over, F32(0), r))
    bits = np.where(over, (np.signbit(v).astype(np.uint8) << 7) | np.uint8(0x7F), bits)
    return r.astype(F32), bits.astype(np.uint8)


def e2m1_round_mag(a):
    """fp4_round_magnitude (kernels/quantization/common/nvfp4_quant.py:33-60)."""
    a = np.asarray(a, dtype=F32)
    with np.errstate(invalid="ignore"):
        return np.where(a <= 0.25, 0.0,
               np.where(a < 0.75, 0.5,
               np.where(a <= 1.25, 1.0,
               np.where(a < 1.75, 1.5,
               np.where(a <= 2.5, 2.0,
               np.where(a < 3.5, 3.0,
               np.where(a <= 5.0, 4.0, 6.0))))))).astype(F32)


def cast_fp4_codes(y):
    """NVFP4QTensor._cast_fp4 (quantization/qtensor/nvfp4_tensor.py:229-251): 4-bit codes."""
    y = np.asarray(y, dtype=F32)
    with np.errstate(invalid="ignore"):
        sign = (y < 0).astype(np.uint8)
    a = np.abs(y)
    ordv = np.searchsorted(E2M1_BOUNDS, a, side="left").astype(np.uint8)
    ordv = np.where(np.isnan(a), np.uint8(7), ordv)
    odd = ((a == F32(0.75)) | (a == F32(1.75)) | (a == F32(3.5))).astype(np.uint8)
    return ((sign << 3) + ordv + odd).astype(np.uint8)


# ------------------------------------------------------------------------------------------------
# (1) calibration collect
# ------------------------------------------------------------------------------------------------
def reduce_amax(x, axis=None, keepdims=True):
    """quantization/utils/core_utils.py:147-183: max(|max(x)|, |min(x)|), NaN-propagating,
    result in the input dtype (exact: max/abs never round)."""
    x = np.asarray(x, dtype=F32)
    if axis is None:
        return np.maximum(np.abs(np.max(x)), np.abs(np.min(x))).astype(F32)
    return np.maximum(np.abs(np.max(x, axis=axis, keepdims=keepdims)),
                      np.abs(np.min(x, axis=axis, keepdims=keepdims))).astype(F32)


def nan_skip_absmax(x, axis, keepdims=False):
    """max |x| over ``axis`` skipping NaN elements, NaN where every element is NaN (fmaxf / tl.max).  Not
    ``np.fmax.reduce``: its vectorized loops return NaN or a smaller element for some blocks holding signaling NaNs
    (the fp32 images of bf16 NaN patterns with a clear quiet bit)."""
    a = np.abs(np.asarray(x, dtype=F32))
    nan = np.isnan(a)
    m = np.max(np.where(nan, F32(0), a), axis=axis, keepdims=keepdims)
    return np.where(np.all(nan, axis=axis, keepdims=keepdims), F32(np.nan), m).astype(F32)


def canonical_nan(v):
    """GPU fp32 arithmetic returns the canonical NaN 0x7fffffff (sign clear) whatever the NaN operand's sign; numpy on
    the host keeps it.  Applied where the reference's tensor op (a CUDA op on a CUDA tensor) produces a NaN that a
    sign-keeping cast then reads."""
    v = np.asarray(v, dtype=F32)
    return np.where(np.isnan(v), F32(np.nan), v).astype(F32)


def reduce_block_amax(x, block):
    """core_utils.py:43-89 for block_sizes={-1: block}: [..., K] -> [..., K/block]."""
    x = np.asarray(x, dtype=F32)
    xb = x.reshape(*x.shape[:-1], x.shape[-1] // block, block)
    return reduce_amax(xb, axis=-1, keepdims=False)


class MaxCalibrator:
    """quantization/calib/max.py:26-94 (running elementwise max of reduce_amax)."""

    def __init__(self, axis=None):
        self.axis = axis
        self.amax = None

    def collect(self, x):
        x = np.asarray(x, dtype=F32)
        if self.axis is None:
            local = reduce_amax(x)
        else:
            ax = self.axis if isinstance(self.axis, (tuple, list)) else (self.axis,)
            red = tuple(i for i in range(x.ndim) if i not in ax and (i - x.ndim) not in ax)
            local = reduce_amax(x, axis=red)
        assert not np.any(np.isnan(local)) and not np.any(np.isinf(local))
        self.amax = local if self.amax is None else np.maximum(self.amax, local)

    def compute_amax(self):
        return self.amax


def histc(x, bins, vmax):
    """torch.histc(x, bins, min=0, max=vmax) as computed by ATen's CUDA kernel
    (aten/src/ATen/native/cuda/SummaryOps.cu getBin, third party -- parity pinned only through
    tests/unit/torch/quantization/test_calibrator.py:141-181, exact counts vs numpy):
    bin = (int)((v - min) * bins / (max - min)) in fp32, bin == bins -> bins - 1, values outside
    [min, max] dropped.  Counts returned as float32 like histc.
    A zero range is histc's: min = max = 0 takes the data's own min and max, and a range that is still empty is
    widened by 1 on each side (all zeros: [-1, 1], the zeros in bin bins // 2).  A product v * bins that overflows fp32
    (vmax above FLT_MAX / bins) has no value in that formula; it saturates to the last bin, as the kernels do
    (DESIGN.md section 4, "Histogram ranges")."""
    x = np.asarray(x, dtype=F32).ravel()
    lo, hi = F32(0), F32(vmax)
    if hi == lo and x.size:
        lo, hi = x.min(), x.max()
    if hi == lo:
        lo, hi = F32(lo - 1), F32(hi + 1)
    keep = (x >= lo) & (x <= hi)
    v = (x[keep] - lo).astype(F32)
    with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
        b = ((v * F32(bins)).astype(F32) / (hi - lo)).astype(F32)
    b = np.where(np.isnan(b), 0, np.minimum(b, F32(bins))).astype(np.int64)
    b = np.where(b == bins, bins - 1, b)
    return np.bincount(b, minlength=bins).astype(F32)


def arange_f32(end, step):
    """torch.arange(0, end, step) in fp32 as the device computes it: length ceil(end / step) in fp64, entry i the fp32
    rounding of the exact product i * step.  np.arange(dtype=float32) and torch's CPU fp32 arange round some entries
    differently."""
    n = int(np.ceil(float(end) / float(step)))
    return (np.arange(n, dtype=np.float64) * float(step)).astype(F32)


class HistogramCalibrator:
    """quantization/calib/histogram.py:77-130 (torch_hist=True branch), collect only."""

    def __init__(self, num_bins=2048):
        self.num_bins = num_bins
        self.hist = None
        self.edges = None
        self.n_growths = 0

    def collect(self, x):
        x = np.asarray(x, dtype=F32)
        if x.min() < 0:
            x = np.abs(x)
        x_max = x.max()
        if self.hist is None:
            self.hist = histc(x, self.num_bins, x_max)
            self.edges = np.linspace(0, x_max, self.num_bins + 1, dtype=F32)
        else:
            if x_max > self.edges[-1]:
                width = self.edges[1] - self.edges[0]
                # x_max / width on the device: before the first growth width is a host scalar (linspace edges), which
                # torch applies as a multiplication by its fp32 reciprocal; later it is a device tensor
                q = F32(x_max) * (F32(1) / F32(width)) if self.n_growths == 0 else F32(x_max) / F32(width)
                self.num_bins = int(np.ceil(F32(q)))
                self.edges = arange_f32(F32(x_max) + F32(width), width)
                self.n_growths += 1
            h = histc(x, self.num_bins, self.edges[-1])
            h[: self.hist.size] += self.hist
            self.hist = h


# ------------------------------------------------------------------------------------------------
# (2) fake quant
# ------------------------------------------------------------------------------------------------
def _bcast_amax(x, amax, outer):
    """amax[(i / outer) % n_amax] (kernels/quantization/gemm/tensor_quant_gpu.cu:115)."""
    amax = np.asarray(amax, dtype=F32).ravel()
    if amax.size == 1:
        return amax[0]
    idx = (np.arange(x.size) // outer) % amax.size
    return amax[idx].reshape(x.shape)


def fake_quant_int(x, amax, num_bits=8, unsigned=False, narrow_range=True, outer=1, dtype="bf16"):
    """CUDA integer fake quant: fake_tensor_quant_device
    (kernels/quantization/gemm/tensor_quant_gpu.cu:38-73, :102-118)."""
    x = np.asarray(x, dtype=F32)
    a = _bcast_amax(x, amax, outer)
    bound = F32((1 << (num_bits - 1 + int(unsigned))) - 1)
    max_bound = bound
    min_bound = F32(-(bound + (0 if narrow_range else 1)))
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        scale = (max_bound / a).astype(F32)
        out = np.rint((x * scale).astype(F32)).astype(F32)
        out = np.where(out > max_bound, max_bound, out)
        out = np.where(out < min_bound, min_bound, out)
        out = (out / scale).astype(F32)
    out = np.where(a < EPS24, F32(0.0), out).astype(F32)
    return round_to(out, dtype)


def tensor_quant_cpu(x, amax, num_bits=8, unsigned=False, narrow_range=True, dtype="bf16"):
    """CPU twin ``_tensor_quant`` (quantization/tensor_quant.py:607-645); amax broadcastable."""
    x = np.asarray(x, dtype=F32)
    amax = np.asarray(amax, dtype=F32)
    max_bound = F32(2.0 ** (num_bits - 1 + int(unsigned)) - 1.0)
    min_bound = F32(0) if unsigned else (-max_bound if narrow_range else -max_bound - 1)
    with np.errstate(divide="ignore", invalid="ignore"):
        scale = (max_bound / amax).astype(F32)
        zero = amax <= EPS24
        scale = np.where(zero, F32(0), scale)
        out = np.clip(np.rint((x * scale).astype(F32)), min_bound, max_bound).astype(F32)
        scale = np.where(zero, F32(1), scale)
        out = (out / scale).astype(F32)
    return round_to(out, dtype)


def _fp8_scales(amax, eager=False):
    """scale = 448 / safe_amax, inv = 1 / scale.

    eager=False: the CUDA extension's C++ ``448.f / safe_amax`` -- ATen ``Scalar / Tensor`` is a true
    IEEE division (tensor_quant_gpu_fp8.cu:94-98).  This is the path the reference runs on a GPU.
    eager=True : the Python twin ``448.0 / safe_amax`` (tensor_quant.py:53) which is
    ``Tensor.__rtruediv__`` == ``safe_amax.reciprocal() * 448.0`` (two roundings); runnable on CPU,
    used to pin this oracle against tests/golden (the two differ in the scale's last bit)."""
    amax = np.asarray(amax, dtype=F32)
    safe = np.where(amax <= EPS24, F32(1.0), amax).astype(F32)
    if eager:
        scale = ((F32(1.0) / safe).astype(F32) * F32(448.0)).astype(F32)
    else:
        scale = (F32(448.0) / safe).astype(F32)
    inv = (F32(1.0) / scale).astype(F32)
    return scale, inv


def fake_quant_fp8(x, amax, outer=1, dtype="bf16", eager=False):
    """fake_e4m3fy[_with_axis] (kernels/quantization/gemm/tensor_quant_gpu_fp8.cu:36-107); with
    eager=True, _fp8_eager (quantization/tensor_quant.py:46-59)."""
    x = np.asarray(x, dtype=F32)
    if amax is None:
        r, _ = e4m3fn_torch_cast(x)
        return round_to(r, dtype)
    scale, inv = _fp8_scales(amax, eager)
    s = _bcast_amax(x, scale, outer)
    i = _bcast_amax(x, inv, outer)
    with np.errstate(over="ignore", invalid="ignore"):
        q = e4m3_round((x * s).astype(F32))
        return round_to((q * i).astype(F32), dtype)


def rdiv_scalar(scalar, t, dtype):
    """``python_scalar / tensor`` == ``tensor.reciprocal() * scalar`` (torch/_tensor.py
    Tensor.__rtruediv__): both steps round to the tensor dtype."""
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        r = round_to((F32(1.0) / np.asarray(t, dtype=F32)).astype(F32), dtype)
        return round_to((r * F32(scalar)).astype(F32), dtype)


def nvfp4_block_scale_dynamic(bmax, global_amax):
    """fp8_quantize_scale + the 1e-5 guard (common/nvfp4_quant.py:105-126,
    gemm/fp4_kernel_hopper.py:70-84, :140), IEEE division."""
    gs = F32(F32(global_amax) / F32(6.0 * 448.0))
    gs_safe = gs if gs > 0 else F32(1e-12)
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        sc = (np.asarray(bmax, dtype=F32) / F32(F32(6.0) * gs_safe)).astype(F32)
        sc = np.fmin(sc, F32(448.0))                      # tl.minimum: NaN-ignoring (FMNMX)
        s = (e4m3_round(sc) * gs_safe).astype(F32)
    return np.where(s >= F32(1e-5), s, F32(1.0)).astype(F32)


def _nvfp4_qdq_with_scale(xb, s):
    """nvfp4 element step: sign(x>=0) * e2m1(|x| / s) * s (fp4_kernel_hopper.py:86-95)."""
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        a = (np.abs(xb) / s).astype(F32)
        r = (e2m1_round_mag(a) * s).astype(F32)
    return np.where(xb >= 0, r, -r).astype(F32)


def fake_quant_nvfp4(x, global_amax, dtype="bf16"):
    """NVFP4 dynamic fake quant, blocks of 16 along the last dim, zero padded at the row end."""
    x = np.asarray(x, dtype=F32)
    shape = x.shape
    k = shape[-1]
    x2 = x.reshape(-1, k)
    pad = (-k) % 16
    if pad:
        x2 = np.concatenate([x2, np.zeros((x2.shape[0], pad), dtype=F32)], axis=1)
    xb = x2.reshape(x2.shape[0], -1, 16)
    bmax = nan_skip_absmax(xb, axis=2, keepdims=True)   # tl.max: NaN elements are skipped, an all-NaN block gives NaN
    s = nvfp4_block_scale_dynamic(bmax, global_amax)
    out = _nvfp4_qdq_with_scale(xb, s).reshape(x2.shape)[:, :k]
    return round_to(out.reshape(shape), dtype)


def compute_fp4_scales(amax, global_amax, quantize_block_scales=True, fp8_max_norm=448.0, eager=False):
    """kernels/quantization/gemm/fp4_kernel.py:217-251 (eager: see _fp8_scales)."""
    amax = np.asarray(amax, dtype=F32)
    scale = (amax / F32(6.0)).astype(F32)
    if quantize_block_scales:
        qa = F32(F32(F32(global_amax) * F32(448.0 / fp8_max_norm)) / F32(6.0))
        sc, inv = _fp8_scales(qa, eager)
        with np.errstate(over="ignore", invalid="ignore"):
            prod = (scale * sc).astype(F32)
            if eager:  # _fp8_eager clamps before the cast (tensor_quant.py:55)
                prod = np.clip(prod, F32(-448.0), F32(448.0))
            scale = (e4m3_round(prod) * inv).astype(F32)
    return scale


def fake_quant_nvfp4_static(x, block_amax, global_amax, quantize_block_scales=True,
                            fp8_max_norm=448.0, dtype="bf16"):
    """static_blockwise_fp4_fake_quant (gemm/fp4_kernel.py:194-316) + nvfp4_scalar_quant
    (common/nvfp4_quant.py:67-100)."""
    x = np.asarray(x, dtype=F32)
    xb = x.reshape(-1, 16)
    scale = compute_fp4_scales(np.asarray(block_amax, dtype=F32).reshape(-1, 1), global_amax,
                               quantize_block_scales, fp8_max_norm)
    zero = scale == 0
    safe = np.where(zero | ~np.isfinite(scale), F32(1.0), scale).astype(F32)
    out = _nvfp4_qdq_with_scale(xb, safe)
    out = np.where(zero, F32(0.0), out)
    return round_to(out.reshape(x.shape), dtype)


# ------------------------------------------------------------------------------------------------
# (3) quant and pack
# ------------------------------------------------------------------------------------------------
def pack_nvfp4(x, global_amax=None, block_amax=None, fp8_max_norm=448.0, block_size=16, wsf2=None):
    """NVFP4QTensor.quantize (quantization/qtensor/nvfp4_tensor.py:253-342); static branch
    (:139-161) when block_amax is given.  ``wsf2``: a caller-given weights_scaling_factor_2, used as is
    (:281-282, get_weights_scaling_factor :169-202); global_amax is then not read.  x last dim must be a
    multiple of block_size.  Returns (packed uint8 [..., K/2], scale bits uint8 [..., K/block_size], wsf2 float32)."""
    x = np.asarray(x, dtype=F32)
    k = x.shape[-1]
    xb = x.reshape(*x.shape[:-1], k // block_size, block_size)
    if wsf2 is not None and block_amax is not None:
        raise ValueError("wsf2 and block_amax are mutually exclusive")
    if global_amax is None and wsf2 is None:
        global_amax = reduce_amax(x)
    g = F32(0.0 if global_amax is None else global_amax)
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        if block_amax is None:
            s2 = F32(wsf2) if wsf2 is not None else F32(g / F32(6.0 * 448.0))
            bmax = np.max(np.abs(xb), axis=-1)
            pbs = (bmax / F32(F32(6.0) * s2)).astype(F32)
            pbs = np.where(pbs == 0, F32(1.0), pbs)
        else:
            s2 = F32(g / F32(6.0 * fp8_max_norm))
            psm = F32(g / F32(6.0))
            pbs = (np.asarray(block_amax, dtype=F32).reshape(xb.shape[:-1]) / F32(6.0)).astype(F32)
            pbs = np.where(pbs == 0, F32(1.0), pbs)
            pbs = ((pbs * F32(fp8_max_norm)).astype(F32) / psm).astype(F32)
        pbs = np.where(np.isnan(pbs), pbs, np.clip(pbs, F32(2.0**-9), F32(448.0))).astype(F32)
        bs_val, bs_bits = e4m3fn_torch_cast(pbs)
        denom = (bs_val * s2).astype(F32)
        y = (xb / denom[..., None]).astype(F32)
    codes = cast_fp4_codes(y).reshape(*x.shape[:-1], k)
    packed = (codes[..., 1::2] << 4) | codes[..., 0::2]
    return packed.astype(np.uint8), bs_bits, s2


def unpack_nvfp4(packed, scale_bits, wsf2, dtype="bf16"):
    """NVFP4QTensor.dequantize slow path (nvfp4_tensor.py:344-407)."""
    packed = np.asarray(packed, dtype=np.uint8)
    k = packed.shape[-1] * 2
    codes = np.empty((*packed.shape[:-1], k), dtype=np.uint8)
    codes[..., 1::2] = packed >> 4
    codes[..., 0::2] = packed & 0x0F
    lut = np.concatenate([E2M1_VALUES, -E2M1_VALUES]).astype(F32)
    lut[8] = F32(0.0)  # e2m1_values[8] is +0 (nvfp4_tensor.py:27)
    bs = k // np.asarray(scale_bits).shape[-1]
    vals = lut[codes].reshape(*packed.shape[:-1], k // bs, bs)
    s = (e4m3_from_bits(scale_bits) * F32(wsf2)).astype(F32)
    out = (vals * s[..., None]).astype(F32)
    return round_to(out.reshape(*packed.shape[:-1], k), dtype)


def _round_half_away(v):
    return np.where(v >= 0, np.floor(v + F32(0.5)), np.ceil(v - F32(0.5))).astype(F32)


def pack_int4_blockwise_cuda(x, block_size, dtype="bf16"):
    """INT4QTensor.quantize on the CUDA-extension branch (quantization/qtensor/int4_tensor.py:52-68
    + INT4_quantize_kernel, kernels/quantization/gemm/tensor_quant_gpu.cu:311-340): every
    intermediate is rounded to the tensor dtype T, roundf = half away from zero.
    Returns (packed uint8 [numel/2], scales [n_blocks, 1] as float32 values on the T grid)."""
    x = np.asarray(x, dtype=F32).ravel()
    xb = x.reshape(-1, block_size)
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        amax = reduce_amax(xb, axis=-1, keepdims=True)
        scales = rdiv_scalar(7.0, amax, dtype)  # int4_tensor.py:62
        v = round_to((xb * scales).astype(F32), dtype)
        v = np.maximum(F32(-8.0), np.minimum(F32(7.0), v))
        u = _round_half_away(round_to((v + F32(8.0)).astype(F32), dtype))
    q = u.astype(np.int32).ravel() & 0xF
    packed = ((q[0::2] << 4) | q[1::2]).astype(np.uint8)
    return packed, scales


def pack_int4_blockwise_cpu(x, block_size, dtype="bf16"):
    """INT4QTensor.quantize CPU branch (int4_tensor.py:70-84): RNE before the clamp."""
    x = np.asarray(x, dtype=F32).ravel()
    xb = x.reshape(-1, block_size)
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        amax = reduce_amax(xb, axis=-1, keepdims=True)
        scales = rdiv_scalar(7.0, amax, dtype)  # int4_tensor.py:62
        v = round_to((xb * scales).astype(F32), dtype).ravel()
        u = np.clip(np.rint(v), -8, 7) + 8
    q = u.astype(np.uint8)
    return ((q[0::2] << 4) | q[1::2]).astype(np.uint8), scales


def unpack_int4_blockwise(packed, scales, block_size, dtype="bf16"):
    """INT4_dequantize_kernel (tensor_quant_gpu.cu:262-279): (nibble - 8) / scale in T."""
    packed = np.asarray(packed, dtype=np.uint8).ravel()
    first = (packed >> 4).astype(F32) - F32(8.0)
    second = (packed & 0xF).astype(F32) - F32(8.0)
    vals = np.stack([first, second], axis=-1).reshape(-1, block_size)
    with np.errstate(divide="ignore", invalid="ignore"):
        out = (vals / np.asarray(scales, dtype=F32).reshape(-1, 1)).astype(F32)
    return round_to(out, dtype).ravel()


def pack_int4_export(w, scale, w_dtype="bf16", scale_dtype="f32"):
    """pack_int4_in_uint8 (export/quant_utils.py:792-833): w [out, in], scale [out, in/block].
    Division in the promoted dtype (bf16/f32 -> f32; same dtype -> that dtype), round half even."""
    w = np.asarray(w, dtype=F32)
    scale = np.asarray(scale, dtype=F32)
    out_dim, in_dim = w.shape
    block = in_dim // scale.shape[-1]
    s_full = scale[:, np.arange(in_dim) // block]
    res_dtype = w_dtype if w_dtype == scale_dtype else "f32"
    with np.errstate(divide="ignore", invalid="ignore"):
        q = np.clip(np.rint(round_to((w / s_full).astype(F32), res_dtype)), -8, 7).astype(np.int8)
    t = q.T.reshape(in_dim, out_dim // 2, 2)
    val0 = t[..., 0] & 0x0F
    val1 = t[..., 1] & 0x0F
    packed = (val0 | (val1 << 4)).astype(np.int8)
    return np.ascontiguousarray(packed.T).view(np.uint8)


def pack_fp8(x, scale, outer=1, x_dtype="bf16", scale_dtype="bf16", scale_is_0dim=False):
    """(x / scale).to(float8_e4m3fn): FP8QTensor.quantize (quantization/qtensor/fp8_tensor.py:107)
    and to_quantized_weight (export/quant_utils.py:854-866).  The quotient is rounded to torch's
    result dtype first: x's dtype when scale has the same dtype or is a 0-dim tensor, else f32."""
    x = np.asarray(x, dtype=F32)
    s = _bcast_amax(x, scale, outer)
    res_dtype = x_dtype if (scale_dtype == x_dtype or scale_is_0dim) else "f32"
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        q = canonical_nan(round_to((x / s).astype(F32), res_dtype))   # x / scale on the GPU: -NaN -> 0x7f
    _, bits = e4m3fn_torch_cast(q)
    return bits


def unpack_fp8(bits, scale, outer=1, dtype="bf16"):
    """FP8QTensor.dequantize (fp8_tensor.py:115-155): q.to(dtype) * scale.to(dtype) in dtype."""
    v = round_to(e4m3_from_bits(bits), dtype)
    s = round_to(_bcast_amax(v, scale, outer), dtype)
    return round_to((v * s).astype(F32), dtype)


def pack_int8(x, scale, outer=1, x_dtype="bf16", scale_dtype="bf16", scale_is_0dim=False):
    """(x / scale).round().clamp(-128, 127).to(int8): INT8QTensor.quantize (quantization/qtensor/int8_tensor.py:86).
    The quotient is rounded to torch's result dtype first (as in pack_fp8); round = half to even."""
    x = np.asarray(x, dtype=F32)
    s = _bcast_amax(x, scale, outer)
    res_dtype = x_dtype if (scale_dtype == x_dtype or scale_is_0dim) else "f32"
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        q = round_to((x / s).astype(F32), res_dtype)
    q = np.clip(np.rint(q), -128, 127)
    return np.where(np.isnan(q), 0, q).astype(np.int8)


def unpack_int8(q, scale, outer=1, dtype="bf16"):
    """INT8QTensor.dequantize (int8_tensor.py:88-124): q.to(dtype) * scale.to(dtype) in dtype."""
    v = np.asarray(q, dtype=np.int8).astype(F32)
    s = round_to(_bcast_amax(v, scale, outer), dtype)
    return round_to((v * s).astype(F32), dtype)


# ------------------------------------------------------------------------------------------------
# scale searches
# ------------------------------------------------------------------------------------------------
def scale_cols(x, s, dtype="bf16"):
    """inputs * pre_quant_scale, both in the tensor dtype (nn/modules/tensor_quantizer.py:1143-1144)."""
    return round_to((np.asarray(x, dtype=F32) * np.asarray(s, dtype=F32).reshape(1, -1)).astype(F32), dtype)


def awq_scale_fake_quant(w, s, block_size, num_bits=4, narrow_range=False, dtype="bf16"):
    """One alpha step of awq_lite's patched forward on the weight side (model_calib.py:1552-1554):
    W * s -> dynamic per-block amax (tensor_quantizer.py:746-748) -> integer fake quant over
    [n_blocks, block] with axis 0 (kernels/quantization/gemm/tensor_quant_gpu.cu:102-118)."""
    ws = scale_cols(w, s, dtype)
    wb = ws.reshape(-1, block_size)
    amax = reduce_amax(wb, axis=1)
    return fake_quant_int(wb, amax, num_bits, False, narrow_range, block_size, dtype).reshape(ws.shape)


def awq_weight_scale(w, block_size, dtype="bf16"):
    """get_weight_scale (model_calib.py:1453-1469): mean over rows of |W| / (blockamax + tiny),
    arithmetic in the weight dtype, result cast to float32."""
    w = np.asarray(w, dtype=F32)
    tiny = F32(6.103515625e-05) if dtype == "f16" else F32(1.17549435e-38)
    wb = np.abs(w).reshape(-1, block_size)
    den = round_to((wb.max(axis=1, keepdims=True) + tiny).astype(F32), dtype)
    with np.errstate(divide="ignore", invalid="ignore"):
        ratio = round_to((wb / den).astype(F32), dtype).reshape(w.shape)
    return round_to(ratio.astype(np.float64).mean(0).astype(F32), dtype)


def awq_get_scale(x_max, w_max, alpha):
    """get_scale (model_calib.py:1474-1487), fp32."""
    x_max = np.asarray(x_max, dtype=F32)
    w_max = np.asarray(w_max, dtype=F32)
    tiny = F32(1.17549435e-38)
    with np.errstate(divide="ignore", invalid="ignore"):
        s = (np.power(x_max, F32(alpha)) / (np.power(w_max, F32(1 - alpha)) + tiny)).astype(F32)
    s = np.clip(s, F32(1e-4), F32(1e4))
    return (s / np.sqrt(s.max() * s.min())).astype(F32)


def smoothquant_scale(act_amax, weight_colmax, alpha=1.0):
    """smoothquant.postprocess (model_calib.py:1309-1335): per-input-channel scale_a."""
    a = np.asarray(act_amax, dtype=F32).ravel()
    w = np.asarray(weight_colmax, dtype=F32).ravel()
    with np.errstate(divide="ignore", invalid="ignore"):
        s = (np.power(w, F32(1 - alpha)) / np.power(a, F32(alpha))).astype(F32)
    eps = F32(1.0 / (1 << 31))
    if s.min() <= eps:
        s = np.where(a <= eps, F32(1.0), s)
    return np.clip(s, F32(1e-4), F32(1e4)).astype(F32)


def mse_sweep_losses(x, amax0, mult, num_bits=8, unsigned=False, narrow_range=False):
    """MseCalibrator.collect (calib/mse.py:84-119), per-tensor: loss[k] = sum (fq(x; amax0*mult[k]) - x)^2
    with the fake quant evaluated in fp32 (x is upcast first, :93).  num_bits=0 selects FP8-E4M3."""
    x = np.asarray(x, dtype=F32)
    out = []
    for m in np.asarray(mult, dtype=F32):
        amax = F32(F32(amax0) * m)
        xq = fake_quant_fp8(x, amax, 1, "f32") if num_bits == 0 else \
            fake_quant_int(x, amax, num_bits, unsigned, narrow_range, 1, "f32")
        out.append(np.sum((x.astype(np.float64) - xq.astype(np.float64)) ** 2))
    return np.array(out, dtype=np.float64)


def fp8_scale_candidates(cuda_rule=False):
    """kernels/quantization/gemm/_fp8_scale_candidates.py: 126 positive finite e4m3 values / 448.  ATen divides a
    tensor by a Python scalar with an IEEE division on CPU (the committed fixtures) and with a multiply by
    fl(1 / 448) on CUDA (``cuda_rule=True``: what a GPU run of the reference sweeps)."""
    v = e4m3_from_bits(np.arange(1, 127, dtype=np.uint8))
    if cuda_rule:
        return (v * (F32(1.0) / F32(448.0))).astype(F32)
    return (v / F32(448.0)).astype(F32)


def nvfp4_fp8_scale_sweep(w, global_amax, cuda_rule=False):
    """nvfp4_fp8_scale_sweep (kernels/quantization/gemm/nvfp4_fp8_sweep.py:59-160) ==
    NVFP4MSECalibrator's 126-step reference sweep (calib/mse.py:175-311): per 16-block argmin over
    candidates of sum (|w| - q(|w| / s) * s)^2, s = c * global_amax / 6; first minimum wins;
    returns best_amax = global_amax * c.  Per-block loss summed with a pairwise fp32 tree."""
    w = np.asarray(w, dtype=F32)
    a = np.abs(w).reshape(-1, 16)
    g = F32(global_amax)
    cand = fp8_scale_candidates(cuda_rule)
    best_loss = np.full(a.shape[0], np.inf, dtype=F32)
    best_k = np.zeros(a.shape[0], dtype=np.int64)
    for k, c in enumerate(cand):
        scale = F32(F32(c * g) / F32(6.0))
        s = F32(1.0) if scale == 0 else scale
        with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
            q = e2m1_round_mag((a / s).astype(F32))
            d = (a - (q * s).astype(F32)).astype(F32)
            t = (d * d).astype(F32)
        n = 8
        while n >= 1:
            t = (t[:, :n] + t[:, n : 2 * n]).astype(F32)
            n //= 2
        loss = t[:, 0]
        better = loss < best_loss
        best_loss = np.where(better, loss, best_loss)
        best_k = np.where(better, k, best_k)
    return (g * cand[best_k]).astype(F32)


def nvfp4_block_log2_hist(x, num_bins=512, log2_min=-40.0, log2_max=40.0):
    """NVFP4ActHeadroomCalibrator.collect (calib/nvfp4_act_headroom.py:110-149): (int64 histogram of the
    log2 bin of every non-zero 16-block amax, running max).  log2 in fp32 (libm; the CUDA log2f may
    differ in the last ulp, which only matters for a value sitting on a bin edge)."""
    x = np.asarray(x, dtype=F32)
    b = reduce_block_amax(x, 16).ravel()
    nz = b[b > 0]
    frac = ((np.log2(nz).astype(F32) - F32(log2_min)) / F32(log2_max - log2_min)).astype(F32)
    # clamp before the integer conversion: +inf (an inf block) lands in the top bin, as CUDA's saturating float -> int64
    # conversion and the kernel put it
    idx = np.clip(np.floor((frac * F32(num_bins)).astype(F32)), 0, num_bins - 1).astype(np.int64)
    return np.bincount(idx, minlength=num_bins).astype(np.int64), (b.max() if b.size else F32(0))


# ------------------------------------------------------------------------------------------------
# (4c) host-side amax searches of the calibrators
# ------------------------------------------------------------------------------------------------
def mse_sweep_losses_rows(x, amax0, mult, num_bits=8, unsigned=False, narrow_range=False, cand_dtype="bf16",
                          cpu_twin=False, round_mult=None):
    """MseCalibrator.collect (calib/mse.py:84-119) with one amax per row: loss[k, r] = sum_j (fq(x[r,j]; a_k(r)) -
    x[r,j])^2, a_k(r) = round_A(amax0[r] * m_k) -- ``_compute_candidate_amax`` (:80-84) multiplies the
    [R,1] amax (dtype A) by a 0-dim fp32 candidate, which torch evaluates in dtype A; m_k = mult[k] on CPU (ATen's
    reduced-float CPU mul keeps the original fp32 scalar -- pinned by the CPU-executed fixture) and round_A(mult[k])
    on CUDA (the 0-dim CUDA operand is cast to A on load): ``round_mult`` (default: not cpu_twin).  The fake quant runs on the
    fp32 copy of x (:93) and is not rounded back.  num_bits=0: FP8-E4M3.  cpu_twin: ``_tensor_quant`` / ``fp8_eager``
    (what the CPU-executed fixture used) instead of the CUDA kernels' formulas."""
    x = np.asarray(x, dtype=F32)
    a0 = np.asarray(amax0, dtype=F32).reshape(-1, 1)
    out = []
    round_mult = (not cpu_twin) if round_mult is None else round_mult
    for m in np.asarray(mult, dtype=F32):
        mk = round_to(m, cand_dtype) if round_mult else m
        amax = round_to((a0 * mk).astype(F32), cand_dtype)
        if num_bits == 0:
            xq = fake_quant_fp8(x, amax, x.shape[1], "f32", eager=cpu_twin)
        elif cpu_twin:
            xq = tensor_quant_cpu(x, amax, num_bits, unsigned, narrow_range, "f32")
        else:
            xq = fake_quant_int(x, amax, num_bits, unsigned, narrow_range, x.shape[1], "f32")
        d = (x - xq).astype(F32)
        out.append(np.sum((d * d).astype(F32).astype(np.float64), axis=1))
    return np.array(out, dtype=np.float64)


def hist_amax_percentile(hist, edges, percentile):
    """_compute_amax_percentile (calib/histogram.py:325-343): sequential fp64 cumsum of hist / total, left
    searchsorted."""
    hist = np.asarray(hist)
    total = hist.sum()
    cdf = np.cumsum(hist / total)
    return F32(edges[int(np.searchsorted(cdf, percentile / 100))])


def hist_entropy_divergences(hist, num_bits, unsigned=False, stride=1, start_bin=128):
    """The KL divergence per candidate of _compute_amax_entropy (calib/histogram.py:210-278), vectorised per
    candidate (the reference loops in Python over bins); fp64 like the reference."""
    bins = np.asarray(hist).astype(np.float64).copy()
    bins[0] = bins[1]
    nq = 1 << (num_bits - 1 + int(unsigned))
    divs = []
    for i in range(start_bin, len(bins) + 1, stride):
        space = np.linspace(0, i, num=nq + 1)
        dig = np.digitize(np.arange(i), space) - 1
        nz = bins[:i] != 0
        sums = np.bincount(dig[nz], weights=bins[:i][nz], minlength=nq)
        cnts = np.bincount(dig[nz], minlength=nq)
        avg = np.divide(sums, cnts, out=np.zeros_like(sums), where=cnts > 0)
        new_density = np.where(nz, avg[dig], 0.0)
        ref = bins[:i].copy()
        ref[-1] += bins[i:].sum()
        p = ref / ref.sum() if ref.sum() else ref
        q = new_density / new_density.sum() if new_density.sum() else new_density
        with np.errstate(divide="ignore", invalid="ignore"):
            kl = np.where(p > 0, p * np.log(p / q), 0.0).sum()      # scipy.stats.entropy(p, q) = sum rel_entr
        divs.append(kl)
    return np.array(divs)


def hist_amax_entropy(hist, edges, num_bits, unsigned=False, stride=1, start_bin=128):
    divs = hist_entropy_divergences(hist, num_bits, unsigned, stride, start_bin)
    last = len(divs) - 1 - int(np.argmin(divs[::-1]))               # the LAST minimum (:276)
    return F32(edges[last * stride + start_bin])


def hist_mse_losses(hist, edges, num_bits, unsigned=False, stride=1, start_bin=128):
    """_compute_amax_mse (calib/histogram.py:281-322) with the call site repaired (bias=None; see
    oracle/gen_golden.py main_calibrators): per candidate bin centre c_i, mean((fq(c; amax=c_i) - c)^2 * counts).
    Fake quant with the default ``narrow_range=True``; num_bits=0: FP8-E4M3 (CUDA-extension scale rule)."""
    counts = np.asarray(hist).astype(F32)
    e = np.asarray(edges, dtype=F32)
    centers = ((e[1:] + e[:-1]).astype(F32) / F32(2)).astype(F32)
    losses = []
    for i in range(start_bin, len(centers), stride):
        amax = centers[i]
        q = fake_quant_fp8(centers, amax, 1, "f32") if num_bits == 0 else \
            fake_quant_int(centers, amax, num_bits, unsigned, True, 1, "f32")
        d = (q - centers).astype(F32)
        losses.append(F32(np.sum(((d * d).astype(F32) * counts).astype(F32).astype(np.float64)) / len(centers)))
    return np.array(losses, dtype=F32), centers


def hist_amax_mse(hist, edges, num_bits, unsigned=False, stride=1, start_bin=128):
    losses, centers = hist_mse_losses(hist, edges, num_bits, unsigned, stride, start_bin)
    return centers[start_bin + int(np.argmin(losses)) * stride]


def act_headroom_amax(hist, running_max, anchor_percentile=1.0, upper_percentile=99.99, rho=16384.0,
                      num_bins=512, log2_min=-40.0, log2_max=40.0):
    """NVFP4ActHeadroomCalibrator.compute_amax / _percentile (calib/nvfp4_act_headroom.py:151-205):
    amax = max(rho * P_anchor, P_upper) with percentiles read at bin centres of the log2 histogram; the anchor
    ignores bins below upper / 1e6."""
    def bin_index(v):
        frac = F32((F32(np.log2(F32(v))) - F32(log2_min)) / F32(log2_max - log2_min))
        return int(np.clip(np.floor(F32(frac * F32(num_bins))), 0, num_bins - 1))

    def pct(p, floor_value=None):
        counts = np.asarray(hist).astype(F32).copy()
        if floor_value is not None and floor_value > 0:
            counts[: bin_index(floor_value)] = 0
        total = counts.sum(dtype=F32)
        if total <= 0:
            return None
        target = F32(p / 100.0 * float(total))
        cdf = np.cumsum(counts, dtype=F32)
        idx = int(np.clip(np.searchsorted(cdf, target), 0, num_bins - 1))
        return float(2.0 ** (log2_min + (idx + 0.5) / num_bins * (log2_max - log2_min)))

    rmax = float(F32(running_max))
    upper = rmax if upper_percentile >= 100.0 else pct(upper_percentile)
    anchor = pct(anchor_percentile, upper / 1e6 if upper else None) if upper else None
    if not upper or upper <= 0 or not anchor or anchor <= 0:
        return F32(rmax)
    return F32(max(rho * anchor, upper))


# ------------------------------------------------------------------------------------------------
# (5) MX formats: power-of-two (E8M0) block scales
# ------------------------------------------------------------------------------------------------
# format ids follow `enum class Types` (kernels/quantization/gemm/tensor_quant_mx.h:40)
MX_E4M3, MX_E5M2, MX_INT8, MX_E0M3, MX_E1M2, MX_E3M0, MX_E2M1, MX_E3M2, MX_E2M3, MX_E8M0 = range(10)
MX_FORMAT_MAX = {MX_E4M3: 448.0, MX_E5M2: 57344.0, MX_INT8: 127.0, MX_E0M3: 7.0, MX_E1M2: 3.5,
                 MX_E3M0: 16.0, MX_E2M1: 6.0, MX_E3M2: 28.0, MX_E2M3: 7.5}   # tensor_quant_mx.h:193-218


def _minifloat_values(ebits, mbits, bias):
    """All non-negative values of a sign/exponent/mantissa format without inf/NaN codes."""
    vals = []
    for code in range(1 << (ebits + mbits)):
        e, m = code >> mbits, code & ((1 << mbits) - 1)
        vals.append(m * 2.0 ** (1 - bias - mbits) if e == 0 else (1 + m / (1 << mbits)) * 2.0 ** (e - bias))
    return np.array(vals, dtype=F32)


_MX_TABLES = {  # same grids as the value tables of tensor_quant_mx.h:42-74, generated from the bit layouts
    MX_E2M1: _minifloat_values(2, 1, 1), MX_E1M2: _minifloat_values(1, 2, 0),
    MX_E0M3: np.arange(8, dtype=F32), MX_E3M0: _minifloat_values(3, 0, 3),
    MX_E3M2: _minifloat_values(3, 2, 3), MX_E2M3: _minifloat_values(2, 3, 1),
}


def _e5m2_round(a):
    """|v| -> float(e5m2_rne_satfinite(|v|)) (__nv_fp8_e5m2, tensor_quant_mx.h:80-82)."""
    a = np.asarray(a, dtype=F32)
    with np.errstate(invalid="ignore", over="ignore"):
        b = a.view(np.uint32).astype(np.uint64)
        r = (b + 0xFFFFF + ((b >> 21) & 1)) & ~np.uint64(0x1FFFFF)   # keep 2 mantissa bits, RNE
        normal = (r & 0xFFFFFFFF).astype(np.uint32).view(F32)
        sub = np.rint(a * F32(65536.0)) / F32(65536.0)                # subnormal grid 2^-16
        out = np.where(a < F32(2.0**-14), sub, normal).astype(F32)
        out = np.minimum(out, F32(57344.0))
    return np.where(np.isnan(a), F32(np.nan), out).astype(F32)


def convert_to_exmy(x, fmt):
    """convert_to_types (tensor_quant_mx.h:163-190): sign-symmetric rounding of x onto the element
    grid.  Table formats round to nearest even (E3M0: ties away from zero) and saturate inf AND NaN
    to the largest value (:120-160); E4M3/E5M2 keep NaN and saturate (cuda_fp8.h); INT8 is
    rint + clamp to +-127 (:84-93; NaN is undefined there and maps to 0 here, like cvt.rni on the GPU)."""
    x = np.asarray(x, dtype=F32)
    if fmt == MX_E4M3:
        return e4m3_round(x)
    neg = x < 0
    a = np.abs(x)
    if fmt == MX_E5M2:
        return np.copysign(_e5m2_round(a), x).astype(F32)
    if fmt == MX_INT8:
        with np.errstate(invalid="ignore"):
            r = np.where(np.isnan(a), F32(0), np.minimum(np.rint(a), F32(127.0))).astype(F32)
        return np.where(neg & (r > 0), -r, r).astype(F32)    # through an int: no negative zero
    if True:
        vals = _MX_TABLES[fmt]
        bounds = ((vals[1:].astype(np.float64) + vals[:-1].astype(np.float64)) / 2).astype(F32)
        idx = np.searchsorted(bounds, a, side="left")        # ties -> lower index
        safe = np.minimum(idx, len(bounds) - 1)
        tie = (idx < len(bounds)) & (a == bounds[safe])
        up = tie if fmt == MX_E3M0 else (tie & (idx % 2 == 1))
        idx = np.where(up, idx + 1, idx)
        idx = np.where(np.isnan(a) | np.isinf(a), len(vals) - 1, idx)
        r = vals[idx]
    return np.where(neg, -r, r).astype(F32)


def e8m0_exponent_nv(amax, fmt):
    """compute_scale_e8m0_NV (kernels/quantization/gemm/tensor_quant_mx.cu:103-131): the exponent e
    with unscale = 2^e, scale = 2^-e; e = ceil(log2(fp32(amax / dmax))) read off the bits of the
    IEEE-rounded ratio (the reference builds with --use_fast_math; IEEE division is what the source says)."""
    amax = np.asarray(amax, dtype=F32)
    with np.errstate(all="ignore"):
        ratio = (amax / F32(MX_FORMAT_MAX[fmt])).astype(F32)
    bits = ratio.view(np.uint32)
    ex = ((bits >> 23) & 0xFF).astype(np.int32)
    sig = (bits & 0x7FFFFF).astype(np.int64)
    up = (sig > 0) & (ex != 0xFE) & ~((ex == 0) & (sig <= 0x400000))
    return np.where(up, ex - 126, ex - 127).astype(np.int32)


def fake_quant_mx(x, block_size, fmt, dtype="bf16"):
    """fused_amax_convert with an E8M0 scale (tensor_quant_mx.cu:240-291, 320-366; quantize :36-54;
    compute_scale :134-151).  Blocks run along the last dim, a ragged tail block is padded with
    zeros.  Block amax ignores NaN (fmaxf); amax 0 / inf / NaN -> scale 1.
    `sign` is uninitialised in the reference for x == 0 and NaN; this restatement uses +1."""
    x = np.asarray(x, dtype=F32)
    k = x.shape[-1]
    pad = (-k) % block_size
    xp = np.concatenate([x, np.zeros((*x.shape[:-1], pad), F32)], axis=-1) if pad else x
    xb = xp.reshape(*x.shape[:-1], -1, block_size)
    with np.errstate(all="ignore"):
        amax = nan_skip_absmax(xb, axis=-1)
        bad = (amax == 0) | np.isinf(amax) | np.isnan(amax)
        e = np.where(bad, 0, e8m0_exponent_nv(np.where(bad, F32(1), amax), fmt))
        scale = np.ldexp(F32(1), -e).astype(F32)[..., None]
        unscale = np.ldexp(F32(1), e).astype(F32)[..., None]
        q = convert_to_exmy((np.abs(xb) * scale).astype(F32), fmt)
        out = (q * unscale).astype(F32)
        out = np.where(xb < 0, -out, out)
    out = out.reshape(xp.shape)[..., :k]
    return round_to(out, dtype)


def _ceil_log2_clamped(r):
    """clamp(ceil(log2(r)), -127, 127) for r > 0, exact (frexp), else -127: MXFP8QTensor.
    _compute_e8m0_exponent (quantization/qtensor/mxfp8_tensor.py:42-65) without libm rounding."""
    r = np.asarray(r, dtype=F32)
    with np.errstate(all="ignore"):
        m, ex = np.frexp(r.astype(np.float64))
        e = np.where(m == 0.5, ex - 1, ex).astype(np.float64)
        e = np.where(np.isinf(r), 127.0, e)
        e = np.where(r > 0, e, -127.0)
    return np.clip(e, -127, 127).astype(np.int32)


def pack_mxfp8(x, scale_bytes=None):
    """MXFP8QTensor.quantize / quantize_with_scale (mxfp8_tensor.py:150-215): block 32 along the last
    dim (zero padded), E8M0 byte = e + 127, data = clamp(x * 2^-e, +-448).to(float8_e4m3fn).
    Returns (e4m3 bits uint8 [..., K], scale bytes uint8 [..., ceil(K/32)])."""
    x = np.asarray(x, dtype=F32)
    k = x.shape[-1]
    pad = (-k) % 32
    xp = np.concatenate([x, np.zeros((*x.shape[:-1], pad), F32)], axis=-1) if pad else x
    xb = xp.reshape(*x.shape[:-1], -1, 32)
    with np.errstate(all="ignore"):
        if scale_bytes is None:
            amax = np.max(np.abs(xb), axis=-1)                       # torch max: NaN propagates
            e = _ceil_log2_clamped((amax / F32(448.0)).astype(F32))
            scale_bytes = (e + 127).astype(np.uint8)
        sf = np.exp2(127.0 - scale_bytes.astype(np.float64)).astype(F32)
        scaled = canonical_nan((xb * sf[..., None]).astype(F32))     # x * 2^-e on the GPU: -NaN -> 0x7f
        scaled = np.where(np.isnan(scaled), scaled, np.clip(scaled, F32(-448.0), F32(448.0)))
    _, bits = e4m3fn_torch_cast(scaled)
    return bits.reshape(xp.shape)[..., :k], np.asarray(scale_bytes, dtype=np.uint8)


def unpack_mxfp8(bits, scale_bytes, dtype="bf16"):
    """MXFP8QTensor.dequantize (mxfp8_tensor.py:217-262)."""
    bits = np.asarray(bits, dtype=np.uint8)
    k = bits.shape[-1]
    pad = (-k) % 32
    v = e4m3_from_bits(bits)
    vp = np.concatenate([v, np.zeros((*v.shape[:-1], pad), F32)], axis=-1) if pad else v
    vb = vp.reshape(*v.shape[:-1], -1, 32)
    d = np.exp2(np.asarray(scale_bytes).astype(np.float64) - 127.0).astype(F32)
    with np.errstate(all="ignore"):
        out = (vb * d[..., None]).astype(F32).reshape(vp.shape)[..., :k]
    return round_to(out, dtype)


def pack_mxfp4(x, block_size=32):
    """MXFP4QTensor.quantize (quantization/qtensor/mxfp4_tensor.py:37-83): flat blocks (numel must
    divide), e = ceil(max(log2(amax / 6), -127)), codes: sign bit set unless x > 0 (zeros get code 8,
    :47-48), magnitude = number of E2M1 bounds strictly below |x| (exact ties round DOWN, :49-51).
    Returns (packed uint8 [..., K/2] odd element in the high nibble, scale bytes [numel/bs, 1])."""
    x = np.asarray(x, dtype=F32)
    xb = x.reshape(-1, block_size)
    with np.errstate(all="ignore"):
        amax = np.max(np.abs(xb), axis=-1, keepdims=True)
        r = (amax / F32(6.0)).astype(F32)
        m, ex = np.frexp(r.astype(np.float64))
        e = np.where(m == 0.5, ex - 1, ex).astype(np.float64)
        e = np.where(r > 0, np.maximum(e, -127.0), -127.0)
        y = (xb / np.exp2(e).astype(F32)).astype(F32)
    sign_bit = (~(y > 0)).astype(np.uint8)
    ordv = np.searchsorted(E2M1_BOUNDS, np.abs(y), side="left").astype(np.uint8)
    codes = ((sign_bit << 3) + ordv).astype(np.uint8).reshape(x.shape)
    packed = ((codes[..., 1::2] << 4) + codes[..., 0::2]).astype(np.uint8)
    return packed, (e + 127).astype(np.uint8)


def unpack_mxfp4(packed, scale_bytes, block_size=32, dtype="bf16"):
    """MXFP4QTensor.dequantize (mxfp4_tensor.py:85-144); code 8 decodes to -0.0."""
    packed = np.asarray(packed, dtype=np.uint8)
    k = packed.shape[-1] * 2
    codes = np.empty((*packed.shape[:-1], k), dtype=np.uint8)
    codes[..., 0::2] = packed & 0x0F
    codes[..., 1::2] = packed >> 4
    sign = (1.0 - 2.0 * ((codes & 8) >> 3)).astype(F32)
    v = (sign * E2M1_VALUES[codes & 7]).astype(F32).reshape(-1, block_size)
    sf = np.exp2(np.asarray(scale_bytes).astype(np.float64) - 127.0).astype(F32).reshape(-1, 1)
    with np.errstate(all="ignore"):
        out = (v * sf).astype(F32).reshape(codes.shape)
    return round_to(out, dtype)


# ------------------------------------------------------------------------------------------------
# (6) NF4 (CUDA-extension semantics; the reference's CPU fallback rounds the table to the tensor dtype
#     and is a different function -- the GPU kernels are pinned against the compiled extension on the GPU)
# ------------------------------------------------------------------------------------------------
NF4_LUT = np.array([-1.0, -0.6962, -0.5251, -0.3949, -0.2844, -0.1848, -0.0911, 0.0, 0.0796, 0.1609, 0.2461,
                    0.3379, 0.4407, 0.5626, 0.7230, 1.0], dtype=F32)      # tensor_quant_gpu.cu:142-144


def pack_nf4(x, block_size, dtype="bf16", scales=None):
    """NF4QTensor.quantize (quantization/qtensor/nf4_tensor.py:74-127) + NF4_quantize_kernel
    (kernels/quantization/gemm/tensor_quant_gpu.cu:198-236): scales = block |x| max, v = T(x / scale),
    index = first minimum of |LUT[i] - v| in fp32 (NaN / inf distances never win -> 0), byte = first << 4 | second."""
    xb = np.asarray(x, dtype=F32).reshape(-1, block_size)
    if scales is None:
        scales = np.max(np.abs(xb), axis=1, keepdims=True)
    s = np.asarray(scales, dtype=F32).reshape(-1, 1)
    with np.errstate(all="ignore"):
        v = round_to((xb / s).astype(F32), dtype)
        d = np.abs((NF4_LUT[None, None, :] - v[..., None]).astype(F32))
        best = d[..., 0].copy()
        idx = np.zeros(v.shape, dtype=np.uint8)
        for i in range(1, 16):
            better = d[..., i] < best
            best = np.where(better, d[..., i], best)
            idx = np.where(better, np.uint8(i), idx)
    idx = idx.reshape(-1)
    return ((idx[0::2] << 4) | idx[1::2]).astype(np.uint8), s.astype(F32)


def unpack_nf4(packed, scales, block_size):
    """NF4_dequantize_kernel (tensor_quant_gpu.cu:146-165): bf16(bf16(LUT[idx]) * bf16(scale)), always bf16."""
    packed = np.asarray(packed, dtype=np.uint8).reshape(-1)
    idx = np.empty(packed.size * 2, dtype=np.uint8)
    idx[0::2] = packed >> 4
    idx[1::2] = packed & 0xF
    s = round_bf16(np.asarray(scales, dtype=F32).reshape(-1))
    with np.errstate(all="ignore"):
        out = (round_bf16(NF4_LUT)[idx].reshape(-1, block_size) * s[:, None]).astype(F32)
    return round_bf16(out.reshape(-1))


# ------------------------------------------------------------------------------------------------
# (7) affine-bias statistics (quantization/calib/bias.py:25-149)
# ------------------------------------------------------------------------------------------------
def bias_reduce_dims(ndim, axis):
    """The dims compute_maxmin REDUCES (bias.py:40-44): those listed in ``axis`` (None: all)."""
    if axis is None:
        return tuple(range(ndim))
    return tuple(i for i in range(ndim) if i in axis or (i - ndim) in axis)


def bias_maxmin(x, axis):
    """compute_maxmin (bias.py:25-52): signed max / min, keepdim (0-dim for axis None)."""
    x = np.asarray(x, dtype=F32)
    if axis is None:
        return x.max(), x.min()
    red = bias_reduce_dims(x.ndim, axis)
    return x.max(axis=red, keepdims=True), x.min(axis=red, keepdims=True)


def bias_mean(x, axis, dtype="bf16"):
    """compute_mean_bias (bias.py:61-76): torch.mean accumulates in fp32 and rounds to the tensor dtype; the
    summation order is ATen's, so this float64 restatement is exact only up to the final rounding."""
    x = np.asarray(x, dtype=F32)
    red = None if axis is None else bias_reduce_dims(x.ndim, axis)
    m = x.astype(np.float64).mean() if red is None else x.astype(np.float64).mean(axis=red, keepdims=True)
    return round_to(np.asarray(m, dtype=F32), dtype)
