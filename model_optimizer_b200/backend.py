"""Drop-in installation into a real ``modelopt`` (when it is importable): the sanctioned hooks of
SURVEY.md 8(b), plus the module-level functions the hooks cannot reach.

1. ``register_quant_backend("b200", entrypoint)`` (nn/modules/tensor_quantizer.py:87-109): fake quant of
   any quantizer whose config carries ``backend: "b200"`` runs the fused sm_90a kernels.
2. ``calibrator`` config field (config.py:599-614): ``B200MaxCalibrator`` / ``B200HistogramCalibrator``
   subclass the reference's ``_Calibrator`` so ``TensorQuantizer.collect`` reaches the collect kernels.
3. ``_register_fp8_sweep_calibrator("b200", factory)`` (model_calib.py:166-179): the per-block FP8-scale
   sweep of ``mse_calibrate(fp8_scale_sweep=True)`` runs ``b200q_nvfp4_fp8_scale_sweep``.
4. Extension-module ABI (extensions.py:28-72): ``get_cuda_ext`` / ``get_cuda_ext_fp8`` / ``get_cuda_ext_mx``
   are replaced by shim modules exporting the same names (``fake_tensor_quant``, ``fake_e4m3fy``,
   ``fused_amax_convert`` ...), so the reference's own autograd Functions and ``INT4QTensor`` call this engine
   even without the ``backend`` field.
5. Not reachable through a hook, so rebound by name (``install(patch_functions=True)``; ``uninstall()`` restores):
   * ``static_blockwise_fp4_fake_quant`` in ``nn/modules/tensor_quantizer.py`` --
     ``StaticBlockScaleQuantizer._fake_quantize`` (:1708-1731) calls it without consulting ``backend``;
   * ``MseCalibrator`` as named in ``model_calib.py`` (:720-728, constructed directly, no registry): the
     multiplier search of ``mse_calibrate`` runs ``b200q_mse_sweep[_rows]`` for quantizers on the b200 backend;
   * ``NVFP4QTensor.quantize`` / ``FP8QTensor.quantize`` (qtensor/nvfp4_tensor.py:253, qtensor/fp8_tensor.py:41):
     the weight quant-and-pack of ``mtq.compress`` / ``TensorQuantizer._real_quantize`` (:796-887) is pure ATen
     in the reference; here one pack kernel each.  Calls outside the engine's scope (CPU tensors,
     pre-computed block scales, ``keep_high_precision``) are handed back to the host application's own function;
   * ``normalized_hadamard_transform`` as named in ``nn/modules/tensor_quantizer.py`` (:67, called by
     ``_rotate_inputs`` :664-668): every ``rotate`` config on CUDA tensors runs ``b200q_hadamard`` instead of needing
     the external ``fast_hadamard_transform`` package (other inputs go to the host application's own function);
   * ``NVFP4ActHeadroomCalibrator`` as named in ``model_calib.py`` (constructed directly by ``nvfp4_act_headroom``):
     a subclass whose ``collect`` is one ``b200q_nvfp4_block_log2_hist`` launch for CUDA inputs in fp32 / fp16 /
     bf16 with blocks of 16 (the reference: a clone, two reductions, a host-synchronising compaction, ``log2`` and
     ``bincount`` per batch); other inputs run the reference's own methods.
6. ``register_gptq_helper("b200", B200GPTQHelper)`` (utils/calib_utils.py:316-326): ``gptq`` builds this
   ``GPTQHelper`` subclass for weight quantizers on the b200 backend.  Its ``_blockwise_update`` runs the GPTQ column
   kernel (``b200q_gptq_block``, one launch per block, plus the reference's trailing ``addmm_``) for the formats the
   kernel covers, and the reference's own loop for everything else.  The reference's ``layerwise_calibrate`` thus
   gives layerwise GPTQ on the kernel.  Like the backend registration, it stays in place after ``uninstall()``.

Nothing here is imported by the engine itself; ``install()`` raises if modelopt is absent.
``stats`` counts kernel-path calls per hook so a test can prove which side executed.
"""

from __future__ import annotations

import collections
import copy
import types

import torch

from . import ops
from .nn.functional import normalized_hadamard_transform
from .nn.tensor_quantizer import fp8_max_for_normalization
from .tensor_quant import dynamic_block_quant, fake_tensor_quant, scaled_e4m3, static_blockwise_fp4_fake_quant

stats: collections.Counter = collections.Counter()
_saved: dict = {}


# ---- (1) functional backend -----------------------------------------------------------------------
def _dynamic_amax(inputs: torch.Tensor, tq) -> torch.Tensor:
    """``TensorQuantizer._get_amax`` (:736-751) without a calibrated ``_amax``: per-tensor dynamic amax through
    the collect kernel; other axes go through the quantizer's own helper."""
    if getattr(tq, "_use_constant_amax", False) or hasattr(tq, "_amax") or tq._axis is not None:
        return tq._get_amax(inputs)
    slot = torch.zeros(1, dtype=torch.float32, device=inputs.device)
    ops.amax_per_tensor_(slot, inputs)
    return ops.amax_export(slot, inputs.dtype).reshape((1,) * inputs.dim())


def b200_fake_quant_entrypoint(inputs: torch.Tensor, tq) -> torch.Tensor:
    """``entrypoint(inputs, tensor_quantizer) -> Tensor`` (tensor_quantizer.py:892-896): inputs are
    contiguous, pre_quant_scale / static-block reshape already applied."""
    bs = tq._block_sizes
    num_bits = tq._num_bits
    ptb = getattr(tq, "_pass_through_bwd", True)
    stats["entrypoint"] += 1
    if bs is not None and bs.get("type", "static") == "dynamic":
        block = bs.get(-1) or bs.get(inputs.dim() - 1)
        scale_bits = bs.get("scale_bits")
        amax = None if scale_bits == (8, 0) else _dynamic_amax(inputs, tq)   # MX: no global amax
        return dynamic_block_quant(inputs, block, amax, None, num_bits, scale_bits, None, "dynamic", ptb)
    if getattr(tq, "_global_amax", None) is not None and num_bits == (2, 1):
        return static_blockwise_fp4_fake_quant(inputs, tq._amax.float(), tq._global_amax, True,
                                               fp8_max_for_normalization(tq), None, ptb)
    amax = _dynamic_amax(inputs, tq)
    if isinstance(num_bits, tuple):
        return scaled_e4m3(inputs, amax, None, num_bits[0], num_bits[1], None, ptb)
    return fake_tensor_quant(inputs, amax, None, num_bits, tq._unsigned, tq._narrow_range, None, ptb)


# ---- (4) extension-module shims (same names as tensor_quant.cpp:63-77 / tensor_quant_gpu_fp8.cu:109-114)
def make_cuda_ext() -> types.SimpleNamespace:
    def fake_tensor_quant_(inputs, amax, num_bits=8, unsigned=False, narrow_range=True):
        stats["ext.fake_tensor_quant"] += 1
        ops.fake_quant_int(inputs, amax, num_bits, unsigned, narrow_range, out=inputs)

    def fake_tensor_quant(inputs, amax, num_bits=8, unsigned=False, narrow_range=True):
        stats["ext.fake_tensor_quant"] += 1
        return ops.fake_quant_int(inputs.contiguous(), amax, num_bits, unsigned, narrow_range)

    def fake_tensor_quant_with_axis(inputs, amax, axis, num_bits=8, unsigned=False, narrow_range=True):
        stats["ext.fake_tensor_quant"] += 1
        x = inputs.contiguous()
        return ops.fake_quant_int(x, amax, num_bits, unsigned, narrow_range, outer=x.stride(axis))

    def INT4_quantize(input, scales, block_size):  # noqa: N802  (scales recomputed in-kernel, identical)
        stats["ext.INT4_quantize"] += 1
        packed, _ = ops.pack_int4_blockwise(input.contiguous(), block_size)
        return packed

    def INT4_dequantize(q, scales, block_size):  # noqa: N802
        stats["ext.INT4_dequantize"] += 1
        return ops.unpack_int4_blockwise(q.contiguous(), scales.contiguous(), block_size)

    def NF4_quantize(input, scales, block_size):  # noqa: N802
        stats["ext.NF4_quantize"] += 1
        return ops.pack_nf4(input.contiguous(), block_size, scales.contiguous())[0]

    def NF4_dequantize(q, scales, block_size):  # noqa: N802
        stats["ext.NF4_dequantize"] += 1
        return ops.unpack_nf4(q.contiguous(), scales.contiguous(), block_size)

    return types.SimpleNamespace(fake_tensor_quant_=fake_tensor_quant_, fake_tensor_quant=fake_tensor_quant,
                                 fake_tensor_quant_with_axis=fake_tensor_quant_with_axis,
                                 INT4_quantize=INT4_quantize, INT4_dequantize=INT4_dequantize,
                                 NF4_quantize=NF4_quantize, NF4_dequantize=NF4_dequantize)


def make_cuda_ext_fp8() -> types.SimpleNamespace:
    def fake_e4m3fy(inputs, amax):
        stats["ext.fake_e4m3fy"] += 1
        return ops.fake_quant_fp8(inputs.contiguous(), amax)

    def fake_e4m3fy_with_axis(inputs, amax, axis):
        stats["ext.fake_e4m3fy"] += 1
        x = inputs.contiguous()
        return ops.fake_quant_fp8(x, amax, outer=x.stride(axis))

    return types.SimpleNamespace(fake_e4m3fy=fake_e4m3fy, fake_e4m3fy_with_axis=fake_e4m3fy_with_axis)


def make_cuda_ext_mx() -> types.SimpleNamespace:
    """``modelopt_cuda_ext_mx`` (tensor_quant_mx.cu:393-411): ``fused_amax_convert``, ``convert_to_exmy``,
    ``Types``.  E8M0 scales run the MX kernel; (E2M1, E4M3 scale, global amax) runs the NVFP4 kernel, whose
    results equal the extension's two-level path away from its fast-math corners."""
    import enum

    Types = enum.IntEnum("Types", list(ops.MX_FORMATS.items()))  # noqa: N806

    def fused_amax_convert(inputs, block_size, format, scale_format, global_amax=None):
        stats["ext.fused_amax_convert"] += 1
        x = inputs.contiguous()
        if int(scale_format) == Types.E8M0:
            return ops.fake_quant_mx(x, block_size, int(format))
        if int(format) == Types.E2M1 and int(scale_format) == Types.E4M3 and global_amax is not None \
                and block_size == 16:
            return ops.fake_quant_nvfp4(x, global_amax.float().amax() if global_amax.numel() > 1 else global_amax)
        raise NotImplementedError("fused_amax_convert: the b200quant engine covers E8M0 scales and NVFP4 (E2M1 / E4M3)")

    return types.SimpleNamespace(fused_amax_convert=fused_amax_convert, convert_to_exmy=ops.convert_to_exmy,
                                 Types=Types)


# ---- (5) functions the hooks do not reach ------------------------------------------------------------
def _make_qtensor_patches(ref_nvfp4_cls, ref_fp8_cls):
    """Kernel-backed replacements for ``NVFP4QTensor.quantize`` and ``FP8QTensor.quantize`` that build the
    REFERENCE's QTensor objects (so ``mtq.compress``, ``dequantize`` and export keep working unchanged)."""
    orig_nvfp4 = ref_nvfp4_cls.__dict__["quantize"].__func__
    orig_fp8 = ref_fp8_cls.__dict__["quantize"].__func__

    def nvfp4_quantize(cls, input, block_size, weights_scaling_factor=None, weights_scaling_factor_2=None,
                       keep_high_precision=False, try_tensorrt=False):
        if (not input.is_cuda or weights_scaling_factor is not None or keep_high_precision
                or block_size not in (16, 32, 64, 128, 256, 512) or input.dtype not in ops._DT):
            return orig_nvfp4(cls, input, block_size, weights_scaling_factor, weights_scaling_factor_2,
                              keep_high_precision, try_tensorrt)
        stats["qtensor.nvfp4_quantize"] += 1
        shape, dtype = input.shape, input.dtype
        pad = (-input.shape[-1]) % block_size
        if pad:
            input = torch.nn.functional.pad(input, (0, pad))     # reduce_block_padding (nvfp4_tensor.py:278)
        x = input.contiguous()
        if weights_scaling_factor_2 is None:
            g = torch.zeros(1, dtype=torch.float32, device=x.device)
            ops.amax_per_tensor_(g, x)
            # get_weights_scaling_factor_2 (:204-207) is `reduce_amax(x).float() / (6 * 448)`: the amax is rounded
            # to the input dtype first (reduce_amax returns the input dtype) -- exact for |max| of the tensor
            packed, scales, wsf2 = ops.pack_nvfp4(x, g, None, 448.0, block_size)
        else:
            packed, scales, wsf2 = ops.pack_nvfp4(x, None, None, 448.0, block_size, wsf2=weights_scaling_factor_2)
            wsf2 = weights_scaling_factor_2
        return cls(shape, dtype, packed), scales, wsf2

    def fp8_quantize(cls, input, scales=None, axis=None, block_sizes=None):
        from .qtensor import FP8QTensor as Mine

        if not input.is_cuda or input.dtype not in ops._DT or input.dim() > 2 and block_sizes:
            return orig_fp8(cls, input, scales, axis, block_sizes)
        if block_sizes:
            keys = sorted(k % input.dim() for k in block_sizes if isinstance(k, int))
            if input.dim() != 2 or keys != [0, 1]:
                return orig_fp8(cls, input, scales, axis, block_sizes)
        stats["qtensor.fp8_quantize"] += 1
        mine, out_scales = Mine.quantize(input, scales, axis, block_sizes)
        return cls(input.shape, input.dtype, mine._quantized_data), out_scales

    return classmethod(nvfp4_quantize), classmethod(fp8_quantize)


# ---- (2), (3) calibrators + install ------------------------------------------------------------------
def _make_sweep_calibrator(base):
    class B200FP8SweepCalibrator(base):
        """``NVFP4MSECalibrator`` (calib/mse.py:175-311) for quantizers with ``backend == "b200"``: the 126
        FP8-E4M3 scale candidates of every 16-element block are evaluated in registers from one read
        (``b200q_nvfp4_fp8_scale_sweep``; first-minimum tie-break like the reference's ``loss < best``)."""

        def __init__(self, amax, axis, quant_func):
            super().__init__(num_bits=None, axis=axis, unsigned=None)
            self._initial_amax = amax
            self._quantizer = getattr(quant_func, "keywords", {}).get("quantizer")
            self._best_amax = None

        @torch.no_grad()
        def collect(self, x):
            if self._best_amax is not None:
                raise RuntimeError("B200FP8SweepCalibrator: multi-collect is not supported; call reset() first")
            g = getattr(self._quantizer, "global_amax", None)
            if g is None:
                raise RuntimeError("B200FP8SweepCalibrator needs the quantizer's global_amax (static NVFP4 only)")
            if x.dim() != 2 or x.shape[-1] != 16 or x.shape[0] != self._initial_amax.numel():
                raise RuntimeError(f"expected the blocked [n_blocks, 16] weight layout, got {tuple(x.shape)}")
            stats["calib.fp8_sweep"] += 1
            best = ops.nvfp4_fp8_scale_sweep(x.detach().contiguous(), g.detach().float().reshape(1))
            self._best_amax = best.reshape(self._initial_amax.shape).to(torch.float32)

        @torch.no_grad()
        def compute_amax(self, verbose=False):
            return self._best_amax

        def reset(self):
            self._best_amax = None

    return B200FP8SweepCalibrator


def _make_mse_factory(base, ref_mse_cls):
    from .calib.mse import MseCalibrator as Mine
    from .calib.mse import is_static_nvfp4_search

    class B200MseCalibrator(ref_mse_cls):
        """Stands in for ``MseCalibrator`` in model_calib.py:720-728 (a subclass, so the reference's
        ``isinstance(..., MseCalibrator)`` checks keep working).  For a quantizer on the b200 backend with an integer
        or FP8 format, or static NVFP4 (16-element blocks, fp32 block amax, a global amax; Four-Over-Six included),
        the search runs as one fused sweep kernel; outside that scope (custom error function, no quantizer behind
        ``quant_func``, other formats / backends) the host application's own methods run."""

        def __init__(self, amax, axis=None, step_size=0.1, start_multiplier=0.25, stop_multiplier=4.0,
                     quant_func=None, error_func=None):
            super().__init__(amax=amax, axis=axis, step_size=step_size, start_multiplier=start_multiplier,
                             stop_multiplier=stop_multiplier, quant_func=quant_func, error_func=error_func)
            q = getattr(quant_func, "keywords", {}).get("quantizer") if quant_func is not None else None
            nb = getattr(q, "_num_bits", None)
            ok = (error_func is None and q is not None and getattr(q, "backend", None) == "b200"
                  and ((isinstance(nb, int) or nb == (4, 3)) and not getattr(q, "is_mx_format", False)
                       or is_static_nvfp4_search(q, amax))
                  and amax is not None and amax.is_cuda)
            self._b200 = Mine(amax, axis, step_size, start_multiplier, stop_multiplier, quant_func, None) if ok else None

        def collect(self, x):
            if self._b200 is None:
                return super().collect(x)
            stats["calib.mse"] += 1
            return self._b200.collect(x)

        def compute_amax(self, verbose=False):
            return super().compute_amax(verbose) if self._b200 is None else self._b200.compute_amax(verbose)

        def reset(self):
            if self._b200 is not None:
                self._b200.reset()
            super().reset()

    return B200MseCalibrator


def _make_headroom_calibrator(ref_cls):
    from .calib.nvfp4_act_headroom import NVFP4ActHeadroomCalibrator as Mine

    class B200NVFP4ActHeadroomCalibrator(ref_cls):
        """Stands in for ``NVFP4ActHeadroomCalibrator`` in ``nvfp4_act_headroom_calibrate`` (a subclass, so
        ``isinstance`` checks keep holding; the reference's constructor validates the arguments).  CUDA inputs in fp32 /
        fp16 / bf16 with blocks of 16 go to this engine's calibrator; a NaN or inf block then raises in
        ``compute_amax`` rather than in the ``collect`` of its batch, which would cost a host sync per batch.  Batches
        that ran the reference's ``collect`` (other inputs) are merged with the engine's statistic before the amax."""

        def __init__(self, num_bits=(2, 1), axis=None, unsigned=False, *, block_size=16, anchor_percentile=1.0,
                     upper_percentile=99.99, rho=16384.0, num_bins=512, log2_min=-40.0, log2_max=40.0):
            kw = dict(anchor_percentile=anchor_percentile, upper_percentile=upper_percentile, rho=rho,
                      num_bins=num_bins, log2_min=log2_min, log2_max=log2_max)
            super().__init__(num_bits, axis, unsigned, block_size=block_size, **kw)
            self._b200 = Mine(num_bits, axis, unsigned, block_size=16, **kw) if block_size == 16 else None

        def collect(self, x):
            if self._b200 is None or not x.is_cuda or x.dtype not in ops._DT:
                return super().collect(x)
            stats["calib.nvfp4_act_headroom"] += 1
            return self._b200.collect(x)

        def compute_amax(self):
            if self._b200 is None or self._b200._hist is None:
                return super().compute_amax()
            stats["calib.nvfp4_act_headroom"] += 1
            if self._running_max is None:
                return self._b200.compute_amax()
            rmax = self._b200._running_max.reshape(()).to(self._running_max.device)
            if not bool(torch.isfinite(rmax)):
                raise AssertionError("detected nan/inf values in amax")
            self._running_max = torch.maximum(self._running_max, rmax)
            if int(self._b200._hist.sum()) > 0:
                h = self._b200._hist.to(self._running_max.device)
                self._hist = h if self._hist is None else self._hist + h
            self._b200.reset()
            return super().compute_amax()

        def reset(self):
            if self._b200 is not None:
                stats["calib.nvfp4_act_headroom"] += 1
                self._b200.reset()
            super().reset()

    return B200NVFP4ActHeadroomCalibrator


def _make_gptq_helper(ref_helper_cls):
    class B200GPTQHelper(ref_helper_cls):
        """``GPTQHelper`` whose blockwise update runs ``ops.gptq_blockwise_update`` for quantizers inside the GPTQ
        kernel's scope (the unfused semantics of ``gptq_blockwise_update`` for every covered format, whatever
        ``fused`` says); other quantizers, and CPU weights, run the host application's own loop."""

        def _blockwise_update(self, block_size):
            q = self.module.weight_quantizer
            w = self.weight
            desc = ops.gptq_quantizer_desc(q, w.shape, block_size, w.device) if w.is_cuda else None
            if desc is None:
                return super()._blockwise_update(block_size)
            stats["gptq.block"] += 1
            ops.gptq_blockwise_update(self.weight, self.h_inv, block_size, q, desc=desc)

    return B200GPTQHelper


def install(patch_extensions: bool = True, patch_functions: bool = True):
    """Register the backend, the calibrator classes, the FP8-sweep factory, the GPTQ helper and (optionally) the extension shims
    and function rebinds in modelopt.  Returns ``(B200MaxCalibrator, B200HistogramCalibrator)``."""
    import modelopt.torch.quantization.calib as ref_calib
    import modelopt.torch.quantization.extensions as ref_ext
    import modelopt.torch.quantization.model_calib as ref_model_calib
    import modelopt.torch.quantization.tensor_quant as ref_tensor_quant
    from modelopt.torch.quantization.nn.modules import tensor_quantizer as ref_tq

    from . import _lib
    from .calib import HistogramCalibrator, MaxCalibrator

    _lib.load()                                        # fail loudly when the CUDA library is missing
    if not ref_tq.is_registered_quant_backend("b200"):
        ref_tq.register_quant_backend("b200", b200_fake_quant_entrypoint)

    base = ref_calib._Calibrator
    if "classes" not in _saved:
        class B200MaxCalibrator(MaxCalibrator, base):  # isinstance(_Calibrator) for the reference's checks
            def collect(self, x):
                stats["calib.max"] += 1
                return MaxCalibrator.collect(self, x)

        class B200HistogramCalibrator(HistogramCalibrator, base):
            def collect(self, x):
                stats["calib.histogram"] += 1
                return HistogramCalibrator.collect(self, x)

        _saved["classes"] = (B200MaxCalibrator, B200HistogramCalibrator, _make_sweep_calibrator(base))
    B200MaxCalibrator, B200HistogramCalibrator, sweep_cls = _saved["classes"]   # noqa: N806
    ref_calib.B200MaxCalibrator = B200MaxCalibrator
    ref_calib.B200HistogramCalibrator = B200HistogramCalibrator
    ref_model_calib._register_fp8_sweep_calibrator("b200", lambda amax, axis, quant_func: sweep_cls(amax, axis, quant_func))
    import modelopt.torch.quantization.utils.calib_utils as ref_calib_utils

    if "gptq" not in _saved:
        _saved["gptq"] = _make_gptq_helper(ref_calib_utils.GPTQHelper)
    ref_calib_utils.register_gptq_helper("b200", _saved["gptq"])

    if patch_extensions and "ext" not in _saved:
        _saved["ext"] = {(m, n): getattr(m, n) for m in (ref_ext, ref_tensor_quant)
                         for n in ("get_cuda_ext", "get_cuda_ext_fp8", "get_cuda_ext_mx") if hasattr(m, n)}
        import modelopt.torch.quantization.qtensor.int4_tensor as ref_int4
        import modelopt.torch.quantization.qtensor.nf4_tensor as ref_nf4

        for m in (ref_int4, ref_nf4):
            if hasattr(m, "get_cuda_ext"):
                _saved["ext"][(m, "get_cuda_ext")] = m.get_cuda_ext
        ext, ext8, extmx = make_cuda_ext(), make_cuda_ext_fp8(), make_cuda_ext_mx()
        shims = {"get_cuda_ext": lambda raise_if_failed=False: ext,
                 "get_cuda_ext_fp8": lambda raise_if_failed=False: ext8,
                 "get_cuda_ext_mx": lambda raise_if_failed=False: extmx}
        for (m, n) in _saved["ext"]:
            setattr(m, n, shims[n])
    if patch_functions and "fn" not in _saved:
        from modelopt.torch.quantization.qtensor import FP8QTensor, NVFP4QTensor

        from .tensor_quant import static_blockwise_fp4_fake_quant as mine

        def static_fp4(x, amax, global_amax=None, quantize_block_scales=True, fp8_max_for_normalization=448.0,
                       out_dtype=None, pass_through_bwd=False):
            stats["fn.static_blockwise_fp4_fake_quant"] += 1
            return mine(x, amax, global_amax, quantize_block_scales, fp8_max_for_normalization, out_dtype,
                        pass_through_bwd)

        orig_hadamard = ref_tq.normalized_hadamard_transform

        def hadamard(inputs, rotate_fp32=False, block_size=None):
            if not inputs.is_cuda or inputs.dtype not in ops._DT:      # outside the engine: the host's own function
                return orig_hadamard(inputs, rotate_fp32=rotate_fp32, block_size=block_size)
            stats["fn.normalized_hadamard_transform"] += 1
            return normalized_hadamard_transform(inputs, rotate_fp32, block_size)

        _saved["fn"] = {"static": ref_tq.static_blockwise_fp4_fake_quant,
                        "nvfp4_quantize": NVFP4QTensor.__dict__["quantize"],
                        "fp8_quantize": FP8QTensor.__dict__["quantize"],
                        "mse": ref_model_calib.MseCalibrator,
                        "headroom": ref_model_calib.NVFP4ActHeadroomCalibrator,
                        "hadamard": orig_hadamard}
        ref_tq.static_blockwise_fp4_fake_quant = static_fp4
        ref_tq.normalized_hadamard_transform = hadamard
        ref_model_calib.MseCalibrator = _make_mse_factory(base, ref_model_calib.MseCalibrator)
        ref_model_calib.NVFP4ActHeadroomCalibrator = _make_headroom_calibrator(ref_model_calib.NVFP4ActHeadroomCalibrator)
        NVFP4QTensor.quantize, FP8QTensor.quantize = _make_qtensor_patches(NVFP4QTensor, FP8QTensor)
    return B200MaxCalibrator, B200HistogramCalibrator


def uninstall():
    """Undo every rebind of ``install()`` (the backend / calibrator registrations are inert and stay)."""
    from modelopt.torch.quantization.nn.modules import tensor_quantizer as ref_tq

    for (m, n), f in _saved.pop("ext", {}).items():
        setattr(m, n, f)
    fn = _saved.pop("fn", None)
    if fn is not None:
        from modelopt.torch.quantization.qtensor import FP8QTensor, NVFP4QTensor

        import modelopt.torch.quantization.model_calib as ref_model_calib

        ref_tq.static_blockwise_fp4_fake_quant = fn["static"]
        ref_tq.normalized_hadamard_transform = fn["hadamard"]
        ref_model_calib.MseCalibrator = fn["mse"]
        ref_model_calib.NVFP4ActHeadroomCalibrator = fn["headroom"]
        NVFP4QTensor.quantize = fn["nvfp4_quantize"]
        FP8QTensor.quantize = fn["fp8_quantize"]


def with_b200_backend(quant_cfg: dict, calibrators: bool = True) -> dict:
    """Return a copy of a modelopt preset with ``backend: "b200"`` on every enabled quantizer entry and (after
    ``install()``) the ``calibrator`` field pointing at the B200 collect classes.  The calibrator is given as the
    constructor tuple ``(cls, (num_bits, axis, unsigned))`` because the reference builds a custom class with no
    arguments (``_calibrator_setter``, tensor_quantizer.py:235-241) and would lose a per-channel ``axis``."""
    cfg = copy.deepcopy(quant_cfg)
    classes = _saved.get("classes") if calibrators else None

    def patch(c: dict):
        if c.get("enable", True) is False:
            return
        c["backend"] = "b200"
        if classes is not None and c.get("type", "static") != "dynamic":
            kind = c.get("calibrator", "max")
            if isinstance(kind, str):
                cls = classes[0] if kind == "max" else classes[1]
                axis = None if c.get("block_sizes") else c.get("axis")
                c["calibrator"] = (cls, (c.get("num_bits", 8), axis, c.get("unsigned", False)))

    for entry in cfg["quant_cfg"]:
        if not isinstance(entry, dict):
            continue
        c = entry.get("cfg")
        if isinstance(c, dict):
            patch(c)
        elif isinstance(c, (list, tuple)):
            for ci in c:
                if isinstance(ci, dict):
                    patch(ci)
    return cfg


__all__ = ["install", "uninstall", "with_b200_backend", "b200_fake_quant_entrypoint", "make_cuda_ext",
           "make_cuda_ext_fp8", "make_cuda_ext_mx", "stats"]
