"""Calibration algorithms -- mirror of ``modelopt/torch/quantization/model_calib.py``:
``max_calibrate`` :311-498, ``enable_stats_collection`` :1128 / ``finish_stats_collection`` :1144,
``weight_only_quantize`` :187, ``smoothquant`` :1274-1358, ``awq_lite`` :1395-1722,
``apply_pre_quant_scale_and_smooth`` :1227.

B200-first differences (results identical, work removed):
  * weights are collected once (``weight_only_quantize``); the reference re-collects every weight on
    every calibration batch because ``QuantLinear.forward`` calls ``weight_quantizer(weight)`` while
    ``_if_calib`` is set (quant_module.py:258-270) -- here weight quantizers leave calibration mode
    as soon as their amax exists;
  * per-quantizer ``dist.all_reduce`` calls (tensor_quantizer.py:1377) become ONE all-reduce over a
    flat fp32 amax arena (``distributed.AmaxArena``).
"""

from __future__ import annotations

import collections
import math
import warnings
from typing import Callable

import torch
import torch.nn.functional as F
from torch import nn

from . import distributed as b200_dist
from . import ops
from .nn import TensorQuantizer, is_quantized_linear


def _quantizers(model):
    if isinstance(model, TensorQuantizer):
        yield "", model
        return
    for name, m in model.named_modules():
        if isinstance(m, TensorQuantizer):
            yield name, m


def enable_stats_collection(model: nn.Module):
    """model_calib.py:1128-1141."""
    for _, q in _quantizers(model):
        if q.is_enabled and q._calibrator is not None and not q._dynamic:
            q.disable_quant()
            q.enable_calib()
        elif q.is_enabled:
            q.disable_quant()


def finish_stats_collection(model: nn.Module, method: str | None = None):
    """model_calib.py:1144-1167."""
    for _, q in _quantizers(model):
        if q._disabled:
            continue
        cal = q._calibrator
        if cal is not None and not q._dynamic and q._if_calib:
            amax = cal.compute_amax() if method is None else cal.compute_amax(method)
            if amax is not None:
                q.load_calib_amax() if method is None else q.load_calib_amax(method)
        if q.bias_calibrator is not None and q.bias_type == "static" and q.bias_calibrator.compute_bias() is not None:
            q.load_calib_bias()          # model_calib.py:1163-1164
        q.enable_quant()
        q.disable_calib()


def weight_only_quantize(model: nn.Module):
    """model_calib.py:187-199: one pass of every enabled weight quantizer over its weight."""
    for m in model.modules():
        if is_quantized_linear(m) and m.weight_quantizer.is_enabled:
            m.weight_quantizer(m.weight)


# Groups export fuses into one GEMM (q/k/v -> qkv, gate/up incl. Mixtral w1/w3 -> gate_up): their weights must share
# ONE NVFP4 per-tensor scale.  Same regexes as utils/shared_input.py:57-61, ``re.fullmatch``-ed against module names;
# the captured parent is the group key (so MoE w1/w3 group per expert).
SHARED_PATTERNS = (
    r"(?:(.*)\.)?(?:q_proj|k_proj|v_proj)",
    r"(?:(.*)\.)?(?:gate_proj|up_proj)",
    r"(?:(.*)\.)?(?:w1|w3)",
)


def find_shared_weight_groups(model: nn.Module, patterns=SHARED_PATTERNS) -> list[list[nn.Module]]:
    """find_shared_input_groups (utils/shared_input.py:420-463): modules with an enabled weight quantizer whose
    fully-qualified name matches the same pattern with the same captured parent; groups of >= 2."""
    import re

    compiled = [re.compile(p) for p in patterns or ()]
    buckets: dict = {}
    for name, m in model.named_modules():
        wq = getattr(m, "weight_quantizer", None)
        if wq is None or not hasattr(wq, "_disabled") or wq._disabled:
            continue
        for i, rx in enumerate(compiled):
            mt = rx.fullmatch(name)
            if mt is not None:
                buckets.setdefault((i, mt.groups()), []).append(m)
                break                                     # first matching pattern wins
    return [g for g in buckets.values() if len(g) >= 2]


def _finalize_static_nvfp4(model, patterns=SHARED_PATTERNS):
    """``_finalize_with_shared_state`` (model_calib.py:143-156) = ``SharedWeightGlobalAmaxState.populate``
    (utils/shared_input.py:258-268, finalize :314-327: one fp32 ``global_amax`` = max over the members' ``_amax``)
    + ``promote_static_block_weight_quantizers`` (utils/core_utils.py:1077-1150): static NVFP4 weight quantizers
    keep their per-block ``_amax`` in fp32 and get ``_global_amax`` -- the group's tensor, ALIASED (one storage
    for all members, shared_input.py:151-185), or their own per-block maximum when they belong to no group.

    Distributed runs call this after the amax sync (like the reference, model_calib.py:497), so the group maximum
    is computed from already-consistent ``_amax`` values and needs no collective of its own."""
    shared: dict[int, torch.Tensor] = {}
    for members in find_shared_weight_groups(model, patterns):
        qs = [m.weight_quantizer for m in members if getattr(m.weight_quantizer, "_amax", None) is not None]
        if not qs or not any(q.is_nvfp4_static for q in qs):
            continue
        g = torch.zeros(1, dtype=torch.float32, device=qs[0]._amax.device)
        for q in qs:                                       # running max over members: one collect kernel each
            ops.amax_per_tensor_(g, q._amax.detach().contiguous())
        g = g.reshape(())
        for q in qs:
            shared[id(q)] = g
    # promotion walks quantized modules (core_utils.py:1101-1109): a bare quantizer passed to max_calibrate is left alone
    weight_quantizers = [m.weight_quantizer for m in model.modules() if is_quantized_linear(m)]
    for q in weight_quantizers:
        if not (q.is_enabled and q.is_static_block_quant and q.amax is not None):
            continue
        if q._amax.dtype != torch.float32:
            # StaticBlockScaleQuantizer._preserve_amax_in_fp32 (tensor_quantizer.py:1501-1514): promoted static-block
            # weight quantizers -- NVFP4 and integer (INT4 block-128) alike, core_utils.py:1143-1146 -- keep fp32 state
            blocks = q._amax.float()
            delattr(q, "_amax")
            q.amax = blocks
        if not q.is_nvfp4_static:
            continue
        g = shared.get(id(q))
        if g is None:
            g = torch.zeros(1, dtype=torch.float32, device=q._amax.device)
            ops.amax_per_tensor_(g, q._amax.contiguous())
            g = g.reshape(())
        if "_global_amax" in q._buffers:
            q._buffers["_global_amax"] = g             # alias, do not copy
        else:
            q.register_buffer("_global_amax", g)
        q._state_gen += 1


@torch.no_grad()
def max_calibrate(model: nn.Module, forward_loop: Callable | None = None, distributed_sync: bool = True):
    """model_calib.py:311-498."""
    enable_stats_collection(model)
    if forward_loop is None:
        weight_only_quantize(model)
    else:
        weight_only_quantize(model)
        # weight amax is final after one pass: take weight quantizers out of calibration mode so the
        # forward loop does not re-reduce every weight per batch
        for m in model.modules():
            if is_quantized_linear(m):
                m.weight_quantizer._b200_hold = m.weight_quantizer._if_calib
                m.weight_quantizer._if_calib = False
        forward_loop(model)
        for m in model.modules():
            if is_quantized_linear(m) and hasattr(m.weight_quantizer, "_b200_hold"):
                m.weight_quantizer._if_calib = m.weight_quantizer._b200_hold
                del m.weight_quantizer._b200_hold
    if distributed_sync and b200_dist.is_initialized():
        b200_dist.sync_calibrator_amax(model)
    finish_stats_collection(model)
    if distributed_sync and b200_dist.is_initialized():
        b200_dist.sync_headroom_amax(model)
    _finalize_static_nvfp4(model)


def _is_nvfp4_dynamic_input_quantizer(name: str, q) -> bool:
    """model_calib.py:501-529: an enabled, non-``_dynamic`` NVFP4 dynamic-block (E2M1, E4M3 scales) input quantizer."""
    return (name.endswith("input_quantizer") and isinstance(q, TensorQuantizer) and not q._disabled
            and not q._dynamic and q.is_nvfp4_dynamic)


@torch.no_grad()
def nvfp4_act_headroom_calibrate(model: nn.Module, forward_loop: Callable | None = None, *,
                                 anchor_percentile: float = 1.0, upper_percentile: float = 99.99, rho: float = 16384.0,
                                 weight_scale_algorithm: dict | None = None):
    """model_calib.py:500-636: every NVFP4 dynamic-block input quantizer gets an ``NVFP4ActHeadroomCalibrator`` for
    the run of ``weight_scale_algorithm`` (``max``, ``mse`` or ``local_hessian``; ``None`` is ``max``), whose max pass
    collects the per-block log2 histograms and loads ``amax = max(rho * P_anchor, P_upper)`` (fp32) into those
    quantizers; the original calibrators are restored afterwards.  Everything is validated before the model changes:
    an NVFP4 input quantizer with blocks other than 16 raises ``NotImplementedError``.  Under data parallelism the
    per-rank amaxes are merged with one MAX all-reduce (``distributed.sync_headroom_amax``): the largest per-rank
    scale, as the reference documents."""
    from .calib import NVFP4ActHeadroomCalibrator
    from .config import NVFP4ActHeadroomCalibConfig

    cfg = NVFP4ActHeadroomCalibConfig(anchor_percentile=anchor_percentile, upper_percentile=upper_percentile, rho=rho,
                                      weight_scale_algorithm=weight_scale_algorithm)
    targets = [(n, q) for n, q in _quantizers(model) if _is_nvfp4_dynamic_input_quantizer(n, q)]
    for n, q in targets:
        if q._block_sizes.get(-1, 16) != 16:
            raise NotImplementedError(f"nvfp4_act_headroom: {n!r} quantizes blocks of {q._block_sizes.get(-1)}; "
                                      f"only NVFP4 input blocks of 16 are supported")
    weight_kw = {k: v for k, v in cfg.weight_scale_algorithm.items() if k != "method"}
    weight_fn = {"max": max_calibrate, "mse": mse_calibrate,
                 "local_hessian": local_hessian_calibrate}[cfg.weight_scale_algorithm["method"]]
    if not targets:
        warnings.warn("nvfp4_act_headroom: no NVFP4 dynamic-block input quantizer matched, so this is equivalent to "
                      "plain max calibration. Check that the recipe enables NVFP4 activation quantizers.")
    swapped = []
    try:
        for _, q in targets:
            swapped.append((q, q._calibrator))
            q._calibrator = NVFP4ActHeadroomCalibrator(q._num_bits, None, q._unsigned, block_size=16,
                                                       anchor_percentile=cfg.anchor_percentile,
                                                       upper_percentile=cfg.upper_percentile, rho=cfg.rho)
        weight_fn(model, forward_loop, **weight_kw)
    finally:
        for q, original in swapped:
            q._calibrator = original


@torch.no_grad()
def mse_calibrate(model: nn.Module, forward_loop: Callable | None = None, distributed_sync: bool = True,
                  step_size: float = 0.1, start_multiplier: float = 0.25, stop_multiplier: float = 4.0,
                  fp8_scale_sweep: bool = False, **kw):
    """model_calib.py:733-827: max-calibrate everything, then refine every eligible WEIGHT amax by MSE.

    ``fp8_scale_sweep=True``: only static NVFP4 weights, per-block argmin over the 126 FP8-E4M3 scale values
    (``NVFP4MSECalibrator``, calib/mse.py:175-311) -- one ``b200q_nvfp4_fp8_scale_sweep`` launch per weight.
    Otherwise: the multiplier search of ``MseCalibrator`` (calib/mse.py:31-172) for every enabled, static,
    non-MX weight quantizer -- one ``b200q_mse_sweep[_rows]`` launch per weight (the reference: 39 x ~4 passes), or
    for static NVFP4 weights one ``b200q_nvfp4_static_mse_sweep`` launch that picks each 16-element block's
    multiplier against the ``global_amax`` set by max calibration (shared by q/k/v and gate/up siblings).  With the
    Four-Over-Six preset's multipliers {1.0, 1.5} this chooses, per block, the grid that ends at 6 or at 4."""
    max_calibrate(model, forward_loop, distributed_sync)
    for m in model.modules():
        if not is_quantized_linear(m):
            continue
        q = m.weight_quantizer
        if (not q.is_enabled or q._dynamic or q.is_mx_format or q._calibrator is None
                or getattr(q, "_amax", None) is None):       # _make_weight_mse_calibrator (:694-707)
            continue
        if fp8_scale_sweep:
            if not q.is_nvfp4_static:
                continue                                     # left at the max-calibrated amax (:717-718)
            # the sweep's candidates and losses do not depend on the FP8 normalization: a Four-Over-Six quantizer is
            # swept like any static NVFP4 one (NVFP4MSECalibrator, calib/mse.py:175-311) and normalizes by 256 after
            best = ops.nvfp4_fp8_scale_sweep(_pad_blocks16(m.weight), q._global_amax.reshape(1))
            q.amax = best.reshape(q._amax.shape)
            continue
        _mse_search_weight(m, step_size, start_multiplier, stop_multiplier)


def _pad_blocks16(w):
    """The weight in the static NVFP4 block layout the sweep searches: the last dim zero-padded to a multiple of 16, as
    ``_process_for_blockquant`` pads it (zeros change no block amax and add no error)."""
    rem = w.shape[-1] % 16
    return (F.pad(w, (0, 16 - rem)) if rem else w).contiguous()


def _mse_search_weight(m, step_size, start_multiplier, stop_multiplier):
    """The multiplier search of one weight (``_make_weight_mse_calibrator`` -> ``MseCalibrator``, :720-728)."""
    from functools import partial

    from .calib.mse import MseCalibrator

    q = m.weight_quantizer
    cal = MseCalibrator(q._amax.clone().detach(), q._calibrator._axis, step_size, start_multiplier,
                        stop_multiplier, quant_func=partial(_mse_quant_func, quantizer=q))
    w = m.weight
    if q.is_static_block_quant:                              # the calibration layout: [n_blocks, block]
        q._setup_for_blockquant(w)
        w = q._process_for_blockquant(w)
    cal.collect(w)
    q.amax = cal.compute_amax()
    cal.reset()


@torch.no_grad()
def local_hessian_calibrate(model: nn.Module, forward_loop: Callable | None = None, distributed_sync: bool = True,
                            step_size: float = 0.1, start_multiplier: float = 0.25, stop_multiplier: float = 4.0,
                            fp8_scale_sweep: bool = True, block_size: int = 16, debug: bool = False, **kw):
    """model_calib.py:1005-1125: weight amax search under the Hessian-weighted error ``dw^T H dw`` with the
    per-cin-block local Hessian ``H = sum X^T X / n_tokens`` (``_LocalHessianAccumulator``, :829-901) captured by
    forward pre-hooks while the weight quantizers are disabled.  Static NVFP4 weights: ONE
    ``b200q_nvfp4_fp8_scale_sweep_hessian`` launch per weight (the reference: a Triton kernel with ``tl.dot``, or 126
    einsum passes); the Hessian itself is a batched GEMM (cuBLAS through ``torch.matmul`` -- a plain library GEMM,
    not part of this engine).  ``fp8_scale_sweep=False``: every eligible static weight (not dynamic, not MX, with an
    ``_amax``) gets the multiplier search, under the Hessian metric where it has a Hessian
    (``_hessian_mse_search_weight``) and under the squared error where it has none (never reached by the forward, or
    ``cin % block_size != 0``), like the reference."""
    if forward_loop is None:
        warnings.warn("forward_loop must be provided for local_hessian; skipping local_hessian")
        return
    if block_size != 16:
        raise NotImplementedError("local_hessian_calibrate: block_size 16 (the NVFP4 scale block)")
    max_calibrate(model, forward_loop, distributed_sync)
    acc: dict[int, list] = {}                              # id(weight_quantizer) -> [H, n_tokens]
    handles = []

    def hook(lin, args):
        if not args:
            return
        cin = lin.weight.shape[1]
        if cin % block_size:
            return
        _local_hessian_update(acc.setdefault(id(lin.weight_quantizer), [None, 0]), args[0], cin, block_size)

    mods = [m for m in model.modules() if is_quantized_linear(m) and m.weight_quantizer.is_enabled]
    for m in mods:
        handles.append(m.register_forward_pre_hook(hook))
        m.weight_quantizer.disable()
    try:
        forward_loop(model)
    finally:
        for h in handles:
            h.remove()
        for m in mods:
            m.weight_quantizer.enable()
    for m in mods:
        q = m.weight_quantizer
        if q._dynamic or q.is_mx_format or getattr(q, "_amax", None) is None:
            continue
        e = acc.get(id(q))
        hess = None if e is None or e[1] == 0 else e[0] / e[1]
        if fp8_scale_sweep and q.is_nvfp4_static:
            best = ops.nvfp4_fp8_scale_sweep(_pad_blocks16(m.weight), q._global_amax.reshape(1), hessian=hess)
            q.amax = best.reshape(q._amax.shape)
        elif not fp8_scale_sweep and q._calibrator is not None:
            # the multiplier search (:720-728): under the Hessian metric where the forward reached this weight, else
            # the plain squared error
            if hess is None:
                _mse_search_weight(m, step_size, start_multiplier, stop_multiplier)
            else:
                _hessian_mse_search_weight(m, hess, step_size, start_multiplier, stop_multiplier)
    if debug:
        model._local_hessian_accumulators = acc


def _local_hessian_update(entry: list, x: torch.Tensor, cin: int, block_size: int = 16) -> list:
    """``_LocalHessianAccumulator.accumulate`` (model_calib.py:848-860) on ``entry = [H, n_tokens]``: add the
    per-cin-block ``X^T X`` of the activation ``x`` (``[..., cin]``, taken in fp32) to ``H`` ([cin / block_size,
    block_size, block_size]; ``None`` before the first batch) and its token count to ``n_tokens``.  The normalized
    Hessian is ``H / n_tokens``."""
    xt = x.reshape(-1, cin).to(torch.float32).T.reshape(cin // block_size, block_size, -1)
    h = xt @ xt.transpose(-1, -2)
    entry[0] = h if entry[0] is None else entry[0].add_(h)
    entry[1] += x.numel() // cin
    return entry


def _hessian_mse_search_weight(m, hess, step_size, start_multiplier, stop_multiplier, round_mult=True):
    """``MseCalibrator`` with the local-Hessian ``error_func`` (calib/mse.py:84-172, model_calib.py:891-896) on one
    weight: for every multiplier ``c`` of ``linspace(start, stop, ceil((stop - start) / step) + 1)``, fake-quantize the
    fp32 weight at ``initial_amax * c`` with the quantizer itself, weight each element's error by the loss
    ``dw^T H dw`` of its 16-element cin block (einsum ``cnb,nbd,cnd->cn``), sum that per amax slot, and keep the
    ``torch.argmin`` multiplier.  ``round_mult``: the candidate amax as torch forms it on CUDA (the multiplier rounded
    to the amax dtype first, ``MseCalibrator``'s default) or, False, on CPU.  A composed loop of torch and the engine's
    fake-quant kernels (calibration only, off the hot path)."""
    q = m.weight_quantizer
    a0 = q._amax.clone().detach()
    w = m.weight
    if q.is_static_block_quant:                              # the calibration layout: [n_blocks, block]
        q._setup_for_blockquant(w)
        w = q._process_for_blockquant(w)
    x = w.detach().to(torch.float32)
    cout, bs = m.weight.shape[0], hess.shape[-1]
    hess = hess.to(device=x.device, dtype=torch.float32)
    axis = q._calibrator._axis                               # convert_quantization_axis_to_reduce_axis (:128-143)
    if axis is not None:
        keep = {a % x.dim() for a in ((axis,) if isinstance(axis, int) else axis)}
        dims = [d for d in range(x.dim()) if d not in keep]
    n_steps = math.ceil((stop_multiplier - start_multiplier) / step_size) + 1
    cands = torch.linspace(start_multiplier, stop_multiplier, steps=n_steps, device=x.device)
    losses = []
    for c in cands:
        amax = a0 * c
        if not round_mult:
            amax = (a0.float() * c).to(amax.dtype)
        dw = (x - _mse_quant_func(x, amax, q)).view(cout, -1, bs)
        block_loss = torch.einsum("cnb,nbd,cnd->cn", dw, hess, dw).reshape(-1)
        err = block_loss.unsqueeze(-1).expand(-1, bs).reshape(x.shape)
        losses.append(err.sum() if axis is None else err.sum(dim=dims) if dims else err)
    best = cands[torch.argmin(torch.stack(losses), dim=0)]
    if best.ndim:
        best = best.view_as(a0)
    q.amax = a0 * best


def _mse_quant_func(x, amax, quantizer):
    """model_calib.py:640-665 (kept for API parity: the fused sweep reads the format off ``quantizer`` instead of
    calling this per candidate)."""
    saved = quantizer._amax
    quantizer._amax = amax
    try:
        return quantizer._fake_quantize(x)
    finally:
        quantizer._amax = saved


# ---- SmoothQuant -----------------------------------------------------------------------------------
@torch.no_grad()
def _apply_weight_pre_quant_scale(linear, pre_quant_scale):
    """model_calib.py:1209-1224."""
    linear.weight.copy_((linear.weight * pre_quant_scale.to(linear.weight.device).squeeze()[None, :])
                        .to(linear.weight.dtype))     # in-place under no_grad: bumps weight._version
    linear.weight_quantizer.reset_amax()
    max_calibrate(linear, lambda lin: lin.weight_quantizer(lin.weight))


@torch.no_grad()
def apply_pre_quant_scale_and_smooth(linear, pre_quant_scale):
    """model_calib.py:1227-1271."""
    assert is_quantized_linear(linear)
    assert linear.input_quantizer.pre_quant_scale is None, "pre_quant_scale should be None first!"
    assert torch.all(pre_quant_scale > 0), "pre_quant_scale should be positive"
    pre_quant_scale = pre_quant_scale.to(torch.float32)
    linear.input_quantizer.pre_quant_scale = pre_quant_scale.to(linear.weight.dtype)
    inv_scale = pre_quant_scale.reciprocal()  # == 1.0 / pre_quant_scale (Tensor.__rtruediv__)
    _apply_weight_pre_quant_scale(linear, inv_scale)
    if linear.input_quantizer.amax is not None:
        a = linear.input_quantizer._amax_for_smoothing.to(device=linear.weight.device, dtype=linear.weight.dtype)
        linear.input_quantizer.amax = (a * pre_quant_scale.to(a.device)).amax().to(linear.weight.dtype)


@torch.no_grad()
def smoothquant(model: nn.Module, forward_loop: Callable | None = None, alpha: float = 1.0):
    """model_calib.py:1274-1358."""
    assert forward_loop is not None, "forward_loop must be provided for smoothquant"
    for m in model.modules():
        if is_quantized_linear(m) and m.input_quantizer.is_enabled and m.input_quantizer.axis is None:
            m.input_quantizer.axis = -1
    max_calibrate(model, forward_loop)
    smoothed = 0
    for name, m in model.named_modules():
        if not is_quantized_linear(m):
            continue
        iq = m.input_quantizer
        if not hasattr(iq, "_amax"):
            warnings.warn(f"{name} is not calibrated, skip smoothing")
            continue
        if iq.num_bits != 8 or m.weight_quantizer.num_bits != 8 or iq.axis != -1:
            warnings.warn(f"Only int8 per-channel smoothing is supported, skip {name}")
            continue
        act_amax = iq.amax.float()
        wslots = torch.zeros(m.weight.shape[1], dtype=torch.float32, device=m.weight.device)
        ops.amax_cols_(wslots, m.weight)  # weight.abs().amax(dim=0, keepdim=True)
        weight_scale = ops.amax_export(wslots, m.weight.dtype).reshape(1, -1)
        scale_a = (weight_scale.pow(1 - alpha) / act_amax.pow(alpha)).squeeze()
        dtype, device = m.weight.dtype, m.weight.device
        iq._amax_for_smoothing = act_amax.cpu()
        iq.reset_amax()
        iq.axis = None
        iq.amax = act_amax.amax().to(dtype=dtype, device=device)
        eps = 1.0 / (1 << 31)
        if scale_a.min() <= eps:
            scale_a[act_amax.squeeze() <= eps] = 1
        scale_a = scale_a.clamp(min=1e-4, max=1e4)
        apply_pre_quant_scale_and_smooth(m, scale_a)
        smoothed += 1
    return smoothed


# ---- AWQ-lite -----------------------------------------------------------------------------------------
def _awq_block_size(weight, wq):
    bs = wq.block_sizes
    if not bs:
        return None
    return bs.get(-1) or bs.get(weight.dim() - 1)


def get_weight_scale(weight, block_size=None):
    """model_calib.py:1453-1469: mean over rows of |W| / (blockamax + tiny), in the weight dtype.  A ragged last
    block is zero-padded before its amax is taken, as in the reference."""
    if block_size and weight.shape[-1] % block_size == 0:
        sums = torch.zeros(weight.shape[-1], dtype=torch.float32, device=weight.device)
        ops.awq_weight_scale_sums_(sums, weight.contiguous(), block_size)
        return (sums / weight.shape[0]).to(weight.dtype).to(torch.float32)
    cin = weight.shape[-1]
    w = weight.abs()
    if block_size:
        w = F.pad(w, (0, (-cin) % block_size))
        shape = w.shape
        w = w.reshape(-1, block_size)
        scale = (w / (w.amax(dim=1, keepdim=True) + torch.finfo(weight.dtype).tiny)).reshape(shape)[..., :cin]
    else:
        scale = w / (w.amax(dim=1, keepdim=True) + torch.finfo(weight.dtype).tiny)
    return scale.mean(0).to(torch.float32)


def get_act_scale_(acc, x):
    """model_calib.py:1471-1472: ``acc += x.abs().view(-1, C).mean(0).to(float32)`` -- one column-sum kernel.  The
    reference's mean is taken IN THE ACTIVATION DTYPE (fp32 accumulation inside ATen, result rounded to bf16 / fp16),
    so the fp32 column sums are divided and rounded to that dtype before they are accumulated."""
    c = x.shape[-1]
    tmp = torch.zeros(c, dtype=torch.float32, device=x.device)
    ops.abssum_cols_(tmp, x.contiguous())
    acc += (tmp / (x.numel() // c)).to(x.dtype).to(torch.float32)
    return acc


def get_scale(x_max, w_max, alpha):
    """model_calib.py:1474-1487."""
    scales = (x_max.pow(alpha) / (w_max.to(x_max.device).pow(1 - alpha) + torch.finfo(torch.float32).tiny)) \
        .clamp(min=1e-4, max=1e4).view(-1)
    return (scales / (scales.max() * scales.min()).sqrt()).view(-1)


class _AWQLiteState:
    def __init__(self, module, alpha_step):
        self.block_size = _awq_block_size(module.weight, module.weight_quantizer)
        self.weight_scale = get_weight_scale(module.weight, self.block_size)
        self.act_scale = torch.zeros(module.weight.shape[1], dtype=torch.float32, device=module.weight.device)
        self.alphas = [round(float(a), 6) for a in torch.arange(0, 1.0 + alpha_step, alpha_step)]
        self.loss = torch.zeros(len(self.alphas), dtype=torch.float32, device=module.weight.device)
        self.num_cache_steps = 0
        self.num_search_steps = 0
        self.is_input_quantized = module.input_quantizer.is_enabled
        self.best_alpha = None
        self.best_scale = None


@torch.no_grad()
def awq_lite(model: nn.Module, forward_loop: Callable, alpha_step: float = 0.1, debug: bool = False, **kw):
    """model_calib.py:1395-1722 for plain (non-MoE, non-TP) quantized linears.

    The search step of the reference runs, per alpha, ``W * s`` -> per-block amax -> INT4 fake quant
    as ~6 ATen passes over W; here it is ONE fused kernel (``ops.awq_scale_fake_quant``).
    """
    if forward_loop is None:
        warnings.warn("forward_loop must be provided for awq_lite; skipping awq_lite")
        return
    mods = [(n, m) for n, m in model.named_modules() if is_quantized_linear(m) and m.weight_quantizer.is_enabled]
    state = {"cache": True}
    for _, m in mods:
        m.awq_lite = _AWQLiteState(m, alpha_step)
        if m.input_quantizer.is_enabled:
            m.input_quantizer.disable()
            m.input_quantizer.axis = -1

        def fwd(self, x, _orig=type(m).forward):
            st = self.awq_lite
            out_actual = F.linear(x, self.weight, self.bias)
            if x.numel() == 0:
                return out_actual
            if state["cache"]:
                get_act_scale_(st.act_scale, x)
                st.num_cache_steps += 1
                if st.is_input_quantized:
                    self.input_quantizer._calibrator.collect(x)
                return out_actual
            wq = self.weight_quantizer
            for i, alpha in enumerate(st.alphas):
                s = get_scale(st.act_scale, st.weight_scale, alpha)
                xs = ops.scale_cols(x.contiguous(), s.reciprocal().to(self.weight.dtype))
                if st.block_size and self.weight.shape[-1] % st.block_size == 0 and isinstance(wq.num_bits, int):
                    wqd = ops.awq_scale_fake_quant(self.weight, s.to(self.weight.dtype), st.block_size,
                                                   wq.num_bits, wq._narrow_range)
                else:  # ragged last dim (padding) or non-integer format: scale kernel + quantizer
                    wqd = wq(ops.scale_cols(self.weight.contiguous(), s.to(self.weight.dtype)))
                out = F.linear(xs, wqd, self.bias)
                st.loss[i] += (out - out_actual).float().pow(2).mean()
            st.num_search_steps += 1
            return out_actual

        m._b200_orig_forward = m.forward
        m.forward = fwd.__get__(m, type(m))

    forward_loop(model)  # pass 1: cache activation statistics
    for _, m in mods:
        st = m.awq_lite
        if st.num_cache_steps > 0:
            st.act_scale = st.act_scale / st.num_cache_steps
        if st.is_input_quantized and m.input_quantizer._calibrator.compute_amax() is not None:
            m.input_quantizer.load_calib_amax()
    state["cache"] = False
    forward_loop(model)  # pass 2: search
    def collapse_input_amax(m):
        """Per-channel input amax of the cache pass -> per-tensor, the per-channel one kept for smoothing."""
        iq = m.input_quantizer
        if iq.amax is not None:
            act_amax = iq.amax
            iq._amax_for_smoothing = act_amax.cpu()
            iq.reset_amax()
            iq.axis = None
            iq.amax = act_amax.amax()
        iq.enable()

    for name, m in mods:
        st = m.awq_lite
        m.forward = m._b200_orig_forward
        del m._b200_orig_forward
        if st.num_cache_steps > 0 and st.num_search_steps == 0:
            warnings.warn(f"awq_lite: Calling `forward_loop(model)` the second time did not forward data through the"
                          f" {name}. Please provide a valid `forward_loop` function that can be used to forward data"
                          " through the model many times.")
        ok = (st.num_cache_steps > 0 and st.num_search_steps > 0 and not bool(torch.isnan(st.act_scale).any())
              and not bool(torch.isnan(st.weight_scale).any()))
        if ok:
            for q in (m.weight_quantizer, m.input_quantizer):
                if hasattr(q, "_pre_quant_scale"):
                    delattr(q, "_pre_quant_scale")
            if st.is_input_quantized:
                collapse_input_amax(m)
            losses = st.loss.tolist()
            st.best_alpha = st.alphas[min(range(len(losses)), key=losses.__getitem__)]
            st.best_scale = get_scale(st.act_scale, st.weight_scale, st.best_alpha)
            apply_pre_quant_scale_and_smooth(m, 1.0 / st.best_scale)
        else:
            # model_calib.py:1673-1714: max calibration (the input quantizer is still disabled) and a neutral all-ones
            # pre_quant_scale, so that export sees the same AWQ format on every linear
            warnings.warn(f"awq_lite: Disabling for {name}, quantizing with max calibration.")
            max_calibrate(m, lambda mod: mod.weight_quantizer(mod.weight))
            m.input_quantizer.pre_quant_scale = torch.ones(m.weight.shape[1], dtype=m.weight.dtype,
                                                           device=m.weight.device)
            if st.is_input_quantized:
                collapse_input_amax(m)
        if not debug:
            delattr(m, "awq_lite")
    _finalize_static_nvfp4(model)


# ---- AWQ-clip ------------------------------------------------------------------------------------------
@torch.no_grad()
def awq_clip(model: nn.Module, forward_loop: Callable, max_co_batch_size: int = 1024, max_tokens_per_batch: int = 64,
             min_clip_ratio: float = 0.5, shrink_step: float = 0.05, debug: bool = False, **kw):
    """model_calib.py:1725-1940: per-block (or per-tensor) clip-ratio search of the weight amax.

    For every shrink ratio the weight is fake-quantized with ``amax * shrink`` (the fused kernels) and the
    per-block partial outputs ``sum_block(x * w)`` of up to ``max_tokens_per_batch`` tokens are compared
    with the unquantized ones; the ratio with the smallest accumulated squared error wins per block.

    Like the reference:
      * only weights with ``block_sizes`` are searched (a dynamic-block weight, e.g. NVFP4, clips its per-tensor
        amax); every other quantizer -- per-channel INT8 or per-tensor FP8 weights too -- is max-calibrated by the
        same forward loop;
      * an input quantizer that was enabled is max-calibrated on every batch and stays disabled during the loop,
        so the search sees unquantized inputs;
      * a searched weight quantizer is disabled during the loop and re-enabled with its best amax only when its
        linear saw tokens.  A linear the loop never reaches keeps its max amax and stays disabled (with its input
        quantizer), as the reference leaves it.
    The weight amax keeps the weight dtype (no fp32 promotion: the reference's awq_clip does not promote)."""
    assert forward_loop is not None, "forward_loop must be provided for awq_clip"
    mods = [(n, m) for n, m in model.named_modules() if is_quantized_linear(m) and m.weight_quantizer.is_enabled
            and m.weight_quantizer.block_sizes is not None]
    ratios = [round(float(k), 2) for k in torch.arange(min_clip_ratio, 1.0, shrink_step)] + [1.0]
    for _, m in mods:
        wq = m.weight_quantizer
        wq.reset_amax()
        enable_stats_collection(wq)
        wq(m.weight)
        finish_stats_collection(wq)
        st = type("AWQClipState", (), {})()
        st.w_amax = wq.amax.clone()
        st.block_size = _awq_block_size(m.weight, wq)
        st.per_tensor = wq.axis is None and wq.block_sizes.get("type") == "dynamic"
        st.num_tokens = 0
        st.is_input_quantized = m.input_quantizer.is_enabled
        co, ci = m.weight.shape
        shape = () if st.per_tensor else (co, math.ceil(ci / st.block_size))
        st.loss = {k: torch.zeros(shape, device=m.weight.device) for k in ratios}
        m.awq_clip = st
        wq.disable()

        def fwd(self, x, _ratios=ratios):
            st, wq, iq = self.awq_clip, self.weight_quantizer, self.input_quantizer
            if st.is_input_quantized:                # model_calib.py:1873-1876
                iq.enable()
                max_calibrate(iq, lambda q: q(x), distributed_sync=False)
                iq.disable()
            inputs = x
            w = self.weight
            wq.enable()
            if st.per_tensor:
                out_actual = inputs @ w.T
                st.num_tokens += inputs.shape[0]
                for shrink in _ratios:
                    wq.amax = st.w_amax * shrink
                    st.loss[shrink] += ((inputs @ wq(w).T) - out_actual).float().pow(2).mean()
            else:
                xs = inputs.reshape(-1, inputs.shape[-1])
                xs = xs[0:: max(1, xs.shape[0] // max_tokens_per_batch)]
                st.num_tokens += xs.shape[0]
                bs, (co, ci) = st.block_size, w.shape
                pad = (-ci) % bs
                wp = F.pad(w, (0, pad)) if pad else w
                xp = F.pad(xs, (0, pad)) if pad else xs
                xb = xp.reshape(1, xp.shape[0], -1, bs)
                for c0 in range(0, co, max_co_batch_size):
                    c1 = min(c0 + max_co_batch_size, co)
                    wb = wp[c0:c1].reshape(c1 - c0, 1, -1, bs)
                    org = (xb * wb).sum(dim=-1)
                    for shrink in _ratios:
                        wq.amax = st.w_amax * shrink
                        cur = wq(w)[c0:c1]
                        cur = (F.pad(cur, (0, pad)) if pad else cur).reshape(wb.shape)
                        st.loss[shrink][c0:c1] += ((xb * cur).sum(dim=-1) - org).float().pow(2).mean(dim=1)
            wq.amax = st.w_amax
            wq.disable()
            return F.linear(x, w, self.bias)

        m._b200_orig_forward = m.forward
        m.forward = fwd.__get__(m, type(m))
    # the loop also max-calibrates every other quantizer (model_calib.py:1911-1920)
    enable_stats_collection(model)
    try:
        forward_loop(model)
    finally:
        for _, m in mods:
            m.forward = m._b200_orig_forward
            del m._b200_orig_forward
    if b200_dist.is_initialized():
        b200_dist.sync_calibrator_amax(model)
    finish_stats_collection(model)
    for _, m in mods:
        st = m.awq_clip
        if st.num_tokens > 0:                        # postprocess (model_calib.py:1922-1935)
            best_loss = torch.full_like(st.w_amax.float(), float("inf"))
            best = torch.zeros_like(st.w_amax)
            for shrink, loss in st.loss.items():
                loss = loss.reshape(st.w_amax.shape)
                better = loss < best_loss
                best_loss = torch.where(better, loss, best_loss)
                best = torch.where(better, st.w_amax * shrink, best)
            st.best_clip_val = best
            m.weight_quantizer.amax = best
            m.weight_quantizer.enable()
            if st.is_input_quantized:
                m.input_quantizer.enable()
        if not debug:
            delattr(m, "awq_clip")


# ---- GPTQ ------------------------------------------------------------------------------------------
# weight updates per path of gptq_blockwise_update: "gptq.kernel" (the column kernel) and "gptq.composed"
stats: collections.Counter = collections.Counter()


def update_hessian(input, hessian, n_samples):
    """utils/calib_utils.py:50-77: running mean of ``2 X X^T`` over tokens; the same torch ops in the same order.
    Zero tokens (an MoE expert that received none) return ``hessian`` itself unchanged."""
    import math

    input_flat = input.reshape(-1, input.shape[-1]).t().float()
    batch_size = input_flat.shape[1]
    if batch_size == 0:
        return hessian, n_samples
    hessian *= n_samples / (n_samples + batch_size)
    n_samples += batch_size
    scaled_input = math.sqrt(2 / n_samples) * input_flat
    hessian.add_((scaled_input @ scaled_input.t()).to(hessian.device))
    return hessian, n_samples


def compute_hessian_inverse(hessian, weight, perc_damp):
    """utils/calib_utils.py:80-113: upper Cholesky factor of the damped inverse Hessian.  Columns that are all zero in
    ``weight`` are zeroed in the Hessian (diagonal 1); a Hessian that is not positive definite gives the identity,
    with a warning."""
    h = hessian.clone()
    zero_cols = torch.nonzero(weight.eq(0).all(dim=0)).unsqueeze(-1)
    h[zero_cols, :] = 0
    h[:, zero_cols] = 0
    h[zero_cols, zero_cols] = 1
    damp = perc_damp * torch.mean(torch.diag(h))
    diag_indices = torch.arange(h.shape[0], device=h.device)
    h[diag_indices, diag_indices] += damp
    try:
        h = torch.cholesky_inverse(torch.linalg.cholesky(h))
        return torch.linalg.cholesky(h, upper=True)
    except (RuntimeError, torch.linalg.LinAlgError):
        warnings.warn("Hessian is not positive definite, using identity matrix")
        return torch.eye(h.shape[0], device=h.device, dtype=h.dtype)


def gptq_blockwise_update_composed(weight, h_inv, block_size, quantize_fn):
    """utils/calib_utils.py:241-276 as written: per column, fake-quantize the whole working matrix with
    ``quantize_fn`` and keep one column, then a rank-1 ``addr_``.  Used for quantizers outside the GPTQ kernel's scope,
    and by tests as the reference on the GPU."""
    num_cols = weight.shape[1]
    for block_start in range(0, num_cols, block_size):
        block_end = min(block_start + block_size, num_cols)
        n_cols_blk = block_end - block_start
        h_inv_cho_blk = h_inv[block_start:block_end, block_start:block_end]
        wblk = weight.clone()
        errs = torch.zeros_like(weight[:, block_start:block_end])
        for i in range(n_cols_blk):
            w_ci = wblk[:, block_start + i]
            d = h_inv_cho_blk[i, i]
            qdq = quantize_fn(wblk)
            weight[:, block_start + i] = qdq[:, block_start + i]
            err = (w_ci - qdq[:, block_start + i]) / d
            wblk[:, block_start + i: block_end].addr_(err, h_inv_cho_blk[i, i:], alpha=-1)
            errs[:, i] = err
        weight[:, block_end:].addmm_(errs, h_inv[block_start:block_end, block_end:], alpha=-1)


def gptq_blockwise_update(weight, h_inv, block_size, quantizer) -> bool:
    """GPTQ update of the fp32 working ``weight`` in place: the column kernel (``ops.gptq_blockwise_update``) when the
    quantizer is inside its scope, else the composed loop.  Returns whether the kernel ran; ``stats`` counts both."""
    desc = ops.gptq_quantizer_desc(quantizer, weight.shape, block_size, weight.device) if weight.is_cuda else None
    if desc is not None:
        ops.gptq_blockwise_update(weight, h_inv, block_size, quantizer, desc=desc)
        stats["gptq.kernel"] += 1
        return True
    stats["gptq.composed"] += 1
    gptq_blockwise_update_composed(weight, h_inv, block_size, quantizer)
    return False


@torch.no_grad()
def gptq(model: nn.Module, forward_loop: Callable | None = None, perc_damp: float = 0.01, block_size: int = 128,
         fused: bool = False, layerwise=None):
    """model_calib.py:2191-2271 (non-layerwise): ``max_calibrate`` (static NVFP4 promotion and shared global amax
    included), one forward that accumulates ``2 X X^T`` per quantized linear with an enabled weight quantizer (X is
    the input quantizer's output when that quantizer is enabled; weight quantizers are disabled during this pass),
    then per module the blockwise update of ``weight.float()`` with the inverse Hessian, written back in the weight's
    dtype.  ``fused`` is accepted for config parity: the kernel implements the unfused semantics."""
    from .config import GPTQCalibConfig

    cfg = GPTQCalibConfig(perc_damp=perc_damp, block_size=block_size, fused=fused, layerwise=layerwise)
    if cfg.layerwise_enabled:
        raise NotImplementedError(
            "gptq: layerwise calibration is not part of model_optimizer_b200's own API; run the reference's "
            "mtq.quantize under model_optimizer_b200.backend.install(), whose layerwise_calibrate drives the GPTQ "
            "kernel through the registered 'b200' GPTQ helper")
    max_calibrate(model, forward_loop)
    layers = [(n, m) for n, m in model.named_modules() if is_quantized_linear(m) and m.weight_quantizer.is_enabled]
    if not layers:
        warnings.warn("No quantized linear layers found, skipping GPTQ")
        return
    state = {}
    for name, m in layers:
        state[name] = [torch.zeros(m.weight.shape[-1], m.weight.shape[-1], dtype=torch.float32,
                                   device=m.weight.device), 0]

    def make_hook(name):
        def hook(lin, args):
            if not args:
                return
            inp = args[0]
            iq = lin.input_quantizer
            x = iq(inp) if iq is not None and iq.is_enabled else inp
            st = state[name]
            st[0], st[1] = update_hessian(x, st[0], st[1])
        return hook

    handles = [m.register_forward_pre_hook(make_hook(name)) for name, m in layers]
    held = [q for n, q in _quantizers(model) if n.endswith("weight_quantizer") and q.is_enabled]
    for q in held:                      # set_quantizer_by_cfg_context(*weight_quantizer: enable False)
        q.disable()
    try:
        if forward_loop is not None:
            forward_loop(model)
    finally:
        for h in handles:
            h.remove()
        for q in held:
            q.enable()
    for name, m in layers:
        hessian = state[name][0].to(m.weight.device)
        weight = m.weight.data.float().clone()
        h_inv = compute_hessian_inverse(hessian, weight, cfg.perc_damp)
        gptq_blockwise_update(weight, h_inv, cfg.block_size, m.weight_quantizer)
        m.weight.data = weight.reshape(m.weight.shape).to(m.weight.data.dtype)
        if hasattr(m, "invalidate_weight_cache"):
            m.invalidate_weight_cache()
        state[name] = None


__all__ = ["max_calibrate", "mse_calibrate", "local_hessian_calibrate", "nvfp4_act_headroom_calibrate", "find_shared_weight_groups", "SHARED_PATTERNS", "smoothquant", "awq_lite", "awq_clip", "enable_stats_collection",
           "gptq", "update_hessian", "compute_hessian_inverse", "gptq_blockwise_update",
           "gptq_blockwise_update_composed",
           "finish_stats_collection", "weight_only_quantize", "apply_pre_quant_scale_and_smooth",
           "get_weight_scale", "get_scale"]
