"""Export-side quant-and-pack -- mirror of the part of ``modelopt/torch/export/quant_utils.py`` that sits
directly after the hot path (SURVEY.md 8f-1): scaling-factor getters (:225-362), ``to_quantized_weight``
(:836-938), ``pack_int4_in_uint8`` (:792-833), ``from_quantized_weight`` (:941-978) and a per-linear
``export_quantized_linear`` producing the unified-HF tensor names (``weight``, ``weight_scale``,
``weight_scale_2``, ``input_scale``, ``pre_quant_scale``; export/unified_export_hf.py:569-700).

Scalar divisions use a 0-dim device tensor as divisor so that CUDA performs the IEEE division the
reference's CPU path performs (``tensor / python_scalar`` multiplies by a reciprocal on CUDA)."""

from __future__ import annotations

import torch

from . import ops
from .nn.tensor_quantizer import fp8_max_for_normalization
from .qtensor import FP8QTensor, MXFP4QTensor, MXFP8QTensor, NVFP4QTensor

QUANTIZATION_NONE = None
QUANTIZATION_FP8 = "fp8"
QUANTIZATION_FP8_PC_PT = "fp8_pc_pt"
QUANTIZATION_FP8_PB_WO = "fp8_pb_wo"
QUANTIZATION_INT8_SQ = "int8_sq"
QUANTIZATION_INT8_WO = "int8_wo"
QUANTIZATION_INT4_AWQ = "int4_awq"
QUANTIZATION_NVFP4 = "nvfp4"
QUANTIZATION_NVFP4_AWQ = "nvfp4_awq"
QUANTIZATION_W4A16_NVFP4 = "w4a16_nvfp4"
QUANTIZATION_W4A8_NVFP4_FP8 = "w4a8_nvfp4_fp8"
QUANTIZATION_MXFP4 = "mxfp4"
QUANTIZATION_MXFP8 = "mxfp8"
QUANTIZATION_W4A8_MXFP4_FP8 = "w4a8_mxfp4_fp8"
_MXFP4_FORMATS = (QUANTIZATION_MXFP4, QUANTIZATION_W4A8_MXFP4_FP8)
_INT8_FORMATS = (QUANTIZATION_INT8_SQ, QUANTIZATION_INT8_WO)
# block scales derived from weight_scale_2 = global amax / (6 * 448) by the pack kernel
_NVFP4_GLOBAL_FORMATS = (QUANTIZATION_NVFP4, QUANTIZATION_NVFP4_AWQ, QUANTIZATION_W4A16_NVFP4)
_NVFP4_FORMATS = (*_NVFP4_GLOBAL_FORMATS, QUANTIZATION_W4A8_NVFP4_FP8)


def _tdiv(t: torch.Tensor, scalar: float) -> torch.Tensor:
    return t / torch.tensor(float(scalar), device=t.device, dtype=torch.float32)


def get_quantization_format(module) -> str | None:
    """quant_utils.py:485-604 restricted to the formats this engine packs, checked in the reference's order."""
    wq = getattr(module, "weight_quantizer", None)
    if wq is None or not wq.is_enabled:
        return QUANTIZATION_NONE
    iq = getattr(module, "input_quantizer", None)
    iq_on = iq is not None and iq.is_enabled
    bs = wq.block_sizes or {}
    if wq.num_bits == 4 and bs:
        return QUANTIZATION_INT4_AWQ
    if wq.num_bits == 8:
        return QUANTIZATION_INT8_SQ if iq_on else QUANTIZATION_INT8_WO
    if wq.num_bits == (4, 3):
        if bs:
            return QUANTIZATION_MXFP8 if wq.is_mx_format else QUANTIZATION_FP8_PB_WO
        return QUANTIZATION_FP8_PC_PT if wq.axis == 0 else QUANTIZATION_FP8
    if wq.num_bits == (2, 1):
        scale_bits = bs.get("scale_bits")
        if getattr(iq, "_pre_quant_scale", None) is not None or getattr(module, "fused_with_prequant", False):
            return QUANTIZATION_NVFP4_AWQ
        if not iq_on and scale_bits == (4, 3):
            return QUANTIZATION_W4A16_NVFP4
        fp8_input = iq_on and iq.num_bits == (4, 3) and iq.block_sizes is None
        if fp8_input and bs.get("type", "static") == "dynamic":
            if scale_bits == (8, 0):
                return QUANTIZATION_W4A8_MXFP4_FP8
            if scale_bits == (4, 3):
                return QUANTIZATION_W4A8_NVFP4_FP8
        if scale_bits == (4, 3):
            return QUANTIZATION_NVFP4
        if scale_bits == (8, 0):
            return QUANTIZATION_MXFP4
    raise NotImplementedError(f"unsupported weight quantizer {wq}")


def get_scaling_factor(quantizer):
    """quant_utils.py:225-242: ``amax.float() / maxbound`` (NVFP4: global amax / (6 * 448), or / (6 * 256) for
    Four-Over-Six, nvfp4_tensor.py:88-107)."""
    if quantizer is None or not quantizer.is_enabled:
        return None
    amax = quantizer.export_amax()
    if amax is None:
        return None
    if quantizer.num_bits == (2, 1):
        g = getattr(quantizer, "_global_amax", None)
        src = g if g is not None else quantizer._amax
        sf = _tdiv(src.float(), 6.0 * fp8_max_for_normalization(quantizer))
    else:
        sf = _tdiv(amax.float(), quantizer.maxbound)
    assert torch.all(sf > 0), f"scaling factor {sf} not positive."
    return sf


def get_activation_scaling_factor(module, input_quantizer_name="input_quantizer"):
    """quant_utils.py:245-260; NVFP4: ``amax / (maxbound * 448)`` (nvfp4_tensor.py:209-227)."""
    q = getattr(module, input_quantizer_name, None)
    if q is None or not q.is_enabled:
        return None
    if get_quantization_format(module) in (QUANTIZATION_NVFP4, QUANTIZATION_NVFP4_AWQ):
        amax = q.export_amax()
        return None if amax is None else _tdiv(amax.float(), q.maxbound * 448.0)
    return get_scaling_factor(q)


def get_weight_scaling_factor_2(module):
    """quant_utils.py:314-336: W4A8-NVFP4-FP8 uses ``amax / 448`` so that the block scales dequantize the weight
    into the FP8 range."""
    fmt = get_quantization_format(module)
    if fmt == QUANTIZATION_W4A8_NVFP4_FP8:
        return _tdiv(module.weight_quantizer._amax.float(), 448.0).reshape(())
    if fmt in _NVFP4_GLOBAL_FORMATS:
        return get_scaling_factor(module.weight_quantizer).reshape(())
    return None


def get_weight_scaling_factor(module):
    """quant_utils.py:263-311 (NVFP4 block scales come out of the pack kernel itself)."""
    fmt = get_quantization_format(module)
    if fmt is None:
        return None
    if fmt in _NVFP4_FORMATS:
        return export_nvfp4_weight(module)[1]
    if fmt in _MXFP4_FORMATS:                     # :304-307
        w = module.weight.detach()
        return MXFP4QTensor.quantize(w, block_size=module.weight_quantizer.block_sizes[-1])[1].reshape(*w.shape[:-1], -1)
    if fmt == QUANTIZATION_MXFP8:                 # :309-310
        return MXFP8QTensor.get_weights_scaling_factor(module.weight.detach())
    return get_scaling_factor(module.weight_quantizer)


def get_prequant_scaling_factor(module):
    q = getattr(module, "input_quantizer", None)
    pqs = getattr(q, "_pre_quant_scale", None) if q is not None else None
    if pqs is None:
        return None
    assert torch.all(pqs > 0), f"prequant scaling factor {pqs} not positive."
    return pqs.squeeze()


def pack_int4_in_uint8(weight, weights_scaling_factor):
    """quant_utils.py:792-833."""
    return ops.pack_int4_export(weight.contiguous(), weights_scaling_factor.contiguous())


def export_nvfp4_weight(module):
    """(packed uint8 [N, K/2], e4m3 block scales [N, K/block], fp32 weight_scale_2): dynamic quantizers pack
    from the calibrated per-tensor amax, static ones from their per-block amax (nvfp4_tensor.py:113-167), with the
    block scales normalized by 256 instead of 448 for Four-Over-Six.  W4A8-NVFP4-FP8 packs against its own
    weight_scale_2 (``get_weight_scaling_factor_2``)."""
    wq = module.weight_quantizer
    w = module.weight.detach().contiguous()
    bs = (wq.block_sizes or {}).get(-1, 16)
    if get_quantization_format(module) == QUANTIZATION_W4A8_NVFP4_FP8:
        return ops.pack_nvfp4(w, None, block_size=bs, wsf2=get_weight_scaling_factor_2(module))
    if getattr(wq, "_global_amax", None) is not None:
        return ops.pack_nvfp4(w, wq._global_amax.reshape(1).float(), wq._amax.float().reshape(-1),
                              fp8_max_norm=fp8_max_for_normalization(wq), block_size=bs)
    return ops.pack_nvfp4(w, wq._amax.reshape(1).float(), block_size=bs)


def _row_outer(weight, scale) -> int:
    """Elements per scale entry of a per-row (``[N]`` / ``[N, 1]``) scale: the row length."""
    return weight.shape[-1] if scale.numel() > 1 else 1


def to_quantized_weight(weight, weights_scaling_factor, quantization, weights_scaling_factor2=None, block_size=None):
    """quant_utils.py:836-938, every format through a pack kernel.  Per-row scales divide as ``weight / scale[:, None]``
    does in torch (an fp32 scale promotes the quotient to fp32)."""
    weight = weight.contiguous()
    if quantization == QUANTIZATION_FP8:
        if weight.dtype == torch.float8_e4m3fn:
            return weight
        return ops.pack_fp8(weight, weights_scaling_factor.to(weight.device))
    if quantization == QUANTIZATION_FP8_PC_PT:     # :879-909 (2-D weights)
        s = weights_scaling_factor.to(weight.device).reshape(-1)
        return ops.pack_fp8(weight, s, outer=_row_outer(weight, s))
    if quantization in _INT8_FORMATS:             # :868-869
        s = weights_scaling_factor.to(weight.device).reshape(-1)
        return ops.pack_int8(weight, s, outer=_row_outer(weight, s))
    if quantization == QUANTIZATION_INT4_AWQ:
        return pack_int4_in_uint8(weight, weights_scaling_factor.to(weight.device))
    if quantization == QUANTIZATION_W4A8_NVFP4_FP8:
        assert block_size and weights_scaling_factor2 is not None
        return ops.pack_nvfp4(weight, None, block_size=block_size, wsf2=weights_scaling_factor2)[0]
    if quantization in _NVFP4_GLOBAL_FORMATS:
        assert block_size and weights_scaling_factor2 is not None
        return NVFP4QTensor.quantize(weight, block_size, None, weights_scaling_factor2)[0]._quantized_data
    if quantization == QUANTIZATION_FP8_PB_WO:    # :874-877
        return FP8QTensor.quantize(weight, weights_scaling_factor.squeeze(),
                                   block_sizes={-1: block_size, -2: block_size})[0]._quantized_data
    if quantization == QUANTIZATION_MXFP8:        # :871-872
        return MXFP8QTensor.quantize_with_scale(weight, weights_scaling_factor)
    if quantization in _MXFP4_FORMATS:            # :935-936
        return MXFP4QTensor.quantize(weight, block_size=block_size)[0]._quantized_data
    raise NotImplementedError(f"quantization format {quantization} not supported")


def from_quantized_weight(weight, weights_scaling_factor, quantization, torch_dtype, weights_scaling_factor2=None,
                          block_size=None):
    """quant_utils.py:941-978 for FP8 and INT8, and the inverse of ``to_quantized_weight`` for every other format
    through the unpack kernels.  ``block_size``: the FP8 2-D block edge; MX and NVFP4 read it from the scale shape."""
    if quantization == QUANTIZATION_FP8:
        return weight.view(torch.float8_e4m3fn).to(torch_dtype) * weights_scaling_factor.to(torch_dtype)
    if quantization == QUANTIZATION_FP8_PC_PT:
        s = weights_scaling_factor.to(weight.device).reshape(-1)
        return ops.unpack_fp8(weight, s, torch_dtype, outer=_row_outer(weight, s))
    if quantization in _INT8_FORMATS:
        s = weights_scaling_factor.to(weight.device).reshape(-1)
        return ops.unpack_int8(weight, s, torch_dtype, outer=_row_outer(weight, s))
    if quantization in _NVFP4_FORMATS:
        return ops.unpack_nvfp4(weight, weights_scaling_factor, weights_scaling_factor2, torch_dtype)
    if quantization == QUANTIZATION_FP8_PB_WO:
        q = FP8QTensor(weight.shape, torch_dtype, weight)
        return q.dequantize(torch_dtype, scale=weights_scaling_factor.float(),
                            block_sizes={-1: block_size, -2: block_size})
    if quantization == QUANTIZATION_MXFP8:
        return ops.unpack_mxfp8(weight, weights_scaling_factor, torch_dtype)
    if quantization in _MXFP4_FORMATS:
        s = weights_scaling_factor.reshape(-1, 1)
        return ops.unpack_mxfp4(weight, s, weight.numel() * 2 // s.numel(), torch_dtype)
    raise NotImplementedError(f"quantization format {quantization} not supported")


def export_quantized_linear(module) -> dict:
    """One quantized linear -> tensors with the unified-HF checkpoint names (unified_export_hf.py:569-800)."""
    fmt = get_quantization_format(module)
    out: dict = {"quantization": fmt}
    if fmt is None:
        out["weight"] = module.weight.detach()
        return out
    wq = module.weight_quantizer
    w = module.weight.detach()
    if fmt in _NVFP4_FORMATS:
        packed, scales, wsf2 = export_nvfp4_weight(module)
        out.update(weight=packed, weight_scale=scales, weight_scale_2=wsf2)
    elif fmt == QUANTIZATION_FP8_PB_WO:
        wsf = get_scaling_factor(wq)                            # amax.float() / 448, shape [N / b, 1, K / b, 1]
        out.update(weight=to_quantized_weight(w, wsf, fmt, block_size=wq.block_sizes[-1]), weight_scale=wsf.squeeze())
    elif fmt == QUANTIZATION_MXFP8:
        scale = MXFP8QTensor.get_weights_scaling_factor(w)
        out.update(weight=to_quantized_weight(w, scale, fmt), weight_scale=scale)
    elif fmt in _MXFP4_FORMATS:
        q, scale = MXFP4QTensor.quantize(w, block_size=wq.block_sizes[-1])
        out.update(weight=q._quantized_data, weight_scale=scale.reshape(*w.shape[:-1], -1))
    elif fmt == QUANTIZATION_INT4_AWQ:
        amax = wq.export_amax()  # [out, in / block]
        wsf = _tdiv(amax.float(), wq.maxbound).reshape(w.shape[0], -1)
        out.update(weight=pack_int4_in_uint8(w, wsf), weight_scale=wsf)
    else:
        # FP8: the scale keeps export_amax()'s shape (1,) in fp32, so `weight / scale` promotes to fp32 in
        # torch and the quotient is NOT rounded to the weight dtype before the e4m3 cast (unified_export_hf.py:
        # 680-683 -> quant_utils.py:854-866); FP8 per-channel and INT8 divide each row by its fp32 scale
        wsf = get_scaling_factor(wq)
        if fmt != QUANTIZATION_FP8:
            wsf = wsf.reshape(-1)
        out.update(weight=to_quantized_weight(w, wsf, fmt), weight_scale=wsf)
    isf = get_activation_scaling_factor(module)
    if isf is not None:
        out["input_scale"] = isf
    pqs = get_prequant_scaling_factor(module)
    if pqs is not None:
        out["pre_quant_scale"] = pqs
    return out


__all__ = ["get_quantization_format", "get_scaling_factor", "get_activation_scaling_factor",
           "get_weight_scaling_factor", "get_weight_scaling_factor_2", "get_prequant_scaling_factor",
           "pack_int4_in_uint8", "to_quantized_weight", "from_quantized_weight", "export_quantized_linear"]
