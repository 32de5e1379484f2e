"""Tensor quantization functionals -- the b200quant counterpart of
``modelopt/torch/quantization/tensor_quant.py``: same names, same argument meaning, every forward
is ONE fused sm_90a kernel reached through the C-ABI; backward is the reference's straight-through
estimator with the ``|x| <= amax`` clip (tensor_quant.py:290-316)."""

from __future__ import annotations

import torch
from torch.autograd import Function

from . import ops


def _ste_backward(ctx, grad_outputs, num_args):
    saved = ctx.saved_tensors
    if len(saved) == 0:
        return (grad_outputs,) + (None,) * (num_args - 1)
    inputs, amax = saved
    grad = torch.where(inputs.abs() <= amax, grad_outputs, grad_outputs.new_zeros(1))
    return (grad,) + (None,) * (num_args - 1)


def _save(ctx, pass_through_bwd, inputs, amax):
    if not pass_through_bwd and amax is not None:
        ctx.save_for_backward(inputs, amax if isinstance(amax, torch.Tensor) else inputs.new_tensor(amax))


def _axis_outer(inputs: torch.Tensor, amax: torch.Tensor) -> int:
    """``axis = amax.shape.index(amax.numel())`` then ``outer = inputs.stride(axis)``
    (tensor_quant.py:106-110 + tensor_quant_gpu.cu:127-129)."""
    if amax.numel() == 1:
        return 1
    if (amax.dim() == inputs.dim() and amax.shape[-1] == 1 and tuple(amax.shape[:-1]) == tuple(inputs.shape[:-1])):
        return inputs.shape[-1]  # per-row (per-token) amax over all leading dims: row r -> amax[r]
    if amax.squeeze().dim() > 1:
        raise ValueError("amax with more than one non-singleton dim is not supported by the fused kernels")
    axis = list(amax.shape).index(amax.numel()) if amax.dim() == inputs.dim() else None
    if axis is None:
        raise ValueError(f"cannot infer the quantization axis from amax shape {tuple(amax.shape)}")
    return inputs.stride(axis) if inputs.is_contiguous() else inputs.contiguous().stride(axis)


class FakeTensorQuantFunction(Function):
    """tensor_quant.py:319-399 -> fake_tensor_quant[_with_axis]."""

    @staticmethod
    def forward(ctx, inputs, amax, bias=None, num_bits=8, unsigned=False, narrow_range=True,
                trt_high_precision_dtype=None, pass_through_bwd=False, block_size=None, axis=None):
        if bias is not None:
            inputs = inputs - bias
        _save(ctx, pass_through_bwd, inputs, amax)
        inputs = inputs.contiguous()
        outputs = ops.fake_quant_int(inputs, amax, num_bits, unsigned, narrow_range, _axis_outer(inputs, amax))
        if bias is not None:
            outputs = outputs + bias
        return outputs

    @staticmethod
    def backward(ctx, grad_outputs):
        return _ste_backward(ctx, grad_outputs, 10)


class ScaledE4M3Function(Function):
    """tensor_quant.py:402-460 -> fake_e4m3fy[_with_axis]."""

    @staticmethod
    def forward(ctx, inputs, amax, bias, E, M, trt_high_precision_dtype=None, pass_through_bwd=False):  # noqa: N803
        if E != 4 or M != 3:
            raise NotImplementedError("Only support E=4 & M=3 for now.")
        if bias is not None:
            inputs = inputs - bias
        _save(ctx, pass_through_bwd, inputs, amax)
        inputs = inputs.contiguous()
        if amax is not None and amax.squeeze().dim() > 1:
            # amax with several non-singleton dims: the reference runs _fp8_eager here (scaled_e4m3_impl,
            # tensor_quant.py:78-79) -- e.g. per-token dynamic amax [B, T, 1] of a 3-D activation, or the
            # [A, 1, B, 1] tile amax of 2-D block quantization on the [A, b1, B, b2] view, whose per-tile amax is
            # spread over the b1 rows of its tile (a tensor b2 times smaller than the input).
            if amax.dim() == inputs.dim() and amax.shape[-1] == 1 and tuple(amax.shape[:-1]) == tuple(inputs.shape[:-1]):
                rows = amax.reshape(-1)
            elif inputs.dim() == 4 and tuple(amax.shape) == (inputs.shape[0], 1, inputs.shape[2], 1):
                rows = amax.float().expand(-1, inputs.shape[1], -1, -1).reshape(-1).contiguous()
            else:
                raise NotImplementedError(f"FP8 fake quant with amax shape {tuple(amax.shape)}")
            outputs = ops.fake_quant_fp8(inputs, rows, inputs.shape[-1], eager=True)
        else:
            outer = 1 if amax is None else _axis_outer(inputs, amax)
            outputs = ops.fake_quant_fp8(inputs, amax, outer)
        if bias is not None:
            outputs = outputs + bias
        return outputs

    @staticmethod
    def backward(ctx, grad_outputs):
        return _ste_backward(ctx, grad_outputs, 7)


# (exponent bits, mantissa bits) | int -> element format name (tensor_quant.py:30-41)
mx_format_map = {(4, 3): "E4M3", (5, 2): "E5M2", (3, 2): "E3M2", (2, 3): "E2M3", 8: "INT8", (8, 0): "E8M0",
                 (2, 1): "E2M1", (1, 2): "E1M2", (0, 3): "E0M3", (3, 0): "E3M0"}


class DynamicBlockQuantizationFunction(Function):
    """tensor_quant.py:497-568 -> _dynamic_block_quantize_impl (:157-195): NVFP4 (E2M1 + E4M3 block
    scale, the Triton branch) or an MX format (any element format + E8M0 scale, fused_amax_convert)."""

    @staticmethod
    def forward(ctx, inputs, block_size, amax, bias, num_bits, scale_bits,
                trt_high_precision_dtype=None, onnx_quantizer_type="dynamic", pass_through_bwd=True):
        # `bias` is accepted and NOT applied, exactly like the reference (_dynamic_block_quantize_forward,
        # tensor_quant.py:463-494, takes no bias)
        _save(ctx, pass_through_bwd, inputs, amax)
        num_bits = tuple(num_bits) if isinstance(num_bits, (list, tuple)) else num_bits
        scale_bits = tuple(scale_bits) if isinstance(scale_bits, (list, tuple)) else scale_bits
        if num_bits not in mx_format_map or num_bits == (8, 0):
            raise NotImplementedError(
                f"Unsupported num_bits: {num_bits}, scale_bits: {scale_bits} for dynamic block quantization.")
        if scale_bits == (8, 0):
            return ops.fake_quant_mx(inputs.contiguous(), block_size, mx_format_map[num_bits])
        if num_bits != (2, 1) or scale_bits != (4, 3):
            raise NotImplementedError(
                f"dynamic block quantization num_bits={num_bits} scale_bits={scale_bits}: the b200quant engine has "
                "kernels for NVFP4 (E2M1 + E4M3 scales) and for E8M0-scaled MX formats")
        # like the reference's Triton branch (tensor_quant.py:175-183, fp4_kernel_hopper.py:102), the NVFP4
        # fake quant always works on 16-element blocks; block_size only matters to the pack / export path
        if amax is None:
            raise ValueError("NVFP4 dynamic block quantization needs the per-tensor (global) amax")
        if amax.numel() != 1:
            amax = amax.amax()  # tensor_quant.py:173-174
        return ops.fake_quant_nvfp4(inputs.contiguous(), amax)

    @staticmethod
    def backward(ctx, grad_outputs):
        return _ste_backward(ctx, grad_outputs, 9)


class StaticBlockwiseFP4FakeQuantFunction(Function):
    """tensor_quant.py:574-604 -> static_blockwise_fp4_fake_quant."""

    @staticmethod
    def forward(ctx, x, amax, global_amax=None, quantize_block_scales=True, fp8_max_for_normalization=448.0,
                out_dtype=None, pass_through_bwd=False):
        _save(ctx, pass_through_bwd, x, amax)
        if out_dtype is not None and out_dtype != x.dtype:
            raise NotImplementedError("out_dtype != input dtype")
        return ops.fake_quant_nvfp4_static(x.contiguous(), amax, global_amax, quantize_block_scales,
                                           fp8_max_for_normalization)

    @staticmethod
    def backward(ctx, grad_outputs):
        return _ste_backward(ctx, grad_outputs, len(ctx.needs_input_grad))


class _NoCtx:
    """Stand-in for the autograd context when no graph is being recorded."""

    needs_input_grad = ()

    @staticmethod
    def save_for_backward(*tensors):
        pass


def _entry(fn):
    """``fn.apply`` under autograd; with grad mode off (calibration, inference, export) the forward is called
    directly -- ``Function.apply`` costs several microseconds per call, more than the launch it wraps."""
    apply, forward, ctx = fn.apply, fn.forward, _NoCtx()

    def call(*args):
        if torch.is_grad_enabled():
            return apply(*args)
        return forward(ctx, *args)

    call.__name__ = fn.__name__
    call.__doc__ = fn.__doc__
    return call


fake_tensor_quant = _entry(FakeTensorQuantFunction)
scaled_e4m3 = _entry(ScaledE4M3Function)
dynamic_block_quant = _entry(DynamicBlockQuantizationFunction)
static_blockwise_fp4_fake_quant = _entry(StaticBlockwiseFP4FakeQuantFunction)

__all__ = ["fake_tensor_quant", "scaled_e4m3", "dynamic_block_quant", "static_blockwise_fp4_fake_quant",
           "mx_format_map"]
