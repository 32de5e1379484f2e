"""Quantizer input rotation -- the b200quant counterpart of ``normalized_hadamard_transform`` in
``modelopt/torch/quantization/nn/functional.py`` (:76-138): the same block selection, checks and messages, with the
transform run by ``b200q_hadamard`` (``model_optimizer_b200.ops.hadamard``) instead of the external
``fast_hadamard_transform`` package.  CPU tensors raise, like every op.
"""

from __future__ import annotations

from torch.autograd import Function

from .. import ops
from ..tensor_quant import _entry


def _largest_pow2_divisor(n: int) -> int:
    """Return the largest power of 2 that divides n."""
    return n & (-n)


def _is_pow2(n: int) -> bool:
    return n > 0 and (n & (n - 1)) == 0


def rotate_block_size(dim: int, block_size: int | None = None) -> int:
    """The block the transform runs on for a last dim of ``dim`` (functional.py:108-130): ``block_size`` when given,
    else the whole dim when it is a power of 2, else its largest power-of-2 divisor."""
    if block_size is None:
        if _is_pow2(dim):
            block_size = dim
        else:
            block_size = _largest_pow2_divisor(dim)
            if block_size < 2:
                raise RuntimeError(
                    f"Block RHT: dimension {dim} has no power-of-2 divisor >= 2. "
                    "Set rotate.block_size explicitly (e.g. 128) or use a dimension divisible by a power of 2."
                )
    if not _is_pow2(block_size):
        raise ValueError(f"Block RHT: block_size must be power of 2, got {block_size}.")
    if dim % block_size != 0:
        raise RuntimeError(
            f"Block RHT: inputs.shape[-1]={dim} is not divisible by block_size={block_size}. "
            f"Use a block_size that divides {dim} (e.g. {_largest_pow2_divisor(dim)})."
        )
    return block_size


class HadamardFunction(Function):
    """y = H x per block; H is symmetric and orthonormal, so the gradient is the same transform of the gradient."""

    @staticmethod
    def forward(ctx, inputs, block_size, amax_slot=None):
        ctx.block_size = block_size
        return ops.hadamard(inputs, block_size, amax_slot)

    @staticmethod
    def backward(ctx, grad_outputs):
        return ops.hadamard(grad_outputs, ctx.block_size), None, None


_hadamard = _entry(HadamardFunction)


def normalized_hadamard_transform(inputs, rotate_fp32=False, block_size=None, *, amax_slot=None):
    """Normalized fast Hadamard transform along the last dim, per block of ``block_size`` elements (see
    ``rotate_block_size`` for the default).

    ``rotate_fp32`` is accepted for parity with the reference: the kernel always works in fp32 and rounds once to the
    input dtype, which is what computing in fp32 and casting back gives, so both settings return the same bits.
    ``amax_slot`` (fp32 [1], optional): the same pass also folds max|y| into it (a per-tensor max calibrator's collect
    of the rotated tensor).
    """
    del rotate_fp32
    bs = rotate_block_size(inputs.shape[-1], block_size)
    return _hadamard(inputs, bs, amax_slot)


__all__ = ["normalized_hadamard_transform", "rotate_block_size", "HadamardFunction"]
