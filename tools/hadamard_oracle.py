"""Host restatement of the normalized Hadamard transform contract of ``b200q_hadamard`` (csrc/hadamard.cu), in numpy.

Test infrastructure, never imported by the product: the GPU tests compare the kernel with it bit for bit, and
``tools/gen_rotate_golden.py`` runs the reference with it standing in for ``fast_hadamard_transform``.
"""

from __future__ import annotations

import numpy as np

F32 = np.float32


def round_to(x, dtype: str):
    """float32 -> nearest value of ``dtype`` ("bf16" | "f16" | "f32"), RNE, returned as float32."""
    x = np.ascontiguousarray(x, dtype=F32)
    if dtype == "f32":
        return x.copy()
    if dtype == "f16":
        with np.errstate(over="ignore"):
            return x.astype(np.float16).astype(F32)
    if dtype != "bf16":
        raise ValueError(dtype)
    b = x.reshape(-1).view(np.uint32).astype(np.uint64)
    r = (((b + 0x7FFF + ((b >> 16) & 1)) >> 16) << 16) & 0xFFFFFFFF
    out = r.astype(np.uint32).view(F32).copy()
    out[np.isnan(x.reshape(-1))] = np.nan
    return out.reshape(x.shape)


def hadamard(x, block: int, dtype: str, scale=None):
    """The transform of every contiguous block of ``block`` (a power of 2) elements along the last dim of ``x`` (values
    of ``dtype``): fp32 stages s = 0 .. k-1 in ascending order, each mapping (x[i], x[i | 2^s]) with bit s of i clear
    to (a + b, a - b) rounded to fp32; one multiply by ``scale`` (default fl32(block ** -0.5)); one RNE rounding to
    ``dtype``.  Returns float32 values of ``dtype``."""
    x = np.asarray(x, dtype=F32)
    if block < 1 or block & (block - 1) or x.shape[-1] % block:
        raise ValueError(f"block {block} does not tile the last dim {x.shape[-1]}")
    v = x.reshape(-1, block).copy()
    with np.errstate(over="ignore", invalid="ignore"):
        h = 1
        while h < block:
            v = v.reshape(-1, block // (2 * h), 2, h)
            a, b = v[:, :, 0, :].copy(), v[:, :, 1, :].copy()
            v[:, :, 0, :] = a + b                 # float32 + float32: one RNE rounding
            v[:, :, 1, :] = a - b
            h *= 2
        v = v.reshape(-1, block) * F32(block ** -0.5 if scale is None else scale)
    return round_to(v, dtype).reshape(x.shape)


def hadamard_f64(x, block: int):
    """The same transform as an fp64 matrix product with scipy's Sylvester Hadamard matrix (no rounding model)."""
    from scipy.linalg import hadamard as sylvester

    x = np.asarray(x, dtype=np.float64)
    hm = sylvester(block).astype(np.float64) / np.sqrt(block)
    return (x.reshape(-1, block) @ hm.T).reshape(x.shape)


__all__ = ["hadamard", "hadamard_f64", "round_to"]
