"""TensorQuantizer -- host-side mirror of
``modelopt/torch/quantization/nn/modules/tensor_quantizer.py`` (``TensorQuantizer`` :136,
``forward`` :1119-1221, ``_fake_quantize`` :890-949, ``_get_amax`` :736-751, ``collect`` :1397-1407,
static block reshape :975-1061, ``load_calib_amax`` :697-720, ``export_amax`` :1082-1117, input rotation :616-668).

Same attribute names and state (``_amax`` buffer in the input dtype, ``_pre_quant_scale``,
``_if_quant`` / ``_if_calib`` / ``_disabled``), same dispatch rules; every numeric step is a
fused sm_90a kernel (``model_optimizer_b200.ops``).  CPU tensors raise.
"""

from __future__ import annotations

import math

import torch
import torch.nn.functional as F
from torch import nn

from .. import calib, ops
from ..config import QuantizerAttributeConfig, RotateConfig
from . import shared_input as _shared
from .functional import normalized_hadamard_transform, rotate_block_size
from ..tensor_quant import dynamic_block_quant, fake_tensor_quant, scaled_e4m3, static_blockwise_fp4_fake_quant


_QT_BASE = None


def _qtensor_base():
    """qtensor.BaseQuantizedTensor, imported once (the qtensor package imports this module's siblings)."""
    global _QT_BASE
    if _QT_BASE is None:
        from ..qtensor import BaseQuantizedTensor

        _QT_BASE = BaseQuantizedTensor
    return _QT_BASE


def fp8_max_for_normalization(quantizer) -> float:
    """The FP8 maximum that normalizes static NVFP4 block scales (utils/numeric_utils.py:181-184): 256 for
    Four-Over-Six (``block_sizes["four_over_six"]`` truthy), else 448.  The fake quant, the real quant, the export
    and the drop-in all take it from here."""
    bs = getattr(quantizer, "block_sizes", None) or {}
    return 256.0 if bool(bs.get("four_over_six", False)) else 448.0


class TensorQuantizer(nn.Module):
    # input quantizers of sibling linears that are handed the very same tensor object (q/k/v, gate/up) do the collect /
    # fake quant once (nn/shared_input.py); bit-identical results
    share_identical_inputs = True

    def __init__(self, quant_attribute_cfg: QuantizerAttributeConfig | dict | None = None,
                 if_quant=True, if_calib=False, amax=None):
        super().__init__()
        cfg = quant_attribute_cfg
        if cfg is None:
            cfg = QuantizerAttributeConfig()
        elif isinstance(cfg, dict):
            cfg = QuantizerAttributeConfig(**cfg)
        self._if_quant = if_quant
        self._if_calib = if_calib
        self._dequantize = False
        self._state_gen = 0  # bumped on every state change; lets callers cache results safely
        self._calibrator = None
        self.set_from_attribute_config(cfg)
        if amax is not None:
            self.amax = amax

    # ---- configuration ---------------------------------------------------------------------------
    def set_from_attribute_config(self, cfg: QuantizerAttributeConfig | dict):
        """tensor_quantizer.py:228-259."""
        if isinstance(cfg, dict):
            cfg = QuantizerAttributeConfig(**cfg)
        self._state_gen = getattr(self, "_state_gen", 0) + 1
        self._num_bits = cfg.num_bits
        self._axis = cfg.axis
        self._block_sizes = dict(cfg.block_sizes) if cfg.block_sizes else None
        self._unsigned = cfg.unsigned
        self._narrow_range = cfg.narrow_range
        self._fake_quant = cfg.fake_quant
        self._pass_through_bwd = cfg.pass_through_bwd
        self._disabled = not cfg.enable
        self._dynamic = cfg.type == "dynamic"
        self._bias = dict(cfg.bias) if cfg.bias else None
        self._rotate = cfg.rotate
        self._bias_calibrator = None
        if hasattr(self, "_bias_value"):
            delattr(self, "_bias_value")
        c = cfg.calibrator
        if isinstance(c, str):
            if c == "max":
                c = calib.MaxCalibrator(self._num_bits, self._axis, self._unsigned)
            elif c == "histogram":
                c = calib.HistogramCalibrator(self._num_bits, self._axis, self._unsigned)
            else:
                raise ValueError(f"Unknown calibrator: {c}")
        elif isinstance(c, type):
            c = c(self._num_bits, self._axis, self._unsigned)
        self._calibrator = c
        if self.is_mx_format:  # tensor_quantizer.py:289-290
            self._pass_through_bwd = True
        for name in ("_block_reshape_size", "_original_shape", "_padding", "_slices"):
            if hasattr(self, name):
                delattr(self, name)

    # ---- properties (same names as the reference) ---------------------------------------------------
    @property
    def num_bits(self):
        return self._num_bits

    @property
    def axis(self):
        return self._axis

    @axis.setter
    def axis(self, value):
        self._axis = value
        if self._calibrator is not None:
            self._calibrator._axis = value

    @property
    def block_sizes(self):
        return self._block_sizes

    @property
    def fake_quant(self):
        return self._fake_quant

    @property
    def is_enabled(self):
        return not self._disabled

    @property
    def maxbound(self):
        """tensor_quantizer.py:401-409."""
        if self._num_bits == (4, 3):
            return 448.0
        if self._num_bits == (2, 1):
            return 6.0
        return (1 << (self._num_bits - 1 + int(self._unsigned))) - 1

    @property
    def is_static_block_quant(self):
        return (self._block_sizes is not None and self._block_sizes.get("type", "static") != "dynamic"
                and self._fake_quant)

    @property
    def is_mx_format(self):
        """tensor_quantizer.py:544-551: dynamic blocks with an E8M0 (power-of-two) scale."""
        bs = self._block_sizes
        return bool(bs) and bs.get("type") == "dynamic" and bs.get("scale_bits") == (8, 0)

    def is_mxfp(self, bits):
        """tensor_quantizer.py:583-604."""
        elem = {4: (2, 1), 6: (3, 2), 8: (4, 3)}.get(bits)
        if elem is None:
            raise NotImplementedError()
        return self.is_mx_format and self._num_bits == elem and self._block_sizes.get(-1) == 32

    @property
    def is_nvfp4_dynamic(self):
        bs = self._block_sizes
        return bool(bs) and bs.get("type") == "dynamic" and self._num_bits == (2, 1) and bs.get("scale_bits") == (4, 3)

    @property
    def is_nvfp4_static(self):
        bs = self._block_sizes
        return bool(bs) and bs.get("type", "static") == "static" and self._num_bits == (2, 1) \
            and bs.get("scale_bits") == (4, 3)

    @property
    def amax(self):
        if self.is_mx_format:  # tensor_quantizer.py:360: MX scales are recomputed per block on every call
            return None
        return getattr(self, "_amax", None)

    @amax.setter
    def amax(self, value):
        """tensor_quantizer.py:366-380: the buffer keeps its shape once registered."""
        if value is None:
            raise AssertionError("amax cannot be set to None.")
        self._state_gen += 1
        if not isinstance(value, torch.Tensor):
            value = torch.tensor(value)
        if not hasattr(self, "_amax"):
            self.register_buffer("_amax", value.clone().detach())
        else:
            if self._amax.shape != value.shape:
                raise RuntimeError("Changing shape when setting amax is not allowed.")
            self._amax.data.copy_(value.clone().detach().to(self._amax.device))

    def reset_amax(self):
        self._state_gen += 1
        if hasattr(self, "_amax"):
            delattr(self, "_amax")
        if self._calibrator is not None:
            self._calibrator.reset()
        self.reset_bias()

    # ---- affine bias (tensor_quantizer.py:389-503, 722-734, 775-786) -------------------------------------
    def reset_bias(self):
        if hasattr(self, "_bias_value"):
            delattr(self, "_bias_value")
        if getattr(self, "_bias_calibrator", None) is not None:
            self._bias_calibrator.reset()

    @property
    def bias(self):
        return getattr(self, "_bias", None)

    @property
    def bias_axis(self):
        return None if self._bias is None else tuple(k for k in self._bias if isinstance(k, int))

    @property
    def bias_method(self):
        return None if self._bias is None else self._bias.get("method", "mean")

    @property
    def bias_type(self):
        return None if self._bias is None else self._bias.get("type", "static")

    @property
    def bias_value(self):
        return getattr(self, "_bias_value", None)

    @bias_value.setter
    def bias_value(self, value):
        assert value is not None, "bias cannot be set to None."
        self._state_gen += 1
        if not hasattr(self, "_bias_value"):
            self.register_buffer("_bias_value", value.clone().detach())
        else:
            if self._bias_value.shape != value.shape:
                raise RuntimeError("Changing shape when setting bias is not allowed.")
            self._bias_value.data.copy_(value.clone().detach().to(self._bias_value.device))

    @property
    def bias_calibrator(self):
        if self._bias_calibrator is None and self._bias is not None:
            self._bias_calibrator = calib.BiasCalibrator(method=self.bias_method, axis=self.bias_axis)
        return self._bias_calibrator

    def load_calib_bias(self):
        b = self.bias_calibrator.compute_bias()
        if b is None:
            raise RuntimeError("Calibrator returned None. This usually happens when calibrator hasn't seen any tensor.")
        self.bias_value = b

    def _get_bias(self, inputs):
        if self.bias_calibrator is None:
            return None
        if self.bias_type == "static":
            return getattr(self, "_bias_value", None)
        if self.bias_type == "dynamic":
            return self.bias_calibrator.compute_dynamic_bias(inputs)
        raise ValueError(f"Unsupported bias type: {self.bias_type}")

    @property
    def pre_quant_scale(self):
        return getattr(self, "_pre_quant_scale", None)

    @pre_quant_scale.setter
    def pre_quant_scale(self, value):
        self._state_gen += 1
        if not isinstance(value, torch.Tensor):
            value = torch.tensor(value)
        if not hasattr(self, "_pre_quant_scale"):
            self.register_buffer("_pre_quant_scale", value.clone().detach())
        else:
            self._pre_quant_scale.data.copy_(value.clone().detach().to(self._pre_quant_scale.device))

    # ---- input rotation (tensor_quantizer.py:616-668) -------------------------------------------------
    @property
    def rotate_is_enabled(self):
        if isinstance(self._rotate, RotateConfig):
            return self._rotate.enable
        if isinstance(self._rotate, dict):  # a state dict of an older checkpoint
            return self._rotate.get("enable", False)
        return self._rotate

    @property
    def rotate_is_fp32(self):
        if isinstance(self._rotate, RotateConfig):
            return self._rotate.rotate_fp32 if self._rotate.enable else False
        if isinstance(self._rotate, dict) and self.rotate_is_enabled:
            return self._rotate.get("rotate_fp32", False)
        return False

    @property
    def rotate_block_size(self):
        if isinstance(self._rotate, RotateConfig):
            return self._rotate.block_size if self._rotate.enable else None
        if isinstance(self._rotate, dict) and self.rotate_is_enabled:
            return self._rotate.get("block_size", None)
        return None

    @property
    def rotate_back_is_enabled(self):
        if isinstance(self._rotate, RotateConfig):
            return self._rotate.enable and self._rotate.mode == "rotate_back"
        if isinstance(self._rotate, dict) and self.rotate_is_enabled:
            return self._rotate.get("mode", "rotate") == "rotate_back"
        return False

    def disable_rotate(self):
        """Disable rotation, keeping the type of the ``_rotate`` field (idempotent)."""
        self._state_gen += 1
        if isinstance(self._rotate, RotateConfig):
            self._rotate = self._rotate.model_copy(update={"enable": False})
        elif isinstance(self._rotate, dict):
            self._rotate = dict(self._rotate, enable=False)
        else:
            self._rotate = False

    def _rotate_inputs(self, inputs, amax_slot=None):
        if amax_slot is not None:  # the collect of a per-tensor max calibrator, folded into the transform
            return normalized_hadamard_transform(inputs, rotate_fp32=self.rotate_is_fp32,
                                                 block_size=self.rotate_block_size, amax_slot=amax_slot)
        return normalized_hadamard_transform(inputs, rotate_fp32=self.rotate_is_fp32, block_size=self.rotate_block_size)

    def _rotate_collect_slot(self, inputs):
        """The fp32 slot the transform can fold the calibration collect into (per-tensor ``MaxCalibrator``, no bias,
        no block reshape or axis conversion before the collect), or None."""
        cal = self._calibrator
        if not (self._if_calib and not self._dynamic and isinstance(cal, calib.MaxCalibrator) and cal._axis is None
                and not cal._track_amax and self._bias is None and inputs.is_cuda
                and (self._block_sizes is None or self.is_nvfp4_dynamic)):
            return None
        return cal.tensor_slot(inputs)

    def _fake_quant_rotated_nvfp4(self, inputs):
        """NVFP4 dynamic block fake quant of the rotated input (rotated back for ``rotate_back``) in one kernel when the
        quantizer has a calibrated per-tensor amax, is not calibrating and no autograd graph is needed; else None."""
        amax = getattr(self, "_amax", None)
        if not (self.is_nvfp4_dynamic and self._if_quant and self._fake_quant and not self._disabled
                and not (self._if_calib and not self._dynamic) and amax is not None and amax.numel() == 1
                and inputs.is_cuda and inputs.dim() > 0 and inputs.shape[-1] % 16 == 0
                and not (torch.is_grad_enabled() and inputs.requires_grad)):
            return None
        bs = rotate_block_size(inputs.shape[-1], self.rotate_block_size)
        return ops.fake_quant_nvfp4_rotated(inputs, bs, amax, self.rotate_back_is_enabled)

    # ---- mode switches (tensor_quantizer.py:640-695) ---------------------------------------------------
    def disable(self):
        self._disabled = True

    def enable(self):
        self._disabled = False

    def disable_calib(self):
        self._if_calib = False

    def enable_calib(self):
        if self._calibrator is None:
            raise ValueError("Calibrator was not created, cannot enable calibration.")
        self._if_calib = True

    def disable_quant(self):
        self._if_quant = False

    def enable_quant(self):
        self._if_quant = True

    # ---- calibration -------------------------------------------------------------------------------------
    def collect(self, inputs):
        """tensor_quantizer.py:1397-1407."""
        if self.bias_calibrator is not None and self.bias_type == "static":
            self.bias_calibrator.collect(inputs)
            inputs = inputs - self.bias_calibrator.compute_bias()
        self._calibrator.collect(inputs)

    def load_calib_amax(self, *args, **kwargs):
        """tensor_quantizer.py:697-720."""
        strict = kwargs.pop("strict", True)
        if self._calibrator is None:
            raise RuntimeError("Calibrator not created.")
        calib_amax = self._calibrator.compute_amax(*args, **kwargs)
        if calib_amax is None:
            msg = "Calibrator returned None. This usually happens when calibrator hasn't seen any tensor."
            if strict:
                raise RuntimeError(msg + " Passing 'strict=False' to `load_calib_amax()` will ignore the error.")
            calib_amax = torch.tensor(math.nan)
        if hasattr(self, "_amax") and self._amax.shape != calib_amax.shape:
            delattr(self, "_amax")
        cal = self._calibrator
        if getattr(cal, "_b200_shared", False):
            # a calibrator shared by sibling input quantizers (nn/shared_input.py): ONE amax buffer, aliased
            buf = getattr(cal, "_b200_amax_buf", None)
            if buf is not None and buf.shape == calib_amax.shape and buf.dtype == calib_amax.dtype:
                if hasattr(self, "_amax"):
                    delattr(self, "_amax")
                self.register_buffer("_amax", buf)
                self._state_gen += 1
                return
            self.amax = calib_amax
            cal._b200_amax_buf = self._amax
            return
        self.amax = calib_amax

    def export_amax(self):
        """tensor_quantizer.py:1082-1117."""
        if self._block_sizes is not None and self._block_sizes.get("type") == "dynamic":
            return self.amax
        if self.amax is None:
            return None
        amax = self.amax.clone()
        if hasattr(self, "_amax_shape_for_export"):
            amax = amax.reshape(self._amax_shape_for_export)
        amax[amax == 0] = self.maxbound
        amax = torch.nan_to_num(amax, nan=self.maxbound)
        amax = amax.clamp(min=torch.finfo(amax.dtype).tiny, max=torch.finfo(amax.dtype).max)
        if self._block_sizes is None:
            if self._axis is None:
                amax = amax.unsqueeze(0) if amax.dim() == 0 else amax
            elif isinstance(self._axis, int) or len(self._axis) == 1:
                amax = amax.squeeze()
        return amax

    def _get_amax(self, inputs):
        """tensor_quantizer.py:736-751: buffer, or dynamic |x| max when none is registered."""
        if hasattr(self, "_amax"):
            amax = self._amax
            return amax.to(inputs.device) if amax.device != inputs.device else amax
        axis = self._axis
        if isinstance(axis, (tuple, list)) and len(axis) > 1:
            # kept axes = all leading dims (per-token / per-row dynamic quantization): rows of the last dim
            nd = inputs.dim()
            if sorted(a % nd for a in axis) != list(range(nd - 1)):
                raise NotImplementedError(f"dynamic amax with axis={axis}")
            slots = torch.zeros(inputs.numel() // inputs.shape[-1], dtype=torch.float32, device=inputs.device)
            ops.amax_rows_(slots, inputs, inputs.shape[-1])
            return ops.amax_export(slots, inputs.dtype).reshape(*inputs.shape[:-1], 1)
        tmp = calib.MaxCalibrator(self._num_bits, axis, self._unsigned)
        tmp.collect(inputs)
        return ops.amax_export(tmp.slots, inputs.dtype).reshape(tmp._shape)

    def _block_sizes_to_axis(self, x):
        """tensor_quantizer.py:1063-1086: ``block_sizes`` whose integer keys all map to None mean
        per-channel / per-token quantization along the remaining axes."""
        bs = self._block_sizes
        if bs is None or not all(v is None for k, v in bs.items() if isinstance(k, int)):
            return
        assert self._axis is None, "Axis and block_sizes are both set."
        reduced = tuple(k if k >= 0 else k + x.dim() for k in bs if isinstance(k, int))
        self.axis = tuple(i for i in range(x.dim()) if i not in reduced) or None
        self._block_sizes = None

    # ---- static block quant reshape (tensor_quantizer.py:975-1061: last-axis and multi-axis blocks) ------
    def _setup_for_blockquant(self, inputs):
        """tensor_quantizer.py:975-1045: reshape sizes, kept axes, paddings and crop slices of static block
        quantization.  Blocks along the last axis only: flatten to [-1, block] (amax per row).  Otherwise every
        blocked dim d is split into [ceil(d / b), b] and the amax keeps the block-count dims (2-D 128 x 128 FP8
        blocks: [N, K] -> [N/128, 128, K/128, 128], amax [N/128, 1, K/128, 1])."""
        if hasattr(self, "_block_reshape_size"):
            return
        bs = self._block_sizes
        nd = inputs.dim()

        def params(ax):
            key = ax if ax in bs else ax - nd
            bsize = bs.get(key)
            padding, ax_slice = None, None
            if bsize is not None and inputs.shape[ax] % bsize != 0:
                padding = (bsize - inputs.shape[ax] % bsize, 0)
                ax_slice = slice(inputs.shape[ax])
            return bsize, padding, ax_slice

        # the reference's criterion (_get_block_quant_axes_and_sizes, :975-1006): ALL integer keys count, also the
        # None-valued ones ({-1: 128, -2: None} keeps the [N, K/128, 1] amax layout, not the flattened one)
        blocked = [k for k in bs if isinstance(k, int)]
        if len(blocked) == 1 and bs[blocked[0]] is not None and blocked[0] in (-1, nd - 1):
            bsize, padding, ax_slice = params(nd - 1)
            self._original_shape = inputs.shape
            if padding:
                self._padding = tuple(reversed(padding))
                self._slices = (*(slice(None),) * (nd - 1), ax_slice)
                self._original_shape = F.pad(inputs, self._padding, "constant", 0).shape
            self._block_reshape_size = torch.Size((-1, bsize))
            self._amax_shape_for_export = (*inputs.shape[:-1], -1)
            self.axis = (0,)
            return
        reshape, keep, paddings, slices = [], [], [], []
        for ax in range(nd):
            bsize, padding, ax_slice = params(ax)
            paddings.append(padding)
            slices.append(ax_slice)
            if bsize is not None:
                reshape += [math.ceil(inputs.shape[ax] / bsize), bsize]
                keep += [True, False]
            else:
                reshape.append(inputs.shape[ax])
                keep.append(True)
        self._original_shape = inputs.shape
        if any(p is not None for p in paddings):
            flat = []
            for p in paddings:
                if not (flat or p):
                    continue
                flat.extend(p or (0, 0))
            self._padding = tuple(reversed(flat))
            self._original_shape = F.pad(inputs, self._padding, "constant", 0).shape
        if any(sl is not None for sl in slices):
            self._slices = tuple(sl or slice(None) for sl in slices)
        self._block_reshape_size = torch.Size(reshape)
        self.axis = tuple(i for i, k in enumerate(keep) if k)

    def _process_for_blockquant(self, inputs):
        if hasattr(self, "_padding"):
            inputs = F.pad(inputs, self._padding, "constant", 0)
        if inputs.shape != self._original_shape:
            raise ValueError(f"Input shape has changed from {self._original_shape} to {inputs.shape}."
                             " Block-quantization requires a fixed input shape.")
        return inputs.reshape(self._block_reshape_size)

    def _reset_to_original_shape(self, outputs):
        outputs = outputs.reshape(self._original_shape)
        if hasattr(self, "_slices"):
            outputs = outputs[self._slices]
        return outputs

    # ---- fake quant dispatch (tensor_quantizer.py:890-949) ------------------------------------------------
    def _fake_quantize(self, inputs):
        bs = self._block_sizes
        if bs is not None and bs.get("type", "static") == "dynamic":
            block_size = bs.get(-1) or bs.get(inputs.dim() - 1)
            if block_size is None:
                raise ValueError("block size for dynamic quantization not found.")
            amax = None if self.is_mx_format else self._get_amax(inputs)  # tensor_quantizer.py:898-900
            return dynamic_block_quant(inputs, block_size, amax, self._get_bias(inputs), self._num_bits,
                                       bs.get("scale_bits"), None, "dynamic", self._pass_through_bwd)
        if self.is_nvfp4_static:  # StaticBlockScaleQuantizer._fake_quantize (:1708-1731)
            gamax = getattr(self, "_global_amax", None)
            return static_blockwise_fp4_fake_quant(inputs, self._get_amax(inputs).float(), gamax, True,
                                                   fp8_max_for_normalization(self), None, self._pass_through_bwd)
        amax = self._get_amax(inputs)
        if isinstance(self._num_bits, tuple):
            e, m = self._num_bits
            return scaled_e4m3(inputs, amax, self._get_bias(inputs), e, m, None, self._pass_through_bwd)
        return fake_tensor_quant(inputs, amax, self._get_bias(inputs), self._num_bits, self._unsigned, self._narrow_range, None,
                                 self._pass_through_bwd, bs.get(-1) if bs else None,
                                 self._axis[0] if isinstance(self._axis, tuple) else self._axis)

    def _real_quantize(self, inputs):
        """tensor_quantizer.py:796-888 (FP8 / INT4 / NVFP4 packs)."""
        from ..qtensor import FP8QTensor, INT4QTensor, MXFP4QTensor, MXFP8QTensor, NF4QTensor, NVFP4QTensor

        bs = self._block_sizes
        if self.is_mx_format:  # checked first: MXFP8 shares num_bits (4, 3) with FP8 (:800-823)
            if self._num_bits == (2, 1):
                q, sc = MXFP4QTensor.quantize(inputs, bs[-1])
            elif self._num_bits == (4, 3):
                assert bs[-1] == MXFP8QTensor.BLOCK_SIZE, (
                    f"MXFP8 requires block size {MXFP8QTensor.BLOCK_SIZE}, got {bs[-1]}")
                q, sc = MXFP8QTensor.quantize(inputs)
            else:
                raise ValueError(f"Unsupported MX format: num_bits={self._num_bits}. "
                                 "Expected (2, 1) for MXFP4 or (4, 3) for MXFP8.")
            self._scale = sc
        elif self._num_bits == (2, 1):
            if bs and bs.get("four_over_six", False):   # tensor_quantizer.py:861-866
                raise NotImplementedError(
                    "NVFP4 Four-Over-Six (4/6) is not supported via mtq.compress: the per-block M=4/M=6 choice baked "
                    "into the quantizer amax by MSE calibration is not preserved by real quantization. Use "
                    "mtq.quantize + export for 4/6 instead.")
            # second-level scale from the calibration when there is one (tensor_quantizer.py:867-875,
            # NVFP4QTensor.get_weights_scaling_factor_2_from_quantizer): the static global amax, else _amax
            wsf2 = None
            if self.amax is not None:
                g = getattr(self, "_global_amax", None) if self.is_static_block_quant else None
                wsf2 = (g if g is not None else self._amax).float() / (6.0 * fp8_max_for_normalization(self))
            q, sf, sf2 = NVFP4QTensor.quantize(inputs, bs[-1], weights_scaling_factor_2=wsf2)
            self._scale, self._double_scale = sf, sf2
        elif bs and bs.get("scale_bits", 0) == 8 and bs.get("scale_block_sizes"):
            # NF4 with double quantization of the scales (tensor_quantizer.py:841-856)
            sbs = bs["scale_block_sizes"][-1]
            q, scales = NF4QTensor.quantize(inputs, bs[-1], sbs)
            self._scale, self._double_scale, self._scale_zeros = NF4QTensor.double_quantization(
                scales, sbs, bs["scale_bits"])
        elif self._num_bits == 4 and bs:
            q, sc = INT4QTensor.quantize(inputs, bs[-1])
            self._scale = sc
        elif self._num_bits == (4, 3):
            # per-tensor / per-channel scales from the calibrated amax (:824-835); 2-D blocks recompute theirs from
            # the weight, which gives the reference's packs and scales bit for bit after max calibration
            use_amax = self.amax is not None and not bs
            q, sc = FP8QTensor.quantize(inputs, axis=self._axis, block_sizes=bs or None,
                                        scales=self.amax / 448.0 if use_amax else None)
            self._scale = sc
        else:
            raise NotImplementedError(f"real quantization for num_bits={self._num_bits}")
        self._dequantize = True
        return q

    def dequantize(self, inputs):
        """tensor_quantizer.py:292-302: de-quantize a real-quantized tensor with this quantizer's scales."""
        from ..qtensor import BaseQuantizedTensor

        assert isinstance(inputs, BaseQuantizedTensor), "Expected input as real quantized tensors."
        return inputs.dequantize(scale=self._scale, block_sizes=self.block_sizes,
                                 double_scale=getattr(self, "_double_scale", None),
                                 scale_zeros=getattr(self, "_scale_zeros", None))

    # ---- forward (tensor_quantizer.py:1119-1221) -----------------------------------------------------------
    def forward(self, inputs):
        if isinstance(inputs, _qtensor_base()):           # tensor_quantizer.py:1135-1137
            assert getattr(self, "_dequantize", False), "No dequantization stats in the tensor quantizer."
            return self.dequantize(inputs)
        if inputs.numel() == 0:
            return inputs
        pqs = self.pre_quant_scale
        if pqs is not None:
            # SmoothQuant / AWQ pre-scale (tensor_quantizer.py:1143-1144): fused column-scale kernel when no
            # autograd graph is needed, plain broadcasting multiply otherwise
            if (inputs.is_cuda and not torch.is_grad_enabled() and pqs.dtype == inputs.dtype
                    and pqs.numel() == inputs.shape[-1] and inputs.dtype in (torch.bfloat16, torch.float16, torch.float32)):
                inputs = ops.scale_cols(inputs, pqs.reshape(-1))
            else:
                inputs = inputs * pqs
        rotate, rotate_back = self.rotate_is_enabled, self.rotate_back_is_enabled
        if rotate_back and self._if_quant and not self._fake_quant:   # tensor_quantizer.py:1146-1147, before rotating
            raise ValueError("rotate_back mode is only supported with fake_quant=True.")
        if self._disabled or not (self._if_quant or (self._if_calib and not self._dynamic)):
            # nothing to do in this phase (e.g. a weight quantizer held during the activation calibration loop): the
            # reference reshapes into blocks and back for the same values.  It still rotates (and rotates back)
            if rotate:
                inputs = self._rotate_inputs(inputs)
                if rotate_back:
                    inputs = self._rotate_inputs(inputs)
            return inputs
        collected = False
        if rotate:
            fused = self._fake_quant_rotated_nvfp4(inputs)
            if fused is not None:
                return fused
            slot = self._rotate_collect_slot(inputs)
            inputs = self._rotate_inputs(inputs, slot)
            collected = slot is not None
        if self._block_sizes is not None and self._fake_quant:
            self._block_sizes_to_axis(inputs)
        if self.is_static_block_quant:
            self._setup_for_blockquant(inputs)
            inputs = self._process_for_blockquant(inputs)
        outputs = inputs
        share = _shared.eligible(self, inputs)
        if self._if_calib and not self._dynamic:
            if self._calibrator is None:
                raise RuntimeError("Calibrator was not created.")
            if not collected and (not share or _shared.collect_once(self, inputs)):
                self.collect(inputs)
        if self._if_quant:
            if share and self._fake_quant:
                hit = _shared.cached_output(self, inputs)
                if hit is not None:
                    return self._rotate_inputs(hit) if rotate_back else hit
            src = inputs
            if not inputs.is_contiguous():
                inputs = inputs.contiguous()
            if self._fake_quant:
                outputs = self._fake_quantize(inputs)
                if share:
                    _shared.store_output(self, src, outputs)
            elif not getattr(self, "_dequantize", False):
                outputs = self._real_quantize(inputs)
            else:                                              # tensor_quantizer.py:1207-1211
                raise ValueError("self._dequantize is True and self.fake_quant is False. "
                                 "This case should have been handled.")
        if self.is_static_block_quant and isinstance(outputs, torch.Tensor):
            outputs = self._reset_to_original_shape(outputs)
        if rotate_back and isinstance(outputs, torch.Tensor):
            outputs = self._rotate_inputs(outputs)
        return outputs

    def _rotate_repr(self):
        """tensor_quantizer.py:1250-1254."""
        s = " rotated" if self.rotate_is_enabled else ""
        s += " (rotate_back)" if self.rotate_back_is_enabled else ""
        s += " (fp32)" if self.rotate_is_fp32 else ""
        if self.rotate_block_size is not None:
            s += f" (block={self.rotate_block_size})"
        return s

    def extra_repr(self):
        if self._disabled:
            return "disabled" + self._rotate_repr()
        a = self.amax
        amax = "dynamic" if a is None else (f"{a.item():.4e}" if a.numel() == 1 else f"[{a.min().item():.2e}, {a.max().item():.2e}]({a.numel()})")
        return (f"{self._num_bits} bit fake={self._fake_quant} axis={self._axis} block_sizes={self._block_sizes} "
                f"amax={amax} calib={self._if_calib} quant={self._if_quant}" + self._rotate_repr())


__all__ = ["TensorQuantizer", "fp8_max_for_normalization"]
