"""Quantizer attribute config and preset PTQ configs.

Mirrors the part of ``modelopt/torch/quantization/config.py`` the hot path reads
(``QuantizerAttributeConfig`` :322-709 -- ``num_bits, axis, block_sizes, fake_quant, unsigned,
narrow_range, calibrator, enable, rotate``) and the preset dictionaries (:1681-1778), which are ordered
lists of ``{"quantizer_name": fnmatch pattern, "cfg": {...} | "enable": bool}`` entries plus an
``"algorithm"``.
"""

from __future__ import annotations

import copy
import dataclasses
from dataclasses import dataclass, field
from typing import Any


@dataclass
class RotateConfig:
    """quantization/config.py:282-319: normalized Hadamard rotation of the quantizer input (RHT / QuaRot / SpinQuant).
    ``mode="rotate_back"`` applies the transform again after fake quantization; ``block_size`` None rotates the whole
    last dim (or its largest power-of-2 divisor, nn/functional.py)."""

    enable: bool = False
    mode: str = "rotate"
    rotate_fp32: bool = False
    block_size: int | None = None

    def __post_init__(self):
        if self.mode not in ("rotate", "rotate_back"):
            raise ValueError(f"rotate mode must be 'rotate' or 'rotate_back', got {self.mode!r}")
        v = self.block_size
        if v is not None and (isinstance(v, bool) or not isinstance(v, int) or v <= 0):
            raise ValueError(f"block_size must be a positive int, got {v!r}")

    def model_copy(self, update=None):
        return dataclasses.replace(self, **(update or {}))


# the non-integer keys block_sizes accepts (config.py:548,564); "four_over_six": static NVFP4 weights whose block
# scales are normalized by 256 instead of 448 (Four-Over-Six, utils/numeric_utils.py:181-184)
BLOCK_SIZES_STR_KEYS = ("type", "scale_bits", "scale_block_sizes", "four_over_six")


@dataclass
class QuantizerAttributeConfig:
    """quantization/config.py:322-709 (fields on the PTQ hot path only)."""

    num_bits: int | tuple[int, int] = 8
    axis: int | tuple[int, ...] | None = None
    block_sizes: dict | None = None
    unsigned: bool = False
    narrow_range: bool = False          # config default (config.py:459-463)
    fake_quant: bool = True
    calibrator: str | Any = "max"
    enable: bool = True
    pass_through_bwd: bool = True
    type: str = "static"                 # "dynamic": amax is recomputed on every call (config.py:560-578)
    # affine bias (config.py:523-585): int keys = dims reduced by the bias statistic, "type" static | dynamic,
    # "method" mean | max_min
    bias: dict | None = None
    effective_bits: float | None = None  # informational (NVFP4 presets carry it)
    trt_high_precision_dtype: str = "Float"
    # input rotation (config.py:616-625): a bool is RotateConfig(enable=...), a dict the RotateConfig fields
    rotate: bool | dict | RotateConfig = False

    def __post_init__(self):
        if isinstance(self.num_bits, list):
            self.num_bits = tuple(self.num_bits)
        if self.block_sizes is not None:
            bs = dict(self.block_sizes)
            if isinstance(bs.get("scale_bits"), list):
                bs["scale_bits"] = tuple(bs["scale_bits"])
            self.block_sizes = bs
            if self.axis is not None:
                raise ValueError("axis and block_sizes are mutually exclusive")
            for k, v in bs.items():                      # config.py:555-566
                if isinstance(k, str):
                    if k not in BLOCK_SIZES_STR_KEYS:
                        raise ValueError(f"unknown block_sizes key {k!r}, expected one of {BLOCK_SIZES_STR_KEYS}")
                elif not (isinstance(k, int) and (v is None or isinstance(v, int))):
                    raise ValueError(f"block_sizes entry {k!r}: {v!r} must map an int axis to an int or None")
        if self.bias is not None:
            if self.bias.get("type", "static") not in ("static", "dynamic"):
                raise ValueError(f"Invalid bias type: {self.bias['type']}, expected 'static' or 'dynamic'")
            if self.bias.get("method", "mean") not in ("mean", "max_min"):
                raise ValueError(f"Invalid bias method: {self.bias['method']}, expected 'mean' or 'max_min'")
            assert any(isinstance(k, int) for k in self.bias), "The axis for bias computation is not specified."
        if self.type not in ("static", "dynamic"):
            raise ValueError(f"type must be 'static' or 'dynamic', got {self.type}")
        if isinstance(self.rotate, dict):
            self.rotate = RotateConfig(**self.rotate)
        elif not isinstance(self.rotate, (bool, RotateConfig)):
            raise ValueError(f"rotate must be a bool, a dict or a RotateConfig, got {self.rotate!r}")


@dataclass
class GPTQCalibConfig:
    """quantization/config.py:1204-1250: GPTQ (second-order blockwise weight update).  ``perc_damp`` in (0, 1] is the
    fraction of the mean Hessian diagonal added as damping; ``block_size`` columns per GPTQ block; ``fused`` is
    accepted for parity (the engine's kernel implements the unfused semantics for every format it covers).
    ``layerwise``: a bool or ``{"enable": ...}``; layer-by-layer calibration is not part of the engine's own API, so
    ``enable: true`` is refused at calibration time (the drop-in into the reference provides it).  ``None`` for
    ``perc_damp`` / ``block_size`` is accepted like the reference's config and means the default."""

    method: str = "gptq"
    perc_damp: float | None = 0.01
    block_size: int | None = 128
    fused: bool = False
    layerwise: bool | dict | None = None

    def __post_init__(self):
        if self.method != "gptq":
            raise ValueError(f"method must be 'gptq', got {self.method!r}")
        if self.perc_damp is None:
            self.perc_damp = 0.01
        if self.block_size is None:
            self.block_size = 128
        p = self.perc_damp
        if isinstance(p, bool) or not isinstance(p, (int, float)) or not (0.0 < p <= 1.0):
            raise ValueError(f"perc_damp must be in (0, 1], got {p!r}")
        b = self.block_size
        if isinstance(b, bool) or not isinstance(b, int) or b <= 0:
            raise ValueError(f"block_size must be a positive int, got {b!r}")
        if not isinstance(self.fused, bool):
            raise ValueError(f"fused must be a bool, got {self.fused!r}")
        lw = self.layerwise
        if lw is not None and not isinstance(lw, (bool, dict)):
            raise ValueError(f"layerwise must be a bool or a dict, got {lw!r}")

    @property
    def layerwise_enabled(self) -> bool:
        lw = self.layerwise
        return bool(lw.get("enable", False)) if isinstance(lw, dict) else bool(lw)


# NVFP4ActHeadroomCalibrator: rho must stay below the FP8-E4M3 normal dynamic range, 448 / 2^-6
FP8_NORMAL_DYNAMIC_RANGE = 448.0 / 2.0**-6
_WEIGHT_SCALE_METHODS = ("max", "mse", "local_hessian")


@dataclass
class NVFP4ActHeadroomCalibConfig:
    """quantization/config.py:1257-1330: the per-tensor global scale of every NVFP4 input quantizer from the
    distribution of its per-block amaxes, ``max(rho * P_anchor, P_upper)``, which leaves headroom above the calibrated
    range.  ``weight_scale_algorithm`` calibrates the weights (and runs the max pass that collects the histograms):
    ``None`` means ``{"method": "max"}``; otherwise a dict whose ``method`` is ``max``, ``mse`` or ``local_hessian``, plus
    that algorithm's own options."""

    method: str = "nvfp4_act_headroom"
    anchor_percentile: float = 1.0
    upper_percentile: float = 99.99
    rho: float = 16384.0
    weight_scale_algorithm: dict | None = None

    def __post_init__(self):
        if self.method != "nvfp4_act_headroom":
            raise ValueError(f"method must be 'nvfp4_act_headroom', got {self.method!r}")
        for name in ("anchor_percentile", "upper_percentile"):
            v = getattr(self, name)
            if isinstance(v, bool) or not isinstance(v, (int, float)) or not (0.0 < v <= 100.0):
                raise ValueError(f"{name} must be in (0, 100], got {v!r}")
        r = self.rho
        if isinstance(r, bool) or not isinstance(r, (int, float)) or not (0.0 < r < FP8_NORMAL_DYNAMIC_RANGE):
            raise ValueError(f"rho must be in (0, {FP8_NORMAL_DYNAMIC_RANGE:g}), got {r!r}")
        w = self.weight_scale_algorithm
        if w is None:
            self.weight_scale_algorithm = {"method": "max"}
        elif not isinstance(w, dict) or w.get("method") not in _WEIGHT_SCALE_METHODS:
            raise ValueError(f"weight_scale_algorithm must be None or a dict whose method is one of "
                             f"{_WEIGHT_SCALE_METHODS}, got {w!r}")


_DEFAULT_DISABLED = [
    "*block_sparse_moe.gate*", "*linear_attn.conv1d*", "*linear_attn.in_proj_a*", "*linear_attn.in_proj_b*",
    "*lm_head*", "*mixer.conv1d*", "*mlp.gate.*", "*mlp.shared_expert_gate.*", "*output_layer*", "*proj_out.*",
    "*router*", "mtp.*", "output.*", "*embed_vision*", "*vision_tower*", "*visual*", "*vision_model*",
    "*multi_modal_projector*",
]
_DISABLED_PARENTS = ["nn.BatchNorm1d", "nn.BatchNorm2d", "nn.BatchNorm3d", "nn.LeakyReLU", "nn.Embedding"]


def _preset_entries(entries, algorithm):
    """Same shape as modelopt_recipes/configs/ptq/presets/model/*.yaml after loading: disable-all, the
    (pattern, cfg) entries in order, the default disabled quantizers."""
    q: list[dict] = [{"quantizer_name": "*", "enable": False}]
    for pattern, cfg in entries:
        q.append({"quantizer_name": pattern, **({"cfg": copy.deepcopy(cfg)} if cfg else {"enable": False})})
    q += [{"quantizer_name": p, "enable": False} for p in _DEFAULT_DISABLED]
    q += [{"quantizer_name": "*", "parent_class": p, "enable": False} for p in _DISABLED_PARENTS]
    return {"quant_cfg": q, "algorithm": algorithm}


def _preset(weight_cfg, input_cfg, algorithm):
    return _preset_entries([("*weight_quantizer", weight_cfg), ("*input_quantizer", input_cfg)], algorithm)


def _wi(patterns, weight_cfg, input_cfg):
    """weight + input entries for every module pattern (the *_ONLY presets)."""
    out = []
    for p in patterns:
        out.append((p + "weight_quantizer", weight_cfg))
        if input_cfg is not None:
            out.append((p + "input_quantizer", input_cfg))
    return out


_NVFP4 = {"num_bits": (2, 1), "effective_bits": 4.5,
          "block_sizes": {-1: 16, "type": "dynamic", "scale_bits": (4, 3)}}
_NVFP4_STATIC = {"num_bits": (2, 1), "block_sizes": {-1: 16, "type": "static", "scale_bits": (4, 3)}}
_NVFP4_B32 = {"num_bits": (2, 1), "block_sizes": {-1: 32, "type": "dynamic", "scale_bits": (4, 3)}}
_INT4_BLOCK = {"num_bits": 4, "block_sizes": {-1: 128, "type": "static"}}
_FP8 = {"num_bits": (4, 3), "axis": None}


def _mx(num_bits):
    return {"num_bits": num_bits, "block_sizes": {-1: 32, "type": "dynamic", "scale_bits": (8, 0)}}


INT8_DEFAULT_CFG = _preset({"num_bits": 8, "axis": 0}, {"num_bits": 8, "axis": None}, "max")
INT8_SMOOTHQUANT_CFG = _preset({"num_bits": 8, "axis": 0}, {"num_bits": 8, "axis": None}, "smoothquant")
INT8_WEIGHT_ONLY_CFG = _preset({"num_bits": 8, "axis": 0}, None, "max")
FP8_DEFAULT_CFG = _preset(_FP8, _FP8, "max")
FP8_PER_CHANNEL_PER_TOKEN_CFG = _preset(
    {"num_bits": (4, 3), "axis": 0},
    {"num_bits": (4, 3), "type": "dynamic", "block_sizes": {-1: None}, "axis": None}, "max")
FP8_2D_BLOCKWISE_WEIGHT_ONLY_CFG = _preset(
    {"num_bits": (4, 3), "axis": None, "block_sizes": {-1: 128, -2: 128}}, None, "max")
NVFP4_DEFAULT_CFG = _preset(_NVFP4, _NVFP4, "max")
NVFP4_W4A4_WEIGHT_MSE_FP8_SWEEP_CFG = _preset(_NVFP4_STATIC, _NVFP4, {"method": "mse", "fp8_scale_sweep": True})
NVFP4_W4A4_WEIGHT_LOCAL_HESSIAN_CFG = _preset(_NVFP4_STATIC, _NVFP4, {"method": "local_hessian", "fp8_scale_sweep": True})
# Four-Over-Six (modelopt_recipes/configs/ptq/presets/model/nvfp4_four_over_six.yaml): static NVFP4 weights with
# block scales normalized by 256; MSE over the multipliers {1.0, 1.5} picks, per 16-element block, the scale that
# maps the block maximum to 6 or the one that maps it to 4
NVFP4_FOUR_OVER_SIX_CFG = _preset({**_NVFP4_STATIC, "block_sizes": {**_NVFP4_STATIC["block_sizes"], "four_over_six": True}},
                                  _NVFP4, {"method": "mse", "fp8_scale_sweep": False, "start_multiplier": 1.0,
                                           "stop_multiplier": 1.5, "step_size": 0.5})
NVFP4_AWQ_LITE_CFG = _preset(_NVFP4, _NVFP4, "awq_lite")
NVFP4_AWQ_CLIP_CFG = _preset(_NVFP4, _NVFP4, {"method": "awq_clip"})
W4A16_NVFP4_CFG = _preset_entries([("*weight_quantizer", _NVFP4)], "max")
W4A8_NVFP4_FP8_CFG = _preset(_NVFP4_B32, _FP8, "max")
_MOE = ["*block_sparse_moe*", "*.experts.*"]
_MLP = ["*mlp*", "*.mixer.up_proj.", "*.mixer.down_proj.", *_MOE]
NVFP4_EXPERTS_ONLY_CFG = _preset_entries(_wi(_MOE, _NVFP4, _NVFP4), "max")
NVFP4_MLP_ONLY_CFG = _preset_entries(_wi(_MLP, _NVFP4, _NVFP4), "max")
NVFP4_OMLP_ONLY_CFG = _preset_entries(_wi(["*o_proj*", *_MLP[:-1]], _NVFP4, _NVFP4), "max")
NVFP4_MLP_WEIGHT_ONLY_CFG = _preset_entries(_wi(["*mlp*", "*block_sparse_moe*"], _NVFP4_B32, None), "max")
INT4_BLOCKWISE_WEIGHT_ONLY_CFG = _preset(_INT4_BLOCK, None, "max")
INT4_AWQ_CFG = _preset(_INT4_BLOCK, None, {"method": "awq_lite", "alpha_step": 0.1})
# MX formats (block 32, E8M0 scales): calibration-free, "algorithm" is None
MXFP8_DEFAULT_CFG = _preset(_mx((4, 3)), _mx((4, 3)), None)
MXFP6_DEFAULT_CFG = _preset(_mx((3, 2)), _mx((3, 2)), None)
MXFP4_DEFAULT_CFG = _preset(_mx((2, 1)), _mx((2, 1)), None)
MXINT8_DEFAULT_CFG = _preset(_mx(8), _mx(8), None)
W4A8_MXFP4_FP8_CFG = _preset(_mx((2, 1)), _FP8, None)
MXFP4_MLP_WEIGHT_ONLY_CFG = _preset_entries(_wi(["*mlp*", "*block_sparse_moe*"], _mx((2, 1)), None), None)

PRESETS = {k: v for k, v in globals().items() if k.endswith("_CFG")}


def get_preset(name: str) -> dict:
    return copy.deepcopy(PRESETS[name])


__all__ = ["QuantizerAttributeConfig", "RotateConfig", "GPTQCalibConfig", "PRESETS", "get_preset", *PRESETS.keys()]
