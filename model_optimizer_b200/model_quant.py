"""User API -- mirror of ``modelopt/torch/quantization/model_quant.py`` (``quantize`` :147,
``calibrate`` :64) and ``conversion.py`` (``replace_quant_module`` :214, ``set_quantizer_by_cfg`` :245).
The mode/state framework (``modelopt.torch.opt``) is out of scope: ``quantize`` converts modules in
place, applies the ordered ``quant_cfg`` entries by fnmatch, then runs the calibration algorithm."""

from __future__ import annotations

import fnmatch
from typing import Callable

from torch import nn

from . import model_calib
from .config import QuantizerAttributeConfig
from .nn import QuantModuleRegistry, TensorQuantizer


def replace_quant_module(model: nn.Module) -> nn.Module:
    for _, module in list(model.named_modules()):
        if QuantModuleRegistry.get(type(module)) is not None:
            QuantModuleRegistry.convert(module)
    return model


_PARENT_CLASSES = {"nn.Embedding": nn.Embedding, "nn.Linear": nn.Linear, "nn.BatchNorm1d": nn.BatchNorm1d,
                   "nn.BatchNorm2d": nn.BatchNorm2d, "nn.BatchNorm3d": nn.BatchNorm3d, "nn.LeakyReLU": nn.LeakyReLU}


def set_quantizer_by_cfg(model: nn.Module, quant_cfg: list[dict]):
    """Apply ordered ``{"quantizer_name": pattern, "cfg": ... | "enable": ...}`` entries
    (conversion.py:245-330); later entries override earlier ones."""
    parents = {}
    for pname, parent in model.named_modules():
        for cname, child in parent.named_children():
            parents[f"{pname}.{cname}" if pname else cname] = parent
    for entry in quant_cfg:
        pattern = entry["quantizer_name"]
        pcls = entry.get("parent_class")
        for name, module in model.named_modules():
            if not isinstance(module, TensorQuantizer):
                continue
            if not fnmatch.fnmatch(name, pattern):
                continue
            if pcls is not None:
                want = _PARENT_CLASSES.get(pcls)
                if want is None or not isinstance(parents.get(name), want):
                    continue
            if "cfg" in entry and entry["cfg"] is not None:
                cfg = dict(entry["cfg"])
                cfg.setdefault("enable", entry.get("enable", True))
                module.set_from_attribute_config(QuantizerAttributeConfig(**cfg))
            elif "enable" in entry:
                module.enable() if entry["enable"] else module.disable()


def calibrate(model: nn.Module, algorithm="max", forward_loop: Callable | None = None):
    """model_quant.py:64-145: dispatch on the algorithm name."""
    if algorithm is None:
        return model
    kwargs = {}
    if isinstance(algorithm, dict):
        kwargs = {k: v for k, v in algorithm.items() if k != "method"}
        algorithm = algorithm["method"]
    fn = {
        "max": model_calib.max_calibrate,
        "smoothquant": model_calib.smoothquant,
        "awq_lite": model_calib.awq_lite,
        "awq_clip": model_calib.awq_clip,
        "mse": model_calib.mse_calibrate,
        "local_hessian": model_calib.local_hessian_calibrate,
        "gptq": model_calib.gptq,
        "nvfp4_act_headroom": model_calib.nvfp4_act_headroom_calibrate,
    }.get(algorithm)
    if fn is None:
        raise ValueError(f"Unsupported calibration algorithm: {algorithm}")
    fn(model, forward_loop, **kwargs)
    return model


def quantize(model: nn.Module, config: dict, forward_loop: Callable | None = None) -> nn.Module:
    """``mtq.quantize`` (model_quant.py:147-270)."""
    replace_quant_module(model)
    set_quantizer_by_cfg(model, config["quant_cfg"])
    return calibrate(model, config.get("algorithm", "max"), forward_loop)


def print_quant_summary(model: nn.Module):
    n = 0
    for name, m in model.named_modules():
        if isinstance(m, TensorQuantizer):
            print(f"{name:80} {m}")
            n += 1
    print(f"{n} TensorQuantizers found in model")


__all__ = ["quantize", "calibrate", "replace_quant_module", "set_quantizer_by_cfg", "print_quant_summary"]
