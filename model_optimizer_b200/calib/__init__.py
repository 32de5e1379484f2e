"""Calibrators -- the b200quant counterpart of ``modelopt/torch/quantization/calib``.

``collect`` is one fused kernel per batch (|x| max / histogram folded into device-resident fp32
state); nothing synchronises with the host until ``compute_amax``."""

from .bias import BiasCalibrator
from .calibrator import _Calibrator
from .histogram import HistogramCalibrator
from .max import MaxCalibrator
from .mse import MseCalibrator
from .nvfp4_act_headroom import NVFP4ActHeadroomCalibrator

__all__ = ["_Calibrator", "MaxCalibrator", "MseCalibrator", "HistogramCalibrator", "NVFP4ActHeadroomCalibrator", "BiasCalibrator"]
