"""model_optimizer_b200 -- a H100-native (sm_90a) PTQ calibration / fake-quant / quant-and-pack
engine behind the ``modelopt.torch.quantization`` API surface.

Layout: ``csrc/`` hand-written CUDA + the C-ABI (``include/b200quant.h``), ``_lib``/``ops`` the
binding, and the host-side mirror of the reference interface (``tensor_quant``, ``calib``, ``nn``,
``qtensor``, ``model_calib``, ``model_quant``).  There is no CPU fallback anywhere in this package.
"""

__version__ = "0.1.0"
