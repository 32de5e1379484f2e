"""Build the REFERENCE's own CUDA extensions for sm_90a from the sources where they lie
(/root/reference/modelopt/torch/kernels/quantization/gemm) into oracle/_ref/ -- nothing is copied into
the repo.  Same source lists and extra flags as the reference's loader (quantization/extensions.py:28-72):

    modelopt_cuda_ext      tensor_quant.cpp + tensor_quant_gpu.cu
    modelopt_cuda_ext_fp8  tensor_quant_gpu_fp8.cu
    modelopt_cuda_ext_mx   tensor_quant_mx.cu            (--use_fast_math)

The .so files travel to the GPU box with the snapshot (oracle/_ref is git-ignored, not gpurun-ignored) where
tests/test_gpu_vs_reference_ext.py runs the reference kernels side by side with this engine's.
Test infrastructure only.  Usage: python oracle/build_ref_ext.py   (cross-compiles without a GPU, ~5 min once)
"""

from __future__ import annotations

import os
import shutil
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = "/root/reference/modelopt/torch/kernels/quantization/gemm"
OUT = os.path.join(HERE, "_ref")
EXTS = {
    "modelopt_cuda_ext": (["tensor_quant.cpp", "tensor_quant_gpu.cu"], []),
    "modelopt_cuda_ext_fp8": (["tensor_quant_gpu_fp8.cu"], []),
    "modelopt_cuda_ext_mx": (["tensor_quant_mx.cu"], ["--use_fast_math"]),
}


def build_one(name: str) -> str:
    from torch.utils import cpp_extension

    srcs, flags = EXTS[name]
    dst = os.path.join(OUT, name + ".so")
    srcs = [os.path.join(SRC, s) for s in srcs]
    # this recipe (its gencode flags) is part of the key: a change of target architecture rebuilds
    if os.path.exists(dst) and all(os.path.getmtime(dst) >= os.path.getmtime(s) for s in srcs + [__file__]):
        return dst
    bdir = os.path.join(OUT, "build_" + name)
    os.makedirs(bdir, exist_ok=True)
    cpp_extension.load(name=name, sources=srcs, build_directory=bdir, verbose=False, is_python_module=False,
                       extra_cuda_cflags=["-gencode", "arch=compute_90a,code=sm_90a", *flags])
    shutil.copyfile(os.path.join(bdir, name + ".so"), dst)
    shutil.rmtree(bdir, ignore_errors=True)
    return dst


def main() -> int:
    if not os.path.isdir(SRC):
        print("reference sources not present: nothing to build")
        return 0
    os.environ.setdefault("TORCH_CUDA_ARCH_LIST", "9.0a")
    os.makedirs(OUT, exist_ok=True)
    with ThreadPoolExecutor(3) as ex:
        for p in ex.map(build_one, EXTS):
            print("built", p)
    return 0


if __name__ == "__main__":
    sys.exit(main())
