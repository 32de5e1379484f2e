"""AOT-compile the REFERENCE's Triton kernels for sm_90 into oracle/_ref/ (cubins + one JSON index).

The kernels are the reference's own ``@triton.jit`` functions, imported from /root/reference where they lie
(nothing is copied into the repo) and compiled with the Triton that ships in this image -- no GPU needed:

  fp4_fake_quant_kernel                    kernels/quantization/gemm/fp4_kernel_hopper.py:33   (NVFP4 dynamic)
  static_blockwise_fp4_fake_quant_kernel   kernels/quantization/gemm/fp4_kernel.py:194        (NVFP4 static)
  _fp8_scale_sweep_kernel                  kernels/quantization/gemm/nvfp4_fp8_sweep.py:58    (126-candidate sweep)

with the launch constants their Python wrappers use by default (tile 16 x 64, block 16, 4 warps; the sweep's
BLOCKS_PER_PROGRAM=64 / 8 warps configuration).  The cubins travel to the GPU box with the snapshot, where
tests/test_gpu_vs_reference_triton.py launches them through the CUDA driver API next to this engine's kernels.
Test infrastructure only.  Usage: python oracle/build_ref_triton.py
"""

from __future__ import annotations

import importlib
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "_ref")
sys.path.insert(0, HERE)


def main() -> int:
    if not os.path.isdir("/root/reference/modelopt"):
        print("reference sources not present: nothing to build")
        return 0
    srcs = [f"/root/reference/modelopt/torch/kernels/quantization/{f}" for f in
            ("gemm/fp4_kernel_hopper.py", "gemm/fp4_kernel.py", "gemm/nvfp4_fp8_sweep.py", "common/nvfp4_quant.py")]
    idx_path = os.path.join(OUT, "triton_kernels.json")
    if os.path.exists(idx_path) and all(os.path.getmtime(idx_path) >= os.path.getmtime(f) for f in srcs + [__file__]):
        print("up to date:", idx_path)
        return 0
    import gen_golden

    gen_golden._install_shim()
    import triton
    import triton.language as tl
    from triton.backends.compiler import GPUTarget
    from triton.compiler import ASTSource

    base = "modelopt.torch.kernels.quantization.gemm."
    hopper = importlib.import_module(base + "fp4_kernel_hopper")
    fp4 = importlib.import_module(base + "fp4_kernel")
    sweep = importlib.import_module(base + "nvfp4_fp8_sweep")
    target = GPUTarget("cuda", 90, 32)
    tdt = {"bf16": tl.bfloat16, "f16": tl.float16, "f32": tl.float32}
    ptr = {"bf16": "*bf16", "f16": "*fp16", "f32": "*fp32"}
    index = {"triton": triton.__version__, "kernels": {}}
    os.makedirs(OUT, exist_ok=True)

    def emit(key, fn, signature, constexprs, num_warps):
        if type(fn).__name__ == "Autotuner":             # unwrap @triton.autotune -> the JITFunction
            fn = fn.fn
        sig = dict(signature)
        sig.update({k: "constexpr" for k in constexprs})
        k = triton.compile(ASTSource(fn, sig, constexprs), target=target, options={"num_warps": num_warps})
        path = os.path.join(OUT, f"triton_{key}.cubin")
        with open(path, "wb") as f:
            f.write(k.asm["cubin"])
        n_entry = k.asm["ptx"].split(".entry")[1].split(")")[0].count(".param")
        index["kernels"][key] = {
            "file": os.path.basename(path), "name": k.metadata.name, "shared": int(k.metadata.shared),
            "num_warps": int(k.metadata.num_warps), "args": [a for a in signature],
            "arg_types": [signature[a] for a in signature], "n_params": n_entry,
            "constexprs": {a: str(v) for a, v in constexprs.items()},
            "fp32_division": sorted({t for t in k.asm["ptx"].split() if t.startswith("div.") and "f32" in t}),
        }

    for d in tdt:
        emit(f"fp4_fake_quant_{d}", hopper.fp4_fake_quant_kernel,
             {"x_ptr": ptr[d], "y_ptr": ptr[d], "M": "i32", "N": "i32", "global_scale_ptr": "*fp32",
              "stride_xm": "i32", "stride_xn": "i32", "stride_ym": "i32", "stride_yn": "i32"},
             {"BLOCK_SIZE": 16, "TILE_M": 16, "TILE_N": 64, "NUM_FP4_BLOCKS": 4, "OUT_DTYPE": tdt[d]}, 4)
        emit(f"fp4_static_{d}", fp4.static_blockwise_fp4_fake_quant_kernel,
             {"x_ptr": ptr[d], "y_ptr": ptr[d], "scale_ptr": "*fp32", "NUM_FP4_BLOCKS": "i32"},
             {"BLOCK_SIZE": 16, "OUT_DTYPE": tdt[d]}, 4)
        emit(f"fp8_sweep_{d}", sweep._fp8_scale_sweep_kernel,
             {"x_ptr": ptr[d], "candidates_ptr": "*fp32", "global_amax_ptr": "*fp32", "best_amax_ptr": "*fp32",
              "N_BLOCKS": "i32"},
             {"BLOCK_SIZE": 16, "NUM_CANDIDATES": 126, "BLOCKS_PER_PROGRAM": 64}, 8)
    with open(os.path.join(OUT, "triton_kernels.json"), "w") as f:
        json.dump(index, f, indent=1)
    print("wrote", len(index["kernels"]), "cubins +", os.path.join(OUT, "triton_kernels.json"))
    return 0


if __name__ == "__main__":
    sys.exit(main())
